"""TEST INFRASTRUCTURE ONLY.

oracle/ holds the checkers for the MTTKRP / CPD-ALS hot path:
  * oracle/_ref/      the UNMODIFIED reference, compiled from the reference sources by
                      oracle/build_ref.sh (+ ref_driver.c, a flat ctypes facade).
                      `oracle.ref` wraps it.
  * oracle/restate.c  a plain-C restatement of the reference's algorithms for this
                      path (each function cites the reference lines it follows),
                      pinned against _ref and the committed golden vectors.
                      `oracle.restate` wraps it.
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this package.  The product (splatt_b200/) never does.
"""
