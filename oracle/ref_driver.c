/*
 * ref_driver.c -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * A flat, ctypes-friendly C interface over the UNMODIFIED reference library
 * (oracle/_ref/libsplatt_ref.so, built from the reference sources by build_ref.sh).
 * Compiled against the reference's own headers, so every struct and call here
 * is the reference's; this file contributes no arithmetic of its own.
 *
 * Used by tests/ (parity oracle), tests/golden/make_golden.py (golden vectors),
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
 */
#include "base.h"
#include "sptensor.h"
#include "csf.h"
#include "mttkrp.h"
#include "matrix.h"
#include "thd_info.h"
#include "cpd.h"
#include "io.h"
#include "timer.h"
#include "thread_partition.h"
#include <omp.h>
#include <stddef.h>

/* ---- tensors ------------------------------------------------------------ */

sptensor_t * refdrv_tt_from_coo(uint64_t nmodes, uint64_t const * dims, uint64_t nnz,
                                uint64_t const * const * ind, double const * vals)
{
  sptensor_t * tt = tt_alloc(nnz, nmodes);
  for(idx_t m=0; m < nmodes; ++m) {
    tt->dims[m] = dims[m];
    memcpy(tt->ind[m], ind[m], nnz * sizeof(idx_t));
  }
  memcpy(tt->vals, vals, nnz * sizeof(val_t));
  return tt;
}

sptensor_t * refdrv_tt_read(char const * fname) { return tt_read(fname); }
void refdrv_tt_free(sptensor_t * tt) { tt_free(tt); }
uint64_t refdrv_tt_nmodes(sptensor_t const * tt) { return tt->nmodes; }
uint64_t refdrv_tt_nnz(sptensor_t const * tt) { return tt->nnz; }
void refdrv_tt_dims(sptensor_t const * tt, uint64_t * dims)
{
  for(idx_t m=0; m < tt->nmodes; ++m) dims[m] = tt->dims[m];
}
void refdrv_tt_copy_out(sptensor_t const * tt, uint64_t ** ind, double * vals)
{
  for(idx_t m=0; m < tt->nmodes; ++m) memcpy(ind[m], tt->ind[m], tt->nnz * sizeof(idx_t));
  memcpy(vals, tt->vals, tt->nnz * sizeof(val_t));
}
uint64_t refdrv_tt_remove_empty(sptensor_t * tt) { return tt_remove_empty(tt); }

/* ---- options ------------------------------------------------------------ */

double * refdrv_default_opts(void) { return splatt_default_opts(); }
void refdrv_free_opts(double * o) { splatt_free_opts(o); }

/* ---- CSF ---------------------------------------------------------------- */

/* NOTE: sorts tt in place (reference behaviour, src/csf.c:475). */
splatt_csf * refdrv_csf_alloc(sptensor_t * tt, double const * opts) { return csf_alloc(tt, opts); }
void refdrv_csf_free(splatt_csf * csf, double const * opts) { csf_free(csf, opts); }

void refdrv_mode_order(uint64_t const * dims, uint64_t nmodes, int which, uint64_t mode,
                       uint64_t * perm)
{
  csf_find_mode_order(dims, nmodes, (csf_mode_type) which, mode, perm);
}

uint64_t * refdrv_partition_weighted(uint64_t const * weights, uint64_t nitems, uint64_t nparts,
                                     uint64_t * bneck)
{
  return partition_weighted(weights, nitems, nparts, bneck);
}
void refdrv_free(void * p) { free(p); }

/* ---- MTTKRP -------------------------------------------------------------- */

static void p_wrap(matrix_t * store, matrix_t ** mats, uint64_t nmodes, uint64_t const * dims,
                   uint64_t R, double ** vals, uint64_t mode, double * out)
{
  for(idx_t m=0; m < nmodes; ++m) {
    store[m].I = dims[m]; store[m].J = R; store[m].rowmajor = 1; store[m].vals = vals[m];
    mats[m] = &store[m];
  }
  store[MAX_NMODES].I = dims[mode]; store[MAX_NMODES].J = R;
  store[MAX_NMODES].rowmajor = 1;   store[MAX_NMODES].vals = out;
  mats[MAX_NMODES] = &store[MAX_NMODES];
}

/* The reference's gold (tests/mttkrp_test.c:66): COO streaming MTTKRP. */
void refdrv_mttkrp_stream(sptensor_t const * tt, uint64_t R, double ** mats_vals, uint64_t mode,
                          double * out, int nthreads)
{
  matrix_t store[MAX_NMODES+1];
  matrix_t * mats[MAX_NMODES+1];
  p_wrap(store, mats, tt->nmodes, tt->dims, R, mats_vals, mode, out);
  omp_set_num_threads(nthreads);
  mttkrp_stream(tt, mats, mode);
}

/* The reference's production path: mttkrp_csf with ws and thds allocated once
 * (pattern of src/cpd.c:285-304).  Runs `warm` untimed + `iters` timed calls,
 * returns per-call seconds in times[] (clock_gettime MONOTONIC, the clock of
 * src/timer.h:137-139). */
void refdrv_mttkrp_csf(splatt_csf const * csf, double const * opts, uint64_t R, double ** mats_vals,
                       uint64_t mode, double * out, int warm, int iters, double * times)
{
  idx_t const nmodes = csf->nmodes;
  idx_t const nthreads = (idx_t) opts[SPLATT_OPTION_NTHREADS];
  matrix_t store[MAX_NMODES+1];
  matrix_t * mats[MAX_NMODES+1];
  p_wrap(store, mats, nmodes, csf->dims, R, mats_vals, mode, out);
  omp_set_num_threads(nthreads);
  thd_info * thds = thd_init(nthreads, 3,
      (nmodes * R * sizeof(val_t)) + 64, 0, (nmodes * R * sizeof(val_t)) + 64);
  splatt_mttkrp_ws * ws = splatt_mttkrp_alloc_ws(csf, R, opts);
  for(int i=0; i < warm + iters; ++i) {
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    mttkrp_csf(csf, mats, mode, thds, ws, opts);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    if(i >= warm && times != NULL) {
      times[i-warm] = (t1.tv_sec - t0.tv_sec) + 1e-9 * (t1.tv_nsec - t0.tv_nsec);
    }
  }
  splatt_mttkrp_free_ws(ws);
  thd_free(thds, nthreads);
}

/* Public API entry (include/splatt/api_kernels.h:98-104). */
int refdrv_splatt_mttkrp(uint64_t mode, uint64_t R, splatt_csf const * csf, double ** mats_vals,
                         double * out, double const * opts)
{
  return splatt_mttkrp(mode, R, csf, mats_vals, out, opts);
}

/* ---- CPD ----------------------------------------------------------------- */

/* splatt_cpd_als with srand(seed) first, as the CLI does (src/cmds/cmd_cpd.c:167).
 * Copies factors (row-major dims[m] x R) and lambda out; returns the fit. */
double refdrv_cpd_als(splatt_csf const * csf, uint64_t R, double const * opts, unsigned seed,
                      double ** factors_out, double * lambda_out)
{
  splatt_kruskal k;
  srand(seed);
  init_timers();
  splatt_cpd_als(csf, R, opts, &k);
  for(idx_t m=0; m < k.nmodes; ++m) {
    if(factors_out != NULL && factors_out[m] != NULL) {
      memcpy(factors_out[m], k.factors[m], k.dims[m] * R * sizeof(val_t));
    }
  }
  if(lambda_out != NULL) memcpy(lambda_out, k.lambda, R * sizeof(val_t));
  double const fit = k.fit;
  splatt_free_kruskal(&k);
  return fit;
}

/* ---- ABI facts for tests/test_abi.py ---------------------------------------- */

#define PUT(x) out[n++] = (uint64_t)(x)
uint64_t refdrv_abi(uint64_t * out)
{
  uint64_t n = 0;
  PUT(sizeof(splatt_idx_t)); PUT(sizeof(splatt_val_t)); PUT(SPLATT_MAX_NMODES);
  PUT(sizeof(csf_sparsity));
  PUT(offsetof(csf_sparsity, nfibs)); PUT(offsetof(csf_sparsity, fptr));
  PUT(offsetof(csf_sparsity, fids));  PUT(offsetof(csf_sparsity, vals));
  PUT(sizeof(splatt_csf));
  PUT(offsetof(splatt_csf, nnz)); PUT(offsetof(splatt_csf, nmodes)); PUT(offsetof(splatt_csf, dims));
  PUT(offsetof(splatt_csf, dim_perm)); PUT(offsetof(splatt_csf, dim_iperm));
  PUT(offsetof(splatt_csf, which_tile)); PUT(offsetof(splatt_csf, ntiles));
  PUT(offsetof(splatt_csf, ntiled_modes)); PUT(offsetof(splatt_csf, tile_dims));
  PUT(offsetof(splatt_csf, pt));
  PUT(sizeof(splatt_kruskal));
  PUT(offsetof(splatt_kruskal, rank)); PUT(offsetof(splatt_kruskal, factors));
  PUT(offsetof(splatt_kruskal, lambda)); PUT(offsetof(splatt_kruskal, nmodes));
  PUT(offsetof(splatt_kruskal, dims)); PUT(offsetof(splatt_kruskal, fit));
  PUT(sizeof(splatt_mttkrp_ws));
  PUT(offsetof(splatt_mttkrp_ws, num_csf)); PUT(offsetof(splatt_mttkrp_ws, mode_csf_map));
  PUT(offsetof(splatt_mttkrp_ws, num_threads)); PUT(offsetof(splatt_mttkrp_ws, tile_partition));
  PUT(offsetof(splatt_mttkrp_ws, tree_partition)); PUT(offsetof(splatt_mttkrp_ws, is_privatized));
  PUT(offsetof(splatt_mttkrp_ws, privatize_buffer)); PUT(offsetof(splatt_mttkrp_ws, reduction_time));
  PUT(sizeof(matrix_t));
  PUT(offsetof(matrix_t, I)); PUT(offsetof(matrix_t, J)); PUT(offsetof(matrix_t, vals));
  PUT(offsetof(matrix_t, rowmajor));
  PUT(SPLATT_SUCCESS); PUT(SPLATT_ERROR_BADINPUT); PUT(SPLATT_ERROR_NOMEMORY);
  PUT(SPLATT_OPTION_NTHREADS); PUT(SPLATT_OPTION_TOLERANCE); PUT(SPLATT_OPTION_REGULARIZE);
  PUT(SPLATT_OPTION_NITER); PUT(SPLATT_OPTION_VERBOSITY); PUT(SPLATT_OPTION_RANDSEED);
  PUT(SPLATT_OPTION_CSF_ALLOC); PUT(SPLATT_OPTION_TILE); PUT(SPLATT_OPTION_TILELEVEL);
  PUT(SPLATT_OPTION_PRIVTHRESH); PUT(SPLATT_OPTION_DECOMP); PUT(SPLATT_OPTION_COMM);
  PUT(SPLATT_OPTION_NOPTIONS);
  return n;
}
