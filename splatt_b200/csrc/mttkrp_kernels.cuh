// sm_90a MTTKRP kernels over fiber streams (see common.h for the layout).
//
// Replaces the reference's CPU kernels (src/mttkrp.c):
//   KIND_ROOT  p_csf_mttkrp_root3_* :390-541, p_csf_mttkrp_root_* :668-799
//              (with p_propagate_up :324-387)
//   KIND_INTL  p_csf_mttkrp_intl3_* :544-607/:1032-1093, p_csf_mttkrp_intl_*
//              :1096-1278
//   KIND_LEAF  p_csf_mttkrp_leaf3_* :610-665/:802-855, p_csf_mttkrp_leaf_*
//              :860-1029
//
// Execution model
// ---------------
//  * A "group" of L lanes owns one record at a time; each lane carries one 128-bit
//    vector of adjacent columns (LaneVec: two fp64 or four fp32 columns), so a factor
//    row is fetched with one 128-bit load per lane (fp64: L = 16 covers R <= 32,
//    L = 32 covers R <= 64; fp32: twice that).  A warp holds 32/L independent groups.
//  * Every group walks ONE contiguous range of the stream (nnz-balanced:
//    ranges are equal record counts, not equal slice counts, so skewed slices
//    cannot unbalance the machine).  The tree is traversed by counting close
//    flags; partial sums of the levels above the output live in registers and
//    reach HBM once per finished output node with red.global.add.f64.  A
//    range boundary is handled by force-closing every level at the range's
//    last record -- MTTKRP is linear, so a split slice just produces two
//    partial rows that the reduction adds.  (These are the only atomics of
//    the root kernel: "atomics only at slice/range boundaries".)
//  * The record stream is staged through shared memory with 1-D TMA bulk
//    copies (cp.async.bulk + mbarrier complete_tx), one private 3-stage ring
//    per warp: no __syncthreads anywhere, the LSU only sees broadcast
//    LDS.128 (one per record) and the row gathers.
#pragma once
#include "common.h"

namespace spb200 {

constexpr int kThreads   = 256;
constexpr int kWarps     = kThreads / 32;
constexpr int kStageRecs = 128;   // records per warp per stage (2 KB)
constexpr int kStages    = 3;     // default ring depth (a template parameter of the kernel)

// Shared-memory layout.  Every lane group owns one region per stage.  With a stagger
// (MttkrpArgs::rpad / apad) the regions of the groups of a warp are 16 bytes further apart
// (one pad record / four pad ids per region), so that the per-group broadcast reads of one
// warp instruction (LDS.128 of G different records, LDS.32 of G different ids) fall into
// different banks; without it the regions are a multiple of 128 bytes apart and every such
// read is a G-way bank conflict (measured: 1.0 / 1.4 shared-memory wavefronts per record
// for 3 / 4 modes).  The price is a TMA destination that is only 16-byte aligned and a
// slightly larger footprint (which can cost an L1 carve-out step): measured, see DESIGN.md.
__host__ __device__ constexpr size_t smem_rec_bytes(int stages, int G, int rpad) {
  return sizeof(SpRec) * kWarps * stages * (kStageRecs + G * rpad);
}
__host__ __device__ constexpr size_t smem_bar_bytes(int stages) { return sizeof(uint64_t) * kWarps * stages; }
// N >= 4 root kernels also stage the per-record level-(N-3) ancestor ids (4 B each)
__host__ __device__ constexpr size_t smem_anc_bytes(int stages, int G, int apad) {
  return sizeof(uint32_t) * kWarps * stages * (kStageRecs + G * apad);
}
__host__ __device__ constexpr size_t smem_bytes(int stages, bool anc, int G, int rpad, int apad) {
  return smem_rec_bytes(stages, G, rpad) + smem_bar_bytes(stages) +
         (anc ? smem_anc_bytes(stages, G, apad) : 0);
}

__device__ __forceinline__ uint32_t smem_u32(const void * p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t * bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t * bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t * bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t * bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// 1-D TMA bulk copy global -> shared, completion signalled on an mbarrier.
__device__ __forceinline__ void tma_bulk_g2s(void * dst, const void * src, uint32_t bytes,
                                             uint64_t * bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// One lane's share of a factor row: 16 bytes, i.e. W columns of the value type T.
template <typename T> struct LaneVec;
template <> struct LaneVec<double> { using type = double2; static constexpr int W = 2; };
template <> struct LaneVec<float>  { using type = float4;  static constexpr int W = 4; };

// Row addressing: `base` already points at this lane's columns; the row offset
// is one 32x32->64 multiply-add (IMAD.WIDE.U32) of the index with the row pitch.
template <typename V = double2>
__device__ __forceinline__ V ld_row(const char * __restrict__ base, uint32_t idx, uint32_t pitch) {
  return __ldg(reinterpret_cast<const V *>(base + static_cast<uint64_t>(idx) * pitch));
}
// Same gather, but the line is not allocated in L1 (parent rows of a leaf-tiled stream
// are touched once per SM: keeping them out leaves L1 to the leaf tile).
template <typename V = double2>
__device__ __forceinline__ V ld_row_na(const char * __restrict__ base, uint32_t idx, uint32_t pitch);
template <>
__device__ __forceinline__ double2 ld_row_na<double2>(const char * __restrict__ base, uint32_t idx,
                                                      uint32_t pitch) {
  double2 r;
  asm("ld.global.nc.L1::no_allocate.v2.f64 {%0, %1}, [%2];"
               : "=d"(r.x), "=d"(r.y)
               : "l"(base + static_cast<uint64_t>(idx) * pitch));
  return r;
}
template <>
__device__ __forceinline__ float4 ld_row_na<float4>(const char * __restrict__ base, uint32_t idx,
                                                    uint32_t pitch) {
  float4 r;
  asm("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(base + static_cast<uint64_t>(idx) * pitch));
  return r;
}
__device__ __forceinline__ void red_row(char * __restrict__ base, uint32_t idx, uint32_t pitch,
                                        double2 x) {
  double * p = reinterpret_cast<double *>(base + static_cast<uint64_t>(idx) * pitch);
  atomicAdd(p, x.x);      // result unused -> RED.E.ADD.F64
  atomicAdd(p + 1, x.y);
}
// One vector reduction for the four columns (REDG.E.ADD.F32x4).  Like every f32 global
// reduction it flushes subnormal operands and results to (sign-preserving) zero.
__device__ __forceinline__ void red_row(char * __restrict__ base, uint32_t idx, uint32_t pitch,
                                        float4 x) {
  float * p = reinterpret_cast<float *>(base + static_cast<uint64_t>(idx) * pitch);
  asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1, %2, %3, %4};"
               ::"l"(p), "f"(x.x), "f"(x.y), "f"(x.z), "f"(x.w) : "memory");
}
// The same reduction through an NVLink MULTICAST address: one instruction adds the value
// into the row of every GPU of the group (NVSwitch fans it out).  Used by the fused
// MTTKRP + exchange path: the finished output rows never take a separate collective.
__device__ __forceinline__ void red_row_mc(char * __restrict__ base, uint32_t idx, uint32_t pitch,
                                           double2 x) {
  double * p = reinterpret_cast<double *>(base + static_cast<uint64_t>(idx) * pitch);
  asm volatile("multimem.red.relaxed.sys.global.add.f64 [%0], %1;" ::"l"(p), "d"(x.x) : "memory");
  asm volatile("multimem.red.relaxed.sys.global.add.f64 [%0], %1;" ::"l"(p + 1), "d"(x.y) : "memory");
}
// Group barrier primitive: GPU `rank` of `world` publishes `epoch` in ITS OWN slot of the
// group's flag array on every GPU (one multicast store), then waits until every slot of the
// local copy has reached `epoch`.  One slot per GPU (not an arrival count): a fast GPU's next
// arrival can never stand in for a slow GPU's current one.
__device__ __forceinline__ void group_signal_and_wait(uint32_t * mc_flags, uint32_t * local_flags,
                                                      uint32_t epoch, uint32_t rank, uint32_t world) {
  asm volatile("multimem.st.release.sys.global.u32 [%0], %1;" ::"l"(mc_flags + rank), "r"(epoch) : "memory");
  for (uint32_t r = 0; r < world; ++r) {
    unsigned int v;
    do {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(local_flags + r) : "memory");
    } while (static_cast<int>(v - epoch) < 0);
  }
}
// A finished output row that no other lane group and no other GPU contributes to (a slice
// lying wholly inside this group's record range) needs no reduction: one 128-bit store to the
// multicast address writes it into every GPU's (zeroed) buffer -- half the NVLink packets of
// two 64-bit multimem.red's and no work for the switch's reduction units.
__device__ __forceinline__ void st_row_mc(char * __restrict__ base, uint32_t idx, uint32_t pitch,
                                          double2 x) {
  double * p = reinterpret_cast<double *>(base + static_cast<uint64_t>(idx) * pitch);
  asm volatile("st.relaxed.sys.global.v2.f64 [%0], {%1, %2};" ::"l"(p), "d"(x.x), "d"(x.y) : "memory");
}
__device__ __forceinline__ double2 vfma(double s, double2 a, double2 c) {
  return make_double2(fma(s, a.x, c.x), fma(s, a.y, c.y));
}
__device__ __forceinline__ double2 vfma(double2 a, double2 b, double2 c) {
  return make_double2(fma(a.x, b.x, c.x), fma(a.y, b.y, c.y));
}
__device__ __forceinline__ double2 vmul(double2 a, double2 b) {
  return make_double2(a.x * b.x, a.y * b.y);
}
__device__ __forceinline__ double2 vmul(double s, double2 a) {
  return make_double2(s * a.x, s * a.y);
}
__device__ __forceinline__ float4 vfma(float s, float4 a, float4 c) {
  return make_float4(fmaf(s, a.x, c.x), fmaf(s, a.y, c.y), fmaf(s, a.z, c.z), fmaf(s, a.w, c.w));
}
__device__ __forceinline__ float4 vfma(float4 a, float4 b, float4 c) {
  return make_float4(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y), fmaf(a.z, b.z, c.z),
                     fmaf(a.w, b.w, c.w));
}
__device__ __forceinline__ float4 vmul(float4 a, float4 b) {
  return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w);
}
__device__ __forceinline__ float4 vmul(float s, float4 a) {
  return make_float4(s * a.x, s * a.y, s * a.z, s * a.w);
}
template <typename V> __device__ __forceinline__ V vzero();
template <> __device__ __forceinline__ double2 vzero<double2>() { return make_double2(0.0, 0.0); }
template <> __device__ __forceinline__ float4 vzero<float4>() { return make_float4(0.f, 0.f, 0.f, 0.f); }
// The record's value in the kernel's value type (fp32: rounded once, to nearest).
template <typename T> __device__ __forceinline__ T rec_val(const uint4 q) {
  return static_cast<T>(__hiloint2double(static_cast<int>(q.y), static_cast<int>(q.x)));
}

// Minimum CTAs per SM a stream kernel is compiled for unless a variant names its own.
__host__ __device__ constexpr int default_minb(int N, int BATCH) { return (BATCH >= 8 || N >= 4) ? 2 : 3; }

// One record of the root traversal (levels above the leaf fold upwards; the
// root row leaves the SM with a RED).  `b`/`r` are the gathered leaf / parent
// rows; for N >= 4 `r2` is the gathered level-(N-3) row (valid when c >= 2).
template <typename Val, int N, bool MC, typename V = typename LaneVec<Val>::type>
__device__ __forceinline__ void root_record(const MttkrpArgs & a, const uint4 q, const V b,
                                            const V r, const V r2,
                                            V (&acc)[N - 1], uint32_t (&pos)[(N > 2) ? N - 2 : 1],
                                            const char * const (&mbase)[N], char * obase,
                                            uint32_t pitch, bool & seen_root, const bool last) {
  const V        zero2 = vzero<V>();
  const Val      v     = rec_val<Val>(q);
  const uint32_t c     = q.w >> SPB200_IDX_BITS;
  acc[N - 2]           = vfma(v, b, acc[N - 2]);
  if (c) {
    acc[N - 3] = vfma(acc[N - 2], r, acc[N - 3]);
    acc[N - 2] = zero2;
    if (c >= 2) {
      if constexpr (N >= 4) {
        ++pos[N - 3];
        acc[N - 4] = vfma(acc[N - 3], r2, acc[N - 4]);
        acc[N - 3] = zero2;
#pragma unroll
        for (int l = N - 4; l >= 1; --l) {
          if (c >= uint32_t(N - 1 - l)) {
            const uint32_t idx = __ldg(&a.up[l][pos[l]]);
            ++pos[l];
            acc[l - 1] = vfma(acc[l], ld_row<V>(mbase[l], idx, pitch), acc[l - 1]);
            acc[l]     = zero2;
          }
        }
      }
      if (c >= uint32_t(N - 1)) {
        const uint32_t row = __ldg(&a.up[0][pos[0]]);
        ++pos[0];
        if constexpr (MC) {
          // the first slice a group closes may have begun before its range and the slice cut by
          // the range's end continues after it: those are partial rows (reduce); every slice in
          // between lies wholly inside the range (store)
          if (a.mc_store && seen_root && !last) st_row_mc(obase, row, pitch, acc[0]);
          else red_row_mc(obase, row, pitch, acc[0]);
        } else {
          red_row(obase, row, pitch, acc[0]);
        }
        seen_root = true;
        acc[0] = zero2;
      }
    }
  }
}

// Val: value type of the factors, the output and the arithmetic (double or float).  The
// records are the same for both: an fp32 kernel rounds each record's fp64 value once.
// MAXREG: register limit on top of the one MINB implies (the tighter applies); 255 = none.
template <typename Val, int N, int L, int KIND, int BATCH, bool KT, bool MC,
          int MINB = default_minb(N, BATCH), int STAGES = kStages, int MAXREG = 255>
__global__ void __launch_bounds__(kThreads, MINB) __maxnreg__(MAXREG)
mttkrp_stream_kernel(const MttkrpArgs a) {
  static_assert(N >= 2 && N <= SPB200_MAXN, "2..8 modes");
  static_assert(!MC || sizeof(Val) == 8, "multicast output is fp64 only");
  using V          = typename LaneVec<Val>::type;
  constexpr int W  = LaneVec<Val>::W;     // columns per lane
  constexpr int G  = 32 / L;            // groups per warp
  constexpr int SU = kStageRecs / G;    // records per group per stage
  constexpr int kStages = STAGES;       // shadows the namespace default inside the kernel
  const int RS = SU + a.rpad;           // region stride in records (rpad = 1: 16-byte stagger)
  const int AS = SU + a.apad;           // region stride in ancestor ids (apad = 4: 16-byte stagger)

  extern __shared__ __align__(128) unsigned char smem_raw[];
  SpRec *    srec = reinterpret_cast<SpRec *>(smem_raw);
  uint64_t * bars = reinterpret_cast<uint64_t *>(smem_raw + smem_rec_bytes(STAGES, G, a.rpad));
  // level-(N-3) ancestor id of every record, staged beside the records (root, N >= 4): all
  // three row gathers of a record then depend on shared memory only -- no id -> row chain
  constexpr bool kAnc = (KIND == SPB200_KIND_ROOT && N >= 4);
  uint32_t * sanc =
      reinterpret_cast<uint32_t *>(smem_raw + smem_rec_bytes(STAGES, G, a.rpad) + smem_bar_bytes(STAGES));

  const int      warp   = threadIdx.x >> 5;
  const int      lane   = threadIdx.x & 31;
  const int      grp    = lane / L;
  const int      gl     = lane % L;
  const bool     act    = (W * gl) < a.ncols;   // lanes past the last column only keep the warp in step
  const bool     leader = (gl == 0);
  const uint32_t pitch  = static_cast<uint32_t>(a.ldm) * static_cast<uint32_t>(sizeof(Val));

  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < kStages; ++s) mbar_init(&bars[warp * kStages + s], G);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncwarp();

  // This group's contiguous range of chunks / records.
  const unsigned long long TG = static_cast<unsigned long long>(gridDim.x) * kWarps * G;
  const unsigned long long gg =
      (static_cast<unsigned long long>(blockIdx.x) * kWarps + warp) * G + grp;
  const unsigned long long cb = gg * a.nchunks / TG;
  const unsigned long long ce = (gg + 1) * a.nchunks / TG;
  const unsigned long long rb = cb * SPB200_CHUNK;
  unsigned long long       re = ce * SPB200_CHUNK;
  if (re > a.nrec) re = a.nrec;
  const uint32_t T      = (re > rb) ? static_cast<uint32_t>(re - rb) : 0u;
  const uint32_t steps  = (T + SU - 1) / SU;
  const uint32_t wsteps = __reduce_max_sync(0xffffffffu, steps);

  auto issue = [&](uint32_t step) {
    if (leader) {
      const uint32_t st  = step % kStages;
      uint64_t *     bar = &bars[warp * kStages + st];
      const uint32_t off = step * SU;
      const uint32_t cnt = (off < T) ? min(static_cast<uint32_t>(SU), T - off) : 0u;
      if (cnt) {
        // generic-proxy accesses to this stage (record reads, the range-end patch) are
        // ordered before the async-proxy refill
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        if constexpr (kAnc) {
          const uint32_t ab = (cnt * 4u + 15u) & ~15u;     // the array is padded to 16 B
          mbar_arrive_expect_tx(bar, cnt * 16u + ab);
          tma_bulk_g2s(&sanc[((warp * kStages + st) * G + grp) * AS], a.anc + rb + off, ab, bar);
        } else {
          mbar_arrive_expect_tx(bar, cnt * 16u);
        }
        tma_bulk_g2s(&srec[((warp * kStages + st) * G + grp) * RS], a.rec + rb + off, cnt * 16u,
                     bar);
      } else {
        mbar_arrive(bar);
      }
    }
  };

  // Per-lane matrix bases (already offset to this lane's columns), by level.
  const int    colx = act ? (a.col0 + W * gl) : a.col0;
  const char * mbase[N];
#pragma unroll
  for (int l = 0; l < N; ++l) mbase[l] = reinterpret_cast<const char *>(static_cast<const Val *>(a.mats[l]) + colx);
  char * obase = reinterpret_cast<char *>(static_cast<Val *>(a.out) + colx);

  // Traversal state.
  const V       zero2 = vzero<V>();
  constexpr int NP = (N > 2) ? N - 2 : 1;
  V             acc[N - 1];   // partial sums of levels 0..N-2 (levels >= outdepth)
  V             pre[N - 1];   // Hadamard prefixes of levels 0..N-2 (levels < outdepth)
  uint32_t      pos[NP];      // current node at levels 0..N-3
#pragma unroll
  for (int l = 0; l < N - 1; ++l) { acc[l] = zero2; pre[l] = zero2; }
#pragma unroll
  for (int l = 0; l < NP; ++l) pos[l] = 0u;
#pragma unroll
  for (int l = 0; l < N - 2; ++l) pos[l] = T ? a.desc[cb * (N - 2) + l] : 0u;
  uint32_t  pc = N - 1;        // close count of the previous record
  bool      seen_root = false; // this group has closed a root slice already (multicast store rule)
  const int d  = a.outdepth;

#pragma unroll
  for (int s = 0; s < kStages; ++s)
    if (s < static_cast<int>(wsteps)) issue(s);

  for (uint32_t step = 0; step < wsteps; ++step) {
    const uint32_t st = step % kStages;
    while (!mbar_try_wait(&bars[warp * kStages + st], (step / kStages) & 1u)) {}

    const uint32_t off = step * SU;
    const uint32_t cnt = (off < T) ? min(static_cast<uint32_t>(SU), T - off) : 0u;
    SpRec *        buf = &srec[((warp * kStages + st) * G + grp) * RS];
    const uint32_t * abuf = &sanc[((warp * kStages + st) * G + grp) * AS];
    // The last record of the range closes every level (range boundary).
    if (leader && cnt && off + cnt == T)
      buf[cnt - 1].aux = (buf[cnt - 1].aux & SPB200_IDX_MASK) | (uint32_t(N - 1) << SPB200_IDX_BITS);
    __syncwarp();

    if (act) {
      if constexpr (N == 2) {
        // Matrices (2 modes): the record's parent IS the root row.  Root output:
        // out[root] += sum v * U_leaf[k]  (sparse x dense);  leaf output: out[k] += v * U_root[root].
        // reference: the generic kernels with nmodes == 2, src/mttkrp.c:668-732 / :860-943.
        for (uint32_t n = 0; n < cnt; ++n) {
          const uint4    q   = *reinterpret_cast<const uint4 *>(&buf[n]);
          const Val      v   = rec_val<Val>(q);
          const uint32_t par = q.w & SPB200_IDX_MASK;
          if constexpr (KIND == SPB200_KIND_ROOT) {
            acc[0] = vfma(v, ld_row<V>(mbase[1], q.z, pitch), acc[0]);
            if (q.w >> SPB200_IDX_BITS) {
              if constexpr (MC) red_row_mc(obase, par, pitch, acc[0]);
              else red_row(obase, par, pitch, acc[0]);
              acc[0] = zero2;
            }
          } else {
            const V row = ld_row<V>(mbase[0], par, pitch);
            red_row(obase, q.z, pitch, vmul(v, row));
          }
        }
      } else if constexpr (KIND == SPB200_KIND_ROOT) {
        uint32_t n0 = 0;
        // full batches: all gathers of BATCH records are in flight before the first FMA
        for (; n0 + BATCH <= cnt; n0 += BATCH) {
          uint4    q[BATCH];
          V        b[BATCH], r[BATCH], r2[BATCH];
          uint32_t hi = 0;
#pragma unroll
          for (int u = 0; u < BATCH; ++u) {
            q[u] = *reinterpret_cast<const uint4 *>(&buf[n0 + u]);
            hi   = max(hi, q[u].w);
          }
#pragma unroll
          for (int u = 0; u < BATCH; ++u) b[u] = ld_row<V>(mbase[N - 1], q[u].z, pitch);
#pragma unroll
          for (int u = 0; u < BATCH; ++u)
            if (q[u].w >> SPB200_IDX_BITS)
              r[u] = KT ? ld_row_na<V>(mbase[N - 2], q[u].w & SPB200_IDX_MASK, pitch)
                        : ld_row<V>(mbase[N - 2], q[u].w & SPB200_IDX_MASK, pitch);
          uint32_t p2 = 0;
          if constexpr (N >= 4) {
            // level N-3 closes are frequent on deep trees; the id of the closing node rides
            // beside the record, so its row gather is issued together with the other two
            p2 = pos[N - 3];
#pragma unroll
            for (int u = 0; u < BATCH; ++u)
              if ((q[u].w >> SPB200_IDX_BITS) >= 2u) {
                r2[u] = ld_row<V>(mbase[N - 3], abuf[n0 + u], pitch);
                ++p2;
              }
          }
          constexpr uint32_t kFast = (N >= 4) ? 3u : 2u;   // close counts handled branch-free
          if ((hi >> SPB200_IDX_BITS) < kFast) {
            // common case: nothing above level N-3 (N-2 for 3 modes) ends in this
            // batch -- straight-line, predicated, no branches
#pragma unroll
            for (int u = 0; u < BATCH; ++u) {
              const Val      v = rec_val<Val>(q[u]);
              const uint32_t c = q[u].w >> SPB200_IDX_BITS;
              acc[N - 2]       = vfma(v, b[u], acc[N - 2]);
              if (c) {
                acc[N - 3] = vfma(acc[N - 2], r[u], acc[N - 3]);
                acc[N - 2] = zero2;
              }
              if constexpr (N >= 4) {
                if (c >= 2u) {
                  acc[N - 4] = vfma(acc[N - 3], r2[u], acc[N - 4]);
                  acc[N - 3] = zero2;
                }
              }
            }
            if constexpr (N >= 4) pos[N - 3] = p2;
          } else {
#pragma unroll
            for (int u = 0; u < BATCH; ++u)
              root_record<Val, N, MC>(a, q[u], b[u], r[u], r2[u], acc, pos, mbase, obase, pitch, seen_root,
                                 off + n0 + u + 1 == T);
          }
        }
        for (; n0 < cnt; ++n0) {   // tail of the range's last stage
          const uint4   q = *reinterpret_cast<const uint4 *>(&buf[n0]);
          const V       b = ld_row<V>(mbase[N - 1], q.z, pitch);
          V             r = zero2, r2 = zero2;
          if (q.w >> SPB200_IDX_BITS) r = ld_row<V>(mbase[N - 2], q.w & SPB200_IDX_MASK, pitch);
          if constexpr (N >= 4) {
            if ((q.w >> SPB200_IDX_BITS) >= 2u) r2 = ld_row<V>(mbase[N - 3], abuf[n0], pitch);
          }
          root_record<Val, N, MC>(a, q, b, r, r2, acc, pos, mbase, obase, pitch, seen_root, off + n0 + 1 == T);
        }
      } else if constexpr (KIND == SPB200_KIND_INTL) {
#pragma unroll 2
        for (uint32_t n = 0; n < cnt; ++n) {
          const uint4    q   = *reinterpret_cast<const uint4 *>(&buf[n]);
          const Val      v   = rec_val<Val>(q);
          const uint32_t c   = q.w >> SPB200_IDX_BITS;
          const uint32_t par = q.w & SPB200_IDX_MASK;
          const V        b   = ld_row<V>(mbase[N - 1], q.z, pitch);
          // (re)open prefix levels that changed after the previous record
          if (pc >= uint32_t(N - d)) {
#pragma unroll
            for (int l = 0; l <= N - 3; ++l) {
              if (l < d && l + int(pc) >= N - 1) {
                const uint32_t idx = __ldg(&a.up[l][pos[l]]);
                const V        row = ld_row<V>(mbase[l], idx, pitch);
                pre[l]             = (l == 0) ? row : vmul(pre[l - 1], row);
              }
            }
          }
          acc[N - 2] = vfma(v, b, acc[N - 2]);
          if (c) {
            // levels below the output level fold upwards
#pragma unroll
            for (int l = N - 2; l >= 2; --l) {
              if (l > d && c >= uint32_t(N - 1 - l)) {
                uint32_t idx;
                if (l == N - 2) idx = par;
                else { idx = __ldg(&a.up[l][pos[l]]); ++pos[l]; }
                acc[l - 1] = vfma(acc[l], ld_row<V>(mbase[l], idx, pitch), acc[l - 1]);
                acc[l]     = zero2;
              }
            }
            // the output level itself
#pragma unroll
            for (int l = 1; l <= N - 2; ++l) {
              if (l == d && c >= uint32_t(N - 1 - l)) {
                uint32_t idx;
                if (l == N - 2) idx = par;
                else { idx = __ldg(&a.up[l][pos[l]]); ++pos[l]; }
                red_row(obase, idx, pitch, vmul(pre[l - 1], acc[l]));
                acc[l] = zero2;
              }
            }
            // prefix levels that ended: advance to their next node
#pragma unroll
            for (int l = 0; l <= N - 3; ++l)
              if (l < d && c >= uint32_t(N - 1 - l)) ++pos[l];
          }
          pc = c;
        }
      } else {   // KIND_LEAF
#pragma unroll 2
        for (uint32_t n = 0; n < cnt; ++n) {
          const uint4    q   = *reinterpret_cast<const uint4 *>(&buf[n]);
          const Val      v   = rec_val<Val>(q);
          const uint32_t c   = q.w >> SPB200_IDX_BITS;
          const uint32_t par = q.w & SPB200_IDX_MASK;
          if (pc) {
#pragma unroll
            for (int l = 0; l <= N - 2; ++l) {
              if (l + int(pc) >= N - 1) {
                uint32_t idx;
                if (l == N - 2) idx = par;
                else idx = __ldg(&a.up[l][pos[l]]);
                const V       row = ld_row<V>(mbase[l], idx, pitch);
                pre[l]            = (l == 0) ? row : vmul(pre[l - 1], row);
              }
            }
          }
          red_row(obase, q.z, pitch, vmul(v, pre[N - 2]));
          if (c) {
#pragma unroll
            for (int l = 0; l <= N - 3; ++l)
              if (c >= uint32_t(N - 1 - l)) ++pos[l];
          }
          pc = c;
        }
      }
    }

    __syncwarp();
    if (step + kStages < wsteps) issue(step + kStages);
  }

  if constexpr (MC) {
    // Group barrier in the kernel's tail (see MttkrpArgs::sync_*).
    if (a.sync_mc != nullptr) {
      __threadfence_system();                 // this thread's multimem.red's are performed
      __syncthreads();
      if (threadIdx.x == 0) {
        const unsigned int done = atomicAdd(a.sync_cta, 1u);
        if (done == gridDim.x - 1) {          // last CTA of this GPU
          *reinterpret_cast<volatile unsigned int *>(a.sync_cta) = 0u;   // ready for the next launch
          __threadfence_system();
          group_signal_and_wait(a.sync_mc, a.sync_local, a.sync_target, a.sync_rank, a.sync_world);
        }
      }
    }
  }
}

}  // namespace spb200
