// The per-record walk of a root stream that completion (tc.cu), Poisson CP (apr.cu) and Tucker
// (tucker.cu) share: one warp per nnz-balanced chunk range of the root MTTKRP, a private TMA
// record ring, and for completion and CP-APR the Hadamard prefix of the inner levels in registers.
// Also the model-sum kernel body (the SSE of completion, the log-likelihood of CP-APR) and the
// host helpers the drivers use.
#pragma once
#include "mttkrp_kernels.cuh"
#include <algorithm>
#include <type_traits>

namespace spb200 {
namespace {

constexpr uint32_t kEmptySlot = 0xffffffffu;

struct TcArgs {
  const SpRec *      rec;
  const uint32_t *   up[SPB200_MAXN - 2];
  const uint32_t *   desc;
  const double *     mats[SPB200_MAXN];   // by LEVEL (level 0 unused by the row update; CP-APR: B)
  unsigned long long nrec;
  unsigned int       nchunks;
  int                ldm, R;
  double             reg;
  double *           out;        // row update: U_m; rows with a solve are stored here (CP-APR: Phi)
  double *           packs;      // boundary slots [2 * warps][P], or per-row packs [dims][P]
  uint32_t *         slot_row;   // row of every boundary slot (kEmptySlot: unused)
  const double *     lambda;     // SSE / log-likelihood: RP weights
  double *           sse;        // SSE / log-likelihood: one double, accumulated into
  double             eps;        // CP-APR: floor of the model value in a division or a log
};

__host__ __device__ constexpr size_t tc_ring_bytes() { return smem_bytes(kStages, false, 1, 0, 0); }

// The upper triangle of an R x R matrix as "pair rows" (completion's row update, CP-APR's PDNR
// Hessian): row i holds the column pairs (2q, 2q+1) for q = i/2 .. H - 1 (H = RP / 2, RP = R
// rounded up to even), so every update is one double2 FMA; tc_pairs(H) pairs in all.
__host__ __device__ constexpr int tc_pairs(int H) { return H * (H + 1); }
// pairs stored before pair row i (H = RP / 2): sum over i' < i of (H - i'/2)
__device__ __forceinline__ int pair_base(int i, int H) {
  const int q = i >> 1;
  return i * H - ((i & 1) ? q * q : q * (q - 1));
}

// Walks this warp's range of the stream (the MTTKRP kernel's nnz-balanced chunk ranges with one
// lane group per warp) through a private TMA ring of kStages x kStageRecs records.  Lane l holds
// columns 2l, 2l + 1.  For every record f(v, h, close, row, last) is called by the whole warp:
// h = the product of the rows of levels L0 .. N-1 (L0 = 1: the row update's h_x; L0 = 0: the
// model's term), close = the record ends its root slice (always at the range's last record),
// row = the root index (valid when close, and with OPEN also at the record that opens a slice,
// i.e. the range's first record and every record after a close), last = the range's last record.
template <int N, int L0, bool OPEN = false, class F>
__device__ __forceinline__ void walk_range(const TcArgs & a, unsigned char * smem, bool act, F && f) {
  constexpr int SU   = kStageRecs;
  const int     warp = threadIdx.x >> 5;
  const int     lane = threadIdx.x & 31;
  SpRec *    ring = reinterpret_cast<SpRec *>(smem) + warp * kStages * SU;
  uint64_t * bars = reinterpret_cast<uint64_t *>(smem + smem_rec_bytes(kStages, 1, 0)) + warp * kStages;
  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < kStages; ++s) mbar_init(&bars[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncwarp();

  const unsigned long long TG = static_cast<unsigned long long>(gridDim.x) * kWarps;
  const unsigned long long gg = static_cast<unsigned long long>(blockIdx.x) * kWarps + warp;
  const unsigned long long cb = gg * a.nchunks / TG;
  const unsigned long long ce = (gg + 1) * a.nchunks / TG;
  const unsigned long long rb = cb * SPB200_CHUNK;
  unsigned long long       re = ce * SPB200_CHUNK;
  if (re > a.nrec) re = a.nrec;
  const uint32_t T     = (re > rb) ? static_cast<uint32_t>(re - rb) : 0u;
  const uint32_t steps = (T + SU - 1) / SU;

  auto issue = [&](uint32_t step) {
    if (lane != 0) return;
    uint64_t *     bar = &bars[step % kStages];
    const uint32_t off = step * SU;
    const uint32_t cnt = min(static_cast<uint32_t>(SU), T - off);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    mbar_arrive_expect_tx(bar, cnt * 16u);
    tma_bulk_g2s(&ring[(step % kStages) * SU], a.rec + rb + off, cnt * 16u, bar);
  };

  const uint32_t pitch = static_cast<uint32_t>(a.ldm) * 8u;
  const char *   mbase[N];
#pragma unroll
  for (int l = 0; l < N; ++l) mbase[l] = reinterpret_cast<const char *>(a.mats[l] + (act ? 2 * lane : 0));
  constexpr int NP = (N > 2) ? N - 2 : 1;
  double2       pre[N - 1];
  uint32_t      pos[NP];
#pragma unroll
  for (int l = 0; l < N - 1; ++l) pre[l] = make_double2(0.0, 0.0);
#pragma unroll
  for (int l = 0; l < NP; ++l) pos[l] = 0u;
#pragma unroll
  for (int l = 0; l < N - 2; ++l) pos[l] = T ? a.desc[cb * (N - 2) + l] : 0u;
  uint32_t pc = N - 1;

#pragma unroll
  for (int s = 0; s < kStages; ++s)
    if (s < static_cast<int>(steps)) issue(s);

  for (uint32_t step = 0; step < steps; ++step) {
    while (!mbar_try_wait(&bars[step % kStages], (step / kStages) & 1u)) {}
    const uint32_t off = step * SU;
    const uint32_t cnt = min(static_cast<uint32_t>(SU), T - off);
    SpRec *        buf = &ring[(step % kStages) * SU];
    // the last record of the range closes every level (range boundary)
    if (lane == 0 && off + cnt == T)
      buf[cnt - 1].aux = (buf[cnt - 1].aux & SPB200_IDX_MASK) | (uint32_t(N - 1) << SPB200_IDX_BITS);
    __syncwarp();
    for (uint32_t n = 0; n < cnt; ++n) {
      const uint4    q   = *reinterpret_cast<const uint4 *>(&buf[n]);
      const double   v   = rec_val<double>(q);
      const uint32_t c   = q.w >> SPB200_IDX_BITS;
      const uint32_t par = q.w & SPB200_IDX_MASK;
      double2        h   = make_double2(0.0, 0.0);
      if (act) {
        // (re)open the prefix levels that changed after the previous record
        if (pc) {
#pragma unroll
          for (int l = L0; l <= N - 2; ++l) {
            if (l + int(pc) >= N - 1) {
              const uint32_t idx = (l == N - 2) ? par : __ldg(&a.up[l][pos[l]]);
              const double2  row = ld_row<double2>(mbase[l], idx, pitch);
              pre[l]             = (l == L0) ? row : vmul(pre[l - 1], row);
            }
          }
        }
        const double2 b = ld_row<double2>(mbase[N - 1], q.z, pitch);
        h = (L0 <= N - 2) ? vmul(pre[N - 2], b) : b;
      }
      const bool close = c >= uint32_t(N - 1);
      uint32_t   row   = 0;
      if (close || (OPEN && pc == uint32_t(N - 1))) {
        if constexpr (N == 2) row = par;
        else row = __ldg(&a.up[0][pos[0]]);
      }
      f(v, h, close, row, off + n + 1 == T);
      if (c) {
#pragma unroll
        for (int l = 0; l <= N - 3; ++l)
          if (c >= uint32_t(N - 1 - l)) ++pos[l];
      }
      pc = c;
    }
    __syncwarp();
    if (step + kStages < steps) issue(step + kStages);
  }
}

// The same walk without the Hadamard prefix, for kernels that need the level structure itself
// (Tucker's TTMc forms a Kronecker product of the levels' rows).  For every record
// g(q, pc, pos, close, row, last) is called by the whole warp: q = the record, pc = the previous
// record's close count (levels N-1-pc .. N-2 have a new node at this record; pc = N-1 at the
// range's first record), pos[l] = the node number of level l = 0 .. N-3 (its index is
// up[l][pos[l]]; level N-2's is the record's parent field), close / row / last as in walk_range
// (row valid when close).  walk_range keeps its own copy of this loop: rebasing it on walk_levels
// reschedules the SASS of the completion and CP-APR kernels.
template <int N, class G>
__device__ __forceinline__ void walk_levels(const TcArgs & a, unsigned char * smem, G && g) {
  constexpr int SU   = kStageRecs;
  const int     warp = threadIdx.x >> 5;
  const int     lane = threadIdx.x & 31;
  SpRec *    ring = reinterpret_cast<SpRec *>(smem) + warp * kStages * SU;
  uint64_t * bars = reinterpret_cast<uint64_t *>(smem + smem_rec_bytes(kStages, 1, 0)) + warp * kStages;
  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < kStages; ++s) mbar_init(&bars[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncwarp();

  const unsigned long long TG = static_cast<unsigned long long>(gridDim.x) * kWarps;
  const unsigned long long gg = static_cast<unsigned long long>(blockIdx.x) * kWarps + warp;
  const unsigned long long cb = gg * a.nchunks / TG;
  const unsigned long long ce = (gg + 1) * a.nchunks / TG;
  const unsigned long long rb = cb * SPB200_CHUNK;
  unsigned long long       re = ce * SPB200_CHUNK;
  if (re > a.nrec) re = a.nrec;
  const uint32_t T     = (re > rb) ? static_cast<uint32_t>(re - rb) : 0u;
  const uint32_t steps = (T + SU - 1) / SU;

  auto issue = [&](uint32_t step) {
    if (lane != 0) return;
    uint64_t *     bar = &bars[step % kStages];
    const uint32_t off = step * SU;
    const uint32_t cnt = min(static_cast<uint32_t>(SU), T - off);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    mbar_arrive_expect_tx(bar, cnt * 16u);
    tma_bulk_g2s(&ring[(step % kStages) * SU], a.rec + rb + off, cnt * 16u, bar);
  };

  constexpr int NP = (N > 2) ? N - 2 : 1;
  uint32_t      pos[NP];
#pragma unroll
  for (int l = 0; l < NP; ++l) pos[l] = 0u;
#pragma unroll
  for (int l = 0; l < N - 2; ++l) pos[l] = T ? a.desc[cb * (N - 2) + l] : 0u;
  uint32_t pc = N - 1;

#pragma unroll
  for (int s = 0; s < kStages; ++s)
    if (s < static_cast<int>(steps)) issue(s);

  for (uint32_t step = 0; step < steps; ++step) {
    while (!mbar_try_wait(&bars[step % kStages], (step / kStages) & 1u)) {}
    const uint32_t off = step * SU;
    const uint32_t cnt = min(static_cast<uint32_t>(SU), T - off);
    SpRec *        buf = &ring[(step % kStages) * SU];
    if (lane == 0 && off + cnt == T)
      buf[cnt - 1].aux = (buf[cnt - 1].aux & SPB200_IDX_MASK) | (uint32_t(N - 1) << SPB200_IDX_BITS);
    __syncwarp();
    for (uint32_t n = 0; n < cnt; ++n) {
      const uint4    q     = *reinterpret_cast<const uint4 *>(&buf[n]);
      const uint32_t c     = q.w >> SPB200_IDX_BITS;
      const bool     close = c >= uint32_t(N - 1);
      uint32_t       row   = 0;
      if (close) {
        if constexpr (N == 2) row = q.w & SPB200_IDX_MASK;
        else row = __ldg(&a.up[0][pos[0]]);
      }
      g(q, pc, pos, close, row, off + n + 1 == T);
      if (c) {
#pragma unroll
        for (int l = 0; l <= N - 3; ++l)
          if (c >= uint32_t(N - 1 - l)) ++pos[l];
      }
      pc = c;
    }
    __syncwarp();
    if (step + kStages < steps) issue(step + kStages);
  }
}

// Body of the model-sum kernels: over this grid's ranges of the stream, s = acc(s, v, x) per
// record with x = sum_r lambda_r prod_m U_m[i_m, r] (a warp sum), then one atomic per CTA into
// *a.sse.  acc is the per-record term: (v - x)^2 for the SSE, v log(max(x, eps)) for CP-APR.
template <int N, class Acc>
__device__ __forceinline__ void model_sum(const TcArgs & a, Acc && acc) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ double part[kWarps];
  const int  lane = threadIdx.x & 31;
  const bool act  = 2 * lane < a.R;
  const bool hasy = 2 * lane + 1 < a.R;
  const double2 lam = act ? reinterpret_cast<const double2 *>(a.lambda)[lane] : make_double2(0.0, 0.0);
  double sum = 0.0;
  walk_range<N, 0>(a, smem, act, [&](double v, double2 h, bool, uint32_t, bool) {
    double x = act ? h.x * lam.x : 0.0;
    if (hasy) x = fma(h.y, lam.y, x);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    sum = acc(sum, v, x);
  });
  if (lane == 0) part[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += part[w];
    atomicAdd(a.sse, s);
  }
}

// ---- host side ---------------------------------------------------------------------------------

int num_sms() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
    return 132;
  return n;
}

// Calls f(std::integral_constant<int, N>{}) for the runtime mode count N in 2..SPB200_MAXN: the
// walker kernels are instantiated per mode count.
template <class F>
auto with_nmodes(int N, F && f) {
  switch (N) {
    case 2: return f(std::integral_constant<int, 2>{});
    case 3: return f(std::integral_constant<int, 3>{});
    case 4: return f(std::integral_constant<int, 4>{});
    case 5: return f(std::integral_constant<int, 5>{});
    case 6: return f(std::integral_constant<int, 6>{});
    case 7: return f(std::integral_constant<int, 7>{});
    default: return f(std::integral_constant<int, 8>{});
  }
}

// The compile-time rank tier of the pair-row kernels: R padded to 16, 32 or 64.
int rank_tier(int R) { return R <= 16 ? 16 : (R <= 32 ? 32 : 64); }

// Sets kernel k's dynamic shared memory to smem bytes and returns the grid of every CTA that can
// be resident at that size, or 0 when k cannot run with it.
template <class Args>
int resident_grid(void (*k)(Args), size_t smem) {
  int nb = 0;
  if (cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k, kThreads, smem) != cudaSuccess || nb < 1)
    return 0;
  return nb * num_sms();
}

// Grid of a kernel that combines boundary slots or solves rows: one warp per item, at most 8 CTAs
// per SM.
unsigned combine_grid(unsigned long long nitems) {
  return (unsigned)std::min<unsigned long long>((nitems + kWarps - 1) / kWarps, (unsigned long long)num_sms() * 8);
}

// One mode's walker launch on its resident grid.  On an untiled stream (rows false) every warp
// stores the first and the last slice of its range into its two boundary slots, and a combine
// (or solve) kernel adds each row's slots; a leaf-tiled stream adds every piece into its row with
// red.add and uses none.
template <class Args>
struct WalkLaunch {
  void (*k)(Args) = nullptr;
  size_t smem = 0;
  int    grid = 0;
  bool   rows = false;
  unsigned long long nslots = 0;

  bool configure(void (*kernel)(Args), size_t smem_bytes, bool leaf_tiled) {
    k      = kernel;
    smem   = smem_bytes;
    rows   = leaf_tiled;
    grid   = resident_grid(k, smem);
    nslots = rows ? 0 : 2ull * grid * kWarps;
    return grid > 0;
  }
  // Marks every boundary slot empty (slot_row: nslots entries), then launches k(a).
  cudaError_t launch(const Args & a, uint32_t * slot_row, cudaStream_t s) const {
    const cudaError_t e = nslots ? cudaMemsetAsync(slot_row, 0xff, nslots * sizeof(uint32_t), s) : cudaSuccess;
    if (e != cudaSuccess) return e;
    k<<<grid, kThreads, smem, s>>>(a);
    spb200_count_launches(1);
    return cudaGetLastError();
  }
};

// The largest slot count of a run's launches: one slot buffer serves every mode.
template <class Launch>
unsigned long long max_slots(const Launch * ml, int N) {
  unsigned long long n = 0;
  for (int m = 0; m < N; ++m) n = std::max(n, ml[m].nslots);
  return n;
}

// Grid of the elementwise kernels over rows x R entries.
unsigned elementwise_grid(uint64_t rows, int R) {
  return (unsigned)std::max<uint64_t>(std::min<uint64_t>((rows * R + kThreads - 1) / kThreads, 1184), 1);
}

// The walker arguments of one stream: its records and levels, the factors by level
// (mats_by_mode[perm[l]]), ldm and R.
TcArgs walk_args(const FiberStream & fs, const double * const * mats_by_mode, int ldm, int R) {
  const int N = fs.nmodes;
  TcArgs a = {};
  a.rec = fs.rec;
  for (int l = 0; l < SPB200_MAXN - 2; ++l) a.up[l] = (l <= N - 3) ? fs.up[l] : nullptr;
  a.desc    = fs.desc;
  a.nrec    = fs.nrec;
  a.nchunks = static_cast<unsigned int>(fs.nchunks);
  for (int l = 0; l < N; ++l) a.mats[l] = mats_by_mode[fs.perm[l]];
  a.ldm = ldm;
  a.R   = R;
  return a;
}

// Launches a model-sum kernel (k(a) over the stream's records, the ring in dynamic shared memory)
// on every resident CTA.
cudaError_t launch_model_sum(void (*k)(TcArgs), const TcArgs & a, cudaStream_t s) {
  const size_t smem = tc_ring_bytes();
  const int grid = resident_grid(k, smem);
  if (grid < 1) return cudaErrorInvalidConfiguration;
  k<<<grid, kThreads, smem, s>>>(a);
  spb200_count_launches(1);
  return cudaGetLastError();
}

bool factors_ok(int N, int R, int ldm, const void * const * d_factors) {
  if (!d_factors || R < 1 || R > 64 || (ldm & 1) || ldm < R) return false;
  for (int m = 0; m < N; ++m)
    if (!d_factors[m] || reinterpret_cast<uintptr_t>(d_factors[m]) % 16 != 0) return false;
  return true;
}

bool stream_fits(const FiberStream & fs) { return fs.nchunks <= 0xffffffffull; }

// A whole ALLROOT tensor with 2..MAXN modes whose every mode m has a root stream with m at its
// root that the walkers can index.
bool root_streams_ok(const splatt_b200_tensor * t) {
  if (!t || t->nmodes < 2 || t->nmodes > SPB200_MAXN || t->shard_count > 1 ||
      t->layout != SPLATT_B200_LAYOUT_ALLROOT || t->streams.empty())
    return false;
  for (int m = 0; m < t->nmodes; ++m) {
    const ModePlan & p = t->plan[m];
    if (p.stream < 0 || p.stream >= (int)t->streams.size() || p.kind != SPB200_KIND_ROOT ||
        t->streams[p.stream].perm[0] != m || !stream_fits(t->streams[p.stream]))
      return false;
  }
  return true;
}

}  // namespace
}  // namespace spb200
