// Tensor completion by row-wise ALS on device-resident tensors (splatt_b200_tc_als_device), and
// the residual sum of squares of a Kruskal model at a tensor's nonzeros (splatt_b200_tensor_sse).
//
// Completion fits x^(i_1..i_N) = sum_r prod_m U_m[i_m, r] to the stored entries only.  Updating
// row i of U_m solves (sum_x h_x h_x^T + reg I) u = sum_x v_x h_x over the nonzeros x whose
// mode-m index is i, with h_x the Hadamard product of the other modes' rows.  On the ALLROOT
// layout every mode has a stream with that mode at its root, so the nonzeros of one output row
// are contiguous: the row-update kernel walks the same nnz-balanced chunk ranges as the root
// MTTKRP kernel (one warp per range, its own TMA record ring, mttkrp_kernels.cuh), keeps the
// Hadamard prefix of levels 1..N-2 in registers, and folds each record's h into the upper
// triangle of its row's R x R matrix and the right-hand side.
//
//   * Storage of the triangle ("pair rows"): row i holds the column pairs (2q, 2q+1) for
//     q = i/2 .. RP/2 - 1 (RP = R rounded up to even), so every update is one double2 FMA.
//     Row i of an odd i carries one unused entry (i, i-1).  NP = (RP/2)(RP/2 + 1) pairs; a row's
//     "pack" is the 2 NP entries followed by the RP right-hand-side entries.
//   * Tiers by the padded rank (compile time, as the ALS tail's 16/32/64): RT = 16 keeps the
//     lane's pairs in registers (3 per lane); RT = 32 and 64 keep the triangle in per-warp
//     shared memory (2112 doubles at R = 64).
//   * A slice that lies wholly inside the warp's range is solved where it closes: the warp adds
//     reg I, factors the matrix by Cholesky and runs the two triangular solves in shared memory,
//     then stores the row with plain stores.  The first and the last slice of a range may be
//     cut by a range boundary: their packs are stored (plain stores, no atomics) into one of the
//     range's two boundary slots, and k_tc_solve adds the slots of each such row in range order
//     and solves it.  The result is deterministic.
//   * Leaf-tiled streams (built CTA-tiled by default for config-2-like 3-mode tensors, or with
//     ktile > 0) regroup a range's records by leaf tile, so a root row closes once per tile.
//     There every closed (row, tile) piece is added with red.add.f64 into a per-row pack
//     (dims[m] packs), and k_tc_solve then solves every row of the mode.
//   * U_m is zeroed before its update and never read during it (the prefix starts at level 1),
//     so rows with no observations stay 0.
#include "mttkrp_kernels.cuh"
#include <algorithm>
#include <cmath>
#include <vector>

namespace spb200 {
namespace {

constexpr uint32_t kEmptySlot = 0xffffffffu;

struct TcArgs {
  const SpRec *      rec;
  const uint32_t *   up[SPB200_MAXN - 2];
  const uint32_t *   desc;
  const double *     mats[SPB200_MAXN];   // by LEVEL (level 0 unused by the row update)
  unsigned long long nrec;
  unsigned int       nchunks;
  int                ldm, R;
  double             reg;
  double *           out;        // row update: U_m; rows with a solve are stored here
  double *           packs;      // boundary slots [2 * warps][P], or per-row packs [dims][P]
  uint32_t *         slot_row;   // row of every boundary slot (kEmptySlot: unused)
  const double *     lambda;     // SSE: RP weights
  double *           sse;        // SSE: one double, accumulated into
};

__host__ __device__ constexpr int tc_pairs(int H) { return H * (H + 1); }
// pairs stored before pair row i (H = RP / 2): sum over i' < i of (H - i'/2)
__device__ __forceinline__ int pair_base(int i, int H) {
  const int q = i >> 1;
  return i * H - ((i & 1) ? q * q : q * (q - 1));
}
// doubles per warp of the row-update / solve workspace: the pack (2 NP + RT) and h (RT)
__host__ __device__ constexpr int tc_ws_doubles(int RT) { return 2 * tc_pairs(RT / 2) + 2 * RT; }
__host__ __device__ constexpr size_t tc_ring_bytes() { return smem_bytes(kStages, false, 1, 0, 0); }
__host__ __device__ constexpr size_t tc_tab_bytes(int RT) { return (sizeof(uint32_t) * tc_pairs(RT / 2) + 15) & ~size_t(15); }
__host__ __device__ constexpr size_t tc_update_smem(int RT) {
  return tc_ring_bytes() + tc_tab_bytes(RT) + sizeof(double) * kWarps * tc_ws_doubles(RT);
}
__host__ __device__ constexpr int tc_minb(int RT) { return RT <= 32 ? 2 : 1; }

// Walks this warp's range of the stream (the MTTKRP kernel's nnz-balanced chunk ranges with one
// lane group per warp) through a private TMA ring of kStages x kStageRecs records.  Lane l holds
// columns 2l, 2l + 1.  For every record f(v, h, close, row, last) is called by the whole warp:
// h = the product of the rows of levels L0 .. N-1 (L0 = 1: the row update's h_x; L0 = 0: the
// model's term), close = the record ends its root slice (always at the range's last record),
// row = the root index (valid when close), last = the range's last record.
template <int N, int L0, class F>
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
      if (close) {
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

// Solves (A + reg I) x = b for the pack at W (pair rows, then b at W + 2 NP) by Cholesky
// (A = U^T U, U upper, in place) and two triangular solves, one warp, and stores x[0..R) to urow.
__device__ __noinline__ void warp_solve(double * W, int R, int H, double reg, double * urow) {
  const int lane = threadIdx.x & 31;
  double *  b    = W + 2 * tc_pairs(H);
  auto A = [&](int i, int j) -> double & { return W[2 * pair_base(i, H) + j - (i & ~1)]; };
  for (int i = lane; i < R; i += 32) A(i, i) += reg;
  __syncwarp();
  for (int k = 0; k < R; ++k) {
    const double d = sqrt(A(k, k));
    __syncwarp();
    const double inv = 1.0 / d;
    for (int j = k + 1 + lane; j < R; j += 32) A(k, j) *= inv;
    if (lane == 0) A(k, k) = d;
    __syncwarp();
    for (int i = k + 1; i < R; ++i) {
      const double aki = A(k, i);
      for (int j = i + lane; j < R; j += 32) A(i, j) = fma(-aki, A(k, j), A(i, j));
    }
    __syncwarp();
  }
  for (int k = 0; k < R; ++k) {                // U^T y = b
    const double yk = b[k] / A(k, k);
    __syncwarp();
    for (int j = k + 1 + lane; j < R; j += 32) b[j] = fma(-A(k, j), yk, b[j]);
    if (lane == 0) b[k] = yk;
    __syncwarp();
  }
  for (int k = R - 1; k >= 0; --k) {           // U x = y
    const double xk = b[k] / A(k, k);
    __syncwarp();
    for (int i = lane; i < k; i += 32) b[i] = fma(-A(i, k), xk, b[i]);
    if (lane == 0) b[k] = xk;
    __syncwarp();
  }
  for (int j = lane; j < R; j += 32) urow[j] = b[j];
  __syncwarp();
}

// Row update of the root mode of one stream.  RT: padded-rank tier (16: triangle in registers,
// 32 / 64: in shared memory).  ROWS: every closed piece goes into its row's pack (leaf-tiled
// streams) instead of being solved here or put into a boundary slot.
template <int N, int RT, bool ROWS>
__global__ void __launch_bounds__(kThreads, tc_minb(RT)) k_tc_update(const TcArgs a) {
  constexpr int  HM  = RT / 2;
  constexpr int  S   = (tc_pairs(HM) + 31) / 32;   // pairs per lane
  constexpr bool REG = (RT <= 16);
  extern __shared__ __align__(128) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int RP = a.R + (a.R & 1), H = RP / 2, NPr = tc_pairs(H), P = 2 * NPr + RP;
  uint32_t * tab = reinterpret_cast<uint32_t *>(smem + tc_ring_bytes());
  double *   ws  = reinterpret_cast<double *>(smem + tc_ring_bytes() + tc_tab_bytes(RT)) +
                   warp * tc_ws_doubles(RT);
  double2 *  W2  = reinterpret_cast<double2 *>(ws);
  double *   hs  = ws + 2 * tc_pairs(HM) + RT;

  // pair p -> (row i, first column j0): i in bits 0..15, j0 / 2 in bits 16..31
  for (int i = warp; i < RP; i += kWarps)
    for (int q = lane; q < H - i / 2; q += 32) tab[pair_base(i, H) + q] = uint32_t(i) | uint32_t(i / 2 + q) << 16;
  for (int p = lane; p < P; p += 32) ws[p] = 0.0;
  __syncthreads();

  const bool act = 2 * lane < a.R;
  const bool hasy = 2 * lane + 1 < a.R;
  double2    acc[REG ? S : 1];
  uint32_t   ent[REG ? S : 1];
  if constexpr (REG) {
#pragma unroll
    for (int k = 0; k < S; ++k) {
      acc[k] = make_double2(0.0, 0.0);
      ent[k] = (k * 32 + lane < NPr) ? tab[k * 32 + lane] : 0u;
    }
  }
  double2  rhs  = make_double2(0.0, 0.0);
  bool     seen = false;   // this warp closed a slice already: later ones (but the last) are whole
  const unsigned long long gw = static_cast<unsigned long long>(blockIdx.x) * kWarps + warp;

  walk_range<N, 1>(a, smem, act, [&](double v, double2 h, bool close, uint32_t row, bool last) {
    if (act) {
      if (!hasy) h.y = 0.0;                   // column R of an odd rank never feeds the result
      rhs = vfma(v, h, rhs);
      reinterpret_cast<double2 *>(hs)[lane] = h;
    }
    __syncwarp();
#pragma unroll
    for (int k = 0; k < S; ++k) {
      const int p = k * 32 + lane;
      if (p < NPr) {
        const uint32_t e  = REG ? ent[k] : tab[p];
        const double   hi = hs[e & 0xffffu];
        const double2  hj = reinterpret_cast<const double2 *>(hs)[e >> 16];
        if constexpr (REG) acc[k] = vfma(hi, hj, acc[k]);
        else W2[p] = vfma(hi, hj, W2[p]);
      }
    }
    __syncwarp();                             // h is rewritten by the next record
    if (!close) return;
    // the pack of the closed slice into ws
    if constexpr (REG) {
#pragma unroll
      for (int k = 0; k < S; ++k) {
        if (k * 32 + lane < NPr) W2[k * 32 + lane] = acc[k];
        acc[k] = make_double2(0.0, 0.0);
      }
    }
    if (act) reinterpret_cast<double2 *>(ws + 2 * NPr)[lane] = rhs;
    rhs = make_double2(0.0, 0.0);
    __syncwarp();
    if constexpr (ROWS) {
      double * dst = a.packs + static_cast<size_t>(row) * P;
      for (int p = lane; p < P; p += 32) atomicAdd(dst + p, ws[p]);
    } else if (!seen || last) {
      const unsigned long long slot = 2 * gw + (seen ? 1 : 0);
      double * dst = a.packs + slot * P;
      for (int p = lane; p < P; p += 32) dst[p] = ws[p];
      if (lane == 0) a.slot_row[slot] = row;
    } else {
      warp_solve(ws, a.R, H, a.reg, a.out + static_cast<size_t>(row) * a.ldm);
    }
    seen = true;
    __syncwarp();
    for (int p = lane; p < P; p += 32) ws[p] = 0.0;
    __syncwarp();
  });
}

// Solves the rows the row-update kernel left: with slot_row, every row of the boundary slots
// (the warp of a row's first slot adds all its slots, in range order); without, every row
// 0..nrows-1 from its pack.
template <int RT>
__global__ void __launch_bounds__(kThreads) k_tc_solve(const double * __restrict__ packs,
                                                       const uint32_t * __restrict__ slot_row,
                                                       unsigned long long nitems, int R, int ldm,
                                                       double reg, double * __restrict__ out) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int RP = R + (R & 1), H = RP / 2, P = 2 * tc_pairs(H) + RP;
  double *  ws = reinterpret_cast<double *>(smem) + warp * tc_ws_doubles(RT);
  const unsigned long long TW = static_cast<unsigned long long>(gridDim.x) * kWarps;
  for (unsigned long long s = static_cast<unsigned long long>(blockIdx.x) * kWarps + warp; s < nitems;
       s += TW) {
    uint32_t row;
    if (slot_row) {
      row = slot_row[s];
      if (row == kEmptySlot) continue;
      long long t = static_cast<long long>(s) - 1;
      while (t >= 0 && slot_row[t] == kEmptySlot) --t;
      if (t >= 0 && slot_row[t] == row) continue;          // not the row's first slot
      for (int p = lane; p < P; p += 32) ws[p] = 0.0;
      for (unsigned long long u = s; u < nitems; ++u) {
        const uint32_t r2 = slot_row[u];
        if (r2 == kEmptySlot) continue;
        if (r2 != row) break;
        const double * src = packs + u * P;
        for (int p = lane; p < P; p += 32) ws[p] += src[p];
      }
    } else {
      row = static_cast<uint32_t>(s);
      const double * src = packs + s * P;
      for (int p = lane; p < P; p += 32) ws[p] = src[p];
    }
    __syncwarp();
    warp_solve(ws, R, H, reg, out + static_cast<size_t>(row) * ldm);
  }
}

// Sum over this grid's ranges of the stream of (v - sum_r lambda_r prod_m U_m[i_m, r])^2: one
// warp per range, the model's value per record by a warp sum, one atomic per CTA.
template <int N>
__global__ void __launch_bounds__(kThreads, 3) k_tc_sse(const TcArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ double part[kWarps];
  const int  lane = threadIdx.x & 31;
  const bool act  = 2 * lane < a.R;
  const bool hasy = 2 * lane + 1 < a.R;
  const double2 lam = act ? reinterpret_cast<const double2 *>(a.lambda)[lane] : make_double2(0.0, 0.0);
  double sse = 0.0;
  walk_range<N, 0>(a, smem, act, [&](double v, double2 h, bool, uint32_t, bool) {
    double x = act ? h.x * lam.x : 0.0;
    if (hasy) x = fma(h.y, lam.y, x);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    const double r = v - x;
    sse = fma(r, r, sse);
  });
  if (lane == 0) part[threadIdx.x >> 5] = sse;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += part[w];
    atomicAdd(a.sse, s);
  }
}

// out += sum of squares of columns [0, R) of a rows x ldm matrix (one atomic per CTA)
__global__ void __launch_bounds__(kThreads) k_tc_sumsq(const double * __restrict__ U, unsigned long long rows,
                                                       int R, int ldm, double * __restrict__ out) {
  __shared__ double part[kWarps];
  double s = 0.0;
  const unsigned long long n = rows * static_cast<unsigned long long>(R);
  for (unsigned long long e = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; e < n;
       e += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
    const double x = U[(e / R) * ldm + e % R];
    s = fma(x, x, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < kWarps; ++w) t += part[w];
    atomicAdd(out, t);
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

int rank_tier(int R) { return R <= 16 ? 16 : (R <= 32 ? 32 : 64); }

// Kernel pointer and grid (resident CTAs) of the row update for (N, tier, rows mode).
template <int N, int RT, bool ROWS>
cudaError_t update_kernel_of(void (**k)(TcArgs), size_t * smem, int * grid) {
  *k    = k_tc_update<N, RT, ROWS>;
  *smem = tc_update_smem(RT);
  cudaError_t e = cudaFuncSetAttribute(*k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)*smem);
  if (e != cudaSuccess) return e;
  int nb = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, *k, kThreads, *smem);
  *grid = std::max(nb, 1) * num_sms();
  return e;
}
template <int N>
cudaError_t update_kernel_n(int RT, bool rows, void (**k)(TcArgs), size_t * smem, int * grid) {
  if (RT == 16) return rows ? update_kernel_of<N, 16, true>(k, smem, grid) : update_kernel_of<N, 16, false>(k, smem, grid);
  if (RT == 32) return rows ? update_kernel_of<N, 32, true>(k, smem, grid) : update_kernel_of<N, 32, false>(k, smem, grid);
  return rows ? update_kernel_of<N, 64, true>(k, smem, grid) : update_kernel_of<N, 64, false>(k, smem, grid);
}
cudaError_t update_kernel(int N, int R, bool rows, void (**k)(TcArgs), size_t * smem, int * grid) {
  const int RT = rank_tier(R);
  switch (N) {
    case 2: return update_kernel_n<2>(RT, rows, k, smem, grid);
    case 3: return update_kernel_n<3>(RT, rows, k, smem, grid);
    case 4: return update_kernel_n<4>(RT, rows, k, smem, grid);
    case 5: return update_kernel_n<5>(RT, rows, k, smem, grid);
    case 6: return update_kernel_n<6>(RT, rows, k, smem, grid);
    case 7: return update_kernel_n<7>(RT, rows, k, smem, grid);
    default: return update_kernel_n<8>(RT, rows, k, smem, grid);
  }
}

cudaError_t launch_solve(const double * packs, const uint32_t * slot_row, unsigned long long nitems,
                         int R, int ldm, double reg, double * out, cudaStream_t s) {
  if (nitems == 0) return cudaSuccess;
  const int RT = rank_tier(R);
  const size_t smem = sizeof(double) * kWarps * tc_ws_doubles(RT);
  void (*k)(const double *, const uint32_t *, unsigned long long, int, int, double, double *) =
      RT == 16 ? k_tc_solve<16> : (RT == 32 ? k_tc_solve<32> : k_tc_solve<64>);
  cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const unsigned long long want = (nitems + kWarps - 1) / kWarps;
  const unsigned grid = (unsigned)std::min<unsigned long long>(want, (unsigned long long)num_sms() * 8);
  k<<<grid, kThreads, smem, s>>>(packs, slot_row, nitems, R, ldm, reg, out);
  spb200_count_launches(1);
  return cudaGetLastError();
}

void fill_stream_args(const FiberStream & fs, TcArgs & a) {
  const int N = fs.nmodes;
  a.rec = fs.rec;
  for (int l = 0; l < SPB200_MAXN - 2; ++l) a.up[l] = (l <= N - 3) ? fs.up[l] : nullptr;
  a.desc    = fs.desc;
  a.nrec    = fs.nrec;
  a.nchunks = static_cast<unsigned int>(fs.nchunks);
}

// SSE of the model (lambda: RP device doubles) over one stream's records, added into *d_sse.
cudaError_t launch_sse(const FiberStream & fs, int R, int ldm, const double * const * d_mats_by_mode,
                       const double * d_lambda, double * d_sse, cudaStream_t s) {
  if (fs.nrec == 0) return cudaSuccess;
  TcArgs a = {};
  fill_stream_args(fs, a);
  for (int l = 0; l < fs.nmodes; ++l) a.mats[l] = d_mats_by_mode[fs.perm[l]];
  a.ldm = ldm; a.R = R; a.lambda = d_lambda; a.sse = d_sse;
  void (*k)(TcArgs) = nullptr;
  switch (fs.nmodes) {
    case 2: k = k_tc_sse<2>; break;
    case 3: k = k_tc_sse<3>; break;
    case 4: k = k_tc_sse<4>; break;
    case 5: k = k_tc_sse<5>; break;
    case 6: k = k_tc_sse<6>; break;
    case 7: k = k_tc_sse<7>; break;
    default: k = k_tc_sse<8>; break;
  }
  const size_t smem = tc_ring_bytes();
  cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  int nb = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, k, kThreads, smem);
  if (e != cudaSuccess) return e;
  k<<<std::max(nb, 1) * num_sms(), kThreads, smem, s>>>(a);
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

// Device buffers of one completion run, released on every return path.
struct TcBuffers {
  double *   packs = nullptr;
  uint32_t * slot_row = nullptr;
  double *   lambda = nullptr;    // RP ones
  double *   sums = nullptr;      // [0] train SSE, [1] validation SSE, [2] sum ||U_m||^2
  ~TcBuffers() { cudaFree(packs); cudaFree(slot_row); cudaFree(lambda); cudaFree(sums); }
};

}  // namespace
}  // namespace spb200

using namespace spb200;

extern "C" int splatt_b200_tensor_sse(splatt_b200_tensor const * t, int ncolumns, int ldm,
                                      double const * const * d_factors, double const * lambda,
                                      double * sse_out, void * stream) {
  if (!t || !sse_out || t->streams.empty() || t->nmodes < 2 || t->nmodes > SPB200_MAXN ||
      !factors_ok(t->nmodes, ncolumns, ldm, reinterpret_cast<const void * const *>(d_factors)) ||
      !stream_fits(t->streams[0])) {
    fprintf(stderr, "SPLATT: splatt_b200_tensor_sse: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  DeviceGuard g(t->device);
  if (!g.ok) return SPLATT_ERROR_BADINPUT;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int RP = ncolumns + (ncolumns & 1);
  std::vector<double> lam(RP, 0.0);
  for (int r = 0; r < ncolumns; ++r) lam[r] = lambda ? lambda[r] : 1.0;
  double * d = nullptr;   // [0] the sum, [1..] lambda
  if (cudaMalloc(&d, sizeof(double) * (RP + 2)) != cudaSuccess) return SPLATT_ERROR_NOMEMORY;
  double h = 0.0;
  bool ok = cudaMemsetAsync(d, 0, sizeof(double), s) == cudaSuccess &&
            cudaMemcpyAsync(d + 2, lam.data(), sizeof(double) * RP, cudaMemcpyHostToDevice, s) == cudaSuccess &&
            launch_sse(t->streams[0], ncolumns, ldm, d_factors, d + 2, d, s) == cudaSuccess &&
            cudaMemcpyAsync(&h, d, sizeof(double), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
            cudaStreamSynchronize(s) == cudaSuccess;
  cudaFree(d);
  if (!ok) {
    fprintf(stderr, "SPLATT: splatt_b200_tensor_sse failed (%s)\n", cudaGetErrorString(cudaGetLastError()));
    return SPLATT_ERROR_BADINPUT;
  }
  *sse_out = h;
  return SPLATT_SUCCESS;
}

extern "C" int splatt_b200_tc_als_device(splatt_b200_tensor const * train,
                                         splatt_b200_tensor const * validate, int ncolumns, int ldm,
                                         double const * options, double * const * d_factors,
                                         double * history, int * iterations_out, void * stream) {
  const int R = ncolumns;
  const double reg = options ? options[SPLATT_OPTION_REGULARIZE] : 0.0;
  bool bad = !train || !options || train->nmodes < 2 || train->nmodes > SPB200_MAXN ||
             !factors_ok(train->nmodes, R, ldm, reinterpret_cast<const void * const *>(d_factors)) ||
             !(std::isfinite(reg) && reg > 0.0) || train->shard_count > 1 ||
             train->layout != SPLATT_B200_LAYOUT_ALLROOT || train->streams.empty();
  for (int m = 0; !bad && m < train->nmodes; ++m) {
    const ModePlan & p = train->plan[m];
    bad = p.stream < 0 || p.stream >= (int)train->streams.size() || p.kind != SPB200_KIND_ROOT ||
          train->streams[p.stream].perm[0] != m || !stream_fits(train->streams[p.stream]);
  }
  if (!bad && validate) {
    bad = validate->nmodes != train->nmodes || validate->shard_count > 1 ||
          validate->device != train->device || validate->streams.empty() ||
          !stream_fits(validate->streams[0]);
    for (int m = 0; !bad && m < train->nmodes; ++m) bad = validate->dims[m] != train->dims[m];
  }
  if (bad) {
    fprintf(stderr, "SPLATT: splatt_b200_tc_als_device: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  DeviceGuard g(train->device);
  if (!g.ok) return SPLATT_ERROR_BADINPUT;
  const int N = train->nmodes;
  const int RP = R + (R & 1), H = RP / 2;
  const size_t P = 2 * (size_t)H * (H + 1) + RP;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const uint64_t niters = (uint64_t)options[SPLATT_OPTION_NITER];
  const double tol = options[SPLATT_OPTION_TOLERANCE];
  const int verbosity = (int)options[SPLATT_OPTION_VERBOSITY];

  // one launch configuration per mode; the pack buffer serves the largest
  struct ModeLaunch { void (*k)(TcArgs); size_t smem; int grid; bool rows; };
  ModeLaunch ml[SPB200_MAXN];
  size_t max_packs = 0, max_slots = 0;
  for (int m = 0; m < N; ++m) {
    const FiberStream & fs = train->streams[train->plan[m].stream];
    ml[m].rows = fs.ktile_rows > 0;
    if (update_kernel(N, R, ml[m].rows, &ml[m].k, &ml[m].smem, &ml[m].grid) != cudaSuccess) {
      fprintf(stderr, "SPLATT: splatt_b200_tc_als_device: cannot configure the row update (%s)\n",
              cudaGetErrorString(cudaGetLastError()));
      return SPLATT_ERROR_BADINPUT;
    }
    const size_t slots = 2 * (size_t)ml[m].grid * kWarps;
    max_packs = std::max<size_t>(max_packs, ml[m].rows ? train->dims[m] : slots);
    if (!ml[m].rows) max_slots = std::max(max_slots, slots);
  }
  TcBuffers b;
  std::vector<double> ones(RP, 0.0);
  std::fill(ones.begin(), ones.begin() + R, 1.0);
  if (cudaMalloc(&b.packs, std::max<size_t>(max_packs, 1) * P * sizeof(double)) != cudaSuccess ||
      cudaMalloc(&b.slot_row, std::max<size_t>(max_slots, 1) * sizeof(uint32_t)) != cudaSuccess ||
      cudaMalloc(&b.lambda, RP * sizeof(double)) != cudaSuccess ||
      cudaMalloc(&b.sums, 3 * sizeof(double)) != cudaSuccess) {
    cudaGetLastError();
    return SPLATT_ERROR_NOMEMORY;
  }
  bool ok = cudaMemcpyAsync(b.lambda, ones.data(), RP * sizeof(double), cudaMemcpyHostToDevice, s) == cudaSuccess;
  const double nnz_train = (double)train->streams[0].nrec;
  const double nnz_val = validate ? (double)validate->streams[0].nrec : 0.0;
  double prev = 0.0;
  uint64_t its = 0;
  auto t0 = std::chrono::steady_clock::now();
  for (uint64_t it = 0; ok && it < niters; ++it) {
    if (verbosity > SPLATT_VERBOSITY_NONE) t0 = std::chrono::steady_clock::now();
    for (int m = 0; ok && m < N; ++m) {
      const FiberStream & fs = train->streams[train->plan[m].stream];
      const ModeLaunch & L = ml[m];
      ok = cudaMemset2DAsync(d_factors[m], (size_t)ldm * 8, 0, (size_t)R * 8, train->dims[m], s) == cudaSuccess;
      const unsigned long long nslots = 2ull * L.grid * kWarps;
      if (L.rows) ok = ok && cudaMemsetAsync(b.packs, 0, train->dims[m] * P * sizeof(double), s) == cudaSuccess;
      else ok = ok && cudaMemsetAsync(b.slot_row, 0xff, nslots * sizeof(uint32_t), s) == cudaSuccess;
      if (!ok) break;
      if (fs.nrec) {
        TcArgs a = {};
        fill_stream_args(fs, a);
        for (int l = 0; l < N; ++l) a.mats[l] = d_factors[fs.perm[l]];
        a.ldm = ldm; a.R = R; a.reg = reg; a.out = d_factors[m];
        a.packs = b.packs; a.slot_row = L.rows ? nullptr : b.slot_row;
        L.k<<<L.grid, kThreads, L.smem, s>>>(a);
        spb200_count_launches(1);
        ok = cudaGetLastError() == cudaSuccess;
      }
      if (L.rows)
        ok = ok && launch_solve(b.packs, nullptr, train->dims[m], R, ldm, reg, d_factors[m], s) == cudaSuccess;
      else if (fs.nrec)
        ok = ok && launch_solve(b.packs, b.slot_row, nslots, R, ldm, reg, d_factors[m], s) == cudaSuccess;
    }
    if (!ok) break;
    ok = cudaMemsetAsync(b.sums, 0, 3 * sizeof(double), s) == cudaSuccess;
    for (int m = 0; ok && m < N; ++m) {
      const unsigned grid = (unsigned)std::min<uint64_t>((train->dims[m] * R + kThreads - 1) / kThreads, 1184);
      k_tc_sumsq<<<std::max(grid, 1u), kThreads, 0, s>>>(d_factors[m], train->dims[m], R, ldm, b.sums + 2);
      spb200_count_launches(1);
      ok = cudaGetLastError() == cudaSuccess;
    }
    const double * const * cf = d_factors;
    ok = ok && launch_sse(train->streams[0], R, ldm, cf, b.lambda, b.sums, s) == cudaSuccess;
    if (validate) ok = ok && launch_sse(validate->streams[0], R, ldm, cf, b.lambda, b.sums + 1, s) == cudaSuccess;
    double h[3] = {0, 0, 0};
    ok = ok && cudaMemcpyAsync(h, b.sums, sizeof(h), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaStreamSynchronize(s) == cudaSuccess;
    if (!ok) break;
    const double L = h[0] + reg * h[2];
    const double trmse = std::sqrt(h[0] / nnz_train);
    const double vrmse = validate ? std::sqrt(h[1] / nnz_val) : std::nan("");
    if (history) { history[3 * it] = L; history[3 * it + 1] = trmse; history[3 * it + 2] = vrmse; }
    its = it + 1;
    if (verbosity > SPLATT_VERBOSITY_NONE) {
      const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
      printf("  its = %3llu (%0.3fs)  loss = %0.5e  train RMSE = %0.5e  validation RMSE = %0.5e\n",
             (unsigned long long)its, sec, L, trmse, vrmse);
    }
    if (it > 0 && std::fabs(prev - L) / prev < tol) break;
    prev = L;
  }
  if (!ok) {
    fprintf(stderr, "SPLATT: splatt_b200_tc_als_device failed (%s)\n", cudaGetErrorString(cudaGetLastError()));
    cudaStreamSynchronize(s);
    return SPLATT_ERROR_BADINPUT;
  }
  if (iterations_out) *iterations_out = (int)its;
  return SPLATT_SUCCESS;
}
