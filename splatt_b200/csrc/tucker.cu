// Sparse Tucker decomposition by HOOI (higher-order orthogonal iteration) on device-resident
// tensors: splatt_b200_ttmc and splatt_b200_tucker_hooi_device.
//
// Model X ~ G x_0 U_0 x_1 U_1 ... x_{N-1} U_{N-1}, U_m dims[m] x R_m with orthonormal columns.
// Its kernel is the TTMc Y_n = X_(n) (kron_{m != n} U_m), dims[n] x C_n, C_n = prod_{m != n} R_m,
// columns in mode order with the highest mode fastest.  On the ALLROOT layout every mode has a
// root stream, and the TTMc walks it like the root MTTKRP (Smith & Karypis, Euro-Par 2017):
//
//   * k_ttmc walks mode n's root stream with walk_levels (walk.cuh: the root MTTKRP's
//     nnz-balanced chunk ranges, one warp per range, a private TMA record ring).  Lane l keeps the
//     fiber sum s[l] = sum v U_leaf[k, l] in a register.  At a fiber close the warp forms
//     t = U_{N-2}[parent] (x) s (R_{N-2} R_leaf entries) in shared memory and adds
//     A (x) t into the slice's C_n-entry accumulator, A = the Kronecker product of the rows of
//     levels 1 .. N-3, kept per warp in shared memory and rebuilt when one of those levels
//     advances.  Lane l owns accumulator entries l + 32 i (i < TT, a register tile of 2, 8 or 32
//     entries: C_n <= 64, 256, 1024).  Entries are in level order; a per-CTA table in shared
//     memory maps them to the mode-ordered column at the store.
//   * Slices wholly inside a range are stored with plain stores; the first and the last slice of
//     a range go into the range's two boundary slots, which k_ttmc_combine adds in range order.
//     So on untiled streams Y_n, and with it the whole HOOI run, is bitwise reproducible.
//     Leaf-tiled streams (CTA-tiled, or ktile > 0) close a root row once per leaf tile; there
//     every piece is added with red.add.f64.
//
// HOOI's dense steps run on the device on tall-skinny matrices (k_atb_part/_fin: A^T B reduced
// over row blocks in a fixed order; k_ab: row-parallel A M + beta C; k_chol_inv: the R x R
// Cholesky factor's inverse for CholeskyQR2; k_sumsq_part/_fin; the sign convention's
// k_absmax_part/_fin), so every reduction has a fixed order.  The Ritz step's R x R eigen-solve
// is the Jacobi rotation loop of jacobi.cuh, run on the host on the R x R matrix read back.
#include "walk.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <numeric>
#include <vector>

namespace spb200 {
namespace {

#include "jacobi.cuh"

constexpr int kMaxTuckerRank = 32;
constexpr int kMaxTuckerCols = 1024;

struct TtmcArgs {
  TcArgs t;                      // the stream; t.mats by level, t.ldm, t.out = Y, t.packs, t.slot_row
  int    rk[SPB200_MAXN];        // rank by level
  int    cs[SPB200_MAXN];        // stride of the level's index in the mode-ordered column
  int    C;                      // columns of Y (and of a boundary slot)
  int    PA;                     // entries of A, the Kronecker product of levels 1 .. N-3
  int    K;                      // entries of t: rk[N-2] * rk[N-1] (N = 2: rk[1])
  int    wsm;                    // doubles of shared scratch per warp
};

// the per-CTA column table and (N >= 4) entry table in shared memory
__host__ __device__ constexpr size_t colmap_bytes(int C) { return ((size_t)C * 8 + 15) / 16 * 16; }

template <int N, int TT, bool ROWS>
__global__ void __launch_bounds__(kThreads, TT >= 32 ? 1 : 2) k_ttmc(const TtmcArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int  warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t * colmap = reinterpret_cast<uint32_t *>(smem + tc_ring_bytes());
  uint32_t * emap   = colmap + a.C;  // N >= 4: entry e -> (index into A) << 16 | (index into t)
  double *   A  = reinterpret_cast<double *>(smem + tc_ring_bytes() + colmap_bytes(a.C)) +
                  static_cast<size_t>(warp) * a.wsm;
  double *   tk = A + a.PA;
  double *   sb = tk + a.K;
  double *   ub = sb + 32;
  double *   rc = ub + 32;           // rows of levels 1 .. N-3, 32 doubles each
  // level-ordered entry e (levels 1 .. N-1, the leaf fastest) -> mode-ordered column
  for (int e = threadIdx.x; e < a.C; e += kThreads) {
    int rem = e, col = 0;
    for (int l = N - 1; l >= 1; --l) {
      const int j = rem % a.rk[l];
      rem /= a.rk[l];
      col += j * a.cs[l];
    }
    colmap[e] = static_cast<uint32_t>(col);
    if (N >= 4) emap[e] = static_cast<uint32_t>(e / a.K) << 16 | static_cast<uint32_t>(e % a.K);
  }
  __syncthreads();

  const size_t   ldm  = static_cast<size_t>(a.t.ldm);
  const int      RL   = a.rk[N - 1];
  const int      K    = a.K;
  const double * leaf = a.t.mats[N - 1];
  const unsigned long long gw = static_cast<unsigned long long>(blockIdx.x) * kWarps + warp;
  double acc[TT];
#pragma unroll
  for (int i = 0; i < TT; ++i) acc[i] = 0.0;
  double s    = 0.0;
  bool   seen = false;   // this warp closed a slice already: later ones (but the last) are whole

  walk_levels<N>(a.t, smem, [&](const uint4 & q, uint32_t pc, const uint32_t * pos, bool close,
                                uint32_t row, bool last) {
    if constexpr (N >= 4) {
      if (pc >= 2u) {    // a level of 1 .. N-3 has a new node: rebuild A
#pragma unroll
        for (int l = 1; l <= N - 3; ++l)
          if (l + int(pc) >= N - 1 && lane < a.rk[l])
            rc[(l - 1) * 32 + lane] = a.t.mats[l][static_cast<size_t>(__ldg(&a.t.up[l][pos[l]])) * ldm + lane];
        __syncwarp();
        for (int p = lane; p < a.PA; p += 32) {
          int    rem = p;
          double x   = 1.0;
#pragma unroll
          for (int l = N - 3; l >= 1; --l) {
            const int j = rem % a.rk[l];
            rem /= a.rk[l];
            x *= rc[(l - 1) * 32 + j];
          }
          A[p] = x;
        }
        __syncwarp();
      }
    }
    const double v = rec_val<double>(q);
    if (lane < RL) s = fma(v, leaf[static_cast<size_t>(q.z) * ldm + lane], s);
    if ((q.w >> SPB200_IDX_BITS) == 0u) return;
    // the fiber closes (N = 2: the slice): acc += A (x) U_{N-2}[parent] (x) s
    if constexpr (N >= 3) {
      if (lane < a.rk[N - 2]) ub[lane] = a.t.mats[N - 2][static_cast<size_t>(q.w & SPB200_IDX_MASK) * ldm + lane];
    }
    sb[lane] = s;
    __syncwarp();
    for (int k = lane; k < K; k += 32) tk[k] = (N >= 3) ? ub[k / RL] * sb[k % RL] : sb[k];
    __syncwarp();
#pragma unroll
    for (int i = 0; i < TT; ++i) {
      const int e = lane + 32 * i;
      if (e >= a.C) continue;
      if constexpr (N >= 4) {
        const uint32_t m = emap[e];
        acc[i] = fma(A[m >> 16], tk[m & 0xffffu], acc[i]);
      } else {
        acc[i] += tk[e];     // N <= 3: A = [1], t has all C entries
      }
    }
    __syncwarp();
    s = 0.0;
    if (!close) return;
    const int C = a.C;
    if constexpr (ROWS) {
      double * dst = a.t.out + static_cast<size_t>(row) * C;
#pragma unroll
      for (int i = 0; i < TT; ++i)
        if (lane + 32 * i < C) atomicAdd(dst + colmap[lane + 32 * i], acc[i]);
    } else {
      double * dst;
      if (!seen || last) {
        const unsigned long long slot = 2 * gw + (seen ? 1 : 0);
        dst = a.t.packs + slot * C;
        if (lane == 0) a.t.slot_row[slot] = row;
      } else {
        dst = a.t.out + static_cast<size_t>(row) * C;
      }
#pragma unroll
      for (int i = 0; i < TT; ++i)
        if (lane + 32 * i < C) dst[colmap[lane + 32 * i]] = acc[i];
    }
    seen = true;
#pragma unroll
    for (int i = 0; i < TT; ++i) acc[i] = 0.0;
  });
}

// Adds the boundary slots of every row the TTMc kernel left there, in range order (the warp of a
// row's first slot adds all its slots), and stores the row.
__global__ void __launch_bounds__(kThreads) k_ttmc_combine(const double * __restrict__ packs,
                                                           const uint32_t * __restrict__ slot_row,
                                                           unsigned long long nslots, int C,
                                                           double * __restrict__ out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned long long TW = static_cast<unsigned long long>(gridDim.x) * kWarps;
  for (unsigned long long s = static_cast<unsigned long long>(blockIdx.x) * kWarps + warp; s < nslots;
       s += TW) {
    const uint32_t row = slot_row[s];
    if (row == kEmptySlot) continue;
    long long t = static_cast<long long>(s) - 1;
    while (t >= 0 && slot_row[t] == kEmptySlot) --t;
    if (t >= 0 && slot_row[t] == row) continue;          // not the row's first slot
    for (int j = lane; j < C; j += 32) {
      double x = 0.0;
      for (unsigned long long u = s; u < nslots; ++u) {
        const uint32_t r2 = slot_row[u];
        if (r2 == kEmptySlot) continue;
        if (r2 != row) break;
        x += packs[u * C + j];
      }
      out[static_cast<size_t>(row) * C + j] = x;
    }
  }
}

// ---- dense steps on tall-skinny matrices --------------------------------------------------------

// part[g] = A[rows_g]^T B[rows_g] (K x J, row-major) over the g-th block of `chunk` rows: CTA
// (x, g) owns columns [32 x, 32 x + 32) of A; thread (k, jg) sums column k of A against columns
// jg + 8 u of B row by row.  J <= 32.
// (__maxnreg__: with the default launch bounds ptxas keeps it at 32 registers and a stack slot.)
__global__ void __maxnreg__(64) k_atb_part(const double * __restrict__ Am, int lda,
                                           const double * __restrict__ Bm, int ldb,
                                           unsigned long long rows, unsigned long long chunk,
                                           int K, int J, double * __restrict__ part) {
  __shared__ double ta[32][33];
  __shared__ double tb[32][33];
  const int kc = threadIdx.x & 31, jg = threadIdx.x >> 5;
  const int k0 = blockIdx.x * 32;
  const unsigned long long lo = chunk * blockIdx.y, hi = min(rows, lo + chunk);
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (unsigned long long r0 = lo; r0 < hi; r0 += 32) {
    const int nr = static_cast<int>(min(32ull, hi - r0));
    for (int x = threadIdx.x; x < 32 * 32; x += kThreads) {
      const int i = x >> 5, c = x & 31;
      ta[i][c] = (i < nr && k0 + c < K) ? Am[(r0 + i) * lda + k0 + c] : 0.0;
      tb[i][c] = (i < nr && c < J) ? Bm[(r0 + i) * ldb + c] : 0.0;
    }
    __syncthreads();
    for (int i = 0; i < nr; ++i) {
      const double x = ta[i][kc];
#pragma unroll
      for (int u = 0; u < 4; ++u) acc[u] = fma(x, tb[i][jg + 8 * u], acc[u]);
    }
    __syncthreads();
  }
  if (k0 + kc >= K) return;
#pragma unroll
  for (int u = 0; u < 4; ++u)
    if (jg + 8 * u < J) part[(static_cast<size_t>(blockIdx.y) * K + k0 + kc) * J + jg + 8 * u] = acc[u];
}
// out = sum over the G partials in order
__global__ void __launch_bounds__(kThreads) k_atb_fin(const double * __restrict__ part, int G, int KJ,
                                                      double * __restrict__ out) {
  for (int e = blockIdx.x * kThreads + threadIdx.x; e < KJ; e += gridDim.x * kThreads) {
    double x = 0.0;
    for (int g = 0; g < G; ++g) x += part[static_cast<size_t>(g) * KJ + e];
    out[e] = x;
  }
}

// Out[i, :J] = A[i, :K] M (M: K x J, row-major, leading dimension J) + beta Cm[i, :J], beta =
// *beta_dev when given.  32 rows per CTA; thread (j, w) computes rows w + 8 u, column j.  Out may
// be A when K <= 32 (the CTA reads its rows whole before it writes).
__global__ void __launch_bounds__(kThreads) k_ab(const double * Am, int lda, int K,
                                                 const double * __restrict__ M, int J,
                                                 double beta, const double * __restrict__ beta_dev,
                                                 const double * __restrict__ Cm, int ldc,
                                                 double * Out, int ldo, unsigned long long rows) {
  __shared__ double ta[32][33];
  __shared__ double tm[32][33];
  const int j = threadIdx.x & 31, w = threadIdx.x >> 5;
  const unsigned long long r0 = static_cast<unsigned long long>(blockIdx.x) * 32;
  const int nr = static_cast<int>(min(32ull, rows - r0));
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (int k0 = 0; k0 < K; k0 += 32) {
    for (int x = threadIdx.x; x < 32 * 32; x += kThreads) {
      const int i = x >> 5, c = x & 31;
      ta[i][c] = (i < nr && k0 + c < K) ? Am[(r0 + i) * lda + k0 + c] : 0.0;
      tm[i][c] = (k0 + i < K && c < J) ? M[static_cast<size_t>(k0 + i) * J + c] : 0.0;
    }
    __syncthreads();
    const int kn = min(32, K - k0);
    for (int k = 0; k < kn; ++k) {
      const double m = tm[k][j];
#pragma unroll
      for (int u = 0; u < 4; ++u) acc[u] = fma(ta[w + 8 * u][k], m, acc[u]);
    }
    __syncthreads();
  }
  if (j >= J) return;
  const double b = beta_dev ? *beta_dev : beta;
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int i = w + 8 * u;
    if (i >= nr) continue;
    double x = acc[u];
    if (Cm) x = fma(b, Cm[(r0 + i) * ldc + j], x);
    Out[(r0 + i) * ldo + j] = x;
  }
}

// Minv = L^-T for the Cholesky factor L of the R x R Gram G (one warp).  *bad = 1 when a pivot is
// not finite or not above 2^-46 times its diagonal entry (dependent columns); Minv is then I.
__global__ void __launch_bounds__(32) k_chol_inv(const double * __restrict__ G, int R,
                                                 double * __restrict__ Minv, int * bad) {
  __shared__ double L[kMaxTuckerRank][kMaxTuckerRank + 1];
  __shared__ double X[kMaxTuckerRank][kMaxTuckerRank + 1];
  __shared__ int fail;
  const int lane = threadIdx.x;
  for (int x = lane; x < R * R; x += 32) L[x / R][x % R] = G[x];
  if (lane == 0) fail = 0;
  __syncwarp();
  for (int j = 0; j < R; ++j) {
    if (lane == 0) {
      double d = L[j][j];
      for (int k = 0; k < j; ++k) d -= L[j][k] * L[j][k];
      if (!(d > G[j * R + j] * 1.4210854715202004e-14) || !(d < INFINITY)) fail = 1;
      L[j][j] = sqrt(fmax(d, 0.0));
    }
    __syncwarp();
    if (fail) break;
    for (int i = j + 1 + lane; i < R; i += 32) {
      double x = L[i][j];
      for (int k = 0; k < j; ++k) x -= L[i][k] * L[j][k];
      L[i][j] = x / L[j][j];
    }
    __syncwarp();
  }
  __syncwarp();
  if (fail) {
    for (int x = lane; x < R * R; x += 32) Minv[x] = (x / R == x % R) ? 1.0 : 0.0;
    if (lane == 0) atomicExch(bad, 1);
    return;
  }
  // column c of L^-1 by forward substitution (lane c)
  if (lane < R) {
    const int c = lane;
    for (int i = 0; i < R; ++i) {
      double x = (i == c) ? 1.0 : 0.0;
      for (int k = c; k < i; ++k) x -= L[i][k] * X[k][c];
      X[i][c] = (i < c) ? 0.0 : x / L[i][i];
    }
  }
  __syncwarp();
  for (int x = lane; x < R * R; x += 32) Minv[x] = X[x % R][x / R];   // Minv[k][j] = Linv[j][k]
}

// sum of squares of the rows x J entries of M (leading dimension ld) in two passes with a fixed
// order: CTA g of kSumCtas sums rows [rows g / G, rows (g + 1) / G) with a fixed tree.
constexpr int kSumCtas = 256;
__global__ void __launch_bounds__(kThreads) k_sumsq_part(const double * __restrict__ M, int ld, int J,
                                                         unsigned long long rows, double * __restrict__ part) {
  __shared__ double sh[kThreads];
  const unsigned long long lo = rows * blockIdx.x / gridDim.x, hi = rows * (blockIdx.x + 1) / gridDim.x;
  const unsigned long long n = (hi - lo) * J;
  double s = 0.0;
  for (unsigned long long e = threadIdx.x; e < n; e += kThreads) {
    const double x = M[(lo + e / J) * ld + e % J];
    s = fma(x, x, s);
  }
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int o = kThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = sh[0];
}
// *out = sum of the parts in order; *shift = (sum > 0 ? mu_rel * sum : 1) when shift is given
__global__ void k_sumsq_fin(const double * __restrict__ part, int n, double * __restrict__ out,
                            double mu_rel, double * __restrict__ shift) {
  double s = 0.0;
  for (int g = 0; g < n; ++g) s += part[g];
  *out = s;
  if (shift) *shift = s > 0.0 ? mu_rel * s : 1.0;
}

// ||X||^2 with duplicate coordinates summed: a run of records of one fiber with equal leaf ids is
// one coordinate; the thread of the run's first record sums it (across range cuts, which this
// kernel does not see).  Two passes with a fixed order like k_sumsq_part.
__global__ void __launch_bounds__(kThreads) k_xnorm_part(const SpRec * __restrict__ rec,
                                                         unsigned long long nrec, double * __restrict__ part) {
  __shared__ double sh[kThreads];
  double s = 0.0;
  for (unsigned long long k = static_cast<unsigned long long>(blockIdx.x) * kThreads + threadIdx.x; k < nrec;
       k += static_cast<unsigned long long>(gridDim.x) * kThreads) {
    const SpRec r = rec[k];
    if (k > 0 && (rec[k - 1].aux >> SPB200_IDX_BITS) == 0u && rec[k - 1].k == r.k) continue;
    double x = r.v;
    for (unsigned long long j = k; (rec[j].aux >> SPB200_IDX_BITS) == 0u && j + 1 < nrec && rec[j + 1].k == r.k; ++j)
      x += rec[j + 1].v;
    s = fma(x, x, s);
  }
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int o = kThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = sh[0];
}

// Sign convention: per column j < J of U (rows x J, leading dimension ld) the entry of largest
// magnitude, the lowest row on a tie.  Pass 1: CTA g over its row block, thread (j, q) every 8th
// row; pass 2 (one warp) in block order; sgn[j] = -1 when that entry is negative, else 1.
__device__ __forceinline__ bool absmax_better(double x, unsigned long long i, double bx, unsigned long long bi) {
  return fabs(x) > fabs(bx) || (fabs(x) == fabs(bx) && i < bi);
}
__global__ void __launch_bounds__(kThreads) k_absmax_part(const double * __restrict__ U, int ld, int J,
                                                          unsigned long long rows, double * __restrict__ pv,
                                                          unsigned long long * __restrict__ pi) {
  __shared__ double sv[kThreads];
  __shared__ unsigned long long si[kThreads];
  const int j = threadIdx.x & 31, q = threadIdx.x >> 5;
  const unsigned long long lo = rows * blockIdx.x / gridDim.x, hi = rows * (blockIdx.x + 1) / gridDim.x;
  double bv = 0.0;
  unsigned long long bi = ~0ull;
  if (j < J)
    for (unsigned long long i = lo + q; i < hi; i += kWarps) {
      const double x = U[i * ld + j];
      if (absmax_better(x, i, bv, bi)) { bv = x; bi = i; }
    }
  sv[threadIdx.x] = bv;
  si[threadIdx.x] = bi;
  __syncthreads();
  if (q == 0) {
    for (int w = 1; w < kWarps; ++w)
      if (absmax_better(sv[w * 32 + j], si[w * 32 + j], bv, bi)) { bv = sv[w * 32 + j]; bi = si[w * 32 + j]; }
    pv[blockIdx.x * 32 + j] = bv;
    pi[blockIdx.x * 32 + j] = bi;
  }
}
__global__ void __launch_bounds__(32) k_absmax_fin(const double * __restrict__ pv,
                                                   const unsigned long long * __restrict__ pi, int G,
                                                   double * __restrict__ sgn) {
  const int j = threadIdx.x;
  double bv = 0.0;
  unsigned long long bi = ~0ull;
  for (int g = 0; g < G; ++g)
    if (absmax_better(pv[g * 32 + j], pi[g * 32 + j], bv, bi)) { bv = pv[g * 32 + j]; bi = pi[g * 32 + j]; }
  sgn[j] = bv < 0.0 ? -1.0 : 1.0;
}
// M[i, j] *= sgn[j], j < J
__global__ void __launch_bounds__(kThreads) k_flip_cols(double * __restrict__ M, int ld, int J,
                                                        unsigned long long rows, const double * __restrict__ sgn) {
  for (unsigned long long e = blockIdx.x * static_cast<unsigned long long>(kThreads) + threadIdx.x; e < rows * J;
       e += static_cast<unsigned long long>(gridDim.x) * kThreads)
    M[(e / J) * ld + e % J] *= sgn[e % J];
}

// ---- host side ---------------------------------------------------------------------------------

// The TTMc kernel of (N, register tile for C columns, rows mode).
template <int N>
void (*ttmc_kernel(int C, bool rows))(TtmcArgs) {
  if (C <= 64) return rows ? k_ttmc<N, 2, true> : k_ttmc<N, 2, false>;
  if (C <= 256) return rows ? k_ttmc<N, 8, true> : k_ttmc<N, 8, false>;
  return rows ? k_ttmc<N, 32, true> : k_ttmc<N, 32, false>;
}

int cols_but(int N, const int * ranks, int n) {
  int C = 1;
  for (int m = 0; m < N; ++m)
    if (m != n) C *= ranks[m];
  return C;
}

// The launch of one mode's TTMc and its arguments.
struct TtmcPlan : WalkLaunch<TtmcArgs> {
  TtmcArgs a = {};
};

bool plan_ttmc(const splatt_b200_tensor * t, int n, const int * ranks, int ldm,
               const double * const * mats_by_mode, double * out, TtmcPlan & p) {
  const int N = t->nmodes;
  const FiberStream & fs = t->streams[t->plan[n].stream];
  TtmcArgs & a = p.a;
  a = {};
  a.t = walk_args(fs, mats_by_mode, ldm, 0);
  a.t.out = out;
  int stride[SPB200_MAXN];
  for (int m = N - 1, s = 1; m >= 0; --m) {
    stride[m] = (m == n) ? 0 : s;
    if (m != n) s *= ranks[m];
  }
  for (int l = 0; l < N; ++l) {
    const int m = fs.perm[l];
    a.rk[l] = ranks[m];
    a.cs[l] = stride[m];
  }
  a.C = cols_but(N, ranks, n);
  a.K = (N >= 3) ? a.rk[N - 2] * a.rk[N - 1] : a.rk[1];
  a.PA = a.C / a.K;
  a.wsm = a.PA + a.K + 64 + std::max(N - 3, 0) * 32;
  const bool rows = fs.ktile_rows > 0;
  if (!p.configure(with_nmodes(N, [&](auto nm) { return ttmc_kernel<nm.value>(a.C, rows); }),
                   tc_ring_bytes() + colmap_bytes(a.C) + (size_t)kWarps * a.wsm * sizeof(double), rows)) {
    fprintf(stderr, "SPLATT: cannot configure the TTMc kernel (%s)\n", cudaGetErrorString(cudaGetLastError()));
    return false;
  }
  return true;
}

// Y = 0, then the TTMc into Y (packs: nslots x C doubles, slot_row: nslots)
bool run_ttmc(const splatt_b200_tensor * t, int n, TtmcPlan & p, double * packs, uint32_t * slot_row,
              cudaStream_t s) {
  const FiberStream & fs = t->streams[t->plan[n].stream];
  if (cudaMemsetAsync(p.a.t.out, 0, t->dims[n] * p.a.C * sizeof(double), s) != cudaSuccess) return false;
  if (!fs.nrec) return true;
  p.a.t.packs = packs;
  p.a.t.slot_row = slot_row;
  // other modes may share this instantiation with less shared memory: set it for this launch
  if (cudaFuncSetAttribute(p.k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem) != cudaSuccess ||
      p.launch(p.a, slot_row, s) != cudaSuccess)
    return false;
  if (!p.rows) {
    k_ttmc_combine<<<combine_grid(p.nslots), kThreads, 0, s>>>(packs, slot_row, p.nslots, p.a.C, p.a.t.out);
    spb200_count_launches(1);
  }
  return cudaGetLastError() == cudaSuccess;
}

bool ranks_ok(const splatt_b200_tensor * t, const int * ranks, int ldm, bool all_modes, int mode) {
  if (!ranks || (ldm & 1)) return false;
  const int N = t->nmodes;
  for (int m = 0; m < N; ++m)
    if (ranks[m] < 1 || ranks[m] > kMaxTuckerRank || (uint64_t)ranks[m] > t->dims[m] || ldm < ranks[m])
      return false;
  for (int n = 0; n < N; ++n) {
    if (!all_modes && n != mode) continue;
    const int C = cols_but(N, ranks, n);
    if (C > kMaxTuckerCols || (all_modes && ranks[n] > C)) return false;
  }
  return true;
}

bool aligned(const void * p) { return p && reinterpret_cast<uintptr_t>(p) % 16 == 0; }

// Device scratch of the dense steps: A^T B partials, and the small matrices and scalars.
constexpr size_t kPartDoubles = 1u << 20;     // k_atb_part: G x K x J <= 1024 / ceil(K/32) x 32 ceil(K/32) x 32
struct Dense {
  double * part = nullptr;
  double * sq = nullptr;         // kSumCtas partial sums
  double * small = nullptr;      // 8 x 32 x 32 doubles: Gram, Minv, M, S, V, ...
  double * scal = nullptr;       // 8 scalars
  double * absv = nullptr;       // kSumCtas x 32
  unsigned long long * absi = nullptr;
  int *    bad = nullptr;
  ~Dense() {
    cudaFree(part); cudaFree(sq); cudaFree(small); cudaFree(scal); cudaFree(absv); cudaFree(absi); cudaFree(bad);
  }
  bool alloc() {
    return cudaMalloc(&part, kPartDoubles * 8) == cudaSuccess && cudaMalloc(&sq, kSumCtas * 8) == cudaSuccess &&
           cudaMalloc(&small, 8 * 1024 * 8) == cudaSuccess && cudaMalloc(&scal, 8 * 8) == cudaSuccess &&
           cudaMalloc(&absv, kSumCtas * 32 * 8) == cudaSuccess &&
           cudaMalloc(&absi, kSumCtas * 32 * 8) == cudaSuccess && cudaMalloc(&bad, sizeof(int)) == cudaSuccess;
  }
  double * mat(int i) { return small + (size_t)i * 1024; }

  // out (K x J) = A^T B over `rows` rows
  void atb(const double * A, int lda, const double * B, int ldb, uint64_t rows, int K, int J, double * out,
           cudaStream_t s) {
    const int kx = (K + 31) / 32;
    const uint64_t G0 = std::max<uint64_t>(1, std::min<uint64_t>((rows + 31) / 32, 1024 / kx));
    const uint64_t chunk = (rows + G0 - 1) / G0;
    const int G = (int)std::max<uint64_t>(1, (rows + chunk - 1) / std::max<uint64_t>(chunk, 1));
    k_atb_part<<<dim3(kx, G), kThreads, 0, s>>>(A, lda, B, ldb, rows, std::max<uint64_t>(chunk, 1), K, J, part);
    k_atb_fin<<<std::min((K * J + kThreads - 1) / kThreads, 1024), kThreads, 0, s>>>(part, G, K * J, out);
    spb200_count_launches(2);
  }
  // Out = A M + beta C
  void ab(const double * A, int lda, int K, const double * M, int J, double beta, const double * beta_dev,
          const double * Cm, int ldc, double * Out, int ldo, uint64_t rows, cudaStream_t s) {
    if (!rows) return;
    k_ab<<<(unsigned)((rows + 31) / 32), kThreads, 0, s>>>(A, lda, K, M, J, beta, beta_dev, Cm, ldc, Out, ldo, rows);
    spb200_count_launches(1);
  }
  void sumsq(const double * M, int ld, int J, uint64_t rows, double * out, double mu_rel, double * shift,
             cudaStream_t s) {
    k_sumsq_part<<<kSumCtas, kThreads, 0, s>>>(M, ld, J, rows, sq);
    k_sumsq_fin<<<1, 1, 0, s>>>(sq, kSumCtas, out, mu_rel, shift);
    spb200_count_launches(2);
  }
  // Q (rows x R, ldq) = CholeskyQR2 of Z (rows x R, ldz); *bad set on a failed pivot.  The second
  // product runs in place: with K = R <= 32 every CTA of k_ab reads its rows whole before it
  // writes them.
  void cholqr2(const double * Z, int ldz, double * Q, int ldq, uint64_t rows, int R, cudaStream_t s) {
    atb(Z, ldz, Z, ldz, rows, R, R, mat(0), s);
    k_chol_inv<<<1, 32, 0, s>>>(mat(0), R, mat(1), bad);
    ab(Z, ldz, R, mat(1), R, 0.0, nullptr, nullptr, 0, Q, ldq, rows, s);
    atb(Q, ldq, Q, ldq, rows, R, R, mat(0), s);
    k_chol_inv<<<1, 32, 0, s>>>(mat(0), R, mat(1), bad);
    ab(Q, ldq, R, mat(1), R, 0.0, nullptr, nullptr, 0, Q, ldq, rows, s);
    spb200_count_launches(2);
  }
  // sgn = the sign convention's column signs of U; U's columns flipped
  void fix_signs(double * U, int ld, int J, uint64_t rows, double * sgn, cudaStream_t s) {
    k_absmax_part<<<kSumCtas, kThreads, 0, s>>>(U, ld, J, rows, absv, absi);
    k_absmax_fin<<<1, 32, 0, s>>>(absv, absi, kSumCtas, sgn);
    flip(U, ld, J, rows, sgn, s);
    spb200_count_launches(2);
  }
  void flip(double * M, int ld, int J, uint64_t rows, const double * sgn, cudaStream_t s) {
    k_flip_cols<<<elementwise_grid(rows, J), kThreads, 0, s>>>(M, ld, J, rows, sgn);
    spb200_count_launches(1);
  }
};

// Eigenvectors of the symmetric R x R matrix S (row-major) in descending eigenvalue order (ties
// by index) as the columns of the row-major V; the eigenvalues into lam.
void ritz_rotation(const double * S, int R, double * V, double * lam) {
  std::vector<double> A(S, S + (size_t)R * R), W((size_t)R * R), P((size_t)R * R);
  jacobi_pinv(A.data(), W.data(), R, P.data());
  std::vector<int> idx(R);
  std::iota(idx.begin(), idx.end(), 0);
  std::stable_sort(idx.begin(), idx.end(), [&](int x, int y) { return A[x + x * R] > A[y + y * R]; });
  for (int j = 0; j < R; ++j) {
    lam[j] = A[idx[j] + idx[j] * R];
    for (int i = 0; i < R; ++i) V[i * R + j] = W[idx[j] + i * R];
  }
}

}  // namespace
}  // namespace spb200

using namespace spb200;

extern "C" int splatt_b200_ttmc(splatt_b200_tensor const * t, int mode, int const * ranks, int ldm,
                                double const * const * d_mats, double * d_out, void * stream) {
  bool bad = !root_streams_ok(t) || mode < 0 || mode >= t->nmodes || !d_mats || !aligned(d_out) ||
             !ranks_ok(t, ranks, ldm, false, mode);
  for (int m = 0; !bad && m < t->nmodes; ++m)
    if (m != mode && !aligned(d_mats[m])) bad = true;
  if (bad) {
    fprintf(stderr, "SPLATT: splatt_b200_ttmc: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  DeviceGuard g(t->device);
  if (!g.ok) return SPLATT_ERROR_BADINPUT;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  TtmcPlan p;
  if (!plan_ttmc(t, mode, ranks, ldm, d_mats, d_out, p)) return SPLATT_ERROR_BADINPUT;
  double * packs = nullptr;
  uint32_t * slot_row = nullptr;
  if (p.nslots &&
      (cudaMallocAsync(&packs, p.nslots * p.a.C * sizeof(double), s) != cudaSuccess ||
       cudaMallocAsync(&slot_row, p.nslots * sizeof(uint32_t), s) != cudaSuccess)) {
    cudaGetLastError();
    if (packs) cudaFreeAsync(packs, s);
    return SPLATT_ERROR_NOMEMORY;
  }
  const bool ok = run_ttmc(t, mode, p, packs, slot_row, s);
  if (packs) cudaFreeAsync(packs, s);
  if (slot_row) cudaFreeAsync(slot_row, s);
  if (!ok) {
    fprintf(stderr, "SPLATT: splatt_b200_ttmc failed (%s)\n", cudaGetErrorString(cudaGetLastError()));
    return SPLATT_ERROR_BADINPUT;
  }
  return SPLATT_SUCCESS;
}

namespace {
// Device buffers of one HOOI run, released on every return path.
struct HooiBuffers {
  double *   F[SPB200_MAXN] = {nullptr};   // working factors, dims[m] x ldm
  double *   Y = nullptr;                   // max dims[n] x C_n
  double *   Qa = nullptr, * Qb = nullptr, * Z = nullptr;   // max dims x 32
  double *   W = nullptr;                   // max C x 32: Y^T Q
  double *   G = nullptr;                   // C_{N-1} x R_{N-1}: the core
  double *   packs = nullptr;
  uint32_t * slot_row = nullptr;
  ~HooiBuffers() {
    for (double * p : F) cudaFree(p);
    cudaFree(Y); cudaFree(Qa); cudaFree(Qb); cudaFree(Z); cudaFree(W); cudaFree(G); cudaFree(packs); cudaFree(slot_row);
  }
};
}  // namespace

extern "C" int splatt_b200_tucker_hooi_device(splatt_b200_tensor const * t, int const * ranks, int ldm,
                                              double const * options, splatt_b200_tucker_opts const * topts,
                                              double * const * d_factors, double * core_out, double * history,
                                              int * iterations_out, void * stream) {
  const splatt_b200_tucker_opts o = topts ? *topts : splatt_b200_tucker_opts{50, 1e-10};
  const double tol = options ? options[SPLATT_OPTION_TOLERANCE] : 0.0;
  const double niter = options ? options[SPLATT_OPTION_NITER] : 0.0;
  bool bad = !root_streams_ok(t) || !options || !core_out || !d_factors || !ranks_ok(t, ranks, ldm, true, 0) ||
             o.max_power < 1 || !(std::isfinite(o.svd_tol) && o.svd_tol >= 0.0) ||
             !(std::isfinite(tol) && tol >= 0.0) || !(niter >= 0.0 && niter <= 2147483647.0);
  for (int m = 0; !bad && m < t->nmodes; ++m)
    if (!aligned(d_factors[m])) bad = true;
  if (bad) {
    fprintf(stderr, "SPLATT: splatt_b200_tucker_hooi_device: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  DeviceGuard g(t->device);
  if (!g.ok) return SPLATT_ERROR_BADINPUT;
  cudaError_t last = cudaSuccess;         // the error a check consumed, for the message
  const int N = t->nmodes;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  // relative shift of the orthogonal iteration: Q <- orth(Y Y^T Q + mu Q), mu = 2^-20 ||Y_n||_F^2
  const double kMuRel = 9.5367431640625e-07;

  TtmcPlan plan[SPB200_MAXN];
  HooiBuffers b;
  Dense d;
  uint64_t max_dim = 1, max_yc = 1;
  unsigned long long max_packs = 1;
  int max_c = 1;
  bool ok = d.alloc();
  for (int m = 0; ok && m < N; ++m) {
    ok = cudaMalloc(&b.F[m], t->dims[m] * ldm * sizeof(double)) == cudaSuccess;
    max_dim = std::max<uint64_t>(max_dim, t->dims[m]);
    const int C = cols_but(N, ranks, m);
    max_c = std::max(max_c, C);
    max_yc = std::max<uint64_t>(max_yc, t->dims[m] * C);
  }
  ok = ok && cudaMalloc(&b.Y, max_yc * sizeof(double)) == cudaSuccess &&
       cudaMalloc(&b.Qa, max_dim * 32 * sizeof(double)) == cudaSuccess &&
       cudaMalloc(&b.Qb, max_dim * 32 * sizeof(double)) == cudaSuccess &&
       cudaMalloc(&b.Z, max_dim * 32 * sizeof(double)) == cudaSuccess &&
       cudaMalloc(&b.W, (size_t)max_c * 32 * sizeof(double)) == cudaSuccess &&
       cudaMalloc(&b.G, (size_t)max_c * 32 * sizeof(double)) == cudaSuccess;
  if (!ok) {
    cudaGetLastError();
    return SPLATT_ERROR_NOMEMORY;
  }
  const double * fmats[SPB200_MAXN];
  for (int m = 0; m < N; ++m) fmats[m] = b.F[m];
  for (int n = 0; n < N; ++n) {
    if (!plan_ttmc(t, n, ranks, ldm, fmats, b.Y, plan[n])) return SPLATT_ERROR_BADINPUT;
    max_packs = std::max(max_packs, plan[n].nslots * (unsigned long long)plan[n].a.C);
  }
  if (cudaMalloc(&b.packs, max_packs * sizeof(double)) != cudaSuccess ||
      cudaMalloc(&b.slot_row, std::max(max_slots(plan, N), 1ull) * sizeof(uint32_t)) != cudaSuccess) {
    cudaGetLastError();
    return SPLATT_ERROR_NOMEMORY;
  }

  // start: CholeskyQR2 of every start factor into the working factors; the caller's stay untouched
  double * dX = d.scal + 0, * dMu = d.scal + 1, * dRes = d.scal + 2, * dG = d.scal + 3, * dY = d.scal + 4;
  double * sgn = d.mat(7);
  ok = cudaMemsetAsync(d.bad, 0, sizeof(int), s) == cudaSuccess;
  for (int m = 0; ok && m < N; ++m) {
    const int R = ranks[m];
    ok = cudaMemcpy2DAsync(b.Z, 32 * 8, d_factors[m], (size_t)ldm * 8, (size_t)R * 8, t->dims[m],
                           cudaMemcpyDeviceToDevice, s) == cudaSuccess;
    d.cholqr2(b.Z, 32, b.F[m], ldm, t->dims[m], R, s);
  }
  // ||X||^2 with duplicates summed
  const FiberStream & fs0 = t->streams[0];
  k_xnorm_part<<<kSumCtas, kThreads, 0, s>>>(fs0.rec, fs0.nrec, d.sq);
  k_sumsq_fin<<<1, 1, 0, s>>>(d.sq, kSumCtas, dX, 0.0, nullptr);
  spb200_count_launches(2);
  int hbad = 1;
  double xsq = 0.0;
  ok = ok && (last = cudaGetLastError()) == cudaSuccess &&
       cudaMemcpyAsync(&hbad, d.bad, sizeof(int), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
       cudaMemcpyAsync(&xsq, dX, sizeof(double), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
       cudaStreamSynchronize(s) == cudaSuccess;
  if (!ok) {
    fprintf(stderr, "SPLATT: splatt_b200_tucker_hooi_device failed (%s)\n", cudaGetErrorString(last != cudaSuccess ? last : cudaGetLastError()));
    return SPLATT_ERROR_BADINPUT;
  }
  if (hbad) {
    fprintf(stderr, "SPLATT: splatt_b200_tucker_hooi_device: a start factor has dependent columns\n");
    return SPLATT_ERROR_BADINPUT;
  }
  const double xnorm = std::sqrt(xsq);

  AlsIterations ctl(options);
  uint64_t its = 0;
  std::vector<double> S(1024), V(1024), lam(32);
  const int CL = cols_but(N, ranks, N - 1), RLast = ranks[N - 1];
  for (uint64_t it = 0; ok && it < ctl.niters; ++it) {
    ctl.start();
    int power_total = 0;
    double res_max = 0.0;
    for (int n = 0; ok && n < N; ++n) {
      const int R = ranks[n], C = plan[n].a.C;
      const uint64_t I = t->dims[n];
      ok = run_ttmc(t, n, plan[n], b.packs, b.slot_row, s);
      d.sumsq(b.Y, C, C, I, dY, kMuRel, dMu, s);
      ok = ok && cudaMemcpy2DAsync(b.Qa, 32 * 8, b.F[n], (size_t)ldm * 8, (size_t)R * 8, I,
                                   cudaMemcpyDeviceToDevice, s) == cudaSuccess;
      double res = 0.0;
      int step = 0;
      while (ok && step < o.max_power) {
        // Z = Y (Y^T Qa) + mu Qa; Qb = CholeskyQR2(Z); res = ||Qb - Qa (Qa^T Qb)||_F
        d.atb(b.Y, C, b.Qa, 32, I, C, R, b.W, s);
        d.ab(b.Y, C, C, b.W, R, 0.0, dMu, b.Qa, 32, b.Z, 32, I, s);
        d.cholqr2(b.Z, 32, b.Qb, 32, I, R, s);
        d.atb(b.Qa, 32, b.Qb, 32, I, R, R, d.mat(2), s);
        d.ab(b.Qa, 32, R, d.mat(2), R, -1.0, nullptr, b.Qb, 32, b.Z, 32, I, s);
        d.sumsq(b.Z, 32, R, I, dRes, 0.0, nullptr, s);
        double hres = 0.0;
        hbad = 0;
        ok = (last = cudaGetLastError()) == cudaSuccess &&
             cudaMemcpyAsync(&hres, dRes, sizeof(double), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
             cudaMemcpyAsync(&hbad, d.bad, sizeof(int), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
             cudaStreamSynchronize(s) == cudaSuccess && !hbad;
        std::swap(b.Qa, b.Qb);
        ++step;
        res = std::sqrt(hres);
        if (res <= o.svd_tol) break;
      }
      if (!ok) break;
      power_total += step;
      res_max = std::max(res_max, res);
      // Rayleigh-Ritz: W = Y^T Q, S = W^T W = V diag(lam) V^T, U_n = Q V, signs fixed
      d.atb(b.Y, C, b.Qa, 32, I, C, R, b.W, s);
      d.atb(b.W, R, b.W, R, C, R, R, d.mat(3), s);
      ok = (last = cudaGetLastError()) == cudaSuccess &&
           cudaMemcpyAsync(S.data(), d.mat(3), (size_t)R * R * 8, cudaMemcpyDeviceToHost, s) == cudaSuccess &&
           cudaStreamSynchronize(s) == cudaSuccess;
      if (!ok) break;
      ritz_rotation(S.data(), R, V.data(), lam.data());
      ok = cudaMemcpyAsync(d.mat(4), V.data(), (size_t)R * R * 8, cudaMemcpyHostToDevice, s) == cudaSuccess;
      d.ab(b.Qa, 32, R, d.mat(4), R, 0.0, nullptr, nullptr, 0, b.F[n], ldm, I, s);
      d.fix_signs(b.F[n], ldm, R, I, sgn, s);
      if (n == N - 1) {
        // the core: G = W V with the same column signs, C_{N-1} x R_{N-1} row-major
        d.ab(b.W, R, R, d.mat(4), R, 0.0, nullptr, nullptr, 0, b.G, R, C, s);
        d.flip(b.G, R, R, C, sgn, s);
        d.sumsq(b.G, R, R, C, dG, 0.0, nullptr, s);
      }
    }
    if (!ok) break;
    double gsq = 0.0;
    ok = (last = cudaGetLastError()) == cudaSuccess &&
         cudaMemcpyAsync(&gsq, dG, sizeof(double), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaMemcpyAsync(core_out, b.G, (size_t)CL * RLast * 8, cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaStreamSynchronize(s) == cudaSuccess;
    if (!ok) break;
    const double fit = xnorm > 0.0 ? 1.0 - std::sqrt(std::max(xsq - gsq, 0.0)) / xnorm : 1.0;
    if (history) {
      history[4 * it] = fit;
      history[4 * it + 1] = std::sqrt(gsq);
      history[4 * it + 2] = power_total;
      history[4 * it + 3] = res_max;
    }
    its = it + 1;
    if (ctl.done(it, fit)) break;
  }
  if (!ok) {
    fprintf(stderr, "SPLATT: splatt_b200_tucker_hooi_device failed (%s%s)\n",
            cudaGetErrorString(last != cudaSuccess ? last : cudaGetLastError()),
            hbad ? ", CholeskyQR broke down" : "");
    cudaStreamSynchronize(s);
    return SPLATT_ERROR_BADINPUT;
  }
  // the result into the caller's factors (columns [0, R_m) only)
  for (int m = 0; ok && m < N; ++m)
    ok = cudaMemcpy2DAsync(d_factors[m], (size_t)ldm * 8, b.F[m], (size_t)ldm * 8, (size_t)ranks[m] * 8,
                           t->dims[m], cudaMemcpyDeviceToDevice, s) == cudaSuccess;
  if (!ok || cudaStreamSynchronize(s) != cudaSuccess) return SPLATT_ERROR_BADINPUT;
  if (iterations_out) *iterations_out = (int)its;
  return SPLATT_SUCCESS;
}
