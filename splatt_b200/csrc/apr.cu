// Poisson CP decomposition by CP-APR (Chi & Kolda, SIMAX 2012, multiplicative updates) on
// device-resident tensors (splatt_b200_cp_apr_device).
//
// The model M = sum_r lambda_r a_r^(1) o ... o a_r^(N) has nonnegative, column-stochastic factors;
// unstored coordinates are zero counts.  Mode n's update repeats B <- B * Phi_n with
//     Phi_n[i, :] = sum over x with i_n(x) = i of (v_x / max(B[i, :] . Pi_x, eps)) Pi_x,
// Pi_x the Hadamard product of the other modes' rows at x.  That is a root-mode traversal much
// like the MTTKRP's, and on the ALLROOT layout every mode has a root stream:
//
//   * k_apr_phi walks mode n's root stream with walk_range (walk.cuh: the root MTTKRP's
//     nnz-balanced chunk ranges, one warp per range, a private TMA record ring, the Hadamard
//     prefix in registers).  Lane l holds columns 2l, 2l + 1 of the current root row of B, loaded
//     when the slice opens, and of the row's Phi accumulator.  Per record the warp forms Pi_x, the
//     dot product B[i] . Pi_x (a 32-lane shfl_xor sum), the weight and the accumulation.
//   * A slice that lies wholly inside the warp's range is stored with plain stores.  The first
//     and the last slice of a range may be cut by a range boundary: their accumulators go into
//     one of the range's two boundary slots, and k_apr_combine adds the slots of each such row in
//     range order.  So on untiled streams Phi, lambda, the factors and the inner-iteration counts
//     are bitwise reproducible from run to run.
//   * Leaf-tiled streams (CTA-tiled, or ktile > 0) close a root row once per leaf tile; there
//     every closed (row, tile) piece is added into Phi with red.add.f64, so the order of the
//     additions, and with it the last bits of the result, may vary from run to run.
//   * The dense steps are elementwise kernels over dims[n] x R: shift + B = A diag(lambda)
//     (k_apr_scale), the KKT value max |min(B, 1 - Phi)| by atomicMax on the bit pattern of a
//     nonnegative double (exact, so deterministic; k_apr_kkt), B <- B * Phi (k_apr_mul), the
//     column sums (row-blocked, in a fixed order, k_apr_colsum_part / _fin) and the normalisation.
//   * The log-likelihood sum v log(max(m, eps)) is the model-sum kernel of completion's SSE with
//     the other per-record term (k_apr_ll).
#include "walk.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace spb200 {
namespace {

// Phi of the root mode of one stream into a.out (zeroed before).  a.mats[0] is B, the other
// levels the current factors.  ROWS: leaf-tiled stream, every closed piece is added with red.add.
template <int N, bool ROWS>
__global__ void __launch_bounds__(kThreads, 3) k_apr_phi(const TcArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int  warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool act  = 2 * lane < a.R;
  const bool hasy = 2 * lane + 1 < a.R;
  const int  RP   = a.R + (a.R & 1);
  const unsigned long long gw = static_cast<unsigned long long>(blockIdx.x) * kWarps + warp;
  double2 b    = make_double2(0.0, 0.0);
  double2 phi  = make_double2(0.0, 0.0);
  bool    open = true;    // the next record opens a slice
  bool    seen = false;   // this warp closed a slice already: later ones (but the last) are whole
  walk_range<N, 1, true>(a, smem, act, [&](double v, double2 h, bool close, uint32_t row, bool last) {
    if (open) {
      if (act) b = reinterpret_cast<const double2 *>(a.mats[0] + static_cast<size_t>(row) * a.ldm)[lane];
      if (!hasy) b.y = 0.0;
      open = false;
    }
    if (!hasy) h.y = 0.0;                   // column R of an odd rank never feeds the result
    double d = b.x * h.x;
    d = fma(b.y, h.y, d);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    phi = vfma(v / fmax(d, a.eps), h, phi);
    if (!close) return;
    open = true;
    if (act) {
      if constexpr (ROWS) {
        double * dst = a.out + static_cast<size_t>(row) * a.ldm + 2 * lane;
        atomicAdd(dst, phi.x);
        if (hasy) atomicAdd(dst + 1, phi.y);
      } else if (!seen || last) {
        const unsigned long long slot = 2 * gw + (seen ? 1 : 0);
        reinterpret_cast<double2 *>(a.packs + slot * RP)[lane] = phi;
        if (lane == 0) a.slot_row[slot] = row;
      } else {
        double * dst = a.out + static_cast<size_t>(row) * a.ldm + 2 * lane;
        dst[0] = phi.x;
        if (hasy) dst[1] = phi.y;
      }
    }
    seen = true;
    phi  = make_double2(0.0, 0.0);
  });
}

// Adds the boundary slots of every row the Phi kernel left there, in range order (the warp of a
// row's first slot adds all its slots), and stores the row.
__global__ void __launch_bounds__(kThreads) k_apr_combine(const double * __restrict__ packs,
                                                          const uint32_t * __restrict__ slot_row,
                                                          unsigned long long nslots, int R, int ldm,
                                                          double * __restrict__ out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int RP = R + (R & 1);
  const unsigned long long TW = static_cast<unsigned long long>(gridDim.x) * kWarps;
  for (unsigned long long s = static_cast<unsigned long long>(blockIdx.x) * kWarps + warp; s < nslots;
       s += TW) {
    const uint32_t row = slot_row[s];
    if (row == kEmptySlot) continue;
    long long t = static_cast<long long>(s) - 1;
    while (t >= 0 && slot_row[t] == kEmptySlot) --t;
    if (t >= 0 && slot_row[t] == row) continue;          // not the row's first slot
    double x0 = 0.0, x1 = 0.0;
    for (unsigned long long u = s; u < nslots; ++u) {
      const uint32_t r2 = slot_row[u];
      if (r2 == kEmptySlot) continue;
      if (r2 != row) break;
      const double * src = packs + u * RP;
      if (lane < R) x0 += src[lane];
      if (lane + 32 < R) x1 += src[lane + 32];
    }
    double * dst = out + static_cast<size_t>(row) * ldm;
    if (lane < R) dst[lane] = x0;
    if (lane + 32 < R) dst[lane + 32] = x1;
  }
}

// Grid-stride loop over the entries (i, c), c < R, of a rows x ldm matrix.
#define APR_FOR_ENTRIES(rows, R)                                                                   \
  for (unsigned long long e = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x, \
                          n_ = (rows) * static_cast<unsigned long long>(R);                          \
       e < n_; e += static_cast<unsigned long long>(gridDim.x) * blockDim.x)

// B = (A + kappa [A < kappa_tol and Phi > 1 and shift]) diag(lambda)
__global__ void __launch_bounds__(kThreads) k_apr_scale(const double * __restrict__ A, const double * __restrict__ Phi,
                                                        const double * __restrict__ lam, double * __restrict__ B,
                                                        unsigned long long rows, int R, int ldm, double kappa,
                                                        double kappa_tol, int shift) {
  APR_FOR_ENTRIES(rows, R) {
    const size_t k = (e / R) * ldm + e % R;
    double x = A[k];
    if (shift && x < kappa_tol && Phi[k] > 1.0) x += kappa;
    B[k] = x * lam[e % R];
  }
}

// *kkt = max(*kkt, max |min(B, 1 - Phi)|) on the bit patterns of nonnegative doubles
__global__ void __launch_bounds__(kThreads) k_apr_kkt(const double * __restrict__ B, const double * __restrict__ Phi,
                                                      unsigned long long rows, int R, int ldm,
                                                      unsigned long long * kkt) {
  double m = 0.0;
  APR_FOR_ENTRIES(rows, R) {
    const size_t k = (e / R) * ldm + e % R;
    m = fmax(m, fabs(fmin(B[k], 1.0 - Phi[k])));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(kkt, static_cast<unsigned long long>(__double_as_longlong(m)));
}

// B <- B * Phi
__global__ void __launch_bounds__(kThreads) k_apr_mul(double * __restrict__ B, const double * __restrict__ Phi,
                                                      unsigned long long rows, int R, int ldm) {
  APR_FOR_ENTRIES(rows, R) {
    const size_t k = (e / R) * ldm + e % R;
    B[k] *= Phi[k];
  }
}

// out = in diag(1 / lam); a column with lam = 0 becomes 0 (in == out allowed)
__global__ void __launch_bounds__(kThreads) k_apr_normalize(const double * in, const double * __restrict__ lam,
                                                            double * out, unsigned long long rows, int R, int ldm) {
  APR_FOR_ENTRIES(rows, R) {
    const size_t k = (e / R) * ldm + e % R;
    const double l = lam[e % R];
    out[k] = l > 0.0 ? in[k] / l : 0.0;
  }
}

// *bad = 1 if an entry (i, c), c < R, of p (row stride `stride` doubles) is negative or not finite
__global__ void __launch_bounds__(kThreads) k_apr_check(const double * __restrict__ p, unsigned long long rows,
                                                        int R, int stride, int * bad) {
  bool b = false;
  APR_FOR_ENTRIES(rows, R) {
    const double x = p[(e / R) * stride + e % R];
    b |= !(x >= 0.0 && x <= 1.7976931348623157e308);
  }
  if (__any_sync(0xffffffffu, b) && (threadIdx.x & 31) == 0) atomicExch(bad, 1);
}

// Column sums in two passes with a fixed order (deterministic): CTA g of kColsumCtas sums the
// rows [rows g / G, rows (g + 1) / G), thread t column t % 64 of every 4th row from t / 64 (a
// warp reads 32 adjacent columns of one row), and the four partials in order into part[g][c];
// k_apr_colsum_fin adds the CTAs' partials in order.
constexpr int kColsumCtas = 256;
__global__ void __launch_bounds__(kThreads) k_apr_colsum_part(const double * __restrict__ M, unsigned long long rows,
                                                              int R, int ldm, double * __restrict__ part) {
  __shared__ double sh[kThreads];
  const int c = threadIdx.x % 64, q = threadIdx.x / 64;
  const unsigned long long lo = rows * blockIdx.x / gridDim.x, hi = rows * (blockIdx.x + 1) / gridDim.x;
  double s = 0.0;
  if (c < R)
    for (unsigned long long i = lo + q; i < hi; i += kThreads / 64) s += M[i * ldm + c];
  sh[threadIdx.x] = s;
  __syncthreads();
  if (q == 0 && c < R) part[blockIdx.x * 64 + c] = ((sh[c] + sh[64 + c]) + sh[128 + c]) + sh[192 + c];
}
__global__ void __launch_bounds__(64) k_apr_colsum_fin(const double * __restrict__ part, int nparts, int R,
                                                       double * __restrict__ out) {
  const int c = threadIdx.x;
  if (c >= R) return;
  double s = 0.0;
  for (int g = 0; g < nparts; ++g) s += part[g * 64 + c];
  out[c] = s;
}

// Sum over this grid's ranges of the stream of v log(max(sum_r lambda_r prod_m A_m[i_m, r], eps))
template <int N>
__global__ void __launch_bounds__(kThreads, 3) k_apr_ll(const TcArgs a) {
  const double eps = a.eps;
  model_sum<N>(a, [eps](double s, double v, double x) { return fma(v, log(fmax(x, eps)), s); });
}

// ---- PDNR: projected damped Newton on the rows ----------------------------------------------------
//
// splatt_b200_cp_apr_pdnr_device (Hansen, Plantenga & Kolda, OMS 2015).  Row i of B = A_n diag(lambda)
// minimises f_i(b) = sum_r b_r - sum_{x in X_i} v_x log(max(b . Pi_x, eps)) on its own, so one
// lockstep iteration of mode n is:
//   * k_pdnr_grad walks mode n's root stream like k_apr_phi and, for every row still to be
//     evaluated (state 1), accumulates per record w Pi_x (w = v / max(m, eps)) and, with
//     k_tc_update's pair-row accumulation, h h^T with h = (sqrt(v) / max(m, eps)) Pi_x: the
//     Hessian.  A whole slice is finished in the warp where it closes (pdnr_step: g, kkt, the
//     epsilon-active set, the reduced damped Cholesky solve, the direction); the first and last
//     slice of a range go to boundary slots and k_pdnr_solve adds them in range order and runs
//     pdnr_step.  k_pdnr_solve also serves the rows without records (g = 1, H = 0) and, on
//     leaf-tiled streams, every row from its red.add-accumulated pack.
//   * k_pdnr_ladder walks the stream again for the rows with a direction (state 2) and sums, for
//     all kPdnrTrials trial points b_k = max(b + 2^-k d, 0) at once, v log(m_k / m) with
//     m = b . Pi_x and m_k - m = (b_k - b) . Pi_x.  The eight dot products per record are reduced
//     by a transposed butterfly (9 shuffles, lane group k ends with sum k) instead of 8 warp sums.
//     Cut slices go through boundary slots and k_apr_combine, leaf-tiled pieces through red.add.
//   * k_pdnr_accept, one thread per row: f(b_k) - f(b) = sum_r (b_k - b)_r - (ladder sum k), the
//     smallest k that passes the Armijo and the decrease test, the damping, and the count of rows
//     that attempted a step (the host reads it once per lockstep iteration).

constexpr int    kPdnrTrials = 8;       // trial points the ladder scores (the largest max_backtrack)
constexpr double kArmijo     = 1e-4;
constexpr double kDamping    = 3.5;

// Row states: 0 stopped (kkt < tol), 1 to be evaluated by the next gradient walk, 2 has a
// direction for the ladder and the accept.
struct PdnrArgs {
  TcArgs          w;           // the walk: mats[0] = B, eps, packs / slot_row
  double *        D;           // rows x ldm: the direction of every row in state 2
  double *        G;           // rows x ldm: the gradient of every row in state 2
  double *        lad;         // rows x kPdnrTrials: sum_x v log(m_k / m)
  double *        kkt;         // rows: the last kkt of every row
  const double *  mu;          // rows: the damping
  int *           state;       // rows
  unsigned char * mark;        // rows: 1 when the row has a record (set by every gradient walk)
  double          tol, eps_active;
};

// doubles per warp of the gradient walk / solve workspace: the pack (2 NP + RT: the pair rows and
// sum w Pi), h, b and the right-hand side / solution
__host__ __device__ constexpr int pdnr_ws_doubles(int RT) { return 2 * tc_pairs(RT / 2) + 4 * RT; }
__host__ __device__ constexpr size_t pdnr_tab_bytes(int RT) { return (sizeof(uint32_t) * tc_pairs(RT / 2) + 15) & ~size_t(15); }
__host__ __device__ constexpr size_t pdnr_grad_smem(int RT) {
  return tc_ring_bytes() + pdnr_tab_bytes(RT) + sizeof(double) * kWarps * pdnr_ws_doubles(RT);
}
__host__ __device__ constexpr int pdnr_minb(int RT) { return RT <= 32 ? 2 : 1; }

// Trial point k of b along d: max(b + 2^-k d, 0).  The ladder and the accept use this one
// expression, so both see bitwise the same point.
__device__ __forceinline__ double pdnr_trial(double b, double d, int k) {
  return fmax(fma(1.0 / static_cast<double>(1 << k), d, b), 0.0);
}

// One row's Newton step, one warp.  W: the row's pack (pair rows of H, then sum w Pi at
// W + 2 tc_pairs(H)); bv, xv: R doubles of scratch each.  Computes g = 1 - sum w Pi and
// kkt = max |min(b, g)|; stops the row when kkt < tol; else the epsilon-active set
// A = {r: b_r <= min(eps_active, ||b - max(b - g, 0)||), g_r > 0}, d_A = -g_A and
// (H_FF + mu I) d_F = -g_F by Cholesky over the free indices only (d = -g when a pivot is <= 0
// or not finite), and stores d, g and state 2.  (The arguments are passed by value: a reference
// to the kernel's parameters would copy them to the stack.)
__device__ __noinline__ void pdnr_step(double * W, int R, int H, uint32_t row, const double * __restrict__ B,
                                       double * __restrict__ D, double * __restrict__ G, int ldm,
                                       double * __restrict__ kkt_out, const double * __restrict__ mu_in,
                                       int * __restrict__ state, double tol, double eps_active,
                                       double * bv, double * xv) {
  const int lane = threadIdx.x & 31;
  double *  g    = W + 2 * tc_pairs(H);
  auto A = [&](int i, int j) -> double & { return W[2 * pair_base(i, H) + j - (i & ~1)]; };
  const double * brow = B + static_cast<size_t>(row) * ldm;
  double kkt = 0.0, e2 = 0.0;
  for (int j = lane; j < R; j += 32) {
    const double bj = brow[j], gj = 1.0 - g[j];
    g[j] = gj;
    bv[j] = bj;
    kkt = fmax(kkt, fabs(fmin(bj, gj)));
    const double t = bj - fmax(bj - gj, 0.0);
    e2 = fma(t, t, e2);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    kkt = fmax(kkt, __shfl_xor_sync(0xffffffffu, kkt, o));
    e2 += __shfl_xor_sync(0xffffffffu, e2, o);
  }
  if (lane == 0) kkt_out[row] = kkt;
  if (kkt < tol) {
    if (lane == 0) state[row] = 0;
    __syncwarp();
    return;
  }
  const double ei = fmin(eps_active, sqrt(e2));
  const unsigned lo = __ballot_sync(0xffffffffu, lane < R && bv[lane] <= ei && g[lane] > 0.0);
  const unsigned hi = __ballot_sync(0xffffffffu, lane + 32 < R && bv[lane + 32] <= ei && g[lane + 32] > 0.0);
  const unsigned long long act = lo | static_cast<unsigned long long>(hi) << 32;
  auto free_ = [act](int j) { return !((act >> j) & 1ull); };
  const double mu = mu_in[row];
  for (int j = lane; j < R; j += 32) {
    xv[j] = -g[j];
    if (free_(j)) A(j, j) += mu;
  }
  __syncwarp();
  bool ok = true;
  for (int k = 0; k < R; ++k) {                // H_FF + mu I = U^T U over the free indices
    if (!free_(k)) continue;
    const double piv = A(k, k);
    if (!(piv > 0.0 && piv <= 1.7976931348623157e308)) { ok = false; break; }
    const double d = sqrt(piv);
    __syncwarp();
    const double inv = 1.0 / d;
    for (int j = k + 1 + lane; j < R; j += 32)
      if (free_(j)) A(k, j) *= inv;
    if (lane == 0) A(k, k) = d;
    __syncwarp();
    for (int i = k + 1; i < R; ++i) {
      if (!free_(i)) continue;
      const double aki = A(k, i);
      for (int j = i + lane; j < R; j += 32)
        if (free_(j)) A(i, j) = fma(-aki, A(k, j), A(i, j));
    }
    __syncwarp();
  }
  __syncwarp();
  if (ok) {
    for (int k = 0; k < R; ++k) {              // U^T y = -g_F
      if (!free_(k)) continue;
      const double yk = xv[k] / A(k, k);
      __syncwarp();
      for (int j = k + 1 + lane; j < R; j += 32)
        if (free_(j)) xv[j] = fma(-A(k, j), yk, xv[j]);
      if (lane == 0) xv[k] = yk;
      __syncwarp();
    }
    for (int k = R - 1; k >= 0; --k) {         // U d_F = y
      if (!free_(k)) continue;
      const double xk = xv[k] / A(k, k);
      __syncwarp();
      for (int i = lane; i < k; i += 32)
        if (free_(i)) xv[i] = fma(-A(i, k), xk, xv[i]);
      if (lane == 0) xv[k] = xk;
      __syncwarp();
    }
  }
  double * drow = D + static_cast<size_t>(row) * ldm;
  double * grow = G + static_cast<size_t>(row) * ldm;
  for (int j = lane; j < R; j += 32) {
    drow[j] = ok ? xv[j] : -g[j];
    grow[j] = g[j];
  }
  if (lane == 0) state[row] = 2;
  __syncwarp();
}

// pdnr_step of row `row` with the pack at W
__device__ __forceinline__ void pdnr_step(double * W, int H, uint32_t row, const PdnrArgs & p, double * bv,
                                          double * xv) {
  pdnr_step(W, p.w.R, H, row, p.w.mats[0], p.D, p.G, p.w.ldm, p.kkt, p.mu, p.state, p.tol, p.eps_active, bv, xv);
}

// Gradient and Hessian walk of the root mode of one stream (RT: the rank tier, the Hessian's
// pair rows in registers at 16 and in per-warp shared memory at 32 / 64; ROWS: leaf-tiled
// stream, every closed piece is added into its row's pack with red.add).
template <int N, int RT, bool ROWS>
__global__ void __launch_bounds__(kThreads, pdnr_minb(RT)) k_pdnr_grad(const PdnrArgs p) {
  constexpr int  HM  = RT / 2;
  constexpr int  S   = (tc_pairs(HM) + 31) / 32;   // pairs per lane
  constexpr bool REG = (RT <= 16);
  const TcArgs & a = p.w;
  extern __shared__ __align__(128) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int RP = a.R + (a.R & 1), H = RP / 2, NPr = tc_pairs(H), P = 2 * NPr + RP;
  uint32_t * tab = reinterpret_cast<uint32_t *>(smem + tc_ring_bytes());
  double *   ws  = reinterpret_cast<double *>(smem + tc_ring_bytes() + pdnr_tab_bytes(RT)) +
                   warp * pdnr_ws_doubles(RT);
  double2 *  W2  = reinterpret_cast<double2 *>(ws);
  double *   hs  = ws + 2 * tc_pairs(HM) + RT;
  double *   bv  = hs + RT;
  double *   xv  = bv + RT;

  // pair p -> (row i, first column j0): i in bits 0..15, j0 / 2 in bits 16..31
  for (int i = warp; i < RP; i += kWarps)
    for (int q = lane; q < H - i / 2; q += 32) tab[pair_base(i, H) + q] = uint32_t(i) | uint32_t(i / 2 + q) << 16;
  for (int q = lane; q < P; q += 32) ws[q] = 0.0;
  __syncthreads();

  const bool act  = 2 * lane < a.R;
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
  double2 b    = make_double2(0.0, 0.0);
  double2 gw   = make_double2(0.0, 0.0);
  bool    open = true;    // the next record opens a slice
  bool    live = false;   // the open slice's row is to be evaluated
  bool    seen = false;   // this warp closed a slice already: later ones (but the last) are whole
  const unsigned long long gwarp = static_cast<unsigned long long>(blockIdx.x) * kWarps + warp;

  walk_range<N, 1, true>(a, smem, act, [&](double v, double2 h, bool close, uint32_t row, bool last) {
    if (open) {
      live = p.state[row] == 1;
      if (live && act) b = reinterpret_cast<const double2 *>(a.mats[0] + static_cast<size_t>(row) * a.ldm)[lane];
      if (!hasy) b.y = 0.0;
      if (lane == 0) p.mark[row] = 1;
      open = false;
    }
    if (live) {
      if (!hasy) h.y = 0.0;                 // column R of an odd rank never feeds the result
      double m = b.x * h.x;
      m = fma(b.y, h.y, m);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m += __shfl_xor_sync(0xffffffffu, m, o);
      const double mm = fmax(m, a.eps);
      gw = vfma(v / mm, h, gw);
      if (act) reinterpret_cast<double2 *>(hs)[lane] = vmul(sqrt(v) / mm, h);
      __syncwarp();
#pragma unroll
      for (int k = 0; k < S; ++k) {
        const int q = k * 32 + lane;
        if (q < NPr) {
          const uint32_t e  = REG ? ent[k] : tab[q];
          const double   hi = hs[e & 0xffffu];
          const double2  hj = reinterpret_cast<const double2 *>(hs)[e >> 16];
          if constexpr (REG) acc[k] = vfma(hi, hj, acc[k]);
          else W2[q] = vfma(hi, hj, W2[q]);
        }
      }
      __syncwarp();                         // h is rewritten by the next record
    }
    if (!close) return;
    open = true;
    if (live) {
      if constexpr (REG) {
#pragma unroll
        for (int k = 0; k < S; ++k) {
          if (k * 32 + lane < NPr) W2[k * 32 + lane] = acc[k];
          acc[k] = make_double2(0.0, 0.0);
        }
      }
      if (act) reinterpret_cast<double2 *>(ws + 2 * NPr)[lane] = gw;
      gw = make_double2(0.0, 0.0);
      __syncwarp();
      if constexpr (ROWS) {
        double * dst = a.packs + static_cast<size_t>(row) * P;
        for (int q = lane; q < P; q += 32) atomicAdd(dst + q, ws[q]);
      } else if (!seen || last) {
        const unsigned long long slot = 2 * gwarp + (seen ? 1 : 0);
        double * dst = a.packs + slot * P;
        for (int q = lane; q < P; q += 32) dst[q] = ws[q];
        if (lane == 0) a.slot_row[slot] = row;
      } else {
        pdnr_step(ws, H, row, p, bv, xv);
      }
      __syncwarp();
      for (int q = lane; q < P; q += 32) ws[q] = 0.0;
      __syncwarp();
    }
    seen = true;
  });
}

// The Newton step of the rows the gradient walk left: with slot_row, every row of the boundary
// slots (the warp of a row's first slot adds all its slots, in range order), then every row in
// state 1 without a record (g = 1, H = 0); without slot_row (leaf-tiled), every row in state 1
// from its pack.
template <int RT>
__global__ void __launch_bounds__(kThreads) k_pdnr_solve(const PdnrArgs p, unsigned long long nslots,
                                                         unsigned long long rows) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int RP = p.w.R + (p.w.R & 1), H = RP / 2, P = 2 * tc_pairs(H) + RP;
  double *  ws = reinterpret_cast<double *>(smem) + warp * pdnr_ws_doubles(RT);
  double *  bv = ws + 2 * tc_pairs(RT / 2) + 2 * RT;
  double *  xv = bv + RT;
  const uint32_t * slot_row = p.w.slot_row;
  const unsigned long long TW = static_cast<unsigned long long>(gridDim.x) * kWarps;
  const unsigned long long nitems = (slot_row ? nslots : 0) + rows;
  for (unsigned long long s = static_cast<unsigned long long>(blockIdx.x) * kWarps + warp; s < nitems;
       s += TW) {
    uint32_t row;
    if (slot_row && s < nslots) {
      row = slot_row[s];
      if (row == kEmptySlot) continue;
      long long t = static_cast<long long>(s) - 1;
      while (t >= 0 && slot_row[t] == kEmptySlot) --t;
      if (t >= 0 && slot_row[t] == row) continue;          // not the row's first slot
      for (int q = lane; q < P; q += 32) ws[q] = 0.0;
      for (unsigned long long u = s; u < nslots; ++u) {
        const uint32_t r2 = slot_row[u];
        if (r2 == kEmptySlot) continue;
        if (r2 != row) break;
        const double * src = p.w.packs + u * P;
        for (int q = lane; q < P; q += 32) ws[q] += src[q];
      }
    } else {
      row = static_cast<uint32_t>(slot_row ? s - nslots : s);
      if (p.state[row] != 1 || (slot_row && p.mark[row])) continue;
      const double * src = p.w.packs + static_cast<size_t>(row) * P;
      for (int q = lane; q < P; q += 32) ws[q] = slot_row ? 0.0 : src[q];
    }
    __syncwarp();
    pdnr_step(ws, H, row, p, bv, xv);
  }
}

// For every row with a direction, sum_x v log(max(m_k, eps) / max(m, eps)) over the trial points
// k < kPdnrTrials into lad (ROWS: leaf-tiled stream, pieces added with red.add).
template <int N, bool ROWS>
__global__ void __launch_bounds__(kThreads, 2) k_pdnr_ladder(const PdnrArgs p) {
  const TcArgs & a = p.w;
  extern __shared__ __align__(128) unsigned char smem[];
  const int  warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool act  = 2 * lane < a.R;
  const bool hasy = 2 * lane + 1 < a.R;
  // after the butterfly, lane group (lane & ~3) holds the sum of trial point k
  const int  kown = ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1);
  const unsigned long long gwarp = static_cast<unsigned long long>(blockIdx.x) * kWarps + warp;
  double2 b = make_double2(0.0, 0.0);
  double2 t[kPdnrTrials];                  // b_k - b, the lane's two columns
#pragma unroll
  for (int k = 0; k < kPdnrTrials; ++k) t[k] = make_double2(0.0, 0.0);
  double acc  = 0.0;
  bool   open = true, live = false, seen = false;
  walk_range<N, 1, true>(a, smem, act, [&](double v, double2 h, bool close, uint32_t row, bool last) {
    if (open) {
      live = p.state[row] == 2;
      if (live) {
        double2 d = make_double2(0.0, 0.0);
        if (act) {
          b = reinterpret_cast<const double2 *>(a.mats[0] + static_cast<size_t>(row) * a.ldm)[lane];
          d = reinterpret_cast<const double2 *>(p.D + static_cast<size_t>(row) * a.ldm)[lane];
        }
        if (!hasy) b.y = d.y = 0.0;
#pragma unroll
        for (int k = 0; k < kPdnrTrials; ++k)
          t[k] = make_double2(pdnr_trial(b.x, d.x, k) - b.x, pdnr_trial(b.y, d.y, k) - b.y);
      }
      open = false;
    }
    if (live) {
      if (!hasy) h.y = 0.0;
      double m = b.x * h.x;
      m = fma(b.y, h.y, m);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m += __shfl_xor_sync(0xffffffffu, m, o);
      double q[kPdnrTrials];
#pragma unroll
      for (int k = 0; k < kPdnrTrials; ++k) q[k] = fma(t[k].y, h.y, t[k].x * h.x);
      // reduce-scatter: each round keeps half of the sums and sends the other half
      {
        const bool up = lane & 16;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const double send = up ? q[i] : q[i + 4], keep = up ? q[i + 4] : q[i];
          q[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
        }
      }
      {
        const bool up = lane & 8;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const double send = up ? q[i] : q[i + 2], keep = up ? q[i + 2] : q[i];
          q[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
        }
      }
      {
        const bool up = lane & 4;
        const double send = up ? q[0] : q[1], keep = up ? q[1] : q[0];
        q[0] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
      }
      q[0] += __shfl_xor_sync(0xffffffffu, q[0], 2);
      q[0] += __shfl_xor_sync(0xffffffffu, q[0], 1);
      const double mk = m + q[0];
      const double lr = (m >= a.eps && mk >= a.eps) ? log1p(q[0] / m) : log(fmax(mk, a.eps)) - log(fmax(m, a.eps));
      acc = fma(v, lr, acc);
    }
    if (!close) return;
    open = true;
    if (live && (lane & 3) == 0) {
      if constexpr (ROWS) {
        atomicAdd(p.lad + static_cast<size_t>(row) * kPdnrTrials + kown, acc);
      } else if (!seen || last) {
        const unsigned long long slot = 2 * gwarp + (seen ? 1 : 0);
        a.packs[slot * kPdnrTrials + kown] = acc;
        if (lane == 0) a.slot_row[slot] = row;
      } else {
        p.lad[static_cast<size_t>(row) * kPdnrTrials + kown] = acc;
      }
    }
    acc  = 0.0;
    seen = true;
  });
}

// The line search's decision for every row with a direction (one thread per row): the smallest
// k < K with df_k <= 1e-4 g.(b_k - b) and df_k <= 0, df_k = sum_r (b_k - b)_r - lad[k]; b <- b_k
// and the damping; the row goes back to state 1 and is counted into *count.
__global__ void __launch_bounds__(kThreads) k_pdnr_accept(double * __restrict__ B, const double * __restrict__ D,
                                                          const double * __restrict__ G,
                                                          const double * __restrict__ lad, double * __restrict__ mu,
                                                          int * __restrict__ state, unsigned long long rows, int R,
                                                          int ldm, int K, double mu0, int * count) {
  int n = 0;
  for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; i < rows;
       i += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
    if (state[i] != 2) continue;
    double * b = B + i * ldm;
    const double * d = D + i * ldm;
    const double * g = G + i * ldm;
    double ds[kPdnrTrials], gd[kPdnrTrials];
#pragma unroll
    for (int k = 0; k < kPdnrTrials; ++k) ds[k] = gd[k] = 0.0;
    for (int r = 0; r < R; ++r) {
      const double br = b[r], dr = d[r], gr = g[r];
#pragma unroll
      for (int k = 0; k < kPdnrTrials; ++k) {
        const double s = pdnr_trial(br, dr, k) - br;
        ds[k] += s;
        gd[k] = fma(gr, s, gd[k]);
      }
    }
    int acc = -1;
#pragma unroll
    for (int k = 0; k < kPdnrTrials; ++k) {
      const double df = ds[k] - lad[i * kPdnrTrials + k];
      if (acc < 0 && k < K && df <= kArmijo * gd[k] && df <= 0.0) acc = k;
    }
    if (acc >= 0)
      for (int r = 0; r < R; ++r) b[r] = pdnr_trial(b[r], d[r], acc);
    mu[i] = acc == 0 ? fmax(mu[i] / kDamping, mu0) : mu[i] * kDamping;
    state[i] = 1;
    ++n;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
  if ((threadIdx.x & 31) == 0 && n) atomicAdd(count, n);
}

// Every row of a mode: state 1 (to be evaluated) and damping mu0.
__global__ void __launch_bounds__(kThreads) k_pdnr_init(double * __restrict__ mu, int * __restrict__ state,
                                                        unsigned long long rows, double mu0) {
  for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; i < rows;
       i += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
    mu[i] = mu0;
    state[i] = 1;
  }
}

// *bits = max(*bits, max of kkt[0..rows)) on the bit patterns of nonnegative doubles
__global__ void __launch_bounds__(kThreads) k_pdnr_kktmax(const double * __restrict__ kkt, unsigned long long rows,
                                                          unsigned long long * bits) {
  double m = 0.0;
  for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; i < rows;
       i += static_cast<unsigned long long>(gridDim.x) * blockDim.x)
    m = fmax(m, kkt[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(bits, static_cast<unsigned long long>(__double_as_longlong(m)));
}

// ---- PQNR: projected quasi-Newton (L-BFGS) on the rows ---------------------------------------------
//
// splatt_b200_cp_apr_pqnr_device.  The row problems of PDNR, with the direction from L-BFGS pairs
// instead of the Hessian.  The gradient is 1 - Phi, and Phi is MU's, so one lockstep iteration
// of mode n is k_apr_phi (+ k_apr_combine), k_pqnr_step for every row in state 1 (the pair
// update and the direction), and -- when some row got a direction -- PDNR's k_pdnr_ladder
// (+ k_apr_combine) and k_pdnr_accept.  The accept's damping goes to a scratch buffer PQNR never
// reads.

constexpr int kPqnrMaxMem = 8;          // the largest lbfgs_mem
constexpr int kPqnrRounds = 3;          // continuation rounds before a row gives up

// Per-row state of the quasi-Newton rows.  Pair slot k of row i is at S / Y + k * slot + i * ldm
// (slot = max dims x ldm: a warp's row loads stay coalesced) and rho[k * rows_max + i].
struct PqnrArgs {
  const double * phi;          // rows x ldm: Phi at b
  const double * B;            // rows x ldm: b
  double *       D;            // rows x ldm: the direction (state 2)
  double *       G;            // rows x ldm: g at b_prev, the accept's gradient
  double *       Bp;           // rows x ldm: b_prev
  double *       S;            // lbfgs_mem x slot
  double *       Y;            // lbfgs_mem x slot
  double *       rho;          // lbfgs_mem x rows_max: 1 / s.y
  int *          head;         // rows: the ring slot the next pair goes to
  int *          npairs;       // rows: pairs stored (<= lbfgs_mem)
  int *          lev;          // rows: continuation level; -1 before the row's first step
  int *          state;        // rows: 0 stopped, 1 to be evaluated, 2 has a direction
  double *       kkt;          // rows: the last kkt
  int *          count;        // rows that got a direction
  unsigned long long rows, rows_max;
  size_t         slot;
  int            R, ldm, mem, max_backtrack;
  double         tol, eps_active;
};

__device__ __forceinline__ double pqnr_wsum(double x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}
__device__ __forceinline__ double pqnr_dot(double2 a, double2 b) { return pqnr_wsum(fma(a.y, b.y, a.x * b.x)); }

// One warp per row in state 1; lane l holds columns 2l, 2l + 1.  g = 1 - Phi and kkt; a row below
// tol stops.  If the last line search left b bitwise unchanged, the level rises (the row stops at
// kPqnrRounds) and d continues the halving (d <- 2^-max_backtrack d); otherwise the pair
// (b - b_prev, g - g_prev) is stored when s.y > 0 and 1 / s.y is finite, and d comes from the
// two-loop recursion on q = -g with q_A = 0, then d_A = -g_A (d = -g when not finite).  Stores
// d, g and b as b_prev and g_prev, state 2, and adds the rows with a direction to *count.
__global__ void __launch_bounds__(kThreads) k_pqnr_step(const PqnrArgs q) {
  const int  warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool act  = 2 * lane < q.R;
  const bool hasy = 2 * lane + 1 < q.R;
  const int  mem  = q.mem;
  int n = 0;
  for (unsigned long long row = static_cast<unsigned long long>(blockIdx.x) * kWarps + warp; row < q.rows;
       row += static_cast<unsigned long long>(gridDim.x) * kWarps) {
    if (q.state[row] != 1) continue;
    const size_t o = static_cast<size_t>(row) * q.ldm;
    auto ld = [&](const double * base) {
      double2 x = act ? reinterpret_cast<const double2 *>(base + o)[lane] : make_double2(0.0, 0.0);
      if (!hasy) x.y = 0.0;
      return x;
    };
    auto st = [&](double * base, double2 x) {
      if (act) reinterpret_cast<double2 *>(base + o)[lane] = x;
    };
    const double2 b  = ld(q.B);
    const double2 ph = ld(q.phi);
    const double2 g  = make_double2(act ? 1.0 - ph.x : 0.0, hasy ? 1.0 - ph.y : 0.0);
    double kkt = fmax(fabs(fmin(b.x, g.x)), fabs(fmin(b.y, g.y)));
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) kkt = fmax(kkt, __shfl_xor_sync(0xffffffffu, kkt, s));
    if (lane == 0) q.kkt[row] = kkt;
    if (kkt < q.tol) {
      if (lane == 0) q.state[row] = 0;
      continue;
    }
    int lev = q.lev[row];
    bool same = false;
    double2 bp = make_double2(0.0, 0.0);
    if (lev >= 0) {
      bp = ld(q.Bp);
      const bool eq = __double_as_longlong(b.x) == __double_as_longlong(bp.x) &&
                      __double_as_longlong(b.y) == __double_as_longlong(bp.y);
      same = __ballot_sync(0xffffffffu, !eq) == 0u;
    }
    double2 d;
    if (same) {
      if (++lev == kPqnrRounds) {
        if (lane == 0) { q.lev[row] = lev; q.state[row] = 0; }
        continue;
      }
      const double h = ldexp(1.0, -q.max_backtrack);
      d = ld(q.D);
      d = make_double2(h * d.x, h * d.y);
    } else {
      int head = q.head[row], np = q.npairs[row];
      if (lev >= 0) {
        const double2 gp  = ld(q.G);
        const double2 s   = make_double2(b.x - bp.x, b.y - bp.y);
        const double2 y   = make_double2(g.x - gp.x, g.y - gp.y);
        const double  sty = pqnr_dot(s, y);
        const double  r   = 1.0 / sty;
        if (sty > 0.0 && isfinite(r)) {
          const size_t k = static_cast<size_t>(head) * q.slot;
          st(q.S + k, s);
          st(q.Y + k, y);
          if (lane == 0) q.rho[static_cast<size_t>(head) * q.rows_max + row] = r;
          head = head + 1 == mem ? 0 : head + 1;
          np   = min(np + 1, mem);
        }
      }
      lev = 0;
      const double tx = b.x - fmax(b.x - g.x, 0.0), ty = b.y - fmax(b.y - g.y, 0.0);
      const double ei = fmin(q.eps_active, sqrt(pqnr_wsum(fma(ty, ty, tx * tx))));
      const bool ax = act && b.x <= ei && g.x > 0.0;
      const bool ay = hasy && b.y <= ei && g.y > 0.0;
      double2 v = make_double2(ax ? 0.0 : -g.x, ay ? 0.0 : -g.y);
      double alpha[kPqnrMaxMem];
      double gamma = 1.0;
#pragma unroll
      for (int i = 0; i < kPqnrMaxMem; ++i) {  // newest to oldest
        if (i < np) {
          const int k = (head - 1 - i + 2 * mem) % mem;
          const double2 sk = ld(q.S + static_cast<size_t>(k) * q.slot);
          const double2 yk = ld(q.Y + static_cast<size_t>(k) * q.slot);
          if (i == 0) gamma = pqnr_dot(sk, yk) / pqnr_dot(yk, yk);
          alpha[i] = q.rho[static_cast<size_t>(k) * q.rows_max + row] * pqnr_dot(sk, v);
          v = make_double2(fma(-alpha[i], yk.x, v.x), fma(-alpha[i], yk.y, v.y));
        }
      }
      v = make_double2(gamma * v.x, gamma * v.y);
#pragma unroll
      for (int i = kPqnrMaxMem - 1; i >= 0; --i) {   // oldest to newest
        if (i < np) {
          const int k = (head - 1 - i + 2 * mem) % mem;
          const double2 sk = ld(q.S + static_cast<size_t>(k) * q.slot);
          const double2 yk = ld(q.Y + static_cast<size_t>(k) * q.slot);
          const double beta = q.rho[static_cast<size_t>(k) * q.rows_max + row] * pqnr_dot(yk, v);
          v = make_double2(fma(alpha[i] - beta, sk.x, v.x), fma(alpha[i] - beta, sk.y, v.y));
        }
      }
      d = make_double2(ax ? -g.x : v.x, ay ? -g.y : v.y);
      if (__ballot_sync(0xffffffffu, !(isfinite(d.x) && isfinite(d.y))) != 0u) d = make_double2(-g.x, -g.y);
      if (lane == 0) { q.head[row] = head; q.npairs[row] = np; }
    }
    st(q.D, d);
    st(q.G, g);
    st(q.Bp, b);
    if (lane == 0) { q.lev[row] = lev; q.state[row] = 2; }
    ++n;
  }
  if (lane == 0 && n) atomicAdd(q.count, n);
}

// Every row of a mode: state 1, no pair, no step yet.
__global__ void __launch_bounds__(kThreads) k_pqnr_init(int * __restrict__ state, int * __restrict__ head,
                                                        int * __restrict__ npairs, int * __restrict__ lev,
                                                        unsigned long long rows) {
  for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; i < rows;
       i += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
    state[i] = 1;
    head[i] = npairs[i] = 0;
    lev[i] = -1;
  }
}

#undef APR_FOR_ENTRIES

// ---- host side ---------------------------------------------------------------------------------

// out[c] = sum over the rows of M[i, c], c < R (part: kColsumCtas x 64 doubles of scratch)
void launch_colsum(const double * M, uint64_t rows, int R, int ldm, double * part, double * out,
                   cudaStream_t s) {
  k_apr_colsum_part<<<kColsumCtas, kThreads, 0, s>>>(M, rows, R, ldm, part);
  k_apr_colsum_fin<<<1, 64, 0, s>>>(part, kColsumCtas, R, out);
  spb200_count_launches(2);
}

// Device buffers of one CP-APR run, released on every return path.
struct AprBuffers {
  double *   B = nullptr;                      // max dims x ldm
  double *   phi[SPB200_MAXN] = {nullptr};     // dims[m] x ldm: the last Phi of every mode
  double *   packs = nullptr;                  // boundary slots x RP
  uint32_t * slot_row = nullptr;
  double *   lam = nullptr;                    // RP
  double *   sums = nullptr;                   // N x RP start column sums
  double *   ll = nullptr;                     // one double
  unsigned long long * kkt = nullptr;          // one bit pattern
  int *      bad = nullptr;
  double *   colsum_part = nullptr;                 // kColsumCtas x 64
  ~AprBuffers() {
    cudaFree(B); cudaFree(packs); cudaFree(slot_row); cudaFree(lam); cudaFree(sums); cudaFree(ll);
    cudaFree(kkt); cudaFree(bad); cudaFree(colsum_part);
    for (double * p : phi) cudaFree(p);
  }
};


// The extra device buffers of one run of a row method, PDNR or PQNR (B, the slots, lambda, the
// sums and the flags are AprBuffers').
struct RowBuffers : AprBuffers {
  double *   D = nullptr;                      // max dims x ldm: directions
  double *   G = nullptr;                      // max dims x ldm: gradients
  double *   lad = nullptr;                    // max dims x kPdnrTrials: ladder sums
  double *   kkt_row = nullptr;                // max dims
  double *   mu = nullptr;                     // max dims
  int *      state = nullptr;                  // max dims
  int *      count = nullptr;                  // one int: rows with a step
  ~RowBuffers() {
    cudaFree(D); cudaFree(G); cudaFree(lad); cudaFree(kkt_row); cudaFree(mu); cudaFree(state); cudaFree(count);
  }
};

// The gradient walk of (N, tier, rows mode).
template <int N>
void (*pdnr_grad_kernel(int RT, bool rows))(PdnrArgs) {
  if (RT == 16) return rows ? k_pdnr_grad<N, 16, true> : k_pdnr_grad<N, 16, false>;
  if (RT == 32) return rows ? k_pdnr_grad<N, 32, true> : k_pdnr_grad<N, 32, false>;
  return rows ? k_pdnr_grad<N, 64, true> : k_pdnr_grad<N, 64, false>;
}

// k_pdnr_solve over nslots boundary slots (p.w.slot_row set) and the rows of the mode.
cudaError_t launch_pdnr_solve(const PdnrArgs & p, unsigned long long nslots, uint64_t rows, cudaStream_t s) {
  const int RT = rank_tier(p.w.R);
  const size_t smem = sizeof(double) * kWarps * pdnr_ws_doubles(RT);
  void (*k)(const PdnrArgs, unsigned long long, unsigned long long) =
      RT == 16 ? k_pdnr_solve<16> : (RT == 32 ? k_pdnr_solve<32> : k_pdnr_solve<64>);
  cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  k<<<combine_grid((p.w.slot_row ? nslots : 0) + rows), kThreads, smem, s>>>(p, nslots, rows);
  spb200_count_launches(1);
  return cudaGetLastError();
}

// The start of both CP-APR solvers.  Checks the input rules on the device (tensor values and start
// entries finite and >= 0, every start column with a positive sum), then divides every start
// column of d_factors by its sum s_{m,r} and sets lambda_r = prod_m s_{m,r} (lam: RP host doubles,
// also copied to b.lam).  Uses b.bad, b.sums, b.colsum_part and b.lam.  A violated rule returns
// SPLATT_ERROR_BADINPUT before anything is written.
int apr_start(const splatt_b200_tensor * t, int R, int ldm, double * const * d_factors, AprBuffers & b,
              std::vector<double> & lam, cudaStream_t s, const char * name) {
  const int N = t->nmodes, RP = R + (R & 1);
  const FiberStream & fs0 = t->streams[0];
  bool ok = cudaMemsetAsync(b.bad, 0, sizeof(int), s) == cudaSuccess &&
            cudaMemsetAsync(b.sums, 0, (size_t)N * RP * sizeof(double), s) == cudaSuccess;
  if (ok && fs0.nrec) {
    // the records' values: the first double of every 16-byte record
    k_apr_check<<<elementwise_grid(fs0.nrec, 1), kThreads, 0, s>>>(reinterpret_cast<const double *>(fs0.rec),
                                                                   fs0.nrec, 1, 2, b.bad);
    spb200_count_launches(1);
  }
  for (int m = 0; ok && m < N; ++m) {
    k_apr_check<<<elementwise_grid(t->dims[m], R), kThreads, 0, s>>>(d_factors[m], t->dims[m], R, ldm, b.bad);
    spb200_count_launches(1);
    launch_colsum(d_factors[m], t->dims[m], R, ldm, b.colsum_part, b.sums + (size_t)m * RP, s);
  }
  std::vector<double> hs((size_t)N * RP, 0.0);
  int hbad = 1;
  ok = ok && cudaGetLastError() == cudaSuccess &&
       cudaMemcpyAsync(hs.data(), b.sums, hs.size() * sizeof(double), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
       cudaMemcpyAsync(&hbad, b.bad, sizeof(int), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
       cudaStreamSynchronize(s) == cudaSuccess;
  if (!ok) {
    fprintf(stderr, "SPLATT: %s failed (%s)\n", name, cudaGetErrorString(cudaGetLastError()));
    return SPLATT_ERROR_BADINPUT;
  }
  for (int m = 0; m < N && !hbad; ++m)
    for (int r = 0; r < R; ++r)
      if (!(std::isfinite(hs[(size_t)m * RP + r]) && hs[(size_t)m * RP + r] > 0.0)) hbad = 1;
  if (hbad) {
    fprintf(stderr, "SPLATT: %s: a tensor value or start entry is negative or not finite, or a start column "
                    "sums to 0\n", name);
    return SPLATT_ERROR_BADINPUT;
  }

  // start: every column divided by its sum, lambda_r = prod_m s_{m,r}
  lam.assign(RP, 0.0);
  for (int r = 0; r < R; ++r) {
    lam[r] = 1.0;
    for (int m = 0; m < N; ++m) lam[r] *= hs[(size_t)m * RP + r];
  }
  ok = cudaMemcpyAsync(b.lam, lam.data(), RP * sizeof(double), cudaMemcpyHostToDevice, s) == cudaSuccess;
  for (int m = 0; ok && m < N; ++m) {
    k_apr_normalize<<<elementwise_grid(t->dims[m], R), kThreads, 0, s>>>(d_factors[m], b.sums + (size_t)m * RP,
                                                                         d_factors[m], t->dims[m], R, ldm);
    spb200_count_launches(1);
  }
  if (!ok) {
    fprintf(stderr, "SPLATT: %s failed (%s)\n", name, cudaGetErrorString(cudaGetLastError()));
    return SPLATT_ERROR_BADINPUT;
  }
  return SPLATT_SUCCESS;
}

// ---- the row methods: one driver, PDNR's and PQNR's lockstep bodies ---------------------------

// The options of both row methods.
struct RowOpts {
  int    max_inner, max_backtrack;
  double eps_active, eps_div_zero;
};

// Reads the count of rows that got a step: a lockstep iteration's one synchronisation.
bool read_count(const int * count, int & cnt, cudaStream_t s) {
  return cudaGetLastError() == cudaSuccess &&
         cudaMemcpyAsync(&cnt, count, sizeof(int), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaStreamSynchronize(s) == cudaSuccess;
}

// PDNR's lockstep iteration: the gradient and Hessian walk with the Newton directions
// (k_pdnr_grad, k_pdnr_solve), the ladder and the accept.
struct PdnrRows {
  double mu0;
  size_t P = 0;                                     // doubles of a gradient pack
  WalkLaunch<PdnrArgs> gl[SPB200_MAXN], ll[SPB200_MAXN];
  unsigned char * mark[SPB200_MAXN] = {nullptr};   // dims[m]: the row has a record
  explicit PdnrRows(double mu0_) : mu0(mu0_) {}
  ~PdnrRows() {
    for (unsigned char * p : mark) cudaFree(p);
  }

  // per mode the gradient walk and the ladder walk; one pack buffer serves the largest need
  // (boundary slots of either walk, or a pack per row on a leaf-tiled stream)
  bool configure(const splatt_b200_tensor * t, int R, size_t & max_pack, unsigned long long & max_slot) {
    const int RT = rank_tier(R), RP = R + (R & 1), H = RP / 2;
    P = 2 * (size_t)H * (H + 1) + RP;
    for (int m = 0; m < t->nmodes; ++m) {
      const bool rows = t->streams[t->plan[m].stream].ktile_rows > 0;
      auto lad = [rows](auto n) { return rows ? k_pdnr_ladder<n.value, true> : k_pdnr_ladder<n.value, false>; };
      if (!gl[m].configure(with_nmodes(t->nmodes, [&](auto n) { return pdnr_grad_kernel<n.value>(RT, rows); }),
                           pdnr_grad_smem(RT), rows) ||
          !ll[m].configure(with_nmodes(t->nmodes, lad), tc_ring_bytes(), rows))
        return false;
      max_pack = std::max<size_t>({max_pack, (rows ? t->dims[m] : gl[m].nslots) * P, ll[m].nslots * kPdnrTrials});
    }
    max_slot = std::max({max_slots(gl, t->nmodes), max_slots(ll, t->nmodes), 1ull});
    return true;
  }
  bool alloc(const splatt_b200_tensor * t, uint64_t, int) {
    bool ok = true;
    for (int m = 0; ok && m < t->nmodes; ++m)
      ok = cudaMalloc(&mark[m], std::max<uint64_t>(t->dims[m], 1)) == cudaSuccess;
    return ok;
  }
  bool reset(const splatt_b200_tensor * t, RowBuffers &, cudaStream_t s) {
    bool ok = true;
    for (int m = 0; ok && m < t->nmodes; ++m) ok = cudaMemsetAsync(mark[m], 0, t->dims[m], s) == cudaSuccess;
    return ok;
  }
  void start_mode(int n, uint64_t rows, RowBuffers & b, PdnrArgs & p, cudaStream_t s) {
    k_pdnr_init<<<elementwise_grid(rows, 1), kThreads, 0, s>>>(b.mu, b.state, rows, mu0);
    spb200_count_launches(1);
    p.w.slot_row = gl[n].rows ? nullptr : b.slot_row;
    p.mark = mark[n];
  }
  bool lockstep(const FiberStream & fs, int n, uint64_t rows, const PdnrArgs & p, RowBuffers & b,
                const RowOpts & o, cudaStream_t s, int & cnt) {
    const WalkLaunch<PdnrArgs> & GL = gl[n];
    const WalkLaunch<PdnrArgs> & LL = ll[n];
    bool ok = true;
    // gradient, Hessian and direction of every row still to be evaluated
    if (GL.rows) ok = cudaMemsetAsync(b.packs, 0, rows * P * sizeof(double), s) == cudaSuccess;
    if (ok && fs.nrec) ok = GL.launch(p, b.slot_row, s) == cudaSuccess;
    ok = ok && launch_pdnr_solve(p, GL.nslots, rows, s) == cudaSuccess;
    // the ladder's sums and the line search's decision
    ok = ok && cudaMemsetAsync(b.lad, 0, rows * kPdnrTrials * sizeof(double), s) == cudaSuccess &&
         cudaMemsetAsync(b.count, 0, sizeof(int), s) == cudaSuccess;
    if (ok && fs.nrec) {
      ok = LL.launch(p, b.slot_row, s) == cudaSuccess;
      if (ok && !LL.rows) {
        k_apr_combine<<<combine_grid(LL.nslots), kThreads, 0, s>>>(b.packs, b.slot_row, LL.nslots, kPdnrTrials,
                                                                   kPdnrTrials, b.lad);
        spb200_count_launches(1);
      }
    }
    k_pdnr_accept<<<elementwise_grid(rows, 1), kThreads, 0, s>>>(b.B, b.D, b.G, b.lad, b.mu, b.state, rows,
                                                                 p.w.R, p.w.ldm, o.max_backtrack, mu0, b.count);
    spb200_count_launches(1);
    return ok && read_count(b.count, cnt, s);
  }
};

// PQNR's lockstep iteration: MU's Phi walk, k_pqnr_step, and -- only when some row got a
// direction -- PDNR's ladder and accept.
struct PqnrRows {
  int mem;
  WalkLaunch<TcArgs>   pl[SPB200_MAXN];
  WalkLaunch<PdnrArgs> ll[SPB200_MAXN];
  double * phi = nullptr;                           // max dims x ldm
  double * Bp = nullptr;                            // max dims x ldm: b_prev
  double * S = nullptr;                             // mem x max dims x ldm
  double * Y = nullptr;                             // mem x max dims x ldm
  double * rho = nullptr;                           // mem x max dims
  int *    head = nullptr;                          // max dims (each)
  int *    npairs = nullptr;
  int *    lev = nullptr;
  PqnrArgs q = {};
  explicit PqnrRows(int mem_) : mem(mem_) {}
  ~PqnrRows() {
    cudaFree(phi); cudaFree(Bp); cudaFree(S); cudaFree(Y); cudaFree(rho); cudaFree(head); cudaFree(npairs);
    cudaFree(lev);
  }

  // per mode the Phi walk and the ladder walk; one slot buffer serves both (a leaf-tiled stream
  // adds its pieces into Phi and the ladder sums directly)
  bool configure(const splatt_b200_tensor * t, int R, size_t & max_pack, unsigned long long & max_slot) {
    const int RP = R + (R & 1);
    for (int m = 0; m < t->nmodes; ++m) {
      const bool rows = t->streams[t->plan[m].stream].ktile_rows > 0;
      auto phik = [rows](auto n) { return rows ? k_apr_phi<n.value, true> : k_apr_phi<n.value, false>; };
      auto lad = [rows](auto n) { return rows ? k_pdnr_ladder<n.value, true> : k_pdnr_ladder<n.value, false>; };
      if (!pl[m].configure(with_nmodes(t->nmodes, phik), tc_ring_bytes(), rows) ||
          !ll[m].configure(with_nmodes(t->nmodes, lad), tc_ring_bytes(), rows))
        return false;
      max_pack = std::max<size_t>({max_pack, pl[m].nslots * RP, ll[m].nslots * kPdnrTrials});
    }
    max_slot = std::max({max_slots(pl, t->nmodes), max_slots(ll, t->nmodes), 1ull});
    return true;
  }
  bool alloc(const splatt_b200_tensor *, uint64_t max_dim, int ldm) {
    const size_t slot = max_dim * ldm;
    q.slot = slot;
    q.rows_max = max_dim;
    return cudaMalloc(&phi, slot * sizeof(double)) == cudaSuccess &&
           cudaMalloc(&Bp, slot * sizeof(double)) == cudaSuccess &&
           cudaMalloc(&S, mem * slot * sizeof(double)) == cudaSuccess &&
           cudaMalloc(&Y, mem * slot * sizeof(double)) == cudaSuccess &&
           cudaMalloc(&rho, mem * max_dim * sizeof(double)) == cudaSuccess &&
           cudaMalloc(&head, max_dim * sizeof(int)) == cudaSuccess &&
           cudaMalloc(&npairs, max_dim * sizeof(int)) == cudaSuccess &&
           cudaMalloc(&lev, max_dim * sizeof(int)) == cudaSuccess;
  }
  // the accept's damping is never read; zero it once so it stays finite (mu0 = 0 keeps it 0)
  bool reset(const splatt_b200_tensor *, RowBuffers & b, cudaStream_t s) {
    return cudaMemsetAsync(b.mu, 0, q.rows_max * sizeof(double), s) == cudaSuccess;
  }
  void start_mode(int, uint64_t rows, RowBuffers & b, PdnrArgs & p, cudaStream_t s) {
    k_pqnr_init<<<elementwise_grid(rows, 1), kThreads, 0, s>>>(b.state, head, npairs, lev, rows);
    spb200_count_launches(1);
    p.w.out = phi;
    q.phi = phi; q.B = b.B; q.D = b.D; q.G = b.G; q.Bp = Bp; q.S = S; q.Y = Y; q.rho = rho;
    q.head = head; q.npairs = npairs; q.lev = lev; q.state = b.state; q.kkt = b.kkt_row; q.count = b.count;
    q.rows = rows; q.R = p.w.R; q.ldm = p.w.ldm; q.mem = mem;
    q.tol = p.tol; q.eps_active = p.eps_active;
  }
  bool lockstep(const FiberStream & fs, int n, uint64_t rows, const PdnrArgs & p, RowBuffers & b,
                const RowOpts & o, cudaStream_t s, int & cnt) {
    const WalkLaunch<TcArgs> &   PL = pl[n];
    const WalkLaunch<PdnrArgs> & LL = ll[n];
    const int R = p.w.R, ldm = p.w.ldm;
    // Phi at every row's b, then the pair update and the direction of every row still active
    bool ok = cudaMemsetAsync(phi, 0, rows * ldm * sizeof(double), s) == cudaSuccess &&
              cudaMemsetAsync(b.count, 0, sizeof(int), s) == cudaSuccess;
    if (ok && fs.nrec) {
      ok = PL.launch(p.w, b.slot_row, s) == cudaSuccess;
      if (ok && !PL.rows) {
        k_apr_combine<<<combine_grid(PL.nslots), kThreads, 0, s>>>(b.packs, b.slot_row, PL.nslots, R, ldm, phi);
        spb200_count_launches(1);
      }
    }
    q.max_backtrack = o.max_backtrack;
    k_pqnr_step<<<combine_grid(rows), kThreads, 0, s>>>(q);
    spb200_count_launches(1);
    ok = ok && read_count(b.count, cnt, s);
    if (!ok || !cnt) return ok;                     // no direction: the mode is done, no ladder
    // the ladder's sums and the line search's decision
    ok = cudaMemsetAsync(b.lad, 0, rows * kPdnrTrials * sizeof(double), s) == cudaSuccess;
    if (ok && fs.nrec) {
      ok = LL.launch(p, b.slot_row, s) == cudaSuccess;
      if (ok && !LL.rows) {
        k_apr_combine<<<combine_grid(LL.nslots), kThreads, 0, s>>>(b.packs, b.slot_row, LL.nslots, kPdnrTrials,
                                                                   kPdnrTrials, b.lad);
        spb200_count_launches(1);
      }
    }
    k_pdnr_accept<<<elementwise_grid(rows, 1), kThreads, 0, s>>>(b.B, b.D, b.G, b.lad, b.mu, b.state, rows, R,
                                                                 ldm, o.max_backtrack, 0.0, b.count);
    spb200_count_launches(1);
    return ok && cudaGetLastError() == cudaSuccess;
  }
};

// The outer loop of both row methods (Body: PdnrRows or PqnrRows): the input rules (bad: the
// body's own options violate them), the start, and per outer iteration and mode B = A_n diag(lambda),
// up to max_inner lockstep iterations of the body, the largest kkt, the column sums and the
// normalisation; the log-likelihood, lambda and the largest kkt are read back once per outer
// iteration.
template <class Body>
int run_apr_rows(const char * name, const splatt_b200_tensor * t, int R, int ldm, const double * options,
                 const RowOpts & o, bool bad, double * const * d_factors, double * lambda_out, double * history,
                 int * iterations_out, void * stream, Body & body) {
  const double tol = options ? options[SPLATT_OPTION_TOLERANCE] : 0.0;
  const double niter = options ? options[SPLATT_OPTION_NITER] : 0.0;
  auto nonneg = [](double x) { return std::isfinite(x) && x >= 0.0; };
  auto positive = [](double x) { return std::isfinite(x) && x > 0.0; };
  bad = bad || !root_streams_ok(t) || !options || !lambda_out ||
        !factors_ok(t->nmodes, R, ldm, reinterpret_cast<const void * const *>(d_factors)) ||
        o.max_inner < 1 || o.max_backtrack < 1 || o.max_backtrack > kPdnrTrials ||
        !nonneg(o.eps_active) || !positive(o.eps_div_zero) || !nonneg(tol) ||
        !(niter >= 0.0 && niter <= 2147483647.0);
  if (bad) {
    fprintf(stderr, "SPLATT: %s: bad arguments\n", name);
    return SPLATT_ERROR_BADINPUT;
  }
  DeviceGuard g(t->device);
  if (!g.ok) return SPLATT_ERROR_BADINPUT;
  const int N = t->nmodes;
  const int RP = R + (R & 1);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const uint64_t niters = (uint64_t)niter;
  const int verbosity = (int)options[SPLATT_OPTION_VERBOSITY];

  uint64_t max_dim = 1;
  for (int m = 0; m < N; ++m) max_dim = std::max<uint64_t>(max_dim, t->dims[m]);
  size_t max_pack = 1;
  unsigned long long max_slot = 1;
  if (!body.configure(t, R, max_pack, max_slot)) {
    fprintf(stderr, "SPLATT: %s: cannot configure the walks (%s)\n", name, cudaGetErrorString(cudaGetLastError()));
    return SPLATT_ERROR_BADINPUT;
  }
  RowBuffers b;
  bool ok = cudaMalloc(&b.B, max_dim * ldm * sizeof(double)) == cudaSuccess &&
            cudaMalloc(&b.D, max_dim * ldm * sizeof(double)) == cudaSuccess &&
            cudaMalloc(&b.G, max_dim * ldm * sizeof(double)) == cudaSuccess &&
            cudaMalloc(&b.lad, max_dim * kPdnrTrials * sizeof(double)) == cudaSuccess &&
            cudaMalloc(&b.kkt_row, max_dim * sizeof(double)) == cudaSuccess &&
            cudaMalloc(&b.mu, max_dim * sizeof(double)) == cudaSuccess &&
            cudaMalloc(&b.state, max_dim * sizeof(int)) == cudaSuccess &&
            cudaMalloc(&b.count, sizeof(int)) == cudaSuccess &&
            cudaMalloc(&b.packs, max_pack * sizeof(double)) == cudaSuccess &&
            cudaMalloc(&b.slot_row, max_slot * sizeof(uint32_t)) == cudaSuccess &&
            cudaMalloc(&b.lam, RP * sizeof(double)) == cudaSuccess &&
            cudaMalloc(&b.sums, (size_t)N * RP * sizeof(double)) == cudaSuccess &&
            cudaMalloc(&b.ll, sizeof(double)) == cudaSuccess &&
            cudaMalloc(&b.kkt, sizeof(unsigned long long)) == cudaSuccess &&
            cudaMalloc(&b.bad, sizeof(int)) == cudaSuccess &&
            cudaMalloc(&b.colsum_part, kColsumCtas * 64 * sizeof(double)) == cudaSuccess &&
            body.alloc(t, max_dim, ldm);
  if (!ok) {
    cudaGetLastError();
    return SPLATT_ERROR_NOMEMORY;
  }

  std::vector<double> lam;
  const int rc = apr_start(t, R, ldm, d_factors, b, lam, s, name);
  if (rc != SPLATT_SUCCESS) return rc;
  const FiberStream & fs0 = t->streams[0];
  ok = cudaMemsetAsync(b.B, 0, max_dim * ldm * sizeof(double), s) == cudaSuccess && body.reset(t, b, s);

  uint64_t its = 0;
  auto t0 = std::chrono::steady_clock::now();
  for (uint64_t it = 0; ok && it < niters; ++it) {
    if (verbosity > SPLATT_VERBOSITY_NONE) t0 = std::chrono::steady_clock::now();
    bool converged = true;
    long long lockstep = 0, steps = 0;
    ok = cudaMemsetAsync(b.kkt, 0, sizeof(unsigned long long), s) == cudaSuccess;
    for (int n = 0; ok && n < N; ++n) {
      const FiberStream & fs = t->streams[t->plan[n].stream];
      const uint64_t rows = t->dims[n];
      const unsigned eg = elementwise_grid(rows, R);
      PdnrArgs p = {};
      p.w = walk_args(fs, d_factors, ldm, R);
      p.w.mats[0] = b.B;
      p.w.eps = o.eps_div_zero;
      p.w.packs = b.packs;
      p.w.slot_row = b.slot_row;
      p.D = b.D; p.G = b.G; p.lad = b.lad; p.kkt = b.kkt_row; p.mu = b.mu; p.state = b.state;
      p.tol = tol; p.eps_active = o.eps_active;
      // B = A_n diag(lambda) (no shift: A_n stands in for the unread Phi)
      k_apr_scale<<<eg, kThreads, 0, s>>>(d_factors[n], d_factors[n], b.lam, b.B, rows, R, ldm, 0.0, 0.0, 0);
      spb200_count_launches(1);
      body.start_mode(n, rows, b, p, s);
      for (int l = 0; ok && l < o.max_inner; ++l) {
        int cnt = 0;
        ok = body.lockstep(fs, n, rows, p, b, o, s, cnt);
        if (!ok) break;
        ++lockstep;
        steps += cnt;
        if (cnt && l == 0) converged = false;
        if (!cnt) break;
      }
      if (!ok) break;
      k_pdnr_kktmax<<<elementwise_grid(rows, 1), kThreads, 0, s>>>(b.kkt_row, rows, b.kkt);
      spb200_count_launches(1);
      launch_colsum(b.B, rows, R, ldm, b.colsum_part, b.lam, s);
      k_apr_normalize<<<eg, kThreads, 0, s>>>(b.B, b.lam, d_factors[n], rows, R, ldm);
      spb200_count_launches(1);
    }
    if (!ok) break;
    // log-likelihood of the iteration's model, lambda and the largest kkt, read back once
    double ll = 0.0, kkt_max = 0.0;
    unsigned long long bits = 0;
    ok = cudaMemsetAsync(b.ll, 0, sizeof(double), s) == cudaSuccess;
    if (ok && fs0.nrec) {
      TcArgs a = walk_args(fs0, d_factors, ldm, R);
      a.lambda = b.lam; a.sse = b.ll; a.eps = o.eps_div_zero;
      ok = launch_model_sum(with_nmodes(N, [](auto n) { return k_apr_ll<n.value>; }), a, s) == cudaSuccess;
    }
    ok = ok && cudaMemcpyAsync(&ll, b.ll, sizeof(double), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaMemcpyAsync(lam.data(), b.lam, RP * sizeof(double), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaMemcpyAsync(&bits, b.kkt, sizeof(bits), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaStreamSynchronize(s) == cudaSuccess;
    if (!ok) break;
    std::memcpy(&kkt_max, &bits, sizeof(kkt_max));
    for (int r = 0; r < R; ++r) ll -= lam[r];
    if (history) {
      history[4 * it] = ll;
      history[4 * it + 1] = kkt_max;
      history[4 * it + 2] = (double)lockstep;
      history[4 * it + 3] = (double)steps;
    }
    its = it + 1;
    if (verbosity > SPLATT_VERBOSITY_NONE) {
      const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
      printf("  its = %3llu (%0.3fs)  log-likelihood = %0.10e  kkt = %0.3e  lockstep = %lld  steps = %lld\n",
             (unsigned long long)its, sec, ll, kkt_max, lockstep, steps);
    }
    if (converged) break;
  }
  if (!ok) {
    fprintf(stderr, "SPLATT: %s failed (%s)\n", name, cudaGetErrorString(cudaGetLastError()));
    cudaStreamSynchronize(s);
    return SPLATT_ERROR_BADINPUT;
  }
  std::copy(lam.begin(), lam.begin() + R, lambda_out);
  if (iterations_out) *iterations_out = (int)its;
  return SPLATT_SUCCESS;
}

}  // namespace
}  // namespace spb200

using namespace spb200;

extern "C" int splatt_b200_cp_apr_device(splatt_b200_tensor const * t, int ncolumns, int ldm,
                                         double const * options, splatt_b200_apr_opts const * apr,
                                         double * const * d_factors, double * lambda_out,
                                         double * history, int * iterations_out, void * stream) {
  const int R = ncolumns;
  const splatt_b200_apr_opts o = apr ? *apr : splatt_b200_apr_opts{10, 0.01, 1e-10, 1e-10};
  const double tol = options ? options[SPLATT_OPTION_TOLERANCE] : 0.0;
  const double niter = options ? options[SPLATT_OPTION_NITER] : 0.0;
  auto nonneg = [](double x) { return std::isfinite(x) && x >= 0.0; };
  bool bad = !root_streams_ok(t) || !options || !lambda_out ||
             !factors_ok(t->nmodes, R, ldm, reinterpret_cast<const void * const *>(d_factors)) ||
             o.max_inner < 1 || !nonneg(o.kappa) || !nonneg(o.kappa_tol) ||
             !(std::isfinite(o.eps_div_zero) && o.eps_div_zero > 0.0) || !nonneg(tol) ||
             !(niter >= 0.0 && niter <= 2147483647.0);
  if (bad) {
    fprintf(stderr, "SPLATT: splatt_b200_cp_apr_device: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  DeviceGuard g(t->device);
  if (!g.ok) return SPLATT_ERROR_BADINPUT;
  const int N = t->nmodes;
  const int RP = R + (R & 1);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const uint64_t niters = (uint64_t)niter;
  const int verbosity = (int)options[SPLATT_OPTION_VERBOSITY];

  // one Phi launch configuration per mode; the slot buffer serves the largest
  WalkLaunch<TcArgs> ml[SPB200_MAXN];
  uint64_t max_dim = 1;
  for (int m = 0; m < N; ++m) {
    const bool rows = t->streams[t->plan[m].stream].ktile_rows > 0;
    auto phi = [rows](auto n) { return rows ? k_apr_phi<n.value, true> : k_apr_phi<n.value, false>; };
    if (!ml[m].configure(with_nmodes(N, phi), tc_ring_bytes(), rows)) {
      fprintf(stderr, "SPLATT: splatt_b200_cp_apr_device: cannot configure the Phi kernel (%s)\n",
              cudaGetErrorString(cudaGetLastError()));
      return SPLATT_ERROR_BADINPUT;
    }
    max_dim = std::max<uint64_t>(max_dim, t->dims[m]);
  }
  const unsigned long long max_slot = std::max(max_slots(ml, N), 1ull);
  AprBuffers b;
  bool ok = cudaMalloc(&b.B, max_dim * ldm * sizeof(double)) == cudaSuccess &&
            cudaMalloc(&b.packs, max_slot * RP * sizeof(double)) == cudaSuccess &&
            cudaMalloc(&b.slot_row, max_slot * sizeof(uint32_t)) == cudaSuccess &&
            cudaMalloc(&b.lam, RP * sizeof(double)) == cudaSuccess &&
            cudaMalloc(&b.sums, (size_t)N * RP * sizeof(double)) == cudaSuccess &&
            cudaMalloc(&b.ll, sizeof(double)) == cudaSuccess &&
            cudaMalloc(&b.kkt, sizeof(unsigned long long)) == cudaSuccess &&
            cudaMalloc(&b.bad, sizeof(int)) == cudaSuccess &&
            cudaMalloc(&b.colsum_part, kColsumCtas * 64 * sizeof(double)) == cudaSuccess;
  for (int m = 0; ok && m < N; ++m)
    ok = cudaMalloc(&b.phi[m], std::max<uint64_t>(t->dims[m], 1) * ldm * sizeof(double)) == cudaSuccess;
  if (!ok) {
    cudaGetLastError();
    return SPLATT_ERROR_NOMEMORY;
  }

  std::vector<double> lam;
  const int rc = apr_start(t, R, ldm, d_factors, b, lam, s, "splatt_b200_cp_apr_device");
  if (rc != SPLATT_SUCCESS) return rc;
  const FiberStream & fs0 = t->streams[0];
  ok = cudaMemsetAsync(b.B, 0, max_dim * ldm * sizeof(double), s) == cudaSuccess;
  for (int m = 0; ok && m < N; ++m)
    ok = cudaMemsetAsync(b.phi[m], 0, t->dims[m] * ldm * sizeof(double), s) == cudaSuccess;

  uint64_t its = 0;
  auto t0 = std::chrono::steady_clock::now();
  for (uint64_t it = 0; ok && it < niters; ++it) {
    if (verbosity > SPLATT_VERBOSITY_NONE) t0 = std::chrono::steady_clock::now();
    bool converged = true;
    double kkt_max = 0.0;
    int inner_total = 0;
    for (int n = 0; ok && n < N; ++n) {
      const FiberStream & fs = t->streams[t->plan[n].stream];
      const WalkLaunch<TcArgs> & L = ml[n];
      const uint64_t rows = t->dims[n];
      const unsigned eg = elementwise_grid(rows, R);
      k_apr_scale<<<eg, kThreads, 0, s>>>(d_factors[n], b.phi[n], b.lam, b.B, rows, R, ldm, o.kappa,
                                          o.kappa_tol, it > 0);
      spb200_count_launches(1);
      TcArgs a = walk_args(fs, d_factors, ldm, R);
      a.mats[0] = b.B;
      a.eps = o.eps_div_zero; a.out = b.phi[n];
      a.packs = b.packs; a.slot_row = b.slot_row;
      double kkt = 0.0;
      int l = 0;
      for (; ok && l < o.max_inner; ++l) {
        ok = cudaMemsetAsync(b.phi[n], 0, rows * ldm * sizeof(double), s) == cudaSuccess &&
             cudaMemsetAsync(b.kkt, 0, sizeof(unsigned long long), s) == cudaSuccess;
        if (ok && fs.nrec) {
          ok = L.launch(a, b.slot_row, s) == cudaSuccess;
          if (ok && !L.rows) {
            k_apr_combine<<<combine_grid(L.nslots), kThreads, 0, s>>>(b.packs, b.slot_row, L.nslots, R, ldm,
                                                                      b.phi[n]);
            spb200_count_launches(1);
          }
        }
        k_apr_kkt<<<eg, kThreads, 0, s>>>(b.B, b.phi[n], rows, R, ldm, b.kkt);
        spb200_count_launches(1);
        unsigned long long bits = 0;
        ok = ok && cudaGetLastError() == cudaSuccess &&
             cudaMemcpyAsync(&bits, b.kkt, sizeof(bits), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
             cudaStreamSynchronize(s) == cudaSuccess;
        if (!ok) break;
        std::memcpy(&kkt, &bits, sizeof(kkt));
        ++inner_total;
        if (kkt < tol) break;
        k_apr_mul<<<eg, kThreads, 0, s>>>(b.B, b.phi[n], rows, R, ldm);
        spb200_count_launches(1);
      }
      if (!ok) break;
      if (!(l == 0 && kkt < tol)) converged = false;
      kkt_max = std::max(kkt_max, kkt);
      launch_colsum(b.B, rows, R, ldm, b.colsum_part, b.lam, s);
      k_apr_normalize<<<eg, kThreads, 0, s>>>(b.B, b.lam, d_factors[n], rows, R, ldm);
      spb200_count_launches(1);
    }
    if (!ok) break;
    // log-likelihood of the iteration's model, and lambda, read back once
    double ll = 0.0;
    ok = cudaMemsetAsync(b.ll, 0, sizeof(double), s) == cudaSuccess;
    if (ok && fs0.nrec) {
      TcArgs a = walk_args(fs0, d_factors, ldm, R);
      a.lambda = b.lam; a.sse = b.ll; a.eps = o.eps_div_zero;
      ok = launch_model_sum(with_nmodes(N, [](auto n) { return k_apr_ll<n.value>; }), a, s) == cudaSuccess;
    }
    ok = ok && cudaMemcpyAsync(&ll, b.ll, sizeof(double), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaMemcpyAsync(lam.data(), b.lam, RP * sizeof(double), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaStreamSynchronize(s) == cudaSuccess;
    if (!ok) break;
    for (int r = 0; r < R; ++r) ll -= lam[r];
    if (history) {
      history[3 * it] = ll;
      history[3 * it + 1] = kkt_max;
      history[3 * it + 2] = inner_total;
    }
    its = it + 1;
    if (verbosity > SPLATT_VERBOSITY_NONE) {
      const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
      printf("  its = %3llu (%0.3fs)  log-likelihood = %0.10e  kkt = %0.3e  inner = %d\n",
             (unsigned long long)its, sec, ll, kkt_max, inner_total);
    }
    if (converged) break;
  }
  if (!ok) {
    fprintf(stderr, "SPLATT: splatt_b200_cp_apr_device failed (%s)\n", cudaGetErrorString(cudaGetLastError()));
    cudaStreamSynchronize(s);
    return SPLATT_ERROR_BADINPUT;
  }
  std::copy(lam.begin(), lam.begin() + R, lambda_out);
  if (iterations_out) *iterations_out = (int)its;
  return SPLATT_SUCCESS;
}

extern "C" int splatt_b200_cp_apr_pdnr_device(splatt_b200_tensor const * t, int ncolumns, int ldm,
                                              double const * options, splatt_b200_pdnr_opts const * pdnr,
                                              double * const * d_factors, double * lambda_out,
                                              double * history, int * iterations_out, void * stream) {
  const splatt_b200_pdnr_opts o = pdnr ? *pdnr : splatt_b200_pdnr_opts{10, 8, 1e-5, 1e-8, 1e-10};
  PdnrRows body(o.mu0);
  return run_apr_rows("splatt_b200_cp_apr_pdnr_device", t, ncolumns, ldm, options,
                      RowOpts{o.max_inner, o.max_backtrack, o.eps_active, o.eps_div_zero},
                      !(std::isfinite(o.mu0) && o.mu0 > 0.0), d_factors, lambda_out, history, iterations_out,
                      stream, body);
}

extern "C" int splatt_b200_cp_apr_pqnr_device(splatt_b200_tensor const * t, int ncolumns, int ldm,
                                              double const * options, splatt_b200_pqnr_opts const * pqnr,
                                              double * const * d_factors, double * lambda_out,
                                              double * history, int * iterations_out, void * stream) {
  const splatt_b200_pqnr_opts o = pqnr ? *pqnr : splatt_b200_pqnr_opts{10, 8, 3, 1e-8, 1e-10};
  PqnrRows body(o.lbfgs_mem);
  return run_apr_rows("splatt_b200_cp_apr_pqnr_device", t, ncolumns, ldm, options,
                      RowOpts{o.max_inner, o.max_backtrack, o.eps_active, o.eps_div_zero},
                      o.lbfgs_mem < 1 || o.lbfgs_mem > kPqnrMaxMem, d_factors, lambda_out, history,
                      iterations_out, stream, body);
}
