// Tensor completion by whole-model L-BFGS with an exact line search on device-resident tensors
// (splatt_b200_tc_lbfgs_device; CP-WOPT, Acar, Dunlavy, Kolda & Morup 2011), and the host root
// finder of its line search (splatt_b200_poly_argmin).
//
// The objective is completion's, L = sum_stored (v - x^)^2 + reg sum_m ||U_m||_F^2, minimised over
// all factors at once.  One iteration is a fixed sequence of kernels with one host read-back:
//   * k_tcg_grad<N, ROWS> walks mode m's root stream (walk_range with OPEN: the root row u is
//     loaded where a slice opens).  Per record x^ = u . h is a warp sum, r = v - x^ and acc += r h.
//     A slice that closes inside the warp's range stores G[i] = 2 reg u - 2 acc; the range's first
//     and last slice go to its two boundary slots (RP doubles each) and k_tcg_combine adds each
//     row's slots in range order.  Rows without records keep the 2 reg U that k_tcg_axpy wrote
//     first.  Leaf-tiled streams add -2 acc with red.add into that 2 reg U.
//   * The direction is the L-BFGS two-loop recursion run as a sequence of vector launches
//     (k_tcg_dot, k_tcg_axpy) whose coefficients are read from device scalars, so the recursion
//     needs no host synchronisation.  The newest pair enters the ring on the device (a kernel
//     checks s.y > 0), and the descent check (g.d < 0, else d = -g) is a gated launch as well.
//   * k_tcg_line<N> walks mode 0's root stream with walk_levels, gathers U and D rows at every
//     level, forms per column the N+1 coefficients of prod_m (u_m + alpha d_m), reduces them over
//     the warp with a transposed butterfly and accumulates the 2N+1 coefficients of
//     (v - p(alpha))^2.  Per-CTA partials go to [grid][2N+1]; the host adds them in CTA order.
//   * Vector kernels run one warp per factor row over the concatenation of the modes' blocks
//     (dims[m] x ldm each, columns [0, R) only).  Dot products are two-stage and fixed-order: each
//     CTA writes its partial, and the last CTA to finish adds the partials in CTA order.
// Nothing that feeds alpha or the factors is reduced with atomics on untiled streams, so the
// factors and alpha are bitwise reproducible there.
#include "walk.cuh"
#include <algorithm>
#include <chrono>
#include <cmath>
#include <vector>

namespace spb200 {

// The SSE kernel of completion (tc.cu), for the validation score.
cudaError_t tc_enqueue_sse(const FiberStream & fs, int R, int ldm, const double * const * d_mats_by_mode,
                           const double * d_lambda, double * d_sse, cudaStream_t s);

namespace {

constexpr int kDotGrid = 264;     // CTAs of every dot product (fixed: the sum order is fixed)

// A vector over all modes: block m is dims[m] rows x ldm at p[m]; entries are columns [0, R).
struct Blocks {
  double * p[SPB200_MAXN];
};
struct VecShape {
  unsigned long long row0[SPB200_MAXN + 1];   // first row of every block; row0[nm] = total rows
  int nm, R, ldm;
};

// a[i] by a compile-time index per candidate, so the per-mode lookups stay in registers
template <class T, int K>
__device__ __forceinline__ T pick(const T (&a)[K], int i) {
  T r = a[0];
#pragma unroll
  for (int k = 1; k < K; ++k)
    if (i == k) r = a[k];
  return r;
}
__device__ __forceinline__ size_t vec_off(const VecShape & sh, int m, unsigned long long row) {
  return static_cast<size_t>(row - pick(sh.row0, m)) * sh.ldm;
}

// Launch gates on a device scalar x: run always, only if x > 0, only if !(x > 0), only if !(x < 0).
enum Gate : int { kAlways = 0, kPos = 1, kNotPos = 2, kNotNeg = 3 };
__device__ __forceinline__ bool gate_open(const double * g, int mode) {
  if (mode == kAlways) return true;
  const double x = *g;
  return mode == kPos ? (x > 0.0) : (mode == kNotPos ? !(x > 0.0) : !(x < 0.0));
}

// One operand of a dot product: a A + z Z elementwise (Z read only when z != 0), computed as
// fma(z, Z, a A) -- the same rounding as k_tcg_axpy's store of that combination.
struct Opnd {
  Blocks A, Z;
  double a, z;
};
__device__ __forceinline__ double opnd(const Opnd & o, int m, size_t off) {
  const double x = o.a * o.A.p[m][off];
  return o.z != 0.0 ? fma(o.z, o.Z.p[m][off], x) : x;
}

// *out = sum x . y over every entry, in a fixed order: one warp per row (grid-stride), lanes over
// columns, a per-CTA partial into part[blockIdx.x], and the last CTA adds the kDotGrid partials
// in CTA order (part[kDotGrid] holds the arrival count and is left at 0).  Skipped entirely when
// the gate is closed.
__global__ void __launch_bounds__(kThreads) k_tcg_dot(const __grid_constant__ VecShape sh, const __grid_constant__ Opnd x,
                                                      const __grid_constant__ Opnd y,
                                                      double * __restrict__ part, double * __restrict__ out,
                                                      const double * gate, int gmode) {
  __shared__ double wp[kWarps];
  __shared__ bool   lastcta;
  if (!gate_open(gate, gmode)) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double s = 0.0;
  int m = 0;
  for (unsigned long long row = static_cast<unsigned long long>(blockIdx.x) * kWarps + warp; row < sh.row0[sh.nm];
       row += static_cast<unsigned long long>(gridDim.x) * kWarps) {
    while (row >= pick(sh.row0, m + 1)) ++m;
    const size_t off = vec_off(sh, m, row);
    const Opnd xm = {{{pick(x.A.p, m)}}, {{pick(x.Z.p, m)}}, x.a, x.z};
    const Opnd ym = {{{pick(y.A.p, m)}}, {{pick(y.Z.p, m)}}, y.a, y.z};
    for (int j = lane; j < sh.R; j += 32) s = fma(opnd(xm, 0, off + j), opnd(ym, 0, off + j), s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) wp[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < kWarps; ++w) t += wp[w];
    part[blockIdx.x] = t;
    __threadfence();
    unsigned int * cnt = reinterpret_cast<unsigned int *>(part + gridDim.x);
    lastcta = atomicAdd(cnt, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!lastcta || threadIdx.x != 0) return;
  __threadfence();
  const volatile double * vp = part;
  double t = 0.0;
  for (unsigned b = 0; b < gridDim.x; ++b) t += vp[b];
  *out = t;
  *reinterpret_cast<unsigned int *>(part + gridDim.x) = 0u;
}

// Y = b Y + c X + z Z over every entry (Y read only when b != 0, Z only when z != 0), with
// c = hc (P ? *P - (Q ? *Q : 0) : 1) / (Dn ? *Dn : 1) from device scalars.  Skipped when the gate
// is closed.
struct Coef {
  const double * P;
  const double * Q;
  const double * Dn;
  double hc;
};
__global__ void __launch_bounds__(kThreads) k_tcg_axpy(const __grid_constant__ VecShape sh, const __grid_constant__ Blocks Y,
                                                       double b, const __grid_constant__ Blocks X, const Coef cf,
                                                       const __grid_constant__ Blocks Z, double z,
                                                       const double * gate, int gmode) {
  if (!gate_open(gate, gmode)) return;
  double c = cf.hc;
  if (cf.P) c *= cf.Q ? *cf.P - *cf.Q : *cf.P;
  if (cf.Dn) c /= *cf.Dn;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int m = 0;
  for (unsigned long long row = static_cast<unsigned long long>(blockIdx.x) * kWarps + warp; row < sh.row0[sh.nm];
       row += static_cast<unsigned long long>(gridDim.x) * kWarps) {
    while (row >= pick(sh.row0, m + 1)) ++m;
    const size_t off = vec_off(sh, m, row);
    double * const       y  = pick(Y.p, m) + off;
    const double * const x  = pick(X.p, m) + off;
    const double * const zz = pick(Z.p, m) + off;
    for (int j = lane; j < sh.R; j += 32) {
      double v = c * x[j];
      if (b != 0.0) v = fma(b, y[j], v);
      if (z != 0.0) v = fma(z, zz[j], v);
      y[j] = v;
    }
  }
}

// dst[0..n) = src[0..n) when the gate is open (one thread).
__global__ void k_tcg_copy(const double * __restrict__ src, double * __restrict__ dst, int n, const double * gate,
                           int gmode) {
  if (threadIdx.x == 0 && gate_open(gate, gmode))
    for (int i = 0; i < n; ++i) dst[i] = src[i];
}

// Gradient block of the root mode of one stream: a.mats[0] = U_m, a.out = G_m (pitch ldm, holding
// 2 reg U_m on entry), a.packs = boundary slots [2 * warps][RP], a.reg = reg.  ROWS: leaf-tiled
// stream, every closed piece is added into G with red.add.
template <int N, bool ROWS>
__global__ void __launch_bounds__(kThreads, 3) k_tcg_grad(const TcArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int  warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool act  = 2 * lane < a.R;
  const bool hasy = 2 * lane + 1 < a.R;
  const int  RP   = a.R + (a.R & 1);
  const unsigned long long gw = static_cast<unsigned long long>(blockIdx.x) * kWarps + warp;
  const double reg2 = 2.0 * a.reg;
  double2 u = make_double2(0.0, 0.0), acc = make_double2(0.0, 0.0);
  bool    open = true, seen = false;
  walk_range<N, 1, true>(a, smem, act, [&](double v, double2 h, bool close, uint32_t row, bool last) {
    if (open) {
      if (act) u = reinterpret_cast<const double2 *>(a.mats[0] + static_cast<size_t>(row) * a.ldm)[lane];
      if (!hasy) u.y = 0.0;
      open = false;
    }
    if (!hasy) h.y = 0.0;
    double x = u.x * h.x;
    x = fma(u.y, h.y, x);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    acc = vfma(v - x, h, acc);
    if (!close) return;
    open = true;
    if constexpr (ROWS) {
      if (act) {
        double * g = a.out + static_cast<size_t>(row) * a.ldm + 2 * lane;
        atomicAdd(g, -2.0 * acc.x);
        if (hasy) atomicAdd(g + 1, -2.0 * acc.y);
      }
    } else if (!seen || last) {
      const unsigned long long slot = 2 * gw + (seen ? 1 : 0);
      if (act) reinterpret_cast<double2 *>(a.packs + slot * RP)[lane] = acc;
      if (lane == 0) a.slot_row[slot] = row;
    } else if (act) {
      double2 * g = reinterpret_cast<double2 *>(a.out + static_cast<size_t>(row) * a.ldm) + lane;
      const double2 gv = make_double2(fma(reg2, u.x, -2.0 * acc.x), fma(reg2, u.y, -2.0 * acc.y));
      if (hasy) *g = gv;
      else g->x = gv.x;
    }
    acc  = make_double2(0.0, 0.0);
    seen = true;
  });
}

// G[row] = 2 reg U[row] - 2 sum of the row's boundary slots, added in range order (the warp of a
// row's first slot adds them all), one warp per slot.
__global__ void __launch_bounds__(kThreads) k_tcg_combine(const double * __restrict__ slots,
                                                          const uint32_t * __restrict__ slot_row,
                                                          unsigned long long nslots, int R, int ldm, double reg,
                                                          const double * __restrict__ U, double * __restrict__ G) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int RP = R + (R & 1);
  const unsigned long long TW = static_cast<unsigned long long>(gridDim.x) * kWarps;
  for (unsigned long long s = static_cast<unsigned long long>(blockIdx.x) * kWarps + warp; s < nslots; s += TW) {
    const uint32_t row = slot_row[s];
    if (row == kEmptySlot) continue;
    long long t = static_cast<long long>(s) - 1;
    while (t >= 0 && slot_row[t] == kEmptySlot) --t;
    if (t >= 0 && slot_row[t] == row) continue;          // not the row's first slot
    for (int j = lane; j < R; j += 32) {
      double acc = 0.0;
      for (unsigned long long q = s; q < nslots; ++q) {
        const uint32_t r2 = slot_row[q];
        if (r2 == kEmptySlot) continue;
        if (r2 != row) break;
        acc += slots[q * RP + j];
      }
      const size_t o = static_cast<size_t>(row) * ldm + j;
      G[o] = fma(2.0 * reg, U[o], -2.0 * acc);
    }
  }
}

// Arguments of the line walk: the walker's (factors U by level), D by level (pitch w.ldm), and the
// per-CTA partials [grid][2N+1].
struct TcgLine {
  TcArgs         w;
  const double * dm[SPB200_MAXN];
  double *       part;
};

// Sum over the warp of q[0..V) (V a power of two, V <= 32) by a transposed butterfly: each round
// keeps half of the sums and sends the other half.  Afterwards q[0] holds the total of value
// butterfly_index(lane) and the other entries are garbage.
template <int V>
__device__ __forceinline__ void butterfly(double (&q)[V], int lane) {
  int n = V;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    if (n > 1) {
      const int  half = n / 2;
      const bool up   = lane & o;
#pragma unroll
      for (int i = 0; i < V / 2; ++i) {
        if (i < half) {
          const double send = up ? q[i] : q[i + half], keep = up ? q[i + half] : q[i];
          q[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
        }
      }
      n = half;
    } else {
      q[0] += __shfl_xor_sync(0xffffffffu, q[0], o);
    }
  }
}
// The lane that holds the total of value j after butterfly<V>.
__host__ __device__ constexpr int butterfly_lane(int j, int V) {
  int lane = 0;
  for (int o = 16, n = V; o > 0 && n > 1; o >>= 1, n /= 2)
    if (j & (n / 2)) lane |= o;
  return lane;
}
__host__ __device__ constexpr int pow2_at_least(int x) { return x <= 1 ? 1 : 2 * pow2_at_least((x + 1) / 2); }

// Coefficients of phi_data(alpha) = sum_x (v - sum_r prod_m (u_m + alpha d_m)_r)^2 over this grid's
// ranges of the stream, per CTA in fixed order, into part[blockIdx.x][0 .. 2N].
template <int N>
__global__ void __launch_bounds__(kThreads, 1) k_tcg_line(const TcgLine p) {
  const TcArgs & a = p.w;
  constexpr int  K = 2 * N + 1;
  constexpr int  V = pow2_at_least(N + 1);
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ double wpart[kWarps][K];
  const int  warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool act  = 2 * lane < a.R;
  const bool hasy = 2 * lane + 1 < a.R;
  const uint32_t pitch = static_cast<uint32_t>(a.ldm) * 8u;
  const char *   ub[N];
  const char *   db[N];
#pragma unroll
  for (int l = 0; l < N; ++l) {
    ub[l] = reinterpret_cast<const char *>(a.mats[l] + (act ? 2 * lane : 0));
    db[l] = reinterpret_cast<const char *>(p.dm[l] + (act ? 2 * lane : 0));
  }
  double2 ur[N], dr[N];
#pragma unroll
  for (int l = 0; l < N; ++l) ur[l] = dr[l] = make_double2(0.0, 0.0);
  double acc[K];
#pragma unroll
  for (int k = 0; k < K; ++k) acc[k] = 0.0;

  walk_levels<N>(a, smem, [&](const uint4 & q, uint32_t pc, const uint32_t * pos, bool, uint32_t, bool) {
    if (act) {
#pragma unroll
      for (int l = 0; l <= N - 2; ++l) {
        if (l + int(pc) >= N - 1) {
          const uint32_t idx = (l == N - 2) ? (q.w & SPB200_IDX_MASK) : __ldg(&a.up[l][pos[l]]);
          ur[l] = ld_row<double2>(ub[l], idx, pitch);
          dr[l] = ld_row<double2>(db[l], idx, pitch);
        }
      }
      ur[N - 1] = ld_row<double2>(ub[N - 1], q.z, pitch);
      dr[N - 1] = ld_row<double2>(db[N - 1], q.z, pitch);
    }
    // the lane's two columns of prod_l (u_l + alpha d_l), coefficient j of alpha^j
    double px[N + 1], py[N + 1];
    px[0] = ur[0].x; px[1] = dr[0].x;
    py[0] = ur[0].y; py[1] = dr[0].y;
#pragma unroll
    for (int j = 2; j <= N; ++j) px[j] = py[j] = 0.0;
#pragma unroll
    for (int l = 1; l < N; ++l) {
#pragma unroll
      for (int j = l + 1; j >= 1; --j) {
        px[j] = fma(px[j], ur[l].x, px[j - 1] * dr[l].x);
        py[j] = fma(py[j], ur[l].y, py[j - 1] * dr[l].y);
      }
      px[0] *= ur[l].x;
      py[0] *= ur[l].y;
    }
    double s[V];
#pragma unroll
    for (int j = 0; j < V; ++j) s[j] = (j <= N && act) ? px[j] + (hasy ? py[j] : 0.0) : 0.0;
    butterfly<V>(s, lane);
    // e(alpha) = v - p(alpha): every lane gathers the N+1 totals
    double e[N + 1];
#pragma unroll
    for (int j = 0; j <= N; ++j) e[j] = -__shfl_sync(0xffffffffu, s[0], butterfly_lane(j, V));
    e[0] += rec_val<double>(q);
#pragma unroll
    for (int k = 0; k < K; ++k) {
      double t = 0.0;
#pragma unroll
      for (int i = 0; i <= N; ++i) {
        const int j = k - i;
        if (j > i && j <= N) t = fma(e[i], e[j], t);
      }
      t = 2.0 * t;
      if ((k & 1) == 0) t = fma(e[k / 2], e[k / 2], t);
      acc[k] += t;
    }
  });
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) wpart[warp][k] = acc[k];
  }
  __syncthreads();
  if (threadIdx.x < K) {
    double t = 0.0;
    for (int w = 0; w < kWarps; ++w) t += wpart[w][threadIdx.x];
    p.part[static_cast<size_t>(blockIdx.x) * K + threadIdx.x] = t;
  }
}

// ---- host side ---------------------------------------------------------------------------------

// The polynomial sum_j c[j] x^j at x (Horner).
double poly_eval(const std::vector<double> & c, double x) {
  double s = 0.0;
  for (size_t j = c.size(); j-- > 0;) s = std::fma(s, x, c[j]);
  return s;
}

// A root of p in [lo, hi] where p(lo) and p(hi) have opposite signs (or p(hi) = 0), by bisection
// until the midpoint equals an endpoint.
double bisect(const std::vector<double> & p, double lo, double hi) {
  const double plo = poly_eval(p, lo);
  for (;;) {
    const double mid = 0.5 * (lo + hi);
    if (!(mid > lo && mid < hi)) break;
    const double pm = poly_eval(p, mid);
    if (pm == 0.0) return mid;
    if ((pm < 0.0) == (plo < 0.0)) lo = mid;
    else hi = mid;
  }
  const double pl = std::fabs(poly_eval(p, lo)), ph = std::fabs(poly_eval(p, hi));
  return ph < pl ? hi : lo;
}

// The real roots in (0, B] of p at which p changes sign or vanishes exactly, ascending.  Between
// consecutive roots of p' p is monotone, so each such interval holds at most one root; the roots
// of p' come from the same rule one degree down (a linear p has its root in closed form).
std::vector<double> roots_in(const std::vector<double> & p, double B) {
  std::vector<double> out;
  const int deg = (int)p.size() - 1;
  if (deg < 1) return out;
  if (deg == 1) {
    const double r = -p[0] / p[1];
    if (r > 0.0 && r <= B) out.push_back(r);
    return out;
  }
  std::vector<double> dp(deg);
  for (int j = 1; j <= deg; ++j) dp[j - 1] = j * p[j];
  std::vector<double> pts{0.0};
  for (double r : roots_in(dp, B))
    if (r > pts.back() && r < B) pts.push_back(r);
  pts.push_back(B);
  for (size_t i = 0; i + 1 < pts.size(); ++i) {
    const double a = pts[i], b = pts[i + 1];
    const double pa = poly_eval(p, a), pb = poly_eval(p, b);
    double r;
    if (pb == 0.0) r = b;
    else if (pa == 0.0) r = a;
    else if ((pa < 0.0) != (pb < 0.0)) r = bisect(p, a, b);
    else continue;
    if (r > 0.0 && (out.empty() || r > out.back())) out.push_back(r);
  }
  return out;
}

// Device buffers of one run, released on every return path.
struct LbfgsBuffers {
  double *   vec = nullptr;       // g, g_prev, d, then the pairs s_0, y_0, s_1, y_1, ...
  double *   slots = nullptr;     // gradient boundary slots
  uint32_t * slot_row = nullptr;
  double *   sc = nullptr;        // device scalars (kSc*)
  double *   dotpart = nullptr;   // kDotGrid partials and the arrival count
  double *   lpart = nullptr;     // line partials [grid][2N+1]
  double *   lambda = nullptr;    // RP ones for the validation SSE
  ~LbfgsBuffers() {
    cudaFree(vec); cudaFree(slots); cudaFree(slot_row); cudaFree(sc); cudaFree(dotpart); cudaFree(lpart);
    cudaFree(lambda);
  }
};

// device scalars: the pending pair's s.y and y.y, |g|^2, g.d, <U,U>, <U,D>, <D,D>, the validation
// SSE; then 4 per ring slot: s.y, y.y, s.q (first loop), y.q (second loop)
enum { kScSy = 0, kScYy, kScGg, kScGd, kScUu, kScUd, kScDd, kScVal, kScHead, kScSlot = kScHead };

}  // namespace
}  // namespace spb200

using namespace spb200;

extern "C" int splatt_b200_poly_argmin(int degree, double const * c, double * alpha_out, double * decrease_out) {
  if (degree < 0 || degree > 16 || !c || !alpha_out || !decrease_out) return SPLATT_ERROR_BADINPUT;
  for (int j = 0; j <= degree; ++j)
    if (!std::isfinite(c[j])) return SPLATT_ERROR_BADINPUT;
  // phi'(x) = sum_{j>=1} j c_j x^(j-1), trailing zero coefficients dropped
  std::vector<double> dp;
  for (int j = 1; j <= degree; ++j) dp.push_back(j * c[j]);
  while (!dp.empty() && dp.back() == 0.0) dp.pop_back();
  double best = 0.0, bestd = 0.0;
  if (!dp.empty()) {
    const double lead = std::fabs(dp.back());
    double mx = 0.0;
    for (size_t j = 0; j + 1 < dp.size(); ++j) mx = std::max(mx, std::fabs(dp[j]) / lead);
    const double B = 1.0 + mx;                             // Cauchy bound of phi's roots
    for (double r : roots_in(dp, B)) {
      double t = 0.0;                                      // phi(r) - phi(0) = sum_{j>=1} c_j r^j
      for (int j = degree; j >= 1; --j) t = std::fma(t, r, c[j]);
      const double dec = -(t * r);
      if (dec > bestd) { bestd = dec; best = r; }
    }
  }
  *alpha_out = best;
  *decrease_out = bestd;
  return SPLATT_SUCCESS;
}

extern "C" int splatt_b200_tc_lbfgs_device(splatt_b200_tensor const * train, splatt_b200_tensor const * validate,
                                           int ncolumns, int ldm, double const * options,
                                           splatt_b200_tc_lbfgs_opts const * lopts, double * const * d_factors,
                                           double * history, int * iterations_out, void * stream) {
  const int R = ncolumns;
  const double reg = options ? options[SPLATT_OPTION_REGULARIZE] : 0.0;
  const int M = lopts ? lopts->memory : 5;
  bool bad = !root_streams_ok(train) || !options ||
             !factors_ok(train->nmodes, R, ldm, reinterpret_cast<const void * const *>(d_factors)) ||
             !(std::isfinite(reg) && reg >= 0.0) || M < 0 || M > 32;
  if (!bad && validate) {
    bad = validate->nmodes != train->nmodes || validate->shard_count > 1 ||
          validate->device != train->device || validate->streams.empty() ||
          !stream_fits(validate->streams[0]);
    for (int m = 0; !bad && m < train->nmodes; ++m) bad = validate->dims[m] != train->dims[m];
  }
  if (bad) {
    fprintf(stderr, "SPLATT: splatt_b200_tc_lbfgs_device: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  DeviceGuard dg(train->device);
  if (!dg.ok) return SPLATT_ERROR_BADINPUT;
  const int N = train->nmodes, RP = R + (R & 1), K = 2 * N + 1;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const uint64_t niters = (uint64_t)options[SPLATT_OPTION_NITER];
  const double tol = options[SPLATT_OPTION_TOLERANCE];
  const int verbosity = (int)options[SPLATT_OPTION_VERBOSITY];

  // launch configurations: the gradient walk of every mode, the line walk of mode 0's stream
  WalkLaunch<TcArgs> gl[SPB200_MAXN];
  for (int m = 0; m < N; ++m) {
    const bool rows = train->streams[train->plan[m].stream].ktile_rows > 0;
    if (!gl[m].configure(with_nmodes(N, [&](auto n) {
                           return rows ? k_tcg_grad<n.value, true> : k_tcg_grad<n.value, false>;
                         }),
                         tc_ring_bytes(), rows)) {
      fprintf(stderr, "SPLATT: splatt_b200_tc_lbfgs_device: cannot configure the gradient walk (%s)\n",
              cudaGetErrorString(cudaGetLastError()));
      return SPLATT_ERROR_BADINPUT;
    }
  }
  void (*lk)(TcgLine) = with_nmodes(N, [](auto n) { return k_tcg_line<n.value>; });
  const int lgrid = resident_grid(lk, tc_ring_bytes());
  if (lgrid < 1) {
    fprintf(stderr, "SPLATT: splatt_b200_tc_lbfgs_device: cannot configure the line walk (%s)\n",
            cudaGetErrorString(cudaGetLastError()));
    return SPLATT_ERROR_BADINPUT;
  }

  VecShape sh = {};
  sh.nm = N; sh.R = R; sh.ldm = ldm;
  for (int m = 0; m < N; ++m) sh.row0[m + 1] = sh.row0[m] + train->dims[m];
  const size_t V = (size_t)sh.row0[N] * ldm;                 // doubles per vector
  LbfgsBuffers b;
  const int nsc = kScHead + 4 * std::max(M, 1);
  if (cudaMalloc(&b.vec, (3 + 2 * (size_t)M) * V * sizeof(double)) != cudaSuccess ||
      cudaMalloc(&b.slots, std::max(max_slots(gl, N), 1ull) * RP * sizeof(double)) != cudaSuccess ||
      cudaMalloc(&b.slot_row, std::max(max_slots(gl, N), 1ull) * sizeof(uint32_t)) != cudaSuccess ||
      cudaMalloc(&b.sc, nsc * sizeof(double)) != cudaSuccess ||
      cudaMalloc(&b.dotpart, (kDotGrid + 1) * sizeof(double)) != cudaSuccess ||
      cudaMalloc(&b.lpart, (size_t)lgrid * K * sizeof(double)) != cudaSuccess ||
      cudaMalloc(&b.lambda, RP * sizeof(double)) != cudaSuccess) {
    cudaGetLastError();
    return SPLATT_ERROR_NOMEMORY;
  }
  auto blocks = [&](double * base) {
    Blocks x = {};
    for (int m = 0; m < N; ++m) x.p[m] = base + sh.row0[m] * ldm;
    return x;
  };
  Blocks U = {};
  for (int m = 0; m < N; ++m) U.p[m] = d_factors[m];
  Blocks gB = blocks(b.vec), gpB = blocks(b.vec + V), D = blocks(b.vec + 2 * V);
  std::vector<Blocks> S(M), Y(M);
  for (int k = 0; k < M; ++k) { S[k] = blocks(b.vec + (3 + 2 * k) * V); Y[k] = blocks(b.vec + (4 + 2 * k) * V); }
  double * const sc = b.sc;
  auto slot_sc = [&](int k, int f) { return sc + kScSlot + 4 * k + f; };   // f: 0 s.y, 1 y.y, 2 s.q, 3 y.q

  const unsigned vgrid = (unsigned)std::max<unsigned long long>(
      std::min<unsigned long long>((sh.row0[N] + kWarps - 1) / kWarps, (unsigned long long)num_sms() * 8), 1);
  bool ok = true;
  auto dot = [&](const Opnd & x, const Opnd & y, double * out, const double * gate = nullptr, int gm = kAlways) {
    if (!ok) return;
    k_tcg_dot<<<kDotGrid, kThreads, 0, s>>>(sh, x, y, b.dotpart, out, gate, gm);
    spb200_count_launches(1);
    ok = cudaGetLastError() == cudaSuccess;
  };
  auto axpy = [&](const Blocks & Yb, double bb, const Blocks & X, Coef cf, const Blocks * Z = nullptr,
                  double z = 0.0, const double * gate = nullptr, int gm = kAlways) {
    if (!ok) return;
    k_tcg_axpy<<<vgrid, kThreads, 0, s>>>(sh, Yb, bb, X, cf, Z ? *Z : Blocks{}, z, gate, gm);
    spb200_count_launches(1);
    ok = cudaGetLastError() == cudaSuccess;
  };
  auto op = [](const Blocks & A, double a = 1.0) { return Opnd{A, Blocks{}, a, 0.0}; };
  const Coef one = {nullptr, nullptr, nullptr, 1.0};
  const double nnz_train = (double)train->streams[0].nrec;
  const double nnz_val = validate ? (double)validate->streams[0].nrec : 0.0;
  const double * const * cf = d_factors;
  auto enqueue_val = [&]() {
    if (!validate || !ok) return;
    ok = cudaMemsetAsync(sc + kScVal, 0, sizeof(double), s) == cudaSuccess &&
         tc_enqueue_sse(validate->streams[0], R, ldm, cf, b.lambda, sc + kScVal, s) == cudaSuccess;
  };
  auto line = [&]() {
    if (!ok) return;
    const FiberStream & fs = train->streams[train->plan[0].stream];
    if (fs.nrec == 0) { ok = cudaMemsetAsync(b.lpart, 0, (size_t)lgrid * K * sizeof(double), s) == cudaSuccess; return; }
    TcgLine p = {};
    p.w = walk_args(fs, cf, ldm, R);
    for (int l = 0; l < N; ++l) p.dm[l] = D.p[fs.perm[l]];
    p.part = b.lpart;
    lk<<<lgrid, kThreads, tc_ring_bytes(), s>>>(p);
    spb200_count_launches(1);
    ok = cudaGetLastError() == cudaSuccess;
  };
  std::vector<double> lh((size_t)lgrid * K), hs(kScHead);
  auto readback = [&]() {
    ok = ok && cudaMemcpyAsync(lh.data(), b.lpart, lh.size() * sizeof(double), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaMemcpyAsync(hs.data(), sc, kScHead * sizeof(double), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaStreamSynchronize(s) == cudaSuccess;
  };
  // phi's coefficients: the line partials added in CTA order, then reg (|U|^2 + 2 a <U,D> + a^2 |D|^2)
  auto coefs = [&](std::vector<double> & cd, std::vector<double> & c) {
    cd.assign(K, 0.0);
    for (int g = 0; g < lgrid; ++g)
      for (int k = 0; k < K; ++k) cd[k] += lh[(size_t)g * K + k];
    c = cd;
    c[0] += reg * hs[kScUu];
    c[1] += 2.0 * reg * hs[kScUd];
    c[2] += reg * hs[kScDd];
  };

  {
    std::vector<double> ones(RP, 0.0);
    std::fill(ones.begin(), ones.begin() + R, 1.0);
    ok = cudaMemsetAsync(b.vec, 0, (3 + 2 * (size_t)M) * V * sizeof(double), s) == cudaSuccess &&
         cudaMemsetAsync(sc, 0, nsc * sizeof(double), s) == cudaSuccess &&
         cudaMemsetAsync(b.dotpart, 0, (kDotGrid + 1) * sizeof(double), s) == cudaSuccess &&
         cudaMemcpyAsync(b.lambda, ones.data(), RP * sizeof(double), cudaMemcpyHostToDevice, s) == cudaSuccess;
    if (ok) ok = cudaStreamSynchronize(s) == cudaSuccess;    // ones[] is a host temporary
  }
  enqueue_val();                               // the validation SSE at the start, read with iteration 0

  int cnt = 0, newest = M - 1;                 // ring: cnt pairs, the newest in slot `newest`
  double alpha_prev = 0.0;
  uint64_t its = 0;
  double * hrow_prev = nullptr;                // history row whose validation RMSE is pending
  std::vector<double> cd, c;
  auto t0 = std::chrono::steady_clock::now();
  for (uint64_t it = 0; ok && it < niters; ++it) {
    if (verbosity > SPLATT_VERBOSITY_NONE) t0 = std::chrono::steady_clock::now();
    if (it > 0) std::swap(gB, gpB);
    // 1. the gradient g = grad L(U): 2 reg U everywhere, then every mode's walk
    axpy(gB, 0.0, U, Coef{nullptr, nullptr, nullptr, 2.0 * reg});
    for (int m = 0; ok && m < N; ++m) {
      const FiberStream & fs = train->streams[train->plan[m].stream];
      if (!fs.nrec) continue;
      TcArgs a = walk_args(fs, cf, ldm, R);
      a.reg = reg; a.out = gB.p[m]; a.packs = b.slots; a.slot_row = gl[m].rows ? nullptr : b.slot_row;
      ok = gl[m].launch(a, b.slot_row, s) == cudaSuccess;
      if (ok && !gl[m].rows) {
        k_tcg_combine<<<combine_grid(gl[m].nslots), kThreads, 0, s>>>(b.slots, b.slot_row, gl[m].nslots, R, ldm, reg,
                                                                      d_factors[m], gB.p[m]);
        spb200_count_launches(1);
        ok = cudaGetLastError() == cudaSuccess;
      }
    }
    // 4 (of the previous iteration). The pair s = alpha d, y = g - g_prev enters slot t when s.y > 0.
    const bool pending = it > 0 && M > 0 && alpha_prev > 0.0;
    const int t = M > 0 ? (newest + 1) % M : 0;
    if (pending) {
      const Opnd so = op(D, alpha_prev), yo = Opnd{gB, gpB, 1.0, -1.0};
      dot(so, yo, sc + kScSy);
      dot(yo, yo, sc + kScYy);
      axpy(S[t], 0.0, D, Coef{nullptr, nullptr, nullptr, alpha_prev}, nullptr, 0.0, sc + kScSy, kPos);
      axpy(Y[t], 0.0, gB, one, &gpB, -1.0, sc + kScSy, kPos);
      if (ok) {
        k_tcg_copy<<<1, 32, 0, s>>>(sc + kScSy, slot_sc(t, 0), 2, sc + kScSy, kPos);
        spb200_count_launches(1);
        ok = cudaGetLastError() == cudaSuccess;
      }
    }
    // 2. the direction: d = -g, then the two-loop recursion over the ring.  Slot t is the newest
    // pair if the pending pair entered it; otherwise, when the ring is full, it still holds the
    // oldest pair.  Both cases are enqueued, gated on the pending s.y.
    axpy(D, 0.0, gB, Coef{nullptr, nullptr, nullptr, -1.0});
    const bool used = cnt > 0 || pending;
    if (used) {
      struct Step { int k; const double * gate; int gm; };
      std::vector<Step> order;                 // newest to oldest
      if (pending) order.push_back({t, sc + kScSy, kPos});
      for (int i = 0; i < cnt; ++i) {
        const int k = ((newest - i) % M + M) % M;
        if (k == t && pending) continue;       // the oldest of a full ring: after the others
        order.push_back({k, nullptr, kAlways});
      }
      if (pending && cnt == M) order.push_back({t, sc + kScSy, kNotPos});
      for (const Step & st : order) {          // q = s_k . d, d -= (q / s.y) y_k
        dot(op(S[st.k]), op(D), slot_sc(st.k, 2), st.gate, st.gm);
        axpy(D, 1.0, Y[st.k], Coef{slot_sc(st.k, 2), nullptr, slot_sc(st.k, 0), -1.0}, nullptr, 0.0, st.gate, st.gm);
      }
      // H0 = gamma I, gamma = s.y / y.y of the newest pair
      if (pending) axpy(D, 0.0, D, Coef{slot_sc(t, 0), nullptr, slot_sc(t, 1), 1.0}, nullptr, 0.0, sc + kScSy, kPos);
      if (cnt > 0)
        axpy(D, 0.0, D, Coef{slot_sc(newest, 0), nullptr, slot_sc(newest, 1), 1.0}, nullptr, 0.0,
             pending ? sc + kScSy : nullptr, pending ? kNotPos : kAlways);
      for (size_t i = order.size(); i-- > 0;) {   // oldest to newest: d += ((q - y_k . d) / s.y) s_k
        const Step & st = order[i];
        dot(op(Y[st.k]), op(D), slot_sc(st.k, 3), st.gate, st.gm);
        axpy(D, 1.0, S[st.k], Coef{slot_sc(st.k, 2), slot_sc(st.k, 3), slot_sc(st.k, 0), 1.0}, nullptr, 0.0,
             st.gate, st.gm);
      }
      // descent check on the device: d = -g unless g.d < 0
      dot(op(gB), op(D), sc + kScGd);
      axpy(D, 0.0, gB, Coef{nullptr, nullptr, nullptr, -1.0}, nullptr, 0.0, sc + kScGd, kNotNeg);
    }
    // 3. the line: |g|^2, <U,U>, <U,D>, <D,D> and the data coefficients
    dot(op(gB), op(gB), sc + kScGg);
    dot(op(U), op(U), sc + kScUu);
    dot(op(U), op(D), sc + kScUd);
    dot(op(D), op(D), sc + kScDd);
    line();
    readback();
    if (!ok) break;
    if (hrow_prev && validate) hrow_prev[2] = std::sqrt(hs[kScVal] / nnz_val);
    // the ring as the device left it; the direction came from pairs if the ring held any
    const bool entered = pending && hs[kScSy] > 0.0;
    bool lbfgs_dir = cnt > 0 || entered;
    if (entered) { newest = t; cnt = std::min(cnt + 1, M); }
    if (used && !(hs[kScGd] < 0.0)) { cnt = 0; lbfgs_dir = false; }
    const double gnorm = std::sqrt(hs[kScGg]);
    coefs(cd, c);
    double alpha = 0.0, dec = 0.0;
    bool stop = false;
    if (hs[kScGg] == 0.0) {
      stop = true;
    } else {
      splatt_b200_poly_argmin(K - 1, c.data(), &alpha, &dec);
      if (!(dec > 0.0) && lbfgs_dir) {       // retry along -g
        cnt = 0;
        axpy(D, 0.0, gB, Coef{nullptr, nullptr, nullptr, -1.0});
        dot(op(U), op(D), sc + kScUd);
        dot(op(D), op(D), sc + kScDd);
        line();
        readback();
        if (!ok) break;
        coefs(cd, c);
        splatt_b200_poly_argmin(K - 1, c.data(), &alpha, &dec);
      }
      if (!(dec > 0.0)) { alpha = 0.0; dec = 0.0; stop = true; }
    }
    // 4. the update U += alpha D
    const double L = c[0] - dec;
    double trs = 0.0;
    for (int k = K - 1; k >= 0; --k) trs = std::fma(trs, alpha, cd[k]);
    double * row = history ? history + 5 * it : nullptr;
    if (row) {
      row[0] = L; row[1] = std::sqrt(std::max(trs, 0.0) / nnz_train);
      row[2] = validate ? (stop ? std::sqrt(hs[kScVal] / nnz_val) : std::nan("")) : std::nan("");
      row[3] = alpha; row[4] = gnorm;
    }
    hrow_prev = nullptr;
    its = it + 1;
    if (!stop) {
      axpy(U, 1.0, D, Coef{nullptr, nullptr, nullptr, alpha});
      enqueue_val();
      hrow_prev = row;
    }
    alpha_prev = alpha;
    if (verbosity > SPLATT_VERBOSITY_NONE) {
      const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
      printf("  its = %3llu (%0.3fs)  loss = %0.5e  train RMSE = %0.5e  alpha = %0.3e  |g| = %0.3e\n",
             (unsigned long long)its, sec, L, std::sqrt(std::max(trs, 0.0) / nnz_train), alpha, gnorm);
    }
    if (stop || (it > 0 && dec / c[0] < tol)) break;
  }
  if (ok && hrow_prev && validate) {          // the validation RMSE after the last step
    double v = 0.0;
    ok = cudaMemcpyAsync(&v, sc + kScVal, sizeof(double), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaStreamSynchronize(s) == cudaSuccess;
    hrow_prev[2] = std::sqrt(v / nnz_val);
  }
  if (!ok) {
    fprintf(stderr, "SPLATT: splatt_b200_tc_lbfgs_device failed (%s)\n", cudaGetErrorString(cudaGetLastError()));
    cudaStreamSynchronize(s);
    return SPLATT_ERROR_BADINPUT;
  }
  cudaStreamSynchronize(s);
  if (iterations_out) *iterations_out = (int)its;
  return SPLATT_SUCCESS;
}
