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

  // input rules on the device: values and start entries finite and >= 0, start columns sum > 0
  const FiberStream & fs0 = t->streams[0];
  ok = cudaMemsetAsync(b.bad, 0, sizeof(int), s) == cudaSuccess &&
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
    fprintf(stderr, "SPLATT: splatt_b200_cp_apr_device failed (%s)\n", cudaGetErrorString(cudaGetLastError()));
    return SPLATT_ERROR_BADINPUT;
  }
  for (int m = 0; m < N && !hbad; ++m)
    for (int r = 0; r < R; ++r)
      if (!(std::isfinite(hs[(size_t)m * RP + r]) && hs[(size_t)m * RP + r] > 0.0)) hbad = 1;
  if (hbad) {
    fprintf(stderr, "SPLATT: splatt_b200_cp_apr_device: a tensor value or start entry is negative or not "
                    "finite, or a start column sums to 0\n");
    return SPLATT_ERROR_BADINPUT;
  }

  // start: every column divided by its sum, lambda_r = prod_m s_{m,r}
  std::vector<double> lam(RP, 0.0);
  for (int r = 0; r < R; ++r) {
    lam[r] = 1.0;
    for (int m = 0; m < N; ++m) lam[r] *= hs[(size_t)m * RP + r];
  }
  ok = cudaMemcpyAsync(b.lam, lam.data(), RP * sizeof(double), cudaMemcpyHostToDevice, s) == cudaSuccess &&
       cudaMemsetAsync(b.B, 0, max_dim * ldm * sizeof(double), s) == cudaSuccess;
  for (int m = 0; ok && m < N; ++m) {
    k_apr_normalize<<<elementwise_grid(t->dims[m], R), kThreads, 0, s>>>(d_factors[m], b.sums + (size_t)m * RP,
                                                                         d_factors[m], t->dims[m], R, ldm);
    spb200_count_launches(1);
    ok = cudaMemsetAsync(b.phi[m], 0, t->dims[m] * ldm * sizeof(double), s) == cudaSuccess;
  }

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
