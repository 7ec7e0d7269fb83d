// Generalized CP decomposition (GCP) by sampled gradients and Adam on device-resident tensors
// (splatt_b200_gcp_device; Hong, Kolda & Duersch 2020, Kolda & Hong 2020), its sampler and kernel
// primitive (splatt_b200_gcp_sample, splatt_b200_gcp_sampled), and the decode of a device tensor
// back to coordinates (splatt_b200_tensor_to_coo).
//
// A step costs the same whatever nnz is: it draws a fixed number of stored entries and uniform
// coordinates and never walks the tensor.  The kernels:
//   * k_gcp_decode: one warp per 64-record chunk of streams[0].  Lane i takes record i of each
//     half-chunk; its node number at level l is the chunk's descriptor plus the records before it
//     in the chunk that close level l (a ballot and a popcount), so the ids come from up[l].
//   * k_gcp_sample: one thread per sample.  Philox4x32-10 (written out below) gives the draws;
//     a stored-entry draw gathers the coordinates and value from the decoded COO.
//   * k_gcp_sampled<N, B, GRAD, VAL>: one warp per B samples at a time, lane l holding columns
//     2l, 2l+1 as in the walkers.  All B x N row gathers are issued before any is used; m is a
//     warp sum; y = w (df or its stored-entry correction) and every mode's row gets
//     y prod_{k != n} row_k (prefix and suffix products, no division) by red.add.f64.  With VAL
//     the weighted loss is summed per warp in sample order, then over warps and written per CTA;
//     the host adds the CTA partials in order.
//   * k_gcp_adam: one launch over every mode's columns [0, R); it also clears G for the next
//     step, so a step is three launches (sample, gradient, Adam) and no host synchronisation.
#include "walk.cuh"
#include <chrono>
#include <cmath>
#include <vector>

namespace spb200 {
namespace {

// ---- Philox4x32-10 -----------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint4 philox(uint32_t k0, uint32_t k1, uint4 c) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const uint64_t p0 = static_cast<uint64_t>(0xD2511F53u) * c.x;
    const uint64_t p1 = static_cast<uint64_t>(0xCD9E8D57u) * c.z;
    c = make_uint4(static_cast<uint32_t>(p1 >> 32) ^ c.y ^ k0, static_cast<uint32_t>(p1),
                   static_cast<uint32_t>(p0 >> 32) ^ c.w ^ k1, static_cast<uint32_t>(p0));
  }
  return c;
}
__device__ __forceinline__ uint64_t hi_lo(uint32_t a, uint32_t b) { return (static_cast<uint64_t>(a) << 32) | b; }

// ---- losses ------------------------------------------------------------------------------------
__device__ __forceinline__ double f_zero(int loss, double m) {
  if (loss == SPLATT_B200_GCP_GAUSSIAN) return m * m;
  if (loss == SPLATT_B200_GCP_BERNOULLI_LOGIT) return fmax(m, 0.0) + log1p(exp(-fabs(m)));
  return exp(m);
}
__device__ __forceinline__ double df_zero(int loss, double m) {
  if (loss == SPLATT_B200_GCP_GAUSSIAN) return 2.0 * m;
  if (loss == SPLATT_B200_GCP_BERNOULLI_LOGIT) {
    const double e = exp(-fabs(m));
    return m >= 0.0 ? 1.0 / (1.0 + e) : e / (1.0 + e);
  }
  return exp(m);
}
// f(x, m) - f(0, m) and df(x, m) - df(0, m)
__device__ __forceinline__ double f_corr(int loss, double x, double m) {
  return loss == SPLATT_B200_GCP_GAUSSIAN ? x * x - 2.0 * x * m : -x * m;
}
__device__ __forceinline__ double df_corr(int loss, double x) {
  return loss == SPLATT_B200_GCP_GAUSSIAN ? -2.0 * x : -x;
}
bool loss_ok(int loss) { return loss >= SPLATT_B200_GCP_GAUSSIAN && loss <= SPLATT_B200_GCP_POISSON_LOG; }

// ---- decode ------------------------------------------------------------------------------------
struct DecodeArgs {
  const SpRec *      rec;
  const uint32_t *   up[SPB200_MAXN - 2];
  const uint32_t *   desc;
  uint32_t *         ind[SPB200_MAXN];     // by LEVEL
  double *           vals;
  unsigned long long nrec, nchunks;
};

template <int N>
__global__ void __launch_bounds__(kThreads) k_gcp_decode(const __grid_constant__ DecodeArgs a) {
  constexpr int NP = N > 2 ? N - 2 : 1;
  const int lane = threadIdx.x & 31;
  const unsigned long long TW = static_cast<unsigned long long>(gridDim.x) * kWarps;
  for (unsigned long long c = static_cast<unsigned long long>(blockIdx.x) * kWarps + (threadIdx.x >> 5);
       c < a.nchunks; c += TW) {
    uint32_t pos[NP];
#pragma unroll
    for (int l = 0; l < N - 2; ++l) pos[l] = a.desc[c * (N - 2) + l];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const unsigned long long n = c * SPB200_CHUNK + h * 32 + lane;
      const bool ok = n < a.nrec;
      uint4 q = make_uint4(0u, 0u, 0u, 0u);
      if (ok) q = *reinterpret_cast<const uint4 *>(a.rec + n);
      const uint32_t cc = q.w >> SPB200_IDX_BITS;
#pragma unroll
      for (int l = 0; l < N - 2; ++l) {
        const unsigned ball = __ballot_sync(0xffffffffu, ok && cc >= uint32_t(N - 1 - l));
        if (ok) a.ind[l][n] = a.up[l][pos[l] + __popc(ball & ((1u << lane) - 1u))];
        pos[l] += __popc(ball);
      }
      if (ok) {
        a.ind[N - 2][n] = q.w & SPB200_IDX_MASK;
        a.ind[N - 1][n] = q.z;
        a.vals[n] = rec_val<double>(q);
      }
    }
  }
}

// *bad = 1 if a stored value breaks the loss's rule
__global__ void k_gcp_check(const SpRec * __restrict__ rec, unsigned long long n, int loss, int * bad) {
  bool b = false;
  for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    const double v = rec[i].v;
    if (loss == SPLATT_B200_GCP_GAUSSIAN) b |= !isfinite(v);
    else if (loss == SPLATT_B200_GCP_BERNOULLI_LOGIT) b |= !(v == 0.0 || v == 1.0);
    else b |= !(isfinite(v) && v >= 0.0);
  }
  if (__any_sync(0xffffffffu, b) && (threadIdx.x & 31) == 0) atomicOr(bad, 1);
}

// ---- sampling ----------------------------------------------------------------------------------
struct SampleArgs {
  const uint32_t *   coo[SPB200_MAXN];     // by MODE
  const double *     coo_vals;
  uint32_t *         ind[SPB200_MAXN];     // by MODE, p + q each
  double *           vals;
  unsigned long long dims[SPB200_MAXN];
  unsigned long long nnz;
  uint32_t           k0, k1, t_lo, t_hi;
  uint32_t           p, q;
  uint32_t           pnz, pz;              // purposes of the stored-entry and coordinate draws
  int                N;
};

__global__ void __launch_bounds__(kThreads) k_gcp_sample(const __grid_constant__ SampleArgs a) {
  const uint32_t j = blockIdx.x * kThreads + threadIdx.x;
  if (j >= a.p + a.q) return;
  if (j < a.p) {
    const uint4 w = philox(a.k0, a.k1, make_uint4(j, a.t_lo, a.t_hi, 4u * a.pnz));
    const unsigned long long pos = __umul64hi(hi_lo(w.x, w.y), a.nnz);
#pragma unroll
    for (int n = 0; n < SPB200_MAXN; ++n)
      if (n < a.N) a.ind[n][j] = __ldg(&a.coo[n][pos]);
    a.vals[j] = __ldg(&a.coo_vals[pos]);
    return;
  }
  const uint32_t k = j - a.p;
#pragma unroll
  for (int b = 0; b < SPB200_MAXN / 2; ++b) {
    if (2 * b >= a.N) break;
    const uint4 w = philox(a.k0, a.k1, make_uint4(k, a.t_lo, a.t_hi, 4u * a.pz + b));
    a.ind[2 * b][j] = static_cast<uint32_t>(__umul64hi(hi_lo(w.x, w.y), a.dims[2 * b]));
    if (2 * b + 1 < a.N) a.ind[2 * b + 1][j] = static_cast<uint32_t>(__umul64hi(hi_lo(w.z, w.w), a.dims[2 * b + 1]));
  }
  a.vals[j] = 0.0;
}

// ---- sampled value and gradient ----------------------------------------------------------------
struct SampledArgs {
  const uint32_t *   ind[SPB200_MAXN];
  const double *     vals;
  const double *     U[SPB200_MAXN];
  double *           G[SPB200_MAXN];
  double *           part;                 // VAL: one partial per CTA
  unsigned long long p, total;
  double             w_nz, w_z;
  int                ldm, R, loss;
};

// samples a warp keeps in flight: B x N row gathers
__host__ __device__ constexpr int gcp_batch(int N) { return N <= 3 ? 4 : 2; }

template <int N, bool GRAD, bool VAL>
__global__ void __launch_bounds__(kThreads, 2) k_gcp_sampled(const __grid_constant__ SampledArgs a) {
  constexpr int B = gcp_batch(N);
  __shared__ double wsum[kWarps];
  const int  warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool act  = 2 * lane < a.R;
  const bool hasy = 2 * lane + 1 < a.R;
  const uint32_t pitch = static_cast<uint32_t>(a.ldm) * 8u;
  const unsigned long long TW = static_cast<unsigned long long>(gridDim.x) * kWarps;
  double acc = 0.0;
  for (unsigned long long s0 = (static_cast<unsigned long long>(blockIdx.x) * kWarps + warp) * B; s0 < a.total;
       s0 += TW * B) {
    uint32_t idx[B][N];
    double   x[B];
#pragma unroll
    for (int u = 0; u < B; ++u) {
      const unsigned long long s = s0 + u;
      const bool ok = s < a.total;
#pragma unroll
      for (int n = 0; n < N; ++n) idx[u][n] = ok ? __ldg(&a.ind[n][s]) : 0u;
      x[u] = (ok && s < a.p) ? __ldg(&a.vals[s]) : 0.0;
    }
    double2 row[B][N];
#pragma unroll
    for (int u = 0; u < B; ++u) {
#pragma unroll
      for (int n = 0; n < N; ++n) {
        row[u][n] = act ? ld_row<double2>(reinterpret_cast<const char *>(a.U[n] + 2 * lane), idx[u][n], pitch)
                        : make_double2(0.0, 0.0);
        if (!hasy) row[u][n].y = 0.0;
      }
    }
    double m[B];
#pragma unroll
    for (int u = 0; u < B; ++u) {
      double2 pr = row[u][0];
#pragma unroll
      for (int n = 1; n < N; ++n) pr = vmul(pr, row[u][n]);
      m[u] = pr.x + pr.y;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
      for (int u = 0; u < B; ++u) m[u] += __shfl_xor_sync(0xffffffffu, m[u], o);
    }
#pragma unroll
    for (int u = 0; u < B; ++u) {
      const unsigned long long s = s0 + u;
      if (s >= a.total) break;
      const bool stored = s < a.p;
      const double w = stored ? a.w_nz : a.w_z;
      if constexpr (VAL) acc += w * (stored ? f_corr(a.loss, x[u], m[u]) : f_zero(a.loss, m[u]));
      if constexpr (GRAD) {
        const double y = w * (stored ? df_corr(a.loss, x[u]) : df_zero(a.loss, m[u]));
        double2 sfx[N];
        sfx[N - 1] = make_double2(1.0, 1.0);
#pragma unroll
        for (int n = N - 2; n >= 0; --n) sfx[n] = vmul(sfx[n + 1], row[u][n + 1]);
        double2 pre = make_double2(y, y);
#pragma unroll
        for (int n = 0; n < N; ++n) {
          const double2 g = vmul(pre, sfx[n]);
          if (act) {
            double * gp = a.G[n] + static_cast<size_t>(idx[u][n]) * a.ldm + 2 * lane;
            atomicAdd(gp, g.x);
            if (hasy) atomicAdd(gp + 1, g.y);
          }
          pre = vmul(pre, row[u][n]);
        }
      }
    }
  }
  if constexpr (VAL) {
    if (lane == 0) wsum[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
      for (int w = 0; w < kWarps; ++w) t += wsum[w];
      a.part[blockIdx.x] = t;
    }
  }
}

// ---- Adam --------------------------------------------------------------------------------------
struct AdamArgs {
  double *           U[SPB200_MAXN];
  double *           M;                    // moments and gradient: every mode's block, pitch ldm
  double *           V;
  double *           G;
  unsigned long long row0[SPB200_MAXN + 1];
  int                N, R, ldm;
  double             lr, b1, b2, eps, c1, c2;   // c1 = 1 / (1 - b1^k), c2 = 1 / (1 - b2^k)
};

__global__ void __launch_bounds__(kThreads) k_gcp_adam(const __grid_constant__ AdamArgs a) {
  const unsigned long long n_ent = a.row0[a.N] * a.R;
  for (unsigned long long e = blockIdx.x * (unsigned long long)kThreads + threadIdx.x; e < n_ent;
       e += (unsigned long long)gridDim.x * kThreads) {
    const unsigned long long row = e / a.R;
    const int col = static_cast<int>(e - row * a.R);
    int n = 0;
#pragma unroll
    for (int k = 1; k < SPB200_MAXN; ++k)
      if (k < a.N && row >= a.row0[k]) n = k;
    double * U = a.U[0];
#pragma unroll
    for (int k = 1; k < SPB200_MAXN; ++k)
      if (n == k) U = a.U[k];
    const size_t o = static_cast<size_t>(row) * a.ldm + col;
    const double g = a.G[o];
    const double m = a.b1 * a.M[o] + (1.0 - a.b1) * g;
    const double v = a.b2 * a.V[o] + (1.0 - a.b2) * (g * g);
    a.M[o] = m;
    a.V[o] = v;
    a.G[o] = 0.0;
    const size_t uo = static_cast<size_t>(row - a.row0[n]) * a.ldm + col;
    U[uo] -= a.lr * (m * a.c1) / (sqrt(v * a.c2) + a.eps);
  }
}

// ---- host side ---------------------------------------------------------------------------------
bool whole_tensor(const splatt_b200_tensor * t) {
  return t && t->nmodes >= 2 && t->nmodes <= SPB200_MAXN && t->shard_count <= 1 && !t->streams.empty() &&
         stream_fits(t->streams[0]);
}

unsigned grid_for(unsigned long long items, unsigned per_cta) {
  return (unsigned)std::max<unsigned long long>(
      std::min<unsigned long long>((items + per_cta - 1) / per_cta, (unsigned long long)num_sms() * 8), 1);
}

cudaError_t enqueue_decode(const FiberStream & fs, uint32_t * const * ind_by_mode, double * vals, cudaStream_t s) {
  if (!fs.nrec) return cudaSuccess;
  DecodeArgs a = {};
  a.rec = fs.rec;
  for (int l = 0; l < fs.nmodes - 2; ++l) a.up[l] = fs.up[l];
  a.desc = fs.desc;
  for (int l = 0; l < fs.nmodes; ++l) a.ind[l] = ind_by_mode[fs.perm[l]];
  a.vals = vals;
  a.nrec = fs.nrec;
  a.nchunks = fs.nchunks;
  with_nmodes(fs.nmodes, [&](auto n) { k_gcp_decode<n.value><<<grid_for(fs.nchunks, kWarps), kThreads, 0, s>>>(a); });
  spb200_count_launches(1);
  return cudaGetLastError();
}

// The decoded stored entries of a tensor: N index arrays and the values, in one allocation.
struct Coo {
  uint32_t * ind[SPB200_MAXN] = {nullptr};
  double *   vals = nullptr;
  void *     base = nullptr;
};
size_t coo_bytes(int N, unsigned long long n) { return (size_t)n * (4 * N + 8) + 16; }
void coo_carve(Coo & c, void * base, int N, unsigned long long n) {
  c.base = base;
  c.vals = static_cast<double *>(base);
  uint32_t * p = reinterpret_cast<uint32_t *>(c.vals + n);
  for (int m = 0; m < N; ++m) c.ind[m] = p + (size_t)m * n;
}

cudaError_t enqueue_sample(const splatt_b200_tensor * t, const Coo & coo, uint64_t seed, uint64_t step,
                           bool estimate, int p, int q, uint32_t * const * ind, double * vals, cudaStream_t s) {
  SampleArgs a = {};
  for (int m = 0; m < t->nmodes; ++m) {
    a.coo[m] = coo.ind[m];
    a.ind[m] = ind[m];
    a.dims[m] = t->dims[m];
  }
  a.coo_vals = coo.vals;
  a.vals = vals;
  a.nnz = t->streams[0].nrec;
  a.k0 = (uint32_t)seed; a.k1 = (uint32_t)(seed >> 32);
  a.t_lo = (uint32_t)step; a.t_hi = (uint32_t)(step >> 32);
  a.p = (uint32_t)p; a.q = (uint32_t)q;
  a.pnz = estimate ? 2 : 0; a.pz = estimate ? 3 : 1;
  a.N = t->nmodes;
  const unsigned long long total = (unsigned long long)p + q;
  if (!total) return cudaSuccess;
  k_gcp_sample<<<(unsigned)((total + kThreads - 1) / kThreads), kThreads, 0, s>>>(a);
  spb200_count_launches(1);
  return cudaGetLastError();
}

using SampledKernel = void (*)(SampledArgs);
SampledKernel sampled_kernel(int N, bool grad, bool val) {
  return with_nmodes(N, [&](auto n) -> SampledKernel {
    if (grad && val) return k_gcp_sampled<n.value, true, true>;
    if (grad) return k_gcp_sampled<n.value, true, false>;
    return k_gcp_sampled<n.value, false, true>;
  });
}
// Fixed grid of the sampled kernel for `total` samples (the value's sum order follows from it).
unsigned sampled_grid(int N, unsigned long long total) {
  return grid_for((total + gcp_batch(N) - 1) / gcp_batch(N), kWarps);
}

cudaError_t enqueue_sampled(int N, bool grad, bool val, const SampledArgs & a, cudaStream_t s) {
  if (!a.total) return cudaSuccess;
  sampled_kernel(N, grad, val)<<<sampled_grid(N, a.total), kThreads, 0, s>>>(a);
  spb200_count_launches(1);
  return cudaGetLastError();
}

// The value of a VAL launch: its CTA partials added in order on the host.
double sum_parts(const std::vector<double> & h) {
  double v = 0.0;
  for (double x : h) v += x;
  return v;
}

bool gopts_ok(const splatt_b200_gcp_opts & g, uint64_t nnz) {
  auto sample_ok = [&](int p, int q) {
    return p >= 0 && q >= 0 && (long long)p + q >= 1 && (long long)p + q < (1ll << 31) && (nnz > 0 || p == 0);
  };
  return loss_ok(g.loss) && sample_ok(g.grad_nnz, g.grad_zeros) && sample_ok(g.est_nnz, g.est_zeros) &&
         g.epoch_iters >= 1 && std::isfinite(g.lr) && g.lr > 0.0 && std::isfinite(g.beta1) && g.beta1 >= 0.0 &&
         g.beta1 < 1.0 && std::isfinite(g.beta2) && g.beta2 >= 0.0 && g.beta2 < 1.0 &&
         std::isfinite(g.epsilon) && g.epsilon > 0.0 && std::isfinite(g.decay) && g.decay > 0.0 &&
         g.decay <= 1.0 && g.max_fails >= 0;
}

// Device buffers of one splatt_b200_gcp_device call, released on every return path.
struct GcpBuffers {
  void *   coo = nullptr;
  void *   gs = nullptr;        // gradient sample
  void *   es = nullptr;        // estimate sample
  double * mv = nullptr;        // M, V, G, saved M and V, saved U: 6 blocks of rows x ldm
  double * part = nullptr;
  int *    bad = nullptr;
  ~GcpBuffers() {
    cudaFree(coo); cudaFree(gs); cudaFree(es); cudaFree(mv); cudaFree(part); cudaFree(bad);
  }
};

}  // namespace
}  // namespace spb200

using namespace spb200;

extern "C" int splatt_b200_tensor_to_coo(splatt_b200_tensor const * t, uint32_t * const * d_ind, double * d_vals,
                                         void * stream) {
  bool bad = !t || t->nmodes < 2 || t->nmodes > SPB200_MAXN || t->streams.empty() || !d_ind || !d_vals ||
             !stream_fits(t->streams[0]);
  for (int m = 0; !bad && m < t->nmodes; ++m) bad = !d_ind[m];
  if (bad) {
    fprintf(stderr, "SPLATT: splatt_b200_tensor_to_coo: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  DeviceGuard dg(t->device);
  if (!dg.ok) return SPLATT_ERROR_BADINPUT;
  return enqueue_decode(t->streams[0], d_ind, d_vals, static_cast<cudaStream_t>(stream)) == cudaSuccess
             ? SPLATT_SUCCESS
             : SPLATT_ERROR_BADINPUT;
}

extern "C" int splatt_b200_gcp_sample(splatt_b200_tensor const * t, uint64_t seed, uint64_t t_step, int estimate,
                                      int p, int q, uint32_t * const * d_ind, double * d_vals, void * stream) {
  bool bad = !whole_tensor(t) || p < 0 || q < 0 || (long long)p + q < 1 || (long long)p + q >= (1ll << 31) ||
             !d_ind || !d_vals;
  if (!bad) bad = p > 0 && t->streams[0].nrec == 0;
  for (int m = 0; !bad && m < t->nmodes; ++m) bad = !d_ind[m];
  if (bad) {
    fprintf(stderr, "SPLATT: splatt_b200_gcp_sample: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  DeviceGuard dg(t->device);
  if (!dg.ok) return SPLATT_ERROR_BADINPUT;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int N = t->nmodes;
  const unsigned long long nnz = p > 0 ? t->streams[0].nrec : 0;
  Coo coo;
  void * base = nullptr;
  if (nnz) {
    if (cudaMallocAsync(&base, coo_bytes(N, nnz), s) != cudaSuccess) { cudaGetLastError(); return SPLATT_ERROR_NOMEMORY; }
    coo_carve(coo, base, N, nnz);
  }
  cudaError_t e = nnz ? enqueue_decode(t->streams[0], coo.ind, coo.vals, s) : cudaSuccess;
  if (e == cudaSuccess) e = enqueue_sample(t, coo, seed, t_step, estimate != 0, p, q, d_ind, d_vals, s);
  if (base) cudaFreeAsync(base, s);
  return e == cudaSuccess ? SPLATT_SUCCESS : SPLATT_ERROR_BADINPUT;
}

extern "C" int splatt_b200_gcp_sampled(splatt_b200_tensor const * t, int loss, int p, int q, double w_nz, double w_z,
                                       uint32_t const * const * d_ind, double const * d_vals, int ncolumns, int ldm,
                                       double const * const * d_factors, double * const * d_grads, double * value_out,
                                       void * stream) {
  const int R = ncolumns;
  bool bad = !t || t->nmodes < 2 || t->nmodes > SPB200_MAXN || !loss_ok(loss) || p < 0 || q < 0 ||
             (long long)p + q >= (1ll << 31) || !std::isfinite(w_nz) || !std::isfinite(w_z) || !d_ind ||
             (p > 0 && !d_vals) ||
             !factors_ok(t ? t->nmodes : 0, R, ldm, reinterpret_cast<const void * const *>(d_factors));
  if (!bad && d_grads) bad = !factors_ok(t->nmodes, R, ldm, reinterpret_cast<const void * const *>(d_grads));
  for (int m = 0; !bad && m < t->nmodes; ++m) bad = !d_ind[m];
  if (bad) {
    fprintf(stderr, "SPLATT: splatt_b200_gcp_sampled: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  DeviceGuard dg(t->device);
  if (!dg.ok) return SPLATT_ERROR_BADINPUT;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int N = t->nmodes;
  SampledArgs a = {};
  for (int m = 0; m < N; ++m) {
    a.ind[m] = d_ind[m];
    a.U[m] = d_factors[m];
    a.G[m] = d_grads ? d_grads[m] : nullptr;
  }
  a.vals = d_vals;
  a.p = (unsigned long long)p;
  a.total = (unsigned long long)p + q;
  a.w_nz = w_nz; a.w_z = w_z;
  a.ldm = ldm; a.R = R; a.loss = loss;
  cudaError_t e = cudaSuccess;
  for (int m = 0; d_grads && e == cudaSuccess && m < N; ++m)
    e = cudaMemset2DAsync(d_grads[m], (size_t)ldm * 8, 0, (size_t)R * 8, t->dims[m], s);
  const unsigned grid = sampled_grid(N, a.total);
  if (e == cudaSuccess && value_out && a.total) e = cudaMallocAsync(&a.part, grid * sizeof(double), s);
  if (e == cudaSuccess && (d_grads || value_out)) e = enqueue_sampled(N, d_grads != nullptr, value_out != nullptr, a, s);
  if (value_out && e == cudaSuccess) {
    std::vector<double> h(a.total ? grid : 0);
    if (a.total) e = cudaMemcpyAsync(h.data(), a.part, grid * sizeof(double), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e == cudaSuccess) *value_out = sum_parts(h);
  }
  if (a.part) cudaFreeAsync(a.part, s);
  if (e != cudaSuccess) {
    fprintf(stderr, "SPLATT: splatt_b200_gcp_sampled failed (%s)\n", cudaGetErrorString(e));
    cudaGetLastError();
    return e == cudaErrorMemoryAllocation ? SPLATT_ERROR_NOMEMORY : SPLATT_ERROR_BADINPUT;
  }
  return SPLATT_SUCCESS;
}

extern "C" int splatt_b200_gcp_device(splatt_b200_tensor const * t, int ncolumns, int ldm, double const * options,
                                      splatt_b200_gcp_opts const * gopts, double * const * d_factors,
                                      double * history, double * f_start_out, int * epochs_out, void * stream) {
  const int R = ncolumns;
  splatt_b200_gcp_opts g = {SPLATT_B200_GCP_BERNOULLI_LOGIT, 1 << 16, 1 << 16, 1 << 20, 1 << 20, 1000,
                            1e-3, 0.9, 0.999, 1e-8, 0.1, 1, 0};
  if (gopts) g = *gopts;
  bool bad = !whole_tensor(t) || !options ||
             !factors_ok(t->nmodes, R, ldm, reinterpret_cast<const void * const *>(d_factors));
  if (!bad) {
    const double ni = options[SPLATT_OPTION_NITER];
    bad = !gopts_ok(g, t->streams[0].nrec) || !std::isfinite(options[SPLATT_OPTION_TOLERANCE]) ||
          !(ni >= 0.0 && ni < 2147483648.0);
  }
  if (bad) {
    fprintf(stderr, "SPLATT: splatt_b200_gcp_device: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  DeviceGuard dg(t->device);
  if (!dg.ok) return SPLATT_ERROR_BADINPUT;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int N = t->nmodes;
  const FiberStream & fs = t->streams[0];
  const unsigned long long nnz = fs.nrec;
  const uint64_t niters = (uint64_t)options[SPLATT_OPTION_NITER];
  const double tol = options[SPLATT_OPTION_TOLERANCE];
  const int verbosity = (int)options[SPLATT_OPTION_VERBOSITY];
  GcpBuffers b;

  // 1. the values against the loss's rule
  {
    int hbad = 0;
    if (cudaMalloc(&b.bad, sizeof(int)) != cudaSuccess) { cudaGetLastError(); return SPLATT_ERROR_NOMEMORY; }
    bool ok = cudaMemsetAsync(b.bad, 0, sizeof(int), s) == cudaSuccess;
    if (ok && nnz) {
      k_gcp_check<<<grid_for(nnz, kThreads), kThreads, 0, s>>>(fs.rec, nnz, g.loss, b.bad);
      spb200_count_launches(1);
      ok = cudaGetLastError() == cudaSuccess;
    }
    ok = ok && cudaMemcpyAsync(&hbad, b.bad, sizeof(int), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaStreamSynchronize(s) == cudaSuccess;
    if (!ok) return SPLATT_ERROR_BADINPUT;
    if (hbad) {
      fprintf(stderr, "SPLATT: splatt_b200_gcp_device: a tensor value is not allowed by the loss\n");
      return SPLATT_ERROR_BADINPUT;
    }
  }

  // 2. buffers: the decoded entries, both samples, the moments, the gradient and the saved state
  unsigned long long row0[SPB200_MAXN + 1] = {0};
  for (int m = 0; m < N; ++m) row0[m + 1] = row0[m] + t->dims[m];
  const size_t blk = (size_t)row0[N] * ldm;
  const unsigned long long gtot = (unsigned long long)g.grad_nnz + g.grad_zeros;
  const unsigned long long etot = (unsigned long long)g.est_nnz + g.est_zeros;
  const unsigned egrid = sampled_grid(N, etot);
  if (cudaMalloc(&b.coo, coo_bytes(N, nnz)) != cudaSuccess || cudaMalloc(&b.gs, coo_bytes(N, gtot)) != cudaSuccess ||
      cudaMalloc(&b.es, coo_bytes(N, etot)) != cudaSuccess ||
      cudaMalloc(&b.mv, 6 * blk * sizeof(double)) != cudaSuccess ||
      cudaMalloc(&b.part, egrid * sizeof(double)) != cudaSuccess) {
    cudaGetLastError();
    return SPLATT_ERROR_NOMEMORY;
  }
  Coo coo, gsmp, esmp;
  coo_carve(coo, b.coo, N, nnz);
  coo_carve(gsmp, b.gs, N, gtot);
  coo_carve(esmp, b.es, N, etot);
  double * const Mo = b.mv;
  double * const Vo = b.mv + blk;
  double * const G = b.mv + 2 * blk;
  double * const Ms = b.mv + 3 * blk;     // saved M, then saved V: both moments move as one block
  double * const Us = b.mv + 5 * blk;
  const double total = [&] { double x = 1.0; for (int m = 0; m < N; ++m) x *= (double)t->dims[m]; return x; }();
  const double gw_nz = g.grad_nnz ? (double)nnz / g.grad_nnz : 0.0, gw_z = g.grad_zeros ? total / g.grad_zeros : 0.0;
  const double ew_nz = g.est_nnz ? (double)nnz / g.est_nnz : 0.0, ew_z = g.est_zeros ? total / g.est_zeros : 0.0;

  bool ok = cudaMemsetAsync(b.mv, 0, 3 * blk * sizeof(double), s) == cudaSuccess &&
            enqueue_decode(fs, coo.ind, coo.vals, s) == cudaSuccess &&
            enqueue_sample(t, coo, g.seed, 0, true, g.est_nnz, g.est_zeros, esmp.ind, esmp.vals, s) == cudaSuccess;

  SampledArgs ga = {}, ea = {};
  for (int m = 0; m < N; ++m) {
    ga.ind[m] = gsmp.ind[m]; ga.U[m] = d_factors[m]; ga.G[m] = G + row0[m] * ldm;
    ea.ind[m] = esmp.ind[m]; ea.U[m] = d_factors[m];
  }
  ga.vals = gsmp.vals; ga.p = g.grad_nnz; ga.total = gtot; ga.w_nz = gw_nz; ga.w_z = gw_z;
  ga.ldm = ldm; ga.R = R; ga.loss = g.loss;
  ea.vals = esmp.vals; ea.p = g.est_nnz; ea.total = etot; ea.w_nz = ew_nz; ea.w_z = ew_z;
  ea.ldm = ldm; ea.R = R; ea.loss = g.loss; ea.part = b.part;
  AdamArgs aa = {};
  for (int m = 0; m < N; ++m) aa.U[m] = d_factors[m];
  for (int m = 0; m <= N; ++m) aa.row0[m] = row0[m];
  aa.M = Mo; aa.V = Vo; aa.G = G; aa.N = N; aa.R = R; aa.ldm = ldm;
  aa.b1 = g.beta1; aa.b2 = g.beta2; aa.eps = g.epsilon;
  const unsigned agrid = grid_for(row0[N] * R, kThreads);

  std::vector<double> eh(egrid);
  auto estimate = [&](double & v) {
    ok = ok && enqueue_sampled(N, false, true, ea, s) == cudaSuccess &&
         cudaMemcpyAsync(eh.data(), b.part, egrid * sizeof(double), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaStreamSynchronize(s) == cudaSuccess;
    v = sum_parts(eh);
  };
  // U's columns [0, R) and the moments: save (to the epoch-start copies) or restore
  auto state = [&](bool save) {
    for (int m = 0; ok && m < N; ++m) {
      double * us = Us + row0[m] * ldm;
      ok = cudaMemcpy2DAsync(save ? us : d_factors[m], (size_t)ldm * 8, save ? d_factors[m] : us, (size_t)ldm * 8,
                             (size_t)R * 8, t->dims[m], cudaMemcpyDeviceToDevice, s) == cudaSuccess;
    }
    ok = ok && cudaMemcpyAsync(save ? Ms : Mo, save ? Mo : Ms, 2 * blk * sizeof(double), cudaMemcpyDeviceToDevice,
                               s) == cudaSuccess;
  };

  double prev = 0.0;
  estimate(prev);
  if (!ok) {
    fprintf(stderr, "SPLATT: splatt_b200_gcp_device failed (%s)\n", cudaGetErrorString(cudaGetLastError()));
    cudaStreamSynchronize(s);
    return SPLATT_ERROR_BADINPUT;
  }
  if (f_start_out) *f_start_out = prev;
  uint64_t step = 0, epochs = 0;
  double lr = g.lr;
  int fails = 0;
  for (uint64_t ep = 0; ok && ep < niters; ++ep) {
    const auto t0 = std::chrono::steady_clock::now();
    const uint64_t step0 = step;
    state(true);
    for (int it = 0; ok && it < g.epoch_iters; ++it, ++step) {
      ok = enqueue_sample(t, coo, g.seed, step, false, g.grad_nnz, g.grad_zeros, gsmp.ind, gsmp.vals, s) == cudaSuccess &&
           enqueue_sampled(N, true, false, ga, s) == cudaSuccess;
      if (!ok) break;
      aa.lr = lr;
      aa.c1 = 1.0 / (1.0 - std::pow(g.beta1, (double)(step + 1)));
      aa.c2 = 1.0 / (1.0 - std::pow(g.beta2, (double)(step + 1)));
      k_gcp_adam<<<agrid, kThreads, 0, s>>>(aa);
      spb200_count_launches(1);
      ok = cudaGetLastError() == cudaSuccess;
    }
    double est = 0.0;
    estimate(est);
    if (!ok) break;
    const bool accepted = std::isfinite(est) && est <= prev;
    if (history) {
      history[3 * ep] = est;
      history[3 * ep + 1] = lr;
      history[3 * ep + 2] = accepted ? 1.0 : 0.0;
    }
    epochs = ep + 1;
    if (verbosity > SPLATT_VERBOSITY_NONE) {
      const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
      printf("  epoch = %3llu (%0.3fs)  f~ = %0.5e  lr = %0.3e  %s\n", (unsigned long long)epochs, sec, est, lr,
             accepted ? "accepted" : "failed");
    }
    if (accepted) {
      const double rel = prev != 0.0 ? (prev - est) / std::fabs(prev) : 0.0;
      prev = est;
      if (rel < tol) break;
    } else {
      state(false);
      step = step0;
      lr *= g.decay;
      if (++fails > g.max_fails) break;
    }
  }
  if (!ok) {
    fprintf(stderr, "SPLATT: splatt_b200_gcp_device failed (%s)\n", cudaGetErrorString(cudaGetLastError()));
    cudaStreamSynchronize(s);
    return SPLATT_ERROR_BADINPUT;
  }
  cudaStreamSynchronize(s);
  if (epochs_out) *epochs_out = (int)epochs;
  return SPLATT_SUCCESS;
}
