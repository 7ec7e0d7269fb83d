// CPD-ALS driver with the MTTKRP on the GPU (drop-in for splatt_cpd_als).
//
// Follows the iteration of the reference's cpd_als_iterate (src/cpd.c:271-387):
//   per mode: M1 = MTTKRP -> A_m = M1 * (hadamard of the other Grams)^-1
//             -> column normalise (2-norm in iteration 0, max-norm afterwards)
//             -> Gram update;   per iteration: fit from the last mode's M1.
// Per the north star the small dense algebra stays on the host; it is written
// here in plain C++ (Cholesky / triangular solves on R x R, R = rank) so the
// library has no BLAS/LAPACK dependency.  Factor matrices are kept resident on
// the device: only the matrix updated in a mode step crosses PCIe (H2D), plus
// the MTTKRP result (D2H).
#include "common.h"
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include <vector>

namespace {

// reference: src/util.c:15-23 (two rand() draws per value)
double rand_val() {
  double v = 3.0 * ((double)rand() / (double)RAND_MAX);
  if (rand() % 2 == 0) v *= -1;
  return v;
}

// G = A^T A, upper triangle in row-major (what the reference's syrk call leaves,
// src/matrix.c:414-455); lower triangle is not referenced by consumers.
void gram(const double * A, uint64_t I, int R, double * G) {
  std::vector<double> acc((size_t)R * R, 0.0);
#pragma omp parallel
  {
    std::vector<double> loc((size_t)R * R, 0.0);
#pragma omp for schedule(static) nowait
    for (int64_t i = 0; i < (int64_t)I; ++i) {
      const double * a = A + (size_t)i * R;
      for (int p = 0; p < R; ++p) {
        const double ap = a[p];
        double * row = loc.data() + (size_t)p * R;
        for (int q = p; q < R; ++q) row[q] += ap * a[q];
      }
    }
#pragma omp critical
    for (size_t x = 0; x < loc.size(); ++x) acc[x] += loc[x];
  }
  memcpy(G, acc.data(), sizeof(double) * R * R);
}

// Normal-equation matrix: Hadamard of the other modes' Grams, symmetrised.
// NOTE: in the reference the `1 + reg` written on the diagonal is immediately
// overwritten by the row fill (src/matrix.c:45-51), i.e. the regularisation
// parameter has no effect; that effective behaviour is reproduced.
// ata: the N Grams, R x R each, one after the other
void form_normal_matrix(const double * ata, int mode, int N, int R, double * neq) {
  for (int x = 0; x < R * R; ++x) neq[x] = 1.0;
  for (int m = 0; m < N; ++m) {
    if (m == mode) continue;
    for (int i = 0; i < R; ++i)
      for (int j = i; j < R; ++j) neq[j + i * R] *= ata[(size_t)m * R * R + j + i * R];
  }
  for (int i = 0; i < R; ++i)
    for (int j = 0; j < i; ++j) neq[j + i * R] = neq[i + j * R];
}

// In-place Cholesky G = L L^T (lower, row-major).  false if not SPD.
bool cholesky(double * G, int R) {
  for (int j = 0; j < R; ++j) {
    double d = G[j + j * R];
    for (int k = 0; k < j; ++k) d -= G[k + j * R] * G[k + j * R];
    if (!(d > 0.0)) return false;
    d = std::sqrt(d);
    G[j + j * R] = d;
    for (int i = j + 1; i < R; ++i) {
      double s = G[j + i * R];
      for (int k = 0; k < j; ++k) s -= G[k + i * R] * G[k + j * R];
      G[j + i * R] = s / d;
    }
  }
  return true;
}

// rows of X <- rows of X * (L L^T)^-1
void cholesky_solve_rows(const double * L, int R, double * X, uint64_t I) {
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < (int64_t)I; ++i) {
    double * x = X + (size_t)i * R;
    for (int p = 0; p < R; ++p) {          // L y = x
      double s = x[p];
      for (int k = 0; k < p; ++k) s -= L[k + p * R] * x[k];
      x[p] = s / L[p + p * R];
    }
    for (int p = R - 1; p >= 0; --p) {     // L^T z = y
      double s = x[p];
      for (int k = p + 1; k < R; ++k) s -= L[p + k * R] * x[k];
      x[p] = s / L[p + p * R];
    }
  }
}

#include "jacobi.cuh"

// Minimum-norm least squares for a symmetric (possibly singular) G: the role of
// the reference's GELSS fallback (src/matrix.c:566-603).
void pinv_solve_rows(const double * Gin, int R, double * X, uint64_t I) {
  std::vector<double> A(Gin, Gin + (size_t)R * R), V((size_t)R * R), P((size_t)R * R);
  const int erank = jacobi_pinv(A.data(), V.data(), R, P.data());
  printf("SPLATT:   pseudo-inverse effective rank: %d\n", erank);
#pragma omp parallel
  {
    std::vector<double> tmp(R);
#pragma omp for schedule(static)
    for (int64_t i = 0; i < (int64_t)I; ++i) {
      double * x = X + (size_t)i * R;
      for (int j = 0; j < R; ++j) {
        double s = 0;
        for (int k = 0; k < R; ++k) s += x[k] * P[j + k * R];
        tmp[j] = s;
      }
      memcpy(x, tmp.data(), sizeof(double) * R);
    }
  }
}

// reference: p_mat_2norm / p_mat_maxnorm (src/matrix.c:86-199)
void normalize_cols(double * A, uint64_t I, int R, double * lambda, bool two_norm) {
  std::vector<double> acc(R, 0.0);
#pragma omp parallel
  {
    std::vector<double> loc(R, 0.0);
#pragma omp for schedule(static) nowait
    for (int64_t i = 0; i < (int64_t)I; ++i) {
      const double * a = A + (size_t)i * R;
      if (two_norm) for (int j = 0; j < R; ++j) loc[j] += a[j] * a[j];
      else for (int j = 0; j < R; ++j) loc[j] = std::max(loc[j], a[j]);
    }
#pragma omp critical
    for (int j = 0; j < R; ++j) acc[j] = two_norm ? acc[j] + loc[j] : std::max(acc[j], loc[j]);
  }
  for (int j = 0; j < R; ++j) lambda[j] = two_norm ? std::sqrt(acc[j]) : std::max(acc[j], 1.0);
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < (int64_t)I; ++i) {
    double * a = A + (size_t)i * R;
    for (int j = 0; j < R; ++j) a[j] /= lambda[j];
  }
}

// reference: p_kruskal_norm src/cpd.c:116-152
double kruskal_norm(const double * ata, const double * lambda, int N, int R) {
  std::vector<double> av((size_t)R * R, 1.0);
  for (int m = 0; m < N; ++m)
    for (int i = 0; i < R; ++i)
      for (int j = i; j < R; ++j) av[j + i * R] *= ata[(size_t)m * R * R + j + i * R];
  double nm = 0;
  for (int i = 0; i < R; ++i) {
    nm += av[i + i * R] * lambda[i] * lambda[i];
    for (int j = i + 1; j < R; ++j) nm += av[j + i * R] * lambda[i] * lambda[j] * 2;
  }
  return std::fabs(nm);
}

// reference: p_tt_kruskal_inner src/cpd.c:171-218
double kruskal_inner(const double * last, const double * m1, uint64_t I, int R,
                     const double * lambda) {
  std::vector<double> acc(R, 0.0);
#pragma omp parallel
  {
    std::vector<double> loc(R, 0.0);
#pragma omp for schedule(static) nowait
    for (int64_t i = 0; i < (int64_t)I; ++i)
      for (int r = 0; r < R; ++r) loc[r] += last[r + (size_t)i * R] * m1[r + (size_t)i * R];
#pragma omp critical
    for (int r = 0; r < R; ++r) acc[r] += loc[r];
  }
  double inner = 0;
  for (int r = 0; r < R; ++r) inner += acc[r] * lambda[r];
  return inner;
}

// fit = 1 - ||X - K|| / ||X||  (reference: p_calc_fit src/cpd.c:237-265)
double cpd_fit(const double * ata, const double * lambda, int N, int R, double ttnormsq,
               double inner) {
  const double norm_mats = kruskal_norm(ata, lambda, N, R);
  double residual = ttnormsq + norm_mats - 2 * inner;
  if (residual > 0.) residual = std::sqrt(residual);
  return 1 - residual / std::sqrt(ttnormsq);
}

}  // namespace

double spb200_csf_frobsq(const splatt_csf * t) {   // reference: src/csf.c:817-851
  double norm = 0;
  const int N = (int)t->nmodes;
  for (uint64_t tile = 0; tile < t->ntiles; ++tile) {
    const double * v = t->pt[tile].vals;
    if (!v) continue;
    const uint64_t n = t->pt[tile].nfibs[N - 1];
#pragma omp parallel for reduction(+ : norm) schedule(static)
    for (int64_t i = 0; i < (int64_t)n; ++i) norm += v[i] * v[i];
  }
  return norm;
}

AlsIterations::AlsIterations(const double * options)
    : niters((uint64_t)options[SPLATT_OPTION_NITER]), tol(options[SPLATT_OPTION_TOLERANCE]),
      verbosity((int)options[SPLATT_OPTION_VERBOSITY]) {}

void AlsIterations::start() { t0 = std::chrono::steady_clock::now(); }

bool AlsIterations::done(uint64_t it, double fit) {
  if (verbosity > SPLATT_VERBOSITY_NONE)
    printf("  its = %3llu (%0.3fs)  fit = %0.5f  delta = %+0.4e\n", (unsigned long long)it + 1,
           std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(), fit,
           fit - oldfit);
  if (fit == 1. || (it > 0 && std::fabs(fit - oldfit) < tol)) return true;
  oldfit = fit;
  return false;
}

HostKruskal::~HostKruskal() {
  for (int m = 0; m < N; ++m) free(mats[m]);
  free(lambda);
}

bool HostKruskal::start(int N_, const uint64_t * dims_, int R_) {
  N = N_; R = R_;
  memcpy(dims, dims_, sizeof(uint64_t) * N);
  lambda = static_cast<double *>(malloc(sizeof(double) * R));
  bool ok = lambda != nullptr;
  for (int m = 0; m < N && ok; ++m) {
    mats[m] = static_cast<double *>(malloc(sizeof(double) * dims[m] * R));
    ok = mats[m] != nullptr;
    if (ok) for (uint64_t x = 0; x < dims[m] * (uint64_t)R; ++x) mats[m][x] = rand_val();
  }
  return ok;
}

void HostKruskal::finish(double fit, splatt_kruskal * out) {
  std::vector<double> tmp(R);
  for (int m = 0; m < N; ++m) {
    normalize_cols(mats[m], dims[m], R, tmp.data(), true);
    for (int f = 0; f < R; ++f) lambda[f] *= tmp[f];
  }
  out->fit = fit;
  out->rank = (splatt_idx_t)R;
  out->nmodes = (splatt_idx_t)N;
  out->lambda = lambda;
  lambda = nullptr;
  for (int m = 0; m < N; ++m) {
    out->dims[m] = dims[m];
    out->factors[m] = mats[m];
    mats[m] = nullptr;
  }
}

namespace {

// ---------------------------------------------------------------------------
// Device-side ALS tail (SURVEY.md 8(f) #1): the same five steps as the host
// functions above, as small kernels on the MTTKRP stream, so that an iteration
// needs no host<->device traffic except one tiny read-back for the fit.
// ---------------------------------------------------------------------------

// G(upper, row-major) += A^T A over a block of rows.  reference: mat_aTa src/matrix.c:414-455
// T is the storage type of A (double or float); G and the arithmetic are fp64.
template <class T>
__global__ void k_gram(const T * __restrict__ A, unsigned long long I, int R, int lda,
                       double * __restrict__ G) {
  extern __shared__ double tile[];           // 32 rows x R
  const int nent = R * (R + 1) / 2;
  constexpr int kMaxPer = 34;                // R <= 128: ceil(8256 / 256) = 33
  double acc[kMaxPer];
  short  ep[kMaxPer], eq[kMaxPer];
  int    mine = 0;
  for (int e = threadIdx.x; e < nent && mine < kMaxPer; e += blockDim.x) {
    int p = 0, rem = e;                      // e -> (p, q >= p), row-major upper triangle
    while (rem >= R - p) { rem -= R - p; ++p; }
    ep[mine] = (short)p; eq[mine] = (short)(p + rem); acc[mine] = 0.0; ++mine;
  }
  for (unsigned long long r0 = (unsigned long long)blockIdx.x * 32; r0 < I;
       r0 += (unsigned long long)gridDim.x * 32) {
    const int rows = (int)min((unsigned long long)32, I - r0);
    for (int x = threadIdx.x; x < rows * R; x += blockDim.x)
      tile[x] = static_cast<double>(A[(r0 + x / R) * lda + (x % R)]);
    __syncthreads();
    for (int t = 0; t < mine; ++t) {
      double a = acc[t];
      for (int i = 0; i < rows; ++i) a = fma(tile[i * R + ep[t]], tile[i * R + eq[t]], a);
      acc[t] = a;
    }
    __syncthreads();
  }
  for (int t = 0; t < mine; ++t) atomicAdd(&G[eq[t] + ep[t] * R], acc[t]);
}

// Normal matrix = Hadamard of the other modes' Grams; Cholesky in shared memory.
// reference: p_form_gram src/matrix.c:29-83 + potrf :554.  info = 1 when not SPD; then P holds
// the pseudo-inverse (the role of the GELSS fallback :566-603).
__global__ void k_form_chol(const double * __restrict__ ata, int nmodes, int mode, int R,
                            double * __restrict__ Lout, double * __restrict__ Pout,
                            double * __restrict__ Vscratch, int * __restrict__ info) {
  extern __shared__ double sm[];             // R*R working copy (the fallback's V is in global)
  double * a = sm;
  __shared__ int bad;
  if (threadIdx.x == 0) bad = 0;
  for (int x = threadIdx.x; x < R * R; x += blockDim.x) {
    const int i = x / R, j = x % R;
    const int p = min(i, j), q = max(i, j);  // Grams are stored upper (row-major)
    double v = 1.0;
    for (int m = 0; m < nmodes; ++m)
      if (m != mode) v *= ata[(size_t)m * R * R + q + p * R];
    a[x] = v;
    Pout[x] = v;                             // keep the unfactored matrix for the fallback
  }
  __syncthreads();
  for (int j = 0; j < R && !bad; ++j) {
    if (threadIdx.x == 0) {
      const double d = a[j + j * R];
      if (!(d > 0.0)) bad = 1; else a[j + j * R] = sqrt(d);
    }
    __syncthreads();
    if (bad) break;
    const double djj = a[j + j * R];
    for (int i = j + 1 + threadIdx.x; i < R; i += blockDim.x) a[j + i * R] /= djj;
    __syncthreads();
    // trailing update of the lower triangle: a[i][k] -= L[i][j] * L[k][j], i >= k > j
    const int rem = R - j - 1;
    for (int x = threadIdx.x; x < rem * rem; x += blockDim.x) {
      const int i = j + 1 + x / rem, k = j + 1 + x % rem;
      if (k <= i) a[k + i * R] -= a[j + i * R] * a[j + k * R];
    }
    __syncthreads();
  }
  __syncthreads();
  if (!bad) {
    for (int x = threadIdx.x; x < R * R; x += blockDim.x) Lout[x] = a[x];
    if (threadIdx.x == 0) *info = 0;
    return;
  }
  // not SPD: pseudo-inverse of the unfactored matrix (one thread; rare path)
  if (threadIdx.x == 0) {
    for (int x = 0; x < R * R; ++x) a[x] = Pout[x];
    jacobi_pinv(a, Vscratch, R, Pout);
    *info = 1;
  }
}

// One thread per row: X[i,:] = M1[i,:] * (L L^T)^-1 (or * P when info != 0).
// reference: potrs call src/matrix.c:563 (nrhs = rows).  Row scratch lives in shared memory,
// laid out [r][thread] so that accesses are conflict-free; L is read as a broadcast.
// Rows are stored as T and solved in fp64; the result is rounded to T once.
template <class T>
__global__ void k_solve_rows(const T * __restrict__ M1, T * __restrict__ X,
                             unsigned long long I, int R, int ld, const double * __restrict__ L,
                             const double * __restrict__ P, const int * __restrict__ info,
                             int only_fallback) {
  extern __shared__ double sm[];
  double * Ls = sm;                         // R*R
  double * xs = sm + R * R;                 // R * blockDim.x
  const bool use_p = (*info != 0);
  if (only_fallback && !use_p) return;      // the register-tiled kernel did the work
  const double * src = use_p ? P : L;
  for (int x = threadIdx.x; x < R * R; x += blockDim.x) Ls[x] = src[x];
  __syncthreads();
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= I) return;
  const int NT = blockDim.x, t = threadIdx.x;
  const T * row = M1 + i * ld;
  for (int r = 0; r < R; ++r) xs[r * NT + t] = static_cast<double>(row[r]);
  T * out = X + i * ld;
  if (!use_p) {
    for (int p = 0; p < R; ++p) {           // L y = x
      double s = xs[p * NT + t];
      for (int k = 0; k < p; ++k) s = fma(-Ls[k + p * R], xs[k * NT + t], s);
      xs[p * NT + t] = s / Ls[p + p * R];
    }
    for (int p = R - 1; p >= 0; --p) {      // L^T z = y
      double s = xs[p * NT + t];
      for (int k = p + 1; k < R; ++k) s = fma(-Ls[p + k * R], xs[k * NT + t], s);
      s /= Ls[p + p * R];
      xs[p * NT + t] = s;
      out[p] = static_cast<T>(s);
    }
  } else {
    for (int j = 0; j < R; ++j) {
      double s = 0;
      for (int k = 0; k < R; ++k) s = fma(xs[k * NT + t], Ls[j + k * R], s);
      out[j] = static_cast<T>(s);
    }
  }
}

// ---------------------------------------------------------------------------
// Register-tiled versions of the two O(I R^2) steps for R <= 64 (RT = R padded to 16/32/64).
// The generic kernels above spend two shared-memory reads per fp64 FMA (ncu launch list of
// one ALS iteration, profiles/r02_cpd_tail.md: 1M x 64 factor: k_solve_rows 2.76 ms, k_gram
// 1.2 ms -- 41 % of the iteration); here the row / the 4x4 output block lives in registers.
// ---------------------------------------------------------------------------

// X[i,:] = M1[i,:] * (L L^T)^-1, one thread per row, the row in registers, L (padded with an
// identity block to RT) and its transpose in shared memory, read as 128-bit broadcasts.
// reference: potrs call src/matrix.c:563.  (*info != 0: the generic kernel handles it.)
// fp32 rows (ld % 4 == 0) move as float4; columns [R, RT) enter as 0 by selection, so the
// unspecified pad columns of an fp32 M1 (NaN included) are loaded but never reach the solve.
template <int RT, class T>
__global__ void __launch_bounds__(128)
k_solve_rows_reg(const T * __restrict__ M1, T * __restrict__ X, unsigned long long I,
                 int R, int ld, const double * __restrict__ L, const int * __restrict__ info) {
  extern __shared__ __align__(16) double sm[];
  double * Ls  = sm;                    // RT*RT, row-major lower factor
  double * Lt  = sm + RT * RT;          // its transpose
  double * inv = sm + 2 * RT * RT;      // 1 / diagonal
  if (*info != 0) return;
  for (int x = threadIdx.x; x < RT * RT; x += blockDim.x) {
    const int i = x / RT, j = x % RT;
    double v;
    if (i < R && j < R) v = (j <= i) ? L[j + i * R] : 0.0;
    else v = (i == j) ? 1.0 : 0.0;
    Ls[i * RT + j] = v;
    Lt[j * RT + i] = v;
  }
  __syncthreads();
  for (int x = threadIdx.x; x < RT; x += blockDim.x) inv[x] = 1.0 / Ls[x * RT + x];
  __syncthreads();
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= I) return;
  double x[RT];
  const T * row = M1 + i * ld;
  if constexpr (sizeof(T) == 8) {
#pragma unroll
    for (int r = 0; r < RT; r += 2) {
      if (r + 1 < R) { const double2 v = *reinterpret_cast<const double2 *>(row + r); x[r] = v.x; x[r + 1] = v.y; }
      else { x[r] = (r < R) ? row[r] : 0.0; x[r + 1] = 0.0; }
    }
  } else {
    // (this shape keeps RT = 64 at 72 B of spill, under the fp64 instance's 88 B)
#pragma unroll
    for (int r = 0; r < RT; r += 4) {
      if (r < R) {
        const float4 v = *reinterpret_cast<const float4 *>(row + r);
        x[r]     = v.x;
        x[r + 1] = (r + 1 < R) ? (double)v.y : 0.0;
        x[r + 2] = (r + 2 < R) ? (double)v.z : 0.0;
        x[r + 3] = (r + 3 < R) ? (double)v.w : 0.0;
      } else {
        x[r] = x[r + 1] = x[r + 2] = x[r + 3] = 0.0;
      }
    }
  }
  // L y = x (forward), four independent partial sums per entry
#pragma unroll
  for (int p = 0; p < RT; ++p) {
    double s0 = x[p], s1 = 0.0, s2 = 0.0, s3 = 0.0;
#pragma unroll
    for (int k = 0; k + 1 < p; k += 2) {
      const double2 l = *reinterpret_cast<const double2 *>(&Ls[p * RT + k]);
      if ((k & 2) == 0) { s0 = fma(-l.x, x[k], s0); s1 = fma(-l.y, x[k + 1], s1); }
      else              { s2 = fma(-l.x, x[k], s2); s3 = fma(-l.y, x[k + 1], s3); }
    }
    if (p & 1) s0 = fma(-Ls[p * RT + p - 1], x[p - 1], s0);
    x[p] = ((s0 + s1) + (s2 + s3)) * inv[p];
  }
  // L^T z = y (backward)
#pragma unroll
  for (int p = RT - 1; p >= 0; --p) {
    double s0 = x[p], s1 = 0.0, s2 = 0.0, s3 = 0.0;
    constexpr int dummy = 0; (void)dummy;
    const int k0 = p + 1 + ((p + 1) & 1);          // first even index above p
    if ((p + 1) & 1) { if (p + 1 < RT) s0 = fma(-Lt[p * RT + p + 1], x[p + 1], s0); }
#pragma unroll
    for (int k = 0; k < RT; k += 2) {
      if (k >= k0) {
        const double2 l = *reinterpret_cast<const double2 *>(&Lt[p * RT + k]);
        if ((k & 2) == 0) { s0 = fma(-l.x, x[k], s0); s1 = fma(-l.y, x[k + 1], s1); }
        else              { s2 = fma(-l.x, x[k], s2); s3 = fma(-l.y, x[k + 1], s3); }
      }
    }
    x[p] = ((s0 + s1) + (s2 + s3)) * inv[p];
  }
  T * out = X + i * ld;
  if constexpr (sizeof(T) == 8) {
#pragma unroll
    for (int r = 0; r < RT; r += 2) {
      if (r + 1 < R) *reinterpret_cast<double2 *>(out + r) = make_double2(x[r], x[r + 1]);
      else if (r < R) out[r] = x[r];
    }
  } else {
#pragma unroll
    for (int r = 0; r < RT; r += 4) {
      if (r + 3 < R) {
        *reinterpret_cast<float4 *>(out + r) = make_float4((float)x[r], (float)x[r + 1],
                                                           (float)x[r + 2], (float)x[r + 3]);
      } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) if (r + c < R) out[r + c] = (float)x[r + c];
      }
    }
  }
}

// G(upper, row-major R x R) += A^T A as a register-tiled SYRK: persistent CTAs stream
// 64-row tiles of A through shared memory; two teams of threads (even / odd tile rows) each
// hold the 4x4 blocks of the upper triangle of G in registers (one block per thread) and
// flush them with one round of atomics per CTA.  reference: mat_aTa src/matrix.c:414-455
template <int RT>
constexpr int kSyrkThreads = 2 * ((RT / 4) * (RT / 4 + 1) / 2 + 31) / 32 * 32;   // two teams
template <int RT, class T>
__global__ void __launch_bounds__(kSyrkThreads<RT>)
k_gram_syrk(const T * __restrict__ A, unsigned long long I, int R, int lda,
            double * __restrict__ G) {
  constexpr int NB     = RT / 4;                       // 4x4 blocks per side
  constexpr int NBLK   = NB * (NB + 1) / 2;            // blocks of the upper triangle
  constexpr int TEAM   = (NBLK + 31) / 32 * 32;        // threads per team (whole warps)
  constexpr int TR     = 64;                           // rows per tile
  extern __shared__ __align__(16) double tile[];       // TR x RT
  const int team = threadIdx.x / TEAM, t = threadIdx.x % TEAM;
  // block t -> (bp, bq >= bp)
  int bp = 0, rem = t;
  while (bp < NB && rem >= NB - bp) { rem -= NB - bp; ++bp; }
  const bool active = t < NBLK;
  const int p0 = 4 * bp, q0 = 4 * (bp + rem);
  double acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
  // zero the padding columns once
  for (int x = threadIdx.x; x < TR * RT; x += blockDim.x) tile[x] = 0.0;
  __syncthreads();
  for (unsigned long long r0 = (unsigned long long)blockIdx.x * TR; r0 < I;
       r0 += (unsigned long long)gridDim.x * TR) {
    const int rows = (int)min((unsigned long long)TR, I - r0);
    for (int x = threadIdx.x; x < TR * R; x += blockDim.x) {
      const int i = x / R, j = x % R;
      tile[i * RT + j] = (i < rows) ? static_cast<double>(A[(r0 + i) * lda + j]) : 0.0;
    }
    __syncthreads();
    if (active) {
#pragma unroll 4
      for (int i = team; i < TR; i += 2) {
        const double2 a01 = *reinterpret_cast<const double2 *>(&tile[i * RT + p0]);
        const double2 a23 = *reinterpret_cast<const double2 *>(&tile[i * RT + p0 + 2]);
        const double2 b01 = *reinterpret_cast<const double2 *>(&tile[i * RT + q0]);
        const double2 b23 = *reinterpret_cast<const double2 *>(&tile[i * RT + q0 + 2]);
        const double av[4] = {a01.x, a01.y, a23.x, a23.y};
        const double bv[4] = {b01.x, b01.y, b23.x, b23.y};
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int b = 0; b < 4; ++b) acc[a][b] = fma(av[a], bv[b], acc[a][b]);
      }
    }
    __syncthreads();
  }
  if (active) {
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int p = p0 + a, q = q0 + b;
        if (p < R && q < R && q >= p) atomicAdd(&G[q + p * R], acc[a][b]);
      }
  }
}

// Column sums of squares (two_norm) or column maxima of max(a, 0).
// reference: p_mat_2norm src/matrix.c:86-144, p_mat_maxnorm :147-199
// (fp32: held to the fp64 instance's 28 registers; left alone ptxas gives it 30)
template <class T>
__global__ void __maxnreg__(sizeof(T) == 4 ? 28 : 255) k_colnorm(const T * __restrict__ A, unsigned long long I, int R, int ld,
                          int two_norm, double * __restrict__ acc) {
  const int j = threadIdx.x % 32 + 32 * blockIdx.y;
  const int ty = threadIdx.x / 32, ny = blockDim.x / 32;
  double v = 0.0;
  if (j < R)
    for (unsigned long long i = (unsigned long long)blockIdx.x * ny + ty; i < I;
         i += (unsigned long long)gridDim.x * ny) {
      const double a = static_cast<double>(A[i * ld + j]);
      v = two_norm ? fma(a, a, v) : fmax(v, a);
    }
  __shared__ double red[8][33];
  red[ty][threadIdx.x % 32] = v;
  __syncthreads();
  if (ty == 0 && j < R) {
    for (int y = 1; y < ny; ++y) v = two_norm ? v + red[y][threadIdx.x] : fmax(v, red[y][threadIdx.x]);
    if (two_norm) atomicAdd(&acc[j], v);
    else atomicMax(reinterpret_cast<unsigned long long *>(&acc[j]), (unsigned long long)__double_as_longlong(v));
  }
}
__global__ void k_finish_lambda(double * __restrict__ acc, int R, int two_norm,
                                double * __restrict__ lambda) {
  const int j = threadIdx.x + blockIdx.x * blockDim.x;
  if (j < R) lambda[j] = two_norm ? sqrt(acc[j]) : fmax(acc[j], 1.0);
}
// a /= lambda in fp64, rounded to T once
template <class T>
__global__ void k_scale_cols(T * __restrict__ A, unsigned long long I, int R, int ld,
                             const double * __restrict__ lambda) {
  const unsigned long long x = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= I * R) return;
  const unsigned long long i = x / R;
  const int j = (int)(x % R);
  A[i * ld + j] = static_cast<T>(static_cast<double>(A[i * ld + j]) / lambda[j]);
}
// *out += the sum of v over the block (whole warps): warp shuffles, then one atomic per block
__device__ __forceinline__ void block_sum_add(double v, double * out) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __shared__ double red[32];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    v = threadIdx.x < blockDim.x / 32 ? red[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) atomicAdd(out, v);
  }
}
// inner += sum_i sum_r A[i,r] * M1[i,r] * lambda[r].  reference: p_tt_kruskal_inner src/cpd.c:171-218
template <class T>
__global__ void k_inner(const T * __restrict__ A, const T * __restrict__ M1,
                        unsigned long long I, int R, int ld, const double * __restrict__ lambda,
                        double * __restrict__ inner) {
  double v = 0.0;
  for (unsigned long long x = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; x < I * R;
       x += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long i = x / R;
    const int j = (int)(x % R);
    v = fma(static_cast<double>(A[i * ld + j]) * static_cast<double>(M1[i * ld + j]), lambda[j], v);
  }
  block_sum_add(v, inner);
}

// ||X||^2 as an fp64 sum of squares over one stream's record values: the device CPD entries
// have no CSF to call csf_frobsq on.  reference: csf_frobsq src/csf.c:817-851
__global__ void k_vals_sumsq(const SpRec * __restrict__ rec, unsigned long long n,
                             double * __restrict__ out) {
  double v = 0.0;
  for (unsigned long long x = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; x < n;
       x += (unsigned long long)gridDim.x * blockDim.x) {
    const double a = rec[x].v;
    v = fma(a, a, v);
  }
  block_sum_add(v, out);
}
// post-processing (src/cpd.c:391-411): lambda_total *= the column 2-norms just divided out
__global__ void k_fold_lambda(double * __restrict__ lambda_total, const double * __restrict__ norms,
                              int R) {
  const int j = threadIdx.x + blockIdx.x * blockDim.x;
  if (j < R) lambda_total[j] *= norms[j];
}

// ---- nonnegative CPD by HALS (Cichocki & Phan 2009; Gillis & Glineur 2012), the update step of
// splatt_b200_cpd_nonneg_device: per mode one Gauss-Seidel sweep over the columns of
// B = A_n diag(lambda),
//   B[:, r] <- max(eps, (M[:, r] - sum_{j != r} B[:, j] G[j, r]) / G[r, r]),
// G the Hadamard product of the other modes' Grams.  Rows are independent given M and G, so a
// thread sweeps one row on its own (no atomics); the division is a product with 1 / G[r, r].
constexpr double kHalsFloor = 1e-16;   // include/splatt_b200.h: keeps every column nonzero

// G = the Hadamard product of the Grams of every mode but `mode`, full R x R (one CTA)
__global__ void k_hals_form(const double * __restrict__ ata, int nmodes, int mode, int R,
                            double * __restrict__ G) {
  for (int x = threadIdx.x; x < R * R; x += blockDim.x) {
    const int i = x / R, j = x % R;
    const int p = min(i, j), q = max(i, j);  // Grams are stored upper (row-major)
    double v = 1.0;
    for (int m = 0; m < nmodes; ++m)
      if (m != mode) v *= ata[(size_t)m * R * R + q + p * R];
    G[x] = v;
  }
}

// One HALS sweep per row for R <= RT (16 / 32 / 64), in place on X = A_n: one thread per row,
// the row of B in registers (A_n[i, :] lambda in fp64), G padded to RT with zeros (1 on the pad
// diagonal) in shared memory, read as 128-bit broadcasts; the row of M1 is loaded as the sweep
// reaches it.  Columns [0, R) are stored once, rounded to T.  As in k_solve_rows_reg, fp32 rows
// move as float4 and columns [R, RT) enter as 0 by selection: pad columns are loaded but never
// feed a result or get written.
template <int RT, class T>
__global__ void __launch_bounds__(128)
k_hals_rows_reg(const T * __restrict__ M1, T * __restrict__ X, unsigned long long I, int R, int ld,
                const double * __restrict__ G, const double * __restrict__ lambda) {
  extern __shared__ __align__(16) double sm[];
  double * Gs  = sm;                    // RT*RT
  double * inv = sm + RT * RT;          // 1 / G[r, r]
  double * lam = sm + RT * RT + RT;     // lambda, 0 on the pad
  for (int x = threadIdx.x; x < RT * RT; x += blockDim.x) {
    const int i = x / RT, j = x % RT;
    Gs[x] = (i < R && j < R) ? G[j + i * R] : (i == j ? 1.0 : 0.0);
  }
  for (int x = threadIdx.x; x < RT; x += blockDim.x) {
    inv[x] = x < R ? 1.0 / G[x + x * R] : 1.0;
    lam[x] = x < R ? lambda[x] : 0.0;
  }
  __syncthreads();
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= I) return;
  double b[RT];
  T * row = X + i * ld;
  const T * m = M1 + i * ld;
  if constexpr (sizeof(T) == 8) {
#pragma unroll
    for (int r = 0; r < RT; r += 2) {
      if (r + 1 < R) {
        const double2 v = *reinterpret_cast<const double2 *>(row + r);
        b[r] = v.x * lam[r]; b[r + 1] = v.y * lam[r + 1];
      } else {
        b[r] = (r < R) ? row[r] * lam[r] : 0.0; b[r + 1] = 0.0;
      }
    }
  } else {
#pragma unroll
    for (int r = 0; r < RT; r += 4) {
      if (r < R) {
        const float4 v = *reinterpret_cast<const float4 *>(row + r);
        b[r]     = (double)v.x * lam[r];
        b[r + 1] = (r + 1 < R) ? (double)v.y * lam[r + 1] : 0.0;
        b[r + 2] = (r + 2 < R) ? (double)v.z * lam[r + 2] : 0.0;
        b[r + 3] = (r + 3 < R) ? (double)v.w * lam[r + 3] : 0.0;
      } else {
        b[r] = b[r + 1] = b[r + 2] = b[r + 3] = 0.0;
      }
    }
  }
  double2 m2 = make_double2(0.0, 0.0);
  float4  m4 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int r = 0; r < RT; ++r) {
    if (r < R) {
      double mr;
      if constexpr (sizeof(T) == 8) {
        if ((r & 1) == 0) {
          if (r + 1 < R) m2 = *reinterpret_cast<const double2 *>(m + r);
          else m2.x = m[r];
        }
        mr = (r & 1) ? m2.y : m2.x;
      } else {
        if ((r & 3) == 0) m4 = *reinterpret_cast<const float4 *>(m + r);
        mr = (r & 3) == 0 ? m4.x : (r & 3) == 1 ? m4.y : (r & 3) == 2 ? m4.z : m4.w;
      }
      // mr - sum_{j != r} B[j] G[r, j], four independent partial sums
      double s0 = mr, s1 = 0.0, s2 = 0.0, s3 = 0.0;
#pragma unroll
      for (int k = 0; k < RT; k += 2) {
        const double2 g = *reinterpret_cast<const double2 *>(&Gs[r * RT + k]);
        if (k != r)     { if ((k & 2) == 0) s0 = fma(-g.x, b[k], s0); else s2 = fma(-g.x, b[k], s2); }
        if (k + 1 != r) { if ((k & 2) == 0) s1 = fma(-g.y, b[k + 1], s1); else s3 = fma(-g.y, b[k + 1], s3); }
      }
      b[r] = fmax(kHalsFloor, ((s0 + s1) + (s2 + s3)) * inv[r]);
    }
  }
  if constexpr (sizeof(T) == 8) {
#pragma unroll
    for (int r = 0; r < RT; r += 2) {
      if (r + 1 < R) *reinterpret_cast<double2 *>(row + r) = make_double2(b[r], b[r + 1]);
      else if (r < R) row[r] = b[r];
    }
  } else {
#pragma unroll
    for (int r = 0; r < RT; r += 4) {
      if (r + 3 < R) {
        *reinterpret_cast<float4 *>(row + r) = make_float4((float)b[r], (float)b[r + 1],
                                                           (float)b[r + 2], (float)b[r + 3]);
      } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) if (r + c < R) row[r + c] = (float)b[r + c];
      }
    }
  }
}

// The same sweep for any R (64 < R <= 128, or SPLATT_B200_TAIL_GENERIC=1): G in shared memory,
// the rows of B in shared memory laid out [r][thread] (as in k_solve_rows), in place on X = A_n.
template <class T>
__global__ void k_hals_rows(const T * __restrict__ M1, T * __restrict__ X, unsigned long long I,
                            int R, int ld, const double * __restrict__ G,
                            const double * __restrict__ lambda) {
  extern __shared__ double sm[];
  double * Gs = sm;                         // R*R
  double * bs = sm + R * R;                 // R * blockDim.x
  for (int x = threadIdx.x; x < R * R; x += blockDim.x) Gs[x] = G[x];
  __syncthreads();
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= I) return;
  const int NT = blockDim.x, t = threadIdx.x;
  T * row = X + i * ld;
  const T * m = M1 + i * ld;
  for (int r = 0; r < R; ++r) bs[r * NT + t] = static_cast<double>(row[r]) * lambda[r];
  for (int r = 0; r < R; ++r) {
    double s = static_cast<double>(m[r]);
    for (int j = 0; j < r; ++j) s = fma(-Gs[j + r * R], bs[j * NT + t], s);
    for (int j = r + 1; j < R; ++j) s = fma(-Gs[j + r * R], bs[j * NT + t], s);
    s = fmax(kHalsFloor, s * (1.0 / Gs[r + r * R]));
    bs[r * NT + t] = s;
    row[r] = static_cast<T>(s);
  }
}

// *bad = 1 if an entry (i, c), c < R, of A is negative or not finite
template <class T>
__global__ void k_nonneg_check(const T * __restrict__ A, unsigned long long I, int R, int ld,
                               int * __restrict__ bad) {
  bool b = false;
  for (unsigned long long x = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; x < I * R;
       x += (unsigned long long)gridDim.x * blockDim.x) {
    const double a = static_cast<double>(A[(x / R) * ld + x % R]);
    b |= !(a >= 0.0 && a <= 1.7976931348623157e308);
  }
  if (__any_sync(0xffffffffu, b) && (threadIdx.x & 31) == 0) atomicExch(bad, 1);
}

// ---- pieces of the ROW-PARTITIONED tail (multi-GPU engine, multi.cu): every device works on
// its own row slice and publishes partial column norms / partial Grams into per-device slots
// of the group's multicast region; all devices then combine the slots in device order, so
// they all end up with bit-identical lambda, Grams and factors.

// publish n doubles to a (multicast) address; zero the source for its next accumulation
__global__ void k_publish_zero(double * __restrict__ src, double * __restrict__ dst, int n) {
  for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < n; x += gridDim.x * blockDim.x) {
    dst[x] = src[x];
    src[x] = 0.0;
  }
}
// lambda from k per-device partial vectors (sum of squares -> sqrt, or max -> max(., 1))
__global__ void k_lambda_from_partials(const double * __restrict__ parts, int k, int stride, int R,
                                       int two_norm, double * __restrict__ lambda) {
  const int j = threadIdx.x + blockIdx.x * blockDim.x;
  if (j >= R) return;
  double v = 0.0;
  for (int d = 0; d < k; ++d) v = two_norm ? v + parts[(size_t)d * stride + j] : fmax(v, parts[(size_t)d * stride + j]);
  lambda[j] = two_norm ? sqrt(v) : fmax(v, 1.0);
}
// rows /= lambda, written to the local replica and (multicast) to every replica
__global__ void k_scale_rows_mc(double * __restrict__ x_local, double * __restrict__ x_mc,
                                unsigned long long I, int R, int ld, const double * __restrict__ lambda) {
  const unsigned long long x = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= I * R) return;
  const unsigned long long i = x / R;
  const int j = (int)(x % R);
  const double v = x_local[i * ld + j] / lambda[j];
  x_local[i * ld + j] = v;
  x_mc[i * ld + j] = v;
}
// dst = sum over devices of the published partials, in device order
__global__ void k_sum_partials(const double * __restrict__ parts, int k, int stride, int n,
                               double * __restrict__ dst) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= n) return;
  double v = 0.0;
  for (int d = 0; d < k; ++d) v += parts[(size_t)d * stride + x];
  dst[x] = v;
}

// f(std::integral_constant<int, RT>()) for the register tile rt = 16, 32 or 64
template <class F>
void with_rt(int rt, F && f) {
  if (rt == 16) f(std::integral_constant<int, 16>());
  else if (rt == 32) f(std::integral_constant<int, 32>());
  else f(std::integral_constant<int, 64>());
}

// The update of a mode's factor from its MTTKRP: the ALS row solve, or the HALS sweep of the
// nonnegative CPD.
enum class Update { als, hals };

struct DevTail {
  int N = 0, R = 0, ld = 0;
  double * ata = nullptr;     // N x R x R
  double * chol = nullptr;    // R x R
  double * hals_g = nullptr;  // R x R: G of the HALS sweep
  double * pinv = nullptr;    // R x R
  double * lam_acc = nullptr; // R
  double * lambda = nullptr;  // R
  double * inner = nullptr;   // 1
  int *    info = nullptr;
  double * jac_v = nullptr;   // R x R scratch of the pseudo-inverse fallback
  double * gpart = nullptr;   // R x R partial Gram of a row slice (zero between uses)
  double * h_back = nullptr;  // pinned: N*R*R + R + 1 (+1 info)
  cudaStream_t s = nullptr;
  int      solve_threads = 128;   // rows per block of k_solve_rows (shared memory permitting)
  int      rt = 0;                // R padded to 16 / 32 / 64: register-tiled solve + SYRK (0 = generic)
  bool     failed = false;        // a launch was rejected: results are not to be trusted

  // shared-memory opt-in of the instances that serve storage type T
  template <class T>
  bool set_smem_attrs() {
    bool ok = cudaFuncSetAttribute(k_solve_rows<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (R * R + R * solve_threads) * 8) == cudaSuccess &&
              cudaFuncSetAttribute(k_hals_rows<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (R * R + R * solve_threads) * 8) == cudaSuccess &&
              cudaFuncSetAttribute(k_gram<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 32 * R * 8) == cudaSuccess;
    if (ok && rt) {
      const int sb = (2 * rt * rt + rt) * 8, gb = 64 * rt * 8;
      cudaError_t e1 = cudaSuccess, e2 = cudaSuccess;
      with_rt(rt, [&](auto c) {
        constexpr int RT = decltype(c)::value;
        e1 = cudaFuncSetAttribute(k_solve_rows_reg<RT, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, sb);
        e2 = cudaFuncSetAttribute(k_gram_syrk<RT, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, gb);
      });
      if (e1 != cudaSuccess || e2 != cudaSuccess) { cudaGetLastError(); rt = 0; }
    }
    return ok;
  }
  bool alloc(int N_, int R_, int ld_, cudaStream_t st) {
    N = N_; R = R_; ld = ld_; s = st;
    bool ok = cudaMalloc(&ata, sizeof(double) * N * R * R) == cudaSuccess &&
              cudaMalloc(&chol, sizeof(double) * R * R) == cudaSuccess &&
              cudaMalloc(&hals_g, sizeof(double) * R * R) == cudaSuccess &&
              cudaMalloc(&pinv, sizeof(double) * R * R) == cudaSuccess &&
              cudaMalloc(&lam_acc, sizeof(double) * R) == cudaSuccess &&
              cudaMalloc(&lambda, sizeof(double) * R) == cudaSuccess &&
              cudaMalloc(&inner, sizeof(double)) == cudaSuccess &&
              cudaMalloc(&info, sizeof(int) * 2) == cudaSuccess &&
              cudaMalloc(&jac_v, sizeof(double) * R * R) == cudaSuccess &&
              cudaMalloc(&gpart, sizeof(double) * R * R) == cudaSuccess &&
              cudaMemset(gpart, 0, sizeof(double) * R * R) == cudaSuccess &&
              cudaMemset(lam_acc, 0, sizeof(double) * R) == cudaSuccess &&
              cudaMallocHost(&h_back, sizeof(double) * ((size_t)N * R * R + R + 2)) == cudaSuccess;
    if (ok) {
      // shared-memory budgets: k_form_chol R*R doubles (128 KB at R = 128); k_solve_rows
      // R*R + R*threads doubles -- shrink its row tile until it fits the opt-in limit
      int dev = 0, lim = 0;
      cudaGetDevice(&dev);
      cudaDeviceGetAttribute(&lim, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
      solve_threads = 128;
      while (solve_threads > 32 && (size_t)(R * R + R * solve_threads) * 8 > (size_t)lim) solve_threads /= 2;
      const char * ge = getenv("SPLATT_B200_TAIL_GENERIC");
      rt = (ge && atoi(ge) != 0) ? 0 : (R <= 16 ? 16 : (R <= 32 ? 32 : (R <= 64 ? 64 : 0)));
      ok = (size_t)(R * R + R * solve_threads) * 8 <= (size_t)lim && (size_t)R * R * 8 <= (size_t)lim &&
           cudaFuncSetAttribute(k_form_chol, cudaFuncAttributeMaxDynamicSharedMemorySize, R * R * 8) == cudaSuccess &&
           set_smem_attrs<double>() && set_smem_attrs<float>();
      if (!ok) fprintf(stderr, "SPLATT: rank %d does not fit the device ALS tail (shared memory)\n", R);
    }
    return ok;
  }
  void check(const char * what) {
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
      fprintf(stderr, "SPLATT: ALS tail launch '%s' failed: %s\n", what, cudaGetErrorString(e));
      failed = true;
    }
  }
  void release() {
    cudaFree(ata); cudaFree(chol); cudaFree(hals_g); cudaFree(pinv); cudaFree(lam_acc); cudaFree(lambda);
    cudaFree(inner); cudaFree(info); cudaFree(jac_v); cudaFree(gpart);
    if (h_back) cudaFreeHost(h_back);
  }
  template <class T>
  void gram(const T * A, uint64_t I, int m) {
    double * G = ata + (size_t)m * R * R;
    cudaMemsetAsync(G, 0, sizeof(double) * R * R, s);
    gram_into(A, I, G);
  }
  // G += A^T A (G is NOT zeroed here)
  template <class T>
  void gram_into(const T * A, uint64_t I, double * G) {
    if (I == 0) return;
    // the persistent SYRK pays one round of atomics per CTA: worth it from ~32 K rows on
    // (measured: 10 K x 32: 22.6 us vs 13.3 us generic; 1 M x 64: 0.74 ms vs 1.2 ms)
    if (rt && I >= 32768) {
      const unsigned blocks = (unsigned)std::min<uint64_t>((I + 63) / 64, 296);
      const size_t sm = (size_t)64 * rt * 8;
      with_rt(rt, [&](auto c) {
        constexpr int RT = decltype(c)::value;
        k_gram_syrk<RT, T><<<blocks, kSyrkThreads<RT>, sm, s>>>(A, I, R, ld, G);
      });
    } else {
      const unsigned blocks = (unsigned)std::min<uint64_t>((I + 31) / 32, 592);
      k_gram<T><<<blocks, 256, 32 * R * 8, s>>>(A, I, R, ld, G);
    }
    check("k_gram");
    spb200_count_launches(1);
  }
  // one mode step after the MTTKRP: d_out (M1) -> d_mat (new factor), lambda, Gram
  template <class T>
  void mode_step(const T * d_out, T * d_mat, uint64_t I, int m, bool two_norm,
                 Update u = Update::als) {
    if (u == Update::hals) hals(d_out, d_mat, I, m);
    else solve(d_out, d_mat, I, m);
    cudaMemsetAsync(lam_acc, 0, sizeof(double) * R, s);
    dim3 g((unsigned)std::min<uint64_t>((I + 7) / 8, 1184), (R + 31) / 32);
    k_colnorm<T><<<g, 256, 0, s>>>(d_mat, I, R, ld, two_norm ? 1 : 0, lam_acc);
    k_finish_lambda<<<(R + 127) / 128, 128, 0, s>>>(lam_acc, R, two_norm ? 1 : 0, lambda);
    k_scale_cols<T><<<(unsigned)((I * R + 255) / 256), 256, 0, s>>>(d_mat, I, R, ld, lambda);
    check("normalise");
    spb200_count_launches(3);
    gram(d_mat, I, m);
  }
  // normal matrix of mode m + Cholesky, then the row solves of `I` rows
  template <class T>
  void solve(const T * d_out, T * d_mat, uint64_t I, int m) {
    k_form_chol<<<1, 256, R * R * 8, s>>>(ata, N, m, R, chol, pinv, jac_v, info);
    check("k_form_chol");
    spb200_count_launches(1);
    if (I == 0) return;
    const int NT = solve_threads;
    if (rt) {
      // register-tiled solve when the Cholesky succeeded (it returns at once otherwise) ...
      const size_t sm = (size_t)(2 * rt * rt + rt) * 8;
      const unsigned nb = (unsigned)((I + 127) / 128);
      with_rt(rt, [&](auto c) {
        k_solve_rows_reg<decltype(c)::value, T><<<nb, 128, sm, s>>>(d_out, d_mat, I, R, ld, chol, info);
      });
      // ... and the generic kernel only for the pseudo-inverse fallback (info != 0)
      k_solve_rows<T><<<(unsigned)((I + NT - 1) / NT), NT, (R * R + R * NT) * 8, s>>>(
          d_out, d_mat, I, R, ld, chol, pinv, info, 1);
      spb200_count_launches(1);
    } else {
      k_solve_rows<T><<<(unsigned)((I + NT - 1) / NT), NT, (R * R + R * NT) * 8, s>>>(
          d_out, d_mat, I, R, ld, chol, pinv, info, 0);
    }
    check("k_solve_rows");
    spb200_count_launches(1);
  }
  // G of mode m, then the HALS sweep of `I` rows: d_mat (A_m) <- B, lambda read as it stands
  template <class T>
  void hals(const T * d_out, T * d_mat, uint64_t I, int m) {
    k_hals_form<<<1, 256, 0, s>>>(ata, N, m, R, hals_g);
    check("k_hals_form");
    spb200_count_launches(1);
    if (I == 0) return;
    if (rt) {
      const size_t sm = (size_t)(rt * rt + 2 * rt) * 8;
      const unsigned nb = (unsigned)((I + 127) / 128);
      with_rt(rt, [&](auto c) {
        k_hals_rows_reg<decltype(c)::value, T><<<nb, 128, sm, s>>>(d_out, d_mat, I, R, ld, hals_g, lambda);
      });
    } else {
      const int NT = solve_threads;
      k_hals_rows<T><<<(unsigned)((I + NT - 1) / NT), NT, (R * R + R * NT) * 8, s>>>(
          d_out, d_mat, I, R, ld, hals_g, lambda);
    }
    check("k_hals_rows");
    spb200_count_launches(1);
  }

  // Start of the nonnegative CPD: checks every entry of columns [0, R) of the start (finite,
  // >= 0) and its column sums of squares (positive, finite; summed into ata, before the Grams are
  // formed), synchronising the stream once.  When they hold, 2-normalises every factor with
  // lambda = the product of the column norms; otherwise writes nothing and returns false (as it
  // does when a launch failed: then `failed` is set).
  template <class T>
  bool nonneg_start(T * const * d_mats, const uint64_t * dims) {
    cudaMemsetAsync(info, 0, sizeof(int), s);
    cudaMemsetAsync(ata, 0, sizeof(double) * N * R, s);
    for (int m = 0; m < N; ++m) {
      const uint64_t I = dims[m];
      if (!I) continue;
      k_nonneg_check<T><<<(unsigned)std::min<uint64_t>((I * R + 255) / 256, 1184), 256, 0, s>>>(
          d_mats[m], I, R, ld, info);
      dim3 g((unsigned)std::min<uint64_t>((I + 7) / 8, 1184), (R + 31) / 32);
      k_colnorm<T><<<g, 256, 0, s>>>(d_mats[m], I, R, ld, 1, ata + (size_t)m * R);
      spb200_count_launches(2);
    }
    check("start check");
    std::vector<double> sums((size_t)N * R);
    int bad = 1;
    if (cudaMemcpyAsync(sums.data(), ata, sizeof(double) * N * R, cudaMemcpyDeviceToHost, s) != cudaSuccess ||
        cudaMemcpyAsync(&bad, info, sizeof(int), cudaMemcpyDeviceToHost, s) != cudaSuccess ||
        cudaStreamSynchronize(s) != cudaSuccess)
      failed = true;
    if (failed) return false;
    for (double x : sums) bad |= !(x > 0.0 && x <= 1.7976931348623157e308);
    if (bad) return false;
    const std::vector<double> ones(R, 1.0);
    if (cudaMemcpyAsync(lambda, ones.data(), sizeof(double) * R, cudaMemcpyHostToDevice, s) != cudaSuccess) {
      failed = true;
      return false;
    }
    for (int m = 0; m < N; ++m) {
      const uint64_t I = dims[m];
      k_finish_lambda<<<(R + 127) / 128, 128, 0, s>>>(ata + (size_t)m * R, R, 1, lam_acc);
      k_scale_cols<T><<<(unsigned)((I * R + 255) / 256), 256, 0, s>>>(d_mats[m], I, R, ld, lam_acc);
      k_fold_lambda<<<(R + 127) / 128, 128, 0, s>>>(lambda, lam_acc, R);
      spb200_count_launches(3);
    }
    check("start normalisation");
    return !failed;
  }

  // post-processing on the device (src/cpd.c:391-411): 2-normalise every factor, folding the
  // norms into lambda_total (R doubles, device; holds the ALS lambda on entry)
  template <class T>
  void postprocess(T * const * d_mats, const uint64_t * dims, double * lambda_total) {
    for (int m = 0; m < N; ++m) {
      const uint64_t I = dims[m];
      cudaMemsetAsync(lam_acc, 0, sizeof(double) * R, s);
      if (I) {
        dim3 g((unsigned)std::min<uint64_t>((I + 7) / 8, 1184), (R + 31) / 32);
        k_colnorm<T><<<g, 256, 0, s>>>(d_mats[m], I, R, ld, 1, lam_acc);
      }
      k_finish_lambda<<<(R + 127) / 128, 128, 0, s>>>(lam_acc, R, 1, lambda);
      if (I) k_scale_cols<T><<<(unsigned)((I * R + 255) / 256), 256, 0, s>>>(d_mats[m], I, R, ld, lambda);
      k_fold_lambda<<<(R + 127) / 128, 128, 0, s>>>(lambda_total, lambda, R);
      check("post-process");
      spb200_count_launches(I ? 4 : 2);
    }
  }

  // Fit after the last mode's update from its factor and M1 (reference: p_calc_fit
  // src/cpd.c:237-265): inner product on the device, one read-back of the Grams, lambda and
  // the inner product (and the solver info when info_out is set), synchronising the stream.
  // lambda_out (R host doubles) and info_out may be null.  Check `failed` afterwards: when it
  // is set (by this synchronisation or an earlier launch) nothing has been written.
  template <class T>
  double fit(const T * last, const T * m1, uint64_t rows, double ttnormsq, double * lambda_out,
             int * info_out) {
    const size_t nb = (size_t)N * R * R;
    cudaMemsetAsync(inner, 0, sizeof(double), s);
    k_inner<T><<<296, 256, 0, s>>>(last, m1, rows, R, ld, lambda, inner);
    spb200_count_launches(1);
    cudaMemcpyAsync(h_back, ata, nb * 8, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(h_back + nb, lambda, R * 8, cudaMemcpyDeviceToHost, s);
    cudaMemcpyAsync(h_back + nb + R, inner, 8, cudaMemcpyDeviceToHost, s);
    if (info_out) cudaMemcpyAsync(h_back + nb + R + 1, info, 4, cudaMemcpyDeviceToHost, s);
    if (cudaStreamSynchronize(s) != cudaSuccess) failed = true;
    if (failed) return 0.0;
    if (lambda_out) memcpy(lambda_out, h_back + nb, sizeof(double) * R);
    if (info_out) memcpy(info_out, h_back + nb + R + 1, sizeof(int));
    return cpd_fit(h_back, h_back + nb, N, R, ttnormsq, h_back[nb + R]);
  }

  // ---- row-partitioned tail (see the kernels above)
  void solve_norm_partial(const double * m1, double * x, uint64_t rows, int m, bool two_norm,
                          double * mc_norm_slot) {
    solve(m1, x, rows, m);
    if (rows) {
      dim3 g((unsigned)std::min<uint64_t>((rows + 7) / 8, 1184), (R + 31) / 32);
      k_colnorm<double><<<g, 256, 0, s>>>(x, rows, R, ld, two_norm ? 1 : 0, lam_acc);
    }
    k_publish_zero<<<1, 128, 0, s>>>(lam_acc, mc_norm_slot, R);
    check("norm partial");
    spb200_count_launches(2);
  }
  void scale_gram_partial(double * x, double * x_mc, uint64_t rows, bool two_norm,
                          const double * norms_all, int k, int norm_stride, double * mc_gram_slot) {
    k_lambda_from_partials<<<(R + 127) / 128, 128, 0, s>>>(norms_all, k, norm_stride, R,
                                                           two_norm ? 1 : 0, lambda);
    if (rows)
      k_scale_rows_mc<<<(unsigned)((rows * R + 255) / 256), 256, 0, s>>>(x, x_mc, rows, R, ld, lambda);
    gram_partial(x, rows, mc_gram_slot);
    check("scale + gram partial");
    spb200_count_launches(2);
  }
  void gram_partial(const double * x, uint64_t rows, double * mc_gram_slot) {
    gram_into(x, rows, gpart);
    k_publish_zero<<<(R * R + 255) / 256, 256, 0, s>>>(gpart, mc_gram_slot, R * R);
    check("gram partial");
    spb200_count_launches(1);
  }
  void finish_gram(int m, const double * grams_all, int k, int gram_stride) {
    k_sum_partials<<<(R * R + 255) / 256, 256, 0, s>>>(grams_all, k, gram_stride, R * R,
                                                        ata + (size_t)m * R * R);
    check("gram sum");
    spb200_count_launches(1);
  }
};

int mttkrp_t(const splatt_b200_tensor * t, int m, int R, int ldm, double * const * d_mats,
             double * d_out, cudaStream_t s) {
  return splatt_b200_mttkrp(t, m, R, ldm, d_mats, d_out, s);
}
int mttkrp_t(const splatt_b200_tensor * t, int m, int R, int ldm, float * const * d_mats,
             float * d_out, cudaStream_t s) {
  return splatt_b200_mttkrp_f32(t, m, R, ldm, d_mats, d_out, s);
}

// CPD-ALS with the dense tail on the device (reference: cpd_als_iterate src/cpd.c:318-373):
// per mode MTTKRP -> tail.mode_step; per iteration one small read-back (Grams, lambda, inner
// product, solver info) for the fit -- the loop's only host synchronisation.  d_mats hold the
// start on entry (their Grams are formed here) and the factors of the last iteration on return,
// not post-processed.  d_out: M1 scratch of max(dims) x ldm.  lambda: R host doubles, the last
// iteration's.  upd: the update step (Update::hals 2-normalises in every iteration and has no
// solver info).  history: NULL or one fit per iteration run.  false when a launch failed.
template <class T>
bool run_device_als(const splatt_b200_tensor * t, T * const * d_mats, T * d_out, int ldm,
                    DevTail & tail, double ttnormsq, const double * options, double * lambda,
                    double * fit_out, uint64_t * iterations_out, Update upd = Update::als,
                    double * history = nullptr) {
  const int N = tail.N, R = tail.R;
  const uint64_t * dims = t->dims;
  AlsIterations iters(options);
  double fit = 0;
  uint64_t its = 0;
  bool ok = true;
  for (int m = 0; m < N; ++m) tail.gram(d_mats[m], dims[m], m);
  for (uint64_t it = 0; it < iters.niters && ok; ++it) {
    iters.start();
    for (int m = 0; m < N && ok; ++m) {
      if (mttkrp_t(t, m, R, ldm, d_mats, d_out, tail.s) != SPLATT_SUCCESS) { ok = false; break; }
      tail.mode_step(d_out, d_mats[m], dims[m], m, it == 0 || upd == Update::hals, upd);
    }
    if (!ok) break;
    int info_last = 0;
    fit = tail.fit(d_mats[N - 1], d_out, dims[N - 1], ttnormsq, lambda,
                   upd == Update::als ? &info_last : nullptr);
    if (tail.failed) { ok = false; break; }
    if (info_last)
      fprintf(stderr, "SPLATT: Gram matrix is not SPD. Used pseudo-inverse.\n");
    if (history) history[it] = fit;
    its = it + 1;
    if (iters.done(it, fit)) break;
  }
  *fit_out = fit;
  *iterations_out = its;
  return ok;
}

// splatt_b200_cpd_als_device / _f32 (Update::als) and splatt_b200_cpd_nonneg_device / _f32
// (Update::hals): CPD of a device tensor from device factors.
template <class T>
int cpd_device(const char * name, Update upd, const splatt_b200_tensor * t, int R, int ldm,
               const double * options, T * const * d_factors, double * lambda_out,
               double * fit_out, int * iterations_out, double * history, void * stream) {
  constexpr int align = sizeof(T) == 4 ? 4 : 2;     // row alignment of the MTTKRP
  bool bad = !t || !options || !d_factors || R < 1 || R > 128 || ldm % align != 0 ||
             ldm < (R + align - 1) / align * align;
  bad = bad || t->nmodes < 2 || t->nmodes > SPB200_MAXN || t->shard_count > 1 || t->streams.empty();
  for (int m = 0; !bad && m < t->nmodes; ++m)
    bad = !d_factors[m] || reinterpret_cast<uintptr_t>(d_factors[m]) % 16 != 0;
  if (bad) {
    fprintf(stderr, "SPLATT: %s: bad arguments\n", name);
    return SPLATT_ERROR_BADINPUT;
  }
  DeviceGuard g(t->device);
  if (!g.ok) return SPLATT_ERROR_BADINPUT;
  const int N = t->nmodes;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  uint64_t maxdim = 0;
  for (int m = 0; m < N; ++m) maxdim = std::max(maxdim, t->dims[m]);
  T * d_out = nullptr;
  double * d_lambda = nullptr;
  DevTail tail;
  bool alloc_ok = cudaMalloc(&d_out, std::max<uint64_t>(maxdim, 1) * (size_t)ldm * sizeof(T)) == cudaSuccess &&
                  cudaMalloc(&d_lambda, sizeof(double) * R) == cudaSuccess &&
                  tail.alloc(N, R, ldm, s);
  bool ok = alloc_ok;
  double ttnormsq = 0, fit = 0;
  uint64_t its = 0;
  std::vector<double> lambda(R);
  if (ok) {
    const FiberStream & fs = t->streams[0];
    cudaMemsetAsync(tail.inner, 0, sizeof(double), s);
    if (fs.nrec) {
      k_vals_sumsq<<<(unsigned)std::min<uint64_t>((fs.nrec + 255) / 256, 1184), 256, 0, s>>>(
          fs.rec, fs.nrec, tail.inner);
      tail.check("k_vals_sumsq");
      spb200_count_launches(1);
    }
    ok = cudaMemcpyAsync(tail.h_back, tail.inner, 8, cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaStreamSynchronize(s) == cudaSuccess && !tail.failed;
    ttnormsq = tail.h_back[0];
  }
  if (ok && upd == Update::hals && !tail.nonneg_start(d_factors, t->dims)) {
    if (!tail.failed)
      fprintf(stderr, "SPLATT: %s: a start entry is negative or not finite, or a start column is "
                      "zero\n", name);
    ok = false;
  }
  ok = ok && run_device_als<T>(t, d_factors, d_out, ldm, tail, ttnormsq, options, lambda.data(),
                               &fit, &its, upd, history);
  if (ok && upd == Update::als) {
    ok = cudaMemcpyAsync(d_lambda, lambda.data(), sizeof(double) * R, cudaMemcpyHostToDevice, s) == cudaSuccess;
    tail.postprocess(d_factors, t->dims, d_lambda);
    ok = ok && cudaMemcpyAsync(tail.h_back, d_lambda, sizeof(double) * R, cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaStreamSynchronize(s) == cudaSuccess && !tail.failed;
  } else if (ok) {
    // HALS leaves 2-normalised factors: lambda as the loop (or, after 0 iterations, the start) left it
    ok = cudaMemcpyAsync(tail.h_back, tail.lambda, sizeof(double) * R, cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaStreamSynchronize(s) == cudaSuccess && !tail.failed;
  }
  if (ok) {
    if (lambda_out) memcpy(lambda_out, tail.h_back, sizeof(double) * R);
    if (fit_out) *fit_out = fit;
    if (iterations_out) *iterations_out = (int)its;
  }
  cudaStreamSynchronize(s);
  cudaFree(d_out);
  cudaFree(d_lambda);
  tail.release();
  if (!ok) {
    fprintf(stderr, "SPLATT: %s failed (%s)\n", name, cudaGetErrorString(cudaGetLastError()));
    return alloc_ok ? SPLATT_ERROR_BADINPUT : SPLATT_ERROR_NOMEMORY;
  }
  return SPLATT_SUCCESS;
}

}  // namespace

extern "C" {

int splatt_cpd_als(splatt_csf const * const tensors, splatt_idx_t const nfactors,
                   double const * const options, splatt_kruskal * factored) {
  if (!tensors || !options || !factored || nfactors == 0) {
    fprintf(stderr, "SPLATT: splatt_cpd_als: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  const int N = (int)tensors[0].nmodes;
  const int R = (int)nfactors;
  const int ldm = R + (R & 1);
  const int verbosity = (int)options[SPLATT_OPTION_VERBOSITY];
  {
    // SPLATT_B200_NGPUS=k / SPLATT_B200_DEVICES=a,b,..: one process, k devices (multi.cu)
    int devs[16];
    const int nd = splatt_b200_multi_env_devices(devs, 16);
    if (nd > 1) {
      splatt_b200_multi * mh = nullptr;
      int mrc = splatt_b200_multi_create(tensors, (int)options[SPLATT_OPTION_CSF_ALLOC], R, devs, nd,
                                         verbosity, &mh);
      if (mrc != SPLATT_SUCCESS) return mrc;
      mrc = splatt_b200_multi_cpd_als(mh, tensors, options, factored);
      splatt_b200_multi_free(mh);
      return mrc;
    }
  }
  uint64_t dims[SPB200_MAXN], maxdim = 0;
  for (int m = 0; m < N; ++m) { dims[m] = tensors[0].dims[m]; maxdim = std::max(maxdim, dims[m]); }
  // Where the dense ALS tail runs.  Default: on the device (SURVEY 8(f) #1).
  // SPLATT_B200_HOST_SOLVE=1 keeps it on the host as the north star words it.
  const char * hs = getenv("SPLATT_B200_HOST_SOLVE");
  const bool host_tail = (hs && atoi(hs) != 0) || R > 128;

  // device mirror (once) -- reference: splatt_mttkrp_alloc_ws at src/cpd.c:304
  splatt_b200_build_opts bo;
  memset(&bo, 0, sizeof(bo));
  bo.device = -1;
  bo.verbosity = verbosity;
  const char * lay = getenv("SPLATT_B200_LAYOUT");
  bo.layout = (lay && !strcmp(lay, "asgiven")) ? SPLATT_B200_LAYOUT_ASGIVEN
                                               : SPLATT_B200_LAYOUT_ALLROOT;
  splatt_b200_tensor * T = nullptr;
  int rc = splatt_b200_tensor_from_csf(tensors, (int)options[SPLATT_OPTION_CSF_ALLOC], &bo, &T);
  if (rc != SPLATT_SUCCESS) return rc;

  // factor matrices: random init in the reference's draw order (src/cpd.c:36-40)
  HostKruskal K;
  double * d_mats[SPB200_MAXN] = {nullptr};
  double * d_out = nullptr;
  double * m1 = nullptr;          // pinned MTTKRP result (host tail only)
  cudaStream_t stream = nullptr;
  DevTail tail;
  bool ok = K.start(N, dims, R);
  double ** mats = K.mats;
  double * lambda = K.lambda;
  ok = ok && cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking) == cudaSuccess;
  for (int m = 0; m < N && ok; ++m) {
    ok = cudaMalloc(&d_mats[m], dims[m] * (size_t)ldm * 8) == cudaSuccess &&
         cudaMemsetAsync(d_mats[m], 0, dims[m] * (size_t)ldm * 8, stream) == cudaSuccess &&
         h2d_matrix(d_mats[m], ldm, mats[m], dims[m], R, stream) == cudaSuccess;
  }
  ok = ok && cudaMalloc(&d_out, maxdim * (size_t)ldm * 8) == cudaSuccess;
  if (host_tail) ok = ok && cudaMallocHost(&m1, maxdim * (size_t)R * 8) == cudaSuccess;
  else ok = ok && tail.alloc(N, R, ldm, stream);
  if (ok && !host_tail && verbosity > SPLATT_VERBOSITY_LOW)
    printf("SPLATT-B200: device ALS tail, %d rows per solve block\n", tail.solve_threads);

  double fit = 0;
  const double ttnormsq = spb200_csf_frobsq(tensors);

  if (ok && host_tail) {
    AlsIterations iters(options);
    std::vector<double> ata((size_t)N * R * R);
    for (int m = 0; m < N; ++m) gram(mats[m], dims[m], R, ata.data() + (size_t)m * R * R);
    std::vector<double> neq((size_t)R * R);
    for (uint64_t it = 0; it < iters.niters && ok; ++it) {
      iters.start();
      for (int m = 0; m < N && ok; ++m) {
        // M1 = X_(m) (khatri-rao of the other factors), on the GPU
        rc = splatt_b200_mttkrp(T, m, R, ldm, d_mats, d_out, stream);
        cudaError_t e = d2h_matrix(m1, d_out, ldm, dims[m], R, stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
        if (rc != SPLATT_SUCCESS || e != cudaSuccess) { ok = false; break; }
        // A_m = M1 * (hadamard Grams)^-1   (src/cpd.c:337-339, src/matrix.c:529-606)
        memcpy(mats[m], m1, dims[m] * (size_t)R * 8);
        form_normal_matrix(ata.data(), m, N, R, neq.data());
        std::vector<double> chol(neq);
        if (cholesky(chol.data(), R)) {
          cholesky_solve_rows(chol.data(), R, mats[m], dims[m]);
        } else {
          fprintf(stderr, "SPLATT: Gram matrix is not SPD. Trying pseudo-inverse.\n");
          pinv_solve_rows(neq.data(), R, mats[m], dims[m]);
        }
        normalize_cols(mats[m], dims[m], R, lambda, it == 0);   // src/cpd.c:343-347
        gram(mats[m], dims[m], R, ata.data() + (size_t)m * R * R);   // src/cpd.c:350
        // keep the device copy current
        ok = h2d_matrix(d_mats[m], ldm, mats[m], dims[m], R, stream) == cudaSuccess;
      }
      if (!ok) break;
      const double inner = kruskal_inner(mats[N - 1], m1, dims[N - 1], R, lambda);
      fit = cpd_fit(ata.data(), lambda, N, R, ttnormsq, inner);
      if (iters.done(it, fit)) break;
    }
  } else if (ok) {
    // ---- everything on the device; one small read-back per iteration for the fit
    uint64_t its = 0;
    ok = run_device_als<double>(T, d_mats, d_out, ldm, tail, ttnormsq, options, lambda, &fit, &its);
    for (int m = 0; m < N && ok; ++m)
      ok = d2h_matrix(mats[m], d_mats[m], ldm, dims[m], R, stream) == cudaSuccess;
    ok = ok && cudaStreamSynchronize(stream) == cudaSuccess;
  }
  if (stream) cudaStreamSynchronize(stream);
  for (int m = 0; m < N; ++m) if (d_mats[m]) cudaFree(d_mats[m]);
  if (d_out) cudaFree(d_out);
  if (m1) cudaFreeHost(m1);
  if (!host_tail) tail.release();
  if (stream) cudaStreamDestroy(stream);
  splatt_b200_tensor_free(T);
  if (!ok) {
    fprintf(stderr, "SPLATT: CPD-ALS failed (%s)\n", cudaGetErrorString(cudaGetLastError()));
    return SPLATT_ERROR_NOMEMORY;
  }
  K.finish(fit, factored);     // post-process (src/cpd.c:391-411)
  return SPLATT_SUCCESS;
}

// ---------------------------------------------------------------------------
// The device ALS tail as engine entry points, so that a multi-GPU driver can run
//   local MTTKRP on its shard -> exchange -> (replicated) tail
// with the same kernels splatt_cpd_als uses (splatt_b200/parallel.py:cpd_als_sharded).
// ---------------------------------------------------------------------------
struct splatt_b200_als_tail { DevTail t; };

}  // extern "C"

namespace {

template <class T>
int tail_gram(splatt_b200_als_tail * h, int mode, const T * d_factor, uint64_t rows) {
  if (!h || mode < 0 || mode >= h->t.N) return SPLATT_ERROR_BADINPUT;
  h->t.gram(d_factor, rows, mode);
  return (cudaGetLastError() == cudaSuccess && !h->t.failed) ? SPLATT_SUCCESS : SPLATT_ERROR_BADINPUT;
}

template <class T>
int tail_update(splatt_b200_als_tail * h, int mode, const T * d_m1, T * d_factor, uint64_t rows,
                int first_iteration) {
  if (!h || mode < 0 || mode >= h->t.N) return SPLATT_ERROR_BADINPUT;
  h->t.mode_step(d_m1, d_factor, rows, mode, first_iteration != 0);
  return (cudaGetLastError() == cudaSuccess && !h->t.failed) ? SPLATT_SUCCESS : SPLATT_ERROR_BADINPUT;
}

template <class T>
int tail_fit(splatt_b200_als_tail * h, const T * d_last_factor, const T * d_last_m1, uint64_t rows,
             double ttnormsq, double * fit_out, double * lambda_out) {
  if (!h || !fit_out) return SPLATT_ERROR_BADINPUT;
  const double fit = h->t.fit(d_last_factor, d_last_m1, rows, ttnormsq, lambda_out, nullptr);
  if (h->t.failed) return SPLATT_ERROR_BADINPUT;
  *fit_out = fit;
  return SPLATT_SUCCESS;
}

// the fp32 tail entries need 16-byte rows (ldm % 4 == 0) and 16-byte aligned matrices
bool f32_tail_ok(const splatt_b200_als_tail * h, const float * a, const float * b) {
  return h && h->t.ld % 4 == 0 && a && b && reinterpret_cast<uintptr_t>(a) % 16 == 0 &&
         reinterpret_cast<uintptr_t>(b) % 16 == 0;
}

}  // namespace

extern "C" {

int splatt_b200_als_tail_create(int nmodes, int ncolumns, int ldm, void * stream,
                                splatt_b200_als_tail ** out) {
  if (!out || nmodes < 2 || nmodes > SPB200_MAXN || ncolumns < 1 || ncolumns > 128 ||
      ldm < ncolumns) return SPLATT_ERROR_BADINPUT;
  splatt_b200_als_tail * h = new splatt_b200_als_tail();
  if (!h->t.alloc(nmodes, ncolumns, ldm, static_cast<cudaStream_t>(stream))) {
    h->t.release();
    delete h;
    return SPLATT_ERROR_NOMEMORY;
  }
  *out = h;
  return SPLATT_SUCCESS;
}

void splatt_b200_als_tail_free(splatt_b200_als_tail * h) {
  if (!h) return;
  h->t.release();
  delete h;
}

// Gram of one factor (call once per factor before the first iteration).
int splatt_b200_als_tail_gram(splatt_b200_als_tail * h, int mode, double const * d_factor,
                              uint64_t rows) {
  return tail_gram(h, mode, d_factor, rows);
}

// One mode update: d_m1 (the summed MTTKRP result) -> d_factor, lambda, Gram of the mode.
int splatt_b200_als_tail_update(splatt_b200_als_tail * h, int mode, double const * d_m1,
                                double * d_factor, uint64_t rows, int first_iteration) {
  return tail_update(h, mode, d_m1, d_factor, rows, first_iteration);
}

// Fit after the last mode's update (reference: p_calc_fit src/cpd.c:237-265).  Synchronises
// the stream; lambda_out (ncolumns doubles, host) may be NULL.
int splatt_b200_als_tail_fit(splatt_b200_als_tail * h, double const * d_last_factor,
                             double const * d_last_m1, uint64_t rows, double ttnormsq,
                             double * fit_out, double * lambda_out) {
  return tail_fit(h, d_last_factor, d_last_m1, rows, ttnormsq, fit_out, lambda_out);
}

int splatt_b200_als_tail_gram_f32(splatt_b200_als_tail * h, int mode, float const * d_factor,
                                  uint64_t rows) {
  if (!f32_tail_ok(h, d_factor, d_factor)) return SPLATT_ERROR_BADINPUT;
  return tail_gram(h, mode, d_factor, rows);
}

int splatt_b200_als_tail_update_f32(splatt_b200_als_tail * h, int mode, float const * d_m1,
                                    float * d_factor, uint64_t rows, int first_iteration) {
  if (!f32_tail_ok(h, d_m1, d_factor)) return SPLATT_ERROR_BADINPUT;
  return tail_update(h, mode, d_m1, d_factor, rows, first_iteration);
}

int splatt_b200_als_tail_fit_f32(splatt_b200_als_tail * h, float const * d_last_factor,
                                 float const * d_last_m1, uint64_t rows, double ttnormsq,
                                 double * fit_out, double * lambda_out) {
  if (!f32_tail_ok(h, d_last_factor, d_last_m1)) return SPLATT_ERROR_BADINPUT;
  return tail_fit(h, d_last_factor, d_last_m1, rows, ttnormsq, fit_out, lambda_out);
}

int splatt_b200_cpd_als_device(splatt_b200_tensor const * t, int ncolumns, int ldm,
                               double const * options, double * const * d_factors,
                               double * lambda_out, double * fit_out, int * iterations_out,
                               void * stream) {
  return cpd_device("splatt_b200_cpd_als_device", Update::als, t, ncolumns, ldm, options,
                    d_factors, lambda_out, fit_out, iterations_out, nullptr, stream);
}

int splatt_b200_cpd_als_device_f32(splatt_b200_tensor const * t, int ncolumns, int ldm,
                                   double const * options, float * const * d_factors,
                                   double * lambda_out, double * fit_out, int * iterations_out,
                                   void * stream) {
  return cpd_device("splatt_b200_cpd_als_device_f32", Update::als, t, ncolumns, ldm, options,
                    d_factors, lambda_out, fit_out, iterations_out, nullptr, stream);
}

int splatt_b200_cpd_nonneg_device(splatt_b200_tensor const * t, int ncolumns, int ldm,
                                  double const * options, double * const * d_factors,
                                  double * lambda_out, double * fit_out, int * iterations_out,
                                  double * history, void * stream) {
  return cpd_device("splatt_b200_cpd_nonneg_device", Update::hals, t, ncolumns, ldm, options,
                    d_factors, lambda_out, fit_out, iterations_out, history, stream);
}

int splatt_b200_cpd_nonneg_device_f32(splatt_b200_tensor const * t, int ncolumns, int ldm,
                                      double const * options, float * const * d_factors,
                                      double * lambda_out, double * fit_out, int * iterations_out,
                                      double * history, void * stream) {
  return cpd_device("splatt_b200_cpd_nonneg_device_f32", Update::hals, t, ncolumns, ldm, options,
                    d_factors, lambda_out, fit_out, iterations_out, history, stream);
}

}  // extern "C"

// Row-partitioned tail steps for the multi-GPU engine (internal, see common.h).
int spb200_tail_solve_norm_partial(splatt_b200_als_tail * h, int mode, const double * d_m1,
                                   double * d_x, uint64_t rows, int first_iteration,
                                   double * mc_norm_slot) {
  h->t.solve_norm_partial(d_m1, d_x, rows, mode, first_iteration != 0, mc_norm_slot);
  return h->t.failed ? SPLATT_ERROR_BADINPUT : SPLATT_SUCCESS;
}
int spb200_tail_scale_gram_partial(splatt_b200_als_tail * h, double * d_x, double * mc_x,
                                   uint64_t rows, int first_iteration, const double * norms_all,
                                   int k, int norm_stride, double * mc_gram_slot) {
  h->t.scale_gram_partial(d_x, mc_x, rows, first_iteration != 0, norms_all, k, norm_stride,
                          mc_gram_slot);
  return h->t.failed ? SPLATT_ERROR_BADINPUT : SPLATT_SUCCESS;
}
int spb200_tail_gram_partial(splatt_b200_als_tail * h, const double * d_rows, uint64_t rows,
                             double * mc_gram_slot) {
  h->t.gram_partial(d_rows, rows, mc_gram_slot);
  return h->t.failed ? SPLATT_ERROR_BADINPUT : SPLATT_SUCCESS;
}
int spb200_tail_finish_gram(splatt_b200_als_tail * h, int mode, const double * grams_all, int k,
                            int gram_stride) {
  h->t.finish_gram(mode, grams_all, k, gram_stride);
  return h->t.failed ? SPLATT_ERROR_BADINPUT : SPLATT_SUCCESS;
}

extern "C" {

void splatt_free_kruskal(splatt_kruskal * factored) {
  if (!factored) return;
  free(factored->lambda);
  for (splatt_idx_t m = 0; m < factored->nmodes; ++m) free(factored->factors[m]);
}

}  // extern "C"
