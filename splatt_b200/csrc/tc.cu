// Tensor completion by row-wise ALS on device-resident tensors (splatt_b200_tc_als_device), and
// the residual sum of squares of a Kruskal model at a tensor's nonzeros (splatt_b200_tensor_sse).
//
// Completion fits x^(i_1..i_N) = sum_r prod_m U_m[i_m, r] to the stored entries only.  Updating
// row i of U_m solves (sum_x h_x h_x^T + reg I) u = sum_x v_x h_x over the nonzeros x whose
// mode-m index is i, with h_x the Hadamard product of the other modes' rows.  On the ALLROOT
// layout every mode has a stream with that mode at its root, so the nonzeros of one output row
// are contiguous: the row-update kernel walks the same nnz-balanced chunk ranges as the root
// MTTKRP kernel (one warp per range, its own TMA record ring: walk_range in walk.cuh), keeps the
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
#include "walk.cuh"
#include <algorithm>
#include <cmath>
#include <vector>

namespace spb200 {
namespace {

// doubles per warp of the row-update / solve workspace: the pack (2 NP + RT) and h (RT)
__host__ __device__ constexpr int tc_ws_doubles(int RT) { return 2 * tc_pairs(RT / 2) + 2 * RT; }
__host__ __device__ constexpr size_t tc_tab_bytes(int RT) { return (sizeof(uint32_t) * tc_pairs(RT / 2) + 15) & ~size_t(15); }
__host__ __device__ constexpr size_t tc_update_smem(int RT) {
  return tc_ring_bytes() + tc_tab_bytes(RT) + sizeof(double) * kWarps * tc_ws_doubles(RT);
}
__host__ __device__ constexpr int tc_minb(int RT) { return RT <= 32 ? 2 : 1; }

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
  model_sum<N>(a, [](double s, double v, double x) {
    const double r = v - x;
    return fma(r, r, s);
  });
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

// The row-update kernel of (N, tier, rows mode).
template <int N>
void (*update_kernel(int RT, bool rows))(TcArgs) {
  if (RT == 16) return rows ? k_tc_update<N, 16, true> : k_tc_update<N, 16, false>;
  if (RT == 32) return rows ? k_tc_update<N, 32, true> : k_tc_update<N, 32, false>;
  return rows ? k_tc_update<N, 64, true> : k_tc_update<N, 64, false>;
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
  k<<<combine_grid(nitems), kThreads, smem, s>>>(packs, slot_row, nitems, R, ldm, reg, out);
  spb200_count_launches(1);
  return cudaGetLastError();
}

// SSE of the model (lambda: RP device doubles) over one stream's records, added into *d_sse.
cudaError_t launch_sse(const FiberStream & fs, int R, int ldm, const double * const * d_mats_by_mode,
                       const double * d_lambda, double * d_sse, cudaStream_t s) {
  if (fs.nrec == 0) return cudaSuccess;
  TcArgs a = walk_args(fs, d_mats_by_mode, ldm, R);
  a.lambda = d_lambda; a.sse = d_sse;
  return launch_model_sum(with_nmodes(fs.nmodes, [](auto n) { return k_tc_sse<n.value>; }), a, s);
}

// Device buffers of one completion run, released on every return path.
struct TcBuffers {
  double *   packs = nullptr;
  uint32_t * slot_row = nullptr;
  double *   lambda = nullptr;    // RP ones
  double *   sums = nullptr;      // [0] train SSE, [1] validation SSE, [2] sum ||U_m||^2
  ~TcBuffers() { cudaFree(packs); cudaFree(slot_row); cudaFree(lambda); cudaFree(sums); }
};

}  // namespace

// launch_sse for the other completion solvers (tc_lbfgs.cu)
cudaError_t tc_enqueue_sse(const FiberStream & fs, int R, int ldm, const double * const * d_mats_by_mode,
                           const double * d_lambda, double * d_sse, cudaStream_t s) {
  return launch_sse(fs, R, ldm, d_mats_by_mode, d_lambda, d_sse, s);
}

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
  bool bad = !root_streams_ok(train) || !options ||
             !factors_ok(train->nmodes, R, ldm, reinterpret_cast<const void * const *>(d_factors)) ||
             !(std::isfinite(reg) && reg > 0.0);
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

  // one launch configuration per mode; the pack buffer serves the largest (a leaf-tiled mode: a
  // pack per row)
  const int RT = rank_tier(R);
  WalkLaunch<TcArgs> ml[SPB200_MAXN];
  size_t max_packs = 0;
  for (int m = 0; m < N; ++m) {
    const bool rows = train->streams[train->plan[m].stream].ktile_rows > 0;
    if (!ml[m].configure(with_nmodes(N, [&](auto n) { return update_kernel<n.value>(RT, rows); }),
                         tc_update_smem(RT), rows)) {
      fprintf(stderr, "SPLATT: splatt_b200_tc_als_device: cannot configure the row update (%s)\n",
              cudaGetErrorString(cudaGetLastError()));
      return SPLATT_ERROR_BADINPUT;
    }
    max_packs = std::max<size_t>(max_packs, rows ? train->dims[m] : ml[m].nslots);
  }
  TcBuffers b;
  std::vector<double> ones(RP, 0.0);
  std::fill(ones.begin(), ones.begin() + R, 1.0);
  if (cudaMalloc(&b.packs, std::max<size_t>(max_packs, 1) * P * sizeof(double)) != cudaSuccess ||
      cudaMalloc(&b.slot_row, std::max(max_slots(ml, N), 1ull) * sizeof(uint32_t)) != cudaSuccess ||
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
      const WalkLaunch<TcArgs> & L = ml[m];
      ok = cudaMemset2DAsync(d_factors[m], (size_t)ldm * 8, 0, (size_t)R * 8, train->dims[m], s) == cudaSuccess;
      if (L.rows) ok = ok && cudaMemsetAsync(b.packs, 0, train->dims[m] * P * sizeof(double), s) == cudaSuccess;
      if (!ok) break;
      if (fs.nrec) {
        TcArgs a = walk_args(fs, d_factors, ldm, R);
        a.reg = reg; a.out = d_factors[m];
        a.packs = b.packs; a.slot_row = L.rows ? nullptr : b.slot_row;
        ok = L.launch(a, b.slot_row, s) == cudaSuccess;
      }
      if (L.rows)
        ok = ok && launch_solve(b.packs, nullptr, train->dims[m], R, ldm, reg, d_factors[m], s) == cudaSuccess;
      else if (fs.nrec)
        ok = ok && launch_solve(b.packs, b.slot_row, L.nslots, R, ldm, reg, d_factors[m], s) == cudaSuccess;
    }
    if (!ok) break;
    ok = cudaMemsetAsync(b.sums, 0, 3 * sizeof(double), s) == cudaSuccess;
    for (int m = 0; ok && m < N; ++m) {
      k_tc_sumsq<<<elementwise_grid(train->dims[m], R), kThreads, 0, s>>>(d_factors[m], train->dims[m], R, ldm,
                                                                          b.sums + 2);
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
