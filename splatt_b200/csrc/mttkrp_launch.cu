// Host-side dispatch of one MTTKRP over a fiber stream.
#include "common.h"
#include <cstdlib>
#include <type_traits>

unsigned long long g_spb200_launches = 0;
unsigned long long g_spb200_builds = 0;

// Tuning knob (experiments): records per gather batch of the root kernel.
int spb200_root_batch() {
  static int v = -1;
  if (v < 0) {
    const char * e = getenv("SPLATT_B200_BATCH");
    v = e ? atoi(e) : 0;   // 0 = per-kernel default (4 for 2-3 modes, 2 for deeper trees)
    if (v != 2 && v != 3 && v != 4 && v != 8) v = 0;
  }
  return v;
}

// Tuning knob (experiments): minimum CTAs per SM the 4-mode root kernel is compiled for.
int spb200_root_minb() {
  static int v = -1;
  if (v < 0) {
    const char * e = getenv("SPLATT_B200_MINB");
    v = e ? atoi(e) : 0;
  }
  return v;
}

namespace spb200 {
int launch_n2(int, const MttkrpArgs &, int, cudaStream_t);
int launch_n3(int, const MttkrpArgs &, int, cudaStream_t);
int launch_n4(int, const MttkrpArgs &, int, cudaStream_t);
int launch_n5(int, const MttkrpArgs &, int, cudaStream_t);
int launch_n6(int, const MttkrpArgs &, int, cudaStream_t);
int launch_n7(int, const MttkrpArgs &, int, cudaStream_t);
int launch_n8(int, const MttkrpArgs &, int, cudaStream_t);
int launch_f32_n2(int, const MttkrpArgs &, int, cudaStream_t);
int launch_f32_n3(int, const MttkrpArgs &, int, cudaStream_t);
int launch_f32_n4(int, const MttkrpArgs &, int, cudaStream_t);
int launch_f32_n5(int, const MttkrpArgs &, int, cudaStream_t);
int launch_f32_n6(int, const MttkrpArgs &, int, cudaStream_t);
int launch_f32_n7(int, const MttkrpArgs &, int, cudaStream_t);
int launch_f32_n8(int, const MttkrpArgs &, int, cudaStream_t);
}  // namespace spb200

static int num_sms_of_current_device() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

// T = double or float.  A lane moves 16 bytes of a row, i.e. W = 16 / sizeof(T) columns: ldm,
// the padded rank and column blocks are multiples of W, and one launch covers 32 * W columns.
template <typename T>
static int launch_mttkrp(const FiberStream & s, int kind, int outdepth, int ncolumns, int ldm,
                         const T * const * d_mats_by_mode, T * d_out,
                         uint64_t out_rows, cudaStream_t stream, bool multicast_out,
                         int col_begin, int col_count, const GroupSync * sync) {
  constexpr int W    = 16 / static_cast<int>(sizeof(T));
  constexpr int kCol = 32 * W;        // columns per launch (L = 32)
  const int N = s.nmodes;
  if (N < 2 || N > SPB200_MAXN) {
    fprintf(stderr, "SPLATT: MTTKRP supports 2..%d modes (got %d)\n", SPB200_MAXN, N);
    return SPLATT_ERROR_BADINPUT;
  }
  // padded rank: ncolumns rounded up to a whole lane vector
  const int rpad_all = (ncolumns + W - 1) & ~(W - 1);
  if (ncolumns <= 0 || ldm < rpad_all || (ldm & (W - 1))) {
    if (W == 2)
      fprintf(stderr, "SPLATT: bad ncolumns/ldm (%d/%d): ldm must be even and >= ncolumns\n",
              ncolumns, ldm);
    else
      fprintf(stderr, "SPLATT: bad ncolumns/ldm (%d/%d): ldm must be a multiple of %d and >= ncolumns\n",
              ncolumns, ldm, W);
    return SPLATT_ERROR_BADINPUT;
  }
  // rows are fetched with 128-bit loads: every matrix base must be 16-byte aligned
  for (int m = 0; m < N; ++m) {
    const T * p = d_mats_by_mode[m];
    if (p && (reinterpret_cast<uintptr_t>(p) & 15u)) {
      fprintf(stderr, "SPLATT: factor matrix %d is not 16-byte aligned\n", m);
      return SPLATT_ERROR_BADINPUT;
    }
  }
  if (reinterpret_cast<uintptr_t>(d_out) & 15u) {
    fprintf(stderr, "SPLATT: output matrix is not 16-byte aligned\n");
    return SPLATT_ERROR_BADINPUT;
  }
  if (multicast_out) {
    // the caller zeroed every GPU's buffer and synchronised the group beforehand
    if (kind != SPB200_KIND_ROOT) {
      fprintf(stderr, "SPLATT: multicast output needs a root-oriented stream (ALLROOT layout)\n");
      return SPLATT_ERROR_BADINPUT;
    }
  }
  if (col_count <= 0) { col_begin = 0; col_count = rpad_all; }        // whole matrix
  // a block is widened to the next multiple of W, which must still lie inside rpad_all:
  // past it the zeroing and the kernel would reach into the next row (or past the buffer)
  if ((col_begin & (W - 1)) || col_begin < 0 || col_count > rpad_all - col_begin ||
      col_begin >= rpad_all) {
    fprintf(stderr, "SPLATT: bad column block [%d, %d) of %d\n", col_begin, col_begin + col_count,
            rpad_all);
    return SPLATT_ERROR_BADINPUT;
  }
  const int col_end = (col_begin + col_count + W - 1) & ~(W - 1);     // <= rpad_all
  if (!multicast_out) {
    if (col_begin == 0 && col_end == rpad_all)
      SPB200_CUDA_OK(cudaMemsetAsync(d_out, 0, sizeof(T) * out_rows * ldm, stream));
    else
      SPB200_CUDA_OK(cudaMemset2DAsync(d_out + col_begin, sizeof(T) * ldm, 0,
                                       sizeof(T) * (col_end - col_begin), out_rows, stream));
  }
  if (s.nrec == 0 && !(multicast_out && sync)) return SPLATT_SUCCESS;

  // leaf factor staged in shared memory (CTA-tiled stream, 3-mode root).  That kernel is fp64
  // only: an fp32 call on such a stream runs the generic kernel (leaf-tiled variant).
  if constexpr (std::is_same<T, double>::value) {
    if (!multicast_out && spb200_tiled_applicable(s, kind)) {
      static int use_tiled = -1;
      if (use_tiled < 0) {
        const char * e = getenv("SPLATT_B200_TILED_KERNEL");
        use_tiled = (e && atoi(e) == 0) ? 0 : 1;
      }
      if (use_tiled)
        return spb200_launch_tiled_root3(s, ldm, col_begin, col_end, d_mats_by_mode[s.perm[2]],
                                         d_mats_by_mode[s.perm[1]], d_out, stream);
    }
  }

  MttkrpArgs a;
  a.rec = s.rec;
  for (int l = 0; l < SPB200_MAXN - 2; ++l) a.up[l] = (l <= N - 3) ? s.up[l] : nullptr;   // none for N = 2
  a.desc = s.desc;
  a.anc  = s.anc;
  for (int l = 0; l < SPB200_MAXN; ++l) a.mats[l] = (l < N) ? d_mats_by_mode[s.perm[l]] : nullptr;
  a.out      = d_out;
  a.nrec     = s.nrec;
  if (s.nchunks > 0xffffffffull) {
    fprintf(stderr, "SPLATT: stream too long for one launch (%llu chunks)\n",
            (unsigned long long)s.nchunks);
    return SPLATT_ERROR_BADINPUT;
  }
  a.nchunks  = static_cast<unsigned int>(s.nchunks);
  a.ldm      = ldm;
  a.outdepth = outdepth;
  a.ktiled   = s.ktile_rows ? 1 : 0;
  a.multicast = multicast_out ? 1 : 0;
  a.sync_mc = a.sync_local = a.sync_cta = nullptr;
  a.sync_target = 0;
  a.sync_rank = 0; a.sync_world = 1;
  {
    // SPLATT_B200_STAGGER: 0 = aligned regions (bank conflicts on the broadcast reads),
    // 1 = stagger the record regions, 2 = records and ancestor ids
    static int stagger = -1;
    if (stagger < 0) {
      const char * e = getenv("SPLATT_B200_STAGGER");
      stagger = e ? atoi(e) : 0;
    }
    a.rpad = stagger >= 1 ? 1 : 0;
    a.apad = stagger >= 2 ? 4 : 0;
    // SPLATT_B200_MC_STORE=0: reduce every row of a multicast launch (the round-1 behaviour)
    static int mc_store = -1;
    if (mc_store < 0) {
      const char * e = getenv("SPLATT_B200_MC_STORE");
      mc_store = (e && atoi(e) == 0) ? 0 : 1;
    }
    // (a leaf-tiled stream closes the same root row once per tile: never stored)
    a.mc_store = (mc_store && !s.ktile_rows) ? 1 : 0;
  }

  using Launch = int (*)(int, const MttkrpArgs &, int, cudaStream_t);
  static constexpr Launch kLaunch[] = {spb200::launch_n2, spb200::launch_n3, spb200::launch_n4,
                                       spb200::launch_n5, spb200::launch_n6, spb200::launch_n7,
                                       spb200::launch_n8};
  static constexpr Launch kLaunchF32[] = {spb200::launch_f32_n2, spb200::launch_f32_n3,
                                          spb200::launch_f32_n4, spb200::launch_f32_n5,
                                          spb200::launch_f32_n6, spb200::launch_f32_n7,
                                          spb200::launch_f32_n8};
  const Launch launch = (std::is_same<T, double>::value ? kLaunch : kLaunchF32)[N - 2];
  const int num_sms = num_sms_of_current_device();
  for (int c0 = col_begin; c0 < col_end; c0 += kCol) {
    a.col0  = c0;
    a.ncols = (col_end - c0 < kCol) ? (col_end - c0) : kCol;
    if (multicast_out && sync && c0 + kCol >= col_end) {   // the last column pass carries the barrier
      a.sync_mc = sync->mc_flag; a.sync_local = sync->local_flag; a.sync_cta = sync->cta_done;
      a.sync_target = sync->target;
      a.sync_rank = sync->rank; a.sync_world = sync->world;
    }
    const int rc = launch(kind, a, num_sms, stream);
    if (rc != SPLATT_SUCCESS) return rc;
  }
  return SPLATT_SUCCESS;
}

int spb200_launch_mttkrp(const FiberStream & s, int kind, int outdepth, int ncolumns, int ldm,
                         const double * const * d_mats_by_mode, double * d_out,
                         uint64_t out_rows, cudaStream_t stream, bool multicast_out,
                         int col_begin, int col_count, const GroupSync * sync) {
  return launch_mttkrp<double>(s, kind, outdepth, ncolumns, ldm, d_mats_by_mode, d_out, out_rows,
                               stream, multicast_out, col_begin, col_count, sync);
}

int spb200_launch_mttkrp_f32(const FiberStream & s, int kind, int outdepth, int ncolumns, int ldm,
                             const float * const * d_mats_by_mode, float * d_out,
                             uint64_t out_rows, cudaStream_t stream) {
  return launch_mttkrp<float>(s, kind, outdepth, ncolumns, ldm, d_mats_by_mode, d_out, out_rows,
                              stream, false, 0, 0, nullptr);
}


// ---------------------------------------------------------------------------
// Gather probe: the speed of light of the MTTKRP's dominant access pattern on
// this GPU.  Every group of `lanes` lanes fetches whole rows (2 doubles per lane,
// one LDG.128 each) of a rows x ld matrix at the indices idx[0..nidx), eight
// rows in flight per group, and does nothing else.  bench.py times it to put a
// MEASURED ceiling next to the kernel's achieved L2->SM gather rate.
// ---------------------------------------------------------------------------
template <int L>
__global__ void __launch_bounds__(256, 3)
gather_probe_kernel(const double * __restrict__ mat, int ld, const uint32_t * __restrict__ idx,
                    unsigned long long nidx, double * __restrict__ sink) {
  constexpr int G = 32 / L;
  const int lane = threadIdx.x & 31, grp = lane / L, gl = lane % L;
  const unsigned long long ngroups = (unsigned long long)gridDim.x * (blockDim.x / 32) * G;
  const unsigned long long g = ((unsigned long long)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5)) * G + grp;
  const unsigned long long b0 = g * nidx / ngroups, b1 = (g + 1) * nidx / ngroups;
  const char * base = reinterpret_cast<const char *>(mat + 2 * gl);
  const uint32_t pitch = (uint32_t)ld * 8u;
  double2 acc = make_double2(0.0, 0.0);
  unsigned long long n = b0;
  for (; n + 8 <= b1; n += 8) {
    uint32_t k[8];
    double2  r[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) k[u] = __ldg(&idx[n + u]);
#pragma unroll
    for (int u = 0; u < 8; ++u)
      r[u] = __ldg(reinterpret_cast<const double2 *>(base + (unsigned long long)k[u] * pitch));
#pragma unroll
    for (int u = 0; u < 8; ++u) { acc.x += r[u].x; acc.y += r[u].y; }
  }
  if (acc.x == 1.2345e300) sink[0] = acc.x + acc.y;   // keep the loads alive
}

extern "C" int splatt_b200_gather_probe(double const * d_mat, int ncolumns, int ldm,
                                        uint32_t const * d_idx, uint64_t nidx, double * d_sink,
                                        void * stream) {
  if (!d_mat || !d_idx || !d_sink || ncolumns <= 0 || (ldm & 1) || ldm < ncolumns) return SPLATT_ERROR_BADINPUT;
  const int grid = num_sms_of_current_device() * 3;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int rp = ncolumns + (ncolumns & 1);
  if (rp <= 8) gather_probe_kernel<4><<<grid, 256, 0, s>>>(d_mat, ldm, d_idx, nidx, d_sink);
  else if (rp <= 16) gather_probe_kernel<8><<<grid, 256, 0, s>>>(d_mat, ldm, d_idx, nidx, d_sink);
  else if (rp <= 32) gather_probe_kernel<16><<<grid, 256, 0, s>>>(d_mat, ldm, d_idx, nidx, d_sink);
  else gather_probe_kernel<32><<<grid, 256, 0, s>>>(d_mat, ldm, d_idx, nidx, d_sink);
  SPB200_CUDA_OK(cudaGetLastError());
  return SPLATT_SUCCESS;
}


// ---------------------------------------------------------------------------
// Probe sweep: the same access pattern at a chosen occupancy (CTAs of 256 threads
// per SM), rows in flight per lane group, L1 allocation policy and shared-memory
// reservation (= how much of the unified L1/shared array is left as L1).  scripts/probe_sweep.py sweeps these to find the
// best the hardware gives for random whole-row gathers -- the ceiling the MTTKRP
// kernel is compared with is the BEST point of the sweep, not one kernel shape.
// ---------------------------------------------------------------------------
template <int L, int ROWS, bool NA>
__global__ void __launch_bounds__(256)
gather_probe_sweep_kernel(const double * __restrict__ mat, int ld, const uint32_t * __restrict__ idx,
                          unsigned long long nidx, double * __restrict__ sink) {
  constexpr int G = 32 / L;
  const int lane = threadIdx.x & 31, grp = lane / L, gl = lane % L;
  const unsigned long long ngroups = (unsigned long long)gridDim.x * (blockDim.x / 32) * G;
  const unsigned long long g = ((unsigned long long)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5)) * G + grp;
  const unsigned long long b0 = g * nidx / ngroups, b1 = (g + 1) * nidx / ngroups;
  const char * base = reinterpret_cast<const char *>(mat + 2 * gl);
  const uint32_t pitch = (uint32_t)ld * 8u;
  double2 acc = make_double2(0.0, 0.0);
  for (unsigned long long n = b0; n + ROWS <= b1; n += ROWS) {
    uint32_t k[ROWS];
    double2  r[ROWS];
#pragma unroll
    for (int u = 0; u < ROWS; ++u) k[u] = __ldg(&idx[n + u]);
#pragma unroll
    for (int u = 0; u < ROWS; ++u) {
      const char * p = base + (unsigned long long)k[u] * pitch;
      if constexpr (NA) {
        asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0, %1}, [%2];"
                     : "=d"(r[u].x), "=d"(r[u].y) : "l"(p));
      } else {
        r[u] = __ldg(reinterpret_cast<const double2 *>(p));
      }
    }
#pragma unroll
    for (int u = 0; u < ROWS; ++u) { acc.x += r[u].x; acc.y += r[u].y; }
  }
  if (acc.x == 1.2345e300) sink[0] = acc.x + acc.y;
}

template <int L, int ROWS, bool NA>
static cudaError_t probe_launch(int grid, size_t smem, cudaStream_t s, const double * m, int ld,
                                const uint32_t * idx, unsigned long long n, double * sink) {
  cudaError_t e = cudaFuncSetAttribute(gather_probe_sweep_kernel<L, ROWS, NA>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  gather_probe_sweep_kernel<L, ROWS, NA><<<grid, 256, smem, s>>>(m, ld, idx, n, sink);
  return cudaGetLastError();
}

extern "C" int splatt_b200_gather_probe_ex(double const * d_mat, int ncolumns, int ldm,
                                           uint32_t const * d_idx, uint64_t nidx, double * d_sink,
                                           int ctas_per_sm, int rows_in_flight, int no_allocate,
                                           int smem_bytes, void * stream) {
  if (!d_mat || !d_idx || !d_sink || ncolumns <= 0 || (ldm & 1) || ldm < ncolumns ||
      ctas_per_sm < 1 || ctas_per_sm > 8) return SPLATT_ERROR_BADINPUT;
  const int rp = ncolumns + (ncolumns & 1);
  if (rp != 16 && rp != 32 && rp != 64) return SPLATT_ERROR_BADINPUT;   // L = 8 / 16 / 32
  const int grid = num_sms_of_current_device() * ctas_per_sm;
  // grid = SMs x ctas_per_sm CTAs of 256 threads, all resident at once (<= 8 per SM): the
  // block scheduler spreads them evenly.  smem_bytes of dynamic shared memory per CTA only
  // shrinks the L1 (unified with shared memory) -- the L1 holds the lines of in-flight misses.
  if (smem_bytes < 0 || (size_t)smem_bytes * ctas_per_sm > 220 * 1024) return SPLATT_ERROR_BADINPUT;
  const size_t smem = (size_t)smem_bytes;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaErrorInvalidValue;
#define SPB200_PROBE(LL, RR)                                                                    \
  e = no_allocate ? probe_launch<LL, RR, true>(grid, smem, s, d_mat, ldm, d_idx, nidx, d_sink)  \
                  : probe_launch<LL, RR, false>(grid, smem, s, d_mat, ldm, d_idx, nidx, d_sink)
#define SPB200_PROBE_L(LL)                                                                      \
  do {                                                                                          \
    if (rows_in_flight == 2) { SPB200_PROBE(LL, 2); }                                           \
    else if (rows_in_flight == 4) { SPB200_PROBE(LL, 4); }                                      \
    else if (rows_in_flight == 8) { SPB200_PROBE(LL, 8); }                                      \
    else if (rows_in_flight == 16) { SPB200_PROBE(LL, 16); }                                    \
  } while (0)
  if (rp == 16) SPB200_PROBE_L(8);
  else if (rp == 32) SPB200_PROBE_L(16);
  else SPB200_PROBE_L(32);
#undef SPB200_PROBE_L
#undef SPB200_PROBE
  SPB200_CUDA_OK(e);
  return SPLATT_SUCCESS;
}
