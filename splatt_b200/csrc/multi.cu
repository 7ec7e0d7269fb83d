// Single-process multi-GPU engine: ONE host process drives k GPUs of one NVSwitch box.
//
// This is the C-ABI counterpart of the reference's distributed driver
// (mpi_cpd_als_iterate, src/mpi/mpi_cpd.c:627-804; per-mode reduction :250-308) for one
// node: the tensor is partitioned, every device computes the MTTKRP of its share, the
// output factor is summed over devices once per mode, the dense tail is row-partitioned
// over the devices (single-valued factors; see splatt_b200_multi_cpd_als).
// Differences that make it native to an NVSwitch box of H100s:
//   * partition = equal-nnz contiguous chunk ranges of every fiber stream (built once on
//     the first device, the shares are cut out and moved device-to-device);
//   * exchange  = inside the MTTKRP kernel: every finished output row goes into ALL devices'
//     buffers through an NVLink multicast mapping created here with the CUDA driver's
//     multicast objects (no NCCL, no torch) -- multimem.red.add.f64 for rows shared between
//     lane groups or devices, a plain 128-bit store for rows one lane group finishes alone --
//     and the group barrier is the kernel's own tail (mttkrp_kernels.cuh);
//   * fallback  = when the box has no multicast support: local kernels, then a peer-memory
//     reduce kernel (each device sums one row slice over all peers' partials and writes
//     the sum into every peer's result buffer), ordered with CUDA events.
#include "common.h"
#include <cuda.h>
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace {

constexpr int kMaxDev = 16;

// ---------------------------------------------------------------------------
// Driver entry points, resolved through the runtime (no link dependency on libcuda:
// the library must load on a machine without a GPU driver).
// ---------------------------------------------------------------------------
#define SPB200_DRV_LIST(X)        \
  X(cuDeviceGet)                  \
  X(cuDeviceGetAttribute)         \
  X(cuMulticastCreate)            \
  X(cuMulticastAddDevice)         \
  X(cuMulticastBindMem)           \
  X(cuMulticastUnbind)            \
  X(cuMulticastGetGranularity)    \
  X(cuMemCreate)                  \
  X(cuMemRelease)                 \
  X(cuMemAddressReserve)          \
  X(cuMemAddressFree)             \
  X(cuMemMap)                     \
  X(cuMemUnmap)                   \
  X(cuMemSetAccess)               \
  X(cuMemGetAllocationGranularity)

struct Drv {
#define X(name) decltype(&name) name##_ = nullptr;
  SPB200_DRV_LIST(X)
#undef X
  bool ok = false;
};

const Drv & drv() {
  static Drv d;
  static bool tried = false;
  if (tried) return d;
  tried = true;
  bool ok = true;
#define X(name)                                                                              \
  {                                                                                          \
    void * fp = nullptr;                                                                     \
    cudaDriverEntryPointQueryResult qr;                                                      \
    if (cudaGetDriverEntryPoint(#name, &fp, cudaEnableDefault, &qr) != cudaSuccess || !fp || \
        qr != cudaDriverEntryPointSuccess) {                                                 \
      ok = false;                                                                            \
      cudaGetLastError();                                                                    \
    }                                                                                        \
    d.name##_ = reinterpret_cast<decltype(&name)>(fp);                                       \
  }
  SPB200_DRV_LIST(X)
#undef X
  d.ok = ok;
  return d;
}

size_t round_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// One region of `bytes` on every device, all bound to one multicast object:
// uc[d] = device d's own (unicast) address of its copy, mc = the multicast address.
struct McRegion {
  int k = 0;
  size_t bytes = 0;
  CUmemGenericAllocationHandle mch = 0;
  CUmemGenericAllocationHandle mem[kMaxDev] = {0};
  CUdeviceptr mc = 0;
  CUdeviceptr uc[kMaxDev] = {0};
  CUdevice cud[kMaxDev] = {0};
  bool bound[kMaxDev] = {false};
  bool mc_mapped = false, uc_mapped[kMaxDev] = {false};

  bool create(int k_, const int * devs, size_t want, int verbosity) {
    const Drv & D = drv();
    if (!D.ok) { if (verbosity > 1) fprintf(stderr, "SPLATT-B200: driver entry points unavailable\n"); return false; }
    k = k_;
    for (int i = 0; i < k; ++i) {
      for (int j = 0; j < i; ++j)
        if (devs[j] == devs[i]) return false;            // a device can join a team once
      if (cudaSetDevice(devs[i]) != cudaSuccess || cudaFree(0) != cudaSuccess) return false;
      if (D.cuDeviceGet_(&cud[i], devs[i]) != CUDA_SUCCESS) return false;
      int sup = 0;
      if (D.cuDeviceGetAttribute_(&sup, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, cud[i]) != CUDA_SUCCESS || !sup) {
        if (verbosity > 1) fprintf(stderr, "SPLATT-B200: device %d has no multicast support\n", devs[i]);
        return false;
      }
    }
    // every step reports its CUresult on failure: the caller falls back to the peer reduce
#define MC_TRY(call)                                                                       \
    do {                                                                                     \
      CUresult r_ = (call);                                                                  \
      if (r_ != CUDA_SUCCESS) {                                                              \
        fprintf(stderr, "SPLATT-B200: multicast set-up: %s -> CUresult %d\n", #call, (int)r_); \
        destroy();                                                                           \
        return false;                                                                        \
      }                                                                                      \
    } while (0)
    CUmulticastObjectProp mp;
    memset(&mp, 0, sizeof(mp));
    mp.numDevices = (unsigned)k;
    mp.handleTypes = 0;
    mp.flags = 0;
    mp.size = want;
    size_t gran = 0;
    MC_TRY(D.cuMulticastGetGranularity_(&gran, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED));
    if (!gran) return false;
    CUmemAllocationProp ap;
    memset(&ap, 0, sizeof(ap));
    ap.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    ap.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    ap.location.id = cud[0];
    size_t g2 = 0;
    if (D.cuMemGetAllocationGranularity_(&g2, &ap, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED) == CUDA_SUCCESS && g2 > gran)
      gran = g2;
    bytes = round_up(want, gran);
    mp.size = bytes;
    MC_TRY(D.cuMulticastCreate_(&mch, &mp));
    for (int i = 0; i < k; ++i) MC_TRY(D.cuMulticastAddDevice_(mch, cud[i]));
    for (int i = 0; i < k; ++i) {
      ap.location.id = cud[i];
      MC_TRY(D.cuMemCreate_(&mem[i], bytes, &ap, 0));
      MC_TRY(D.cuMulticastBindMem_(mch, 0, mem[i], 0, bytes, 0));
      bound[i] = true;
      MC_TRY(D.cuMemAddressReserve_(&uc[i], bytes, gran, 0, 0));
      MC_TRY(D.cuMemMap_(uc[i], bytes, 0, mem[i], 0));
      uc_mapped[i] = true;
      CUmemAccessDesc ad;
      memset(&ad, 0, sizeof(ad));
      ad.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
      ad.location.id = cud[i];
      ad.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
      MC_TRY(D.cuMemSetAccess_(uc[i], bytes, &ad, 1));
    }
    MC_TRY(D.cuMemAddressReserve_(&mc, bytes, gran, 0, 0));
    MC_TRY(D.cuMemMap_(mc, bytes, 0, mch, 0));
    mc_mapped = true;
    CUmemAccessDesc ads[kMaxDev];
    memset(ads, 0, sizeof(ads));
    for (int i = 0; i < k; ++i) {
      ads[i].location.type = CU_MEM_LOCATION_TYPE_DEVICE;
      ads[i].location.id = cud[i];
      ads[i].flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    }
    MC_TRY(D.cuMemSetAccess_(mc, bytes, ads, (size_t)k));
#undef MC_TRY
    return true;
  }

  void destroy() {
    const Drv & D = drv();
    if (!D.ok) return;
    if (mc) {
      if (mc_mapped) D.cuMemUnmap_(mc, bytes);
      D.cuMemAddressFree_(mc, bytes);
      mc = 0; mc_mapped = false;
    }
    for (int i = 0; i < k; ++i) {
      if (uc[i]) {
        if (uc_mapped[i]) D.cuMemUnmap_(uc[i], bytes);
        D.cuMemAddressFree_(uc[i], bytes);
        uc[i] = 0; uc_mapped[i] = false;
      }
      if (bound[i]) {
        D.cuMulticastUnbind_(mch, cud[i], 0, bytes);
        bound[i] = false;
      }
      if (mem[i]) { D.cuMemRelease_(mem[i]); mem[i] = 0; }
    }
    if (mch) { D.cuMemRelease_(mch); mch = 0; }
  }
};

struct PeerReduceArgs {
  const double2 * part[kMaxDev];
  double2 *       res[kMaxDev];
  int             k;
};

// Fallback exchange: sum the partial outputs of all devices over the element range
// [e0, e1) (double2 units) and write the sum into every device's result buffer.
__global__ void k_peer_reduce(const PeerReduceArgs a, unsigned long long e0, unsigned long long e1) {
  for (unsigned long long i = e0 + (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < e1;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    double2 s = a.part[0][i];
    for (int p = 1; p < a.k; ++p) {
      const double2 v = a.part[p][i];
      s.x += v.x; s.y += v.y;
    }
    for (int p = 0; p < a.k; ++p) a.res[p][i] = s;
  }
}

// Stand-alone group barrier (same flag array and sequence numbers as the MTTKRP kernel's
// tail): the kernels before it on this stream have completed, so their multicast stores are
// performed; publish the sequence number in this GPU's slot on every GPU, wait for all slots.
__device__ __forceinline__ void mg_signal_and_wait(uint32_t * mc_flags, uint32_t * local_flags,
                                                   uint32_t epoch, uint32_t rank, uint32_t world) {
  asm volatile("multimem.st.release.sys.global.u32 [%0], %1;" ::"l"(mc_flags + rank), "r"(epoch) : "memory");
  for (uint32_t r = 0; r < world; ++r) {
    unsigned int v;
    do {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(local_flags + r) : "memory");
    } while (static_cast<int>(v - epoch) < 0);
  }
}
__global__ void k_group_barrier(uint32_t * mc_flags, uint32_t * local_flags, uint32_t epoch,
                                uint32_t rank, uint32_t world) {
  if (threadIdx.x == 0) {
    __threadfence_system();
    mg_signal_and_wait(mc_flags, local_flags, epoch, rank, world);
  }
}

struct DevState {
  int dev = 0;
  splatt_b200_tensor * T = nullptr;
  cudaStream_t stream = nullptr;
  double * mats[SPB200_MAXN] = {nullptr};   // factor replicas, dims[m] x ldm
  double * out[SPB200_MAXN] = {nullptr};    // this device's (unicast) output buffer per mode
  double * part = nullptr;                  // fallback: local partial, maxdim x ldm
  uint32_t * flag_local = nullptr;
  double * norms_local = nullptr;           // this device's copy of the k norm slots
  double * grams_local = nullptr;           // ... and of the k Gram slots
  cudaEvent_t ev_k = nullptr, ev_r = nullptr;
  cudaEvent_t ev_tail = nullptr;            // device 0: the mode's new factor is ready
  cudaStream_t copy = nullptr;              // PCIe copies of the host-buffer call's column pipeline
  cudaEvent_t ev_h2d[2] = {nullptr, nullptr}, ev_kb[2] = {nullptr, nullptr};
  splatt_b200_als_tail * tail = nullptr;    // device 0 only (see splatt_b200_multi_cpd_als)
};

#define MCK(call)                                                                               \
  do {                                                                                          \
    cudaError_t e_ = (call);                                                                    \
    if (e_ != cudaSuccess) {                                                                    \
      fprintf(stderr, "SPLATT: CUDA error '%s' at %s:%d (%s)\n", cudaGetErrorString(e_),       \
              __FILE__, __LINE__, #call);                                                       \
      return (e_ == cudaErrorMemoryAllocation) ? SPLATT_ERROR_NOMEMORY : SPLATT_ERROR_BADINPUT; \
    }                                                                                           \
  } while (0)

}  // namespace

struct splatt_b200_multi {
  int k = 0;
  int N = 0;
  uint64_t dims[SPB200_MAXN] = {0};
  uint64_t maxdim = 0;
  uint64_t nnz = 0;
  int R = 0, ldm = 0;
  bool multicast = false;
  bool distinct = true;            // all devices distinct (false only in tests: "0,0")
  McRegion mc;
  size_t out_off[SPB200_MAXN] = {0};
  size_t mat_off[SPB200_MAXN] = {0};
  size_t norm_off = 0, gram_off = 0;
  int norm_stride = 0, gram_stride = 0;      // doubles per device slot
  double * mc_out[SPB200_MAXN] = {nullptr};
  double * mc_mats[SPB200_MAXN] = {nullptr}; // multicast addresses of the factor replicas
  double * mc_norms = nullptr;               // k slots of partial column norms
  double * mc_grams = nullptr;               // k slots of partial Grams
  uint32_t * mc_flag = nullptr;
  uint32_t epoch = 0;
  DevState d[kMaxDev];
  int prev_dev = 0;
  double last_ms = 0;
  // page-locked bounce buffers for pageable caller memory (see dropin.cu)
  double * stage_in = nullptr;  size_t stage_in_cap = 0;
  double * stage_out = nullptr; size_t stage_out_cap = 0;
};

namespace {

int multi_alloc_buffers(splatt_b200_multi * h, int verbosity) {
  const int k = h->k, N = h->N;
  int devs[kMaxDev];
  for (int i = 0; i < k; ++i) devs[i] = h->d[i].dev;
  // multicast region: [flags 4 KB][k norm slots][k Gram slots][out mode 0..][factor mode 0..]
  size_t off = 4096;
  h->norm_stride = (h->R + 15) / 16 * 16;
  h->gram_stride = h->R * h->R;
  h->norm_off = off;
  off += round_up((size_t)k * h->norm_stride * 8, 4096);
  h->gram_off = off;
  off += round_up((size_t)k * h->gram_stride * 8, 4096);
  for (int m = 0; m < N; ++m) {
    h->out_off[m] = off;
    off += round_up(h->dims[m] * (size_t)h->ldm * 8, 4096);
  }
  for (int m = 0; m < N; ++m) {
    h->mat_off[m] = off;
    off += round_up(h->dims[m] * (size_t)h->ldm * 8, 4096);
  }
  const char * me = getenv("SPLATT_B200_MULTICAST");
  const bool want_mc = !(me && atoi(me) == 0) && h->distinct && k > 1;
  h->multicast = want_mc && h->mc.create(k, devs, off, verbosity);
  if (want_mc && !h->multicast && verbosity > 0)
    fprintf(stderr, "SPLATT-B200: NVLink multicast unavailable; using the peer-memory reduce\n");
  for (int i = 0; i < k; ++i) {
    DevState & s = h->d[i];
    MCK(cudaSetDevice(s.dev));
    MCK(cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking));
    if (s.T && !s.T->cta_done) {     // scratch of the in-kernel barrier: not lazily, later launches
      MCK(cudaMalloc(&s.T->cta_done, 64));   // come from one host thread per device
      MCK(cudaMemset(s.T->cta_done, 0, 64));
    }
    MCK(cudaEventCreateWithFlags(&s.ev_k, cudaEventDisableTiming));
    MCK(cudaEventCreateWithFlags(&s.ev_r, cudaEventDisableTiming));
    MCK(cudaEventCreateWithFlags(&s.ev_tail, cudaEventDisableTiming));
    MCK(cudaStreamCreateWithFlags(&s.copy, cudaStreamNonBlocking));
    for (int b = 0; b < 2; ++b) {
      MCK(cudaEventCreateWithFlags(&s.ev_h2d[b], cudaEventDisableTiming));
      MCK(cudaEventCreateWithFlags(&s.ev_kb[b], cudaEventDisableTiming));
    }
    if (h->multicast) {
      char * base = reinterpret_cast<char *>(h->mc.uc[i]);
      MCK(cudaMemset(base, 0, h->mc.bytes));
      s.flag_local = reinterpret_cast<uint32_t *>(base);
      s.norms_local = reinterpret_cast<double *>(base + h->norm_off);
      s.grams_local = reinterpret_cast<double *>(base + h->gram_off);
      for (int m = 0; m < N; ++m) {
        s.out[m] = reinterpret_cast<double *>(base + h->out_off[m]);
        s.mats[m] = reinterpret_cast<double *>(base + h->mat_off[m]);   // replicas live in the region
      }
    } else {
      for (int m = 0; m < N; ++m) {
        MCK(cudaMalloc(&s.mats[m], h->dims[m] * (size_t)h->ldm * 8));
        MCK(cudaMemset(s.mats[m], 0, h->dims[m] * (size_t)h->ldm * 8));
      }
      MCK(cudaMalloc(&s.part, h->maxdim * (size_t)h->ldm * 8));
      for (int m = 0; m < N; ++m) MCK(cudaMalloc(&s.out[m], h->dims[m] * (size_t)h->ldm * 8));
    }
    MCK(cudaDeviceSynchronize());
  }
  if (h->multicast) {
    char * mb = reinterpret_cast<char *>(h->mc.mc);
    h->mc_flag = reinterpret_cast<uint32_t *>(mb);
    h->mc_norms = reinterpret_cast<double *>(mb + h->norm_off);
    h->mc_grams = reinterpret_cast<double *>(mb + h->gram_off);
    for (int m = 0; m < N; ++m) {
      h->mc_out[m] = reinterpret_cast<double *>(mb + h->out_off[m]);
      h->mc_mats[m] = reinterpret_cast<double *>(mb + h->mat_off[m]);
    }
  }
  if (h->distinct && k > 1) {
    // peer access: the reduce kernel of the fallback reads / writes peer buffers directly, and
    // the CPD driver's factor hand-off (cudaMemcpyPeerAsync) then goes straight over NVLink
    for (int i = 0; i < k; ++i) {
      MCK(cudaSetDevice(h->d[i].dev));
      for (int j = 0; j < k; ++j) {
        if (i == j) continue;
        int can = 0;
        MCK(cudaDeviceCanAccessPeer(&can, h->d[i].dev, h->d[j].dev));
        if (!can) {
          if (h->multicast) continue;            // copies fall back to staging; still correct
          fprintf(stderr, "SPLATT: devices %d and %d have no peer access\n", h->d[i].dev, h->d[j].dev);
          return SPLATT_ERROR_BADINPUT;
        }
        cudaError_t e = cudaDeviceEnablePeerAccess(h->d[j].dev, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) MCK(e);
        cudaGetLastError();
      }
    }
  }
  return SPLATT_SUCCESS;
}

// The fused kernel of device i for barrier sequence number `epoch`.
int enqueue_mc_device(splatt_b200_multi * h, int i, int mode, uint32_t epoch) {
  DevState & s = h->d[i];
  splatt_b200_group_sync gs;
  gs.mc_flag = h->mc_flag;
  gs.local_flag = s.flag_local;
  gs.target = epoch;
  gs.rank = (uint32_t)i;
  gs.world = (uint32_t)h->k;
  gs.reserved = 0;
  return splatt_b200_mttkrp_multicast_sync(s.T, mode, h->R, h->ldm, s.mats, h->mc_out[mode], &gs,
                                           s.stream);
}

// In the multicast path nothing orders the devices on the host (the barriers are on the
// devices), so every device gets its own host thread for the enqueue: with 8 devices the
// ~10 API calls per device and mode otherwise add up to the duration of the kernels.
// All host-side parallel regions of this file use ONE team size: libgomp re-creates threads
// when consecutive regions ask for different team sizes (measured: 16-thread staging copies
// alternating with 2-thread device regions cost 0.3-0.4 ms per switch).
constexpr int kHostTeam = 16;

template <class F>
int for_each_device_parallel(int k, F f) {
  int rc_all = SPLATT_SUCCESS;
#pragma omp parallel for num_threads(kHostTeam) schedule(static, 1) reduction(max : rc_all)
  for (int i = 0; i < k; ++i) {
    const int r = f(i);
    if (r != SPLATT_SUCCESS && r > rc_all) rc_all = r;
  }
  return rc_all;
}

// One MTTKRP over all devices; on return (in stream order of every device) out[d][mode]
// holds the full sum on every device.
int multi_mttkrp_enqueue(splatt_b200_multi * h, int mode) {
  const int k = h->k;
  if (h->multicast) {
    const uint32_t epoch = ++h->epoch;
    return for_each_device_parallel(k, [&](int i) { return enqueue_mc_device(h, i, mode, epoch); });
  }
  // fallback: local partials, then the peer reduce
  for (int i = 0; i < k; ++i) {
    DevState & s = h->d[i];
    int rc = splatt_b200_mttkrp(s.T, mode, h->R, h->ldm, s.mats, k > 1 ? s.part : s.out[mode], s.stream);
    if (rc != SPLATT_SUCCESS) return rc;
    if (k > 1) { MCK(cudaSetDevice(s.dev)); MCK(cudaEventRecord(s.ev_k, s.stream)); }
  }
  if (k == 1) return SPLATT_SUCCESS;
  PeerReduceArgs a;
  a.k = k;
  for (int p = 0; p < k; ++p) {
    a.part[p] = reinterpret_cast<const double2 *>(h->d[p].part);
    a.res[p] = reinterpret_cast<double2 *>(h->d[p].out[mode]);
  }
  const unsigned long long I = h->dims[mode], half = (unsigned long long)h->ldm / 2;
  for (int i = 0; i < k; ++i) {
    DevState & s = h->d[i];
    MCK(cudaSetDevice(s.dev));
    for (int p = 0; p < k; ++p)
      if (p != i) MCK(cudaStreamWaitEvent(s.stream, h->d[p].ev_k, 0));
    const unsigned long long e0 = I * i / k * half, e1 = I * (i + 1) / k * half;
    if (e1 > e0) {
      const unsigned blocks = (unsigned)std::min<unsigned long long>((e1 - e0 + 255) / 256, 132ull * 8);
      k_peer_reduce<<<blocks, 256, 0, s.stream>>>(a, e0, e1);
      spb200_count_launches(1);
      MCK(cudaGetLastError());
    }
    MCK(cudaEventRecord(s.ev_r, s.stream));
  }
  for (int i = 0; i < k; ++i) {
    DevState & s = h->d[i];
    MCK(cudaSetDevice(s.dev));
    for (int p = 0; p < k; ++p)
      if (p != i) MCK(cudaStreamWaitEvent(s.stream, h->d[p].ev_r, 0));
  }
  return SPLATT_SUCCESS;
}

// Result of `mode` consumed on device i: make its buffer ready for the next use.
int multi_release(splatt_b200_multi * h, int i, int mode) {
  if (!h->multicast) return SPLATT_SUCCESS;
  DevState & s = h->d[i];
  MCK(cudaSetDevice(s.dev));
  MCK(cudaMemsetAsync(s.out[mode], 0, h->dims[mode] * (size_t)h->ldm * 8, s.stream));
  return SPLATT_SUCCESS;
}

bool host_pinned(const void * p, size_t bytes) {
  cudaPointerAttributes a0, a1;
  if (cudaPointerGetAttributes(&a0, p) != cudaSuccess) { cudaGetLastError(); return false; }
  if (a0.type != cudaMemoryTypeHost) return false;
  if (bytes <= 1) return true;
  if (cudaPointerGetAttributes(&a1, static_cast<const char *>(p) + bytes - 1) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a1.type == cudaMemoryTypeHost;
}

void par_memcpy(void * dst, const void * src, size_t bytes) {
  const size_t chunk = 1 << 17;
  const int64_t n = (int64_t)((bytes + chunk - 1) / chunk);
#pragma omp parallel for schedule(static) num_threads(kHostTeam)
  for (int64_t c = 0; c < n; ++c) {
    const size_t o = (size_t)c * chunk;
    memcpy(static_cast<char *>(dst) + o, static_cast<const char *>(src) + o, std::min(chunk, bytes - o));
  }
}

int parse_devices(int * devs) {
  // SPLATT_B200_DEVICES="0,1,2,3" wins; else SPLATT_B200_NGPUS=k -> devices 0..k-1
  int n = 0;
  const char * dl = getenv("SPLATT_B200_DEVICES");
  if (dl && *dl) {
    const char * p = dl;
    while (*p && n < kMaxDev) {
      char * end = nullptr;
      long v = strtol(p, &end, 10);
      if (end == p) break;
      devs[n++] = (int)v;
      p = (*end == ',') ? end + 1 : end;
    }
    return n;
  }
  const char * ng = getenv("SPLATT_B200_NGPUS");
  if (ng && atoi(ng) > 1) {
    n = std::min(atoi(ng), kMaxDev);
    for (int i = 0; i < n; ++i) devs[i] = i;
  }
  return n;
}

}  // namespace

extern "C" {

int splatt_b200_multi_env_devices(int * devices, int cap) {
  int devs[kMaxDev];
  const int n = parse_devices(devs);
  for (int i = 0; i < n && i < cap; ++i) devices[i] = devs[i];
  return n;
}

void splatt_b200_multi_free(splatt_b200_multi * h) {
  if (!h) return;
  for (int i = 0; i < h->k; ++i) {
    DevState & s = h->d[i];
    cudaSetDevice(s.dev);
    if (s.stream) cudaStreamSynchronize(s.stream);
  }
  for (int i = 0; i < h->k; ++i) {
    DevState & s = h->d[i];
    cudaSetDevice(s.dev);
    if (s.tail) splatt_b200_als_tail_free(s.tail);
    for (int m = 0; m < SPB200_MAXN; ++m) {
      if (!h->multicast && s.mats[m]) cudaFree(s.mats[m]);
      if (!h->multicast && s.out[m]) cudaFree(s.out[m]);
    }
    if (s.part) cudaFree(s.part);
    if (s.ev_k) cudaEventDestroy(s.ev_k);
    if (s.ev_r) cudaEventDestroy(s.ev_r);
    if (s.ev_tail) cudaEventDestroy(s.ev_tail);
    for (int b = 0; b < 2; ++b) {
      if (s.ev_h2d[b]) cudaEventDestroy(s.ev_h2d[b]);
      if (s.ev_kb[b]) cudaEventDestroy(s.ev_kb[b]);
    }
    if (s.copy) { cudaStreamSynchronize(s.copy); cudaStreamDestroy(s.copy); }
    if (s.stream) cudaStreamDestroy(s.stream);
    if (s.T) splatt_b200_tensor_free(s.T);
  }
  if (h->multicast) h->mc.destroy();
  if (h->stage_in) cudaFreeHost(h->stage_in);
  if (h->stage_out) cudaFreeHost(h->stage_out);
  cudaSetDevice(h->prev_dev);
  delete h;
}

int splatt_b200_multi_create(splatt_csf const * tensors, int csf_alloc, int ncolumns,
                             int const * devices, int ndevices, int verbosity,
                             splatt_b200_multi ** out) {
  if (!tensors || !out || ncolumns < 1 || !devices || ndevices < 1 || ndevices > kMaxDev) {
    fprintf(stderr, "SPLATT: splatt_b200_multi_create: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  int ndev_sys = 0;
  MCK(cudaGetDeviceCount(&ndev_sys));
  for (int i = 0; i < ndevices; ++i)
    if (devices[i] < 0 || devices[i] >= ndev_sys) {
      fprintf(stderr, "SPLATT: CUDA device %d requested, %d present\n", devices[i], ndev_sys);
      return SPLATT_ERROR_BADINPUT;
    }
  splatt_b200_multi * h = new splatt_b200_multi();
  cudaGetDevice(&h->prev_dev);
  h->k = ndevices;
  h->N = (int)tensors[0].nmodes;
  h->R = ncolumns;
  h->ldm = ncolumns + (ncolumns & 1);
  h->nnz = tensors[0].nnz;
  for (int m = 0; m < h->N; ++m) {
    h->dims[m] = tensors[0].dims[m];
    h->maxdim = std::max(h->maxdim, h->dims[m]);
  }
  for (int i = 0; i < ndevices; ++i) {
    h->d[i].dev = devices[i];
    for (int j = 0; j < i; ++j)
      if (devices[j] == devices[i]) h->distinct = false;
  }
  // 1. whole tensor on the first device (one upload, one sort per stream) ...
  splatt_b200_build_opts bo;
  memset(&bo, 0, sizeof(bo));
  bo.layout = SPLATT_B200_LAYOUT_ALLROOT;   // the fused exchange needs root kernels
  bo.device = devices[0];
  bo.verbosity = verbosity;
  bo.ktile = -1;
  splatt_b200_tensor * whole = nullptr;
  int rc = splatt_b200_tensor_from_csf(tensors, csf_alloc, &bo, &whole);
  // 2. ... cut into equal-nnz shares, moved device to device
  for (int i = 0; i < ndevices && rc == SPLATT_SUCCESS; ++i)
    rc = splatt_b200_tensor_shard(whole, i, ndevices, devices[i], &h->d[i].T);
  if (whole) splatt_b200_tensor_free(whole);
  if (rc == SPLATT_SUCCESS) rc = multi_alloc_buffers(h, verbosity);
  if (rc != SPLATT_SUCCESS) { splatt_b200_multi_free(h); return rc; }
  cudaSetDevice(h->prev_dev);
  if (verbosity > 1)
    printf("SPLATT-B200: %d devices, exchange = %s\n", h->k,
           h->multicast ? "fused NVLink multicast (multimem.red in the MTTKRP kernel)"
                        : (h->k > 1 ? "peer-memory reduce kernel" : "none"));
  *out = h;
  return SPLATT_SUCCESS;
}

int splatt_b200_multi_info(splatt_b200_multi const * h, int * ndevices, int * multicast,
                           uint64_t * nnz_local, uint64_t * device_bytes) {
  if (!h) return SPLATT_ERROR_BADINPUT;
  if (ndevices) *ndevices = h->k;
  if (multicast) *multicast = h->multicast ? 1 : 0;
  for (int i = 0; i < h->k; ++i) {
    uint64_t nl = 0, db = 0;
    splatt_b200_tensor_info(h->d[i].T, nullptr, nullptr, nullptr, &nl, &db);
    if (nnz_local) nnz_local[i] = nl;
    if (device_bytes) device_bytes[i] = db;
  }
  return SPLATT_SUCCESS;
}

// Host-buffer MTTKRP over all devices (what splatt_mttkrp_csf runs when several GPUs are
// configured): factors H2D to every device over its own PCIe link, fused kernel +
// exchange, result D2H as k row slices (one per device, k PCIe links in parallel).
int splatt_b200_multi_mttkrp_host(splatt_b200_multi * h, int mode, double const * const * mats,
                                  double * out_host) {
  if (!h || !mats || !out_host || mode < 0 || mode >= h->N) return SPLATT_ERROR_BADINPUT;
  auto t0 = std::chrono::steady_clock::now();
  const int k = h->k, N = h->N;
  const size_t J = (size_t)h->R, ld = (size_t)h->ldm;
  // pageable caller buffers: one packed copy into page-locked staging serves all k devices
  bool pinned = host_pinned(out_host, h->dims[mode] * J * 8);
  size_t in_doubles = 0;
  for (int m = 0; m < N; ++m)
    if (m != mode) { pinned = pinned && host_pinned(mats[m], h->dims[m] * J * 8); in_doubles += h->dims[m] * J; }
  const double * src[SPB200_MAXN] = {nullptr};
  for (int m = 0; m < N; ++m) src[m] = mats[m];
  if (!pinned) {
    if (in_doubles > h->stage_in_cap) {
      if (h->stage_in) cudaFreeHost(h->stage_in);
      h->stage_in = nullptr; h->stage_in_cap = 0;
      MCK(cudaMallocHost(&h->stage_in, in_doubles * 8));
      h->stage_in_cap = in_doubles;
    }
    if (h->dims[mode] * J > h->stage_out_cap) {
      if (h->stage_out) cudaFreeHost(h->stage_out);
      h->stage_out = nullptr; h->stage_out_cap = 0;
      MCK(cudaMallocHost(&h->stage_out, h->dims[mode] * J * 8));
      h->stage_out_cap = h->dims[mode] * J;
    }
  }
  static int use_pipe = -1;
  if (use_pipe < 0) {
    const char * pe = getenv("SPLATT_B200_PIPELINE");
    use_pipe = (pe && atoi(pe) == 0) ? 0 : 1;
  }
  if (h->multicast && use_pipe && J >= 16) {
    // ---- column-block pipeline over all devices (same idea as dropin.cu:pipelined_call):
    // MTTKRP is independent per column, so the factor columns of block 1 are packed and cross
    // PCIe while the fused kernels run on block 0, and block 0's result slices return while the
    // kernels run on block 1.  Per device: a copy stream for PCIe, the compute stream for the
    // kernels (each with the group barrier in its tail), events between them.
    const int rpad = (int)ld;
    const int half = ((rpad / 2) + 1) & ~1;
    const int cb[3] = {0, half, rpad};
    const uint64_t I = h->dims[mode];
    size_t in_off = 0, out_off[2] = {0, 0};
    int rc = SPLATT_SUCCESS;
    for (int b = 0; b < 2; ++b) {
      const size_t c0 = cb[b], wcols = std::min<size_t>(cb[b + 1], J) - std::min<size_t>(c0, J);
      const double * bsrc[SPB200_MAXN] = {nullptr};
      size_t bpitch[SPB200_MAXN] = {0};
      for (int m = 0; m < N; ++m) {
        if (m == mode || !wcols) continue;
        if (pinned) { bsrc[m] = mats[m] + c0; bpitch[m] = J * 8; continue; }
        double * st = h->stage_in + in_off;              // dense rows x wcols
        const double * from = mats[m] + c0;
        const uint64_t rows = h->dims[m];
#pragma omp parallel for schedule(static) num_threads(kHostTeam)
        for (int64_t r = 0; r < (int64_t)rows; ++r)
          memcpy(st + (size_t)r * wcols, from + (size_t)r * J, wcols * 8);
        bsrc[m] = st; bpitch[m] = wcols * 8;
        in_off += rows * wcols;
      }
      rc = for_each_device_parallel(k, [&](int i) -> int {
        DevState & s = h->d[i];
        MCK(cudaSetDevice(s.dev));
        for (int m = 0; m < N; ++m)
          if (m != mode && wcols)
            MCK(cudaMemcpy2DAsync(s.mats[m] + c0, ld * 8, bsrc[m], bpitch[m], wcols * 8, h->dims[m],
                                  cudaMemcpyHostToDevice, s.copy));
        MCK(cudaEventRecord(s.ev_h2d[b], s.copy));
        return SPLATT_SUCCESS;
      });
      if (rc != SPLATT_SUCCESS) return rc;
    }
    out_off[1] = I * std::min<size_t>(cb[1], J);
    const uint32_t e0 = ++h->epoch, e1 = ++h->epoch;
    rc = for_each_device_parallel(k, [&](int i) -> int {
      DevState & s = h->d[i];
      MCK(cudaSetDevice(s.dev));
      const uint64_t r0 = I * i / k, r1 = I * (i + 1) / k;
      for (int b = 0; b < 2; ++b) {
        const size_t c0 = cb[b], wcols = std::min<size_t>(cb[b + 1], J) - std::min<size_t>(c0, J);
        MCK(cudaStreamWaitEvent(s.stream, s.ev_h2d[b], 0));
        splatt_b200_group_sync gs;
        gs.mc_flag = h->mc_flag; gs.local_flag = s.flag_local; gs.target = b == 0 ? e0 : e1;
        gs.rank = (uint32_t)i; gs.world = (uint32_t)k; gs.reserved = 0;
        const int r = splatt_b200_mttkrp_multicast_sync_columns(s.T, mode, h->R, h->ldm, s.mats,
                                                                h->mc_out[mode], cb[b],
                                                                cb[b + 1] - cb[b], &gs, s.stream);
        if (r != SPLATT_SUCCESS) return r;
        MCK(cudaSetDevice(s.dev));
        MCK(cudaEventRecord(s.ev_kb[b], s.stream));
        MCK(cudaStreamWaitEvent(s.copy, s.ev_kb[b], 0));
        if (r1 > r0 && wcols) {
          if (pinned)
            MCK(cudaMemcpy2DAsync(out_host + r0 * J + c0, J * 8, s.out[mode] + r0 * ld + c0, ld * 8,
                                  wcols * 8, r1 - r0, cudaMemcpyDeviceToHost, s.copy));
          else
            MCK(cudaMemcpy2DAsync(h->stage_out + out_off[b] + r0 * wcols, wcols * 8,
                                  s.out[mode] + r0 * ld + c0, ld * 8, wcols * 8, r1 - r0,
                                  cudaMemcpyDeviceToHost, s.copy));
        }
      }
      // buffer ready for its next use (after the slices have left it)
      MCK(cudaMemsetAsync(s.out[mode], 0, I * ld * 8, s.copy));
      return SPLATT_SUCCESS;
    });
    if (rc != SPLATT_SUCCESS) return rc;
    for (int i = 0; i < k; ++i) {
      MCK(cudaSetDevice(h->d[i].dev));
      MCK(cudaStreamSynchronize(h->d[i].copy));
      MCK(cudaStreamSynchronize(h->d[i].stream));
    }
    if (!pinned) {
      for (int b = 0; b < 2; ++b) {
        const size_t c0 = cb[b], wcols = std::min<size_t>(cb[b + 1], J) - std::min<size_t>(c0, J);
        if (!wcols) continue;
        const double * st = h->stage_out + out_off[b];
        double * to = out_host + c0;
#pragma omp parallel for schedule(static) num_threads(kHostTeam)
        for (int64_t r = 0; r < (int64_t)I; ++r)
          memcpy(to + (size_t)r * J, st + (size_t)r * wcols, wcols * 8);
      }
    }
    cudaSetDevice(h->prev_dev);
    h->last_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return SPLATT_SUCCESS;
  }
  size_t off = 0;
  for (int m = 0; m < N; ++m) {
    if (m == mode) continue;                            // never read (may alias the output)
    if (!pinned) {
      par_memcpy(h->stage_in + off, mats[m], h->dims[m] * J * 8);
      src[m] = h->stage_in + off;
      off += h->dims[m] * J;
    }
    // issue this matrix to every device as soon as it is staged (k PCIe links in parallel,
    // one host thread per device)
    const int rcm = for_each_device_parallel(k, [&](int i) -> int {
      DevState & s = h->d[i];
      cudaError_t e = cudaSetDevice(s.dev);
      if (e == cudaSuccess)
        e = (ld == J) ? cudaMemcpyAsync(s.mats[m], src[m], h->dims[m] * J * 8, cudaMemcpyHostToDevice, s.stream)
                      : cudaMemcpy2DAsync(s.mats[m], ld * 8, src[m], J * 8, J * 8, h->dims[m],
                                          cudaMemcpyHostToDevice, s.stream);
      return e == cudaSuccess ? SPLATT_SUCCESS : SPLATT_ERROR_BADINPUT;
    });
    if (rcm != SPLATT_SUCCESS) return rcm;
  }
  double * dst_host = pinned ? out_host : h->stage_out;
  const uint64_t I = h->dims[mode];
  int rc = SPLATT_SUCCESS;
  auto tail_of_device = [&](int i) -> int {       // result slice back + buffer ready for its next use
    DevState & s = h->d[i];
    MCK(cudaSetDevice(s.dev));
    const uint64_t r0 = I * i / k, r1 = I * (i + 1) / k;
    if (r1 > r0) {
      if (ld == J)
        MCK(cudaMemcpyAsync(dst_host + r0 * J, s.out[mode] + r0 * ld, (r1 - r0) * J * 8,
                            cudaMemcpyDeviceToHost, s.stream));
      else
        MCK(cudaMemcpy2DAsync(dst_host + r0 * J, J * 8, s.out[mode] + r0 * ld, ld * 8, J * 8, r1 - r0,
                              cudaMemcpyDeviceToHost, s.stream));
    }
    return multi_release(h, i, mode);
  };                                              // enqueue only: never block inside the region
                                                  // (a thread may serve several devices)
  if (h->multicast) {
    const uint32_t epoch = ++h->epoch;
    rc = for_each_device_parallel(k, [&](int i) -> int {
      const int r = enqueue_mc_device(h, i, mode, epoch);
      return r == SPLATT_SUCCESS ? tail_of_device(i) : r;
    });
    if (rc != SPLATT_SUCCESS) return rc;
  } else {
    rc = multi_mttkrp_enqueue(h, mode);
    if (rc != SPLATT_SUCCESS) return rc;
    for (int i = 0; i < k; ++i) {
      rc = tail_of_device(i);
      if (rc != SPLATT_SUCCESS) return rc;
    }
  }
  for (int i = 0; i < k; ++i) {
    MCK(cudaSetDevice(h->d[i].dev));
    MCK(cudaStreamSynchronize(h->d[i].stream));
  }
  // (measured: unstaging per device from k threads, or a 32-thread team, is slower than this)
  if (!pinned) par_memcpy(out_host, h->stage_out, I * J * 8);
  cudaSetDevice(h->prev_dev);
  h->last_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  return SPLATT_SUCCESS;
}

// CPD-ALS over all devices: per mode the fused MTTKRP + exchange on every device, then the
// dense tail ONCE -- row-partitioned over the devices when the multicast mapping exists (each
// device solves, normalises and Grams its own row slice and multicasts it; partial norms and
// Grams are summed in device order on every device), otherwise on device 0 (the same kernels
// splatt_cpd_als uses on one GPU), whose new factor every other device pulls over NVLink
// before its next MTTKRP.  Either way the factor matrices
// are single-valued: replicated tails would agree only to rounding (their
// atomics and the multimem.red's arrive in a different order on every GPU) and on
// ill-conditioned problems such replicas drift apart until the shards multiply with
// inconsistent factors (measured: 300^3, 200 K nnz, rank 32 diverges after ~10 iterations).
// The fit and the stop decision also come from device 0, so there is one decision.
// reference: cpd_als_iterate src/cpd.c:271-387 / mpi_cpd_als_iterate src/mpi/mpi_cpd.c:627-804
int splatt_b200_multi_cpd_als(splatt_b200_multi * h, splatt_csf const * tensors,
                              double const * options, splatt_kruskal * factored) {
  if (!h || !tensors || !options || !factored) return SPLATT_ERROR_BADINPUT;
  const int k = h->k, N = h->N, R = h->R, ldm = h->ldm;
  if (R > 128) {
    fprintf(stderr, "SPLATT: multi-GPU CPD-ALS supports rank <= 128\n");
    return SPLATT_ERROR_BADINPUT;
  }
  // multicast available: the tail is ROW-PARTITIONED over the devices (each solves, normalises
  // and Grams its own row slice and multicasts it); otherwise one tail on device 0 + pulls
  const char * pe = getenv("SPLATT_B200_PARTITIONED_TAIL");
  const bool part = h->multicast && !(pe && atoi(pe) == 0);
  HostKruskal K;
  auto fail = [&](int rc) {
    cudaSetDevice(h->prev_dev);
    return rc;
  };
  if (!K.start(N, h->dims, R)) return fail(SPLATT_ERROR_NOMEMORY);
  int rc = SPLATT_SUCCESS;
  for (int i = 0; i < k && rc == SPLATT_SUCCESS; ++i) {
    DevState & s = h->d[i];
    if (cudaSetDevice(s.dev) != cudaSuccess) return fail(SPLATT_ERROR_BADINPUT);
    for (int m = 0; m < N; ++m)
      if (h2d_matrix(s.mats[m], ldm, K.mats[m], h->dims[m], R, s.stream) != cudaSuccess)
        return fail(SPLATT_ERROR_BADINPUT);
    if (i == 0 || part) {
      if (!s.tail) rc = splatt_b200_als_tail_create(N, R, ldm, s.stream, &s.tail);
      if (!part)
        for (int m = 0; m < N && rc == SPLATT_SUCCESS; ++m)
          rc = splatt_b200_als_tail_gram(s.tail, m, s.mats[m], h->dims[m]);
    }
  }
  if (rc != SPLATT_SUCCESS) return fail(rc);
  // one group barrier on every device's stream (multicast path)
  auto group_barrier = [&]() -> int {
    ++h->epoch;
    for (int i = 0; i < k; ++i) {
      DevState & s = h->d[i];
      if (cudaSetDevice(s.dev) != cudaSuccess) return SPLATT_ERROR_BADINPUT;
      k_group_barrier<<<1, 32, 0, s.stream>>>(h->mc_flag, s.flag_local, h->epoch, (uint32_t)i,
                                              (uint32_t)k);
      if (cudaGetLastError() != cudaSuccess) return SPLATT_ERROR_BADINPUT;
      spb200_count_launches(1);
    }
    return SPLATT_SUCCESS;
  };
  auto slice = [&](int m, int i, uint64_t * r0, uint64_t * r1) {
    *r0 = h->dims[m] * (uint64_t)i / k;
    *r1 = h->dims[m] * (uint64_t)(i + 1) / k;
  };
  // SPLATT_B200_MULTI_TIMING=1: synchronise all devices after every phase and report where an
  // iteration's wall time goes (diagnostics; it serialises the phases)
  const char * te = getenv("SPLATT_B200_MULTI_TIMING");
  const bool timing = te && atoi(te) != 0;
  double tphase[5] = {0, 0, 0, 0, 0};
  auto tmark = std::chrono::steady_clock::now();
  auto phase_done = [&](int ph) {
    if (!timing) return;
    for (int i = 0; i < k; ++i) { cudaSetDevice(h->d[i].dev); cudaStreamSynchronize(h->d[i].stream); }
    auto now = std::chrono::steady_clock::now();
    tphase[ph] += std::chrono::duration<double, std::milli>(now - tmark).count();
    tmark = now;
  };
  if (part) {
    // initial Grams: per-device partials of the row slices, summed in device order everywhere
    for (int m = 0; m < N; ++m) {
      for (int i = 0; i < k; ++i) {
        DevState & s = h->d[i];
        uint64_t r0, r1;
        slice(m, i, &r0, &r1);
        if (cudaSetDevice(s.dev) != cudaSuccess) return fail(SPLATT_ERROR_BADINPUT);
        rc = spb200_tail_gram_partial(s.tail, s.mats[m] + r0 * ldm, r1 - r0,
                                      h->mc_grams + (size_t)i * h->gram_stride);
        if (rc != SPLATT_SUCCESS) return fail(rc);
      }
      rc = group_barrier();
      if (rc != SPLATT_SUCCESS) return fail(rc);
      for (int i = 0; i < k; ++i) {
        DevState & s = h->d[i];
        if (cudaSetDevice(s.dev) != cudaSuccess) return fail(SPLATT_ERROR_BADINPUT);
        rc = spb200_tail_finish_gram(s.tail, m, s.grams_local, k, h->gram_stride);
        if (rc != SPLATT_SUCCESS) return fail(rc);
      }
      rc = group_barrier();      // the slots may be overwritten from here on
      if (rc != SPLATT_SUCCESS) return fail(rc);
    }
  }

  const double ttnormsq = spb200_csf_frobsq(tensors);
  AlsIterations iters(options);
  double fit = 0;
  for (uint64_t it = 0; it < iters.niters; ++it) {
    iters.start();
    for (int m = 0; m < N; ++m) {
      if (timing) { phase_done(4); }
      if (!(part && !timing)) {
        rc = multi_mttkrp_enqueue(h, m);
        if (rc != SPLATT_SUCCESS) return fail(rc);
        phase_done(0);
      }
      if (part && !timing) {
        // One host thread per device enqueues the device's whole mode step: fused MTTKRP
        // (barrier e0 in its tail), solve of its row slice + partial column norms -> slot,
        // barrier e1, lambda from all slots, scale + multicast of the slice, partial Gram ->
        // slot, barrier e2, Gram = sum of the slots in device order.  Identical factors, lambda
        // and Grams on every device; the next mode's kernel barrier orders the reads of the
        // slots before their next writes.  Nothing orders the devices on the host.
        const uint32_t e0 = ++h->epoch, e1 = ++h->epoch, e2 = ++h->epoch;
        const int rcp = for_each_device_parallel(k, [&](int i) -> int {
          DevState & s = h->d[i];
          uint64_t r0, r1;
          slice(m, i, &r0, &r1);
          int r = enqueue_mc_device(h, i, m, e0);
          if (r != SPLATT_SUCCESS) return r;
          if (cudaSetDevice(s.dev) != cudaSuccess) return (int)SPLATT_ERROR_BADINPUT;
          r = spb200_tail_solve_norm_partial(s.tail, m, s.out[m] + r0 * ldm, s.mats[m] + r0 * ldm,
                                             r1 - r0, it == 0 ? 1 : 0,
                                             h->mc_norms + (size_t)i * h->norm_stride);
          if (r != SPLATT_SUCCESS) return r;
          k_group_barrier<<<1, 32, 0, s.stream>>>(h->mc_flag, s.flag_local, e1, (uint32_t)i, (uint32_t)k);
          r = spb200_tail_scale_gram_partial(s.tail, s.mats[m] + r0 * ldm, h->mc_mats[m] + r0 * ldm,
                                             r1 - r0, it == 0 ? 1 : 0, s.norms_local, k,
                                             h->norm_stride, h->mc_grams + (size_t)i * h->gram_stride);
          if (r != SPLATT_SUCCESS) return r;
          k_group_barrier<<<1, 32, 0, s.stream>>>(h->mc_flag, s.flag_local, e2, (uint32_t)i, (uint32_t)k);
          spb200_count_launches(2);
          r = spb200_tail_finish_gram(s.tail, m, s.grams_local, k, h->gram_stride);
          if (r != SPLATT_SUCCESS) return r;
          if (!(m == N - 1 && i == 0)) r = multi_release(h, i, m);   // device 0 keeps the last M1 for the fit
          return r;
        });
        if (rcp != SPLATT_SUCCESS) return fail(rcp);
        continue;
      }
      if (part) {
        // the same step, phase by phase from one host thread (SPLATT_B200_MULTI_TIMING)
        for (int i = 0; i < k; ++i) {
          DevState & s = h->d[i];
          uint64_t r0, r1;
          slice(m, i, &r0, &r1);
          if (cudaSetDevice(s.dev) != cudaSuccess) return fail(SPLATT_ERROR_BADINPUT);
          rc = spb200_tail_solve_norm_partial(s.tail, m, s.out[m] + r0 * ldm, s.mats[m] + r0 * ldm,
                                              r1 - r0, it == 0 ? 1 : 0,
                                              h->mc_norms + (size_t)i * h->norm_stride);
          if (rc != SPLATT_SUCCESS) return fail(rc);
        }
        rc = group_barrier();
        if (rc != SPLATT_SUCCESS) return fail(rc);
        phase_done(1);
        for (int i = 0; i < k; ++i) {
          DevState & s = h->d[i];
          uint64_t r0, r1;
          slice(m, i, &r0, &r1);
          if (cudaSetDevice(s.dev) != cudaSuccess) return fail(SPLATT_ERROR_BADINPUT);
          rc = spb200_tail_scale_gram_partial(s.tail, s.mats[m] + r0 * ldm, h->mc_mats[m] + r0 * ldm,
                                              r1 - r0, it == 0 ? 1 : 0, s.norms_local, k,
                                              h->norm_stride, h->mc_grams + (size_t)i * h->gram_stride);
          if (rc != SPLATT_SUCCESS) return fail(rc);
        }
        rc = group_barrier();
        if (rc != SPLATT_SUCCESS) return fail(rc);
        phase_done(2);
        for (int i = 0; i < k; ++i) {
          DevState & s = h->d[i];
          if (cudaSetDevice(s.dev) != cudaSuccess) return fail(SPLATT_ERROR_BADINPUT);
          rc = spb200_tail_finish_gram(s.tail, m, s.grams_local, k, h->gram_stride);
          if (rc != SPLATT_SUCCESS) return fail(rc);
          if (!(m == N - 1 && i == 0)) {        // device 0 still needs the last M1 for the fit
            rc = multi_release(h, i, m);
            if (rc != SPLATT_SUCCESS) return fail(rc);
          }
        }
        phase_done(3);
        continue;
      }
      // device 0: the tail; everybody else: result consumed, wait for the new factor, pull it
      {
        DevState & s0 = h->d[0];
        if (cudaSetDevice(s0.dev) != cudaSuccess) return fail(SPLATT_ERROR_BADINPUT);
        rc = splatt_b200_als_tail_update(s0.tail, m, s0.out[m], s0.mats[m], h->dims[m], it == 0 ? 1 : 0);
        if (rc != SPLATT_SUCCESS) return fail(rc);
        if (cudaEventRecord(s0.ev_tail, s0.stream) != cudaSuccess) return fail(SPLATT_ERROR_BADINPUT);
        if (m != N - 1) {                        // the last M1 is still needed for the fit
          rc = multi_release(h, 0, m);
          if (rc != SPLATT_SUCCESS) return fail(rc);
        }
      }
      for (int i = 1; i < k; ++i) {
        DevState & s = h->d[i];
        if (cudaSetDevice(s.dev) != cudaSuccess) return fail(SPLATT_ERROR_BADINPUT);
        rc = multi_release(h, i, m);
        if (rc != SPLATT_SUCCESS) return fail(rc);
        // device 0 overwrites this factor again only one iteration later, after N-1 more
        // group exchanges that this device takes part in AFTER the copy below (stream order)
        const size_t bytes = h->dims[m] * (size_t)ldm * 8;
        cudaError_t e = cudaStreamWaitEvent(s.stream, h->d[0].ev_tail, 0);
        if (e == cudaSuccess)
          e = (s.dev == h->d[0].dev)
                  ? cudaMemcpyAsync(s.mats[m], h->d[0].mats[m], bytes, cudaMemcpyDeviceToDevice, s.stream)
                  : cudaMemcpyPeerAsync(s.mats[m], s.dev, h->d[0].mats[m], h->d[0].dev, bytes, s.stream);
        if (e != cudaSuccess) return fail(SPLATT_ERROR_BADINPUT);
      }
    }
    if (cudaSetDevice(h->d[0].dev) != cudaSuccess) return fail(SPLATT_ERROR_BADINPUT);
    rc = splatt_b200_als_tail_fit(h->d[0].tail, h->d[0].mats[N - 1], h->d[0].out[N - 1],
                                  h->dims[N - 1], ttnormsq, &fit, K.lambda);
    if (rc != SPLATT_SUCCESS) return fail(rc);
    rc = multi_release(h, 0, N - 1);
    if (rc != SPLATT_SUCCESS) return fail(rc);
    if (iters.done(it, fit)) break;
  }
  if (timing)
    printf("SPLATT-B200: multi CPD phases (ms, all iterations): mttkrp %.2f | solve+norm %.2f | "
           "scale+gram %.2f | gram sum+release %.2f | fit/other %.2f\n",
           tphase[0], tphase[1], tphase[2], tphase[3], tphase[4]);
  // factors back from device 0 (every device holds the same bits)
  {
    DevState & s = h->d[0];
    if (cudaSetDevice(s.dev) != cudaSuccess) return fail(SPLATT_ERROR_BADINPUT);
    for (int m = 0; m < N; ++m)
      if (d2h_matrix(K.mats[m], s.mats[m], ldm, h->dims[m], R, s.stream) != cudaSuccess)
        return fail(SPLATT_ERROR_BADINPUT);
  }
  for (int i = 0; i < k; ++i) {
    cudaSetDevice(h->d[i].dev);
    if (cudaStreamSynchronize(h->d[i].stream) != cudaSuccess) return fail(SPLATT_ERROR_BADINPUT);
  }
  cudaSetDevice(h->prev_dev);
  K.finish(fit, factored);     // post-process (src/cpd.c:391-411)
  return SPLATT_SUCCESS;
}

double splatt_b200_multi_last_ms(splatt_b200_multi const * h) { return h ? h->last_ms : 0.0; }

}  // extern "C"
