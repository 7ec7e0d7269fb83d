// Drop-in symbols (include/splatt_b200.h, group 1): host-buffer wrappers with the
// reference's names and semantics around the device engine.
#include "common.h"
#include <cfloat>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <chrono>
#include <algorithm>
#include <mutex>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

void spb200_mode_csf_map(int N, int csf_alloc, const int perm0[SPB200_MAXN], int * map);

namespace {

constexpr uint64_t kWsMagic = 0x53504232303057ull;   // "SPB200W"

// Private workspace: the public struct first (callers only hold a pointer to it,
// reference: src/cpd.c:304, src/mttkrp.c:1796), engine state behind it.
struct WsPriv {
  splatt_mttkrp_ws pub;
  uint64_t magic;
  splatt_b200_tensor * T;
  splatt_b200_multi * multi;     // several GPUs configured (SPLATT_B200_NGPUS / _DEVICES): multi.cu
  int N;
  uint64_t dims[SPB200_MAXN];
  int ncolumns;
  int ldm;
  double * d_mats[SPB200_MAXN];
  double * d_out;
  uint64_t out_rows_cap;
  cudaStream_t stream;
  cudaStream_t copy_stream;       // PCIe copies of the column-block pipeline
  cudaEvent_t ev_h2d[2], ev_k[2];
  double last_ms;
  // SPLATT_B200_PIN=1: caller buffers seen by splatt_mttkrp_csf are page-locked on first
  // sight (cudaHostRegister) so the H2D/D2H copies run at full PCIe rate; released in
  // splatt_mttkrp_free_ws.  Opt-in because it assumes the buffers outlive the workspace
  // (true for the reference's CPD driver, src/cpd.c:304-379).
  bool pin;
  int npinned;
  void * pinned[4 * SPB200_MAXN];
  size_t pinned_bytes[4 * SPB200_MAXN];
  // Pageable caller buffers (the reference's splatt_malloc memory): copies are staged through
  // page-locked bounce buffers owned by the workspace, filled / drained by a few host threads,
  // so that the PCIe copies stay asynchronous and the column-block pipeline still overlaps.
  double * stage_in;  size_t stage_in_cap;     // doubles
  double * stage_out; size_t stage_out_cap;
  cudaEvent_t ev_d2h[2];
};

int layout_from_env() {
  const char * e = getenv("SPLATT_B200_LAYOUT");
  if (e && (!strcmp(e, "asgiven") || !strcmp(e, "ASGIVEN") || !strcmp(e, "1")))
    return SPLATT_B200_LAYOUT_ASGIVEN;
  return SPLATT_B200_LAYOUT_ALLROOT;
}

void pin_once(WsPriv * w, void * p, size_t bytes) {
  if (!w->pin || !p) return;
  for (int i = 0; i < w->npinned; ++i)
    if (w->pinned[i] == p) {
      if (w->pinned_bytes[i] >= bytes) return;
      // the same buffer seen with a larger extent (the reference's CPD driver reuses one
      // maxdim x J output for every mode, src/cpd.c:322-327): register the larger range
      cudaHostUnregister(p);
      if (cudaHostRegister(p, bytes, cudaHostRegisterDefault) == cudaSuccess) w->pinned_bytes[i] = bytes;
      else { cudaGetLastError(); w->pinned[i] = w->pinned[--w->npinned]; w->pinned_bytes[i] = w->pinned_bytes[w->npinned]; }
      return;
    }
  if (w->npinned >= 4 * SPB200_MAXN) return;
  if (cudaHostRegister(p, bytes, cudaHostRegisterDefault) == cudaSuccess) {
    w->pinned[w->npinned] = p;
    w->pinned_bytes[w->npinned++] = bytes;
  } else {
    cudaGetLastError();   // already pinned / not registrable: copy works either way
  }
}

void free_priv(WsPriv * w) {
  if (!w) return;
  for (int i = 0; i < w->npinned; ++i) cudaHostUnregister(w->pinned[i]);
  for (int m = 0; m < SPB200_MAXN; ++m)
    if (w->d_mats[m]) cudaFree(w->d_mats[m]);
  if (w->d_out) cudaFree(w->d_out);
  if (w->stream) cudaStreamDestroy(w->stream);
  if (w->copy_stream) cudaStreamDestroy(w->copy_stream);
  for (int i = 0; i < 2; ++i) {
    if (w->ev_h2d[i]) cudaEventDestroy(w->ev_h2d[i]);
    if (w->ev_k[i]) cudaEventDestroy(w->ev_k[i]);
    if (w->ev_d2h[i]) cudaEventDestroy(w->ev_d2h[i]);
  }
  if (w->stage_in) cudaFreeHost(w->stage_in);
  if (w->stage_out) cudaFreeHost(w->stage_out);
  if (w->T) splatt_b200_tensor_free(w->T);
  if (w->multi) splatt_b200_multi_free(w->multi);
  w->magic = 0;
  free(w);
}

bool is_pinned(const void * p, size_t bytes) {
  // both ends of the range must be page-locked host memory
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

int stage_threads() {
  static int v = 0;
  if (v == 0) {
    const char * e = getenv("SPLATT_B200_STAGE_THREADS");
    v = e ? atoi(e) : 16;
    if (v < 1) v = 1;
    if (v > 64) v = 64;
  }
  return v;
}

// rows x wcols block of a row-major (ld_src) matrix -> dense rows x wcols, and back
void pack_cols(double * dst, const double * src, uint64_t rows, size_t ld_src, size_t wcols) {
#pragma omp parallel for schedule(static) num_threads(stage_threads())
  for (int64_t i = 0; i < (int64_t)rows; ++i)
    memcpy(dst + (size_t)i * wcols, src + (size_t)i * ld_src, wcols * sizeof(double));
}
void unpack_cols(double * dst, size_t ld_dst, const double * src, uint64_t rows, size_t wcols) {
#pragma omp parallel for schedule(static) num_threads(stage_threads())
  for (int64_t i = 0; i < (int64_t)rows; ++i)
    memcpy(dst + (size_t)i * ld_dst, src + (size_t)i * wcols, wcols * sizeof(double));
}

bool ensure_stage(WsPriv * w, size_t in_doubles, size_t out_doubles) {
  if (in_doubles > w->stage_in_cap) {
    if (w->stage_in) cudaFreeHost(w->stage_in);
    w->stage_in = nullptr; w->stage_in_cap = 0;
    if (cudaMallocHost(&w->stage_in, in_doubles * 8) != cudaSuccess) { cudaGetLastError(); return false; }
    w->stage_in_cap = in_doubles;
  }
  if (out_doubles > w->stage_out_cap) {
    if (w->stage_out) cudaFreeHost(w->stage_out);
    w->stage_out = nullptr; w->stage_out_cap = 0;
    if (cudaMallocHost(&w->stage_out, out_doubles * 8) != cudaSuccess) { cudaGetLastError(); return false; }
    w->stage_out_cap = out_doubles;
  }
  return true;
}

// Column-block pipeline: MTTKRP is independent per column, so the factor columns of block 1
// cross PCIe while the kernel runs on block 0, and block 0's result goes back while the
// kernel runs on block 1.
//   host (staged): pack blk0 | pack blk1 |                      unpack blk0 | unpack blk1
//   copy stream  :      H2D blk0 | H2D blk1 |        D2H blk0 |          D2H blk1
//   kernel stream:                kernel blk0        | kernel blk1
// `staged`: the caller's buffers are pageable -- go through the workspace's page-locked
// bounce buffers (packed per column block); otherwise DMA straight from/to the caller.
cudaError_t pipelined_call(WsPriv * w, splatt_b200_matrix_t ** mats, int mode, uint64_t J,
                           int nblocks, bool staged, int * rc) {
  const int N = w->N;
  const int rpad = w->ldm;
  const int half = ((rpad / 2) + 1) & ~1;                 // even split point
  int cb[3] = {0, half, rpad};
  if (nblocks == 1) { cb[1] = rpad; cb[2] = rpad; }
  splatt_b200_matrix_t * M = mats[SPLATT_B200_MAX_NMODES];
  size_t in_rows = 0;
  for (int m = 0; m < N; ++m) if (m != mode) in_rows += w->dims[m];
  if (staged && !ensure_stage(w, in_rows * J, w->dims[mode] * J)) return cudaErrorMemoryAllocation;
  cudaError_t e = cudaSuccess;
  size_t in_off = 0;
  for (int b = 0; b < nblocks && e == cudaSuccess; ++b) {
    const size_t c0 = cb[b], wcols = std::min<size_t>(cb[b + 1], J) - std::min<size_t>(c0, J);
    for (int m = 0; m < N && e == cudaSuccess && wcols; ++m) {
      if (m == mode) continue;
      const double * src = mats[m]->vals + c0;
      size_t spitch = J * 8;
      if (staged) {
        double * st = w->stage_in + in_off;
        pack_cols(st, src, w->dims[m], J, wcols);
        in_off += w->dims[m] * wcols;
        src = st;
        spitch = wcols * 8;
      }
      e = cudaMemcpy2DAsync(w->d_mats[m] + c0, (size_t)w->ldm * 8, src, spitch, wcols * 8,
                            w->dims[m], cudaMemcpyHostToDevice, w->copy_stream);
    }
    if (e == cudaSuccess) e = cudaEventRecord(w->ev_h2d[b], w->copy_stream);
  }
  for (int b = 0; b < nblocks && e == cudaSuccess; ++b) {
    e = cudaStreamWaitEvent(w->stream, w->ev_h2d[b], 0);
    if (e != cudaSuccess) break;
    *rc = splatt_b200_mttkrp_columns(w->T, mode, w->ncolumns, w->ldm, w->d_mats, w->d_out, cb[b],
                                     cb[b + 1] - cb[b], w->stream);
    if (*rc != SPLATT_SUCCESS) return cudaSuccess;
    e = cudaEventRecord(w->ev_k[b], w->stream);
  }
  size_t out_off[2] = {0, 0};
  for (int b = 0; b < nblocks && e == cudaSuccess; ++b) {
    const size_t c0 = cb[b], wcols = std::min<size_t>(cb[b + 1], J) - std::min<size_t>(c0, J);
    e = cudaStreamWaitEvent(w->copy_stream, w->ev_k[b], 0);
    if (b == 1) out_off[1] = w->dims[mode] * (std::min<size_t>(cb[1], J));
    if (e == cudaSuccess && wcols) {
      if (staged)
        e = cudaMemcpy2DAsync(w->stage_out + out_off[b], wcols * 8, w->d_out + c0, (size_t)w->ldm * 8,
                              wcols * 8, w->dims[mode], cudaMemcpyDeviceToHost, w->copy_stream);
      else
        e = cudaMemcpy2DAsync(M->vals + c0, J * 8, w->d_out + c0, (size_t)w->ldm * 8, wcols * 8,
                              w->dims[mode], cudaMemcpyDeviceToHost, w->copy_stream);
    }
    if (e == cudaSuccess) e = cudaEventRecord(w->ev_d2h[b], w->copy_stream);
  }
  if (staged) {
    for (int b = 0; b < nblocks && e == cudaSuccess; ++b) {
      const size_t c0 = cb[b], wcols = std::min<size_t>(cb[b + 1], J) - std::min<size_t>(c0, J);
      e = cudaEventSynchronize(w->ev_d2h[b]);
      if (e == cudaSuccess && wcols)
        unpack_cols(M->vals + c0, J, w->stage_out + out_off[b], w->dims[mode], wcols);
    }
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(w->copy_stream);
  return e;
}

// ---------------------------------------------------------------------------
// Device-mirror cache of the bare splatt_mttkrp entry point.  The reference pays an
// O(nslices) workspace build per call (src/mttkrp.c:1796); a per-call device mirror would
// cost the CSF expansion, the upload of the whole tensor and one radix sort per stream.  So
// workspaces built by splatt_mttkrp are kept (LRU, SPLATT_B200_CACHE entries, default 2,
// 0 = off) and found again by (tensors, policy, rank, shape, array addresses) plus a content
// fingerprint of the first CSF -- a tensor freed and another one allocated at the same
// addresses does not match.  matlab/splatt_mttkrp.c:47-68 is the caller this serves.
// ---------------------------------------------------------------------------
struct MirrorKey {
  const void * tensors;
  const void * pt0;
  const void * vals0;
  uint64_t nnz, fingerprint;
  uint64_t dims[SPB200_MAXN];
  int nmodes, csf_alloc, ncolumns, layout, ndev, devs[16];
  bool operator==(const MirrorKey & o) const { return memcmp(this, &o, sizeof(MirrorKey)) == 0; }
};
struct MirrorEntry { MirrorKey key; splatt_mttkrp_ws * ws; uint64_t stamp; };
std::mutex g_mirror_mu;
std::vector<MirrorEntry> g_mirror;
uint64_t g_mirror_stamp = 0;

int mirror_cap() {
  const char * e = getenv("SPLATT_B200_CACHE");
  const int v = e ? atoi(e) : 2;
  return v < 0 ? 0 : (v > 64 ? 64 : v);
}

uint64_t fnv(uint64_t h, const void * p, size_t n) {
  const unsigned char * b = static_cast<const unsigned char *>(p);
  for (size_t i = 0; i < n; ++i) { h ^= b[i]; h *= 1099511628211ull; }
  return h;
}

MirrorKey mirror_key(const splatt_csf * tensors, int csf_alloc, int ncolumns) {
  MirrorKey k;
  memset(&k, 0, sizeof(k));
  const splatt_csf & t = tensors[0];
  const int N = (int)t.nmodes;
  k.tensors = tensors;
  k.pt0 = t.pt;
  k.vals0 = t.pt ? t.pt[0].vals : nullptr;
  k.nnz = t.nnz;
  k.nmodes = N;
  k.csf_alloc = csf_alloc;
  k.ncolumns = ncolumns;
  k.layout = layout_from_env();
  for (int m = 0; m < N; ++m) k.dims[m] = t.dims[m];
  k.ndev = splatt_b200_multi_env_devices(k.devs, 16);
  // content fingerprint: shape of the tree + strided samples of values and leaf indices
  uint64_t h = 1469598103934665603ull;
  h = fnv(h, &t.ntiles, sizeof(t.ntiles));
  h = fnv(h, t.dim_perm, sizeof(t.dim_perm[0]) * N);
  for (uint64_t tile = 0; tile < t.ntiles && tile < 64; ++tile) {
    const csf_sparsity & pt = t.pt[tile];
    h = fnv(h, pt.nfibs, sizeof(pt.nfibs[0]) * N);
    const uint64_t n = pt.vals ? pt.nfibs[N - 1] : 0;
    const uint64_t step = n > 2048 ? n / 2048 : 1;
    for (uint64_t i = 0; i < n; i += step) {
      h = fnv(h, &pt.vals[i], sizeof(double));
      if (pt.fids[N - 1]) h = fnv(h, &pt.fids[N - 1][i], sizeof(splatt_idx_t));
    }
    if (n) h = fnv(h, &pt.vals[n - 1], sizeof(double));
  }
  k.fingerprint = h;
  return k;
}

}  // namespace

extern "C" {

void splatt_b200_cache_clear(void) {
  std::lock_guard<std::mutex> lk(g_mirror_mu);
  for (auto & e : g_mirror) splatt_mttkrp_free_ws(e.ws);
  g_mirror.clear();
}

splatt_mttkrp_ws * splatt_mttkrp_alloc_ws(splatt_csf const * const tensors,
                                          splatt_idx_t const ncolumns,
                                          double const * const opts) {
  if (!tensors || !opts || ncolumns == 0) {
    fprintf(stderr, "SPLATT: splatt_mttkrp_alloc_ws: bad arguments\n");
    return nullptr;
  }
  const int csf_alloc = (int)opts[SPLATT_OPTION_CSF_ALLOC];
  if (csf_alloc < SPLATT_CSF_ONEMODE || csf_alloc > SPLATT_CSF_ALLMODE) {
    // reference: src/mttkrp.c:1856-1858
    fprintf(stderr, "SPLATT: CSF type '%d' not recognized.\n", csf_alloc);
    abort();
  }
  WsPriv * w = static_cast<WsPriv *>(calloc(1, sizeof(WsPriv)));
  if (!w) return nullptr;
  w->magic = kWsMagic;
  {
    const char * e = getenv("SPLATT_B200_PIN");
    w->pin = e && atoi(e) != 0;
  }
  const int N = (int)tensors[0].nmodes;
  w->N = N;
  for (int m = 0; m < N; ++m) w->dims[m] = tensors[0].dims[m];

  // public, CPU-facing fields (reference: src/mttkrp.c:1822-1880)
  w->pub.num_threads = (splatt_idx_t)opts[SPLATT_OPTION_NTHREADS];
  int perm0[SPB200_MAXN], map[SPB200_MAXN];
  for (int l = 0; l < N; ++l) perm0[l] = (int)tensors[0].dim_perm[l];
  spb200_mode_csf_map(N, csf_alloc, perm0, map);
  for (int m = 0; m < N; ++m) w->pub.mode_csf_map[m] = (splatt_idx_t)map[m];
  w->pub.num_csf = csf_alloc == SPLATT_CSF_ONEMODE ? 1 : (csf_alloc == SPLATT_CSF_TWOMODE ? 2 : N);
  w->pub.privatize_buffer = nullptr;
  w->pub.reduction_time = 0.;

  w->ncolumns = (int)ncolumns;
  w->ldm = (int)(ncolumns + (ncolumns & 1));
  {
    int devs[16];
    const int nd = splatt_b200_multi_env_devices(devs, 16);
    if (nd > 1) {
      // one process, several GPUs: shards + fused exchange live in the multi engine
      if (splatt_b200_multi_create(tensors, csf_alloc, (int)ncolumns, devs, nd,
                                   (int)opts[SPLATT_OPTION_VERBOSITY], &w->multi) != SPLATT_SUCCESS) {
        free_priv(w);
        return nullptr;
      }
      return &w->pub;
    }
  }
  splatt_b200_build_opts bo;
  memset(&bo, 0, sizeof(bo));
  bo.layout = layout_from_env();
  bo.device = -1;
  bo.verbosity = (int)opts[SPLATT_OPTION_VERBOSITY];
  // untiled streams: the copy/compute pipeline launches column blocks, and the tiled kernel
  // re-walks every record per block (measured slower on config 2 with page-locked buffers)
  bo.ktile = -1;
  if (splatt_b200_tensor_from_csf(tensors, csf_alloc, &bo, &w->T) != SPLATT_SUCCESS) {
    free_priv(w);
    return nullptr;
  }
  w->ncolumns = (int)ncolumns;
  w->ldm = (int)(ncolumns + (ncolumns & 1));
  uint64_t maxdim = 0;
  bool ok = true;
  for (int m = 0; m < N && ok; ++m) {
    maxdim = w->dims[m] > maxdim ? w->dims[m] : maxdim;
    ok = cudaMalloc(&w->d_mats[m], w->dims[m] * (size_t)w->ldm * 8) == cudaSuccess &&
         cudaMemset(w->d_mats[m], 0, w->dims[m] * (size_t)w->ldm * 8) == cudaSuccess;
  }
  w->out_rows_cap = maxdim;
  ok = ok && cudaMalloc(&w->d_out, maxdim * (size_t)w->ldm * 8) == cudaSuccess;
  ok = ok && cudaStreamCreateWithFlags(&w->stream, cudaStreamNonBlocking) == cudaSuccess;
  ok = ok && cudaStreamCreateWithFlags(&w->copy_stream, cudaStreamNonBlocking) == cudaSuccess;
  for (int i = 0; i < 2 && ok; ++i)
    ok = cudaEventCreateWithFlags(&w->ev_h2d[i], cudaEventDisableTiming) == cudaSuccess &&
         cudaEventCreateWithFlags(&w->ev_k[i], cudaEventDisableTiming) == cudaSuccess &&
         cudaEventCreateWithFlags(&w->ev_d2h[i], cudaEventDisableTiming) == cudaSuccess;
  if (!ok) {
    fprintf(stderr, "SPLATT: out of device memory for MTTKRP workspace (%s)\n",
            cudaGetErrorString(cudaGetLastError()));
    free_priv(w);
    return nullptr;
  }
  return &w->pub;
}

void splatt_mttkrp_free_ws(splatt_mttkrp_ws * const ws) {
  if (!ws) return;
  WsPriv * w = reinterpret_cast<WsPriv *>(ws);
  if (w->magic != kWsMagic) {
    fprintf(stderr, "SPLATT: splatt_mttkrp_free_ws: workspace was not allocated by "
                    "libsplatt_b200\n");
    return;
  }
  free_priv(w);
}

void splatt_mttkrp_csf(splatt_csf const * const tensors, splatt_b200_matrix_t ** mats,
                       splatt_idx_t const mode, void * const thds, splatt_mttkrp_ws * const ws,
                       double const * const opts) {
  (void)thds;
  WsPriv * w = reinterpret_cast<WsPriv *>(ws);
  if (!w || w->magic != kWsMagic || !mats || (int)mode >= w->N) {
    // the reference has no error channel here; fatal like src/mttkrp.c:1857
    fprintf(stderr, "SPLATT: splatt_mttkrp_csf: workspace not created by libsplatt_b200 "
                    "or bad mode\n");
    abort();
  }
  const int N = w->N;
  splatt_b200_matrix_t * M = mats[SPLATT_B200_MAX_NMODES];
  M->I = tensors[0].dims[mode];                       // reference: src/mttkrp.c:1303-1305
  const uint64_t J = M->J;
  if ((int)J != w->ncolumns) {
    fprintf(stderr, "SPLATT: splatt_mttkrp_csf: workspace built for %d columns, got %llu\n",
            w->ncolumns, (unsigned long long)J);
    abort();
  }
  auto t0 = std::chrono::steady_clock::now();
  cudaError_t e = cudaSuccess;
  int rc = SPLATT_SUCCESS;
  bool all_pinned = true;
  for (int m = 0; m < N; ++m) {
    if (m == (int)mode) continue;                      // never read (may alias the output)
    pin_once(w, mats[m]->vals, w->dims[m] * J * sizeof(double));
    all_pinned = all_pinned && is_pinned(mats[m]->vals, w->dims[m] * J * sizeof(double));
  }
  pin_once(w, M->vals, w->dims[mode] * J * sizeof(double));
  all_pinned = all_pinned && is_pinned(M->vals, w->dims[mode] * J * sizeof(double));
  if (w->multi) {
    const double * hm[SPB200_MAXN] = {nullptr};
    for (int m = 0; m < N; ++m) hm[m] = (m == (int)mode) ? nullptr : mats[m]->vals;
    if (splatt_b200_multi_mttkrp_host(w->multi, (int)mode, hm, M->vals) != SPLATT_SUCCESS) {
      fprintf(stderr, "SPLATT: multi-GPU MTTKRP failed\n");
      abort();
    }
    w->last_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (opts && (int)opts[SPLATT_OPTION_VERBOSITY] == SPLATT_VERBOSITY_MAX)
      printf("MTTKRP mode %llu: %0.6fs (B200 x N, host buffers)\n", (unsigned long long)mode + 1,
             w->last_ms * 1e-3);
    return;
  }
  static int use_pipe = -1, use_stage = -1;
  if (use_pipe < 0) {
    const char * pe = getenv("SPLATT_B200_PIPELINE");
    use_pipe = (pe && atoi(pe) == 0) ? 0 : 1;
    const char * se = getenv("SPLATT_B200_STAGE");
    use_stage = (se && atoi(se) == 0) ? 0 : 1;
  }
  if (all_pinned || use_stage) {
    // narrow matrices: one block is enough
    e = pipelined_call(w, mats, (int)mode, J, (J >= 16 && use_pipe) ? 2 : 1, !all_pinned, &rc);
  } else {
    for (int m = 0; m < N && e == cudaSuccess; ++m) {
      if (m == (int)mode) continue;
      e = h2d_matrix(w->d_mats[m], w->ldm, mats[m]->vals, w->dims[m], J, w->stream);
    }
    if (e == cudaSuccess)
      rc = splatt_b200_mttkrp(w->T, (int)mode, w->ncolumns, w->ldm, w->d_mats, w->d_out, w->stream);
    if (e == cudaSuccess && rc == SPLATT_SUCCESS)
      e = d2h_matrix(M->vals, w->d_out, w->ldm, w->dims[mode], J, w->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(w->stream);
  }
  if (e != cudaSuccess || rc != SPLATT_SUCCESS) {
    fprintf(stderr, "SPLATT: GPU MTTKRP failed (%s)\n", cudaGetErrorString(e));
    abort();
  }
  w->last_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  if (opts && (int)opts[SPLATT_OPTION_VERBOSITY] == SPLATT_VERBOSITY_MAX) {
    // counterpart of the per-thread time report, reference: src/mttkrp.c:1333-1339
    printf("MTTKRP mode %llu: %0.6fs (B200, host buffers)\n", (unsigned long long)mode + 1,
           w->last_ms * 1e-3);
  }
}

int splatt_mttkrp(splatt_idx_t const mode, splatt_idx_t const ncolumns,
                  splatt_csf const * const tensors, splatt_val_t ** matrices,
                  splatt_val_t * const matout, double const * const options) {
  if (!tensors || !matrices || !matout || !options || ncolumns == 0 ||
      mode >= tensors[0].nmodes) {
    fprintf(stderr, "SPLATT: splatt_mttkrp: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  const int N = (int)tensors[0].nmodes;
  // the device mirror of a tensor seen before is reused (see MirrorKey above)
  const int cap = mirror_cap();
  std::unique_lock<std::mutex> lk(g_mirror_mu, std::defer_lock);
  splatt_mttkrp_ws * ws = nullptr;
  if (cap > 0) {
    lk.lock();                       // also serialises calls that share a cached workspace
    const MirrorKey key = mirror_key(tensors, (int)options[SPLATT_OPTION_CSF_ALLOC], (int)ncolumns);
    for (auto & e : g_mirror)
      if (e.key == key) { ws = e.ws; e.stamp = ++g_mirror_stamp; break; }
    if (!ws) {
      ws = splatt_mttkrp_alloc_ws(tensors, ncolumns, options);
      if (!ws) return SPLATT_ERROR_NOMEMORY;
      if ((int)g_mirror.size() >= cap) {
        size_t lru = 0;
        for (size_t i = 1; i < g_mirror.size(); ++i)
          if (g_mirror[i].stamp < g_mirror[lru].stamp) lru = i;
        splatt_mttkrp_free_ws(g_mirror[lru].ws);
        g_mirror.erase(g_mirror.begin() + lru);
      }
      g_mirror.push_back(MirrorEntry{key, ws, ++g_mirror_stamp});
    }
  } else {
    ws = splatt_mttkrp_alloc_ws(tensors, ncolumns, options);
    if (!ws) return SPLATT_ERROR_NOMEMORY;
  }
  // same wrapping as the reference (src/mttkrp.c:1773-1786)
  splatt_b200_matrix_t store[SPLATT_B200_MAX_NMODES + 1];
  splatt_b200_matrix_t * mats[SPLATT_B200_MAX_NMODES + 1] = {nullptr};
  for (int m = 0; m < N; ++m) {
    store[m].I = tensors[0].dims[m];
    store[m].J = ncolumns;
    store[m].rowmajor = 1;
    store[m].vals = matrices[m];
    mats[m] = &store[m];
  }
  store[SPLATT_B200_MAX_NMODES].I = tensors[0].dims[mode];
  store[SPLATT_B200_MAX_NMODES].J = ncolumns;
  store[SPLATT_B200_MAX_NMODES].rowmajor = 1;
  store[SPLATT_B200_MAX_NMODES].vals = matout;
  mats[SPLATT_B200_MAX_NMODES] = &store[SPLATT_B200_MAX_NMODES];
  splatt_mttkrp_csf(tensors, mats, mode, nullptr, ws, options);
  if (cap == 0) splatt_mttkrp_free_ws(ws);
  return SPLATT_SUCCESS;
}

double * splatt_default_opts(void) {
  // reference: src/opts.c:10-47 (SPLATT_VAL_OFF = -DBL_MAX, include/splatt/constants.h)
  double * opts = static_cast<double *>(malloc(SPLATT_OPTION_NOPTIONS * sizeof(double)));
  if (!opts) return nullptr;
  for (int i = 0; i < SPLATT_OPTION_NOPTIONS; ++i) opts[i] = -DBL_MAX;
  opts[SPLATT_OPTION_TOLERANCE]  = 1e-5;
  opts[SPLATT_OPTION_REGULARIZE] = 0.;
  opts[SPLATT_OPTION_NITER]      = 50;
  opts[SPLATT_OPTION_VERBOSITY]  = SPLATT_VERBOSITY_LOW;
  opts[SPLATT_OPTION_CSF_ALLOC]  = SPLATT_CSF_TWOMODE;
  opts[SPLATT_OPTION_TILE]       = SPLATT_NOTILE;
  opts[SPLATT_OPTION_PRIVTHRESH] = 0.02;
  opts[SPLATT_OPTION_TILELEVEL]  = 1;
  opts[SPLATT_OPTION_DECOMP]     = 1;   /* SPLATT_DECOMP_MEDIUM */
  opts[SPLATT_OPTION_COMM]       = 1;   /* SPLATT_COMM_ALL2ALL  */
  opts[SPLATT_OPTION_RANDSEED]   = (double)time(nullptr);
#ifdef _OPENMP
  opts[SPLATT_OPTION_NTHREADS] = omp_in_parallel() ? 1 : omp_get_max_threads();
#else
  opts[SPLATT_OPTION_NTHREADS] = 1;
#endif
  return opts;
}

void splatt_free_opts(double * opts) { free(opts); }

}  // extern "C"
