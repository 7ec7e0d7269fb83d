// Device-side construction of fiber streams (and of reference-shaped CSF arrays)
// from coordinate data.
//
// Reference semantics followed (not code): tt_sort orders nonzeros
// lexicographically by the level permutation (src/sort.c:912-918 via
// src/csf.c:475); p_mk_outerptr / p_mk_fptr start a new node at level l wherever
// the index at any level <= l changes (src/csf.c:248-458).  Here the same rule
// is evaluated per nonzero as "first differing level" dl[n], and everything else
// (node numbering, fids, fptr, close counts) follows from prefix sums over
// dl[n] <= l.  Sorting and scans use CUB (one-time set-up, not the hot path).
#include "common.h"
#include <cub/cub.cuh>
#include <algorithm>
#include <cstring>
#include <cstdlib>

namespace {

struct DevBuf {
  void * p = nullptr;
  size_t bytes = 0;
  ~DevBuf() { if (p) cudaFree(p); }
  cudaError_t alloc(size_t b) {
    if (p) { cudaFree(p); p = nullptr; }
    bytes = b;
    return cudaMalloc(&p, b ? b : 16);
  }
  template <class T> T * as() { return static_cast<T *>(p); }
  void * release() { void * r = p; p = nullptr; return r; }
};

int bits_for(uint64_t dim) {
  int b = 1;
  while (b < 64 && (1ull << b) < dim) ++b;
  return b;
}

struct KeySpec {
  const uint32_t * src[SPB200_MAXN];
  int shift[SPB200_MAXN];
  int n;
};

__global__ void k_iota(uint32_t * o, uint64_t n) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) o[i] = (uint32_t)i;
}

__global__ void k_make_keys(KeySpec ks, const uint32_t * __restrict__ order, uint64_t n,
                            uint64_t * __restrict__ keys) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t o = order[i];
  uint64_t k = 0;
  for (int j = 0; j < ks.n; ++j) k |= (uint64_t)ks.src[j][o] << ks.shift[j];
  keys[i] = k;
}

__global__ void k_gather_u32(const uint32_t * __restrict__ src, const uint32_t * __restrict__ order,
                             uint64_t n, uint32_t * __restrict__ dst) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) dst[i] = order ? src[order[i]] : src[i];
}

struct LevelPtrs { const uint32_t * s[SPB200_MAXN]; };

// dl[n] = first level at which nonzero n differs from n-1 (0 for n == 0,
// N if all coordinates are equal).
__global__ void k_first_diff(LevelPtrs lp, int N, uint64_t n, uint8_t * __restrict__ dl) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int d = 0;
  if (i > 0) {
    d = N;
    for (int l = 0; l < N; ++l)
      if (lp.s[l][i] != lp.s[l][i - 1]) { d = l; break; }
  }
  dl[i] = (uint8_t)d;
}

__global__ void k_flags(const uint8_t * __restrict__ dl, int level, uint64_t n,
                        uint32_t * __restrict__ flag) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) flag[i] = (dl[i] <= level) ? 1u : 0u;
}

// nid = inclusive scan of flags.  Node f (= nid-1) starts at position i.
__global__ void k_scatter_nodes(const uint8_t * __restrict__ dl, int level,
                                const uint32_t * __restrict__ nid,
                                const uint32_t * __restrict__ sidx_level, uint64_t n,
                                uint32_t * __restrict__ ids_out,      // may be null
                                uint32_t * __restrict__ start_out,    // may be null: position i
                                const uint32_t * __restrict__ child_nid,  // may be null
                                uint32_t * __restrict__ child_out) {  // may be null
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n || dl[i] > level) return;
  const uint32_t f = nid[i] - 1u;
  if (ids_out) ids_out[f] = sidx_level[i];
  if (start_out) start_out[f] = (uint32_t)i;
  if (child_out) child_out[f] = child_nid[i] - 1u;
}

__global__ void k_desc(const uint32_t * __restrict__ nid, uint64_t n, uint64_t chunk0,
                       uint64_t nchunks, int level, int stride, uint32_t * __restrict__ desc) {
  uint64_t c = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (c >= nchunks) return;
  const uint64_t pos = (chunk0 + c) * SPB200_CHUNK;
  desc[c * stride + level] = nid[pos] - 1u;
}

__global__ void k_fill_rec(const double * __restrict__ vals, const uint32_t * __restrict__ order,
                           const uint32_t * __restrict__ leaf, const uint32_t * __restrict__ parent,
                           const uint8_t * __restrict__ dl, int N, uint64_t n_total, uint64_t first,
                           uint64_t count, SpRec * __restrict__ rec) {
  uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (j >= count) return;
  const uint64_t i = first + j;
  uint32_t c;
  if (i + 1 == n_total) c = (uint32_t)(N - 1);
  else {
    const int d = dl[i + 1];
    c = (d >= N - 1) ? 0u : (uint32_t)(N - 1 - d);
  }
  SpRec r;
  r.v   = vals[order ? order[i] : i];
  r.k   = leaf[i];
  r.aux = parent[i] | (c << SPB200_IDX_BITS);
  rec[j] = r;
}

__global__ void k_gather_f64(const double * __restrict__ src, const uint32_t * __restrict__ order,
                             uint64_t n, double * __restrict__ dst) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) dst[i] = order ? src[order[i]] : src[i];
}

inline unsigned nblk(uint64_t n) { return (unsigned)((n + 255) / 256); }

// Sorted view of the COO data in level order.
struct SortedCoo {
  int N = 0;
  uint64_t nnz = 0;
  DevBuf order;                 // uint32[nnz]: source nonzero of every record
  DevBuf sidx[SPB200_MAXN];     // uint32[nnz] per level
  DevBuf dl;                    // uint8[nnz]
};

#define CK(call)                                                                        \
  do {                                                                                  \
    cudaError_t e_ = (call);                                                            \
    if (e_ != cudaSuccess) {                                                            \
      fprintf(stderr, "SPLATT: CUDA error '%s' at %s:%d\n", cudaGetErrorString(e_),     \
              __FILE__, __LINE__);                                                      \
      return (e_ == cudaErrorMemoryAllocation) ? SPLATT_ERROR_NOMEMORY                  \
                                               : SPLATT_ERROR_BADINPUT;                 \
    }                                                                                   \
  } while (0)

// Sort the whole tensor lexicographically in level order: leaves sc->order
// (empty when presorted).  LSD radix passes; as many trailing levels as fit are
// packed into one 64-bit key.
int sort_order(int N, const uint64_t * dims, uint64_t nnz, const uint32_t * const * d_ind,
               const int * perm, bool presorted, DevBuf * order) {
  if (nnz >= 0xffffffffull) {
    fprintf(stderr, "SPLATT: tensors with >= 2^32 nonzeros per device are not supported\n");
    return SPLATT_ERROR_BADINPUT;
  }
  for (int m = 0; m < N; ++m) {
    // leaf indices use 32 bits; every other level is a 'parent' in some stream
    if (dims[m] > (1ull << SPB200_IDX_BITS)) {
      fprintf(stderr, "SPLATT: mode %d has %llu > 2^%d rows; not supported by the "
              "device stream format\n", m, (unsigned long long)dims[m], SPB200_IDX_BITS);
      return SPLATT_ERROR_BADINPUT;
    }
  }
  if (presorted || nnz == 0) return SPLATT_SUCCESS;
  CK(order->alloc(nnz * 4));
  DevBuf order_alt, keys, keys_alt, tmp;
  CK(order_alt.alloc(nnz * 4));
  CK(keys.alloc(nnz * 8));
  CK(keys_alt.alloc(nnz * 8));
  k_iota<<<nblk(nnz), 256>>>(order->as<uint32_t>(), nnz);
  int l = N - 1;
  while (l >= 0) {
    KeySpec ks; ks.n = 0;
    int used = 0;
    while (l >= 0) {
      const int b = bits_for(dims[perm[l]]);
      if (used + b > 64) break;
      ks.src[ks.n] = d_ind[perm[l]];
      ks.shift[ks.n] = used;
      ++ks.n;
      used += b;
      --l;
    }
    k_make_keys<<<nblk(nnz), 256>>>(ks, order->as<uint32_t>(), nnz, keys.as<uint64_t>());
    cub::DoubleBuffer<uint64_t> kb(keys.as<uint64_t>(), keys_alt.as<uint64_t>());
    cub::DoubleBuffer<uint32_t> vb(order->as<uint32_t>(), order_alt.as<uint32_t>());
    size_t tb = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, tb, kb, vb, (int64_t)nnz, 0, used));
    if (tb > tmp.bytes) CK(tmp.alloc(tb));
    CK(cub::DeviceRadixSort::SortPairs(tmp.p, tb, kb, vb, (int64_t)nnz, 0, used));
    if (vb.Current() != order->as<uint32_t>()) std::swap(order->p, order_alt.p);
    if (kb.Current() != keys.as<uint64_t>()) std::swap(keys.p, keys_alt.p);
  }
  CK(cudaGetLastError());
  return SPLATT_SUCCESS;
}

// Leaf-tile re-ordering ("k-tiling").  The local records are cut into `nranges`
// chunk-aligned ranges (the same cut the kernel makes when it hands ranges to
// lane groups); inside every range the records are regrouped by
// leaf-index tile = leaf / tile_rows, keeping CSF order inside a (range, tile)
// segment.  All groups of an SM then sweep the leaf factor tile by tile at the
// same pace, so the rows of the current tile stay L1-resident and are re-used
// instead of being fetched from L2 once per nonzero.  seg[n] = segment id of
// local record n (segment changes force a node break at every level).
__global__ void k_tile_keys(const uint32_t * __restrict__ leaf_src,
                            const uint32_t * __restrict__ lorder, uint64_t n0, uint64_t nrec,
                            uint64_t nchunks, uint32_t nranges, uint32_t tile_rows,
                            uint32_t ntiles, uint32_t * __restrict__ keys,
                            uint32_t * __restrict__ pos) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= nrec) return;
  const uint64_t c = i / SPB200_CHUNK;
  uint64_t r = ((c + 1) * nranges - 1) / nchunks;        // largest r with r*nchunks/nranges <= c
  if (r >= nranges) r = nranges - 1;
  const uint32_t src = lorder ? lorder[i] : (uint32_t)(n0 + i);
  keys[i] = (uint32_t)r * ntiles + leaf_src[src] / tile_rows;
  pos[i]  = src;
}

int tile_local_order(const uint32_t * leaf_src, const uint32_t * lorder, uint64_t n0,
                     uint64_t nrec, uint32_t nranges, uint32_t tile_rows, uint32_t ntiles,
                     DevBuf * new_order, DevBuf * seg) {
  const uint64_t nchunks = (nrec + SPB200_CHUNK - 1) / SPB200_CHUNK;
  DevBuf keys_alt, pos_alt, tmp;
  CK(seg->alloc(nrec * 4));
  CK(new_order->alloc(nrec * 4));
  CK(keys_alt.alloc(nrec * 4));
  CK(pos_alt.alloc(nrec * 4));
  k_tile_keys<<<nblk(nrec), 256>>>(leaf_src, lorder, n0, nrec, nchunks, nranges, tile_rows,
                                   ntiles, seg->as<uint32_t>(), new_order->as<uint32_t>());
  cub::DoubleBuffer<uint32_t> kb(seg->as<uint32_t>(), keys_alt.as<uint32_t>());
  cub::DoubleBuffer<uint32_t> vb(new_order->as<uint32_t>(), pos_alt.as<uint32_t>());
  int bits = 1;
  while (bits < 32 && (1ull << bits) < (uint64_t)nranges * ntiles) ++bits;
  size_t tb = 0;
  CK(cub::DeviceRadixSort::SortPairs(nullptr, tb, kb, vb, (int64_t)nrec, 0, bits));
  CK(tmp.alloc(tb));
  CK(cub::DeviceRadixSort::SortPairs(tmp.p, tb, kb, vb, (int64_t)nrec, 0, bits));   // stable
  if (vb.Current() != new_order->as<uint32_t>()) std::swap(new_order->p, pos_alt.p);
  if (kb.Current() != seg->as<uint32_t>()) std::swap(seg->p, keys_alt.p);
  CK(cudaGetLastError());
  return SPLATT_SUCCESS;
}

// seg_off[key] = first local record whose segment id is >= key (segment ids ascend).
__global__ void k_seg_offsets(const uint32_t * __restrict__ seg, uint64_t n, uint32_t nkeys,
                              uint32_t * __restrict__ seg_off) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i > n) return;
  const uint32_t lo = (i == 0) ? 0u : seg[i - 1] + 1u;
  const uint32_t hi = (i == n) ? nkeys : seg[i];          // keys in [lo, hi] start at i
  if (i == n) { for (uint32_t k = lo; k <= nkeys; ++k) seg_off[k] = (uint32_t)n; return; }
  for (uint32_t k = lo; k <= hi; ++k) seg_off[k] = (uint32_t)i;
}

// rroot[2r], rroot[2r + 1] = least / greatest root index of the records of range r
// (seg_off[r * ntiles] .. seg_off[(r + 1) * ntiles]); an empty range gets 1, 0.
__global__ void k_range_roots(const uint32_t * __restrict__ rootid,
                              const uint32_t * __restrict__ seg_off, uint32_t ntiles,
                              uint32_t * __restrict__ rroot) {
  __shared__ uint32_t lo, hi;
  if (threadIdx.x == 0) { lo = 0xffffffffu; hi = 0u; }
  __syncthreads();
  const uint32_t b = seg_off[(size_t)blockIdx.x * ntiles], e = seg_off[(size_t)(blockIdx.x + 1) * ntiles];
  uint32_t l = 0xffffffffu, h = 0u;
  for (uint32_t i = b + threadIdx.x; i < e; i += blockDim.x) {
    l = min(l, rootid[i]);
    h = max(h, rootid[i]);
  }
  atomicMin(&lo, l);
  atomicMax(&hi, h);
  __syncthreads();
  if (threadIdx.x == 0) {
    rroot[2 * blockIdx.x]     = (b < e) ? lo : 1u;
    rroot[2 * blockIdx.x + 1] = (b < e) ? hi : 0u;
  }
}

__global__ void k_offset_iota(uint32_t * o, uint64_t n0, uint64_t n) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) o[i] = (uint32_t)(n0 + i);
}

__global__ void k_seg_breaks(const uint32_t * __restrict__ seg, uint64_t n,
                             uint8_t * __restrict__ dl) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i > 0 && i < n && seg[i] != seg[i - 1]) dl[i] = 0;
}

// Gather the per-level indices of `count` records taken in the order `ord`
// (ord[i] = source nonzero) and compute their first-differing levels.
int gather_levels(int N, const uint32_t * const * d_ind, const int * perm, const uint32_t * ord,
                  uint64_t n0, uint64_t count, const uint32_t * seg, SortedCoo * sc) {
  sc->N = N;
  sc->nnz = count;
  // materialise the order so later stages can index values with it
  CK(sc->order.alloc(count * 4));
  if (count) {
    if (ord) CK(cudaMemcpy(sc->order.p, ord, count * 4, cudaMemcpyDeviceToDevice));
    else k_offset_iota<<<nblk(count), 256>>>(sc->order.as<uint32_t>(), n0, count);
  }
  for (int lv = 0; lv < N; ++lv) {
    CK(sc->sidx[lv].alloc(count * 4));
    if (count)
      k_gather_u32<<<nblk(count), 256>>>(d_ind[perm[lv]], sc->order.as<uint32_t>(), count,
                                         sc->sidx[lv].as<uint32_t>());
  }
  CK(sc->dl.alloc(count));
  if (count) {
    LevelPtrs lp;
    for (int lv = 0; lv < SPB200_MAXN; ++lv) lp.s[lv] = lv < N ? sc->sidx[lv].as<uint32_t>() : nullptr;
    k_first_diff<<<nblk(count), 256>>>(lp, N, count, sc->dl.as<uint8_t>());
    if (seg) k_seg_breaks<<<nblk(count), 256>>>(seg, count, sc->dl.as<uint8_t>());
  }
  CK(cudaGetLastError());
  return SPLATT_SUCCESS;
}

// Inclusive scan of (dl <= level) into nid; returns the node count.
int scan_level(SortedCoo & sc, int level, DevBuf & flag, DevBuf & nid, DevBuf & tmp,
               uint64_t * nnodes) {
  const uint64_t nnz = sc.nnz;
  *nnodes = 0;
  if (nnz == 0) return SPLATT_SUCCESS;
  k_flags<<<nblk(nnz), 256>>>(sc.dl.as<uint8_t>(), level, nnz, flag.as<uint32_t>());
  size_t tb = 0;
  CK(cub::DeviceScan::InclusiveSum(nullptr, tb, flag.as<uint32_t>(), nid.as<uint32_t>(),
                                   (int64_t)nnz));
  if (tb > tmp.bytes) CK(tmp.alloc(tb));
  CK(cub::DeviceScan::InclusiveSum(tmp.p, tb, flag.as<uint32_t>(), nid.as<uint32_t>(),
                                   (int64_t)nnz));
  uint32_t last = 0;
  CK(cudaMemcpy(&last, nid.as<uint32_t>() + (nnz - 1), 4, cudaMemcpyDeviceToHost));
  *nnodes = last;
  return SPLATT_SUCCESS;
}

}  // namespace

void spb200_free_stream(FiberStream * s) {
  if (!s) return;
  if (s->rec) cudaFree(s->rec);
  if (s->seg_off) cudaFree(s->seg_off);
  if (s->rootid) cudaFree(s->rootid);
  if (s->rroot) cudaFree(s->rroot);
  for (int l = 0; l < SPB200_MAXN; ++l)
    if (s->up[l]) cudaFree(s->up[l]);
  if (s->desc) cudaFree(s->desc);
  if (s->anc) cudaFree(s->anc);
  *s = FiberStream();
}

int spb200_build_stream(int N, const uint64_t * dims, uint64_t nnz,
                        const uint32_t * const * d_ind, const double * d_vals, const int * perm,
                        bool presorted, int shard_rank, int shard_count,
                        const StreamTiling & tiling, FiberStream * out) {
  *out = FiberStream();
  __atomic_fetch_add(&g_spb200_builds, 1ull, __ATOMIC_RELAXED);
  out->nmodes = N;
  for (int l = 0; l < N; ++l) out->perm[l] = perm[l];
  out->nrec_total = nnz;
  out->leaf_rows = dims[perm[N - 1]];

  // 1. whole-tensor CSF order
  DevBuf order;
  int rc = sort_order(N, dims, nnz, d_ind, perm, presorted, &order);
  if (rc != SPLATT_SUCCESS) return rc;

  // 2. this shard = a contiguous, equal-count range of 64-record chunks
  uint64_t c0 = 0, c1 = 0;
  spb200_shard_chunks(nnz, shard_rank, shard_count, &c0, &c1);
  const uint64_t r0 = c0 * SPB200_CHUNK;
  const uint64_t r1 = std::min<uint64_t>(c1 * SPB200_CHUNK, nnz);
  out->nchunks = c1 - c0;
  out->nrec = (r1 > r0) ? (r1 - r0) : 0;
  const uint64_t nrec = out->nrec;
  const uint32_t * lorder = order.p ? order.as<uint32_t>() + r0 : nullptr;

  // 3. optional leaf-tile re-ordering inside kernel ranges
  DevBuf tiled_order, seg;
  const bool tiled = tiling.tile_rows > 0 && tiling.nranges > 0 && nrec > 0 &&
                     dims[perm[N - 1]] > tiling.tile_rows;
  if (tiled) {
    const uint32_t ntiles = (uint32_t)((dims[perm[N - 1]] + tiling.tile_rows - 1) / tiling.tile_rows);
    rc = tile_local_order(d_ind[perm[N - 1]], lorder, r0, nrec, tiling.nranges, tiling.tile_rows,
                          ntiles, &tiled_order, &seg);
    if (rc != SPLATT_SUCCESS) return rc;
    lorder = tiled_order.as<uint32_t>();
    out->ktile_rows = tiling.tile_rows;
    out->kranges = tiling.nranges;
  }

  // 4. per-level structure of the local records
  SortedCoo sc;
  rc = gather_levels(N, d_ind, perm, lorder, r0, nrec, tiled ? seg.as<uint32_t>() : nullptr, &sc);
  if (rc != SPLATT_SUCCESS) return rc;
  order.alloc(0);
  tiled_order.alloc(0);

  size_t held = 0;
  if (tiled && tiling.cta) {
    const uint32_t ntiles = (uint32_t)((dims[perm[N - 1]] + tiling.tile_rows - 1) / tiling.tile_rows);
    const uint32_t nkeys = tiling.nranges * ntiles;
    void * so = nullptr; void * ri = nullptr; void * rr = nullptr;
    if (cudaMalloc(&so, ((size_t)nkeys + 1) * 4) != cudaSuccess ||
        cudaMalloc(&ri, std::max<uint64_t>(nrec, 1) * 4) != cudaSuccess ||
        cudaMalloc(&rr, (size_t)tiling.nranges * 2 * 4) != cudaSuccess) {
      if (so) cudaFree(so);
      if (ri) cudaFree(ri);
      return SPLATT_ERROR_NOMEMORY;
    }
    out->seg_off = static_cast<uint32_t *>(so);
    out->rootid = static_cast<uint32_t *>(ri);
    out->rroot = static_cast<uint32_t *>(rr);
    out->ntiles = ntiles;
    k_seg_offsets<<<nblk(nrec + 1), 256>>>(seg.as<uint32_t>(), nrec, nkeys, out->seg_off);
    CK(cudaMemcpy(out->rootid, sc.sidx[0].as<uint32_t>(), nrec * 4, cudaMemcpyDeviceToDevice));
    k_range_roots<<<tiling.nranges, 256>>>(out->rootid, out->seg_off, ntiles, out->rroot);
    std::vector<uint32_t> rh((size_t)tiling.nranges * 2);
    CK(cudaMemcpy(rh.data(), out->rroot, rh.size() * 4, cudaMemcpyDeviceToHost));
    for (uint32_t r = 0; r < tiling.nranges; ++r)
      if (rh[2 * r + 1] >= rh[2 * r]) out->acc_rows = std::max(out->acc_rows, rh[2 * r + 1] - rh[2 * r] + 1);
    held += ((size_t)nkeys + 1) * 4 + nrec * 4 + rh.size() * 4;
  }
  DevBuf flag, nid, tmp, desc;
  CK(flag.alloc(nrec * 4));
  CK(nid.alloc(nrec * 4));
  const int stride = N - 2;
  CK(desc.alloc(std::max<uint64_t>(out->nchunks, 1) * stride * 4));
  for (int l = 0; l <= N - 2; ++l) {
    uint64_t nn = 0;
    rc = scan_level(sc, l, flag, nid, tmp, &nn);
    if (rc != SPLATT_SUCCESS) { spb200_free_stream(out); return rc; }
    out->nnodes[l] = nn;
    if (l <= N - 3) {
      // +1 pad so a one-past-the-end read stays in bounds
      void * up = nullptr;
      cudaError_t e = cudaMalloc(&up, (nn + 1) * 4);
      if (e != cudaSuccess) { spb200_free_stream(out); return SPLATT_ERROR_NOMEMORY; }
      cudaMemset(up, 0, (nn + 1) * 4);
      out->up[l] = static_cast<uint32_t *>(up);
      held += (nn + 1) * 4;
      if (nrec) {
        k_scatter_nodes<<<nblk(nrec), 256>>>(sc.dl.as<uint8_t>(), l, nid.as<uint32_t>(),
                                             sc.sidx[l].as<uint32_t>(), nrec, out->up[l], nullptr,
                                             nullptr, nullptr);
        k_desc<<<nblk(out->nchunks), 256>>>(nid.as<uint32_t>(), nrec, 0, out->nchunks, l, stride,
                                            desc.as<uint32_t>());
      }
    }
  }
  out->nnodes[N - 1] = nrec;
  {
    void * rec = nullptr;
    cudaError_t e = cudaMalloc(&rec, std::max<uint64_t>(nrec, 1) * sizeof(SpRec));
    if (e != cudaSuccess) { spb200_free_stream(out); return SPLATT_ERROR_NOMEMORY; }
    out->rec = static_cast<SpRec *>(rec);
    held += nrec * sizeof(SpRec);
    if (nrec)
      k_fill_rec<<<nblk(nrec), 256>>>(d_vals, sc.order.as<uint32_t>(), sc.sidx[N - 1].as<uint32_t>(),
                                      sc.sidx[N - 2].as<uint32_t>(), sc.dl.as<uint8_t>(), N, nrec, 0,
                                      nrec, out->rec);
  }
  if (N >= 4) {
    // level-(N-3) index of every record, beside the records (root kernels of deep trees);
    // padded so 16-byte TMA copies of a range tail stay inside the allocation
    const size_t ab = (std::max<uint64_t>(nrec, 1) * 4 + 15) & ~(size_t)15;
    void * anc = nullptr;
    if (cudaMalloc(&anc, ab) != cudaSuccess) { spb200_free_stream(out); return SPLATT_ERROR_NOMEMORY; }
    out->anc = static_cast<uint32_t *>(anc);
    cudaMemset(anc, 0, ab);
    if (nrec)
      CK(cudaMemcpy(anc, sc.sidx[N - 3].as<uint32_t>(), nrec * 4, cudaMemcpyDeviceToDevice));
    held += ab;
  }
  held += desc.bytes;
  out->desc = static_cast<uint32_t *>(desc.release());
  out->bytes = held;
  CK(cudaGetLastError());
  CK(cudaDeviceSynchronize());
  return SPLATT_SUCCESS;
}

// ---------------------------------------------------------------------------
// Slicing a whole stream into shards (multi-GPU from one build).
// ---------------------------------------------------------------------------
namespace {
__global__ void k_rebase_desc(uint32_t * __restrict__ desc, uint64_t nchunks, int stride,
                              const uint32_t * __restrict__ base) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < nchunks * (uint64_t)stride) desc[i] -= base[i % stride];
}
__global__ void k_count_fibers(const SpRec * __restrict__ rec, uint64_t n,
                               unsigned long long * __restrict__ count) {
  uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  unsigned c = 0;
  if (i < n) c = ((rec[i].aux >> SPB200_IDX_BITS) != 0u) || (i + 1 == n);
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, (unsigned long long)c);
}
}  // namespace

int spb200_slice_stream(const FiberStream & w, int src_dev, uint64_t c0, uint64_t c1, int dst_dev,
                        FiberStream * out) {
  *out = FiberStream();
  if (w.ktile_rows || w.nrec != w.nrec_total) {
    fprintf(stderr, "SPLATT: only whole, untiled streams can be sliced\n");
    return SPLATT_ERROR_BADINPUT;
  }
  const int N = w.nmodes;
  const int stride = N - 2;
  if (c1 > w.nchunks) c1 = w.nchunks;
  if (c0 > c1) c0 = c1;
  const uint64_t r0 = c0 * SPB200_CHUNK;
  const uint64_t r1 = std::min<uint64_t>(c1 * SPB200_CHUNK, w.nrec);
  const uint64_t nrec = r1 > r0 ? r1 - r0 : 0;
  out->nmodes = N;
  for (int l = 0; l < N; ++l) out->perm[l] = w.perm[l];
  out->nrec_total = w.nrec_total;
  out->leaf_rows = w.leaf_rows;
  out->nrec = nrec;
  out->nchunks = c1 - c0;

  // node numbers at the cut points (from the source device)
  uint32_t first[SPB200_MAXN] = {0}, next[SPB200_MAXN] = {0};
  uint32_t last_aux = 0;
  CK(cudaSetDevice(src_dev));
  if (nrec && stride > 0) {
    CK(cudaMemcpy(first, w.desc + c0 * stride, sizeof(uint32_t) * stride, cudaMemcpyDeviceToHost));
    if (c1 < w.nchunks)
      CK(cudaMemcpy(next, w.desc + c1 * stride, sizeof(uint32_t) * stride, cudaMemcpyDeviceToHost));
  }
  if (nrec) CK(cudaMemcpy(&last_aux, &w.rec[r1 - 1].aux, 4, cudaMemcpyDeviceToHost));
  const uint32_t last_c = last_aux >> SPB200_IDX_BITS;

  CK(cudaSetDevice(dst_dev));
  size_t held = 0;
  auto peer_copy = [&](void * dst, const void * src, size_t bytes) -> cudaError_t {
    if (!bytes) return cudaSuccess;
    if (src_dev == dst_dev) return cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToDevice);
    return cudaMemcpyPeer(dst, dst_dev, src, src_dev, bytes);
  };
  {
    void * rec = nullptr;
    if (cudaMalloc(&rec, std::max<uint64_t>(nrec, 1) * sizeof(SpRec)) != cudaSuccess)
      return SPLATT_ERROR_NOMEMORY;
    out->rec = static_cast<SpRec *>(rec);
    CK(peer_copy(rec, w.rec + r0, nrec * sizeof(SpRec)));
    held += nrec * sizeof(SpRec);
  }
  if (w.anc) {
    const size_t ab = (std::max<uint64_t>(nrec, 1) * 4 + 15) & ~(size_t)15;
    void * anc = nullptr;
    if (cudaMalloc(&anc, ab) != cudaSuccess) { spb200_free_stream(out); return SPLATT_ERROR_NOMEMORY; }
    out->anc = static_cast<uint32_t *>(anc);
    CK(cudaMemset(anc, 0, ab));
    CK(peer_copy(anc, w.anc + r0, nrec * 4));
    held += ab;
  }
  for (int l = 0; l <= N - 3; ++l) {
    uint64_t nn = 0;
    if (nrec) {
      // node holding the shard's last record: the one before `next` if that record ends
      // level l (close count >= N-1-l), else `next` itself continues it
      const uint64_t lastn = (c1 < w.nchunks)
                                 ? (uint64_t)next[l] - ((last_c >= (uint32_t)(N - 1 - l)) ? 1u : 0u)
                                 : w.nnodes[l] - 1;
      nn = lastn - first[l] + 1;
    }
    void * up = nullptr;
    if (cudaMalloc(&up, (nn + 1) * 4) != cudaSuccess) { spb200_free_stream(out); return SPLATT_ERROR_NOMEMORY; }
    out->up[l] = static_cast<uint32_t *>(up);
    CK(cudaMemset(up, 0, (nn + 1) * 4));
    CK(peer_copy(up, w.up[l] + first[l], nn * 4));
    out->nnodes[l] = nn;
    held += (nn + 1) * 4;
  }
  {
    const size_t db = std::max<uint64_t>(out->nchunks, 1) * (stride > 0 ? stride : 1) * 4;
    void * desc = nullptr;
    if (cudaMalloc(&desc, db) != cudaSuccess) { spb200_free_stream(out); return SPLATT_ERROR_NOMEMORY; }
    out->desc = static_cast<uint32_t *>(desc);
    held += db;
    if (stride > 0 && out->nchunks) {
      CK(peer_copy(desc, w.desc + c0 * stride, out->nchunks * stride * 4));
      DevBuf base;
      CK(base.alloc(sizeof(uint32_t) * stride));
      CK(cudaMemcpy(base.p, first, sizeof(uint32_t) * stride, cudaMemcpyHostToDevice));
      k_rebase_desc<<<nblk(out->nchunks * stride), 256>>>(out->desc, out->nchunks, stride,
                                                          base.as<uint32_t>());
      CK(cudaDeviceSynchronize());
    }
  }
  // fibers (level N-2 nodes) intersecting the shard
  if (N >= 2) {
    unsigned long long nf = 0;
    if (nrec) {
      DevBuf cnt;
      CK(cnt.alloc(8));
      CK(cudaMemset(cnt.p, 0, 8));
      k_count_fibers<<<nblk(nrec), 256>>>(out->rec, nrec, cnt.as<unsigned long long>());
      CK(cudaMemcpy(&nf, cnt.p, 8, cudaMemcpyDeviceToHost));
    }
    out->nnodes[N - 2] = nf;
  }
  out->nnodes[N - 1] = nrec;
  out->bytes = held;
  CK(cudaGetLastError());
  CK(cudaDeviceSynchronize());
  return SPLATT_SUCCESS;
}

// ---------------------------------------------------------------------------
// Reference-shaped host CSF (one tile, untiled) from device COO.
// Mirrors what p_csf_alloc_untiled builds (reference: src/csf.c:468-502):
//   fids[N-1] = sorted leaf indices, vals = sorted values,
//   for l < N-1: fids[l][f] / fptr[l][f] per node, fptr[l][nfibs] = #children
//   level; fids[0] == NULL iff every root index occurs (src/csf.c:303-309).
// ---------------------------------------------------------------------------
static splatt_idx_t * widen_to_host(const uint32_t * d, uint64_t n, uint64_t extra_slots) {
  std::vector<uint32_t> h(n ? n : 1);
  if (n && cudaMemcpy(h.data(), d, n * 4, cudaMemcpyDeviceToHost) != cudaSuccess) return nullptr;
  splatt_idx_t * o = static_cast<splatt_idx_t *>(malloc((n + extra_slots + 1) * sizeof(splatt_idx_t)));
  if (!o) return nullptr;
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < (int64_t)n; ++i) o[i] = h[i];
  return o;
}

int spb200_build_host_csf(int N, const uint64_t * dims, uint64_t nnz,
                          const uint32_t * const * d_ind, const double * d_vals, const int * perm,
                          splatt_csf * csf) {
  memset(csf, 0, sizeof(*csf));
  csf->nnz = nnz;
  csf->nmodes = N;
  for (int m = 0; m < N; ++m) {
    csf->dims[m] = dims[m];
    csf->dim_perm[m] = perm[m];
    csf->dim_iperm[perm[m]] = m;
    csf->tile_dims[m] = 1;
  }
  csf->which_tile = SPLATT_NOTILE;
  csf->ntiles = 1;
  csf->ntiled_modes = 0;
  csf->pt = static_cast<csf_sparsity *>(calloc(1, sizeof(csf_sparsity)));
  if (!csf->pt) return SPLATT_ERROR_NOMEMORY;
  csf_sparsity * pt = csf->pt;

  DevBuf order;
  int rc = sort_order(N, dims, nnz, d_ind, perm, false, &order);
  if (rc != SPLATT_SUCCESS) return rc;
  SortedCoo sc;
  rc = gather_levels(N, d_ind, perm, order.p ? order.as<uint32_t>() : nullptr, 0, nnz, nullptr, &sc);
  if (rc != SPLATT_SUCCESS) return rc;
  order.alloc(0);

  // leaves
  pt->nfibs[N - 1] = nnz;
  pt->fids[N - 1] = widen_to_host(sc.sidx[N - 1].as<uint32_t>(), nnz, 0);
  pt->vals = static_cast<splatt_val_t *>(malloc((nnz + 1) * sizeof(double)));
  if (!pt->fids[N - 1] || !pt->vals) return SPLATT_ERROR_NOMEMORY;
  {
    DevBuf sv;
    CK(sv.alloc(nnz * 8));
    if (nnz) {
      k_gather_f64<<<nblk(nnz), 256>>>(d_vals, sc.order.as<uint32_t>(), nnz, sv.as<double>());
      CK(cudaMemcpy(pt->vals, sv.p, nnz * 8, cudaMemcpyDeviceToHost));
    }
  }

  DevBuf flag, nid, nid_child, tmp, ids, starts;
  CK(flag.alloc(nnz * 4));
  CK(nid.alloc(nnz * 4));
  CK(nid_child.alloc(nnz * 4));
  CK(ids.alloc(nnz * 4));
  CK(starts.alloc(nnz * 4));
  uint64_t nn_child = nnz;
  for (int l = N - 2; l >= 0; --l) {
    uint64_t nn = 0;
    rc = scan_level(sc, l, flag, nid, tmp, &nn);
    if (rc != SPLATT_SUCCESS) return rc;
    if (nnz) {
      // fptr[l][f]: for l == N-2 the leaf position, else the child node number
      k_scatter_nodes<<<nblk(nnz), 256>>>(
          sc.dl.as<uint8_t>(), l, nid.as<uint32_t>(), sc.sidx[l].as<uint32_t>(), nnz,
          ids.as<uint32_t>(), (l == N - 2) ? starts.as<uint32_t>() : nullptr,
          (l == N - 2) ? nullptr : nid_child.as<uint32_t>(),
          (l == N - 2) ? nullptr : starts.as<uint32_t>());
      CK(cudaGetLastError());
    }
    pt->nfibs[l] = nn;
    pt->fids[l] = widen_to_host(ids.as<uint32_t>(), nn, 0);
    pt->fptr[l] = widen_to_host(starts.as<uint32_t>(), nn, 1);
    if (!pt->fids[l] || !pt->fptr[l]) return SPLATT_ERROR_NOMEMORY;
    pt->fptr[l][nn] = nn_child;
    nn_child = nn;
    std::swap(nid.p, nid_child.p);
  }
  // root ids are implicit when the root mode has no empty slices
  if (pt->nfibs[0] == dims[perm[0]]) {
    free(pt->fids[0]);
    pt->fids[0] = nullptr;
  }
  return SPLATT_SUCCESS;
}
