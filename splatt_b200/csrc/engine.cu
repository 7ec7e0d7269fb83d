// Engine entry points (include/splatt_b200.h, group 2): HBM-resident tensors and
// device-pointer MTTKRP.
#include "common.h"
#include <algorithm>
#include <cstring>
#include <cstdlib>
#include <vector>
#include <cstdlib>

// ---------------------------------------------------------------------------
// Level orders.  Semantics of csf_find_mode_order (reference: src/csf.c:694-726):
// SORTED_SMALLFIRST sorts modes by length, ties by mode number
// (p_order_dims_small :111-136); SORTED_MINUSONE moves one chosen mode to the
// root and keeps the rest in that order (p_order_dims_minusone :177-195).
// ---------------------------------------------------------------------------
void spb200_order_small_first(const uint64_t * dims, int N, int * perm) {
  for (int m = 0; m < N; ++m) perm[m] = m;
  std::stable_sort(perm, perm + N, [&](int a, int b) { return dims[a] < dims[b]; });
}
void spb200_order_minus_one(const uint64_t * dims, int N, int mode, int * perm) {
  int tmp[SPB200_MAXN];
  spb200_order_small_first(dims, N, tmp);
  perm[0] = mode;
  int w = 1;
  for (int i = 0; i < N; ++i)
    if (tmp[i] != mode) perm[w++] = tmp[i];
}

// How many CSFs an allocation policy yields and their level orders
// (reference: csf_alloc src/csf.c:770-814).
int spb200_csf_orders(const uint64_t * dims, int N, int csf_alloc, int perms[][SPB200_MAXN]) {
  switch (csf_alloc) {
    case SPLATT_CSF_ONEMODE:
      spb200_order_small_first(dims, N, perms[0]);
      return 1;
    case SPLATT_CSF_TWOMODE:
      spb200_order_small_first(dims, N, perms[0]);
      spb200_order_minus_one(dims, N, perms[0][N - 1], perms[1]);
      return 2;
    case SPLATT_CSF_ALLMODE:
      for (int m = 0; m < N; ++m) spb200_order_minus_one(dims, N, m, perms[m]);
      return N;
    default:
      return 0;
  }
}

// Mode -> CSF map of the MTTKRP workspace (reference: src/mttkrp.c:1832-1861).
void spb200_mode_csf_map(int N, int csf_alloc, const int perm0[SPB200_MAXN], int * map) {
  for (int m = 0; m < N; ++m) {
    switch (csf_alloc) {
      case SPLATT_CSF_ONEMODE: map[m] = 0; break;
      case SPLATT_CSF_TWOMODE: map[m] = (perm0[N - 1] == m) ? 1 : 0; break;
      default: map[m] = m; break;
    }
  }
}

// Chunk range [c0, c1) of shard `rank`: equal chunk counts (+-1).
void spb200_shard_chunks(uint64_t nnz, int rank, int nshards, uint64_t * c0, uint64_t * c1) {
  const uint64_t nchunks = (nnz + SPB200_CHUNK - 1) / SPB200_CHUNK;
  if (nshards < 1) nshards = 1;
  if (rank < 0) rank = 0;
  if (rank >= nshards) rank = nshards - 1;
  *c0 = nchunks * (uint64_t)rank / (uint64_t)nshards;
  *c1 = nchunks * (uint64_t)(rank + 1) / (uint64_t)nshards;
}

namespace {

struct DevCoo {
  int N = 0;
  uint64_t nnz = 0;
  uint32_t * ind[SPB200_MAXN] = {nullptr};
  double * vals = nullptr;
  bool owned = false;
  ~DevCoo() {
    if (!owned) return;
    for (int m = 0; m < SPB200_MAXN; ++m)
      if (ind[m]) cudaFree(ind[m]);
    if (vals) cudaFree(vals);
  }
};

int upload_coo(int N, uint64_t nnz, const uint32_t * const * ind, const double * vals,
               int on_device, DevCoo * dc) {
  dc->N = N;
  dc->nnz = nnz;
  if (on_device) {
    for (int m = 0; m < N; ++m) dc->ind[m] = const_cast<uint32_t *>(ind[m]);
    dc->vals = const_cast<double *>(vals);
    dc->owned = false;
    return SPLATT_SUCCESS;
  }
  dc->owned = true;
  for (int m = 0; m < N; ++m) {
    SPB200_CUDA_OK(cudaMalloc(&dc->ind[m], std::max<uint64_t>(nnz, 1) * 4));
    SPB200_CUDA_OK(cudaMemcpy(dc->ind[m], ind[m], nnz * 4, cudaMemcpyHostToDevice));
  }
  SPB200_CUDA_OK(cudaMalloc(&dc->vals, std::max<uint64_t>(nnz, 1) * 8));
  SPB200_CUDA_OK(cudaMemcpy(dc->vals, vals, nnz * 8, cudaMemcpyHostToDevice));
  return SPLATT_SUCCESS;
}

// Expand one reference CSF (all tiles) to coordinates in storage order.
// Walks the tree exactly as the reference's kernels do: children of node f at
// level l are fptr[l][f]..fptr[l][f+1] (include/splatt/structs.h:51-68); the
// root id is f itself when fids[0] == NULL (src/csf.c:303-309).
// One big tile (untiled CSF): loops are parallel inside the tile.  Many tiles
// (SPLATT_DENSETILE builds up to nthreads^nmodes of them, most tiny or empty):
// tiles are expanded concurrently, each one serially.
template <bool PAR>
void expand_tile(const splatt_csf * ct, const csf_sparsity * pt, uint64_t off, uint32_t ** ind,
                 double * vals) {
  const int N = (int)ct->nmodes;
  const uint64_t tn = pt->nfibs[N - 1];
  memcpy(vals + off, pt->vals, tn * sizeof(double));
  {
    uint32_t * dst = ind[ct->dim_perm[N - 1]] + off;
    const splatt_idx_t * src = pt->fids[N - 1];
#pragma omp parallel for schedule(static) if (PAR)
    for (int64_t n = 0; n < (int64_t)tn; ++n) dst[n] = (uint32_t)src[n];
  }
  // leaf-range start of every node, level by level from the bottom
  std::vector<uint64_t> ls_child, ls;
  for (int l = N - 2; l >= 0; --l) {
    const uint64_t nf = pt->nfibs[l];
    const splatt_idx_t * fp = pt->fptr[l];
    ls.resize(nf + 1);
    if (l == N - 2) {
#pragma omp parallel for schedule(static) if (PAR)
      for (int64_t f = 0; f <= (int64_t)nf; ++f) ls[f] = fp[f];
    } else {
#pragma omp parallel for schedule(static) if (PAR)
      for (int64_t f = 0; f <= (int64_t)nf; ++f) ls[f] = ls_child[fp[f]];
    }
    uint32_t * dst = ind[ct->dim_perm[l]] + off;
    const splatt_idx_t * ids = pt->fids[l];
#pragma omp parallel for schedule(dynamic, 256) if (PAR)
    for (int64_t f = 0; f < (int64_t)nf; ++f) {
      const uint32_t id = ids ? (uint32_t)ids[f] : (uint32_t)f;
      for (uint64_t n = ls[f]; n < ls[f + 1]; ++n) dst[n] = id;
    }
    ls_child.swap(ls);
  }
}

int csf_to_coo(const splatt_csf * ct, std::vector<uint32_t> * ind, std::vector<double> * vals) {
  const int N = (int)ct->nmodes;
  const uint64_t nnz = ct->nnz;
  uint32_t * ip[SPB200_MAXN] = {nullptr};
  for (int m = 0; m < N; ++m) { ind[m].assign(nnz, 0u); ip[m] = ind[m].data(); }
  vals->assign(nnz, 0.0);
  // storage offset of every tile (empty tiles have vals == NULL, src/mttkrp.c:682-685)
  std::vector<uint64_t> off(ct->ntiles + 1, 0);
  for (uint64_t t = 0; t < ct->ntiles; ++t)
    off[t + 1] = off[t] + (ct->pt[t].vals ? ct->pt[t].nfibs[N - 1] : 0);
  if (off[ct->ntiles] != nnz) return SPLATT_ERROR_BADINPUT;
  if (ct->ntiles == 1) {
    if (ct->pt[0].vals) expand_tile<true>(ct, ct->pt, 0, ip, vals->data());
  } else {
#pragma omp parallel for schedule(dynamic, 4)
    for (int64_t t = 0; t < (int64_t)ct->ntiles; ++t)
      if (ct->pt[t].vals) expand_tile<false>(ct, ct->pt + t, off[t], ip, vals->data());
  }
  return SPLATT_SUCCESS;
}

struct PermSpec { int perm[SPB200_MAXN]; bool presorted; };

int build_tensor(int N, const uint64_t * dims, const DevCoo & dc,
                 const std::vector<PermSpec> & stream_perms, const ModePlan * plan,
                 const splatt_b200_build_opts & bo, splatt_b200_tensor ** out) {
  splatt_b200_tensor * T = new splatt_b200_tensor();
  T->nmodes = N;
  for (int m = 0; m < N; ++m) T->dims[m] = dims[m];
  T->nnz_total = dc.nnz;
  T->layout = bo.layout;
  T->shard_rank = bo.shard_rank;
  T->shard_count = bo.shard_count > 1 ? bo.shard_count : 1;
  if (cudaGetDevice(&T->device) != cudaSuccess) { delete T; return SPLATT_ERROR_BADINPUT; }
  T->streams.resize(stream_perms.size());
  int num_sms = 132;
  cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, T->device);
  for (size_t i = 0; i < stream_perms.size(); ++i) {
    // Leaf-tile re-ordering.  Two layouts, both valid for the generic kernels too:
    //  (a) CTA-tiled: one range per SM, leaf tiles staged in shared memory by
    //      mttkrp_tiled.cu; chosen by splatt_b200_cta_tiling (DESIGN.md 4.1);
    //  (b) L1-tiled (opt-in, ktile > 0): many small ranges, tiles kept hot in L1 only
    //      statistically -- measured not to pay off (DESIGN.md 4.3).
    StreamTiling tiling;
    uint64_t local = 0;
    {
      uint64_t c0, c1;
      spb200_shard_chunks(dc.nnz, T->shard_rank, T->shard_count, &c0, &c1);
      local = std::min<uint64_t>(c1 * SPB200_CHUNK, dc.nnz) - c0 * SPB200_CHUNK;
    }
    if (bo.ktile > 0) {
      tiling.tile_rows = (uint32_t)bo.ktile;
      tiling.nranges = (uint32_t)num_sms * 48u;
    } else if (bo.ktile == 0) {
      bool root_only = true;            // every mode served by this stream runs the root kernel
      for (int m = 0; m < N; ++m)
        if (plan[m].stream == (int)i && plan[m].kind != SPB200_KIND_ROOT) root_only = false;
      const char * te = getenv("SPLATT_B200_TILED");
      const int force = (te && atoi(te) == 2) ? 1 : 0;             // testing: ignore the heuristics
      uint32_t rows = 0, acc = 0;
      if (splatt_b200_cta_tiling(N, dims, stream_perms[i].perm, local, T->shard_count,
                                 root_only ? 1 : 0, num_sms, force, &rows, &acc)) {
        const char * re = getenv("SPLATT_B200_TILE_ROWS");          // testing / tuning
        if (re && atoi(re) > 0) rows = std::min<uint32_t>(rows, (uint32_t)atoi(re));
        tiling.tile_rows = rows;
        tiling.nranges = (uint32_t)num_sms;
        tiling.cta = true;
        tiling.acc_rows = acc;
      }
    }
    if (tiling.tile_rows) {
      const uint64_t leaf_dim = dims[stream_perms[i].perm[N - 1]];
      const uint64_t ntiles = (leaf_dim + tiling.tile_rows - 1) / tiling.tile_rows;
      if ((uint64_t)tiling.nranges * ntiles >= 0x7fffffffull) tiling = StreamTiling();
    }
    int rc = spb200_build_stream(N, dims, dc.nnz, dc.ind, dc.vals, stream_perms[i].perm,
                                 stream_perms[i].presorted, T->shard_rank, T->shard_count,
                                 tiling, &T->streams[i]);
    if (rc == SPLATT_SUCCESS && tiling.cta && T->streams[i].acc_rows > tiling.acc_rows) {
      // a range touches more root rows than the shared accumulator holds: build it untiled
      spb200_free_stream(&T->streams[i]);
      rc = spb200_build_stream(N, dims, dc.nnz, dc.ind, dc.vals, stream_perms[i].perm,
                               stream_perms[i].presorted, T->shard_rank, T->shard_count,
                               StreamTiling(), &T->streams[i]);
    }
    if (rc != SPLATT_SUCCESS) { splatt_b200_tensor_free(T); return rc; }
    if (bo.verbosity >= SPLATT_VERBOSITY_MAX) {
      const FiberStream & s = T->streams[i];
      printf("SPLATT-B200: stream %zu order [", i);
      for (int l = 0; l < N; ++l) printf("%d%s", s.perm[l], l + 1 < N ? " " : "");
      printf("] nodes [");
      for (int l = 0; l < N; ++l)
        printf("%llu%s", (unsigned long long)s.nnodes[l], l + 1 < N ? " " : "");
      printf("] local records %llu, %.1f MB", (unsigned long long)s.nrec, s.bytes / 1e6);
      if (s.ktile_rows) printf(", leaf tiles of %u rows in %u ranges", s.ktile_rows, s.kranges);
      printf("\n");
    }
  }
  for (int m = 0; m < N; ++m) T->plan[m] = plan[m];
  *out = T;
  return SPLATT_SUCCESS;
}

bool same_perm(const int * a, const int * b, int N) {
  for (int l = 0; l < N; ++l)
    if (a[l] != b[l]) return false;
  return true;
}

int kind_of_depth(int depth, int N) {
  return depth == 0 ? SPB200_KIND_ROOT : (depth == N - 1 ? SPB200_KIND_LEAF : SPB200_KIND_INTL);
}

}  // namespace

extern "C" {

int splatt_b200_tensor_from_coo(int nmodes, uint64_t const * dims, uint64_t nnz,
                                uint32_t const * const * ind, double const * vals, int on_device,
                                int csf_alloc, splatt_b200_build_opts const * bopts,
                                splatt_b200_tensor ** out) {
  if (!out || !dims || nmodes < 2 || nmodes > SPB200_MAXN || (nnz && (!ind || !vals))) {
    fprintf(stderr, "SPLATT: splatt_b200_tensor_from_coo: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  splatt_b200_build_opts bo;
  memset(&bo, 0, sizeof(bo));
  bo.device = -1;
  if (bopts) bo = *bopts;
  int cur = 0;
  if (cudaGetDevice(&cur) != cudaSuccess) return SPLATT_ERROR_BADINPUT;
  DeviceGuard guard(bo.device >= 0 ? bo.device : cur);     // restored on every return path
  if (!guard.ok) return SPLATT_ERROR_BADINPUT;
  int rc = SPLATT_SUCCESS;

  const int N = nmodes;
  std::vector<PermSpec> sp;
  ModePlan plan[SPB200_MAXN];
  if (bo.layout == SPLATT_B200_LAYOUT_ALLROOT) {
    for (int m = 0; m < N; ++m) {
      PermSpec p; p.presorted = false;
      spb200_order_minus_one(dims, N, m, p.perm);
      sp.push_back(p);
      plan[m].stream = m; plan[m].kind = SPB200_KIND_ROOT; plan[m].outdepth = 0;
    }
  } else {
    int perms[SPB200_MAXN][SPB200_MAXN];
    const int nc = spb200_csf_orders(dims, N, csf_alloc, perms);
    if (nc == 0) {
      fprintf(stderr, "SPLATT: CSF type '%d' not recognized.\n", csf_alloc);
      return SPLATT_ERROR_BADINPUT;
    }
    for (int c = 0; c < nc; ++c) {
      PermSpec p; p.presorted = false;
      memcpy(p.perm, perms[c], sizeof(int) * SPB200_MAXN);
      sp.push_back(p);
    }
    int map[SPB200_MAXN];
    spb200_mode_csf_map(N, csf_alloc, perms[0], map);
    for (int m = 0; m < N; ++m) {
      int depth = 0;
      for (int l = 0; l < N; ++l)
        if (perms[map[m]][l] == m) depth = l;
      plan[m].stream = map[m]; plan[m].outdepth = depth; plan[m].kind = kind_of_depth(depth, N);
    }
  }
  DevCoo dc;
  rc = upload_coo(N, nnz, ind, vals, on_device, &dc);
  if (rc == SPLATT_SUCCESS) rc = build_tensor(N, dims, dc, sp, plan, bo, out);
  return rc;
}

int splatt_b200_tensor_from_csf(splatt_csf const * tensors, int csf_alloc,
                                splatt_b200_build_opts const * bopts, splatt_b200_tensor ** out) {
  if (!tensors || !out) return SPLATT_ERROR_BADINPUT;
  const int N = (int)tensors[0].nmodes;
  if (N < 2 || N > SPB200_MAXN) {
    fprintf(stderr, "SPLATT: the B200 engine supports 2..%d modes (got %d)\n", SPB200_MAXN, N);
    return SPLATT_ERROR_BADINPUT;
  }
  int ncsf;
  switch (csf_alloc) {
    case SPLATT_CSF_ONEMODE: ncsf = 1; break;
    case SPLATT_CSF_TWOMODE: ncsf = 2; break;
    case SPLATT_CSF_ALLMODE: ncsf = N; break;
    default:
      fprintf(stderr, "SPLATT: CSF type '%d' not recognized.\n", csf_alloc);
      return SPLATT_ERROR_BADINPUT;
  }
  splatt_b200_build_opts bo;
  memset(&bo, 0, sizeof(bo));
  bo.device = -1;
  if (bopts) bo = *bopts;
  int cur = 0;
  if (cudaGetDevice(&cur) != cudaSuccess) return SPLATT_ERROR_BADINPUT;
  DeviceGuard guard(bo.device >= 0 ? bo.device : cur);     // restored on every return path
  if (!guard.ok) return SPLATT_ERROR_BADINPUT;
  int rc = SPLATT_SUCCESS;

  uint64_t dims[SPB200_MAXN];
  for (int m = 0; m < N; ++m) dims[m] = tensors[0].dims[m];

  // coordinates in CSF 0's storage order
  std::vector<uint32_t> ind[SPB200_MAXN];
  std::vector<double> vals;
  for (int m = 0; m < N; ++m)
    if (dims[m] > 0xffffffffull) {
      fprintf(stderr, "SPLATT: mode %d too long for 32-bit device indices\n", m);
      return SPLATT_ERROR_BADINPUT;
    }
  rc = csf_to_coo(&tensors[0], ind, &vals);
  if (rc != SPLATT_SUCCESS) {
    fprintf(stderr, "SPLATT: inconsistent CSF (tile nnz do not add up)\n");
    return rc;
  }
  const bool csf0_sorted = (tensors[0].ntiles == 1);   // untiled storage order is lexicographic
  int perm0[SPB200_MAXN];
  for (int l = 0; l < N; ++l) perm0[l] = (int)tensors[0].dim_perm[l];

  std::vector<PermSpec> sp;
  ModePlan plan[SPB200_MAXN];
  if (bo.layout == SPLATT_B200_LAYOUT_ALLROOT) {
    for (int m = 0; m < N; ++m) {
      PermSpec p; p.presorted = false;
      // reuse the order of a given CSF rooted at m, else the reference's MINUSONE order
      bool found = false;
      for (int c = 0; c < ncsf && !found; ++c)
        if ((int)tensors[c].dim_perm[0] == m) {
          for (int l = 0; l < N; ++l) p.perm[l] = (int)tensors[c].dim_perm[l];
          found = true;
        }
      if (!found) spb200_order_minus_one(dims, N, m, p.perm);
      p.presorted = csf0_sorted && same_perm(p.perm, perm0, N);
      sp.push_back(p);
      plan[m].stream = m; plan[m].kind = SPB200_KIND_ROOT; plan[m].outdepth = 0;
    }
  } else {
    for (int c = 0; c < ncsf; ++c) {
      PermSpec p;
      for (int l = 0; l < N; ++l) p.perm[l] = (int)tensors[c].dim_perm[l];
      p.presorted = csf0_sorted && same_perm(p.perm, perm0, N);
      sp.push_back(p);
    }
    int map[SPB200_MAXN];
    spb200_mode_csf_map(N, csf_alloc, perm0, map);
    for (int m = 0; m < N; ++m) {
      const int depth = (int)tensors[map[m]].dim_iperm[m];
      plan[m].stream = map[m]; plan[m].outdepth = depth; plan[m].kind = kind_of_depth(depth, N);
    }
  }
  const uint32_t * hp[SPB200_MAXN];
  for (int m = 0; m < N; ++m) hp[m] = ind[m].data();
  DevCoo dc;
  rc = upload_coo(N, tensors[0].nnz, hp, vals.data(), 0, &dc);
  if (rc == SPLATT_SUCCESS) rc = build_tensor(N, dims, dc, sp, plan, bo, out);
  return rc;
}

int splatt_b200_tensor_shard(splatt_b200_tensor const * whole, int rank, int count, int device,
                             splatt_b200_tensor ** out) {
  if (!whole || !out || count < 1 || rank < 0 || rank >= count || whole->shard_count != 1) {
    fprintf(stderr, "SPLATT: splatt_b200_tensor_shard: needs a whole (unsharded) tensor\n");
    return SPLATT_ERROR_BADINPUT;
  }
  int prev = 0;
  SPB200_CUDA_OK(cudaGetDevice(&prev));
  const int dst = device >= 0 ? device : whole->device;
  splatt_b200_tensor * T = new splatt_b200_tensor();
  T->nmodes = whole->nmodes;
  for (int m = 0; m < whole->nmodes; ++m) { T->dims[m] = whole->dims[m]; T->plan[m] = whole->plan[m]; }
  T->nnz_total = whole->nnz_total;
  T->layout = whole->layout;
  T->shard_rank = rank;
  T->shard_count = count;
  T->device = dst;
  T->streams.resize(whole->streams.size());
  uint64_t c0 = 0, c1 = 0;
  spb200_shard_chunks(whole->nnz_total, rank, count, &c0, &c1);
  int rc = SPLATT_SUCCESS;
  for (size_t i = 0; i < whole->streams.size() && rc == SPLATT_SUCCESS; ++i)
    rc = spb200_slice_stream(whole->streams[i], whole->device, c0, c1, dst, &T->streams[i]);
  cudaSetDevice(prev);
  if (rc != SPLATT_SUCCESS) { splatt_b200_tensor_free(T); return rc; }
  *out = T;
  return SPLATT_SUCCESS;
}

void splatt_b200_tensor_free(splatt_b200_tensor * t) {
  if (!t) return;
  int prev = 0;
  cudaGetDevice(&prev);
  if (prev != t->device) cudaSetDevice(t->device);
  for (auto & s : t->streams) spb200_free_stream(&s);
  if (t->cta_done) cudaFree(t->cta_done);
  if (prev != t->device) cudaSetDevice(prev);
  delete t;
}

int splatt_b200_tensor_info(splatt_b200_tensor const * t, int * nmodes, uint64_t * dims,
                            uint64_t * nnz_total, uint64_t * nnz_local, uint64_t * device_bytes) {
  if (!t) return SPLATT_ERROR_BADINPUT;
  if (nmodes) *nmodes = t->nmodes;
  if (dims) for (int m = 0; m < t->nmodes; ++m) dims[m] = t->dims[m];
  if (nnz_total) *nnz_total = t->nnz_total;
  if (nnz_local) *nnz_local = t->streams.empty() ? 0 : t->streams[0].nrec;
  if (device_bytes) {
    uint64_t b = 0;
    for (auto & s : t->streams) b += s.bytes;
    *device_bytes = b;
  }
  return SPLATT_SUCCESS;
}

int splatt_b200_mode_info(splatt_b200_tensor const * t, int mode, int ncolumns, int * kind,
                          int * level_perm, uint64_t * nfibs, uint64_t * alg_bytes) {
  if (!t || mode < 0 || mode >= t->nmodes) return SPLATT_ERROR_BADINPUT;
  const ModePlan & p = t->plan[mode];
  const FiberStream & s = t->streams[p.stream];
  const int N = t->nmodes;
  if (kind) *kind = p.kind;
  if (level_perm) for (int l = 0; l < N; ++l) level_perm[l] = s.perm[l];
  if (nfibs) for (int l = 0; l < N; ++l) nfibs[l] = s.nnodes[l];
  if (alg_bytes) {
    // SURVEY.md 8(d): every array touched once, at the widths stored on device
    // (values 8 B, indices 4 B; fptr replaced by per-record flags that ride
    // in the index words, so the fptr term is the 4 B/nnz parent word).
    uint64_t b = s.nrec * sizeof(SpRec);
    for (int l = 0; l <= N - 3; ++l) b += s.nnodes[l] * 4;   // node counts are this shard's
    // root kernels of 4+-mode streams read the level-(N-3) id beside every record (4 B per
    // nonzero) instead of the up[N-3] node array
    if (p.kind == SPB200_KIND_ROOT && N >= 4) b += s.nrec * 4 - s.nnodes[N - 3] * 4;
    for (int m = 0; m < N; ++m) b += t->dims[m] * (uint64_t)ncolumns * 8;   // N-1 reads + 1 write
    *alg_bytes = b;
  }
  return SPLATT_SUCCESS;
}

int splatt_b200_mttkrp(splatt_b200_tensor const * t, int mode, int ncolumns, int ldm,
                       double const * const * d_mats, double * d_out, void * stream) {
  if (!t || !d_mats || !d_out || mode < 0 || mode >= t->nmodes) {
    fprintf(stderr, "SPLATT: splatt_b200_mttkrp: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  const ModePlan & p = t->plan[mode];
  DeviceGuard g(t->device);
  if (!g.ok) return SPLATT_ERROR_BADINPUT;
  return spb200_launch_mttkrp(t->streams[p.stream], p.kind, p.outdepth, ncolumns, ldm, d_mats,
                              d_out, t->dims[mode], static_cast<cudaStream_t>(stream));
}

int splatt_b200_mttkrp_f32(splatt_b200_tensor const * t, int mode, int ncolumns, int ldm,
                           float const * const * d_mats, float * d_out, void * stream) {
  if (!t || !d_mats || !d_out || mode < 0 || mode >= t->nmodes) {
    fprintf(stderr, "SPLATT: splatt_b200_mttkrp_f32: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  const ModePlan & p = t->plan[mode];
  DeviceGuard g(t->device);
  if (!g.ok) return SPLATT_ERROR_BADINPUT;
  return spb200_launch_mttkrp_f32(t->streams[p.stream], p.kind, p.outdepth, ncolumns, ldm, d_mats,
                                  d_out, t->dims[mode], static_cast<cudaStream_t>(stream));
}

int splatt_b200_mttkrp_columns(splatt_b200_tensor const * t, int mode, int ncolumns, int ldm,
                               double const * const * d_mats, double * d_out, int col_begin,
                               int col_count, void * stream) {
  if (!t || !d_mats || !d_out || mode < 0 || mode >= t->nmodes) {
    fprintf(stderr, "SPLATT: splatt_b200_mttkrp_columns: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  const ModePlan & p = t->plan[mode];
  DeviceGuard g(t->device);
  if (!g.ok) return SPLATT_ERROR_BADINPUT;
  return spb200_launch_mttkrp(t->streams[p.stream], p.kind, p.outdepth, ncolumns, ldm, d_mats,
                              d_out, t->dims[mode], static_cast<cudaStream_t>(stream), false,
                              col_begin, col_count);
}

int splatt_b200_mttkrp_multicast(splatt_b200_tensor const * t, int mode, int ncolumns, int ldm,
                                 double const * const * d_mats, double * mc_out, void * stream) {
  if (!t || !d_mats || !mc_out || mode < 0 || mode >= t->nmodes) {
    fprintf(stderr, "SPLATT: splatt_b200_mttkrp_multicast: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  const ModePlan & p = t->plan[mode];
  DeviceGuard g(t->device);
  if (!g.ok) return SPLATT_ERROR_BADINPUT;
  return spb200_launch_mttkrp(t->streams[p.stream], p.kind, p.outdepth, ncolumns, ldm, d_mats,
                              mc_out, t->dims[mode], static_cast<cudaStream_t>(stream), true);
}

int splatt_b200_mttkrp_multicast_sync(splatt_b200_tensor const * t, int mode, int ncolumns, int ldm,
                                      double const * const * d_mats, double * mc_out,
                                      splatt_b200_group_sync const * sync, void * stream) {
  return splatt_b200_mttkrp_multicast_sync_columns(t, mode, ncolumns, ldm, d_mats, mc_out, 0, 0, sync,
                                                   stream);
}

int splatt_b200_mttkrp_multicast_sync_columns(splatt_b200_tensor const * t, int mode, int ncolumns,
                                              int ldm, double const * const * d_mats,
                                              double * mc_out, int col_begin, int col_count,
                                              splatt_b200_group_sync const * sync, void * stream) {
  if (!t || !d_mats || !mc_out || !sync || !sync->mc_flag || !sync->local_flag ||
      mode < 0 || mode >= t->nmodes) {
    fprintf(stderr, "SPLATT: splatt_b200_mttkrp_multicast_sync: bad arguments\n");
    return SPLATT_ERROR_BADINPUT;
  }
  const ModePlan & p = t->plan[mode];
  DeviceGuard g(t->device);
  if (!g.ok) return SPLATT_ERROR_BADINPUT;
  if (!t->cta_done) {
    // finished-CTA counter of the in-kernel barrier (zero between launches)
    splatt_b200_tensor * tm = const_cast<splatt_b200_tensor *>(t);
    SPB200_CUDA_OK(cudaMalloc(&tm->cta_done, 64));
    SPB200_CUDA_OK(cudaMemset(tm->cta_done, 0, 64));
    SPB200_CUDA_OK(cudaDeviceSynchronize());   // callers' streams do not synchronise with the null stream
  }
  GroupSync gs;
  gs.mc_flag = sync->mc_flag; gs.local_flag = sync->local_flag; gs.cta_done = t->cta_done;
  gs.target = sync->target;
  gs.rank = sync->rank; gs.world = sync->world;
  if (gs.world < 1 || gs.world > 64 || gs.rank >= gs.world) {
    fprintf(stderr, "SPLATT: splatt_b200_mttkrp_multicast_sync: bad rank/world (%u/%u)\n", gs.rank, gs.world);
    return SPLATT_ERROR_BADINPUT;
  }
  return spb200_launch_mttkrp(t->streams[p.stream], p.kind, p.outdepth, ncolumns, ldm, d_mats,
                              mc_out, t->dims[mode], static_cast<cudaStream_t>(stream), true,
                              col_begin, col_count, &gs);
}

int splatt_b200_csf_alloc(int nmodes, uint64_t const * dims, uint64_t nnz,
                          uint32_t const * const * ind, double const * vals, int on_device,
                          int csf_alloc, splatt_csf ** out) {
  if (!out || !dims || nmodes < 2 || nmodes > SPB200_MAXN) return SPLATT_ERROR_BADINPUT;
  int perms[SPB200_MAXN][SPB200_MAXN];
  const int nc = spb200_csf_orders(dims, nmodes, csf_alloc, perms);
  if (nc == 0) {
    fprintf(stderr, "SPLATT: CSF type '%d' not recognized.\n", csf_alloc);
    return SPLATT_ERROR_BADINPUT;
  }
  DevCoo dc;
  int rc = upload_coo(nmodes, nnz, ind, vals, on_device, &dc);
  if (rc != SPLATT_SUCCESS) return rc;
  splatt_csf * csf = static_cast<splatt_csf *>(calloc(nc, sizeof(splatt_csf)));
  if (!csf) return SPLATT_ERROR_NOMEMORY;
  for (int c = 0; c < nc; ++c) {
    rc = spb200_build_host_csf(nmodes, dims, nnz, dc.ind, dc.vals, perms[c], &csf[c]);
    if (rc != SPLATT_SUCCESS) { splatt_b200_csf_free(csf, csf_alloc); return rc; }
  }
  *out = csf;
  return SPLATT_SUCCESS;
}

void splatt_b200_csf_free(splatt_csf * csf, int csf_alloc) {
  if (!csf) return;
  int nc = 1;
  if (csf_alloc == SPLATT_CSF_TWOMODE) nc = 2;
  else if (csf_alloc == SPLATT_CSF_ALLMODE) nc = (int)csf[0].nmodes;
  for (int c = 0; c < nc; ++c) {
    if (!csf[c].pt) continue;
    for (uint64_t t = 0; t < csf[c].ntiles; ++t) {
      free(csf[c].pt[t].vals);
      for (int l = 0; l < SPB200_MAXN; ++l) {
        free(csf[c].pt[t].fptr[l]);
        free(csf[c].pt[t].fids[l]);
      }
    }
    free(csf[c].pt);
  }
  free(csf);
}

int splatt_b200_cta_tiling(int nmodes, uint64_t const * dims, int const * perm,
                           uint64_t nnz_local, int shard_count, int root_only, int num_sms,
                           int force, uint32_t * tile_rows, uint32_t * acc_rows) {
  if (tile_rows) *tile_rows = 0;
  if (acc_rows) *acc_rows = 0;
  if (!dims || !perm || !tile_rows || !acc_rows || nmodes != 3 || num_sms < 1 || nnz_local == 0)
    return 0;
  const uint64_t root_dim = dims[perm[0]], leaf_dim = dims[perm[nmodes - 1]];
  // root rows one range (1 / num_sms of the records) spans if roots are spread evenly, plus
  // a margin; the build checks the real spans and drops the tiling when one does not fit
  const uint64_t slices = std::max<uint64_t>(1, std::min(root_dim, nnz_local));
  uint64_t acc = (root_dim + num_sms - 1) / num_sms;
  acc += acc / 4 + 8;
  if (force) acc = std::max<uint64_t>(acc, std::min<uint64_t>(root_dim, 256));
  if (acc > 0xffffu) return 0;
  const uint32_t rows = spb200_tiled_rows_for((uint32_t)acc);
  if (force) {
    if (rows < 1) return 0;
  } else {
    const double reuse = (double)nnz_local / num_sms / (double)std::max<uint64_t>(leaf_dim, 1);
    const uint64_t ntiles = (leaf_dim + std::max<uint32_t>(rows, 1) - 1) / std::max<uint32_t>(rows, 1);
    const double per_piece = (double)nnz_local / (double)slices / (double)ntiles;
    if (shard_count > 1 || !root_only || rows < 16 || leaf_dim <= rows || reuse < 3.0 ||
        nnz_local < (uint64_t)num_sms * 4096 || per_piece < SPB200_MIN_NNZ_PER_PIECE)
      return 0;
  }
  *tile_rows = rows;
  *acc_rows = (uint32_t)acc;
  return 1;
}

int splatt_b200_level_orders(uint64_t const * dims, int nmodes, int csf_alloc, int * perms,
                             int * mode_csf_map) {
  if (!dims || nmodes < 1 || nmodes > SPB200_MAXN) return 0;
  int p[SPB200_MAXN][SPB200_MAXN];
  const int nc = spb200_csf_orders(dims, nmodes, csf_alloc, p);
  if (nc == 0) return 0;
  if (perms)
    for (int c = 0; c < nc; ++c)
      for (int l = 0; l < SPB200_MAXN; ++l) perms[c * SPB200_MAXN + l] = l < nmodes ? p[c][l] : 0;
  if (mode_csf_map) spb200_mode_csf_map(nmodes, csf_alloc, p[0], mode_csf_map);
  return nc;
}

int splatt_b200_csf_to_coo(splatt_csf const * csf, uint32_t ** ind, double * vals) {
  if (!csf || !ind || !vals) return SPLATT_ERROR_BADINPUT;
  const int N = (int)csf->nmodes;
  std::vector<uint32_t> iv[SPB200_MAXN];
  std::vector<double> vv;
  const int rc = csf_to_coo(csf, iv, &vv);
  if (rc != SPLATT_SUCCESS) return rc;
  for (int m = 0; m < N; ++m) memcpy(ind[m], iv[m].data(), csf->nnz * sizeof(uint32_t));
  memcpy(vals, vv.data(), csf->nnz * sizeof(double));
  return SPLATT_SUCCESS;
}

void splatt_b200_shard_range(uint64_t nnz, int rank, int count_shards, uint64_t * first,
                             uint64_t * count) {
  uint64_t c0, c1;
  spb200_shard_chunks(nnz, rank, count_shards, &c0, &c1);
  const uint64_t r0 = c0 * SPB200_CHUNK;
  uint64_t r1 = c1 * SPB200_CHUNK;
  if (r1 > nnz) r1 = nnz;
  if (first) *first = r0;
  if (count) *count = r1 > r0 ? r1 - r0 : 0;
}

uint64_t splatt_b200_launch_count(void) { return g_spb200_launches; }
uint64_t splatt_b200_build_count(void) { return g_spb200_builds; }

char const * splatt_b200_version(void) { return "splatt_b200 0.1 (sm_90a fiber-stream MTTKRP)"; }

}  // extern "C"
