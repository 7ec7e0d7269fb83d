// Shared declarations of the splatt_b200 engine (host side + kernel arguments).
//
// Data layout in HBM -- the "fiber stream"
// ----------------------------------------
// A CSF tensor with level order perm[0..N-1] (root .. leaf; reference:
// include/splatt/structs.h:76-114) is stored as a linearised tree:
//
//   rec[n]     one 16-byte record per nonzero, in CSF (lexicographic) order:
//                { double v; uint32 k; uint32 aux }
//                k   = leaf index (mode perm[N-1])
//                aux = parent index (mode perm[N-2]) in bits 0..28,
//                      close count c in bits 29..31: how many ancestor levels
//                      END after this nonzero (c>=1: the level-(N-2) fiber
//                      ends, c>=2: its level-(N-3) parent ends too, ...,
//                      c==N-1: the root slice ends).  This replaces the
//                      reference's fptr[] arrays: the tree is walked by
//                      counting, never by pointer chasing.
//   up[l][f]   uint32 index (mode perm[l]) of node f at level l, l = 0..N-3
//                (the reference's fids[l], always materialised for l = 0).
//   anc[n]     (N >= 4 only) uint32 index (mode perm[N-3]) of record n's level-(N-3)
//                ancestor: the root kernel gathers that row whenever c >= 2 without
//                first fetching an id from up[N-3] (no dependent load chain).
//   desc[c][l] for every chunk of SPB200_CHUNK records, the node number at
//                level l (l = 0..N-3) that contains the chunk's first record,
//                so any chunk boundary is a legal place to start a traversal.
//
// Everything a traversal needs arrives as three perfectly sequential streams
// (rec, up[*], desc); the only random accesses are the factor-row gathers.
#pragma once
#include <cstdint>
#include <cstddef>
#include <cstdio>
#include <vector>
#include <cuda_runtime.h>
#include "../../include/splatt_b200.h"

#define SPB200_MAXN 8
#define SPB200_CHUNK 64u             // records per descriptor chunk
#define SPB200_IDX_BITS 29           // parent index bits in rec.aux
#define SPB200_IDX_MASK 0x1fffffffu
// CTA tiling pays only when a (root slice, leaf tile) piece holds this many nonzeros on
// average: every piece ends a slice partial sum and splits fibers
#define SPB200_MIN_NNZ_PER_PIECE 8.0

struct __align__(16) SpRec {
  double   v;
  uint32_t k;
  uint32_t aux;
};
static_assert(sizeof(SpRec) == 16, "record must be 16 bytes");

// One sorted stream, device resident (a shard holds a contiguous chunk range).
struct FiberStream {
  int      nmodes = 0;
  int      perm[SPB200_MAXN] = {0};       // level -> mode
  uint64_t nrec = 0;                       // records held (local)
  uint64_t nrec_total = 0;                 // records in the whole tensor
  uint64_t nnodes[SPB200_MAXN] = {0};     // nodes per level (of the records held)
  SpRec *    rec = nullptr;
  uint32_t * up[SPB200_MAXN] = {nullptr}; // levels 0..N-3 (of the records held)
  uint32_t * anc = nullptr;                // N >= 4: level-(N-3) index of every record (padded to 16 B)
  uint32_t * desc = nullptr;               // local chunks x (N-2)
  uint64_t nchunks = 0;                    // local chunks
  size_t   bytes = 0;                      // HBM held
  uint32_t ktile_rows = 0;                 // >0: leaf-tile re-ordered (rows per tile)
  uint32_t kranges = 0;                    //     ... inside this many chunk-aligned ranges
  // CTA-tiled variant (one range per CTA, leaf tile staged in shared memory):
  uint32_t * seg_off = nullptr;            // [kranges * ntiles + 1] first record of every segment
  uint32_t * rootid = nullptr;             // [nrec] root index of every record
  uint32_t * rroot = nullptr;              // [2 * kranges] first / last root index of every range
  uint32_t ntiles = 0;
  uint32_t acc_rows = 0;                   // rows of the kernel's shared accumulator
  uint64_t leaf_rows = 0;                  // rows of the leaf-mode factor
};

// Leaf-tile re-ordering request for spb200_build_stream (tile_rows == 0: off).
struct StreamTiling {
  uint32_t tile_rows = 0;
  uint32_t nranges = 0;
  bool     cta = false;      // build seg_off / rootid / rroot for the shared-memory tile kernel
  uint32_t acc_rows = 0;     // cta: root rows the kernel can accumulate per range
};

enum { SPB200_KIND_ROOT = 0, SPB200_KIND_INTL = 1, SPB200_KIND_LEAF = 2 };

struct ModePlan {
  int stream = -1;
  int kind = SPB200_KIND_ROOT;
  int outdepth = 0;
};

struct splatt_b200_tensor {
  int      nmodes = 0;
  uint64_t dims[SPB200_MAXN] = {0};
  uint64_t nnz_total = 0;
  int      device = 0;
  int      layout = 0;
  int      shard_rank = 0, shard_count = 1;
  std::vector<FiberStream> streams;
  ModePlan plan[SPB200_MAXN];
  uint32_t * cta_done = nullptr;   // scratch of the in-kernel group barrier (lazily allocated)
};

// Run on the tensor's device, restore the caller's afterwards.
struct DeviceGuard {
  int prev = -1, want = -1;
  bool ok = true;
  explicit DeviceGuard(int dev) : want(dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) { ok = false; return; }
    if (prev != want && cudaSetDevice(want) != cudaSuccess) {
      fprintf(stderr, "SPLATT: cannot switch to CUDA device %d\n", want);
      ok = false;
    }
  }
  ~DeviceGuard() { if (ok && prev != want) cudaSetDevice(prev); }
};

// Kernel argument block (passed by value).
struct MttkrpArgs {
  const SpRec *    rec;
  const uint32_t * up[SPB200_MAXN - 2];
  const uint32_t * desc;
  const uint32_t * anc;                 // N >= 4 root kernels: level-(N-3) index per record
  const void *     mats[SPB200_MAXN];   // by LEVEL: factor of mode perm[l] (the kernel's value type)
  void *           out;
  unsigned long long nrec;
  unsigned int     nchunks;
  int              ldm;       // leading dimension of every matrix (elements; 16 B multiple)
  int              ncols;     // active columns in this launch (16 B multiple, <= L * 16 B)
  int              col0;      // first column of this launch
  int              outdepth;  // level of the output mode
  int              ktiled;    // stream is leaf-tile ordered: keep non-leaf gathers out of L1
  int              multicast; // `out` is an NVLink multicast address: reduce with multimem.red
  int              rpad, apad; // shared-memory stagger: pad records / pad ids per group region (0 = none)
  int              mc_store;   // multicast launches: rows owned by one lane group are stored, not reduced
  // Group barrier folded into the kernel's tail (multicast launches only; null = off):
  // after its last row reduction every CTA fences at system scope; the last CTA to finish
  // stores sync_target (the barrier's sequence number) into THIS GPU's slot of the group's
  // flag array on EVERY GPU (multimem.st on sync_mc + sync_rank) and spins on this GPU's copy
  // until all sync_world slots have reached it.  When the kernel exits, every peer's
  // reductions have landed in this GPU's output buffer.
  uint32_t *       sync_mc;
  uint32_t *       sync_local;
  uint32_t *       sync_cta;   // this GPU's finished-CTA counter (device memory, starts at 0)
  uint32_t         sync_target;
  uint32_t         sync_rank, sync_world;
};

// Host-side description of the group barrier (see MttkrpArgs).
struct GroupSync {
  uint32_t * mc_flag = nullptr;
  uint32_t * local_flag = nullptr;
  uint32_t * cta_done = nullptr;
  uint32_t   target = 0;
  uint32_t   rank = 0, world = 1;
};

#define SPB200_CUDA_OK(call)                                                   \
  do {                                                                         \
    cudaError_t e_ = (call);                                                   \
    if (e_ != cudaSuccess) {                                                   \
      fprintf(stderr, "SPLATT: CUDA error '%s' at %s:%d (%s)\n",               \
              cudaGetErrorString(e_), __FILE__, __LINE__, #call);              \
      return (e_ == cudaErrorMemoryAllocation) ? SPLATT_ERROR_NOMEMORY         \
                                               : SPLATT_ERROR_BADINPUT;        \
    }                                                                          \
  } while (0)

void spb200_shard_chunks(uint64_t nnz, int rank, int nshards, uint64_t * c0, uint64_t * c1);

// stream_build.cu -----------------------------------------------------------
// Build one stream from device COO (ind[m] uint32[nnz], vals) in level order
// `perm`.  If `presorted`, the input is already lexicographically sorted in
// that order.  Keeps only this shard's chunk range.
int spb200_build_stream(int nmodes, const uint64_t * dims, uint64_t nnz,
                        const uint32_t * const * d_ind, const double * d_vals,
                        const int * perm, bool presorted,
                        int shard_rank, int shard_count,
                        const StreamTiling & tiling, FiberStream * out);
void spb200_free_stream(FiberStream * s);
// Cut the chunk range [c0, c1) out of a WHOLE (unsharded, untiled) stream living on device
// `src_dev` into a stand-alone stream on device `dst_dev` (node numbers re-based): what a
// shard built by spb200_build_stream(shard_rank, shard_count) holds, without re-sorting.
int spb200_slice_stream(const FiberStream & whole, int src_dev, uint64_t c0, uint64_t c1,
                        int dst_dev, FiberStream * out);

// Host CSF arrays from device COO (for splatt_b200_csf_alloc).
int spb200_build_host_csf(int nmodes, const uint64_t * dims, uint64_t nnz,
                          const uint32_t * const * d_ind, const double * d_vals,
                          const int * perm, splatt_csf * csf);

// mttkrp_launch.cu ------------------------------------------------------------
int spb200_launch_mttkrp(const FiberStream & s, int kind, int outdepth,
                         int ncolumns, int ldm,
                         const double * const * d_mats_by_mode, double * d_out,
                         uint64_t out_rows, cudaStream_t stream, bool multicast_out = false,
                         int col_begin = 0, int col_count = 0, const GroupSync * sync = nullptr);
// The same in fp32 (factors and output float, records rounded to fp32, fp32 arithmetic): whole
// matrices only, never multicast, never the CTA-tiled kernel.  ldm % 4 == 0.
int spb200_launch_mttkrp_f32(const FiberStream & s, int kind, int outdepth, int ncolumns, int ldm,
                             const float * const * d_mats_by_mode, float * d_out,
                             uint64_t out_rows, cudaStream_t stream);
extern unsigned long long g_spb200_launches;
extern unsigned long long g_spb200_builds;     // fiber streams built (sort + scans) so far
inline void spb200_count_launches(unsigned n) { __atomic_fetch_add(&g_spb200_launches, n, __ATOMIC_RELAXED); }

// mttkrp_tiled.cu -- 3-mode root kernel with the leaf factor staged tile by tile in smem
bool spb200_tiled_applicable(const FiberStream & s, int kind);
// columns [col_begin, col_end) (even bounds) of the output
int spb200_launch_tiled_root3(const FiberStream & s, int ldm, int col_begin, int col_end,
                              const double * leaf, const double * parent, double * d_out,
                              cudaStream_t stream);
// rows of a leaf tile that fit the kernel's smem beside an accumulator of acc_rows rows
uint32_t spb200_tiled_rows_for(uint32_t acc_rows);

// cpd.cu -- row-partitioned ALS tail steps (multi-GPU engine).  Every device works on its own
// row slice; partial column norms / Grams go to per-device slots of the multicast region and
// are combined in device order on every device, so all replicas stay bit-identical.
struct splatt_b200_als_tail;
int spb200_tail_solve_norm_partial(splatt_b200_als_tail * h, int mode, const double * d_m1,
                                   double * d_x, uint64_t rows, int first_iteration,
                                   double * mc_norm_slot);
int spb200_tail_scale_gram_partial(splatt_b200_als_tail * h, double * d_x, double * mc_x,
                                   uint64_t rows, int first_iteration, const double * norms_all,
                                   int k, int norm_stride, double * mc_gram_slot);
int spb200_tail_gram_partial(splatt_b200_als_tail * h, const double * d_rows, uint64_t rows,
                             double * mc_gram_slot);
int spb200_tail_finish_gram(splatt_b200_als_tail * h, int mode, const double * grams_all, int k,
                            int gram_stride);
