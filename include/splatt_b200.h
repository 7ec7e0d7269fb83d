/*
 * splatt_b200.h -- C ABI of libsplatt_b200.so, the Hopper (H100, sm_90a) MTTKRP engine
 * that drops in behind SPLATT's MTTKRP / CPD-ALS entry points.
 *
 * Two groups of symbols:
 *
 *  (1) DROP-IN symbols.  Same names, argument meaning, ownership and return
 *      codes as the reference, so that a SPLATT build can link this library
 *      in place of src/mttkrp.c (+ src/cpd.c's driver).  Every declaration
 *      cites the reference declaration it replaces (paths relative to the
 *      ShadenSmith/splatt tree).  The struct layouts below are written to be
 *      binary compatible with the reference's default configuration
 *      (idx = uint64, val = double, SPLATT_MAX_NMODES = 8); tests/test_abi.py
 *      proves the offsets against ones recorded from the reference headers.
 *
 *  (2) ENGINE symbols (prefix splatt_b200_).  The device-resident interface:
 *      tensors live in HBM as per-mode "fiber streams", factor matrices and
 *      outputs are device pointers, and a call only enqueues kernels on a CUDA
 *      stream.  bench.py, the Python host layer and the multi-GPU path use
 *      these; the drop-in symbols are thin host-buffer wrappers around them.
 *
 * Plain pointers and sizes only; no C++ or torch types cross this boundary.
 */
#ifndef SPLATT_B200_H
#define SPLATT_B200_H

#include <stdint.h>
#include <stddef.h>
#include <stdbool.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------
 * Scalar types and constants (reference: include/splatt/types_config.h:38-89,
 * include/splatt/constants.h:14-16, default build widths cmake/types.cmake:3-4)
 * ---------------------------------------------------------------------- */
typedef uint64_t splatt_idx_t;
typedef double   splatt_val_t;

#ifndef SPLATT_MAX_NMODES
#define SPLATT_MAX_NMODES ((splatt_idx_t) 8)
#endif
#define SPLATT_B200_MAX_NMODES 8

/* Return codes (reference: include/splatt/types_config.h:129-137).
 * NOTE: success is 1, not 0. */
enum {
  SPLATT_SUCCESS        = 1,
  SPLATT_ERROR_BADINPUT = 2,
  SPLATT_ERROR_NOMEMORY = 3
};

/* Slots of the `double opts[]` array (reference:
 * include/splatt/types_config.h:103-123).  The order is ABI. */
enum {
  SPLATT_OPTION_NTHREADS   = 0,
  SPLATT_OPTION_TOLERANCE  = 1,
  SPLATT_OPTION_REGULARIZE = 2,
  SPLATT_OPTION_NITER      = 3,
  SPLATT_OPTION_VERBOSITY  = 4,
  SPLATT_OPTION_RANDSEED   = 5,
  SPLATT_OPTION_CSF_ALLOC  = 6,
  SPLATT_OPTION_TILE       = 7,
  SPLATT_OPTION_TILELEVEL  = 8,
  SPLATT_OPTION_PRIVTHRESH = 9,
  SPLATT_OPTION_DECOMP     = 10,
  SPLATT_OPTION_COMM       = 11,
  SPLATT_OPTION_NOPTIONS   = 12
};

/* reference: include/splatt/types_config.h:143-149 */
enum { SPLATT_VERBOSITY_NONE = 0, SPLATT_VERBOSITY_LOW, SPLATT_VERBOSITY_HIGH,
       SPLATT_VERBOSITY_MAX };
/* reference: include/splatt/types_config.h:155-162 */
typedef enum { SPLATT_NOTILE = 0, SPLATT_DENSETILE, SPLATT_SYNCTILE,
               SPLATT_COOPTILE } splatt_tile_type;
/* reference: include/splatt/types_config.h:168-173 */
typedef enum { SPLATT_CSF_ONEMODE = 0, SPLATT_CSF_TWOMODE,
               SPLATT_CSF_ALLMODE } splatt_csf_type;

/* ------------------------------------------------------------------------
 * Boundary structs.  Layout-compatible with the reference; field names kept
 * so reference-side code compiles against either header.
 * ---------------------------------------------------------------------- */

/* One tile's sparsity pattern (reference: include/splatt/structs.h:51-68).
 * Level l has nfibs[l] nodes; children of node f at level l are
 * fptr[l][f] .. fptr[l][f+1]-1 at level l+1; fids[l][f] is the node's index
 * in mode dim_perm[l].  fids[0] may be NULL (root ids are then 0..nfibs[0]-1,
 * reference: src/csf.c:303-309).  vals has nfibs[nmodes-1] entries. */
typedef struct
{
  splatt_idx_t   nfibs[SPLATT_B200_MAX_NMODES];
  splatt_idx_t * fptr [SPLATT_B200_MAX_NMODES];
  splatt_idx_t * fids [SPLATT_B200_MAX_NMODES];
  splatt_val_t * vals;
} csf_sparsity;

/* Compressed sparse fiber tensor (reference: include/splatt/structs.h:76-114). */
typedef struct splatt_csf
{
  splatt_idx_t nnz;
  splatt_idx_t nmodes;
  splatt_idx_t dims     [SPLATT_B200_MAX_NMODES];
  splatt_idx_t dim_perm [SPLATT_B200_MAX_NMODES];  /* level -> mode */
  splatt_idx_t dim_iperm[SPLATT_B200_MAX_NMODES];  /* mode  -> level */
  splatt_tile_type which_tile;
  splatt_idx_t ntiles;
  splatt_idx_t ntiled_modes;
  splatt_idx_t tile_dims[SPLATT_B200_MAX_NMODES];
  csf_sparsity * pt;                               /* ntiles entries */
} splatt_csf;

/* CPD output (reference: include/splatt/structs.h:26-45).  factors[m] and
 * lambda are malloc()-family memory released by splatt_free_kruskal. */
typedef struct splatt_kruskal
{
  splatt_idx_t   rank;
  splatt_val_t * factors[SPLATT_B200_MAX_NMODES];
  splatt_val_t * lambda;
  splatt_idx_t   nmodes;
  splatt_idx_t   dims[SPLATT_B200_MAX_NMODES];
  double         fit;
} splatt_kruskal;

/* MTTKRP workspace (reference: include/splatt/api_kernels.h:22-67).  Only ever
 * created by splatt_mttkrp_alloc_ws and handled by pointer, so this library
 * allocates a larger private object whose first member is this public struct;
 * the tail carries the device mirror (fiber streams, staging buffers, stream).
 * The CPU-only fields are filled with the values the reference would compute
 * where cheap (num_csf, mode_csf_map, num_threads) and NULL/false elsewhere. */
typedef struct
{
  splatt_idx_t   num_csf;
  splatt_idx_t   mode_csf_map[SPLATT_B200_MAX_NMODES];
  splatt_idx_t   num_threads;
  splatt_idx_t * tile_partition[SPLATT_B200_MAX_NMODES];
  splatt_idx_t * tree_partition[SPLATT_B200_MAX_NMODES];
  bool           is_privatized[SPLATT_B200_MAX_NMODES];
  splatt_val_t ** privatize_buffer;
  double         reduction_time;
} splatt_mttkrp_ws;

/* Dense matrix used by the internal entry point (reference: src/matrix.h:10-16). */
typedef struct
{
  splatt_idx_t   I;
  splatt_idx_t   J;
  splatt_val_t * vals;
  int            rowmajor;
} splatt_b200_matrix_t;   /* == reference matrix_t */

/* ------------------------------------------------------------------------
 * (1) DROP-IN symbols
 * ---------------------------------------------------------------------- */

/* MTTKRP of a CSF tensor with host factor matrices.
 * Replaces: include/splatt/api_kernels.h:98-104, src/mttkrp.c:1763-1811.
 *  mode      output mode;  ncolumns = rank R
 *  tensors   1, 2 or nmodes CSFs according to options[SPLATT_OPTION_CSF_ALLOC]
 *  matrices  matrices[m] is row-major dims[m] x ncolumns (host); matrices[mode]
 *            is never read and may alias matout
 *  matout    dims[mode] x ncolumns, fully overwritten
 * Returns SPLATT_SUCCESS (1), or SPLATT_ERROR_* with a "SPLATT:" line on stderr.
 * Like the reference it builds and destroys a workspace per call. */
int splatt_mttkrp(
    splatt_idx_t const mode,
    splatt_idx_t const ncolumns,
    splatt_csf const * const tensors,
    splatt_val_t ** matrices,
    splatt_val_t * const matout,
    double const * const options);

/* Replaces: include/splatt/api_kernels.h:107-110, src/mttkrp.c:1814-1912.
 * Builds the device mirror of `tensors` once (all HBM allocation happens here). */
splatt_mttkrp_ws * splatt_mttkrp_alloc_ws(
    splatt_csf const * const tensors,
    splatt_idx_t const ncolumns,
    double const * const options);

/* Replaces: include/splatt/api_kernels.h:118-119, src/mttkrp.c:1915-1928. */
void splatt_mttkrp_free_ws(
    splatt_mttkrp_ws * const ws);

/* The entry the reference's CPD driver, bench harness and tests call
 * (reference: src/mttkrp.h:19,35-41 `#define mttkrp_csf splatt_mttkrp_csf`,
 * src/mttkrp.c:1287-1341; call sites src/cpd.c:327, src/bench.c:191,
 * tests/mttkrp_test.c:75).  mats[m] are reference matrix_t*, the output is
 * mats[SPLATT_MAX_NMODES] whose I is reset to dims[mode]; `thds` (the CPU
 * per-thread scratch, src/thd_info.h:25-30) is accepted and ignored. */
void splatt_mttkrp_csf(
    splatt_csf const * const tensors,
    splatt_b200_matrix_t ** mats,
    splatt_idx_t const mode,
    void * const thds,
    splatt_mttkrp_ws * const ws,
    double const * const opts);

/* CPD-ALS with the MTTKRP on the GPU.
 * Replaces: include/splatt/api_factorization.h:41-45, src/cpd.c:22-63 and the
 * loop of src/cpd.c:271-387 (MTTKRP -> normal equations -> normalise -> Gram,
 * fit from the last mode's MTTKRP). */
int splatt_cpd_als(
    splatt_csf const * const tensors,
    splatt_idx_t const nfactors,
    double const * const options,
    splatt_kruskal * factored);

/* Replaces: include/splatt/api_kruskal.h:34-35, src/cpd.c:66-73. */
void splatt_free_kruskal(
    splatt_kruskal * factored);

/* Replaces: include/splatt/api_options.h (splatt_default_opts, src/opts.c:10-47;
 * splatt_free_opts src/opts.c:50-54).  Same defaults. */
double * splatt_default_opts(void);
void     splatt_free_opts(double * opts);


/* ------------------------------------------------------------------------
 * (2) ENGINE symbols -- device-resident interface
 * ---------------------------------------------------------------------- */

/* Opaque handle: a sparse tensor resident in HBM as fiber streams. */
typedef struct splatt_b200_tensor splatt_b200_tensor;

/* How MTTKRP modes map to device streams. */
enum {
  /* one root-oriented stream per mode (every mode runs the root kernel; uses
   * nmodes x 16 B/nnz of HBM).  Default. */
  SPLATT_B200_LAYOUT_ALLROOT = 0,
  /* mirror exactly the CSFs handed in (ONEMODE/TWOMODE/ALLMODE): modes that
   * are not a root of some CSF run the internal / leaf kernels (atomics). */
  SPLATT_B200_LAYOUT_ASGIVEN = 1
};

/* Build-time knobs; zero-initialise for defaults. */
typedef struct
{
  int32_t layout;        /* SPLATT_B200_LAYOUT_*                           */
  int32_t device;        /* CUDA device ordinal, -1 = current              */
  int32_t shard_rank;    /* this process's rank among shard_count          */
  int32_t shard_count;   /* 0/1 = whole tensor; >1 = keep only this rank's
                            nnz-balanced share of every stream             */
  int32_t verbosity;     /* SPLATT_VERBOSITY_*                             */
  int32_t ncolumns_hint; /* rank the tensor will be used with (0 = unknown);
                            not needed by the leaf-tiling policy            */
  int32_t ktile;         /* leaf-tile re-ordering: 0 = automatic (shared-
                            memory tiles where splatt_b200_cta_tiling says
                            so), -1 = off, > 0 = this many rows per tile    */
  int32_t reserved[9];
} splatt_b200_build_opts;

/* Mirror reference CSF(s) (host memory) into HBM.  `csf_alloc` says how many
 * CSFs `tensors` holds (SPLATT_CSF_*; reference: src/csf.c:770-814). */
int splatt_b200_tensor_from_csf(
    splatt_csf const * tensors,
    int csf_alloc,
    splatt_b200_build_opts const * bopts,
    splatt_b200_tensor ** out);

/* Build straight from coordinate data.  ind[m] has nnz entries (0-based);
 * pointers are host or device according to `on_device`. */
int splatt_b200_tensor_from_coo(
    int nmodes,
    uint64_t const * dims,
    uint64_t nnz,
    uint32_t const * const * ind,
    double const * vals,
    int on_device,
    int csf_alloc,
    splatt_b200_build_opts const * bopts,
    splatt_b200_tensor ** out);

void splatt_b200_tensor_free(splatt_b200_tensor * t);

/* Introspection: *nnz_local is what this shard holds. */
int splatt_b200_tensor_info(
    splatt_b200_tensor const * t,
    int * nmodes, uint64_t * dims, uint64_t * nnz_total, uint64_t * nnz_local,
    uint64_t * device_bytes);

/* Per-mode facts used for the roofline: kernel kind (0 root, 1 internal,
 * 2 leaf), level order, node counts per level, algorithmic bytes moved by
 * one launch at rank R (SURVEY.md section 8d formula at the widths stored). */
int splatt_b200_mode_info(
    splatt_b200_tensor const * t, int mode, int ncolumns,
    int * kind, int * level_perm, uint64_t * nfibs, uint64_t * alg_bytes);

/* Materialise a host splatt_csf array equal to what the reference's
 * csf_alloc would build from the same nonzeros (reference: src/csf.c:770-814,
 * :468-502; untiled only).  Arrays are malloc()ed; release with
 * splatt_b200_csf_free. */
int splatt_b200_csf_alloc(
    int nmodes, uint64_t const * dims, uint64_t nnz,
    uint32_t const * const * ind, double const * vals, int on_device,
    int csf_alloc, splatt_csf ** out);
void splatt_b200_csf_free(splatt_csf * csf, int csf_alloc);

/* Host logic, no GPU needed: the level orders csf_alloc would use for each CSF
 * of an allocation policy (perms: ncsf x SPLATT_B200_MAX_NMODES ints, row c =
 * level -> mode of CSF c; reference: csf_find_mode_order src/csf.c:694-726) and
 * the mode -> CSF map of the MTTKRP workspace (reference: src/mttkrp.c:1832-1861).
 * Returns the number of CSFs, 0 on a bad policy. */
int splatt_b200_level_orders(
    uint64_t const * dims, int nmodes, int csf_alloc, int * perms, int * mode_csf_map);

/* Host logic, no GPU needed: whether the stream with level order perm (root .. leaf) is built
 * CTA-tiled, i.e. multiplied at its root by the kernel that serves leaf-factor rows from
 * shared memory.  Needs 3 modes, an unsharded build, a stream whose every mode runs the
 * root kernel (root_only), leaf rows re-used >= 3x by one SM's nonzeros, enough nonzeros per
 * (root slice, leaf tile) piece, and an accumulator for a range's root rows that fits beside
 * the tiles.  force = 1 skips the performance rules (testing).  Returns 1 and the tile and
 * accumulator rows if so, 0 otherwise.  The build still falls back to an untiled stream when
 * a range spans more root rows than *acc_rows. */
int splatt_b200_cta_tiling(
    int nmodes, uint64_t const * dims, int const * perm, uint64_t nnz_local, int shard_count,
    int root_only, int num_sms, int force, uint32_t * tile_rows, uint32_t * acc_rows);

/* Host logic, no GPU needed: the records [first, first+count) of a sorted stream
 * of `nnz` nonzeros that shard `rank` of `count_shards` keeps (equal numbers of
 * 64-record chunks, so shares differ by at most one chunk; slices may be split
 * at a share boundary -- the all-reduce adds the two partial rows).  Plays the
 * role of the reference's per-thread slice partition (csf_partition_1d,
 * src/csf.c:854-872 -> partition_weighted, src/thread_partition.c:156-195) at
 * the granularity a GPU needs. */
void splatt_b200_shard_range(
    uint64_t nnz, int rank, int count_shards, uint64_t * first, uint64_t * count);

/* Host logic, no GPU needed: expand one CSF (any tiling) to coordinates in storage order --
 * the first step of mirroring a reference CSF to the device.  ind[m] (nnz uint32 each) and
 * vals (nnz doubles) are caller-allocated. */
int splatt_b200_csf_to_coo(splatt_csf const * csf, uint32_t ** ind, double * vals);

/* Enqueue one MTTKRP on `stream` (a cudaStream_t passed as void*; NULL =
 * default stream).  d_mats[m] are DEVICE pointers, row-major with leading
 * dimension ldm (>= ncolumns, even so rows are 16-byte aligned); d_mats[mode]
 * is ignored.  d_out (dims[mode] x ldm) is zeroed and then accumulated into.
 * No host synchronisation.  Sharded tensors produce a partial sum that the
 * caller all-reduces (NCCL). */
int splatt_b200_mttkrp(
    splatt_b200_tensor const * t,
    int mode,
    int ncolumns,
    int ldm,
    double const * const * d_mats,
    double * d_out,
    void * stream);

/* Single precision: the same product with float factors and a float output, for callers whose
 * factors are fp32 (e.g. PyTorch defaults).  Every nonzero's value is rounded to fp32 once
 * and products and sums are formed in fp32; the tensor is the one splatt_b200_mttkrp uses
 * (no rebuild).  Contract as splatt_b200_mttkrp -- d_out zeroed, then accumulated into;
 * sharded tensors give partial sums; no host synchronisation; d_mats[mode] ignored -- except
 * the alignment rules: ldm % 4 == 0, ldm >= (ncolumns + 3) & ~3, and every base pointer
 * 16-byte aligned.  A violation returns SPLATT_ERROR_BADINPUT and writes nothing.
 * Columns [(ncolumns + 3) & ~3, ldm) of d_out are left zero; [ncolumns, (ncolumns + 3) & ~3)
 * are unspecified.  The f32 reductions flush subnormal sums to zero. */
int splatt_b200_mttkrp_f32(
    splatt_b200_tensor const * t,
    int mode,
    int ncolumns,
    int ldm,
    float const * const * d_mats,
    float * d_out,
    void * stream);

/* The same for a block of columns only: [col_begin, col_begin + col_count) (col_begin even).
 * MTTKRP is independent per column, so a caller can pipeline column blocks against the
 * PCIe copies of the corresponding factor columns (the drop-in symbols do exactly that
 * when the host buffers are page-locked).  Only those columns of d_out are zeroed/written;
 * an odd col_count also zeroes and writes the one column after the block, so the block must
 * end at or before the padded rank ncolumns + (ncolumns & 1).  A block with an odd
 * col_begin, col_begin past the padded rank or col_begin + col_count > ncolumns +
 * (ncolumns & 1) returns SPLATT_ERROR_BADINPUT and writes nothing. */
int splatt_b200_mttkrp_columns(
    splatt_b200_tensor const * t,
    int mode,
    int ncolumns,
    int ldm,
    double const * const * d_mats,
    double * d_out,
    int col_begin,
    int col_count,
    void * stream);

/* Fused MTTKRP + exchange for sharded tensors on one NVSwitch domain.  `mc_out` is
 * an NVLink MULTICAST address (CUDA multicast object / torch symmetric memory
 * `multicast_ptr`) bound to one dims[mode] x ldm buffer on every GPU of the
 * group.  The kernel puts every finished output row into ALL the buffers as it
 * goes -- `multimem.red.add.f64` for rows that several lane groups or GPUs
 * contribute to, a plain 128-bit store to the multicast address for rows one lane
 * group finishes alone (SPLATT_B200_MC_STORE=0: reductions only) -- so the per-mode
 * all-reduce of the north star happens inside the MTTKRP kernel instead of after
 * it.  Contract: every rank zeroes its own buffer and the group synchronises BEFORE
 * the call (the call does NOT accumulate into what the buffers held); after the
 * call the group synchronises once more and every buffer holds the full sum.
 * Requires the ALLROOT layout (root kernels).  Not zeroed, not synchronised here. */
int splatt_b200_mttkrp_multicast(
    splatt_b200_tensor const * t,
    int mode,
    int ncolumns,
    int ldm,
    double const * const * d_mats,
    double * mc_out,
    void * stream);

/* The same with the group barrier folded into the kernel's tail (no separate barrier
 * launch).  The group owns an array of `world` (<= 64) uint32 flags in its symmetric /
 * multicast memory, zero before first use: `sync->mc_flag` is the array's multicast address,
 * `sync->local_flag` this GPU's own address of it.  `sync->target` is the barrier's sequence
 * number (1, 2, 3, ... -- the caller counts; every GPU of the group passes the same number),
 * `rank` / `world` this GPU's slot and the group size.  The last CTA of the kernel stores the
 * number into its slot on every GPU and waits until all slots of the local copy hold it; when
 * the kernel completes on a GPU, every peer's reductions have landed in that GPU's buffer.
 * All GPUs of the group must launch (an empty shard too). */
typedef struct
{
  uint32_t * mc_flag;
  uint32_t * local_flag;
  uint32_t   target;
  uint32_t   rank;
  uint32_t   world;
  uint32_t   reserved;
} splatt_b200_group_sync;
int splatt_b200_mttkrp_multicast_sync(
    splatt_b200_tensor const * t,
    int mode,
    int ncolumns,
    int ldm,
    double const * const * d_mats,
    double * mc_out,
    splatt_b200_group_sync const * sync,
    void * stream);

/* ... for a block of columns only ([col_begin, col_begin + col_count), col_begin even;
 * col_count <= 0: all columns): lets a host pipeline column blocks against the PCIe copies of
 * the factor columns while the exchange stays fused (the multi-GPU engine's host-buffer call). */
int splatt_b200_mttkrp_multicast_sync_columns(
    splatt_b200_tensor const * t,
    int mode,
    int ncolumns,
    int ldm,
    double const * const * d_mats,
    double * mc_out,
    int col_begin,
    int col_count,
    splatt_b200_group_sync const * sync,
    void * stream);

/* Cut shard `rank` of `count` out of a WHOLE device tensor (built with shard_count <= 1)
 * onto CUDA device `device` (-1 = the whole tensor's device): the same equal-nnz chunk
 * range splatt_b200_shard_range names, copied device-to-device (P2P) instead of being
 * re-sorted on every GPU.  Used by the single-process multi-GPU engine. */
int splatt_b200_tensor_shard(
    splatt_b200_tensor const * whole, int rank, int count, int device,
    splatt_b200_tensor ** out);

/* ---- Single-process multi-GPU engine (multi.cu) ------------------------------------
 * One host process drives `ndevices` GPUs of one NVSwitch box: the reference's
 * distributed driver for one node (mpi_cpd_als_iterate, src/mpi/mpi_cpd.c:627-804; the
 * per-mode reduction :250-308) behind the unchanged C API.  The drop-in symbols use it
 * when the environment says so:
 *     SPLATT_B200_NGPUS=k            devices 0..k-1
 *     SPLATT_B200_DEVICES=0,2,5      an explicit list
 * (splatt_cpd_als, splatt_mttkrp_alloc_ws/_csf and splatt_mttkrp then run on all of
 * them).  The tensor is built once on the first device, cut into equal-nnz shares that
 * move device-to-device; the per-mode sum over devices happens inside the MTTKRP kernel
 * through an NVLink multicast mapping (CUDA driver multicast objects) with the group
 * barrier in the kernel's tail; without multicast support a peer-memory reduce kernel
 * ordered by CUDA events takes over (SPLATT_B200_MULTICAST=0 forces that path). */
typedef struct splatt_b200_multi splatt_b200_multi;
int  splatt_b200_multi_env_devices(int * devices, int cap);   /* parsed env, 0 = single GPU */
int  splatt_b200_multi_create(splatt_csf const * tensors, int csf_alloc, int ncolumns,
                              int const * devices, int ndevices, int verbosity,
                              splatt_b200_multi ** out);
void splatt_b200_multi_free(splatt_b200_multi * h);
int  splatt_b200_multi_info(splatt_b200_multi const * h, int * ndevices, int * multicast,
                            uint64_t * nnz_local, uint64_t * device_bytes);
/* MTTKRP of `mode` with HOST matrices (row-major dims[m] x ncolumns; mats[mode] ignored):
 * factors go to every device, result comes back as one row slice per device. */
int  splatt_b200_multi_mttkrp_host(splatt_b200_multi * h, int mode,
                                   double const * const * mats, double * out_host);
/* CPD-ALS over all devices; same contract as splatt_cpd_als (`tensors` only supplies the
 * Frobenius norm for the fit). */
int  splatt_b200_multi_cpd_als(splatt_b200_multi * h, splatt_csf const * tensors,
                               double const * options, splatt_kruskal * factored);
double splatt_b200_multi_last_ms(splatt_b200_multi const * h);

/* The dense tail of one ALS mode update on the device -- the kernels splatt_cpd_als uses --
 * as separate entry points, so a multi-GPU driver can interleave them with its exchange:
 *   local MTTKRP (shard) -> sum over ranks -> splatt_b200_als_tail_update (replicated).
 * Replaces, per call: mat_solve_normals src/matrix.c:529-606, mat_normalize :501-525,
 * mat_aTa :414-455, p_calc_fit src/cpd.c:237-265.  All matrices are device pointers with
 * leading dimension ldm; work is enqueued on the stream given at creation. */
typedef struct splatt_b200_als_tail splatt_b200_als_tail;
int  splatt_b200_als_tail_create(int nmodes, int ncolumns, int ldm, void * stream,
                                 splatt_b200_als_tail ** out);
void splatt_b200_als_tail_free(splatt_b200_als_tail * h);
int  splatt_b200_als_tail_gram(splatt_b200_als_tail * h, int mode, double const * d_factor,
                               uint64_t rows);
int  splatt_b200_als_tail_update(splatt_b200_als_tail * h, int mode, double const * d_m1,
                                 double * d_factor, uint64_t rows, int first_iteration);
int  splatt_b200_als_tail_fit(splatt_b200_als_tail * h, double const * d_last_factor,
                              double const * d_last_m1, uint64_t rows, double ttnormsq,
                              double * fit_out, double * lambda_out);
/* The same three steps with fp32 factors and an fp32 M1 (the output of splatt_b200_mttkrp_f32),
 * on the same handle.  Grams, the normal matrix, its Cholesky factor or pseudo-inverse, lambda,
 * the fit's inner product and the fit stay fp64; each row is solved in fp64 from its fp32 values
 * and rounded to fp32 once, and the column scaling is done in fp64 and rounded once.  Columns
 * [ncolumns, ldm) of d_m1 never feed the results (they may hold anything, NaN included; the
 * row solve loads whole float4 groups and discards those columns by selection), and columns
 * [ncolumns, ldm) of d_factor are never written.  Needs a handle created with ldm % 4 == 0 and
 * 16-byte aligned matrices; otherwise SPLATT_ERROR_BADINPUT and nothing is enqueued. */
int  splatt_b200_als_tail_gram_f32(splatt_b200_als_tail * h, int mode, float const * d_factor,
                                   uint64_t rows);
int  splatt_b200_als_tail_update_f32(splatt_b200_als_tail * h, int mode, float const * d_m1,
                                     float * d_factor, uint64_t rows, int first_iteration);
int  splatt_b200_als_tail_fit_f32(splatt_b200_als_tail * h, float const * d_last_factor,
                                  float const * d_last_m1, uint64_t rows, double ttnormsq,
                                  double * fit_out, double * lambda_out);

/* CPD-ALS of a device-resident tensor from device-resident factors (no host CSF, no host
 * factors): the iteration of splatt_cpd_als with the dense tail on the device, then its
 * post-processing.
 *   d_factors[m]  dims[m] x ldm, row-major, in/out.  On entry the caller's initial factors; on
 *                 return the 2-normalised factors.  Columns [ncolumns, ldm) never feed the
 *                 results and are never written (they may be read: the MTTKRP loads rows in
 *                 16-byte groups, up to column (ncolumns + 3) & ~3 in fp32).
 *   lambda_out    ncolumns host doubles: the weights (may be NULL).
 *   fit_out       the fit of the last iteration (may be NULL).
 *   iterations_out the number of iterations run (may be NULL).
 * Reads options[SPLATT_OPTION_NITER], [SPLATT_OPTION_TOLERANCE] and [SPLATT_OPTION_VERBOSITY]
 * and stops as splatt_cpd_als does: after NITER iterations, at fit == 1, or when the fit moved
 * by less than TOLERANCE (from the second iteration on).  ||X||^2 is summed from the tensor's
 * own values.  Runs on t->device and enqueues on `stream` (a cudaStream_t; NULL = default
 * stream); synchronises the stream once before the first iteration (||X||^2), once per
 * iteration (the fit) and once at the end.
 * Input rules: 1 <= ncolumns <= 128; fp64: ldm even and >= ncolumns; fp32: ldm % 4 == 0 and
 * ldm >= (ncolumns + 3) & ~3; every d_factors[m] 16-byte aligned; the tensor is whole (built
 * with shard_count <= 1: a shard's values are only a part of ||X||^2).  A violation returns
 * SPLATT_ERROR_BADINPUT before anything is enqueued, and the factors are left untouched.
 * _f32: factors and MTTKRP in fp32 (splatt_b200_mttkrp_f32), the dense tail as in
 * splatt_b200_als_tail_update_f32.  The fit's inner product <X,K> is formed from the fp32
 * MTTKRP result, and the fit 1 - sqrt(||X||^2 + ||K||^2 - 2<X,K>) / ||X|| cancels digits as it
 * approaches 1: there it is resolved only to about sqrt(2 eps) for a relative error eps in <X,K>
 * (about 1e-4 on a dense 30^3 tensor of exact rank 3, where fp64 reaches 1.0).  Near such a fit
 * the fp32 fit moves by about that much from one iteration to the next, so a TOLERANCE below it
 * may never stop the run before NITER. */
int splatt_b200_cpd_als_device(splatt_b200_tensor const * t, int ncolumns, int ldm,
                               double const * options, double * const * d_factors,
                               double * lambda_out, double * fit_out, int * iterations_out,
                               void * stream);
int splatt_b200_cpd_als_device_f32(splatt_b200_tensor const * t, int ncolumns, int ldm,
                                   double const * options, float * const * d_factors,
                                   double * lambda_out, double * fit_out, int * iterations_out,
                                   void * stream);

/* Nonnegative CPD of a device-resident tensor by HALS (hierarchical ALS: Cichocki & Phan 2009,
 * Gillis & Glineur 2012).  The model is K = sum_r lambda_r a_r^(0) o ... o a_r^(N-1) with
 * nonnegative factors whose columns have 2-norm 1 and lambda >= 0; the call minimises
 * 1/2 ||X - K||^2 over the stored entries, unstored entries read as zeros (as CPD-ALS does).
 * Tensor values may have any sign: the constraint is on the factors.
 *   Start: the caller's factors, columns [0, ncolumns).  Every column is 2-normalised and lambda
 *     is the product of the norms; then the Grams are formed.
 *   One iteration, for n = 0 .. N-1:
 *     M = the MTTKRP of mode n;  G = the Hadamard product of the other modes' Grams;
 *     B = A_n diag(lambda);  one Gauss-Seidel sweep over the columns r = 0 .. R-1,
 *       B[:, r] <- max(eps, (M[:, r] - sum_{j != r} B[:, j] G[j, r]) / G[r, r])
 *     (columns j < r already hold their new values);  lambda = the column 2-norms of B,
 *     A_n = B diag(1 / lambda) (always the 2-norm), and the Gram of A_n.
 *   The floor eps = 1e-16 is applied in fp64.  It keeps every column nonzero, so after the
 *   normalisation every G[r, r] is 1 up to rounding.  The division by G[r, r] is computed as a
 *   product with its reciprocal.
 * Fit, stopping and verbosity are those of splatt_b200_cpd_als_device: the fit
 * 1 - sqrt(||X||^2 + ||K||^2 - 2<X,K>) / ||X|| is formed from the last mode's M, and the run stops
 * after NITER iterations, at fit == 1, or when the fit moved by less than TOLERANCE (from the
 * second iteration on).
 *   d_factors[m]  in/out: the start on entry; on return the loop's factors as they stand (already
 *                 2-normalised, no post-processing).  Columns [ncolumns, ldm) are never written
 *                 and never feed the results.
 *   lambda_out, fit_out, iterations_out: as for splatt_b200_cpd_als_device (each may be NULL).
 *   history       NULL, or room for NITER doubles: the fit of every iteration run.
 * Input rules: those of splatt_b200_cpd_als_device; in addition every start entry in columns
 * [0, ncolumns) must be finite and >= 0, and every start column must have a positive, finite sum
 * of squares (so a nonzero entry; the sums are formed in fp64).  The start is checked on the
 * device before anything is written; a violation returns SPLATT_ERROR_BADINPUT and leaves the
 * factors bit-identical.  Synchronises the stream as splatt_b200_cpd_als_device does, and once
 * more for the start check.
 * _f32: fp32 factors and MTTKRP (splatt_b200_mttkrp_f32); G, the sweep's arithmetic, lambda and the
 * fit are fp64, and each swept row is rounded to fp32 once.  The fp32 fit resolves only about
 * 1e-4 near 1, as described for splatt_b200_cpd_als_device_f32. */
int splatt_b200_cpd_nonneg_device(splatt_b200_tensor const * t, int ncolumns, int ldm,
                                  double const * options, double * const * d_factors,
                                  double * lambda_out, double * fit_out, int * iterations_out,
                                  double * history, void * stream);
int splatt_b200_cpd_nonneg_device_f32(splatt_b200_tensor const * t, int ncolumns, int ldm,
                                      double const * options, float * const * d_factors,
                                      double * lambda_out, double * fit_out, int * iterations_out,
                                      double * history, void * stream);

/* Sum over the tensor's nonzeros of (v - sum_r lambda_r prod_m U_m[i_m, r])^2: the residual of a
 * Kruskal model at the stored entries (e.g. a Tensor.cpd_als result scored on a held-out tensor).
 *   d_factors[m]  dims[m] x ldm device matrices, row-major; columns [ncolumns, ldm) never feed
 *                 the result (they may hold anything, NaN included).
 *   lambda        ncolumns HOST doubles, or NULL for all ones.
 * Works on any layout (it walks the tensor's first stream); a shard sums its own nonzeros.  Runs
 * on t->device, enqueues on `stream` and synchronises it once.  Input rules: 1 <= ncolumns <= 64,
 * ldm even and >= ncolumns, every d_factors[m] 16-byte aligned; otherwise SPLATT_ERROR_BADINPUT
 * and nothing is enqueued. */
int splatt_b200_tensor_sse(splatt_b200_tensor const * t, int ncolumns, int ldm,
                           double const * const * d_factors, double const * lambda,
                           double * sse_out, void * stream);

/* Tensor completion by row-wise ALS: fits x^(i_1..i_N) = sum_r prod_m U_m[i_m, r] (no lambda) to
 * the stored entries of `train` only (a coordinate that is not stored is unobserved, not zero;
 * duplicate coordinates are separate observations), minimising
 *     L = sum_{x stored} (v_x - x^_x)^2 + reg * sum_m ||U_m||_F^2,   reg = options[REGULARIZE].
 * One iteration updates the modes 0 .. N-1 in order; row i of U_m becomes
 *     (sum_x h_x h_x^T + reg I)^-1 sum_x v_x h_x   over the nonzeros x with mode-m index i,
 * h_x the Hadamard product of the other modes' current rows (modes updated earlier in the same
 * iteration with their new values).  A row with no observations becomes 0.
 *   validate      may be NULL; else a tensor with train's nmodes and dims, on the same device,
 *                 scored after every iteration.
 *   d_factors[m]  dims[m] x ldm device matrices, in/out: the start on entry, the factors of the
 *                 last iteration on return.  Columns [ncolumns, ldm) never feed the results and
 *                 are never written.
 *   history       NULL, or 3 doubles per iteration run: L, the training RMSE
 *                 sqrt(sum (v - x^)^2 / nnz), and the validation RMSE (NaN without `validate`).
 *   iterations_out the number of iterations run (may be NULL).
 * Stops after options[NITER] iterations or, from the second iteration on, when
 * |L_prev - L| / L_prev < options[TOLERANCE].  VERBOSITY above NONE prints one line per iteration.
 * Runs on train->device, enqueues on `stream`, synchronises it once per iteration (the history).
 * Input rules: 1 <= ncolumns <= 64; ldm even and >= ncolumns; every d_factors[m] 16-byte aligned;
 * reg finite and > 0; both tensors whole (shard_count <= 1); train built with the ALLROOT layout
 * (every mode served by a root stream; ASGIVEN is rejected).  Leaf-tiled streams (CTA-tiled by
 * default, or ktile > 0) are accepted.  A violation returns SPLATT_ERROR_BADINPUT before anything is
 * enqueued, and the factors are left untouched. */
int splatt_b200_tc_als_device(splatt_b200_tensor const * train,
                              splatt_b200_tensor const * validate,
                              int ncolumns, int ldm, double const * options,
                              double * const * d_factors, double * history,
                              int * iterations_out, void * stream);

/* Parameters of completion by L-BFGS beyond options[NITER], [TOLERANCE] and [REGULARIZE]. */
typedef struct {
  int memory;   /* L-BFGS pairs kept, 0..32 (default 5); 0 = steepest descent with the exact line search */
} splatt_b200_tc_lbfgs_opts;

/* Tensor completion by whole-model L-BFGS with an exact line search (CP-WOPT; Acar, Dunlavy, Kolda
 * & Morup, Chemometr. Intell. Lab. Syst. 2011).  Model and objective are those of
 * splatt_b200_tc_als_device: x^ = sum_r prod_m U_m[i_m, r] and
 *     L = sum_{x stored} (v_x - x^_x)^2 + reg * sum_m ||U_m||_F^2,   reg = options[REGULARIZE] >= 0,
 * minimised over all factors at once.  U stands for the concatenation of the factors (columns
 * [0, ncolumns) of every mode); g, d, s and y are vectors of that shape.  Iteration k, at U_k:
 *   1. Gradient g_k = grad L(U_k), every mode's block at the same U_k:
 *        G_m[i,:] = -2 sum_{x : i_m(x) = i} r_x h_x + 2 reg U_m[i,:],   r_x = v_x - x^_x,
 *      h_x the Hadamard product of the other modes' rows (a row with no observations gets
 *      2 reg U_m[i,:]).  From the second iteration on, the pair s = alpha_{k-1} d_{k-1},
 *      y = g_k - g_{k-1} enters a ring of `memory` pairs (the oldest dropped) when s.y > 0.
 *   2. Direction: if ||g_k||_2 = 0, alpha_k = 0 is recorded and the run stops.  Otherwise
 *      d = -H g_k by the two-loop recursion over the stored pairs (newest to oldest, a scaling by
 *      gamma = s.y / y.y of the newest pair, then oldest to newest); with no pair d = -g_k.  If
 *      g.d is not negative the pairs are cleared and d = -g_k.
 *   3. Exact line search: phi(a) = L(U_k + a d) = sum_{j=0}^{2N} c_j a^j, the data part from one
 *      walk over the nonzeros and reg (||U||^2 + 2 a <U,d> + a^2 ||d||^2).  alpha_k minimises phi
 *      over [0, B], B the Cauchy root bound of phi': the candidates are 0 and the real roots of
 *      phi' in (0, B], and the smallest candidate with the least value is taken (alpha_k = 0 when
 *      phi' is identically 0).  The decrease Delta = -sum_{j>=1} c_j alpha_k^j is evaluated from
 *      the coefficients, not as a difference of two objectives.  If Delta <= 0 along a direction
 *      from stored pairs, the pairs are cleared and the search is redone along -g_k in the same
 *      iteration; if Delta <= 0 along -g_k, alpha_k = 0 is recorded, the factors stay unchanged
 *      and the run stops.
 *   4. U_{k+1} = U_k + alpha_k d.
 * Stops after options[NITER] iterations, by the rules of steps 2 and 3, or, from the second
 * iteration on, after an iteration with Delta / phi(0) < options[TOLERANCE].
 *   lopts         NULL for the default (memory 5).
 *   validate      may be NULL; else a tensor with train's nmodes and dims, on the same device,
 *                 scored after every step.
 *   d_factors[m]  dims[m] x ldm device matrices, in/out: the start on entry, U after the last step
 *                 on return.  Columns [ncolumns, ldm) never feed a result and are never written.
 *   history       NULL, or 5 doubles per iteration run: L after the step (phi(0) - Delta), the
 *                 training RMSE after the step (from the data part of phi at alpha_k), the
 *                 validation RMSE after the step (NaN without `validate`), alpha_k and ||g_k||_2.
 *                 The first three columns are those of splatt_b200_tc_als_device.
 *   iterations_out the number of iterations run (may be NULL).
 * On untiled streams the factors, alpha and the first two history columns are bitwise
 * reproducible from run to run (no sum that feeds them uses atomics); on leaf-tiled streams the
 * gradient rows are added with atomics and may vary in the last bits.  Runs on train->device,
 * enqueues on `stream` and synchronises it once per iteration (the line coefficients, ||g|| and
 * g.d), twice in an iteration that retries along -g, and once at the end.  VERBOSITY above NONE
 * prints one line per iteration.
 * Input rules: those of splatt_b200_tc_als_device except that reg = 0 is allowed (reg finite and
 * >= 0), and 0 <= memory <= 32.  A violation returns SPLATT_ERROR_BADINPUT before anything is
 * enqueued, and the factors are left untouched. */
int splatt_b200_tc_lbfgs_device(splatt_b200_tensor const * train, splatt_b200_tensor const * validate,
                                int ncolumns, int ldm, double const * options,
                                splatt_b200_tc_lbfgs_opts const * lopts,
                                double * const * d_factors, double * history,
                                int * iterations_out, void * stream);

/* Host logic, no GPU needed: the exact line search of splatt_b200_tc_lbfgs_device.  For
 * phi(a) = sum_{j=0}^{degree} c[j] a^j (0 <= degree <= 16, coefficients finite) writes the alpha
 * of its step 3 and the decrease Delta = -sum_{j>=1} c[j] alpha^j.  The real roots of phi' in
 * (0, B] are found where phi' changes sign (or vanishes exactly) between consecutive roots of
 * phi'' -- found the same way one degree down -- and are bisected to full precision; a root where
 * phi' touches 0 without changing sign cannot be a minimiser and is not returned.  Returns
 * SPLATT_SUCCESS, or SPLATT_ERROR_BADINPUT (outputs untouched) on a bad argument. */
int splatt_b200_poly_argmin(int degree, double const * c, double * alpha_out, double * decrease_out);

/* Parameters of CP-APR beyond options[NITER] and options[TOLERANCE]. */
typedef struct {
  int    max_inner;      /* inner (multiplicative-update) iterations per mode, >= 1 (default 10) */
  double kappa;          /* shift added to entries pinned at zero, >= 0 (default 0.01) */
  double kappa_tol;      /* entries below this may be shifted, >= 0 (default 1e-10) */
  double eps_div_zero;   /* floor of the model value in a division or a log, > 0 (default 1e-10) */
} splatt_b200_apr_opts;

/* Poisson CP decomposition by CP-APR (Chi & Kolda, SIMAX 2012, multiplicative updates) for count
 * tensors.  The model M = sum_r lambda_r a_r^(1) o ... o a_r^(N) has lambda >= 0 and nonnegative
 * factors whose columns sum to 1; unstored coordinates are zero counts and duplicate coordinates
 * separate observations.  The call maximises
 *     LL = sum_{x stored} v_x log(max(m_x, eps)) - sum_r lambda_r     (m_x: the model at x).
 * Start: columns [0, ncolumns) of d_factors, every column divided by its sum s_{m,r}, and
 * lambda_r = prod_m s_{m,r}.  One outer iteration runs, for n = 0 .. N-1:
 *   1. from the second outer iteration on, add kappa to every A_n[i,r] < kappa_tol whose last
 *      Phi_n[i,r] > 1;
 *   2. B = A_n diag(lambda);
 *   3. up to max_inner times: Phi_n[i,:] = sum over x with i_n(x) = i of
 *      (v_x / max(B[i,:] . Pi_x, eps)) Pi_x, Pi_x the Hadamard product of the other modes' rows;
 *      kkt_n = max |min(B, 1 - Phi_n)|; stop if kkt_n < options[TOLERANCE], else B <- B * Phi_n;
 *   4. lambda = the column sums of B, A_n = B diag(1 / lambda) (a column with lambda_r = 0
 *      becomes 0).
 * Stops after options[NITER] outer iterations, or after the first in which every mode met
 * kkt_n < TOLERANCE at its first inner iteration.
 *   apr           NULL for the defaults (10, 0.01, 1e-10, 1e-10).
 *   d_factors[m]  dims[m] x ldm device matrices, in/out: the start on entry, the column-stochastic
 *                 factors on return.  Columns [ncolumns, ldm) never feed a result and are never
 *                 written.
 *   lambda_out    ncolumns HOST doubles.
 *   history       NULL, or 3 doubles per outer iteration run: LL after it, the largest final
 *                 kkt_n, and the inner iterations run, summed over the modes.
 *   iterations_out the number of outer iterations run (may be NULL).
 * On untiled streams lambda, the factors and the inner-iteration counts are bitwise reproducible
 * from run to run; on leaf-tiled streams Phi is summed with atomics and may vary in the last bits.
 * Runs on t->device, enqueues on `stream`, synchronises it once per inner iteration (the kkt
 * value) and once per outer iteration (the history).  VERBOSITY above NONE prints one line per
 * outer iteration.
 * Input rules: 1 <= ncolumns <= 64; ldm even and >= ncolumns; every d_factors[m] 16-byte aligned;
 * the tensor whole (shard_count <= 1) and built with the ALLROOT layout (leaf-tiled streams, CTA-
 * tiled or ktile > 0, are accepted); every tensor value finite and >= 0; every start entry in
 * columns [0, ncolumns) finite and >= 0 and every start column with a positive (finite) sum;
 * max_inner >= 1, kappa >= 0, kappa_tol >= 0, eps > 0 and TOLERANCE >= 0, all finite;
 * 0 <= NITER < 2^31.  A violation
 * returns SPLATT_ERROR_BADINPUT and the factors are left bit-identical. */
int splatt_b200_cp_apr_device(splatt_b200_tensor const * t, int ncolumns, int ldm,
                              double const * options, splatt_b200_apr_opts const * apr,
                              double * const * d_factors, double * lambda_out,
                              double * history, int * iterations_out, void * stream);

/* Parameters of CP-APR by PDNR beyond options[NITER] and options[TOLERANCE]. */
typedef struct {
  int    max_inner;      /* lockstep Newton iterations per mode, >= 1 (default 10) */
  int    max_backtrack;  /* trial steps of the line search, 1..8 (default 8) */
  double mu0;            /* initial and smallest damping, > 0 (default 1e-5) */
  double eps_active;     /* bound of the epsilon-active set, >= 0 (default 1e-8) */
  double eps_div_zero;   /* floor of the model value in a division or a log, > 0 (default 1e-10) */
} splatt_b200_pdnr_opts;

/* Poisson CP decomposition by CP-APR with row-wise projected damped Newton steps (PDNR; Hansen,
 * Plantenga & Kolda, Optim. Methods Softw. 2015).  Model, objective LL, start and outputs are
 * those of splatt_b200_cp_apr_device; there is no shift.  One outer iteration runs, for
 * n = 0 .. N-1:
 *   1. B = A_n diag(lambda).
 *   2. Every row i of B is its own problem: minimise
 *        f_i(b) = sum_r b_r - sum_{x in X_i} v_x log(max(m_x(b), eps)),  m_x(b) = b . Pi_x,
 *      X_i the stored x with i_n(x) = i and Pi_x the Hadamard product of the other modes' rows,
 *      from b = B[i,:] with mu_i = mu0; g = 1 - sum_x (v_x / max(m_x, eps)) Pi_x and
 *      H = sum_x (v_x / max(m_x, eps)^2) Pi_x Pi_x^T.  Up to max_inner lockstep iterations, every
 *      row still active:
 *      - kkt_i = max_r |min(b_r, g_r)|; if kkt_i < TOLERANCE the row stops and keeps b;
 *      - eps_i = min(eps_active, ||b - max(b - g, 0)||_2); the active set is
 *        A = {r : b_r <= eps_i and g_r > 0}, F the rest;
 *      - d_A = -g_A, and (H_FF + mu_i I) d_F = -g_F by Cholesky; if a pivot is <= 0 or not
 *        finite, d = -g for this iteration;
 *      - trial points b_k = max(b + 2^-k d, 0), k = 0 .. max_backtrack-1; the smallest k with
 *        f_i(b_k) <= f_i(b) + 1e-4 g^T (b_k - b) and f_i(b_k) <= f_i(b) is accepted, b <- b_k.
 *        The change f_i(b_k) - f_i(b) is evaluated as
 *        sum_r (b_k - b)_r - sum_x v_x log(max(m_x + delta_x, eps) / max(m_x, eps)),
 *        delta_x = (b_k - b) . Pi_x, the log of the ratio by log1p(delta_x / m_x) where neither
 *        value is floored, so a decrease stays visible near the row's minimum;
 *      - if k = 0 was accepted mu_i <- max(mu_i / 3.5, mu0), else (a larger k, or none passed,
 *        b unchanged) mu_i <- 3.5 mu_i.
 *      The lockstep loop of a mode ends early when no row is active.
 *   3. lambda = the column sums of B, A_n = B diag(1 / lambda) (a column with lambda_r = 0
 *      becomes 0).
 * Stops after options[NITER] outer iterations, or after one in which every row of every mode had
 * kkt_i < TOLERANCE at its first evaluation.  sum_i f_i(B[i]) = -LL and the accept rule never
 * raises an f_i, so LL does not decrease from mode to mode, up to rounding in the sums.
 *   pdnr          NULL for the defaults (10, 8, 1e-5, 1e-8, 1e-10).
 *   d_factors[m], lambda_out, iterations_out: as splatt_b200_cp_apr_device.
 *   history       NULL, or 4 doubles per outer iteration run: LL after it, the largest
 *                 last-computed kkt_i over all rows and modes, the lockstep iterations run summed
 *                 over the modes, and the Newton steps attempted (a line search run, whether
 *                 or not a trial point passed) summed over rows and modes.
 * On untiled streams lambda, the factors and the history's last three columns are bitwise
 * reproducible from run to run; on leaf-tiled streams the gradient, Hessian and line-search sums
 * are added with atomics and may vary in the last bits.  Runs on t->device, enqueues on `stream`,
 * synchronises it once per lockstep iteration (the count of rows that attempted a step) and once per
 * outer iteration (the history).  VERBOSITY above NONE prints one line per outer iteration.
 * Input rules: those of splatt_b200_cp_apr_device, and max_inner >= 1, 1 <= max_backtrack <= 8,
 * mu0 > 0, eps_active >= 0 and eps > 0, all finite.  A violation returns SPLATT_ERROR_BADINPUT and
 * the factors are left bit-identical. */
int splatt_b200_cp_apr_pdnr_device(splatt_b200_tensor const * t, int ncolumns, int ldm,
                                   double const * options, splatt_b200_pdnr_opts const * pdnr,
                                   double * const * d_factors, double * lambda_out,
                                   double * history, int * iterations_out, void * stream);

/* Parameters of CP-APR by PQNR beyond options[NITER] and options[TOLERANCE]. */
typedef struct {
  int    max_inner;      /* lockstep quasi-Newton iterations per mode, >= 1 (default 10) */
  int    max_backtrack;  /* trial steps of the line search, 1..8 (default 8) */
  int    lbfgs_mem;      /* L-BFGS pairs kept per row, 1..8 (default 3) */
  double eps_active;     /* bound of the epsilon-active set, >= 0 (default 1e-8) */
  double eps_div_zero;   /* floor of the model value in a division or a log, > 0 (default 1e-10) */
} splatt_b200_pqnr_opts;

/* Poisson CP decomposition by CP-APR with row-wise projected quasi-Newton steps (PQNR; Hansen,
 * Plantenga & Kolda, Optim. Methods Softw. 2015).  Model, objective LL, start, outputs, outer
 * loop, stop rule and the absence of a shift are those of splatt_b200_cp_apr_pdnr_device; only
 * the direction differs, and it needs no Hessian.  In mode n every row i of B = A_n diag(lambda)
 * starts from b = B[i,:] with no stored pair and level j = 0, and runs up to max_inner lockstep
 * evaluations:
 *   1. g = 1 - sum_x (v_x / max(m_x, eps)) Pi_x and kkt_i = max_r |min(b_r, g_r)|; if
 *      kkt_i < TOLERANCE the row stops and keeps b.
 *   2. After a previous step, if b is bitwise equal to b_prev (the last line search moved
 *      nothing): j <- j + 1; at j = 3 the row stops; otherwise d <- 2^-max_backtrack d, so the
 *      trial points continue the halving, and go to 5.
 *   3. Otherwise j = 0, and after a previous step the pair s = b - b_prev, y = g - g_prev is
 *      stored in a ring of lbfgs_mem pairs (the oldest dropped) if s.y > 0 and 1 / s.y is finite.
 *   4. eps_i and the active set A are PDNR's; q = -g with q_A = 0; the L-BFGS two-loop recursion
 *      over the stored pairs, newest to oldest, then a scaling by gamma = s.y / y.y of the newest
 *      pair (1 when none is stored), then oldest to newest; d = q, then d_A = -g_A, and d = -g
 *      when d is not finite.
 *   5. b_prev = b, g_prev = g, and PDNR's line search along d: trial points
 *      max(b + 2^-k d, 0), k = 0 .. max_backtrack-1, its Armijo and decrease tests and its
 *      evaluation of the change; b stays unchanged when no trial point passes.
 * Every scaling of d is a power of two, so the trial points do not depend on how the scalings
 * are grouped.  A lockstep iteration in which no row gets a direction ends the mode without
 * running the line search.
 *   pqnr          NULL for the defaults (10, 8, 3, 1e-8, 1e-10).
 *   d_factors[m], lambda_out, iterations_out: as splatt_b200_cp_apr_device.
 *   history       NULL, or 4 doubles per outer iteration run: LL after it, the largest
 *                 last-computed kkt_i over all rows and modes, the lockstep iterations run summed
 *                 over the modes, and the line searches run (continuations included, whether or
 *                 not a trial point passed) summed over rows and modes.
 * On untiled streams lambda, the factors and the history's last three columns are bitwise
 * reproducible from run to run; on leaf-tiled streams Phi and the line-search sums are added
 * with atomics and may vary in the last bits.  Runs on t->device, enqueues on `stream`,
 * synchronises it once per lockstep iteration (the count of rows with a direction) and once per
 * outer iteration (the history).  VERBOSITY above NONE prints one line per outer iteration.
 * Input rules: those of splatt_b200_cp_apr_device, and max_inner >= 1, 1 <= max_backtrack <= 8,
 * 1 <= lbfgs_mem <= 8, eps_active >= 0 and eps > 0, all finite.  A violation returns
 * SPLATT_ERROR_BADINPUT and the factors are left bit-identical. */
int splatt_b200_cp_apr_pqnr_device(splatt_b200_tensor const * t, int ncolumns, int ldm,
                                   double const * options, splatt_b200_pqnr_opts const * pqnr,
                                   double * const * d_factors, double * lambda_out,
                                   double * history, int * iterations_out, void * stream);

/* TTMc, the kernel of Tucker: d_out = X_(mode) (kron_{m != mode} U_m), a dims[mode] x C_mode
 * row-major device matrix with leading dimension C_mode = prod_{m != mode} ranks[m], U_m =
 * columns [0, ranks[m]) of d_mats[m] (dims[m] x ldm, row-major).  Column order: the other modes
 * in increasing mode order, the highest fastest (c = sum_{m != mode} j_m prod_{m' > m, m' != mode}
 * ranks[m']), whatever the stream's level order.  Unstored coordinates are zeros; duplicate
 * coordinates add.  d_out is zeroed, then written.  d_mats[mode] is not read (may be NULL).
 * Runs on t->device and enqueues on `stream` (boundary-slot scratch is allocated and freed
 * stream-ordered); no host synchronisation.  On untiled streams the result is bitwise
 * reproducible; on leaf-tiled streams (CTA-tiled or ktile > 0) pieces of a row are added with
 * atomics and may vary in the last bits.
 * Input rules: the tensor whole (shard_count <= 1) and built with the ALLROOT layout; 2 <= N <= 8;
 * 0 <= mode < N; 1 <= ranks[m] <= min(32, dims[m]) for every m; C_mode <= 1024; ldm even and
 * >= every ranks[m]; d_out and every d_mats[m], m != mode, 16-byte aligned.  A violation returns
 * SPLATT_ERROR_BADINPUT and nothing is enqueued. */
int splatt_b200_ttmc(splatt_b200_tensor const * t, int mode, int const * ranks, int ldm,
                     double const * const * d_mats, double * d_out, void * stream);

/* Parameters of HOOI's subspace step beyond options[NITER] and options[TOLERANCE]. */
typedef struct {
  int    max_power;      /* orthogonal-iteration steps per mode and iteration, >= 1 (default 50) */
  double svd_tol;        /* stop the steps when the subspace moved by <= this, >= 0 (default 1e-10) */
} splatt_b200_tucker_opts;

/* Sparse Tucker decomposition by HOOI (higher-order orthogonal iteration):
 *     X ~ G x_0 U_0 x_1 U_1 ... x_{N-1} U_{N-1},
 * U_m dims[m] x ranks[m] with orthonormal columns, G the ranks[0] x ... x ranks[N-1] core.
 * Unstored coordinates are zeros; duplicate coordinates add (in the TTMc and in ||X||^2).
 * Start: columns [0, ranks[m]) of d_factors[m], each orthonormalised by CholeskyQR2 in fp64.
 * One iteration runs, for n = 0 .. N-1 (modes updated earlier in the iteration with their new
 * values):
 *   1. Y_n = splatt_b200_ttmc(n), dims[n] x C_n;
 *   2. from Q = U_n, up to max_power steps of Q <- orth(Y_n Y_n^T Q + mu Q), orth = CholeskyQR2,
 *      mu = 2^-20 ||Y_n||_F^2 (1 when Y_n = 0): the shift keeps CholeskyQR well posed when Y_n
 *      has rank below R_n and leaves the eigenvectors unchanged; the steps stop early once
 *      ||Q_new - Q_old (Q_old^T Q_new)||_F <= svd_tol;
 *   3. Rayleigh-Ritz: W = Y_n^T Q, W^T W = V diag(lam) V^T (Jacobi, lam descending),
 *      U_n = Q V; in every column the entry of largest magnitude is made positive (the lowest
 *      row on a tie).
 * After the last mode G = (W V with U_{N-1}'s column signs), whose C_{N-1} x R_{N-1} row-major
 * array is the C-order array of shape (ranks[0], ..., ranks[N-1]), and
 *     fit = 1 - sqrt(max(||X||^2 - ||G||_F^2, 0)) / ||X||.
 * Stops after options[NITER] iterations, or when fit = 1, or from the second iteration on when
 * |fit - previous fit| < options[TOLERANCE].  VERBOSITY above NONE prints one line per
 * iteration.  A rank-deficient Y_n still gives orthonormal U_n (the columns past its rank are
 * some orthonormal completion, with zero core entries).
 *   topts         NULL for the defaults (50, 1e-10).
 *   d_factors[m]  dims[m] x ldm device matrices, in/out: the start on entry, the factors of the
 *                 last iteration on return (the orthonormalised start when NITER = 0).  Columns
 *                 [ranks[m], ldm) never feed a result and are never written.
 *   core_out      prod ranks[m] HOST doubles, the core of the last iteration (untouched when no
 *                 iteration ran).
 *   history       NULL, or 4 doubles per iteration run: the fit, ||G||_F, the orthogonal-
 *                 iteration steps summed over the modes, and the largest final subspace residual.
 *   iterations_out the number of iterations run (may be NULL).
 * The factors are only written on success.  On untiled streams the factors, the core and the
 * history are bitwise reproducible from run to run (every reduction has a fixed order); on
 * leaf-tiled streams the TTMc adds with atomics.  Runs on t->device, enqueues on `stream` and
 * synchronises it once per orthogonal-iteration step (the residual), once per mode (the R x R
 * Ritz matrix, diagonalised on the host) and once per iteration (the fit and the core).
 * Input rules: the tensor whole and ALLROOT (leaf-tiled streams accepted); 2 <= N <= 8;
 * 1 <= ranks[m] <= min(32, dims[m]); ranks[n] <= C_n <= 1024 for every n; ldm even and >= every
 * ranks[m]; every d_factors[m] 16-byte aligned; max_power >= 1; svd_tol, TOLERANCE >= 0 and
 * finite; 0 <= NITER < 2^31; every start factor with independent columns (a Gram pivot above
 * 2^-46 of its diagonal entry in CholeskyQR).  A violation returns SPLATT_ERROR_BADINPUT and the
 * factors are left bit-identical. */
int splatt_b200_tucker_hooi_device(splatt_b200_tensor const * t, int const * ranks, int ldm,
                                   double const * options, splatt_b200_tucker_opts const * topts,
                                   double * const * d_factors, double * core_out,
                                   double * history, int * iterations_out, void * stream);

/* The nonzeros of a device tensor as coordinates, in the record order of its first stream
 * (t->streams[0]: lexicographic in that stream's level order on an untiled stream; leaf-tiled
 * streams regroup records inside ranges).  d_ind[m] (nnz_local uint32 each) and d_vals
 * (nnz_local doubles) are caller-allocated DEVICE buffers; a shard writes its own nonzeros.
 * One pass over the records, each 64-record chunk decoded from its descriptor, the records'
 * close counts and the level ids up[l].  Works on every layout and tiling.  Runs on t->device,
 * enqueues on `stream`; no host synchronisation.  Input rules: t non-NULL, every d_ind[m] and
 * d_vals non-NULL; otherwise SPLATT_ERROR_BADINPUT and nothing is enqueued. */
int splatt_b200_tensor_to_coo(splatt_b200_tensor const * t, uint32_t * const * d_ind, double * d_vals,
                              void * stream);

/* Losses of generalized CP (splatt_b200_gcp_*).  f(x, m), its derivative in m, and the values
 * x a tensor may hold:
 *   GAUSSIAN          (x - m)^2                                   2 (m - x)     finite
 *   BERNOULLI_LOGIT   softplus(m) - x m,                          sigma(m) - x  0 or 1
 *                     softplus(m) = max(m, 0) + log1p(exp(-|m|))
 *   POISSON_LOG       exp(m) - x m                                exp(m) - x    finite, >= 0
 * The stored-entry corrections f(x, m) - f(0, m) and df(x, m) - df(0, m) are evaluated as
 * x^2 - 2 x m and -2 x (GAUSSIAN), -x m and -x (the others). */
typedef enum {
  SPLATT_B200_GCP_GAUSSIAN = 0,
  SPLATT_B200_GCP_BERNOULLI_LOGIT = 1,
  SPLATT_B200_GCP_POISSON_LOG = 2
} splatt_b200_gcp_loss;

/* Parameters of GCP-Adam beyond options[NITER], [TOLERANCE] and [VERBOSITY]. */
typedef struct {
  int      loss;         /* splatt_b200_gcp_loss (default BERNOULLI_LOGIT) */
  int      grad_nnz;     /* p of every gradient sample: stored entries, >= 0 (default 65536) */
  int      grad_zeros;   /* q of every gradient sample: uniform coordinates, >= 0 (default 65536) */
  int      est_nnz;      /* p of the estimate sample, >= 0 (default 1048576) */
  int      est_zeros;    /* q of the estimate sample, >= 0 (default 1048576) */
  int      epoch_iters;  /* Adam steps per epoch, >= 1 (default 1000) */
  double   lr;           /* learning rate of the first epoch, > 0 (default 1e-3) */
  double   beta1;        /* first-moment decay, in [0, 1) (default 0.9) */
  double   beta2;        /* second-moment decay, in [0, 1) (default 0.999) */
  double   epsilon;      /* Adam's denominator floor, > 0 (default 1e-8) */
  double   decay;        /* lr factor after a failed epoch, in (0, 1] (default 0.1) */
  int      max_fails;    /* failed epochs tolerated, >= 0 (default 1) */
  uint64_t seed;         /* key of every draw (default 0) */
} splatt_b200_gcp_opts;

/* Draws one sample set of GCP exactly as splatt_b200_gcp_device does.  Philox4x32-10 keyed by
 * (seed & 0xffffffff, seed >> 32); draw j of step t_step under purpose P uses block b with counter
 * (j, t_step & 0xffffffff, t_step >> 32, 4 P + b), and each 64-bit value is two consecutive words,
 * the first one high.  Purposes: 0 gradient stored entries, 1 gradient coordinates, 2 estimate
 * stored entries, 3 estimate coordinates (`estimate` 0 selects 0 and 1, else 2 and 3).
 *   - sample j < p is a stored entry: the record position __umul64hi(v, nnz) in the record order
 *     of splatt_b200_tensor_to_coo, v from block 0 words 0-1 with j the draw index;
 *   - sample p + j (j < q) is a coordinate: mode n's index __umul64hi(v_n, dims[n]), v_n from
 *     words 2 (n mod 2), 2 (n mod 2) + 1 of block n / 2, with j the draw index; its value is 0.
 * d_ind[m] (p + q uint32 each) and d_vals (p + q doubles) are caller-allocated DEVICE buffers.
 * The draws do not depend on the launch shape.  Decodes the tensor once into stream-ordered
 * scratch of (4 N + 8) nnz bytes.  Runs on t->device and enqueues on `stream`; no host
 * synchronisation.  Input rules: a whole tensor (shard_count <= 1); p, q >= 0, p + q >= 1 and
 * p + q < 2^31; p = 0 when the tensor has no nonzero; every pointer non-NULL; otherwise
 * SPLATT_ERROR_BADINPUT and nothing is enqueued. */
int splatt_b200_gcp_sample(splatt_b200_tensor const * t, uint64_t seed, uint64_t t_step, int estimate,
                           int p, int q, uint32_t * const * d_ind, double * d_vals, void * stream);

/* The kernel primitive of GCP on an explicit sample of p + q coordinates (d_ind[m], p + q uint32
 * each, on the device): samples 0 .. p-1 are stored entries with values d_vals[0 .. p-1] and weight
 * w_nz, samples p .. p+q-1 are coordinates (value 0) with weight w_z.  With m_s the model
 * sum_r prod_n U_n[i_n, r] at sample s,
 *     value = sum_{s < p} w_nz (f(x_s, m_s) - f(0, m_s)) + sum_{s >= p} w_z f(0, m_s),
 *     G_n[i, :] = sum_{s : i_n(s) = i} y_s prod_{k != n} U_k[i_k(s), :],
 *     y_s = w_nz (df(x_s, m_s) - df(0, m_s)) (s < p),  w_z df(0, m_s) (s >= p).
 *   d_factors[m]  dims[m] x ldm device matrices; columns [ncolumns, ldm) are never read.
 *   d_grads       NULL (value only), or dims[m] x ldm device matrices: columns [0, ncolumns) are
 *                 zeroed and then accumulated into, the other columns never written.
 *   value_out     NULL (no value, no host synchronisation), or one HOST double.
 * The value is summed in a fixed order (per warp in sample order, then warps, then CTAs in order)
 * and is bitwise reproducible; the gradient rows are added with red.add.f64 atomics and are not.
 * Runs on t->device and enqueues on `stream`; synchronises it once when value_out is given.
 * Input rules: loss one of splatt_b200_gcp_loss; 1 <= ncolumns <= 64; ldm even and >= ncolumns;
 * every d_factors[m] (and d_grads[m]) non-NULL and 16-byte aligned; p, q >= 0, p + q < 2^31; w_nz
 * and w_z finite; d_vals non-NULL when p > 0.  Indices must lie inside dims (not checked).  A
 * violation returns SPLATT_ERROR_BADINPUT and nothing is enqueued. */
int splatt_b200_gcp_sampled(splatt_b200_tensor const * t, int loss, int p, int q, double w_nz,
                            double w_z, uint32_t const * const * d_ind, double const * d_vals,
                            int ncolumns, int ldm, double const * const * d_factors,
                            double * const * d_grads, double * value_out, void * stream);

/* Generalized CP decomposition (GCP; Hong, Kolda & Duersch, SIAM Rev. 2020) by sampled gradients
 * and Adam (GCP-Adam; Kolda & Hong, SIMODS 2020, Alg. 5.1).  The model m_x = sum_r prod_n
 * U_n[i_n, r] (no lambda) is fitted to every coordinate, unstored ones being x = 0:
 *     F(U) = sum_{all coordinates} f(0, m) + sum_{stored x} (f(x_v, m_x) - f(0, m_x)),
 * f the loss of gopts->loss; duplicate coordinates count separately.  With nnz the stored entries
 * and P = prod dims[n] (in fp64), a sample of p stored entries and q coordinates
 * (splatt_b200_gcp_sample) weighted w_nz = nnz / p and w_z = P / q (0 when p or q is 0) gives
 * unbiased estimates of F and grad F (splatt_b200_gcp_sampled).
 *   Steps.  The global step count t starts at 0.  A step draws the gradient sample of step t,
 *     forms every mode's gradient G at the same U, and applies Adam to columns [0, ncolumns):
 *       M = b1 M + (1 - b1) G,  V = b2 V + (1 - b2) G^2,
 *       U -= lr (M / (1 - b1^(t+1))) / (sqrt(V / (1 - b2^(t+1))) + eps);
 *     then t = t + 1.  M and V start at 0.
 *   Epochs.  An epoch is epoch_iters steps; at its end F is estimated on one estimate sample
 *     drawn once per call (t_step = 0, purposes 2 and 3).  The epoch is accepted if the estimate
 *     is finite and <= the last accepted estimate (the start's estimate at first).  Otherwise it
 *     fails: U, M, V and t return bitwise to their values at the epoch's start and lr *= decay.
 *   Stops after options[NITER] epochs, after more than max_fails failed epochs, or after an
 *     accepted epoch whose relative decrease (prev - est) / |prev| is < options[TOLERANCE] (a
 *     previous estimate of 0 counts as no decrease).
 *   gopts         NULL for the defaults (BERNOULLI_LOGIT, 65536, 65536, 1048576, 1048576, 1000,
 *                 1e-3, 0.9, 0.999, 1e-8, 0.1, 1, 0).
 *   d_factors[m]  dims[m] x ldm device matrices, in/out: the start on entry, U after the last
 *                 accepted (or the start, when none) epoch's end on return.  Columns
 *                 [ncolumns, ldm) never feed a result and are never written.
 *   history       NULL, or 3 doubles per epoch run: the estimate at its end, the lr it used, and
 *                 1 if it was accepted, else 0.
 *   f_start_out   NULL, or one HOST double: the estimate at the start.
 *   epochs_out    the number of epochs run (may be NULL).
 * The gradients are summed with atomics, so U is not bitwise reproducible from run to run; given
 * the gradient, the estimate and the Adam update are elementwise and deterministic.  The stored
 * entries are decoded once per call into (4 N + 8) nnz bytes of device memory beside the sample
 * buffers.  Runs on t->device, enqueues on `stream` and synchronises it once per epoch (the
 * estimate) and a bounded number of times at the start (the value check, the start's estimate);
 * never within an epoch.  VERBOSITY above NONE prints one line per epoch.
 * Input rules: a whole tensor (shard_count <= 1) of 2..8 modes, any layout; 1 <= ncolumns <= 64;
 * ldm even and >= ncolumns; every d_factors[m] 16-byte aligned; every tensor value allowed by
 * the loss (checked on the device); p, q >= 0 and 1 <= p + q < 2^31 for both samples, p = 0 when
 * the tensor has no nonzero; epoch_iters >= 1; lr > 0, 0 <= beta1, beta2 < 1, epsilon > 0,
 * 0 < decay <= 1, all finite; max_fails >= 0; TOLERANCE finite; 0 <= NITER < 2^31.  A violation
 * returns SPLATT_ERROR_BADINPUT, and the factors are left bit-identical. */
int splatt_b200_gcp_device(splatt_b200_tensor const * t, int ncolumns, int ldm, double const * options,
                           splatt_b200_gcp_opts const * gopts, double * const * d_factors,
                           double * history, double * f_start_out, int * epochs_out, void * stream);

/* Measurement aid: a pure gather kernel with the MTTKRP's access pattern (whole
 * fp64 rows of a rows x ldm matrix at d_idx[0..nidx), 128-bit loads, eight rows in
 * flight per lane group, no arithmetic).  bench.py times it to report a MEASURED
 * ceiling for the L2->SM gather path next to the kernel's achieved rate.  Reads
 * only the first min(ncolumns, 64) columns. */
int splatt_b200_gather_probe(
    double const * d_mat, int ncolumns, int ldm,
    uint32_t const * d_idx, uint64_t nidx, double * d_sink, void * stream);

/* The same probe at a chosen shape: `ctas_per_sm` (1..8) CTAs of 256 threads resident per
 * SM, `rows_in_flight` (2/4/8/16) independent row loads per lane group, `no_allocate` != 0
 * loads with ld.global.nc.L1::no_allocate, `smem_bytes` of dynamic shared memory reserved
 * per CTA (shrinks the L1).  ncolumns must be 16, 32 or 64.
 * scripts/probe_sweep.py sweeps the shapes; the best point is the access pattern's ceiling. */
int splatt_b200_gather_probe_ex(
    double const * d_mat, int ncolumns, int ldm,
    uint32_t const * d_idx, uint64_t nidx, double * d_sink,
    int ctas_per_sm, int rows_in_flight, int no_allocate, int smem_bytes, void * stream);

/* Number of kernels the engine has launched in this process (bench.py's
 * gpu_launches evidence). */
uint64_t splatt_b200_launch_count(void);

/* Number of fiber streams built (sorted + scanned) in this process so far. */
uint64_t splatt_b200_build_count(void);

/* The bare splatt_mttkrp entry keeps the device mirrors it builds (LRU of
 * SPLATT_B200_CACHE entries, default 2, 0 = rebuild on every call as the reference
 * rebuilds its workspace, src/mttkrp.c:1796).  A mirror is reused only when the CSF array,
 * its policy / rank / shape, the addresses of its arrays AND a content fingerprint match.
 * Call this before freeing a CSF whose mirror should release its HBM now. */
void splatt_b200_cache_clear(void);

/* Library / build identification, e.g. "splatt_b200 0.1 (sm_90a fiber-stream MTTKRP)". */
char const * splatt_b200_version(void);

#ifdef __cplusplus
}
#endif
#endif /* SPLATT_B200_H */
