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
