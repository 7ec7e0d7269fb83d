// 3-mode root MTTKRP with the LEAF factor staged tile by tile in shared memory.
//
// The generic root kernel sits on the measured ceiling of its access pattern: two
// factor rows per nonzero gathered through L2 -> SM (DESIGN.md 4.1).  When one SM's
// nonzeros touch every leaf row several times (nnz per SM >> rows of the leaf factor),
// half of those gathers can be served from shared memory instead:
//
//   * the stream is built "CTA-tiled" (stream_build.cu): the records of CTA r's range
//     are regrouped by leaf tile, seg_off[r * ntiles + t] marks the segments, and
//     rroot[2r], rroot[2r + 1] bound the root rows the range touches;
//   * one persistent CTA per SM walks its range tile by tile; the leaf-factor tiles are
//     streamed in with TMA bulk copies, double buffered (mbarrier full, a counter of the
//     warps done with a buffer);
//   * every warp stages its records through a private TMA ring, reads the leaf row from
//     the tile (LDS.128) and gathers only the parent row from L2;
//   * slice / sub-range ends add into a shared-memory block holding the range's root
//     rows; at the end interior rows are stored, and only the first and last row (which
//     the neighbouring ranges may share) are reduced into the output.
//
// Columns are processed in slabs of kSlab: the tile and the accumulator hold one slab, and
// the CTA re-walks its records once per slab, all inside one launch.  Same results as the
// generic kernel (linearity); chosen by spb200_launch_mttkrp whenever the stream carries the
// tiling.
#include "mttkrp_kernels.cuh"

namespace spb200 {

constexpr int kTW   = 32;         // warps per CTA, all of them consuming records
constexpr int kTRS  = 72;         // records per warp per staging round
constexpr int kTB   = 3;          // records whose gathers are issued together
constexpr int kSlab = 32;         // columns held in shared memory at a time
static_assert(kTB <= 4, "a batch's close counts are packed one byte per record");

struct TiledArgs {
  const SpRec *    rec;
  const uint32_t * rootid;
  const uint32_t * seg_off;       // this grid's ranges: [gridDim.x * ntiles + 1]
  const uint32_t * rroot;         // [2 * gridDim.x] first / last root row of every range
  const double *   leaf;
  const double *   parent;
  double *         out;
  uint32_t         ntiles, tile_rows, leaf_rows;
  uint32_t         tile_bytes;    // bytes reserved per tile buffer (tile_rows * kSlab * 8)
  uint32_t         tpitch;        // bytes per row of a staged tile
  uint32_t         acc_rows;      // rows of the shared accumulator
  int              ldm, col0, col_end;
  int              whole;         // 1: one slab and ldm <= kSlab: a tile is one contiguous copy
};

__device__ __forceinline__ void mbar_wait(uint64_t * bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {}
}

// shared-memory load by 32-bit address (volatile: stays after the mbarrier wait that guards it)
__device__ __forceinline__ double2 lds_f64x2(uint32_t addr) {
  double2 r;
  asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(r.x), "=d"(r.y) : "r"(addr));
  return r;
}

// 32 warps, one CTA per SM, all of them consuming records (no producer warp).  The parent-row
// gathers are bound by how many warps keep them in flight, not by how deep one warp's batch is
// (gather probe, DESIGN.md 4.1), and a 1024-thread CTA leaves 64 registers per thread.  The
// batch loop fits them without spilling: a batch's parent gathers are issued straight from the
// records' aux words, and the leaf rows are folded into the fiber sums while they are in flight,
// so only the closing records' fiber products, the parent rows, acc0 / acc1 and the close
// counts live across the wait.  At 4 records per batch the kernel still spilled (32 B); at 3 it
// does not.  Per-tile values (segment bounds, the issue side's next round) are re-read rather
// than held across the batch loop.  Leaf tiles are double buffered; the last warp to finish
// tile gt loads tile gt + 2 into the buffer gt leaves.
template <int L>
__global__ void __launch_bounds__(kTW * 32, 1) mttkrp_tiled_root3(const TiledArgs a) {
  constexpr int G  = 32 / L;
  constexpr int NG = kTW * G;     // lane groups per CTA

  extern __shared__ __align__(128) unsigned char smem[];
  unsigned char * tiles = smem;                                              // 2 x tile_bytes
  double *   accs = reinterpret_cast<double *>(smem + 2 * a.tile_bytes);    // [acc_rows][kSlab]
  SpRec *    ring = reinterpret_cast<SpRec *>(accs + static_cast<size_t>(a.acc_rows) * kSlab);
  uint64_t * bars = reinterpret_cast<uint64_t *>(ring + kTW * 2 * kTRS);
  uint64_t * tile_full = bars;                                               // [2]
  uint32_t * tile_left = reinterpret_cast<uint32_t *>(bars + 2);            // [2] warps done with a buffer
  uint64_t * rec_full  = bars + 4;                                           // [kTW][2]

  const int      warp  = threadIdx.x >> 5;
  const int      lane  = threadIdx.x & 31;
  const uint32_t pitch = static_cast<uint32_t>(a.ldm) * 8u;
  const uint32_t NT    = a.ntiles;
  const uint32_t NS    = static_cast<uint32_t>(a.col_end - a.col0 + kSlab - 1) / kSlab;
  // the range's first root row, its row count and its segment offsets are re-read where needed
  // rather than held in registers across the main loop
  auto range_lo   = [&]() { return __ldg(&a.rroot[2 * blockIdx.x]); };
  auto range_rows = [&]() {
    const uint32_t r_lo = range_lo(), r_hi = __ldg(&a.rroot[2 * blockIdx.x + 1]);
    return (r_hi >= r_lo) ? r_hi - r_lo + 1 : 0u;
  };

  for (uint32_t i = threadIdx.x, nrows = range_rows(); i < nrows * (kSlab / 2); i += blockDim.x)
    reinterpret_cast<double2 *>(accs)[i] = make_double2(0.0, 0.0);
  if (threadIdx.x == 0) {
    for (int b = 0; b < 2; ++b) { mbar_init(&tile_full[b], 1); tile_left[b] = 0; }
    for (int w = 0; w < kTW * 2; ++w) mbar_init(&rec_full[w], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  // one warp loads tile gt (slab gt / NT, tile gt % NT) into buffer gt & 1
  auto load_tile = [&](uint32_t gt) {
    const uint32_t t = gt % NT, b = gt & 1u;
    const uint32_t rows = min(a.tile_rows, a.leaf_rows - t * a.tile_rows);
    unsigned char * dst = tiles + b * a.tile_bytes;
    // generic-proxy reads of this buffer (the tile gt - 2) are ordered before the async writes
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    if (a.whole) {
      if (lane == 0) {
        const uint32_t bytes = rows * pitch;
        mbar_arrive_expect_tx(&tile_full[b], bytes);
        const char * src = reinterpret_cast<const char *>(a.leaf) +
                           static_cast<size_t>(t) * a.tile_rows * pitch;
        // bulk copies of at most 32 KB each
        for (uint32_t off = 0; off < bytes; off += 32768u)
          tma_bulk_g2s(dst + off, src + off, min(32768u, bytes - off), &tile_full[b]);
      }
    } else {
      // one slab of every row: a strided block, one bulk copy per row spread over the lanes
      const int      sc0 = a.col0 + static_cast<int>(gt / NT) * kSlab;
      const uint32_t sb  = static_cast<uint32_t>(min(kSlab, a.col_end - sc0)) * 8u;
      if (lane == 0) mbar_arrive_expect_tx(&tile_full[b], rows * sb);
      __syncwarp();
      const double * src = a.leaf + static_cast<size_t>(t) * a.tile_rows * a.ldm + sc0;
      for (uint32_t i = lane; i < rows; i += 32)
        tma_bulk_g2s(dst + i * a.tpitch, src + static_cast<size_t>(i) * a.ldm, sb, &tile_full[b]);
    }
  };
  if (warp == 0) {
    load_tile(0);
    if (NS * NT > 1) load_tile(1);
  }

  const int  grp    = lane / L;
  const int  gl     = lane % L;
  const bool leader = (gl == 0);
  SpRec *    myring = ring + warp * 2 * kTRS;
  uint64_t * mybars = rec_full + warp * 2;

  // part of segment t that belongs to lane-group gi / to this warp
  auto part = [&](uint32_t t, uint32_t g0, uint32_t g1, uint32_t & lo, uint32_t & hi) {
    const uint32_t * so = a.seg_off + blockIdx.x * NT + t;
    const uint32_t s0 = __ldg(so), len = __ldg(so + 1) - s0;
    lo = s0 + static_cast<uint32_t>(static_cast<unsigned long long>(g0) * len / NG);
    hi = s0 + static_cast<uint32_t>(static_cast<unsigned long long>(g1) * len / NG);
  };

  // issue side, run by lane 0: rounds are enumerated slab-major, then tile-major, at least one
  // (possibly empty) per tile; the next round to issue (tile, offset) is kept in shared memory
  uint32_t * inext = reinterpret_cast<uint32_t *>(rec_full + 2 * kTW) + 2 * warp;
  if (lane == 0) { inext[0] = 0; inext[1] = 0; }
  auto issue_next = [&](uint32_t ij) {      // round ij into stage ij & 1
    if (lane != 0) return;
    uint32_t it = inext[0], ioff = inext[1];
    if (it >= NS * NT) return;
    uint32_t ws, we;
    part(it % NT, warp * G, (warp + 1) * G, ws, we);
    const uint32_t rs  = ws + ioff;
    const uint32_t cnt = (rs < we) ? min(static_cast<uint32_t>(kTRS), we - rs) : 0u;
    uint64_t * bar = &mybars[ij & 1u];
    if (cnt) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      mbar_arrive_expect_tx(bar, cnt * 16u);
      tma_bulk_g2s(myring + (ij & 1u) * kTRS, a.rec + rs, cnt * 16u, bar);
    } else {
      mbar_arrive(bar);
    }
    ioff += kTRS;
    if (ws + ioff >= we) { ++it; ioff = 0; }
    inext[0] = it; inext[1] = ioff;
  };
  issue_next(0);
  issue_next(1);

  const double2 zero2 = make_double2(0.0, 0.0);
  double2 acc1 = zero2, acc0 = zero2;      // fiber / slice partial sums
  uint32_t j = 0;                          // rounds consumed

  // tiles gt in order, slab-major: slab gt / NT, leaf tile gt % NT
  for (uint32_t gt = 0; gt < NS * NT; ++gt) {
    const uint32_t s    = gt / NT, t = gt - s * NT;
    const int      sc0  = a.col0 + static_cast<int>(s) * kSlab;
    const int      sw   = min(kSlab, a.col_end - sc0);
    const bool     act  = (2 * gl) < sw;
    const int      c2   = act ? 2 * gl : 0;                    // this lane's columns in the slab
    const uint32_t poff = static_cast<uint32_t>(sc0 + c2) * 8u;   // this lane's columns of a parent row
    const uint32_t tcol = static_cast<uint32_t>((a.whole ? sc0 : 0) + c2) * 8u;
    double *       abase = accs + c2;
    // the lanes of this lane group that run the batch loop (they take the same trips)
    const uint32_t gmask = ((1u << min(L, (sw + 1) / 2)) - 1u) << (grp * L);
    auto flush = [&](uint32_t n) {                           // the slice closed: into smem
      double * p = abase + static_cast<size_t>(__ldg(&a.rootid[n]) - range_lo()) * kSlab;
      atomicAdd(p, acc0.x);
      atomicAdd(p + 1, acc0.y);
      acc0 = zero2;
    };
    // shared address of leaf row 0 (this lane's columns) as if the tile started there
    const uint32_t tile = smem_u32(tiles) + (gt & 1u) * a.tile_bytes + tcol - t * a.tile_rows * a.tpitch;
    // one or more rounds per tile (one, for a tile no larger than the policy picks); the
    // segment bounds are re-read every round rather than held across the batch loop
    for (uint32_t i = 0, more = 1; more; ++i, ++j) {
      uint32_t ws, we, gs, ge;
      part(t, warp * G, (warp + 1) * G, ws, we);
      part(t, warp * G + grp, warp * G + grp + 1, gs, ge);
      mbar_wait(&mybars[j & 1u], (j >> 1) & 1u);
      const uint32_t rs  = ws + i * kTRS;
      const uint32_t re  = min(we, rs + kTRS);
      const uint32_t lo  = max(gs, rs), hi = min(ge, re);
      more = (re < we) ? 1u : 0u;
      if (i == 0) mbar_wait(&tile_full[gt & 1u], (gt >> 1) & 1u);
      SpRec *        buf = myring + (j & 1u) * kTRS;
      // the group's last record of this tile closes the slice (sub-range boundary)
      if (leader && hi > lo && hi == ge)
        buf[hi - 1 - rs].aux = (buf[hi - 1 - rs].aux & SPB200_IDX_MASK) | (2u << SPB200_IDX_BITS);
      __syncwarp();
      if (act && hi > lo) {
        uint32_t n = lo;
        for (; n + kTB <= hi; n += kTB) {
          const SpRec * bq = buf + (n - rs);
          // parent gathers first, from the records' aux words; the close counts are kept one
          // byte per record
          double2  r[kTB];
          uint32_t cc = 0;
#pragma unroll
          for (int u = 0; u < kTB; ++u) {
            const uint32_t w = bq[u].aux;
            cc |= (w >> SPB200_IDX_BITS) << (8 * u);
            if (w >> SPB200_IDX_BITS) r[u] = ld_row_na(reinterpret_cast<const char *>(a.parent) + poff, w & SPB200_IDX_MASK, pitch);
          }
          // keeps the gathers ahead of the leaf fold: without it ptxas sinks them below the
          // first records' leaf reads to save registers (0.46 against 0.45 ms per mode)
          __syncwarp(gmask);
          // while they are in flight, the leaf rows fold into the fiber sums; a closing
          // record's fiber product waits in p[u] for its parent row (the last record's stays
          // in acc1, and p[kTB - 1] is never set)
          double2 p[kTB];
#pragma unroll
          for (int u = 0; u < kTB; ++u) {
            const uint4  q = *reinterpret_cast<const uint4 *>(&bq[u]);
            const double v = __hiloint2double(static_cast<int>(q.y), static_cast<int>(q.x));
            acc1           = vfma(v, lds_f64x2(tile + q.z * a.tpitch), acc1);
            if (u + 1 < kTB && ((cc >> (8 * u)) & 0xffu)) { p[u] = acc1; acc1 = zero2; }
          }
          auto close = [&](int u) {
            acc0 = vfma(u + 1 < kTB ? p[u] : acc1, r[u], acc0);
            if (u + 1 == kTB) acc1 = zero2;
          };
          if ((cc & 0xfefefefeu) == 0) {             // no slice ends in the batch
#pragma unroll
            for (int u = 0; u < kTB; ++u)
              if ((cc >> (8 * u)) & 0xffu) close(u);
          } else {
#pragma unroll
            for (int u = 0; u < kTB; ++u) {
              const uint32_t c = (cc >> (8 * u)) & 0xffu;
              if (c) {
                close(u);
                if (c >= 2) flush(n + u);
              }
            }
          }
        }
#pragma unroll 1
        for (; n < hi; ++n) {
          const uint4    q = *reinterpret_cast<const uint4 *>(&buf[n - rs]);
          const double   v = __hiloint2double(static_cast<int>(q.y), static_cast<int>(q.x));
          const uint32_t c = q.w >> SPB200_IDX_BITS;
          const double2  b = lds_f64x2(tile + q.z * a.tpitch);
          acc1             = vfma(v, b, acc1);
          if (c) {
            acc0 = vfma(acc1, ld_row_na(reinterpret_cast<const char *>(a.parent) + poff, q.w & SPB200_IDX_MASK, pitch), acc0);
            acc1 = zero2;
            if (c >= 2) flush(n);
          }
        }
      }
      __syncwarp();
      issue_next(j + 2);   // refill the stage just consumed
    }
    // this warp is done with tile gt; the last warp to get here loads tile gt + 2 in its place
    __syncwarp();
    uint32_t last = 0;
    if (lane == 0) {
      __threadfence_block();
      last = ((atomicAdd(&tile_left[gt & 1u], 1u) + 1u) % kTW == 0) ? 1u : 0u;   // counts on
      __threadfence_block();
    }
    if (__shfl_sync(0xffffffffu, last, 0) && gt + 2 < NS * NT) load_tile(gt + 2);

    if (t + 1 < NT) continue;
    // the slab is complete: interior rows belong to this range alone and are stored; the
    // first and last row may be shared with the neighbouring ranges and are reduced
    __syncthreads();
    const uint32_t pairs = static_cast<uint32_t>(sw) / 2u;
    const uint32_t nrows = range_rows(), r_lo = range_lo();
    for (uint32_t i = threadIdx.x; i < nrows * pairs; i += kTW * 32) {
      const uint32_t row = i / pairs, c = 2u * (i % pairs);
      double2 *      src = reinterpret_cast<double2 *>(accs + static_cast<size_t>(row) * kSlab + c);
      const double2  v   = *src;
      *src = zero2;
      double * dst = a.out + static_cast<size_t>(r_lo + row) * a.ldm + sc0 + c;
      if (row == 0 || row + 1 == nrows) {
        atomicAdd(dst, v.x);
        atomicAdd(dst + 1, v.y);
      } else {
        *reinterpret_cast<double2 *>(dst) = v;
      }
    }
    __syncthreads();
  }
}

}  // namespace spb200

// smem the kernel needs for a tile of `tile_rows` and an accumulator of `acc_rows` rows
static size_t tiled_smem_bytes(uint32_t tile_rows, uint32_t acc_rows) {
  using namespace spb200;
  return (2 * (size_t)tile_rows + acc_rows) * kSlab * 8 + sizeof(SpRec) * kTW * 2 * kTRS +
         sizeof(uint64_t) * (4 + 3 * kTW) + 128;
}

uint32_t spb200_tiled_rows_for(uint32_t acc_rows) {
  const size_t fixed = tiled_smem_bytes(0, acc_rows);
  if (fixed >= 227 * 1024) return 0;
  return (uint32_t)((227 * 1024 - fixed) / 2 / (spb200::kSlab * 8));
}

bool spb200_tiled_applicable(const FiberStream & s, int kind) {
  return s.nmodes == 3 && kind == SPB200_KIND_ROOT && s.seg_off && s.rootid && s.rroot &&
         s.ntiles > 0 && tiled_smem_bytes(s.ktile_rows, s.acc_rows) <= 227 * 1024;
}

int spb200_launch_tiled_root3(const FiberStream & s, int ldm, int col_begin, int col_end,
                              const double * leaf, const double * parent, double * d_out,
                              cudaStream_t stream) {
  using namespace spb200;
  TiledArgs a;
  a.rec = s.rec; a.rootid = s.rootid; a.seg_off = s.seg_off; a.rroot = s.rroot;
  a.leaf = leaf; a.parent = parent; a.out = d_out;
  a.ntiles = s.ntiles; a.tile_rows = s.ktile_rows; a.leaf_rows = (uint32_t)s.leaf_rows;
  a.acc_rows = s.acc_rows;
  a.ldm = ldm; a.col0 = col_begin; a.col_end = col_end;
  a.whole = (col_end - col_begin <= kSlab && ldm <= kSlab) ? 1 : 0;
  a.tile_bytes = s.ktile_rows * kSlab * 8u;
  a.tpitch = a.whole ? (uint32_t)ldm * 8u : kSlab * 8u;
  const size_t smem = tiled_smem_bytes(s.ktile_rows, s.acc_rows);
  const int threads = kTW * 32;
  const unsigned grid = s.kranges;
#define SPB200_TILED_LAUNCH(LL)                                                                   \
  do {                                                                                            \
    static bool set[64] = {false};          /* function attributes are per device */            \
    int dev_ = 0;                                                                                 \
    SPB200_CUDA_OK(cudaGetDevice(&dev_));                                                         \
    if (dev_ < 0 || dev_ >= 64 || !set[dev_]) {                                                   \
      SPB200_CUDA_OK(cudaFuncSetAttribute(mttkrp_tiled_root3<LL>,                                 \
                                          cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024)); \
      SPB200_CUDA_OK(cudaFuncSetAttribute(mttkrp_tiled_root3<LL>,                                 \
                                          cudaFuncAttributePreferredSharedMemoryCarveout,         \
                                          cudaSharedmemCarveoutMaxShared));                       \
      if (dev_ >= 0 && dev_ < 64) set[dev_] = true;                                               \
    }                                                                                             \
    mttkrp_tiled_root3<LL><<<grid, threads, smem, stream>>>(a);                                   \
  } while (0)
  const int width = col_end - col_begin;
  if (width <= 8) SPB200_TILED_LAUNCH(4);
  else if (width <= 16) SPB200_TILED_LAUNCH(8);
  else SPB200_TILED_LAUNCH(16);
#undef SPB200_TILED_LAUNCH
  spb200_count_launches(1);
  SPB200_CUDA_OK(cudaGetLastError());
  return SPLATT_SUCCESS;
}
