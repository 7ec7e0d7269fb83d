// Instantiation unit: compiled once per mode count (-DSPB200_INST_N=2..8) so the
// 6 x 4 x 3 kernel variants build in parallel; with -DSPB200_INST_F32 the fp32 kernels of
// that mode count (launch_f32_n<N>) instead of the fp64 ones (launch_n<N>).
#include <type_traits>
#include "mttkrp_kernels.cuh"

#ifndef SPB200_INST_N
#error "compile with -DSPB200_INST_N=<nmodes>"
#endif

int spb200_root_batch();
int spb200_root_minb();

namespace spb200 {

#ifdef SPB200_INST_F32
using Val = float;
#else
using Val = double;
#endif

// fp32 register budget by (N, kind): the registers of the fp64 default-batch kernel of the same
// N and kind (ptxas, sm_90a, CUDA 12.9; the lowest over L).  Left to itself ptxas gives many
// fp32 kernels 1-8 registers more than their fp64 counterpart, and the 5-mode leaf kernels go
// from 64 to 68-70, i.e. from 4 to 3 CTAs per SM; held to these counts an fp32 kernel never
// runs fewer CTAs per SM than the fp64 one (and none spills).  tests/test_mttkrp_f32.py checks
// the built library kernel by kernel against its fp64 counterpart.
constexpr int kF32Regs[SPB200_MAXN - 1][3] = {
    // root, internal, leaf
    {42, 54, 54},    // N = 2
    {80, 46, 48},    // N = 3
    {80, 62, 56},    // N = 4
    {80, 72, 64},    // N = 5
    {90, 90, 77},    // N = 6
    {94, 103, 84},   // N = 7
    {96, 114, 96},   // N = 8
};

template <int N, int L, int KIND, int BATCH, bool KT = false, bool MC = false, int MINB = 0,
          int STAGES = kStages>
static int launch_variant(const MttkrpArgs & args, int num_sms, cudaStream_t stream) {
  auto kern = [] {
    if constexpr (std::is_same<Val, float>::value)
      return mttkrp_stream_kernel<Val, N, L, KIND, BATCH, KT, MC, default_minb(N, BATCH), STAGES,
                                  kF32Regs[N - 2][KIND]>;
    else if constexpr (MINB == 0) return mttkrp_stream_kernel<Val, N, L, KIND, BATCH, KT, MC>;
    else return mttkrp_stream_kernel<Val, N, L, KIND, BATCH, KT, MC, MINB, STAGES>;
  }();
  static_assert(MINB != 0 || STAGES == kStages, "a non-default ring depth needs an explicit MINB");
  const size_t smem = smem_bytes(STAGES, KIND == SPB200_KIND_ROOT && N >= 4, 32 / L, args.rpad, args.apad);
  // function attributes and occupancy are per DEVICE (and per stagger setting): cache them
  static int occ_of[64] = {0};
  static size_t smem_of[64] = {0};
  int dev = 0;
  SPB200_CUDA_OK(cudaGetDevice(&dev));
  const int slot = (dev >= 0 && dev < 64) ? dev : 0;
  if (occ_of[slot] == 0 || dev != slot || smem_of[slot] != smem) {
    smem_of[slot] = smem;
    SPB200_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        static_cast<int>(smem)));
    int o = 0;
    SPB200_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, kern, kThreads, smem));
    occ_of[slot] = o > 0 ? o : 1;
  }
  const int occ = occ_of[slot];
  constexpr int G = 32 / L;
  // never launch more groups than there are chunks
  unsigned long long want = (static_cast<unsigned long long>(args.nchunks) + kWarps * G - 1) / (kWarps * G);
  unsigned long long grid = static_cast<unsigned long long>(num_sms) * occ;
  if (grid > want) grid = want;
  if (grid == 0) {
    if (args.sync_mc == nullptr) return SPLATT_SUCCESS;
    grid = 1;                      // an empty shard still takes part in the group barrier
  }
  kern<<<static_cast<unsigned>(grid), kThreads, smem, stream>>>(args);
  spb200_count_launches(1);
  SPB200_CUDA_OK(cudaGetLastError());
  return SPLATT_SUCCESS;
}

template <int N, int L>
static int launch_kind(int kind, const MttkrpArgs & args, int num_sms, cudaStream_t stream) {
  switch (kind) {
    case SPB200_KIND_ROOT:
      if constexpr (std::is_same<Val, float>::value) {
        // fp32: only the default batch of each N (multicast and the tuning knobs are fp64 only)
        if constexpr (N >= 4) return launch_variant<N, L, SPB200_KIND_ROOT, 2>(args, num_sms, stream);
        else if (args.ktiled) return launch_variant<N, L, SPB200_KIND_ROOT, 4, true>(args, num_sms, stream);
        else return launch_variant<N, L, SPB200_KIND_ROOT, 4>(args, num_sms, stream);
      } else {
        if (args.multicast) return launch_variant<N, L, SPB200_KIND_ROOT, 4, false, true>(args, num_sms, stream);
        if (spb200_root_batch() >= 8) return launch_variant<N, L, SPB200_KIND_ROOT, 8>(args, num_sms, stream);
        if constexpr (N == 4) {   // tuning variants of the 4-mode kernel (SPLATT_B200_BATCH / _MINB)
          const int b = spb200_root_batch(), mb = spb200_root_minb();
          if (b == 3 && mb == 3) return launch_variant<N, L, SPB200_KIND_ROOT, 3, false, false, 3>(args, num_sms, stream);
          if (b == 3) return launch_variant<N, L, SPB200_KIND_ROOT, 3, false, false, 2>(args, num_sms, stream);
          if (b == 4 && mb == 3) return launch_variant<N, L, SPB200_KIND_ROOT, 4, false, false, 3>(args, num_sms, stream);
          if (b == 2 && mb == 4) return launch_variant<N, L, SPB200_KIND_ROOT, 2, false, false, 4, 2>(args, num_sms, stream);
        }
        if constexpr (N == 3) {   // 32 warps per SM: 4 CTAs of <= 64 registers
          if (spb200_root_batch() == 2 && spb200_root_minb() == 4)
            return launch_variant<N, L, SPB200_KIND_ROOT, 2, false, false, 4>(args, num_sms, stream);
          if (spb200_root_batch() == 4 && spb200_root_minb() == 4)
            return launch_variant<N, L, SPB200_KIND_ROOT, 4, false, false, 4>(args, num_sms, stream);
          if (spb200_root_batch() == 3 && spb200_root_minb() == 4)
            return launch_variant<N, L, SPB200_KIND_ROOT, 3, false, false, 4>(args, num_sms, stream);
          if (spb200_root_batch() == 3 && spb200_root_minb() == 3)
            return launch_variant<N, L, SPB200_KIND_ROOT, 3, false, false, 3>(args, num_sms, stream);
        }
        // deeper trees hold a third gathered row per record: two-record batches keep the
        // kernel at 80 registers / 3 CTAs per SM (measured 1014 vs 1052 us on config 3)
        if (spb200_root_batch() == 2 || (spb200_root_batch() == 0 && N >= 4))
          return launch_variant<N, L, SPB200_KIND_ROOT, 2>(args, num_sms, stream);
        if (args.ktiled) return launch_variant<N, L, SPB200_KIND_ROOT, 4, true>(args, num_sms, stream);
        return launch_variant<N, L, SPB200_KIND_ROOT, 4>(args, num_sms, stream);
      }
    case SPB200_KIND_INTL: return launch_variant<N, L, SPB200_KIND_INTL, 4>(args, num_sms, stream);
    default:               return launch_variant<N, L, SPB200_KIND_LEAF, 4>(args, num_sms, stream);
  }
}

#define SPB200_CAT_(a, b) a##b
#define SPB200_CAT(a, b) SPB200_CAT_(a, b)

#ifdef SPB200_INST_F32
#define SPB200_LAUNCH_NAME SPB200_CAT(launch_f32_n, SPB200_INST_N)
#else
#define SPB200_LAUNCH_NAME SPB200_CAT(launch_n, SPB200_INST_N)
#endif

// ncols: active columns of this launch (a multiple of W), <= 32 * W (fp64: 64, fp32: 128).
int SPB200_LAUNCH_NAME(int kind, const MttkrpArgs & args, int num_sms, cudaStream_t stream) {
  constexpr int N = SPB200_INST_N;
  constexpr int W = LaneVec<Val>::W;
  if (args.ncols <= 4 * W)  return launch_kind<N, 4>(kind, args, num_sms, stream);
  if (args.ncols <= 8 * W)  return launch_kind<N, 8>(kind, args, num_sms, stream);
  if (args.ncols <= 16 * W) return launch_kind<N, 16>(kind, args, num_sms, stream);
  return launch_kind<N, 32>(kind, args, num_sms, stream);
}

}  // namespace spb200
