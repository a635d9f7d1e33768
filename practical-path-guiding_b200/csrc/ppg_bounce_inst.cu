// ppg_bounce_inst.cu -- one (SMEM, FULL) family of bounce_kernel instantiations per translation unit:
//   nvcc -DPPG_INST_SMEM={0,1} -DPPG_INST_FULL={0,1} -c ppg_bounce_inst.cu
#include "ppg_bounce.cuh"

using namespace ppg;

#define PPG_CAT2(a, b, c) a##b##c
#define PPG_CAT(a, b, c) PPG_CAT2(a, b, c)
#define LAUNCH_NAME PPG_CAT(ppg_launch_bounce_, PPG_INST_SMEM, PPG_INST_FULL)
#define OCC_NAME PPG_CAT(ppg_bounce_occupancy_, PPG_INST_SMEM, PPG_INST_FULL)

namespace {
constexpr bool kSmem = PPG_INST_SMEM != 0, kFull = PPG_INST_FULL != 0;
constexpr int kBlock = kSmem ? PPG_BOUNCE_BLOCK : PPG_BOUNCE_BLOCK_HBM;
template <bool FIRST> void launch(const RenderParams &P, const BounceLaunch &L) {
    const size_t sm = P.sceneSmemBytes;
    if (L.nee) {      // next event estimation always runs with full records
        if (L.record == 0) bounce_kernel<FIRST, 0, true, kSmem, kFull><<<L.grid, kBlock, sm, L.stream>>>(P);
        else bounce_kernel<FIRST, 2, true, kSmem, kFull><<<L.grid, kBlock, sm, L.stream>>>(P);
    } else if (L.record == 0) bounce_kernel<FIRST, 0, false, kSmem, kFull><<<L.grid, kBlock, sm, L.stream>>>(P);
    else if (L.record == 1) bounce_kernel<FIRST, 1, false, kSmem, kFull><<<L.grid, kBlock, sm, L.stream>>>(P);
    else bounce_kernel<FIRST, 2, false, kSmem, kFull><<<L.grid, kBlock, sm, L.stream>>>(P);
}
}  // namespace

namespace ppg {
void LAUNCH_NAME(const RenderParams &P, const BounceLaunch &L) { if (L.first) launch<true>(P, L); else launch<false>(P, L); }
int OCC_NAME(size_t smem) {
    int occ = 0;
    if (kFull) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, bounce_kernel<false, 2, true, kSmem, kFull>, kBlock, smem);
    else cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, bounce_kernel<false, 1, false, kSmem, kFull>, kBlock, smem);
    return occ;
}
}  // namespace ppg
