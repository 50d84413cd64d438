// The parts of the weight-stationary wgmma GEMMs (conv_ws.cu: convolutions, fc_ws.cu: fully-connected layers) that do not
// depend on the layer's geometry:
//   - the CTA of twelve warps: warps 0-7 two consumer warpgroups (wgmma), warps 8-11 producers (staging + weight decode);
//   - one k-step of the MMA loop: A = bf16x2 rows of the staged planes ([x1 | x2]: K-core-matrix 0 in the x1 plane, 1 in
//     the x2 plane, LBO = the plane distance), B = decoded weights [w1, w2][channel] 16-byte rows in shared memory with
//     the duplicated half read twice (LBO = 0), two MMAs into one accumulator per m64 block:
//         [x1|x2].[w1|w1] + [x1|x2].[w2|w2] = (x1 + x2)(w1 + w2);
//   - the release of a weight stage by the consumers (its MMAs have retired) and the mbarrier set-up of the rings;
//   - the accumulator fragment -> (row, channel) mapping of the epilogues.
#ifndef QCNN_WS_COMMON_CUH_
#define QCNN_WS_COMMON_CUH_

#include <stdint.h>

#include "async_copy.h"
#include "wgmma.h"

namespace qcnn {

constexpr int kWsThreads = 384;
constexpr int kWsConsumers = 256;   // warps 0-7
constexpr int kWsProducers = 128;   // warps 8-11

// the four producer warps only (named barrier 1; barrier 0 is __syncthreads)
__device__ __forceinline__ void WsProducerSync() { asm volatile("bar.sync 1, %0;" :: "n"(kWsProducers) : "memory"); }

// Rings of plane buffers (nPB) and the two weight buffers: full[i] counts the producers' arrivals (fullCount: every
// producer thread, or 1 when the buffer arrives by bulk copy with its byte count), empty[i] one arrival per consumer warp.
__device__ __forceinline__ void WsInitBarriers(uint64_t* fullP, uint64_t* emptyP, int nPB, int fullPCount, uint64_t* fullW,
                                               uint64_t* emptyW) {
  for (int i = 0; i < nPB; i++) { MbarInit(fullP + i, fullPCount); MbarInit(emptyP + i, kWsConsumers / 32); }
  for (int i = 0; i < 2; i++) { MbarInit(fullW + i, kWsProducers); MbarInit(emptyW + i, kWsConsumers / 32); }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// One k-step into the MB accumulators of a consumer warpgroup: the A rows of m64 block m start at row bStart + 64 m of
// the x1 plane at plA (the x2 plane lboBytes further), the k-step's weights [w1 | w2][NC channels] at wb.
template <int NC, int MB>
__device__ __forceinline__ void WsMmaKStep(float (&acc)[MB][NC / 2], uint32_t plA, int bStart, uint32_t lboBytes, uint32_t wb) {
  const uint64_t d1 = WgmmaDesc(wb, 0, 128), d2 = WgmmaDesc(wb + NC * 16, 0, 128);
#pragma unroll
  for (int m = 0; m < MB; m++) {
    const uint64_t dA = WgmmaDesc(plA + static_cast<uint32_t>(bStart + m * 64) * 16u, lboBytes, 128);
    WgmmaSS<NC>::Bf16(acc[m], dA, d1);
    WgmmaSS<NC>::Bf16(acc[m], dA, d2);
  }
}

// end of a weight stage: every MMA of the warpgroup has retired, then one arrival per warp frees the stage's buffer
__device__ __forceinline__ void WsRetireStage(uint64_t* emptyW, int lane) {
  WgmmaCommit();
  WgmmaWaitAll();
  __syncwarp();
  if (lane == 0) MbarArrive(emptyW);
}

// Accumulator fragment of a consumer thread (m64 x N, one 16-row slice per warp): acc[4 i + 2 h] and acc[4 i + 2 h + 1]
// hold row r0 + 8 h, columns 8 i + 2 t4 and 8 i + 2 t4 + 1
struct WsFrag {
  int r0, t4;
};
__device__ __forceinline__ WsFrag WsFragOf(int warp, int lane) { return {(warp & 3) * 16 + (lane >> 2), lane & 3}; }

}  // namespace qcnn

#endif  // QCNN_WS_COMMON_CUH_
