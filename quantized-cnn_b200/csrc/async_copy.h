// Asynchronous global -> shared copies and the mbarriers that count them (sm_90), shared by the kernels of the library.
#ifndef QCNN_ASYNC_COPY_H_
#define QCNN_ASYNC_COPY_H_

#include <stdint.h>

namespace qcnn {

__device__ __forceinline__ uint32_t SmemU32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// cp.async of 4 / 16 bytes; src-size 0 (valid = false): nothing is read, the destination bytes are zero-filled
__device__ __forceinline__ void CpAsync4(void* smemDst, const void* gsrc, bool valid) {
  const int sz = valid ? 4 : 0;
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(SmemU32(smemDst)), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void CpAsync16(void* smemDst, const void* gsrc, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(SmemU32(smemDst)), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void CpAsyncCommit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void CpAsyncWaitAll() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ void MbarInit(uint64_t* b, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(SmemU32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void MbarArrive(uint64_t* b) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(SmemU32(b)) : "memory");
}
__device__ __forceinline__ void MbarExpectTx(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(SmemU32(b)), "r"(bytes) : "memory");
}
// bounded spin: a protocol error traps (launch failure) after 2^kSpinLog2 polls instead of hanging the GPU
template <int kSpinLog2>
__device__ __forceinline__ void MbarWait(uint64_t* b, uint32_t parity) {
  uint32_t done = 0;
  for (uint32_t spins = 0; !done; spins++) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(SmemU32(b)), "r"(parity) : "memory");
    if (spins > (1u << kSpinLog2)) __trap();
  }
}
// bulk copy of `bytes` (multiple of 16) whose completion is counted on the mbarrier `bar`
__device__ __forceinline__ void BulkLoad(void* smemDst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(SmemU32(smemDst)), "l"(gsrc), "r"(bytes), "r"(SmemU32(bar)) : "memory");
}

}  // namespace qcnn

#endif  // QCNN_ASYNC_COPY_H_
