// Convolutions as a weight-stationary GEMM on the Hopper tensor cores, with the roles of pq_gemm_tc transposed:
//
//     dst[q][c] = bias[c] + sum_{k-steps} sum_{j<16} X_kstep[q][j] * W_kstep[c][j]       (M = positions, N = channels)
//
// Two position geometries, the ones pq_gemm_tc uses for the same layers (its k-step tables, Mode0Table / Mode1Table):
//   stride 1 (mode 0, conv2-conv5, VGG16): all images form one flat padded grid; a chunk is 8 input channels x all taps,
//     and a 16-byte row of a plane holds the 8 channels of one position; a tap is a start-address shift of the A
//     descriptor.  A group of <= 3 channels (an RGB first layer) is one chunk whose second half is zeros.
//   strided over <= 4 input channels (mode 1, conv1: 11x11 / 4 over 3 channels): the input is de-interleaved into phase
//     planes; a 16-byte row holds two phase columns x 4 channels of one position; a chunk is one phase row.
//
// A = positions: bf16x2 planes (x = x1 + x2; K-core-matrix 0 in the x1 plane, 1 in the x2 plane: LBO = plane distance),
//     read by descriptor.
// B = decoded weights in shared memory, N = the channels of one CTA: Cout / grp, or a 1/nct tile of it (any instantiated
//     width up to 256: no channel padding).  Per k-step, [w1 | w1] and [w2 | w2] are 16-byte rows per channel; the
//     duplicated half is the same core matrix read twice (LBO = 0).  Two MMAs per k-step into one accumulator:
//     [x1|x2].[w1|w1] + [x1|x2].[w2|w2] = (x1 + x2)(w1 + w2), the same k-steps in the same order as pq_gemm_tc's one-
//     accumulator tiling of the same geometry (the error bound depends on that chain, DESIGN.md 2).
//
// Roles inside a CTA of twelve warps:
//   warps 0-7   two consumer warpgroups; each owns MB m64 blocks of the CTA's 128 MB positions and issues
//               wgmma.mma_async (both operands in shared memory) into MB accumulators of N / 2 registers per thread.
//   warps 8-11  producers: stage the position planes (global -> bf16x2 split -> planes; mode 1: every phase row resident,
//               mode 0: a ring of plane buffers, one chunk each, with a full / empty mbarrier pair per buffer), and decode
//               the weights of one stage (<= KS k-steps of one chunk, all N channels) from the pre-split codebook and the
//               channel-major index block into one of two weight buffers.  The decode is done once per CTA and reused by
//               both warpgroups and every m64 block; decoded weights never reach global memory.
//   epilogue    the consumers add the bias (+ ReLU) and store pairs of consecutive channels of one NHWC pixel.
#include "qcnn_internal.h"
#include "wgmma.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>

namespace {

using qcnn::ByteOf32;
using qcnn::MbarArrive;
using qcnn::MbarInit;
using qcnn::MbarWait;
using qcnn::SmemU32;
using qcnn::SplitBf16x4;
using qcnn::WgmmaDesc;

constexpr int kWsThreads = 384;
constexpr int kWsConsumers = 256;   // warps 0-7
constexpr int kWsProducers = 128;   // warps 8-11
constexpr int kWsRegPos = 8;        // mode 0: float4 of a chunk's planes a producer thread stages per register pass

// the four producer warps only (named barrier 1; barrier 0 is __syncthreads)
__device__ __forceinline__ void ProducerSync() { asm volatile("bar.sync 1, %0;" :: "n"(kWsProducers) : "memory"); }

// Shared-memory carve, read by the planner (fits / does not fit) and by the kernel.  a.NT = positions per CTA,
// a.GT = k-steps per weight stage (KS), a.Kg / a.nct = channels per CTA (N of the MMA), a.nPB = plane buffers (mode 1:
// one per phase row, mode 0: the ring).
struct WsSmem {  // byte offsets inside the dynamic shared memory
  int planes, wts, cb, outoff, bias, bars, total;
};
__host__ __device__ inline WsSmem MapWsSmem(const GemmArgs& a) {
  const int nc = a.Kg / a.nct;
  WsSmem m;
  int o = 0;
  m.planes = o; o += a.nPB * 2 * a.planeRows * 16;        // [buffer][x1, x2][planeRows] 16-byte rows
  m.wts = o;    o += 2 * a.GT * 2 * nc * 16;              // [buffer][k-step][w1, w2][channel] 16-byte rows
  m.cb = o;     o += (a.mode == 0 ? 2 : 1) * a.K * 16;    // pre-split codebook slices {w1, w2} (mode 0: one per half)
  m.outoff = o; o += a.NT * 4;                            // destination element offset of every position (-1: none)
  m.bias = o;   o += nc * 4;                              // (nc is a multiple of 16: the barriers stay 8-byte aligned)
  m.bars = o;   o += 8 * (2 * a.nPB + 4);
  m.total = o;
  return m;
}

// NC: channels per CTA; MB: m64 blocks per consumer warpgroup; S1: the stride-1 geometry (mode 0), else mode 1;
// WIDE (stride 1): a chunk's planes take more than one register pass of the producers, or a group has <= 3 channels
// (kept apart so that the single-pass kernels AlexNet runs carry none of that staging)
template <int NC, int MB, bool S1, bool WIDE>
__global__ void __launch_bounds__(kWsThreads, 1) conv_ws_kernel(const GemmArgs a) {
  constexpr int P = 128 * MB;   // positions per CTA
  extern __shared__ __align__(128) unsigned char smem[];
  const WsSmem sm = MapWsSmem(a);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int KS = a.GT, nPB = a.nPB;
  const int nCh = S1 ? a.nChunks : a.stride;   // chunks: 8-channel groups (mode 0) / phase rows (mode 1)
  uint4* planes = reinterpret_cast<uint4*>(smem + sm.planes);
  uint4* wts = reinterpret_cast<uint4*>(smem + sm.wts);
  uint4* cb = reinterpret_cast<uint4*>(smem + sm.cb);
  int* outoff = reinterpret_cast<int*>(smem + sm.outoff);
  float* biasS = reinterpret_cast<float*>(smem + sm.bias);
  uint64_t* fullP = reinterpret_cast<uint64_t*>(smem + sm.bars);   // [nPB] planes of a chunk staged: producers -> consumers
  uint64_t* emptyP = fullP + nPB;                                   // [nPB] (mode 0) planes' MMAs retired: consumers -> producers
  uint64_t* fullW = emptyP + nPB;                                   // [2] weight buffer decoded: producers -> consumers
  uint64_t* emptyW = fullW + 2;                                     // [2] weight buffer's MMAs retired: consumers -> producers
  int bi = blockIdx.x;
  const int ct = bi % a.nct; bi /= a.nct;   // (channel tile, group, position tile)
  const int g = bi % a.G, tile = bi / a.G;
  const int ch0 = ct * NC;                  // first channel of the tile inside the group
  const int Q0 = tile * P;                  // first flat position (grid of IB positions per image)
  const int i0 = Q0 / a.IB;                 // first image touched
  float* dstBase = a.dst + static_cast<size_t>(i0) * a.dstImg + g * a.Kg + ch0;

  // ---- set-up (all threads) ----
  for (int p = tid; p < P; p += kWsThreads) {
    const int Q = Q0 + p;
    const int i = Q / a.IB, rem = Q - i * a.IB;
    const int ho = rem / a.PW, wo = rem - ho * a.PW;
    outoff[p] = (i < a.N && ho < a.Ho && wo < a.Wo) ? (((i - i0) * a.Ho + ho) * a.Wo + wo) * a.Cout : -1;
  }
  if (!S1)
    for (int k = tid; k < a.K; k += kWsThreads) cb[k] = __ldg(reinterpret_cast<const uint4*>(a.ctrd) + k);
  for (int c = tid; c < NC; c += kWsThreads) biasS[c] = __ldg(a.bias + g * a.Kg + ch0 + c);
  if (tid == 0) {
    for (int i = 0; i < nPB; i++) { MbarInit(fullP + i, kWsProducers); MbarInit(emptyP + i, kWsConsumers / 32); }
    for (int i = 0; i < 2; i++) { MbarInit(fullW + i, kWsProducers); MbarInit(emptyW + i, kWsConsumers / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int warpU = __shfl_sync(0xffffffffu, warp, 0);   // provably warp-uniform role selector
  if (warpU >= kWsConsumers / 32) {
    // =========================== producers ===========================
    const int pt = tid - kWsConsumers;
    int j = 0;   // weight stage counter (buffer j & 1)
    if constexpr (S1) {
      // float4 p = pt + (q * kWsRegPos + i) * kWsProducers of pass q of a chunk's planes: half = p / NPOS (channels 0-3 /
      // 4-7 of the chunk), position = p % NPOS -> pixel (r - pad, c - pad) of image i of the flat padded grid.  The 2 NPOS
      // float4 of a chunk take nPass register passes; the source offsets and validity of a pass are chunk-invariant
      // (computed once with a single pass, per pass otherwise)
      const int taps = a.ntab;
      const int nPass = WIDE ? (2 * a.NPOS + kWsRegPos * kWsProducers - 1) / (kWsRegPos * kWsProducers) : 1;
      const float* srcBase = a.src + static_cast<size_t>(i0) * a.srcImg + g * a.Cg;
      int poff[kWsRegPos];
      uint32_t pvalid = 0, phalf = 0;
      auto passPos = [&](int q) {
        pvalid = 0; phalf = 0;
#pragma unroll
        for (int i = 0; i < kWsRegPos; i++) {
          const int p = pt + (q * kWsRegPos + i) * kWsProducers;
          poff[i] = 0;
          if (p < 2 * a.NPOS) {
            const bool hb = p >= a.NPOS;
            const int F = Q0 + (hb ? p - a.NPOS : p);
            const int im = F / a.IB, rem = F - im * a.IB;
            const int r = rem / a.PW, c = rem - r * a.PW;
            if (im < a.N && r >= a.pad && c >= a.pad) {
              poff[i] = (((im - i0) * a.Hi + (r - a.pad)) * a.Wi + (c - a.pad)) * a.Cin + (hb ? 4 : 0);
              pvalid |= 1u << i;
            }
            if (hb) phalf |= 1u << i;
          }
        }
      };
      float4 rg[kWsRegPos];
      // the current pass's positions of chunk kc into registers; a half beyond the group's channels (Cg % 8 == 4, Cg <= 3)
      // stages zeros
      auto loadPos = [&](int kc) {
        const int chA = kc * 8;
        const uint32_t m = chA + 4 >= a.Cg ? pvalid & ~phalf : pvalid;
        const float* srcG = srcBase + chA;
        if (!WIDE || a.Cg >= 4) {
#pragma unroll
          for (int i = 0; i < kWsRegPos; i++) {
            rg[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
            if ((m >> i) & 1u) rg[i] = __ldg(reinterpret_cast<const float4*>(srcG + poff[i]));
          }
        } else {
          // <= 3 channels (one chunk): the pixel pitch is not 16-byte aligned, the channels are read as scalars
#pragma unroll
          for (int i = 0; i < kWsRegPos; i++) {
            rg[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
            if ((m >> i) & 1u) {
              const float* px = srcG + poff[i];
              rg[i].x = __ldg(px);
              if (a.Cg > 1) rg[i].y = __ldg(px + 1);
              if (a.Cg > 2) rg[i].z = __ldg(px + 2);
            }
          }
        }
      };
      // pass q of the registers v into the plane buffer {x1, x2}: row = position (16 bytes = the chunk's 8 channels), the
      // half selects bytes 0-7 / 8-15
      auto storePass = [&](const float4 (&v)[kWsRegPos], int q, char* x1, char* x2) {
#pragma unroll
        for (int i = 0; i < kWsRegPos; i++) {
          const int p = pt + (q * kWsRegPos + i) * kWsProducers;
          if (p < 2 * a.NPOS) {
            uint2 p1, p2;
            SplitBf16x4(v[i], p1, p2);
            const int db = p >= a.NPOS ? (p - a.NPOS) * 16 + 8 : p * 16;
            *reinterpret_cast<uint2*>(x1 + db) = p1;
            *reinterpret_cast<uint2*>(x2 + db) = p2;
          }
        }
      };
      passPos(0);
      loadPos(0);
      for (int kc = 0; kc < nCh; kc++) {
        const int pb = kc % nPB;
        if (kc >= nPB) MbarWait<24>(emptyP + pb, ((kc / nPB) - 1) & 1);   // buffer last read by the MMAs of chunk kc - nPB
        char* x1 = reinterpret_cast<char*>(planes + pb * 2 * a.planeRows);
        char* x2 = x1 + a.planeRows * 16;
        if (nPass == 1) {
          storePass(rg, 0, x1, x2);
        } else {
          for (int q = 0; q < nPass; q++) {
            float4 cur[kWsRegPos];
#pragma unroll
            for (int i = 0; i < kWsRegPos; i++) cur[i] = rg[i];
            if (q + 1 < nPass) { passPos(q + 1); loadPos(kc); }   // the next pass's loads are in flight during this split
            storePass(cur, q, x1, x2);
          }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // planes are read by the tensor core
        MbarArrive(fullP + pb);
        if (kc + 1 < nCh) {   // in flight during the decode below
          if (nPass > 1) passPos(0);
          loadPos(kc + 1);
        }
        // the chunk's two 4-channel halves: subspace and piece of each (as pq_gemm_tc's fetchChunk); a half beyond the
        // group's channels gets a zero codebook slice (its positions are zeros too)
        const int chA = kc * 8, chB = chA + 4;
        const bool okB = chB < a.Cg;
        const int sA = chA / a.d, jA = chA - sA * a.d;
        const int sB = okB ? chB / a.d : 0, jB = okB ? chB - sB * a.d : 0;
        const uint4* cA = reinterpret_cast<const uint4*>(a.ctrd) + static_cast<size_t>(sA * (a.d >> 2) + (jA >> 2)) * a.K;
        const uint4* cB = reinterpret_cast<const uint4*>(a.ctrd) + static_cast<size_t>(sB * (a.d >> 2) + (jB >> 2)) * a.K;
        ProducerSync();   // every producer is done decoding from the previous chunk's slices
        for (int k = pt; k < a.K; k += kWsProducers) {
          cb[k] = __ldg(cA + k);
          cb[a.K + k] = okB ? __ldg(cB + k) : make_uint4(0u, 0u, 0u, 0u);
        }
        ProducerSync();
        // weights of the chunk's stages: a thread owns channel c, its tap indices of either half are one or two 16-byte
        // granules of the channel-major block d_asmt_t ([grp][S][KgPad][tapsPad])
        const uint8_t* rowA = a.asmtT + (static_cast<size_t>(g * a.S + sA) * a.KgPad + ch0) * a.tapsPad;
        const uint8_t* rowB = a.asmtT + (static_cast<size_t>(g * a.S + sB) * a.KgPad + ch0) * a.tapsPad;
        for (int s0 = 0; s0 < taps; s0 += KS, j++) {
          const int n = min(KS, taps - s0), b = j & 1;
          if (j >= 2) MbarWait<24>(emptyW + b, ((j >> 1) - 1) & 1);   // buffer last read by the MMAs of stage j - 2
          uint4* w = wts + b * KS * 2 * NC;
          for (int c = pt; c < NC; c += kWsProducers) {
            const uint4* iA = reinterpret_cast<const uint4*>(rowA + static_cast<size_t>(c) * a.tapsPad);
            const uint4* iB = reinterpret_cast<const uint4*>(rowB + static_cast<size_t>(c) * a.tapsPad);
            const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
            const uint4 a0 = __ldg(iA), a1 = a.tapsPad > 16 ? __ldg(iA + 1) : zero;
            const uint4 b0 = __ldg(iB), b1 = a.tapsPad > 16 ? __ldg(iB + 1) : zero;
            // (no unroll pragma: see the mode-1 decode loop below)
            for (int e = 0; e < n; e++) {
              const int t = a.tab[s0 + e].idx0;   // the tap of k-step s0 + e
              const uint4 qa = cb[ByteOf32(a0, a1, t)];
              const uint4 qb = cb[a.K + ByteOf32(b0, b1, t)];
              w[(2 * e + 0) * NC + c] = make_uint4(qa.x, qa.y, qb.x, qb.y);   // [w1 of half A | w1 of half B]
              w[(2 * e + 1) * NC + c] = make_uint4(qa.z, qa.w, qb.z, qb.w);   // [w2 of half A | w2 of half B]
            }
          }
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          MbarArrive(fullW + b);
        }
      }
      return;
    }
    const int st = a.stride;
    const float* srcBase = a.src + static_cast<size_t>(i0) * a.srcImg + static_cast<size_t>(g) * a.Cg * a.chStride;
    for (int ph = 0; ph < st; ph++) {
      // planes of phase row ph: staged float4 p = (phase column pw, position pos) -> pixel (r*stride + ph - pad,
      // c*stride + pw - pad) of image i; zero outside the image (and beyond the batch)
      char* x1 = reinterpret_cast<char*>(planes + ph * 2 * a.planeRows);
      char* x2 = x1 + a.planeRows * 16;
      for (int p = pt; p < st * a.NPOS; p += kWsProducers) {
        const int pw = p / a.NPOS, pos = p - pw * a.NPOS;
        const int F = Q0 + pos;
        const int i = F / a.IB, rem = F - i * a.IB;
        const int r = rem / a.PW, c = rem - r * a.PW;
        const int hi = r * st + ph - a.pad, wi = c * st + pw - a.pad;
        float4 v = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (i < a.N && static_cast<unsigned>(hi) < static_cast<unsigned>(a.Hi) && static_cast<unsigned>(wi) < static_cast<unsigned>(a.Wi)) {
          const float* px = srcBase + static_cast<size_t>(i - i0) * a.srcImg + hi * a.rowStride + wi * a.colStride;
          v.x = __ldg(px);
          if (a.Cg > 1) v.y = __ldg(px + a.chStride);
          if (a.Cg > 2) v.z = __ldg(px + 2 * a.chStride);
          if (a.Cg > 3) v.w = __ldg(px + 3 * a.chStride);
        }
        // row = (pair of phase columns, position), the parity selects the half
        uint2 p1, p2;
        SplitBf16x4(v, p1, p2);
        const int db = ((pw >> 1) * a.NPOS + pos) * 16 + (pw & 1) * 8;
        *reinterpret_cast<uint2*>(x1 + db) = p1;
        *reinterpret_cast<uint2*>(x2 + db) = p2;
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // planes are read by the tensor core
      MbarArrive(fullP + ph);
      // weights of the phase row's stages: a thread owns channel c, its index row is [tapsPad] bytes of d_asmt_t
      const int first = a.chunkFirst[ph], cnt = a.chunkCount[ph];
      for (int s0 = 0; s0 < cnt; s0 += KS, j++) {
        const int n = min(KS, cnt - s0), b = j & 1;
        if (j >= 2) MbarWait<24>(emptyW + b, ((j >> 1) - 1) & 1);   // buffer last read by the MMAs of stage j - 2
        uint4* w = wts + b * KS * 2 * NC;
        for (int c = pt; c < NC; c += kWsProducers) {
          const uint8_t* row = a.asmtT + (static_cast<size_t>(g * st + ph) * a.KgPad + c) * a.tapsPad;
          // (no unroll pragma here: under `#pragma unroll 3` the compiled loop was seen running an iteration with e == n
          // for n = 8 on the device, writing past the weight buffer into the codebook / offset regions)
          for (int e = 0; e < n; e++) {
            const KStep ks = a.tab[first + s0 + e];
            const uint4 q0 = cb[__ldg(row + ks.idx0)];
            const uint4 q1 = ks.cb1 ? make_uint4(0u, 0u, 0u, 0u) : cb[__ldg(row + ks.idx1)];   // unpaired tap: zero half
            w[(2 * e + 0) * NC + c] = make_uint4(q0.x, q0.y, q1.x, q1.y);   // [w1 of half 0 | w1 of half 1]
            w[(2 * e + 1) * NC + c] = make_uint4(q0.z, q0.w, q1.z, q1.w);   // [w2 of half 0 | w2 of half 1]
          }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        MbarArrive(fullW + b);
      }
    }
    return;
  }

  // =========================== consumers: wgmma ===========================
  const int wg = warp >> 2;
  float acc[MB][NC / 2];
#pragma unroll
  for (int m = 0; m < MB; m++)
#pragma unroll
    for (int i = 0; i < NC / 2; i++) acc[m][i] = 0.0f;
  const uint32_t planes0 = SmemU32(planes), wts0 = SmemU32(wts);
  int j = 0;
  for (int kc = 0; kc < nCh; kc++) {
    // mode 0: chunk kc = 8 channels, every tap (table entries [0, ntab)), plane buffer kc % nPB of the ring;
    // mode 1: chunk kc = phase row kc (entries [chunkFirst, + chunkCount)), its own resident plane buffer
    const int pb = S1 ? kc % nPB : kc;
    MbarWait<24>(fullP + pb, S1 ? (kc / nPB) & 1 : 0);
    const uint32_t plA = planes0 + static_cast<uint32_t>(pb * 2 * a.planeRows) * 16u + static_cast<uint32_t>(wg * MB * 64) * 16u;
    const int first = S1 ? 0 : a.chunkFirst[kc], cnt = S1 ? a.ntab : a.chunkCount[kc];
    for (int s0 = 0; s0 < cnt; s0 += KS, j++) {
      const int n = min(KS, cnt - s0), b = j & 1;
      MbarWait<24>(fullW + b, (j >> 1) & 1);
      qcnn::WgmmaFence();
      for (int e = 0; e < n; e++) {
        const KStep ks = a.tab[first + s0 + e];
        const uint32_t wb = wts0 + static_cast<uint32_t>((b * KS + e) * 2 * NC) * 16u;
        const uint64_t d1 = WgmmaDesc(wb, 0, 128), d2 = WgmmaDesc(wb + NC * 16, 0, 128);
#pragma unroll
        for (int m = 0; m < MB; m++) {
          const uint64_t dA = WgmmaDesc(plA + static_cast<uint32_t>(ks.bStart + m * 64) * 16u, static_cast<uint32_t>(a.planeRows) * 16u, 128);
          qcnn::WgmmaSS<NC>::Bf16(acc[m], dA, d1);
          qcnn::WgmmaSS<NC>::Bf16(acc[m], dA, d2);
        }
      }
      qcnn::WgmmaCommit();
      qcnn::WgmmaWaitAll();
      __syncwarp();
      if (lane == 0) MbarArrive(emptyW + b);
    }
    if (S1 && lane == 0) MbarArrive(emptyP + pb);   // (the chunk's MMAs have retired: the last stage waited for them)
  }

  // ---- epilogue: accumulator fragments (rows = positions r0, r0 + 8; columns = channels 8 i + 2 t4, +1) -> NHWC ----
  const int r0 = (warp & 3) * 16 + (lane >> 2), t4 = lane & 3;
  const bool v2 = (reinterpret_cast<uintptr_t>(a.dst) & 7u) == 0;   // (Cout, g * Kg and ch0 are even: pairs are 8-byte aligned)
#pragma unroll
  for (int m = 0; m < MB; m++) {
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int off = outoff[(wg * MB + m) * 64 + r0 + 8 * h];
      if (off < 0) continue;
      float* o = dstBase + off;
#pragma unroll
      for (int i = 0; i < NC / 8; i++) {
        const int ch = 8 * i + 2 * t4;
        float v0 = acc[m][4 * i + 2 * h] + biasS[ch], v1 = acc[m][4 * i + 2 * h + 1] + biasS[ch + 1];
        if (a.relu) { v0 = fmaxf(v0, 0.0f); v1 = fmaxf(v1, 0.0f); }
        if (v2) *reinterpret_cast<float2*>(o + ch) = make_float2(v0, v1);
        else { o[ch] = v0; o[ch + 1] = v1; }
      }
    }
  }
}

// channel counts per CTA with an instantiation (N of the MMA; 192 and 256 with one m64 block per warpgroup only)
constexpr int kWsWidths[] = {16, 32, 64, 96, 128, 192, 256};

// the dynamic shared-memory limit of an instantiation is raised once per device to the opt-in maximum (as in pq_gemm_tc.cu)
template <int NC, int MB, bool S1, bool WIDE>
int SetSmemAndLaunch(const GemmArgs& a, unsigned blocks, size_t smem, cudaStream_t st, qcnn_ctx* ctx) {
  static bool done[64] = {false};
  if (ctx->device < 0 || ctx->device >= 64 || !done[ctx->device]) {
    const int lim = static_cast<int>(qcnn::SmemOptin(ctx));
    QCNN_CUDA(cudaFuncSetAttribute(conv_ws_kernel<NC, MB, S1, WIDE>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
    if (ctx->device >= 0 && ctx->device < 64) done[ctx->device] = true;
  }
  conv_ws_kernel<NC, MB, S1, WIDE><<<blocks, kWsThreads, smem, st>>>(a);
  QCNN_CUDA(cudaGetLastError());
  return 0;
}

template <bool S1, bool WIDE>
int LaunchWidth(const GemmArgs& a, int nc, unsigned nb, size_t smem, cudaStream_t st, qcnn_ctx* ctx) {
#define QCNN_WS(NC)                                                                               \
  if (nc == NC) return a.NT == 256 ? SetSmemAndLaunch<NC, 2, S1, WIDE>(a, nb, smem, st, ctx)      \
                                   : SetSmemAndLaunch<NC, 1, S1, WIDE>(a, nb, smem, st, ctx);
  QCNN_WS(16) QCNN_WS(32) QCNN_WS(64) QCNN_WS(96) QCNN_WS(128)
#undef QCNN_WS
  if (nc == 192 && a.NT == 128) return SetSmemAndLaunch<192, 1, S1, WIDE>(a, nb, smem, st, ctx);
  if (nc == 256 && a.NT == 128) return SetSmemAndLaunch<256, 1, S1, WIDE>(a, nb, smem, st, ctx);
  qcnn::SetError("internal: no conv_ws instantiation for N=%d positions=%d", nc, a.NT);
  return 1;
}

bool WsWidth(int w) { return std::find(std::begin(kWsWidths), std::end(kWsWidths), w) != std::end(kWsWidths); }

}  // namespace

namespace qcnn {

// Stride-1 tilings (mode-0 geometry): positions per CTA x channels per CTA (an instantiated width dividing Cout / grp)
// x k-steps per weight stage, under the conditions of pq_gemm_tc mode 0 (or <= 3 channels per group) plus the pre-split
// codebook and the channel-major index block of at most 32 taps.  The positions of a CTA need not fit one register pass
// of the producers: any plane ring that fits in shared memory is a tiling.
static void PlanConvWsS1(const qcnn_layer* L, int N, ConvCands* cands) {
  const int G = L->grp, Cg = L->Cin / G, Kg = L->Cout / G, taps = L->ksz * L->ksz;
  // (Cg <= 3: one chunk, half A read as scalars; wider groups: whole 4-channel halves read as float4)
  if (L->src_nchw || L->d % 4 != 0 || (Cg > 3 && (Cg % 4 != 0 || L->Cin % 4 != 0)) || L->S * L->d < Cg || taps > kMaxKSteps) return;
  if (L->asmt_t_mode != 0 || RoundUp(taps, 16) > 32) return;
  const int PW = L->Win + L->pad, IB = (L->Hin + L->pad) * PW;
  if (L->Ho > L->Hin + L->pad || L->Wo > PW || static_cast<double>(N) * IB > 2.0e9) return;
  const size_t smemMax = SmemOptin(L->ctx);
  // widths: every instantiated divisor of Kg from 64 up (narrower tiles re-stage the same positions for few channels),
  // or the widest divisor when all are narrower
  int widest = 0;
  for (int w : kWsWidths) if (Kg % w == 0) widest = w;
  for (int W : kWsWidths) {
    if (Kg % W != 0 || (W < 64 && W != widest)) continue;
    for (int MB = 2; MB >= 1; MB--) {
      if (MB == 2 && W > 128) continue;   // (2 x 128 accumulator registers do not fit)
      const int P = 128 * MB;
      ConvPlan p;
      memset(&p, 0, sizeof(p));
      p.kernel = kConvWs; p.threads = kWsThreads;
      GemmArgs& ga = p.g;
      ga.mode = 0; ga.bf = 1;
      ga.PW = PW; ga.IB = IB; ga.NT = P;
      ga.NPOS = RoundUp(P + (L->ksz - 1) * (PW + 1), 8);
      ga.planeRows = ga.NPOS; ga.planeF4 = 2 * ga.NPOS;
      ga.nChunks = CeilDiv(Cg, 8); ga.nct = Kg / W; ga.nsplit = 1;
      ga.stride = 1; ga.Kg = Kg; ga.K = L->K;
      ga.tapsPad = RoundUp(taps, 16);
      Mode0Table(L, ga);
      // k-steps per weight stage: the chunk's taps in as few equal stages as fit; a ring of three plane buffers if it fits
      bool fit = false;
      for (int stages = 1; stages <= taps && !fit; stages++) {
        ga.GT = CeilDiv(taps, stages);
        for (ga.nPB = 3; ga.nPB >= 2; ga.nPB--)
          if (static_cast<size_t>(MapWsSmem(ga).total) <= smemMax) { fit = true; break; }
      }
      if (!fit) continue;
      p.smem = static_cast<size_t>(MapWsSmem(ga).total);
      p.key = {P, ga.GT, ga.nct};
      const int stages = ga.nChunks * CeilDiv(taps, ga.GT);
      const double ne = static_cast<double>(ga.nChunks) * taps;
      // tensor work on PlanPqGemm's scale (as PlanConvWs below), a pipeline drain per weight stage, the set-up
      const double perCta = ne * 2.0 * (P / 64) * (W / 128.0) * (3.0 * 64.0 * 1.15 / 4.0) + 600.0 * stages + 4000.0 + P * 24.0;
      const double ctas = static_cast<double>(CeilDiv(N * IB, P)) * G * ga.nct;
      cands->emplace_back(perCta * std::ceil(ctas / L->ctx->sm_count), p);
    }
  }
}

// Candidate tilings for batch N (cost in SM-cycles, the scale of PlanPqGemm's model): positions per CTA x k-steps per
// weight stage (x channel tiles, stride 1).  Eligible: bf16x2 operands, an instantiated channel width, the pre-split
// codebook and the channel-major index block; stride 1 under the conditions of pq_gemm_tc mode 0, strided layers under
// those of its mode 1.
void PlanConvWs(const qcnn_layer* L, int N, ConvCands* cands) {
  const int G = L->grp, Cg = L->Cin / G, Kg = L->Cout / G, st = L->stride;
  if (!L->opt_tc_bf || L->K < 1 || L->K > 256) return;
  if (st == 1) { PlanConvWsS1(L, N, cands); return; }
  if (st < 2 || st > 4 || (st & 1)) return;
  if (Cg > 4 || L->S != 1 || L->d < Cg || L->d % 4 != 0 || L->asmt_t_mode != 1) return;
  if (!WsWidth(Kg)) return;
  const int PWp = CeilDiv(L->Win + 2 * L->pad, st), PHp = CeilDiv(L->Hin + 2 * L->pad, st);
  if (L->Wo > PWp) return;
  const int IB = PHp * PWp;
  if (static_cast<double>(N) * IB > 2.0e9 || static_cast<double>(L->Hin) * L->Win * L->Cin * 4 > 2.0e9) return;
  const size_t smemMax = SmemOptin(L->ctx);
  for (int MB = 2; MB >= 1; MB--) {
    if (MB == 2 && Kg > 128) continue;   // (2 x 128 accumulator registers do not fit)
    const int P = 128 * MB;
    ConvPlan p;
    memset(&p, 0, sizeof(p));
    p.kernel = kConvWs; p.threads = kWsThreads;
    GemmArgs& ga = p.g;
    ga.mode = 1; ga.bf = 1;
    ga.PW = PWp; ga.IB = IB; ga.NT = P;
    ga.NPOS = RoundUp(P + ((L->ksz - 1) / st) * (PWp + 1), 8);
    ga.planeRows = (st / 2) * ga.NPOS;
    ga.planeF4 = st * ga.NPOS;
    ga.nChunks = st; ga.nct = 1; ga.nsplit = 1; ga.nPB = st;   // every phase row resident
    ga.stride = st; ga.Kg = Kg; ga.K = L->K;
    ga.tapsPad = RoundUp(CeilDiv(L->ksz, st) * L->ksz, 16);
    const int ne = Mode1Table(L, ga);
    if (ne > kMaxKSteps) continue;
    int maxCnt = 0;
    for (int ph = 0; ph < st; ph++) maxCnt = std::max(maxCnt, ga.chunkCount[ph]);
    // k-steps per weight stage: a whole phase row when it fits, else the largest count that does
    for (ga.GT = maxCnt; ga.GT >= 1 && static_cast<size_t>(MapWsSmem(ga).total) > smemMax; ga.GT--) {}
    if (ga.GT < 1) continue;
    p.smem = static_cast<size_t>(MapWsSmem(ga).total);
    p.key = {P, ga.GT, ga.nct};
    int stages = 0;
    for (int ph = 0; ph < st; ph++) stages += CeilDiv(ga.chunkCount[ph], ga.GT);
    // tensor work on PlanPqGemm's scale (its 4 MMAs of m64 n128 k16 per k-step cost 3 * 64 * 1.15), a pipeline drain per
    // weight stage, the set-up and the staging of the first phase row
    const double perCta = ne * 2.0 * (P / 64) * (Kg / 128.0) * (3.0 * 64.0 * 1.15 / 4.0) + 600.0 * stages + 9000.0 + P * 24.0;
    const double ctas = static_cast<double>(CeilDiv(N * IB, P)) * G;
    cands->emplace_back(perCta * std::ceil(ctas / L->ctx->sm_count), p);
  }
}

int LaunchConvWs(qcnn_layer* L, const ConvPlan& p, const float* src, int N, float* dst, int relu, cudaStream_t st) {
  GemmArgs a = p.g;
  a.src = src; a.dst = dst; a.ctrd = L->d_ctrd_bf.as<float>(); a.bias = L->d_bias.as<float>();
  a.asmtT = L->d_asmt_t.as<uint8_t>();
  a.N = N; a.relu = relu;
  SetGemmGeometry(L, a);
  QCNN_CHECK(a.mode == 1 || !L->src_nchw, "qcnn_conv_aprx_forward: the stride-1 weight-stationary tiling reads NHWC sources only");
  const long long blocks = static_cast<long long>(CeilDiv(N * a.IB, a.NT)) * a.G * a.nct;
  QCNN_CHECK(blocks <= 2147483647LL, "qcnn_conv_aprx_forward: batch too large for the weight-stationary tiling");
  QCNN_CHECK(static_cast<size_t>(MapWsSmem(a).total) == p.smem, "internal: conv_ws shared-memory carve changed after planning");
  const unsigned nb = static_cast<unsigned>(blocks);
  const int nc = a.Kg / a.nct;
  if (a.mode == 1) return LaunchWidth<false, false>(a, nc, nb, p.smem, st, L->ctx);
  const bool wide = 2 * a.NPOS > kWsRegPos * kWsProducers || a.Cg < 4;
  return wide ? LaunchWidth<true, true>(a, nc, nb, p.smem, st, L->ctx) : LaunchWidth<true, false>(a, nc, nb, p.smem, st, L->ctx);
}

void DescribeConvWs(const qcnn_layer* L, const ConvPlan& p, int N, char* buf, size_t cap) {
  if (p.g.mode == 0) {
    // stride 1: N = channels per CTA, ctiles = channel tiles per group, ksteps = chunks x taps (a CTA's k-steps), so
    // that grid x ksteps x 32 x positions x N is the executed MAC count
    const int stages = p.g.nChunks * CeilDiv(p.g.ntab, p.g.GT);
    snprintf(buf, cap, " mode=0 N=%d positions=%d ctiles=%d KS=%d smem=%zuB grid=%d NPOS=%d planebufs=%d chunks=%d stages=%d "
             "ksteps=%d", p.g.Kg / p.g.nct, p.g.NT, p.g.nct, p.g.GT, p.smem, CeilDiv(N * p.g.IB, p.g.NT) * L->grp * p.g.nct,
             p.g.NPOS, p.g.nPB, p.g.nChunks, stages, p.g.nChunks * p.g.ntab);
    return;
  }
  // (no "NT=": the executed-MAC count that bench.py derives from pq_gemm_tc( plans assumes 128-channel tiles)
  int stages = 0;
  for (int c = 0; c < p.g.nChunks; c++) stages += CeilDiv(p.g.chunkCount[c], p.g.GT);
  snprintf(buf, cap, " N=%d positions=%d KS=%d smem=%zuB grid=%d NPOS=%d chunks=%d stages=%d ksteps=%d", p.g.Kg, p.g.NT,
           p.g.GT, p.smem, CeilDiv(N * p.g.IB, p.g.NT) * L->grp, p.g.NPOS, p.g.nChunks, stages, p.g.ntab);
}

}  // namespace qcnn
