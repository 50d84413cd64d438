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
//     width up to 256: no channel padding).  They are decoded once per layer, at its creation, into the weight image
//     qcnn_layer::d_w_ws (conv_ws_image_kernel below), and a CTA streams them into a ring of nWB stage buffers by bulk
//     copy.  Per k-step, [w1 | w1] and [w2 | w2] are 16-byte rows per channel; the duplicated half is the same core
//     matrix read twice (LBO = 0).  Two MMAs per k-step into one accumulator:
//     [x1|x2].[w1|w1] + [x1|x2].[w2|w2] = (x1 + x2)(w1 + w2), the same k-steps in the same order as pq_gemm_tc's one-
//     accumulator tiling of the same geometry (the error bound depends on that chain, DESIGN.md 2).
//
// Roles inside a CTA of twelve warps:
//   warps 0-7   two consumer warpgroups; each owns MB m64 blocks of the CTA's 128 MB positions and issues
//               wgmma.mma_async (both operands in shared memory) into MB accumulators of N / 2 registers per thread.
//   warps 8-11  producers: stage the position planes (global -> bf16x2 split -> planes; mode 1: every phase row resident,
//               mode 0: a ring of plane buffers, one chunk each, with a full / empty mbarrier pair per buffer).  One
//               producer thread also fills the weight ring: a stage (<= KS k-steps of one chunk, all N channels) is one
//               bulk copy from the image (nct > 1: one per k-step and piece), counted on the buffer's full mbarrier.
//   epilogue    the consumers add the bias (+ ReLU) and store pairs of consecutive channels of one NHWC pixel.
#include "qcnn_internal.h"
#include "wgmma.h"
#include "ws_common.cuh"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>

namespace {

using qcnn::kWsConsumers;
using qcnn::kWsProducers;
using qcnn::kWsThreads;
using qcnn::MbarArrive;
using qcnn::MbarWait;
using qcnn::SmemU32;
using qcnn::SplitBf16x4;

constexpr int kWsRegPos = 8;        // mode 0: float4 of a chunk's planes a producer thread stages per register pass
constexpr int kWsRegItems1 = 12;    // mode 1: float4 of a phase row's planes a producer thread holds (st * NPOS <= 1536)
constexpr int kNoRow = -(1 << 30);  // mode 1: input row of an item that stages zeros in every phase row

// Shared-memory carve, read by the planner (fits / does not fit) and by the kernel.  The channel count is computed as
// Kg / nct rather than read from NC: reading NC changed the kernels' register allocation.
struct WsSmem {  // byte offsets inside the dynamic shared memory
  int planes, wts, outoff, bias, bars, total;
};
__host__ __device__ inline WsSmem MapWsSmem(const ConvWsArgs& a) {
  const int nc = a.Kg / a.nct;
  WsSmem m;
  int o = 0;
  m.planes = o; o += a.nPB * 2 * a.planeRows * 16;        // [buffer][x1, x2][planeRows] 16-byte rows
  m.wts = o;    o += a.nWB * a.KS * 2 * nc * 16;          // [buffer][k-step][w1, w2][channel] 16-byte rows (bulk-copy targets)
  m.outoff = o; o += a.P * 4;                             // destination element offset of every position (-1: none)
  m.bias = o;   o += nc * 4;                              // (nc is a multiple of 16: the barriers stay 8-byte aligned)
  m.bars = o;   o += 8 * (2 * a.nPB + 2 * a.nWB);
  m.total = o;
  return m;
}

// NC: channels per CTA; MB: m64 blocks per consumer warpgroup; S1: the stride-1 geometry (mode 0), else mode 1;
// WIDE (stride 1): a chunk's planes take more than one register pass of the producers, or a group has <= 3 channels
// (kept apart so that the single-pass kernels AlexNet runs carry none of that staging)
template <int NC, int MB, bool S1, bool WIDE>
__global__ void __launch_bounds__(kWsThreads, 1) conv_ws_kernel(const ConvWsArgs a) {
  constexpr int P = 128 * MB;   // positions per CTA
  extern __shared__ __align__(128) unsigned char smem[];
  const WsSmem sm = MapWsSmem(a);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int KS = a.KS, nPB = a.nPB, nWB = a.nWB;
  const int nCh = S1 ? a.nChunks : a.stride;   // chunks: 8-channel groups (mode 0) / phase rows (mode 1)
  uint4* planes = reinterpret_cast<uint4*>(smem + sm.planes);
  uint4* wts = reinterpret_cast<uint4*>(smem + sm.wts);
  int* outoff = reinterpret_cast<int*>(smem + sm.outoff);
  float* biasS = reinterpret_cast<float*>(smem + sm.bias);
  uint64_t* fullP = reinterpret_cast<uint64_t*>(smem + sm.bars);   // [nPB] planes of a chunk staged: producers -> consumers
  uint64_t* emptyP = fullP + nPB;                                   // [nPB] (mode 0) planes' MMAs retired: consumers -> producers
  uint64_t* fullW = emptyP + nPB;                                   // [nWB] weight stage copied: bulk copy -> consumers
  uint64_t* emptyW = fullW + nWB;                                   // [nWB] weight stage's MMAs retired: consumers -> producer
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
  for (int c = tid; c < NC; c += kWsThreads) biasS[c] = __ldg(a.bias + g * a.Kg + ch0 + c);
  if (tid == 0) {
    for (int i = 0; i < nPB; i++) { qcnn::MbarInit(fullP + i, kWsProducers); qcnn::MbarInit(emptyP + i, kWsConsumers / 32); }
    for (int i = 0; i < nWB; i++) { qcnn::MbarInit(fullW + i, 1); qcnn::MbarInit(emptyW + i, kWsConsumers / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int warpU = __shfl_sync(0xffffffffu, warp, 0);   // provably warp-uniform role selector
  if (warpU >= kWsConsumers / 32) {
    // =========================== producers ===========================
    const int pt = tid - kWsConsumers;
    // the weight ring, filled by producer thread 0: stage jI = k-steps [s0I, + KS) of chunk kcI into buffer jI % nWB, once
    // the MMAs of stage jI - nWB have retired.  The image holds [grp][entry][w1, w2][Kg] 16-byte rows, an entry being a
    // k-step of the layer (mode 0: chunk x tap, mode 1: the k-step table's order); a stage's entries are consecutive.
    // The stages are exactly those the consumers wait for: ceil(count / KS) per chunk, none for a phase row without
    // k-steps (ksz < stride: the trailing rows; the chunk advance steps over them).
    const int nE = S1 ? nCh * a.kt.ntab : a.kt.ntab;
    int jI = 0, kcI = 0, s0I = 0;
    auto issueStage = [&]() {
      const int cnt = S1 ? a.kt.ntab : a.kt.chunkCount[kcI];
      const int n = min(KS, cnt - s0I), b = jI % nWB;
      if (jI >= nWB) MbarWait<24>(emptyW + b, ((jI / nWB) - 1) & 1);
      const uint32_t bytes = static_cast<uint32_t>(n * 2 * NC * 16);
      qcnn::MbarExpectTx(fullW + b, bytes);
      uint4* w = wts + b * KS * 2 * NC;
      const int e0 = (S1 ? kcI * a.kt.ntab : a.kt.chunkFirst[kcI]) + s0I;
      const uint4* src = a.wimg + (static_cast<size_t>(g) * nE + e0) * 2 * a.Kg + ch0;
      if (a.nct == 1) {
        qcnn::BulkLoad(w, src, bytes, fullW + b);   // (NC = Kg: the stage's rows are contiguous in the image)
      } else {
        for (int r = 0; r < 2 * n; r++) qcnn::BulkLoad(w + r * NC, src + static_cast<size_t>(r) * a.Kg, NC * 16, fullW + b);
      }
      jI++;
      s0I += KS;
      if (s0I >= cnt) {
        s0I = 0;
        kcI++;
        if constexpr (!S1)
          while (kcI < nCh && a.kt.chunkCount[kcI] == 0) kcI++;
      }
    };
    if (pt == 0)   // the first stages are in flight before any position is loaded
      while (jI < nWB && kcI < nCh) issueStage();
    if constexpr (S1) {
      // float4 p = pt + (q * kWsRegPos + i) * kWsProducers of pass q of a chunk's planes: half = p / NPOS (channels 0-3 /
      // 4-7 of the chunk), position = p % NPOS -> pixel (r - pad, c - pad) of image i of the flat padded grid.  The 2 NPOS
      // float4 of a chunk take nPass register passes; the source offsets and validity of a pass are chunk-invariant
      // (computed once with a single pass, per pass otherwise)
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
        if (kc + 1 < nCh) {   // in flight during the weight copies below
          if (nPass > 1) passPos(0);
          loadPos(kc + 1);
        }
        if (pt == 0)
          while (kcI <= kc) issueStage();   // the chunk's stages not issued yet
      }
      return;
    }
    // A phase row's planes are st * NPOS float4 items p = (position pos, phase column pw), pw fastest, so that a warp reads
    // consecutive pixels of an input row; thread pt holds items pt + i * kWsProducers (i < kWsRegItems1) in registers.  Per
    // item, computed once per tile: the source offset of phase row 0 and its input row hr (phase row ph reads input row
    // hr + ph, one row pitch further per phase; kNoRow: the item is outside the image or the batch, or past the planes).
    const int st = a.stride, sh = st >> 1, nItems = st * a.NPOS;   // (stride 2 or 4: pos = p >> sh, pw = p & (st - 1))
    const float* srcBase = a.src + static_cast<size_t>(i0) * a.srcImg + static_cast<size_t>(g) * a.Cg * a.chStride;
    int poff[kWsRegItems1], hr[kWsRegItems1];
#pragma unroll
    for (int i = 0; i < kWsRegItems1; i++) {
      const int p = pt + i * kWsProducers, pos = p >> sh, pw = p & (st - 1);
      const int F = Q0 + pos;
      const int im = F / a.IB, rem = F - im * a.IB;
      const int r = rem / a.PW, c = rem - r * a.PW;
      const int wi = c * st + pw - a.pad;
      poff[i] = 0; hr[i] = kNoRow;
      if (p < nItems && im < a.N && static_cast<unsigned>(wi) < static_cast<unsigned>(a.Wi)) {
        hr[i] = r * st - a.pad;
        poff[i] = (im - i0) * static_cast<int>(a.srcImg) + hr[i] * a.rowStride + wi * a.colStride;
      }
    }
    float4 rg[kWsRegItems1];
    auto loadRow = [&](int ph) {   // every load of the phase row is issued before any is used
      const float* s = srcBase + ph * a.rowStride;
#pragma unroll
      for (int i = 0; i < kWsRegItems1; i++) {
        rg[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (static_cast<unsigned>(hr[i] + ph) < static_cast<unsigned>(a.Hi)) {
          const float* px = s + poff[i];
          rg[i].x = __ldg(px);
          if (a.Cg > 1) rg[i].y = __ldg(px + a.chStride);
          if (a.Cg > 2) rg[i].z = __ldg(px + 2 * a.chStride);
          if (a.Cg > 3) rg[i].w = __ldg(px + 3 * a.chStride);
        }
      }
    };
    loadRow(0);
    for (int ph = 0; ph < st; ph++) {
      // planes of phase row ph: item p -> pixel (r*stride + ph - pad, c*stride + pw - pad) of its image (zero outside);
      // plane row = (pair of phase columns, position), the parity of pw selects the half
      char* x1 = reinterpret_cast<char*>(planes + ph * 2 * a.planeRows);
      char* x2 = x1 + a.planeRows * 16;
#pragma unroll
      for (int i = 0; i < kWsRegItems1; i++) {
        const int p = pt + i * kWsProducers, pos = p >> sh, pw = p & (st - 1);
        if (p < nItems) {
          uint2 p1, p2;
          SplitBf16x4(rg[i], p1, p2);
          const int db = ((pw >> 1) * a.NPOS + pos) * 16 + (pw & 1) * 8;
          *reinterpret_cast<uint2*>(x1 + db) = p1;
          *reinterpret_cast<uint2*>(x2 + db) = p2;
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // planes are read by the tensor core
      MbarArrive(fullP + ph);
      if (ph + 1 < st) loadRow(ph + 1);   // in flight during the weight copies below
      if (pt == 0)
        while (kcI <= ph) issueStage();   // the phase row's stages not issued yet
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
    const int first = S1 ? 0 : a.kt.chunkFirst[kc], cnt = S1 ? a.kt.ntab : a.kt.chunkCount[kc];
    for (int s0 = 0; s0 < cnt; s0 += KS, j++) {
      const int n = min(KS, cnt - s0), b = j % nWB;
      MbarWait<24>(fullW + b, (j / nWB) & 1);
      qcnn::WgmmaFence();
      for (int e = 0; e < n; e++) {
        const KStep ks = a.kt.tab[first + s0 + e];
        const uint32_t wb = wts0 + static_cast<uint32_t>((b * KS + e) * 2 * NC) * 16u;
        qcnn::WsMmaKStep<NC, MB>(acc, plA, ks.bStart, static_cast<uint32_t>(a.planeRows) * 16u, wb);
      }
      qcnn::WsRetireStage(emptyW + b, lane);
    }
    if (S1 && lane == 0) MbarArrive(emptyP + pb);   // (the chunk's MMAs have retired: the last stage waited for them)
  }

  // ---- epilogue: accumulator fragments (rows = positions r0, r0 + 8; columns = channels 8 i + 2 t4, +1) -> NHWC ----
  const qcnn::WsFrag fr = qcnn::WsFragOf(warp, lane);
  const int r0 = fr.r0, t4 = fr.t4;
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

template <int NC, int MB, bool S1, bool WIDE>
int LaunchInstance(const ConvWsArgs& a, unsigned blocks, size_t smem, cudaStream_t st, qcnn_ctx* ctx) {
  if (int rc = qcnn::OptInSmem<conv_ws_kernel<NC, MB, S1, WIDE>>(ctx)) return rc;
  conv_ws_kernel<NC, MB, S1, WIDE><<<blocks, kWsThreads, smem, st>>>(a);
  QCNN_CUDA(cudaGetLastError());
  return 0;
}

template <bool S1, bool WIDE>
int LaunchWidth(const ConvWsArgs& a, unsigned nb, size_t smem, cudaStream_t st, qcnn_ctx* ctx) {
#define QCNN_WS(W)                                                                          \
  if (a.NC == W) return a.P == 256 ? LaunchInstance<W, 2, S1, WIDE>(a, nb, smem, st, ctx)   \
                                   : LaunchInstance<W, 1, S1, WIDE>(a, nb, smem, st, ctx);
  QCNN_WS(16) QCNN_WS(32) QCNN_WS(64) QCNN_WS(96) QCNN_WS(128)
#undef QCNN_WS
  if (a.NC == 192 && a.P == 128) return LaunchInstance<192, 1, S1, WIDE>(a, nb, smem, st, ctx);
  if (a.NC == 256 && a.P == 128) return LaunchInstance<256, 1, S1, WIDE>(a, nb, smem, st, ctx);
  qcnn::SetError("internal: no conv_ws instantiation for N=%d positions=%d", a.NC, a.P);
  return 1;
}

bool WsWidth(int w) { return std::find(std::begin(kWsWidths), std::end(kWsWidths), w) != std::end(kWsWidths); }

// The weight image of a layer (qcnn_layer::d_w_ws), [grp][entry][w1, w2][Kg] 16-byte rows: one thread per (group, entry,
// channel) writes the entry's rows [w1 of half 0 | w1 of half 1] and [w2 of half 0 | w2 of half 1] of the channel from
// the pre-split codebook (d_ctrd_bf) and the channel-major index block (d_asmt_t).  These are the rows that conv_ws
// stages for the k-step, so its MMAs read the same bits as pq_gemm_tc's decoders produce.
struct WsImageArgs {
  const uint4* ctrd;
  const uint8_t* asmtT;
  uint4* img;
  int G, Kg, KgPad, S, K, d, Cg, stride, tapsPad, nE;   // nE: entries per group
  KStepTable kt;                                        // Mode0Table / Mode1Table (only the index fields are read)
};

__global__ void conv_ws_image_kernel(const WsImageArgs a) {
  const long long total = static_cast<long long>(a.G) * a.nE * a.Kg;
  const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % a.Kg);
    const long long r = i / a.Kg;
    const int e = static_cast<int>(r % a.nE), g = static_cast<int>(r / a.nE);
    uint4 q0, q1;
    if (a.stride == 1) {
      // entry = (chunk kc of 8 input channels, tap t); the chunk's two 4-channel halves: subspace and piece of each (as
      // pq_gemm_tc's fetchChunk); a half beyond the group's channels is zero (its positions are zeros too)
      const int taps = a.kt.ntab, kc = e / taps, t = e - kc * taps;
      const int chA = kc * 8, chB = chA + 4;
      const int sA = chA / a.d, jA = chA - sA * a.d;
      const int iA = a.asmtT[(static_cast<size_t>(g * a.S + sA) * a.KgPad + c) * a.tapsPad + t];
      q0 = a.ctrd[static_cast<size_t>(sA * (a.d >> 2) + (jA >> 2)) * a.K + iA];
      q1 = zero;
      if (chB < a.Cg) {
        const int sB = chB / a.d, jB = chB - sB * a.d;
        const int iB = a.asmtT[(static_cast<size_t>(g * a.S + sB) * a.KgPad + c) * a.tapsPad + t];
        q1 = a.ctrd[static_cast<size_t>(sB * (a.d >> 2) + (jB >> 2)) * a.K + iB];
      }
    } else {
      // entry = k-step e of the table, in phase row ph: its taps' indices are bytes idx0 / idx1 of the channel's row of
      // the phase row; an unpaired tap's second half is zero
      int ph = 0;
      while (ph + 1 < a.stride && e >= a.kt.chunkFirst[ph + 1]) ph++;
      const KStep ks = a.kt.tab[e];
      const uint8_t* row = a.asmtT + (static_cast<size_t>(g * a.stride + ph) * a.KgPad + c) * a.tapsPad;
      q0 = a.ctrd[row[ks.idx0]];
      q1 = ks.cb1 ? zero : a.ctrd[row[ks.idx1]];
    }
    uint4* o = a.img + static_cast<size_t>(g * a.nE + e) * 2 * a.Kg + c;
    o[0] = make_uint4(q0.x, q0.y, q1.x, q1.y);      // [w1 of half 0 | w1 of half 1]
    o[a.Kg] = make_uint4(q0.z, q0.w, q1.z, q1.w);   // [w2 of half 0 | w2 of half 1]
  }
}

// mode 1: staged positions per phase plane for P positions per CTA (P + the taps' reach in phase rows and columns)
int StridedNpos(const qcnn_layer* L, int P) {
  const int st = L->stride, PWp = qcnn::CeilDiv(L->Win + 2 * L->pad, st);
  return qcnn::RoundUp(P + ((L->ksz - 1) / st) * (PWp + 1), 8);
}

// A strided layer's tile of P positions: a phase row's planes in one register pass of the producers, and source offsets
// relative to the CTA's first image in int
bool StridedTileFits(const qcnn_layer* L, int P) {
  const int st = L->stride, NPOS = StridedNpos(L, P);
  const int IB = qcnn::CeilDiv(L->Hin + 2 * L->pad, st) * qcnn::CeilDiv(L->Win + 2 * L->pad, st);
  return st * NPOS <= kWsRegItems1 * kWsProducers &&
         static_cast<double>(qcnn::CeilDiv(NPOS, IB) + 1) * L->Hin * L->Win * L->Cin <= 2.0e9;
}

// The conditions of conv_ws that depend on the layer alone (not on the batch, the operand format or the source layout):
// the layers that get a weight image.  Stride 1: those of pq_gemm_tc mode 0 (or <= 3 channels per group) with at most
// 32 taps per channel-major index row.  Strided: those of its mode 1 over <= 4 input channels, an instantiated width,
// and a tile height whose phase row fits one register pass.
bool WsLayerTakes(const qcnn_layer* L) {
  const int G = L->grp, Cg = L->Cin / G, Kg = L->Cout / G, st = L->stride, taps = L->ksz * L->ksz;
  if (L->kind != QCNN_KIND_CONV || L->K < 1 || L->K > 256) return false;
  if (st == 1) {
    return L->d % 4 == 0 && (Cg <= 3 || (Cg % 4 == 0 && L->Cin % 4 == 0)) && L->S * L->d >= Cg && taps <= kMaxKSteps &&
           L->asmt_t_mode == 0 && qcnn::RoundUp(taps, 16) <= 32 && L->Ho <= L->Hin + L->pad && L->Wo <= L->Win + L->pad;
  }
  if (st > 4 || (st & 1)) return false;
  if (Cg > 4 || L->S != 1 || L->d < Cg || L->d % 4 != 0 || L->asmt_t_mode != 1 || !WsWidth(Kg)) return false;
  if (L->Wo > qcnn::CeilDiv(L->Win + 2 * L->pad, st) || static_cast<double>(L->Hin) * L->Win * L->Cin * 4 > 2.0e9) return false;
  KStepTable t;
  if (qcnn::Mode1Table(L, 0, true, 0, t) > kMaxKSteps) return false;
  return StridedTileFits(L, 128) || (Kg <= 128 && StridedTileFits(L, 256));
}

}  // namespace

namespace qcnn {

int BuildConvWsImage(qcnn_layer* L) {
  if (!WsLayerTakes(L) || L->d_w_ws.get()) return 0;
  WsImageArgs a;
  memset(&a, 0, sizeof(a));
  a.G = L->grp; a.Kg = L->Cout / L->grp; a.KgPad = RoundUp(a.Kg, 16); a.S = L->S; a.K = L->K; a.d = L->d;
  a.Cg = L->Cin / L->grp; a.stride = L->stride;
  if (a.stride == 1) {
    Mode0Table(L, 0, 0, a.kt);
    a.nE = CeilDiv(a.Cg, 8) * a.kt.ntab;
    a.tapsPad = RoundUp(a.kt.ntab, 16);
  } else {
    a.nE = Mode1Table(L, 0, true, 0, a.kt);
    a.tapsPad = RoundUp(CeilDiv(L->ksz, a.stride) * L->ksz, 16);
  }
  const size_t rows = static_cast<size_t>(a.G) * a.nE * 2 * a.Kg;
  QCNN_CUDA(L->d_w_ws.Reserve(L->ctx, rows * sizeof(uint4)));
  a.ctrd = L->d_ctrd_bf.as<uint4>(); a.asmtT = L->d_asmt_t.as<uint8_t>(); a.img = L->d_w_ws.as<uint4>();
  conv_ws_image_kernel<<<static_cast<unsigned>(std::min<size_t>((rows / 2 + 255) / 256, 4096)), 256>>>(a);
  QCNN_CUDA(cudaGetLastError());
  QCNN_CUDA(cudaDeviceSynchronize());
  return 0;
}

// Stride-1 tilings (mode-0 geometry): positions per CTA x channels per CTA (an instantiated width dividing Cout / grp)
// x k-steps per weight stage x weight buffers.  The positions of a CTA need not fit one register pass of the producers:
// any plane ring that fits in shared memory is a tiling.
static void PlanConvWsS1(const qcnn_layer* L, int N, ConvCands* cands) {
  const int G = L->grp, Cg = L->Cin / G, Kg = L->Cout / G, taps = L->ksz * L->ksz;
  if (L->src_nchw) return;
  const int PW = L->Win + L->pad, IB = (L->Hin + L->pad) * PW;
  if (static_cast<double>(N) * IB > 2.0e9) return;
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
      ConvWsArgs& a = p.ws;
      SetGemmGeometry(L, a);
      a.PW = PW; a.IB = IB; a.P = P; a.NC = W; a.nct = Kg / W;
      a.NPOS = RoundUp(P + (L->ksz - 1) * (PW + 1), 8);
      a.planeRows = a.NPOS;
      a.nChunks = CeilDiv(Cg, 8);
      Mode0Table(L, PW, a.NPOS, a.kt);
      // per depth of the weight ring (4, 3, 2 buffers): k-steps per stage = the chunk's taps in as few equal stages as
      // fit (gemm_gt: that many), a ring of three plane buffers if it fits
      for (a.nWB = 4; a.nWB >= 2; a.nWB--) {
        bool fit = false;
        for (int stages = 1; stages <= taps && !fit; stages++) {
          a.KS = L->opt_gemm_gt ? L->opt_gemm_gt : CeilDiv(taps, stages);
          if (a.KS > taps) break;
          for (a.nPB = 3; a.nPB >= 2; a.nPB--)
            if (static_cast<size_t>(MapWsSmem(a).total) <= smemMax) { fit = true; break; }
          if (L->opt_gemm_gt) break;
        }
        if (!fit) continue;
        p.smem = static_cast<size_t>(MapWsSmem(a).total);
        p.key = {P, a.KS, a.nct, a.nWB};
        const double ne = static_cast<double>(a.nChunks) * taps;
        // tensor work on PlanPqGemm's scale (as PlanConvWs below) and the set-up
        const double perCta = ne * 2.0 * (P / 64) * (W / 128.0) * (3.0 * 64.0 * 1.15 / 4.0) + 4000.0 + P * 24.0;
        const double ctas = static_cast<double>(CeilDiv(N * IB, P)) * G * a.nct;
        cands->emplace_back(perCta * std::ceil(ctas / L->ctx->sm_count), p);
      }
    }
  }
}

// Candidate tilings for batch N (cost in SM-cycles, the scale of PlanPqGemm's model): positions per CTA x k-steps per
// weight stage x weight buffers (x channel tiles, stride 1), for the layers with a weight image (WsLayerTakes) at bf16x2
// operands.
void PlanConvWs(const qcnn_layer* L, int N, ConvCands* cands) {
  const int G = L->grp, Kg = L->Cout / G, st = L->stride;
  if (!L->opt_tc_bf || !L->d_w_ws.get()) return;
  if (st == 1) { PlanConvWsS1(L, N, cands); return; }
  const int PWp = CeilDiv(L->Win + 2 * L->pad, st), PHp = CeilDiv(L->Hin + 2 * L->pad, st);
  const int IB = PHp * PWp;
  if (static_cast<double>(N) * IB > 2.0e9) return;
  const size_t smemMax = SmemOptin(L->ctx);
  for (int MB = 2; MB >= 1; MB--) {
    if (MB == 2 && Kg > 128) continue;   // (2 x 128 accumulator registers do not fit)
    const int P = 128 * MB;
    if (!StridedTileFits(L, P)) continue;
    ConvPlan p;
    memset(&p, 0, sizeof(p));
    p.kernel = kConvWs; p.threads = kWsThreads;
    ConvWsArgs& a = p.ws;
    SetGemmGeometry(L, a);
    a.PW = PWp; a.IB = IB; a.P = P; a.NC = Kg; a.nct = 1;
    a.NPOS = StridedNpos(L, P);
    a.planeRows = (st / 2) * a.NPOS;
    a.nChunks = st; a.nPB = st;   // every phase row resident
    const int ne = Mode1Table(L, a.NPOS, true, a.planeRows, a.kt);
    int maxCnt = 0;
    for (int ph = 0; ph < st; ph++) maxCnt = std::max(maxCnt, a.kt.chunkCount[ph]);
    // per depth of the weight ring: k-steps per stage = a whole phase row when it fits, else the largest count that does
    // (gemm_gt: that many)
    for (a.nWB = 4; a.nWB >= 2; a.nWB--) {
      if (L->opt_gemm_gt) {
        a.KS = L->opt_gemm_gt;
        if (a.KS > maxCnt || static_cast<size_t>(MapWsSmem(a).total) > smemMax) continue;
      } else {
        for (a.KS = maxCnt; a.KS >= 1 && static_cast<size_t>(MapWsSmem(a).total) > smemMax; a.KS--) {}
        if (a.KS < 1) continue;
      }
      p.smem = static_cast<size_t>(MapWsSmem(a).total);
      p.key = {P, a.KS, a.nct, a.nWB};
      // tensor work on PlanPqGemm's scale (its 4 MMAs of m64 n128 k16 per k-step cost 3 * 64 * 1.15), the set-up and the
      // staging of the first phase row
      const double perCta = ne * 2.0 * (P / 64) * (Kg / 128.0) * (3.0 * 64.0 * 1.15 / 4.0) + 9000.0 + P * 24.0;
      const double ctas = static_cast<double>(CeilDiv(N * IB, P)) * G;
      cands->emplace_back(perCta * std::ceil(ctas / L->ctx->sm_count), p);
    }
  }
}

int LaunchConvWs(qcnn_layer* L, const ConvPlan& p, const float* src, int N, float* dst, int relu, cudaStream_t st) {
  ConvWsArgs a = p.ws;
  a.src = src; a.dst = dst; a.wimg = L->d_w_ws.as<uint4>(); a.bias = L->d_bias.as<float>();
  a.N = N; a.relu = relu;
  SetGemmGeometry(L, a);
  QCNN_CHECK(a.wimg, "internal: conv_ws planned for a layer without a weight image");
  QCNN_CHECK(a.stride > 1 || !L->src_nchw, "qcnn_conv_aprx_forward: the stride-1 weight-stationary tiling reads NHWC sources only");
  const long long blocks = static_cast<long long>(CeilDiv(N * a.IB, a.P)) * a.G * a.nct;
  QCNN_CHECK(blocks <= 2147483647LL, "qcnn_conv_aprx_forward: batch too large for the weight-stationary tiling");
  QCNN_CHECK(static_cast<size_t>(MapWsSmem(a).total) == p.smem, "internal: conv_ws shared-memory carve changed after planning");
  const unsigned nb = static_cast<unsigned>(blocks);
  if (a.stride > 1) return LaunchWidth<false, false>(a, nb, p.smem, st, L->ctx);
  const bool wide = 2 * a.NPOS > kWsRegPos * kWsProducers || a.Cg < 4;
  return wide ? LaunchWidth<true, true>(a, nb, p.smem, st, L->ctx) : LaunchWidth<true, false>(a, nb, p.smem, st, L->ctx);
}

void DescribeConvWs(const qcnn_layer* L, const ConvPlan& p, int N, char* buf, size_t cap) {
  const ConvWsArgs& a = p.ws;
  const int grid = CeilDiv(N * a.IB, a.P) * L->grp * a.nct;
  if (a.stride == 1) {
    // stride 1: N = channels per CTA, ctiles = channel tiles per group, ksteps = chunks x taps (a CTA's k-steps), so
    // that grid x ksteps x 32 x positions x N is the executed MAC count; wbufs = weight stage buffers
    const int stages = a.nChunks * CeilDiv(a.kt.ntab, a.KS);
    snprintf(buf, cap, " mode=0 N=%d positions=%d ctiles=%d KS=%d smem=%zuB grid=%d NPOS=%d planebufs=%d chunks=%d stages=%d "
             "ksteps=%d wbufs=%d", a.NC, a.P, a.nct, a.KS, p.smem, grid, a.NPOS, a.nPB, a.nChunks, stages,
             a.nChunks * a.kt.ntab, a.nWB);
    return;
  }
  // (no "NT=": the executed-MAC count that bench.py derives from pq_gemm_tc( plans assumes 128-channel tiles)
  int stages = 0;
  for (int c = 0; c < a.nChunks; c++) stages += CeilDiv(a.kt.chunkCount[c], a.KS);
  snprintf(buf, cap, " N=%d positions=%d KS=%d smem=%zuB grid=%d NPOS=%d chunks=%d stages=%d ksteps=%d wbufs=%d", a.NC, a.P,
           a.KS, p.smem, grid, a.NPOS, a.nChunks, stages, a.kt.ntab, a.nWB);
}

}  // namespace qcnn
