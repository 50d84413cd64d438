// Fully-connected layers at large batch as a weight-stationary GEMM on the Hopper tensor cores (the FC form of conv_ws.cu):
//
//     dst[n][o] = bias[o] + sum_{k-steps} sum_{j<8} X_kstep[n][j] * W_kstep[o][j]          (M = images, N = channels)
//
// A k-step is eight consecutive input features (NCHW-flatten order).  d % 4 == 0: its two 4-feature halves are one
// (subspace, piece) slice each of the pre-split codebook d_ctrd_bf; d == 1: eight subspaces of scalar codewords, split
// into bf16 pieces by the decoder.
//
// A = images: the bf16x2 plane image that fc_prep_bf_kernel writes, [tile][chunk][x1, x2][KS k-steps][P images] 16-byte
//     rows, made with P = the images of one CTA and KS = the k-steps of one stage, so that a stage of a CTA is ONE
//     contiguous run, staged by one cp.async.bulk into a ring of plane buffers (full / empty mbarrier per buffer).
//     Row (k-step e, image) of the x1 plane is K-core-matrix 0 of the A descriptor, the same row of the x2 plane (LBO =
//     the plane distance) K-core-matrix 1.
// B = decoded weights in shared memory, N = the channels of one CTA (a tile of Dout; tail channels decode to zero and
//     are never stored), [buffer][k-step][w1, w2][channel] 16-byte rows with the duplicated half read twice (LBO = 0):
//     two MMAs per k-step into one accumulator (ws_common.cuh).  The k-steps of a CTA go in ascending order into that
//     accumulator: the chain and the error bound are those of pq_gemm_tc mode 2 with 128 images per MMA.
//
// Roles inside a CTA of twelve warps (ws_common.cuh):
//   warps 0-7   two consumer warpgroups; each owns MB m64 blocks of the CTA's 128 MB images.
//   warps 8-11  producers: one thread issues the bulk copies of the plane ring; all of them copy the stage's rows of
//               the byte table [S][DoutPad] (this CTA's channels; a bit-packed table is expanded into the same bytes) into
//               shared memory one stage ahead, and decode the stage's weights from them into one of two weight
//               buffers (a thread owns a channel: the index reads are conflict-free).  d % 4 == 0: the codebook pieces are read through L1; d == 1: the
//               stage's scalar codewords are copied into shared memory with its table rows (a decode that waited on
//               L2 for eight codewords per k-step was slower than the MMAs).
//   epilogue    nsplit == 1: bias (+ ReLU) and [N][Dout]; else [split][N][DoutPad] partial sums, split 0 carrying the
//               bias, reduced in fixed order by fc_reduce_kernel (deterministic: no atomics).
#include "packed_asmt.h"
#include "qcnn_internal.h"
#include "ws_common.cuh"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>

namespace {

using qcnn::BulkLoad;
using qcnn::CpAsync16;
using qcnn::CpAsyncCommit;
using qcnn::CpAsyncWaitAll;
using qcnn::kWsConsumers;
using qcnn::kWsProducers;
using qcnn::kWsThreads;
using qcnn::MbarArrive;
using qcnn::MbarExpectTx;
using qcnn::MbarWait;
using qcnn::SmemU32;
using qcnn::SplitBf16x4;
using qcnn::StagePackedRow;

constexpr int kFcWsMaxKS = 8;   // k-steps per stage: 8 or 4

struct FcWsArgs {
  const uint4* xprep;     // plane image [tile][chunk][x1, x2][KS][P] 16-byte rows
  const uint8_t* asmt;    // byte table [S][DoutPad], index << kshift; pkBits != 0: bit-packed rows of pkPitch bytes
  const float* ctrd;      // d == 1: [S][K] scalar codewords
  const uint4* ctrdBf;    // d % 4 == 0: [S][d / 4][K] {w1, w2} pieces (qcnn_layer::d_ctrd_bf)
  const float* bias;
  float* dst;             // nsplit == 1: [N][Dout]; else partial sums [nsplit][N][DoutPad]
  int N, Dout, DoutPad, K, d, kshift;
  int KS, nPB, nct, nsplit, kAll, kPerSplit, nChunksAll, idxRows;
  int pkBits, pkPitch;    // bit-packed table (packed_asmt.h): bits per index, bytes per row (0: the byte table)
  int relu;
};

struct FcWsSmem {  // byte offsets inside the dynamic shared memory
  int planes, wts, idx, cb, bias, bars, total;
};
__host__ __device__ inline FcWsSmem MapFcWsSmem(const FcWsArgs& a, int P, int NC) {
  FcWsSmem m;
  int o = 0;
  m.planes = o; o += a.nPB * 2 * a.KS * P * 16;   // [buffer][x1, x2][KS][P] 16-byte rows
  m.wts = o;    o += 2 * a.KS * 2 * NC * 16;      // [buffer][k-step][w1, w2][channel] 16-byte rows
  m.idx = o;    o += 2 * a.idxRows * NC;          // [buffer][table row][channel] bytes (NC is a multiple of 64)
  m.cb = o;     o += a.d == 1 ? 2 * a.idxRows * a.K * 4 : 0;   // d == 1: [buffer][subspace][K] scalar codewords
  m.bias = o;   o += NC * 4;
  m.bars = o;   o += 8 * (2 * a.nPB + 4);
  m.total = o;
  return m;
}

// first table row and row count of the k-steps [kb, kb + n)
__device__ __forceinline__ void StageRows(const FcWsArgs& a, bool d1, int kb, int n, int& s0, int& nr) {
  if (d1) { s0 = kb * 8; nr = n * 8; return; }
  s0 = kb * 8 / a.d;
  nr = ((kb + n) * 8 - 1) / a.d - s0 + 1;
}

// NC: channels per CTA; MB: m64 blocks per consumer warpgroup; D1: scalar codewords (d == 1), else d % 4 == 0
template <int NC, int MB, bool D1>
__global__ void __launch_bounds__(kWsThreads, 1) fc_ws_kernel(const FcWsArgs a) {
  constexpr int P = 128 * MB;   // images per CTA
  extern __shared__ __align__(128) unsigned char smem[];
  const FcWsSmem sm = MapFcWsSmem(a, P, NC);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int KS = a.KS, nPB = a.nPB;
  uint4* planes = reinterpret_cast<uint4*>(smem + sm.planes);
  uint4* wts = reinterpret_cast<uint4*>(smem + sm.wts);
  uint8_t* idx = smem + sm.idx;
  float* cbS = reinterpret_cast<float*>(smem + sm.cb);
  float* biasS = reinterpret_cast<float*>(smem + sm.bias);
  uint64_t* fullP = reinterpret_cast<uint64_t*>(smem + sm.bars);   // [nPB] planes of a stage landed (bulk copy)
  uint64_t* emptyP = fullP + nPB;                                   // [nPB] planes' MMAs retired: consumers -> producers
  uint64_t* fullW = emptyP + nPB;                                   // [2] weight buffer decoded: producers -> consumers
  uint64_t* emptyW = fullW + 2;                                     // [2] weight buffer's MMAs retired: consumers -> producers
  int bi = blockIdx.x;
  const int ct = bi % a.nct; bi /= a.nct;   // (channel tile, split, image tile): the channel tiles of one plane stage run together
  const int split = bi % a.nsplit, tile = bi / a.nsplit;
  const int ch0 = ct * NC;
  const int kBeg = split * a.kPerSplit, kEnd = min(a.kAll, kBeg + a.kPerSplit);
  const int nSt = (kEnd - kBeg + KS - 1) / KS;
  const int planeRows = KS * P;             // 16-byte rows of one plane (x1 or x2) of a stage

  for (int c = tid; c < NC; c += kWsThreads) biasS[c] = (split == 0 && ch0 + c < a.Dout) ? __ldg(a.bias + ch0 + c) : 0.0f;
  if (tid == 0) qcnn::WsInitBarriers(fullP, emptyP, nPB, 1, fullW, emptyW);
  __syncthreads();

  const int warpU = __shfl_sync(0xffffffffu, warp, 0);   // provably warp-uniform role selector
  if (warpU >= kWsConsumers / 32) {
    // =========================== producers ===========================
    const int pt = tid - kWsConsumers;
    // stage j's plane image into ring buffer j % nPB: one bulk copy, counted on the buffer's full barrier
    auto issuePlanes = [&](int j) {
      const int pb = j % nPB;
      if (j >= nPB) MbarWait<24>(emptyP + pb, ((j / nPB) - 1) & 1);   // buffer last read by the MMAs of stage j - nPB
      const uint32_t bytes = static_cast<uint32_t>(planeRows) * 32u;
      MbarExpectTx(fullP + pb, bytes);
      BulkLoad(planes + pb * 2 * planeRows,
               a.xprep + (static_cast<size_t>(tile) * a.nChunksAll + kBeg / KS + j) * 2 * planeRows, bytes, fullP + pb);
    };
    // stage j's table rows (this CTA's NC channels; granules past DoutPad are zero-filled) into index buffer j & 1
    auto issueIdx = [&](int j) {
      const int kb = kBeg + j * KS, n = min(KS, kEnd - kb);
      int s0, nr;
      StageRows(a, D1, kb, n, s0, nr);
      uint8_t* dstI = idx + (j & 1) * a.idxRows * NC;
      constexpr int G = NC / 16;
      for (int e = pt; e < nr * G; e += kWsProducers) {
        const int r = e / G, ch = ch0 + (e - r * G) * 16;
        const bool ok = ch < a.DoutPad;
        uint8_t* dq = dstI + r * NC + (e - r * G) * 16;
        if (!a.pkBits) CpAsync16(dq, a.asmt + (ok ? static_cast<size_t>(s0 + r) * a.DoutPad + ch : 0), ok);
        // packed rows are expanded into the same bytes by plain stores: visible to every producer after the barrier
        // that starts the stage's decode
        else if (ok) StagePackedRow(dq, a.asmt + static_cast<size_t>(s0 + r) * a.pkPitch, ch, a.pkBits, a.kshift);
        else *reinterpret_cast<uint4*>(dq) = make_uint4(0u, 0u, 0u, 0u);
      }
      if (D1) {   // and the stage's codewords (K floats per subspace, contiguous): the decode reads shared memory only
        float* dstC = cbS + (j & 1) * a.idxRows * a.K;
        const float* srcC = a.ctrd + static_cast<size_t>(s0) * a.K;
        for (int e = pt; e < nr * a.K / 4; e += kWsProducers) CpAsync16(dstC + 4 * e, srcC + 4 * e, true);
      }
      CpAsyncCommit();
    };
    if (pt == 0)
      for (int j = 0; j < min(nPB - 1, nSt); j++) issuePlanes(j);
    issueIdx(0);
    for (int j = 0; j < nSt; j++) {
      const int b = j & 1, kb = kBeg + j * KS, n = min(KS, kEnd - kb);
      CpAsyncWaitAll();          // this thread's rows of stage j landed ...
      qcnn::WsProducerSync();    // ... and everyone's; every producer is done decoding stage j - 1 from the other buffer
      if (j + 1 < nSt) issueIdx(j + 1);
      if (j >= 2) MbarWait<24>(emptyW + b, ((j >> 1) - 1) & 1);   // buffer last read by the MMAs of stage j - 2
      int s0, nr;
      StageRows(a, D1, kb, n, s0, nr);
      const uint8_t* ib = idx + b * a.idxRows * NC;
      const float* cbb = cbS + b * a.idxRows * a.K;
      uint4* w = wts + b * KS * 2 * NC;
      if constexpr (D1) {
        // k-step e = subspaces kb * 8 + 8 e + i (i < 8), one scalar codeword each: table row and codebook row 8 e + i of
        // the stage (unrolled over the k-steps as well, the loop spills)
        for (int c = pt; c < NC; c += kWsProducers) {
          const bool ok = ch0 + c < a.Dout;
#pragma unroll 1
          for (int e = 0; e < n; e++) {
            {
              float v[8];
#pragma unroll
              for (int i = 0; i < 8; i++) v[i] = ok ? cbb[(8 * e + i) * a.K + (ib[(8 * e + i) * NC + c] >> a.kshift)] : 0.0f;
              uint2 p1a, p2a, p1b, p2b;
              SplitBf16x4(make_float4(v[0], v[1], v[2], v[3]), p1a, p2a);
              SplitBf16x4(make_float4(v[4], v[5], v[6], v[7]), p1b, p2b);
              w[(2 * e + 0) * NC + c] = make_uint4(p1a.x, p1a.y, p1b.x, p1b.y);   // w1 of the eight features
              w[(2 * e + 1) * NC + c] = make_uint4(p2a.x, p2a.y, p2b.x, p2b.y);   // w2
            }
          }
        }
      } else {
        // k-step e = features f = (kb + e) * 8: halves [f, f + 4) and [f + 4, f + 8), each one (subspace, piece) slice of
        // K pieces; the slices and the halves' table rows are the same for every channel
        const int dq = a.d >> 2;
        int pA[kFcWsMaxKS], pB[kFcWsMaxKS], rA[kFcWsMaxKS], rB[kFcWsMaxKS];
#pragma unroll
        for (int e = 0; e < kFcWsMaxKS; e++) {
          const int f = (kb + e) * 8, sA = f / a.d, sB = (f + 4) / a.d;
          pA[e] = (sA * dq + ((f - sA * a.d) >> 2)) * a.K; rA[e] = (sA - s0) * NC;
          pB[e] = (sB * dq + ((f + 4 - sB * a.d) >> 2)) * a.K; rB[e] = (sB - s0) * NC;
        }
        for (int c = pt; c < NC; c += kWsProducers) {
          const bool ok = ch0 + c < a.Dout;
          uint4 qa[kFcWsMaxKS], qb[kFcWsMaxKS];
#pragma unroll
          for (int e = 0; e < kFcWsMaxKS; e++) {
            qa[e] = make_uint4(0u, 0u, 0u, 0u);
            qb[e] = qa[e];
            if (e < n && ok) {
              qa[e] = __ldg(a.ctrdBf + pA[e] + (ib[rA[e] + c] >> a.kshift));
              qb[e] = __ldg(a.ctrdBf + pB[e] + (ib[rB[e] + c] >> a.kshift));
            }
          }
#pragma unroll
          for (int e = 0; e < kFcWsMaxKS; e++) {
            if (e < n) {
              w[(2 * e + 0) * NC + c] = make_uint4(qa[e].x, qa[e].y, qb[e].x, qb[e].y);   // [w1 of half A | w1 of half B]
              w[(2 * e + 1) * NC + c] = make_uint4(qa[e].z, qa[e].w, qb[e].z, qb[e].w);   // [w2 of half A | w2 of half B]
            }
          }
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // weights are read by the tensor core
      MbarArrive(fullW + b);
      if (pt == 0 && j + nPB - 1 < nSt) issuePlanes(j + nPB - 1);
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
  const uint32_t lbo = static_cast<uint32_t>(planeRows) * 16u;   // x1 plane -> x2 plane
  for (int j = 0; j < nSt; j++) {
    const int pb = j % nPB, b = j & 1, n = min(KS, kEnd - kBeg - j * KS);
    MbarWait<24>(fullP + pb, (j / nPB) & 1);
    MbarWait<24>(fullW + b, (j >> 1) & 1);
    qcnn::WgmmaFence();
    const uint32_t plA = planes0 + static_cast<uint32_t>(pb * 2 * planeRows) * 16u;
    for (int e = 0; e < n; e++)
      qcnn::WsMmaKStep<NC, MB>(acc, plA, e * P + wg * MB * 64, lbo, wts0 + static_cast<uint32_t>((b * KS + e) * 2 * NC) * 16u);
    qcnn::WsRetireStage(emptyW + b, lane);
    if (lane == 0) MbarArrive(emptyP + pb);   // (the stage's MMAs have retired)
  }

  // ---- epilogue: accumulator fragments (rows = images, columns = channels) -> [N][Dout] or the split's partial sums ----
  const qcnn::WsFrag fr = qcnn::WsFragOf(warp, lane);
  const bool part = a.nsplit > 1;
  const int pitch = part ? a.DoutPad : a.Dout;
  float* out = a.dst + (part ? static_cast<size_t>(split) * a.N * a.DoutPad : 0) + ch0;
  const bool v2 = (pitch & 1) == 0 && (reinterpret_cast<uintptr_t>(a.dst) & 7u) == 0;   // (ch0 and the columns are even)
#pragma unroll
  for (int m = 0; m < MB; m++) {
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int img = tile * P + (wg * MB + m) * 64 + fr.r0 + 8 * h;
      if (img >= a.N) continue;
      float* o = out + static_cast<size_t>(img) * pitch;
#pragma unroll
      for (int i = 0; i < NC / 8; i++) {
        const int ch = 8 * i + 2 * fr.t4;
        if (ch0 + ch >= a.Dout) continue;
        float v0 = acc[m][4 * i + 2 * h] + biasS[ch], v1 = acc[m][4 * i + 2 * h + 1] + biasS[ch + 1];
        if (a.relu) { v0 = fmaxf(v0, 0.0f); v1 = fmaxf(v1, 0.0f); }
        const bool two = ch0 + ch + 1 < a.Dout;
        if (two && v2) *reinterpret_cast<float2*>(o + ch) = make_float2(v0, v1);
        else { o[ch] = v0; if (two) o[ch + 1] = v1; }
      }
    }
  }
}

// (channels per CTA, m64 blocks per consumer warpgroup) with an instantiation, in the planner's order of preference
constexpr int kFcWsShapes[][2] = {{256, 1}, {128, 1}, {128, 2}, {64, 1}, {64, 2}};

template <int NC, int MB, bool D1>
int LaunchInstance(const FcWsArgs& a, unsigned blocks, size_t smem, cudaStream_t st, qcnn_ctx* ctx) {
  if (int rc = qcnn::OptInSmem<fc_ws_kernel<NC, MB, D1>>(ctx)) return rc;
  fc_ws_kernel<NC, MB, D1><<<blocks, kWsThreads, smem, st>>>(a);
  QCNN_CUDA(cudaGetLastError());
  return 0;
}

template <bool D1>
int LaunchShape(const FcWsArgs& a, int nc, int mb, unsigned nb, size_t smem, cudaStream_t st, qcnn_ctx* ctx) {
  if (nc == 256 && mb == 1) return LaunchInstance<256, 1, D1>(a, nb, smem, st, ctx);
  if (nc == 128 && mb == 1) return LaunchInstance<128, 1, D1>(a, nb, smem, st, ctx);
  if (nc == 128 && mb == 2) return LaunchInstance<128, 2, D1>(a, nb, smem, st, ctx);
  if (nc == 64 && mb == 1) return LaunchInstance<64, 1, D1>(a, nb, smem, st, ctx);
  if (nc == 64 && mb == 2) return LaunchInstance<64, 2, D1>(a, nb, smem, st, ctx);
  qcnn::SetError("internal: no fc_ws instantiation for N=%d images=%d", nc, 128 * mb);
  return 1;
}

// cost-model constants on PlanPqGemm's scale (SM-cycles): the L2 -> shared bandwidth one SM can count on for the plane
// image, and the GPU's HBM bandwidth for the partial sums of a K-split and their reduction (H100 SXM: ~5.5 TB/s and
// 3.35 TB/s at ~1.75 GHz)
constexpr double kL2BytesPerSmCycle = 24.0;
constexpr double kHbmBytesPerCycle = 1900.0;

// the layer's arguments of a tiling (the activations, the output and N are bound at launch)
FcWsArgs ArgsOf(const qcnn_layer* L, const FcPlan& c) {
  const auto& p = c.ws;
  FcWsArgs a;
  memset(&a, 0, sizeof(a));
  a.asmt = L->d_asmt.as<uint8_t>(); a.ctrd = L->d_ctrd.as<float>(); a.ctrdBf = L->d_ctrd_bf.as<uint4>(); a.bias = L->d_bias.as<float>();
  a.Dout = L->Dout; a.DoutPad = L->DoutPad; a.K = L->K; a.d = L->d; a.kshift = L->kshift;
  a.KS = p.KS; a.nPB = p.nPB; a.nct = qcnn::CeilDiv(L->Dout, p.NC); a.nsplit = c.nsplit; a.kAll = L->Din / 8;
  a.kPerSplit = p.kPerSplit; a.nChunksAll = qcnn::CeilDiv(a.kAll, p.KS);
  a.idxRows = L->d == 1 ? 8 * p.KS : qcnn::CeilDiv(8 * p.KS, L->d) + 1;
  a.pkBits = L->asmt_bits; a.pkPitch = L->asmt_pitch;
  return a;
}

}  // namespace

namespace qcnn {

// The cheapest tiling of batch N under the gemm_nt / gemm_gt / gemm_ct / gemm_nsplit pins (no on-device timing: a
// layer at a given batch computes the same sums in every process); fails when the pins leave none.
int PlanFcWs(const qcnn_layer* L, int N, FcPlan* out) {
  const int kAll = L->Din / 8;
  const size_t smemMax = SmemOptin(L->ctx);
  const int sms = L->ctx->sm_count;
  double best = 0.0;
  bool found = false;
  for (const auto& shape : kFcWsShapes) {
    const int NC = shape[0], P = 128 * shape[1];
    if (L->opt_gemm_nt && P != L->opt_gemm_nt) continue;
    if (L->opt_gemm_ct && NC != L->opt_gemm_ct) continue;
    const int tiles = CeilDiv(N, P), nct = CeilDiv(L->Dout, NC);
    for (int KS = kFcWsMaxKS; KS >= 4; KS -= 4) {
      if (L->opt_gemm_gt && KS != L->opt_gemm_gt) continue;
      FcPlan c;
      auto& p = c.ws;
      p.P = P; p.NC = NC; p.KS = KS;
      const int nChunksAll = CeilDiv(kAll, KS);
      // a ring of three plane buffers if it fits, else two
      bool fit = false;
      for (p.nPB = 3; p.nPB >= 2 && !fit; p.nPB--) {
        c.nsplit = 1; p.kPerSplit = kAll;
        p.smem = static_cast<size_t>(MapFcWsSmem(ArgsOf(L, c), P, NC).total);
        if (p.smem <= smemMax) { fit = true; break; }
      }
      if (!fit) continue;
      const int maxSplit = std::min(nChunksAll, 64);
      for (int ns = 1; ns <= maxSplit; ns++) {
        const int cps = CeilDiv(nChunksAll, ns);
        if (CeilDiv(nChunksAll, cps) != ns) continue;   // (the same split as a smaller ns)
        if (L->opt_gemm_nsplit && ns != L->opt_gemm_nsplit) continue;
        const double ks = static_cast<double>(cps) * KS;   // k-steps of the busiest CTA
        // tensor work (as PlanConvWs), or the plane image it reads from L2 when that takes longer (every channel tile
        // reads the same image again), a pipeline drain per stage, the set-up
        const double tensor = ks * 2.0 * (P / 64) * (NC / 128.0) * (3.0 * 64.0 * 1.15 / 4.0);
        const double l2 = ks * P * 32.0 / kL2BytesPerSmCycle;
        const double perCta = std::max(tensor, l2) + 600.0 * cps + 4000.0 + P * 24.0;
        const double ctas = static_cast<double>(tiles) * nct * ns;
        double cost = perCta * std::ceil(ctas / sms);
        // a K-split writes and the reduction reads ns partial sums and writes the output, in a launch of its own
        if (ns > 1) cost += (2.0 * ns + 1.0) * N * L->Dout * 4.0 / kHbmBytesPerCycle + 3000.0;
        if (!found || cost < best) {
          best = cost;
          found = true;
          out->ws = p;
          out->nsplit = ns;
          out->ws.kPerSplit = cps * KS;
        }
      }
    }
  }
  QCNN_CHECK(found, "qcnn_fc_aprx_forward: gemm_nt=%d gemm_gt=%d gemm_nsplit=%d gemm_ct=%d has no fc_ws tiling for this layer "
             "at batch %d", L->opt_gemm_nt, L->opt_gemm_gt, L->opt_gemm_nsplit, L->opt_gemm_ct, N);
  return 0;
}

void DescribeFcWs(const qcnn_layer* L, const FcPlan& p, int N, char* buf, size_t cap) {
  // (no "NT=": the executed-MAC count that bench.py derives from pq_gemm_tc( plans assumes 128-channel tiles)
  const int nct = CeilDiv(L->Dout, p.ws.NC);
  snprintf(buf, cap, "pq_gemm_tc_ws(weight-stationary wgmma, weights decoded once per CTA into shared memory, bf16x2) mode=2 "
           "N=%d images=%d ctiles=%d KS=%d smem=%zuB grid=%d planebufs=%d nsplit=%d ksteps=%d", p.ws.NC, p.ws.P, nct, p.ws.KS,
           p.ws.smem, CeilDiv(N, p.ws.P) * nct * p.nsplit, p.ws.nPB, p.nsplit, p.ws.kPerSplit);
}

int LaunchFcWs(qcnn_layer* L, const FcPlan& p, const float* src, int N, float* dst, int relu, cudaStream_t st) {
  FcWsArgs a = ArgsOf(L, p);
  a.N = N; a.relu = relu; a.dst = dst;
  QCNN_CHECK(static_cast<size_t>(MapFcWsSmem(a, p.ws.P, p.ws.NC).total) == p.ws.smem,
             "internal: fc_ws shared-memory carve changed after planning");
  const long long blocks = static_cast<long long>(CeilDiv(N, p.ws.P)) * a.nct * a.nsplit;
  QCNN_CHECK(blocks <= 2147483647LL, "qcnn_fc_aprx_forward: batch too large for the weight-stationary tiling");
  if (int rc = PrepFcPlanes(L, src, N, p.ws.P, p.ws.KS, a.nChunksAll, true, st)) return rc;
  a.xprep = L->d_flat.as<uint4>();
  const unsigned nb = static_cast<unsigned>(blocks);
  return L->d == 1 ? LaunchShape<true>(a, p.ws.NC, p.ws.P / 128, nb, p.ws.smem, st, L->ctx)
                   : LaunchShape<false>(a, p.ws.NC, p.ws.P / 128, nb, p.ws.smem, st, L->ctx);
}

}  // namespace qcnn
