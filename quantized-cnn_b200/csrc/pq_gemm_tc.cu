// PQ layers as decode-at-use GEMMs on the Hopper tensor cores (wgmma), weights decoded straight into registers.
//
//     dst[q][c] = bias[c] + sum_{k-steps} sum_{j<8}  W_kstep[c][j] * X_kstep[q][j]
//
// One k-step is 8 input values of every position q (two 4-float halves); W_kstep[c][half] is the 4-float piece of the
// codeword that channel c's uint8 assignment index names for that half -- the same codebook + index arrays the LUT /
// gather kernels use (reference CaffeEva::CalcFeatMap_ConvAprx / _FCntAprx + GetInPdMat, src/CaffeEva.cc:760-868,
// 968-1025, 1261-1296, evaluated as x . (decoded w) instead of gather(LUT(x)); same sums, different association).
//
// Roles inside a CTA of twelve warps (warp-specialised, mbarrier pipelines, no CTA-wide barrier in the main loop):
//   warps 0-7  two consumer warpgroups, 64 of the tile's 128 output channels each.  A thread decodes exactly the elements
//              of the wgmma A fragment it owns (two channels x one or two value pairs per k-step): index byte -> codeword
//              piece from the staged codebook slice -> registers, then the warpgroup issues wgmma.mma_async (M = 64,
//              N = NT positions) with A from those registers and B = the position planes in shared memory.  Decoded
//              weights never touch shared memory.  bf16x2 operands (default): the codebook was split into bf16 pieces
//              {w1, w2} once at layer creation and the decoders convert nothing; per k-step two MMAs of K = 16
//              ([w1|w1].[x1|x2] + [w2|w2].[x1|x2]).  3xTF32: three MMAs of K = 8 (Ah*Bh + Ah*Bl + Al*Bh).  Conv layers: all
//              tap indices of a chunk sit in registers (channel-major index block, one or two 128-bit loads per chunk).
//              A stage of up to four k-steps is decoded, issued and waited for; the two warpgroups overlap each other.
//   warps 8-11 stagers: the next chunk's positions go global -> registers -> planes (K-major core matrices without
//              swizzle: 8 positions x 16 B, SBO = 128 B, LBO = distance between the two halves / pieces), double-buffered
//              against the MMAs of the current chunk; a chunk's codebook slices and index blocks arrive by
//              cp.async.bulk counted on the chunk's mbarrier (3xTF32: cp.async), four chunks deep.
//              FC layers: the planes were pre-split by fc_prep_kernel and arrive by one cp.async.bulk per chunk.
//   epilogue   the consumers add the bias (+ ReLU) to their accumulator fragments and store them NHWC.
// Instantiations: operands (bf16x2 | 3xTF32) x positions per CTA (NT = 128: one accumulator; NT = 64: the terms with a
// low-order operand piece have an accumulator of their own, added in the epilogue -- the tensor core's accumulation
// error grows with the number of chained MMAs per accumulator, DESIGN.md 2).
//
// Layer geometries are expressed as a table of k-steps (KStep: B start / half distance inside the staged planes, index
// row and codebook slot of either half), so one main loop serves
//   mode 0  stride-1 convolutions: all images form one flat padded grid (image block = (Hi+pad) rows of pitch Wi+pad;
//           the leading pad rows / columns are zero and double as the previous row's / image's trailing padding), a tap
//           is a start-address shift of the B descriptor, a chunk is 8 input channels x all taps;
//   mode 1  strided convolutions with <= 4 input channels (conv1: 11x11 / 4): input de-interleaved into stride x stride
//           phase planes so that a tap again is a shift; a k-step pairs two taps (4 floats each: channels + zero pad);
//           a chunk is one phase row;
//   mode 2  fully-connected layers: position = image, a chunk is a run of k-steps over consecutive input features.
#include "qcnn_internal.h"
#include "wgmma.h"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <cstdio>

namespace {

using qcnn::BulkLoad;
using qcnn::CpAsync16;
using qcnn::CpAsyncCommit;
using qcnn::CpAsyncWaitAll;
using qcnn::MbarArrive;
using qcnn::MbarExpectTx;
using qcnn::MbarInit;
using qcnn::MbarWait;
using qcnn::SmemU32;
using qcnn::SplitTf32x4;
using qcnn::Wgmma;

constexpr int kThreads = 384;
constexpr int kConsumers = 256;  // warps 0-7
constexpr int kStagers = 128;    // warps 8-11
constexpr int kMaxGT = 4;        // k-steps per stage (decoded A fragments of a stage live in registers)
constexpr int kRegPos = 12;      // float4 a stager thread holds in registers (convolution modes: planeF4 <= 12 * 128)
constexpr int kCbBufs = 4;       // codebook / index buffers: the decoders run ahead of the position planes

// ---- bf16x2 operands: v = v1 + v2 with v1 = bf16(v), v2 = bf16(v - v1) (|v - v1 - v2| <= 2^-17 |v|).  One k-step of
// eight values is TWO kind::f16 MMAs of K = 16: [w1 | w1] . [x1 | x2] + [w2 | w2] . [x1 | x2] = (w1 + w2)(x1 + x2) --
// all four cross terms, at the fp16/bf16 rate (twice tf32's), against three K = 8 tf32 MMAs for 3xTF32.
__device__ __forceinline__ uint32_t PackBf16x2(float lo, float hi) {   // low 16 bits = bf16(lo), high 16 bits = bf16(hi)
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ void SplitBf16x4(const float4 v, uint2& p1, uint2& p2) {
  p1.x = PackBf16x2(v.x, v.y);
  p1.y = PackBf16x2(v.z, v.w);
  // residuals against the rounded pieces (exact in fp32)
  const float rx = v.x - __uint_as_float(p1.x << 16), ry = v.y - __uint_as_float(p1.x & 0xFFFF0000u);
  const float rz = v.z - __uint_as_float(p1.y << 16), rw = v.w - __uint_as_float(p1.y & 0xFFFF0000u);
  p2.x = PackBf16x2(rx, ry);
  p2.y = PackBf16x2(rz, rw);
}

// fp32 codebook [S][K][P pieces of 4 floats] -> [S][P][K] x {w1, w2}: the K pieces of one (subspace, piece) are contiguous
__global__ void split_codebook_kernel(const float4* __restrict__ src, uint4* __restrict__ dst, int S, int K, int P) {
  const size_t n = static_cast<size_t>(S) * K * P;
  const size_t gs = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += gs) {
    const int pc = static_cast<int>(i % P);
    const size_t sk = i / P;
    const int k = static_cast<int>(sk % K);
    const size_t sidx = sk / K;
    uint2 p1, p2;
    SplitBf16x4(src[i], p1, p2);
    dst[(sidx * P + pc) * K + k] = make_uint4(p1.x, p1.y, p2.x, p2.y);
  }
}

// byte t (< 32) of the 32 bytes {lo, hi} held in registers (t is warp-uniform: selects, no local memory)
__device__ __forceinline__ int ByteOf32(const uint4 lo, const uint4 hi, int t) {
  const uint32_t x = (t & 16) ? hi.x : lo.x, y = (t & 16) ? hi.y : lo.y, z = (t & 16) ? hi.z : lo.z, w = (t & 16) ? hi.w : lo.w;
  const uint32_t xy = (t & 4) ? y : x, zw = (t & 4) ? w : z;
  const uint32_t v = (t & 8) ? zw : xy;
  return static_cast<int>((v >> ((t & 3) * 8)) & 0xFFu);
}

// byte t (< 48) of the 48 bytes {q0, q1, q2}
__device__ __forceinline__ int ByteOf48(const uint4 q0, const uint4 q1, const uint4 q2, int t) {
  const int hi = t >> 4;
  const uint4 q = hi == 0 ? q0 : (hi == 1 ? q1 : q2);
  const uint32_t xy = (t & 4) ? q.y : q.x, zw = (t & 4) ? q.w : q.z;
  const uint32_t v = (t & 8) ? zw : xy;
  return static_cast<int>((v >> ((t & 3) * 8)) & 0xFFu);
}

struct SmemMap {  // byte offsets inside the dynamic shared memory
  int planes, cbs, ids, tab, posoff, posrow, posdst, outoff, bias, bars, total;
};
__host__ __device__ inline SmemMap MapSmem(const GemmArgs& a) {
  SmemMap m;
  int o = 0;
  m.planes = o; o += a.nPB * 2 * a.planeRows * 16;      // [buf][hi,lo | x1,x2][planeRows] 16-byte rows
  m.cbs = o;    o += kCbBufs * a.cbSlots * a.cbF4 * 16; // [cbuf][slot][cbF4] codeword pieces
  m.ids = o;    o += kCbBufs * a.idRows * 128;          // [cbuf][row][128 channels] assignment indices
  m.tab = o;    o += a.ntab * 16;                       // k-step table for the decoders that do not keep their indices in registers
  m.posoff = o; o += a.planeF4 * 4;                     // source element offset of every staged float4 (-1: zero)
  m.posrow = o; o += a.mode == 1 ? a.planeF4 * 4 : 0;   // mode 1: first input row of the position (phase row 0)
  m.posdst = o; o += (a.bf && a.mode != 2) ? a.planeF4 * 4 : 0;   // bf16x2: byte offset of every staged float4 inside a plane
  m.outoff = o; o += 128 * 4;                           // destination element offset of every position (-1: none)
  m.bias = o;   o += 128 * 4;
  m.bars = o;   o += 8 * (8 + 2 * kCbBufs);
  m.total = o;
  return m;
}

// BF: bf16x2 operands (else 3xTF32); NT: positions per CTA = wgmma N; NT = 64 keeps the second accumulator (a.corr)
template <bool BF, int NT>
__global__ void __launch_bounds__(kThreads, 1) pq_gemm_tc_kernel(const GemmArgs a) {
  constexpr int NTHR = kThreads;
  constexpr int NSTG = kStagers;
  constexpr int RP = kRegPos;
  constexpr bool CORR = NT <= 64;
  extern __shared__ __align__(128) unsigned char smem[];
  const SmemMap sm = MapSmem(a);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int K = a.K, GT = a.GT;

  float4* planes = reinterpret_cast<float4*>(smem + sm.planes);
  float4* cbs = reinterpret_cast<float4*>(smem + sm.cbs);
  uint8_t* ids = smem + sm.ids;
  KStep* tabS = reinterpret_cast<KStep*>(smem + sm.tab);   // (FC tiles: shared memory is lightly loaded there and an LDS beats an indexed LDC)
  int* posoff = reinterpret_cast<int*>(smem + sm.posoff);
  int* posrow = reinterpret_cast<int*>(smem + sm.posrow);
  int* posdst = reinterpret_cast<int*>(smem + sm.posdst);
  int* outoff = reinterpret_cast<int*>(smem + sm.outoff);
  float* biasS = reinterpret_cast<float*>(smem + sm.bias);
  uint64_t* fullB = reinterpret_cast<uint64_t*>(smem + sm.bars);   // [<=4] position planes: stagers -> consumers
  uint64_t* emptyB = fullB + 4;                                    // [<=4] chunk's MMAs retired -> stagers
  uint64_t* fullC = emptyB + 4;                                    // [kCbBufs] codebook + indices: stagers -> consumers
  uint64_t* emptyC = fullC + kCbBufs;                              // [kCbBufs] consumers done with the chunk -> stagers
  int b = blockIdx.x;
  const int ct = b % a.nct; b /= a.nct;
  int g = 0, split = 0;
  if (a.nsplit > 1) { split = b % a.nsplit; b /= a.nsplit; }
  if (a.mode != 2) { g = b % a.G; b /= a.G; }
  const int tile = b;
  const int ch0 = ct * 128;                            // first channel of the tile inside the group
  const int CTv = min(128, a.Kg - ch0);                // valid channels
  const int Q0 = tile * NT;                            // first flat position
  const int i0 = Q0 / a.IB;                            // first image touched
  const float* srcBase = a.src + static_cast<size_t>(i0) * a.srcImg;
  float* dstBase = a.dst + static_cast<size_t>(i0) * a.dstImg + g * a.Kg + ch0;
  // mode 2: this CTA's k-step range [k0, k0 + kTotal) of the layer; partial sums go to their own plane
  const int k0 = split * a.kPerSplit;
  const int kTotal = a.mode == 2 ? min(a.kPerSplit, a.kAll - k0) : 0;
  // convolution modes: K split by chunks [kcBase, kcBase + nChunks) (small batches: more CTAs than position tiles)
  const int kcBase = a.mode == 2 ? 0 : split * a.kPerSplit;
  const int nChunks = a.mode == 2 ? (kTotal + a.chunkCount[0] - 1) / a.chunkCount[0]
                                  : (a.nsplit > 1 ? min(a.kPerSplit, a.nChunks - kcBase) : a.nChunks);
  // mode 2: rows = images, so the tile starts at row Q0 of the output (or of this split's partial sums)
  if (a.mode == 2)
    dstBase = (a.nsplit > 1 ? a.partial + static_cast<size_t>(split) * a.N * a.dstRow : a.dst) + static_cast<size_t>(Q0) * a.dstRow + ch0;
  if (a.mode != 2 && a.nsplit > 1)
    dstBase = a.partial + (static_cast<size_t>(split) * a.N + i0) * a.dstImg + g * a.Kg + ch0;

  // ---- set-up (all threads) ----
  for (int e = tid; e < a.ntab; e += NTHR) tabS[e] = a.tab[e];
  for (int p = tid; p < a.planeF4; p += NTHR) {
    int off = -1;
    if (a.mode == 0) {
      // float4 p: half = p / NPOS, position = p % NPOS; the half only selects the channel offset (added per chunk)
      const int pos = p % a.NPOS;
      const int F = Q0 + pos;
      const int i = F / a.IB, rem = F - i * a.IB;
      const int r = rem / a.PW, c = rem - r * a.PW;
      if (i < a.N && r >= a.pad && c >= a.pad) off = (((i - i0) * a.Hi + (r - a.pad)) * a.Wi + (c - a.pad)) * a.Cin;
    } else if (a.mode == 1) {
      // float4 p: phase column pw = p / NPOS, position = p % NPOS -> pixel (r*stride + ph - pad, c*stride + pw - pad);
      // the phase row ph is the chunk, so the row part is resolved per chunk from posrow
      const int pw = p / a.NPOS, pos = p - pw * a.NPOS;
      const int F = Q0 + pos;
      const int i = F / a.IB, rem = F - i * a.IB;
      const int r = rem / a.PW, c = rem - r * a.PW;
      const int wi = c * a.stride + pw - a.pad;
      const bool colOk = i < a.N && wi >= 0 && wi < a.Wi;
      off = static_cast<int>((i - i0) * a.srcImg) + (r * a.stride - a.pad) * a.rowStride + wi * a.colStride;
      posrow[p] = colOk ? r * a.stride - a.pad : -(1 << 28);
    }
    posoff[p] = off;   // (mode 2 stages its planes by bulk copy: no offsets)
    if (BF && a.mode != 2) {
      // bf16x2 planes hold 16-byte rows of eight values: mode 0 row = position, the half selects bytes 0-7 / 8-15;
      // mode 1 row = (phase-column pair, position), the column's parity selects the half
      const int grp = p / a.NPOS, pos = p - grp * a.NPOS;
      posdst[p] = a.mode == 0 ? pos * 16 + grp * 8 : ((grp >> 1) * a.NPOS + pos) * 16 + (grp & 1) * 8;
    }
  }
  for (int p = tid; p < 128; p += NTHR) {
    int off = -1;
    if (p < NT) {
      const int Q = Q0 + p;
      const int i = Q / a.IB, rem = Q - i * a.IB;
      const int ho = rem / a.PW, wo = rem - ho * a.PW;
      if (a.mode == 2) { if (Q < a.N) off = p * a.dstRow; }
      else if (i < a.N && ho < a.Ho && wo < a.Wo) off = (((i - i0) * a.Ho + ho) * a.Wo + wo) * a.Cout;
    }
    outoff[p] = off;
  }
  if (a.mode == 1 && a.bulkC)      // slot 1 (unpaired taps) stays zero; slot 0 arrives by bulk copy
    for (int e = tid; e < kCbBufs * K; e += NTHR) cbs[(e / K) * a.cbSlots * K + K + (e % K)] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  for (int c = tid; c < 128; c += NTHR) biasS[c] = (c < CTv && split == 0) ? __ldg(a.bias + g * a.Kg + ch0 + c) : 0.0f;
  if (tid == 0) {
    for (int i = 0; i < 4; i++) { MbarInit(fullB + i, NSTG); MbarInit(emptyB + i, kConsumers / 32); }
    for (int i = 0; i < kCbBufs; i++) { MbarInit(fullC + i, a.bulkC ? 1 : NSTG); MbarInit(emptyC + i, kConsumers / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int warpU = __shfl_sync(0xffffffffu, warp, 0);   // provably warp-uniform role selector
  if (warpU >= kConsumers / 32) {
    // =========================== stagers ===========================
    const int st = tid - kConsumers;
    const int sw = st >> 5;                      // stager warp 0 .. NSTG/32 - 1
    // 4-float piece j0/4 of codeword k of subspace s: fp32 codebook [S][K][d] or the pre-split one [S][d/4][K][4 words]
    auto piece = [&](int s, int j0, int k) -> const float* {
      return a.cbPre ? a.ctrd + ((static_cast<size_t>(s) * (a.d >> 2) + (j0 >> 2)) * K + k) * 4
                     : a.ctrd + (static_cast<size_t>(s) * K + k) * a.d + j0;
    };
    // chunk kc: codebook slices + index rows by cp.async (one group); the positions travel through registers
    auto fetchChunk = [&](int kc) {
      const int cbuf = kc % kCbBufs;
      if (a.mode == 0) {
        // per-chunk scalars: the two 4-channel halves, their subspaces and the offsets inside the codewords
        const int taps = a.ksz * a.ksz;
        const int chA = (kcBase + kc) * 8, chB = chA + 4;
        const bool okA = chA < a.Cg, okB = chB < a.Cg;
        const int sA = okA ? chA / a.d : 0, jA = okA ? chA - sA * a.d : 0;
        const int sB = okB ? chB / a.d : 0, jB = okB ? chB - sB * a.d : 0;
        // (positions travel through registers: loadPos / storePos)
        // codebook slices: slot = half
        float4* cdst = cbs + cbuf * a.cbSlots * K;
        if (a.bulkC) {
          // four bulk copies (two contiguous codebook slices, two contiguous index blocks), completion counted on fullC;
          // a half beyond the group's channels stages valid data (its positions are staged as zeros)
          if (st == 0) {
            const uint32_t cbBytes = static_cast<uint32_t>(K) * 16u, idBytes = static_cast<uint32_t>(CTv * a.tapsPad);
            uint64_t* bar = fullC + cbuf;
            uint8_t* idst = ids + cbuf * a.idRows * 128;
            const uint8_t* tA = a.asmtT + (static_cast<size_t>(g * a.S + sA) * a.KgPad + ch0) * a.tapsPad;
            const uint8_t* tB = a.asmtT + (static_cast<size_t>(g * a.S + sB) * a.KgPad + ch0) * a.tapsPad;
            MbarExpectTx(bar, 2u * cbBytes + 2u * idBytes);
            BulkLoad(cdst, piece(sA, jA, 0), cbBytes, bar);
            BulkLoad(cdst + K, piece(sB, jB, 0), cbBytes, bar);
            BulkLoad(idst, tA, idBytes, bar);
            BulkLoad(idst + 128 * a.tapsPad, tB, idBytes, bar);
          }
          return;
        }
        for (int k = st; k < K; k += NSTG) {
          CpAsync16(cdst + k, piece(sA, jA, k), okA);
          CpAsync16(cdst + K + k, piece(sB, jB, k), okB);
        }
        if (a.idxT) {
          // channel-major index block [half][channel][tapsPad]: contiguous CTv * tapsPad bytes per half
          const int gran = (CTv * a.tapsPad) >> 4;
          const uint8_t* tA = a.asmtT + (static_cast<size_t>(g * a.S + sA) * a.KgPad + ch0) * a.tapsPad;
          const uint8_t* tB = a.asmtT + (static_cast<size_t>(g * a.S + sB) * a.KgPad + ch0) * a.tapsPad;
          uint8_t* idst = ids + cbuf * a.idRows * 128;
          for (int e = st; e < 2 * gran; e += NSTG) {
            const bool hb = e >= gran;
            const int q = hb ? e - gran : e;
            CpAsync16(idst + (hb ? 128 * a.tapsPad : 0) + (q << 4), (hb ? tB : tA) + (static_cast<size_t>(q) << 4), true);
          }
        }
        // index rows [half][tap]: stager warp w takes rows w, w+3, ...; lane < gran copies one 16-byte granule
        const int gran = CTv >> 4;
        if (!a.idxT && lane < gran) {
          const uint8_t* asA = a.asmt + static_cast<size_t>(g * a.S + sA) * taps * a.KgPad + ch0 + (lane << 4);
          const uint8_t* asB = a.asmt + static_cast<size_t>(g * a.S + sB) * taps * a.KgPad + ch0 + (lane << 4);
          uint8_t* idst = ids + cbuf * a.idRows * 128 + (lane << 4);
          for (int row = sw; row < 2 * taps; row += NSTG / 32) {
            const bool hb = row >= taps;
            const int tap = hb ? row - taps : row;
            CpAsync16(idst + row * 128, (hb ? asB : asA) + static_cast<size_t>(tap) * a.KgPad, true);
          }
        }
      }
      if (a.mode == 1) {
        // chunk = phase row ph: pixels of input rows r*stride + ph - pad, one 4-byte copy per channel
        const int ph = kcBase + kc;
        // (positions travel through registers: loadPos / storePos)
        // codebook: slot 0 = the first 4 floats of every codeword of subspace 0, slot 1 = zeros (unpaired taps)
        float4* cdst = cbs + cbuf * a.cbSlots * K;
        if (a.bulkC) {
          if (st == 0) {
            const uint32_t cbBytes = static_cast<uint32_t>(K) * 16u, idBytes = static_cast<uint32_t>(CTv * a.tapsPad);
            uint64_t* bar = fullC + cbuf;
            const uint8_t* tA = a.asmtT + (static_cast<size_t>(g * a.stride + ph) * a.KgPad + ch0) * a.tapsPad;
            MbarExpectTx(bar, cbBytes + idBytes);
            BulkLoad(cdst, piece(0, 0, 0), cbBytes, bar);
            BulkLoad(ids + cbuf * a.idRows * 128, tA, idBytes, bar);
          }
          return;
        }
        for (int k = st; k < K; k += NSTG) {
          CpAsync16(cdst + k, piece(0, 0, k), true);
          CpAsync16(cdst + K + k, a.ctrd, false);
        }
        // index rows of the taps with kh % stride == ph, in (kh, kw) order
        const int gran = CTv >> 4;
        if (lane < gran) {
          const uint8_t* as0 = a.asmt + static_cast<size_t>(g * a.S) * a.ksz * a.ksz * a.KgPad + ch0 + (lane << 4);
          uint8_t* idst = ids + cbuf * a.idRows * 128 + (lane << 4);
          const int nrow = ((a.ksz - ph + a.stride - 1) / a.stride) * a.ksz;
          for (int row = sw; row < nrow; row += NSTG / 32) {
            const int kh = ph + (row / a.ksz) * a.stride, kw = row % a.ksz;
            CpAsync16(idst + row * 128, as0 + static_cast<size_t>(kh * a.ksz + kw) * a.KgPad, true);
          }
        }
      }
      if (a.mode == 2) {
        // chunk = KS consecutive k-steps of this CTA's range: features [f0, f0 + 8 ne)
        const int KS = a.chunkCount[0];
        const int ne = min(KS, kTotal - kc * KS);
        const int f0 = (k0 + kc * KS) * 8;
        const int gran = (CTv + 15) >> 4;
        if (a.d == 1) {
          // slot q = subspace f0 + q: its K scalar codewords; index row q
          const int kq = K >> 2;
          float4* cdst = cbs + cbuf * a.cbSlots * a.cbF4;
          for (int e = st; e < 8 * ne * kq; e += NSTG) CpAsync16(cdst + e, a.ctrd + static_cast<size_t>(f0) * K + e * 4, true);
          if (lane < gran) {
            const uint8_t* as0 = a.asmt + static_cast<size_t>(f0) * a.KgPad + ch0 + (lane << 4);
            uint8_t* idst = ids + cbuf * a.idRows * 128 + (lane << 4);
            for (int row = sw; row < 8 * ne; row += NSTG / 32) CpAsync16(idst + row * 128, as0 + static_cast<size_t>(row) * a.KgPad, true);
          }
        } else {
          // slot q = features [f0 + 4q, +4): piece j0 of every codeword of subspace s; index row q = row s of the layer
          float4* cdst = cbs + cbuf * a.cbSlots * a.cbF4;
          for (int e = st; e < 2 * ne * K; e += NSTG) {
            const int q = e / K, k = e - q * K;
            const int f = f0 + 4 * q;
            const int s = f / a.d, j0 = f - s * a.d;
            CpAsync16(cdst + e, piece(s, j0, k), true);
          }
          if (lane < gran) {
            uint8_t* idst = ids + cbuf * a.idRows * 128 + (lane << 4);
            for (int row = sw; row < 2 * ne; row += NSTG / 32) {
              const int s = (f0 + 4 * row) / a.d;
              CpAsync16(idst + row * 128, a.asmt + static_cast<size_t>(s) * a.KgPad + ch0 + (lane << 4), true);
            }
          }
        }
      }
      CpAsyncCommit();
    };
    // Positions of the convolution modes: global -> registers -> hi/lo planes.  (16-byte cp.async of scattered pieces
    // costs one shared-memory wavefront per THREAD, whereas a 128-bit store of 32 consecutive float4 costs four per
    // warp.)  A thread owns float4 st, st + kStagers, ...: at most kRegPos of them.
    float4 rg[RP];
    int poffR[RP];        // chunk-invariant source offset of the thread's float4 (mode 0: incl. the half's +4)
    int prowR[RP];        // mode 1: first input row (phase row 0), very negative when the column is outside
    uint32_t pvalid = 0;       // mode 0: bit i = the float4 exists and its position is inside an image
    uint32_t phalf = 0;        // mode 0: bit i = second half (channels 4..7 of the chunk)
    if (a.mode != 2) {
#pragma unroll
      for (int i = 0; i < RP; i++) {
        const int p = st + i * NSTG;
        poffR[i] = 0; prowR[i] = -(1 << 28);
        if (p < a.planeF4) {
          const int off = posoff[p];
          if (a.mode == 0) {
            const bool hb = p >= a.NPOS;
            poffR[i] = off + (hb ? 4 : 0);
            if (off >= 0) pvalid |= 1u << i;
            if (hb) phalf |= 1u << i;
          } else {
            poffR[i] = off;
            prowR[i] = posrow[p];
          }
        }
      }
    }
    auto loadPos = [&](int kc) {
      if (a.mode == 0) {
        const int chA = (kcBase + kc) * 8;
        uint32_t m = pvalid;
        if (chA >= a.Cg) m = 0;
        else if (chA + 4 >= a.Cg) m &= ~phalf;
        const float* srcG = srcBase + g * a.Cg + chA;
#pragma unroll
        for (int i = 0; i < RP; i++) {
          rg[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
          if ((m >> i) & 1u) rg[i] = __ldg(reinterpret_cast<const float4*>(srcG + poffR[i]));
        }
      } else {
        const int ph = kcBase + kc;
        const float* srcG = srcBase + static_cast<size_t>(g) * a.Cg * a.chStride + ph * a.rowStride;
#pragma unroll
        for (int i = 0; i < RP; i++) {
          rg[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
          if (static_cast<unsigned>(prowR[i] + ph) < static_cast<unsigned>(a.Hi)) {
            const float* px = srcG + poffR[i];
            rg[i].x = __ldg(px);
            if (a.Cg > 1) rg[i].y = __ldg(px + a.chStride);
            if (a.Cg > 2) rg[i].z = __ldg(px + 2 * a.chStride);
            if (a.Cg > 3) rg[i].w = __ldg(px + 3 * a.chStride);
          }
        }
      }
    };
    fetchChunk(0);
    if (a.mode != 2) loadPos(0);
    if (nChunks > 1) fetchChunk(1);
    for (int kc = 0; kc < nChunks; kc++) {
      const int buf = kc % a.nPB;
      if (!a.bulkC) {
        if (kc + 1 < nChunks) asm volatile("cp.async.wait_group 1;" ::: "memory");   // chunk kc landed, kc+1 may be in flight
        else CpAsyncWaitAll();
        // (each stager arrives after its own copies have landed; the barrier completes when all of them have)
        MbarArrive(fullC + kc % kCbBufs);                  // the consumers may start on chunk kc
      }
      if (kc >= a.nPB) MbarWait<24>(emptyB + buf, ((kc / a.nPB) - 1) & 1);   // planes last read by the MMAs of chunk kc-nPB
      float4* pHi = planes + (buf * 2 + 0) * a.planeRows;
      float4* pLo = planes + (buf * 2 + 1) * a.planeRows;
      if (a.mode == 2) {
        // the plane image of (tile, chunk) was written by fc_prep_kernel: one bulk copy (hi + lo, contiguous) straight
        // into the planes, completion counted on the same mbarrier the stagers arrive on
        if (st == 0) {
          const uint32_t bytes = static_cast<uint32_t>(a.planeRows) * 32u;
          const float* gsrc = a.xprep + (static_cast<size_t>(tile) * a.nChunksAll + (k0 / a.chunkCount[0] + kc)) * a.planeRows * 8;
          MbarExpectTx(fullB + buf, bytes);
          BulkLoad(pHi, gsrc, bytes, fullB + buf);
        } else {
          MbarArrive(fullB + buf);
        }
      } else {
#pragma unroll
        for (int i = 0; i < RP; i++) {
          const int p = st + i * NSTG;
          if (p < a.planeF4) {
            if (BF) {
              uint2 p1, p2;
              SplitBf16x4(rg[i], p1, p2);
              const int db = posdst[p];
              *reinterpret_cast<uint2*>(reinterpret_cast<char*>(pHi) + db) = p1;
              *reinterpret_cast<uint2*>(reinterpret_cast<char*>(pLo) + db) = p2;
            } else {
              float4 hi, lo;
              SplitTf32x4(rg[i], hi, lo);
              pHi[p] = hi;
              pLo[p] = lo;
            }
          }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // planes are read by the tensor core
        MbarArrive(fullB + buf);
        if (kc + 1 < nChunks) loadPos(kc + 1);
      }
      if (kc + 2 < nChunks) {
        const int nb = (kc + 2) % kCbBufs;
        if (kc + 2 >= kCbBufs) MbarWait<24>(emptyC + nb, (((kc + 2) / kCbBufs) - 1) & 1);
        fetchChunk(kc + 2);
      }
    }
    return;
  }

  // =========================== consumers: decode + wgmma ===========================
  // Fragment ownership (wgmma A / D, one 16-row slice per warp): this thread holds rows r0 = 16 * (warp in group) + lane / 4
  // and r0 + 8 of its warpgroup's 64 channels; of a k-step's eight values it holds the pair 2 * (lane % 4), +1 (bf16x2: both
  // copies of [w | w]) or the values lane % 4 of either half (tf32).
  const int gid = lane >> 2, t4 = lane & 3;
  const int row0 = (warp >> 2) * 64 + (warp & 3) * 16 + gid, row1 = row0 + 8;
  const int cc0 = min(row0, CTv - 1), cc1 = min(row1, CTv - 1);   // rows beyond the valid channels decode a copy (never stored)
  const int myHalf = t4 >> 1, myWord = t4 & 1;                    // bf16x2: the half and the value pair inside its piece
  const bool pre = BF && a.cbPre != 0;
  float acc[NT / 2], acc2[CORR ? NT / 2 : 1];
#pragma unroll
  for (int i = 0; i < NT / 2; i++) acc[i] = 0.0f;
#pragma unroll
  for (int i = 0; i < (CORR ? NT / 2 : 1); i++) acc2[i] = 0.0f;
  float (&accLo)[CORR ? NT / 2 : 1] = acc2;
  const uint64_t descFixed = static_cast<uint64_t>(8) << 32;     // SBO = 128 B; LBO and the start address come per k-step
  const uint32_t planes0 = SmemU32(planes);

  for (int kc = 0; kc < nChunks; kc++) {
    const int cbuf = kc % kCbBufs, buf = kc % a.nPB;
    MbarWait<24>(fullC + cbuf, (kc / kCbBufs) & 1);
    const uint8_t* idb = ids + cbuf * a.idRows * 128;
    const float4* cb = cbs + cbuf * a.cbSlots * a.cbF4;
    const float* cbf = reinterpret_cast<const float*>(cb);
    const uint32_t* cbw = reinterpret_cast<const uint32_t*>(cb);
    const int e0 = a.chunkFirst[a.mode == 1 ? kcBase + kc : 0];
    const int ne = a.mode == 2 ? min(a.chunkCount[0], kTotal - kc * a.chunkCount[0]) : a.chunkCount[a.mode == 1 ? kcBase + kc : 0];
    // idxT: every tap index of the thread's two channels for the chunk in registers (one to three 128-bit loads each): the
    // per-k-step chain is one dependent shared-memory round trip (the codeword piece)
    //   mode 0: iq[ch][2 h], iq[ch][2 h + 1] = the taps of half-slot h (bf16x2: the thread's own half; tf32: both halves)
    //   mode 1: iq[ch][0..2] = the <= 48 rows of the phase row
    uint4 iq[2][4];
#pragma unroll
    for (int c = 0; c < 2; c++)
#pragma unroll
      for (int j = 0; j < 4; j++) iq[c][j] = make_uint4(0, 0, 0, 0);
    if (a.idxT) {
      const uint4* ip = reinterpret_cast<const uint4*>(idb);
      const int W = a.tapsPad >> 4;
#pragma unroll
      for (int c = 0; c < 2; c++) {
        const int cc = c ? cc1 : cc0;
        if (a.mode == 1) {
          iq[c][0] = ip[cc * W];
          if (W > 1) iq[c][1] = ip[cc * W + 1];
          if (W > 2) iq[c][2] = ip[cc * W + 2];
        } else {
#pragma unroll
          for (int h = 0; h < (BF ? 1 : 2); h++) {
            const int half = BF ? myHalf : h;
            iq[c][2 * h] = ip[(half * 128 + cc) * W];
            if (W > 1) iq[c][2 * h + 1] = ip[(half * 128 + cc) * W + 1];
          }
        }
      }
    }
    // float4 index (inside the chunk's staged codebook) of the piece that `half` of k-step (ks, tap) takes for channel c
    auto pieceOf = [&](const KStep& ks, int tap, int half, int c) -> int {
      if (a.idxT && a.mode == 1)
        return (half ? ks.cb1 : ks.cb0) * K + ByteOf48(iq[c][0], iq[c][1], iq[c][2], half ? ks.idx1 : ks.idx0);
      if (a.idxT) {
        const int h = BF ? 0 : half;
        return half * K + ByteOf32(iq[c][2 * h], iq[c][2 * h + 1], tap);
      }
      return (half ? ks.cb1 : ks.cb0) * K + (idb[(half ? ks.idx1 : ks.idx0) * 128 + (c ? cc1 : cc0)] >> a.kshift);
    };
    // scalar codewords (d = 1): value j (< 4) of `half` is its own subspace: row / slot idx + j
    auto scalarOf = [&](const KStep& ks, int half, int j, int c) -> float {
      const int row = (half ? ks.idx1 : ks.idx0) + j, slot = (half ? ks.cb1 : ks.cb0) + j;
      return cbf[slot * K + (idb[row * 128 + (c ? cc1 : cc0)] >> a.kshift)];
    };
    MbarWait<24>(fullB + buf, (kc / a.nPB) & 1);
    const uint64_t dHi = descFixed | (((planes0 + static_cast<uint32_t>((buf * 2 + 0) * a.planeRows) * 16u) >> 4) & 0x3FFFu);
    const uint64_t dLo = descFixed | (((planes0 + static_cast<uint32_t>((buf * 2 + 1) * a.planeRows) * 16u) >> 4) & 0x3FFFu);
    for (int s0 = 0; s0 < ne; s0 += GT) {
      const int n = min(GT, ne - s0);
      // the stage's k-steps are independent: index bytes and codeword pieces of all of them are in flight together
      uint32_t fa[kMaxGT][BF ? 4 : 8];
      uint64_t boff[kMaxGT];
#pragma unroll
      for (int i = 0; i < kMaxGT; i++) {
        if (i < n) {
          const KStep ks = (a.idxT || a.mode != 2) ? a.tab[e0 + s0 + i] : tabS[e0 + s0 + i];
          boff[i] = static_cast<uint64_t>(static_cast<uint32_t>(ks.bStart)) | (static_cast<uint64_t>(static_cast<uint32_t>(ks.lbo)) << 16);
          if constexpr (BF) {
            // [w1 | w1] -> fa[0..1] (rows r0, r1; both K halves read the same registers), [w2 | w2] -> fa[2..3]
#pragma unroll
            for (int c = 0; c < 2; c++) {
              if (a.d == 1) {
                const float v0 = scalarOf(ks, myHalf, 2 * myWord, c), v1 = scalarOf(ks, myHalf, 2 * myWord + 1, c);
                const uint32_t p1 = PackBf16x2(v0, v1);
                fa[i][c] = p1;
                fa[i][2 + c] = PackBf16x2(v0 - __uint_as_float(p1 << 16), v1 - __uint_as_float(p1 & 0xFFFF0000u));
              } else {
                const int pi = pieceOf(ks, s0 + i, myHalf, c);
                if (pre) {
                  fa[i][c] = cbw[pi * 4 + myWord];
                  fa[i][2 + c] = cbw[pi * 4 + 2 + myWord];
                } else {
                  const float2 v = reinterpret_cast<const float2*>(cb)[pi * 2 + myWord];
                  const uint32_t p1 = PackBf16x2(v.x, v.y);
                  fa[i][c] = p1;
                  fa[i][2 + c] = PackBf16x2(v.x - __uint_as_float(p1 << 16), v.y - __uint_as_float(p1 & 0xFFFF0000u));
                }
              }
            }
          } else {
            // tf32 fragment: (r0, half 0), (r1, half 0), (r0, half 1), (r1, half 1), value t4 of the half; hi -> fa[0..3], lo -> fa[4..7]
#pragma unroll
            for (int h = 0; h < 2; h++)
#pragma unroll
              for (int c = 0; c < 2; c++) {
                const float v = a.d == 1 ? scalarOf(ks, h, t4, c) : cbf[pieceOf(ks, s0 + i, h, c) * 4 + t4];
                const uint32_t hi = __float_as_uint(v) & 0xFFFFE000u;
                fa[i][2 * h + c] = hi;
                fa[i][4 + 2 * h + c] = __float_as_uint(v - __uint_as_float(hi));
              }
          }
        }
      }
      qcnn::WgmmaFence();
#pragma unroll
      for (int i = 0; i < kMaxGT; i++) {
        if (i < n) {
          if constexpr (BF) {
            // B = [x1 | x2]: K-core-matrix 0 in the first plane, 1 in the second (the table's lbo is the plane distance)
            Wgmma<NT>::Bf16RS(acc, fa[i][0], fa[i][1], fa[i][0], fa[i][1], dHi + boff[i]);
            if constexpr (CORR) Wgmma<NT>::Bf16RS(accLo, fa[i][2], fa[i][3], fa[i][2], fa[i][3], dHi + boff[i]);
            else Wgmma<NT>::Bf16RS(acc, fa[i][2], fa[i][3], fa[i][2], fa[i][3], dHi + boff[i]);
          } else {
            Wgmma<NT>::Tf32RS(acc, fa[i][0], fa[i][1], fa[i][2], fa[i][3], dHi + boff[i]);
            if constexpr (CORR) {
              Wgmma<NT>::Tf32RS(accLo, fa[i][0], fa[i][1], fa[i][2], fa[i][3], dLo + boff[i]);
              Wgmma<NT>::Tf32RS(accLo, fa[i][4], fa[i][5], fa[i][6], fa[i][7], dHi + boff[i]);
            } else {
              Wgmma<NT>::Tf32RS(acc, fa[i][0], fa[i][1], fa[i][2], fa[i][3], dLo + boff[i]);
              Wgmma<NT>::Tf32RS(acc, fa[i][4], fa[i][5], fa[i][6], fa[i][7], dHi + boff[i]);
            }
          }
        }
      }
      qcnn::WgmmaCommit();
      qcnn::WgmmaWaitAll();
    }
    // the chunk's MMAs have retired: its planes and its codebook / index buffer may be refilled
    __syncwarp();
    if (lane == 0) { MbarArrive(emptyB + buf); MbarArrive(emptyC + cbuf); }
  }

  // ---- epilogue: accumulator fragments (rows = channels r0, r1; columns = positions 8 i + 2 t4, +1) -> + bias, ReLU -> NHWC ----
  {
    const bool ok0 = row0 < CTv, ok1 = row1 < CTv;
    const float b0 = biasS[row0], b1 = biasS[row1];
#pragma unroll
    for (int i = 0; i < NT / 8; i++) {
#pragma unroll
      for (int j = 0; j < 2; j++) {
        const int off = outoff[8 * i + 2 * t4 + j];
        if (off < 0) continue;
        float v0 = acc[4 * i + j] + b0, v1 = acc[4 * i + 2 + j] + b1;
        if constexpr (CORR) { v0 += acc2[CORR ? 4 * i + j : 0]; v1 += acc2[CORR ? 4 * i + 2 + j : 0]; }
        if (a.relu) { v0 = fmaxf(v0, 0.0f); v1 = fmaxf(v1, 0.0f); }   // (never set together with split-K partial sums)
        if (ok0) dstBase[off + row0] = v0;
        if (ok1) dstBase[off + row1] = v1;
      }
    }
  }
}

}  // namespace

namespace qcnn {

// Candidate tilings for batch N (cost in SM-cycles, comparable with PlanConv's model); on-device timing chooses among them.
void PlanPqGemm(const qcnn_layer* L, int N, std::vector<std::pair<double, ConvPlan>>* cands) {
  const int G = L->grp, Cg = L->Cin / G, Kg = L->Cout / G, taps = L->ksz * L->ksz;
  if (L->K < 1 || L->K > 256 || Kg % 16 != 0) return;
  const size_t smemMax0 = L->ctx->smem_optin ? L->ctx->smem_optin : 227 * 1024;
  if (L->stride > 1) {
    // mode 1: strided convolution with one subspace over <= 4 input channels (conv1), input on stride x stride phase planes
    const int st = L->stride, rowsPer = CeilDiv(L->ksz, st);
    if (Cg > 4 || L->S != 1 || L->d < Cg || st > 8 || L->Wo > CeilDiv(L->Win + 2 * L->pad, st)) return;
    const int pairs = (L->ksz + 1) / 2;
    if (rowsPer * pairs > 32 || L->ksz * pairs > kMaxKSteps) return;
    const int PWp = CeilDiv(L->Win + 2 * L->pad, st), PHp = CeilDiv(L->Hin + 2 * L->pad, st);
    const int IB = PHp * PWp;
    if (static_cast<double>(N) * IB > 2.0e9 || static_cast<double>(L->Hin) * L->Win * L->Cin * 4 > 2.0e9) return;
    const int nts1[2] = {128, 64};
    for (int ni = 0; ni < 2; ni++) {
      const int NT = nts1[ni];
      const int gts1[2] = {4, 3};
      for (int gi = 0; gi < 2; gi++) {
        const int GT = gts1[gi];
        ConvPlan p;
        memset(&p, 0, sizeof(p));
        p.kernel = kPqGemmTc; p.CPT = NT; p.J = GT; p.threads = kThreads;
        GemmArgs& ga = p.g;
        ga.mode = 1;
        ga.PW = PWp; ga.IB = IB; ga.NT = NT; ga.GT = GT;
        ga.NPOS = RoundUp(NT + ((L->ksz - 1) / st) * (PWp + 1), 8);
        ga.planeF4 = st * ga.NPOS;
        if (ga.planeF4 > kRegPos * kStagers) continue;
        ga.corr = NT <= 64 ? 1 : 0;
        ga.bf = L->opt_tc_bf ? 1 : 0;
        if (ga.bf && (st & 1)) continue;       // bf16x2 rows hold a PAIR of phase columns
        ga.planeRows = ga.bf ? (st / 2) * ga.NPOS : ga.planeF4;
        ga.cbSlots = 2; ga.idRows = rowsPer * L->ksz;
        ga.tapsPad = RoundUp(rowsPer * L->ksz, 16);
        ga.idxT = (ga.tapsPad <= 48 && L->d_asmt_t.get() && L->asmt_t_mode == 1) ? 1 : 0;
        if (ga.idxT) ga.idRows = ga.tapsPad;       // [128 channels][tapsPad] bytes
        ga.nChunks = st;
        ga.K = L->K; ga.cbF4 = L->K; ga.nPB = 2;
        // bf16x2 planes are half the size: keep EVERY phase row of the tile resident (no plane reuse), so that the stagers
        // never wait for the MMAs and the few k-steps of a phase row (conv1: 16-18) are not what hides a global-load latency
        if (ga.bf && st <= 4) ga.nPB = st;
        ga.nct = CeilDiv(Kg, 128);
        int ne = 0;
        for (int ph = 0; ph < st; ph++) {
          ga.chunkFirst[ph] = ne;
          for (int kh = ph; kh < L->ksz; kh += st)
            for (int kw = 0; kw < L->ksz; kw += 2, ne++) {
              if (ne >= kMaxKSteps) { ne = kMaxKSteps + 1000; break; }
              KStep& ks = ga.tab[ne];
              // partner in the next phase column, same shift (bf16x2: the partner must be the odd column of the same pair)
              const bool paired = kw + 1 < L->ksz && (kw % st) + 1 < st && !(ga.bf && ((kw % st) & 1));
              ks.bStart = (kw % st) * ga.NPOS + (kh / st) * PWp + kw / st;
              // an unpaired tap's second half (zero codebook slot) aliases its first half (LBO = 0): a shift would read
              // the next position -- for a tile's last position, or a tap at the end of an image, another image's
              // pixel -- and 0 * NaN / Inf would carry that image's non-finite values into this one's output
              ks.lbo = paired ? ga.NPOS : 0;
              if (ga.bf) {   // row = (pair of phase columns, position); K-core-matrix 1 = the x2 plane
                ks.bStart = ((kw % st) >> 1) * ga.NPOS + (kh / st) * PWp + kw / st;
                ks.lbo = ga.planeRows;
              }
              ks.idx0 = static_cast<short>((kh - ph) / st * L->ksz + kw);
              ks.idx1 = static_cast<short>(paired ? ks.idx0 + 1 : ks.idx0);
              ks.cb0 = 0; ks.cb1 = paired ? 0 : 1;
              if (!paired && kw + 1 < L->ksz) kw--;   // the partner starts its own k-step
            }
          ga.chunkCount[ph] = ne - ga.chunkFirst[ph];
        }
        if (ne > kMaxKSteps) continue;
        ga.ntab = ne;
        p.smem = static_cast<size_t>(MapSmem(ga).total);
        if (p.smem > smemMax0) continue;
        p.a.CT = 128; p.a.nct = ga.nct; p.a.R = NT; p.a.nstrips = GT;
        const double ctas0 = static_cast<double>(CeilDiv(N * IB, NT)) * G * ga.nct;
        // small batches: split the phase rows over CTAs (partial sums reduced by LaunchSplitReduce)
        for (int nsplit = 1; nsplit <= st; nsplit *= 2) {
          if (nsplit > 1 && ctas0 * nsplit > 1.5 * L->ctx->sm_count) break;
          ga.kPerSplit = CeilDiv(st, nsplit);
          ga.nsplit = CeilDiv(st, ga.kPerSplit);
          if (ga.nsplit != nsplit) continue;
          p.a.rgroups = nsplit;
          const double perCta = ne * 3.0 * (NT / 2.0) * 1.15 / nsplit + 120.0 * ne / GT / nsplit + 9000.0 + NT * 24.0 +
                                (nsplit > 1 ? 6000.0 : 0.0);
          cands->emplace_back(perCta * std::ceil(ctas0 * nsplit / L->ctx->sm_count), p);
        }
      }
    }
    return;
  }
  if (L->src_nchw) return;
  if (L->d % 4 != 0 || Cg % 4 != 0 || L->Cin % 4 != 0 || L->S * L->d < Cg || taps > kMaxKSteps) return;
  const int PW = L->Win + L->pad, IB = (L->Hin + L->pad) * PW;
  if (L->Ho > L->Hin + L->pad || L->Wo > PW) return;
  if (static_cast<double>(N) * IB > 2.0e9) return;
  const size_t smemMax = L->ctx->smem_optin ? L->ctx->smem_optin : 227 * 1024;
  const int nts[2] = {128, 64};
  for (int ni = 0; ni < 2; ni++) {
    const int NT = nts[ni];
    const int gts[2] = {4, 3};
    for (int gi = 0; gi < 2; gi++) {
      const int GT = gts[gi];
      ConvPlan p;
      memset(&p, 0, sizeof(p));
      p.kernel = kPqGemmTc; p.CPT = NT; p.J = GT; p.threads = kThreads;
      GemmArgs& ga = p.g;
      ga.mode = 0;
      ga.PW = PW; ga.IB = IB; ga.NT = NT; ga.GT = GT;
      ga.NPOS = RoundUp(NT + (L->ksz - 1) * (PW + 1), 8);
      if (ga.NPOS > 16000) continue;
      ga.planeF4 = 2 * ga.NPOS;
      if (ga.planeF4 > kRegPos * kStagers) continue;
      ga.corr = NT <= 64 ? 1 : 0;
      ga.bf = L->opt_tc_bf ? 1 : 0;
      ga.planeRows = ga.bf ? ga.NPOS : ga.planeF4;   // (bf16x2: lbo = NPOS rows is the x1 -> x2 plane distance as well)
      ga.cbSlots = 2; ga.idRows = 2 * taps;
      ga.tapsPad = RoundUp(taps, 16);
      ga.idxT = (ga.tapsPad <= 32 && L->d_asmt_t.get() && L->asmt_t_mode == 0) ? 1 : 0;
      if (ga.idxT) ga.idRows = 2 * ga.tapsPad;      // [half][128 channels][tapsPad] bytes = 2 * tapsPad rows of 128
      ga.nChunks = CeilDiv(Cg, 8);
      ga.ntab = taps;
      ga.chunkFirst[0] = 0; ga.chunkCount[0] = taps;
      for (int t = 0; t < taps; t++) {
        KStep& ks = ga.tab[t];
        ks.bStart = (t / L->ksz) * PW + (t % L->ksz);
        ks.lbo = ga.NPOS;
        ks.idx0 = static_cast<short>(t); ks.idx1 = static_cast<short>(taps + t);
        ks.cb0 = 0; ks.cb1 = 1;
      }
      ga.K = L->K; ga.cbF4 = L->K; ga.nPB = 2;
      ga.nct = CeilDiv(Kg, 128);
      p.smem = static_cast<size_t>(MapSmem(ga).total);
      if (p.smem > smemMax) continue;
      p.a.CT = 128; p.a.nct = ga.nct; p.a.R = NT; p.a.nstrips = GT;   // (candidate de-duplication keys)
      const double ksteps = static_cast<double>(ga.nChunks) * taps;
      const double ctas0 = static_cast<double>(CeilDiv(N * IB, NT)) * G * ga.nct;
      // small batches: split the 8-channel chunks over CTAs (partial sums reduced by LaunchSplitReduce)
      for (int nsplit = 1; nsplit <= ga.nChunks; nsplit *= 2) {
        if (nsplit > 1 && ctas0 * nsplit > 1.5 * L->ctx->sm_count) break;
        ga.kPerSplit = CeilDiv(ga.nChunks, nsplit);
        ga.nsplit = CeilDiv(ga.nChunks, ga.kPerSplit);
        if (ga.nsplit != nsplit) continue;
        p.a.rgroups = nsplit;
        const double perCta = ksteps * 3.0 * (NT / 2.0) * 1.1 / nsplit + 120.0 * ksteps / GT / nsplit + 4000.0 + NT * 24.0 +
                              (nsplit > 1 ? 6000.0 : 0.0);
        cands->emplace_back(perCta * std::ceil(ctas0 * nsplit / L->ctx->sm_count), p);
      }
    }
  }
}
// dynamic shared-memory limit of the instantiations: raised once per device to the opt-in maximum (not per launch,
// which would make the limit follow whichever layer ran last -- fragile under graph capture / concurrent streams)
static int SetSmemLimitOnce(qcnn_ctx* ctx) {
  static bool done[64] = {false};
  if (ctx->device >= 0 && ctx->device < 64 && done[ctx->device]) return 0;
  const int lim = static_cast<int>(ctx->smem_optin ? ctx->smem_optin : 227 * 1024);
#define QCNN_SMEM_ATTR(...) QCNN_CUDA(cudaFuncSetAttribute(pq_gemm_tc_kernel<__VA_ARGS__>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim))
  QCNN_SMEM_ATTR(true, 128); QCNN_SMEM_ATTR(true, 64); QCNN_SMEM_ATTR(false, 128); QCNN_SMEM_ATTR(false, 64);
#undef QCNN_SMEM_ATTR
  if (ctx->device >= 0 && ctx->device < 64) done[ctx->device] = true;
  return 0;
}

static int LaunchKernel(const GemmArgs& a, unsigned blocks, size_t smem, cudaStream_t st) {
  QCNN_CHECK((a.NT == 128 || a.NT == 64) && a.corr == (a.NT == 64 ? 1 : 0) && a.GT >= 1 && a.GT <= kMaxGT,
             "pq_gemm_tc: no instantiation for NT=%d GT=%d", a.NT, a.GT);
  if (a.bf) {
    if (a.NT == 128) pq_gemm_tc_kernel<true, 128><<<blocks, kThreads, smem, st>>>(a);
    else pq_gemm_tc_kernel<true, 64><<<blocks, kThreads, smem, st>>>(a);
  } else {
    if (a.NT == 128) pq_gemm_tc_kernel<false, 128><<<blocks, kThreads, smem, st>>>(a);
    else pq_gemm_tc_kernel<false, 64><<<blocks, kThreads, smem, st>>>(a);
  }
  QCNN_CUDA(cudaGetLastError());
  return 0;
}

// bf16x2 form of the codebook, made once per layer: every aligned 4-float piece becomes {w1 (4 x bf16), w2 (4 x bf16)},
// stored [S][d/4][K] so that the K pieces a chunk stages are one contiguous run (bulk-copyable)
int BuildCtrdBf(qcnn_layer* L) {
  if (L->d % 4 != 0 || L->d_ctrd_bf.get()) return 0;
  const size_t n = static_cast<size_t>(L->S) * L->K * L->d / 4;
  QCNN_CUDA(L->d_ctrd_bf.Reserve(L->ctx, n * sizeof(uint4)));
  split_codebook_kernel<<<static_cast<unsigned>(std::min<size_t>((n + 255) / 256, 1024)), 256>>>(
      L->d_ctrd.as<const float4>(), L->d_ctrd_bf.as<uint4>(), L->S, L->K, L->d / 4);
  QCNN_CUDA(cudaGetLastError());
  QCNN_CUDA(cudaDeviceSynchronize());
  return 0;
}

int LaunchPqGemm(qcnn_layer* L, const ConvPlan& p, const float* src, int N, float* dst, int relu, cudaStream_t st) {
  GemmArgs a = p.g;
  a.src = src; a.dst = dst; a.ctrd = L->d_ctrd.as<float>(); a.asmt = L->d_asmt.as<uint8_t>(); a.bias = L->d_bias.as<float>();
  if (a.bf && L->d_ctrd_bf.get()) { a.ctrd = L->d_ctrd_bf.as<float>(); a.cbPre = 1; }
  a.asmtT = L->d_asmt_t.as<uint8_t>();
  a.bulkC = (a.mode != 2 && a.idxT && a.cbPre) ? 1 : 0;
  if (a.mode == 1 && !a.bulkC) a.idxT = 0;   // (3xTF32 operands: index rows by cp.async in tap-major order; the planned buffer is large enough)
  a.N = N; a.relu = a.nsplit > 1 ? 0 : relu;
  if (a.nsplit < 1) a.nsplit = 1;
  a.Hi = L->Hin; a.Wi = L->Win; a.Cin = L->Cin; a.Ho = L->Ho; a.Wo = L->Wo; a.Cout = L->Cout;
  a.ksz = L->ksz; a.pad = L->pad; a.stride = L->stride; a.G = L->grp; a.Cg = L->Cin / L->grp; a.Kg = L->Cout / L->grp;
  a.KgPad = RoundUp(a.Kg, 16); a.S = L->S; a.K = L->K; a.d = L->d;
  a.srcImg = static_cast<long long>(a.Hi) * a.Wi * a.Cin;
  if (L->src_nchw) { a.rowStride = a.Wi; a.colStride = 1; a.chStride = a.Hi * a.Wi; }
  else { a.rowStride = a.Wi * a.Cin; a.colStride = a.Cin; a.chStride = 1; }
  a.dstImg = static_cast<long long>(a.Ho) * a.Wo * a.Cout;
  const long long blocks = static_cast<long long>(CeilDiv(N * a.IB, a.NT)) * a.G * a.nct * a.nsplit;
  QCNN_CHECK(blocks <= 2147483647LL, "qcnn_conv_aprx_forward: batch too large for the tensor-core tiling");
  if (a.nsplit > 1) {
    QCNN_CUDA(L->d_partial.Reserve(L->ctx, sizeof(float) * static_cast<size_t>(a.nsplit) * N * a.dstImg, st));
    a.partial = L->d_partial.as<float>();
  }
  if (int rc = SetSmemLimitOnce(L->ctx)) return rc;
  if (int rc = LaunchKernel(a, static_cast<unsigned>(blocks), p.smem, st)) return rc;
  if (a.nsplit > 1)
    return LaunchSplitReduce(L->ctx, a.partial, dst, N * a.Ho * a.Wo, a.Cout, a.Cout, a.nsplit, relu, st);
  return 0;
}

// generic entry for callers that fill GemmArgs themselves (the fully-connected path in fc_aprx.cu)
size_t PqGemmSmemBytes(const GemmArgs& a) { return static_cast<size_t>(MapSmem(a).total); }
int LaunchPqGemmArgs(qcnn_ctx* ctx, const GemmArgs& a, long long blocks, cudaStream_t st) {
  QCNN_CHECK(blocks >= 1 && blocks <= 2147483647LL, "pq_gemm_tc: bad grid");
  if (int rc = SetSmemLimitOnce(ctx)) return rc;
  return LaunchKernel(a, static_cast<unsigned>(blocks), PqGemmSmemBytes(a), st);
}

}  // namespace qcnn
