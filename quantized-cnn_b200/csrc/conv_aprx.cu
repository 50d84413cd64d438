// Fused PQ convolution for sm_90a: per-subspace LUT (codebook x input inner products) built in shared memory
// and consumed by the uint8 gather-accumulate of the same CTA -- the LUT never touches HBM.
// Replaces CaffeEva::CalcFeatMap_ConvAprx + GetInPdMat (reference src/CaffeEva.cc:760-868, 1261-1296):
//     LUT[n][hi][wi][s][k] = sum_j src[n][hi][wi][g*Cg + s*d + j] * ctrd[s][k][j]
//     dst[n][ho][wo][g*Kg+c] = bias + sum_{kh,kw in bounds} sum_s LUT[n][ho*st-pad+kh][wo*st-pad+kw][s][asmt[kh][kw][s][g*Kg+c]]
//
// Design (SURVEY.md 7, hard parts 1/4): the binding resource is shared-memory gather bandwidth
// (32 four-byte lookups / clk / SM), so the gather is laid out to be bank-conflict free and issue-light:
//   * lane = output pixel, LUT stored TRANSPOSED as lut[k][position]; the codeword index of a (tap, s, channel)
//     is warp-uniform, so the 32 lanes read 32 consecutive floats (one wavefront, no conflicts);
//   * zero padding is realised by zero LUT columns (padded flat grid), so no per-lane bounds predicate exists in
//     the inner loop -- out-of-image taps add +0.0f, which is what the reference's tap skipping amounts to;
//   * a thread owns J positions x CPT channels (<= 64 accumulators, held as float2 pairs so two positions are
//     accumulated as a float2); per 4 channels it issues one 128-bit broadcast load of 4 pre-multiplied LUT row
//     offsets, then 4 x (1 IADD + J LDS + J FADD);
//   * the per-(s) assignment slice is staged in shared memory already multiplied by the LUT row pitch.
// Two kernel templates walk the LUT + gather steps; the kernel body owns the CTA decode, the LUT position -> pixel
// table, the gather and the epilogue:
//   conv_s1_kernel   stride 1 (conv2..conv5, sweep): a CTA owns (image, row strip, group, channel tile) and the
//                    flat padded grid of the strip; a step is a subspace; tap (kh,kw) is a constant shift kh*PW+kw.
//   conv_roll_kernel any stride (conv1: 11x11 / 4): a CTA walks the input rows of its strip once; a step is an
//                    (input row, subspace) pair, and each input row's LUT is used by the <= ceil(k/stride) output rows
//                    that see it, each owned by a different "row group" of warps; columns are de-interleaved by stride
//                    phase so that a tap again is a constant shift.
// The LUT stage of a step is a [K x d] x [d x positions] contraction, produced by one of two policies (template
// argument Lut) that own their shared-memory carve and operand staging:
//   FfmaLut   the FP32 pipe, a register-blocked mini-GEMM: 8 codewords x 4 positions per thread, float2 FFMA pairs,
//             codebook rows broadcast from shared memory, 128-bit LUT stores (fp32, ascending j: parity with the
//             reference's saxpy order up to FMA contraction -- SURVEY.md 7.5).  Any K, subspaces wider than 8 dims in
//             chunks of 8.
//   WgmmaLut  the tensor cores (K = 128, d <= 8): 3xTF32 wgmma, ~5e-6 from the FFMA stage.
#include "qcnn_internal.h"
#include "async_copy.h"
#include "wgmma.h"

#include <algorithm>
#include <cmath>
#include <cstdlib>

namespace {

using qcnn::CpAsync4;
using qcnn::CpAsyncCommit;
using qcnn::CpAsyncWaitAll;

// float2 arithmetic, element by element (sm_90 has no packed fp32 instructions)
__device__ __forceinline__ float2 Ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 Fadd2(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }

constexpr int kMaxThreads = 512;

// ------------------------------------------------------------------------------------------------------------
// Operand staging.  Everything the LUT stage of step i+1 needs from global memory (input pixels of the
// subspace's channels, its codebook rows, its assignment slice) is copied ASYNCHRONOUSLY (cp.async, no registers)
// into shared-memory staging buffers right before the gather of step i starts, and picked up after it ends,
// so no global-load latency is exposed between the two stages.
// ------------------------------------------------------------------------------------------------------------
// raw codebook chunk: cbN[k*8 + jj] <- ctrd[s][k][jc + jj]   (zero beyond the subspace's real dims)
__device__ __forceinline__ void FetchCodebook(float* __restrict__ cbN, const float* __restrict__ ctrd, int s, int K,
                                              int d, int jc, int nj, int tid, int T) {
  const float* base = ctrd + static_cast<size_t>(s) * K * d + jc;
  for (int e = tid; e < K * 8; e += T) {
    const int k = e >> 3, jj = e & 7;
    CpAsync4(cbN + e, base + (jj < nj ? k * d + jj : 0), jj < nj);
  }
}
// cb2[jj][k] = (c, c)
__device__ __forceinline__ void CommitCodebook(const float* __restrict__ cbN, float2* __restrict__ cb2, int K, int tid,
                                               int T) {
  for (int e = tid; e < K * 8; e += T) {
    const float c = cbN[e];
    cb2[(e & 7) * K + (e >> 3)] = make_float2(c, c);
  }
}

// raw assignment slice of (group, s, channel tile): idN[tap*CT + c] (bytes), fetched as 4-channel words
__device__ __forceinline__ void FetchOffsets(uint8_t* __restrict__ idN, const uint8_t* __restrict__ ap, int taps,
                                             int CT, int KgPad, int tid, int T) {
  const int wpt = CT >> 2;
  for (int w = tid; w < taps * wpt; w += T) {
    const int tap = w / wpt, c4 = w - tap * wpt;
    CpAsync4(idN + 4 * w, ap + static_cast<size_t>(tap) * KgPad + 4 * c4, true);
  }
}
// idx[tap][c] = asmt * (PP * 4): byte offset of LUT row k
__device__ __forceinline__ void CommitOffsets(const uint8_t* __restrict__ idN, uint32_t* __restrict__ idx, int taps,
                                              int CT, uint32_t rowBytes, int tid, int T) {
  const int wpt = CT >> 2;
  for (int w = tid; w < taps * wpt; w += T) {
    const uint32_t v = *reinterpret_cast<const uint32_t*>(idN + 4 * w);
    *reinterpret_cast<uint4*>(idx + 4 * w) = make_uint4((v & 0xFFu) * rowBytes, ((v >> 8) & 0xFFu) * rowBytes,
                                                        ((v >> 16) & 0xFFu) * rowBytes, (v >> 24) * rowBytes);
  }
}

// input pixels: xs[jj][pos] <- channel ch0+jj of the pixel behind LUT position pos; posoff[pos] = element offset
// of the pixel's channel 0 (or -1 for zero padding); chStride = 1 for NHWC, H*W for NCHW
__device__ __forceinline__ void FetchPixels(float* __restrict__ xs, const float* __restrict__ src,
                                            const int* __restrict__ posoff, int PP, int ch0, size_t chStride, int nj,
                                            int tid, int T) {
  for (int pos = tid; pos < PP; pos += T) {
    const int off = posoff[pos];
#pragma unroll
    for (int jj = 0; jj < 8; jj++) {
      const bool ok = off >= 0 && jj < nj;
      CpAsync4(xs + jj * PP + pos, src + (ok ? off + (ch0 + jj) * chStride : 0), ok);
    }
  }
}

// dims of subspace s that exist (reference CaffeEva.cc:1277)
__device__ __forceinline__ int SubspaceDims(const ConvArgs& a, int s) { return min(a.Cg - s * a.d, a.d); }
// ... of them in the first chunk of 8
__device__ __forceinline__ int FirstChunkDims(const ConvArgs& a, int s) { return max(0, min(8, SubspaceDims(a, s))); }

// ------------------------------------------------------------------------------------------------------------
// FFMA LUT stage: lut[k][p] (+)= sum_{jj<nj} cb[jj][k] * xs[jj][p], tile of 8 codewords x 4 positions per thread.
// Lanes walk the position tiles (128-bit LUT stores and x loads are conflict-free, codebook loads broadcast).
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void LutStep(float2 (&acc)[8][2], const float2* __restrict__ cb2, const float* __restrict__ xs,
                                        int K, int PP, int j, int k0, int p0) {
  const float4 xv = *reinterpret_cast<const float4*>(xs + j * PP + p0);
  const float2 x01 = make_float2(xv.x, xv.y), x23 = make_float2(xv.z, xv.w);
  const float4* cp = reinterpret_cast<const float4*>(cb2 + j * K + k0);
#pragma unroll
  for (int kk = 0; kk < 4; kk++) {
    const float4 cc = cp[kk];  // (c[2kk], c[2kk], c[2kk+1], c[2kk+1])
    const float2 ca = make_float2(cc.x, cc.y), cb = make_float2(cc.z, cc.w);
    acc[2 * kk][0] = Ffma2(ca, x01, acc[2 * kk][0]);
    acc[2 * kk][1] = Ffma2(ca, x23, acc[2 * kk][1]);
    acc[2 * kk + 1][0] = Ffma2(cb, x01, acc[2 * kk + 1][0]);
    acc[2 * kk + 1][1] = Ffma2(cb, x23, acc[2 * kk + 1][1]);
  }
}

__device__ __forceinline__ void BuildLut(float* __restrict__ lut, const float2* __restrict__ cb2,
                                         const float* __restrict__ xs, int K, int PP, int nj, bool first, int tid,
                                         int T) {
  const int npt = PP >> 2;
  const int ntiles = npt * (K >> 3);
  for (int t = tid; t < ntiles; t += T) {
    const int kt = t / npt;
    const int p0 = (t - kt * npt) << 2;
    const int k0 = kt << 3;
    float2 acc[8][2];
    if (first) {
#pragma unroll
      for (int k = 0; k < 8; k++) { acc[k][0] = make_float2(0.f, 0.f); acc[k][1] = make_float2(0.f, 0.f); }
    } else {
#pragma unroll
      for (int k = 0; k < 8; k++) {
        const float4 v = *reinterpret_cast<const float4*>(lut + (k0 + k) * PP + p0);
        acc[k][0] = make_float2(v.x, v.y);
        acc[k][1] = make_float2(v.z, v.w);
      }
    }
    if (nj == 8) {  // two steps in flight: enough ILP to cover the LDS latency without blowing the register file
#pragma unroll 2
      for (int j = 0; j < 8; j++) LutStep(acc, cb2, xs, K, PP, j, k0, p0);
    } else {
#pragma unroll 1
      for (int j = 0; j < nj; j++) LutStep(acc, cb2, xs, K, PP, j, k0, p0);
    }
#pragma unroll
    for (int k = 0; k < 8; k++)
      *reinterpret_cast<float4*>(lut + (k0 + k) * PP + p0) = make_float4(acc[k][0].x, acc[k][0].y, acc[k][1].x, acc[k][1].y);
  }
}

// ------------------------------------------------------------------------------------------------------------
// wgmma LUT stage (K = 128 codewords, subspaces of <= 8 dims)
//
// The LUT of a step is the dense contraction  LUT[k][p] = sum_j ctrd[s][k][j] * x[p][j]  = C (128 x 8) * X^T (8 x N).
// Per 32 LUT columns a warpgroup issues three wgmma.mma_async of tf32 operands (M = 64 codewords, N = 32, K = 8) -- the
// 3xTF32 split  C_hi*X_hi + C_hi*X_lo + C_lo*X_hi  keeps fp32-level accuracy -- with both operands in shared memory and
// the accumulator in its registers, which it then writes to lut[k][p].  The first two warpgroups of the CTA (the first
// one alone in CTAs of fewer than eight warps) produce the LUT of a step at the stage boundary; all warps gather.
// Operands reach the canonical K-major unswizzled tiles through cp.async (raw) + a hi/lo split pass.
// ------------------------------------------------------------------------------------------------------------
// canonical K-major operand tile without swizzle (tf32): rows in groups of 8, per group K-chunk 0 (8 rows x 16 B) then
// K-chunk 1; element (row r, k) -> float index below.  Descriptor: LBO = 128 B (K chunks), SBO = 256 B (row groups).
__device__ __forceinline__ int TileIdx(int r, int k) { return (r >> 3) * 64 + (k >> 2) * 32 + (r & 7) * 4 + (k & 3); }
// LUT[128][NM] = A (128 codewords x 8) * B^T (NM positions x 8) as 3xTF32, written to lut (row pitch PP floats).
// Called by all threads of warps 0 .. 4 nwg - 1 (nwg = 1 or 2 warpgroups); the tiles are published to the async proxy.
__device__ __forceinline__ void LutMma(const float* aHi, const float* aLo, const float* bHi, const float* bLo, float* lut,
                                       int PP, int NM, int warp, int lane, int nwg) {
  const int wg = warp >> 2;
  for (int half = wg; half < 2; half += nwg) {          // codewords [64 half, +64)
    const uint64_t dAh = qcnn::WgmmaDesc(qcnn::SmemU32(aHi + half * 512), 128, 256);
    const uint64_t dAl = qcnn::WgmmaDesc(qcnn::SmemU32(aLo + half * 512), 128, 256);
    const int r0 = half * 64 + (warp & 3) * 16 + (lane >> 2);
    for (int c = 0; c < (NM >> 5); c++) {               // 32 LUT columns = 4 row groups of the B tile
      const uint64_t dBh = qcnn::WgmmaDesc(qcnn::SmemU32(bHi + c * 256), 128, 256);
      const uint64_t dBl = qcnn::WgmmaDesc(qcnn::SmemU32(bLo + c * 256), 128, 256);
      float d[16];
#pragma unroll
      for (int i = 0; i < 16; i++) d[i] = 0.0f;
      qcnn::WgmmaFence();
      qcnn::Wgmma<32>::Tf32SS(d, dAh, dBh);
      qcnn::Wgmma<32>::Tf32SS(d, dAh, dBl);
      qcnn::Wgmma<32>::Tf32SS(d, dAl, dBh);
      qcnn::WgmmaCommit();
      qcnn::WgmmaWaitAll();
      // fragment: d[4 i + {0, 1}] = row r0, columns 8 i + 2 (lane % 4) + {0, 1}; d[4 i + {2, 3}] = row r0 + 8
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int col = c * 32 + 8 * i + 2 * (lane & 3);
        *reinterpret_cast<float2*>(lut + r0 * PP + col) = make_float2(d[4 * i], d[4 * i + 1]);
        *reinterpret_cast<float2*>(lut + (r0 + 8) * PP + col) = make_float2(d[4 * i + 2], d[4 * i + 3]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// LUT stage policies.  A kernel walks steps 0 .. steps-1 as
//     Prologue                                  operands of step 0 (wgmma: also step 1) in flight
//     per step:  cp.async.wait_all; __syncthreads()   (A) staged operands have landed; the previous gather is done
//                Produce(step)                  lut + idx of the step, complete for every thread on return
//                Prefetch(step)                 operands of later steps fly in while this one is gathered
//                gather
// A step reads input LutSrc::src (the strip of the image, or one input row, of the CTA's group) and subspace
// LutSrc::s; `at(i)` gives those of step i.  idx holds the LUT row offsets of the step's assignment slice; the rolling-row
// kernel with one subspace keeps the slice of step 0 (commitOffsets / fetchOffsets false).
// ------------------------------------------------------------------------------------------------------------
struct LutSrc {
  const float* src;
  int s;
};

// What both policies take from the kernel
struct LutBase {
  const ConvArgs& a;
  size_t chStride;        // source element stride between channels
  const uint8_t* asmtG;   // assignments of the CTA's group and channel tile, subspace 0
  int taps, tid, T;
  uint32_t rowBytes;      // LUT row pitch in bytes
  __device__ LutBase(const ConvArgs& a_, size_t chStride_, const uint8_t* asmtG_, int taps_)
      : a(a_), chStride(chStride_), asmtG(asmtG_), taps(taps_), tid(threadIdx.x), T(blockDim.x),
        rowBytes(static_cast<uint32_t>(a_.PP) * 4u) {}
};

struct FfmaLut : LutBase {
  float* lut;      // [K][PP]
  uint32_t* idx;   // [taps][CT]   LUT row byte offsets of the current step
  float2* cb2;     // [8][K]       duplicated codebook chunk of the current step
  float* xs;       // [2][8][PP]   input pixels, double-buffered (even / odd steps)
  int* posoff;     // [PP]         LUT position -> element offset of its pixel (-1: zero padding), written by the kernel
  float* cbN;      // [K*8]        raw codebook chunk of the next step (cp.async target)
  uint8_t* idN;    // [taps*CT]    raw assignment slice of the next step (cp.async target)
  int npos;        // entries of posoff

  struct Map { int idx, cb2, xs, posoff, cbN, idN, bytes; };   // byte offsets; bytes = dynamic shared memory of a CTA
  static __host__ __device__ Map MapSmem(int K, int PP, int NM, int taps, int CT) {
    Map m;
    int o = 4 * K * PP;                         // lut
    m.idx = o;    o += 4 * taps * CT;
    m.cb2 = o;    o += 8 * 8 * K;
    m.xs = o;     o += 2 * 4 * 8 * PP;
    m.posoff = o; o += 4 * PP;
    m.cbN = o;    o += 4 * 8 * K;
    m.idN = o;    o += (taps * CT + 15) & ~15;
    m.bytes = o;
    return m;
  }

  __device__ FfmaLut(unsigned char* smem, const LutBase& b) : LutBase(b), npos(b.a.PP) {
    const Map m = MapSmem(a.K, a.PP, a.NM, taps, a.CT);
    lut = reinterpret_cast<float*>(smem);
    idx = reinterpret_cast<uint32_t*>(smem + m.idx);
    cb2 = reinterpret_cast<float2*>(smem + m.cb2);
    xs = reinterpret_cast<float*>(smem + m.xs);
    posoff = reinterpret_cast<int*>(smem + m.posoff);
    cbN = reinterpret_cast<float*>(smem + m.cbN);
    idN = smem + m.idN;
  }

  __device__ float* Xs(int step) const { return xs + (step & 1) * 8 * a.PP; }

  template <class At>
  __device__ void Prologue(At at, int) {
    const LutSrc in = at(0);
    const int nj0 = FirstChunkDims(a, in.s);
    FetchCodebook(cbN, a.ctrd, in.s, a.K, a.d, 0, nj0, tid, T);
    FetchOffsets(idN, asmtG, taps, a.CT, a.KgPad, tid, T);
    FetchPixels(Xs(0), in.src, posoff, a.PP, in.s * a.d, chStride, nj0, tid, T);
    CpAsyncCommit();
  }

  __device__ void Produce(int step, int, LutSrc in, bool commitOffsets) {
    const int dsel = SubspaceDims(a, in.s);
    float* x = Xs(step);
    CommitCodebook(cbN, cb2, a.K, tid, T);
    if (commitOffsets) CommitOffsets(idN, idx, taps, a.CT, rowBytes, tid, T);
    __syncthreads();  // (B)
    BuildLut(lut, cb2, x, a.K, a.PP, max(0, min(8, dsel)), true, tid, T);
    // the rare further chunks of subspaces wider than 8 dims, staged with exposed latency
    for (int jc = 8; jc < dsel; jc += 8) {
      const int nj = min(8, dsel - jc);
      __syncthreads();
      FetchCodebook(cbN, a.ctrd, in.s, a.K, a.d, jc, nj, tid, T);
      FetchPixels(x, in.src, posoff, a.PP, in.s * a.d + jc, chStride, nj, tid, T);
      CpAsyncCommit();
      CpAsyncWaitAll();
      __syncthreads();
      CommitCodebook(cbN, cb2, a.K, tid, T);
      __syncthreads();
      BuildLut(lut, cb2, x, a.K, a.PP, nj, false, tid, T);
    }
    __syncthreads();  // (C) lut complete; cbN / idN / the other xs buffer are free
  }

  // operands of step + 1 (= next)
  template <class At>
  __device__ void Prefetch(int step, int steps, LutSrc next, At, bool fetchOffsets) {
    if (step + 1 < steps) {
      const int njn = FirstChunkDims(a, next.s);
      FetchCodebook(cbN, a.ctrd, next.s, a.K, a.d, 0, njn, tid, T);
      if (fetchOffsets) FetchOffsets(idN, asmtG + static_cast<size_t>(next.s) * taps * a.KgPad, taps, a.CT, a.KgPad, tid, T);
      FetchPixels(Xs(step + 1), next.src, posoff, a.PP, next.s * a.d, chStride, njn, tid, T);
      CpAsyncCommit();
    }
  }
};

struct WgmmaLut : LutBase {
  float* lut;       // [128][PP]
  uint32_t* idx;    // [taps][CT]
  float* aHi;       // [128 x 8] canonical
  float* aLo;
  float* bHi;       // [NM x 8] canonical
  float* bLo;
  float* xr;        // [NM][8] raw pixels of a later step (cp.async target)
  float* cr;        // [128][8] raw codebook of a later step
  int* posoff;      // [NM]
  uint8_t* idN;     // [taps*CT] raw assignment slice of the next step
  int npos;         // entries of posoff: NM
  int warp, lane;
  int nwg;          // warpgroups that run the LUT MMAs

  struct Map { int idx, aHi, aLo, bHi, bLo, xr, cr, posoff, idN, bytes; };
  static __host__ __device__ Map MapSmem(int, int PP, int NM, int taps, int CT) {
    Map m;
    int o = 4 * 128 * PP;                       // lut
    m.idx = o;    o += 4 * taps * CT;
    m.aHi = o;    o += 4 * 1024;
    m.aLo = o;    o += 4 * 1024;
    m.bHi = o;    o += 4 * 8 * NM;
    m.bLo = o;    o += 4 * 8 * NM;
    m.xr = o;     o += 4 * 8 * NM;
    m.cr = o;     o += 4 * 1024;
    m.posoff = o; o += 4 * (NM + 8);
    m.idN = o;    o += (taps * CT + 15) & ~15;
    m.bytes = o;
    return m;
  }

  __device__ WgmmaLut(unsigned char* smem, const LutBase& b) : LutBase(b), npos(b.a.NM) {
    const Map m = MapSmem(a.K, a.PP, a.NM, taps, a.CT);
    lut = reinterpret_cast<float*>(smem);
    idx = reinterpret_cast<uint32_t*>(smem + m.idx);
    aHi = reinterpret_cast<float*>(smem + m.aHi);
    aLo = reinterpret_cast<float*>(smem + m.aLo);
    bHi = reinterpret_cast<float*>(smem + m.bHi);
    bLo = reinterpret_cast<float*>(smem + m.bLo);
    xr = reinterpret_cast<float*>(smem + m.xr);
    cr = reinterpret_cast<float*>(smem + m.cr);
    posoff = reinterpret_cast<int*>(smem + m.posoff);
    idN = smem + m.idN;
    warp = tid >> 5;
    lane = tid & 31;
    nwg = (T >> 5) >= 8 ? 2 : 1;
  }

  // raw operands of a step: pixels [NM][8] and codebook [128][8], zero beyond the subspace's real dims
  __device__ void FetchRaw(LutSrc in) {
    const int nj = FirstChunkDims(a, in.s);
    const float* cg = a.ctrd + static_cast<size_t>(in.s) * 128 * a.d;
    for (int e = tid; e < 1024; e += T) {
      const int k = e >> 3, jj = e & 7;
      CpAsync4(cr + e, cg + (jj < nj ? k * a.d + jj : 0), jj < nj);
    }
    const int ch0 = in.s * a.d;
    for (int e = tid; e < a.NM * 8; e += T) {
      const int pos = e >> 3, jj = e & 7;
      const int off = posoff[pos];
      const bool ok = off >= 0 && jj < nj;
      CpAsync4(xr + e, in.src + (ok ? off + (ch0 + jj) * chStride : 0), ok);
    }
  }
  // raw -> hi/lo canonical operand tiles (generic-proxy writes, published to the async proxy by the caller's fence)
  __device__ void SplitOperands() {
    for (int e = tid; e < 1024; e += T) {
      float hi, lo;
      qcnn::SplitTf32(cr[e], hi, lo);
      const int i = TileIdx(e >> 3, e & 7);
      aHi[i] = hi;
      aLo[i] = lo;
    }
    for (int e = tid; e < a.NM * 8; e += T) {
      float hi, lo;
      qcnn::SplitTf32(xr[e], hi, lo);
      const int i = TileIdx(e >> 3, e & 7);
      bHi[i] = hi;
      bLo[i] = lo;
    }
  }

  // operand tiles of step 0 published, raw operands of step 1 + assignment slice 0 in flight
  template <class At>
  __device__ void Prologue(At at, int steps) {
    FetchRaw(at(0));
    CpAsyncCommit();
    CpAsyncWaitAll();
    __syncthreads();
    SplitOperands();
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (steps > 1) FetchRaw(at(1));
    FetchOffsets(idN, asmtG, taps, a.CT, a.KgPad, tid, T);
    CpAsyncCommit();
  }

  // tensor cores -> accumulator fragments -> lut; the operand tiles of step + 1 are split from the raw operands
  __device__ void Produce(int step, int steps, LutSrc, bool commitOffsets) {
    if (warp < 4 * nwg) LutMma(aHi, aLo, bHi, bLo, lut, a.PP, a.NM, warp, lane, nwg);
    if (commitOffsets) CommitOffsets(idN, idx, taps, a.CT, rowBytes, tid, T);
    if (step + 1 < steps) {
      __syncthreads();  // the MMAs of this step have read the operand tiles
      SplitOperands();
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();  // (B) lut + idx ready, operand tiles of step + 1 published
  }

  // raw operands of step + 2, assignment slice of step + 1 (= next)
  template <class At>
  __device__ void Prefetch(int step, int steps, LutSrc next, At at, bool fetchOffsets) {
    if (step + 1 < steps) {
      if (step + 2 < steps) FetchRaw(at(step + 2));
      if (fetchOffsets) FetchOffsets(idN, asmtG + static_cast<size_t>(next.s) * taps * a.KgPad, taps, a.CT, a.KgPad, tid, T);
      CpAsyncCommit();
    }
  }
};

// ------------------------------------------------------------------------------------------------------------
// gather stage
// ------------------------------------------------------------------------------------------------------------
// Accumulators of one thread: J positions x CPT channels.  For even J two positions share a float2 so that one
// float2 add retires two lookups.
template <int CPT, int J>
struct Acc {
  static constexpr int JP = (J % 2 == 0) ? J / 2 : J;
  static constexpr bool kPaired = (J % 2 == 0);
  float2 v[JP][CPT];  // paired: (pos 2jp, pos 2jp+1); unpaired: .x only

  __device__ __forceinline__ void Fill(const float (&b)[CPT]) {
#pragma unroll
    for (int jp = 0; jp < JP; jp++)
#pragma unroll
      for (int c = 0; c < CPT; c++) v[jp][c] = make_float2(b[c], b[c]);
  }
  __device__ __forceinline__ float Get(int j, int c) const {
    if (kPaired) return (j & 1) ? v[j >> 1][c].y : v[j >> 1][c].x;
    return v[j][c].x;
  }
};

// one tap: acc[j][c] += lut[idx[c]][q_j + shift]; `base` = byte address of lut[0][q_0 + shift]; positions of a
// thread are 32 apart (j * 128 bytes), so the J loads of a channel share one address register.
template <int CPT, int J>
__device__ __forceinline__ void GatherTap(Acc<CPT, J>& acc, const char* base, const uint32_t* __restrict__ ip) {
#pragma unroll
  for (int c4 = 0; c4 < CPT; c4 += 4) {
    const uint4 o = *reinterpret_cast<const uint4*>(ip + c4);
    const char* b[4] = {base + o.x, base + o.y, base + o.z, base + o.w};
#pragma unroll
    for (int u = 0; u < 4; u++) {
      if (Acc<CPT, J>::kPaired) {
#pragma unroll
        for (int jp = 0; jp < J / 2; jp++) {
          const float2 val = make_float2(*reinterpret_cast<const float*>(b[u] + (2 * jp) * 128),
                                         *reinterpret_cast<const float*>(b[u] + (2 * jp + 1) * 128));
          acc.v[jp][c4 + u] = Fadd2(acc.v[jp][c4 + u], val);
        }
      } else {
#pragma unroll
        for (int j = 0; j < J; j++) acc.v[j][c4 + u].x += *reinterpret_cast<const float*>(b[u] + j * 128);
      }
    }
  }
}

template <int CPT, int J>
__device__ __forceinline__ void StoreChannels(float* __restrict__ out, const Acc<CPT, J>& acc, int j, int relu) {
#pragma unroll
  for (int c = 0; c < CPT; c += 4) {
    float4 o = make_float4(acc.Get(j, c), acc.Get(j, c + 1), acc.Get(j, c + 2), acc.Get(j, c + 3));
    if (relu) {
      o.x = fmaxf(o.x, 0.0f); o.y = fmaxf(o.y, 0.0f); o.z = fmaxf(o.z, 0.0f); o.w = fmaxf(o.w, 0.0f);
    }
    *reinterpret_cast<float4*>(out + c) = o;
  }
}

// CTA coordinates of the LUT + gather and direct kernels: blockIdx.x = (group, channel tile, strip), strip fastest;
// blockIdx.y = image
struct CtaTile {
  int strip, ct, g, n;
  __device__ explicit CtaTile(const ConvArgs& a) {
    int b = blockIdx.x;
    strip = b % a.nstrips; b /= a.nstrips;
    ct = b % a.nct;
    g = b / a.nct;
    n = blockIdx.y;
  }
};

// ------------------------------------------------------------------------------------------------------------
// stride-1 kernel
// ------------------------------------------------------------------------------------------------------------
// MAXT: launch bound (256 / 384 / 512 threads) -> register cap 255 / 168 / 128, so small CTAs never spill
template <class Lut, int CPT, int J, int MAXT>
__global__ void __launch_bounds__(MAXT, 1) conv_s1_kernel(const ConvArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int taps = a.ksz * a.ksz;
  const int tid = threadIdx.x, T = blockDim.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int pw = warp % a.pwarps, cw = warp / a.pwarps;
  const CtaTile t(a);
  // strip = row strip x ncol + column tile.  Whole rows (ncol = 1) share their padding: the right padding of a row is
  // the left padding of the next (pitch Win + pad, positions shifted by pad).  A column tile (rows wider than a LUT
  // holds) has pitch CW + ksz - 1 with its own left halo.
  const int r0 = (t.strip / a.ncol) * a.R;   // first output row of the strip
  const int c0 = (t.strip % a.ncol) * a.CW;  // first output column of the tile
  const int shift = a.ncol > 1 ? 0 : a.pad, wi0 = a.ncol > 1 ? c0 - a.pad : 0;
  const int Wt = a.ncol > 1 ? min(a.CW, a.Wo - c0) : a.Wo;   // output columns of the tile
  const int hin0 = r0 - a.pad;             // input row held at ri = 0
  const int q0 = pw * 32 * J + lane;       // first flat position of this thread (others at +32 j)
  const int cbase = t.ct * a.CT + cw * CPT;  // first channel (within the group) of this thread
  const float* src = a.src + static_cast<size_t>(t.n) * a.Hi * a.Wi * a.Cin + t.g * a.Cg;
  Lut lut(smem, LutBase(a, 1, a.asmt + static_cast<size_t>(t.g) * a.S * taps * a.KgPad + t.ct * a.CT, taps));

  // LUT position -> source pixel (NHWC element offset within this image/group), -1 = zero padding
  for (int pos = tid; pos < lut.npos; pos += T) {
    int off = -1;
    const int pp = pos - shift;
    if (pp >= 0) {
      const int ri = pp / a.PW, wi = wi0 + pp - ri * a.PW;
      const int hi = hin0 + ri;
      if (ri < a.RI && wi >= 0 && wi < a.Wi && hi >= 0 && hi < a.Hi) off = (hi * a.Wi + wi) * a.Cin;
    }
    lut.posoff[pos] = off;
  }

  Acc<CPT, J> acc;
  {
    float bv[CPT];
#pragma unroll
    for (int c = 0; c < CPT; c++) bv[c] = __ldg(a.bias + t.g * a.Kg + cbase + c);
    acc.Fill(bv);
  }
  __syncthreads();  // posoff visible

  const auto at = [&](int s) { return LutSrc{src, s}; };   // step = subspace
  lut.Prologue(at, a.S);
  for (int s = 0; s < a.S; s++) {
    CpAsyncWaitAll();
    __syncthreads();  // (A)
    lut.Produce(s, a.S, at(s), true);
    lut.Prefetch(s, a.S, at(s + 1), at, true);
    const char* lutq = reinterpret_cast<const char*>(lut.lut) + q0 * 4;
    const uint32_t* ip = lut.idx + cw * CPT;
    for (int kh = 0; kh < a.ksz; kh++) {
      for (int kw = 0; kw < a.ksz; kw++) {
        GatherTap<CPT, J>(acc, lutq + (kh * a.PW + kw) * 4, ip);
        ip += a.CT;
      }
    }
  }

#pragma unroll
  for (int j = 0; j < J; j++) {
    const int q = q0 + 32 * j;
    const int r = q / a.PW, wo = q - r * a.PW;
    const int ho = r0 + r;
    if (r < a.R && wo < Wt && ho < a.Ho) {
      float* out = a.dst + ((static_cast<size_t>(t.n) * a.Ho + ho) * a.Wo + c0 + wo) * a.Cout + t.g * a.Kg + cbase;
      StoreChannels<CPT, J>(out, acc, j, a.relu);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// rolling-row kernel (any stride)
// ------------------------------------------------------------------------------------------------------------
template <class Lut, int CPT, int J, int MAXT>
__global__ void __launch_bounds__(MAXT, 1) conv_roll_kernel(const ConvArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int taps = a.ksz * a.ksz;
  const int tid = threadIdx.x, T = blockDim.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int rg = warp % a.rgroups;
  const int rest = warp / a.rgroups;
  const int pw = rest % a.pwarps, cw = rest / a.pwarps;
  const CtaTile t(a);
  const int ho0 = t.strip * a.R;
  const int ho_end = min(a.Ho, ho0 + a.R);
  const int PH = a.PW;
  const int wo0 = pw * 32 * J + lane;
  const int cbase = t.ct * a.CT + cw * CPT;
  // source addressing: pixel (hi, wi), channel ch  ->  base + hi*rowStride + wi*pixStride + ch*chStride
  const size_t chStride = a.src_nchw ? static_cast<size_t>(a.Hi) * a.Wi : 1;
  const int pixStride = a.src_nchw ? 1 : a.Cin;
  const size_t rowStride = static_cast<size_t>(a.Wi) * pixStride;
  const float* src = a.src + static_cast<size_t>(t.n) * a.Hi * a.Wi * a.Cin + static_cast<size_t>(t.g) * a.Cg * chStride;
  Lut lut(smem, LutBase(a, chStride, a.asmt + static_cast<size_t>(t.g) * a.S * taps * a.KgPad + t.ct * a.CT, taps));

  // LUT position (phase-major de-interleaved column) -> element offset of the pixel inside its input row
  for (int pos = tid; pos < lut.npos; pos += T) {
    const int phase = pos / PH, i = pos - phase * PH;
    const int wi = i * a.stride + phase - a.pad;
    lut.posoff[pos] = (phase < a.stride && wi >= 0 && wi < a.Wi) ? wi * pixStride : -1;
  }

  float bias[CPT];
#pragma unroll
  for (int c = 0; c < CPT; c++) bias[c] = __ldg(a.bias + t.g * a.Kg + cbase + c);
  Acc<CPT, J> acc;
  acc.Fill(bias);
  int ho_cur = ho0 + rg;  // output row this warp is accumulating
  __syncthreads();        // posoff visible

  const int hi_begin = ho0 * a.stride - a.pad;
  const int hi_end = (ho_end - 1) * a.stride - a.pad + a.ksz;
  const int hi_lo = max(hi_begin, 0), hi_hi = min(hi_end, a.Hi);  // rows outside the image contribute nothing
  const int steps = (hi_hi - hi_lo) * a.S;                         // (input row, subspace) pairs, row-major
  const auto at = [&](int step) { return LutSrc{src + (hi_lo + step / a.S) * rowStride, step % a.S}; };
  // the current output row has seen its last input row: store it and move on to the row group's next one
  const auto emitRow = [&]() {
#pragma unroll
    for (int j = 0; j < J; j++) {
      const int wo = wo0 + 32 * j;
      if (wo < a.Wo) {
        float* out = a.dst + ((static_cast<size_t>(t.n) * a.Ho + ho_cur) * a.Wo + wo) * a.Cout + t.g * a.Kg + cbase;
        StoreChannels<CPT, J>(out, acc, j, a.relu);
      }
    }
    acc.Fill(bias);
    ho_cur += a.rgroups;
  };

  if (steps > 0) lut.Prologue(at, steps);
  int hi = hi_lo, s = 0;
  for (int it = 0; it < steps; it++) {
    const int kh = hi + a.pad - ho_cur * a.stride;  // warp-uniform
    const bool active = ho_cur < ho_end && kh >= 0 && kh < a.ksz;
    CpAsyncWaitAll();
    __syncthreads();  // (A)
    lut.Produce(it, steps, LutSrc{src + hi * rowStride, s}, a.S > 1 || it == 0);
    int hin = hi, sn = s + 1;  // next (row, subspace)
    if (sn == a.S) { sn = 0; hin = hi + 1; }
    lut.Prefetch(it, steps, LutSrc{src + hin * rowStride, sn}, at, a.S > 1);
    if (active) {
      const char* lutq = reinterpret_cast<const char*>(lut.lut) + wo0 * 4;
      const uint32_t* ip = lut.idx + (kh * a.ksz) * a.CT + cw * CPT;
      for (int kw = 0; kw < a.ksz; kw++) {
        const int phase = kw % a.stride, sh = kw / a.stride;
        GatherTap<CPT, J>(acc, lutq + (phase * PH + sh) * 4, ip);
        ip += a.CT;
      }
    }
    if (s == a.S - 1 && ho_cur < ho_end && kh == a.ksz - 1) emitRow();
    hi = hin; s = sn;
  }
  // output rows whose window ends below the image (padding rows were skipped above)
  for (int h = max(hi_hi, hi_begin); h < hi_end; h++) {
    const int kh = h + a.pad - ho_cur * a.stride;
    if (ho_cur < ho_end && kh == a.ksz - 1) emitRow();
  }
}

// ------------------------------------------------------------------------------------------------------------
// single-subspace, narrow-subspace layers (AlexNet conv1: S = 1, 3 of the 8 codebook dims exist).
// With S = 1 every LUT entry  LUT[pixel][k] = <x_pixel, c_k>  would be read only ~ (k/stride)^2 * Cout / K ~ 5 times,
// so tabulating costs more than it saves.  This kernel keeps the layer in PQ form (codebook + uint8 assignments) but
// evaluates the inner product where it is consumed:  acc[p][c] += <x[p + tap], c_{asmt[tap][c]}>  -- the same sum,
// the codeword (not the partial product) is what the warp-uniform assignment index gathers (128-bit broadcast load).
// A thread owns 2 output rows x 2 columns x CPT channels (float2 pairs); the strip's input rows live in shared
// memory, de-interleaved by stride phase, so a tap is a constant shift and there are no barriers after the tile load.
// ------------------------------------------------------------------------------------------------------------
template <int CPT, int NJ, int ROWS>
__global__ void __launch_bounds__(384, 1) conv_direct_kernel(const ConvArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int taps = a.ksz * a.ksz;
  const int PH = a.PW, PITCH = a.PP;                // phase length, padded row pitch (floats)
  const int rowsIn = (a.R - 1) * a.stride + a.ksz;  // input rows of the strip
  float* xin = reinterpret_cast<float*>(smem);                                   // [rowsIn][NJ][PITCH]
  float2* cb = reinterpret_cast<float2*>(xin + static_cast<size_t>(rowsIn) * NJ * PITCH + 64);  // [K][4] (c,c) pairs
  uint32_t* idxa = reinterpret_cast<uint32_t*>(cb + a.K * 4);                    // [taps][CT] smem address of cb[k]

  const int tid = threadIdx.x, T = blockDim.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int cw = warp % a.cwarps, rw = warp / a.cwarps;   // channel warp, row-pair warp
  int b = blockIdx.x;
  const int strip = b % a.nstrips; b /= a.nstrips;
  const int ct = b % a.nct;
  const int g = b / a.nct;
  const int n = blockIdx.y;
  const int ho0 = strip * a.R;
  const int ho_end = min(a.Ho, ho0 + a.R);
  const int cbase = ct * a.CT + cw * CPT;
  const size_t chStride = a.src_nchw ? static_cast<size_t>(a.Hi) * a.Wi : 1;
  const int pixStride = a.src_nchw ? 1 : a.Cin;
  const size_t rowStride = static_cast<size_t>(a.Wi) * pixStride;
  const float* src = a.src + static_cast<size_t>(n) * a.Hi * a.Wi * a.Cin + static_cast<size_t>(g) * a.Cg * chStride;
  const int nj = min(NJ, min(a.Cg, a.d));
  const int hi0 = ho0 * a.stride - a.pad;

  // input tile: element (row r, dim jj, column position) <- pixel (hi0 + r, wi), zero outside the image
  for (int e = tid; e < rowsIn * NJ * PITCH; e += T) {
    const int pos = e % PITCH;
    const int rj = e / PITCH;
    const int jj = rj % NJ, r = rj / NJ;
    const int phase = pos / PH, i = pos - phase * PH;
    const int wi = i * a.stride + phase - a.pad;
    const int hi = hi0 + r;
    const bool ok = phase < a.stride && wi >= 0 && wi < a.Wi && hi >= 0 && hi < a.Hi && jj < nj;
    CpAsync4(xin + e, src + (ok ? hi * rowStride + static_cast<size_t>(wi) * pixStride + jj * chStride : 0), ok);
  }
  CpAsyncCommit();
  for (int e = tid; e < a.K * 4; e += T) {
    const int k = e >> 2, jj = e & 3;
    const float c = (jj < nj) ? __ldg(a.ctrd + static_cast<size_t>(k) * a.d + jj) : 0.0f;
    cb[e] = make_float2(c, c);
  }
  {
    const uint8_t* ap = a.asmt + static_cast<size_t>(g) * taps * a.KgPad + ct * a.CT;  // S == 1
    const uint32_t cbBase = static_cast<uint32_t>(__cvta_generic_to_shared(cb));
    for (int e = tid; e < taps * a.CT; e += T) {
      const int tap = e / a.CT, c = e - tap * a.CT;
      idxa[e] = cbBase + static_cast<uint32_t>(__ldg(ap + tap * a.KgPad + c)) * 32u;
    }
  }
  float bias[CPT];
#pragma unroll
  for (int c = 0; c < CPT; c++) bias[c] = __ldg(a.bias + g * a.Kg + cbase + c);
  CpAsyncWaitAll();
  __syncthreads();

  const int groups = (ho_end - ho0 + ROWS - 1) / ROWS;
  for (int gr = rw; gr < groups; gr += a.rgroups) {
    const int ra = ROWS * gr;                    // strip-local output rows ra .. ra + ROWS - 1
    float2 acc[ROWS][CPT];
#pragma unroll
    for (int r = 0; r < ROWS; r++)
#pragma unroll
      for (int c = 0; c < CPT; c++) acc[r][c] = make_float2(bias[c], bias[c]);
    int rowOff[ROWS];                            // rows past the strip re-read row ra (results discarded)
#pragma unroll
    for (int r = 0; r < ROWS; r++) rowOff[r] = (ho0 + ra + r < ho_end ? r * a.stride : 0) * NJ * PITCH;
    for (int kh = 0; kh < a.ksz; kh++) {
      const float* rowA = xin + static_cast<size_t>(ra * a.stride + kh) * NJ * PITCH + lane;
      const uint32_t* ip = idxa + (kh * a.ksz) * a.CT + cw * CPT;
      for (int kw = 0; kw < a.ksz; kw++) {
        const int shift = (kw % a.stride) * PH + kw / a.stride;
        float2 x[ROWS][NJ];
#pragma unroll
        for (int r = 0; r < ROWS; r++)
#pragma unroll
          for (int jj = 0; jj < NJ; jj++)
            x[r][jj] = make_float2(rowA[rowOff[r] + jj * PITCH + shift], rowA[rowOff[r] + jj * PITCH + shift + 32]);
#pragma unroll
        for (int c4 = 0; c4 < CPT; c4 += 4) {
          const uint4 ad = *reinterpret_cast<const uint4*>(ip + c4);
          const uint32_t adr[4] = {ad.x, ad.y, ad.z, ad.w};
#pragma unroll
          for (int u = 0; u < 4; u++) {
            float4 c01;
            float2 c2 = make_float2(0.f, 0.f), c3 = make_float2(0.f, 0.f);
            asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(c01.x), "=f"(c01.y), "=f"(c01.z), "=f"(c01.w) : "r"(adr[u]));
            if (NJ > 2) {
              if (NJ > 3) asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4+16];" : "=f"(c2.x), "=f"(c2.y), "=f"(c3.x), "=f"(c3.y) : "r"(adr[u]));
              else asm volatile("ld.shared.v2.f32 {%0,%1}, [%2+16];" : "=f"(c2.x), "=f"(c2.y) : "r"(adr[u]));
            }
            const int c = c4 + u;
#pragma unroll
            for (int r = 0; r < ROWS; r++) {
              acc[r][c] = Ffma2(make_float2(c01.x, c01.y), x[r][0], acc[r][c]);
              if (NJ > 1) acc[r][c] = Ffma2(make_float2(c01.z, c01.w), x[r][1 % NJ], acc[r][c]);
              if (NJ > 2) acc[r][c] = Ffma2(c2, x[r][2 % NJ], acc[r][c]);
              if (NJ > 3) acc[r][c] = Ffma2(c3, x[r][3 % NJ], acc[r][c]);
            }
          }
        }
        ip += a.CT;
      }
    }
    // emit: lanes hold columns lane and lane + 32 of each row
#pragma unroll
    for (int r = 0; r < ROWS; r++) {
      if (ho0 + ra + r >= ho_end) break;
#pragma unroll
      for (int half = 0; half < 2; half++) {
        const int wo = lane + 32 * half;
        if (wo < a.Wo) {
          float* out = a.dst + ((static_cast<size_t>(n) * a.Ho + ho0 + ra + r) * a.Wo + wo) * a.Cout + g * a.Kg + cbase;
#pragma unroll
          for (int c = 0; c < CPT; c += 4) {
            float4 o = half ? make_float4(acc[r][c].y, acc[r][c + 1].y, acc[r][c + 2].y, acc[r][c + 3].y)
                            : make_float4(acc[r][c].x, acc[r][c + 1].x, acc[r][c + 2].x, acc[r][c + 3].x);
            if (a.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
            *reinterpret_cast<float4*>(out + c) = o;
          }
        }
      }
    }
  }
}

template <int CPT, int J, int MAXT>
int LaunchBound(const ConvPlan& p, const ConvArgs& a, cudaStream_t st) {
  dim3 grid(a.G * a.nct * a.nstrips, a.N);
  void (*kern)(ConvArgs);
  switch (p.kernel) {
    case kConvS1: kern = conv_s1_kernel<FfmaLut, CPT, J, MAXT>; break;
    case kConvS1Tc: kern = conv_s1_kernel<WgmmaLut, CPT, J, MAXT>; break;
    case kConvRoll: kern = conv_roll_kernel<FfmaLut, CPT, J, MAXT>; break;
    case kConvRollTc: kern = conv_roll_kernel<WgmmaLut, CPT, J, MAXT>; break;
    default: ::qcnn::SetError("internal: kernel %d is not a LUT + gather kernel", p.kernel); return 1;
  }
  QCNN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
  kern<<<grid, p.threads, p.smem, st>>>(a);
  QCNN_CUDA(cudaGetLastError());
  return 0;
}

template <int CPT, int J>
int LaunchOne(const ConvPlan& p, const ConvArgs& a, cudaStream_t st) {
  if (p.threads <= 256) return LaunchBound<CPT, J, 256>(p, a, st);
  if (p.threads <= 384) return LaunchBound<CPT, J, 384>(p, a, st);
  return LaunchBound<CPT, J, 512>(p, a, st);
}

}  // namespace

namespace qcnn {

// Candidate tilings of the LUT + gather kernels for batch size N.  Cost model in SM-cycles per CTA, times the number of
// waves the whole batch needs on this GPU (so small batches trade LUT rebuilds for parallelism):
//   gather  = shared-memory wavefronts: one per (warp, tap, s, channel, position-slot) plus one 128-bit offset load
//             per 4 channels -> (1 + 1/(4J)) per lookup slot, 1 wavefront / clk / SM
//   build   = LUT entries built (incl. halo rows, garbage columns and per-channel-tile rebuilds) x
//             (0.66 * dims + 0.3) issue slots / 32 lanes / ~2.5 warp-instructions per clk
//   sync    = ~300 clk per (s [, input row]) phase pair
// The two stages do not overlap inside a CTA (one CTA per SM), so the costs add.
void PlanLutGather(const qcnn_layer* L, int N, ConvCands* cands) {
  bool found = false;   // a tiling exists (while ncol = 1: a whole-row one)
  const int G = L->grp, Cg = L->Cin / G, Kg = L->Cout / G;
  const int taps = L->ksz * L->ksz;
  const size_t smemMax = SmemOptin(L->ctx);
  ConvPlan p0;   // every candidate: the layer's geometry, the tiling fields zero
  memset(&p0, 0, sizeof(p0));
  ConvArgs& a0 = p0.a;
  a0.Hi = L->Hin; a0.Wi = L->Win; a0.Cin = L->Cin; a0.Ho = L->Ho; a0.Wo = L->Wo; a0.Cout = L->Cout;
  a0.ksz = L->ksz; a0.pad = L->pad; a0.stride = L->stride; a0.G = G; a0.Cg = Cg; a0.Kg = Kg;
  a0.KgPad = RoundUp(Kg, 16);
  a0.S = L->S; a0.K = L->K; a0.d = L->d;
  double dimsSum = 0;  // sum over subspaces of the dims that exist
  for (int s = 0; s < L->S; s++) dimsSum += std::max(0, std::min(Cg - s * L->d, L->d));
  const double ipe = 0.66 * (dimsSum / L->S) + 0.3;  // issue slots per LUT entry
  // tensor-core LUT stage: 128 codewords (MMA M), every subspace <= 8 dims (one K = 8 tf32 step)
  const bool tcOk = L->K == 128 && L->d <= 8;
  // stride 1: whole rows per CTA; column tiles (ncol > 1) only for layers whose rows fit no LUT (VGG16's 224-wide block 1)
  for (int ncol = 1; ncol <= (L->stride == 1 ? std::min(16, L->Wo) : 1) && !(ncol > 1 && found); ncol++)
  for (const int CPT : {32, 16}) {
    if (Kg % CPT != 0) continue;
    for (int J = 1; J * CPT <= 64 && J <= 4; J++) {
      for (int nct = 1; nct <= Kg / CPT; nct++) {
        if (Kg % nct != 0) continue;
        const int CT = Kg / nct;
        if (CT % CPT != 0 || CT % 16 != 0) continue;
        const int cwarps = CT / CPT;
        for (int R = 1; R <= L->Ho; R++) {
          for (int tc = 0; tc <= (tcOk ? 1 : 0); tc++) {
            ConvPlan p = p0;
            ConvArgs& a = p.a;
            a.R = R;
            a.nstrips = CeilDiv(L->Ho, R) * ncol;
            a.ncol = ncol; a.CW = CeilDiv(L->Wo, ncol);
            a.CT = CT; a.nct = nct; a.cwarps = cwarps;
            double gatherSlots, builtEntries, phases;
            int warps;
            if (L->stride == 1) {
              p.kernel = tc ? kConvS1Tc : kConvS1;
              a.PW = ncol > 1 ? a.CW + L->ksz - 1 : L->Win + L->pad;
              a.RI = R + L->ksz - 1;
              a.pwarps = CeilDiv(R * a.PW, 32 * J);
              a.rgroups = 1;
              const int need1 = a.RI * a.PW + std::max(L->pad, L->ksz - 1) + 1;
              const int need2 = a.pwarps * 32 * J + (L->ksz - 1) * a.PW + (L->ksz - 1) + 1;
              warps = a.pwarps * cwarps;
              if (tc) {
                a.NM = RoundUp(std::max(need1, need2), 32);  // MMA N = LUT columns per subspace
                if (a.NM > 256 || warps < 4) continue;
                a.PP = a.NM + 4;    // row pitch = 4 (mod 32) words
              } else {
                a.PP = RoundUp(std::max(need1, need2), 4);
              }
              gatherSlots = static_cast<double>(a.pwarps) * J * taps * L->S * CT;   // wavefronts of LUT reads
              builtEntries = static_cast<double>(a.PP) * L->K * L->S;
              phases = L->S;
            } else {
              p.kernel = tc ? kConvRollTc : kConvRoll;
              a.rgroups = CeilDiv(L->ksz, L->stride);
              a.pwarps = CeilDiv(L->Wo, 32 * J);
              const int ph1 = CeilDiv(L->Win + 2 * L->pad, L->stride);
              const int ph2 = a.pwarps * 32 * J + (L->ksz - 1) / L->stride + 1;
              warps = a.pwarps * cwarps * a.rgroups;
              const double rowsIn = (R - 1) * L->stride + L->ksz;
              if (tc) {
                // phase length = the real columns only; idle lanes beyond Wo then read into the next phase's columns
                // (valid shared memory, results discarded), so the row must hold (stride-1)*PH + lanes + shift entries
                a.PW = ph1;
                a.NM = RoundUp(std::max(ph1 * L->stride, (L->stride - 1) * ph1 + ph2), 32);
                if (a.NM > 256 || warps < 4) continue;
                a.PP = a.NM + 4;
              } else {
                a.PW = std::max(ph1, ph2);           // phase length
                a.PP = RoundUp(a.PW * L->stride, 4);
              }
              gatherSlots = static_cast<double>(a.pwarps) * J * R * taps * L->S * CT;
              builtEntries = static_cast<double>(a.PP) * L->K * L->S * rowsIn;
              phases = L->S * rowsIn;
            }
            p.CPT = CPT; p.J = J;
            p.threads = warps * 32;
            if (p.threads > kMaxThreads || p.threads < 64) continue;
            p.smem = tc ? WgmmaLut::MapSmem(L->K, a.PP, a.NM, taps, CT).bytes : FfmaLut::MapSmem(L->K, a.PP, a.NM, taps, CT).bytes;
            if (p.smem > smemMax) continue;
            // model constants (they only order the candidates; on-device timing picks among the cheapest): ~1.3 clk per
            // gather wavefront, FFMA LUT stage ~0.12 clk per entry at d = 8, tensor-core LUT stage = MMA + fragment
            // stores + operand split; gather latency hiding improves with resident warps
            const double gather = gatherSlots * (1.0 + 1.0 / (4.0 * J)) * (1.15 + 1.6 / warps);
            const double build = tc ? builtEntries * 0.02 + 300.0 * phases : builtEntries * ipe / 5.5 * 0.12;
            const double perCta = gather + build + 400.0 * phases;
            // few resident warps cannot keep ~30 LDS in flight per SM nor feed the FMA pipe during the LUT stage
            // (model constants, not measurements); 64 accumulators at 512 threads spill
            double occPenalty = warps < 4 ? 2.5 : (warps < 6 ? 1.6 : (warps < 8 ? 1.25 : 1.0));
            if (p.threads > 384 && J * CPT >= 64) occPenalty *= 1.1;
            const double ctas = static_cast<double>(G) * nct * a.nstrips * N;
            const double waves = std::ceil(ctas / L->ctx->sm_count);
            const double cost = perCta * waves * occPenalty;
            p.key = {CPT, J, nct, a.nstrips, a.rgroups, R};
            cands->emplace_back(cost, p);
            found = true;
          }
        }
      }
    }
  }
  // single subspace of <= 4 existing dims: evaluate <x, codeword> at the point of use (conv_direct_kernel)
  if (L->S == 1 && std::min(Cg, L->d) <= 4 && L->Wo <= 64) {
    const int NJ = std::min(Cg, L->d) <= 3 ? 3 : 4;
    for (const int CPT : {16, 8}) {
      if (Kg % CPT != 0 || Kg % 16 != 0) continue;
      for (int nct = 1; nct <= 2; nct++) {
        if (Kg % nct != 0 || (Kg / nct) % 16 != 0 || (Kg / nct) % CPT != 0) continue;
        const int CT = Kg / nct, cwarps = CT / CPT;
        for (const int R : {2, 4, 6, 8, 14}) {
          if (R > L->Ho + 1) continue;
          for (int rgroups = 1; rgroups <= 2; rgroups++)
          for (int rowsPer = 2; rowsPer <= (CPT == 8 ? 4 : 2); rowsPer += 2) {
            if (rgroups > R / rowsPer) continue;
            ConvPlan p = p0;
            ConvArgs& a = p.a;
            p.kernel = kConvDirect; p.CPT = CPT; p.J = rowsPer;
            a.R = std::min(R, L->Ho + (L->Ho & 1)); a.nstrips = CeilDiv(L->Ho, a.R);
            a.CT = CT; a.nct = nct; a.cwarps = cwarps; a.pwarps = 1; a.rgroups = rgroups;
            a.PW = CeilDiv(L->Win + 2 * L->pad, L->stride);       // phase length
            a.PP = RoundUp(a.PW * L->stride, 4);                   // row pitch
            p.threads = 32 * cwarps * rgroups;
            if (p.threads > 384 || p.threads < 128) continue;
            const int rowsIn = (a.R - 1) * L->stride + L->ksz;
            p.smem = sizeof(float) * (static_cast<size_t>(rowsIn) * NJ * a.PP + 64 + 8 * static_cast<size_t>(L->K) +
                                      static_cast<size_t>(taps) * CT);
            if (p.smem > smemMax) continue;
            const int pairs = CeilDiv(a.R, rowsPer);
            // issue slots: per (row pair, tap, channel) 2 loads + 2*NJ FFMA pairs, plus 4*NJ pixel loads per tap
            const double perWarp = static_cast<double>(CeilDiv(pairs, rgroups)) * taps * (CPT * (2.0 + rowsPer * NJ) + 2.0 * rowsPer * NJ + CPT / 4.0);
            const double perCta = perWarp * cwarps * rgroups / 2.6 + rowsIn * NJ * a.PP * 0.5;
            const double ctas = static_cast<double>(G) * nct * a.nstrips * N;
            const double waves = std::ceil(ctas / L->ctx->sm_count);
            p.key = {CPT, rowsPer, nct, a.nstrips, rgroups, a.R};
            cands->emplace_back(perCta * waves, p);
          }
        }
      }
    }
  }
}

template <int CPT, int NJ, int ROWS>
static int LaunchDirect(const ConvPlan& p, const ConvArgs& a, cudaStream_t st) {
  dim3 grid(a.G * a.nct * a.nstrips, a.N);
  auto kern = conv_direct_kernel<CPT, NJ, ROWS>;
  QCNN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
  kern<<<grid, p.threads, p.smem, st>>>(a);
  QCNN_CUDA(cudaGetLastError());
  return 0;
}

int LaunchLutGather(qcnn_layer* L, const ConvPlan& p, const float* src, int N, float* dst, int relu, cudaStream_t st) {
  ConvArgs a = p.a;
  a.src = src; a.dst = dst; a.ctrd = L->d_ctrd.as<float>(); a.asmt = L->d_asmt.as<uint8_t>(); a.bias = L->d_bias.as<float>();
  a.N = N; a.relu = relu; a.src_nchw = L->src_nchw;
  if (p.kernel == kConvDirect) {
    const int nj = std::min(a.Cg, a.d);
    // p.J carries the output rows per thread (2 or 4)
    if (p.CPT == 16) return nj <= 3 ? LaunchDirect<16, 3, 2>(p, a, st) : LaunchDirect<16, 4, 2>(p, a, st);
    if (p.J == 4) return nj <= 3 ? LaunchDirect<8, 3, 4>(p, a, st) : LaunchDirect<8, 4, 4>(p, a, st);
    return nj <= 3 ? LaunchDirect<8, 3, 2>(p, a, st) : LaunchDirect<8, 4, 2>(p, a, st);
  }
  QCNN_CHECK(!(a.src_nchw && (p.kernel == kConvS1 || p.kernel == kConvS1Tc)), "qcnn_conv_aprx_forward: NCHW source is only supported by the strided kernel");
  int rc = 1;
#define QCNN_DISPATCH(C, JJ) if (p.CPT == C && p.J == JJ) rc = LaunchOne<C, JJ>(p, a, st); else
  QCNN_DISPATCH(32, 1) QCNN_DISPATCH(32, 2) QCNN_DISPATCH(16, 1) QCNN_DISPATCH(16, 2) QCNN_DISPATCH(16, 3)
  QCNN_DISPATCH(16, 4) { SetError("internal: no conv instantiation for CPT=%d J=%d", p.CPT, p.J); return 1; }
#undef QCNN_DISPATCH
  return rc;
}

void DescribeLutGather(const qcnn_layer* L, const ConvPlan& p, int N, char* buf, size_t cap) {
  snprintf(buf, cap, " CPT=%d J=%d threads=%d smem=%zuB grid=(%d,%d) R=%d strips=%d CT=%d nct=%d PP=%d pwarps=%d "
           "cwarps=%d rgroups=%d", p.CPT, p.J, p.threads, p.smem, p.a.G * p.a.nct * p.a.nstrips, N, p.a.R, p.a.nstrips,
           p.a.CT, p.a.nct, p.a.PP, p.a.pwarps, p.a.cwarps, p.a.rgroups);
}

}  // namespace qcnn
