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
using qcnn::ByteOf32;
using qcnn::CpAsync16;
using qcnn::CpAsyncCommit;
using qcnn::CpAsyncWaitAll;
using qcnn::MbarArrive;
using qcnn::MbarExpectTx;
using qcnn::MbarInit;
using qcnn::MbarWait;
using qcnn::PackBf16x2;
using qcnn::SmemU32;
using qcnn::SplitBf16x4;
using qcnn::SplitTf32x4;
using qcnn::Wgmma;

constexpr int kThreads = 384;
constexpr int kConsumers = 256;  // warps 0-7
constexpr int kStagers = 128;    // warps 8-11
constexpr int kMaxGT = 4;        // k-steps per stage (decoded A fragments of a stage live in registers)
constexpr int kRegPos = 12;      // float4 a stager thread holds in registers (convolution modes: planeF4 <= 12 * 128)
constexpr int kCbBufs = 4;       // codebook / index buffers: the decoders run ahead of the position planes

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

// Mode 2 with a bit-packed FC table (packed_asmt.h): the 16 indices of channels [ch, ch + 16) of one row (2 b bytes, from
// the four aligned words that cover them) -> 16 bytes idx << kshift at dst, the index block the byte table would stage
__device__ __forceinline__ void StagePackedRow(uint8_t* dst, const uint8_t* row, int ch, int b, int kshift) {
  const uint32_t bit0 = static_cast<uint32_t>(ch) * b, sh = bit0 & 31u;
  const uint32_t* wp = reinterpret_cast<const uint32_t*>(row) + (bit0 >> 5);
  const uint32_t w0 = __ldg(wp), w1 = __ldg(wp + 1), w2 = __ldg(wp + 2), w3 = __ldg(wp + 3);
  const uint32_t u0 = __funnelshift_r(w0, w1, sh), u1 = __funnelshift_r(w1, w2, sh), u2 = __funnelshift_r(w2, w3, sh), u3 = w3 >> sh;
  const uint32_t mask = (1u << b) - 1u;
  uint32_t o[4] = {0u, 0u, 0u, 0u};
#pragma unroll
  for (int c = 0; c < 16; c++) {
    const int pos = c * b, j = pos >> 5;   // (16 b + sh <= 128 bits: the fields end inside u3)
    const uint32_t lo = j == 0 ? u0 : (j == 1 ? u1 : (j == 2 ? u2 : u3));
    const uint32_t hi = j == 0 ? u1 : (j == 1 ? u2 : (j == 2 ? u3 : 0u));
    o[c >> 2] |= ((__funnelshift_r(lo, hi, pos & 31) & mask) << kshift) << (8 * (c & 3));
  }
  *reinterpret_cast<uint4*>(dst) = make_uint4(o[0], o[1], o[2], o[3]);
}

// BF: bf16x2 operands (else 3xTF32); NT: positions per CTA = wgmma N; NT = 64 keeps the second accumulator (a.corr).
// The kernel body lives in pq_gemm_tc_body.cuh and is compiled into two kernels: pq_gemm_tc_kernel (byte index tables) and
// pq_gemm_tc_packed_kernel (PK: mode 2 with a bit-packed FC table of pkBits bits per index and rows of pkPitch bytes).
// Including the body, rather than calling a shared device function, leaves the code of pq_gemm_tc_kernel exactly what it
// was before the packed form existed (register allocation of these spilling kernels is sensitive to the call structure).
template <bool BF, int NT>
__global__ void __launch_bounds__(kThreads, 1) pq_gemm_tc_kernel(const GemmArgs a) {
  constexpr bool PK = false;
  constexpr int pkBits = 0, pkPitch = 0;
#include "pq_gemm_tc_body.cuh"
}
template <bool BF, int NT>
__global__ void __launch_bounds__(kThreads, 1) pq_gemm_tc_packed_kernel(const GemmArgs a, int pkBits, int pkPitch) {
  constexpr bool PK = true;
#include "pq_gemm_tc_body.cuh"
}

}  // namespace

namespace qcnn {

// Mode 1 k-step table (strided layer on phase planes): for every phase row ph, its k-steps in (kh, kw) order, as entries
// [chunkFirst[ph], + chunkCount[ph]) of ga.tab.  Reads ga.NPOS, ga.bf and ga.planeRows.  Returns the number of k-steps
// (> kMaxKSteps: the table does not fit) and sets ga.ntab.  The weight-stationary kernel (conv_ws.cu) runs the same table.
int Mode1Table(const qcnn_layer* L, GemmArgs& ga) {
  const int st = L->stride, PWp = CeilDiv(L->Win + 2 * L->pad, st);
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
  ga.ntab = ne;
  return ne;
}

// Mode 0 k-step table (stride-1 layer on the flat padded grid): the taps of a chunk in (kh, kw) order, a tap being a shift
// of the position operand's start by kh * PW + kw rows, K-core-matrix 1 (the chunk's second half / the x2 plane) NPOS rows
// further; index row and codebook slot = (half, tap).  Reads ga.PW and ga.NPOS, sets ga.ntab and the chunk range, returns
// the number of k-steps per chunk.  The weight-stationary kernel (conv_ws.cu) runs the same table.
int Mode0Table(const qcnn_layer* L, GemmArgs& ga) {
  const int taps = L->ksz * L->ksz;
  ga.ntab = taps;
  ga.chunkFirst[0] = 0; ga.chunkCount[0] = taps;
  for (int t = 0; t < taps; t++) {
    KStep& ks = ga.tab[t];
    ks.bStart = (t / L->ksz) * ga.PW + (t % L->ksz);
    ks.lbo = ga.NPOS;
    ks.idx0 = static_cast<short>(t); ks.idx1 = static_cast<short>(taps + t);
    ks.cb0 = 0; ks.cb1 = 1;
  }
  return taps;
}

// Candidate tilings for batch N (cost in SM-cycles, comparable with PlanLutGather's model); on-device timing chooses among them.
void PlanPqGemm(const qcnn_layer* L, int N, ConvCands* cands) {
  const int G = L->grp, Cg = L->Cin / G, Kg = L->Cout / G, taps = L->ksz * L->ksz;
  if (L->K < 1 || L->K > 256 || Kg % 16 != 0) return;
  const size_t smemMax = SmemOptin(L->ctx);
  if (L->stride > 1) {
    // mode 1: strided convolution with one subspace over <= 4 input channels (conv1), input on stride x stride phase planes
    const int st = L->stride, rowsPer = CeilDiv(L->ksz, st);
    if (Cg > 4 || L->S != 1 || L->d < Cg || st > 8 || L->Wo > CeilDiv(L->Win + 2 * L->pad, st)) return;
    const int pairs = (L->ksz + 1) / 2;
    if (rowsPer * pairs > 32 || L->ksz * pairs > kMaxKSteps) return;
    const int PWp = CeilDiv(L->Win + 2 * L->pad, st), PHp = CeilDiv(L->Hin + 2 * L->pad, st);
    const int IB = PHp * PWp;
    if (static_cast<double>(N) * IB > 2.0e9 || static_cast<double>(L->Hin) * L->Win * L->Cin * 4 > 2.0e9) return;
    for (const int NT : {128, 64}) {
      for (const int GT : {4, 3}) {
        ConvPlan p;
        memset(&p, 0, sizeof(p));
        p.kernel = kPqGemmTc; p.threads = kThreads;
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
        ga.idxT = (ga.tapsPad <= 48 && L->asmt_t_mode == 1) ? 1 : 0;
        if (ga.idxT) ga.idRows = ga.tapsPad;       // [128 channels][tapsPad] bytes
        ga.nChunks = st;
        ga.K = L->K; ga.cbF4 = L->K; ga.nPB = 2;
        // bf16x2 planes are half the size: keep EVERY phase row of the tile resident (no plane reuse), so that the stagers
        // never wait for the MMAs and the few k-steps of a phase row (conv1: 16-18) are not what hides a global-load latency
        if (ga.bf && st <= 4) ga.nPB = st;
        ga.nct = CeilDiv(Kg, 128);
        const int ne = Mode1Table(L, ga);
        if (ne > kMaxKSteps) continue;
        p.smem = static_cast<size_t>(MapSmem(ga).total);
        if (p.smem > smemMax) continue;
        const double ctas0 = static_cast<double>(CeilDiv(N * IB, NT)) * G * ga.nct;
        // small batches: split the phase rows over CTAs (partial sums reduced by LaunchSplitReduce)
        for (int nsplit = 1; nsplit <= st; nsplit *= 2) {
          if (nsplit > 1 && ctas0 * nsplit > 1.5 * L->ctx->sm_count) break;
          ga.kPerSplit = CeilDiv(st, nsplit);
          ga.nsplit = CeilDiv(st, ga.kPerSplit);
          if (ga.nsplit != nsplit) continue;
          p.key = {NT, GT, ga.nct, nsplit};
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
  for (const int NT : {128, 64}) {
    for (const int GT : {4, 3}) {
      ConvPlan p;
      memset(&p, 0, sizeof(p));
      p.kernel = kPqGemmTc; p.threads = kThreads;
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
      ga.idxT = (ga.tapsPad <= 32 && L->asmt_t_mode == 0) ? 1 : 0;
      if (ga.idxT) ga.idRows = 2 * ga.tapsPad;      // [half][128 channels][tapsPad] bytes = 2 * tapsPad rows of 128
      ga.nChunks = CeilDiv(Cg, 8);
      Mode0Table(L, ga);
      ga.K = L->K; ga.cbF4 = L->K; ga.nPB = 2;
      ga.nct = CeilDiv(Kg, 128);
      p.smem = static_cast<size_t>(MapSmem(ga).total);
      if (p.smem > smemMax) continue;
      const double ksteps = static_cast<double>(ga.nChunks) * taps;
      const double ctas0 = static_cast<double>(CeilDiv(N * IB, NT)) * G * ga.nct;
      // small batches: split the 8-channel chunks over CTAs (partial sums reduced by LaunchSplitReduce)
      for (int nsplit = 1; nsplit <= ga.nChunks; nsplit *= 2) {
        if (nsplit > 1 && ctas0 * nsplit > 1.5 * L->ctx->sm_count) break;
        ga.kPerSplit = CeilDiv(ga.nChunks, nsplit);
        ga.nsplit = CeilDiv(ga.nChunks, ga.kPerSplit);
        if (ga.nsplit != nsplit) continue;
        p.key = {NT, GT, ga.nct, nsplit};
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
  const int lim = static_cast<int>(SmemOptin(ctx));
#define QCNN_SMEM_ATTR(...) QCNN_CUDA(cudaFuncSetAttribute(pq_gemm_tc_kernel<__VA_ARGS__>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim))
  QCNN_SMEM_ATTR(true, 128); QCNN_SMEM_ATTR(true, 64); QCNN_SMEM_ATTR(false, 128); QCNN_SMEM_ATTR(false, 64);
#undef QCNN_SMEM_ATTR
#define QCNN_SMEM_ATTR(...) QCNN_CUDA(cudaFuncSetAttribute(pq_gemm_tc_packed_kernel<__VA_ARGS__>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim))
  QCNN_SMEM_ATTR(true, 128); QCNN_SMEM_ATTR(true, 64); QCNN_SMEM_ATTR(false, 128); QCNN_SMEM_ATTR(false, 64);
#undef QCNN_SMEM_ATTR
  if (ctx->device >= 0 && ctx->device < 64) done[ctx->device] = true;
  return 0;
}

static int LaunchKernel(const GemmArgs& a, unsigned blocks, size_t smem, cudaStream_t st, int pkBits = 0, int pkPitch = 0) {
  QCNN_CHECK((a.NT == 128 || a.NT == 64) && a.corr == (a.NT == 64 ? 1 : 0) && a.GT >= 1 && a.GT <= kMaxGT,
             "pq_gemm_tc: no instantiation for NT=%d GT=%d", a.NT, a.GT);
  if (pkBits) {
    QCNN_CHECK(a.mode == 2 && pkBits >= 4 && pkBits <= 7, "pq_gemm_tc: a bit-packed table is only read by mode 2 (FC)");
    if (a.bf) {
      if (a.NT == 128) pq_gemm_tc_packed_kernel<true, 128><<<blocks, kThreads, smem, st>>>(a, pkBits, pkPitch);
      else pq_gemm_tc_packed_kernel<true, 64><<<blocks, kThreads, smem, st>>>(a, pkBits, pkPitch);
    } else {
      if (a.NT == 128) pq_gemm_tc_packed_kernel<false, 128><<<blocks, kThreads, smem, st>>>(a, pkBits, pkPitch);
      else pq_gemm_tc_packed_kernel<false, 64><<<blocks, kThreads, smem, st>>>(a, pkBits, pkPitch);
    }
  } else if (a.bf) {
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

void SetGemmGeometry(const qcnn_layer* L, GemmArgs& a) {
  a.Hi = L->Hin; a.Wi = L->Win; a.Cin = L->Cin; a.Ho = L->Ho; a.Wo = L->Wo; a.Cout = L->Cout;
  a.ksz = L->ksz; a.pad = L->pad; a.stride = L->stride; a.G = L->grp; a.Cg = L->Cin / L->grp; a.Kg = L->Cout / L->grp;
  a.KgPad = RoundUp(a.Kg, 16); a.S = L->S; a.K = L->K; a.d = L->d;
  a.srcImg = static_cast<long long>(a.Hi) * a.Wi * a.Cin;
  if (L->src_nchw) { a.rowStride = a.Wi; a.colStride = 1; a.chStride = a.Hi * a.Wi; }
  else { a.rowStride = a.Wi * a.Cin; a.colStride = a.Cin; a.chStride = 1; }
  a.dstImg = static_cast<long long>(a.Ho) * a.Wo * a.Cout;
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
  SetGemmGeometry(L, a);
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

void DescribePqGemm(const qcnn_layer* L, const ConvPlan& p, int N, char* buf, size_t cap) {
  int ksteps = 0;
  for (int c = 0; c < p.g.nChunks; c++) ksteps += p.g.chunkCount[p.g.mode == 1 ? c : 0];
  snprintf(buf, cap, "(wgmma, weights decoded into registers%s) mode=%d NT=%d GT=%d smem=%zuB grid=%d NPOS=%d "
           "chunks=%d ksteps=%d nsplit=%d", p.g.bf ? ", bf16x2" : "", p.g.mode, p.g.NT, p.g.GT, p.smem,
           CeilDiv(N * p.g.IB, p.g.NT) * L->grp * p.g.nct * std::max(1, p.g.nsplit), p.g.NPOS, p.g.nChunks,
           ksteps / std::max(1, p.g.nsplit), std::max(1, p.g.nsplit));
}

// generic entry for callers that fill GemmArgs themselves (the fully-connected path in fc_aprx.cu)
size_t PqGemmSmemBytes(const GemmArgs& a) { return static_cast<size_t>(MapSmem(a).total); }
int LaunchPqGemmArgs(qcnn_ctx* ctx, const GemmArgs& a, long long blocks, cudaStream_t st, int asmtBits, int asmtPitch) {
  QCNN_CHECK(blocks >= 1 && blocks <= 2147483647LL, "pq_gemm_tc: bad grid");
  if (int rc = SetSmemLimitOnce(ctx)) return rc;
  return LaunchKernel(a, static_cast<unsigned>(blocks), PqGemmSmemBytes(a), st, asmtBits, asmtPitch);
}

}  // namespace qcnn
