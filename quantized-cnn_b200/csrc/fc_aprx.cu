// Fused PQ fully-connected layer for sm_90a: LUT stage + uint8 gather-accumulate in ONE kernel.
// Replaces CaffeEva::CalcFeatMap_FCntAprx + GetInPdMat (reference src/CaffeEva.cc:968-1025, 1261-1296):
//     LUT[n][s][k] = sum_j x[n][s*d+j] * ctrd[s][k][j]        (ascending j, rounded mul then rounded add)
//     dst[n][o]    = bias[o] + sum_s LUT[n][s][asmt[s][o]]    (ascending s)
//
// Mapping (HBM/L2 stream of the assignment matrix is the only large operand):
//   * lane = output channel.  A thread owns CPT consecutive channels and TN images -> TN*CPT accumulators.
//   * the device assignment table is [S][DoutPad] bytes, so a warp reads 32*CPT contiguous bytes per subspace
//     row (128-bit loads at CPT=16); rows stream through a rolling register window (one block of 8 rows in flight
//     while the previous block is consumed), the first block being issued BEFORE the chunk's LUT slice is built,
//     so the HBM/L2 stream overlaps the LUT arithmetic;
//   * the input slice and codebook rows of chunk c+1 are staged by cp.async while chunk c is gathered.
//   * the LUT slice of the chunk ([TN][PF][K] floats) lives in shared memory.  With K <= 32 one LUT row is
//     <= 128 B = one bank sweep: distinct codewords hit distinct banks and equal codewords broadcast, so the
//     lane-dependent gather is bank-conflict free by construction.
//   * assignments are stored pre-multiplied by 4 (byte offsets) when K <= 64, saving the shift per lookup.
//   * S can be split over blockIdx.z (needed at small N to fill the SMs); partial sums are reduced in a fixed
//     order by fc_reduce_kernel (deterministic; no atomics).  With nsplit == 1 the accumulation order is
//     exactly the reference's (bias, then s ascending) and the result is bit-identical to the CPU path.
#include "qcnn_internal.h"
#include "async_copy.h"
#include "packed_asmt.h"

#include <algorithm>
#include <cstring>
#include <cstdio>

namespace {

using qcnn::CpAsync16;
using qcnn::CpAsync4;
using qcnn::CpAsyncCommit;
using qcnn::CpAsyncWaitAll;

constexpr int kFcThreads = 256;

template <int CPT> struct AsmtVec;
template <> struct AsmtVec<4>  { using type = uint32_t; };
template <> struct AsmtVec<8>  { using type = uint2; };
template <> struct AsmtVec<16> { using type = uint4; };

__device__ __forceinline__ uint32_t LoadStream(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ uint2 LoadStream(const uint2* p) {
  uint2 v;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
  return v;
}
__device__ __forceinline__ uint4 LoadStream(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ void Zero(uint32_t& v) { v = 0u; }
__device__ __forceinline__ void Zero(uint2& v) { v = make_uint2(0u, 0u); }
__device__ __forceinline__ void Zero(uint4& v) { v = make_uint4(0u, 0u, 0u, 0u); }
__device__ __forceinline__ uint32_t Word(const uint32_t& v, int) { return v; }
__device__ __forceinline__ uint32_t Word(const uint2& v, int i) { return i == 0 ? v.x : v.y; }
__device__ __forceinline__ uint32_t Word(const uint4& v, int i) {
  return i == 0 ? v.x : (i == 1 ? v.y : (i == 2 ? v.z : v.w));
}

constexpr int kRowBlock = 8;  // assignment rows held in registers per block of the rolling prefetch window

// K: codewords per subspace; CPT: channels per thread; TN: images per CTA; PFL: subspaces per LUT chunk;
// PRE: assignments stored as byte offsets (idx*4)
//
// Per chunk of PFL subspaces:  (1) the chunk's input slice and codebook rows were copied into shared memory by
// cp.async while the PREVIOUS chunk was being gathered; (2) the LUT slice [TN][PFL][K] is built from them
// (shared -> shared, no global latency); (3) the chunk's assignment rows stream through a rolling register window
// (block r+1 is in flight while block r is consumed) and are gathered against the LUT slice.
//
// PACKED: the bit-packed table of packed_asmt.h (rows of `pitch` bytes, b = log2(K) bits per channel).  A thread streams the
// aligned words that cover its CPT * b bits of a row and unpacks them just before the lookups; tiling, chunking and the
// order of the adds are those of the byte table, so both give bit-identical sums.
template <int CPT, int NW> struct PackedWords { uint32_t w[NW]; };
template <bool PACKED, typename A, typename B> struct Pick { using type = A; };
template <typename A, typename B> struct Pick<false, A, B> { using type = B; };
template <int CPT, int NW>
__device__ __forceinline__ PackedWords<CPT, NW> LoadStream(const PackedWords<CPT, NW>* p) {
  PackedWords<CPT, NW> v;
#pragma unroll
  for (int i = 0; i < NW; i++) v.w[i] = LoadStream(reinterpret_cast<const uint32_t*>(p) + i);
  return v;
}
template <int CPT, int NW>
__device__ __forceinline__ void Zero(PackedWords<CPT, NW>& v) {
#pragma unroll
  for (int i = 0; i < NW; i++) v.w[i] = 0u;
}

template <int K, int CPT, int TN, int PFL, bool PRE, bool PACKED>
__device__ __forceinline__ void FcAprxBody(const FcArgs a, int pitch) {
  extern __shared__ __align__(16) unsigned char smraw[];
  constexpr int B = PACKED ? (K == 16 ? 4 : (K == 32 ? 5 : (K == 64 ? 6 : 7))) : 8;
  constexpr int NW = qcnn::PackedSpan<B, CPT>::kWords;
  using AV = typename Pick<PACKED, PackedWords<CPT, NW>, typename AsmtVec<CPT>::type>::type;
  constexpr int U = kRowBlock;
  static_assert(PFL % U == 0, "chunk must be a whole number of row blocks");
  const int d = a.d;
  const int xlen = TN * PFL * d;            // staged input slice of one chunk (floats)
  const int xpad = (xlen + 3) & ~3;
  const int clen = PFL * K * d;             // staged codebook rows of one chunk (floats, multiple of 4)
  float* lut = reinterpret_cast<float*>(smraw);  // [TN][PFL][K]
  float* xN = lut + TN * PFL * K;                 // [2][xpad]
  float* cN = xN + 2 * xpad;                      // [2][clen]

  const int tid = threadIdx.x;
  const int o0 = (blockIdx.x * kFcThreads + tid) * CPT;
  const int n0 = blockIdx.y * TN;
  const int split = blockIdx.z;
  const int s_begin = split * a.s_per_split;
  const int s_end = min(a.S, s_begin + a.s_per_split);
  const bool live = o0 < a.DoutPad;
  // PACKED: first bit of the thread's channels inside a row -> its first aligned word, and the bit offset inside that word
  const uint32_t bit0 = static_cast<uint32_t>(o0) * B, sh = bit0 & 31u;
  const uint8_t* pbase = a.asmt + (bit0 >> 5) * 4;
  auto rowPtr = [&](int s) -> const AV* {
    if constexpr (PACKED) return reinterpret_cast<const AV*>(pbase + static_cast<size_t>(s) * pitch);
    else return reinterpret_cast<const AV*>(a.asmt + static_cast<size_t>(s) * a.DoutPad + o0);
  };

  // asynchronous staging of chunk `sc` into buffer `buf`
  auto fetch = [&](int sc, int buf) {
    float* xb = xN + buf * xpad;
    float* cb = cN + buf * clen;
    const int per = PFL * d;
    for (int e = tid; e < xlen; e += kFcThreads) {
      const int nl = e / per, i = e - nl * per;
      const int f = sc * d + i;
      const int n = n0 + nl;
      const bool ok = n < a.N && f < a.Din && (sc + i / d) < s_end;
      int off = 0;
      if (ok) off = a.srcoff ? __ldg(a.srcoff + f) : f;  // NHWC source read in NCHW-flatten order
      CpAsync4(xb + e, a.src + (ok ? static_cast<size_t>(n) * a.Din + off : 0), ok);
    }
    const float* cg = a.ctrd + static_cast<size_t>(sc) * K * d;
    for (int v = tid; v < clen / 4; v += kFcThreads) {
      const bool ok = (sc + (4 * v) / (K * d)) < s_end;
      CpAsync16(cb + 4 * v, cg + (ok ? 4 * v : 0), ok);
    }
    CpAsyncCommit();
  };

  float acc[TN][CPT];
#pragma unroll
  for (int c = 0; c < CPT; c++) {
    const float bv = (split == 0 && o0 + c < a.Dout) ? __ldg(a.bias + o0 + c) : 0.0f;
#pragma unroll
    for (int nl = 0; nl < TN; nl++) acc[nl][c] = bv;
  }

  if (s_begin < s_end) fetch(s_begin, 0);
  int buf = 0;
  for (int sc = s_begin; sc < s_end; sc += PFL, buf ^= 1) {
    // (0) first block of assignment rows: in flight during the LUT build
    AV win[U];
#pragma unroll
    for (int r = 0; r < U; r++) {
      const int s = sc + r;
      if (live && s < s_end) win[r] = LoadStream(rowPtr(s));
      else Zero(win[r]);
    }
    // (1) staged operands of this chunk have landed; the previous gather is done with `lut`
    CpAsyncWaitAll();
    __syncthreads();
    // (2) LUT slice: thread owns (subspace r, codeword k) pairs and sweeps the TN images
    {
      const float* xb = xN + buf * xpad;
      const float* cb = cN + buf * clen;
      for (int pr = tid; pr < PFL * K; pr += kFcThreads) {
        const int r = pr / K, k = pr % K;
        const float* c = cb + static_cast<size_t>(pr) * d;
        if (d == 4) {
          const float4 cv = *reinterpret_cast<const float4*>(c);
#pragma unroll
          for (int nl = 0; nl < TN; nl++) {
            const float4 xv = *reinterpret_cast<const float4*>(xb + nl * PFL * 4 + r * 4);
            float v = __fmul_rn(xv.x, cv.x);           // 0 + x0*c0 == x0*c0 exactly
            v = __fadd_rn(v, __fmul_rn(xv.y, cv.y));
            v = __fadd_rn(v, __fmul_rn(xv.z, cv.z));
            v = __fadd_rn(v, __fmul_rn(xv.w, cv.w));
            lut[(nl * PFL + r) * K + k] = v;
          }
        } else {
#pragma unroll
          for (int nl = 0; nl < TN; nl++) {
            const float* x = xb + nl * PFL * d + r * d;
            float v = 0.0f;
            for (int j = 0; j < d; j++) v = __fadd_rn(v, __fmul_rn(x[j], c[j]));
            lut[(nl * PFL + r) * K + k] = v;
          }
        }
      }
    }
    __syncthreads();
    // (3) next chunk's operands fly in while this one is gathered
    if (sc + PFL < s_end) fetch(sc + PFL, buf ^ 1);
    const char* lutb = reinterpret_cast<const char*>(lut);
#pragma unroll
    for (int rb = 0; rb < PFL; rb += U) {
      AV cur[U];
#pragma unroll
      for (int r = 0; r < U; r++) cur[r] = win[r];
      if (rb + U < PFL) {
#pragma unroll
        for (int r = 0; r < U; r++) {
          const int s = sc + rb + U + r;
          if (live && s < s_end) win[r] = LoadStream(rowPtr(s));
          else Zero(win[r]);
        }
      }
      // rows past s_end hold index 0 and their LUT rows are zero, so no tail guard is needed
#pragma unroll
      for (int r = 0; r < U; r++) {
        if constexpr (PACKED) {
          uint32_t idx[CPT];
          qcnn::UnpackFields<B, CPT, NW>(cur[r].w, sh, idx);
#pragma unroll
          for (int c = 0; c < CPT; c++) {
            const uint32_t off = idx[c] << 2;
#pragma unroll
            for (int nl = 0; nl < TN; nl++)
              acc[nl][c] += *reinterpret_cast<const float*>(lutb + (nl * PFL + rb + r) * K * 4 + off);
          }
        } else {
#pragma unroll
          for (int c = 0; c < CPT; c++) {
            const uint32_t w = Word(cur[r], c >> 2);
            uint32_t off = (w >> (8 * (c & 3))) & 0xFFu;
            if (!PRE) off <<= 2;
#pragma unroll
            for (int nl = 0; nl < TN; nl++)
              acc[nl][c] += *reinterpret_cast<const float*>(lutb + (nl * PFL + rb + r) * K * 4 + off);
          }
        }
      }
    }
  }

  if (!live) return;
#pragma unroll
  for (int nl = 0; nl < TN; nl++) {
    const int n = n0 + nl;
    if (n >= a.N) break;
    if (a.nsplit == 1) {
      float* out = a.dst + static_cast<size_t>(n) * a.Dout;
#pragma unroll
      for (int c = 0; c < CPT; c++) {
        if (o0 + c < a.Dout) out[o0 + c] = a.relu ? fmaxf(acc[nl][c], 0.0f) : acc[nl][c];
      }
    } else {
      float* out = a.partial + (static_cast<size_t>(split) * a.N + n) * a.DoutPad;
#pragma unroll
      for (int c = 0; c < CPT; c++) out[o0 + c] = acc[nl][c];
    }
  }
}

template <int K, int CPT, int TN, int PFL, bool PRE>
__global__ void __launch_bounds__(kFcThreads, 2) fc_aprx_kernel(const FcArgs a) {
  FcAprxBody<K, CPT, TN, PFL, PRE, false>(a, 0);
}
template <int K, int CPT, int TN, int PFL>
__global__ void __launch_bounds__(kFcThreads, 2) fc_aprx_packed_kernel(const FcArgs a, int pitch) {
  FcAprxBody<K, CPT, TN, PFL, false, true>(a, pitch);
}

// dst[n][o] = sum over splits (ascending; split 0 already carries the bias)
__global__ void fc_reduce_kernel(const float* __restrict__ partial, float* __restrict__ dst, int N, int Dout,
                                 int DoutPad, int nsplit, int relu) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * Dout) return;
  const int n = i / Dout, o = i % Dout;
  float v = 0.0f;
  for (int sp = 0; sp < nsplit; sp++) v += partial[(static_cast<size_t>(sp) * N + n) * DoutPad + o];
  dst[i] = relu ? fmaxf(v, 0.0f) : v;
}

// Activations of the tensor-core FC path, pre-split (3xTF32 hi / lo) and laid out as the shared-memory plane image of
// every (image tile, k-chunk): [tile][chunk][hi, lo][2*KS halves][NT images] float4, so that a CTA stages a chunk with
// ONE bulk copy.  Folds the NHWC -> NCHW-flatten map of the first FC layer (srcoff) and zero-pads images / features.
__global__ void fc_prep_kernel(const float* __restrict__ src, const int* __restrict__ srcoff, float4* __restrict__ dst,
                               int N, int Din, int NT, int KS, int nChunksAll, int tiles) {
  const size_t per = static_cast<size_t>(2 * KS) * NT;                       // float4 per plane (hi or lo)
  const size_t total = static_cast<size_t>(tiles) * nChunksAll * per;
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const size_t blk = i / per;
  const int r = static_cast<int>(i - blk * per);
  const int ih = r / NT, n = r - ih * NT;
  const int tile = static_cast<int>(blk / nChunksAll), chunk = static_cast<int>(blk - static_cast<size_t>(tile) * nChunksAll);
  const int Q = tile * NT + n, f = (chunk * KS * 2 + ih) * 4;
  float v[4] = {0.0f, 0.0f, 0.0f, 0.0f};
  if (Q < N) {
    const float* row = src + static_cast<size_t>(Q) * Din;
#pragma unroll
    for (int j = 0; j < 4; j++)
      if (f + j < Din) v[j] = __ldg(row + (srcoff ? __ldg(srcoff + f + j) : f + j));
  }
  float4 hi, lo;
  hi.x = __uint_as_float(__float_as_uint(v[0]) & 0xFFFFE000u); lo.x = v[0] - hi.x;
  hi.y = __uint_as_float(__float_as_uint(v[1]) & 0xFFFFE000u); lo.y = v[1] - hi.y;
  hi.z = __uint_as_float(__float_as_uint(v[2]) & 0xFFFFE000u); lo.z = v[2] - hi.z;
  hi.w = __uint_as_float(__float_as_uint(v[3]) & 0xFFFFE000u); lo.w = v[3] - hi.w;
  float4* base = dst + blk * per * 2;
  base[r] = hi;
  base[per + r] = lo;
}

// bf16x2 form of the same image: [tile][chunk][x1, x2][KS k-steps][NT images] rows of 16 bytes = eight consecutive
// features as bf16 (x = x1 + x2); half the bytes of the 3xTF32 image.
__device__ __forceinline__ uint32_t PackBf(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__global__ void fc_prep_bf_kernel(const float* __restrict__ src, const int* __restrict__ srcoff, uint4* __restrict__ dst,
                                  int N, int Din, int NT, int KS, int nChunksAll, int tiles) {
  const size_t per = static_cast<size_t>(KS) * NT;                           // rows per plane (x1 or x2)
  const size_t total = static_cast<size_t>(tiles) * nChunksAll * per;
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const size_t blk = i / per;
  const int r = static_cast<int>(i - blk * per);
  const int ks = r / NT, n = r - ks * NT;
  const int tile = static_cast<int>(blk / nChunksAll), chunk = static_cast<int>(blk - static_cast<size_t>(tile) * nChunksAll);
  const int Q = tile * NT + n, f = (chunk * KS + ks) * 8;
  float v[8] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
  if (Q < N) {
    const float* row = src + static_cast<size_t>(Q) * Din;
#pragma unroll
    for (int j = 0; j < 8; j++)
      if (f + j < Din) v[j] = __ldg(row + (srcoff ? __ldg(srcoff + f + j) : f + j));
  }
  uint32_t p1[4], p2[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    p1[j] = PackBf(v[2 * j], v[2 * j + 1]);
    const float r0 = v[2 * j] - __uint_as_float(p1[j] << 16), r1 = v[2 * j + 1] - __uint_as_float(p1[j] & 0xFFFF0000u);
    p2[j] = PackBf(r0, r1);
  }
  uint4* base = dst + blk * per * 2;
  base[r] = make_uint4(p1[0], p1[1], p1[2], p1[3]);
  base[per + r] = make_uint4(p2[0], p2[1], p2[2], p2[3]);
}

// PACKED: the bit-packed table, rows of `pitch` bytes (PRE is then false: the kernel scales the unpacked index itself)
template <int K, int CPT, int TN, int PF, bool PRE, bool PACKED>
int Launch(const FcArgs& a, int pitch, dim3 grid, cudaStream_t st) {
  const size_t smem = qcnn::FcGatherSmemBytes(K, TN, a.d);   // (PlanFcGather chose a TN that fits: this is a backstop)
  if (smem > qcnn::kFcGatherSmemMax) {
    qcnn::SetError("qcnn_fc_aprx_forward: K=%d d=%d needs %zu bytes of shared memory per CTA", K, a.d, smem);
    return 1;
  }
  if constexpr (PACKED) {
    auto kern = fc_aprx_packed_kernel<K, CPT, TN, PF>;
    if (smem > 48 * 1024) QCNN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, kFcThreads, smem, st>>>(a, pitch);
  } else {
    auto kern = fc_aprx_kernel<K, CPT, TN, PF, PRE>;
    if (smem > 48 * 1024) QCNN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, kFcThreads, smem, st>>>(a);
  }
  QCNN_CUDA(cudaGetLastError());
  return 0;
}

// subspaces per LUT chunk of the instantiation for K codewords and tn images per CTA (LaunchK's PF, PlanFcGather's pf)
constexpr int FcChunkLen(int K, int tn) { return tn == 1 ? (K <= 64 ? 16 : 8) : (K <= 32 ? 32 : (K <= 64 ? 16 : 8)); }

template <int K, bool PRE, bool PACKED = false>
int LaunchK(const FcArgs& a, int tn, int cpt, dim3 grid, cudaStream_t st, int pitch = 0) {
  if (cpt == 4 && tn == 8) return Launch<K, 4, 8, FcChunkLen(K, 8), PRE, PACKED>(a, pitch, grid, st);
  switch (tn) {
    case 1: return Launch<K, 16, 1, FcChunkLen(K, 1), PRE, PACKED>(a, pitch, grid, st);
    case 4: return Launch<K, 8, 4, FcChunkLen(K, 4), PRE, PACKED>(a, pitch, grid, st);
    default: return Launch<K, 8, 8, FcChunkLen(K, 8), PRE, PACKED>(a, pitch, grid, st);
  }
}

}  // namespace

namespace qcnn {

// dst[r][c] = sum over splits of partial[split][r][c] (+ ReLU); split 0 carries the bias.  The K-split of every FC family
// (fc_plan.cu) and of the pq_gemm_tc convolutions (rows = positions).
int LaunchSplitReduce(qcnn_ctx* ctx, const float* partial, float* dst, int rows, int cols, int colsPad, int nsplit, int relu,
                      cudaStream_t st) {
  const int total = rows * cols;
  fc_reduce_kernel<<<CeilDiv(total, 256), 256, 0, st>>>(partial, dst, rows, cols, colsPad, nsplit, relu);
  QCNN_CUDA(cudaGetLastError());
  ctx->launches++;
  return 0;
}

// k-steps per chunk of the tensor-core FC path (plane image of a chunk: 2 * 3 halves x NT images, hi + lo)
constexpr int kFcKs = 3;

// Large batches: the layer as a decode-at-use GEMM on the tensor cores (pq_gemm_tc.cu, mode 2): M = 128 outputs per CTA,
// N = up to 128 images, K split over CTAs so that the grid fills the GPU.  Fills p->tc (everything but the pointers) and
// p->nsplit; false when the staging does not fit in shared memory.
bool PlanFcMode2(const qcnn_layer* L, int N, FcPlan* p) {
  GemmArgs& a = p->tc;
  memset(&a, 0, sizeof(a));
  a.mode = 2;
  a.N = N; a.Cin = L->Din; a.Cout = L->Dout; a.G = 1; a.Cg = L->Din; a.Kg = L->Dout; a.KgPad = L->DoutPad;
  a.S = L->S; a.K = L->K; a.d = L->d; a.kshift = L->kshift;
  a.srcImg = L->Din; a.dstImg = 0;
  a.IB = 1; a.PW = 1;
  a.NT = N > 64 ? 128 : 64;   // the two wgmma N of pq_gemm_tc
  a.corr = a.NT <= 64 ? 1 : 0;
  a.bf = L->opt_tc_bf ? 1 : 0;
  a.cbPre = a.bf && L->d_ctrd_bf.get() ? 1 : 0;   // (d % 4 == 0)
  a.GT = kFcKs;
  a.nPB = 3; a.nChunksAll = CeilDiv(L->Din / 8, kFcKs);
  a.planeF4 = kFcKs * 2 * a.NT;
  a.planeRows = a.bf ? kFcKs * a.NT : a.planeF4;
  a.NPOS = a.NT;
  a.cbSlots = L->d == 1 ? 8 * kFcKs : 2 * kFcKs;
  a.idRows = a.cbSlots;
  a.cbF4 = L->d == 1 ? L->K / 4 : L->K;
  a.ntab = kFcKs;
  a.chunkFirst[0] = 0; a.chunkCount[0] = kFcKs;
  for (int i = 0; i < kFcKs; i++) {
    KStep& ks = a.tab[i];
    ks.bStart = 2 * i * a.NT; ks.lbo = a.NT;
    if (a.bf) { ks.bStart = i * a.NT; ks.lbo = kFcKs * a.NT; }   // row = (k-step, image); x2 plane = K-core-matrix 1
    if (L->d == 1) { ks.idx0 = static_cast<short>(8 * i); ks.idx1 = static_cast<short>(8 * i + 4); }
    else { ks.idx0 = static_cast<short>(2 * i); ks.idx1 = static_cast<short>(2 * i + 1); }
    ks.cb0 = ks.idx0; ks.cb1 = ks.idx1;
  }
  a.nct = CeilDiv(L->Dout, 128);
  const int tiles = CeilDiv(N, a.NT);
  a.kAll = L->Din / 8;
  a.nsplit = std::max(1, L->ctx->sm_count / (tiles * a.nct));
  a.kPerSplit = RoundUp(CeilDiv(a.kAll, a.nsplit), kFcKs);
  a.nsplit = CeilDiv(a.kAll, a.kPerSplit);
  a.dstRow = a.nsplit > 1 ? L->DoutPad : L->Dout;
  p->nsplit = a.nsplit;
  return PqGemmSmemBytes(a) <= SmemOptin(L->ctx);
}

void DescribeFcMode2(const qcnn_layer* L, const FcPlan& p, int N, char* buf, size_t cap) {
  const GemmArgs& a = p.tc;
  snprintf(buf, cap, "pq_gemm_tc(wgmma, weights decoded into registers%s) mode=2 NT=%d GT=3 grid=%d nsplit=%d ksteps=%d",
           a.bf ? ", bf16x2" : "", a.NT, CeilDiv(N, a.NT) * a.nsplit * a.nct, a.nsplit, a.kPerSplit);
}

// The activations as the plane image of every (image tile, chunk): NT images per tile, KS k-steps per chunk, bf16x2
// (fc_prep_bf_kernel) or 3xTF32 (fc_prep_kernel) pieces, in L->d_flat
int PrepFcPlanes(qcnn_layer* L, const float* src, int N, int NT, int KS, int nChunksAll, bool bf, cudaStream_t st) {
  qcnn_ctx* ctx = L->ctx;
  const int tiles = CeilDiv(N, NT);
  const size_t total = static_cast<size_t>(tiles) * nChunksAll * KS * NT * (bf ? 1 : 2);   // 16-byte rows of one plane (hi or lo)
  QCNN_CUDA(L->d_flat.Reserve(ctx, total * 2 * sizeof(float4), st));
  if (bf)
    fc_prep_bf_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(src, L->d_srcoff.as<int>(), L->d_flat.as<uint4>(),
                                                                               N, L->Din, NT, KS, nChunksAll, tiles);
  else
    fc_prep_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(src, L->d_srcoff.as<int>(), L->d_flat.as<float4>(),
                                                                            N, L->Din, NT, KS, nChunksAll, tiles);
  QCNN_CUDA(cudaGetLastError());
  ctx->launches++;
  return 0;
}

int LaunchFcMode2(qcnn_layer* L, const FcPlan& p, const float* src, int N, float* dst, int relu, cudaStream_t st) {
  GemmArgs a = p.tc;
  a.src = src; a.dst = a.partial = dst; a.relu = relu;   // (partial: read with nsplit > 1 only)
  a.ctrd = a.cbPre ? L->d_ctrd_bf.as<float>() : L->d_ctrd.as<float>();
  a.asmt = L->d_asmt.as<uint8_t>(); a.bias = L->d_bias.as<float>();
  if (int rc = PrepFcPlanes(L, src, N, a.NT, kFcKs, a.nChunksAll, a.bf != 0, st)) return rc;
  a.xprep = L->d_flat.as<float>();
  return LaunchPqGemmArgs(L->ctx, a, static_cast<long long>(CeilDiv(N, a.NT)) * a.nsplit * a.nct, st, L->asmt_bits, L->asmt_pitch);
}

// [TN][PF][K] LUT slice + two buffers of the input slice (TN PF d floats, padded to 4) + two of the codebook rows (PF K d)
size_t FcGatherSmemBytes(int K, int tn, int d) {
  const size_t pf = FcChunkLen(K, tn);
  const size_t xpad = (static_cast<size_t>(tn) * pf * d + 3) & ~static_cast<size_t>(3);
  return sizeof(float) * (static_cast<size_t>(tn) * pf * K + 2 * xpad + 2 * pf * K * d);
}

// batch tile: 1 (latency path, 16 channels/thread, 128-bit loads), 4 or 8 images per CTA; fc_tn / fc_nsplit pin the tiling.
// Unpinned, the tile is the widest that fits in shared memory (K = 256: tn = 8 up to d = 8, 4 up to d = 10, else 1).
int PlanFcGather(const qcnn_layer* L, int N, FcPlan* p) {
  int tn = L->opt_fc_tn ? L->opt_fc_tn : (N >= 8 ? 8 : (N >= 4 ? 4 : 1));
  if (tn != 1 && tn != 4) tn = 8;
  if (!L->opt_fc_tn)
    while (tn > 1 && FcGatherSmemBytes(L->K, tn, L->d) > kFcGatherSmemMax) tn = tn == 8 ? 4 : 1;
  if (FcGatherSmemBytes(L->K, tn, L->d) > kFcGatherSmemMax) {
    SetError("qcnn_fc_aprx_forward: fc_tn=%d with K=%d d=%d needs %zu bytes of shared memory per CTA (limit %zu)", tn, L->K,
             L->d, FcGatherSmemBytes(L->K, tn, L->d), kFcGatherSmemMax);
    return 1;
  }
  // narrow layers (fc8: 1000 outputs) take 4 channels per thread so that a 256-thread CTA is fully populated
  const int cpt = (tn == 1) ? 16 : ((tn == 8 && L->DoutPad <= 1024) ? 4 : 8);
  const int pf = FcChunkLen(L->K, tn);
  const int chunks = CeilDiv(L->S, pf);
  int nsplit = L->opt_fc_nsplit;
  if (nsplit <= 0) {
    // aim for >= 3 CTAs of 8 warps per SM; never more splits than chunks
    const int want = 3 * L->ctx->sm_count;
    nsplit = CeilDiv(want, CeilDiv(L->DoutPad, kFcThreads * cpt) * CeilDiv(N, tn));
  }
  nsplit = std::max(1, std::min(nsplit, chunks));
  const int chunks_per_split = CeilDiv(chunks, nsplit);
  p->nsplit = CeilDiv(chunks, chunks_per_split);
  p->gather = {tn, cpt, chunks_per_split * pf};
  return 0;
}

// the tiling of a LUT + gather plan; describe() writes it after the layer's geometry (no " via ": the plain kernel)
void DescribeFcGather(const qcnn_layer* L, const FcPlan& p, int, char* buf, size_t cap) {
  snprintf(buf, cap, "gather(tn=%d cpt=%d pf=%d nsplit=%d)", p.gather.tn, p.gather.cpt, FcChunkLen(L->K, p.gather.tn),
           p.nsplit);
}

int LaunchFcGather(qcnn_layer* L, const FcPlan& p, const float* src, int N, float* dst, int relu, cudaStream_t st) {
  const int tn = p.gather.tn, cpt = p.gather.cpt;
  FcArgs a;
  a.src = src; a.dst = dst; a.partial = p.nsplit > 1 ? dst : nullptr;
  a.ctrd = L->d_ctrd.as<float>(); a.asmt = L->d_asmt.as<uint8_t>(); a.bias = L->d_bias.as<float>();
  a.N = N; a.Din = L->Din; a.Dout = L->Dout; a.DoutPad = L->DoutPad; a.S = L->S; a.K = L->K; a.d = L->d;
  a.srcoff = L->d_srcoff.as<int>();
  a.relu = relu;
  a.s_per_split = p.gather.sPerSplit;
  a.nsplit = p.nsplit;
  const dim3 grid(CeilDiv(L->DoutPad, kFcThreads * cpt), CeilDiv(N, tn), p.nsplit);
  const bool pre = L->kshift == 2;
  if (L->asmt_bits) {   // bit-packed table: same grid, chunking and splits as the byte table
    const int pt = L->asmt_pitch;
    switch (L->K) {
      case 16:  return LaunchK<16, false, true>(a, tn, cpt, grid, st, pt);
      case 32:  return LaunchK<32, false, true>(a, tn, cpt, grid, st, pt);
      case 64:  return LaunchK<64, false, true>(a, tn, cpt, grid, st, pt);
      case 128: return LaunchK<128, false, true>(a, tn, cpt, grid, st, pt);
      default:
        SetError("qcnn_fc_aprx_forward: no packed-table kernel for K=%d", L->K);
        return 1;
    }
  }
  switch (L->K) {
    case 16:  return pre ? LaunchK<16, true>(a, tn, cpt, grid, st) : LaunchK<16, false>(a, tn, cpt, grid, st);
    case 32:  return pre ? LaunchK<32, true>(a, tn, cpt, grid, st) : LaunchK<32, false>(a, tn, cpt, grid, st);
    case 64:  return pre ? LaunchK<64, true>(a, tn, cpt, grid, st) : LaunchK<64, false>(a, tn, cpt, grid, st);
    case 128: return LaunchK<128, false>(a, tn, cpt, grid, st);
    case 256: return LaunchK<256, false>(a, tn, cpt, grid, st);
    default:
      SetError("qcnn_fc_aprx_forward: unsupported codebook size K=%d (supported: 16, 32, 64, 128, 256)", L->K);
      return 1;
  }
}

}  // namespace qcnn
