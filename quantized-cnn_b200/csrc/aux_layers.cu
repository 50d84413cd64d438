// Supporting (non-PQ) layers of the forward pass, kept on the device so activations never bounce to the host.
// They replace the remaining CalcFeatMap_* loop nests and the OpenVML / cblas elementwise calls they make
// (reference src/CaffeEva.cc:870-921, 1027-1116; include/BlasWrapper.h:101-162).  All are HBM-streaming kernels:
// NHWC maps, channel index fastest across lanes (coalesced), grid-stride loops sized to the SM count.
#include "qcnn_internal.h"

#include <cstdlib>

namespace {

constexpr int kThreads = 256;

__global__ void relu_kernel(const float* __restrict__ src, float* __restrict__ dst, size_t n) {
  // CalcFeatMap_ReLu (CaffeEva.cc:1027-1036): max(0, x)
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
    dst[i] = fmaxf(src[i], 0.0f);
}

// CalcFeatMap_LoRN (CaffeEva.cc:1038-1089), same operation order as the reference:
//   t_c  = (x_c * x_c) * (alpha / size)                      vsSqr, cblas_sscal
//   sum  = k; sum += t_{c-rad+w} for w = 0..size-1            vsAdd over the zero-padded window
//   y_c  = x_c * expf(-beta * logf(sum))                      vsPowx_m fallback (BlasWrapper.h:134-147)
__device__ __forceinline__ float LrnAt(const float* __restrict__ px, int c, int C, int size, int rad, float coeff,
                                       float kini, float nbeta) {
  float sum = kini;
  for (int w = 0; w < size; w++) {
    const int cc = c - rad + w;
    float t = 0.0f;
    if (cc >= 0 && cc < C) {
      const float v = __ldg(px + cc);
      t = __fmul_rn(__fmul_rn(v, v), coeff);
    }
    sum = __fadd_rn(sum, t);
  }
  return __fmul_rn(__ldg(px + c), expf(__fmul_rn(nbeta, logf(sum))));
}

__global__ void lrn_kernel(const float* __restrict__ src, float* __restrict__ dst, size_t total, int C, int size,
                           float coeff, float kini, float nbeta) {
  const int rad = (size - 1) / 2;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const size_t p = i / C;
    const int c = static_cast<int>(i - p * C);
    dst[i] = LrnAt(src + p * C, c, C, size, rad, coeff, kini, nbeta);
  }
}

// CalcFeatMap_Pool (CaffeEva.cc:870-921): window clipped to the image, out = ceil((H+2p-k)/s)+1
__global__ void maxpool_kernel(const float* __restrict__ src, float* __restrict__ dst, int N, int H, int W, int C,
                               int Ho, int Wo, int ksz, int pad, int stride) {
  const size_t total = static_cast<size_t>(N) * Ho * Wo * C;
  const size_t gs = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += gs) {
    const int c = static_cast<int>(i % C);
    size_t t = i / C;
    const int wo = static_cast<int>(t % Wo); t /= Wo;
    const int ho = static_cast<int>(t % Ho);
    const int n = static_cast<int>(t / Ho);
    const int hL = max(0, ho * stride - pad), hU = min(H, ho * stride + ksz - pad) - 1;
    const int wL = max(0, wo * stride - pad), wU = min(W, wo * stride + ksz - pad) - 1;
    float m = -INFINITY;
    for (int h = hL; h <= hU; h++)
      for (int w = wL; w <= wU; w++)
        m = fmaxf(m, __ldg(src + ((static_cast<size_t>(n) * H + h) * W + w) * C + c));
    dst[i] = m;
  }
}

// LRN immediately followed by max-pool (AlexNet / VggCnnS order): the normalised map is never written.
__global__ void lrn_maxpool_kernel(const float* __restrict__ src, float* __restrict__ dst, int N, int H, int W, int C,
                                   int Ho, int Wo, int size, float coeff, float kini, float nbeta, int ksz, int pad,
                                   int stride) {
  const int rad = (size - 1) / 2;
  const size_t total = static_cast<size_t>(N) * Ho * Wo * C;
  const size_t gs = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += gs) {
    const int c = static_cast<int>(i % C);
    size_t t = i / C;
    const int wo = static_cast<int>(t % Wo); t /= Wo;
    const int ho = static_cast<int>(t % Ho);
    const int n = static_cast<int>(t / Ho);
    const int hL = max(0, ho * stride - pad), hU = min(H, ho * stride + ksz - pad) - 1;
    const int wL = max(0, wo * stride - pad), wU = min(W, wo * stride + ksz - pad) - 1;
    float m = -INFINITY;
    for (int h = hL; h <= hU; h++)
      for (int w = wL; w <= wU; w++)
        m = fmaxf(m, LrnAt(src + ((static_cast<size_t>(n) * H + h) * W + w) * C, c, C, size, rad, coeff, kini, nbeta));
    dst[i] = m;
  }
}

// 8 consecutive channels of one pixel at once: the squared/scaled window terms are computed once and shared by the
// 8 sliding sums (same per-output operation order as LrnAt / the reference).  C % 4 == 0, c0 % 8 == 0.
// FAST075: beta == 0.75 (every layer table of the reference, CaffePara.cc:31,35,...): sum^-0.75 = r * sqrt(r) with
// r = rsqrt(sum), both by the special-function unit -- within ~5 ulp of the reference's expf(-0.75 * logf(sum)) (itself
// ~4 ulp from the true value; the LRN parity tolerance is 1e-5, i.e. ~80 ulp) at a tenth of the instructions, which is
// what bounds this kernel.
template <int SIZE, bool FAST075>
__device__ __forceinline__ void LrnChunk8(const float* __restrict__ px, int c0, int C, float coeff, float kini,
                                          float nbeta, float (&out)[8]) {
  constexpr int RAD = (SIZE - 1) / 2;
  constexpr int LO = (RAD + 3) / 4 * 4;        // floats loaded below c0 (multiple of 4 so 128-bit loads stay aligned)
  constexpr int NV = (LO + 8 + LO) / 4;        // float4 loads
  float x[NV * 4];
#pragma unroll
  for (int v = 0; v < NV; v++) {
    const int cc = c0 - LO + 4 * v;
    float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
    if (cc >= 0 && cc < C) q = __ldg(reinterpret_cast<const float4*>(px + cc));
    x[4 * v] = q.x; x[4 * v + 1] = q.y; x[4 * v + 2] = q.z; x[4 * v + 3] = q.w;
  }
  float t[8 + 2 * RAD];
#pragma unroll
  for (int i = 0; i < 8 + 2 * RAD; i++) {
    const float v = x[LO - RAD + i];
    t[i] = __fmul_rn(__fmul_rn(v, v), coeff);
  }
#pragma unroll
  for (int c = 0; c < 8; c++) {
    float sum = kini;
#pragma unroll
    for (int w = 0; w < SIZE; w++) sum = __fadd_rn(sum, t[c + w]);
    if (FAST075) {
      // one MUFU.RSQ + one MUFU.SQRT (the IEEE square root costs ~10 instructions and a slow-path call per value, and
      // instruction issue is what bounds this kernel); sum >= k >= 1e-20 (checked by the launcher): no denormals
      float r, q;
      asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(sum));
      asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(q) : "f"(r));
      out[c] = __fmul_rn(x[LO + c], __fmul_rn(r, q));
    } else {
      out[c] = __fmul_rn(x[LO + c], expf(__fmul_rn(nbeta, logf(sum))));
    }
  }
}

// Tiled variant: one CTA per (image, `ro` output rows).  The input rows those output rows need are normalised ONCE
// into shared memory and then pooled, so the power function runs ~((ro-1)*stride+ksz)/(ro*stride) times per input element
// instead of ksz^2/stride^2 times, and the normalised map still never reaches HBM.
template <int SIZE, bool FAST075, bool K3>
__global__ void __launch_bounds__(512, 3) lrn_maxpool_tiled_kernel(const float* __restrict__ src, float* __restrict__ dst, int H, int W, int C,
                                         int Ho, int Wo, int size, float coeff, float kini, float nbeta, int ksz,
                                         int pad, int stride, int ro) {
  extern __shared__ __align__(16) float tile[];  // [rows][W][C]
  const int ho0 = blockIdx.x * ro, n = blockIdx.y;
  const int hoN = min(Ho, ho0 + ro);
  const int hL = max(0, ho0 * stride - pad), hU = min(H, (hoN - 1) * stride + ksz - pad) - 1;
  const int rows = hU - hL + 1;
  const int rowLen = W * C;
  const float* base = src + (static_cast<size_t>(n) * H + hL) * rowLen;
  const int nthr = blockDim.x;
  if (SIZE > 0) {
    // (pixel, 8-channel chunk) pairs walked incrementally: one division per thread, none per element
    const int cpp = C >> 3, npix = rows * W;
    int p = threadIdx.x / cpp, ch = threadIdx.x - p * cpp;
    const int dp = nthr / cpp, dc = nthr - dp * cpp;
    while (p < npix) {
      float o[8];
      LrnChunk8<(SIZE > 0 ? SIZE : 1), FAST075>(base + static_cast<size_t>(p) * C, ch << 3, C, coeff, kini, nbeta, o);
      float4* tp = reinterpret_cast<float4*>(tile + static_cast<size_t>(p) * C + (ch << 3));
      tp[0] = make_float4(o[0], o[1], o[2], o[3]);
      tp[1] = make_float4(o[4], o[5], o[6], o[7]);
      p += dp; ch += dc;
      if (ch >= cpp) { ch -= cpp; p++; }
    }
  } else {
    const int rad = (size - 1) / 2;
    for (int e = threadIdx.x; e < rows * rowLen; e += nthr) {
      const int p = e / C, c = e - p * C;
      tile[e] = LrnAt(base + static_cast<size_t>(p) * C, c, C, size, rad, coeff, kini, nbeta);
    }
  }
  __syncthreads();
  const int rowOut = Wo * C;
  float* out = dst + (static_cast<size_t>(n) * Ho + ho0) * rowOut;
  if ((C & 3) == 0) {
    // four channels per thread: 128-bit shared-memory reads and global stores; (row, column, channel quad) walked
    // incrementally.  K3: 3x3 window with the clipped taps CLAMPED into the window (max is idempotent): nine reads, no branches
    const int c4n = C >> 2, rowOut4 = Wo * c4n;
    const float4* tile4 = reinterpret_cast<const float4*>(tile);
    float4* out4 = reinterpret_cast<float4*>(out);
    int e = threadIdx.x;
    int r0 = e / rowOut4, rem = e - r0 * rowOut4;
    int wo = rem / c4n, c4 = rem - wo * c4n;
    const int dwo = nthr / c4n, dc4 = nthr - dwo * c4n;
    const int total = (hoN - ho0) * rowOut4;
    for (; e < total; e += nthr) {
      const int ho = ho0 + r0;
      const int rL = max(0, ho * stride - pad) - hL, rU = min(H, ho * stride + ksz - pad) - 1 - hL;
      const int wL = max(0, wo * stride - pad), wU = min(W, wo * stride + ksz - pad) - 1;
      float4 m;
      if (K3) {
        const int rM = min(rL + 1, rU), wM = min(wL + 1, wU);
        const float4* t0 = tile4 + rL * W * c4n + c4;
        const float4* t1 = tile4 + rM * W * c4n + c4;
        const float4* t2 = tile4 + rU * W * c4n + c4;
        const int o0 = wL * c4n, o1 = wM * c4n, o2 = wU * c4n;
        const float4 a0 = t0[o0], a1 = t0[o1], a2 = t0[o2];
        const float4 b0 = t1[o0], b1 = t1[o1], b2 = t1[o2];
        const float4 d0 = t2[o0], d1 = t2[o1], d2 = t2[o2];
#define QCNN_MAX9(f) fmaxf(fmaxf(fmaxf(a0.f, a1.f), fmaxf(a2.f, b0.f)), fmaxf(fmaxf(b1.f, b2.f), fmaxf(fmaxf(d0.f, d1.f), d2.f)))
        m = make_float4(QCNN_MAX9(x), QCNN_MAX9(y), QCNN_MAX9(z), QCNN_MAX9(w));
#undef QCNN_MAX9
      } else {
        m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
        for (int r = rL; r <= rU; r++)
          for (int w = wL; w <= wU; w++) {
            const float4 v = tile4[(r * W + w) * c4n + c4];
            m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
          }
      }
      out4[e] = m;
      wo += dwo; c4 += dc4;
      if (c4 >= c4n) { c4 -= c4n; wo++; }
      while (wo >= Wo) { wo -= Wo; r0++; }
    }
    return;
  }
  for (int e = threadIdx.x; e < (hoN - ho0) * rowOut; e += nthr) {
    const int r0 = e / rowOut, rem = e - r0 * rowOut;
    const int wo = rem / C, c = rem - wo * C;
    const int ho = ho0 + r0;
    const int rL = max(0, ho * stride - pad) - hL, rU = min(H, ho * stride + ksz - pad) - 1 - hL;
    const int wL = max(0, wo * stride - pad), wU = min(W, wo * stride + ksz - pad) - 1;
    float m = -INFINITY;
    for (int r = rL; r <= rU; r++)
      for (int w = wL; w <= wU; w++) m = fmaxf(m, tile[(r * W + w) * C + c]);
    out[e] = m;
  }
}

// Max-pool of an NHWC map with C % 4 == 0: one thread per output channel quad, 128-bit loads; 3x3 windows read their
// clipped taps clamped into the window (nine loads, no branches).  Same result as maxpool_kernel.
template <bool K3>
__global__ void maxpool4_kernel(const float4* __restrict__ src, float4* __restrict__ dst, int N, int H, int W, int c4n,
                                int Ho, int Wo, int ksz, int pad, int stride) {
  const size_t total = static_cast<size_t>(N) * Ho * Wo * c4n;
  const size_t gs = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += gs) {
    const int c4 = static_cast<int>(i % c4n);
    size_t t = i / c4n;
    const int wo = static_cast<int>(t % Wo); t /= Wo;
    const int ho = static_cast<int>(t % Ho);
    const int n = static_cast<int>(t / Ho);
    const int hL = max(0, ho * stride - pad), hU = min(H, ho * stride + ksz - pad) - 1;
    const int wL = max(0, wo * stride - pad), wU = min(W, wo * stride + ksz - pad) - 1;
    const float4* img = src + static_cast<size_t>(n) * H * W * c4n + c4;
    float4 m;
    if (K3) {
      const int hM = min(hL + 1, hU), wM = min(wL + 1, wU);
      const float4* t0 = img + static_cast<size_t>(hL) * W * c4n;
      const float4* t1 = img + static_cast<size_t>(hM) * W * c4n;
      const float4* t2 = img + static_cast<size_t>(hU) * W * c4n;
      const int o0 = wL * c4n, o1 = wM * c4n, o2 = wU * c4n;
      const float4 a0 = __ldg(t0 + o0), a1 = __ldg(t0 + o1), a2 = __ldg(t0 + o2);
      const float4 b0 = __ldg(t1 + o0), b1 = __ldg(t1 + o1), b2 = __ldg(t1 + o2);
      const float4 d0 = __ldg(t2 + o0), d1 = __ldg(t2 + o1), d2 = __ldg(t2 + o2);
#define QCNN_MAX9(f) fmaxf(fmaxf(fmaxf(a0.f, a1.f), fmaxf(a2.f, b0.f)), fmaxf(fmaxf(b1.f, b2.f), fmaxf(fmaxf(d0.f, d1.f), d2.f)))
      m = make_float4(QCNN_MAX9(x), QCNN_MAX9(y), QCNN_MAX9(z), QCNN_MAX9(w));
#undef QCNN_MAX9
    } else {
      m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
      for (int h = hL; h <= hU; h++)
        for (int w = wL; w <= wU; w++) {
          const float4 v = __ldg(img + (static_cast<size_t>(h) * W + w) * c4n);
          m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
        }
    }
    dst[i] = m;
  }
}

// CalcFeatMap_SMax (CaffeEva.cc:1098-1116): y = exp(x) / sum(exp(x)), NO max subtraction (kept: parity).
// One CTA per image; the float sum is reduced in a fixed tree order (deterministic).
__global__ void softmax_kernel(const float* __restrict__ src, float* __restrict__ dst, int C) {
  __shared__ float red[kThreads / 32];
  __shared__ float total;
  const float* x = src + static_cast<size_t>(blockIdx.x) * C;
  float* y = dst + static_cast<size_t>(blockIdx.x) * C;
  float part = 0.0f;
  for (int c = threadIdx.x; c < C; c += kThreads) {
    const float e = expf(x[c]);
    y[c] = e;
    part += e;
  }
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = part;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.0f;
    for (int w = 0; w < kThreads / 32; w++) s += red[w];
    total = s;
  }
  __syncthreads();
  const float s = total;
  for (int c = threadIdx.x; c < C; c += kThreads) y[c] = __fdiv_rn(y[c], s);
}

// Matrix::Permute(0,2,3,1) / (0,3,1,2) call sites (CaffeEva.cc:225-228, 236-238)
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ src, float* __restrict__ dst, int N, int C, int H, int W) {
  const size_t total = static_cast<size_t>(N) * C * H * W;
  const size_t gs = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += gs) {
    // i indexes dst (NHWC)
    const int c = static_cast<int>(i % C);
    size_t t = i / C;
    const int w = static_cast<int>(t % W); t /= W;
    const int h = static_cast<int>(t % H);
    const int n = static_cast<int>(t / H);
    dst[i] = __ldg(src + ((static_cast<size_t>(n) * C + c) * H + h) * W + w);
  }
}
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ src, float* __restrict__ dst, int N, int H, int W, int C) {
  const size_t total = static_cast<size_t>(N) * C * H * W;
  const size_t gs = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += gs) {
    // i indexes dst (NCHW)
    const int w = static_cast<int>(i % W);
    size_t t = i / W;
    const int h = static_cast<int>(t % H); t /= H;
    const int c = static_cast<int>(t % C);
    const int n = static_cast<int>(t / C);
    dst[i] = __ldg(src + ((static_cast<size_t>(n) * H + h) * W + w) * C + c);
  }
}

int GridFor(const qcnn_ctx* ctx, size_t total) {
  const size_t want = (total + kThreads - 1) / kThreads;
  const size_t cap = static_cast<size_t>(ctx->sm_count) * 8;  // 8 CTAs of 256 threads per SM, grid-stride beyond
  return static_cast<int>(std::max<size_t>(1, std::min(want, cap)));
}

}  // namespace

namespace qcnn {

int LaunchRelu(qcnn_ctx* ctx, const float* src, float* dst, size_t n, cudaStream_t st) {
  if (n == 0) return 0;
  relu_kernel<<<GridFor(ctx, n), kThreads, 0, st>>>(src, dst, n);
  QCNN_CUDA(cudaGetLastError());
  ctx->launches++;
  return 0;
}

int LaunchLrn(qcnn_ctx* ctx, const float* src, float* dst, size_t pixels, int C, int size, float alpha, float beta,
              float k, cudaStream_t st) {
  QCNN_CHECK(C >= 1 && size >= 1, "qcnn_lrn: bad arguments");
  const size_t total = pixels * C;
  if (total == 0) return 0;
  lrn_kernel<<<GridFor(ctx, total), kThreads, 0, st>>>(src, dst, total, C, size, alpha / size, k, -beta);
  QCNN_CUDA(cudaGetLastError());
  ctx->launches++;
  return 0;
}

int LaunchMaxPool(qcnn_ctx* ctx, const float* src, float* dst, int N, int H, int W, int C, int ksz, int pad,
                  int stride, cudaStream_t st) {
  QCNN_CHECK(N >= 1 && ksz >= 1 && stride >= 1, "qcnn_maxpool: bad arguments");
  QCNN_CHECK(PoolWindowsNonEmpty(H, pad, ksz, stride) && PoolWindowsNonEmpty(W, pad, ksz, stride),
             "qcnn_maxpool: %dx%d map, %dx%d window, pad %d, stride %d: an output window holds no input pixel", H, W, ksz,
             ksz, pad, stride);
  const int Ho = PoolOut(H, pad, ksz, stride), Wo = PoolOut(W, pad, ksz, stride);
  const size_t total = static_cast<size_t>(N) * Ho * Wo * C;
  // (fmaxf of a window that contains a NaN: both kernels return the maximum of the other taps, in any order)
  if ((C & 3) == 0) {
    const size_t total4 = total / 4;
    if (ksz == 3 && stride <= 3 && pad <= 2) maxpool4_kernel<true><<<GridFor(ctx, total4), kThreads, 0, st>>>(reinterpret_cast<const float4*>(src), reinterpret_cast<float4*>(dst), N, H, W, C / 4, Ho, Wo, ksz, pad, stride);
    else maxpool4_kernel<false><<<GridFor(ctx, total4), kThreads, 0, st>>>(reinterpret_cast<const float4*>(src), reinterpret_cast<float4*>(dst), N, H, W, C / 4, Ho, Wo, ksz, pad, stride);
  } else {
    maxpool_kernel<<<GridFor(ctx, total), kThreads, 0, st>>>(src, dst, N, H, W, C, Ho, Wo, ksz, pad, stride);
  }
  QCNN_CUDA(cudaGetLastError());
  ctx->launches++;
  return 0;
}

int LaunchLrnMaxPool(qcnn_ctx* ctx, const float* src, float* dst, int N, int H, int W, int C, int size, float alpha,
                     float beta, float k, int ksz, int pad, int stride, cudaStream_t st) {
  QCNN_CHECK(N >= 1 && ksz >= 1 && stride >= 1 && size >= 1, "qcnn_lrn_maxpool: bad arguments");
  QCNN_CHECK(PoolWindowsNonEmpty(H, pad, ksz, stride) && PoolWindowsNonEmpty(W, pad, ksz, stride),
             "qcnn_lrn_maxpool: %dx%d map, %dx%d window, pad %d, stride %d: an output window holds no input pixel", H, W,
             ksz, ksz, pad, stride);
  const int Ho = PoolOut(H, pad, ksz, stride), Wo = PoolOut(W, pad, ksz, stride);
  const size_t total = static_cast<size_t>(N) * Ho * Wo * C;
  // output rows per CTA: as many as keep two CTAs per SM (less re-normalisation of shared input rows)
  int ro = 1;
  static const int roMax = getenv("QCNN_LRN_RO") ? atoi(getenv("QCNN_LRN_RO")) : 1;
  static const int lrnThreads = getenv("QCNN_LRN_THREADS") ? atoi(getenv("QCNN_LRN_THREADS")) : 512;   // threads per CTA of the LRN kernels
  while (ro < roMax && ro < Ho && sizeof(float) * static_cast<size_t>(ro * stride + ksz) * W * C <= 110 * 1024) ro++;
  const size_t tileBytes = sizeof(float) * static_cast<size_t>((ro - 1) * stride + ksz) * W * C;
  if (tileBytes <= 160 * 1024 && N <= 65535) {
    // specialised 8-channel path for the 5-wide window every reference table uses (CaffePara.cc:31,35,...)
    const bool fast = beta == 0.75f && k >= 1e-20f && alpha >= 0.0f;
    const bool k3 = ksz == 3 && C % 4 == 0 && stride <= 3 && pad <= 2;   // (no empty windows: the clamped taps stay inside)
    auto kern = (size == 5 && C % 8 == 0)
                    ? (fast ? (k3 ? lrn_maxpool_tiled_kernel<5, true, true> : lrn_maxpool_tiled_kernel<5, true, false>)
                            : (k3 ? lrn_maxpool_tiled_kernel<5, false, true> : lrn_maxpool_tiled_kernel<5, false, false>))
                    : lrn_maxpool_tiled_kernel<0, false, false>;
    if (tileBytes > 48 * 1024)
      QCNN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tileBytes));
    kern<<<dim3(CeilDiv(Ho, ro), N), lrnThreads, tileBytes, st>>>(src, dst, H, W, C, Ho, Wo, size, alpha / size, k, -beta,
                                                                ksz, pad, stride, ro);
  } else {
    lrn_maxpool_kernel<<<GridFor(ctx, total), kThreads, 0, st>>>(src, dst, N, H, W, C, Ho, Wo, size, alpha / size, k,
                                                                 -beta, ksz, pad, stride);
  }
  QCNN_CUDA(cudaGetLastError());
  ctx->launches++;
  return 0;
}

int LaunchSoftmax(qcnn_ctx* ctx, const float* src, float* dst, int N, int C, cudaStream_t st) {
  QCNN_CHECK(N >= 1 && C >= 1, "qcnn_softmax: bad arguments");
  softmax_kernel<<<N, kThreads, 0, st>>>(src, dst, C);
  QCNN_CUDA(cudaGetLastError());
  ctx->launches++;
  return 0;
}

int LaunchNchwToNhwc(qcnn_ctx* ctx, const float* src, float* dst, int N, int C, int H, int W, cudaStream_t st) {
  const size_t total = static_cast<size_t>(N) * C * H * W;
  nchw_to_nhwc_kernel<<<GridFor(ctx, total), kThreads, 0, st>>>(src, dst, N, C, H, W);
  QCNN_CUDA(cudaGetLastError());
  ctx->launches++;
  return 0;
}

int LaunchNhwcToNchw(qcnn_ctx* ctx, const float* src, float* dst, int N, int H, int W, int C, cudaStream_t st) {
  const size_t total = static_cast<size_t>(N) * C * H * W;
  nhwc_to_nchw_kernel<<<GridFor(ctx, total), kThreads, 0, st>>>(src, dst, N, H, W, C);
  QCNN_CUDA(cudaGetLastError());
  ctx->launches++;
  return 0;
}

}  // namespace qcnn
