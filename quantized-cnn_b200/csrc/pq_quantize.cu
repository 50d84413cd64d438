// Product quantization of dense conv / FC weights on the device: per subspace, Lloyd k-means over the weight sub-vectors
// (the paper's quantization without error correction).  Output is what CaffePara::LoadLayerPara(true, ...) holds:
// ctrdLst [S][K][d], asmtLst [Cout][k][k][S] / [Dout][S] (0-based).  Semantics, normative (DESIGN.md 4e):
//   points     conv p = (o k + kh) k + kw, x_p[j] = knl[o][s d + j][kh][kw], j < w_s = min(d, Cg - s d); FC is conv with
//              k = 1 and Cg = Din.  One codebook per subspace is shared by all groups (src/CaffeEva.cc:795-811).
//   distance   fp32, ascending j, no contraction; argmin with the lowest index winning ties.
//   update     c_k[j] = (float)(sum_{a_p = k} (double) x_p[j] / n_k) in a fixed order; empty clusters keep their codeword.
//   iterations a_0 = assign(C_0); C_t = update(a_{t-1}, C_{t-1}), a_t = assign(C_t) for t = 1..iters.
// Nothing depends on timing, atomics on floating-point values, or thread order, so every result is reproducible bit for
// bit.  All iterations are stream-ordered launches; the host waits once, when the results are copied back.
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <unordered_map>
#include <vector>

#include "../host/CaffePara.h"
#include "../host/FileIO.h"
#include "qcnn_internal.h"

using namespace qcnn;

namespace {

constexpr int kMaxD = 64;            // widest sub-vector
constexpr int kMaxK = 256;           // uint8 assignments
constexpr int kMaxP = 1 << 24;       // the LCG's (x >> 8) draws 24 bits
constexpr int kAssignThreads = 128;
constexpr int kUpdateThreads = 256;
constexpr int kUpdateChunk = 1024;   // points per CTA of the update's partial sums

// Points and codewords are padded to D = 4, 8, 16, 32 or 64 floats with zeros.  A padded dim adds t * t = +0 to a
// non-negative fp32 sum, which leaves it bit-identical, so the distance loops need no bound on the valid dims.
int PadDims(int w) {
  int D = 4;
  while (D < w) D *= 2;
  return D;
}

// weights [Cout][Cg][k][k] -> points [S][P][D], zero past each subspace's valid dims
__global__ void pq_relayout_kernel(const float* __restrict__ w, float* __restrict__ x, int Cg, int taps, int S, int P,
                                   int d, int D) {
  const size_t total = static_cast<size_t>(S) * P * D;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int j = static_cast<int>(i % D);
    const size_t sp = i / D;
    const int p = static_cast<int>(sp % P), s = static_cast<int>(sp / P);
    const int c = s * d + j;
    float v = 0.0f;
    if (j < d && c < Cg) {
      const int o = p / taps, t = p % taps;
      v = w[(static_cast<size_t>(o) * Cg + c) * taps + t];
    }
    x[i] = v;
  }
}

// Deterministic sum of one double per thread: a fixed shuffle tree per warp, then the warps in ascending order.
template <int THREADS>
__device__ double BlockSumFixed(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double r = 0.0;
  if (threadIdx.x == 0)
    for (int i = 0; i < THREADS / 32; i++) r += red[i];
  return r;
}

// Assignment of R points per thread to the nearest codeword of their subspace.  The codebook sits in shared memory and
// every codeword read (one broadcast 16-byte load per four dims) serves the thread's R points.  Writes each CTA's fp64
// sum of the minimum distances to sse_part[blockIdx.y * gridDim.x + blockIdx.x].
template <int D, int R>
__global__ void __launch_bounds__(kAssignThreads) pq_assign_kernel(const float* __restrict__ x, const float* __restrict__ cb,
                                                                   uint8_t* __restrict__ a, double* __restrict__ sse_part,
                                                                   int P, int K) {
  extern __shared__ float4 sc[];   // [K][D / 4], then the block sum's kAssignThreads / 32 doubles (all shared memory is
                                   // dynamic: the opt-in limit is for dynamic plus static)
  constexpr int Q = D / 4;
  double* red = reinterpret_cast<double*>(sc + K * Q);
  const int s = blockIdx.y;
  const float4* c4 = reinterpret_cast<const float4*>(cb + static_cast<size_t>(s) * K * D);
  for (int i = threadIdx.x; i < K * Q; i += kAssignThreads) sc[i] = c4[i];
  const int p0 = blockIdx.x * (kAssignThreads * R) + threadIdx.x;
  float4 xv[R][Q];
#pragma unroll
  for (int r = 0; r < R; r++) {
    const int p = p0 + r * kAssignThreads;
    const float4* src = reinterpret_cast<const float4*>(x + (static_cast<size_t>(s) * P + (p < P ? p : 0)) * D);
#pragma unroll
    for (int q = 0; q < Q; q++) xv[r][q] = src[q];
  }
  __syncthreads();
  float best[R];
  int bi[R];
#pragma unroll
  for (int r = 0; r < R; r++) { best[r] = INFINITY; bi[r] = 0; }
  for (int k = 0; k < K; k++) {
    float acc[R];
#pragma unroll
    for (int r = 0; r < R; r++) acc[r] = 0.0f;
#pragma unroll
    for (int q = 0; q < Q; q++) {
      const float4 cv = sc[k * Q + q];
#pragma unroll
      for (int r = 0; r < R; r++) {
        float t = __fsub_rn(xv[r][q].x, cv.x);
        acc[r] = __fadd_rn(acc[r], __fmul_rn(t, t));
        t = __fsub_rn(xv[r][q].y, cv.y);
        acc[r] = __fadd_rn(acc[r], __fmul_rn(t, t));
        t = __fsub_rn(xv[r][q].z, cv.z);
        acc[r] = __fadd_rn(acc[r], __fmul_rn(t, t));
        t = __fsub_rn(xv[r][q].w, cv.w);
        acc[r] = __fadd_rn(acc[r], __fmul_rn(t, t));
      }
    }
#pragma unroll
    for (int r = 0; r < R; r++)
      if (acc[r] < best[r]) { best[r] = acc[r]; bi[r] = k; }
  }
  double part = 0.0;
#pragma unroll
  for (int r = 0; r < R; r++) {
    const int p = p0 + r * kAssignThreads;
    if (p < P) {
      a[static_cast<size_t>(s) * P + p] = static_cast<uint8_t>(bi[r]);
      part += static_cast<double>(best[r]);
    }
  }
  const double tot = BlockSumFixed<kAssignThreads>(part, red);
  if (threadIdx.x == 0) sse_part[static_cast<size_t>(blockIdx.y) * gridDim.x + blockIdx.x] = tot;
}

// Per (subspace, chunk of kUpdateChunk points): a stable counting sort of the chunk's points by cluster, then one fp64
// sum per (cluster, dim) over the cluster's points in ascending point order.  Partials [S][chunks][K][D], counts
// [S][chunks][K].
__global__ void __launch_bounds__(kUpdateThreads) pq_update_partial_kernel(const float* __restrict__ x,
                                                                           const uint8_t* __restrict__ a,
                                                                           double* __restrict__ sum_part,
                                                                           int* __restrict__ cnt_part, int P, int K, int D) {
  __shared__ uint8_t sa[kUpdateChunk];
  __shared__ short order[kUpdateChunk];
  __shared__ int cnt[kMaxK], beg[kMaxK + 1], cur[kMaxK];
  const int s = blockIdx.y, chunk = blockIdx.x, chunks = gridDim.x;
  const int base = chunk * kUpdateChunk, n = min(kUpdateChunk, P - base);
  for (int k = threadIdx.x; k < K; k += kUpdateThreads) cnt[k] = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += kUpdateThreads) {
    const uint8_t v = a[static_cast<size_t>(s) * P + base + i];
    sa[i] = v;
    atomicAdd(&cnt[v], 1);   // integer counts: the same in any order
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int k = 0; k < K; k++) { beg[k] = acc; cur[k] = acc; acc += cnt[k]; }
    beg[K] = acc;
  }
  __syncthreads();
  if (threadIdx.x < 32) {   // one warp places the points, 32 at a time, in ascending order within each cluster
    const int lane = threadIdx.x;
    for (int i0 = 0; i0 < n; i0 += 32) {
      const int i = i0 + lane;
      const bool valid = i < n;
      const int c = valid ? sa[i] : kMaxK + lane;
      const unsigned peers = __match_any_sync(0xffffffffu, c);
      const int rank = __popc(peers & ((1u << lane) - 1u));
      if (valid) order[cur[c] + rank] = static_cast<short>(i);
      __syncwarp();
      if (valid && rank == 0) cur[c] += __popc(peers);
      __syncwarp();
    }
  }
  __syncthreads();
  const float* xs = x + (static_cast<size_t>(s) * P + base) * D;
  double* out = sum_part + (static_cast<size_t>(s) * chunks + chunk) * K * D;
  for (int e = threadIdx.x; e < K * D; e += kUpdateThreads) {
    const int k = e / D, j = e % D;
    double acc = 0.0;
    for (int q = beg[k]; q < beg[k + 1]; q++) acc += static_cast<double>(xs[static_cast<size_t>(order[q]) * D + j]);
    out[e] = acc;
  }
  for (int k = threadIdx.x; k < K; k += kUpdateThreads)
    cnt_part[(static_cast<size_t>(s) * chunks + chunk) * K + k] = cnt[k];
}

// New codeword (s, k = blockIdx.x): partials combined in ascending chunk order; an empty cluster keeps its codeword.
__global__ void pq_update_final_kernel(const double* __restrict__ sum_part, const int* __restrict__ cnt_part,
                                       float* __restrict__ cb, int K, int D, int chunks) {
  const int s = blockIdx.y, k = blockIdx.x, j = threadIdx.x;
  if (j >= D) return;
  long long n = 0;
  double sum = 0.0;
  for (int c = 0; c < chunks; c++) {
    const size_t pc = (static_cast<size_t>(s) * chunks + c) * K + k;
    n += cnt_part[pc];
    sum += sum_part[pc * D + j];
  }
  if (n > 0) cb[(static_cast<size_t>(s) * K + k) * D + j] = static_cast<float>(sum / static_cast<double>(n));
}

// sse[t] = sum of the assignment CTAs' partials of step t, in a fixed order
__global__ void __launch_bounds__(kUpdateThreads) pq_sse_reduce_kernel(const double* __restrict__ sse_part,
                                                                       double* __restrict__ sse, int per_step) {
  __shared__ double red[kUpdateThreads / 32];
  const double* p = sse_part + static_cast<size_t>(blockIdx.x) * per_step;
  double v = 0.0;
  for (int i = threadIdx.x; i < per_step; i += kUpdateThreads) v += p[i];
  const double tot = BlockSumFixed<kUpdateThreads>(v, red);
  if (threadIdx.x == 0) sse[blockIdx.x] = tot;
}

typedef void (*AssignKernel)(const float*, const float*, uint8_t*, double*, int, int);

// Points per thread: as many as the registers allow (R * D <= 128 floats) while the grid still gives every SM two CTAs,
// and at least two
template <int D>
int PickAssign(qcnn_ctx* ctx, int S, int P, AssignKernel* kern, int* R) {
  constexpr int Rmax = D <= 16 ? 8 : 128 / D;
  int r = Rmax;
  while (r > 2 && static_cast<long long>(S) * CeilDiv(P, kAssignThreads * r) < 2LL * ctx->sm_count) r /= 2;
  *R = r;
  if constexpr (Rmax >= 8)
    if (r == 8) { *kern = pq_assign_kernel<D, 8>; return OptInSmem<pq_assign_kernel<D, 8>>(ctx); }
  if constexpr (Rmax >= 4)
    if (r == 4) { *kern = pq_assign_kernel<D, 4>; return OptInSmem<pq_assign_kernel<D, 4>>(ctx); }
  *kern = pq_assign_kernel<D, 2>;
  return OptInSmem<pq_assign_kernel<D, 2>>(ctx);
}

int PickAssignKernel(qcnn_ctx* ctx, int D, int S, int P, AssignKernel* kern, int* R) {
  switch (D) {
    case 4: return PickAssign<4>(ctx, S, P, kern, R);
    case 8: return PickAssign<8>(ctx, S, P, kern, R);
    case 16: return PickAssign<16>(ctx, S, P, kern, R);
    case 32: return PickAssign<32>(ctx, S, P, kern, R);
    default: return PickAssign<64>(ctx, S, P, kern, R);
  }
}

bool AllFinite(const float* v, size_t n) {
  for (size_t i = 0; i < n; i++)
    if (!isfinite(v[i])) return false;
  return true;
}

// One layer: weights [Cout][Cg][k][k] (FC: k = 1, Cg = Din).  K and d are checked by the entry points.
int Quantize(qcnn_ctx* ctx, const char* who, int Cout, int Cg, int ksz, int K, int d, int iters, uint32_t seed,
             const float* w_h, const float* init_h, float* ctrd_h, uint8_t* asmt_h, double* sse_h) {
  QCNN_CHECK(ctx && w_h && ctrd_h && asmt_h, "%s: NULL argument", who);
  QCNN_CHECK(Cout >= 1 && Cg >= 1 && ksz >= 1, "%s: bad dimensions", who);
  QCNN_CHECK(d >= 1 && d <= kMaxD, "%s: d=%d is outside 1..%d", who, d, kMaxD);
  QCNN_CHECK(iters >= 0, "%s: iters=%d is negative", who, iters);
  const int taps = ksz * ksz;
  const long long P64 = static_cast<long long>(Cout) * taps;
  QCNN_CHECK(P64 <= kMaxP, "%s: %lld points per subspace exceed 2^24", who, P64);
  const int P = static_cast<int>(P64), S = CeilDiv(Cg, d), D = PadDims(std::min(d, Cg));
  QCNN_CHECK(init_h || P >= K, "%s: %d points per subspace cannot seed K=%d distinct codewords", who, P, K);
  const size_t nw = static_cast<size_t>(P) * Cg;
  QCNN_CHECK(AllFinite(w_h, nw), "%s: the weights contain a non-finite value", who);
  QCNN_CHECK(!init_h || AllFinite(init_h, static_cast<size_t>(S) * K * d), "%s: the initial codebook contains a non-finite value",
             who);
  // C_0 on the host, [S][K][D]: the given codebook, or K distinct points drawn by the project's LCG
  std::vector<float> cb(static_cast<size_t>(S) * K * D, 0.0f);
  for (int s = 0; s < S; s++) {
    const int ws = std::min(d, Cg - s * d);
    uint32_t xr = seed + static_cast<uint32_t>(s);
    std::unordered_map<int, int> perm;   // the entries of [0, 1, ..., P-1] that the partial shuffle moved
    auto at = [&perm](int i) { auto it = perm.find(i); return it == perm.end() ? i : it->second; };
    for (int k = 0; k < K; k++) {
      float* c = &cb[(static_cast<size_t>(s) * K + k) * D];
      if (init_h) {
        for (int j = 0; j < ws; j++) c[j] = init_h[(static_cast<size_t>(s) * K + k) * d + j];
        continue;
      }
      xr = 1664525u * xr + 1013904223u;
      const int j = k + static_cast<int>((xr >> 8) % static_cast<uint32_t>(P - k));
      const int pk = at(j), pj = at(k);
      perm[k] = pk;
      perm[j] = pj;
      const int o = pk / taps, t = pk % taps;
      for (int jj = 0; jj < ws; jj++) c[jj] = w_h[(static_cast<size_t>(o) * Cg + s * d + jj) * taps + t];
    }
  }
  QCNN_ON_DEVICE(ctx->device);
  AssignKernel assign = nullptr;
  int R = 1;
  if (int rc = PickAssignKernel(ctx, D, S, P, &assign, &R)) return rc;
  const int chunksA = CeilDiv(P, kAssignThreads * R), chunksU = CeilDiv(P, kUpdateChunk);
  const size_t perStep = static_cast<size_t>(S) * chunksA;
  DeviceBuffer dw, dx, dcb, da, dsum, dcnt, dssep, dsse;
  QCNN_CUDA(dw.Upload(ctx, w_h, sizeof(float) * nw));
  QCNN_CUDA(dx.Reserve(ctx, sizeof(float) * S * static_cast<size_t>(P) * D));
  QCNN_CUDA(dcb.Upload(ctx, cb.data(), sizeof(float) * cb.size()));
  QCNN_CUDA(da.Reserve(ctx, static_cast<size_t>(S) * P));
  QCNN_CUDA(dsum.Reserve(ctx, sizeof(double) * S * static_cast<size_t>(chunksU) * K * D));
  QCNN_CUDA(dcnt.Reserve(ctx, sizeof(int) * S * static_cast<size_t>(chunksU) * K));
  QCNN_CUDA(dssep.Reserve(ctx, sizeof(double) * perStep * (iters + 1)));
  QCNN_CUDA(dsse.Reserve(ctx, sizeof(double) * (iters + 1)));
  const size_t nx = static_cast<size_t>(S) * P * D;
  const int relayoutBlocks = static_cast<int>(std::min<size_t>((nx + 255) / 256, 32u * ctx->sm_count));
  pq_relayout_kernel<<<relayoutBlocks, 256>>>(dw.as<float>(), dx.as<float>(), Cg, taps, S, P, d, D);
  QCNN_CUDA(cudaGetLastError());
  const size_t smemA = sizeof(float) * K * D + sizeof(double) * (kAssignThreads / 32);
  const dim3 gridA(chunksA, S), gridU(chunksU, S), gridF(K, S);
  for (int t = 0; t <= iters; t++) {
    if (t > 0) {
      pq_update_partial_kernel<<<gridU, kUpdateThreads>>>(dx.as<float>(), da.as<uint8_t>(), dsum.as<double>(), dcnt.as<int>(),
                                                         P, K, D);
      pq_update_final_kernel<<<gridF, kMaxD>>>(dsum.as<double>(), dcnt.as<int>(), dcb.as<float>(), K, D, chunksU);
    }
    assign<<<gridA, kAssignThreads, smemA>>>(dx.as<float>(), dcb.as<float>(), da.as<uint8_t>(),
                                             dssep.as<double>() + perStep * t, P, K);
    QCNN_CUDA(cudaGetLastError());
  }
  pq_sse_reduce_kernel<<<iters + 1, kUpdateThreads>>>(dssep.as<double>(), dsse.as<double>(), static_cast<int>(perStep));
  QCNN_CUDA(cudaGetLastError());
  std::vector<uint8_t> a(static_cast<size_t>(S) * P);
  std::vector<double> sse(iters + 1);
  QCNN_CUDA(cudaMemcpy(cb.data(), dcb.get(), sizeof(float) * cb.size(), cudaMemcpyDeviceToHost));
  QCNN_CUDA(cudaMemcpy(a.data(), da.get(), a.size(), cudaMemcpyDeviceToHost));
  QCNN_CUDA(cudaMemcpy(sse.data(), dsse.get(), sizeof(double) * sse.size(), cudaMemcpyDeviceToHost));
  for (int s = 0; s < S; s++)
    for (int k = 0; k < K; k++)
      for (int j = 0; j < d; j++)
        ctrd_h[(static_cast<size_t>(s) * K + k) * d + j] = j < D ? cb[(static_cast<size_t>(s) * K + k) * D + j] : 0.0f;
  for (int p = 0; p < P; p++)
    for (int s = 0; s < S; s++) asmt_h[static_cast<size_t>(p) * S + s] = a[static_cast<size_t>(s) * P + p];
  if (sse_h) std::copy(sse.begin(), sse.end(), sse_h);
  return 0;
}

struct QuantizedLayer {
  int l;
  Matrix<float> ctrd;
  Matrix<uint8_t> asmt;   // 1-based, as the .cbn writer takes it
  int bits;
};

bool ReadFile(const std::string& path, std::vector<char>* buf) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) return false;
  char tmp[1 << 16];
  size_t n;
  while ((n = fread(tmp, 1, sizeof(tmp), f)) > 0) buf->insert(buf->end(), tmp, tmp + n);
  const bool ok = !ferror(f);
  fclose(f);
  return ok;
}

bool WriteFile(const std::string& path, const std::vector<char>& buf) {
  FILE* f = fopen(path.c_str(), "wb");
  if (!f) return false;
  const bool ok = fwrite(buf.data(), 1, buf.size(), f) == buf.size();
  return (fclose(f) == 0) && ok;
}

}  // namespace

// K as qcnn_conv_layer_create / qcnn_fc_layer_create accept it, so that the output always loads
int qcnn::CheckConvK(const char* who, int K) {
  QCNN_CHECK(K >= 8 && K <= kMaxK && K % 8 == 0, "%s: K=%d must be a multiple of 8 in 8..%d", who, K, kMaxK);
  return 0;
}

int qcnn::CheckFcK(const char* who, int K) {
  QCNN_CHECK(K == 16 || K == 32 || K == 64 || K == 128 || K == 256, "%s: unsupported codebook size K=%d (supported: 16, 32, 64, 128, 256)",
             who, K);
  return 0;
}

extern "C" {

int qcnn_pq_quantize_conv(qcnn_ctx* ctx, int Cout, int Cg, int ksz, int K, int d, int iters, uint32_t seed, const float* knl_h,
                          const float* init_ctrd_h, float* ctrd_h, uint8_t* asmt_h, double* sse_h) {
  if (int rc = CheckConvK("qcnn_pq_quantize_conv", K)) return rc;
  return Quantize(ctx, "qcnn_pq_quantize_conv", Cout, Cg, ksz, K, d, iters, seed, knl_h, init_ctrd_h, ctrd_h, asmt_h, sse_h);
}

int qcnn_pq_quantize_fc(qcnn_ctx* ctx, int Din, int Dout, int K, int d, int iters, uint32_t seed, const float* wei_h,
                        const float* init_ctrd_h, float* ctrd_h, uint8_t* asmt_h, double* sse_h) {
  if (int rc = CheckFcK("qcnn_pq_quantize_fc", K)) return rc;
  return Quantize(ctx, "qcnn_pq_quantize_fc", Dout, Din, 1, K, d, iters, seed, wei_h, init_ctrd_h, ctrd_h, asmt_h, sse_h);
}

int qcnn_pq_quantize_model(qcnn_ctx* ctx, const char* model_name, const char* dir, const char* pfx, const int* K, const int* d,
                           int iters, uint32_t seed, const char* out_dir, const char* out_pfx) {
  const char* who = "qcnn_pq_quantize_model";
  QCNN_CHECK(ctx && model_name && dir && pfx && K && d && out_dir && out_pfx, "%s: NULL argument", who);
  CaffePara para;
  para.Init(dir, pfx);
  QCNN_CHECK(para.ConfigLayer_ByName(model_name), "%s: unrecognized caffe model name: %s", who, model_name);
  QCNN_CHECK(para.LoadLayerPara(false, ENUM_AsmtEnc::Compact), "%s: could not load dense parameters from %s/%s.*", who, dir, pfx);
  const std::vector<qcnn_layer_info> infos = LayerInfos(para);
  const std::vector<LayerDims> dims = LayerInputDims(infos, para.imgChnIn, para.imgHeiIn, para.imgWidIn);
  std::vector<QuantizedLayer> out;
  for (int l = 0; l < para.layerCnt; l++) {
    const qcnn_layer_info& li = infos[l];
    if (li.type != QCNN_CONV && li.type != QCNN_FCNT) continue;
    const bool conv = li.type == QCNN_CONV;
    const LayerPara& lp = para.layerParaLst[l];
    const LayerDims& in = dims[l];
    const int Kl = K[l], dl = d[l];
    char layerWho[64];
    snprintf(layerWho, sizeof(layerWho), "%s: layer %d", who, l + 1);
    if (int rc = conv ? CheckConvK(layerWho, Kl) : CheckFcK(layerWho, Kl)) return rc;
    QCNN_CHECK(dl >= 1 && dl <= kMaxD, "%s: d=%d is outside 1..%d", layerWho, dl, kMaxD);
    const Matrix<float>& w = conv ? lp.convKnlLst : lp.fcntWeiMat;
    int Cout, Cg, k;
    if (conv) {
      QCNN_CHECK(li.grpCnt >= 1 && in.C % li.grpCnt == 0, "%s: layer %d: %d input channels are not divisible into %d groups", who,
                 l + 1, in.C, li.grpCnt);
      Cout = li.knlCnt; Cg = in.C / li.grpCnt; k = li.knlSiz;
      QCNN_CHECK(w.GetDimCnt() == 4 && w.GetDimLen(0) == Cout && w.GetDimLen(1) == Cg && w.GetDimLen(2) == k && w.GetDimLen(3) == k,
                 "%s: layer %d: convKnl is not [%d][%d][%d][%d]", who, l + 1, Cout, Cg, k, k);
    } else {
      Cout = li.nodCnt; Cg = in.H * in.W * in.C; k = 1;
      QCNN_CHECK(w.GetDimCnt() == 2 && w.GetDimLen(0) == Cout && w.GetDimLen(1) == Cg, "%s: layer %d: fcntWei is not [%d][%d]", who,
                 l + 1, Cout, Cg);
    }
    QCNN_CHECK(lp.biasVec.GetEleCnt() == Cout, "%s: layer %d: biasVec does not hold %d values", who, l + 1, Cout);
    const int S = CeilDiv(Cg, dl);
    QuantizedLayer q;
    q.l = l;
    q.ctrd.Create(S, Kl, dl);
    if (conv) q.asmt.Create(Cout, k, k, S); else q.asmt.Create(Cout, S);
    if (int rc = Quantize(ctx, layerWho, Cout, Cg, k, Kl, dl, iters, seed + 65536u * static_cast<uint32_t>(l + 1), w.GetDataPtr(),
                          nullptr, q.ctrd.GetDataPtr(), q.asmt.GetDataPtr(), nullptr))
      return rc;
    uint8_t* a = q.asmt.GetDataPtr();
    for (int i = 0, n = q.asmt.GetEleCnt(); i < n; i++) a[i] = static_cast<uint8_t>(a[i] + 1);   // K = 256 wraps; the writer masks
    // CaffePara::CalcBitCntPerEle of a table whose 1-based maximum is K
    q.bits = 0;
    for (int m = Kl - 1; m != 0; m /= 2) q.bits++;
    out.push_back(std::move(q));
  }
  // every layer is quantized: write the files, and leave none behind if one fails
  CaffePara dst;
  dst.Init(out_dir, out_pfx);
  std::vector<std::string> written;
  bool ok = true;
  std::string failed;
  for (const QuantizedLayer& q : out) {
    std::vector<char> bias;
    const std::string biasSrc = para.ParaPath("biasVec", q.l, "bin"), biasDst = dst.ParaPath("biasVec", q.l, "bin");
    const std::string ctrdDst = dst.ParaPath("ctrdLst", q.l, "bin"), asmtDst = dst.ParaPath("asmtLst", q.l, "cbn");
    ok = ReadFile(biasSrc, &bias);
    if (ok) { written.push_back(biasDst); ok = WriteFile(biasDst, bias); }
    if (ok) { written.push_back(ctrdDst); ok = FileIO::WriteBinFile(ctrdDst, q.ctrd); }
    if (ok) { written.push_back(asmtDst); ok = FileIO::WriteCbnFile(asmtDst, q.asmt, q.bits); }
    if (!ok) { failed = written.empty() ? biasSrc : written.back(); break; }
  }
  if (!ok) {
    for (const std::string& p : written) remove(p.c_str());
    SetError("%s: cannot write %s", who, failed.c_str());
    return 1;
  }
  return 0;
}

}  // extern "C"
