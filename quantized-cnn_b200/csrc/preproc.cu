// The steps either side of the PQ path, on the device (SURVEY.md 8(f1), 8(f2)):
//   * image entry  -- BmpImgIO::Load after the file decode (reference src/BmpImgIO.cc:105-224: ReszImg, RmMeanImg,
//     CropImg) for a batch of decoded BMPs, and the uint8 -> mean-subtracted fp32 conversion of ready-made crops; a
//     host that ships uint8 pixels instead of fp32 tensors moves 4x fewer bytes over PCIe;
//   * result exit  -- the k-fold arg-max of CaffeEva::CvtFeatMapToLablVec (src/CaffeEva.cc:1162-1190) and
//     CaffeEvaWrapper::Proc (src/CaffeEvaWrapper.cc:188-206), so only k (index, probability) pairs per image go back.
// All arithmetic follows the reference expression by expression (same float / double steps, no FMA contraction), so the
// preprocessing is bit-identical to the CPU path (tests/test_gpu_preproc.py).
#include <float.h>

#include <vector>

#include "qcnn_internal.h"

using namespace qcnn;

struct qcnn_preproc {
  qcnn_ctx* ctx;
  int reszType, meanType;      // ENUM_ReszType { Strict, Relaxed }, ENUM_MeanType { Full, Crop } (include/BmpImgIO.h:19-20)
  int heiFull, widFull, heiCrop, widCrop;
  int meanHei, meanWid;
  DeviceBuffer d_mean;         // float [3][meanHei][meanWid]
  DeviceBuffer d_desc;         // per-image descriptors of the last run
};

namespace {

struct ImgDesc {
  long long off;     // byte offset of the image's pixels
  int hs, ws;        // source size
  int hd, wd;        // size after ReszImg
  float sh, sw;      // source step per resized pixel
};

// one thread = one pixel of the final crop, all three channels
__global__ void bmp_preproc_kernel(const uint8_t* __restrict__ pix, const ImgDesc* __restrict__ desc, const float* __restrict__ mean,
                                   int meanHei, int meanWid, int meanFull, int heiCrop, int widCrop, float* __restrict__ dst) {
  const int n = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= heiCrop * widCrop) return;
  const ImgDesc d = desc[n];
  const int yc_ = i / widCrop, xc_ = i - yc_ * widCrop;
  // CropImg (:180-201): centre crop of the resized image
  const int yo = (d.hd - heiCrop) / 2, xo = (d.wd - widCrop) / 2;
  const int y = yc_ + yo, x = xc_ + xo;
  // ReszImg (:119-176): weight-normalised bilinear interpolation, weights formed in double like `1.0 - (yc - yl)`
  const float yc = __fmul_rn(d.sh, static_cast<float>(y));
  const int yl = max(0, static_cast<int>(yc));
  const int yh = min(d.hs - 1, yl + 1);
  const float wyl = static_cast<float>(1.0 - static_cast<double>(__fsub_rn(yc, static_cast<float>(yl))));
  const float wyh = static_cast<float>(1.0 - static_cast<double>(__fsub_rn(static_cast<float>(yh), yc)));
  const float xc = __fmul_rn(d.sw, static_cast<float>(x));
  const int xl = max(0, static_cast<int>(xc));
  const int xh = min(d.ws - 1, xl + 1);
  const float wxl = static_cast<float>(1.0 - static_cast<double>(__fsub_rn(xc, static_cast<float>(xl))));
  const float wxh = static_cast<float>(1.0 - static_cast<double>(__fsub_rn(static_cast<float>(xh), xc)));
  const float wLT = __fmul_rn(wyl, wxl), wRT = __fmul_rn(wyl, wxh), wLB = __fmul_rn(wyh, wxl), wRB = __fmul_rn(wyh, wxh);
  const float wSum = __fadd_rn(__fadd_rn(__fadd_rn(wLT, wRT), wLB), wRB);
  const uint8_t* p = pix + d.off;
  const size_t rl = static_cast<size_t>(yl) * d.ws, rh = static_cast<size_t>(yh) * d.ws;
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const float a = static_cast<float>(p[(rl + xl) * 3 + c]), b = static_cast<float>(p[(rl + xh) * 3 + c]);
    const float e = static_cast<float>(p[(rh + xl) * 3 + c]), f = static_cast<float>(p[(rh + xh) * 3 + c]);
    float v = __fmul_rn(a, wLT);
    v = __fadd_rn(v, __fmul_rn(b, wRT));
    v = __fadd_rn(v, __fmul_rn(e, wLB));
    v = __fadd_rn(v, __fmul_rn(f, wRB));
    v = __fdiv_rn(v, wSum);
    // RmMeanImg (:203-224): the mean image has the resized ("Full") or the cropped ("Crop") size
    const float m = meanFull ? mean[(static_cast<size_t>(c) * meanHei + y) * meanWid + x]
                             : mean[(static_cast<size_t>(c) * meanHei + yc_) * meanWid + xc_];
    dst[((static_cast<size_t>(n) * 3 + c) * heiCrop + yc_) * widCrop + xc_] = __fsub_rn(v, m);
  }
}

// src u8 [N][H][W][C] (interleaved) -> dst f32 [N][C][H][W], minus mean [C][H][W] when given
__global__ void u8hwc_to_f32chw_kernel(const uint8_t* __restrict__ src, const float* __restrict__ mean, float* __restrict__ dst,
                                       int N, int C, int HW) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;   // (n, pixel)
  if (i >= static_cast<size_t>(N) * HW) return;
  const size_t n = i / HW;
  const int px = static_cast<int>(i - n * HW);
  const uint8_t* s = src + i * C;
  for (int c = 0; c < C; c++) {
    const float v = static_cast<float>(s[c]);
    dst[(n * C + c) * HW + px] = mean ? __fsub_rn(v, __ldg(mean + static_cast<size_t>(c) * HW + px)) : v;
  }
}

// k rounds of "first maximum wins, winner zeroed" on one row per block (works on a private copy in shared memory)
__global__ void topk_kernel(const float* __restrict__ prob, int C, int k, int mode, int* __restrict__ idx, float* __restrict__ val) {
  extern __shared__ float row[];
  __shared__ float wv[32];
  __shared__ int wi[32];
  const int n = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  for (int c = tid; c < C; c += blockDim.x) row[c] = prob[static_cast<size_t>(n) * C + c];
  __syncthreads();
  for (int r = 0; r < k; r++) {
    // first maximum of the thread's elements (ascending index, strict <), then of the block (ties -> lower index)
    float bv = -INFINITY;
    int bi = C;
    for (int c = tid; c < C; c += blockDim.x)
      if (bi == C || bv < row[c]) { bv = row[c]; bi = c; }
    for (int m = 16; m >= 1; m >>= 1) {
      const float ov = __shfl_xor_sync(0xFFFFFFFFu, bv, m);
      const int oi = __shfl_xor_sync(0xFFFFFFFFu, bi, m);
      if (oi < C && (bi == C || bv < ov || (bv == ov && oi < bi))) { bv = ov; bi = oi; }
    }
    if (lane == 0) { wv[warp] = bv; wi[warp] = bi; }
    __syncthreads();
    if (warp == 0) {
      bv = lane < nw ? wv[lane] : -INFINITY;
      bi = lane < nw ? wi[lane] : C;
      for (int m = 16; m >= 1; m >>= 1) {
        const float ov = __shfl_xor_sync(0xFFFFFFFFu, bv, m);
        const int oi = __shfl_xor_sync(0xFFFFFFFFu, bi, m);
        if (oi < C && (bi == C || bv < ov || (bv == ov && oi < bi))) { bv = ov; bi = oi; }
      }
      if (lane == 0) {
        // mode 1 (CvtFeatMapToLablVec): the scan starts from FLT_MIN with index 0, so nothing <= FLT_MIN can win
        if (mode == 1 && !(FLT_MIN < bv)) bi = 0;
        if (bi >= C) bi = 0;
        idx[static_cast<size_t>(n) * k + r] = bi;
        val[static_cast<size_t>(n) * k + r] = row[bi];
        row[bi] = 0.0f;
      }
    }
    __syncthreads();
  }
}

}  // namespace

namespace qcnn {

int LaunchU8ToF32(qcnn_ctx* ctx, const uint8_t* src, const float* mean, float* dst, int N, int C, int HW, cudaStream_t st) {
  const size_t total = static_cast<size_t>(N) * HW;
  u8hwc_to_f32chw_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(src, mean, dst, N, C, HW);
  QCNN_CUDA(cudaGetLastError());
  ctx->launches++;
  return 0;
}

int LaunchTopK(qcnn_ctx* ctx, const float* prob, int N, int C, int k, int mode, int* idx, float* val, cudaStream_t st) {
  QCNN_CHECK(k >= 1 && k <= C && C >= 1 && C <= 12000, "qcnn_topk: need 1 <= k <= C <= 12000 (got k=%d C=%d)", k, C);
  topk_kernel<<<N, 256, sizeof(float) * C, st>>>(prob, C, k, mode, idx, val);
  QCNN_CUDA(cudaGetLastError());
  ctx->launches++;
  return 0;
}

}  // namespace qcnn

extern "C" {

int qcnn_topk(qcnn_ctx* ctx, const float* prob, int N, int C, int k, int mode, int* idx, float* val, void* stream) {
  QCNN_CHECK(ctx && prob && idx && val && N >= 1, "qcnn_topk: bad argument");
  QCNN_ON_DEVICE(ctx->device);
  return LaunchTopK(ctx, prob, N, C, k, mode, idx, val, static_cast<cudaStream_t>(stream));
}

int qcnn_u8hwc_to_f32chw(qcnn_ctx* ctx, const uint8_t* src, const float* mean, float* dst, int N, int C, int H, int W, void* stream) {
  QCNN_CHECK(ctx && src && dst && N >= 1 && C >= 1 && H >= 1 && W >= 1, "qcnn_u8hwc_to_f32chw: bad argument");
  QCNN_ON_DEVICE(ctx->device);
  return LaunchU8ToF32(ctx, src, mean, dst, N, C, H * W, static_cast<cudaStream_t>(stream));
}

int qcnn_preproc_create(qcnn_ctx* ctx, int resz_type, int mean_type, int hei_full, int wid_full, int hei_crop, int wid_crop,
                        const float* mean_h, int mean_hei, int mean_wid, qcnn_preproc** out) {
  QCNN_CHECK(ctx && out && mean_h, "qcnn_preproc_create: NULL argument");
  *out = nullptr;
  QCNN_CHECK((resz_type == 0 || resz_type == 1) && (mean_type == 0 || mean_type == 1), "qcnn_preproc_create: bad enum value");
  QCNN_CHECK(hei_full >= 2 && wid_full >= 2 && hei_crop >= 1 && wid_crop >= 1 && hei_crop <= hei_full && wid_crop <= wid_full,
             "qcnn_preproc_create: bad sizes");
  if (mean_type == 0) {
    // RmMeanImg on the resized image: sizes must match (reference :208-211), which only a Strict resize guarantees
    QCNN_CHECK(resz_type == 0 && mean_hei == hei_full && mean_wid == wid_full,
               "qcnn_preproc_create: a full-size mean needs a Strict resize to exactly the mean's size");
  } else {
    QCNN_CHECK(mean_hei == hei_crop && mean_wid == wid_crop, "qcnn_preproc_create: a crop-size mean must have the crop's size");
  }
  QCNN_ON_DEVICE(ctx->device);
  qcnn_preproc* p = new qcnn_preproc();
  p->ctx = ctx; p->reszType = resz_type; p->meanType = mean_type;
  p->heiFull = hei_full; p->widFull = wid_full; p->heiCrop = hei_crop; p->widCrop = wid_crop;
  p->meanHei = mean_hei; p->meanWid = mean_wid;
  const size_t bytes = sizeof(float) * 3 * static_cast<size_t>(mean_hei) * mean_wid;
  if (cudaError_t e = p->d_mean.Upload(ctx, mean_h, bytes)) {
    CudaFail(e, "preproc mean upload", __FILE__, __LINE__);
    delete p;
    return 2;
  }
  *out = p;
  return 0;
}

void qcnn_preproc_destroy(qcnn_preproc* p) {
  if (!p) return;
  DeviceGuard guard(p->ctx->device);
  delete p;
}

int qcnn_preproc_run(qcnn_preproc* p, const uint8_t* pix, const long long* off_h, const int* hei_h, const int* wid_h, int N,
                     float* dst, void* stream) {
  QCNN_CHECK(p && pix && off_h && hei_h && wid_h && dst && N >= 1 && N <= 65535, "qcnn_preproc_run: bad argument");
  QCNN_ON_DEVICE(p->ctx->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  std::vector<ImgDesc> desc(N);
  for (int i = 0; i < N; i++) {
    const int hs = hei_h[i], ws = wid_h[i];
    QCNN_CHECK(hs >= 2 && ws >= 2, "qcnn_preproc_run: image %d is %dx%d (need at least 2x2)", i, hs, ws);
    // ReszImg (:119-138): scale = (src - 1) / (dst - 1); Relaxed keeps the aspect ratio and covers the target
    float sh = static_cast<float>(hs - 1) / (p->heiFull - 1);
    float sw = static_cast<float>(ws - 1) / (p->widFull - 1);
    int hd = p->heiFull, wd = p->widFull;
    if (p->reszType == 1) {
      sh = std::min(sh, sw);
      sw = std::min(sh, sw);
      hd = static_cast<int>((hs - 1) / sh + 0.0000001) + 1;
      wd = static_cast<int>((ws - 1) / sw + 0.0000001) + 1;
    }
    QCNN_CHECK(hd >= p->heiCrop && wd >= p->widCrop, "qcnn_preproc_run: image %d resizes to %dx%d, smaller than the crop", i, hd, wd);
    desc[i].off = off_h[i]; desc[i].hs = hs; desc[i].ws = ws; desc[i].hd = hd; desc[i].wd = wd; desc[i].sh = sh; desc[i].sw = sw;
  }
  const size_t need = sizeof(ImgDesc) * N;
  QCNN_CUDA(p->d_desc.Reserve(p->ctx, need, st));
  // (pageable source: the copy is staged by the runtime before the call returns, so `desc` may go out of scope)
  QCNN_CUDA(cudaMemcpyAsync(p->d_desc.get(), desc.data(), need, cudaMemcpyHostToDevice, st));
  dim3 grid(CeilDiv(p->heiCrop * p->widCrop, 256), N);
  bmp_preproc_kernel<<<grid, 256, 0, st>>>(pix, p->d_desc.as<const ImgDesc>(), p->d_mean.as<float>(), p->meanHei, p->meanWid,
                                           p->meanType == 0 ? 1 : 0, p->heiCrop, p->widCrop, dst);
  QCNN_CUDA(cudaGetLastError());
  p->ctx->launches++;
  return 0;
}

}  // extern "C"
