// C-ABI entry points of libqcnn_b200.so (include/qcnn.h): context, PQ layer set-up (the device-side equivalent of
// CaffeEva::PrepCtrdBuf / PrepAsmtBuf, reference src/CaffeEva.cc:534-623), per-layer forward calls, file formats.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../host/CaffePara.h"
#include "../host/FileIO.h"
#include "packed_asmt.h"
#include "qcnn_internal.h"

namespace qcnn {

static thread_local char g_err[1024] = "";

void SetError(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int CudaFail(cudaError_t e, const char* what, const char* file, int line) {
  SetError("CUDA error %d (%s) at %s:%d: %s", static_cast<int>(e), cudaGetErrorString(e), file, line, what);
  cudaGetLastError();   // reported: do not leave it behind for the next, unrelated, launch check to find
  return 2;
}

}  // namespace qcnn

using namespace qcnn;

extern "C" {

const char* qcnn_version(void) { return "qcnn-b200 0.1 (sm_90a)"; }
const char* qcnn_last_error(void) { return g_err; }

int qcnn_ctx_create(int device, qcnn_ctx** out) {
  QCNN_CHECK(out != nullptr, "qcnn_ctx_create: out is NULL");
  *out = nullptr;
  int cnt = 0;
  cudaError_t e = cudaGetDeviceCount(&cnt);
  if (e != cudaSuccess || cnt == 0) {
    SetError("qcnn_ctx_create: no CUDA device available (%s); this library has no CPU fallback",
             e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    return 2;
  }
  QCNN_CHECK(device >= 0 && device < cnt, "qcnn_ctx_create: device %d out of range (have %d)", device, cnt);
  cudaDeviceProp prop;
  QCNN_CUDA(cudaGetDeviceProperties(&prop, device));
  QCNN_CHECK(prop.major == 9 && prop.minor == 0, "qcnn_ctx_create: device %d is sm_%d%d; this build carries sm_90a code only", device,
             prop.major, prop.minor);
  QCNN_ON_DEVICE(device);
  qcnn_ctx* ctx = new qcnn_ctx();
  ctx->device = device;
  ctx->sm_count = prop.multiProcessorCount;
  ctx->cc_major = prop.major;
  ctx->cc_minor = prop.minor;
  ctx->smem_optin = prop.sharedMemPerBlockOptin;
  ctx->launches = 0;
  *out = ctx;
  return 0;
}

void qcnn_ctx_destroy(qcnn_ctx* ctx) { delete ctx; }
int qcnn_ctx_device(const qcnn_ctx* ctx) { return ctx ? ctx->device : -1; }
int qcnn_ctx_sm_count(const qcnn_ctx* ctx) { return ctx ? ctx->sm_count : 0; }

int qcnn_dev_alloc(qcnn_ctx* ctx, size_t bytes, void** out) {
  QCNN_CHECK(ctx && out, "qcnn_dev_alloc: NULL argument");
  QCNN_ON_DEVICE(ctx->device);
  QCNN_CUDA(cudaMalloc(out, bytes ? bytes : 1));
  return 0;
}
int qcnn_dev_free(qcnn_ctx* ctx, void* ptr) {
  QCNN_CHECK(ctx, "qcnn_dev_free: NULL ctx");
  QCNN_ON_DEVICE(ctx->device);
  if (ptr) QCNN_CUDA(cudaFree(ptr));
  return 0;
}
int qcnn_copy_h2d(qcnn_ctx* ctx, void* dst, const void* src_h, size_t bytes, void* stream) {
  QCNN_CHECK(ctx && dst && src_h, "qcnn_copy_h2d: NULL argument");
  QCNN_ON_DEVICE(ctx->device);
  QCNN_CUDA(cudaMemcpyAsync(dst, src_h, bytes, cudaMemcpyHostToDevice, static_cast<cudaStream_t>(stream)));
  return 0;
}
int qcnn_copy_d2h(qcnn_ctx* ctx, void* dst_h, const void* src, size_t bytes, void* stream) {
  QCNN_CHECK(ctx && dst_h && src, "qcnn_copy_d2h: NULL argument");
  QCNN_ON_DEVICE(ctx->device);
  QCNN_CUDA(cudaMemcpyAsync(dst_h, src, bytes, cudaMemcpyDeviceToHost, static_cast<cudaStream_t>(stream)));
  return 0;
}
int qcnn_stream_sync(qcnn_ctx* ctx, void* stream) {
  QCNN_CHECK(ctx, "qcnn_stream_sync: NULL ctx");
  QCNN_ON_DEVICE(ctx->device);
  QCNN_CUDA(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
  return 0;
}

static qcnn_layer* NewLayer(qcnn_ctx* ctx, int kind) {
  qcnn_layer* L = new qcnn_layer();
  L->ctx = ctx;
  L->kind = kind;
  // default operand format of the tensor-core GEMMs: bf16x2 (two MMAs per k-step at twice the tf32 rate; error at the
  // level of 3xTF32's, DESIGN.md 2); tensor_core = 1 or QCNN_TC_BF=0 selects 3xTF32
  static const bool bfDefault = !(getenv("QCNN_TC_BF") && getenv("QCNN_TC_BF")[0] == '0');
  L->opt_tc_bf = bfDefault ? 1 : 0;
  // process-wide default of "tensor_core": QCNN_NO_DECTC=1 starts every layer on the strict LUT + gather path
  static const bool strictDefault = getenv("QCNN_NO_DECTC") != nullptr;
  L->opt_no_tc = strictDefault ? 1 : 0;
  return L;
}

static int CheckPq(const char* who, int S, int K, int d, const uint8_t* asmt, size_t n) {
  QCNN_CHECK(S >= 1 && d >= 1, "%s: S and d must be >= 1", who);
  QCNN_CHECK(K >= 1 && K <= 256, "%s: K=%d does not fit uint8 assignments", who, K);
  for (size_t i = 0; i < n; i++) {
    if (asmt[i] >= K) {
      SetError("%s: assignment[%zu]=%d is not < K=%d", who, i, static_cast<int>(asmt[i]), K);
      return 1;
    }
  }
  return 0;
}

int qcnn_conv_layer_create(qcnn_ctx* ctx, int Cin, int Hin, int Win, int Cout, int ksz, int pad, int stride, int grp,
                           int S, int K, int d, const float* ctrd_h, const uint8_t* asmt_h, const float* bias_h,
                           qcnn_layer** out) {
  QCNN_CHECK(ctx && out && ctrd_h && asmt_h && bias_h, "qcnn_conv_layer_create: NULL argument");
  *out = nullptr;
  QCNN_CHECK(grp >= 1 && Cin % grp == 0 && Cout % grp == 0, "qcnn_conv_layer_create: channels not divisible by grp");
  QCNN_CHECK(ksz >= 1 && stride >= 1 && pad >= 0 && pad < ksz, "qcnn_conv_layer_create: bad kernel geometry");
  QCNN_CHECK(Hin + 2 * pad >= ksz && Win + 2 * pad >= ksz, "qcnn_conv_layer_create: kernel larger than input");
  QCNN_CHECK(K % 8 == 0, "qcnn_conv_layer_create: K=%d must be a multiple of 8 (LUT stage tiles 8 codewords)", K);
  const int taps = ksz * ksz;
  if (int rc = CheckPq("qcnn_conv_layer_create", S, K, d, asmt_h, static_cast<size_t>(Cout) * taps * S)) return rc;
  QCNN_ON_DEVICE(ctx->device);
  qcnn_layer* L = NewLayer(ctx, QCNN_KIND_CONV);
  L->Cin = Cin; L->Hin = Hin; L->Win = Win; L->Cout = Cout; L->ksz = ksz; L->pad = pad; L->stride = stride;
  L->grp = grp; L->S = S; L->K = K; L->d = d;
  L->Ho = (Hin + 2 * pad - ksz) / stride + 1;  // reference CaffeEva.cc:361-362
  L->Wo = (Win + 2 * pad - ksz) / stride + 1;
  const int Kg = Cout / grp, KgPad = RoundUp(Kg, 16);
  // assignments: file order [Cout][kh][kw][S] -> device [grp][S][tap][KgPad]
  // (the reference's asmtBuf is [kh][kw][S][Cout], CaffeEva.cc:585-586; we additionally make the subspace the
  //  slow index because the fused kernel walks s in its outer loop)
  std::vector<uint8_t> dev(static_cast<size_t>(grp) * S * taps * KgPad, 0);
  for (int g = 0; g < grp; g++)
    for (int c = 0; c < Kg; c++)
      for (int t = 0; t < taps; t++)
        for (int s = 0; s < S; s++)
          dev[((static_cast<size_t>(g) * S + s) * taps + t) * KgPad + c] =
              asmt_h[((static_cast<size_t>(g) * Kg + c) * taps + t) * S + s];
  // channel-major copy for the tensor-core GEMM's decoders: [grp][S][KgPad][tapsPad]
  const int tapsPad = RoundUp(taps, 16);
  std::vector<uint8_t> devT;
  if (stride > 1 && S == 1) {
    // strided layers (conv1): one block per phase row ph, row r <-> tap (kh = ph + (r / ksz) * stride, kw = r % ksz)
    const int rowsPad = RoundUp(((ksz + stride - 1) / stride) * ksz, 16);
    L->asmt_t_mode = 1;
    devT.assign(static_cast<size_t>(grp) * stride * KgPad * rowsPad, 0);
    for (int g = 0; g < grp; g++)
      for (int ph = 0; ph < stride; ph++)
        for (int c = 0; c < Kg; c++)
          for (int kh = ph, r0 = 0; kh < ksz; kh += stride, r0 += ksz)
            for (int kw = 0; kw < ksz; kw++)
              devT[((static_cast<size_t>(g) * stride + ph) * KgPad + c) * rowsPad + r0 + kw] =
                  dev[(static_cast<size_t>(g) * taps + kh * ksz + kw) * KgPad + c];
  } else {
    devT.assign(static_cast<size_t>(grp) * S * KgPad * tapsPad, 0);
    for (int g = 0; g < grp; g++)
      for (int s = 0; s < S; s++)
        for (int c = 0; c < Kg; c++)
          for (int t = 0; t < taps; t++)
            devT[((static_cast<size_t>(g) * S + s) * KgPad + c) * tapsPad + t] = dev[((static_cast<size_t>(g) * S + s) * taps + t) * KgPad + c];
  }
  cudaError_t e = L->d_asmt.Upload(ctx, dev.data(), dev.size());
  if (!e) e = L->d_asmt_t.Upload(ctx, devT.data(), devT.size());
  if (!e) e = L->d_ctrd.Upload(ctx, ctrd_h, sizeof(float) * S * K * d);
  if (!e) e = L->d_bias.Upload(ctx, bias_h, sizeof(float) * Cout);
  if (e) {
    CudaFail(e, "conv layer upload", __FILE__, __LINE__);
    qcnn_layer_destroy(L);
    return 2;
  }
  if (BuildCtrdBf(L) || BuildConvWsImage(L)) { qcnn_layer_destroy(L); return 2; }
  if (PlanConv(L, 256)) {  // validates that a tiling exists; re-planned per batch size at launch
    qcnn_layer_destroy(L);
    return 1;
  }
  *out = L;
  return 0;
}

int qcnn_fc_layer_create(qcnn_ctx* ctx, int Din, int Dout, int S, int K, int d, const float* ctrd_h,
                         const uint8_t* asmt_h, const float* bias_h, qcnn_layer** out) {
  QCNN_CHECK(ctx && out && ctrd_h && asmt_h && bias_h, "qcnn_fc_layer_create: NULL argument");
  *out = nullptr;
  QCNN_CHECK(Din >= 1 && Dout >= 1, "qcnn_fc_layer_create: bad dimensions");
  if (int rc = CheckPq("qcnn_fc_layer_create", S, K, d, asmt_h, static_cast<size_t>(Dout) * S)) return rc;
  QCNN_CHECK(K == 16 || K == 32 || K == 64 || K == 128 || K == 256,
             "qcnn_fc_layer_create: unsupported codebook size K=%d (supported: 16, 32, 64, 128, 256)", K);
  // every batch size must have a kernel: the LUT + gather kernel (batches 5-95, tensor_core = 0, fc_* pins) stages the
  // codebook rows of a chunk in shared memory, which bounds d (K = 256: d <= 11)
  QCNN_CHECK(FcGatherSmemBytes(K, 1, d) <= kFcGatherSmemMax,
             "qcnn_fc_layer_create: K=%d d=%d is not supported: the LUT + gather kernel would stage %zu bytes of shared memory "
             "per CTA (limit %zu)", K, d, FcGatherSmemBytes(K, 1, d), kFcGatherSmemMax);
  QCNN_ON_DEVICE(ctx->device);
  qcnn_layer* L = NewLayer(ctx, QCNN_KIND_FC);
  L->Din = Din; L->Dout = Dout; L->S = S; L->K = K; L->d = d;
  L->Ho = 1; L->Wo = 1; L->Cout = Dout;
  L->DoutPad = RoundUp(Dout, 16);
  L->asmt_pitch = L->DoutPad;
  L->kshift = (K <= 64) ? 2 : 0;
  // assignments: file order [Dout][S] -> device [S][DoutPad] (reference asmtBuf [S][Dout], CaffeEva.cc:610-611),
  // stored as byte offsets into a LUT row (idx * 4) when that fits a byte
  std::vector<uint8_t> dev(static_cast<size_t>(S) * L->DoutPad, 0);
  for (int o = 0; o < Dout; o++)
    for (int s = 0; s < S; s++)
      dev[static_cast<size_t>(s) * L->DoutPad + o] = static_cast<uint8_t>(asmt_h[static_cast<size_t>(o) * S + s] << L->kshift);
  cudaError_t e = L->d_asmt.Upload(ctx, dev.data(), dev.size());
  if (!e) e = L->d_ctrd.Upload(ctx, ctrd_h, sizeof(float) * S * K * d);
  if (!e) e = L->d_bias.Upload(ctx, bias_h, sizeof(float) * Dout);
  if (e) {
    CudaFail(e, "fc layer upload", __FILE__, __LINE__);
    qcnn_layer_destroy(L);
    return 2;
  }
  if (BuildCtrdBf(L)) { qcnn_layer_destroy(L); return 2; }
  *out = L;
  return 0;
}

int qcnn_fc_layer_set_src_nhwc(qcnn_layer* L, int H, int W, int C) {
  QCNN_CHECK(L && L->kind == QCNN_KIND_FC, "qcnn_fc_layer_set_src_nhwc: not an FC layer");
  QCNN_ON_DEVICE(L->ctx->device);
  L->ctx->alloc_epoch++;   // captured graphs may hold the old offset table / kernel choice
  QCNN_CUDA(L->d_srcoff.Release());
  if (H == 0 && W == 0 && C == 0) { L->src_h = L->src_w = L->src_c = 0; return 0; }
  QCNN_CHECK(H >= 1 && W >= 1 && C >= 1 && H * W * C == L->Din, "qcnn_fc_layer_set_src_nhwc: H*W*C=%d != Din=%d",
             H * W * C, L->Din);
  L->src_h = H; L->src_w = W; L->src_c = C;
  // flattened NCHW feature f = c*H*W + hw  ->  NHWC element offset hw*C + c
  std::vector<int> off(L->Din);
  const int hw = H * W;
  for (int f = 0; f < L->Din; f++) off[f] = (f % hw) * C + f / hw;
  QCNN_CUDA(L->d_srcoff.Upload(L->ctx, off.data(), sizeof(int) * L->Din));
  return 0;
}

int qcnn_conv_layer_set_src_nchw(qcnn_layer* L, int enable) {
  QCNN_CHECK(L && L->kind == QCNN_KIND_CONV, "qcnn_conv_layer_set_src_nchw: not a conv layer");
  QCNN_CHECK(!enable || L->stride > 1, "qcnn_conv_layer_set_src_nchw: only the strided kernel reads NCHW");
  L->ctx->alloc_epoch++;
  L->src_nchw = enable ? 1 : 0;
  return 0;
}

}  // extern "C"

// FC assignment table on the host as plain 0-based indices [S][DoutPad], whichever form d_asmt holds
static int ReadFcIndices(const qcnn_layer* L, std::vector<uint8_t>* idx) {
  std::vector<uint8_t> dev(L->d_asmt.bytes());
  QCNN_CUDA(cudaMemcpy(dev.data(), L->d_asmt.get(), dev.size(), cudaMemcpyDeviceToHost));
  idx->assign(static_cast<size_t>(L->S) * L->DoutPad, 0);
  const int b = L->asmt_bits;
  for (int s = 0; s < L->S; s++) {
    const uint8_t* row = dev.data() + static_cast<size_t>(s) * L->asmt_pitch;
    uint8_t* out = idx->data() + static_cast<size_t>(s) * L->DoutPad;
    for (int o = 0; o < L->DoutPad; o++) {
      if (!b) { out[o] = row[o] >> L->kshift; continue; }
      int v = 0;
      for (int i = 0; i < b; i++) {
        const int bit = o * b + i;
        v |= ((row[bit >> 3] >> (bit & 7)) & 1) << i;
      }
      out[o] = static_cast<uint8_t>(v);
    }
  }
  return 0;
}

// Replaces d_asmt by the byte table (enable = 0) or the bit-packed table (packed_asmt.h).  Layers with K = 256 keep the
// byte table either way: at 8 bits packing changes nothing.
static int SetAsmtPacked(qcnn_layer* L, int enable) {
  const int b = (enable && PackedBits(L->K) < 8) ? PackedBits(L->K) : 0;
  if (b == L->asmt_bits) return 0;
  QCNN_ON_DEVICE(L->ctx->device);
  std::vector<uint8_t> idx;
  if (int rc = ReadFcIndices(L, &idx)) return rc;
  const int pitch = b ? PackedPitch(L->DoutPad, b) : L->DoutPad;
  std::vector<uint8_t> host(static_cast<size_t>(L->S) * pitch + (b ? kPackedTail : 0), 0);
  for (int s = 0; s < L->S; s++) {
    uint8_t* row = host.data() + static_cast<size_t>(s) * pitch;
    const uint8_t* in = idx.data() + static_cast<size_t>(s) * L->DoutPad;
    for (int o = 0; o < L->DoutPad; o++) {
      if (!b) { row[o] = static_cast<uint8_t>(in[o] << L->kshift); continue; }
      for (int i = 0; i < b; i++) {
        const int bit = o * b + i;
        row[bit >> 3] |= static_cast<uint8_t>(((in[o] >> i) & 1) << (bit & 7));
      }
    }
  }
  // kernels still queued on any stream may read the old table
  QCNN_CUDA(cudaDeviceSynchronize());
  DeviceBuffer nb;
  QCNN_CUDA(nb.Upload(L->ctx, host.data(), host.size()));   // (bumps alloc_epoch: graphs captured before hold the old table)
  L->d_asmt = std::move(nb);                                 // the old table is freed here
  L->asmt_bits = b;
  L->asmt_pitch = pitch;
  return 0;
}

extern "C" {

int qcnn_layer_set_param(qcnn_layer* L, const char* name, int value) {
  QCNN_CHECK(L && name, "qcnn_layer_set_param: NULL argument");
  L->ctx->alloc_epoch++;   // every parameter changes kernel choice or buffers: graphs captured before are stale
  if (!strcmp(name, "asmt_packed")) {
    // FC only: 1 keeps the assignment table bit-packed at log2(K) bits per index (kernels unpack it), 0 = byte table
    QCNN_CHECK(L->kind == QCNN_KIND_FC, "qcnn_layer_set_param: 'asmt_packed' applies to FC layers");
    return SetAsmtPacked(L, value);
  }
  if (!strcmp(name, "fc_ws")) {
    // FC only: 1 runs the batched tensor-core path as the weight-stationary GEMM (fc_ws.cu) where it applies (bf16x2
    // operands, byte table), 0 (the default of a standalone layer) keeps pq_gemm_tc mode 2
    QCNN_CHECK(L->kind == QCNN_KIND_FC, "qcnn_layer_set_param: 'fc_ws' applies to FC layers");
    L->opt_fc_ws = value ? 1 : 0;
  }
  else if (!strcmp(name, "fc_nsplit")) L->opt_fc_nsplit = value;
  else if (!strcmp(name, "fc_tn")) L->opt_fc_tn = value;
  else if (!strcmp(name, "tensor_core")) {
    // 0: LUT + gather kernels only (fp32 adds in the reference's association; the strict-parity path);
    // 2 (default): eligible layers run the decode-at-use tensor-core GEMMs with bf16x2 operands (two MMAs per k-step at
    // the bf16 rate); 1: the same GEMMs with 3xTF32 operands (both with a wider tolerance: DESIGN.md)
    L->opt_no_tc = value ? 0 : 1;
    L->opt_tc_bf = value == 2 ? 1 : 0;
    L->plan_N = 0; L->tuned = 0;
    L->tunedPlans.clear();
  }
  else if (!strcmp(name, "gemm_nt") || !strcmp(name, "gemm_gt") || !strcmp(name, "gemm_nsplit") || !strcmp(name, "gemm_ct")) {
    // 0 = any.  Conv: gemm_nt: positions per CTA of the pq_gemm_tc tilings (128 = one accumulator, 64 = two) and of the
    // conv_ws tilings; gemm_gt: k-steps per stage of the pq_gemm_tc tilings (4 or 3); gemm_nsplit: their K-split factor
    // (1 = no split, > 1 = partial sums reduced by a second kernel); gemm_ct: channels per CTA of the conv_ws tilings.
    // FC with fc_ws = 1: the fc_ws tilings with that many images per CTA (128 / 256), k-steps per stage (8 / 4), K-split
    // factor and channels per CTA; pq_gemm_tc mode 2 has a single tiling per batch and ignores them.
    // A pin that no tiling of the layer matches fails the forward.
    const int v = value < 0 ? 0 : value;
    if (!strcmp(name, "gemm_nt")) L->opt_gemm_nt = v;
    else if (!strcmp(name, "gemm_gt")) L->opt_gemm_gt = v;
    else if (!strcmp(name, "gemm_nsplit")) L->opt_gemm_nsplit = v;
    else L->opt_gemm_ct = v;
    L->plan_N = 0; L->tuned = 0;
    L->tunedPlans.clear();
  }
  else if (!strcmp(name, "gemm_wb")) {
    // conv only, 0 = any: the conv_ws tilings with that many weight stage buffers (2, 3 or 4) in their ring.  A pin that
    // no tiling of the layer matches fails the forward.
    QCNN_CHECK(L->kind == QCNN_KIND_CONV, "qcnn_layer_set_param: 'gemm_wb' applies to conv layers");
    L->opt_gemm_wb = value < 0 ? 0 : value;
    L->plan_N = 0; L->tuned = 0;
    L->tunedPlans.clear();
  }
  else if (!strcmp(name, "lut_cpt") || !strcmp(name, "lut_j") || !strcmp(name, "lut_nct") || !strcmp(name, "lut_r") ||
           !strcmp(name, "lut_rgroups")) {
    // conv only, 0 = any: the LUT + gather tilings (force_kernel 0-4) with that many channels per thread, positions per
    // lane (conv_direct: output rows per thread), channel tiles per group, output rows per strip (conv_direct: the value
    // after its clamp to Ho + (Ho & 1)) and row groups.  A pin that no tiling of the layer matches fails the forward.
    QCNN_CHECK(L->kind == QCNN_KIND_CONV, "qcnn_layer_set_param: '%s' applies to conv layers", name);
    const int v = value < 0 ? 0 : value;
    if (!strcmp(name, "lut_cpt")) L->opt_lut_cpt = v;
    else if (!strcmp(name, "lut_j")) L->opt_lut_j = v;
    else if (!strcmp(name, "lut_nct")) L->opt_lut_nct = v;
    else if (!strcmp(name, "lut_r")) L->opt_lut_r = v;
    else L->opt_lut_rgroups = v;
    L->plan_N = 0; L->tuned = 0;
    L->tunedPlans.clear();
  }
  else if (!strcmp(name, "force_kernel") || !strcmp(name, "autotune")) {
    // conv only.  force_kernel: -1 none, else 0 s1 | 1 roll | 2 s1_tc | 3 roll_tc | 4 direct | 6 pq_gemm_tc | 7 conv_ws;
    // autotune: 0 keeps the cost model's first tiling instead of timing the candidates on the device
    QCNN_CHECK(L->kind == QCNN_KIND_CONV, "qcnn_layer_set_param: '%s' applies to conv layers", name);
    if (name[0] == 'f') L->opt_force_kernel = value < 0 ? 0 : value + 1;
    else L->opt_no_autotune = value ? 0 : 1;
    L->plan_N = 0; L->tuned = 0;
    L->tunedPlans.clear();
  }
  else { SetError("qcnn_layer_set_param: unknown parameter '%s'", name); return 1; }
  return 0;
}

int qcnn_layer_describe(qcnn_layer* L, int N, char* buf, size_t cap) {
  QCNN_CHECK(L && buf && cap > 0 && N >= 1, "qcnn_layer_describe: bad argument");
  if (L->kind == QCNN_KIND_CONV) return DescribeConv(L, N, buf, cap);
  return DescribeFc(L, N, buf, cap);
}

void qcnn_layer_destroy(qcnn_layer* L) {
  if (!L) return;
  DeviceGuard guard(L->ctx->device);
  delete L;
}

int qcnn_layer_out_dims(const qcnn_layer* L, int* out3) {
  QCNN_CHECK(L && out3, "qcnn_layer_out_dims: NULL argument");
  out3[0] = L->Ho; out3[1] = L->Wo; out3[2] = L->Cout;
  return 0;
}

// SURVEY.md 8(d): conv 4*N*Hi*Wi*Cin + 4*N*Ho*Wo*Cout + k^2*S*Cout + 4*S*K*d + 4*Cout ;
//                 FC   4*N*Din + 4*N*Dout + S*Dout + 4*S*K*d + 4*Dout
int qcnn_layer_work(const qcnn_layer* L, int N, double* alg_bytes, double* lookups, double* lut_macs) {
  QCNN_CHECK(L, "qcnn_layer_work: NULL layer");
  double bytes, lk, macs;
  if (L->kind == QCNN_KIND_CONV) {
    const double taps = static_cast<double>(L->ksz) * L->ksz;
    bytes = 4.0 * N * L->Hin * L->Win * L->Cin + 4.0 * N * L->Ho * L->Wo * L->Cout + taps * L->S * L->Cout +
            4.0 * L->S * L->K * L->d + 4.0 * L->Cout;
    // valid (in-bounds) taps only, as the reference counts them
    double vt = 0;
    for (int ho = 0; ho < L->Ho; ho++) {
      const int hL = ho * L->stride - L->pad;
      const int nh = std::min(L->ksz - 1, L->Hin - 1 - hL) - std::max(0, -hL) + 1;
      for (int wo = 0; wo < L->Wo; wo++) {
        const int wL = wo * L->stride - L->pad;
        const int nw = std::min(L->ksz - 1, L->Win - 1 - wL) - std::max(0, -wL) + 1;
        vt += static_cast<double>(nh) * nw;
      }
    }
    lk = vt * L->S * L->Cout * N;
    const int Cg = L->Cin / L->grp;
    double dims = 0;
    for (int s = 0; s < L->S; s++) dims += std::max(0, std::min(Cg - s * L->d, L->d));
    macs = static_cast<double>(N) * L->Hin * L->Win * L->grp * dims * L->K;
  } else {
    // assignment term: S * Dout bytes, or S * ceil(Dout * b / 8) when the table is bit-packed
    const double asmtRow = L->asmt_bits ? static_cast<double>((L->Dout * L->asmt_bits + 7) / 8) : static_cast<double>(L->Dout);
    bytes = 4.0 * N * L->Din + 4.0 * N * L->Dout + static_cast<double>(L->S) * asmtRow + 4.0 * L->S * L->K * L->d +
            4.0 * L->Dout;
    lk = static_cast<double>(N) * L->S * L->Dout;
    double dims = 0;
    for (int s = 0; s < L->S; s++) dims += std::max(0, std::min(L->Din - s * L->d, L->d));
    macs = static_cast<double>(N) * dims * L->K;
  }
  if (alg_bytes) *alg_bytes = bytes;
  if (lookups) *lookups = lk;
  if (lut_macs) *lut_macs = macs;
  return 0;
}

int qcnn_layer_read_asmt_h(const qcnn_layer* L, uint8_t* out_h, size_t cap) {
  QCNN_CHECK(L && out_h, "qcnn_layer_read_asmt_h: NULL argument");
  QCNN_ON_DEVICE(L->ctx->device);
  if (L->kind != QCNN_KIND_CONV) {
    QCNN_CHECK(cap >= static_cast<size_t>(L->S) * L->Dout, "qcnn_layer_read_asmt_h: buffer too small");
    std::vector<uint8_t> idx;
    if (int rc = ReadFcIndices(L, &idx)) return rc;
    for (int s = 0; s < L->S; s++)
      memcpy(out_h + static_cast<size_t>(s) * L->Dout, idx.data() + static_cast<size_t>(s) * L->DoutPad, L->Dout);
    return 0;
  }
  std::vector<uint8_t> dev(L->d_asmt.bytes());
  QCNN_CUDA(cudaMemcpy(dev.data(), L->d_asmt.get(), dev.size(), cudaMemcpyDeviceToHost));
  const int taps = L->ksz * L->ksz, Kg = L->Cout / L->grp, KgPad = RoundUp(Kg, 16);
  QCNN_CHECK(cap >= static_cast<size_t>(taps) * L->S * L->Cout, "qcnn_layer_read_asmt_h: buffer too small");
  for (int t = 0; t < taps; t++)
    for (int s = 0; s < L->S; s++)
      for (int c = 0; c < L->Cout; c++) {
        const int g = c / Kg, cl = c % Kg;
        out_h[(static_cast<size_t>(t) * L->S + s) * L->Cout + c] =
            dev[((static_cast<size_t>(g) * L->S + s) * taps + t) * KgPad + cl];
      }
  return 0;
}

int qcnn_layer_read_w_ws(const qcnn_layer* L, void* out_h, size_t cap, size_t* bytes) {
  QCNN_CHECK(L && bytes, "qcnn_layer_read_w_ws: NULL argument");
  *bytes = L->d_w_ws.bytes();
  if (!out_h || *bytes == 0) return 0;
  QCNN_CHECK(cap >= *bytes, "qcnn_layer_read_w_ws: buffer too small (%zu < %zu bytes)", cap, *bytes);
  QCNN_ON_DEVICE(L->ctx->device);
  QCNN_CUDA(cudaMemcpy(out_h, L->d_w_ws.get(), *bytes, cudaMemcpyDeviceToHost));
  return 0;
}

int qcnn_conv_aprx_forward(qcnn_layer* L, const float* src, int N, float* dst, int fuse_relu, void* stream) {
  QCNN_CHECK(L && src && dst, "qcnn_conv_aprx_forward: NULL argument");
  QCNN_ON_DEVICE(L->ctx->device);
  return LaunchConv(L, src, N, dst, fuse_relu, static_cast<cudaStream_t>(stream));
}

int qcnn_fc_aprx_forward(qcnn_layer* L, const float* src, int N, float* dst, int fuse_relu, void* stream) {
  QCNN_CHECK(L && src && dst, "qcnn_fc_aprx_forward: NULL argument");
  QCNN_ON_DEVICE(L->ctx->device);
  return LaunchFc(L, src, N, dst, fuse_relu, static_cast<cudaStream_t>(stream));
}

int qcnn_fc_aprx_forward_flat(qcnn_layer* L, const float* src, int N, float* dst, int fuse_relu, void* stream) {
  QCNN_CHECK(L && src && dst, "qcnn_fc_aprx_forward_flat: NULL argument");
  QCNN_ON_DEVICE(L->ctx->device);
  DeviceBuffer saved = std::move(L->d_srcoff);   // every FC path sees no offset table while the source is flat
  const int rc = LaunchFc(L, src, N, dst, fuse_relu, static_cast<cudaStream_t>(stream));
  L->d_srcoff = std::move(saved);
  return rc;
}

int qcnn_fc_chain_forward(qcnn_layer* const* layers, const int* relu, int n, const float* src, int N, float* dst,
                          unsigned long long* stamps, void* stream) {
  QCNN_CHECK(layers && relu && src && dst && n >= 1 && n <= 4, "qcnn_fc_chain_forward: bad argument (1..4 layers)");
  for (int l = 0; l < n; l++) QCNN_CHECK(layers[l] && layers[l]->kind == QCNN_KIND_FC, "qcnn_fc_chain_forward: layer %d is not fully-connected", l);
  QCNN_CHECK(N >= 1 && N <= 4, "qcnn_fc_chain_forward: N must be in [1, 4] (got %d)", N);
  QCNN_ON_DEVICE(layers[0]->ctx->device);
  bool handled = false;
  if (int rc = LaunchFcChain(layers[0]->ctx, layers, relu, n, src, N, dst, static_cast<cudaStream_t>(stream), stamps, &handled)) return rc;
  QCNN_CHECK(handled, "qcnn_fc_chain_forward: these layers are not supported by the fused kernel (shape, shared memory, "
             "fc_nsplit / fc_tn override, or QCNN_FC_CHAIN=0)");
  return 0;
}

int qcnn_relu(qcnn_ctx* ctx, const float* src, float* dst, size_t n, void* stream) {
  QCNN_CHECK(ctx && src && dst, "qcnn_relu: NULL argument");
  QCNN_ON_DEVICE(ctx->device);
  return LaunchRelu(ctx, src, dst, n, static_cast<cudaStream_t>(stream));
}
int qcnn_lrn(qcnn_ctx* ctx, const float* src, float* dst, size_t pixels, int C, int size, float alpha, float beta,
             float k, void* stream) {
  QCNN_CHECK(ctx && src && dst, "qcnn_lrn: NULL argument");
  QCNN_ON_DEVICE(ctx->device);
  return LaunchLrn(ctx, src, dst, pixels, C, size, alpha, beta, k, static_cast<cudaStream_t>(stream));
}
int qcnn_maxpool(qcnn_ctx* ctx, const float* src, float* dst, int N, int H, int W, int C, int ksz, int pad, int stride,
                 void* stream) {
  QCNN_CHECK(ctx && src && dst, "qcnn_maxpool: NULL argument");
  QCNN_ON_DEVICE(ctx->device);
  return LaunchMaxPool(ctx, src, dst, N, H, W, C, ksz, pad, stride, static_cast<cudaStream_t>(stream));
}
int qcnn_lrn_maxpool(qcnn_ctx* ctx, const float* src, float* dst, int N, int H, int W, int C, int size, float alpha,
                     float beta, float k, int ksz, int pad, int stride, void* stream) {
  QCNN_CHECK(ctx && src && dst, "qcnn_lrn_maxpool: NULL argument");
  QCNN_ON_DEVICE(ctx->device);
  return LaunchLrnMaxPool(ctx, src, dst, N, H, W, C, size, alpha, beta, k, ksz, pad, stride,
                          static_cast<cudaStream_t>(stream));
}
int qcnn_softmax(qcnn_ctx* ctx, const float* src, float* dst, int N, int C, void* stream) {
  QCNN_CHECK(ctx && src && dst, "qcnn_softmax: NULL argument");
  QCNN_ON_DEVICE(ctx->device);
  return LaunchSoftmax(ctx, src, dst, N, C, static_cast<cudaStream_t>(stream));
}
int qcnn_nchw_to_nhwc(qcnn_ctx* ctx, const float* src, float* dst, int N, int C, int H, int W, void* stream) {
  QCNN_CHECK(ctx && src && dst, "qcnn_nchw_to_nhwc: NULL argument");
  QCNN_ON_DEVICE(ctx->device);
  return LaunchNchwToNhwc(ctx, src, dst, N, C, H, W, static_cast<cudaStream_t>(stream));
}
int qcnn_nhwc_to_nchw(qcnn_ctx* ctx, const float* src, float* dst, int N, int H, int W, int C, void* stream) {
  QCNN_CHECK(ctx && src && dst, "qcnn_nhwc_to_nchw: NULL argument");
  QCNN_ON_DEVICE(ctx->device);
  return LaunchNhwcToNchw(ctx, src, dst, N, H, W, C, static_cast<cudaStream_t>(stream));
}

// ---- file formats (host) ---------------------------------------------------------------------------------
long qcnn_read_bin_f32(const char* path, int* dim_cnt, int* dims4, float* data_h, long cap) {
  Matrix<float> m;
  if (!path || !FileIO::ReadBinFile(path, &m)) { SetError("qcnn_read_bin_f32: cannot read %s", path ? path : "(null)"); return -1; }
  if (dim_cnt) *dim_cnt = m.GetDimCnt();
  if (dims4) for (int i = 0; i < 4; i++) dims4[i] = m.GetDimLen(i);
  const long n = m.GetEleCnt();
  if (data_h) memcpy(data_h, m.GetDataPtr(), sizeof(float) * std::min(n, cap));
  return n;
}

int qcnn_write_bin_f32(const char* path, int dim_cnt, const int* dims, const float* data_h) {
  QCNN_CHECK(path && dims && data_h && dim_cnt >= 1 && dim_cnt <= 4, "qcnn_write_bin_f32: bad argument");
  Matrix<float> m(dim_cnt, dims);
  memcpy(m.GetDataPtr(), data_h, sizeof(float) * m.GetEleCnt());
  QCNN_CHECK(FileIO::WriteBinFile(path, m), "qcnn_write_bin_f32: cannot write %s", path);
  return 0;
}

long qcnn_read_cbn_u8(const char* path, int* dim_cnt, int* dims4, int* bits, uint8_t* data_h, long cap) {
  Matrix<uint8_t> m;
  if (!path || !FileIO::ReadCbnFile(path, &m)) { SetError("qcnn_read_cbn_u8: cannot read %s", path ? path : "(null)"); return -1; }
  if (dim_cnt) *dim_cnt = m.GetDimCnt();
  if (dims4) for (int i = 0; i < 4; i++) dims4[i] = m.GetDimLen(i);
  if (bits) *bits = FileIO::PeekCbnBits(path);
  const long n = m.GetEleCnt();
  if (data_h) {
    const uint8_t* p = m.GetDataPtr();
    for (long i = 0; i < std::min(n, cap); i++) data_h[i] = static_cast<uint8_t>(p[i] - 1);  // CaffePara.cc:285-288
  }
  return n;
}

int qcnn_write_cbn_u8(const char* path, int dim_cnt, const int* dims, const uint8_t* idx0_h, int bits) {
  QCNN_CHECK(path && dims && idx0_h && dim_cnt >= 1 && dim_cnt <= 4, "qcnn_write_cbn_u8: bad argument");
  Matrix<uint8_t> m(dim_cnt, dims);
  uint8_t* p = m.GetDataPtr();
  for (int i = 0, n = m.GetEleCnt(); i < n; i++) p[i] = static_cast<uint8_t>(idx0_h[i] + 1);  // writer takes 1-based
  QCNN_CHECK(FileIO::WriteCbnFile(path, m, bits), "qcnn_write_cbn_u8: cannot write %s", path);
  return 0;
}

}  // extern "C"
