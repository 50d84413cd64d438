/*
 * qcnn.h -- C ABI of the H100-native (sm_90a) product-quantized (PQ) forward path.
 *
 * Drop-in boundary for the reference's CalcFeatMap_ConvAprx / CalcFeatMap_FCntAprx path
 * (CAS-CLab/quantized-cnn, src/CaffeEva.cc).  The reference has no FFI of its own: the path sits behind
 * private C++ members of class CaffeEva (include/CaffeEva.h:145-170).  Each entry point below names the
 * reference member it replaces; INTEGRATION.md shows the binding a maintainer adds inside CaffeEva.cc.
 *
 * Conventions
 *   - plain C types only; every function returns 0 on success, non-zero on error with the text available from
 *     qcnn_last_error() (thread-local).  No exceptions cross the boundary.
 *   - pointers are DEVICE pointers unless the parameter name ends in _h (host).
 *   - `stream` is a cudaStream_t passed as void* (NULL = default stream); forward calls are asynchronous on it.
 *   - activations are fp32; conv/pool/LRN maps are NHWC ([N][H][W][C]) exactly like the reference's featMapLst;
 *     assignment indices are uint8, 0-based, "file order" as CaffePara::layerParaLst holds them after
 *     LoadLayerPara (src/CaffePara.cc:239-306).
 *   - one qcnn_ctx per GPU; a ctx and its layers are not thread-safe; distinct ctxs may be used concurrently.
 *   - there is NO CPU fallback: every compute entry point fails with an error if no sm_90 device is usable.
 */
#ifndef QCNN_H_
#define QCNN_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define QCNN_API __attribute__((visibility("default")))
#else
#define QCNN_API
#endif

typedef struct qcnn_ctx qcnn_ctx;
typedef struct qcnn_layer qcnn_layer;
typedef struct qcnn_net qcnn_net;

/* ---- context ------------------------------------------------------------------------------------------- */
QCNN_API const char* qcnn_version(void);
QCNN_API const char* qcnn_last_error(void);
QCNN_API int qcnn_ctx_create(int device, qcnn_ctx** out);
QCNN_API void qcnn_ctx_destroy(qcnn_ctx* ctx);
QCNN_API int qcnn_ctx_device(const qcnn_ctx* ctx);
QCNN_API int qcnn_ctx_sm_count(const qcnn_ctx* ctx);

/* device-memory helpers: a host program (e.g. the reference's CaffeEva.cc) can drive the library without the CUDA
 * toolkit.  Copies are asynchronous on `stream` when the host buffer is pinned; qcnn_stream_sync waits for it. */
QCNN_API int qcnn_dev_alloc(qcnn_ctx* ctx, size_t bytes, void** out);
QCNN_API int qcnn_dev_free(qcnn_ctx* ctx, void* ptr);
QCNN_API int qcnn_copy_h2d(qcnn_ctx* ctx, void* dst, const void* src_h, size_t bytes, void* stream);
QCNN_API int qcnn_copy_d2h(qcnn_ctx* ctx, void* dst_h, const void* src, size_t bytes, void* stream);
QCNN_API int qcnn_stream_sync(qcnn_ctx* ctx, void* stream);

/* ---- PQ layers (one-time set-up) ---------------------------------------------------------------------------
 * Take the HOST arrays exactly as CaffePara::layerParaLst[l] holds them and do the re-layout + upload that
 * CaffeEva::PrepCtrdBuf / PrepAsmtBuf (src/CaffeEva.cc:534-623) do on the CPU.
 *   ctrd_h  [S][K][d]            f32   (ctrdLst, file order)
 *   asmt_h  [Cout][k][k][S]      u8    (conv asmtLst)   |   [Dout][S] (FC asmtLst), 0-based, values < K
 *   bias_h  [Cout] / [Dout]      f32
 * Conv: ONE codebook is shared by all `grp` groups; group g reads input channels [g*Cin/grp, (g+1)*Cin/grp) and
 * assignment columns [g*Cout/grp, ...) (src/CaffeEva.cc:795-811,847).  Subspace s covers the per-group channels
 * [s*d, s*d + min(Cin/grp - s*d, d)) (src/CaffeEva.cc:1276-1277).
 * FC: K is 16, 32, 64, 128 or 256, and d is bounded so that the LUT + gather kernel, which runs every batch of 5 to 95
 * images and every batch under tensor_core = 0, can stage a chunk of codebook rows in shared memory: d <= 93 (K = 16),
 * 48 (K = 32), 24 (K = 64, 128) or 11 (K = 256).  Larger d is refused at creation, with a message naming K and d.
 * That kernel takes the widest batch tile that fits: at K = 256, 8 images per CTA up to d = 8, 4 up to d = 10, else 1. */
QCNN_API int qcnn_conv_layer_create(qcnn_ctx* ctx, int Cin, int Hin, int Win, int Cout, int ksz, int pad,
                                    int stride, int grp, int S, int K, int d, const float* ctrd_h,
                                    const uint8_t* asmt_h, const float* bias_h, qcnn_layer** out);
QCNN_API int qcnn_fc_layer_create(qcnn_ctx* ctx, int Din, int Dout, int S, int K, int d, const float* ctrd_h,
                                  const uint8_t* asmt_h, const float* bias_h, qcnn_layer** out);
/* FC only: the source is an NHWC map [N][H][W][C] that the reference would first permute to NCHW
 * (CaffeEva.cc:187-189, 236-238); fold that permute into the LUT stage's addressing (H*W*C must equal Din). */
QCNN_API int qcnn_fc_layer_set_src_nhwc(qcnn_layer* layer, int H, int W, int C);
/* Conv only: the source is NCHW [N][C][H][W] (the API input of CaffeEva::ExecForwardPass, CaffeEva.cc:225-228). */
QCNN_API int qcnn_conv_layer_set_src_nchw(qcnn_layer* layer, int enable);
/* tuning overrides for tests/benchmarks: "fc_nsplit" (subspace splits, 0 = automatic; 1 reproduces the reference's
 * accumulation order exactly), "fc_tn" (images per CTA: 1, 4 or 8; 0 = automatic; a tile whose staging does not fit fails the forward), "tensor_core" (2 = default: eligible layers
 * run as decode-at-use GEMMs on the tensor cores with bf16x2 operands; 1 = the same GEMMs with 3xTF32 operands; 0 = LUT +
 * gather kernels only, the fp32 strict-parity path -- tolerances of all three in DESIGN.md);
 * conv layers, for tests that must know which kernel they check: "force_kernel" (-1 none | 0 s1 | 1 roll | 2 s1_tc |
 * 3 roll_tc | 4 direct | 6 pq_gemm_tc | 7 conv_ws: stride-1 layers (NHWC source; Cg % 4 == 0 or Cg <= 3, d % 4 == 0,
 * S*d >= Cg, <= 32 taps, any width whose plane ring fits in shared memory) and strided layers over <= 4 input
 * channels per group, with bf16x2 operands (tensor_core = 2), as a weight-stationary GEMM whose N is the channels of one
 * CTA: Cout/grp or a tile of it, in {16, 32, 64, 96, 128, 192, 256}; describe() names it pq_gemm_tc_ws), "gemm_nt" (positions per CTA of the pq_gemm_tc tilings, and 128 / 256 for conv_ws; 0 = any), "gemm_gt"
 * (k-steps per stage of those tilings, 0 = any), "gemm_nsplit" (their K-split factor, 0 = any), "gemm_ct" (channels per
 * CTA of the conv_ws tilings, 0 = any), "gemm_wb" (conv only: weight stage buffers of the conv_ws tilings' ring, 2, 3
 * or 4, 0 = any; the other families ignore it; a pin that no tiling of the layer matches makes the forward fail), "lut_cpt",
 * "lut_j", "lut_nct", "lut_r", "lut_rgroups" (the LUT + gather tilings, force_kernel 0-4, with that many channels per
 * thread, positions per lane -- conv_direct: output rows per thread --, channel tiles per group, output rows per strip --
 * conv_direct: after its clamp to Ho + (Ho & 1) -- and row groups; 0 = any; a pin that no tiling matches makes the
 * forward fail; describe() prints them as CPT, J, nct, R, rgroups), "autotune"
 * (0 = keep the cost model's first tiling instead of timing the candidates of the chosen family on the device);
 * FC layers only: "fc_ws" (1 = at N >= 96 with bf16x2 operands, run the layer as a weight-stationary
 * GEMM, describe() "pq_gemm_tc_ws(...) mode=2"; 0 = pq_gemm_tc mode 2, the default of a standalone layer; the network
 * executor sets 1 on every FC layer it creates), where "gemm_nt" (images per CTA: 128 / 256), "gemm_gt" (k-steps per
 * stage: 8 / 4), "gemm_ct" (channels per CTA: 64 / 128 / 256) and "gemm_nsplit" (K-split) restrict its tilings, and
 * "asmt_packed" (1 = keep the assignment table in device memory bit-packed at b = log2(K) bits per
 * index instead of one byte, and unpack it inside the FC kernels; 0 = the byte table, the default).  Switching repacks the
 * table on the host, waits for the work queued on the layer's device, frees the previous table and makes graphs captured
 * before stale.  Every FC path (batch <= 4 chain, gather kernel, tensor-core GEMM) makes the same plan and adds the same
 * LUT entries in the same order either way, so outputs are bit-identical; K = 256 is accepted and keeps its byte table.
 * Device layout: row s at byte s * RoundUp(DoutPad * b / 8, 16) (DoutPad = Dout rounded up to 16), channel o in bits
 * [o b, o b + b) of the row as a little-endian bit string.  Fails on a conv layer. */
QCNN_API int qcnn_layer_set_param(qcnn_layer* layer, const char* name, int value);
/* one-line description of the kernel + tiling chosen for batch N (FC layers with a packed table end in " asmt=<b>bit") */
QCNN_API int qcnn_layer_describe(qcnn_layer* layer, int N, char* buf, size_t cap);
QCNN_API void qcnn_layer_destroy(qcnn_layer* layer);
/* out[0..2] = Ho, Wo, Cout (FC: 1, 1, Dout) */
QCNN_API int qcnn_layer_out_dims(const qcnn_layer* layer, int* out3);
/* algorithmic HBM bytes of one forward launch at batch N (SURVEY.md 8(d)) and lookup-add / LUT MAC counts; the
 * assignment term of a packed FC table is S * ceil(Dout * b / 8) bytes */
QCNN_API int qcnn_layer_work(const qcnn_layer* layer, int N, double* alg_bytes, double* lookups, double* lut_macs);
/* device copy of the re-laid-out assignment table, decoded back to plain 0-based indices in the reference's
 * asmtBuf order ([kh][kw][S][Cout] / [S][Dout], CaffeEva.cc:585-586, 610-611) -- for bit-exact index tests */
QCNN_API int qcnn_layer_read_asmt_h(const qcnn_layer* layer, uint8_t* out_h, size_t cap);
/* device copy of a conv layer's weight image, the decoded bf16x2 weights conv_ws streams into shared memory (for
 * byte-exact tests): *bytes = its size, G x entries x 2 x (Cout/grp) x 16 bytes, laid out [grp][entry][w1, w2][Cout/grp]
 * 16-byte rows, an entry being one k-step (stride 1: a chunk of 8 input channels x one tap, chunk by chunk; strided: the
 * k-steps of each phase row in turn).  A k-step has two halves of 4 weights (stride 1: input channels 0-3 and 4-7 of the
 * chunk; strided: a tap and its paired tap), each split as w = w1 + w2 into bf16 pieces: the w1 row holds the 4 w1 of
 * either half, the w2 row the w2; a half the k-step does not have is zero.  0 bytes for a layer without an image (an FC
 * layer, a conv layer conv_ws does not take).  out_h may be NULL to query the size; otherwise cap must be >= *bytes. */
QCNN_API int qcnn_layer_read_w_ws(const qcnn_layer* layer, void* out_h, size_t cap, size_t* bytes);

/* ---- hot path -------------------------------------------------------------------------------------------- */
/* replaces CaffeEva::CalcFeatMap_ConvAprx (src/CaffeEva.cc:760-868) incl. its GetInPdMat call (:810, :1261-1296)
 * src [N][Hin][Win][Cin] -> dst [N][Ho][Wo][Cout]; fuse_relu != 0 additionally applies CalcFeatMap_ReLu (:1027). */
QCNN_API int qcnn_conv_aprx_forward(qcnn_layer* layer, const float* src, int N, float* dst, int fuse_relu,
                                    void* stream);
/* replaces CaffeEva::CalcFeatMap_FCntAprx (src/CaffeEva.cc:968-1025); src [N][Din] -> dst [N][Dout] */
QCNN_API int qcnn_fc_aprx_forward(qcnn_layer* layer, const float* src, int N, float* dst, int fuse_relu,
                                  void* stream);

/* same, but src is always the flat [N][Din] vector in the reference's (NCHW-flatten) feature order, even for a layer
 * whose NHWC fold (qcnn_fc_layer_set_src_nhwc) is enabled -- what CaffeEva::CalcFeatMap_FCntAprx itself receives */
QCNN_API int qcnn_fc_aprx_forward_flat(qcnn_layer* layer, const float* src, int N, float* dst, int fuse_relu,
                                       void* stream);

/* A run of consecutive FC layers of ONE forward pass (the FCnt [ReLU] [Drpt] iterations of the layer loop in
 * CaffeEva::ExecForwardPass, src/CaffeEva.cc:213-261, each iteration being CalcFeatMap_FCntAprx :968-1025) as a single
 * persistent launch; batch <= 4 (the latency path, bound by the HBM stream of the assignment matrices).  relu[l] != 0
 * applies CalcFeatMap_ReLu after layer l.  src [N][Din of layers[0]] (or the NHWC map its set_src_nhwc folds),
 * dst [N][Dout of layers[n-1]].  stamps (nullable, device, 32 * sm_count u64; per CTA: [0],[1] %globaltimer and [2],[3]
 * clock64 at its first / last instruction, [4 + 5 l + i] clock64 after phase i of layer l: input slice, LUT, first
 * assignment chunk landed, gather, publish), for latency measurements.  Fails if the shapes are not supported by the fused kernel
 * (qcnn_fc_aprx_forward per layer always works). */
QCNN_API int qcnn_fc_chain_forward(qcnn_layer* const* layers, const int* relu, int n, const float* src, int N,
                                   float* dst, unsigned long long* stamps, void* stream);

/* ---- supporting layers (src/CaffeEva.cc:1027-1116, 870-921) ---------------------------------------------- */
QCNN_API int qcnn_relu(qcnn_ctx* ctx, const float* src, float* dst, size_t n, void* stream);
QCNN_API int qcnn_lrn(qcnn_ctx* ctx, const float* src, float* dst, size_t pixels, int C, int size, float alpha,
                      float beta, float k, void* stream);
QCNN_API int qcnn_maxpool(qcnn_ctx* ctx, const float* src, float* dst, int N, int H, int W, int C, int ksz,
                          int pad, int stride, void* stream);
/* LRN followed by max-pool in one pass (the reference always runs them back to back in AlexNet-family tables) */
QCNN_API int qcnn_lrn_maxpool(qcnn_ctx* ctx, const float* src, float* dst, int N, int H, int W, int C, int size,
                              float alpha, float beta, float k, int ksz, int pad, int stride, void* stream);
QCNN_API int qcnn_softmax(qcnn_ctx* ctx, const float* src, float* dst, int N, int C, void* stream);
QCNN_API int qcnn_nchw_to_nhwc(qcnn_ctx* ctx, const float* src, float* dst, int N, int C, int H, int W,
                               void* stream);
QCNN_API int qcnn_nhwc_to_nchw(qcnn_ctx* ctx, const float* src, float* dst, int N, int H, int W, int C,
                               void* stream);

/* ---- whole network (CaffeEva::LoadCaffePara + ExecForwardPass, src/CaffeEva.cc:109-149, 213-261) ------------
 * Layer table record == the reference's LayerInfo (include/CaffePara.h:28-41); type uses ENUM_LyrType order. */
enum { QCNN_CONV = 0, QCNN_POOL = 1, QCNN_FCNT = 2, QCNN_RELU = 3, QCNN_LORN = 4, QCNN_DRPT = 5, QCNN_SMAX = 6 };
typedef struct {
  int type;
  int padSiz, knlSiz, knlCnt, grpCnt, stride, nodCnt, lrnSiz;
  float lrnAlp, lrnBet, lrnIni, drpRat;
} qcnn_layer_info;

/* model_name: "AlexNet" | "CaffeNet" | "VggCnnS" | "VGG16" | "CaffeNetFGB" | "CaffeNetFGD" (CaffeEva.cc:117-132);
 * parameters are read from <dir>/<pfx>.{biasVec,ctrdLst}.NN.bin and <pfx>.asmtLst.NN.cbn (CaffePara.cc:262-281). */
QCNN_API int qcnn_net_create(qcnn_ctx* ctx, const char* model_name, const char* dir, const char* pfx,
                             qcnn_net** out);
QCNN_API int qcnn_net_create_custom(qcnn_ctx* ctx, int layer_cnt, const qcnn_layer_info* layers, int img_chn,
                                    int img_hei, int img_wid, const char* dir, const char* pfx, qcnn_net** out);
/* Same, from parameters the caller already holds in host memory -- what CaffeEva::LoadCaffePara has after
 * CaffePara::LoadLayerPara (src/CaffeEva.cc:134-139): one record per layer == the reference's LayerPara
 * (include/CaffePara.h:45-58) restricted to the PQ members; all pointers NULL for layers without parameters.
 *   ctrd [S][K][d] f32 (ctrdLst), asmt u8 0-based ([Cout][k][k][S] conv / [Dout][S] FC, asmtLst), bias f32 (biasVec) */
typedef struct {
  const float* ctrd;
  const uint8_t* asmt;
  const float* bias;
  int S, K, d;
} qcnn_layer_para;
QCNN_API int qcnn_net_create_from_para(qcnn_ctx* ctx, int layer_cnt, const qcnn_layer_info* layers,
                                       const qcnn_layer_para* para, int img_chn, int img_hei, int img_wid,
                                       qcnn_net** out);
QCNN_API void qcnn_net_destroy(qcnn_net* net);
QCNN_API int qcnn_net_layer_count(const qcnn_net* net);
QCNN_API int qcnn_net_out_len(const qcnn_net* net);
/* keep != 0: every feature map featMapLst[0..layerCnt] is materialised un-fused (parity tests); default 0: ReLU is
 * fused into the producing PQ kernel, LRN+pool are fused, dropout is elided. */
QCNN_API int qcnn_net_set_keep_maps(qcnn_net* net, int keep);
/* device-resident forward: img [N][C][H][W] (NCHW, as ExecForwardPass takes it) -> prob [N][out_len];
 * logits (nullable) receives the input of the final softmax layer. */
QCNN_API int qcnn_net_forward(qcnn_net* net, const float* img, int N, float* prob, float* logits, void* stream);
/* host-buffer forward == CaffeEva::ExecForwardPass(imgDataIn, pProbVecOut): H2D, forward, D2H, synchronises. */
QCNN_API int qcnn_net_forward_h(qcnn_net* net, const float* img_h, int N, float* prob_h, float* logits_h);
/* same, with the k-fold arg-max of CaffeEvaWrapper::Proc (src/CaffeEvaWrapper.cc:188-206; topk_mode 0) or
 * CaffeEva::CvtFeatMapToLablVec (src/CaffeEva.cc:1162-1190: the scan starts from FLT_MIN; topk_mode 1) done on the
 * device: topk_idx_h [N][topk] int32 and topk_prob_h [N][topk] come back instead of (prob_h nullable) the whole rows */
QCNN_API int qcnn_net_forward_topk_h(qcnn_net* net, const float* img_h, int N, int topk, int topk_mode, int* topk_idx_h,
                                     float* topk_prob_h, float* prob_h);
/* uint8 entry: images as interleaved pixels [N][H][W][C] (C = B, G, R for the shipped models), the crop-sized mean image
 * [C][H][W] (NULL: none) subtracted on the device -- (float)pixel - mean, the element BmpImgIO::RmMeanImg produces
 * (src/BmpImgIO.cc:203-224) -- before the first layer.  4x fewer bytes cross the host link than with fp32 tensors. */
QCNN_API int qcnn_net_set_input_mean(qcnn_net* net, const float* mean_h);
QCNN_API int qcnn_net_forward_u8(qcnn_net* net, const uint8_t* img, int N, float* prob, float* logits, void* stream);
/* host pixels in, top-k (topk > 0) and / or probabilities (prob_h != NULL) out; synchronises */
QCNN_API int qcnn_net_forward_u8_h(qcnn_net* net, const uint8_t* img_h, int N, int topk, int topk_mode, int* topk_idx_h,
                                   float* topk_prob_h, float* prob_h);
/* asynchronous form: queues copy-in, conversion, forward pass, top-k and copy-out, then returns a ticket (0 or 1); the
 * host buffers (pinned, or the copies are not asynchronous) belong to the step until qcnn_net_wait(ticket).  Two tickets
 * may be outstanding -- the pixels of step i+1 travel while step i computes -- and a third submit first waits for the
 * ticket two steps back.  Do not mix with the synchronous host entry points while tickets are outstanding. */
QCNN_API int qcnn_net_submit_u8_h(qcnn_net* net, const uint8_t* img_h, int N, int topk, int topk_mode, int* topk_idx_h,
                                  float* topk_prob_h, float* prob_h, int* ticket);
QCNN_API int qcnn_net_wait(qcnn_net* net, int ticket);
/* images per pipeline chunk of the host-buffer entry points (default 128; the first chunk of a call is a quarter of
 * that): H2D of chunk c+1 overlaps the layers of chunk c */
QCNN_API int qcnn_net_set_chunk(qcnn_net* net, int chunk);
/* qcnn_layer_set_param(layer, "asmt_packed", enable) for every FC layer of the net (multi-GPU: call it on every
 * replica, qcnn_multi_net); the batch-1 graph is recaptured on the next forward */
QCNN_API int qcnn_net_set_asmt_packed(qcnn_net* net, int enable);
/* after a forward with keep_maps: device pointer + dims [N,H,W,C] of featMapLst[idx] */
QCNN_API int qcnn_net_featmap(qcnn_net* net, int idx, const float** ptr, int* dims4);
/* per-layer CUDA-event timing of the LAST forward (ms); enable before the forward.  Mirrors the reference's
 * swIndvLayerLst stop-watches (CaffeEva.cc:192-194, 317-320). */
QCNN_API int qcnn_net_set_profiling(qcnn_net* net, int enable);
QCNN_API int qcnn_net_layer_time_ms(qcnn_net* net, int layer, float* ms);
QCNN_API int qcnn_net_layer_work(qcnn_net* net, int layer, int N, double* alg_bytes, double* lookups,
                                 double* lut_macs);
/* number of kernels the last forward launched */
QCNN_API int qcnn_net_launch_count(const qcnn_net* net);
/* PQ layer handle of layer `l` (NULL for non-PQ layers); owned by the net */
QCNN_API qcnn_layer* qcnn_net_pq_layer(qcnn_net* net, int l);

/* ---- image entry and result exit on the device (SURVEY.md 8(f1), 8(f2)) -------------------------------------------
 * k-fold arg-max of N rows of C values: first maximum wins, winner zeroed (mode: see qcnn_net_forward_topk_h);
 * 1 <= k <= C <= 12000.  NaNs follow the reference scans: mode 0 returns (0, NaN) for a row starting with NaN and
 * otherwise skips them, mode 1 always skips them.  idx [N][k] int32, val [N][k], device */
QCNN_API int qcnn_topk(qcnn_ctx* ctx, const float* prob, int N, int C, int k, int mode, int* idx, float* val, void* stream);
/* src u8 [N][H][W][C] -> dst f32 [N][C][H][W] minus mean [C][H][W] (nullable), device */
QCNN_API int qcnn_u8hwc_to_f32chw(qcnn_ctx* ctx, const uint8_t* src, const float* mean, float* dst, int N, int C, int H, int W,
                                  void* stream);
/* BmpImgIO on the device: == BmpImgIO::Init (src/BmpImgIO.cc:28-38).  resz_type 0 Strict / 1 Relaxed, mean_type 0 Full /
 * 1 Crop (include/BmpImgIO.h:19-20); mean_h [3][mean_hei][mean_wid] in B, G, R plane order (imagenet_mean.single.bin) */
typedef struct qcnn_preproc qcnn_preproc;
QCNN_API int qcnn_preproc_create(qcnn_ctx* ctx, int resz_type, int mean_type, int hei_full, int wid_full, int hei_crop,
                                 int wid_crop, const float* mean_h, int mean_hei, int mean_wid, qcnn_preproc** out);
QCNN_API void qcnn_preproc_destroy(qcnn_preproc* p);
/* == BmpImgIO::Load after the file decode -- ReszImg, RmMeanImg, CropImg (src/BmpImgIO.cc:105-224) -- for N decoded
 * images in one launch, bit-identical to the CPU path: pix (device) holds the images' interleaved B, G, R bytes, top row
 * first, image i of hei_h[i] x wid_h[i] pixels starting at byte off_h[i] (host arrays); dst [N][3][hei_crop][wid_crop]
 * f32 NCHW (device), what ExecForwardPass takes.  Runs of one object on one stream are ordered; one object must not
 * run on two streams at once (they share its descriptor buffer) */
QCNN_API int qcnn_preproc_run(qcnn_preproc* p, const uint8_t* pix, const long long* off_h, const int* hei_h, const int* wid_h,
                              int N, float* dst, void* stream);

/* ---- multi-GPU (SURVEY.md 8(e)): ONE process drives n_dev GPUs of a box -----------------------------------------
 * The batch is sharded by image (rank r owns rows [r*per, min(N, (r+1)*per)), per = ceil(N / n_dev)), the weights are
 * replicated, and the only exchange is one ncclAllGather of the per-rank probabilities over NVLink, after which every
 * GPU holds the [N][out_len] result -- what CaffeEva::ExecForwardPass (src/CaffeEva.cc:213-261) leaves in
 * featMapLst[layerCnt].  devices == NULL means 0 .. n_dev-1.  NCCL is loaded at run time (libnccl.so.2); the calls fail
 * if it is missing (no host-staged fallback). */
typedef struct qcnn_multi qcnn_multi;
QCNN_API int qcnn_multi_create(int n_dev, const int* devices, const char* model_name, const char* dir, const char* pfx,
                               qcnn_multi** out);
QCNN_API int qcnn_multi_create_from_para(int n_dev, const int* devices, int layer_cnt, const qcnn_layer_info* layers,
                                         const qcnn_layer_para* para, int img_chn, int img_hei, int img_wid,
                                         qcnn_multi** out);
QCNN_API void qcnn_multi_destroy(qcnn_multi* m);
QCNN_API int qcnn_multi_device_count(const qcnn_multi* m);
QCNN_API int qcnn_multi_out_len(const qcnn_multi* m);
QCNN_API int qcnn_multi_nccl_version(const qcnn_multi* m);
/* the replica of rank `rank` (owned by m): for qcnn_net_pq_layer / qcnn_layer_set_param on every replica */
QCNN_API qcnn_net* qcnn_multi_net(qcnn_multi* m, int rank);
/* == CaffeEva::ExecForwardPass(imgDataIn, pProbVecOut) on n_dev GPUs: img_h [N][C][H][W] host (pinned for concurrent
 * copies), prob_h [N][out_len] host; shards go up on every GPU's own link, forward, all-gather, rank 0's copy comes
 * back; synchronises. */
QCNN_API int qcnn_multi_forward_h(qcnn_multi* m, const float* img_h, int N, float* prob_h);
/* device-resident, asynchronous step: img_dev[r] = rank r's shard on device r; prob_all_dev[r] (nullable array) receives
 * the device-r pointer of the gathered [N][out_len] probabilities (library-owned, valid until the step after next).  The
 * all-gather runs on a side stream, so consecutive steps overlap it with the next step's layers; qcnn_multi_sync waits
 * for everything issued. */
QCNN_API int qcnn_multi_forward(qcnn_multi* m, const float* const* img_dev, int N, const float** prob_all_dev);
QCNN_API int qcnn_multi_sync(qcnn_multi* m);

/* ---- product quantization of dense weights (DESIGN.md 4e) ------------------------------------------------------
 * Per subspace s of d input channels, Lloyd k-means over the weight sub-vectors, on the device; synchronous, host arrays.
 * Points: conv p = (o k + kh) k + kw over all Cout channels (one codebook for all groups), x_p[j] = knl[o][s d + j][kh][kw];
 * FC p = o, x_p[j] = wei[o][s d + j]; j < w_s = min(d, Cg - s d) (FC: Din), S = ceil(Cg / d).  Distances are fp32 in
 * ascending j, the lowest index wins ties, means are fp64 sums in a fixed order, an empty cluster keeps its codeword and
 * codebook dims j >= w_s are 0.  a_0 = assign(C_0); then iters x (update, assign): every returned index is the nearest
 * codeword of the returned codebook.  sse_h[t] (nullable, iters + 1 values) = sum over all points and subspaces of the
 * distance to the assigned codeword after step t.  C_0 = init_ctrd_h [S][K][d] when given, else per subspace the points
 * perm[0..K-1] of an LCG partial shuffle: x = seed + s; for i < K: x = 1664525 x + 1013904223 (mod 2^32),
 * j = i + (x >> 8) mod (P - i), swap(perm[i], perm[j]).  Results are bit-reproducible.  Fails on non-finite weights, K that
 * the matching layer_create refuses (conv: multiple of 8; FC: 16, 32, 64, 128, 256), d outside 1..64, iters < 0, more than
 * 2^24 points, or fewer points than K without an init codebook. */
QCNN_API int qcnn_pq_quantize_conv(qcnn_ctx* ctx, int Cout, int Cg, int ksz, int K, int d, int iters, uint32_t seed,
                                   const float* knl_h /*[Cout][Cg][k][k]*/, const float* init_ctrd_h /*nullable [S][K][d]*/,
                                   float* ctrd_h /*[S][K][d]*/, uint8_t* asmt_h /*[Cout][k][k][S], 0-based*/,
                                   double* sse_h /*nullable [iters+1]*/);
QCNN_API int qcnn_pq_quantize_fc(qcnn_ctx* ctx, int Din, int Dout, int K, int d, int iters, uint32_t seed,
                                 const float* wei_h /*[Dout][Din]*/, const float* init_ctrd_h, float* ctrd_h,
                                 uint8_t* asmt_h /*[Dout][S]*/, double* sse_h);
/* model table by name (as qcnn_net_create): reads <dir>/<pfx>.{convKnl|fcntWei,biasVec}.NN.bin (CaffePara::LoadLayerPara
 * with enblAprx = false), writes <out_dir>/<out_pfx>.{ctrdLst,biasVec}.NN.bin and .asmtLst.NN.cbn (bits of the 1-based
 * maximum K); K[l], d[l] per layer index (ignored for non-PQ layers); layer l uses seed + 65536 (l + 1) and a random
 * init.  Dense shapes are checked against the table; biasVec is copied unchanged; no file is written unless every
 * layer is quantized, and none is left behind by a failed write. */
QCNN_API int qcnn_pq_quantize_model(qcnn_ctx* ctx, const char* model_name, const char* dir, const char* pfx,
                                    const int* K, const int* d, int iters, uint32_t seed,
                                    const char* out_dir, const char* out_pfx);
/* Error-correcting PQ of an FC layer (DESIGN.md 4e): block coordinate descent on (ctrd, asmt) that lowers
 * loss = sum_n |(W - W^) x_n|^2 = sum_o E_o^T G E_o, E = W - W^ (fp64), G = X^T X (fp64, fixed order), on the inputs
 * x [N][Din] (device, fcntWei column order).  A sweep visits m = 0..S-1 in order; subspace m (dims m d .. m d + w_m - 1)
 * is skipped when tr(G_mm) = 0, else with h_o = [G E_o]_m + G_mm w^_o:  for every non-empty cluster k,
 * D = fp32((G_mm + lambda I)^-1 H_k / n_k) by Cholesky (H_k = sum of h_o over the cluster, lambda = 1e-10 tr(G_mm) / w_m)
 * replaces c_k only if f(D) < f(c_k), f(D) = n_k D^T G_mm D - 2 D^T H_k; then a_o = argmin_k c_k^T G_mm c_k - 2 c_k^T h_o
 * (lowest index on ties), and E is updated before m + 1.  ctrd_h [S][K][d] and asmt_h [Dout][S] (0-based) are the start
 * and receive the result; loss_h (nullable, sweeps + 1 values) = the start's loss, then the loss after each sweep.
 * Results are bit-reproducible.  Runs on `stream` (ordered after whatever produced x) and synchronises it before
 * returning.  Device memory: 8 Din^2 bytes for G plus about 20 Dout Din bytes (E and G E^T in fp64, the weights in
 * fp32).  Fails on what
 * qcnn_pq_quantize_fc refuses (K, d, non-finite weights or codebook), sweeps < 0, N < 1, an assignment >= K, non-finite
 * x, or a failed allocation (with its byte count). */
QCNN_API int qcnn_pq_refine_fc(qcnn_ctx* ctx, int Din, int Dout, int K, int d, int sweeps,
                               const float* wei_h /*[Dout][Din]*/, const float* x /*device [N][Din]*/, int N,
                               float* ctrd_h /*in/out [S][K][d]*/, uint8_t* asmt_h /*in/out [Dout][S], 0-based*/,
                               double* loss_h /*nullable [sweeps + 1]*/, void* stream);
/* Error-correcting PQ of a conv layer (DESIGN.md 4e): block coordinate descent on (ctrd, asmt) that lowers
 * loss = sum_{n,o,y,x} conv(x, W - W^)^2 = sum_g sum_{o in g} E_o^T G_g E_o, E = W - W^ (fp64), on the layer inputs
 * x [N][Hin][Win][Cin] (device, NHWC: what Net.featmap returns for the layer's input under keep_maps).  Geometry as
 * qcnn_conv_layer_create; Cg = Cin / grp, S = ceil(Cg / d), subspace m covers the per-group channels m d .. m d + w_m - 1,
 * tap t = kh k + kw, output o is in group o / (Cout / grp), and one codebook serves all taps and groups.
 * G_g = sum p p^T (fp64, fixed order, exactly symmetric) over every image and output position, p the zero-padded
 * Cg k^2 patch of group g's channels.  A sweep visits m = 0..S-1 in order; m is skipped when sum_g sum_t tr G^m_{g,tt} = 0
 * (G^m_{g,tt'}: the w_m x w_m block of G_g between the dims of (m, t) and (m, t')), else:
 *   h_{o,t} = [G_g R_o]_(m,t), R_o = E_o + W^_o(m) (the residual of the other subspaces);
 *   codebook: over U = {k : n_k > 0} (ascending), M = sum_g sum_{t,t'} Cnt^g_{tt'} (x) G^m_{g,tt'} (Cnt^g_{tt'}[k][k'] =
 *     |{o in g : A[o][t][m] = k, A[o][t'][m] = k'}|, g, t, t' ascending), b_k = sum of h_{o,t} over A[o][t][m] = k
 *     (o, then t ascending); D = fp32((M + mu I)^-1 b) by fp64 Cholesky, mu = 1e-10 tr(M) / (|U| w_m), replaces C[m][U]
 *     only if (D - C)^T (M (D + C) - 2 b) < 0; empty clusters keep their codeword, dims j >= w_m stay 0;
 *   assignment: taps t = 0..k^2-1 in order, per output A[o][t][m] = argmin_k c_k^T G^m_{g,tt} c_k - 2 c_k^T h'_{o,t} (fp64,
 *     lowest index on ties), h'_{o,t} = [G_g E_o]_(m,t) + G^m_{g,tt} w^_{o,t} with E current (earlier taps' changes
 *     included); a (g, t) with tr G^m_{g,tt} = 0 keeps its assignments; E is updated before m + 1.
 * ctrd_h [S][K][d] and asmt_h [Cout][k][k][S] (0-based) are the start and receive the result; loss_h (nullable, sweeps + 1
 * values) = the start's loss, then the loss after each sweep.  Results are bit-reproducible.  Runs on `stream` (ordered
 * after whatever produced x) and synchronises it before returning.  Device memory: 8 grp (Cg k^2)^2 bytes for the Grams,
 * 20 Cout Cg k^2 for E, G E and the weights, 16 (K min(d, Cg))^2 for M and its factor, and 24 Cout k^2 min(d, Cg) for
 * one subspace's responses; the Grams read the patches straight from x.  Fails on what qcnn_pq_quantize_conv refuses (K not
 * a multiple of 8 in 8..256, d outside 1..64, non-finite weights or codebook), non-finite x, sweeps < 0, N < 1, an
 * assignment >= K, Cin or Cout not divisible by grp, an empty output, K min(d, Cg) > 2048 (the size of the joint
 * system), or a failed allocation (with its byte count). */
QCNN_API int qcnn_pq_refine_conv(qcnn_ctx* ctx, int Cin, int Hin, int Win, int Cout, int ksz, int pad, int stride,
                                 int grp, int K, int d, int sweeps,
                                 const float* knl_h /*[Cout][Cin/grp][k][k]*/,
                                 const float* x /*device NHWC [N][Hin][Win][Cin]*/, int N,
                                 float* ctrd_h /*in/out [S][K][d]*/, uint8_t* asmt_h /*in/out [Cout][k][k][S], 0-based*/,
                                 double* loss_h /*nullable [sweeps + 1]*/, void* stream);
/* Error-correcting PQ toward target responses (DESIGN.md 4e, the paper's multi-layer error correction): the layer's
 * inputs y come from the quantized network (every earlier layer already quantized) and the targets t are the original
 * network's responses of the layer, without bias and before ReLU (e.g. t_n = W x_n on the original network's input x_n).
 * The calls lower loss = sum_n |t_n - W^ y_n|^2 and take no dense weights: the targets carry what the weights did.
 * FC: y [N][Din] and t [N][Dout] on the device; G = Y^T Y exactly as qcnn_pq_refine_fc forms it (same kernel and order,
 * so bit-identical for the same y), P = T^T Y (fp64 [Dout][Din], k ascending in the GEMM's fixed steps), and
 * loss = |T|^2 - 2 sum_o w^_o^T P_o + sum_o w^_o^T G w^_o.  The sweeps are those of qcnn_pq_refine_fc (skip rule, Cholesky
 * codebook step with strict acceptance, argmin with the lowest index on ties, Gauss-Seidel order) with the residual
 * response h_o = [R_o]_m + G_mm w^_o(m), R_o = P_o - G w^_o, in place of G E_o.
 * Conv: y [N][Hin][Win][Cin] and t [N][Ho][Wo][Cout] (NHWC) on the device, geometry as qcnn_pq_refine_conv;
 * P_g[o][q] = sum over every image and output position of t[pos][o] p_g(pos)[q] for o in group g (p_g the zero-padded
 * patch of y, accumulated over the same patch chunks in the same ascending order as G_g), and R = P - G W^ replaces G E
 * everywhere in qcnn_pq_refine_conv's sweep (h_{o,t}, h'_{o,t} and the update after each subspace); the joint codebook
 * system, the tap-ordered assignment, the skip rule and every tie rule are unchanged.  The loss is formed as for FC.
 * loss_h (nullable, sweeps + 1 values) = the start's loss, then the loss after each sweep.  This loss is a difference of
 * large terms: its absolute rounding error is of order 1e-15 (|T|^2 + sum_o w^_o^T G w^_o), so it can rise by that much
 * across a sweep.  |T|^2 is an fp64 sum of fp32 squares, which cannot overflow: it is non-finite exactly when t holds a
 * NaN or Inf.  Results are bit-reproducible.  Runs on `stream` and synchronises it.  Device memory: that of the
 * same-input call plus 8 Dout Din bytes for P (FC) or 8 Cout Cg k^2 (conv).  Fails on what the same-input call refuses
 * apart from the weight checks (K, d, sweeps < 0, N < 1, an assignment >= K, a non-finite codebook, non-finite y, the
 * conv geometry, the joint-system limit, a failed allocation with its byte count), and on a NULL or non-finite t. */
QCNN_API int qcnn_pq_refine_fc_target(qcnn_ctx* ctx, int Din, int Dout, int K, int d, int sweeps,
                                      const float* y /*device [N][Din]*/, const float* t /*device [N][Dout]*/, int N,
                                      float* ctrd_h /*in/out [S][K][d]*/, uint8_t* asmt_h /*in/out [Dout][S], 0-based*/,
                                      double* loss_h /*nullable [sweeps + 1]*/, void* stream);
QCNN_API int qcnn_pq_refine_conv_target(qcnn_ctx* ctx, int Cin, int Hin, int Win, int Cout, int ksz, int pad, int stride,
                                        int grp, int K, int d, int sweeps,
                                        const float* y /*device NHWC [N][Hin][Win][Cin]*/,
                                        const float* t /*device NHWC [N][Ho][Wo][Cout]*/, int N,
                                        float* ctrd_h /*in/out [S][K][d]*/, uint8_t* asmt_h /*in/out [Cout][k][k][S], 0-based*/,
                                        double* loss_h /*nullable [sweeps + 1]*/, void* stream);
/* Calibration statistics of one layer for one subspace width d (DESIGN.md 4e), so that the calibration set can be
 * streamed in batches: the refine calls above reduce their inputs to sums over images before the first sweep (G, and for
 * the target form P and |T|^2), and these objects accumulate those sums batch by batch.  Device memory does not depend
 * on the number of images: an FC object holds 8 Din^2 bytes (plus 8 Dout Din for a target object), a conv object
 * 8 grp Dg^2 (plus 8 Cout Dg), Dg = Cg k^2, and about 4 KiB more.  The qcnn_pq_refine_* calls above are create, one add
 * of all N images, refine and destroy on these objects.
 * Dim order: FC, the input column; conv, the internal order of the refine code for d, q = m d k^2 + t w_m + j (subspace
 *   m, tap t = kh k + kw, channel m d + j of the group, w_m = min(d, Cg - m d)), so each G^m is a diagonal block.
 * Accumulation order (normative; one add of all N images is exactly the arithmetic of the one-shot call):
 *   FC: an add is one fold, G <- G + Y_b^T Y_b and P <- P + T_b^T Y_b, each a fresh fixed-order GEMM; the first add
 *   stores instead of adding.  Conv: an add folds its positions (n Ho + oy) Wo + ox (n counted within the batch) in runs
 *   of F = max(1, min(P_b, floor(2^28 / (4 Dg)))) positions, each run a fresh sum over 16-position k-steps in ascending
 *   order, added to G_g (and P_g) in ascending order.  |T|^2 <- |T|^2 + |T_b|^2, |T_b|^2 a fixed-order fp64 sum of the
 *   fp32 squares.
 * create: target != 0 also keeps P and |T|^2 (and then every add needs t).  Fails on the geometry the matching refine
 *   call refuses, d outside 1..64, or a failed allocation.
 * add: scans y and (target) t for NaN or Inf, synchronising `stream` once, then queues the accumulation on `stream` and
 *   returns; y and t must stay valid until the stream reaches it.  A rejected add (non-finite y or t, t given to a
 *   same-input object or missing on a target object, N < 1, NULL y) leaves the statistics and the count unchanged.
 * read_h: waits for the queued adds and copies each non-NULL output (G [grp][Dg][Dg], FC [Din][Din]; P [Cout][Dg], FC
 *   [Dout][Din]; |T|^2 one double); P and |T|^2 need a target object.  Before any add the sums are zero.
 * refine / refine_target: the sweeps of qcnn_pq_refine_{fc,conv} / _target on the statistics, with the same arguments,
 *   results and checks (K, the joint-system limit, an assignment >= K, a non-finite codebook or weights) plus a call
 *   before any add; refine works on either kind of object (it reads only G), refine_target needs a target object.  They
 *   read the statistics and never change them, so either may run any number of times.  They wait for the queued adds,
 *   run on `stream` and synchronise it; device memory is that of the one-shot call less G and P.
 * First moments (for the bias refit below): every object also sums, in fp64, s = the sum of y (FC [Din]; conv [grp][Dg]
 *   in the dim order above, the zero-padded patches summed over every image and output position, so a tap outside the map
 *   adds 0) and, for a target object, u = the sum of t (FC [Dout]; conv [Cout], over every image and output position);
 *   n = the rows summed: images (FC) or images Ho Wo (conv).  Fold rule (normative): each add forms its batch's sums
 *   fresh, in a fixed order that does not depend on the values, and adds them to the running sums with one addition per
 *   element; the first add stores instead of adding.  So adds of y and -y leave s = 0 exactly, and the same sequence of
 *   adds gives the same bits.  The sums are queued after the scan, so a rejected add leaves them unchanged.  They take
 *   8 (Din + Dout) bytes (FC) or 8 (grp Dg + Cout) (conv; u only for a target object), and a conv object another
 *   8 Hin Win Cin (target: 8 max(Hin Win Cin, Ho Wo Cout)) for an add's per-image-position sum.
 * read_sums_h: waits for the queued adds and copies each non-NULL output; u needs a target object.
 * refine_bias / refine_target_bias: refine / refine_target with the bias free as well.  For fixed W^ the best bias is
 *   b^ = b + mean(t - W^ y) (target) or b + (W - W^) mean(y) (same input); with it the loss is the same quadratic in the
 *   centered sums, so the unchanged sweeps run on centered copies, formed elementwise with every operation rounded (no
 *   contraction): Gc[i][j] = G[i][j] - (s[i] s[j]) / n (per group for conv; exactly symmetric), Pc[o][q] = P[o][q] -
 *   (u[o] s_g[q]) / n, |T_c|^2 = |T|^2 - sum over o ascending of (u[o] u[o]) / n.  Every rule of the sweeps (skip, ridge,
 *   acceptance, ties) is evaluated on the centered sums.  Then, in fp64 from the final (ctrd, asmt) and g the group of
 *   output o: delta_o = (u_o - w^_o . s_g) / n (target) or (w_o - w^_o) . s_g / n (same input), and bias_h[o] becomes
 *   fp32(bias_h[o] + delta_o).  loss_h = the bias-optimal loss: the start's, then one value after each sweep.  The calls
 *   reject what refine / refine_target reject, plus a NULL or non-finite bias_h; they never change the statistics.
 *   Device memory: that of refine / refine_target plus the centered copies, 8 Din^2 (+ 8 Dout Din for the target form)
 *   bytes (FC; VGG16 fc6: +5.0 GB) or 8 grp Dg^2 (+ 8 Cout Dg) (conv).
 * Skip rule of every sweep: a subspace (conv: a (group, tap) in the assignment step) is skipped when !(tr > 0) for the
 *   trace of its diagonal block, so a centered block with a rounding-level negative trace is skipped; on raw sums the
 *   trace is a sum of squares, so this is tr == 0.  A codeword solve that is not finite (a centered block that is
 *   singular at rounding level) fails the strict acceptance test and never enters the codebook.
 * refine_damped: the sweeps with a damping term that pulls the fit toward the original weights W (wei_h, fcntWei /
 *   convKnl, required in both forms), minimising loss + sum_g lambda_g |W_g - W^_g|_F^2 over the groups g.  target = 0 runs
 *   the same-input form on either kind of object, target = 1 the target form on a target object; bias_h NULL runs on the
 *   raw sums, otherwise on the centered sums with the bias refit of refine_bias / refine_target_bias (the damping term
 *   does not involve the bias, so its closed form is unchanged).  Base sums: the sums those calls' sweeps read.
 *   Per group, on the base sums: tr_g = sum over i ascending of G_g[i][i] (fp64), lambda_g = damp (tr_g / Dg) with each
 *   operation rounded, and lambda_g = 0 when !(tr_g > 0) (such a group is skipped as before); FC is one group, Dg = Din.
 *   The sweeps run unchanged (skip rule, ridge, acceptance, ties, order) on damped copies formed elementwise with every
 *   operation rounded (no contraction): G'_g[i][i] = G_g[i][i] + lambda_g, every other entry copied (so G' stays exactly
 *   symmetric); target form: P'[o][q] = P[o][q] + lambda_g W[o][q] (W in the dim order above, g the group of output o)
 *   and |T'|^2 = |T|^2 + (sum over g ascending of lambda_g |W_g|^2), |W_g|^2 the fixed-order fp64 sum of group g's squared
 *   weights; |T'|^2 enters only the reported loss.  With lambda_g > 0 no subspace of group g has a zero trace, so a
 *   subspace without input energy is no longer skipped: its codewords and assignments are fitted to W in the Euclidean
 *   metric, which is what the damping term asks for.  loss_h = the damped objective (bias-optimal with bias_h): the
 *   start's, then one value after each sweep.  damp = 0 gives the bits of refine, refine_target, refine_bias or
 *   refine_target_bias, whichever matches.  Rejects what those calls reject, plus a NULL wei_h, damp < 0, NaN or Inf,
 *   target not 0 or 1, target = 1 on a same-input object, and non-finite weights in either form; never changes the
 *   statistics.  Device memory: that of the matching call plus the damped copies, 8 grp Dg^2 (+ 8 Cout Dg for the target
 *   form) bytes, and for the target form 4 Cout Dg bytes of weights until the sweeps start; with bias_h the centered
 *   copies are damped in place, so no more than refine_bias / refine_target_bias. */
typedef struct qcnn_pq_stats qcnn_pq_stats;
QCNN_API int qcnn_pq_stats_create_fc(qcnn_ctx* ctx, int Din, int Dout, int d, int target, qcnn_pq_stats** out);
QCNN_API int qcnn_pq_stats_create_conv(qcnn_ctx* ctx, int Cin, int Hin, int Win, int Cout, int ksz, int pad, int stride,
                                       int grp, int d, int target, qcnn_pq_stats** out);
/* y: device [N][Din] / NHWC [N][Hin][Win][Cin]; t: device [N][Dout] / NHWC [N][Ho][Wo][Cout], NULL unless target */
QCNN_API int qcnn_pq_stats_add(qcnn_pq_stats* s, const float* y, const float* t, int N, void* stream);
QCNN_API int qcnn_pq_stats_count(const qcnn_pq_stats* s, long long* images);
/* host copies (each nullable): G [grp][Dg][Dg] (FC: [Din][Din]), P [Cout][Dg] (FC: [Dout][Din]), |T|^2 */
QCNN_API int qcnn_pq_stats_read_h(const qcnn_pq_stats* s, double* G_h, double* P_h, double* tt_h);
QCNN_API int qcnn_pq_stats_refine(qcnn_pq_stats* s, int K, int sweeps, const float* wei_h /* fcntWei or convKnl */,
                                  float* ctrd_h, uint8_t* asmt_h, double* loss_h, void* stream);
QCNN_API int qcnn_pq_stats_refine_target(qcnn_pq_stats* s, int K, int sweeps, float* ctrd_h, uint8_t* asmt_h,
                                         double* loss_h, void* stream);
/* s [grp][Dg] (FC [Din]), internal dim order; u [Cout] (FC [Dout]), target objects only; n = images (FC) or images*Ho*Wo */
QCNN_API int qcnn_pq_stats_read_sums_h(const qcnn_pq_stats* s, double* s_h, double* u_h, long long* n_h);
/* refine / refine_target on the centered sums; bias_h [Dout] / [Cout] in/out: the layer's bias, replaced by the refit one */
QCNN_API int qcnn_pq_stats_refine_bias(qcnn_pq_stats* s, int K, int sweeps, const float* wei_h, float* ctrd_h,
                                       uint8_t* asmt_h, float* bias_h, double* loss_h, void* stream);
QCNN_API int qcnn_pq_stats_refine_target_bias(qcnn_pq_stats* s, int K, int sweeps, float* ctrd_h, uint8_t* asmt_h,
                                              float* bias_h, double* loss_h, void* stream);
/* refine or refine_target (target = 0 / 1) with the weight anchor; bias_h nullable: with it, _bias's refit */
QCNN_API int qcnn_pq_stats_refine_damped(qcnn_pq_stats* s, int target, double damp, int K, int sweeps,
                                         const float* wei_h /* fcntWei or convKnl */, float* ctrd_h, uint8_t* asmt_h,
                                         float* bias_h, double* loss_h, void* stream);
QCNN_API void qcnn_pq_stats_destroy(qcnn_pq_stats* s);

/* ---- file formats (include/FileIO.h:56-178, 229-350), host only ------------------------------------------- */
/* .bin: returns element count or -1; dims4 padded with 1; data_h may be NULL to query the shape */
QCNN_API long qcnn_read_bin_f32(const char* path, int* dim_cnt, int* dims4, float* data_h, long cap);
QCNN_API int qcnn_write_bin_f32(const char* path, int dim_cnt, const int* dims, const float* data_h);
/* .cbn: 0-based indices as held after CaffePara::LoadLayerPara (reader's +1 and the loader's -1 both applied) */
QCNN_API long qcnn_read_cbn_u8(const char* path, int* dim_cnt, int* dims4, int* bits, uint8_t* data_h, long cap);
QCNN_API int qcnn_write_cbn_u8(const char* path, int dim_cnt, const int* dims, const uint8_t* idx0_h, int bits);

#ifdef __cplusplus
}
#endif
#endif /* QCNN_H_ */
