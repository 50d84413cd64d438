// Whole-network executor on the device: the layer loop of CaffeEva::ExecForwardPass (reference
// src/CaffeEva.cc:213-261) + CaffeEva::LoadCaffePara (:109-149) with every feature map resident in HBM.
// Differences from the reference executor, none of which change results beyond fp32 rounding:
//   * runtime batch size (the reference hard-codes kDataCntInBatch = 1, CaffeEva.cc:23);
//   * NCHW->NHWC of the input is folded into the first conv's loads when that conv runs the strided kernel,
//     NHWC->NCHW before the first FC layer is folded into that layer's LUT addressing (never materialised);
//   * ReLU is fused into the producing PQ kernel, LRN+pool into one pass, dropout (identity at test time,
//     CaffeEva.cc:1091-1096) is elided by aliasing -- unless keep_maps asks for the un-fused featMapLst.
#include <string.h>

#include <algorithm>
#include <string>
#include <vector>

#include "../host/CaffePara.h"
#include "qcnn_internal.h"

#include <cstdlib>

using namespace qcnn;

struct NetLayer {
  qcnn_layer_info info;
  qcnn_layer* pq;
  int Hin, Win, Cin;     // NHWC dims of featMapLst[l]
  int Hout, Wout, Cout;  // NHWC dims of featMapLst[l+1]
};

struct qcnn_net {
  qcnn_ctx* ctx = nullptr;
  std::vector<NetLayer> layers;
  int imgC = 0, imgH = 0, imgW = 0;
  int keep = 0;
  int profiling = 0;
  std::vector<DeviceBuffer> maps;  // featMapLst[0..L] (float); maps[0] only used when the input must be permuted
  std::vector<const float*> mapPtr;  // where featMapLst[i] of the last forward actually lives (NULL if fused away)
  std::vector<cudaEvent_t> evBeg, evEnd;
  std::vector<char> evUsed;
  unsigned long long lastLaunches = 0;
  // host-buffer forward: double-buffered input chunks (float) + output staging
  DeviceBuffer d_in[2];
  // uint8 entry points: crop-sized mean image, staging of the uint8 chunks, on-device top-k results
  DeviceBuffer d_mean;      // float [C][H][W] or empty
  DeviceBuffer d_in8[2];    // uint8_t
  DeviceBuffer d_f32;       // converted chunk (device-resident uint8 entry)
  DeviceBuffer d_topi;      // int
  DeviceBuffer d_topv;      // float
  // asynchronous host-buffer steps (qcnn_net_submit_u8_h): two input slots so that the copy of step i+1 overlaps step i
  DeviceBuffer d_sub8[2];   // uint8_t
  cudaEvent_t evSubIn[2] = {}, evSubRead[2] = {}, evSubDone[2] = {};
  int subInit = 0;
  unsigned long long subCount = 0;
  DeviceBuffer d_prob;      // float
  DeviceBuffer d_logit;     // float
  cudaStream_t stCopy = nullptr, stComp = nullptr;
  cudaEvent_t evH2D[2] = {}, evDone[2] = {};
  int chunk = 128;
  // small batches: the launch sequence of a forward pass is captured once per (N, buffers, stream) and replayed
  struct GraphEntry {
    int N; const float* img; float* prob; float* logits; cudaStream_t st;
    unsigned long long epoch; // ctx->alloc_epoch at capture
    int seen;                 // eager passes so far (tilings are autotuned and scratch is allocated during these)
    int disabled;             // capture failed once: stay eager
    cudaGraphExec_t exec;
    unsigned long long launches;
  };
  std::vector<GraphEntry> graphs;
};

static size_t MapElems(const NetLayer& L) { return static_cast<size_t>(L.Hout) * L.Wout * L.Cout; }

// Feature-map buffers are reserved on first use for the batch at hand: the fused production path touches about half of
// featMapLst (ReLU / LRN / dropout outputs are fused away), so the other half is never allocated unless keep_maps asks
// for it.
static float* MapBuf(qcnn_net* net, int idx, int N, cudaStream_t st) {
  const size_t elems = idx == 0 ? static_cast<size_t>(net->imgC) * net->imgH * net->imgW : MapElems(net->layers[idx - 1]);
  const cudaError_t e = net->maps[idx].Reserve(net->ctx, sizeof(float) * N * elems, st);
  if (e == cudaErrorStreamCaptureUnsupported) { SetError("internal: feature map %d is not allocated inside a stream capture", idx); return nullptr; }
  if (e) { CudaFail(e, "feature map reservation", __FILE__, __LINE__); return nullptr; }
  return net->maps[idx].as<float>();
}

namespace qcnn {

std::vector<LayerDims> LayerInputDims(const std::vector<qcnn_layer_info>& infos, int imgC, int imgH, int imgW) {
  std::vector<LayerDims> dims(infos.size() + 1);
  int H = imgH, W = imgW, C = imgC;
  for (size_t l = 0; l < infos.size(); l++) {
    const qcnn_layer_info& li = infos[l];
    dims[l] = {H, W, C};
    switch (li.type) {
      case QCNN_CONV: {
        const int stride = std::max(li.stride, 1);   // qcnn_conv_layer_create refuses a stride < 1
        H = (H + 2 * li.padSiz - li.knlSiz) / stride + 1;  // reference CaffeEva.cc:361-362
        W = (W + 2 * li.padSiz - li.knlSiz) / stride + 1;
        C = li.knlCnt;
        break;
      }
      case QCNN_FCNT:
        H = 1; W = 1; C = li.nodCnt;
        break;
      case QCNN_POOL: {
        const int stride = std::max(li.stride, 1);   // BuildNet refuses a stride < 1
        H = PoolOut(H, li.padSiz, li.knlSiz, stride);
        W = PoolOut(W, li.padSiz, li.knlSiz, stride);
        break;
      }
      default:
        break;
    }
  }
  dims[infos.size()] = {H, W, C};
  return dims;
}

std::vector<qcnn_layer_info> LayerInfos(const CaffePara& para) {
  std::vector<qcnn_layer_info> infos(para.layerCnt);
  for (int l = 0; l < para.layerCnt; l++) {
    const LayerInfo& li = para.layerInfoLst[l];
    qcnn_layer_info& o = infos[l];
    o.type = static_cast<int>(li.type);
    o.padSiz = li.padSiz; o.knlSiz = li.knlSiz; o.knlCnt = li.knlCnt; o.grpCnt = li.grpCnt; o.stride = li.stride;
    o.nodCnt = li.nodCnt; o.lrnSiz = li.lrnSiz; o.lrnAlp = li.lrnAlp; o.lrnBet = li.lrnBet; o.lrnIni = li.lrnIni; o.drpRat = li.drpRat;
  }
  return infos;
}

}  // namespace qcnn

static int BuildNet(qcnn_ctx* ctx, int layerCnt, const qcnn_layer_info* infos, const qcnn_layer_para* paras, int imgC, int imgH,
                    int imgW, qcnn_net** out) {
  qcnn_net* net = new qcnn_net();
  net->ctx = ctx;
  net->imgC = imgC; net->imgH = imgH; net->imgW = imgW;
  const std::vector<LayerDims> dims = LayerInputDims(std::vector<qcnn_layer_info>(infos, infos + layerCnt), imgC, imgH, imgW);
  bool seenFc = false;
  int rc = 0;
  for (int l = 0; l < layerCnt && rc == 0; l++) {
    NetLayer nl;
    memset(&nl, 0, sizeof(nl));
    nl.info = infos[l];
    const qcnn_layer_info& li = nl.info;
    const int H = dims[l].H, W = dims[l].W, C = dims[l].C;
    nl.Hin = H; nl.Win = W; nl.Cin = C;
    const qcnn_layer_para& lp = paras[l];
    switch (li.type) {
      case QCNN_CONV: {
        if (!lp.ctrd || !lp.asmt || !lp.bias) {
          SetError("layer %d: conv layer without product-quantized parameters", l + 1);
          rc = 1;
          break;
        }
        rc = qcnn_conv_layer_create(ctx, C, H, W, li.knlCnt, li.knlSiz, li.padSiz, li.stride, li.grpCnt, lp.S, lp.K, lp.d,
                                    lp.ctrd, lp.asmt, lp.bias, &nl.pq);
        break;
      }
      case QCNN_FCNT: {
        if (!lp.ctrd || !lp.asmt || !lp.bias) {
          SetError("layer %d: FC layer without product-quantized parameters", l + 1);
          rc = 1;
          break;
        }
        const int Din = H * W * C;
        rc = qcnn_fc_layer_create(ctx, Din, li.nodCnt, lp.S, lp.K, lp.d, lp.ctrd, lp.asmt, lp.bias, &nl.pq);
        if (rc) break;
        nl.pq->opt_fc_ws = 1;   // the weight-stationary GEMM for batched FC layers (standalone layers keep mode 2: DESIGN.md 4a)
        // first FC layer: the reference permutes its NHWC input to NCHW first (CaffeEva.cc:236-238)
        if (!seenFc && (H > 1 || W > 1)) rc = qcnn_fc_layer_set_src_nhwc(nl.pq, H, W, C);
        seenFc = true;
        break;
      }
      case QCNN_POOL:
        if (li.knlSiz < 1 || li.stride < 1 || !PoolWindowsNonEmpty(H, li.padSiz, li.knlSiz, li.stride) ||
            !PoolWindowsNonEmpty(W, li.padSiz, li.knlSiz, li.stride)) {
          SetError("layer %d: pooling a %dx%d map with a %dx%d window, pad %d, stride %d leaves an output window without "
                   "input pixels", l + 1, H, W, li.knlSiz, li.knlSiz, li.padSiz, li.stride);
          rc = 1;
        }
        break;
      default:
        break;
    }
    nl.Hout = dims[l + 1].H; nl.Wout = dims[l + 1].W; nl.Cout = dims[l + 1].C;
    net->layers.push_back(nl);
  }
  if (rc) {
    qcnn_net_destroy(net);
    return rc;
  }
  // the first conv reads the NCHW API input directly when it runs the strided kernel
  if (!net->layers.empty() && net->layers[0].pq && net->layers[0].info.type == QCNN_CONV &&
      net->layers[0].info.stride > 1)
    qcnn_conv_layer_set_src_nchw(net->layers[0].pq, 1);
  const size_t L = net->layers.size();
  net->maps.resize(L + 1);
  net->mapPtr.assign(L + 1, nullptr);
  net->evBeg.resize(L); net->evEnd.resize(L); net->evUsed.assign(L, 0);
  for (size_t l = 0; l < L; l++) {
    cudaEventCreate(&net->evBeg[l]);
    cudaEventCreate(&net->evEnd[l]);
  }
  *out = net;
  return 0;
}

// parameters loaded from files: shape checks against the layer table, then the common builder
static int BuildFromCaffePara(qcnn_ctx* ctx, CaffePara& para, qcnn_net** out) {
  const std::vector<qcnn_layer_info> infos = LayerInfos(para);
  std::vector<qcnn_layer_para> paras(para.layerCnt);
  for (int l = 0; l < para.layerCnt; l++) {
    const LayerInfo& li = para.layerInfoLst[l];
    memset(&paras[l], 0, sizeof(qcnn_layer_para));
    if (li.type != ENUM_LyrType::Conv && li.type != ENUM_LyrType::FCnt) continue;
    const LayerPara& lp = para.layerParaLst[l];
    const bool conv = li.type == ENUM_LyrType::Conv;
    QCNN_CHECK(lp.ctrdLst.GetDimCnt() == 3 && lp.asmtLst.GetDimCnt() == (conv ? 4 : 2),
               "layer %d: %s parameters have unexpected rank", l + 1, conv ? "conv" : "FC");
    const int S = lp.ctrdLst.GetDimLen(0);
    if (conv)
      QCNN_CHECK(lp.asmtLst.GetDimLen(0) == li.knlCnt && lp.asmtLst.GetDimLen(1) == li.knlSiz && lp.asmtLst.GetDimLen(2) == li.knlSiz &&
                 lp.asmtLst.GetDimLen(3) == S && lp.biasVec.GetEleCnt() == li.knlCnt,
                 "layer %d: conv parameter shapes do not match the layer table", l + 1);
    else
      QCNN_CHECK(lp.asmtLst.GetDimLen(0) == li.nodCnt && lp.asmtLst.GetDimLen(1) == S && lp.biasVec.GetEleCnt() == li.nodCnt,
                 "layer %d: FC parameter shapes do not match the layer table", l + 1);
    paras[l].ctrd = lp.ctrdLst.GetDataPtr(); paras[l].asmt = lp.asmtLst.GetDataPtr(); paras[l].bias = lp.biasVec.GetDataPtr();
    paras[l].S = S; paras[l].K = lp.ctrdLst.GetDimLen(1); paras[l].d = lp.ctrdLst.GetDimLen(2);
  }
  return BuildNet(ctx, para.layerCnt, infos.data(), paras.data(), para.imgChnIn, para.imgHeiIn, para.imgWidIn, out);
}

extern "C" {

int qcnn_net_create_from_para(qcnn_ctx* ctx, int layer_cnt, const qcnn_layer_info* layers, const qcnn_layer_para* para,
                              int img_chn, int img_hei, int img_wid, qcnn_net** out) {
  QCNN_CHECK(ctx && layers && para && out && layer_cnt >= 1, "qcnn_net_create_from_para: bad argument");
  *out = nullptr;
  for (int l = 0; l < layer_cnt; l++)
    QCNN_CHECK(layers[l].type >= 0 && layers[l].type <= QCNN_SMAX, "qcnn_net_create_from_para: layer %d has invalid type", l);
  QCNN_ON_DEVICE(ctx->device);
  return BuildNet(ctx, layer_cnt, layers, para, img_chn, img_hei, img_wid, out);
}

int qcnn_net_create(qcnn_ctx* ctx, const char* model_name, const char* dir, const char* pfx, qcnn_net** out) {
  QCNN_CHECK(ctx && model_name && dir && pfx && out, "qcnn_net_create: NULL argument");
  *out = nullptr;
  CaffePara para;
  para.Init(dir, pfx);
  QCNN_CHECK(para.ConfigLayer_ByName(model_name), "qcnn_net_create: unrecognized caffe model name: %s", model_name);
  QCNN_CHECK(para.LoadLayerPara(true, ENUM_AsmtEnc::Compact), "qcnn_net_create: could not load parameters from %s/%s.*",
             dir, pfx);
  return BuildFromCaffePara(ctx, para, out);
}

int qcnn_net_create_custom(qcnn_ctx* ctx, int layer_cnt, const qcnn_layer_info* layers, int img_chn, int img_hei,
                           int img_wid, const char* dir, const char* pfx, qcnn_net** out) {
  QCNN_CHECK(ctx && layers && dir && pfx && out && layer_cnt >= 1, "qcnn_net_create_custom: bad argument");
  *out = nullptr;
  CaffePara para;
  para.Init(dir, pfx);
  para.layerCnt = layer_cnt;
  para.imgChnIn = img_chn; para.imgHeiIn = img_hei; para.imgWidIn = img_wid;
  para.layerInfoLst.resize(layer_cnt);
  for (int l = 0; l < layer_cnt; l++) {
    LayerInfo& li = para.layerInfoLst[l];
    QCNN_CHECK(layers[l].type >= 0 && layers[l].type <= QCNN_SMAX, "qcnn_net_create_custom: layer %d has invalid type", l);
    li.type = static_cast<ENUM_LyrType>(layers[l].type);
    li.padSiz = layers[l].padSiz; li.knlSiz = layers[l].knlSiz; li.knlCnt = layers[l].knlCnt;
    li.grpCnt = layers[l].grpCnt; li.stride = layers[l].stride; li.nodCnt = layers[l].nodCnt;
    li.lrnSiz = layers[l].lrnSiz; li.lrnAlp = layers[l].lrnAlp; li.lrnBet = layers[l].lrnBet;
    li.lrnIni = layers[l].lrnIni; li.drpRat = layers[l].drpRat;
  }
  QCNN_CHECK(para.LoadLayerPara(true, ENUM_AsmtEnc::Compact),
             "qcnn_net_create_custom: could not load parameters from %s/%s.*", dir, pfx);
  return BuildFromCaffePara(ctx, para, out);
}

void qcnn_net_destroy(qcnn_net* net) {
  if (!net) return;
  DeviceGuard guard(net->ctx->device);
  for (NetLayer& L : net->layers) qcnn_layer_destroy(L.pq);
  for (size_t l = 0; l < net->evBeg.size(); l++) {
    cudaEventDestroy(net->evBeg[l]);
    cudaEventDestroy(net->evEnd[l]);
  }
  for (int i = 0; i < 2; i++) {
    if (net->subInit) { cudaEventDestroy(net->evSubIn[i]); cudaEventDestroy(net->evSubRead[i]); cudaEventDestroy(net->evSubDone[i]); }
    if (net->stCopy) { cudaEventDestroy(net->evH2D[i]); cudaEventDestroy(net->evDone[i]); }
  }
  for (qcnn_net::GraphEntry& g : net->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
  if (net->stCopy) cudaStreamDestroy(net->stCopy);
  if (net->stComp) cudaStreamDestroy(net->stComp);
  delete net;
}

int qcnn_net_layer_count(const qcnn_net* net) { return net ? static_cast<int>(net->layers.size()) : 0; }

int qcnn_net_out_len(const qcnn_net* net) {
  if (!net || net->layers.empty()) return 0;
  const NetLayer& L = net->layers.back();
  return L.Hout * L.Wout * L.Cout;
}

int qcnn_net_set_keep_maps(qcnn_net* net, int keep) {
  QCNN_CHECK(net, "qcnn_net_set_keep_maps: NULL net");
  net->keep = keep ? 1 : 0;
  return 0;
}

int qcnn_net_set_profiling(qcnn_net* net, int enable) {
  QCNN_CHECK(net, "qcnn_net_set_profiling: NULL net");
  net->profiling = enable ? 1 : 0;
  return 0;
}

qcnn_layer* qcnn_net_pq_layer(qcnn_net* net, int l) {
  if (!net || l < 0 || l >= static_cast<int>(net->layers.size())) return nullptr;
  return net->layers[l].pq;
}

int qcnn_net_launch_count(const qcnn_net* net) { return net ? static_cast<int>(net->lastLaunches) : 0; }

static int ForwardEager(qcnn_net* net, const float* img, int N, float* prob, float* logits, cudaStream_t st);

// Batches of <= kGraphMaxN images are launch-bound (20 kernels of 10-30 us): after two eager passes (autotuning, scratch
// allocation) the sequence is captured into a CUDA graph keyed by (N, buffers, stream) and replayed.  Not used on the
// legacy default stream (it cannot be captured), while profiling / keeping maps, or with QCNN_GRAPH=0.
constexpr int kGraphMaxN = 8;

int qcnn_net_forward(qcnn_net* net, const float* img, int N, float* prob, float* logits, void* stream) {
  QCNN_CHECK(net && img && prob, "qcnn_net_forward: NULL argument");
  QCNN_CHECK(N >= 1, "qcnn_net_forward: N must be >= 1");
  QCNN_ON_DEVICE(net->ctx->device);   // one process may drive several GPUs (qcnn_multi_*)
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  static const bool graphsOn = !(getenv("QCNN_GRAPH") && getenv("QCNN_GRAPH")[0] == '0');
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  if (st) cudaStreamIsCapturing(st, &cap);
  if (!graphsOn || N > kGraphMaxN || st == nullptr || net->keep || net->profiling || cap != cudaStreamCaptureStatusNone)
    return ForwardEager(net, img, N, prob, logits, st);
  qcnn_net::GraphEntry* ge = nullptr;
  for (qcnn_net::GraphEntry& g : net->graphs)
    if (g.N == N && g.img == img && g.prob == prob && g.logits == logits && g.st == st) ge = &g;
  if (!ge) {
    if (net->graphs.size() >= 8) {   // bounded cache: drop the oldest entry
      if (net->graphs.front().exec) cudaGraphExecDestroy(net->graphs.front().exec);
      net->graphs.erase(net->graphs.begin());
    }
    net->graphs.push_back({N, img, prob, logits, st, 0, 0, 0, nullptr, 0});
    ge = &net->graphs.back();
  }
  if (ge->exec && ge->epoch != net->ctx->alloc_epoch) {   // a scratch buffer moved since the capture
    cudaGraphExecDestroy(ge->exec);
    ge->exec = nullptr;
    ge->seen = 1;
  }
  if (ge->exec) {
    QCNN_CUDA(cudaGraphLaunch(ge->exec, st));
    net->ctx->launches += ge->launches;
    net->lastLaunches = ge->launches;
    return 0;
  }
  if (ge->disabled || ge->seen < 2) {
    ge->seen++;
    return ForwardEager(net, img, N, prob, logits, st);
  }
  // third pass with the same arguments: capture, instantiate, replay
  if (cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) != cudaSuccess) {
    cudaGetLastError();
    ge->disabled = 1;
    return ForwardEager(net, img, N, prob, logits, st);
  }
  const int rc = ForwardEager(net, img, N, prob, logits, st);
  cudaGraph_t graph = nullptr;
  const cudaError_t ce = cudaStreamEndCapture(st, &graph);
  if (rc != 0 || ce != cudaSuccess || graph == nullptr) {
    cudaGetLastError();
    if (graph) cudaGraphDestroy(graph);
    ge->disabled = 1;
    return rc ? rc : ForwardEager(net, img, N, prob, logits, st);
  }
  ge->launches = net->lastLaunches;
  ge->epoch = net->ctx->alloc_epoch;
  const cudaError_t ie = cudaGraphInstantiate(&ge->exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ie != cudaSuccess) {
    cudaGetLastError();
    ge->exec = nullptr;
    ge->disabled = 1;
    return ForwardEager(net, img, N, prob, logits, st);
  }
  QCNN_CUDA(cudaGraphLaunch(ge->exec, st));
  return 0;
}

static int ForwardEager(qcnn_net* net, const float* img, int N, float* prob, float* logits, cudaStream_t st) {
  qcnn_ctx* ctx = net->ctx;
  const int L = static_cast<int>(net->layers.size());
  const unsigned long long launches0 = ctx->launches;
  std::fill(net->mapPtr.begin(), net->mapPtr.end(), nullptr);
  std::fill(net->evUsed.begin(), net->evUsed.end(), 0);

  // featMapLst[0]: NHWC copy of the input unless the first conv consumes NCHW directly
  const float* cur = nullptr;
  const bool firstReadsNchw = L > 0 && net->layers[0].pq && net->layers[0].pq->kind == QCNN_KIND_CONV &&
                              net->layers[0].pq->src_nchw;
  if (firstReadsNchw && !net->keep) {
    cur = img;
  } else {
    if (firstReadsNchw) {
      cur = img;  // conv still reads the NCHW input; also materialise the NHWC map for inspection
      float* m0 = MapBuf(net, 0, N, st);
      if (!m0) return 2;
      if (int rc = LaunchNchwToNhwc(ctx, img, m0, N, net->imgC, net->imgH, net->imgW, st)) return rc;
    } else {
      float* m0 = MapBuf(net, 0, N, st);
      if (!m0) return 2;
      if (int rc = LaunchNchwToNhwc(ctx, img, m0, N, net->imgC, net->imgH, net->imgW, st)) return rc;
      cur = m0;
    }
    net->mapPtr[0] = net->maps[0].as<float>();
  }

  int l = 0;
  while (l < L) {
    NetLayer& nl = net->layers[l];
    const int type = nl.info.type;
    const int first = l;
    if (net->profiling) { QCNN_CUDA(cudaEventRecord(net->evBeg[first], st)); }
    int rc = 0;
    const bool lastLayer = (l == L - 1);
    switch (type) {
      case QCNN_CONV:
      case QCNN_FCNT: {
        if (type == QCNN_FCNT && !net->keep) {
          // batch <= 4: the whole run FC [ReLU] [Drpt] FC ... as ONE persistent launch (fc_chain.cu)
          qcnn_layer* chain[4];
          int crelu[4];
          int n = 0, j = l, outIdx = l;
          while (j < L && net->layers[j].info.type == QCNN_FCNT && n < 4) {
            chain[n] = net->layers[j].pq;
            crelu[n] = 0;
            j++;
            if (j < L && net->layers[j].info.type == QCNN_RELU) { crelu[n] = 1; j++; }
            n++;
            outIdx = j;
            int k = j;
            while (k < L && net->layers[k].info.type == QCNN_DRPT) k++;   // identity at test time (CaffeEva.cc:1091-1096)
            if (k < L && net->layers[k].info.type == QCNN_FCNT) j = k; else break;
          }
          if (n >= 1 && FcChainEligible(ctx, chain, crelu, n, N)) {
            bool handled = false;
            float* dst = MapBuf(net, outIdx, N, st);
        if (!dst) return 2;
            rc = LaunchFcChain(ctx, chain, crelu, n, cur, N, dst, st, nullptr, &handled);
            if (rc) break;
            if (handled) {
              net->mapPtr[outIdx] = dst;
              cur = dst;
              l = outIdx;
              break;
            }
          }
        }
        const bool fuse = !net->keep && l + 1 < L && net->layers[l + 1].info.type == QCNN_RELU;
        const int outIdx = fuse ? l + 2 : l + 1;
        float* dst = MapBuf(net, outIdx, N, st);
        if (!dst) return 2;
        if (type == QCNN_CONV) rc = LaunchConv(nl.pq, cur, N, dst, fuse ? 1 : 0, st);
        else rc = LaunchFc(nl.pq, cur, N, dst, fuse ? 1 : 0, st);
        net->mapPtr[outIdx] = dst;
        cur = dst;
        l = outIdx;
        break;
      }
      case QCNN_RELU: {
        float* dst = MapBuf(net, l + 1, N, st);
        if (!dst) return 2;
        rc = LaunchRelu(ctx, cur, dst, static_cast<size_t>(N) * MapElems(nl), st);
        net->mapPtr[l + 1] = dst; cur = dst; l++;
        break;
      }
      case QCNN_LORN: {
        const bool fuse = !net->keep && l + 1 < L && net->layers[l + 1].info.type == QCNN_POOL;
        if (fuse) {
          const NetLayer& pl = net->layers[l + 1];
          float* dst = MapBuf(net, l + 2, N, st);
        if (!dst) return 2;
          rc = LaunchLrnMaxPool(ctx, cur, dst, N, nl.Hin, nl.Win, nl.Cin, nl.info.lrnSiz, nl.info.lrnAlp,
                                nl.info.lrnBet, nl.info.lrnIni, pl.info.knlSiz, pl.info.padSiz, pl.info.stride, st);
          net->mapPtr[l + 2] = dst; cur = dst; l += 2;
        } else {
          float* dst = MapBuf(net, l + 1, N, st);
        if (!dst) return 2;
          rc = LaunchLrn(ctx, cur, dst, static_cast<size_t>(N) * nl.Hin * nl.Win, nl.Cin, nl.info.lrnSiz,
                         nl.info.lrnAlp, nl.info.lrnBet, nl.info.lrnIni, st);
          net->mapPtr[l + 1] = dst; cur = dst; l++;
        }
        break;
      }
      case QCNN_POOL: {
        float* dst = MapBuf(net, l + 1, N, st);
        if (!dst) return 2;
        rc = LaunchMaxPool(ctx, cur, dst, N, nl.Hin, nl.Win, nl.Cin, nl.info.knlSiz, nl.info.padSiz, nl.info.stride, st);
        net->mapPtr[l + 1] = dst; cur = dst; l++;
        break;
      }
      case QCNN_DRPT: {
        if (net->keep) {
          float* dst = MapBuf(net, l + 1, N, st);
        if (!dst) return 2;
          QCNN_CUDA(cudaMemcpyAsync(dst, cur, sizeof(float) * N * MapElems(nl), cudaMemcpyDeviceToDevice, st));
          net->mapPtr[l + 1] = dst; cur = dst;
        } else {
          net->mapPtr[l + 1] = cur;  // identity: alias
        }
        l++;
        break;
      }
      case QCNN_SMAX: {
        if (logits && lastLayer)
          QCNN_CUDA(cudaMemcpyAsync(logits, cur, sizeof(float) * N * MapElems(nl), cudaMemcpyDeviceToDevice, st));
        float* dst = lastLayer ? prob : MapBuf(net, l + 1, N, st);
        if (!dst) return 2;
        rc = LaunchSoftmax(ctx, cur, dst, N, nl.Hout * nl.Wout * nl.Cout, st);
        net->mapPtr[l + 1] = dst; cur = dst; l++;
        break;
      }
      default:
        SetError("qcnn_net_forward: invalid layer type %d", type);
        return 1;
    }
    if (rc) return rc;
    if (net->profiling) {
      QCNN_CUDA(cudaEventRecord(net->evEnd[first], st));
      net->evUsed[first] = 1;
    }
  }
  // networks that do not end in softmax: copy the last map out
  if (L == 0 || net->layers[L - 1].info.type != QCNN_SMAX) {
    QCNN_CUDA(cudaMemcpyAsync(prob, cur, sizeof(float) * N * qcnn_net_out_len(net), cudaMemcpyDeviceToDevice, st));
    if (logits) QCNN_CUDA(cudaMemcpyAsync(logits, cur, sizeof(float) * N * qcnn_net_out_len(net), cudaMemcpyDeviceToDevice, st));
  }
  net->lastLaunches = ctx->launches - launches0;
  return 0;
}

// The copy and compute streams of the host-buffer pipelines and their events, created on first use
static int CreatePipeline(qcnn_net* net) {
  if (net->stCopy) return 0;
  QCNN_CUDA(cudaStreamCreateWithFlags(&net->stCopy, cudaStreamNonBlocking));
  QCNN_CUDA(cudaStreamCreateWithFlags(&net->stComp, cudaStreamNonBlocking));
  for (int i = 0; i < 2; i++) {
    QCNN_CUDA(cudaEventCreateWithFlags(&net->evH2D[i], cudaEventDisableTiming));
    QCNN_CUDA(cudaEventCreateWithFlags(&net->evDone[i], cudaEventDisableTiming));
  }
  return 0;
}

// Device-side results of a host-buffer call for N images: probabilities, logits and (topk > 0) the top-k pairs
static int ReserveOutputs(qcnn_net* net, int N, int topk) {
  const size_t out = sizeof(float) * static_cast<size_t>(N) * qcnn_net_out_len(net), top = static_cast<size_t>(N) * topk;
  QCNN_CUDA(net->d_prob.Reserve(net->ctx, out));
  QCNN_CUDA(net->d_logit.Reserve(net->ctx, out));
  QCNN_CUDA(net->d_topi.Reserve(net->ctx, sizeof(int) * top));
  QCNN_CUDA(net->d_topv.Reserve(net->ctx, sizeof(float) * top));
  return 0;
}

// Host-buffer forward pass: a pipeline of chunks on two streams -- H2D of chunk c+1 (copy stream) overlaps the layers of
// chunk c (compute stream).  Images arrive as fp32 NCHW (ExecForwardPass's own input) or as uint8 HWC pixels that are
// converted (and mean-subtracted) on the device: 4x fewer bytes over the host link.  With topk > 0 the k-fold arg-max runs
// on the device and only [N][k] (index, probability) pairs come back; prob_h / logits_h are optional then.
static int ForwardHost(qcnn_net* net, const float* img_h, const uint8_t* img8_h, int N, float* prob_h, float* logits_h, int topk,
                       int topk_mode, int* topi_h, float* topv_h) {
  QCNN_ON_DEVICE(net->ctx->device);
  if (int rc = CreatePipeline(net)) return rc;
  const size_t imgLen = static_cast<size_t>(net->imgC) * net->imgH * net->imgW;
  const int outLen = qcnn_net_out_len(net);
  const int chunk = std::min(N, net->chunk);
  for (DeviceBuffer& b : net->d_in) QCNN_CUDA(b.Reserve(net->ctx, sizeof(float) * chunk * imgLen));
  if (img8_h)
    for (DeviceBuffer& b : net->d_in8) QCNN_CUDA(b.Reserve(net->ctx, chunk * imgLen));
  if (int rc = ReserveOutputs(net, N, topk)) return rc;
  unsigned long long launches = 0;
  int ci = 0;
  // the first chunk is a quarter of the others: its host-to-device copy is the only one nothing overlaps
  const int first = (N > chunk) ? std::max(1, chunk / 4) : chunk;
  for (int n0 = 0; n0 < N; ci++) {
    const int cn = std::min(ci == 0 ? first : chunk, N - n0);
    const int b = ci & 1;
    if (ci >= 2) QCNN_CUDA(cudaStreamWaitEvent(net->stCopy, net->evDone[b], 0));
    if (img8_h)
      QCNN_CUDA(cudaMemcpyAsync(net->d_in8[b].get(), img8_h + n0 * imgLen, cn * imgLen, cudaMemcpyHostToDevice, net->stCopy));
    else
      QCNN_CUDA(cudaMemcpyAsync(net->d_in[b].get(), img_h + n0 * imgLen, sizeof(float) * cn * imgLen, cudaMemcpyHostToDevice, net->stCopy));
    QCNN_CUDA(cudaEventRecord(net->evH2D[b], net->stCopy));
    QCNN_CUDA(cudaStreamWaitEvent(net->stComp, net->evH2D[b], 0));
    if (img8_h) {
      if (int rc = LaunchU8ToF32(net->ctx, net->d_in8[b].as<uint8_t>(), net->d_mean.as<float>(), net->d_in[b].as<float>(), cn,
                                 net->imgC, net->imgH * net->imgW, net->stComp))
        return rc;
      launches++;
    }
    if (int rc = qcnn_net_forward(net, net->d_in[b].as<float>(), cn, net->d_prob.as<float>() + static_cast<size_t>(n0) * outLen,
                                  logits_h ? net->d_logit.as<float>() + static_cast<size_t>(n0) * outLen : nullptr, net->stComp))
      return rc;
    launches += net->lastLaunches;
    QCNN_CUDA(cudaEventRecord(net->evDone[b], net->stComp));
    n0 += cn;
  }
  if (topk > 0) {
    if (int rc = LaunchTopK(net->ctx, net->d_prob.as<float>(), N, outLen, topk, topk_mode, net->d_topi.as<int>(), net->d_topv.as<float>(),
                            net->stComp))
      return rc;
    launches++;
    QCNN_CUDA(cudaMemcpyAsync(topi_h, net->d_topi.get(), sizeof(int) * N * topk, cudaMemcpyDeviceToHost, net->stComp));
    QCNN_CUDA(cudaMemcpyAsync(topv_h, net->d_topv.get(), sizeof(float) * N * topk, cudaMemcpyDeviceToHost, net->stComp));
  }
  if (prob_h) QCNN_CUDA(cudaMemcpyAsync(prob_h, net->d_prob.get(), sizeof(float) * N * outLen, cudaMemcpyDeviceToHost, net->stComp));
  if (logits_h)
    QCNN_CUDA(cudaMemcpyAsync(logits_h, net->d_logit.get(), sizeof(float) * N * outLen, cudaMemcpyDeviceToHost, net->stComp));
  QCNN_CUDA(cudaStreamSynchronize(net->stComp));
  net->lastLaunches = launches;
  return 0;
}

int qcnn_net_forward_h(qcnn_net* net, const float* img_h, int N, float* prob_h, float* logits_h) {
  QCNN_CHECK(net && img_h && prob_h, "qcnn_net_forward_h: NULL argument");
  QCNN_CHECK(N >= 1, "qcnn_net_forward_h: N must be >= 1");
  return ForwardHost(net, img_h, nullptr, N, prob_h, logits_h, 0, 0, nullptr, nullptr);
}

int qcnn_net_forward_topk_h(qcnn_net* net, const float* img_h, int N, int topk, int topk_mode, int* topk_idx_h, float* topk_prob_h,
                            float* prob_h) {
  QCNN_CHECK(net && img_h && topk_idx_h && topk_prob_h, "qcnn_net_forward_topk_h: NULL argument");
  QCNN_CHECK(N >= 1 && topk >= 1 && topk <= qcnn_net_out_len(net), "qcnn_net_forward_topk_h: bad N / topk");
  return ForwardHost(net, img_h, nullptr, N, prob_h, nullptr, topk, topk_mode, topk_idx_h, topk_prob_h);
}

int qcnn_net_set_input_mean(qcnn_net* net, const float* mean_h) {
  QCNN_CHECK(net, "qcnn_net_set_input_mean: NULL net");
  QCNN_ON_DEVICE(net->ctx->device);
  if (!mean_h) {
    QCNN_CUDA(net->d_mean.Release());
    return 0;
  }
  QCNN_CUDA(net->d_mean.Upload(net->ctx, mean_h, sizeof(float) * net->imgC * net->imgH * net->imgW));
  return 0;
}

int qcnn_net_forward_u8(qcnn_net* net, const uint8_t* img, int N, float* prob, float* logits, void* stream) {
  QCNN_CHECK(net && img && prob && N >= 1, "qcnn_net_forward_u8: bad argument");
  QCNN_ON_DEVICE(net->ctx->device);
  const size_t imgLen = static_cast<size_t>(net->imgC) * net->imgH * net->imgW;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  QCNN_CUDA(net->d_f32.Reserve(net->ctx, sizeof(float) * N * imgLen, st));
  if (int rc = LaunchU8ToF32(net->ctx, img, net->d_mean.as<float>(), net->d_f32.as<float>(), N, net->imgC, net->imgH * net->imgW, st))
    return rc;
  return qcnn_net_forward(net, net->d_f32.as<float>(), N, prob, logits, st);
}

int qcnn_net_forward_u8_h(qcnn_net* net, const uint8_t* img_h, int N, int topk, int topk_mode, int* topk_idx_h, float* topk_prob_h,
                          float* prob_h) {
  QCNN_CHECK(net && img_h && N >= 1, "qcnn_net_forward_u8_h: bad argument");
  QCNN_CHECK(topk >= 0 && topk <= qcnn_net_out_len(net), "qcnn_net_forward_u8_h: bad topk");
  QCNN_CHECK(topk == 0 || (topk_idx_h && topk_prob_h), "qcnn_net_forward_u8_h: topk > 0 needs the index and probability buffers");
  QCNN_CHECK(topk > 0 || prob_h, "qcnn_net_forward_u8_h: nothing to return (topk == 0 and prob_h == NULL)");
  return ForwardHost(net, nullptr, img_h, N, prob_h, nullptr, topk, topk_mode, topk_idx_h, topk_prob_h);
}

// Asynchronous host-buffer step: queues H2D (copy stream) -> uint8 conversion, forward pass, top-k (compute stream) ->
// D2H of the results, and returns a ticket.  Two tickets may be outstanding: the pixels of step i+1 travel while step i
// computes, so a caller that keeps two steps in flight is bound by max(copy, compute) instead of their sum.
int qcnn_net_submit_u8_h(qcnn_net* net, const uint8_t* img_h, int N, int topk, int topk_mode, int* topk_idx_h, float* topk_prob_h,
                         float* prob_h, int* ticket) {
  QCNN_CHECK(net && img_h && ticket && N >= 1, "qcnn_net_submit_u8_h: bad argument");
  QCNN_CHECK(topk >= 0 && topk <= qcnn_net_out_len(net), "qcnn_net_submit_u8_h: bad topk");
  QCNN_CHECK(topk == 0 || (topk_idx_h && topk_prob_h), "qcnn_net_submit_u8_h: topk > 0 needs the index and probability buffers");
  QCNN_CHECK(topk > 0 || prob_h, "qcnn_net_submit_u8_h: nothing to return (topk == 0 and prob_h == NULL)");
  QCNN_ON_DEVICE(net->ctx->device);
  if (int rc = CreatePipeline(net)) return rc;
  if (!net->subInit) {
    for (int i = 0; i < 2; i++) {
      QCNN_CUDA(cudaEventCreateWithFlags(&net->evSubIn[i], cudaEventDisableTiming));
      QCNN_CUDA(cudaEventCreateWithFlags(&net->evSubRead[i], cudaEventDisableTiming));
      QCNN_CUDA(cudaEventCreateWithFlags(&net->evSubDone[i], cudaEventDisableTiming));
    }
    net->subInit = 1;
  }
  const size_t imgLen = static_cast<size_t>(net->imgC) * net->imgH * net->imgW;
  const int outLen = qcnn_net_out_len(net);
  const int s = static_cast<int>(net->subCount & 1);
  if (net->subCount >= 2) QCNN_CUDA(cudaEventSynchronize(net->evSubDone[s]));   // the ticket two steps back must be over
  // (re)allocations only while nothing is in flight that uses the buffers
  const size_t in8 = static_cast<size_t>(N) * imgLen;
  if (net->d_sub8[0].bytes() < in8 || net->d_f32.bytes() < sizeof(float) * in8 ||
      net->d_prob.bytes() < sizeof(float) * N * outLen || net->d_topi.bytes() < sizeof(int) * N * topk) {
    QCNN_CUDA(cudaStreamSynchronize(net->stCopy));
    QCNN_CUDA(cudaStreamSynchronize(net->stComp));
  }
  for (DeviceBuffer& b : net->d_sub8) QCNN_CUDA(b.Reserve(net->ctx, in8));
  QCNN_CUDA(net->d_f32.Reserve(net->ctx, sizeof(float) * in8));
  if (int rc = ReserveOutputs(net, N, topk)) return rc;
  // copy stream: the slot's pixels were last read by the conversion two steps back
  if (net->subCount >= 2) QCNN_CUDA(cudaStreamWaitEvent(net->stCopy, net->evSubRead[s], 0));
  QCNN_CUDA(cudaMemcpyAsync(net->d_sub8[s].get(), img_h, in8, cudaMemcpyHostToDevice, net->stCopy));
  QCNN_CUDA(cudaEventRecord(net->evSubIn[s], net->stCopy));
  // compute stream: conversion, layers, top-k, results home
  QCNN_CUDA(cudaStreamWaitEvent(net->stComp, net->evSubIn[s], 0));
  if (int rc = LaunchU8ToF32(net->ctx, net->d_sub8[s].as<uint8_t>(), net->d_mean.as<float>(), net->d_f32.as<float>(), N, net->imgC,
                             net->imgH * net->imgW, net->stComp))
    return rc;
  QCNN_CUDA(cudaEventRecord(net->evSubRead[s], net->stComp));
  if (int rc = qcnn_net_forward(net, net->d_f32.as<float>(), N, net->d_prob.as<float>(), nullptr, net->stComp)) return rc;
  if (topk > 0) {
    if (int rc = LaunchTopK(net->ctx, net->d_prob.as<float>(), N, outLen, topk, topk_mode, net->d_topi.as<int>(), net->d_topv.as<float>(),
                            net->stComp))
      return rc;
    QCNN_CUDA(cudaMemcpyAsync(topk_idx_h, net->d_topi.get(), sizeof(int) * N * topk, cudaMemcpyDeviceToHost, net->stComp));
    QCNN_CUDA(cudaMemcpyAsync(topk_prob_h, net->d_topv.get(), sizeof(float) * N * topk, cudaMemcpyDeviceToHost, net->stComp));
  }
  if (prob_h) QCNN_CUDA(cudaMemcpyAsync(prob_h, net->d_prob.get(), sizeof(float) * N * outLen, cudaMemcpyDeviceToHost, net->stComp));
  QCNN_CUDA(cudaEventRecord(net->evSubDone[s], net->stComp));
  *ticket = s;
  net->subCount++;
  return 0;
}

int qcnn_net_wait(qcnn_net* net, int ticket) {
  QCNN_CHECK(net && (ticket == 0 || ticket == 1) && net->subInit, "qcnn_net_wait: bad ticket");
  QCNN_ON_DEVICE(net->ctx->device);
  QCNN_CUDA(cudaEventSynchronize(net->evSubDone[ticket]));
  return 0;
}

int qcnn_net_set_chunk(qcnn_net* net, int chunk) {
  QCNN_CHECK(net && chunk >= 1, "qcnn_net_set_chunk: bad argument");
  net->chunk = chunk;
  return 0;
}

int qcnn_net_set_asmt_packed(qcnn_net* net, int enable) {
  QCNN_CHECK(net, "qcnn_net_set_asmt_packed: NULL net");
  for (const NetLayer& nl : net->layers)
    if (nl.pq && nl.pq->kind == QCNN_KIND_FC)
      if (int rc = qcnn_layer_set_param(nl.pq, "asmt_packed", enable ? 1 : 0)) return rc;
  return 0;
}

int qcnn_net_featmap(qcnn_net* net, int idx, const float** ptr, int* dims4) {
  QCNN_CHECK(net && ptr && dims4, "qcnn_net_featmap: NULL argument");
  const int L = static_cast<int>(net->layers.size());
  QCNN_CHECK(idx >= 0 && idx <= L, "qcnn_net_featmap: index %d out of range", idx);
  *ptr = net->mapPtr[idx];
  if (idx == 0) { dims4[1] = net->imgH; dims4[2] = net->imgW; dims4[3] = net->imgC; }
  else { const NetLayer& nl = net->layers[idx - 1]; dims4[1] = nl.Hout; dims4[2] = nl.Wout; dims4[3] = nl.Cout; }
  dims4[0] = 0;
  return 0;
}

int qcnn_net_layer_time_ms(qcnn_net* net, int layer, float* ms) {
  QCNN_CHECK(net && ms, "qcnn_net_layer_time_ms: NULL argument");
  QCNN_CHECK(layer >= 0 && layer < static_cast<int>(net->layers.size()), "qcnn_net_layer_time_ms: bad layer index");
  *ms = 0.0f;
  if (!net->evUsed[layer]) return 0;
  QCNN_ON_DEVICE(net->ctx->device);
  QCNN_CUDA(cudaEventSynchronize(net->evEnd[layer]));
  QCNN_CUDA(cudaEventElapsedTime(ms, net->evBeg[layer], net->evEnd[layer]));
  return 0;
}

int qcnn_net_layer_work(qcnn_net* net, int layer, int N, double* alg_bytes, double* lookups, double* lut_macs) {
  QCNN_CHECK(net, "qcnn_net_layer_work: NULL net");
  QCNN_CHECK(layer >= 0 && layer < static_cast<int>(net->layers.size()), "qcnn_net_layer_work: bad layer index");
  const NetLayer& nl = net->layers[layer];
  if (nl.pq) return qcnn_layer_work(nl.pq, N, alg_bytes, lookups, lut_macs);
  // non-PQ layers stream their input and output maps once
  const double in = 4.0 * N * nl.Hin * nl.Win * nl.Cin, outb = 4.0 * N * nl.Hout * nl.Wout * nl.Cout;
  if (alg_bytes) *alg_bytes = (nl.info.type == QCNN_DRPT) ? 0.0 : in + outb;
  if (lookups) *lookups = 0.0;
  if (lut_macs) *lut_macs = 0.0;
  return 0;
}

}  // extern "C"
