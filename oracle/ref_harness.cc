// TEST INFRASTRUCTURE ONLY -- never linked into, imported by, or called from the product path.
//
// Thin extern-"C" harness around the UNMODIFIED reference sources
// (/root/reference/src/{CaffeEva,CaffePara,BlasWrapper}.cc), compiled where they lie by
// oracle/Makefile into oracle/_ref/libqcnn_ref.so (git-ignored).  It exposes the reference's own
// CaffeEva object so tests / bench.py's cpu_baseline leg can
//   * run the whole PQ forward pass  (CaffeEva::ExecForwardPass(img,prob), CaffeEva.cc:213-261),
//   * run ONE layer kernel            (CaffeEva::CalcFeatMap, CaffeEva.cc:625-670 -> _ConvAprx/_FCntAprx/...),
//   * read back every feature map and the decoded parameters (CaffePara::layerParaLst),
//   * drive the reference with a caller-supplied layer table (synthetic S x K sweeps).
// The private members are reached with the "#define private public" include trick (SURVEY.md 8(c)).
// No reference source text is copied here: only its public/private *names* are used.

#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdint.h>
#include <unistd.h>
#include <fcntl.h>
#include <math.h>
#include <time.h>

#include <algorithm>
#include <iostream>
#include <sstream>
#include <string>
#include <typeinfo>
#include <vector>

#define private public
#include "include/CaffeEva.h"
#include "include/FileIO.h"
#include "include/CaffeEvaWrapper.h"
#undef private

namespace {

// The reference printf()s on every call; silence fd 1 while it runs.
struct StdoutMute {
  int saved;
  explicit StdoutMute(bool on) : saved(-1) {
    if (!on) return;
    fflush(stdout);
    saved = dup(1);
    int nul = open("/dev/null", O_WRONLY);
    if (nul >= 0) { dup2(nul, 1); close(nul); }
  }
  ~StdoutMute() {
    if (saved < 0) return;
    fflush(stdout);
    dup2(saved, 1);
    close(saved);
  }
};

struct RefNet {
  CaffeEva eva;
  bool quiet;
};

double NowMs() {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6;
}

}  // namespace

extern "C" {

// layer spec record used by ref_net_create_custom (one per layer), mirrors LayerInfo (CaffePara.h:28-41)
struct RefLayerSpec {
  int type;      // ENUM_LyrType order: 0 Conv, 1 Pool, 2 FCnt, 3 ReLU, 4 LoRN, 5 Drpt, 6 SMax
  int padSiz, knlSiz, knlCnt, grpCnt, stride, nodCnt, lrnSiz;
  float lrnAlp, lrnBet, lrnIni, drpRat;
};

// Standard model tables (ConfigLayer_<name>), parameters loaded through the reference's own LoadCaffePara.
void* ref_net_create(const char* dir, const char* pfx, const char* model, int quiet) {
  RefNet* net = new RefNet();
  net->quiet = quiet != 0;
  StdoutMute mute(net->quiet);
  net->eva.Init(true);
  net->eva.SetModelName(model);
  net->eva.SetModelPath(dir, pfx);
  if (!net->eva.LoadCaffePara()) {
    // NOTE: the reference destructor assumes featMapLst was allocated; leak instead of crashing.
    return nullptr;
  }
  return net;
}

// Caller-supplied layer table: same steps as CaffeEva::LoadCaffePara (CaffeEva.cc:109-149) with the
// ConfigLayer_* call replaced by the given table.
void* ref_net_create_custom(const char* dir, const char* pfx, int layerCnt, const RefLayerSpec* specs,
                            int imgChn, int imgHei, int imgWid, int quiet) {
  RefNet* net = new RefNet();
  net->quiet = quiet != 0;
  StdoutMute mute(net->quiet);
  CaffeEva& eva = net->eva;
  eva.Init(true);
  eva.SetModelName("custom");
  eva.SetModelPath(dir, pfx);
  CaffePara& para = eva.caffeParaObj;
  para.Init(dir, pfx);
  para.layerCnt = layerCnt;
  para.imgChnIn = imgChn;
  para.imgHeiIn = imgHei;
  para.imgWidIn = imgWid;
  para.layerInfoLst.resize(layerCnt);
  for (int l = 0; l < layerCnt; l++) {
    LayerInfo& li = para.layerInfoLst[l];
    memset(&li, 0, sizeof(li));
    li.type = static_cast<ENUM_LyrType>(specs[l].type);
    li.padSiz = specs[l].padSiz;
    li.knlSiz = specs[l].knlSiz;
    li.knlCnt = specs[l].knlCnt;
    li.grpCnt = specs[l].grpCnt;
    li.stride = specs[l].stride;
    li.nodCnt = specs[l].nodCnt;
    li.lrnSiz = specs[l].lrnSiz;
    li.lrnAlp = specs[l].lrnAlp;
    li.lrnBet = specs[l].lrnBet;
    li.lrnIni = specs[l].lrnIni;
    li.drpRat = specs[l].drpRat;
  }
  if (!para.LoadLayerPara(true, ENUM_AsmtEnc::Compact)) return nullptr;
  eva.PrepFeatMap();
  eva.PrepFeatBuf();
  eva.PrepCtrdBuf();
  eva.PrepAsmtBuf();
  return net;
}

void ref_net_destroy(void* h) { delete static_cast<RefNet*>(h); }

int ref_net_layer_count(void* h) { return static_cast<RefNet*>(h)->eva.caffeParaObj.layerCnt; }

int ref_net_layer_type(void* h, int l) {
  return static_cast<int>(static_cast<RefNet*>(h)->eva.caffeParaObj.layerInfoLst[l].type);
}

// Whole forward pass on ONE image (the reference hard-codes kDataCntInBatch = 1, CaffeEva.cc:23).
// img: [1,C,H,W] f32 (NCHW, BGR, mean-subtracted); prob: [nodCnt of last layer].
int ref_net_forward(void* h, const float* img, float* prob, int probLen) {
  RefNet* net = static_cast<RefNet*>(h);
  StdoutMute mute(net->quiet);
  CaffePara& para = net->eva.caffeParaObj;
  Matrix<float> in(1, para.imgChnIn, para.imgHeiIn, para.imgWidIn);
  memcpy(in.GetDataPtr(), img, sizeof(float) * in.GetEleCnt());
  Matrix<float> out;
  net->eva.ExecForwardPass(in, &out);
  int n = std::min(probLen, out.GetEleCnt());
  memcpy(prob, out.GetDataPtr(), sizeof(float) * n);
  return out.GetEleCnt();
}

// featMapLst[idx] (idx in 0..layerCnt): writes up to 4 dims, returns element count; data may be null.
int ref_net_featmap(void* h, int idx, int* dims, float* data, int cap) {
  RefNet* net = static_cast<RefNet*>(h);
  const Matrix<float>& m = net->eva.featMapLst[idx];
  for (int i = 0; i < 4; i++) dims[i] = (i < m.GetDimCnt()) ? m.GetDimLen(i) : 1;
  int n = m.GetEleCnt();
  if (data != nullptr) memcpy(data, m.GetDataPtr(), sizeof(float) * std::min(n, cap));
  return n;
}

// One layer: copies src into featMapLst[l] (element order exactly as the reference kernel expects it:
// NHWC for conv/pool/lrn/relu, flat [N,Din] for FC) and calls CaffeEva::CalcFeatMap.
int ref_net_layer_forward(void* h, int l, const float* src, int srcLen, float* dst, int dstCap) {
  RefNet* net = static_cast<RefNet*>(h);
  StdoutMute mute(net->quiet);
  Matrix<float>& fs = net->eva.featMapLst[l];
  Matrix<float>& fd = net->eva.featMapLst[l + 1];
  if (srcLen != fs.GetEleCnt()) return -1;
  memcpy(fs.GetDataPtr(), src, sizeof(float) * srcLen);
  net->eva.CalcFeatMap(fs, l, &fd);
  int n = fd.GetEleCnt();
  memcpy(dst, fd.GetDataPtr(), sizeof(float) * std::min(n, dstCap));
  return n;
}

// LUT stage alone (CaffeEva::GetInPdMat, CaffeEva.cc:1261-1296) on caller data.
// data [P,D]; ctrd [S,d,K] (already permuted like ctrdBuf); out [P,S,K].
void ref_get_inpd(const float* data, int P, int D, const float* ctrd, int S, int d, int K, float* out) {
  CaffeEva eva;
  eva.featMapLst = nullptr;
  eva.caffeParaObj.layerCnt = 0;
  Matrix<float> dataLst(P, D), ctrdLst(S, d, K), inPd(P, S, K);
  memcpy(dataLst.GetDataPtr(), data, sizeof(float) * P * D);
  memcpy(ctrdLst.GetDataPtr(), ctrd, sizeof(float) * S * d * K);
  eva.GetInPdMat(dataLst, ctrdLst, &inPd);
  memcpy(out, inPd.GetDataPtr(), sizeof(float) * P * S * K);
}

// Decoded parameters as CaffePara holds them after LoadLayerPara (0-based assignments, file order).
// which: 0 biasVec, 1 ctrdLst, 2 asmtLst.  Returns element count; data may be null.
int ref_net_param(void* h, int l, int which, int* dims, void* data, int capBytes) {
  RefNet* net = static_cast<RefNet*>(h);
  const LayerPara& lp = net->eva.caffeParaObj.layerParaLst[l];
  if (which == 2) {
    const Matrix<uint8_t>& m = lp.asmtLst;
    for (int i = 0; i < 4; i++) dims[i] = (i < m.GetDimCnt()) ? m.GetDimLen(i) : 1;
    int n = m.GetEleCnt();
    if (data != nullptr) memcpy(data, m.GetDataPtr(), std::min(n, capBytes));
    return n;
  }
  const Matrix<float>& m = (which == 0) ? lp.biasVec : lp.ctrdLst;
  for (int i = 0; i < 4; i++) dims[i] = (i < m.GetDimCnt()) ? m.GetDimLen(i) : 1;
  int n = m.GetEleCnt();
  if (data != nullptr) memcpy(data, m.GetDataPtr(), std::min<size_t>(sizeof(float) * n, capBytes));
  return n;
}

// The device-order buffers the reference builds (PrepCtrdBuf / PrepAsmtBuf, CaffeEva.cc:534-623).
int ref_net_ctrdbuf(void* h, int l, int* dims, float* data, int cap) {
  RefNet* net = static_cast<RefNet*>(h);
  const Matrix<float>& m = *(net->eva.ctrdBufStrLst[l].pCtrdBuf);
  for (int i = 0; i < 4; i++) dims[i] = (i < m.GetDimCnt()) ? m.GetDimLen(i) : 1;
  int n = m.GetEleCnt();
  if (data != nullptr) memcpy(data, m.GetDataPtr(), sizeof(float) * std::min(n, cap));
  return n;
}

int ref_net_asmtbuf(void* h, int l, int* dims, uint8_t* data, int cap) {
  RefNet* net = static_cast<RefNet*>(h);
  const Matrix<uint8_t>& m = *(net->eva.asmtBufStrLst[l].pAsmtBuf);
  for (int i = 0; i < 4; i++) dims[i] = (i < m.GetDimCnt()) ? m.GetDimLen(i) : 1;
  int n = m.GetEleCnt();
  if (data != nullptr) memcpy(data, m.GetDataPtr(), std::min(n, cap));
  return n;
}

// Times `iters` forward passes over `imgCnt` images (round-robin), wall clock, single thread.
// Returns total milliseconds; msEach (nullable) gets per-iteration times.
double ref_net_time_forward(void* h, const float* imgs, int imgCnt, int warmup, int iters, double* msEach) {
  RefNet* net = static_cast<RefNet*>(h);
  StdoutMute mute(net->quiet);
  CaffePara& para = net->eva.caffeParaObj;
  Matrix<float> in(1, para.imgChnIn, para.imgHeiIn, para.imgWidIn);
  Matrix<float> out;
  const int len = in.GetEleCnt();
  for (int i = 0; i < warmup; i++) {
    memcpy(in.GetDataPtr(), imgs + static_cast<size_t>(i % imgCnt) * len, sizeof(float) * len);
    net->eva.ExecForwardPass(in, &out);
  }
  double total = 0.0;
  for (int i = 0; i < iters; i++) {
    memcpy(in.GetDataPtr(), imgs + static_cast<size_t>(i % imgCnt) * len, sizeof(float) * len);
    double t0 = NowMs();
    net->eva.ExecForwardPass(in, &out);
    double t1 = NowMs();
    if (msEach != nullptr) msEach[i] = t1 - t0;
    total += t1 - t0;
  }
  return total;
}

// FileIO round trips through the reference's own reader/writer (FileIO.h:56-178, 229-350).
int ref_read_cbn(const char* path, int* dims, uint8_t* data, int cap) {
  StdoutMute mute(true);
  Matrix<uint8_t> m;
  if (!FileIO::ReadCbnFile(path, &m)) return -1;
  for (int i = 0; i < 4; i++) dims[i] = (i < m.GetDimCnt()) ? m.GetDimLen(i) : 1;
  int n = m.GetEleCnt();
  if (data != nullptr) memcpy(data, m.GetDataPtr(), std::min(n, cap));  // 1-based, as the reader returns
  return n;
}

int ref_write_cbn(const char* path, int dimCnt, const int* dims, const uint8_t* data1based, int bits) {
  StdoutMute mute(true);
  Matrix<uint8_t> m(dimCnt, dims);
  memcpy(m.GetDataPtr(), data1based, m.GetEleCnt());
  return FileIO::WriteCbnFile(path, m, bits) ? 0 : -1;
}

int ref_read_bin_f32(const char* path, int* dims, float* data, int cap) {
  StdoutMute mute(true);
  Matrix<float> m;
  if (!FileIO::ReadBinFile(path, &m)) return -1;
  for (int i = 0; i < 4; i++) dims[i] = (i < m.GetDimCnt()) ? m.GetDimLen(i) : 1;
  int n = m.GetEleCnt();
  if (data != nullptr) memcpy(data, m.GetDataPtr(), sizeof(float) * std::min(n, cap));
  return n;
}

int ref_write_bin_f32(const char* path, int dimCnt, const int* dims, const float* data) {
  StdoutMute mute(true);
  Matrix<float> m(dimCnt, dims);
  memcpy(m.GetDataPtr(), data, sizeof(float) * m.GetEleCnt());
  return FileIO::WriteBinFile(path, m) ? 0 : -1;
}

// CaffeEvaWrapper::SetPath + SetModel(AlexNet, Aprx) (CaffeEvaWrapper.cc:15-151); returns a handle or NULL
void* ref_wrapper_create(const char* mainDir, const char* clsNames, const char* imgLabels) {
  StdoutMute mute(true);
  CaffeEvaWrapper* w = new CaffeEvaWrapper();
  if (!w->SetPath(mainDir, clsNames, imgLabels ? imgLabels : "")) return nullptr;
  if (!w->SetModel(ENUM_CaffeModel::AlexNet, ENUM_CompMethod::Aprx)) return nullptr;
  return w;
}

// CaffeEvaWrapper::Proc (CaffeEvaWrapper.cc:153-209): top-k indices / probabilities of one BMP
int ref_wrapper_proc(void* h, const char* bmpPath, int k, int* idx, float* prob) {
  StdoutMute mute(true);
  CaffeEvaWrapper* w = static_cast<CaffeEvaWrapper*>(h);
  CaffeEvaRslt r;
  r.clsCntPred = k;
  if (!w->Proc(bmpPath, &r)) return -1;
  for (int i = 0; i < k; i++) { idx[i] = r.clsIdxLst[i]; prob[i] = r.clsProbLst[i]; }
  return 0;
}

// BmpImgIO::Init + Load (BmpImgIO.cc:16-71) with any recipe: resz_type / mean_type in ENUM_ReszType / ENUM_MeanType
// order, mean file [3][H][W] (FileIO .bin); out [3][hei_crop][wid_crop] BGR, mean-subtracted.  Returns the element
// count or -1.
int ref_bmp_load(const char* bmpPath, const char* meanPath, int reszType, int meanType, int heiFull, int widFull,
                 int heiCrop, int widCrop, float* out, int cap) {
  StdoutMute mute(true);
  BmpImgIOPara para;
  para.reszType = static_cast<ENUM_ReszType>(reszType);
  para.meanType = static_cast<ENUM_MeanType>(meanType);
  para.imgHeiFull = heiFull;
  para.imgWidFull = widFull;
  para.imgHeiCrop = heiCrop;
  para.imgWidCrop = widCrop;
  para.filePathMean = meanPath;
  BmpImgIO io;
  if (!io.Init(para)) return -1;
  Matrix<float> img;
  if (!io.Load(bmpPath, &img)) return -1;
  int n = img.GetEleCnt();
  memcpy(out, img.GetDataPtr(), sizeof(float) * std::min(n, cap));
  return n;
}

// CaffeEva::CvtFeatMapToLablVec (CaffeEva.cc:1162-1190) on a caller's [N][C] matrix: out [N][5] labels
void ref_cvt_featmap_to_labl(const float* prob, int N, int C, uint16_t* out) {
  CaffeEva eva;
  eva.featMapLst = nullptr;
  eva.caffeParaObj.layerCnt = 0;
  Matrix<float> featMap(N, C, 1, 1);
  memcpy(featMap.GetDataPtr(), prob, sizeof(float) * N * C);
  Matrix<uint16_t> labl(N, 5, 1, 1);
  eva.CvtFeatMapToLablVec(0, N - 1, featMap, &labl);
  memcpy(out, labl.GetDataPtr(), sizeof(uint16_t) * N * 5);
}

// BmpImgIO::Load (BmpImgIO.cc:40-71) with the wrapper's AlexNet recipe: out [3][227][227] BGR, mean-subtracted
int ref_wrapper_load_bmp(void* h, const char* bmpPath, float* out, int cap) {
  StdoutMute mute(true);
  CaffeEvaWrapper* w = static_cast<CaffeEvaWrapper*>(h);
  Matrix<float> img;
  if (!w->bmpImgIOObj.Load(bmpPath, &img)) return -1;
  int n = img.GetEleCnt();
  memcpy(out, img.GetDataPtr(), sizeof(float) * std::min(n, cap));
  return n;
}

}  // extern "C"
