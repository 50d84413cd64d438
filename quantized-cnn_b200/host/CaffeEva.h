// Network executor with the reference's CaffeEva interface (/root/reference/include/CaffeEva.h:60-195), running the
// PQ forward pass on the GPU through the C ABI of include/qcnn.h -- this file uses NOTHING but that C ABI, so it is
// also the template for the binding a maintainer adds to the reference's own CaffeEva.cc (see INTEGRATION.md).
//
// Same public methods and semantics; differences:
//   * the batch size is whatever the caller passes (the reference hard-codes kDataCntInBatch = 1, CaffeEva.cc:23);
//   * only the approximate (PQ) path exists: Init(false) makes LoadCaffePara fail with a message -- there is no
//     exact (sgemm) path and no CPU fallback;
//   * the CalcFeatMap_* kernels are public so each one can be driven and checked on its own;
//   * timings reported by DispElpsTime come from CUDA events, not clock().
#ifndef QCNN_HOST_CAFFEEVA_H_
#define QCNN_HOST_CAFFEEVA_H_

#include <string>
#include <vector>

#include "../../include/qcnn.h"
#include "CaffePara.h"
#include "Matrix.h"

class CaffeEva {
 public:
  CaffeEva(void);
  ~CaffeEva(void);

 public:
  void Init(const bool enblAprxSrc);
  void SetModelName(const std::string& modelNameSrc);
  void SetModelPath(const std::string& dirPathMainSrc, const std::string& fileNamePfxSrc);
  bool LoadDataset(const std::string& dirPathData);
  bool LoadCaffePara(void);
  void ExecForwardPass(void);
  void ExecForwardPass(const Matrix<float>& imgDataIn, Matrix<float>* pProbVecOut);
  void CalcPredAccu(void);
  float DispElpsTime(void);

  // extensions (not in the reference)
  void SetDevice(const int deviceInd) { device = deviceInd; }
  // > 1: ExecForwardPass shards every batch over GPUs 0 .. n-1 of this process (qcnn_multi_*: replicas + NCCL all-gather
  // of the probabilities); call before LoadCaffePara
  void SetDeviceCount(const int deviceCntSrc) { deviceCnt = deviceCntSrc < 1 ? 1 : deviceCntSrc; }
  void SetEvalCount(const int imgCnt, const int batchSiz) { evalCnt = imgCnt; evalBatch = batchSiz; }
  // Decoded pictures in, top-k out, everything between on the GPU: BmpImgIO's ReszImg / RmMeanImg / CropImg
  // (qcnn_preproc_run), the forward pass, and the k-fold arg-max of CaffeEvaWrapper::Proc (qcnn_topk).  `pixels` holds
  // imgCnt images back to back (interleaved B, G, R bytes, top row first; image i is hei[i] x wid[i]).
  bool SetPreproc(const int reszType, const int meanType, const int heiFull, const int widFull, const int heiCrop,
                  const int widCrop, const Matrix<float>& meanImg);
  bool ClassifyPixels(const unsigned char* pixels, const int* hei, const int* wid, const int imgCnt, const int topk,
                      std::vector<int>* pClsIdxLst, std::vector<float>* pClsProbLst);
  const std::string& GetErrorMsg(void) const { return errorMsg; }
  const CaffePara& GetCaffePara(void) const { return caffeParaObj; }
  const Matrix<uint16_t>& GetPredLabels(void) const { return lablVecPred; }

  // per-layer kernels, same signatures as the reference's private members (CaffeEva.h:145-170); host matrices in,
  // host matrices out (NHWC maps; FC: [N, Din] -> [N,1,1,Dout])
  void CalcFeatMap(const Matrix<float>& featMapSrc, const int layerInd, Matrix<float>* pFeatMapDst);
  void CalcFeatMap_ConvAprx(const Matrix<float>& featMapSrc, const int layerInd, Matrix<float>* pFeatMapDst);
  void CalcFeatMap_FCntAprx(const Matrix<float>& featMapSrc, const int layerInd, Matrix<float>* pFeatMapDst);
  void CalcFeatMap_Pool(const Matrix<float>& featMapSrc, const int layerInd, Matrix<float>* pFeatMapDst);
  void CalcFeatMap_ReLu(const Matrix<float>& featMapSrc, const int layerInd, Matrix<float>* pFeatMapDst);
  void CalcFeatMap_LoRN(const Matrix<float>& featMapSrc, const int layerInd, Matrix<float>* pFeatMapDst);
  void CalcFeatMap_Drpt(const Matrix<float>& featMapSrc, const int layerInd, Matrix<float>* pFeatMapDst);
  void CalcFeatMap_SMax(const Matrix<float>& featMapSrc, const int layerInd, Matrix<float>* pFeatMapDst);

 private:
  bool enblAprx;
  int device;
  int deviceCnt;
  int evalCnt, evalBatch;
  std::string modelName, dirPathMain, fileNamePfx, errorMsg;
  CaffePara caffeParaObj;
  Matrix<float> dataLst;
  Matrix<uint16_t> lablVecGrth;
  Matrix<uint16_t> lablVecPred;
  qcnn_ctx* ctx;
  qcnn_net* net;
  qcnn_preproc* preproc;             // GPU BmpImgIO (SetPreproc)
  qcnn_multi* multi;                 // deviceCnt > 1: the sharded executor (net stays for the per-layer members)
  double msAllLayers;                // accumulated device time of ExecForwardPass calls since the last DispElpsTime
  std::vector<double> msIndvLayerLst;

  bool Fail(const std::string& what);
  void AccumulateTimes(void);
  // upload src, run `op` on device buffers, download into pFeatMapDst (already sized)
  template <typename Op>
  void RunOnDevice(const Matrix<float>& src, Matrix<float>* dst, Op op);
  void CvtFeatMapToLablVec(const int dataIndL, const int dataIndU, const float* probs, const int probVecLen);
};

#endif  // QCNN_HOST_CAFFEEVA_H_
