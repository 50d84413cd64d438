// Model description + parameter loading, same public interface as the reference's CaffePara
// (/root/reference/include/CaffePara.h:24-107); host-only, not a GPU target (SURVEY.md section 2: "KEPT").
// The six architecture tables are carried as compact builder chains (CaffePara.cc) instead of the
// reference's one-call-per-layer listings; the resulting layerInfoLst contents are identical.
#ifndef QCNN_HOST_CAFFEPARA_H_
#define QCNN_HOST_CAFFEPARA_H_

#include <cstdint>
#include <string>
#include <vector>

#include "Matrix.h"

enum class ENUM_AsmtEnc { Raw, Compact };
enum class ENUM_LyrType { Conv, Pool, FCnt, ReLU, LoRN, Drpt, SMax };

typedef struct {
  ENUM_LyrType type;
  int padSiz;    // zero padding on each side (conv / pool)
  int knlSiz;    // kernel width == height
  int knlCnt;    // conv: number of output channels
  int grpCnt;    // conv: number of channel groups
  int stride;    // conv / pool stride
  int nodCnt;    // fully-connected: number of outputs
  int lrnSiz;    // LRN window (channels)
  float lrnAlp;  // LRN alpha
  float lrnBet;  // LRN beta
  float lrnIni;  // LRN k
  float drpRat;  // dropout ratio (unused at test time)
} LayerInfo;
typedef std::vector<LayerInfo> LayerInfoLst;

typedef struct {
  Matrix<float> convKnlLst;  // exact path only (not shipped / out of scope)
  Matrix<float> fcntWeiMat;  // exact path only
  Matrix<float> biasVec;     // [Cout] / [Dout]
  Matrix<float> ctrdLst;     // [S][K][d]
  Matrix<uint8_t> asmtLst;   // conv [Cout][k][k][S] / FC [Dout][S], 0-based after LoadLayerPara
} LayerPara;
typedef std::vector<LayerPara> LayerParaLst;

class CaffePara {
 public:
  void Init(const std::string& dirPathSrc, const std::string& filePfxSrc);
  void ConfigLayer_AlexNet(void);
  void ConfigLayer_CaffeNet(void);
  void ConfigLayer_VggCnnS(void);
  void ConfigLayer_VGG16(void);
  void ConfigLayer_CaffeNetFGB(void);
  void ConfigLayer_CaffeNetFGD(void);
  // by name, as CaffeEva::LoadCaffePara dispatches (reference src/CaffeEva.cc:117-132); false if unknown
  bool ConfigLayer_ByName(const std::string& modelName);
  bool LoadLayerPara(const bool enblAprx, const ENUM_AsmtEnc asmtEnc);
  bool CvtAsmtEnc(const ENUM_AsmtEnc asmtEncSrc, const ENUM_AsmtEnc asmtEncDst);
  // <dirPath>/<filePfx>.<kind>.NN.<ext>, NN = layerInd + 1 (reference src/CaffePara.cc:262-281)
  std::string ParaPath(const char* kind, int layerInd, const char* ext) const;

 public:
  std::string dirPath;
  std::string filePfx;
  int layerCnt;
  int imgChnIn;
  int imgHeiIn;
  int imgWidIn;
  LayerInfoLst layerInfoLst;
  LayerParaLst layerParaLst;

 private:
  int CalcBitCntPerEle(const Matrix<uint8_t>& asmtLst);
};

#endif  // QCNN_HOST_CAFFEPARA_H_
