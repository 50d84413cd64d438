// Single-image classification API, same interface as the reference's CaffeEvaWrapper
// (/root/reference/include/CaffeEvaWrapper.h:38-142): SetPath / SetModel / Proc / GetErrorMsg / ClrErrorMsg and the
// CaffeEvaRslt result record.  Host glue only; the forward pass runs on the GPU through CaffeEva -> C ABI.
#ifndef QCNN_HOST_CAFFEEVAWRAPPER_H_
#define QCNN_HOST_CAFFEEVAWRAPPER_H_

#include <string>
#include <vector>

#include "BmpImgIO.h"
#include "CaffeEva.h"

enum class ENUM_CaffeModel { AlexNet, CaffeNet, VggCnnS, VGG16, CaffeNetFGB, CaffeNetFGD };
enum class ENUM_CompMethod { Prec, Aprx };

typedef struct {
  int clsCntPred;                       // in: how many top classes to return
  float timeTotal;                      // out: forward-pass time (s), CUDA events
  bool hasGrthClsName;
  std::string clsNameGrth;
  std::vector<int> clsIdxLst;
  std::vector<float> clsProbLst;
  std::vector<std::string> clsNameLst;
} CaffeEvaRslt;

class CaffeEvaWrapper {
 public:
  CaffeEvaWrapper(void);
  bool SetPath(const std::string& mainDirPathSrc, const std::string& clsNameFilePath,
               const std::string& imgLablFilePath = "");
  bool SetModel(const ENUM_CaffeModel& caffeModelSrc, const ENUM_CompMethod& compMethodSrc);
  bool Proc(const std::string& filePathProcImg, CaffeEvaRslt* pCaffeEvaRslt);
  std::string GetErrorMsg(void);
  void ClrErrorMsg(void);

 private:
  struct GrthEntry { std::string fileName, clsName; };
  std::string mainDirPath;
  BmpImgIO bmpImgIOObj;
  CaffeEva caffeEvaObj;
  std::vector<std::string> clsNameLst;
  std::vector<GrthEntry> clsNameGrthLst;
  std::string errorMsg;

  bool LoadClsName(const std::string& filePath);
  bool LoadImgLabl(const std::string& filePath);
  static std::string ExtrFileName(const std::string& filePath);
};

#endif  // QCNN_HOST_CAFFEEVAWRAPPER_H_
