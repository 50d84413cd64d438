// extern-"C" test hooks into the C++ host layer (libqcnn_host.so) for the Python test-suite.
#include <cstring>

#include "BmpImgIO.h"
#include "CaffePara.h"

extern "C" {

// BmpImgIO with the AlexNet recipe of CaffeEvaWrapper::SetModel (resize 256x256 strict, full-size mean, crop 227):
// out [3][227][227] BGR mean-subtracted; returns the element count or -1
__attribute__((visibility("default"))) int qcnn_host_load_bmp_alexnet(const char* meanPath, const char* bmpPath,
                                                                      float* out, int cap) {
  BmpImgIOPara p;
  p.reszType = ENUM_ReszType::Strict;
  p.meanType = ENUM_MeanType::Full;
  p.imgHeiFull = p.imgWidFull = 256;
  p.imgHeiCrop = p.imgWidCrop = 227;
  p.filePathMean = meanPath;
  BmpImgIO io;
  if (!io.Init(p)) return -1;
  Matrix<float> img;
  if (!io.Load(bmpPath, &img)) return -1;
  const int n = img.GetEleCnt();
  memcpy(out, img.GetDataPtr(), sizeof(float) * (n < cap ? n : cap));
  return n;
}

// BmpImgIO with any recipe: resz_type 0 Strict / 1 Relaxed, mean_type 0 Full / 1 Crop (the ENUM orders), mean file
// [3][H][W]; out [3][hei_crop][wid_crop] BGR mean-subtracted; returns the element count or -1
__attribute__((visibility("default"))) int qcnn_host_load_bmp(const char* bmpPath, const char* meanPath, int reszType,
                                                              int meanType, int heiFull, int widFull, int heiCrop,
                                                              int widCrop, float* out, int cap) {
  BmpImgIOPara p;
  p.reszType = static_cast<ENUM_ReszType>(reszType);
  p.meanType = static_cast<ENUM_MeanType>(meanType);
  p.imgHeiFull = heiFull;
  p.imgWidFull = widFull;
  p.imgHeiCrop = heiCrop;
  p.imgWidCrop = widCrop;
  p.filePathMean = meanPath;
  BmpImgIO io;
  if (!io.Init(p)) return -1;
  Matrix<float> img;
  if (!io.Load(bmpPath, &img)) return -1;
  const int n = img.GetEleCnt();
  memcpy(out, img.GetDataPtr(), sizeof(float) * (n < cap ? n : cap));
  return n;
}

// layer table of a named model: writes up to cap records of 12 ints/floats (LayerInfo order); returns layerCnt
__attribute__((visibility("default"))) int qcnn_host_layer_table(const char* model, int* imgChw, int* types, int cap) {
  CaffePara para;
  if (!para.ConfigLayer_ByName(model)) return -1;
  imgChw[0] = para.imgChnIn; imgChw[1] = para.imgHeiIn; imgChw[2] = para.imgWidIn;
  for (int l = 0; l < para.layerCnt && l < cap; l++) types[l] = static_cast<int>(para.layerInfoLst[l].type);
  return para.layerCnt;
}

}  // extern "C"
