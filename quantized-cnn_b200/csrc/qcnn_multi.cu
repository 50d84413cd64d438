// Multi-GPU behind the C ABI (SURVEY.md 8(e)): ONE process drives R GPUs of a box.  The path shards by image -- rank r
// owns a contiguous slice of the batch, the weights (20.4 MB for AlexNet) are replicated, nothing is exchanged while the
// layers run -- and the only collective is one ncclAllGather of the [N/R, out_len] probabilities per rank over
// NVLink / NVSwitch, after which every GPU holds the [N, out_len] result (what CaffeEva::ExecForwardPass would leave in
// featMapLst[layerCnt], reference src/CaffeEva.cc:213-261, had the batch run on one device).
//
// Streams: each rank has a compute stream and a gather stream.  The all-gather of step i waits (event) for step i's
// softmax and runs on the gather stream, so step i+1's layers start on the compute stream at once and the collective
// overlaps them; shard buffers alternate between two sets so a gather in flight is never overwritten.
//
// NCCL is bound at run time (dlopen of libnccl.so.2, the copy the process already has if any): single-GPU users of the
// library do not need it, and nothing here falls back to host staging when it is missing -- the call fails.
#include <dlfcn.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "qcnn_internal.h"

using namespace qcnn;

namespace {

// minimal NCCL surface (nccl.h: ncclResult_t, ncclComm_t, ncclDataType_t; ncclFloat32 == 7, ncclSuccess == 0)
typedef struct ncclComm* NcclComm;
struct NcclApi {
  void* lib;
  int (*CommInitAll)(NcclComm*, int, const int*);
  int (*CommDestroy)(NcclComm);
  int (*AllGather)(const void*, void*, size_t, int, NcclComm, cudaStream_t);
  int (*GroupStart)(void);
  int (*GroupEnd)(void);
  const char* (*GetErrorString)(int);
  int (*GetVersion)(int*);
};

NcclApi* LoadNccl() {
  static NcclApi api;
  static int state = 0;   // 0 untried, 1 ok, -1 failed
  if (state == 1) return &api;
  if (state == -1) return nullptr;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  void* lib = nullptr;
  for (const char* n : names) {
    lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (lib) break;
  }
  if (!lib) { state = -1; SetError("qcnn_multi: cannot load libnccl.so.2 (%s)", dlerror()); return nullptr; }
  api.lib = lib;
#define QCNN_SYM(field, name)                                                     \
  *reinterpret_cast<void**>(&api.field) = dlsym(lib, name);                       \
  if (!api.field) { state = -1; SetError("qcnn_multi: libnccl has no %s", name); return nullptr; }
  QCNN_SYM(CommInitAll, "ncclCommInitAll")
  QCNN_SYM(CommDestroy, "ncclCommDestroy")
  QCNN_SYM(AllGather, "ncclAllGather")
  QCNN_SYM(GroupStart, "ncclGroupStart")
  QCNN_SYM(GroupEnd, "ncclGroupEnd")
  QCNN_SYM(GetErrorString, "ncclGetErrorString")
  QCNN_SYM(GetVersion, "ncclGetVersion")
#undef QCNN_SYM
  state = 1;
  return &api;
}

}  // namespace

// puts the caller's current device back when a multi-GPU call returns
struct RestoreDevice {
  int prev;
  RestoreDevice() : prev(-1) { if (cudaGetDevice(&prev) != cudaSuccess) prev = -1; }
  ~RestoreDevice() { if (prev >= 0) cudaSetDevice(prev); }
};

struct qcnn_multi {
  int R;
  std::vector<int> dev;
  std::vector<qcnn_ctx*> ctx;
  std::vector<qcnn_net*> net;
  std::vector<NcclComm> comm;
  std::vector<cudaStream_t> stComp, stGath;
  std::vector<cudaEvent_t> evFwd[2], evGath[2];   // per buffer set: forward of the shard done / gather done
  std::vector<DeviceBuffer> dImg;                 // host-buffer entry: device copy of the rank's image shard
  std::vector<DeviceBuffer> dShard[2];            // [per][out] probabilities of the rank's shard (two sets)
  std::vector<DeviceBuffer> dAll[2];              // [R * per][out] gathered probabilities (two sets)
  unsigned long long step;
  NcclApi* nccl;
  int outLen, imgLen;
};

static int NcclFail(qcnn_multi* m, int rc, const char* what) {
  SetError("NCCL error %d (%s) in %s", rc, m->nccl->GetErrorString(rc), what);
  return 3;
}

static int EnsureMultiCapacity(qcnn_multi* m, int per, bool needImg) {
  const size_t shard = sizeof(float) * static_cast<size_t>(per) * m->outLen;
  for (int r = 0; r < m->R; r++) {
    for (int b = 0; b < 2; b++) {
      bool grown = false;
      QCNN_CUDA(m->dShard[b][r].Reserve(m->ctx[r], shard, nullptr, &grown));
      if (grown) {
        QCNN_ON_DEVICE(m->dev[r]);
        QCNN_CUDA(cudaMemset(m->dShard[b][r].get(), 0, shard));
      }
      QCNN_CUDA(m->dAll[b][r].Reserve(m->ctx[r], m->R * shard));
    }
    if (needImg) QCNN_CUDA(m->dImg[r].Reserve(m->ctx[r], sizeof(float) * static_cast<size_t>(per) * m->imgLen));
  }
  return 0;
}

// rows [lo, hi) of the batch owned by rank r: contiguous shards of `per` = ceil(N / R) images
static void ShardRange(int N, int R, int r, int* per, int* lo, int* hi) {
  *per = CeilDiv(N, R);
  *lo = std::min(N, r * *per);
  *hi = std::min(N, (r + 1) * *per);
}

static int FinishCreate(qcnn_multi* m) {
  m->outLen = qcnn_net_out_len(m->net[0]);
  const float* dummy = nullptr;
  int d4[4];
  qcnn_net_featmap(m->net[0], 0, &dummy, d4);
  m->imgLen = d4[1] * d4[2] * d4[3];
  // communicator clique of the R devices of this process (NVLink / NVSwitch underneath)
  int rc = m->nccl->CommInitAll(m->comm.data(), m->R, m->dev.data());
  if (rc != 0) return NcclFail(m, rc, "ncclCommInitAll");
  for (int r = 0; r < m->R; r++) {
    QCNN_CUDA(cudaSetDevice(m->dev[r]));
    QCNN_CUDA(cudaStreamCreateWithFlags(&m->stComp[r], cudaStreamNonBlocking));
    QCNN_CUDA(cudaStreamCreateWithFlags(&m->stGath[r], cudaStreamNonBlocking));
    for (int b = 0; b < 2; b++) {
      QCNN_CUDA(cudaEventCreateWithFlags(&m->evFwd[b][r], cudaEventDisableTiming));
      QCNN_CUDA(cudaEventCreateWithFlags(&m->evGath[b][r], cudaEventDisableTiming));
    }
  }
  return 0;
}

static qcnn_multi* NewMulti(int R, const int* devices) {
  qcnn_multi* m = new qcnn_multi();
  m->R = R;
  m->dev.resize(R);
  for (int r = 0; r < R; r++) m->dev[r] = devices ? devices[r] : r;
  m->ctx.assign(R, nullptr); m->net.assign(R, nullptr); m->comm.assign(R, nullptr);
  m->stComp.assign(R, nullptr); m->stGath.assign(R, nullptr);
  for (int b = 0; b < 2; b++) {
    m->evFwd[b].assign(R, nullptr); m->evGath[b].assign(R, nullptr);
    m->dShard[b].resize(R); m->dAll[b].resize(R);
  }
  m->dImg.resize(R);
  m->step = 0; m->nccl = nullptr; m->outLen = 0; m->imgLen = 0;
  return m;
}

extern "C" {

void qcnn_multi_destroy(qcnn_multi* m) {
  if (!m) return;
  RestoreDevice restore;
  for (int r = 0; r < m->R; r++) {
    if (!m->ctx[r]) continue;          // creation failed before this rank (e.g. a device that does not exist)
    cudaSetDevice(m->dev[r]);
    if (m->stComp[r]) cudaStreamSynchronize(m->stComp[r]);
    if (m->stGath[r]) cudaStreamSynchronize(m->stGath[r]);
  }
  for (int r = 0; r < m->R; r++) {
    if (!m->ctx[r]) continue;
    cudaSetDevice(m->dev[r]);
    if (m->comm[r] && m->nccl) m->nccl->CommDestroy(m->comm[r]);
    for (int b = 0; b < 2; b++) {
      if (m->evFwd[b][r]) cudaEventDestroy(m->evFwd[b][r]);
      if (m->evGath[b][r]) cudaEventDestroy(m->evGath[b][r]);
    }
    if (m->stComp[r]) cudaStreamDestroy(m->stComp[r]);
    if (m->stGath[r]) cudaStreamDestroy(m->stGath[r]);
    if (m->net[r]) qcnn_net_destroy(m->net[r]);
    if (m->ctx[r]) qcnn_ctx_destroy(m->ctx[r]);
  }
  cudaGetLastError();
  delete m;
}

int qcnn_multi_create(int n_dev, const int* devices, const char* model_name, const char* dir, const char* pfx, qcnn_multi** out) {
  QCNN_CHECK(out && model_name && dir && pfx && n_dev >= 1 && n_dev <= 64, "qcnn_multi_create: bad argument");
  RestoreDevice restore;
  *out = nullptr;
  NcclApi* api = LoadNccl();
  if (!api) return 3;
  qcnn_multi* m = NewMulti(n_dev, devices);
  m->nccl = api;
  int rc = 0;
  for (int r = 0; r < n_dev && rc == 0; r++) {
    rc = qcnn_ctx_create(m->dev[r], &m->ctx[r]);
    if (rc == 0) rc = qcnn_net_create(m->ctx[r], model_name, dir, pfx, &m->net[r]);
  }
  if (rc == 0) rc = FinishCreate(m);
  if (rc) { qcnn_multi_destroy(m); return rc; }
  *out = m;
  return 0;
}

int qcnn_multi_create_from_para(int n_dev, const int* devices, int layer_cnt, const qcnn_layer_info* layers,
                                const qcnn_layer_para* para, int img_chn, int img_hei, int img_wid, qcnn_multi** out) {
  QCNN_CHECK(out && layers && para && n_dev >= 1 && n_dev <= 64, "qcnn_multi_create_from_para: bad argument");
  RestoreDevice restore;
  *out = nullptr;
  NcclApi* api = LoadNccl();
  if (!api) return 3;
  qcnn_multi* m = NewMulti(n_dev, devices);
  m->nccl = api;
  int rc = 0;
  for (int r = 0; r < n_dev && rc == 0; r++) {
    rc = qcnn_ctx_create(m->dev[r], &m->ctx[r]);
    if (rc == 0) rc = qcnn_net_create_from_para(m->ctx[r], layer_cnt, layers, para, img_chn, img_hei, img_wid, &m->net[r]);
  }
  if (rc == 0) rc = FinishCreate(m);
  if (rc) { qcnn_multi_destroy(m); return rc; }
  *out = m;
  return 0;
}

int qcnn_multi_device_count(const qcnn_multi* m) { return m ? m->R : 0; }
int qcnn_multi_out_len(const qcnn_multi* m) { return m ? m->outLen : 0; }
qcnn_net* qcnn_multi_net(qcnn_multi* m, int rank) { return (m && rank >= 0 && rank < m->R) ? m->net[rank] : nullptr; }

int qcnn_multi_nccl_version(const qcnn_multi* m) {
  int v = 0;
  if (m && m->nccl) m->nccl->GetVersion(&v);
  return v;
}

// One step, device-resident and asynchronous: img_dev[r] = rank r's shard of the batch ([hi - lo][C][H][W] on device r,
// shards of ceil(N / R) images, the last one shorter); afterwards (qcnn_multi_sync) *prob_all_dev[r] points at the
// [N][out_len] probabilities on device r (a library-owned buffer, valid until the step after next).
int qcnn_multi_forward(qcnn_multi* m, const float* const* img_dev, int N, const float** prob_all_dev) {
  QCNN_CHECK(m && img_dev && N >= 1, "qcnn_multi_forward: bad argument");
  RestoreDevice restore;
  int per, lo, hi;
  ShardRange(N, m->R, 0, &per, &lo, &hi);
  if (int rc = EnsureMultiCapacity(m, per, false)) return rc;
  const int b = static_cast<int>(m->step & 1);
  for (int r = 0; r < m->R; r++) {
    ShardRange(N, m->R, r, &per, &lo, &hi);
    QCNN_CUDA(cudaSetDevice(m->dev[r]));
    // the shard buffer of this set was last read by the gather two steps ago
    if (m->step >= 2) QCNN_CUDA(cudaStreamWaitEvent(m->stComp[r], m->evGath[b][r], 0));
    if (hi > lo) {
      QCNN_CHECK(img_dev[r] != nullptr, "qcnn_multi_forward: img_dev[%d] is NULL", r);
      if (int rc = qcnn_net_forward(m->net[r], img_dev[r], hi - lo, m->dShard[b][r].as<float>(), nullptr, m->stComp[r])) return rc;
    }
    QCNN_CUDA(cudaEventRecord(m->evFwd[b][r], m->stComp[r]));
    QCNN_CUDA(cudaStreamWaitEvent(m->stGath[r], m->evFwd[b][r], 0));
  }
  // the path's only exchange: all ranks gather every shard (equal counts: `per` rows each, the tail shard padded)
  int rc = m->nccl->GroupStart();
  if (rc != 0) return NcclFail(m, rc, "ncclGroupStart");
  for (int r = 0; r < m->R; r++) {
    rc = m->nccl->AllGather(m->dShard[b][r].get(), m->dAll[b][r].get(), static_cast<size_t>(per) * m->outLen, 7 /* ncclFloat32 */,
                            m->comm[r], m->stGath[r]);
    if (rc != 0) { m->nccl->GroupEnd(); return NcclFail(m, rc, "ncclAllGather"); }
  }
  rc = m->nccl->GroupEnd();
  if (rc != 0) return NcclFail(m, rc, "ncclGroupEnd");
  for (int r = 0; r < m->R; r++) {
    QCNN_CUDA(cudaSetDevice(m->dev[r]));
    QCNN_CUDA(cudaEventRecord(m->evGath[b][r], m->stGath[r]));
    if (prob_all_dev) prob_all_dev[r] = m->dAll[b][r].as<float>();
  }
  m->step++;
  return 0;
}

int qcnn_multi_sync(qcnn_multi* m) {
  QCNN_CHECK(m, "qcnn_multi_sync: NULL argument");
  RestoreDevice restore;
  for (int r = 0; r < m->R; r++) {
    QCNN_CUDA(cudaSetDevice(m->dev[r]));
    QCNN_CUDA(cudaStreamSynchronize(m->stComp[r]));
    QCNN_CUDA(cudaStreamSynchronize(m->stGath[r]));
  }
  return 0;
}

// host-buffer step == CaffeEva::ExecForwardPass(imgDataIn, pProbVecOut) on R GPUs: the image shards go host -> device on
// every rank's own stream (concurrent copies over every GPU's own link), forward, all-gather, rank 0's copy of the
// gathered [N][out_len] probabilities comes back; synchronises.
int qcnn_multi_forward_h(qcnn_multi* m, const float* img_h, int N, float* prob_h) {
  QCNN_CHECK(m && img_h && prob_h && N >= 1, "qcnn_multi_forward_h: bad argument");
  RestoreDevice restore;
  int per, lo, hi;
  ShardRange(N, m->R, 0, &per, &lo, &hi);
  if (int rc = EnsureMultiCapacity(m, per, true)) return rc;
  std::vector<const float*> img(m->R, nullptr);
  for (int r = 0; r < m->R; r++) {
    ShardRange(N, m->R, r, &per, &lo, &hi);
    QCNN_CUDA(cudaSetDevice(m->dev[r]));
    if (hi > lo)
      QCNN_CUDA(cudaMemcpyAsync(m->dImg[r].get(), img_h + static_cast<size_t>(lo) * m->imgLen, sizeof(float) * (hi - lo) * m->imgLen,
                                cudaMemcpyHostToDevice, m->stComp[r]));
    img[r] = m->dImg[r].as<float>();
  }
  std::vector<const float*> all(m->R, nullptr);
  if (int rc = qcnn_multi_forward(m, img.data(), N, all.data())) return rc;
  QCNN_CUDA(cudaSetDevice(m->dev[0]));
  QCNN_CUDA(cudaMemcpyAsync(prob_h, all[0], sizeof(float) * static_cast<size_t>(N) * m->outLen, cudaMemcpyDeviceToHost, m->stGath[0]));
  return qcnn_multi_sync(m);
}

}  // extern "C"
