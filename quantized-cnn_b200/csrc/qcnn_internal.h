// Internal declarations shared by the .cu / .cc files of libqcnn_b200.so (not part of the C ABI).
#ifndef QCNN_INTERNAL_H_
#define QCNN_INTERNAL_H_

#include <cuda_runtime.h>
#include <stdint.h>

#include <array>
#include <string>
#include <utility>
#include <vector>

#include "../../include/qcnn.h"

class CaffePara;

namespace qcnn {

// thread-local error text behind qcnn_last_error()
void SetError(const char* fmt, ...);
int CudaFail(cudaError_t e, const char* what, const char* file, int line);

#define QCNN_CUDA(call)                                                      \
  do {                                                                       \
    cudaError_t e__ = (call);                                                \
    if (e__ != cudaSuccess) return ::qcnn::CudaFail(e__, #call, __FILE__, __LINE__); \
  } while (0)

#define QCNN_CHECK(cond, ...)            \
  do {                                   \
    if (!(cond)) {                       \
      ::qcnn::SetError(__VA_ARGS__);     \
      return 1;                          \
    }                                    \
  } while (0)

// Every entry point that needs a particular GPU makes it current for the duration of the call and puts the caller's
// device back on return: the CUDA "current device" is process-visible state (PyTorch's default device IS the runtime's),
// and a library that leaves it changed silently moves the caller's next allocation to another GPU.
class DeviceGuard {
 public:
  explicit DeviceGuard(int device) : prev_(-1), err_(cudaSuccess) {
    if (cudaGetDevice(&prev_) != cudaSuccess) prev_ = -1;
    if (prev_ != device) err_ = cudaSetDevice(device); else prev_ = -1;   // nothing to restore when already current
  }
  ~DeviceGuard() { if (prev_ >= 0) cudaSetDevice(prev_); }
  cudaError_t error() const { return err_; }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
 private:
  int prev_;
  cudaError_t err_;
};
#define QCNN_ON_DEVICE(dev)                 \
  ::qcnn::DeviceGuard device_guard__(dev);  \
  QCNN_CUDA(device_guard__.error())

inline int CeilDiv(int a, int b) { return (a + b - 1) / b; }
inline int RoundUp(int a, int b) { return CeilDiv(a, b) * b; }

}  // namespace qcnn

struct qcnn_ctx {
  int device;
  int sm_count;
  int cc_major, cc_minor;
  size_t smem_optin;  // max dynamic shared memory per block (opt-in)
  unsigned long long launches;  // kernels launched through this ctx (monotonic)
  unsigned long long alloc_epoch;  // bumped whenever a device scratch buffer is (re)allocated: captured graphs go stale
};

namespace qcnn {

// dynamic shared memory a block may opt in to (the H100's 227 KiB when the device did not report it)
inline size_t SmemOptin(const qcnn_ctx* ctx) { return ctx->smem_optin ? ctx->smem_optin : 227 * 1024; }

// The one owner of every device allocation the library makes for itself (layer parameters, scratch, executor staging).
// Invariant: bytes() > 0 if and only if get() owns that many bytes on device().  Freed on destruction.
class DeviceBuffer {
 public:
  DeviceBuffer() = default;
  ~DeviceBuffer() { Release(); }
  DeviceBuffer(DeviceBuffer&& o) noexcept : ptr_(o.ptr_), bytes_(o.bytes_), device_(o.device_) { o.ptr_ = nullptr; o.bytes_ = 0; }
  DeviceBuffer& operator=(DeviceBuffer&& o) noexcept {
    if (this != &o) {
      Release();
      ptr_ = o.ptr_; bytes_ = o.bytes_; device_ = o.device_;
      o.ptr_ = nullptr; o.bytes_ = 0;
    }
    return *this;
  }
  DeviceBuffer(const DeviceBuffer&) = delete;
  DeviceBuffer& operator=(const DeviceBuffer&) = delete;

  // Grow-only: makes the buffer hold at least `bytes` on ctx's device (the contents do not survive a growth).  A real
  // (re)allocation bumps ctx->alloc_epoch, since graphs captured before hold the old address, and sets *grown for
  // first-use initialisation.  Refused with cudaErrorStreamCaptureUnsupported while `st` is being captured.
  cudaError_t Reserve(qcnn_ctx* ctx, size_t bytes, cudaStream_t st = nullptr, bool* grown = nullptr) {
    if (grown) *grown = false;
    if (bytes <= bytes_) return cudaSuccess;
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    if (st) cudaStreamIsCapturing(st, &cap);
    if (cap != cudaStreamCaptureStatusNone) return cudaErrorStreamCaptureUnsupported;
    if (cudaError_t e = Release()) return e;
    DeviceGuard guard(ctx->device);
    if (guard.error()) return guard.error();
    if (cudaError_t e = cudaMalloc(&ptr_, bytes)) { ptr_ = nullptr; return e; }
    bytes_ = bytes;
    device_ = ctx->device;
    ctx->alloc_epoch++;
    if (grown) *grown = true;
    return cudaSuccess;
  }
  // Immutable contents: exactly `bytes` copied from the host.
  cudaError_t Upload(qcnn_ctx* ctx, const void* host, size_t bytes) {
    if (cudaError_t e = Release()) return e;
    if (cudaError_t e = Reserve(ctx, bytes)) return e;
    DeviceGuard guard(device_);
    return cudaMemcpy(ptr_, host, bytes, cudaMemcpyHostToDevice);
  }
  cudaError_t Release() {
    cudaError_t e = cudaSuccess;
    if (ptr_) {
      DeviceGuard guard(device_);
      e = guard.error() ? guard.error() : cudaFree(ptr_);
    }
    ptr_ = nullptr;
    bytes_ = 0;
    return e;
  }
  void* get() const { return ptr_; }
  template <class T> T* as() const { return static_cast<T*>(ptr_); }
  size_t bytes() const { return bytes_; }

 private:
  void* ptr_ = nullptr;
  size_t bytes_ = 0;
  int device_ = 0;
};

}  // namespace qcnn

enum { QCNN_KIND_CONV = 0, QCNN_KIND_FC = 1 };

// ---- kernel argument blocks --------------------------------------------------------------------------------
struct FcArgs {
  const float* src;
  float* dst;
  float* partial;      // [nsplit][N][DoutPad] when nsplit > 1
  const float* ctrd;   // [S][K][d] (file order)
  const uint8_t* asmt; // [S][DoutPad], value = idx << kshift
  const float* bias;
  int N, Din, Dout, DoutPad, S, K, d;
  const int* srcoff;   // [Din] element offset of flattened feature f inside one source image (NULL: identity)
  int s_per_split, nsplit;
  int relu;
};

struct ConvArgs {
  const float* src;
  float* dst;
  const float* ctrd;    // [S][K][d] (file order), shared by all groups
  const uint8_t* asmt;  // [G][S][taps][KgPad]
  const float* bias;
  int N, Hi, Wi, Cin, Ho, Wo, Cout, ksz, pad, stride, G, Cg, Kg, KgPad, S, K, d;
  int src_nchw;
  // tiling plan
  int R, nstrips;       // output rows per CTA / strips per image
  int PW;               // s1: row pitch of the flat padded grid; roll: phase length PH
  int RI;               // s1: input rows held per strip
  int CW, ncol;         // s1: output columns per column tile / column tiles per row (1: whole rows)
  int PP;               // LUT pitch in floats (positions per codeword row), multiple of 4
  int NM;               // wgmma LUT stage: LUT columns produced per step (MMA N, multiple of 32, <= 256)
  int CT, nct;          // output channels per CTA (per group) / channel tiles per group
  int pwarps, cwarps, rgroups;
  int relu;
};

// ---- decode-at-use tensor-core GEMM (pq_gemm_tc.cu) ----
constexpr int kMaxKSteps = 96;
struct KStep {           // one K = 8 step of the GEMM: two 4-float halves
  int bStart;            // B operand: first float4 of half 0 inside the staged planes (position 0 of the tile)
  int lbo;               // distance (in float4) from half 0 to half 1
  short idx0, idx1;      // assignment-index row of either half inside the chunk's staged rows
  short cb0, cb1;        // codebook slot of either half inside the chunk's staged slices
};
// A tensor-core GEMM's k-steps in the order its accumulator chains them (Mode0Table / Mode1Table fill it)
struct KStepTable {
  int ntab;
  int chunkFirst[8], chunkCount[8];   // k-step range of a chunk (mode 1: per phase row; else entry 0)
  KStep tab[kMaxKSteps];
};
struct GemmArgs {
  const float* src;
  float* dst;
  const float* ctrd;
  const uint8_t* asmt;
  const float* bias;
  long long srcImg, dstImg;   // elements per source / destination image
  int N, Hi, Wi, Cin, Ho, Wo, Cout, ksz, pad, stride, G, Cg, Kg, KgPad, S, K, d;
  int mode;                   // 0 stride-1 conv, 1 strided conv on phase planes, 2 fully connected
  int PW, IB;                 // flat grid: row pitch / positions per image
  int rowStride, colStride, chStride;   // mode 1: source element strides of an input row / column / channel
  int nsplit, kAll, kPerSplit;  // mode 2: K splits, k-steps of the layer / per split (partial sums -> fc_reduce)
  int kshift;                   // stored assignment byte = index << kshift
  float* partial;               // mode 2, nsplit > 1: [nsplit][N][dstRow]
  int dstRow;                   // mode 2: floats per destination row
  int nPB;                      // position-plane buffers (2; 3 for mode 2, whose planes arrive by bulk copy)
  const float* xprep;           // mode 2: activations pre-split into the plane image (fc_prep_kernel), [tile][chunk][hi,lo][2KS][NT][4]
  int nChunksAll;               // mode 2: chunks of the whole layer (xprep indexing)
  int cbF4;                     // float4 per codebook slot (K for d % 4 == 0 pieces, K/4 for d == 1 scalars)
  int NT;                     // positions per CTA = wgmma N (128 or 64)
  int corr;                   // 1 (NT = 64): the terms with a low-order operand piece have their own accumulator (added in the epilogue)
  int bf;                     // 1: bf16x2 operands (x = x1 + x2, w = w1 + w2 as bf16 pieces; TWO bf16 MMAs of K = 16 per
                              //    k-step: [w1|w1].[x1|x2] + [w2|w2].[x1|x2]) instead of 3xTF32 (three tf32 MMAs of K = 8)
  const uint8_t* asmtT;       // qcnn_layer::d_asmt_t (mode 0 with idxT)
  int idxT, tapsPad;          // 1: the chunk's indices are staged channel-major ([half][128 channels][tapsPad bytes])
  int bulkC;                  // mode 0 with idxT and cbPre: codebook slices + index blocks arrive by four cp.async.bulk per chunk
  int cbPre;                  // 1: `ctrd` is the pre-split codebook (qcnn_layer::d_ctrd_bf): the decoders convert nothing
  int planeRows;              // 16-byte rows per staged plane (3xTF32: planeF4; bf16x2: positions x k-step groups)
  int NPOS;                   // staged positions per plane (NT + halo)
  int planeF4;                // float4 per staged plane set (one of hi / lo, one buffer)
  int cbSlots, idRows;        // codebook slices / index rows staged per chunk
  int nChunks;
  int GT;                     // k-steps per stage (decoded into registers together, <= 4)
  int nct;                    // channel tiles of 128 channels per group
  int relu;
  // a KStepTable's fields, kept flat: as one nested member they cost the 3xTF32 instantiations 1-2 % of their time
  int ntab;
  int chunkFirst[8], chunkCount[8];
  KStep tab[kMaxKSteps];
};

// ConvPlan::kernel.  The values are the "force_kernel" / QCNN_FORCE_KERNEL numbers of include/qcnn.h (5 is retired).
enum ConvKernel {
  kConvS1 = 0,        // LUT + gather, stride 1, FFMA LUT stage
  kConvRoll = 1,      // LUT + gather, rolling rows (any stride), FFMA LUT stage
  kConvS1Tc = 2,      // as kConvS1 with the 3xTF32 wgmma LUT stage
  kConvRollTc = 3,    // as kConvRoll with the 3xTF32 wgmma LUT stage
  kConvDirect = 4,    // single narrow subspace, codewords evaluated at the point of use
  kPqGemmTc = 6,      // decode-at-use GEMMs on wgmma (pq_gemm_tc.cu)
  kConvWs = 7,        // stride-1 and strided narrow-input layers (bf16x2) as a weight-stationary wgmma GEMM (conv_ws.cu)
  kConvKernelIds = 8
};

// The arguments of conv_ws_kernel (conv_ws.cu), its only reader; declared here so that ConvPlan holds a tiling by value.
// Field order chosen so that conv_ws_kernel's parameter loads and register allocation match those of its GemmArgs form.
struct ConvWsArgs {
  const float* src;
  float* dst;
  const uint4* wimg;          // weight image (qcnn_layer::d_w_ws)
  const float* bias;
  long long srcImg, dstImg;   // elements per source / destination image
  int N, Hi, Wi, Cin, Ho, Wo, Cout, ksz, pad, stride, G, Cg, Kg, KgPad, S, K, d;
  int NC, PW, IB;             // channels per CTA (N of the MMA) / grid row pitch / positions per image
  int rowStride, colStride, chStride;   // source element strides of an input row / column / channel
  int nPB, P, nWB;            // plane buffers (strided: one per phase row) / positions per CTA / weight stage buffers
  int planeRows, NPOS;        // 16-byte rows per plane / staged positions per plane (P + halo)
  int KS, nct, nChunks;       // k-steps per weight stage / channel tiles per group (Kg / NC) / chunks (8 channels or a phase row)
  int relu;
  KStepTable kt;
};

struct ConvPlan {
  int kernel;           // ConvKernel
  int CPT, J;           // LUT + gather kernels: channels per thread / positions per lane (conv_direct: output rows)
  int threads;
  size_t smem;
  std::array<int, 6> key;   // equal keys of one kernel: near-duplicates.  LUT + gather: CPT, J, nct, nstrips, rgroups, R;
                            // pq_gemm_tc: NT, GT, nct, nsplit; conv_ws: P, KS, nct, nWB (unused entries 0)
  ConvArgs a;           // kernels 0-4: geometry + tiling (pointers/N filled at launch)
  GemmArgs g;           // kernel 6 (pq_gemm_tc)
  ConvWsArgs ws;        // kernel 7 (conv_ws)
};

// FcPlan::kernel, in the order the rule of fc_plan.cu tries them: fc_chain.cu, fc_ws.cu, pq_gemm_tc mode 2, LUT + gather
enum FcKernel { kFcChain, kFcWs, kFcMode2, kFcGather, kFcKernelIds };

// An FC layer's family at one batch size and that family's tiling, without device pointers (bound at launch).  Made on
// every call: qcnn_fc_aprx_forward_flat hides d_srcoff for the length of one call.
struct FcPlan {
  int kernel;    // FcKernel
  int nsplit;    // K-split: > 1 = partial sums [nsplit][N][DoutPad] in d_partial, reduced in fixed order (chain: 1)
  struct { int P, NC, KS, nPB, kPerSplit; size_t smem; } ws;   // fc_ws: images, channels per CTA, k-steps per stage and
                                                                 // per split, plane buffers, shared memory
  GemmArgs tc;   // mode 2
  struct { int tn, cpt, sPerSplit; } gather;   // LUT + gather: images per CTA, channels per thread, subspaces per split
};

struct qcnn_layer {
  qcnn_ctx* ctx = nullptr;
  int kind = 0;
  // geometry
  int Cin = 0, Hin = 0, Win = 0, Cout = 0, ksz = 0, pad = 0, stride = 0, grp = 0, S = 0, K = 0, d = 0;
  int Ho = 0, Wo = 0;
  int Din = 0, Dout = 0, DoutPad = 0;
  // FC source permutation (NHWC map) / conv NCHW source
  int src_h = 0, src_w = 0, src_c = 0;
  qcnn::DeviceBuffer d_srcoff;  // FC: int [Din], NCHW-flatten index -> NHWC element offset (empty when the source is flat)
  int src_nchw = 0;
  // device parameters
  qcnn::DeviceBuffer d_ctrd;    // float
  qcnn::DeviceBuffer d_asmt;    // uint8_t
  int asmt_t_mode = 0;    // layout of d_asmt_t: 0 = [grp][S][KgPad][tapsPad] (stride 1), 1 = [grp][stride phase rows][KgPad][rowsPad] (strided, S = 1)
  qcnn::DeviceBuffer d_asmt_t;  // every conv layer: the same indices channel-major (layout: asmt_t_mode; tapsPad = taps rounded up to 16): a
                                // decoder thread (= channel) reads a chunk's taps with one or two 128-bit loads (pq_gemm_tc.cu modes 0-1, conv_ws.cu)
  qcnn::DeviceBuffer d_bias;    // float
  int kshift = 0;       // FC: stored assignment = idx << kshift
  int asmt_bits = 0;    // FC: 0 = d_asmt is the byte table [S][DoutPad]; 4..7 = bit-packed rows of asmt_pitch bytes (packed_asmt.h)
  int asmt_pitch = 0;   // FC: bytes per row of d_asmt (DoutPad for the byte table)
  // plans
  ConvPlan plan{};
  int plan_N = 0;        // batch size the cached plan was made for (0 = none)
  int tuned = 0;         // the plan for plan_N was confirmed by on-device timing
  std::vector<ConvPlan> cands;  // the model's best tilings for plan_N (autotune candidates)
  std::vector<std::pair<int, ConvPlan>> tunedPlans;  // timed winners per batch size
  // FC scratch
  qcnn::DeviceBuffer d_partial;  // float
  qcnn::DeviceBuffer d_flat;     // tensor-core FC path: source pre-split into hi/lo plane images (fc_prep_kernel)
  qcnn::DeviceBuffer d_ctrd_bf;  // present exactly when d % 4 == 0: codebook pre-split into bf16 pieces (pq_gemm_tc.cu, conv_ws.cu, bf16x2 operands): [S][d/4 pieces][K] x {w1 (4 x bf16), w2 (4 x bf16)}: a (subspace, piece) slice is contiguous
  qcnn::DeviceBuffer d_w_ws;     // conv layers conv_ws can take: the decoded weights of every k-step, [grp][k-step][w1, w2][Kg]
                                 // 16-byte rows (conv_ws.cu builds and reads it); a CTA bulk-copies its stages from here
  qcnn::DeviceBuffer d_cpart;    // chain kernel (fc_chain.cu): per-CTA partial sums [sm_count][DoutPad], words double as ready flags
  // tuning overrides (0 = automatic)
  int opt_fc_nsplit = 0;
  int opt_fc_tn = 0;
  int opt_no_tc = 0;         // 1: never use the decode-at-use tensor-core kernels for this layer
  int opt_tc_bf = 0;         // 1: the tensor-core kernels take bf16x2 operands (tensor_core = 2) instead of 3xTF32
  int opt_force_kernel = 0;  // conv: 1 + kernel id the plan is restricted to (0 = none); tests pin the kernel they check
  int opt_no_autotune = 0;   // conv: 1 = keep the cost model's first tiling (no on-device timing)
  int opt_gemm_nt = 0;       // conv: restrict pq_gemm_tc tilings to this many positions per CTA (0 = any)
  int opt_gemm_gt = 0;       // conv: ... to this many k-steps per stage (0 = any)
  int opt_gemm_nsplit = 0;   // conv: ... to this K-split factor (0 = any)
  int opt_gemm_ct = 0;       // conv: restrict conv_ws tilings to this many channels per CTA (0 = any)
  int opt_gemm_wb = 0;       // conv: ... to this many weight stage buffers (0 = any)
                             // (FC with fc_ws: gemm_nt / gemm_gt / gemm_ct / gemm_nsplit restrict the fc_ws tilings)
  int opt_lut_cpt = 0;       // conv: restrict LUT + gather tilings (kernels 0-4) to this ConvPlan::key[0] (CPT) (0 = any)
  int opt_lut_j = 0;         // ... key[1]: positions per lane (conv_direct: output rows per thread)
  int opt_lut_nct = 0;       // ... key[2]: channel tiles per group
  int opt_lut_r = 0;         // ... key[5]: output rows per strip (conv_direct: after its clamp to Ho + (Ho & 1))
  int opt_lut_rgroups = 0;   // ... key[4]: row groups
  int opt_fc_ws = 0;        // FC: 1 = the batched tensor-core path runs as the weight-stationary GEMM (fc_ws.cu) where
                             // it can, instead of pq_gemm_tc mode 2 (the network executor sets it on every FC layer)
};

namespace qcnn {

// conv_plan.cu: the choice among the conv kernel families, their launch and describe()
int PlanConv(qcnn_layer* L, int N);
int DescribeConv(qcnn_layer* L, int N, char* buf, size_t cap);
int LaunchConv(qcnn_layer* L, const float* src, int N, float* dst, int relu, cudaStream_t st);
// Every conv family provides a planner (candidate tilings for batch N, each with its cost in SM-cycles on one scale), a
// launch of a plan and a describe() that writes the plan's text after the family's name (conv_plan.cu adds the name).
using ConvCands = std::vector<std::pair<double, ConvPlan>>;
// conv_aprx.cu: the LUT + gather kernels (ids 0-4)
void PlanLutGather(const qcnn_layer* L, int N, ConvCands* cands);
int LaunchLutGather(qcnn_layer* L, const ConvPlan& p, const float* src, int N, float* dst, int relu, cudaStream_t st);
void DescribeLutGather(const qcnn_layer* L, const ConvPlan& p, int N, char* buf, size_t cap);

// fc_plan.cu: the choice among the FC kernel families (each plans into an FcPlan, launches and describes a plan)
int LaunchFc(qcnn_layer* L, const float* src, int N, float* dst, int relu, cudaStream_t st);
int DescribeFc(qcnn_layer* L, int N, char* buf, size_t cap);
// fc_chain.cu: one persistent launch for a run of consecutive FC layers at batch <= 4 (relu[l]: ReLU after layer l);
// *handled = false when the kernel does not take the layers, or cannot allocate its partial sums inside a stream capture
bool FcChainEligible(qcnn_ctx* ctx, const qcnn_layer* const* layers, const int* relu, int n, int N);
int LaunchFcChain(qcnn_ctx* ctx, qcnn_layer* const* layers, const int* relu, int n, const float* src, int N, float* dst,
                  cudaStream_t st, unsigned long long* dbg, bool* handled);
void DescribeFcChain(const qcnn_layer* L, const FcPlan& p, int N, char* buf, size_t cap);
// fc_ws.cu: the weight-stationary FC GEMM (bf16x2 operands); PlanFcWs fails when the gemm_* pins leave no tiling
int PlanFcWs(const qcnn_layer* L, int N, FcPlan* p);
int LaunchFcWs(qcnn_layer* L, const FcPlan& p, const float* src, int N, float* dst, int relu, cudaStream_t st);
void DescribeFcWs(const qcnn_layer* L, const FcPlan& p, int N, char* buf, size_t cap);
// fc_aprx.cu: pq_gemm_tc mode 2 (false when it does not fit in shared memory), LUT + gather, and the activations of the
// tensor-core families as the plane image [tile][chunk][x1, x2 (3xTF32: hi, lo)][KS][NT] in L->d_flat
bool PlanFcMode2(const qcnn_layer* L, int N, FcPlan* p);
int LaunchFcMode2(qcnn_layer* L, const FcPlan& p, const float* src, int N, float* dst, int relu, cudaStream_t st);
void DescribeFcMode2(const qcnn_layer* L, const FcPlan& p, int N, char* buf, size_t cap);
// LUT + gather: shared memory one CTA stages for K codewords, tn images per CTA and subspaces of d dims, and its limit.
// PlanFcGather takes the widest batch tile that fits and fails when a pinned fc_tn does not; qcnn_fc_layer_create
// refuses (K, d) where not even tn = 1 fits (K = 256: d <= 11).
constexpr size_t kFcGatherSmemMax = 200 * 1024;
size_t FcGatherSmemBytes(int K, int tn, int d);
int PlanFcGather(const qcnn_layer* L, int N, FcPlan* p);
void DescribeFcGather(const qcnn_layer* L, const FcPlan& p, int N, char* buf, size_t cap);
int LaunchFcGather(qcnn_layer* L, const FcPlan& p, const float* src, int N, float* dst, int relu, cudaStream_t st);
int PrepFcPlanes(qcnn_layer* L, const float* src, int N, int NT, int KS, int nChunksAll, bool bf, cudaStream_t st);
int LaunchSplitReduce(qcnn_ctx* ctx, const float* partial, float* dst, int rows, int cols, int colsPad, int nsplit, int relu,
                      cudaStream_t st);

// pq_gemm_tc.cu
void PlanPqGemm(const qcnn_layer* L, int N, ConvCands* cands);
void DescribePqGemm(const qcnn_layer* L, const ConvPlan& p, int N, char* buf, size_t cap);
size_t PqGemmSmemBytes(const GemmArgs& a);
// asmtBits != 0 (mode 2): a.asmt is the bit-packed FC table of packed_asmt.h with rows of asmtPitch bytes
int LaunchPqGemmArgs(qcnn_ctx* ctx, const GemmArgs& a, long long blocks, cudaStream_t st, int asmtBits = 0, int asmtPitch = 0);
int BuildCtrdBf(qcnn_layer* L);   // layer creation: the bf16x2 form of the codebook (d % 4 == 0)
int LaunchPqGemm(qcnn_layer* L, const ConvPlan& p, const float* src, int N, float* dst, int relu, cudaStream_t st);
// A conv layer's geometry and image strides in the argument block of pq_gemm_tc (GemmArgs) or conv_ws (ConvWsArgs).  Set
// at every launch: qcnn_conv_layer_set_src_nchw may change the source strides after planning.
template <class A>
void SetGemmGeometry(const qcnn_layer* L, A& a) {
  a.Hi = L->Hin; a.Wi = L->Win; a.Cin = L->Cin; a.Ho = L->Ho; a.Wo = L->Wo; a.Cout = L->Cout;
  a.ksz = L->ksz; a.pad = L->pad; a.stride = L->stride; a.G = L->grp; a.Cg = L->Cin / L->grp; a.Kg = L->Cout / L->grp;
  a.KgPad = RoundUp(a.Kg, 16); a.S = L->S; a.K = L->K; a.d = L->d;
  a.srcImg = static_cast<long long>(a.Hi) * a.Wi * a.Cin;
  if (L->src_nchw) { a.rowStride = a.Wi; a.colStride = 1; a.chStride = a.Hi * a.Wi; }
  else { a.rowStride = a.Wi * a.Cin; a.colStride = a.Cin; a.chStride = 1; }
  a.dstImg = static_cast<long long>(a.Ho) * a.Wo * a.Cout;
}

// Mode 1 k-step table (strided layer on phase planes of NPOS positions, bf: bf16x2 planes of planeRows rows): for every
// phase row ph, its k-steps in (kh, kw) order, as entries [chunkFirst[ph], + chunkCount[ph]) of t.tab.  Returns the number
// of k-steps (> kMaxKSteps: the table does not fit).  t: a KStepTable (conv_ws) or the same fields of GemmArgs (pq_gemm_tc).
template <class T> int Mode1Table(const qcnn_layer* L, int NPOS, bool bf, int planeRows, T& t) {
  const int st = L->stride, PWp = CeilDiv(L->Win + 2 * L->pad, st);
  int ne = 0;
  for (int ph = 0; ph < st; ph++) {
    t.chunkFirst[ph] = ne;
    for (int kh = ph; kh < L->ksz; kh += st)
      for (int kw = 0; kw < L->ksz; kw += 2, ne++) {
        if (ne >= kMaxKSteps) { ne = kMaxKSteps + 1000; break; }
        KStep& ks = t.tab[ne];
        // partner in the next phase column, same shift (bf16x2: the partner must be the odd column of the same pair)
        const bool paired = kw + 1 < L->ksz && (kw % st) + 1 < st && !(bf && ((kw % st) & 1));
        ks.bStart = (kw % st) * NPOS + (kh / st) * PWp + kw / st;
        // an unpaired tap's second half (zero codebook slot) aliases its first half (LBO = 0): a shift would read
        // the next position -- for a tile's last position, or a tap at the end of an image, another image's
        // pixel -- and 0 * NaN / Inf would carry that image's non-finite values into this one's output
        ks.lbo = paired ? NPOS : 0;
        if (bf) {   // row = (pair of phase columns, position); K-core-matrix 1 = the x2 plane
          ks.bStart = ((kw % st) >> 1) * NPOS + (kh / st) * PWp + kw / st;
          ks.lbo = planeRows;
        }
        ks.idx0 = static_cast<short>((kh - ph) / st * L->ksz + kw);
        ks.idx1 = static_cast<short>(paired ? ks.idx0 + 1 : ks.idx0);
        ks.cb0 = 0; ks.cb1 = paired ? 0 : 1;
        if (!paired && kw + 1 < L->ksz) kw--;   // the partner starts its own k-step
      }
    t.chunkCount[ph] = ne - t.chunkFirst[ph];
  }
  t.ntab = ne;
  return ne;
}

// Mode 0 k-step table (stride-1 layer on the flat padded grid): the taps of a chunk in (kh, kw) order, a tap being a shift
// of the position operand's start by kh * PW + kw rows, K-core-matrix 1 (the chunk's second half / the x2 plane) NPOS rows
// further; index row and codebook slot = (half, tap).  Returns the number of k-steps per chunk.  t: as for Mode1Table.
template <class T> int Mode0Table(const qcnn_layer* L, int PW, int NPOS, T& t) {
  const int taps = L->ksz * L->ksz;
  t.ntab = taps;
  t.chunkFirst[0] = 0; t.chunkCount[0] = taps;
  for (int i = 0; i < taps; i++) {
    KStep& ks = t.tab[i];
    ks.bStart = (i / L->ksz) * PW + (i % L->ksz);
    ks.lbo = NPOS;
    ks.idx0 = static_cast<short>(i); ks.idx1 = static_cast<short>(taps + i);
    ks.cb0 = 0; ks.cb1 = 1;
  }
  return taps;
}

// Raises a kernel's dynamic shared-memory limit to the opt-in maximum once per kernel and device (per launch, the limit
// would follow whichever layer ran last: fragile under graph capture).  A device id past the table is raised every call.
template <auto Kernel>
int OptInSmem(qcnn_ctx* ctx) {
  static bool done[64] = {false};
  const bool inTable = ctx->device >= 0 && ctx->device < 64;
  if (inTable && done[ctx->device]) return 0;
  QCNN_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(SmemOptin(ctx))));
  if (inTable) done[ctx->device] = true;
  return 0;
}

// pq_quantize.cu: K as qcnn_fc_layer_create accepts it (16, 32, 64, 128 or 256), and as qcnn_conv_layer_create accepts
// it (a multiple of 8 in 8..256); each sets the error and returns 1 otherwise
int CheckFcK(const char* who, int K);
int CheckConvK(const char* who, int K);

// pq_refine.cu / pq_refine_conv.cu: a layer's geometry as the error-correcting quantizer reads it (an FC layer of Din
// inputs and Dout outputs is the one-group 1x1 conv on a 1x1 map: Cg = Dg = Din, Cpg = Cout = Dout, T = Ho = Wo = 1),
// and the halves of the quantizer on a qcnn_pq_stats: folding a batch into the statistics, and the sweeps that read them
struct PqGeometry { int Cin, Hin, Win, Cout, ksz, pad, stride, grp, Ho, Wo, Cg, Cpg, T, Dg; };
int FcStatsAdd(qcnn_pq_stats* s, const char* who, const float* y, const float* t, int N, cudaStream_t st);
int ConvStatsAdd(qcnn_pq_stats* s, const char* who, const float* y, const float* t, int N, cudaStream_t st);
// K and the joint-system limit of a conv refine
int CheckConvSystem(const char* who, int K, int d, int Cg);
// The conv sweeps on the sums G, P and |T|^2 (those of s, or their centered copies), from the weights wts in the internal
// dim order (not read by the target form) and the assignments at [S][Cout][T].  bias_h non-NULL: replaced by the refit
// bias.
int SweepConv(qcnn_pq_stats* s, const char* who, bool target, int K, int sweeps, const float* wts, std::vector<uint8_t>& at,
              const double* G, const double* P, const double* TT, float* ctrd_h, uint8_t* asmt_h, float* bias_h,
              double* loss_h, cudaStream_t st);
// The one-shot calls after their own argument checks: check the start, create the statistics (without the first
// moments, which they never read), one add of all N inputs, the sweeps, destroy
int RefineOnce(qcnn_ctx* ctx, const char* who, bool conv, bool target, const PqGeometry& geo, int K, int d, int sweeps,
               const float* w_h, const float* x, const float* t, int N, float* ctrd_h, uint8_t* asmt_h, double* loss_h,
               cudaStream_t st);

// conv_ws.cu: the tensor-core family's weight-stationary tilings of stride-1 layers (mode-0 geometry, channel tiles) and
// of strided narrow-input layers (mode-1 geometry)
void PlanConvWs(const qcnn_layer* L, int N, ConvCands* cands);
int BuildConvWsImage(qcnn_layer* L);   // layer creation, after BuildCtrdBf: d_w_ws for the layers conv_ws can take
int LaunchConvWs(qcnn_layer* L, const ConvPlan& p, const float* src, int N, float* dst, int relu, cudaStream_t st);
void DescribeConvWs(const qcnn_layer* L, const ConvPlan& p, int N, char* buf, size_t cap);

int LaunchRelu(qcnn_ctx* ctx, const float* src, float* dst, size_t n, cudaStream_t st);
int LaunchLrn(qcnn_ctx* ctx, const float* src, float* dst, size_t pixels, int C, int size, float alpha, float beta,
              float k, cudaStream_t st);
int LaunchMaxPool(qcnn_ctx* ctx, const float* src, float* dst, int N, int H, int W, int C, int ksz, int pad,
                  int stride, cudaStream_t st);
int LaunchLrnMaxPool(qcnn_ctx* ctx, const float* src, float* dst, int N, int H, int W, int C, int size, float alpha,
                     float beta, float k, int ksz, int pad, int stride, cudaStream_t st);
int LaunchSoftmax(qcnn_ctx* ctx, const float* src, float* dst, int N, int C, cudaStream_t st);
int LaunchNchwToNhwc(qcnn_ctx* ctx, const float* src, float* dst, int N, int C, int H, int W, cudaStream_t st);
int LaunchNhwcToNchw(qcnn_ctx* ctx, const float* src, float* dst, int N, int H, int W, int C, cudaStream_t st);

// preproc.cu
int LaunchU8ToF32(qcnn_ctx* ctx, const uint8_t* src, const float* mean, float* dst, int N, int C, int HW, cudaStream_t st);
int LaunchTopK(qcnn_ctx* ctx, const float* prob, int N, int C, int k, int mode, int* idx, float* val, cudaStream_t st);

// qcnn_net.cu: a CaffePara layer table as C-ABI records, and the NHWC input dims of every layer of a table (entry
// layerCnt: the output) -- the one shape walk of the executor and of qcnn_pq_quantize_model
struct LayerDims { int H, W, C; };
std::vector<qcnn_layer_info> LayerInfos(const CaffePara& para);
std::vector<LayerDims> LayerInputDims(const std::vector<qcnn_layer_info>& infos, int imgC, int imgH, int imgW);

inline int PoolOut(int in, int pad, int ksz, int stride) {
  // ceil((in + 2p - k) / s) + 1   (reference src/CaffeEva.cc:365-372)
  int num = in + 2 * pad - ksz;
  int q = num >= 0 ? (num + stride - 1) / stride : -((-num) / stride);
  return q + 1;
}
// The windows of a pooling layer are clipped to the map, not padded, so each must hold at least one input pixel: the
// first needs pad < ksz, the last (out - 1) * stride - pad < in.  (An empty window has no defined output: the reference
// leaves it unwritten.)  ksz, stride >= 1.
inline bool PoolWindowsNonEmpty(int in, int pad, int ksz, int stride) {
  const int out = PoolOut(in, pad, ksz, stride);
  return in >= 1 && pad >= 0 && pad < ksz && out >= 1 && (out - 1) * stride - pad < in;
}

}  // namespace qcnn

// The calibration statistics of one PQ layer for one subspace width d (DESIGN.md 4e): the sums over images that the
// error-correcting quantizer reads, in the dim order of its sweeps.  Device buffers are owned; `done` is recorded on the
// stream of the last add, so a refine or a read waits for the queued accumulation.
struct qcnn_pq_stats {
  qcnn_ctx* ctx = nullptr;
  bool conv = false, target = false;   // conv: chooses the add and the sweep loop
  int d = 0;
  qcnn::PqGeometry geo{};
  long long images = 0;
  qcnn::DeviceBuffer G, P, tt;    // G [grp][Dg][Dg] (FC [Din][Din]); target: P [Cout][Dg] (FC [Dout][Din]) and |T|^2
  // first moments (with sums): sy = sum of y [grp][Dg] in the dim order of G (FC [Din]); target: su = sum of t [Cout]
  // (FC [Dout]); conv: plane, an add's fresh sum over its images of y [Hin][Win][Cin] or of t [Ho][Wo][Cout]
  bool sums = true;               // false only inside the one-shot refine calls, which never read the first moments
  qcnn::DeviceBuffer sy, su, plane;
  qcnn::DeviceBuffer scratch;     // the |T_b|^2 partials [kLossBlocks] fp64, then the add's two scan flags
  cudaEvent_t done = nullptr;
  ~qcnn_pq_stats() {
    if (done) cudaEventDestroy(done);
  }
};

#endif  // QCNN_INTERNAL_H_
