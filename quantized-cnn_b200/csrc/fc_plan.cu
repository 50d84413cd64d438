// The choice among the FC kernel families, common to all of them.  Each family plans, launches and describes its own
// tiling (fc_chain.cu: the persistent kernel at batch <= 4, fc_ws.cu: weight-stationary GEMM, fc_aprx.cu: pq_gemm_tc
// mode 2 and LUT + gather); this file states the rule that picks one, and the K-split reduction they share.
#include "qcnn_internal.h"

#include <cstdio>
#include <cstdlib>

namespace qcnn {

namespace {

struct FcFamily {
  // runs plan p; with p.nsplit > 1 it writes the partial sums to dst and is given relu = 0 (LaunchFc reduces them)
  int (*launch)(qcnn_layer* L, const FcPlan& p, const float* src, int N, float* dst, int relu, cudaStream_t st);
  // the text describe() writes after " via " (none: the plain LUT + gather kernel)
  void (*describe)(const qcnn_layer* L, const FcPlan& p, int N, char* buf, size_t cap);
};

// one row per FcKernel id.  The chain has no launch here: LaunchFc runs it itself, since it can decline at launch.
constexpr FcFamily kFamilies[kFcKernelIds] = {
    {nullptr, DescribeFcChain},
    {LaunchFcWs, DescribeFcWs},
    {LaunchFcMode2, DescribeFcMode2},
    {LaunchFcGather, nullptr},
};

// The rule: the first family that takes the layer at batch N, in FcKernel order (withChain = false leaves the chain out).
// The tensor-core families need N >= 96 (QCNN_FC_TC=1: any N, QCNN_FC_TC=0: none), tensor cores allowed, no gather-kernel
// pin (fc_nsplit = 1 is the bit-exact reference order) and a geometry their decoders read.
int PlanFc(const qcnn_layer* L, int N, FcPlan* p, bool withChain = true) {
  p->nsplit = 1;
  const int relu0 = 0;   // (the chain takes a layer or not whatever its ReLU)
  if (withChain && FcChainEligible(L->ctx, &L, &relu0, 1, N)) { p->kernel = kFcChain; return 0; }
  static const char* env = getenv("QCNN_FC_TC");
  const bool tc = !(env && env[0] == '0') && (N >= 96 || (env && env[0] == '1')) &&
                  !L->opt_fc_nsplit && !L->opt_fc_tn && !L->opt_no_tc && L->Din % 8 == 0 &&
                  (L->d == 1 || L->d % 4 == 0) && L->S * L->d >= L->Din && L->K <= 256 && L->K % 4 == 0;
  if (tc && L->opt_fc_ws && L->opt_tc_bf && (L->d == 1 || (L->d % 4 == 0 && L->d_ctrd_bf.get()))) {
    p->kernel = kFcWs;
    return PlanFcWs(L, N, p);
  }
  if (tc && PlanFcMode2(L, N, p)) { p->kernel = kFcMode2; return 0; }
  p->kernel = kFcGather;
  return PlanFcGather(L, N, p);
}

}  // namespace

int LaunchFc(qcnn_layer* L, const float* src, int N, float* dst, int relu, cudaStream_t st) {
  QCNN_CHECK(L->kind == QCNN_KIND_FC, "qcnn_fc_aprx_forward: layer is not fully-connected");
  QCNN_CHECK(N >= 1, "qcnn_fc_aprx_forward: N must be >= 1");
  FcPlan p;
  if (int rc = PlanFc(L, N, &p)) return rc;
  if (p.kernel == kFcChain) {
    bool handled = false;
    if (int rc = LaunchFcChain(L->ctx, &L, &relu, 1, src, N, dst, st, nullptr, &handled)) return rc;
    if (handled) return 0;
    // d_cpart cannot grow inside a stream capture: this call runs what the rule gives without the chain
    if (int rc = PlanFc(L, N, &p, false)) return rc;
  }
  float* out = dst;
  if (p.nsplit > 1) {
    QCNN_CUDA(L->d_partial.Reserve(L->ctx, sizeof(float) * static_cast<size_t>(p.nsplit) * N * L->DoutPad, st));
    out = L->d_partial.as<float>();
  }
  if (int rc = kFamilies[p.kernel].launch(L, p, src, N, out, p.nsplit > 1 ? 0 : relu, st)) return rc;
  L->ctx->launches++;
  if (p.nsplit > 1) return LaunchSplitReduce(L->ctx, out, dst, N, L->Dout, L->DoutPad, p.nsplit, relu, st);
  return 0;
}

// "fc_aprx Din=... [via <family's text> | gather(<tiling>)][ asmt=<b>bit]" for batch N (bench / DESIGN bookkeeping)
int DescribeFc(qcnn_layer* L, int N, char* buf, size_t cap) {
  FcPlan p;
  if (int rc = PlanFc(L, N, &p)) return rc;
  char via[256] = "", gather[96] = "", packed[16] = "";
  if (kFamilies[p.kernel].describe) kFamilies[p.kernel].describe(L, p, N, via, sizeof(via));
  if (p.kernel == kFcGather) DescribeFcGather(L, p, N, gather, sizeof(gather));
  if (L->asmt_bits) snprintf(packed, sizeof(packed), " asmt=%dbit", L->asmt_bits);
  snprintf(buf, cap, "fc_aprx Din=%d Dout=%d S=%d K=%d d=%d%s%s%s%s%s", L->Din, L->Dout, L->S, L->K, L->d, via[0] ? " via " : "",
           via, gather[0] ? " " : "", gather, packed);
  return 0;
}

}  // namespace qcnn
