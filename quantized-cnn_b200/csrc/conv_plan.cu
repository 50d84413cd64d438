// The choice among the conv kernel families, common to all of them.  Each family plans, launches and describes its own
// tilings (conv_aprx.cu: LUT + gather, pq_gemm_tc.cu: decode-at-use GEMM, conv_ws.cu: weight-stationary GEMM); this
// file picks the candidates, times them on the device and dispatches a plan to its family.
#include "qcnn_internal.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>

namespace qcnn {

namespace {

// Numerical classes, which on-device timing never chooses between: fp32 LUT (or decode, conv_direct), 3xTF32 LUT (~5e-6
// apart), and the tensor-core GEMMs, whose operand format (bf16x2 / 3xTF32) is a layer setting, not a timing result (at
// bf16x2, conv_ws and pq_gemm_tc of one geometry chain the same k-steps and share one error bound: DESIGN.md 2)
enum ConvClass { kFp32Lut, kTf32Lut, kGemm };

struct ConvFamily {
  const char* name;   // describe(): the plan's text starts with it
  ConvClass cls;
  int seats;          // candidates the kernel is guaranteed (when it has that many tilings) before the rest go by cost
  int (*launch)(qcnn_layer* L, const ConvPlan& p, const float* src, int N, float* dst, int relu, cudaStream_t st);
  void (*describe)(const qcnn_layer* L, const ConvPlan& p, int N, char* buf, size_t cap);
};

// one row per ConvKernel id
constexpr ConvFamily kFamilies[kConvKernelIds] = {
    {"conv_s1", kFp32Lut, 2, LaunchLutGather, DescribeLutGather},
    {"conv_roll", kFp32Lut, 2, LaunchLutGather, DescribeLutGather},
    {"conv_s1_tc(wgmma LUT)", kTf32Lut, 2, LaunchLutGather, DescribeLutGather},
    {"conv_roll_tc(wgmma LUT)", kTf32Lut, 2, LaunchLutGather, DescribeLutGather},
    {"conv_direct", kFp32Lut, 8, LaunchLutGather, DescribeLutGather},
    {nullptr, kGemm, 0, nullptr, nullptr},   // 5: retired
    {"pq_gemm_tc", kGemm, 6, LaunchPqGemm, DescribePqGemm},
    {"pq_gemm_tc_ws(weight-stationary wgmma, weights decoded once per layer and bulk-copied into shared memory, bf16x2)", kGemm, 6, LaunchConvWs,
     DescribeConvWs},
};

constexpr size_t kMaxCand = 18;

}  // namespace

// Chooses the tiling of a conv layer for batch size N.  The candidates are the tensor-core GEMM tilings whenever the layer
// allows tensor cores (tensor_core = 1 or 2) and any GEMM family has a tiling; otherwise the LUT + gather tilings,
// restricted to the numerical class of the cheapest; then the pins apply.  The kMaxCand cheapest are kept, every kernel
// first getting its seats, near-duplicates (equal kernel and key) dropped.  cands[0] is the plan when autotuning is off.
int PlanConv(qcnn_layer* L, int N) {
  if (L->plan_N == N) return 0;
  for (const std::pair<int, ConvPlan>& e : L->tunedPlans)  // a batch size seen (and timed) before: reuse its plan
    if (e.first == N) { L->plan = e.second; L->plan_N = N; L->tuned = 1; return 0; }
  ConvCands cands;
  if (!L->opt_no_tc) {
    PlanPqGemm(L, N, &cands);
    PlanConvWs(L, N, &cands);
  }
  if (cands.empty()) PlanLutGather(L, N, &cands);
  QCNN_CHECK(!cands.empty(), "qcnn_conv_layer_create: no tiling fits (Cout/grp=%d must be a multiple of 16; K=%d must be a "
             "multiple of 8; k=%d, W=%d)", L->Cout / L->grp, L->K, L->ksz, L->Win);
  std::stable_sort(cands.begin(), cands.end(), [](const std::pair<double, ConvPlan>& x, const std::pair<double, ConvPlan>& y) { return x.first < y.first; });
  auto keepIf = [&cands](auto pred) {
    cands.erase(std::remove_if(cands.begin(), cands.end(), [&](const std::pair<double, ConvPlan>& c) { return !pred(c.second); }),
                cands.end());
  };
  // layer parameter "force_kernel" / QCNN_FORCE_KERNEL=<0 s1 | 1 roll | 2 s1_tc | 3 roll_tc | 4 direct | 6 pq_gemm_tc |
  // 7 conv_ws> restricts the choice instead of the class (tests pin the kernel they check; fails when that kernel has no
  // tiling).  It goes first: a gemm_* pin that no tiling of the pinned family matches is reported as such.
  const char* force = getenv("QCNN_FORCE_KERNEL");
  if (L->opt_force_kernel || force) {
    const int want = L->opt_force_kernel ? L->opt_force_kernel - 1 : atoi(force);
    const bool any = std::any_of(cands.begin(), cands.end(), [&](const std::pair<double, ConvPlan>& c) { return c.second.kernel == want; });
    QCNN_CHECK(any || !L->opt_force_kernel, "qcnn_conv_aprx_forward: force_kernel=%d has no tiling for this layer at batch %d", want, N);
    if (any) keepIf([&](const ConvPlan& c) { return c.kernel == want; });
  } else {
    const ConvClass want = kFamilies[cands[0].second.kernel].cls;
    keepIf([&](const ConvPlan& c) { return kFamilies[c.kernel].cls == want; });
  }
  // layer parameters "gemm_nt" / "gemm_gt" / "gemm_nsplit": only pq_gemm_tc tilings with that many positions per CTA,
  // k-steps per stage and K-split factor (0 = any); "gemm_nt" and "gemm_gt" also restrict the positions per CTA and the
  // k-steps per weight stage of conv_ws, "gemm_ct" its channels per CTA and "gemm_wb" the depth of its weight ring
  if (L->opt_gemm_nt || L->opt_gemm_gt || L->opt_gemm_nsplit || L->opt_gemm_ct || L->opt_gemm_wb) {
    keepIf([L](const ConvPlan& c) {
      if (c.kernel == kConvWs)
        return (!L->opt_gemm_nt || c.ws.P == L->opt_gemm_nt) && (!L->opt_gemm_gt || c.ws.KS == L->opt_gemm_gt) &&
               (!L->opt_gemm_ct || c.ws.NC == L->opt_gemm_ct) && (!L->opt_gemm_wb || c.ws.nWB == L->opt_gemm_wb);
      const GemmArgs& g = c.g;
      return c.kernel != kPqGemmTc || ((!L->opt_gemm_nt || g.NT == L->opt_gemm_nt) && (!L->opt_gemm_gt || g.GT == L->opt_gemm_gt) &&
                                       (!L->opt_gemm_nsplit || g.nsplit == L->opt_gemm_nsplit));
    });
    QCNN_CHECK(!cands.empty(), "qcnn_conv_aprx_forward: gemm_nt=%d gemm_gt=%d gemm_nsplit=%d gemm_ct=%d gemm_wb=%d has no "
               "tiling for this layer at batch %d", L->opt_gemm_nt, L->opt_gemm_gt, L->opt_gemm_nsplit, L->opt_gemm_ct,
               L->opt_gemm_wb, N);
  }
  // layer parameters "lut_cpt" / "lut_j" / "lut_nct" / "lut_r" / "lut_rgroups": only LUT + gather tilings (kernels 0-4) with
  // that key entry (0 = any): channels per thread, positions per lane (conv_direct: output rows per thread), channel tiles
  // per group, output rows per strip (conv_direct: after its clamp), row groups.  Tests pin the tiling they check.
  if (L->opt_lut_cpt || L->opt_lut_j || L->opt_lut_nct || L->opt_lut_r || L->opt_lut_rgroups) {
    keepIf([L](const ConvPlan& c) {
      if (c.kernel > kConvDirect) return true;
      return (!L->opt_lut_cpt || c.key[0] == L->opt_lut_cpt) && (!L->opt_lut_j || c.key[1] == L->opt_lut_j) &&
             (!L->opt_lut_nct || c.key[2] == L->opt_lut_nct) && (!L->opt_lut_r || c.key[5] == L->opt_lut_r) &&
             (!L->opt_lut_rgroups || c.key[4] == L->opt_lut_rgroups);
    });
    QCNN_CHECK(!cands.empty(), "qcnn_conv_aprx_forward: lut_cpt=%d lut_j=%d lut_nct=%d lut_r=%d lut_rgroups=%d has no tiling "
               "for this layer at batch %d", L->opt_lut_cpt, L->opt_lut_j, L->opt_lut_nct, L->opt_lut_r, L->opt_lut_rgroups, N);
  }
  L->cands.clear();
  for (int pass = 0; pass < 2; pass++) {
    int perKernel[kConvKernelIds] = {};
    for (size_t i = 0; i < cands.size() && L->cands.size() < kMaxCand; i++) {
      const ConvPlan& c = cands[i].second;
      if (pass == 0 && perKernel[c.kernel] >= kFamilies[c.kernel].seats) continue;
      bool dup = false;
      for (const ConvPlan& e : L->cands) dup |= e.kernel == c.kernel && e.key == c.key;
      if (dup) continue;
      L->cands.push_back(c);
      perKernel[c.kernel]++;
    }
  }
  L->plan = L->cands[0];
  L->plan_N = N;
  L->tuned = 0;
  return 0;
}

int LaunchConv(qcnn_layer* L, const float* src, int N, float* dst, int relu, cudaStream_t st) {
  QCNN_CHECK(L->kind == QCNN_KIND_CONV, "qcnn_conv_aprx_forward: layer is not convolutional");
  QCNN_CHECK(N >= 1 && N <= 65535, "qcnn_conv_aprx_forward: N must be in [1, 65535] (got %d)", N);
  if (int prc = PlanConv(L, N)) return prc;
  // empirical choice among the model's best tilings: time each once on this device for this batch size
  static const bool autotune = !(getenv("QCNN_AUTOTUNE") && getenv("QCNN_AUTOTUNE")[0] == '0');
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(st, &cap);
  if (autotune && !L->opt_no_autotune && !L->tuned && L->cands.size() > 1 && cap == cudaStreamCaptureStatusNone) {
    cudaEvent_t e0, e1;
    QCNN_CUDA(cudaEventCreate(&e0));
    if (cudaEventCreate(&e1) != cudaSuccess) { cudaEventDestroy(e0); return CudaFail(cudaGetLastError(), "cudaEventCreate", __FILE__, __LINE__); }
    float bestMs = 1e30f;
    size_t bestI = 0;
    for (size_t i = 0; i < L->cands.size(); i++) {
      const ConvPlan& c = L->cands[i];
      if (kFamilies[c.kernel].launch(L, c, src, N, dst, relu, st)) continue;   // warm-up (also sets the smem attribute)
      // best of two timed samples (a sample = 1 launch at large batches, 3 at small ones): single samples made the choice
      // between near-equal candidates vary from run to run
      const int reps = N >= 64 ? 1 : 3;
      float ms = 1e30f;
      bool ok = true;
      for (int sample = 0; sample < 2 && ok; sample++) {
        if (cudaEventRecord(e0, st) != cudaSuccess) { cudaGetLastError(); ok = false; break; }
        for (int r = 0; r < reps; r++) kFamilies[c.kernel].launch(L, c, src, N, dst, relu, st);
        if (cudaEventRecord(e1, st) != cudaSuccess) { cudaGetLastError(); ok = false; break; }
        if (cudaEventSynchronize(e1) != cudaSuccess) { cudaGetLastError(); ok = false; break; }
        float t = 0.0f;
        cudaEventElapsedTime(&t, e0, e1);
        ms = std::min(ms, t);
      }
      if (!ok) continue;
      static const bool tuneLog = getenv("QCNN_AUTOTUNE_LOG") != nullptr;
      if (tuneLog) {   // (conv_ws: positions per CTA, KS, bf16x2, no K-split, and its weight buffers)
        const bool ws = c.kernel == kConvWs, tc = c.kernel == kPqGemmTc;
        char wsTail[16] = "";
        if (ws) snprintf(wsTail, sizeof(wsTail), " wb=%d", c.ws.nWB);
        fprintf(stderr, "[qcnn autotune] N=%d Cout=%d k=%d cand %zu: kernel=%d NT/CPT=%d GT/J=%d bf=%d nsplit=%d%s smem=%zu -> %.4f ms\n",
                N, L->Cout, L->ksz, i, c.kernel, ws ? c.ws.P : tc ? c.g.NT : c.CPT, ws ? c.ws.KS : tc ? c.g.GT : c.J,
                ws ? 1 : c.g.bf, ws ? 1 : c.g.nsplit, wsTail, c.smem, ms);
      }
      if (ms < bestMs) { bestMs = ms; bestI = i; }
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    L->plan = L->cands[bestI];
    L->tuned = 1;
    L->tunedPlans.emplace_back(N, L->plan);
  }
  const int rc = kFamilies[L->plan.kernel].launch(L, L->plan, src, N, dst, relu, st);
  if (rc == 0) L->ctx->launches++;
  return rc;
}

// human-readable tiling of the plan for batch N (bench / DESIGN bookkeeping)
int DescribeConv(qcnn_layer* L, int N, char* buf, size_t cap) {
  if (int prc = PlanConv(L, N)) return prc;
  const ConvFamily& f = kFamilies[L->plan.kernel];
  const int n = snprintf(buf, cap, "%s", f.name);
  if (n >= 0 && static_cast<size_t>(n) < cap) f.describe(L, L->plan, N, buf + n, cap - n);
  return 0;
}

}  // namespace qcnn
