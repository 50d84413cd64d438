// Error-correcting product quantization of FC layers on the device: block coordinate descent on the codebook and the
// assignments so that the layer's response W x is kept on given inputs (the paper's quantization with error correction).
// Semantics, normative (DESIGN.md 4e):
//   G = X^T X (fp64, fixed order), E = W - W^ (fp64), loss = sum_o E_o^T G E_o = sum_n |(W - W^) x_n|^2.
//   A sweep visits subspaces m = 0..S-1 in order (Gauss-Seidel); a subspace with !(tr(G_mm) > 0) is skipped.
//   h_o = [G E_o]_m + G_mm w^_o(m); H_k = sum_{a_o = k} h_o (fixed order), n_k = |{o : a_o = k}|.
//   codebook   D = (G_mm + lambda I)^-1 H_k / n_k by the Cholesky factor, lambda = 1e-10 tr(G_mm) / w_m, rounded to fp32;
//              D replaces c_k only if f(D) < f(c_k), f(D) = n_k D^T G_mm D - 2 D^T H_k; empty clusters keep their codeword.
//   assign     a_o = argmin_k c_k^T G_mm c_k - 2 c_k^T h_o (fp64, new codewords), the lowest index wins ties.
// Target form (qcnn_pq_refine_fc_target): inputs y, targets t [N][Dout], P = T^T Y (fp64), and
//   loss = sum_n |t_n - W^ y_n|^2 = |T|^2 - 2 sum_o w^_o^T P_o + sum_o w^_o^T G w^_o; the sweep is the same with
//   G E_o replaced by R_o = P_o - G w^_o.  It runs on the same kernels: E = -W^ (the residual against zero weights) and
//   the initial GE = P + E G, after which every update of E and GE is the same-input one.
// No floating-point atomics: two calls return identical bits.
//
// Cost structure: G, the initial G E^T and the update of G E^T after every block of subspaces are fp64 tensor-core GEMMs
// (DMMA m16n8k16).  Inside a block, every per-subspace step runs in one cooperative launch with two grid-wide barriers
// per subspace (codebook step, then assignment step); a CTA owns a fixed set of outputs for the whole block, so the
// per-output work needs no grid barrier.
#include <cooperative_groups.h>
#include <math.h>

#include <algorithm>
#include <memory>
#include <vector>

#include "pq_refine_common.cuh"
#include "qcnn_internal.h"

using namespace qcnn;
namespace cg = cooperative_groups;

namespace {

constexpr int kBlockDims = 256;      // dims per block of subspaces (a multiple of d): the K of the trailing GEMM

// Per subspace m (blockIdx.x): the lower-triangular inverse of the Cholesky factor of G_mm + lambda I, [w][w] at row
// pitch d.  G does not change between sweeps, so this runs once per call.  Skipped subspaces (!(tr(G_mm) > 0)) get none.
__global__ void __launch_bounds__(kSweepThreads) pqr_chol_kernel(const double* __restrict__ G, double* __restrict__ Linv, int Din,
                                                                 int d) {
  extern __shared__ double chol_sm[];
  const int m = blockIdx.x, c0 = m * d, w = min(d, Din - c0), ld = w + 1, tid = threadIdx.x;
  double* L = chol_sm;            // [w][w + 1]
  double* Li = chol_sm + w * ld;  // [w][w + 1]
  double tr = 0.0;
  for (int j = 0; j < w; j++) tr += G[static_cast<size_t>(c0 + j) * (Din + 1)];
  if (!(tr > 0.0)) return;   // also a centered G's rounding-level negative or NaN trace
  const double lam = 1e-10 * tr / w;
  for (int e = tid; e < w * w; e += blockDim.x) {
    const int i = e / w, j = e % w;
    L[i * ld + j] = G[static_cast<size_t>(c0 + i) * Din + c0 + j] + (i == j ? lam : 0.0);
  }
  __syncthreads();
  for (int k = 0; k < w; k++) {   // right-looking Cholesky, lower triangle
    if (tid == 0) L[k * ld + k] = sqrt(L[k * ld + k]);
    __syncthreads();
    for (int i = k + 1 + tid; i < w; i += blockDim.x) L[i * ld + k] /= L[k * ld + k];
    __syncthreads();
    const int r = w - k - 1;
    for (int e = tid; e < r * r; e += blockDim.x) {
      const int i = k + 1 + e / r, j = k + 1 + e % r;
      if (j <= i) L[i * ld + j] -= L[i * ld + k] * L[j * ld + k];
    }
    __syncthreads();
  }
  if (tid < w) {   // column c of L^-1 by forward substitution
    const int c = tid;
    Li[c * ld + c] = 1.0 / L[c * ld + c];
    for (int i = c + 1; i < w; i++) {
      double s = 0.0;
      for (int k = c; k < i; k++) s += L[i * ld + k] * Li[k * ld + c];
      Li[i * ld + c] = -s / L[i * ld + i];
    }
  }
  __syncthreads();
  for (int e = tid; e < w * w; e += blockDim.x) {
    const int i = e / w, j = e % w;
    Linv[(static_cast<size_t>(m) * d + i) * d + j] = j <= i ? Li[i * ld + j] : 0.0;
  }
}

struct BlockArgs {
  const double* G;        // [Din][Din]
  const double* GE;       // [Dout][Din], as of the start of the block
  const double* Linv;     // [S][d][d]
  double* E;              // [Dout][Din]
  double* dlt;            // [Dout][ld]: per block dim, the change of E (the old decoded weight while its subspace runs)
  double* h;              // [Dout][d]
  double* cconst;         // [K]: c_k^T G_mm c_k of the current subspace
  float* C;               // [S][K][d]
  uint8_t* A;             // [S][Dout]
  int Din, Dout, K, d, ld, m0, m1;
};

// Subspaces [m0, m1) of one sweep, dims [blk0 = m0 d, ...).  GE is not written: the block's own earlier changes enter
// h through dlt, and the trailing GEMM brings GE up to date afterwards.
__global__ void __launch_bounds__(kSweepThreads) pqr_block_kernel(BlockArgs p) {
  cg::grid_group grid = cg::this_grid();
  extern __shared__ float4 blk_sm[];   // assignment step: Cs [K][w] fp32, then cs [K] fp64
  __shared__ double sPart[kSweepThreads], sH[kMaxD], sY[kMaxD], sD[kMaxD], sCu[kMaxD], sRed[kMaxD];
  __shared__ int sCnt[kSweepThreads], sN, sAcc;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int Din = p.Din, Dout = p.Dout, K = p.K, d = p.d, ld = p.ld, blk0 = p.m0 * d;
  const int R = (Dout + gridDim.x - 1) / gridDim.x, r0 = min(Dout, static_cast<int>(blockIdx.x) * R), r1 = min(Dout, r0 + R);
  for (size_t e = tid; e < static_cast<size_t>(r1 - r0) * ld; e += kSweepThreads) p.dlt[static_cast<size_t>(r0) * ld + e] = 0.0;
  __syncthreads();
  for (int m = p.m0; m < p.m1; m++) {
    const int c0 = m * d, w = min(d, Din - c0), cb = c0 - blk0;
    double tr = 0.0;
    for (int j = 0; j < w; j++) tr += p.G[static_cast<size_t>(c0 + j) * (Din + 1)];
    if (!(tr > 0.0)) continue;   // no input energy: codebook and assignments stay
    const uint8_t* Am = p.A + static_cast<size_t>(m) * Dout;
    const float* Cm = p.C + static_cast<size_t>(m) * K * d;
    // (1) h_o = GE_o[c0 + j] + sum_{c in block, c < c0} dlt_o[c] G[c0 + j][c] + sum_i G[c0 + j][c0 + i] w^_o[i]:
    // eight lanes per (output, dim), each over every eighth dim, combined by a fixed shuffle tree
    const int items = (r1 - r0) * w;
    for (int base = 0; base < items * 8; base += kSweepThreads) {
      const int it = base + tid, item = it >> 3, sub = it & 7;
      const bool ok = item < items;
      double acc = 0.0, wold = 0.0;
      int o = 0, j = 0;
      if (ok) {
        o = r0 + item / w;
        j = item % w;
        const double* grow = p.G + static_cast<size_t>(c0 + j) * Din + blk0;
        const double* drow = p.dlt + static_cast<size_t>(o) * ld;
        for (int c = sub; c < cb; c += 8) acc += drow[c] * grow[c];
        const float* cw = Cm + static_cast<size_t>(Am[o]) * d;
        for (int i = sub; i < w; i += 8) acc += static_cast<double>(cw[i]) * grow[cb + i];
        wold = static_cast<double>(cw[j]);
      }
      acc += __shfl_xor_sync(0xffffffffu, acc, 4);
      acc += __shfl_xor_sync(0xffffffffu, acc, 2);
      acc += __shfl_xor_sync(0xffffffffu, acc, 1);
      if (ok && sub == 0) p.h[static_cast<size_t>(o) * d + j] = p.GE[static_cast<size_t>(o) * Din + c0 + j] + acc;
      if (ok && sub == 1) p.dlt[static_cast<size_t>(o) * ld + cb + j] = wold;   // read by step (3); lanes above read c < cb
    }
    grid.sync();
    // (2) codebook: cluster k per CTA.  H_k: nseg contiguous runs of outputs, each summed in ascending o, the runs
    // combined in ascending order.
    const int nseg = kSweepThreads / w;
    for (int k = blockIdx.x; k < K; k += gridDim.x) {
      if (tid < nseg * w) {
        const int j = tid % w, seg = tid / w;
        const int o0 = static_cast<int>(static_cast<long long>(Dout) * seg / nseg);
        const int o1 = static_cast<int>(static_cast<long long>(Dout) * (seg + 1) / nseg);
        double s = 0.0;
        int n = 0;
        for (int o = o0; o < o1; o++)
          if (__ldcg(Am + o) == k) {
            s += __ldcg(p.h + static_cast<size_t>(o) * d + j);
            n++;
          }
        sPart[tid] = s;
        if (j == 0) sCnt[seg] = n;
      }
      __syncthreads();
      float* ck = p.C + (static_cast<size_t>(m) * K + k) * d;
      if (tid < w) {
        double s = 0.0;
        for (int seg = 0; seg < nseg; seg++) s += sPart[seg * w + tid];
        sH[tid] = s;
        sCu[tid] = static_cast<double>(ck[tid]);
      }
      if (tid == 0) {
        int n = 0;
        for (int seg = 0; seg < nseg; seg++) n += sCnt[seg];
        sN = n;
      }
      __syncthreads();
      const int n = sN;
      const double* Gmm = p.G + static_cast<size_t>(c0) * Din + c0;
      if (n > 0) {
        const double* Lm = p.Linv + static_cast<size_t>(m) * d * d;
        if (tid < w) {   // y = L^-1 H / n
          double s = 0.0;
          for (int j = 0; j <= tid; j++) s += Lm[tid * d + j] * (sH[j] / n);
          sY[tid] = s;
        }
        __syncthreads();
        if (tid < w) {   // D = L^-T y, rounded to fp32
          double s = 0.0;
          for (int j = tid; j < w; j++) s += Lm[j * d + tid] * sY[j];
          sD[tid] = static_cast<double>(static_cast<float>(s));
        }
        __syncthreads();
        if (tid < w) {   // f(D) - f(c) = (D - c)^T (n G_mm (D + c) - 2 H), without the cancellation of two f values
          double s = 0.0;
          for (int j = 0; j < w; j++) s += Gmm[static_cast<size_t>(tid) * Din + j] * (sD[j] + sCu[j]);
          sRed[tid] = (sD[tid] - sCu[tid]) * (static_cast<double>(n) * s - 2.0 * sH[tid]);
        }
        __syncthreads();
        if (tid == 0) {
          double s = 0.0;
          for (int j = 0; j < w; j++) s += sRed[j];
          sAcc = s < 0.0;
        }
        __syncthreads();
        if (sAcc && tid < w) {
          ck[tid] = static_cast<float>(sD[tid]);
          sCu[tid] = sD[tid];
        }
        __syncthreads();
      }
      if (tid < w) {
        double s = 0.0;
        for (int j = 0; j < w; j++) s += Gmm[static_cast<size_t>(tid) * Din + j] * sCu[j];
        sRed[tid] = sCu[tid] * s;
      }
      __syncthreads();
      if (tid == 0) {
        double s = 0.0;
        for (int j = 0; j < w; j++) s += sRed[j];
        p.cconst[k] = s;
      }
      __syncthreads();
    }
    grid.sync();
    // (3) assignment, one warp per output; then E and dlt of the subspace's dims
    float* Cs = reinterpret_cast<float*>(blk_sm);
    double* cs = reinterpret_cast<double*>(blk_sm) + (K * w + 1) / 2;
    for (int e = tid; e < K * w; e += kSweepThreads) Cs[e] = __ldcg(Cm + static_cast<size_t>(e / w) * d + e % w);
    for (int k = tid; k < K; k += kSweepThreads) cs[k] = __ldcg(p.cconst + k);
    __syncthreads();
    for (int o = r0 + warp; o < r1; o += kSweepThreads / 32) {
      const double* ho = p.h + static_cast<size_t>(o) * d;
      double best = INFINITY;
      int bi = K;
      for (int k = lane; k < K; k += 32) {
        double dot = 0.0;
        for (int j = 0; j < w; j++) dot += static_cast<double>(Cs[k * w + j]) * ho[j];
        const double v = cs[k] - 2.0 * dot;
        if (v < best) { best = v; bi = k; }
      }
      for (int off = 16; off > 0; off >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, off);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
        if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
      }
      if (lane == 0) p.A[static_cast<size_t>(m) * Dout + o] = static_cast<uint8_t>(bi);
      for (int j = lane; j < w; j += 32) {
        double* dp = p.dlt + static_cast<size_t>(o) * ld + cb + j;
        const double dE = *dp - static_cast<double>(Cs[bi * w + j]);   // E changes by w^_old - w^_new
        *dp = dE;
        p.E[static_cast<size_t>(o) * Din + c0 + j] += dE;
      }
    }
    __syncthreads();
  }
}

// The FC sweeps (arguments as SweepConv's): the inverse Cholesky factors of every subspace once, then per block of
// subspaces the cooperative block kernel and the trailing GEMM
int SweepFc(qcnn_pq_stats* s, const char* who, bool target, int K, int sweeps, const float* wts, std::vector<uint8_t>& at,
            const double* G, const double* P, const double* TT, float* ctrd_h, uint8_t* asmt_h, float* bias_h, double* loss_h,
            cudaStream_t st) {
  qcnn_ctx* ctx = s->ctx;
  const int Din = s->geo.Dg, Dout = s->geo.Cout, d = s->d, S = CeilDiv(Din, d);
  QCNN_ON_DEVICE(ctx->device);
  SweepState ss;
  if (int rc = BeginSweeps(&ss, s, who, target, K, sweeps, wts, at, ctrd_h, G, P, TT, st)) return rc;
  const int spb = std::max(1, kBlockDims / d), ld = spb * d;
  DeviceBuffer dL, dDlt, dH, dCc;
  if (Reserve(ctx, who, dL, sizeof(double) * static_cast<size_t>(S) * d * d, "the Cholesky factors") ||
      Reserve(ctx, who, dDlt, sizeof(double) * Dout * static_cast<size_t>(ld), "the block's changes") ||
      Reserve(ctx, who, dH, sizeof(double) * Dout * static_cast<size_t>(d), "the subspace responses") ||
      Reserve(ctx, who, dCc, sizeof(double) * K, "the codeword norms"))
    return 1;
  const size_t cholSmem = sizeof(double) * 2 * std::min(d, Din) * (std::min(d, Din) + 1);
  if (int rc = OptInSmem<pqr_chol_kernel>(ctx)) return rc;
  pqr_chol_kernel<<<S, kSweepThreads, cholSmem, st>>>(G, dL.as<double>(), Din, d);
  QCNN_CUDA(cudaGetLastError());
  if (sweeps > 0) {
    const size_t blkSmem = sizeof(float) * K * std::min(d, Din) + sizeof(double) * (K + 1);
    cudaFuncAttributes fa;   // the opt-in limit covers static plus dynamic shared memory
    QCNN_CUDA(cudaFuncGetAttributes(&fa, pqr_block_kernel));
    QCNN_CUDA(cudaFuncSetAttribute(pqr_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   static_cast<int>(SmemOptin(ctx) - fa.sharedSizeBytes)));
    int perSm = 0;
    QCNN_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, pqr_block_kernel, kSweepThreads, blkSmem));
    QCNN_CHECK(perSm >= 1, "%s: the sweep kernel does not fit on an SM", who);
    const int grid = std::min(std::min(perSm, 2) * ctx->sm_count, std::max(Dout, K));
    const dim3 gemmGrid(CeilDiv(Din, kTile), CeilDiv(Dout, kTile));
    BlockArgs a{G, ss.GE.as<double>(), dL.as<double>(), ss.E.as<double>(), dDlt.as<double>(), dH.as<double>(),
                dCc.as<double>(), ss.C.as<float>(), ss.A.as<uint8_t>(), Din, Dout, K, d, ld, 0, 0};
    for (int sw = 1; sw <= sweeps; sw++) {
      for (int m0 = 0; m0 < S; m0 += spb) {
        a.m0 = m0;
        a.m1 = std::min(S, m0 + spb);
        void* args[] = {&a};
        QCNN_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(pqr_block_kernel), grid, kSweepThreads, args, blkSmem, st));
        // GE += dlt G[block dims][:]
        const int blk0 = m0 * d, bw = std::min(Din, a.m1 * d) - blk0;
        pqr_gemm_kernel<kGemmF64><<<gemmGrid, kGemmThreads, 0, st>>>(dDlt.get(), ld, G + static_cast<size_t>(blk0) * Din, Din,
                                                                  ss.GE.as<double>(), Din, Dout, Din, bw, 1);
        QCNN_CUDA(cudaGetLastError());
      }
      if (int rc = ss.Loss(sw, st)) return rc;
    }
  }
  return EndSweeps(ss, ctrd_h, asmt_h, bias_h, loss_h, st);
}

// An FC layer of Din inputs and Dout outputs as its 1x1 conv geometry
PqGeometry FcGeometry(int Din, int Dout) { return PqGeometry{Din, 1, 1, Dout, 1, 0, 1, 1, 1, 1, Din, Dout, 1, Din}; }

// The one-shot FC calls' argument checks, in the order of their messages
int Refine(qcnn_ctx* ctx, bool target, int Din, int Dout, int K, int d, int sweeps, const float* w_h, const float* x, const float* t,
           int N, float* ctrd_h, uint8_t* asmt_h, double* loss_h, cudaStream_t st) {
  const char* who = target ? "qcnn_pq_refine_fc_target" : "qcnn_pq_refine_fc";
  QCNN_CHECK(ctx && (target || w_h) && ctrd_h && asmt_h, "%s: NULL argument", who);
  QCNN_CHECK(Din >= 1 && Dout >= 1, "%s: bad dimensions", who);
  if (int rc = CheckFcK(who, K)) return rc;
  QCNN_CHECK(d >= 1 && d <= kMaxD, "%s: d=%d is outside 1..%d", who, d, kMaxD);
  QCNN_CHECK(sweeps >= 0, "%s: sweeps=%d is negative", who, sweeps);
  QCNN_CHECK(N >= 1, "%s: N=%d: at least one input is needed", who, N);
  QCNN_CHECK(x, "%s: NULL argument", who);
  QCNN_CHECK(!target || t, "%s: NULL t", who);
  return RefineOnce(ctx, who, false, target, FcGeometry(Din, Dout), K, d, sweeps, w_h, x, t, N, ctrd_h, asmt_h, loss_h, st);
}

// The sweeps of s's kind on its sums, or with bias_h on their centered copies and followed by the bias refit; with
// damp > 0 on the damped copies of those (damp = 0: on them as they are)
int Sweep(qcnn_pq_stats* s, const char* who, bool target, int K, int sweeps, Start& start, double damp, float* ctrd_h,
          uint8_t* asmt_h, float* bias_h, double* loss_h, cudaStream_t st) {
  const double *G = s->G.as<double>(), *P = s->P.as<double>(), *TT = s->tt.as<double>();
  CenteredSums c;
  if (bias_h) {
    if (int rc = CenterSums(s, who, target, &c, st)) return rc;
    G = c.G.as<double>();
    P = c.P.as<double>();
    TT = c.tt.as<double>();
  }
  if (damp > 0.0) {
    if (int rc = DampSums(s, who, target, damp, start.w, G, P, TT, &c, st)) return rc;
    G = c.G.as<double>();
    P = c.P.as<double>();
    TT = c.tt.as<double>();
  }
  return (s->conv ? SweepConv : SweepFc)(s, who, target, K, sweeps, start.w, start.at, G, P, TT, ctrd_h, asmt_h, bias_h, loss_h,
                                         st);
}

}  // namespace

namespace qcnn {

// An FC add: the scan (its message names the first input column holding a NaN or Inf), then one fold of the sums
// (G, then s; for a target |T|^2, P, then u)
int FcStatsAdd(qcnn_pq_stats* s, const char* who, const float* y, const float* t, int N, cudaStream_t st) {
  const int Din = s->geo.Cin, Dout = s->geo.Cout;
  unsigned first[2];
  if (int rc = ScanAdd(s, y, static_cast<size_t>(N) * Din, Din, t, static_cast<size_t>(N) * Dout, first, st)) return rc;
  QCNN_CHECK(first[0] == kNoneFound, "%s: %s contains a non-finite value (input column %u)", who, s->target ? "y" : "x", first[0]);
  QCNN_CHECK(first[1] == kNoneFound, "%s: t contains a non-finite value", who);
  QCNN_ON_DEVICE(s->ctx->device);
  const int acc = s->images > 0, tiles = CeilDiv(Din, kTile);
  pqr_gemm_kernel<kGemmGram><<<tiles * (tiles + 1) / 2, kGemmThreads, 0, st>>>(y, Din, nullptr, 0, s->G.as<double>(), Din, Din, Din, N,
                                                                              acc);
  QCNN_CUDA(cudaGetLastError());
  if (s->sums && LaunchColSum(s->ctx, y, N, Din, s->sy.as<double>(), acc, st)) return 1;
  if (s->target) {   // |T|^2 and P = T^T Y
    if (int rc = LaunchSqNorm(t, static_cast<size_t>(N) * Dout, s->scratch.as<double>(), s->tt.as<double>(), acc, st)) return rc;
    pqr_gemm_kernel<kGemmCross><<<dim3(tiles, CeilDiv(Dout, kTile)), kGemmThreads, 0, st>>>(t, Dout, y, Din, s->P.as<double>(), Din,
                                                                                         Dout, Din, N, acc);
    QCNN_CUDA(cudaGetLastError());
    if (s->sums && LaunchColSum(s->ctx, t, N, Dout, s->su.as<double>(), acc, st)) return 1;
  }
  QCNN_CUDA(cudaEventRecord(s->done, st));
  s->images += N;
  return 0;
}

int RefineOnce(qcnn_ctx* ctx, const char* who, bool conv, bool target, const PqGeometry& geo, int K, int d, int sweeps,
               const float* w_h, const float* x, const float* t, int N, float* ctrd_h, uint8_t* asmt_h, double* loss_h,
               cudaStream_t st) {
  Start start;
  if (int rc = CheckStart(who, conv, geo, K, d, w_h, ctrd_h, asmt_h, &start)) return rc;
  qcnn_pq_stats* sp = nullptr;
  if (int rc = CreateStats(ctx, who, conv, geo, d, target, false, &sp)) return rc;
  std::unique_ptr<qcnn_pq_stats> s(sp);
  if (int rc = conv ? ConvStatsAdd(s.get(), who, x, t, N, st) : FcStatsAdd(s.get(), who, x, t, N, st)) return rc;
  return Sweep(s.get(), who, target, K, sweeps, start, 0.0, ctrd_h, asmt_h, nullptr, loss_h, st);
}

}  // namespace qcnn

extern "C" int qcnn_pq_refine_fc(qcnn_ctx* ctx, int Din, int Dout, int K, int d, int sweeps, const float* wei_h, const float* x,
                                 int N, float* ctrd_h, uint8_t* asmt_h, double* loss_h, void* stream) {
  return Refine(ctx, false, Din, Dout, K, d, sweeps, wei_h, x, nullptr, N, ctrd_h, asmt_h, loss_h, static_cast<cudaStream_t>(stream));
}

extern "C" int qcnn_pq_refine_fc_target(qcnn_ctx* ctx, int Din, int Dout, int K, int d, int sweeps, const float* y, const float* t,
                                        int N, float* ctrd_h, uint8_t* asmt_h, double* loss_h, void* stream) {
  return Refine(ctx, true, Din, Dout, K, d, sweeps, nullptr, y, t, N, ctrd_h, asmt_h, loss_h, static_cast<cudaStream_t>(stream));
}

// ---- the statistics objects (both kinds; the conv creation and the conv halves are in pq_refine_conv.cu)

extern "C" int qcnn_pq_stats_create_fc(qcnn_ctx* ctx, int Din, int Dout, int d, int target, qcnn_pq_stats** out) {
  const char* who = "qcnn_pq_stats_create_fc";
  QCNN_CHECK(ctx && out, "%s: NULL argument", who);
  *out = nullptr;
  QCNN_CHECK(Din >= 1 && Dout >= 1, "%s: bad dimensions", who);
  QCNN_CHECK(d >= 1 && d <= kMaxD, "%s: d=%d is outside 1..%d", who, d, kMaxD);
  return CreateStats(ctx, who, false, FcGeometry(Din, Dout), d, target != 0, true, out);
}

extern "C" int qcnn_pq_stats_add(qcnn_pq_stats* s, const float* y, const float* t, int N, void* stream) {
  const char* who = "qcnn_pq_stats_add";
  QCNN_CHECK(s, "%s: NULL argument", who);
  QCNN_CHECK(N >= 1, "%s: N=%d: at least one input is needed", who, N);
  QCNN_CHECK(y, "%s: NULL argument", who);
  QCNN_CHECK(s->target || !t, "%s: t given to statistics created without a target", who);
  QCNN_CHECK(!s->target || t, "%s: NULL t (the statistics were created with a target)", who);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  return s->conv ? ConvStatsAdd(s, who, y, t, N, st) : FcStatsAdd(s, who, y, t, N, st);
}

extern "C" int qcnn_pq_stats_count(const qcnn_pq_stats* s, long long* images) {
  QCNN_CHECK(s && images, "qcnn_pq_stats_count: NULL argument");
  *images = s->images;
  return 0;
}

extern "C" int qcnn_pq_stats_read_h(const qcnn_pq_stats* s, double* G_h, double* P_h, double* tt_h) {
  const char* who = "qcnn_pq_stats_read_h";
  QCNN_CHECK(s, "%s: NULL argument", who);
  QCNN_CHECK(s->target || (!P_h && !tt_h), "%s: P and |T|^2 are kept only by statistics created with a target", who);
  QCNN_ON_DEVICE(s->ctx->device);
  QCNN_CUDA(cudaEventSynchronize(s->done));
  if (G_h) QCNN_CUDA(cudaMemcpy(G_h, s->G.get(), s->G.bytes(), cudaMemcpyDeviceToHost));
  if (P_h) QCNN_CUDA(cudaMemcpy(P_h, s->P.get(), s->P.bytes(), cudaMemcpyDeviceToHost));
  if (tt_h) QCNN_CUDA(cudaMemcpy(tt_h, s->tt.get(), sizeof(double), cudaMemcpyDeviceToHost));
  return 0;
}

extern "C" int qcnn_pq_stats_read_sums_h(const qcnn_pq_stats* s, double* s_h, double* u_h, long long* n_h) {
  const char* who = "qcnn_pq_stats_read_sums_h";
  QCNN_CHECK(s, "%s: NULL argument", who);
  QCNN_CHECK(s->target || !u_h, "%s: the targets' sum is kept only by statistics created with a target", who);
  QCNN_ON_DEVICE(s->ctx->device);
  QCNN_CUDA(cudaEventSynchronize(s->done));
  if (s_h) QCNN_CUDA(cudaMemcpy(s_h, s->sy.get(), s->sy.bytes(), cudaMemcpyDeviceToHost));
  if (u_h) QCNN_CUDA(cudaMemcpy(u_h, s->su.get(), s->su.bytes(), cudaMemcpyDeviceToHost));
  if (n_h) *n_h = StatsRows(s);
  return 0;
}

namespace {

// bias: the bias calls, which also need bias_h (finite, [Cout]); without it the sweeps run on the raw sums.  damped: the
// damped call, which needs the weights in both forms and a finite damp >= 0 (the others pass damp = 0).
int RefineStats(qcnn_pq_stats* s, const char* who, bool target, bool bias, bool damped, double damp, int K, int sweeps,
                const float* wei_h, float* ctrd_h, uint8_t* asmt_h, float* bias_h, double* loss_h, void* stream) {
  QCNN_CHECK(s && ((target && !damped) || wei_h) && ctrd_h && asmt_h && (!bias || bias_h), "%s: NULL argument", who);
  QCNN_CHECK(!target || s->target, "%s: the statistics were created without a target", who);
  QCNN_CHECK(s->images > 0, "%s: no calibration data has been added", who);
  QCNN_CHECK(sweeps >= 0, "%s: sweeps=%d is negative", who, sweeps);
  if (damped) QCNN_CHECK(isfinite(damp) && damp >= 0.0, "%s: damp=%g is not a finite number >= 0", who, damp);
  if (bias) QCNN_CHECK(AllFinite(bias_h, s->geo.Cout), "%s: the bias contains a non-finite value", who);
  if (int rc = s->conv ? CheckConvSystem(who, K, s->d, s->geo.Cg) : CheckFcK(who, K)) return rc;
  Start start;
  if (int rc = CheckStart(who, s->conv, s->geo, K, s->d, wei_h, ctrd_h, asmt_h, &start)) return rc;
  return Sweep(s, who, target, K, sweeps, start, damp, ctrd_h, asmt_h, bias ? bias_h : nullptr, loss_h,
               static_cast<cudaStream_t>(stream));
}

}  // namespace

extern "C" int qcnn_pq_stats_refine(qcnn_pq_stats* s, int K, int sweeps, const float* wei_h, float* ctrd_h, uint8_t* asmt_h,
                                    double* loss_h, void* stream) {
  return RefineStats(s, "qcnn_pq_stats_refine", false, false, false, 0.0, K, sweeps, wei_h, ctrd_h, asmt_h, nullptr, loss_h,
                     stream);
}

extern "C" int qcnn_pq_stats_refine_target(qcnn_pq_stats* s, int K, int sweeps, float* ctrd_h, uint8_t* asmt_h, double* loss_h,
                                           void* stream) {
  return RefineStats(s, "qcnn_pq_stats_refine_target", true, false, false, 0.0, K, sweeps, nullptr, ctrd_h, asmt_h, nullptr,
                     loss_h, stream);
}

extern "C" int qcnn_pq_stats_refine_bias(qcnn_pq_stats* s, int K, int sweeps, const float* wei_h, float* ctrd_h, uint8_t* asmt_h,
                                         float* bias_h, double* loss_h, void* stream) {
  return RefineStats(s, "qcnn_pq_stats_refine_bias", false, true, false, 0.0, K, sweeps, wei_h, ctrd_h, asmt_h, bias_h, loss_h,
                     stream);
}

extern "C" int qcnn_pq_stats_refine_target_bias(qcnn_pq_stats* s, int K, int sweeps, float* ctrd_h, uint8_t* asmt_h,
                                                float* bias_h, double* loss_h, void* stream) {
  return RefineStats(s, "qcnn_pq_stats_refine_target_bias", true, true, false, 0.0, K, sweeps, nullptr, ctrd_h, asmt_h, bias_h,
                     loss_h, stream);
}

extern "C" int qcnn_pq_stats_refine_damped(qcnn_pq_stats* s, int target, double damp, int K, int sweeps, const float* wei_h,
                                           float* ctrd_h, uint8_t* asmt_h, float* bias_h, double* loss_h, void* stream) {
  const char* who = "qcnn_pq_stats_refine_damped";
  QCNN_CHECK(target == 0 || target == 1, "%s: target=%d is not 0 or 1", who, target);
  return RefineStats(s, who, target != 0, bias_h != nullptr, true, damp, K, sweeps, wei_h, ctrd_h, asmt_h, bias_h, loss_h, stream);
}

extern "C" void qcnn_pq_stats_destroy(qcnn_pq_stats* s) {
  if (!s) return;
  DeviceGuard guard(s->ctx->device);
  if (s->done) cudaEventSynchronize(s->done);   // queued adds still use the buffers
  delete s;
}
