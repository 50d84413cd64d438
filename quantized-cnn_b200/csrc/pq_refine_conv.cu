// Error-correcting product quantization of conv layers on the device: block coordinate descent on the codebook and the
// assignments so that the layer's response conv(x, W) is kept on given inputs (the paper's quantization with error
// correction).  Semantics, normative (DESIGN.md 4e, "Error correction for conv layers"):
//   Cg = Cin / grp, T = k^2 taps, S = ceil(Cg / d); subspace m covers the per-group channels [m d, m d + w_m).
//   Per group g, G_g = sum p p^T (fp64, fixed order) over the zero-padded Cg T patches p of the group's channels.
//   E = W - W^ (fp64), loss = sum_g sum_{o in g} E_o^T G_g E_o; one codebook per subspace serves every tap and group.
//   A sweep visits m = 0..S-1 in order; m is skipped when !(sum_g sum_t tr G^m_{g,tt} > 0).
//   h_{o,t} = [G_g R_o]_{(m,t)}, R_o = E_o with m's taps replaced by the weights (the other subspaces' residual).
//   codebook   over U = {k : n_k > 0}, M = sum_g sum_{t,t'} Cnt^g_{tt'} (x) G^m_{g,tt'} (ascending g, t, t'),
//              b_k = sum of h_{o,t} assigned to k (o, then t ascending), D = fp32((M + mu I)^-1 b) by blocked Cholesky,
//              mu = 1e-10 tr(M) / (|U| w_m); D replaces C[m][U] only if (D - C)^T (M (D + C) - 2 b) < 0.
//   assign     per output, taps t = 0..T-1 in order: a = argmin_k c_k^T G_tt c_k - 2 c_k^T h'_{o,t} (fp64, lowest index
//              on ties), h' with E current (earlier taps' new assignments included); a (g, t) with !(tr G_tt > 0) keeps.
// Target form (qcnn_pq_refine_conv_target): inputs y, targets t [N][Ho][Wo][Cout], per group
//   P_g[o][q] = sum over positions of t[pos][o] p_g(pos)[q] (the same patch chunks, ascending), and R = P - G W^ in place
//   of G E everywhere above; loss = |T|^2 + sum_o (-2 w^_o^T P_o + w^_o^T G_g w^_o).  It runs on the same kernels:
//   the weights are zeros, so E = -W^, and the initial GE = P + E G.
// No floating-point atomics: two calls return identical bits.
//
// Internal dim order (patches, G, E, GE, the weights): subspace-major, q = m d T + t w_m + j, so subspace m's dims are
// one contiguous block of T w_m and G^m is a diagonal block of G_g.  Per subspace the work is ordinary launches: the
// responses and the trailing update of GE are fp64 tensor-core GEMMs, M is built per pair of used clusters from
// per-tap member lists, the Cholesky is blocked by 64 with its trailing updates on the same GEMM, and the tap-ordered
// assignment step gives a warp to each output.  The host reads |U| once per subspace to size the solve.
#include <math.h>

#include <algorithm>
#include <memory>
#include <vector>

#include "pq_refine_common.cuh"
#include "qcnn_internal.h"

using namespace qcnn;

namespace {

constexpr int kMaxSystem = 2048;                 // K w_m: the size of the joint codebook system
constexpr int kCholBlock = 64;                   // panel width of the blocked Cholesky
constexpr int kSolveThreads = 1024;
constexpr int kNormalThreads = 128;
constexpr int kAssignWarps = 8;
constexpr size_t kRunBytes = size_t(256) << 20;     // an add folds its positions in runs of 2^28 / (4 Dg)

// s[g][q] (accumulate: s[g][q] +) the sum over output positions (oy, then ox ascending) of the image sum `plane`
// [Hin][Win][Cin] at the input pixel tap t of dim q reads, for every (g, q) (thread g Dg + q); a tap outside the map
// adds nothing (the zero padding)
__global__ void pqrc_tapsum_kernel(const double* __restrict__ plane, int Hin, int Win, int Cin, int ksz, int pad, int stride,
                                   int Ho, int Wo, int Cg, int d, int grp, double* __restrict__ s, int accumulate) {
  const int T = ksz * ksz, Dg = Cg * T;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= grp * Dg) return;
  const int g = i / Dg;
  const Dim q = DecodeDim(i - g * Dg, Cg, d, T);
  const int ky = q.t / ksz, kx = q.t % ksz;
  const double* p = plane + g * Cg + q.m * d + q.j;
  double f = 0.0;
  for (int oy = 0; oy < Ho; oy++) {
    const int iy = oy * stride - pad + ky;
    if (iy < 0 || iy >= Hin) continue;
    for (int ox = 0; ox < Wo; ox++) {
      const int ix = ox * stride - pad + kx;
      if (ix >= 0 && ix < Win) f += p[(static_cast<size_t>(iy) * Win + ix) * Cin];
    }
  }
  s[i] = accumulate ? s[i] + f : f;
}

// Subspace m, nb = T w dims from q0: Wh[o][r] = the decoded weight w^ (fp64), H[o][r] = GE[o][q0 + r] (the responses'
// first term; the GEMM adds W^_m G^m).
__global__ void pqrc_decode_kernel(const float* __restrict__ C, const uint8_t* __restrict__ A, const double* __restrict__ GE,
                                   double* __restrict__ Wh, double* __restrict__ H, int m, int Cout, int Dg, int K, int d, int w,
                                   int T, int q0) {
  const int nb = T * w;
  const size_t total = static_cast<size_t>(Cout) * nb;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int o = static_cast<int>(i / nb), r = static_cast<int>(i % nb), t = r / w, j = r % w;
    const uint8_t a = A[(static_cast<size_t>(m) * Cout + o) * T + t];
    Wh[i] = static_cast<double>(C[(static_cast<size_t>(m) * K + a) * d + j]);
    H[i] = GE[static_cast<size_t>(o) * Dg + q0 + r];
  }
}

// Per (g, t) (blockIdx.x = g T + t): the outputs o of group g with A[m][o][t] = k, for every k, in ascending o.
// Mem[gt][Off[gt][k] .. Off[gt][k + 1]) (global output indices), Off [grp T][K + 1].
__global__ void __launch_bounds__(256) pqrc_lists_kernel(const uint8_t* __restrict__ A, int* __restrict__ Mem, int* __restrict__ Off,
                                                         int m, int Cout, int Cpg, int K, int T) {
  __shared__ int cnt[257];
  const int gt = blockIdx.x, g = gt / T, t = gt % T, k = threadIdx.x;
  const uint8_t* Am = A + static_cast<size_t>(m) * Cout * T + t;
  int n = 0;
  if (k < K)
    for (int o = g * Cpg; o < (g + 1) * Cpg; o++) n += Am[static_cast<size_t>(o) * T] == k;
  cnt[k] = n;
  __syncthreads();
  if (k == 0) {
    int s = 0;
    for (int i = 0; i < K; i++) {
      const int c = cnt[i];
      cnt[i] = s;
      s += c;
    }
    cnt[K] = s;
  }
  __syncthreads();
  int* off = Off + static_cast<size_t>(gt) * (K + 1);
  if (k < K) off[k] = cnt[k];
  if (k == 0) off[K] = cnt[K];
  if (k < K) {
    int* mem = Mem + static_cast<size_t>(gt) * Cpg + cnt[k];
    for (int o = g * Cpg; o < (g + 1) * Cpg; o++)
      if (Am[static_cast<size_t>(o) * T] == k) *mem++ = o;
  }
}

// U = {k : n_k > 0} in ascending k -> Uk[0 .. *nU)
__global__ void __launch_bounds__(256) pqrc_used_kernel(const int* __restrict__ Off, int* __restrict__ Uk, int* __restrict__ nU, int GT,
                                                        int K) {
  __shared__ int used[256];
  const int k = threadIdx.x;
  int n = 0;
  if (k < K)
    for (int gt = 0; gt < GT; gt++) n += Off[static_cast<size_t>(gt) * (K + 1) + k + 1] - Off[static_cast<size_t>(gt) * (K + 1) + k];
  used[k] = n > 0;
  __syncthreads();
  if (k == 0) {
    int u = 0;
    for (int i = 0; i < K; i++)
      if (used[i]) Uk[u++] = i;
    *nU = u;
  }
}

// The block (u, u') of M (blockIdx.x = u', blockIdx.y = u): for k = Uk[u], k' = Uk[u'] and every (j, j'),
// M[u w + j][u' w + j'] = sum over g, t, t' ascending of Cnt^g_{tt'}[k][k'] G_g[(m, t, j)][(m, t', j')], each product
// rounded before it is added (no contraction).  Cnt^g_{tt'}[k][k'] counts the members o of (g, t, k) with
// A[m][o][t'] = k'.  A thread owns fixed (j, j') entries, so only the counts need a barrier.
__global__ void __launch_bounds__(kNormalThreads) pqrc_normal_kernel(const double* __restrict__ G, const uint8_t* __restrict__ A,
                                                                     const int* __restrict__ Mem, const int* __restrict__ Off,
                                                                     const int* __restrict__ Uk, double* __restrict__ M, int m,
                                                                     int grp, int Cout, int Cpg, int Dg, int K, int T, int w,
                                                                     int q0, int n) {
  extern __shared__ double nrm_sm[];   // acc [w w], then the counts [T] as int
  double* acc = nrm_sm;
  int* sc = reinterpret_cast<int*>(nrm_sm + w * w);
  const int tid = threadIdx.x, u = blockIdx.y, v = blockIdx.x, k = Uk[u], k2 = Uk[v], ww = w * w;
  for (int e = tid; e < ww; e += kNormalThreads) acc[e] = 0.0;
  const uint8_t* Am = A + static_cast<size_t>(m) * Cout * T;
  for (int g = 0; g < grp; g++) {
    const double* Gg = G + static_cast<size_t>(g) * Dg * Dg;
    for (int t = 0; t < T; t++) {
      const int gt = g * T + t;
      const int b0 = Off[static_cast<size_t>(gt) * (K + 1) + k], b1 = Off[static_cast<size_t>(gt) * (K + 1) + k + 1];
      if (b0 == b1) continue;
      const int* mem = Mem + static_cast<size_t>(gt) * Cpg;
      __syncthreads();   // the previous tap's counts are read
      for (int t2 = tid; t2 < T; t2 += kNormalThreads) {
        int c = 0;
        for (int e = b0; e < b1; e++) c += Am[static_cast<size_t>(mem[e]) * T + t2] == k2;
        sc[t2] = c;
      }
      __syncthreads();
      for (int t2 = 0; t2 < T; t2++) {
        const int c = sc[t2];
        if (c == 0) continue;
        const double cd = static_cast<double>(c);
        for (int e = tid; e < ww; e += kNormalThreads) {
          const int j = e / w, j2 = e % w;
          acc[e] = __dadd_rn(acc[e], __dmul_rn(cd, Gg[static_cast<size_t>(q0 + t * w + j) * Dg + q0 + t2 * w + j2]));
        }
      }
    }
  }
  for (int e = tid; e < ww; e += kNormalThreads)
    M[static_cast<size_t>(u * w + e / w) * n + v * w + e % w] = acc[e];
}

// b[u w + j] = sum of H[o][t w + j] over (o, t) with A[m][o][t] = Uk[u], o ascending, then t
__global__ void pqrc_rhs_kernel(const double* __restrict__ H, const uint8_t* __restrict__ A, const int* __restrict__ Uk,
                                double* __restrict__ b, int m, int Cout, int T, int w, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int k = Uk[i / w], j = i % w, nb = T * w;
  const uint8_t* Am = A + static_cast<size_t>(m) * Cout * T;
  double s = 0.0;
  for (int o = 0; o < Cout; o++)
    for (int t = 0; t < T; t++)
      if (Am[static_cast<size_t>(o) * T + t] == k) s += H[static_cast<size_t>(o) * nb + t * w + j];
  b[i] = s;
}

// F = M + mu I, mu = 1e-10 tr(M) / n (the trace in ascending order, by every CTA)
__global__ void pqrc_ridge_kernel(const double* __restrict__ M, double* __restrict__ F, int n) {
  __shared__ double mu;
  if (threadIdx.x == 0) {
    double tr = 0.0;
    for (int i = 0; i < n; i++) tr += M[static_cast<size_t>(i) * (n + 1)];
    mu = 1e-10 * tr / n;
  }
  __syncthreads();
  const size_t total = static_cast<size_t>(n) * n;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    F[i] = M[i] + (i % (n + 1) == 0 ? mu : 0.0);
}

// Cholesky of the diagonal block F[kb .. kb + bw)^2 (already updated by the earlier panels), in place, lower triangle
__global__ void __launch_bounds__(256) pqrc_potrf_kernel(double* __restrict__ F, int n, int kb, int bw) {
  __shared__ double L[kCholBlock][kCholBlock + 1];
  const int tid = threadIdx.x;
  for (int e = tid; e < bw * bw; e += blockDim.x) L[e / bw][e % bw] = F[static_cast<size_t>(kb + e / bw) * n + kb + e % bw];
  __syncthreads();
  for (int k = 0; k < bw; k++) {
    if (tid == 0) L[k][k] = sqrt(L[k][k]);
    __syncthreads();
    for (int i = k + 1 + tid; i < bw; i += blockDim.x) L[i][k] /= L[k][k];
    __syncthreads();
    const int r = bw - k - 1;
    for (int e = tid; e < r * r; e += blockDim.x) {
      const int i = k + 1 + e / r, j = k + 1 + e % r;
      if (j <= i) L[i][j] -= L[i][k] * L[j][k];
    }
    __syncthreads();
  }
  for (int e = tid; e < bw * bw; e += blockDim.x)
    if (e % bw <= e / bw) F[static_cast<size_t>(kb + e / bw) * n + kb + e % bw] = L[e / bw][e % bw];
}

// Panel below the diagonal block: row r >= kb + bw solves x L_kk^T = F[r][kb ..), in place; Pt[j][r - kb - bw] = -x_j
// feeds the trailing update F -= P P^T as a GEMM.
__global__ void __launch_bounds__(kCholBlock) pqrc_trsm_kernel(double* __restrict__ F, double* __restrict__ Pt, int n, int kb, int bw) {
  __shared__ double L[kCholBlock][kCholBlock + 1];
  for (int e = threadIdx.x; e < bw * bw; e += blockDim.x) L[e / bw][e % bw] = F[static_cast<size_t>(kb + e / bw) * n + kb + e % bw];
  __syncthreads();
  const int r0 = kb + bw, r = r0 + blockIdx.x * kCholBlock + threadIdx.x;
  if (r >= n) return;
  double* row = F + static_cast<size_t>(r) * n + kb;
  for (int j = 0; j < bw; j++) {
    double s = row[j];
    for (int i = 0; i < j; i++) s -= row[i] * L[j][i];
    s /= L[j][j];
    row[j] = s;
    Pt[static_cast<size_t>(j) * n + r - r0] = -s;
  }
}

// With L (lower triangle of F): z = L^-T L^-1 b, D = fp32(z); if (D - C)^T (M (D + C) - 2 b) < 0, C[m][Uk[u]][j] = D.
// One CTA; each 64-row block's triangle is solved by warp 0, the rest of the vector updated by all threads.
__global__ void __launch_bounds__(kSolveThreads) pqrc_solve_kernel(const double* __restrict__ F, const double* __restrict__ M,
                                                                   const double* __restrict__ b, const int* __restrict__ Uk,
                                                                   float* __restrict__ C, int m, int K, int d, int w, int n) {
  __shared__ double r[kMaxSystem], z[kMaxSystem], red[kSolveThreads / 32];
  __shared__ int accept;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < n; i += kSolveThreads) r[i] = b[i];
  __syncthreads();
  // forward: L y = b (y into z)
  for (int kb = 0; kb < n; kb += kCholBlock) {
    const int bw = min(kCholBlock, n - kb);
    if (warp == 0) {
      for (int j = 0; j < bw; j++) {
        const double y = r[kb + j] / F[static_cast<size_t>(kb + j) * n + kb + j];
        for (int i = j + 1 + lane; i < bw; i += 32) r[kb + i] -= F[static_cast<size_t>(kb + i) * n + kb + j] * y;
        if (lane == 0) z[kb + j] = y;
        __syncwarp();
      }
    }
    __syncthreads();
    for (int i = kb + bw + tid; i < n; i += kSolveThreads) {
      double s = 0.0;
      for (int j = 0; j < bw; j++) s += F[static_cast<size_t>(i) * n + kb + j] * z[kb + j];
      r[i] -= s;
    }
    __syncthreads();
  }
  for (int i = tid; i < n; i += kSolveThreads) r[i] = z[i];
  __syncthreads();
  // backward: L^T z = y
  for (int kb = (n - 1) / kCholBlock * kCholBlock; kb >= 0; kb -= kCholBlock) {
    const int bw = min(kCholBlock, n - kb);
    if (warp == 0) {
      for (int j = bw - 1; j >= 0; j--) {
        const double x = r[kb + j] / F[static_cast<size_t>(kb + j) * n + kb + j];
        for (int i = lane; i < j; i += 32) r[kb + i] -= F[static_cast<size_t>(kb + j) * n + kb + i] * x;
        if (lane == 0) z[kb + j] = x;
        __syncwarp();
      }
    }
    __syncthreads();
    for (int i = tid; i < kb; i += kSolveThreads) {
      double s = 0.0;
      for (int j = 0; j < bw; j++) s += F[static_cast<size_t>(kb + j) * n + i] * z[kb + j];
      r[i] -= s;
    }
    __syncthreads();
  }
  // D into z (rounded), the current codewords into r
  for (int i = tid; i < n; i += kSolveThreads) {
    z[i] = static_cast<double>(static_cast<float>(z[i]));
    r[i] = static_cast<double>(C[(static_cast<size_t>(m) * K + Uk[i / w]) * d + i % w]);
  }
  __syncthreads();
  // acceptance: a warp per row of M (lanes over columns, a fixed shuffle tree), rows summed per warp in ascending order
  double part = 0.0;
  for (int i = warp; i < n; i += kSolveThreads / 32) {
    const double* Mi = M + static_cast<size_t>(i) * n;
    double s = 0.0;
    for (int j = lane; j < n; j += 32) s += Mi[j] * (z[j] + r[j]);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    part += (z[i] - r[i]) * (s - 2.0 * b[i]);
  }
  if (lane == 0) red[warp] = part;
  __syncthreads();
  if (tid == 0) {
    double s = 0.0;
    for (int i = 0; i < kSolveThreads / 32; i++) s += red[i];
    accept = s < 0.0;
  }
  __syncthreads();
  if (accept)
    for (int i = tid; i < n; i += kSolveThreads) C[(static_cast<size_t>(m) * K + Uk[i / w]) * d + i % w] = static_cast<float>(z[i]);
}

// CC[g][t][k] = c_k^T G^m_{g,tt} c_k (blockIdx.x = g T + t, thread k)
__global__ void __launch_bounds__(256) pqrc_ccost_kernel(const double* __restrict__ G, const float* __restrict__ C,
                                                         double* __restrict__ CC, int m, int Dg, int K, int d, int w, int T,
                                                         int q0) {
  const int gt = blockIdx.x, g = gt / T, t = gt % T, k = threadIdx.x;
  if (k >= K) return;
  const double* Gt = G + static_cast<size_t>(g) * Dg * Dg + static_cast<size_t>(q0 + t * w) * Dg + q0 + t * w;
  const float* c = C + (static_cast<size_t>(m) * K + k) * d;
  double s = 0.0;
  for (int i = 0; i < w; i++) {
    double gi = 0.0;
    for (int j = 0; j < w; j++) gi += Gt[static_cast<size_t>(i) * Dg + j] * static_cast<double>(c[j]);
    s += static_cast<double>(c[i]) * gi;
  }
  CC[static_cast<size_t>(gt) * K + k] = s;
}

// A warp per output o walks the taps in order: h'_t = h_t - sum_{t'' != t} G^m_{g,tt''} w^_{t''} (the current decoded
// weights, earlier taps already reassigned), a_t = argmin_k CC[g][t][k] - 2 c_k^T h'_t.  Then E's block gets the new
// decoded weights and Dlt = E_new - E_old feeds the trailing GEMM.
__global__ void __launch_bounds__(kAssignWarps * 32) pqrc_assign_kernel(const double* __restrict__ G, const float* __restrict__ C,
                                                                        const double* __restrict__ CC, const double* __restrict__ H,
                                                                        const float* __restrict__ W, uint8_t* __restrict__ A,
                                                                        double* __restrict__ E, double* __restrict__ Dlt, int m,
                                                                        int Cout, int Cpg, int Dg, int K, int d, int w, int T,
                                                                        int q0) {
  extern __shared__ double asg_sm[];   // per warp: h' [kMaxD], then the row's assignments [T] as int
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int o = blockIdx.x * kAssignWarps + warp;
  if (o >= Cout) return;
  double* hp = asg_sm + static_cast<size_t>(warp) * (kMaxD + (T + 1) / 2);
  int* a = reinterpret_cast<int*>(hp + kMaxD);
  const int g = o / Cpg, nb = T * w;
  const double* Gg = G + static_cast<size_t>(g) * Dg * Dg;
  const float* Cm = C + static_cast<size_t>(m) * K * d;
  uint8_t* Ao = A + (static_cast<size_t>(m) * Cout + o) * T;
  const double* Ho = H + static_cast<size_t>(o) * nb;
  for (int t = lane; t < T; t += 32) a[t] = Ao[t];
  __syncwarp();
  for (int t = 0; t < T; t++) {
    const double* Grow = Gg + static_cast<size_t>(q0 + t * w) * Dg + q0;   // rows (m, t, j), columns from the block's start
    double tr = 0.0;
    for (int j = 0; j < w; j++) tr += Grow[static_cast<size_t>(j) * Dg + t * w + j];
    if (!(tr > 0.0)) continue;
    for (int j = lane; j < w; j += 32) {
      double s = 0.0;
#pragma unroll 1
      for (int t2 = 0; t2 < T; t2++) {
        if (t2 == t) continue;
        const float* c = Cm + static_cast<size_t>(a[t2]) * d;
        const double* gr = Grow + static_cast<size_t>(j) * Dg + t2 * w;
        for (int i = 0; i < w; i++) s += gr[i] * static_cast<double>(c[i]);
      }
      hp[j] = Ho[t * w + j] - s;
    }
    __syncwarp();
    const double* cc = CC + (static_cast<size_t>(g) * T + t) * K;
    double best = INFINITY;
    int bi = K;
#pragma unroll 1
    for (int k = lane; k < K; k += 32) {
      const float* c = Cm + static_cast<size_t>(k) * d;
      double dot = 0.0;
      for (int j = 0; j < w; j++) dot += static_cast<double>(c[j]) * hp[j];
      const double v = cc[k] - 2.0 * dot;
      if (v < best) { best = v; bi = k; }
    }
    for (int off = 16; off > 0; off >>= 1) {
      const double ob = __shfl_xor_sync(0xffffffffu, best, off);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
      if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (lane == 0) a[t] = bi;
    __syncwarp();
  }
  for (int t = lane; t < T; t += 32) Ao[t] = static_cast<uint8_t>(a[t]);
  for (int r = lane; r < nb; r += 32) {
    const size_t qi = static_cast<size_t>(o) * Dg + q0 + r;
    const double e = static_cast<double>(W[qi]) - static_cast<double>(Cm[static_cast<size_t>(a[r / w]) * d + r % w]);
    Dlt[static_cast<size_t>(o) * nb + r] = e - E[qi];
    E[qi] = e;
  }
}

// The geometry checks of every conv entry point, then the derived sizes
int CheckGeometry(const char* who, int Cin, int Hin, int Win, int Cout, int ksz, int pad, int stride, int grp, PqGeometry* geo) {
  QCNN_CHECK(Cin >= 1 && Hin >= 1 && Win >= 1 && Cout >= 1 && ksz >= 1 && pad >= 0 && stride >= 1 && grp >= 1,
             "%s: bad geometry (Cin=%d Hin=%d Win=%d Cout=%d ksz=%d pad=%d stride=%d grp=%d)", who, Cin, Hin, Win, Cout, ksz, pad,
             stride, grp);
  QCNN_CHECK(Cin % grp == 0 && Cout % grp == 0, "%s: Cin=%d and Cout=%d must be divisible by grp=%d", who, Cin, Cout, grp);
  QCNN_CHECK(Hin + 2 * pad >= ksz && Win + 2 * pad >= ksz, "%s: empty output (%dx%d input, pad %d, kernel %d)", who, Hin, Win, pad, ksz);
  geo->Cin = Cin; geo->Hin = Hin; geo->Win = Win; geo->Cout = Cout; geo->ksz = ksz; geo->pad = pad; geo->stride = stride; geo->grp = grp;
  geo->Ho = (Hin + 2 * pad - ksz) / stride + 1;
  geo->Wo = (Win + 2 * pad - ksz) / stride + 1;
  geo->Cg = Cin / grp; geo->Cpg = Cout / grp; geo->T = ksz * ksz; geo->Dg = geo->Cg * geo->T;
  return 0;
}

// The one-shot calls' argument checks, the same for both forms and in the order of their messages
int RefineConv(bool target, qcnn_ctx* ctx, int Cin, int Hin, int Win, int Cout, int ksz, int pad, int stride, int grp, int K,
               int d, int sweeps, const float* knl_h, const float* x, const float* t, int N, float* ctrd_h, uint8_t* asmt_h,
               double* loss_h, void* stream) {
  const char* who = target ? "qcnn_pq_refine_conv_target" : "qcnn_pq_refine_conv";
  QCNN_CHECK(ctx && (target || knl_h) && ctrd_h && asmt_h, "%s: NULL argument", who);
  PqGeometry geo;
  if (int rc = CheckGeometry(who, Cin, Hin, Win, Cout, ksz, pad, stride, grp, &geo)) return rc;
  if (int rc = CheckConvK(who, K)) return rc;
  QCNN_CHECK(d >= 1 && d <= kMaxD, "%s: d=%d is outside 1..%d", who, d, kMaxD);
  QCNN_CHECK(sweeps >= 0, "%s: sweeps=%d is negative", who, sweeps);
  QCNN_CHECK(N >= 1, "%s: N=%d: at least one input is needed", who, N);
  QCNN_CHECK(x, "%s: NULL argument", who);
  QCNN_CHECK(!target || t, "%s: NULL t", who);
  if (int rc = CheckConvSystem(who, K, d, geo.Cg)) return rc;
  return RefineOnce(ctx, who, true, target, geo, K, d, sweeps, knl_h, x, t, N, ctrd_h, asmt_h, loss_h,
                    static_cast<cudaStream_t>(stream));
}

}  // namespace

namespace qcnn {

int CheckConvSystem(const char* who, int K, int d, int Cg) {
  if (int rc = CheckConvK(who, K)) return rc;
  const long long sys = static_cast<long long>(K) * std::min(d, Cg);
  QCNN_CHECK(sys <= kMaxSystem, "%s: K*min(d, Cin/grp) = %d*%d = %lld exceeds %d, the size of the joint codebook system", who, K,
             std::min(d, Cg), sys, kMaxSystem);
  return 0;
}

// The conv sweeps: the subspaces the sweeps skip, then per subspace the responses, the joint codebook step, the
// tap-ordered assignment and the update of GE
int SweepConv(qcnn_pq_stats* s, const char* who, bool target, int K, int sweeps, const float* wts, std::vector<uint8_t>& at,
              const double* G, const double* P, const double* TT, float* ctrd_h, uint8_t* asmt_h, float* bias_h,
              double* loss_h, cudaStream_t st) {
  qcnn_ctx* ctx = s->ctx;
  const PqGeometry& geo = s->geo;
  const int d = s->d, Cout = geo.Cout, Cg = geo.Cg, Cpg = geo.Cpg, T = geo.T, Dg = geo.Dg, grp = geo.grp;
  const int S = CeilDiv(Cg, d), wmax = std::min(d, Cg);
  QCNN_ON_DEVICE(ctx->device);
  SweepState ss;
  if (int rc = BeginSweeps(&ss, s, who, target, K, sweeps, wts, at, ctrd_h, G, P, TT, st)) return rc;
  const size_t nbMax = static_cast<size_t>(T) * wmax, nMax = static_cast<size_t>(K) * wmax;
  DeviceBuffer dWh, dH, dDlt, dM, dF, dPt, dB, dMem, dOff, dUk, dNU, dCC;
  if (Reserve(ctx, who, dWh, sizeof(double) * Cout * nbMax, "the decoded subspace") ||
      Reserve(ctx, who, dH, sizeof(double) * Cout * nbMax, "the subspace responses") ||
      Reserve(ctx, who, dDlt, sizeof(double) * Cout * nbMax, "the subspace's changes") ||
      Reserve(ctx, who, dM, sizeof(double) * nMax * nMax, "the joint system") ||
      Reserve(ctx, who, dF, sizeof(double) * nMax * nMax, "its Cholesky factor") ||
      Reserve(ctx, who, dPt, sizeof(double) * kCholBlock * nMax, "the Cholesky panel") ||
      Reserve(ctx, who, dB, sizeof(double) * nMax, "the right-hand side") ||
      Reserve(ctx, who, dMem, sizeof(int) * grp * static_cast<size_t>(T) * Cpg, "the cluster members") ||
      Reserve(ctx, who, dOff, sizeof(int) * grp * static_cast<size_t>(T) * (K + 1), "the cluster members") ||
      Reserve(ctx, who, dUk, sizeof(int) * K, "the used clusters") || Reserve(ctx, who, dNU, sizeof(int), "the used clusters") ||
      Reserve(ctx, who, dCC, sizeof(double) * grp * static_cast<size_t>(T) * K, "the codeword norms"))
    return 1;
  std::vector<double> diag(static_cast<size_t>(grp) * Dg);
  for (int g = 0; g < grp; g++)
    QCNN_CUDA(cudaMemcpy2DAsync(diag.data() + static_cast<size_t>(g) * Dg, sizeof(double), G + static_cast<size_t>(g) * Dg * Dg,
                                sizeof(double) * (static_cast<size_t>(Dg) + 1), sizeof(double), Dg, cudaMemcpyDeviceToHost, st));
  QCNN_CUDA(cudaStreamSynchronize(st));
  std::vector<bool> skip(S);
  for (int m = 0; m < S; m++) {
    const int w = std::min(d, Cg - m * d);
    double tr = 0.0;
    for (int g = 0; g < grp; g++)
      for (int r = 0; r < T * w; r++) tr += diag[static_cast<size_t>(g) * Dg + m * d * T + r];
    skip[m] = !(tr > 0.0);
  }
  const int tiles = CeilDiv(Dg, kTile);
  const size_t assignSmem = sizeof(double) * kAssignWarps * (kMaxD + (T + 1) / 2);
  if (assignSmem > 48 * 1024)
    QCNN_CUDA(cudaFuncSetAttribute(pqrc_assign_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(assignSmem)));
  for (int sw = 1; sw <= sweeps; sw++) {
    for (int m = 0; m < S; m++) {
      if (skip[m]) continue;
      const int w = std::min(d, Cg - m * d), nb = T * w, q0 = m * d * T;
      const size_t nwb = static_cast<size_t>(Cout) * nb;
      const int gridB = static_cast<int>(std::min<size_t>((nwb + 255) / 256, 32u * ctx->sm_count));
      // responses h = GE[:, block] + W^_m G^m
      pqrc_decode_kernel<<<gridB, 256, 0, st>>>(ss.C.as<float>(), ss.A.as<uint8_t>(), ss.GE.as<double>(), dWh.as<double>(),
                                                dH.as<double>(), m, Cout, Dg, K, d, w, T, q0);
      for (int g = 0; g < grp; g++) {
        const size_t ro = static_cast<size_t>(g) * Cpg * nb;
        const double* Gm = G + static_cast<size_t>(g) * Dg * Dg + static_cast<size_t>(q0) * Dg + q0;
        pqr_gemm_kernel<kGemmF64><<<dim3(CeilDiv(nb, kTile), CeilDiv(Cpg, kTile)), kGemmThreads, 0, st>>>(
            dWh.as<double>() + ro, nb, Gm, Dg, dH.as<double>() + ro, nb, Cpg, nb, nb, 1);
      }
      // the used clusters and, per (g, t, k), their members
      pqrc_lists_kernel<<<grp * T, 256, 0, st>>>(ss.A.as<uint8_t>(), dMem.as<int>(), dOff.as<int>(), m, Cout, Cpg, K, T);
      pqrc_used_kernel<<<1, 256, 0, st>>>(dOff.as<int>(), dUk.as<int>(), dNU.as<int>(), grp * T, K);
      QCNN_CUDA(cudaGetLastError());
      int nU = 0;
      QCNN_CUDA(cudaMemcpyAsync(&nU, dNU.get(), sizeof(int), cudaMemcpyDeviceToHost, st));
      QCNN_CUDA(cudaStreamSynchronize(st));
      const int n = nU * w;
      // codebook: M, b, the blocked Cholesky of M + mu I, the solve and the acceptance test
      const size_t nrmSmem = sizeof(double) * w * w + sizeof(int) * T;
      pqrc_normal_kernel<<<dim3(nU, nU), kNormalThreads, nrmSmem, st>>>(G, ss.A.as<uint8_t>(), dMem.as<int>(), dOff.as<int>(),
                                                                        dUk.as<int>(), dM.as<double>(), m, grp, Cout, Cpg, Dg, K, T, w,
                                                                        q0, n);
      pqrc_rhs_kernel<<<CeilDiv(n, 128), 128, 0, st>>>(dH.as<double>(), ss.A.as<uint8_t>(), dUk.as<int>(), dB.as<double>(), m, Cout,
                                                       T, w, n);
      const int gridF = static_cast<int>(std::min<size_t>((static_cast<size_t>(n) * n + 255) / 256, 8u * ctx->sm_count));
      pqrc_ridge_kernel<<<gridF, 256, 0, st>>>(dM.as<double>(), dF.as<double>(), n);
      for (int kb = 0; kb < n; kb += kCholBlock) {
        const int bw = std::min(kCholBlock, n - kb), n2 = n - kb - bw;
        pqrc_potrf_kernel<<<1, 256, 0, st>>>(dF.as<double>(), n, kb, bw);
        if (n2 == 0) break;
        pqrc_trsm_kernel<<<CeilDiv(n2, kCholBlock), kCholBlock, 0, st>>>(dF.as<double>(), dPt.as<double>(), n, kb, bw);
        double* Fp = dF.as<double>() + static_cast<size_t>(kb + bw) * n + kb;
        pqr_gemm_kernel<kGemmF64><<<dim3(CeilDiv(n2, kTile), CeilDiv(n2, kTile)), kGemmThreads, 0, st>>>(Fp, n, dPt.as<double>(), n,
                                                                                                         Fp + bw, n, n2, n2, bw, 1);
      }
      pqrc_solve_kernel<<<1, kSolveThreads, 0, st>>>(dF.as<double>(), dM.as<double>(), dB.as<double>(), dUk.as<int>(),
                                                     ss.C.as<float>(), m, K, d, w, n);
      // assignment, tap by tap per output; then GE += Dlt G[block, :]
      pqrc_ccost_kernel<<<grp * T, 256, 0, st>>>(G, ss.C.as<float>(), dCC.as<double>(), m, Dg, K, d, w, T, q0);
      pqrc_assign_kernel<<<CeilDiv(Cout, kAssignWarps), kAssignWarps * 32, assignSmem, st>>>(
          G, ss.C.as<float>(), dCC.as<double>(), dH.as<double>(), ss.W.as<float>(), ss.A.as<uint8_t>(), ss.E.as<double>(),
          dDlt.as<double>(), m, Cout, Cpg, Dg, K, d, w, T, q0);
      for (int g = 0; g < grp; g++) {
        const double* Gb = G + static_cast<size_t>(g) * Dg * Dg + static_cast<size_t>(q0) * Dg;
        pqr_gemm_kernel<kGemmF64><<<dim3(tiles, CeilDiv(Cpg, kTile)), kGemmThreads, 0, st>>>(
            dDlt.as<double>() + static_cast<size_t>(g) * Cpg * nb, nb, Gb, Dg, ss.GE.as<double>() + static_cast<size_t>(g) * Cpg * Dg,
            Dg, Cpg, Dg, nb, 1);
      }
      QCNN_CUDA(cudaGetLastError());
    }
    if (int rc = ss.Loss(sw, st)) return rc;
  }
  return EndSweeps(ss, ctrd_h, asmt_h, bias_h, loss_h, st);
}

// A conv add: the scan, then per group the positions in runs of F, each run's Gram (and cross product) read straight
// from the maps and added in ascending order; then the first moments (s from the image sum of y, u from that of t)
int ConvStatsAdd(qcnn_pq_stats* s, const char* who, const float* y, const float* t, int N, cudaStream_t st) {
  const PqGeometry& geo = s->geo;
  const int Cout = geo.Cout, Cpg = geo.Cpg, Dg = geo.Dg, grp = geo.grp;
  const size_t positions = static_cast<size_t>(N) * geo.Ho * geo.Wo;
  unsigned first[2];
  if (int rc = ScanAdd(s, y, static_cast<size_t>(N) * geo.Hin * geo.Win * geo.Cin, 1, t, positions * Cout, first, st)) return rc;
  QCNN_CHECK(first[0] == kNoneFound, "%s: %s contains a non-finite value", who, s->target ? "y" : "x");
  QCNN_CHECK(first[1] == kNoneFound, "%s: t contains a non-finite value", who);
  QCNN_ON_DEVICE(s->ctx->device);
  const bool acc0 = s->images > 0;
  if (s->target && LaunchSqNorm(t, positions * Cout, s->scratch.as<double>(), s->tt.as<double>(), acc0, st)) return 1;
  const size_t run = std::max<size_t>(1, std::min<size_t>(positions, kRunBytes / (sizeof(float) * Dg)));
  const int tiles = CeilDiv(Dg, kTile);
  for (int g = 0; g < grp; g++) {
    double* Gg = s->G.as<double>() + static_cast<size_t>(g) * Dg * Dg;
    for (size_t p0 = 0; p0 < positions; p0 += run) {
      const int np = static_cast<int>(std::min<size_t>(run, positions - p0));
      const int acc = acc0 || p0 > 0;
      const MapOperand map{y, static_cast<long long>(p0), geo.Hin, geo.Win, geo.Cin, geo.ksz, geo.pad, geo.stride, geo.Ho, geo.Wo,
                           geo.Cg, s->d, g};
      pqr_gemm_kernel<kGemmGramMap><<<tiles * (tiles + 1) / 2, kGemmThreads, 0, st>>>(nullptr, 0, nullptr, 0, Gg, Dg, Dg, Dg, np, acc,
                                                                                     map);
      if (s->target)   // the run's target rows of group g's outputs against its patches
        pqr_gemm_kernel<kGemmCrossMap><<<dim3(tiles, CeilDiv(Cpg, kTile)), kGemmThreads, 0, st>>>(
            t + p0 * Cout + static_cast<size_t>(g) * Cpg, Cout, nullptr, 0, s->P.as<double>() + static_cast<size_t>(g) * Cpg * Dg, Dg,
            Cpg, Dg, np, acc, map);
      QCNN_CUDA(cudaGetLastError());
    }
  }
  if (s->sums) {
    double* plane = s->plane.as<double>();
    const size_t inPlane = static_cast<size_t>(geo.Hin) * geo.Win * geo.Cin, hw = static_cast<size_t>(geo.Ho) * geo.Wo;
    if (LaunchColSum(s->ctx, y, N, inPlane, plane, 0, st)) return 1;
    pqrc_tapsum_kernel<<<CeilDiv(grp * Dg, 128), 128, 0, st>>>(plane, geo.Hin, geo.Win, geo.Cin, geo.ksz, geo.pad, geo.stride, geo.Ho,
                                                               geo.Wo, geo.Cg, s->d, grp, s->sy.as<double>(), acc0);
    QCNN_CUDA(cudaGetLastError());
    if (s->target) {
      if (LaunchColSum(s->ctx, t, N, hw * Cout, plane, 0, st)) return 1;
      if (LaunchColSum(s->ctx, static_cast<const double*>(plane), hw, Cout, s->su.as<double>(), acc0, st)) return 1;
    }
  }
  QCNN_CUDA(cudaEventRecord(s->done, st));
  s->images += N;
  return 0;
}

}  // namespace qcnn

extern "C" int qcnn_pq_refine_conv(qcnn_ctx* ctx, int Cin, int Hin, int Win, int Cout, int ksz, int pad, int stride, int grp, int K,
                                   int d, int sweeps, const float* knl_h, const float* x, int N, float* ctrd_h, uint8_t* asmt_h,
                                   double* loss_h, void* stream) {
  return RefineConv(false, ctx, Cin, Hin, Win, Cout, ksz, pad, stride, grp, K, d, sweeps, knl_h, x, nullptr, N,
                    ctrd_h, asmt_h, loss_h, stream);
}

extern "C" int qcnn_pq_refine_conv_target(qcnn_ctx* ctx, int Cin, int Hin, int Win, int Cout, int ksz, int pad, int stride, int grp,
                                          int K, int d, int sweeps, const float* y, const float* t, int N, float* ctrd_h,
                                          uint8_t* asmt_h, double* loss_h, void* stream) {
  return RefineConv(true, ctx, Cin, Hin, Win, Cout, ksz, pad, stride, grp, K, d, sweeps, nullptr, y, t, N,
                    ctrd_h, asmt_h, loss_h, stream);
}

extern "C" int qcnn_pq_stats_create_conv(qcnn_ctx* ctx, int Cin, int Hin, int Win, int Cout, int ksz, int pad, int stride, int grp,
                                         int d, int target, qcnn_pq_stats** out) {
  const char* who = "qcnn_pq_stats_create_conv";
  QCNN_CHECK(ctx && out, "%s: NULL argument", who);
  *out = nullptr;
  PqGeometry geo;
  if (int rc = CheckGeometry(who, Cin, Hin, Win, Cout, ksz, pad, stride, grp, &geo)) return rc;
  QCNN_CHECK(d >= 1 && d <= kMaxD, "%s: d=%d is outside 1..%d", who, d, kMaxD);
  return CreateStats(ctx, who, true, geo, d, target != 0, true, out);
}
