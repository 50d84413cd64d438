// Pieces shared by the error-correcting quantizers of FC layers (pq_refine.cu) and conv layers (pq_refine_conv.cu):
// the fp64 tensor-core GEMM, the fixed-order block reduction, the residual and loss kernels (same-input and target
// form), and the host code around the sweeps, which treats an FC layer as its 1x1 conv geometry (PqGeometry).  They
// sit in an anonymous namespace because each including .cu file is its own device module and links its own copy.
#ifndef QCNN_PQ_REFINE_COMMON_CUH_
#define QCNN_PQ_REFINE_COMMON_CUH_

#include <math.h>

#include <algorithm>
#include <memory>
#include <vector>

#include "qcnn_internal.h"

namespace {

constexpr int kMaxD = 64;            // the widest subspace
constexpr int kTile = 64;            // GEMM output tile (kTile x kTile per CTA, 2 x 2 warps of 32 x 32)
constexpr int kKStep = 16;           // the DMMA's k
constexpr int kLd = kTile + 4;       // smem row pitch in doubles: fragment reads hit 16 distinct 8-byte bank pairs
constexpr int kGemmThreads = 128;
constexpr int kSweepThreads = 256;
constexpr int kLossBlocks = 512;     // fixed, so the loss reduction order does not depend on the device

__device__ __forceinline__ void Dmma(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
      "{%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

// What pqr_gemm_kernel computes (its template argument)
constexpr int kGemmF64 = 0;     // C [M][N] = (accumulate ? C : 0) + A [M][Kd] B [Kd][N], all fp64
constexpr int kGemmGram = 1;    // C = (accumulate ? C : 0) + X^T X for X = A [Kd][lda] fp32 (M = N = the column count)
constexpr int kGemmCross = 2;   // C [M][N] = (accumulate ? C : 0) + A^T B for A [Kd][lda], B [Kd][ldb] fp32
constexpr int kGemmGramMap = 3;   // kGemmGram with X = the patches of an NHWC map (MapOperand), M = N = Dg
constexpr int kGemmCrossMap = 4;  // kGemmCross with B = the patches of an NHWC map (MapOperand), N = Dg

// (m, t, j) of a conv layer's internal dim q = m d T + t w_m + j: subspace m, tap t, channel m d + j of the group
struct Dim { int m, t, j, w; };
__device__ __forceinline__ Dim DecodeDim(int q, int Cg, int d, int T) {
  Dim r;
  r.m = q / (d * T);
  const int rem = q - r.m * d * T;
  r.w = min(d, Cg - r.m * d);
  r.t = rem / r.w;
  r.j = rem - r.t * r.w;
  return r;
}

// E[o][q] = W[o][q] - C[m][A[m][o][t]][j] in fp64 (A held [S][Cout][T]; FC: T = 1, q the input column)
__global__ void pqrc_residual_kernel(const float* __restrict__ W, const float* __restrict__ C, const uint8_t* __restrict__ A,
                                     double* __restrict__ E, int Cout, int Cg, int K, int d, int T) {
  const int Dg = Cg * T;
  const size_t total = static_cast<size_t>(Cout) * Dg;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int o = static_cast<int>(i / Dg);
    const Dim q = DecodeDim(static_cast<int>(i % Dg), Cg, d, T);
    const uint8_t a = A[(static_cast<size_t>(q.m) * Cout + o) * T + q.t];
    E[i] = static_cast<double>(W[i]) - static_cast<double>(C[(static_cast<size_t>(q.m) * K + a) * d + q.j]);
  }
}

// The patch operand of the map modes: row k is output position pos0 + k = (n Ho + oy) Wo + ox of the NHWC map
// x [N][Hin][Win][Cin], column q the internal dim (m, t, j) of group g, and the element is
// x[n][oy stride - pad + t / ksz][ox stride - pad + t % ksz][g Cg + m d + j], zero outside the map.
struct MapOperand {
  const float* x;
  long long pos0;
  int Hin, Win, Cin, ksz, pad, stride, Ho, Wo, Cg, d, g;
};
constexpr int kMapFar = -(1 << 28);   // a row offset that puts an element outside any map: dims past Dg, rows past Kd

// fp64 tensor-core GEMM, one kTile x kTile output tile per CTA, k in ascending steps of 16 (a fixed order per element).
//   kGemmGram:  lower-triangle tiles only (blockIdx.x is the linear lower-triangle index); each element with row >= col
//               is written to both (row, col) and (col, row), so G is exactly symmetric.
//   otherwise:  the full tile grid, blockIdx.y over M and blockIdx.x over N.
// Operands are staged through registers (the next k-step is loaded while the current one is multiplied), widened to
// fp64 and stored k-major, [16][kLd], in shared memory.
// Map modes: the patch operand's address is the sum of a row part (per k-step, its 16 positions decoded by warp 0 into
// a double-buffered table while the previous k-step is multiplied) and a column part (per thread, its dim decoded once
// into registers), so every element is the value the im2col patch would hold, and the products and their order are those of
// kGemmGram / kGemmCross on the patches.
template <int kMode>
__global__ void __launch_bounds__(kGemmThreads) pqr_gemm_kernel(const void* __restrict__ Ap, int lda, const void* __restrict__ Bp,
                                                                int ldb, double* __restrict__ C, int ldc, int M, int N, int Kd,
                                                                int accumulate, MapOperand map = MapOperand{}) {
  constexpr bool kMap = kMode == kGemmGramMap || kMode == kGemmCrossMap;
  constexpr bool kGram = kMode == kGemmGram || kMode == kGemmGramMap;
  __shared__ double As[2][kKStep][kLd], Bs[2][kKStep][kLd];
  // map modes: per row (k-step buffer, position) the element offset of tap (0, 0) and its map row and column
  __shared__ long long sRowOff[kMap ? 2 : 1][kKStep];
  __shared__ int sRowY[kMap ? 2 : 1][kKStep], sRowX[kMap ? 2 : 1][kKStep];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t = lane & 3, wm = warp >> 1, wn = warp & 1;
  int tm, tn;
  if (kGram) {
    const int i = blockIdx.x;
    tm = static_cast<int>((sqrt(8.0 * i + 1.0) - 1.0) * 0.5);
    while (tm * (tm + 1) / 2 > i) tm--;
    while ((tm + 1) * (tm + 2) / 2 <= i) tm++;
    tn = i - tm * (tm + 1) / 2;
  } else {
    tm = blockIdx.y;
    tn = blockIdx.x;
  }
  const int m0 = tm * kTile, n0 = tn * kTile;
  constexpr int kPer = kKStep * kTile / kGemmThreads;   // 8 elements of each operand per thread and k-step
  double ra[kPer], rb[kPer];
  // map modes: the k-step's raw fp32 elements, widened when they are stored, so that nothing waits for the loads until
  // the k-step's DMMAs are issued
  float fa_[kMap ? kPer : 1], fb_[kMap ? kPer : 1];
  // map modes: a thread loads one column of each operand (nn = tid % kTile), so its dims are decoded once into
  // registers: the offset of the tap and channel, and the tap's row and column (side 0: the tile's rows m0.., side 1
  // its columns n0..; the cross mode reads only side 1); a dim past M / N is far outside the map
  int cOff[2] = {0, 0}, cY[2] = {kMapFar, kMapFar}, cX[2] = {0, 0};
  if (kMap) {
#pragma unroll
    for (int side = 0; side < 2; side++) {
      const int q = (side ? n0 : m0) + tid % kTile;
      if (q < (side ? N : M)) {
        const int T = map.ksz * map.ksz;
        const Dim dm = DecodeDim(q, map.Cg, map.d, T);
        cY[side] = dm.t / map.ksz;
        cX[side] = dm.t % map.ksz;
        cOff[side] = (cY[side] * map.Win + cX[side]) * map.Cin + map.g * map.Cg + dm.m * map.d + dm.j;
      }
    }
  }
  // map modes: lanes 0..15 of warp 0 decode the rows of consecutive k-steps into buffer kt & 1, each lane stepping its
  // position (n, oy, ox) by 16; a row past Kd is far outside the map
  long long rn = 0;
  int ry = 0, rx = 0;
  if (kMap && tid < kKStep) {
    const long long pos = map.pos0 + tid, hw = static_cast<long long>(map.Ho) * map.Wo;
    rn = pos / hw;
    const int yx = static_cast<int>(pos - rn * hw);
    ry = yx / map.Wo;
    rx = yx - ry * map.Wo;
  }
  auto decodeRows = [&](int kt) {
    if (!kMap || tid >= kKStep) return;
    long long off = 0;
    int iy = kMapFar, ix = 0;
    if (kt * kKStep + tid < Kd) {
      iy = ry * map.stride - map.pad;
      ix = rx * map.stride - map.pad;
      off = ((rn * map.Hin + iy) * map.Win + ix) * map.Cin;
    }
    sRowOff[kt & 1][tid] = off;
    sRowY[kt & 1][tid] = iy;
    sRowX[kt & 1][tid] = ix;
    rx += kKStep;
    while (rx >= map.Wo) {
      rx -= map.Wo;
      if (++ry == map.Ho) {
        ry = 0;
        rn++;
      }
    }
  };
  auto mapAt = [&](int buf, int kk, int side) -> float {
    const int iy = sRowY[buf][kk] + cY[side], ix = sRowX[buf][kk] + cX[side];
    const bool in = static_cast<unsigned>(iy) < static_cast<unsigned>(map.Hin) &&
                    static_cast<unsigned>(ix) < static_cast<unsigned>(map.Win);
    return in ? __ldg(map.x + sRowOff[buf][kk] + cOff[side]) : 0.0f;
  };
  if (kMap) {
    decodeRows(0);
    decodeRows(1);
    __syncthreads();
  }
  auto load = [&](int k0) {
    const int rbuf = (k0 / kKStep) & 1;
#pragma unroll
    for (int r = 0; r < kPer; r++) {
      const int e = tid + r * kGemmThreads;
      const int kk = e / kTile, nn = e % kTile;   // B (and the Gram's A): row kk of the k-step, column nn
      const int k = k0 + kk;
      if (kMode == kGemmGramMap) {
        fa_[r] = mapAt(rbuf, kk, 0);
        fb_[r] = mapAt(rbuf, kk, 1);
      } else if (kMode == kGemmCrossMap) {
        const float* A = static_cast<const float*>(Ap);
        fa_[r] = (k < Kd && m0 + nn < M) ? __ldg(A + static_cast<size_t>(k) * lda + m0 + nn) : 0.0f;
        fb_[r] = mapAt(rbuf, kk, 1);
      } else if (kMode == kGemmGram) {
        const float* X = static_cast<const float*>(Ap);
        ra[r] = (k < Kd && m0 + nn < M) ? static_cast<double>(X[static_cast<size_t>(k) * lda + m0 + nn]) : 0.0;
        rb[r] = (k < Kd && n0 + nn < N) ? static_cast<double>(X[static_cast<size_t>(k) * lda + n0 + nn]) : 0.0;
      } else if (kMode == kGemmCross) {
        const float* A = static_cast<const float*>(Ap);
        const float* B = static_cast<const float*>(Bp);
        ra[r] = (k < Kd && m0 + nn < M) ? static_cast<double>(A[static_cast<size_t>(k) * lda + m0 + nn]) : 0.0;
        rb[r] = (k < Kd && n0 + nn < N) ? static_cast<double>(B[static_cast<size_t>(k) * ldb + n0 + nn]) : 0.0;
      } else {
        const double* A = static_cast<const double*>(Ap);
        const double* B = static_cast<const double*>(Bp);
        const int mm = e / kKStep, ka = k0 + e % kKStep;   // A: row mm, k-column ka (rows of A are contiguous in k)
        ra[r] = (ka < Kd && m0 + mm < M) ? A[static_cast<size_t>(m0 + mm) * lda + ka] : 0.0;
        rb[r] = (k < Kd && n0 + nn < N) ? B[static_cast<size_t>(k) * ldb + n0 + nn] : 0.0;
      }
    }
  };
  auto store = [&](int buf) {
#pragma unroll
    for (int r = 0; r < kPer; r++) {
      const int e = tid + r * kGemmThreads;
      if (kMap) {
        As[buf][e / kTile][e % kTile] = static_cast<double>(fa_[r]);
        Bs[buf][e / kTile][e % kTile] = static_cast<double>(fb_[r]);
        continue;
      }
      if (kMode != kGemmF64) As[buf][e / kTile][e % kTile] = ra[r];
      else As[buf][e % kKStep][e / kKStep] = ra[r];
      Bs[buf][e / kTile][e % kTile] = rb[r];
    }
  };
  double acc[2][4][4];
#pragma unroll
  for (int a = 0; a < 2; a++)
#pragma unroll
    for (int b = 0; b < 4; b++)
#pragma unroll
      for (int c = 0; c < 4; c++) acc[a][b][c] = 0.0;
  const int nk = (Kd + kKStep - 1) / kKStep;
  load(0);
  store(0);
  __syncthreads();
  for (int kt = 0; kt < nk; kt++) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load((kt + 1) * kKStep);
    // buffer kt & 1 of the row table was last read by the loads of k-step kt, before the previous barrier
    if (kMap && kt + 2 < nk) decodeRows(kt + 2);
    double fa[2][8], fb[4][4];
#pragma unroll
    for (int mt = 0; mt < 2; mt++)
#pragma unroll
      for (int i = 0; i < 8; i++) fa[mt][i] = As[buf][t + 4 * (i >> 1)][wm * 32 + mt * 16 + g + 8 * (i & 1)];
#pragma unroll
    for (int nt = 0; nt < 4; nt++)
#pragma unroll
      for (int i = 0; i < 4; i++) fb[nt][i] = Bs[buf][t + 4 * i][wn * 32 + nt * 8 + g];
#pragma unroll
    for (int mt = 0; mt < 2; mt++)
#pragma unroll
      for (int nt = 0; nt < 4; nt++) Dmma(acc[mt][nt], fa[mt], fb[nt]);
    if (kt + 1 < nk) store(buf ^ 1);
    __syncthreads();
  }
#pragma unroll
  for (int mt = 0; mt < 2; mt++)
#pragma unroll
    for (int nt = 0; nt < 4; nt++)
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int row = m0 + wm * 32 + mt * 16 + g + 8 * (i >> 1), col = n0 + wn * 32 + nt * 8 + 2 * t + (i & 1);
        if (row >= M || col >= N) continue;
        if (kGram) {
          if (row < col) continue;
          double* p = C + static_cast<size_t>(row) * ldc + col;
          const double v = accumulate ? *p + acc[mt][nt][i] : acc[mt][nt][i];
          *p = v;
          C[static_cast<size_t>(col) * ldc + row] = v;
        } else {
          double* p = C + static_cast<size_t>(row) * ldc + col;
          *p = (accumulate ? *p : 0.0) + acc[mt][nt][i];
        }
      }
}

// Deterministic sum of one double per thread: a fixed shuffle tree per warp, then the warps in ascending order.
__device__ double BlockSum(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double r = 0.0;
  if (threadIdx.x == 0)
    for (int i = 0; i < kSweepThreads / 32; i++) r += red[i];
  return r;
}

// loss partials: CTA b sums E * GE (kTarget: E * (P + GE)) over a fixed range of kLossBlocks equal ranges
template <bool kTarget>
__global__ void __launch_bounds__(kSweepThreads) pqr_loss_partial_kernel(const double* __restrict__ E, const double* __restrict__ GE,
                                                                         const double* __restrict__ P, size_t n,
                                                                         double* __restrict__ part) {
  __shared__ double red[kSweepThreads / 32];
  const size_t chunk = (n + kLossBlocks - 1) / kLossBlocks, b0 = blockIdx.x * chunk, b1 = min(n, b0 + chunk);
  double v = 0.0;
  for (size_t i = b0 + threadIdx.x; i < b1; i += kSweepThreads) v += kTarget ? E[i] * (P[i] + GE[i]) : E[i] * GE[i];
  const double tot = BlockSum(v, red);
  if (threadIdx.x == 0) part[blockIdx.x] = tot;
}

// partials of |t|^2 = sum of fp32 squares in fp64, over the same fixed ranges (exact products, so no overflow)
__global__ void __launch_bounds__(kSweepThreads) pqr_sqnorm_partial_kernel(const float* __restrict__ t, size_t n,
                                                                           double* __restrict__ part) {
  __shared__ double red[kSweepThreads / 32];
  const size_t chunk = (n + kLossBlocks - 1) / kLossBlocks, b0 = blockIdx.x * chunk, b1 = min(n, b0 + chunk);
  double v = 0.0;
  for (size_t i = b0 + threadIdx.x; i < b1; i += kSweepThreads) {
    const double x = static_cast<double>(t[i]);
    v += x * x;
  }
  const double tot = BlockSum(v, red);
  if (threadIdx.x == 0) part[blockIdx.x] = tot;
}

// *loss = the partials' sum (kTarget: *tt plus it)
template <bool kTarget>
__global__ void __launch_bounds__(kSweepThreads) pqr_loss_final_kernel(const double* __restrict__ part, const double* __restrict__ tt,
                                                                       double* __restrict__ loss) {
  __shared__ double red[kSweepThreads / 32];
  double v = 0.0;
  for (int i = threadIdx.x; i < kLossBlocks; i += kSweepThreads) v += part[i];
  const double tot = BlockSum(v, red);
  if (threadIdx.x == 0) *loss = kTarget ? *tt + tot : tot;
}

// loss = sum E * GE over n elements, in a fixed order, written to *loss.  With a target (P non-null):
// loss = *tt + sum E * (P + GE), which for E = -W^, P = T^T Y and GE = P + E G is |T|^2 - 2 sum W^ . P + sum W^ . G W^.
inline int LaunchLoss(const double* E, const double* GE, size_t n, double* part, double* loss, cudaStream_t st,
                      const double* P = nullptr, const double* tt = nullptr) {
  if (P) {
    pqr_loss_partial_kernel<true><<<kLossBlocks, kSweepThreads, 0, st>>>(E, GE, P, n, part);
    pqr_loss_final_kernel<true><<<1, kSweepThreads, 0, st>>>(part, tt, loss);
  } else {
    pqr_loss_partial_kernel<false><<<kLossBlocks, kSweepThreads, 0, st>>>(E, GE, nullptr, n, part);
    pqr_loss_final_kernel<false><<<1, kSweepThreads, 0, st>>>(part, nullptr, loss);
  }
  QCNN_CUDA(cudaGetLastError());
  return 0;
}

// *tt = the partials' sum (accumulate: *tt plus it), in pqr_loss_final_kernel's order
__global__ void __launch_bounds__(kSweepThreads) pqr_sqnorm_final_kernel(const double* __restrict__ part, double* __restrict__ tt,
                                                                         int accumulate) {
  __shared__ double red[kSweepThreads / 32];
  double v = 0.0;
  for (int i = threadIdx.x; i < kLossBlocks; i += kSweepThreads) v += part[i];
  const double tot = BlockSum(v, red);
  if (threadIdx.x == 0) *tt = accumulate ? *tt + tot : tot;
}

// *tt (accumulate: *tt +) |t|^2 over n fp32 values in a fixed order; part holds kLossBlocks doubles
inline int LaunchSqNorm(const float* t, size_t n, double* part, double* tt, int accumulate, cudaStream_t st) {
  pqr_sqnorm_partial_kernel<<<kLossBlocks, kSweepThreads, 0, st>>>(t, n, part);
  pqr_sqnorm_final_kernel<<<1, kSweepThreads, 0, st>>>(part, tt, accumulate);
  QCNN_CUDA(cudaGetLastError());
  return 0;
}

// *first = min(*first, the column i % cols of every non-finite x[i]); *first starts at 0xffffffff (none)
__global__ void pqr_nonfinite_kernel(const float* __restrict__ x, size_t n, unsigned cols, unsigned* __restrict__ first) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x)
    if (!isfinite(x[i])) atomicMin(first, static_cast<unsigned>(i % cols));
}

constexpr unsigned kNoneFound = 0xffffffffu;

// An add's scan, ordered after the earlier adds of s: first[0] = the lowest column (index mod ycols) of a NaN or Inf in
// y, first[1] = 0 if t (when given) holds one, kNoneFound otherwise.  One synchronisation of st.
inline int ScanAdd(qcnn_pq_stats* s, const float* y, size_t ny, unsigned ycols, const float* t, size_t nt, unsigned first[2],
                   cudaStream_t st) {
  QCNN_ON_DEVICE(s->ctx->device);
  unsigned* flags = reinterpret_cast<unsigned*>(s->scratch.as<double>() + kLossBlocks);
  QCNN_CUDA(cudaStreamWaitEvent(st, s->done, 0));
  QCNN_CUDA(cudaMemsetAsync(flags, 0xff, 2 * sizeof(unsigned), st));
  auto scan = [&](const float* v, size_t n, unsigned cols, unsigned* flag) {
    const int grid = static_cast<int>(std::min<size_t>((n + 255) / 256, 32u * s->ctx->sm_count));
    pqr_nonfinite_kernel<<<grid, 256, 0, st>>>(v, n, cols, flag);
  };
  scan(y, ny, ycols, flags);
  if (t) scan(t, nt, 1, flags + 1);
  QCNN_CUDA(cudaGetLastError());
  QCNN_CUDA(cudaMemcpyAsync(first, flags, 2 * sizeof(unsigned), cudaMemcpyDeviceToHost, st));
  QCNN_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// Makes b hold at least bytes on ctx's device; on failure sets who's error, which names what the buffer is for
inline int Reserve(qcnn_ctx* ctx, const char* who, qcnn::DeviceBuffer& b, size_t bytes, const char* what) {
  const cudaError_t e = b.Reserve(ctx, bytes);
  if (e == cudaSuccess) return 0;
  cudaGetLastError();
  qcnn::SetError("%s: cannot allocate %zu bytes of device memory for %s (%s)", who, bytes, what, cudaGetErrorString(e));
  return 1;
}

// A statistics object of either kind with its sums zero until the first add: G [grp][Dg][Dg], for a target P [Cout][Dg]
// and |T|^2, the scratch and the event.  sums: also the first moments, s [grp][Dg] and for a target u [Cout], and for
// conv the per-add plane (FC: none).
inline int CreateStats(qcnn_ctx* ctx, const char* who, bool conv, const qcnn::PqGeometry& geo, int d, bool target, bool sums,
                       qcnn_pq_stats** out) {
  std::unique_ptr<qcnn_pq_stats> s(new qcnn_pq_stats);
  s->ctx = ctx;
  s->conv = conv;
  s->target = target;
  s->d = d;
  s->geo = geo;
  s->sums = sums;
  const size_t gBytes = sizeof(double) * geo.grp * static_cast<size_t>(geo.Dg) * geo.Dg;
  const size_t pBytes = target ? sizeof(double) * geo.Cout * static_cast<size_t>(geo.Dg) : 0;
  const size_t syBytes = sums ? sizeof(double) * geo.grp * static_cast<size_t>(geo.Dg) : 0;
  const size_t suBytes = sums && target ? sizeof(double) * geo.Cout : 0;
  const size_t inPlane = static_cast<size_t>(geo.Hin) * geo.Win * geo.Cin, outPlane = static_cast<size_t>(geo.Ho) * geo.Wo * geo.Cout;
  const size_t planeBytes = sums && conv ? sizeof(double) * (target ? std::max(inPlane, outPlane) : inPlane) : 0;
  if (Reserve(ctx, who, s->G, gBytes, "the Gram matrices") || Reserve(ctx, who, s->P, pBytes, "the targets' cross product") ||
      Reserve(ctx, who, s->tt, target ? sizeof(double) : 0, "the targets' norm") ||
      Reserve(ctx, who, s->sy, syBytes, "the inputs' sum") || Reserve(ctx, who, s->su, suBytes, "the targets' sum") ||
      Reserve(ctx, who, s->plane, planeBytes, "the per-add image sum") ||
      Reserve(ctx, who, s->scratch, sizeof(double) * kLossBlocks + 2 * sizeof(unsigned), "the scan flags"))
    return 1;
  QCNN_ON_DEVICE(ctx->device);
  QCNN_CUDA(cudaEventCreateWithFlags(&s->done, cudaEventDisableTiming));
  QCNN_CUDA(cudaMemset(s->G.get(), 0, gBytes));
  if (target) {
    QCNN_CUDA(cudaMemset(s->P.get(), 0, pBytes));
    QCNN_CUDA(cudaMemset(s->tt.get(), 0, sizeof(double)));
  }
  if (syBytes) QCNN_CUDA(cudaMemset(s->sy.get(), 0, syBytes));
  if (suBytes) QCNN_CUDA(cudaMemset(s->su.get(), 0, suBytes));
  QCNN_CUDA(cudaEventRecord(s->done, nullptr));
  *out = s.release();
  return 0;
}

// ---- first moments and the bias refit (DESIGN.md 4e, "Bias refit")

// The rows n the first moments are summed over: images Ho Wo (FC: images)
inline long long StatsRows(const qcnn_pq_stats* s) { return s->images * s->geo.Ho * s->geo.Wo; }

// out[c] = (accumulate ? out[c] + f : f), f = sum over r = 0..rows-1 ascending of x[r cols + c] in fp64: one fresh
// fixed-order sum per column, folded with one addition
template <typename In>
__global__ void pqr_colsum_kernel(const In* __restrict__ x, size_t rows, size_t cols, double* __restrict__ out, int accumulate) {
  for (size_t c = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; c < cols; c += static_cast<size_t>(gridDim.x) * blockDim.x) {
    double f = 0.0;
    for (size_t r = 0; r < rows; r++) f += static_cast<double>(x[r * cols + c]);
    out[c] = accumulate ? out[c] + f : f;
  }
}

template <typename In>
inline int LaunchColSum(qcnn_ctx* ctx, const In* x, size_t rows, size_t cols, double* out, int accumulate, cudaStream_t st) {
  const int grid = static_cast<int>(std::min<size_t>((cols + 255) / 256, 32u * ctx->sm_count));
  pqr_colsum_kernel<In><<<grid, 256, 0, st>>>(x, rows, cols, out, accumulate);
  QCNN_CUDA(cudaGetLastError());
  return 0;
}

// out[r][c] = X[r][c] - (a[r] b[r / rpg][c]) / n, each operation rounded (no contraction): the centered G (a = s,
// b = s per group) and P (a = u, b = s of the output's group)
__global__ void pqr_center_kernel(const double* __restrict__ X, const double* __restrict__ a, const double* __restrict__ b,
                                  size_t rows, size_t cols, size_t rpg, double n, double* __restrict__ out) {
  const size_t total = rows * cols;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t r = i / cols, c = i % cols;
    out[i] = __dsub_rn(X[i], __ddiv_rn(__dmul_rn(a[r], b[(r / rpg) * cols + c]), n));
  }
}

// *ttc = *tt - sum over o ascending of (u[o] u[o]) / n, each operation rounded
__global__ void pqr_center_tt_kernel(const double* __restrict__ tt, const double* __restrict__ u, int Dout, double n,
                                     double* __restrict__ ttc) {
  double acc = 0.0;
  for (int o = 0; o < Dout; o++) acc = __dadd_rn(acc, __ddiv_rn(__dmul_rn(u[o], u[o]), n));
  *ttc = __dsub_rn(*tt, acc);
}

// delta[o] = (u[o] + E_o . s_g) / n, g = o / Cpg, u = 0 without a target (E = W - W^, or -W^ for the target form): a
// warp per output, lanes over every 32nd dim, a fixed shuffle tree
__global__ void pqr_bias_delta_kernel(const double* __restrict__ E, const double* __restrict__ sy, const double* __restrict__ u,
                                      int Dout, int D, int Cpg, double n, double* __restrict__ delta) {
  const int lane = threadIdx.x & 31;
  const int o = static_cast<int>((blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x) >> 5);
  if (o >= Dout) return;
  const double* e = E + static_cast<size_t>(o) * D;
  const double* sg = sy + static_cast<size_t>(o / Cpg) * D;
  double v = 0.0;
  for (int q = lane; q < D; q += 32) v += e[q] * sg[q];
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  if (lane == 0) delta[o] = __ddiv_rn(u ? __dadd_rn(u[o], v) : v, n);
}

// The centered copies of a stats object's sums: G [grp][Dg][Dg] always, P [Cout][Dg] and |T_c|^2 for the target form
// (DampSums also damps them in place, or holds its damped copies of the raw sums here)
struct CenteredSums {
  qcnn::DeviceBuffer G, P, tt;
};

inline int CenterSums(qcnn_pq_stats* s, const char* who, bool target, CenteredSums* c, cudaStream_t st) {
  qcnn_ctx* ctx = s->ctx;
  const int grp = s->geo.grp, D = s->geo.Dg, Dout = s->geo.Cout;
  const size_t gn = static_cast<size_t>(grp) * D * D, pn = static_cast<size_t>(Dout) * D;
  if (Reserve(ctx, who, c->G, sizeof(double) * gn, "the centered Gram matrices") ||
      Reserve(ctx, who, c->P, target ? sizeof(double) * pn : 0, "the centered cross product") ||
      Reserve(ctx, who, c->tt, target ? sizeof(double) : 0, "the centered targets' norm"))
    return 1;
  QCNN_ON_DEVICE(ctx->device);
  QCNN_CUDA(cudaStreamWaitEvent(st, s->done, 0));
  const double n = static_cast<double>(StatsRows(s));
  const double* sy = s->sy.as<double>();
  auto grid = [&](size_t total) { return static_cast<int>(std::min<size_t>((total + 255) / 256, 32u * ctx->sm_count)); };
  pqr_center_kernel<<<grid(gn), 256, 0, st>>>(s->G.as<double>(), sy, sy, static_cast<size_t>(grp) * D, D, D, n, c->G.as<double>());
  if (target) {
    const double* su = s->su.as<double>();
    pqr_center_kernel<<<grid(pn), 256, 0, st>>>(s->P.as<double>(), su, sy, Dout, D, Dout / grp, n, c->P.as<double>());
    pqr_center_tt_kernel<<<1, 1, 0, st>>>(s->tt.as<double>(), su, Dout, n, c->tt.as<double>());
  }
  QCNN_CUDA(cudaGetLastError());
  return 0;
}

// ---- damping toward the original weights (DESIGN.md 4e, "Damping toward the original weights")

constexpr int kTraceChunk = 1024;   // diagonal entries staged per step of pqr_damp_lambda_kernel

// Per group g (blockIdx.x): lam[g] = damp (tr_g / Dg), tr_g = the sum over i ascending of G_g[i][i], every operation
// rounded; 0 when !(tr_g > 0).  The block stages the strided diagonal in chunks, thread 0 adds them in order.
__global__ void __launch_bounds__(kSweepThreads) pqr_damp_lambda_kernel(const double* __restrict__ G, int Dg, double damp,
                                                                        double* __restrict__ lam) {
  __shared__ double diag[kTraceChunk];
  const double* Gg = G + static_cast<size_t>(blockIdx.x) * Dg * Dg;
  double tr = 0.0;
  for (int i0 = 0; i0 < Dg; i0 += kTraceChunk) {
    const int n = min(kTraceChunk, Dg - i0);
    for (int i = threadIdx.x; i < n; i += kSweepThreads) diag[i] = Gg[static_cast<size_t>(i0 + i) * (Dg + 1)];
    __syncthreads();
    if (threadIdx.x == 0)
      for (int i = 0; i < n; i++) tr = __dadd_rn(tr, diag[i]);
    __syncthreads();
  }
  if (threadIdx.x == 0) lam[blockIdx.x] = tr > 0.0 ? __dmul_rn(damp, __ddiv_rn(tr, static_cast<double>(Dg))) : 0.0;
}

// The damped copies, elementwise with every operation rounded; X and out may be the same array.
//   W NULL:  the diagonals, out[g][i][i] = X[g][i][i] + lam[g] over rows = grp Dg entries (rpg = Dg, cols = Dg).
//   else:    out[o][q] = X[o][q] + lam[o / rpg] W[o][q] over rows = Cout outputs of cols = Dg dims (rpg = Cpg).
__global__ void pqr_damp_kernel(const double* X, const float* __restrict__ W, const double* __restrict__ lam, size_t rows,
                                size_t cols, size_t rpg, double* out) {
  const size_t total = W ? rows * cols : rows;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    if (W) {
      out[i] = __dadd_rn(X[i], __dmul_rn(lam[i / cols / rpg], static_cast<double>(W[i])));
    } else {
      const size_t e = (i / rpg) * rpg * cols + (i % rpg) * (cols + 1);   // group i / Dg, diagonal entry i % Dg
      out[e] = __dadd_rn(X[e], lam[i / rpg]);
    }
  }
}

// *ttd = *tt + sum over g ascending of lam[g] wsq[g], every operation rounded (*ttd may be *tt)
__global__ void pqr_damp_tt_kernel(const double* tt, const double* __restrict__ lam, const double* __restrict__ wsq, int grp,
                                   double* ttd) {
  double acc = 0.0;
  for (int g = 0; g < grp; g++) acc = __dadd_rn(acc, __dmul_rn(lam[g], wsq[g]));
  *ttd = __dadd_rn(*tt, acc);
}

// The damped copies of the sums G, P and TT the sweeps would otherwise read (the statistics' own, or c's centered
// copies): per group lam_g from G's trace, G' = G + lam_g I, and for the target form P' = P + lam_g W (g the output's
// group) and |T'|^2 = |T|^2 + sum_g lam_g |W_g|^2, w_h the host weights [Cout][Dg] in the internal dim order.  They are
// written to c: in place when the base sums are c's, otherwise into c's buffers, reserved here.  Synchronises st.
inline int DampSums(qcnn_pq_stats* s, const char* who, bool target, double damp, const float* w_h, const double* G,
                    const double* P, const double* TT, CenteredSums* c, cudaStream_t st) {
  qcnn_ctx* ctx = s->ctx;
  const int grp = s->geo.grp, D = s->geo.Dg, Dout = s->geo.Cout, Cpg = s->geo.Cpg;
  const size_t gn = static_cast<size_t>(grp) * D * D, pn = static_cast<size_t>(Dout) * D;
  qcnn::DeviceBuffer scratch, dW;   // lam [grp], |W_g|^2 [grp], the |W_g|^2 partials [kLossBlocks]; the weights
  if (Reserve(ctx, who, c->G, sizeof(double) * gn, "the damped Gram matrices") ||
      Reserve(ctx, who, c->P, target ? sizeof(double) * pn : 0, "the damped cross product") ||
      Reserve(ctx, who, c->tt, target ? sizeof(double) : 0, "the damped targets' norm") ||
      Reserve(ctx, who, scratch, sizeof(double) * (2 * grp + kLossBlocks), "the damping weights") ||
      Reserve(ctx, who, dW, target ? sizeof(float) * pn : 0, "the weights"))
    return 1;
  QCNN_ON_DEVICE(ctx->device);
  QCNN_CUDA(cudaStreamWaitEvent(st, s->done, 0));
  double *lam = scratch.as<double>(), *wsq = lam + grp, *part = wsq + grp;
  auto grid = [&](size_t total) { return static_cast<int>(std::min<size_t>((total + 255) / 256, 32u * ctx->sm_count)); };
  pqr_damp_lambda_kernel<<<grp, kSweepThreads, 0, st>>>(G, D, damp, lam);
  double* Gd = c->G.as<double>();
  if (Gd != G) QCNN_CUDA(cudaMemcpyAsync(Gd, G, sizeof(double) * gn, cudaMemcpyDeviceToDevice, st));
  pqr_damp_kernel<<<grid(static_cast<size_t>(grp) * D), 256, 0, st>>>(Gd, nullptr, lam, static_cast<size_t>(grp) * D, D, D, Gd);
  QCNN_CUDA(cudaGetLastError());
  if (target) {
    QCNN_CUDA(cudaMemcpyAsync(dW.get(), w_h, sizeof(float) * pn, cudaMemcpyHostToDevice, st));
    pqr_damp_kernel<<<grid(pn), 256, 0, st>>>(P, dW.as<float>(), lam, Dout, D, Cpg, c->P.as<double>());
    for (int g = 0; g < grp; g++)
      if (int rc = LaunchSqNorm(dW.as<float>() + static_cast<size_t>(g) * Cpg * D, static_cast<size_t>(Cpg) * D, part, wsq + g, 0,
                                st))
        return rc;
    pqr_damp_tt_kernel<<<1, 1, 0, st>>>(TT, lam, wsq, grp, c->tt.as<double>());
    QCNN_CUDA(cudaGetLastError());
  }
  QCNN_CUDA(cudaStreamSynchronize(st));   // scratch and dW are freed on return
  return 0;
}

// bias_h[o] = fp32(bias_h[o] + delta_o) from the final residual E [Cout][Dg] on the device (pqr_bias_delta_kernel)
inline int RefitBias(qcnn_pq_stats* s, const char* who, bool target, const double* E, float* bias_h, cudaStream_t st) {
  const int Dout = s->geo.Cout;
  qcnn::DeviceBuffer dDelta;
  if (Reserve(s->ctx, who, dDelta, sizeof(double) * Dout, "the bias change")) return 1;
  pqr_bias_delta_kernel<<<qcnn::CeilDiv(Dout, 8), 256, 0, st>>>(E, s->sy.as<double>(), target ? s->su.as<double>() : nullptr, Dout,
                                                                s->geo.Dg, s->geo.Cpg, static_cast<double>(StatsRows(s)),
                                                                dDelta.as<double>());
  QCNN_CUDA(cudaGetLastError());
  std::vector<double> delta(Dout);
  QCNN_CUDA(cudaMemcpyAsync(delta.data(), dDelta.get(), sizeof(double) * Dout, cudaMemcpyDeviceToHost, st));
  QCNN_CUDA(cudaStreamSynchronize(st));
  for (int o = 0; o < Dout; o++) bias_h[o] = static_cast<float>(static_cast<double>(bias_h[o]) + delta[o]);
  return 0;
}

// ---- the start and the end of the sweeps (SweepFc, SweepConv)

bool AllFinite(const float* v, size_t n) {
  for (size_t i = 0; i < n; i++)
    if (!isfinite(v[i])) return false;
  return true;
}

// A refine's start as the sweeps read it: at, the assignments [Cout][T][S] as [S][Cout][T], and w, the weights
// [Cout][Cg][T] in the internal dim order (NULL when the call takes none; the target form reads them only to damp P):
// the caller's own array when T == 1, where the two orders agree, else the permuted copy wp
struct Start {
  std::vector<uint8_t> at;
  std::vector<float> wp;
  const float* w = nullptr;
};

// The host-side checks of a refine (weights when given, codebook, assignments; the FC message names no tap), then
// the start.  Both forms go through the same checks: the target calls pass w_h NULL, the damped call its anchor.
inline int CheckStart(const char* who, bool conv, const qcnn::PqGeometry& geo, int K, int d, const float* w_h,
                      const float* ctrd_h, const uint8_t* asmt_h, Start* start) {
  const int Cout = geo.Cout, Cg = geo.Cg, T = geo.T, Dg = geo.Dg, S = qcnn::CeilDiv(Cg, d);
  const size_t nw = static_cast<size_t>(Cout) * Dg, nc = static_cast<size_t>(S) * K * d;
  if (w_h) QCNN_CHECK(AllFinite(w_h, nw), "%s: the weights contain a non-finite value", who);
  QCNN_CHECK(AllFinite(ctrd_h, nc), "%s: the codebook contains a non-finite value", who);
  start->at.assign(static_cast<size_t>(S) * Cout * T, 0);
  for (int o = 0; o < Cout; o++)
    for (int t = 0; t < T; t++)
      for (int m = 0; m < S; m++) {
        const uint8_t a = asmt_h[(static_cast<size_t>(o) * T + t) * S + m];
        QCNN_CHECK(a < K || conv, "%s: assignment %d of output %d, subspace %d is not below K=%d", who, a, o, m, K);
        QCNN_CHECK(a < K, "%s: assignment %d of output %d, tap %d, subspace %d is not below K=%d", who, a, o, t, m, K);
        start->at[(static_cast<size_t>(m) * Cout + o) * T + t] = a;
      }
  start->w = w_h;
  if (!w_h || T == 1) return 0;
  start->wp.resize(nw);
  for (int o = 0; o < Cout; o++)
    for (int c = 0; c < Cg; c++) {
      const int m = c / d, j = c % d, w = std::min(d, Cg - m * d);
      for (int t = 0; t < T; t++)
        start->wp[static_cast<size_t>(o) * Dg + m * d * T + t * w + j] = w_h[(static_cast<size_t>(o) * Cg + c) * T + t];
    }
  start->w = start->wp.data();
  return 0;
}

// What both sweep loops share: the residual E [Cout][Dg] = W - W^ in fp64 (target form: the weights are zeros, so
// E = -W^), GE = E G per group (target: P + E G), the weights, codebook and assignments on the device, and the losses.
// G, P and TT are the sums the sweeps run on (P and TT NULL in the same-input form); at is the start's assignments.
struct SweepState {
  qcnn_pq_stats* s;
  const char* who;
  bool target;
  int K, sweeps;
  const double *G, *P, *TT;
  std::vector<uint8_t>* at;
  size_t nw, nc;
  qcnn::DeviceBuffer E, GE, W, C, A, part, loss;

  void Residual(cudaStream_t st) {   // E afresh from W, C and A
    const qcnn::PqGeometry& geo = s->geo;
    const int grid = static_cast<int>(std::min<size_t>((nw + 255) / 256, 32u * s->ctx->sm_count));
    pqrc_residual_kernel<<<grid, 256, 0, st>>>(W.as<float>(), C.as<float>(), A.as<uint8_t>(), E.as<double>(), geo.Cout, geo.Cg, K,
                                               s->d, geo.T);
  }
  int Loss(int sw, cudaStream_t st) {   // loss[sw] from E and GE
    return LaunchLoss(E.as<double>(), GE.as<double>(), nw, part.as<double>(), loss.as<double>() + sw, st, P, TT);
  }
};

// The set-up of the sweeps on s's current device: reserves the shared buffers, uploads the weights w (zeros for the
// target form), the codebook and the assignments at, forms E, seeds GE per group and writes loss[0]
inline int BeginSweeps(SweepState* ss, qcnn_pq_stats* s, const char* who, bool target, int K, int sweeps, const float* w,
                       std::vector<uint8_t>& at, const float* ctrd_h, const double* G, const double* P, const double* TT,
                       cudaStream_t st) {
  qcnn_ctx* ctx = s->ctx;
  const qcnn::PqGeometry& geo = s->geo;
  const int Cpg = geo.Cpg, Dg = geo.Dg;
  const size_t nw = static_cast<size_t>(geo.Cout) * Dg, nc = static_cast<size_t>(qcnn::CeilDiv(geo.Cg, s->d)) * K * s->d;
  ss->s = s;
  ss->who = who;
  ss->target = target;
  ss->K = K;
  ss->sweeps = sweeps;
  ss->G = G;
  ss->P = target ? P : nullptr;   // P = T^T Y
  ss->TT = target ? TT : nullptr;
  ss->at = &at;
  ss->nw = nw;
  ss->nc = nc;
  if (Reserve(ctx, who, ss->E, sizeof(double) * nw, "the residual") ||
      Reserve(ctx, who, ss->GE, sizeof(double) * nw, "G times the residual") ||
      Reserve(ctx, who, ss->W, sizeof(float) * nw, "the weights") || Reserve(ctx, who, ss->C, sizeof(float) * nc, "the codebook") ||
      Reserve(ctx, who, ss->A, at.size(), "the assignments") ||
      Reserve(ctx, who, ss->part, sizeof(double) * kLossBlocks, "the loss") ||
      Reserve(ctx, who, ss->loss, sizeof(double) * (sweeps + 1), "the loss"))
    return 1;
  QCNN_CUDA(cudaStreamWaitEvent(st, s->done, 0));
  if (target) QCNN_CUDA(cudaMemsetAsync(ss->W.get(), 0, sizeof(float) * nw, st));   // E = 0 - W^
  else QCNN_CUDA(cudaMemcpyAsync(ss->W.get(), w, sizeof(float) * nw, cudaMemcpyHostToDevice, st));
  QCNN_CUDA(cudaMemcpyAsync(ss->C.get(), ctrd_h, sizeof(float) * nc, cudaMemcpyHostToDevice, st));
  QCNN_CUDA(cudaMemcpyAsync(ss->A.get(), at.data(), at.size(), cudaMemcpyHostToDevice, st));
  ss->Residual(st);
  // GE = E G, or P + E G for a target
  if (target) QCNN_CUDA(cudaMemcpyAsync(ss->GE.get(), P, sizeof(double) * nw, cudaMemcpyDeviceToDevice, st));
  for (int g = 0; g < geo.grp; g++) {
    const size_t ro = static_cast<size_t>(g) * Cpg * Dg;
    pqr_gemm_kernel<kGemmF64><<<dim3(qcnn::CeilDiv(Dg, kTile), qcnn::CeilDiv(Cpg, kTile)), kGemmThreads, 0, st>>>(
        ss->E.as<double>() + ro, Dg, G + static_cast<size_t>(g) * Dg * Dg, Dg, ss->GE.as<double>() + ro, Dg, Cpg, Dg, Dg, target);
  }
  QCNN_CUDA(cudaGetLastError());
  return ss->Loss(0, st);
}

// The end of the sweeps: with bias_h, E afresh from the final codebook and assignments (target: -W^) and the bias refit;
// then the codebook, the assignments in the caller's layout [Cout][T][S] and the losses to the host
inline int EndSweeps(SweepState& ss, float* ctrd_h, uint8_t* asmt_h, float* bias_h, double* loss_h, cudaStream_t st) {
  if (bias_h) {
    ss.Residual(st);
    if (int rc = RefitBias(ss.s, ss.who, ss.target, ss.E.as<double>(), bias_h, st)) return rc;
  }
  const qcnn::PqGeometry& geo = ss.s->geo;
  const int Cout = geo.Cout, T = geo.T, S = qcnn::CeilDiv(geo.Cg, ss.s->d);
  std::vector<uint8_t>& at = *ss.at;
  std::vector<double> lossv(ss.sweeps + 1);
  QCNN_CUDA(cudaMemcpyAsync(ctrd_h, ss.C.get(), sizeof(float) * ss.nc, cudaMemcpyDeviceToHost, st));
  QCNN_CUDA(cudaMemcpyAsync(at.data(), ss.A.get(), at.size(), cudaMemcpyDeviceToHost, st));
  QCNN_CUDA(cudaMemcpyAsync(lossv.data(), ss.loss.get(), sizeof(double) * lossv.size(), cudaMemcpyDeviceToHost, st));
  QCNN_CUDA(cudaStreamSynchronize(st));
  for (int o = 0; o < Cout; o++)
    for (int t = 0; t < T; t++)
      for (int m = 0; m < S; m++) asmt_h[(static_cast<size_t>(o) * T + t) * S + m] = at[(static_cast<size_t>(m) * Cout + o) * T + t];
  if (loss_h) std::copy(lossv.begin(), lossv.end(), loss_h);
  return 0;
}

}  // namespace

#endif  // QCNN_PQ_REFINE_COMMON_CUH_
