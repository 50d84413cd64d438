// Latency path of the PQ fully-connected layers (batch 1..4): ONE persistent launch for a whole run of consecutive FC
// layers (AlexNet: fc6 -> ReLU -> fc7 -> ReLU -> fc8), bound by the HBM stream of the uint8 assignment matrices.
// Replaces CaffeEva::CalcFeatMap_FCntAprx + GetInPdMat (reference src/CaffeEva.cc:968-1025, 1261-1296) for each layer:
//     LUT[s][k] = sum_j x[s*d+j] * ctrd[s][k][j]            (ascending j, rounded mul then rounded add)
//     dst[o]    = bias[o] + sum_s LUT[s][asmt[s][o]]
//
// Design (one CTA per SM, cooperative launch so that all CTAs are co-resident):
//   * the subspaces (rows of the device assignment table [S][DoutPad]) of EVERY layer are split evenly over the CTAs,
//     so a CTA's share of a layer is one contiguous block of bytes.  A producer warp streams these blocks -- all
//     layers back to back, it never waits for the arithmetic -- into a shared-memory ring with cp.async.bulk
//     (mbarrier complete_tx); with ~150 KB of ring per SM the whole 17.7 MB of AlexNet's three FC layers is in flight
//     from the first cycle of the kernel, so the HBM stream is not interrupted by the layer-to-layer dependency.
//   * a CTA builds only the LUT rows of its own subspaces (its share of the codebook, one CTA per SM, arrives by one bulk copy), then
//     512 consumer threads gather: thread = 4/8/16 consecutive output channels, one 32/64/128-bit shared-memory load
//     of assignment bytes per row, LUT row = one bank sweep for K <= 32 (conflict-free by construction).
//   * a CTA's result is a partial sum over ITS subspaces for ALL output channels.  It is published to an L2-resident
//     buffer [CTA][DoutPad]; the word itself is the ready flag (the buffer holds a NaN pattern no arithmetic produces
//     until it is written, and the one consumer of a word resets it), so there is no grid barrier, no fence and no
//     atomic between the layers: the consumer of the next layer polls exactly the 4-float groups it needs
//     (its own subspaces' inputs), lanes over the producing CTAs, and reduces them with a fixed shuffle tree
//     (deterministic; bias and ReLU are applied there).  The last layer's partials are reduced the same way, eight
//     output channels per CTA.
// Accumulation order: per CTA s ascending, then CTAs in a fixed tree -- a re-association of the reference's
// bias + s-ascending sum (fp32 adds only; tolerance in tests/test_gpu_layers.py).  fc_nsplit = 1 keeps the bit-exact kernel.
#include "qcnn_internal.h"
#include "async_copy.h"
#include "packed_asmt.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace {

using qcnn::BulkLoad;
using qcnn::MbarArrive;
using qcnn::MbarExpectTx;
using qcnn::MbarInit;
using qcnn::MbarWait;   // the chain's waits trap after 2^26 polls
using qcnn::SmemU32;

constexpr int kConsumers = 512;
constexpr int kConsumerWarps = kConsumers / 32;
constexpr int kThreads = kConsumers + 32;
constexpr int kMaxChain = 4;
constexpr int kMaxParts = 160;       // 5 polls per lane
constexpr int kMaxStage = 32;
constexpr int kChunkBytes = 16384;
constexpr int kBarBytes = 1024;      // mbarrier block at the start of shared memory
constexpr uint32_t kSentinel = 0xFFFFFFFFu;

struct ChainLayer {
  const float* ctrd;      // [S][K][d]
  const uint8_t* asmt;    // [S][DoutPad], stored byte = idx << kshift
  const float* bias;
  const int* srcoff;      // first layer only: flattened feature -> source element offset (NULL: identity / arithmetic fold)
  float* partial;         // [G][DoutPad]
  int Din, Dout, DoutPad, S, K, d;
  int log2K;
  int pre;                // stored byte = byte offset inside a LUT row (K <= 64)
  int lutPitch;           // bytes per LUT row in shared memory (256 when pre, else 4 K)
  int unit, unitsBase, unitsRem;   // subspace split in units of `unit` rows
  int cpt, tpr, rg;       // channels per thread, threads per row, row groups
  float tprInv;           // 1 / tpr (host-verified: floor((tid + 0.5) * tprInv) == tid / tpr for all consumer threads)
  int rpc;                // rows per ring chunk
  int relu;               // ReLU on this layer's output
  int ctrdOff;            // float offset of the codebook slice in shared memory
  int srcHW, srcC;        // first layer reading an NHWC map: feature f = c * HW + pos lives at pos * C + c (0: not folded)
  float srcHWInv;         // 1 / HW (host-verified like tprInv)
};

struct ChainArgs {
  ChainLayer L[kMaxChain];
  const float* src;
  float* dst;
  unsigned long long* dbg;   // optional [G][32] stamps: [0],[1] %globaltimer at the CTA's first / last instruction; [2],[3] clock64
                             // there; [4 + 5 l + i] clock64 after phase i of layer l (input slice, LUT, first chunk, gather, publish)
  int nLayers, G, nStage;
  int cpcLast;               // output channels of the last layer reduced per CTA (multiple of 4)
  int xFloats, lutFloats, ctrdFloats, rgFloats, scrFloats, ringOff;
};

static_assert(8 * (2 * kMaxStage + kMaxChain) <= kBarBytes, "shared-memory header layout");

__device__ __forceinline__ void ConsumerSync() { asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory"); }
__device__ __forceinline__ unsigned long long GlobalTimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ uint4 LdRelaxed4(const float* p) {
  uint4 v;
  asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void StRelaxed4(float* p, float a, float b, float c, float d) {
  asm volatile("st.relaxed.gpu.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ bool Pending(const uint4& v) {
  return v.x == kSentinel || v.y == kSentinel || v.z == kSentinel || v.w == kSentinel;
}

// subspaces [r0, r1) of layer L owned by CTA c
__device__ __forceinline__ void RowRange(const ChainLayer& L, int c, int* r0, int* r1) {
  const int u0 = c * L.unitsBase + min(c, L.unitsRem);
  const int nu = L.unitsBase + (c < L.unitsRem ? 1 : 0);
  *r0 = min(L.S, u0 * L.unit);
  *r1 = min(L.S, (u0 + nu) * L.unit);
}

// Cross-CTA reduction of a slice of a layer's output: sums[j] = sum over the G producing CTAs of partial[p][f0 + j],
// j < 4 * ngroups (ngroups <= 16), by ALL consumer threads.  Returns (only in the threads with `*owner`) the sum of
// feature *fc.
//   pass 1  thread = (producer p, 4-float group g): consecutive lanes read consecutive 16-byte pieces of one producer's
//           row, so a warp touches a few 128-byte lines per load (a lane-per-producer mapping costs 32 lines per load
//           and blocks the load/store unit -- shared memory included -- for a microsecond).  Every word is polled
//           until it is written, parked in shared memory [p][4 GP + 4], then reset (armed for the next call).
//   pass 2  thread = (feature, chain c of 8): chain c adds producers c, c + 8, ... in ascending order, the eight chains
//           are combined by a fixed shuffle tree: deterministic, no atomics.
__device__ __forceinline__ float CollectSlice(float* partial, int pitch, int G, int f0, int ngroups, float* scr, int tid,
                                              int* fc, bool* owner, unsigned long long* dbg) {
  int log2GP = 0;
  while ((1 << log2GP) < ngroups) log2GP++;
  const int GP = 1 << log2GP, scrPitch = 4 * GP + 4;   // = 4 (mod 32) for GP >= 8: pass 2 is bank-conflict free
  const int g = tid & (GP - 1), p0 = tid >> log2GP, pstep = kConsumers >> log2GP;
  constexpr int NP = 5;    // passes over the producers: ceil(kMaxParts / (kConsumers / 16))
  if (dbg) dbg[0] = clock64();
  if (g < ngroups) {
    float* base = partial + static_cast<size_t>(p0) * pitch + f0 + 4 * g;
    const size_t dp = static_cast<size_t>(pstep) * pitch;
    uint4 v[NP];
#pragma unroll
    for (int j = 0; j < NP; j++) {
      if (p0 + j * pstep < G) v[j] = LdRelaxed4(base + j * dp);
      else v[j] = make_uint4(0u, 0u, 0u, 0u);
    }
    // words not written yet are polled again TOGETHER: one round trip after the slowest producer, not one per word
    for (uint32_t spins = 0;; spins++) {
      bool pend = false;
#pragma unroll
      for (int j = 0; j < NP; j++) pend = pend || Pending(v[j]);
      if (!pend) break;
      if (spins > (1u << 22)) __trap();     // seconds: a producer that never publishes is a bug, not something to wait for
#pragma unroll
      for (int j = 0; j < NP; j++)
        if (Pending(v[j])) v[j] = LdRelaxed4(base + j * dp);
    }
#pragma unroll
    for (int j = 0; j < NP; j++) {
      const int p = p0 + j * pstep;
      if (p < G) *reinterpret_cast<uint4*>(scr + p * scrPitch + 4 * g) = v[j];
    }
#pragma unroll
    for (int j = 0; j < NP; j++)      // armed for the next call (off the critical path: after the values are parked)
      if (p0 + j * pstep < G) *reinterpret_cast<uint4*>(base + j * dp) = make_uint4(kSentinel, kSentinel, kSentinel, kSentinel);
  }
  if (dbg) dbg[1] = clock64();
  ConsumerSync();
  const int f = tid >> 3, c = tid & 7;
  float s = 0.0f;
  if (f < 4 * ngroups) {
    constexpr int NQ = kMaxParts / 8;
    float t[NQ];
#pragma unroll
    for (int q = 0; q < NQ; q++) t[q] = (c + 8 * q < G) ? scr[(c + 8 * q) * scrPitch + f] : 0.0f;
#pragma unroll
    for (int q = 0; q < NQ; q++) s += t[q];      // producers c, c + 8, ... in ascending order (+0.0f past the last one)
  }
  s += __shfl_xor_sync(0xFFFFFFFFu, s, 4);
  s += __shfl_xor_sync(0xFFFFFFFFu, s, 2);
  s += __shfl_xor_sync(0xFFFFFFFFu, s, 1);
  if (dbg) dbg[2] = clock64();
  *fc = f;
  *owner = c == 0 && f < 4 * ngroups;
  return s;
}

// the 32-byte sectors CollectSlice will poll -- partial[p][f0 .. f0 + nf) of every producer p -- requested into L2 ahead of
// time by the (otherwise idle) producer warp: after an L2 flush the first poll would go to DRAM and back while the
// producers are already done
__device__ __forceinline__ void PrefetchSlice(const float* partial, int pitch, int G, int f0, int nf, int lane) {
  const int sectors = (nf + 7) >> 3;
  for (int i = lane; i < G * sectors; i += 32) {
    const int p = i / sectors, sct = i - p * sectors;
    asm volatile("prefetch.global.L2 [%0];" ::"l"(partial + static_cast<size_t>(p) * pitch + f0 + 8 * sct));
  }
}

template <int CPT> struct Idx;
template <> struct Idx<4>  { using type = uint32_t; };
template <> struct Idx<8>  { using type = uint2; };
template <> struct Idx<16> { using type = uint4; };
__device__ __forceinline__ uint32_t IdxWord(const uint32_t& v, int) { return v; }
__device__ __forceinline__ uint32_t IdxWord(const uint2& v, int i) { return i == 0 ? v.x : v.y; }
__device__ __forceinline__ uint32_t IdxWord(const uint4& v, int i) { return i == 0 ? v.x : (i == 1 ? v.y : (i == 2 ? v.z : v.w)); }

// not volatile: the compiler may schedule the lookups of several rows together (they only depend on the index words,
// which are loaded after the chunk's mbarrier wait)
__device__ __forceinline__ float LdShared(uint32_t addr) {
  float v;
  asm("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}

// the CPT lookups of one assignment row.  PRE: the stored byte is already the byte offset inside a LUT row (K <= 64) and
// LUT rows are 256-byte aligned, so ONE byte-permute both extracts the index and forms the shared-memory address:
// 3 instructions per lookup (PRMT, LDS, FADD).
template <int CPT, bool PRE, typename IV>
__device__ __forceinline__ void GatherRow(const IV& w, uint32_t lr, float (&acc)[CPT]) {
#pragma unroll
  for (int c = 0; c < CPT; c++) {
    uint32_t addr;
    if (PRE) addr = __byte_perm(IdxWord(w, c >> 2), lr, 0x7650u | (c & 3));          // (lr & ~0xFF) | byte
    else addr = lr + (__byte_perm(IdxWord(w, c >> 2), 0u, 0x4440u | (c & 3)) << 2);
    acc[c] += LdShared(addr);
  }
}

// the CPT lookups of one row of the bit-packed table (packed_asmt.h): w = the NW aligned words that cover the thread's
// CPT * B bits, the first one starting at bit `sh`.  The LUT row is at lr either way (PRE rows are 256 bytes apart).
template <int CPT, int B, int NW>
__device__ __forceinline__ void GatherRowPacked(const uint32_t (&w)[NW], uint32_t sh, uint32_t lr, float (&acc)[CPT]) {
  uint32_t idx[CPT];
  qcnn::UnpackFields<B, CPT, NW>(w, sh, idx);
#pragma unroll
  for (int c = 0; c < CPT; c++) acc[c] += LdShared(lr + (idx[c] << 2));
}
template <int NW>
__device__ __forceinline__ void LoadWords(const uint8_t* p, uint32_t (&w)[NW]) {
#pragma unroll
  for (int i = 0; i < NW; i++) w[i] = reinterpret_cast<const uint32_t*>(p)[i];
}

// Steps (3) and (4) of a layer for one consumer thread: gather-accumulate the CTA's assignment rows as their ring chunks
// arrive (thread = CPT consecutive channels of the rows rgIdx, rgIdx + rg, ...; four rows are in flight together), then
// publish the partial sums.  B < 8: the rows are bit-packed at B bits per index, packedPitch bytes apart in the ring (the row
// groups own the same rows as with the byte table, so the partial sums are the same).
template <int CPT, bool PRE, int B = 8>
__device__ __forceinline__ void GatherAndPublish(const ChainLayer& L, int rows, int nStage, uint64_t* fullB, uint64_t* emptyB,
                                                 const uint8_t* ring, const float* lut, float* rgred, float* out, int tid,
                                                 int lane, int* stagep, uint32_t* roundp, unsigned long long* dbg,
                                                 int packedPitch = 0) {
  using IV = typename Idx<CPT>::type;
  float acc[CPT];
#pragma unroll
  for (int c = 0; c < CPT; c++) acc[c] = 0.0f;
  const int rgIdx = __float2int_rd((static_cast<float>(tid) + 0.5f) * L.tprInv), cgIdx = tid - rgIdx * L.tpr;
  const bool active = rgIdx < L.rg;
  const int rowBytes = L.lutPitch, pitch = L.DoutPad, rg = L.rg;
  const uint32_t lutBase = SmemU32(lut);
  int stage = *stagep;
  uint32_t round = *roundp;
  for (int r = 0; r < rows; r += L.rpc) {
    MbarWait<26>(fullB + stage, round & 1u);
    if (dbg && tid == 0 && r == 0) dbg[0] = clock64();
    if constexpr (B < 8) {
      if (active) {
        constexpr int NW = qcnn::PackedSpan<B, CPT>::kWords;
        const uint32_t bit0 = static_cast<uint32_t>(cgIdx) * CPT * B, sh = bit0 & 31u;
        const uint8_t* chunk = ring + static_cast<size_t>(stage) * kChunkBytes + (bit0 >> 5) * 4;
        const int n = min(L.rpc, rows - r), pp = packedPitch;
        const uint32_t lr0 = lutBase + static_cast<uint32_t>(r) * rowBytes;
        int q = rgIdx;
        for (; q + 3 * rg < n; q += 4 * rg) {
          const uint8_t* p = chunk + static_cast<size_t>(q) * pp;
          uint32_t w0[NW], w1[NW], w2[NW], w3[NW];
          LoadWords(p, w0);
          LoadWords(p + static_cast<size_t>(rg) * pp, w1);
          LoadWords(p + static_cast<size_t>(2 * rg) * pp, w2);
          LoadWords(p + static_cast<size_t>(3 * rg) * pp, w3);
          const uint32_t lr = lr0 + static_cast<uint32_t>(q) * rowBytes, dl = static_cast<uint32_t>(rg) * rowBytes;
          GatherRowPacked<CPT, B>(w0, sh, lr, acc);
          GatherRowPacked<CPT, B>(w1, sh, lr + dl, acc);
          GatherRowPacked<CPT, B>(w2, sh, lr + 2 * dl, acc);
          GatherRowPacked<CPT, B>(w3, sh, lr + 3 * dl, acc);
        }
        for (; q < n; q += rg) {
          uint32_t w0[NW];
          LoadWords(chunk + static_cast<size_t>(q) * pp, w0);
          GatherRowPacked<CPT, B>(w0, sh, lr0 + static_cast<uint32_t>(q) * rowBytes, acc);
        }
      }
    } else if (active) {
      const uint8_t* chunk = ring + static_cast<size_t>(stage) * kChunkBytes + cgIdx * CPT;
      const int n = min(L.rpc, rows - r);
      const uint32_t lr0 = lutBase + static_cast<uint32_t>(r) * rowBytes;
      int q = rgIdx;
      for (; q + 3 * rg < n; q += 4 * rg) {
        const uint8_t* p = chunk + static_cast<size_t>(q) * pitch;
        const IV w0 = *reinterpret_cast<const IV*>(p);
        const IV w1 = *reinterpret_cast<const IV*>(p + static_cast<size_t>(rg) * pitch);
        const IV w2 = *reinterpret_cast<const IV*>(p + static_cast<size_t>(2 * rg) * pitch);
        const IV w3 = *reinterpret_cast<const IV*>(p + static_cast<size_t>(3 * rg) * pitch);
        const uint32_t lr = lr0 + static_cast<uint32_t>(q) * rowBytes, dl = static_cast<uint32_t>(rg) * rowBytes;
        GatherRow<CPT, PRE>(w0, lr, acc);
        GatherRow<CPT, PRE>(w1, lr + dl, acc);
        GatherRow<CPT, PRE>(w2, lr + 2 * dl, acc);
        GatherRow<CPT, PRE>(w3, lr + 3 * dl, acc);
      }
      for (; q < n; q += rg) {
        const IV w0 = *reinterpret_cast<const IV*>(chunk + static_cast<size_t>(q) * pitch);
        GatherRow<CPT, PRE>(w0, lr0 + static_cast<uint32_t>(q) * rowBytes, acc);
      }
    }
    __syncwarp();
    if (lane == 0) MbarArrive(emptyB + stage);
    if (++stage == nStage) { stage = 0; round++; }
  }
  *stagep = stage;
  *roundp = round;
  if (dbg && tid == 0) dbg[1] = clock64();
  if (rg > 1) {
    if (active) {
      float* mine = rgred + static_cast<size_t>(rgIdx) * pitch + cgIdx * CPT;
#pragma unroll
      for (int c = 0; c < CPT; c += 4) *reinterpret_cast<float4*>(mine + c) = make_float4(acc[c], acc[c + 1], acc[c + 2], acc[c + 3]);
    }
    ConsumerSync();
    for (int q = tid; q < (pitch >> 2); q += kConsumers) {
      float4 s = *reinterpret_cast<const float4*>(rgred + 4 * q);
      for (int g = 1; g < rg; g++) {
        const float4 t = *reinterpret_cast<const float4*>(rgred + static_cast<size_t>(g) * pitch + 4 * q);
        s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
      }
      StRelaxed4(out + 4 * q, s.x, s.y, s.z, s.w);
    }
  } else if (active) {
    float* o = out + cgIdx * CPT;
#pragma unroll
    for (int c = 0; c < CPT; c += 4) StRelaxed4(o + c, acc[c], acc[c + 1], acc[c + 2], acc[c + 3]);
  }
  if (dbg && tid == 0) dbg[2] = clock64();
}

// layers whose assignment table is bit-packed (packed_asmt.h): bits[l] (0 = byte table) and the bytes per table row
struct ChainPack {
  int bits[kMaxChain];
  int pitch[kMaxChain];
};

// PK: some layer of the chain has a bit-packed table (fc_chain_packed_kernel), pk describes them; else pk is NULL
template <bool PK>
__device__ __forceinline__ void ChainBody(const ChainArgs& a, const ChainPack* pk) {
  extern __shared__ __align__(128) unsigned char sm[];
  uint64_t* fullB = reinterpret_cast<uint64_t*>(sm);
  uint64_t* emptyB = fullB + kMaxStage;
  uint64_t* ctrdB = emptyB + kMaxStage;
  float* xs = reinterpret_cast<float*>(sm + kBarBytes);
  float* lut = xs + a.xFloats;
  float* ctrdS = lut + a.lutFloats;
  float* rgred = ctrdS + a.ctrdFloats;
  float* scr = rgred + a.rgFloats;
  uint8_t* ring = sm + a.ringOff;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, cta = blockIdx.x;
  if (a.dbg && tid == 0) { a.dbg[32 * cta] = GlobalTimer(); a.dbg[32 * cta + 2] = clock64(); }
  if (tid < a.nStage) { MbarInit(fullB + tid, 1); MbarInit(emptyB + tid, kConsumerWarps); }
  if (tid >= 32 && tid < 32 + a.nLayers) MbarInit(ctrdB + (tid - 32), 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  // the argument block lives in the constant bank: touch every layer's lines now, together, instead of taking one cache
  // miss (~0.2 us) on the critical path of each layer's first phase
  if ((a.L[0].relu | a.L[1].relu | a.L[2].relu | a.L[3].relu | a.L[0].rpc | a.L[1].rpc | a.L[2].rpc | a.L[3].rpc) < 0) __trap();
  __syncthreads();

  if (warp == kConsumerWarps) {
    // ---- producer: codebook slices of every layer, then the assignment rows of every layer through the ring ----
    int issued = 0;
    if (lane == 0) {
      for (int l = 0; l < a.nLayers; l++) {
        const ChainLayer& L = a.L[l];
        int r0, r1;
        RowRange(L, cta, &r0, &r1);
        if (r1 > r0) {
          const uint32_t bytes = static_cast<uint32_t>(r1 - r0) * L.K * L.d * 4u;
          MbarExpectTx(ctrdB + l, bytes);
          BulkLoad(ctrdS + L.ctrdOff, L.ctrd + static_cast<size_t>(r0) * L.K * L.d, bytes, ctrdB + l);
        }
      }
      int stage = 0;
      uint32_t round = 0;
      for (int l = 0; l < a.nLayers; l++) {
        const ChainLayer& L = a.L[l];
        int r0, r1;
        RowRange(L, cta, &r0, &r1);
        const int rowB = PK ? pk->pitch[l] : L.DoutPad;   // bytes per table row
        for (int r = r0; r < r1; r += L.rpc, issued++) {
          if (round > 0) MbarWait<26>(emptyB + stage, (round - 1) & 1u);
          const uint32_t bytes = static_cast<uint32_t>(min(L.rpc, r1 - r)) * rowB;
          MbarExpectTx(fullB + stage, bytes);
          BulkLoad(ring + static_cast<size_t>(stage) * kChunkBytes, L.asmt + static_cast<size_t>(r) * rowB, bytes, fullB + stage);
          if (++stage == a.nStage) { stage = 0; round++; }
        }
      }
    }
    // every slice of partial sums this CTA will wait for, requested into L2 now (all lanes)
    for (int l = 0; l < a.nLayers; l++) {
      const ChainLayer& P = a.L[l];
      if (l + 1 < a.nLayers) {
        const ChainLayer& N = a.L[l + 1];
        int r0, r1;
        RowRange(N, cta, &r0, &r1);
        PrefetchSlice(P.partial, P.DoutPad, a.G, r0 * N.d, min((r1 - r0) * N.d, max(0, N.Din - r0 * N.d)), lane);
      } else {
        const int o0 = cta * a.cpcLast;
        PrefetchSlice(P.partial, P.DoutPad, a.G, o0, max(0, min(a.cpcLast, P.Dout - o0)), lane);
      }
    }
    if (lane == 0) {
      if (a.dbg) {   // measurement only: when the first 8 chunks landed ([24 + i]); only while the ring is not recycled
        a.dbg[32 * cta + 23] = clock64();   // all copies issued
        for (int i = 0; i < (issued <= a.nStage ? min(issued, 8) : 0); i++) {
          MbarWait<26>(fullB + i, 0);
          a.dbg[32 * cta + 24 + i] = clock64();
        }
      }
    }
    return;
  }

  // ---- consumers ----
  int stage = 0;
  uint32_t round = 0;
  for (int l = 0; l < a.nLayers; l++) {
    const ChainLayer& L = a.L[l];
    int r0, r1;
    RowRange(L, cta, &r0, &r1);
    const int rows = r1 - r0;
    const int f0 = r0 * L.d, nf = rows * L.d;
    // (1) this CTA's slice of the layer input
    if (l == 0) {
      for (int i = tid; i < nf; i += kConsumers) {
        const int f = f0 + i;
        int off = f;
        if (L.srcHW) {          // NHWC map read in the reference's NCHW-flatten order (CaffeEva.cc:236-238)
          const int c = __float2int_rd((static_cast<float>(f) + 0.5f) * L.srcHWInv);
          off = (f - c * L.srcHW) * L.srcC + c;
        } else if (L.srcoff && f < L.Din) {
          off = __ldg(L.srcoff + f);
        }
        xs[i] = f < L.Din ? __ldg(a.src + off) : 0.0f;
      }
    } else {
      // sum of the previous layer's per-CTA partial sums (+ bias, ReLU) for this CTA's input features only
      const ChainLayer& P = a.L[l - 1];
      const int groups = (min(nf, max(0, L.Din - f0)) + 3) >> 2;   // Din == P.Dout <= P.DoutPad (multiple of 16)
      for (int i = 4 * groups + tid; i < nf; i += kConsumers) xs[i] = 0.0f;
      for (int b = 0; b < groups; b += 16) {
        if (b) ConsumerSync();      // the scratch of the previous batch has been read
        int fc;
        bool owner;
        const int fb = f0 + 4 * b + (tid >> 3);         // the feature this thread will own: its bias is fetched meanwhile
        const float bv = (fb < L.Din) ? __ldg(P.bias + fb) : 0.0f;
        const float v = CollectSlice(P.partial, P.DoutPad, a.G, f0 + 4 * b, min(16, groups - b), scr, tid, &fc, &owner, nullptr);
        if (owner) {
          const int f = f0 + 4 * b + fc;
          float o = f < L.Din ? v + bv : 0.0f;
          if (P.relu) o = fmaxf(o, 0.0f);
          xs[4 * b + fc] = o;
        }
      }
    }
    ConsumerSync();
    if (a.dbg && tid == 0) a.dbg[32 * cta + 4 + 5 * l] = clock64();
    // (2) LUT rows of the CTA's subspaces (reference GetInPdMat: ascending j, separate multiply and add)
    if (rows > 0) {
      MbarWait<26>(ctrdB + l, 0);
      const float* cs = ctrdS + L.ctrdOff;
      const int d = L.d, kmask = L.K - 1, lutRowF = L.lutPitch >> 2;
      for (int e = tid; e < rows * L.K; e += kConsumers) {
        const int r = e >> L.log2K;
        const int dims = min(d, L.Din - (r0 + r) * d);
        const float* c = cs + static_cast<size_t>(e) * d;
        const float* x = xs + r * d;
        float v = 0.0f;
        if (d == 4 && dims == 4) {
          const float4 cv = *reinterpret_cast<const float4*>(c);
          const float4 xv = *reinterpret_cast<const float4*>(x);
          v = __fmul_rn(xv.x, cv.x);
          v = __fadd_rn(v, __fmul_rn(xv.y, cv.y));
          v = __fadd_rn(v, __fmul_rn(xv.z, cv.z));
          v = __fadd_rn(v, __fmul_rn(xv.w, cv.w));
        } else {
          for (int j = 0; j < dims; j++) v = __fadd_rn(v, __fmul_rn(x[j], c[j]));
        }
        lut[r * lutRowF + (e & kmask)] = v;
      }
    }
    ConsumerSync();
    if (a.dbg && tid == 0) a.dbg[32 * cta + 5 + 5 * l] = clock64();
    // (3) + (4) gather-accumulate the assignment rows as they arrive, publish the partial sums of all DoutPad channels
    float* out = L.partial + static_cast<size_t>(cta) * L.DoutPad;
#define QCNN_GP(C, P) GatherAndPublish<C, P>(L, rows, a.nStage, fullB, emptyB, ring, lut, rgred, out, tid, lane, &stage, &round, \
                                             a.dbg ? a.dbg + 32 * cta + 6 + 5 * l : nullptr)
#define QCNN_GPK(C, B) GatherAndPublish<C, false, B>(L, rows, a.nStage, fullB, emptyB, ring, lut, rgred, out, tid, lane, &stage, \
                                                      &round, a.dbg ? a.dbg + 32 * cta + 6 + 5 * l : nullptr, pk->pitch[l])
#define QCNN_GPK_B(B) do { if (L.cpt == 8) QCNN_GPK(8, B); else if (L.cpt == 4) QCNN_GPK(4, B); else QCNN_GPK(16, B); } while (0)
    if (PK && pk->bits[l]) {
      if (pk->bits[l] == 5) QCNN_GPK_B(5);
      else if (pk->bits[l] == 4) QCNN_GPK_B(4);
      else if (pk->bits[l] == 6) QCNN_GPK_B(6);
      else QCNN_GPK_B(7);
    }
    else if (L.pre) { if (L.cpt == 8) QCNN_GP(8, true); else if (L.cpt == 4) QCNN_GP(4, true); else QCNN_GP(16, true); }
    else { if (L.cpt == 8) QCNN_GP(8, false); else if (L.cpt == 4) QCNN_GP(4, false); else QCNN_GP(16, false); }
#undef QCNN_GPK_B
#undef QCNN_GPK
#undef QCNN_GP
  }

  // ---- output of the last layer: a multiple of four channels per CTA ----
  {
    const ChainLayer& P = a.L[a.nLayers - 1];
    const int o0 = cta * a.cpcLast;
    const int groups = (max(0, min(a.cpcLast, P.Dout - o0)) + 3) >> 2;
    for (int b = 0; b < groups; b += 16) {
      if (b) ConsumerSync();   // the scratch of the previous batch has been read (its last use before: many barriers ago)
      int fc;
      bool owner;
      const int ob = o0 + 4 * b + (tid >> 3);
      const float bv = (ob < P.Dout) ? __ldg(P.bias + ob) : 0.0f;
      const float v = CollectSlice(P.partial, P.DoutPad, a.G, o0 + 4 * b, min(16, groups - b), scr, tid, &fc, &owner,
                                   (a.dbg && tid == 0 && b == 0) ? a.dbg + 32 * cta + 19 : nullptr);
      const int o = o0 + 4 * b + fc;
      if (owner && o < P.Dout) {
        const float t = v + bv;
        a.dst[o] = P.relu ? fmaxf(t, 0.0f) : t;
      }
    }
  }
  if (a.dbg && tid == 0) { a.dbg[32 * cta + 1] = GlobalTimer(); a.dbg[32 * cta + 3] = clock64(); }
}

__global__ void __launch_bounds__(kThreads, 1) fc_chain_kernel(const __grid_constant__ ChainArgs a) { ChainBody<false>(a, nullptr); }
__global__ void __launch_bounds__(kThreads, 1) fc_chain_packed_kernel(const __grid_constant__ ChainArgs a,
                                                                      const __grid_constant__ ChainPack pk) {
  ChainBody<true>(a, &pk);
}

int Gcd(int a, int b) { return b ? Gcd(b, a % b) : a; }

}  // namespace

namespace qcnn {

// Largest batch the chain kernel is launched for (once per image; the assignment bytes of the later images come from L2)
constexpr int kChainMaxN = 4;

static bool ChainEnabled() {
  static const bool on = !(getenv("QCNN_FC_CHAIN") && getenv("QCNN_FC_CHAIN")[0] == '0');
  return on;
}

// Fills the kernel arguments for a run of FC layers; false when the kernel does not apply (the caller falls back to
// the per-layer kernels of fc_aprx.cu).
// *packed: some layer keeps a bit-packed table (launch fc_chain_packed_kernel with *pk).  Eligibility and every figure
// but the ring chunking of a packed layer are those of the byte table.
static bool PlanChain(qcnn_ctx* ctx, const qcnn_layer* const* layers, const int* relu, int n, ChainArgs* out, size_t* smemBytes,
                      ChainPack* pk = nullptr, bool* packed = nullptr) {
  if (!ChainEnabled() || n < 1 || n > kMaxChain) return false;
  const int G = ctx->sm_count;
  if (G < 1 || G > kMaxParts) return false;
  ChainArgs& a = *out;
  memset(&a, 0, sizeof(a));
  ChainPack pkLocal;
  if (!pk) pk = &pkLocal;
  memset(pk, 0, sizeof(*pk));
  if (packed) *packed = false;
  a.nLayers = n; a.G = G;
  int xF = 64, lutF = 64, ctrdF = 0, rgF = 0;
  for (int l = 0; l < n; l++) {
    const qcnn_layer* Q = layers[l];
    if (Q->kind != QCNN_KIND_FC || Q->opt_fc_nsplit || Q->opt_fc_tn) return false;
    if (l > 0 && (Q->Din != layers[l - 1]->Dout || Q->d_srcoff.get())) return false;
    if (Q->DoutPad > kChunkBytes || Q->K * Q->d % 4 != 0) return false;
    ChainLayer& L = a.L[l];
    L.ctrd = Q->d_ctrd.as<float>(); L.asmt = Q->d_asmt.as<uint8_t>(); L.bias = Q->d_bias.as<float>(); L.srcoff = Q->d_srcoff.as<int>();
    L.Din = Q->Din; L.Dout = Q->Dout; L.DoutPad = Q->DoutPad; L.S = Q->S; L.K = Q->K; L.d = Q->d;
    L.log2K = 0;
    while ((1 << L.log2K) < Q->K) L.log2K++;
    if ((1 << L.log2K) != Q->K) return false;
    L.pre = Q->kshift == 2 ? 1 : 0;
    L.lutPitch = L.pre ? 256 : Q->K * 4;
    L.relu = relu[l];
    L.cpt = (Q->DoutPad / 4 <= kConsumers) ? 4 : ((Q->DoutPad / 8 <= kConsumers) ? 8 : 16);
    if (Q->DoutPad / L.cpt > kConsumers) return false;
    L.tpr = Q->DoutPad / L.cpt;
    L.rg = std::min(kConsumers / L.tpr, 16);
    L.tprInv = 1.0f / static_cast<float>(L.tpr);
    for (int t = 0; t < kConsumers; t++)     // the kernel divides by multiplying: must be exact for every thread index
      if (static_cast<int>(floorf((static_cast<float>(t) + 0.5f) * L.tprInv)) != t / L.tpr) return false;
    if (Q->d_srcoff.get() && Q->src_h > 0 && l == 0) {   // NHWC fold by arithmetic (same check); otherwise the offset table is used
                                                         // (d_srcoff is empty while qcnn_fc_aprx_forward_flat passes a flat vector)
      const int hw = Q->src_h * Q->src_w;
      const float inv = 1.0f / static_cast<float>(hw);
      bool exact = true;
      for (int f = 0; f < Q->Din && exact; f++) exact = static_cast<int>(floorf((static_cast<float>(f) + 0.5f) * inv)) == f / hw;
      if (exact) { L.srcHW = hw; L.srcC = Q->src_c; L.srcHWInv = inv; }
    }
    L.rpc = std::max(1, kChunkBytes / Q->DoutPad);
    pk->bits[l] = Q->asmt_bits;
    pk->pitch[l] = Q->asmt_bits ? Q->asmt_pitch : Q->DoutPad;
    if (Q->asmt_bits) {
      // packed rows are shorter, so a chunk holds more of them; the count stays a multiple of rg when the byte table's
      // is (row group g then owns rows g, g + rg, ... of the CTA's share either way: same partial sums), and leaves
      // room after the last row for the aligned word reads that run past it (packed_asmt.h)
      const int P = Q->asmt_pitch;
      int rpc = L.rpc;
      if (rpc % L.rg == 0) rpc = (kChunkBytes - qcnn::kPackedTail) / P / L.rg * L.rg;
      if (rpc < 1 || rpc * P + qcnn::kPackedTail > kChunkBytes) return false;
      L.rpc = rpc;
      if (packed) *packed = true;
    }
    L.unit = 4 / Gcd(Q->d, 4);
    const int units = CeilDiv(Q->S, L.unit);
    L.unitsBase = units / G; L.unitsRem = units % G;
    const int rowsMax = std::min(Q->S, (L.unitsBase + (L.unitsRem ? 1 : 0)) * L.unit);
    L.ctrdOff = ctrdF;
    ctrdF += rowsMax * Q->K * Q->d;
    xF = std::max(xF, RoundUp(rowsMax * Q->d, 64));       // keeps the LUT 256-byte aligned
    lutF = std::max(lutF, RoundUp(rowsMax * (L.lutPitch / 4), 64));
    if (L.rg > 1) rgF = std::max(rgF, L.rg * Q->DoutPad);
  }
  a.cpcLast = RoundUp(CeilDiv(layers[n - 1]->Dout, G), 4);
  // scratch of the cross-CTA reduction: [G][4 GP + 4] floats, GP = groups of 4 features reduced together (<= 16)
  int gmax = std::min(16, a.cpcLast / 4);
  for (int l = 1; l < n; l++) {
    const int rowsMax = std::min(a.L[l].S, (a.L[l].unitsBase + (a.L[l].unitsRem ? 1 : 0)) * a.L[l].unit);
    gmax = std::max(gmax, std::min(16, CeilDiv(rowsMax * a.L[l].d, 4)));
  }
  int gp = 1;
  while (gp < gmax) gp *= 2;
  a.scrFloats = G * (4 * gp + 4);
  a.xFloats = xF; a.lutFloats = lutF; a.ctrdFloats = ctrdF; a.rgFloats = rgF;
  const size_t fixed = kBarBytes + sizeof(float) * (static_cast<size_t>(xF) + lutF + ctrdF + rgF + a.scrFloats);
  a.ringOff = static_cast<int>((fixed + 127) & ~static_cast<size_t>(127));
  const size_t cap = SmemOptin(ctx);
  if (static_cast<size_t>(a.ringOff) + 2 * kChunkBytes > cap) return false;
  a.nStage = static_cast<int>(std::min<size_t>(kMaxStage, (cap - a.ringOff) / kChunkBytes));
  *smemBytes = a.ringOff + static_cast<size_t>(a.nStage) * kChunkBytes;
  return true;
}

bool FcChainEligible(qcnn_ctx* ctx, const qcnn_layer* const* layers, const int* relu, int n, int N) {
  if (N < 1 || N > kChainMaxN) return false;
  ChainArgs a;
  size_t smem;
  return PlanChain(ctx, layers, relu, n, &a, &smem);
}

// The chain row of fc_plan.cu: one layer as a chain of one
void DescribeFcChain(const qcnn_layer* L, const FcPlan&, int, char* buf, size_t cap) {
  ChainArgs a;
  size_t smem = 0;
  const int relu0 = 0;
  if (PlanChain(L->ctx, &L, &relu0, 1, &a, &smem))
    snprintf(buf, cap, "fc_chain(persistent, 1 layer, grid=%d, ring=%dx%dB, smem=%zuB)", a.G, a.nStage, kChunkBytes, smem);
}

// src: [N][Din of the first layer] (or the NHWC map the first layer's srcoff folds); dst: [N][Dout of the last layer]
int LaunchFcChain(qcnn_ctx* ctx, qcnn_layer* const* layers, const int* relu, int n, const float* src, int N, float* dst,
                  cudaStream_t st, unsigned long long* dbg, bool* handled) {
  *handled = false;
  if (N < 1 || N > kChainMaxN) return 0;
  ChainArgs a;
  ChainPack pk;
  bool packed = false;
  size_t smem = 0;
  if (!PlanChain(ctx, layers, relu, n, &a, &smem, &pk, &packed)) return 0;
  // partial-sum buffers: one per layer, [G][DoutPad], every word armed with the "not yet written" pattern
  for (int l = 0; l < n; l++) {
    qcnn_layer* Q = layers[l];
    const size_t need = sizeof(float) * static_cast<size_t>(ctx->sm_count) * Q->DoutPad;
    bool grown = false;
    const cudaError_t e = Q->d_cpart.Reserve(ctx, need, st, &grown);
    if (e == cudaErrorStreamCaptureUnsupported) return 0;   // cannot allocate inside a capture: per-layer kernels this time
    QCNN_CUDA(e);
    if (grown) QCNN_CUDA(cudaMemsetAsync(Q->d_cpart.get(), 0xFF, need, st));
    a.L[l].partial = Q->d_cpart.as<float>();
  }
  if (int rc = packed ? OptInSmem<fc_chain_packed_kernel>(ctx) : OptInSmem<fc_chain_kernel>(ctx)) return rc;
  a.dbg = dbg;
  const size_t srcImg = layers[0]->Din, dstImg = layers[n - 1]->Dout;
  for (int i = 0; i < N; i++) {
    a.src = src + i * srcImg;
    a.dst = dst + i * dstImg;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(a.G); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;   // all CTAs co-resident (they wait for each other's partial sums)
    attr[0].val.cooperative = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    if (packed) QCNN_CUDA(cudaLaunchKernelEx(&cfg, fc_chain_packed_kernel, a, pk));
    else QCNN_CUDA(cudaLaunchKernelEx(&cfg, fc_chain_kernel, a));
    ctx->launches++;
  }
  *handled = true;
  return 0;
}

}  // namespace qcnn
