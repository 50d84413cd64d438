// Bit-packed assignment tables of the fully-connected layers (qcnn_layer_set_param "asmt_packed"), shared by the three FC
// paths (fc_chain.cu, fc_aprx.cu, pq_gemm_tc.cu mode 2).
//
// Layout: b = log2(K) bits per index (4..7; K = 256 keeps its byte table).  Row s of the [S][DoutPad] table starts at byte
// s * pitch, pitch = RoundUp(DoutPad * b / 8, 16), so rows stay 16-byte aligned for cp.async / cp.async.bulk.  Inside a
// row, channel o occupies bits [o b, o b + b) of a little-endian bit string (bit i = bit i % 8 of byte i / 8).  The value
// is the plain 0-based index (the byte table stores idx << kshift); padding channels hold 0.
//
// A thread that owns CPT consecutive channels starting at a multiple of CPT reads the aligned 32-bit words covering its
// CPT * b bits: the first bit sits at a multiple of gcd(CPT b, 32) inside the first word, so PackedSpan<b, CPT>::kWords
// words always suffice.  Those reads may run up to 15 bytes past the end of a row; the table carries kPackedTail bytes
// after its last row, and the chain kernel leaves as many free after the rows of a ring chunk.
#ifndef QCNN_PACKED_ASMT_H_
#define QCNN_PACKED_ASMT_H_

#include <stdint.h>

namespace qcnn {

constexpr int kPackedTail = 16;

// bits per packed index of a codebook of K (a power of two) words; 8 = the byte table is kept
inline int PackedBits(int K) {
  int b = 0;
  while ((1 << b) < K) b++;
  return b;
}
inline int PackedPitch(int DoutPad, int b) { return (DoutPad * b / 8 + 15) / 16 * 16; }

template <int B, int CPT>
struct PackedSpan {
  static constexpr int kBits = CPT * B;
  static constexpr int kAlign = kBits % 32 == 0 ? 32 : (kBits % 16 == 0 ? 16 : (kBits % 8 == 0 ? 8 : 4));   // gcd(kBits, 32)
  static constexpr int kWords = (32 - kAlign + kBits + 31) / 32;
};

#ifdef __CUDACC__
// idx[c] = field c (B bits) of the bit string that starts at bit `sh` of the words w[0..NW): the words are first shifted
// down by `sh` (NW - 1 funnel shifts), then every field is one compile-time shift (or funnel shift) and a mask
template <int B, int CPT, int NW>
__device__ __forceinline__ void UnpackFields(const uint32_t (&w)[NW], uint32_t sh, uint32_t (&idx)[CPT]) {
  uint32_t u[NW];
#pragma unroll
  for (int i = 0; i + 1 < NW; i++) u[i] = __funnelshift_r(w[i], w[i + 1], sh);
  u[NW - 1] = w[NW - 1] >> sh;
#pragma unroll
  for (int c = 0; c < CPT; c++) {
    const int bit = c * B, j = bit >> 5, o = bit & 31;
    uint32_t v;
    if (o + B <= 32 || j + 1 >= NW) v = u[j] >> o;
    else v = __funnelshift_r(u[j], u[j + 1], o);
    idx[c] = v & ((1u << B) - 1u);
  }
}

// The tensor-core FC GEMMs (pq_gemm_tc mode 2, fc_ws) with a bit-packed table: the 16 indices of channels [ch, ch + 16)
// of one row (2 b bytes, from the four aligned words that cover them) -> 16 bytes idx << kshift at dst, the index block
// the byte table would stage
__device__ __forceinline__ void StagePackedRow(uint8_t* dst, const uint8_t* row, int ch, int b, int kshift) {
  const uint32_t bit0 = static_cast<uint32_t>(ch) * b, sh = bit0 & 31u;
  const uint32_t* wp = reinterpret_cast<const uint32_t*>(row) + (bit0 >> 5);
  const uint32_t w0 = __ldg(wp), w1 = __ldg(wp + 1), w2 = __ldg(wp + 2), w3 = __ldg(wp + 3);
  const uint32_t u0 = __funnelshift_r(w0, w1, sh), u1 = __funnelshift_r(w1, w2, sh), u2 = __funnelshift_r(w2, w3, sh), u3 = w3 >> sh;
  const uint32_t mask = (1u << b) - 1u;
  uint32_t o[4] = {0u, 0u, 0u, 0u};
#pragma unroll
  for (int c = 0; c < 16; c++) {
    const int pos = c * b, j = pos >> 5;   // (16 b + sh <= 128 bits: the fields end inside u3)
    const uint32_t lo = j == 0 ? u0 : (j == 1 ? u1 : (j == 2 ? u2 : u3));
    const uint32_t hi = j == 0 ? u1 : (j == 1 ? u2 : (j == 2 ? u3 : 0u));
    o[c >> 2] |= ((__funnelshift_r(lo, hi, pos & 31) & mask) << kshift) << (8 * (c & 3));
  }
  *reinterpret_cast<uint4*>(dst) = make_uint4(o[0], o[1], o[2], o[3]);
}
#endif

}  // namespace qcnn

#endif  // QCNN_PACKED_ASMT_H_
