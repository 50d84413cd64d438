/*
 * TEST INFRASTRUCTURE ONLY -- CPU oracle for the product-quantized forward path.
 *
 * Plain-C restatement of the reference algorithm (CAS-CLab/quantized-cnn), written from the
 * behaviour of the reference sources; every function cites the file:line it follows
 * (paths relative to /root/reference).  Built by oracle/Makefile into oracle/_build/libpq_oracle.so
 * with -ffp-contract=off so the float arithmetic is the same mul-then-add sequence the reference
 * executes (x86-64 g++ -O2, no FMA).
 *
 * Pinned: tests/test_oracle_vs_reference.py checks every function here bit-for-bit against the
 * compiled reference itself (oracle/_ref/libqcnn_ref.so) and against the committed golden vectors
 * in tests/golden/ that were generated from the compiled reference (tests/golden/make_golden.py).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load
 * this library.  The product library (quantized-cnn_b200/libqcnn_b200.so) never does.
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define PQO_EXPORT __attribute__((visibility("default")))

static int imin(int a, int b) { return a < b ? a : b; }
static int imax(int a, int b) { return a > b ? a : b; }

/* ------------------------------------------------------------------------------------------------
 * File formats (include/FileIO.h)
 * ---------------------------------------------------------------------------------------------- */

/* .bin : int32 dimCnt, int32 dimLen[dimCnt], raw elements row-major (FileIO.h:56-107).
 * Returns element count (or -1); dims gets up to 4 entries (missing = 1); at most cap elements are
 * stored in data (data may be NULL to query the shape). elemSize = sizeof(T). */
PQO_EXPORT long pqo_read_bin(const char* path, int* dims, void* data, long cap, int elemSize) {
  FILE* f = fopen(path, "rb");
  if (!f) return -1;
  int32_t dimCnt = 0;
  if (fread(&dimCnt, 4, 1, f) != 1 || dimCnt < 1 || dimCnt > 4) { fclose(f); return -1; }
  int32_t dl[4] = {1, 1, 1, 1};
  if (fread(dl, 4, dimCnt, f) != (size_t)dimCnt) { fclose(f); return -1; }
  long n = 1;
  for (int i = 0; i < 4; i++) { dims[i] = dl[i]; n *= dl[i]; }
  if (data) {
    long want = n < cap ? n : cap;
    if ((long)fread(data, elemSize, want, f) != want) { fclose(f); return -1; }
  }
  fclose(f);
  return n;
}

/* .cbn : header as .bin plus int32 bitCntPerEle, then 4096-byte blocks; each block holds
 * floor(32768/bits) values, MSB-first, contiguous across byte boundaries inside the block, block
 * tail bits unused (FileIO.h:110-178).  The reference reader returns value+1 (FileIO.h:165) and
 * CaffePara::LoadLayerPara subtracts 1 again in uint8 arithmetic (CaffePara.cc:285-288); the net
 * effect -- reproduced here -- is the stored 0-based index modulo 256.
 * Returns element count; *bitsOut receives bitCntPerEle. */
PQO_EXPORT long pqo_read_cbn(const char* path, int* dims, uint8_t* data, long cap, int* bitsOut) {
  FILE* f = fopen(path, "rb");
  if (!f) return -1;
  int32_t dimCnt = 0, bits = 0;
  if (fread(&dimCnt, 4, 1, f) != 1 || dimCnt < 1 || dimCnt > 4) { fclose(f); return -1; }
  int32_t dl[4] = {1, 1, 1, 1};
  if (fread(dl, 4, dimCnt, f) != (size_t)dimCnt) { fclose(f); return -1; }
  if (fread(&bits, 4, 1, f) != 1 || bits < 1 || bits > 8) { fclose(f); return -1; }
  long n = 1;
  for (int i = 0; i < 4; i++) { dims[i] = dl[i]; n *= dl[i]; }
  if (bitsOut) *bitsOut = bits;
  if (data) {
    const long perBlk = 4096 * 8 / bits;
    uint8_t blk[4096];
    long done = 0;
    long want = n < cap ? n : cap;
    while (done < want) {
      if (fread(blk, 1, 4096, f) != 4096) { fclose(f); return -1; }
      long cnt = want - done < perBlk ? want - done : perBlk;
      long bitPos = 0;
      for (long i = 0; i < cnt; i++, bitPos += bits) {
        /* take `bits` bits starting at bitPos, most-significant bit first */
        unsigned v = 0;
        for (int b = 0; b < bits; b++) {
          long p = bitPos + b;
          v = (v << 1) | ((blk[p >> 3] >> (7 - (p & 7))) & 1u);
        }
        data[done + i] = (uint8_t)((uint8_t)(v + 1) - 1); /* +1 (reader) then -- (LoadLayerPara) */
      }
      done += cnt;
    }
  }
  fclose(f);
  return n;
}

/* Writer counterpart of the .cbn layout (FileIO.h:281-350): input is 0-based, stored as is. */
PQO_EXPORT int pqo_write_cbn(const char* path, int dimCnt, const int* dims, const uint8_t* idx0, int bits) {
  FILE* f = fopen(path, "wb");
  if (!f) return -1;
  int32_t dc = dimCnt;
  fwrite(&dc, 4, 1, f);
  long n = 1;
  for (int i = 0; i < dimCnt; i++) { int32_t d = dims[i]; fwrite(&d, 4, 1, f); n *= d; }
  int32_t b32 = bits;
  fwrite(&b32, 4, 1, f);
  const long perBlk = 4096 * 8 / bits;
  uint8_t blk[4096];
  for (long done = 0; done < n; done += perBlk) {
    memset(blk, 0, sizeof(blk));
    long cnt = n - done < perBlk ? n - done : perBlk;
    long bitPos = 0;
    for (long i = 0; i < cnt; i++) {
      unsigned v = idx0[done + i];
      for (int b = bits - 1; b >= 0; b--, bitPos++) {
        if ((v >> b) & 1u) blk[bitPos >> 3] |= (uint8_t)(1u << (7 - (bitPos & 7)));
      }
    }
    fwrite(blk, 1, 4096, f);
  }
  fclose(f);
  return 0;
}

PQO_EXPORT int pqo_write_bin(const char* path, int dimCnt, const int* dims, const void* data, int elemSize) {
  FILE* f = fopen(path, "wb");
  if (!f) return -1;
  int32_t dc = dimCnt;
  fwrite(&dc, 4, 1, f);
  long n = 1;
  for (int i = 0; i < dimCnt; i++) { int32_t d = dims[i]; fwrite(&d, 4, 1, f); n *= d; }
  fwrite(data, elemSize, n, f);
  fclose(f);
  return 0;
}

/* CaffePara::CalcBitCntPerEle (CaffePara.cc:360-378) on 1-based values: bits needed for (max-1). */
PQO_EXPORT int pqo_bits_per_ele(const uint8_t* idx1, long n) {
  uint8_t mx = 0;
  for (long i = 0; i < n; i++) if (idx1[i] > mx) mx = idx1[i];
  mx = (uint8_t)(mx - 1);
  int bits = 0;
  while (mx != 0) { mx /= 2; bits++; }
  return bits;
}

/* ------------------------------------------------------------------------------------------------
 * LUT stage: CaffeEva::GetInPdMat (src/CaffeEva.cc:1261-1296)
 *   inPd[p][s][k] = sum_{j < min(D - s*d, d)} data[p][s*d+j] * ctrd[s][k][j]
 * zero start, ascending j, one rounded multiply and one rounded add per term (the reference runs
 * cblas_saxpy(K, x, ctrdRow, 1, out, 1), include/BlasWrapper.h:164-184: y[i] += a * x[i]).
 * ctrdLst here is in FILE order [S][K][d] (the reference permutes it to [S][d][K] first,
 * CaffeEva.cc:556-557; only the addressing differs).
 * ---------------------------------------------------------------------------------------------- */
PQO_EXPORT void pqo_get_inpd(const float* data, long P, int D, const float* ctrdLst, int S, int K, int d,
                             float* inPd /* [P][S][K] */) {
  for (int s = 0; s < S; s++) {
    int lo = s * d;
    int sel = imin(D - lo, d);
    for (long p = 0; p < P; p++) {
      const float* x = data + p * D + lo;
      float* out = inPd + (p * S + s) * (long)K;
      for (int k = 0; k < K; k++) out[k] = 0.0f;
      for (int j = 0; j < sel; j++) {
        const float a = x[j];
        for (int k = 0; k < K; k++) {
          float prod = a * ctrdLst[((long)s * K + k) * d + j];
          out[k] = out[k] + prod;
        }
      }
    }
  }
}

/* ------------------------------------------------------------------------------------------------
 * Conv: CaffeEva::CalcFeatMap_ConvAprx (src/CaffeEva.cc:760-868)
 * src  [N][Hi][Wi][Cin] NHWC, dst [N][Ho][Wo][Cout] NHWC (bias included, no ReLU)
 * ctrdLst [S][K][d] (file order) -- ONE codebook shared by all groups (CaffeEva.cc:810)
 * asmtLst [Cout][kh][kw][S] 0-based (file order; the reference permutes to [kh][kw][S][Cout], :585-586)
 * Accumulation order per output: bias, then kh, kw ascending over the in-bounds window, then s ascending.
 * ---------------------------------------------------------------------------------------------- */
PQO_EXPORT void pqo_conv_aprx(const float* src, int N, int Hi, int Wi, int Cin, int Cout, int ksz, int pad,
                              int stride, int G, const float* ctrdLst, int S, int K, int d,
                              const uint8_t* asmtLst, const float* bias, float* dst) {
  const int Ho = (Hi + 2 * pad - ksz) / stride + 1; /* CaffeEva.cc:361-362 */
  const int Wo = (Wi + 2 * pad - ksz) / stride + 1;
  const int Cg = Cin / G, Kg = Cout / G;
  const long P = (long)N * Hi * Wi;
  float* grp = (float*)malloc(sizeof(float) * P * Cg);
  float* inPd = (float*)malloc(sizeof(float) * P * S * K);
  for (int g = 0; g < G; g++) {
    /* per-group channel slice (CaffeEva.cc:802-809) */
    for (long p = 0; p < P; p++) memcpy(grp + p * Cg, src + p * Cin + (long)g * Cg, sizeof(float) * Cg);
    pqo_get_inpd(grp, P, Cg, ctrdLst, S, K, d, inPd);
    for (int ho = 0; ho < Ho; ho++) {
      for (int wo = 0; wo < Wo; wo++) {
        const int hL = ho * stride - pad, wL = wo * stride - pad;
        const int khL = imax(0, -hL), khU = imin(ksz - 1, Hi - 1 - hL); /* :824-827 */
        const int kwL = imax(0, -wL), kwU = imin(ksz - 1, Wi - 1 - wL);
        for (int n = 0; n < N; n++) {
          float* out = dst + (((long)n * Ho + ho) * Wo + wo) * Cout + (long)g * Kg;
          for (int c = 0; c < Kg; c++) out[c] = bias[g * Kg + c];
          for (int kh = khL; kh <= khU; kh++) {
            for (int kw = kwL; kw <= kwU; kw++) {
              const float* lut = inPd + (((long)n * Hi + (hL + kh)) * Wi + (wL + kw)) * S * (long)K;
              for (int s = 0; s < S; s++) {
                for (int c = 0; c < Kg; c++) {
                  const uint8_t a = asmtLst[(((long)(g * Kg + c) * ksz + kh) * ksz + kw) * S + s];
                  out[c] = out[c] + lut[(long)s * K + a];
                }
              }
            }
          }
        }
      }
    }
  }
  free(grp);
  free(inPd);
}

/* ------------------------------------------------------------------------------------------------
 * FC: CaffeEva::CalcFeatMap_FCntAprx (src/CaffeEva.cc:968-1025)
 * src [N][Din], dst [N][Dout]; ctrdLst [S][K][d]; asmtLst [Dout][S] 0-based (file order).
 * Accumulation: bias, then s ascending.
 * ---------------------------------------------------------------------------------------------- */
PQO_EXPORT void pqo_fc_aprx(const float* src, int N, int Din, int Dout, const float* ctrdLst, int S, int K,
                            int d, const uint8_t* asmtLst, const float* bias, float* dst) {
  float* inPd = (float*)malloc(sizeof(float) * (long)N * S * K);
  pqo_get_inpd(src, N, Din, ctrdLst, S, K, d, inPd);
  for (int n = 0; n < N; n++) {
    float* out = dst + (long)n * Dout;
    const float* lut = inPd + (long)n * S * K;
    for (int o = 0; o < Dout; o++) out[o] = bias[o];
    for (int s = 0; s < S; s++) {
      for (int o = 0; o < Dout; o++) {
        out[o] = out[o] + lut[(long)s * K + asmtLst[(long)o * S + s]];
      }
    }
  }
  free(inPd);
}

/* ReLU: CaffeEva::CalcFeatMap_ReLu (src/CaffeEva.cc:1027-1036) */
PQO_EXPORT void pqo_relu(const float* src, long n, float* dst) {
  for (long i = 0; i < n; i++) dst[i] = src[i] > 0.0f ? src[i] : 0.0f;
}

/* LRN across channels: CaffeEva::CalcFeatMap_LoRN (src/CaffeEva.cc:1038-1089)
 *   sq[c] = (x[c]*x[c]) * (alpha/size)       vsSqr then cblas_sscal (:1066-1067)
 *   sum[c] = k; for w in 0..size-1: sum[c] = sum[c] + sqExt[c + w]   (zero-padded by radius, :1070-1075)
 *   y[c] = x[c] * expf(-beta * logf(sum[c]))                         vsPowx_m fallback, BlasWrapper.h:134-147 */
PQO_EXPORT void pqo_lrn(const float* src, long pixels, int C, int size, float alpha, float beta, float k,
                        float* dst) {
  const int rad = (size - 1) / 2;
  const float coeff = alpha / size;
  float* ext = (float*)calloc(C + 2 * rad, sizeof(float));
  const float nb = -beta;
  for (long p = 0; p < pixels; p++) {
    const float* x = src + p * C;
    float* y = dst + p * C;
    for (int c = 0; c < C; c++) {
      float sq = x[c] * x[c];
      ext[rad + c] = sq * coeff;
    }
    for (int c = 0; c < C; c++) {
      float sum = k;
      for (int w = 0; w < size; w++) sum = sum + ext[c + w];
      float f = expf(nb * logf(sum));
      y[c] = x[c] * f;
    }
  }
  free(ext);
}

/* Max-pool: CaffeEva::CalcFeatMap_Pool (src/CaffeEva.cc:870-921); Ho = ceil((Hi+2p-k)/s)+1 (:365-372);
 * window clipped to the image. NHWC. */
PQO_EXPORT void pqo_pool(const float* src, int N, int Hi, int Wi, int C, int ksz, int pad, int stride,
                         float* dst) {
  const int Ho = (int)ceil((Hi + 2 * pad - ksz) / (double)stride) + 1;
  const int Wo = (int)ceil((Wi + 2 * pad - ksz) / (double)stride) + 1;
  for (int n = 0; n < N; n++)
    for (int ho = 0; ho < Ho; ho++) {
      int hL = imax(0, ho * stride - pad), hU = imin(Hi, ho * stride + ksz - pad) - 1;
      for (int wo = 0; wo < Wo; wo++) {
        int wL = imax(0, wo * stride - pad), wU = imin(Wi, wo * stride + ksz - pad) - 1;
        float* out = dst + (((long)n * Ho + ho) * Wo + wo) * C;
        int first = 1;
        for (int h = hL; h <= hU; h++)
          for (int w = wL; w <= wU; w++) {
            const float* in = src + (((long)n * Hi + h) * Wi + w) * C;
            if (first) { memcpy(out, in, sizeof(float) * C); first = 0; }
            else for (int c = 0; c < C; c++) out[c] = in[c] > out[c] ? in[c] : out[c];
          }
      }
    }
}

/* Softmax WITHOUT max subtraction, float accumulator: CaffeEva::CalcFeatMap_SMax (src/CaffeEva.cc:1098-1116) */
PQO_EXPORT void pqo_softmax(const float* src, int N, int C, float* dst) {
  for (int n = 0; n < N; n++) {
    const float* x = src + (long)n * C;
    float* y = dst + (long)n * C;
    float sum = 0.0f;
    for (int c = 0; c < C; c++) { y[c] = expf(x[c]); sum = sum + y[c]; }
    for (int c = 0; c < C; c++) y[c] = y[c] / sum;
  }
}

/* Layout permutes the executor performs (CaffeEva.cc:225-228 NCHW->NHWC on input, :236-238 NHWC->NCHW before
 * the first FC layer; Matrix::Permute, include/Matrix.h:508-553). */
PQO_EXPORT void pqo_nchw_to_nhwc(const float* src, int N, int C, int H, int W, float* dst) {
  for (int n = 0; n < N; n++)
    for (int c = 0; c < C; c++)
      for (int h = 0; h < H; h++)
        for (int w = 0; w < W; w++)
          dst[(((long)n * H + h) * W + w) * C + c] = src[(((long)n * C + c) * H + h) * W + w];
}
PQO_EXPORT void pqo_nhwc_to_nchw(const float* src, int N, int H, int W, int C, float* dst) {
  for (int n = 0; n < N; n++)
    for (int h = 0; h < H; h++)
      for (int w = 0; w < W; w++)
        for (int c = 0; c < C; c++)
          dst[(((long)n * C + c) * H + h) * W + w] = src[(((long)n * H + h) * W + w) * C + c];
}

/* Top-k by repeated arg-max exactly as CaffeEvaWrapper::Proc does (src/CaffeEvaWrapper.cc:188-206):
 * start from element 0, strict '<' comparison (first maximum wins), winner zeroed for the next round. */
PQO_EXPORT void pqo_topk(const float* prob, int C, int k, int* idx, float* val) {
  float* tmp = (float*)malloc(sizeof(float) * C);
  memcpy(tmp, prob, sizeof(float) * C);
  for (int r = 0; r < k; r++) {
    int bi = 0;
    float best = tmp[0];
    for (int c = 1; c < C; c++) if (best < tmp[c]) { best = tmp[c]; bi = c; }
    idx[r] = bi;
    val[r] = best;
    tmp[bi] = 0.0f;
  }
  free(tmp);
}

/* k-fold arg-max of CaffeEva::CvtFeatMapToLablVec (src/CaffeEva.cc:1162-1190): each round scans from
 * (FLT_MIN, index 0) with a strict '<', so a value <= FLT_MIN or a NaN never wins, and index 0 is taken (and
 * zeroed) when nothing beats FLT_MIN.  Labels only; the reference records no probability. */
PQO_EXPORT void pqo_topk_labl(const float* prob, int C, int k, int* idx) {
  float* tmp = (float*)malloc(sizeof(float) * C);
  memcpy(tmp, prob, sizeof(float) * C);
  for (int r = 0; r < k; r++) {
    float best = 1.17549435e-38f; /* FLT_MIN */
    int bi = 0;
    for (int c = 0; c < C; c++) if (best < tmp[c]) { best = tmp[c]; bi = c; }
    idx[r] = bi;
    tmp[bi] = 0.0f;
  }
  free(tmp);
}

/* Synthetic image generator of SURVEY.md 8(d) / BASELINE.md 3: LCG s <- 1664525 s + 1013904223 (mod 2^32),
 * x = ((s >> 8) & 0xFFFF) / 65536 * 256 - 128, value taken after each update. */
PQO_EXPORT void pqo_lcg_fill(uint32_t seed, float* out, long n) {
  uint32_t s = seed;
  for (long i = 0; i < n; i++) {
    s = s * 1664525u + 1013904223u;
    out[i] = (float)((s >> 8) & 0xFFFFu) / 65536.0f * 256.0f - 128.0f;
  }
}
