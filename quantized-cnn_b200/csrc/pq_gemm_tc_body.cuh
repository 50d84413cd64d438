// Body of the decode-at-use GEMM kernels (pq_gemm_tc.cu), included inside pq_gemm_tc_kernel and pq_gemm_tc_packed_kernel:
// in scope are the kernel parameter `a` (GemmArgs), the template parameters BF and NT, and PK / pkBits / pkPitch (mode 2
// index rows come from a bit-packed FC table), and the device helpers of wgmma.h.  Not a header: no include guard.
  constexpr int NTHR = kThreads;
  constexpr int NSTG = kStagers;
  constexpr int RP = kRegPos;
  constexpr bool CORR = NT <= 64;
  extern __shared__ __align__(128) unsigned char smem[];
  const SmemMap sm = MapSmem(a);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int K = a.K, GT = a.GT;

  float4* planes = reinterpret_cast<float4*>(smem + sm.planes);
  float4* cbs = reinterpret_cast<float4*>(smem + sm.cbs);
  uint8_t* ids = smem + sm.ids;
  KStep* tabS = reinterpret_cast<KStep*>(smem + sm.tab);   // (FC tiles: shared memory is lightly loaded there and an LDS beats an indexed LDC)
  int* posoff = reinterpret_cast<int*>(smem + sm.posoff);
  int* posrow = reinterpret_cast<int*>(smem + sm.posrow);
  int* posdst = reinterpret_cast<int*>(smem + sm.posdst);
  int* outoff = reinterpret_cast<int*>(smem + sm.outoff);
  float* biasS = reinterpret_cast<float*>(smem + sm.bias);
  uint64_t* fullB = reinterpret_cast<uint64_t*>(smem + sm.bars);   // [<=4] position planes: stagers -> consumers
  uint64_t* emptyB = fullB + 4;                                    // [<=4] chunk's MMAs retired -> stagers
  uint64_t* fullC = emptyB + 4;                                    // [kCbBufs] codebook + indices: stagers -> consumers
  uint64_t* emptyC = fullC + kCbBufs;                              // [kCbBufs] consumers done with the chunk -> stagers
  int b = blockIdx.x;
  const int ct = b % a.nct; b /= a.nct;
  int g = 0, split = 0;
  if (a.nsplit > 1) { split = b % a.nsplit; b /= a.nsplit; }
  if (a.mode != 2) { g = b % a.G; b /= a.G; }
  const int tile = b;
  const int ch0 = ct * 128;                            // first channel of the tile inside the group
  const int CTv = min(128, a.Kg - ch0);                // valid channels
  const int Q0 = tile * NT;                            // first flat position
  const int i0 = Q0 / a.IB;                            // first image touched
  const float* srcBase = a.src + static_cast<size_t>(i0) * a.srcImg;
  float* dstBase = a.dst + static_cast<size_t>(i0) * a.dstImg + g * a.Kg + ch0;
  // mode 2: this CTA's k-step range [k0, k0 + kTotal) of the layer; partial sums go to their own plane
  const int k0 = split * a.kPerSplit;
  const int kTotal = a.mode == 2 ? min(a.kPerSplit, a.kAll - k0) : 0;
  // convolution modes: K split by chunks [kcBase, kcBase + nChunks) (small batches: more CTAs than position tiles)
  const int kcBase = a.mode == 2 ? 0 : split * a.kPerSplit;
  const int nChunks = a.mode == 2 ? (kTotal + a.chunkCount[0] - 1) / a.chunkCount[0]
                                  : (a.nsplit > 1 ? min(a.kPerSplit, a.nChunks - kcBase) : a.nChunks);
  // mode 2: rows = images, so the tile starts at row Q0 of the output (or of this split's partial sums)
  if (a.mode == 2)
    dstBase = (a.nsplit > 1 ? a.partial + static_cast<size_t>(split) * a.N * a.dstRow : a.dst) + static_cast<size_t>(Q0) * a.dstRow + ch0;
  if (a.mode != 2 && a.nsplit > 1)
    dstBase = a.partial + (static_cast<size_t>(split) * a.N + i0) * a.dstImg + g * a.Kg + ch0;

  // ---- set-up (all threads) ----
  for (int e = tid; e < a.ntab; e += NTHR) tabS[e] = a.tab[e];
  for (int p = tid; p < a.planeF4; p += NTHR) {
    int off = -1;
    if (a.mode == 0) {
      // float4 p: half = p / NPOS, position = p % NPOS; the half only selects the channel offset (added per chunk)
      const int pos = p % a.NPOS;
      const int F = Q0 + pos;
      const int i = F / a.IB, rem = F - i * a.IB;
      const int r = rem / a.PW, c = rem - r * a.PW;
      if (i < a.N && r >= a.pad && c >= a.pad) off = (((i - i0) * a.Hi + (r - a.pad)) * a.Wi + (c - a.pad)) * a.Cin;
    } else if (a.mode == 1) {
      // float4 p: phase column pw = p / NPOS, position = p % NPOS -> pixel (r*stride + ph - pad, c*stride + pw - pad);
      // the phase row ph is the chunk, so the row part is resolved per chunk from posrow
      const int pw = p / a.NPOS, pos = p - pw * a.NPOS;
      const int F = Q0 + pos;
      const int i = F / a.IB, rem = F - i * a.IB;
      const int r = rem / a.PW, c = rem - r * a.PW;
      const int wi = c * a.stride + pw - a.pad;
      const bool colOk = i < a.N && wi >= 0 && wi < a.Wi;
      off = static_cast<int>((i - i0) * a.srcImg) + (r * a.stride - a.pad) * a.rowStride + wi * a.colStride;
      posrow[p] = colOk ? r * a.stride - a.pad : -(1 << 28);
    }
    posoff[p] = off;   // (mode 2 stages its planes by bulk copy: no offsets)
    if (BF && a.mode != 2) {
      // bf16x2 planes hold 16-byte rows of eight values: mode 0 row = position, the half selects bytes 0-7 / 8-15;
      // mode 1 row = (phase-column pair, position), the column's parity selects the half
      const int grp = p / a.NPOS, pos = p - grp * a.NPOS;
      posdst[p] = a.mode == 0 ? pos * 16 + grp * 8 : ((grp >> 1) * a.NPOS + pos) * 16 + (grp & 1) * 8;
    }
  }
  for (int p = tid; p < 128; p += NTHR) {
    int off = -1;
    if (p < NT) {
      const int Q = Q0 + p;
      const int i = Q / a.IB, rem = Q - i * a.IB;
      const int ho = rem / a.PW, wo = rem - ho * a.PW;
      if (a.mode == 2) { if (Q < a.N) off = p * a.dstRow; }
      else if (i < a.N && ho < a.Ho && wo < a.Wo) off = (((i - i0) * a.Ho + ho) * a.Wo + wo) * a.Cout;
    }
    outoff[p] = off;
  }
  if (a.mode == 1 && a.bulkC)      // slot 1 (unpaired taps) stays zero; slot 0 arrives by bulk copy
    for (int e = tid; e < kCbBufs * K; e += NTHR) cbs[(e / K) * a.cbSlots * K + K + (e % K)] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  for (int c = tid; c < 128; c += NTHR) biasS[c] = (c < CTv && split == 0) ? __ldg(a.bias + g * a.Kg + ch0 + c) : 0.0f;
  if (tid == 0) {
    for (int i = 0; i < 4; i++) { MbarInit(fullB + i, NSTG); MbarInit(emptyB + i, kConsumers / 32); }
    for (int i = 0; i < kCbBufs; i++) { MbarInit(fullC + i, a.bulkC ? 1 : NSTG); MbarInit(emptyC + i, kConsumers / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int warpU = __shfl_sync(0xffffffffu, warp, 0);   // provably warp-uniform role selector
  if (warpU >= kConsumers / 32) {
    // =========================== stagers ===========================
    const int st = tid - kConsumers;
    const int sw = st >> 5;                      // stager warp 0 .. NSTG/32 - 1
    // 4-float piece j0/4 of codeword k of subspace s: fp32 codebook [S][K][d] or the pre-split one [S][d/4][K][4 words]
    auto piece = [&](int s, int j0, int k) -> const float* {
      return a.cbPre ? a.ctrd + ((static_cast<size_t>(s) * (a.d >> 2) + (j0 >> 2)) * K + k) * 4
                     : a.ctrd + (static_cast<size_t>(s) * K + k) * a.d + j0;
    };
    // chunk kc: codebook slices + index rows by cp.async (one group); the positions travel through registers
    auto fetchChunk = [&](int kc) {
      const int cbuf = kc % kCbBufs;
      if (a.mode == 0) {
        // per-chunk scalars: the two 4-channel halves, their subspaces and the offsets inside the codewords
        const int taps = a.ksz * a.ksz;
        const int chA = (kcBase + kc) * 8, chB = chA + 4;
        const bool okA = chA < a.Cg, okB = chB < a.Cg;
        const int sA = okA ? chA / a.d : 0, jA = okA ? chA - sA * a.d : 0;
        const int sB = okB ? chB / a.d : 0, jB = okB ? chB - sB * a.d : 0;
        // (positions travel through registers: loadPos / storePos)
        // codebook slices: slot = half
        float4* cdst = cbs + cbuf * a.cbSlots * K;
        if (a.bulkC) {
          // four bulk copies (two contiguous codebook slices, two contiguous index blocks), completion counted on fullC;
          // a half beyond the group's channels stages valid data (its positions are staged as zeros)
          if (st == 0) {
            const uint32_t cbBytes = static_cast<uint32_t>(K) * 16u, idBytes = static_cast<uint32_t>(CTv * a.tapsPad);
            uint64_t* bar = fullC + cbuf;
            uint8_t* idst = ids + cbuf * a.idRows * 128;
            const uint8_t* tA = a.asmtT + (static_cast<size_t>(g * a.S + sA) * a.KgPad + ch0) * a.tapsPad;
            const uint8_t* tB = a.asmtT + (static_cast<size_t>(g * a.S + sB) * a.KgPad + ch0) * a.tapsPad;
            MbarExpectTx(bar, 2u * cbBytes + 2u * idBytes);
            BulkLoad(cdst, piece(sA, jA, 0), cbBytes, bar);
            BulkLoad(cdst + K, piece(sB, jB, 0), cbBytes, bar);
            BulkLoad(idst, tA, idBytes, bar);
            BulkLoad(idst + 128 * a.tapsPad, tB, idBytes, bar);
          }
          return;
        }
        for (int k = st; k < K; k += NSTG) {
          CpAsync16(cdst + k, piece(sA, jA, k), okA);
          CpAsync16(cdst + K + k, piece(sB, jB, k), okB);
        }
        if (a.idxT) {
          // channel-major index block [half][channel][tapsPad]: contiguous CTv * tapsPad bytes per half
          const int gran = (CTv * a.tapsPad) >> 4;
          const uint8_t* tA = a.asmtT + (static_cast<size_t>(g * a.S + sA) * a.KgPad + ch0) * a.tapsPad;
          const uint8_t* tB = a.asmtT + (static_cast<size_t>(g * a.S + sB) * a.KgPad + ch0) * a.tapsPad;
          uint8_t* idst = ids + cbuf * a.idRows * 128;
          for (int e = st; e < 2 * gran; e += NSTG) {
            const bool hb = e >= gran;
            const int q = hb ? e - gran : e;
            CpAsync16(idst + (hb ? 128 * a.tapsPad : 0) + (q << 4), (hb ? tB : tA) + (static_cast<size_t>(q) << 4), true);
          }
        }
        // index rows [half][tap]: stager warp w takes rows w, w+3, ...; lane < gran copies one 16-byte granule
        const int gran = CTv >> 4;
        if (!a.idxT && lane < gran) {
          const uint8_t* asA = a.asmt + static_cast<size_t>(g * a.S + sA) * taps * a.KgPad + ch0 + (lane << 4);
          const uint8_t* asB = a.asmt + static_cast<size_t>(g * a.S + sB) * taps * a.KgPad + ch0 + (lane << 4);
          uint8_t* idst = ids + cbuf * a.idRows * 128 + (lane << 4);
          for (int row = sw; row < 2 * taps; row += NSTG / 32) {
            const bool hb = row >= taps;
            const int tap = hb ? row - taps : row;
            CpAsync16(idst + row * 128, (hb ? asB : asA) + static_cast<size_t>(tap) * a.KgPad, true);
          }
        }
      }
      if (a.mode == 1) {
        // chunk = phase row ph: pixels of input rows r*stride + ph - pad, one 4-byte copy per channel
        const int ph = kcBase + kc;
        // (positions travel through registers: loadPos / storePos)
        // codebook: slot 0 = the first 4 floats of every codeword of subspace 0, slot 1 = zeros (unpaired taps)
        float4* cdst = cbs + cbuf * a.cbSlots * K;
        if (a.bulkC) {
          if (st == 0) {
            const uint32_t cbBytes = static_cast<uint32_t>(K) * 16u, idBytes = static_cast<uint32_t>(CTv * a.tapsPad);
            uint64_t* bar = fullC + cbuf;
            const uint8_t* tA = a.asmtT + (static_cast<size_t>(g * a.stride + ph) * a.KgPad + ch0) * a.tapsPad;
            MbarExpectTx(bar, cbBytes + idBytes);
            BulkLoad(cdst, piece(0, 0, 0), cbBytes, bar);
            BulkLoad(ids + cbuf * a.idRows * 128, tA, idBytes, bar);
          }
          return;
        }
        for (int k = st; k < K; k += NSTG) {
          CpAsync16(cdst + k, piece(0, 0, k), true);
          CpAsync16(cdst + K + k, a.ctrd, false);
        }
        // index rows of the taps with kh % stride == ph, in (kh, kw) order
        const int gran = CTv >> 4;
        if (lane < gran) {
          const uint8_t* as0 = a.asmt + static_cast<size_t>(g * a.S) * a.ksz * a.ksz * a.KgPad + ch0 + (lane << 4);
          uint8_t* idst = ids + cbuf * a.idRows * 128 + (lane << 4);
          const int nrow = ((a.ksz - ph + a.stride - 1) / a.stride) * a.ksz;
          for (int row = sw; row < nrow; row += NSTG / 32) {
            const int kh = ph + (row / a.ksz) * a.stride, kw = row % a.ksz;
            CpAsync16(idst + row * 128, as0 + static_cast<size_t>(kh * a.ksz + kw) * a.KgPad, true);
          }
        }
      }
      if (a.mode == 2) {
        // chunk = KS consecutive k-steps of this CTA's range: features [f0, f0 + 8 ne)
        const int KS = a.chunkCount[0];
        const int ne = min(KS, kTotal - kc * KS);
        const int f0 = (k0 + kc * KS) * 8;
        const int gran = (CTv + 15) >> 4;
        // PK: the stagers expand the packed rows into the same u8 index block with plain st.shared instead of cp.async.
        // The block is published by the same arrive on fullC[cbuf] as the copies: every stager thread stores its rows
        // before it arrives (program order), mbarrier.arrive has release and the decoders' mbarrier.try_wait acquire
        // semantics (both .cta), so the stores are visible to every decoder that passed the wait.  The buffer is not
        // rewritten before the decoders arrived on emptyC[cbuf], which the stagers wait for first.
        if (a.d == 1) {
          // slot q = subspace f0 + q: its K scalar codewords; index row q
          const int kq = K >> 2;
          float4* cdst = cbs + cbuf * a.cbSlots * a.cbF4;
          for (int e = st; e < 8 * ne * kq; e += NSTG) CpAsync16(cdst + e, a.ctrd + static_cast<size_t>(f0) * K + e * 4, true);
          if (PK && lane < gran) {
            uint8_t* idst = ids + cbuf * a.idRows * 128 + (lane << 4);
            for (int row = sw; row < 8 * ne; row += NSTG / 32)
              StagePackedRow(idst + row * 128, a.asmt + static_cast<size_t>(f0 + row) * pkPitch, ch0 + (lane << 4), pkBits, a.kshift);
          } else if (lane < gran) {
            const uint8_t* as0 = a.asmt + static_cast<size_t>(f0) * a.KgPad + ch0 + (lane << 4);
            uint8_t* idst = ids + cbuf * a.idRows * 128 + (lane << 4);
            for (int row = sw; row < 8 * ne; row += NSTG / 32) CpAsync16(idst + row * 128, as0 + static_cast<size_t>(row) * a.KgPad, true);
          }
        } else {
          // slot q = features [f0 + 4q, +4): piece j0 of every codeword of subspace s; index row q = row s of the layer
          float4* cdst = cbs + cbuf * a.cbSlots * a.cbF4;
          for (int e = st; e < 2 * ne * K; e += NSTG) {
            const int q = e / K, k = e - q * K;
            const int f = f0 + 4 * q;
            const int s = f / a.d, j0 = f - s * a.d;
            CpAsync16(cdst + e, piece(s, j0, k), true);
          }
          if (lane < gran) {
            uint8_t* idst = ids + cbuf * a.idRows * 128 + (lane << 4);
            for (int row = sw; row < 2 * ne; row += NSTG / 32) {
              const int s = (f0 + 4 * row) / a.d;
              if (PK) StagePackedRow(idst + row * 128, a.asmt + static_cast<size_t>(s) * pkPitch, ch0 + (lane << 4), pkBits, a.kshift);
              else CpAsync16(idst + row * 128, a.asmt + static_cast<size_t>(s) * a.KgPad + ch0 + (lane << 4), true);
            }
          }
        }
      }
      CpAsyncCommit();
    };
    // Positions of the convolution modes: global -> registers -> hi/lo planes.  (16-byte cp.async of scattered pieces
    // costs one shared-memory wavefront per THREAD, whereas a 128-bit store of 32 consecutive float4 costs four per
    // warp.)  A thread owns float4 st, st + kStagers, ...: at most kRegPos of them.
    float4 rg[RP];
    int poffR[RP];        // chunk-invariant source offset of the thread's float4 (mode 0: incl. the half's +4)
    int prowR[RP];        // mode 1: first input row (phase row 0), very negative when the column is outside
    uint32_t pvalid = 0;       // mode 0: bit i = the float4 exists and its position is inside an image
    uint32_t phalf = 0;        // mode 0: bit i = second half (channels 4..7 of the chunk)
    if (a.mode != 2) {
#pragma unroll
      for (int i = 0; i < RP; i++) {
        const int p = st + i * NSTG;
        poffR[i] = 0; prowR[i] = -(1 << 28);
        if (p < a.planeF4) {
          const int off = posoff[p];
          if (a.mode == 0) {
            const bool hb = p >= a.NPOS;
            poffR[i] = off + (hb ? 4 : 0);
            if (off >= 0) pvalid |= 1u << i;
            if (hb) phalf |= 1u << i;
          } else {
            poffR[i] = off;
            prowR[i] = posrow[p];
          }
        }
      }
    }
    auto loadPos = [&](int kc) {
      if (a.mode == 0) {
        const int chA = (kcBase + kc) * 8;
        uint32_t m = pvalid;
        if (chA >= a.Cg) m = 0;
        else if (chA + 4 >= a.Cg) m &= ~phalf;
        const float* srcG = srcBase + g * a.Cg + chA;
#pragma unroll
        for (int i = 0; i < RP; i++) {
          rg[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
          if ((m >> i) & 1u) rg[i] = __ldg(reinterpret_cast<const float4*>(srcG + poffR[i]));
        }
      } else {
        const int ph = kcBase + kc;
        const float* srcG = srcBase + static_cast<size_t>(g) * a.Cg * a.chStride + ph * a.rowStride;
#pragma unroll
        for (int i = 0; i < RP; i++) {
          rg[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
          if (static_cast<unsigned>(prowR[i] + ph) < static_cast<unsigned>(a.Hi)) {
            const float* px = srcG + poffR[i];
            rg[i].x = __ldg(px);
            if (a.Cg > 1) rg[i].y = __ldg(px + a.chStride);
            if (a.Cg > 2) rg[i].z = __ldg(px + 2 * a.chStride);
            if (a.Cg > 3) rg[i].w = __ldg(px + 3 * a.chStride);
          }
        }
      }
    };
    fetchChunk(0);
    if (a.mode != 2) loadPos(0);
    if (nChunks > 1) fetchChunk(1);
    for (int kc = 0; kc < nChunks; kc++) {
      const int buf = kc % a.nPB;
      if (!a.bulkC) {
        if (kc + 1 < nChunks) asm volatile("cp.async.wait_group 1;" ::: "memory");   // chunk kc landed, kc+1 may be in flight
        else CpAsyncWaitAll();
        // (each stager arrives after its own copies have landed; the barrier completes when all of them have)
        MbarArrive(fullC + kc % kCbBufs);                  // the consumers may start on chunk kc
      }
      if (kc >= a.nPB) MbarWait<24>(emptyB + buf, ((kc / a.nPB) - 1) & 1);   // planes last read by the MMAs of chunk kc-nPB
      float4* pHi = planes + (buf * 2 + 0) * a.planeRows;
      float4* pLo = planes + (buf * 2 + 1) * a.planeRows;
      if (a.mode == 2) {
        // the plane image of (tile, chunk) was written by fc_prep_kernel: one bulk copy (hi + lo, contiguous) straight
        // into the planes, completion counted on the same mbarrier the stagers arrive on
        if (st == 0) {
          const uint32_t bytes = static_cast<uint32_t>(a.planeRows) * 32u;
          const float* gsrc = a.xprep + (static_cast<size_t>(tile) * a.nChunksAll + (k0 / a.chunkCount[0] + kc)) * a.planeRows * 8;
          MbarExpectTx(fullB + buf, bytes);
          BulkLoad(pHi, gsrc, bytes, fullB + buf);
        } else {
          MbarArrive(fullB + buf);
        }
      } else {
#pragma unroll
        for (int i = 0; i < RP; i++) {
          const int p = st + i * NSTG;
          if (p < a.planeF4) {
            if (BF) {
              uint2 p1, p2;
              SplitBf16x4(rg[i], p1, p2);
              const int db = posdst[p];
              *reinterpret_cast<uint2*>(reinterpret_cast<char*>(pHi) + db) = p1;
              *reinterpret_cast<uint2*>(reinterpret_cast<char*>(pLo) + db) = p2;
            } else {
              float4 hi, lo;
              SplitTf32x4(rg[i], hi, lo);
              pHi[p] = hi;
              pLo[p] = lo;
            }
          }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // planes are read by the tensor core
        MbarArrive(fullB + buf);
        if (kc + 1 < nChunks) loadPos(kc + 1);
      }
      if (kc + 2 < nChunks) {
        const int nb = (kc + 2) % kCbBufs;
        if (kc + 2 >= kCbBufs) MbarWait<24>(emptyC + nb, (((kc + 2) / kCbBufs) - 1) & 1);
        fetchChunk(kc + 2);
      }
    }
    return;
  }

  // =========================== consumers: decode + wgmma ===========================
  // Fragment ownership (wgmma A / D, one 16-row slice per warp): this thread holds rows r0 = 16 * (warp in group) + lane / 4
  // and r0 + 8 of its warpgroup's 64 channels; of a k-step's eight values it holds the pair 2 * (lane % 4), +1 (bf16x2: both
  // copies of [w | w]) or the values lane % 4 of either half (tf32).
  const int gid = lane >> 2, t4 = lane & 3;
  const int row0 = (warp >> 2) * 64 + (warp & 3) * 16 + gid, row1 = row0 + 8;
  const int cc0 = min(row0, CTv - 1), cc1 = min(row1, CTv - 1);   // rows beyond the valid channels decode a copy (never stored)
  const int myHalf = t4 >> 1, myWord = t4 & 1;                    // bf16x2: the half and the value pair inside its piece
  const bool pre = BF && a.cbPre != 0;
  float acc[NT / 2], acc2[CORR ? NT / 2 : 1];
#pragma unroll
  for (int i = 0; i < NT / 2; i++) acc[i] = 0.0f;
#pragma unroll
  for (int i = 0; i < (CORR ? NT / 2 : 1); i++) acc2[i] = 0.0f;
  float (&accLo)[CORR ? NT / 2 : 1] = acc2;
  const uint64_t descFixed = static_cast<uint64_t>(8) << 32;     // SBO = 128 B; LBO and the start address come per k-step
  const uint32_t planes0 = SmemU32(planes);

  for (int kc = 0; kc < nChunks; kc++) {
    const int cbuf = kc % kCbBufs, buf = kc % a.nPB;
    MbarWait<24>(fullC + cbuf, (kc / kCbBufs) & 1);
    const uint8_t* idb = ids + cbuf * a.idRows * 128;
    const float4* cb = cbs + cbuf * a.cbSlots * a.cbF4;
    const float* cbf = reinterpret_cast<const float*>(cb);
    const uint32_t* cbw = reinterpret_cast<const uint32_t*>(cb);
    const int e0 = a.chunkFirst[a.mode == 1 ? kcBase + kc : 0];
    const int ne = a.mode == 2 ? min(a.chunkCount[0], kTotal - kc * a.chunkCount[0]) : a.chunkCount[a.mode == 1 ? kcBase + kc : 0];
    // idxT: every tap index of the thread's two channels for the chunk in registers (one to three 128-bit loads each): the
    // per-k-step chain is one dependent shared-memory round trip (the codeword piece)
    //   mode 0: iq[ch][2 h], iq[ch][2 h + 1] = the taps of half-slot h (bf16x2: the thread's own half; tf32: both halves)
    //   mode 1: iq[ch][0..2] = the <= 48 rows of the phase row
    uint4 iq[2][4];
#pragma unroll
    for (int c = 0; c < 2; c++)
#pragma unroll
      for (int j = 0; j < 4; j++) iq[c][j] = make_uint4(0, 0, 0, 0);
    if (a.idxT) {
      const uint4* ip = reinterpret_cast<const uint4*>(idb);
      const int W = a.tapsPad >> 4;
#pragma unroll
      for (int c = 0; c < 2; c++) {
        const int cc = c ? cc1 : cc0;
        if (a.mode == 1) {
          iq[c][0] = ip[cc * W];
          if (W > 1) iq[c][1] = ip[cc * W + 1];
          if (W > 2) iq[c][2] = ip[cc * W + 2];
        } else {
#pragma unroll
          for (int h = 0; h < (BF ? 1 : 2); h++) {
            const int half = BF ? myHalf : h;
            iq[c][2 * h] = ip[(half * 128 + cc) * W];
            if (W > 1) iq[c][2 * h + 1] = ip[(half * 128 + cc) * W + 1];
          }
        }
      }
    }
    // float4 index (inside the chunk's staged codebook) of the piece that `half` of k-step (ks, tap) takes for channel c
    auto pieceOf = [&](const KStep& ks, int tap, int half, int c) -> int {
      if (a.idxT && a.mode == 1)
        return (half ? ks.cb1 : ks.cb0) * K + ByteOf48(iq[c][0], iq[c][1], iq[c][2], half ? ks.idx1 : ks.idx0);
      if (a.idxT) {
        const int h = BF ? 0 : half;
        return half * K + ByteOf32(iq[c][2 * h], iq[c][2 * h + 1], tap);
      }
      return (half ? ks.cb1 : ks.cb0) * K + (idb[(half ? ks.idx1 : ks.idx0) * 128 + (c ? cc1 : cc0)] >> a.kshift);
    };
    // scalar codewords (d = 1): value j (< 4) of `half` is its own subspace: row / slot idx + j
    auto scalarOf = [&](const KStep& ks, int half, int j, int c) -> float {
      const int row = (half ? ks.idx1 : ks.idx0) + j, slot = (half ? ks.cb1 : ks.cb0) + j;
      return cbf[slot * K + (idb[row * 128 + (c ? cc1 : cc0)] >> a.kshift)];
    };
    MbarWait<24>(fullB + buf, (kc / a.nPB) & 1);
    const uint64_t dHi = descFixed | (((planes0 + static_cast<uint32_t>((buf * 2 + 0) * a.planeRows) * 16u) >> 4) & 0x3FFFu);
    const uint64_t dLo = descFixed | (((planes0 + static_cast<uint32_t>((buf * 2 + 1) * a.planeRows) * 16u) >> 4) & 0x3FFFu);
    for (int s0 = 0; s0 < ne; s0 += GT) {
      const int n = min(GT, ne - s0);
      // the stage's k-steps are independent: index bytes and codeword pieces of all of them are in flight together
      uint32_t fa[kMaxGT][BF ? 4 : 8];
      uint64_t boff[kMaxGT];
#pragma unroll
      for (int i = 0; i < kMaxGT; i++) {
        if (i < n) {
          const KStep ks = (a.idxT || a.mode != 2) ? a.tab[e0 + s0 + i] : tabS[e0 + s0 + i];
          boff[i] = static_cast<uint64_t>(static_cast<uint32_t>(ks.bStart)) | (static_cast<uint64_t>(static_cast<uint32_t>(ks.lbo)) << 16);
          if constexpr (BF) {
            // [w1 | w1] -> fa[0..1] (rows r0, r1; both K halves read the same registers), [w2 | w2] -> fa[2..3]
#pragma unroll
            for (int c = 0; c < 2; c++) {
              if (a.d == 1) {
                const float v0 = scalarOf(ks, myHalf, 2 * myWord, c), v1 = scalarOf(ks, myHalf, 2 * myWord + 1, c);
                const uint32_t p1 = PackBf16x2(v0, v1);
                fa[i][c] = p1;
                fa[i][2 + c] = PackBf16x2(v0 - __uint_as_float(p1 << 16), v1 - __uint_as_float(p1 & 0xFFFF0000u));
              } else {
                const int pi = pieceOf(ks, s0 + i, myHalf, c);
                if (pre) {
                  fa[i][c] = cbw[pi * 4 + myWord];
                  fa[i][2 + c] = cbw[pi * 4 + 2 + myWord];
                } else {
                  const float2 v = reinterpret_cast<const float2*>(cb)[pi * 2 + myWord];
                  const uint32_t p1 = PackBf16x2(v.x, v.y);
                  fa[i][c] = p1;
                  fa[i][2 + c] = PackBf16x2(v.x - __uint_as_float(p1 << 16), v.y - __uint_as_float(p1 & 0xFFFF0000u));
                }
              }
            }
          } else {
            // tf32 fragment: (r0, half 0), (r1, half 0), (r0, half 1), (r1, half 1), value t4 of the half; hi -> fa[0..3], lo -> fa[4..7]
#pragma unroll
            for (int h = 0; h < 2; h++)
#pragma unroll
              for (int c = 0; c < 2; c++) {
                const float v = a.d == 1 ? scalarOf(ks, h, t4, c) : cbf[pieceOf(ks, s0 + i, h, c) * 4 + t4];
                const uint32_t hi = __float_as_uint(v) & 0xFFFFE000u;
                fa[i][2 * h + c] = hi;
                fa[i][4 + 2 * h + c] = __float_as_uint(v - __uint_as_float(hi));
              }
          }
        }
      }
      qcnn::WgmmaFence();
#pragma unroll
      for (int i = 0; i < kMaxGT; i++) {
        if (i < n) {
          if constexpr (BF) {
            // B = [x1 | x2]: K-core-matrix 0 in the first plane, 1 in the second (the table's lbo is the plane distance)
            Wgmma<NT>::Bf16RS(acc, fa[i][0], fa[i][1], fa[i][0], fa[i][1], dHi + boff[i]);
            if constexpr (CORR) Wgmma<NT>::Bf16RS(accLo, fa[i][2], fa[i][3], fa[i][2], fa[i][3], dHi + boff[i]);
            else Wgmma<NT>::Bf16RS(acc, fa[i][2], fa[i][3], fa[i][2], fa[i][3], dHi + boff[i]);
          } else {
            Wgmma<NT>::Tf32RS(acc, fa[i][0], fa[i][1], fa[i][2], fa[i][3], dHi + boff[i]);
            if constexpr (CORR) {
              Wgmma<NT>::Tf32RS(accLo, fa[i][0], fa[i][1], fa[i][2], fa[i][3], dLo + boff[i]);
              Wgmma<NT>::Tf32RS(accLo, fa[i][4], fa[i][5], fa[i][6], fa[i][7], dHi + boff[i]);
            } else {
              Wgmma<NT>::Tf32RS(acc, fa[i][0], fa[i][1], fa[i][2], fa[i][3], dLo + boff[i]);
              Wgmma<NT>::Tf32RS(acc, fa[i][4], fa[i][5], fa[i][6], fa[i][7], dHi + boff[i]);
            }
          }
        }
      }
      qcnn::WgmmaCommit();
      qcnn::WgmmaWaitAll();
    }
    // the chunk's MMAs have retired: its planes and its codebook / index buffer may be refilled
    __syncwarp();
    if (lane == 0) { MbarArrive(emptyB + buf); MbarArrive(emptyC + cbuf); }
  }

  // ---- epilogue: accumulator fragments (rows = channels r0, r1; columns = positions 8 i + 2 t4, +1) -> + bias, ReLU -> NHWC ----
  {
    const bool ok0 = row0 < CTv, ok1 = row1 < CTv;
    const float b0 = biasS[row0], b1 = biasS[row1];
#pragma unroll
    for (int i = 0; i < NT / 8; i++) {
#pragma unroll
      for (int j = 0; j < 2; j++) {
        const int off = outoff[8 * i + 2 * t4 + j];
        if (off < 0) continue;
        float v0 = acc[4 * i + j] + b0, v1 = acc[4 * i + 2 + j] + b1;
        if constexpr (CORR) { v0 += acc2[CORR ? 4 * i + j : 0]; v1 += acc2[CORR ? 4 * i + 2 + j : 0]; }
        if (a.relu) { v0 = fmaxf(v0, 0.0f); v1 = fmaxf(v1, 0.0f); }   // (never set together with split-K partial sums)
        if (ok0) dstBase[off + row0] = v0;
        if (ok1) dstBase[off + row1] = v1;
      }
    }
  }
