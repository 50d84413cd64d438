"""The decode-at-use tensor-core GEMM (pq_gemm_tc) against a float64 reference, at every tiling and at the shapes where its
code paths branch.

Reference and metric
  The weights are decoded once, W[c, kh, kw, cin] = ctrd[s][asmt[c, kh, kw, s]][cin - s d] (only the dims that exist), and
  the convolution (groups, stride, zero padding) or the FC layer (NCHW flatten order) is evaluated in float64.  The same
  code evaluated on |x| and |ctrd| gives the magnitude map M = sum |w x| + |bias|.  The metric is
      err = max |gpu - ref64| / M,
  the natural scale of a floating-point sum's error: it does not depend on how much the sum cancels.  ReLU outputs are
  compared with max(ref64, 0) under the same M (ReLU does not increase a difference).

Error bounds (U = 2^-24), one per numerical class, as a function of the k-steps ks chained in one CTA's accumulator
  operands   bf16x2: x = x1 + x2 with round-to-nearest-even bf16 pieces leaves |x - x1 - x2| <= 2^-17 |x| (the remainder
             is at most half a bf16 ulp of x, and its own rounding at most half a bf16 ulp of that), so one product
             (w1 + w2)(x1 + x2) is off by <= 2^-16 (1 + 2^-18) |w x|.  3xTF32: hi = x truncated to tf32, the remainder is
             read truncated to tf32 too (<= 2^-20 |x| lost) and xl wl is dropped (<= 2^-20 |w x|): <= 3 2^-20 |w x|.
  summation  products of bf16 or tf32 pieces are exact in fp32.  A chained wgmma adds its products to the fp32
             accumulator, whose magnitude stays below M; the tensor core aligns the addends to the largest exponent and
             truncates, which we take as at most 2 ulps of the accumulator, C_MMA U M per chained MMA (C_MMA = 4).
             Chained MMAs per k-step: bf16x2 NT = 128: 2 ([w1|w1].[x1|x2] and [w2|w2].[x1|x2] into one accumulator);
             NT = 64: 1 (the w2 term has an accumulator of its own, whose values are 2^-8 smaller); 3xTF32 NT = 128: 3;
             NT = 64: 1 (plus 2 into the small accumulator).  The epilogue adds bias and the second accumulator, the
             K-split reduction adds nsplit partial sums: (nsplit + 3) U.
      bound = op + (C_MMA (chain + 2^-8 chain_lo) + nsplit + 3) U        (tc_bound)
  The LUT + gather families (tensor_core = 0) add fp32 LUT entries of d products: any order of that sum stays within
  (max(d + taps S, taps min(Cg, d)) + 3) U; the 3xTF32 LUT stage (conv_s1_tc / conv_roll_tc) adds the 3xTF32 operand term
  and one chain of three MMAs (strict_bound).
  Measured worst case on one NVIDIA H100 80GB HBM3 (700 W power limit), max err / bound over this file's cases (with and
  without ReLU): conv bf16x2 NT = 128 0.43 (err 6.9e-6), NT = 64 0.44 (7.2e-6); conv 3xTF32 NT = 128 0.28 (1.1e-6),
  NT = 64 0.26 (8.6e-7); FC bf16x2 NT = 128 0.19, NT = 64 0.09; FC 3xTF32 NT = 128 0.12, NT = 64 0.04; LUT + gather
  families <= 0.30.  The worst cases are the short reductions, where the operand term is nearly reached.  Every case's
  err, bound and plan string go to pq_gemm_f64.json in the directory named by QCNN_REPORT_DIR (default: qcnn_reports
  under the system temporary directory), so that the suite writes nothing into the source tree unless asked to.

What the bounds can catch
  On short reductions (Cg = 8 with 1x1 and 3x3 kernels, an FC layer with Din = 64) the operand term dominates, and
  test_degraded_operands_exceed_bound (CPU) shows that each bound rejects, by at least 4x, every way of losing an operand
  piece: bf16 single piece, x-lo or w-lo dropped, one-pass tf32, 3xTF32 with either cross term dropped.  On the long
  reductions the summation term (~ks U) is larger than those operand errors, so there the bound catches structural
  errors only (a lost k-step, a wrong tap, a wrong codeword; errors of 1e-2 and more).

Coverage
  Every conv case pins family, operand format and the whole tiling (force_kernel = 6, gemm_nt, gemm_gt, gemm_nsplit) and
  asserts the plan from describe() after the forward.  CONV_ROWS is designed to reach every branch of the kernel
  (test_table_reaches_every_branch lists them), and across it every NT x GT x nsplit in {1, >1} x ReLU runs in both
  operand formats.  FC mode 2 has no timed choice; its rows pick (N, Dout) so that nsplit = 1 and nsplit > 1 both occur,
  and the NT = 64 instantiation (reachable only through QCNN_FC_TC=1 at N <= 64) runs in a child process.  Besides:
  neighbour poisoning (an image's output is bit-identical whether the other images are 0 or NaN), the exact write set of
  the output (a NaN-filled guard region around it stays untouched), run-to-run bit identity of a plan, and the LUT +
  gather families on the same table against the same reference.
"""
import collections
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import zlib

import numpy as np
import pytest

from test_gpu_layers import CONV_CASES, CONV_FAMILY_NAMES, FC_CASES, rand_act
from test_oracle_vs_reference import SYNTH, golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))
REPORT = {}

U = 2.0 ** -24
C_MMA = 4
OP_BF = 2.0 ** -16 * (1 + 2.0 ** -18)
OP_TF = 3 * 2.0 ** -20
H100_SMS = 132


# ------------------------------------------------------------------------------------------------------------------
# float64 reference
# ------------------------------------------------------------------------------------------------------------------
def decode_conv_weights(ctrd, asmt, Cg):
    """W[c, kh, kw, cin] in float64 from codebook [S, K, d] and assignments [Cout, k, k, S] (one codebook for all groups)."""
    S, K, d = ctrd.shape
    c64 = np.asarray(ctrd, np.float64)
    W = np.zeros(asmt.shape[:3] + (Cg,), np.float64)
    for s in range(S):
        lo, hi = s * d, min(Cg, (s + 1) * d)
        if lo >= Cg:
            break
        W[..., lo:hi] = c64[s][asmt[..., s]][..., :hi - lo]
    return W


def conv_sum(x, ctrd, asmt, pad, stride, G):
    """sum over taps and input channels of w x, float64, x NHWC [N, H, W, Cin] -> [N, Ho, Wo, Cout] (no bias)."""
    x = np.asarray(x, np.float64)
    Cin = x.shape[3]
    Cout, k = asmt.shape[0], asmt.shape[1]
    Cg, Kg = Cin // G, Cout // G
    W = decode_conv_weights(ctrd, asmt, Cg)
    xp = np.pad(x, ((0, 0), (pad, pad), (pad, pad), (0, 0)))
    win = np.lib.stride_tricks.sliding_window_view(xp, (k, k), axis=(1, 2))[:, ::stride, ::stride]   # [N,Ho,Wo,Cin,k,k]
    out = np.empty(win.shape[:3] + (Cout,), np.float64)
    for g in range(G):
        out[..., g * Kg:(g + 1) * Kg] = np.tensordot(win[:, :, :, g * Cg:(g + 1) * Cg], W[g * Kg:(g + 1) * Kg],
                                                     axes=([3, 4, 5], [3, 1, 2]))
    return out


def fc_sum(x, ctrd, asmt):
    """sum over input features of w x, float64, x [N, Din] (NCHW flatten order) -> [N, Dout] (no bias)."""
    x = np.asarray(x, np.float64)
    N, Din = x.shape
    S, K, d = ctrd.shape
    c64 = np.asarray(ctrd, np.float64)
    out = np.zeros((N, asmt.shape[0]), np.float64)
    for s in range(S):
        lo, hi = s * d, min(Din, (s + 1) * d)
        if lo >= Din:
            break
        lut = x[:, lo:hi] @ c64[s][:, :hi - lo].T          # [N, K]
        out += lut[:, asmt[:, s]]
    return out


def nhwc_flatten(x):
    """NHWC map [N, H, W, C] -> the reference's NCHW-flattened FC input [N, C*H*W]."""
    return np.ascontiguousarray(np.transpose(x, (0, 3, 1, 2))).reshape(x.shape[0], -1)


def ref64(kind, x, ctrd, asmt, bias, geom=None):
    """(ref, M): the layer in float64 and the magnitude map sum |w x| + |bias|."""
    b = np.asarray(bias, np.float64)
    if kind == "conv":
        f = lambda xx, cc: conv_sum(xx, cc, asmt, *geom)
    else:
        f = lambda xx, cc: fc_sum(xx, cc, asmt)
    return f(x, ctrd) + b, f(np.abs(x), np.abs(ctrd)) + np.abs(b)


def f64_err(gpu, ref, mag):
    gpu = np.asarray(gpu, np.float64)
    assert gpu.shape == ref.shape, (gpu.shape, ref.shape)
    if not np.isfinite(gpu).all():
        return float("inf")
    return float((np.abs(gpu - ref) / np.maximum(mag, 1e-30)).max())


def tc_bound(bf, NT, ks, nsplit):
    """Error bound (units of M) of pq_gemm_tc with ks k-steps chained in one accumulator (module docstring)."""
    op = OP_BF if bf else OP_TF
    chain = ks * (2 if bf else 3) if NT == 128 else ks
    chain_lo = 0 if NT == 128 else ks * (1 if bf else 2)
    return op + (C_MMA * (chain + chain_lo * 2.0 ** -8) + nsplit + 3) * U


def strict_bound(family, taps, S, d, Cg):
    """Error bound of the LUT + gather families: fp32 LUT entries of d products gathered over taps x S."""
    b = (max(d + taps * S, taps * min(Cg, d)) + 3) * U
    if family in (2, 3):       # 3xTF32 wgmma LUT stage
        b += OP_TF + 3 * C_MMA * U
    return b


# ------------------------------------------------------------------------------------------------------------------
# numpy emulation of the kernel's operand splits (round-to-nearest-even bf16, tf32 truncation as & 0xFFFFE000)
# ------------------------------------------------------------------------------------------------------------------
def bf16_rn(v):
    u = np.ascontiguousarray(v, np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32).view(np.float32)


def split_bf16(v):
    v = np.asarray(v, np.float32)
    v1 = bf16_rn(v)
    return v1, bf16_rn(v - v1)          # (the remainder is exact in fp32)


def tf32_trunc(v):
    return (np.ascontiguousarray(v, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def split_tf32(v):
    v = np.asarray(v, np.float32)
    hi = tf32_trunc(v)
    return hi, tf32_trunc(v - hi)       # the tensor core reads the remainder as tf32 as well


def operand_variants(x, ctrd):
    """{class: {variant: [(x piece, codebook piece), ...]}} whose products the tensor core would sum; the first variant
    of a class is what the kernel computes, the others lose an operand piece."""
    f = lambda *a: sum(np.asarray(t, np.float64) for t in a)
    x1, x2 = split_bf16(x)
    w1, w2 = split_bf16(ctrd)
    xh, xl = split_tf32(x)
    wh, wl = split_tf32(ctrd)
    return {
        "bf16x2": collections.OrderedDict([
            ("bf16x2 (w1+w2)(x1+x2)", [(f(x1, x2), f(w1, w2))]),
            ("bf16 single piece w1 x1", [(x1, w1)]),
            ("x-lo dropped (w1+w2) x1", [(x1, f(w1, w2))]),
            ("w-lo dropped w1 (x1+x2)", [(f(x1, x2), w1)])]),
        "3xTF32": collections.OrderedDict([
            ("3xTF32 wh xh + wh xl + wl xh", [(xh, wh), (xl, wh), (xh, wl)]),
            ("one-pass tf32 wh xh", [(xh, wh)]),
            ("x-lo dropped wh xh + wl xh", [(xh, wh), (xh, wl)]),
            ("w-lo dropped wh xh + wh xl", [(xh, wh), (xl, wh)])]),
    }


# ------------------------------------------------------------------------------------------------------------------
# the designed shape table
# ------------------------------------------------------------------------------------------------------------------
Row = collections.namedtuple("Row", "name N Hi Wi Cin Cout k pad stride G S K d nchw")
CONV_ROWS = [
    # mode 0 (stride 1): channel tiles, chunk counts, half-B masking, partial subspaces, index staging, grid edges
    Row("kg16_1x1_cg8", 6, 9, 9, 8, 16, 1, 0, 1, 1, 1, 64, 8, False),       # CTv = 16, one k-step per chunk (< GT)
    Row("kg48_3x3_cg8", 4, 10, 11, 8, 48, 3, 1, 1, 1, 2, 32, 4, False),     # CTv = 48, d = 4, one chunk
    Row("g2_cg12_kg80_pad2", 3, 12, 10, 24, 160, 3, 2, 1, 2, 2, 128, 8, False),  # Cg % 8 == 4, S d > Cg, pad = k-1
    Row("tiny_images_pad2", 40, 3, 3, 16, 64, 3, 2, 1, 1, 4, 16, 4, False),  # 25-position images: a tile spans ~5
    Row("d12_cg36_kg144", 2, 8, 8, 36, 144, 3, 1, 1, 1, 3, 64, 12, False),   # 5 chunks, nct = 2 with a 16-channel tile
    Row("d16_kg192_5x5", 2, 7, 9, 32, 192, 5, 2, 1, 1, 2, 128, 16, False),   # 4 chunks, nct = 2 with a 64-channel tile
    Row("k7_tap_rows", 2, 9, 9, 24, 32, 7, 3, 1, 1, 3, 64, 8, False),        # 49 taps: tap-row cp.async, 3 chunks
    Row("k9_tap_rows", 2, 10, 10, 8, 64, 9, 4, 1, 1, 1, 32, 8, False),       # 81 taps
    Row("cg80_10_chunks", 2, 6, 6, 80, 128, 3, 1, 1, 1, 10, 256, 8, False),  # 10 chunks (> 2 turns of the ring)
    Row("plane_limit_w318", 1, 2, 318, 8, 32, 3, 1, 1, 1, 2, 16, 4, False),  # planeF4 = 1536 at NT = 128
    Row("cg4_valid", 3, 11, 7, 4, 32, 3, 0, 1, 1, 1, 128, 4, False),         # Cg = 4: second half masked throughout
    Row("g2_cg20_k5_pad4", 2, 6, 6, 40, 96, 5, 4, 1, 2, 5, 32, 4, False),    # Cg = 20, Kg = 48, pad = k-1
    # mode 1 (strided, Cg <= 4, S = 1): strides 2-4, paired / unpaired taps, groups, NCHW source
    Row("s4_k11_cg3", 2, 39, 39, 3, 64, 11, 0, 4, 1, 1, 128, 8, False),      # conv1-like
    Row("s2_k3_cg1_nchw", 5, 13, 12, 1, 32, 3, 1, 2, 1, 1, 16, 4, True),
    Row("s3_k5_g2_cg2", 3, 17, 16, 4, 64, 5, 2, 3, 2, 1, 64, 4, False),      # odd stride: bf16x2 not eligible
    Row("s2_k7_cg4", 2, 21, 21, 4, 48, 7, 3, 2, 1, 1, 32, 4, False),
    Row("s4_k9_cg2_nchw", 3, 25, 25, 2, 16, 9, 1, 4, 1, 1, 128, 8, True),
    # not eligible for the tensor-core GEMM in either format
    Row("s1_k11_ineligible", 1, 13, 13, 4, 16, 11, 0, 1, 1, 1, 32, 4, False),  # 121 taps
    Row("cg6_ineligible", 2, 7, 7, 6, 32, 3, 1, 1, 1, 1, 32, 8, False),         # Cg % 4 != 0
]
ROWS = {r.name: r for r in CONV_ROWS}

FcRow = collections.namedtuple("FcRow", "name N Din Dout S K d nhwc")
FC_ROWS = [
    FcRow("din64_short", 96, 64, 256, 16, 16, 4, None),
    FcRow("d16_partial_sub", 129, 1000, 200, 63, 64, 16, None),    # Din = 1000: the last subspace has 8 of 16 dims
    FcRow("d1_k256", 300, 512, 128, 512, 256, 1, None),
    FcRow("d12_k128", 100, 480, 96, 40, 128, 12, None),
    FcRow("d8_nhwc_fold", 130, 512, 64, 64, 64, 8, (4, 4, 32)),
    FcRow("nsplit1_n1100", 1100, 64, 2048, 8, 16, 8, None),         # 9 tiles x 16 channel tiles >= 132 CTAs: no split
]
FC_NT64_ROWS = [
    FcRow("nt64_n64", 64, 256, 160, 32, 32, 8, None),
    FcRow("nt64_n33_d12", 33, 240, 48, 20, 64, 12, None),
]


def _ceil(a, b):
    return -(-a // b)


def _rup(a, b):
    return _ceil(a, b) * b


def mode1_counts(k, st, bf):
    """k-steps of every phase row of a strided layer (mirror of PlanPqGemm's tap pairing)."""
    counts = []
    for ph in range(st):
        c = 0
        for _kh in range(ph, k, st):
            kw = 0
            while kw < k:
                paired = kw + 1 < k and (kw % st) + 1 < st and not (bf and ((kw % st) & 1))
                c += 1
                kw += 2 if paired else 1
        counts.append(c)
    return counts


def geometry(row):
    """(mode, IB, NPOS(NT), per-chunk k-steps(bf)) of a TC-eligible row, or None (mirror of PlanPqGemm's eligibility)."""
    Cg, Kg = row.Cin // row.G, row.Cout // row.G
    k, st, pad = row.k, row.stride, row.pad
    if row.K > 256 or Kg % 16:
        return None
    if st > 1:
        PWp, PHp = _ceil(row.Wi + 2 * pad, st), _ceil(row.Hi + 2 * pad, st)
        Wo = (row.Wi + 2 * pad - k) // st + 1
        pairs = (k + 1) // 2
        if Cg > 4 or row.S != 1 or row.d < Cg or st > 8 or Wo > PWp or _ceil(k, st) * pairs > 32 or k * pairs > 96:
            return None
        return (1, PHp * PWp, lambda NT: _rup(NT + ((k - 1) // st) * (PWp + 1), 8) * st,
                lambda bf: mode1_counts(k, st, bf))
    if row.nchw or row.d % 4 or Cg % 4 or row.Cin % 4 or row.S * row.d < Cg or k * k > 96:
        return None
    PW = row.Wi + pad
    return (0, (row.Hi + pad) * PW, lambda NT: 2 * _rup(NT + (k - 1) * (PW + 1), 8),
            lambda bf: [k * k] * _ceil(Cg, 8))


def tc_space(row, bf, sms):
    """[(NT, GT, nsplit, ks)] of the pq_gemm_tc tilings the planner offers for row at batch row.N on sms SMs."""
    g = geometry(row)
    if g is None or (bf and row.stride > 1 and row.stride % 2):
        return []
    mode, IB, planeF4, counts_of = g
    counts = counts_of(bf)
    nChunks, nct = len(counts), _ceil(row.Cout // row.G, 128)
    out = []
    for NT in (128, 64):
        if planeF4(NT) > 1536:
            continue
        ctas0 = _ceil(row.N * IB, NT) * row.G * nct
        for GT in (4, 3):
            ns = 1
            while ns <= nChunks:
                if ns > 1 and ctas0 * ns > 1.5 * sms:
                    break
                kper = _ceil(nChunks, ns)
                if _ceil(nChunks, kper) == ns:
                    out.append((NT, GT, ns, max(sum(counts[i:i + kper]) for i in range(0, nChunks, kper))))
                ns *= 2
    return out


def tc_pins(row, bf, sms=H100_SMS):
    """Tilings each row runs: every (NT, GT) with nsplit = 1 and with the largest split the batch admits."""
    sp = tc_space(row, bf, sms)
    pins = []
    for NT in (128, 64):
        for GT in (4, 3):
            splits = sorted(ns for (a, b, ns, _) in sp if (a, b) == (NT, GT))
            if splits:
                pins += [(NT, GT, 1)] + ([(NT, GT, splits[-1])] if splits[-1] > 1 else [])
    return pins


def fmt(bf):
    return "bf16x2" if bf else "3xTF32"


TC_PINS = [pytest.param(r, bf, NT, GT, ns, id="%s-N%d-%s-NT%d-GT%d-ns%d" % (r.name, r.N, fmt(bf), NT, GT, ns))
           for r in CONV_ROWS for bf in (True, False) for (NT, GT, ns) in tc_pins(r, bf)]
INELIGIBLE = [pytest.param(r, bf, id="%s-%s" % (r.name, fmt(bf))) for r in CONV_ROWS for bf in (True, False)
              if not tc_space(r, bf, H100_SMS)]


def fc_plan(N, Din, Dout, sms):
    """(NT, nsplit, k-steps per split) PlanFcMode2 derives for batch N."""
    NT = 128 if N > 64 else 64
    tiles, nct, kall = _ceil(N, NT), _ceil(Dout, 128), Din // 8
    ns = max(1, sms // (tiles * nct))
    kper = _rup(_ceil(kall, ns), 3)
    return NT, _ceil(kall, kper), kper


FC_PARAMS = [pytest.param(r, bf, id="%s-N%d-%s-NT%d-GT3-ns%d" % ((r.name, r.N, fmt(bf)) + fc_plan(r.N, r.Din, r.Dout, H100_SMS)[:2]))
             for r in FC_ROWS for bf in (True, False)]


# ------------------------------------------------------------------------------------------------------------------
# data
# ------------------------------------------------------------------------------------------------------------------
def _seed(name):
    return zlib.crc32(name.encode()) & 0x7FFFFFFF


def conv_data(row):
    rng = np.random.RandomState(_seed(row.name))
    fan = (row.Cin // row.G) * row.k * row.k
    ctrd = (rng.randn(row.S, row.K, row.d) / np.sqrt(fan)).astype(np.float32)
    asmt = rng.randint(0, row.K, size=(row.Cout, row.k, row.k, row.S)).astype(np.uint8)
    bias = (rng.randn(row.Cout) * 0.1).astype(np.float32)
    x = rand_act(rng, (row.N, row.Hi, row.Wi, row.Cin), scale=4.0)
    return x, ctrd, asmt, bias


def fc_data(row):
    rng = np.random.RandomState(_seed(row.name))
    ctrd = (rng.randn(row.S, row.K, row.d) / np.sqrt(row.Din)).astype(np.float32)
    asmt = rng.randint(0, row.K, size=(row.Dout, row.S)).astype(np.uint8)
    bias = (rng.randn(row.Dout) * 0.1).astype(np.float32)
    shape = (row.N,) + tuple(row.nhwc) if row.nhwc else (row.N, row.Din)
    x = rand_act(rng, shape, scale=4.0)
    return x, ctrd, asmt, bias


def fc_input(row, x):
    return nhwc_flatten(x) if row.nhwc else x


# ------------------------------------------------------------------------------------------------------------------
# CPU: the reference itself, the discrimination of the bounds, the table's coverage
# ------------------------------------------------------------------------------------------------------------------
def _oracle_bound(n_terms, d):
    n = n_terms + d + 2
    return n * U / (1 - n * U)


@pytest.mark.parametrize("case", CONV_CASES)
def test_ref64_conv_matches_oracle(case, po):
    """The fp32 oracle (pinned bit-for-bit to the reference implementation by test_oracle_vs_reference) stays within
    the fp32 summation bound of the float64 reference: LUT entries of d products, then k*k*S lookups."""
    N, Hi, Wi, Cin, Cout, k, pad, stride, G, S, K, d = case
    rng = np.random.RandomState(hash(case) % (2 ** 31))
    ctrd = (rng.randn(S, K, d) * 0.05).astype(np.float32)
    asmt = rng.randint(0, K, size=(Cout, k, k, S)).astype(np.uint8)
    bias = (rng.randn(Cout) * 0.1).astype(np.float32)
    x = rand_act(rng, (N, Hi, Wi, Cin))
    ora = po.conv_aprx(x, po.conv(pad, k, Cout, G, stride), ctrd, asmt, bias)
    ref, mag = ref64("conv", x, ctrd, asmt, bias, (pad, stride, G))
    assert f64_err(ora, ref, mag) <= _oracle_bound(k * k * S, d), f64_err(ora, ref, mag)


@pytest.mark.parametrize("case", FC_CASES + [(5, 6 * 6 * 32, 128, 288, 32, 4, "nhwc")])
def test_ref64_fc_matches_oracle(case, po):
    N, Din, Dout, S, K, d = case[:6]
    rng = np.random.RandomState(hash(case[:6]) % (2 ** 31))
    ctrd = (rng.randn(S, K, d) * 0.05).astype(np.float32)
    asmt = rng.randint(0, K, size=(Dout, S)).astype(np.uint8)
    bias = (rng.randn(Dout) * 0.1).astype(np.float32)
    if len(case) > 6:   # NHWC source: the oracle's permute against nhwc_flatten
        xm = rand_act(rng, (N, 6, 6, 32))
        ora = po.fc_aprx(po.nhwc_to_nchw(xm).reshape(N, -1), ctrd, asmt, bias)
        x = nhwc_flatten(xm)
    else:
        x = rand_act(rng, (N, Din))
        ora = po.fc_aprx(x, ctrd, asmt, bias)
    ref, mag = ref64("fc", x, ctrd, asmt, bias)
    assert f64_err(ora, ref, mag) <= _oracle_bound(S, d), f64_err(ora, ref, mag)


@pytest.mark.parametrize("name", sorted(SYNTH))
def test_ref64_matches_reference_golden(name):
    """Directly against the outputs of the compiled reference implementation (tests/golden/synth_layers.npz)."""
    g = golden("synth_layers.npz")
    kind, spec, chw = SYNTH[name]
    x = g[name + "_fm0"]
    ctrd, asmt, bias = g[name + "_ctrd0"], g[name + "_asmt0"], g[name + "_bias0"]
    S, K, d = ctrd.shape
    if kind == "conv":
        pad, k, cnt, grp, stride = spec
        ref, mag = ref64("conv", x, ctrd, asmt, bias, (pad, stride, grp))
        n = k * k * S
    else:
        ref, mag = ref64("fc", nhwc_flatten(x), ctrd, asmt, bias)
        n = S
    got = g[name + "_fm1"].reshape(ref.shape)
    assert f64_err(got, ref, mag) <= _oracle_bound(n, d), f64_err(got, ref, mag)


DISCRIM_SHAPES = {
    # short reductions: name -> (kind, row); ks = k-steps chained without a K-split
    "conv_1x1_cg8": ("conv", ROWS["kg16_1x1_cg8"]),
    "conv_3x3_cg8": ("conv", ROWS["kg48_3x3_cg8"]),
    "fc_din64": ("fc", FC_ROWS[0]),
}


@pytest.mark.parametrize("shape", sorted(DISCRIM_SHAPES))
def test_degraded_operands_exceed_bound(shape):
    """The class bounds reject a lost operand piece on short reductions: each degraded variant, emulated in numpy on the
    same tensors with the kernel's exact splits, errs by >= 4x the bound of every class it would belong to, while the
    correct split stays within its operand term (the per-product claim of DESIGN.md 2 included)."""
    kind, row = DISCRIM_SHAPES[shape]
    if kind == "conv":
        x, ctrd, asmt, bias = conv_data(row)
        geom = (row.pad, row.stride, row.G)
        bil = lambda xx, cc: conv_sum(xx, cc, asmt, *geom)
        ks = row.k * row.k * _ceil(row.Cin // row.G, 8)
    else:
        x, ctrd, asmt, bias = fc_data(row)
        x = fc_input(row, x)
        bil = lambda xx, cc: fc_sum(xx, cc, asmt)
        ks = row.Din // 8
    ref, mag = ref64(kind, x, ctrd, asmt, bias, geom if kind == "conv" else None)
    lines = []
    for cls, variants in operand_variants(x, ctrd).items():
        bf = cls == "bf16x2"
        bounds = {NT: tc_bound(bf, NT, ks, 1) for NT in (128, 64)}
        for i, (vname, terms) in enumerate(variants.items()):
            y = sum(bil(xx, cc) for xx, cc in terms) + np.asarray(bias, np.float64)
            e = f64_err(y, ref, mag)
            lines.append("%-14s %-32s err %.3e  bound NT=128 %.3e  NT=64 %.3e" % (shape, vname, e, bounds[128], bounds[64]))
            if i == 0:
                assert e <= (OP_BF if bf else OP_TF), (vname, e)
            else:
                assert e >= 4 * max(bounds.values()), (vname, e, bounds)
    print("\n" + "\n".join(lines))
    # per product: |(w1 + w2)(x1 + x2) - w x| <= 2^-16 (1 + 2^-18) |w x| and the 3xTF32 counterpart
    w = np.unique(np.asarray(ctrd, np.float32).ravel())[:3000]
    v = np.asarray(x, np.float32).ravel()[:3000]
    v = v[v != 0]
    exact = np.outer(w.astype(np.float64), v.astype(np.float64))
    (w1, w2), (v1, v2) = split_bf16(w), split_bf16(v)
    pb = np.outer(w1.astype(np.float64) + w2, v1.astype(np.float64) + v2)
    assert (np.abs(pb - exact) <= OP_BF * np.abs(exact)).all()
    (wh, wl), (vh, vl) = split_tf32(w), split_tf32(v)
    pt = np.outer(wh.astype(np.float64), vh) + np.outer(wh.astype(np.float64), vl) + np.outer(wl.astype(np.float64), vh)
    assert (np.abs(pt - exact) <= OP_TF * np.abs(exact)).all()


def test_table_reaches_every_branch():
    """CONV_ROWS / FC_ROWS are designed, not sampled: every branch of pq_gemm_tc named here is reached, and every
    NT x GT x nsplit in {1, >1} runs in both operand formats (each pin runs with and without ReLU)."""
    combos = {(bf, NT, GT, ns > 1) for r in CONV_ROWS for bf in (True, False) for (NT, GT, ns) in tc_pins(r, bf)}
    assert combos == {(bf, NT, GT, sp) for bf in (True, False) for NT in (128, 64) for GT in (4, 3) for sp in (False, True)}
    tc = [r for r in CONV_ROWS if tc_pins(r, False)]
    m0 = [r for r in tc if r.stride == 1]
    m1 = [r for r in tc if r.stride > 1]
    Kg = {r.Cout // r.G for r in tc}
    Cg = lambda r: r.Cin // r.G
    assert {16, 48, 80, 144, 192} <= Kg                                          # CTv < 128, nct = 2 with a partial tile
    assert any(Cg(r) % 8 == 4 for r in m0) and any(r.S * r.d > Cg(r) for r in m0)
    assert {4, 12, 16} <= {r.d for r in m0}
    assert {r.k * r.k > 32 for r in m0} == {True, False} and {7, 9} <= {r.k for r in m0}   # idxT and tap rows
    assert {1, 2, 3, 4, 5} <= {_ceil(Cg(r), 8) for r in m0} and max(_ceil(Cg(r), 8) for r in m0) > 8
    assert any(r.k == 1 for r in m0) and any(r.pad == r.k - 1 and r.k > 1 for r in m0)
    assert any((r.Hi + r.pad) * (r.Wi + r.pad) < 64 and r.N > 8 for r in m0)      # a tile spans many images
    assert any(geometry(r)[2](128) == 1536 for r in m0)
    assert any((r.N * geometry(r)[1]) % 64 for r in m0) and any((r.N * geometry(r)[1]) % 64 for r in m1)  # tails
    assert {2, 3, 4} <= {r.stride for r in m1} and {1, 2, 3, 4} <= {Cg(r) for r in m1}
    assert any(r.G > 1 for r in m1) and any(r.nchw for r in m1) and {3, 5, 7, 9, 11} <= {r.k for r in m1}
    assert any(not tc_pins(r, True) and tc_pins(r, False) for r in m1)             # odd stride: no bf16x2
    assert {1, 4, 8, 12, 16} <= {r.d for r in FC_ROWS + FC_NT64_ROWS}
    assert {16, 64, 128, 256} <= {r.K for r in FC_ROWS}
    assert {96, 129, 300} <= {r.N for r in FC_ROWS} and any(r.nhwc for r in FC_ROWS)
    assert {fc_plan(r.N, r.Din, r.Dout, H100_SMS)[1] > 1 for r in FC_ROWS} == {True, False}
    assert any(r.Din % 16 and r.S * r.d > r.Din for r in FC_ROWS)
    assert INELIGIBLE


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def save_report():
    out = os.environ.get("QCNN_REPORT_DIR") or os.path.join(tempfile.gettempdir(), "qcnn_reports")
    try:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "pq_gemm_f64.json"), "w") as f:
            json.dump(REPORT, f, indent=1, sort_keys=True)
    except OSError:
        pass


class _Cache(object):
    """One layer, input and float64 reference per row, shared by the cases of the module."""

    def __init__(self, qcnn, ctx):
        self.qcnn, self.ctx, self.items = qcnn, ctx, {}

    def conv(self, row):
        if row.name not in self.items:
            import torch
            x, ctrd, asmt, bias = conv_data(row)
            L = self.qcnn.ConvLayer(self.ctx, row.Cin, row.Hi, row.Wi, row.Cout, row.k, row.pad, row.stride, row.G,
                                    ctrd, asmt, bias)
            ref, mag = ref64("conv", x, ctrd, asmt, bias, (row.pad, row.stride, row.G))
            self.items[row.name] = dict(L=L, x=x, xd=torch.from_numpy(x).cuda(),
                                        xn=torch.from_numpy(np.ascontiguousarray(x.transpose(0, 3, 1, 2))).cuda(),
                                        ref=ref, mag=mag)
        return self.items[row.name]

    def close(self):
        for it in self.items.values():
            it["L"].close()


@pytest.fixture(scope="module")
def cache(qcnn, ctx):
    c = _Cache(qcnn, ctx)
    yield c
    c.close()


def pin(L, tc, kernel=6, nt=0, gt=0, ns=0):
    L.set_param("tensor_core", tc)
    L.set_param("force_kernel", kernel)
    L.set_param("gemm_nt", nt)
    L.set_param("gemm_gt", gt)
    L.set_param("gemm_nsplit", ns)


def conv_src(row, it, L, nchw=None):
    nchw = row.nchw if nchw is None else nchw
    if row.stride > 1:
        L.set_src_nchw(nchw)
    return it["xn"] if nchw else it["xd"]


def assert_plan(desc, mode, bf, NT, GT, ns):
    assert desc.startswith("pq_gemm_tc("), desc
    for f in ("mode=%d" % mode, "NT=%d" % NT, "GT=%d" % GT, "nsplit=%d" % ns):
        assert " %s " % f in desc + " ", (f, desc)
    assert ("bf16x2" in desc) == bf, desc


def bits(y):
    return np.ascontiguousarray(y, np.float32).view(np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize("row,bf,NT,GT,ns", TC_PINS)
def test_conv_pinned_tiling_f64(row, bf, NT, GT, ns, cache, ctx):
    space = {(a, b, c): ks for (a, b, c, ks) in tc_space(row, bf, ctx.sm_count)}
    if (NT, GT, ns) not in space:
        pytest.skip("tiling not offered on a GPU with %d SMs" % ctx.sm_count)
    it = cache.conv(row)
    L = it["L"]
    pin(L, 2 if bf else 1, 6, NT, GT, ns)
    xd = conv_src(row, it, L)
    y = L.forward(xd).cpu().numpy()
    desc = L.describe(row.N)          # after the forward: the plan that just ran
    assert_plan(desc, 1 if row.stride > 1 else 0, bf, NT, GT, ns)
    bound = tc_bound(bf, NT, space[(NT, GT, ns)], ns)
    e = f64_err(y, it["ref"], it["mag"])
    # same plan, same sums: bit-identical run to run
    y2 = L.forward(xd).cpu().numpy()
    yr = L.forward(xd, relu=True).cpu().numpy()
    er = f64_err(yr, np.maximum(it["ref"], 0), it["mag"])
    REPORT["conv/%s/N=%d/%s/NT=%d/GT=%d/nsplit=%d" % (row.name, row.N, fmt(bf), NT, GT, ns)] = {
        "plan": desc, "err": e, "err_relu": er, "bound": bound, "ksteps": space[(NT, GT, ns)]}
    save_report()
    assert e <= bound, (e, bound, desc)
    assert er <= bound, (er, bound, desc)
    assert np.array_equal(bits(y), bits(y2))


@pytest.mark.gpu
@pytest.mark.parametrize("row,bf", INELIGIBLE)
def test_conv_ineligible_plan_says_so(row, bf, qcnn, cache):
    """Where the tensor-core GEMM is not eligible the plan names the LUT + gather family that runs instead."""
    it = cache.conv(row)
    L = it["L"]
    pin(L, 2 if bf else 1, -1)
    y = L.forward(conv_src(row, it, L)).cpu().numpy()
    desc = L.describe(row.N)
    assert not desc.startswith("pq_gemm_tc"), desc
    fam = [f for f, p in CONV_FAMILY_NAMES.items() if desc.startswith(p)]
    assert len(fam) == 1, desc
    bound = strict_bound(fam[0], row.k * row.k, row.S, row.d, row.Cin // row.G)
    e = f64_err(y, it["ref"], it["mag"])
    REPORT["ineligible/%s/%s" % (row.name, fmt(bf))] = {"plan": desc, "err": e, "bound": bound}
    save_report()
    assert e <= bound, (e, bound, desc)
    # a pq_gemm_tc pin on such a layer is an error, not a silent change of family
    L.set_param("force_kernel", 6)
    with pytest.raises(qcnn.QcnnError):
        L.describe(row.N)


@pytest.mark.gpu
@pytest.mark.parametrize("row", CONV_ROWS, ids=[r.name for r in CONV_ROWS])
def test_conv_strict_families_f64(row, qcnn, cache):
    """tensor_core = 0, each LUT + gather family pinned where it has a tiling, against the same float64 reference."""
    it = cache.conv(row)
    L = it["L"]
    ran = []
    for fam, prefix in sorted(CONV_FAMILY_NAMES.items()):
        pin(L, 0, fam)
        xd = conv_src(row, it, L, nchw=False)
        try:
            desc = L.describe(row.N)
        except qcnn.QcnnError as ex:
            assert "has no tiling" in str(ex), str(ex)
            continue
        assert desc.startswith(prefix), desc
        y = L.forward(xd).cpu().numpy()
        bound = strict_bound(fam, row.k * row.k, row.S, row.d, row.Cin // row.G)
        e = f64_err(y, it["ref"], it["mag"])
        REPORT["strict/%s/%s" % (row.name, prefix.strip(" ("))] = {"plan": desc, "err": e, "bound": bound}
        assert e <= bound, (fam, e, bound, desc)
        ran.append(fam)
    save_report()
    assert ran


@pytest.mark.gpu
def test_conv_unmatched_pin_fails(qcnn, cache):
    row = ROWS["kg16_1x1_cg8"]          # one 8-channel chunk: no K-split exists
    L = cache.conv(row)["L"]
    for name, value in (("gemm_nsplit", 2), ("gemm_gt", 5), ("gemm_nt", 96)):
        pin(L, 2, 6)
        L.set_param(name, value)
        with pytest.raises(qcnn.QcnnError, match="%s=%d" % (name, value)):
            L.describe(row.N)


def _fc_layer(qcnn, ctx, row, ctrd, asmt, bias):
    L = qcnn.FcLayer(ctx, row.Din, ctrd, asmt, bias)
    if row.nhwc:
        L.set_src_nhwc(*row.nhwc)
    return L


def _ksteps(desc):
    return int(desc.split("ksteps=")[1].split()[0])


@pytest.mark.gpu
@pytest.mark.parametrize("row,bf", FC_PARAMS)
def test_fc_mode2_f64(row, bf, qcnn, ctx):
    import torch
    x, ctrd, asmt, bias = fc_data(row)
    ref, mag = ref64("fc", fc_input(row, x), ctrd, asmt, bias)
    L = _fc_layer(qcnn, ctx, row, ctrd, asmt, bias)
    L.set_param("tensor_core", 2 if bf else 1)
    xd = torch.from_numpy(x).cuda().view(row.N, -1)
    y = L.forward(xd).cpu().numpy()
    desc = L.describe(row.N)
    NT, ns, _ = fc_plan(row.N, row.Din, row.Dout, ctx.sm_count)
    assert " via pq_gemm_tc(" in desc, desc
    assert_plan(desc.split(" via ")[1], 2, bf, NT, 3, ns)
    bound = tc_bound(bf, NT, _ksteps(desc), ns)
    e = f64_err(y, ref, mag)
    y2 = L.forward(xd).cpu().numpy()
    er = f64_err(L.forward(xd, relu=True).cpu().numpy(), np.maximum(ref, 0), mag)
    L.close()
    REPORT["fc/%s/N=%d/%s/NT=%d/nsplit=%d" % (row.name, row.N, fmt(bf), NT, ns)] = {
        "plan": desc, "err": e, "err_relu": er, "bound": bound, "ksteps": _ksteps(desc)}
    save_report()
    assert e <= bound, (e, bound, desc)
    assert er <= bound, (er, bound, desc)
    assert np.array_equal(bits(y), bits(y2))


_CHILD = r"""
import importlib, json, sys
sys.path[:0] = [%r, %r]
import numpy as np, torch
import test_gpu_pq_gemm as t
q = importlib.import_module("quantized-cnn_b200")
ctx = q.Context(0)
res = []
for row in t.FC_NT64_ROWS:
    x, ctrd, asmt, bias = t.fc_data(row)
    ref, mag = t.ref64("fc", t.fc_input(row, x), ctrd, asmt, bias)
    L = q.FcLayer(ctx, row.Din, ctrd, asmt, bias)
    xd = torch.from_numpy(x).cuda().view(row.N, -1)
    for tc in (2, 1):
        L.set_param("tensor_core", tc)
        y = L.forward(xd).cpu().numpy()
        y2 = L.forward(xd).cpu().numpy()
        yr = L.forward(xd, relu=True).cpu().numpy()
        res.append(dict(name=row.name, N=row.N, Din=row.Din, Dout=row.Dout, tc=tc, plan=L.describe(row.N),
                        err=t.f64_err(y, ref, mag), err_relu=t.f64_err(yr, np.maximum(ref, 0), mag),
                        same=bool(np.array_equal(t.bits(y), t.bits(y2)))))
    L.close()
ctx.close()
print("RESULT " + json.dumps(res))
"""


@pytest.mark.gpu
def test_fc_mode2_nt64_child_process():
    """The NT = 64 instantiation of mode 2 runs only when QCNN_FC_TC=1 (read once per process) sends N <= 64 to the
    tensor cores: a child process with that environment."""
    env = dict(os.environ, QCNN_FC_TC="1")
    p = subprocess.run([sys.executable, "-c", _CHILD % (ROOT, TESTS)], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-4000:]
    res = json.loads([l for l in p.stdout.splitlines() if l.startswith("RESULT ")][-1][7:])
    assert len(res) == 2 * len(FC_NT64_ROWS)
    for r in res:
        bf = r["tc"] == 2
        assert " via " in r["plan"], r["plan"]
        desc = r["plan"].split(" via ")[1]
        ns = int(desc.split("nsplit=")[1].split()[0])
        assert_plan(desc, 2, bf, 64, 3, ns)
        r["bound"] = tc_bound(bf, 64, _ksteps(desc), ns)
        REPORT["fc_nt64/%s/N=%d/%s" % (r["name"], r["N"], fmt(bf))] = r
        save_report()
        assert r["err"] <= r["bound"] and r["err_relu"] <= r["bound"], r
        assert r["same"], r


def _pins_for_isolation(row, bf, sms):
    sp = tc_space(row, bf, sms)
    first = [(a, b, c) for (a, b, c, _) in sp if (a, b, c) == (128, 4, 1)]
    split = [(a, b, c) for (a, b, c, _) in sp if a == 64 and b == 3 and c > 1]
    return first + split[-1:]


POISON_CONV = [pytest.param(ROWS[n], bf, id="%s-%s" % (n, fmt(bf)))
               for n in ("tiny_images_pad2", "g2_cg20_k5_pad4", "s2_k3_cg1_nchw", "s2_k7_cg4", "s4_k11_cg3")
               for bf in (True, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("row,bf", POISON_CONV)
def test_conv_neighbour_poison(row, bf, cache, ctx):
    """Image i's output is bit-identical whether every other image is 0 or NaN (tiles straddle image boundaries)."""
    import torch
    it = cache.conv(row)
    L = it["L"]
    i = (row.N - 1) // 2              # an image with a successor: its last positions' taps reach into the next image
    pins = _pins_for_isolation(row, bf, ctx.sm_count)
    assert pins
    for (NT, GT, ns) in pins:
        pin(L, 2 if bf else 1, 6, NT, GT, ns)
        outs = []
        for fill in (0.0, np.nan):
            xp = np.full_like(it["x"], fill)
            xp[i] = it["x"][i]
            if row.nchw:
                xp = np.ascontiguousarray(xp.transpose(0, 3, 1, 2))
            conv_src(row, it, L)
            outs.append(L.forward(torch.from_numpy(xp).cuda()).cpu().numpy()[i])
        assert_plan(L.describe(row.N), 1 if row.stride > 1 else 0, bf, NT, GT, ns)
        assert np.array_equal(bits(outs[0]), bits(outs[1])), (NT, GT, ns)
        assert f64_err(outs[0], it["ref"][i], it["mag"][i]) <= tc_bound(bf, NT, 10 ** 4, ns)


@pytest.mark.gpu
@pytest.mark.parametrize("bf", [True, False], ids=fmt)
def test_fc_neighbour_poison(bf, qcnn, ctx):
    import torch
    row = FC_ROWS[1]
    x, ctrd, asmt, bias = fc_data(row)
    L = _fc_layer(qcnn, ctx, row, ctrd, asmt, bias)
    L.set_param("tensor_core", 2 if bf else 1)
    outs = []
    for i in (0, 64, 128):
        for fill in (0.0, np.nan):
            xp = np.full_like(x, fill)
            xp[i] = x[i]
            outs.append(L.forward(torch.from_numpy(xp).cuda()).cpu().numpy()[i])
        assert np.array_equal(bits(outs[-2]), bits(outs[-1])), i
    assert "pq_gemm_tc(" in L.describe(row.N)
    L.close()


SENTINEL = 0x7FC0BEEF     # a quiet NaN no kernel writes
GUARD = 4096              # floats on either side of the output


def _guarded_call(fn, n_out, relu):
    import torch
    buf = torch.full((n_out + 2 * GUARD,), SENTINEL, dtype=torch.int32, device="cuda")
    dst = ctypes.c_void_p(buf.data_ptr() + 4 * GUARD)
    fn(dst, relu)
    torch.cuda.synchronize()
    h = buf.cpu().numpy()
    out = h[GUARD:GUARD + n_out].view(np.float32)
    guard_ok = (h[:GUARD] == SENTINEL).all() and (h[GUARD + n_out:] == SENTINEL).all()
    return out, guard_ok


WRITE_SET_CONV = [pytest.param(ROWS[n], bf, id="%s-%s" % (n, fmt(bf)))
                  for n in ("g2_cg12_kg80_pad2", "d12_cg36_kg144", "tiny_images_pad2", "s4_k11_cg3") for bf in (True, False)] + \
                 [pytest.param(ROWS["s3_k5_g2_cg2"], False, id="s3_k5_g2_cg2-3xTF32")]


@pytest.mark.gpu
@pytest.mark.parametrize("row,bf", WRITE_SET_CONV)
def test_conv_exact_write_set(row, bf, qcnn, cache, ctx):
    """qcnn_conv_aprx_forward writes every output element and nothing around them (partial channel tiles, G > 1,
    position tails, K-split reduction)."""
    import torch
    it = cache.conv(row)
    L = it["L"]
    ho, wo, co = L.out_dims()
    n_out = row.N * ho * wo * co
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for (NT, GT, ns) in _pins_for_isolation(row, bf, ctx.sm_count):
        pin(L, 2 if bf else 1, 6, NT, GT, ns)
        xd = conv_src(row, it, L)
        for relu in (0, 1):
            out, guard_ok = _guarded_call(
                lambda dst, r: qcnn._check(qcnn.lib.qcnn_conv_aprx_forward(L.h, ctypes.c_void_p(xd.data_ptr()), row.N,
                                                                           dst, r, stream)), n_out, relu)
            assert_plan(L.describe(row.N), 1 if row.stride > 1 else 0, bf, NT, GT, ns)
            assert guard_ok, (NT, GT, ns, relu)
            assert np.isfinite(out).all(), (NT, GT, ns, relu, int((~np.isfinite(out)).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("ri,bf", [(ri, bf) for ri in (1, 3, 5) for bf in (True, False)],
                         ids=["%s-%s" % (FC_ROWS[ri].name, fmt(bf)) for ri in (1, 3, 5) for bf in (True, False)])
def test_fc_exact_write_set(ri, bf, qcnn, ctx):
    import torch
    row = FC_ROWS[ri]
    x, ctrd, asmt, bias = fc_data(row)
    L = _fc_layer(qcnn, ctx, row, ctrd, asmt, bias)
    L.set_param("tensor_core", 2 if bf else 1)
    xd = torch.from_numpy(x).cuda().view(row.N, -1)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for relu in (0, 1):
        out, guard_ok = _guarded_call(
            lambda dst, r: qcnn._check(qcnn.lib.qcnn_fc_aprx_forward(L.h, ctypes.c_void_p(xd.data_ptr()), row.N, dst, r,
                                                                     stream)), row.N * row.Dout, relu)
        assert guard_ok, relu
        assert np.isfinite(out).all(), relu
    assert "pq_gemm_tc(" in L.describe(row.N)
    L.close()
