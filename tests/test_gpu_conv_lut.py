"""The LUT + gather conv kernels (conv_aprx.cu: conv_s1, conv_roll, each with the FFMA or the 3xTF32 wgmma LUT stage, and
conv_direct) against a float64 reference, at every instantiation and at the shapes where their code paths branch.

Reference, metric and bound
  ref64 / f64_err / strict_bound of test_gpu_pq_gemm: err = max |gpu - ref64| / M with M = sum |w x| + |bias|, and
      bound = (max(d + taps S, taps min(Cg, d)) + 3) U                    (FFMA LUT stage, conv_direct)
              + 3 2^-20 + 3 C_MMA U                                       (3xTF32 wgmma LUT stage)
  with U = 2^-24: a LUT entry is an fp32 sum of d products, an output the fp32 sum of taps x S entries and the bias;
  conv_direct sums taps x min(Cg, d) products.  ReLU outputs are compared with max(ref64, 0) under the same M.
  Measured worst err / bound over the 121 cases, with and without ReLU, on one NVIDIA H100 80GB HBM3 (700 W power limit):
  conv_s1 0.073, conv_roll 0.053, conv_s1_tc 0.052, conv_roll_tc 0.111 (err 6.5e-7), conv_direct 0.111 (err 2.6e-7).
  The bound is loose on these short reductions; what it catches is a structural error (a lost subspace, tap or row, a
  wrong codeword, a doubled bias), each of which errs by far more than the bound.

Pins
  Each case pins the family (force_kernel) and the whole tiling (lut_cpt, lut_j, lut_nct, lut_r, lut_rgroups), turns
  autotuning off, and asserts the plan from describe() after the forward.  lut_space() mirrors PlanLutGather's
  candidate enumeration (not its cost model), so the table is checked on the CPU: every pin names exactly one tiling,
  and the pins together reach every kernel instantiation (test_pins_reach_every_instantiation) and every branch the
  table claims (test_table_reaches_every_branch).  On the GPU, test_every_instantiation_ran collects (kernel, LUT
  stage, CPT, J, launch bound) from the plans that ran.

Besides
  neighbour poisoning (an image's output is bit-identical whether the other images are 0 or NaN), the exact write set
  (a NaN guard around the output stays untouched, every output is finite), run-to-run bit identity, and bit identity of
  image i computed alone and inside the batch under the same pinned tiling.  Every case's err, bound and plan go to
  conv_lut_f64.json in the directory named by QCNN_REPORT_DIR (default: qcnn_reports under the system temporary
  directory).
"""
import collections
import ctypes
import json
import os
import tempfile
import zlib

import numpy as np
import pytest

from test_gpu_layers import rand_act
from test_gpu_pq_gemm import _guarded_call, bits, f64_err, ref64, strict_bound

REPORT = {}
SMEM_OPTIN = 227 * 1024     # H100: cudaDevAttrMaxSharedMemoryPerBlockOptin
FAMILY = {0: "conv_s1", 1: "conv_roll", 2: "conv_s1_tc(wgmma LUT)", 3: "conv_roll_tc(wgmma LUT)", 4: "conv_direct"}


def _ceil(a, b):
    return -(-a // b)


def _rup(a, b):
    return _ceil(a, b) * b


# ------------------------------------------------------------------------------------------------------------------
# mirror of PlanLutGather's candidates (conv_aprx.cu)
# ------------------------------------------------------------------------------------------------------------------
Row = collections.namedtuple("Row", "name N Hi Wi Cin Cout k pad stride G S K d")
Plan = collections.namedtuple("Plan", "kernel CPT J nct R rgroups threads smem nstrips ncol CW CT PP pwarps cwarps NJ")


def out_hw(row):
    return ((row.Hi + 2 * row.pad - row.k) // row.stride + 1, (row.Wi + 2 * row.pad - row.k) // row.stride + 1)


def _ffma_smem(K, PP, taps, CT):
    return 4 * K * PP + 4 * taps * CT + 64 * K + 64 * PP + 4 * PP + 32 * K + ((taps * CT + 15) & ~15)


def _wgmma_smem(PP, NM, taps, CT):
    return 4 * 128 * PP + 4 * taps * CT + 3 * 4096 + 96 * NM + 4 * (NM + 8) + ((taps * CT + 15) & ~15)


def lut_space(row, smem_max=SMEM_OPTIN):
    """Every tiling PlanLutGather offers for the row (any batch size: the candidates do not depend on it)."""
    G, k, p, s = row.G, row.k, row.pad, row.stride
    Cg, Kg, taps = row.Cin // G, row.Cout // G, k * k
    Ho, Wo = out_hw(row)
    tc_ok = row.K == 128 and row.d <= 8
    out, found = [], False
    for ncol in range(1, (min(16, Wo) if s == 1 else 1) + 1):
        if ncol > 1 and found:
            break
        for CPT in (32, 16):
            if Kg % CPT:
                continue
            for J in range(1, 5):
                if J * CPT > 64:
                    break
                for nct in range(1, Kg // CPT + 1):
                    CT = Kg // nct
                    if Kg % nct or CT % CPT or CT % 16:
                        continue
                    cwarps = CT // CPT
                    for R in range(1, Ho + 1):
                        for tc in ((0, 1) if tc_ok else (0,)):
                            nstrips, CW = _ceil(Ho, R) * ncol, _ceil(Wo, ncol)
                            if s == 1:
                                kernel, rgroups = (2 if tc else 0), 1
                                PW = CW + k - 1 if ncol > 1 else row.Wi + p
                                pwarps = _ceil(R * PW, 32 * J)
                                need = max((R + k - 1) * PW + max(p, k - 1) + 1, pwarps * 32 * J + (k - 1) * PW + k)
                                warps = pwarps * cwarps
                            else:
                                kernel, rgroups = (3 if tc else 1), _ceil(k, s)
                                pwarps = _ceil(Wo, 32 * J)
                                ph1 = _ceil(row.Wi + 2 * p, s)
                                ph2 = pwarps * 32 * J + (k - 1) // s + 1
                                need = max(ph1 * s, (s - 1) * ph1 + ph2) if tc else _rup(max(ph1, ph2) * s, 4)
                                warps = pwarps * cwarps * rgroups
                            if tc:
                                NM = _rup(need, 32)
                                if NM > 256 or warps < 4:
                                    continue
                                PP = NM + 4
                                smem = _wgmma_smem(PP, NM, taps, CT)
                            else:
                                PP = _rup(need, 4)
                                smem = _ffma_smem(row.K, PP, taps, CT)
                            threads = warps * 32
                            if threads > 512 or threads < 64 or smem > smem_max:
                                continue
                            out.append(Plan(kernel, CPT, J, nct, R, rgroups, threads, smem, nstrips, ncol, CW, CT, PP,
                                            pwarps, cwarps, 0))
                            found = True
    if row.S == 1 and min(Cg, row.d) <= 4 and Wo <= 64:
        NJ = 3 if min(Cg, row.d) <= 3 else 4
        for CPT in (16, 8):
            if Kg % CPT or Kg % 16:
                continue
            for nct in (1, 2):
                CT = Kg // nct
                if Kg % nct or CT % 16 or CT % CPT:
                    continue
                cwarps = CT // CPT
                for R in (2, 4, 6, 8, 14):
                    if R > Ho + 1:
                        continue
                    for rgroups in (1, 2):
                        for rows in range(2, (4 if CPT == 8 else 2) + 1, 2):
                            if rgroups > R // rows:
                                continue
                            aR = min(R, Ho + (Ho & 1))
                            PW = _ceil(row.Wi + 2 * p, s)
                            PP = _rup(PW * s, 4)
                            threads = 32 * cwarps * rgroups
                            smem = 4 * (((aR - 1) * s + k) * NJ * PP + 64 + 8 * row.K + taps * CT)
                            if threads > 384 or threads < 128 or smem > smem_max:
                                continue
                            out.append(Plan(4, CPT, rows, nct, aR, rgroups, threads, smem, _ceil(Ho, aR), 1, Wo, CT,
                                            PP, 1, cwarps, NJ))
    return out


def pinned(row, pin):
    """The tilings a pin (kernel, CPT, J, nct, R, rgroups) keeps, duplicates (equal plans) merged."""
    return sorted({p for p in lut_space(row) if (p.kernel, p.CPT, p.J, p.nct, p.R, p.rgroups) == pin})


def bound_of(threads):
    return 256 if threads <= 256 else 384 if threads <= 384 else 512


def instantiation(p):
    """The kernel template instance a plan launches (LaunchLutGather's dispatch)."""
    if p.kernel == 4:
        return ("conv_direct", p.CPT, p.NJ, p.J)
    return ("conv_s1" if p.kernel in (0, 2) else "conv_roll", "wgmma" if p.kernel in (2, 3) else "ffma", p.CPT, p.J,
            bound_of(p.threads))


ALL_INSTANTIATIONS = {(k, lut, c, j, b) for k in ("conv_s1", "conv_roll") for lut in ("ffma", "wgmma")
                      for (c, j) in ((32, 1), (32, 2), (16, 1), (16, 2), (16, 3), (16, 4)) for b in (256, 384, 512)} | \
                     {("conv_direct", 16, 3, 2), ("conv_direct", 16, 4, 2), ("conv_direct", 8, 3, 4),
                      ("conv_direct", 8, 4, 4), ("conv_direct", 8, 3, 2), ("conv_direct", 8, 4, 2)}
# An instantiation that no geometry the planner accepts can reach, with the constraint that excludes it (none today).
UNREACHABLE = {}


# ------------------------------------------------------------------------------------------------------------------
# the designed table
# ------------------------------------------------------------------------------------------------------------------
ROWS = {r.name: r for r in [
    # stride 1: groups, a partial last subspace (S d > Cg), several FFMA LUT chunks (d = 12, 16), K = 16 ... 256
    Row("s1_g2_partial_sub", 3, 7, 9, 24, 64, 3, 1, 1, 2, 2, 128, 8),      # Cg = 12 < S d = 16
    Row("s1_k5_valid_d12", 2, 8, 8, 24, 48, 5, 0, 1, 1, 2, 64, 12),         # pad = 0, two LUT chunks per subspace
    Row("s1_pad2_d16_k256", 2, 6, 7, 32, 32, 3, 2, 1, 1, 2, 256, 16),       # pad = k - 1
    Row("s1_k16_kg128", 2, 5, 6, 16, 128, 3, 1, 1, 1, 2, 16, 8),
    Row("s1_kg256_k128", 1, 6, 12, 8, 256, 3, 1, 1, 1, 1, 128, 8),          # up to 16 channel warps
    Row("s1_kg192", 2, 5, 13, 16, 192, 3, 1, 1, 1, 2, 128, 8),
    Row("s1_wide_ncol", 1, 2, 298, 8, 16, 3, 1, 1, 1, 1, 256, 8),           # no whole row fits a LUT: 6 column tiles
    # rolling rows: rgroups = ceil(k / stride) in {2, 3, 4}, strides 2-4, windows ending below the image
    Row("roll_s2_kg192", 1, 9, 11, 4, 192, 3, 1, 2, 1, 1, 128, 4),
    Row("roll_s2_k3", 3, 9, 11, 8, 32, 3, 1, 2, 1, 2, 128, 4),
    Row("roll_s3_k5_g2", 2, 11, 13, 12, 64, 5, 2, 3, 2, 1, 64, 8),          # Cg = 6 < d = 8
    Row("roll_s4_k11", 2, 23, 23, 3, 64, 11, 0, 4, 1, 1, 128, 8),           # conv1-like
    Row("roll_s2_kg256", 1, 7, 9, 4, 256, 3, 1, 2, 1, 1, 128, 4),
    Row("roll_s2_k7_k16", 2, 13, 13, 8, 64, 7, 3, 2, 1, 2, 16, 4),          # VggCnnS-like stem
    # conv_direct: NJ = 4 (Cg = 4) and NJ = 3 (Cg = 2), odd Ho
    Row("direct_cg4_odd", 2, 7, 9, 4, 64, 3, 0, 1, 1, 1, 32, 4),
    Row("direct_cg2_s2", 2, 13, 15, 2, 32, 5, 2, 2, 1, 1, 16, 4),
]}

# (row, (force_kernel, lut_cpt, lut_j, lut_nct, lut_r, lut_rgroups)): every instantiation, plus per row and family a
# partial last strip and R = 1 where the row has them
PINS = [
    ("s1_g2_partial_sub", (0, 16, 1, 1, 1, 1)), ("s1_g2_partial_sub", (0, 32, 1, 1, 4, 1)),
    ("s1_g2_partial_sub", (0, 32, 2, 1, 7, 1)), ("s1_g2_partial_sub", (2, 16, 1, 1, 4, 1)),
    ("s1_g2_partial_sub", (2, 16, 1, 1, 7, 1)), ("s1_g2_partial_sub", (2, 16, 2, 1, 7, 1)),
    ("s1_k5_valid_d12", (0, 16, 1, 1, 1, 1)), ("s1_k5_valid_d12", (0, 16, 1, 1, 3, 1)),
    ("s1_k5_valid_d12", (0, 16, 1, 1, 4, 1)),
    ("s1_pad2_d16_k256", (0, 16, 1, 1, 1, 1)), ("s1_pad2_d16_k256", (0, 16, 2, 2, 8, 1)),
    ("s1_pad2_d16_k256", (0, 32, 1, 1, 5, 1)),
    ("s1_k16_kg128", (0, 16, 1, 1, 5, 1)), ("s1_k16_kg128", (0, 32, 1, 2, 1, 1)), ("s1_k16_kg128", (0, 32, 1, 2, 3, 1)),
    ("s1_kg256_k128", (0, 16, 2, 2, 6, 1)), ("s1_kg256_k128", (0, 16, 3, 1, 6, 1)),
    ("s1_kg256_k128", (0, 16, 3, 8, 6, 1)), ("s1_kg256_k128", (0, 16, 4, 1, 6, 1)),
    ("s1_kg256_k128", (0, 32, 1, 1, 3, 1)), ("s1_kg256_k128", (0, 32, 1, 4, 1, 1)),
    ("s1_kg256_k128", (0, 32, 1, 8, 4, 1)), ("s1_kg256_k128", (0, 32, 2, 1, 6, 1)),
    ("s1_kg256_k128", (2, 16, 1, 2, 3, 1)), ("s1_kg256_k128", (2, 16, 1, 4, 6, 1)),
    ("s1_kg256_k128", (2, 16, 2, 2, 6, 1)), ("s1_kg256_k128", (2, 16, 3, 1, 6, 1)),
    ("s1_kg256_k128", (2, 16, 4, 1, 6, 1)), ("s1_kg256_k128", (2, 16, 4, 4, 6, 1)),
    ("s1_kg256_k128", (2, 32, 1, 1, 3, 1)), ("s1_kg256_k128", (2, 32, 1, 2, 1, 1)),
    ("s1_kg256_k128", (2, 32, 1, 2, 6, 1)), ("s1_kg256_k128", (2, 32, 1, 4, 4, 1)),
    ("s1_kg256_k128", (2, 32, 2, 1, 6, 1)), ("s1_kg256_k128", (2, 32, 2, 4, 6, 1)),
    ("s1_kg192", (0, 16, 1, 4, 5, 1)), ("s1_kg192", (0, 16, 2, 2, 5, 1)), ("s1_kg192", (0, 16, 3, 1, 5, 1)),
    ("s1_kg192", (0, 16, 4, 1, 5, 1)), ("s1_kg192", (0, 16, 4, 6, 5, 1)), ("s1_kg192", (0, 32, 1, 2, 5, 1)),
    ("s1_kg192", (0, 32, 1, 3, 1, 1)), ("s1_kg192", (0, 32, 1, 6, 3, 1)), ("s1_kg192", (0, 32, 2, 1, 5, 1)),
    ("s1_kg192", (2, 16, 1, 3, 1, 1)), ("s1_kg192", (2, 16, 2, 2, 5, 1)), ("s1_kg192", (2, 16, 3, 1, 5, 1)),
    ("s1_kg192", (2, 16, 3, 3, 5, 1)), ("s1_kg192", (2, 16, 4, 1, 5, 1)), ("s1_kg192", (2, 32, 1, 3, 3, 1)),
    ("s1_kg192", (2, 32, 1, 3, 5, 1)), ("s1_kg192", (2, 32, 2, 1, 5, 1)),
    ("s1_wide_ncol", (0, 16, 1, 1, 1, 1)),
    ("roll_s2_kg192", (1, 16, 1, 12, 5, 2)), ("roll_s2_kg192", (1, 16, 3, 2, 5, 2)),
    ("roll_s2_kg192", (1, 16, 4, 2, 5, 2)), ("roll_s2_kg192", (1, 16, 4, 12, 5, 2)),
    ("roll_s2_kg192", (1, 32, 1, 1, 5, 2)), ("roll_s2_kg192", (1, 32, 1, 6, 1, 2)),
    ("roll_s2_kg192", (1, 32, 1, 6, 3, 2)), ("roll_s2_kg192", (1, 32, 2, 1, 5, 2)),
    ("roll_s2_kg192", (3, 16, 2, 6, 5, 2)), ("roll_s2_kg192", (3, 32, 1, 1, 5, 2)),
    ("roll_s2_kg192", (3, 32, 1, 3, 1, 2)), ("roll_s2_kg192", (3, 32, 1, 3, 3, 2)),
    ("roll_s2_kg192", (3, 32, 2, 1, 5, 2)), ("roll_s2_kg192", (4, 16, 2, 2, 6, 1)),
    ("roll_s2_k3", (1, 16, 2, 2, 5, 2)), ("roll_s2_k3", (1, 32, 1, 1, 1, 2)), ("roll_s2_k3", (1, 32, 1, 1, 3, 2)),
    ("roll_s2_k3", (3, 16, 1, 1, 1, 2)), ("roll_s2_k3", (3, 16, 1, 1, 3, 2)), ("roll_s2_k3", (3, 16, 1, 1, 5, 2)),
    ("roll_s2_k3", (3, 16, 3, 1, 5, 2)),
    ("roll_s3_k5_g2", (1, 32, 1, 1, 1, 2)), ("roll_s3_k5_g2", (1, 32, 1, 1, 3, 2)),
    ("roll_s4_k11", (1, 16, 1, 1, 4, 3)), ("roll_s4_k11", (1, 16, 2, 1, 4, 3)), ("roll_s4_k11", (1, 32, 1, 2, 1, 3)),
    ("roll_s4_k11", (1, 32, 1, 2, 3, 3)), ("roll_s4_k11", (3, 16, 1, 1, 4, 3)), ("roll_s4_k11", (3, 16, 2, 1, 4, 3)),
    ("roll_s4_k11", (3, 16, 3, 1, 4, 3)), ("roll_s4_k11", (3, 16, 4, 1, 4, 3)), ("roll_s4_k11", (3, 32, 1, 1, 1, 3)),
    ("roll_s4_k11", (3, 32, 1, 1, 3, 3)), ("roll_s4_k11", (3, 32, 2, 1, 4, 3)), ("roll_s4_k11", (4, 16, 2, 1, 4, 1)),
    ("roll_s2_kg256", (1, 32, 1, 1, 4, 2)), ("roll_s2_kg256", (1, 32, 1, 8, 1, 2)),
    ("roll_s2_kg256", (1, 32, 1, 8, 3, 2)), ("roll_s2_kg256", (1, 32, 2, 1, 4, 2)),
    ("roll_s2_kg256", (1, 32, 2, 8, 1, 2)), ("roll_s2_kg256", (3, 16, 1, 2, 4, 2)),
    ("roll_s2_kg256", (3, 16, 2, 2, 4, 2)), ("roll_s2_kg256", (3, 16, 3, 2, 4, 2)),
    ("roll_s2_kg256", (3, 16, 4, 2, 4, 2)), ("roll_s2_kg256", (3, 16, 4, 8, 4, 2)),
    ("roll_s2_kg256", (3, 32, 1, 1, 4, 2)), ("roll_s2_kg256", (3, 32, 1, 4, 1, 2)),
    ("roll_s2_kg256", (3, 32, 1, 4, 3, 2)), ("roll_s2_kg256", (3, 32, 1, 4, 4, 2)),
    ("roll_s2_kg256", (3, 32, 2, 1, 4, 2)),
    ("roll_s2_k7_k16", (1, 16, 1, 1, 7, 4)), ("roll_s2_k7_k16", (1, 16, 2, 1, 7, 4)),
    ("roll_s2_k7_k16", (1, 16, 3, 1, 7, 4)), ("roll_s2_k7_k16", (1, 16, 3, 4, 7, 4)),
    ("roll_s2_k7_k16", (1, 16, 4, 1, 7, 4)), ("roll_s2_k7_k16", (1, 32, 1, 2, 1, 4)),
    ("roll_s2_k7_k16", (1, 32, 1, 2, 4, 4)),
    ("direct_cg4_odd", (0, 32, 1, 1, 1, 1)), ("direct_cg4_odd", (0, 32, 1, 1, 3, 1)),
    ("direct_cg4_odd", (4, 8, 2, 2, 6, 1)), ("direct_cg4_odd", (4, 8, 4, 2, 6, 1)),
    ("direct_cg4_odd", (4, 16, 2, 1, 6, 1)), ("direct_cg4_odd", (4, 16, 2, 2, 6, 2)),
    ("direct_cg2_s2", (1, 32, 1, 1, 1, 3)), ("direct_cg2_s2", (1, 32, 1, 1, 4, 3)),
    ("direct_cg2_s2", (4, 8, 2, 2, 8, 2)), ("direct_cg2_s2", (4, 8, 4, 2, 8, 2)),
    ("direct_cg2_s2", (4, 16, 2, 1, 8, 2)),
]


def pin_id(name, pin):
    return "%s-%s-CPT%d-J%d-nct%d-R%d-rg%d" % ((name, FAMILY[pin[0]].split("(")[0]) + tuple(pin[1:]))


CASES = [pytest.param(ROWS[n], pin, id=pin_id(n, pin)) for n, pin in PINS]


def plan_text(row, p, N):
    """describe() of a LUT + gather plan (DescribeLutGather's format)."""
    return ("%s CPT=%d J=%d threads=%d smem=%dB grid=(%d,%d) R=%d strips=%d ncol=%d CW=%d CT=%d nct=%d PP=%d pwarps=%d "
            "cwarps=%d rgroups=%d" % (FAMILY[p.kernel], p.CPT, p.J, p.threads, p.smem, row.G * p.nct * p.nstrips, N, p.R,
                                      p.nstrips, p.ncol, p.CW, p.CT, p.nct, p.PP, p.pwarps, p.cwarps, p.rgroups))


def the_plan(row, pin):
    (p,) = pinned(row, pin)
    return p


# ------------------------------------------------------------------------------------------------------------------
# CPU: the table
# ------------------------------------------------------------------------------------------------------------------
def test_pins_name_one_tiling():
    for n, pin in PINS:
        assert len(pinned(ROWS[n], pin)) == 1, (n, pin, pinned(ROWS[n], pin))
    assert len(set(PINS)) == len(PINS)


def test_pins_reach_every_instantiation():
    reached = {instantiation(the_plan(ROWS[n], pin)) for n, pin in PINS}
    assert len(ALL_INSTANTIATIONS) == 78
    assert reached == ALL_INSTANTIATIONS - set(UNREACHABLE), sorted(ALL_INSTANTIATIONS - set(UNREACHABLE) - reached)


def test_table_reaches_every_branch():
    plans = [(ROWS[n], the_plan(ROWS[n], pin)) for n, pin in PINS]
    Ho = lambda r: out_hw(r)[0]
    Cg = lambda r: r.Cin // r.G
    for fam in (0, 1, 2, 3):
        fp = [(r, p) for r, p in plans if p.kernel == fam]
        assert any(p.R == 1 for r, p in fp) and any(Ho(r) % p.R for r, p in fp), fam   # R = 1, a partial last strip
        assert any(p.nct > 1 for r, p in fp), fam
    rows = {r.name: r for r, _ in plans}.values()
    assert any(r.G > 1 and r.stride == 1 for r in rows) and any(r.G > 1 and r.stride > 1 for r in rows)
    assert {r.pad == 0 for r in rows} == {True, False} and any(r.pad == r.k - 1 and r.stride == 1 for r in rows)
    assert any(r.S * r.d > Cg(r) for r in rows)
    assert {12, 16} <= {r.d for r in rows}
    assert {16, 64, 128, 256} <= {r.K for r in rows}
    roll = [(r, p) for r, p in plans if p.kernel in (1, 3)]
    assert {2, 3, 4} <= {r.stride for r, p in roll if p.rgroups > 1}
    # the trailing loop of conv_roll: the last output row's window ends below the image
    assert any((Ho(r) - 1) * r.stride - r.pad + r.k > r.Hi for r, p in roll)
    assert any(p.ncol > 1 and out_hw(r)[1] % p.CW for r, p in plans)                # column tiles, partial last one
    direct = [(r, p) for r, p in plans if p.kernel == 4]
    assert {p.NJ for r, p in direct} == {3, 4} and {p.CPT for r, p in direct} == {8, 16}
    assert {p.J for r, p in direct} == {2, 4} and {p.rgroups for r, p in direct} == {1, 2}
    assert any(p.nct == 2 for r, p in direct)
    assert any(Ho(r) % 2 and p.R > Ho(r) for r, p in direct)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def save_report():
    out = os.environ.get("QCNN_REPORT_DIR") or os.path.join(tempfile.gettempdir(), "qcnn_reports")
    try:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "conv_lut_f64.json"), "w") as f:
            json.dump(REPORT, f, indent=1, sort_keys=True)
    except OSError:
        pass


def conv_data(row):
    rng = np.random.RandomState(zlib.crc32(row.name.encode()) & 0x7FFFFFFF)
    fan = (row.Cin // row.G) * row.k * row.k
    ctrd = (rng.randn(row.S, row.K, row.d) / np.sqrt(fan)).astype(np.float32)
    asmt = rng.randint(0, row.K, size=(row.Cout, row.k, row.k, row.S)).astype(np.uint8)
    bias = (rng.randn(row.Cout) * 0.1).astype(np.float32)
    x = rand_act(rng, (row.N, row.Hi, row.Wi, row.Cin), scale=4.0)
    return x, ctrd, asmt, bias


class _Cache(object):
    """One layer, input and float64 reference per row, shared by the cases of the module."""

    def __init__(self, qcnn, ctx):
        self.qcnn, self.ctx, self.items = qcnn, ctx, {}

    def get(self, row):
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


LUT_PINS = ("lut_cpt", "lut_j", "lut_nct", "lut_r", "lut_rgroups")


def pin_lut(L, pin):
    L.set_param("tensor_core", 0)
    L.set_param("autotune", 0)
    L.set_param("force_kernel", pin[0])
    for name, v in zip(LUT_PINS, pin[1:]):
        L.set_param(name, v)


RAN = set()     # instantiations whose plan ran and was checked


def run_case(row, pin, it):
    """Forward (twice, and with ReLU) under the pin; returns (y, yr, plan text) after checking the plan that ran."""
    L = it["L"]
    pin_lut(L, pin)
    if row.stride > 1:
        L.set_src_nchw(False)
    y = L.forward(it["xd"]).cpu().numpy()
    desc = L.describe(row.N)          # after the forward: the plan that just ran
    p = the_plan(row, pin)
    assert desc == plan_text(row, p, row.N), (desc, plan_text(row, p, row.N))
    y2 = L.forward(it["xd"]).cpu().numpy()
    yr = L.forward(it["xd"], relu=True).cpu().numpy()
    assert np.array_equal(bits(y), bits(y2)), desc            # same plan, same sums: bit-identical run to run
    if row.stride > 1:                # the NCHW source: the same sums in the same order
        L.set_src_nchw(True)
        yn = L.forward(it["xn"]).cpu().numpy()
        L.set_src_nchw(False)
        assert np.array_equal(bits(yn), bits(y)), desc
    RAN.add(instantiation(p))
    return y, yr, desc


@pytest.mark.gpu
@pytest.mark.parametrize("row,pin", CASES)
def test_conv_lut_pinned_f64(row, pin, cache):
    it = cache.get(row)
    y, yr, desc = run_case(row, pin, it)
    bound = strict_bound(pin[0], row.k * row.k, row.S, row.d, row.Cin // row.G)
    e = f64_err(y, it["ref"], it["mag"])
    er = f64_err(yr, np.maximum(it["ref"], 0), it["mag"])
    REPORT[pin_id(row.name, pin)] = {"plan": desc, "err": e, "err_relu": er, "bound": bound,
                                     "instantiation": list(instantiation(the_plan(row, pin)))}
    save_report()
    assert e <= bound, (e, bound, desc)
    assert er <= bound, (er, bound, desc)


@pytest.mark.gpu
def test_every_instantiation_ran(cache):
    """Every kernel instantiation of conv_aprx.cu ran under a pin and matched its plan (cases not run yet in this
    session, e.g. under -k, run here)."""
    for n, pin in PINS:
        if instantiation(the_plan(ROWS[n], pin)) not in RAN:
            run_case(ROWS[n], pin, cache.get(ROWS[n]))
    assert RAN == ALL_INSTANTIATIONS - set(UNREACHABLE), sorted(ALL_INSTANTIATIONS - set(UNREACHABLE) - RAN)


@pytest.mark.gpu
def test_unmatched_lut_pin_fails(qcnn, cache):
    row = ROWS["s1_g2_partial_sub"]
    L = cache.get(row)["L"]
    for name, value in (("lut_cpt", 8), ("lut_j", 5), ("lut_nct", 3), ("lut_r", 99), ("lut_rgroups", 2)):
        pin_lut(L, (0, 0, 0, 0, 0, 0))
        L.set_param(name, value)
        with pytest.raises(qcnn.QcnnError, match="%s=%d" % (name, value)):
            L.describe(row.N)
    pin_lut(L, (0, 0, 0, 0, 0, 0))
    with pytest.raises(qcnn.QcnnError, match="applies to conv layers"):
        fc = qcnn.FcLayer(cache.ctx, 64, np.zeros((16, 16, 4), np.float32), np.zeros((8, 16), np.uint8),
                          np.zeros(8, np.float32))
        try:
            fc.set_param("lut_cpt", 16)
        finally:
            fc.close()


# a representative pin per family (several images, a partial last strip where the family has one)
ISOLATION = [("s1_g2_partial_sub", (0, 32, 1, 1, 4, 1)), ("s1_g2_partial_sub", (2, 16, 1, 1, 4, 1)),
             ("roll_s2_k3", (1, 32, 1, 1, 3, 2)), ("roll_s2_k3", (3, 16, 1, 1, 3, 2)),
             ("direct_cg4_odd", (4, 16, 2, 2, 6, 2)), ("direct_cg2_s2", (4, 8, 4, 2, 8, 2))]
ISO_CASES = [pytest.param(ROWS[n], pin, id=pin_id(n, pin)) for n, pin in ISOLATION]


@pytest.mark.gpu
@pytest.mark.parametrize("row,pin", ISO_CASES)
def test_conv_lut_neighbour_poison_and_alone(row, pin, cache):
    """Image i's output is bit-identical whether every other image is 0 or NaN, and to image i computed alone (the
    pinned tiling does not depend on N; per-image work does not either)."""
    import torch
    it = cache.get(row)
    L = it["L"]
    pin_lut(L, pin)
    if row.stride > 1:
        L.set_src_nchw(False)
    full = L.forward(it["xd"]).cpu().numpy()
    for i in range(row.N):
        outs = []
        for fill in (0.0, np.nan):
            xp = np.full_like(it["x"], fill)
            xp[i] = it["x"][i]
            outs.append(L.forward(torch.from_numpy(xp).cuda()).cpu().numpy()[i])
        assert L.describe(row.N) == plan_text(row, the_plan(row, pin), row.N)
        assert np.array_equal(bits(outs[0]), bits(outs[1])), i
        assert np.array_equal(bits(outs[0]), bits(full[i])), i
        alone = L.forward(it["xd"][i:i + 1].contiguous()).cpu().numpy()
        assert L.describe(1) == plan_text(row, the_plan(row, pin), 1)
        assert np.array_equal(bits(alone[0]), bits(full[i])), i


@pytest.mark.gpu
@pytest.mark.parametrize("row,pin", ISO_CASES)
def test_conv_lut_exact_write_set(row, pin, qcnn, cache):
    """qcnn_conv_aprx_forward writes every output element and nothing around them."""
    import torch
    it = cache.get(row)
    L = it["L"]
    pin_lut(L, pin)
    if row.stride > 1:
        L.set_src_nchw(False)
    ho, wo, co = L.out_dims()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    xd = it["xd"]
    for relu in (0, 1):
        out, guard_ok = _guarded_call(
            lambda dst, r: qcnn._check(qcnn.lib.qcnn_conv_aprx_forward(L.h, ctypes.c_void_p(xd.data_ptr()), row.N, dst,
                                                                       r, stream)), row.N * ho * wo * co, relu)
        assert L.describe(row.N) == plan_text(row, the_plan(row, pin), row.N)
        assert guard_ok, relu
        assert np.isfinite(out).all(), (relu, int((~np.isfinite(out)).sum()))
