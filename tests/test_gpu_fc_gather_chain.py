"""The FC layers' LUT + gather kernel (fc_aprx.cu, batches 5-95, every batch under tensor_core = 0, and every fc_tn /
fc_nsplit pin) and the persistent batch <= 4 chain kernel (fc_chain.cu) against float64 references, at every
instantiation and at the shapes where their code paths branch.

Reference, metric and bounds
  ref64 / fc_sum / f64_err / strict_bound of test_gpu_pq_gemm: err = max |gpu - ref64| / M with M = sum |w x| + |bias|.
  Every output is a tree of S LUT entries (each an fp32 sum of d products) plus the bias, and adding the exact zero
  partial sums of idle CTAs or splits changes nothing, so one layer is within
      beta = strict_bound(0, 1, S, d, Din) = (d + S + 3) U        (+ nsplit U for the gather kernel's K-split)
  in any association: the gather kernel's s-ascending order, its K-split reduced by fc_reduce_kernel, and the chain's
  per-CTA rows, row groups and cross-CTA shuffle tree.  A chain of layers propagates the error elementwise,
      E_1 = beta_1 M_1,   E_l = beta_l M_l + fc_sum(E_{l-1}, |ctrd_l|, asmt_l),
  with M_l evaluated on |x_ref| + E_{l-1} (ReLU does not widen a difference), and every output must satisfy
  |gpu - ref64| <= E_L.  Gather with nsplit = 1 adds in the reference's order: it is compared bit for bit with the oracle.
  Measured worst err / bound on one NVIDIA H100 80GB HBM3 (700 W power limit), with and without ReLU: LUT + gather
  0.044 (err 5.8e-8, k64_n tn = 4 packed; 36 pinned cases and the K = 256 rows), chain 0.0098 (one layer,
  rg9_k128_partial; every branch row at N = 1..4 and the re-arm sequence).  Multi-layer chains sit far lower (<= 4.4e-5),
  because the propagated term sums |w| E where the real errors cancel.  The bounds are loose on these short
  reductions; what they catch is a structural error (a lost row or split, a doubled partial, a dropped bias), each of
  which errs by far more.

Mirrors (CPU)
  gather_plan mirrors PlanFcGather and the staging size of Launch; chain_plan mirrors PlanChain, including the float32
  NHWC fold check.  test_gather_table_reaches_every_branch and test_chain_table_reaches_every_branch show that the rows
  reach every instantiation and branch they claim, with G = 132 (rows that depend on G are derived from it, so on the
  GPU they are built from ctx.sm_count).  The first layer's offset-table branch of the chain is recorded as unreachable.

GPU checks
  Gather: each case pins tensor_core = 0, fc_tn, fc_nsplit and the table format, asserts the plan from describe(), the
  bound with and without ReLU, neighbour NaN isolation inside a tile, the exact write set (a NaN guard around the
  output), run-to-run bit identity, and that image i alone equals image i inside the batch.  Chain: every row at
  N = 1..4 against the propagated bound, its exact write set, image i alone vs inside a batch of 4, and describe()'s
  grid / ring / smem against the mirror for chains of one layer.  The re-arm test runs [A, B, C], [B, C], [C], [A] and
  [A, B, C] on fresh inputs, on the default and on a side stream: a partial-sum word a consumer failed to re-arm would
  hand a later call a stale value.  Only ordinary NaN is used as poison.  Every case's err, bound and plan go to
  fc_gather_chain_f64.json in the directory named by QCNN_REPORT_DIR (default: qcnn_reports under the system temporary
  directory).
"""
import collections
import ctypes
import json
import math
import os
import tempfile
import zlib

import numpy as np
import pytest

from test_gpu_fc_chain import make_fc
from test_gpu_pq_gemm import _guarded_call, bits, f64_err, fc_sum, nhwc_flatten, ref64, strict_bound

REPORT = {}
U = 2.0 ** -24
G_CPU = 132                  # H100 SXM: SMs, the chain's grid
SMEM_OPTIN = 227 * 1024      # H100: cudaDevAttrMaxSharedMemoryPerBlockOptin
GATHER_SMEM_MAX = 200 * 1024
CHUNK_BYTES = 16384
PACKED_TAIL = 16


def _ceil(a, b):
    return -(-a // b)


def _rup(a, b):
    return _ceil(a, b) * b


def save_report():
    out = os.environ.get("QCNN_REPORT_DIR") or os.path.join(tempfile.gettempdir(), "qcnn_reports")
    try:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "fc_gather_chain_f64.json"), "w") as f:
            json.dump(REPORT, f, indent=1, sort_keys=True)
    except OSError:
        pass


def packed_bits(K, packed):
    return int(math.log2(K)) if packed and K < 256 else 0


# ------------------------------------------------------------------------------------------------------------------
# mirror of PlanFcGather / Launch (fc_aprx.cu)
# ------------------------------------------------------------------------------------------------------------------
Row = collections.namedtuple("Row", "name Din Dout S K d")
GPlan = collections.namedtuple("GPlan", "tn cpt pf nsplit sPerSplit grid smem fits")


def chunk_len(K, tn):
    return (16 if K <= 64 else 8) if tn == 1 else (32 if K <= 32 else (16 if K <= 64 else 8))


def gather_smem(K, tn, d):
    pf = chunk_len(K, tn)
    return 4 * (tn * pf * K + 2 * _rup(tn * pf * d, 4) + 2 * pf * K * d)


def gather_plan(row, N, tn_pin=0, nsplit_pin=0, G=G_CPU):
    DoutPad = _rup(row.Dout, 16)
    tn = tn_pin or (8 if N >= 8 else (4 if N >= 4 else 1))
    if tn not in (1, 4):
        tn = 8
    if not tn_pin:
        while tn > 1 and gather_smem(row.K, tn, row.d) > GATHER_SMEM_MAX:
            tn = 4 if tn == 8 else 1
    cpt = 16 if tn == 1 else (4 if tn == 8 and DoutPad <= 1024 else 8)
    pf = chunk_len(row.K, tn)
    chunks = _ceil(row.S, pf)
    ns = nsplit_pin
    if ns <= 0:
        ns = _ceil(3 * G, _ceil(DoutPad, 256 * cpt) * _ceil(N, tn))
    ns = max(1, min(ns, chunks))
    cps = _ceil(chunks, ns)
    smem = gather_smem(row.K, tn, row.d)
    return GPlan(tn, cpt, pf, _ceil(chunks, cps), cps * pf, (_ceil(DoutPad, 256 * cpt), _ceil(N, tn), _ceil(chunks, cps)),
                 smem, smem <= GATHER_SMEM_MAX)


def gather_text(p):
    return "gather(tn=%d cpt=%d pf=%d nsplit=%d)" % (p.tn, p.cpt, p.pf, p.nsplit)


def gather_key(row, packed, p):
    """The kernel instantiation: (K, table, TN, CPT); table = PRE (byte offsets, K <= 64), byte, or b<bits> (packed)."""
    b = packed_bits(row.K, packed)
    return (row.K, "b%d" % b if b else ("PRE" if row.K <= 64 else "byte"), p.tn, p.cpt)


# narrow rows (DoutPad <= 1024) take tn = 1, 4 and 8 with 4 channels per thread; wide rows tn = 8 with 8
GROWS = {r.name: r for r in [
    Row("k16_n", 1000, 200, 250, 16, 4),     # d == 4, Dout % 16 != 0
    Row("k16_w", 301, 1100, 101, 16, 3),     # partial last subspace, grid-x tail
    Row("k32_n", 130, 90, 130, 32, 1),       # d = 1, S % pf != 0
    Row("k32_w", 1024, 1030, 256, 32, 4),
    Row("k64_n", 90, 77, 9, 64, 10),         # S < pf
    Row("k64_w", 600, 2100, 150, 64, 4),     # two CTAs in x, the second one partly idle
    Row("k128_n", 700, 250, 88, 128, 8),     # partial last subspace
    Row("k128_w", 256, 1500, 128, 128, 2),
    Row("k256_n", 80, 40, 10, 256, 8),       # S % pf != 0
    Row("k256_w", 512, 1040, 128, 256, 4),
]}
NMAX = 11
NS_CYCLE = (1, 0, 3, 999)      # reference order, automatic, an uneven split, a pin above the chunk count (clamped)


def _gather_cases():
    out = []
    i = 0
    for K in (16, 32, 64, 128, 256):
        for packed in ((0, 1) if K < 256 else (0,)):
            for name, tn in (("k%d_n" % K, 1), ("k%d_n" % K, 4), ("k%d_n" % K, 8), ("k%d_w" % K, 8)):
                N = {1: 3, 4: 6, 8: NMAX}[tn]
                out.append((GROWS[name], N, tn, NS_CYCLE[i % len(NS_CYCLE)], packed))
                i += 1
    return out


GATHER_CASES = _gather_cases()


def _gid(c):
    row, N, tn, ns, packed = c
    return "%s-N%d-tn%d-ns%d%s" % (row.name, N, tn, ns, "-packed" if packed else "")


def test_gather_table_reaches_every_branch():
    keys, reached = set(), collections.Counter()
    for (row, N, tn, ns, packed) in GATHER_CASES:
        p = gather_plan(row, N, tn, ns)
        assert p.fits and p.tn == tn, (row, p)
        keys.add(gather_key(row, packed, p))
        DoutPad = _rup(row.Dout, 16)
        chunks = _ceil(row.S, p.pf)
        reached["d == 4" if row.d == 4 else "generic d"] += 1
        reached["partial last subspace"] += row.S * row.d > row.Din
        reached["S % pf != 0"] += row.S % p.pf != 0
        reached["S < pf"] += row.S < p.pf
        reached["nsplit = 1"] += p.nsplit == 1
        reached["nsplit > 1"] += p.nsplit > 1
        reached["uneven last split"] += p.nsplit > 1 and row.S - (p.nsplit - 1) * p.sPerSplit < p.sPerSplit
        reached["pin above the chunk count"] += ns > chunks
        reached["N % tn != 0"] += N % p.tn != 0
        reached["grid-x tail"] += DoutPad % (256 * p.cpt) != 0
        reached["Dout % 16 != 0"] += row.Dout % 16 != 0
    # 5 byte-table variants (PRE at K <= 64) and 4 packed widths, each at the 4 (tn, cpt) tilings
    want = {(K, t, tn, cpt) for K in (16, 32, 64, 128, 256)
            for t in (("PRE" if K <= 64 else "byte"),) + (("b%d" % int(math.log2(K)),) if K < 256 else ())
            for (tn, cpt) in ((1, 16), (4, 8), (8, 4), (8, 8))}
    assert len(want) == 36 and keys == want, sorted(want ^ keys)
    missing = [b for b in ("d == 4", "generic d", "partial last subspace", "S % pf != 0", "S < pf", "nsplit = 1",
                           "nsplit > 1", "uneven last split", "pin above the chunk count", "N % tn != 0", "grid-x tail",
                           "Dout % 16 != 0") if not reached[b]]
    assert not missing, missing
    # ReLU: in the kernel's epilogue (nsplit = 1) and in fc_reduce_kernel (nsplit > 1); every case runs both


def test_gather_staging_limits():
    """Largest d per K that the gather kernel stages (include/qcnn.h), and the tile it picks at K = 256."""
    def dmax(K, tn):
        return max(d for d in range(1, 200) if gather_smem(K, tn, d) <= GATHER_SMEM_MAX)
    assert [dmax(K, 1) for K in (16, 32, 64, 128, 256)] == [93, 48, 24, 24, 11]
    assert [dmax(256, tn) for tn in (8, 4, 1)] == [8, 10, 11]
    for d, tn in ((8, 8), (9, 4), (10, 4), (11, 1)):
        p = gather_plan(Row("k256", 40 * d, 64, 40, 256, d), 8)
        assert p.fits and p.tn == tn, (d, p)
    assert not gather_plan(Row("k256", 120, 64, 10, 256, 12), 8).fits
    assert not gather_plan(Row("k256", 100, 64, 10, 256, 10), 8, tn_pin=8).fits     # a pin is not moved


# ------------------------------------------------------------------------------------------------------------------
# mirror of PlanChain (fc_chain.cu)
# ------------------------------------------------------------------------------------------------------------------
Layer = collections.namedtuple("Layer", "Din Dout S K d packed")
CPlan = collections.namedtuple("CPlan", "eligible why layers nStage smem cpcLast gp chunks recycled_within recycled_across "
                                        "collect_calls out_groups fold")


def _f32_floor_div_exact(divisor, count):
    """floor((t + 0.5) * (1 / divisor)) in float32 equals t // divisor for every t < count (the kernel's division)."""
    inv = np.float32(1.0) / np.float32(divisor)
    t = np.arange(count, dtype=np.int64)
    q = np.floor((t.astype(np.float32) + np.float32(0.5)) * inv).astype(np.int64)
    return bool((q == t // divisor).all())


def row_range(unit, ub, ur, S, c):
    u0 = c * ub + min(c, ur)
    nu = ub + (1 if c < ur else 0)
    return min(S, u0 * unit), min(S, (u0 + nu) * unit)


def chain_plan(layers, G=G_CPU, smem_optin=SMEM_OPTIN, nhwc=None):
    """Per-layer figures of PlanChain, and what the kernel will do with them (ring use, CollectSlice batches)."""
    def no(why):
        return CPlan(False, why, [], 0, 0, 0, 0, [], False, False, [], [], False)
    n = len(layers)
    if not 1 <= n <= 4 or not 1 <= G <= 160:
        return no("length / G")
    xF, lutF, ctrdF, rgF = 64, 64, 0, 0
    per, fold = [], False
    for l, Q in enumerate(layers):
        if l > 0 and Q.Din != layers[l - 1].Dout:
            return no("Din != previous Dout")
        DoutPad = _rup(Q.Dout, 16)
        if DoutPad > CHUNK_BYTES or Q.K * Q.d % 4:
            return no("DoutPad / K d")
        pre = Q.K <= 64
        lutPitch = 256 if pre else 4 * Q.K
        cpt = 4 if DoutPad // 4 <= 512 else (8 if DoutPad // 8 <= 512 else 16)
        if DoutPad // cpt > 512:
            return no("too wide")
        tpr = DoutPad // cpt
        rg = min(512 // tpr, 16)
        if not _f32_floor_div_exact(tpr, 512):
            return no("tprInv")
        if l == 0 and nhwc:
            fold = _f32_floor_div_exact(nhwc[0] * nhwc[1], Q.Din)
        rpc = rpc_byte = max(1, CHUNK_BYTES // DoutPad)
        b = packed_bits(Q.K, Q.packed)
        pitch = DoutPad
        if b:
            pitch = _rup(DoutPad * b // 8, 16)
            if rpc % rg == 0:
                rpc = (CHUNK_BYTES - PACKED_TAIL) // pitch // rg * rg
            if rpc < 1 or rpc * pitch + PACKED_TAIL > CHUNK_BYTES:
                return no("packed chunk")
        unit = 4 // math.gcd(Q.d, 4)
        units = _ceil(Q.S, unit)
        ub, ur = divmod(units, G)
        rowsMax = min(Q.S, (ub + (1 if ur else 0)) * unit)
        ctrdF += rowsMax * Q.K * Q.d
        xF = max(xF, _rup(rowsMax * Q.d, 64))
        lutF = max(lutF, _rup(rowsMax * (lutPitch // 4), 64))
        if rg > 1:
            rgF = max(rgF, rg * DoutPad)
        per.append(dict(DoutPad=DoutPad, pre=pre, cpt=cpt, tpr=tpr, rg=rg, rpc=rpc, rpc_byte=rpc_byte, bits=b, pitch=pitch,
                        rpc_kept=bool(b) and rpc == rpc_byte, unit=unit, ub=ub, ur=ur, rowsMax=rowsMax,
                        idle_ctas=G - min(G, units)))
    cpcLast = _rup(_ceil(layers[-1].Dout, G), 4)
    gmax = min(16, cpcLast // 4)
    for l in range(1, n):
        gmax = max(gmax, min(16, _ceil(per[l]["rowsMax"] * layers[l].d, 4)))
    gp = 1
    while gp < gmax:
        gp *= 2
    scr = G * (4 * gp + 4)
    ringOff = _rup(1024 + 4 * (xF + lutF + ctrdF + rgF + scr), 128)
    if ringOff + 2 * CHUNK_BYTES > smem_optin:
        return no("shared memory")
    nStage = min(32, (smem_optin - ringOff) // CHUNK_BYTES)
    # the ring as CTA c's producer fills it: chunk j goes to stage j % nStage, after chunk j - nStage was consumed
    chunks, within, across = [], False, False
    for c in range(G):
        j = 0
        for l, Q in enumerate(layers):
            P = per[l]
            r0, r1 = row_range(P["unit"], P["ub"], P["ur"], Q.S, c)
            k = _ceil(r1 - r0, P["rpc"])
            if c == 0:
                chunks.append(k)
            within = within or k > nStage                      # a stage's previous chunk was this layer's
            across = across or (k > 0 and 0 < j and j + k > nStage)   # ... or an earlier layer's
            j += k
    # CollectSlice calls: groups of 4 features per call, by the consumers of layers 1.. and of the last layer's output
    calls, out_groups = [], []
    for c in range(G):
        for l in range(1, n):
            Q, P = layers[l], per[l]
            r0, r1 = row_range(P["unit"], P["ub"], P["ur"], Q.S, c)
            f0, nf = r0 * Q.d, (r1 - r0) * Q.d
            groups = (min(nf, max(0, Q.Din - f0)) + 3) >> 2
            calls += [min(16, groups - b) for b in range(0, groups, 16)]
            if groups > 16:
                calls.append(groups)        # (recorded as the > 16 marker: more than one batch)
        o0 = c * cpcLast
        og = (max(0, min(cpcLast, layers[-1].Dout - o0)) + 3) >> 2
        out_groups.append(og)
        calls += [min(16, og - b) for b in range(0, og, 16)]
    return CPlan(True, "", per, nStage, ringOff + nStage * CHUNK_BYTES, cpcLast, gp, chunks, within, across, calls,
                 out_groups, fold)


def L_(Din, Dout, S, K, d, packed=0):
    return Layer(Din, Dout, S, K, d, packed)


def chain_rows(G):
    """(name, layers, relu, nhwc): rows that depend on G are derived from it."""
    S12 = 5 * G + G // 6                 # d = 12: 6 rows = 72 features = 18 groups per CTA of the later layer
    S3 = 4 * S12 + 2                     # d = 3: 6 units of 4 rows = 72 features (G = 132: Din = 8190)
    return [
        ("alexnet_fc678", [L_(9216, 4096, 2304, 32, 4), L_(4096, 4096, 1024, 32, 4), L_(4096, 1000, 4096, 16, 1)],
         [1, 1, 0], None),
        ("rg16_one_layer", [L_(256, 100, 64, 32, 4)], [0], None),
        ("rg9_k128_partial", [L_(300, 200, 38, 128, 8)], [1], None),
        ("cpt8_d2", [L_(640, 2500, 320, 64, 2)], [0], None),
        ("cpt16_packed5", [L_(2048, 6000, 512, 32, 4, 1)], [1], None),
        ("packed_each_cpt", [L_(512, 2000, 128, 16, 4, 1), L_(2000, 3000, 500, 64, 4, 1), L_(3000, 5000, 750, 128, 4, 1),
                             L_(5000, 42, 1250, 16, 4, 1)], [1, 1, 1, 0], None),
        ("packed_cpt4_kept", [L_(256, 200, 64, 32, 4, 1), L_(200, 2048, 50, 64, 4, 1), L_(2048, 4096, 512, 128, 4, 1),
                              L_(4096, 8000, 1024, 16, 4, 1)], [1, 0, 1, 0], None),
        ("packed_b6_b7_cpt16", [L_(128, 5000, 32, 64, 4, 1), L_(5000, 8100, 1250, 128, 4, 1), L_(8100, 3000, 2025, 32, 4, 1)],
         [1, 0, 1], None),
        ("packed_b7_cpt4_b4_cpt8", [L_(128, 300, 32, 128, 4, 1), L_(300, 4000, 75, 16, 4, 1)], [0, 1], None),
        ("unit4_idle_ctas", [L_(512, 200, 128, 32, 4), L_(200, 96, 50, 64, 4), L_(96, 40, 96, 16, 1)], [1, 0, 1], None),
        ("groups_gt16_d12", [L_(512, 12 * S12, 128, 16, 4), L_(12 * S12, 100, S12, 32, 12)], [1, 0], None),
        ("groups_gt16_d3", [L_(256, 3 * S3, 64, 16, 4), L_(3 * S3, 100, S3, 32, 3)], [0, 1], None),
        ("ring_recycled", [L_(28416, 4096, 54 * G, 32, 4), L_(4096, 520, 1024, 32, 4)], [1, 0], None),
        ("nhwc_fold", [L_(6 * 6 * 64, 520, 6 * 6 * 16, 32, 4), L_(520, 42, 130, 16, 4)], [1, 0], (6, 6, 64)),
    ]


def test_chain_table_reaches_every_branch():
    G = G_CPU
    reached = collections.Counter()
    for name, layers, relu, nhwc in chain_rows(G):
        p = chain_plan(layers, G, nhwc=nhwc)
        assert p.eligible, (name, p.why)
        reached["chain length %d" % len(layers)] += 1
        for l, (Q, P) in enumerate(zip(layers, p.layers)):
            reached["cpt %d" % P["cpt"]] += 1
            reached["rg = 1" if P["rg"] == 1 else ("rg = 16" if P["rg"] == 16 else "1 < rg < 16")] += 1
            reached["PRE" if P["pre"] and not P["bits"] else ("packed" if P["bits"] else "not PRE")] += 1
            if P["bits"]:
                reached["packed b=%d cpt %d" % (P["bits"], P["cpt"])] += 1
                reached["packed rpc kept" if P["rpc_kept"] else "packed rpc recomputed"] += 1
            reached["unit > 1"] += P["unit"] > 1
            reached["CTAs that own no rows"] += P["idle_ctas"] > 0
            reached["partial last subspace"] += Q.S * Q.d > Q.Din
        reached["ring recycled within a layer"] += p.recycled_within
        reached["ring recycled across a layer boundary"] += p.recycled_across
        for g in p.collect_calls:
            reached["CollectSlice %s" % ("1 group" if g == 1 else ("16 groups" if g == 16 else
                                                                   ("> 16 groups" if g > 16 else "2-15 groups")))] += 1
        reached["last Dout % 4 != 0"] += layers[-1].Dout % 4 != 0
        reached["CTAs with no output channels"] += min(p.out_groups) == 0
        reached["NHWC fold"] += p.fold
    want = (["chain length %d" % n for n in (1, 2, 3, 4)] + ["cpt 4", "cpt 8", "cpt 16", "rg = 1", "1 < rg < 16", "rg = 16",
            "PRE", "not PRE", "packed rpc kept", "packed rpc recomputed", "unit > 1", "CTAs that own no rows",
            "partial last subspace", "ring recycled within a layer", "ring recycled across a layer boundary",
            "CollectSlice 1 group", "CollectSlice 2-15 groups", "CollectSlice 16 groups", "CollectSlice > 16 groups",
            "last Dout % 4 != 0", "CTAs with no output channels", "NHWC fold"] +
            ["packed b=%d cpt %d" % (b, c) for b in (4, 5, 6, 7) for c in (4, 8, 16)])
    missing = [w for w in want if not reached[w]]
    assert not missing, missing


def test_chain_offset_table_branch_unreachable():
    """The first layer's offset-table branch (L.srcoff) runs only when the float32 fold check fails; it passes for every
    NHWC map of fewer than 400 positions and fewer than 30000 features, so no realistic layer reaches it."""
    for hw in range(1, 400):
        assert _f32_floor_div_exact(hw, 30000), hw


def test_chain_groups_gt16_on_smaller_parts():
    """The > 16-group rows stay > 16 groups at the SM counts of other Hopper parts."""
    for G in (114, 132):
        rows = {r[0]: r for r in chain_rows(G)}
        for name in ("groups_gt16_d12", "groups_gt16_d3"):
            p = chain_plan(rows[name][1], G)
            assert p.eligible and max(p.collect_calls) > 16, (G, name)


# ------------------------------------------------------------------------------------------------------------------
# GPU: LUT + gather
# ------------------------------------------------------------------------------------------------------------------
def _seed(name):
    return zlib.crc32(name.encode()) & 0x7FFFFFFF


def _data(rng, Din, Dout, S, K, d, N):
    x = (rng.randn(N, Din) * 2.0).astype(np.float32)
    ctrd = (rng.randn(S, K, d) * 0.05).astype(np.float32)
    asmt = rng.randint(0, K, size=(Dout, S)).astype(np.uint8)
    bias = (rng.randn(Dout) * 0.1).astype(np.float32)
    return x, ctrd, asmt, bias


class _GatherCache(object):
    def __init__(self, qcnn, ctx):
        self.qcnn, self.ctx, self.items = qcnn, ctx, {}

    def get(self, row):
        if row.name not in self.items:
            import torch
            x, ctrd, asmt, bias = _data(np.random.RandomState(_seed(row.name)), row.Din, row.Dout, row.S, row.K, row.d, NMAX)
            ref, mag = ref64("fc", x, ctrd, asmt, bias)
            L = self.qcnn.FcLayer(self.ctx, row.Din, ctrd, asmt, bias)
            self.items[row.name] = dict(L=L, x=x, xd=torch.from_numpy(x).cuda(), ref=ref, mag=mag, p=(ctrd, asmt, bias))
        return self.items[row.name]

    def close(self):
        for it in self.items.values():
            it["L"].close()


@pytest.fixture(scope="module")
def gcache(qcnn, ctx):
    c = _GatherCache(qcnn, ctx)
    yield c
    c.close()


def gpin(L, tn, ns, packed):
    L.set_param("asmt_packed", packed)
    L.set_param("tensor_core", 0)
    L.set_param("fc_tn", tn)
    L.set_param("fc_nsplit", ns)


def gather_desc(row, plan, packed):
    b = packed_bits(row.K, packed)
    return "fc_aprx Din=%d Dout=%d S=%d K=%d d=%d %s%s" % (row.Din, row.Dout, row.S, row.K, row.d, gather_text(plan),
                                                           " asmt=%dbit" % b if b else "")


@pytest.mark.gpu
@pytest.mark.parametrize("case", GATHER_CASES, ids=[_gid(c) for c in GATHER_CASES])
def test_gather_pinned_f64(case, gcache, qcnn, ctx, po):
    import torch
    row, N, tn, ns, packed = case
    it = gcache.get(row)
    L = it["L"]
    gpin(L, tn, ns, packed)
    plan = gather_plan(row, N, tn, ns, ctx.sm_count)
    xd, x = it["xd"][:N], it["x"][:N]
    ref, mag = it["ref"][:N], it["mag"][:N]
    y = L.forward(xd).cpu().numpy()
    desc = L.describe(N)
    assert desc == gather_desc(row, plan, packed), (desc, plan)
    bound = strict_bound(0, 1, row.S, row.d, row.Din) + (plan.nsplit * U if plan.nsplit > 1 else 0.0)
    e = f64_err(y, ref, mag)
    yr = L.forward(xd, relu=True).cpu().numpy()
    er = f64_err(yr, np.maximum(ref, 0), mag)
    REPORT["gather/%s" % _gid(case)] = {"plan": desc, "err": e, "err_relu": er, "bound": bound}
    save_report()
    assert e <= bound, (e, bound, desc)
    assert er <= bound, (er, bound, desc)
    assert np.array_equal(bits(L.forward(xd).cpu().numpy()), bits(y))         # run to run
    if plan.nsplit == 1:                                                        # the reference's order: bit-exact
        assert np.array_equal(bits(y), bits(po.fc_aprx(x, *it["p"]))), desc
    # neighbour isolation inside a tile: image i is the same whether the other images are 0 or NaN
    for i in sorted({0, N - 1}):
        outs = []
        for fill in (0.0, np.nan):
            xp = np.full_like(x, fill)
            xp[i] = x[i]
            outs.append(L.forward(torch.from_numpy(xp).cuda()).cpu().numpy()[i])
        assert np.array_equal(bits(outs[0]), bits(outs[1])), (i, desc)
        assert np.array_equal(bits(outs[0]), bits(y[i])), (i, desc)
    # image i alone, under the same pins (the same sums whenever the pinned plan is the same at N = 1)
    if gather_plan(row, 1, tn, ns, ctx.sm_count).nsplit == plan.nsplit:
        i = N - 1
        assert np.array_equal(bits(L.forward(it["xd"][i:i + 1]).cpu().numpy()[0]), bits(y[i])), desc
    # exact write set: a NaN guard around the output stays untouched and every output is written
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for relu in (0, 1):
        out, guard_ok = _guarded_call(
            lambda dst, r: qcnn._check(qcnn.lib.qcnn_fc_aprx_forward(L.h, ctypes.c_void_p(xd.data_ptr()), N, dst, r, stream)),
            N * row.Dout, relu)
        assert guard_ok, (relu, desc)
        assert np.isfinite(out).all(), (relu, desc)
        assert np.array_equal(bits(out.reshape(N, row.Dout)), bits(yr if relu else y)), (relu, desc)


@pytest.mark.gpu
def test_gather_wide_codewords_every_batch(qcnn, ctx):
    """K = 256: d = 10 runs at N = 8 on 4-image tiles and d = 11 on 1-image tiles, within the bound; d = 12 is refused
    at creation, and a pinned tile that cannot be staged fails the forward naming the pin."""
    import torch
    for d, tn in ((10, 4), (11, 1)):
        row = Row("k256_d%d" % d, 20 * d - 3, 70, 20, 256, d)
        x, ctrd, asmt, bias = _data(np.random.RandomState(d), row.Din, row.Dout, row.S, row.K, row.d, 8)
        ref, mag = ref64("fc", x, ctrd, asmt, bias)
        L = qcnn.FcLayer(ctx, row.Din, ctrd, asmt, bias)
        L.set_param("tensor_core", 0)
        for N in (5, 8):
            plan = gather_plan(row, N, 0, 0, ctx.sm_count)
            y = L.forward(torch.from_numpy(x[:N]).cuda()).cpu().numpy()
            desc = L.describe(N)
            assert desc == gather_desc(row, plan, 0) and plan.tn == (tn if N == 8 else min(tn, 4)), desc
            bound = strict_bound(0, 1, row.S, row.d, row.Din) + plan.nsplit * U
            e = f64_err(y, ref[:N], mag[:N])
            REPORT["gather_k256/d=%d/N=%d" % (d, N)] = {"plan": desc, "err": e, "bound": bound}
            save_report()
            assert e <= bound, (e, bound, desc)
        L.set_param("fc_tn", 8)
        with pytest.raises(qcnn.QcnnError, match="fc_tn=8 with K=256 d=%d" % d):
            L.forward(torch.from_numpy(x).cuda())
        L.close()
    with pytest.raises(qcnn.QcnnError, match="K=256 d=12 is not supported"):
        qcnn.FcLayer(ctx, 120, np.zeros((10, 256, 12), np.float32), np.zeros((8, 10), np.uint8), np.zeros(8, np.float32))


# ------------------------------------------------------------------------------------------------------------------
# GPU: chain
# ------------------------------------------------------------------------------------------------------------------
def chain_ref(params, relu, x):
    """(ref, E): the chain in float64 and the elementwise error bound propagated through it (module docstring)."""
    xr = np.asarray(x, np.float64)
    E = np.zeros_like(xr)
    for (ctrd, asmt, bias), r in zip(params, relu):
        S, K, d = ctrd.shape
        beta = strict_bound(0, 1, S, d, xr.shape[1])
        ac = np.abs(ctrd)
        ref = fc_sum(xr, ctrd, asmt) + bias.astype(np.float64)
        M = fc_sum(np.abs(xr) + E, ac, asmt) + np.abs(bias.astype(np.float64))
        E = beta * M + fc_sum(E, ac, asmt)
        xr = np.maximum(ref, 0) if r else ref
    return xr, E


def _bound_ratio(y, ref, E):
    y = np.asarray(y, np.float64)
    assert y.shape == ref.shape
    if not np.isfinite(y).all():
        return float("inf")
    return float((np.abs(y - ref) / np.maximum(E, 1e-300)).max())


class _ChainCache(object):
    def __init__(self, qcnn, ctx):
        self.qcnn, self.ctx, self.items = qcnn, ctx, {}

    def get(self, name):
        if name not in self.items:
            rows = {r[0]: r for r in chain_rows(self.ctx.sm_count)}
            _, shapes, relu, nhwc = rows[name]
            rng = np.random.RandomState(_seed(name))
            layers, params = [], []
            for Q in shapes:
                L, p = make_fc(rng, self.qcnn, self.ctx, Q.Din, Q.Dout, Q.S, Q.K, Q.d)
                if Q.packed:
                    L.set_param("asmt_packed", 1)
                layers.append(L)
                params.append(p)
            if nhwc:
                layers[0].set_src_nhwc(*nhwc)
                x = (rng.randn(4, *nhwc) * 2.0).astype(np.float32)
                xf = nhwc_flatten(x)
                x = x.reshape(4, -1)
            else:
                x = xf = (rng.randn(4, shapes[0].Din) * 2.0).astype(np.float32)
            ref, E = chain_ref(params, relu, xf)
            self.items[name] = dict(layers=layers, shapes=shapes, relu=relu, x=x, ref=ref, E=E)
        return self.items[name]

    def close(self):
        for it in self.items.values():
            for L in it["layers"]:
                L.close()


@pytest.fixture(scope="module")
def ccache(qcnn, ctx):
    c = _ChainCache(qcnn, ctx)
    yield c
    c.close()


CHAIN_NAMES = [r[0] for r in chain_rows(G_CPU)]


def _chain_call(qcnn, layers, relu, xd, N, stream):
    n = len(layers)
    hs = (ctypes.c_void_p * n)(*[L.h for L in layers])
    rl = (ctypes.c_int * n)(*[int(r) for r in relu])
    return lambda dst, _r: qcnn._check(qcnn.lib.qcnn_fc_chain_forward(hs, rl, n, ctypes.c_void_p(xd.data_ptr()), N, dst,
                                                                      None, stream))


@pytest.mark.gpu
@pytest.mark.parametrize("name", CHAIN_NAMES)
def test_chain_rows_f64(name, ccache, qcnn, ctx):
    import torch
    it = ccache.get(name)
    layers, relu = it["layers"], it["relu"]
    xd = torch.from_numpy(it["x"]).cuda()
    worst = 0.0
    outs = {}
    for N in (1, 2, 3, 4):
        y = qcnn.fc_chain_forward(layers, relu, xd[:N]).cpu().numpy()
        r = _bound_ratio(y, it["ref"][:N], it["E"][:N])
        worst = max(worst, r)
        outs[N] = y
        assert r <= 1.0, (N, r)
    REPORT["chain/%s" % name] = {"err_over_bound": worst, "plan": layers[0].describe(1) if len(layers) == 1 else
                                 "fc_chain(%d layers)" % len(layers), "G": ctx.sm_count}
    save_report()
    # image i alone equals image i inside the batch (one launch per image: the same sums)
    for i in range(4):
        assert np.array_equal(bits(outs[1][0] if i == 0 else
                                   qcnn.fc_chain_forward(layers, relu, xd[i:i + 1]).cpu().numpy()[0]), bits(outs[4][i])), i
    # exact write set
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    Dout = it["shapes"][-1].Dout
    out, guard_ok = _guarded_call(_chain_call(qcnn, layers, relu, xd, 3, stream), 3 * Dout, 0)
    assert guard_ok
    assert np.array_equal(bits(out.reshape(3, Dout)), bits(outs[3]))
    # the mirror agrees with describe() for a chain of one layer
    if len(layers) == 1:
        p = chain_plan(it["shapes"], ctx.sm_count, nhwc=None)
        desc = layers[0].describe(1)
        want = "fc_chain(persistent, 1 layer, grid=%d, ring=%dx%dB, smem=%dB)" % (ctx.sm_count, p.nStage, CHUNK_BYTES, p.smem)
        assert " via " + want in desc, (desc, want)


@pytest.mark.gpu
def test_chain_rearm_fresh_inputs(qcnn, ctx):
    """Each layer's partial-sum words are re-armed by whoever consumed them, whatever chain the layer was part of: every
    call of [A, B, C], [B, C], [C], [A], [A, B, C] on a fresh input meets its own float64 bound, on two streams."""
    import torch
    rng = np.random.RandomState(77)
    shapes = [(640, 520, 160, 32, 4), (520, 300, 130, 16, 4), (300, 42, 150, 64, 2)]
    layers, params = [], []
    for s in shapes:
        L, p = make_fc(rng, qcnn, ctx, *s)
        layers.append(L)
        params.append(p)
    relu = [1, 1, 0]
    seq = [(0, 1, 2), (1, 2), (2,), (0,), (0, 1, 2)]
    side = torch.cuda.Stream()
    k = 0
    for use_side in (False, True):
        for idx in seq:
            N = 1 + k % 4
            k += 1
            x = (rng.randn(N, shapes[idx[0]][0]) * 2.0).astype(np.float32)
            ls, ps, rs = [layers[i] for i in idx], [params[i] for i in idx], [relu[i] for i in idx]
            ref, E = chain_ref(ps, rs, x)
            xd = torch.from_numpy(x).cuda()
            torch.cuda.synchronize()
            if use_side:
                with torch.cuda.stream(side):
                    y = qcnn.fc_chain_forward(ls, rs, xd)
                side.synchronize()
            else:
                y = qcnn.fc_chain_forward(ls, rs, xd)
            r = _bound_ratio(y.cpu().numpy(), ref, E)
            REPORT["chain_rearm/%s/%s/N=%d" % ("side" if use_side else "default", "-".join("ABC"[i] for i in idx), N)] = {
                "err_over_bound": r}
            save_report()
            assert r <= 1.0, (idx, use_side, r)
    for L in layers:
        L.close()
