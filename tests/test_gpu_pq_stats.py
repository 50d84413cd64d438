"""Calibration statistics (qcnn_pq_stats_*): the sums an error-correcting refinement reads, accumulated batch by batch.
read() after one or many adds against fp64 references within the summation bound, the fold rule (a CPU mirror), the
sweeps on accumulated statistics against the restatements fed the read-back sums, refine leaving the statistics as they
were, and every rejection."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

import test_gpu_pq_refine as fcr
import test_gpu_pq_refine_conv as cvr
import test_gpu_pq_refine_target as tgr
from test_gpu_pq_quantize import ulps

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import pq_refine_golden as golden   # noqa: E402

GOLDEN_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pq_refine_conv_bits.npz")
GOLDEN_ROWS = golden.ROWS

EPS = 2.0 ** -53
RUN_BYTES = 1 << 28   # an add folds its positions in runs of 2^28 / (4 Dg) (DESIGN.md 4e)

STATS_SYMBOLS = ["qcnn_pq_stats_create_fc", "qcnn_pq_stats_create_conv", "qcnn_pq_stats_add", "qcnn_pq_stats_count",
                 "qcnn_pq_stats_read_h", "qcnn_pq_stats_refine", "qcnn_pq_stats_refine_target", "qcnn_pq_stats_destroy"]


# ---- the fold rule, mirrored on the CPU ------------------------------------------------------------------------------
def runs(P_b, Dg):
    """the runs [p0, p1) of one add of P_b positions"""
    F = max(1, min(P_b, RUN_BYTES // (4 * Dg)))
    return [(p0, min(P_b, p0 + F)) for p0 in range(0, P_b, F)]


def batchings(N):
    """the batchings of N images each test adds: all at once, uneven (1, 2 and the rest), one image per add"""
    uneven = [b for b in (1, 2, N - 3) if b > 0][:3] if N > 3 else [1] * N
    return {"one": [N], "uneven": uneven, "single": [1] * N}


def conv_geometry(Cin, H, k, pad, stride, grp):
    Ho = cvr.out_size(H, k, pad, stride)
    return Ho * Ho, Cin // grp * k * k


def test_stats_symbols_declared_and_exported(qcnn):
    text = open(qcnn.HEADER_PATH).read()
    lib = C.CDLL(qcnn.LIB_PATH)
    for name in STATS_SYMBOLS:
        assert re.search(r"QCNN_API\s+\w+\s+%s\s*\(" % name, text), name
        assert hasattr(lib, name), name
        assert name in qcnn.EXPORTS, name


def test_rows_cover_the_fold_rule():
    """The conv rows reach padding, stride 4, groups, Cin = 3, partial 64-dim tiles, position counts that are not
    multiples of 16 and more than one fold in one add; in the uneven batching of a multi-fold row, a batch boundary
    falls inside a run that the single add sums as one fold."""
    seen = set()
    for name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed in cvr.ONE_SWEEP:
        hw, Dg = conv_geometry(Cin, H, k, pad, stride, grp)
        one = runs(N * hw, Dg)
        seen |= {"pad"} if pad else set()
        seen |= {"stride4"} if stride == 4 else set()
        seen |= {"groups"} if grp > 1 else set()
        seen |= {"cin3"} if Cin == 3 else set()
        seen |= {"partial_tile"} if Dg % 64 else set()
        seen |= {"not16"} if any((p1 - p0) % 16 for p0, p1 in one) else set()
        if len(one) > 1:
            seen.add("multi_fold")
            base, inside = 0, False
            for b in batchings(N)["uneven"][:-1]:
                base += b * hw
                inside |= any(p0 < base < p1 for p0, p1 in one)
            assert inside, name
            seen.add("boundary_inside_run")
    assert seen == {"pad", "stride4", "groups", "cin3", "partial_tile", "not16", "multi_fold", "boundary_inside_run"}, seen


# ---- helpers -----------------------------------------------------------------------------------------------------
def cuda(a):
    return cvr.cuda(a)


def add_batches(st, y, t, batches):
    i, n0 = 0, st.count
    for b in batches:
        st.add(y[i:i + b], None if t is None else t[i:i + b])
        i += b
    assert st.count == n0 + i


def conv_refs(x, t, Cin, H, k, pad, stride, grp, d):
    """fp64 references of G, |patches| Gram (the bound's sum of |products|), P, |t| P and |T|^2, by torch F.unfold"""
    Cg = Cin // grp
    batch = max(1, (64 << 20) // (8 * Cg * k * k * cvr.out_size(H, k, pad, stride) ** 2))
    G = np.stack(cvr.grams_torch(x, Cg, k, pad, stride, grp, d, batch))
    Ga = np.stack(cvr.grams_torch(x.abs(), Cg, k, pad, stride, grp, d, batch))
    if t is None:
        return G, Ga, None, None, None
    P = tgr.conv_cross_torch(x, t, Cg, k, pad, stride, grp, d, batch)
    Pa = tgr.conv_cross_torch(x.abs(), t.abs(), Cg, k, pad, stride, grp, d, batch)
    return G, Ga, P, Pa, tgr.tsq(t)


def within(got, want, absum, n):
    """|got - want| <= 2 n 2^-53 sum|products| (the device's and the reference's summation error, products exact)"""
    err = np.abs(got - want)
    bound = 2.0 * n * EPS * absum
    assert (err <= bound).all(), (err.max(), float(np.max(err - bound)))


def check_conv(st, ref, n_pos):
    G, Ga, P, Pa, tt = ref
    g, p, t2 = st.read()
    for gg in g:
        assert np.array_equal(gg, gg.T)
    within(g, G, Ga, n_pos)
    if P is not None:
        within(p, P, Pa, n_pos)
        assert abs(t2 - tt) <= 2.0 * n_pos * EPS * tt
    return g, p, t2


def fc_data(Din, Dout, K, d, seed):
    W, ctrd, asmt = fcr.start(Din, Dout, K, d, seed)
    X = fcr.gaussian_inputs(2 * Din + 7, Din, seed + 1)
    T = tgr.fc_targets(X, W, seed + 2)
    return W, ctrd, asmt, X, T


def check_fc(st, X, T):
    X64, T64 = X.astype(np.float64), T.astype(np.float64)
    n = X.shape[0]
    g, p, t2 = st.read()
    assert np.array_equal(g, g.T)
    within(g, X64.T @ X64, np.abs(X64).T @ np.abs(X64), n)
    if T is not None and st.target:
        within(p, T64.T @ X64, np.abs(T64).T @ np.abs(X64), n)
        tt = float((T64 * T64).sum())
        assert abs(t2 - tt) <= 2.0 * T.size * EPS * tt
    return g, p, t2


class Fed(object):
    """Stands for the data matrix in the FC restatements, which form G = Y^T Y and P = T^T Y: both products return
    the matrix it was given, so the restatements run on read-back sums."""

    def __init__(self, M, cols):
        self.M, self.shape = M, (0, cols)

    def astype(self, _):
        return self

    @property
    def T(self):
        return self

    def __matmul__(self, other):
        return self.M


# ---- one add, many adds ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,Cin,H,Cout,k,pad,stride,grp,K,d,N,seed", cvr.ONE_SWEEP, ids=[c[0] for c in cvr.ONE_SWEEP])
def test_conv_adds_match_fp64(name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed, qcnn, ctx):
    W, ctrd, asmt = cvr.start(Cout, Cin // grp, k, K, d, seed)
    x = cuda(cvr.maps(N, H, H, Cin, seed + 1))
    t = tgr.conv_targets(x, W, pad, stride, grp, seed + 2)
    ref = conv_refs(x, t, Cin, H, k, pad, stride, grp, d)
    hw, _ = conv_geometry(Cin, H, k, pad, stride, grp)
    bits = {}
    for how, batches in sorted(batchings(N).items()):
        for rep in range(2 if how == "uneven" else 1):
            st = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, stride=stride, grp=grp, target=True)
            add_batches(st, x, t, batches)
            g, p, t2 = check_conv(st, ref, N * hw)
            key = (how, rep)
            bits[key] = g.tobytes() + p.tobytes() + np.float64(t2).tobytes()
            st.close()
    assert bits[("uneven", 0)] == bits[("uneven", 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,Din,Dout,K,d,seed", fcr.ONE_SWEEP, ids=[c[0] for c in fcr.ONE_SWEEP])
def test_fc_adds_match_fp64(name, Din, Dout, K, d, seed, qcnn, ctx):
    W, ctrd, asmt, X, T = fc_data(Din, Dout, K, d, seed)
    x, t = cuda(X), cuda(T)
    bits = {}
    for how, batches in sorted(batchings(X.shape[0]).items()):
        for rep in range(2 if how == "uneven" else 1):
            st = qcnn.PqStats.fc(ctx, Din, Dout, d, target=True)
            add_batches(st, x, t, batches)
            g, p, t2 = check_fc(st, X, T)
            bits[(how, rep)] = g.tobytes() + p.tobytes() + np.float64(t2).tobytes()
            st.close()
    assert bits[("uneven", 0)] == bits[("uneven", 1)]


# ---- refine from accumulated statistics --------------------------------------------------------------------------
def conv_loss(W, G, ctrd, asmt, grp, d):
    """sum_g sum_{o in g} E_o^T G_g E_o from the read-back Grams"""
    Cout, Cg, k, _ = W.shape
    perm = cvr.dim_order(Cg, d, k * k)
    E = (W.astype(np.float64) - cvr.decode(dict(ctrd=ctrd, asmt=asmt), Cg)).reshape(Cout, -1)[:, perm]
    Cpg = Cout // grp
    return sum(float(((E[g * Cpg:(g + 1) * Cpg] @ G[g]) * E[g * Cpg:(g + 1) * Cpg]).sum()) for g in range(grp))


def conv_target_loss(G, P, tt, ctrd, asmt, Cout, Cg, k, grp, d):
    """(|T|^2 - 2 sum w^ P + sum w^ G w^, its scale) from the read-back sums"""
    perm = cvr.dim_order(Cg, d, k * k)
    Wh = cvr.decode(dict(ctrd=ctrd, asmt=asmt), Cg).reshape(Cout, -1)[:, perm].astype(np.float64)
    Cpg = Cout // grp
    quad = sum(float(((Wh[g * Cpg:(g + 1) * Cpg] @ G[g]) * Wh[g * Cpg:(g + 1) * Cpg]).sum()) for g in range(grp))
    return tt - 2 * float((Wh * P).sum()) + quad, tt + abs(quad)


REFINE_CONV = [r for r in cvr.ONE_SWEEP if r[0] in ("3x3_grp2_partial", "5x5_s2_p2", "conv1_like", "chunked_grp2")]


@pytest.mark.gpu
@pytest.mark.parametrize("name,Cin,H,Cout,k,pad,stride,grp,K,d,N,seed", REFINE_CONV, ids=[c[0] for c in REFINE_CONV])
def test_conv_refine_from_accumulated_statistics(name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed, qcnn, ctx):
    Cg = Cin // grp
    W, ctrd, asmt = cvr.start(Cout, Cg, k, K, d, seed)
    x = cuda(cvr.maps(N, H, H, Cin, seed + 1))
    t = tgr.conv_targets(x, W, pad, stride, grp, seed + 2)
    st = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, stride=stride, grp=grp, target=True)
    add_batches(st, x, t, batchings(N)["uneven"])
    G, P, tt = st.read()
    # same input
    c, a, loss = st.refine(W, ctrd, asmt, sweeps=1)
    want_c, want_a, stats = cvr.sweep_ref(W, list(G), ctrd, asmt, grp, 1, follow=(c, a))
    assert ulps(c, want_c).max() <= 1.0 and np.array_equal(a, want_a)
    for got, (cc, aa) in zip(loss, [(ctrd, asmt), (c, a)]):
        want = conv_loss(W, G, cc, aa, grp, d)
        assert abs(got - want) <= 1e-12 * want, (got, want)
    # target
    c2, a2, loss2 = st.refine_target(ctrd, asmt, sweeps=1)
    want_c, want_a, stats = tgr.conv_target_sweep_ref(list(G), P, ctrd, asmt, grp, k, 1, follow=(c2, a2))
    assert ulps(c2, want_c).max() <= 1.0 and np.array_equal(a2, want_a)
    for got, (cc, aa) in zip(loss2, [(ctrd, asmt), (c2, a2)]):
        want, scale = conv_target_loss(G, P, tt, cc, aa, Cout, Cg, k, grp, d)
        assert abs(got - want) <= 1e-12 * scale, (got, want, scale)
    st.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,Din,Dout,K,d,seed", fcr.ONE_SWEEP, ids=[c[0] for c in fcr.ONE_SWEEP])
def test_fc_refine_from_accumulated_statistics(name, Din, Dout, K, d, seed, qcnn, ctx):
    W, ctrd, asmt, X, T = fc_data(Din, Dout, K, d, seed)
    st = qcnn.PqStats.fc(ctx, Din, Dout, d, target=True)
    add_batches(st, cuda(X), cuda(T), batchings(X.shape[0])["uneven"])
    G, P, tt = st.read()
    c, a, loss = st.refine(W, ctrd, asmt, sweeps=1)
    want_c, want_a, _ = fcr.refine_ref(W, Fed(G, Din), ctrd, asmt, 1, follow=(c, a))
    assert ulps(c, want_c).max() <= 1.0 and np.array_equal(a, want_a)
    for got, (cc, aa) in zip(loss, [(ctrd, asmt), (c, a)]):
        E = W.astype(np.float64) - fcr.decoded(cc, aa, Din)
        want = float(((E @ G) * E).sum())
        assert abs(got - want) <= 1e-12 * want, (got, want)
    c2, a2, loss2 = st.refine_target(ctrd, asmt, sweeps=1)
    want_c, want_a, _ = tgr.fc_target_ref(Fed(G, Din), Fed(P, Din), ctrd, asmt, 1, follow=(c2, a2))
    assert ulps(c2, want_c).max() <= 1.0 and np.array_equal(a2, want_a)
    for got, (cc, aa) in zip(loss2, [(ctrd, asmt), (c2, a2)]):
        Wh = fcr.decoded(cc, aa, Din)
        quad = float(((Wh @ G) * Wh).sum())
        want = tt - 2 * float((Wh * P).sum()) + quad
        assert abs(got - want) <= 1e-12 * (tt + quad), (got, want)
    st.close()


# ---- one add is the one-shot call; refine leaves the statistics unchanged ----------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("row", GOLDEN_ROWS, ids=[r[0] for r in GOLDEN_ROWS])
def test_results_keep_the_stored_bits(row, qcnn, ctx):
    """The one-shot calls and refine after one add of all N images reproduce, bit for bit, the results stored in
    tests/golden/pq_refine_conv_bits.npz by the im2col implementation the map-operand Gram replaced (written on an
    NVIDIA H100 by tools/pq_refine_golden.py from the same seeded inputs)."""
    name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed = row
    W, X, T, ctrd, asmt = golden.inputs(Cin, H, Cout, k, pad, stride, grp, K, d, N, seed)
    ref = np.load(GOLDEN_PATH)
    x, t = cuda(X), cuda(T)
    same = qcnn.pq_refine_conv(ctx, W, x, ctrd, asmt, pad=pad, stride=stride, grp=grp, sweeps=golden.SWEEPS)
    tgt = qcnn.pq_refine_conv_target(ctx, x, t, ctrd, asmt, k, pad=pad, stride=stride, grp=grp, sweeps=golden.SWEEPS)
    st = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, stride=stride, grp=grp, target=True)
    st.add(x, t)
    same_st = st.refine(W, ctrd, asmt, sweeps=golden.SWEEPS)
    tgt_st = st.refine_target(ctrd, asmt, sweeps=golden.SWEEPS)
    st.close()
    for got in (same, same_st):
        for part, arr in zip(("ctrd", "asmt", "loss"), got):
            assert arr.tobytes() == ref[name + "/" + part].tobytes(), (name, part)
    for got in (tgt, tgt_st):
        for part, arr in zip(("ctrd", "asmt", "loss"), got):
            assert arr.tobytes() == ref[name + "/target_" + part].tobytes(), (name, "target", part)


@pytest.mark.gpu
def test_refine_leaves_the_statistics_unchanged(qcnn, ctx):
    Cin, H, Cout, k, pad, stride, grp, K, d, N = 12, 11, 24, 5, 2, 2, 1, 32, 4, 4
    W, ctrd, asmt = cvr.start(Cout, Cin, k, K, d, 51)
    x = cuda(cvr.maps(N, H, H, Cin, 52))
    t = tgr.conv_targets(x, W, pad, stride, grp, 53)
    st = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, stride=stride, target=True)
    same = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, stride=stride)
    for b in ([1, 3], [2, 2]):
        add_batches(st, x[:sum(b)], t[:sum(b)], b)
        add_batches(same, x[:sum(b)], None, b)
    before = [a.tobytes() if isinstance(a, np.ndarray) else np.float64(a).tobytes() for a in st.read()]
    r1 = st.refine(W, ctrd, asmt, sweeps=2)
    r2 = st.refine(W, ctrd, asmt, sweeps=2)
    r3 = same.refine(W, ctrd, asmt, sweeps=2)
    t1 = st.refine_target(ctrd, asmt, sweeps=2)
    t2 = st.refine_target(ctrd, asmt, sweeps=2)
    after = [a.tobytes() if isinstance(a, np.ndarray) else np.float64(a).tobytes() for a in st.read()]
    assert before == after
    assert st.count == 8
    for u, v in ((r1, r2), (r1, r3), (t1, t2)):
        assert all(a.tobytes() == b.tobytes() for a, b in zip(u, v))
    assert same.read()[0].tobytes() == st.read()[0].tobytes()
    st.close()
    same.close()


# ---- rejections ---------------------------------------------------------------------------------------------------
def _raises(qcnn, fn, text):
    with pytest.raises(qcnn.QcnnError) as e:
        fn()
    assert text in str(e.value), (text, str(e.value))


@pytest.mark.gpu
def test_rejected_calls(qcnn, ctx):
    import torch
    Cin, H, Cout, k, pad, K, d, N = 16, 8, 24, 3, 1, 16, 4, 3
    W, ctrd, asmt = cvr.start(Cout, Cin, k, K, d, 61)
    x = cuda(cvr.maps(N, H, H, Cin, 62))
    t = tgr.conv_targets(x, W, pad, 1, 1, 63)
    st = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, target=True)
    same = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad)
    # before any add
    _raises(qcnn, lambda: st.refine_target(ctrd, asmt, sweeps=1), "no calibration data")
    _raises(qcnn, lambda: same.refine(W, ctrd, asmt, sweeps=1), "no calibration data")
    assert st.count == 0 and not st.read()[0].any()
    st.add(x[:2], t[:2])
    same.add(x[:2])
    snap = [a.tobytes() if isinstance(a, np.ndarray) else np.float64(a).tobytes() for a in st.read()]
    # non-finite y or t: nothing changes
    for bad_y, bad_t, text in ((float("nan"), None, "y contains a non-finite value"),
                               (None, float("inf"), "t contains a non-finite value")):
        yb, tb = x[2:].clone(), t[2:].clone()
        if bad_y is not None:
            yb[0, 3, 4, 5] = bad_y
        if bad_t is not None:
            tb[0, 1, 2, 3] = bad_t
        _raises(qcnn, lambda: st.add(yb, tb), text)
    xb = x[2:].clone()
    xb[0, 0, 0, 0] = float("-inf")
    _raises(qcnn, lambda: same.add(xb), "x contains a non-finite value")
    assert [a.tobytes() if isinstance(a, np.ndarray) else np.float64(a).tobytes() for a in st.read()] == snap
    assert st.count == 2 and same.count == 2
    # t on a same-input object, none on a target object, N < 1
    _raises(qcnn, lambda: same.add(x[2:], t[2:]), "created without a target")
    _raises(qcnn, lambda: st.add(x[2:]), "NULL t")
    _raises(qcnn, lambda: st.add(x[:0], t[:0]), "at least one input")
    # refine_target on a same-input object, K, the joint system, assignments, codebook, weights
    _raises(qcnn, lambda: same.refine_target(ctrd, asmt, sweeps=1), "created without a target")
    c12 = np.zeros((ctrd.shape[0], 12, d), np.float32)
    _raises(qcnn, lambda: st.refine(W, c12, np.zeros_like(asmt), sweeps=1), "K=12")
    big = qcnn.PqStats.conv(ctx, 40, 6, 6, 16, 3, 16, pad=1)
    big.add(cuda(cvr.maps(1, 6, 6, 40, 64)))
    Wb, cb, ab = cvr.start(16, 40, 3, 256, 16, 65)
    _raises(qcnn, lambda: big.refine(Wb, cb, ab, sweeps=1), "joint codebook system")
    big.close()
    a_bad = asmt.copy()
    a_bad[0, 0, 0, 0] = K
    _raises(qcnn, lambda: st.refine(W, ctrd, a_bad, sweeps=1), "not below K")
    c_bad = ctrd.copy()
    c_bad[0, 0, 0] = np.nan
    _raises(qcnn, lambda: st.refine_target(c_bad, asmt, sweeps=1), "codebook contains a non-finite value")
    w_bad = W.copy()
    w_bad[0, 0, 0, 0] = np.inf
    _raises(qcnn, lambda: st.refine(w_bad, ctrd, asmt, sweeps=1), "weights contain a non-finite value")
    _raises(qcnn, lambda: st.refine(W, ctrd, asmt, sweeps=-1), "negative")
    # shapes in Python
    _raises(qcnn, lambda: st.add(x[:, :4], t), "y must be")
    _raises(qcnn, lambda: st.add(x, t[:, 1:]), "t must be")
    _raises(qcnn, lambda: st.add(x.double(), t), "float32")
    _raises(qcnn, lambda: st.refine(W[:, :3], ctrd, asmt), "wei must be")
    _raises(qcnn, lambda: st.refine(W, ctrd[:, :, :2], asmt), "must be [S, K, d]")
    _raises(qcnn, lambda: st.add(x.permute(0, 2, 1, 3), t), "contiguous")
    # NULL arguments through the C ABI
    lib = qcnn.lib
    out = C.c_void_p()
    assert lib.qcnn_pq_stats_create_fc(None, 4, 4, 2, 0, C.byref(out)) != 0 and "NULL" in qcnn.last_error()
    assert lib.qcnn_pq_stats_create_fc(ctx.h, 4, 4, 2, 0, None) != 0 and "NULL" in qcnn.last_error()
    assert lib.qcnn_pq_stats_create_conv(ctx.h, 4, 4, 4, 4, 3, 1, 1, 1, 65, 0, C.byref(out)) != 0
    assert "d=65" in qcnn.last_error()
    assert lib.qcnn_pq_stats_add(None, C.c_void_p(x.data_ptr()), None, 1, None) != 0 and "NULL" in qcnn.last_error()
    assert lib.qcnn_pq_stats_add(same.h, None, None, 1, None) != 0 and "NULL" in qcnn.last_error()
    assert lib.qcnn_pq_stats_count(None, None) != 0 and "NULL" in qcnn.last_error()
    assert lib.qcnn_pq_stats_read_h(None, None, None, None) != 0 and "NULL" in qcnn.last_error()
    assert lib.qcnn_pq_stats_read_h(same.h, None, None, C.byref(C.c_double())) != 0
    assert lib.qcnn_pq_stats_refine(same.h, K, 1, None, ctrd.ctypes.data_as(C.c_void_p), asmt.ctypes.data_as(C.c_void_p),
                                    None, None) != 0 and "NULL" in qcnn.last_error()
    assert lib.qcnn_pq_stats_refine_target(None, K, 1, None, None, None, None) != 0 and "NULL" in qcnn.last_error()
    lib.qcnn_pq_stats_destroy(None)
    assert st.count == 2
    torch.cuda.synchronize()
    st.close()
    same.close()
    # FC: a rejected add names the input column, and a target FC object needs t
    sf = qcnn.PqStats.fc(ctx, 12, 5, 4, target=True)
    Y = np.ones((3, 12), np.float32)
    Y[1, 7] = np.nan
    _raises(qcnn, lambda: sf.add(cuda(Y), cuda(np.ones((3, 5)))), "input column 7")
    _raises(qcnn, lambda: sf.add(cuda(np.ones((3, 12))), cuda(np.ones((3, 4)))), "t must be")
    assert sf.count == 0
    sf.close()
