"""The bias refit of error-correcting PQ on calibration statistics (qcnn_pq_stats_read_sums_h, qcnn_pq_stats_refine_bias
and _refine_target_bias, DESIGN.md 4e "Bias refit"): the first moments s = sum y and u = sum t against fp64 references
within the summation bound, adds of y and -y (and t and -t) leaving them exactly zero so that the bias calls are the plain
ones bit for bit, the sweeps on the centered sums Gc = G - s s^T / n, Pc = P - u s^T / n against the restatements fed
them, the refit bias and the bias-optimal loss against the calibration data, degenerate (constant) input channels, and
every rejection."""
import ctypes as C
import re

import numpy as np
import pytest

import test_gpu_pq_refine as fcr
import test_gpu_pq_refine_conv as cvr
import test_gpu_pq_refine_target as tgr
import test_gpu_pq_stats as sts
from test_gpu_pq_quantize import decode, ulps

EPS = 2.0 ** -53
BIAS_SYMBOLS = ["qcnn_pq_stats_read_sums_h", "qcnn_pq_stats_refine_bias", "qcnn_pq_stats_refine_target_bias"]
SHIFT = 1.0   # added to the inputs, so that their means, and with them the centering, are not small

SUM_CONV = [r for r in cvr.ONE_SWEEP if not r[0].startswith("chunked")]
REFINE_CONV = sts.REFINE_CONV
FC_ROWS = fcr.ONE_SWEEP


def test_bias_symbols_declared_and_exported(qcnn):
    text = open(qcnn.HEADER_PATH).read()
    lib = C.CDLL(qcnn.LIB_PATH)
    for name in BIAS_SYMBOLS:
        assert re.search(r"QCNN_API\s+\w+\s+%s\s*\(" % name, text), name
        assert hasattr(lib, name), name
        assert name in qcnn.EXPORTS, name


def test_sum_rows_reach_padding_stride4_groups_and_three_channels():
    seen = set()
    for name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed in SUM_CONV:
        seen |= {"pad"} if pad else set()
        seen |= {"stride4"} if stride == 4 else set()
        seen |= {"groups"} if grp == 2 else set()
        seen |= {"cin3"} if Cin == 3 else set()
    assert seen == {"pad", "stride4", "groups", "cin3"}, seen


# ---- references ---------------------------------------------------------------------------------------------------
def centered(G, P, tt, s, u, n, grp):
    """Gc, Pc and |T_c|^2 by the normative formula, every operation rounded: bit-identical to the device's copies"""
    n = float(n)
    if G.ndim == 2:   # FC
        Gc = G - np.multiply.outer(s, s) / n
        if P is None:
            return Gc, None, None
        Pc = P - np.multiply.outer(u, s) / n
    else:
        Gc = np.stack([G[g] - np.multiply.outer(s[g], s[g]) / n for g in range(grp)])
        if P is None:
            return Gc, None, None
        Cpg = P.shape[0] // grp
        Pc = np.concatenate([P[g * Cpg:(g + 1) * Cpg] - np.multiply.outer(u[g * Cpg:(g + 1) * Cpg], s[g]) / n
                             for g in range(grp)])
    acc = 0.0
    for v in (u * u) / n:
        acc += float(v)
    return Gc, Pc, tt - acc


def conv_sums_torch(x, Cg, k, pad, stride, grp, d):
    """(s [grp][Dg] in the internal dim order, the same of |x|) in fp64 from the zero-padded patches (F.unfold)"""
    import torch
    import torch.nn.functional as F
    Dg = Cg * k * k
    perm = torch.from_numpy(cvr.dim_order(Cg, d, k * k)).to(x.device)
    s = torch.zeros((grp, Dg), dtype=torch.float64, device=x.device)
    sa = torch.zeros_like(s)
    for i in range(x.shape[0]):
        xb = x[i:i + 1].permute(0, 3, 1, 2).double()
        for g in range(grp):
            Pt = F.unfold(xb[:, g * Cg:(g + 1) * Cg], k, padding=pad, stride=stride)   # [1][Dg][positions]
            s[g] += Pt.sum((0, 2))[perm]
            sa[g] += Pt.abs().sum((0, 2))[perm]
    return s.cpu().numpy(), sa.cpu().numpy()


def within(got, want, absum, n):
    err = np.abs(got - want)
    bound = 2.0 * n * EPS * absum
    assert (err <= bound).all(), (err.max(), float(np.max(err - bound)))


def snapshot(st):
    s, u, n = st.read_sums()
    return s.tobytes() + (b"" if u is None else u.tobytes()) + np.int64(n).tobytes()


def conv_setup(Cin, H, Cout, k, pad, stride, grp, K, d, N, seed):
    W, ctrd, asmt = cvr.start(Cout, Cin // grp, k, K, d, seed)
    x = sts.cuda(cvr.maps(N, H, H, Cin, seed + 1) + SHIFT)
    t = tgr.conv_targets(x, W, pad, stride, grp, seed + 2)
    bias = np.random.RandomState(seed + 3).randn(Cout).astype(np.float32)
    return W, ctrd, asmt, x, t, bias


def fc_setup(Din, Dout, K, d, seed):
    W, ctrd, asmt = fcr.start(Din, Dout, K, d, seed)
    X = fcr.gaussian_inputs(2 * Din + 7, Din, seed + 1) + np.float32(SHIFT)
    T = tgr.fc_targets(X, W, seed + 2)
    bias = np.random.RandomState(seed + 3).randn(Dout).astype(np.float32)
    return W, ctrd, asmt, X, T, bias


# ---- 1. the first moments -------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,Cin,H,Cout,k,pad,stride,grp,K,d,N,seed", SUM_CONV, ids=[c[0] for c in SUM_CONV])
def test_conv_sums_match_fp64(name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed, qcnn, ctx):
    W, ctrd, asmt, x, t, bias = conv_setup(Cin, H, Cout, k, pad, stride, grp, K, d, N, seed)
    s_ref, sa_ref = conv_sums_torch(x, Cin // grp, k, pad, stride, grp, d)
    t64 = t.double().reshape(-1, Cout)
    u_ref, ua_ref = t64.sum(0).cpu().numpy(), t64.abs().sum(0).cpu().numpy()
    Ho = cvr.out_size(H, k, pad, stride)
    rows = N * Ho * Ho
    bits = {}
    for how, batches in sorted(sts.batchings(N).items()):
        for rep in range(2 if how == "uneven" else 1):
            st = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, stride=stride, grp=grp, target=True)
            sts.add_batches(st, x, t, batches)
            s, u, n = st.read_sums()
            assert n == rows and s.shape == (grp, Cin // grp * k * k) and u.shape == (Cout,)
            within(s, s_ref, sa_ref, rows)
            within(u, u_ref, ua_ref, rows)
            bits[(how, rep)] = snapshot(st)
            st.close()
    assert bits[("uneven", 0)] == bits[("uneven", 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,Din,Dout,K,d,seed", FC_ROWS, ids=[c[0] for c in FC_ROWS])
def test_fc_sums_match_fp64(name, Din, Dout, K, d, seed, qcnn, ctx):
    W, ctrd, asmt, X, T, bias = fc_setup(Din, Dout, K, d, seed)
    X64, T64 = X.astype(np.float64), T.astype(np.float64)
    x, t = sts.cuda(X), sts.cuda(T)
    bits = {}
    for how, batches in sorted(sts.batchings(X.shape[0]).items()):
        for rep in range(2 if how == "uneven" else 1):
            st = qcnn.PqStats.fc(ctx, Din, Dout, d, target=True)
            sts.add_batches(st, x, t, batches)
            s, u, n = st.read_sums()
            assert n == X.shape[0] and s.shape == (Din,) and u.shape == (Dout,)
            within(s, X64.sum(0), np.abs(X64).sum(0), n)
            within(u, T64.sum(0), np.abs(T64).sum(0), n)
            bits[(how, rep)] = snapshot(st)
            st.close()
    assert bits[("uneven", 0)] == bits[("uneven", 1)]
    same = qcnn.PqStats.fc(ctx, Din, Dout, d)
    same.add(x)
    s, u, n = same.read_sums()
    assert u is None and n == X.shape[0]
    within(s, X64.sum(0), np.abs(X64).sum(0), n)
    same.close()


def _raises(qcnn, fn, text):
    with pytest.raises(qcnn.QcnnError) as e:
        fn()
    assert text in str(e.value), (text, str(e.value))


@pytest.mark.gpu
def test_rejected_adds_leave_the_sums_unchanged(qcnn, ctx):
    Cin, H, Cout, k, pad, stride, grp, K, d, N = 16, 8, 24, 3, 1, 1, 2, 16, 4, 3
    W, ctrd, asmt, x, t, bias = conv_setup(Cin, H, Cout, k, pad, stride, grp, K, d, N, 71)
    st = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, stride=stride, grp=grp, target=True)
    assert snapshot(st) == np.zeros(grp * Cin // grp * k * k + Cout).tobytes() + np.int64(0).tobytes()
    st.add(x[:2], t[:2])
    snap = snapshot(st)
    yb, tb = x[2:].clone(), t[2:].clone()
    yb[0, 3, 4, 5] = float("nan")
    _raises(qcnn, lambda: st.add(yb, t[2:]), "y contains a non-finite value")
    tb[0, 1, 2, 3] = float("nan")
    _raises(qcnn, lambda: st.add(x[2:], tb), "t contains a non-finite value")
    assert snapshot(st) == snap
    st.close()
    Din, Dout = 12, 5
    sf = qcnn.PqStats.fc(ctx, Din, Dout, 4, target=True)
    Y = np.random.RandomState(72).randn(3, Din).astype(np.float32)
    Tt = np.random.RandomState(73).randn(3, Dout).astype(np.float32)
    sf.add(sts.cuda(Y), sts.cuda(Tt))
    snap = snapshot(sf)
    Yb, Tb = Y.copy(), Tt.copy()
    Yb[1, 7], Tb[2, 1] = np.nan, np.nan
    _raises(qcnn, lambda: sf.add(sts.cuda(Yb), sts.cuda(Tt)), "input column 7")
    _raises(qcnn, lambda: sf.add(sts.cuda(Y), sts.cuda(Tb)), "t contains a non-finite value")
    assert snapshot(sf) == snap and sf.count == 3
    sf.close()


# ---- 2. zero means: the bias calls are the plain ones -------------------------------------------------------------
def _same_bits(a, b):
    return all(u.tobytes() == v.tobytes() for u, v in zip(a, b))


@pytest.mark.gpu
@pytest.mark.parametrize("sweeps", [1, 2])
def test_zero_means_give_the_plain_calls(sweeps, qcnn, ctx):
    name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed = REFINE_CONV[0]
    W, ctrd, asmt, x, t, bias = conv_setup(Cin, H, Cout, k, pad, stride, grp, K, d, N, seed)
    sc = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, stride=stride, grp=grp, target=True)
    sc.add(x, t)
    sc.add(-x, -t)
    Wf, cf, af, X, T, bf = fc_setup(250, 200, 32, 4, 81)
    sf = qcnn.PqStats.fc(ctx, 250, 200, 4, target=True)
    sf.add(sts.cuda(X), sts.cuda(T))
    sf.add(sts.cuda(-X), sts.cuda(-T))
    for st, Wl, c0, a0, b0 in ((sc, W, ctrd, asmt, bias), (sf, Wf, cf, af, bf)):
        s, u, n = st.read_sums()
        assert not s.any() and not u.any()
        c, a, b, loss = st.refine_bias(Wl, c0, a0, b0, sweeps=sweeps)
        assert _same_bits((c, a, loss), st.refine(Wl, c0, a0, sweeps=sweeps))
        assert b.tobytes() == b0.tobytes()
        c, a, b, loss = st.refine_target_bias(c0, a0, b0, sweeps=sweeps)
        assert _same_bits((c, a, loss), st.refine_target(c0, a0, sweeps=sweeps))
        assert b.tobytes() == b0.tobytes()
        assert loss[-1] < loss[0]
        st.close()


# ---- 3. the sweeps on the centered sums against the restatements --------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,Cin,H,Cout,k,pad,stride,grp,K,d,N,seed", REFINE_CONV, ids=[c[0] for c in REFINE_CONV])
def test_conv_centered_sweep_matches_restatement(name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed, qcnn, ctx):
    Cg = Cin // grp
    W, ctrd, asmt, x, t, bias = conv_setup(Cin, H, Cout, k, pad, stride, grp, K, d, N, seed)
    st = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, stride=stride, grp=grp, target=True)
    sts.add_batches(st, x, t, sts.batchings(N)["uneven"])
    G, P, tt = st.read()
    s, u, n = st.read_sums()
    Gc, Pc, ttc = centered(G, P, tt, s, u, n, grp)
    c, a, b, loss = st.refine_bias(W, ctrd, asmt, bias, sweeps=1)
    want_c, want_a, _ = cvr.sweep_ref(W, list(Gc), ctrd, asmt, grp, 1, follow=(c, a))
    assert ulps(c, want_c).max() <= 1.0 and np.array_equal(a, want_a)
    for got, (cc, aa) in zip(loss, [(ctrd, asmt), (c, a)]):
        want = sts.conv_loss(W, Gc, cc, aa, grp, d)
        assert abs(got - want) <= 1e-12 * want, (got, want)
    c2, a2, b2, loss2 = st.refine_target_bias(ctrd, asmt, bias, sweeps=1)
    want_c, want_a, _ = tgr.conv_target_sweep_ref(list(Gc), Pc, ctrd, asmt, grp, k, 1, follow=(c2, a2))
    assert ulps(c2, want_c).max() <= 1.0 and np.array_equal(a2, want_a)
    for got, (cc, aa) in zip(loss2, [(ctrd, asmt), (c2, a2)]):
        want, scale = sts.conv_target_loss(Gc, Pc, ttc, cc, aa, Cout, Cg, k, grp, d)
        assert abs(got - want) <= 1e-12 * (scale + tt), (got, want, scale)
    st.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,Din,Dout,K,d,seed", FC_ROWS, ids=[c[0] for c in FC_ROWS])
def test_fc_centered_sweep_matches_restatement(name, Din, Dout, K, d, seed, qcnn, ctx):
    W, ctrd, asmt, X, T, bias = fc_setup(Din, Dout, K, d, seed)
    st = qcnn.PqStats.fc(ctx, Din, Dout, d, target=True)
    sts.add_batches(st, sts.cuda(X), sts.cuda(T), sts.batchings(X.shape[0])["uneven"])
    G, P, tt = st.read()
    s, u, n = st.read_sums()
    Gc, Pc, ttc = centered(G, P, tt, s, u, n, 1)
    c, a, b, loss = st.refine_bias(W, ctrd, asmt, bias, sweeps=1)
    want_c, want_a, _ = fcr.refine_ref(W, sts.Fed(Gc, Din), ctrd, asmt, 1, follow=(c, a))
    assert ulps(c, want_c).max() <= 1.0 and np.array_equal(a, want_a)
    for got, (cc, aa) in zip(loss, [(ctrd, asmt), (c, a)]):
        E = W.astype(np.float64) - fcr.decoded(cc, aa, Din)
        want = float(((E @ Gc) * E).sum())
        assert abs(got - want) <= 1e-12 * want, (got, want)
    c2, a2, b2, loss2 = st.refine_target_bias(ctrd, asmt, bias, sweeps=1)
    want_c, want_a, _ = tgr.fc_target_ref(sts.Fed(Gc, Din), sts.Fed(Pc, Din), ctrd, asmt, 1, follow=(c2, a2))
    assert ulps(c2, want_c).max() <= 1.0 and np.array_equal(a2, want_a)
    for got, (cc, aa) in zip(loss2, [(ctrd, asmt), (c2, a2)]):
        Wh = fcr.decoded(cc, aa, Din)
        quad = float(((Wh @ Gc) * Wh).sum())
        want = ttc - 2 * float((Wh * Pc).sum()) + quad
        assert abs(got - want) <= 1e-12 * (tt + quad), (got, want)
    st.close()


# ---- 4. the refit bias and the loss against the calibration data ---------------------------------------------------
def _check_against_data(resid, b0, b, loss, loss_plain0, scale, rows):
    """resid(dbias) = the fp64 residual rows [rows][Dout] of the data with the bias changed by dbias"""
    r = resid(b.astype(np.float64) - b0.astype(np.float64))
    got = float((r * r).sum())
    rounding = rows * float((np.spacing(np.abs(b)).astype(np.float64) ** 2).sum())   # b^ is rounded to fp32
    tol = 1e-13 * (3 * scale + 2 * loss_plain0) + rounding
    assert abs(got - loss[-1]) <= tol, (got, loss[-1], tol)
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("sweeps", [0, 2])
def test_bias_and_loss_agree_with_the_data(sweeps, qcnn, ctx):
    import torch
    # FC
    W, ctrd, asmt, X, T, bias = fc_setup(250, 200, 32, 4, 91)
    st = qcnn.PqStats.fc(ctx, 250, 200, 4, target=True)
    sts.add_batches(st, sts.cuda(X), sts.cuda(T), sts.batchings(X.shape[0])["uneven"])
    X64, T64, W64 = X.astype(np.float64), T.astype(np.float64), W.astype(np.float64)
    n = X.shape[0]
    for target in (False, True):
        if target:
            c, a, b, loss = st.refine_target_bias(ctrd, asmt, bias, sweeps=sweeps)
            plain = st.refine_target(ctrd, asmt, sweeps=0)[2]
            ref = T64
        else:
            c, a, b, loss = st.refine_bias(W, ctrd, asmt, bias, sweeps=sweeps)
            plain = st.refine(W, ctrd, asmt, sweeps=0)[2]
            ref = X64 @ W64.T
        R = ref - X64 @ fcr.decoded(c, a, 250).T
        _check_against_data(lambda db: R - db[None, :], bias, b, loss, plain[0], float((ref * ref).sum()), n)
        if sweeps == 0:
            mean = R.mean(0)
            want = plain[0] - n * float(mean @ mean)
            assert abs(loss[0] - want) <= 1e-13 * (3 * float((ref * ref).sum()) + 2 * plain[0]), (loss[0], want)
            assert np.array_equal(c, ctrd) and np.array_equal(a, asmt)
        assert np.all(np.diff(loss) <= 1e-13 * (3 * float((ref * ref).sum()) + 2 * plain[0]))
    st.close()
    # conv
    name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed = REFINE_CONV[1]
    Cg = Cin // grp
    W, ctrd, asmt, x, t, bias = conv_setup(Cin, H, Cout, k, pad, stride, grp, K, d, N, seed)
    st = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, stride=stride, grp=grp, target=True)
    sts.add_batches(st, x, t, sts.batchings(N)["uneven"])
    rows = N * cvr.out_size(H, k, pad, stride) ** 2
    for target in (False, True):
        if target:
            c, a, b, loss = st.refine_target_bias(ctrd, asmt, bias, sweeps=sweeps)
            plain = st.refine_target(ctrd, asmt, sweeps=0)[2]
            ref = t.double()
        else:
            c, a, b, loss = st.refine_bias(W, ctrd, asmt, bias, sweeps=sweeps)
            plain = st.refine(W, ctrd, asmt, sweeps=0)[2]
            ref = tgr.conv_fwd(x, W, pad, stride, grp)
        R = (ref - tgr.conv_fwd(x, decode(dict(ctrd=c, asmt=a), Cg), pad, stride, grp)).reshape(-1, Cout)
        scale = float((ref * ref).sum())

        def resid(db):
            return (R - torch.from_numpy(db).to(R.device)[None, :]).cpu().numpy()

        _check_against_data(resid, bias, b, loss, plain[0], scale, rows)
        if sweeps == 0:
            mean = R.mean(0).cpu().numpy()
            want = plain[0] - rows * float(mean @ mean)
            assert abs(loss[0] - want) <= 1e-13 * (3 * scale + 2 * plain[0]), (loss[0], want)
        assert np.all(np.diff(loss) <= 1e-13 * (3 * scale + 2 * plain[0]))
    st.close()


# ---- 5. a constant input channel: centered blocks singular at rounding level ---------------------------------------
def _finite_descent(c, b, loss, tol):
    assert np.isfinite(c).all() and np.isfinite(b).all() and np.isfinite(loss).all()
    assert np.all(np.diff(loss) <= tol), (loss, tol)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [1, 4])
def test_constant_channel(d, qcnn, ctx):
    # FC: input column 5 is 0.1 in every row (its centered Gram row is zero up to rounding)
    Din, Dout, K = 24, 64, 16
    W, ctrd, asmt = fcr.start(Din, Dout, K, d, 101)
    X = fcr.gaussian_inputs(60, Din, 102) + np.float32(SHIFT)
    X[:, 5] = np.float32(0.1)
    T = tgr.fc_targets(X, W, 103)
    bias = np.random.RandomState(104).randn(Dout).astype(np.float32)
    st = qcnn.PqStats.fc(ctx, Din, Dout, d, target=True)
    sts.add_batches(st, sts.cuda(X), sts.cuda(T), [25, 35])
    tt = st.read()[2]
    c, a, b, loss = st.refine_bias(W, ctrd, asmt, bias, sweeps=3)
    _finite_descent(c, b, loss, 1e-12 * loss[0])
    c, a, b, loss = st.refine_target_bias(ctrd, asmt, bias, sweeps=3)
    _finite_descent(c, b, loss, 1e-13 * (3 * tt + 2 * loss[0]))
    st.close()
    # conv: channel 2 is 0.1 in every pixel of every image, no padding, so every patch sees it in every tap
    Cin, H, Cout, k = 4, 7, 16, 3
    W, ctrd, asmt = cvr.start(Cout, Cin, k, K, d, 105)
    X = cvr.maps(5, H, H, Cin, 106) + np.float32(SHIFT)
    X[..., 2] = np.float32(0.1)
    x = sts.cuda(X)
    t = tgr.conv_targets(x, W, 0, 1, 1, 107)
    bias = np.random.RandomState(108).randn(Cout).astype(np.float32)
    st = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, target=True)
    sts.add_batches(st, x, t, [2, 3])
    tt = st.read()[2]
    c, a, b, loss = st.refine_bias(W, ctrd, asmt, bias, sweeps=3)
    _finite_descent(c, b, loss, 1e-12 * loss[0])
    c, a, b, loss = st.refine_target_bias(ctrd, asmt, bias, sweeps=3)
    _finite_descent(c, b, loss, 1e-13 * (3 * tt + 2 * loss[0]))
    st.close()


# ---- 6. rejections --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rejected_bias_calls(qcnn, ctx):
    Cin, H, Cout, k, pad, stride, grp, K, d, N = 16, 8, 24, 3, 1, 1, 1, 16, 4, 3
    W, ctrd, asmt, x, t, bias = conv_setup(Cin, H, Cout, k, pad, stride, grp, K, d, N, 111)
    st = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, target=True)
    same = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad)
    _raises(qcnn, lambda: st.refine_target_bias(ctrd, asmt, bias, sweeps=1), "no calibration data")
    _raises(qcnn, lambda: same.refine_bias(W, ctrd, asmt, bias, sweeps=1), "no calibration data")
    st.add(x, t)
    same.add(x)
    snap = snapshot(st) + b"".join(a.tobytes() if isinstance(a, np.ndarray) else np.float64(a).tobytes() for a in st.read())
    b_bad = bias.copy()
    b_bad[3] = np.nan
    _raises(qcnn, lambda: st.refine_bias(W, ctrd, asmt, b_bad, sweeps=1), "qcnn_pq_stats_refine_bias: the bias contains a non-finite value")
    b_bad[3] = np.inf
    _raises(qcnn, lambda: st.refine_target_bias(ctrd, asmt, b_bad, sweeps=1),
            "qcnn_pq_stats_refine_target_bias: the bias contains a non-finite value")
    _raises(qcnn, lambda: same.refine_target_bias(ctrd, asmt, bias, sweeps=1), "created without a target")
    _raises(qcnn, lambda: st.refine_bias(W, ctrd, asmt, bias, sweeps=-1), "negative")
    a_bad = asmt.copy()
    a_bad[0, 0, 0, 0] = K
    _raises(qcnn, lambda: st.refine_bias(W, ctrd, a_bad, bias, sweeps=1), "not below K")
    c_bad = ctrd.copy()
    c_bad[0, 0, 0] = np.nan
    _raises(qcnn, lambda: st.refine_target_bias(c_bad, asmt, bias, sweeps=1), "codebook contains a non-finite value")
    w_bad = W.copy()
    w_bad[0, 0, 0, 0] = np.inf
    _raises(qcnn, lambda: st.refine_bias(w_bad, ctrd, asmt, bias, sweeps=1), "weights contain a non-finite value")
    c12 = np.zeros((ctrd.shape[0], 12, d), np.float32)
    _raises(qcnn, lambda: st.refine_bias(W, c12, np.zeros_like(asmt), bias, sweeps=1), "K=12")
    # shapes in Python
    _raises(qcnn, lambda: st.refine_bias(W, ctrd, asmt, bias[:-1], sweeps=1), "bias must be")
    _raises(qcnn, lambda: st.refine_target_bias(ctrd, asmt, np.zeros((Cout, 1)), sweeps=1), "bias must be")
    # NULL arguments through the C ABI
    lib = qcnn.lib
    vp = C.c_void_p
    cp, ap, bp = ctrd.ctypes.data_as(vp), asmt.ctypes.data_as(vp), bias.ctypes.data_as(vp)
    assert lib.qcnn_pq_stats_refine_bias(st.h, K, 1, W.ctypes.data_as(vp), cp, ap, None, None, None) != 0
    assert "qcnn_pq_stats_refine_bias: NULL argument" in qcnn.last_error()
    assert lib.qcnn_pq_stats_refine_target_bias(st.h, K, 1, cp, ap, None, None, None) != 0
    assert "qcnn_pq_stats_refine_target_bias: NULL argument" in qcnn.last_error()
    assert lib.qcnn_pq_stats_refine_target_bias(None, K, 1, cp, ap, bp, None, None) != 0 and "NULL" in qcnn.last_error()
    assert lib.qcnn_pq_stats_read_sums_h(None, None, None, None) != 0
    assert "qcnn_pq_stats_read_sums_h: NULL argument" in qcnn.last_error()
    u = np.empty(Cout)
    assert lib.qcnn_pq_stats_read_sums_h(same.h, None, u.ctypes.data_as(vp), None) != 0
    assert "kept only by statistics created with a target" in qcnn.last_error()
    # none of them changed the statistics
    assert snap == snapshot(st) + b"".join(a.tobytes() if isinstance(a, np.ndarray) else np.float64(a).tobytes()
                                           for a in st.read())
    st.close()
    same.close()
