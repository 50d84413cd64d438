"""Error correction damped toward the original weights (qcnn_pq_stats_refine_damped, DESIGN.md 4e "Damping toward the
original weights"): damp = 0 reproducing the four undamped calls bit for bit, the sweeps on the damped copies
G' = G + lambda_g I, P' = P + lambda_g W (numpy forms them bit for bit) against the existing restatements, the damped
loss against the calibration data, the skip rule with and without damping, a weakly spanned calibration set where
damping lowers the held-out error of the target form, reproducibility and every rejection."""
import ctypes as C
import re

import numpy as np
import pytest

import test_gpu_pq_bias as bia
import test_gpu_pq_refine as fcr
import test_gpu_pq_refine_conv as cvr
import test_gpu_pq_refine_target as tgr
import test_gpu_pq_stats as sts
from test_gpu_pq_bias import centered, snapshot
from test_gpu_pq_quantize import decode, ulps

SYMBOL = "qcnn_pq_stats_refine_damped"
DAMP = 0.1
FC_ROWS = [r for r in fcr.ONE_SWEEP if r[0] in ("d4_blocks", "d1_blocks")]     # several sweep blocks, d = 4 and 1
CONV_ROWS = [r for r in cvr.ONE_SWEEP if r[0] in ("3x3_grp2_partial", "conv1_like")]   # groups + partial; stride 4, Cin 3


def test_damped_symbol_declared_and_exported(qcnn):
    text = open(qcnn.HEADER_PATH).read()
    lib = C.CDLL(qcnn.LIB_PATH)
    assert re.search(r"QCNN_API\s+\w+\s+%s\s*\(" % SYMBOL, text)
    assert hasattr(lib, SYMBOL) and SYMBOL in qcnn.EXPORTS


def test_rows_reach_blocks_groups_stride4_and_partial_subspaces():
    assert {r[4] for r in FC_ROWS} == {1, 4}
    assert all(len(fcr.blocks(r[1], r[4])) > 1 for r in FC_ROWS)
    seen = set()
    for name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed in CONV_ROWS:
        seen |= {"groups"} if grp > 1 else set()
        seen |= {"stride4_cin3"} if stride == 4 and Cin == 3 else set()
        seen |= {"partial"} if (Cin // grp) % d else set()
    assert seen == {"groups", "stride4_cin3", "partial"}, seen


# ---- the damped copies, restated --------------------------------------------------------------------------------------
def lambdas(G, damp):
    """lambda_g = damp (tr_g / Dg) per group, tr_g the sequential sum of G_g's diagonal in ascending order, 0 unless
    tr_g > 0: the device's values bit for bit"""
    Gs = G[None] if G.ndim == 2 else G
    Dg = Gs.shape[-1]
    lam = []
    for Gg in Gs:
        tr = float(np.cumsum(np.diagonal(Gg))[-1])
        lam.append(damp * (tr / Dg) if tr > 0 else 0.0)
    return lam


def damped(G, P, tt, Wq, lam):
    """(G', P', |T'|^2): G' and P' bit for bit (elementwise, every operation rounded), |T'|^2 with numpy's sum of the
    squared weights; Wq [Cout][Dg] the weights in the internal dim order"""
    Gs = (G[None] if G.ndim == 2 else G).copy()
    i = np.arange(Gs.shape[-1])
    for g, lg in enumerate(lam):
        Gs[g, i, i] = Gs[g, i, i] + lg
    Gd = Gs[0] if G.ndim == 2 else Gs
    if P is None:
        return Gd, None, None
    Cpg = P.shape[0] // len(lam)
    W64 = Wq.astype(np.float64)
    Pd = P + np.repeat(np.array(lam), Cpg)[:, None] * W64
    acc = 0.0
    for g, lg in enumerate(lam):
        acc += lg * float((W64[g * Cpg:(g + 1) * Cpg] ** 2).sum())
    return Gd, Pd, tt + acc


def internal(W, d):
    """the weights [Cout][Dg] in the refine's internal dim order (FC: as given)"""
    if W.ndim == 2:
        return W
    Cout, Cg, k, _ = W.shape
    return W.reshape(Cout, -1)[:, cvr.dim_order(Cg, d, k * k)]


def base_sums(st, bias):
    """the sums the sweeps read: raw, or centered (with the bias refit)"""
    G, P, tt = st.read()
    if not bias:
        return G, P, tt
    s, u, n = st.read_sums()
    return centered(G, P, tt, s, u, n, G.shape[0] if G.ndim == 3 else 1)


def fc_stats(qcnn, ctx, Din, Dout, K, d, seed):
    W, ctrd, asmt, X, T, b = bia.fc_setup(Din, Dout, K, d, seed)
    st = qcnn.PqStats.fc(ctx, Din, Dout, d, target=True)
    sts.add_batches(st, sts.cuda(X), sts.cuda(T), sts.batchings(X.shape[0])["uneven"])
    return st, W, ctrd, asmt, X, T, b


def conv_stats(qcnn, ctx, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed):
    W, ctrd, asmt, x, t, b = bia.conv_setup(Cin, H, Cout, k, pad, stride, grp, K, d, N, seed)
    st = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, stride=stride, grp=grp, target=True)
    sts.add_batches(st, x, t, sts.batchings(N)["uneven"])
    return st, W, ctrd, asmt, x, t, b


def _call(st, W, ctrd, asmt, damp, target, bias, sweeps):
    """(ctrd, asmt, bias or None, loss) of one damped call"""
    r = st.refine_damped(W, ctrd, asmt, damp, target=target, bias=bias, sweeps=sweeps)
    return r if bias is not None else (r[0], r[1], None, r[2])


def _same_bits(a, b):
    return len(a) == len(b) and all(u.tobytes() == v.tobytes() for u, v in zip(a, b))


# ---- 2. damp = 0 is the undamped call ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("sweeps", [0, 1, 2])
def test_zero_damp_gives_the_undamped_calls(sweeps, qcnn, ctx):
    name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed = CONV_ROWS[0]
    sc, Wc, cc, ac, _, _, bc = conv_stats(qcnn, ctx, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed)
    sf, Wf, cf, af, _, _, bf = fc_stats(qcnn, ctx, 250, 200, 32, 4, 81)
    for st, W, c0, a0, b0 in ((sc, Wc, cc, ac, bc), (sf, Wf, cf, af, bf)):
        assert _same_bits(st.refine_damped(W, c0, a0, 0.0, sweeps=sweeps), st.refine(W, c0, a0, sweeps=sweeps))
        assert _same_bits(st.refine_damped(W, c0, a0, 0.0, target=True, sweeps=sweeps),
                          st.refine_target(c0, a0, sweeps=sweeps))
        assert _same_bits(st.refine_damped(W, c0, a0, 0.0, bias=b0, sweeps=sweeps),
                          st.refine_bias(W, c0, a0, b0, sweeps=sweeps))
        assert _same_bits(st.refine_damped(W, c0, a0, 0.0, target=True, bias=b0, sweeps=sweeps),
                          st.refine_target_bias(c0, a0, b0, sweeps=sweeps))
        st.close()


# ---- 3. the sweeps on the damped copies against the restatements ---------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("name,Din,Dout,K,d,seed", FC_ROWS, ids=[r[0] for r in FC_ROWS])
def test_fc_damped_sweep_matches_restatement(name, Din, Dout, K, d, seed, bias, qcnn, ctx):
    st, W, ctrd, asmt, X, T, b0 = fc_stats(qcnn, ctx, Din, Dout, K, d, seed)
    G, P, tt = base_sums(st, bias)
    lam = lambdas(G, DAMP)
    assert lam[0] > 0
    Gd, Pd, ttd = damped(G, P, tt, W, lam)
    bb = b0 if bias else None
    c, a, _, loss = _call(st, W, ctrd, asmt, DAMP, False, bb, 1)
    want_c, want_a, _ = fcr.refine_ref(W, sts.Fed(Gd, Din), ctrd, asmt, 1, follow=(c, a))
    assert ulps(c, want_c).max() <= 1.0 and np.array_equal(a, want_a)
    for got, (cc, aa) in zip(loss, [(ctrd, asmt), (c, a)]):
        E = W.astype(np.float64) - fcr.decoded(cc, aa, Din)
        want = float(((E @ Gd) * E).sum())
        assert abs(got - want) <= 1e-12 * want, (got, want)
    c2, a2, _, loss2 = _call(st, W, ctrd, asmt, DAMP, True, bb, 1)
    want_c, want_a, _ = tgr.fc_target_ref(sts.Fed(Gd, Din), sts.Fed(Pd, Din), ctrd, asmt, 1, follow=(c2, a2))
    assert ulps(c2, want_c).max() <= 1.0 and np.array_equal(a2, want_a)
    for got, (cc, aa) in zip(loss2, [(ctrd, asmt), (c2, a2)]):
        Wh = fcr.decoded(cc, aa, Din)
        quad = float(((Wh @ Gd) * Wh).sum())
        want = ttd - 2 * float((Wh * Pd).sum()) + quad
        assert abs(got - want) <= 1e-12 * (ttd + quad), (got, want)
    st.close()


@pytest.mark.gpu
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("name,Cin,H,Cout,k,pad,stride,grp,K,d,N,seed", CONV_ROWS, ids=[r[0] for r in CONV_ROWS])
def test_conv_damped_sweep_matches_restatement(name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed, bias, qcnn, ctx):
    Cg = Cin // grp
    st, W, ctrd, asmt, x, t, b0 = conv_stats(qcnn, ctx, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed)
    G, P, tt = base_sums(st, bias)
    lam = lambdas(G, DAMP)
    assert min(lam) > 0 and len(lam) == grp
    Gd, Pd, ttd = damped(G, P, tt, internal(W, d), lam)
    bb = b0 if bias else None
    c, a, _, loss = _call(st, W, ctrd, asmt, DAMP, False, bb, 1)
    want_c, want_a, _ = cvr.sweep_ref(W, list(Gd), ctrd, asmt, grp, 1, follow=(c, a))
    assert ulps(c, want_c).max() <= 1.0 and np.array_equal(a, want_a)
    for got, (cc, aa) in zip(loss, [(ctrd, asmt), (c, a)]):
        want = sts.conv_loss(W, Gd, cc, aa, grp, d)
        assert abs(got - want) <= 1e-12 * want, (got, want)
    c2, a2, _, loss2 = _call(st, W, ctrd, asmt, DAMP, True, bb, 1)
    want_c, want_a, _ = tgr.conv_target_sweep_ref(list(Gd), Pd, ctrd, asmt, grp, k, 1, follow=(c2, a2))
    assert ulps(c2, want_c).max() <= 1.0 and np.array_equal(a2, want_a)
    for got, (cc, aa) in zip(loss2, [(ctrd, asmt), (c2, a2)]):
        want, scale = sts.conv_target_loss(Gd, Pd, ttd, cc, aa, Cout, Cg, k, grp, d)
        assert abs(got - want) <= 1e-12 * (scale + ttd), (got, want, scale)
    st.close()


# ---- 4. the damped loss against the calibration data ---------------------------------------------------------------
def _anchor_term(W, Wh, lam):
    """(sum_g lambda_g |W_g - W^_g|^2, sum_g lambda_g (|W_g|^2 + |W^_g|^2)) in fp64, W and W^ [Cout][...]"""
    Cpg = W.shape[0] // len(lam)
    D = (W.astype(np.float64) - Wh).reshape(W.shape[0], -1)
    S = (W.astype(np.float64) ** 2 + Wh ** 2).reshape(W.shape[0], -1)
    term = sum(lg * float((D[g * Cpg:(g + 1) * Cpg] ** 2).sum()) for g, lg in enumerate(lam))
    scale = sum(lg * float(S[g * Cpg:(g + 1) * Cpg].sum()) for g, lg in enumerate(lam))
    return term, scale


def _check_losses(runs, data_loss, lam, W, decode_fn, scale, rows):
    """runs[s] = (ctrd, asmt, bias, loss) after s sweeps; every loss[s] of the longest run against the data"""
    full = runs[-1][3]
    for s, (c, a, b, loss) in enumerate(runs):
        assert loss.tobytes() == full[:s + 1].tobytes()
        Wh = np.asarray(decode_fn(c, a), np.float64)
        resid, bround = data_loss(Wh, b)
        term, tscale = _anchor_term(W, Wh, lam)
        got = resid + term
        tol = 1e-12 * (scale + tscale + full[0]) + rows * bround
        assert abs(got - full[s]) <= tol, (s, got, full[s], tol)
    assert np.all(np.diff(full) <= 1e-12 * (scale + full[0])), full


@pytest.mark.gpu
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("target", [False, True])
def test_damped_loss_agrees_with_the_data(target, bias, qcnn, ctx):
    import torch
    sweeps = 2
    # FC
    st, W, ctrd, asmt, X, T, b0 = fc_stats(qcnn, ctx, 250, 200, 32, 4, 91)
    lam = lambdas(base_sums(st, bias)[0], DAMP)
    X64, W64 = X.astype(np.float64), W.astype(np.float64)
    ref = T.astype(np.float64) if target else X64 @ W64.T
    bb = b0 if bias else None
    runs = [_call(st, W, ctrd, asmt, DAMP, target, bb, s) for s in range(sweeps + 1)]

    def fc_data(Wh, b):
        db = np.zeros(W.shape[0]) if b is None else b.astype(np.float64) - b0.astype(np.float64)
        R = ref - X64 @ Wh.T - db[None, :]
        bround = 0.0 if b is None else float((np.spacing(np.abs(b)).astype(np.float64) ** 2).sum())
        return float((R * R).sum()), bround

    _check_losses(runs, fc_data, lam, W, lambda c, a: fcr.decoded(c, a, 250), float((ref * ref).sum()), X.shape[0])
    st.close()
    # conv
    name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed = sts.REFINE_CONV[1]
    Cg = Cin // grp
    st, W, ctrd, asmt, x, t, b0 = conv_stats(qcnn, ctx, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed)
    lam = lambdas(base_sums(st, bias)[0], DAMP)
    ref = t.double() if target else tgr.conv_fwd(x, W, pad, stride, grp)
    bb = b0 if bias else None
    runs = [_call(st, W, ctrd, asmt, DAMP, target, bb, s) for s in range(sweeps + 1)]

    def conv_data(Wh, b):
        R = (ref - tgr.conv_fwd(x, Wh, pad, stride, grp)).reshape(-1, Cout)
        if b is not None:
            R = R - torch.from_numpy(b.astype(np.float64) - b0.astype(np.float64)).to(R.device)[None, :]
        bround = 0.0 if b is None else float((np.spacing(np.abs(b)).astype(np.float64) ** 2).sum())
        return float((R * R).sum()), bround

    rows = N * cvr.out_size(H, k, pad, stride) ** 2
    _check_losses(runs, conv_data, lam, W, lambda c, a: decode(dict(ctrd=c, asmt=a), Cg).astype(np.float64),
                  float((ref * ref).sum()), rows)
    st.close()


# ---- 5. the skip rule --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("target", [False, True])
def test_zero_input_subspace_is_fitted_when_damped(target, qcnn, ctx):
    Din, Dout, K, d = 48, 96, 16, 4
    W, ctrd, asmt = fcr.start(Din, Dout, K, d, 121)
    X = fcr.gaussian_inputs(100, Din, 122)
    X[:, 8:12] = 0   # subspace 2 has no input energy
    T = tgr.fc_targets(X, W, 123)
    st = qcnn.PqStats.fc(ctx, Din, Dout, d, target=True)
    st.add(sts.cuda(X), sts.cuda(T))
    G, P, tt = st.read()
    assert not G[8:12, 8:12].any()
    plain = st.refine_target(ctrd, asmt, sweeps=1) if target else st.refine(W, ctrd, asmt, sweeps=1)
    assert np.array_equal(plain[0][2], ctrd[2]) and np.array_equal(plain[1][:, 2], asmt[:, 2])   # skipped
    lam = lambdas(G, DAMP)
    Gd, Pd, _ = damped(G, P, tt, W, lam)
    c, a, loss = st.refine_damped(W, ctrd, asmt, DAMP, target=target, sweeps=1)
    if target:
        want_c, want_a, _ = tgr.fc_target_ref(sts.Fed(Gd, Din), sts.Fed(Pd, Din), ctrd, asmt, 1, follow=(c, a))
    else:
        want_c, want_a, _ = fcr.refine_ref(W, sts.Fed(Gd, Din), ctrd, asmt, 1, follow=(c, a))
    assert ulps(c, want_c).max() <= 1.0 and np.array_equal(a, want_a)
    assert not np.array_equal(c[2], ctrd[2])   # fitted to the weights
    # in the Euclidean metric: each used codeword of subspace 2 is at least as close to its members' weights as before
    Ws = W[:, 8:12].astype(np.float64)
    before = ((Ws - ctrd[2][asmt[:, 2]]) ** 2).sum()
    after = ((Ws - c[2][a[:, 2]]) ** 2).sum()
    assert after < before, (after, before)
    st.close()


@pytest.mark.gpu
@pytest.mark.parametrize("bias", [False, True])
def test_groups_without_input_keep_their_start(bias, qcnn, ctx):
    # FC: every input zero, so the one group's trace is 0 and lambda = 0
    Din, Dout, K, d = 40, 64, 16, 4
    W, ctrd, asmt = fcr.start(Din, Dout, K, d, 131)
    b0 = np.random.RandomState(132).randn(Dout).astype(np.float32)
    st = qcnn.PqStats.fc(ctx, Din, Dout, d, target=True)
    st.add(sts.cuda(np.zeros((30, Din))), sts.cuda(tgr.fc_targets(np.zeros((30, Din), np.float32), W, 133)))
    assert lambdas(base_sums(st, bias)[0], DAMP) == [0.0]
    for target in (False, True):
        c, a, b, loss = _call(st, W, ctrd, asmt, DAMP, target, b0 if bias else None, 2)
        assert np.array_equal(c, ctrd) and np.array_equal(a, asmt)
        plain = _call(st, W, ctrd, asmt, 0.0, target, b0 if bias else None, 2)
        assert _same_bits([x for x in (c, a, b, loss) if x is not None], [x for x in plain if x is not None])
    st.close()
    # conv: both groups' maps zero
    Cin, H, Cout, k, pad, stride, grp = 8, 6, 16, 3, 1, 1, 2
    W, ctrd, asmt = cvr.start(Cout, Cin // grp, k, K, d, 134)
    b0 = np.random.RandomState(135).randn(Cout).astype(np.float32)
    x = sts.cuda(np.zeros((2, H, H, Cin), np.float32))
    t = tgr.conv_targets(x, W, pad, stride, grp, 136)
    st = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, stride=stride, grp=grp, target=True)
    st.add(x, t)
    assert lambdas(base_sums(st, bias)[0], DAMP) == [0.0, 0.0]
    for target in (False, True):
        c, a, b, loss = _call(st, W, ctrd, asmt, DAMP, target, b0 if bias else None, 2)
        assert np.array_equal(c, ctrd) and np.array_equal(a, asmt)
    st.close()


@pytest.mark.gpu
@pytest.mark.parametrize("bias", [False, True])
def test_one_group_without_input_next_to_a_damped_group(bias, qcnn, ctx):
    """Group 1's input channels are zero, group 0's are live: lambda = [> 0, 0].  Group 0 is damped and group 1 keeps
    its assignments (its (group, tap) blocks have zero trace), in both forms and against the restatements, so a wrong
    group index in the damping would show as a mismatch."""
    Cin, H, Cout, k, pad, stride, grp, K, d, N = 20, 9, 32, 3, 1, 1, 2, 16, 4, 3
    Cg, Cpg = Cin // grp, Cout // grp
    W, ctrd, asmt = cvr.start(Cout, Cg, k, K, d, 171)
    X = cvr.maps(N, H, H, Cin, 172) + np.float32(bia.SHIFT)
    X[..., Cg:] = 0
    x = sts.cuda(X)
    t = tgr.conv_targets(x, W, pad, stride, grp, 173)
    b0 = np.random.RandomState(174).randn(Cout).astype(np.float32)
    st = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, stride=stride, grp=grp, target=True)
    sts.add_batches(st, x, t, [1, 2])
    G, P, tt = base_sums(st, bias)
    assert not G[1].any()
    lam = lambdas(G, DAMP)
    assert lam[0] > 0 and lam[1] == 0.0
    Gd, Pd, _ = damped(G, P, tt, internal(W, d), lam)
    bb = b0 if bias else None
    c, a, _, _ = _call(st, W, ctrd, asmt, DAMP, False, bb, 1)
    want_c, want_a, _ = cvr.sweep_ref(W, list(Gd), ctrd, asmt, grp, 1, follow=(c, a))
    assert ulps(c, want_c).max() <= 1.0 and np.array_equal(a, want_a)
    c2, a2, _, _ = _call(st, W, ctrd, asmt, DAMP, True, bb, 1)
    want_c, want_a, _ = tgr.conv_target_sweep_ref(list(Gd), Pd, ctrd, asmt, grp, k, 1, follow=(c2, a2))
    assert ulps(c2, want_c).max() <= 1.0 and np.array_equal(a2, want_a)
    for aa in (a, a2):
        assert np.array_equal(aa[Cpg:], asmt[Cpg:])       # group 1: skipped
        assert not np.array_equal(aa[:Cpg], asmt[:Cpg])   # group 0: refined
    st.close()


# ---- 6. what damping is for: a weakly spanned calibration set -------------------------------------------------------
@pytest.mark.gpu
def test_damping_lowers_the_held_out_error_of_a_weakly_spanned_fit(qcnn, ctx):
    """Calibration inputs y barely span dims 32..47 (scaled by 1e-3); the targets come from different inputs x (y is x
    passed through a re-quantized earlier layer, modelled as x plus noise); the held-out inputs have full energy in
    those dims.  The undamped target fit reaches into them; damping holds it near the original weights."""
    Din, Dout, K, d, N, sweeps = 64, 128, 16, 4, 256, 4
    W, ctrd, asmt = fcr.start(Din, Dout, K, d, 141)
    rng = np.random.RandomState(142)
    x = rng.randn(N, Din)
    y = x + 0.1 * rng.randn(N, Din)
    weak = slice(32, 48)
    x[:, weak] *= 1e-3
    y[:, weak] *= 1e-3
    T = (x @ W.astype(np.float64).T).astype(np.float32)
    st = qcnn.PqStats.fc(ctx, Din, Dout, d, target=True)
    st.add(sts.cuda(y.astype(np.float32)), sts.cuda(T))
    Z = np.random.RandomState(143).randn(512, Din)
    ref = Z @ W.astype(np.float64).T

    def held_out(c, a):
        R = ref - Z @ fcr.decoded(c, a, Din).T
        return float(np.linalg.norm(R) / np.linalg.norm(ref))

    c, a, loss = st.refine_target(ctrd, asmt, sweeps=sweeps)
    plain = held_out(c, a)
    c, a, loss = st.refine_damped(W, ctrd, asmt, 1e-2, target=True, sweeps=sweeps)
    damp = held_out(c, a)
    start = held_out(ctrd, asmt)
    print("held-out relative response error: start %.4f, target %.4f, target damp=1e-2 %.4f" % (start, plain, damp))
    assert damp < plain, (damp, plain)
    st.close()


# ---- 7. reproducibility and rejections -----------------------------------------------------------------------------
def _sums_bits(st):
    return snapshot(st) + b"".join(v.tobytes() if isinstance(v, np.ndarray) else np.float64(v).tobytes()
                                   for v in st.read())


@pytest.mark.gpu
def test_two_calls_give_the_same_bits(qcnn, ctx):
    name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed = CONV_ROWS[0]
    sc, Wc, cc, ac, _, _, bc = conv_stats(qcnn, ctx, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed)
    sf, Wf, cf, af, _, _, bf = fc_stats(qcnn, ctx, 250, 200, 32, 4, 151)
    for st, W, c0, a0, b0 in ((sc, Wc, cc, ac, bc), (sf, Wf, cf, af, bf)):
        before = _sums_bits(st)
        for target in (False, True):
            for bb in (None, b0):
                r1 = st.refine_damped(W, c0, a0, DAMP, target=target, bias=bb, sweeps=2)
                r2 = st.refine_damped(W, c0, a0, DAMP, target=target, bias=bb, sweeps=2)
                assert _same_bits(r1, r2)
                assert np.all(np.isfinite(r1[-1]))
        assert _sums_bits(st) == before
        st.close()


@pytest.mark.gpu
def test_rejected_damped_calls(qcnn, ctx):
    Cin, H, Cout, k, pad, stride, grp, K, d, N = 16, 8, 24, 3, 1, 1, 2, 16, 4, 3
    W, ctrd, asmt, x, t, bias = bia.conv_setup(Cin, H, Cout, k, pad, stride, grp, K, d, N, 161)
    st = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, grp=grp, target=True)
    same = qcnn.PqStats.conv(ctx, Cin, H, H, Cout, k, d, pad=pad, grp=grp)
    raises = lambda fn, text: bia._raises(qcnn, fn, text)   # noqa: E731
    raises(lambda: st.refine_damped(W, ctrd, asmt, DAMP, target=True), "no calibration data")
    raises(lambda: same.refine_damped(W, ctrd, asmt, DAMP), "no calibration data")
    st.add(x, t)
    same.add(x)
    snaps = [_sums_bits(st), snapshot(same) + same.read()[0].tobytes()]
    who = SYMBOL + ": "
    for target in (False, True):
        for damp in (-1e-3, float("nan"), float("inf"), -float("inf")):
            raises(lambda: st.refine_damped(W, ctrd, asmt, damp, target=target, sweeps=1), who + "damp=")
        w_bad = W.copy()
        w_bad[1, 2, 0, 1] = np.nan
        raises(lambda: st.refine_damped(w_bad, ctrd, asmt, DAMP, target=target, sweeps=1),
               who + "the weights contain a non-finite value")
        raises(lambda: st.refine_damped(W, ctrd, asmt, DAMP, target=target, sweeps=-1), "negative")
        a_bad = asmt.copy()
        a_bad[0, 0, 0, 0] = K
        raises(lambda: st.refine_damped(W, ctrd, a_bad, DAMP, target=target, sweeps=1), "not below K")
        c_bad = ctrd.copy()
        c_bad[0, 0, 0] = np.inf
        raises(lambda: st.refine_damped(W, c_bad, asmt, DAMP, target=target, sweeps=1), "codebook contains a non-finite")
        b_bad = bias.copy()
        b_bad[3] = np.nan
        raises(lambda: st.refine_damped(W, ctrd, asmt, DAMP, target=target, bias=b_bad, sweeps=1),
               who + "the bias contains a non-finite value")
        c12 = np.zeros((ctrd.shape[0], 12, d), np.float32)
        raises(lambda: st.refine_damped(W, c12, np.zeros_like(asmt), DAMP, target=target, sweeps=1), "K=12")
    raises(lambda: same.refine_damped(W, ctrd, asmt, DAMP, target=True, sweeps=1), "created without a target")
    raises(lambda: same.refine_damped(W, ctrd, asmt, DAMP, target=True, bias=bias, sweeps=1), "created without a target")
    # shapes in Python
    raises(lambda: st.refine_damped(W[:, :3], ctrd, asmt, DAMP), "wei must be")
    raises(lambda: st.refine_damped(W, ctrd, asmt, DAMP, bias=bias[:-1]), "bias must be")
    # through the C ABI: NULL weights in either form, target not 0 or 1, NULL statistics
    lib, vp = qcnn.lib, C.c_void_p
    wp, cp, ap = W.ctypes.data_as(vp), ctrd.copy().ctypes.data_as(vp), asmt.copy().ctypes.data_as(vp)
    for target in (0, 1):
        assert lib.qcnn_pq_stats_refine_damped(st.h, target, DAMP, K, 1, None, cp, ap, None, None, None) != 0
        assert who + "NULL argument" in qcnn.last_error()
    assert lib.qcnn_pq_stats_refine_damped(st.h, 2, DAMP, K, 1, wp, cp, ap, None, None, None) != 0
    assert who + "target=2 is not 0 or 1" in qcnn.last_error()
    assert lib.qcnn_pq_stats_refine_damped(None, 0, DAMP, K, 1, wp, cp, ap, None, None, None) != 0
    assert who + "NULL argument" in qcnn.last_error()
    # none of them changed the statistics
    assert _sums_bits(st) == snaps[0] and snapshot(same) + same.read()[0].tobytes() == snaps[1]
    st.close()
    same.close()
