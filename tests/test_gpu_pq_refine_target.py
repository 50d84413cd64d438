"""Error-correcting product quantization toward target responses (qcnn_pq_refine_fc_target / _conv_target, DESIGN.md
4e): the layer's inputs y come from the quantized network and the targets t from the original one, and the sweeps
lower sum_n |t_n - W^ y_n|^2.  Checked against numpy fp64 restatements in which R = P - G W^ (P = T^T Y) takes the
place of G E, and those restatements against the same-input ones when t = y W^T."""
import ctypes as C
import re
import tempfile

import numpy as np
import pytest

import test_gpu_pq_refine as fcr
import test_gpu_pq_refine_conv as cvr
from test_gpu_pq_quantize import decode, ulps


# ---- the restatements -----------------------------------------------------------------------------------------------
def fc_target_ref(Y, T, ctrd, asmt, sweeps, follow=None):
    """(ctrd, asmt, inside) after `sweeps` target sweeps on inputs Y [N][Din] and targets T [N][Dout]; the margins and
    `follow` as in test_gpu_pq_refine.refine_ref."""
    assert follow is None or sweeps == 1
    Y = Y.astype(np.float64)
    G = Y.T @ Y
    P = T.astype(np.float64).T @ Y
    Din = Y.shape[1]
    S, K, d = ctrd.shape
    ctrd, asmt = ctrd.copy(), asmt.copy()
    inside = 0
    for _ in range(sweeps):
        for m in range(S):
            c0, w = m * d, min(d, Din - m * d)
            sl = slice(c0, c0 + w)
            Gmm = G[sl, sl]
            tr = np.trace(Gmm)
            if tr == 0:
                continue
            R = P[:, sl] - fcr.decoded(ctrd, asmt, Din) @ G[:, sl]
            h = R + ctrd[m, asmt[:, m], :w].astype(np.float64) @ Gmm
            L = np.linalg.cholesky(Gmm + 1e-10 * tr / w * np.eye(w))
            for k in range(K):
                mem = asmt[:, m] == k
                n = int(mem.sum())
                if n == 0:
                    continue
                H = h[mem].sum(axis=0)
                D = np.linalg.solve(L.T, np.linalg.solve(L, H / n)).astype(np.float32)
                c = ctrd[m, k, :w]
                f = lambda v: n * (v @ Gmm @ v) - 2 * (v @ H)
                fD, fc = f(D.astype(np.float64)), f(c.astype(np.float64))
                if not np.array_equal(D, c):
                    scale = n * abs(D @ Gmm @ D) + n * abs(c @ Gmm @ c) + 2 * abs(D @ H) + 2 * abs(c @ H)
                    if abs(fD - fc) <= 1e-9 * scale:
                        assert follow is not None, ("accept-or-keep inside its margin", m, k, fD, fc)
                        got = follow[0][m, k, :w]
                        assert ulps(got, D).max() <= 1.0 or ulps(got, c).max() <= 1.0, (m, k)
                        ctrd[m, k, :w] = got
                        inside += 1
                        continue
                if fD < fc:
                    ctrd[m, k, :w] = D
            Cm = ctrd[m, :, :w].astype(np.float64)
            cc = ((Cm @ Gmm) * Cm).sum(axis=1)
            dot = h @ Cm.T
            v = cc[None, :] - 2 * dot
            two = np.sort(v, axis=1)[:, :2]
            scale = np.abs(cc).max() + 2 * np.abs(dot).max(axis=1)
            asmt[:, m], n_in = fcr.follow_argmin(v, two, 1e-6 * scale, m, follow)
            inside += n_in
    return ctrd, asmt, inside


def conv_cross(X, Tm, Cg, k, pad, stride, grp, d):
    """[Cout][Cg k k] fp64: row o = sum over positions of t[pos][o] p_g(pos), g = o's group, in the internal dim order"""
    perm = cvr.dim_order(Cg, d, k * k)
    Cout = Tm.shape[-1]
    Cpg = Cout // grp
    Tf = Tm.reshape(-1, Cout).astype(np.float64)
    P = np.empty((Cout, Cg * k * k))
    for g in range(grp):
        Pg = cvr.patches(X.astype(np.float64), g, Cg, k, pad, stride)[:, perm]
        P[g * Cpg:(g + 1) * Cpg] = Tf[:, g * Cpg:(g + 1) * Cpg].T @ Pg
    return P


def conv_cross_torch(x, t, Cg, k, pad, stride, grp, d, batch):
    """The same from device maps x [N][H][W][Cin] and t [N][Ho][Wo][Cout]: fp64 F.unfold over `batch` images at a time"""
    import torch
    import torch.nn.functional as F
    Dg, Cout = Cg * k * k, t.shape[-1]
    Cpg = Cout // grp
    perm = torch.from_numpy(cvr.dim_order(Cg, d, k * k)).to(x.device)
    P = torch.zeros((Cout, Dg), dtype=torch.float64, device=x.device)
    for i in range(0, x.shape[0], batch):
        xb = x[i:i + batch].permute(0, 3, 1, 2).double()
        tb = t[i:i + batch].reshape(-1, Cout).double()
        for g in range(grp):
            Pt = F.unfold(xb[:, g * Cg:(g + 1) * Cg], k, padding=pad, stride=stride)
            Pt = Pt.permute(0, 2, 1).reshape(-1, Dg)[:, perm]
            P[g * Cpg:(g + 1) * Cpg] += tb[:, g * Cpg:(g + 1) * Cpg].T @ Pt
    return P.cpu().numpy()


def conv_target_sweep_ref(G, P, ctrd, asmt, grp, k, sweeps, follow=None):
    """(ctrd, asmt, stats) after `sweeps` target sweeps from the Grams G (per group) and the cross products P [Cout][Dg];
    the margins, `follow` and stats as in test_gpu_pq_refine_conv.sweep_ref."""
    assert follow is None or sweeps == 1
    T = k * k
    S, K, d = ctrd.shape
    Cout, Dg = P.shape
    Cg, Cpg = Dg // T, Cout // grp
    perm = cvr.dim_order(Cg, d, T)
    ctrd, asmt = ctrd.copy(), asmt.copy()
    A = asmt.reshape(Cout, T, S)
    FA = None if follow is None else follow[1].reshape(Cout, T, S)
    grp_of = np.arange(Cout) // Cpg
    stats = {"inside": 0, "n": []}

    def decoded():
        return decode(dict(ctrd=ctrd, asmt=asmt), Cg).reshape(Cout, Dg)[:, perm].astype(np.float64)

    for _ in range(sweeps):
        for m in range(S):
            w = min(d, Cg - m * d)
            q0, nb = m * d * T, T * w
            blk = slice(q0, q0 + nb)
            if sum(np.trace(G[g][blk, blk]) for g in range(grp)) == 0:
                continue
            Wh = decoded()
            h = np.empty((Cout, nb))
            for g in range(grp):
                og = grp_of == g
                h[og] = P[og][:, blk] - Wh[og] @ G[g][:, blk] + Wh[og][:, blk] @ G[g][blk, blk]
            h = h.reshape(Cout, T, w)
            Am = A[:, :, m].astype(np.int64)
            U = np.nonzero(np.bincount(Am.ravel(), minlength=K))[0]
            nU = len(U)
            uidx = -np.ones(K, np.int64)
            uidx[U] = np.arange(nU)
            M4 = np.zeros((nU, w, nU, w))
            jj = np.arange(w)
            for g in range(grp):
                Gb = G[g][blk, blk].reshape(T, w, T, w)
                ug = uidx[Am[grp_of == g]]
                for t in range(T):
                    key = (np.arange(T)[None, :] * nU + ug[:, t:t + 1]) * nU + ug
                    keys, cnt = np.unique(key.ravel(), return_counts=True)
                    t2, u, u2 = keys // (nU * nU), (keys // nU) % nU, keys % nU
                    vals = cnt[:, None, None].astype(np.float64) * Gb[t][:, t2, :].transpose(1, 0, 2)
                    np.add.at(M4, (u[:, None, None], jj[None, :, None], u2[:, None, None], jj[None, None, :]), vals)
            n = nU * w
            stats["n"].append(n)
            M = M4.reshape(n, n)
            b = np.zeros((nU, w))
            np.add.at(b, uidx[Am.ravel()], h.reshape(-1, w))
            b = b.ravel()
            mu = 1e-10 * np.trace(M) / n
            L = np.linalg.cholesky(M + mu * np.eye(n))
            D = np.linalg.solve(L.T, np.linalg.solve(L, b)).astype(np.float32)
            Cu = ctrd[m, U, :w].ravel()
            Dd, Cd = D.astype(np.float64), Cu.astype(np.float64)
            diff = (Dd - Cd) @ (M @ (Dd + Cd) - 2 * b)
            scale = abs(Dd @ M @ Dd) + abs(Cd @ M @ Cd) + 2 * abs(Dd @ b) + 2 * abs(Cd @ b)
            if not np.array_equal(D, Cu) and abs(diff) <= 1e-9 * scale:
                assert follow is not None, ("accept-or-keep inside its margin", m, diff, scale)
                got = follow[0][m, U, :w].ravel()
                assert ulps(got, D).max() <= 1.0 or ulps(got, Cu).max() <= 1.0, m
                ctrd[m, U, :w] = got.reshape(nU, w)
                stats["inside"] += 1
            elif diff < 0:
                ctrd[m, U, :w] = D.reshape(nU, w)
            # assignment, taps in order, W^ current: h' = [P - G W^]_(m,t) + G_tt w^_t
            Wh = decoded()
            Cm = ctrd[m, :, :w].astype(np.float64)
            for o in range(Cout):
                Gg = G[grp_of[o]]
                for t in range(T):
                    r = slice(q0 + t * w, q0 + (t + 1) * w)
                    Gtt = Gg[r, r]
                    if np.trace(Gtt) == 0:
                        continue
                    hp = P[o, r] - Gg[r, :] @ Wh[o] + Gtt @ Wh[o, r]
                    cc = ((Cm @ Gtt) * Cm).sum(axis=1)
                    dot = Cm @ hp
                    v = cc - 2 * dot
                    two = np.sort(v)[:2]
                    margin = 1e-6 * (np.abs(cc).max() + 2 * np.abs(dot).max())
                    if two[1] - two[0] <= margin:
                        assert follow is not None, ("argmin inside its margin", m, o, t)
                        a = int(FA[o, t, m])
                        assert v[a] - two[0] <= margin, (m, o, t)
                        stats["inside"] += 1
                    else:
                        a = int(np.argmin(v))
                    A[o, t, m] = a
                    Wh[o, r] = Cm[a]
    return ctrd, asmt, stats


# ---- data -----------------------------------------------------------------------------------------------------------
def fc_targets(X, W, seed):
    """t = X W^T + 0.3 Z V^T in fp64, rounded to fp32: Z is an independent seeded input, V independent weights"""
    rng = np.random.RandomState(seed)
    Z = rng.randn(*X.shape)
    V = rng.randn(*W.shape) / np.sqrt(W.shape[1])
    return (X.astype(np.float64) @ W.astype(np.float64).T + 0.3 * Z @ V.T).astype(np.float32)


def conv_fwd(x, W, pad, stride, grp):
    """conv(x, W) in fp64, NHWC in and out (x a numpy array or a torch tensor; the result is a torch tensor)"""
    import torch
    import torch.nn.functional as F
    if not isinstance(x, torch.Tensor):
        x = torch.from_numpy(np.ascontiguousarray(x))
    Wt = torch.from_numpy(np.ascontiguousarray(W, np.float64)).to(x.device)
    return F.conv2d(x.double().permute(0, 3, 1, 2), Wt, stride=stride, padding=pad, groups=grp).permute(0, 2, 3, 1)


def conv_targets(x, W, pad, stride, grp, seed):
    """t = conv(x, W) + 0.3 conv(z, V), fp32 NHWC, with z independent seeded maps and V independent weights"""
    import torch
    rng = np.random.RandomState(seed)
    V = rng.randn(*W.shape) / np.sqrt(np.prod(W.shape[1:]))
    g = torch.Generator(device=x.device).manual_seed(seed)
    z = torch.randn(x.shape, generator=g, device=x.device, dtype=torch.float32)
    return (conv_fwd(x, W, pad, stride, grp) + 0.3 * conv_fwd(z, V, pad, stride, grp)).float().contiguous()


def fc_target_loss(Y, T, ctrd, asmt):
    """sum_n |t_n - W^ y_n|^2 from the data themselves"""
    R = T.astype(np.float64) - Y.astype(np.float64) @ fcr.decoded(ctrd, asmt, Y.shape[1]).T
    return float((R * R).sum())


def conv_target_loss(y, t, ctrd, asmt, k, pad, stride, grp):
    """sum (t - conv(y, W^))^2 in fp64 (torch, on y's device)"""
    Cg = y.shape[-1] // grp
    r = t.double() - conv_fwd(y, decode(dict(ctrd=ctrd, asmt=asmt), Cg), pad, stride, grp)
    return float((r * r).sum())


def tsq(t):
    return float((t.double() ** 2).sum()) if hasattr(t, "double") else float((t.astype(np.float64) ** 2).sum())


def dyadic_fc(Din, Dout, K, d, N, seed):
    """small-integer inputs, weights and codebook in multiples of 1/8, t = y W^T: every product and sum is exact"""
    rng = np.random.RandomState(seed)
    Y = rng.randint(-3, 4, size=(N, Din)).astype(np.float32)
    W = (rng.randint(-8, 9, size=(Dout, Din)) / 8.0).astype(np.float32)
    S = -(-Din // d)
    ctrd = (rng.randint(-8, 9, size=(S, K, d)) / 8.0).astype(np.float32)
    for m in range(S):
        ctrd[m, :, min(d, Din - m * d):] = 0
    asmt = rng.randint(0, K, size=(Dout, S)).astype(np.uint8)
    T = (Y.astype(np.float64) @ W.astype(np.float64).T).astype(np.float32)
    assert np.array_equal(T.astype(np.float64), Y.astype(np.float64) @ W.astype(np.float64).T)
    return Y, T, W, ctrd, asmt


def dyadic_conv(Cin, H, Cout, k, pad, stride, grp, K, d, N, seed):
    rng = np.random.RandomState(seed)
    Cg = Cin // grp
    X = rng.randint(-3, 4, size=(N, H, H, Cin)).astype(np.float32)
    W = (rng.randint(-8, 9, size=(Cout, Cg, k, k)) / 8.0).astype(np.float32)
    S = -(-Cg // d)
    ctrd = (rng.randint(-8, 9, size=(S, K, d)) / 8.0).astype(np.float32)
    for m in range(S):
        ctrd[m, :, min(d, Cg - m * d):] = 0
    asmt = rng.randint(0, K, size=(Cout, k, k, S)).astype(np.uint8)
    return X, W, ctrd, asmt


cuda = fcr.cuda


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_target_symbols_declared_and_exported(qcnn):
    text = open(qcnn.HEADER_PATH).read()
    for name in ("qcnn_pq_refine_fc_target", "qcnn_pq_refine_conv_target"):
        assert re.search(r"QCNN_API\s+int\s+%s\s*\(" % name, text), name
        assert hasattr(C.CDLL(qcnn.LIB_PATH), name), name
        assert name in qcnn.EXPORTS, name


@pytest.mark.parametrize("Din,Dout,K,d,seed", [(24, 40, 8, 4, 3), (30, 64, 16, 8, 4), (13, 20, 8, 1, 6)])
def test_fc_target_restatement_reduces_to_same_input(Din, Dout, K, d, seed):
    """With t = y W^T in fp64, P = W G and R = G (W - W^): the target restatement is the same-input one."""
    W, ctrd, asmt = fcr.start(Din, Dout, K, d, seed)
    X = fcr.gaussian_inputs(3 * Din, Din, seed + 1)
    T = X.astype(np.float64) @ W.astype(np.float64).T
    want_c, want_a, _ = fcr.refine_ref(W, X, ctrd, asmt, 2)
    c, a, _ = fc_target_ref(X, T, ctrd, asmt, 2)
    assert ulps(c, want_c).max() <= 1.0
    assert np.array_equal(a, want_a)
    assert not np.array_equal(a, asmt)


@pytest.mark.parametrize("Cin,H,Cout,k,pad,stride,grp,K,d,N,seed",
                         [(20, 7, 32, 3, 1, 1, 2, 16, 4, 2, 3), (12, 9, 24, 5, 2, 2, 1, 16, 8, 2, 4)])
def test_conv_target_restatement_reduces_to_same_input(Cin, H, Cout, k, pad, stride, grp, K, d, N, seed):
    Cg = Cin // grp
    W, ctrd, asmt = cvr.start(Cout, Cg, k, K, d, seed)
    X = cvr.maps(N, H, H, Cin, seed + 1)
    G = cvr.grams(X, Cg, k, pad, stride, grp, d)
    T = conv_fwd(X.astype(np.float64), W, pad, stride, grp).numpy()
    P = conv_cross(X, T, Cg, k, pad, stride, grp, d)
    want_c, want_a, want_s = cvr.sweep_ref(W, G, ctrd, asmt, grp, 2)
    c, a, s = conv_target_sweep_ref(G, P, ctrd, asmt, grp, k, 2)
    assert s["n"] == want_s["n"]
    assert ulps(c, want_c).max() <= 1.0
    assert np.array_equal(a, want_a)
    assert not np.array_equal(a, asmt)


# ---- sweeps = 0: the start and its loss -----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,Din,Dout,K,d,N,z0,zeros", fcr.ZERO_SWEEP, ids=[c[0] for c in fcr.ZERO_SWEEP])
def test_fc_zero_sweeps(name, Din, Dout, K, d, N, z0, zeros, qcnn, ctx):
    W, ctrd, asmt = fcr.start(Din, Dout, K, d, 11)
    X = fcr.gaussian_inputs(N, Din, 12)
    X[:, z0:z0 + zeros] = 0
    T = fc_targets(X, W, 13)
    c, a, loss = qcnn.pq_refine_fc_target(ctx, cuda(X), cuda(T), ctrd, asmt, sweeps=0)
    assert c.tobytes() == ctrd.tobytes() and a.tobytes() == asmt.tobytes()
    assert loss.shape == (1,)
    want = fc_target_loss(X, T, ctrd, asmt)
    assert abs(loss[0] - want) <= 1e-10 * tsq(T), (loss[0], want)


@pytest.mark.gpu
@pytest.mark.parametrize("name,Cin,H,Cout,k,pad,stride,grp,K,d,N", cvr.ZERO_SWEEP, ids=[c[0] for c in cvr.ZERO_SWEEP])
def test_conv_zero_sweeps(name, Cin, H, Cout, k, pad, stride, grp, K, d, N, qcnn, ctx):
    W, ctrd, asmt = cvr.start(Cout, Cin // grp, k, K, d, 11)
    x = cuda(cvr.maps(N, H, H, Cin, 12))
    t = conv_targets(x, W, pad, stride, grp, 13)
    c, a, loss = qcnn.pq_refine_conv_target(ctx, x, t, ctrd, asmt, k, pad=pad, stride=stride, grp=grp, sweeps=0)
    assert c.tobytes() == ctrd.tobytes() and a.tobytes() == asmt.tobytes()
    assert loss.shape == (1,)
    want = conv_target_loss(x, t, ctrd, asmt, k, pad, stride, grp)
    assert abs(loss[0] - want) <= 1e-10 * tsq(t), (loss[0], want)


# ---- one sweep against the restatement ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,Din,Dout,K,d,seed", fcr.ONE_SWEEP, ids=[c[0] for c in fcr.ONE_SWEEP])
def test_fc_one_sweep_matches_restatement(name, Din, Dout, K, d, seed, qcnn, ctx):
    W, ctrd, asmt = fcr.start(Din, Dout, K, d, seed)
    X = fcr.gaussian_inputs(2 * Din, Din, seed + 1)
    T = fc_targets(X, W, seed + 2)
    c, a, loss = qcnn.pq_refine_fc_target(ctx, cuda(X), cuda(T), ctrd, asmt, sweeps=1)
    want_c, want_a, inside = fc_target_ref(X, T, ctrd, asmt, 1, follow=(c, a))
    print("%s: %d of %d assignments and codewords decided inside their margins"
          % (name, inside, a.size + ctrd.shape[0] * K))
    assert ulps(c, want_c).max() <= 1.0
    assert np.array_equal(a, want_a)
    tt = tsq(T)
    assert loss[1] <= loss[0] + 1e-13 * (3 * tt + 2 * loss[0])
    want = fc_target_loss(X, T, c, a)
    assert abs(loss[1] - want) <= 1e-10 * (tt + want), (loss[1], want)


@pytest.mark.gpu
@pytest.mark.parametrize("name,Cin,H,Cout,k,pad,stride,grp,K,d,N,seed", cvr.ONE_SWEEP, ids=[c[0] for c in cvr.ONE_SWEEP])
def test_conv_one_sweep_matches_restatement(name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed, qcnn, ctx):
    """The chunked rows cross 3 and 4 patch chunks per group, so each chunk's target rows must be the right ones."""
    Cg = Cin // grp
    W, ctrd, asmt = cvr.start(Cout, Cg, k, K, d, seed)
    X = cvr.maps(N, H, H, Cin, seed + 1)
    x = cuda(X)
    t = conv_targets(x, W, pad, stride, grp, seed + 2)
    if cvr.patch_chunks(N, H, k, pad, stride, Cg) > 1:
        c0, a0, l0 = qcnn.pq_refine_conv_target(ctx, x, t, ctrd, asmt, k, pad=pad, stride=stride, grp=grp, sweeps=0)
        want = conv_target_loss(x, t, ctrd, asmt, k, pad, stride, grp)
        assert abs(l0[0] - want) <= 1e-10 * tsq(t), (l0[0], want)
        batch = max(1, (64 << 20) // (8 * Cg * k * k * cvr.out_size(H, k, pad, stride) ** 2))
        G = cvr.grams_torch(x, Cg, k, pad, stride, grp, d, batch)
        P = conv_cross_torch(x, t, Cg, k, pad, stride, grp, d, batch)
    else:
        G = cvr.grams(X, Cg, k, pad, stride, grp, d)
        P = conv_cross(X, t.cpu().numpy(), Cg, k, pad, stride, grp, d)
    c, a, loss = qcnn.pq_refine_conv_target(ctx, x, t, ctrd, asmt, k, pad=pad, stride=stride, grp=grp, sweeps=1)
    want_c, want_a, stats = conv_target_sweep_ref(G, P, ctrd, asmt, grp, k, 1, follow=(c, a))
    print("%s: systems n = %s, %d of %d decisions inside their margins"
          % (name, stats["n"], stats["inside"], a.size + len(stats["n"])))
    assert stats["n"] == cvr.system_sizes(Cg, d, k * k, asmt)
    assert ulps(c, want_c).max() <= 1.0
    assert np.array_equal(a, want_a)
    tt = tsq(t)
    assert loss[1] <= loss[0] + 1e-13 * (3 * tt + 2 * loss[0])
    want = conv_target_loss(x, t, c, a, k, pad, stride, grp)
    assert abs(loss[1] - want) <= 1e-10 * (tt + want), (loss[1], want)


# ---- reduction to the same-input form and the fixed point, on exact (dyadic) data -----------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("Din,Dout,K,d,N", [(300, 200, 16, 4, 400), (130, 96, 32, 8, 256)])
def test_fc_dyadic_target_equals_same_input(Din, Dout, K, d, N, qcnn, ctx):
    Y, T, W, ctrd, asmt = dyadic_fc(Din, Dout, K, d, N, 81)
    c1, a1, l1 = qcnn.pq_refine_fc(ctx, W, cuda(Y), ctrd, asmt, sweeps=2)
    c2, a2, l2 = qcnn.pq_refine_fc_target(ctx, cuda(Y), cuda(T), ctrd, asmt, sweeps=2)
    assert c2.tobytes() == c1.tobytes() and a2.tobytes() == a1.tobytes()
    assert not np.array_equal(a2, asmt)
    assert np.all(np.abs(l2 - l1) <= 1e-12 * l1), (l1, l2)


@pytest.mark.gpu
def test_conv_dyadic_target_equals_same_input(qcnn, ctx):
    """grouped 3x3 layer over 2 patch chunks per group (Dg = 1800: 37 282 positions a chunk, 64 800 in all)"""
    Cin, H, Cout, k, pad, stride, grp, K, d, N = 400, 18, 32, 3, 1, 1, 2, 16, 8, 200
    assert cvr.patch_chunks(N, H, k, pad, stride, Cin // grp) == 2
    X, W, ctrd, asmt = dyadic_conv(Cin, H, Cout, k, pad, stride, grp, K, d, N, 82)
    x = cuda(X)
    t = conv_fwd(x, W, pad, stride, grp)
    tf = t.float().contiguous()
    assert bool((tf.double() == t).all())
    c1, a1, l1 = qcnn.pq_refine_conv(ctx, W, x, ctrd, asmt, pad=pad, stride=stride, grp=grp, sweeps=2)
    c2, a2, l2 = qcnn.pq_refine_conv_target(ctx, x, tf, ctrd, asmt, k, pad=pad, stride=stride, grp=grp, sweeps=2)
    assert c2.tobytes() == c1.tobytes() and a2.tobytes() == a1.tobytes()
    assert not np.array_equal(a2, asmt)
    assert np.all(np.abs(l2 - l1) <= 1e-12 * l1), (l1, l2)


def _fixed_point_check(c, a, loss, Cs, As, m_axis):
    assert c.tobytes() == Cs.tobytes()
    assert (loss == 0).all(), loss
    differ = a != As
    if differ.any():   # only onto an equal codeword of lower index
        m_idx = np.nonzero(differ)[m_axis]
        assert np.array_equal(c[m_idx, a[differ]], c[m_idx, As[differ]])
        assert (a[differ] < As[differ]).all()


@pytest.mark.gpu
def test_fc_fixed_point(qcnn, ctx):
    Din, Dout, K, d, N = 130, 200, 32, 8, 260
    Y, _, _, Cs, As = dyadic_fc(Din, Dout, K, d, N, 83)
    W = fcr.decoded(Cs, As, Din).astype(np.float32)
    T = (Y.astype(np.float64) @ W.astype(np.float64).T).astype(np.float32)
    c, a, loss = qcnn.pq_refine_fc_target(ctx, cuda(Y), cuda(T), Cs, As, sweeps=3)
    _fixed_point_check(c, a, loss, Cs, As, 1)


@pytest.mark.gpu
def test_conv_fixed_point(qcnn, ctx):
    Cin, H, Cout, k, pad, stride, grp, K, d, N = 20, 9, 32, 3, 1, 1, 2, 16, 4, 3
    X, _, Cs, As = dyadic_conv(Cin, H, Cout, k, pad, stride, grp, K, d, N, 84)
    W = decode(dict(ctrd=Cs, asmt=As), Cin // grp).astype(np.float32)
    x = cuda(X)
    t = conv_fwd(x, W, pad, stride, grp).float().contiguous()
    c, a, loss = qcnn.pq_refine_conv_target(ctx, x, t, Cs, As, k, pad=pad, stride=stride, grp=grp, sweeps=3)
    _fixed_point_check(c, a, loss, Cs, As, 3)


# ---- descent and reproducibility ------------------------------------------------------------------------------------
def _descends(loss, tt):
    """no sweep raises the loss beyond its rounding (of order 1e-15 (|T|^2 + sum w^ G w^), and w^ G w^ <= 2 |T|^2 +
    2 loss), and the sweeps lower it in all"""
    slack = 1e-13 * (3 * tt + 2 * loss[0])
    return bool((loss[1:] <= loss[:-1] + slack).all() and loss[-1] < loss[0])


@pytest.mark.gpu
def test_fc_descent_and_reproducibility(qcnn, ctx):
    Din, Dout, K, d = 1024, 512, 32, 4
    W = (np.random.RandomState(51).randn(Dout, Din) / 32).astype(np.float32)
    X = fcr.gaussian_inputs(2048, Din, 52)
    T = fc_targets(X, W, 53)
    x, t, tt = cuda(X), cuda(T), tsq(T)
    c0, a0, _ = qcnn.pq_quantize_fc(ctx, W, K, d, iters=5, seed=3)
    c, a, loss = qcnn.pq_refine_fc_target(ctx, x, t, c0, a0, sweeps=4)
    assert loss.shape == (5,) and _descends(loss, tt), loss
    want = fc_target_loss(X, T, c, a)
    assert abs(loss[-1] - want) <= 1e-10 * (tt + want), (loss[-1], want)
    c2, a2, l2 = qcnn.pq_refine_fc_target(ctx, x, t, c0, a0, sweeps=4)
    assert c2.tobytes() == c.tobytes() and a2.tobytes() == a.tobytes() and l2.tobytes() == loss.tobytes()
    # from the same-input optimum on the same inputs, the target sweeps still lower the target loss
    cs, as_, _ = qcnn.pq_refine_fc(ctx, W, x, c0, a0, sweeps=4)
    _, _, lt = qcnn.pq_refine_fc_target(ctx, x, t, cs, as_, sweeps=3)
    assert abs(lt[0] - fc_target_loss(X, T, cs, as_)) <= 1e-10 * tt
    assert _descends(lt, tt), lt


@pytest.mark.gpu
def test_conv_descent_and_reproducibility(qcnn, ctx):
    Cin, Cout, k, pad, grp, K, d = 64, 96, 3, 1, 2, 32, 8
    W = (np.random.RandomState(51).randn(Cout, Cin // grp, k, k) / 17).astype(np.float32)
    x = cuda(cvr.maps(16, 13, 13, Cin, 52))
    t = conv_targets(x, W, pad, 1, grp, 53)
    tt = tsq(t)
    c0, a0, _ = qcnn.pq_quantize_conv(ctx, W, K, d, iters=5, seed=3)
    c, a, loss = qcnn.pq_refine_conv_target(ctx, x, t, c0, a0, k, pad=pad, grp=grp, sweeps=4)
    assert loss.shape == (5,) and _descends(loss, tt), loss
    want = conv_target_loss(x, t, c, a, k, pad, 1, grp)
    assert abs(loss[-1] - want) <= 1e-10 * (tt + want), (loss[-1], want)
    c2, a2, l2 = qcnn.pq_refine_conv_target(ctx, x, t, c0, a0, k, pad=pad, grp=grp, sweeps=4)
    assert c2.tobytes() == c.tobytes() and a2.tobytes() == a.tobytes() and l2.tobytes() == loss.tobytes()
    cs, as_, _ = qcnn.pq_refine_conv(ctx, W, x, c0, a0, pad=pad, grp=grp, sweeps=4)
    _, _, lt = qcnn.pq_refine_conv_target(ctx, x, t, cs, as_, k, pad=pad, grp=grp, sweeps=3)
    assert abs(lt[0] - conv_target_loss(x, t, cs, as_, k, pad, 1, grp)) <= 1e-10 * tt
    assert _descends(lt, tt), lt


# ---- the paper's claim on the shipped AlexNet -----------------------------------------------------------------------
def _requantized_net(po, qcnn, ctx, params, layer, K, d, W, tmp):
    """The shipped net with `layer` replaced by k-means PQ of its decoded weights W at (K, d)"""
    p = dict(params[layer])
    quant = qcnn.pq_quantize_conv if W.ndim == 4 else qcnn.pq_quantize_fc
    p["ctrd"], p["asmt"], _ = quant(ctx, W, K, d, iters=20, seed=1)
    p["bits"] = po.bits_for(K)
    q = dict(params)
    q[layer] = p
    po.save_model(tmp, po.ALEXNET_PFX, q)
    return qcnn.Net(ctx, tmp, po.ALEXNET_PFX, "AlexNet")


def _inputs(po, net, layer, n_img, batch, seed0):
    """featMapLst[layer] (the layer's input) of the seeded LCG images seed0 .. seed0 + n_img - 1"""
    import torch
    net.set_keep_maps(True)
    xs = []
    for i in range(0, n_img, batch):
        net.forward(torch.from_numpy(po.lcg_images(batch, seed0 + i)).cuda())
        xs.append(net.featmap(layer, batch))
    return torch.cat(xs)


@pytest.mark.gpu
@pytest.mark.parametrize("layer,prev,name", [(18, 15, "fc7"), (4, 0, "conv2")])
def test_shipped_alexnet_target_beats_same_input(layer, prev, name, po, qcnn, ctx):
    """Re-quantize the layer before `layer` (fc6 at K = 16, d = 8; conv1 at K = 32 with its 3 channels in one subspace,
    stored d = 4 wide, which quantizes as d = 3 does: see DESIGN.md 4e), then re-quantize `layer`
    (fc7 at K = 16, d = 8; conv2 at K = 32, d = 8) and refine it on the new net's inputs, same-input and toward the
    original net's responses.  On held-out images the target-refined layer is closer to the original layer's response."""
    import torch
    if not po.have_alexnet():
        pytest.skip("shipped AlexNet parameters not staged under oracle/_ref/data")
    layers = po.alexnet_layers()
    params = po.load_model(po.ALEXNET_DIR, po.ALEXNET_PFX, layers)
    fc = layers[layer]["type"] == po.FCNT
    n_train, n_held, batch = (8192, 1024, 256) if fc else (192, 64, 64)
    seed0 = 900000
    net = qcnn.Net(ctx, po.ALEXNET_DIR, po.ALEXNET_PFX, "AlexNet")
    X = _inputs(po, net, layer, n_train + n_held, batch, seed0)
    net.close()
    if fc:
        Wp, Kp, dp = fcr.decoded(params[prev]["ctrd"], params[prev]["asmt"], 9216).astype(np.float32), 16, 8
        W = fcr.decoded(params[layer]["ctrd"], params[layer]["asmt"], 4096).astype(np.float32)
        K, d = 16, 8
    else:
        Wp, Kp, dp = decode(params[prev], 3).astype(np.float32), 32, 4
        W = decode(params[layer], X.shape[-1] // layers[layer]["grp"]).astype(np.float32)
        K, d = 32, 8
    with tempfile.TemporaryDirectory() as tmp:
        qnet = _requantized_net(po, qcnn, ctx, params, prev, Kp, dp, Wp, tmp)
        Y = _inputs(po, qnet, layer, n_train + n_held, batch, seed0)
        qnet.close()
    if fc:
        X, Y = X.reshape(X.shape[0], -1), Y.reshape(Y.shape[0], -1)
        resp = lambda inp, w: inp.double() @ torch.from_numpy(w).cuda().double().T
        quant, refine = qcnn.pq_quantize_fc, lambda y, c, a: qcnn.pq_refine_fc(ctx, W, y, c, a, sweeps=4)
        refine_t = lambda y, t, c, a: qcnn.pq_refine_fc_target(ctx, y, t, c, a, sweeps=4)
        dec = lambda c, a: fcr.decoded(c, a, 4096)
    else:
        L = layers[layer]
        kw = dict(pad=L["pad"], stride=L["stride"], grp=L["grp"])
        resp = lambda inp, w: conv_fwd(inp, w, L["pad"], L["stride"], L["grp"])
        quant = qcnn.pq_quantize_conv
        refine = lambda y, c, a: qcnn.pq_refine_conv(ctx, W, y, c, a, sweeps=4, **kw)
        refine_t = lambda y, t, c, a: qcnn.pq_refine_conv_target(ctx, y, t, c, a, L["k"], sweeps=4, **kw)
        dec = lambda c, a: decode(dict(ctrd=c, asmt=a), X.shape[-1] // L["grp"])
    T = resp(X, W).float().contiguous()
    y_tr, y_ho = Y[:n_train].contiguous(), Y[n_train:].contiguous()
    t_tr, ref = T[:n_train].contiguous(), T[n_train:].double()
    c0, a0, _ = quant(ctx, W, K, d, iters=20, seed=1)
    cs, as_, ls = refine(y_tr, c0, a0)
    ct, at, lt = refine_t(y_tr, t_tr, c0, a0)
    assert _descends(lt, tsq(t_tr)), lt
    errs = []
    for c, a in ((c0, a0), (cs, as_), (ct, at)):
        out = resp(y_ho, dec(c, a).astype(np.float32))
        errs.append(((out - ref).norm() / ref.norm()).item())
    print("AlexNet %s after re-quantizing the layer before it: held-out relative error against the original layer's "
          "response: k-means %.4f, same-input %.4f, target %.4f (target training loss x%.3f)"
          % (name, errs[0], errs[1], errs[2], lt[-1] / lt[0]))
    assert errs[2] < errs[1]


# ---- errors ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_fc_rejected_inputs(qcnn, ctx):
    import torch
    Din, Dout, K, d = 32, 40, 16, 4
    W, ctrd, asmt = fcr.start(Din, Dout, K, d, 71)
    X = fcr.gaussian_inputs(20, Din, 72)
    T = fc_targets(X, W, 73)
    Xn, Tn, Ti = X.copy(), T.copy(), T.copy()
    Xn[7, 5] = np.nan
    Tn[3, 9] = np.nan
    Ti[19, 39] = -np.inf
    Cn = ctrd.copy()
    Cn[1, 2, 3] = np.nan
    Ak = asmt.copy()
    Ak[5, 2] = K
    _, c48, a48 = fcr.start(Din, Dout, 48, d, 71)
    _, c65, a65 = fcr.start(130, Dout, 16, 65, 71)
    x, t = cuda(X), cuda(T)
    ref = qcnn.pq_refine_fc_target
    bad = [
        (lambda: ref(ctx, x, cuda(Tn), ctrd, asmt, 1), "t contains a non-finite value"),
        (lambda: ref(ctx, x, cuda(Ti), ctrd, asmt, 1), "t contains a non-finite value"),
        (lambda: ref(ctx, cuda(Xn), t, ctrd, asmt, 1), "y contains a non-finite value"),
        (lambda: ref(ctx, x, t, Cn, asmt, 1), "codebook contains a non-finite value"),
        (lambda: ref(ctx, x, t, ctrd, Ak, 1), "not below K=16"),
        (lambda: ref(ctx, x, t, c48, a48, 1), "K=48"),
        (lambda: ref(ctx, cuda(fcr.gaussian_inputs(20, 130, 1)), t, c65, a65, 1), "d=65"),
        (lambda: ref(ctx, x, t, ctrd, asmt, -1), "sweeps=-1"),
        (lambda: ref(ctx, torch.empty((0, Din), dtype=torch.float32, device="cuda"),
                     torch.empty((0, Dout), dtype=torch.float32, device="cuda"), ctrd, asmt, 1), "N=0"),
        (lambda: ref(ctx, x, t[:19].contiguous(), ctrd, asmt, 1), "the same N"),
        (lambda: ref(ctx, x, t[:, :39].contiguous(), ctrd, asmt, 1), "do not match"),
        (lambda: ref(ctx, x[:, :28].contiguous(), t, ctrd, asmt, 1), "do not match"),
        (lambda: ref(ctx, x, t.double(), ctrd, asmt, 1), "contiguous float32 CUDA tensor"),
    ]
    for fn, msg in bad:
        with pytest.raises(qcnn.QcnnError) as e:
            fn()
        assert msg in str(e.value), (msg, str(e.value))
    with pytest.raises(qcnn.QcnnError) as e:   # the C ABI itself, with t = NULL
        qcnn._check(qcnn.lib.qcnn_pq_refine_fc_target(ctx.h, Din, Dout, K, d, 1, qcnn._dptr(x), None, 20,
                                                       ctrd.ctypes.data_as(C.c_void_p), asmt.ctypes.data_as(C.c_void_p),
                                                       None, qcnn._stream(None)))
    assert "NULL t" in str(e.value)


@pytest.mark.gpu
def test_conv_rejected_inputs(qcnn, ctx):
    import torch
    Cin, Cout, k, K, d = 8, 16, 3, 16, 4
    W, ctrd, asmt = cvr.start(Cout, Cin, k, K, d, 71)
    x = cuda(cvr.maps(2, 6, 6, Cin, 72))
    t = conv_targets(x, W, 1, 1, 1, 73)
    xn, tn = x.clone(), t.clone()
    xn[1, 2, 3, 4] = float("nan")
    tn[0, 5, 5, 15] = float("inf")
    Cnan = ctrd.copy()
    Cnan[0, 3, 1] = np.nan
    Ak = asmt.copy()
    Ak[5, 1, 1, 0] = K
    _, c12, a12 = cvr.start(Cout, Cin, k, 12, d, 71)
    _, c65, a65 = cvr.start(Cout, 130, 1, 16, 65, 71)
    _, cb, ab = cvr.start(Cout, 16, k, 256, 16, 71)
    _, cg, ag = cvr.start(15, Cin // 2, k, K, d, 71)
    ref = qcnn.pq_refine_conv_target
    bad = [
        (lambda: ref(ctx, x, tn, ctrd, asmt, k, pad=1, sweeps=1), "t contains a non-finite value"),
        (lambda: ref(ctx, xn, t, ctrd, asmt, k, pad=1, sweeps=1), "y contains a non-finite value"),
        (lambda: ref(ctx, x, t, Cnan, asmt, k, pad=1, sweeps=1), "codebook contains a non-finite value"),
        (lambda: ref(ctx, x, t, ctrd, Ak, k, pad=1, sweeps=1), "not below K=16"),
        (lambda: ref(ctx, x, t, c12, a12, k, pad=1, sweeps=1), "K=12"),
        (lambda: ref(ctx, cuda(cvr.maps(1, 3, 3, 130, 1)), torch.zeros((1, 3, 3, Cout), device="cuda"), c65, a65, 1,
                     sweeps=1), "d=65"),
        (lambda: ref(ctx, x, t, ctrd, asmt, k, pad=1, sweeps=-1), "sweeps=-1"),
        (lambda: ref(ctx, torch.empty((0, 6, 6, Cin), dtype=torch.float32, device="cuda"),
                     torch.empty((0, 6, 6, Cout), dtype=torch.float32, device="cuda"), ctrd, asmt, k, pad=1, sweeps=1),
         "N=0"),
        (lambda: ref(ctx, x, torch.zeros((2, 6, 6, 15), device="cuda"), cg, ag, k, pad=1, grp=2, sweeps=1),
         "divisible by grp=2"),
        (lambda: ref(ctx, cuda(cvr.maps(1, 1, 1, Cin, 1)), torch.zeros((1, 1, 1, Cout), device="cuda"), ctrd, asmt, k,
                     sweeps=1), "empty output"),
        (lambda: ref(ctx, cuda(cvr.maps(2, 6, 6, 16, 1)), t, cb, ab, k, pad=1, sweeps=1), "256*16 = 4096 exceeds 2048"),
        (lambda: ref(ctx, x, t[:1].contiguous(), ctrd, asmt, k, pad=1, sweeps=1), "the same N"),
        (lambda: ref(ctx, x, t, ctrd, asmt, k, pad=0, sweeps=1), "t must be [2, 4, 4, Cout]"),
        (lambda: ref(ctx, x, t[..., :15].contiguous(), ctrd, asmt, k, pad=1, sweeps=1), "do not match"),
        (lambda: ref(ctx, x, t, ctrd, asmt, 1, pad=0, sweeps=1), "do not match"),
    ]
    for fn, msg in bad:
        with pytest.raises(qcnn.QcnnError) as e:
            fn()
        assert msg in str(e.value), (msg, str(e.value))
    with pytest.raises(qcnn.QcnnError) as e:
        qcnn._check(qcnn.lib.qcnn_pq_refine_conv_target(ctx.h, Cin, 6, 6, Cout, k, 1, 1, 1, K, d, 1, qcnn._dptr(x), None, 2,
                                                         ctrd.ctypes.data_as(C.c_void_p), asmt.ctypes.data_as(C.c_void_p),
                                                         None, qcnn._stream(None)))
    assert "NULL t" in str(e.value)
