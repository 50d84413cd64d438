"""Error-correcting product quantization of conv layers on the GPU (qcnn_pq_refine_conv) against a numpy fp64
restatement of one sweep (DESIGN.md 4e): per group the patch Gram G_g, per subspace the joint codebook system
M = sum_g sum_{t,t'} Cnt^g_{tt'} (x) G^m_{g,tt'} solved by Cholesky and kept only if it lowers f, then the tap-ordered
assignment argmin_k c_k^T G_tt c_k - 2 c_k^T h'_{o,t}."""
import ctypes as C
import re

import numpy as np
import pytest

from test_gpu_pq_quantize import decode, dists, ulps


# ---- the restatement ----------------------------------------------------------------------------------------------
def dim_order(Cg, d, T):
    """original flat index c T + t of every internal dim q = m d T + t w_m + j"""
    out = []
    for m in range(-(-Cg // d)):
        w = min(d, Cg - m * d)
        for t in range(T):
            for j in range(w):
                out.append((m * d + j) * T + t)
    return np.array(out)


def out_size(n, k, pad, stride):
    return (n + 2 * pad - k) // stride + 1


def patches(X, g, Cg, k, pad, stride):
    """[N Ho Wo][Cg k k] fp64 patches of group g's channels (original order c, kh, kw), zero-padded"""
    N, H, W, _ = X.shape
    Ho, Wo = out_size(H, k, pad, stride), out_size(W, k, pad, stride)
    Xp = np.zeros((N, H + 2 * pad, W + 2 * pad, Cg))
    Xp[:, pad:pad + H, pad:pad + W] = X[..., g * Cg:(g + 1) * Cg]
    P = np.empty((N, Ho, Wo, Cg, k, k))
    for kh in range(k):
        for kw in range(k):
            P[..., kh, kw] = Xp[:, kh:kh + stride * (Ho - 1) + 1:stride, kw:kw + stride * (Wo - 1) + 1:stride]
    return P.reshape(N * Ho * Wo, Cg * k * k)


def grams(X, Cg, k, pad, stride, grp, d):
    """per group the fp64 patch Gram G_g in the internal dim order, from numpy patches"""
    perm = dim_order(Cg, d, k * k)
    G = []
    for g in range(grp):
        P = patches(X.astype(np.float64), g, Cg, k, pad, stride)[:, perm]
        G.append(P.T @ P)
    return G


def grams_torch(x, Cg, k, pad, stride, grp, d, batch):
    """The same from maps x [N][H][W][Cin] on the GPU: fp64 F.unfold over `batch` images at a time, accumulated.  For
    layers whose fp64 patches are too large to build in numpy; it sums in another order than the device, so the two
    differ in the last bits, which the restatement's margins absorb."""
    import torch
    import torch.nn.functional as F
    Dg = Cg * k * k
    perm = torch.from_numpy(dim_order(Cg, d, k * k)).to(x.device)
    G = [torch.zeros((Dg, Dg), dtype=torch.float64, device=x.device) for _ in range(grp)]
    for i in range(0, x.shape[0], batch):
        xb = x[i:i + batch].permute(0, 3, 1, 2).double()
        for g in range(grp):
            P = F.unfold(xb[:, g * Cg:(g + 1) * Cg], k, padding=pad, stride=stride)   # [n][Cg k k][positions]
            P = P.permute(0, 2, 1).reshape(-1, Dg)[:, perm]
            G[g] += P.T @ P
    return [Gg.cpu().numpy() for Gg in G]


def system_sizes(Cg, d, T, asmt):
    """n = |U| w_m of every subspace's joint codebook system in the first sweep (U: the start's used clusters)"""
    S = -(-Cg // d)
    A = asmt.reshape(-1, T, S)
    return [len(np.unique(A[:, :, m])) * min(d, Cg - m * d) for m in range(S)]


def sweep_ref(W, G, ctrd, asmt, grp, sweeps, follow=None):
    """(ctrd, asmt, stats) after `sweeps` sweeps from the Grams G (grams / grams_torch).  A decision is exact outside its
    margin: an argmin whose best and second best differ by more than 1e-6 of the terms' scale, an accept-or-keep
    decision with D != C and |f(D) - f(C)| above 1e-9 of the terms' scale.  A decision inside its margin needs
    `follow`, the device's (ctrd, asmt) after one sweep, in which every codebook and assignment is decided once: the
    device's choice must be one of the options inside the margin (an index within the gap, a codebook within 1 ulp of
    D or of C), and the restatement continues with it.  stats: "inside" counts those decisions, "n" lists the size
    |U| w_m of every subspace's system."""
    assert follow is None or sweeps == 1
    Cout, Cg, k, _ = W.shape
    T = k * k
    S, K, d = ctrd.shape
    Cpg, Dg = Cout // grp, Cg * T
    perm = dim_order(Cg, d, T)
    Wq = W.reshape(Cout, Dg)[:, perm].astype(np.float64)
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
            E = Wq - Wh
            h = np.empty((Cout, nb))
            for g in range(grp):
                og = grp_of == g
                h[og] = E[og] @ G[g][:, blk] + Wh[og][:, blk] @ G[g][blk, blk]
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
                ug = uidx[Am[grp_of == g]]            # [Cpg][T]
                for t in range(T):
                    key = (np.arange(T)[None, :] * nU + ug[:, t:t + 1]) * nU + ug   # (t', u, u') for every (o, t')
                    keys, cnt = np.unique(key.ravel(), return_counts=True)        # ascending t'
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
            # assignment, taps in order, E current
            E = Wq - decoded()
            Cm = ctrd[m, :, :w].astype(np.float64)
            for o in range(Cout):
                Gg = G[grp_of[o]]
                for t in range(T):
                    r = slice(q0 + t * w, q0 + (t + 1) * w)
                    Gtt = Gg[r, r]
                    if np.trace(Gtt) == 0:
                        continue
                    hp = Gg[r, :] @ E[o] + Gtt @ (Wq[o, r] - E[o, r])
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
                    E[o, r] = Wq[o, r] - Cm[a]
    return ctrd, asmt, stats


def refine_ref(W, X, ctrd, asmt, pad, stride, grp, sweeps, follow=None):
    """sweep_ref from the numpy Grams of the maps X"""
    S, K, d = ctrd.shape
    return sweep_ref(W, grams(X, W.shape[1], W.shape[2], pad, stride, grp, d), ctrd, asmt, grp, sweeps, follow)


def response_loss(W, X, ctrd, asmt, pad, stride, grp):
    """sum conv(x, W - W^)^2 from the maps themselves (torch, fp64; on the GPU when X is a CUDA tensor, else the CPU)"""
    import torch
    import torch.nn.functional as F
    dW = torch.from_numpy(W.astype(np.float64) - decode(dict(ctrd=ctrd, asmt=asmt), W.shape[1]))
    if isinstance(X, torch.Tensor):
        x, dW = X.double().permute(0, 3, 1, 2), dW.to(X.device)
    else:
        x = torch.from_numpy(np.ascontiguousarray(X, np.float64)).permute(0, 3, 1, 2)
    y = F.conv2d(x, dW, stride=stride, padding=pad, groups=grp)
    return float((y * y).sum())


def start(Cout, Cg, k, K, d, seed):
    """dense weights and a starting point: codewords drawn from the weights' sub-vectors, random assignments"""
    rng = np.random.RandomState(seed)
    W = (rng.randn(Cout, Cg, k, k) / np.sqrt(Cg * k * k)).astype(np.float32)
    S = -(-Cg // d)
    Wp = np.zeros((Cout, k, k, S * d), np.float32)
    Wp[..., :Cg] = W.transpose(0, 2, 3, 1)
    pts = Wp.reshape(-1, S, d)
    ctrd = pts[rng.randint(0, len(pts), size=(S, K)), np.arange(S)[:, None]]
    ctrd = (ctrd + 0.1 * rng.randn(S, K, d) / np.sqrt(Cg * k * k)).astype(np.float32)
    for m in range(S):
        ctrd[m, :, min(d, Cg - m * d):] = 0
    asmt = rng.randint(0, K, size=(Cout, k, k, S)).astype(np.uint8)
    return W, ctrd, asmt


def maps(N, H, W, C, seed):
    return np.random.RandomState(seed).randn(N, H, W, C).astype(np.float32)


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


# ---- CPU ----------------------------------------------------------------------------------------------------------
def test_refine_conv_symbol_declared_and_exported(qcnn):
    text = open(qcnn.HEADER_PATH).read()
    assert re.search(r"QCNN_API\s+int\s+qcnn_pq_refine_conv\s*\(", text)
    assert hasattr(C.CDLL(qcnn.LIB_PATH), "qcnn_pq_refine_conv")
    assert "qcnn_pq_refine_conv" in qcnn.EXPORTS


# ---- sweeps = 0: the starting point and its loss -------------------------------------------------------------------
# (name, Cin, H, Cout, k, pad, stride, grp, K, d, N)
ZERO_SWEEP = [
    ("1x1", 20, 6, 24, 1, 0, 1, 1, 16, 4, 3),
    ("3x3_grp2", 20, 7, 32, 3, 1, 1, 2, 16, 4, 2),       # Cg = 10: subspaces of 4, 4, 2
    ("11x11_s4", 3, 31, 16, 11, 0, 4, 1, 32, 8, 2),
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,Cin,H,Cout,k,pad,stride,grp,K,d,N", ZERO_SWEEP, ids=[c[0] for c in ZERO_SWEEP])
def test_zero_sweeps_return_the_start_and_its_loss(name, Cin, H, Cout, k, pad, stride, grp, K, d, N, qcnn, ctx):
    W, ctrd, asmt = start(Cout, Cin // grp, k, K, d, 11)
    X = maps(N, H, H, Cin, 12)
    c, a, loss = qcnn.pq_refine_conv(ctx, W, cuda(X), ctrd, asmt, pad=pad, stride=stride, grp=grp, sweeps=0)
    assert c.tobytes() == ctrd.tobytes() and a.tobytes() == asmt.tobytes()
    assert loss.shape == (1,)
    want = response_loss(W, X, ctrd, asmt, pad, stride, grp)
    assert abs(loss[0] - want) <= 1e-10 * want, (loss[0], want)


@pytest.mark.gpu
def test_zero_input_channels_skip_their_subspaces(qcnn, ctx):
    Cin, Cout, k, K, d = 16, 24, 3, 16, 4
    W, ctrd, asmt = start(Cout, Cin, k, K, d, 13)
    X = maps(2, 8, 8, Cin, 14)
    X[..., 4:12] = 0   # subspaces 1 and 2 see no input
    c, a, loss = qcnn.pq_refine_conv(ctx, W, cuda(X), ctrd, asmt, pad=1, sweeps=1)
    assert np.array_equal(c[1:3], ctrd[1:3]) and np.array_equal(a[..., 1:3], asmt[..., 1:3])
    assert not np.array_equal(a[..., 0], asmt[..., 0])
    assert loss[1] <= loss[0]


# ---- one sweep against the restatement -----------------------------------------------------------------------------
PATCH_BYTES = 256 << 20   # one chunk of one group's fp32 patches (pq_refine_conv.cu)


def patch_chunks(N, H, k, pad, stride, Cg):
    """chunks of output positions the device's Gram of one group is accumulated over"""
    positions, Dg = N * out_size(H, k, pad, stride) ** 2, Cg * k * k
    return -(-positions // max(1, min(positions, PATCH_BYTES // (4 * Dg))))


# (name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed).  The chunked rows' patches span several chunks per group,
# the last partial; their Grams come from grams_torch, since fp64 numpy patches that large do not fit.
ONE_SWEEP = [
    ("1x1", 24, 6, 48, 1, 0, 1, 1, 16, 8, 4, 21),
    ("3x3_grp2_partial", 20, 9, 32, 3, 1, 1, 2, 16, 4, 3, 21),   # Cg = 10, d = 4
    ("5x5_s2_p2", 12, 11, 24, 5, 2, 2, 1, 32, 4, 4, 21),
    ("conv1_like", 3, 63, 32, 11, 0, 4, 1, 128, 8, 6, 21),        # w = 3, K = 128
    ("kw_2048", 8, 6, 160, 3, 1, 1, 1, 256, 8, 6, 21),            # K w = 2048
    ("chunked_conv1", 3, 227, 96, 11, 0, 4, 1, 128, 8, 128, 21),  # AlexNet conv1: 387 200 positions, 184 872 a chunk
    ("chunked_grp2", 464, 32, 32, 3, 1, 1, 2, 16, 8, 100, 21),    # Dg = 2088: 102 400 positions, 32 140 a chunk
]


def test_rows_cover_chunks_and_cholesky_panels():
    """Every row's first-sweep system sizes n = |U| w_m (from the start alone: subspace m's assignments are still the
    start's when its codebook is solved) reach a single panel (n < 64), whole panels, a partial last panel and more
    than 16 panels; the chunked rows reach three and four patch chunks per group."""
    ns, chunked = [], set()
    for name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed in ONE_SWEEP:
        _, _, asmt = start(Cout, Cin // grp, k, K, d, seed)
        n = system_sizes(Cin // grp, d, k * k, asmt)
        chunks = patch_chunks(N, H, k, pad, stride, Cin // grp)
        print("%s: %d patch chunks per group, systems n = %s" % (name, chunks, n))
        assert (chunks >= 3) == name.startswith("chunked"), name
        if chunks > 1:
            chunked.add(chunks)
        ns += n
    assert chunked == {3, 4}, chunked
    assert min(ns) < 64, ns
    assert any(n % 64 == 0 for n in ns), ns
    assert any(n > 64 and n % 64 for n in ns), ns
    assert max(ns) > 1024, ns


@pytest.mark.gpu
@pytest.mark.parametrize("name,Cin,H,Cout,k,pad,stride,grp,K,d,N,seed", ONE_SWEEP, ids=[c[0] for c in ONE_SWEEP])
def test_one_sweep_matches_restatement(name, Cin, H, Cout, k, pad, stride, grp, K, d, N, seed, qcnn, ctx):
    Cg = Cin // grp
    W, ctrd, asmt = start(Cout, Cg, k, K, d, seed)
    X = maps(N, H, H, Cin, seed + 1)
    x = cuda(X)
    chunked = patch_chunks(N, H, k, pad, stride, Cg) > 1
    if chunked:   # the chunked Gram alone, against the response loss
        c0, a0, l0 = qcnn.pq_refine_conv(ctx, W, x, ctrd, asmt, pad=pad, stride=stride, grp=grp, sweeps=0)
        assert c0.tobytes() == ctrd.tobytes() and a0.tobytes() == asmt.tobytes()
        want = response_loss(W, x, ctrd, asmt, pad, stride, grp)
        assert abs(l0[0] - want) <= 1e-10 * want, (l0[0], want)
        G = grams_torch(x, Cg, k, pad, stride, grp, d, batch=max(1, (64 << 20) // (8 * Cg * k * k * out_size(H, k, pad, stride) ** 2)))
    else:
        G = grams(X, Cg, k, pad, stride, grp, d)
    c, a, loss = qcnn.pq_refine_conv(ctx, W, x, ctrd, asmt, pad=pad, stride=stride, grp=grp, sweeps=1)
    want_c, want_a, stats = sweep_ref(W, G, ctrd, asmt, grp, 1, follow=(c, a))
    print("%s: systems n = %s, %d of %d decisions inside their margins"
          % (name, stats["n"], stats["inside"], a.size + len(stats["n"])))
    assert stats["n"] == system_sizes(Cg, d, k * k, asmt)
    assert ulps(c, want_c).max() <= 1.0
    assert np.array_equal(a, want_a)
    assert loss[1] <= loss[0]


@pytest.mark.gpu
def test_every_sweeps_loss(qcnn, ctx):
    Cin, H, Cout, k, pad, stride, grp, K, d, N = 20, 9, 32, 3, 1, 1, 2, 16, 4, 3
    W, ctrd, asmt = start(Cout, Cin // grp, k, K, d, 24)
    X = maps(N, H, H, Cin, 25)
    x = cuda(X)
    prev = np.zeros(0)
    for sweeps in (1, 2, 3):
        c, a, loss = qcnn.pq_refine_conv(ctx, W, x, ctrd, asmt, pad=pad, stride=stride, grp=grp, sweeps=sweeps)
        assert loss.shape == (sweeps + 1,)
        assert loss[:len(prev)].tobytes() == prev.tobytes(), (sweeps, loss, prev)
        want = response_loss(W, X, c, a, pad, stride, grp)
        assert abs(loss[-1] - want) <= 1e-9 * want, (sweeps, loss[-1], want)
        prev = loss


def unit_patch_maps(Cg, k, grp):
    """stride = k, pad = 0: the non-overlapping patches are the unit vectors, in every group's channels at once"""
    Dg = Cg * k * k
    side = int(np.ceil(np.sqrt(Dg)))
    X = np.zeros((1, side * k, side * k, Cg * grp), np.float32)
    for i in range(Dg):
        c, t = divmod(i, k * k)
        y, x = divmod(i, side)
        for g in range(grp):
            X[0, y * k + t // k, x * k + t % k, g * Cg + c] = 1
    return X


@pytest.mark.gpu
def test_identity_gram_gives_one_kmeans_iteration(qcnn, ctx):
    Cg, k, grp, Cout, K, d = 6, 2, 2, 80, 16, 4
    W, C0, _ = start(Cout, Cg, k, K, d, 31)
    _, a0, _ = qcnn.pq_quantize_conv(ctx, W, K, d, iters=0, init=C0)
    C1, a1, _ = qcnn.pq_quantize_conv(ctx, W, K, d, iters=1, init=C0)
    c, a, _ = qcnn.pq_refine_conv(ctx, W, cuda(unit_patch_maps(Cg, k, grp)), C0, a0, stride=k, grp=grp, sweeps=1)
    assert ulps(c, C1).max() <= 1.0
    for m in range(-(-Cg // d)):
        x = np.ascontiguousarray(W[:, m * d:(m + 1) * d].transpose(0, 2, 3, 1).reshape(-1, min(d, Cg - m * d)))
        dist = dists(x, C1[m][:, :x.shape[1]]).astype(np.float64)
        am, a1m = a[..., m].ravel(), a1[..., m].ravel()
        for p in np.nonzero(am != a1m)[0]:
            d1, d2 = dist[p, am[p]], dist[p, a1m[p]]
            assert abs(d1 - d2) <= 1e-5 * max(d1, d2), (m, p, d1, d2)


@pytest.mark.gpu
def test_exact_weights_are_a_fixed_point(qcnn, ctx):
    Cin, Cout, k, grp, K, d = 20, 32, 3, 2, 16, 4
    _, Cs, As = start(Cout, Cin // grp, k, K, d, 41)
    Cs[1, 7] = Cs[1, 2]   # two equal codewords: the lower index may take the other's outputs
    W = decode(dict(ctrd=Cs, asmt=As), Cin // grp).astype(np.float32)
    X = maps(3, 9, 9, Cin, 42)
    c, a, loss = qcnn.pq_refine_conv(ctx, W, cuda(X), Cs, As, pad=1, grp=grp, sweeps=3)
    assert c.tobytes() == Cs.tobytes()
    assert (loss == 0).all(), loss
    differ = a != As
    if differ.any():
        m_idx = np.nonzero(differ)[3]
        assert np.array_equal(c[m_idx, a[differ]], c[m_idx, As[differ]])
        assert (a[differ] < As[differ]).all()


@pytest.mark.gpu
def test_descent_and_reproducibility(qcnn, ctx):
    Cin, Cout, k, grp, K, d = 64, 96, 3, 2, 32, 8
    W = (np.random.RandomState(51).randn(Cout, Cin // grp, k, k) / 17).astype(np.float32)
    X = maps(16, 13, 13, Cin, 52)
    c0, a0, _ = qcnn.pq_quantize_conv(ctx, W, K, d, iters=5, seed=3)
    x = cuda(X)
    c, a, loss = qcnn.pq_refine_conv(ctx, W, x, c0, a0, pad=1, grp=grp, sweeps=4)
    assert loss.shape == (5,)
    assert (loss[1:] <= loss[:-1] * (1 + 1e-12)).all(), loss
    assert loss[-1] < loss[0]
    want = response_loss(W, X, c, a, 1, 1, grp)
    assert abs(loss[-1] - want) <= 1e-9 * want, (loss[-1], want)
    c2, a2, l2 = qcnn.pq_refine_conv(ctx, W, x, c0, a0, pad=1, grp=grp, sweeps=4)
    assert c2.tobytes() == c.tobytes() and a2.tobytes() == a.tobytes() and l2.tobytes() == loss.tobytes()


def correlated_maps(N, H, C, seed):
    """Gaussian maps with channel covariance spectrum exp(-i / (C / 8)) in a random basis, smoothed over 3x3 pixels"""
    rng = np.random.RandomState(seed)
    Q, _ = np.linalg.qr(rng.randn(C, C))
    s = np.exp(-np.arange(C) / (C / 8.0)) ** 0.5
    X = (rng.randn(N, H + 2, H + 2, C) * s) @ Q.T
    X = sum(X[:, dy:dy + H, dx:dx + H] for dy in range(3) for dx in range(3)) / 3.0
    return X.astype(np.float32)


@pytest.mark.gpu
def test_corrects_error_on_unseen_maps(qcnn, ctx):
    Cin, Cout, k, K, d = 64, 128, 3, 32, 8
    W = (np.random.RandomState(61).randn(Cout, Cin, k, k) / 24).astype(np.float32)
    X = correlated_maps(64, 12, Cin, 62)
    train, held = X[:32], X[32:]
    c0, a0, _ = qcnn.pq_quantize_conv(ctx, W, K, d, iters=20, seed=7)
    c, a, loss = qcnn.pq_refine_conv(ctx, W, cuda(train), c0, a0, pad=1, sweeps=8)
    assert (loss[1:] <= loss[:-1] * (1 + 1e-12)).all(), loss
    held0, held1 = response_loss(W, held, c0, a0, 1, 1, 1), response_loss(W, held, c, a, 1, 1, 1)
    print("training loss %.4g -> %.4g (x%.3f), held-out error %.4g -> %.4g (x%.3f)"
          % (loss[0], loss[-1], loss[-1] / loss[0], held0, held1, held1 / held0))
    assert loss[-1] <= 0.5 * loss[0]
    assert held1 <= 0.5 * held0


# ---- shipped AlexNet conv2 / conv4 ----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("layer,name", [(4, "conv2"), (10, "conv4")])
def test_shipped_alexnet_conv_on_its_own_inputs(layer, name, po, qcnn, ctx):
    import torch
    import torch.nn.functional as F
    if not po.have_alexnet():
        pytest.skip("shipped AlexNet parameters not staged under oracle/_ref/data")
    layers = po.alexnet_layers()
    L = layers[layer]
    params = po.load_model(po.ALEXNET_DIR, po.ALEXNET_PFX, layers)
    p = params[layer]
    net = qcnn.Net(ctx, po.ALEXNET_DIR, po.ALEXNET_PFX, "AlexNet")
    net.set_keep_maps(True)
    xs = []
    for i in range(4):
        net.forward(torch.from_numpy(po.lcg_images(64, 800000 + 64 * i)).cuda())
        xs.append(net.featmap(layer, 64).clone())
    net.close()
    X = torch.cat(xs)
    train, held = X[:192].contiguous(), X[192:].contiguous()
    N, H, Wd, Cin = X.shape
    grp, k, pad, stride = L["grp"], L["k"], L["pad"], L["stride"]
    W = decode(p, Cin // grp).astype(np.float32)
    Cout = W.shape[0]
    c0, a0, _ = qcnn.pq_quantize_conv(ctx, W, 32, 8, iters=20, seed=1)
    c, a, loss = qcnn.pq_refine_conv(ctx, W, train, c0, a0, pad=pad, stride=stride, grp=grp, sweeps=4)
    assert (loss[1:] <= loss[:-1] * (1 + 1e-12)).all(), loss
    ref = F.conv2d(held.double().permute(0, 3, 1, 2), torch.from_numpy(W).cuda().double(), stride=stride, padding=pad,
                   groups=grp) + torch.from_numpy(p["bias"]).cuda().double()[None, :, None, None]
    ref = ref.permute(0, 2, 3, 1)
    errs = []
    for cc, aa in ((c0, a0), (c, a)):
        lay = qcnn.ConvLayer(ctx, Cin, H, Wd, Cout, k, pad, stride, grp, cc, aa, p["bias"])
        lay.set_param("tensor_core", 0)
        y = lay.forward(held)
        errs.append(((y.double() - ref).norm() / ref.norm()).item())
        lay.close()
    print("AlexNet %s re-quantized at K=32, d=8: held-out relative output error k-means %.4f, refined %.4f "
          "(training loss x%.3f)" % (name, errs[0], errs[1], loss[-1] / loss[0]))
    assert errs[1] < errs[0]


# ---- errors -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rejected_inputs(qcnn, ctx):
    import torch
    Cin, Cout, k, K, d = 8, 16, 3, 16, 4
    W, ctrd, asmt = start(Cout, Cin, k, K, d, 71)
    X = maps(2, 6, 6, Cin, 72)
    Xn = X.copy()
    Xn[1, 2, 3, 4] = np.nan
    Winf = W.copy()
    Winf[3, 1, 0, 0] = np.inf
    Cnan = ctrd.copy()
    Cnan[0, 3, 1] = np.nan
    Ak = asmt.copy()
    Ak[5, 1, 1, 0] = K
    _, c12, a12 = start(Cout, Cin, k, 12, d, 71)
    W65, c65, a65 = start(Cout, 130, 1, 16, 65, 71)
    Wb, cb, ab = start(Cout, 16, k, 256, 16, 71)
    Wg, cg, ag = start(15, Cin // 2, k, K, d, 71)
    ref = qcnn.pq_refine_conv
    bad = [
        (lambda: ref(ctx, W, cuda(Xn), ctrd, asmt, pad=1, sweeps=1), "non-finite"),
        (lambda: ref(ctx, Winf, cuda(X), ctrd, asmt, pad=1, sweeps=1), "non-finite"),
        (lambda: ref(ctx, W, cuda(X), Cnan, asmt, pad=1, sweeps=1), "non-finite"),
        (lambda: ref(ctx, W, cuda(X), ctrd, Ak, pad=1, sweeps=1), "not below K=16"),
        (lambda: ref(ctx, W, cuda(X), c12, a12, pad=1, sweeps=1), "K=12"),
        (lambda: ref(ctx, W65, cuda(maps(1, 3, 3, 130, 1)), c65, a65, sweeps=1), "d=65"),
        (lambda: ref(ctx, W, cuda(X), ctrd, asmt, pad=1, sweeps=-1), "sweeps=-1"),
        (lambda: ref(ctx, W, torch.empty((0, 6, 6, Cin), dtype=torch.float32, device="cuda"), ctrd, asmt, pad=1,
                     sweeps=1), "N=0"),
        (lambda: ref(ctx, Wg, cuda(X), cg, ag, pad=1, grp=2, sweeps=1), "divisible by grp=2"),
        (lambda: ref(ctx, W, cuda(maps(1, 1, 1, Cin, 1)), ctrd, asmt, sweeps=1), "empty output"),
        (lambda: ref(ctx, Wb, cuda(maps(2, 6, 6, 16, 1)), cb, ab, pad=1, sweeps=1), "256*16 = 4096 exceeds 2048"),
    ]
    for fn, msg in bad:
        with pytest.raises(qcnn.QcnnError) as e:
            fn()
        assert msg in str(e.value), (msg, str(e.value))
