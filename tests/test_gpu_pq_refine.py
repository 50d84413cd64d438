"""Error-correcting product quantization of FC layers on the GPU (qcnn_pq_refine_fc) against a numpy fp64 restatement
of one sweep (DESIGN.md 4e): Gram G = X^T X, h_o = [G E_o]_m + G_mm w^_o, per cluster a ridge Cholesky solve rounded to
fp32 and kept only if it lowers f, then the assignment argmin_k c_k^T G_mm c_k - 2 c_k^T h_o, subspace by subspace."""
import ctypes as C
import re

import numpy as np
import pytest

from test_gpu_pq_quantize import decode, dists, ulps


# ---- the restatement ----------------------------------------------------------------------------------------------
def decoded(ctrd, asmt, Din):
    return decode(dict(ctrd=ctrd, asmt=asmt), Din)


def follow_argmin(v, two, margin, m, follow):
    """Per row of v the argmin, except that a row whose best and second best differ by at most `margin` takes the
    device's index follow[1][:, m], which must lie within `margin` of the best.  Returns (indices, rows inside)."""
    a = np.argmin(v, axis=1)
    inside = (two[:, 1] - two[:, 0]) <= margin
    if inside.any():
        assert follow is not None, ("argmin inside its margin", m, np.nonzero(inside)[0])
        ad = follow[1][inside, m].astype(np.int64)
        assert (v[inside, ad] - two[inside, 0] <= margin[inside]).all(), m
        a[inside] = ad
    return a, int(inside.sum())


def refine_ref(W, X, ctrd, asmt, sweeps, follow=None):
    """(ctrd, asmt, inside) after `sweeps` sweeps.  A decision is exact outside its margin: an argmin whose best and
    second best differ by more than 1e-6 of the terms' scale, an accept-or-keep decision of the codebook step with
    D != c_k and |f(D) - f(c_k)| above 1e-9 of the terms' scale.  A decision inside its margin needs `follow`, the
    device's (ctrd, asmt) after one sweep, in which every codeword and assignment is decided once: the device's choice
    must be one of the options inside the margin (an index within the gap, a codeword within 1 ulp of D or of c_k), and
    the restatement continues with it.  `inside` counts those decisions."""
    assert follow is None or sweeps == 1
    X = X.astype(np.float64)
    G = X.T @ X
    Dout, Din = W.shape
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
            E = W.astype(np.float64) - decoded(ctrd, asmt, Din)
            h = E @ G[:, sl] + ctrd[m, asmt[:, m], :w].astype(np.float64) @ Gmm
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
            asmt[:, m], n_in = follow_argmin(v, two, 1e-6 * scale, m, follow)
            inside += n_in
    return ctrd, asmt, inside


def response_loss(W, X, ctrd, asmt):
    """sum_n |(W - W^) x_n|^2 from the inputs themselves (not from G)"""
    R = X.astype(np.float64) @ (W.astype(np.float64) - decoded(ctrd, asmt, W.shape[1])).T
    return float((R * R).sum())


def start(Din, Dout, K, d, seed):
    """dense weights and a starting point: codewords drawn from the weights' sub-vectors, random assignments"""
    rng = np.random.RandomState(seed)
    W = (rng.randn(Dout, Din) / np.sqrt(Din)).astype(np.float32)
    S = -(-Din // d)
    Wp = np.zeros((Dout, S * d), np.float32)
    Wp[:, :Din] = W
    ctrd = Wp.reshape(Dout, S, d)[rng.randint(0, Dout, size=(S, K)), np.arange(S)[:, None]]
    ctrd = (ctrd + 0.1 * rng.randn(S, K, d) / np.sqrt(Din)).astype(np.float32)
    for m in range(S):
        ctrd[m, :, min(d, Din - m * d):] = 0
    asmt = rng.randint(0, K, size=(Dout, S)).astype(np.uint8)
    return W, ctrd, asmt


def gaussian_inputs(N, Din, seed):
    return np.random.RandomState(seed).randn(N, Din).astype(np.float32)


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


# ---- CPU ----------------------------------------------------------------------------------------------------------
def test_refine_symbol_declared_and_exported(qcnn):
    text = open(qcnn.HEADER_PATH).read()
    assert re.search(r"QCNN_API\s+int\s+qcnn_pq_refine_fc\s*\(", text)
    assert hasattr(C.CDLL(qcnn.LIB_PATH), "qcnn_pq_refine_fc")
    assert "qcnn_pq_refine_fc" in qcnn.EXPORTS


# ---- sweeps = 0: the starting point and its loss -------------------------------------------------------------------
# (name, Din, Dout, K, d, N, first zero input column, zero input columns)
ZERO_SWEEP = [
    ("d1", 40, 300, 16, 1, 64, 20, 0),
    ("d4_partial", 30, 200, 32, 4, 50, 20, 0),        # Din % d = 2
    ("d64_k256", 100, 64, 256, 64, 120, 20, 0),       # subspaces of 64 and 36 dims
    ("n1", 48, 32, 16, 4, 1, 20, 0),
    ("singular", 96, 64, 32, 4, 40, 20, 10),          # N < Din, ten zero columns: G_mm singular, whole subspaces skipped
    ("singular_block2", 700, 301, 32, 4, 200, 300, 41),   # skipped subspaces 75..84 in the second block of 64
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,Din,Dout,K,d,N,z0,zeros", ZERO_SWEEP, ids=[c[0] for c in ZERO_SWEEP])
def test_zero_sweeps_return_the_start_and_its_loss(name, Din, Dout, K, d, N, z0, zeros, qcnn, ctx):
    W, ctrd, asmt = start(Din, Dout, K, d, 11)
    X = gaussian_inputs(N, Din, 12)
    X[:, z0:z0 + zeros] = 0
    c, a, loss = qcnn.pq_refine_fc(ctx, W, cuda(X), ctrd, asmt, sweeps=0)
    assert c.tobytes() == ctrd.tobytes() and a.tobytes() == asmt.tobytes()
    assert loss.shape == (1,)
    want = response_loss(W, X, ctrd, asmt)
    assert abs(loss[0] - want) <= 1e-10 * want, (loss[0], want)
    if zeros:   # a skipped subspace keeps everything even in a sweep, and the others still lower the loss
        c1, a1, l1 = qcnn.pq_refine_fc(ctx, W, cuda(X), ctrd, asmt, sweeps=1)
        skipped = [m for m in range(-(-Din // d)) if z0 <= m * d and (m + 1) * d <= z0 + zeros]
        assert skipped
        assert np.array_equal(c1[skipped], ctrd[skipped]) and np.array_equal(a1[:, skipped], asmt[:, skipped])
        want = response_loss(W, X, c1, a1)
        assert abs(l1[1] - want) <= 1e-9 * want, (l1[1], want)
        assert l1[1] <= l1[0]


# ---- one sweep against the restatement -----------------------------------------------------------------------------
BLOCK_DIMS = 256   # dims per cooperative launch of the sweep: floor(256 / d) subspaces (pq_refine.cu)


def blocks(Din, d):
    """subspaces per block of one sweep"""
    S, spb = -(-Din // d), max(1, BLOCK_DIMS // d)
    return [min(spb, S - m0) for m0 in range(0, S, spb)]


# (name, Din, Dout, K, d, seed).  The block rows span three blocks with a partial last one.  With the sweep kernel's grid
# of min(2 x SMs, max(Dout, K)) CTAs (264 on 132 SMs, 228 on 114), Dout = 701 gives each CTA several outputs and the
# last CTA with outputs a partial range, and Dout = 200 < K = 256 leaves CTAs without outputs.
ONE_SWEEP = [
    ("d1", 24, 300, 16, 1, 22),
    ("d4_partial", 250, 200, 32, 4, 21),
    ("d8_k64", 256, 256, 64, 8, 21),
    ("d64_k256", 160, 128, 256, 64, 21),
    ("d4_blocks", 610, 701, 32, 4, 23),        # 64 + 64 + 25 subspaces, the last of 2 dims
    ("d12_blocks", 610, 701, 32, 12, 23),      # 21 + 21 + 9 subspaces (252 dims a block: the trailing GEMM's K % 16 = 12)
    ("d1_blocks", 600, 701, 32, 1, 23),        # 256 + 256 + 88 subspaces
    ("d64_blocks", 600, 200, 256, 64, 23),     # 4 + 4 + 2 subspaces, the last of 24 dims; Dout < K
]


def test_block_rows_cross_blocks():
    """Two sweep CTAs fit on an SM at every row's shared memory, so the grid is min(2 x SMs, max(Dout, K))."""
    for name, Din, Dout, K, d, seed in ONE_SWEEP:
        b = blocks(Din, d)
        print("%s: blocks of %s subspaces, the last subspace %d dims" % (name, b, Din - (-(-Din // d) - 1) * d))
        if name.endswith("_blocks"):
            assert len(b) >= 3 and b[-1] < b[0], name
            assert d == 1 or Din % d, name
            for sm in (132, 114):
                grid = min(2 * sm, max(Dout, K))
                R = -(-Dout // grid)
                assert grid > Dout if Dout < K else (R >= 2 and Dout % R), (name, sm)
    assert {tuple(blocks(Din, d)) for _, Din, _, _, d, _ in ONE_SWEEP} >= {(64, 64, 25), (21, 21, 9), (256, 256, 88), (4, 4, 2)}


@pytest.mark.gpu
@pytest.mark.parametrize("name,Din,Dout,K,d,seed", ONE_SWEEP, ids=[c[0] for c in ONE_SWEEP])
def test_one_sweep_matches_restatement(name, Din, Dout, K, d, seed, qcnn, ctx):
    W, ctrd, asmt = start(Din, Dout, K, d, seed)
    X = gaussian_inputs(2 * Din, Din, seed + 1)
    c, a, loss = qcnn.pq_refine_fc(ctx, W, cuda(X), ctrd, asmt, sweeps=1)
    want_c, want_a, inside = refine_ref(W, X, ctrd, asmt, 1, follow=(c, a))
    print("%s: %d blocks, %d of %d assignments and codewords decided inside their margins"
          % (name, len(blocks(Din, d)), inside, a.size + ctrd.shape[0] * K))
    assert ulps(c, want_c).max() <= 1.0
    assert np.array_equal(a, want_a)
    assert loss[1] <= loss[0]
    want = response_loss(W, X, c, a)
    assert abs(loss[1] - want) <= 1e-9 * want, (loss[1], want)


@pytest.mark.gpu
def test_every_sweeps_loss(qcnn, ctx):
    Din, Dout, K, d = 610, 701, 32, 4
    W, ctrd, asmt = start(Din, Dout, K, d, 24)
    X = gaussian_inputs(2 * Din, Din, 25)
    x = cuda(X)
    prev = np.zeros(0)
    for sweeps in (1, 2, 3):
        c, a, loss = qcnn.pq_refine_fc(ctx, W, x, ctrd, asmt, sweeps=sweeps)
        assert loss.shape == (sweeps + 1,)
        assert loss[:len(prev)].tobytes() == prev.tobytes(), (sweeps, loss, prev)
        want = response_loss(W, X, c, a)
        assert abs(loss[-1] - want) <= 1e-9 * want, (sweeps, loss[-1], want)
        prev = loss


@pytest.mark.gpu
def test_identity_inputs_give_one_kmeans_iteration(qcnn, ctx):
    Din, Dout, K, d = 64, 400, 32, 4
    W, C0, _ = start(Din, Dout, K, d, 31)
    _, a0, _ = qcnn.pq_quantize_fc(ctx, W, K, d, iters=0, init=C0)
    C1, a1, _ = qcnn.pq_quantize_fc(ctx, W, K, d, iters=1, init=C0)
    c, a, _ = qcnn.pq_refine_fc(ctx, W, cuda(np.eye(Din)), C0, a0, sweeps=1)
    assert ulps(c, C1).max() <= 1.0
    for m in range(-(-Din // d)):
        x = np.ascontiguousarray(W[:, m * d:(m + 1) * d])
        dist = dists(x, C1[m][:, :x.shape[1]]).astype(np.float64)
        differ = np.nonzero(a[:, m] != a1[:, m])[0]
        for o in differ:
            d1, d2 = dist[o, a[o, m]], dist[o, a1[o, m]]
            assert abs(d1 - d2) <= 1e-5 * max(d1, d2), (m, o, d1, d2)


@pytest.mark.gpu
def test_exact_weights_are_a_fixed_point(qcnn, ctx):
    Din, Dout, K, d = 130, 200, 32, 8
    _, Cs, As = start(Din, Dout, K, d, 41)
    Cs[3, 7] = Cs[3, 2]   # two equal codewords: the lower index may take the other's outputs
    W = decoded(Cs, As, Din).astype(np.float32)
    X = gaussian_inputs(2 * Din, Din, 42)
    c, a, loss = qcnn.pq_refine_fc(ctx, W, cuda(X), Cs, As, sweeps=3)
    assert c.tobytes() == Cs.tobytes()
    assert (loss == 0).all(), loss
    differ = a != As
    if differ.any():
        m_idx = np.nonzero(differ)[1]
        assert np.array_equal(c[m_idx, a[differ]], c[m_idx, As[differ]])
        assert (a[differ] < As[differ]).all()


@pytest.mark.gpu
def test_descent_and_reproducibility(qcnn, ctx):
    Din, Dout, K, d = 1024, 512, 32, 4
    W = (np.random.RandomState(51).randn(Dout, Din) / 32).astype(np.float32)
    X = gaussian_inputs(2048, Din, 52)
    c0, a0, _ = qcnn.pq_quantize_fc(ctx, W, K, d, iters=5, seed=3)
    x = cuda(X)
    c, a, loss = qcnn.pq_refine_fc(ctx, W, x, c0, a0, sweeps=4)
    assert loss.shape == (5,)
    assert (loss[1:] <= loss[:-1] * (1 + 1e-12)).all(), loss
    assert loss[-1] < loss[0]
    want = response_loss(W, X, c, a)
    assert abs(loss[-1] - want) <= 1e-9 * want, (loss[-1], want)
    c2, a2, l2 = qcnn.pq_refine_fc(ctx, W, x, c0, a0, sweeps=4)
    assert c2.tobytes() == c.tobytes() and a2.tobytes() == a.tobytes() and l2.tobytes() == loss.tobytes()


def correlated_inputs(N, Din, seed):
    """Gaussian inputs with covariance spectrum exp(-i / (Din / 10)) in a random orthonormal basis"""
    rng = np.random.RandomState(seed)
    Q, _ = np.linalg.qr(rng.randn(Din, Din))
    s = np.exp(-np.arange(Din) / (Din / 10.0)) ** 0.5
    return ((rng.randn(N, Din) * s) @ Q.T).astype(np.float32)


@pytest.mark.gpu
def test_corrects_error_on_unseen_inputs(qcnn, ctx):
    Din = Dout = 1024
    K, d = 32, 4
    W = (np.random.RandomState(61).randn(Dout, Din) / 32).astype(np.float32)
    X = correlated_inputs(8192, Din, 62)
    train, held = X[:4096], X[4096:]
    c0, a0, _ = qcnn.pq_quantize_fc(ctx, W, K, d, iters=20, seed=7)
    c, a, loss = qcnn.pq_refine_fc(ctx, W, cuda(train), c0, a0, sweeps=8)
    assert (loss[1:] <= loss[:-1] * (1 + 1e-12)).all(), loss
    held0, held1 = response_loss(W, held, c0, a0), response_loss(W, held, c, a)
    print("training loss %.4g -> %.4g (x%.3f), held-out error %.4g -> %.4g (x%.3f)"
          % (loss[0], loss[-1], loss[-1] / loss[0], held0, held1, held1 / held0))
    assert loss[-1] <= 0.5 * loss[0]
    assert held1 <= 0.5 * held0


# ---- shipped AlexNet fc7 ------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_shipped_alexnet_fc7_on_its_own_inputs(po, qcnn, ctx):
    import torch
    if not po.have_alexnet():
        pytest.skip("shipped AlexNet parameters not staged under oracle/_ref/data")
    params = po.load_model(po.ALEXNET_DIR, po.ALEXNET_PFX, po.alexnet_layers())
    p = params[18]
    W = decoded(p["ctrd"], p["asmt"], 4096).astype(np.float32)
    net = qcnn.Net(ctx, po.ALEXNET_DIR, po.ALEXNET_PFX, "AlexNet")
    net.set_keep_maps(True)
    maps = []
    for i in range((16384 + 2048) // 256):
        net.forward(torch.from_numpy(po.lcg_images(256, 700000 + 256 * i)).cuda())
        maps.append(net.featmap(18, 256).reshape(256, 4096))   # fc6 after ReLU
    net.close()
    X = torch.cat(maps)
    train, held = X[:16384].contiguous(), X[16384:].contiguous()
    c0, a0, _ = qcnn.pq_quantize_fc(ctx, W, 16, 8, iters=20, seed=1)
    c, a, loss = qcnn.pq_refine_fc(ctx, W, train, c0, a0, sweeps=4)
    assert (loss[1:] <= loss[:-1] * (1 + 1e-12)).all(), loss
    ref = held.double() @ torch.from_numpy(W).cuda().double().T + torch.from_numpy(p["bias"]).cuda().double()
    errs = []
    for cc, aa in ((c0, a0), (c, a)):
        fc = qcnn.FcLayer(ctx, 4096, cc, aa, p["bias"])
        y = fc.forward(held)
        errs.append(((y.double() - ref).norm() / ref.norm()).item())
        fc.close()
    print("AlexNet fc7 re-quantized at K=16, d=8: held-out relative output error k-means %.4f, refined %.4f "
          "(training loss x%.3f)" % (errs[0], errs[1], loss[-1] / loss[0]))
    assert errs[1] < errs[0]


# ---- errors -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rejected_inputs(qcnn, ctx):
    import torch
    Din, Dout, K, d = 32, 40, 16, 4
    W, ctrd, asmt = start(Din, Dout, K, d, 71)
    X = gaussian_inputs(20, Din, 72)
    Xn = X.copy()
    Xn[7, 5] = np.nan
    Winf = W.copy()
    Winf[3, 3] = np.inf
    Ak = asmt.copy()
    Ak[5, 2] = K
    _, c48, a48 = start(Din, Dout, 48, d, 71)
    _, c65, a65 = start(130, Dout, 16, 65, 71)
    bad = [
        (lambda: qcnn.pq_refine_fc(ctx, W, cuda(Xn), ctrd, asmt, 1), "non-finite"),
        (lambda: qcnn.pq_refine_fc(ctx, Winf, cuda(X), ctrd, asmt, 1), "non-finite"),
        (lambda: qcnn.pq_refine_fc(ctx, W, cuda(X), ctrd, Ak, 1), "not below K=16"),
        (lambda: qcnn.pq_refine_fc(ctx, W, cuda(X), c48, a48, 1), "K=48"),
        (lambda: qcnn.pq_refine_fc(ctx, start(130, Dout, 16, 65, 71)[0], cuda(gaussian_inputs(20, 130, 1)), c65, a65, 1),
         "d=65"),
        (lambda: qcnn.pq_refine_fc(ctx, W, cuda(X), ctrd, asmt, -1), "sweeps=-1"),
        (lambda: qcnn.pq_refine_fc(ctx, W, torch.empty((0, Din), dtype=torch.float32, device="cuda"), ctrd, asmt, 1),
         "N=0"),
    ]
    for fn, msg in bad:
        with pytest.raises(qcnn.QcnnError) as e:
            fn()
        assert msg in str(e.value), (msg, str(e.value))
