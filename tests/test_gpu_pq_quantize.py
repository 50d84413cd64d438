"""k-means product quantization of dense conv / FC weights on the GPU (qcnn_pq_quantize_conv / _fc / _model) against a
numpy restatement of its semantics (DESIGN.md 4e): fp32 distances summed in ascending j, np.argmin for the lowest index
on ties, fp64 means, the project's LCG for the seeded initialisation."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from test_gpu_layers import close
from test_gpu_net import MODES, set_mode

NEW_SYMBOLS = ("qcnn_pq_quantize_conv", "qcnn_pq_quantize_fc", "qcnn_pq_quantize_model")


# ---- the restatement ----------------------------------------------------------------------------------------------
def subspaces(w, d):
    """w [Cout][Cg][k][k] (FC: [Dout][Din] as k = 1) -> per subspace the points [P][w_s]."""
    if w.ndim == 2:
        w = w[:, :, None, None]
    Cout, Cg, k, _ = w.shape
    return [np.ascontiguousarray(w[:, s * d:s * d + min(d, Cg - s * d)].transpose(0, 2, 3, 1).reshape(Cout * k * k, -1))
            for s in range(-(-Cg // d))]


def dists(x, c):
    """[P][K] fp32: acc = acc + (x[j] - c[j])^2 over the valid dims in ascending j, each operation rounded to fp32."""
    acc = np.zeros((x.shape[0], c.shape[0]), np.float32)
    for j in range(x.shape[1]):
        t = x[:, j:j + 1] - c[None, :, j]
        acc = acc + t * t
    return acc


def assign(x, c):
    return np.argmin(dists(x, c), axis=1).astype(np.uint8)


def seeded_init(x, K, seed, s):
    P = x.shape[0]
    r = (seed + s) & 0xFFFFFFFF
    perm = {}
    pick = []
    for i in range(K):
        r = (1664525 * r + 1013904223) & 0xFFFFFFFF
        j = i + (r >> 8) % (P - i)
        pi, pj = perm.get(i, i), perm.get(j, j)
        perm[i], perm[j] = pj, pi
        pick.append(pj)
    return x[pick]


def exact_means(x, a, c_prev):
    c = c_prev.copy()
    for k in range(c.shape[0]):
        m = a == k
        if m.any():
            c[k, :x.shape[1]] = (x[m].astype(np.float64).sum(axis=0) / m.sum()).astype(np.float32)
    return c


def ulps(a, b):
    return np.abs(a.astype(np.float64) - b.astype(np.float64)) / np.spacing(np.maximum(np.abs(a), np.abs(b)).astype(np.float32))


def sse_of(xs, ctrd, asmt):
    a = asmt.reshape(-1, len(xs))
    return sum(float(dists(x, ctrd[s][:, :x.shape[1]])[np.arange(x.shape[0]), a[:, s]].astype(np.float64).sum())
               for s, x in enumerate(xs))


def quantize(qcnn, ctx, w, K, d, **kw):
    return (qcnn.pq_quantize_conv if w.ndim == 4 else qcnn.pq_quantize_fc)(ctx, w, K, d, **kw)


# ---- which assignment kernel a shape runs (PickAssign / PadDims in pq_quantize.cu) ------------------------------------
ASSIGN_THREADS = 128
UPDATE_CHUNK = 1024   # points per CTA of the update's partial sums
ASSIGN_KERNELS = {(D, R) for D in (4, 8, 16) for R in (8, 4, 2)} | {(32, 4), (32, 2), (64, 2)}   # the 12 instantiations


def pad_dims(w):
    D = 4
    while D < w:
        D *= 2
    return D


def points(shape):
    """points per subspace: Cout k^2 (FC: Dout)"""
    return shape[0] * (shape[2] * shape[3] if len(shape) == 4 else 1)


def assign_plan(shape, d, sm_count):
    """(D, R) of the pq_assign_kernel<D, R> that weights of `shape` at subspace width d run on sm_count SMs"""
    Cg, P = shape[1], points(shape)
    S, D = -(-Cg // d), pad_dims(min(d, Cg))
    R = 8 if D <= 16 else 128 // D
    while R > 2 and S * -(-P // (ASSIGN_THREADS * R)) < 2 * sm_count:
        R //= 2
    return D, R


# (name, weight shape, K, d)
CASES = [
    ("conv1", (96, 3, 11, 11), 128, 8),      # d > Cg: one partial subspace of 3 dims
    ("conv2g", (256, 48, 5, 5), 128, 8),     # the grouped conv2 of AlexNet (48 channels per group)
    ("k256_d64", (64, 100, 2, 2), 256, 64),  # subspaces of 64 and 36 dims
    ("fc_d1", (300, 40), 16, 1),
    ("fc_d4", (200, 30), 32, 4),             # Din % d = 2
]
# One row per assignment kernel (D, R), on 114 and on 132 SMs alike (test_assign_rows_cover_every_kernel).  Every row
# has a partial last CTA of points and a partial last update chunk, and a partial last subspace where d > 1.  Rows at
# d = 16 and d = 32 fill D, so the last float4 of a point carries data; the d = 12 and d = 24 rows leave it padding.
ASSIGN_CASES = [
    ("fc_D4_R8", (2500, 602), 32, 4),
    ("fc_D4_R4", (1500, 402), 32, 4),
    ("fc_D4_R2", (300, 130), 32, 4),
    ("fc_D8_R8", (2500, 1202), 32, 8),
    ("fc_D8_R4", (1500, 802), 32, 8),
    ("fc_D8_R2", (300, 130), 32, 8),
    ("fc_D16_R8", (2500, 1450), 32, 16),
    ("fc_D16_R4", (1500, 1210), 32, 12),
    ("fc_D16_R2", (300, 250), 32, 16),
    ("fc_D16_R2_d12", (300, 130), 32, 12),
    ("fc_D32_R4", (1500, 3210), 32, 32),
    ("fc_D32_R2", (300, 250), 32, 24),
    ("fc_D64_R2", (300, 250), 32, 64),
]
CASES += ASSIGN_CASES


def weights(shape, seed):
    return np.random.RandomState(seed).randn(*shape).astype(np.float32)


# ---- CPU ----------------------------------------------------------------------------------------------------------
def test_quantize_symbols_declared_and_exported(qcnn):
    text = open(qcnn.HEADER_PATH).read()
    lib = C.CDLL(qcnn.LIB_PATH)
    for name in NEW_SYMBOLS:
        assert re.search(r"QCNN_API\s+int\s+%s\s*\(" % name, text), name
        assert hasattr(lib, name), name
        assert name in qcnn.EXPORTS


def assign_coverage(sm_count):
    """{(D, R): names of the ASSIGN_CASES rows that run it}; asserts every row's point and subspace tails"""
    out = {}
    for name, shape, K, d in ASSIGN_CASES:
        D, R = assign_plan(shape, d, sm_count)
        P, Cg = points(shape), shape[1]
        assert P % (ASSIGN_THREADS * R) and P % UPDATE_CHUNK, (name, sm_count)   # partial last CTA and update chunk
        assert d == 1 or Cg % d, name                                           # partial last subspace
        out.setdefault((D, R), []).append(name)
    return out


@pytest.mark.parametrize("sm_count", [132, 114])
def test_assign_rows_cover_every_kernel(sm_count):
    cov = assign_coverage(sm_count)
    print("sm_count %d: %s" % (sm_count, ", ".join("D=%d R=%d: %s" % (D, R, "/".join(n)) for (D, R), n in sorted(cov.items()))))
    assert set(cov) == ASSIGN_KERNELS
    for D in (16, 32):   # subspaces that fill D, and subspaces that leave the last float4 padding
        ds = {d for _, shape, _, d in ASSIGN_CASES if assign_plan(shape, d, sm_count)[0] == D}
        assert D in ds and any(d <= D - 4 for d in ds), (D, ds)


@pytest.mark.gpu
def test_assign_rows_cover_every_kernel_on_this_gpu(ctx):
    assert set(assign_coverage(ctx.sm_count)) == ASSIGN_KERNELS, ctx.sm_count


# ---- exact steps --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,shape,K,d", CASES, ids=[c[0] for c in CASES])
def test_seeded_init_and_first_assignment_exact(name, shape, K, d, qcnn, ctx):
    w = weights(shape, 1)
    ctrd, asmt, sse = quantize(qcnn, ctx, w, K, d, iters=0, seed=77)
    xs = subspaces(w, d)
    assert ctrd.shape == (len(xs), K, d) and sse.shape == (1,)
    a = asmt.reshape(-1, len(xs))
    for s, x in enumerate(xs):
        ws = x.shape[1]
        assert np.array_equal(ctrd[s][:, :ws], seeded_init(x, K, 77, s)), s   # C_0 is exactly the drawn points
        assert not ctrd[s][:, ws:].any(), s                                    # unused dims are 0
        assert np.array_equal(a[:, s], assign(x, ctrd[s][:, :ws])), s
    assert abs(sse[0] - sse_of(xs, ctrd, asmt)) <= 1e-9 * max(1.0, sse[0])


@pytest.mark.gpu
@pytest.mark.parametrize("name,shape,K,d", CASES, ids=[c[0] for c in CASES])
def test_one_update_from_given_codebook(name, shape, K, d, qcnn, ctx):
    w = weights(shape, 2)
    xs = subspaces(w, d)
    rng = np.random.RandomState(3)
    init = rng.randn(len(xs), K, d).astype(np.float32)
    init[:, ::5] += np.float32(1000.0)   # far away: these clusters stay empty
    ctrd, asmt, _ = quantize(qcnn, ctx, w, K, d, iters=1, init=init)
    _, a0, _ = quantize(qcnn, ctx, w, K, d, iters=0, init=init)
    a0 = a0.reshape(-1, len(xs))
    a = asmt.reshape(-1, len(xs))
    for s, x in enumerate(xs):
        ws = x.shape[1]
        assert np.array_equal(a0[:, s], assign(x, init[s][:, :ws])), s
        want = exact_means(x, a0[:, s], init[s][:, :ws])
        empty = np.setdiff1d(np.arange(K), a0[:, s])
        assert len(empty) >= K // 5
        assert np.array_equal(ctrd[s][empty, :ws], init[s][empty, :ws]), s
        assert ulps(ctrd[s][:, :ws], want).max() <= 1.0, s
        assert not ctrd[s][:, ws:].any(), s
        assert np.array_equal(a[:, s], assign(x, ctrd[s][:, :ws])), s


# ---- many iterations ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,shape,K,d", CASES, ids=[c[0] for c in CASES])
def test_twenty_iterations(name, shape, K, d, qcnn, ctx):
    w = weights(shape, 4)
    xs = subspaces(w, d)
    ctrd, asmt, sse = quantize(qcnn, ctx, w, K, d, iters=20, seed=5)
    assert sse.shape == (21,)
    assert np.all(sse[1:] <= sse[:-1] * (1 + 1e-6)), sse
    assert abs(sse[-1] - sse_of(xs, ctrd, asmt)) <= 1e-9 * sse[-1]
    c2, a2, s2 = quantize(qcnn, ctx, w, K, d, iters=20, seed=5)
    assert c2.tobytes() == ctrd.tobytes() and a2.tobytes() == asmt.tobytes() and s2.tobytes() == sse.tobytes()
    a = asmt.reshape(-1, len(xs))
    for s, x in enumerate(xs):
        assert np.array_equal(a[:, s], assign(x, ctrd[s][:, :x.shape[1]])), s


# ---- shipped AlexNet ----------------------------------------------------------------------------------------------
def decode(p, cin):
    """Dense weights of a PQ layer: conv [Cout][Cg][k][k], FC [Dout][Din] (W = ctrd[s][asmt])."""
    ctrd, asmt = p["ctrd"], p["asmt"]
    S, K, d = ctrd.shape
    g = ctrd[np.arange(S), asmt]                    # [..., S, d]
    g = g.reshape(g.shape[:-2] + (S * d,))[..., :cin]
    return np.ascontiguousarray(np.moveaxis(g, -1, 1)) if g.ndim == 4 else np.ascontiguousarray(g)


def input_widths(po):
    layers = po.alexnet_layers()
    shapes = po.infer_shapes(layers, po.ALEXNET_IN)
    out = {}
    for l, L in enumerate(layers):
        h, w, c = shapes[l]
        if L["type"] == po.CONV:
            out[l] = c // L["grp"]
        elif L["type"] == po.FCNT:
            out[l] = h * w * c
    return out


@pytest.fixture(scope="module")
def shipped(po):
    if not po.have_alexnet():
        pytest.skip("shipped AlexNet parameters not staged under oracle/_ref/data")
    params = po.load_model(po.ALEXNET_DIR, po.ALEXNET_PFX, po.alexnet_layers())
    widths = input_widths(po)
    dense = {l: decode(p, widths[l]) for l, p in params.items()}
    return params, dense


def no_autotune(po, net):
    """Conv layers keep the cost model's first tiling, so that two nets run the same kernels."""
    for l, L in enumerate(po.alexnet_layers()):
        if L["type"] == po.CONV:
            net.pq_layer(l).set_param("autotune", 0)


@pytest.mark.gpu
def test_shipped_alexnet_is_a_fixed_point(po, qcnn, ctx, shipped, tmp_path):
    import torch
    params, dense = shipped
    out = {}
    for l, p in params.items():
        S, K, d = p["ctrd"].shape
        ctrd, asmt, sse = quantize(qcnn, ctx, dense[l], K, d, iters=3, init=p["ctrd"])
        assert np.array_equal(ctrd, p["ctrd"]), l
        assert sse[-1] == 0.0, (l, sse)
        differ = asmt != p["asmt"]
        if differ.any():   # only where two codewords are equal, and then the lower index
            s_idx = np.nonzero(differ)[-1]
            assert np.array_equal(ctrd[s_idx, asmt[differ]], ctrd[s_idx, p["asmt"][differ]]), l
            assert (asmt[differ] < p["asmt"][differ]).all(), l
        q = dict(p, ctrd=ctrd, asmt=asmt)
        assert np.array_equal(decode(q, dense[l].shape[1]), dense[l]), l
        out[l] = q
    d = str(tmp_path)
    po.save_model(d, "fp", out)
    ref = qcnn.Net(ctx, po.ALEXNET_DIR, po.ALEXNET_PFX, "AlexNet")
    got = qcnn.Net(ctx, d, "fp", "AlexNet")
    img = torch.from_numpy(po.lcg_images(8, 2024)).cuda()
    for mode in ("default", "strict"):
        res = []
        for net in (ref, got):
            set_mode(net, mode)
            no_autotune(po, net)
            lg = torch.empty((8, 1000), dtype=torch.float32, device="cuda")
            pr = net.forward(img, logits=lg)
            res.append((lg.cpu().numpy(), pr.cpu().numpy()))
        assert np.array_equal(res[0][0], res[1][0]), mode
        assert np.array_equal(res[0][1], res[1][1]), mode
    ref.close()
    got.close()


@pytest.mark.gpu
def test_model_level_matches_per_layer_calls(po, qcnn, ctx, shipped, tmp_path):
    import torch
    params, dense = shipped
    layers = po.alexnet_layers()
    src, out, per = (str(tmp_path / n) for n in ("dense", "model", "layers"))
    for p in (src, out, per):
        os.makedirs(p)
    for l, w in dense.items():
        kind = "convKnl" if w.ndim == 4 else "fcntWei"
        po.write_bin(os.path.join(src, "a.%s.%02d.bin" % (kind, l + 1)), w)
        po.write_bin(os.path.join(src, "a.biasVec.%02d.bin" % (l + 1)), params[l]["bias"])
    pq = {l: p["ctrd"].shape[1:] for l, p in params.items()}
    seed = 99
    qcnn.pq_quantize_model(ctx, "AlexNet", src, "a", out, "q", pq, iters=10, seed=seed)
    mine = {}
    for l, w in dense.items():
        K, d = pq[l]
        ctrd, asmt, _ = quantize(qcnn, ctx, w, K, d, iters=10, seed=(seed + 65536 * (l + 1)) & 0xFFFFFFFF)
        mine[l] = dict(ctrd=ctrd, asmt=asmt, bias=params[l]["bias"], bits=po.bits_for(K))
    po.save_model(per, "q", mine)
    assert sorted(os.listdir(out)) == sorted(os.listdir(per))
    for f in os.listdir(out):
        assert open(os.path.join(out, f), "rb").read() == open(os.path.join(per, f), "rb").read(), f
    loaded = po.load_model(out, "q", layers)
    for l in params:
        assert np.array_equal(loaded[l]["ctrd"], mine[l]["ctrd"]) and np.array_equal(loaded[l]["asmt"], mine[l]["asmt"])
    net = qcnn.Net(ctx, out, "q", "AlexNet")
    img = po.lcg_images(3, 4242)
    ref_prob, ref_maps = po.net_forward(layers, loaded, img, keep=True)
    for mode in ("strict", "default"):
        set_mode(net, mode)
        RT, PT = MODES[mode]
        logits = torch.empty((3, 1000), dtype=torch.float32, device="cuda")
        prob = net.forward(torch.from_numpy(img).cuda(), logits=logits).cpu().numpy()
        assert close(logits.cpu().numpy(), ref_maps[len(layers) - 1].reshape(3, -1)) <= RT, mode
        assert np.abs(prob - ref_prob).max() <= PT, mode
    shipped_net = qcnn.Net(ctx, po.ALEXNET_DIR, po.ALEXNET_PFX, "AlexNet")
    imgs = torch.from_numpy(po.lcg_images(64, 12345)).cuda()
    agree = (net.forward(imgs).argmax(1) == shipped_net.forward(imgs).argmax(1)).float().mean().item()
    print("top-1 agreement of the k-means model (iters=10) with the shipped AlexNet on 64 LCG images: %.3f" % agree)
    net.close()
    shipped_net.close()


# ---- errors -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_rejected_inputs(qcnn, ctx, tmp_path):
    w = weights((16, 8, 3, 3), 6)
    bad = [
        (lambda: qcnn.pq_quantize_conv(ctx, np.where(np.arange(w.size).reshape(w.shape) == 7, np.nan, w), 16, 4), "non-finite"),
        (lambda: qcnn.pq_quantize_fc(ctx, np.full((32, 8), np.inf, np.float32), 16, 4), "non-finite"),
        (lambda: qcnn.pq_quantize_conv(ctx, w, 12, 4), "K=12"),
        (lambda: qcnn.pq_quantize_fc(ctx, w.reshape(16, -1), 48, 4), "K=48"),
        (lambda: qcnn.pq_quantize_fc(ctx, weights((64, 130), 1), 16, 65), "d=65"),
        (lambda: qcnn.pq_quantize_conv(ctx, weights((2, 8, 1, 1), 1), 16, 4), "points"),
        (lambda: qcnn.pq_quantize_conv(ctx, w, 16, 4, iters=-1), "iters=-1"),
    ]
    for fn, msg in bad:
        with pytest.raises(qcnn.QcnnError) as e:
            fn()
        assert msg in str(e.value), (msg, str(e.value))
    # with an init codebook, fewer points than K is fine
    init = weights((2, 16, 4), 2)
    ctrd, _, _ = qcnn.pq_quantize_conv(ctx, weights((2, 8, 1, 1), 1), 16, 4, iters=2, init=init)
    assert ctrd.shape == (2, 16, 4)


@pytest.mark.gpu
def test_model_level_errors_leave_no_files(po, qcnn, ctx, tmp_path):
    layers = po.alexnet_layers()
    widths = input_widths(po)
    src, out = str(tmp_path / "dense"), str(tmp_path / "out")
    os.makedirs(src)
    os.makedirs(out)
    rng = np.random.RandomState(8)
    for l, L in enumerate(layers):
        if l not in widths:
            continue
        if L["type"] == po.CONV:
            w, n = rng.randn(L["cnt"], widths[l], L["k"], L["k"]), L["cnt"]
            po.write_bin(os.path.join(src, "a.convKnl.%02d.bin" % (l + 1)), w.astype(np.float32))
        else:
            w, n = rng.randn(L["nod"], widths[l]) * 0.01, L["nod"]
            po.write_bin(os.path.join(src, "a.fcntWei.%02d.bin" % (l + 1)), w.astype(np.float32))
        po.write_bin(os.path.join(src, "a.biasVec.%02d.bin" % (l + 1)), rng.randn(n).astype(np.float32))
    pq = {l: (K, d) for l, (S, K, d) in po.ALEXNET_PQ.items()}
    for bad, msg in (({21: (48, 1)}, "layer 22: unsupported codebook size K=48"), ({4: (128, 80)}, "layer 5: d=80")):
        with pytest.raises(qcnn.QcnnError) as e:
            qcnn.pq_quantize_model(ctx, "AlexNet", src, "a", out, "q", {**pq, **bad}, iters=1)
        assert msg in str(e.value), str(e.value)
        assert os.listdir(out) == []
    with pytest.raises(qcnn.QcnnError) as e:
        qcnn.pq_quantize_model(ctx, "AlexNet", src, "a", str(tmp_path / "missing"), "q", pq, iters=1)
    assert "cannot write" in str(e.value)
    with pytest.raises(qcnn.QcnnError) as e:
        qcnn.pq_quantize_model(ctx, "NoSuchNet", src, "a", out, "q", pq, iters=1)
    assert "unrecognized" in str(e.value)
    # a dense file whose shape does not match the table
    po.write_bin(os.path.join(src, "a.convKnl.05.bin"), rng.randn(256, 96, 5, 5).astype(np.float32))
    with pytest.raises(qcnn.QcnnError) as e:
        qcnn.pq_quantize_model(ctx, "AlexNet", src, "a", out, "q", pq, iters=1)
    assert "layer 5: convKnl is not [256][48][5][5]" in str(e.value)
    assert os.listdir(out) == []
