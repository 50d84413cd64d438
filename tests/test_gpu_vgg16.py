"""VGG16 on the GPU: its 224-wide and 3-channel stride-1 convolutions on the weight-stationary tensor-core GEMM (conv_ws,
force_kernel = 7) against the float64 reference of test_gpu_pq_gemm.py, and the whole 39-layer net, built by name,
against the CPU oracle.

Layer cases.  conv_ws stages a CTA's positions in as many register passes of its producer threads as the halo needs,
so a stride-1 layer of any width whose plane ring fits in shared memory has a tiling; a group of <= 3 input channels
(conv1_1: RGB) is one chunk read as scalars, with a zero second half.  Every case pins the family at every tiling the
planner offers and checks tc_bound(bf16x2, 128, chunks x taps, 1) (the k-step chain of pq_gemm_tc mode 0), ReLU and
run-to-run bit identity; some also the neighbour NaN isolation and the exact write set (helpers of
test_gpu_conv_ws_s1.py).  With tensor_core = 0 the same layers run the stride-1 LUT + gather kernels, on column tiles
where whole rows do not fit a LUT.  conv1_1 and conv1_2 run at batch 1, 3 and 256; batch-256 inputs are generated on the device
and the reference runs on a sample of images (both ends, the middle, a spread).  Widths either side of the limit
of one register pass (126 / 127 with P = 256, 190 / 191 with P = 128) and beyond it (318), with k = 3 and k = 5.

Net.  Seeded synthetic parameters in the reference's file formats (tests/test_oracle_vgg16.py, which pins the oracle
and this table against the compiled reference).  Tolerances are MODES of test_gpu_net.py: VGG16 chains 16 PQ layers."""
import ctypes
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from test_gpu_conv_ws_s1 import Row, assert_plan, ksteps, pin, positions, unpin, widths
from test_gpu_layers import CONV_FAMILY_NAMES, close
from test_gpu_net import MODES, set_mode
from test_gpu_pq_gemm import _guarded_call, _seed, bits, conv_data, f64_err, ref64, strict_bound, tc_bound
from test_oracle_vgg16 import VGG16_CONVS, VGG16_IN, synth_vgg16, vgg16_images

ROWS = [
    # VGG16 block 1 exactly
    Row("conv1_1_n1", 1, 224, 224, 3, 64, 3, 1, 1, 1, 1, 128, 4, False),
    Row("conv1_1_n3", 3, 224, 224, 3, 64, 3, 1, 1, 1, 1, 128, 4, False),
    Row("conv1_1_n256", 256, 224, 224, 3, 64, 3, 1, 1, 1, 1, 128, 4, False),
    Row("conv1_2_n1", 1, 224, 224, 64, 64, 3, 1, 1, 1, 8, 128, 8, False),
    Row("conv1_2_n3", 3, 224, 224, 64, 64, 3, 1, 1, 1, 8, 128, 8, False),
    Row("conv1_2_n256", 256, 224, 224, 64, 64, 3, 1, 1, 1, 8, 128, 8, False),
    # widths around the single-pass limit and beyond (2 NPOS float4 over 1024 per pass), k = 3 and 5
    Row("w126_k3", 2, 6, 126, 16, 64, 3, 1, 1, 1, 2, 128, 8, False),
    Row("w127_k3", 2, 6, 127, 16, 64, 3, 1, 1, 1, 2, 128, 8, False),
    Row("w190_k3_cg12", 2, 5, 190, 12, 64, 3, 1, 1, 1, 3, 64, 4, False),
    Row("w191_k3", 2, 5, 191, 16, 128, 3, 1, 1, 1, 2, 128, 8, False),
    Row("w318_k3", 2, 4, 318, 16, 64, 3, 1, 1, 1, 2, 128, 8, False),
    Row("w126_k5", 2, 7, 126, 16, 64, 5, 2, 1, 1, 2, 128, 8, False),
    Row("w191_k5_g2", 2, 6, 191, 32, 64, 5, 2, 1, 2, 2, 64, 8, False),
    Row("w318_k5", 2, 5, 318, 8, 32, 5, 2, 1, 1, 1, 128, 8, False),
    # <= 3 channels per group: pad 0 / 1 / 2, G = 2, d = 4 / 8
    Row("cg1_pad0", 3, 17, 19, 1, 32, 3, 0, 1, 1, 1, 64, 4, False),
    Row("cg2_pad1_d8", 2, 20, 15, 2, 64, 3, 1, 1, 1, 1, 64, 8, False),
    Row("cg3_pad1_g2", 2, 16, 18, 6, 128, 3, 1, 1, 2, 1, 128, 4, False),
    Row("cg3_k5_pad2", 2, 30, 33, 3, 48, 5, 2, 1, 1, 1, 32, 4, False),
    Row("cg3_pad0_w200", 1, 9, 200, 3, 64, 3, 0, 1, 1, 1, 128, 4, False),
]
BYNAME = {r.name: r for r in ROWS}
BIG = 200_000_000   # input elements above which the input is generated on the device


def sample(N):
    return sorted({0, 1, 2, 127, 128, 254, 255} | set(range(5, 256, 31))) if N == 256 else list(range(N))


class _Cache(object):
    def __init__(self, qcnn, ctx):
        self.qcnn, self.ctx, self.items = qcnn, ctx, {}

    def get(self, row):
        import torch
        if row.name not in self.items:
            big = row.N * row.Hi * row.Wi * row.Cin > BIG
            small = row._replace(N=1) if big else row
            x, ctrd, asmt, bias = conv_data(small)
            if big:
                g = torch.Generator(device="cuda").manual_seed(_seed(row.name))
                xd = torch.randn((row.N, row.Hi, row.Wi, row.Cin), generator=g, device="cuda").abs_().mul_(4.0)
            else:
                xd = torch.from_numpy(x).cuda()
            L = self.qcnn.ConvLayer(self.ctx, row.Cin, row.Hi, row.Wi, row.Cout, row.k, row.pad, row.stride, row.G,
                                    ctrd, asmt, bias)
            sel = sample(row.N)
            xs = xd[sel].cpu().numpy()
            refs = [ref64("conv", xs[i:i + 1], ctrd, asmt, bias, (row.pad, row.stride, row.G)) for i in range(len(sel))]
            self.items[row.name] = dict(L=L, xd=xd, xs=xs, sel=sel, ref=np.concatenate([r[0] for r in refs]),
                                        mag=np.concatenate([r[1] for r in refs]))
        return self.items[row.name]

    def drop(self, row):
        it = self.items.pop(row.name, None)
        if it:
            it["L"].close()

    def close(self):
        for it in self.items.values():
            it["L"].close()


@pytest.fixture(scope="module")
def cache(qcnn, ctx):
    c = _Cache(qcnn, ctx)
    yield c
    c.close()


def _cases(rows):
    return [pytest.param(r, P, W, id="%s-P%d-N%d" % (r.name, P, W)) for r in rows for W in widths(r) for P in positions(W)]


def _sel(y, sel):
    import torch
    return y[torch.as_tensor(sel, device=y.device)].cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("row,P,W", _cases(ROWS))
def test_vgg16_conv_ws_f64(row, P, W, cache):
    it = cache.get(row)
    L = it["L"]
    pin(L, P, W)
    y = _sel(L.forward(it["xd"]), it["sel"])
    assert_plan(L.describe(row.N), row, P, W)
    bound = tc_bound(True, 128, ksteps(row), 1)
    e = f64_err(y, it["ref"], it["mag"])
    assert e <= bound, (e, bound)
    yr = _sel(L.forward(it["xd"], relu=True), it["sel"])
    er = f64_err(yr, np.maximum(it["ref"], 0), it["mag"])
    assert er <= bound, (er, bound)
    y2 = _sel(L.forward(it["xd"]), it["sel"])
    assert np.array_equal(bits(y), bits(y2))
    if row.N == 256 and P == positions(W)[-1] and W == widths(row)[-1]:
        cache.drop(row)   # (last tiling of a batch-256 row: release its device input)


POISON = [pytest.param(BYNAME[n], P, W, id="%s-P%d-N%d" % (n, P, W))
          for n in ("conv1_1_n3", "conv1_2_n3", "w127_k3", "w318_k5", "cg3_pad1_g2", "cg1_pad0")
          for W in widths(BYNAME[n]) for P in positions(W)]


@pytest.mark.gpu
@pytest.mark.parametrize("row,P,W", POISON)
def test_vgg16_conv_ws_neighbour_poison(row, P, W, cache):
    """Image i's output is bit-identical whether every other image is 0 or NaN (multi-pass tiles straddle images)."""
    import torch
    it = cache.get(row)
    L = it["L"]
    pin(L, P, W)
    i = (row.N - 1) // 2
    x = it["xd"].cpu().numpy()
    outs = []
    for fill in (0.0, np.nan):
        xp = np.full_like(x, fill)
        xp[i] = x[i]
        outs.append(L.forward(torch.from_numpy(xp).cuda()).cpu().numpy()[i])
    assert_plan(L.describe(row.N), row, P, W)
    assert np.array_equal(bits(outs[0]), bits(outs[1]))
    assert f64_err(outs[0], it["ref"][it["sel"].index(i)], it["mag"][it["sel"].index(i)]) <= tc_bound(True, 128, ksteps(row), 1)


WRITE_SET = [pytest.param(BYNAME[n], P, W, id="%s-P%d-N%d" % (n, P, W))
             for n in ("conv1_1_n1", "w191_k5_g2", "w318_k3", "cg3_k5_pad2", "cg2_pad1_d8")
             for W in widths(BYNAME[n]) for P in positions(W)]


@pytest.mark.gpu
@pytest.mark.parametrize("row,P,W", WRITE_SET)
def test_vgg16_conv_ws_exact_write_set(row, P, W, qcnn, cache):
    import torch
    it = cache.get(row)
    L = it["L"]
    pin(L, P, W)
    ho, wo, co = L.out_dims()
    n_out = row.N * ho * wo * co
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    xd = it["xd"]
    for relu in (0, 1):
        out, guard_ok = _guarded_call(
            lambda dst, r: qcnn._check(qcnn.lib.qcnn_conv_aprx_forward(L.h, ctypes.c_void_p(xd.data_ptr()), row.N, dst,
                                                                       r, stream)), n_out, relu)
        assert_plan(L.describe(row.N), row, P, W)
        assert guard_ok, relu
        assert np.isfinite(out).all(), (relu, int((~np.isfinite(out)).sum()))


@pytest.mark.gpu
def test_vgg16_cg3_unpinned_runs_conv_ws(cache):
    """A 3-channel stride-1 layer at bf16x2 has conv_ws as its only GEMM (pq_gemm_tc mode 0 does not take it)."""
    row = BYNAME["conv1_1_n3"]
    it = cache.get(row)
    L = it["L"]
    L.set_param("tensor_core", 2)
    unpin(L)
    y = _sel(L.forward(it["xd"]), it["sel"])
    desc = L.describe(row.N)
    assert desc.startswith("pq_gemm_tc_ws(") and " mode=0 " in desc, desc
    assert f64_err(y, it["ref"], it["mag"]) <= tc_bound(True, 128, ksteps(row), 1), desc


STRICT = [pytest.param(BYNAME[n], id=n) for n in ("conv1_1_n1", "conv1_2_n3", "w318_k5", "w191_k5_g2")]


@pytest.mark.gpu
@pytest.mark.parametrize("row", STRICT)
def test_vgg16_strict_lut_column_tiles(row, qcnn, cache):
    """tensor_core = 0: rows too wide for one LUT (3 rows x 225 positions x 128 codewords) run the stride-1 LUT + gather
    kernel (fp32 LUT stage) on column tiles, each with its own left halo; against the float64 reference within the
    strict families' bound.  (The tensor-core LUT stage holds at most 256 positions: it has no tiling at these widths.)"""
    fam = 0
    it = cache.get(row)
    L = it["L"]
    L.set_param("tensor_core", 0)
    L.set_param("force_kernel", fam)
    for name in ("gemm_nt", "gemm_ct"):
        L.set_param(name, 0)
    try:
        y = _sel(L.forward(it["xd"]), it["sel"])
        desc = L.describe(row.N)
        assert desc.startswith(CONV_FAMILY_NAMES[fam]), desc
        bound = strict_bound(fam, row.k * row.k, row.S, row.d, row.Cin // row.G)
        e = f64_err(y, it["ref"], it["mag"])
        assert e <= bound, (e, bound, desc)
        assert np.array_equal(bits(y), bits(_sel(L.forward(it["xd"]), it["sel"])))
    finally:
        L.set_param("tensor_core", 2)
        unpin(L)


# ---------------------------------------------------------------------------------------------------------------------
# the whole net
# ---------------------------------------------------------------------------------------------------------------------
NET_IMAGES = 256
NET_SAMPLE = sorted({0, 1, 2, 3, 100, 127, 128, 200, 254, 255})


@pytest.fixture(scope="module")
def vgg(po, tmp_path_factory):
    """Synthetic VGG16 files, a batch of 256 images and the oracle's maps of the sampled images."""
    layers, params = synth_vgg16(po, seed=16)
    d = str(tmp_path_factory.mktemp("synth_vgg16"))
    po.save_model(d, "vgg", params)
    img = vgg16_images(NET_IMAGES, 2016)
    with ThreadPoolExecutor(8) as ex:
        res = list(ex.map(lambda i: po.net_forward(layers, params, img[i:i + 1], keep=True), NET_SAMPLE))
    ref = {i: r for i, r in zip(NET_SAMPLE, res)}
    return dict(dir=d, layers=layers, img=img, prob={i: r[0][0] for i, r in ref.items()},
                maps={i: r[1] for i, r in ref.items()})


def _logits_ref(g, i):
    return g["maps"][i][len(g["layers"]) - 1].reshape(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["strict", "default"])
def test_vgg16_net_all_feature_maps_n2(mode, qcnn, ctx, vgg):
    import torch
    g = vgg
    N = 2
    net = qcnn.Net(ctx, g["dir"], "vgg", "VGG16")
    try:
        assert net.layer_count == 39 and net.out_len == 1000
        set_mode(net, mode)
        RT, PT = MODES[mode]
        net.set_keep_maps(True)
        logits = torch.empty((N, 1000), dtype=torch.float32, device="cuda")
        prob_d = net.forward(torch.from_numpy(g["img"][:N]).cuda(), logits=logits)   # keep alive: the last map lives in it
        for l in range(len(g["layers"]) + 1):
            fm = net.featmap(l, N)
            assert fm is not None, l
            want = np.stack([g["maps"][i][l][0] for i in range(N)])
            e = close(fm.cpu().numpy().reshape(-1), want.reshape(-1))
            assert e <= RT, (mode, l, e)
        assert close(logits.cpu().numpy(), np.stack([_logits_ref(g, i) for i in range(N)])) <= RT
        assert np.abs(prob_d.cpu().numpy() - np.stack([g["prob"][i] for i in range(N)])).max() <= PT
        if mode == "default":
            assert net.pq_layer(0).describe(N).startswith("pq_gemm_tc_ws(")
    finally:
        net.close()


@pytest.mark.gpu
def test_vgg16_net_graph_replay_n1_and_fc_chain_n4(qcnn, ctx, vgg):
    """N = 1 replayed from a captured CUDA graph on a side stream; N = 4 through the small-batch FC chain."""
    import torch
    g = vgg
    RT, PT = MODES["default"]
    net = qcnn.Net(ctx, g["dir"], "vgg", "VGG16")
    try:
        one = torch.from_numpy(g["img"][:1]).cuda()
        pg = torch.empty((1, 1000), dtype=torch.float32, device="cuda")
        side = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            for _ in range(4):
                net.forward(one, prob=pg)
                side.synchronize()
                assert np.abs(pg.cpu().numpy()[0] - g["prob"][0]).max() <= PT
        N = 4
        logits = torch.empty((N, 1000), dtype=torch.float32, device="cuda")
        prob = net.forward(torch.from_numpy(g["img"][:N]).cuda(), logits=logits).cpu().numpy()
        assert close(logits.cpu().numpy(), np.stack([_logits_ref(g, i) for i in range(N)])) <= RT
        assert np.abs(prob - np.stack([g["prob"][i] for i in range(N)])).max() <= PT
    finally:
        net.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pinned", [True, False], ids=["conv_ws_pinned", "unpinned"])
def test_vgg16_net_b256(pinned, qcnn, ctx, vgg):
    """Batch 256 on the default path: with force_kernel = 7 every conv layer runs conv_ws; unpinned, conv1_1 still does
    (its only GEMM) and the others run conv_ws or pq_gemm_tc mode 0 by timing.  Sampled images against the oracle."""
    import torch
    g = vgg
    N = NET_IMAGES
    RT, PT = MODES["default"]
    net = qcnn.Net(ctx, g["dir"], "vgg", "VGG16")
    try:
        if pinned:
            for l in VGG16_CONVS:
                net.pq_layer(l).set_param("tensor_core", 2)
                net.pq_layer(l).set_param("force_kernel", 7)
        imgd = torch.from_numpy(g["img"]).cuda()
        logits = torch.empty((N, 1000), dtype=torch.float32, device="cuda")
        prob = net.forward(imgd, logits=logits).cpu().numpy()
        for l in VGG16_CONVS:
            desc = net.pq_layer(l).describe(N)
            if pinned or l == 0:
                assert desc.startswith("pq_gemm_tc_ws(") and " mode=0 " in desc, (l, desc)
            else:
                assert (desc.startswith("pq_gemm_tc(") or desc.startswith("pq_gemm_tc_ws(")) and " mode=0 " in desc, (l, desc)
        lg = logits.cpu().numpy()
        for i in NET_SAMPLE:
            assert close(lg[i], _logits_ref(g, i)) <= RT, i
            assert np.abs(prob[i] - g["prob"][i]).max() <= PT, i
        del imgd
    finally:
        net.close()

