"""The weight-stationary tensor-core conv family (conv_ws, force_kernel = 7) on stride-1 layers (conv2-conv5 of AlexNet:
the mode-0 geometry of pq_gemm_tc) against the float64 reference of test_gpu_pq_gemm.py.

conv_ws runs a stride-1 layer with bf16x2 operands as a GEMM with positions as M and one tile of the Cout/grp channels as
N (gemm_ct: 16 ... 256 channels, 192 included, Cout/grp = ctiles x N).  Each accumulator chains the same k-steps in the
same order as pq_gemm_tc mode 0 with one accumulator (two MMAs per k-step, chunks x taps k-steps), so the bound is
tc_bound(bf16x2, NT=128, chunks x taps, nsplit=1).  Every case pins the family, the positions per CTA (gemm_nt = 256 or
128) and the channels per CTA, and asserts the plan from describe() after the forward.  Besides the bound: ReLU, run-to-run
bit identity, neighbour poisoning (an image's output is bit-identical whether the other images are 0 or NaN), the exact
write set (a NaN guard around the output stays untouched and every element is written), the layers the family does not
take, and AlexNet at batch 256 with conv2-conv5 pinned to it against the CPU oracle."""
import collections
import ctypes

import numpy as np
import pytest

from test_gpu_layers import close
from test_gpu_net import MODES
from test_gpu_parity_b256 import alexnet_b256  # noqa: F401  (module-scoped fixture: model files, images, oracle maps)
from test_gpu_pq_gemm import _guarded_call, bits, conv_data, f64_err, ref64, tc_bound

Row = collections.namedtuple("Row", "name N Hi Wi Cin Cout k pad stride G S K d nchw")
ROWS = [
    # conv2-conv5 of AlexNet exactly, at the benchmarked batch and at batch 1-3
    Row("conv2_n256", 256, 27, 27, 96, 256, 5, 2, 1, 2, 6, 128, 8, False),
    Row("conv3_n256", 256, 13, 13, 256, 384, 3, 1, 1, 1, 32, 128, 8, False),
    Row("conv4_n256", 256, 13, 13, 384, 384, 3, 1, 1, 2, 24, 128, 8, False),
    Row("conv5_n256", 256, 13, 13, 384, 256, 3, 1, 1, 2, 24, 128, 8, False),
    Row("conv2_n1", 1, 27, 27, 96, 256, 5, 2, 1, 2, 6, 128, 8, False),
    Row("conv3_n2", 2, 13, 13, 256, 384, 3, 1, 1, 1, 32, 128, 8, False),
    Row("conv4_n3", 3, 13, 13, 384, 384, 3, 1, 1, 2, 24, 128, 8, False),
    Row("conv5_n1", 1, 13, 13, 384, 256, 3, 1, 1, 2, 24, 128, 8, False),
    # widths, kernel sizes 1 / 3 / 5 with pad 0 / 1 / 2, d = 4 / 8 / 12, Cg % 8 == 4, groups, channel tiles
    Row("kg16_k1_pad0_d4", 5, 9, 9, 8, 16, 1, 0, 1, 1, 2, 64, 4, False),        # halves in different subspaces
    Row("kg32_k3_cg12_d12", 3, 10, 11, 12, 32, 3, 1, 1, 1, 1, 32, 12, False),   # Cg % 8 == 4; pieces 0-2 of one subspace
    Row("g2_kg64_k5_pad2_d4", 2, 12, 10, 16, 128, 5, 2, 1, 2, 2, 128, 4, False),
    Row("kg96_cg20_k3", 4, 8, 8, 20, 96, 3, 1, 1, 1, 3, 64, 8, False),           # Cg % 8 == 4 over three chunks
    Row("kg192_k5_cg36_d12", 2, 9, 7, 36, 192, 5, 2, 1, 1, 3, 128, 12, False),  # 25 taps: stages split a chunk
    Row("tiny_kg256_pad2", 40, 3, 3, 16, 256, 3, 2, 1, 1, 4, 16, 4, False),     # 25-position images: tiles span many
    Row("kg384_k3", 3, 7, 9, 32, 384, 3, 1, 1, 1, 4, 64, 8, False),              # 3 x 128, 2 x 192, 4 x 96, 6 x 64
    Row("g3_kg48_k3_cg8", 2, 6, 6, 24, 144, 3, 1, 1, 3, 1, 256, 8, False),      # 3 x 16-channel tiles per group
]
BYNAME = {r.name: r for r in ROWS}
# images of the batch-256 rows the float64 reference is evaluated on: both ends, both sides of the middle, and a spread
REF_IMAGES = {r.name: sorted({0, 1, 2, 127, 128, 254, 255} | set(range(5, 256, 31))) for r in ROWS if r.N == 256}

WIDTHS = (16, 32, 64, 96, 128, 192, 256)


def widths(row):
    """Channels per CTA the planner offers: instantiated divisors of Cout/grp from 64 up, else the widest divisor."""
    kg = row.Cout // row.G
    ds = [w for w in WIDTHS if kg % w == 0]
    return [w for w in ds if w >= 64 or w == ds[-1]]


def positions(width):
    """Positions per CTA: 256 (two m64 blocks per warpgroup) needs <= 128 channels per CTA."""
    return [256, 128] if width <= 128 else [128]


def ksteps(row):
    return -(-(row.Cin // row.G) // 8) * row.k * row.k


class _Cache(object):
    def __init__(self, qcnn, ctx):
        self.qcnn, self.ctx, self.items = qcnn, ctx, {}

    def get(self, row):
        if row.name not in self.items:
            import torch
            x, ctrd, asmt, bias = conv_data(row)
            L = self.qcnn.ConvLayer(self.ctx, row.Cin, row.Hi, row.Wi, row.Cout, row.k, row.pad, row.stride, row.G,
                                    ctrd, asmt, bias)
            sel = REF_IMAGES.get(row.name, list(range(row.N)))
            ref, mag = ref64("conv", x[sel], ctrd, asmt, bias, (row.pad, row.stride, row.G))
            self.items[row.name] = dict(L=L, x=x, xd=torch.from_numpy(x).cuda(), sel=sel, ref=ref, mag=mag)
        return self.items[row.name]

    def close(self):
        for it in self.items.values():
            it["L"].close()


@pytest.fixture(scope="module")
def cache(qcnn, ctx):
    c = _Cache(qcnn, ctx)
    yield c
    c.close()


def pin(L, P, W):
    L.set_param("tensor_core", 2)
    L.set_param("force_kernel", 7)
    L.set_param("gemm_nt", P)
    L.set_param("gemm_ct", W)
    L.set_param("gemm_gt", 0)
    L.set_param("gemm_nsplit", 0)


def unpin(L):
    for name in ("force_kernel", "gemm_nt", "gemm_ct"):
        L.set_param(name, -1 if name == "force_kernel" else 0)


def assert_plan(desc, row, P, W):
    assert desc.startswith("pq_gemm_tc_ws("), desc
    kg = row.Cout // row.G
    for f in ("mode=0", "N=%d" % W, "positions=%d" % P, "ctiles=%d" % (kg // W), "ksteps=%d" % ksteps(row)):
        assert " %s " % f in desc + " ", (f, desc)
    assert "bf16x2" in desc and "NT=" not in desc, desc
    grid = -(-row.N * (row.Hi + row.pad) * (row.Wi + row.pad) // P) * row.G * (kg // W)
    assert " grid=%d " % grid in desc, (grid, desc)


def _cases(rows, all_widths=True):
    out = []
    for r in rows:
        ws = widths(r) if all_widths else widths(r)[-1:]
        out += [pytest.param(r, P, W, id="%s-P%d-N%d" % (r.name, P, W)) for W in ws for P in positions(W)]
    return out


CASES = _cases([r for r in ROWS if r.N == 256 or not r.name.startswith("conv")]) + \
    _cases([r for r in ROWS if r.N < 256 and r.name.startswith("conv")], all_widths=False)


@pytest.mark.gpu
@pytest.mark.parametrize("row,P,W", CASES)
def test_conv_ws_s1_f64(row, P, W, cache):
    it = cache.get(row)
    L = it["L"]
    pin(L, P, W)
    y = L.forward(it["xd"]).cpu().numpy()
    assert_plan(L.describe(row.N), row, P, W)
    bound = tc_bound(True, 128, ksteps(row), 1)
    e = f64_err(y[it["sel"]], it["ref"], it["mag"])
    assert e <= bound, (e, bound)
    yr = L.forward(it["xd"], relu=True).cpu().numpy()
    er = f64_err(yr[it["sel"]], np.maximum(it["ref"], 0), it["mag"])
    assert er <= bound, (er, bound)
    y2 = L.forward(it["xd"]).cpu().numpy()
    assert np.array_equal(bits(y), bits(y2))


POISON = [pytest.param(BYNAME[n], P, W, id="%s-P%d-N%d" % (n, P, W))
          for n, W in (("conv4_n3", 192), ("kg32_k3_cg12_d12", 32), ("tiny_kg256_pad2", 256), ("tiny_kg256_pad2", 128),
                       ("kg96_cg20_k3", 96), ("g2_kg64_k5_pad2_d4", 64))
          for P in positions(W)]


@pytest.mark.gpu
@pytest.mark.parametrize("row,P,W", POISON)
def test_conv_ws_s1_neighbour_poison(row, P, W, cache):
    """Image i's output is bit-identical whether every other image is 0 or NaN (tiles straddle image boundaries)."""
    import torch
    it = cache.get(row)
    L = it["L"]
    pin(L, P, W)
    i = (row.N - 1) // 2
    outs = []
    for fill in (0.0, np.nan):
        xp = np.full_like(it["x"], fill)
        xp[i] = it["x"][i]
        outs.append(L.forward(torch.from_numpy(xp).cuda()).cpu().numpy()[i])
    assert_plan(L.describe(row.N), row, P, W)
    assert np.array_equal(bits(outs[0]), bits(outs[1]))
    assert f64_err(outs[0], it["ref"][it["sel"].index(i)], it["mag"][it["sel"].index(i)]) <= tc_bound(True, 128, ksteps(row), 1)


WRITE_SET = [pytest.param(BYNAME[n], P, W, id="%s-P%d-N%d" % (n, P, W))
             for n, W in (("kg16_k1_pad0_d4", 16), ("kg384_k3", 192), ("kg384_k3", 64), ("tiny_kg256_pad2", 256),
                          ("g3_kg48_k3_cg8", 16), ("conv2_n1", 128))
             for P in positions(W)]


@pytest.mark.gpu
@pytest.mark.parametrize("row,P,W", WRITE_SET)
def test_conv_ws_s1_exact_write_set(row, P, W, qcnn, cache):
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
def test_conv_ws_s1_not_offered_for_3xtf32(qcnn, cache):
    """3xTF32 operands (tensor_core = 1) keep pq_gemm_tc mode 0: a conv_ws pin is an error, not a change of format."""
    row = BYNAME["kg32_k3_cg12_d12"]
    L = cache.get(row)["L"]
    L.set_param("tensor_core", 1)
    L.set_param("force_kernel", 7)
    L.set_param("gemm_nt", 0)
    L.set_param("gemm_ct", 0)
    with pytest.raises(qcnn.QcnnError):
        L.describe(row.N)
    unpin(L)
    desc = L.describe(row.N)
    assert desc.startswith("pq_gemm_tc(") and " mode=0 " in desc and "bf16x2" not in desc, desc


@pytest.mark.gpu
@pytest.mark.parametrize("what", ["nchw_source", "d6"])
def test_conv_ws_s1_ineligible(what, qcnn, ctx):
    """An NCHW source or d % 4 != 0 on a stride-1 layer: the NCHW source is refused when it is set; with d % 4 != 0 a
    conv_ws pin is an error and, unpinned, the layer keeps a LUT + gather family (pq_gemm_tc mode 0 does not take it
    either)."""
    import torch
    if what == "nchw_source":
        row = Row("nchw", 2, 9, 9, 16, 64, 3, 1, 1, 1, 2, 64, 8, True)
    else:
        row = Row("d6", 2, 9, 9, 12, 64, 3, 1, 1, 1, 2, 64, 6, False)
    x, ctrd, asmt, bias = conv_data(row)
    L = qcnn.ConvLayer(ctx, row.Cin, row.Hi, row.Wi, row.Cout, row.k, row.pad, row.stride, row.G, ctrd, asmt, bias)
    try:
        if row.nchw:
            # a stride-1 layer refuses an NCHW source outright: conv_ws (like pq_gemm_tc mode 0) never sees one
            with pytest.raises(qcnn.QcnnError):
                L.set_src_nchw(True)
            return
        pin(L, 0, 0)
        with pytest.raises(qcnn.QcnnError):
            L.describe(row.N)
        unpin(L)
        y = L.forward(torch.from_numpy(x).cuda()).cpu().numpy()
        desc = L.describe(row.N)
        assert not desc.startswith("pq_gemm_tc"), desc
        ref, mag = ref64("conv", x, ctrd, asmt, bias, (row.pad, row.stride, row.G))
        assert f64_err(y, ref, mag) <= 1e-5, desc
    finally:
        L.close()


@pytest.mark.gpu
def test_conv_ws_s1_unpinned_runs_a_gemm(cache):
    """Without a pin an eligible stride-1 layer at bf16x2 runs one of the two GEMMs of its geometry (timing chooses)."""
    row = BYNAME["conv5_n256"]
    it = cache.get(row)
    L = it["L"]
    L.set_param("tensor_core", 2)
    unpin(L)
    y = L.forward(it["xd"]).cpu().numpy()
    desc = L.describe(row.N)
    assert (desc.startswith("pq_gemm_tc(") or desc.startswith("pq_gemm_tc_ws(")) and " mode=0 " in desc, desc
    assert f64_err(y[it["sel"]], it["ref"], it["mag"]) <= tc_bound(True, 128, ksteps(row), 1), desc


@pytest.mark.gpu
def test_alexnet_b256_conv2_5_pinned(qcnn, ctx, alexnet_b256):  # noqa: F811
    """AlexNet at batch 256 with conv2-conv5 pinned to conv_ws: the feature maps of the kept images up to the logits, the
    logits and the probabilities within the default path's tolerance of the CPU oracle."""
    import torch
    g = alexnet_b256
    N = 256
    RT, PT = MODES["default"]
    net = qcnn.Net(ctx, g["dirpath"], g["pfx"], "AlexNet")
    try:
        for l in (4, 8, 10, 12):
            pl = net.pq_layer(l)
            pl.set_param("tensor_core", 2)
            pl.set_param("force_kernel", 7)
        imgd = torch.from_numpy(g["img"]).cuda()
        logits = torch.empty((N, 1000), dtype=torch.float32, device="cuda")
        net.forward(imgd)      # tilings of this batch size are timed here; describe() then reports the plans that run
        for l in (4, 8, 10, 12):
            desc = net.pq_layer(l).describe(N)
            assert desc.startswith("pq_gemm_tc_ws(") and " mode=0 " in desc, (l, desc)
        net.set_keep_maps(True)
        prob = net.forward(imgd, logits=logits).cpu().numpy()
        for l in range(23):    # (the softmax output, map 23, is checked through the probabilities below)
            fm = net.featmap(l, N).cpu().numpy()
            ref = np.stack([g["maps"][i][l].reshape(fm.shape[1:]) for i in g["keep"]])
            assert close(fm[g["keep"]], ref) <= RT, l
        assert close(logits.cpu().numpy(), g["logits"]) <= RT
        assert np.abs(prob - g["prob"]).max() <= PT
    finally:
        net.close()
