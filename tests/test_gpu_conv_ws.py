"""The weight-stationary tensor-core conv family (conv_ws, force_kernel = 7; describe() names it pq_gemm_tc_ws) against
the float64 reference of test_gpu_pq_gemm.py.

conv_ws runs strided layers over <= 4 input channels per group (the mode-1 geometry of pq_gemm_tc, i.e. conv1) with
bf16x2 operands as a GEMM with positions as M and the Cout/grp channels as N.  Each accumulator chains the same k-steps in
the same order as pq_gemm_tc mode 1 with one accumulator (two MMAs per k-step), so the bound is tc_bound(bf16x2, NT=128,
k-steps, nsplit=1).  Every case pins the family and the positions per CTA (gemm_nt = 256 or 128) and asserts the plan from
describe() after the forward.  Besides the bound: ReLU, run-to-run bit identity, neighbour poisoning (an image's output is
bit-identical whether the other images are 0 or NaN) and the exact write set (a NaN guard around the output stays
untouched and every element is written)."""
import collections
import ctypes

import numpy as np
import pytest

from test_gpu_pq_gemm import (_guarded_call, bits, conv_data, f64_err, mode1_counts, ref64, tc_bound)

Row = collections.namedtuple("Row", "name N Hi Wi Cin Cout k pad stride G S K d nchw")
ROWS = [
    # conv1 of AlexNet exactly (N = 96 channels, 11x11 / 4, Cg = 3)
    Row("conv1_n1", 1, 227, 227, 3, 96, 11, 0, 4, 1, 1, 128, 8, False),
    Row("conv1_n3", 3, 227, 227, 3, 96, 11, 0, 4, 1, 1, 128, 8, False),
    Row("conv1_n256", 256, 227, 227, 3, 96, 11, 0, 4, 1, 1, 128, 8, False),
    # channel widths, kernel sizes, strides, input channels, NCHW source, partial tiles
    Row("kg16_k3_s2_cg1_nchw", 5, 13, 12, 1, 16, 3, 1, 2, 1, 1, 16, 4, True),
    Row("kg128_k7_s2_cg4", 2, 21, 21, 4, 128, 7, 3, 2, 1, 1, 32, 4, False),
    Row("kg256_k11_s4_cg3", 2, 39, 39, 3, 256, 11, 0, 4, 1, 1, 128, 8, False),
    Row("kg64_k3_s2_cg4_tiny", 7, 9, 9, 4, 64, 3, 0, 2, 1, 1, 64, 8, False),
    # 8 and 4 k-steps per phase row (not multiples of 3), padding with stride 4, groups
    Row("kg96_k7_s4_cg1_pad2", 3, 29, 30, 1, 96, 7, 2, 4, 1, 1, 64, 4, False),
    Row("g2_kg96_k7_s4_cg1", 3, 29, 30, 2, 192, 7, 2, 4, 2, 1, 64, 4, False),
    Row("g2_kg32_k3_s4_cg3_nchw", 4, 17, 19, 6, 64, 3, 1, 4, 2, 1, 32, 4, True),
]
BYNAME = {r.name: r for r in ROWS}
# images of conv1_n256 the float64 reference is evaluated on: both ends, both sides of the middle, and a spread
REF_IMAGES = {"conv1_n256": sorted({0, 1, 2, 127, 128, 254, 255} | set(range(5, 256, 31)))}


def ksteps(row):
    return sum(mode1_counts(row.k, row.stride, True))


def tilings(row):
    """Positions per CTA the planner offers: 256 (two m64 blocks per warpgroup) needs Cout/grp <= 128."""
    return [256, 128] if row.Cout // row.G <= 128 else [128]


class _Cache(object):
    def __init__(self, qcnn, ctx):
        self.qcnn, self.ctx, self.items = qcnn, ctx, {}

    def get(self, row):
        if row.name not in self.items:
            import torch
            x, ctrd, asmt, bias = conv_data(row)
            L = self.qcnn.ConvLayer(self.ctx, row.Cin, row.Hi, row.Wi, row.Cout, row.k, row.pad, row.stride, row.G,
                                    ctrd, asmt, bias)
            L.set_src_nchw(row.nchw)
            sel = REF_IMAGES.get(row.name, list(range(row.N)))
            ref, mag = ref64("conv", x[sel], ctrd, asmt, bias, (row.pad, row.stride, row.G))
            xs = np.ascontiguousarray(x.transpose(0, 3, 1, 2)) if row.nchw else x
            self.items[row.name] = dict(L=L, x=x, xd=torch.from_numpy(xs).cuda(), sel=sel, ref=ref, mag=mag)
        return self.items[row.name]

    def close(self):
        for it in self.items.values():
            it["L"].close()


@pytest.fixture(scope="module")
def cache(qcnn, ctx):
    c = _Cache(qcnn, ctx)
    yield c
    c.close()


def pin(L, positions):
    L.set_param("tensor_core", 2)
    L.set_param("force_kernel", 7)
    L.set_param("gemm_nt", positions)
    L.set_param("gemm_gt", 0)
    L.set_param("gemm_nsplit", 0)


def assert_plan(desc, row, positions):
    assert desc.startswith("pq_gemm_tc_ws("), desc
    for f in ("N=%d" % (row.Cout // row.G), "positions=%d" % positions, "ksteps=%d" % ksteps(row)):
        assert " %s " % f in desc + " ", (f, desc)
    assert "bf16x2" in desc and " NT=" not in desc, desc


CASES = [pytest.param(r, P, id="%s-P%d" % (r.name, P)) for r in ROWS for P in tilings(r)]


@pytest.mark.gpu
@pytest.mark.parametrize("row,positions", CASES)
def test_conv_ws_f64(row, positions, cache):
    it = cache.get(row)
    L = it["L"]
    pin(L, positions)
    y = L.forward(it["xd"]).cpu().numpy()
    assert_plan(L.describe(row.N), row, positions)
    bound = tc_bound(True, 128, ksteps(row), 1)
    e = f64_err(y[it["sel"]], it["ref"], it["mag"])
    assert e <= bound, (e, bound)
    yr = L.forward(it["xd"], relu=True).cpu().numpy()
    er = f64_err(yr[it["sel"]], np.maximum(it["ref"], 0), it["mag"])
    assert er <= bound, (er, bound)
    y2 = L.forward(it["xd"]).cpu().numpy()
    assert np.array_equal(bits(y), bits(y2))


POISON = [pytest.param(BYNAME[n], P, id="%s-P%d" % (n, P))
          for n in ("conv1_n3", "kg64_k3_s2_cg4_tiny", "kg16_k3_s2_cg1_nchw", "g2_kg96_k7_s4_cg1", "g2_kg32_k3_s4_cg3_nchw")
          for P in tilings(BYNAME[n])]


@pytest.mark.gpu
@pytest.mark.parametrize("row,positions", POISON)
def test_conv_ws_neighbour_poison(row, positions, cache):
    """Image i's output is bit-identical whether every other image is 0 or NaN (tiles straddle image boundaries)."""
    import torch
    it = cache.get(row)
    L = it["L"]
    pin(L, positions)
    i = (row.N - 1) // 2
    outs = []
    for fill in (0.0, np.nan):
        xp = np.full_like(it["x"], fill)
        xp[i] = it["x"][i]
        if row.nchw:
            xp = np.ascontiguousarray(xp.transpose(0, 3, 1, 2))
        outs.append(L.forward(torch.from_numpy(xp).cuda()).cpu().numpy()[i])
    assert_plan(L.describe(row.N), row, positions)
    assert np.array_equal(bits(outs[0]), bits(outs[1]))
    assert f64_err(outs[0], it["ref"][it["sel"].index(i)], it["mag"][it["sel"].index(i)]) <= tc_bound(True, 128, ksteps(row), 1)


WRITE_SET = [pytest.param(BYNAME[n], P, id="%s-P%d" % (n, P))
             for n in ("conv1_n3", "kg16_k3_s2_cg1_nchw", "kg256_k11_s4_cg3", "kg96_k7_s4_cg1_pad2", "g2_kg96_k7_s4_cg1")
             for P in tilings(BYNAME[n])]


@pytest.mark.gpu
@pytest.mark.parametrize("row,positions", WRITE_SET)
def test_conv_ws_exact_write_set(row, positions, qcnn, cache):
    import torch
    it = cache.get(row)
    L = it["L"]
    pin(L, positions)
    ho, wo, co = L.out_dims()
    n_out = row.N * ho * wo * co
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    xd = it["xd"]
    for relu in (0, 1):
        out, guard_ok = _guarded_call(
            lambda dst, r: qcnn._check(qcnn.lib.qcnn_conv_aprx_forward(L.h, ctypes.c_void_p(xd.data_ptr()), row.N, dst,
                                                                       r, stream)), n_out, relu)
        assert_plan(L.describe(row.N), row, positions)
        assert guard_ok, relu
        assert np.isfinite(out).all(), (relu, int((~np.isfinite(out)).sum()))


@pytest.mark.gpu
def test_conv_ws_not_offered_for_3xtf32(qcnn, cache):
    """3xTF32 operands (tensor_core = 1) keep pq_gemm_tc mode 1: a conv_ws pin is an error, not a change of format."""
    row = BYNAME["conv1_n3"]
    L = cache.get(row)["L"]
    L.set_param("tensor_core", 1)
    L.set_param("force_kernel", 7)
    L.set_param("gemm_nt", 0)
    with pytest.raises(qcnn.QcnnError):
        L.describe(row.N)
    L.set_param("force_kernel", -1)
    assert L.describe(row.N).startswith("pq_gemm_tc("), L.describe(row.N)
