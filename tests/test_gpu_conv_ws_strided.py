"""conv_ws on strided layers (the mode-1 geometry, conv1): what the producers' phase-row staging and index decode add to
test_gpu_conv_ws.py.

Each producer thread holds its items of a phase row's planes (twelve float4 at most, st x NPOS <= 1536 per CTA, the
limit pq_gemm_tc mode 1 has as well) and reads its channel's index row of the phase row into registers when the row has
at most 48 taps, byte by byte at each k-step when it is longer.  The rows here sit on those limits: exactly 1536 items,
one layer too wide for 256 positions per CTA, index rows of 64 and 80 bytes (one with a second channel per thread), and
a VggCnnS-shaped 7 x 7 / 2 stem.  Every case checks the float64 bound of test_gpu_conv_ws.py, run-to-run bit identity,
neighbour poisoning and the exact write set.  conv1-shaped layers also give bit-identical outputs through conv_ws and
through pq_gemm_tc mode 1 with one accumulator (128 positions, no K-split): both chain the same k-steps in the same order.
"""
import ctypes

import numpy as np
import pytest

from test_gpu_conv_ws import Row, assert_plan, ksteps, pin, tilings
from test_gpu_pq_gemm import _guarded_call, bits, conv_data, f64_err, ref64, tc_bound

ROWS = [
    # 252 wide, 11 x 11 / 4: NPOS = 384 at 256 positions, 4 x 384 = 1536 items (every register of every producer)
    Row("items1536_k11_s4", 3, 23, 252, 3, 96, 11, 0, 4, 1, 1, 128, 8, True),
    # 256 wide: 1568 items at 256 positions (not offered), 1056 at 128
    Row("items1568_k11_s4", 2, 23, 256, 3, 96, 11, 0, 4, 1, 1, 128, 8, False),
    # VggCnnS conv1 geometry (7 x 7 / 2 over RGB, 224 wide): 1200 items at 256 positions
    Row("vggs_k7_s2", 2, 19, 224, 3, 96, 7, 0, 2, 1, 1, 128, 4, True),
    # index rows longer than 48 bytes: 11 x 11 / 2 (66 taps per phase row -> 80 bytes), 13 x 13 / 4 with groups, Cg = 4
    # and NCHW (52 -> 64), 10 x 10 / 2 at 256 channels (two channels per producer thread; 50 -> 64)
    Row("longrow80_k11_s2", 2, 31, 31, 3, 32, 11, 1, 2, 1, 1, 64, 4, False),
    Row("longrow64_g2_k13_s4_cg4_nchw", 3, 30, 30, 8, 64, 13, 2, 4, 2, 1, 64, 4, True),
    Row("longrow64_kg256_k10_s2_cg2", 2, 24, 24, 2, 256, 10, 0, 2, 1, 1, 32, 4, False),
]
BYNAME = {r.name: r for r in ROWS}
# 256 positions per CTA would stage more than 1536 items
NOT_OFFERED = {"items1568_k11_s4": 256}


class _Cache(object):
    def __init__(self, qcnn, ctx):
        self.qcnn, self.ctx, self.items = qcnn, ctx, {}

    def get(self, row, ref=True):
        if row.name not in self.items:
            import torch
            x, ctrd, asmt, bias = conv_data(row)
            L = self.qcnn.ConvLayer(self.ctx, row.Cin, row.Hi, row.Wi, row.Cout, row.k, row.pad, row.stride, row.G,
                                    ctrd, asmt, bias)
            L.set_src_nchw(row.nchw)
            it = dict(L=L, x=x, data=(ctrd, asmt, bias))
            it["xd"] = torch.from_numpy(self.src(row, x)).cuda()
            self.items[row.name] = it
        it = self.items[row.name]
        if ref and "ref" not in it:
            it["ref"], it["mag"] = ref64("conv", it["x"], *it["data"], (row.pad, row.stride, row.G))
        return it

    @staticmethod
    def src(row, x):
        return np.ascontiguousarray(x.transpose(0, 3, 1, 2)) if row.nchw else x

    def close(self):
        for it in self.items.values():
            it["L"].close()


@pytest.fixture(scope="module")
def cache(qcnn, ctx):
    c = _Cache(qcnn, ctx)
    yield c
    c.close()


CASES = [pytest.param(r, P, id="%s-P%d" % (r.name, P)) for r in ROWS for P in tilings(r) if NOT_OFFERED.get(r.name) != P]


@pytest.mark.gpu
@pytest.mark.parametrize("row,positions", CASES)
def test_conv_ws_strided_edges(row, positions, qcnn, cache):
    import torch
    it = cache.get(row)
    L = it["L"]
    pin(L, positions)
    bound = tc_bound(True, 128, ksteps(row), 1)
    y = L.forward(it["xd"]).cpu().numpy()
    assert_plan(L.describe(row.N), row, positions)
    e = f64_err(y, it["ref"], it["mag"])
    assert e <= bound, (e, bound)
    assert np.array_equal(bits(y), bits(L.forward(it["xd"]).cpu().numpy()))
    # neighbour poisoning: image i's output does not depend on whether the other images are 0 or NaN
    i = (row.N - 1) // 2
    outs = []
    for fill in (0.0, np.nan):
        xp = np.full_like(it["x"], fill)
        xp[i] = it["x"][i]
        outs.append(L.forward(torch.from_numpy(cache.src(row, xp)).cuda()).cpu().numpy()[i])
    assert np.array_equal(bits(outs[0]), bits(outs[1]))
    assert np.array_equal(bits(outs[0]), bits(y[i]))
    # exact write set: a NaN guard around the output stays untouched and every element is written
    ho, wo, co = L.out_dims()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    xd = it["xd"]
    for relu in (0, 1):
        out, guard_ok = _guarded_call(
            lambda dst, r: qcnn._check(qcnn.lib.qcnn_conv_aprx_forward(L.h, ctypes.c_void_p(xd.data_ptr()), row.N, dst,
                                                                       r, stream)), row.N * ho * wo * co, relu)
        assert guard_ok, relu
        assert np.isfinite(out).all(), (relu, int((~np.isfinite(out)).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("name,positions", sorted(NOT_OFFERED.items()))
def test_conv_ws_strided_too_many_items(name, positions, qcnn, cache):
    """A tiling whose phase row would stage more than 1536 items is not offered: a pin on it is an error."""
    row = BYNAME[name]
    L = cache.get(row, ref=False)["L"]
    pin(L, positions)
    with pytest.raises(qcnn.QcnnError):
        L.describe(row.N)


CONV1 = [pytest.param(N, nchw, id="N%d-%s" % (N, "nchw" if nchw else "nhwc"))
         for N, nchw in ((1, True), (3, True), (3, False), (256, True))]


@pytest.mark.gpu
@pytest.mark.parametrize("N,nchw", CONV1)
def test_conv_ws_conv1_equals_mode1(N, nchw, cache):
    """conv1 (227 x 227 x 3, 11 x 11 / 4, 96 channels) through conv_ws at 256 and 128 positions per CTA and through
    pq_gemm_tc mode 1 with one accumulator: bit-identical outputs."""
    row = Row("conv1_n%d_%s" % (N, "nchw" if nchw else "nhwc"), N, 227, 227, 3, 96, 11, 0, 4, 1, 1, 128, 8, nchw)
    it = cache.get(row, ref=False)
    L = it["L"]
    pin(L, 128)
    L.set_param("force_kernel", 6)
    L.set_param("gemm_nsplit", 1)
    want = L.forward(it["xd"]).cpu().numpy()
    desc = L.describe(N)
    assert desc.startswith("pq_gemm_tc(") and " mode=1 " in desc and " NT=128 " in desc, desc
    for positions in tilings(row):
        pin(L, positions)
        y = L.forward(it["xd"]).cpu().numpy()
        assert_plan(L.describe(N), row, positions)
        assert np.array_equal(bits(y), bits(want)), positions
