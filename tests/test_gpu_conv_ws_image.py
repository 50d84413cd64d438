"""conv_ws on stride-1 layers reads each k-step's decoded weights from the layer's weight image (qcnn_layer::d_w_ws, built
once at layer creation) through a ring of bulk-copied stage buffers.  Its accumulator chains the same k-steps in the same
order, on the same bf16x2 pieces, as pq_gemm_tc mode 0 with one accumulator (force_kernel = 6, 128 positions per CTA, no
K-split), which decodes its weights at use: the two outputs are compared bit for bit.

  - AlexNet conv2-conv5 at batch 1, 3 and 256, at every channel width the planner offers;
  - the stride-1 rows of test_gpu_conv_ws_s1.py with d = 4 / 12, Cg % 8 == 4, groups and 2, 3 or 6 channel tiles;
  - the weight ring: k-steps per stage pinned to 1, 2 and 5 (gemm_gt) on a 25-tap row with one channel tile (one copy
    per stage) and on a 9-tap row with six channel tiles (one copy per k-step and piece): many more stages than buffers,
    stages that end inside a chunk, and run-to-run bit identity."""
import numpy as np
import pytest

from test_gpu_conv_ws_s1 import BYNAME, Row, widths
from test_gpu_pq_gemm import bits, conv_data

ALEXNET = [Row("%s_n%d" % (name, N), N, *geo) for N in (1, 3, 256) for name, geo in (
    ("conv2", (27, 27, 96, 256, 5, 2, 1, 2, 6, 128, 8, False)),
    ("conv3", (13, 13, 256, 384, 3, 1, 1, 1, 32, 128, 8, False)),
    ("conv4", (13, 13, 384, 384, 3, 1, 1, 2, 24, 128, 8, False)),
    ("conv5", (13, 13, 384, 256, 3, 1, 1, 2, 24, 128, 8, False)))]
ODD = [BYNAME[n] for n in ("kg16_k1_pad0_d4", "kg32_k3_cg12_d12", "g2_kg64_k5_pad2_d4", "kg96_cg20_k3",
                           "kg192_k5_cg36_d12", "kg384_k3", "g3_kg48_k3_cg8")]
ROWS = {r.name: r for r in ALEXNET + ODD}


class _Cache(object):
    def __init__(self, qcnn, ctx):
        self.qcnn, self.ctx, self.items = qcnn, ctx, {}

    def get(self, row):
        if row.name not in self.items:
            import torch
            x, ctrd, asmt, bias = conv_data(row)
            L = self.qcnn.ConvLayer(self.ctx, row.Cin, row.Hi, row.Wi, row.Cout, row.k, row.pad, row.stride, row.G,
                                    ctrd, asmt, bias)
            self.items[row.name] = dict(L=L, xd=torch.from_numpy(x).cuda(), tc=None)
        return self.items[row.name]

    def close(self):
        for it in self.items.values():
            it["L"].close()


@pytest.fixture(scope="module")
def cache(qcnn, ctx):
    c = _Cache(qcnn, ctx)
    yield c
    c.close()


def set_pins(L, kernel, nt=0, gt=0, ct=0, nsplit=0):
    L.set_param("tensor_core", 2)
    L.set_param("force_kernel", kernel)
    L.set_param("gemm_nt", nt)
    L.set_param("gemm_gt", gt)
    L.set_param("gemm_ct", ct)
    L.set_param("gemm_nsplit", nsplit)


def decode_at_use(row, it):
    """pq_gemm_tc mode 0 with one accumulator: the bits conv_ws must reproduce (computed once per row)."""
    if it["tc"] is None:
        L = it["L"]
        set_pins(L, 6, nt=128, nsplit=1)
        y = L.forward(it["xd"]).cpu().numpy()
        desc = L.describe(row.N)
        assert desc.startswith("pq_gemm_tc(") and " mode=0 " in desc and "bf16x2" in desc, desc
        assert " NT=128 " in desc and " nsplit=1" in desc, desc
        it["tc"] = y
    return it["tc"]


def field(desc, name):
    return int(desc.split(" %s=" % name)[1].split()[0])


CASES = [pytest.param(r, W, id="%s-N%d" % (r.name, W)) for r in ALEXNET + ODD for W in widths(r)]


@pytest.mark.gpu
@pytest.mark.parametrize("row,W", CASES)
def test_conv_ws_image_bit_identical_to_decode_at_use(row, W, cache):
    it = cache.get(row)
    ref = decode_at_use(row, it)
    L = it["L"]
    set_pins(L, 7, ct=W)
    y = L.forward(it["xd"]).cpu().numpy()
    desc = L.describe(row.N)
    assert desc.startswith("pq_gemm_tc_ws(") and " mode=0 " in desc and " N=%d " % W in desc, desc
    assert 2 <= field(desc, "wbufs") <= 4, desc
    assert np.array_equal(bits(y), bits(ref)), (desc, int((bits(y) != bits(ref)).sum()))


RING = [pytest.param(ROWS[n], W, ks, id="%s-N%d-KS%d" % (n, W, ks))
        for n, W in (("kg192_k5_cg36_d12", 192), ("kg384_k3", 64)) for ks in (1, 2, 5)]


@pytest.mark.gpu
@pytest.mark.parametrize("row,W,ks", RING)
def test_conv_ws_weight_ring(row, W, ks, cache):
    it = cache.get(row)
    ref = decode_at_use(row, it)
    L = it["L"]
    set_pins(L, 7, gt=ks, ct=W)
    try:
        y = L.forward(it["xd"]).cpu().numpy()
        desc = L.describe(row.N)
        taps = row.k * row.k
        chunks = -(-(row.Cin // row.G) // 8)
        assert " KS=%d " % ks in desc and " N=%d " % W in desc, desc
        assert field(desc, "stages") == chunks * -(-taps // ks), desc
        assert field(desc, "stages") > field(desc, "wbufs"), desc
        assert np.array_equal(bits(y), bits(ref)), (desc, int((bits(y) != bits(ref)).sum()))
        y2 = L.forward(it["xd"]).cpu().numpy()
        assert np.array_equal(bits(y), bits(y2))
    finally:
        L.set_param("gemm_gt", 0)


@pytest.mark.gpu
def test_conv_ws_unmatched_ks_pin_fails(qcnn, cache):
    """A k-steps-per-stage pin longer than a chunk's taps leaves conv_ws no tiling: an error, not another tiling."""
    row = ROWS["conv3_n1"]
    L = cache.get(row)["L"]
    set_pins(L, 7, gt=10)
    try:
        with pytest.raises(qcnn.QcnnError):
            L.describe(row.N)
    finally:
        L.set_param("gemm_gt", 0)
