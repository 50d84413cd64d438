"""conv_ws's weight image and its weight ring, in both geometries.

conv_ws reads each k-step's decoded weights from the layer's weight image (qcnn_layer::d_w_ws, [grp][entry][w1, w2][Kg]
16-byte rows, built once at layer creation) and streams stages of KS k-steps into a ring of nWB = 2-4 shared-memory
buffers by bulk copy.  Every tiling (positions P, channels per CTA N, KS, nWB) chains the same k-steps in the same order,
on the same bf16x2 pieces, as pq_gemm_tc with one accumulator (force_kernel = 6, 128 positions per CTA, no K-split; mode 0
at stride 1, mode 1 on strided layers), which decodes its weights at use: all of them are compared bit for bit.  Where
pq_gemm_tc has no such tiling (stride-1 groups of <= 3 channels, index rows longer than it stages) every tiling is
compared with the first, and that one with the float64 bound.

  - the image, byte for byte: a numpy build of it from the codebook and assignments as ConvLayer receives them, checked
    against the float64 weights without a GPU and against read_w_ws() on one;
  - the sweep: a Python mirror of the planners' tiling space (MapWsSmem and the fit rules of PlanConvWsS1 / PlanConvWs)
    and, per row, every (P, N, nWB) with every KS that fits (at batch 256 a subset: 1, 2, a KS leaving a one-k-step
    remainder, a divisor, the default), pinned with gemm_nt / gemm_ct / gemm_gt / gemm_wb; describe() must show the
    mirror's carve, and pins outside the space must fail;
  - phase rows without k-steps (ksz < stride) get no weight stage;
  - at the ring's extremes (KS = 1 over 2 and 3 buffers, the default KS over 3): neighbour poisoning, the exact write set,
    ReLU and run-to-run bit identity.
Large outputs are compared on the device."""
import ctypes

import numpy as np
import pytest

from test_gpu_conv_ws import BYNAME as STRIDED
from test_gpu_conv_ws_s1 import BYNAME, Row, widths
from test_gpu_conv_ws_strided import BYNAME as STRIDED_EDGES
from test_gpu_pq_gemm import (H100_SMS, _guarded_call, _seed, bits, conv_data, decode_conv_weights, f64_err, mode1_counts,
                              ref64, split_bf16, tc_bound, tc_space)
from test_gpu_vgg16 import BYNAME as VGG

ALEXNET = [Row("%s_n%d" % (name, N), N, *geo) for N in (1, 3, 256) for name, geo in (
    ("conv2", (27, 27, 96, 256, 5, 2, 1, 2, 6, 128, 8, False)),
    ("conv3", (13, 13, 256, 384, 3, 1, 1, 1, 32, 128, 8, False)),
    ("conv4", (13, 13, 384, 384, 3, 1, 1, 2, 24, 128, 8, False)),
    ("conv5", (13, 13, 384, 256, 3, 1, 1, 2, 24, 128, 8, False)))]
ODD = [BYNAME[n] for n in ("kg16_k1_pad0_d4", "kg32_k3_cg12_d12", "g2_kg64_k5_pad2_d4", "kg96_cg20_k3",
                           "kg192_k5_cg36_d12", "kg384_k3", "g3_kg48_k3_cg8")]
CONV1 = [Row("conv1_n3_nchw", 3, 227, 227, 3, 96, 11, 0, 4, 1, 1, 128, 8, True), STRIDED["conv1_n3"],
         Row("conv1_n256_nchw", 256, 227, 227, 3, 96, 11, 0, 4, 1, 1, 128, 8, True)]
# strided layers whose trailing phase rows have no k-steps: 2 x 2 / 4 (rows 2 and 3), 1 x 1 / 2 (one k-step, row 1)
EMPTY_ROWS = [Row("k2_s4_pad1_cg3", 3, 18, 21, 3, 32, 2, 1, 4, 1, 1, 64, 4, False),
              Row("k1_s2_cg4", 4, 11, 13, 4, 64, 1, 0, 2, 1, 1, 32, 4, False)]
VGG_KG512 = Row("vgg_conv5_kg512", 1, 14, 14, 512, 512, 3, 1, 1, 1, 64, 128, 8, False)
ROWS = {r.name: r for r in ALEXNET + ODD + CONV1 + EMPTY_ROWS + [VGG_KG512, BYNAME["tiny_kg256_pad2"]]}
ROWS.update({n: r for n, r in list(STRIDED.items()) + list(STRIDED_EDGES.items()) + list(VGG.items())
             if n in ("kg96_k7_s4_cg1_pad2", "g2_kg32_k3_s4_cg3_nchw", "vggs_k7_s2", "longrow80_k11_s2",
                      "conv1_n1", "cg3_k5_pad2")})


def _ceil(a, b):
    return -(-a // b)


def _rup(a, b):
    return _ceil(a, b) * b


# ------------------------------------------------------------------------------------------------------------------
# the weight image in numpy
# ------------------------------------------------------------------------------------------------------------------
def layer_params(row):
    """(ctrd, asmt, bias) of conv_data(row) without its input (the same draws of the same generator)."""
    rng = np.random.RandomState(_seed(row.name))
    fan = (row.Cin // row.G) * row.k * row.k
    ctrd = (rng.randn(row.S, row.K, row.d) / np.sqrt(fan)).astype(np.float32)
    asmt = rng.randint(0, row.K, size=(row.Cout, row.k, row.k, row.S)).astype(np.uint8)
    bias = (rng.randn(row.Cout) * 0.1).astype(np.float32)
    return ctrd, asmt, bias


def mode1_entries(k, st):
    """The k-steps of a strided layer per phase row, in Mode1Table's order (bf16x2 pairing): [[(kh, kw, paired)]]."""
    rows = []
    for ph in range(st):
        ents = []
        for kh in range(ph, k, st):
            kw = 0
            while kw < k:
                paired = kw + 1 < k and (kw % st) + 1 < st and not ((kw % st) & 1)
                ents.append((kh, kw, paired))
                kw += 2 if paired else 1
        rows.append(ents)
    assert [len(e) for e in rows] == mode1_counts(k, st, True)
    return rows


def ws_image(row, ctrd, asmt):
    """The weight image as uint16 bf16 bit patterns [G, entries, {w1, w2}, Kg, 8]: per entry and channel the two
    4-value halves of the k-step (stride 1: input channels 8 kc + 0-3 and + 4-7 of tap t, each from its own subspace and
    piece; strided: a tap and its paired tap), split w = w1 + w2 as the codebook's bf16 pieces; a half the k-step does
    not have is 0."""
    S, K, d = ctrd.shape
    G, Cg, Kg, k = row.G, row.Cin // row.G, row.Cout // row.G, row.k
    w1, w2 = split_bf16(ctrd)
    pieces = (np.stack([w1, w2]).view(np.uint32) >> 16).astype(np.uint16)   # [2, S, K, d]
    A = asmt.reshape(G, Kg, k * k, S)
    if row.stride == 1:
        nch, taps = _ceil(Cg, 8), k * k
        img = np.zeros((G, nch, taps, 2, Kg, 8), np.uint16)
        for kc in range(nch):
            for h, ch in enumerate((8 * kc, 8 * kc + 4)):
                if ch >= Cg:
                    continue
                s, j = divmod(ch, d)
                vals = pieces[:, s][:, A[..., s]][..., j:j + 4]                 # [2, G, Kg, taps, 4]
                img[:, kc, :, :, :, 4 * h:4 * h + 4] = vals.transpose(1, 3, 0, 2, 4)
        return img.reshape(G, nch * taps, 2, Kg, 8)
    ents = [e for r in mode1_entries(k, row.stride) for e in r]
    img = np.zeros((G, len(ents), 2, Kg, 8), np.uint16)
    for e, (kh, kw, paired) in enumerate(ents):
        for h, tw in enumerate((kw, kw + 1) if paired else (kw,)):
            vals = pieces[:, 0][:, A[:, :, kh * k + tw, 0]][..., 0:4]               # [2, G, Kg, 4]
            img[:, e, :, :, 4 * h:4 * h + 4] = vals.transpose(1, 0, 2, 3)
    return img


def image_weights(img):
    """float64 w1 + w2 of every value of an image [G, entries, Kg, 8]."""
    f = (img.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    return f[:, :, 0] + f[:, :, 1]


# ------------------------------------------------------------------------------------------------------------------
# the tiling space (mirror of MapWsSmem, PlanConvWsS1 and PlanConvWs)
# ------------------------------------------------------------------------------------------------------------------
_SMEM = []


def smem_optin():
    """Dynamic shared memory a block may opt in to: the device's, else the H100's 227 KB (as SmemOptin)."""
    if not _SMEM:
        v = 0
        try:
            import torch
            if torch.cuda.is_available():
                v = getattr(torch.cuda.get_device_properties(0), "shared_memory_per_block_optin", 0)
        except Exception:
            v = 0
        _SMEM.append(v or 227 * 1024)
    return _SMEM[0]


def carve(P, NC, KS, nWB, nPB, planeRows):
    """MapWsSmem(...).total: plane buffers, weight buffers, output offsets, bias, mbarriers."""
    return nPB * 2 * planeRows * 16 + nWB * KS * 2 * NC * 16 + P * 4 + NC * 4 + 8 * (2 * nPB + 2 * nWB)


class Tiling(object):
    """One (P, N, nWB) of a row: the KS that fit (1 .. ksmax), the default KS and the carve of each."""

    def __init__(self, row, P, W, nWB, lim):
        self.row, self.P, self.W, self.nWB = row, P, W, nWB
        k, st = row.k, row.stride
        if st == 1:
            PW = row.Wi + row.pad
            self.NPOS = _rup(P + (k - 1) * (PW + 1), 8)
            self.counts = [k * k] * _ceil(row.Cin // row.G, 8)
            self.planeRows, nPBs = self.NPOS, (3, 2)
        else:
            PWp = _ceil(row.Wi + 2 * row.pad, st)
            self.NPOS = _rup(P + ((k - 1) // st) * (PWp + 1), 8)
            self.counts = mode1_counts(k, st, True)
            self.planeRows, nPBs = (st // 2) * self.NPOS, (st,)
        self.nPB = {}
        for KS in range(1, max(self.counts) + 1):
            fit = [n for n in nPBs if carve(P, W, KS, nWB, n, self.planeRows) <= lim]
            if fit:
                self.nPB[KS] = fit[0]
        self.ksmax = max(self.nPB) if self.nPB else 0
        if st == 1:   # the fewest equal stages that fit
            taps = k * k
            self.default = next((_ceil(taps, s) for s in range(1, taps + 1) if _ceil(taps, s) in self.nPB), 0)
        else:         # the largest count that fits
            self.default = self.ksmax

    def smem(self, KS):
        return carve(self.P, self.W, KS, self.nWB, self.nPB[KS], self.planeRows)

    def stages(self, KS):
        return sum(_ceil(c, KS) for c in self.counts)

    def ks_subset(self):
        """KS 1, 2, the largest leaving a one-k-step remainder in some chunk, the largest divisor of every non-empty
        chunk's count, and the default."""
        cs = [c for c in self.counts if c]
        rng = range(2, self.ksmax + 1)
        rem1 = [ks for ks in rng if any(c % ks == 1 for c in cs)]
        div = [ks for ks in rng if all(c % ks == 0 for c in cs) and ks != self.default]
        return sorted({1, min(2, self.ksmax), self.default} | set(rem1[-1:]) | set(div[-1:]))


def strided_tile_fits(row, P):
    st = row.stride
    PWp, PHp = _ceil(row.Wi + 2 * row.pad, st), _ceil(row.Hi + 2 * row.pad, st)
    NPOS = _rup(P + ((row.k - 1) // st) * (PWp + 1), 8)
    return st * NPOS <= 1536 and (_ceil(NPOS, PHp * PWp) + 1) * row.Hi * row.Wi * row.Cin <= 2.0e9


def space(row, only_widths=None):
    """Every (P, N, nWB) tiling the planner offers for row (those with at least one KS that fits)."""
    lim, Kg, out = smem_optin(), row.Cout // row.G, []
    if row.stride == 1:
        pw = [(P, W) for W in widths(row) for P in ((256, 128) if W <= 128 else (128,))]
    else:
        pw = [(P, Kg) for P in (256, 128) if (P == 128 or Kg <= 128) and strided_tile_fits(row, P)]
    for P, W in pw:
        if only_widths and W not in only_widths:
            continue
        for nWB in (4, 3, 2):
            t = Tiling(row, P, W, nWB, lim)
            if t.ksmax:
                out.append(t)
    return out


def test_mirror_reproduces_conv1_ring_depths():
    """conv1 (Kg = 96, 11 x 11 / 4, counts 18 / 18 / 18 / 12) at 227 KB: the mirror's default KS per ring depth."""
    if smem_optin() != 227 * 1024:
        pytest.skip("device opt-in limit is not 227 KB")
    row = ROWS["conv1_n3_nchw"]
    got = {(t.P, t.nWB): t.default for t in space(row)}
    assert got == {(256, 4): 10, (256, 3): 14, (256, 2): 18, (128, 4): 13, (128, 3): 18, (128, 2): 18}, got


# ------------------------------------------------------------------------------------------------------------------
# CPU: the numpy image against the float64 weights
# ------------------------------------------------------------------------------------------------------------------
IMAGE_ROWS = sorted({n for n in ROWS if not n.endswith("_n256")} | {"conv2_n256", "conv1_n256_nchw"})


@pytest.mark.parametrize("name", IMAGE_ROWS)
def test_image_builder_reproduces_decoded_weights(name):
    """Summing each image row's bf16 pieces back per (channel, tap, input channel) gives decode_conv_weights to within
    the bf16x2 split (|w - w1 - w2| <= 2^-17 |w|); every half a k-step does not have is exactly 0."""
    row = ROWS[name]
    ctrd, asmt, _ = layer_params(row)
    G, Cg, Kg, k = row.G, row.Cin // row.G, row.Cout // row.G, row.k
    W = decode_conv_weights(ctrd, asmt, Cg).reshape(G, Kg, k * k, Cg)
    img = ws_image(row, ctrd, asmt)
    v = image_weights(img)                                           # [G, entries, Kg, 8]
    if row.stride == 1:
        nch = _ceil(Cg, 8)
        assert img.shape == (G, nch * k * k, 2, Kg, 8)
        got = v.reshape(G, nch, k * k, Kg, 8).transpose(0, 3, 2, 1, 4).reshape(G, Kg, k * k, nch * 8)[..., :Cg]
        for kc in range(nch):
            if 8 * kc + 4 >= Cg:
                assert not img.reshape(G, nch, k * k, 2, Kg, 8)[:, kc, ..., 4:].any(), kc
    else:
        ents = [e for r in mode1_entries(k, row.stride) for e in r]
        assert img.shape == (G, len(ents), 2, Kg, 8)
        got = np.full(W.shape, np.nan)
        for e, (kh, kw, paired) in enumerate(ents):
            for h, tw in enumerate((kw, kw + 1) if paired else (kw,)):
                assert np.isnan(got[:, :, kh * k + tw, 0]).all(), (kh, tw)   # every tap once
                got[:, :, kh * k + tw] = v[:, e, :, 4 * h:4 * h + Cg]
            if not paired:
                assert not img[:, e, :, :, 4:].any(), e
        assert not np.isnan(got).any()
    assert (np.abs(got - W) <= 2.0 ** -17 * np.abs(W)).all(), float((np.abs(got - W) / np.maximum(np.abs(W), 1e-30)).max())


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
class _Cache(object):
    def __init__(self, qcnn, ctx):
        self.qcnn, self.ctx, self.items = qcnn, ctx, {}

    def get(self, row, data=True):
        if row.name not in self.items:
            ctrd, asmt, bias = layer_params(row)
            L = self.qcnn.ConvLayer(self.ctx, row.Cin, row.Hi, row.Wi, row.Cout, row.k, row.pad, row.stride, row.G,
                                    ctrd, asmt, bias)
            L.set_src_nchw(row.nchw)
            self.items[row.name] = dict(L=L, params=(ctrd, asmt, bias), ref=None)
        it = self.items[row.name]
        if data and "x" not in it:
            import torch
            it["x"] = conv_data(row)[0]
            it["xd"] = torch.from_numpy(self.src(row, it["x"])).cuda()
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


def set_pins(L, kernel, nt=0, gt=0, ct=0, nsplit=0, wb=0):
    L.set_param("tensor_core", 2)
    L.set_param("force_kernel", kernel)
    for name, v in (("gemm_nt", nt), ("gemm_gt", gt), ("gemm_ct", ct), ("gemm_nsplit", nsplit), ("gemm_wb", wb)):
        L.set_param(name, v)


def field(desc, name):
    return int(desc.split(" %s=" % name)[1].split()[0].rstrip("B"))


def as_bits(y):
    """int32 view of a float32 device tensor (bitwise torch.equal)."""
    import torch
    return y.contiguous().view(torch.int32)


def bit_mismatches(a, b):
    return int((as_bits(a) != as_bits(b)).sum().item())


def twin_free(row):
    """pq_gemm_tc has no bf16x2 tiling of 128 positions without a K-split for the layer (mirror of PlanPqGemm's
    eligibility): stride-1 groups of <= 3 channels, and strided layers whose index rows are longer than it stages
    (ceil(k / stride) x ceil(k / 2) > 32 bytes, e.g. 11 x 11 / 2)."""
    return not any(NT == 128 and ns == 1 for NT, _, ns, _ in tc_space(row, True, H100_SMS))


def reference(row, it):
    """The bits every conv_ws tiling of row must produce, on the device (computed once per row): pq_gemm_tc with one
    accumulator, or, without a twin, the first tiling of the space checked against the float64 bound."""
    if it["ref"] is None:
        L = it["L"]
        if twin_free(row):
            t = space(row)[0]
            set_pins(L, 7, nt=t.P, ct=t.W, wb=t.nWB)
            y = L.forward(it["xd"])
            assert L.describe(row.N).startswith("pq_gemm_tc_ws(")
            ref, mag = ref64("conv", it["x"], *it["params"], (row.pad, row.stride, row.G))
            ksteps = sum(t.counts)
            assert f64_err(y.cpu().numpy(), ref, mag) <= tc_bound(True, 128, ksteps, 1)
        else:
            set_pins(L, 6, nt=128, nsplit=1)
            y = L.forward(it["xd"])
            desc = L.describe(row.N)
            assert desc.startswith("pq_gemm_tc(") and " mode=%d " % (row.stride > 1) in desc and "bf16x2" in desc, desc
            assert " NT=128 " in desc and " nsplit=1" in desc, desc
        it["ref"] = y
    return it["ref"]


def assert_carve(desc, t, KS):
    row = t.row
    assert desc.startswith("pq_gemm_tc_ws("), desc
    want = dict(positions=t.P, N=t.W, KS=KS, wbufs=t.nWB, stages=t.stages(KS), smem=t.smem(KS), NPOS=t.NPOS,
                ksteps=sum(t.counts) if row.stride > 1 else t.counts[0] * len(t.counts))
    if row.stride == 1:
        want["planebufs"] = t.nPB[KS]
        assert " mode=0 " in desc, desc
    got = {f: field(desc, f) for f in want}
    assert got == want, (desc, want)


def run_tiling(row, t, it, KS, reps):
    """Forward at tiling t with KS pinned (0: unpinned, the default), describe() against the mirror, the output against
    the reference bit for bit, reps times."""
    L = it["L"]
    ref = reference(row, it)
    set_pins(L, 7, nt=t.P, gt=KS, ct=t.W, wb=t.nWB)
    for _ in range(reps):
        y = L.forward(it["xd"])
        desc = L.describe(row.N)
        assert_carve(desc, t, KS or t.default)
        assert as_bits(y).equal(as_bits(ref)), (desc, bit_mismatches(y, ref))


# the sweep: (row, channels per CTA to run (None = every width offered))
SWEEP = [(ROWS[n], w) for n, w in (
    ("conv2_n3", None), ("conv2_n256", None), ("conv3_n3", None), ("kg384_k3", (64,)), ("kg96_cg20_k3", None),
    ("tiny_kg256_pad2", (256,)), ("kg192_k5_cg36_d12", (192,)), ("cg3_k5_pad2", None),
    ("conv1_n3_nchw", None), ("conv1_n3", None), ("conv1_n256_nchw", None), ("kg96_k7_s4_cg1_pad2", None),
    ("vggs_k7_s2", None), ("longrow80_k11_s2", None), ("g2_kg32_k3_s4_cg3_nchw", None), ("k2_s4_pad1_cg3", None),
    ("k1_s2_cg4", None))]
SWEEP_CASES = [pytest.param(r, t, id="%s-P%d-N%d-wb%d" % (r.name, t.P, t.W, t.nWB)) for r, w in SWEEP for t in space(r, w)]


def test_sweep_covers_every_depth_and_empty_rows():
    """Every ring depth in both geometries, and an empty phase row at every depth."""
    for s1 in (True, False):
        assert {t.nWB for r, w in SWEEP if (r.stride == 1) == s1 for t in space(r, w)} == {2, 3, 4}, s1
    assert {t.nWB for r, w in SWEEP if r.stride > 1 and 0 in mode1_counts(r.k, r.stride, True)
            for t in space(r, w)} == {2, 3, 4}
    assert [r.name for r, _ in SWEEP if r.stride > 1 and mode1_counts(r.k, r.stride, True).count(0) == 2] == ["k2_s4_pad1_cg3"]


@pytest.mark.gpu
@pytest.mark.parametrize("row,t", SWEEP_CASES)
def test_conv_ws_ring_sweep(row, t, cache):
    """Every KS of tiling t (a subset at batch 256) and the unpinned default, bit for bit against the reference; at
    small batches each twice (run-to-run identity)."""
    it = cache.get(row)
    big = row.N >= 64
    ks_list = t.ks_subset() if big else list(range(1, t.ksmax + 1))
    try:
        run_tiling(row, t, it, 0, 1)
        for KS in ks_list:
            run_tiling(row, t, it, KS, 1 if big else 2)
    finally:
        set_pins(it["L"], -1)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["k2_s4_pad1_cg3", "k1_s2_cg4"])
def test_conv_ws_takes_layers_with_empty_phase_rows(name, cache):
    """conv_ws takes a strided layer whose trailing phase rows have no k-steps: a pin on the family alone gives a plan
    over every phase row."""
    row = ROWS[name]
    assert 0 in mode1_counts(row.k, row.stride, True)
    it = cache.get(row, data=False)
    set_pins(it["L"], 7)
    try:
        desc = it["L"].describe(row.N)
        assert desc.startswith("pq_gemm_tc_ws(") and field(desc, "chunks") == row.stride, desc
        assert field(desc, "ksteps") == sum(mode1_counts(row.k, row.stride, True)), desc
    finally:
        set_pins(it["L"], -1)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["conv2_n3", "conv1_n3_nchw"])
def test_conv_ws_pins_outside_the_space_fail(name, qcnn, cache):
    """KS above every chunk's count, a ring of 1 or 5 buffers, and a (KS, nWB) whose carve exceeds the opt-in limit
    leave conv_ws no tiling: an error, not another tiling."""
    row = ROWS[name]
    L = cache.get(row, data=False)["L"]
    over = [t for t in space(row) if t.ksmax < max(t.counts)]
    assert over, "no tiling of %s is limited by shared memory" % row.name
    bad = [dict(gt=max(over[0].counts) + 1), dict(wb=1), dict(wb=5)]
    bad += [dict(nt=t.P, ct=t.W, wb=t.nWB, gt=t.ksmax + 1) for t in over[:2]]
    try:
        for pins in bad:
            set_pins(L, 7, **pins)
            with pytest.raises(qcnn.QcnnError):
                L.describe(row.N)
        for nWB in (2, 3, 4):   # each depth alone is offered
            set_pins(L, 7, wb=nWB)
            assert field(L.describe(row.N), "wbufs") == nWB
    finally:
        set_pins(L, -1)


@pytest.mark.gpu
def test_gemm_wb_refused_on_fc_layer(qcnn, ctx):
    """gemm_wb is a conv parameter, and an FC layer has no weight image."""
    rng = np.random.RandomState(7)
    fc = qcnn.FcLayer(ctx, 64, rng.randn(16, 16, 4).astype(np.float32), rng.randint(0, 16, (32, 16)).astype(np.uint8),
                      np.zeros(32, np.float32))
    try:
        with pytest.raises(qcnn.QcnnError):
            fc.set_param("gemm_wb", 2)
        assert fc.read_w_ws().size == 0
    finally:
        fc.close()


# the ring's extremes on rows whose images straddle tiles: 25-position images at stride 1, 30-position images with an
# empty phase row (3 x 3 / 4, groups, NCHW) in mode 1
EXTREMES = [pytest.param(ROWS[n], W, ks, wb, id="%s-N%d-KS%s-wb%d" % (n, W, ks or "default", wb))
            for n, W in (("tiny_kg256_pad2", 128), ("g2_kg32_k3_s4_cg3_nchw", 32)) for ks, wb in ((1, 2), (1, 3), (0, 3))]


@pytest.mark.gpu
@pytest.mark.parametrize("row,W,ks,wb", EXTREMES)
def test_conv_ws_ring_extremes(row, W, ks, wb, qcnn, cache):
    import torch
    it = cache.get(row)
    L = it["L"]
    t = next(tt for tt in space(row) if tt.W == W and tt.nWB == wb)
    assert t.P == 256
    try:
        run_tiling(row, t, it, ks, 2)                     # bits, carve, run-to-run
        y = L.forward(it["xd"]).cpu().numpy()
        yr = L.forward(it["xd"], relu=True).cpu().numpy()
        assert np.array_equal(yr, np.where(y > 0, y, np.float32(0)))
        # neighbour poisoning: image i's output does not depend on whether the other images are 0 or NaN
        i = (row.N - 1) // 2
        for fill in (0.0, np.nan):
            xp = np.full_like(it["x"], fill)
            xp[i] = it["x"][i]
            yi = L.forward(torch.from_numpy(cache.src(row, xp)).cuda()).cpu().numpy()[i]
            assert np.array_equal(bits(yi), bits(y[i])), fill
        # exact write set: a NaN guard around the output stays untouched and every element is written
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        xd = it["xd"]
        for relu, want in ((0, y), (1, yr)):
            out, guard_ok = _guarded_call(
                lambda dst, r: qcnn._check(qcnn.lib.qcnn_conv_aprx_forward(L.h, ctypes.c_void_p(xd.data_ptr()), row.N,
                                                                           dst, r, stream)), y.size, relu)
            assert guard_ok, relu
            assert np.array_equal(bits(out), bits(want.reshape(-1))), relu
        assert_carve(L.describe(row.N), t, ks or t.default)
    finally:
        set_pins(L, -1)


# every channel width the stride-1 planner offers, at batch 1, 3 and 256, unpinned KS and depth
CASES = [pytest.param(r, W, id="%s-N%d" % (r.name, W)) for r in ALEXNET + ODD for W in widths(r)]


@pytest.mark.gpu
@pytest.mark.parametrize("row,W", CASES)
def test_conv_ws_image_bit_identical_to_decode_at_use(row, W, cache):
    it = cache.get(row)
    ref = reference(row, it)
    L = it["L"]
    set_pins(L, 7, ct=W)
    y = L.forward(it["xd"])
    desc = L.describe(row.N)
    assert desc.startswith("pq_gemm_tc_ws(") and " mode=0 " in desc and " N=%d " % W in desc, desc
    assert 2 <= field(desc, "wbufs") <= 4, desc
    assert as_bits(y).equal(as_bits(ref)), (desc, bit_mismatches(y, ref))


@pytest.mark.gpu
def test_conv_ws_unmatched_ks_pin_fails(qcnn, cache):
    """A k-steps-per-stage pin longer than a chunk's taps leaves conv_ws no tiling: an error, not another tiling."""
    row = ROWS["conv3_n1"]
    L = cache.get(row, data=False)["L"]
    set_pins(L, 7, gt=10)
    try:
        with pytest.raises(qcnn.QcnnError):
            L.describe(row.N)
    finally:
        L.set_param("gemm_gt", 0)


IMAGE_GPU_ROWS = sorted(set(IMAGE_ROWS) - {"conv2_n256", "conv1_n256_nchw"})


@pytest.mark.gpu
@pytest.mark.parametrize("name", IMAGE_GPU_ROWS)
def test_weight_image_bytes(name, cache):
    """read_w_ws() is the numpy image byte for byte: G x entries x 2 x Kg x 16 bytes."""
    row = ROWS[name]
    it = cache.get(row, data=False)
    want = ws_image(row, *it["params"][:2])
    got = it["L"].read_w_ws()
    assert got.size == want.shape[0] * want.shape[1] * 2 * (row.Cout // row.G) * 16, (got.size, want.shape)
    got = got.view(np.uint16).reshape(want.shape)
    assert np.array_equal(got, want), int((got != want).sum())


@pytest.mark.gpu
def test_layer_without_image(qcnn, ctx):
    """A conv layer conv_ws does not take (d = 6) has no weight image."""
    row = Row("d6", 2, 9, 9, 12, 64, 3, 1, 1, 1, 2, 64, 6, False)
    ctrd, asmt, bias = layer_params(row)
    L = qcnn.ConvLayer(ctx, row.Cin, row.Hi, row.Wi, row.Cout, row.k, row.pad, row.stride, row.G, ctrd, asmt, bias)
    try:
        assert L.read_w_ws().size == 0
    finally:
        L.close()
