"""The weight-stationary FC GEMM (fc_ws, describe() "pq_gemm_tc_ws(...) mode=2") against a float64 reference, at every
tiling it offers and at the shapes where its code paths branch.

Reference, metric and bound are those of test_gpu_pq_gemm.py: err = max |gpu - ref64| / M with M = sum |w x| + |bias|, and
the bound of the bf16x2 class with one accumulator per 128 images, tc_bound(bf16x2, 128, ks, nsplit), where ks is the
k-steps one CTA chains (describe()'s ksteps) and nsplit the K-split (describe()'s nsplit).  The layers of network size
(AlexNet fc6-fc8, VGG16 fc6) take the same float64 reference evaluated with torch on the GPU (the decoded weight matrix
times the input); test_gpu_ref_matches_ref64 checks that it agrees with ref64 on a small row.

Coverage: d in {1, 4, 8, 12, 16}; K in {16, 32, 64, 128, 256} (the byte table holds index << 2 for K <= 64); a partial
last subspace; the NHWC fold of a first FC layer; Dout tails (1000, 200, 96); N in {96, 129, 256, 300, 1024}; nsplit = 1
and > 1; ReLU on and off.  Every case pins the images per CTA (gemm_nt), the channels per CTA (gemm_ct) and the k-steps
per stage (gemm_gt) of each tiling fc_ws offers, with the planner's K-split and with gemm_nsplit = 1.  Besides: run-to-run
bit identity, neighbour NaN isolation, the exact write set of the output, the fall-back to pq_gemm_tc mode 2 where fc_ws
does not apply (tensor_core = 1, fc_ws = 0), bit-identical outputs from the byte and the bit-packed table, and the plans
of a network's FC layers.
"""
import ctypes

import numpy as np
import pytest

from test_gpu_pq_gemm import FcRow, _guarded_call, bits, f64_err, fc_data, fc_input, ref64, save_report, tc_bound, REPORT

# (channels per CTA, images per CTA) of the fc_ws instantiations, and the k-steps per stage
SHAPES = [(256, 128), (128, 128), (128, 256), (64, 128), (64, 256)]
STAGES = (8, 4)

FC_WS_ROWS = [
    FcRow("d4_k16_n96", 96, 64, 256, 16, 16, 4, None),
    FcRow("d16_partial_sub_dout200", 129, 1000, 200, 63, 64, 16, None),   # Din = 1000: the last subspace has 8 of 16 dims
    FcRow("d1_k256_dout1000", 300, 512, 1000, 512, 256, 1, None),
    FcRow("d12_k128_dout96", 256, 480, 96, 40, 128, 12, None),
    FcRow("d8_k32_nhwc_fold", 130, 512, 64, 64, 32, 8, (4, 4, 32)),
    FcRow("d8_k16_n1024", 1024, 64, 2048, 8, 16, 8, None),
    FcRow("d4_k16_n1024", 1024, 256, 512, 64, 16, 4, None),
]
BIG_ROWS = [
    FcRow("alexnet_fc6_n256", 256, 9216, 4096, 2304, 32, 4, (6, 6, 256)),
    FcRow("alexnet_fc7_n256", 256, 4096, 4096, 1024, 32, 4, None),
    FcRow("alexnet_fc8_n256", 256, 4096, 1000, 4096, 16, 1, None),
    FcRow("alexnet_fc6_n1024", 1024, 9216, 4096, 2304, 32, 4, (6, 6, 256)),
    FcRow("alexnet_fc7_n1024", 1024, 4096, 4096, 1024, 32, 4, None),
    FcRow("alexnet_fc8_n1024", 1024, 4096, 1000, 4096, 16, 1, None),
    FcRow("vgg16_fc6_n256", 256, 25088, 4096, 6272, 32, 4, (7, 7, 512)),
]
ROWS = {r.name: r for r in FC_WS_ROWS + BIG_ROWS}


def _field(desc, name):
    return int(desc.split(" %s=" % name)[1].split()[0])


def test_rows_cover_the_branches():
    rows = FC_WS_ROWS + BIG_ROWS
    assert {1, 4, 8, 12, 16} <= {r.d for r in rows}
    assert {16, 32, 64, 128, 256} <= {r.K for r in rows}
    assert {96, 129, 256, 300, 1024} <= {r.N for r in rows}
    assert {1000, 200, 96} <= {r.Dout for r in rows}
    assert any(r.nhwc for r in rows) and any(r.Din % 16 and r.S * r.d > r.Din for r in rows)


def _layer(qcnn, ctx, row, ctrd, asmt, bias):
    L = qcnn.FcLayer(ctx, row.Din, ctrd, asmt, bias)
    if row.nhwc:
        L.set_src_nhwc(*row.nhwc)
    L.set_param("fc_ws", 1)
    return L


def _pin(L, nt=0, ct=0, gt=0, ns=0):
    for name, v in (("gemm_nt", nt), ("gemm_ct", ct), ("gemm_gt", gt), ("gemm_nsplit", ns)):
        L.set_param(name, v)


def _ref_gpu(row, x, ctrd, asmt, bias):
    """(ref, M) in float64 on the GPU: the decoded weight matrix [Dout, Din] times the NCHW-flattened input."""
    import torch
    dev = "cuda"
    c = torch.from_numpy(ctrd).to(dev, torch.float64)                                # [S, K, d]
    a = torch.from_numpy(asmt.astype(np.int64)).to(dev)                              # [Dout, S]
    W = c[torch.arange(row.S, device=dev)[None, :], a].reshape(row.Dout, -1)[:, :row.Din]
    xf = torch.from_numpy(fc_input(row, x)).to(dev, torch.float64)
    b = torch.from_numpy(bias).to(dev, torch.float64)
    ref = xf @ W.T + b
    mag = xf.abs() @ W.abs().T + b.abs()
    return ref.cpu().numpy(), mag.cpu().numpy()


def _reference(row, x, ctrd, asmt, bias):
    if row.name in {r.name for r in BIG_ROWS}:
        return _ref_gpu(row, x, ctrd, asmt, bias)
    return ref64("fc", fc_input(row, x), ctrd, asmt, bias)


def _check(L, row, xd, ref, mag, key):
    y = L.forward(xd).cpu().numpy()
    yr = L.forward(xd, relu=True).cpu().numpy()
    desc = L.describe(row.N)
    plan = desc.split(" via ")[1]
    assert plan.startswith("pq_gemm_tc_ws(") and " mode=2 " in plan and "NT=" not in plan, desc
    ks, ns = _field(plan, "ksteps"), _field(plan, "nsplit")
    bound = tc_bound(True, 128, ks, ns)
    e, er = f64_err(y, ref, mag), f64_err(yr, np.maximum(ref, 0), mag)
    REPORT["fc_ws/%s/%s" % (row.name, key)] = {"plan": plan, "err": e, "err_relu": er, "bound": bound}
    assert e <= bound, (e, bound, plan)
    assert er <= bound, (er, bound, plan)
    return y, plan


@pytest.mark.gpu
@pytest.mark.parametrize("name", [r.name for r in FC_WS_ROWS + BIG_ROWS])
def test_fc_ws_tilings_f64(name, qcnn, ctx):
    """Every tiling fc_ws offers for the row (with the planner's K-split and unsplit) within the bf16x2 bound."""
    import torch
    row = ROWS[name]
    x, ctrd, asmt, bias = fc_data(row)
    ref, mag = _reference(row, x, ctrd, asmt, bias)
    L = _layer(qcnn, ctx, row, ctrd, asmt, bias)
    xd = torch.from_numpy(x).cuda().view(row.N, -1)
    seen = set()
    # (network-size rows: the widest tilings only, besides the unpinned plan below)
    pins = [(ct, nt, gt, ns) for ct, nt in SHAPES for gt in STAGES for ns in (0, 1)]
    if row in BIG_ROWS:
        pins = [p for p in pins if p[0] >= 128 and p[1] == 128]
    for ct, nt, gt, ns in pins:
        _pin(L, nt, ct, gt, ns)
        try:
            L.describe(row.N)
        except qcnn.QcnnError as ex:
            assert "has no fc_ws tiling" in str(ex), str(ex)
            continue
        y, plan = _check(L, row, xd, ref, mag, "ct=%d/nt=%d/gt=%d/ns=%d" % (ct, nt, gt, ns))
        assert " N=%d images=%d " % (ct, nt) in plan and " KS=%d " % gt in plan, plan
        assert ns == 0 or " nsplit=1 " in plan, plan
        seen.add(plan)
    _pin(L)
    y, plan = _check(L, row, xd, ref, mag, "default")
    y2 = L.forward(xd).cpu().numpy()
    assert np.array_equal(bits(y), bits(y2)), plan
    L.close()
    save_report()
    assert seen


@pytest.mark.gpu
def test_gpu_ref_matches_ref64(qcnn, ctx):
    row = ROWS["d16_partial_sub_dout200"]
    x, ctrd, asmt, bias = fc_data(row)
    r1, m1 = ref64("fc", fc_input(row, x), ctrd, asmt, bias)
    r2, m2 = _ref_gpu(row, x, ctrd, asmt, bias)
    assert np.abs(r1 - r2).max() <= 1e-12 * m1.max() and np.abs(m1 - m2).max() <= 1e-12 * m1.max()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["d4_k16_n96", "d1_k256_dout1000"])
def test_fc_ws_neighbour_poison(name, qcnn, ctx):
    """An image's outputs are bit-identical whether the other images of the batch are 0 or NaN."""
    import torch
    row = ROWS[name]
    x, ctrd, asmt, bias = fc_data(row)
    L = _layer(qcnn, ctx, row, ctrd, asmt, bias)
    for ns in (0, 1):
        _pin(L, ns=ns)
        for i in (0, 64, row.N - 1):
            outs = []
            for fill in (0.0, np.nan):
                xp = np.full_like(x, fill)
                xp[i] = x[i]
                outs.append(L.forward(torch.from_numpy(xp).cuda().view(row.N, -1)).cpu().numpy()[i])
            assert np.array_equal(bits(outs[0]), bits(outs[1])), (ns, i)
        assert "pq_gemm_tc_ws(" in L.describe(row.N)
    L.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["d1_k256_dout1000", "d12_k128_dout96", "d16_partial_sub_dout200"])
def test_fc_ws_exact_write_set(name, qcnn, ctx):
    """[N][Dout] and nothing else: a NaN-filled guard region on either side of the output stays untouched."""
    import torch
    row = ROWS[name]
    x, ctrd, asmt, bias = fc_data(row)
    L = _layer(qcnn, ctx, row, ctrd, asmt, bias)
    xd = torch.from_numpy(x).cuda().view(row.N, -1)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for ns in (0, 1):
        _pin(L, ns=ns)
        assert "pq_gemm_tc_ws(" in L.describe(row.N)
        for relu in (0, 1):
            out, guard_ok = _guarded_call(
                lambda dst, r: qcnn._check(qcnn.lib.qcnn_fc_aprx_forward(L.h, ctypes.c_void_p(xd.data_ptr()), row.N, dst, r,
                                                                         stream)), row.N * row.Dout, relu)
            assert guard_ok, (ns, relu)
            assert np.isfinite(out).all(), (ns, relu)
    L.close()


@pytest.mark.gpu
def test_fc_ws_ineligible_falls_back_to_mode2(qcnn, ctx):
    """fc_ws applies to bf16x2 operands only; with 3xTF32 or fc_ws = 0 the layer runs pq_gemm_tc mode 2 as before."""
    row = ROWS["d4_k16_n96"]
    x, ctrd, asmt, bias = fc_data(row)
    L = _layer(qcnn, ctx, row, ctrd, asmt, bias)
    assert "pq_gemm_tc_ws(" in L.describe(row.N)
    L.set_param("tensor_core", 1)
    d = L.describe(row.N)
    assert "pq_gemm_tc(" in d and "mode=2" in d and "bf16x2" not in d, d
    L.set_param("tensor_core", 2)
    L.set_param("fc_ws", 0)
    d = L.describe(row.N)
    assert "pq_gemm_tc(" in d and "mode=2" in d, d
    L.close()


@pytest.mark.gpu
def test_alexnet_net_plans_fc_ws(po, qcnn, ctx, tmp_path):
    """A network's FC layers (AlexNet fc6, fc7, fc8 at N = 256) run fc_ws."""
    import torch
    if po.have_alexnet():
        dirpath, pfx = po.ALEXNET_DIR, po.ALEXNET_PFX
    else:
        dirpath, pfx = str(tmp_path), "synth"
        po.save_model(dirpath, pfx, po.synth_alexnet(seed=1))
    net = qcnn.Net(ctx, dirpath, pfx, "AlexNet")
    img = torch.from_numpy(po.lcg_images(256, 4242)).cuda()
    p = net.forward(img).cpu().numpy()
    assert np.isfinite(p).all()
    for l in (15, 18, 21):
        d = net.pq_layer(l).describe(256)
        assert "pq_gemm_tc_ws(" in d and "NT=" not in d, (l, d)
    net.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["d4_k16_n96", "d1_k256_dout1000", "alexnet_fc8_n256", "alexnet_fc7_n256"])
def test_fc_ws_packed_table_bit_identical(name, qcnn, ctx):
    """A bit-packed table is expanded into the bytes the byte table holds: same tiling, bit-identical outputs."""
    import torch
    row = ROWS[name]
    x, ctrd, asmt, bias = fc_data(row)
    L = _layer(qcnn, ctx, row, ctrd, asmt, bias)
    xd = torch.from_numpy(x).cuda().view(row.N, -1)
    outs, plans = [], []
    for packed in (0, 1):
        L.set_param("asmt_packed", packed)
        outs.append(L.forward(xd).cpu().numpy())
        plans.append(L.describe(row.N))
    assert "pq_gemm_tc_ws(" in plans[1] and ("asmt=" in plans[1]) == (row.K < 256), plans[1]
    assert plans[0].split(" via ")[1] == plans[1].split(" via ")[1].split(" asmt=")[0]
    assert np.array_equal(bits(outs[0]), bits(outs[1])), name
    L.close()
