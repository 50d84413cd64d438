"""Per-layer parity of the CUDA kernels (through the C ABI) against the CPU oracle.

Tolerances (stated once, used everywhere):
  * assignment indexing: bit-exact (decoded device table == reference asmtBuf)
  * FC with one subspace split: bit-exact (same operation order as the reference, separate mul/add)
  * everything else (conv, split FC): |gpu - ref| <= RTOL * max(1, |ref|, 0.1 * max|ref|) elementwise, RTOL = 1e-4.
    The third term scales the bound with the magnitude of the tensor: an output is a sum of 10^2..10^4 fp32 LUT
    entries that partly cancel, so the *reference's own* sequential-sum rounding noise is ~sqrt(n)*2^-24*|partial
    sums|; re-associating that sum (s-major instead of tap-major, split-S) and FMA contraction in the LUT stage move
    results by the same order.  LRN / softmax (libm vs CUDA expf/logf): 1e-5 relative / 1e-6 absolute.
"""
import numpy as np
import pytest

RTOL = 1e-4
# decode-at-use tensor-core kernels (bf16x2 or 3xTF32 operands, fp32 accumulation inside the tensor core over all k-steps): measured
# on an H100 <= 1.1e-4 per layer on the AlexNet shapes at batch 256; the LUT + gather kernels stay within RTOL (measured 5.5e-6)
RTOL_TC = 3e-4


def close(gpu, ref, rtol=RTOL):
    gpu = np.asarray(gpu, np.float64)
    ref = np.asarray(ref, np.float64)
    if not ref.size:
        return 0.0
    scale = np.maximum(np.maximum(1.0, np.abs(ref)), 0.1 * np.abs(ref).max())
    return float((np.abs(gpu - ref) / scale).max())


def rand_act(rng, shape, scale=20.0):
    # post-ReLU-like, non-negative (SURVEY.md 8(d) sweep tensors)
    return (np.abs(rng.randn(*shape)) * scale).astype(np.float32)


FC_CASES = [
    # (N, Din, Dout, S, K, d)
    (1, 9216, 4096, 2304, 32, 4),    # fc6
    (1, 4096, 4096, 1024, 32, 4),    # fc7
    (1, 4096, 1000, 4096, 16, 1),    # fc8 (Dout not a multiple of 16)
    (3, 512, 200, 128, 32, 4),
    (4, 512, 200, 128, 32, 4),
    (9, 640, 1000, 160, 16, 4),
    (37, 256, 520, 64, 64, 4),
    (8, 300, 96, 40, 128, 8),        # Din not a multiple of d: last subspace is partial
    (16, 128, 64, 16, 256, 8),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", FC_CASES)
def test_fc_parity(case, po, qcnn, ctx):
    import torch
    N, Din, Dout, S, K, d = case
    rng = np.random.RandomState(hash(case) % (2 ** 31))
    ctrd = (rng.randn(S, K, d) * 0.05).astype(np.float32)
    asmt = rng.randint(0, K, size=(Dout, S)).astype(np.uint8)
    bias = (rng.randn(Dout) * 0.1).astype(np.float32)
    x = rand_act(rng, (N, Din))
    ref = po.fc_aprx(x, ctrd, asmt, bias)
    layer = qcnn.FcLayer(ctx, Din, ctrd, asmt, bias)
    # bit-exact decoded assignment table, reference asmtBuf order [S][Dout]
    assert np.array_equal(layer.read_asmt(S * Dout).reshape(S, Dout), asmt.T)
    xd = torch.from_numpy(x).cuda()
    # (a) automatic configuration
    y = layer.forward(xd).cpu().numpy()
    assert close(y, ref) <= RTOL
    # (b) one split: same accumulation order as the reference -> bit-exact
    layer.set_param("fc_nsplit", 1)
    for tn in (1, 4, 8):
        layer.set_param("fc_tn", tn)
        y1 = layer.forward(xd).cpu().numpy()
        assert np.array_equal(y1, ref), "tn=%d max err %g" % (tn, close(y1, ref))
    # (c) fused ReLU
    yr = layer.forward(xd, relu=True).cpu().numpy()
    assert np.array_equal(yr, np.maximum(ref, 0))
    layer.close()


FC_TC_CASES = [
    # large batches take the tensor-core path (decode-at-use GEMM, split-K): (N, Din, Dout, S, K, d)
    (128, 512, 200, 128, 32, 4),
    (200, 4096, 1000, 4096, 16, 1),   # fc8-like: scalar codewords, Dout not a multiple of 16
    (300, 1024, 520, 128, 64, 8),     # two batch tiles, d = 8
    (256, 2048, 4096, 512, 32, 4),    # fc7-like
    (100, 304, 96, 38, 128, 8),       # odd k-step count (Din/8 = 38)
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", FC_TC_CASES)
def test_fc_tc_parity(case, po, qcnn, ctx):
    import torch
    N, Din, Dout, S, K, d = case
    rng = np.random.RandomState(hash(case) % (2 ** 31))
    ctrd = (rng.randn(S, K, d) * 0.05).astype(np.float32)
    asmt = rng.randint(0, K, size=(Dout, S)).astype(np.uint8)
    bias = (rng.randn(Dout) * 0.1).astype(np.float32)
    x = rand_act(rng, (N, Din))
    ref = po.fc_aprx(x, ctrd, asmt, bias)
    layer = qcnn.FcLayer(ctx, Din, ctrd, asmt, bias)
    xd = torch.from_numpy(x).cuda()
    y = layer.forward(xd).cpu().numpy()
    assert close(y, ref) <= RTOL_TC, close(y, ref)
    yr = layer.forward(xd, relu=True).cpu().numpy()
    assert close(yr, np.maximum(ref, 0)) <= RTOL_TC
    assert "bf16x2" in layer.describe(N)       # the default operand format
    layer.set_param("tensor_core", 1)          # 3xTF32 operands
    assert "bf16x2" not in layer.describe(N)
    yb = layer.forward(xd).cpu().numpy()
    assert close(yb, ref) <= RTOL_TC, close(yb, ref)
    layer.set_param("tensor_core", 2)
    # explicit single split keeps the gather kernel and the reference's accumulation order: bit-exact
    layer.set_param("fc_nsplit", 1)
    assert np.array_equal(layer.forward(xd).cpu().numpy(), ref)
    layer.close()


@pytest.mark.gpu
def test_fc_tc_nhwc_source(po, qcnn, ctx):
    import torch
    rng = np.random.RandomState(11)
    N, H, W, Cc, Dout, K, d = 130, 6, 6, 32, 256, 32, 4
    Din = H * W * Cc
    S = Din // d
    ctrd = (rng.randn(S, K, d) * 0.05).astype(np.float32)
    asmt = rng.randint(0, K, size=(Dout, S)).astype(np.uint8)
    bias = (rng.randn(Dout) * 0.1).astype(np.float32)
    x = rand_act(rng, (N, H, W, Cc))
    ref = po.fc_aprx(po.nhwc_to_nchw(x).reshape(N, -1), ctrd, asmt, bias)
    layer = qcnn.FcLayer(ctx, Din, ctrd, asmt, bias)
    layer.set_src_nhwc(H, W, Cc)
    y = layer.forward(torch.from_numpy(x).cuda().view(N, -1)).cpu().numpy()
    assert close(y, ref) <= RTOL_TC, close(y, ref)
    layer.set_param("tensor_core", 0)
    y = layer.forward(torch.from_numpy(x).cuda().view(N, -1)).cpu().numpy()
    assert close(y, ref) <= RTOL, close(y, ref)
    layer.close()


@pytest.mark.gpu
def test_fc_nhwc_source_fold(po, qcnn, ctx):
    """fc6-style: the NHWC->NCHW permute of the reference (CaffeEva.cc:236-238) folded into the LUT addressing."""
    import torch
    rng = np.random.RandomState(7)
    N, H, W, Cc, Dout, K, d = 5, 6, 6, 32, 128, 32, 4
    Din = H * W * Cc
    S = Din // d
    ctrd = (rng.randn(S, K, d) * 0.05).astype(np.float32)
    asmt = rng.randint(0, K, size=(Dout, S)).astype(np.uint8)
    bias = (rng.randn(Dout) * 0.1).astype(np.float32)
    x = rand_act(rng, (N, H, W, Cc))
    ref = po.fc_aprx(po.nhwc_to_nchw(x).reshape(N, -1), ctrd, asmt, bias)
    layer = qcnn.FcLayer(ctx, Din, ctrd, asmt, bias)
    layer.set_src_nhwc(H, W, Cc)
    layer.set_param("fc_nsplit", 1)
    y = layer.forward(torch.from_numpy(x).cuda().view(N, -1)).cpu().numpy()
    assert np.array_equal(y, ref)
    # explicit permute kernels agree with the oracle's permutes bit-for-bit
    xd = torch.from_numpy(x).cuda()
    assert np.array_equal(ctx.nhwc_to_nchw(xd).cpu().numpy(), po.nhwc_to_nchw(x))
    assert np.array_equal(ctx.nchw_to_nhwc(ctx.nhwc_to_nchw(xd)).cpu().numpy(), x)
    layer.close()


CONV_CASES = [
    # (N, Hi, Wi, Cin, Cout, k, pad, stride, G, S, K, d)
    (2, 27, 27, 96, 256, 5, 2, 1, 2, 6, 128, 8),      # conv2
    (2, 13, 13, 256, 384, 3, 1, 1, 1, 32, 128, 8),    # conv3
    (3, 13, 13, 384, 384, 3, 1, 1, 2, 24, 128, 8),    # conv4
    (2, 13, 13, 384, 256, 3, 1, 1, 2, 24, 128, 8),    # conv5
    (1, 227, 227, 3, 96, 11, 0, 4, 1, 1, 128, 8),     # conv1 (d=8 in the file, 3 dims used)
    (2, 9, 11, 32, 64, 3, 1, 1, 1, 4, 64, 8),         # non-square, K=64
    (1, 13, 13, 64, 128, 3, 1, 1, 2, 4, 256, 8),      # K=256
    (2, 12, 12, 48, 32, 3, 0, 1, 1, 4, 128, 12),      # "valid" conv, d=12 (two LUT chunks)
    (1, 13, 13, 256, 384, 3, 1, 1, 1, 16, 64, 16),    # sweep point S=16, K=64, d=16
    (2, 31, 29, 8, 32, 7, 0, 2, 1, 2, 128, 4),        # VggCnnS-like stride 2, S>1
    (1, 20, 20, 16, 32, 5, 2, 3, 2, 2, 32, 4),        # stride 3 with padding and groups
    (2, 17, 19, 3, 32, 5, 1, 2, 1, 1, 64, 4),         # conv1-like: 3 input channels, stride 2 with padding, one subspace
    (3, 14, 14, 4, 48, 3, 0, 3, 1, 1, 128, 4),        # 4 input channels, stride 3, one subspace
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_parity(case, po, qcnn, ctx):
    import torch
    N, Hi, Wi, Cin, Cout, k, pad, stride, G, S, K, d = case
    rng = np.random.RandomState(hash(case) % (2 ** 31))
    ctrd = (rng.randn(S, K, d) * 0.05).astype(np.float32)
    asmt = rng.randint(0, K, size=(Cout, k, k, S)).astype(np.uint8)
    bias = (rng.randn(Cout) * 0.1).astype(np.float32)
    x = rand_act(rng, (N, Hi, Wi, Cin))
    L = po.conv(pad, k, Cout, G, stride)
    ref = po.conv_aprx(x, L, ctrd, asmt, bias)
    layer = qcnn.ConvLayer(ctx, Cin, Hi, Wi, Cout, k, pad, stride, G, ctrd, asmt, bias)
    got = layer.read_asmt(asmt.size).reshape(k, k, S, Cout)
    assert np.array_equal(got, np.transpose(asmt, (1, 2, 3, 0)))  # reference asmtBuf order (CaffeEva.cc:585-586)
    xd = torch.from_numpy(x).cuda()
    # (a) default: the autotuner may pick a decode-at-use tensor-core kernel
    y = layer.forward(xd).cpu().numpy()
    assert y.shape == ref.shape
    assert close(y, ref) <= RTOL_TC, close(y, ref)
    if stride > 1:
        layer.set_src_nchw(True)
        yn = layer.forward(torch.from_numpy(po.nhwc_to_nchw(x)).cuda()).cpu().numpy()
        assert close(yn, ref) <= RTOL_TC, close(yn, ref)
        layer.set_src_nchw(False)
    # (a2) both operand formats of the tensor-core GEMM explicitly: 2 = bf16x2 (the default), 1 = 3xTF32
    for tc in (2, 1):
        layer.set_param("tensor_core", tc)
        yb = layer.forward(xd).cpu().numpy()
        assert close(yb, ref) <= RTOL_TC, (tc, close(yb, ref), layer.describe(N))
    # (b) strict parity: LUT + gather kernels only (fp32 adds)
    layer.set_param("tensor_core", 0)
    y = layer.forward(xd).cpu().numpy()
    assert close(y, ref) <= RTOL, close(y, ref)
    yr = layer.forward(xd, relu=True).cpu().numpy()
    assert close(yr, np.maximum(ref, 0)) <= RTOL
    # batch invariance: image 0 alone gives the same result as image 0 inside the batch (tilings differ per batch size)
    y0 = layer.forward(xd[:1].contiguous()).cpu().numpy()
    assert close(y0[0], y[0]) <= RTOL
    if stride > 1:
        layer.set_src_nchw(True)
        yn = layer.forward(torch.from_numpy(po.nhwc_to_nchw(x)).cuda()).cpu().numpy()
        assert np.array_equal(yn, y)
    layer.close()


# Each LUT + gather family pinned on CONV_CASES shapes (with the cost model alone some families never run): (case index,
# force_kernel id); every family twice, both rolling-row families on an NCHW source too.
CONV_FAMILY_NAMES = {0: "conv_s1 ", 1: "conv_roll ", 2: "conv_s1_tc(", 3: "conv_roll_tc(", 4: "conv_direct "}
CONV_FAMILY_PAIRS = [(0, 0), (8, 0), (9, 1), (10, 1), (1, 2), (3, 2), (4, 3), (9, 3), (4, 4), (11, 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("idx,family", CONV_FAMILY_PAIRS)
def test_conv_family_pinned(idx, family, po, qcnn, ctx):
    import torch
    case = CONV_CASES[idx]
    N, Hi, Wi, Cin, Cout, k, pad, stride, G, S, K, d = case
    rng = np.random.RandomState(hash(case) % (2 ** 31))
    ctrd = (rng.randn(S, K, d) * 0.05).astype(np.float32)
    asmt = rng.randint(0, K, size=(Cout, k, k, S)).astype(np.uint8)
    bias = (rng.randn(Cout) * 0.1).astype(np.float32)
    x = rand_act(rng, (N, Hi, Wi, Cin))
    ref = po.conv_aprx(x, po.conv(pad, k, Cout, G, stride), ctrd, asmt, bias)
    layer = qcnn.ConvLayer(ctx, Cin, Hi, Wi, Cout, k, pad, stride, G, ctrd, asmt, bias)
    layer.set_param("tensor_core", 0)
    layer.set_param("force_kernel", family)
    assert layer.describe(N).startswith(CONV_FAMILY_NAMES[family]), layer.describe(N)
    xd = torch.from_numpy(x).cuda()
    y = layer.forward(xd).cpu().numpy()
    assert close(y, ref) <= RTOL, close(y, ref)
    yr = layer.forward(xd, relu=True).cpu().numpy()
    assert close(yr, np.maximum(ref, 0)) <= RTOL
    if family in (1, 3):
        layer.set_src_nchw(True)
        yn = layer.forward(torch.from_numpy(po.nhwc_to_nchw(x)).cuda()).cpu().numpy()
        assert np.array_equal(yn, y)
    layer.close()


@pytest.mark.gpu
def test_supporting_layers(po, qcnn, ctx):
    import torch
    rng = np.random.RandomState(3)
    x = (rng.randn(3, 13, 15, 96) * 30).astype(np.float32)
    xd = torch.from_numpy(x).cuda()
    assert np.array_equal(ctx.relu(xd).cpu().numpy(), po.relu_f(x))
    lr = po.lrn_f(x, 5, 1e-4, 0.75, 1.0)
    assert close(ctx.lrn(xd, 5, 1e-4, 0.75, 1.0).cpu().numpy(), lr, 1e-5) <= 1e-5
    for (k, p, s) in [(3, 0, 2), (2, 0, 2), (3, 0, 3), (3, 1, 2)]:
        assert np.array_equal(ctx.maxpool(xd, k, p, s).cpu().numpy(), po.pool_f(x, k, p, s))
    fused = ctx.lrn_maxpool(xd, 5, 1e-4, 0.75, 1.0, 3, 0, 2).cpu().numpy()
    assert close(fused, po.pool_f(lr, 3, 0, 2), 1e-5) <= 1e-5
    z = (rng.randn(7, 1000) * 4).astype(np.float32)
    sm = ctx.softmax(torch.from_numpy(z).cuda()).cpu().numpy()
    ref = po.softmax_f(z)
    assert np.abs(sm - ref).max() <= 1e-6
    assert np.array_equal(sm.argmax(1), ref.argmax(1))
