"""Batch-1..4 latency path of the FC layers: the persistent assignment-stream kernel (csrc/fc_chain.cu) through the
C ABI (qcnn_fc_chain_forward, and qcnn_fc_aprx_forward / qcnn_net_forward, which route small batches to it) against
the CPU oracle.

Tolerance: the kernel adds the same fp32 LUT entries as the reference (LUT entries bit-identical: separate rounded
multiply and add, ascending j) but associates the sum differently -- per CTA s-ascending over its share (one CTA per SM) of the
subspaces, then a fixed tree over the CTAs -- so results agree to fp32 re-association noise: RTOL = 1e-4 under the
metric of test_gpu_layers.close (measured ~1e-6), and are bit-identical from run to run (no atomics).  The stricter check
is test_gpu_fc_gather_chain.py: every branch of the kernel against a float64 bound propagated through the chain,
(d + S + 3) U M per layer (measured worst err / bound 0.0098 on an H100 80GB HBM3 at 700 W)."""
import numpy as np
import pytest

from test_gpu_layers import RTOL, close, rand_act


def make_fc(rng, qcnn, ctx, Din, Dout, S, K, d, std=0.05):
    ctrd = (rng.randn(S, K, d) * std).astype(np.float32)
    asmt = rng.randint(0, K, size=(Dout, S)).astype(np.uint8)
    bias = (rng.randn(Dout) * 0.1).astype(np.float32)
    return qcnn.FcLayer(ctx, Din, ctrd, asmt, bias), (ctrd, asmt, bias)


def ref_chain(po, x, params, relu):
    for (ctrd, asmt, bias), r in zip(params, relu):
        x = po.fc_aprx(x, ctrd, asmt, bias)
        if r:
            x = np.maximum(x, 0)
    return x


CHAINS = [
    # list of (Din, Dout, S, K, d) per layer, relu flags
    ([(9216, 4096, 2304, 32, 4), (4096, 4096, 1024, 32, 4), (4096, 1000, 4096, 16, 1)], [1, 1, 0]),   # AlexNet fc6-fc8
    ([(512, 200, 128, 32, 4), (200, 96, 50, 64, 4)], [1, 0]),          # fewer subspaces than CTAs, Dout % 16 != 0
    ([(300, 96, 40, 128, 8)], [0]),                                    # Din not a multiple of d: partial last subspace
    ([(128, 64, 16, 256, 8), (64, 520, 16, 16, 4), (520, 40, 130, 32, 4), (40, 24, 40, 16, 1)], [0, 1, 1, 1]),  # 4 layers
    ([(2048, 6000, 512, 32, 4)], [1]),                                 # 16 channels per thread (Dout > 4096)
    ([(640, 2500, 320, 64, 2)], [0]),                                  # 8 channels per thread, d = 2
    ([(28416, 4096, 7104, 32, 4), (4096, 520, 1024, 32, 4)], [1, 0]),  # 48 rows x 4 KB per CTA: the ring is recycled
]


@pytest.mark.gpu
@pytest.mark.parametrize("ci", range(len(CHAINS)))
@pytest.mark.parametrize("N", [1, 3])
def test_fc_chain_parity(ci, N, po, qcnn, ctx):
    import torch
    shapes, relu = CHAINS[ci]
    rng = np.random.RandomState(100 + ci)
    layers, params = [], []
    for (Din, Dout, S, K, d) in shapes:
        L, p = make_fc(rng, qcnn, ctx, Din, Dout, S, K, d)
        layers.append(L)
        params.append(p)
    x = rand_act(rng, (N, shapes[0][0]), scale=2.0)
    ref = ref_chain(po, x, params, relu)
    xd = torch.from_numpy(x).cuda()
    y = qcnn.fc_chain_forward(layers, relu, xd).cpu().numpy()
    assert y.shape == ref.shape
    assert close(y, ref) <= RTOL, close(y, ref)
    # the ready-flag words were re-armed by their consumers: the same buffers serve the next calls; deterministic
    for _ in range(3):
        y2 = qcnn.fc_chain_forward(layers, relu, xd).cpu().numpy()
        assert np.array_equal(y2, y)
    # on another stream
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        y3 = qcnn.fc_chain_forward(layers, relu, xd)
    side.synchronize()
    assert np.array_equal(y3.cpu().numpy(), y)
    # the per-layer entry point takes the same kernel at batch <= 4 (a chain of one layer) ...
    assert "fc_chain" in layers[0].describe(N)
    z = xd
    for L, r in zip(layers, relu):
        z = L.forward(z, relu=bool(r))
    assert close(z.cpu().numpy(), ref) <= RTOL
    # ... unless the reference's exact accumulation order is requested: bit-exact against the oracle
    z = xd
    for L, r in zip(layers, relu):
        L.set_param("fc_nsplit", 1)
        z = L.forward(z, relu=bool(r))
    assert np.array_equal(z.cpu().numpy(), ref)
    with pytest.raises(qcnn.QcnnError):
        qcnn.fc_chain_forward(layers, relu, xd)     # overrides select the per-layer kernels: the fused call says so
    for L in layers:
        L.close()


@pytest.mark.gpu
def test_fc_chain_nhwc_source_and_stamps(po, qcnn, ctx):
    """First layer reading an NHWC map (the reference permutes to NCHW first, CaffeEva.cc:236-238) + the timing stamps."""
    import torch
    rng = np.random.RandomState(5)
    H, W, Cc = 6, 6, 256
    Din = H * W * Cc
    l1, p1 = make_fc(rng, qcnn, ctx, Din, 4096, Din // 4, 32, 4, std=0.02)
    l2, p2 = make_fc(rng, qcnn, ctx, 4096, 1000, 4096, 16, 1, std=0.02)
    l1.set_src_nhwc(H, W, Cc)
    x = rand_act(rng, (2, H, W, Cc), scale=1.0)
    ref = ref_chain(po, po.nhwc_to_nchw(x).reshape(2, -1), [p1, p2], [1, 0])
    stamps = torch.zeros(32 * ctx.sm_count, dtype=torch.int64, device="cuda")
    y = qcnn.fc_chain_forward([l1, l2], [1, 0], torch.from_numpy(x).cuda().view(2, -1), stamps=stamps).cpu().numpy()
    assert close(y, ref) <= RTOL, close(y, ref)
    st = stamps.cpu().numpy().reshape(-1, 32)
    assert (st[:, 0] > 0).all() and (st[:, 1] > st[:, 0]).all()
    span_us = (st[:, 1].max() - st[:, 0].min()) / 1e3
    assert span_us < 1000.0      # sanity: one launch of the second image, microseconds
    l1.close()
    l2.close()
