"""Bit-packed FC assignment tables (qcnn_layer_set_param "asmt_packed", qcnn_net_set_asmt_packed): the table is kept at
b = log2(K) bits per index and every FC path unpacks it in the kernel.  The storage format never changes the plan, and the
same LUT entries are added in the same order, so packed and byte-table outputs are compared BIT FOR BIT, on every path:
the batch <= 4 chain (fc_chain.cu), the gather kernel (fc_aprx.cu: strict path and batches 5-95) and the tensor-core GEMM
(pq_gemm_tc.cu mode 2, batch >= 96; its NT = 64 instantiation in a child process with QCNN_FC_TC=1)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from test_gpu_fc_chain import CHAINS, make_fc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))

# (Din, Dout, S, K, d, NHWC source (H, W, C) or None): every FC shape of the chain tests (AlexNet fc6-fc8 among them:
# K = 16-256, d = 1, 2, 4, 8, Dout % 16 != 0, Dout > 4096, a partial last subspace, a recycled chain ring) + an NHWC source
ROWS = sorted({s + (None,) for shapes, _ in CHAINS for s in shapes}) + [(9216, 4096, 2304, 32, 4, (6, 6, 256))]
BATCHES = [1, 3, 40, 130, 256]


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def packed_width(K):
    b = int(np.log2(K))
    return b if b < 8 else 0


def make_row(rng, qcnn, ctx, row):
    Din, Dout, S, K, d, nhwc = row
    L, p = make_fc(rng, qcnn, ctx, Din, Dout, S, K, d)
    if nhwc:
        L.set_src_nhwc(*nhwc)
    return L, p


def run_cells(L, xd):
    """Output and describe() of every (N, tensor_core, fc_nsplit) cell."""
    out = {}
    for tc in (2, 1, 0):
        for ns in (0, 1):
            L.set_param("tensor_core", tc)
            L.set_param("fc_nsplit", ns)
            for N in BATCHES:
                out[(N, tc, ns)] = (L.forward(xd[:N]).cpu().numpy(), L.describe(N))
    L.set_param("tensor_core", 2)
    L.set_param("fc_nsplit", 0)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("ri", range(len(ROWS)))
def test_packed_bit_identity_matrix(ri, qcnn, ctx):
    import torch
    row = ROWS[ri]
    rng = np.random.RandomState(700 + ri)
    L, (ctrd, asmt, bias) = make_row(rng, qcnn, ctx, row)
    x = (np.abs(rng.randn(max(BATCHES), row[0])) * 2.0).astype(np.float32)
    xd = torch.from_numpy(x).cuda()
    base = run_cells(L, xd)
    L.set_param("asmt_packed", 1)
    packed = run_cells(L, xd)
    b = packed_width(row[3])
    paths = set()
    for key, (y, desc) in base.items():
        yp, descp = packed[key]
        assert np.array_equal(bits(yp), bits(y)), (row, key, desc)
        assert descp == desc + (" asmt=%dbit" % b if b else ""), (descp, desc)
        paths.add("chain" if "fc_chain" in desc else ("tc" if "pq_gemm_tc" in desc else "gather"))
    assert "gather" in paths, paths
    # the decoded table is the original one, and the layer goes back to its byte table and forth again unchanged
    assert np.array_equal(L.read_asmt(asmt.size), asmt.T.reshape(-1))
    y0 = base[(3, 2, 0)][0]
    L.set_param("asmt_packed", 0)
    assert np.array_equal(L.read_asmt(asmt.size), asmt.T.reshape(-1))
    assert np.array_equal(bits(L.forward(xd[:3]).cpu().numpy()), bits(y0))
    L.set_param("asmt_packed", 1)
    assert np.array_equal(bits(L.forward(xd[:3]).cpu().numpy()), bits(y0))
    assert np.array_equal(L.read_asmt(asmt.size), asmt.T.reshape(-1))
    L.close()


@pytest.mark.gpu
@pytest.mark.parametrize("ci", range(len(CHAINS)))
@pytest.mark.parametrize("N", [1, 3])
def test_packed_fc_chain_forward(ci, N, qcnn, ctx):
    import torch
    shapes, relu = CHAINS[ci]
    rng = np.random.RandomState(800 + ci)
    layers = [make_fc(rng, qcnn, ctx, *s)[0] for s in shapes]
    xd = torch.from_numpy((np.abs(rng.randn(N, shapes[0][0])) * 2.0).astype(np.float32)).cuda()
    y = qcnn.fc_chain_forward(layers, relu, xd).cpu().numpy()
    # only the first layer packed (a chain may mix both forms), then all of them
    for packed in ([1] + [0] * (len(layers) - 1), [1] * len(layers)):
        for L, p in zip(layers, packed):
            L.set_param("asmt_packed", p)
        for _ in range(3):
            yp = qcnn.fc_chain_forward(layers, relu, xd).cpu().numpy()
            assert np.array_equal(bits(yp), bits(y)), (ci, packed)
    for L in layers:
        L.close()


@pytest.mark.gpu
def test_packed_fc_chain_nhwc_source(qcnn, ctx):
    import torch
    rng = np.random.RandomState(5)
    H, W, Cc = 6, 6, 256
    l1, _ = make_fc(rng, qcnn, ctx, H * W * Cc, 4096, H * W * Cc // 4, 32, 4, std=0.02)
    l2, _ = make_fc(rng, qcnn, ctx, 4096, 1000, 4096, 16, 1, std=0.02)
    l1.set_src_nhwc(H, W, Cc)
    xd = torch.from_numpy((np.abs(rng.randn(2, H, W, Cc))).astype(np.float32)).cuda().view(2, -1)
    y = qcnn.fc_chain_forward([l1, l2], [1, 0], xd).cpu().numpy()
    l1.set_param("asmt_packed", 1)
    l2.set_param("asmt_packed", 1)
    assert "asmt=5bit" in l1.describe(1) and "asmt=4bit" in l2.describe(1)
    assert np.array_equal(bits(qcnn.fc_chain_forward([l1, l2], [1, 0], xd).cpu().numpy()), bits(y))
    l1.close()
    l2.close()


@pytest.mark.gpu
def test_packed_work_bytes(qcnn, ctx):
    rng = np.random.RandomState(9)
    total = 0
    for row in ROWS:
        Din, Dout, S, K = row[:4]
        L, _ = make_row(rng, qcnn, ctx, row)
        w0 = L.work(7)["alg_bytes"]
        L.set_param("asmt_packed", 1)
        w1 = L.work(7)["alg_bytes"]
        b = packed_width(K)
        if b:
            assert w1 - w0 == S * (-(-Dout * b // 8)) - S * Dout, row
        else:
            assert w1 == w0
        if row[5] is None and (Din, Dout, S, K) in [(9216, 4096, 2304, 32), (4096, 4096, 1024, 32), (4096, 1000, 4096, 16)]:
            total += S * (-(-Dout * b // 8))
        L.set_param("asmt_packed", 0)
        assert L.work(7)["alg_bytes"] == w0
        L.close()
    assert total == 10567680      # AlexNet fc6-fc8 at 5, 5 and 4 bits


@pytest.mark.gpu
def test_packed_errors_and_k256(qcnn, ctx):
    rng = np.random.RandomState(3)
    ctrd = (rng.randn(8, 16, 8) * 0.05).astype(np.float32)
    asmt = rng.randint(0, 16, size=(32, 3, 3, 8)).astype(np.uint8)
    conv = qcnn.ConvLayer(ctx, 64, 9, 9, 32, 3, 1, 1, 1, ctrd, asmt, np.zeros(32, np.float32))
    with pytest.raises(qcnn.QcnnError):
        conv.set_param("asmt_packed", 1)
    conv.close()
    L, (_, a, _) = make_fc(rng, qcnn, ctx, 128, 64, 16, 256, 8)
    d0, w0 = L.describe(3), L.work(3)
    L.set_param("asmt_packed", 1)        # accepted; at 8 bits the byte table stays
    assert L.describe(3) == d0 and L.work(3) == w0
    assert np.array_equal(L.read_asmt(a.size), a.T.reshape(-1))
    L.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["default", "strict"])
def test_packed_alexnet_net(po, qcnn, ctx, mode):
    """The shipped AlexNet: probabilities and logits of the packed net equal the byte-table net's bit for bit, including
    the captured batch-1 graph (recaptured after the switch)."""
    import torch
    if not po.have_alexnet():
        pytest.skip("shipped AlexNet parameters not staged under oracle/_ref/data")
    net = qcnn.Net(ctx, po.ALEXNET_DIR, po.ALEXNET_PFX, "AlexNet")
    fc = [l for l in range(net.layer_count) if net.pq_layer(l) is not None and
          net.pq_layer(l).describe(1).startswith("fc_aprx")]
    assert len(fc) == 3
    if mode == "strict":
        for l in range(net.layer_count):
            if net.pq_layer(l) is not None:
                net.pq_layer(l).set_param("tensor_core", 0)
    imgs = torch.from_numpy(po.lcg_images(256, 4242)).cuda()

    def run(N, reps):
        outs = []
        for _ in range(reps):
            lg = torch.empty((N, 1000), dtype=torch.float32, device="cuda")
            p = net.forward(imgs[:N].contiguous(), logits=lg)
            outs.append((p.cpu().numpy(), lg.cpu().numpy()))
        for p, lg in outs[1:]:
            assert np.array_equal(bits(p), bits(outs[0][0])) and np.array_equal(bits(lg), bits(outs[0][1]))
        return outs[0]

    plan = {N: (4 if N == 1 else 1) for N in (1, 3, 40, 256)}   # batch 1 runs eagerly first, then from its graph
    base = {N: run(N, r) for N, r in plan.items()}
    net.set_asmt_packed(True)
    for l in fc:
        assert " asmt=" in net.pq_layer(l).describe(1)
    for N, r in plan.items():
        p, lg = run(N, r)
        assert np.array_equal(bits(p), bits(base[N][0])), (mode, N)
        assert np.array_equal(bits(lg), bits(base[N][1])), (mode, N)
    net.set_asmt_packed(False)
    p, lg = run(1, 3)
    assert np.array_equal(bits(lg), bits(base[1][1]))
    net.close()


# NT = 64 tensor-core FC instantiation: QCNN_FC_TC=1 (read once per process) sends N <= 64 to the tensor cores
_CHILD = r"""
import importlib, json, sys
sys.path[:0] = [%r, %r]
import numpy as np, torch
import test_gpu_packed_asmt as t
q = importlib.import_module("quantized-cnn_b200")
ctx = q.Context(0)
res = []
for ri, row in enumerate(t.ROWS):
    rng = np.random.RandomState(900 + ri)
    L, _ = t.make_row(rng, q, ctx, row)
    xd = torch.from_numpy((np.abs(rng.randn(40, row[0])) * 2.0).astype(np.float32)).cuda()
    for tc in (2, 1):
        L.set_param("tensor_core", tc)
        for N in (5, 40):
            L.set_param("asmt_packed", 0)
            y, desc = L.forward(xd[:N]).cpu().numpy(), L.describe(N)
            L.set_param("asmt_packed", 1)
            yp = L.forward(xd[:N]).cpu().numpy()
            res.append(dict(row=ri, tc=tc, N=N, plan=desc, same=bool(np.array_equal(t.bits(y), t.bits(yp)))))
    L.close()
ctx.close()
print("RESULT " + json.dumps(res))
"""


@pytest.mark.gpu
def test_packed_fc_tc_nt64_child_process():
    env = dict(os.environ, QCNN_FC_TC="1")
    p = subprocess.run([sys.executable, "-c", _CHILD % (ROOT, TESTS)], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=900)
    assert p.returncode == 0, p.stderr[-4000:]
    res = json.loads([l for l in p.stdout.splitlines() if l.startswith("RESULT ")][-1][7:])
    assert any("NT=64" in r["plan"] for r in res)
    for r in res:
        assert r["same"], r
