"""The choice among the FC kernel families (fc_plan.cu), seen through describe().

The rule, first that applies:
  chain    N <= 4 and the persistent kernel takes the layer ("fc_chain(")
  fc_ws    fc_ws = 1, bf16x2 operands (tensor_core = 2) and the tensor-core conditions ("pq_gemm_tc_ws(")
  mode 2   the tensor-core conditions: tensor_core != 0, no fc_nsplit / fc_tn pin, N >= 96 (QCNN_FC_TC=1: any N) and a
           geometry the decoders read ("pq_gemm_tc(... mode=2")
  gather   otherwise (no " via ")
Every layer below has a geometry that the chain, fc_ws and mode 2 all take, so the cell alone decides the family.  A
forward runs what describe() names: describe() is the same before and after it.  A child process checks the case where
QCNN_FC_TC=1 sends a batch <= 4 to the tensor cores while QCNN_FC_CHAIN=0 keeps the chain out (both read once per
process): describe() names the tensor-core family and the output is within that family's float64 bound.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from test_gpu_pq_gemm import FcRow, fc_data

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))

ROWS = [
    FcRow("alexnet_fc6", 256, 9216, 4096, 2304, 32, 4, None),
    FcRow("alexnet_fc7", 256, 4096, 4096, 1024, 32, 4, None),
    FcRow("alexnet_fc8", 256, 4096, 1000, 4096, 16, 1, None),
    FcRow("d1_k64", 256, 512, 200, 512, 64, 1, None),
    FcRow("k256_d8", 256, 1024, 300, 128, 256, 8, None),
    FcRow("alexnet_fc6_nhwc", 256, 9216, 4096, 2304, 32, 4, (6, 6, 256)),
]
BATCHES = (1, 4, 5, 95, 96, 256)


def expected_family(N, tc, fc_ws, fc_nsplit):
    if N <= 4 and not fc_nsplit:
        return "fc_chain("
    if tc and not fc_nsplit and N >= 96:
        return "pq_gemm_tc_ws(" if fc_ws and tc == 2 else "pq_gemm_tc("
    return None


def assert_family(desc, fam, tc, packed_bits):
    assert desc.endswith(" asmt=%dbit" % packed_bits) == bool(packed_bits), desc
    if fam is None:
        assert " via " not in desc, desc
        return
    via = desc.split(" via ")[1]
    assert via.startswith(fam), (fam, desc)
    if fam == "pq_gemm_tc(":
        assert " mode=2 " in via and ("bf16x2" in via) == (tc == 2), desc


@pytest.mark.gpu
@pytest.mark.parametrize("name", [r.name for r in ROWS])
def test_fc_plan_table(name, qcnn, ctx):
    """Every (N, tensor_core, fc_ws, fc_nsplit, asmt_packed) cell: describe() names the family the rule gives, and the
    same one after a forward."""
    import torch
    row = {r.name: r for r in ROWS}[name]
    x, ctrd, asmt, bias = fc_data(row)
    L = qcnn.FcLayer(ctx, row.Din, ctrd, asmt, bias)
    if row.nhwc:
        L.set_src_nhwc(*row.nhwc)
    xd = torch.from_numpy(x).cuda().view(row.N, -1)
    seen = set()
    for packed in (0, 1):
        L.set_param("asmt_packed", packed)
        bits = int(np.log2(row.K)) if packed and row.K < 256 else 0
        for tc in (0, 1, 2):
            for fc_ws in (0, 1):
                for ns in (0, 1):
                    L.set_param("tensor_core", tc)
                    L.set_param("fc_ws", fc_ws)
                    L.set_param("fc_nsplit", ns)
                    for N in BATCHES:
                        fam = expected_family(N, tc, fc_ws, ns)
                        before = L.describe(N)
                        assert_family(before, fam, tc, bits)
                        y = L.forward(xd[:N]).cpu().numpy()
                        assert y.shape == (N, row.Dout) and np.isfinite(y).all(), before
                        assert L.describe(N) == before
                        seen.add(fam)
    L.close()
    assert seen == {"fc_chain(", "pq_gemm_tc_ws(", "pq_gemm_tc(", None}


_CHILD = r"""
import importlib, json, sys
sys.path[:0] = [%r, %r]
import numpy as np, torch
import test_gpu_pq_gemm as t
import test_gpu_fc_plan as p
q = importlib.import_module("quantized-cnn_b200")
ctx = q.Context(0)
res = []
for row in p.CHILD_ROWS:
    x, ctrd, asmt, bias = t.fc_data(row)
    L = q.FcLayer(ctx, row.Din, ctrd, asmt, bias)
    for tc in (2, 1):
        for fc_ws in (0, 1):
            L.set_param("tensor_core", tc)
            L.set_param("fc_ws", fc_ws)
            for N in (1, 4):
                ref, mag = t.ref64("fc", x[:N], ctrd, asmt, bias)
                before = L.describe(N)
                y = L.forward(torch.from_numpy(x[:N]).cuda()).cpu().numpy()
                res.append(dict(name=row.name, N=N, tc=tc, fc_ws=fc_ws, plan=before, after=L.describe(N),
                                err=t.f64_err(y, ref, mag)))
    L.close()
ctx.close()
print("RESULT " + json.dumps(res))
"""

CHILD_ROWS = [
    FcRow("child_d4", 4, 1024, 300, 256, 32, 4, None),
    FcRow("child_d1", 4, 512, 200, 512, 16, 1, None),
]


@pytest.mark.gpu
def test_fc_tc_small_batch_without_chain_child_process():
    """QCNN_FC_TC=1 and QCNN_FC_CHAIN=0 at N = 1 and 4: describe() names what runs (fc_ws, or mode 2 at NT = 64), and the
    output is within that family's bound."""
    from test_gpu_pq_gemm import tc_bound
    env = dict(os.environ, QCNN_FC_TC="1", QCNN_FC_CHAIN="0")
    p = subprocess.run([sys.executable, "-c", _CHILD % (ROOT, TESTS)], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-4000:]
    res = json.loads([l for l in p.stdout.splitlines() if l.startswith("RESULT ")][-1][7:])
    assert len(res) == 8 * len(CHILD_ROWS)
    for r in res:
        assert r["after"] == r["plan"], r
        assert " via " in r["plan"], r
        via = r["plan"].split(" via ")[1]
        ks = int(via.split(" ksteps=")[1].split()[0])
        ns = int(via.split(" nsplit=")[1].split()[0])
        if r["tc"] == 2 and r["fc_ws"]:
            assert via.startswith("pq_gemm_tc_ws("), r
            bound = tc_bound(True, 128, ks, ns)
        else:
            assert via.startswith("pq_gemm_tc(") and " mode=2 " in via and " NT=64 " in via, r
            assert ("bf16x2" in via) == (r["tc"] == 2), r
            bound = tc_bound(r["tc"] == 2, 64, ks, ns)
        assert r["err"] <= bound, (r, bound)
