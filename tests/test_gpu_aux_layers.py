"""The supporting layers of aux_layers.cu (max-pool, LRN, fused LRN + max-pool, softmax, permutes) against numpy and
float64 references, at every kernel and branch their launchers choose between.

Max-pool is exact: a window's maximum is one of its inputs.  The inputs are distinct and nonzero, so ties and +-0 (whose
order fmaxf leaves unspecified) do not occur, and every output is compared bit for bit.  A pooling geometry in which an
output window holds no input pixel (pad >= ksz, or (Ho - 1) stride - pad >= H) is rejected on the host.

LRN, y = x (k + alpha / size sum_window x^2)^-beta, against float64, relative to |y64| (U = 2^-24):
  window sum  each term fl(fl(x x) coeff) carries <= 3 U (alpha = 2^-13 is exact, coeff = alpha / size is rounded once);
              the `size` fp32 additions of nonnegative terms add <= size U of the sum:  e_s <= (size + 3) U
  power       exact path, expf(fl(-beta logf(s))): logf <= 1 ulp (2 U |ln s|), the product with -beta U |beta ln s|, expf
              <= 2 ulp (4 U) (CUDA C++ Programming Guide, single-precision function error bounds); beta is a binary
              fraction, so exact.  FAST075 (beta = 0.75): r = rsqrt.approx(s) <= 2^-22.9 relative, q = sqrt.approx(r) <=
              2^-23 + r's error halved, fl(r q) U (PTX ISA: rsqrt.approx.f32 / sqrt.approx.f32 maximum relative errors)
  output      beta e_s + power + U for the final product:
      exact    B = beta (size + 3) U + 3 beta U |ln s| + 5 U
      FAST075  B = 0.75 (size + 3) U + 1.5 2^-22.9 + 2^-23 + 2 U
  Fused LRN + max-pool: |max a - max b| <= max |a - b|, so the bound of an output is the max-pool of the LRN bounds.
Softmax, exp(x) / sum exp(x) without max subtraction: each exp <= 2 ulp (4 U), the sum of C positive terms has at most
  ceil(C / 256) + 5 + 8 roundings on any path (per-thread loop, warp tree, the 8 warp sums), the division U:
      B = (9 + ceil(C / 256) + 13) U  relative.
Measured worst err / bound on one NVIDIA H100 80GB HBM3 (700 W power limit): lrn_kernel 0.36, fused LRN + max-pool 0.43
(QCNN_LRN_RO=4: 0.41), softmax 0.15.  Every case's ratio goes to aux_layers_f64.json in the directory named by
QCNN_REPORT_DIR (default: qcnn_reports under the system temporary directory).
"""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))
U = 2.0 ** -24
ALPHA = 2.0 ** -13


# ------------------------------------------------------------------------------------------------------------------
# references
# ------------------------------------------------------------------------------------------------------------------
def pool_out(n, k, p, s):
    return -((-(n + 2 * p - k)) // s) + 1


def windows_nonempty(n, k, p, s):
    o = pool_out(n, k, p, s)
    return p < k and o >= 1 and (o - 1) * s - p < n


def legal(H, W, k, p, s):
    return windows_nonempty(H, k, p, s) and windows_nonempty(W, k, p, s)


def maxpool_ref(x, k, p, s):
    """NHWC max-pool with windows clipped to the map (reference CalcFeatMap_Pool), any dtype."""
    N, H, W, C = x.shape
    Ho, Wo = pool_out(H, k, p, s), pool_out(W, k, p, s)
    out = np.empty((N, Ho, Wo, C), x.dtype)
    for ho in range(Ho):
        h0, h1 = max(0, ho * s - p), min(H, ho * s + k - p)
        for wo in range(Wo):
            w0, w1 = max(0, wo * s - p), min(W, wo * s + k - p)
            out[:, ho, wo] = x[:, h0:h1, w0:w1].max(axis=(1, 2))
    return out


def lrn64(x, size, alpha, beta, k):
    """(y, s): float64 LRN across the channels of an NHWC map, and its window sums."""
    x = np.asarray(x, np.float64)
    C, rad = x.shape[-1], (size - 1) // 2
    sq = np.pad(x * x, [(0, 0)] * (x.ndim - 1) + [(rad, size - 1 - rad)])
    s = k + alpha / size * sum(sq[..., w:w + C] for w in range(size))
    return x * s ** -beta, s


def lrn_bound(s, size, beta, fast):
    if fast:
        return 0.75 * (size + 3) * U + 1.5 * 2.0 ** -22.9 + 2.0 ** -23 + 2 * U
    return beta * (size + 3) * U + 3 * beta * U * np.abs(np.log(s)) + 5 * U


def distinct(rng, shape):
    """Distinct nonzero values of both signs over several binades (no ties, no +-0)."""
    n = int(np.prod(shape))
    u = np.sort(10.0 ** rng.uniform(-2, 3, size=n)).astype(np.float32).view(np.int32).astype(np.int64)
    i = np.arange(n)
    u = np.maximum.accumulate(u - i) + i            # strictly increasing bit patterns: distinct positive floats
    v = u.astype(np.int32).view(np.float32)
    assert len(np.unique(v)) == n and (v > 0).all()
    v = v * np.where(rng.rand(n) < 0.5, -1, 1).astype(np.float32)
    return rng.permutation(v).reshape(shape)


def bits(y):
    return np.ascontiguousarray(y, np.float32).view(np.uint32)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the geometry rule and the references
# ------------------------------------------------------------------------------------------------------------------
def test_windows_nonempty_matches_enumeration():
    for n in range(1, 12):
        for k in range(1, 5):
            for p in range(0, 4):
                for s in range(1, 5):
                    o = pool_out(n, k, p, s)
                    brute = o >= 1 and all(max(0, i * s - p) < min(n, i * s + k - p) for i in range(o))
                    assert windows_nonempty(n, k, p, s) == brute, (n, k, p, s)


def test_reject_cases_are_empty_windows():
    for (H, k, p, s) in REJECT:
        assert not windows_nonempty(H, k, p, s)
    # the example: N = 1, H = W = 2, 3x3 pool, stride 3, pad 1: Ho = 2, and output row 1 would start at input row 2
    assert pool_out(2, 3, 1, 3) == 2 and 1 * 3 - 1 == 2


def test_lrn_bound_covers_fp32_emulation():
    """A numpy fp32 emulation of the exact path (same operation order, libm-rounded exp / log) stays within B."""
    rng = np.random.RandomState(5)
    x = distinct(rng, (64, 24))
    for size in (3, 5, 7):
        for beta in (0.75, 0.625):
            ref, s = lrn64(x, size, ALPHA, beta, 1.0)
            coeff = np.float32(np.float32(ALPHA) / np.float32(size))
            C, rad = x.shape[-1], (size - 1) // 2
            t = np.pad((x * x) * coeff, [(0, 0), (rad, size - 1 - rad)])
            acc = np.full(x.shape, np.float32(1.0), np.float32)
            for w in range(size):
                acc = acc + t[:, w:w + C]
            y = x * np.exp(np.float32(-beta) * np.log(acc))
            assert y.dtype == np.float32
            err = np.abs(y.astype(np.float64) - ref) / np.abs(ref)
            assert (err <= lrn_bound(s, size, beta, False)).all(), (size, beta, float(err.max()))


# ------------------------------------------------------------------------------------------------------------------
# GPU: rejected geometries (host checks: nothing is launched)
# ------------------------------------------------------------------------------------------------------------------
# (H = W, ksz, pad, stride): pad >= ksz; stride 3 / pad 1; stride 3 / pad 2; stride 2 / pad 2
REJECT = [(5, 2, 2, 1), (6, 3, 3, 2), (2, 3, 1, 3), (5, 3, 1, 3), (4, 3, 2, 3), (4, 3, 2, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("H,k,p,s", REJECT)
def test_empty_pool_window_rejected(H, k, p, s, po, qcnn, ctx, tmp_path):
    import torch
    for C in (4, 5, 8):
        x = torch.ones((1, H, H, C), dtype=torch.float32, device="cuda")
        with pytest.raises(qcnn.QcnnError, match="holds no input pixel"):
            ctx.maxpool(x, k, p, s)
        with pytest.raises(qcnn.QcnnError, match="holds no input pixel"):
            ctx.lrn_maxpool(x, 5, ALPHA, 0.75, 1.0, k, p, s)
    # at net creation, from a custom layer table
    layers = [po.conv(0, 1, 16, 1, 1), po.relu(), po.pool(p, k, s)]
    chw = (4, H, H)
    po.save_model(str(tmp_path), "c", po.synth_model(layers, chw, {0: (1, 16, 4)}, seed=1))
    infos = [qcnn.LayerInfo(L["type"], L.get("pad", 0), L.get("k", 0), L.get("cnt", 0), L.get("grp", 0),
                            L.get("stride", 0), L.get("nod", 0), L.get("size", 0), L.get("alpha", 0.0),
                            L.get("beta", 0.0), L.get("kini", 0.0), L.get("ratio", 0.0)) for L in layers]
    with pytest.raises(qcnn.QcnnError, match="without input pixels"):
        qcnn.Net(ctx, str(tmp_path), "c", layers=infos, in_chw=chw)


# ------------------------------------------------------------------------------------------------------------------
# GPU: max-pool, bit-exact
# ------------------------------------------------------------------------------------------------------------------
def pool_geometries(H, W):
    return [(k, p, s) for k in (2, 3) for s in (1, 2, 3) for p in (0, 1, 2) if legal(H, W, k, p, s)]


MAPS = [(2, 9, 13), (1, 10, 7), (3, 6, 6)]


def test_pool_geometries_reach_every_branch():
    g = [(H, W, k, p, s) for (_, H, W) in MAPS for (k, p, s) in pool_geometries(H, W)]
    assert {(k, s) for (_, _, k, _, s) in g} == {(k, s) for k in (2, 3) for s in (1, 2, 3)}
    assert {p for (_, _, _, p, _) in g} == {0, 1, 2}
    assert any(H != W for (H, W, _, _, _) in g)
    # the last window clipped on the bottom / right edge (ceil output size)
    assert any((pool_out(H, k, p, s) - 1) * s - p + k > H for (H, W, k, p, s) in g)
    assert any((pool_out(W, k, p, s) - 1) * s - p + k > W for (H, W, k, p, s) in g)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [5, 6, 8, 12], ids=["C5-scalar", "C6-scalar", "C8-float4", "C12-float4"])
def test_maxpool_bit_exact(C, ctx):
    """C % 4 != 0: maxpool_kernel; C % 4 == 0: maxpool4_kernel, <true> for 3x3 windows, <false> for 2x2."""
    import torch
    rng = np.random.RandomState(C)
    for (N, H, W) in MAPS:
        x = distinct(rng, (N, H, W, C))
        xd = torch.from_numpy(x).cuda()
        for (k, p, s) in pool_geometries(H, W):
            y = ctx.maxpool(xd, k, p, s).cpu().numpy()
            assert np.array_equal(bits(y), bits(maxpool_ref(x, k, p, s))), (N, H, W, k, p, s)


# ------------------------------------------------------------------------------------------------------------------
# GPU: LRN and fused LRN + max-pool against float64
# ------------------------------------------------------------------------------------------------------------------
REPORT = {}


def check_lrn(name, y, ref, bound_map):
    ratio = float((np.abs(np.asarray(y, np.float64) - ref) / np.maximum(bound_map, 1e-300)).max())
    REPORT[name] = ratio
    assert np.isfinite(y).all(), name
    assert ratio <= 1.0, (name, ratio)


@pytest.mark.gpu
@pytest.mark.parametrize("size", [3, 5, 7])
def test_lrn_f64(size, ctx):
    """lrn_kernel (exact power path), C >= size and C < size."""
    import torch
    rng = np.random.RandomState(size)
    for C in (size - 1, 16, 37):
        for beta in (0.75, 0.625):
            x = distinct(rng, (2, 5, 7, C))
            ref, s = lrn64(x, size, ALPHA, beta, 1.0)
            y = ctx.lrn(torch.from_numpy(x).cuda(), size, ALPHA, beta, 1.0).cpu().numpy()
            check_lrn("lrn/size%d/C%d/beta%g" % (size, C, beta), y, ref, lrn_bound(s, size, beta, False) * np.abs(ref))


def tiled_kernel(size, C, beta, k, p, s):
    """The instantiation LaunchLrnMaxPool's tiled path picks: (SIZE, FAST075, K3)."""
    if size == 5 and C % 8 == 0:
        return (5, beta == 0.75, k == 3 and s <= 3 and p <= 2)
    return (0, False, False)


# (N, H, W, C, size, beta, ksz, pad, stride): the five tiled instantiations, both pooling loops of <0, ...>, a tile
# over 48 KB (opt-in shared memory), the untiled fallback through a tile over 160 KB
FUSED = [
    (2, 9, 11, 16, 5, 0.75, 3, 0, 2),      # <5, true, true>
    (2, 8, 9, 24, 5, 0.75, 2, 0, 2),       # <5, true, false>
    (2, 9, 10, 16, 5, 0.625, 3, 1, 2),     # <5, false, true>
    (1, 7, 8, 8, 5, 0.625, 2, 1, 1),       # <5, false, false>
    (2, 7, 9, 12, 5, 0.75, 3, 0, 2),       # <0, ...>, C % 4 == 0, C % 8 != 0: float4 pooling loop
    (2, 7, 9, 7, 3, 0.75, 3, 1, 3),        # <0, ...>, C odd: scalar pooling loop
    (1, 8, 8, 16, 7, 0.625, 2, 0, 2),      # <0, ...>, size 7
    (1, 6, 56, 96, 5, 0.75, 3, 0, 2),      # tile 3 x 56 x 96 floats = 63 KB
    (1, 5, 112, 128, 5, 0.75, 3, 0, 2),    # tile 168 KB: lrn_maxpool_kernel
]


def fused_ref(x, size, beta, k, p, s, fast):
    lr, sums = lrn64(x, size, ALPHA, beta, 1.0)
    return maxpool_ref(lr, k, p, s), maxpool_ref(lrn_bound(sums, size, beta, fast) * np.abs(lr), k, p, s)


def fused_fast(N, H, W, C, size, beta, k, p, s):
    """The FAST075 power path runs (tiled kernel, one output row per CTA's tile size)."""
    tile = 4 * k * W * C
    return tile <= 160 * 1024 and N <= 65535 and tiled_kernel(size, C, beta, k, p, s)[1]


def test_fused_table_reaches_every_branch():
    kern = lambda r: tiled_kernel(r[4], r[3], r[5], r[6], r[7], r[8])
    tiled = [r for r in FUSED if 4 * r[6] * r[2] * r[3] <= 160 * 1024]
    assert {kern(r) for r in tiled} == {(5, True, True), (5, True, False), (5, False, True), (5, False, False),
                                        (0, False, False)}
    zero = [r for r in tiled if kern(r)[0] == 0]
    assert any(r[3] % 4 == 0 for r in zero) and any(r[3] % 4 for r in zero)
    assert any(4 * r[6] * r[2] * r[3] > 48 * 1024 for r in tiled)
    assert any(4 * r[6] * r[2] * r[3] > 160 * 1024 for r in FUSED)
    assert all(legal(r[1], r[2], *r[6:]) for r in FUSED)


@pytest.mark.gpu
@pytest.mark.parametrize("case", FUSED, ids=["N%d-%dx%dx%d-size%d-beta%g-k%dp%ds%d" % c for c in FUSED])
def test_lrn_maxpool_f64(case, ctx):
    import torch
    N, H, W, C, size, beta, k, p, s = case
    rng = np.random.RandomState(H * W + C)
    x = distinct(rng, (N, H, W, C))
    ref, bmap = fused_ref(x, size, beta, k, p, s, fused_fast(*case))
    xd = torch.from_numpy(x).cuda()
    y = ctx.lrn_maxpool(xd, size, ALPHA, beta, 1.0, k, p, s).cpu().numpy()
    check_lrn("lrn_maxpool/%s" % (case,), y, ref, bmap)
    assert np.array_equal(bits(y), bits(ctx.lrn_maxpool(xd, size, ALPHA, beta, 1.0, k, p, s).cpu().numpy()))


@pytest.mark.gpu
def test_lrn_maxpool_untiled_by_batch(ctx):
    """N = 65536 images exceed the tiled kernel's grid: lrn_maxpool_kernel on a 3 x 3 x 8 map (~19 MB)."""
    import torch
    rng = np.random.RandomState(65536)
    x = (rng.uniform(1, 1e3, size=(65536, 3, 3, 8)) * np.where(rng.rand(65536, 3, 3, 8) < 0.5, -1, 1)).astype(np.float32)
    ref, bmap = fused_ref(x, 5, 0.75, 2, 0, 1, False)
    y = ctx.lrn_maxpool(torch.from_numpy(x).cuda(), 5, ALPHA, 0.75, 1.0, 2, 0, 1).cpu().numpy()
    check_lrn("lrn_maxpool/N65536", y, ref, bmap)


_CHILD = r"""
import importlib, json, sys
sys.path[:0] = [%r, %r]
import numpy as np, torch
import test_gpu_aux_layers as t
q = importlib.import_module("quantized-cnn_b200")
ctx = q.Context(0)
res = []
for case in t.FUSED[:7] + [(3, 13, 15, 96, 5, 0.75, 3, 0, 2)]:
    N, H, W, C, size, beta, k, p, s = case
    rng = np.random.RandomState(H * W + C + 1)
    x = t.distinct(rng, (N, H, W, C))
    ref, bmap = t.fused_ref(x, size, beta, k, p, s, t.fused_fast(*case))
    xd = torch.from_numpy(x).cuda()
    y = ctx.lrn_maxpool(xd, size, t.ALPHA, beta, 1.0, k, p, s).cpu().numpy()
    y2 = ctx.lrn_maxpool(xd, size, t.ALPHA, beta, 1.0, k, p, s).cpu().numpy()
    ratio = float((np.abs(y.astype(np.float64) - ref) / np.maximum(bmap, 1e-300)).max())
    res.append(dict(case=case, ratio=ratio, finite=bool(np.isfinite(y).all()),
                    same=bool(np.array_equal(t.bits(y), t.bits(y2)))))
ctx.close()
print("RESULT " + json.dumps(res))
"""


@pytest.mark.gpu
def test_lrn_maxpool_ro4_child_process():
    """Several output rows per CTA (ro > 1) only through QCNN_LRN_RO, read once per process: a child process."""
    env = dict(os.environ, QCNN_LRN_RO="4")
    p = subprocess.run([sys.executable, "-c", _CHILD % (ROOT, TESTS)], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-4000:]
    res = json.loads([l for l in p.stdout.splitlines() if l.startswith("RESULT ")][-1][7:])
    assert len(res) == 8
    for r in res:
        REPORT["lrn_maxpool_ro4/%s" % (tuple(r["case"]),)] = r["ratio"]
        assert r["finite"] and r["same"] and r["ratio"] <= 1.0, r


# ------------------------------------------------------------------------------------------------------------------
# GPU: softmax and permutes
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 31, 257, 1000, 4097])
def test_softmax_f64(C, ctx):
    import torch
    rng = np.random.RandomState(C)
    z = (rng.randn(5, C) * 4).astype(np.float32)
    e = np.exp(z.astype(np.float64))
    ref = e / e.sum(axis=1, keepdims=True)
    zd = torch.from_numpy(z).cuda()
    y = ctx.softmax(zd).cpu().numpy()
    bound = (9 + -(-C // 256) + 13) * U
    ratio = float((np.abs(y - ref) / ref).max()) / bound
    REPORT["softmax/C%d" % C] = ratio
    assert ratio <= 1.0, ratio
    assert np.array_equal(bits(y), bits(ctx.softmax(zd).cpu().numpy()))


@pytest.mark.gpu
def test_permutes_bit_exact(ctx):
    import torch
    rng = np.random.RandomState(9)
    for (N, C, H, W) in [(3, 5, 7, 9), (1, 1, 3, 5), (2, 33, 1, 7)]:
        x = distinct(rng, (N, C, H, W))
        xd = torch.from_numpy(x).cuda()
        nhwc = ctx.nchw_to_nhwc(xd)
        assert np.array_equal(bits(nhwc.cpu().numpy()), bits(np.transpose(x, (0, 2, 3, 1))))
        assert np.array_equal(bits(ctx.nhwc_to_nchw(nhwc).cpu().numpy()), bits(x))


@pytest.mark.gpu
def test_report(ctx):
    """Writes err / bound of the LRN and softmax cases that ran in this session to aux_layers_f64.json."""
    out = os.environ.get("QCNN_REPORT_DIR") or os.path.join(tempfile.gettempdir(), "qcnn_reports")
    try:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "aux_layers_f64.json"), "w") as f:
            json.dump(REPORT, f, indent=1, sort_keys=True)
    except OSError:
        pass
    print("\nworst err/bound: %s" % (max(REPORT.values()) if REPORT else None))
