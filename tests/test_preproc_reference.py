"""Both ends of the PQ path against the compiled reference, without a GPU: the BMP recipe of BmpImgIO::Load (reference
src/BmpImgIO.cc) on generated pictures, and the k-fold arg-max of CaffeEva::CvtFeatMapToLablVec (src/CaffeEva.cc:
1162-1190) on generated probability vectors.

This module also owns the generated inputs that tests/test_gpu_preproc_edges.py feeds to the device:
  * a BMP writer (24 bpp, bottom-up, row padding of 0-3 bytes, optionally a gap between the header and the pixels);
  * a set of (recipe, source size) cases and a CPU mirror of the resize / crop index arithmetic that names the branch
    each case reaches: upscaling, a source equal to the full size, yh / xh clamping at the last source row / column
    (with fl(s*y) exactly on hs - 1 and past it), fl(s*y) rounding up onto an integer, odd and even crop offsets,
    non-square sizes, crop equal to full, every accepted (resize, mean) pair;
  * probability rows with NaN (at index 0, inside a thread's stride, past 256, everywhere), +-inf, -0.0 / 0.0 ties,
    equal, negative and sub-FLT_MIN values.
The reference, the C++ host port (qcnn_host_load_bmp) and the numpy restatement must agree bit for bit on every
case; the oracle's restatement of CvtFeatMapToLablVec must equal the reference on every row."""
import ctypes as C
import hashlib
import os
import struct

import numpy as np
import pytest

from test_gpu_preproc import decode_bmp, resz_crop_numpy

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "quantized-cnn_b200")
FLT_MIN = np.float32(1.17549435e-38)
GOLDEN = os.path.join(ROOT, "tests", "golden", "preproc_topk_ref.npz")


def _ref_has(*names):
    path = os.path.join(ROOT, "oracle", "_ref", "libqcnn_ref.so")
    if not os.path.exists(path):
        return False
    lib = C.CDLL(path)
    return all(hasattr(lib, n) for n in names)


needs_ref = pytest.mark.skipif(not _ref_has("ref_bmp_load", "ref_cvt_featmap_to_labl"),
                               reason="compiled reference with ref_bmp_load / ref_cvt_featmap_to_labl not built "
                                      "under oracle/_ref")


# ------------------------------------------------------------------------------------------------
# BMP writer
# ------------------------------------------------------------------------------------------------
def write_bmp(path, img, gap=0):
    """uint8 [H, W, 3] (B, G, R, top row first) -> 24-bpp uncompressed bottom-up BMP; `gap` bytes of junk sit between
    the 54-byte header and the pixels (off_bits says where the pixels start)."""
    h, w = img.shape[:2]
    row = (w * 3 + 3) & ~3
    body = np.zeros((h, row), np.uint8)
    body[:, :w * 3] = img[::-1].reshape(h, w * 3)
    body[:, w * 3:] = 0xA5                                       # padding bytes are never pixels
    off = 54 + gap
    hdr = struct.pack("<2sIHHI", b"BM", off + body.size, 0, 0, off)
    hdr += struct.pack("<IiiHHIIiiII", 40, w, h, 1, 24, 0, body.size, 2835, 2835, 0, 0)
    with open(path, "wb") as f:
        f.write(hdr + bytes([0x5A]) * gap + body.tobytes())


def make_image(hs, ws, seed):
    return np.random.RandomState(seed).randint(0, 256, size=(hs, ws, 3)).astype(np.uint8)


# ------------------------------------------------------------------------------------------------
# recipes, sizes and the CPU mirror of the index arithmetic
# ------------------------------------------------------------------------------------------------
# (name, resz_type 0 Strict / 1 Relaxed, mean_type 0 Full / 1 Crop, hei_full, wid_full, hei_crop, wid_crop)
RECIPES = [
    ("alexnet", 0, 0, 256, 256, 227, 227),          # CaffeEvaWrapper's recipe: odd offsets (29) on both axes
    ("strict_cropmean", 0, 1, 256, 256, 227, 227),
    ("vgg", 1, 1, 256, 256, 224, 224),              # VggCnnS: Relaxed, crop-size mean
    ("rect_strict", 0, 0, 256, 320, 224, 288),      # non-square full and crop
    ("rect_relaxed", 1, 1, 256, 320, 224, 288),
    ("rect_odd", 0, 1, 33, 20, 30, 17),             # odd offsets 3 / 3 at non-square sizes
    ("whole_strict", 0, 0, 48, 64, 48, 64),         # crop == full: the crop reaches the last resized row / column
    ("whole_relaxed", 1, 1, 40, 40, 40, 40),
]
RECIPE = {r[0]: r for r in RECIPES}
BASE_SIZES = [(2, 2), (2, 700), (700, 2), (3, 3), (2, 5), (100, 100), (13, 7), (256, 256), (517, 333), (240, 700),
              (1999, 1500), (1200, 2000), (2000, 37)]
MAX_RESIZED = 3 << 20                               # the reference resizes the whole picture: keep that cheap


def geometry(recipe, hs, ws):
    """(sh, sw, hd, wd, q_h, q_w) exactly as ReszImg computes them (float scales, double + kEpsilon)."""
    _, resz, _, hf, wf, _, _ = recipe
    f32 = np.float32
    sh, sw = f32(hs - 1) / f32(hf - 1), f32(ws - 1) / f32(wf - 1)
    hd, wd, qh, qw = hf, wf, None, None
    if resz == 1:
        sh = min(sh, sw)
        sw = min(sh, sw)
        qh, qw = f32(hs - 1) / sh, f32(ws - 1) / sw
        hd = int(np.float64(qh) + 0.0000001) + 1
        wd = int(np.float64(qw) + 0.0000001) + 1
    return sh, sw, hd, wd, qh, qw


def accepted(recipe, hs, ws):
    """What qcnn_preproc_run accepts (and where the reference's CropImg stays inside the resized picture)."""
    _, _, _, _, _, hc, wc = recipe
    _, _, hd, wd, _, _ = geometry(recipe, hs, ws)
    return hs >= 2 and ws >= 2 and hd >= hc and wd >= wc


def _axis_branches(s, n_src, n_dst, crop, tag):
    off = (n_dst - crop) // 2
    pos = np.arange(off, off + crop)
    c32 = (s * pos.astype(np.float32)).astype(np.float32)            # fl(s * y), as the kernel computes it
    exact = np.float64(s) * pos                                      # exact: 24-bit s times an 11-bit integer
    lo = np.maximum(0, c32.astype(np.int64))
    out = {"odd_%soff" % tag if (n_dst - crop) % 2 else "even_%soff" % tag}
    if s < 1:
        out.add("upscale_" + tag)
    if np.any(lo + 1 > n_src - 1):
        out.add(tag + "clamp")
        if np.any(c32 == n_src - 1):
            out.add(tag + "clamp_exact")
        if np.any(c32 > n_src - 1):
            out.add(tag + "clamp_past")
    if np.any(np.floor(exact) != lo):
        out.add(tag + "round_up")                                    # fl(s*y) rounded up onto an integer
    return out


def branches(recipe, hs, ws):
    name, resz, mean, hf, wf, hc, wc = recipe
    sh, sw, hd, wd, _, _ = geometry(recipe, hs, ws)
    out = _axis_branches(sh, hs, hd, hc, "y") | _axis_branches(sw, ws, wd, wc, "x")
    out.add(("Strict", "Relaxed")[resz] + "/" + ("Full", "Crop")[mean])
    if (hs, ws) == (hf, wf):
        out.add("src_eq_full")
    if max(hs, ws) >= 1500:
        out.add("large")
    if (hc, wc) == (hf, wf):
        out.add("crop_eq_full")
    if hf != wf and hc != wc:
        out.add("non_square")
    return out


def _search(recipe, want, hs_range, ws_of, count=2):
    """First `count` accepted source sizes (hs, ws_of(hs)) whose mirror reaches `want`."""
    found = []
    for hs in hs_range:
        ws = ws_of(hs)
        if accepted(recipe, hs, ws) and want in branches(recipe, hs, ws):
            found.append((hs, ws))
            if len(found) == count:
                break
    return found


def recipe_sizes(recipe):
    name, resz, _, hf, wf, hc, wc = recipe
    sizes = list(BASE_SIZES) + [(hf, wf)]
    # rounding searches: fl(s*y) landing on an integer that the exact product stays below
    sizes += _search(recipe, "yround_up", range(2, 3000), lambda h: h + 61)
    sizes += _search(recipe, "xround_up", range(2, 3000), lambda h: h + 11 if resz else 3 * h + 7)
    if (hc, wc) == (hf, wf):
        # hs - 1 a multiple of full - 1: fl(s * (hd - 1)) is exactly hs - 1 and yh clamps; then a search for a product
        # that rounds past hs - 1
        sizes += [(3 * (hf - 1) + 1, 2 * (wf - 1) + 1), (hf - 1 + 1, 5 * (wf - 1) + 1)]
        sizes += _search(recipe, "yclamp_past", range(2, 3000), lambda h: h if resz else 2 * h + 1, 1)
        sizes += _search(recipe, "xclamp_past", range(2, 3000), lambda h: h if resz else h + 3, 1)
    keep = []
    for hs, ws in sizes:
        if (hs, ws) in keep or not accepted(recipe, hs, ws):
            continue
        _, _, hd, wd, _, _ = geometry(recipe, hs, ws)
        if hd * wd <= MAX_RESIZED:
            keep.append((hs, ws))
    return keep


def preproc_cases():
    """[(recipe, [(hs, ws, seed, gap), ...])]: every recipe with its sources; gaps of 0-7 bytes before the pixels."""
    out = []
    for r, recipe in enumerate(RECIPES):
        imgs = [(hs, ws, 1000 * r + i, (i * 3) % 8) for i, (hs, ws) in enumerate(recipe_sizes(recipe))]
        out.append((recipe, imgs))
    return out


def write_mean(po, d, recipe, seed=5):
    name, _, mean_type, hf, wf, hc, wc = recipe
    h, w = (hf, wf) if mean_type == 0 else (hc, wc)
    mean = (np.random.RandomState(seed).rand(3, h, w) * 120 + 0.37).astype(np.float32)
    if po is None:
        return mean, None
    path = os.path.join(d, "%s_mean.bin" % name)
    po.write_bin(path, mean)
    return mean, path


REQUIRED = {"upscale_y", "upscale_x", "src_eq_full", "large", "yclamp", "xclamp", "yclamp_exact", "xclamp_exact",
            "yround_up", "xround_up", "odd_yoff", "odd_xoff", "even_yoff", "even_xoff", "non_square", "crop_eq_full",
            "Strict/Full", "Strict/Crop", "Relaxed/Crop"}


def test_generated_cases_reach_every_branch():
    seen, per = set(), {}
    for recipe, imgs in preproc_cases():
        for hs, ws, _, _ in imgs:
            b = branches(recipe, hs, ws)
            seen |= b
            per.setdefault(recipe[0], set()).update(b)
    assert REQUIRED <= seen, REQUIRED - seen
    # clamping past hs - 1 (fl(s * (hd - 1)) > hs - 1, both weights ~1) is reached too
    assert {"yclamp_past", "xclamp_past"} <= seen
    for name, (_, resz, _, hf, wf, hc, wc) in RECIPE.items():
        if (hc, wc) == (hf, wf):
            assert {"yclamp", "xclamp"} <= per[name], name
    # row padding 0-3 bytes and a gap before the pixels both occur
    pads = {(4 - ws * 3 % 4) % 4 for _, imgs in preproc_cases() for _, ws, _, _ in imgs}
    gaps = {g for _, imgs in preproc_cases() for _, _, _, g in imgs}
    assert pads == {0, 1, 2, 3} and 0 in gaps and max(gaps) > 0


def test_kepsilon_never_changes_the_relaxed_size():
    """ReszImg adds kEpsilon = 1e-7 to (src - 1) / s before truncating.  s <= (src - 1) / (full - 1) makes the float
    quotient >= 1, and the largest float below any integer n >= 2 is at least 2^-23 > 1e-7 away, so the addition never
    carries the quotient onto the next integer: the branch that would need it is unreachable.  A sweep confirms it."""
    f32 = np.float32
    hs = np.arange(2, 4001)
    for hf, wf in [(2, 2), (3, 7), (40, 40), (227, 227), (256, 256), (256, 320), (224, 288)]:
        for ws in [2, 3, 5, 17, 100, 255, 256, 257, 700, 1000, 2000, 3999]:
            s = np.minimum((hs - 1).astype(f32) / f32(hf - 1), f32(ws - 1) / f32(wf - 1))
            for q in ((hs - 1).astype(f32) / s, f32(ws - 1) / s):
                assert q.min() >= 1
                assert np.array_equal((q.astype(np.float64) + 1e-7).astype(np.int64), q.astype(np.int64))


def test_bmp_writer_round_trips(tmp_path):
    for hs, ws, gap in [(1, 1, 0), (3, 1, 5), (2, 2, 0), (5, 3, 1), (4, 4, 7), (7, 13, 2)]:
        img = make_image(hs, ws, hs * 31 + ws)
        p = str(tmp_path / ("r%d_%d.bmp" % (hs, ws)))
        write_bmp(p, img, gap)
        assert os.path.getsize(p) == 54 + gap + hs * ((ws * 3 + 3) & ~3)
        assert np.array_equal(decode_bmp(p), img)


def host_load_bmp(host, bmp, mean_path, recipe):
    _, resz, mean_type, hf, wf, hc, wc = recipe
    out = np.empty((3, hc, wc), np.float32)
    n = host.qcnn_host_load_bmp(bmp.encode(), mean_path.encode(), resz, mean_type, hf, wf, hc, wc,
                                out.ctypes.data_as(C.c_void_p), out.size)
    assert n == out.size, (bmp, n)
    return out


@needs_ref
def test_reference_host_port_and_numpy_agree_on_generated_bmps(po, tmp_path):
    host = C.CDLL(os.path.join(PKG, "libqcnn_host.so"))
    checked = 0
    for recipe, imgs in preproc_cases():
        name, resz, mean_type, hf, wf, hc, wc = recipe
        mean, mean_path = write_mean(po, str(tmp_path), recipe)
        for hs, ws, seed, gap in imgs:
            img = make_image(hs, ws, seed)
            bmp = str(tmp_path / ("%s_%d_%d.bmp" % (name, hs, ws)))
            write_bmp(bmp, img, gap)
            want = po.ref_bmp_load(bmp, mean_path, resz, mean_type, hf, wf, hc, wc)
            got = host_load_bmp(host, bmp, mean_path, recipe)
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (name, hs, ws)
            npy = resz_crop_numpy(img, mean, (hf, wf), (hc, wc), resz == 1, mean_type == 0)
            assert np.array_equal(npy.view(np.uint32), want.view(np.uint32)), (name, hs, ws)
            checked += 1
    assert checked >= 90


# ------------------------------------------------------------------------------------------------
# top-k rows
# ------------------------------------------------------------------------------------------------
TOPK_C = [1, 2, 31, 32, 33, 255, 256, 257, 1000, 4097, 12000]


def topk_rows(Cc, n_rand=0, seed=0):
    """(names, float32 [N, C]) of probability-like rows with the edge values of a k-fold arg-max."""
    rng = np.random.RandomState(seed + Cc)
    nan, inf = np.float32(np.nan), np.float32(np.inf)
    rows = []

    def base():
        return (rng.rand(Cc) * 0.5).astype(np.float32)

    def add(name, r):
        rows.append((name, r))

    for i in range(3):
        add("rand%d" % i, base())
    r = base(); r[Cc // 2] = 0.9; r[0] = nan; add("nan_at_0", r)
    if Cc > 1:
        r = base(); r[0] = nan; r[Cc - 1] = nan; add("nan_at_0_and_last", r)
    for t in sorted({1, 5, 37, 200, 255} & set(range(1, min(Cc, 256)))):
        # NaN in thread t's first slot, the row maximum later in the same thread's stride when there is one
        r = base(); r[t] = nan; r[t + 256 if t + 256 < Cc else Cc - 1] = 0.9; add("nan_mid_%d" % t, r)
    if Cc > 1:
        r = base(); r[1] = nan; r[0] = 0.95; add("nan_at_1_max_at_0", r)
    if Cc > 300:
        r = base(); r[261] = 0.9; r[5] = nan; add("issue_nan5", r)
        r = base(); r[261] = 0.9; r[0] = nan; add("issue_nan0", r)
        r = base(); r[299] = nan; r[Cc - 1] = 0.9; r[300] = nan; add("nan_past_256", r)
        r = base(); r[rng.rand(Cc) < 0.3] = nan; r[0] = 0.1; add("nan_scattered", r)
    add("all_nan", np.full(Cc, nan, np.float32))
    r = base(); r[Cc - 1] = inf; r[Cc // 3] = inf; add("pos_inf", r)
    r = base(); r[0] = -inf; add("neg_inf_at_0", r)
    add("all_neg_inf", np.full(Cc, -inf, np.float32))
    r = np.where(rng.rand(Cc) < 0.5, np.float32(-0.0), np.float32(0.0)).astype(np.float32); r[0] = -0.0
    add("signed_zeros", r)
    add("all_equal", np.full(Cc, 0.25, np.float32))
    add("all_negative", (-rng.rand(Cc) - 0.01).astype(np.float32))
    r = (rng.rand(Cc) * FLT_MIN).astype(np.float32); add("below_flt_min", r)
    r = (rng.rand(Cc) * FLT_MIN).astype(np.float32); r[Cc // 2] = FLT_MIN; r[-1] = FLT_MIN; add("at_flt_min", r)
    r = (rng.rand(Cc) * FLT_MIN).astype(np.float32); r[Cc - 1] = np.nextafter(FLT_MIN, np.float32(1)); add("above_flt_min", r)
    for i in range(n_rand):
        add("fill%d" % i, base())
    return [n for n, _ in rows], np.stack([r for _, r in rows]).astype(np.float32)


def topk_case(Cc):
    """The rows the device top-k test runs: 300 for C <= 1000, else only the named rows (k = C costs O(C^2))."""
    names, P = topk_rows(Cc, seed=1)
    if Cc <= 1000:
        names, P = topk_rows(Cc, n_rand=300 - len(names), seed=1)
    return names, P


def sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def case_key(recipe, hs, ws):
    return "%s/%dx%d" % (recipe[0], hs, ws)


def reference_goldens(po, d):
    """What the compiled reference computes on every generated input, as tests/golden/preproc_topk_ref.npz stores it:
    per BMP case the sha256 of the input (pixels, mean) and of BmpImgIO::Load's float32 output; per top-k C the sha256
    of the rows and CvtFeatMapToLablVec's labels.  Needs the compiled reference (tests/golden/make_golden.py)."""
    keys, ins, outs, out = [], [], [], {}
    for recipe, imgs in preproc_cases():
        name, resz, mean_type, hf, wf, hc, wc = recipe
        mean, mean_path = write_mean(po, d, recipe)
        for hs, ws, seed, gap in imgs:
            img = make_image(hs, ws, seed)
            bmp = os.path.join(d, "%s_%d_%d.bmp" % (name, hs, ws))
            write_bmp(bmp, img, gap)
            keys.append(case_key(recipe, hs, ws))
            ins.append(sha(img, mean))
            outs.append(sha(po.ref_bmp_load(bmp, mean_path, resz, mean_type, hf, wf, hc, wc)))
    out["bmp_key"], out["bmp_in"], out["bmp_out"] = np.array(keys), np.array(ins), np.array(outs)
    for Cc in TOPK_C:
        _, P = topk_case(Cc)
        out["topk_rows_%d" % Cc] = np.array(sha(P))
        out["topk_labl_%d" % Cc] = po.ref_cvt_featmap_to_labl(P)
    return out


def load_goldens():
    g = np.load(GOLDEN)
    bmp = {k: (i, o) for k, i, o in zip(g["bmp_key"], g["bmp_in"], g["bmp_out"])}
    return bmp, g


def _model_topk(row, k, mode, fixed, threads=256):
    """CPU model of topk_kernel: per-thread scan over c = t, t + 256, ..., two xor-shuffle trees, the FLT_MIN rule."""
    row = row.copy()
    Cc = row.size
    out = []

    def merge(bv, bi):
        for m in (16, 8, 4, 2, 1):
            ov, oi = bv[np.arange(32) ^ m], bi[np.arange(32) ^ m]
            take = (oi < Cc) & ((bi == Cc) | (bv < ov) | ((bv == ov) & (oi < bi)))
            bv, bi = np.where(take, ov, bv), np.where(take, oi, bi)
        return bv[0], bi[0]

    for _ in range(k):
        bv, bi = np.full(threads, -np.inf, np.float32), np.full(threads, Cc)
        for t in range(threads):
            for c in range(t, Cc, threads):
                v = row[c]
                if (v == v or not fixed) and (bi[t] == Cc or bv[t] < v):
                    bv[t], bi[t] = v, c
        wv, wi = zip(*[merge(bv[w * 32:(w + 1) * 32], bi[w * 32:(w + 1) * 32]) for w in range(threads // 32)])
        v, i = merge(np.array(list(wv) + [-np.inf] * 24, np.float32), np.array(list(wi) + [Cc] * 24))
        if fixed and mode == 0 and row[0] != row[0]:
            i = 0
        if mode == 1 and not (FLT_MIN < v):
            i = 0
        i = 0 if i >= Cc else int(i)
        out.append(i)
        row[i] = 0.0
    return out


def test_kernel_model_shows_the_nan_defect_and_its_fix(po):
    """The issue's table: the old per-thread rule (first element taken unconditionally, then strict <) keeps a NaN in a
    thread's first slot and hides that thread's later elements; the fixed rule matches both reference scans."""
    rng = np.random.RandomState(0)
    p = (rng.rand(1000) * 0.5).astype(np.float32)
    p[261] = 0.9
    a = p.copy(); a[5] = np.nan
    b = p.copy(); b[0] = np.nan
    truth = {(5, 0): list(po.topk(a, 3)[0]), (5, 1): list(po.topk_labl(a, 3)),
             (0, 0): list(po.topk(b, 3)[0]), (0, 1): list(po.topk_labl(b, 3))}
    assert truth[(5, 0)][0] == 261 and truth[(5, 1)][0] == 261 and truth[(0, 0)][:2] == [0, 261]
    assert truth[(0, 1)][0] == 261
    for (at, mode), want in truth.items():
        row = a if at == 5 else b
        old = _model_topk(row, 3, mode, fixed=False)
        assert (old == want) == (at == 0 and mode == 0), (at, mode, old, want)
        assert _model_topk(row, 3, mode, fixed=True) == want, (at, mode)
    for Cc in [1, 33, 257, 1000]:
        names, P = topk_rows(Cc)
        for n, row in zip(names, P):
            k = min(5, Cc)
            assert _model_topk(row, k, 0, True) == list(po.topk(row, k)[0]), (Cc, n)
            assert _model_topk(row, k, 1, True) == list(po.topk_labl(row, k)), (Cc, n)


@needs_ref
def test_topk_labl_restatement_equals_the_reference(po):
    for Cc in TOPK_C:
        names, P = topk_rows(Cc, n_rand=4)
        ref = po.ref_cvt_featmap_to_labl(P)
        for n, row in enumerate(P):
            assert np.array_equal(po.topk_labl(row, 5), ref[n].astype(np.int32)), (Cc, names[n])


def test_golden_fixture_covers_every_generated_input():
    """The committed reference outputs belong to exactly the inputs this module generates (no reference needed)."""
    bmp, g = load_goldens()
    keys = set()
    for recipe, imgs in preproc_cases():
        mean = write_mean(None, None, recipe)[0]
        for hs, ws, seed, _ in imgs:
            k = case_key(recipe, hs, ws)
            keys.add(k)
            assert bmp[k][0] == sha(make_image(hs, ws, seed), mean), k
    assert keys == set(bmp)
    for Cc in TOPK_C:
        assert str(g["topk_rows_%d" % Cc]) == sha(topk_case(Cc)[1]), Cc


@needs_ref
def test_golden_fixture_equals_the_compiled_reference(po, tmp_path):
    want = reference_goldens(po, str(tmp_path))
    _, g = load_goldens()
    assert set(want) == set(g.files)
    for k in want:
        assert np.array_equal(want[k], g[k]), k
