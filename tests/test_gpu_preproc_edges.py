"""The two ends of the PQ path on the device (csrc/preproc.cu) against the compiled reference, at the sizes and values
where they go wrong.

  * bmp_preproc_kernel (qcnn_preproc_run): every generated case of tests/test_preproc_reference.py -- upscaling,
    clamped last rows / columns, products that round onto an integer, odd offsets, non-square sizes, crop == full, all
    accepted (resize, mean) pairs -- in one launch per recipe with mixed sizes and unaligned byte offsets, bit for bit
    against the compiled reference (BmpImgIO::Load, through the sha256 of its outputs that
    tests/golden/preproc_topk_ref.npz keeps), the C++ host port and the numpy restatement; a launch of 300
    images; back-to-back runs of one object on one stream; the refusals.
  * u8hwc_to_f32chw_kernel: (float)pixel - mean bit for bit at C = 1, 3, 4, with an exact write set.
  * topk_kernel: idx and val bit for bit against the oracle's restatement of CaffeEvaWrapper::Proc (mode 0), idx
    against CaffeEva::CvtFeatMapToLablVec (mode 1: the compiled reference's labels in the same fixture and the oracle's
    restatement), across C
    around the 32-lane and 256-thread strides and NaN / inf / signed-zero / sub-FLT_MIN rows."""
import ctypes as C
import os

import numpy as np
import pytest

from test_gpu_preproc import resz_crop_numpy
from test_preproc_reference import (PKG, RECIPE, RECIPES, TOPK_C, accepted, case_key, geometry, host_load_bmp,
                                    load_goldens, make_image, preproc_cases, sha, topk_case, write_bmp, write_mean)

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _pack(imgs, seed):
    """One uint8 buffer holding the pictures at unaligned offsets (1-13 junk bytes before each)."""
    rng = np.random.RandomState(seed)
    parts, offs, pos = [], [], 0
    for im in imgs:
        gap = int(rng.randint(1, 14))
        parts.append(np.full(gap, 0xEE, np.uint8))
        parts.append(np.ascontiguousarray(im, np.uint8).reshape(-1))
        offs.append(pos + gap)
        pos += gap + im.size
    return np.concatenate(parts), offs


def _run(qcnn, pp, dev_pix, offs, imgs, out, stream=None):
    N = len(imgs)
    rc = qcnn.lib.qcnn_preproc_run(pp.h, C.c_void_p(dev_pix.data_ptr()), (C.c_longlong * N)(*offs),
                                   (C.c_int * N)(*[im.shape[0] for im in imgs]),
                                   (C.c_int * N)(*[im.shape[1] for im in imgs]), N, C.c_void_p(out.data_ptr()),
                                   qcnn._stream(stream))
    return rc


def _preproc(qcnn, ctx, recipe, mean):
    _, resz, mean_type, hf, wf, hc, wc = recipe
    return qcnn.Preproc(ctx, mean, hf, wf, hc, wc, resz_type=resz, mean_type=mean_type)


@pytest.mark.parametrize("name", [r[0] for r in RECIPES])
def test_preproc_equals_the_reference_on_generated_bmps(po, qcnn, ctx, tmp_path, name):
    import torch
    recipe, imgs_spec = [c for c in preproc_cases() if c[0][0] == name][0]
    _, resz, mean_type, hf, wf, hc, wc = recipe
    host = C.CDLL(os.path.join(PKG, "libqcnn_host.so"))
    golden, _ = load_goldens()
    mean, mean_path = write_mean(po, str(tmp_path), recipe)
    imgs = [make_image(hs, ws, seed) for hs, ws, seed, _ in imgs_spec]
    flat, offs = _pack(imgs, 7)
    pp = _preproc(qcnn, ctx, recipe, mean)
    out = torch.empty((len(imgs), 3, hc, wc), dtype=torch.float32, device="cuda")
    assert _run(qcnn, pp, torch.from_numpy(flat).cuda(), offs, imgs, out) == 0
    got = out.cpu().numpy()
    pp.close()
    for i, ((hs, ws, _, gap), im) in enumerate(zip(imgs_spec, imgs)):
        bmp = str(tmp_path / ("%d.bmp" % i))
        write_bmp(bmp, im, gap)
        tag = (name, hs, ws)
        # the compiled reference's output, by its sha256 (tests/golden/preproc_topk_ref.npz)
        ref_in, ref_out = golden[case_key(recipe, hs, ws)]
        assert ref_in == sha(im, mean) and sha(got[i]) == ref_out, tag
        assert np.array_equal(_bits(got[i]), _bits(host_load_bmp(host, bmp, mean_path, recipe))), tag
        assert np.array_equal(_bits(got[i]), _bits(resz_crop_numpy(im, mean, (hf, wf), (hc, wc), resz == 1,
                                                                   mean_type == 0))), tag


def _random_sizes(recipe, n, seed, lo=2, hi=600):
    rng = np.random.RandomState(seed)
    out = []
    while len(out) < n:
        hs, ws = int(rng.randint(lo, hi)), int(rng.randint(lo, hi))
        if accepted(recipe, hs, ws) and np.prod(geometry(recipe, hs, ws)[2:4]) <= (1 << 21):
            out.append((hs, ws))
    return out


def test_preproc_launch_of_300_images(qcnn, ctx):
    import torch
    recipe = RECIPE["rect_relaxed"]
    _, resz, mean_type, hf, wf, hc, wc = recipe
    mean = (np.random.RandomState(3).rand(3, hc, wc) * 120).astype(np.float32)
    sizes = _random_sizes(recipe, 300, 11)
    imgs = [make_image(hs, ws, 50 + i) for i, (hs, ws) in enumerate(sizes)]
    flat, offs = _pack(imgs, 8)
    pp = _preproc(qcnn, ctx, recipe, mean)
    out = torch.empty((300, 3, hc, wc), dtype=torch.float32, device="cuda")
    assert _run(qcnn, pp, torch.from_numpy(flat).cuda(), offs, imgs, out) == 0
    got = out.cpu().numpy()
    pp.close()
    for i, im in enumerate(imgs):
        want = resz_crop_numpy(im, mean, (hf, wf), (hc, wc), True, False)
        assert np.array_equal(_bits(got[i]), _bits(want)), (i, im.shape)


def test_back_to_back_runs_of_one_object_keep_stream_order(qcnn, ctx):
    """Three runs on one side stream with no host sync between them: the second needs a larger descriptor buffer, the
    third reuses it while the second's kernel may still be reading it.  Each run must see its own descriptors."""
    import torch
    recipe = RECIPE["alexnet"]
    _, resz, mean_type, hf, wf, hc, wc = recipe
    mean = (np.random.RandomState(4).rand(3, hf, wf) * 120).astype(np.float32)
    sets = [[make_image(hs, ws, 900 + 100 * k + i) for i, (hs, ws) in enumerate(_random_sizes(recipe, n, 20 + k))]
            for k, n in enumerate([3, 40, 7])]
    packs = [_pack(imgs, 30 + k) for k, imgs in enumerate(sets)]
    devs = [torch.from_numpy(f).cuda() for f, _ in packs]
    outs = [torch.full((len(imgs), 3, hc, wc), float("nan"), device="cuda") for imgs in sets]
    pp = _preproc(qcnn, ctx, recipe, mean)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    for dev, (_, offs), imgs, out in zip(devs, packs, sets, outs):
        assert _run(qcnn, pp, dev, offs, imgs, out, stream=side.cuda_stream) == 0
    side.synchronize()
    for imgs, out in zip(sets, outs):
        got = out.cpu().numpy()
        for i, im in enumerate(imgs):
            want = resz_crop_numpy(im, mean, (hf, wf), (hc, wc), False, True)
            assert np.array_equal(_bits(got[i]), _bits(want)), (len(imgs), i, im.shape)
    pp.close()


def test_preproc_refusals(qcnn, ctx):
    import torch
    mean = np.zeros((3, 40, 40), np.float32)
    with pytest.raises(qcnn.QcnnError):
        qcnn.Preproc(ctx, np.zeros((3, 256, 256), np.float32), 256, 256, 224, 224, resz_type=1, mean_type=0)
    with pytest.raises(qcnn.QcnnError):
        qcnn.Preproc(ctx, mean, 40, 40, 40, 40, resz_type=1, mean_type=0)
    pp = _preproc(qcnn, ctx, RECIPE["whole_relaxed"], mean)
    # Relaxed: fl((hs - 1) / fl((hs - 1) / 39)) can fall just below 39, which resizes to 39 rows, one short of the crop
    short = [(hs, hs + 50) for hs in range(2, 400) if not accepted(RECIPE["whole_relaxed"], hs, hs + 50)]
    assert short and geometry(RECIPE["whole_relaxed"], *short[0])[2] == 39
    ok = make_image(50, 60, 1)
    out = torch.empty((2, 3, 40, 40), dtype=torch.float32, device="cuda")
    for bad in [make_image(1, 5, 2), make_image(5, 1, 3), make_image(1, 1, 4), make_image(*short[0], seed=5)]:
        flat, offs = _pack([ok, bad], 1)
        assert _run(qcnn, pp, torch.from_numpy(flat).cuda(), offs, [ok, bad], out) != 0, bad.shape
    pix = torch.zeros(16, dtype=torch.uint8, device="cuda")
    z = (C.c_longlong * 1)(0)
    one = (C.c_int * 1)(2)
    for N in (0, 65536, -1):
        assert qcnn.lib.qcnn_preproc_run(pp.h, C.c_void_p(pix.data_ptr()), z, one, one, N, C.c_void_p(out.data_ptr()),
                                         qcnn._stream(None)) != 0, N
    torch.cuda.synchronize()
    pp.close()


@pytest.mark.parametrize("Cc", [1, 3, 4])
def test_u8hwc_to_f32chw_is_exact(qcnn, ctx, Cc):
    import torch
    G = 67                                                       # NaN guard either side of dst
    for H, W in [(1, 1), (7, 13), (227, 227)]:
        for N in (1, 5, 300):
            rng = np.random.RandomState(H * 1000 + W * 10 + N + Cc)
            pix = rng.randint(0, 256, size=(N, H, W, Cc)).astype(np.uint8)
            mean = (rng.rand(Cc, H, W) * 255 - 60).astype(np.float32)
            src = torch.from_numpy(pix).cuda()
            dm = torch.from_numpy(mean).cuda()
            for with_mean in (False, True):
                n = N * Cc * H * W
                buf = torch.full((n + 2 * G,), float("nan"), device="cuda")
                rc = qcnn.lib.qcnn_u8hwc_to_f32chw(ctx.h, C.c_void_p(src.data_ptr()),
                                                  C.c_void_p(dm.data_ptr() if with_mean else 0),
                                                  C.c_void_p(buf.data_ptr() + 4 * G), N, Cc, H, W, qcnn._stream(None))
                assert rc == 0
                got = buf.cpu().numpy()
                want = np.transpose(pix, (0, 3, 1, 2)).astype(np.float32)
                if with_mean:
                    want = want - mean[None]
                tag = (Cc, H, W, N, with_mean)
                assert np.array_equal(_bits(got[G:G + n]), _bits(want.reshape(-1))), tag
                assert np.isnan(got[:G]).all() and np.isnan(got[G + n:]).all(), tag


@pytest.mark.parametrize("Cc", TOPK_C)
def test_topk_matches_both_reference_scans(po, qcnn, ctx, Cc):
    import torch
    names, P = topk_case(Cc)
    _, g = load_goldens()
    assert sha(P) == str(g["topk_rows_%d" % Cc])
    ref = g["topk_labl_%d" % Cc].astype(np.int32)             # the compiled CvtFeatMapToLablVec on these rows
    dev = torch.from_numpy(P).cuda()
    bad = []
    for k in sorted({1, 5, Cc} & set(range(1, Cc + 1))):
        idx, val = ctx.topk(dev, k, mode=0)
        idx, val = idx.cpu().numpy(), val.cpu().numpy()
        for n in range(P.shape[0]):
            ri, rv = po.topk(P[n], k)
            if not (np.array_equal(idx[n], ri) and np.array_equal(_bits(val[n]), _bits(rv))):
                bad.append(("mode0", k, names[n]))
        if k > 5:
            continue
        idx1, _ = ctx.topk(dev, k, mode=1)
        idx1 = idx1.cpu().numpy()
        for n in range(P.shape[0]):
            ok = np.array_equal(idx1[n], po.topk_labl(P[n], k)) and np.array_equal(idx1[n], ref[n, :k])
            if not ok:
                bad.append(("mode1", k, names[n]))
    assert not bad, "C=%d: %s" % (Cc, sorted(set(bad)))


def test_topk_refusals(qcnn, ctx):
    import torch
    p = torch.rand((3, 100), device="cuda")
    for k in (0, 101):
        with pytest.raises(qcnn.QcnnError):
            ctx.topk(p, k)
    with pytest.raises(qcnn.QcnnError):
        ctx.topk(torch.rand((2, 12001), device="cuda"), 1)
    idx, _ = ctx.topk(torch.rand((2, 12000), device="cuda"), 1)
    torch.cuda.synchronize()
    assert idx.shape == (2, 1)
