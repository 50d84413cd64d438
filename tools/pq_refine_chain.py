"""The paper's multi-layer error correction on the shipped AlexNet, as a caller loop over the per-layer primitives.

The shipped parameters, decoded, are the "original" network.  In layer order (conv1 ... fc8) every PQ layer is
re-quantized coarser than shipped (conv K = 32, d = 8; fc6 / fc7 K = 16, d = 8; fc8 K = 16, d = 4) in three ways.
conv1 has 3 input channels, so any d >= 3 gives it one 3-dim subspace; its codebook is stored d = 4 wide by default
(the same quantization as d = 3; DESIGN.md 4e says why):
  kmeans      pq_quantize_* only (iters = 20);
  same-input  that start refined with pq_refine_* on the layer's inputs in the quantized network;
  target      that start refined with pq_refine_*_target: the same inputs toward the original network's pre-bias
              responses of the layer (t = W x on the original network's inputs x).
The inputs of layer l come from a net in which every layer before l is already replaced by that mode's result
(po.save_model into a temporary directory, Net.featmap under keep_maps).  Calibration and held-out images are seeded
LCG images (po.lcg_images).  Reports per layer and mode the training loss ratio and the call time, per mode the held-out
relative error of the final logits against the original network's (over all images, and the median of the per-image
errors) and the top-1 / top-5 agreement with its
predictions (top-5: the original's top-1 class is among the mode's five best), and the card, its power limit and max SM
clock, all from the same run.
With --stats the calibration images stream through in batches of --batch: per layer and mode, each batch's inputs y
(and for the target mode the original network's responses t) are added to a PqStats object and dropped, and the
refinement runs on the accumulated statistics (qcnn_pq_stats_refine / _refine_target), so no layer's inputs or targets
are ever held whole and device memory does not grow with --train.  Each call time is then the accumulation plus the
refinement, printed with the peak device memory of that layer and mode (torch's peak allocation plus the statistics;
the buffers the library allocates for the refine call itself are not included).
With --stats --bias two more modes run, same-input+bias and target+bias: the same refinements with the bias refit as
well (qcnn_pq_stats_refine_bias / _refine_target_bias on the centered statistics).  Each saves its refit bias into its
own model, so the next layer's inputs come from the corrected network; their training loss ratios are of the
bias-optimal losses.
With --stats --damp R [R ...] each value adds the mode target+damp=R (and with --bias also target+bias+damp=R): the
target refinement damped toward the original weights (qcnn_pq_stats_refine_damped, lambda_g = R tr(G_g) / Dg); their
training loss ratios are of the damped losses.
--modes M [M ...] runs only those of the modes above (each mode's chain depends on no other mode), so that a large
--train can be split over several runs.
    python tools/pq_refine_chain.py [--train 4096] [--held 1024] [--sweeps 4] [--conv 32 8] [--fc8 16 4] [--stats]
                                    [--bias] [--damp R [R ...]] [--modes M [M ...]] [--out f.json]"""
import argparse
import importlib
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from pq_refine_time import card   # noqa: E402

NAMES = {0: "conv1", 4: "conv2", 8: "conv3", 10: "conv4", 12: "conv5", 15: "fc6", 18: "fc7", 21: "fc8"}
MODES = ("kmeans", "same-input", "target")
BIAS_MODES = ("same-input+bias", "target+bias")


def decode(ctrd, asmt, cin):
    """dense weights of a PQ layer: conv [Cout][Cg][k][k] from asmt [Cout][k][k][S], FC [Dout][Din] from asmt [Dout][S]"""
    S = ctrd.shape[0]
    g = ctrd[np.arange(S), asmt]
    g = g.reshape(g.shape[:-2] + (-1,))[..., :cin]
    return np.ascontiguousarray(np.moveaxis(g, -1, 1) if g.ndim == 4 else g, np.float32)


def layer_inputs(net, l, imgs, batch, first_fc):
    """featMapLst[l] on every image: NHWC for a conv layer, [N][Din] in fcntWei column order for an FC layer (the first
    FC layer's NHWC map permuted to the NCHW flattening its weights use)"""
    import torch
    net.set_keep_maps(True)
    out = []
    for i in range(0, imgs.shape[0], batch):
        xb = imgs[i:i + batch]
        net.forward(xb)
        m = net.featmap(l, xb.shape[0])
        if l == first_fc:
            m = m.permute(0, 3, 1, 2)
        out.append(m.reshape(m.shape[0], -1).contiguous() if l >= first_fc else m)
    return torch.cat(out)


def response(L, x, W, batch):
    """the original layer's pre-bias response, fp64 arithmetic rounded to fp32 (NHWC for conv)"""
    import torch
    import torch.nn.functional as F
    Wt = torch.from_numpy(W).cuda().double()
    out = []
    for i in range(0, x.shape[0], batch):
        xb = x[i:i + batch].double()
        if W.ndim == 4:
            y = F.conv2d(xb.permute(0, 3, 1, 2), Wt, stride=L["stride"], padding=L["pad"], groups=L["grp"])
            out.append(y.permute(0, 2, 3, 1).float().contiguous())
        else:
            out.append((xb @ Wt.T).float())
    return torch.cat(out)


def logits(net, imgs, batch):
    import torch
    out = []
    for i in range(0, imgs.shape[0], batch):
        xb = imgs[i:i + batch]
        lg = torch.empty((xb.shape[0], net.out_len), dtype=torch.float32, device="cuda")
        net.forward(xb, logits=lg)
        out.append(lg)
    return torch.cat(out)


class LcgImages(object):
    """po.lcg_images on the device, bit for bit: image i's values are s_j = a^j seed + c (a^j - 1) / (a - 1) mod 2^32
    (a = 1664525, c = 1013904223, j = 1 .. 3 x 227 x 227), so a batch of images is one elementwise pass from two
    precomputed per-value tables instead of a sequential host loop per image."""

    def __init__(self, chw):
        import torch
        n = int(np.prod(chw))
        A, Cc = np.empty(n, np.int64), np.empty(n, np.int64)
        a, c = 1, 0
        for j in range(n):
            a, c = (a * 1664525) & 0xFFFFFFFF, (c * 1664525 + 1013904223) & 0xFFFFFFFF
            A[j], Cc[j] = a, c
        self.A, self.C, self.chw = torch.from_numpy(A).cuda(), torch.from_numpy(Cc).cuda(), tuple(chw)

    def __call__(self, count, seed0, chunk=16):
        import torch
        out = torch.empty((count,) + self.chw, dtype=torch.float32, device="cuda")
        flat = out.view(count, -1)
        for i in range(0, count, chunk):
            seeds = (torch.arange(i, min(count, i + chunk), device="cuda", dtype=torch.int64) + seed0) & 0xFFFFFFFF
            lo, hi = (seeds & 0xFFFF)[:, None], (seeds >> 16)[:, None]
            s = (self.A * lo + (((self.A * hi) & 0xFFFF) << 16) + self.C) & 0xFFFFFFFF
            flat[i:i + seeds.shape[0]] = ((s >> 8) & 0xFFFF).float() / 65536.0 * 256.0 - 128.0
        return out


def refine_streamed(q, po, ctx, args, orig, net, l, L, W, c0, a0, first_fc, target, bias=None, damp=None):
    """Accumulate layer l's statistics over the calibration images batch by batch (inputs from `net`, targets from the
    original network), then refine on them: (ctrd, asmt, bias, loss, seconds in the adds and the refine, peak device
    bytes).  bias: the layer's bias, refit with the codebook and assignments (else returned as None).  damp: the
    refinement damped toward W with this weight."""
    import torch
    conv = W.ndim == 4
    d = c0.shape[2]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    st, secs = None, 0.0
    for i in range(0, args.train, args.batch):
        b = min(args.batch, args.train - i)
        imgs = args.lcg(b, args.seed + i)
        y = layer_inputs(net, l, imgs, b, first_fc)
        t = response(L, layer_inputs(orig, l, imgs, b, first_fc), W, b) if target else None
        if st is None:
            if conv:
                _, Hin, Win, Cin = y.shape
                st = q.PqStats.conv(ctx, Cin, Hin, Win, W.shape[0], L["k"], d, pad=L["pad"], stride=L["stride"],
                                    grp=L["grp"], target=target)
            else:
                st = q.PqStats.fc(ctx, y.shape[1], W.shape[0], d, target=target)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        st.add(y, t)
        torch.cuda.synchronize()   # y and t may be freed once the add has run
        secs += time.perf_counter() - t0
        del imgs, y, t
    t0 = time.perf_counter()
    b = None
    if damp is not None:
        r = st.refine_damped(W, c0, a0, damp, target=target, bias=bias, sweeps=args.sweeps)
        c, a, loss = r[0], r[1], r[-1]
        b = r[2] if bias is not None else None
    elif bias is not None and target:
        c, a, b, loss = st.refine_target_bias(c0, a0, bias, sweeps=args.sweeps)
    elif bias is not None:
        c, a, b, loss = st.refine_bias(W, c0, a0, bias, sweeps=args.sweeps)
    elif target:
        c, a, loss = st.refine_target(c0, a0, sweeps=args.sweeps)
    else:
        c, a, loss = st.refine(W, c0, a0, sweeps=args.sweeps)
    secs += time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated() + st.nbytes
    st.close()
    return c, a, b, loss, secs, peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--train", type=int, default=4096, help="calibration images")
    ap.add_argument("--held", type=int, default=1024, help="held-out images")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--sweeps", type=int, default=4)
    ap.add_argument("--conv", type=int, nargs=2, default=(32, 8), metavar=("K", "d"))
    ap.add_argument("--conv1-d", type=int, default=4)
    ap.add_argument("--fc", type=int, nargs=2, default=(16, 8), metavar=("K", "d"), help="fc6 and fc7")
    ap.add_argument("--fc8", type=int, nargs=2, default=(16, 4), metavar=("K", "d"))
    ap.add_argument("--seed", type=int, default=1000000, help="image seed: calibration, then held-out")
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    ap.add_argument("--stats", action="store_true", help="stream the calibration images through PqStats objects")
    ap.add_argument("--bias", action="store_true", help="with --stats: also the modes that refit each layer's bias")
    ap.add_argument("--damp", nargs="+", default=[], metavar="R",
                    help="with --stats: also target+damp=R (and with --bias target+bias+damp=R) for each R")
    ap.add_argument("--modes", nargs="+", default=None, metavar="M", help="run only these modes")
    args = ap.parse_args()
    if args.bias and not args.stats:
        ap.error("--bias needs --stats (the bias refit runs on calibration statistics)")
    if args.damp and not args.stats:
        ap.error("--damp needs --stats (the damped refinement runs on calibration statistics)")
    damp_of = {}   # mode: its damping weight
    for r in args.damp:
        damp_of["target+damp=" + r] = float(r)
        if args.bias:
            damp_of["target+bias+damp=" + r] = float(r)
    modes = MODES + (BIAS_MODES if args.bias else ()) + tuple(damp_of)
    if args.modes:
        unknown = sorted(set(args.modes) - set(modes))
        if unknown:
            ap.error("--modes: %s not among %s" % (", ".join(unknown), ", ".join(modes)))
        modes = tuple(m for m in modes if m in args.modes)
    width = max([15] + [len(m) for m in modes])
    import torch
    from oracle import pyoracle as po
    assert torch.cuda.is_available(), "needs a GPU"
    assert po.have_alexnet(), "needs the shipped AlexNet parameters under oracle/_ref/data"
    q = importlib.import_module("quantized-cnn_b200")
    ctx = q.Context(0)
    cfg = {l: tuple(args.conv) for l in (0, 4, 8, 10, 12)}
    cfg[0] = (args.conv[0], args.conv1_d)
    cfg.update({15: tuple(args.fc), 18: tuple(args.fc), 21: tuple(args.fc8)})
    layers = po.alexnet_layers()
    shapes = po.infer_shapes(layers, po.ALEXNET_IN)
    first_fc = min(l for l in NAMES if layers[l]["type"] == po.FCNT)
    params = po.load_model(po.ALEXNET_DIR, po.ALEXNET_PFX, layers)
    cin = {l: shapes[l][2] // layers[l]["grp"] if layers[l]["type"] == po.CONV else int(np.prod(shapes[l])) for l in NAMES}
    dense = {l: decode(params[l]["ctrd"], params[l]["asmt"], cin[l]) for l in NAMES}
    train = None if args.stats else torch.from_numpy(po.lcg_images(args.train, args.seed)).cuda()
    args.lcg = LcgImages(po.ALEXNET_IN) if args.stats else None
    held = torch.from_numpy(po.lcg_images(args.held, args.seed + args.train)).cuda()
    hw = card()
    print("card: %s (name, power limit, max SM clock)" % hw)
    orig = q.Net(ctx, po.ALEXNET_DIR, po.ALEXNET_PFX, "AlexNet")
    ref = logits(orig, held, args.batch).double()
    qparams = {m: dict(params) for m in modes}
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        def net_of(mode):
            path = os.path.join(tmp, mode)
            po.save_model(path, po.ALEXNET_PFX, qparams[mode])
            return q.Net(ctx, path, po.ALEXNET_PFX, "AlexNet")

        for l in sorted(NAMES):
            L, W, (K, d) = layers[l], dense[l], cfg[l]
            conv = L["type"] == po.CONV
            quant = q.pq_quantize_conv if conv else q.pq_quantize_fc
            c0, a0, _ = quant(ctx, W, K, d, iters=20, seed=1)
            t = None if args.stats else response(L, layer_inputs(orig, l, train, args.batch, first_fc), W, args.batch)
            for mode in modes:
                c, a, b, ratio, secs, peak = c0, a0, None, None, None, None
                if mode != "kmeans" and args.stats:
                    net = net_of(mode)
                    c, a, b, loss, secs, peak = refine_streamed(q, po, ctx, args, orig, net, l, L, W, c0, a0, first_fc,
                                                                mode.startswith("target"),
                                                                params[l]["bias"] if "+bias" in mode else None,
                                                                damp_of.get(mode))
                    net.close()
                    ratio = float(loss[-1] / loss[0])
                elif mode != "kmeans":
                    net = net_of(mode)
                    y = layer_inputs(net, l, train, args.batch, first_fc)
                    net.close()
                    geo = dict(pad=L["pad"], stride=L["stride"], grp=L["grp"]) if conv else {}
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    if mode == "same-input":
                        fn = q.pq_refine_conv if conv else q.pq_refine_fc
                        c, a, loss = fn(ctx, W, y, c0, a0, sweeps=args.sweeps, **geo)
                    elif conv:
                        c, a, loss = q.pq_refine_conv_target(ctx, y, t, c0, a0, L["k"], sweeps=args.sweeps, **geo)
                    else:
                        c, a, loss = q.pq_refine_fc_target(ctx, y, t, c0, a0, sweeps=args.sweeps)
                    secs = time.perf_counter() - t0
                    ratio = float(loss[-1] / loss[0])
                    del y
                qparams[mode][l] = dict(bias=params[l]["bias"] if b is None else b, ctrd=c, asmt=a, bits=po.bits_for(K))
                rows.append(dict(layer=NAMES[l], K=K, d=d, mode=mode, loss_ratio=ratio, call_s=secs, peak_bytes=peak))
                if ratio is not None:
                    print("%-6s K=%-3d d=%-2d %-*s training loss x%.4f  call %.2f s%s"
                          % (NAMES[l], K, d, width, mode, ratio, secs,
                             "" if peak is None else "  peak %.2f GB" % (peak / 1e9)))
            del t
            torch.cuda.empty_cache()
        orig.close()
        top1 = ref.argmax(1)
        summary = []
        for mode in modes:
            net = net_of(mode)
            lg = logits(net, held, args.batch).double()
            net.close()
            err = ((lg - ref).norm() / ref.norm()).item()
            med = ((lg - ref).norm(dim=1) / ref.norm(dim=1)).median().item()
            agree1 = (lg.argmax(1) == top1).double().mean().item()
            agree5 = (lg.topk(5, 1).indices == top1[:, None]).any(1).double().mean().item()
            summary.append(dict(mode=mode, logit_rel_err=err, logit_rel_err_median=med, top1_agree=agree1,
                                top5_agree=agree5))
            print("%-*s held-out logits relative error %.4f (per image, median %.4f)  top-1 agreement %.4f  "
                  "top-5 agreement %.4f" % (width, mode, err, med, agree1, agree5))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(card=hw, train=args.train, held=args.held, sweeps=args.sweeps, stats=args.stats, layers=rows,
                           modes=summary), f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
