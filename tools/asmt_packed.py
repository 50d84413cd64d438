#!/usr/bin/env python
"""Bit-packed FC assignment tables against byte tables on one GPU, in one process: the two forms alternate, round by
round, and every figure is the median over the rounds with the spread (min - max) beside it.

    fc_chain   AlexNet fc6 -> fc7 -> fc8 at batch 1 (one persistent launch), L2 flushed before every launch, CUDA events
    net        the shipped AlexNet, qcnn_net_forward at N = 1 (captured graph), 4, 40 and 256, default and strict path
    bytes      the assignment table of each FC layer, byte table and packed

    python tools/asmt_packed.py [--rounds 7] [--iters 200] [--out results/asmt_packed.json]

Needs the shipped AlexNet staged under oracle/_ref/data (built by __graft_entry__.build() where the reference exists).
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        lim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        lim = "unknown"
    return name, lim


def stats(v):
    v = np.asarray(v, np.float64)
    return dict(median=float(np.median(v)), min=float(v.min()), max=float(v.max()))


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=200, help="launches per fc_chain round")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from oracle import pyoracle as po
    if not po.have_alexnet():
        sys.exit("shipped AlexNet parameters not staged under oracle/_ref/data")
    q = importlib.import_module("quantized-cnn_b200")
    name, lim = card()
    print("card: %s  power.limit, clocks.max.sm: %s" % (name, lim), flush=True)
    ctx = q.Context(0)
    net = q.Net(ctx, po.ALEXNET_DIR, po.ALEXNET_PFX, "AlexNet")
    fcl = [l for l in range(net.layer_count) if net.pq_layer(l) is not None and net.pq_layer(l).describe(1).startswith("fc_aprx")]
    fcs = [net.pq_layer(l) for l in fcl]
    res = dict(card=name, power_limit_and_max_sm_clock=lim, rounds=args.rounds)

    # ---- assignment bytes per FC layer ----
    res["bytes"] = {}
    for l, L in zip(fcl, fcs):
        desc = L.describe(1)
        f = dict(kv.split("=") for kv in desc.split()[1:6])
        Dout, S, K = int(f["Dout"]), int(f["S"]), int(f["K"])
        b = int(np.log2(K))
        res["bytes"]["layer%d" % l] = dict(S=S, Dout=Dout, K=K, byte_table=S * Dout, packed=S * ((Dout * b + 7) // 8), bits=b)
    print("assignment bytes:", json.dumps(res["bytes"]), flush=True)

    # ---- fc_chain, batch 1, L2 flushed ----
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    x = torch.rand((1, 9216), dtype=torch.float32, device="cuda")
    relu = [1, 1, 0]
    chain = {0: [], 1: []}
    outs = {}
    for rnd in range(args.rounds + 1):
        for packed in (0, 1):
            for L in fcs:
                L.set_param("asmt_packed", packed)
            outs[packed] = q.fc_chain_forward(fcs, relu, x).cpu().numpy()
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.iters)]
            for k in range(args.iters):
                flush.fill_(k & 0xFF)
                ev[k][0].record()
                q.fc_chain_forward(fcs, relu, x)
                ev[k][1].record()
            torch.cuda.synchronize()
            if rnd:   # round 0 warms up both forms
                chain[packed].append(float(np.median([a.elapsed_time(b) * 1e3 for a, b in ev])))
    assert np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32)), "packed and byte-table chain outputs differ"
    res["fc_chain_b1_l2flushed_us"] = {"byte": stats(chain[0]), "packed": stats(chain[1])}
    print("fc_chain b1 (L2 flushed, us):", json.dumps(res["fc_chain_b1_l2flushed_us"]), flush=True)
    del flush

    # ---- whole network ----
    imgs = torch.from_numpy(po.lcg_images(256, 77)).cuda()
    res["net_ms"] = {}
    for mode in ("default", "strict"):
        for l in range(net.layer_count):
            pl = net.pq_layer(l)
            if pl is not None:
                pl.set_param("tensor_core", 0 if mode == "strict" else 2)
        for N in (1, 4, 40, 256):
            xin = imgs[:N].contiguous()
            prob = torch.empty((N, net.out_len), dtype=torch.float32, device="cuda")
            reps = max(5, min(200, 2000 // N))
            t = {0: [], 1: []}
            ref = {}
            for rnd in range(args.rounds + 1):
                for packed in (0, 1):
                    net.set_asmt_packed(packed)
                    for _ in range(4):                   # eager passes, graph capture at small N
                        net.forward(xin, prob)
                    ref[packed] = prob.cpu().numpy().copy()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    for _ in range(reps):
                        net.forward(xin, prob)
                    b.record()
                    torch.cuda.synchronize()
                    if rnd:
                        t[packed].append(a.elapsed_time(b) / reps)
            assert np.array_equal(ref[0].view(np.uint32), ref[1].view(np.uint32)), (mode, N)
            key = "%s/N=%d" % (mode, N)
            res["net_ms"][key] = {"byte": stats(t[0]), "packed": stats(t[1]),
                                  "packed_over_byte": float(np.median(t[1]) / np.median(t[0]))}
            print("net %-12s byte %.4f ms  packed %.4f ms  (x%.3f)" % (key, np.median(t[0]), np.median(t[1]),
                                                                       np.median(t[1]) / np.median(t[0])), flush=True)
    net.set_asmt_packed(False)
    net.close()
    ctx.close()
    print("RESULT " + json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
