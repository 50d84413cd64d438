"""The network executor (qcnn_net.cu: BuildNet, ForwardEager, the graph cache of qcnn_net_forward) on generated layer
tables, beyond the four fixed model tables.

Every kernel the executor launches is pinned to a float64 reference in its own test file.  What is checked here is how
the executor composes them: where ReLU is fused, where LRN + pool become one pass, where dropout aliases the previous
map, which FC runs go to the persistent chain kernel at batch <= 4, how the input layout is folded into the first layer,
what `logits` and `prob` receive, and when a captured CUDA graph is replayed.

* `plan_forward` restates ForwardEager's grouping on the CPU; a CPU test shows that the tables reach every branch.
* Against the oracle (keep_maps = 1): every feature map within the mode's tolerance of `po.net_forward`.
* Composition (keep_maps = 1): map[l+1] is bit for bit the net's own layer l applied to map[l] (same handle, same N:
  same tuned plan), so any difference is a wrong pointer, shape, stride, ReLU flag or source layout.
* Fused path (keep_maps = 0): the maps that survive and the maps that alias another are the mirror's, and every
  surviving map is bit for bit the fused op applied to the map it was computed from.
* Graph cache: replays equal the eager pass, and a layer setting, a regrown map, a repacked table or an evicted entry
  never replays a stale graph.
* qcnn_net_create_from_para builds the same net as qcnn_net_create_custom.
* CPU only: the oracle's feature maps equal the compiled reference's on every table, bit for bit.
"""
import ctypes as C

import numpy as np
import pytest

from test_gpu_layers import close
from test_gpu_net import MODES, set_mode

CONV, POOL, FCNT, RELU, LORN, DRPT, SMAX = range(7)

NS = (1, 3, 4, 5, 8, 9, 40, 130)   # <= 4: chain; <= 8: graph (side stream); 5..95: FC gather; >= 96: fc_ws
CHAIN_MAX_N = 4
FC_TN_PIN = 1


def _tables():
    """name -> (layers, in_chw, {layer: (S, K, d)}, {layer: codebook scale}, pinned FC layer or None).

    Cout/grp is 16 or 32 and every Dout a multiple of 8 (the reference's gathers are unrolled x8); conv K is a multiple
    of 8 and FC K a power of two.  The PQ layer before a softmax has its codebook scaled down as in synth_alexnet."""
    from oracle import pyoracle as po
    T = {}
    # ReLU first, then a stride-1 conv (nchw_to_nhwc), fused LRN + pool (beta 0.75), a grouped conv without ReLU,
    # dropout after a conv and after FC + ReLU, a chain of 3 ending in the softmax
    T["relu_first"] = ([po.relu(), po.conv(1, 3, 16, 1, 1), po.relu(), po.lorn(5, 1e-4, 0.75, 1.0), po.pool(0, 3, 2),
                        po.conv(1, 3, 32, 2, 1), po.drpt(0.5), po.fcnt(32), po.relu(), po.drpt(0.5), po.fcnt(32),
                        po.relu(), po.fcnt(16), po.smax()],
                       (8, 16, 16), {1: (2, 32, 4), 5: (2, 32, 4), 7: (512, 32, 4), 10: (8, 32, 4), 12: (8, 32, 4)},
                       {12: 0.25}, None)
    # CaffeNet order (pool, then a standalone LRN at beta 0.6) before the first FC, FC -> FC, a net ending in dropout
    T["pool_lrn"] = ([po.conv(1, 3, 16, 1, 1), po.relu(), po.pool(0, 2, 2), po.lorn(3, 2e-4, 0.6, 2.0), po.fcnt(32),
                      po.fcnt(24), po.relu(), po.drpt(0.5)],
                     (8, 16, 16), {0: (2, 32, 4), 4: (256, 32, 4), 5: (8, 32, 4)}, {}, None)
    # strided first conv on 3 channels (NCHW fold), fused LRN + pool at beta 0.6, a grouped conv as the last layer
    T["strided3"] = ([po.conv(0, 5, 16, 1, 2), po.relu(), po.lorn(5, 2e-4, 0.6, 1.5), po.pool(0, 3, 2),
                      po.conv(1, 3, 32, 2, 1)],
                     (3, 31, 31), {0: (1, 32, 4), 4: (2, 32, 4)}, {}, None)
    # strided first conv on 8 channels (NCHW fold through a LUT + gather kernel), ReLU after dropout and after pool,
    # a standalone LRN as the last layer
    T["strided8"] = ([po.conv(1, 3, 16, 1, 2), po.drpt(0.5), po.relu(), po.pool(0, 2, 2), po.relu(),
                      po.lorn(5, 1e-4, 0.75, 1.0)],
                     (8, 16, 16), {0: (2, 32, 4)}, {}, None)
    # an FC reading the image; five FC layers with ReLU: a chain of 4, then the fifth on its own
    T["fc_first"] = ([po.fcnt(64), po.relu(), po.fcnt(32), po.relu(), po.fcnt(32), po.relu(), po.fcnt(32), po.relu(),
                      po.fcnt(16), po.smax()],
                     (8, 4, 4), {0: (32, 32, 4), 2: (16, 32, 4), 4: (8, 32, 4), 6: (8, 32, 4), 8: (8, 32, 4)},
                     {8: 0.25}, None)
    # pool first; a chain of 4 with 2, 1 and 0 dropouts between its layers, ReLU on one of them; dropout last
    T["drpt_chain"] = ([po.pool(0, 2, 2), po.fcnt(64), po.drpt(0.5), po.drpt(0.5), po.fcnt(32), po.relu(), po.drpt(0.5),
                        po.fcnt(32), po.fcnt(16), po.drpt(0.5)],
                       (8, 16, 16), {1: (128, 32, 4), 4: (16, 32, 4), 7: (8, 32, 4), 8: (8, 32, 4)}, {}, None)
    # dropout first, a stride-1 conv that is not first, FC -> softmax -> FC, no final softmax
    T["smax_mid"] = ([po.drpt(0.5), po.conv(1, 3, 16, 1, 1), po.relu(), po.pool(0, 2, 2), po.fcnt(32), po.relu(),
                      po.drpt(0.5), po.fcnt(16), po.smax(), po.fcnt(8)],
                     (8, 16, 16), {1: (2, 32, 4), 4: (256, 32, 4), 7: (8, 32, 4), 9: (4, 32, 4)}, {7: 0.25}, None)
    # a softmax over a spatial map read by the first FC (the reference permutes its input to NCHW all the same)
    T["conv_smax_fc"] = ([po.conv(1, 3, 16, 1, 1), po.smax(), po.fcnt(16), po.smax()],
                         (3, 8, 8), {0: (1, 32, 4), 2: (256, 32, 4)}, {0: 0.25, 2: 64.0}, None)
    # fc_tn pinned on the middle FC: no run through it is chain-eligible, the last FC runs as a chain of one
    T["pinned"] = ([po.conv(1, 3, 16, 1, 1), po.relu(), po.fcnt(32), po.relu(), po.fcnt(32), po.relu(), po.fcnt(16),
                    po.smax()],
                   (8, 8, 8), {0: (2, 32, 4), 2: (256, 32, 4), 4: (8, 32, 4), 6: (8, 32, 4)}, {6: 0.25}, 4)
    return T


TABLES = _tables()


def chain_ok(name):
    """Which FC runs the GPU takes as one chain launch at N <= 4 (a per-table fact, not derived from PlanChain): all of
    them, except any run through a layer with a gather-kernel pin."""
    pin = TABLES[name][4]
    return lambda run: pin is None or pin not in run


# ------------------------------------------------------------------------------------------------
# CPU mirror of ForwardEager's grouping
# ------------------------------------------------------------------------------------------------
def plan_forward(table, N, keep, chain_ok):
    """ForwardEager's layer loop restated: a list of steps dict(op, src, dst, relu, layers).

    op is conv, fc, chain, relu, lrn, lrn_maxpool, pool, drpt-alias, drpt-copy or softmax; src / dst are featMapLst
    indices; relu is the flag of the fused kernel (a list for a chain); layers are the PQ layers a step runs."""
    L = len(table)
    ty = [t["type"] for t in table]
    steps = []
    l = 0
    while l < L:
        t = ty[l]
        if t in (CONV, FCNT):
            if t == FCNT and not keep and N <= CHAIN_MAX_N:
                run, relus, j, out = [], [], l, l
                while j < L and ty[j] == FCNT and len(run) < 4:
                    run.append(j)
                    j += 1
                    r = 0
                    if j < L and ty[j] == RELU:
                        r = 1
                        j += 1
                    relus.append(r)
                    out = j
                    k = j
                    while k < L and ty[k] == DRPT:
                        k += 1
                    if k < L and ty[k] == FCNT:
                        j = k
                    else:
                        break
                if chain_ok(tuple(run)):
                    steps.append(dict(op="chain", src=l, dst=out, relu=relus, layers=run))
                    l = out
                    continue
            fuse = not keep and l + 1 < L and ty[l + 1] == RELU
            out = l + 2 if fuse else l + 1
            steps.append(dict(op="conv" if t == CONV else "fc", src=l, dst=out, relu=int(fuse), layers=[l]))
            l = out
        elif t == LORN:
            if not keep and l + 1 < L and ty[l + 1] == POOL:
                steps.append(dict(op="lrn_maxpool", src=l, dst=l + 2, relu=0, layers=[l, l + 1]))
                l += 2
            else:
                steps.append(dict(op="lrn", src=l, dst=l + 1, relu=0, layers=[l]))
                l += 1
        else:
            op = {RELU: "relu", POOL: "pool", SMAX: "softmax", DRPT: "drpt-copy" if keep else "drpt-alias"}[t]
            steps.append(dict(op=op, src=l, dst=l + 1, relu=0, layers=[l]))
            l += 1
    return steps


def first_reads_nchw(table):
    return table[0]["type"] == CONV and table[0]["stride"] > 1


def surviving_maps(table, steps, keep):
    """(maps with a non-NULL mapPtr, {map: the map it aliases})."""
    live = set() if (first_reads_nchw(table) and not keep) else {0}
    alias = {}
    for s in steps:
        live.add(s["dst"])
        if s["op"] == "drpt-alias":
            alias[s["dst"]] = alias.get(s["src"], s["src"])
    return live, alias


def branches(name, N, keep):
    """The executor branches one forward of table `name` at batch N takes, as labels."""
    layers, chw = TABLES[name][0], TABLES[name][1]
    from oracle import pyoracle as po
    shapes = po.infer_shapes(layers, chw)
    L = len(layers)
    ty = [t["type"] for t in layers]
    steps = plan_forward(layers, N, keep, chain_ok(name))
    out = set()
    f = layers[0]
    if ty[0] == CONV:
        cg = chw[0] // f["grp"]
        out.add("first:conv_s1" if f["stride"] == 1 else ("first:conv_strided_cg<=4" if cg <= 4 else "first:conv_strided_cg8"))
    else:
        out.add("first:" + {FCNT: "fc", RELU: "relu", DRPT: "drpt", POOL: "pool", LORN: "lrn", SMAX: "smax"}[ty[0]])
    for s in steps:
        op, a, b = s["op"], s["src"], s["dst"]
        nxt = ty[b] if b < L else None
        if op in ("conv", "fc"):
            l = s["layers"][0]
            if s["relu"]:
                out.add(op + ":fused_relu")
            elif not keep:
                out.add(op + ":no_relu")
            if op == "conv" and layers[l]["grp"] > 1:
                out.add("conv:grouped")
            if op == "conv" and l == L - 1:
                out.add("conv:last")
            if op == "fc" and l + 1 < L and ty[l + 1] == FCNT:
                out.add("fc:fc_direct")
        if op == "chain":
            run = s["layers"]
            out.add("chain:%d" % len(run))
            out.add("chain:relu" if any(s["relu"]) else "chain:no_relu")
            for x, y in zip(run, run[1:]):
                out.add("chain:drpt%d" % sum(1 for t in ty[x + 1:y] if t == DRPT))
            if len(run) == 4 and any(st["op"] in ("chain", "fc") and st["src"] > run[-1] for st in steps):
                out.add("chain:cap_then_next")
            if b < L and ty[b] == DRPT:
                out.add("chain:ends_drpt")
            if b < L and ty[b] == SMAX:
                out.add("chain:ends_smax")
            if b == L:
                out.add("chain:ends_net")
        if op == "fc" and N <= CHAIN_MAX_N and not keep:
            out.add("chain:rejected")
        if op == "lrn_maxpool":
            out.add("lrn:fused_b075" if layers[a]["beta"] == 0.75 else "lrn:fused_general")
        if op == "lrn":
            out.add("lrn:last" if b == L else "lrn:standalone")
        if op == "pool":
            out.add("pool:standalone")
        if op == "relu" and a > 0:
            out.add({POOL: "relu:after_pool", DRPT: "relu:after_drpt"}.get(ty[a - 1], "relu:after_other"))
        if op.startswith("drpt") and a > 0:
            prev = ty[a - 1]
            if prev == CONV:
                out.add("drpt:after_conv")
            if prev == RELU and a > 1 and ty[a - 2] == FCNT:
                out.add("drpt:after_fc_relu")
            if prev == DRPT:
                out.add("drpt:twice")
            if b == L:
                out.add("drpt:last")
        if op == "softmax":
            if b == L:
                out.add("smax:last")
            else:
                if a > 0 and ty[a - 1] == FCNT:
                    out.add("smax:mid_after_fc")
                if shapes[a][0] * shapes[a][1] > 1 and nxt == FCNT:
                    out.add("smax:spatial_then_fc")
    if ty[-1] != SMAX:
        out.add("smax:absent_last")
    return out


REQUIRED = {
    "first:conv_s1", "first:conv_strided_cg<=4", "first:conv_strided_cg8", "first:fc", "first:relu", "first:drpt",
    "first:pool",
    "conv:fused_relu", "conv:no_relu", "conv:last", "conv:grouped",
    "fc:fused_relu", "fc:no_relu", "fc:fc_direct",
    "chain:1", "chain:2", "chain:3", "chain:4", "chain:cap_then_next", "chain:relu", "chain:no_relu",
    "chain:drpt0", "chain:drpt1", "chain:drpt2", "chain:rejected", "chain:ends_smax", "chain:ends_drpt", "chain:ends_net",
    "lrn:fused_b075", "lrn:fused_general", "lrn:standalone", "lrn:last",
    "pool:standalone", "relu:after_pool", "relu:after_drpt",
    "drpt:after_conv", "drpt:after_fc_relu", "drpt:twice", "drpt:last",
    "smax:last", "smax:mid_after_fc", "smax:spatial_then_fc", "smax:absent_last",
}


def test_tables_reach_every_executor_branch(po):
    reached = set()
    for name, (layers, chw, pq, _, pin) in TABLES.items():
        shapes = po.infer_shapes(layers, chw)
        for l, t in enumerate(layers):
            h, w, c = shapes[l]
            if t["type"] == CONV:
                assert t["cnt"] // t["grp"] in (16, 32) and pq[l][1] % 8 == 0, (name, l)
                S, K, d = pq[l]
                assert S == -(-(c // t["grp"]) // d), (name, l)
            elif t["type"] == FCNT:
                S, K, d = pq[l]
                assert t["nod"] % 8 == 0 and K in (16, 32, 64, 128, 256) and S * d == h * w * c, (name, l)
            elif t["type"] == POOL:
                assert min(shapes[l + 1][:2]) >= 1 and (shapes[l + 1][0] - 1) * t["stride"] < h + t["pad"], (name, l)
        assert np.prod(chw) <= max(3 * 31 * 31, 8 * 16 * 16), name
        for N in (1, 130):
            for keep in (0, 1):
                reached |= branches(name, N, keep)
    assert REQUIRED <= reached, sorted(REQUIRED - reached)


def test_mirror_groups_as_the_executor_does():
    """Hand-checked steps: the chain cap, rejected runs, dropouts inside a chain, the keep_maps walk."""
    fc_first = plan_forward(TABLES["fc_first"][0], 1, False, chain_ok("fc_first"))
    assert [(s["op"], s["src"], s["dst"]) for s in fc_first] == [("chain", 0, 8), ("chain", 8, 9), ("softmax", 9, 10)]
    assert fc_first[0]["relu"] == [1, 1, 1, 1] and fc_first[1]["relu"] == [0]
    pinned = plan_forward(TABLES["pinned"][0], 4, False, chain_ok("pinned"))
    assert [(s["op"], s["src"], s["dst"], s["relu"]) for s in pinned] == [
        ("conv", 0, 2, 1), ("fc", 2, 4, 1), ("fc", 4, 6, 1), ("chain", 6, 7, [0]), ("softmax", 7, 8, 0)]
    drpt = plan_forward(TABLES["drpt_chain"][0], 3, False, chain_ok("drpt_chain"))
    assert [(s["op"], s["src"], s["dst"]) for s in drpt] == [("pool", 0, 1), ("chain", 1, 9), ("drpt-alias", 9, 10)]
    assert drpt[1]["layers"] == [1, 4, 7, 8] and drpt[1]["relu"] == [0, 1, 0, 0]
    live, alias = surviving_maps(TABLES["drpt_chain"][0], drpt, False)
    assert live == {0, 1, 9, 10} and alias == {10: 9}
    live, alias = surviving_maps(TABLES["strided8"][0], plan_forward(TABLES["strided8"][0], 9, False, None), False)
    assert live == {1, 2, 3, 4, 5, 6} and alias == {2: 1}
    keep = plan_forward(TABLES["relu_first"][0], 1, True, chain_ok("relu_first"))
    assert [s["dst"] for s in keep] == list(range(1, 15)) and all(s["relu"] == 0 for s in keep)


# ------------------------------------------------------------------------------------------------
# the oracle against the compiled reference (CPU)
# ------------------------------------------------------------------------------------------------
def synth(po, name):
    layers, chw, pq, scale, _ = TABLES[name]
    params = po.synth_model(layers, chw, pq, seed=sorted(TABLES).index(name) + 7, ctrd_std=None, bias_std=0.1)
    for l, s in scale.items():
        params[l]["ctrd"] = (params[l]["ctrd"] * np.float32(s)).astype(np.float32)
    return params


def images(name, N, seed=0):
    chw = TABLES[name][1]
    rng = np.random.RandomState(1000 + seed)
    return (rng.randn(N, *chw) * 4).astype(np.float32)


def first_fc_input(layers):
    return next((l for l, t in enumerate(layers) if t["type"] == FCNT), None)


@pytest.mark.parametrize("name", sorted(TABLES))
def test_oracle_matches_reference_on_table(po, tmp_path, name):
    """net_forward(keep=True) against the reference's featMapLst, bit for bit, at batch 1.  The reference leaves the
    first FC layer's input in NCHW element order."""
    if not po.have_ref():
        pytest.skip("oracle/_ref not built")
    layers, chw = TABLES[name][0], TABLES[name][1]
    params = synth(po, name)
    po.save_model(str(tmp_path), "t", params)
    ref = po.RefNet(str(tmp_path), "t", layers=layers, in_chw=chw)
    shapes = po.infer_shapes(layers, chw)
    ffc = first_fc_input(layers)
    try:
        img = images(name, 1, seed=3)
        prob = ref.forward(img[0])
        mine, maps = po.net_forward(layers, params, img, keep=True)
        assert np.array_equal(mine.reshape(-1), prob)
        for l in range(len(layers) + 1):
            m = maps[l]
            if l == ffc:
                m = po.nhwc_to_nchw(m.reshape((1,) + tuple(shapes[l])))
            assert np.array_equal(m.reshape(-1), ref.featmap(l).reshape(-1)), (name, l)
    finally:
        ref.close()


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
class LayerPara(C.Structure):
    """== qcnn_layer_para (include/qcnn.h)."""
    _fields_ = [("ctrd", C.c_void_p), ("asmt", C.c_void_p), ("bias", C.c_void_p), ("S", C.c_int), ("K", C.c_int),
                ("d", C.c_int)]


def layer_infos(qcnn, layers):
    return [qcnn.LayerInfo(L["type"], L.get("pad", 0), L.get("k", 0), L.get("cnt", 0), L.get("grp", 0),
                           L.get("stride", 0), L.get("nod", 0), L.get("size", 0), L.get("alpha", 0.0),
                           L.get("beta", 0.0), L.get("kini", 0.0), L.get("ratio", 0.0)) for L in layers]


@pytest.fixture(scope="module")
def models(po, tmp_path_factory):
    out = {}
    for name in TABLES:
        d = str(tmp_path_factory.mktemp("table_" + name))
        params = synth(po, name)
        po.save_model(d, "t", params)
        out[name] = (d, params)
    return out


def open_net(qcnn, ctx, models, name, mode):
    layers, chw, _, _, pin = TABLES[name]
    net = qcnn.Net(ctx, models[name][0], "t", layers=layer_infos(qcnn, layers), in_chw=chw)
    set_mode(net, mode)
    if pin is not None:
        net.pq_layer(pin).set_param("fc_tn", FC_TN_PIN)
    return net


def net_from_para(qcnn, ctx, name, params):
    """The same table through qcnn_net_create_from_para (asmt 0-based in file order)."""
    layers, chw = TABLES[name][0], TABLES[name][1]
    paras = (LayerPara * len(layers))()
    hold = []
    for l, p in params.items():
        ctrd = np.ascontiguousarray(p["ctrd"], np.float32)
        asmt = np.ascontiguousarray(p["asmt"], np.uint8)
        bias = np.ascontiguousarray(p["bias"], np.float32)
        hold += [ctrd, asmt, bias]
        S, K, d = ctrd.shape
        paras[l] = LayerPara(ctrd.ctypes.data, asmt.ctypes.data, bias.ctypes.data, S, K, d)
    infos = (qcnn.LayerInfo * len(layers))(*layer_infos(qcnn, layers))
    h = C.c_void_p()
    rc = qcnn.lib.qcnn_net_create_from_para(ctx.h, len(layers), infos, C.cast(paras, C.c_void_p), chw[0], chw[1],
                                            chw[2], C.byref(h))
    if rc:
        raise qcnn.QcnnError(qcnn.last_error())
    net = qcnn.Net.__new__(qcnn.Net)
    net.h, net.ctx = h, ctx
    net.out_len = qcnn.lib.qcnn_net_out_len(h)
    net.layer_count = qcnn.lib.qcnn_net_layer_count(h)
    return net


def raw_maps(qcnn, net):
    """mapPtr[0..L] of the last forward, as integers (0: fused away)."""
    out = []
    for l in range(net.layer_count + 1):
        p = C.c_void_p()
        d = (C.c_int * 4)()
        assert qcnn.lib.qcnn_net_featmap(net.h, l, C.byref(p), d) == 0
        out.append(p.value or 0)
    return out


def view(ptr, shape):
    import torch

    class _View(object):
        pass
    v = _View()
    v.__cuda_array_interface__ = dict(shape=tuple(shape), typestr="<f4", data=(ptr, False), version=2)
    return torch.as_tensor(v, device="cuda").clone()


def pq_forward(qcnn, net, conv, l, x, N, out_shape, relu):
    """The net's own PQ layer l (its handle, hence its tuned plan for batch N) on x."""
    import torch
    y = torch.empty((N,) + tuple(out_shape), dtype=torch.float32, device="cuda")
    fn = qcnn.lib.qcnn_conv_aprx_forward if conv else qcnn.lib.qcnn_fc_aprx_forward
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = fn(net.pq_layer(l).h, C.c_void_p(x.data_ptr()), N, C.c_void_p(y.data_ptr()), int(relu), stream)
    if rc:
        raise qcnn.QcnnError(qcnn.last_error())
    return y


def apply_step(qcnn, ctx, net, layers, step, x, N, shapes, img):
    """The op a step of the mirror runs, applied to x (the map at step['src'], or the NCHW image)."""
    op, a, b = step["op"], step["src"], step["dst"]
    t = layers[a]
    if op in ("conv", "fc"):
        src = img if (op == "conv" and a == 0 and first_reads_nchw(layers)) else x
        return pq_forward(qcnn, net, op == "conv", a, src, N, shapes[b], step["relu"])
    if op == "chain":
        return qcnn.fc_chain_forward([net.pq_layer(l) for l in step["layers"]], step["relu"], x.view(N, -1))
    if op == "relu":
        return ctx.relu(x)
    if op == "lrn":
        return ctx.lrn(x, t["size"], t["alpha"], t["beta"], t["kini"])
    if op == "lrn_maxpool":
        p = layers[a + 1]
        return ctx.lrn_maxpool(x, t["size"], t["alpha"], t["beta"], t["kini"], p["k"], p["pad"], p["stride"])
    if op == "pool":
        return ctx.maxpool(x, t["k"], t["pad"], t["stride"])
    if op == "softmax":
        return ctx.softmax(x.reshape(N, -1).contiguous())
    assert op in ("drpt-copy", "drpt-alias")
    return x


def check_against_oracle(po, layers, l, got, ref, RT, PT):
    """Probabilities (softmax outputs) to PT absolute, every other map to RT under close()."""
    got = np.asarray(got, np.float64).reshape(-1)
    ref = np.asarray(ref, np.float64).reshape(-1)
    if l > 0 and layers[l - 1]["type"] == SMAX:
        e = np.abs(got - ref).max()
        assert e <= PT, ("prob", l, e)
    else:
        e = close(got, ref)
        assert e <= RT, ("map", l, e)


def forward(net, imgd, keep, stream=None):
    import torch
    N = imgd.shape[0]
    net.set_keep_maps(keep)
    prob = torch.full((N, net.out_len), float("nan"), dtype=torch.float32, device="cuda")
    logits = torch.full((N, net.out_len), float("nan"), dtype=torch.float32, device="cuda")
    net.forward(imgd, prob=prob, logits=logits, stream=stream)
    torch.cuda.synchronize()
    return prob, logits


@pytest.mark.gpu
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("name", sorted(TABLES))
def test_table_keep_maps_oracle_and_composition(po, qcnn, ctx, models, name, mode):
    """keep_maps = 1: every featMapLst entry within the mode's tolerance of the oracle, and bit for bit the net's own
    layer applied to the map before it; the exits (logits, prob, out_len) as ForwardEager defines them."""
    import torch
    layers, chw = TABLES[name][0], TABLES[name][1]
    params = models[name][1]
    RT, PT = MODES[mode]
    shapes = po.infer_shapes(layers, chw)
    L = len(layers)
    net = open_net(qcnn, ctx, models, name, mode)
    assert net.layer_count == L and net.out_len == int(np.prod(shapes[-1]))
    if first_reads_nchw(layers) and chw[0] > 4:
        for N in (1, 130):   # conv_ws and pq_gemm_tc mode 1 fold at most 4 channels: the LUT + gather kernel does it
            plan = net.pq_layer(0).describe(N)
            assert plan.startswith("conv_") and not plan.startswith("conv_s1"), plan
    try:
        for N in NS:
            img = images(name, N, seed=N)
            imgd = torch.from_numpy(img).cuda()
            _, ref_maps = po.net_forward(layers, params, img, keep=True)
            prob, logits = forward(net, imgd, True)
            maps = [net.featmap(l, N) for l in range(L + 1)]
            for l in range(L + 1):
                assert maps[l] is not None, (N, l)
                check_against_oracle(po, layers, l, maps[l].cpu().numpy(), ref_maps[l], RT, PT)
            for l in range(L):
                t = layers[l]["type"]
                op = {CONV: "conv", FCNT: "fc", RELU: "relu", LORN: "lrn", POOL: "pool", DRPT: "drpt-copy",
                      SMAX: "softmax"}[t]
                y = apply_step(qcnn, ctx, net, layers, dict(op=op, src=l, dst=l + 1, relu=0, layers=[l]), maps[l], N, shapes,
                               imgd)
                assert torch.equal(y.reshape(-1), maps[l + 1].reshape(-1)), (name, mode, N, l)
            assert torch.equal(prob.reshape(-1), maps[L].reshape(-1))
            if layers[-1]["type"] == SMAX:
                assert torch.equal(logits.reshape(-1), maps[L - 1].reshape(-1)), (N, "logits")
            else:
                assert torch.equal(logits, prob), (N, "logits")
    finally:
        net.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("name", sorted(TABLES))
def test_table_fused_path(po, qcnn, ctx, models, name, mode):
    """keep_maps = 0: the maps that survive and alias are the mirror's, every surviving map is the fused op applied to
    the map it came from (bit for bit), and prob / logits are within the oracle tolerance."""
    import torch
    layers, chw = TABLES[name][0], TABLES[name][1]
    params = models[name][1]
    RT, PT = MODES[mode]
    shapes = po.infer_shapes(layers, chw)
    L = len(layers)
    net = open_net(qcnn, ctx, models, name, mode)
    try:
        for N in NS:
            img = images(name, N, seed=N)
            imgd = torch.from_numpy(img).cuda()
            ref_prob, ref_maps = po.net_forward(layers, params, img, keep=True)
            prob, logits = forward(net, imgd, False)
            ptr = raw_maps(qcnn, net)
            steps = plan_forward(layers, N, False, chain_ok(name))
            live, alias = surviving_maps(layers, steps, False)
            assert {l for l in range(L + 1) if ptr[l]} == live, (N, ptr)
            for b, a in alias.items():
                assert ptr[b] == ptr[a], (N, b, a)
            owners = [l for l in live if l not in alias]
            assert len({ptr[l] for l in owners}) == len(owners), (N, ptr)
            if layers[-1]["type"] == SMAX:
                assert ptr[L] == prob.data_ptr()
            for s in steps:
                if s["op"] == "drpt-alias":
                    continue
                a, b = s["src"], s["dst"]
                x = view(ptr[a], (N,) + tuple(shapes[a])) if ptr[a] else None
                y = apply_step(qcnn, ctx, net, layers, s, x, N, shapes, imgd)
                assert torch.equal(y.reshape(-1), view(ptr[b], (N,) + tuple(shapes[b])).reshape(-1)), (name, mode, N, s)
            last = view(ptr[L], (N,) + tuple(shapes[L]))
            if layers[-1]["type"] == SMAX:
                assert torch.equal(logits.reshape(-1), view(ptr[L - 1], (N,) + tuple(shapes[L - 1])).reshape(-1))
                check_against_oracle(po, layers, L, prob.cpu().numpy(), ref_prob, RT, PT)
                assert close(logits.cpu().numpy(), ref_maps[L - 1]) <= RT
            else:
                assert torch.equal(prob.reshape(-1), last.reshape(-1)) and torch.equal(logits, prob)
                check_against_oracle(po, layers, L, prob.cpu().numpy(), ref_maps[L], RT, PT)
    finally:
        net.close()


GRAPH_NS = (1, 4, 8)


def side_passes(net, imgd, prob, logits, side, n):
    import torch
    out = []
    with torch.cuda.stream(side):
        for _ in range(n):
            net.forward(imgd, prob=prob, logits=logits)
            side.synchronize()
            out.append((prob.clone(), logits.clone()))
    return out


def eager(net, imgd):
    """A forward on the legacy default stream, which is never captured."""
    import torch
    N = imgd.shape[0]
    prob = torch.empty((N, net.out_len), dtype=torch.float32, device="cuda")
    logits = torch.empty((N, net.out_len), dtype=torch.float32, device="cuda")
    net.forward(imgd, prob=prob, logits=logits, stream=0)
    torch.cuda.synchronize()
    return prob, logits


def same(a, b):
    import torch
    return torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def pick_tc_layer(net, N):
    """The first conv layer that runs a tensor-core GEMM at batch N, which tensor_core = 0 moves to the LUT + gather
    kernels (FC layers run them below 96 images anyway), else the first PQ layer; and whether the plan changes."""
    pq = [l for l in range(net.layer_count) if net.pq_layer(l) is not None]
    for l in pq:
        if net.pq_layer(l).describe(N).startswith("pq_gemm_tc"):
            return l, True
    return pq[0], False


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(TABLES))
def test_graph_replay_follows_set_param(po, qcnn, ctx, models, name):
    """Passes 3-6 on a side stream are replays of pass 1; after tensor_core = 0 on one layer the next call equals a
    fresh eager strict run, not the graph captured before."""
    import torch
    layers = TABLES[name][0]
    side = torch.cuda.Stream()
    for N in GRAPH_NS:
        net = open_net(qcnn, ctx, models, name, "default")
        try:
            net.set_keep_maps(False)
            imgd = torch.from_numpy(images(name, N, seed=50 + N)).cuda()
            prob = torch.empty((N, net.out_len), dtype=torch.float32, device="cuda")
            logits = torch.empty_like(prob)
            outs = side_passes(net, imgd, prob, logits, side, 6)
            for i in range(1, 6):
                assert same(outs[i], outs[0]), (N, i)
            assert same(eager(net, imgd), outs[0]), N
            l, changes = pick_tc_layer(net, N)
            net.pq_layer(l).set_param("tensor_core", 0)
            after = side_passes(net, imgd, prob, logits, side, 4)
            fresh = eager(net, imgd)
            for i in range(4):
                assert same(after[i], fresh), (N, l, i)
            if changes:   # the strict plan computes other sums: a stale replay would be seen
                assert not same(fresh, outs[0]), (N, l)
        finally:
            net.close()
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(TABLES))
def test_graph_cache_regrow_repack_evict(po, qcnn, ctx, models, name):
    """A larger batch that regrows the maps, a repacked FC assignment table and a 9th buffer set (the cache holds 8)
    never leave a stale graph: every side-stream result equals the eager pass."""
    import torch
    layers, chw = TABLES[name][0], TABLES[name][1]
    params = models[name][1]
    RT, PT = MODES["default"]
    side = torch.cuda.Stream()
    net = open_net(qcnn, ctx, models, name, "default")
    net.set_keep_maps(False)
    try:
        grow = 16
        for N in GRAPH_NS:
            img = images(name, N, seed=70 + N)
            imgd = torch.from_numpy(img).cuda()
            prob = torch.empty((N, net.out_len), dtype=torch.float32, device="cuda")
            logits = torch.empty_like(prob)
            outs = side_passes(net, imgd, prob, logits, side, 4)
            assert all(same(o, outs[0]) for o in outs), N
            _, ref_maps = po.net_forward(layers, params, img, keep=True)
            check_against_oracle(po, layers, len(layers), outs[0][0].cpu().numpy(), ref_maps[-1], RT, PT)
            # a larger batch regrows the feature maps (and bumps the allocation epoch)
            grow += 8
            eager(net, torch.from_numpy(images(name, grow, seed=grow)).cuda())
            for o in side_passes(net, imgd, prob, logits, side, 4):
                assert same(o, outs[0]), (N, "regrow")
            # nine buffer sets, each replayed: the oldest graph is evicted and re-created on its next use
            bufs = [(torch.empty_like(prob), torch.empty_like(prob)) for _ in range(9)]
            for _ in range(2):
                for pb, lb in bufs:
                    for o in side_passes(net, imgd, pb, lb, side, 3):
                        assert same(o, outs[0]), (N, "evict")
        if any(t["type"] == FCNT for t in layers):
            net.set_asmt_packed(True)
            for N in GRAPH_NS:
                img = images(name, N, seed=90 + N)
                imgd = torch.from_numpy(img).cuda()
                prob = torch.empty((N, net.out_len), dtype=torch.float32, device="cuda")
                logits = torch.empty_like(prob)
                outs = side_passes(net, imgd, prob, logits, side, 5)
                fresh = eager(net, imgd)
                assert all(same(o, fresh) for o in outs), (N, "packed")
                _, ref_maps = po.net_forward(layers, params, img, keep=True)
                check_against_oracle(po, layers, len(layers), fresh[0].cpu().numpy(), ref_maps[-1], RT, PT)
    finally:
        net.close()
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("name", sorted(TABLES))
def test_create_from_para_equals_create_custom(po, qcnn, ctx, models, name, mode):
    """Both construction entries build the same net: bit-identical prob and logits (autotuning off, so both pick the
    cost model's first tiling)."""
    import torch
    a = open_net(qcnn, ctx, models, name, mode)
    b = net_from_para(qcnn, ctx, name, models[name][1])
    set_mode(b, mode)
    pin = TABLES[name][4]
    if pin is not None:
        b.pq_layer(pin).set_param("fc_tn", FC_TN_PIN)
    try:
        for net in (a, b):
            for l, t in enumerate(TABLES[name][0]):
                if t["type"] == CONV:
                    net.pq_layer(l).set_param("autotune", 0)
        for N in (1, 5, 130):
            imgd = torch.from_numpy(images(name, N, seed=200 + N)).cuda()
            for keep in (True, False):
                assert same(forward(a, imgd, keep), forward(b, imgd, keep)), (N, keep)
    finally:
        a.close()
        b.close()
