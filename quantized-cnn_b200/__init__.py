"""quantized-cnn_b200: Python binding (ctypes) of the H100-native (sm_90a) PQ forward path.

The product is ``libqcnn_b200.so`` (hand-written sm_90a CUDA + C++ host code behind the C ABI of
``include/qcnn.h``).  This module only marshals pointers: torch supplies device memory and streams, every
computation happens inside the shared library.  There is no CPU or PyTorch fallback -- if the library is
missing or no H100 is visible the calls raise.

The directory name contains a hyphen, so import it with::

    import importlib; q = importlib.import_module("quantized-cnn_b200")
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libqcnn_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "qcnn.h")


class QcnnError(RuntimeError):
    pass


def build(verbose=False):
    """Compile libqcnn_b200.so in-tree with nvcc for sm_90a (see Makefile)."""
    import subprocess
    cmd = ["make", "-C", _HERE, "-j8"]
    if not verbose:
        cmd.insert(1, "-s")
    subprocess.check_call(cmd)


def _load():
    if not os.path.exists(LIB_PATH):
        raise QcnnError("%s is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                        "(there is no fallback path)" % LIB_PATH)
    return C.CDLL(LIB_PATH)


lib = _load()


class LayerInfo(C.Structure):
    """== qcnn_layer_info == the reference's LayerInfo (include/CaffePara.h:28-41)."""
    _fields_ = [("type", C.c_int), ("padSiz", C.c_int), ("knlSiz", C.c_int), ("knlCnt", C.c_int),
                ("grpCnt", C.c_int), ("stride", C.c_int), ("nodCnt", C.c_int), ("lrnSiz", C.c_int),
                ("lrnAlp", C.c_float), ("lrnBet", C.c_float), ("lrnIni", C.c_float), ("drpRat", C.c_float)]


_vp, _i, _f, _sz, _cp = C.c_void_p, C.c_int, C.c_float, C.c_size_t, C.c_char_p
_dp = C.POINTER(C.c_double)
_SIGS = {
    "qcnn_version": (_cp, []),
    "qcnn_last_error": (_cp, []),
    "qcnn_ctx_create": (_i, [_i, C.POINTER(_vp)]),
    "qcnn_ctx_destroy": (None, [_vp]),
    "qcnn_ctx_device": (_i, [_vp]),
    "qcnn_ctx_sm_count": (_i, [_vp]),
    "qcnn_dev_alloc": (_i, [_vp, _sz, C.POINTER(_vp)]),
    "qcnn_dev_free": (_i, [_vp, _vp]),
    "qcnn_copy_h2d": (_i, [_vp, _vp, _vp, _sz, _vp]),
    "qcnn_copy_d2h": (_i, [_vp, _vp, _vp, _sz, _vp]),
    "qcnn_stream_sync": (_i, [_vp, _vp]),
    "qcnn_conv_layer_create": (_i, [_vp] + [_i] * 11 + [_vp, _vp, _vp, C.POINTER(_vp)]),
    "qcnn_fc_layer_create": (_i, [_vp] + [_i] * 5 + [_vp, _vp, _vp, C.POINTER(_vp)]),
    "qcnn_fc_layer_set_src_nhwc": (_i, [_vp, _i, _i, _i]),
    "qcnn_conv_layer_set_src_nchw": (_i, [_vp, _i]),
    "qcnn_layer_set_param": (_i, [_vp, _cp, _i]),
    "qcnn_layer_describe": (_i, [_vp, _i, _cp, _sz]),
    "qcnn_layer_destroy": (None, [_vp]),
    "qcnn_layer_out_dims": (_i, [_vp, C.POINTER(_i)]),
    "qcnn_layer_work": (_i, [_vp, _i, _dp, _dp, _dp]),
    "qcnn_layer_read_asmt_h": (_i, [_vp, _vp, _sz]),
    "qcnn_layer_read_w_ws": (_i, [_vp, _vp, _sz, C.POINTER(_sz)]),
    "qcnn_conv_aprx_forward": (_i, [_vp, _vp, _i, _vp, _i, _vp]),
    "qcnn_fc_aprx_forward": (_i, [_vp, _vp, _i, _vp, _i, _vp]),
    "qcnn_fc_aprx_forward_flat": (_i, [_vp, _vp, _i, _vp, _i, _vp]),
    "qcnn_fc_chain_forward": (_i, [C.POINTER(_vp), C.POINTER(_i), _i, _vp, _i, _vp, _vp, _vp]),
    "qcnn_relu": (_i, [_vp, _vp, _vp, _sz, _vp]),
    "qcnn_lrn": (_i, [_vp, _vp, _vp, _sz, _i, _i, _f, _f, _f, _vp]),
    "qcnn_maxpool": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "qcnn_lrn_maxpool": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _f, _f, _i, _i, _i, _vp]),
    "qcnn_softmax": (_i, [_vp, _vp, _vp, _i, _i, _vp]),
    "qcnn_nchw_to_nhwc": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "qcnn_nhwc_to_nchw": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "qcnn_net_create": (_i, [_vp, _cp, _cp, _cp, C.POINTER(_vp)]),
    "qcnn_net_create_custom": (_i, [_vp, _i, C.POINTER(LayerInfo), _i, _i, _i, _cp, _cp, C.POINTER(_vp)]),
    "qcnn_net_create_from_para": (_i, [_vp, _i, C.POINTER(LayerInfo), _vp, _i, _i, _i, C.POINTER(_vp)]),
    "qcnn_net_destroy": (None, [_vp]),
    "qcnn_net_layer_count": (_i, [_vp]),
    "qcnn_net_out_len": (_i, [_vp]),
    "qcnn_net_set_keep_maps": (_i, [_vp, _i]),
    "qcnn_net_forward": (_i, [_vp, _vp, _i, _vp, _vp, _vp]),
    "qcnn_net_forward_h": (_i, [_vp, _vp, _i, _vp, _vp]),
    "qcnn_net_forward_topk_h": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "qcnn_net_set_input_mean": (_i, [_vp, _vp]),
    "qcnn_net_forward_u8": (_i, [_vp, _vp, _i, _vp, _vp, _vp]),
    "qcnn_net_forward_u8_h": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "qcnn_net_submit_u8_h": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, C.POINTER(_i)]),
    "qcnn_net_wait": (_i, [_vp, _i]),
    "qcnn_net_set_chunk": (_i, [_vp, _i]),
    "qcnn_net_set_asmt_packed": (_i, [_vp, _i]),
    "qcnn_net_featmap": (_i, [_vp, _i, C.POINTER(_vp), C.POINTER(_i)]),
    "qcnn_net_set_profiling": (_i, [_vp, _i]),
    "qcnn_net_layer_time_ms": (_i, [_vp, _i, C.POINTER(_f)]),
    "qcnn_net_layer_work": (_i, [_vp, _i, _i, _dp, _dp, _dp]),
    "qcnn_net_launch_count": (_i, [_vp]),
    "qcnn_net_pq_layer": (_vp, [_vp, _i]),
    "qcnn_topk": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "qcnn_u8hwc_to_f32chw": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "qcnn_preproc_create": (_i, [_vp, _i, _i, _i, _i, _i, _i, _vp, _i, _i, C.POINTER(_vp)]),
    "qcnn_preproc_destroy": (None, [_vp]),
    "qcnn_preproc_run": (_i, [_vp, _vp, C.POINTER(C.c_longlong), C.POINTER(_i), C.POINTER(_i), _i, _vp, _vp]),
    "qcnn_multi_create": (_i, [_i, C.POINTER(_i), _cp, _cp, _cp, C.POINTER(_vp)]),
    "qcnn_multi_create_from_para": (_i, [_i, C.POINTER(_i), _i, C.POINTER(LayerInfo), _vp, _i, _i, _i, C.POINTER(_vp)]),
    "qcnn_multi_destroy": (None, [_vp]),
    "qcnn_multi_device_count": (_i, [_vp]),
    "qcnn_multi_out_len": (_i, [_vp]),
    "qcnn_multi_nccl_version": (_i, [_vp]),
    "qcnn_multi_net": (_vp, [_vp, _i]),
    "qcnn_multi_forward_h": (_i, [_vp, _vp, _i, _vp]),
    "qcnn_multi_forward": (_i, [_vp, C.POINTER(_vp), _i, C.POINTER(_vp)]),
    "qcnn_multi_sync": (_i, [_vp]),
    "qcnn_read_bin_f32": (C.c_long, [_cp, C.POINTER(_i), C.POINTER(_i), _vp, C.c_long]),
    "qcnn_write_bin_f32": (_i, [_cp, _i, C.POINTER(_i), _vp]),
    "qcnn_read_cbn_u8": (C.c_long, [_cp, C.POINTER(_i), C.POINTER(_i), C.POINTER(_i), _vp, C.c_long]),
    "qcnn_write_cbn_u8": (_i, [_cp, _i, C.POINTER(_i), _vp, _i]),
    "qcnn_pq_quantize_conv": (_i, [_vp] + [_i] * 6 + [C.c_uint32, _vp, _vp, _vp, _vp, _vp]),
    "qcnn_pq_quantize_fc": (_i, [_vp] + [_i] * 5 + [C.c_uint32, _vp, _vp, _vp, _vp, _vp]),
    "qcnn_pq_quantize_model": (_i, [_vp, _cp, _cp, _cp, C.POINTER(_i), C.POINTER(_i), _i, C.c_uint32, _cp, _cp]),
    "qcnn_pq_refine_fc": (_i, [_vp] + [_i] * 5 + [_vp, _vp, _i, _vp, _vp, _vp, _vp]),
    "qcnn_pq_refine_conv": (_i, [_vp] + [_i] * 11 + [_vp, _vp, _i, _vp, _vp, _vp, _vp]),
    "qcnn_pq_refine_fc_target": (_i, [_vp] + [_i] * 5 + [_vp, _vp, _i, _vp, _vp, _vp, _vp]),
    "qcnn_pq_refine_conv_target": (_i, [_vp] + [_i] * 11 + [_vp, _vp, _i, _vp, _vp, _vp, _vp]),
    "qcnn_pq_stats_create_fc": (_i, [_vp] + [_i] * 4 + [C.POINTER(_vp)]),
    "qcnn_pq_stats_create_conv": (_i, [_vp] + [_i] * 10 + [C.POINTER(_vp)]),
    "qcnn_pq_stats_add": (_i, [_vp, _vp, _vp, _i, _vp]),
    "qcnn_pq_stats_count": (_i, [_vp, C.POINTER(C.c_longlong)]),
    "qcnn_pq_stats_read_h": (_i, [_vp, _vp, _vp, _vp]),
    "qcnn_pq_stats_refine": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "qcnn_pq_stats_refine_target": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp]),
    "qcnn_pq_stats_read_sums_h": (_i, [_vp, _vp, _vp, C.POINTER(C.c_longlong)]),
    "qcnn_pq_stats_refine_bias": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "qcnn_pq_stats_refine_target_bias": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "qcnn_pq_stats_refine_damped": (_i, [_vp, _i, C.c_double, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "qcnn_pq_stats_destroy": (None, [_vp]),
}
for _name, (_res, _args) in _SIGS.items():
    _fn = getattr(lib, _name)
    _fn.restype = _res
    _fn.argtypes = _args
EXPORTS = sorted(_SIGS)


def last_error():
    return lib.qcnn_last_error().decode()


def _check(rc):
    if rc != 0:
        raise QcnnError(last_error())


def _np(a, dt):
    return np.ascontiguousarray(a, dtype=dt)


def _stream(stream):
    if stream is not None:
        return C.c_void_p(int(stream))
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _dptr(t):
    """Device pointer of a contiguous float32 CUDA tensor."""
    import torch
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
        raise QcnnError("expected a contiguous float32 CUDA tensor")
    return C.c_void_p(t.data_ptr())


class Context(object):
    def __init__(self, device=0):
        h = _vp()
        _check(lib.qcnn_ctx_create(device, C.byref(h)))
        self.h = h
        self.device = device

    @property
    def sm_count(self):
        return lib.qcnn_ctx_sm_count(self.h)

    def close(self):
        if self.h:
            lib.qcnn_ctx_destroy(self.h)
            self.h = None

    # ---- supporting layers; tensors are NHWC float32 on the context's device ----
    def relu(self, x, stream=None):
        import torch
        y = torch.empty_like(x)
        _check(lib.qcnn_relu(self.h, _dptr(x), _dptr(y), x.numel(), _stream(stream)))
        return y

    def lrn(self, x, size, alpha, beta, k, stream=None):
        import torch
        y = torch.empty_like(x)
        _check(lib.qcnn_lrn(self.h, _dptr(x), _dptr(y), x.numel() // x.shape[-1], x.shape[-1], size, alpha, beta, k,
                            _stream(stream)))
        return y

    @staticmethod
    def _pool_out(n, pad, ksz, stride):
        return -((-(n + 2 * pad - ksz)) // stride) + 1

    def maxpool(self, x, ksz, pad, stride, stream=None):
        import torch
        N, H, W, Cc = x.shape
        y = torch.empty((N, self._pool_out(H, pad, ksz, stride), self._pool_out(W, pad, ksz, stride), Cc),
                        dtype=torch.float32, device=x.device)
        _check(lib.qcnn_maxpool(self.h, _dptr(x), _dptr(y), N, H, W, Cc, ksz, pad, stride, _stream(stream)))
        return y

    def lrn_maxpool(self, x, size, alpha, beta, k, ksz, pad, stride, stream=None):
        import torch
        N, H, W, Cc = x.shape
        y = torch.empty((N, self._pool_out(H, pad, ksz, stride), self._pool_out(W, pad, ksz, stride), Cc),
                        dtype=torch.float32, device=x.device)
        _check(lib.qcnn_lrn_maxpool(self.h, _dptr(x), _dptr(y), N, H, W, Cc, size, alpha, beta, k, ksz, pad, stride,
                                    _stream(stream)))
        return y

    def softmax(self, x, stream=None):
        import torch
        y = torch.empty_like(x)
        _check(lib.qcnn_softmax(self.h, _dptr(x), _dptr(y), x.shape[0], x.numel() // x.shape[0], _stream(stream)))
        return y

    def topk(self, prob, k, mode=0, stream=None):
        """k-fold arg-max (first maximum wins, winner zeroed) of every row; returns (idx int32 [N,k], val [N,k])."""
        import torch
        N, Cc = prob.shape
        idx = torch.empty((N, k), dtype=torch.int32, device=prob.device)
        val = torch.empty((N, k), dtype=torch.float32, device=prob.device)
        _check(lib.qcnn_topk(self.h, _dptr(prob), N, Cc, k, mode, C.c_void_p(idx.data_ptr()), _dptr(val), _stream(stream)))
        return idx, val

    def nchw_to_nhwc(self, x, stream=None):
        import torch
        N, Cc, H, W = x.shape
        y = torch.empty((N, H, W, Cc), dtype=torch.float32, device=x.device)
        _check(lib.qcnn_nchw_to_nhwc(self.h, _dptr(x), _dptr(y), N, Cc, H, W, _stream(stream)))
        return y

    def nhwc_to_nchw(self, x, stream=None):
        import torch
        N, H, W, Cc = x.shape
        y = torch.empty((N, Cc, H, W), dtype=torch.float32, device=x.device)
        _check(lib.qcnn_nhwc_to_nchw(self.h, _dptr(x), _dptr(y), N, H, W, Cc, _stream(stream)))
        return y


class _Layer(object):
    def __init__(self, ctx, h, owned=True):
        self.ctx, self.h, self.owned = ctx, h, owned

    def close(self):
        if self.h and self.owned:
            lib.qcnn_layer_destroy(self.h)
        self.h = None

    def out_dims(self):
        d = (_i * 3)()
        _check(lib.qcnn_layer_out_dims(self.h, d))
        return tuple(d)

    def work(self, N):
        b, l, m = C.c_double(), C.c_double(), C.c_double()
        _check(lib.qcnn_layer_work(self.h, N, C.byref(b), C.byref(l), C.byref(m)))
        return dict(alg_bytes=b.value, lookups=l.value, lut_macs=m.value)

    def describe(self, N):
        buf = C.create_string_buffer(512)
        _check(lib.qcnn_layer_describe(self.h, N, buf, 512))
        return buf.value.decode()

    def set_param(self, name, value):
        _check(lib.qcnn_layer_set_param(self.h, name.encode(), value))

    def read_asmt(self, n):
        out = np.empty(n, np.uint8)
        _check(lib.qcnn_layer_read_asmt_h(self.h, out.ctypes.data_as(_vp), out.size))
        return out

    def read_w_ws(self):
        """The layer's weight image as uint8 bytes (include/qcnn.h: qcnn_layer_read_w_ws); empty without one."""
        n = _sz()
        _check(lib.qcnn_layer_read_w_ws(self.h, None, 0, C.byref(n)))
        out = np.empty(n.value, np.uint8)
        if out.size:
            _check(lib.qcnn_layer_read_w_ws(self.h, out.ctypes.data_as(_vp), out.size, C.byref(n)))
        return out


class ConvLayer(_Layer):
    """PQ convolution; parameters as CaffePara holds them (ctrd [S,K,d], asmt [Cout,k,k,S] 0-based, bias [Cout])."""

    def __init__(self, ctx, Cin, Hin, Win, Cout, ksz, pad, stride, grp, ctrd, asmt, bias):
        ctrd, asmt, bias = _np(ctrd, np.float32), _np(asmt, np.uint8), _np(bias, np.float32)
        S, K, d = ctrd.shape
        assert asmt.shape == (Cout, ksz, ksz, S), asmt.shape
        h = _vp()
        _check(lib.qcnn_conv_layer_create(ctx.h, Cin, Hin, Win, Cout, ksz, pad, stride, grp, S, K, d,
                                          ctrd.ctypes.data_as(_vp), asmt.ctypes.data_as(_vp),
                                          bias.ctypes.data_as(_vp), C.byref(h)))
        _Layer.__init__(self, ctx, h)
        self.shape_in = (Hin, Win, Cin)
        self.n_asmt = asmt.size

    def set_src_nchw(self, enable=True):
        _check(lib.qcnn_conv_layer_set_src_nchw(self.h, int(enable)))

    def forward(self, x, relu=False, stream=None):
        import torch
        ho, wo, co = self.out_dims()
        y = torch.empty((x.shape[0], ho, wo, co), dtype=torch.float32, device=x.device)
        _check(lib.qcnn_conv_aprx_forward(self.h, _dptr(x), x.shape[0], _dptr(y), int(relu), _stream(stream)))
        return y


class FcLayer(_Layer):
    """PQ fully-connected layer; ctrd [S,K,d], asmt [Dout,S] 0-based, bias [Dout]."""

    def __init__(self, ctx, Din, ctrd, asmt, bias):
        ctrd, asmt, bias = _np(ctrd, np.float32), _np(asmt, np.uint8), _np(bias, np.float32)
        S, K, d = ctrd.shape
        Dout = asmt.shape[0]
        assert asmt.shape == (Dout, S)
        h = _vp()
        _check(lib.qcnn_fc_layer_create(ctx.h, Din, Dout, S, K, d, ctrd.ctypes.data_as(_vp),
                                        asmt.ctypes.data_as(_vp), bias.ctypes.data_as(_vp), C.byref(h)))
        _Layer.__init__(self, ctx, h)
        self.Din, self.Dout = Din, Dout
        self.n_asmt = asmt.size

    def set_src_nhwc(self, H, W, Cc):
        _check(lib.qcnn_fc_layer_set_src_nhwc(self.h, H, W, Cc))

    def forward(self, x, relu=False, stream=None):
        import torch
        N = x.shape[0]
        y = torch.empty((N, self.Dout), dtype=torch.float32, device=x.device)
        _check(lib.qcnn_fc_aprx_forward(self.h, _dptr(x), N, _dptr(y), int(relu), _stream(stream)))
        return y


def fc_chain_forward(layers, relu, x, stamps=None, stream=None):
    """Consecutive FC layers (FcLayer objects) as one persistent launch; x [N<=4, Din]; returns [N, Dout of the last]."""
    import torch
    n = len(layers)
    hs = (_vp * n)(*[l.h for l in layers])
    rl = (_i * n)(*[int(r) for r in relu])
    N = x.shape[0]
    y = torch.empty((N, layers[-1].out_dims()[2]), dtype=torch.float32, device=x.device)
    sp = C.c_void_p(stamps.data_ptr()) if stamps is not None else None
    _check(lib.qcnn_fc_chain_forward(hs, rl, n, _dptr(x), N, _dptr(y), sp, _stream(stream)))
    return y


class Net(object):
    """Device-resident network == CaffeEva::LoadCaffePara + ExecForwardPass (reference src/CaffeEva.cc:109-261)."""

    def __init__(self, ctx, dirpath, pfx, model="AlexNet", layers=None, in_chw=None):
        h = _vp()
        if layers is None:
            _check(lib.qcnn_net_create(ctx.h, model.encode(), dirpath.encode(), pfx.encode(), C.byref(h)))
        else:
            arr = (LayerInfo * len(layers))(*layers)
            _check(lib.qcnn_net_create_custom(ctx.h, len(layers), arr, in_chw[0], in_chw[1], in_chw[2],
                                              dirpath.encode(), pfx.encode(), C.byref(h)))
        self.h, self.ctx = h, ctx
        self.out_len = lib.qcnn_net_out_len(h)
        self.layer_count = lib.qcnn_net_layer_count(h)

    def close(self):
        if self.h:
            lib.qcnn_net_destroy(self.h)
            self.h = None

    def set_keep_maps(self, keep):
        _check(lib.qcnn_net_set_keep_maps(self.h, int(keep)))

    def set_profiling(self, on):
        _check(lib.qcnn_net_set_profiling(self.h, int(on)))

    def set_chunk(self, n):
        _check(lib.qcnn_net_set_chunk(self.h, n))

    def set_asmt_packed(self, enable=True):
        """Keep every FC assignment table bit-packed at log2(K) bits per index on the device (outputs are unchanged)."""
        _check(lib.qcnn_net_set_asmt_packed(self.h, int(enable)))

    def forward(self, img, prob=None, logits=None, stream=None):
        """img: CUDA float32 [N,C,H,W]; returns prob [N,out_len] (device)."""
        import torch
        N = img.shape[0]
        if prob is None:
            prob = torch.empty((N, self.out_len), dtype=torch.float32, device=img.device)
        _check(lib.qcnn_net_forward(self.h, _dptr(img), N, _dptr(prob), _dptr(logits) if logits is not None else None,
                                    _stream(stream)))
        return prob

    def forward_host(self, img_h, prob_h=None, logits_h=None):
        """img_h: host float32 array/tensor [N,C,H,W] (pinned for full overlap); returns host probs."""
        def ptr(a):
            if hasattr(a, "data_ptr"):
                return C.c_void_p(a.data_ptr())
            return a.ctypes.data_as(_vp)
        N = img_h.shape[0]
        if prob_h is None:
            prob_h = np.empty((N, self.out_len), np.float32)
        _check(lib.qcnn_net_forward_h(self.h, ptr(img_h), N, ptr(prob_h), ptr(logits_h) if logits_h is not None else None))
        return prob_h

    def set_input_mean(self, mean_chw):
        if mean_chw is None:
            _check(lib.qcnn_net_set_input_mean(self.h, None))
        else:
            m = _np(mean_chw, np.float32)
            _check(lib.qcnn_net_set_input_mean(self.h, m.ctypes.data_as(_vp)))

    def forward_u8(self, img_u8, prob=None, logits=None, stream=None):
        """img_u8: CUDA uint8 [N,H,W,C] interleaved pixels; returns prob [N,out_len] (device)."""
        import torch
        N = img_u8.shape[0]
        if prob is None:
            prob = torch.empty((N, self.out_len), dtype=torch.float32, device=img_u8.device)
        assert img_u8.dtype == torch.uint8 and img_u8.is_contiguous()
        _check(lib.qcnn_net_forward_u8(self.h, C.c_void_p(img_u8.data_ptr()), N, _dptr(prob),
                                       _dptr(logits) if logits is not None else None, _stream(stream)))
        return prob

    @staticmethod
    def _hptr(a):
        if a is None:
            return None
        return C.c_void_p(a.data_ptr()) if hasattr(a, "data_ptr") else a.ctypes.data_as(_vp)

    def forward_topk_host(self, img_h, k, mode=0, idx_h=None, val_h=None, prob_h=None):
        """fp32 host images in, on-device top-k out: (idx int32 [N,k], prob [N,k])."""
        N = img_h.shape[0]
        idx_h = np.empty((N, k), np.int32) if idx_h is None else idx_h
        val_h = np.empty((N, k), np.float32) if val_h is None else val_h
        _check(lib.qcnn_net_forward_topk_h(self.h, self._hptr(img_h), N, k, mode, self._hptr(idx_h), self._hptr(val_h),
                                           self._hptr(prob_h)))
        return idx_h, val_h

    def forward_u8_host(self, img_h, k=0, mode=0, idx_h=None, val_h=None, prob_h=None):
        """uint8 host pixels [N,H,W,C] in; top-k (k > 0) and / or probabilities (prob_h) out."""
        N = img_h.shape[0]
        if k > 0:
            idx_h = np.empty((N, k), np.int32) if idx_h is None else idx_h
            val_h = np.empty((N, k), np.float32) if val_h is None else val_h
        elif prob_h is None:
            prob_h = np.empty((N, self.out_len), np.float32)
        _check(lib.qcnn_net_forward_u8_h(self.h, self._hptr(img_h), N, k, mode, self._hptr(idx_h), self._hptr(val_h),
                                         self._hptr(prob_h)))
        return (idx_h, val_h) if k > 0 else prob_h

    def submit_u8_host(self, img_h, k=0, mode=0, idx_h=None, val_h=None, prob_h=None):
        """Asynchronous uint8 step (pinned buffers); returns a ticket for wait()."""
        t = _i()
        _check(lib.qcnn_net_submit_u8_h(self.h, self._hptr(img_h), img_h.shape[0], k, mode, self._hptr(idx_h), self._hptr(val_h),
                                        self._hptr(prob_h), C.byref(t)))
        return t.value

    def wait(self, ticket):
        _check(lib.qcnn_net_wait(self.h, ticket))

    def featmap(self, idx, N):
        """featMapLst[idx] of the last forward as a torch view [N,H,W,C] (None if fused away)."""
        import torch
        p = _vp()
        d = (_i * 4)()
        _check(lib.qcnn_net_featmap(self.h, idx, C.byref(p), d))
        if not p.value:
            return None
        class _View(object):
            pass
        v = _View()
        v.__cuda_array_interface__ = dict(shape=(N, d[1], d[2], d[3]), typestr="<f4", data=(p.value, False), version=2)
        return torch.as_tensor(v, device="cuda:%d" % self.ctx.device).clone()

    def layer_time_ms(self, l):
        v = _f()
        _check(lib.qcnn_net_layer_time_ms(self.h, l, C.byref(v)))
        return v.value

    def layer_work(self, l, N):
        b, lk, m = C.c_double(), C.c_double(), C.c_double()
        _check(lib.qcnn_net_layer_work(self.h, l, N, C.byref(b), C.byref(lk), C.byref(m)))
        return dict(alg_bytes=b.value, lookups=lk.value, lut_macs=m.value)

    def launch_count(self):
        return lib.qcnn_net_launch_count(self.h)

    def pq_layer(self, l):
        h = lib.qcnn_net_pq_layer(self.h, l)
        return _Layer(self.ctx, _vp(h), owned=False) if h else None


class Preproc(object):
    """BmpImgIO on the device (ReszImg, RmMeanImg, CropImg of decoded BMP pixels), qcnn_preproc_*."""

    def __init__(self, ctx, mean_chw, hei_full=256, wid_full=256, hei_crop=227, wid_crop=227, resz_type=0, mean_type=0):
        m = _np(mean_chw, np.float32)
        assert m.ndim == 3 and m.shape[0] == 3
        h = _vp()
        _check(lib.qcnn_preproc_create(ctx.h, resz_type, mean_type, hei_full, wid_full, hei_crop, wid_crop,
                                       m.ctypes.data_as(_vp), m.shape[1], m.shape[2], C.byref(h)))
        self.h, self.ctx, self.crop = h, ctx, (hei_crop, wid_crop)

    def close(self):
        if self.h:
            lib.qcnn_preproc_destroy(self.h)
            self.h = None

    def run(self, images, stream=None):
        """images: list of uint8 numpy arrays [H,W,3] (B,G,R interleaved, top row first); returns CUDA f32 [N,3,hc,wc]."""
        import torch
        N = len(images)
        offs, total = [], 0
        for im in images:
            offs.append(total)
            total += im.size
        flat = np.concatenate([np.ascontiguousarray(im, np.uint8).reshape(-1) for im in images])
        pix = torch.from_numpy(flat).to("cuda:%d" % self.ctx.device)
        out = torch.empty((N, 3) + self.crop, dtype=torch.float32, device=pix.device)
        off = (C.c_longlong * N)(*offs)
        hei = (_i * N)(*[im.shape[0] for im in images])
        wid = (_i * N)(*[im.shape[1] for im in images])
        _check(lib.qcnn_preproc_run(self.h, C.c_void_p(pix.data_ptr()), off, hei, wid, N, _dptr(out), _stream(stream)))
        return out


class MultiNet(object):
    """One process, several GPUs: batch-sharded replicas + NCCL all-gather of the probabilities (qcnn_multi_*)."""

    def __init__(self, dirpath, pfx, model="AlexNet", devices=(0,)):
        devices = list(devices)
        arr = (_i * len(devices))(*devices)
        h = _vp()
        _check(lib.qcnn_multi_create(len(devices), arr, model.encode(), dirpath.encode(), pfx.encode(), C.byref(h)))
        self.h, self.devices = h, devices
        self.out_len = lib.qcnn_multi_out_len(h)

    def close(self):
        if self.h:
            lib.qcnn_multi_destroy(self.h)
            self.h = None

    @property
    def nccl_version(self):
        return lib.qcnn_multi_nccl_version(self.h)

    def pq_layer(self, rank, l):
        net = lib.qcnn_multi_net(self.h, rank)
        h = lib.qcnn_net_pq_layer(net, l)
        return _Layer(None, _vp(h), owned=False) if h else None

    def forward_host(self, img_h, prob_h=None):
        def ptr(a):
            return C.c_void_p(a.data_ptr()) if hasattr(a, "data_ptr") else a.ctypes.data_as(_vp)
        N = img_h.shape[0]
        if prob_h is None:
            prob_h = np.empty((N, self.out_len), np.float32)
        _check(lib.qcnn_multi_forward_h(self.h, ptr(img_h), N, ptr(prob_h)))
        return prob_h

    def shard(self, N, r):
        per = -(-N // len(self.devices))
        return min(N, r * per), min(N, (r + 1) * per)

    def forward(self, shards, N):
        """shards[r]: CUDA float32 tensor on device r with rank r's images; returns device pointers of the gathered probs."""
        R = len(self.devices)
        ins = (_vp * R)(*[(_dptr(t).value if t is not None else None) for t in shards])
        outs = (_vp * R)()
        _check(lib.qcnn_multi_forward(self.h, ins, N, outs))
        return [outs[r] for r in range(R)]

    def sync(self):
        _check(lib.qcnn_multi_sync(self.h))

    def gathered(self, ptr, N, rank):
        """torch view [N, out_len] of a gathered buffer returned by forward() (after sync)."""
        import torch

        class _View(object):
            pass
        v = _View()
        v.__cuda_array_interface__ = dict(shape=(N, self.out_len), typestr="<f4", data=(int(ptr), False), version=2)
        return torch.as_tensor(v, device="cuda:%d" % self.devices[rank])


# ---- file formats (host) ----------------------------------------------------------------------------------
def read_bin_f32(path):
    dc, dims = _i(), (_i * 4)()
    n = lib.qcnn_read_bin_f32(path.encode(), C.byref(dc), dims, None, 0)
    if n < 0:
        raise QcnnError(last_error())
    out = np.empty(n, np.float32)
    lib.qcnn_read_bin_f32(path.encode(), C.byref(dc), dims, out.ctypes.data_as(_vp), n)
    return out.reshape([dims[k] for k in range(dc.value)])


def write_bin_f32(path, arr):
    arr = _np(arr, np.float32)
    dims = (_i * arr.ndim)(*arr.shape)
    _check(lib.qcnn_write_bin_f32(path.encode(), arr.ndim, dims, arr.ctypes.data_as(_vp)))


def read_cbn_u8(path):
    dc, dims, bits = _i(), (_i * 4)(), _i()
    n = lib.qcnn_read_cbn_u8(path.encode(), C.byref(dc), dims, C.byref(bits), None, 0)
    if n < 0:
        raise QcnnError(last_error())
    out = np.empty(n, np.uint8)
    lib.qcnn_read_cbn_u8(path.encode(), C.byref(dc), dims, C.byref(bits), out.ctypes.data_as(_vp), n)
    return out.reshape([dims[k] for k in range(dc.value)]), bits.value


def write_cbn_u8(path, idx0, bits):
    idx0 = _np(idx0, np.uint8)
    dims = (_i * idx0.ndim)(*idx0.shape)
    _check(lib.qcnn_write_cbn_u8(path.encode(), idx0.ndim, dims, idx0.ctypes.data_as(_vp), bits))


# ---- product quantization of dense weights (k-means on the device, DESIGN.md 4e) -----------------------------------
def _pq_quantize(fn, ctx, w, shape_args, Cg, K, d, iters, seed, init, asmt_shape):
    S = -(-Cg // d)
    init_p = None
    if init is not None:
        init = _np(init, np.float32)
        if init.shape != (S, K, d):
            raise QcnnError("init codebook must be [%d, %d, %d], got %s" % (S, K, d, init.shape))
        init_p = init.ctypes.data_as(_vp)
    ctrd = np.empty((S, K, d), np.float32)
    asmt = np.empty(asmt_shape + (S,), np.uint8)
    sse = np.empty(max(iters, 0) + 1, np.float64)
    _check(fn(ctx.h, *shape_args, K, d, iters, seed & 0xFFFFFFFF, w.ctypes.data_as(_vp), init_p,
              ctrd.ctypes.data_as(_vp), asmt.ctypes.data_as(_vp), sse.ctypes.data_as(_vp)))
    return ctrd, asmt, sse


def pq_quantize_conv(ctx, knl, K, d, iters=20, seed=0, init=None):
    """k-means PQ of conv weights knl [Cout, Cg, k, k]: (ctrd [S, K, d], asmt [Cout, k, k, S] 0-based, sse [iters + 1])."""
    knl = _np(knl, np.float32)
    Cout, Cg, k, k2 = knl.shape
    assert k == k2, knl.shape
    return _pq_quantize(lib.qcnn_pq_quantize_conv, ctx, knl, (Cout, Cg, k), Cg, K, d, iters, seed, init, (Cout, k, k))


def pq_quantize_fc(ctx, wei, K, d, iters=20, seed=0, init=None):
    """k-means PQ of FC weights wei [Dout, Din]: (ctrd [S, K, d], asmt [Dout, S] 0-based, sse [iters + 1])."""
    wei = _np(wei, np.float32)
    Dout, Din = wei.shape
    return _pq_quantize(lib.qcnn_pq_quantize_fc, ctx, wei, (Din, Dout), Din, K, d, iters, seed, init, (Dout,))


def pq_quantize_model(ctx, model, dir, pfx, out_dir, out_pfx, pq, iters=20, seed=0):
    """Dense <dir>/<pfx>.{convKnl|fcntWei,biasVec}.NN.bin of a model table -> PQ files under <out_dir>/<out_pfx>;
    pq = {layerInd: (K, d)} for every conv / FC layer (layer l is seeded with seed + 65536 (l + 1))."""
    n = max(pq) + 1 if pq else 0
    n = max(n, 256)   # one entry per layer index of the table: unlisted layers are 0, which the call rejects
    Ks, ds = (_i * n)(), (_i * n)()
    for l, (K, d) in pq.items():
        Ks[l], ds[l] = K, d
    _check(lib.qcnn_pq_quantize_model(ctx.h, model.encode(), dir.encode(), pfx.encode(), Ks, ds, iters,
                                      seed & 0xFFFFFFFF, out_dir.encode(), out_pfx.encode()))


def _refine_start(ctrd, asmt):
    """Fresh C-ordered copies of a refine call's start (ctrd float32, asmt uint8), which the call overwrites."""
    return np.array(ctrd, np.float32, order="C", copy=True), np.array(asmt, np.uint8, order="C", copy=True)


def _refine_call(fn, args, ctrd, asmt, sweeps, stream):
    """fn(*args, ctrd, asmt, loss, stream) with loss [sweeps + 1]: (ctrd, asmt, loss)."""
    loss = np.empty(max(sweeps, 0) + 1, np.float64)
    _check(fn(*args, ctrd.ctypes.data_as(_vp), asmt.ctypes.data_as(_vp), loss.ctypes.data_as(_vp), _stream(stream)))
    return ctrd, asmt, loss


def pq_refine_fc(ctx, wei, x, ctrd, asmt, sweeps=8, stream=None):
    """Error-correcting PQ of FC weights wei [Dout, Din] on layer inputs x (contiguous float32 CUDA tensor [N, Din],
    fcntWei column order), starting from (ctrd [S, K, d], asmt [Dout, S] 0-based), e.g. pq_quantize_fc's output:
    (ctrd, asmt, loss [sweeps + 1]) with loss[t] = sum_n |(W - W^) x_n|^2 after sweep t.  The arguments are not modified."""
    wei = _np(wei, np.float32)
    Dout, Din = wei.shape
    ctrd, asmt = _refine_start(ctrd, asmt)
    S, K, d = ctrd.shape
    if S != -(-Din // d) or asmt.shape != (Dout, S):
        raise QcnnError("ctrd [%d, K, d] and asmt [%d, %d] do not match a [%d, %d] layer with d=%d"
                        % (S, Dout, S, Dout, Din, d))
    if x.dim() != 2 or x.shape[1] != Din:
        raise QcnnError("x must be [N, %d], got %s" % (Din, tuple(x.shape)))
    return _refine_call(lib.qcnn_pq_refine_fc, (ctx.h, Din, Dout, K, d, sweeps, wei.ctypes.data_as(_vp), _dptr(x), x.shape[0]),
                        ctrd, asmt, sweeps, stream)


def pq_refine_conv(ctx, knl, x, ctrd, asmt, pad=0, stride=1, grp=1, sweeps=8, stream=None):
    """Error-correcting PQ of conv weights knl [Cout, Cin / grp, k, k] on layer inputs x (contiguous float32 CUDA tensor
    [N, Hin, Win, Cin], NHWC as Net.featmap returns it), starting from (ctrd [S, K, d], asmt [Cout, k, k, S] 0-based),
    e.g. pq_quantize_conv's output: (ctrd, asmt, loss [sweeps + 1]) with loss[t] = sum conv(x, W - W^)^2 after sweep t.
    The arguments are not modified."""
    knl = _np(knl, np.float32)
    Cout, Cg, k, k2 = knl.shape
    ctrd, asmt = _refine_start(ctrd, asmt)
    S, K, d = ctrd.shape
    if k != k2 or S != -(-Cg // d) or asmt.shape != (Cout, k, k, S):
        raise QcnnError("ctrd [%d, K, d] and asmt %s do not match a %s kernel with d=%d"
                        % (S, tuple(asmt.shape), tuple(knl.shape), d))
    if x.dim() != 4 or x.shape[3] != Cg * grp:
        raise QcnnError("x must be [N, Hin, Win, %d], got %s" % (Cg * grp, tuple(x.shape)))
    N, Hin, Win, Cin = x.shape
    return _refine_call(lib.qcnn_pq_refine_conv, (ctx.h, Cin, Hin, Win, Cout, k, pad, stride, grp, K, d, sweeps,
                                                  knl.ctypes.data_as(_vp), _dptr(x), N), ctrd, asmt, sweeps, stream)


def pq_refine_fc_target(ctx, y, t, ctrd, asmt, sweeps=8, stream=None):
    """Error-correcting PQ of an FC layer toward target responses: y [N, Din] are the layer's inputs in the quantized
    network and t [N, Dout] the original layer's responses without bias and before ReLU (both contiguous float32 CUDA
    tensors, y in fcntWei column order), starting from (ctrd [S, K, d], asmt [Dout, S] 0-based): (ctrd, asmt,
    loss [sweeps + 1]) with loss[s] = sum_n |t_n - W^ y_n|^2 after sweep s.  The arguments are not modified."""
    ctrd, asmt = _refine_start(ctrd, asmt)
    S, K, d = ctrd.shape
    if y.dim() != 2 or t.dim() != 2 or t.shape[0] != y.shape[0]:
        raise QcnnError("y must be [N, Din] and t [N, Dout] with the same N, got %s and %s"
                        % (tuple(y.shape), tuple(t.shape)))
    N, Din = y.shape
    Dout = t.shape[1]
    if S != -(-Din // d) or asmt.shape != (Dout, S):
        raise QcnnError("ctrd [%d, K, d] and asmt %s do not match a [%d, %d] layer with d=%d"
                        % (S, tuple(asmt.shape), Dout, Din, d))
    return _refine_call(lib.qcnn_pq_refine_fc_target, (ctx.h, Din, Dout, K, d, sweeps, _dptr(y), _dptr(t), N), ctrd, asmt,
                        sweeps, stream)


def pq_refine_conv_target(ctx, y, t, ctrd, asmt, ksz, pad=0, stride=1, grp=1, sweeps=8, stream=None):
    """Error-correcting PQ of a conv layer toward target responses: y [N, Hin, Win, Cin] are the layer's inputs in the
    quantized network and t [N, Ho, Wo, Cout] the original layer's responses without bias and before ReLU (both NHWC,
    contiguous float32 CUDA tensors), starting from (ctrd [S, K, d], asmt [Cout, ksz, ksz, S] 0-based): (ctrd, asmt,
    loss [sweeps + 1]) with loss[s] = sum (t - conv(y, W^))^2 after sweep s.  The arguments are not modified."""
    ctrd, asmt = _refine_start(ctrd, asmt)
    S, K, d = ctrd.shape
    if y.dim() != 4 or t.dim() != 4 or t.shape[0] != y.shape[0]:
        raise QcnnError("y must be [N, Hin, Win, Cin] and t [N, Ho, Wo, Cout] with the same N, got %s and %s"
                        % (tuple(y.shape), tuple(t.shape)))
    N, Hin, Win, Cin = y.shape
    Cout = t.shape[3]
    # a geometry the call refuses (grp not dividing Cin, an empty output, ...) is left to its own message
    if ksz >= 1 and stride >= 1 and grp >= 1 and Cin % grp == 0 and Hin + 2 * pad >= ksz and Win + 2 * pad >= ksz:
        Ho, Wo = (Hin + 2 * pad - ksz) // stride + 1, (Win + 2 * pad - ksz) // stride + 1
        if tuple(t.shape) != (N, Ho, Wo, Cout):
            raise QcnnError("t must be [%d, %d, %d, Cout] for a %dx%d kernel, pad %d, stride %d on %s, got %s"
                            % (N, Ho, Wo, ksz, ksz, pad, stride, tuple(y.shape), tuple(t.shape)))
        if S != -(-(Cin // grp) // d) or asmt.shape != (Cout, ksz, ksz, S):
            raise QcnnError("ctrd [%d, K, d] and asmt %s do not match a [%d, %d, %d, %d] kernel with d=%d"
                            % (S, tuple(asmt.shape), Cout, Cin // grp, ksz, ksz, d))
    return _refine_call(lib.qcnn_pq_refine_conv_target, (ctx.h, Cin, Hin, Win, Cout, ksz, pad, stride, grp, K, d, sweeps,
                                                         _dptr(y), _dptr(t), N), ctrd, asmt, sweeps, stream)


_ABSENT = object()   # PqStats._refine: an argument the call does not take


class PqStats(object):
    """Calibration statistics of one layer for one subspace width d (include/qcnn.h, DESIGN.md 4e): add() folds a batch
    of layer inputs y (and, with target=True, the original layer's responses t) into the sums the error-correcting
    refinement reads, so the calibration set can be streamed in batches; refine() / refine_target() then run the sweeps
    of pq_refine_* / pq_refine_*_target on the sums, any number of times; refine_bias() / refine_target_bias() also
    refit the layer's bias, from the first moments read_sums() returns; refine_damped() runs either form, with or
    without the bias, damped toward the dense weights.  Device memory does not grow with the number of images."""

    def __init__(self, ctx, h, conv, shape, target):
        self.ctx, self.h, self.conv, self.target = ctx, h, conv, target
        # d, the sums' dims (G [grp, Dg, Dg], P [outputs, Dg]), and the shapes add() and the refines check: y and t
        # without N, wei, asmt
        self._shape = shape
        self._groups = (shape["grp"],) if conv else ()   # FC: G [Din, Din] and s [Din]

    @classmethod
    def fc(cls, ctx, Din, Dout, d, target=False):
        h = _vp()
        _check(lib.qcnn_pq_stats_create_fc(ctx.h, Din, Dout, d, int(bool(target)), C.byref(h)))
        return cls(ctx, h, False, dict(d=d, grp=1, Dg=Din, outputs=Dout, y=(Din,), t=(Dout,), wei=(Dout, Din),
                                       asmt=(Dout, -(-Din // d))), bool(target))

    @classmethod
    def conv(cls, ctx, Cin, Hin, Win, Cout, ksz, d, pad=0, stride=1, grp=1, target=False):
        h = _vp()
        _check(lib.qcnn_pq_stats_create_conv(ctx.h, Cin, Hin, Win, Cout, ksz, pad, stride, grp, d, int(bool(target)),
                                             C.byref(h)))
        Ho, Wo = (Hin + 2 * pad - ksz) // stride + 1, (Win + 2 * pad - ksz) // stride + 1
        Cg = Cin // grp
        return cls(ctx, h, True, dict(d=d, grp=grp, Dg=Cg * ksz * ksz, outputs=Cout, y=(Hin, Win, Cin), t=(Ho, Wo, Cout),
                                      wei=(Cout, Cg, ksz, ksz), asmt=(Cout, ksz, ksz, -(-Cg // d))), bool(target))

    def _live(self):
        if not self.h:
            raise QcnnError("PqStats: closed")

    def add(self, y, t=None, stream=None):
        """Fold a batch: y [N, Din] (FC) or [N, Hin, Win, Cin] (NHWC conv), t [N, Dout] or [N, Ho, Wo, Cout] for a
        target object, contiguous float32 CUDA tensors that must stay alive until the stream has run the add."""
        self._live()
        N = y.shape[0] if y.dim() >= 1 else 0
        want_y = (N,) + self._shape["y"]
        if tuple(y.shape) != want_y:
            raise QcnnError("y must be %s, got %s" % (want_y, tuple(y.shape)))
        if t is not None:
            want_t = (N,) + self._shape["t"]
            if tuple(t.shape) != want_t:
                raise QcnnError("t must be %s, got %s" % (want_t, tuple(t.shape)))
        _check(lib.qcnn_pq_stats_add(self.h, _dptr(y), None if t is None else _dptr(t), N, _stream(stream)))

    @property
    def count(self):
        """images added so far"""
        self._live()
        n = C.c_longlong()
        _check(lib.qcnn_pq_stats_count(self.h, C.byref(n)))
        return n.value

    def read(self):
        """(G, P, tt): G [grp, Dg, Dg] conv / [Din, Din] FC in the internal dim order, and for a target object
        P [Cout, Dg] / [Dout, Din] and |T|^2 (else None, None), as float64 host arrays."""
        self._live()
        Dg, outputs = self._shape["Dg"], self._shape["outputs"]
        G = np.empty(self._groups + (Dg, Dg), np.float64)
        P = np.empty((outputs, Dg), np.float64) if self.target else None
        tt = np.empty(1, np.float64) if self.target else None
        _check(lib.qcnn_pq_stats_read_h(self.h, G.ctypes.data_as(_vp), None if P is None else P.ctypes.data_as(_vp),
                                        None if tt is None else tt.ctypes.data_as(_vp)))
        return G, P, None if tt is None else float(tt[0])

    def read_sums(self):
        """(s, u, n): the sum of y, s [grp, Dg] conv (internal dim order) / [Din] FC, the sum of t, u [Cout] / [Dout]
        for a target object (else None), as float64 host arrays, and n, the rows summed (images, conv images Ho Wo)."""
        self._live()
        sy = np.empty(self._groups + (self._shape["Dg"],), np.float64)
        u = np.empty(self._shape["outputs"], np.float64) if self.target else None
        n = C.c_longlong()
        _check(lib.qcnn_pq_stats_read_sums_h(self.h, sy.ctypes.data_as(_vp), None if u is None else u.ctypes.data_as(_vp),
                                             C.byref(n)))
        return sy, u, n.value

    def _start(self, ctrd, asmt):
        ctrd, asmt = _refine_start(ctrd, asmt)
        g = self._shape
        S, K, d = ctrd.shape if ctrd.ndim == 3 else (0, 0, 0)
        want = g["asmt"]
        if not (d == g["d"] and S == want[-1] and asmt.shape == want):
            raise QcnnError("ctrd [%d, K, %d] and asmt %s must be [S, K, d] and %s" % (S, g["d"], tuple(asmt.shape), want))
        return ctrd, asmt, K

    def _refine(self, fn, ctrd, asmt, sweeps, stream, wei=_ABSENT, bias=_ABSENT, lead=()):
        """fn(h, *lead, K, sweeps, ...) on the statistics from the start (ctrd, asmt), with the dense weights and the
        bias when the call takes them (bias None: a NULL bias): (ctrd, asmt, loss), or (ctrd, asmt, bias, loss) with a
        bias."""
        self._live()
        ctrd, asmt, K = self._start(ctrd, asmt)
        args = []
        if wei is not _ABSENT:
            wei = _np(wei, np.float32)
            if wei.shape != self._shape["wei"]:
                raise QcnnError("wei must be %s, got %s" % (self._shape["wei"], wei.shape))
            args.append(wei.ctypes.data_as(_vp))
        args += [ctrd.ctypes.data_as(_vp), asmt.ctypes.data_as(_vp)]
        if bias is None:
            args.append(None)
        elif bias is not _ABSENT:
            bias = np.array(bias, np.float32, order="C", copy=True)
            if bias.shape != (self._shape["outputs"],):
                raise QcnnError("bias must be (%d,), got %s" % (self._shape["outputs"], bias.shape))
            args.append(bias.ctypes.data_as(_vp))
        loss = np.empty(max(sweeps, 0) + 1, np.float64)
        _check(fn(self.h, *lead, K, sweeps, *args, loss.ctypes.data_as(_vp), _stream(stream)))
        return (ctrd, asmt, loss) if bias is _ABSENT or bias is None else (ctrd, asmt, bias, loss)

    def refine(self, wei, ctrd, asmt, sweeps=8, stream=None):
        """The same-input sweeps (pq_refine_fc / pq_refine_conv) on the statistics and the dense weights wei
        [Dout, Din] / [Cout, Cin / grp, k, k]: (ctrd, asmt, loss [sweeps + 1]).  The arguments are not modified."""
        return self._refine(lib.qcnn_pq_stats_refine, ctrd, asmt, sweeps, stream, wei=wei)

    def refine_target(self, ctrd, asmt, sweeps=8, stream=None):
        """The target sweeps (pq_refine_*_target) on the statistics of a target object: (ctrd, asmt, loss [sweeps + 1]).
        The arguments are not modified."""
        return self._refine(lib.qcnn_pq_stats_refine_target, ctrd, asmt, sweeps, stream)

    def refine_bias(self, wei, ctrd, asmt, bias, sweeps=8, stream=None):
        """refine() with the bias free as well: the sweeps on the centered sums, then the bias refit (include/qcnn.h).
        bias [Dout] / [Cout] is the layer's bias.  Returns (ctrd, asmt, bias, loss [sweeps + 1]), loss the bias-optimal
        one; the arguments are not modified."""
        return self._refine(lib.qcnn_pq_stats_refine_bias, ctrd, asmt, sweeps, stream, wei=wei, bias=bias)

    def refine_target_bias(self, ctrd, asmt, bias, sweeps=8, stream=None):
        """refine_target() with the bias free as well: (ctrd, asmt, bias, loss [sweeps + 1]).  The arguments are not
        modified."""
        return self._refine(lib.qcnn_pq_stats_refine_target_bias, ctrd, asmt, sweeps, stream, bias=bias)

    def refine_damped(self, wei, ctrd, asmt, damp, target=False, bias=None, sweeps=8, stream=None):
        """refine() (target=False) or refine_target() (target=True, a target object) with a damping term that pulls the
        fit toward the dense weights wei: the loss plus lambda_g |W_g - W^_g|^2 per group, lambda_g = damp tr(G_g) / Dg
        (include/qcnn.h).  With bias [Dout] / [Cout] the bias is refit as by refine_bias() / refine_target_bias().
        Returns (ctrd, asmt, loss [sweeps + 1]), or (ctrd, asmt, bias, loss) with a bias, loss the damped objective;
        damp = 0 gives the undamped call's bits.  The arguments are not modified."""
        return self._refine(lib.qcnn_pq_stats_refine_damped, ctrd, asmt, sweeps, stream, wei=wei, bias=bias,
                            lead=(int(bool(target)), float(damp)))

    @property
    def nbytes(self):
        """device bytes of the sums (G and s, and for a target object P, |T|^2 and u)"""
        g = self._shape
        return 8 * (g["grp"] * g["Dg"] * (g["Dg"] + 1) + ((g["Dg"] + 1) * g["outputs"] + 1 if self.target else 0))

    def close(self):
        if self.h:
            lib.qcnn_pq_stats_destroy(self.h)
            self.h = None
