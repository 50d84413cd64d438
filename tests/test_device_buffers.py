"""Device memory has one owner: qcnn::DeviceBuffer (csrc/qcnn_internal.h).

CPU: no file under csrc/ calls the CUDA allocator except the buffer type and the C ABI's qcnn_dev_alloc / qcnn_dev_free.
GPU: a reservation that fails leaves the buffer empty, not a stale capacity beside a null pointer, so the next call with
a batch that fits the old buffers reserves again instead of running on the null pointer."""
import ctypes as C
import glob
import os
import re

import numpy as np
import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "quantized-cnn_b200", "csrc")
ALLOC = re.compile(r"\bcuda(?:Malloc|Free)\w*")


def _strip_comments_and_strings(src):
    pat = re.compile(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])*\'', re.S)
    return pat.sub(lambda m: " " if m.group(0)[0] in "/" else '""', src)


def _cut_block(src, head):
    """src without the brace-delimited body that follows `head`, and that body."""
    i = src.index(head)
    j = src.index("{", i)
    depth = 0
    for k in range(j, len(src)):
        depth += {"{": 1, "}": -1}.get(src[k], 0)
        if depth == 0:
            return src[:i] + src[k + 1:], src[i:k + 1]
    raise AssertionError("unbalanced braces after %r" % head)


def test_only_the_buffer_type_calls_the_allocator():
    files = sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.h")))
    assert files
    owners = {}
    leftovers = []
    for f in files:
        src = _strip_comments_and_strings(open(f).read())
        for head in ("class DeviceBuffer", "int qcnn_dev_alloc(", "int qcnn_dev_free("):
            if head in src:
                src, body = _cut_block(src, head)
                owners[head] = body
        leftovers += ["%s: %s" % (os.path.basename(f), m.group(0)) for m in ALLOC.finditer(src)]
    assert not leftovers, "device allocations outside DeviceBuffer: %s" % leftovers
    # the owners are where the allocator is called
    assert "cudaMalloc(" in owners["class DeviceBuffer"] and "cudaFree(" in owners["class DeviceBuffer"]
    assert "cudaMalloc(" in owners["int qcnn_dev_alloc("]
    assert "cudaFree(" in owners["int qcnn_dev_free("]


@pytest.mark.gpu
def test_failed_output_growth_leaves_a_usable_net(po, qcnn, ctx, tmp_path):
    d = str(tmp_path)
    po.save_model(d, "synth", po.synth_alexnet(seed=1))
    net = qcnn.Net(ctx, d, "synth", "AlexNet")
    try:
        img = po.lcg_images(2, 777)
        first = net.forward_host(img)
        # 2^28 images: after the input staging of one 128-image chunk, the output reservation (about 1 TB) fails before
        # any host-to-device copy, so the two-image host buffers are never read past their end
        prob = np.empty((2, net.out_len), np.float32)
        rc = qcnn.lib.qcnn_net_forward_h(net.h, img.ctypes.data_as(C.c_void_p), 1 << 28, prob.ctypes.data_as(C.c_void_p), None)
        assert rc != 0
        assert "out of memory" in qcnn.last_error()
        again = net.forward_host(img)
        assert np.array_equal(again, first)
    finally:
        net.close()
