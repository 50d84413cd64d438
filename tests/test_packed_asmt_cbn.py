"""The width of a packed FC assignment table (qcnn_layer_set_param "asmt_packed") is b = log2(K): for the shipped AlexNet
that is the width the reference itself stores each FC layer's indices at (the bit count in the .cbn header)."""
import os

import numpy as np
import pytest


def test_packed_width_matches_cbn_header(po, qcnn):
    if not po.have_alexnet():
        pytest.skip("shipped AlexNet parameters not staged under oracle/_ref/data")
    layers = po.alexnet_layers()
    params = po.load_model(po.ALEXNET_DIR, po.ALEXNET_PFX, layers)
    widths = []
    for l, p in sorted(params.items()):
        if p["asmt"].ndim != 2:        # FC tables are [Dout][S]
            continue
        _, hdr_bits = qcnn.read_cbn_u8(os.path.join(po.ALEXNET_DIR, "%s.asmtLst.%02d.cbn" % (po.ALEXNET_PFX, l + 1)))
        K = p["ctrd"].shape[1]
        assert hdr_bits == int(np.log2(K)), (l, hdr_bits, K)
        widths.append(hdr_bits)
    assert widths == [5, 5, 4]         # fc6, fc7 (K = 32), fc8 (K = 16)
