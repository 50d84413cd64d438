"""VGG16 (CaffePara's 39-layer table: thirteen 3x3 stride-1 convolutions, five 2x2 / 2 max-pools, fc6 over 7x7x512)
on the CPU: the compiled reference, built BY NAME (CaffeEva::SetModelName("VGG16")), against the CPU oracle driven by the
Python transcription of the table below, every feature map of one image bit for bit.  This pins both the oracle and the
transcription that tests/test_gpu_vgg16.py compares the GPU with.  No shipped VGG16 parameters exist: seeded synthetic
parameters in the reference's file formats stand in (He-scaled codebooks, as tests/test_gpu_models.py).  No GPU."""
import numpy as np
import pytest

VGG16_IN = (3, 224, 224)
# conv layer indices of the table (fc6, fc7, fc8 are 31, 34, 37)
VGG16_CONVS = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
VGG16_FC6 = 31


def vgg16_layers(po):
    """reference src/CaffePara.cc:121-169"""
    L = []
    for cnt, times in ((64, 2), (128, 2), (256, 3), (512, 3), (512, 3)):
        for _ in range(times):
            L += [po.conv(1, 3, cnt, 1, 1), po.relu()]
        L.append(po.pool(0, 2, 2))
    for _ in range(2):
        L += [po.fcnt(4096), po.relu(), po.drpt(0.5)]
    return L + [po.fcnt(1000), po.smax()]


def vgg16_pq(layers):
    """{layerInd: (S, K, d)}: conv1_1 one 4-wide subspace over its 3 channels, the other convolutions 8-wide subspaces,
    fc6 / fc7 4-wide with K = 32 and fc8 scalar with K = 16 (the shapes of the shipped AlexNet's FC files)."""
    pq, cin = {}, VGG16_IN[0]
    for l, L in enumerate(layers):
        if l in VGG16_CONVS:
            pq[l] = (1, 128, 4) if cin == 3 else (cin // 8, 128, 8)
            cin = L["cnt"]
    pq[31] = (7 * 7 * 512 // 4, 32, 4)
    pq[34] = (4096 // 4, 32, 4)
    pq[37] = (4096, 16, 1)
    return pq


def synth_vgg16(po, seed):
    layers = vgg16_layers(po)
    params = po.synth_model(layers, VGG16_IN, vgg16_pq(layers), seed=seed, ctrd_std=None, bias_std=0.05)
    # keep the logits well inside expf's range: the reference softmax does not subtract the maximum
    params[37]["ctrd"] = (params[37]["ctrd"] * np.float32(0.25)).astype(np.float32)
    return layers, params


def vgg16_images(n, seed):
    rng = np.random.RandomState(seed)
    return (rng.rand(n, *VGG16_IN) * 256 - 128).astype(np.float32)


def test_vgg16_table_shapes(po):
    layers = vgg16_layers(po)
    assert len(layers) == 39
    shapes = po.infer_shapes(layers, VGG16_IN)
    assert [i for i, L in enumerate(layers) if L["type"] == po.CONV] == list(VGG16_CONVS)
    assert tuple(shapes[VGG16_FC6]) == (7, 7, 512)
    assert tuple(shapes[2]) == (224, 224, 64) and tuple(shapes[-1]) == (1, 1, 1000)


def test_oracle_vgg16_matches_reference_by_name(po, tmp_path):
    if not po.have_ref():
        pytest.skip("compiled reference not built under oracle/_ref")
    layers, params = synth_vgg16(po, seed=16)
    d = str(tmp_path)
    po.save_model(d, "vgg", params)
    img = vgg16_images(1, 7)
    prob, maps = po.net_forward(layers, params, img, keep=True)
    assert np.isfinite(prob).all()
    net = po.RefNet(d, "vgg", model="VGG16")
    try:
        assert np.array_equal(net.forward(img[0]), prob[0])
        for l in range(len(layers) + 1):
            want = maps[l]
            if l == VGG16_FC6:    # the reference leaves fc6's input in NCHW order (as AlexNet's featMapLst[15])
                want = po.nhwc_to_nchw(want)
            assert np.array_equal(net.featmap(l).reshape(-1), want.reshape(-1)), l
    finally:
        net.close()
