"""CPU tests of the INT8 heads' host side: weight quantisation, the max / entropy threshold search, calibration tables, and
the accuracy of the INT8-emulating oracle heads against the fp32 oracle (the bar the GPU match-rate test derives from)."""
import json

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import int8_oracle
from oracle import model_ref
from retinanet_examples_b200 import calib, engine
from retinanet_examples_b200.model import make_state_dict


def test_weight_quantisation_per_channel_with_zero_channel():
    g = torch.Generator().manual_seed(0)
    w = torch.randn((5, 128, 3, 3), generator=g) * 0.02
    w[2] = 0.0
    w[4, 7, 1, 1] = 0.5                                         # one large weight sets its channel's scale
    q, s_w = engine.pack_weight_s8(w)
    assert q.dtype == torch.int8 and q.shape == (5, 9 * 128) and s_w.dtype == torch.float32
    assert float(s_w[2]) == 1.0 and int(q[2].abs().max()) == 0
    for c in (0, 1, 3, 4):
        assert float(s_w[c]) == float(torch.tensor(float(w[c].abs().max())) / 127.0)
        assert int(q[c].abs().max()) == 127
    # tap-major, channel-minor K order (engine.pack_weight) and round-half-even of W / s_w
    ref = torch.round(w / s_w.view(-1, 1, 1, 1)).clamp(-127, 127).permute(0, 2, 3, 1).reshape(5, -1)
    assert torch.equal(q.float(), ref)
    assert int(q[4].reshape(3, 3, 128)[1, 1, 7]) == 127
    # dequantised weights are within half a step of the fp32 weights
    err = (q.float() * s_w.view(-1, 1) - w.permute(0, 2, 3, 1).reshape(5, -1)).abs()
    assert bool((err <= s_w.view(-1, 1) / 2 + 1e-9).all())


def _gauss_hist(absmax, n=200000, sigma=1.0, outlier=None):
    x = np.abs(np.random.default_rng(0).normal(0, sigma, n))
    if outlier is not None:
        x = np.append(x, outlier)
    top = x.max() if absmax is None else absmax
    h, _ = np.histogram(x, bins=calib.NBINS, range=(0, top))
    return h.astype(np.float64), float(top)


def test_max_and_entropy_thresholds():
    # a far outlier: max keeps it (threshold = absmax), entropy clips it close to the bulk of the distribution
    h, top = _gauss_hist(None, outlier=100.0)
    assert top == 100.0
    assert calib.max_threshold(top) == 100.0
    t = calib.entropy_threshold(h, top)
    assert 2.0 < t < 10.0, t
    # no outlier: the threshold stays near the tail, never above absmax
    h, top = _gauss_hist(None)
    t = calib.entropy_threshold(h, top)
    assert 0.5 * top < t <= top, (t, top)
    # a uniform histogram needs no clipping
    t = calib.entropy_threshold(np.ones(calib.NBINS), 3.0)
    assert t == 3.0
    assert calib.entropy_threshold(np.zeros(calib.NBINS), 0.0) == 0.0
    assert calib.scale_from_threshold(0.0) == 1.0
    assert calib.scale_from_threshold(127.0) == 1.0


def test_collector_two_passes():
    col = calib.Collector()
    x = torch.randn(1000, generator=torch.Generator().manual_seed(1))
    for phase in (0, 1):
        col.phase = phase
        for n in calib.TENSORS:
            col.observe(n, x)
    assert col.absmax["heads.input"] == float(x.abs().max())
    assert col.hist["heads.input"].sum() == 1000
    sm, se = col.scales("max"), col.scales("entropy")
    assert set(sm) == set(se) == set(calib.TENSORS)
    assert all(0 < se[n] <= sm[n] for n in calib.TENSORS)
    with pytest.raises(ValueError):
        col.scales("percentile")


def test_table_write_read_and_mismatch(tmp_path):
    scales = {n: 0.01 * (i + 1) for i, n in enumerate(calib.TENSORS)}
    t = calib.make_table("ResNet18FPN", 6, 9, "entropy", 8, scales)
    p = str(tmp_path / "table.json")
    calib.save_table(t, p)
    back = calib.load_table(p)
    assert back == t and json.load(open(p))["format"] == 1
    assert calib.check_table(back, "ResNet18FPN", 6, 9) is back
    for args in (("ResNet50FPN", 6, 9), ("ResNet18FPN", 80, 9), ("ResNet18FPN", 6, 27)):
        with pytest.raises(ValueError):
            calib.check_table(back, *args)
    broken = dict(t, scales=dict(scales))
    del broken["scales"]["box_head.4"]
    with pytest.raises(ValueError):
        calib.check_table(broken, "ResNet18FPN", 6, 9)
    with pytest.raises(ValueError):
        calib.check_table(dict(t, format=2), "ResNet18FPN", 6, 9)
    # fp32 epilogue constants: alpha = s_in * s_w, inv_out = 1 / s_out, layer by layer
    ls = calib.layer_scales(scales, "box_head")
    assert ls[0][0] == np.float32(scales["heads.input"]) and ls[0][1] == np.float32(1) / np.float32(scales["box_head.0"])
    assert ls[4] == (np.float32(scales["box_head.6"]), None)


def _oracle_scales(sd, feats, method="entropy"):
    """CPU calibration on the oracle: the fp16-emulated heads' input and tower outputs, all pixels of every level."""
    col = calib.Collector()
    for phase in (0, 1):
        col.phase = phase
        for head in calib.HEADS:
            for f in feats:
                if head == "cls_head":
                    col.observe("heads.input", f)
                t = f
                for i in calib.TOWER:
                    t = model_ref._q(F.relu(model_ref._cb(sd, "%s.%d" % (head, i), None, t, 1, 1, True)), True)
                    col.observe("%s.%d" % (head, i), t)
    return col.scales(method)


def test_int8_oracle_heads_sqnr_vs_fp32():
    """SQNR of the INT8-emulating heads against the all-fp32 oracle heads (ResNet18FPN, 2 x 3 x 256 x 384, entropy
    calibration on the same batch), per head, over all five levels, of the convolution part of the logits (the final
    layer's bias, which no quantisation touches, is left out of both).  Measured: cls 29.9 dB, box 30.4 dB (max
    calibration: 29.8 / 30.3 dB); asserted with 3 dB of margin."""
    backbone, classes = "ResNet18FPN", 6
    sd = {k: v.float() for k, v in make_state_dict(backbone, classes, 9, False, 3).items()}
    x = torch.randn((2, 3, 256, 384), generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        feats = model_ref.features(sd, backbone, x, True)
        scales = _oracle_scales(sd, feats)
        rc, rb = model_ref.forward_heads(sd, backbone, x, sigmoid=False)
        qc, qb = int8_oracle.forward_heads(sd, backbone, x, scales, sigmoid=False)
    for name, ref, got in (("cls", rc, qc), ("box", rb, qb)):
        b = sd["%s_head.8.bias" % name].view(1, -1, 1, 1)
        sig = sum(float(((r - b) ** 2).sum()) for r in ref)
        noise = sum(float(((g - r) ** 2).sum()) for g, r in zip(got, ref))
        sqnr = 10 * np.log10(sig / noise)
        assert sqnr > 27.0, (name, sqnr)
