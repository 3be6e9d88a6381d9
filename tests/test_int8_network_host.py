"""CPU tests of the INT8 network scope's host side: format-2 calibration tables, the list of tensors the scope quantises,
and the accuracy of the network oracle (tests/int8_network_oracle.py) against the fp32 oracle and the fp16 oracle's
detections -- the bars the GPU tests derive from."""
import numpy as np
import pytest
import torch

import int8_network_oracle as net_oracle
import int8_oracle
from oracle import model_ref
from retinanet_examples_b200 import calib
from retinanet_examples_b200.model import make_state_dict


def _scales(backbone):
    return {n: 0.01 * (i + 1) for i, n in enumerate(calib.table_tensors(backbone, "network"))}


def test_network_table_round_trip_format1_compat_and_rejections(tmp_path):
    t = calib.make_table("ResNet18FPN", 6, 9, "entropy", 8, _scales("ResNet18FPN"), scope="network")
    assert t["format"] == 2 and t["scope"] == "network"
    assert set(t["scales"]) == set(calib.TENSORS) | set(calib.network_tensors("ResNet18FPN"))
    p = str(tmp_path / "net.json")
    calib.save_table(t, p)
    back = calib.load_table(p)
    assert back == t
    for scope in ("heads", "network"):                       # a network table also serves the heads scope
        assert calib.check_table(back, "ResNet18FPN", 6, 9, scope) is back
    heads = calib.make_table("ResNet18FPN", 6, 9, "entropy", 8, _scales("ResNet18FPN"))
    assert heads["format"] == 1 and "scope" not in heads and set(heads["scales"]) == set(calib.TENSORS)
    assert calib.check_table(heads, "ResNet18FPN", 6, 9) is heads
    with pytest.raises(ValueError):
        calib.check_table(heads, "ResNet18FPN", 6, 9, "network")
    for args in (("ResNet50FPN", 6, 9), ("ResNet18FPN", 80, 9), ("ResNet18FPN", 6, 27)):
        for scope in ("heads", "network"):
            with pytest.raises(ValueError):
                calib.check_table(back, *args, scope)
    broken = dict(t, scales=dict(t["scales"]))
    del broken["scales"]["backbones.ResNet18FPN.features.layer3.1.conv1"]
    with pytest.raises(ValueError):
        calib.check_table(broken, "ResNet18FPN", 6, 9, "network")
    with pytest.raises(ValueError):
        calib.check_table(dict(t, scope="heads"), "ResNet18FPN", 6, 9)
    with pytest.raises(ValueError):
        calib.check_table(t, "ResNet18FPN", 6, 9, "backbone")


@pytest.mark.parametrize("backbone,count", [("ResNet18FPN", 14), ("ResNet34FPN", 24), ("ResNet50FPN", 33),
                                            ("ResNet101FPN", 84), ("ResNet152FPN", 123)])
def test_network_tensors_every_s8_tensor_once(backbone, count):
    """C3; per layer3 / layer4 block the ReLU outputs of its convolutions but the last, the downsample output (first
    block) and the block output; P5 / P4 / P3 -- named by state_dict prefix, each exactly once, and exactly what the fp16
    oracle records."""
    names = calib.network_tensors(backbone)
    assert len(names) == len(set(names)) == count
    f = "backbones.%s.features." % backbone
    assert names[0] == f + "layer2" and names[-3:] == ["backbones.%s.lateral%d" % (backbone, k) for k in (5, 4, 3)]
    assert f + "layer3.0.downsample" in names and f + "layer3.1.downsample" not in names
    keys = make_state_dict(backbone, 2, 9, False, 0).keys()
    for n in names:
        assert any(k.startswith(n + ".") for k in keys), n
    if backbone in ("ResNet18FPN", "ResNet50FPN"):
        x = torch.randn((1, 3, 128, 128), generator=torch.Generator().manual_seed(0))
        sd = {k: v.float() for k, v in make_state_dict(backbone, 2, 9, False, 0).items()}
        with torch.no_grad():
            taps, feats = net_oracle.fp16_network(sd, backbone, x)
            ref = model_ref.features(sd, backbone, x, True)
        assert set(taps) == set(names)
        assert all(torch.equal(a, b) for a, b in zip(feats, ref))
    for other in ("ResNeXt50_32x4dFPN", "MobileNetV2FPN"):
        with pytest.raises(ValueError):
            calib.network_tensors(other)


def test_network_oracle_pieces_exact():
    """conv_int is exact for every K, stride and kernel size; fma_add rounds once."""
    g = torch.Generator().manual_seed(2)
    q = torch.randint(-127, 128, (1, 256, 9, 11), generator=g).double()
    for ks, stride in ((1, 1), (3, 1), (1, 2), (3, 2)):
        w = torch.randint(-127, 128, (32, 256, ks, ks), generator=g).double()
        ref = torch.nn.functional.conv2d(q, w, stride=stride, padding=ks // 2)
        assert torch.equal(net_oracle.conv_int(q, w, stride), ref)
    r = torch.tensor([3.0, -127.0, 1.0]).double()
    t = torch.tensor([1.0, 2.5, 2.0 ** 24], dtype=torch.float32)
    s = torch.tensor(0.1, dtype=torch.float32)
    exact = r * s.double() + t.double()
    assert torch.equal(net_oracle.fma_add(r, s, t), exact.float())


def _sqnr(ref, got, bias):
    sig = sum(float(((r - bias) ** 2).sum()) for r in ref)
    return 10 * np.log10(sig / sum(float(((g - r) ** 2).sum()) for g, r in zip(got, ref)))


def test_network_oracle_sqnr_vs_fp32():
    """SQNR of the network-scope INT8 heads against the all-fp32 oracle (ResNet18FPN, 2 x 3 x 256 x 384, entropy
    calibration on the batch, the set-up of test_int8_host's heads-only test), over all five levels, final bias left out.
    Measured: cls 27.0 dB, box 27.2 dB, against 29.9 / 30.4 dB with INT8 heads only -- the 3 dB the quantised layer3,
    layer4 and FPN cost.  Asserted with 3 dB of margin."""
    backbone = "ResNet18FPN"
    sd = {k: v.float() for k, v in make_state_dict(backbone, 6, 9, False, 3).items()}
    x = torch.randn((2, 3, 256, 384), generator=torch.Generator().manual_seed(1))
    c3 = "backbones.%s.features.layer2" % backbone
    with torch.no_grad():
        scales, taps, _ = net_oracle.calibrate(sd, backbone, x)
        q3 = int8_oracle.quant_s8(taps[c3], int8_oracle.f32(1.0) / int8_oracle.f32(scales[c3]))
        qc, qb = net_oracle.forward_heads(sd, backbone, q3, scales, sigmoid=False)
        rc, rb = model_ref.forward_heads(sd, backbone, x, sigmoid=False)
    for name, ref, got in (("cls", rc, qc), ("box", rb, qb)):
        assert _sqnr(ref, got, sd["%s_head.8.bias" % name].view(1, -1, 1, 1)) > 24.0, name


def spread_head(sd, std=0.05, prior=0.02):
    """The detection set-up of the GPU INT8 tests (test_gpu_int8._spread_head): a class head with some dynamic range."""
    g = torch.Generator().manual_seed(123)
    sd = dict(sd)
    sd["cls_head.8.weight"] = torch.randn(sd["cls_head.8.weight"].shape, generator=g) * std
    sd["cls_head.8.bias"] = torch.full_like(sd["cls_head.8.bias"], -float(np.log((1 - prior) / prior)))
    sd["box_head.8.weight"] = torch.randn(sd["box_head.8.weight"].shape, generator=g) * 0.02
    return sd


def match(got, ref, score_tol=0.02, px=2.0):
    """Detections of `ref` found in `got`: same class, every box coordinate within px, score within score_tol."""
    gs, gb, gc = got
    rs, rb, rc = ref
    n = int((rs > 0).sum())
    hit = 0
    for i in range(n):
        ok = (gc == rc[i]) & (np.abs(gb - rb[i]).max(axis=1) <= px) & (np.abs(gs - rs[i]) <= score_tol)
        hit += bool(ok.any())
    return hit, n


# Network-scope INT8 vs fp16 detections of the oracles (int8_network_oracle vs model_ref fp16, entropy calibration on the
# batch, the set-up of test_gpu_int8's match-rate test), 200 reference detections each: measured 177 / 200 and 133 / 200.
# With INT8 heads only the same set-up gives 182 / 200 and 179 / 200.  ResNet50FPN loses far more than ResNet18FPN, most
# likely because the requantisation error of its 9 quantised residual blocks (against 4) compounds (not analysed further).
MATCH_NETWORK_ORACLE = {"ResNet18FPN": 0.885, "ResNet50FPN": 0.665}


@pytest.mark.parametrize("backbone", ["ResNet18FPN", "ResNet50FPN"])
def test_network_oracle_match_rate_vs_fp16(backbone):
    sd = {k: v.float() for k, v in spread_head(make_state_dict(backbone, 6, 9, False, 10)).items()}
    x = torch.randn((2, 3, 256, 384), generator=torch.Generator().manual_seed(4))
    c3 = "backbones.%s.features.layer2" % backbone
    with torch.no_grad():
        scales, taps, _ = net_oracle.calibrate(sd, backbone, x)
        q3 = int8_oracle.quant_s8(taps[c3], int8_oracle.f32(1.0) / int8_oracle.f32(scales[c3]))
        cls, box = net_oracle.forward_heads(sd, backbone, q3, scales)
        got, _ = model_ref.postprocess(cls, box, x.shape[-1])
        ref = model_ref.forward(sd, backbone, x, fp16=True)
    hit = n = 0
    for img in range(x.shape[0]):
        h, k = match([t[img] for t in got], [t[img] for t in ref])
        hit, n = hit + h, n + k
    assert n == 200
    assert abs(hit / n - MATCH_NETWORK_ORACLE[backbone]) <= 0.02, (hit, n)
