"""INT8-emulating oracle of the network scope -- TEST INFRASTRUCTURE ONLY (imported by tests/test_*int8_network*.py).

Model.set_precision("int8", table, scope="network") runs ResNet layer3, layer4 and the FPN on s8 from layer2's output C3
quantised once, and the FPN writes the s8 atlas the INT8 heads read.  Every convolution is an exact integer convolution
followed by one correctly rounded fp32 operation per term (include/odtk_b200.h, odtk_conv2d_s8_ex):

    t = fmaf(acc, alpha[c], bias[c]);  t = fmaf(r, res_scale, t) (residual);  t = fmaf(u, up_scale, t) (upsample)
    ReLU (optional);  q = clamp(rint(t * inv_out), -127, 127)

so this emulation is bit-exact.  It starts from an s8 C3 (the GPU tests pass the model's own, so that the fp32 summation
order of the fp16 stem / layer1 / layer2 cannot leak in) and ends with int8_oracle.head on the s8 atlas levels.
fp16_network is oracle/model_ref.py's fp16-emulating backbone + FPN with the tensors the network scope quantises recorded
(CPU calibration)."""
import torch
import torch.nn.functional as F

import int8_oracle
from int8_oracle import f32, fmaf, quant_s8, quant_weight
from oracle import model_ref
from retinanet_examples_b200 import calib

CHUNK = (2 ** 24 - 1) // (127 * 127)     # 1040 products: every fp32 partial sum stays below 2^24, exact in any order


def conv_int(q, wq, stride=1):
    """Exact ksize x ksize (pad ksize // 2) stride-1 / stride-2 convolution of integer tensors (|values| <= 127): fp32
    GEMMs over K chunks of CHUNK products, summed in float64."""
    n, cin, h, w = q.shape
    cout, _, k, _ = wq.shape
    pad = k // 2
    oh, ow = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
    if k == 1:
        cols = q[:, :, ::stride, ::stride].float().reshape(n, cin, oh * ow)
    else:
        cols = F.unfold(q.float(), k, padding=pad, stride=stride)       # [n, cin * k * k, oh * ow], K order (c, r, s)
    wm = wq.float().reshape(cout, -1)
    acc = None
    for k0 in range(0, cols.shape[1], CHUNK):
        part = torch.matmul(wm[:, k0:k0 + CHUNK], cols[:, k0:k0 + CHUNK]).double()
        acc = part if acc is None else acc + part
    return acc.view(n, cout, oh, ow)


def fma_add(r, scale, t):
    """fp32 fmaf(r, scale, t) elementwise: r float64 integers (|r| <= 127), scale a fp32 scalar, t fp32.  r * scale is exact
    in float64; the float64 sum's double rounding is corrected as in int8_oracle.fmaf."""
    p = r * scale.double()
    b = t.double()
    s = p + b
    bb = s - p
    e = (p - (s - bb)) + (b - bb)                                # TwoSum: p + b == s + e exactly
    res = s.float()
    rd = res.double()
    lo = torch.where(rd <= s, res, torch.nextafter(res, torch.tensor(-float("inf"))))
    hi = torch.nextafter(lo, torch.tensor(float("inf")))
    mid = (s - lo.double()) == (hi.double() - s)
    return torch.where(mid & (e != 0), torch.where(e > 0, hi, lo), res)


def upsample2(q):
    """Nearest 2x (FPN top-down path, F.interpolate(scale_factor=2))."""
    return q.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)


def conv(q, w, bias, s_in, inv_out, stride=1, relu=False, res=None, res_scale=None, up=None, up_scale=None):
    """One s8 convolution: integer tensor q -> integer tensor (float64)."""
    wq, s_w = quant_weight(w)
    y = fmaf(conv_int(q, wq, stride), s_w * s_in, bias.float() if bias is not None else None)
    if res is not None:
        y = fma_add(res, res_scale, y)
    if up is not None:
        y = fma_add(upsample2(up), up_scale, y)
    if relu:
        y = F.relu(y)
    return quant_s8(y, inv_out)


def fold(sd, pc, pb):
    """conv + eval BatchNorm -> (weight, bias), fp32, the arithmetic of engine.fold_bn / model_ref._cb."""
    scale = sd[pb + ".weight"] / torch.sqrt(sd[pb + ".running_var"] + 1e-5)
    return sd[pc + ".weight"] * scale.view(-1, 1, 1, 1), sd[pb + ".bias"] - sd[pb + ".running_mean"] * scale


def network(sd, backbone, q3, scales):
    """The s8 atlas levels [P3, P4, P5, P6, P7] (float64 integers, NCHW) of the network scope from the s8 C3 q3."""
    block, layers = model_ref.LAYERS[backbone]
    f, n = "backbones.%s.features." % backbone, "backbones.%s." % backbone

    def S(name):
        return f32(scales[name])

    def inv(name):
        return f32(1.0) / S(name)

    x, xn = q3, f + "layer2"
    taps = {}
    for li in (3, 4):
        for b in range(layers[li - 1]):
            p = f + "layer%d.%d" % (li, b)
            stride = 2 if b == 0 else 1
            mids = [p + ".conv1", p + ".conv2"] if block == "bottleneck" else [p + ".conv1"]
            ins, outs = [xn] + mids, mids + [p]
            strided = 1 if block == "bottleneck" else 0
            ident, rs = x, S(xn)
            if (p + ".downsample.0.weight") in sd:
                ident = conv(x, *fold(sd, p + ".downsample.0", p + ".downsample.1"), S(xn), inv(p + ".downsample"), stride)
                rs = S(p + ".downsample")
            t = x
            for k in range(len(ins)):
                last = k == len(ins) - 1
                t = conv(t, *fold(sd, p + ".conv%d" % (k + 1), p + ".bn%d" % (k + 1)), S(ins[k]), inv(outs[k]),
                         stride if k == strided else 1, relu=True, res=ident if last else None, res_scale=rs)
            x, xn = t, p
        taps[li] = (x, xn)
    (c4, c4n), (c5, c5n) = taps[3], taps[4]

    def plain(name, q, s_in, out, stride=1, **kw):
        return conv(q, sd[n + name + ".weight"], sd.get(n + name + ".bias"), s_in, inv(out), stride, **kw)

    p5 = plain("lateral5", c5, S(c5n), n + "lateral5")
    p4 = plain("lateral4", c4, S(c4n), n + "lateral4", up=p5, up_scale=S(n + "lateral5"))
    p3 = plain("lateral3", q3, S(f + "layer2"), n + "lateral3", up=p4, up_scale=S(n + "lateral4"))
    hi = "heads.input"
    levels = [plain("smooth%d" % k, t, S(n + "lateral%d" % k), hi) for k, t in ((3, p3), (4, p4), (5, p5))]
    p6 = plain("pyramid6", c5, S(c5n), hi, 2)
    p7 = plain("pyramid7", F.relu(p6), S(hi), hi, 2)                 # ReLU on symmetric s8 values is exact
    return levels + [p6, p7]


def heads(sd, levels, scales, sigmoid=True):
    """int8_oracle.head on the s8 atlas levels.  head() quantises its input with "heads.input"; the levels are handed to it
    as q * s_in, which that quantisation maps back to exactly q."""
    s_in = f32(scales["heads.input"])
    feats = []
    for q in levels:
        t = q.float() * s_in
        assert torch.equal(quant_s8(t, f32(1.0) / s_in), q)
        feats.append(t)
    cls = [int8_oracle.head(sd, "cls_head", t, scales) for t in feats]
    box = [int8_oracle.head(sd, "box_head", t, scales) for t in feats]
    if sigmoid:
        cls = [c.sigmoid() for c in cls]
    return cls, box


def forward_heads(sd, backbone, q3, scales, sigmoid=True):
    """Model.forward_heads in network scope from the s8 C3 q3 (NCHW integers)."""
    with torch.no_grad():
        sd = {k: v.float() for k, v in sd.items()}
        return heads(sd, network(sd, backbone, q3.double(), scales), scales, sigmoid)


def fp16_network(sd, backbone, x):
    """oracle/model_ref.py's fp16-emulating ResNet + FPN (same roundings), recording every tensor of
    calib.network_tensors(backbone).  Returns (taps, the five FPN levels)."""
    _q, _cb = model_ref._q, model_ref._cb
    block, layers = model_ref.LAYERS[backbone]
    f, n = "backbones.%s.features." % backbone, "backbones.%s." % backbone
    taps, outs = {}, []
    x = _q(x, True)
    x = _q(F.relu(_cb(sd, f + "conv1", f + "bn1", x, 2, 3, True)), True)
    x = F.max_pool2d(x, 3, 2, 1)
    for li, nblocks in enumerate(layers):
        for b in range(nblocks):
            stride = 2 if (b == 0 and li > 0) else 1
            p = f + "layer%d.%d" % (li + 1, b)
            identity = x
            if block == "bottleneck":
                o1 = _q(F.relu(_cb(sd, p + ".conv1", p + ".bn1", x, 1, 0, True)), True)
                o2 = _q(F.relu(_cb(sd, p + ".conv2", p + ".bn2", o1, stride, 1, True)), True)
                out, mids = _cb(sd, p + ".conv3", p + ".bn3", o2, 1, 0, True), [o1, o2]
            else:
                o1 = _q(F.relu(_cb(sd, p + ".conv1", p + ".bn1", x, stride, 1, True)), True)
                out, mids = _cb(sd, p + ".conv2", p + ".bn2", o1, 1, 1, True), [o1]
            if (p + ".downsample.0.weight") in sd:
                identity = _cb(sd, p + ".downsample.0", p + ".downsample.1", x, stride, 0, True)
                if not (block == "bottleneck" and stride == 1):
                    identity = _q(identity, True)
                if li >= 2:
                    taps[p + ".downsample"] = identity
            x = _q(F.relu(out + identity), True)
            if li >= 2:
                taps.update({p + ".conv%d" % (k + 1): m for k, m in enumerate(mids)})
                taps[p] = x
        if li >= 1:
            outs.append(x)
    c3, c4, c5 = outs
    taps[f + "layer2"] = c3
    p5 = _q(_cb(sd, n + "lateral5", None, c5, 1, 0, True), True)
    p4 = _q(F.interpolate(p5, scale_factor=2) + _cb(sd, n + "lateral4", None, c4, 1, 0, True), True)
    p3 = _q(F.interpolate(p4, scale_factor=2) + _cb(sd, n + "lateral3", None, c3, 1, 0, True), True)
    taps.update({n + "lateral5": p5, n + "lateral4": p4, n + "lateral3": p3})
    return taps, model_ref._fpn(sd, backbone, c3, c4, c5, True)


def calibrate(sd, backbone, x, method="entropy"):
    """CPU network-scope calibration on the fp16 oracle: every tensor of calib.table_tensors(backbone, "network"); the
    heads' input and tower outputs over all pixels of every level."""
    sd = {k: v.float() for k, v in sd.items()}
    with torch.no_grad():
        taps, feats = fp16_network(sd, backbone, x.float())
        col = calib.Collector()
        for phase in (0, 1):
            col.phase = phase
            for name in calib.network_tensors(backbone):
                col.observe(name, taps[name])
            for head in calib.HEADS:
                for t0 in feats:
                    if head == "cls_head":
                        col.observe("heads.input", t0)
                    t = t0
                    for i in calib.TOWER:
                        t = model_ref._q(F.relu(model_ref._cb(sd, "%s.%d" % (head, i), None, t, 1, 1, True)), True)
                        col.observe("%s.%d" % (head, i), t)
    return col.scales(method, calib.table_tensors(backbone, "network")), taps, feats
