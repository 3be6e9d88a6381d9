"""INT8-emulating oracle of the detection heads -- TEST INFRASTRUCTURE ONLY (imported by tests/test_*int8*.py).

The INT8 heads: symmetric per-output-channel weights (s_w = max|W| / 127, 1 for an all-zero channel,
q = clamp(rint(W / s_w), -127, 127)), one symmetric scale per activation tensor (zero-point 0), exact integer
accumulation, then y = fmaf(acc, alpha, bias) with alpha = s_in * s_w in fp32, ReLU, and requantisation
clamp(rint(y * (1 / s_out)), -127, 127) -- or, after the final layer, fp32 output.  Every step is exact integer
arithmetic or one correctly rounded fp32 operation, so this emulation is bit-exact: the integer convolution is exact
(conv_int; |acc| <= 2304 * 127^2 < 2^53 in float64), the fp32 fma runs in float64 with its double rounding corrected.

The fp16 backbone + FPN in front of the heads are oracle/model_ref.py's fp16-emulating mode."""
import torch
import torch.nn.functional as F

from oracle import model_ref


def f32(v):
    return torch.tensor(float(v), dtype=torch.float32)


def quant_s8(x, inv):
    """fp32 x * fp32 inv (one rounding), round half to even, saturate: the float64 tensor of the s8 values."""
    return torch.round(x.float() * inv).clamp_(-127, 127).double()


def fmaf(acc, alpha, bias):
    """fp32 fmaf(acc, alpha[c], bias[c]) over NCHW float64 integers acc: alpha / bias fp32 [C] (bias may be None)."""
    p = acc * alpha.double().view(1, -1, 1, 1)                 # exact: < 2^26 times a 24-bit significand
    b = bias.double().view(1, -1, 1, 1) if bias is not None else torch.zeros_like(p)
    s = p + b
    bb = s - p
    e = (p - (s - bb)) + (b - bb)                                # TwoSum: p + b == s + e exactly
    r = s.float()
    # s rounded to fp32 is the correctly rounded fma unless s sits exactly halfway between two fp32 neighbours while the
    # exact sum does not (e != 0): then round towards e
    rd = r.double()
    lo = torch.where(rd <= s, r, torch.nextafter(r, torch.tensor(-float("inf"))))
    hi = torch.nextafter(lo, torch.tensor(float("inf")))
    mid = (s - lo.double()) == (hi.double() - s)
    return torch.where(mid & (e != 0), torch.where(e > 0, hi, lo), r)


def conv_int(q, wq):
    """Exact 3x3 pad-1 convolution of integer tensors (|values| <= 127): fp32 GEMMs over K chunks of 576 products, whose
    partial sums stay below 576 * 127^2 < 2^24 and are therefore exact in any order, summed in float64."""
    n, cin, h, w = q.shape
    cols = F.unfold(q.float(), 3, padding=1)                       # [n, cin * 9, h * w], K order (c, r, s)
    wm = wq.float().reshape(wq.shape[0], -1)
    acc = None
    for k0 in range(0, cols.shape[1], 576):
        part = torch.matmul(wm[:, k0:k0 + 576], cols[:, k0:k0 + 576]).double()
        acc = part if acc is None else acc + part
    return acc.view(n, wq.shape[0], h, w)


def quant_weight(w):
    """fp32 [Cout, Cin, kh, kw] -> (integer-valued fp32 weights, s_w fp32 [Cout])."""
    w = w.float()
    amax = w.abs().amax(dim=(1, 2, 3))
    s_w = torch.where(amax > 0, amax / 127.0, torch.ones_like(amax))
    return torch.round(w / s_w.view(-1, 1, 1, 1)).clamp_(-127, 127), s_w


def head(sd, name, t, scales):
    """One head (`cls_head` / `box_head`) in INT8 on one level's fp16 features t [N, 256, H, W] (fp32 tensor holding fp16
    values); scales: the 9 activation scales of a calibration table.  Returns the fp32 logits / box deltas."""
    s_in = f32(scales["heads.input"])
    q = quant_s8(t, f32(1.0) / s_in)
    for i in (0, 2, 4, 6, 8):
        wq, s_w = quant_weight(sd["%s.%d.weight" % (name, i)])
        bias = sd.get("%s.%d.bias" % (name, i))
        y = fmaf(conv_int(q, wq), s_w * s_in, bias.float() if bias is not None else None)
        if i == 8:
            return y
        s_out = f32(scales["%s.%d" % (name, i)])
        q = quant_s8(F.relu(y), f32(1.0) / s_out)
        s_in = s_out


def forward_heads(sd, backbone, x, scales, sigmoid=True):
    """Reference Model.forward with exporting=True, fp16 backbone + FPN (model_ref's fp16-emulating mode), INT8 heads."""
    with torch.no_grad():
        sd = {k: v.float() for k, v in sd.items()}
        feats = model_ref.features(sd, backbone, x.float(), True)
        cls = [head(sd, "cls_head", t, scales) for t in feats]
        box = [head(sd, "box_head", t, scales) for t in feats]
        if sigmoid:
            cls = [c.sigmoid() for c in cls]
    return cls, box
