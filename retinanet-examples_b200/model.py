"""RetinaNet inference model -- host-side mirror of the reference's odtk/model.py `Model`
(constructor arguments, `config` keys, state_dict key names, `forward(x) -> (scores, boxes,
classes)`), executing on the sm_90a kernels behind the C ABI instead of nn.Conv2d/cuDNN +
odtk._C.  `_compute_loss` (training-mode forward) runs target assignment + ONE fused loss kernel; `save` / `load` /
`initialize(pre_trained)` read and write the reference's checkpoint dict; ONNX/TensorRT export is outside the
hot path; `load_state_dict` ingests exactly the reference's key layout
(odtk/model.py:217-258): `backbones.<Name>.features.*`, `backbones.<Name>.{lateral,pyramid,smooth}*`,
`cls_head.{0,2,4,6,8}.*`, `box_head.{0,2,4,6,8}.*`.

Data flow of forward() (reference: odtk/model.py:125-165, odtk/backbones/fpn.py:45-61,
odtk/backbones/resnet.py:24-39, torchvision BasicBlock/Bottleneck):
  NHWC fp16 activations; every conv is one launch of the wgmma kernel with BatchNorm folded
  into weights/bias, ReLU / residual add / FPN upsample-add fused in its epilogue; the last conv
  of each head writes fp32 NCHW (sigmoid fused for the class head) which feeds the all-levels
  decode (3 launches) and the batched NMS (1 launch)."""
import math
import os

import numpy as np
import torch

from . import _C, box, calib, engine

RESNET_LAYERS = {"ResNet18FPN": ("basic", [2, 2, 2, 2]), "ResNet34FPN": ("basic", [3, 4, 6, 3]),
                 "ResNet50FPN": ("bottleneck", [3, 4, 6, 3]), "ResNet101FPN": ("bottleneck", [3, 4, 23, 3]),
                 "ResNet152FPN": ("bottleneck", [3, 8, 36, 3]),
                 "ResNeXt50_32x4dFPN": ("bottleneck", [3, 4, 6, 3]), "ResNeXt101_32x8dFPN": ("bottleneck", [3, 4, 23, 3])}
# grouped bottlenecks (odtk/backbones/fpn.py:85-91): (groups, width_per_group); conv2 has planes * width_per_group / 64 * groups channels
RESNEXT = {"ResNeXt50_32x4dFPN": (32, 4), "ResNeXt101_32x8dFPN": (32, 8)}
# MobileNetV2 (odtk/backbones/mobilenet.py:5-25, fpn.py:92-93; torchvision mobilenetv2.py inverted_residual_setting):
# (expansion t, output channels c, repeats n, first stride s); FPN taps features[6 / 13 / 17] = 32 / 96 / 320 channels
MOBILENET = {"MobileNetV2FPN": [(1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1), (6, 160, 3, 2), (6, 320, 1, 1)]}
MOBILENET_TAPS = (6, 13, 17)
BACKBONES = tuple(RESNET_LAYERS) + tuple(MOBILENET)
# backbones of the full-precision mode (set_precision("fp32")): the plain ResNets (no grouped or depthwise convolutions)
FP32_BACKBONES = tuple(b for b in RESNET_LAYERS if b not in RESNEXT)


def mobilenet_blocks(backbone):
    """[(features index, cin, cout, stride, t)] of the inverted residual blocks (features[1 .. 17])."""
    out, cin, idx = [], 32, 1
    for t, c, n, s in MOBILENET[backbone]:
        for i in range(n):
            out.append((idx, cin, c, s if i == 0 else 1, t))
            cin, idx = c, idx + 1
    return out


def _head_specs(classes, num_anchors, rotated):
    specs = []
    nbox = 6 if rotated else 4
    for head, out in (("cls_head", classes * num_anchors), ("box_head", nbox * num_anchors)):
        for i in (0, 2, 4, 6):
            specs.append(("%s.%d" % (head, i), "convb", (256, 256, 3, 3)))
        specs.append(("%s.8" % head, "convb_final", (out, 256, 3, 3)))
    return specs


def _fpn_specs(n, ch):
    return [(n + "lateral3", "convb", (256, ch[0], 1, 1)), (n + "lateral4", "convb", (256, ch[1], 1, 1)),
            (n + "lateral5", "convb", (256, ch[2], 1, 1)), (n + "pyramid6", "convb", (256, ch[2], 3, 3)),
            (n + "pyramid7", "convb", (256, 256, 3, 3)), (n + "smooth3", "convb", (256, 256, 3, 3)),
            (n + "smooth4", "convb", (256, 256, 3, 3)), (n + "smooth5", "convb", (256, 256, 3, 3))]


def mobilenet_specs(backbone, classes, num_anchors, rotated):
    f = "backbones.%s.features.features." % backbone       # FPN.features = MobileNet module, MobileNet.features = Sequential
    specs = [(f + "0.0", "conv", (32, 3, 3, 3)), (f + "0.1", "bn", 32)]
    for idx, cin, cout, stride, t in mobilenet_blocks(backbone):
        hidden, k = cin * t, 0
        p = f + "%d.conv." % idx
        if t != 1:
            specs += [(p + "0.0", "conv", (hidden, cin, 1, 1)), (p + "0.1", "bn", hidden)]
            k = 1
        specs += [(p + "%d.0" % k, "conv", (hidden, 1, 3, 3)), (p + "%d.1" % k, "bn", hidden),
                  (p + "%d" % (k + 1), "conv", (cout, hidden, 1, 1)), (p + "%d" % (k + 2), "bn_last", cout)]
    return specs + _fpn_specs("backbones.%s." % backbone, [32, 96, 320]) + _head_specs(classes, num_anchors, rotated)


def conv_specs(backbone, classes=80, num_anchors=9, rotated=False):
    """Every convolution / batch-norm of the model as (state_dict prefix, kind, shape info), in
    forward order.  kind: 'conv' (weight only, followed by 'bn') or 'convb' (weight + bias)."""
    if backbone in MOBILENET:
        return mobilenet_specs(backbone, classes, num_anchors, rotated)
    block, layers = RESNET_LAYERS[backbone]
    f = "backbones.%s.features." % backbone
    specs = [(f + "conv1", "conv", (64, 3, 7, 7)), (f + "bn1", "bn", 64)]
    inplanes = 64
    exp = 4 if block == "bottleneck" else 1
    for li, (planes, nblocks) in enumerate(zip([64, 128, 256, 512], layers)):
        for b in range(nblocks):
            stride = 2 if (b == 0 and li > 0) else 1
            p = f + "layer%d.%d." % (li + 1, b)
            if block == "bottleneck":
                groups, wpg = RESNEXT.get(backbone, (1, 64))
                width = planes * wpg // 64 * groups
                specs += [(p + "conv1", "conv", (width, inplanes, 1, 1)), (p + "bn1", "bn", width),
                          (p + "conv2", "conv", (width, width // groups, 3, 3)), (p + "bn2", "bn", width),
                          (p + "conv3", "conv", (planes * 4, width, 1, 1)), (p + "bn3", "bn_last", planes * 4)]
            else:
                specs += [(p + "conv1", "conv", (planes, inplanes, 3, 3)), (p + "bn1", "bn", planes),
                          (p + "conv2", "conv", (planes, planes, 3, 3)), (p + "bn2", "bn_last", planes)]
            if b == 0 and (stride != 1 or inplanes != planes * exp):
                specs += [(p + "downsample.0", "conv", (planes * exp, inplanes, 1, 1)),
                          (p + "downsample.1", "bn", planes * exp)]
            inplanes = planes * exp
    ch = [128, 256, 512] if block == "basic" else [512, 1024, 2048]
    return specs + _fpn_specs("backbones.%s." % backbone, ch) + _head_specs(classes, num_anchors, rotated)


def make_state_dict(backbone="ResNet50FPN", classes=80, num_anchors=9, rotated=False, seed=0, cls_prior=0.01):
    """Deterministic random-init weights in the reference's state_dict layout (no checkpoint or
    pretrained weights exist offline).  BatchNorm statistics are randomised so that folding is
    exercised; the last BN of each residual block is damped so
    that activations stay well inside fp16 range through 50+ layers."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, kind, shp in conv_specs(backbone, classes, num_anchors, rotated):
        if kind.startswith("conv"):
            cout, cin, kh, kw = shp
            std = 0.01 if name.startswith(("cls_head", "box_head")) else math.sqrt(2.0 / (cin * kh * kw))   # cin = per-group fan-in
            sd[name + ".weight"] = torch.randn(shp, generator=g) * std
            if kind != "conv":
                sd[name + ".bias"] = torch.randn(cout, generator=g) * 0.01
                if kind == "convb_final" and name.startswith("cls_head"):
                    sd[name + ".bias"] = torch.full((cout,), -math.log((1 - cls_prior) / cls_prior))
        else:
            c = shp
            lo, hi = (0.1, 0.3) if kind == "bn_last" else (0.5, 1.5)
            sd[name + ".weight"] = torch.rand(c, generator=g) * (hi - lo) + lo
            sd[name + ".bias"] = torch.randn(c, generator=g) * 0.1
            sd[name + ".running_mean"] = torch.randn(c, generator=g) * 0.1
            sd[name + ".running_var"] = torch.rand(c, generator=g) + 0.5
    return sd


def network_walk(backbone):
    """Every convolution of the model once, in the shape of a packed layer set: "stem", "blocks" [{convs, down, level,
    last, name}], "lateral3-5", "smooth3-5", "pyramid6-7", "cls_head", "box_head" (MobileNetV2FPN: the heads only, its
    backbone is packed by Model._pack_mobilenet).  A convolution is a dict: conv / bn (state-dict prefixes; bn None for a
    convolution with its own bias), stride, groups, x / y (the names of its input and output tensors, those of
    calib.network_tensors and the calibration tables) and, for the convolutions that add one, res / up (the name of the
    residual / upsample addend)."""
    def conv(c, bn=None, stride=1, groups=1, x=None, y=None, **addend):
        return dict(conv=c, bn=bn, stride=stride, groups=groups, x=x, y=y, **addend)

    walk = {}
    for head in calib.HEADS:
        names = ["heads.input"] + ["%s.%d" % (head, i) for i in (0, 2, 4, 6, 8)]
        walk[head] = [conv(names[k + 1], x=names[k], y=names[k + 1]) for k in range(5)]
    if backbone in MOBILENET:
        return walk
    block, layers = RESNET_LAYERS[backbone]
    f, n = "backbones.%s.features." % backbone, "backbones.%s." % backbone
    groups = RESNEXT.get(backbone, (1, 64))[0]
    exp = 4 if block == "bottleneck" else 1
    walk["stem"] = conv(f + "conv1", f + "bn1", 2, x="input", y=f + "conv1")
    blocks, taps, x, inplanes = [], {}, f + "maxpool", 64
    for li, (planes, nblocks) in enumerate(zip((64, 128, 256, 512), layers)):
        for b in range(nblocks):
            stride = 2 if (b == 0 and li > 0) else 1
            p = f + "layer%d.%d" % (li + 1, b)
            y = f + "layer2" if (li == 1 and b == nblocks - 1) else p      # C3 is named after its layer
            down = None
            if b == 0 and (stride != 1 or inplanes != planes * exp):
                down = conv(p + ".downsample.0", p + ".downsample.1", stride, x=x, y=p + ".downsample")
            if block == "bottleneck":       # torchvision v1.5: the 3x3 carries the stride
                ins, strides, gs = [x, p + ".conv1", p + ".conv2"], [1, stride, 1], [1, groups, 1]
            else:
                ins, strides, gs = [x, p + ".conv1"], [stride, 1], [1, 1]
            outs = ins[1:] + [y]
            convs = [conv(p + ".conv%d" % (k + 1), p + ".bn%d" % (k + 1), strides[k], gs[k], x=ins[k], y=outs[k])
                     for k in range(len(ins))]
            convs[-1]["res"] = down["y"] if down else x
            blocks.append({"convs": convs, "down": down, "level": li + 2, "last": b == nblocks - 1, "name": p})
            x, inplanes = y, planes * exp
        taps[li + 2] = x
    walk["blocks"] = blocks
    walk["lateral5"] = conv(n + "lateral5", x=taps[5], y=n + "lateral5")
    walk["lateral4"] = conv(n + "lateral4", x=taps[4], y=n + "lateral4", up=n + "lateral5")
    walk["lateral3"] = conv(n + "lateral3", x=taps[3], y=n + "lateral3", up=n + "lateral4")
    for k in (3, 4, 5):       # smooth and pyramid write the atlas the heads read
        walk["smooth%d" % k] = conv(n + "smooth%d" % k, x=n + "lateral%d" % k, y="heads.input")
    walk["pyramid6"] = conv(n + "pyramid6", stride=2, x=taps[5], y="heads.input")
    walk["pyramid7"] = conv(n + "pyramid7", stride=2, x="heads.input", y="heads.input")
    return walk


def pack_walk(walk, make):
    """The packed layer set of `walk` with every convolution replaced by make(convolution) (None: not in this set)."""
    P = {}
    for k, v in walk.items():
        if k == "blocks":
            P[k] = [dict(b, convs=[make(c) for c in b["convs"]], down=make(b["down"]) if b["down"] else None) for b in v]
        else:
            P[k] = [make(c) for c in v] if isinstance(v, list) else make(v)
    return P


def walk_weights(sd, c):
    """(weight, bias) of a convolution of network_walk, BatchNorm folded (fp32)."""
    if c["bn"] is None:
        return sd[c["conv"] + ".weight"], sd.get(c["conv"] + ".bias")
    bn = c["bn"]
    return engine.fold_bn(sd[c["conv"] + ".weight"], sd[bn + ".weight"], sd[bn + ".bias"], sd[bn + ".running_mean"],
                          sd[bn + ".running_var"])


def _out_size(x, stride):
    return (x.shape[1] - 1) // stride + 1, (x.shape[2] - 1) // stride + 1


class _Conv:
    """One packed convolution: fp16 weights in the kernel's K order, fp32 bias, geometry.  Packed layers of every precision
    take (x, relu, residual, upsample, out, out_mode, sink, tile_tab, valid_px) and count their FLOPs."""

    def __init__(self, weight, bias, stride=1, device="cuda", groups=1):
        cout, cin, kh, kw = weight.shape
        self.groups = groups
        if groups > 1:                       # grouped 3x3 (ResNeXt): block-diagonal packing, see engine.pack_weight_grouped
            self.cout, self.cin, self.ks, self.stride = cout, cin * groups, kh, stride
            self.direct, self.stem, self.w_stem = stride == 1, False, None
            self.kpad = kh * kw * 64
            self.w = engine.pack_weight_grouped(weight, groups).to(device)
            self.b = bias.float().contiguous().to(device) if bias is not None else None
            return
        self.cout, self.cin, self.ks, self.stride = cout, cin, kh, stride
        self.direct = stride == 1 and kh in (1, 3) and cin % 64 == 0
        self.stem = (cin == 3 and kh == 7 and stride == 2 and cout % 16 == 0 and cout <= 256)
        self.w_stem = engine.pack_stem_weight(weight).to(device) if self.stem else None
        kreal = kh * kw * cin
        self.kpad = kreal if self.direct else (kreal + 63) // 64 * 64
        self.w = engine.pack_weight(weight, self.kpad).to(device)
        self.b = bias.float().contiguous().to(device) if bias is not None else None

    def __call__(self, x, relu=False, residual=None, upsample=None, out=None, out_mode=engine.OUT_NHWC_F16, sink=None,
                 tile_tab=None, valid_px=None):
        oh, ow = _out_size(x, self.stride)
        px = x.shape[0] * oh * ow if valid_px is None else valid_px          # atlas launches: only the pixels of the levels count
        engine.STATS["conv_flops"] += 2 * px * self.cout * self.ks * self.ks * self.cin // self.groups
        if self.stem and x.shape[1] % 2 == 0 and x.shape[2] % 2 == 0 and residual is None and upsample is None:
            return engine.stem_conv(x, self.w_stem, self.b, self.cout, relu)
        if self.direct:
            return engine.conv2d(x, self.w, self.b, self.cout, self.ks, relu, residual, upsample, out_mode,
                                 sink=sink, groups=self.groups, out=out, tile_tab=tile_tab)
        assert sink is None
        if self.stride == 2 and self.ks in (1, 3) and self.cin % 64 == 0 and upsample is None:
            # stride-2 convolution, any size: strided TMA view (even sizes: parity split, odd sizes: element-strided
            # boxes), no gather pre-pass
            return engine.conv2d(x, self.w, self.b, self.cout, self.ks, relu, residual, None, out_mode, stride=2,
                                 groups=self.groups, out=out)
        low = engine.lower_conv(x, self.ks, self.stride, self.ks // 2, self.kpad if self.cin % 8 else None)
        return engine.conv2d(low, self.w, self.b, self.cout, 1, relu, residual, upsample, out_mode)


class _ConvS8:
    """One packed INT8 convolution: symmetric per-channel s8 weights and its epilogue constants from the calibration scales
    of its tensors -- alpha[c] = s_in * s_w[c] (fp32), the fp32 bias, inv_out = 1 / s_out (None: an fp32 output), and the
    scales of its residual / upsample addends."""

    def __init__(self, weight, bias, s_in, s_out, stride=1, device="cuda", res_scale=None, up_scale=None):
        q, s_w = engine.pack_weight_s8(weight)
        self.w = q.to(device)
        self.alpha = (s_w * torch.tensor(s_in, dtype=torch.float32)).contiguous().to(device)
        self.b = bias.float().contiguous().to(device) if bias is not None else None
        self.cout, self.ks, self.stride = weight.shape[0], weight.shape[2], stride
        self.inv_out = float(np.float32(1.0) / s_out) if s_out is not None else None
        self.res_scale, self.up_scale = res_scale, up_scale

    def __call__(self, x, relu=False, residual=None, upsample=None, out=None, out_mode=engine.OUT_NHWC_S8, sink=None,
                 tile_tab=None, valid_px=None):
        oh, ow = _out_size(x, self.stride)
        px = x.shape[0] * oh * ow if valid_px is None else valid_px
        engine.STATS["conv_flops"] += 2 * px * self.cout * self.ks * self.ks * x.shape[3]
        return engine.conv2d_s8(x, self.w, self.alpha, self.b, self.cout, self.ks, relu=relu, out_mode=out_mode, out=out,
                                inv_out_scale=self.inv_out if self.inv_out is not None else 1.0, sink=sink,
                                tile_tab=tile_tab, stride=self.stride, residual=residual,
                                res_scale=self.res_scale if residual is not None else 0.0, upsample=upsample,
                                up_scale=self.up_scale if upsample is not None else 0.0)


class _ConvF32:
    """One packed full-precision convolution: the fp32 weights split into two tf32-valued halves
    (engine.pack_weight_tf32x2; the stem in its window K order), the fp32 bias, geometry."""

    def __init__(self, weight, bias, stride=1, device="cuda", stem=False):
        hi, lo = engine.pack_stem_weight_tf32x2(weight) if stem else engine.pack_weight_tf32x2(weight)
        self.hi, self.lo = hi.to(device), lo.to(device)
        self.b = bias.float().contiguous().to(device) if bias is not None else None
        self.cout, self.ks, self.stride = weight.shape[0], weight.shape[2], stride

    def __call__(self, x, relu=False, residual=None, upsample=None, out=None, out_mode=engine.OUT_NHWC_F32, sink=None,
                 tile_tab=None, valid_px=None):
        oh, ow = _out_size(x, self.stride)
        px = x.shape[0] * oh * ow if valid_px is None else valid_px
        engine.STATS["conv_flops"] += 2 * px * self.cout * self.ks * self.ks * x.shape[3]
        return engine.conv2d_f32(x, self.hi, self.lo, self.b, self.cout, self.ks, relu=relu, residual=residual,
                                 upsample=upsample, out_mode=out_mode, out=out, stride=self.stride, sink=sink,
                                 tile_tab=tile_tab)


FPN_LAYERS = ("lateral3", "lateral4", "lateral5", "pyramid6", "pyramid7", "smooth3", "smooth4", "smooth5")   # fpn.py:26-33


class _HeadsTrain(torch.autograd.Function):
    """(cls_loss, box_loss) of the training forward as a function of the parameters of the training scope (the heads, or
    the FPN and the heads: Model._train_forward / Model._train_backward)."""

    @staticmethod
    def forward(ctx, model, x, targets, *params):
        cls_loss, box_loss, state = model._train_forward(x, targets)
        ctx.model, ctx.state = model, state
        ctx.set_materialize_grads(False)       # a loss outside the graph gives None: its head gets no gradient
        return cls_loss, box_loss

    @staticmethod
    def backward(ctx, g_cls, g_box):
        grads = ctx.model._train_backward(ctx.state, g_cls, g_box, ctx.needs_input_grad[3:])
        return (None, None, None) + tuple(grads)


class Model:
    'RetinaNet - https://arxiv.org/abs/1708.02002 (reference: odtk/model.py:15-72)'

    def __init__(self, backbones='ResNet50FPN', classes=80, ratios=[1.0, 2.0, 0.5],
                 scales=[4 * 2 ** (i / 3) for i in range(3)], angles=None, rotated_bbox=False,
                 anchor_ious=[0.4, 0.5], config={}):
        if isinstance(backbones, (list, tuple)):
            if len(backbones) != 1:
                raise ValueError("one backbone per model on this path")
            backbones = backbones[0]
        if backbones not in BACKBONES:
            raise ValueError("unsupported backbone %r (hot path: %s)" % (backbones, ", ".join(BACKBONES)))
        self.backbone = backbones
        self.name = 'RetinaNet'
        self.exporting = False
        self.training = False
        self.rotated_bbox = rotated_bbox
        self.anchor_ious = anchor_ious
        self.ratios, self.scales = ratios, scales
        self.angles = angles if angles is not None else [-np.pi / 6, 0, np.pi / 6] if rotated_bbox else None
        self.anchors = {}
        self.classes = classes
        self.threshold = config.get('threshold', 0.05)
        self.top_n = config.get('top_n', 1000)
        self.nms = config.get('nms', 0.5)
        self.detections = config.get('detections', 100)
        self.stride = 128
        if self.top_n > 4096 or self.detections > 1024 or 5 * self.top_n > 6144:
            raise ValueError("config outside the sm_90a kernels' limits (include/odtk_b200.h): top_n <= 4096, "
                             "5 * top_n <= 6144 candidates per image into NMS, detections <= 1024; got top_n=%d detections=%d"
                             % (self.top_n, self.detections))
        self.num_anchors = len(ratios) * len(scales) * (len(self.angles) if rotated_bbox else 1)
        self._sd = None
        self._packed = None
        self.device = None
        self.parallel_heads = True
        self.fused_candidates = os.environ.get("ODTK_FUSED_CANDIDATES", "1") != "0"
        self._atlas = {}
        self._fused = {}
        self._head_streams = None
        self.gather = None            # peer.PeerGather: image-wise sharding, detections pushed to all ranks by the NMS kernel
        self._packed_out = {}
        self.precision = "fp16"
        self._int8_table = None       # calibration table of the INT8 heads (set_precision)
        self._int8 = None             # the INT8 network: fp16 layers with the s8 ones of int8_scope in their place
        self.int8_scope = "heads"     # "heads" or "network" (layer3, layer4 and the FPN in INT8 as well)
        self._calib_hook = None
        self._calib_net = False       # calibration also records the network scope's tensors
        self._f32 = None              # full precision: split-TF32 weights of every layer (packed on first use)
        self._params = None           # trainable parameters by name (created by named_parameters / parameters)
        self._walk = network_walk(backbones)   # read by every training forward (_trainable_layers)
        self.train_scope = "heads"    # "heads" or "fpn": which parameters named_parameters lists (set_train_scope)
        self._param_versions = {}     # weight name -> the layer's (weight, bias) _version when its fp16 weights were packed
        self._sd_versions = {}        # parameter name -> its _version when it was last copied into the state dict
        self._dgrad_w = {}            # weight name -> ((_version, id), pack_weight_dgrad weights)
        self._fwd_gen = 0             # counts forward passes: a backward must follow its own forward
        # test hooks, both only while want_atlas_grad is set: the training backward also computes d(loss)/d(atlas) into
        # last_atlas_grad, which ALIASES a gradient buffer of the atlas geometry (the next backward overwrites it), and
        # last_train keeps the last training forward's atlas views, head outputs and loss gradients
        self.want_atlas_grad = False
        self.last_train = None
        self.last_atlas_grad = None

    def __repr__(self):
        return '\n'.join(['     model: {}'.format(self.name), '  backbone: {}'.format(self.backbone),
                          '   classes: {}, anchors: {}'.format(self.classes, self.num_anchors)])

    # ---- weights ---------------------------------------------------------------------------------
    def initialize(self, pre_trained=None, seed=0):
        """Reference odtk/model.py:79-123.  `pre_trained`: a checkpoint file written by `save` (or by the reference):
        every weight except the class head's last layer (and, rotated, the box head's) is taken from it -- fine-tuning, as
        the reference does; those layers get the prior initialisation.  Otherwise seeded random init (no ImageNet
        backbone checkpoints exist offline)."""
        sd = make_state_dict(self.backbone, self.classes, self.num_anchors, self.rotated_bbox, seed)
        if pre_trained:
            if not os.path.isfile(pre_trained):
                raise ValueError('No checkpoint {}'.format(pre_trained))
            chk = torch.load(pre_trained, map_location="cpu", weights_only=False)
            ignored = ['cls_head.8.bias', 'cls_head.8.weight']
            if self.rotated_bbox:
                ignored += ['box_head.8.bias', 'box_head.8.weight']
            sd.update({k: v for k, v in chk['state_dict'].items() if k not in ignored and k in sd})
        self.load_state_dict(sd)
        return self

    # ---- checkpoint files (reference odtk/model.py:217-258: same dict layout, readable by either side) ---------
    def save(self, state):
        checkpoint = {'backbone': [self.backbone], 'classes': self.classes, 'state_dict': self.state_dict(),
                      'ratios': self.ratios, 'scales': self.scales}
        if self.rotated_bbox and self.angles:
            checkpoint['angles'] = self.angles
        for key in ('iteration', 'optimizer', 'scheduler'):
            if key in state:
                checkpoint[key] = state[key]
        torch.save(checkpoint, state['path'])

    @classmethod
    def load(cls, filename, rotated_bbox=False):
        if not os.path.isfile(filename):
            raise ValueError('No checkpoint {}'.format(filename))
        checkpoint = torch.load(filename, map_location="cpu", weights_only=False)
        kwargs = {k: checkpoint[k] for k in ('ratios', 'scales', 'angles') if k in checkpoint}
        if ('angles' in checkpoint) or rotated_bbox:
            kwargs['rotated_bbox'] = True
        model = cls(backbones=checkpoint['backbone'], classes=checkpoint['classes'], **kwargs)
        model.load_state_dict(checkpoint['state_dict'])
        state = {key: checkpoint[key] for key in ('iteration', 'optimizer', 'scheduler') if key in checkpoint}
        return model, state

    def state_dict(self):
        """The reference's state_dict (CPU fp32 tensors); trained head parameters are copied in first."""
        self._params_to_sd()
        return self._sd

    def load_state_dict(self, sd):
        need = [n + ".weight" for n, _, _ in conv_specs(self.backbone, self.classes, self.num_anchors, self.rotated_bbox)]
        missing = [k for k in need if k not in sd]
        if missing:
            raise RuntimeError("missing keys in state_dict: %s" % missing[:4])
        self._sd = {k: v.detach().float().cpu() for k, v in sd.items() if torch.is_tensor(v)}
        self._packed = None
        self._f32 = None
        if self._params is not None:       # as nn.Module: the existing parameter tensors take the new values in place
            with torch.no_grad():
                for n, p in self._params.items():
                    p.copy_(self._sd[n])
            self._param_versions = {}
            self._sd_versions = {n: p._version for n, p in self._params.items()}
        return self

    # ---- trainable parameters ---------------------------------------------------------------------------------------
    def _head_param_names(self):
        return ["%s.%d.%s" % (head, i, k) for head in ("cls_head", "box_head") for i in (0, 2, 4, 6, 8) for k in ("weight", "bias")]

    def _fpn_param_names(self):
        return ["backbones.%s.%s.%s" % (self.backbone, l, k) for l in FPN_LAYERS for k in ("weight", "bias")]

    def _param_names(self):
        """The training scope's parameter names in the reference's named_parameters() order: the FPN's before the heads'."""
        return (self._fpn_param_names() if self.train_scope == "fpn" else []) + self._head_param_names()

    def _trainable_layers(self):
        """(packed-layer key, index in a head list or None, stride, weight name, bias name) of every layer whose
        parameters exist, the FPN's before the heads'."""
        walk = self._walk
        layers = [(l, None, walk[l]) for l in FPN_LAYERS if l in walk]
        layers += [(head, k, c) for head in calib.HEADS for k, c in enumerate(walk[head])]
        return [(key, k, c["stride"], c["conv"] + ".weight", c["conv"] + ".bias") for key, k, c in layers
                if self._params is not None and c["conv"] + ".weight" in self._params]

    def set_train_scope(self, scope):
        """What training updates: "heads" (default: the class and box heads, the backbone and the FPN frozen) or "fpn"
        (the FPN's 16 tensors as well; ResNet18/34/50/101/152 and ResNeXt FPNs -- not MobileNetV2FPN, whose 64-channel
        padded C3 does not fit the weight-gradient GEMM's 128-channel tiles).  named_parameters / parameters list the
        scope's tensors, so build the optimizer after this call.  A parameter keeps its identity across scope changes.
        Returns self."""
        if scope not in ("heads", "fpn"):
            raise ValueError("training scope must be 'heads' or 'fpn', got %r" % (scope,))
        if scope == "fpn" and self.backbone in MOBILENET:
            raise ValueError("the fpn training scope needs C3 with a multiple of 128 channels; %s's padded C3 has 64 channels"
                             % self.backbone)
        self.train_scope = scope
        return self

    def named_parameters(self, prefix="", recurse=True):
        """(name, parameter) of the training scope (set_train_scope), with the reference's names, shapes and order: the
        default scope "heads" lists cls_head.{0,2,4,6,8}.{weight,bias}, then box_head.*; scope "fpn" lists
        backbones.<backbone>.{lateral3,lateral4,lateral5,pyramid6,pyramid7,smooth3,smooth4,smooth5}.{weight,bias} first.
        fp32 CUDA leaf tensors, created from the state dict on first request (after .cuda()).  The backbone is frozen: it
        has no backward kernels here and is never listed.  Once the parameters exist, the training-mode forward returns
        losses connected to them (the backward runs on the sm_90a kernels: odtk_conv_wgrad, odtk_conv_wgrad_ex,
        odtk_conv2d_dgrad, odtk_pool_add_f16, odtk_dilate_f16), and every forward uses their current values (the fp16
        weights are repacked when a parameter changed, e.g. after optimizer.step())."""
        names = self._param_names()
        if self._params is None or any(n not in self._params for n in names):
            if self._packed is None or self.device is None:
                raise RuntimeError("call .cuda() before asking for parameters: they are CUDA tensors")
            if self._params is None:
                self._params = {}
            for n in names:
                if n not in self._params:
                    self._params[n] = torch.nn.Parameter(self._sd[n].to(self.device, torch.float32).clone())
                    self._sd_versions[n] = self._params[n]._version
            for _, _, _, wn, bn in self._trainable_layers():
                if wn not in self._param_versions:      # the packed layer holds the state dict's values
                    self._param_versions[wn] = (self._params[wn]._version, self._params[bn]._version)
        for n in names:
            yield prefix + n, self._params[n]

    def parameters(self, recurse=True):
        for _, p in self.named_parameters():
            yield p

    def zero_grad(self, set_to_none=True):
        for p in self.parameters():
            if set_to_none:
                p.grad = None
            elif p.grad is not None:
                p.grad.zero_()

    def _params_to_sd(self):
        """Copy every parameter that changed since its last copy into the state dict (read by state_dict(), save()
        and the fp32 / INT8 weight packing)."""
        if self._params is not None:
            for n, p in self._params.items():
                if self._sd_versions.get(n) != p._version:
                    self._sd[n] = p.detach().float().cpu().clone()
                    self._sd_versions[n] = p._version

    def _sync_params(self):
        """Repack the fp16 weights of every head or FPN layer whose parameters changed since they were packed (then the
        fp32 weights are dropped, the INT8 network is rebuilt and CUDA graphs are recaptured); counts the forward pass."""
        self._fwd_gen += 1
        if self._params is None or self._packed is None:
            return
        P, changed = self._packed, False
        for key, k, stride, wn, bn in self._trainable_layers():
            w, b = self._params[wn], self._params[bn]
            v = (w._version, b._version)
            if self._param_versions.get(wn) != v:
                with torch.no_grad():
                    conv = _Conv(w.detach(), b.detach().clone(), stride, self.device)
                if k is None:
                    P[key] = conv
                else:
                    P[key][k] = conv
                self._param_versions[wn] = v
                changed = True
        if changed:
            self._f32 = None
            if self._int8 is not None:
                self._params_to_sd()
                self._pack_int8()
            if getattr(self, "_graphs", None):
                self._graphs = {}

    def cuda(self, device=None):
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self._params_to_sd()
        self._pack()
        return self

    def to(self, *args, **kwargs):   # memory_format / dtype arguments of the reference call sites are accepted
        for a in args:
            if isinstance(a, (str, torch.device)) and str(a).startswith("cuda"):
                return self.cuda(torch.device(a).index)
        return self

    def eval(self):
        self.training = False
        return self

    def train(self, mode=True):
        """Training-mode forward (odtk/model.py:130-138): `model([images, targets])` returns (cls_loss, box_loss).  Once
        the parameters of the training scope exist (set_train_scope, then named_parameters / parameters), the losses are
        connected to them and .backward() fills their .grad on the sm_90a backward kernels: the heads, and in scope "fpn"
        the FPN too; the backbone is frozen (no backward kernels).  An INT8 network table calibrated before training
        describes the old weights: recalibrate after training.
        Without them, the losses and -- `_compute_loss(..., with_grad=True)` -- their gradients w.r.t. the head outputs
        are what this provides.  The training forward runs in fp16 over the pyramid atlas whatever set_precision chose."""
        self.training = bool(mode)
        return self

    def share_memory(self):
        return self

    def _pack(self):
        self._f32 = None
        sd, dev = self._sd, self.device
        if self.backbone in MOBILENET:
            P = {}
            self._pack_mobilenet(P)
        else:
            P = pack_walk(network_walk(self.backbone),
                          lambda c: _Conv(*walk_weights(sd, c), c["stride"], dev, c["groups"]))
        self._packed = P
        self._pack_int8()

    def _pack_int8(self):
        """The INT8 network (set_precision("int8")): the fp16 layers with s8 ones in place of the layers `int8_scope` runs on
        the s8 tensor cores -- the 10 head layers, and in scope "network" layer3, layer4 and the FPN too.  Every s8
        convolution reads a tensor quantised with the scale of its table entry and requantises its output with the scale of
        its own (calib.network_tensors); residual / upsample addends are dequantised with the scale of the tensor they are;
        the smooth and pyramid convolutions write the s8 atlas with the "heads.input" scale.  Also the inverse scales of
        the two fp16 -> s8 quantisations: C3 (network scope) and the atlas (heads scope)."""
        self._int8 = None
        if self._int8_table is None or self.device is None:
            return
        self._params_to_sd()              # trained parameters
        S, sd, dev = self._int8_table["scales"], self._sd, self.device
        names = calib.table_tensors(self.backbone, self.int8_scope)
        walk = network_walk(self.backbone)
        if self.int8_scope == "heads":
            walk = {h: walk[h] for h in calib.HEADS}

        def s32(name):
            return np.float32(S[name]) if name is not None and name in S else None

        def make(c):
            if c["x"] not in names:
                return None
            res, up = s32(c.get("res")), s32(c.get("up"))
            return _ConvS8(*walk_weights(sd, c), s32(c["x"]), s32(c["y"]), c["stride"], dev,
                           float(res) if res is not None else None, float(up) if up is not None else None)

        N = dict(self._packed)
        for k, v in pack_walk(walk, make).items():
            if k == "blocks":
                N[k] = [b8 if b8["convs"][0] is not None else b16 for b16, b8 in zip(N[k], v)]
            elif v is not None:
                N[k] = v
        N["inv_in"] = float(np.float32(1.0) / np.float32(S["heads.input"]))
        if self.int8_scope == "network":
            N["inv_c3"] = float(np.float32(1.0) / s32("backbones.%s.features.layer2" % self.backbone))
        self._int8 = N

    def _f32_layers(self):
        """Full precision: every convolution of the ResNet backbone, the FPN and the heads with BatchNorm folded in fp32,
        packed on first use."""
        if self._f32 is None:
            self._params_to_sd()          # trained head parameters
            sd, dev = self._sd, self.device
            self._f32 = pack_walk(network_walk(self.backbone),
                                  lambda c: _ConvF32(*walk_weights(sd, c), c["stride"], dev, stem=c["x"] == "input"))
        return self._f32

    def _stem_dtype(self):
        """The precision decision: fp32 activations from the stem input on (set_precision("fp32"), inference only), else
        fp16 (the training-mode forward is always fp16)."""
        return torch.float32 if self.precision == "fp32" and not self.training else torch.float16

    def _net(self):
        """The packed layers the forward runs: fp32, the INT8 network (inference only) or fp16."""
        if self._stem_dtype() == torch.float32:
            return self._f32_layers()
        if self._int8 is not None and not self.training:
            return self._int8
        return self._packed

    def set_precision(self, precision, table=None, scope="heads"):
        """"fp16" (default), "fp32" or "int8".  "fp32" (full precision, the reference's --full-precision): fp32
        activations end to end and every convolution on split-TF32 tensor-core products (odtk_conv2d_f32); its head outputs
        are within 1e-4 - 2.3e-4 * max|ref| of fp32 PyTorch (measured on the H100) instead of fp16's 1.4e-3 - 2.1e-3 --
        ResNet18/34/50/101/152FPN (not ResNeXt or
        MobileNetV2); the fused stem-pool and bottleneck kernels are not
        used, and the split weights are packed on the first fp32 forward.  "int8": the head towers and the two final head layers run on the s8 tensor cores with the
        activation scales of `table` (a path or a dict, from `calibrate`).  scope "heads" (default): the backbone and the
        FPN stay fp16; "network" (a table from calibrate(..., scope="network")): ResNet layer3, layer4 and the FPN run in
        INT8 too, from layer2's output quantised once, and the FPN writes the s8 atlas the heads read -- the stem, layer1 and
        layer2 stay fp16 (ResNet18/34/50/101/152 backbones; ResNeXt and MobileNetV2 take "heads" only).  The training-mode
        forward stays fp16.  Captured CUDA graphs are dropped."""
        if precision == "fp16":
            self._int8_table = None
            self._int8 = None
            self.int8_scope = "heads"
        elif precision == "fp32":
            if self.backbone not in FP32_BACKBONES:
                raise ValueError("full precision covers %s, not %s" % (", ".join(FP32_BACKBONES), self.backbone))
            self._int8_table = None
            self._int8 = None
            self.int8_scope = "heads"
        elif precision == "int8":
            if table is None:
                raise ValueError("set_precision('int8') needs a calibration table (Model.calibrate)")
            if scope == "network":
                calib.network_tensors(self.backbone)            # ValueError for the backbones the scope does not cover
            self._int8_table = calib.check_table(calib.load_table(table), self.backbone, self.classes, self.num_anchors, scope)
            self.int8_scope = scope
            if self._packed is not None:
                self._pack_int8()
        else:
            raise ValueError("precision must be 'fp16', 'fp32' or 'int8', got %r" % (precision,))
        if precision != "fp32":
            self._f32 = None
        self.precision = precision
        if getattr(self, "_graphs", None):
            self._graphs = {}
        return self

    def calibrate(self, batches, table=None, method="entropy", scope="heads"):
        """INT8 calibration: eager fp16 forwards over `batches` (each one what `forward` takes) record, for the 9 tensors the
        INT8 heads quantise (calib.TENSORS), max|x| and then a 2048-bin |x| histogram over the valid atlas pixels (the gap
        rows / columns are left out).  method "max": threshold max|x|; "entropy": TensorRT's KL-divergence search.
        scope "network" also records every tensor of layer3, layer4 and the FPN that scope quantises
        (calib.network_tensors) and returns a format-2 table; its 9 head scales are those scope "heads" finds.  Runs on
        the fp16 network, as TensorRT's calibrator does.  Returns the calibration table and, if `table` is a path, writes it
        there."""
        if self._packed is None:
            raise RuntimeError("call .cuda() after loading weights: there is no CPU path")
        if method not in ("max", "entropy"):
            raise ValueError("unknown calibration method %r (max, entropy)" % (method,))
        if scope not in calib.SCOPES:
            raise ValueError("INT8 scope must be 'heads' or 'network', got %r" % (scope,))
        names = calib.table_tensors(self.backbone, scope)
        batches = list(batches)
        col = calib.Collector()
        saved = (self._int8, self.parallel_heads, self.training, self.precision)
        self._int8, self.parallel_heads, self.training = None, False, False
        self.precision = "fp16" if self.precision == "fp32" else self.precision
        self._calib_hook = col.observe
        self._calib_net = scope == "network"
        images = 0
        try:
            with torch.no_grad():
                for phase in ((0, 1) if method == "entropy" else (0,)):
                    col.phase = phase
                    for x in batches:
                        x = x.to(self.device)
                        if x.dtype == torch.uint8:
                            self.forward_heads_u8(x)
                        else:
                            self.forward_heads(x)
                        images += x.shape[0] if phase == 0 else 0
            torch.cuda.synchronize()
        finally:
            self._int8, self.parallel_heads, self.training, self.precision = saved
            self._calib_hook = None
            self._calib_net = False
        t = calib.make_table(self.backbone, self.classes, self.num_anchors, method, images, col.scales(method, names), scope)
        if table is not None:
            calib.save_table(t, table)
        return t

    def _pack_mobilenet(self, P):
        """MobileNetV2FPN (odtk/backbones/mobilenet.py, fpn.py:92-93).  The tensor-core kernels work on 64-channel K
        blocks: every activation is carried with its channel count padded to a multiple of 64 (zero weights / zero bias in
        the padding, so the padding stays exactly 0 through ReLU6 and the residual adds)."""
        sd, dev = self._sd, self.device
        f = "backbones.%s.features.features." % self.backbone

        def up64(c):
            return (c + 63) // 64 * 64

        def fold(pc, pb):
            return engine.fold_bn(sd[pc + ".weight"], sd[pb + ".weight"], sd[pb + ".bias"], sd[pb + ".running_mean"], sd[pb + ".running_var"])

        def padded_conv(w, b, stride=1, pad_in=True):
            cout, cin = w.shape[0], w.shape[1]
            wp = w.new_zeros((up64(cout), up64(cin) if pad_in else cin, w.shape[2], w.shape[3]))
            wp[:cout, :cin] = w
            bp = b.new_zeros(up64(cout))
            bp[:cout] = b
            return _Conv(wp, bp, stride, dev)

        P["stem"] = padded_conv(*fold(f + "0.0", f + "0.1"), stride=2, pad_in=False)       # 3x3 s2, 3 -> 32: receptive-field gather + GEMM
        blocks = []
        for idx, cin, cout, stride, t in mobilenet_blocks(self.backbone):
            p, k = f + "%d.conv." % idx, 0
            blk = {"idx": idx, "stride": stride, "res": stride == 1 and cin == cout, "expand": None}
            if t != 1:
                blk["expand"] = padded_conv(*fold(p + "0.0", p + "0.1"))
                k = 1
            wd, bd = fold(p + "%d.0" % k, p + "%d.1" % k)                                 # depthwise [hidden, 1, 3, 3]
            hidden = wd.shape[0]
            wdp = wd.new_zeros((9, up64(hidden)))
            wdp[:, :hidden] = wd.reshape(hidden, 9).t()
            bdp = bd.new_zeros(up64(hidden))
            bdp[:hidden] = bd
            blk["dw_w"], blk["dw_b"] = wdp.to(torch.float16).contiguous().to(dev), bdp.float().contiguous().to(dev)
            blk["hidden"] = hidden
            blk["project"] = padded_conv(*fold(p + "%d" % (k + 1), p + "%d" % (k + 2)))
            blocks.append(blk)
        P["blocks"] = blocks
        n = "backbones.%s." % self.backbone
        for kname in ("lateral3", "lateral4", "lateral5"):
            P[kname] = padded_conv(sd[n + kname + ".weight"], sd[n + kname + ".bias"])
        for kname in ("smooth3", "smooth4", "smooth5"):
            P[kname] = _Conv(sd[n + kname + ".weight"], sd.get(n + kname + ".bias"), 1, dev)
        P["pyramid6"] = _Conv(sd[n + "pyramid6.weight"], sd.get(n + "pyramid6.bias"), 2, dev)
        P["pyramid7"] = _Conv(sd[n + "pyramid7.weight"], sd.get(n + "pyramid7.bias"), 2, dev)
        for head in ("cls_head", "box_head"):
            P[head] = [_Conv(sd["%s.%d.weight" % (head, i)], sd.get("%s.%d.bias" % (head, i)), 1, dev) for i in (0, 2, 4, 6, 8)]

    def _features_mobilenet(self, x):
        """`x`: NHWC fp16 image [N, H, W, 3].  torchvision MobileNetV2.features[0 .. 17] with ReLU6, taps after blocks
        6 / 13 / 17 (odtk/backbones/mobilenet.py:18-25), then the shared FPN."""
        P = self._packed
        x = P["stem"](x, relu=2)
        outs = {}
        for blk in P["blocks"]:
            inp = x
            hcur = blk["expand"](x, relu=2) if blk["expand"] is not None else x
            engine.STATS["conv_flops"] += 2 * hcur.shape[0] * ((hcur.shape[1] - 1) // blk["stride"] + 1) * ((hcur.shape[2] - 1) // blk["stride"] + 1) * blk["hidden"] * 9
            hcur = engine.depthwise3x3(hcur, blk["dw_w"], blk["dw_b"], blk["stride"], act=2)
            x = blk["project"](hcur, relu=False, residual=inp if blk["res"] else None)
            if blk["idx"] in MOBILENET_TAPS:
                outs[blk["idx"]] = x
        return self._fpn(outs[6], outs[13], outs[17])

    # ---- forward ---------------------------------------------------------------------------------
    def _stem(self, x=None, padded=None):
        """conv1 + bn1 + relu + maxpool (odtk/backbones/resnet.py:25-28).  fp16: one fused kernel when the stem has the
        standard 64 output channels and the image size is even; `padded` = (xp, h, w) from engine.preprocess_u8 (fp32: the
        NHWC4 fp32 stem buffer, stem convolution then max-pool)."""
        if self.backbone in MOBILENET:
            if padded is not None:
                raise RuntimeError("the fused uint8 input path feeds the ResNet stem; pass a float / half image to MobileNetV2FPN")
            return x                                        # the 3x3 stem runs inside _features_mobilenet
        stem = self._net()["stem"]
        if padded is not None:
            xp, h, w = padded
            n = xp.shape[0]
        else:
            n, h, w = x.shape[0], x.shape[1], x.shape[2]
        flops = 2 * n * ((h - 1) // 2 + 1) * ((w - 1) // 2 + 1) * stem.cout * 49 * 3
        engine.STATS["conv_flops"] += flops
        if isinstance(stem, _ConvF32):
            return engine.maxpool3x3s2_f32(engine.stem_conv_f32(xp, h, w, stem.hi, stem.lo, stem.b, stem.cout, relu=True))
        fused = stem.stem and stem.cout == 64 and h % 2 == 0 and w % 2 == 0
        if padded is not None:
            if fused:
                return engine.stem_pool_padded(xp, h, w, stem.w_stem, stem.b, stem.cout, relu=True)
            return engine.maxpool3x3s2(engine.stem_conv_padded(xp, h, w, stem.w_stem, stem.b, stem.cout, relu=True))
        if fused:
            return engine.stem_pool(x, stem.w_stem, stem.b, stem.cout, relu=True)
        engine.STATS["conv_flops"] -= flops      # _Conv.__call__ counts it
        return engine.maxpool3x3s2(stem(x, relu=True))

    def _features_of(self, x):
        """(pyramid level views, (h, w)) of an NCHW float batch, or of a uint8 HWC batch normalised and stride-padded on the
        GPU (h, w: the padded size): the stem input of the current precision."""
        f32 = self._stem_dtype() == torch.float32
        if x.dtype == torch.uint8:
            xp, hs, ws = (engine.preprocess_u8_f32 if f32 else engine.preprocess_u8)(x, self.stride)
            return self._features(self._stem(padded=(xp, hs, ws))), (hs, ws)
        if f32:
            if x.dim() != 4:
                raise ValueError("expected a [B, 3, H, W] batch")
            xp = engine.pad_input_f32(x.permute(0, 2, 3, 1).contiguous().float())
            return self._features(self._stem(padded=(xp, x.shape[2], x.shape[3]))), (x.shape[2], x.shape[3])
        return self._features(self._stem(self._to_nhwc_half(x))), (x.shape[2], x.shape[3])

    def _features(self, x, keep=None):
        """`x`: the POOLED stem output [N, H/4, W/4, C] (from _stem).  The residual blocks, then the FPN (`keep`: see _fpn).  fp16 blocks whose
        shapes fit take the fused bottleneck kernels; every other block runs its downsample, then its convolutions with
        the residual added in the last one's epilogue.  The INT8 network quantises C3 once, at its first s8 block."""
        if self.backbone in MOBILENET:
            return self._features_mobilenet(x)
        P = self._net()
        outs = {}
        blocks = P["blocks"]
        hook = self._calib_hook if self._calib_net else None     # network-scope calibration: layer3 / layer4 tensors
        z_next = None                 # conv1 of THIS block, already computed by the previous block's fused tail (GEMM3)
        for bi, blk in enumerate(blocks):
            cs = blk["convs"]
            dn = blk["down"]
            if isinstance(cs[0], _ConvS8) and x.dtype == torch.float16:
                x = outs[3] = engine.quantize_f16_s8(x, P["inv_c3"])
            fp16 = isinstance(cs[0], _Conv)
            tap = hook if blk["level"] >= 4 else None
            z_in, z_next = z_next, None
            if (fp16 and dn is not None and len(cs) == 3 and dn.ks == 1 and dn.stride == 1 and dn.cin == 64 and
                    dn.groups == 1 and cs[1].stride == 1 and cs[1].groups == 1 and cs[1].ks == 3 and cs[1].cin == 64 and
                    cs[1].cout == 64 and cs[2].cin == 64 and cs[2].cout == dn.cout and dn.cout % 128 == 0 and dn.cout <= 512):
                # first block of layer1: conv2 + conv3 + the 1x1 PROJECTION of the block input (torchvision `downsample`)
                # + ReLU in one kernel: the 3x3's output stays in shared memory, the projected identity is one more K block
                # of the 1x1's fp32 accumulator
                if "b3d" not in blk:
                    blk["b3d"] = (cs[2].b + dn.b).contiguous()
                out = cs[0](x, relu=True)
                px = out.shape[0] * out.shape[1] * out.shape[2]
                engine.STATS["conv_flops"] += 2 * px * (64 * (9 * 64 + cs[2].cout) + 64 * dn.cout)
                x = engine.bottleneck_tail(out, cs[1].w, cs[1].b, cs[2].w, blk["b3d"], None, relu=True, xproj=x, wproj=dn.w)
                if blk["last"]:
                    outs[blk["level"]] = x
                continue
            identity = x if dn is None else dn(x)
            if tap is not None and dn is not None:
                tap(blk["name"] + ".downsample", identity)
            if (fp16 and tap is None and len(cs) == 3 and cs[1].stride == 1 and cs[1].groups == 1 and cs[1].ks == 3 and
                    cs[1].cin in (64, 128) and cs[1].cout == cs[1].cin and cs[2].cin == cs[1].cin and cs[2].cout % 128 == 0 and
                    cs[2].cout <= 512):
                # conv2 (3x3) + conv3 (1x1) + identity + ReLU in one kernel: the 3x3's output never leaves the SM
                out = z_in if z_in is not None else cs[0](x, relu=True)
                px = out.shape[0] * out.shape[1] * out.shape[2]
                engine.STATS["conv_flops"] += 2 * px * cs[1].cin * (9 * cs[1].cin + cs[2].cout)
                # GEMM3: the NEXT block's conv1 (1x1, C2 -> 64 / 128, + ReLU) from this block's output while it is still in
                # shared memory -- removes a full read of the widest tensor of the level
                nxt = blocks[bi + 1]["convs"] if bi + 1 < len(blocks) else None
                if (cs[1].cin == 64 and nxt is not None and len(nxt) == 3 and isinstance(nxt[0], _Conv) and nxt[0].ks == 1 and
                        nxt[0].stride == 1 and nxt[0].groups == 1 and nxt[0].cin == cs[2].cout and nxt[0].cout in (64, 128) and
                        nxt[0].b is not None):
                    engine.STATS["conv_flops"] += 2 * px * nxt[0].cin * nxt[0].cout
                    x, z_next = engine.bottleneck_tail(out, cs[1].w, cs[1].b, cs[2].w, cs[2].b, identity, relu=True,
                                                       w_next=nxt[0].w, b_next=nxt[0].b)
                else:
                    x = engine.bottleneck_tail(out, cs[1].w, cs[1].b, cs[2].w, cs[2].b, identity, relu=True)
            else:
                out = z_in if z_in is not None else x
                for k, c in enumerate(cs[1:-1] if z_in is not None else cs[:-1]):
                    out = c(out, relu=True)
                    if tap is not None:
                        tap("%s.conv%d" % (blk["name"], k + 1), out)
                x = cs[-1](out, relu=True, residual=identity)
            if tap is not None:
                tap(blk["name"], x)
            if blk["last"]:
                outs[blk["level"]] = x
        if hook is not None:
            hook("backbones.%s.features.layer2" % self.backbone, outs[3])
        return self._fpn(outs[3], outs[4], outs[5], keep)

    def _fpn(self, c3, c4, c5, keep=None):
        """FPN (odtk/backbones/fpn.py:45-61) on the three backbone taps, into the pyramid atlas: the five levels stacked in
        ONE zero-separated NHWC buffer of the activation dtype, so that every head-tower layer is one launch over all
        levels instead of five.  Returns the five level views; a `keep` dict receives what the FPN backward reads: c3-c5,
        the pre-smooth p3-p5 and relu(P6)."""
        P = self._net()
        p5 = P["lateral5"](c5)
        p4 = P["lateral4"](c4, upsample=p5)
        p3 = P["lateral3"](c3, upsample=p4)
        if self._calib_net:
            for k, t in ((5, p5), (4, p4), (3, p3)):
                self._calib_hook("backbones.%s.lateral%d" % (self.backbone, k), t)
        n = c5.shape[0]
        h6, w6 = (c5.shape[1] - 1) // 2 + 1, (c5.shape[2] - 1) // 2 + 1
        sizes = ((p3.shape[1], p3.shape[2]), (p4.shape[1], p4.shape[2]), (p5.shape[1], p5.shape[2]), (h6, w6),
                 ((h6 - 1) // 2 + 1, (w6 - 1) // 2 + 1))
        at = self._atlas_for(n, sizes, c5.device)
        v = [engine.AtlasView(self._atlas_bufs(at, p3.dtype)[0], r, h, w) for r, (h, w) in zip(at["rows"], sizes)]
        P["smooth3"](p3, out=v[0])
        P["smooth4"](p4, out=v[1])
        P["smooth5"](p5, out=v[2])
        P["pyramid6"](c5, out=v[3])
        r6 = engine.relu_from_view(v[3])
        P["pyramid7"](r6, out=v[4])
        if keep is not None:
            keep.update(c3=c3, c4=c4, c5=c5, p3=p3, p4=p4, p5=p5, r6=r6)
        return v

    def _atlas_for(self, n, sizes, device):
        """Geometry + persistent, zero-initialised buffers of the pyramid atlas for one batch size / level geometry.
        Level l occupies rows [rows[l], rows[l] + h_l) x columns [0, w_l); level starts are multiples of 8 (the tile
        height) with at least one gap row in between; gap rows / columns are never written and stay zero (they ARE the
        convolutions' zero padding between levels).  tab: every 8 x 16 tile of one image as (row0, col0, row_limit,
        col_limit), ordered by level; tabs: each level's contiguous slice of it."""
        key = (n, sizes, str(device))
        at = self._atlas.get(key)
        if at is None:
            rows, r = [], 0
            for (h, w) in sizes:
                rows.append(r)
                r = (r + h + 1 + 7) // 8 * 8
            ha, wa = rows[-1] + sizes[-1][0], max(w for _, w in sizes)
            tiles = [(r0 + 8 * ty, 16 * tx, r0 + h, w) for (h, w), r0 in zip(sizes, rows)
                     for ty in range((h + 7) // 8) for tx in range((w + 15) // 16)]
            tab = torch.tensor(tiles, dtype=torch.int32, device=device)
            starts = np.cumsum([0] + [((h + 7) // 8) * ((w + 15) // 16) for h, w in sizes]).tolist()
            at = {"rows": rows, "ha": ha, "wa": wa, "px": n * sum(h * w for h, w in sizes), "tab": tab,
                  "tabs": [tab[starts[l]:starts[l + 1]] for l in range(len(sizes))],
                  "buf": [torch.zeros((n, ha, wa, 256), dtype=torch.float16, device=device) for _ in range(5)]}
            self._atlas[key] = at
        return at

    @staticmethod
    def _atlas_bufs(at, dtype):
        """The five buffers of an atlas geometry in `dtype`: at["buf"] for fp16, int8 (INT8) and fp32 (full precision) ones
        zero-initialised on first use."""
        if dtype == torch.float16:
            return at["buf"]
        key = "buf_" + str(dtype).split(".")[-1]
        if key not in at:
            buf = at["buf"][0]
            at[key] = [torch.zeros(buf.shape, dtype=dtype, device=buf.device) for _ in range(5)]
        return at[key]

    def _heads(self, features, sigmoid=True, sinks=None):
        """Class / box heads on the five levels of the pyramid atlas (odtk/model.py:134-135)."""
        return self._heads_atlas(features, engine.OUT_NCHW_F32_SIGMOID if sigmoid else engine.OUT_NCHW_F32, sinks)

    def _heads_atlas(self, views, cls_mode, sinks):
        """Heads over the pyramid atlas: each of the 4 + 4 tower layers is ONE launch over all five levels (a tile table
        lists the 8 x 16 tiles of every level; weights are shared between levels anyway, odtk/model.py:134-135); the
        two final layers run per level on views of the last tower output (their outputs are per-level tensors).  The class
        and the box tower are independent: two streams / two graph branches.  INT8 heads on an fp16 atlas quantise it
        once, on the main stream before the fork."""
        P = self._net()
        atlas0 = views[0].atlas
        sizes = tuple((v.h, v.w) for v in views)
        at = self._atlas_for(atlas0.shape[0], sizes, atlas0.device)
        hook = self._calib_hook
        if hook is not None:              # calibration: the valid atlas pixels of the heads' input and of every tower output
            if "valid" not in at:
                valid = torch.zeros(atlas0.shape[1:3], dtype=torch.bool, device=atlas0.device)
                for r, (h, w) in zip(at["rows"], sizes):
                    valid[r:r + h, :w] = True
                at["valid"] = valid
            hook("heads.input", atlas0[:, at["valid"]])
        if isinstance(P["cls_head"][0], _ConvS8) and atlas0.dtype == torch.float16:
            atlas0 = engine.quantize_f16_s8(atlas0, P["inv_in"], out=self._atlas_bufs(at, torch.int8)[0])
        bufs = self._atlas_bufs(at, atlas0.dtype)

        def tower(head, bufs, final_mode, use_sinks):
            t = atlas0
            for i, conv in enumerate(P[head][:-1]):
                nxt = bufs[i & 1]
                conv(t, relu=True, out=nxt, tile_tab=at["tab"], valid_px=at["px"])
                if hook is not None:
                    hook("%s.%d" % (head, 2 * i), nxt[:, at["valid"]])
                t = nxt
            outs = []
            for l, v in enumerate(views):
                lv = engine.AtlasView(t, at["rows"][l], v.h, v.w)
                if use_sinks is not None:
                    outs.append(P[head][-1](lv, out_mode=engine.OUT_CANDIDATES, sink=use_sinks[l]))
                else:
                    outs.append(P[head][-1](lv, out_mode=final_mode))
            return outs

        if not self.parallel_heads:
            cls_heads = tower("cls_head", bufs[1:3], cls_mode, sinks)
            box_heads = tower("box_head", bufs[3:5], engine.OUT_NCHW_F32, None)
            return cls_heads, box_heads
        main = torch.cuda.current_stream()
        if self._head_streams is None:
            self._head_streams = [torch.cuda.Stream(device=self.device)]
        side = self._head_streams[0]
        fork = torch.cuda.Event()
        fork.record(main)
        side.wait_event(fork)
        with torch.cuda.stream(side):
            box_heads = tower("box_head", bufs[3:5], engine.OUT_NCHW_F32, None)
            join = torch.cuda.Event()
            join.record(side)
        cls_heads = tower("cls_head", bufs[1:3], cls_mode, sinks)
        main.wait_event(join)
        return cls_heads, box_heads

    @staticmethod
    def _to_nhwc_half(x):
        if x.dim() != 4:
            raise ValueError("expected a [B, 3, H, W] batch")
        return x.permute(0, 2, 3, 1).contiguous().to(torch.float16)   # zero-copy for channels_last fp16

    def forward_heads_u8(self, images, sigmoid=True):
        """Input side of `odtk infer` fused in: `images` is a uint8 HWC batch
        [B, H, W, 3]; normalisation, stride padding (odtk/data.py:113-123) and the stem's zero border are one
        kernel that writes the stem's input buffer directly."""
        if self._packed is None:
            raise RuntimeError("call .cuda() after loading weights: there is no CPU path")
        features, size = self._features_of(images)
        return self._heads(features, sigmoid), size

    def forward_heads(self, x, sigmoid=True):
        """The `exporting=True` view of the reference (odtk/model.py:142-144): per-level
        (sigmoid) class maps [B, A*C, H, W] and box maps [B, A*4|6, H, W], fp32 NCHW."""
        if self._packed is None:
            raise RuntimeError("call .cuda() after loading weights: there is no CPU path")
        self._sync_params()
        return self._heads(self._features_of(x)[0], sigmoid)

    def _level_anchors(self, widths, width):
        strides, anchors = [], []
        for w in widths:
            stride = width // w                            # width only (odtk/model.py:155)
            if stride not in self.anchors:
                self.anchors[stride] = (box.generate_anchors_rotated(stride, self.ratios, self.scales, self.angles)
                                        if self.rotated_bbox else box.generate_anchors(stride, self.ratios, self.scales))
            a = self.anchors[stride][0] if self.rotated_bbox else self.anchors[stride]
            strides.append(stride)
            anchors.append(a.reshape(-1).tolist())
        return strides, anchors

    def _forward_fused(self, x):
        """Inference branch with the class head's last convolution appending its above-threshold scores
        directly to the decode workspace (odtk_decode_fused_begin/_finish): the dense [B, A*C, H, W] score maps
        of odtk/model.py:140 are never written or re-read.  Same detections as the dense route."""
        if self._packed is None:
            raise RuntimeError("call .cuda() after loading weights: there is no CPU path")
        features, (_, width) = self._features_of(x)
        return self._detect_fused(features, width)

    def _detect_fused(self, features, width):
        sizes = tuple((f.shape[1], f.shape[2]) for f in features)
        batch = features[0].shape[0]
        key = (batch, sizes, width, self.threshold, self.top_n, self.rotated_bbox)
        fd = self._fused.get(key)
        if fd is None:
            strides, anchors = self._level_anchors([s[1] for s in sizes], width)
            num_anchors = len(anchors[0]) // 4
            fd = self._fused[key] = _C.FusedDecode(batch, sizes, num_anchors, self.classes, anchors, strides,
                                                   self.threshold, self.top_n, self.rotated_bbox, features[0].device)
        sinks = fd.begin()
        _, box_heads = self._heads(features, True, sinks)
        return self._nms(fd.finish(box_heads))

    def _nms(self, decoded):
        """box.nms / nms_rotated (odtk/model.py:162-165) + the packed [B, D, 2 + nbox] rows (self.last_packed) and, when a
        PeerGather is attached, the exchange with the other ranks -- all in the one NMS launch."""
        b = decoded[0].shape[0]
        key = (b, self.detections, self.rotated_bbox, decoded[0].device)
        packed = self._packed_out.get(key)
        if packed is None:
            packed = self._packed_out[key] = torch.empty((b, self.detections, 2 + (6 if self.rotated_bbox else 4)),
                                                         dtype=torch.float32, device=decoded[0].device)
        self.last_packed = packed
        return tuple(_C.nms(*decoded, self.nms, self.detections, self.rotated_bbox, packed=packed, gather=self.gather))

    def attach_gather(self, gather):
        """Image-wise sharded inference: every forward also delivers this rank's detections to all ranks
        (peer.PeerGather.gathered()).  Attach BEFORE the CUDA graph of a shape is captured."""
        self.gather = gather
        if getattr(self, "_graphs", None):
            self._graphs = {}
        return self

    # ---- training-side losses (reference odtk/model.py:167-210) ---------------------------------------------------
    def _extract_targets(self, targets, stride, size):
        """Per level: class-index targets [B, A, H, W] int32, box targets [B, A, nbox, H, W], depth [B, A, 1, H, W].
        Axis-aligned: the whole batch in one launch (odtk_snap_to_anchors); rotated: per image, polygon IoUs on
        odtk_iou (odtk/model.py:167-184)."""
        if stride not in self.anchors:
            self.anchors[stride] = (box.generate_anchors_rotated(stride, self.ratios, self.scales, self.angles)
                                    if self.rotated_bbox else box.generate_anchors(stride, self.ratios, self.scales))
        anchors = self.anchors[stride]
        h, w = int(size[0]), int(size[1])
        if not self.rotated_bbox:
            _, box_target, depth, cls_index = box.snap_to_anchors_batch(targets, (h, w), stride, anchors, self.classes,
                                                                        self.anchor_ious, dense=False)
            return cls_index, box_target, depth
        bts, dps = [], []
        for target in targets:
            target = target[target[:, -1] > -1]
            _, bt, dp = box.snap_to_anchors_rotated(target, [w * stride, h * stride], stride, anchors, self.classes,
                                                    targets.device, self.anchor_ious)
            bts.append(bt)
            dps.append(dp)
        box_target, depth = torch.stack(bts), torch.stack(dps)
        d = depth[:, :, 0]
        cls_index = torch.where(d > 0, d - 1, torch.where(d == 0, torch.full_like(d, -1), torch.full_like(d, -2))).int()
        return cls_index.contiguous(), box_target, depth

    def _compute_loss(self, x, cls_heads, box_heads, targets, with_grad=False):
        """odtk/model.py:186-210: target assignment per level, then ONE fused launch for the focal + smooth-L1 losses of
        all levels, the masks, the foreground counts and the normalisation (loss.retina_loss -> odtk_retina_loss)."""
        from . import loss as loss_mod
        width = x.shape[-1] if torch.is_tensor(x) else int(x)
        cls_idx, box_tgt = [], []
        for cls_head in cls_heads:
            size = cls_head.shape[-2:]
            stride = width // cls_head.shape[-1]
            ci, bt, _ = self._extract_targets(targets, stride, size)
            cls_idx.append(ci)
            box_tgt.append(bt)
        return loss_mod.retina_loss(cls_heads, box_heads, cls_idx, box_tgt, self.classes, with_grad=with_grad)

    # ---- training the heads: forward with saved tower outputs, backward on odtk_conv_wgrad / odtk_conv2d_dgrad ----------
    def _train_forward(self, x, targets):
        """Training forward of the heads over the pyramid atlas with every tower output kept (the inference path
        ping-pongs two buffers) and the loss gradients from the same odtk_retina_loss launch.  Returns the two losses
        and the state the backward needs."""
        if self._packed is None:
            raise RuntimeError("call .cuda() after loading weights: there is no CPU path")
        keep = {} if self.train_scope == "fpn" else None
        views = self._features(self._stem(self._to_nhwc_half(x)), keep)
        P = self._packed
        atlas0 = views[0].atlas
        at = self._atlas_for(atlas0.shape[0], tuple((v.h, v.w) for v in views), atlas0.device)
        if "train" not in at:        # zero-initialised once: gap rows / columns are never written
            at["train"] = {h: [torch.zeros_like(atlas0) for _ in range(4)] for h in ("cls_head", "box_head")}
        outs = {}
        for head in ("cls_head", "box_head"):
            t = atlas0
            for i, conv in enumerate(P[head][:-1]):
                conv(t, relu=True, out=at["train"][head][i], tile_tab=at["tab"], valid_px=at["px"])
                t = at["train"][head][i]
            outs[head] = [P[head][-1](engine.AtlasView(t, at["rows"][l], v.h, v.w), out_mode=engine.OUT_NCHW_F32)
                          for l, v in enumerate(views)]
        cls_loss, box_loss, cls_grads, box_grads = self._compute_loss(x, outs["cls_head"], outs["box_head"], targets,
                                                                      with_grad=True)
        state = {"gen": self._fwd_gen, "at": at, "views": views, "heads": outs, "fpn": keep, "names": self._param_names(),
                 "grads": {"cls_head": cls_grads, "box_head": box_grads}}
        self.last_train = state if self.want_atlas_grad else None
        return cls_loss.clone(), box_loss.clone(), state

    def _train_backward(self, state, g_cls, g_box, needs):
        """Gradients of the training forward's parameters (state["names"]; None where `needs` is False) for upstream
        gradients g_cls / g_box of the two losses.  Per head, from the last layer down: the loss gradients times the
        upstream factor into the fp16 gradient atlas, then per layer the weight / bias gradient (odtk_conv_wgrad) and the
        input gradient masked by the ReLU of the layer's input (odtk_conv2d_dgrad).  The first tower layer's input
        gradient, d(atlas), is only computed when an FPN parameter needs a gradient or want_atlas_grad is set (the box
        tower's with the class tower's as its residual addend); then the FPN backward (_fpn_backward) runs from it."""
        if state["gen"] != self._fwd_gen:
            raise RuntimeError("the model ran another forward pass after this training forward: its saved activations "
                               "are gone; call backward() before the next forward")
        at, tab = state["at"], state["at"]["tab"]
        P = self._packed
        names = state["names"]
        need = dict(zip(names, needs))
        need_fpn = any(need.get(n, False) for n in self._fpn_param_names())
        got = {}
        atlas0 = state["views"][0].atlas
        gbuf = [self._atlas_zeros(at, "gbuf%d" % i) for i in range(4)]    # tower gradient ping-pong + d(atlas) (cls, sum)
        d_atlas = None
        want_atlas = self.want_atlas_grad or need_fpn
        for head, g in (("cls_head", g_cls), ("box_head", g_box)):
            lname = ["%s.%d" % (head, i) for i in (0, 2, 4, 6, 8)]
            needed = [need[n + ".weight"] or need[n + ".bias"] for n in lname]
            if g is None or not (any(needed) or want_atlas):
                continue
            cpad = engine.pad64(P[head][-1].cout)
            G = self._atlas_zeros(at, "grad%d" % cpad, cpad)
            G = engine.grad_to_atlas(state["grads"][head], at["rows"], g, G)   # g stays on the device: no sync
            inputs = [atlas0] + at["train"][head]
            for k in range(4, -1, -1):
                self._wgrad(need, got, lname[k], engine.conv_wgrad, G, inputs[k], P[head][k].cout, tile_tab=tab)
                if not (want_atlas or any(needed[:k])):
                    break
                wpk = self._dgrad_weights(lname[k] + ".weight", cpad if k == 4 else 256)
                if k > 0:
                    G = engine.conv2d_dgrad(G, wpk, 256, mask=inputs[k], tile_tab=tab, out=gbuf[k & 1])
                else:
                    d_atlas = engine.conv2d_dgrad(G, wpk, 256, residual=d_atlas, tile_tab=tab,
                                                  out=gbuf[2] if d_atlas is None else gbuf[3])
        if need_fpn and d_atlas is not None:
            self._fpn_backward(state, d_atlas, need, got)
        self.last_atlas_grad = d_atlas if self.want_atlas_grad else None
        return [got.get(n) for n in names]

    def _fpn_backward(self, state, d_atlas, need, got):
        """The FPN's weight and bias gradients from d(atlas), the gradient w.r.t. the five FPN outputs, into `got`:
        pyramid7 (odtk_conv_wgrad_ex, stride 2 over relu(P6)); dP6 = d(atlas)'s P6 level + the input gradient of pyramid7 --
        dP7 dilated into P6's geometry (odtk_dilate_f16), the stride-1 masked dgrad over P6's tiles, then the plain add
        (odtk_pool_add_f16, pool 1: the dgrad's mask would also zero a residual addend); pyramid6 (stride 2 over C5);
        smooth3-5 (3x3 over the pre-smooth p3-p5); their unmasked input gradients into a pre-smooth gradient atlas, the
        top-down pathway's upsample-add backward (pool 2, level 0 -> 1, then 1 -> 2), then lateral3-5 (1x1 over C3-C5).
        Only the launches whose results a needed gradient reads run; the backbone gets no gradient."""
        S, at, views = state["fpn"], state["at"], state["views"]
        pre = "backbones.%s." % self.backbone
        rows, tabs, atlas0 = at["rows"], at["tabs"], views[0].atlas
        lv = [(r, v.h, v.w) for r, v in zip(rows, views)]

        def wants(layer):
            return need.get(pre + layer + ".weight", False) or need.get(pre + layer + ".bias", False)

        def wgrad(layer, g, x, ksize, stride, l):
            self._wgrad(need, got, pre + layer, engine.conv_wgrad_ex, g, x, 256, ksize, stride, tabs[l], rows[l])

        wgrad("pyramid7", d_atlas, S["r6"], 3, 2, 4)
        if wants("pyramid6"):
            gd = engine.dilate(d_atlas, self._atlas_zeros(at, "fpn_dilated"), lv[4], rows[3])
            dp6 = engine.conv2d_dgrad(gd, self._dgrad_weights(pre + "pyramid7.weight", 256), 256, mask=atlas0,
                                      tile_tab=tabs[3], out=self._atlas_zeros(at, "fpn_dp6"))
            engine.pool_add(d_atlas, dp6, lv[3], lv[3], pool=1)
            wgrad("pyramid6", dp6, S["c5"], 3, 2, 3)
        for l in range(3):
            wgrad("smooth%d" % (l + 3), d_atlas, S["p%d" % (l + 3)], 3, 1, l)
        top = max([l for l in range(3) if wants("lateral%d" % (l + 3))], default=-1)    # lateral l reads levels 0..l
        if top >= 0:
            dpre = self._atlas_zeros(at, "fpn_dpre")
            for l in range(top + 1):
                engine.conv2d_dgrad(d_atlas, self._dgrad_weights(pre + "smooth%d.weight" % (l + 3), 256), 256,
                                    tile_tab=tabs[l], out=dpre)
            for l in range(top):
                engine.pool_add(dpre, dpre, lv[l], lv[l + 1], pool=2)
            for l in range(top + 1):
                wgrad("lateral%d" % (l + 3), dpre, S["c%d" % (l + 3)], 1, 1, l)

    @staticmethod
    def _wgrad(need, got, layer, launch, *args, **kwargs):
        """Weight and bias gradient of `layer` (a parameter prefix) by launch(*args, bias=...) -> (dw, db), run only when
        one of them is needed, stored into `got`."""
        wn, bn = layer + ".weight", layer + ".bias"
        if need.get(wn, False) or need.get(bn, False):
            dw, db = launch(*args, bias=need.get(bn, False), **kwargs)
            if need.get(wn, False):
                got[wn] = dw
            if need.get(bn, False):
                got[bn] = db

    def _dgrad_weights(self, name, cout_pad):
        """engine.pack_weight_dgrad of parameter `name`, cached until the parameter changes."""
        p = self._params[name]
        cached = self._dgrad_w.get(name)
        if cached is None or cached[0] != (p._version, id(p)):
            cached = self._dgrad_w[name] = ((p._version, id(p)), engine.pack_weight_dgrad(p, cout_pad))
        return cached[1]

    @staticmethod
    def _atlas_zeros(at, key, channels=256):
        """at[key]: an fp16 buffer of the atlas geometry with `channels` channels, zero-initialised on first use (the
        backward writes only the levels' tiles, so everything else stays zero)."""
        if key not in at:
            a = at["buf"][0]
            at[key] = torch.zeros(a.shape[:3] + (channels,), dtype=torch.float16, device=a.device)
        return at[key]

    def forward(self, x, rotated_bbox=None):
        self._sync_params()
        if self.training:
            x, targets = x
            params = [p for _, p in self.named_parameters()] if self._params is not None else []
            if torch.is_grad_enabled() and any(p.requires_grad for p in params):
                return _HeadsTrain.apply(self, x, targets.float().to(x.device), *params)
            cls_heads, box_heads = self.forward_heads(x, sigmoid=False)
            return self._compute_loss(x, cls_heads, box_heads, targets.float().to(cls_heads[0].device))
        if self.fused_candidates and not self.exporting:
            return self._forward_fused(x)
        if x.dtype == torch.uint8:                       # raw HWC images: fused input side
            (cls_heads, box_heads), (_, width) = self.forward_heads_u8(x)
        else:
            cls_heads, box_heads = self.forward_heads(x)
            width = x.shape[-1]
        if self.exporting:
            self.strides = [width // c.shape[-1] for c in cls_heads]
            return cls_heads, box_heads
        return self._detect_dense(cls_heads, box_heads, width)

    def _detect_dense(self, cls_heads, box_heads, width):
        strides, anchors = self._level_anchors([c.shape[-1] for c in cls_heads], width)
        decoded = _C.decode_levels(cls_heads, box_heads, anchors, strides, self.threshold, self.top_n, self.rotated_bbox)
        return self._nms(decoded)

    # ---- raw images of any size (the PIL data loader of `odtk infer`, odtk/data.py:55-60, 113-123, 154-176) ------------
    def _forward_padded(self, xp, hs, width):
        """Detections from the stem's padded NHWC4 input buffer (fp32 in full precision): the fused-candidate or the dense
        route of forward()."""
        features = self._features(self._stem(padded=(xp, hs, width)))
        if self.fused_candidates:
            return self._detect_fused(features, width)
        return self._detect_dense(*self._heads(features), width)

    def forward_images(self, images, resize=800, max_size=1333, canvas=None):
        """Inference on a list of raw uint8 [h_i, w_i, 3] RGB images of any sizes (CPU or CUDA tensors): each image is
        resized by the reference's ratio with Pillow-exact BILINEAR resampling, normalised and padded into one batch
        canvas by one kernel (engine.preprocess_resize_u8), then the network runs as forward() does.  `canvas` (hs, ws):
        a fixed canvas (multiples of 128) shared by every batch, hence one CUDA graph; default the reference collate's
        batch maximum.  Returns ((scores, boxes, classes), ratios): boxes in resized coordinates, as the reference model
        returns them; ratios float32 [n] (divide by them for original coordinates, infer.detections_to_coco).
        With enable_cuda_graph() one graph per (n, canvas) is replayed; its staging buffers grow (and the graph is
        captured again) when a batch has more bytes than they hold."""
        if self._packed is None:
            raise RuntimeError("call .cuda() after loading weights: there is no CPU path")
        if self.training or self.exporting:
            raise RuntimeError("forward_images runs inference: call .eval() and leave exporting off")
        self._sync_params()
        plan = engine.ResizePlan(engine.image_shapes(images), resize, max_size, self.stride, canvas)
        hs, ws = plan.canvas
        if getattr(self, "_graphs", None) is None:
            xp, _, _, ratios = engine.preprocess_resize_u8(images, resize, max_size, self.stride, (hs, ws),
                                                           f32=self._stem_dtype() == torch.float32)
            return self._forward_padded(xp, hs, ws), ratios
        key = ("images", plan.n, hs, ws)
        entry = self._graphs.get(key)
        if entry is None or entry["capacity"] < plan.nbytes:
            entry = self._graphs[key] = self._capture_images(images, plan, max(plan.nbytes, 2 * entry["capacity"] if entry else 0))
        engine.stage_images(images, plan, entry["buf"])
        entry["graph"].replay()
        if self.gather is not None:
            self.gather.steps += 1
        return entry["out"], plan.ratios

    def _capture_images(self, images, plan, capacity):
        """CUDA graph of resize + network over static device buffers: [size table | packed pixels] of `capacity` bytes and
        the stem buffer.  The kernel reads the sizes from the device table, so any batch that fits the canvas replays it."""
        dev = self._packed["stem"].w_stem.device
        tpad = engine.table_pad(plan.n)
        buf = torch.empty(tpad + capacity, dtype=torch.uint8, device=dev)
        hs, ws = plan.canvas
        xp = torch.empty((plan.n, hs + 6, ws + 8, 4), dtype=self._stem_dtype(), device=dev)

        def run():
            self._resize_launch(buf[tpad:], capacity, plan, buf[:tpad], out=xp)
            return self._forward_padded(xp, hs, ws)

        engine.stage_images(images, plan, buf)
        for _ in range(2):                      # warm-up: lazy attribute set-up, allocator, anchors
            run()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = run()
        return {"graph": graph, "buf": buf, "xp": xp, "out": out, "capacity": capacity}

    def _resize_launch(self, *args, **kwargs):
        """engine.resize_launch into the stem buffer of the current precision."""
        return (engine.resize_launch_f32 if self._stem_dtype() == torch.float32 else engine.resize_launch)(*args, **kwargs)

    # ---- JPEG streams (the Image.open(path).convert("RGB") of odtk/data.py:50, then the raw-image path) ------------------
    def forward_jpeg(self, datas, resize=800, max_size=1333, canvas=None):
        """Inference on a list of baseline JPEG streams (bytes-like, e.g. open(path, "rb").read()): the GPU decodes them
        bit-exactly as Pillow's Image.open(f).convert("RGB") does (engine.decode_jpeg), then they go through
        forward_images' resize + network path.  Returns ((scores, boxes, classes), ratios, status): status int32 [n]
        CUDA, 0 or the ODTK_JPEG_* bits of an image whose scan is corrupt (its detections are then meaningless, the
        other images are unaffected).  A stream the decoder does not take (progressive, CMYK, ...) raises ValueError
        naming the image: decode it with Pillow and use forward_images.
        With enable_cuda_graph() one graph per (n, canvas) covers decode, resize and network; its staging, workspace
        and pixel buffers grow (and the graph is captured again) when a batch needs more than they hold."""
        from . import jpeg
        if self._packed is None:
            raise RuntimeError("call .cuda() after loading weights: there is no CPU path")
        if self.training or self.exporting:
            raise RuntimeError("forward_jpeg runs inference: call .eval() and leave exporting off")
        self._sync_params()
        batch = jpeg.JpegBatch(datas)
        plan = engine.ResizePlan(batch.shapes, resize, max_size, self.stride, canvas)
        hs, ws = plan.canvas
        need = (batch.nbytes, batch.workspace_bytes(), plan.nbytes)
        if getattr(self, "_graphs", None) is None:
            bufs = self._jpeg_buffers(plan.n, need)
            batch.stage(plan.table, bufs["buf"])
            xp = self._jpeg_decode_resize(batch, plan, bufs)
            return self._forward_padded(xp, hs, ws), plan.ratios, bufs["status"]
        key = ("jpeg", plan.n, hs, ws)
        entry = self._graphs.get(key)
        if entry is None or any(a > b for a, b in zip(need, entry["capacity"])):
            cap = tuple(max(a, 2 * b) for a, b in zip(need, entry["capacity"])) if entry else need
            entry = self._graphs[key] = self._capture_jpeg(batch, plan, cap)
        else:
            bufs = entry["bufs"]
            engine.jpeg_launch(batch, bufs["buf"], plan.table, None, bufs["pixels"], None)    # validate the host tables
            batch.stage(plan.table, bufs["buf"])
        entry["graph"].replay()
        if self.gather is not None:
            self.gather.steps += 1
        return entry["out"], plan.ratios, entry["bufs"]["status"]

    def _jpeg_buffers(self, n, capacity):
        dev = self._packed["stem"].w_stem.device
        staging, workspace, pixels = capacity
        return {"buf": torch.empty(staging, dtype=torch.uint8, device=dev),
                "workspace": torch.empty(workspace, dtype=torch.uint8, device=dev),
                "pixels": torch.empty(pixels, dtype=torch.uint8, device=dev),
                "status": torch.empty(n, dtype=torch.int32, device=dev)}

    def _jpeg_decode_resize(self, batch, plan, bufs, xp=None):
        """Decode into the packed pixel buffer at the resize plan's offsets, then resize it into the stem buffer; the
        resize kernel reads the size table staged with the batch."""
        engine.jpeg_launch(batch, bufs["buf"], plan.table, bufs["workspace"], bufs["pixels"], bufs["status"])
        return self._resize_launch(bufs["pixels"], bufs["pixels"].numel(), plan, bufs["buf"][batch.resize_off:], out=xp)

    def _capture_jpeg(self, batch, plan, capacity):
        """CUDA graph of decode + resize + network over static buffers of `capacity` (staging, workspace, pixel bytes)
        and the stem buffer.  Every kernel reads its sizes from the staged tables, so any batch of n JPEGs that fits the
        canvas and the buffers replays it."""
        bufs = self._jpeg_buffers(plan.n, capacity)
        hs, ws = plan.canvas
        xp = torch.empty((plan.n, hs + 6, ws + 8, 4), dtype=self._stem_dtype(), device=bufs["buf"].device)

        def run():
            self._jpeg_decode_resize(batch, plan, bufs, xp)
            return self._forward_padded(xp, hs, ws)

        batch.stage(plan.table, bufs["buf"])
        for _ in range(2):                      # warm-up: lazy attribute set-up, allocator, anchors
            run()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = run()
        return {"graph": graph, "bufs": bufs, "xp": xp, "out": out, "capacity": capacity}

    # ---- CUDA graph replay ---------------------------------------------------------------------
    def enable_cuda_graph(self, enabled=True):
        """Capture the whole forward (≈125 kernel launches, no host sync anywhere on the path) into a
        CUDA graph per input shape and replay it: removes the per-launch host cost, which dominates at
        small batch.  The reference has no equivalent (its decode/nms block the host B*5+B times)."""
        self._graphs = {} if enabled else None
        return self

    def _forward_graphed(self, x, rotated_bbox=None, static_input=False):
        """static_input=True: the caller promises to reuse THIS tensor's storage for every call (e.g. the
        device side of a double-buffered upload): the graph reads it in place, no staging copy."""
        key = (tuple(x.shape), x.dtype, bool(x.is_contiguous(memory_format=torch.channels_last)),
               x.data_ptr() if static_input else 0)
        entry = self._graphs.get(key)
        if entry is None:
            static_in = x if static_input else x.clone()
            for _ in range(2):                      # warm-up: lazy attribute set-up, allocator, anchors
                self.forward(static_in, rotated_bbox)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                static_out = self.forward(static_in, rotated_bbox)
            entry = self._graphs[key] = (graph, static_in, static_out)
        graph, static_in, static_out = entry
        if not static_input:
            static_in.copy_(x, non_blocking=True)
        graph.replay()
        if self.gather is not None:
            self.gather.steps += 1
        return static_out

    def __call__(self, x, rotated_bbox=None, static_input=False):
        if getattr(self, "_graphs", None) is not None and not self.exporting and not self.training:
            self._sync_params()
            return self._forward_graphed(x, rotated_bbox, static_input)
        return self.forward(x, rotated_bbox)
