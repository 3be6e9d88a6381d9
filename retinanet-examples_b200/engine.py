"""Thin host wrappers over the convolution engine of the C ABI (include/odtk_b200.h): weight
packing / BatchNorm folding and per-layer calls.  Activations are NHWC fp16 CUDA tensors."""
import ctypes

import torch

from . import _lib

OUT_NHWC_F16, OUT_NCHW_F32, OUT_NCHW_F32_SIGMOID, OUT_CANDIDATES = 0, 1, 2, 3

# host-side accounting of what was launched (bench.py reads it): kernels launched by this
# module and algorithmic convolution FLOPs (2 * pixels * Cout * taps * Cin, unpadded)
STATS = {"launches": 0, "conv_flops": 0, "trace": None}


def _trace(kind, flops, nbytes, **shape):
    """When STATS["trace"] is a list, every kernel launch appends (kind, algorithmic FLOPs, algorithmic HBM bytes =
    every operand read once + the output written once, shape): bench.py's layer-wise roofline is keyed on this
    order."""
    if STATS["trace"] is not None:
        STATS["trace"].append(dict(kind=kind, flops=int(flops), bytes=int(nbytes), **shape))



class ConvDesc(ctypes.Structure):
    """odtk_conv_t (include/odtk_b200.h)."""
    _fields_ = [("x", ctypes.c_void_p), ("w", ctypes.c_void_p), ("bias", ctypes.c_void_p),
                ("residual", ctypes.c_void_p), ("upsample", ctypes.c_void_p), ("y", ctypes.c_void_p),
                ("n", ctypes.c_int), ("h", ctypes.c_int), ("width", ctypes.c_int), ("cin", ctypes.c_int),
                ("cout", ctypes.c_int), ("ksize", ctypes.c_int), ("relu", ctypes.c_int), ("out_mode", ctypes.c_int),
                ("ldy", ctypes.c_int), ("ldr", ctypes.c_int), ("stride", ctypes.c_int), ("bias_op", ctypes.c_void_p),
                ("sink", ctypes.c_void_p), ("groups", ctypes.c_int), ("x_rows", ctypes.c_int), ("x_width", ctypes.c_int),
                ("y_rows", ctypes.c_int), ("y_row_off", ctypes.c_int), ("y_width", ctypes.c_int), ("tile_tab", ctypes.c_void_p),
                ("tab_tiles", ctypes.c_int)]


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def last_plan():
    """The kernel variant the last conv launch of this thread used (odtk_conv_last_plan), as a dict."""
    pl = _lib.ConvPlan()
    _lib.check(_lib.lib().odtk_conv_last_plan(ctypes.byref(pl)), "conv_last_plan")
    return {n: getattr(pl, n) for n, _ in pl._fields_}


def fold_bn(weight, bn_weight, bn_bias, running_mean, running_var, eps=1e-5):
    """conv (no bias) followed by eval-mode BatchNorm == conv with scaled weights + a bias
    (torchvision BasicBlock/Bottleneck, odtk/backbones/layers.py:5-15).  fp32 in, fp32 out."""
    scale = bn_weight.float() / torch.sqrt(running_var.float() + eps)
    return weight.float() * scale.view(-1, 1, 1, 1), bn_bias.float() - running_mean.float() * scale


def pack_weight(weight, kpad=None):
    """[Cout, Cin, kh, kw] fp32 -> [Cout, kh*kw*Cin (zero padded to kpad)] fp16, tap-major /
    channel-minor: the K order of the kernel's (tap, 64-channel chunk) loop."""
    cout, cin, kh, kw = weight.shape
    w = weight.permute(0, 2, 3, 1).reshape(cout, kh * kw * cin)
    if kpad is not None and kpad > w.shape[1]:
        w = torch.cat([w, w.new_zeros(cout, kpad - w.shape[1])], dim=1)
    return w.to(torch.float16).contiguous()


def pack_weight_grouped(weight, groups):
    """Grouped 3x3 weights [C, C/groups, kh, kw] fp32 (ResNeXt conv2) -> [C, kh*kw*64] fp16: output channel o reads only
    the 64-channel input chunk it lives in (a group never straddles a chunk), its group's weights sit at the columns of
    their input channels inside that chunk, zeros elsewhere (block-diagonal)."""
    cout, cg, kh, kw = weight.shape
    assert cout % groups == 0 and cout // groups == cg and 64 % cg == 0 and cout % 64 == 0
    w = weight.new_zeros((cout, kh * kw, 64))
    o = torch.arange(cout)
    first = (o // cg) * cg % 64                        # column of the group's first input channel inside the chunk
    cols = first[:, None] + torch.arange(cg)[None, :]  # [cout, cg]
    src = weight.permute(0, 2, 3, 1).reshape(cout, kh * kw, cg)
    w.scatter_(2, cols[:, None, :].expand(cout, kh * kw, cg), src)
    return w.reshape(cout, kh * kw * 64).to(torch.float16).contiguous()


def pack_bias(bias):
    """fp32 bias [Cout] (CUDA) -> the [Cout, 64] fp16 (hi, lo) layout of odtk_conv_t.bias_op.  The sm_90a kernel adds
    the fp32 bias in its epilogue and does not read it."""
    out = torch.empty((bias.numel(), 64), dtype=torch.float16, device=bias.device)
    _lib.check(_lib.lib().odtk_conv_pack_bias(ctypes.c_void_p(bias.data_ptr()), ctypes.c_void_p(out.data_ptr()),
                                              bias.numel(), _stream()), "conv_pack_bias")
    return out


class AtlasView:
    """A level of the pyramid atlas: the top-left h x w rectangle at row `row_off` of an atlas tensor [N, rows, width, C]."""

    def __init__(self, atlas, row_off, h, w):
        self.atlas, self.row_off, self.h, self.w = atlas, int(row_off), int(h), int(w)

    @property
    def shape(self):
        return (self.atlas.shape[0], self.h, self.w, self.atlas.shape[3])

    @property
    def device(self):
        return self.atlas.device

    def dense(self):
        """A contiguous copy of the level (tests / debugging)."""
        return self.atlas[:, self.row_off:self.row_off + self.h, :self.w, :].contiguous()

    def data_ptr(self):
        return self.atlas.data_ptr() + self.row_off * self.atlas.shape[2] * self.atlas.shape[3] * 2


def conv2d(x, w, bias, cout, ksize, relu=False, residual=None, upsample=None, out_mode=OUT_NHWC_F16, out=None,
           stride=1, bias_op=None, sink=None, groups=1, tile_tab=None):
    """x: NHWC fp16 [N,H,W,Cin] (or an AtlasView); w: packed fp16 [Cout, ksize*ksize*Cin]; bias fp32 [Cout] or None.
    Stride 1 / 2, pad ksize//2.  Returns NHWC fp16 [N,H,W,Cout] or NCHW fp32 [N,Cout,H,W]; `out` may be an AtlasView
    (the result lands in that rectangle).  tile_tab (device int32 [T, 4]): x and out are whole atlases, one launch
    covers all the levels the table lists."""
    xv = x if isinstance(x, AtlasView) else None
    assert xv is not None or (x.is_cuda and x.dtype == torch.float16 and x.is_contiguous())
    n, h, wd, cin = x.shape
    oh, ow = ((h - 1) // 2 + 1, (wd - 1) // 2 + 1) if stride == 2 else (h, wd)
    if out_mode == OUT_CANDIDATES:
        assert sink is not None
    elif out is None:
        if out_mode == OUT_NHWC_F16:
            out = torch.empty((n, oh, ow, cout), dtype=torch.float16, device=x.device)
        else:
            out = torch.empty((n, cout, oh, ow), dtype=torch.float32, device=x.device)
    d = ConvDesc()
    d.x, d.w, d.y = x.data_ptr(), w.data_ptr(), (out.data_ptr() if out is not None else None)
    if xv is not None:
        d.x_rows, d.x_width = xv.atlas.shape[1], xv.atlas.shape[2]
    if isinstance(out, AtlasView):
        d.y_rows, d.y_row_off, d.y_width = out.atlas.shape[1], 0, out.atlas.shape[2]      # data_ptr() already points at the level
        d.y_row_off = 0
    if tile_tab is not None:
        d.tile_tab, d.tab_tiles = tile_tab.data_ptr(), tile_tab.shape[0]
    d.sink = ctypes.addressof(sink) if sink is not None else None
    d.bias = bias.data_ptr() if bias is not None else None
    d.residual = residual.data_ptr() if residual is not None else None
    d.upsample = upsample.data_ptr() if upsample is not None else None
    d.n, d.h, d.width, d.cin, d.cout, d.ksize = n, h, wd, cin, cout, ksize
    d.relu, d.out_mode, d.ldy, d.ldr, d.stride = int(relu), out_mode, 0, 0, int(stride)
    d.bias_op = bias_op.data_ptr() if bias_op is not None else None
    d.groups = int(groups)
    _lib.check(_lib.lib().odtk_conv2d(ctypes.byref(d), _stream()), "conv2d")
    STATS["launches"] += 1
    if STATS["trace"] is not None:
        px = n * oh * ow if tile_tab is None else n * int(((tile_tab[:, 2] - tile_tab[:, 0]).clamp(max=8) * (tile_tab[:, 3] - tile_tab[:, 1]).clamp(max=16)).sum())
        obytes = 0 if out_mode == OUT_CANDIDATES else px * cout * (2 if out_mode == OUT_NHWC_F16 else 4)
        _trace("conv%dx%d" % (ksize, ksize), 2 * px * cout * ksize * ksize * cin // groups,
               (px * cin * 2 if ((ksize == 1 and stride == 2) or tile_tab is not None) else n * h * wd * cin * 2) + w.numel() * 2 + obytes + (px * cout * 2 if residual is not None else 0)
               + (px * cout // 2 if upsample is not None else 0),
               n=n, h=h, w=wd, cin=cin, cout=cout, stride=int(stride), residual=residual is not None,
               upsample=upsample is not None, out_mode=out_mode)
    return out


def lower_conv(x, ksize, stride, pad, kpad=None, relu=False):
    """Gather receptive fields: NHWC fp16 [N,H,W,C] -> [N, OH, OW, kpad] fp16."""
    n, h, w, c = x.shape
    oh, ow = (h + 2 * pad - ksize) // stride + 1, (w + 2 * pad - ksize) // stride + 1
    kpad = kpad or ksize * ksize * c
    out = torch.empty((n, oh, ow, kpad), dtype=torch.float16, device=x.device)
    _lib.check(_lib.lib().odtk_lower_conv(ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(out.data_ptr()), n, h, w, c,
                                          ksize, stride, pad, kpad, int(relu), _stream()), "lower_conv")
    STATS["launches"] += 1
    _trace("lower_conv", 0, x.numel() * 2 + out.numel() * 2, n=n, h=h, w=w, cin=c)
    return out


def relu(x):
    """max(x, 0) into a new tensor (input of FPN pyramid7, odtk/backbones/fpn.py:55)."""
    out = torch.empty_like(x)
    _lib.check(_lib.lib().odtk_relu_f16(ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(out.data_ptr()), x.numel(), _stream()),
               "relu_f16")
    STATS["launches"] += 1
    _trace("relu", 0, x.numel() * 4, n=x.shape[0], h=x.shape[1], w=x.shape[2], cin=x.shape[3])
    return out


def relu_from_view(view):
    """ReLU of a pyramid level that lives inside the atlas, into a new dense tensor [N, h, w, C]."""
    n, h, w, c = view.shape
    a = view.atlas
    out = torch.empty((n, h, w, c), dtype=torch.float16, device=a.device)
    _lib.check(_lib.lib().odtk_copy_rows_f16(ctypes.c_void_p(view.data_ptr()), ctypes.c_void_p(out.data_ptr()), n, h, w * c,
                                             a.shape[1] * a.shape[2] * c, a.shape[2] * c, h * w * c, w * c, 1, _stream()), "copy_rows_f16")
    STATS["launches"] += 1
    _trace("relu", 0, out.numel() * 4, n=n, h=h, w=w, cin=c)
    return out


def maxpool3x3s2(x):
    n, h, w, c = x.shape
    out = torch.empty((n, (h - 1) // 2 + 1, (w - 1) // 2 + 1, c), dtype=torch.float16, device=x.device)
    _lib.check(_lib.lib().odtk_maxpool3x3s2(ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(out.data_ptr()), n, h, w, c,
                                            _stream()), "maxpool3x3s2")
    STATS["launches"] += 1
    _trace("maxpool", 0, x.numel() * 2 + out.numel() * 2, n=n, h=h, w=w, cin=c)
    return out


def pack_stem_weight(weight):
    """[Cout, 3, 7, 7] fp32 -> [Cout, 7*32] fp16 with k = r*32 + s*4 + c (zero for s = 7 or c = 3):
    the K order of the stem's overlapping-window tensor map (odtk_stem_conv)."""
    cout = weight.shape[0]
    w = weight.new_zeros((cout, 7, 8, 4))
    w[:, :, :7, :3] = weight.permute(0, 2, 3, 1)          # [cout, r, s, c]
    return w.reshape(cout, 224).to(torch.float16).contiguous()


IMAGENET_MEAN, IMAGENET_STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]   # odtk/data.py:25-26


def preprocess_u8(images, stride=128, mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """uint8 HWC batch [N,H,W,3] (CUDA) -> normalised, stride-padded, zero-bordered NHWC4 fp16
    [N, Hs+6, Ws+8, 4] ready for the stem (reference: odtk/data.py:113-123).  Returns (buffer, Hs, Ws)."""
    assert images.is_cuda and images.dtype == torch.uint8 and images.is_contiguous() and images.shape[-1] == 3
    n, h, w, _ = images.shape
    hs, ws = (h + stride - 1) // stride * stride, (w + stride - 1) // stride * stride
    xp = torch.empty((n, hs + 6, ws + 8, 4), dtype=torch.float16, device=images.device)
    m = (ctypes.c_float * 3)(*mean)
    s = (ctypes.c_float * 3)(*std)
    _lib.check(_lib.lib().odtk_preprocess_u8(ctypes.c_void_p(images.data_ptr()), ctypes.c_void_p(xp.data_ptr()), n, h, w,
                                             hs, ws, m, s, _stream()), "preprocess_u8")
    STATS["launches"] += 1
    _trace("preprocess_u8", 0, images.numel() + xp.numel() * 2, n=n, h=h, w=w, cin=3)
    return xp, hs, ws


def stem_conv_padded(xp, h, wd, w, bias, cout, relu=True):
    """Stem over an already padded NHWC4 buffer [N, h+6, wd+8, 4] (from preprocess_u8)."""
    n = xp.shape[0]
    out = torch.empty((n, h // 2, wd // 2, cout), dtype=torch.float16, device=xp.device)
    _lib.check(_lib.lib().odtk_stem_conv(ctypes.c_void_p(xp.data_ptr()), ctypes.c_void_p(w.data_ptr()),
                                         ctypes.c_void_p(bias.data_ptr()) if bias is not None else None,
                                         ctypes.c_void_p(out.data_ptr()), n, h, wd, cout, int(relu), _stream()), "stem_conv")
    STATS["launches"] += 1
    _trace("stem7x7", 2 * out.numel() * 147, xp.numel() * 2 + w.numel() * 2 + out.numel() * 2, n=n, h=h, w=wd, cin=3,
           cout=cout, stride=2)
    return out


def stem_conv(x, w, bias, cout, relu=True):
    """7x7 stride-2 pad-3 convolution of an NHWC fp16 RGB batch [N,H,W,3] on the tensor cores:
    zero-pad to NHWC4 (one small kernel), then the conv kernel in stem mode.  Returns
    NHWC fp16 [N, H/2, W/2, cout]."""
    n, h, wd, c = x.shape
    assert c == 3 and x.dtype == torch.float16 and x.is_contiguous()
    xp = torch.empty((n, h + 6, wd + 8, 4), dtype=torch.float16, device=x.device)
    L = _lib.lib()
    _lib.check(L.odtk_pad_input(ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(xp.data_ptr()), n, h, wd, _stream()), "pad_input")
    out = torch.empty((n, h // 2, wd // 2, cout), dtype=torch.float16, device=x.device)
    _lib.check(L.odtk_stem_conv(ctypes.c_void_p(xp.data_ptr()), ctypes.c_void_p(w.data_ptr()),
                                ctypes.c_void_p(bias.data_ptr()) if bias is not None else None,
                                ctypes.c_void_p(out.data_ptr()), n, h, wd, cout, int(relu), _stream()), "stem_conv")
    STATS["launches"] += 2
    _trace("pad_input", 0, x.numel() * 2 + xp.numel() * 2, n=n, h=h, w=wd, cin=3)
    _trace("stem7x7", 2 * out.numel() * 147, xp.numel() * 2 + w.numel() * 2 + out.numel() * 2, n=n, h=h, w=wd, cin=3,
           cout=cout, stride=2)
    return out


def stem_pool_padded(xp, h, wd, w, bias, cout, relu=True):
    """Stem conv + BN + ReLU + 3x3/2 max-pool in ONE kernel over a padded NHWC4 buffer [N, h+6, wd+8, 4] (odtk_stem_pool):
    the stem activation is never written.  Returns NHWC fp16 [N, (h/2-1)/2+1, (wd/2-1)/2+1, cout]."""
    n = xp.shape[0]
    oh, ow = h // 2, wd // 2
    out = torch.empty((n, (oh - 1) // 2 + 1, (ow - 1) // 2 + 1, cout), dtype=torch.float16, device=xp.device)
    _lib.check(_lib.lib().odtk_stem_pool(ctypes.c_void_p(xp.data_ptr()), ctypes.c_void_p(w.data_ptr()),
                                         ctypes.c_void_p(bias.data_ptr()) if bias is not None else None,
                                         ctypes.c_void_p(out.data_ptr()), n, h, wd, cout, int(relu), _stream()), "stem_pool")
    STATS["launches"] += 1
    _trace("stem_pool", 2 * n * oh * ow * cout * 147, xp.numel() * 2 + w.numel() * 2 + out.numel() * 2, n=n, h=h, w=wd, cin=3,
           cout=cout, stride=2)
    return out


def bottleneck_tail(x, w2, b2, w3, b3, residual, relu=True, out=None, xproj=None, wproj=None, w_next=None, b_next=None):
    """Tail of a stride-1 bottleneck block in one kernel (odtk_bottleneck_tail):
    relu(conv1x1(relu(conv3x3(x, w2) + b2), w3) + b3 + residual).  x: NHWC fp16 [N,H,W,C1] (C1 64 / 128); w2 packed
    [C1, 9*C1]; w3 packed [C2, C1]; residual NHWC fp16 [N,H,W,C2].  Returns NHWC fp16 [N,H,W,C2]."""
    assert x.is_cuda and x.dtype == torch.float16 and x.is_contiguous()
    n, h, wd, c1 = x.shape
    c2 = w3.shape[0]
    if xproj is not None:          # identity = xproj x wproj^T computed by the kernel (b3 already holds both biases)
        assert xproj.is_contiguous() and xproj.shape == (n, h, wd, 64) and wproj.shape == (c2, 64)
    else:
        assert residual.is_contiguous() and residual.shape == (n, h, wd, c2)
    if out is None:
        out = torch.empty((n, h, wd, c2), dtype=torch.float16, device=x.device)
    d = _lib.BneckDesc()
    d.x, d.w2, d.w3, d.y = x.data_ptr(), w2.data_ptr(), w3.data_ptr(), out.data_ptr()
    d.residual = residual.data_ptr() if residual is not None else None
    d.xproj = xproj.data_ptr() if xproj is not None else None
    d.wproj = wproj.data_ptr() if wproj is not None else None
    d.b2 = b2.data_ptr() if b2 is not None else None
    d.b3 = b3.data_ptr() if b3 is not None else None
    d.n, d.h, d.width, d.c1, d.c2, d.relu = n, h, wd, c1, c2, int(relu)
    z = None
    if w_next is not None:          # GEMM3: the next block's conv1 (+ bias + ReLU) from the block output, in the same kernel
        z = torch.empty((n, h, wd, w_next.shape[0]), dtype=torch.float16, device=x.device)
        d.w_next, d.z, d.c_next = w_next.data_ptr(), z.data_ptr(), w_next.shape[0]
        d.b_next = b_next.data_ptr() if b_next is not None else None
    _lib.check(_lib.lib().odtk_bottleneck_tail(ctypes.byref(d), _stream()), "bottleneck_tail")
    STATS["launches"] += 1
    px = n * h * wd
    if xproj is not None:
        _trace("bneck_tail", 2 * px * (c1 * (9 * c1 + c2) + 64 * c2), px * (c1 + 64 + c2) * 2 + w2.numel() * 2 + w3.numel() * 2 + wproj.numel() * 2,
               n=n, h=h, w=wd, cin=c1, cout=c2, upsample=False, residual=False)
    else:
        c3 = w_next.shape[0] if w_next is not None else 0
        _trace("bneck_tail", 2 * px * (c1 * (9 * c1 + c2) + c2 * c3), px * (c1 + 2 * c2 + c3) * 2 + w2.numel() * 2 + w3.numel() * 2,
               n=n, h=h, w=wd, cin=c1, cout=c2, residual=True, upsample=bool(c3))
    return out if z is None else (out, z)


def depthwise3x3(x, w, bias, stride=1, act=2):
    """Depthwise 3x3 (pad 1) + bias + activation (act: 0 none, 1 ReLU, 2 ReLU6) -- odtk_depthwise3x3.
    x: NHWC fp16 [N,H,W,C]; w: fp16 [9, C]; bias fp32 [C]."""
    assert x.is_cuda and x.dtype == torch.float16 and x.is_contiguous()
    n, h, wd, c = x.shape
    oh, ow = (h - 1) // stride + 1, (wd - 1) // stride + 1
    out = torch.empty((n, oh, ow, c), dtype=torch.float16, device=x.device)
    _lib.check(_lib.lib().odtk_depthwise3x3(ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(w.data_ptr()),
                                            ctypes.c_void_p(bias.data_ptr()) if bias is not None else None,
                                            ctypes.c_void_p(out.data_ptr()), n, h, wd, c, int(stride), int(act), _stream()), "depthwise3x3")
    STATS["launches"] += 1
    _trace("depthwise3x3", 2 * out.numel() * 9, x.numel() * 2 + out.numel() * 2 + w.numel() * 2, n=n, h=h, w=wd, cin=c, cout=c, stride=int(stride))
    return out


def pad_input(x):
    """NHWC fp16 RGB batch [N,H,W,3] -> zero-bordered NHWC4 [N, H+6, W+8, 4] (the stem kernels' input layout)."""
    n, h, wd, c = x.shape
    assert c == 3 and x.dtype == torch.float16 and x.is_contiguous()
    xp = torch.empty((n, h + 6, wd + 8, 4), dtype=torch.float16, device=x.device)
    _lib.check(_lib.lib().odtk_pad_input(ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(xp.data_ptr()), n, h, wd, _stream()), "pad_input")
    STATS["launches"] += 1
    _trace("pad_input", 0, x.numel() * 2 + xp.numel() * 2, n=n, h=h, w=wd, cin=3)
    return xp


def stem_pool(x, w, bias, cout, relu=True):
    """NHWC fp16 RGB batch [N,H,W,3] -> zero-pad to NHWC4 (one small kernel) -> fused stem + max-pool."""
    return stem_pool_padded(pad_input(x), x.shape[1], x.shape[2], w, bias, cout, relu)
