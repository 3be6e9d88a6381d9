"""Thin host wrappers over the convolution engine of the C ABI (include/odtk_b200.h): weight
packing / BatchNorm folding and per-layer calls.  Activations are NHWC fp16 CUDA tensors."""
import ctypes

import torch

from . import _lib

OUT_NHWC_F16, OUT_NCHW_F32, OUT_NCHW_F32_SIGMOID, OUT_CANDIDATES, OUT_NHWC_S8, OUT_NHWC_F32 = 0, 1, 2, 3, 4, 5

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


class ConvS8Desc(ctypes.Structure):
    """odtk_conv_s8_t (include/odtk_b200.h)."""
    _fields_ = [("x", ctypes.c_void_p), ("w", ctypes.c_void_p), ("alpha", ctypes.c_void_p), ("bias", ctypes.c_void_p),
                ("y", ctypes.c_void_p), ("n", ctypes.c_int), ("h", ctypes.c_int), ("width", ctypes.c_int),
                ("cin", ctypes.c_int), ("cout", ctypes.c_int), ("ksize", ctypes.c_int), ("relu", ctypes.c_int),
                ("out_mode", ctypes.c_int), ("inv_out_scale", ctypes.c_float), ("sink", ctypes.c_void_p),
                ("x_rows", ctypes.c_int), ("x_width", ctypes.c_int), ("tile_tab", ctypes.c_void_p), ("tab_tiles", ctypes.c_int)]


class ConvS8ExDesc(ctypes.Structure):
    """odtk_conv_s8_ex_t (include/odtk_b200.h)."""
    _fields_ = [("base", ConvS8Desc), ("stride", ctypes.c_int), ("residual", ctypes.c_void_p), ("res_scale", ctypes.c_float),
                ("upsample", ctypes.c_void_p), ("up_scale", ctypes.c_float), ("y_rows", ctypes.c_int),
                ("y_row_off", ctypes.c_int), ("y_width", ctypes.c_int)]


class ConvF32Desc(ctypes.Structure):
    """odtk_conv_f32_t (include/odtk_b200.h)."""
    _fields_ = [("x", ctypes.c_void_p), ("w_hi", ctypes.c_void_p), ("w_lo", ctypes.c_void_p), ("bias", ctypes.c_void_p),
                ("residual", ctypes.c_void_p), ("upsample", ctypes.c_void_p), ("y", ctypes.c_void_p)] + \
               [(f, ctypes.c_int) for f in ("n", "h", "width", "cin", "cout", "ksize", "stride", "relu", "out_mode", "ldy", "ldr")] + \
               [("sink", ctypes.c_void_p), ("x_rows", ctypes.c_int), ("x_width", ctypes.c_int), ("y_rows", ctypes.c_int),
                ("y_row_off", ctypes.c_int), ("y_width", ctypes.c_int), ("tile_tab", ctypes.c_void_p), ("tab_tiles", ctypes.c_int)]


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
    scale, bias = bn_affine(bn_weight, bn_bias, running_mean, running_var, eps)
    return weight.float() * scale.view(-1, 1, 1, 1), bias


def bn_affine(bn_weight, bn_bias, running_mean, running_var, eps=1e-5):
    """Eval-mode BatchNorm as y = x * scale + bias per channel (fp32): the factor fold_bn scales the weights by."""
    scale = bn_weight.float() / torch.sqrt(running_var.float() + eps)
    return scale, bn_bias.float() - running_mean.float() * scale


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


def pack_weight_s8(weight):
    """[Cout, Cin, kh, kw] fp32 -> (q, s_w): symmetric per-output-channel INT8 weights in the K order of pack_weight,
    q = clamp(rint(W / s_w[c]), -127, 127) int8 [Cout, kh*kw*Cin], s_w[c] = max|W[c]| / 127 (1 for an all-zero channel)
    fp32 [Cout]."""
    w = weight.float()
    amax = w.abs().amax(dim=(1, 2, 3))
    s_w = torch.where(amax > 0, amax / 127.0, torch.ones_like(amax))
    q = torch.round(w / s_w.view(-1, 1, 1, 1)).clamp_(-127, 127)
    return pack_weight(q).to(torch.int8).contiguous(), s_w.contiguous()


class AtlasView:
    """A level of the pyramid atlas: the top-left h x w rectangle at row `row_off` of an atlas tensor [N, rows, width, C]
    (fp16, or int8 for the INT8 heads: `elem` bytes per element)."""

    def __init__(self, atlas, row_off, h, w):
        self.atlas, self.row_off, self.h, self.w = atlas, int(row_off), int(h), int(w)
        self.elem = atlas.element_size()

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
        return self.atlas.data_ptr() + self.row_off * self.atlas.shape[2] * self.atlas.shape[3] * self.elem


def _conv_setup(d, yd, x, cout, ksize, stride, out_mode, out, sink, tile_tab, nhwc_mode, nhwc_dtype):
    """The fields odtk_conv_t, odtk_conv_s8_t and odtk_conv_f32_t share: x, y (allocated unless given: NHWC of the
    precision's dtype or NCHW fp32), the atlas views of x and y (yd: the struct with the y_* fields), the tile table, the
    sink and the sizes.  Returns the output."""
    n, h, wd, cin = x.shape
    oh, ow = ((h - 1) // 2 + 1, (wd - 1) // 2 + 1) if stride == 2 else (h, wd)
    if out_mode == OUT_CANDIDATES:
        assert sink is not None
    elif out is None:
        if out_mode == nhwc_mode:
            out = torch.empty((n, oh, ow, cout), dtype=nhwc_dtype, device=x.device)
        else:
            out = torch.empty((n, cout, oh, ow), dtype=torch.float32, device=x.device)
    d.x, d.y = x.data_ptr(), (out.data_ptr() if out is not None else None)
    if isinstance(x, AtlasView):
        d.x_rows, d.x_width = x.atlas.shape[1], x.atlas.shape[2]
    if isinstance(out, AtlasView):
        yd.y_rows, yd.y_row_off, yd.y_width = out.atlas.shape[1], 0, out.atlas.shape[2]   # data_ptr() already points at the level
    if tile_tab is not None:
        d.tile_tab, d.tab_tiles = tile_tab.data_ptr(), tile_tab.shape[0]
    d.sink = ctypes.addressof(sink) if sink is not None else None
    d.n, d.h, d.width, d.cin, d.cout, d.ksize = n, h, wd, cin, cout, ksize
    return out


def _conv_launched(suffix, es, x, cout, ksize, stride, out_mode, nhwc_mode, tile_tab, wbytes, residual, upsample, groups=1):
    """Trace entry of a convolution with es-byte activations: activations read once (atlas launches: the pixels of the
    levels; 1x1 stride 2: the pixels it samples), the weights, the output, the addends."""
    STATS["launches"] += 1
    if STATS["trace"] is None:
        return
    n, h, wd, cin = x.shape
    oh, ow = ((h - 1) // 2 + 1, (wd - 1) // 2 + 1) if stride == 2 else (h, wd)
    px = n * oh * ow if tile_tab is None else _tab_px(n, h, wd, tile_tab)
    obytes = 0 if out_mode == OUT_CANDIDATES else px * cout * (es if out_mode == nhwc_mode else 4)
    xbytes = px * cin * es if (tile_tab is not None or (ksize == 1 and stride == 2)) else n * h * wd * cin * es
    _trace("conv%dx%d%s" % (ksize, ksize, suffix), 2 * px * cout * ksize * ksize * cin // groups,
           xbytes + wbytes + obytes + (px * cout * es if residual is not None else 0)
           + (px * cout * es // 4 if upsample is not None else 0),
           n=n, h=h, w=wd, cin=cin, cout=cout, stride=int(stride), residual=residual is not None,
           upsample=upsample is not None, out_mode=out_mode)


def conv2d(x, w, bias, cout, ksize, relu=False, residual=None, upsample=None, out_mode=OUT_NHWC_F16, out=None,
           stride=1, bias_op=None, sink=None, groups=1, tile_tab=None):
    """x: NHWC fp16 [N,H,W,Cin] (or an AtlasView); w: packed fp16 [Cout, ksize*ksize*Cin]; bias fp32 [Cout] or None.
    Stride 1 / 2, pad ksize//2.  Returns NHWC fp16 [N,H,W,Cout] or NCHW fp32 [N,Cout,H,W]; `out` may be an AtlasView
    (the result lands in that rectangle).  tile_tab (device int32 [T, 4]): x and out are whole atlases, one launch
    covers all the levels the table lists."""
    assert isinstance(x, AtlasView) or (x.is_cuda and x.dtype == torch.float16 and x.is_contiguous())
    d = ConvDesc()
    out = _conv_setup(d, d, x, cout, ksize, stride, out_mode, out, sink, tile_tab, OUT_NHWC_F16, torch.float16)
    d.w = w.data_ptr()
    d.bias = bias.data_ptr() if bias is not None else None
    d.residual = residual.data_ptr() if residual is not None else None
    d.upsample = upsample.data_ptr() if upsample is not None else None
    d.relu, d.out_mode, d.ldy, d.ldr, d.stride = int(relu), out_mode, 0, 0, int(stride)
    d.bias_op = bias_op.data_ptr() if bias_op is not None else None
    d.groups = int(groups)
    _lib.check(_lib.lib().odtk_conv2d(ctypes.byref(d), _stream()), "conv2d")
    _conv_launched("", 2, x, cout, ksize, stride, out_mode, OUT_NHWC_F16, tile_tab, w.numel() * 2, residual, upsample, groups)
    return out


def conv2d_s8(x, w, alpha, bias, cout, ksize, relu=False, out_mode=OUT_NHWC_S8, out=None, inv_out_scale=1.0, sink=None,
              tile_tab=None, stride=1, residual=None, res_scale=0.0, upsample=None, up_scale=0.0):
    """INT8 convolution (odtk_conv2d_s8 / odtk_conv2d_s8_ex), stride 1 / 2, pad ksize//2.  x: NHWC int8 [N,H,W,Cin] (or an
    int8 AtlasView); w: int8 [Cout, ksize*ksize*Cin] from pack_weight_s8; alpha fp32 [Cout] = s_in * s_w; bias fp32 [Cout]
    or None.  Returns NHWC int8 [N,OH,OW,Cout] (out_mode OUT_NHWC_S8, requantised with inv_out_scale) or NCHW fp32
    [N,Cout,OH,OW]; `out` may be an int8 AtlasView (3x3 only: the result lands in that level of the atlas).
    tile_tab: x and out are whole int8 atlases, one launch covers every level the table lists.  NHWC int8 outputs may add
    residual (NHWC int8 [N,OH,OW,Cout], dequantised with res_scale) and / or upsample (NHWC int8 [N,H/2,W/2,Cout], nearest
    2x, dequantised with up_scale), one fmaf each before ReLU."""
    xv = x if isinstance(x, AtlasView) else None
    assert xv is not None or (x.is_cuda and x.dtype == torch.int8 and x.is_contiguous())
    assert (xv.atlas if xv is not None else x).dtype == torch.int8 and w.dtype == torch.int8
    for t in (residual, upsample):
        assert t is None or (t.is_cuda and t.dtype == torch.int8 and t.is_contiguous())
    e = ConvS8ExDesc()
    d = e.base
    out = _conv_setup(d, e, x, cout, ksize, stride, out_mode, out, sink, tile_tab, OUT_NHWC_S8, torch.int8)
    d.w, d.alpha = w.data_ptr(), alpha.data_ptr()
    d.bias = bias.data_ptr() if bias is not None else None
    d.relu, d.out_mode, d.inv_out_scale = int(relu), out_mode, float(inv_out_scale)
    e.stride = int(stride)
    e.residual, e.res_scale = (residual.data_ptr() if residual is not None else None), float(res_scale)
    e.upsample, e.up_scale = (upsample.data_ptr() if upsample is not None else None), float(up_scale)
    if stride == 1 and residual is None and upsample is None and not isinstance(out, AtlasView):
        _lib.check(_lib.lib().odtk_conv2d_s8(ctypes.byref(d), _stream()), "conv2d_s8")
    else:
        _lib.check(_lib.lib().odtk_conv2d_s8_ex(ctypes.byref(e), _stream()), "conv2d_s8_ex")
    _conv_launched("_s8", 1, x, cout, ksize, stride, out_mode, OUT_NHWC_S8, tile_tab, w.numel(), residual, upsample)
    return out


def quantize_f16_s8(x, inv_scale, out=None):
    """fp16 tensor -> int8 of the same shape, q = clamp(rint(x * inv_scale), -127, 127) (odtk_quantize_f16_s8)."""
    assert x.is_cuda and x.dtype == torch.float16 and x.is_contiguous()
    if out is None:
        out = torch.empty(x.shape, dtype=torch.int8, device=x.device)
    assert out.dtype == torch.int8 and out.numel() == x.numel() and out.is_contiguous()
    _lib.check(_lib.lib().odtk_quantize_f16_s8(ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(out.data_ptr()), x.numel(),
                                               float(inv_scale), _stream()), "quantize_f16_s8")
    STATS["launches"] += 1
    _trace("quantize_s8", 0, x.numel() * 3, n=x.shape[0], h=x.shape[1], w=x.shape[2], cin=x.shape[3])
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
    """ReLU of a pyramid level that lives inside the atlas (fp16, int8 or fp32) into a new dense tensor [N, h, w, C] of its
    dtype: the input of FPN pyramid7, ReLU(P6)."""
    n, h, w, c = view.shape
    a = view.atlas
    out = torch.empty((n, h, w, c), dtype=a.dtype, device=a.device)
    args = (ctypes.c_void_p(view.data_ptr()), ctypes.c_void_p(out.data_ptr()), n, h, w * c, a.shape[1] * a.shape[2] * c,
            a.shape[2] * c, h * w * c, w * c)
    L = _lib.lib()
    if a.dtype == torch.float16:
        _lib.check(L.odtk_copy_rows_f16(*args, 1, _stream()), "copy_rows_f16")
    else:
        name = {torch.int8: "relu_copy_rows_s8", torch.float32: "relu_copy_rows_f32"}[a.dtype]
        _lib.check(getattr(L, "odtk_" + name)(*args, _stream()), name)
    STATS["launches"] += 1
    _trace({torch.float16: "relu", torch.int8: "relu_s8", torch.float32: "relu_f32"}[a.dtype], 0,
           out.numel() * 2 * a.element_size(), n=n, h=h, w=w, cin=c)
    return out


relu_from_view_s8 = relu_from_view_f32 = relu_from_view   # the names of the INT8 and fp32 atlas ReLU before they merged


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


def resize_ratio(h, w, resize, max_size):
    """The inference resize of odtk/data.py:55-60 with the same Python float expressions: ratio = resize / shorter side,
    lowered to max_size / longer side when the longer side would exceed max_size.  Returns (ratio, dst_h, dst_w)."""
    ratio = resize / min(h, w)
    if ratio * max(h, w) > max_size:
        ratio = max_size / max(h, w)
    return ratio, int(ratio * h), int(ratio * w)


class ResizePlan:
    """Sizes of one batch of raw images for odtk_preprocess_resize_u8: `table` (odtk_resize_image_t[n], offsets into the
    packed uint8 bytes of the images in order), `nbytes` (packed size), `ratios` (float32 [n], what odtk/data.py's
    collate returns), `canvas` (hs, ws): the batch maximum of each stride-padded dst size (collate_fn, odtk/data.py:154-176),
    or the caller's canvas."""

    def __init__(self, shapes, resize, max_size, stride=128, canvas=None):
        n = len(shapes)
        if n == 0:
            raise ValueError("no images")
        self.table = (_lib.ResizeImage * n)()
        ratios, off, hs, ws = [], 0, 0, 0
        for i, (h, w) in enumerate(shapes):
            ratio, dh, dw = resize_ratio(h, w, resize, max_size)
            if dh <= 0 or dw <= 0:
                raise ValueError("image %d (%dx%d) resizes to %dx%d" % (i, h, w, dh, dw))
            t = self.table[i]
            t.offset, t.src_h, t.src_w, t.dst_h, t.dst_w = off, h, w, dh, dw
            off += h * w * 3
            ratios.append(ratio)
            hs, ws = max(hs, -(-dh // stride) * stride), max(ws, -(-dw // stride) * stride)
        if canvas is not None:
            ch, cw = int(canvas[0]), int(canvas[1])
            if ch % stride or cw % stride or ch < hs or cw < ws:
                raise ValueError("canvas %dx%d must be a multiple of %d and hold the batch's %dx%d" % (ch, cw, stride, hs, ws))
            hs, ws = ch, cw
        self.n, self.nbytes, self.canvas = n, off, (hs, ws)
        self.ratios = torch.tensor(ratios, dtype=torch.float32)

    def table_bytes(self):
        return torch.frombuffer(bytearray(bytes(self.table)), dtype=torch.uint8)


def image_shapes(images):
    """[(h, w)] of a list of uint8 [h, w, 3] images; ValueError for anything else."""
    shapes = []
    for i, im in enumerate(images):
        if im.dtype != torch.uint8 or im.dim() != 3 or im.shape[-1] != 3:
            raise ValueError("image %d: expected a uint8 [h, w, 3] tensor, got %s %s" % (i, im.dtype, tuple(im.shape)))
        shapes.append((im.shape[0], im.shape[1]))
    return shapes


TABLE_ALIGN = 256


def table_pad(n):
    """Bytes the size table of n images takes at the front of a staging buffer (the pixels start 256-byte aligned)."""
    return -(-n * ctypes.sizeof(_lib.ResizeImage) // TABLE_ALIGN) * TABLE_ALIGN


def stage_images(images, plan, buf):
    """Copy the plan's size table and the images (uint8 [h, w, 3], CPU or CUDA) into the device buffer `buf`, laid out
    [table | pixels packed one after another], on the current stream.  CPU images go through one pinned buffer: table
    and pixels leave in ONE H2D copy.  Returns (table view, pixel view) of buf."""
    tpad = table_pad(plan.n)
    assert buf.dtype == torch.uint8 and buf.numel() >= tpad + plan.nbytes
    tb = plan.table_bytes()
    if all(not im.is_cuda for im in images):
        pinned = torch.empty(tpad + plan.nbytes, dtype=torch.uint8, pin_memory=True)
        pinned[:tb.numel()].copy_(tb)
        torch.cat([im.reshape(-1) for im in images], out=pinned[tpad:])
        buf[:tpad + plan.nbytes].copy_(pinned, non_blocking=True)
    else:
        buf[:tb.numel()].copy_(tb.pin_memory(), non_blocking=True)
        torch.cat([im.to(buf.device).reshape(-1) for im in images], out=buf[tpad:tpad + plan.nbytes])
    return buf[:tpad], buf[tpad:]


def resize_launch(x_dev, x_bytes, plan, table_dev, out=None, mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """odtk_preprocess_resize_u8 over already staged bytes: returns the stem buffer [n, hs+6, ws+8, 4] fp16 (or writes
    `out`)."""
    hs, ws = plan.canvas
    L = _lib.lib()
    nbytes = _lib.check(L.odtk_preprocess_resize_u8(None, x_bytes, ctypes.byref(plan.table), None, plan.n, hs, ws, None, None,
                                                    None, None), "preprocess_resize_u8")
    if out is None:
        out = torch.empty((plan.n, hs + 6, ws + 8, 4), dtype=torch.float16, device=x_dev.device)
    assert out.dtype == torch.float16 and out.is_contiguous() and out.numel() * 2 == nbytes
    m = (ctypes.c_float * 3)(*mean)
    s = (ctypes.c_float * 3)(*std)
    _lib.check(L.odtk_preprocess_resize_u8(ctypes.c_void_p(x_dev.data_ptr()), x_bytes, ctypes.byref(plan.table),
                                           ctypes.c_void_p(table_dev.data_ptr()), plan.n, hs, ws, ctypes.c_void_p(out.data_ptr()),
                                           m, s, _stream()), "preprocess_resize_u8")
    STATS["launches"] += 1
    _trace("preprocess_resize_u8", 0, resize_bytes(plan), n=plan.n, h=hs, w=ws, cin=3)
    return out


def resize_bytes(plan):
    """Algorithmic HBM bytes of one odtk_preprocess_resize_u8 launch: every source byte read once, the size table, the
    whole fp16 NHWC4 canvas written once."""
    hs, ws = plan.canvas
    return plan.nbytes + ctypes.sizeof(plan.table) + plan.n * (hs + 6) * (ws + 8) * 8


def preprocess_resize_u8(images, resize, max_size, stride=128, canvas=None, mean=IMAGENET_MEAN, std=IMAGENET_STD, f32=False):
    """Input side of `odtk infer` for a list of raw uint8 [h_i, w_i, 3] RGB images of any sizes (odtk/data.py:55-60,
    113-123, collate_fn :154-176): Pillow-exact BILINEAR resize by the reference's ratio, normalisation, stride and batch
    padding, written straight into the stem's zero-bordered NHWC4 fp16 buffer [n, hs+6, ws+8, 4] by one kernel.  CPU
    images are staged through pinned memory with one H2D copy; CUDA images are read in place.  `canvas` (hs, ws): a fixed
    batch canvas (multiples of `stride`); default the batch maximum of the stride-padded sizes.  Returns (xp, hs, ws,
    ratios float32 [n]).  f32: the fp32 stem buffer of the full-precision mode (resize_launch_f32)."""
    plan = ResizePlan(image_shapes(images), resize, max_size, stride, canvas)
    dev = next((im.device for im in images if im.is_cuda), torch.device("cuda", torch.cuda.current_device()))
    if all(im.is_cuda and im.is_contiguous() for im in images):
        # in place: offsets from the lowest image address (one flat device address space)
        base = min(im.data_ptr() for im in images)
        for t, im in zip(plan.table, images):
            t.offset = im.data_ptr() - base
        x_bytes = max(im.data_ptr() + im.numel() for im in images) - base
        table_dev = plan.table_bytes().pin_memory().to(dev, non_blocking=True)
        x_dev = _DevPtr(base, dev)
    else:
        table_dev, x_dev = stage_images(images, plan, torch.empty(table_pad(plan.n) + plan.nbytes, dtype=torch.uint8, device=dev))
        x_bytes = plan.nbytes
    xp = (resize_launch_f32 if f32 else resize_launch)(x_dev, x_bytes, plan, table_dev, mean=mean, std=std)
    return xp, plan.canvas[0], plan.canvas[1], plan.ratios


def jpeg_launch(batch, buf, outs, workspace, y, status):
    """odtk_decode_jpeg over a staged batch (jpeg.JpegBatch.stage): `buf` the staging buffer (its odtk_resize_image_t
    copy at batch.resize_off is the device output table), `outs` the host output table, `y` the packed uint8 pixels,
    `status` int32 [n].  workspace=None returns the workspace bytes the batch needs (and validates the tables)."""
    L = _lib.lib()
    ws_ptr = ctypes.c_void_p(workspace.data_ptr()) if workspace is not None else None
    rc = _lib.check(L.odtk_decode_jpeg(ctypes.c_void_p(buf.data_ptr()) if workspace is not None else None, buf.numel(),
                                       ctypes.byref(batch.images), batch.n, ctypes.byref(outs),
                                       ctypes.c_void_p(buf.data_ptr() + batch.resize_off), ws_ptr,
                                       workspace.numel() if workspace is not None else 0,
                                       ctypes.c_void_p(y.data_ptr()), y.numel(),
                                       ctypes.c_void_p(status.data_ptr()) if status is not None else None, _stream()),
                    "decode_jpeg")
    if workspace is not None:
        STATS["launches"] += 4
        _trace("decode_jpeg", 0, jpeg_bytes(batch), n=batch.n, h=0, w=0, cin=3)
    return rc


def jpeg_bytes(batch):
    """Algorithmic HBM bytes of one odtk_decode_jpeg call: the staged input read once (the marker scan and the entropy
    decode each read the scan bytes), coefficients written and read (128 B per block), planes written and read (64 B per
    block, chroma read up to 4 times by the colour kernel, counted once), RGB pixels written."""
    return batch.nbytes + sum(t.scan_bytes for t in batch.images) + batch.blocks * (256 + 128) + batch.pixels * 3


def _output_table(shapes):
    """odtk_resize_image_t[n] packing uint8 [h, w, 3] images one after another (dst = src) and the total bytes."""
    outs = (_lib.ResizeImage * len(shapes))()
    off = 0
    for t, (h, w) in zip(outs, shapes):
        t.offset, t.src_h, t.src_w, t.dst_h, t.dst_w = off, h, w, h, w
        off += h * w * 3
    return outs, off


def decode_jpeg(datas, device=None):
    """Decode a list of baseline JPEG streams (bytes-like) on the GPU, bit-exact to Pillow's
    np.asarray(Image.open(f).convert("RGB")).  The host parses headers and stages the batch with one pinned H2D copy.
    Returns (list of uint8 [h, w, 3] CUDA views into one packed buffer, status int32 [n] CUDA: 0 or ODTK_JPEG_* bits).
    ValueError names the image and the reason for a stream the decoder does not take (progressive, CMYK, ...)."""
    from . import jpeg
    batch = jpeg.JpegBatch(datas)
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    outs, nbytes = _output_table(batch.shapes)
    buf = batch.stage(outs, torch.empty(batch.nbytes, dtype=torch.uint8, device=dev))
    y = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    workspace = torch.empty(batch.workspace_bytes(), dtype=torch.uint8, device=dev)
    status = torch.empty(batch.n, dtype=torch.int32, device=dev)
    jpeg_launch(batch, buf, outs, workspace, y, status)
    return [y[t.offset:t.offset + h * w * 3].view(h, w, 3) for t, (h, w) in zip(outs, batch.shapes)], status


def resize_u8_launch(x_dev, x_bytes, table, table_dev, out_off, out_off_dev, y):
    """odtk_resize_u8_packed over already staged bytes: Pillow's uint8 BILINEAR result of image i, dst_h x dst_w x 3,
    written at y[out_off[i]:] (y a uint8 CUDA tensor).  table: _lib.ResizeImage[n] (host) and table_dev its device copy;
    out_off: host int64 tensor [n] and out_off_dev its device copy.  y=None returns the packed bytes the images need."""
    L = _lib.lib()
    off = ctypes.c_void_p(out_off.data_ptr())
    if y is None:
        return _lib.check(L.odtk_resize_u8_packed(None, x_bytes, ctypes.byref(table), None, off, None, len(table), None, 0,
                                                  None), "resize_u8_packed")
    _lib.check(L.odtk_resize_u8_packed(ctypes.c_void_p(x_dev.data_ptr()), x_bytes, ctypes.byref(table),
                                       ctypes.c_void_p(table_dev.data_ptr()), off, ctypes.c_void_p(out_off_dev.data_ptr()),
                                       len(table), ctypes.c_void_p(y.data_ptr()), y.numel(), _stream()), "resize_u8_packed")
    STATS["launches"] += 1
    return y


def augment_launch(x, table, table_dev, canvas, out=None, workspace=None, mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """odtk_augment_u8: the rotation, flip, colour adjustments and normalisation of CocoDataset.__getitem__ on the uint8
    images in x (uint8 CUDA tensor, each at table[i].offset), collated into fp32 [n, canvas_h, canvas_w, 3] (returned as
    the [n, 3, canvas_h, canvas_w] channels_last view).  table: _lib.AugmentImage[n] (host); table_dev: its device copy."""
    ch, cw = canvas
    n = len(table)
    L = _lib.lib()
    need = _lib.check(L.odtk_augment_u8(None, x.numel(), ctypes.byref(table), None, n, ch, cw, None, 0, None, None, None,
                                        None), "augment_u8")
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, dtype=torch.uint8, device=x.device)
    if out is None:
        out = torch.empty((n, ch, cw, 3), dtype=torch.float32, device=x.device)
    assert out.dtype == torch.float32 and out.is_contiguous() and out.shape == (n, ch, cw, 3)
    m = (ctypes.c_float * 3)(*mean)
    s = (ctypes.c_float * 3)(*std)
    _lib.check(L.odtk_augment_u8(ctypes.c_void_p(x.data_ptr()), x.numel(), ctypes.byref(table),
                                 ctypes.c_void_p(table_dev.data_ptr()), n, ch, cw, ctypes.c_void_p(workspace.data_ptr()),
                                 workspace.numel(), ctypes.c_void_p(out.data_ptr()), m, s, _stream()), "augment_u8")
    STATS["launches"] += 2
    return out.permute(0, 3, 1, 2)


class _DevPtr:
    """A raw device address with the two tensor attributes resize_launch reads."""

    def __init__(self, ptr, device):
        self.ptr, self.device = ptr, device

    def data_ptr(self):
        return self.ptr


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


# ---- full precision: fp32 activations, split-TF32 convolutions (odtk_conv2d_f32) ------------------------------------
def tf32_rna(x):
    """Round fp32 values to the nearest tf32 value, ties away from zero, as cvt.rna.tf32.f32 does: the low 13 bits of the
    magnitude are rounded off (finite inputs)."""
    b = x.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


def pack_weight_tf32x2(weight, kpad=None):
    """[Cout, Cin, kh, kw] fp32 -> (hi, lo): fp32 [Cout, kh*kw*Cin (zero padded to kpad)] in the K order of pack_weight,
    hi = rna_tf32(w), lo = rna_tf32(w - hi), both tf32-valued (low 13 bits zero); |w - hi - lo| <= 2^-22 |w|."""
    cout, cin, kh, kw = weight.shape
    w = weight.float().permute(0, 2, 3, 1).reshape(cout, kh * kw * cin)
    if kpad is not None and kpad > w.shape[1]:
        w = torch.cat([w, w.new_zeros(cout, kpad - w.shape[1])], dim=1)
    return split_tf32x2(w)


def split_tf32x2(w):
    """(hi, lo) = (rna_tf32(w), rna_tf32(w - hi)) of an fp32 tensor, contiguous."""
    hi = tf32_rna(w)
    return hi.contiguous(), tf32_rna(w.float() - hi).contiguous()


def pack_stem_weight_tf32x2(weight):
    """[Cout, 3, 7, 7] fp32 -> (hi, lo) fp32 [Cout, 224] in the K order of pack_stem_weight (k = r*32 + s*4 + c)."""
    cout = weight.shape[0]
    w = weight.new_zeros((cout, 7, 8, 4))
    w[:, :, :7, :3] = weight.float().permute(0, 2, 3, 1)
    return split_tf32x2(w.reshape(cout, 224))


def conv2d_f32(x, w_hi, w_lo, bias, cout, ksize, relu=False, residual=None, upsample=None, out_mode=OUT_NHWC_F32, out=None,
               stride=1, sink=None, tile_tab=None):
    """Full-precision convolution (odtk_conv2d_f32): x NHWC fp32 [N,H,W,Cin] (or an fp32 AtlasView); w_hi / w_lo from
    pack_weight_tf32x2; bias fp32 [Cout] or None; stride 1 / 2, pad ksize//2.  Returns NHWC fp32 [N,OH,OW,Cout]
    (OUT_NHWC_F32, + residual NHWC fp32 [N,OH,OW,Cout] and / or upsample NHWC fp32 [N,H/2,W/2,Cout] before ReLU) or NCHW
    fp32 [N,Cout,OH,OW]; `out` may be an fp32 AtlasView; tile_tab as for conv2d."""
    xv = x if isinstance(x, AtlasView) else None
    assert (xv.atlas if xv is not None else x).dtype == torch.float32
    assert xv is not None or (x.is_cuda and x.is_contiguous())
    assert w_hi.dtype == torch.float32 and w_lo.dtype == torch.float32
    for t in (residual, upsample):
        assert t is None or (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous())
    d = ConvF32Desc()
    out = _conv_setup(d, d, x, cout, ksize, stride, out_mode, out, sink, tile_tab, OUT_NHWC_F32, torch.float32)
    d.w_hi, d.w_lo = w_hi.data_ptr(), w_lo.data_ptr()
    d.bias = bias.data_ptr() if bias is not None else None
    d.residual = residual.data_ptr() if residual is not None else None
    d.upsample = upsample.data_ptr() if upsample is not None else None
    d.stride, d.relu, d.out_mode = int(stride), int(relu), out_mode
    _lib.check(_lib.lib().odtk_conv2d_f32(ctypes.byref(d), _stream()), "conv2d_f32")
    _conv_launched("_f32", 4, x, cout, ksize, stride, out_mode, OUT_NHWC_F32, tile_tab, (w_hi.numel() + w_lo.numel()) * 4,
                residual, upsample)
    return out


def stem_conv_f32(xp, h, wd, w_hi, w_lo, bias, cout, relu=True):
    """7x7 stride-2 pad-3 stem over the NHWC4 fp32 image [N, h+6, wd+8, 4] (pad_input_f32 / preprocess_u8_f32):
    odtk_conv2d_f32 with ksize 7.  Returns NHWC fp32 [N, (h-1)/2+1, (wd-1)/2+1, cout]."""
    assert xp.dtype == torch.float32 and xp.is_contiguous() and xp.shape[1:] == (h + 6, wd + 8, 4)
    n = xp.shape[0]
    out = torch.empty((n, (h - 1) // 2 + 1, (wd - 1) // 2 + 1, cout), dtype=torch.float32, device=xp.device)
    d = ConvF32Desc()
    d.x, d.w_hi, d.w_lo, d.y = xp.data_ptr(), w_hi.data_ptr(), w_lo.data_ptr(), out.data_ptr()
    d.bias = bias.data_ptr() if bias is not None else None
    d.n, d.h, d.width, d.cin, d.cout, d.ksize, d.stride = n, h, wd, 3, cout, 7, 2
    d.relu, d.out_mode = int(relu), OUT_NHWC_F32
    _lib.check(_lib.lib().odtk_conv2d_f32(ctypes.byref(d), _stream()), "conv2d_f32")
    STATS["launches"] += 1
    _trace("stem7x7_f32", 2 * out.numel() * 147, xp.numel() * 4 + (w_hi.numel() + w_lo.numel()) * 4 + out.numel() * 4,
           n=n, h=h, w=wd, cin=3, cout=cout, stride=2)
    return out


def pad_input_f32(x):
    """NHWC fp32 RGB batch [N,H,W,3] -> zero-bordered NHWC4 fp32 [N, H+6, W+8, 4] (odtk_pad_input_f32)."""
    n, h, wd, c = x.shape
    assert c == 3 and x.dtype == torch.float32 and x.is_contiguous()
    xp = torch.empty((n, h + 6, wd + 8, 4), dtype=torch.float32, device=x.device)
    _lib.check(_lib.lib().odtk_pad_input_f32(ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(xp.data_ptr()), n, h, wd, _stream()),
               "pad_input_f32")
    STATS["launches"] += 1
    _trace("pad_input_f32", 0, x.numel() * 4 + xp.numel() * 4, n=n, h=h, w=wd, cin=3)
    return xp


def preprocess_u8_f32(images, stride=128, mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """preprocess_u8 into the fp32 NHWC4 stem buffer [N, Hs+6, Ws+8, 4] (odtk_preprocess_u8_f32): the normalised values
    without the fp16 rounding.  Returns (buffer, Hs, Ws)."""
    assert images.is_cuda and images.dtype == torch.uint8 and images.is_contiguous() and images.shape[-1] == 3
    n, h, w, _ = images.shape
    hs, ws = (h + stride - 1) // stride * stride, (w + stride - 1) // stride * stride
    xp = torch.empty((n, hs + 6, ws + 8, 4), dtype=torch.float32, device=images.device)
    m = (ctypes.c_float * 3)(*mean)
    s = (ctypes.c_float * 3)(*std)
    _lib.check(_lib.lib().odtk_preprocess_u8_f32(ctypes.c_void_p(images.data_ptr()), ctypes.c_void_p(xp.data_ptr()), n, h, w,
                                                 hs, ws, m, s, _stream()), "preprocess_u8_f32")
    STATS["launches"] += 1
    _trace("preprocess_u8_f32", 0, images.numel() + xp.numel() * 4, n=n, h=h, w=w, cin=3)
    return xp, hs, ws


def resize_launch_f32(x_dev, x_bytes, plan, table_dev, out=None, mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """resize_launch into the fp32 NHWC4 stem buffer [n, hs+6, ws+8, 4] (odtk_preprocess_resize_u8_f32)."""
    hs, ws = plan.canvas
    L = _lib.lib()
    nbytes = _lib.check(L.odtk_preprocess_resize_u8_f32(None, x_bytes, ctypes.byref(plan.table), None, plan.n, hs, ws, None,
                                                        None, None, None), "preprocess_resize_u8_f32")
    if out is None:
        out = torch.empty((plan.n, hs + 6, ws + 8, 4), dtype=torch.float32, device=x_dev.device)
    assert out.dtype == torch.float32 and out.is_contiguous() and out.numel() * 4 == nbytes
    m = (ctypes.c_float * 3)(*mean)
    s = (ctypes.c_float * 3)(*std)
    _lib.check(L.odtk_preprocess_resize_u8_f32(ctypes.c_void_p(x_dev.data_ptr()), x_bytes, ctypes.byref(plan.table),
                                               ctypes.c_void_p(table_dev.data_ptr()), plan.n, hs, ws,
                                               ctypes.c_void_p(out.data_ptr()), m, s, _stream()), "preprocess_resize_u8_f32")
    STATS["launches"] += 1
    _trace("preprocess_resize_u8_f32", 0, resize_bytes(plan) + plan.n * (hs + 6) * (ws + 8) * 8, n=plan.n, h=hs, w=ws, cin=3)
    return out


def maxpool3x3s2_f32(x):
    """3x3 stride-2 pad-1 max-pool of NHWC fp32 [N,H,W,C] (odtk_maxpool3x3s2_f32)."""
    n, h, w, c = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous()
    out = torch.empty((n, (h - 1) // 2 + 1, (w - 1) // 2 + 1, c), dtype=torch.float32, device=x.device)
    _lib.check(_lib.lib().odtk_maxpool3x3s2_f32(ctypes.c_void_p(x.data_ptr()), ctypes.c_void_p(out.data_ptr()), n, h, w, c,
                                                _stream()), "maxpool3x3s2_f32")
    STATS["launches"] += 1
    _trace("maxpool_f32", 0, x.numel() * 4 + out.numel() * 4, n=n, h=h, w=w, cin=c)
    return out


# ---- training: backward of the 3x3 stride-1 head convolutions -----------------------------------------------------------
class WgradDesc(ctypes.Structure):
    """odtk_wgrad_t (include/odtk_b200.h)."""
    _fields_ = [("g", ctypes.c_void_p), ("x", ctypes.c_void_p), ("dw", ctypes.c_void_p), ("db", ctypes.c_void_p)] + \
               [(f, ctypes.c_int) for f in ("n", "h", "width", "cin", "cout", "cout_pad")] + \
               [("tile_tab", ctypes.c_void_p), ("tab_tiles", ctypes.c_int)]


class GradLevel(ctypes.Structure):
    """odtk_grad_level_t (include/odtk_b200.h)."""
    _fields_ = [("grad", ctypes.c_void_p), ("height", ctypes.c_int), ("width", ctypes.c_int), ("row0", ctypes.c_int)]


class ConvDgradDesc(ctypes.Structure):
    """odtk_conv_dgrad_t (include/odtk_b200.h)."""
    _fields_ = [("base", ConvDesc), ("mask", ctypes.c_void_p)]


def pad64(c):
    return (c + 63) // 64 * 64


def _tab_px(n, h, w, tile_tab):
    """Pixels a launch covers: n * h * w dense, or the pixels of the levels a tile table lists."""
    if tile_tab is None:
        return n * h * w
    return n * int(((tile_tab[:, 2] - tile_tab[:, 0]).clamp(max=8) * (tile_tab[:, 3] - tile_tab[:, 1]).clamp(max=16)).sum())


def pack_weight_dgrad(weight, cout_pad=None):
    """Weights of the input gradient of a 3x3 (or 1x1) stride-1 convolution: [Cout, Cin, k, k] -> the forward convolution
    with Cin outputs over Cout_pad inputs (pad_out zero-padded to a multiple of 64), rotated by 180 degrees:
    w'[ci, co, ky, kx] = w[co, ci, k - 1 - ky, k - 1 - kx], packed like pack_weight ([Cin, k * k * Cout_pad] fp16)."""
    cout, cin, kh, kw = weight.shape
    assert kh == kw and kh in (1, 3)
    cout_pad = pad64(cout) if cout_pad is None else cout_pad
    w = weight.detach().float()
    if cout_pad > cout:
        w = torch.cat([w, w.new_zeros((cout_pad - cout, cin, kh, kw))], dim=0)
    out = pack_weight(w.transpose(0, 1).flip(2, 3))
    _trace("pack_weight_dgrad", 0, weight.numel() * 4 + out.numel() * 2, cin=cin, cout=cout)
    return out


def _wgrad_launch(name, d, g, x, cout, ksize, bias):
    """odtk_<name> on descriptor d (its geometry filled) into new fp32 dw [cout, Cin, k, k], db [cout] or None."""
    dw = torch.empty((cout, x.shape[3], ksize, ksize), dtype=torch.float32, device=g.device)
    db = torch.empty((cout,), dtype=torch.float32, device=g.device) if bias else None
    d.g, d.x, d.dw, d.db = g.data_ptr(), x.data_ptr(), dw.data_ptr(), (db.data_ptr() if db is not None else None)
    f = getattr(_lib.lib(), "odtk_" + name)
    size = _lib.check(f(ctypes.byref(d), None, 0, None), name + " (workspace query)")
    ws = torch.empty(int(size), dtype=torch.uint8, device=g.device)
    _lib.check(f(ctypes.byref(d), ctypes.c_void_p(ws.data_ptr()), size, _stream()), name)
    STATS["launches"] += 1
    return dw, db, size


def conv_wgrad(g, x, cout, tile_tab=None, bias=True):
    """Weight (and bias) gradient of a 3x3 stride-1 pad-1 convolution (odtk_conv_wgrad): g NHWC fp16 [N, H, W, Cout_pad]
    (the gradient w.r.t. its output before the ReLU, zero outside the levels and in the channels >= cout), x NHWC fp16
    [N, H, W, Cin] (its input).  tile_tab: both are whole atlases and only the listed tiles count.  Returns fp32
    (dw [cout, Cin, 3, 3], db [cout] or None), bit-identical run to run."""
    assert g.is_cuda and g.dtype == torch.float16 and g.is_contiguous()
    assert x.is_cuda and x.dtype == torch.float16 and x.is_contiguous()
    n, h, wd, cpad = g.shape
    cin = x.shape[3]
    assert tuple(x.shape[:3]) == (n, h, wd)
    d = WgradDesc()
    d.n, d.h, d.width, d.cin, d.cout, d.cout_pad = n, h, wd, cin, cout, cpad
    if tile_tab is not None:
        d.tile_tab, d.tab_tiles = tile_tab.data_ptr(), tile_tab.shape[0]
    dw, db, size = _wgrad_launch("conv_wgrad", d, g, x, cout, 3, bias)
    if STATS["trace"] is not None:
        px = _tab_px(n, h, wd, tile_tab)
        # G once per output-channel tile row, X once per tap; the fp32 partials and the result
        _trace("wgrad3x3", 2 * px * cout * 9 * cin, px * (cpad + cin) * 2 + int(size) * 2 + dw.numel() * 4,
               n=n, h=h, w=wd, cin=cin, cout=cout)
    return dw, db


class WgradExDesc(ctypes.Structure):
    """odtk_wgrad_ex_t (include/odtk_b200.h)."""
    _fields_ = [("g", ctypes.c_void_p), ("x", ctypes.c_void_p), ("dw", ctypes.c_void_p), ("db", ctypes.c_void_p)] + \
               [(f, ctypes.c_int) for f in ("n", "g_rows", "g_width", "g_row0", "cout_pad", "x_h", "x_width", "cin", "cout",
                                            "ksize", "stride")] + \
               [("tile_tab", ctypes.c_void_p), ("tab_tiles", ctypes.c_int), ("row_scale", ctypes.c_void_p)]


def conv_wgrad_ex(g, x, cout, ksize, stride, tile_tab, g_row0, bias=True, row_scale=None):
    """Weight (and bias) gradient of an FPN or backbone convolution (odtk_conv_wgrad_ex): 1x1 stride 1, 3x3 stride 1 or 3x3
    stride 2 (pad ksize // 2), and with a dense g 1x1 stride 2.  g: the NHWC fp16 gradient atlas [N, rows, width,
    Cout_pad] whose level at row g_row0 is the convolution's output ((H - 1) // stride + 1 rows and columns; zero in its
    tiles outside the level and in the channels >= cout), tile_tab: that level's slice of the atlas tile table; or, with
    tile_tab None (g_row0 0), g is that dense output itself.  x: the dense NHWC fp16 input [N, H, W, Cin].  row_scale:
    fp32 [cout] on the device or None, multiplies dw's rows (d/dw of a BatchNorm-folded weight w * row_scale).  Returns
    fp32 (dw [cout, Cin, k, k], db [cout] or None: the level's rows only), bit-identical run to run."""
    assert g.is_cuda and g.dtype == torch.float16 and g.is_contiguous()
    assert x.is_cuda and x.dtype == torch.float16 and x.is_contiguous() and x.device == g.device
    assert tile_tab is None or (tile_tab.is_contiguous() and tile_tab.device == g.device)
    assert row_scale is None or (row_scale.device == g.device and row_scale.dtype == torch.float32 and
                                 row_scale.is_contiguous() and row_scale.numel() == cout)
    n, rows, aw, cpad = g.shape
    xn, xh, xw, cin = x.shape
    assert xn == n
    d = WgradExDesc()
    d.n, d.g_rows, d.g_width, d.g_row0, d.cout_pad = n, rows, aw, int(g_row0), cpad
    d.x_h, d.x_width, d.cin, d.cout, d.ksize, d.stride = xh, xw, cin, cout, ksize, stride
    if tile_tab is not None:
        d.tile_tab, d.tab_tiles = tile_tab.data_ptr(), tile_tab.shape[0]
    d.row_scale = row_scale.data_ptr() if row_scale is not None else None
    dw, db, size = _wgrad_launch("conv_wgrad_ex", d, g, x, cout, ksize, bias)
    if STATS["trace"] is not None:
        px = n * ((xh - 1) // stride + 1) * ((xw - 1) // stride + 1)
        # the level's G once, X once per tap (1x1 and stride 2: the pixels it samples), the fp32 partials and the result
        xpx = n * xh * xw if (ksize == 3 and stride == 1) else px
        _trace("wgrad%dx%d%s" % (ksize, ksize, "s2" if stride == 2 else ""), 2 * px * cout * ksize * ksize * cin,
               px * cpad * 2 + xpx * cin * 2 + int(size) * 2 + dw.numel() * 4, n=n, h=xh, w=xw, cin=cin, cout=cout,
               stride=stride)
    return dw, db


def _level_args(atlas, level):
    n, rows, aw, c = atlas.shape
    return [n, rows, aw, c] + [int(v) for v in level]


def pool_add(src, dst, src_level, dst_level, pool=2):
    """dst level += the pool x pool window sums of the src level (odtk_pool_add_f16), both NHWC fp16 atlases of one
    geometry, levels (row0, h, w): pool 2 is the backward of the FPN's nearest 2x upsample-add, pool 1 a plain add.
    fp16_rn((float)dst + ((s00 + s01) + (s10 + s11))).  src may be dst when the levels' rows are disjoint."""
    for t in (src, dst):
        assert t.is_cuda and t.dtype == torch.float16 and t.is_contiguous() and t.shape == dst.shape
    args = _level_args(dst, src_level) + [int(v) for v in dst_level] + [pool]
    _lib.check(_lib.lib().odtk_pool_add_f16(ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(dst.data_ptr()), *args,
                                            _stream()), "pool_add_f16")
    STATS["launches"] += 1
    n, _, _, c = dst.shape
    px = n * int(dst_level[1]) * int(dst_level[2])
    _trace("pool_add", px * c * pool * pool, px * c * 2 * (2 + pool * pool), n=n, h=int(dst_level[1]), w=int(dst_level[2]),
           cin=c, cout=c)
    return dst


def dilate(src, dst, src_level, dst_row0):
    """dst[dst_row0 + 2y, 2x] = src level (row0, h, w) [y, x] (odtk_dilate_f16), NHWC fp16 atlases of one geometry;
    nothing else of dst is written."""
    for t in (src, dst):
        assert t.is_cuda and t.dtype == torch.float16 and t.is_contiguous() and t.shape == dst.shape
    args = _level_args(dst, src_level) + [int(dst_row0)]
    _lib.check(_lib.lib().odtk_dilate_f16(ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(dst.data_ptr()), *args, _stream()),
               "dilate_f16")
    STATS["launches"] += 1
    n, _, _, c = dst.shape
    px = n * int(src_level[1]) * int(src_level[2])
    _trace("dilate", 0, px * c * 4, n=n, h=int(src_level[1]), w=int(src_level[2]), cin=c, cout=c)
    return dst


def dilate_into(src, src_level, dst, stride, dst_row0=0):
    """dst[:, dst_row0 + s y, s x] = src level (row0, h, w) [y, x] (odtk_dilate_ex_f16): NHWC fp16 tensors of their own
    geometries (a dense tensor is one level at row 0).  Stride 1 copies an atlas level into a dense tensor; stride 2
    scatters a gradient into a stride-2 layer's input geometry (a zeroed dst keeps zeros at the odd positions)."""
    for t in (src, dst):
        assert t.is_cuda and t.dtype == torch.float16 and t.is_contiguous()
    n, rows, aw, c = src.shape
    assert dst.shape[0] == n and dst.shape[3] == c and dst.device == src.device
    args = [n, c, rows, aw] + [int(v) for v in src_level] + [dst.shape[1], dst.shape[2], int(dst_row0), int(stride)]
    _lib.check(_lib.lib().odtk_dilate_ex_f16(ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(dst.data_ptr()), *args,
                                             _stream()), "dilate_ex_f16")
    STATS["launches"] += 1
    px = n * int(src_level[1]) * int(src_level[2])
    _trace("dilate", 0, px * c * 4, n=n, h=int(src_level[1]), w=int(src_level[2]), cin=c, cout=c, stride=int(stride))
    return dst


def grad_to_atlas(grads, rows0, scale, atlas):
    """Per-level fp32 NCHW loss gradients [B, C, H_l, W_l] * scale (a number, or a one-element fp32 tensor on the atlas's
    device, read there without a host sync) -> the fp16 NHWC gradient atlas [B, rows, width, C_pad]
    (odtk_grad_to_atlas): level l at rows [rows0[l], + H_l), columns [0, W_l); channels >= C are written as 0; nothing
    else is written (the caller's atlas is zero there).  fp16 overflow is +-inf."""
    assert atlas.is_cuda and atlas.dtype == torch.float16 and atlas.is_contiguous()
    b, rows, aw, cpad = atlas.shape
    ch = grads[0].shape[1]
    gs = [t.float().contiguous() for t in grads]
    assert all(t.device == atlas.device for t in gs)
    sc = (scale if torch.is_tensor(scale) else torch.tensor(float(scale))).to(atlas.device, torch.float32).reshape(1).contiguous()
    levels = (GradLevel * len(gs))()
    for l, (t, r0) in enumerate(zip(gs, rows0)):
        assert t.shape[0] == b and t.shape[1] == ch
        levels[l].grad, levels[l].height, levels[l].width, levels[l].row0 = t.data_ptr(), t.shape[2], t.shape[3], int(r0)
    _lib.check(_lib.lib().odtk_grad_to_atlas(b, len(gs), ctypes.cast(levels, ctypes.c_void_p), ch, ctypes.c_void_p(sc.data_ptr()),
                                             ctypes.c_void_p(atlas.data_ptr()), rows, aw, cpad, _stream()), "grad_to_atlas")
    STATS["launches"] += 1
    px = sum(t.shape[0] * t.shape[2] * t.shape[3] for t in gs)
    _trace("grad_to_atlas", 0, px * ch * 4 + px * cpad * 2, n=b, h=rows, w=aw, cin=ch, cout=cpad)
    return atlas


def conv2d_dgrad(g, w, cout, mask=None, residual=None, tile_tab=None, out=None):
    """Input gradient of a 3x3 or 1x1 stride-1 convolution (odtk_conv2d_dgrad): g NHWC fp16 [N, H, W, Cout_pad] convolved
    with w = pack_weight_dgrad(weight) into NHWC fp16 [N, H, W, cout] (cout = the forward layer's Cin), + residual (same
    shape), then zero wherever mask (NHWC fp16, same shape: the forward layer's input) is not > 0.  tile_tab: whole
    atlases (3x3), only the listed tiles are written (`out` must then be zero outside them).  1x1 (w [cout, Cout_pad]):
    dense, with a mask, cout % 128 == 0.  A stride-2 layer's input gradient is this call on g scattered by dilate_into."""
    assert g.is_cuda and g.dtype == torch.float16 and g.is_contiguous()
    ksize = 3 if w.shape[1] == 9 * g.shape[3] else 1
    assert w.device == g.device and w.dtype == torch.float16 and w.is_contiguous() and w.shape[1] == ksize * ksize * g.shape[3]
    n, h, wd, cpad = g.shape
    if out is None:
        out = (torch.zeros if tile_tab is not None else torch.empty)((n, h, wd, cout), dtype=torch.float16, device=g.device)
    for t in (mask, residual, out):
        assert t is None or (t.device == g.device and t.dtype == torch.float16 and t.is_contiguous() and tuple(t.shape) == (n, h, wd, cout))
    e = ConvDgradDesc()
    d = e.base
    d.x, d.w, d.y = g.data_ptr(), w.data_ptr(), out.data_ptr()
    d.residual = residual.data_ptr() if residual is not None else None
    if tile_tab is not None:
        d.tile_tab, d.tab_tiles = tile_tab.data_ptr(), tile_tab.shape[0]
    d.n, d.h, d.width, d.cin, d.cout, d.ksize = n, h, wd, cpad, cout, ksize
    d.out_mode = OUT_NHWC_F16
    e.mask = mask.data_ptr() if mask is not None else None
    _lib.check(_lib.lib().odtk_conv2d_dgrad(ctypes.byref(e), _stream()), "conv2d_dgrad")
    STATS["launches"] += 1
    if STATS["trace"] is not None:
        px = _tab_px(n, h, wd, tile_tab)
        _trace("dgrad%dx%d" % (ksize, ksize), 2 * px * cout * ksize * ksize * cpad,
               px * cpad * 2 + w.numel() * 2 + px * cout * 2 * (1 + (mask is not None) + (residual is not None)),
               n=n, h=h, w=wd, cin=cpad, cout=cout, residual=residual is not None, mask=mask is not None)
    return out
