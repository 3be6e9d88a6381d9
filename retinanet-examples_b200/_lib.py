"""ctypes loader for libodtk_b200.so (the C ABI declared in include/odtk_b200.h).

The library is built in-tree by `make -C retinanet-examples_b200/csrc` (see
__graft_entry__.build).  Loading fails loudly: there is no fallback implementation."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ODTK_B200_LIB", os.path.join(_HERE, "libodtk_b200.so"))  # override: A/B builds

ODTK_OK = 0
_ERRORS = {-1: "invalid argument", -2: "workspace is too small", -3: "size not supported by the sm_90a kernels",
           -4: "CUDA runtime error"}

_c_vpp = ctypes.POINTER(ctypes.c_void_p)
_c_f32p = ctypes.POINTER(ctypes.c_float)

# name -> (restype, argtypes); must list every symbol include/odtk_b200.h declares
SIGNATURES = {
    "odtk_b200_version": (ctypes.c_char_p, []),
    "odtk_decode": (ctypes.c_longlong, [ctypes.c_int, _c_vpp, _c_vpp] + [ctypes.c_size_t] * 5 +
                    [_c_f32p, ctypes.c_size_t, ctypes.c_float, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t,
                     ctypes.c_void_p]),
    "odtk_decode_rotate": (ctypes.c_longlong, [ctypes.c_int, _c_vpp, _c_vpp] + [ctypes.c_size_t] * 5 +
                           [_c_f32p, ctypes.c_size_t, ctypes.c_float, ctypes.c_int, ctypes.c_void_p,
                            ctypes.c_size_t, ctypes.c_void_p]),
    "odtk_decode_ex": (ctypes.c_longlong, [ctypes.c_int, _c_vpp, _c_vpp] + [ctypes.c_size_t] * 5 +
                       [_c_f32p, ctypes.c_size_t, ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_size_t,
                        ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "odtk_decode_levels": (ctypes.c_longlong, [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t,
                                               ctypes.c_size_t, ctypes.c_size_t, ctypes.c_float, ctypes.c_int,
                                               ctypes.c_int, _c_vpp, ctypes.c_size_t, ctypes.c_size_t,
                                               ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "odtk_decode_fused_begin": (ctypes.c_longlong, [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t,
                                                    ctypes.c_size_t, ctypes.c_float, ctypes.c_int, ctypes.c_void_p,
                                                    ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "odtk_decode_fused_finish": (ctypes.c_longlong, [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t,
                                                     ctypes.c_size_t, ctypes.c_size_t, ctypes.c_float, ctypes.c_int,
                                                     ctypes.c_int, _c_vpp, ctypes.c_size_t, ctypes.c_size_t,
                                                     ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "odtk_nms": (ctypes.c_longlong, [ctypes.c_int, _c_vpp, _c_vpp, ctypes.c_size_t, ctypes.c_int, ctypes.c_float,
                                     ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "odtk_nms_rotate": (ctypes.c_longlong, [ctypes.c_int, _c_vpp, _c_vpp, ctypes.c_size_t, ctypes.c_int,
                                            ctypes.c_float, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "odtk_nms_ex": (ctypes.c_longlong, [ctypes.c_int, _c_vpp, _c_vpp, ctypes.c_size_t, ctypes.c_int, ctypes.c_float,
                                        ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                        ctypes.c_size_t, ctypes.c_void_p]),
    "odtk_nms_gather": (ctypes.c_longlong, [ctypes.c_int, _c_vpp, _c_vpp, ctypes.c_size_t, ctypes.c_int, ctypes.c_float,
                                            ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                            ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "odtk_gather_wait": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]),
    "odtk_iou": (ctypes.c_int, [_c_vpp, _c_vpp, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "odtk_conv2d": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    "odtk_conv2d_s8": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    "odtk_conv2d_s8_ex": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    "odtk_relu_copy_rows_s8": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int] +
                               [ctypes.c_longlong] * 4 + [ctypes.c_void_p]),
    "odtk_conv2d_f32": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    "odtk_conv_wgrad": (ctypes.c_longlong, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "odtk_conv_wgrad_ex": (ctypes.c_longlong, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]),
    "odtk_pool_add_f16": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 11 + [ctypes.c_void_p]),
    "odtk_dilate_f16": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 8 + [ctypes.c_void_p]),
    "odtk_grad_to_atlas": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                          ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "odtk_conv2d_dgrad": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    "odtk_pad_input_f32": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "odtk_preprocess_u8_f32": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 5 + [_c_f32p, _c_f32p, ctypes.c_void_p]),
    "odtk_preprocess_resize_u8_f32": (ctypes.c_longlong, [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p] +
                                      [ctypes.c_int] * 3 + [ctypes.c_void_p, _c_f32p, _c_f32p, ctypes.c_void_p]),
    "odtk_maxpool3x3s2_f32": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_void_p]),
    "odtk_relu_copy_rows_f32": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int] +
                                [ctypes.c_longlong] * 4 + [ctypes.c_void_p]),
    "odtk_quantize_f16_s8": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_float, ctypes.c_void_p]),
    "odtk_conv_last_plan": (ctypes.c_int, [ctypes.c_void_p]),
    "odtk_conv_map_cache_stats": (ctypes.c_int, [ctypes.POINTER(ctypes.c_longlong), ctypes.POINTER(ctypes.c_longlong)]),
    "odtk_conv_pack_bias": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]),
    "odtk_lower_conv": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 9 + [ctypes.c_void_p]),
    "odtk_copy_rows_f16": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int] +
                           [ctypes.c_longlong] * 4 + [ctypes.c_int, ctypes.c_void_p]),
    "odtk_relu_f16": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p]),
    "odtk_maxpool3x3s2": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_void_p]),
    "odtk_stem_conv": (ctypes.c_int, [ctypes.c_void_p] * 4 + [ctypes.c_int] * 5 + [ctypes.c_void_p]),
    "odtk_stem_pool": (ctypes.c_int, [ctypes.c_void_p] * 4 + [ctypes.c_int] * 5 + [ctypes.c_void_p]),
    "odtk_bottleneck_tail": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    "odtk_set_sm_budget": (ctypes.c_int, [ctypes.c_int]),
    "odtk_peer_alloc": (ctypes.c_int, [ctypes.c_size_t, ctypes.POINTER(ctypes.c_void_p), ctypes.c_void_p]),
    "odtk_peer_open": (ctypes.c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p)]),
    "odtk_peer_close": (ctypes.c_int, [ctypes.c_void_p]),
    "odtk_peer_free": (ctypes.c_int, [ctypes.c_void_p]),
    "odtk_depthwise3x3": (ctypes.c_int, [ctypes.c_void_p] * 4 + [ctypes.c_int] * 6 + [ctypes.c_void_p]),
    "odtk_pad_input": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    "odtk_focal_loss": (ctypes.c_longlong, [ctypes.c_void_p] * 4 + [ctypes.c_longlong, ctypes.c_int, ctypes.c_int,
                                            ctypes.c_float, ctypes.c_float, ctypes.c_float] + [ctypes.c_void_p] * 4 +
                        [ctypes.c_size_t, ctypes.c_void_p]),
    "odtk_smooth_l1_loss": (ctypes.c_longlong, [ctypes.c_void_p] * 3 + [ctypes.c_longlong, ctypes.c_float, ctypes.c_float] +
                            [ctypes.c_void_p] * 4 + [ctypes.c_size_t, ctypes.c_void_p]),
    "odtk_retina_loss": (ctypes.c_longlong, [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                             ctypes.c_float, ctypes.c_float, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p,
                                             ctypes.c_size_t, ctypes.c_void_p]),
    "odtk_snap_to_anchors": (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 5 + [_c_f32p, ctypes.c_int, ctypes.c_int,
                                            ctypes.c_float, ctypes.c_float] + [ctypes.c_void_p] * 5),
    "odtk_preprocess_u8": (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 5 + [_c_f32p, _c_f32p, ctypes.c_void_p]),
    "odtk_preprocess_resize_u8": (ctypes.c_longlong, [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p] +
                                  [ctypes.c_int] * 3 + [ctypes.c_void_p, _c_f32p, _c_f32p, ctypes.c_void_p]),
    "odtk_decode_jpeg": (ctypes.c_longlong, [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p,
                                             ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t,
                                             ctypes.c_void_p, ctypes.c_void_p]),
    "odtk_prof_enable": (None, [ctypes.c_int]),
    "odtk_prof_reset": (None, []),
    "odtk_prof_get_list": (ctypes.c_longlong, [ctypes.c_int, ctypes.POINTER(ctypes.c_float), ctypes.c_longlong]),
    "odtk_prof_get": (ctypes.c_int, [ctypes.c_int, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_longlong)]),
}



class Level(ctypes.Structure):
    """odtk_level_t (include/odtk_b200.h)."""
    _fields_ = [("scores", ctypes.c_void_p), ("deltas", ctypes.c_void_p), ("height", ctypes.c_size_t),
                ("width", ctypes.c_size_t), ("scale", ctypes.c_size_t), ("anchors", _c_f32p)]


class Gather(ctypes.Structure):
    """odtk_gather_t (include/odtk_b200.h)."""
    _fields_ = [("packed", ctypes.c_void_p * 8), ("flags", ctypes.c_void_p * 8), ("epoch", ctypes.c_void_p),
                ("num_peers", ctypes.c_int), ("rank", ctypes.c_int)]


class LossLevel(ctypes.Structure):
    """odtk_loss_level_t (include/odtk_b200.h)."""
    _fields_ = [("cls_logits", ctypes.c_void_p), ("box_pred", ctypes.c_void_p), ("cls_index", ctypes.c_void_p),
                ("box_target", ctypes.c_void_p), ("cls_grad", ctypes.c_void_p), ("box_grad", ctypes.c_void_p),
                ("height", ctypes.c_int), ("width", ctypes.c_int)]


class ConvPlan(ctypes.Structure):
    """odtk_conv_plan_t (include/odtk_b200.h)."""
    _fields_ = [(n, ctypes.c_int) for n in ("mode", "cluster", "bn", "num_m_tiles", "num_n_tiles", "nstages", "npatch",
                                            "tile_t", "b_resident", "bias_mma", "res_mma", "tma_store", "th", "tw", "grid",
                                            "up_mma")]


class BneckDesc(ctypes.Structure):
    """odtk_bneck_t (include/odtk_b200.h)."""
    _fields_ = [("x", ctypes.c_void_p), ("w2", ctypes.c_void_p), ("w3", ctypes.c_void_p), ("residual", ctypes.c_void_p),
                ("b2", ctypes.c_void_p), ("b3", ctypes.c_void_p), ("y", ctypes.c_void_p),
                ("n", ctypes.c_int), ("h", ctypes.c_int), ("width", ctypes.c_int), ("c1", ctypes.c_int), ("c2", ctypes.c_int),
                ("relu", ctypes.c_int), ("xproj", ctypes.c_void_p), ("wproj", ctypes.c_void_p),
                ("w_next", ctypes.c_void_p), ("b_next", ctypes.c_void_p), ("z", ctypes.c_void_p), ("c_next", ctypes.c_int)]


class ResizeImage(ctypes.Structure):
    """odtk_resize_image_t (include/odtk_b200.h)."""
    _fields_ = [("offset", ctypes.c_longlong), ("src_h", ctypes.c_int), ("src_w", ctypes.c_int), ("dst_h", ctypes.c_int),
                ("dst_w", ctypes.c_int)]


class JpegImage(ctypes.Structure):
    """odtk_jpeg_image_t (include/odtk_b200.h)."""
    _fields_ = [("scan_offset", ctypes.c_longlong), ("blk_base", ctypes.c_longlong), ("pix_base", ctypes.c_longlong)] + \
               [(f, ctypes.c_int) for f in ("scan_bytes", "height", "width", "ncomp", "hmax", "vmax", "restart_interval", "nseg",
                                            "seg_base")] + [(f, ctypes.c_int * 3) for f in ("quant", "dc", "ac")]


class JpegHuff(ctypes.Structure):
    """odtk_jpeg_huff_t (include/odtk_b200.h)."""
    _fields_ = [("look", ctypes.c_uint16 * 256), ("maxcode", ctypes.c_int * 18), ("valoff", ctypes.c_int * 18),
                ("val", ctypes.c_uint8 * 256)]


class CandSink(ctypes.Structure):
    """odtk_cand_sink_t (include/odtk_b200.h)."""
    _fields_ = [("counts", ctypes.c_void_p), ("hist", ctypes.c_void_p), ("cand", ctypes.c_void_p),
                ("cap", ctypes.c_longlong), ("key_thresh", ctypes.c_uint32), ("shift", ctypes.c_int),
                ("hist_bins", ctypes.c_int), ("thresh", ctypes.c_float)]


_LIB = None


def lib():
    """Returns the loaded library; raises RuntimeError if it has not been built."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "libodtk_b200.so is missing (%s): build it with `make -C retinanet-examples_b200/csrc` or "
                "`python -c 'import __graft_entry__ as g; g.build()'`. There is no CPU fallback." % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _LIB = L
    return _LIB


def check(rc, what):
    if rc < 0:
        raise RuntimeError("%s failed: %s (code %d)" % (what, _ERRORS.get(int(rc), "unknown error"), rc))
    return rc


def ptr_array(ptrs):
    return (ctypes.c_void_p * len(ptrs))(*[ctypes.c_void_p(p) for p in ptrs])
