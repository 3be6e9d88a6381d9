"""INT8 calibration of the detection heads: activation statistics, threshold selection and calibration tables.

The reference deploys INT8 through a TensorRT engine built with TensorRT's entropy calibrator.  Here the head towers and the
two final head layers run on the s8 wgmma kernel (engine.conv2d_s8); this module picks their 9 per-tensor activation scales
(one for the atlas the FPN writes, one per tower layer output) from fp16 forward passes.  One scale covers all five pyramid
levels, because the atlas is one tensor read by one launch (TensorRT scales P3 ... P7 separately).

Network scope (Model.set_precision("int8", table, scope="network")) also runs ResNet layer3, layer4 and the FPN in INT8; its
tables (format 2) add one scale per tensor that scope quantises (network_tensors), named by state_dict prefix.  The FPN's
smooth / pyramid outputs are the atlas, so they use "heads.input".

Offline code: it uses torch / numpy ops and never runs on the inference path."""
import json

import numpy as np
import torch

FORMAT = 1             # heads scope
FORMAT_NETWORK = 2     # network scope: a superset of the heads scales
SCOPES = ("heads", "network")
NBINS = 2048
LEVELS = 128          # quantisation levels of the symmetric s8 range on one side of zero (TensorRT: 128)
HEADS = ("cls_head", "box_head")
TOWER = (0, 2, 4, 6)
TENSORS = ("heads.input",) + tuple("%s.%d" % (h, i) for h in HEADS for i in TOWER)


def network_tensors(backbone):
    """The tensors the network scope quantises besides the 9 head tensors, in forward order: C3 (layer2's output), then per
    block of layer3 / layer4 its convolutions' ReLU outputs except the last, its downsample output (first block) and the
    block output, then P5, P4 and P3 (lateral5, and lateral4 / lateral3 after the top-down add).  ValueError for a backbone
    the scope does not cover (ResNeXt's grouped 3x3, MobileNetV2)."""
    from .model import RESNET_LAYERS, RESNEXT, network_walk
    if backbone not in RESNET_LAYERS or backbone in RESNEXT:
        raise ValueError("INT8 network scope covers the ResNet18/34/50/101/152 FPN backbones, not %r" % (backbone,))
    walk = network_walk(backbone)
    names = ["backbones.%s.features.layer2" % backbone]
    for blk in walk["blocks"]:
        if blk["level"] >= 4:
            names += [c["y"] for c in blk["convs"][:-1]] + ([blk["down"]["y"]] if blk["down"] else []) + [blk["convs"][-1]["y"]]
    return names + [walk["lateral%d" % k]["y"] for k in (5, 4, 3)]


def max_threshold(absmax):
    """"max" calibration: the threshold is the largest |x| seen."""
    return float(absmax)


def _kl(p, q, eps=1e-4):
    """KL(P || Q) of two count vectors.  Empty bins of Q receive eps counts taken evenly from its non-empty ones (the
    smoothing of the public MXNet implementation of this search): a clipped tail folded into an empty last bin then
    costs a finite divergence instead of ruling the candidate out."""
    nzq = q > 0
    if not nzq.any():
        return np.inf
    q = q + np.where(nzq, -eps * (q.size - nzq.sum()) / nzq.sum(), eps)
    p = p / p.sum()
    q = q / q.sum()
    nz = p > 0
    return float(np.sum(p[nz] * np.log(p[nz] / q[nz])))


def entropy_threshold(hist, absmax, levels=LEVELS):
    """TensorRT's entropy calibration over a |x| histogram of len(hist) bins spanning [0, absmax]: for every candidate
    threshold i = levels ... len(hist) bins, P is the histogram clipped at i with the outliers folded into its last bin, Q
    is hist[:i] quantised to `levels` levels (each level's count spread evenly over its non-empty source bins); the
    threshold is the upper edge of the i with the smallest KL(P || Q) (the largest such i on ties).  The histogram should
    not count exact zeros (Collector leaves them out): they are exact at every scale, and the ReLU outputs' spike of zeros
    in bin 0, spread over a whole level by Q, would otherwise pull the search towards small thresholds."""
    hist = np.asarray(hist, np.float64)
    nbins = len(hist)
    if absmax <= 0 or hist.sum() <= 0:
        return 0.0
    best_i, best_kl = nbins, np.inf
    tail = np.concatenate([np.cumsum(hist[::-1])[::-1], [0.0]])      # tail[i] = sum(hist[i:])
    for i in range(levels, nbins + 1):
        src = hist[:i]
        p = src.copy()
        p[-1] += tail[i]
        idx = (np.arange(i) * levels) // i
        nz = src > 0
        mass = np.bincount(idx, weights=src, minlength=levels)
        cnt = np.bincount(idx, weights=nz.astype(np.float64), minlength=levels)
        q = np.where(nz, mass[idx] / np.maximum(cnt[idx], 1.0), 0.0)
        kl = _kl(p, q)
        if kl <= best_kl:
            best_i, best_kl = i, kl
    return float(best_i) * float(absmax) / nbins


def scale_from_threshold(t):
    """Activation scale (fp32): threshold / 127, or 1 for a tensor that was never non-zero."""
    return float(np.float32(t) / np.float32(127.0)) if t > 0 else 1.0


class Collector:
    """Two passes over the calibration batches: pass 0 records max|x| per tensor, pass 1 a NBINS-bin histogram of the
    non-zero |x| over [0, max|x|].  `observe(name, values)` takes any tensor of the values to count (the valid atlas
    pixels)."""

    def __init__(self):
        self.phase = 0
        self.absmax = {}
        self.hist = {}
        self.count = {}

    def observe(self, name, values):
        a = values.detach().abs().float()
        if self.phase == 0:
            self.absmax[name] = max(self.absmax.get(name, 0.0), float(a.max()) if a.numel() else 0.0)
            self.count[name] = self.count.get(name, 0) + a.numel()
            return
        top = self.absmax[name]
        if top <= 0:
            return
        a = a.flatten()
        h = torch.histc(a[a > 0], bins=NBINS, min=0.0, max=top).double().cpu().numpy()   # exact zeros left out
        self.hist[name] = self.hist.get(name, 0.0) + h

    def thresholds(self, method):
        if method == "max":
            return {n: max_threshold(self.absmax[n]) for n in self.absmax}
        if method == "entropy":
            return {n: entropy_threshold(self.hist.get(n, np.zeros(NBINS)), self.absmax[n]) for n in self.absmax}
        raise ValueError("unknown calibration method %r (max, entropy)" % (method,))

    def scales(self, method, names=TENSORS):
        th = self.thresholds(method)
        missing = [n for n in names if n not in th]
        if missing:
            raise RuntimeError("calibration saw no values for %s" % missing)
        return {n: scale_from_threshold(th[n]) for n in names}


def table_tensors(backbone, scope="heads"):
    return TENSORS + (tuple(network_tensors(backbone)) if scope == "network" else ())


def make_table(backbone, classes, num_anchors, method, images, scales, scope="heads"):
    t = {"format": FORMAT, "backbone": backbone, "classes": int(classes), "num_anchors": int(num_anchors),
         "method": method, "images": int(images), "scales": {n: float(scales[n]) for n in table_tensors(backbone, scope)}}
    if scope == "network":
        t.update(format=FORMAT_NETWORK, scope="network")
    return t


def save_table(table, path):
    with open(path, "w") as f:
        json.dump(table, f, indent=1, sort_keys=True)


def load_table(table):
    """A table dict, or the path of a JSON file written by save_table."""
    if isinstance(table, dict):
        return table
    with open(table) as f:
        return json.load(f)


def check_table(table, backbone, classes, num_anchors, scope="heads"):
    """Raises ValueError unless `table` is a calibration table of this model for `scope`: "heads" takes a format-1 table or
    a format-2 network table (whose head scales it uses), "network" only a format-2 one."""
    if scope not in SCOPES:
        raise ValueError("INT8 scope must be 'heads' or 'network', got %r" % (scope,))
    if not isinstance(table, dict) or table.get("format") not in (FORMAT, FORMAT_NETWORK):
        raise ValueError("not an INT8 calibration table (format %d or %d)" % (FORMAT, FORMAT_NETWORK))
    if table["format"] == FORMAT_NETWORK and table.get("scope") != "network":
        raise ValueError("a format-%d calibration table must have scope 'network'" % FORMAT_NETWORK)
    if scope == "network" and table["format"] != FORMAT_NETWORK:
        raise ValueError("INT8 network scope needs a network calibration table (format %d): calibrate(..., scope='network')"
                         % FORMAT_NETWORK)
    for key, want in (("backbone", backbone), ("classes", classes), ("num_anchors", num_anchors)):
        if table.get(key) != want:
            raise ValueError("calibration table is for %s=%r, the model has %r" % (key, table.get(key), want))
    scales = table.get("scales", {})
    names = table_tensors(backbone, "network" if table["format"] == FORMAT_NETWORK else "heads")
    bad = [n for n in names if not (isinstance(scales.get(n), (int, float)) and scales[n] > 0 and np.isfinite(scales[n]))]
    if bad:
        raise ValueError("calibration table lacks a positive scale for %s" % bad)
    return table


def layer_scales(scales, head):
    """[(s_in, inv_out)] for the 5 layers of `head` as fp32 numbers: layer k reads the tensor scaled by s_in; tower layers
    requantise their output with inv_out = 1 / s_out (fp32 division), the final layer has inv_out None."""
    names = ["heads.input"] + ["%s.%d" % (head, i) for i in TOWER]
    out = []
    for k in range(5):
        s_in = np.float32(scales[names[k]])
        inv = np.float32(1.0) / np.float32(scales[names[k + 1]]) if k < 4 else None
        out.append((s_in, inv))
    return out
