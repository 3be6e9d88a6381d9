"""GPU tests of the raw-image input side (odtk_preprocess_resize_u8, engine.preprocess_resize_u8, Model.forward_images,
infer.infer_images): the kernel's stem buffer is bit-identical to Pillow's BILINEAR resize (digests in tests/golden/resize_pil.npz)
followed by the reference's normalisation and padding, and to the numpy resampler (tests/resize_oracle.py) on random
sizes; ragged batches equal the reference collate; detections equal the network run on the batch built on the CPU,
eager and under CUDA graphs."""
import ctypes
import os

import numpy as np
import pytest
import torch

import resize_oracle
from oracle import oracle
from retinanet_examples_b200 import _lib, engine, infer
from retinanet_examples_b200.model import Model, make_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _stem_buffer(pre, canvas):
    """float32 [3, h, w] (oracle.preprocess_u8 of one image) -> the fp16 NHWC4 stem buffer [canvas_h+6, canvas_w+8, 4]."""
    hs, ws = canvas
    out = torch.zeros((hs + 6, ws + 8, 4), dtype=torch.float16)
    out[3:3 + pre.shape[1], 3:3 + pre.shape[2], :3] = torch.from_numpy(pre).permute(1, 2, 0).half()
    return out


def _reference_batch(images, resize, max_size, canvas=None, stride=128):
    """The reference's data loader on the CPU: PIL-exact resize, normalise, stride pad (odtk/data.py:55-123), collate to
    the batch maximum (:154-176).  Returns (float32 [n, 3, hs, ws], NHWC4 fp16 stem buffers, ratios)."""
    pres, ratios = [], []
    for im in images:
        ratio, dh, dw = resize_oracle.resize_ratio(im.shape[0], im.shape[1], resize, max_size)
        pres.append(oracle.preprocess_u8(resize_oracle.resize_bilinear(np.asarray(im), dh, dw), stride))
        ratios.append(ratio)
    hs = max(p.shape[1] for p in pres) if canvas is None else canvas[0]
    ws = max(p.shape[2] for p in pres) if canvas is None else canvas[1]
    x = np.zeros((len(pres), 3, hs, ws), np.float32)
    for i, p in enumerate(pres):
        x[i, :, :p.shape[1], :p.shape[2]] = p
    return torch.from_numpy(x), torch.stack([_stem_buffer(p, (hs, ws)) for p in pres]), torch.tensor(ratios, dtype=torch.float32)


def _images(shapes, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, generator=g) for h, w in shapes]


# ---- the kernel ------------------------------------------------------------------------------------------------------
def test_kernel_matches_pil_fixture(golden_dir):
    g = np.load(os.path.join(golden_dir, "resize_pil.npz"))
    resize, max_size = int(g["resize"]), int(g["max_size"])
    for name in g["names"]:
        img = torch.from_numpy(g[name + "_img"])
        pre = oracle.preprocess_u8(resize_oracle.fixture_output(g, name))          # Pillow's output, digest-checked
        want = _stem_buffer(pre, pre.shape[1:])
        for src in (img, img.to(DEV)):                       # staged through pinned memory / read in place
            xp, hs, ws, ratios = engine.preprocess_resize_u8([src], resize, max_size)
            assert (hs + 6, ws + 8) == tuple(want.shape[:2]), name
            assert float(ratios[0]) == np.float32(g[name + "_ratio"])
            assert torch.equal(xp[0].cpu(), want), name


def _launch_pairs(srcs, dsts):
    """One launch over images with explicit dst sizes; canvas = the largest even-rounded dst.  Returns the buffer."""
    plan = engine.ResizePlan([s.shape[:2] for s in srcs], 4000, 1 << 30)
    for t, (dh, dw) in zip(plan.table, dsts):
        t.dst_h, t.dst_w = dh, dw
    plan.canvas = (max(-(-d[0] // 2) * 2 for d in dsts), max(-(-d[1] // 2) * 2 for d in dsts))
    buf = torch.empty(engine.table_pad(plan.n) + plan.nbytes, dtype=torch.uint8, device=DEV)
    tab, x = engine.stage_images([torch.from_numpy(s) for s in srcs], plan, buf)
    return engine.resize_launch(x, plan.nbytes, plan, tab).cpu(), plan.canvas


def test_random_sizes_match_numpy_oracle():
    """50 seeded (src, dst) pairs, 1-4000 px per side, up and down (some beyond the shared-memory tap tables' 7x)."""
    rng = np.random.default_rng(7)
    pairs = []
    while len(pairs) < 50:
        sh, sw, dh, dw = (int(v) for v in np.exp(rng.uniform(0, np.log(4000), 4)).round().clip(1, 4000))
        if sh * sw > 3_000_000 or dh * dw > 3_000_000 or (2 * sh / dh + 2) * (2 * sw / dw + 2) > 20000:
            continue
        pairs.append((sh, sw, dh, dw))
    assert any(p[0] > 7 * p[2] or p[1] > 7 * p[3] for p in pairs) and any(p[0] < p[2] for p in pairs)
    for k in range(0, len(pairs), 5):
        group = pairs[k:k + 5]
        srcs = [rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8) for sh, sw, _, _ in group]
        got, canvas = _launch_pairs(srcs, [(dh, dw) for _, _, dh, dw in group])
        for i, (s, (sh, sw, dh, dw)) in enumerate(zip(srcs, group)):
            want = _stem_buffer(oracle.preprocess_u8(resize_oracle.resize_bilinear(s, dh, dw), 2), canvas)
            assert torch.equal(got[i], want), (sh, sw, dh, dw)


def test_ragged_batch_equals_reference_collate():
    imgs = _images([(240, 320), (300, 200), (97, 161), (512, 300)], 3)
    _, want, ratios = _reference_batch(imgs, 320, 512)
    xp, hs, ws, r = engine.preprocess_resize_u8(imgs, 320, 512)
    assert (hs, ws) == (512, 512) and torch.equal(r, ratios)
    assert torch.equal(xp.cpu(), want)
    # an explicit larger canvas: the same images at the top left, zeros around
    _, want, _ = _reference_batch(imgs, 320, 512, canvas=(640, 768))
    xp, hs, ws, _ = engine.preprocess_resize_u8([i.to(DEV) for i in imgs], 320, 512, canvas=(640, 768))
    assert (hs, ws) == (640, 768) and torch.equal(xp.cpu(), want)


def test_error_cases():
    img = torch.zeros((20, 30, 3), dtype=torch.uint8, device=DEV)
    with pytest.raises(ValueError):
        engine.preprocess_resize_u8([img], 64, 100, canvas=(128, 100))          # canvas not a stride multiple
    with pytest.raises(ValueError):
        engine.preprocess_resize_u8([img], 256, 512, canvas=(128, 128))         # dst 256 x 384 does not fit
    with pytest.raises(ValueError):
        engine.preprocess_resize_u8([], 64, 100)
    plan = engine.ResizePlan([(20, 30)], 64, 100)
    buf = torch.zeros(4096, dtype=torch.uint8, device=DEV)
    L = _lib.lib()
    m = (ctypes.c_float * 3)(*engine.IMAGENET_MEAN)
    y = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    args = lambda tab, n, ch, cw, mean: (ctypes.c_void_p(buf.data_ptr()), 4096, ctypes.byref(tab), ctypes.c_void_p(buf.data_ptr()),
                                          n, ch, cw, ctypes.c_void_p(y.data_ptr()), mean, m, None)
    assert L.odtk_preprocess_resize_u8(*args(plan.table, 1, 128, 128, None)) == -1     # no mean
    assert L.odtk_preprocess_resize_u8(*args(plan.table, 1, 128, 127, m)) == -1        # odd canvas
    assert L.odtk_preprocess_resize_u8(*args(plan.table, 1, 63, 128, m)) == -1         # dst 64 rows
    plan.table[0].src_w = 0
    assert L.odtk_preprocess_resize_u8(*args(plan.table, 1, 128, 128, m)) == -1
    torch.cuda.synchronize()


# ---- the model ---------------------------------------------------------------------------------------------------------
def _spread_head(sd, std=0.05, prior=0.02):
    g = torch.Generator().manual_seed(123)
    sd = dict(sd)
    sd["cls_head.8.weight"] = torch.randn(sd["cls_head.8.weight"].shape, generator=g) * std
    sd["cls_head.8.bias"] = torch.full_like(sd["cls_head.8.bias"], -float(np.log((1 - prior) / prior)))
    sd["box_head.8.weight"] = torch.randn(sd["box_head.8.weight"].shape, generator=g) * 0.02
    return sd


def _model(backbone, x, classes=6, rotated=False, seed=14, keep=300):
    """A model whose score threshold leaves about `keep` candidates on the float batch x (a fresh model has few
    detections at these small sizes)."""
    sd = _spread_head(make_state_dict(backbone, classes, 27 if rotated else 9, rotated, seed))
    m = Model(backbone, classes=classes, rotated_bbox=rotated).load_state_dict(sd).cuda()
    scores = torch.cat([c.flatten() for c in m.forward_heads(x.to(DEV))[0]])
    m.threshold = float(scores.topk(keep).values[-1])
    return m


def _assert_same(a, b):
    for u, v in zip(a, b):
        assert torch.equal(u, v)


@pytest.mark.parametrize("backbone,rotated,shapes,resize,max_size", [
    ("ResNet18FPN", False, [(120, 160), (200, 133), (77, 101)], 256, 400),
    ("ResNet18FPN", True, [(120, 160), (160, 120)], 256, 400),
    ("ResNet50FPN", False, [(480, 640), (427, 640), (640, 480)], 800, 1333)])
def test_forward_images_equals_cpu_built_batch(backbone, rotated, shapes, resize, max_size):
    imgs = _images(shapes, 11)
    x, _, ratios = _reference_batch(imgs, resize, max_size)
    m = _model(backbone, x, rotated=rotated)
    for fused in (True, False):
        m.fused_candidates = fused
        want = [t.clone() for t in m(x.to(DEV))]
        assert (want[0] > 0).sum() > 5
        got, r = m.forward_images(imgs, resize, max_size)
        _assert_same(got, want)
        assert torch.equal(r, ratios)
    m.fused_candidates = True
    m.parallel_heads = False
    got, _ = m.forward_images([i.to(DEV) for i in imgs], resize, max_size)
    _assert_same(got, [t.clone() for t in m(x.to(DEV))])


@pytest.mark.parametrize("scope", ["heads", "network"])
def test_forward_images_int8(scope):
    imgs = _images([(120, 160), (200, 133)], 12)
    x, _, _ = _reference_batch(imgs, 256, 400)
    m = _model("ResNet18FPN", x)
    m.set_precision("int8", m.calibrate([x], scope=scope), scope=scope)
    want = [t.clone() for t in m(x.to(DEV))]
    assert (want[0] > 0).sum() > 5
    got, _ = m.forward_images(imgs, 256, 400)
    _assert_same(got, want)


def test_cuda_graph_replay_and_recapture():
    canvas = (384, 512)
    batches = [_images([(120, 160), (200, 133)], 21), _images([(90, 200), (150, 150)], 22), _images([(300, 400), (333, 250)], 23)]
    xs = [_reference_batch(b, 256, 400, canvas)[0] for b in batches]
    m = _model("ResNet18FPN", xs[0])
    eager = [[t.clone() for t in m.forward_images(b, 256, 400, canvas)[0]] for b in batches]
    for e, x in zip(eager, xs):
        assert (e[0] > 0).sum() > 5
        _assert_same(e, m(x.to(DEV)))
    m.enable_cuda_graph()
    key = ("images", 2, 384, 512)
    out, _ = m.forward_images(batches[0], 256, 400, canvas)
    _assert_same(out, eager[0])
    entry = m._graphs[key]
    out, _ = m.forward_images(batches[1], 256, 400, canvas)             # fewer bytes: same graph
    _assert_same(out, eager[1])
    assert m._graphs[key] is entry
    out, _ = m.forward_images(batches[2], 256, 400, canvas)             # more bytes than staged: grow + capture again
    _assert_same(out, eager[2])
    assert m._graphs[key] is not entry and m._graphs[key]["capacity"] >= sum(i.numel() for i in batches[2])
    entry = m._graphs[key]
    for k in (0, 1, 2, 0):
        _assert_same(m.forward_images(batches[k], 256, 400, canvas)[0], eager[k])
    assert m._graphs[key] is entry
    m.enable_cuda_graph(False)


def test_infer_images_and_detections_to_coco():
    batches = [_images([(120, 160), (200, 133)], 31), _images([(77, 101), (160, 120)], 32)]
    m = _model("ResNet18FPN", _reference_batch(batches[0], 256, 400)[0])
    scores, boxes, classes, ratios = infer.infer_images(m, batches, 256, 400)
    assert scores.shape[0] == 4 and ratios.shape == (4,)
    want = [m.forward_images(b, 256, 400) for b in batches]
    torch.testing.assert_close(ratios, torch.cat([w[1] for w in want]), rtol=0, atol=0)
    assert torch.equal(scores, torch.cat([w[0][0] for w in want]))
    dets = infer.detections_to_coco(scores, boxes, classes, ratios)
    assert len(dets) == int((scores > 0).sum()) > 0
    i = int((scores[:, 0] > 0).nonzero()[0])
    b = (boxes[i, 0].cpu() / ratios[i]).tolist()
    d = [d for d in dets if d["image_id"] == i][0]
    assert d["bbox"] == [b[0], b[1], b[2] - b[0] + 1, b[3] - b[1] + 1]
