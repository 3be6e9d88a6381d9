"""GPU tests of the JPEG decode path (odtk_decode_jpeg, engine.decode_jpeg, Model.forward_jpeg, infer.infer_jpeg): every
fixture of tests/golden/jpeg_pil.npz decodes to exactly Pillow's digest and to the numpy oracle's array, alone and in a
ragged batch; a truncated stream sets its status and leaves the rest of its batch exact; detections of forward_jpeg
equal forward_images on the oracle-decoded images, eager and under CUDA graphs.  No Pillow here."""
import os

import numpy as np
import pytest
import torch

import jpeg_oracle
from retinanet_examples_b200 import engine, infer
from retinanet_examples_b200.model import Model, make_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def fixture(golden_dir):
    return np.load(os.path.join(golden_dir, "jpeg_pil.npz"))


@pytest.fixture(scope="module")
def streams(fixture):
    return jpeg_oracle.fixture_streams(fixture)


def _check(fixture, name, got, want=None):
    got = got.cpu().numpy()
    assert got.shape == tuple(fixture[name + "_shape"]), name
    assert jpeg_oracle.sha256(got) == str(fixture[name + "_pil_sha256"]), name
    if want is not None:
        assert np.array_equal(got, want), name


def test_every_fixture_alone_matches_pillow_and_oracle(fixture, streams):
    for name, data in streams.items():
        imgs, status = engine.decode_jpeg([data])
        assert status.cpu().tolist() == [0], name
        _check(fixture, name, imgs[0], jpeg_oracle.decode(data))


def test_ragged_batch(fixture, streams):
    names = list(streams)
    order = [n for n in names if "640" in n or "480x640" in n] + [n for n in names if "640" not in n]
    rng = np.random.default_rng(3)
    order = [order[0], order[1]] + list(rng.permutation(order[2:]))
    imgs, status = engine.decode_jpeg([streams[n] for n in order])
    assert status.cpu().tolist() == [0] * len(order)
    for n, im in zip(order, imgs):
        _check(fixture, n, im)
    samplings = {jpeg_oracle.jpeg.parse(streams[n]).sampling for n in order}
    assert samplings == {"4:2:0", "4:2:2", "4:4:4", "gray"}


def test_truncated_stream_sets_status(fixture, streams):
    names = ["420_q75", "420_restart3", "gray_restart_rows", "444_480x640"]
    bad = fixture["truncated_jpeg"].tobytes()
    datas = [streams[names[0]], bad, streams[names[1]], streams[names[2]], streams[names[3]]]
    imgs, status = engine.decode_jpeg(datas)
    s = status.cpu().tolist()
    assert s[1] & 4 and s[:1] + s[2:] == [0, 0, 0, 0], s
    for n, im in zip(names, imgs[:1] + imgs[2:]):
        _check(fixture, n, im)
    # a restart-marker stream cut short loses segments: truncated or missing restart markers
    rs = streams["420_restart3"]
    imgs, status = engine.decode_jpeg([rs[:len(rs) // 2], streams["gray_q75"]])
    s = status.cpu().tolist()
    assert s[0] & (4 | 8) and s[1] == 0
    _check(fixture, "gray_q75", imgs[1])


def test_unsupported_streams_raise(fixture, streams):
    with pytest.raises(ValueError, match="image 1: progressive"):
        engine.decode_jpeg([streams["420_q75"], fixture["reject_progressive"].tobytes()])
    with pytest.raises(ValueError, match="image 0: CMYK"):
        engine.decode_jpeg([fixture["reject_cmyk"].tobytes()])


# ---- the model ---------------------------------------------------------------------------------------------------------
def _spread_head(sd, std=0.05, prior=0.02):
    g = torch.Generator().manual_seed(123)
    sd = dict(sd)
    sd["cls_head.8.weight"] = torch.randn(sd["cls_head.8.weight"].shape, generator=g) * std
    sd["cls_head.8.bias"] = torch.full_like(sd["cls_head.8.bias"], -float(np.log((1 - prior) / prior)))
    sd["box_head.8.weight"] = torch.randn(sd["box_head.8.weight"].shape, generator=g) * 0.02
    return sd


def _model(backbone, images, resize, max_size, classes=6, rotated=False, seed=14, keep=300):
    """A model whose score threshold leaves about `keep` candidates on the batch of images."""
    sd = _spread_head(make_state_dict(backbone, classes, 27 if rotated else 9, rotated, seed))
    m = Model(backbone, classes=classes, rotated_bbox=rotated).load_state_dict(sd).cuda()
    xp, hs, ws, _ = engine.preprocess_resize_u8(images, resize, max_size)
    heads = m._heads(m._features(m._stem(padded=(xp, hs, ws))))[0]
    scores = torch.cat([c.flatten() for c in heads])
    m.threshold = float(scores.topk(keep).values[-1])
    return m


def _assert_same(a, b):
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def _decoded(streams, names):
    datas = [streams[n] for n in names]
    return datas, [torch.from_numpy(jpeg_oracle.decode(d)) for d in datas]


@pytest.mark.parametrize("backbone,rotated,names,resize,max_size", [
    ("ResNet18FPN", False, ["420_q75", "gray_q100", "422_optimize"], 256, 400),
    ("ResNet18FPN", True, ["444_q75", "420_restart3"], 256, 400),
    ("ResNet50FPN", False, ["420_640x480", "444_480x640", "rand15_gray_190x269"], 800, 1333)])
def test_forward_jpeg_equals_forward_images(streams, backbone, rotated, names, resize, max_size):
    datas, imgs = _decoded(streams, names)
    m = _model(backbone, imgs, resize, max_size, rotated=rotated)
    for fused in (True, False):
        m.fused_candidates = fused
        want, wr = m.forward_images(imgs, resize, max_size)
        want = [t.clone() for t in want]
        assert (want[0] > 0).sum() > 5
        got, r, status = m.forward_jpeg(datas, resize, max_size)
        _assert_same(got, want)
        assert torch.equal(r, wr) and status.cpu().tolist() == [0] * len(datas)


@pytest.mark.parametrize("scope", ["heads", "network"])
def test_forward_jpeg_int8(streams, scope):
    datas, imgs = _decoded(streams, ["420_q75", "422_q75"])
    m = _model("ResNet18FPN", imgs, 256, 400)
    xp, hs, ws, _ = engine.preprocess_resize_u8(imgs, 256, 400)
    x = torch.from_numpy(np.stack([_unpad(xp[i].cpu(), hs, ws) for i in range(len(imgs))]))
    m.set_precision("int8", m.calibrate([x], scope=scope), scope=scope)
    want = [t.clone() for t in m.forward_images(imgs, 256, 400)[0]]
    assert (want[0] > 0).sum() > 5
    got, _, _ = m.forward_jpeg(datas, 256, 400)
    _assert_same(got, want)


def _unpad(buf, hs, ws):
    """The float32 [3, hs, ws] network input inside one NHWC4 stem buffer."""
    return buf[3:3 + hs, 3:3 + ws, :3].permute(2, 0, 1).float().numpy()


def test_cuda_graph_replay_and_recapture(streams):
    canvas = (384, 512)
    groups = [["420_q75", "gray_q75"], ["gray_8x8", "444_8x8"], ["420_q100", "rand24_420_149x172"]]
    batches = [_decoded(streams, g) for g in groups]
    m = _model("ResNet18FPN", batches[0][1], 256, 400)
    eager = []
    for datas, imgs in batches:
        want = [t.clone() for t in m.forward_images(imgs, 256, 400, canvas)[0]]
        got, _, _ = m.forward_jpeg(datas, 256, 400, canvas)
        _assert_same(got, want)
        eager.append(want)
    assert (eager[0][0] > 0).sum() > 5
    m.enable_cuda_graph()
    key = ("jpeg", 2, 384, 512)
    out, _, st = m.forward_jpeg(batches[0][0], 256, 400, canvas)
    _assert_same(out, eager[0])
    entry = m._graphs[key]
    out, _, st = m.forward_jpeg(batches[1][0], 256, 400, canvas)             # fits: same graph
    _assert_same(out, eager[1])
    assert m._graphs[key] is entry and st.cpu().tolist() == [0, 0]
    out, _, _ = m.forward_jpeg(batches[2][0], 256, 400, canvas)              # larger: grow + capture again
    _assert_same(out, eager[2])
    assert m._graphs[key] is not entry
    entry = m._graphs[key]
    for k in (0, 1, 2, 0):
        _assert_same(m.forward_jpeg(batches[k][0], 256, 400, canvas)[0], eager[k])
    assert m._graphs[key] is entry
    m.enable_cuda_graph(False)


def test_infer_jpeg(streams):
    batches = [_decoded(streams, ["420_q75", "gray_q75"]), _decoded(streams, ["444_q75", "422_q75"])]
    m = _model("ResNet18FPN", batches[0][1], 256, 400)
    scores, boxes, classes, ratios, status = infer.infer_jpeg(m, [b[0] for b in batches], 256, 400)
    want = infer.infer_images(m, [b[1] for b in batches], 256, 400)
    assert torch.equal(scores, want[0]) and torch.equal(boxes, want[1]) and torch.equal(ratios, want[3])
    assert status.tolist() == [0, 0, 0, 0]


def test_cuda_graph_replay_with_more_blocks_than_captured(streams):
    """A replayed batch that fits the grown buffers but has more 8x8 blocks (and restart segments) than the batch the
    graph was captured with: the workspace regions move with the batch, so its coefficients do not overlap its planes."""
    from retinanet_examples_b200 import jpeg
    canvas = (384, 512)
    groups = [["420_q75", "gray_q75"], ["420_q75", "420_q100"], ["420_q10", "420_q10"], ["420_restart3", "420_restart3"]]
    batches = [_decoded(streams, g) for g in groups]
    jb = [jpeg.JpegBatch(b[0]) for b in batches]
    m = _model("ResNet18FPN", batches[0][1], 256, 400)
    eager = [[t.clone() for t in m.forward_images(imgs, 256, 400, canvas)[0]] for _, imgs in batches]
    m.enable_cuda_graph()
    key = ("jpeg", 2, 384, 512)
    m.forward_jpeg(batches[0][0], 256, 400, canvas)
    _assert_same(m.forward_jpeg(batches[1][0], 256, 400, canvas)[0], eager[1])     # grows: captured with batch 1
    entry = m._graphs[key]
    cap = entry["capacity"]
    for k in (2, 3):
        need = (jb[k].nbytes, jb[k].workspace_bytes(), 3 * jb[k].pixels)
        assert all(a <= b for a, b in zip(need, cap))
    assert jb[2].blocks > jb[1].blocks and jb[3].segments > jb[1].segments
    for k in (2, 3, 1, 2):
        out, _, st = m.forward_jpeg(batches[k][0], 256, 400, canvas)
        assert m._graphs[key] is entry and st.cpu().tolist() == [0, 0]
        _assert_same(out, eager[k])
    m.enable_cuda_graph(False)


def test_trailer_after_eoi(fixture, streams):
    """Bytes after EOI (here restart and EOI markers, then a second JPEG) are not decoded and raise no status."""
    rs = streams["420_restart3"]
    imgs, status = engine.decode_jpeg([rs + b"\xff\xd0\x00\xff\xd3\xff\xd9" + rs, streams["gray_q75"]])
    assert status.cpu().tolist() == [0, 0]
    _check(fixture, "420_restart3", imgs[0])
    _check(fixture, "gray_q75", imgs[1])
