"""GPU tests of the in-kernel detection gather (odtk_nms_gather / odtk_gather_wait, retinanet-examples_b200/peer.py):
`infer.infer` over image-wise shards with the detections of all ranks delivered to every
rank -- on the real Model, on NCCL ranks, compared with a single-GPU run of the same images.
The 2-rank tests need 2 GPUs; the single-GPU ones exercise the same kernel path with world size 1."""
import ctypes
import os
import socket
import sys

import numpy as np
import pytest
import torch

from retinanet_examples_b200 import _C, _lib, infer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _nms_case(rng, batch, n):
    s = rng.uniform(0.01, 1.0, size=(batch, n)).astype(np.float32)
    s[rng.uniform(size=s.shape) < 0.3] = 0.0
    xy = rng.uniform(0, 300, size=(batch, n, 2))
    wh = rng.uniform(5, 80, size=(batch, n, 2))
    b = np.concatenate([xy, xy + wh], 2).astype(np.float32)
    c = rng.integers(0, 5, size=(batch, n)).astype(np.float32)
    return [torch.from_numpy(a).to(DEV) for a in (s, b, c)]


def test_nms_packed_rows_equal_the_three_outputs():
    rng = np.random.default_rng(2)
    s, b, c = _nms_case(rng, 3, 700)
    packed = torch.full((3, 100, 6), -7.0, device=DEV)
    os_, ob, oc = _C.nms(s, b, c, 0.5, 100, packed=packed)
    ps, pb, pc = infer.split_packed(packed)
    assert torch.equal(ps, os_) and torch.equal(pb, ob) and torch.equal(pc, oc)
    assert float(os_.max()) > 0


def test_gather_single_rank_self_delivery_and_epochs():
    """World size 1 through the raw C ABI: the kernel stores its rows into 'peer 0' (itself), counts the arrivals, the wait
    kernel advances the epoch; two steps land in the two parity halves."""
    rng = np.random.default_rng(3)
    B, D, n = 2, 50, 400
    g = _lib.Gather()
    buf = torch.zeros(2 * B * D * 6, device=DEV)
    flags = torch.zeros(1, dtype=torch.int32, device=DEV)
    epoch = torch.zeros(1, dtype=torch.int32, device=DEV)
    g.packed[0], g.flags[0], g.epoch, g.num_peers, g.rank = buf.data_ptr(), flags.data_ptr(), epoch.data_ptr(), 1, 0
    L = _lib.lib()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    ws = torch.empty(256, dtype=torch.uint8, device=DEV)
    outs = []
    for step in range(3):
        s, b, c = _nms_case(rng, B, n)
        inputs = _lib.ptr_array([s.data_ptr(), b.data_ptr(), c.data_ptr()])
        _lib.check(L.odtk_nms_gather(B, inputs, None, n, D, 0.5, 4, 0, None, None, ctypes.byref(g), ctypes.c_void_p(ws.data_ptr()), 256, st), "nms_gather")
        _lib.check(L.odtk_gather_wait(ctypes.byref(g), B, st), "gather_wait")
        torch.cuda.synchronize()
        ref = _C.nms(s, b, c, 0.5, D)
        half = buf[(step & 1) * B * D * 6:((step & 1) + 1) * B * D * 6].view(B, D, 6)
        assert torch.equal(half[..., 0], ref[0]) and torch.equal(half[..., 1:5], ref[1]) and torch.equal(half[..., 5], ref[2])
        outs.append(half.clone())
        assert int(epoch.item()) == step + 1 and int(flags.item()) == (step + 1) * B


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
        sys.path.insert(0, ROOT)
        import torch.distributed as dist
        from retinanet_examples_b200 import peer
        from retinanet_examples_b200.model import Model, make_state_dict
        torch.cuda.set_device(rank)
        dev = torch.device("cuda", rank)
        dist.init_process_group("nccl", device_id=dev)
        classes, per = 4, 2
        sd = make_state_dict("ResNet18FPN", classes, 9, False, seed=1)
        gsd = torch.Generator().manual_seed(5)
        sd["cls_head.8.weight"] = torch.randn(sd["cls_head.8.weight"].shape, generator=gsd) * 0.05
        sd["cls_head.8.bias"] = torch.full_like(sd["cls_head.8.bias"], -3.0)
        model = Model("ResNet18FPN", classes=classes).load_state_dict(sd).cuda(rank)
        images = torch.randn((world * per, 3, 128, 256), generator=torch.Generator().manual_seed(9))
        shard = images[list(infer.shard_batch(world * per, world, rank))].to(dev)
        # (1) NCCL all-gather of the reference-style loop, real Model (F1)
        s, b, c = infer.infer(model, [shard], world=world)
        # (2) in-kernel peer gather, eager then CUDA-graph replayed (the collective is inside the graph)
        pg = peer.PeerGather(per, detections=model.detections, nbox=4)
        model.attach_gather(pg)
        model(shard)
        torch.cuda.synchronize()
        eager = pg.gathered().clone()
        model.enable_cuda_graph()
        for _ in range(3):
            model(shard)
        torch.cuda.synchronize()
        graphed = pg.gathered().clone()
        dist.barrier()
        full = None
        if rank == 0:      # single-GPU run of ALL images for comparison
            ref_model = Model("ResNet18FPN", classes=classes).load_state_dict(sd).cuda(rank)
            full = [t.cpu() for t in ref_model(images.to(dev))]
        q.put((rank, [t.cpu() for t in (s, b, c)], eager.cpu(), graphed.cpu(), full))
        dist.barrier()
        dist.destroy_process_group()
    except Exception as e:   # surface the failure in the parent
        import traceback
        q.put((rank, "error", traceback.format_exc(), None, None))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.timeout(600)
def test_two_rank_gather_matches_single_gpu_run():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = {}
    for _ in range(2):
        item = q.get(timeout=500)
        assert item[1] != "error", item[2]
        res[item[0]] = item[1:]
    for p in procs:
        p.join(60)
    full = res[0][3]
    assert full is not None and float(full[0].max()) > 0          # the case produces detections
    for r in (0, 1):
        (s, b, c), eager, graphed, _ = res[r]
        # NCCL route: rank-major concatenation == the single-GPU result on all images
        assert torch.equal(s, full[0]) and torch.equal(b, full[1]) and torch.equal(c, full[2])
        # peer route, eager and inside the CUDA graph: same rows on every rank
        for got in (eager, graphed):
            assert torch.equal(got[..., 0], full[0]) and torch.equal(got[..., 1:5], full[1]) and torch.equal(got[..., 5], full[2])
