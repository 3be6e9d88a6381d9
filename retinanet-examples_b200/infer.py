"""Host-side mirror of the hot loop of the reference's odtk/infer.py:71-102 on tensors that are
already in memory (datasets, COCO json/eval, DALI and apex are outside the hot path
section 2): per batch `model(data)`, collect, and -- when several ranks shard the images -- gather the
detections of all ranks.  The reference issues five all_gathers (scores, boxes, classes, ids, ratios)
after the loop (infer.py:98-102); here the three detection tensors travel as ONE packed
[N, D, 2 + nbox] fp32 buffer in ONE collective (latency-bound: 2.4-3.2 KB per image)."""
import torch
import torch.distributed as dist


def pack_detections(scores, boxes, classes):
    """[N, D], [N, D, nbox], [N, D] -> [N, D, 2 + nbox] (score, box..., class)."""
    return torch.cat([scores.unsqueeze(-1), boxes, classes.unsqueeze(-1)], dim=-1).contiguous()


def unpack_detections(packed):
    return packed[..., 0].contiguous(), packed[..., 1:-1].contiguous(), packed[..., -1].contiguous()


def split_packed(packed):
    """[N, D, 2 + nbox] -> (scores [N, D], boxes [N, D, nbox], classes [N, D]) as views (no copies)."""
    return packed[..., 0], packed[..., 1:-1], packed[..., -1]


def gather_detections(scores, boxes, classes, world=None):
    """All ranks receive the detections of every rank, rank-major (== the torch.cat of the
    reference's all_gather lists, infer.py:100-102).  One collective."""
    if world is None:
        world = dist.get_world_size() if dist.is_initialized() else 1
    if world <= 1:
        return scores, boxes, classes
    packed = pack_detections(scores, boxes, classes)
    out = torch.empty((world * packed.shape[0],) + tuple(packed.shape[1:]), dtype=packed.dtype, device=packed.device)
    dist.all_gather_into_tensor(out, packed)   # rank-major concatenation along dim 0
    return unpack_detections(out)


def shard_batch(batch_size, world, rank):
    """Image-wise sharding: rank r owns images [r*B/W, (r+1)*B/W) (reference: main.py:170-171,
    data.py:202-205)."""
    if batch_size % world != 0:
        raise RuntimeError("Batch size should be a multiple of the number of GPUs")
    per = batch_size // world
    return range(rank * per, (rank + 1) * per)


def infer(model, path, detections_file=None, resize=None, max_size=None, batch_size=None, mixed_precision=True,
          is_master=True, world=0, annotations=None, with_apex=False, use_dali=True, is_validation=False,
          verbose=True, rotated_bbox=False):
    """`path` is an iterable of image batches ([B, 3, H, W] tensors on the model's device) instead of
    a dataset directory; the remaining reference arguments are accepted for call-site compatibility.
    Returns (scores [N, D], boxes [N, D, nbox], classes [N, D]) for the images of ALL ranks."""
    results = []
    with torch.no_grad():
        for data in path:
            scores, boxes, classes = model(data, rotated_bbox)
            results.append(pack_detections(scores, boxes, classes))
    packed = torch.cat(results, dim=0)
    return gather_detections(*unpack_detections(packed), world=max(world, 1))


def detections_to_coco(scores, boxes, classes, ratios, image_ids=None, category_ids=None):
    """Output side of `odtk infer` (odtk/infer.py:104-148, axis-aligned branch): keep score > 0, undo the
    resize ratio, convert (x1, y1, x2, y2) to COCO (x, y, w, h) with the +1 width convention.
    scores [N, D], boxes [N, D, 4], classes [N, D]; ratios [N] or scalar.  Returns a list of dicts."""
    scores, boxes, classes = scores.float().cpu(), boxes.float().cpu(), classes.float().cpu()
    ratios = torch.as_tensor(ratios, dtype=torch.float32).reshape(-1).expand(scores.shape[0]) if not torch.is_tensor(ratios) \
        else ratios.float().cpu().reshape(-1).expand(scores.shape[0])
    out = []
    for i in range(scores.shape[0]):
        keep = (scores[i] > 0).nonzero(as_tuple=False).view(-1)
        b = boxes[i][keep] / ratios[i]
        for score, box, cat in zip(scores[i][keep].tolist(), b.tolist(), classes[i][keep].int().tolist()):
            x1, y1, x2, y2 = box
            out.append({"image_id": int(image_ids[i]) if image_ids is not None else i, "score": score,
                        "category_id": category_ids[cat] if category_ids is not None else cat,
                        "bbox": [x1, y1, x2 - x1 + 1, y2 - y1 + 1]})
    return out
