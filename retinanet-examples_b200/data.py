"""Training and evaluation batches on the GPU, a drop-in for odtk/data.py's DataIterator / RotatedDataIterator.

Per batch: the host reads the files, parses the JPEG headers and makes the reference's random draws; the GPU decodes
the baseline JPEGs (odtk_decode_jpeg), resizes every image with Pillow's uint8 BILINEAR (odtk_resize_u8_packed) and
applies rotation, flip, brightness, contrast, hue, saturation, normalisation and the collate padding in one pass
(odtk_augment_u8).  Files the GPU decoder does not take (progressive, CMYK, PNG, ...) are decoded by Pillow on the host
and join the same packed buffer.  For the same draws, `data` is torch.equal to the reference dataset's collated batch
(as a channels_last view of fp32 [B, H, W, 3]) and `target` is torch.equal to its target."""
import ctypes
import json
import math
import os
import random
from collections import OrderedDict

import numpy as np
import torch

from . import _lib, engine, jpeg

MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]   # odtk/data.py:25-26
_ALIGN = 256


class Coco:
    """The part of pycocotools.coco.COCO the datasets use, over the annotation JSON: `imgs` in the file's image order,
    each image's annotations in file order, `cat_ids` in the file's category order."""

    def __init__(self, annotations):
        with open(annotations) as f:
            self.dataset = json.load(f)
        self.imgs = OrderedDict((im["id"], im) for im in self.dataset.get("images", []))
        self.img_to_anns = {}
        for ann in self.dataset.get("annotations", []):
            self.img_to_anns.setdefault(ann["image_id"], []).append(ann)
        self.cat_ids = [c["id"] for c in self.dataset.get("categories", [])]


def _align(x):
    return -(-x // _ALIGN) * _ALIGN


class DataIterator:
    """odtk.data.DataIterator's constructor arguments and iteration: yields (data, target) when training, else
    (data, ids, ratio), all on the current CUDA device.  rng: the random source of the draws (default the `random`
    module, as the reference)."""
    rotated = False

    def __init__(self, path, resize, max_size, batch_size, stride, world, annotations, training=False,
                 rotate_augment=False, augment_brightness=0.0, augment_contrast=0.0, augment_hue=0.0,
                 augment_saturation=0.0, absolute_angle=False, rng=None):
        self.path = os.path.expanduser(path)
        self.resize, self.max_size, self.stride = resize, max_size, stride
        self.training, self.rotate_augment, self.absolute_angle = training, rotate_augment, absolute_angle
        self.augment = (augment_brightness, augment_contrast, augment_hue, augment_saturation)
        self.rng = rng if rng is not None else random
        self.coco = Coco(annotations)
        self.ids = list(self.coco.imgs.keys())
        self.categories_inv = {k: i for i, k in enumerate(self.coco.cat_ids)} if "categories" in self.coco.dataset else None
        self.batch_size = batch_size // world
        # the reference shards the dataset's images (DistributedSampler over len(ids)), then batches each rank's share
        self.sampler = torch.utils.data.distributed.DistributedSampler(range(len(self.ids))) if world > 1 else None
        self._pending = None     # (event, pinned status, file names) of the previous batch's GPU decode
        self._staging = _Staging()

    def __repr__(self):
        return "\n".join(["    loader: odtk_b200 (GPU decode + augment)",
                          "    resize: {}, max: {}".format(self.resize, self.max_size)])

    def __len__(self):
        n = len(self.sampler) if self.sampler is not None else len(self.ids)
        return -(-n // self.batch_size)

    # ---- the per-image host work of __getitem__ --------------------------------------------------------------------
    def _target(self, id):
        ncol = 5 if self.rotated else 4
        boxes, cats = [], []
        for ann in self.coco.img_to_anns.get(id, []):
            if ann["bbox"][2] < 1 and ann["bbox"][3] < 1:
                continue
            box = list(ann["bbox"])
            if self.rotated:
                if len(box) == 4:
                    box.append(0.0)
                if len(box) != 5:
                    raise ValueError("Bounding box for id %i does not contain five entries." % id)
            boxes.append(box)
            cat = ann["category_id"]
            cats.append(self.categories_inv[cat] if self.categories_inv is not None else cat)
        if boxes:
            return torch.tensor(boxes, dtype=torch.float32), torch.tensor(cats, dtype=torch.float32).unsqueeze(1)
        return torch.ones([1, ncol]), torch.ones([1, 1]) * -1

    def _draw(self, h, w):
        """The reference's draws for one image of h x w, in its order.  Returns (ratio, dst_h, dst_w, angle, flip,
        factors): factors (brightness, contrast, hue, saturation), None when disabled."""
        resize = self.resize
        if isinstance(resize, list):
            resize = self.rng.randint(self.resize[0], self.resize[-1])
        ratio, dh, dw = engine.resize_ratio(h, w, resize, self.max_size)
        if not self.training:
            return ratio, dh, dw, 0, 0, (None,) * 4
        angle = self.rng.randint(0, 3) * 90
        flip = self.rng.randint(0, 1)
        b, c, hu, s = self.augment
        fb = fc = fh = fs = None
        if b:
            fb = max(0, self.rng.normalvariate(1, b))
        if c:
            fc = max(0, self.rng.normalvariate(1, c))
        if hu:
            fh = min(0.5, max(-0.5, self.rng.normalvariate(0, hu)))
        if s:
            fs = max(0, self.rng.normalvariate(1, s))
        return ratio, dh, dw, angle, flip, (fb, fc, fh, fs)

    def _transform(self, boxes, ratio, angle, flip, dh, dw):
        """The target transforms of CocoDataset.__getitem__ (float32 torch, the reference's operation order)."""
        boxes *= ratio
        W, H = dw, dh
        if self.rotate_augment and angle != 0:
            x, y, w, h = boxes[:, 0].clone(), boxes[:, 1].clone(), boxes[:, 2].clone(), boxes[:, 3].clone()
            if angle == 90:
                boxes[:, 0] = y - H / 2 + W / 2
                boxes[:, 1] = W / 2 + H / 2 - x - w
                boxes[:, 2], boxes[:, 3] = h, w
            elif angle == 180:
                boxes[:, 0] = W - x - w
                boxes[:, 1] = H - y - h
            else:
                boxes[:, 0] = W / 2 + H / 2 - y - h
                boxes[:, 1] = x - W / 2 + H / 2
                boxes[:, 2], boxes[:, 3] = h, w
        if flip:
            boxes[:, 0] = W - boxes[:, 0] - boxes[:, 2]
        return boxes

    def _sample(self, index):
        """(id, file name, file bytes) of dataset index `index`."""
        id = self.ids[index]
        name = self.coco.imgs[id]["file_name"]
        with open("{}/{}".format(self.path, name), "rb") as f:
            data = f.read()
        return id, name, data

    # ---- iteration -------------------------------------------------------------------------------------------------
    def _indices(self):
        return list(self.sampler) if self.sampler is not None else list(range(len(self.ids)))

    def _check_pending(self):
        if self._pending is None:
            return
        event, status, names = self._pending
        self._pending = None
        event.synchronize()
        for s, name in zip(status.tolist(), names):
            if s:
                raise RuntimeError("JPEG decode of %s failed on the GPU (status %d)" % (name, s))

    def __iter__(self):
        idx = self._indices()
        for i in range(0, len(idx), self.batch_size):
            out = self.batch([idx[j] for j in range(i, min(i + self.batch_size, len(idx)))])
            yield out
        self._check_pending()

    def batch(self, indices):
        """One collated batch of the dataset indices, with fresh draws: what the iterator yields."""
        dev = torch.device("cuda", torch.cuda.current_device())
        samples = [self._sample(i) for i in indices]
        # headers: GPU decode where odtk_decode_jpeg takes the stream, Pillow otherwise
        gpu, infos, host, shapes = [], [], {}, []
        for k, (_, name, data) in enumerate(samples):
            try:
                info = jpeg.parse(data)
                gpu.append(k)
                infos.append(info)
                shapes.append((info.height, info.width))
            except ValueError:
                host[k] = _pillow_decode(data, name)
                shapes.append(host[k].shape[:2])
        n = len(samples)
        raw_off, off = [], 0
        for h, w in shapes:
            raw_off.append(off)
            off += h * w * 3
        raw = torch.empty(max(off, 1), dtype=torch.uint8, device=dev)
        # draws and targets, per image in the reference's order
        rtab = (_lib.ResizeImage * n)()
        atab = (_lib.AugmentImage * n)()
        targets, ratios, canvas_h, canvas_w, rsz_off = [], [], 0, 0, 0
        out_off = torch.empty(n, dtype=torch.int64)
        for k, ((id, name, _), (h, w)) in enumerate(zip(samples, shapes)):
            ratio, dh, dw, angle, flip, (fb, fc, fh, fs) = self._draw(h, w)
            if dh <= 0 or dw <= 0:
                raise ValueError("%s (%dx%d) resizes to %dx%d" % (name, h, w, dh, dw))
            r = rtab[k]
            r.offset, r.src_h, r.src_w, r.dst_h, r.dst_w = raw_off[k], h, w, dh, dw
            out_off[k] = rsz_off
            a = atab[k]
            a.offset, a.h, a.w = rsz_off, dh, dw
            rsz_off += dh * dw * 3
            a.rot = angle // 90 if self.rotate_augment else 0
            a.expand = int(self.rotated)
            a.flip = flip
            flags = 0
            for bit, f, field in ((_lib.AUGMENT_BRIGHTNESS, fb, "brightness"), (_lib.AUGMENT_CONTRAST, fc, "contrast"),
                                  (_lib.AUGMENT_SATURATION, fs, "saturation")):
                if f is not None:
                    flags |= bit
                    setattr(a, field, f)
            if fh is not None:
                flags |= _lib.AUGMENT_HUE
                a.hue_shift = int(np.int32(fh * 255).astype(np.uint8))
            a.flags = flags
            oh, ow = (dw, dh) if (a.rot & 1) and a.expand else (dh, dw)
            canvas_h = max(canvas_h, -(-oh // self.stride) * self.stride)
            canvas_w = max(canvas_w, -(-ow // self.stride) * self.stride)
            ratios.append(ratio)
            if self.training:
                boxes, cats = self._target(id)
                targets.append(torch.cat([self._transform(boxes, ratio, angle, flip, dh, dw), cats], dim=1))
        if self.training:
            max_det = max(t.size(0) for t in targets)
            ncol = targets[0].size(1)
            side = torch.stack([torch.cat([t, torch.ones([max_det - t.size(0), ncol]) * -1]) for t in targets], 0)
        else:
            side = torch.tensor([s[0] for s in samples], dtype=torch.int32)
        # everything the batch uploads goes in one H2D copy from one of two pinned staging buffers:
        # [resize table | output offsets | augment table | target or ids | JPEG staging | host-decoded pixels]
        jb = jpeg.JpegBatch([samples[k][2] for k in gpu], infos) if gpu else None
        t0 = _align(ctypes.sizeof(rtab))
        t1 = t0 + _align(8 * n)
        t2 = t1 + _align(ctypes.sizeof(atab))
        t3 = t2 + _align(side.numel() * 4)
        t4 = t3 + (_align(jb.nbytes) if jb is not None else 0)
        hoff, o = {}, t4
        for k, im in host.items():
            hoff[k] = o
            o += im.size
        stage = self._staging.take(o)
        stage[:ctypes.sizeof(rtab)].copy_(torch.frombuffer(bytearray(bytes(rtab)), dtype=torch.uint8))
        stage[t0:t0 + 8 * n].copy_(out_off.view(torch.uint8))
        stage[t1:t1 + ctypes.sizeof(atab)].copy_(torch.frombuffer(bytearray(bytes(atab)), dtype=torch.uint8))
        stage[t2:t2 + side.numel() * 4].copy_(side.reshape(-1).view(torch.uint8))
        outs = None
        if jb is not None:
            outs = (_lib.ResizeImage * len(gpu))()
            for t, k in zip(outs, gpu):
                h, w = shapes[k]
                t.offset, t.src_h, t.src_w, t.dst_h, t.dst_w = raw_off[k], h, w, h, w
            jb.fill(outs, stage[t3:t3 + jb.nbytes].numpy())
        for k, im in host.items():
            stage[hoff[k]:hoff[k] + im.size].copy_(torch.from_numpy(im.reshape(-1)))
        staged = stage.to(dev, non_blocking=True)
        # pixels: the GPU-decoded streams, then the host-decoded images, into one packed buffer
        self._check_pending()
        status_h = None
        if jb is not None:
            workspace = torch.empty(jb.workspace_bytes(), dtype=torch.uint8, device=dev)
            status = torch.empty(jb.n, dtype=torch.int32, device=dev)
            engine.jpeg_launch(jb, staged[t3:t3 + jb.nbytes], outs, workspace, raw, status)
            status_h = self._staging.status(jb.n)
            status_h.copy_(status, non_blocking=True)
        for k, im in host.items():
            raw[raw_off[k]:raw_off[k] + im.size].copy_(staged[hoff[k]:hoff[k] + im.size])
        event = self._staging.release()
        if jb is not None:
            self._pending = (event, status_h, [samples[k][1] for k in gpu])
        resized = torch.empty(max(rsz_off, 1), dtype=torch.uint8, device=dev)
        engine.resize_u8_launch(raw, raw.numel(), rtab, staged, out_off, staged[t0:], resized)
        data = engine.augment_launch(resized, atab, staged[t1:], (canvas_h, canvas_w))
        side_dev = staged[t2:t2 + side.numel() * 4].view(side.dtype).view(side.shape)
        if self.training:
            return data, side_dev
        return data, side_dev, torch.FloatTensor(ratios).view(-1, 1, 1).to(dev, non_blocking=True)


class _Staging:
    """Two pinned host buffers used in turn for a batch's uploads (and the decode status it reads back).  A buffer is
    written again only after the event recorded behind the copies out of (and into) it has completed, i.e. two batches
    later; that wait covers the copies only, never a training step enqueued after them."""

    def __init__(self):
        self.bufs, self.stats, self.events, self.i = [None, None], [None, None], [None, None], 0

    def take(self, nbytes):
        self.i ^= 1
        if self.events[self.i] is not None:
            self.events[self.i].synchronize()
        b = self.bufs[self.i]
        if b is None or b.numel() < nbytes:
            b = self.bufs[self.i] = torch.empty(max(nbytes, 2 * (b.numel() if b is not None else 0)), dtype=torch.uint8,
                                                pin_memory=True)
        return b[:nbytes]

    def status(self, n):
        s = self.stats[self.i]
        if s is None or s.numel() < n:
            s = self.stats[self.i] = torch.empty(max(n, 64), dtype=torch.int32, pin_memory=True)
        return s[:n]

    def release(self):
        e = torch.cuda.Event()
        e.record()
        self.events[self.i] = e
        return e


class RotatedDataIterator(DataIterator):
    """odtk.data.RotatedDataIterator: [x, y, w, h, theta] boxes, rotation with expand, absolute_angle."""
    rotated = True

    def _transform(self, boxes, ratio, angle, flip, dh, dw):
        boxes[:, :4] *= ratio
        W, H = dw, dh
        if self.rotate_augment and angle != 0:
            x, y, w, h, t = (boxes[:, k].clone() for k in range(5))
            if angle == 90:
                boxes[:, 0] = y
                boxes[:, 1] = W - x - w
                if not self.absolute_angle:
                    boxes[:, 2], boxes[:, 3] = h, w
            elif angle == 180:
                boxes[:, 0] = W - x - w
                boxes[:, 1] = H - y - h
            else:
                boxes[:, 0] = H - y - h
                boxes[:, 1] = x
                if not self.absolute_angle:
                    boxes[:, 2], boxes[:, 3] = h, w
            if self.absolute_angle:
                t += math.radians(angle)
                t = torch.remainder(torch.abs(t), math.pi) * torch.sign(t)
            boxes[:, 4] = t
            if angle != 180:
                W = dh
        if flip:
            boxes[:, 0] = W - boxes[:, 0] - boxes[:, 2]
            boxes[:, 4] = -boxes[:, 4]
        return boxes


def _pillow_decode(data, name):
    """Image.open(f).convert("RGB") as uint8 [h, w, 3], for the files the GPU decoder does not take."""
    try:
        import io
        from PIL import Image
    except ImportError:
        raise RuntimeError("%s is not a baseline JPEG and Pillow is not installed to decode it" % name) from None
    return np.array(Image.open(io.BytesIO(data)).convert("RGB"), dtype=np.uint8)
