"""Host side of the GPU JPEG decoder (odtk_decode_jpeg, include/odtk_b200.h): a marker parser for baseline sequential
Huffman-coded JPEG (ITU-T T.81, SOF0 / SOF1, 8-bit, grayscale or YCbCr 4:4:4 / 4:2:2 / 4:2:0) and the packer that lays
a batch out in one staging buffer

    [odtk_jpeg_image_t[n] | odtk_resize_image_t[n] | quantisation and Huffman tables | entropy-coded bytes]

which leaves in one pinned host-to-device copy.  The host reads headers only: the end of the scan is found with
bytes.find (the first EOI after SOS) and the scan bytes are copied as one slice each; everything per pixel or per
coefficient (Huffman decoding, restart markers, dequantisation, IDCT, upsampling, colour conversion) runs on the GPU.

Anything else (progressive, arithmetic-coded, lossless or hierarchical, 12-bit, CMYK / YCCK, RGB-coded, other sampling
factors such as 4:4:0, multi-scan) raises ValueError: decode such an image with Pillow and use Model.forward_images."""
import ctypes

import numpy as np
import torch

from . import _lib

# T.81 figure A.6: position k of the zig-zag sequence -> row-major index in the 8x8 block
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7,
                   14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39,
                   46, 53, 60, 61, 54, 47, 55, 62, 63], np.int64)

SAMPLINGS = {(1, 1): "4:4:4", (2, 1): "4:2:2", (2, 2): "4:2:0"}      # luma (h, v) with chroma 1x1
ALIGN = 256
TABLE_ALIGN = 16

_SOF_NAMES = {0xC2: "progressive", 0xC3: "lossless", 0xC5: "hierarchical", 0xC6: "hierarchical progressive",
              0xC7: "hierarchical lossless", 0xC9: "arithmetic-coded", 0xCA: "arithmetic-coded progressive",
              0xCB: "arithmetic-coded lossless", 0xCD: "arithmetic-coded hierarchical",
              0xCE: "arithmetic-coded hierarchical progressive", 0xCF: "arithmetic-coded hierarchical lossless"}


class JpegInfo:
    """What parse() reads from one stream.  height, width; ncomp (1 or 3); hmax, vmax (luma sampling; 1x1 for
    grayscale); comps: per component (quant slot, dc slot, ac slot) in frame order; quant: slot -> int64 [64]
    quantisation table in row-major (natural) order; huff: (class 0 = DC / 1 = AC, slot) -> (bits int64 [16], values
    uint8 [n]); restart_interval (MCUs, 0 = none); scan: (start, end) byte range of the entropy-coded data (restart
    markers included, EOI excluded; the end of the stream when EOI is missing)."""

    def __init__(self):
        self.quant, self.huff, self.restart_interval = {}, {}, 0
        self.adobe_transform = None
        self.jfif = False

    @property
    def mcus(self):
        """(MCU columns, MCU rows)."""
        return -(-self.width // (8 * self.hmax)), -(-self.height // (8 * self.vmax))

    @property
    def nseg(self):
        mx, my = self.mcus
        return -(-(mx * my) // self.restart_interval) if self.restart_interval else 1

    def comp_blocks(self):
        """[(blocks across, blocks down)] of each component's coefficient plane (whole MCUs)."""
        mx, my = self.mcus
        return [(mx * self.hmax, my * self.vmax)] + [(mx, my)] * (self.ncomp - 1)

    @property
    def blocks(self):
        return sum(bw * bh for bw, bh in self.comp_blocks())

    @property
    def sampling(self):
        return "gray" if self.ncomp == 1 else SAMPLINGS[(self.hmax, self.vmax)]


def _u16(data, p):
    return (data[p] << 8) | data[p + 1]


def parse(data):
    """Reads the markers of one JPEG stream (bytes-like) up to its scan.  Returns a JpegInfo; raises ValueError with the
    reason for a stream the GPU decoder does not take or a malformed header."""
    data = bytes(data) if not isinstance(data, (bytes, bytearray)) else data
    n = len(data)
    if n < 4 or data[0] != 0xFF or data[1] != 0xD8:
        raise ValueError("not a JPEG stream (no SOI marker)")
    info, frame, p = JpegInfo(), None, 2
    while True:
        if p >= n:
            raise ValueError("malformed header: stream ends before SOS")
        if data[p] != 0xFF:
            raise ValueError("malformed header: expected a marker at byte %d" % p)
        while p < n and data[p] == 0xFF:          # fill bytes
            p += 1
        if p >= n:
            raise ValueError("malformed header: stream ends before SOS")
        m = data[p]
        p += 1
        if m == 0xD9:
            raise ValueError("malformed header: EOI before SOS")
        if m == 0x01 or 0xD0 <= m <= 0xD7:
            continue                              # TEM / stray RSTn: no length
        if p + 2 > n:
            raise ValueError("malformed header: truncated marker 0x%02X" % m)
        length = _u16(data, p)
        if length < 2 or p + length > n:
            raise ValueError("malformed header: marker 0x%02X has length %d at byte %d of %d" % (m, length, p, n))
        seg, q = data[p + 2:p + length], p + length
        if m in _SOF_NAMES:
            raise ValueError("%s JPEG is not supported" % _SOF_NAMES[m])
        if m == 0xCC:
            raise ValueError("arithmetic-coded JPEG is not supported")
        if m == 0xDC:
            raise ValueError("DNL marker (height defined after the scan) is not supported")
        if m in (0xC0, 0xC1):
            frame = _parse_sof(info, seg)
        elif m == 0xC4:
            _parse_dht(info, seg)
        elif m == 0xDB:
            _parse_dqt(info, seg)
        elif m == 0xDD:
            if len(seg) != 2:
                raise ValueError("malformed header: DRI length %d" % length)
            info.restart_interval = _u16(seg, 0)
        elif m == 0xE0 and seg[:5] == b"JFIF\0" and len(seg) >= 14:
            info.jfif = True
        elif m == 0xEE and seg[:5] == b"Adobe" and len(seg) >= 12:
            info.adobe_transform = seg[11]
        elif m == 0xDA:
            if frame is None:
                raise ValueError("malformed header: SOS before SOF")
            _parse_sos(info, frame, seg)
            # entropy-coded data never holds FF D9 (an FF byte is followed by 00 or a restart marker), so the first EOI
            # ends the scan; bytes after it (a trailer with a second image or a video) are not part of it
            end = data.find(b"\xff\xd9", q)
            info.scan = (q, end if end >= 0 else n)
            return info
        p = q


def _parse_sof(info, seg):
    if len(seg) < 6:
        raise ValueError("malformed header: SOF too short")
    prec, h, w, nf = seg[0], _u16(seg, 1), _u16(seg, 3), seg[5]
    if prec != 8:
        raise ValueError("%d-bit JPEG is not supported" % prec)
    if len(seg) != 6 + 3 * nf:
        raise ValueError("malformed header: SOF length %d for %d components" % (len(seg) + 2, nf))
    if h == 0 or w == 0:
        raise ValueError("image size %dx%d is not supported" % (h, w))
    if nf == 4:
        raise ValueError("CMYK / YCCK JPEG is not supported")
    if nf not in (1, 3):
        raise ValueError("%d-component JPEG is not supported" % nf)
    ids = [seg[6 + 3 * i] for i in range(nf)]
    samp = [(seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15) for i in range(nf)]
    tq = [seg[8 + 3 * i] for i in range(nf)]
    if len(set(ids)) != nf:
        raise ValueError("malformed header: repeated component id")
    if nf == 3:
        if samp[1] != (1, 1) or samp[2] != (1, 1) or samp[0] not in SAMPLINGS:
            raise ValueError("sampling factors %s are not supported (4:4:4, 4:2:2 and 4:2:0 are)" %
                             "/".join("%dx%d" % s for s in samp))
        info.hmax, info.vmax = samp[0]
    else:
        info.hmax = info.vmax = 1                # one component: non-interleaved, one block per MCU
    if any(t > 3 for t in tq):
        raise ValueError("malformed header: quantisation table slot > 3")
    info.height, info.width, info.ncomp = h, w, nf
    return ids, tq


def _parse_dht(info, seg):
    p = 0
    while p < len(seg):
        if p + 17 > len(seg):
            raise ValueError("malformed header: DHT too short")
        tc, th = seg[p] >> 4, seg[p] & 15
        bits = np.frombuffer(seg, np.uint8, 16, p + 1).astype(np.int64)
        total = int(bits.sum())
        if tc > 1 or th > 3 or total > 256 or p + 17 + total > len(seg):
            raise ValueError("malformed header: bad DHT table (class %d, slot %d, %d codes)" % (tc, th, total))
        info.huff[(tc, th)] = (bits, np.frombuffer(seg, np.uint8, total, p + 17).copy())
        p += 17 + total


def _parse_dqt(info, seg):
    p = 0
    while p < len(seg):
        pq, tq = seg[p] >> 4, seg[p] & 15
        size = 128 if pq else 64
        if pq > 1 or tq > 3 or p + 1 + size > len(seg):
            raise ValueError("malformed header: bad DQT table (precision %d, slot %d)" % (pq, tq))
        vals = np.frombuffer(seg, ">u2" if pq else np.uint8, 64, p + 1).astype(np.int64)
        q = np.zeros(64, np.int64)
        q[ZIGZAG] = vals
        info.quant[tq] = q
        p += 1 + size


def _parse_sos(info, frame, seg):
    ids, tq = frame
    # libjpeg's colour space of a 3-component stream: YCbCr under a JFIF marker; else an Adobe marker decides (transform
    # 0 is RGB); else component ids 'R', 'G', 'B' mean RGB; anything else is YCbCr
    if info.ncomp == 3 and not info.jfif:
        if info.adobe_transform == 0:
            raise ValueError("RGB-coded JPEG (Adobe transform 0) is not supported")
        if info.adobe_transform is None and ids == [0x52, 0x47, 0x42]:
            raise ValueError("RGB-coded JPEG (component ids 'R', 'G', 'B') is not supported")
    ns = seg[0] if seg else 0
    if len(seg) != 4 + 2 * ns:
        raise ValueError("malformed header: SOS length %d" % (len(seg) + 2))
    if ns != info.ncomp:
        raise ValueError("multi-scan JPEG (a scan of %d of %d components) is not supported" % (ns, info.ncomp))
    ss, se, ahl = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
    if ss != 0 or se != 63 or ahl != 0:
        raise ValueError("malformed header: scan spectral range %d-%d / approximation 0x%02X in a sequential JPEG"
                         % (ss, se, ahl))
    comps = []
    for i in range(ns):
        cid, t = seg[1 + 2 * i], seg[2 + 2 * i]
        if cid != ids[i]:
            raise ValueError("malformed header: scan components are not in frame order")
        td, ta = t >> 4, t & 15
        if (0, td) not in info.huff or (1, ta) not in info.huff:
            raise ValueError("malformed header: component %d uses an undefined Huffman table" % i)
        if tq[i] not in info.quant:
            raise ValueError("malformed header: component %d uses an undefined quantisation table" % i)
        comps.append((tq[i], td, ta))
    info.comps = comps


# ---- device tables ------------------------------------------------------------------------------------------------------
def huff_table(bits, vals):
    """odtk_jpeg_huff_t of one table (T.81 annex C canonical codes): an 8-bit lookahead table for codes up to 8 bits,
    libjpeg-style maxcode / valoff for the longer ones.  ValueError when the lengths overflow the code space."""
    t = _lib.JpegHuff()
    look = np.zeros(256, np.uint16)
    maxcode = np.full(18, -1, np.int64)
    valoff = np.zeros(18, np.int64)
    code, k = 0, 0
    for ln in range(1, 17):
        cnt = int(bits[ln - 1])
        if cnt:
            if code + cnt > (1 << ln):
                raise ValueError("malformed header: Huffman code lengths overflow the code space")
            valoff[ln] = k - code
            if ln <= 8:
                for j in range(cnt):
                    lo = (code + j) << (8 - ln)
                    look[lo:lo + (1 << (8 - ln))] = (ln << 8) | int(vals[k + j])
            code += cnt
            k += cnt
            maxcode[ln] = code - 1
        code <<= 1
    maxcode[17] = 0x7FFFFFFF
    ctypes.memmove(t.look, look.ctypes.data, 512)
    t.maxcode[:] = maxcode.tolist()
    t.valoff[:] = valoff.tolist()
    ctypes.memmove(t.val, bytes(vals.tobytes()).ljust(256, b"\0"), 256)
    return bytes(t)


_HUFF_CACHE = {}


def _huff_bytes(bits, vals):
    key = bits.tobytes() + vals.tobytes()
    b = _HUFF_CACHE.get(key)
    if b is None:
        if len(_HUFF_CACHE) > 4096:
            _HUFF_CACHE.clear()
        b = _HUFF_CACHE[key] = huff_table(bits, vals)
    return b


def _align(x, a):
    return -(-x // a) * a


class JpegBatch:
    """A batch of parsed streams packed for odtk_decode_jpeg.  `infos` (JpegInfo per image), `shapes` [(h, w)],
    `images` (odtk_jpeg_image_t[n], offsets from the start of the staging buffer), `nbytes` (staging bytes), `segments`
    and `blocks` (totals), `resize_off` (byte offset of the odtk_resize_image_t table in the staging buffer).
    ValueError names the image and the reason."""

    def __init__(self, datas, infos=None):
        if len(datas) == 0:
            raise ValueError("no images")
        self.datas = [d if isinstance(d, (bytes, bytearray)) else bytes(d) for d in datas]
        if infos is not None:             # headers the caller already parsed with parse()
            self.infos = list(infos)
        else:
            self.infos = []
            for i, d in enumerate(self.datas):
                try:
                    self.infos.append(parse(d))
                except ValueError as e:
                    raise ValueError("image %d: %s" % (i, e)) from None
        n = self.n = len(self.datas)
        self.shapes = [(f.height, f.width) for f in self.infos]
        self.resize_off = _align(n * ctypes.sizeof(_lib.JpegImage), ALIGN)
        off = self.resize_off + _align(n * ctypes.sizeof(_lib.ResizeImage), ALIGN)
        self.images = (_lib.JpegImage * n)()
        tables, self._tables = {}, []
        seg, blk = 0, 0
        for i, f in enumerate(self.infos):
            t = self.images[i]
            for c, (tq, td, ta) in enumerate(f.comps):
                for kind, key, make in (("quant", ("q", f.quant[tq].tobytes()), lambda: f.quant[tq].astype("<u2").tobytes()),
                                        ("dc", ("h",) + tuple(x.tobytes() for x in f.huff[(0, td)]), lambda: _huff_bytes(*f.huff[(0, td)])),
                                        ("ac", ("h",) + tuple(x.tobytes() for x in f.huff[(1, ta)]), lambda: _huff_bytes(*f.huff[(1, ta)]))):
                    if key not in tables:
                        b = make()
                        tables[key] = off
                        self._tables.append((off, b))
                        off += _align(len(b), TABLE_ALIGN)
                    getattr(t, kind)[c] = tables[key]
            t.height, t.width, t.ncomp, t.hmax, t.vmax = f.height, f.width, f.ncomp, f.hmax, f.vmax
            t.restart_interval, t.nseg, t.seg_base, t.blk_base = f.restart_interval, f.nseg, seg, blk
            seg += f.nseg
            blk += f.blocks
        off = _align(off, ALIGN)
        pix = 0
        for i, f in enumerate(self.infos):
            t = self.images[i]
            t.scan_offset, t.scan_bytes, t.pix_base = off, f.scan[1] - f.scan[0], pix
            off += t.scan_bytes
            pix += f.height * f.width
        self.nbytes, self.segments, self.blocks, self.pixels = off, seg, blk, pix

    def workspace_bytes(self):
        return workspace_bytes(self.segments, self.blocks)

    def stage(self, resize_table, buf):
        """Write [descriptors | resize_table | tables | scans] into the device buffer `buf` with one pinned H2D copy on the
        current stream.  `resize_table`: odtk_resize_image_t[n], the output offsets and sizes."""
        assert buf.dtype == torch.uint8 and buf.numel() >= self.nbytes
        pinned = torch.empty(self.nbytes, dtype=torch.uint8, pin_memory=True)
        self.fill(resize_table, pinned.numpy())
        buf[:self.nbytes].copy_(pinned, non_blocking=True)
        return buf

    def fill(self, resize_table, h):
        """The staging bytes, written into the uint8 numpy array h [nbytes]."""
        h[:self.images[0].scan_offset] = 0               # headers, tables and their padding
        d = bytes(self.images)
        h[:len(d)] = np.frombuffer(d, np.uint8)
        r = bytes(resize_table)
        h[self.resize_off:self.resize_off + len(r)] = np.frombuffer(r, np.uint8)
        for off, b in self._tables:
            h[off:off + len(b)] = np.frombuffer(b, np.uint8)
        for t, f, data in zip(self.images, self.infos, self.datas):
            h[t.scan_offset:t.scan_offset + t.scan_bytes] = np.frombuffer(data, np.uint8, t.scan_bytes, f.scan[0])
        return h


def workspace_bytes(segments, blocks):
    """Device workspace of odtk_decode_jpeg: restart segment bounds (8 bytes each), int16 coefficient blocks (128
    bytes each) and uint8 component planes (64 bytes per block)."""
    return _align(segments * 8, ALIGN) + blocks * 128 + blocks * 64
