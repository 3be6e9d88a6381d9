"""Numpy restatement of the baseline JPEG decode that `Image.open(f).convert("RGB")` performs with Pillow's libjpeg(-turbo)
defaults, the decode of the reference's data loader (odtk/data.py:50), written from ITU-T T.81 and libjpeg's documented
arithmetic:

- Huffman decoding of each restart segment (T.81 F.2.2), the DC predictor reset to 0 at each segment, de-zig-zag;
- dequantisation and the JDCT_ISLOW integer IDCT: 13-bit fixed-point constants, 2 extra bits between the column and the
  row pass, rounding right shifts, and the range limit that wraps the result to 10 bits before clamping to [0, 255];
- "fancy" upsampling: h2v1 is the triangle filter 3/4 * nearer + 1/4 * further sample with biases 1 (even output) and
  2 (odd output) before >> 2; h2v2 is the same filter vertically into 16x column sums, then horizontally with biases 8
  and 7 before >> 4; samples past an edge replicate the last one.  A chroma plane at most 2 samples wide is replicated
  instead (libjpeg takes its plain upsampler there);
- YCbCr -> RGB with 16-bit fixed-point tables: R = Y + round(1.402 (Cr - 128)), B = Y + round(1.772 (Cb - 128)),
  G = Y + (-0.71414 (Cr - 128) - 0.34414 (Cb - 128) + 1/2) >> 16 (constants rounded to 1/65536), clamped to [0, 255].

Grayscale is replicated to three channels, as convert("RGB") does.  Huffman decoding is a Python loop over symbols; the
rest is vectorised.  tests/test_jpeg_host.py pins this to Pillow's digests in tests/golden/jpeg_pil.npz."""
import hashlib
import re

import numpy as np

from retinanet_examples_b200 import jpeg

CONST_BITS, PASS1_BITS = 13, 2
F = {k: v for k, v in (("0_298631336", 2446), ("0_390180644", 3196), ("0_541196100", 4433), ("0_765366865", 6270),
                        ("0_899976223", 7373), ("1_175875602", 9633), ("1_501321110", 12299), ("1_847759065", 15137),
                        ("1_961570560", 16069), ("2_053119869", 16819), ("2_562915447", 20995), ("3_072711026", 25172))}


class DecodeError(ValueError):
    pass


def _lut16(bits, vals):
    """(length, symbol) of the code at the head of every 16-bit window; length 0: no code."""
    ln = np.zeros(65536, np.int64)
    sym = np.zeros(65536, np.int64)
    code, k = 0, 0
    for l in range(1, 17):
        for _ in range(int(bits[l - 1])):
            lo = code << (16 - l)
            ln[lo:lo + (1 << (16 - l))] = l
            sym[lo:lo + (1 << (16 - l))] = vals[k]
            code += 1
            k += 1
        code <<= 1
    return ln, sym


def _segments(scan, nseg):
    segs = re.split(rb"\xff[\xd0-\xd7]", scan)
    if len(segs) < nseg:
        raise DecodeError("%d restart segments, %d expected" % (len(segs), nseg))
    return [s.replace(b"\xff\x00", b"\xff") for s in segs[:nseg]]


def _windows(seg):
    """16-bit big-endian window at every bit position and the number of real bits.  Zeros follow the end for more than
    one block's worth of bits (64 codes + values of at most 32 bits): running out is detected after each block."""
    bits = np.unpackbits(np.frombuffer(seg, np.uint8)).astype(np.int64)
    L = bits.size
    b = np.concatenate([bits, np.zeros(4096 + 16, np.int64)])
    w = np.zeros(L + 4096, np.int64)
    for i in range(16):
        w += b[i:i + L + 4096] << (15 - i)
    return w.tolist(), L


def _extend(v, s):
    return v - (1 << s) + 1 if v < (1 << (s - 1)) else v


def entropy_decode(info, scan):
    """Coefficient blocks of each component: list of int64 [bh, bw, 64] (row-major within the block)."""
    planes = [np.zeros((bh, bw, 64), np.int64) for bw, bh in info.comp_blocks()]
    luts = [(_lut16(*info.huff[(0, td)]), _lut16(*info.huff[(1, ta)])) for _, td, ta in info.comps]
    zz = jpeg.ZIGZAG.tolist()
    mx, my = info.mcus
    total = mx * my
    ri = info.restart_interval or total
    layout = [(info.hmax, info.vmax)] + [(1, 1)] * (info.ncomp - 1)
    for k, seg in enumerate(_segments(scan, info.nseg)):
        w, L = _windows(seg)
        pos = 0
        pred = [0] * info.ncomp
        for m in range(k * ri, min((k + 1) * ri, total)):
            ux, uy = m % mx, m // mx
            for c, (h, v) in enumerate(layout):
                (dl, ds), (al, as_) = luts[c]
                for bv in range(v):
                    for bh in range(h):
                        blk = planes[c][uy * v + bv, ux * h + bh]
                        p = w[pos]
                        ln = dl[p]
                        if ln == 0:
                            raise DecodeError("bad DC code")
                        s = ds[p]
                        pos += ln
                        d = 0
                        if s:
                            d = _extend(w[pos] >> (16 - s), s) if s <= 16 else 0
                            pos += s
                        pred[c] += d
                        blk[0] = pred[c]
                        i = 1
                        while i < 64:
                            p = w[pos]
                            ln = al[p]
                            if ln == 0:
                                raise DecodeError("bad AC code")
                            rs = as_[p]
                            pos += ln
                            r, s = rs >> 4, rs & 15
                            if s:
                                i += r
                                if i > 63:
                                    raise DecodeError("coefficient index past 63")
                                blk[zz[i]] = _extend(w[pos] >> (16 - s), s)
                                pos += s
                                i += 1
                            elif r == 15:
                                i += 16
                            else:
                                break
                        if pos > L:
                            raise DecodeError("segment %d ran out of data" % k)
    return planes


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _idct_1d(d, shift):
    """The islow butterfly over 8 arrays (inputs in natural order 0..7); returns 8 outputs descaled by `shift`."""
    z2, z3 = d[2], d[6]
    z1 = (z2 + z3) * F["0_541196100"]
    tmp2 = z1 + z3 * -F["1_847759065"]
    tmp3 = z1 + z2 * F["0_765366865"]
    tmp0 = (d[0] + d[4]) << CONST_BITS
    tmp1 = (d[0] - d[4]) << CONST_BITS
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = d[7], d[5], d[3], d[1]
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * F["1_175875602"]
    t0, t1, t2, t3 = t0 * F["0_298631336"], t1 * F["2_053119869"], t2 * F["3_072711026"], t3 * F["1_501321110"]
    z1, z2 = z1 * -F["0_899976223"], z2 * -F["2_562915447"]
    z3, z4 = z3 * -F["1_961570560"] + z5, z4 * -F["0_390180644"] + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    return [_descale(v, shift) for v in (t10 + t3, t11 + t2, t12 + t1, t13 + t0, t13 - t0, t12 - t1, t11 - t2, t10 - t3)]


def idct_islow(coef, quant):
    """int64 [..., 64] coefficients x quantisation steps -> uint8 [..., 8, 8] samples."""
    x = (coef * quant).reshape(coef.shape[:-1] + (8, 8))
    cols = _idct_1d([x[..., k, :] for k in range(8)], CONST_BITS - PASS1_BITS)      # pass 1: columns
    ws = np.stack(cols, axis=-2)                                                        # [..., row, col]
    rows = _idct_1d([ws[..., :, k] for k in range(8)], CONST_BITS + PASS1_BITS + 3)    # pass 2: rows
    out = np.stack(rows, axis=-1)
    return np.clip(((out + 512) & 1023) - 512 + 128, 0, 255).astype(np.uint8)


def _plane(blocks):
    bh, bw = blocks.shape[:2]
    return blocks.transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)


def _edge(a, axis, step):
    """a shifted by one sample along axis (step -1: the previous sample, +1: the next), edges replicated."""
    n = a.shape[axis]
    idx = np.clip(np.arange(n) + step, 0, n - 1)
    return np.take(a, idx, axis=axis)


def _interleave(even, odd, axis):
    out = np.stack([even, odd], axis=axis + 1)
    shape = list(even.shape)
    shape[axis] *= 2
    return out.reshape(shape)


def upsample(c, h, v, H, W):
    """Chroma plane (already cropped to its ceil(W / h) x ceil(H / v) samples) -> H x W, libjpeg's fancy filters."""
    c = c.astype(np.int64)
    if h == 1 and v == 1:
        out = c
    elif c.shape[1] <= 2:
        out = c.repeat(h, 1).repeat(v, 0)
    elif v == 1:
        out = _interleave((3 * c + _edge(c, 1, -1) + 1) >> 2, (3 * c + _edge(c, 1, 1) + 2) >> 2, 1)
    else:
        t = _interleave(3 * c + _edge(c, 0, -1), 3 * c + _edge(c, 0, 1), 0)
        out = _interleave((3 * t + _edge(t, 1, -1) + 8) >> 4, (3 * t + _edge(t, 1, 1) + 7) >> 4, 1)
    return out[:H, :W]


def ycc_to_rgb(y, cb, cr):
    y, cb, cr = (a.astype(np.int64) for a in (y, cb, cr))
    fix = lambda f: int(f * 65536 + 0.5)
    r = y + ((fix(1.40200) * (cr - 128) + 32768) >> 16)
    g = y + ((-fix(0.71414) * (cr - 128) - fix(0.34414) * (cb - 128) + 32768) >> 16)
    b = y + ((fix(1.77200) * (cb - 128) + 32768) >> 16)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def component_planes(data):
    """uint8 sample planes of each component over whole blocks (what the IDCT kernel writes) and the JpegInfo."""
    info = jpeg.parse(data)
    coefs = entropy_decode(info, bytes(data[info.scan[0]:info.scan[1]]))
    planes = [_plane(idct_islow(co, info.quant[tq])) for co, (tq, _, _) in zip(coefs, info.comps)]
    return planes, info


def decode(data):
    """uint8 [h, w, 3]: np.asarray(Image.open(f).convert("RGB")) of a baseline JPEG.  DecodeError for a corrupt scan."""
    planes, info = component_planes(data)
    H, W = info.height, info.width
    y = planes[0][:H, :W]
    if info.ncomp == 1:
        return np.repeat(y[..., None], 3, -1)
    ch, cw = -(-H // info.vmax), -(-W // info.hmax)
    cb, cr = (upsample(p[:ch, :cw], info.hmax, info.vmax, H, W) for p in planes[1:])
    return ycc_to_rgb(y, cb, cr)


def sha256(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def fixture_streams(g):
    """name -> JPEG bytes of the decodable cases of tests/golden/jpeg_pil.npz."""
    return {str(n): g[str(n) + "_jpeg"].tobytes() for n in g["names"]}
