"""CPU tests of the JPEG decode path: the numpy oracle (tests/jpeg_oracle.py) reproduces Pillow's decode of every stream
in tests/golden/jpeg_pil.npz bit for bit; jpeg.parse reads the header fields and rejects unsupported or malformed
streams with their reason; the staging layout of jpeg.JpegBatch; the argument checks of odtk_decode_jpeg's size query
(no GPU needed)."""
import ctypes
import os
import struct

import numpy as np
import pytest

import jpeg_oracle
from retinanet_examples_b200 import _lib, engine, jpeg


@pytest.fixture(scope="module")
def fixture(golden_dir):
    return np.load(os.path.join(golden_dir, "jpeg_pil.npz"))


@pytest.fixture(scope="module")
def streams(fixture):
    return jpeg_oracle.fixture_streams(fixture)


def test_fixture_covers_the_cases(fixture, streams):
    assert str(fixture["pillow_version"]) == "12.2.0"
    names = list(streams)
    assert len(names) >= 80
    infos = {n: jpeg.parse(d) for n, d in streams.items()}
    assert {f.sampling for f in infos.values()} == {"4:2:0", "4:2:2", "4:4:4", "gray"}
    assert any(f.restart_interval for f in infos.values())
    assert any((f.height, f.width) == (480, 640) for f in infos.values())
    assert any((f.height, f.width) == (1, 1) for f in infos.values())


def test_oracle_matches_pillow_bit_for_bit(fixture, streams):
    for name, data in streams.items():
        out = jpeg_oracle.decode(data)
        assert out.shape == tuple(fixture[name + "_shape"]), name
        assert jpeg_oracle.sha256(out) == str(fixture[name + "_pil_sha256"]), name


def test_oracle_rejects_truncated_stream(fixture):
    with pytest.raises(jpeg_oracle.DecodeError):
        jpeg_oracle.decode(fixture["truncated_jpeg"].tobytes())


def test_parse_fields(streams):
    f = jpeg.parse(streams["420_q75"])
    assert (f.height, f.width, f.ncomp, f.hmax, f.vmax, f.restart_interval) == (61, 90, 3, 2, 2, 0)
    assert f.mcus == (6, 4) and f.nseg == 1 and f.blocks == 6 * 4 * 6
    assert f.comps == [(0, 0, 0), (1, 1, 1), (1, 1, 1)]
    assert f.quant[0][0] == 8 and f.quant[0][1] == 6                 # IJG luminance table at quality 75, natural order
    assert f.quant[0][8] == 6                                       # row 1, column 0: zig-zag position 2
    assert int(f.huff[(0, 0)][0].sum()) == 12 and int(f.huff[(1, 0)][0].sum()) == 162
    data = streams["420_q75"]
    assert data[f.scan[1]:] == b"\xff\xd9" and data[f.scan[0] - 14:f.scan[0] - 12] == b"\xff\xda"
    g = jpeg.parse(streams["gray_q75"])
    assert (g.ncomp, g.hmax, g.vmax, g.sampling, g.comp_blocks()) == (1, 1, 1, "gray", [(12, 8)])
    assert jpeg.parse(streams["422_q75"]).sampling == "4:2:2"
    assert jpeg.parse(streams["444_q75"]).comp_blocks() == [(12, 8)] * 3
    r = jpeg.parse(streams["420_restart3"])
    assert r.restart_interval == 3 and r.nseg == -(-(6 * 5) // 3)
    rows = jpeg.parse(streams["422_restart_rows"])
    assert rows.restart_interval == rows.mcus[0] and rows.nseg == rows.mcus[1]


def _replace_segment(data, marker, fn):
    """data with the payload of the first `marker` segment replaced by fn(payload)."""
    p = data.index(bytes([0xFF, marker]))
    ln = struct.unpack(">H", data[p + 2:p + 4])[0]
    new = fn(bytearray(data[p + 4:p + 2 + ln]))
    return data[:p + 2] + struct.pack(">H", len(new) + 2) + bytes(new) + data[p + 2 + ln:]


def test_parse_rejects_unsupported_streams(fixture, streams):
    with pytest.raises(ValueError, match="progressive"):
        jpeg.parse(fixture["reject_progressive"].tobytes())
    with pytest.raises(ValueError, match="CMYK"):
        jpeg.parse(fixture["reject_cmyk"].tobytes())
    base = streams["420_q75"]
    sof = base.index(b"\xff\xc0")
    for marker, reason in ((0xC9, "arithmetic-coded"), (0xC3, "lossless"), (0xC2, "progressive"), (0xC5, "hierarchical")):
        with pytest.raises(ValueError, match=reason):
            jpeg.parse(base[:sof + 1] + bytes([marker]) + base[sof + 2:])

    def set_byte(i, v):
        def f(seg):
            seg[i] = v
            return seg
        return f

    with pytest.raises(ValueError, match="12-bit"):
        jpeg.parse(_replace_segment(base, 0xC0, set_byte(0, 12)))
    with pytest.raises(ValueError, match="sampling factors 1x2"):          # 4:4:0
        jpeg.parse(_replace_segment(base, 0xC0, set_byte(7, 0x12)))
    with pytest.raises(ValueError, match="sampling factors"):              # chroma not 1x1
        jpeg.parse(_replace_segment(base, 0xC0, set_byte(10, 0x21)))
    # RGB-coded: component ids 'R', 'G', 'B' without JFIF, or an Adobe marker with transform 0
    no_jfif = base[:2] + base[2 + 2 + struct.unpack(">H", base[4:6])[0]:]
    assert jpeg.parse(no_jfif).ncomp == 3

    def rgb_ids(data):
        """Component ids 'R', 'G', 'B' in the frame header and the scan header."""
        def sof(seg):
            seg[6], seg[9], seg[12] = 0x52, 0x47, 0x42
            return seg

        def sos(seg):
            seg[1], seg[3], seg[5] = 0x52, 0x47, 0x42
            return seg
        return _replace_segment(_replace_segment(data, 0xC0, sof), 0xDA, sos)
    rgb = rgb_ids(no_jfif)
    with pytest.raises(ValueError, match="RGB-coded"):
        jpeg.parse(rgb)
    adobe = b"\xff\xee" + struct.pack(">H", 14) + b"Adobe" + bytes([0, 100, 0, 0, 0, 0, 0])
    with pytest.raises(ValueError, match="Adobe transform 0"):
        jpeg.parse(no_jfif[:2] + adobe + no_jfif[2:])
    # libjpeg decodes these as YCbCr (a JFIF marker wins over Adobe and ids; an Adobe marker wins over ids): accepted
    assert jpeg.parse(base[:2] + adobe + base[2:]).ncomp == 3
    assert jpeg.parse(no_jfif[:2] + adobe[:-1] + b"\x01" + no_jfif[2:]).ncomp == 3
    assert jpeg.parse(rgb[:2] + adobe[:-1] + b"\x01" + rgb[2:]).ncomp == 3
    assert jpeg.parse(rgb_ids(base)).ncomp == 3
    with pytest.raises(ValueError, match="image 1: CMYK"):
        jpeg.JpegBatch([base, fixture["reject_cmyk"].tobytes()])


def test_parse_rejects_malformed_headers(streams):
    base = streams["420_q75"]
    with pytest.raises(ValueError, match="no SOI"):
        jpeg.parse(base[2:])
    sos = base.index(b"\xff\xda")
    with pytest.raises(ValueError, match="before SOS"):
        jpeg.parse(base[:sos])                                            # no SOS
    with pytest.raises(ValueError, match="EOI before SOS"):
        jpeg.parse(base[:sos] + b"\xff\xd9")
    dqt = base.index(b"\xff\xdb")
    with pytest.raises(ValueError, match="length"):
        jpeg.parse(base[:dqt + 2] + b"\xff\xf0" + base[dqt + 4:])         # length past the end
    with pytest.raises(ValueError, match="length"):
        jpeg.parse(base[:dqt + 2] + b"\x00\x01" + base[dqt + 4:])         # length < 2
    with pytest.raises(ValueError, match="DQT"):
        jpeg.parse(_replace_segment(base, 0xDB, lambda s: s[:40]))        # table cut short
    with pytest.raises(ValueError, match="undefined Huffman"):
        jpeg.parse(_replace_segment(base, 0xDA, lambda s: s[:2] + bytes([0x33]) + s[3:]))
    with pytest.raises(ValueError, match="spectral"):
        jpeg.parse(_replace_segment(base, 0xDA, lambda s: s[:-2] + b"\x3f\x01"))
    with pytest.raises(ValueError, match="code space"):
        dht = jpeg.parse(base).huff[(0, 0)]
        jpeg.huff_table(np.array([3] + [0] * 15), dht[1])


def test_scan_ends_at_the_first_eoi(streams):
    """Data after EOI (a trailer holding another JPEG or a video) is not part of the scan, even when it contains restart
    and EOI markers."""
    for name in ("420_restart3", "420_q75"):
        data = streams[name]
        trailer = data + b"\xff\xd8\xff\xd0\x00\xff\xd3\xff\xd9" + data
        assert jpeg.parse(trailer).scan == jpeg.parse(data).scan
        assert np.array_equal(jpeg_oracle.decode(trailer), jpeg_oracle.decode(data))


def test_huffman_table_layout(streams):
    bits, vals = jpeg.parse(streams["420_q75"]).huff[(1, 0)]
    t = _lib.JpegHuff.from_buffer_copy(jpeg.huff_table(bits, vals))
    lut_len, lut_sym = jpeg_oracle._lut16(bits, vals)
    for p in range(0, 65536, 97):
        ln = lut_len[p]
        if ln <= 8:
            assert t.look[p >> 8] == (ln << 8 | lut_sym[p]), p
        else:
            assert t.look[p >> 8] == 0
            code = p >> (16 - ln)
            assert code <= t.maxcode[ln] and all(p >> (16 - l) > t.maxcode[l] for l in range(9, ln))
            assert t.val[code + t.valoff[ln]] == lut_sym[p]


def _batch(streams, names):
    return jpeg.JpegBatch([streams[n] for n in names])


def test_staging_layout(streams):
    names = ["420_q75", "gray_q75", "420_restart3", "444_q75", "420_q75"]
    b = _batch(streams, names)
    outs, nbytes = engine._output_table(b.shapes)
    h = b.fill(outs, np.full(b.nbytes, 0xAB, np.uint8))
    assert bytes(h[:ctypes.sizeof(b.images)]) == bytes(b.images)
    assert b.resize_off % 256 == 0 and bytes(h[b.resize_off:b.resize_off + ctypes.sizeof(outs)]) == bytes(outs)
    seg = blk = pix = 0
    for t, n, f in zip(b.images, names, b.infos):
        data = streams[n]
        assert bytes(h[t.scan_offset:t.scan_offset + t.scan_bytes]) == data[f.scan[0]:f.scan[1]]
        assert (t.seg_base, t.blk_base, t.pix_base) == (seg, blk, pix)
        seg, blk, pix = seg + f.nseg, blk + f.blocks, pix + f.height * f.width
        for c, (tq, td, ta) in enumerate(f.comps):
            assert t.quant[c] % 16 == 0 and t.dc[c] % 16 == 0 and t.ac[c] % 16 == 0
            q = np.frombuffer(bytes(h[t.quant[c]:t.quant[c] + 128]), "<u2")
            assert np.array_equal(q, f.quant[tq])
            assert bytes(h[t.dc[c]:t.dc[c] + ctypes.sizeof(_lib.JpegHuff)]) == jpeg.huff_table(*f.huff[(0, td)])
        assert all(v == 0 for v in list(t.quant)[f.ncomp:])
    # tables shared by identical streams: the repeated image points at the same bytes
    assert list(b.images[0].quant) == list(b.images[4].quant) and list(b.images[0].ac) == list(b.images[4].ac)
    assert (b.segments, b.blocks, b.pixels) == (seg, blk, pix)
    assert nbytes == 3 * pix


def _query(b, outs, in_bytes=None, y_bytes=None):
    return _lib.lib().odtk_decode_jpeg(None, b.nbytes if in_bytes is None else in_bytes, ctypes.byref(b.images), b.n,
                                       ctypes.byref(outs), None, None, 0, None,
                                       3 * b.pixels if y_bytes is None else y_bytes, None, None)


def test_abi_size_query_and_validation_need_no_gpu(streams):
    b = _batch(streams, ["420_q75", "gray_restart_rows", "444_restart3", "422_q75"])
    outs, _ = engine._output_table(b.shapes)
    assert _query(b, outs) == b.workspace_bytes() == jpeg.workspace_bytes(b.segments, b.blocks)
    assert _query(b, outs, in_bytes=b.nbytes - 1) == -1                  # last scan past the input
    assert _query(b, outs, y_bytes=3 * b.pixels - 1) == -1               # last image past the output
    L = _lib.lib()
    assert L.odtk_decode_jpeg(None, b.nbytes, None, b.n, ctypes.byref(outs), None, None, 0, None, 0, None, None) == -1
    assert L.odtk_decode_jpeg(None, b.nbytes, ctypes.byref(b.images), 0, ctypes.byref(outs), None, None, 0, None, 0,
                              None, None) == -1

    def check(field, value, want, obj="images", i=1):
        tab = getattr(b, "images") if obj == "images" else outs
        old = getattr(tab[i], field)
        if isinstance(value, tuple):
            getattr(tab[i], field)[value[0]] = value[1]
        else:
            setattr(tab[i], field, value)
        try:
            assert _query(b, outs) == want, (field, value)
        finally:
            if isinstance(value, tuple):
                getattr(tab[i], field)[value[0]] = old[value[0]] if not isinstance(old, int) else old
            else:
                setattr(tab[i], field, old)

    check("ncomp", 4, -3)
    b.images[0].height = b.images[0].width = 65535           # 2^32 pixels: beyond the kernels' int pixel index
    assert _query(b, outs) == -3
    b.images[0].height, b.images[0].width = b.infos[0].height, b.infos[0].width
    check("hmax", 2, -3)                     # grayscale with 2x1 sampling
    check("vmax", 2, -3, i=2)                # 1x2 luma on a YCbCr image: 4:4:0
    check("height", 0, -1)
    check("scan_bytes", 0, -1)
    check("nseg", 1, -1)                     # restart segments do not match the interval
    check("seg_base", 0, -1, i=2)
    check("blk_base", 0, -1, i=2)
    check("pix_base", 0, -1, i=2)
    check("src_w", 1, -1, obj="outs")
    check("offset", -3, -1, obj="outs")
    saved = b.images[0].quant[1]
    for bad in (saved + 4, 0, b.nbytes):
        b.images[0].quant[1] = bad           # misaligned, null, past the input
        assert _query(b, outs) == -1
    b.images[0].quant[1] = saved
    assert _query(b, outs) == b.workspace_bytes()
