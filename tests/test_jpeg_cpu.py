"""The JPEG decoder's host side, without a GPU: the restatement (tests/jpeg_refs.py) against the installed readers byte for byte
under both gray rules, why the IDCT envelope and the Exif refusal exist, jpeg_size / jpeg_plan, and the `images` feed's and
test_model's handling of JPEG bytes."""
import io
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import jpeg_refs as J  # noqa: E402

CV2_SAMPLING = {411: 0x411111, 420: 0x221111, 422: 0x211111, 440: 0x121111, 444: 0x111111}


def host(data, rule):
    import cv2
    from PIL import Image
    if rule == 0:
        return cv2.imdecode(np.frombuffer(data, np.uint8), 0)
    return np.asarray(Image.open(io.BytesIO(data)).convert("L"), dtype=np.uint8)


def _pil(im, **kw):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(im).save(b, "JPEG", **kw)
    return b.getvalue()


def _cv2(im, *params):
    import cv2
    ok, enc = cv2.imencode(".jpg", im, list(params))
    assert ok
    return enc.tobytes()


def _line(rng, h, w):
    return (rng.integers(0, 2, (h, w)) * 200 + rng.integers(0, 40, (h, w))).astype(np.uint8)


def corpus(seed=1, big=True):
    """[(name, file bytes)] of files the device reads under both rules, except the 4:1:1 colour files (`rule1_refused`)."""
    import cv2
    rng = np.random.default_rng(seed)
    out = []
    line = _line(rng, 60, 300)
    colour = np.stack([line, line[::-1], 255 - line], -1)
    for q in list(range(1, 101, 9)) + [100]:
        for ss in (0, 1, 2):
            out.append((f"pil_q{q}_ss{ss}", _pil(colour[:45, :133], quality=q, subsampling=ss)))
        out.append((f"pil_gray_q{q}", _pil(line[:45, :133], quality=q)))
    for kw in (dict(optimize=True), dict(restart_marker_blocks=3), dict(restart_marker_rows=1), dict(optimize=True, subsampling=2,
               restart_marker_blocks=1)):
        out.append(("pil_" + "_".join(f"{k}{v}" for k, v in kw.items()), _pil(colour[:33, :77], quality=80, **kw)))
        out.append(("pil_gray_" + "_".join(f"{k}{v}" for k, v in kw.items()), _pil(line[:33, :77], quality=80, **kw)))
    for sf, code in CV2_SAMPLING.items():
        for rst in (0, 1, 5):
            out.append((f"cv2_{sf}_rst{rst}", _cv2(colour[:37, :101], cv2.IMWRITE_JPEG_SAMPLING_FACTOR, code,
                                                   cv2.IMWRITE_JPEG_RST_INTERVAL, rst, cv2.IMWRITE_JPEG_QUALITY, 90)))
    out.append(("cv2_gray", _cv2(line, cv2.IMWRITE_JPEG_QUALITY, 95)))
    out.append(("cv2_gray_rst2", _cv2(line, cv2.IMWRITE_JPEG_RST_INTERVAL, 2)))
    out.append(("cv2_gray_opt", _cv2(line, cv2.IMWRITE_JPEG_OPTIMIZE, 1)))
    sizes = [(1, 1), (1, 2), (2, 1), (3, 3), (7, 9), (8, 8), (9, 17), (15, 16), (16, 15), (17, 33), (31, 31), (33, 65)]
    if big:
        sizes += [(1024, 8), (1024, 3), (5, 4096), (1, 4096)]
    for h, w in sizes:
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        for ss in (0, 1, 2):
            out.append((f"pil_{h}x{w}_ss{ss}", _pil(img, quality=85, subsampling=ss)))
        out.append((f"pil_gray_{h}x{w}", _pil(img[..., 0], quality=85)))
        out.append((f"cv2_440_{h}x{w}", _cv2(img, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x121111)))
        out.append((f"cv2_411_{h}x{w}", _cv2(img, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x411111)))
    out += written(rng)
    return out


def written(rng):
    """Files from the test writer: gray files declaring 2 x 2 sampling, custom tables, fill bytes, and extreme coefficients
    inside the IDCT envelope (outputs in the clamped parts of the range-limit table)."""
    out = []
    q1 = np.ones(64, np.int64)
    for h, w in ((9, 17), (16, 16), (23, 5)):
        blocks = J.quantise(_line(rng, h, w), q1 * 4)
        out.append((f"w_gray_2x2_{h}x{w}", J.encode([blocks], {0: q1 * 4}, h, w, sampling=[(2, 2)])))
    img = _line(rng, 21, 40)
    blocks = J.quantise(img, q1 * 3)
    long_dc = ([0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 6], list(range(12)))     # codes of 10 .. 16 bits
    tables = {(0, 0): long_dc, (1, 0): J.STD_AC_LUMA}
    out.append(("w_long_dc_codes", J.encode([blocks], {0: q1 * 3}, 21, 40, tables=tables)))
    out.append(("w_fill_rst", J.encode([blocks], {0: q1 * 3}, 21, 40, ri=2, fill=3)))
    out.append(("w_16bit_dqt", J.encode([J.quantise(img, q1 * 300)], {0: q1 * 300}, 21, 40)))
    out.append(("w_sof1", J.encode([blocks], {0: q1 * 3}, 21, 40, sof_marker=0xC1)))
    # extreme DC and AC: output sums in [-512, 511] beyond [-128, 127], the table's clamped parts
    ext = np.zeros((3, 5, 64), np.int64)
    ext[..., 0] = np.array([0, 1700, 3400, 1700, 0, -1700, -3400, -1700, 0, 1600, 3200, 1600, 0, -1600, -3200]).reshape(3, 5)
    ext[..., 1:] = rng.integers(-20, 21, (3, 5, 63)) * (rng.random((3, 5, 63)) < 0.2)
    out.append(("w_extreme", J.encode([ext], {0: q1}, 24, 40)))
    ext3 = [ext, -ext, ext]
    out.append(("w_extreme_colour", J.encode(ext3, {0: q1, 1: q1}, 24, 40, app=J.segment(0xE0, b"JFIF\0\1\1\0\0\1\0\1\0\0"))))
    return out


def rule1_refused(name):
    return name.startswith("cv2_411")


@pytest.mark.parametrize("rule", [0, 1])
def test_restatement_equals_the_host_reader(rule):
    bad = []
    for name, data in corpus():
        want = host(data, rule)
        try:
            got = J.decode(data, rule)
        except J.Refused as r:
            if not (rule == 1 and rule1_refused(name) and r.status == J.HOST_DIFFERS):
                bad.append((name, "refused", r.status))
            continue
        if rule == 1 and rule1_refused(name):
            bad.append((name, "read under rule 1"))
        elif got.shape != want.shape or not np.array_equal(got, want):
            bad.append((name, int((got != want).sum()) if got.shape == want.shape else "shape"))
    assert not bad, bad[:10]


def test_zero_ac_shortcuts_are_exact():
    """jidctint.c's column and row shortcuts give what the full butterflies give, on every block of the corpus."""
    for name, data in corpus(seed=2, big=False)[::3]:
        _, geo, coef = J.coefficients(data, 1 if not rule1_refused(name) else 0)
        for c in coef:
            q = np.arange(1, 65)
            a, ia = J.idct_islow(c.reshape(-1, 64), q, True)
            b, ib = J.idct_islow(c.reshape(-1, 64), q, False)
            assert np.array_equal(a, b) and np.array_equal(ia, ib), name


def test_host_saturates_where_the_range_limit_table_wraps():
    """Why blocks outside the envelope are refused: an output sum of 600 wraps to 0 through jidctint.c's table, while the host
    readers (libjpeg-turbo's SIMD IDCT) give 255."""
    blk = np.zeros((1, 1, 64), np.int64)
    blk[0, 0, 0] = 1200                                    # DC only, dequantised 4800: every output sum (4800 * 4 + 16) >> 5 = 600
    data = J.encode([blk], {0: np.full(64, 4, np.int64)}, 8, 8)
    px, inside = J.idct_islow(blk.reshape(1, 64), np.full(64, 4))
    assert not inside[0] and (px == 0).all()
    for rule in (0, 1):
        assert (host(data, rule) == 255).all()
        with pytest.raises(J.Refused) as e:
            J.decode(data, rule)
        assert e.value.status == J.HOST_DIFFERS


def _exif(orientation, le=True):
    bo = "little" if le else "big"
    ifd = (1).to_bytes(2, bo) + (0x0112).to_bytes(2, bo) + (3).to_bytes(2, bo) + (1).to_bytes(4, bo) + \
        orientation.to_bytes(2, bo) + b"\0\0" + bytes(4)
    tiff = (b"II*\0" if le else b"MM\0*") + (8).to_bytes(4, bo) + ifd
    return J.segment(0xE1, b"Exif\0\0" + tiff)


def with_exif(data, orientation, le=True):
    return data[:2] + _exif(orientation, le) + data[2:]


def test_opencv_turns_by_exif_orientation_and_pillow_does_not():
    rng = np.random.default_rng(3)
    img = _line(rng, 16, 40)
    base = _pil(img, quality=90)
    for o in range(1, 9):
        for le in (True, False):
            data = with_exif(base, o, le)
            assert np.array_equal(host(data, 1), host(base, 1))
            if o == 1:
                assert np.array_equal(host(data, 0), host(base, 0)) and np.array_equal(J.decode(data, 0), host(base, 0))
            else:
                assert not np.array_equal(host(data, 0), host(base, 0)) or host(data, 0).shape != host(base, 0).shape
                with pytest.raises(J.Refused):
                    J.decode(data, 0)
            assert np.array_equal(J.decode(data, 1), host(data, 1))


def test_jpeg_size_and_sof():
    from lstm_ctc_ocr_b200 import engine
    data = _pil(np.zeros((37, 91, 3), np.uint8))
    assert engine.jpeg_size(data) == (37, 91) and engine.jpeg_sof(data)[0] == 0xC0
    prog = _pil(np.zeros((5, 9), np.uint8), progressive=True)
    assert engine.jpeg_size(prog) == (5, 9) and engine.jpeg_sof(prog)[0] == 0xC2
    assert engine.jpeg_size(b"\xff\xd8\xff\xe0" + bytes(40)) is None           # APP0 of length 0
    assert engine.jpeg_size(b"\xff\xd8\xff\xe0") is None
    assert engine.jpeg_size(data[:20]) is None
    assert engine.jpeg_size(b"\xff\xd8\xff\xd9") is None                       # EOI before a frame
    assert engine.jpeg_size(b"\xff\xd8\xff\xff\xff" + data[3:]) == (37, 91)    # fill bytes
    assert engine.jpeg_size(b"\x89PNG") is None


def test_planner_against_the_python_layout():
    from lstm_ctc_ocr_b200 import engine
    recs, flen, want = [], [], {0: [], 1: []}
    for nf, samp in ((1, [(1, 1)]), (1, [(2, 2)]), (3, [(1, 1)] * 3), (3, [(2, 2), (1, 1), (1, 1)]), (3, [(2, 1), (1, 1), (1, 1)]),
                     (3, [(1, 2), (1, 1), (1, 1)]), (3, [(4, 1), (1, 1), (1, 1)]), (3, [(1, 1), (2, 2), (1, 1)])):
        for h, w in ((1, 1), (7, 9), (8, 8), (17, 33), (1024, 3), (2, 65535)):
            sof = bytes([8]) + h.to_bytes(2, "big") + w.to_bytes(2, "big") + bytes([nf]) + b"".join(
                bytes([c + 1, (H << 4) | V, 0]) for c, (H, V) in enumerate(samp))
            recs.append(np.frombuffer(sof.ljust(16, b"\0"), np.uint8))
            flen.append(1000)
            fr = dict(h=h, w=w, comps=[(c + 1, H, V, 0) for c, (H, V) in enumerate(samp)])
            geo, hmax, vmax, mcux, mcuy = J.geometry(fr, 0)
            for rule in (0, 1):
                stored = geo if rule == 1 and nf == 3 else geo[:1]
                n = 512 + -(-((mcux * mcuy + 1) * 8) // 16) * 16 + sum(g[2] * g[3] * 128 for g in stored)
                if rule == 1 and nf == 3:
                    n += sum(g[2] * g[3] * 64 for g in geo)
                want[rule].append(n)
    for bad in (b"\x0c\0\5\0\5\1\1\x11\0", b"\x08\0\0\0\5\1\1\x11\0", b"\x08\4\1\0\5\1\1\x11\0", b"\x08\0\5\0\0\1\1\x11\0",
                b"\x08\0\5\0\5\2\1\x11\0\2\x11\0", b"\x08\0\5\0\5\1\1\x51\0", b"\x08\0\5\0\5\3\1\x22\0\2\x22\0\3\x22\0"):
        recs.append(np.frombuffer(bad.ljust(16, b"\0"), np.uint8))
        flen.append(50)
        want[0].append(0)
        want[1].append(0)
    for rule in (0, 1):
        off, total = engine.jpeg_plan(np.stack(recs), np.array(flen, np.int64), rule)
        assert off[0] == 0 and np.array_equal(np.diff(off), want[rule]) and total == off[-1] == sum(want[rule])


def test_images_feed_takes_jpeg_bytes_and_refuses_bad_ones():
    from lstm_ctc_ocr_b200.session import Session
    good = _pil(np.zeros((3, 4), np.uint8))
    assert Session._images_feed([good, np.zeros((2, 2), np.uint8), bytearray(good)])[0] is good
    for data in (b"\xff\xd8\xff\xe0" + bytes(40), good[:10], J.encode([np.zeros((129, 1, 64))], {0: np.ones(64)}, 1025, 8),
                 good[:5] + b"\0\0" + good[7:]):
        with pytest.raises(ValueError):
            Session._images_feed([good, data])


def test_test_model_feeds_only_jpegs_the_device_reads(tmp_path, monkeypatch):
    from lstm_ctc_ocr_b200.lib.lstm import test as T
    monkeypatch.setattr(T, "load_line_image", lambda path: "host")
    good = _pil(np.zeros((3, 4), np.uint8))
    for name, data in (("progressive", _pil(np.zeros((3, 4), np.uint8), progressive=True)), ("truncated", good[:8]),
                       ("tall", J.encode([np.zeros((129, 1, 64))], {0: np.ones(64)}, 1025, 8))):
        (tmp_path / name).write_bytes(data)
        assert T._line_entry(str(tmp_path / name)) == "host", name
    (tmp_path / "good").write_bytes(good)
    assert T._line_entry(str(tmp_path / "good")) == good
    assert T._entry_size(good) == (3, 4)


def test_decode_error_classes():
    from lstm_ctc_ocr_b200 import engine
    p, j = engine.PngDecodeError([1], [3]), engine.JpegDecodeError([2, 4], [5, 7])
    assert isinstance(p, engine.ImageDecodeError) and isinstance(j, engine.ImageDecodeError)
    assert str(p) == "images: entries [1] are PNG files the device decoder refused (bad CRC)"
    assert j.entries == [2, 4] and j.status == [5, 7] and "JPEG" in str(j)


def test_jpeg_size_reads_frames_behind_large_segments():
    """Segments before the frame may be long (ICC profiles, thumbnails): the walk reads only their headers."""
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.session import Session
    data = _pil(np.zeros((37, 91), np.uint8))
    big = data[:2] + J.segment(0xE2, bytes(65000)) * 20 + data[2:]
    assert len(big) > 1 << 20 and engine.jpeg_size(big) == (37, 91) and engine.jpeg_size(bytearray(big)) == (37, 91)
    assert Session._images_feed([big])[0] is big
    assert np.array_equal(J.decode(big, 0), host(big, 0))


def test_mixed_decode_error_names_each_codec():
    from lstm_ctc_ocr_b200 import engine
    e = engine.ImageDecodeError.mixed([(4, 7, "JPEG"), (1, 3, "PNG")])
    assert type(e) is engine.ImageDecodeError and e.entries == [1, 4] and e.status == [3, 7]
    assert str(e) == ("images: entries [1, 4] are files the device decoders refused (PNG bad CRC, "
                      "JPEG the host reader computes something else)")
