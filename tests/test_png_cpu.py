"""The PNG decoder's host side, without a GPU: the two gray rules against the installed readers, the test's PNG writer, the
workspace planner against a Python restatement, and the `images` feed's refusals of bad bytes before any launch."""
import io
import os
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import png_refs as P  # noqa: E402


def _cv2(data):
    import cv2
    return cv2.imdecode(np.frombuffer(data, np.uint8), 0)


def _pil(data):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(data)).convert("L"), dtype=np.uint8)


READERS = {0: _cv2, 1: _pil}


@pytest.mark.parametrize("rule", [0, 1])
def test_8bit_colour_rule_on_all_colours(rule):
    """Every one of the 2^24 colours, as a 4096 x 4096 RGB file, through the reader."""
    c = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([c >> 16, (c >> 8) & 255, c & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    data = P.write_png(img, 8, 2, level=1)
    got = READERS[rule](data)
    assert np.array_equal(got, P.gray(img, 8, 2, rule))


@pytest.mark.parametrize("rule", [0, 1])
def test_16bit_and_alpha_rules(rule):
    rng = np.random.default_rng(rule)
    edge = np.array([0, 1, 127, 128, 255, 256, 32767, 32768, 65280, 65534, 65535], np.uint16)
    for ctype in (0, 2, 4, 6):
        img = P.random_image(rng, 256, 512, 16, ctype)
        flat = img.reshape(256 * 512, -1)
        flat[:edge.size] = edge[:, None]                   # equal channels at the edge values
        flat[edge.size:2 * edge.size, 0] = edge
        got = READERS[rule](P.write_png(img, 16, ctype, filters="random", rng=rng))
        assert np.array_equal(got, P.gray(img, 16, ctype, rule)), ctype


@pytest.mark.parametrize("rule", [0, 1])
def test_writer_and_rules_on_every_colour_type(rule):
    rng = np.random.default_rng(10 + rule)
    for ctype, depths in P.DEPTHS.items():
        for depth in depths:
            for il in (0, 1):
                pal = rng.integers(0, 256, (1 << depth, 3)).astype(np.uint8) if ctype == 3 else None
                img = P.random_image(rng, 19, 21, depth, ctype, None if pal is None else len(pal))
                data = P.write_png(img, depth, ctype, il, pal, filters="random", rng=rng, split=40, zero_chunks=True)
                assert len(zlib.decompress(b"".join(d for t, d in P.chunks_of(data) if t == b"IDAT"))) == P.raw_len(19, 21, depth,
                                                                                                                 ctype, il)
                assert np.array_equal(READERS[rule](data), P.gray(img, depth, ctype, rule, pal)), (ctype, depth, il)


def test_host_readers_act_on_gamma_and_orientation():
    """Why the decoder refuses these files: OpenCV gamma-corrects colour files that carry gAMA or sRGB and turns files by their
    eXIf orientation; Pillow does neither."""
    rng = np.random.default_rng(3)
    img = P.random_image(rng, 5, 9, 8, 2)
    for extra in (P.chunk(b"gAMA", (45455).to_bytes(4, "big")), P.chunk(b"sRGB", b"\0")):
        data = P.write_png(img, 8, 2, extra=extra)
        assert not np.array_equal(_cv2(data), P.gray(img, 8, 2, 0))
        assert np.array_equal(_pil(data), P.gray(img, 8, 2, 1))
    exif = P.chunk(b"eXIf", b"MM\0*\0\0\0\x08\0\x01\x01\x12\0\x03\0\0\0\x01\0\x06\0\0\0\0\0\0")
    assert _cv2(P.write_png(img, 8, 2, extra=exif)).shape == (9, 5)


def test_planner_against_the_python_layout():
    from lstm_ctc_ocr_b200 import engine
    ihdr, flen, want = [], [], []
    for ctype, depths in P.DEPTHS.items():
        for depth in depths:
            for il in (0, 1):
                for h in range(1, 18):
                    for w in range(1, 18):
                        ihdr.append(np.frombuffer(P.ihdr(h, w, depth, ctype, il), np.uint8))
                        flen.append(100 + h * w)
                        want.append((flen[-1] + 15) // 16 * 16 + (P.raw_len(h, w, depth, ctype, il) + 15) // 16 * 16)
    for bad in (P.ihdr(0, 5, 8, 0), P.ihdr(5, 0, 8, 0), P.ihdr(1025, 5, 8, 0), P.ihdr(5, 5, 3, 0), P.ihdr(5, 5, 8, 5),
                P.ihdr(5, 5, 16, 3), b"\0\0\0\5\0\0\0\5\x08\0\1\0\0", b"\0\0\0\5\0\0\0\5\x08\0\0\0\2"):
        ihdr.append(np.frombuffer(bad, np.uint8))
        flen.append(50)
        want.append(0)
    off, total = engine.png_plan(np.stack(ihdr), np.array(flen, np.int64))
    assert off[0] == 0 and np.array_equal(np.diff(off), want) and total == off[-1] == sum(want)


def test_images_feed_refuses_bad_bytes_before_any_launch():
    from lstm_ctc_ocr_b200.session import Session
    good = P.write_png(np.zeros((3, 4), np.uint8), 8, 0)
    assert Session._images_feed([good, np.zeros((2, 2), np.uint8), bytearray(good)])[0] is good
    cases = {"jpeg": b"\xff\xd8\xff\xe0" + bytes(40), "truncated": good[:30], "no_ihdr": good[:12] + b"IHDX" + good[16:],
             "zero_w": good[:16] + bytes(4) + good[20:], "zero_h": good[:20] + bytes(4) + good[24:],
             "tall": good[:20] + (1025).to_bytes(4, "big") + good[24:], "empty": b"",
             "wide": good[:16] + (1000001).to_bytes(4, "big") + good[20:], "wider_than_int32": good[:16] + b"\xff" * 4 + good[20:]}
    for name, data in cases.items():
        with pytest.raises(ValueError):
            Session._images_feed([good, data])


def test_test_model_feeds_only_pngs_the_device_reads(tmp_path, monkeypatch):
    from lstm_ctc_ocr_b200.lib.lstm import test as T
    good = P.write_png(np.zeros((3, 4), np.uint8), 8, 0)
    monkeypatch.setattr(T, "load_line_image", lambda path: "host")
    for name, data in (("wide", P.assemble([(b"IHDR", P.ihdr(3, 1000001, 8, 0)), (b"IEND", b"")])),
                       ("tall", P.assemble([(b"IHDR", P.ihdr(1025, 4, 8, 0)), (b"IEND", b"")])), ("jpeg", b"\xff\xd8\xff\xe0")):
        (tmp_path / name).write_bytes(data)
        assert T._line_entry(str(tmp_path / name)) == "host", name
    (tmp_path / "good").write_bytes(good)
    assert T._line_entry(str(tmp_path / "good")) == good


@pytest.mark.parametrize("chunk_type", [b"zTXt", b"iCCP", b"iTXt"])
def test_pillow_refuses_text_that_inflates_past_one_mib(chunk_type):
    """Why rule 1 refuses compressed payloads above 1016 bytes: Pillow raises past 1 MiB of inflated text (DEFLATE inflates a byte
    to at most 1032), while OpenCV reads the file."""
    payload = zlib.compress(b"\0" * (2 << 20), 9)
    assert 1016 < len(payload) < 4096 and 1016 * 1032 < 1 << 20
    head = b"k\0\1\0\0\0" if chunk_type == b"iTXt" else b"k\0\0"
    img = np.zeros((3, 4), np.uint8)
    data = P.write_png(img, 8, 0, extra=P.chunk(chunk_type, head + payload))
    assert np.array_equal(_cv2(data), img)
    with pytest.raises(ValueError):
        _pil(data)
