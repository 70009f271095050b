"""PNG files decoded on the GPU (crnn_png_decode_gray_u8, the `images` feed's PNG entries) against the installed host readers.

  1. Byte equality with cv2.imdecode(..., 0) (rule 0) and Pillow's convert("L") (rule 1) over a seeded corpus built here: every
     colour type x bit depth x interlace, each filter forced and drawn per row, zlib levels 0-9, its strategies and windows
     9-15, IDAT split into 1-byte and zero-length chunks, 1 x 1 to 1024-row and 4096-column images, files written by
     cv2.imwrite and Pillow (optimize too), rendered lines, and files with the ancillary chunks both readers ignore.  The
     output is filled with 0xA5 first, so every byte is shown written; every status is 0.
  2. The workspace stages: the gathered zlib stream equals the IDAT payloads, and the scanline region zlib.decompress of it
     with each row's filter undone (restated in png_refs.unfilter).
  3. One defect per file of each class the decoder refuses: its status, an all-zero slot, and the other files of the call
     identical to decoding them alone, in any order; repeat runs bit-identical.
  4. Guarded buffers of exactly the planned sizes (tests/bounds.py): no guard written, no read past an input (a truncated file
     last); status codes of bad arguments with the outputs untouched; a gated stream behind a busy default stream; graph
     capture and replay.
  5. Session.run with bytes, arrays and a mix, and test_model on a directory of PNGs of every kind, a JPEG and refused PNGs,
     under both rules, against the host path."""
import io
import os
import random
import sys
import zlib
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import png_refs as P  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _host(data, rule):
    import cv2
    from PIL import Image
    if rule == 0:
        return cv2.imdecode(np.frombuffer(data, np.uint8), 0)
    return np.asarray(Image.open(io.BytesIO(data)).convert("L"), dtype=np.uint8)


def _plan(files):
    from lstm_ctc_ocr_b200 import engine
    ihdr = np.stack([np.frombuffer(f[16:29].ljust(13, b"\0"), np.uint8) for f in files])
    return engine.png_plan(ihdr, np.array([len(f) for f in files], np.int64))


def _args(files, sizes=None):
    """Device arguments for `files`: (files, file_offset, file_len, h, w, out_offset, ws_offset), the ws bytes, the out bytes."""
    from lstm_ctc_ocr_b200 import engine
    sizes = sizes or [engine.png_size(f) or (1, 1) for f in files]
    flen = np.array([len(f) for f in files], np.int64)
    foff = np.zeros(len(files), np.int64)
    np.cumsum(flen[:-1], out=foff[1:])
    hw = np.array(sizes, np.int64).reshape(-1, 2)
    dec = hw[:, 0] * hw[:, 1]
    ooff = np.zeros(len(files), np.int64)
    np.cumsum(dec[:-1], out=ooff[1:])
    ws_offset, ws_bytes = _plan(files)
    t = lambda a: torch.tensor(np.ascontiguousarray(a), device=DEV)  # noqa: E731
    return ((t(np.frombuffer(b"".join(files), np.uint8)), t(foff), t(flen), t(hw[:, 0].astype(np.int32)), t(hw[:, 1].astype(np.int32)),
             t(ooff), t(ws_offset)), ws_bytes, int(dec.sum()), hw, ooff)


def _decode(files, rule, sizes=None, keep_ws=False):
    """[(image or None, status)] for each file of one call, after 0xA5 fills of the output and the workspace."""
    from lstm_ctc_ocr_b200 import engine
    a, ws_bytes, nout, hw, ooff = _args(files, sizes)
    out = torch.full((max(nout, 1),), 0xA5, dtype=torch.uint8, device=DEV)
    ws = torch.full((max(ws_bytes, 1),), 0xA5, dtype=torch.uint8, device=DEV)
    _, st = engine.decode_png_gray(*a, rule, out=out, workspace=ws)
    o, s = out.cpu().numpy(), st.cpu().numpy()
    res = [(o[ooff[i]:ooff[i] + hw[i, 0] * hw[i, 1]].reshape(hw[i, 0], hw[i, 1]), int(s[i])) for i in range(len(files))]
    return (res, ws.cpu().numpy(), a[6].cpu().numpy()) if keep_ws else res


# ------------------------------------------------------------------------------------------------ the corpus
def _palette(rng, depth, n=None):
    return rng.integers(0, 256, (n or (1 << depth), 3)).astype(np.uint8)


def _corpus(seed=1):
    """[(name, file bytes)] of valid files; each must decode with status 0 under both rules and equal the host readers."""
    import cv2
    from PIL import Image
    rng = np.random.default_rng(seed)
    out = []

    def add(name, img, depth, ctype, **kw):
        pal = kw.pop("palette", None)
        if ctype == 3 and pal is None:
            pal = _palette(rng, depth)
        out.append((name, P.write_png(img, depth, ctype, palette=pal, rng=rng, **kw)))

    for ctype, depths in P.DEPTHS.items():
        for depth in depths:
            for il in (0, 1):
                for h, w in ((1, 1), (1, 13), (13, 1), (3, 5), (7, 9), (17, 23), (33, 70)):
                    npal = (1 << depth) if ctype == 3 else None
                    img = P.random_image(rng, h, w, depth, ctype, npal)
                    add(f"c{ctype}d{depth}i{il}_{h}x{w}", img, depth, ctype, interlace=il, filters="random")
    for f in range(5):                                   # each filter on every row
        for depth, ctype in ((8, 0), (16, 2), (8, 6), (2, 0), (8, 4)):
            img = P.random_image(rng, 11, 37, depth, ctype)
            add(f"filter{f}_c{ctype}d{depth}", img, depth, ctype, filters=f)
            add(f"filter{f}_c{ctype}d{depth}_adam7", img, depth, ctype, filters=f, interlace=1)
    line = (rng.integers(0, 2, (60, 300)) * 200 + rng.integers(0, 40, (60, 300))).astype(np.uint8)
    strategies = (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE, zlib.Z_FIXED)
    for level in range(10):
        for s in strategies:
            add(f"zlib_l{level}_s{s}", line, 8, 0, level=level, strategy=s, filters="random")
    for wbits in range(9, 16):
        add(f"zlib_w{wbits}", line, 8, 0, wbits=wbits, filters="random")
    big = rng.integers(0, 256, (60, 2300), dtype=np.uint8)          # 138 060 raw bytes: 65 535-byte stored blocks
    add("stored_big", big, 8, 0, level=0)
    small = P.random_image(rng, 6, 7, 8, 2)
    add("idat_1byte", small, 8, 2, split=1)
    add("idat_zero_chunks", small, 8, 2, split=17, zero_chunks=True)
    add("idat_only_zero_chunks_around", small, 8, 2, zero_chunks=True)
    add("tall_1024", rng.integers(0, 256, (1024, 5), dtype=np.uint8), 8, 0, filters="random")
    add("tall_1024_x1_adam7", rng.integers(0, 2, (1024, 1), dtype=np.uint8), 1, 0, interlace=1)
    add("wide_4096", rng.integers(0, 256, (3, 4096), dtype=np.uint8), 8, 0, filters=4)
    add("wide_4096_rgb16", P.random_image(rng, 2, 4096, 16, 2), 16, 2)
    add("pal_short", rng.integers(0, 5, (9, 9)).astype(np.uint8), 8, 3, palette=_palette(rng, 8, 5))
    # writers the project's users have: cv2.imwrite and Pillow
    gray_line = line
    color_line = np.stack([line, line[::-1], 255 - line], -1)
    for level in range(10):
        for s in range(5):
            for name, im in (("gray", gray_line), ("bgr", color_line)):
                ok, enc = cv2.imencode(".png", im, [cv2.IMWRITE_PNG_COMPRESSION, level, cv2.IMWRITE_PNG_STRATEGY, s])
                assert ok
                out.append((f"cv2_{name}_l{level}_s{s}", enc.tobytes()))
    ok, enc = cv2.imencode(".png", (line.astype(np.uint16) * 257))
    out.append(("cv2_gray16", enc.tobytes()))
    for mode in ("L", "RGB", "RGBA", "LA", "P", "1", "I;16"):
        base = Image.fromarray(gray_line)
        im = base.convert(mode) if mode not in ("I;16",) else Image.fromarray((line.astype(np.uint16) * 251))
        if mode == "P":
            im = Image.fromarray(color_line).convert("P")
        for opt in (False, True):
            b = io.BytesIO()
            im.save(b, "PNG", optimize=opt)
            out.append((f"pil_{mode}_opt{int(opt)}", b.getvalue()))
    # ancillary chunks that change neither reader, the colour-space ones before PLTE where the specification puts them (libpng
    # ignores them after it).  gAMA, sRGB and iCCP on palette and colour files change OpenCV's bytes: test_colour_gamma_...
    chrm = P.chunk(b"cHRM", b"".join(v.to_bytes(4, "big") for v in (31270, 32900, 64000, 33000, 30000, 60000, 15000, 6000)))
    for ctype, depth in ((0, 8), (3, 4), (0, 16), (4, 8), (3, 8)):
        img = P.random_image(rng, 9, 21, depth, ctype, 16 if ctype == 3 else None)
        trns = (P.chunk(b"tRNS", bytes(2)) if ctype == 0 else P.chunk(b"tRNS", bytes(range(5))) if ctype == 3 else b"")
        sbit = P.chunk(b"sBIT", bytes([min(depth, 8)] * (3 if ctype == 3 else P.CHANNELS[ctype])))
        space = chrm + sbit
        if ctype != 3:
            space += (P.chunk(b"gAMA", (45455).to_bytes(4, "big")) + P.chunk(b"sRGB", b"\0")
                      + P.chunk(b"iCCP", b"icc\0\0" + zlib.compress(b"\0" * 200)))
        extra = trns + P.chunk(b"tEXt", b"Title\0a line") + P.chunk(b"zTXt", b"k\0\0" + zlib.compress(b"text" * 50)) \
            + P.chunk(b"pHYs", bytes(9))
        add(f"ancillary_c{ctype}d{depth}", img, depth, ctype, pre_plte=space, extra=extra,
            palette=_palette(rng, 8, 16) if ctype == 3 else None)
    return out


def _rendered(n=2048, seed=7):
    """Lines as the evaluation set holds them: 30-70 characters, rendered, saved by Pillow (as genImg saves them)."""
    from PIL import Image
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    r = random.Random(seed)
    font = gen.embedded_font(42)
    out = []
    for i in range(n):
        b = io.BytesIO()
        Image.fromarray(gen.render_line(gen.gen_rand(r, 30, 70), rng=r, font=font)).save(b, "PNG")
        out.append((f"line{i}", b.getvalue()))
    return out


def _check_equal(corpus, rule, chunk=512):
    bad = []
    for k in range(0, len(corpus), chunk):
        part = corpus[k:k + chunk]
        got = _decode([f for _, f in part], rule)
        for (name, f), (img, st) in zip(part, got):
            want = _host(f, rule)
            if st != 0 or want is None or img.shape != want.shape or not np.array_equal(img, want):
                bad.append((name, st, None if want is None else int((img != want).sum()) if img.shape == want.shape else "shape"))
    assert not bad, f"{len(bad)} of {len(corpus)} files differ from the rule-{rule} reader (name, status, bytes): {bad[:12]}"


@pytest.mark.parametrize("rule", [0, 1])
def test_corpus_equals_the_host_reader_byte_for_byte(rule):
    _check_equal(_corpus(), rule)


@pytest.mark.parametrize("rule", [0, 1])
def test_rendered_lines_equal_the_host_reader(rule, monkeypatch):
    monkeypatch.setenv("CRNN_FONT", "default")
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    gen._FONT_CACHE.clear()
    _check_equal(_rendered(), rule)


def test_colour_gamma_is_refused_under_opencv_only():
    """libpng gamma-corrects its RGB -> gray conversion, palette entries included, when a colour or palette file carries gAMA,
    sRGB or iCCP: rule 0 refuses those files, rule 1 (Pillow ignores them) reads them."""
    rng = np.random.default_rng(4)
    img = P.random_image(rng, 5, 9, 8, 2)
    gama = P.chunk(b"gAMA", (45455).to_bytes(4, "big"))
    srgb = P.chunk(b"sRGB", b"\0")
    pal8, pal4 = _palette(rng, 8), _palette(rng, 4)
    pimg8, pimg4 = P.random_image(rng, 16, 16, 8, 3, 256), P.random_image(rng, 16, 16, 4, 3, 16)
    files = [P.write_png(img, 8, 2, extra=gama), P.write_png(img, 8, 2, extra=srgb),
             P.write_png(P.random_image(rng, 5, 9, 16, 6), 16, 6, extra=P.chunk(b"iCCP", b"icc\0\0" + zlib.compress(b"x" * 99))),
             P.write_png(pimg8, 8, 3, palette=pal8, pre_plte=gama), P.write_png(pimg4, 4, 3, palette=pal4, pre_plte=srgb),
             P.write_png(pimg4, 4, 3, palette=pal4, pre_plte=P.chunk(b"iCCP", b"icc\0\0" + zlib.compress(b"x" * 99)))]
    assert [s for _, s in _decode(files, 0)] == [8] * len(files)
    for f, (img1, st) in zip(files, _decode(files, 1)):
        assert st == 0 and np.array_equal(img1, _host(f, 1))
    # the reason: OpenCV's bytes do change, for colour and for palette files
    assert not np.array_equal(_host(files[0], 0), P.gray(img, 8, 2, 0))
    assert not np.array_equal(_host(files[3], 0), P.gray(pimg8, 8, 3, 0, pal8))
    assert not np.array_equal(_host(files[4], 0), P.gray(pimg4, 4, 3, 0, pal4))


def test_text_pillow_refuses_is_refused_under_pillow_only():
    """Pillow raises on a zTXt, iTXt or iCCP payload that inflates past 1 MiB: rule 1 refuses every compressed payload above
    1016 bytes (DEFLATE inflates a byte to at most 1032) and files whose text may pass Pillow's 64 MiB in all; OpenCV reads
    them, so rule 0 accepts them."""
    img = np.arange(12, dtype=np.uint8).reshape(3, 4)
    bomb = zlib.compress(b"\0" * (2 << 20), 9)
    small = zlib.compress(b"text" * 100)
    many = b"".join(P.chunk(b"zTXt", b"k%d\0\0" % i + bytes(1016)) for i in range(65))   # a bound of 65 MiB, not a real one
    files = [P.write_png(img, 8, 0, extra=P.chunk(b"zTXt", b"k\0\0" + bomb)),
             P.write_png(img, 8, 0, extra=P.chunk(b"iTXt", b"k\0\1\0\0\0" + bomb)),
             P.write_png(img, 8, 0, pre_plte=P.chunk(b"iCCP", b"icc\0\0" + bomb)),
             P.write_png(img, 8, 0, extra=many),
             P.write_png(img, 8, 0, extra=P.chunk(b"zTXt", b"k\0\0" + small) + P.chunk(b"iTXt", b"k\0\1\0\0\0" + small)
                         + P.chunk(b"iTXt", b"k\0\0\0\0\0" + bytes(5000)))]
    for f in files[:3]:
        with pytest.raises(ValueError):
            _host(f, 1)
    assert [s for _, s in _decode(files, 1)] == [8, 8, 8, 8, 0]
    for f, (got, st) in zip(files, _decode(files, 0)):
        assert st == 0 and np.array_equal(got, _host(f, 0)) and np.array_equal(got, img)


# ------------------------------------------------------------------------------------------------ 2. stages
def test_workspace_stages_equal_zlib():
    corpus = _corpus(seed=3)[::7]
    files = [f for _, f in corpus]
    res, ws, ws_offset = _decode(files, 0, keep_ws=True)
    for (name, f), (_, st), r0 in zip(corpus, res, ws_offset[:-1]):
        assert st == 0, name
        stream = b"".join(d for t, d in P.chunks_of(f) if t == b"IDAT")
        zcap = (len(f) + 15) // 16 * 16
        ih = f[16:29]
        h, w = int.from_bytes(ih[4:8], "big"), int.from_bytes(ih[:4], "big")
        raw = P.unfilter(zlib.decompress(stream), h, w, ih[8], ih[9], ih[12])
        assert ws[r0:r0 + len(stream)].tobytes() == stream, name
        assert ws[r0 + zcap:r0 + zcap + len(raw)].tobytes() == raw, name


# ------------------------------------------------------------------------------------------------ 3. malformed files
def _deflate_file(img, bits):
    """A file whose zlib stream is a valid header and the DEFLATE bits written by `bits(BitWriter)`."""
    w = P.BitWriter()
    bits(w)
    return P.file_with_stream(img, 8, 0, b"\x78\x01" + w.bytes() + b"\0\0\0\0")


def _malformed(seed=5):
    """[(name, bytes, expected status)]: one defect per file."""
    rng = np.random.default_rng(seed)
    img = P.random_image(rng, 7, 11, 8, 0)
    good = P.write_png(img, 8, 0, filters="random", rng=rng)
    ch = P.chunks_of(good)
    raw = P.scanlines(img, 8, 0)
    out = []

    def flip_crc(ctype):
        b = bytearray(P.write_png(img, 8, 0, extra=P.chunk(b"tEXt", b"k\0v")))
        pos = 8
        while True:
            n = int.from_bytes(b[pos:pos + 4], "big")
            if b[pos + 4:pos + 8] == ctype:
                b[pos + 8 + n] ^= 1
                return bytes(b)
            pos += 12 + n

    out += [("crc_idat", flip_crc(b"IDAT"), 3), ("crc_text", flip_crc(b"tEXt"), 3), ("crc_ihdr", flip_crc(b"IHDR"), 3)]
    z = P.compress(raw)
    out.append(("zlib_method", P.file_with_stream(img, 8, 0, b"\x77" + z[1:]), 4))
    out.append(("zlib_check", P.file_with_stream(img, 8, 0, z[:1] + bytes([z[1] ^ 1]) + z[2:]), 4))
    out.append(("zlib_dict", P.file_with_stream(img, 8, 0, b"\x78\xbb" + z[2:]), 4))
    out.append(("adler", P.file_with_stream(img, 8, 0, z[:-1] + bytes([z[-1] ^ 0x10])), 4))
    out.append(("zlib_trailing", P.file_with_stream(img, 8, 0, z + b"\0"), 4))
    out.append(("zlib_truncated", P.file_with_stream(img, 8, 0, z[:-6]), 5))
    out.append(("btype3", _deflate_file(img, lambda w: (w.put(1, 1), w.put(3, 2))), 5))
    out.append(("stored_nlen", _deflate_file(img, lambda w: (w.put(1, 1), w.put(0, 2), w.put(0, 5), w.put(5, 16), w.put(5, 16))), 5))

    def oversub(w):                                  # 19 code length codes of length 1
        w.put(1, 1); w.put(2, 2); w.put(0, 5); w.put(0, 5); w.put(15, 4)
        for _ in range(19):
            w.put(1, 3)

    def incomplete(w):                               # two code length codes of length 2
        w.put(1, 1); w.put(2, 2); w.put(0, 5); w.put(0, 5); w.put(0, 4)
        for v in (2, 2, 0, 0):
            w.put(v, 3)

    def dist_past_output(w):                         # fixed block opening with a match: length 3, distance 1
        w.put(1, 1); w.put(1, 2); w.code(1, 7); w.code(0, 5); w.code(0, 7)

    def bad_dist_code(w):                            # a literal, then distance code 30
        w.put(1, 1); w.put(1, 2); w.code(0x30, 8); w.code(1, 7); w.code(30, 5); w.code(0, 7)

    def bad_len_code(w):                             # literal/length code 286
        w.put(1, 1); w.put(1, 2); w.code(0xC6, 8); w.code(0, 7)

    for name, fn in (("oversubscribed", oversub), ("incomplete", incomplete), ("dist_past_output", dist_past_output),
                     ("dist_code_30", bad_dist_code), ("len_code_286", bad_len_code)):
        out.append((name, _deflate_file(img, fn), 5))
    far = P.random_image(rng, 60, 40, 8, 0)                 # repeats 600 bytes back under a declared 512-byte window
    rawfar = P.scanlines(np.tile(far[:15], (4, 1)), 8, 0)
    zfar = P.compress(rawfar, wbits=15)
    zfar = bytes([0x18 | (zfar[0] & 0x0F), 0]) + zfar[2:]
    zfar = zfar[:1] + bytes([(31 - (zfar[0] * 256) % 31) % 31]) + zfar[2:]
    out.append(("dist_past_window", P.file_with_stream(np.tile(far[:15], (4, 1)), 8, 0, zfar), 5))
    out.append(("too_little", P.file_with_stream(img, 8, 0, P.compress(raw[:-1])), 6))
    out.append(("too_much", P.file_with_stream(img, 8, 0, P.compress(raw + b"\0")), 6))
    out.append(("filter5", P.file_with_stream(img, 8, 0, P.compress(b"\x05" + raw[1:])), 7))
    pal = _palette(rng, 8, 4)
    out.append(("palette_index", P.write_png(np.array([[0, 1, 2, 3, 4]], np.uint8), 8, 3, palette=pal), 7))
    ihdr, idat, iend = ch[0], [c for c in ch if c[0] == b"IDAT"], ch[-1]
    out.append(("critical_unknown", P.assemble([ihdr, (b"XXXX", b"hi")] + idat + [iend]), 2))
    zs = P.compress(raw)
    split = [(b"IDAT", zs[:10]), (b"tEXt", b"k\0v"), (b"IDAT", zs[10:])]
    out.append(("idat_not_consecutive", P.assemble([ihdr] + split + [iend]), 2))
    out.append(("no_iend", P.assemble([ihdr] + idat), 2))
    out.append(("after_iend", good + b"\0", 2))
    out.append(("truncated", good[:len(good) // 2], 2))
    out.append(("no_idat", P.assemble([ihdr, iend]), 2))
    out.append(("plte_in_gray", P.assemble([ihdr, (b"PLTE", bytes(6))] + idat + [iend]), 2))
    out.append(("palette_missing", P.file_with_stream(img, 8, 3, P.compress(raw)), 2))
    out.append(("depth3", P.assemble([(b"IHDR", P.ihdr(7, 11, 3, 0))] + idat + [iend]), 1))
    out.append(("signature", b"\x89PNG\r\n\x1a\x0b" + good[8:], 1))
    out.append(("actl", P.assemble([ihdr, (b"acTL", bytes(8))] + idat + [iend]), 8))
    out.append(("exif", P.assemble([ihdr, (b"eXIf", b"MM\0*\0\0\0\x08\0\0")] + idat + [iend]), 8))
    out.append(("gama_size", P.assemble([ihdr, (b"gAMA", bytes(3))] + idat + [iend]), 2))
    return out, good, img


def test_malformed_files_are_flagged_and_neighbours_unchanged():
    bad, good, img = _malformed()
    names = [n for n, _, _ in bad]
    files = [f for _, f, _ in bad]
    from lstm_ctc_ocr_b200 import engine
    # each file's IHDR size where it reads; a file without one gets (7, 11), the size of the image it was made from
    sizes = [engine.png_size(f) or (7, 11) for f in files]
    for rule in (0, 1):
        got = _decode(files, rule, sizes)
        for (name, _, want), (im, st) in zip(bad, got):
            assert st == want, (name, st, want)
            assert not im.any(), name
        # the valid file between malformed ones, at every position: the same bytes as alone
        alone = _decode([good], rule)[0]
        assert alone[1] == 0 and np.array_equal(alone[0], _host(good, rule))
        for pos in (0, 5, len(files)):
            mixed = files[:pos] + [good] + files[pos:]
            res = _decode(mixed, rule, sizes[:pos] + [(7, 11)] + sizes[pos:])
            assert res[pos][1] == 0 and np.array_equal(res[pos][0], alone[0]), pos
            assert [s for _, s in res[:pos] + res[pos + 1:]] == [w for _, _, w in bad]
    # a height unlike the planned one
    assert _decode([good], 0, [(8, 11)])[0][1] == 1
    assert set(names) >= {"crc_idat", "adler", "oversubscribed", "too_little", "palette_index", "after_iend", "exif", "actl"}


def test_repeat_runs_and_orders_are_bit_identical():
    corpus = _corpus(seed=9)[::5]
    files = [f for _, f in corpus]
    a = _decode(files, 1)
    b = _decode(files, 1)
    perm = list(range(len(files)))[::-1]
    c = _decode([files[i] for i in perm], 1)
    for i in range(len(files)):
        assert a[i][1] == b[i][1] == 0 and np.array_equal(a[i][0], b[i][0])
        assert np.array_equal(a[perm[i]][0], c[i][0])


# ------------------------------------------------------------------------------------------------ 4. memory, codes, streams
def test_guarded_buffers_of_the_planned_sizes():
    import bounds as B
    from lstm_ctc_ocr_b200 import _lib, engine
    corpus = _corpus(seed=11)[::9]
    bad, good, _ = _malformed()
    files = [f for _, f in corpus] + [f for n, f, _ in bad if n != "truncated"] + [good[:len(good) // 2]]   # truncated last
    sizes = [engine.png_size(f) or (7, 11) for f in files]
    (d_files, foff, flen, h, w, ooff, wso), ws_bytes, nout, hw, _ = _args(files, sizes)
    ins = [B.input_of(n, a.cpu().numpy()) for n, a in (("files", d_files), ("file_offset", foff), ("file_len", flen), ("h", h),
                                                       ("w", w), ("out_offset", ooff), ("ws_offset", wso))]
    out = B.output_of("out", (nout,), torch.uint8, align=1)
    status = B.output_of("status", (len(files),), torch.int32)
    ws = B.output_of("workspace", (ws_bytes,), torch.uint8, align=1)
    lib = _lib.load()

    def call():
        return lib.crnn_png_decode_gray_u8(ins[0].ptr, ins[1].ptr, ins[2].ptr, len(files), ins[3].ptr, ins[4].ptr, ins[5].ptr, 0,
                                           out.ptr, status.ptr, ws.ptr, ins[6].ptr, ws_bytes, torch.cuda.current_stream().cuda_stream)
    problems, last = B.run_case(call, ins + [out, status, ws])
    assert not problems, problems
    st = last["status"].cpu().numpy()
    assert not st[:len(corpus)].any() and st[-1] == 2


def test_status_codes_and_untouched_outputs():
    from lstm_ctc_ocr_b200 import _lib
    lib = _lib.load()
    files = [f for _, f in _corpus(seed=2)[:3]]
    (d_files, foff, flen, h, w, ooff, wso), ws_bytes, nout, hw, _ = _args(files)
    out = torch.full((nout + 8,), 0xA5, dtype=torch.uint8, device=DEV)
    status = torch.full((8,), -7, dtype=torch.int32, device=DEV)
    ws = torch.empty(ws_bytes + 64, dtype=torch.uint8, device=DEV)
    p = lambda t: t.data_ptr()  # noqa: E731
    base = dict(files=p(d_files), foff=p(foff), flen=p(flen), N=3, h=p(h), w=p(w), ooff=p(ooff), rule=0, out=p(out),
                st=p(status), ws=p(ws), wso=p(wso))
    cases = {"N0": dict(N=0), "Nneg": dict(N=-2), "rule2": dict(rule=2), "rule_neg": dict(rule=-1)}
    for k in base:
        if k not in ("N", "rule"):
            cases[k + "_null"] = {k: 0}
    for k, al in (("foff", 8), ("flen", 8), ("ooff", 8), ("wso", 8), ("h", 4), ("w", 4), ("st", 4)):
        cases[k + "_misaligned"] = {k: base[k] + al // 2}
    for name, c in cases.items():
        a = dict(base, **c)
        s = lib.crnn_png_decode_gray_u8(a["files"], a["foff"], a["flen"], a["N"], a["h"], a["w"], a["ooff"], a["rule"], a["out"],
                                        a["st"], a["ws"], a["wso"], ws_bytes, torch.cuda.current_stream().cuda_stream)
        assert s == 1, (name, s)
    torch.cuda.synchronize()
    assert (out == 0xA5).all() and (status == -7).all()
    # a workspace shorter than the plan: the files beyond it are refused with CRNN_PNG_WORKSPACE and zero slots
    a = base
    assert lib.crnn_png_decode_gray_u8(a["files"], a["foff"], a["flen"], 3, a["h"], a["w"], a["ooff"], 0, a["out"], a["st"], a["ws"],
                                       a["wso"], ws_bytes - 1, torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    st = status[:3].cpu().numpy()
    assert st[2] == 9 and not st[:2].any()
    n2 = int(hw[2, 0] * hw[2, 1])
    assert not out[nout - n2:nout].any()
    with pytest.raises(Exception):
        from lstm_ctc_ocr_b200 import engine
        engine.decode_png_gray(d_files.cpu(), foff, flen, h, w, ooff, wso, 0)


def test_gated_stream_and_graph_replay():
    import test_gpu_streams as SG
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200._lib import check
    corpus = _corpus(seed=13)[::11]
    files = [f for _, f in corpus]
    (s_files, foff, flen, s_h, s_w, ooff, wso), ws_bytes, nout, hw, offs = _args(files)
    d_files, h, w = (torch.empty_like(v) for v in (s_files, s_h, s_w))
    out = torch.empty(nout, dtype=torch.uint8, device=DEV)
    status = torch.empty(len(files), dtype=torch.int32, device=DEV)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)

    def call():
        check(engine._lib.load().crnn_png_decode_gray_u8(d_files.data_ptr(), foff.data_ptr(), flen.data_ptr(), len(files),
                                                         h.data_ptr(), w.data_ptr(), ooff.data_ptr(), 1, out.data_ptr(),
                                                         status.data_ptr(), ws.data_ptr(), wso.data_ptr(), ws_bytes, engine._stream()))
        return {"out": out.clone(), "status": status.clone()}
    got = SG._gated("png_decode_gray_u8", call, [(d_files, s_files), (h, s_h), (w, s_w)], [out, status])
    o = got["out"].cpu().numpy()
    assert not got["status"].cpu().numpy().any()
    for i, f in enumerate(files):
        assert np.array_equal(o[offs[i]:offs[i] + hw[i, 0] * hw[i, 1]].reshape(hw[i]), _host(f, 1)), corpus[i][0]
    # graph capture and replay
    d_files.copy_(s_files), h.copy_(s_h), w.copy_(s_w)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            engine.decode_png_gray(d_files, foff, flen, h, w, ooff, wso, 1, out=out, workspace=ws, status=status)
    torch.cuda.current_stream().wait_stream(s)
    out.fill_(0xA5)
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), o) and not status.cpu().numpy().any()


# ------------------------------------------------------------------------------------------------ 5. Session and test_model
def _weights():
    import test_gpu_packed_eval as PE
    return PE._load("make_decode10k", "tests", "golden", "make_decode10k.py").load_weights()


def test_session_bytes_arrays_and_mixed_feeds_are_bit_identical(monkeypatch):
    from lstm_ctc_ocr_b200.lib.lstm.test import gray_rule
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.session import Session
    from lstm_ctc_ocr_b200 import engine
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    files = [f for _, f in _rendered(40, seed=3)] + [f for n, f in _corpus(seed=6) if n.startswith(("pil_", "cv2_gray_l6"))]
    arrays = [_host(f, gray_rule()) for f in files]
    mixed = [f if i % 2 else a for i, (f, a) in enumerate(zip(files, arrays))]
    net = get_network("LSTM_test")
    with Session(device=DEV) as sess:
        sess.assign(net, _weights())
        fetches = [Fetch(net, k) for k in ("logits", "dense_decoded")]
        ref = sess.run(fetches, {net.images: arrays, net.keep_prob: 1.0})
        for feed in (files, mixed):
            got = sess.run(fetches, {net.images: feed, net.keep_prob: 1.0})
            for a, b in zip(ref, got):
                assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
        got = sess.run(fetches, {net.images: files, net.keep_prob: 1.0})
        # the encoded bytes, and per line its offset, sizes and time steps, and its file's offsets, length and plan entry
        assert sess.h2d_bytes == sum(len(f) for f in files) + 68 * len(files) + 8
        bad, good, _ = _malformed()
        with pytest.raises(engine.PngDecodeError) as e:
            sess.run(fetches, {net.images: [good, bad[0][1], arrays[0], bad[1][1]], net.keep_prob: 1.0})
        assert e.value.entries == [1, 3]


def _write_eval_dir(path, seed=17):
    """Rendered lines as PNG of every kind, a JPEG, and PNGs the device refuses but the host reads."""
    import cv2
    from PIL import Image
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    r = random.Random(seed)
    rng = np.random.default_rng(seed)
    font = gen.embedded_font(42)
    k = 0
    for i in range(36):
        text = gen.gen_rand(r, 4, 20)
        im = gen.render_line(text, rng=r, font=font)
        name = os.path.join(path, f"{k:04d}_{text}")
        k += 1
        kind = i % 9
        if kind == 0:
            Image.fromarray(im).save(name + ".png")
        elif kind == 1:
            Image.fromarray(im).convert("RGB").save(name + ".png", optimize=True)
        elif kind == 2:
            cv2.imwrite(name + ".png", im, [cv2.IMWRITE_PNG_COMPRESSION, 9])
        elif kind == 3:
            open(name + ".png", "wb").write(P.write_png(im, 8, 0, interlace=1, filters="random", rng=rng))
        elif kind == 4:
            open(name + ".png", "wb").write(P.write_png((im.astype(np.uint16) * 257), 16, 0, filters=4))
        elif kind == 5:
            cv2.imwrite(name + ".jpg", im)
        elif kind == 6:                                        # gAMA on colour: refused under rule 0, read under rule 1
            rgb = np.stack([im, im, im // 2], -1)
            open(name + ".png", "wb").write(P.write_png(rgb, 8, 2, extra=P.chunk(b"gAMA", (45455).to_bytes(4, "big"))))
        elif kind == 7:                                        # a bad IDAT CRC: the host reads it (Pillow), the device refuses it
            b = bytearray(P.write_png(im, 8, 0))
            b[-13] ^= 1
            open(name + ".png", "wb").write(bytes(b))
        else:
            open(name + ".png", "wb").write(P.write_png(im, 8, 0, level=1, split=64, zero_chunks=True))


@pytest.mark.parametrize("opencv", [True, False])
def test_test_model_output_equals_the_host_path(opencv, tmp_path, monkeypatch):
    import test_gpu_resize as RZ
    from lstm_ctc_ocr_b200.lib.lstm import test as T
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    _write_eval_dir(str(tmp_path))
    if not opencv:
        monkeypatch.setitem(sys.modules, "cv2", None)          # `import cv2` raises: load_line_image and the decoder use Pillow
    assert T.gray_rule() == (0 if opencv else 1)
    strip = lambda text: [ln.split(" cost time")[0] if "cost time" in ln else ln for ln in text.splitlines()]  # noqa: E731
    old = cfg.TEST.BATCH_SIZE
    try:
        for bs in (1, 16):
            cfg.TEST.BATCH_SIZE = bs
            net = get_network("LSTM_test")
            with Session(device=DEV) as sess:
                sess.assign(net, _weights())
                sw = T.SolverWrapper(sess, net, None, str(tmp_path), None)
                new, host = io.StringIO(), io.StringIO()
                with redirect_stdout(new):
                    r_new = sw.test_model(sess, testDir=str(tmp_path), restore=False)
                with redirect_stdout(host):
                    r_host = RZ._host_test_model(sess, net, str(tmp_path), bs)
            assert r_new == r_host and r_new[1] == 36
            assert strip(new.getvalue()) == strip(host.getvalue()), bs
    finally:
        cfg.TEST.BATCH_SIZE = old


def _eval_images():
    """The 67 evaluation lines of test_gpu_width_edges._eval_inputs at their native size: 64 rendered lines of 30 - 70
    characters and crops 8, 9 and 12 px wide of a 32-high line."""
    from PIL import Image
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    rng = random.Random(4242)
    texts, imgs = [], []
    for _ in range(64):
        texts.append(gen.gen_rand(rng, 30, 70))
        imgs.append(gen.render_line(texts[-1], rng=rng))
    h32 = np.asarray(Image.fromarray(imgs[0]).resize((int(32 / imgs[0].shape[0] * imgs[0].shape[1]), 32), Image.BILINEAR),
                     dtype=np.uint8)
    return texts + ["crop"] * 3, imgs + [np.ascontiguousarray(h32[:, 40:40 + w]) for w in (8, 9, 12)]


def _fixture_images():
    """The decode-10k fixture's 10 240 rendered lines (tests/golden/make_decode10k.py) as 8-bit gray 32-row images."""
    import test_gpu_packed_eval as PE
    from lstm_ctc_ocr_b200.lib.lstm.test import decodeRes
    mk = PE._load("make_decode10k", "tests", "golden", "make_decode10k.py")
    s = mk.sampler()
    texts, imgs = [], []
    for k in range(mk.NBATCH):
        data, lab, ll, _ = s.batch(k)
        ends = np.cumsum(ll)
        for i, d in enumerate(data):
            imgs.append(np.ascontiguousarray(np.rint(np.asarray(d, np.float64) * 255).astype(np.uint8).T))
            texts.append("".join(decodeRes(lab[ends[i] - ll[i]:ends[i]])))
    return texts, imgs


@pytest.mark.parametrize("which", ["eval67", "fixture10k"])
def test_test_model_on_saved_evaluation_lines_equals_the_host_path(which, tmp_path, monkeypatch):
    """The 67 evaluation lines and the 10 240 fixture lines saved as PNG by Pillow: test_model's reads and accuracy equal the host
    path's on every line."""
    from PIL import Image
    import test_gpu_resize as RZ
    from lstm_ctc_ocr_b200.lib.lstm import test as T
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    texts, imgs = _eval_images() if which == "eval67" else _fixture_images()
    for i, (t, im) in enumerate(zip(texts, imgs)):
        Image.fromarray(im).save(os.path.join(str(tmp_path), f"{i:05d}_{t}.png"))
    strip = lambda text: [ln.split(" cost time")[0] if "cost time" in ln else ln for ln in text.splitlines()]  # noqa: E731
    old = cfg.TEST.BATCH_SIZE
    try:
        cfg.TEST.BATCH_SIZE = 64 if which == "eval67" else 256
        net = get_network("LSTM_test")
        with Session(device=DEV) as sess:
            sess.assign(net, _weights())
            sw = T.SolverWrapper(sess, net, None, str(tmp_path), None)
            new, host = io.StringIO(), io.StringIO()
            with redirect_stdout(new):
                r_new = sw.test_model(sess, testDir=str(tmp_path), restore=False)
            with redirect_stdout(host):
                r_host = RZ._host_test_model(sess, net, str(tmp_path), cfg.TEST.BATCH_SIZE)
        assert r_new == r_host and r_new[1] == len(imgs)
        assert strip(new.getvalue()) == strip(host.getvalue())
    finally:
        cfg.TEST.BATCH_SIZE = old
