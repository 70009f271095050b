"""PNG files written from scratch for the device decoder's tests (crnn_png_decode_gray_u8), and the two gray rules restated.

``write_png`` builds any valid file: every colour type and bit depth, Adam7, a filter per row (forced or drawn), any zlib level,
strategy and window, the IDAT stream split as asked, extra chunks placed before the first IDAT.  ``gray`` restates what the host
readers return for a decoded image: rule 0 is ``cv2.imread(path, 0)`` (OpenCV 4.13 on libpng 1.6), rule 1 Pillow's
``convert("L")``; tests/test_png_cpu.py pins both against the installed readers."""
import struct
import zlib

import numpy as np

SIG = b"\x89PNG\r\n\x1a\n"
DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
ADAM7 = ((0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2))


def chunk(ctype, data):
    return struct.pack(">I", len(data)) + ctype + data + struct.pack(">I", zlib.crc32(ctype + data) & 0xFFFFFFFF)


def ihdr(h, w, depth, ctype, interlace=0):
    return struct.pack(">IIBBBBB", w, h, depth, ctype, 0, 0, interlace)


def passes(h, w, interlace):
    """(y0, x0, dy, dx, ph, pw) of each non-empty pass."""
    if not interlace:
        return [(0, 0, 1, 1, h, w)]
    out = []
    for x0, y0, dx, dy in ADAM7:
        pw, ph = (w - x0 + dx - 1) // dx, (h - y0 + dy - 1) // dy
        if pw > 0 and ph > 0:
            out.append((y0, x0, dy, dx, ph, pw))
    return out


def row_bytes(pw, depth, ctype):
    return (pw * CHANNELS[ctype] * depth + 7) // 8


def raw_len(h, w, depth, ctype, interlace):
    """Bytes of the inflated (still filtered) scanlines: a filter byte and the packed samples per row of each non-empty pass."""
    return sum(ph * (1 + row_bytes(pw, depth, ctype)) for _, _, _, _, ph, pw in passes(h, w, interlace))


def _pack(samples, depth):
    """[rows, n] unsigned samples -> [rows, rowbytes] bytes, big-endian, MSB first below 8 bits."""
    samples = np.asarray(samples)
    if depth == 16:
        return samples.astype(">u2").view(np.uint8).reshape(samples.shape[0], -1)
    if depth == 8:
        return samples.astype(np.uint8)
    per = 8 // depth
    n = samples.shape[1]
    pad = (-n) % per
    s = np.concatenate([samples, np.zeros((samples.shape[0], pad), samples.dtype)], 1).astype(np.uint16)
    s = s.reshape(samples.shape[0], -1, per)
    out = np.zeros(s.shape[:2], np.uint16)
    for k in range(per):
        out |= s[:, :, k] << (8 - depth * (k + 1))
    return out.astype(np.uint8)


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return a if pa <= pb and pa <= pc else (b if pb <= pc else c)


def _filter_row(ftype, row, prior, bpp):
    row = row.astype(np.int32)
    prior = prior.astype(np.int32)
    left = np.concatenate([np.zeros(bpp, np.int32), row[:-bpp]]) if row.size else row
    upleft = np.concatenate([np.zeros(bpp, np.int32), prior[:-bpp]]) if row.size else row
    if ftype == 0:
        pred = np.zeros_like(row)
    elif ftype == 1:
        pred = left
    elif ftype == 2:
        pred = prior
    elif ftype == 3:
        pred = (left + prior) >> 1
    else:
        p = left + prior - upleft
        pa, pb, pc = np.abs(p - left), np.abs(p - prior), np.abs(p - upleft)
        pred = np.where((pa <= pb) & (pa <= pc), left, np.where(pb <= pc, prior, upleft))
    return ((row - pred) & 0xFF).astype(np.uint8)


def scanlines(img, depth, ctype, interlace=0, filters=None, rng=None):
    """The filtered scanlines of `img` ([h, w] or [h, w, c] samples): `filters` None (all 0), an int (every row) or "random"."""
    img = np.asarray(img)
    if img.ndim == 2:
        img = img[:, :, None]
    h, w, c = img.shape
    bpp = max(1, c * depth // 8)
    out = []
    for y0, x0, dy, dx, ph, pw in passes(h, w, interlace):
        sub = img[y0::dy, x0::dx][:ph, :pw].reshape(ph, pw * c)
        packed = _pack(sub, depth)
        prior = np.zeros(packed.shape[1], np.uint8)
        for r in range(ph):
            f = (filters if isinstance(filters, int) else int(rng.integers(0, 5)) if filters == "random" else 0)
            out.append(bytes([f]) + _filter_row(f, packed[r], prior, bpp).tobytes())
            prior = packed[r]
    return b"".join(out)


def compress(raw, level=6, wbits=15, strategy=zlib.Z_DEFAULT_STRATEGY, memlevel=8):
    co = zlib.compressobj(level, zlib.DEFLATED, wbits, memlevel, strategy)
    return co.compress(raw) + co.flush()


def split_idat(stream, split=None, zero_chunks=False):
    """The IDAT chunks of `stream`: one chunk (split None), chunks of `split` bytes, zero-length chunks between them if asked."""
    if split is None:
        parts = [stream]
    else:
        parts = [stream[i:i + split] for i in range(0, len(stream), split)] or [b""]
    out = b""
    for k, p in enumerate(parts):
        if zero_chunks:
            out += chunk(b"IDAT", b"")
        out += chunk(b"IDAT", p)
    if zero_chunks:
        out += chunk(b"IDAT", b"")
    return out


def write_png(img, depth, ctype, interlace=0, palette=None, filters=None, rng=None, level=6, wbits=15,
              strategy=zlib.Z_DEFAULT_STRATEGY, split=None, zero_chunks=False, extra=b"", pre_plte=b""):
    """A valid PNG file of `img` (samples, not bytes).  `palette`: [n, 3] uint8 for colour type 3.  `pre_plte`: whole chunks put
    right after IHDR, where the PNG specification places the colour-space chunks (gAMA, cHRM, sRGB, iCCP, sBIT) -- libpng ignores
    those after PLTE.  `extra`: whole chunks put after PLTE and before the first IDAT."""
    h, w = img.shape[:2]
    out = SIG + chunk(b"IHDR", ihdr(h, w, depth, ctype, interlace)) + pre_plte
    if ctype == 3:
        out += chunk(b"PLTE", np.asarray(palette, np.uint8).tobytes())
    out += extra
    raw = scanlines(img, depth, ctype, interlace, filters, rng)
    out += split_idat(compress(raw, level, wbits, strategy), split, zero_chunks)
    return out + chunk(b"IEND", b"")


def random_image(rng, h, w, depth, ctype, palette_len=None):
    """Random samples for (depth, ctype); palette indices stay below palette_len."""
    c = CHANNELS[ctype]
    hi = (palette_len if ctype == 3 else 1 << depth)
    img = rng.integers(0, hi, size=(h, w, c) if c > 1 else (h, w), dtype=np.int64)
    return img.astype(np.uint16 if depth == 16 else np.uint8)


def gray(img, depth, ctype, rule, palette=None):
    """The [h, w] uint8 the host reader gives for samples `img` (rule 0: cv2.imread(path, 0); rule 1: Pillow convert("L"))."""
    img = np.asarray(img).astype(np.int64)
    if ctype == 3:
        img = np.asarray(palette, np.int64)[img]
        depth = 8
    if ctype in (0, 4):
        g = img if ctype == 0 else img[:, :, 0]
        if depth < 8:
            return (g * 255 // ((1 << depth) - 1)).astype(np.uint8)
        if depth == 16:
            return (g >> 8 if rule == 0 else np.minimum(g, 255) if ctype == 0 else g >> 8).astype(np.uint8)
        return g.astype(np.uint8)
    r, g_, b = img[:, :, 0], img[:, :, 1], img[:, :, 2]
    if depth == 16:
        if rule == 0:
            return (((9797 * r + 19234 * g_ + 3737 * b + 16384) >> 15) >> 8).astype(np.uint8)
        r, g_, b = r >> 8, g_ >> 8, b >> 8
    if rule == 0:
        return ((9797 * r + 19234 * g_ + 3737 * b) >> 15).astype(np.uint8)
    return ((19595 * r + 38470 * g_ + 7471 * b + 0x8000) >> 16).astype(np.uint8)


class BitWriter:
    """DEFLATE bits, least significant first; Huffman codes are given MSB first and reversed here."""

    def __init__(self):
        self.bits = []

    def put(self, value, n):
        self.bits += [(value >> k) & 1 for k in range(n)]

    def code(self, value, n):
        self.bits += [(value >> (n - 1 - k)) & 1 for k in range(n)]

    def bytes(self):
        b = self.bits + [0] * (-len(self.bits) % 8)
        return bytes(sum(b[i + k] << k for k in range(8)) for i in range(0, len(b), 8))


def file_with_stream(img, depth, ctype, stream):
    """A file of img's IHDR whose IDAT holds `stream` (any bytes)."""
    h, w = img.shape[:2]
    return (SIG + chunk(b"IHDR", ihdr(h, w, depth, ctype)) + chunk(b"IDAT", stream) + chunk(b"IEND", b""))


def chunks_of(data):
    """[(type, payload)] of a file."""
    out, pos = [], 8
    while pos + 12 <= len(data):
        n = struct.unpack(">I", data[pos:pos + 4])[0]
        out.append((data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]))
        pos += 12 + n
    return out


def assemble(chunks):
    return SIG + b"".join(chunk(t, d) for t, d in chunks)


def unfilter(raw, h, w, depth, ctype, interlace):
    """The inflated scanlines `raw` with each row's filter undone, filter bytes kept: what the decoder leaves in a file's
    scanline region of the workspace."""
    out = bytearray(raw)
    bpp = max(1, CHANNELS[ctype] * depth // 8)
    pos = 0
    for _, _, _, _, ph, pw in passes(h, w, interlace):
        rb = row_bytes(pw, depth, ctype)
        prior = [0] * rb
        for _ in range(ph):
            f, x = out[pos], out[pos + 1:pos + 1 + rb]
            for k in range(rb):
                a = x[k - bpp] if k >= bpp else 0
                c = prior[k - bpp] if k >= bpp else 0
                pred = (0, a, prior[k], (a + prior[k]) >> 1, _paeth(a, prior[k], c))[f]
                x[k] = (x[k] + pred) & 0xFF
            out[pos + 1:pos + 1 + rb] = x
            prior = list(x)
            pos += 1 + rb
    return bytes(out)
