"""A host restatement of the device JPEG decoder (csrc/jpeg.cu), used only by tests, and a small baseline JPEG writer.

decode(data, rule) -> (gray image, info): marker walk, canonical Huffman decode, libjpeg-turbo's jidctint.c (ISLOW) with the
range-limit table, the envelope where it agrees with libjpeg-turbo's SIMD IDCT, fancy upsampling, jdcolor.c's tables and L24.
It reads the files the device reads and raises Refused(status) on the rest it is asked about.

encode(blocks, ...) encodes given quantised coefficient blocks with given DQT / DHT / DRI, for files neither host writer
makes: extreme coefficients, custom tables, fill bytes, broken restart markers and each malformed class."""
import numpy as np

NATURAL = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
                    21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53,
                    60, 61, 54, 47, 55, 62, 63])
ENVELOPE = 16383
OK, BAD_HEADER, UNSUPPORTED, BAD_MARKER, BAD_HUFFMAN, BAD_DATA, BAD_RESTART, HOST_DIFFERS, WORKSPACE = range(9)

# ITU T.81 Annex K tables: (bits[1..16], values)
STD_DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
STD_DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
STD_AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], bytes.fromhex(
    "01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a3435363738393a"
    "434445464748494a535455565758595a636465666768696a737475767778797a838485868788898a92939495969798999aa2a3a4a5a6a7a8a9"
    "aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9eaf1f2f3f4f5f6f7f8f9fa"))
STD_AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], bytes.fromhex(
    "000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f11718191a262728292a35363738"
    "393a434445464748494a535455565758595a636465666768696a737475767778797a82838485868788898a92939495969798999aa2a3a4a5"
    "a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7e8e9eaf2f3f4f5f6f7f8f9fa"))


class Refused(Exception):
    def __init__(self, status, why=""):
        super().__init__(f"status {status}: {why}")
        self.status = status


def canonical_codes(bits, vals):
    """{symbol: (code, length)} of a DHT table, or Refused(BAD_HUFFMAN) where libjpeg's jpeg_make_d_derived_tbl refuses it."""
    out, code, p = {}, 0, 0
    for l in range(1, 17):
        for _ in range(bits[l - 1]):
            if code + 1 >= 1 << l:
                raise Refused(BAD_HUFFMAN, "over-subscribed")
            out.setdefault(vals[p], (code, l))
            code += 1
            p += 1
        code <<= 1
    return out


# ------------------------------------------------------------------------------------------------ IDCT
FIX = dict(c0298=2446, c0390=3196, c0541=4433, c0765=6270, c0899=7373, c1175=9633, c1501=12299, c1847=15137, c1961=16069,
           c2053=16819, c2562=20995, c3072=25172)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _islow_1d(v):
    """jidctint.c's butterflies on v[..., 0..7] (int64) -> the 8 sums before the descale."""
    z2, z3 = v[..., 2], v[..., 6]
    z1 = (z2 + z3) * FIX["c0541"]
    tmp2, tmp3 = z1 - z3 * FIX["c1847"], z1 + z2 * FIX["c0765"]
    z2, z3 = v[..., 0], v[..., 4]
    tmp0, tmp1 = (z2 + z3) << 13, (z2 - z3) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    tmp0, tmp1, tmp2, tmp3 = v[..., 7], v[..., 5], v[..., 3], v[..., 1]
    z1, z2, z3, z4 = tmp0 + tmp3, tmp1 + tmp2, tmp0 + tmp2, tmp1 + tmp3
    z5 = (z3 + z4) * FIX["c1175"]
    tmp0, tmp1, tmp2, tmp3 = tmp0 * FIX["c0298"], tmp1 * FIX["c2053"], tmp2 * FIX["c3072"], tmp3 * FIX["c1501"]
    z1, z2 = -z1 * FIX["c0899"], -z2 * FIX["c2562"]
    z3, z4 = -z3 * FIX["c1961"] + z5, -z4 * FIX["c0390"] + z5
    tmp0, tmp1, tmp2, tmp3 = tmp0 + z1 + z3, tmp1 + z2 + z4, tmp2 + z2 + z3, tmp3 + z1 + z4
    return np.stack([t10 + tmp3, t11 + tmp2, t12 + tmp1, t13 + tmp0, t13 - tmp0, t12 - tmp1, t11 - tmp2, t10 - tmp3], -1)


def range_limit(x):
    """IDCT_range_limit[x & RANGE_MASK]: the post-IDCT half of jdmaster.c's sample_range_limit table."""
    k = np.asarray(x, np.int64) & 1023
    return np.where(k < 128, k + 128, np.where(k < 512, 255, np.where(k < 896, 0, k - 896))).astype(np.uint8)


def idct_islow(coef, q, shortcut=True):
    """coef [n, 64] int16 (natural order), q [64] -> (pixels [n, 8, 8] uint8, inside [n] bool: the block lies in the envelope
    where jidctint.c and the SIMD IDCT agree).  shortcut=False skips jidctint.c's zero-AC column and row shortcuts."""
    c = np.asarray(coef, np.int64).reshape(-1, 8, 8)                     # [n, row, col]
    dq = c * np.asarray(q, np.int64).reshape(8, 8)
    cols = np.swapaxes(dq, 1, 2)                                         # [n, col, row]
    ws = _descale(_islow_1d(cols), 11)
    if shortcut:
        zero = ~np.any(np.swapaxes(c, 1, 2)[:, :, 1:], -1)
        ws = np.where(zero[..., None], cols[..., :1] << 2, ws)
    ws = np.swapaxes(ws, 1, 2)                                           # [n, row, col]
    out = _descale(_islow_1d(ws), 18)
    if shortcut:
        zero = ~np.any(ws[:, :, 1:], -1)
        out = np.where(zero[..., None], _descale(ws[:, :, :1], 5), out)
    inside = (np.abs(dq).max((1, 2)) <= ENVELOPE) & (np.abs(ws).max((1, 2)) <= ENVELOPE) & (out.min((1, 2)) >= -512) & \
        (out.max((1, 2)) <= 511)
    return range_limit(out), inside


# ------------------------------------------------------------------------------------------------ parsing and entropy decoding
def _segments(data):
    """[(marker, payload, position)] from SOI through SOS, then the scan's entropy-coded bytes up to EOI."""
    if data[:2] != b"\xff\xd8":
        raise Refused(BAD_HEADER, "no SOI")
    pos, segs = 2, []
    while True:
        if pos >= len(data) or data[pos] != 0xFF:
            raise Refused(BAD_MARKER, "no marker")
        while pos < len(data) and data[pos] == 0xFF:
            pos += 1
        if pos + 3 > len(data):
            raise Refused(BAD_MARKER, "truncated")
        m = data[pos]
        if m in (0, 1) or 0xD0 <= m <= 0xD9:
            raise Refused(BAD_MARKER, "marker without a segment")
        n = int.from_bytes(data[pos + 1:pos + 3], "big")
        if n < 2 or pos + 1 + n > len(data):
            raise Refused(BAD_MARKER, "segment length")
        segs.append((m, data[pos + 3:pos + 1 + n], pos + 3))
        pos += 1 + n
        if m == 0xDA:
            return segs, pos


def _exif_turns(d):
    if d[:6] != b"Exif\0\0":
        return False
    t = d[6:]
    if len(t) < 8 or t[:2] not in (b"II", b"MM"):
        return True
    bo = "little" if t[:2] == b"II" else "big"
    u16 = lambda o: int.from_bytes(t[o:o + 2], bo)   # noqa: E731
    ifd = int.from_bytes(t[4:8], bo)
    if ifd + 2 > len(t):
        return True
    cnt = u16(ifd)
    if ifd + 2 + 12 * cnt > len(t):
        return True
    for j in range(cnt):
        e = ifd + 2 + 12 * j
        if u16(e) == 0x0112:
            return u16(e + 2) != 3 or u16(e + 8) != 1
    return False


def parse(data, rule):
    """The header as the device reads it: dict(frame, scan, tables, restart interval, scan start), or Refused."""
    segs, scan_start = _segments(data)
    frame, dht, dqt, ri, jfif, adobe, turns = None, {}, {}, 0, False, None, False
    for m, d, _ in segs:
        if m in (0xC0, 0xC1):
            if frame is not None:
                raise Refused(BAD_MARKER, "second SOF")
            if len(d) < 6 or d[5] == 0 or len(d) != 6 + 3 * d[5]:
                raise Refused(BAD_HEADER, "SOF length")
            nf = d[5]
            if d[0] != 8 or int.from_bytes(d[1:3], "big") == 0 or nf not in (1, 3):
                raise Refused(UNSUPPORTED, "precision / DNL / components")
            comps = [(d[6 + 3 * c], d[7 + 3 * c] >> 4, d[7 + 3 * c] & 15, d[8 + 3 * c]) for c in range(nf)]
            if any(not (1 <= H <= 4 and 1 <= V <= 4 and tq <= 3) for _, H, V, tq in comps) or len({c[0] for c in comps}) < nf:
                raise Refused(BAD_HEADER, "SOF components")
            if nf == 3 and sum(H * V for _, H, V, _ in comps) > 10:
                raise Refused(BAD_HEADER, "blocks per MCU")
            frame = dict(h=int.from_bytes(d[1:3], "big"), w=int.from_bytes(d[3:5], "big"), comps=comps, sof=bytes(d))
        elif 0xC2 <= m <= 0xCF and m != 0xC4:
            raise Refused(UNSUPPORTED, "process")
        elif m == 0xC4:
            k = 0
            while k < len(d):
                if k + 17 > len(d):
                    raise Refused(BAD_MARKER, "DHT length")
                tc, th = d[k] >> 4, d[k] & 15
                bits = list(d[k + 1:k + 17])
                if tc > 1 or th > 3 or sum(bits) > 256 or k + 17 + sum(bits) > len(d):
                    raise Refused(BAD_HUFFMAN, "DHT")
                dht[(tc, th)] = (bits, list(d[k + 17:k + 17 + sum(bits)]))
                k += 17 + sum(bits)
        elif m == 0xDB:
            k = 0
            while k < len(d):
                pq, tq = d[k] >> 4, d[k] & 15
                if pq > 1 or tq > 3 or k + 1 + 64 * (pq + 1) > len(d):
                    raise Refused(BAD_MARKER, "DQT")
                raw = d[k + 1:k + 1 + 64 * (pq + 1)]
                vals = np.frombuffer(raw, ">u2" if pq else np.uint8).astype(np.int64)
                q = np.zeros(64, np.int64)
                q[NATURAL] = vals
                dqt[tq] = q
                k += 1 + 64 * (pq + 1)
        elif m == 0xDD:
            if len(d) != 2:
                raise Refused(BAD_MARKER, "DRI")
            ri = int.from_bytes(d, "big")
        elif m == 0xDA:
            if frame is None:
                raise Refused(BAD_HEADER, "SOS before SOF")
            nf, ns = len(frame["comps"]), d[0] if d else 0
            if not 1 <= ns <= nf or len(d) != 1 + 2 * ns + 3:
                raise Refused(BAD_MARKER, "SOS length")
            if ns < nf:
                raise Refused(UNSUPPORTED, "several scans")
            ids = [c[0] for c in frame["comps"]]
            scan = []
            for s in range(ns):
                if d[1 + 2 * s] not in ids or ids.index(d[1 + 2 * s]) in [c for c, _, _ in scan]:
                    raise Refused(BAD_MARKER, "scan component")
                td, ta = d[2 + 2 * s] >> 4, d[2 + 2 * s] & 15
                if td > 3 or ta > 3 or (0, td) not in dht or (1, ta) not in dht:
                    raise Refused(BAD_MARKER, "scan tables")
                scan.append((ids.index(d[1 + 2 * s]), td, ta))
            if tuple(d[1 + 2 * ns:]) != (0, 63, 0):
                raise Refused(BAD_MARKER, "spectral selection")
            if any(c[3] not in dqt for c in frame["comps"]):
                raise Refused(BAD_MARKER, "no DQT")
            if nf == 3 and not jfif and ((adobe != 1) if adobe is not None else ids == [82, 71, 66]):
                raise Refused(UNSUPPORTED, "RGB")
            if rule == 0 and turns:
                raise Refused(HOST_DIFFERS, "Exif orientation")
            return dict(frame=frame, scan=scan, dht=dht, dqt=dqt, ri=ri, start=scan_start)
        elif m == 0xE0:
            jfif |= len(d) >= 14 and d[:5] == b"JFIF\0"
        elif m == 0xEE:
            if len(d) >= 12 and d[:5] == b"Adobe":
                adobe = d[11]
        elif m == 0xE1:
            turns |= _exif_turns(d)
        elif not (0xE2 <= m <= 0xEF or m == 0xFE):
            raise Refused(BAD_MARKER, "marker")


def geometry(frame, rule):
    """Per component (H, V, block columns, block rows, samples wide, samples high) and (mcux, mcuy), as csrc/jpeg.cu lays them."""
    comps = frame["comps"]
    if len(comps) == 1:
        comps = [(comps[0][0], 1, 1, comps[0][3])]
    hmax, vmax = max(c[1] for c in comps), max(c[2] for c in comps)
    mcux, mcuy = -(-frame["w"] // (8 * hmax)), -(-frame["h"] // (8 * vmax))
    geo = [(H, V, mcux * H, mcuy * V, -(-frame["w"] * H // hmax), -(-frame["h"] * V // vmax)) for _, H, V, _ in comps]
    return geo, hmax, vmax, mcux, mcuy


class _Bits:
    """A restart segment's bits: 16-bit windows at every bit position (zeros past the data)."""

    def __init__(self, raw):
        bits = np.unpackbits(np.frombuffer(bytes(raw) + bytes(260), np.uint8)).astype(np.int64)
        self.n = 8 * len(raw)
        k = np.arange(16)
        idx = np.arange(self.n + 2048)[:, None] + k       # a block reads at most 64 x 27 bits past the data
        self.win = (bits[idx] << (15 - k)).sum(1)
        self.p = 0

    def get(self, s):
        v = int(self.win[self.p]) >> (16 - s)
        self.p += s
        return v


def _lut(bits, vals, dc):
    codes = canonical_codes(bits, vals)
    if dc and any(v > 15 for v in vals):
        raise Refused(BAD_HUFFMAN, "DC symbol")
    ln = np.zeros(1 << 16, np.int64)
    sym = np.zeros(1 << 16, np.int64)
    for s, (c, l) in codes.items():
        ln[c << (16 - l):(c + 1) << (16 - l)] = l
        sym[c << (16 - l):(c + 1) << (16 - l)] = s
    return ln, sym


def _split_scan(data, start, nseg):
    """The entropy-coded segments (unstuffed) between start and EOI, checked as the device checks its RSTn markers."""
    segs, pos, k, cur = [], start, 0, bytearray()
    while True:
        if pos + 1 >= len(data):
            raise Refused(BAD_MARKER, "no EOI")
        b = data[pos]
        if b != 0xFF:
            cur.append(b)
            pos += 1
            continue
        c = data[pos + 1]
        if c == 0:
            cur.append(0xFF)
            pos += 2
            continue
        if c == 0xFF:                      # fill bytes: the data ends; only more fill may follow before the marker
            q = pos
            while q < len(data) and data[q] == 0xFF:
                q += 1
            if q >= len(data) or data[q] == 0:
                raise Refused(BAD_DATA, "FF FF 00")
            pos = q - 1
            continue
        if 0xD0 <= c <= 0xD7:
            if c != 0xD0 + (k & 7) or k + 1 >= nseg:
                raise Refused(BAD_RESTART, "RSTn")
            k += 1
            segs.append(bytes(cur))
            cur = bytearray()
            pos += 2
            continue
        if c == 0xD9:
            segs.append(bytes(cur))
            if k != nseg - 1:
                raise Refused(BAD_RESTART, "missing RSTn")
            return segs
        raise Refused(UNSUPPORTED if c in (0xDA, 0xDC) else BAD_MARKER, "marker in the scan")


def extend(v, s):
    return v - (1 << s) + 1 if v < 1 << (s - 1) else v


def coefficients(data, rule):
    """(header, geometry, [coefficient array [bh, bw, 64] int16 per frame component]) -- every component is decoded."""
    hd = parse(data, rule)
    fr = hd["frame"]
    geo, hmax, vmax, mcux, mcuy = geometry(fr, rule)
    nf = len(geo)
    if nf == 3:
        if rule == 0 and (geo[0][0] != hmax or geo[0][1] != vmax):
            raise Refused(HOST_DIFFERS, "Y upsampled")
        if rule == 1 and any(hmax % H or vmax % V or hmax // H > 2 or vmax // V > 2 for H, V, *_ in geo):
            raise Refused(HOST_DIFFERS, "sampling ratio")
    mcus = mcux * mcuy
    ri = min(hd["ri"], mcus) if hd["ri"] else mcus
    nseg = -(-mcus // ri)
    luts = {}
    for ci, td, ta in hd["scan"]:
        luts.setdefault((0, td), _lut(*hd["dht"][(0, td)], True))
        luts.setdefault((1, ta), _lut(*hd["dht"][(1, ta)], False))
    segs = _split_scan(data, hd["start"], nseg)
    coef = [np.zeros((g[3], g[2], 64), np.int16) for g in geo]
    for s, raw in enumerate(segs):
        br = _Bits(raw)
        pred = [0] * 3
        for m in range(s * ri, min(mcus, (s + 1) * ri)):
            mx, my = m % mcux, m // mcux
            for sc, (ci, td, ta) in enumerate(hd["scan"]):
                H, V = geo[ci][0], geo[ci][1]
                dln, dsym = luts[(0, td)]
                aln, asym = luts[(1, ta)]
                for v in range(V):
                    for u in range(H):
                        blk = coef[ci][my * V + v, mx * H + u]
                        w = int(br.win[br.p])
                        if not dln[w]:
                            raise Refused(BAD_DATA, "code")
                        br.p += int(dln[w])
                        t = int(dsym[w])
                        if t > 11:
                            raise Refused(BAD_DATA, "DC category")
                        if t:
                            pred[sc] += extend(br.get(t), t)
                        blk[0] = np.int16(((pred[sc] + 32768) & 0xFFFF) - 32768)
                        k = 1
                        while k < 64:
                            w = int(br.win[br.p])
                            if not aln[w]:
                                raise Refused(BAD_DATA, "code")
                            br.p += int(aln[w])
                            rs = int(asym[w])
                            r, t = rs >> 4, rs & 15
                            if t:
                                k += r
                                if k > 63 or t > 10:
                                    raise Refused(BAD_DATA, "index / AC category")
                                blk[NATURAL[k]] = extend(br.get(t), t)
                            elif r != 15:
                                break
                            else:
                                k += 15
                            k += 1
            if br.p > br.n:
                raise Refused(BAD_DATA, "premature end")
        if br.n - br.p >= 8:
            raise Refused(BAD_DATA, "bytes after the segment's MCUs")
    return hd, geo, coef


def _up(P, rh, rv, dw, dh, h, w):
    """Component plane P (real size dh x dw at its top left) upsampled to h x w: jdsample.c's fancy h2v1 / h1v2 / h2v2 (plain
    for components 2 or fewer samples wide where libjpeg-turbo falls back)."""
    P = P[:dh, :dw].astype(np.int64)
    if rh == 1 and rv == 1:
        return P[:h, :w]
    y, x = np.arange(h)[:, None], np.arange(w)[None, :]
    j, r = x >> 1, y >> 1
    if rv == 1:
        if dw <= 2:
            return P[y, j]
        odd = x & 1
        right = np.where(j == dw - 1, P[y, j], (3 * P[y, j] + P[y, np.minimum(j + 1, dw - 1)] + 2) >> 2)
        left = np.where(j == 0, P[y, j], (3 * P[y, j] + P[y, np.maximum(j - 1, 0)] + 1) >> 2)
        return np.where(odd, right, left)
    nb = np.where(y & 1, np.minimum(r + 1, dh - 1), np.maximum(r - 1, 0))
    if rh == 1:
        return (3 * P[r, x] + P[nb, x] + np.where(y & 1, 2, 1)) >> 2
    if dw <= 2:
        return P[r, j]
    cs = lambda jj: 3 * P[r, jj] + P[nb, jj]   # noqa: E731
    right = np.where(j == dw - 1, (cs(j) * 4 + 7) >> 4, (3 * cs(j) + cs(np.minimum(j + 1, dw - 1)) + 7) >> 4)
    left = np.where(j == 0, (cs(j) * 4 + 8) >> 4, (3 * cs(j) + cs(np.maximum(j - 1, 0)) + 8) >> 4)
    return np.where(x & 1, right, left)


def ycc_gray(Y, cb, cr):
    """jdcolor.c's YCbCr -> RGB (Cr_r, Cb_b, Cr_g, Cb_g tables, SCALEBITS 16) and Pillow's L24."""
    cb, cr = cb - 128, cr - 128
    R = np.clip(Y + ((91881 * cr + 32768) >> 16), 0, 255)
    G = np.clip(Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16), 0, 255)
    B = np.clip(Y + ((116130 * cb + 32768) >> 16), 0, 255)
    return ((19595 * R + 38470 * G + 7471 * B + 0x8000) >> 16).astype(np.uint8)


def decode(data, rule, shortcut=True):
    """The gray image the device gives (rule 0 OpenCV, 1 Pillow), or Refused(status)."""
    hd, geo, coef = coefficients(data, rule)
    fr = hd["frame"]
    h, w = fr["h"], fr["w"]
    comps = [0] if rule == 0 or len(geo) == 1 else [0, 1, 2]
    planes = []
    for ci in comps:
        H, V, bw, bh, pw, ph = geo[ci]
        q = hd["dqt"][fr["comps"][ci][3]]
        px, inside = idct_islow(coef[ci].reshape(-1, 64), q, shortcut)
        if not inside.all():
            raise Refused(HOST_DIFFERS, "outside the IDCT envelope")
        planes.append(px.reshape(bh, bw, 8, 8).transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8))
    if len(planes) == 1:
        return np.ascontiguousarray(planes[0][:h, :w])
    hmax, vmax = max(g[0] for g in geo), max(g[1] for g in geo)
    up = [_up(P, hmax // g[0], vmax // g[1], g[4], g[5], h, w) for P, g in zip(planes, geo)]
    return ycc_gray(*up)


# ------------------------------------------------------------------------------------------------ the writer
def segment(marker, payload):
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + payload


def dqt(tables):
    """tables: {index: q [64] in natural order}; 16-bit entries where a value passes 255."""
    out = b""
    for tq, q in tables.items():
        q = np.asarray(q, np.int64)
        wide = int(q.max() > 255)
        zz = q[NATURAL]
        out += bytes([(wide << 4) | tq]) + (zz.astype(">u2").tobytes() if wide else zz.astype(np.uint8).tobytes())
    return segment(0xDB, out)


def dht(tables):
    """tables: {(class, index): (bits, values)}."""
    return segment(0xC4, b"".join(bytes([(tc << 4) | th]) + bytes(bits) + bytes(vals) for (tc, th), (bits, vals) in tables.items()))


def _category(v):
    return int(abs(int(v))).bit_length()


def encode(blocks, qs, h, w, sampling=None, tables=None, scan_tables=None, ri=0, ids=None, sof_marker=0xC0, app=b"", fill=0,
           rst=None, after_scan=b"", eoi=True, qindex=None, written_tables=None):
    """A sequential Huffman JPEG, h x w, of quantised coefficient blocks: blocks[c] [bh_c, bw_c, 64] int (natural order, the
    grid of whole MCUs the device lays out), qs {index: q [64] natural order}, qindex[c] each component's table (default c > 0).
    sampling [(H, V)] per component; tables {(class, index): (bits, values)} (Annex K luma 0 / chroma 1 by default); scan_tables
    [(td, ta)] per component; ri the restart interval; ids the component ids (1, 2, 3 by default); fill extra 0xFF bytes before
    every RSTn and EOI; rst(k): the marker code before segment k + 1 (RST k mod 8 by default); app raw segments after SOI;
    after_scan raw bytes before EOI; eoi False drops it; written_tables: the DHT segment's tables when they are to differ from
    the ones the data is coded with (tables the writer could not code with: invalid or remapped ones)."""
    nf = len(blocks)
    sampling = sampling or [(1, 1)] * nf
    ids = ids or list(range(1, nf + 1))
    qindex = qindex or [min(c, 1) for c in range(nf)]
    tables = tables or {(0, 0): STD_DC_LUMA, (1, 0): STD_AC_LUMA, (0, 1): STD_DC_CHROMA, (1, 1): STD_AC_CHROMA}
    scan_tables = scan_tables or [(min(c, 1), min(c, 1)) for c in range(nf)]
    codes = {k: canonical_codes(*v) for k, v in tables.items()}
    geo = [(H if nf > 1 else 1, V if nf > 1 else 1) for H, V in sampling]
    hmax, vmax = max(g[0] for g in geo), max(g[1] for g in geo)
    mcux, mcuy = -(-w // (8 * hmax)), -(-h // (8 * vmax))
    mcus = mcux * mcuy
    ri_eff = min(ri, mcus) if ri else mcus
    out = bytearray(b"\xff\xd8" + app + dqt(qs))
    sof = bytes([8]) + h.to_bytes(2, "big") + w.to_bytes(2, "big") + bytes([nf])
    for c in range(nf):
        sof += bytes([ids[c], (sampling[c][0] << 4) | sampling[c][1], qindex[c]])
    out += segment(sof_marker, sof)
    out += dht(written_tables or tables)
    if ri:
        out += segment(0xDD, ri.to_bytes(2, "big"))
    sos = bytes([nf]) + b"".join(bytes([ids[c], (scan_tables[c][0] << 4) | scan_tables[c][1]]) for c in range(nf)) + b"\x00\x3f\x00"
    out += segment(0xDA, sos)
    for s in range(-(-mcus // ri_eff)):
        bits, pred = [], [0] * nf
        for m in range(s * ri_eff, min(mcus, (s + 1) * ri_eff)):
            mx, my = m % mcux, m // mcux
            for c in range(nf):
                H, V = geo[c]
                dcc, acc = codes[(0, scan_tables[c][0])], codes[(1, scan_tables[c][1])]
                for v in range(V):
                    for u in range(H):
                        blk = np.asarray(blocks[c][my * V + v, mx * H + u], np.int64)
                        diff = int(blk[0]) - pred[c]
                        pred[c] = int(blk[0])
                        t = _category(diff)
                        bits.append(dcc[t])
                        if t:
                            bits.append((diff if diff > 0 else diff + (1 << t) - 1, t))
                        zz = blk[NATURAL]
                        run = 0
                        last = max([k for k in range(1, 64) if zz[k]], default=0)
                        for k in range(1, last + 1):
                            if zz[k] == 0:
                                run += 1
                                continue
                            while run > 15:
                                bits.append(acc[0xF0])
                                run -= 16
                            t = _category(zz[k])
                            bits.append(acc[(run << 4) | t])
                            bits.append((int(zz[k]) if zz[k] > 0 else int(zz[k]) + (1 << t) - 1, t))
                            run = 0
                        if last < 63:
                            bits.append(acc[0x00])
        acc_bits = "".join(format(c, f"0{n}b") for c, n in bits)
        acc_bits += "1" * (-len(acc_bits) % 8)
        raw = int(acc_bits, 2).to_bytes(len(acc_bits) // 8, "big") if acc_bits else b""
        out += raw.replace(b"\xff", b"\xff\x00")
        last_seg = (s + 1) * ri_eff >= mcus
        if not last_seg:
            out += b"\xff" * fill + bytes([0xFF, rst(s) if rst else 0xD0 + (s & 7)])
    out += after_scan
    if eoi:
        out += b"\xff" * fill + b"\xff\xd9"
    return bytes(out)


def quantise(img, q):
    """A gray image [h, w] uint8 -> [ceil(h / 8), ceil(w / 8), 64] quantised coefficients (an fp64 forward DCT, edges
    replicated), natural order -- input for encode()."""
    h, w = img.shape
    H, W = -(-h // 8) * 8, -(-w // 8) * 8
    x = np.pad(img.astype(np.float64), ((0, H - h), (0, W - w)), mode="edge") - 128
    k = np.arange(8)
    C = np.cos((2 * k[None, :] + 1) * k[:, None] * np.pi / 16) * np.where(k == 0, np.sqrt(0.125), 0.5)[:, None]
    b = x.reshape(H // 8, 8, W // 8, 8).transpose(0, 2, 1, 3)
    d = C @ b @ C.T
    return np.rint(d.reshape(H // 8, W // 8, 64) / np.asarray(q, np.float64)).astype(np.int64)
