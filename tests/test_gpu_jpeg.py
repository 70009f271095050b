"""JPEG files decoded on the GPU (crnn_jpeg_decode_gray_u8, the `images` feed's JPEG entries) against the installed host readers
and the restatement in tests/jpeg_refs.py.

  1. Byte equality with cv2.imdecode(..., 0) (rule 0) and Pillow's convert("L") (rule 1) over test_jpeg_cpu's seeded corpus
     (Pillow qualities, subsamplings, optimize and restart markers, cv2 sampling factors and restart intervals, 1 x 1 to
     1024-row and 4096-column files, gray files declaring 2 x 2, the writer's custom tables, fill bytes and extreme
     coefficients) and on rendered lines saved by both writers; the output filled with 0xA5 first, every status 0.
  2. The workspace stage: the stored coefficients equal the restatement's, block for block.
  3. One defect per refusal class: its status, an all-zero slot, and the other files of the call identical to decoding them
     alone, in any order; the rule-specific refusals; repeat runs bit-identical.
  4. Guarded buffers of exactly the planned sizes (a truncated file last), status codes of bad arguments with the outputs
     untouched, a gated stream behind a busy default stream, graph capture and replay.
  5. Session.run with JPEG bytes and with JPEG, PNG and arrays mixed, bit-identical to the arrays feed; the staged bytes; the
     errors naming refused entries.
  6. test_model against the host path under both rules on a directory of JPEGs, PNGs and refused files, and on the decode-10k
     fixture's 10 240 lines saved as JPEG."""
import io
import os
import random
import sys
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import jpeg_refs as J  # noqa: E402
import test_jpeg_cpu as JC  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
host = JC.host


def _args(files, rule, sizes=None):
    from lstm_ctc_ocr_b200 import engine
    sizes = sizes or [engine.jpeg_size(f) or (1, 1) for f in files]
    flen = np.array([len(f) for f in files], np.int64)
    foff = np.zeros(len(files), np.int64)
    np.cumsum(flen[:-1], out=foff[1:])
    hw = np.array(sizes, np.int64).reshape(-1, 2)
    dec = hw[:, 0] * hw[:, 1]
    ooff = np.zeros(len(files), np.int64)
    np.cumsum(dec[:-1], out=ooff[1:])
    ws_offset, ws_bytes = engine.jpeg_plan(engine.jpeg_sof_records(files), flen, rule)
    t = lambda a: torch.tensor(np.ascontiguousarray(a), device=DEV)  # noqa: E731
    return ((t(np.frombuffer(b"".join(files), np.uint8)), t(foff), t(flen), t(hw[:, 0].astype(np.int32)), t(hw[:, 1].astype(np.int32)),
             t(ooff), t(ws_offset)), ws_bytes, int(dec.sum()), hw, ooff)


def _decode(files, rule, sizes=None, keep_ws=False):
    """[(image, status)] for each file of one call, after 0xA5 fills of the output and the workspace."""
    from lstm_ctc_ocr_b200 import engine
    a, ws_bytes, nout, hw, ooff = _args(files, rule, sizes)
    out = torch.full((max(nout, 1),), 0xA5, dtype=torch.uint8, device=DEV)
    ws = torch.full((max(ws_bytes, 1),), 0xA5, dtype=torch.uint8, device=DEV)
    _, st = engine.decode_jpeg_gray(*a, rule, out=out, workspace=ws)
    o, s = out.cpu().numpy(), st.cpu().numpy()
    res = [(o[ooff[i]:ooff[i] + hw[i, 0] * hw[i, 1]].reshape(hw[i, 0], hw[i, 1]), int(s[i])) for i in range(len(files))]
    return (res, ws.cpu().numpy(), a[6].cpu().numpy()) if keep_ws else res


def _rendered(n=512, seed=7):
    """Rendered lines of 30-70 characters saved by Pillow (gray, quality 75 and 4:2:0 colour) and cv2 (quality 95)."""
    import cv2
    from PIL import Image
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    r = random.Random(seed)
    font = gen.embedded_font(42)
    out = []
    for i in range(n):
        im = gen.render_line(gen.gen_rand(r, 30, 70), rng=r, font=font)
        if i % 3 == 0:
            out.append((f"line{i}_cv2", cv2.imencode(".jpg", im, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes()))
        elif i % 3 == 1:
            b = io.BytesIO()
            Image.fromarray(im).save(b, "JPEG")
            out.append((f"line{i}_pil_gray", b.getvalue()))
        else:
            b = io.BytesIO()
            Image.fromarray(np.stack([im, im, im // 2 + 64], -1)).save(b, "JPEG", quality=75, subsampling=2)
            out.append((f"line{i}_pil_420", b.getvalue()))
    return out


def _check_equal(corpus, rule, chunk=256):
    bad = []
    for k in range(0, len(corpus), chunk):
        part = corpus[k:k + chunk]
        got = _decode([f for _, f in part], rule)
        for (name, f), (img, st) in zip(part, got):
            if rule == 1 and JC.rule1_refused(name):
                if st != J.HOST_DIFFERS or img.any():
                    bad.append((name, st, "not refused"))
                continue
            want = host(f, rule)
            if st != 0 or img.shape != want.shape or not np.array_equal(img, want):
                bad.append((name, st, int((img != want).sum()) if img.shape == want.shape else "shape"))
    assert not bad, f"{len(bad)} of {len(corpus)} files differ from the rule-{rule} reader (name, status, bytes): {bad[:12]}"


@pytest.mark.parametrize("rule", [0, 1])
def test_corpus_equals_the_host_reader_byte_for_byte(rule):
    _check_equal(JC.corpus(), rule)


@pytest.mark.parametrize("rule", [0, 1])
def test_rendered_lines_equal_the_host_reader(rule, monkeypatch):
    monkeypatch.setenv("CRNN_FONT", "default")
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    gen._FONT_CACHE.clear()
    _check_equal(_rendered(), rule)


# ------------------------------------------------------------------------------------------------ 2. the workspace stage
@pytest.mark.parametrize("rule", [0, 1])
def test_stored_coefficients_equal_the_restatement(rule):
    corpus = [(n, f) for n, f in JC.corpus(seed=3, big=False)[::4] if not (rule == 1 and JC.rule1_refused(n))]
    files = [f for _, f in corpus]
    res, ws, ws_offset = _decode(files, rule, keep_ws=True)
    for (name, f), (_, st), r0 in zip(corpus, res, ws_offset[:-1]):
        assert st == 0, name
        hd, geo, coef = J.coefficients(f, rule)
        mcus = -(-hd["frame"]["w"] // (8 * max(g[0] for g in geo))) * -(-hd["frame"]["h"] // (8 * max(g[1] for g in geo)))
        off = r0 + 512 + -(-((mcus + 1) * 8) // 16) * 16
        for c in range(3 if rule == 1 and len(geo) == 3 else 1):
            n = coef[c].size
            got = ws[off:off + 2 * n].view(np.int16).reshape(coef[c].shape)
            assert np.array_equal(got, coef[c]), (name, c)
            off += 2 * n


# ------------------------------------------------------------------------------------------------ 3. refusals
def _malformed():
    """[(name, bytes, status under rule 0, status under rule 1)]: one defect per file, made from one valid gray file and one
    colour file."""
    rng = np.random.default_rng(5)
    img = JC._line(rng, 16, 24)
    q = np.full(64, 2, np.int64)
    blocks = J.quantise(img, q)
    good = J.encode([blocks], {0: q}, 16, 24, ri=2)
    enc = lambda **kw: J.encode([blocks], {0: q}, 16, 24, **kw)   # noqa: E731
    sos = good.index(b"\xff\xda")
    out = []

    def both(name, data, st):
        out.append((name, data, st, st))

    both("no_soi", b"\xff\xd9" + good[2:], J.BAD_HEADER)
    both("progressive", JC._pil(img, progressive=True), J.UNSUPPORTED)
    both("arithmetic", good.replace(b"\xff\xc0", b"\xff\xc9", 1), J.UNSUPPORTED)
    both("lossless", good.replace(b"\xff\xc0", b"\xff\xc3", 1), J.UNSUPPORTED)
    both("precision12", enc().replace(b"\xff\xc0\x00\x0b\x08", b"\xff\xc0\x00\x0b\x0c", 1), J.UNSUPPORTED)
    two = J.encode([blocks, blocks], {0: q, 1: q}, 16, 24)
    both("two_components", two, J.UNSUPPORTED)
    both("adobe_rgb", J.encode([blocks] * 3, {0: q, 1: q}, 16, 24, app=J.segment(0xEE, b"Adobe\0\x64\0\0\0\0\0")), J.UNSUPPORTED)
    both("rgb_ids", J.encode([blocks] * 3, {0: q, 1: q}, 16, 24, ids=[82, 71, 66]), J.UNSUPPORTED)
    both("dnl_zero_height", good.replace(b"\x08\x00\x10\x00\x18", b"\x08\x00\x00\x00\x18", 1), J.UNSUPPORTED)
    both("segment_length", good[:sos] + b"\xff\xfe\x00\x01" + good[sos:], J.BAD_MARKER)
    both("no_eoi", enc()[:-2], J.BAD_MARKER)
    both("truncated", good[:len(good) - 9], J.BAD_MARKER)
    both("com_in_scan", good[:-2] + J.segment(0xFE, b"x") + b"\xff\xd9", J.BAD_MARKER)
    both("second_scan", good[:-2] + good[sos:], J.UNSUPPORTED)
    both("spectral", good[:sos + 4 + 1 + 2] + b"\x01\x3f\x00" + good[sos + 4 + 1 + 2 + 3:], J.BAD_MARKER)
    std = {(0, 0): J.STD_DC_LUMA, (1, 0): J.STD_AC_LUMA}
    written = lambda k, t: enc(written_tables={**std, k: t})   # noqa: E731
    both("oversubscribed", written((0, 0), ([3] + [0] * 15, [0, 1, 2])), J.BAD_HUFFMAN)
    both("all_ones_code", written((0, 0), ([2] + [0] * 15, [0, 1])), J.BAD_HUFFMAN)
    both("dc_symbol_16", written((0, 0), (J.STD_DC_LUMA[0], [16] + list(range(1, 12)))), J.BAD_HUFFMAN)
    both("dht_index", written((0, 5), J.STD_DC_LUMA), J.BAD_HUFFMAN)
    # entropy-coded data: the data coded with the standard tables, read through remapped ones
    both("ac_category_11", written((1, 0), (J.STD_AC_LUMA[0], bytes([0x0B if v == 0x01 else v for v in J.STD_AC_LUMA[1]]))),
         J.BAD_DATA)
    cat0 = int(abs(int(blocks[0, 0, 0]))).bit_length()
    both("dc_category_12", written((0, 0), (J.STD_DC_LUMA[0], [12 if v == cat0 else v for v in range(12)])), J.BAD_DATA)
    blk = np.zeros_like(blocks)
    blk[..., 0] = blocks[..., 0]
    blk[..., 63] = 1                                               # ZRL x 3, then (14, 1); read with ZRL as (15, 1), k passes 63
    both("index_past_63", J.encode([blk], {0: q}, 16, 24, written_tables={**std, (1, 0): (
        J.STD_AC_LUMA[0], bytes([0xF1 if v == 0xF0 else v for v in J.STD_AC_LUMA[1]]))}), J.BAD_DATA)
    one = J.encode([blocks[:1, :1]], {0: q}, 8, 8)
    head = one[:one.index(b"\xff\xda") + 2 + int.from_bytes(one[one.index(b"\xff\xda") + 2:one.index(b"\xff\xda") + 4], "big")]
    both("invalid_code", head + b"\xff\x00\xff\x00\xff\xd9", J.BAD_DATA)               # sixteen 1 bits: no DC code
    r0 = good.index(b"\xff\xd0")
    both("premature_end", good[:r0 - 3] + good[r0:], J.BAD_DATA)
    both("extra_bytes", good.replace(b"\xff\xd0", b"\x12\x34\xff\xd0", 1), J.BAD_DATA)
    both("rst_order", good.replace(b"\xff\xd1", b"\xff\xd2", 1), J.BAD_RESTART)
    both("rst_missing", good.replace(b"\xff\xd0", b"", 1), J.BAD_RESTART)
    both("rst_extra", good[:-2] + b"\xff\xd3\xff\xd9", J.BAD_RESTART)
    both("rst_without_dri", J.encode([blocks], {0: q}, 16, 24, ri=2).replace(b"\xff\xdd\x00\x04\x00\x02", b"", 1), J.BAD_RESTART)
    # rule-specific
    for o in range(2, 9):
        out.append((f"exif_{o}", JC.with_exif(good, o), J.HOST_DIFFERS, 0))
    col = np.stack([img, img[::-1], 255 - img], -1)
    import cv2
    out.append(("cv2_411", JC._cv2(col, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x411111), 0, J.HOST_DIFFERS))
    cb = np.zeros((2, 4, 64), np.int64)
    cb[..., 0] = 20
    y_small = J.encode([blocks[:1, :2], cb, blocks[:1, :2]], {0: q, 1: q}, 16, 24, sampling=[(1, 1), (2, 2), (1, 1)])
    out.append(("y_not_largest", y_small, J.HOST_DIFFERS, 0))
    wrap = np.zeros((1, 1, 64), np.int64)
    wrap[0, 0, 0] = 1200
    both("idct_wraps", J.encode([wrap], {0: np.full(64, 4)}, 8, 8), J.HOST_DIFFERS)
    return out, good, img


def test_malformed_files_are_flagged_and_neighbours_unchanged():
    from lstm_ctc_ocr_b200 import engine
    bad, good, img = _malformed()
    files = [f for _, f, _, _ in bad]
    sizes = [engine.jpeg_size(f) if engine.jpeg_size(f) and engine.jpeg_size(f)[0] > 0 else (16, 24) for f in files]
    for rule in (0, 1):
        got = _decode(files, rule, sizes)
        for (name, f, w0, w1), (im, st) in zip(bad, got):
            want = (w0, w1)[rule]
            assert st == want, (rule, name, st, want)
            if want:
                assert not im.any(), name
            else:
                assert np.array_equal(im, host(f, rule)), name
        # the host readers do read what the device refuses for the rule alone
        alone = _decode([good], rule)[0]
        assert alone[1] == 0 and np.array_equal(alone[0], host(good, rule))
        for pos in (0, 7, len(files)):
            mixed = files[:pos] + [good] + files[pos:]
            res = _decode(mixed, rule, sizes[:pos] + [(16, 24)] + sizes[pos:])
            assert res[pos][1] == 0 and np.array_equal(res[pos][0], alone[0]), pos
            assert [s for _, s in res[:pos] + res[pos + 1:]] == [s for _, s in got]
    assert _decode([good], 0, [(17, 24)])[0][1] == J.BAD_HEADER       # a size unlike the frame's


def test_repeat_runs_and_orders_are_bit_identical():
    corpus = JC.corpus(seed=9, big=False)[::3]
    files = [f for _, f in corpus]
    a, b = _decode(files, 1), _decode(files, 1)
    perm = list(range(len(files)))[::-1]
    c = _decode([files[i] for i in perm], 1)
    for i in range(len(files)):
        assert a[i][1] == b[i][1] and np.array_equal(a[i][0], b[i][0])
        assert a[perm[i]][1] == c[i][1] and np.array_equal(a[perm[i]][0], c[i][0])


# ------------------------------------------------------------------------------------------------ 4. memory, codes, streams
@pytest.mark.parametrize("rule", [0, 1])
def test_guarded_buffers_of_the_planned_sizes(rule):
    import bounds as B
    from lstm_ctc_ocr_b200 import _lib, engine
    corpus = JC.corpus(seed=11, big=False)[::5]
    bad, good, _ = _malformed()
    files = [f for _, f in corpus] + [f for n, f, _, _ in bad if n != "truncated"] + [good[:len(good) - 9]]   # truncated last
    sizes = [engine.jpeg_size(f) if engine.jpeg_size(f) and engine.jpeg_size(f)[0] > 0 else (16, 24) for f in files]
    (d_files, foff, flen, h, w, ooff, wso), ws_bytes, nout, hw, _ = _args(files, rule, sizes)
    ins = [B.input_of(n, a.cpu().numpy()) for n, a in (("files", d_files), ("file_offset", foff), ("file_len", flen), ("h", h),
                                                       ("w", w), ("out_offset", ooff), ("ws_offset", wso))]
    out = B.output_of("out", (nout,), torch.uint8, align=1)
    status = B.output_of("status", (len(files),), torch.int32)
    ws = B.output_of("workspace", (ws_bytes,), torch.uint8, align=16)
    lib = _lib.load()

    def call():
        return lib.crnn_jpeg_decode_gray_u8(ins[0].ptr, ins[1].ptr, ins[2].ptr, len(files), ins[3].ptr, ins[4].ptr, ins[5].ptr, rule,
                                            out.ptr, status.ptr, ws.ptr, ins[6].ptr, ws_bytes, torch.cuda.current_stream().cuda_stream)
    problems, last = B.run_case(call, ins + [out, status, ws])
    assert not problems, problems
    st = last["status"].cpu().numpy()
    ok = [not (rule == 1 and JC.rule1_refused(n)) for n, _ in corpus]
    assert not st[:len(corpus)][ok].any() and st[-1] == J.BAD_MARKER


def test_status_codes_and_untouched_outputs():
    from lstm_ctc_ocr_b200 import _lib, engine
    lib = _lib.load()
    files = [f for _, f in JC.corpus(seed=2, big=False)[:3]]
    (d_files, foff, flen, h, w, ooff, wso), ws_bytes, nout, hw, _ = _args(files, 0)
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
    for k, al in (("foff", 8), ("flen", 8), ("ooff", 8), ("wso", 8), ("h", 4), ("w", 4), ("st", 4), ("ws", 16)):
        cases[k + "_misaligned"] = {k: base[k] + al // 2}
    for name, c in cases.items():
        a = dict(base, **c)
        s = lib.crnn_jpeg_decode_gray_u8(a["files"], a["foff"], a["flen"], a["N"], a["h"], a["w"], a["ooff"], a["rule"], a["out"],
                                         a["st"], a["ws"], a["wso"], ws_bytes, torch.cuda.current_stream().cuda_stream)
        assert s == 1, (name, s)
    torch.cuda.synchronize()
    assert (out == 0xA5).all() and (status == -7).all()
    a = base
    assert lib.crnn_jpeg_decode_gray_u8(a["files"], a["foff"], a["flen"], 3, a["h"], a["w"], a["ooff"], 0, a["out"], a["st"], a["ws"],
                                        a["wso"], ws_bytes - 1, torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    st = status[:3].cpu().numpy()
    assert st[2] == J.WORKSPACE and not st[:2].any()
    n2 = int(hw[2, 0] * hw[2, 1])
    assert not out[nout - n2:nout].any()
    with pytest.raises(Exception):
        engine.decode_jpeg_gray(d_files.cpu(), foff, flen, h, w, ooff, wso, 0)


def test_gated_stream_and_graph_replay():
    import test_gpu_streams as SG
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200._lib import check
    corpus = [(n, f) for n, f in JC.corpus(seed=13, big=False)[::7] if not JC.rule1_refused(n)]
    files = [f for _, f in corpus]
    (s_files, foff, flen, s_h, s_w, ooff, wso), ws_bytes, nout, hw, offs = _args(files, 1)
    d_files, h, w = (torch.empty_like(v) for v in (s_files, s_h, s_w))
    out = torch.empty(nout, dtype=torch.uint8, device=DEV)
    status = torch.empty(len(files), dtype=torch.int32, device=DEV)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)

    def call():
        check(engine._lib.load().crnn_jpeg_decode_gray_u8(d_files.data_ptr(), foff.data_ptr(), flen.data_ptr(), len(files),
                                                          h.data_ptr(), w.data_ptr(), ooff.data_ptr(), 1, out.data_ptr(),
                                                          status.data_ptr(), ws.data_ptr(), wso.data_ptr(), ws_bytes, engine._stream()))
        return {"out": out.clone(), "status": status.clone()}
    got = SG._gated("jpeg_decode_gray_u8", call, [(d_files, s_files), (h, s_h), (w, s_w)], [out, status])
    o = got["out"].cpu().numpy()
    assert not got["status"].cpu().numpy().any()
    for i, f in enumerate(files):
        assert np.array_equal(o[offs[i]:offs[i] + hw[i, 0] * hw[i, 1]].reshape(hw[i]), host(f, 1)), corpus[i][0]
    d_files.copy_(s_files), h.copy_(s_h), w.copy_(s_w)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            engine.decode_jpeg_gray(d_files, foff, flen, h, w, ooff, wso, 1, out=out, workspace=ws, status=status)
    torch.cuda.current_stream().wait_stream(s)
    out.fill_(0xA5)
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), o) and not status.cpu().numpy().any()


# ------------------------------------------------------------------------------------------------ 5. Session and test_model
def _weights():
    import test_gpu_packed_eval as PE
    return PE._load("make_decode10k", "tests", "golden", "make_decode10k.py").load_weights()


def test_session_jpeg_png_and_arrays_mixed_are_bit_identical(monkeypatch):
    import png_refs as P
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.lstm.test import gray_rule
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.session import Session
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    jpegs = [f for _, f in _rendered(30, seed=3)]
    arrays = [host(f, gray_rule()) for f in jpegs]
    pngs = [P.write_png(a, 8, 0) for a in arrays]
    mixed = [(jpegs[i], pngs[i], arrays[i])[i % 3] for i in range(len(jpegs))]
    net = get_network("LSTM_test")
    with Session(device=DEV) as sess:
        sess.assign(net, _weights())
        fetches = [Fetch(net, k) for k in ("logits", "dense_decoded")]
        ref = sess.run(fetches, {net.images: arrays, net.keep_prob: 1.0})
        for feed in (jpegs, mixed):
            got = sess.run(fetches, {net.images: feed, net.keep_prob: 1.0})
            for a, b in zip(ref, got):
                assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
        sess.run(fetches, {net.images: jpegs, net.keep_prob: 1.0})
        # the encoded bytes, and per line its offset, sizes and time steps, and its file's offsets, length and plan entry
        assert sess.h2d_bytes == sum(len(f) for f in jpegs) + 68 * len(jpegs) + 8
        bad, good, _ = _malformed()
        png_bad = bytearray(pngs[0])
        png_bad[-13] ^= 1
        with pytest.raises(engine.JpegDecodeError) as e:
            sess.run(fetches, {net.images: [good, bad[1][1], arrays[0], bad[-1][1]], net.keep_prob: 1.0})
        assert e.value.entries == [1, 3] and e.value.status == [J.UNSUPPORTED, J.HOST_DIFFERS]
        with pytest.raises(engine.ImageDecodeError) as e:
            sess.run(fetches, {net.images: [bytes(png_bad), good, bad[-1][1], pngs[1]], net.keep_prob: 1.0})
        assert type(e.value) is engine.ImageDecodeError and e.value.entries == [0, 2] and e.value.status == [3, J.HOST_DIFFERS]
        with pytest.raises(engine.PngDecodeError):
            sess.run(fetches, {net.images: [bytes(png_bad), good], net.keep_prob: 1.0})


def _write_eval_dir(path, seed=17):
    """Rendered lines as JPEG from both writers, gray and colour, mixed with PNGs and with files the device refuses."""
    import cv2
    from PIL import Image
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    r = random.Random(seed)
    font = gen.embedded_font(42)
    for k in range(40):
        text = gen.gen_rand(r, 4, 20)
        im = gen.render_line(text, rng=r, font=font)
        col = np.stack([im, im // 2 + 100, 255 - im // 3], -1)
        name = os.path.join(path, f"{k:04d}_{text}")
        kind = k % 10
        if kind == 0:
            cv2.imwrite(name + ".jpg", im)
        elif kind == 1:
            cv2.imwrite(name + ".jpg", col, [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x221111, cv2.IMWRITE_JPEG_RST_INTERVAL, 4])
        elif kind == 2:
            Image.fromarray(im).save(name + ".jpg", quality=60, optimize=True)
        elif kind == 3:
            Image.fromarray(col).save(name + ".jpg", quality=75, subsampling=1)
        elif kind == 4:
            Image.fromarray(col).save(name + ".jpg", quality=90, subsampling=0, restart_marker_rows=1)
        elif kind == 5:
            Image.fromarray(im).save(name + ".png")
        elif kind == 6:                                   # progressive: read on the host
            Image.fromarray(im).save(name + ".jpg", progressive=True)
        elif kind == 7:                                   # 4:1:1 colour: refused under rule 1, read under rule 0
            cv2.imwrite(name + ".jpg", col, [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x411111])
        elif kind == 8:                                   # Exif orientation 1 (read) and 3 (refused under rule 0)
            data = cv2.imencode(".jpg", im)[1].tobytes()
            open(name + ".jpg", "wb").write(JC.with_exif(data, 1 if k % 20 == 8 else 3))
        else:                                             # bytes before a restart marker: the device refuses, the host reads
            data = cv2.imencode(".jpg", im, [cv2.IMWRITE_JPEG_RST_INTERVAL, 2])[1].tobytes()
            open(name + ".jpg", "wb").write(data.replace(b"\xff\xd0", b"\x00\xff\xd0", 1))


def _compare_test_model(path, bs):
    import test_gpu_resize as RZ
    from lstm_ctc_ocr_b200.lib.lstm import test as T
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    strip = lambda text: [ln.split(" cost time")[0] if "cost time" in ln else ln for ln in text.splitlines()]  # noqa: E731
    old = cfg.TEST.BATCH_SIZE
    try:
        cfg.TEST.BATCH_SIZE = bs
        net = get_network("LSTM_test")
        with Session(device=DEV) as sess:
            sess.assign(net, _weights())
            sw = T.SolverWrapper(sess, net, None, path, None)
            new, hst = io.StringIO(), io.StringIO()
            with redirect_stdout(new):
                r_new = sw.test_model(sess, testDir=path, restore=False)
            with redirect_stdout(hst):
                r_host = RZ._host_test_model(sess, net, path, bs)
        assert r_new == r_host
        assert strip(new.getvalue()) == strip(hst.getvalue()), bs
        return r_new
    finally:
        cfg.TEST.BATCH_SIZE = old


@pytest.mark.parametrize("opencv", [True, False])
def test_test_model_output_equals_the_host_path(opencv, tmp_path, monkeypatch):
    from lstm_ctc_ocr_b200.lib.lstm import test as T
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    _write_eval_dir(str(tmp_path))
    if not opencv:
        monkeypatch.setitem(sys.modules, "cv2", None)
    assert T.gray_rule() == (0 if opencv else 1)
    for bs in (1, 16):
        assert _compare_test_model(str(tmp_path), bs)[1] == 40


def test_test_model_on_the_fixture_lines_saved_as_jpeg(tmp_path, monkeypatch):
    """The decode-10k fixture's 10 240 lines saved as JPEG by OpenCV (quality 95): reads and accuracy equal the host path's."""
    import cv2
    import test_gpu_png as TP
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    texts, imgs = TP._fixture_images()
    for i, (t, im) in enumerate(zip(texts, imgs)):
        cv2.imwrite(os.path.join(str(tmp_path), f"{i:05d}_{t}.jpg"), im)
    assert _compare_test_model(str(tmp_path), 256)[1] == len(imgs)
