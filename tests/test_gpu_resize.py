"""Native-size lines resized on the GPU (crnn_resize_lines_u8, the `images` feed) against the host path of prepare_line + pack_lines.

  1. The kernel byte for byte.  The output is filled with 0xA5 before every call; each slot must then equal the uint8 pack of
     prepare_line (Pillow's resize on the host), padding included, so every byte of [N, W, 32] is shown to be written.  Heights
     1, 8, 20, 31, 32, 33, 48, 60, 64, 100, 200 and 1024, widths 1 .. 4000 (upscales, the nw = 1 corner, the vertical-first order
     of sources over 100 times taller than wide), rendered lines; batched with slots wider than their lines, and one line per
     call at its own width.
  2. Session.run with `images` against the prepared data_u8 + line_width + time_step_len feed: bit-identical logits, equal
     greedy and beam decodes, alignments and lexicon reads under bf16, fp8 and moving BatchNorm statistics; loss, costs,
     gradient and label alignment of a training network.
  3. test_model: identical output (apart from the time per line) to the host-path rendition, at TEST.BATCH_SIZE 1 and 64, on a
     directory that mixes those heights.
  4. The entry point on a gated non-blocking stream behind a busy default stream (test_gpu_streams' window), and its status codes
     with the output left untouched."""
import io
import os
import random
import sys
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_packed_eval as PE  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HEIGHTS = (1, 8, 20, 31, 32, 33, 48, 60, 64, 100, 200, 1024)


def _lines(seed=3):
    """Gray lines at every height of HEIGHTS and widths 1 .. 4000, plus tall narrow sources and rendered lines."""
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    rng = np.random.default_rng(seed)
    out = []
    for h in HEIGHTS:
        for w in (1, 2, 3, 5, 9, 31, 32, 33, 100, 257, 999, 2048, 4000):
            if h * w > 1 << 22:
                w = (1 << 22) // h
            out.append(rng.integers(0, 256, (h, w), dtype=np.uint8))
    for h, w in ((1024, 2), (1024, 10), (201, 2), (300, 2), (1001, 10), (700, 6)):    # vertical pass first (h > 100 w)
        out.append(rng.integers(0, 256, (h, w), dtype=np.uint8))
    out.append(np.full((60, 500), 255, np.uint8))
    out.append((rng.integers(0, 2, (45, 700)) * 255).astype(np.uint8))
    r = random.Random(seed)
    font = gen.embedded_font(42)
    for _ in range(24):
        out.append(gen.render_line(gen.gen_rand(r, 1, 70), rng=r, font=font))
    return out


def _host_slots(images):
    """pack_lines([prepare_line(im, uint8)]) of each line alone: [width_i, 32] uint8."""
    from lstm_ctc_ocr_b200.lib.lstm.test import pack_lines, prepare_line
    return [pack_lines([prepare_line(im, dtype=np.uint8)])[0][0] for im in images]


def _device_batch(images):
    from lstm_ctc_ocr_b200.lib.lstm.test import line_size
    sizes = np.array([line_size(*im.shape) for im in images], np.int32).reshape(-1, 3)
    nbytes = np.array([im.size for im in images], np.int64)
    off = np.zeros(len(images), np.int64)
    np.cumsum(nbytes[:-1], out=off[1:])
    src = torch.tensor(np.concatenate([im.reshape(-1) for im in images]), device=DEV)
    t = lambda a: torch.tensor(np.ascontiguousarray(a), device=DEV)  # noqa: E731
    h = np.array([im.shape[0] for im in images], np.int32)
    w = np.array([im.shape[1] for im in images], np.int32)
    return src, t(off), t(h), t(w), t(sizes[:, 0]), int(sizes[:, 1].max()), int(h.max())


# ------------------------------------------------------------------------------------------------ 1. the kernel byte for byte
def test_kernel_equals_the_host_pack_byte_for_byte():
    from lstm_ctc_ocr_b200 import engine
    images = _lines()
    want = _host_slots(images)
    order = sorted(range(len(images)), key=lambda i: want[i].shape[0])
    bad = []
    # batches of mixed widths (slots wider than their lines) and every line alone at its own width
    for idx in [order[k:k + 16] for k in range(0, len(order), 16)] + [[i] for i in range(len(images))]:
        src, off, h, w, ow, W, max_h = _device_batch([images[i] for i in idx])
        out = torch.full((len(idx), W, 32), 0xA5, dtype=torch.uint8, device=DEV)
        engine.resize_lines_u8(src, off, h, w, ow, W, max_h, out=out)
        got = out.cpu().numpy()
        for r, i in enumerate(idx):
            slot = np.zeros((W, 32), np.uint8)
            slot[:want[i].shape[0]] = want[i]
            if not np.array_equal(got[r], slot):
                bad.append((images[i].shape, len(idx), int((got[r] != slot).sum())))
    assert not bad, f"{len(bad)} slots differ from the host pack (shape, batch, bytes): {bad[:10]}"


def test_kernel_equals_the_host_pack_on_random_shapes():
    from lstm_ctc_ocr_b200 import engine
    rng = np.random.default_rng(11)
    for rep in range(4):
        images = []
        for _ in range(64):
            h = int(np.exp(rng.uniform(0, np.log(1025))))
            w = int(np.exp(rng.uniform(0, np.log(4001 if h <= 200 else 600))))
            images.append(rng.integers(0, 256, (max(h, 1), max(w, 1)), dtype=np.uint8))
        want = _host_slots(images)
        src, off, h, w, ow, W, max_h = _device_batch(images)
        out = torch.full((len(images), W, 32), 0xA5, dtype=torch.uint8, device=DEV)
        got = engine.resize_lines_u8(src, off, h, w, ow, W, max_h, out=out).cpu().numpy()
        for i in range(len(images)):
            assert np.array_equal(got[i, :want[i].shape[0]], want[i]), (rep, images[i].shape)
            assert not got[i, want[i].shape[0]:].any(), (rep, images[i].shape)


# ------------------------------------------------------------------------------------------------ 2. Session.run
def _eval_lines(seed=21, n=40):
    """Rendered 60-row lines and a few at other heights, with their texts."""
    from PIL import Image
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    r = random.Random(seed)
    font = gen.embedded_font(42)
    texts, images = [], []
    for i in range(n):
        t = gen.gen_rand(r, 4, 30)
        im = gen.render_line(t, rng=r, font=font)
        h = HEIGHTS[i % len(HEIGHTS)]
        if i % 3 == 0 and h not in (1, 1024):            # the same text at another native height
            im = np.asarray(Image.fromarray(im).resize((max(1, im.shape[1] * h // im.shape[0]), h), Image.BILINEAR), np.uint8)
        texts.append(t)
        images.append(np.ascontiguousarray(im))
    return texts, images


def _same(a, b, path=""):
    if isinstance(a, dict):
        assert set(a) == set(b), path
        for k in a:
            _same(a[k], b[k], f"{path}/{k}")
    else:
        a, b = np.asarray(a), np.asarray(b)
        assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), path


@pytest.mark.parametrize("dtype,bn", [("bf16", "batch"), ("fp8", "batch"), ("bf16", "moving")])
def test_session_images_equal_the_prepared_feed(dtype, bn, tmp_path, monkeypatch):
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg, get_encode_decode_dict
    from lstm_ctc_ocr_b200.lib.lstm.test import pack_lines, prepare_line
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.session import Session
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    weights = dict(PE._load("make_decode10k", "tests", "golden", "make_decode10k.py").load_weights())
    if bn == "moving":
        rng = np.random.default_rng(2)
        for i, k in enumerate(engine.BN_MOVING_KEYS):
            weights[k] = (rng.normal(0, 0.2, 512) if i % 2 == 0 else rng.uniform(0.5, 2.0, 512)).astype(np.float32)
    texts, images = _eval_lines()
    data, lw, tsl = pack_lines([prepare_line(im, dtype=np.uint8) for im in images])
    enc, _ = get_encode_decode_dict()
    words = sorted(set(texts))
    lex = tmp_path / "words.txt"
    lex.write_text("\n".join(words) + "\n", encoding="utf-8")
    saved = (cfg.TEST.COMPUTE_DTYPE, cfg.TEST.BN_STATS, cfg.DECODER, cfg.TEST.LEXICON)
    try:
        cfg.TEST.COMPUTE_DTYPE, cfg.TEST.BN_STATS, cfg.TEST.LEXICON = dtype, bn, str(lex)
        net = get_network("LSTM_test")
        with Session(device=DEV) as sess:
            sess.assign(net, weights)
            for decoder in ("greedy", "beam"):
                cfg.DECODER = decoder
                fetches = [Fetch(net, k) for k in ("logits", "dense_decoded", "read_alignment", "lexicon_decoded")]
                ref = sess.run(fetches, {net.data_u8: data, net.line_width: lw, net.time_step_len: tsl, net.keep_prob: 1.0})
                got = sess.run(fetches, {net.images: images, net.keep_prob: 1.0})
                assert sess.last_feed_path.startswith("native-size")
                assert sess.h2d_bytes == sum(im.size for im in images) + len(images) * (8 + 5 * 4)
                for f, a, b in zip(fetches, ref, got):
                    _same(a, b, f"{dtype}/{bn}/{decoder}/{f.kind}")
    finally:
        cfg.TEST.COMPUTE_DTYPE, cfg.TEST.BN_STATS, cfg.DECODER, cfg.TEST.LEXICON = saved
    if dtype == "bf16" and bn == "batch":
        labels = np.concatenate([[enc[c] for c in t] for t in texts]).astype(np.int32)
        llen = np.array([len(t) for t in texts], np.int32)
        tnet = get_network("LSTM_train")
        with Session(device=DEV) as sess:
            sess.assign(tnet, weights)
            fetches = [Fetch(tnet, k) for k in ("loss", "ctc_costs", "ctc_grad", "label_alignment", "logits")]
            ref = sess.run(fetches, {tnet.data_u8: data, tnet.line_width: lw, tnet.time_step_len: tsl, tnet.labels: labels,
                                     tnet.labels_len: llen})
            got = sess.run(fetches, {tnet.images: images, tnet.labels: labels, tnet.labels_len: llen})
            for f, a, b in zip(fetches, ref, got):
                _same(a, b, f"train/{f.kind}")
            with pytest.raises(ValueError, match="train_op"):
                sess.run(Fetch(tnet, "train_op"), {tnet.images: images, tnet.labels: labels, tnet.labels_len: llen})


# ------------------------------------------------------------------------------------------------ 3. test_model
def _write_mixed_dir(path, n=80, seed=99):
    from PIL import Image
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    rng = random.Random(seed)
    for i in range(n):
        text = gen.gen_rand(rng, 4, 30)
        im = gen.render_line(text, rng=rng)
        h = HEIGHTS[i % len(HEIGHTS)]
        if h != im.shape[0]:
            im = np.asarray(Image.fromarray(im).resize((max(1, im.shape[1] * h // im.shape[0]), h), Image.BILINEAR), np.uint8)
        Image.fromarray(im).save(os.path.join(path, f"{i:04d}_{text}.png"))


def _host_test_model(sess, net, test_dir, bs):
    """test_model's loop as it ran before the `images` feed: prepare_line per file on the host, pack_lines, the data_u8 feed."""
    from lstm_ctc_ocr_b200.lib.lstm import test as T
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    files = sorted(os.listdir(test_dir))
    lines = [T.prepare_line(T.load_line_image(os.path.join(test_dir, f)), dtype=np.uint8) for f in files]
    order = sorted(range(len(files)), key=lambda i: lines[i][0].shape[1])
    res = {}
    for b0 in range(0, len(order), bs):
        idx = order[b0:b0 + bs]
        data, lw, tsl = T.pack_lines([lines[i] for i in idx])
        dense = sess.run(Fetch(net, "dense_decoded"), {net.data_u8: data, net.line_width: lw, net.time_step_len: tsl})
        for r, i in enumerate(idx):
            res[i] = "".join(T.decodeRes(dense[r]))
    correct = 0
    for i, f in enumerate(files):
        correct += f.split(".")[0].split("_")[1] == res[i]
        print(f, end=" ")
        print("cost time: {:.3f},\n    res: {}".format(0.0, res[i]))
    print("total acc:{}/{}={:.4f}".format(correct, len(files), correct / max(len(files), 1)))
    return correct, len(files)


def test_test_model_output_equals_the_host_path(tmp_path, monkeypatch):
    from lstm_ctc_ocr_b200.lib.lstm import test as T
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    _write_mixed_dir(str(tmp_path))
    weights = PE._load("make_decode10k", "tests", "golden", "make_decode10k.py").load_weights()
    strip = lambda text: [ln.split(" cost time")[0] if "cost time" in ln else ln for ln in text.splitlines()]  # noqa: E731
    old = cfg.TEST.BATCH_SIZE
    try:
        for bs in (1, 64):
            cfg.TEST.BATCH_SIZE = bs
            net = get_network("LSTM_test")
            with Session(device=DEV) as sess:
                sess.assign(net, weights)
                sw = T.SolverWrapper(sess, net, None, str(tmp_path), None)
                new, host = io.StringIO(), io.StringIO()
                with redirect_stdout(new):
                    r_new = sw.test_model(sess, testDir=str(tmp_path), restore=False)
                with redirect_stdout(host):
                    r_host = _host_test_model(sess, net, str(tmp_path), bs)
            assert r_new == r_host and r_new[1] == 80
            assert strip(new.getvalue()) == strip(host.getvalue()), bs
            assert sum("cost time" in ln for ln in new.getvalue().splitlines()) == 80
    finally:
        cfg.TEST.BATCH_SIZE = old


# ------------------------------------------------------------------------------------------------ 4. streams and status codes
def test_entry_point_on_a_gated_stream_behind_a_busy_default_stream():
    import test_gpu_streams as SG
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200._lib import check
    images = _lines(seed=5)[::3]
    s_src, off, s_h, s_w, s_ow, W, max_h = _device_batch(images)
    src, h, w, ow = (torch.empty_like(v) for v in (s_src, s_h, s_w, s_ow))
    out = torch.empty((len(images), W, 32), dtype=torch.uint8, device=DEV)

    def call():
        check(engine._lib.load().crnn_resize_lines_u8(src.data_ptr(), off.data_ptr(), h.data_ptr(), w.data_ptr(), ow.data_ptr(),
                                                      len(images), W, max_h, out.data_ptr(), engine._stream()))
        return {"out": out.clone()}
    got = SG._gated("resize_lines_u8", call, [(src, s_src), (h, s_h), (w, s_w), (ow, s_ow)], [out])
    want = _host_slots(images)
    g = got["out"].cpu().numpy()
    for i in range(len(images)):
        slot = np.zeros((W, 32), np.uint8)
        slot[:want[i].shape[0]] = want[i]
        assert np.array_equal(g[i], slot), images[i].shape


def test_status_codes_and_untouched_output():
    from lstm_ctc_ocr_b200 import _lib, engine
    lib = _lib.load()
    images = [np.full((40, 50), 7, np.uint8), np.full((20, 9), 9, np.uint8)]
    src, off, h, w, ow, W, max_h = _device_batch(images)
    out = torch.full((2, 64, 32), 0xA5, dtype=torch.uint8, device=DEV)
    p = lambda t: t.data_ptr()  # noqa: E731
    st = torch.cuda.current_stream().cuda_stream
    base = dict(src=p(src), off=p(off), h=p(h), w=p(w), ow=p(ow), N=2, W=64, max_h=max_h, out=p(out))
    cases = {"N0": dict(N=0), "Nneg": dict(N=-1), "W4": dict(W=4), "W62": dict(W=62), "maxh0": dict(max_h=0),
             "maxh_over": dict(max_h=engine.RESIZE_MAX_HEIGHT + 1), "src0": dict(src=0), "off0": dict(off=0), "h0": dict(h=0),
             "w0": dict(w=0), "ow0": dict(ow=0), "out0": dict(out=0), "out_misaligned": dict(out=p(out) + 1)}
    for name, c in cases.items():
        a = dict(base, **c)
        s = lib.crnn_resize_lines_u8(a["src"], a["off"], a["h"], a["w"], a["ow"], a["N"], a["W"], a["max_h"], a["out"], st)
        assert s == 1, (name, s)                       # CRNN_INVALID_VALUE
    torch.cuda.synchronize()
    assert (out == 0xA5).all()
    a = base
    assert lib.crnn_resize_lines_u8(a["src"], a["off"], a["h"], a["w"], a["ow"], 2, 64, engine.RESIZE_MAX_HEIGHT, a["out"], st) == 0
    torch.cuda.synchronize()
    want = _host_slots(images)
    got = out.cpu().numpy()
    for i in range(2):
        assert np.array_equal(got[i, :want[i].shape[0]], want[i]) and not got[i, want[i].shape[0]:].any()
