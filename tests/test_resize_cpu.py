"""The native-size line feed without a GPU: the numpy restatement of Pillow's 8-bit BILINEAR (tests/resize_refs.py) against Pillow
itself, the size rule (lib.lstm.test.line_size) against prepare_line, the tap tables of crnn_resize_lines_u8 against the size rule,
and the host-side refusals of the `images` feed."""
import os
import random
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import resize_refs as R  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIMIT = 1024


def _pillow(img, nw, nh=32):
    from PIL import Image
    return np.asarray(Image.fromarray(img).resize((nw, nh), Image.BILINEAR), dtype=np.uint8)


def _cases():
    """2100 random gray lines: heights 1, 2, 31, 32, 33 and the limit, log-uniform heights up to the limit, widths 1 .. 4000
    (log-uniform, so narrow lines and the nw = 1 corner are common), constant images and rendered lines."""
    rng = np.random.default_rng(2024)
    out = []
    fixed_h = [1, 2, 31, 32, 33, LIMIT]
    for i in range(2000):
        h = fixed_h[i % len(fixed_h)] if i < 300 else int(np.exp(rng.uniform(0, np.log(LIMIT + 1))))
        h = min(max(h, 1), LIMIT)
        wmax = 4000 if h <= 200 else 600        # tall lines stay a few MB each
        w = int(np.exp(rng.uniform(0, np.log(wmax + 1))))
        w = min(max(w, 1), wmax)
        kind = i % 7
        if kind == 0:
            img = np.full((h, w), int(rng.integers(0, 256)), np.uint8)
        elif kind == 1:                          # extremes only: clamping of the integer accumulator
            img = (rng.integers(0, 2, (h, w)) * 255).astype(np.uint8)
        else:
            img = rng.integers(0, 256, (h, w), dtype=np.uint8)
        out.append(img)
    for w in (1, 2, 3, 4, 5, 7, 8, 9, 3999, 4000):
        out.append(rng.integers(0, 256, (LIMIT, w), dtype=np.uint8))
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    r = random.Random(7)
    font = gen.embedded_font(42)
    for _ in range(90):
        out.append(gen.render_line(gen.gen_rand(r, 1, 70), rng=r, font=font))
    return out


_CASES = None


def _all():
    global _CASES
    if _CASES is None:
        _CASES = _cases()
    return _CASES


def test_restatement_equals_pillow_byte_for_byte():
    from lstm_ctc_ocr_b200.lib.lstm.test import line_size
    cases = _all()
    assert len(cases) >= 2000
    assert {1, 2, 31, 32, 33, LIMIT} <= {im.shape[0] for im in cases}
    assert max(im.shape[1] for im in cases) == 4000 and min(im.shape[1] for im in cases) == 1
    ups = bad = 0
    for im in cases:
        nw = line_size(*im.shape)[0]
        ups += im.shape[0] < 32 or nw > im.shape[1]
        if not np.array_equal(R.resize_bilinear(im, nw, 32), _pillow(im, nw)):
            bad += 1
    assert ups > 300
    assert bad == 0, f"{bad} of {len(cases)} images differ from Pillow"


def test_restatement_equals_pillow_on_both_axes_at_other_sizes():
    """Sizes the evaluation rule never asks for: the taps of any in -> out pair, upscales and downscales on both axes."""
    rng = np.random.default_rng(5)
    for _ in range(200):
        h, w = (int(v) for v in rng.integers(1, 300, 2))
        nw, nh = (int(v) for v in rng.integers(1, 300, 2))
        img = rng.integers(0, 256, (h, w), dtype=np.uint8)
        assert np.array_equal(R.resize_bilinear(img, nw, nh), _pillow(img, nw, nh)), (h, w, nw, nh)


def test_size_rule_and_slot_equal_prepare_line():
    """line_size's (nw, line_width, time_step_len) and the packed slot built from the restatement against prepare_line (uint8 and
    f32) on every case."""
    from lstm_ctc_ocr_b200.lib.lstm.test import line_size, pack_lines, prepare_line
    for im in _all()[::3]:
        h, w = im.shape
        nw, width, tsl = line_size(h, w)
        assert nw == (w if h == 32 else max(1, int(32 / h * w)))
        assert width == max(8, -(-nw // 4) * 4) and tsl == max(nw // 4 - 1, 0)
        d8, t8 = prepare_line(im, dtype=np.uint8)
        df, tf = prepare_line(im)
        assert d8.shape == (1, width, 32) and df.shape == (1, width, 32) and t8.tolist() == [tsl] and tf.tolist() == [tsl]
        assert np.array_equal(d8[0], R.pack_slot(im, width, line_size))
        assert np.array_equal(df, d8.astype(np.float32) / 255.0)
    lines = [prepare_line(im, dtype=np.uint8) for im in _all()[:40]]
    data, lw, tsl = pack_lines(lines)
    W = data.shape[1]
    for i, im in enumerate(_all()[:40]):
        assert np.array_equal(data[i], R.pack_slot(im, W, line_size))
        assert (lw[i], tsl[i]) == line_size(*im.shape)[1:]


def test_tap_tables_hold_every_line_the_size_rule_makes():
    """crnn_resize_lines_u8 sizes its tap tables from max_h: 2 * (ceil(max_h / 16) + 1) + 1 horizontal taps and
    2 * ceil(max_h / 32) + 1 vertical ones.  Pillow's window is 2 * ceil(support) + 1 taps: every line of 1 .. 1024 rows and
    1 .. 4096 columns under the size rule fits in the tables of its own height."""
    src = open(os.path.join(ROOT, "lstm_ctc_ocr_b200", "csrc", "resize.cu")).read()
    assert re.search(r"RS_MAX_H = (\d+);", src).group(1) == str(LIMIT)
    h = np.arange(1, LIMIT + 1, dtype=np.int64)[:, None]
    w = np.arange(1, 4097, dtype=np.int64)[None, :]
    nw = np.where(h == 32, w, np.maximum(1, np.trunc(32.0 / h * w).astype(np.int64)))     # Python's double expression
    scale = w / nw
    ks_h = np.where(nw != w, 2 * np.ceil(np.maximum(scale, 1.0)).astype(np.int64) + 1, 0)
    assert (ks_h <= 2 * ((h + 15) // 16 + 1) + 1).all()
    ks_v = np.where(h != 32, 2 * np.ceil(np.maximum(h / 32.0, 1.0)).astype(np.int64) + 1, 0)
    assert (ks_v <= 2 * ((h + 31) // 32) + 1).all()


def test_limit_is_the_engines():
    from lstm_ctc_ocr_b200 import engine
    assert engine.RESIZE_MAX_HEIGHT == LIMIT
    hdr = open(os.path.join(ROOT, "include", "crnn_ctc.h")).read()
    assert "at most 1024 (CRNN_INVALID_VALUE outside [1, 1024])" in hdr


def _bare_session():
    """A Session without a device: run() refuses a bad `images` feed before it touches an engine or the GPU."""
    from lstm_ctc_ocr_b200.session import Session
    return Session.__new__(Session)


@pytest.mark.parametrize("bad", ["float", "3d", "1d", "empty_rows", "empty_cols", "too_tall", "no_lines", "one_array", "list"])
def test_bad_images_are_refused_before_any_launch(bad):
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    net = get_network("LSTM_test")
    ok = np.zeros((40, 100), np.uint8)
    feeds = {"float": [ok, ok.astype(np.float32)], "3d": [ok[:, :, None]], "1d": [ok[0]], "empty_rows": [ok[:0]],
             "empty_cols": [ok[:, :0]], "too_tall": [np.zeros((LIMIT + 1, 8), np.uint8)], "no_lines": [],
             "one_array": np.zeros((2, 40, 100), np.uint8), "list": [ok.tolist()]}
    with pytest.raises(ValueError):
        _bare_session().run(Fetch(net, "dense_decoded"), {net.images: feeds[bad]})


@pytest.mark.parametrize("other", ["data", "data_u8", "line_width", "time_step_len"])
def test_images_fed_with_another_batch_feed_is_refused(other):
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    net = get_network("LSTM_test")
    with pytest.raises(ValueError, match="images"):
        _bare_session().run(Fetch(net, "dense_decoded"), {net.images: [np.zeros((40, 100), np.uint8)],
                                                          getattr(net, other): np.zeros(1, np.int32)})


def test_images_with_train_op_or_a_training_model_is_refused():
    from lstm_ctc_ocr_b200.session import Session

    class _Eng:
        training = False
    with pytest.raises(ValueError, match="train_op"):
        Session._check_lines(["train_op"], _Eng(), "images")
    _Eng.training = True
    with pytest.raises(ValueError, match="training"):
        Session._check_lines(["dense_decoded"], _Eng(), "images")


def test_images_placeholder_is_lazy_and_shared():
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    net = get_network("LSTM_test")
    assert "_images" not in net.__dict__
    ph = net.images
    assert ph is net.images and ph.name == "images" and ph.dtype == "uint8"
    assert get_network("LSTM_train").images.name == "images"


def test_engine_refuses_host_tensors():
    import torch
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200._lib import CrnnError
    one = torch.ones(1, dtype=torch.int32)
    with pytest.raises(CrnnError, match="CUDA"):
        engine.resize_lines_u8(torch.zeros(8, dtype=torch.uint8), torch.zeros(1, dtype=torch.int64), one, one, one, 8, 1)
