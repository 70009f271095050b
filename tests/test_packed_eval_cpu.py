"""Packed evaluation without a GPU: the semantics crnn_forward_lines implements, restated on the fp64 oracle, and the packer.

A packed batch holds line i in columns [0, W_i) of slot i.  Each line's logits at frames t < W_i/4 - 1 must equal what the oracle
computes for that line alone, [1, W_i, 32].  That takes two things, which the restatement below does in fp64:
  - every activation a SAME convolution reads is zero at and past the line's boundary in that layer's resolution (W_i * H / W);
  - conv4_1 and conv4_2 normalise each line with its own batch statistics, over its own W_i / 4 x 4 positions.
The same restatement without the masks must fail, which shows the masks are what makes it right."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import crnn_oracle as O  # noqa: E402

WIDTHS = [8, 12, 36, 100, 260]
W = 260


def packed_forward(p, data, line_width, tsl, masks=True):
    """fp64 restatement of crnn_forward_lines: data [N, W, 32], line_width [N] -> logits [W/4-1, N, 64]."""
    x = torch.as_tensor(data, dtype=torch.float64)[:, None, :, :]
    Wp = x.shape[2]
    lw = [int(v) for v in line_width]

    def mask(y):
        if masks:
            for i, w in enumerate(lw):
                y[i, :, w * y.shape[2] // Wp:, :] = 0
        return y

    for name, kh, kw, ci, co, bn, relu, pad in O.CONV_SPECS:
        w_ = p[f"{name}/weights"].permute(3, 2, 0, 1)
        y = F.conv2d(x, w_, p[f"{name}/biases"], padding=(kh // 2, kw // 2) if pad == "SAME" else 0)
        if bn:
            beta, gamma = p[f"{name}/{name}/beta"], p[f"{name}/{name}/gamma"]
            rows = []
            for i, w in enumerate(lw):
                yi = y[i:i + 1, :, :w * y.shape[2] // Wp]          # the line's own positions
                mean = yi.mean(dim=(0, 2, 3))
                var = yi.var(dim=(0, 2, 3), unbiased=False)
                rows.append((y[i:i + 1] - mean[None, :, None, None]) / torch.sqrt(var[None, :, None, None] + O.BN_EPS)
                            * gamma[None, :, None, None] + beta[None, :, None, None])
            y = torch.cat(rows)
        if relu:
            y = torch.relu(y)
        if name in O.POOL_AFTER:
            y = F.max_pool2d(y, O.POOL_AFTER[name], O.POOL_AFTER[name])
        x = mask(y) if name != "conv5" else y
    N = x.shape[0]
    feat = x.permute(0, 2, 3, 1).reshape(N, -1, O.NUM_HID)
    fw = O.lstm_direction(feat, tsl, p[f"{O.LSTM_FW}/weights"], p[f"{O.LSTM_FW}/biases"], False)
    bw = O.lstm_direction(feat, tsl, p[f"{O.LSTM_BW}/weights"], p[f"{O.LSTM_BW}/biases"], True)
    out = torch.cat([fw, bw], dim=2).reshape(-1, O.NUM_HID) @ p["logits/weights"] + p["logits/biases"]
    return out.reshape(N, -1, O.NCLASSES).permute(1, 0, 2).contiguous()


def _lines(seed=7):
    rng = np.random.default_rng(seed)
    data = np.zeros((len(WIDTHS), W, 32))
    for i, w in enumerate(WIDTHS):
        data[i, :w] = rng.random((w, 32))
    tsl = np.array([w // 4 - 1 for w in WIDTHS], np.int32)
    return data, np.array(WIDTHS, np.int32), tsl


def _worst_error(masks):
    p = O.to_torch(O.randomize_params(O.init_params(3), seed=5, scale=0.3))
    data, lw, tsl = _lines()
    packed = packed_forward(p, data, lw, tsl, masks=masks)
    worst = 0.0
    for i, w in enumerate(WIDTHS):
        alone = O.forward(p, data[i:i + 1, :w], tsl[i:i + 1])
        t = int(tsl[i])
        d = (packed[:t, i] - alone[:t, 0]).abs().max().item()
        worst = max(worst, d / max(alone[:t, 0].abs().max().item(), 1e-30))
    return worst


def test_packed_restatement_equals_each_line_alone():
    assert _worst_error(masks=True) < 1e-12


def test_packed_restatement_without_masks_differs():
    assert _worst_error(masks=False) > 1e-6


# ---------------------------------------------------------------------------------------------------------------- packer
def _prepared(widths, seed=0):
    from lstm_ctc_ocr_b200.lib.lstm.test import prepare_line
    rng = np.random.default_rng(seed)
    return [prepare_line(rng.integers(0, 256, size=(32, w), dtype=np.uint8)) for w in widths]


def test_pack_lines_slots_padding_and_width():
    from lstm_ctc_ocr_b200.lib.lstm.test import pack_lines
    lines = _prepared([5, 8, 37, 100, 64])
    data, lw, tsl = pack_lines(lines)
    assert data.dtype == np.float32 and lw.dtype == np.int32 and tsl.dtype == np.int32
    assert data.shape == (5, max(d.shape[1] for d, _ in lines), 32)
    for i, (d, t) in enumerate(lines):
        w = d.shape[1]
        assert lw[i] == w and tsl[i] == t[0]
        assert np.array_equal(data[i, :w], d[0])
        assert not data[i, w:].any()


@pytest.mark.parametrize("bad", ["width_not_multiple", "too_narrow", "tsl_too_long", "tsl_negative", "shape", "empty"])
def test_pack_lines_rejects_bad_lines(bad):
    from lstm_ctc_ocr_b200.lib.lstm.test import pack_lines
    d, t = _prepared([40])[0]
    cases = {"width_not_multiple": [(np.zeros((1, 42, 32), np.float32), t)],
             "too_narrow": [(np.zeros((1, 4, 32), np.float32), np.array([0], np.int32))],
             "tsl_too_long": [(d, np.array([d.shape[1] // 4], np.int32))],
             "tsl_negative": [(d, np.array([-1], np.int32))],
             "shape": [(d[0], t)],
             "empty": []}
    with pytest.raises(ValueError):
        pack_lines(cases[bad])


@pytest.mark.parametrize("bad", ["line_width_not_multiple", "line_width_above_W", "line_width_below_8", "tsl_past_line", "shape"])
def test_validate_feed_checks_line_widths(bad):
    from lstm_ctc_ocr_b200.session import Session
    data = np.zeros((3, 64, 32), np.float32)
    lw = np.array([64, 32, 8], np.int32)
    tsl = np.array([15, 7, 1], np.int32)
    Session.validate_feed(data, tsl, None, None, lw)          # the good feed passes
    if bad == "line_width_not_multiple":
        lw = np.array([64, 30, 8], np.int32)
    elif bad == "line_width_above_W":
        lw = np.array([68, 32, 8], np.int32)
    elif bad == "line_width_below_8":
        lw = np.array([64, 32, 4], np.int32)
    elif bad == "tsl_past_line":
        tsl = np.array([15, 8, 1], np.int32)
    else:
        lw = np.array([64, 32], np.int32)
    with pytest.raises(ValueError):
        Session.validate_feed(data, tsl, None, None, lw)


def test_test_batch_size_is_a_config_key():
    from lstm_ctc_ocr_b200.lib.lstm import config
    old = config.cfg.TEST.BATCH_SIZE
    try:
        config.cfg_from_list(["TEST.BATCH_SIZE", "7"])
        assert config.cfg.TEST.BATCH_SIZE == 7
    finally:
        config.cfg.TEST.BATCH_SIZE = old


def test_line_width_placeholder_on_both_networks():
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    for name in ("LSTM_train", "LSTM_test"):
        net = get_network(name)
        assert net.line_width.name == "line_width" and net.line_width.dtype == "int32"
