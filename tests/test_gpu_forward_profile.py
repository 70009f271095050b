"""Per-stage profiling of every forward (include/crnn_ctc.h: crnn_profile_begin / crnn_profile_read).

Every bf16- and fp8-path forward records kNumStages + 1 events on the caller's stream, whatever its feed: device, uint8, page-locked
host memory in one or four image ranges (a chunked front end records its four front-end marks back to back), ordinary host memory,
packed lines, moving BatchNorm statistics (two marks per conv4 layer).  Calibration and the f32-class forwards (compute_dtype 2, 3)
record none.  bench.py reads these rows by stage name.

Each variant runs on a fresh model, whose events have never been recorded: a forward that recorded fewer than kNumStages + 1 events
would leave one unrecorded, and cudaEventElapsedTime fails on it inside crnn_profile_read."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N, W = 8, 64                  # four ranges of two images start on tile-pair boundaries: forward_host(chunks=4) runs chunked


def _t(a):
    return torch.tensor(a, device=DEV)


def _moving():
    from lstm_ctc_ocr_b200 import engine
    rng = np.random.default_rng(7)
    return {k: (rng.normal(0.0, 0.05, 512) if i % 2 == 0 else rng.uniform(0.002, 0.02, 512)).astype(np.float32)
            for i, k in enumerate(engine.BN_MOVING_KEYS)}


def _run(m, feed, data, lw, tsl):
    if feed == "device":
        m.forward(_t(data), _t(tsl))
    elif feed == "u8":
        m.forward(_t((data * 255).astype(np.uint8)), _t(tsl))
    elif feed in ("host1", "host4"):
        pin = torch.empty(data.shape, dtype=torch.float32).pin_memory()
        pin.numpy()[...] = data
        m.forward_host(pin.numpy(), _t(tsl), chunks=int(feed[-1]))
    elif feed == "pageable":
        staging = torch.empty(data.size, dtype=torch.float32).pin_memory()
        m.forward_pageable(data.copy(), staging, _t(tsl), chunks=4, host_threads=2)
    elif feed == "lines":
        m.forward_lines(_t(data), _t(lw), _t(tsl))


# (compute_dtype, moving statistics, feed, rows the read returns)
VARIANTS = [("bf16", False, f, 1) for f in ("device", "u8", "host1", "host4", "pageable", "lines")] + [
    ("bf16", True, "device", 1), ("bf16", True, "lines", 1),
    ("fp8", False, "device", 1), ("fp8", False, "host4", 1), ("fp8", False, "lines", 1), ("fp8", True, "device", 1),
    ("fp8", True, "lines", 1), ("fp8", False, None, 0),
    ("f32", False, "device", 0), ("tf32", False, "host4", 0)]


@pytest.mark.parametrize("dtype,moving,feed,rows", VARIANTS,
                         ids=[f"{d}-{'moving' if mv else 'batch'}-{f or 'calibration_only'}" for d, mv, f, _ in VARIANTS])
def test_forward_records_one_row_of_stage_times(dtype, moving, feed, rows):
    from lstm_ctc_ocr_b200 import engine
    from oracle import crnn_oracle as O
    m = engine.CrnnModel(device=DEV, compute_dtype=dtype)
    m.load_params(O.randomize_params(O.init_params(3, dtype=np.float32, logits_scale=10.0)))
    lw = np.random.default_rng(4).integers(2, W // 4 + 1, size=N).astype(np.int32) * 4
    data, _, _, tsl = O.synth_batch(N, W, seed=13, widths=[int(w) for w in lw] if feed == "lines" else None)
    if feed == "lines":
        tsl = np.minimum(tsl, lw // 4 - 1).astype(np.int32)
    if moving:
        m.load_bn_moving(_moving())
        m.set_bn_statistics("moving")
    engine.check(m.lib.crnn_profile_begin(m.handle, 4))
    if dtype == "fp8":
        m.calibrate_fp8(_t(data), _t(tsl))        # calibration records no row
    if feed is not None:
        _run(m, feed, data, lw, tsl)
    torch.cuda.synchronize()
    nst = m.lib.crnn_profile_num_stages()
    ms = np.full((4, nst), np.nan, np.float32)
    nf = ctypes.c_int(-1)
    engine.check(m.lib.crnn_profile_read(m.handle, ms.ctypes.data, nf))
    assert nf.value == rows
    assert np.isfinite(ms[:rows]).all() and (ms[:rows] >= 0).all(), ms[:rows]
