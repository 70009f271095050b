"""Packed evaluation (crnn_forward_lines) on the GPU: every line of a packed batch computed as if it were evaluated alone.

  1. Line-alone equality.  The 67 evaluation lines of test_gpu_width_edges (64 rendered lines 396 - 944 px wide and crops
     8, 9 and 12 px wide) with the decode-10k fixture's trained weights, packed in one batch and in batches of 7, against
     crnn_forward of each line alone ([1, W_i, 32]).  Logits are compared per element at t < time_step_len; the only
     difference the design allows is the order of the per-line f64 statistics atomics.  Greedy and beam labels must equal the
     line-alone decode on every line, and the oracle's decode on every line above test_gpu_decode10k.MARGIN.
  2. Every stage per line.  Batches with lines of W_i = 8 .. 1024 in one W = 1024 batch, N = 1 with W_i < W, N = 130 (across
     a 128-sample LSTM tile) and N = 1024 mixed widths at W = 256: masked positions of a1, a2, a3, a3p, a4a (and the pre-BN
     a4a / a4b) are exactly zero; each line's conv1 .. conv3_2 activations equal its line-alone run's bit for bit (they do
     not depend on other lines), its conv4_x pre-BN values, BN and later activations within one bf16 ulp; each line's "stats"
     equal fp64 sums of its own pre-BN values and its "bn" the fp64 finalize of those, within 4.5x the measured error.  Lines of equal width and different content get different coefficients, each its own
     line-alone run's, none the whole-batch forward's.
  3. Interfaces: test_model with TEST.BATCH_SIZE 1 and 64, Session.run with line_width (greedy, beam, train_op refused),
     status codes.
Rows go to build/packed_eval_report.jsonl."""
import importlib.util
import io
import os
import random
import sys
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from stage_check import Checker  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REPORT = "packed_eval_report.jsonl"
# Measured on an H100 80GB HBM3 (SXM, 700 W power limit); every bound is 4.5x its measurement.
# |packed - line alone| / max|line alone logit|: 0 -- all 67 lines bit-identical in both batchings (f64 sums of f32 partials are
# exact here, so the atomics' order does not show), hence the bound is exact equality.
MEASURED_LOGITS = 0.0
LOGIT_BOUND = 4.5 * MEASURED_LOGITS
# per-line "stats" against fp64 sums of the line's own bf16 pre-BN values (relative to sum |x| resp. sum x^2), and "bn" scale /
# shift against the fp64 finalize of those sums (relative to |scale| resp. |shift| + |mean * scale|): largest over the four shapes
MEASURED_STATS, MEASURED_BN = 1.37e-7, 2.75e-6
STATS_BOUND, BN_BOUND = 4.5 * MEASURED_STATS, 4.5 * MEASURED_BN


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _model(weights=None, seed=3):
    from lstm_ctc_ocr_b200 import engine, synthetic
    m = engine.CrnnModel(weight_decay=1e-5, device=DEV)
    m.load_params(weights if weights is not None else synthetic.init_params(seed, logits_scale=10.0))
    return m


def _alone(m, data, w, t):
    """crnn_forward of one line fed alone: logits [w/4-1, 64]."""
    d = torch.tensor(np.ascontiguousarray(data[None, :w]), device=DEV)
    return m.forward(d, torch.tensor([t], dtype=torch.int32, device=DEV))[:, 0]


def _packed(m, lines, idx):
    from lstm_ctc_ocr_b200.lib.lstm.test import pack_lines
    data, lw, tsl = pack_lines([lines[i] for i in idx])
    d = lambda a: torch.tensor(a, device=DEV)  # noqa: E731
    return m.forward_lines(d(data), d(lw), d(tsl)), tsl


# ------------------------------------------------------------------------------------------------ 1. line-alone equality
def test_packed_equals_line_alone_on_evaluation_lines(monkeypatch):
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from oracle import crnn_oracle as O
    we = _load("test_gpu_width_edges", "tests", "test_gpu_width_edges.py")
    margin = _load("test_gpu_decode10k", "tests", "test_gpu_decode10k.py").MARGIN
    mk = _load("make_decode10k", "tests", "golden", "make_decode10k.py")
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    weights = mk.load_weights()
    lines = we._eval_inputs()
    m = _model(weights)
    alone = [_alone(m, d[0], d.shape[1], int(t[0])) for d, t in lines]
    p32 = O.to_torch({k: v.astype(np.float32) for k, v in weights.items()}, torch.float32)
    ck = Checker("packed_eval", {}, REPORT)
    for batching in ("one_batch", "batches_of_7"):
        n = len(lines)
        groups = [list(range(n))] if batching == "one_batch" else [list(range(i, min(i + 7, n))) for i in range(0, n, 7)]
        identical = 0
        worst = 0.0
        dec_alone_eq = {"greedy": 0, "beam": 0}
        oracle_eq = {"greedy": 0, "beam": 0}
        clear_lines = 0
        for g in groups:
            logits, tsl = _packed(m, lines, g)
            d_tsl = torch.tensor(tsl, device=DEV)
            go, gl = engine.ctc_greedy(logits, d_tsl)
            bo, bl, _ = engine.ctc_beam_search_device(logits, d_tsl, beam_width=100)
            for r, i in enumerate(g):
                t = int(tsl[r])
                a = alone[i][:t]
                p = logits[:t, r]
                if torch.equal(a, p):
                    identical += 1
                else:
                    worst = max(worst, float((a - p).abs().max() / a.abs().max().clamp_min(1e-30)))
                t1 = torch.tensor([t], dtype=torch.int32, device=DEV)
                ag, agl = engine.ctc_greedy(a[:, None].contiguous(), t1)
                ab, abl, _ = engine.ctc_beam_search_device(a[:, None].contiguous(), t1, beam_width=100)
                got_g, got_b = go[r, :gl[r]].tolist(), bo[r, :bl[r]].tolist()
                dec_alone_eq["greedy"] += int(got_g == ag[0, :agl[0]].tolist())
                dec_alone_eq["beam"] += int(got_b == ab[0, :abl[0]].tolist())
                data, tl = lines[i]
                lo = O.forward(p32, data, tl).numpy()
                if t > 0:
                    srt = np.sort(lo[:t, 0], axis=1)
                    mg = float((srt[:, -1] - srt[:, -2]).min())
                else:
                    mg = 99.0
                if mg > margin:
                    clear_lines += 1
                    hb, hbl, _ = engine.ctc_beam_search(lo, tl, beam_width=100, merge_repeated=True)
                    oracle_eq["greedy"] += int(got_g == O.greedy_decode(lo, tl)[0])
                    oracle_eq["beam"] += int(got_b == [int(v) for v in hb[0, :hbl[0]] if v != 0])
        ok = (worst <= LOGIT_BOUND and all(v == n for v in dec_alone_eq.values())
              and all(v == clear_lines for v in oracle_eq.values()))
        ck._record(f"line_alone/{batching}", 0.0 if ok else float("inf"), lines=n, bit_identical=identical, worst_rel=worst,
                   bound=LOGIT_BOUND, decode_equal_alone=dec_alone_eq, clear_margin_lines=clear_lines, oracle_equal=oracle_eq)
    ck.assert_ok()


# ------------------------------------------------------------------------------------------------ 2. every stage per line
SHAPES = {
    "W1024_mixed": (1024, [8, 12, 16, 32, 36, 100, 256, 260, 516, 1024]),
    "N1_narrow": (100, [36]),
    "N130": (260, None),
    "N1024_W256": (256, None),
}
ACTS = [("conv1", 2), ("conv2", 4), ("conv3_1", 4), ("conv3_2", 4), ("conv4_1", 4), ("a4a_pre", 4), ("a4b_pre", 4)]
EXACT = ("conv1", "conv2", "conv3_1", "conv3_2")


def _shape_lines(name, seed=11):
    W, widths = SHAPES[name]
    rng = np.random.default_rng(seed)
    if widths is None:
        N = 130 if name == "N130" else 1024
        widths = [int(v) for v in rng.integers(2, W // 4 + 1, size=N) * 4]
        widths[:4] = [8, W, W, 12]
        widths[4:8] = [64, 64, 64, 64]                # equal widths, different content
    data = np.zeros((len(widths), W, 32), np.float32)
    for i, w in enumerate(widths):
        data[i, :w] = rng.random((w, 32), dtype=np.float32)
    tsl = np.array([w // 4 - 1 for w in widths], np.int32)
    return W, np.array(widths, np.int32), data, tsl


@pytest.mark.parametrize("shape", list(SHAPES))
def test_every_stage_per_line(shape):
    from stage_check import ulp_bf16
    W, lw, data, tsl = _shape_lines(shape)
    N = len(lw)
    m = _model()
    d = lambda a: torch.tensor(a, device=DEV)  # noqa: E731
    m.forward_lines(d(data), d(lw), d(tsl))
    taps = {k: m.tap(k, N, W) for k, _ in ACTS + [("conv4_2", 4)]}
    stats = m.tap_raw("stats", N, W, lines=True).double()
    bn = m.tap_raw("bn", N, W, lines=True).double()
    torch.cuda.synchronize()
    ck = Checker(f"packed_stages/{shape}", {}, REPORT)
    # masked positions: exactly zero
    nonzero = {}
    for k, div in ACTS:
        t = taps[k]
        H = t.shape[1]
        h = torch.arange(H, device=DEV)[None, :]
        lim = torch.tensor(lw, device=DEV)[:, None] * H // W
        outside = (h >= lim).view(N, H, *([1] * (t.dim() - 2)))
        nonzero[k] = int((t * outside).ne(0).sum())
    ck._record("masked_zero", 0.0 if not any(nonzero.values()) else float("inf"), **nonzero)
    # per-line stats and bn against fp64 on each line's own pre-BN values
    gamma = {l: m.tensor(f"{l}/{l}/gamma").double() for l in ("conv4_1", "conv4_2")}
    beta = {l: m.tensor(f"{l}/{l}/beta").double() for l in ("conv4_1", "conv4_2")}
    err_s = err_b = 0.0
    for li, (lname, pre) in enumerate((("conv4_1", "a4a_pre"), ("conv4_2", "a4b_pre"))):
        x = taps[pre].double()                                       # [N, H2, 4, 512], zero past each line
        s1 = x.sum(dim=(1, 2))
        s2 = (x * x).sum(dim=(1, 2))
        cnt = torch.tensor(lw, device=DEV, dtype=torch.float64)[:, None]
        scale_s = (x * x).sum(dim=(1, 2)).clamp_min(1e-30)
        err_s = max(err_s, float(((stats[li, :, 0] - s1).abs() / x.abs().sum(dim=(1, 2)).clamp_min(1e-30)).max()),
                    float(((stats[li, :, 1] - s2).abs() / scale_s).max()))
        mean = s1 / cnt
        var = (s2 / cnt - mean * mean).clamp_min(0)
        inv = 1.0 / torch.sqrt(var + 1e-3)
        sc = gamma[lname] * inv
        sh = beta[lname] - mean * sc
        err_b = max(err_b, float(((bn[li, :, 0] - sc).abs() / sc.abs().clamp_min(1e-30)).max()),
                    float(((bn[li, :, 1] - sh).abs() / (sh.abs() + (mean * sc).abs()).clamp_min(1e-30)).max()))
    # f64 sums of f32 partials over 32 rows: a few f32 roundings of the partial sums; coefficients rounded to f32
    ck._record("stats_fp64", err_s / STATS_BOUND, rel=err_s, bound=STATS_BOUND)
    ck._record("bn_fp64", err_b / BN_BOUND, rel=err_b, bound=BN_BOUND)
    # each line against its own line-alone run (sampled at N = 1024)
    sample = list(range(N)) if N <= 130 else list(range(8)) + list(np.random.default_rng(1).choice(np.arange(8, N), 56, replace=False))
    mism = {k: 0 for k in taps}
    bn_alone_equal = 0
    for i in sample:
        w = int(lw[i])
        m.forward(d(np.ascontiguousarray(data[i:i + 1, :w])), d(tsl[i:i + 1]))
        for k in taps:
            a = m.tap(k, 1, w)[0]
            p = taps[k][i, :a.shape[0]]
            if k in EXACT:
                mism[k] += int(not torch.equal(a, p))
            else:
                mism[k] += int(bool(((a - p).abs() > ulp_bf16(torch.maximum(a.abs(), p.abs()))).any()))
        ba = m.tap_raw("bn", 1, w).double()
        bn_alone_equal += int(bool(((ba[:, :2] - bn[:, i, :2]).abs() <= 1e-6 * ba[:, :2].abs().clamp_min(1e-6)).all()))
    ck._record("line_alone_taps", 0.0 if not any(mism.values()) else float("inf"), lines=len(sample), **mism)
    ck._record("bn_line_alone", 0.0 if bn_alone_equal == len(sample) else float("inf"), equal=bn_alone_equal, lines=len(sample))
    if shape == "N1024_W256":
        # equal widths (lines 4..7, W_i = 64), different content: different coefficients, none the whole-batch forward's
        m.forward(d(data), d(tsl))
        whole = m.tap_raw("bn", N, W).double()
        eqw = [bool(torch.equal(bn[:, a, :2], bn[:, b, :2])) for a in range(4, 8) for b in range(a + 1, 8)]
        eqwhole = [bool(torch.allclose(bn[:, a, :2], whole[:, :2], rtol=1e-6, atol=0)) for a in range(4, 8)]
        ck._record("per_line_not_whole_batch", 0.0 if not any(eqw) and not any(eqwhole) else float("inf"),
                   equal_pairs=sum(eqw), equal_to_whole_batch=sum(eqwhole))
    ck.assert_ok()


# ------------------------------------------------------------------------------------------------ 3. interfaces
def _write_dir(path, n=70, seed=99):
    from PIL import Image
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    rng = random.Random(seed)
    for i in range(n):
        text = gen.gen_rand(rng, 4, 30)
        Image.fromarray(gen.render_line(text, rng=rng)).save(os.path.join(path, f"{i:04d}_{text}.png"))


def test_test_model_same_decodes_for_batch_sizes(tmp_path, monkeypatch):
    from lstm_ctc_ocr_b200.lib.lstm import test as T
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    mk = _load("make_decode10k", "tests", "golden", "make_decode10k.py")
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    _write_dir(str(tmp_path))
    weights = mk.load_weights()
    outs = {}
    old = cfg.TEST.BATCH_SIZE
    try:
        for bs in (1, 64):
            cfg.TEST.BATCH_SIZE = bs
            net = get_network("LSTM_test")
            with Session(device=DEV) as sess:
                sess.assign(net, weights)
                sw = T.SolverWrapper(sess, net, None, str(tmp_path), None)
                buf = io.StringIO()
                with redirect_stdout(buf):
                    sw.test_model(sess, testDir=str(tmp_path), restore=False)
            text = buf.getvalue().splitlines()
            outs[bs] = ([ln for ln in text if ln.strip().startswith("res:") or ln.endswith(".png") or ".png cost" in ln or "res:" in ln],
                        [ln for ln in text if ln.startswith("total acc")])
    finally:
        cfg.TEST.BATCH_SIZE = old
    strip = lambda ls: [ln.split(" cost time")[0] if "cost time" in ln else ln for ln in ls]  # noqa: E731
    assert strip(outs[1][0]) == strip(outs[64][0])
    assert outs[1][1] == outs[64][1] and len(outs[1][1]) == 1
    assert sum("cost time" in ln for ln in outs[64][0]) == 70


def test_session_run_with_line_width(monkeypatch):
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.test import pack_lines, prepare_line
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.session import Session
    from lstm_ctc_ocr_b200 import synthetic
    rng = np.random.default_rng(5)
    lines = [prepare_line(rng.integers(0, 256, size=(32, w), dtype=np.uint8)) for w in (30, 90, 200, 9)]
    data, lw, tsl = pack_lines(lines)
    params = synthetic.init_params(3, logits_scale=10.0)
    old = cfg.get("DECODER", "greedy")
    try:
        net = get_network("LSTM_test")
        with Session(device=DEV) as sess:
            sess.assign(net, params)
            eng = sess.engine_for(net)
            for decoder in ("greedy", "beam"):
                cfg.DECODER = decoder
                packed = sess.run(Fetch(net, "dense_decoded"), {net.data: data, net.line_width: lw, net.time_step_len: tsl})
                for i, (d1, t1) in enumerate(lines):
                    alone = sess.run(Fetch(net, "dense_decoded"), {net.data: d1, net.time_step_len: t1})
                    assert [v for v in packed[i] if v] == [v for v in alone[0] if v], (decoder, i)
            with pytest.raises(ValueError):
                sess.run(Fetch(net, "dense_decoded"), {net.data: data, net.line_width: lw,
                                                       net.time_step_len: tsl + np.array([2, 0, 0, 0], np.int32)})
            assert not eng.training
        tnet = get_network("LSTM_train")
        with Session(device=DEV) as sess:
            sess.assign(tnet, params)
            lab = np.array([1, 2, 3, 4], np.int32)
            ll = np.array([1, 1, 1, 1], np.int32)
            feed = {tnet.data: data, tnet.line_width: lw, tnet.time_step_len: tsl, tnet.labels: lab, tnet.labels_len: ll}
            loss, costs = sess.run([Fetch(tnet, "loss"), Fetch(tnet, "ctc_costs")], feed)
            assert np.isfinite(loss) and costs.shape == (4,)
            with pytest.raises(ValueError):
                sess.run([Fetch(tnet, "train_op")], feed)
    finally:
        cfg.DECODER = old


def test_status_codes_and_untouched_outputs():
    from lstm_ctc_ocr_b200 import _lib, engine, synthetic
    lib = _lib.load()
    N, W = 2, 64
    data = torch.rand((N, W, 32), device=DEV)
    lw = torch.tensor([64, 32], dtype=torch.int32, device=DEV)
    tsl = torch.tensor([15, 7], dtype=torch.int32, device=DEV)
    out = torch.full((W // 4 - 1, N, 64), 7.0, device=DEV)
    nbytes = _lib.c_size_t()
    m = _model()
    assert lib.crnn_lines_workspace_size(m.handle, N, W, nbytes) == 0
    plain = _lib.c_size_t()
    assert lib.crnn_model_workspace_size(m.handle, N, W, 0, plain) == 0 and nbytes.value > plain.value
    ws = torch.empty(nbytes.value + 1024, dtype=torch.uint8, device=DEV)
    wp = (ws.data_ptr() + 1023) // 1024 * 1024
    m.set_training(True)
    st = lib.crnn_forward_lines(m.handle, data.data_ptr(), lw.data_ptr(), tsl.data_ptr(), N, W, out.data_ptr(), wp, nbytes.value,
                                torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert st == 1 and bool((out == 7.0).all())                       # CRNN_INVALID_VALUE
    for cd in ("f32", "tf32"):
        mx = engine.CrnnModel(device=DEV, compute_dtype=cd)
        mx.load_params(synthetic.init_params(3))
        assert lib.crnn_lines_workspace_size(mx.handle, N, W, nbytes) == 4
        st = lib.crnn_forward_lines(mx.handle, data.data_ptr(), lw.data_ptr(), tsl.data_ptr(), N, W, out.data_ptr(), wp,
                                    ws.numel() - 1024, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert st == 4 and bool((out == 7.0).all())                   # CRNN_UNSUPPORTED
    m2 = _model()
    assert lib.crnn_forward_lines(m2.handle, data.data_ptr(), lw.data_ptr(), tsl.data_ptr(), N, W + 2, out.data_ptr(), wp,
                                  ws.numel() - 1024, 0) == 1
    # widths are clamped on the device: 4 -> 8, 100 -> W
    got = m2.forward_lines(data, torch.tensor([100, 4], dtype=torch.int32, device=DEV), torch.tensor([15, 1], dtype=torch.int32, device=DEV))
    ref = m2.forward_lines(data, torch.tensor([64, 8], dtype=torch.int32, device=DEV), torch.tensor([15, 1], dtype=torch.int32, device=DEV))
    assert torch.equal(got[:15, 0], ref[:15, 0]) and torch.equal(got[:1, 1], ref[:1, 1])
