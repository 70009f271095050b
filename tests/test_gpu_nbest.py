"""The n-best beam-search decoder on the device (crnn_ctc_beam_search_topk_device, csrc/beam.cu) against the host decoder
(crnn_ctc_beam_search_topk, csrc/beam.cpp): identical labels, lengths and num_paths, log-probabilities within one f32 ulp,
path 0 bit for bit the single-best device decode; the exact prefix-search checks of tests/nbest_refs.py run on device decodes;
a gated non-blocking stream; the "beam_decoded" fetch on every feed; test_model with TEST.TOP_PATHS 5."""
import importlib.util
import io
import os
import re
import sys
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import beam_refs as BR  # noqa: E402
import nbest_refs as NR  # noqa: E402


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


CPU = _load("test_nbest_cpu", "tests", "test_nbest_cpu.py")


def _ulp_equal(a, b):
    a = np.asarray(a, np.float32); b = np.asarray(b, np.float32)
    ia = a.view(np.int32).astype(np.int64); ib = b.view(np.int32).astype(np.int64)
    return bool(np.all((a == b) | ((np.sign(a) == np.sign(b)) & (np.abs(ia - ib) <= 1))))


def _both(x, il, width, K, merge_repeated=True, strip=0):
    """Device and host top-k of the same logits: asserts identical outputs and returns the device's (numpy)."""
    from lstm_ctc_ocr_b200 import engine
    x = np.ascontiguousarray(x, np.float32)
    il = np.asarray(il, np.int32)
    d = [a.cpu().numpy() for a in engine.ctc_beam_search_topk_device(torch.tensor(x, device=DEV), torch.tensor(il, device=DEV),
                                                                     beam_width=width, top_paths=K, merge_repeated=merge_repeated,
                                                                     strip=strip)]
    h = engine.ctc_beam_search_topk(x, il, beam_width=width, top_paths=K, merge_repeated=merge_repeated, strip=strip)
    key = (x.shape, width, K, merge_repeated, strip)
    assert np.array_equal(d[0], h[0]), key                     # labels and zero padding
    assert np.array_equal(d[1], h[1]) and np.array_equal(d[3], h[3]), key
    assert _ulp_equal(d[2], h[2]), key
    return d


def _path0_is_the_single_best(x, il, width, d, merge_repeated=True, strip=0):
    from lstm_ctc_ocr_b200 import engine
    xt = x if torch.is_tensor(x) else torch.tensor(np.ascontiguousarray(x, np.float32), device=DEV)
    ilt = il if torch.is_tensor(il) else torch.tensor(np.asarray(il, np.int32), device=DEV)
    o, ol, nlp = (a.cpu().numpy() for a in engine.ctc_beam_search_device(xt, ilt, beam_width=width, merge_repeated=merge_repeated,
                                                                          strip=strip))
    assert np.array_equal(d[0][:, 0], o) and np.array_equal(d[1][:, 0], ol)
    assert np.array_equal((-d[2][:, 0]).view(np.int32), nlp.view(np.int32))


@pytest.mark.parametrize("width", [1, 2, 33, 100, 128])
def test_device_topk_equals_host_on_the_cpu_grid(width):
    for name, x, il in CPU._grid_cases():
        for K in sorted({1, min(2, width), min(7, width), width}):
            for merge, strip in ((True, 0), (False, -1)):
                d = _both(x, il, width, K, merge, strip)
                _path0_is_the_single_best(x, il, width, d, merge, strip)
    for name, x, il in CPU._pruned_and_blank_free_cases():
        d = _both(x, il, width, width, False, -1)
        bad, _ = NR.check_lower_bound_topk(x, il, [[d[0][n, k, :d[1][n, k]].tolist() for k in range(width)] for n in range(len(il))],
                                           d[2], d[3])
        assert not bad, (name, width, bad[:3])


def test_device_topk_equals_host_on_trained_logits():
    """The trained fixture weights at C3 (T = 63, N = 1024), widths 100 and 128, K 1, 10 and 100."""
    from lstm_ctc_ocr_b200 import engine, synthetic
    mk = _load("make_decode10k", "tests", "golden", "make_decode10k.py")
    data, _, _, tsl = synthetic.synth_batch(1024, 256, seed=5)
    m = engine.CrnnModel(weight_decay=1e-5, device=DEV)
    m.load_params(mk.load_weights())
    d_tsl = torch.tensor(tsl, dtype=torch.int32, device=DEV)
    x = m.forward(torch.tensor(data, dtype=torch.float32, device=DEV), d_tsl)
    torch.cuda.synchronize()
    xh = x.cpu().numpy()
    for width in (100, 128):
        for K in (1, 10, 100):
            d = _both(xh, tsl, width, K)
            _path0_is_the_single_best(x, d_tsl, width, d)
            assert np.all(d[3] >= 1) and np.all(d[3] <= K)


def test_device_topk_against_exact_prefix_search():
    def device_topk(x, il, width, K, merge, strip):
        from lstm_ctc_ocr_b200 import engine
        o, ol, lp, npaths = (a.cpu().numpy() for a in engine.ctc_beam_search_topk_device(
            torch.tensor(x, device=DEV), torch.tensor(il, device=DEV), beam_width=width, top_paths=K, merge_repeated=merge, strip=strip))
        return [[o[n, k, :ol[n, k]].tolist() for k in range(K)] for n in range(len(il))], lp, npaths
    st, bad = NR.run_exhaustive_topk(device_topk, NR.exhaustive_topk_cases())
    print(st)
    assert not bad, bad[:5]
    assert st["decided"] > 50_000, st


def test_device_topk_on_a_gated_non_blocking_stream():
    """Outputs and arena poisoned on a fresh non-blocking stream gated behind a sleep, the legacy stream busy for longer: the
    decode, read on the side stream alone, equals the one on the default stream."""
    from lstm_ctc_ocr_b200 import engine
    ST = _load("test_gpu_streams", "tests", "test_gpu_streams.py")
    x, il = BR.dense_case(17, 19, 64, seed=3)
    d_x, d_il = torch.tensor(x, device=DEV), torch.tensor(il, device=DEV)
    src_x, src_il = d_x.clone(), d_il.clone()
    engine.ctc_beam_search_topk_device(d_x, d_il, beam_width=100, top_paths=10)          # the workspace, allocated once
    ws = engine._beam_ws[torch.device(DEV)][1]

    def call():
        o, ol, lp, npaths = engine.ctc_beam_search_topk_device(d_x, d_il, beam_width=100, top_paths=10)
        return {"out": o.clone(), "len": ol.clone(), "log_prob": lp.clone(), "num_paths": npaths.clone()}
    ref = call()
    torch.cuda.synchronize()
    got, _ = ST._window(call, [(d_x, src_x), (d_il, src_il)], [ws], call_ms=5.0)
    for k in ref:
        assert torch.equal(got[k], ref[k]), k


def _check_beam_fetch(logits, tsl, bd, width, K):
    from lstm_ctc_ocr_b200 import engine
    o, ol, lp, npaths = engine.ctc_beam_search_topk(logits, tsl, beam_width=width, top_paths=K)
    L = bd["labels"].shape[2]
    assert L == int(ol.max())
    assert np.array_equal(bd["labels"], o[:, :, :L]) and not o[:, :, L:].any()
    assert np.array_equal(bd["len"], ol) and np.array_equal(bd["num_paths"], npaths)
    assert _ulp_equal(bd["log_prob"], lp)


def test_beam_decoded_fetch_on_every_feed(tmp_path, monkeypatch):
    from lstm_ctc_ocr_b200 import synthetic
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.test import load_line_image, pack_lines, prepare_line
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.session import Session
    mk = _load("make_decode10k", "tests", "golden", "make_decode10k.py")
    pe = _load("test_gpu_packed_eval", "tests", "test_gpu_packed_eval.py")
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    pe._write_dir(str(tmp_path), n=12)
    images = [load_line_image(os.path.join(tmp_path, f)) for f in sorted(os.listdir(tmp_path))]
    data, _, _, tsl = synthetic.synth_batch(32, 128, seed=9)
    u8 = np.clip(np.round(data * 255), 0, 255).astype(np.uint8)
    old = (cfg.TEST.TOP_PATHS, cfg.BEAM_WIDTH, cfg.DECODER)
    try:
        for width, K in ((100, 5), (33, 33)):
            cfg.TEST.TOP_PATHS, cfg.BEAM_WIDTH = K, width
            net = get_network("LSTM_test")
            with Session(device=DEV) as sess:
                sess.assign(net, mk.load_weights())
                fl = [Fetch(net, "logits"), Fetch(net, "beam_decoded")]
                for feed in ({net.data: data, net.time_step_len: tsl}, {net.data_u8: u8, net.time_step_len: tsl}):
                    x, bd = sess.run(fl, feed)
                    assert sess.d2h_bytes == x.nbytes + sum(a.nbytes for a in bd.values())
                    _check_beam_fetch(x, feed[net.time_step_len], bd, width, K)
                    cfg.DECODER = "beam"
                    dense = sess.run(Fetch(net, "dense_decoded"), feed)
                    cfg.DECODER = old[2]
                    assert np.array_equal(dense, bd["labels"][:, 0, :dense.shape[1]])
                lines = [prepare_line(im) for im in images]
                pdata, lw, ptsl = pack_lines(lines)
                x, bd = sess.run(fl, {net.data: pdata, net.line_width: lw, net.time_step_len: ptsl})
                _check_beam_fetch(x, ptsl, bd, width, K)
                x2, bd2 = sess.run(fl, {net.images: images})
                _check_beam_fetch(x2, ptsl, bd2, width, K)
                assert sess.d2h_bytes == x2.nbytes + sum(a.nbytes for a in bd2.values())
    finally:
        cfg.TEST.TOP_PATHS, cfg.BEAM_WIDTH, cfg.DECODER = old


def test_test_model_prints_the_n_best_reads(tmp_path, monkeypatch):
    """TEST.TOP_PATHS 5 with the beam decoder: every line's first n-best read is its read, and the accuracy is the one
    TOP_PATHS 1 prints."""
    from lstm_ctc_ocr_b200.lib.lstm import test as T
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    mk = _load("make_decode10k", "tests", "golden", "make_decode10k.py")
    pe = _load("test_gpu_packed_eval", "tests", "test_gpu_packed_eval.py")
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    pe._write_dir(str(tmp_path), n=40)
    outs = {}
    old = (cfg.TEST.TOP_PATHS, cfg.DECODER)
    try:
        cfg.DECODER = "beam"
        for K in (1, 5):
            cfg.TEST.TOP_PATHS = K
            net = get_network("LSTM_test")
            with Session(device=DEV) as sess:
                sess.assign(net, mk.load_weights())
                buf = io.StringIO()
                with redirect_stdout(buf):
                    T.SolverWrapper(sess, net, None, str(tmp_path), None).test_model(sess, testDir=str(tmp_path), restore=False)
            outs[K] = [ln for ln in buf.getvalue().splitlines() if "res:" in ln or ln.startswith("total acc")]
    finally:
        cfg.TEST.TOP_PATHS, cfg.DECODER = old
    assert outs[1][-1] == outs[5][-1]
    res = [ln for ln in outs[5] if "res:" in ln]
    assert len(res) == 40
    pat = re.compile(r"^    res: (\S*), n-best: (\S*) \((\d\.\d{4})\)(, \S* \(\d\.\d{4}\)){0,4}(, margin: \S+)?$")
    for a, b in zip([ln for ln in outs[1] if "res:" in ln], res):
        m = pat.match(b)
        assert m, b
        assert m.group(1) == m.group(2) and a == "    res: " + m.group(1), (a, b)
