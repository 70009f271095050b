"""CTC forced alignment (crnn_ctc_align) on the GPU against the fp64 restatement of tests/align_refs.py.

Per utterance: spans valid (ordered, non-empty, disjoint, inside [0, T_n), a gap between equal neighbours); the GPU's own path,
rescored in fp64, within eps(P_gpu) + eps(P_opt) of the reference optimum and within eps(P_gpu) of the returned path_logprob;
spans equal to the reference's wherever its margin exceeds 2 * max(eps(P_gpu), eps(P_opt)); peak within the f32 softmax
bound of the fp64 y over the GPU's span.  The eps are the analytic bounds of align_refs.  Infeasible labellings give -inf,
invalid ones NaN, both with spans -1 and peaks 0.  End to end on the decode-10k fixture: greedy reads align on their argmax
runs, label and read alignments agree on correct reads, beam reads align, packed lines align as if alone, test_model prints
the confidence fields only when asked.  Counts go to build/align_report.jsonl."""
import importlib.util
import io
import json
import os
import sys
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import align_refs as A  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _report(**row):
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    with open(os.path.join(ROOT, "build", "align_report.jsonl"), "a") as f:
        f.write(json.dumps(row) + "\n")


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _t(a, dt=torch.int32):
    return torch.tensor(np.asarray(a), dtype=dt, device=DEV)


def _align(x, lab, ll, il, blank=0, max_label_len=None, **kw):
    from lstm_ctc_ocr_b200 import engine
    r = engine.ctc_align(x, lab, ll, il, blank=blank, max_label_len=max_label_len, **kw)
    torch.cuda.synchronize()
    return [a.cpu().numpy() for a in r]


def _rows(a, ll, dense):
    """Per-utterance slices of a flat or dense output."""
    out, off = [], 0
    for n, L in enumerate(ll):
        L = max(int(L), 0)
        out.append(a[n, :L] if dense else a[off:off + L])
        off += 0 if dense else L
    return out


def check(name, x, labels, ll, il, blank=0, max_label_len=None):
    """Run the kernel on x [T, N, 64] (cuda f32) with labels (numpy, flat or dense) and check every utterance against the
    reference.  Returns the statistics recorded in the report."""
    labels, ll, il = np.asarray(labels, np.int32), np.asarray(ll, np.int32), np.asarray(il, np.int32)
    dense = labels.ndim == 2
    st, en, pk, lp = _align(x, _t(labels), _t(ll), _t(il), blank, max_label_len)
    R = A.align_fp64(x.cpu().numpy(), labels, ll, il, blank, max_label_len if max_label_len is not None else
                     (labels.shape[1] if dense else None))
    S_, E_, P_ = _rows(st, ll, dense), _rows(en, ll, dense), _rows(pk, ll, dense)
    stats = dict(case=name, lines=len(ll), aligned=0, compared_spans=0, equal_spans=0, infeasible=0, invalid=0,
                 worst_score_over_eps=0.0, worst_peak_over_bound=0.0)
    rows = A.to_rows(labels, ll)
    for n in range(len(ll)):
        if dense:                                           # dense rows are written in full: padding past L
            L = max(int(ll[n]), 0) if R["valid"][n] else 0
            assert (st[n, L:] == -1).all() and (en[n, L:] == -1).all() and (pk[n, L:] == 0).all(), (name, n)
        if not R["valid"][n]:
            stats["invalid"] += 1
            assert np.isnan(lp[n]), (name, n)
            assert (S_[n] == -1).all() and (E_[n] == -1).all() and (P_[n] == 0).all()
            continue
        if not R["feasible"][n]:
            stats["infeasible"] += 1
            assert lp[n] == -np.inf, (name, n, lp[n])
            assert (S_[n] == -1).all() and (E_[n] == -1).all() and (P_[n] == 0).all()
            continue
        Tn, L, seq = R["Tn"][n], R["L"][n], rows[n]
        if Tn == 0:
            assert lp[n] == 0.0
            continue
        s, e = S_[n].astype(np.int64), E_[n].astype(np.int64)
        assert ((s >= 0) & (s < e) & (e <= Tn)).all(), (name, n, s, e)
        assert (e[:-1] <= s[1:]).all(), (name, n)
        eq = np.array([seq[k] == seq[k + 1] for k in range(L - 1)], bool)
        assert (e[:-1][eq] < s[1:][eq]).all(), (name, n, "no blank between equal labels")
        ext = R["ext"][n]
        path = A.path_of_spans(s, e, Tn)
        ev = R["lp"][np.arange(Tn), n, ext[path]]
        errv = R["err"][np.arange(Tn), n, ext[path]]
        resc = float(ev.sum())
        eg, er = A.path_eps(ev, errv), R["eps"][n]
        ref = R["score"][n]
        assert abs(resc - ref) <= eg + er, (name, n, resc, ref, eg, er)
        assert abs(resc - float(lp[n])) <= eg, (name, n, resc, float(lp[n]), eg)
        stats["worst_score_over_eps"] = max(stats["worst_score_over_eps"], abs(resc - float(lp[n])) / eg)
        if R["margin"][n] > 2 * max(eg, er):
            stats["compared_spans"] += 1
            assert np.array_equal(s, R["start"][n]) and np.array_equal(e, R["end"][n]), (name, n)
        stats["equal_spans"] += int(np.array_equal(s, R["start"][n]) and np.array_equal(e, R["end"][n]))
        y = np.exp(R["lp"][:Tn, n])
        for k in range(L):
            yk = y[s[k]:e[k], seq[k]]
            bound = yk.max() * A.peak_rel_err(R["err"][s[k]:e[k], n, seq[k]].max())
            d = abs(float(P_[n][k]) - yk.max())
            assert d <= bound, (name, n, k, float(P_[n][k]), yk.max(), bound)
            stats["worst_peak_over_bound"] = max(stats["worst_peak_over_bound"], d / bound if bound else 0.0)
        stats["aligned"] += 1
    _report(**stats)
    return stats


def _random(T, N, seed, scale=3.0):
    rng = np.random.default_rng(seed)
    return torch.tensor(rng.normal(0, scale, size=(T, N, 64)).astype(np.float32), device=DEV), rng


def _draw(rng, L, blank):
    """L ids uniform over [0, 64) minus the blank."""
    v = rng.integers(0, A.C - 1, size=int(L))
    return v + (v >= blank)


def _labels(rng, lens, blank=0):
    return np.concatenate([np.zeros(0, np.int64)] + [_draw(rng, L, blank) for L in lens]).astype(np.int32)


# ------------------------------------------------------------------------------------------------------------- shapes
def test_model_logits_c3():
    """Logits of the model at C3 (W = 256: T = 63, N = 1024), the batch's own labels."""
    from lstm_ctc_ocr_b200 import engine, synthetic
    params = synthetic.init_params(3, logits_scale=10.0)
    data, lab, ll, tsl = synthetic.synth_batch(1024, 256, seed=5)
    m = engine.CrnnModel(weight_decay=1e-5, device=DEV)
    m.load_params(params)
    x = m.forward(_t(data, torch.float32), _t(tsl))
    st = check("c3_model", x, lab, ll, tsl)
    assert st["aligned"] == 1024


@pytest.mark.parametrize("T", [1, 2, 3])
def test_few_frames(T):
    x, rng = _random(T, 12, 100 + T)
    ll = np.array([0, 1, 1, 2, 2, 3, 1, 2, 0, 1, 2, 4], np.int32)
    il = np.array([T, T, 1, T, 2, T, 0, T + 5, 0, T, 1, T], np.int32)
    lab = _labels(rng, ll)
    lab[3:5] = 9                                            # an equal pair: needs 3 frames
    check(f"T{T}", x, lab, ll, il)


@pytest.mark.parametrize("L", [64, 255, 639])
def test_long_lines(L):
    T = 2048
    x, rng = _random(T, 4, 200 + L)
    ll = np.array([L, L, L // 2, L], np.int32)
    il = np.array([T, 2 * L + 1, T - 7, L], np.int32)        # the last is feasible only without equal neighbours
    lab = _labels(rng, ll)
    st = check(f"long_L{L}", x, lab, ll, il, max_label_len=L)
    assert st["aligned"] + st["infeasible"] == 4


def test_empty_labels_and_lengths():
    T = 20
    x, rng = _random(T, 8, 300)
    ll = np.zeros(8, np.int32)
    il = np.array([0, 1, T, T + 5, -3, 7, T, 0], np.int32)
    st = check("L0", x, np.zeros(0, np.int32), ll, il, max_label_len=0)
    assert st["aligned"] == 5                                 # T_n > 0
    _, _, _, lp = _align(x, _t(np.zeros(0, np.int32)), _t(ll), _t(il), max_label_len=0)
    assert lp[0] == 0.0 and lp[4] == 0.0
    lps, _ = A.log_softmax(x.cpu().numpy())
    assert abs(lp[2] - lps[:, 2, 0].sum()) < 1e-3


def test_repeats_infeasible_and_invalid():
    T = 16
    x, rng = _random(T, 10, 400)
    ll = np.array([8, 8, 9, 4, 3, 3, 3, 2, 70, -1], np.int32)
    il = np.array([T, 15, T, 3, T, T, T, T, T, T], np.int32)
    parts = [[5] * 8, [5] * 8, [5] * 9, [1, 2, 3, 4], [1, 64, 2], [1, -1, 2], [1, 0, 2], [3, 3], list(range(1, 71)), []]
    lab = np.array([v for p in parts for v in p], np.int32)
    st = check("repeats_infeasible_invalid", x, lab, ll, il, max_label_len=64)
    # 8 fives need 15 frames: 16 feasible, 15 feasible; 9 fives need 17: infeasible; 4 labels in 3 frames: infeasible
    assert st["infeasible"] == 2 and st["invalid"] == 5, st


@pytest.mark.parametrize("blank", [0, 17, 63])
def test_blanks_and_layouts_give_the_same_bits(blank):
    T, N = 80, 64
    x, rng = _random(T, N, 500 + blank, scale=4.0)
    ll = rng.integers(0, 30, size=N).astype(np.int32)
    il = rng.integers(20, T + 1, size=N).astype(np.int32)
    lab = np.concatenate([_draw(rng, L, blank) for L in ll]).astype(np.int32)
    lab[:4] = lab[0]
    check(f"blank{blank}_flat", x, lab, ll, il, blank=blank)
    dense = np.full((N, 40), 7, np.int32)
    off = np.r_[0, np.cumsum(ll)]
    for n in range(N):
        dense[n, :ll[n]] = lab[off[n]:off[n + 1]]
    check(f"blank{blank}_dense", x, dense, ll, il, blank=blank, max_label_len=40)
    f = _align(x, _t(lab), _t(ll), _t(il), blank, 40)
    d = _align(x, _t(dense), _t(ll), _t(il), blank, 40)
    assert np.array_equal(f[3].view(np.int32), d[3].view(np.int32))
    for a, b in zip(f[:3], d[:3]):
        assert all(np.array_equal(p.view(np.int32), q.view(np.int32)) for p, q in zip(_rows(a, ll, False), _rows(b, ll, True)))


# ------------------------------------------------------------------------------------------------------------- determinism
def test_prefilled_outputs_repeat_runs_and_offset_logits_give_the_same_bits():
    from lstm_ctc_ocr_b200 import engine
    T, N = 300, 96
    x, rng = _random(T, N, 600)
    ll = rng.integers(0, 100, size=N).astype(np.int32)
    il = rng.integers(1, T + 1, size=N).astype(np.int32)
    lab = _labels(rng, ll)
    m = int(ll.max())
    d_lab, d_ll, d_il = _t(lab), _t(ll), _t(il)
    nbytes = engine.ctc_align_workspace_bytes(T, N, 64, m)

    def run(fill, logits, ws_off=0):
        ws = torch.full((nbytes + 64,), fill, dtype=torch.uint8, device=DEV)
        outs = [torch.full(lab.shape, -1 if fill else 0, dtype=dt, device=DEV) for dt in (torch.int32, torch.int32)]
        outs.append(torch.full(lab.shape, float("nan") if fill else 0.0, device=DEV))
        lp = torch.full((N,), float("nan") if fill else 0.0, device=DEV)
        from lstm_ctc_ocr_b200 import _lib
        _lib.check(_lib.load().crnn_ctc_align(logits.data_ptr(), d_lab.data_ptr(), 0, d_ll.data_ptr(), d_il.data_ptr(), T, N, 64, 0, m,
                                              outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), lp.data_ptr(),
                                              ws.data_ptr() + ws_off, nbytes, torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        return [o.cpu().numpy().view(np.int32) for o in outs + [lp]]

    ref = run(0, x)
    shifted = torch.empty(x.numel() + 1, device=DEV)
    shifted[1:] = x.reshape(-1)
    for got in (run(0xFF, x), run(0, x), run(0xFF, shifted[1:].view(T, N, 64), ws_off=4)):
        assert all(np.array_equal(a, b) for a, b in zip(ref, got))


def test_status_codes_leave_the_outputs_untouched():
    from lstm_ctc_ocr_b200 import _lib, engine
    lib = _lib.load()
    T, N, m = 40, 8, 10
    x, rng = _random(T, N, 700)
    ll = np.full(N, m, np.int32)
    lab, d_ll, d_il = _t(_labels(rng, ll)), _t(ll), _t(np.full(N, T, np.int32))
    need = engine.ctc_align_workspace_bytes(T, N, 64, m)
    ws = torch.zeros(need, dtype=torch.uint8, device=DEV)
    outs = [torch.full((N * m,), 123, dtype=torch.int32, device=DEV) for _ in range(2)] + [torch.full((N * m,), 5.0, device=DEV)]
    lp = torch.full((N,), 5.0, device=DEV)
    st = torch.cuda.current_stream().cuda_stream

    def call(C=64, mll=m, nbytes=need, start=None, logits=None):
        return lib.crnn_ctc_align(x.data_ptr() if logits is None else logits, lab.data_ptr(), 0, d_ll.data_ptr(), d_il.data_ptr(),
                                  T, N, C, 0, mll, outs[0].data_ptr() if start is None else start, outs[1].data_ptr(),
                                  outs[2].data_ptr(), lp.data_ptr(), ws.data_ptr(), nbytes, st)

    assert call(C=65) == 4
    assert call(mll=640) == 4
    assert call(nbytes=need - 1) == 5
    assert call(start=0) == 1
    assert call(logits=0) == 1
    torch.cuda.synchronize()
    assert (outs[0] == 123).all() and (outs[1] == 123).all() and (outs[2] == 5.0).all() and (lp == 5.0).all()
    assert call() == 0
    torch.cuda.synchronize()
    assert torch.isfinite(lp).all() and not (outs[0] == 123).any()


# ------------------------------------------------------------------------------------------------------------- end to end
def _argmax_ok(x, Tn):
    """Greedy-read property preconditions on x [T, 64]: no frame's argmax is 63, no frame has a tied maximum."""
    xs = np.sort(x[:Tn], axis=1)
    return not (np.argmax(x[:Tn], axis=1) == 63).any() and not (xs[:, -1] == xs[:, -2]).any()


def test_decode10k_read_and_label_alignment():
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.session import Session
    mk = _load("make_decode10k", "tests", "golden", "make_decode10k.py")
    if not os.path.exists(os.path.join(ROOT, "tests", "golden", "decode10k_oracle.npz")):
        pytest.skip("fixture missing: run tests/golden/make_decode10k.py")
    weights = mk.load_weights()
    s = mk.sampler()
    net = get_network("LSTM_train")
    fetch = [Fetch(net, "logits"), Fetch(net, "read_alignment"), Fetch(net, "label_alignment")]
    st = dict(lines=0, argmax_lines=0, correct=0, beam_lines=0)
    old = cfg.get("DECODER", "greedy")
    try:
        with Session(device=DEV) as sess:
            sess.assign(net, weights)
            for k in range(mk.NBATCH):
                imgs, lab, ll, tsl = s.batch(k)
                feed = {net.data: np.stack(imgs), net.time_step_len: np.asarray(tsl, np.int32),
                        net.labels: np.asarray(lab, np.int32), net.labels_len: np.asarray(ll, np.int32)}
                cfg.DECODER = "greedy"
                x, rd, la = sess.run(fetch, feed)
                lps, lse = A.log_softmax(x)
                err = A.emission_err(lse[..., None], lps)
                truth = A.to_rows(lab, ll)
                for n in range(x.shape[1]):
                    st["lines"] += 1
                    Tn = int(tsl[n])
                    L = int((rd["labels"][n] != 0).sum())
                    read = [int(v) for v in rd["labels"][n, :L]]
                    if _argmax_ok(x[:, n], Tn):
                        st["argmax_lines"] += 1
                        r, s0, e0 = A.argmax_runs(x[:, n], Tn)
                        assert r == read
                        assert np.array_equal(rd["start"][n, :L], s0) and np.array_equal(rd["end"][n, :L], e0), (k, n)
                        am = np.argmax(x[:Tn, n], axis=1)
                        ev = lps[np.arange(Tn), n, am]
                        assert abs(float(rd["path_logprob"][n]) - ev.sum()) <= A.path_eps(ev, err[np.arange(Tn), n, am]), (k, n)
                    assert np.array_equal(rd["x0"][n, :L], 4 * rd["start"][n, :L]) and np.array_equal(rd["x1"][n, :L], 4 * rd["end"][n, :L] + 4)
                    if read == truth[n]:
                        st["correct"] += 1
                        for key in ("labels", "start", "end", "x0", "x1", "peak"):
                            assert np.array_equal(la[key][n, :L].view(np.int32), rd[key][n, :L].view(np.int32)), (k, n, key)
                        assert la["path_logprob"][n].view(np.int32) == rd["path_logprob"][n].view(np.int32)
                if k < 4:                                   # beam: 2048 lines
                    cfg.DECODER = "beam"
                    dense, bd = sess.run([Fetch(net, "dense_decoded"), Fetch(net, "read_alignment")], feed)
                    assert np.array_equal(bd["labels"], dense)
                    for n in range(x.shape[1]):
                        L = int((dense[n] != 0).sum())
                        s_, e_ = bd["start"][n, :L], bd["end"][n, :L]
                        assert np.isfinite(bd["path_logprob"][n]) and ((s_ >= 0) & (s_ < e_) & (e_ <= int(tsl[n]))).all()
                        assert (e_[:-1] <= s_[1:]).all()
                        st["beam_lines"] += 1
    finally:
        cfg.DECODER = old
    _report(case="decode10k", **st)
    assert st["lines"] == 10240 and st["argmax_lines"] > 5000 and st["correct"] > 9000 and st["beam_lines"] == 2048, st


def test_packed_lines_align_as_if_alone(monkeypatch):
    from lstm_ctc_ocr_b200.lib.lstm.test import pack_lines
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.session import Session
    we = _load("test_gpu_width_edges", "tests", "test_gpu_width_edges.py")
    mk = _load("make_decode10k", "tests", "golden", "make_decode10k.py")
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    lines = we._eval_inputs()
    net = get_network("LSTM_test")
    with Session(device=DEV) as sess:
        sess.assign(net, mk.load_weights())
        data, lw, tsl = pack_lines(lines)
        packed = sess.run(Fetch(net, "read_alignment"), {net.data: data, net.line_width: lw, net.time_step_len: tsl})
        for i, (d, t) in enumerate(lines):
            alone = sess.run(Fetch(net, "read_alignment"), {net.data: d, net.time_step_len: t})
            L = int((alone["labels"][0] != 0).sum())
            assert int((packed["labels"][i] != 0).sum()) == L
            for key in ("labels", "start", "end", "x0", "x1", "peak"):
                assert np.array_equal(packed[key][i, :L].view(np.int32), alone[key][0, :L].view(np.int32)), (i, key)
            assert packed["path_logprob"][i].view(np.int32) == alone["path_logprob"][0].view(np.int32), i
    _report(case="packed_67", lines=len(lines))


def test_test_model_prints_confidence_only_when_asked(tmp_path, monkeypatch):
    from lstm_ctc_ocr_b200.lib.lstm import test as T
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    pe = _load("test_gpu_packed_eval", "tests", "test_gpu_packed_eval.py")
    mk = _load("make_decode10k", "tests", "golden", "make_decode10k.py")
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    pe._write_dir(str(tmp_path))
    outs = {}
    try:
        for conf in (False, True):
            cfg.TEST.CONFIDENCE = conf
            net = get_network("LSTM_test")
            with Session(device=DEV) as sess:
                sess.assign(net, mk.load_weights())
                buf = io.StringIO()
                with redirect_stdout(buf):
                    T.SolverWrapper(sess, net, None, str(tmp_path), None).test_model(sess, testDir=str(tmp_path), restore=False)
            outs[conf] = [ln for ln in buf.getvalue().splitlines() if "res:" in ln or ln.startswith("total acc")]
    finally:
        cfg.TEST.CONFIDENCE = False
    assert not any("conf:" in ln for ln in outs[False])
    res_true = [ln for ln in outs[True] if "res:" in ln]
    assert len(res_true) == 70 and all(", conf: " in ln and ", peaks: [" in ln for ln in res_true)
    assert [ln.split(", conf: ")[0] for ln in outs[True]] == outs[False]
    for ln in res_true:
        conf = float(ln.split(", conf: ")[1].split(",")[0])
        peaks = ln.split("peaks: [")[1].rstrip("]").split()
        read = ln.split("res: ")[1].split(", conf")[0]
        assert 0.0 <= conf <= 1.0 and len(peaks) == len(read) and all(0.0 <= float(p) <= 1.0 for p in peaks)
