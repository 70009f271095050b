"""The device beam-search decoder (crnn_ctc_beam_search_device, csrc/beam.cu) against the host decoder it restates
(crnn_ctc_beam_search, csrc/beam.cpp) and, where the CPU suite uses it, the oracle's restatement of TensorFlow's
CTCBeamSearchDecoder (network.py:656).  Every case must give IDENTICAL labellings, and neg_log_prob within one float ulp."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _lines(out, out_len):
    return [out[i, :out_len[i]].tolist() for i in range(len(out_len))]


def _within_one_ulp(a, b):
    a = np.asarray(a, np.float32); b = np.asarray(b, np.float32)
    ia = a.view(np.int32).astype(np.int64); ib = b.view(np.int32).astype(np.int64)
    return bool(np.all((a == b) | ((np.sign(a) == np.sign(b)) & (np.abs(ia - ib) <= 1))))


def _both(x, il, **kw):
    """Device and host decode of the same logits; asserts identical outputs and returns the labellings."""
    from lstm_ctc_ocr_b200 import engine
    x = np.ascontiguousarray(x, np.float32)
    il = np.asarray(il, np.int32)
    o, ol, nlp = engine.ctc_beam_search_device(torch.tensor(x, device=DEV), torch.tensor(il, device=DEV), **kw)
    o, ol, nlp = o.cpu().numpy(), ol.cpu().numpy(), nlp.cpu().numpy()
    ho, hol, hnlp = engine.ctc_beam_search(x, np.clip(il, 0, x.shape[0]), **kw)
    got, ref = _lines(o, ol), _lines(ho, hol)
    bad = [i for i in range(len(il)) if got[i] != ref[i]]
    assert not bad, (kw, bad[:5], [(got[i], ref[i]) for i in bad[:3]])
    assert np.array_equal(o, ho) and np.array_equal(ol, hol)            # zero padding included
    assert _within_one_ulp(nlp, hnlp), (kw, nlp, hnlp)
    return got, nlp


def test_device_beam_rule_table():
    def onehot(seq):
        x = np.zeros((len(seq), 1, 64), np.float32)
        for t, a in enumerate(seq):
            x[t, 0, a] = 8.0
        return x
    beam = lambda seq, **kw: _both(onehot(seq), [len(seq)], **kw)[0][0]
    assert beam([1, 2, 3, 4]) == [1, 2, 3, 4]
    assert beam([63, 63, 63]) == []
    assert beam([5, 5, 63, 5, 0, 7], merge_repeated=False) == [5, 5, 7]
    assert beam([5, 5, 63, 5, 0, 7]) == [5, 7]
    assert beam([3, 63, 3, 63, 4]) == [3, 4]
    assert beam([0, 1, 0, 2], strip=-1) == [0, 1, 0, 2]
    assert beam([5, 5, 63, 5, 0, 7], merge_repeated=False, strip=-1) == [5, 5, 0, 7]
    assert beam([5, 5, 63, 5, 0, 7], strip=-1) == [5, 0, 7]


def _peaked_lines(n, T, seed, margin=6.0):
    r = np.random.default_rng(seed)
    path = r.choice(64, size=(T, n), p=np.r_[0.25, np.full(62, 0.65 / 62), 0.10])
    rep = r.random((T, n)) < 0.3
    for t in range(1, T):
        path[t] = np.where(rep[t], path[t - 1], path[t])
    y = r.standard_normal((T, n, 64))
    y[np.arange(T)[:, None], np.arange(n)[None, :], path] += margin
    return y


@pytest.mark.parametrize("kind,seed", [("peaked", 2), ("soft", 5), ("flat", 7), ("peaked", 12), ("soft", 15), ("flat", 17)])
def test_device_beam_matches_host_and_oracle(kind, seed):
    """The generators of test_beam_search_matches_oracle_restatement: ragged lengths including 0, both merge modes, widths
    100 and 3."""
    from oracle import crnn_oracle as O
    rng = np.random.default_rng(seed)
    T, N = 19, 10
    if kind == "peaked":
        x = _peaked_lines(N, T, seed=seed)
    elif kind == "soft":
        x = _peaked_lines(N, T, seed=seed, margin=2.0)
    else:
        x = rng.standard_normal((T, N, 64)) * 0.3
    x = x.astype(np.float32)
    il = rng.integers(0, T + 1, size=N).astype(np.int32)
    il[0] = T; il[1] = 0
    for merge in (True, False):
        for bw in (100, 3):
            got, nlp = _both(x, il, beam_width=bw, merge_repeated=merge)
            assert got == O.beam_search_decode(x, il, beam_width=bw, merge_repeated=merge), (kind, merge, bw)
            assert np.isfinite(nlp).all() and nlp[1] == 0.0


EDGE_C = (2, 32, 33, 34, 63)                   # the second lane slot (c = lane + 32) partly used, class masks of 31 ... 62 bits
EDGE_WIDTHS = (31, 32, 33, 63, 64, 65, 127)     # heap depth boundaries


@pytest.mark.parametrize("seed", range(36 + 2 * len(EDGE_C)))
def test_device_beam_ties_and_narrow_beams(seed):
    """Quantised logits with exact ties, all-equal frames, C in {3, 6, 17} and (seeds 36 on) the edge class counts EDGE_C,
    widths that evict constantly and the heap-depth widths EDGE_WIDTHS, both merge modes: the inputs on which the visit
    order and the tie rules decide the result.  The oracle is compared at the narrow widths and 100."""
    from oracle import crnn_oracle as O
    rng = np.random.default_rng(100 + seed)
    C = int(rng.choice([3, 6, 17])) if seed < 36 else EDGE_C[seed % len(EDGE_C)]
    T, N = int(rng.integers(4, 15)), 8
    kind = seed % 3
    if kind == 0:
        x = np.round(rng.standard_normal((T, N, C)) * 2) / 2
    elif kind == 1:
        x = rng.integers(0, 2, size=(T, N, C)).astype(np.float64) * float(rng.choice([1, 5]))
        x[T // 2] = 0.0
    else:
        x = rng.standard_normal((T, N, C)) * float(rng.choice([0.3, 3.0]))
    x = x.astype(np.float32)
    il = rng.integers(0, T + 1, size=N).astype(np.int32)
    il[0] = T
    for bw in (1, 2, 3, 5, 7, 100) + EDGE_WIDTHS:
        for merge in (True, False):
            got, _ = _both(x, il, beam_width=bw, merge_repeated=merge, strip=-1)
            if bw not in EDGE_WIDTHS:
                assert got == O.beam_search_decode(x, il, beam_width=bw, merge_repeated=merge, strip=-1), (C, T, bw, merge)


def test_device_beam_reproduces_tensorflows_own_known_answer():
    K = _load("third_party_kats", "tests", "golden", "third_party_kats.py")
    x, il = K.beam_case()
    assert _both(x, il, beam_width=K.BEAM_WIDTH, merge_repeated=True, strip=-1)[0] == [K.BEAM_TOP_PATHS[0]]
    for bw in (1, 3, 100):
        assert _both(x, il, beam_width=bw, merge_repeated=True, strip=-1)[0] == [K.BEAM_TOP_PATHS[1]]


@pytest.mark.parametrize("C", [6, 64])
def test_device_beam_non_finite_logits(C):
    """NaN, +inf and -inf entries, an all -inf frame, an all-NaN frame, and a -inf blank column (the re-scores then depend
    on the order: a parent re-scored earlier in the frame may have turned inactive)."""
    rng = np.random.default_rng(3 + C)
    T, N = 12, 8
    x = (rng.standard_normal((T, N, C)) * 2).astype(np.float32)
    x[2, 0, 1] = np.nan; x[1, 0, 3] = -np.inf
    x[3, 1, :] = -np.inf                        # all -inf frame
    x[4, 2, 0] = np.inf                         # +inf logit: the frame's normaliser is NaN
    x[5, 3, 2] = -np.inf
    x[:, 4, C - 1] = -np.inf                    # no blank at all
    x[6, 5, :] = np.nan                         # all-NaN frame
    x[7:, 5, C - 1] = -np.inf
    q = np.round(x[:, 6] * 2) / 2
    q[:, C - 1] = -np.inf; q[::3, 0] = -np.inf  # ties with a -inf blank column
    x[:, 6] = q
    x[:, 7, C - 1] = -np.inf; x[::2, 7, 1] = -np.inf
    il = np.array([T, T, T, 9, T, T, T, T], np.int32)
    for bw in (1, 3, 100):
        for merge in (True, False):
            _both(x, il, beam_width=bw, merge_repeated=merge)
            _both(x, il, beam_width=bw, merge_repeated=merge, strip=-1)


def test_device_beam_benchmark_shape():
    """N = 1024, T = 63, C = 64, width 100 on tools/beam_bench.py's peaked, soft and flat frames."""
    bb = _load("beam_bench", "tools", "beam_bench.py")
    rng = np.random.default_rng(0)
    for kind in ("peaked", "soft", "flat"):
        x = bb.frames(kind, 63, 1024, rng)
        _both(x, np.full(1024, 63, np.int32), beam_width=100)


def test_device_beam_is_deterministic_and_graph_capturable():
    """Two calls give bit-identical results; after one warm-up call the call can be captured in a CUDA graph (no host sync,
    no allocation inside) and the replay on new logits equals a direct call."""
    from lstm_ctc_ocr_b200 import engine
    bb = _load("beam_bench", "tools", "beam_bench.py")
    rng = np.random.default_rng(1)
    T, N = 40, 96
    x1 = torch.tensor(bb.frames("soft", T, N, rng), device=DEV)
    x2 = torch.tensor(bb.frames("flat", T, N, rng), device=DEV)
    il = torch.tensor(rng.integers(0, T + 1, size=N), dtype=torch.int32, device=DEV)
    a = engine.ctc_beam_search_device(x1, il)
    b = engine.ctc_beam_search_device(x1, il)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    static_x = x1.clone()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        res = engine.ctc_beam_search_device(static_x, il)
    static_x.copy_(x2)
    g.replay()
    ref = engine.ctc_beam_search_device(x2, il)
    torch.cuda.synchronize()
    for u, v in zip(res, ref):
        assert torch.equal(u, v)
    assert not torch.equal(res[0], a[0])


def test_device_beam_argument_statuses_and_length_clamp():
    from lstm_ctc_ocr_b200 import _lib, engine
    from lstm_ctc_ocr_b200._lib import CrnnError
    lib = _lib.load()
    T, N, C = 10, 4, 64
    x = torch.randn(T, N, C, device=DEV)
    il = torch.full((N,), T, dtype=torch.int32, device=DEV)
    out = torch.empty((N, T), dtype=torch.int32, device=DEV)
    ol = torch.empty(N, dtype=torch.int32, device=DEV)
    need = engine.beam_workspace_bytes(T, N, C, 100)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    call = lambda Cx, bw, nbytes: lib.crnn_ctc_beam_search_device(x.data_ptr(), il.data_ptr(), T, N, Cx, bw, 1, 0, out.data_ptr(),
                                                                   ol.data_ptr(), 0, ws.data_ptr(), nbytes, st)
    assert call(C, 100, need - 1) == 5                                   # CRNN_WORKSPACE_TOO_SMALL
    for Cx, bw in ((C, 0), (C, 129), (65, 100), (1, 100)):
        assert call(Cx, bw, need) == 4, (Cx, bw)                         # CRNN_UNSUPPORTED
    assert call(C, 100, need) == 0
    torch.cuda.synchronize()
    for bw in (0, 129):
        with pytest.raises(CrnnError):
            engine.ctc_beam_search_device(x, il, beam_width=bw)
    # input_len is clamped on the device: below 0 acts as 0, above T as T
    xs = np.random.default_rng(4).standard_normal((T, N, C)).astype(np.float32)
    d = engine.ctc_beam_search_device(torch.tensor(xs, device=DEV), torch.tensor([-3, T + 5, 0, T], dtype=torch.int32, device=DEV))
    h = engine.ctc_beam_search(xs, np.array([0, T, 0, T], np.int32))
    assert np.array_equal(d[0].cpu().numpy(), h[0]) and np.array_equal(d[1].cpu().numpy(), h[1])
    assert _within_one_ulp(d[2].cpu().numpy(), h[2])


def test_device_beam_decodes_the_10k_rendered_lines_through_the_session():
    """cfg.DECODER = "beam" through Session.run on the 10 240 rendered lines of the decode-equality fixture (trained weights),
    logits fetched in the same run: the device decode equals the host decode of those logits on every line.  Agreement with
    greedy and with the truth is reported."""
    if not os.path.exists(os.path.join(ROOT, "tests", "golden", "decode10k_oracle.npz")):
        pytest.skip("fixture missing: run tests/golden/make_decode10k.py")
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.session import Session
    mk = _load("make_decode10k", "tests", "golden", "make_decode10k.py")
    fx = np.load(os.path.join(ROOT, "tests", "golden", "decode10k_oracle.npz"))
    s = mk.sampler()
    B = int(fx["batch"])
    lab_off = np.concatenate([[0], np.cumsum(fx["lab_len"].astype(np.int64))])
    net = get_network("LSTM_test")
    f_logits, f_dense = Fetch(net, "logits"), Fetch(net, "dense_decoded")
    st = dict(lines=0, device_equals_host=0, beam_equals_greedy=0, beam_correct=0, greedy_correct=0)
    old = cfg.get("DECODER", "greedy")
    cfg.DECODER = "beam"
    try:
        with Session(device=DEV) as sess:
            sess.assign(net, mk.load_weights())
            for k in range(len(fx["crc"])):
                imgs, _, _, tsl = s.batch(k)
                tsl = np.asarray(tsl, np.int32)
                logits, dec = sess.run([f_logits, f_dense], feed_dict={net.data: np.stack(imgs), net.time_step_len: tsl,
                                                                       net.keep_prob: 1.0})
                ho, hol, _ = engine.ctc_beam_search(logits, tsl, beam_width=100, merge_repeated=True)
                go, gol = engine.ctc_greedy(torch.tensor(logits, device=DEV), torch.tensor(tsl, device=DEV))
                go, gol = go.cpu().numpy(), gol.cpu().numpy()
                for n in range(B):
                    g = k * B + n
                    got = [int(v) for v in dec[n] if v != 0] if dec.size else []
                    host = [int(v) for v in ho[n, :hol[n]] if v != 0]
                    greedy = go[n, :gol[n]].tolist()
                    truth = fx["lab_flat"][lab_off[g]:lab_off[g + 1]].astype(np.int64).tolist()
                    st["lines"] += 1
                    st["device_equals_host"] += int(got == host)
                    st["beam_equals_greedy"] += int(got == greedy)
                    st["beam_correct"] += int(got == truth)
                    st["greedy_correct"] += int(greedy == truth)
    finally:
        cfg.DECODER = old
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    with open(os.path.join(ROOT, "build", "parity_report.jsonl"), "a") as f:
        f.write(json.dumps(dict(test="decode10k_device_beam", **st)) + "\n")
    print(json.dumps(st))
    assert st["lines"] == 10240
    assert st["device_equals_host"] == st["lines"], st
