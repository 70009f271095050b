"""Lexicon-based reading on the GPU (crnn_lexicon_candidates, crnn_ctc_lexicon_score, Session.run "lexicon_decoded") against the
references of tests/lexicon_refs.py.

Candidates: cand / cand_dist / cand_total equal, element for element, the row-by-row Levenshtein DP (run in torch on the same
GPU) with the header's (d, index) order, truncation and totals.  Scores: every element within the analytic f32 bound
(lexicon_refs.score_allow) of the fp64 log2-space alpha recursion on the kernel's own logits, -inf / NaN exactly where the
semantics put them, agreement with -crnn_ctc_loss, TF's ctc_loss known answer.  Selection: best equals the fp64 argmax under the
tie rule on every line whose top-two margin exceeds twice its bound; a control that allows the skip between equal labels does
not.  End to end on the 10 240-line fixture, packed evaluation and test_model.  Counts go to build/lexicon_report.jsonl."""
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
import ctc_refs as R  # noqa: E402
import lexicon_refs as X  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _report(**row):
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    with open(os.path.join(ROOT, "build", "lexicon_report.jsonl"), "a") as f:
        f.write(json.dumps(row) + "\n")


def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _t(a, dt=torch.int32):
    return torch.tensor(np.asarray(a), dtype=dt, device=DEV)


class _Raw(object):
    """A CSR lexicon with any ids and lengths (engine.Lexicon refuses the edge cases these tests need)."""

    def __init__(self, entries, max_entry_len=None):
        self.entries = [tuple(int(v) for v in e) for e in entries]
        self.lens = np.array([len(e) for e in self.entries], np.int32)
        self.ids = _t(np.array([v for e in self.entries for v in e] or [0], np.int32))
        self.off = _t(np.r_[0, np.cumsum(self.lens)].astype(np.int32))
        self.max_entry_len = int(self.lens.max()) if max_entry_len is None else int(max_entry_len)

    def __len__(self):
        return len(self.entries)

    def padded(self, width=None):
        out = np.zeros((len(self.entries), max(int(self.lens.max()), 1) if width is None else width), np.int32)
        for k, e in enumerate(self.entries):
            out[k, :len(e)] = e
        return out


def _words(rng, K, lo=2, hi=15):
    return [list(rng.integers(1, 63, size=int(rng.integers(lo, hi + 1)))) for _ in range(K)]


def _edit(rng, w, k):
    """w with k random edits (substitute, delete, insert) over ids 1 .. 62."""
    w = list(w)
    for _ in range(k):
        op = int(rng.integers(0, 3))
        i = int(rng.integers(0, len(w) + 1))
        if op == 0 and i < len(w):
            w[i] = int(rng.integers(1, 63))
        elif op == 1 and i < len(w) and len(w) > 1:
            del w[i]
        else:
            w.insert(i, int(rng.integers(1, 63)))
    return w


def _dense(rows, width=None):
    width = max([len(r) for r in rows] + [0]) if width is None else width
    out = np.zeros((len(rows), width), np.int32)
    for i, r in enumerate(rows):
        out[i, :min(len(r), width)] = r[:width]
    return out, np.array([len(r) for r in rows], np.int32)


# ------------------------------------------------------------------------------------------------------------- candidates
def _ref_distances(reads, rl, lex):
    E = _t(lex.padded(), torch.int64)
    return X.distances_torch(_t(reads, torch.int64), _t(rl, torch.int64), E, _t(lex.lens, torch.int64))


def check_candidates(name, reads, rl, lex, deltas, mcs):
    from lstm_ctc_ocr_b200 import engine
    D = _ref_distances(reads, rl, lex)
    d_reads, d_rl = _t(reads), _t(rl)
    st = dict(case=name, lines=len(rl), entries=len(lex), checked=0, truncated=0)
    for delta in deltas:
        for mc in mcs:
            got = engine.lexicon_candidates(d_reads, d_rl, lex, delta, mc)
            ref = X.candidates_torch(D, delta, mc)
            for g, r, what in zip(got, ref, ("cand", "cand_dist", "cand_total")):
                assert torch.equal(g, r), (name, delta, mc, what, int((g != r).sum()))
            st["checked"] += 1
            st["truncated"] += int((ref[2] > mc).sum())
    _report(**st)
    return st


@pytest.mark.parametrize("K", [1000, 50000])
def test_candidates_1024_lines(K):
    rng = np.random.default_rng(K)
    lex = _Raw(_words(rng, K))
    rows = []
    for i in range(1024):
        if i % 16 == 0:
            rows.append([] if i % 32 == 0 else [int(rng.integers(1, 63))])
        elif i % 5 == 0:
            rows.append(_words(rng, 1, 1, 20)[0])
        else:
            rows.append(_edit(rng, lex.entries[int(rng.integers(0, K))], int(rng.integers(0, 5))))
    reads, rl = _dense(rows)
    st = check_candidates(f"lines1024_K{K}", reads, rl, lex, (0, 1, 3, 8, -1), (1, 64, 256))
    assert st["truncated"] > 0


def test_candidates_across_the_word_boundaries():
    """Reads of 0, 1, 63, 64, 65 and 255 ids (one to four 64-row words) against entries of up to 63 ids; reads made from
    entries so that some are near."""
    rng = np.random.default_rng(3)
    ents = _words(rng, 1000, 1, 63)
    lex = _Raw(ents)
    rows = []
    for i in range(96):
        L = [0, 1, 63, 64, 65, 255][i % 6]
        base = []
        while len(base) < L:
            base += list(ents[int(rng.integers(0, 1000))])
        rows.append(_edit(rng, base[:L], int(rng.integers(0, 3))) if L else [])
    reads, rl = _dense(rows, 255)
    rl = np.minimum(rl, 255)
    check_candidates("word_boundary", reads, rl, lex, (0, 1, 3, 8, -1), (1, 64, 256))
    lone = _Raw([ents[0]])
    check_candidates("one_entry", reads[2:3], rl[2:3], lone, (0, 3, -1), (1, 64))
    # Session.run's lexicon_decoded passes dense_decoded with stride T: strides 257 ... 512 run the 8-word kernel, 513 ... 1024
    # the 16-word one; with delta = -1 the histogram has 1025 bins at stride 1024
    for stride in (300, 512, 513, 1024):
        lens = [L for L in (0, 1, 64, 256, 257, 511, 512, 513, 1023, 1024) if L <= stride]
        rows = []
        for i in range(4 * len(lens)):
            L = lens[i % len(lens)]
            base = []
            while len(base) < L:
                base += list(ents[int(rng.integers(0, 1000))])
            rows.append(_edit(rng, base[:L], int(rng.integers(0, 3)))[:stride] if L else [])
        reads, rl = _dense(rows, stride)
        rl = np.minimum(rl, stride)
        wt = 8 if stride <= 512 else 16
        check_candidates(f"stride{stride}_wt{wt}", reads, rl, lex, (0, 3, 8, -1), (1, 64, 256))


def test_out_of_range_ids_match_nothing():
    rng = np.random.default_rng(4)
    ents = _words(rng, 500, 1, 12)
    for k in range(0, 500, 7):
        ents[k][int(rng.integers(0, len(ents[k])))] = int(rng.choice([64, 70, -1, -100, 1 << 20]))
    lex = _Raw(ents)
    rows = [_edit(rng, ents[int(rng.integers(0, 500))], int(rng.integers(0, 3))) for _ in range(128)]
    for i in range(0, 128, 3):
        rows[i][int(rng.integers(0, len(rows[i])))] = int(rng.choice([64, 70, -1, -5]))
    reads, rl = _dense(rows)
    check_candidates("out_of_range_ids", reads, rl, lex, (0, 1, 3, -1), (64,))
    # an entry equal to a read, both holding the same out-of-range id, is one substitution away
    same = _Raw([[5, 70, 6]])
    c, d, t = _run_candidates(np.array([[5, 70, 6]], np.int32), np.array([3], np.int32), same, 3, 4)
    assert d[0, 0] == 1 and c[0, 0] == 0


def _run_candidates(reads, rl, lex, delta, mc, fill=None):
    """The raw C ABI on output buffers filled with the byte `fill` (None: engine wrapper)."""
    from lstm_ctc_ocr_b200 import _lib, engine
    if fill is None:
        return [a.cpu().numpy() for a in engine.lexicon_candidates(_t(reads), _t(rl), lex, delta, mc)]
    N, M = reads.shape
    outs = [torch.full((N * mc * 4,), fill, dtype=torch.uint8, device=DEV) for _ in range(2)]
    outs.append(torch.full((N * 4,), fill, dtype=torch.uint8, device=DEV))
    d_reads, d_rl = _t(reads), _t(rl)
    _lib.check(_lib.load().crnn_lexicon_candidates(d_reads.data_ptr(), M, d_rl.data_ptr(), N, lex.ids.data_ptr(), lex.off.data_ptr(),
                                                   len(lex), lex.max_entry_len, delta, mc, outs[0].data_ptr(), outs[1].data_ptr(),
                                                   outs[2].data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return [outs[0].view(torch.int32).view(N, mc).cpu().numpy(), outs[1].view(torch.int32).view(N, mc).cpu().numpy(),
            outs[2].view(torch.int32).cpu().numpy()]


def test_candidates_same_bits_on_repeats_and_prefilled_outputs():
    rng = np.random.default_rng(6)
    lex = _Raw(_words(rng, 20000))
    rows = [_edit(rng, lex.entries[int(rng.integers(0, 20000))], int(rng.integers(0, 4))) for _ in range(512)]
    reads, rl = _dense(rows)
    for delta, mc in ((3, 64), (8, 256), (-1, 16)):
        ref = _run_candidates(reads, rl, lex, delta, mc)
        for fill in (0x00, 0xFF, 0x5A, None):
            got = _run_candidates(reads, rl, lex, delta, mc, fill)
            assert all(np.array_equal(a, b) for a, b in zip(ref, got)), (delta, mc, fill)


# ------------------------------------------------------------------------------------------------------------- scores
def check_scores(name, x, il, lex, cand, blank=0, record=None):
    """Every score element against score_fp64 within its analytic bound, -inf / NaN exactly where the reference has them, and
    best / best_score against the fp64 selection on every line above twice its bound.  Returns (ref, allow, gpu score, best)."""
    from lstm_ctc_ocr_b200 import engine
    cand = np.asarray(cand, np.int32)
    sc, best, bsc = engine.ctc_lexicon_score(x, _t(il), lex, _t(cand), blank=blank)
    g, best, bsc = sc.cpu().numpy().astype(np.float64), best.cpu().numpy(), bsc.cpu().numpy()
    ref, allow = X.score_fp64(x, il, lex.entries, cand, blank)
    assert np.array_equal(np.isnan(g), np.isnan(ref)), name
    ninf = ref == -np.inf
    assert (g[ninf] == -np.inf).all(), name
    fin = np.isfinite(ref)
    assert np.isfinite(g[fin]).all(), name
    with np.errstate(invalid="ignore"):
        err = np.abs(g - ref)
    assert (err[fin] <= allow[fin]).all(), (name, float((err[fin] / allow[fin]).max()))
    bref, _, margin = X.select_ref(ref, cand)
    line_allow = np.where(fin, allow, 0).max(axis=1) if cand.shape[1] else np.zeros(len(il))
    sure = margin > 2 * line_allow
    assert np.array_equal(best[sure], bref[sure]), name
    none = ~fin.any(axis=1)
    assert (best[none] == -1).all() and (bsc[none] == -np.inf).all(), name
    some = ~none
    gmax = np.where(np.isfinite(g), g, -np.inf).max(axis=1) if cand.shape[1] else np.zeros(len(il))
    assert np.array_equal(bsc[some].astype(np.float64), gmax[some]), name
    st = dict(case=name, lines=len(il), slots=int(cand.size), finite=int(fin.sum()),
              worst_over_allow=float((err[fin] / np.maximum(allow[fin], 1e-300)).max()) if fin.any() else 0.0, selection_checked=int(sure.sum()))
    _report(**st)
    return ref, allow, g, best


def test_scores_c3_trained_model_and_the_ctc_loss():
    """The trained fixture weights at C3 (T = 63, N = 1024): greedy reads, their 64 nearest entries of a 50 000-word lexicon
    (no threshold), the scores; then -crnn_ctc_loss of every finite (line, entry) pair, within the score's bound plus the
    loss's relative 1e-4 (the bound of tests/test_zz_gpu_known_answers.py)."""
    from lstm_ctc_ocr_b200 import engine, synthetic
    mk = _load("make_decode10k", "tests", "golden", "make_decode10k.py")
    data, _, _, tsl = synthetic.synth_batch(1024, 256, seed=5)
    m = engine.CrnnModel(weight_decay=1e-5, device=DEV)
    m.load_params(mk.load_weights())
    d_tsl = _t(tsl)
    x = m.forward(_t(data, torch.float32), d_tsl)
    o, ol = engine.ctc_greedy(x, d_tsl)
    reads = engine.dense_decoded(o, ol)
    rng = np.random.default_rng(9)
    lex = engine.Lexicon(_words(rng, 50000), device=DEV)
    cand, _, _ = engine.lexicon_candidates(reads, ol, lex, -1, 64)
    cand = cand.cpu().numpy()
    ref, allow, g, _ = check_scores("c3_trained", x, tsl, lex, cand)
    nn, jj = np.nonzero(np.isfinite(ref))
    xs = x[:, torch.tensor(nn, device=DEV)].contiguous()
    ents = [lex.entries[cand[n, j]] for n, j in zip(nn, jj)]
    costs, _ = engine.ctc_loss(xs, _t(np.concatenate(ents)), _t([len(e) for e in ents]), _t(tsl[nn]), max_label_len=15)
    costs = costs.cpu().numpy().astype(np.float64)
    d = np.abs(-costs - g[nn, jj])
    assert (d <= 2 * allow[nn, jj] + 1e-4 * np.abs(costs)).all(), float(d.max())


def _score_case(T, blank, seed, N=16, J=24):
    rng = np.random.default_rng(seed)
    x = torch.tensor(rng.normal(0, 3.0, size=(T, N, 64)).astype(np.float32), device=DEV)
    draw = lambda L: [int(v) for v in R.draw_labels(rng, L, blank)]
    ents = [[], draw(1), draw(15), draw(63), draw(5), [draw(1)[0]] * 3, [draw(1)[0]] * 63]
    rep = draw(8)
    rep[3] = rep[2]
    ents += [rep, draw(2) + [blank], [64] + draw(2), [-1], draw(40)]
    ents += [draw(int(rng.integers(1, 20))) for _ in range(20)]
    il = np.array([[0, 1, T, T + 5][i % 4] for i in range(N)], np.int32)
    cand = rng.integers(-1, len(ents), size=(N, J)).astype(np.int32)
    cand[:4] = np.arange(J) % len(ents)                  # every entry in some slot
    return x, il, _Raw(ents, 63), cand


@pytest.mark.parametrize("T, blank", [(1, 0), (2, 0), (3, 0), (255, 0), (255, 17), (255, 63), (768, 0)])
def test_scores_frames_lengths_blanks(T, blank):
    x, il, lex, cand = _score_case(T, blank, 100 + T + blank)
    ref, _, g, _ = check_scores(f"T{T}_blank{blank}", x, il, lex, cand, blank)
    assert np.isnan(g).any() and (g == -np.inf).any()
    if T >= 255:
        assert np.isfinite(g).sum() > 0


def test_scores_reproduce_the_tensorflow_known_answer():
    from lstm_ctc_ocr_b200 import engine
    K = _load("third_party_kats", "tests", "golden", "third_party_kats.py")
    x, flat, ll, il, cost, _ = K.ctc_case(num_classes=64, blank=0)
    off = np.r_[0, np.cumsum(ll)]
    lex = _Raw([flat[off[i]:off[i + 1]] for i in range(len(ll))], 63)
    sc, best, _ = engine.ctc_lexicon_score(_t(x, torch.float32), _t(il), lex, _t([[0, -1], [1, -1]]))
    sc = sc.cpu().numpy()
    assert np.allclose(-sc[:, 0], cost, rtol=1e-4, atol=0), sc
    assert list(best.cpu().numpy()) == [0, 1] and (sc[:, 1] == -np.inf).all()


def test_status_codes_leave_the_outputs_untouched():
    from lstm_ctc_ocr_b200 import _lib
    lib = _lib.load()
    T, N, J = 40, 4, 8
    x = torch.zeros((769, N, 64), device=DEV)
    lex = _Raw([[1, 2], [3]], 63)
    cand, il = _t(np.zeros((N, J), np.int32)), _t(np.full(N, T, np.int32))
    score, best, bsc = torch.full((N, J), 5.0, device=DEV), torch.full((N,), 7, dtype=torch.int32, device=DEV), torch.full((N,), 5.0, device=DEV)
    st = torch.cuda.current_stream().cuda_stream

    def call(T=T, C=64, mel=63, logits=None):
        return lib.crnn_ctc_lexicon_score(x.data_ptr() if logits is None else logits, il.data_ptr(), T, N, C, 0, lex.ids.data_ptr(),
                                          lex.off.data_ptr(), mel, cand.data_ptr(), J, score.data_ptr(), best.data_ptr(),
                                          bsc.data_ptr(), st)
    assert call(T=769) == 4 and "769" in lib.crnn_last_error().decode()
    assert call(C=65) == 4
    assert call(mel=64) == 4 and "64" in lib.crnn_last_error().decode()
    assert call(logits=0) == 1
    reads, rl = _t(np.ones((N, 4), np.int32)), _t(np.full(N, 4, np.int32))
    cd, cdist, ct = _t(np.full((N, J), 9, np.int32)), _t(np.full((N, J), 9, np.int32)), _t(np.full(N, 9, np.int32))
    assert lib.crnn_lexicon_candidates(reads.data_ptr(), 1025, rl.data_ptr(), N, lex.ids.data_ptr(), lex.off.data_ptr(), 2, 63, 3, J,
                                       cd.data_ptr(), cdist.data_ptr(), ct.data_ptr(), st) == 4
    assert lib.crnn_lexicon_candidates(reads.data_ptr(), 4, rl.data_ptr(), N, lex.ids.data_ptr(), lex.off.data_ptr(), 2, 64, 3, J,
                                       cd.data_ptr(), cdist.data_ptr(), ct.data_ptr(), st) == 4
    assert lib.crnn_lexicon_candidates(reads.data_ptr(), 4, rl.data_ptr(), N, lex.ids.data_ptr(), lex.off.data_ptr(), 2, 63, 3, J,
                                       0, cdist.data_ptr(), ct.data_ptr(), st) == 1
    torch.cuda.synchronize()
    assert (score == 5.0).all() and (best == 7).all() and (bsc == 5.0).all()
    assert (cd == 9).all() and (cdist == 9).all() and (ct == 9).all()
    assert call() == 0
    torch.cuda.synchronize()
    assert not (score == 5.0).any()


# ------------------------------------------------------------------------------------------------------------- end to end
def _control_scores(x, il, entries, cand):
    """score_fp64's recursion with the skip also allowed between equal labels (a wrong lattice), finite slots only."""
    saved = R.transitions

    def loose(ext, S, blank):
        s = torch.arange(ext.shape[1], device=ext.device)
        live = s[None] < S[:, None]
        skin = (s[None] >= 2) & live & (ext != blank)
        return live, skin, None
    R.transitions = loose
    try:
        return X.score_fp64(x, il, entries, cand)[0]
    finally:
        R.transitions = saved


def _neighbours(rng, w):
    """Edit-distance-1 neighbours of w: a substitution, a deletion and a doubled letter."""
    out = []
    i = int(rng.integers(0, len(w)))
    s = list(w)
    s[i] = int(rng.integers(1, 63))
    out.append(s)
    if len(w) > 1:
        out.append(w[:i] + w[i + 1:])
    out.append(w[:i + 1] + [w[i]] + w[i + 1:])
    return out


def test_decode10k_lexicon_reads(tmp_path):
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg, get_encode_decode_dict
    from lstm_ctc_ocr_b200.lib.lstm.lexicon import load_lexicon
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.session import Session
    mk = _load("make_decode10k", "tests", "golden", "make_decode10k.py")
    fx = np.load(os.path.join(ROOT, "tests", "golden", "decode10k_oracle.npz"))
    off = np.r_[0, np.cumsum(fx["lab_len"].astype(np.int64))]
    truths = [tuple(int(v) for v in fx["lab_flat"][off[i]:off[i + 1]]) for i in range(len(fx["lab_len"]))]
    distinct = sorted(set(truths))
    rng = np.random.default_rng(2024)
    words = [list(w) for w in distinct]
    for w in distinct:
        words += _neighbours(rng, list(w))
    words += _words(rng, 40000)
    _, dec = get_encode_decode_dict()
    path = tmp_path / "words.txt"
    path.write_text("\n".join("".join(dec[v] for v in w) for w in words) + "\n", encoding="utf-8")
    lex = engine.Lexicon(load_lexicon(str(path)), device=DEV)
    s = mk.sampler()
    net = get_network("LSTM_train")
    st = dict(case="decode10k", lines=0, distinct_truths=len(distinct), lexicon=len(lex), greedy_correct=0, lexicon_correct=0,
              selection_checked=0, control_differs=0)
    old = cfg.TEST.LEXICON
    cfg.TEST.LEXICON = str(path)
    try:
        with Session(device=DEV) as sess:
            sess.assign(net, mk.load_weights())
            for k in range(mk.NBATCH):
                imgs, lab, ll, tsl = s.batch(k)
                feed = {net.data: np.stack(imgs), net.time_step_len: np.asarray(tsl, np.int32)}
                x, dense, lx = sess.run([Fetch(net, "logits"), Fetch(net, "dense_decoded"), Fetch(net, "lexicon_decoded")], feed)
                xt = torch.tensor(x, device=DEV)
                rl = (dense != 0).sum(1).astype(np.int32)
                cand, dist, tot = (a.cpu().numpy() for a in engine.lexicon_candidates(_t(dense), _t(rl), lex, 3, 64))
                assert np.array_equal(lx["candidates"], tot)
                ref, allow, _, _ = check_scores(f"decode10k_b{k}", xt, tsl, lex, cand)
                bref, _, margin = X.select_ref(ref, cand)
                line_allow = np.where(np.isfinite(ref), allow, 0).max(axis=1)
                sure = margin > 2 * line_allow
                assert np.array_equal(lx["index"][sure], bref[sure]), k
                ctl, _, _ = X.select_ref(_control_scores(xt, tsl, lex.entries, cand), cand)
                st["control_differs"] += int((ctl[sure] != bref[sure]).sum())
                st["selection_checked"] += int(sure.sum())
                truth = [list(lab[o:o + n]) for o, n in zip(np.r_[0, np.cumsum(ll)[:-1]], ll)]
                for n in range(len(ll)):
                    st["lines"] += 1
                    read = [int(v) for v in dense[n] if v]
                    chosen = [int(v) for v in lx["labels"][n] if v]
                    if lx["index"][n] >= 0:
                        assert chosen == list(lex.entries[lx["index"][n]]) and lx["distance"][n] == dist[n][cand[n] == lx["index"][n]][0]
                    else:
                        assert chosen == read and lx["distance"][n] == -1 and lx["score"][n] == -np.inf
                    st["greedy_correct"] += int(read == [int(v) for v in truth[n]])
                    st["lexicon_correct"] += int(chosen == [int(v) for v in truth[n]])
    finally:
        cfg.TEST.LEXICON = old
    _report(**st)
    print(st)
    assert st["lines"] == 10240 and st["selection_checked"] > 9000, st
    assert st["control_differs"] > 0, st                      # the wrong lattice picks other words: the check can fail


def test_packed_lines_and_test_model(tmp_path, monkeypatch):
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.lstm import test as TM
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg, get_encode_decode_dict
    from lstm_ctc_ocr_b200.lib.lstm.test import pack_lines
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.session import Session
    we = _load("test_gpu_width_edges", "tests", "test_gpu_width_edges.py")
    pe = _load("test_gpu_packed_eval", "tests", "test_gpu_packed_eval.py")
    mk = _load("make_decode10k", "tests", "golden", "make_decode10k.py")
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    lines = we._eval_inputs()
    enc, dec = get_encode_decode_dict()
    rng = np.random.default_rng(31)
    d = tmp_path / "eval"
    d.mkdir()
    pe._write_dir(str(d))
    names = [f.split(".")[0].split("_")[1] for f in sorted(os.listdir(str(d)))]
    old = cfg.TEST.LEXICON
    try:
        net = get_network("LSTM_test")
        with Session(device=DEV) as sess:
            sess.assign(net, mk.load_weights())
            reads = [sess.run(Fetch(net, "dense_decoded"), {net.data: a, net.time_step_len: t})[0] for a, t in lines]
            words = []
            for r in reads:
                w = [int(v) for v in r if v]
                if w:
                    words += [w] + _neighbours(rng, w)
            words += [[enc[ch] for ch in nm] for nm in names] + _words(rng, 5000)
            words = [w for w in words if len(w) <= 63]       # a long line's read is no word
            path = tmp_path / "words.txt"
            path.write_text("\n".join("".join(dec[v] for v in w) for w in words) + "\n", encoding="utf-8")
            cfg.TEST.LEXICON = str(path)
            data, lw, tsl = pack_lines(lines)
            packed = sess.run(Fetch(net, "lexicon_decoded"), {net.data: data, net.line_width: lw, net.time_step_len: tsl})
            for i, (a, t) in enumerate(lines):
                alone = sess.run(Fetch(net, "lexicon_decoded"), {net.data: a, net.time_step_len: t})
                for key in ("index", "score", "distance", "candidates"):
                    assert np.asarray(packed[key][i]).view(np.int32) == np.asarray(alone[key][0]).view(np.int32), (i, key)
                L = alone["labels"].shape[1]
                assert np.array_equal(packed["labels"][i, :L], alone["labels"][0]) and not packed["labels"][i, L:].any(), i
        outs = {}
        for lexicon in ("", str(path)):
            cfg.TEST.LEXICON = lexicon
            net = get_network("LSTM_test")
            with Session(device=DEV) as sess:
                sess.assign(net, mk.load_weights())
                buf = io.StringIO()
                with redirect_stdout(buf):
                    TM.SolverWrapper(sess, net, None, str(d), None).test_model(sess, testDir=str(d), restore=False)
            outs[lexicon] = [ln for ln in buf.getvalue().splitlines() if "res:" in ln or ln.startswith("total acc")]
        cfg.TEST.LEXICON = ""
        with pytest.raises(ValueError):
            with Session(device=DEV) as sess:
                net = get_network("LSTM_test")
                sess.assign(net, mk.load_weights())
                sess.run(Fetch(net, "lexicon_decoded"), {net.data: lines[0][0], net.time_step_len: lines[0][1]})
    finally:
        cfg.TEST.LEXICON = old
    plain, lexed = outs[""], outs[str(path)]
    assert not any(", read: " in ln for ln in plain) and len(plain) == len(lexed) == 71
    vocab = {"".join(dec[v] for v in w) for w in words}
    changed = 0
    for p, q in zip(plain[:-1], lexed[:-1]):
        pr = p.split("res: ")[1]
        if ", read: " in q:
            lr, rd = q.split("res: ")[1].split(", read: ")
            assert rd == pr and lr != pr and lr in vocab
            changed += 1
        else:
            assert q == p
    acc = lambda ln: int(ln.split(":")[1].split("/")[0])
    _report(case="test_model", lines=70, changed=changed, plain_correct=acc(plain[-1]), lexicon_correct=acc(lexed[-1]))
