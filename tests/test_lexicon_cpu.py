"""CPU checks of lexicon-based reading: the Levenshtein references (the plain DP on known answers, the bit-parallel
restatement the kernel runs against the DP), the candidate semantics, the score reference against ctc_refs.ctc_fp64 and
path enumeration, the selection's tie rule, engine.Lexicon, the word-list loader, the cfg keys, the C ABI's prototypes and
the absence of a CPU fallback."""
import os
import re
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ctc_refs as R  # noqa: E402
import lexicon_refs as X  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ids(word):
    return [ord(ch) - ord("a") + 1 for ch in word]


# ------------------------------------------------------------------------------------------------------------- distances
@pytest.mark.parametrize("a, b, d", [("kitten", "sitting", 3), ("", "", 0), ("", "abc", 3), ("abc", "", 3),
                                     ("flaw", "lawn", 2), ("intention", "execution", 5), ("same", "same", 0),
                                     ("abc", "acb", 2), ("a", "b", 1), ("book", "back", 2)])
def test_dp_known_answers(a, b, d):
    assert X.levenshtein(_ids(a), _ids(b)) == d
    assert X.levenshtein(_ids(b), _ids(a)) == d
    assert X.myers_distance(_ids(a), _ids(b)) == d


def test_dp_vectorised_equals_pairwise():
    rng = np.random.default_rng(1)
    reads = [list(rng.integers(0, 6, size=rng.integers(0, 12))) for _ in range(40)]
    entries = [list(rng.integers(0, 6, size=rng.integers(1, 12))) for _ in range(30)]
    M = max(len(r) for r in reads)
    rd = np.zeros((len(reads), M), np.int64)
    for i, r in enumerate(reads):
        rd[i, :len(r)] = r
    D = X.pair_distances(rd, [len(r) for r in reads], entries)
    for i, r in enumerate(reads):
        for k, e in enumerate(entries):
            assert D[i, k] == X.levenshtein(r, e)


@pytest.mark.parametrize("seed", range(3))
def test_bit_parallel_restatement_equals_the_dp(seed):
    """Reads of 0 .. 200 ids (across the 64-row word boundaries), entries of 0 .. 63; small alphabets for many matches, and ids
    outside [0, 64) in both, which match nothing (not even themselves)."""
    rng = np.random.default_rng(10 + seed)
    for it in range(150):
        m = int(rng.choice([0, 1, 2, 63, 64, 65, 127, 128, 129, 200, rng.integers(0, 201)]))
        n = int(rng.integers(0, 64))
        alpha = int(rng.choice([2, 4, 64]))
        read = list(rng.integers(0, alpha, size=m))
        entry = list(rng.integers(0, alpha, size=n))
        if it % 5 == 0 and m and n:
            read[int(rng.integers(0, m))] = 64 + int(rng.integers(0, 3))
            entry[int(rng.integers(0, n))] = -1 if it % 2 else 64
        if it % 7 == 0 and n:
            read = entry[:min(n, m)] + read[min(n, m):]                              # near matches
        assert X.myers_distance(read, entry) == X.levenshtein(read, entry), (it, m, n)
    assert X.levenshtein([70], [70]) == 1 and X.myers_distance([70], [70]) == 1
    assert X.levenshtein([-1, 3], [-1, 3]) == 1


# ------------------------------------------------------------------------------------------------------------- candidates
def test_candidate_order_truncation_and_totals():
    entries = [_ids(w) for w in ("cat", "cart", "bat", "act", "cat", "dog", "ca", "cats", "at", "c")]
    reads = np.array([_ids("cat") + [0]], np.int64)
    D = X.pair_distances(reads, [3], entries)
    assert list(D[0]) == [0, 1, 1, 2, 0, 3, 1, 1, 1, 2]
    cand, dist, tot = X.candidates_ref(D, 1, 8)
    assert list(cand[0]) == [0, 4, 1, 2, 6, 7, 8, -1] and list(dist[0]) == [0, 0, 1, 1, 1, 1, 1, -1] and tot[0] == 7
    cand, dist, tot = X.candidates_ref(D, 1, 3)                                     # truncated at distance 1 by index
    assert list(cand[0]) == [0, 4, 1] and list(dist[0]) == [0, 0, 1] and tot[0] == 7
    cand, dist, tot = X.candidates_ref(D, 0, 4)
    assert list(cand[0]) == [0, 4, -1, -1] and tot[0] == 2
    cand, dist, tot = X.candidates_ref(D, -1, 10)                                   # no threshold: every entry, nearest first
    assert list(cand[0]) == [0, 4, 1, 2, 6, 7, 8, 3, 9, 5] and tot[0] == 10
    cand, _, tot = X.candidates_ref(D, -1, 1)
    assert list(cand[0]) == [0] and tot[0] == 10


def test_lexicon_keeps_the_first_of_exact_duplicates_and_rejects_bad_entries():
    from lstm_ctc_ocr_b200 import engine
    lex = engine.Lexicon([[1, 2, 3], [4], [1, 2, 3], [4, 4], [4]], device="cpu")
    assert lex.entries == [(1, 2, 3), (4,), (4, 4)] and list(lex.index_of) == [0, 1, 3]
    assert lex.off.tolist() == [0, 3, 4, 6] and lex.ids.tolist() == [1, 2, 3, 4, 4, 4] and lex.max_entry_len == 3
    assert lex.padded().tolist() == [[1, 2, 3], [4, 0, 0], [4, 4, 0]]
    for bad in ([[]], [[0, 1]], [[63]], [[1, 64]], [[-1]], [[1] * 64], []):
        with pytest.raises(ValueError):
            engine.Lexicon(bad, device="cpu")
    assert len(engine.Lexicon([[62] * 63], device="cpu")) == 1


# ------------------------------------------------------------------------------------------------------------- scores
@pytest.mark.parametrize("blank", [0, 17, 63])
def test_score_reference_is_minus_the_ctc_cost(blank):
    rng = np.random.default_rng(20 + blank)
    T, N, J = 12, 6, 5
    x = torch.tensor(rng.normal(0, 2.0, size=(T, N, 64)).astype(np.float32))
    il = np.array([T, T, 5, 1, 0, T + 3], np.int32)
    entries = [list(R.draw_labels(rng, int(L), blank)) for L in rng.integers(0, 7, size=12)]
    entries[0] = [entries[1][0]] * 4 if entries[1] else [5, 5, 5, 5]                 # repeats
    entries[2] = [blank if blank else 7, 3]                                         # invalid at blank != 0 ... and below
    entries[3] = [70, 1]                                                            # invalid: outside [0, 64)
    cand = rng.integers(-1, len(entries), size=(N, J))
    cand[0, :4] = [0, 1, 2, 3]
    sc, allow = X.score_fp64(x, il, entries, cand, blank)
    for n in range(N):
        for j in range(J):
            k = int(cand[n, j])
            if k < 0:
                assert sc[n, j] == -np.inf
                continue
            e = entries[k]
            if any(v == blank or not 0 <= v < 64 for v in e):
                assert np.isnan(sc[n, j])
                continue
            if not e:                                   # the all-blank path (ctc_fp64 needs a label)
                Tn = min(max(int(il[n]), 0), T)
                assert abs(sc[n, j] - float(torch.log_softmax(x[:Tn, n].double(), 1)[:, blank].sum())) < 1e-9
                continue
            ref = R.ctc_fp64(x[:, n:n + 1], np.array(e, np.int64), [len(e)], [il[n]], blank=blank)
            if not bool(ref["feasible"][0]):
                assert sc[n, j] == (0.0 if (len(e) == 0 and min(max(il[n], 0), T) == 0) else -np.inf), (n, j)
                continue
            assert abs(sc[n, j] + float(ref["costs"][0])) < 1e-9, (n, j)
            assert 0 < allow[n, j] < 1e-2


def test_score_reference_equals_path_enumeration():
    rng = np.random.default_rng(5)
    Cn = 4                                               # small alphabet: classes 4 .. 63 get -inf logits
    T, N = 5, 4
    xs = np.full((T, N, 64), -1e30, np.float32)
    xs[:, :, :Cn] = rng.normal(0, 1.0, size=(T, N, Cn))
    x = torch.tensor(xs)
    entries = [[], [1], [1, 1], [2, 3], [1, 2, 1], [3, 3, 3]]
    cand = np.tile(np.arange(len(entries)), (N, 1))
    il = [T, 4, 3, 2]
    sc, _ = X.score_fp64(x, il, entries, cand, 0)
    lp = torch.log_softmax(x.double(), 2).numpy()
    for n in range(N):
        for j, e in enumerate(entries):
            ref = X.enumerate_score(lp[:il[n], n, :Cn], e, il[n], 0)
            assert (sc[n, j] == ref == -np.inf) or abs(sc[n, j] - ref) < 1e-9, (n, j, sc[n, j], ref)


def test_selection_tie_rule():
    score = np.array([[-1.0, -1.0, -3.0], [-np.inf, np.nan, -2.0], [-np.inf, np.nan, -np.inf], [-0.5, -0.25, -0.25]])
    cand = np.array([[7, 3, 1], [2, 4, 9], [1, 2, -1], [5, 6, 0]])
    best, slot, margin = X.select_ref(score, cand)
    assert list(best) == [7, 9, -1, 6] and list(slot) == [0, 2, -1, 1]
    assert margin[0] == 0.0 and margin[1] == np.inf and margin[3] == 0.0


# ------------------------------------------------------------------------------------------------------------- loader, cfg
def test_word_list_loader(tmp_path):
    from lstm_ctc_ocr_b200.lib.lstm.lexicon import load_lexicon
    p = tmp_path / "words.txt"
    p.write_text("abc\n\n  Z9 \r\nabc\n", encoding="utf-8")
    assert load_lexicon(str(p)) == [(11, 12, 13), (62, 10), (11, 12, 13)]
    p.write_text("ok\nbad-word\n", encoding="utf-8")
    with pytest.raises(ValueError, match=r"words.txt:2"):
        load_lexicon(str(p))
    p.write_text("ok\n\nnäh\n", encoding="utf-8")
    with pytest.raises(ValueError, match=r"words.txt:3"):
        load_lexicon(str(p))
    p.write_text("\n\n", encoding="utf-8")
    with pytest.raises(ValueError):
        load_lexicon(str(p))


def test_cfg_defaults_and_merges(tmp_path):
    from lstm_ctc_ocr_b200.lib.lstm import config as K
    assert K.cfg.TEST.LEXICON == "" and K.cfg.TEST.LEXICON_MAX_EDIT == 3 and K.cfg.TEST.LEXICON_CANDIDATES == 64
    try:
        K.cfg_from_list(["TEST.LEXICON", "words.txt", "TEST.LEXICON_MAX_EDIT", "-1", "TEST.LEXICON_CANDIDATES", "256"])
        assert K.cfg.TEST.LEXICON == "words.txt" and K.cfg.TEST.LEXICON_MAX_EDIT == -1 and K.cfg.TEST.LEXICON_CANDIDATES == 256
        y = tmp_path / "c.yml"
        y.write_text("TEST:\n  LEXICON: other.txt\n  LEXICON_MAX_EDIT: 2\n")
        K.cfg_from_file(str(y))
        assert K.cfg.TEST.LEXICON == "other.txt" and K.cfg.TEST.LEXICON_MAX_EDIT == 2
        with pytest.raises(AssertionError):
            K.cfg_from_list(["TEST.LEXICON_MAX_EDIT", "two"])
    finally:
        K.cfg.TEST.LEXICON, K.cfg.TEST.LEXICON_MAX_EDIT, K.cfg.TEST.LEXICON_CANDIDATES = "", 3, 64


# ------------------------------------------------------------------------------------------------------------- ABI
def test_header_ctypes_and_binding_table_agree_on_the_lexicon_entries():
    from lstm_ctc_ocr_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "crnn_ctc.h")).read(), flags=re.S)
    for name, nargs in (("crnn_lexicon_candidates", 14), ("crnn_ctc_lexicon_score", 15)):
        m = re.search(r"\bint\s+" + name + r"\s*\(([^;]*)\)\s*;", src)
        assert m, name
        assert len([p for p in m.group(1).split(",") if p.strip()]) == nargs
        assert len(_lib.SIGNATURES[name][1]) == nargs
        assert hasattr(_lib.load(), name)


def test_status_codes_without_touching_the_device():
    """Argument checks come before any launch: null pointers, bad shapes and unsupported limits return without a CUDA call."""
    from lstm_ctc_ocr_b200 import _lib
    lib = _lib.load()
    p = 16                                                  # never dereferenced: every call below fails its checks first
    assert lib.crnn_lexicon_candidates(0, 8, p, 4, p, p, 10, 15, 3, 64, p, p, p, None) == 1
    assert lib.crnn_lexicon_candidates(p, 8, p, 4, p, p, 10, 15, 3, 257, p, p, p, None) == 1
    assert lib.crnn_lexicon_candidates(p, 8, p, 4, p, p, 10, 15, 3, 0, p, p, p, None) == 1
    assert lib.crnn_lexicon_candidates(p, 8, p, 4, p, p, 10, 64, 3, 64, p, p, p, None) == 4
    assert lib.crnn_lexicon_candidates(p, 1025, p, 4, p, p, 10, 15, 3, 64, p, p, p, None) == 4
    assert lib.crnn_ctc_lexicon_score(p, p, 63, 4, 64, 0, p, p, 15, p, 64, p, p, 0, None) == 1
    assert lib.crnn_ctc_lexicon_score(p, p, 769, 4, 64, 0, p, p, 15, p, 64, p, p, p, None) == 4
    assert "769" in lib.crnn_last_error().decode()
    assert lib.crnn_ctc_lexicon_score(p, p, 63, 4, 65, 0, p, p, 15, p, 64, p, p, p, None) == 4
    assert lib.crnn_ctc_lexicon_score(p, p, 63, 4, 64, 0, p, p, 64, p, 64, p, p, p, None) == 4
    assert "64" in lib.crnn_last_error().decode()
    assert lib.crnn_ctc_lexicon_score(p, p, 63, 4, 64, 64, p, p, 15, p, 64, p, p, p, None) == 1


def test_lexicon_calls_fail_loudly_without_a_gpu():
    from lstm_ctc_ocr_b200 import CrnnError, engine
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lex = engine.Lexicon([[1, 2]], device="cpu")
    i = torch.ones(1, dtype=torch.int32)
    with pytest.raises(CrnnError):
        engine.lexicon_candidates(torch.ones((1, 2), dtype=torch.int32), i, lex)
    with pytest.raises(CrnnError):
        engine.ctc_lexicon_score(torch.zeros((4, 1, 64)), i, lex, torch.zeros((1, 1), dtype=torch.int32))


def test_torch_dp_and_candidates_equal_the_numpy_references():
    """The GPU tests' reference (lexicon_refs.distances_torch / candidates_torch) against levenshtein_dp / candidates_ref, on the CPU."""
    rng = np.random.default_rng(8)
    entries = [list(rng.integers(-1, 66, size=rng.integers(1, 10))) for _ in range(60)]
    reads = [list(rng.integers(0, 6, size=rng.integers(0, 14))) + [int(rng.integers(60, 70))] * int(rng.integers(0, 2)) for _ in range(40)]
    M = max(len(r) for r in reads)
    rd = np.zeros((len(reads), M), np.int64)
    for i, r in enumerate(reads):
        rd[i, :len(r)] = r
    el = np.array([len(e) for e in entries])
    E = np.zeros((len(entries), el.max()), np.int64)
    for k, e in enumerate(entries):
        E[k, :len(e)] = e
    D = X.distances_torch(torch.tensor(rd), torch.tensor([len(r) for r in reads]), torch.tensor(E), torch.tensor(el))
    ref = X.pair_distances(rd, [len(r) for r in reads], entries)
    assert np.array_equal(D.numpy(), ref)
    for delta, mc in ((0, 3), (2, 5), (-1, 64), (-1, 1)):
        got, want = X.candidates_torch(D, delta, mc), X.candidates_ref(ref, delta, mc)
        assert all(np.array_equal(g.numpy(), w) for g, w in zip(got, want)), (delta, mc)
