"""CPU checks of CTC forced alignment (crnn_ctc_align): the fp64 restatement in align_refs against exhaustive enumeration, against
the oracle's CTC cost and against the greedy read; the C ABI's size query, the header and the ctypes table; no CPU fallback."""
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import align_refs as A  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("seed", range(4))
def test_reference_equals_brute_force_with_ties(seed):
    """Every path enumerated at T <= 8, C = 4, L <= 3 on emissions of a 1/8 grid (exact sums, frequent ties): the same best score,
    the same path under the tie rules, and the margin of the two best distinct paths."""
    cases = ties = 0
    for e, skip, seq, _lp, _blank in A.small_cases(seed, 150):
        best, path, npaths = A.brute_force(e, skip)
        v = A.viterbi_ext(e, skip)
        Tn, S = e.shape
        if npaths == 0:
            assert v["path"] is None and v["score"] == -np.inf
            continue
        cases += 1
        assert v["score"] == best
        np.testing.assert_array_equal(v["path"], path)
        scores = sorted((sum(e[t, p[t]] for t in range(Tn)) for p in A.all_paths(Tn, S, skip)), reverse=True)
        second = scores[1] if len(scores) > 1 else -np.inf
        assert v["margin"] == best - second
        ties += int(second == best)
        st, en = A.spans_of(path)
        np.testing.assert_array_equal(A.path_of_spans(st, en, Tn), path)
        assert abs(A.count_paths(Tn, skip) - np.log(npaths)) < 1e-12
    assert cases > 80 and ties > 10, (cases, ties)


def test_tie_rules_on_a_flat_row():
    """All emissions equal: every path ties; the rules stay in the later state as long as possible (end in S-1, enter each
    label as late as the frames allow)."""
    e = np.full((5, 5), -1.0)
    _, skip = A.ext_of([1, 2], 0)
    v = A.viterbi_ext(e, skip)
    np.testing.assert_array_equal(v["path"], [1, 3, 4, 4, 4])
    assert v["margin"] == 0.0


def test_best_path_lies_between_the_oracle_cost_and_the_cost_minus_log_paths():
    """max_path log p(path) <= log p(labels) = -cost <= max_path + log(#paths)."""
    from oracle import crnn_oracle as O
    rng = np.random.default_rng(7)
    T, N = 12, 16
    x = rng.normal(0, 2.0, size=(T, N, 64)).astype(np.float32)
    ll = rng.integers(0, 6, size=N).astype(np.int32)
    ll[0], ll[1] = 0, 6
    il = rng.integers(1, T + 1, size=N).astype(np.int32)     # the oracle needs a frame
    il[2] = T
    lab = rng.integers(1, 64, size=int(ll.sum())).astype(np.int32)
    lab[:3] = 5                                                   # a repeat
    R = A.align_fp64(x, lab, ll, il)
    costs, _ = O.ctc_loss_np(x.astype(np.float64), lab, ll, il, want_grad=False)
    checked = 0
    for n in range(N):
        if not R["feasible"][n]:
            assert R["score"][n] == -np.inf
            continue
        sc = R["score"][n]
        _, skip = A.ext_of(A.to_rows(lab, ll)[n], 0)
        logn = A.count_paths(R["Tn"][n], skip) if R["Tn"][n] else 0.0
        assert sc <= -costs[n] + 1e-9
        assert sc >= -costs[n] - logn - 1e-9
        checked += 1
    assert checked >= 8


def test_greedy_read_aligns_on_its_argmax_runs():
    """On peaked logits whose argmax never hits 63 and has no tied frame, the alignment of the greedy read (blank 0) is the
    argmax path: spans are the argmax runs and the score is sum_t max_c log y_t(c)."""
    rng = np.random.default_rng(3)
    T, N = 40, 64
    x = rng.normal(0, 1.0, size=(T, N, 64)).astype(np.float32)
    hot = np.where(rng.random((T, N)) < 0.5, 0, rng.integers(1, 5, size=(T, N)) * 7)     # few classes: repeats and runs
    np.put_along_axis(x, hot[..., None], 6.0 + rng.random((T, N, 1)).astype(np.float32), axis=2)
    il = rng.integers(T // 2, T + 1, size=N).astype(np.int32)
    reads, runs = [], []
    for n in range(N):
        r, s, e = A.argmax_runs(x[:, n], int(il[n]))
        reads.append(r); runs.append((s, e))
    ll = np.array([len(r) for r in reads], np.int32)
    lab = np.array([v for r in reads for v in r], np.int32)
    R = A.align_fp64(x, lab, ll, il)
    lp, _ = A.log_softmax(x)
    for n in range(N):
        np.testing.assert_array_equal(R["start"][n], runs[n][0])
        np.testing.assert_array_equal(R["end"][n], runs[n][1])
        assert abs(R["score"][n] - lp[:il[n], n].max(axis=1).sum()) < 1e-9
    # dense rows give the same alignment as the flat layout
    dense = np.zeros((N, max(ll.max(), 1)), np.int32)
    for n, r in enumerate(reads):
        dense[n, :len(r)] = r
    Rd = A.align_fp64(x, dense, ll, il)
    assert all(np.array_equal(a, b) for a, b in zip(R["start"], Rd["start"])) and R["score"] == Rd["score"]


def test_workspace_size_query_and_its_status_codes():
    """crnn_ctc_align_workspace_size makes no CUDA call: T * (8 + S_pad) bytes per utterance plus 256; CRNN_UNSUPPORTED for
    C != 64 and max_label_len above 639, CRNN_INVALID_VALUE for bad arguments."""
    from lstm_ctc_ocr_b200 import CrnnError, _lib, engine
    for T, N, m in ((63, 1024, 30), (1, 1, 0), (2048, 300, 639)):
        s_pad = (2 * m + 1 + 3) // 4 * 4
        assert engine.ctc_align_workspace_bytes(T, N, 64, m) == T * N * (8 + s_pad) + 256
    lib = _lib.load()
    nb = _lib.c_size_t()
    assert lib.crnn_ctc_align_workspace_size(63, 4, 65, 10, nb) == 4
    assert lib.crnn_ctc_align_workspace_size(63, 4, 64, 640, nb) == 4
    assert lib.crnn_ctc_align_workspace_size(0, 4, 64, 10, nb) == 1
    assert lib.crnn_ctc_align_workspace_size(63, 4, 64, -1, nb) == 1
    with pytest.raises(CrnnError):
        engine.ctc_align_workspace_bytes(63, 4, 64, 640)


def test_header_ctypes_and_binding_table_agree_on_the_align_entries():
    from lstm_ctc_ocr_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "crnn_ctc.h")).read(), flags=re.S)
    for name, nargs in (("crnn_ctc_align_workspace_size", 5), ("crnn_ctc_align", 17)):
        m = re.search(r"\bint\s+" + name + r"\s*\(([^;]*)\)\s*;", src)
        assert m, name
        assert len([p for p in m.group(1).split(",") if p.strip()]) == nargs
        assert len(_lib.SIGNATURES[name][1]) == nargs
        assert hasattr(_lib.load(), name)


def test_ctc_align_fails_loudly_without_a_gpu():
    import torch
    from lstm_ctc_ocr_b200 import CrnnError, engine
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    x = torch.zeros((4, 1, 64))
    i = torch.ones(1, dtype=torch.int32)
    with pytest.raises(CrnnError):
        engine.ctc_align(x, torch.ones(1, dtype=torch.int32), i, i)
