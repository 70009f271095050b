"""The host beam-search decoder (crnn_ctc_beam_search, csrc/beam.cpp) and the oracle's restatement of TF's
CTCBeamSearchDecoder against the fp64 exact prefix search of tests/beam_refs.py, without a GPU.

Where the beam is exhaustive (every frame's count of non-zero prefixes fits the width) the decoder's labelling must be the
most probable one and its neg_log_prob that labelling's -log P within one f32 ulp; where it prunes, neg_log_prob may only
overstate -log P(out).  Each check is shown to reject a decoder that is wrong in the way it targets.  Counts go to
build/beam_exact_report.jsonl."""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import beam_refs as BR  # noqa: E402
import ctc_refs as R  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def report(**row):
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    with open(os.path.join(ROOT, "build", "beam_exact_report.jsonl"), "a") as f:
        f.write(json.dumps(row) + "\n")
    print(json.dumps(row))


def host_decoder(x, il, width, merge_repeated, strip):
    from lstm_ctc_ocr_b200 import engine
    out, out_len, nlp = engine.ctc_beam_search(x, il, beam_width=width, merge_repeated=merge_repeated, strip=strip)
    return [out[i, :out_len[i]].tolist() for i in range(len(il))], nlp


def oracle_decoder(x, il, width, merge_repeated, strip):
    from oracle import crnn_oracle as O
    return O.beam_search_decode(x, il, beam_width=width, merge_repeated=merge_repeated, strip=strip), np.zeros(len(il), np.float32)


@pytest.fixture(scope="module")
def cases():
    return BR.exhaustive_cases()


def test_exact_search_sums_to_one_and_equals_the_ctc_forward(cases):
    """Every alignment collapses to exactly one labelling, so sum_l P(l | x) = 1; each labelling's log P equals the fp64 CTC
    forward probability (torch.ctc_loss, and ctc_refs.ctc_fp64 at C = 64) and, at T <= 6, the sum over every frame path."""
    checked = enumerated = 0
    for name, x, il, refs in cases:
        C = x.shape[2]
        for n, (P, _) in enumerate(refs):
            assert abs(math.fsum(math.exp(v) for v in P.values()) - 1.0) < 1e-12, (name, n)
            labs = list(P)
            lp = BR.labelling_logp(np.repeat(x[:, n:n + 1], len(labs), axis=1), np.full(len(labs), il[n]), labs)
            ex = np.array([P[l] for l in labs])
            assert np.all(np.abs(lp - ex) <= 1e-12 * (1 + np.abs(ex))), (name, n)
            if C == 64 and il[n] > 0:
                xs = torch.tensor(np.repeat(x[:, n:n + 1], len(labs), axis=1))
                lab = np.array([v for l in labs for v in l] or [0], np.int64)
                r = R.ctc_fp64(xs, lab, [len(l) for l in labs], np.full(len(labs), il[n]), blank=63)
                got = -r["costs"].numpy()
                assert np.all(np.abs(got - ex) <= 1e-12 * (1 + np.abs(ex))), (name, n)
            if il[n] <= 6 and C ** int(il[n]) <= 4096:
                E = BR.path_enumeration(x[:, n], int(il[n]))
                assert set(E) == set(P), (name, n)
                assert all(abs(E[l] - P[l]) <= 1e-12 * (1 + abs(P[l])) for l in P), (name, n)
                enumerated += 1
            checked += len(labs)
    report(test="exact_search_self_check", labellings=checked, enumerated_lines=enumerated)
    assert enumerated > 0


def test_host_decoder_equals_the_exact_search(cases):
    """Widths 128, 33, each line's measured count and one below it; both merge modes, strip 0 and -1."""
    st, bad, slack = BR.run_exhaustive(host_decoder, cases)
    report(test="host_exhaustive", min_slack_ulps=float(slack.min()), **st)
    assert not bad, bad[:5]
    assert st["decided"] > 0 and st["pruned"] > 0


def test_host_decoder_lower_bound_on_pruned_decodes():
    """Dense frames far beyond the width, C 3 ... 64 at T = 19 and 63, widths 1 ... 128: neg_log_prob >= -log P(out)."""
    st = dict(bound_fail=0)
    bad, slack = [], []
    for name, x, il in BR.pruned_cases():
        for width in (1, 2, 7, 33, 64, 100, 128):
            lines, nlp = host_decoder(x, il, width, False, -1)
            b, s = BR.check_lower_bound(x, il, lines, nlp, st)
            bad += [(name, width) + e for e in b]
            slack.append(s)
    slack = np.concatenate(slack)
    report(test="host_lower_bound", min_slack_ulps=float(slack.min()), median_slack_ulps=float(np.median(slack)), **st)
    assert not bad, bad[:5]


def test_oracle_restatement_equals_the_exact_search(cases):
    """oracle.beam_search_decode's labellings at width 128 and each line's measured count (its neg_log_prob is not
    reported, so only the labelling is checked)."""
    st = BR.new_stats()
    bad = []
    for name, x, il, refs in cases:
        peak = np.array([p for _, p in refs])
        for merge, strip in ((True, 0), (False, -1)):
            for width in (128, "peak"):
                groups = [(128, np.arange(len(il)))] if width == 128 else [(int(p), np.flatnonzero(peak == p)) for p in np.unique(peak)]
                for w, idx in groups:
                    lines, _ = oracle_decoder(np.ascontiguousarray(x[:, idx]), il[idx], w, merge, strip)
                    for k, n in enumerate(idx):
                        best, l1, l2 = BR.top_two(refs[n][0])
                        st["lines"] += 1
                        if BR.decided(l1, l2):
                            st["decided"] += 1
                            if lines[k] != BR.expected(best, merge, strip):
                                bad.append((name, w, merge, strip, n, lines[k]))
                        else:
                            st["undecided"] += 1
    report(test="oracle_exhaustive", **st)
    assert not bad, bad[:5]


def test_controls_are_rejected(cases):
    """Each check rejects a decoder wrong in the way it targets: the best path (greedy) fails the labelling check on soft
    frames, a blank-only score the neg_log_prob check, a repeated label extended from the parent's total the labelling
    check or the lower bound."""
    soft = [(n, x, il, refs) for n, x, il, refs in cases if n.startswith("dense")]
    rows = {}
    for mutant in ("best_path", "blank_only_score", "repeat_from_total"):
        st, _, _ = BR.run_exhaustive(BR.reference_decoder(mutant), soft, widths=(128,))
        rows[mutant] = st
        report(test="control", mutant=mutant, **st)
    assert rows["best_path"]["label_fail"] > 0
    assert rows["blank_only_score"]["nlp_fail"] > 0
    assert rows["repeat_from_total"]["label_fail"] + rows["repeat_from_total"]["bound_fail"] > 0
    st, bad, _ = BR.run_exhaustive(BR.reference_decoder(None), soft, widths=(128,))
    assert not bad, bad[:3]
