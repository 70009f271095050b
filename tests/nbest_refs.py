"""References for the n-best beam-search decoders (crnn_ctc_beam_search_topk, crnn_ctc_beam_search_topk_device).

  - beam_search_topk: TensorFlow's CTCBeamSearchDecoder with top_paths, restated in Python: the beam of
    oracle.crnn_oracle.beam_search_decode, frame for frame, ending in TopPaths -- the listed entries by total, highest first,
    exact ties in insertion order.  Its path 0 is beam_search_decode's result.
  - check_exhaustive_topk / check_lower_bound_topk: the top-k version of beam_refs' checks against the fp64 exact prefix
    search.  Where the beam never evicts a finite entry and no frame makes the blank impossible, it lists every prefix of
    non-zero probability, so paths 0 .. K-1 are the K most probable prefixes with their exact log-probabilities; where it
    prunes, each path's total sums a subset of its prefix's alignments and is a lower bound on log P(prefix).
    Why the blank matters: TF's visit of a branch wipes a child it rejects, and on a frame whose blank (and the child's own
    label) has probability 0 a listed child re-scores to -inf and its parent's extension of it is rejected too; the wipe then
    keeps the child from being expanded in that frame, although its own extensions have non-zero probability.  The child
    comes after its parent in the frame's order, so the best entry is never lost this way (beam_refs' single-best claim
    holds), but runners-up are: beam_refs.sparse_case has such frames, sparse_live_blank_batch does not.

Test infrastructure only (imported by tests/)."""
import math

import numpy as np

from beam_refs import (DENSE_GRID, NEG, decided, dense_case, exact_prefix_search, expected, labelling_logp, lower_bound_slack,
                       references, sparse_case, within_one_ulp)
from oracle.crnn_oracle import _Beam


def _lse(a, b):
    return (max(a, b) + np.log1p(np.exp(-abs(a - b)))) if max(a, b) > -np.inf else -np.inf


def beam_search_topk(logits, input_len, beam_width=100, top_paths=1, merge_repeated=True, strip=0):
    """Per utterance, a list of (labels, total) for its min(top_paths, listed entries) best entries, in the decoders' order.
    The frame loop is oracle.crnn_oracle.beam_search_decode's, with the decoders' rule for NaN logits; the end is TopPaths."""
    x = np.asarray(logits, dtype=np.float64)
    T, N, C = x.shape
    blank = C - 1
    out = []
    for n in range(N):
        root = _Beam(None, -1)
        root.new = [0.0, 0.0, -np.inf]
        leaves = [root]
        for t in range(int(input_len[n])):
            row = x[t, n]
            live = ~np.isnan(row)                      # the decoders' rule: a NaN logit counts as -inf, and a frame without a
            mx = float(row[live].max()) if live.any() else -np.inf        # finite normaliser makes every class impossible
            se = 0.0
            for v in row[live]:
                se += math.exp(float(v) - mx)
            norm = mx + math.log(se) if se > 0 and se == se else float("nan")
            lp = np.where(live, row - norm, -np.inf) if norm == norm else np.full(C, -np.inf)
            branches = sorted(leaves, key=lambda b: -b.new[0])
            leaves = []
            for b in branches:
                b.old = list(b.new)
            for b in branches:
                if b.parent is not None:
                    if b.parent.active():
                        prev = b.parent.old[1] if b.label == b.parent.label else b.parent.old[0]
                        b.new[2] = _lse(b.new[2], prev)
                    b.new[2] += lp[b.label]
                b.new[1] = b.old[0] + lp[blank]
                b.new[0] = _lse(b.new[1], b.new[2])
                leaves.append(b)
            bottom = lambda: min(leaves, key=lambda e: e.new[0])
            state = {"bot": bottom().new[0]}

            def is_candidate(total):
                return total > -np.inf and (len(leaves) < beam_width or total > state["bot"])
            for b in branches:
                if not is_candidate(b.old[0]):
                    continue
                if b.children is None:
                    b.children = {}
                base = np.full(C - 1, b.old[0])
                if 0 <= b.label < C - 1:
                    base[b.label] = b.old[1]
                cand = base + lp[:C - 1]
                if len(leaves) < beam_width:
                    visit = range(C - 1)
                else:
                    visit = sorted(set(np.nonzero(cand > state["bot"])[0].tolist()) | set(b.children))
                for c in visit:
                    ch = b.children.get(c)
                    if ch is not None and ch.active():
                        continue
                    total = float(cand[c])
                    if is_candidate(total):
                        if ch is None:
                            ch = b.children[c] = _Beam(b, c)
                        ch.new = [total, -np.inf, total]
                        if len(leaves) == beam_width:
                            bt = bottom()
                            bt.new = [-np.inf, -np.inf, -np.inf]
                            leaves.remove(bt)
                        leaves.append(ch)
                        state["bot"] = bottom().new[0]
                    elif ch is not None:
                        ch.old = [-np.inf, -np.inf, -np.inf]
                        ch.new = [-np.inf, -np.inf, -np.inf]
        ranked = sorted(leaves, key=lambda e: -e.new[0])          # stable: exact ties keep insertion order
        out.append([([v for v in e.label_seq(merge_repeated) if v != strip], e.new[0]) for e in ranked[:top_paths]])
    return out


def _ranked(P):
    """The exact search's labellings by log P, highest first (ties by labelling, so the order does not depend on dict order)."""
    return sorted(P.items(), key=lambda kv: (-kv[1], kv[0]))


def check_exhaustive_topk(paths, logp, num_paths, refs, top_paths, merge_repeated, strip, stats):
    """One top-k decode of utterances whose beam was exhaustive against the exact search.  paths[n][i]: labels of path i,
    logp [N, K] f32, num_paths [N].  Path i < min(K, M) (M prefixes of non-zero probability) must carry the i-th largest exact
    log P within one f32 ulp; its labels must be expected() of that prefix, or, when its probability lies within the `decided`
    threshold of a neighbour's, of one prefix of that run of near-ties.  Listed paths past M have log_prob -inf; paths past
    num_paths are empty with -inf.  Adds to `stats` and returns the failures."""
    bad = []
    for n, (P, _) in enumerate(refs):
        items = _ranked(P)
        M = len(items)
        vals = [v for _, v in items]
        stats["lines"] += 1
        real = int(num_paths[n])
        if not min(top_paths, M) <= real <= top_paths:
            bad.append(("num_paths", n, real, M))
        for i in range(top_paths):
            if i < min(top_paths, M, real):
                lo, hi = i, i
                while lo > 0 and not decided(vals[lo - 1], vals[lo]):
                    lo -= 1
                while hi + 1 < M and not decided(vals[hi], vals[hi + 1]):
                    hi += 1
                stats["decided" if lo == hi else "undecided"] += 1
                allowed = [expected(items[j][0], merge_repeated, strip) for j in range(lo, hi + 1)]
                if list(paths[n][i]) not in allowed:
                    stats["label_fail"] += 1
                    bad.append(("label", n, i, list(paths[n][i]), allowed[:3]))
                if not within_one_ulp(logp[n][i], np.float32(vals[i])):
                    stats["logp_fail"] += 1
                    bad.append(("log_prob", n, i, float(logp[n][i]), vals[i]))
            elif i < real:
                stats["listed_zero"] += 1
                if logp[n][i] != NEG:
                    bad.append(("listed past the non-zero prefixes", n, i, float(logp[n][i])))
            elif list(paths[n][i]) != [] or logp[n][i] != NEG:
                bad.append(("padding", n, i, list(paths[n][i]), float(logp[n][i])))
    return bad


def new_stats():
    return dict(lines=0, decided=0, undecided=0, label_fail=0, logp_fail=0, listed_zero=0)


def check_lower_bound_topk(x, il, paths, logp, num_paths):
    """On a merge_repeated=False, strip=-1 decode (the labels are the prefix itself): every real path of finite total has
    log_prob <= log P(prefix) plus one f32 ulp, log P by the CTC forward DP.  Returns (failures, slack in ulps)."""
    bad, slack = [], []
    K = logp.shape[1]
    for i in range(K):
        rows = [n for n in range(len(il)) if i < num_paths[n] and np.isfinite(logp[n][i])]
        if not rows:
            continue
        lines = [list(paths[n][i]) for n in rows]
        lp = labelling_logp(np.ascontiguousarray(x[:, rows]), np.asarray(il)[rows], lines)
        ulps, _ = lower_bound_slack(-np.asarray([logp[n][i] for n in rows], np.float32), lp)
        bad += [("lower_bound", rows[k], i, lines[k], float(logp[rows[k]][i]), float(lp[k])) for k in np.flatnonzero(~(ulps >= -1.0))]
        slack.append(ulps)
    return bad, np.concatenate(slack) if slack else np.zeros(0)


def run_exhaustive_topk(decode, cases, widths=(128, 33, "peak"), ks=(1, 2, 7, "width")):
    """Decode every beam_refs.exhaustive_cases case at every width, K and output mode; lines whose measured prefix count fits
    the width go through check_exhaustive_topk.  `decode(x, il, width, K, merge_repeated, strip)` -> (paths [N][K] label
    lists, log_prob [N,K], num_paths [N]).  "peak" decodes each line at its own measured prefix count.  Returns (stats,
    failures)."""
    from beam_refs import MODES
    st = new_stats()
    bad = []
    for name, x, il, refs in cases:
        peak = np.array([p for _, p in refs])
        groups = []
        for w in widths:
            if w == "peak":
                groups += [(int(p), np.flatnonzero(peak == p)) for p in np.unique(peak)]
            else:
                groups.append((w, np.arange(len(il))))
        for width, idx in groups:
            xs, ils = np.ascontiguousarray(x[:, idx]), il[idx]
            ex = [k for k in range(len(idx)) if peak[idx[k]] <= width]
            if not ex:
                continue
            for K in sorted({width if k == "width" else min(k, width) for k in ks}):
                for merge, strip in MODES:
                    paths, logp, npaths = decode(xs, ils, width, K, merge, strip)
                    for b in check_exhaustive_topk([paths[k] for k in ex], logp[ex], npaths[ex], [refs[idx[k]] for k in ex], K,
                                                   merge, strip, st):
                        bad.append((name, width, K, merge, strip) + b)
    return st, bad


def reference_topk_decoder(mutant):
    """A top-k decoder made of the exact search (or one of beam_refs' controls): its K most probable labellings; width
    ignored."""
    def decode(x, il, width, K, merge_repeated, strip):
        N = x.shape[1]
        paths = [[[] for _ in range(K)] for _ in range(N)]
        logp = np.full((N, K), NEG, np.float32)
        npaths = np.zeros(N, np.int32)
        for n, (P, _) in enumerate(references(x, il, mutant)):
            items = _ranked(P)[:K]
            npaths[n] = len(items)
            for i, (lab, v) in enumerate(items):
                paths[n][i] = expected(lab, merge_repeated, strip)
                logp[n, i] = np.float32(v)
        return paths, logp, npaths
    return decode


def exact_top(x_n, length, K):
    """The K most probable labellings of one utterance and their log P (the exact search)."""
    return _ranked(exact_prefix_search(x_n, length)[0])[:K]


def sparse_live_blank_batch(T, width, count, seed0=0):
    """beam_refs.sparse_batch with every -inf blank of sparse_case set to a finite logit (0.0): mostly blank-only frames, a few
    with two labels, a label repeated over three frames, and no frame whose blank is impossible.  Returns (x, input_len)."""
    xs = []
    s = seed0
    while len(xs) < count:
        x = sparse_case(T, s)
        x[np.isneginf(x[:, 0, -1]), 0, -1] = 0.0
        if exact_prefix_search(x[:, 0], T)[1] <= width:
            xs.append(x)
        s += 1
    return np.concatenate(xs, axis=1), np.full(count, T, np.int32)


def exhaustive_topk_cases(N=24):
    """(name, x, input_len, references): beam_refs' dense grid and sparse_live_blank_batch at T = 63 and 255."""
    out = []
    for C, T in DENSE_GRID:
        x, il = dense_case(C, T, N, seed=1000 * C + T)
        out.append((f"dense_C{C}_T{T}", x, il, references(x, il)))
    for T in (63, 255):
        x, il = sparse_live_blank_batch(T, 128, 6)
        out.append((f"sparse_live_blank_T{T}", x, il, references(x, il)))
    return out
