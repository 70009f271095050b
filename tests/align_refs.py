"""fp64 restatement of crnn_ctc_align (csrc/align.cu, include/crnn_ctc.h) and the bounds its results are checked against.

viterbi_ext() runs the max-plus recursion over log-probabilities with the kernel's tie rules -- among predecessors s beats s-1 beats
s-2, at the end S-1 beats S-2 -- and keeps, beside the best, the second-best path score per state, so each utterance's margin
(best minus second-best complete path, over distinct paths) is known.  With exact arithmetic those rules pick, among the
optimal paths, the one whose state sequence read from the last frame back is lexicographically largest: brute_force() states
that directly, by enumerating every path.

Bounds (f32, u = 2^-24), analytic, from the kernel's arithmetic:
  emission   e = x - lse with lse = m + log(sum_c exp(x_c - m)) (m exact, expf <= 2 ulp, logf <= 1 ulp, a 6-deep add tree):
             the sum's relative error is at most u*(ln 64 + 4 + 6) (the posterior-weighted mean of x_c - m is below ln 64), log
             adds 2u*ln 64 absolute, m + log and x - lse one rounding each:  |e32 - e| <= u * (|lse| + |e| + 32)  (emission_err)
  path       a path's f32 score is its emissions added frame by frame (max picks a value exactly):
             eps(P) = sum_t emission_err_t(P) + 1.01 * u * sum_{t>=1} |V_t(P)|, V_t the partial sums  (path_eps)
  optimum    f32 addition is monotonic, so the kernel's score of its path is at least its score of any other path:
             |score(P_gpu) - score(P_opt)| <= eps(P_gpu) + eps(P_opt); paths differ only where the margin is below that sum.
  peak       exp of an emission: relative error <= emission_err + 6u (expf, the store)  (peak_rel_err)

Test infrastructure only (imported by tests/)."""
import math

import numpy as np

C = 64
U = 2.0 ** -24
NEG = -np.inf


def log_softmax(x):
    """x [T, N, C] (any float) -> (lp, lse) in fp64: lp = x - lse, lse [T, N]."""
    xd = np.asarray(x, np.float64)
    m = xd.max(axis=2, keepdims=True)
    lse = (m + np.log(np.exp(xd - m).sum(axis=2, keepdims=True)))[..., 0]
    return xd - lse[..., None], lse


def to_rows(labels, label_len):
    """Flat labels ([sum L]) or dense rows ([N, M]) -> list of per-utterance id lists (None where the length is negative)."""
    labels, ll = np.asarray(labels), np.asarray(label_len, np.int64)
    rows = []
    if labels.ndim == 2:
        for n, L in enumerate(ll):
            rows.append(None if L < 0 or L > labels.shape[1] else [int(v) for v in labels[n, :L]])
        return rows
    off = 0
    for L in ll:
        rows.append(None if L < 0 else [int(v) for v in labels[off:off + L]])
        off += int(L)
    return rows


def ext_of(seq, blank):
    """(blank, l_1, blank, ..., l_L, blank) and the skip mask: s-2 -> s allowed."""
    ext = [blank]
    for v in seq:
        ext += [v, blank]
    ext = np.array(ext, np.int64)
    skip = np.zeros(len(ext), bool)
    for s in range(2, len(ext)):
        skip[s] = ext[s] != blank and ext[s] != ext[s - 2]
    return ext, skip


def _top2(vals):
    """vals [k, S] -> the largest and second-largest per column (with multiplicity)."""
    srt = np.sort(vals, axis=0)
    return srt[-1], srt[-2]


def viterbi_ext(e, skip):
    """e [Tn, S] fp64 emissions along the extended labelling, skip [S] -> dict(score, path [Tn] states, margin) with the
    kernel's tie rules; score -inf when no path exists (path None)."""
    Tn, S = e.shape
    b1 = np.full(S, NEG)
    b2 = np.full(S, NEG)
    b1[:min(2, S)] = e[0, :min(2, S)]
    back = np.zeros((Tn, S), np.int64)
    for t in range(1, Tn):
        p1 = np.r_[NEG, b1[:-1]]
        p2 = np.where(skip, np.r_[NEG, NEG, b1[:-2]] if S >= 2 else np.full(S, NEG), NEG)[:S]
        q1 = np.r_[NEG, b2[:-1]]
        q2 = np.where(skip, np.r_[NEG, NEG, b2[:-2]] if S >= 2 else np.full(S, NEG), NEG)[:S]
        stack = np.stack([b1, p1, p2])
        back[t] = np.argmax(stack, axis=0)             # first maximum: s, then s-1, then s-2
        n1, n2 = _top2(np.stack([b1, p1, p2, b2, q1, q2]))
        b1, b2 = n1 + e[t], n2 + e[t]
    ends = [S - 1] + ([S - 2] if S >= 2 else [])
    s = S - 1 if S < 2 or not (b1[S - 2] > b1[S - 1]) else S - 2
    f1, f2 = _top2(np.array([[b1[i]] for i in ends] + [[b2[i]] for i in ends] + [[NEG]]))
    score, second = float(f1[0]), float(f2[0])
    if not score > NEG:
        return dict(score=score, path=None, margin=0.0)
    path = np.zeros(Tn, np.int64)
    path[-1] = s
    for t in range(Tn - 1, 0, -1):
        s -= back[t, s]
        path[t - 1] = s
    return dict(score=score, path=path, margin=score - second)


def all_paths(Tn, S, skip):
    """Every valid state sequence of Tn frames over S states (starts in 0 or 1, ends in S-1 or S-2)."""
    out = []

    def rec(prefix):
        if len(prefix) == Tn:
            if prefix[-1] >= S - 2:
                out.append(tuple(prefix))
            return
        s = prefix[-1]
        for d in (0, 1, 2):
            q = s + d
            if q < S and (d < 2 or skip[q]):
                rec(prefix + [q])

    for s0 in range(min(2, S)):
        rec([s0])
    return out


def brute_force(e, skip):
    """Exhaustive: (best score, the optimal path whose reversed state sequence is lexicographically largest, number of paths)."""
    Tn, S = e.shape
    paths = all_paths(Tn, S, skip)
    if not paths:
        return NEG, None, 0
    scores = [sum(e[t, p[t]] for t in range(Tn)) for p in paths]   # the same order of additions as the recursion
    best = max(scores)
    cands = [p for p, sc in zip(paths, scores) if sc == best]
    return best, np.array(max(cands, key=lambda p: p[::-1])), len(paths)


def count_paths(Tn, skip):
    """Number of valid alignments (log, fp64) by the counting form of the recursion."""
    S = len(skip)
    c = np.zeros(S)
    c[:min(2, S)] = 1.0
    for _ in range(1, Tn):
        n = c.copy()
        n[1:] += c[:-1]
        n[2:] += np.where(skip[2:], c[:-2], 0.0)
        c = n
    tot = c[S - 1] + (c[S - 2] if S >= 2 else 0.0)
    return math.log(tot) if tot > 0 else NEG


def spans_of(path):
    """State path [Tn] -> (start, end) per label, from the odd states."""
    L = (int(path.max()) + 1) // 2 if len(path) else 0
    start, end = np.full(L, -1, np.int64), np.full(L, -1, np.int64)
    for t, s in enumerate(path):
        if s & 1:
            k = s >> 1
            if start[k] < 0:
                start[k] = t
            end[k] = t + 1
    return start, end


def path_of_spans(start, end, Tn):
    """The state path the spans describe: label k's state 2k+1 inside its span, the blank state between labels elsewhere."""
    path = np.zeros(Tn, np.int64)
    k = 0
    for t in range(Tn):
        while k < len(start) and t >= end[k]:
            k += 1
        path[t] = 2 * k + 1 if k < len(start) and start[k] <= t < end[k] else 2 * k
    return path


def emission_err(lse, lp):
    """Bound on |f32 e - fp64 e| per element (log units), lse broadcast against lp."""
    return U * (np.abs(lse) + np.abs(lp) + 32.0)


def path_eps(ev, err):
    """eps(P) of a path from its fp64 emissions ev [Tn] and their bounds err [Tn]."""
    V = np.cumsum(ev)
    return float(err.sum() + 1.01 * U * np.abs(V[1:]).sum())


def peak_rel_err(err):
    return err + 6 * U


def align_fp64(x, labels, label_len, input_len, blank=0, max_label_len=None):
    """x [T, N, 64] logits (the kernel's own f32 values), labels flat or dense (see to_rows).  Per utterance, dict of lists:
    valid, feasible, Tn, L, score (path_logprob in fp64: NaN invalid, -inf infeasible), path, start / end [L] (-1 when no path),
    peak [L] (max fp64 y over the span), margin, eps (eps of the optimum path), plus lp / lse [T, N(, 64)] and err."""
    lp, lse = log_softmax(x)
    err = emission_err(lse[..., None], lp)
    T, N, _ = lp.shape
    rows = to_rows(labels, label_len)
    ll = np.asarray(label_len, np.int64)
    mll = int(ll.max(initial=0)) if max_label_len is None else int(max_label_len)
    R = dict(lp=lp, lse=lse, err=err, valid=[], feasible=[], Tn=[], L=[], score=[], path=[], start=[], end=[], peak=[], margin=[],
             eps=[], ext=[])
    for n in range(N):
        Tn = int(min(max(int(input_len[n]), 0), T))
        seq = rows[n]
        L = int(ll[n])
        valid = seq is not None and 0 <= L <= mll and all(0 <= v < C and v != blank for v in seq)
        R["Tn"].append(Tn); R["L"].append(L); R["valid"].append(valid)
        none = (np.full(max(L, 0), -1, np.int64), np.full(max(L, 0), -1, np.int64), np.zeros(max(L, 0)))
        if not valid:
            R["feasible"].append(False); R["score"].append(float("nan")); R["path"].append(None); R["margin"].append(0.0)
            R["eps"].append(0.0); R["ext"].append(None)
            for k, v in zip(("start", "end", "peak"), none):
                R[k].append(v)
            continue
        ext, skip = ext_of(seq, blank)
        R["ext"].append(ext)
        rep = sum(seq[i] == seq[i - 1] for i in range(1, L))
        feas = L + rep <= Tn
        R["feasible"].append(feas)
        if not feas or Tn == 0:
            R["score"].append(NEG if not feas else 0.0); R["path"].append(None); R["margin"].append(np.inf); R["eps"].append(0.0)
            for k, v in zip(("start", "end", "peak"), none):
                R[k].append(v)
            continue
        e = lp[:Tn, n][:, ext]
        v = viterbi_ext(e, skip)
        st, en = spans_of(v["path"])
        st = np.r_[st, np.full(L - len(st), -1)].astype(np.int64)
        en = np.r_[en, np.full(L - len(en), -1)].astype(np.int64)
        y = np.exp(lp[:Tn, n])
        pk = np.array([y[st[k]:en[k], seq[k]].max() for k in range(L)]) if L else np.zeros(0)
        ev = e[np.arange(Tn), v["path"]]
        R["score"].append(v["score"]); R["path"].append(v["path"]); R["margin"].append(v["margin"])
        R["eps"].append(path_eps(ev, err[:Tn, n][np.arange(Tn), ext[v["path"]]]))
        R["start"].append(st); R["end"].append(en); R["peak"].append(pk)
    return R


def argmax_runs(x, Tn, blank=0):
    """Greedy read of x [T, 64] under blank `blank` (argmax, lowest index on ties, repeats merged, blank dropped) and the argmax
    runs as spans: (read, start, end)."""
    am = np.argmax(np.asarray(x)[:Tn], axis=1)
    read, start, end = [], [], []
    for t in range(Tn):
        c = int(am[t])
        if c == blank:
            continue
        if t > 0 and am[t - 1] == c:
            end[-1] = t + 1
            continue
        read.append(c); start.append(t); end.append(t + 1)
    return read, np.array(start, np.int64), np.array(end, np.int64)


def small_cases(seed, n_cases):
    """Random small problems for brute force: (e [Tn, S], skip, seq) with C = 4 classes, Tn <= 8, L <= 3, emissions on a grid
    of 1/8 (exact sums, so ties are exact and frequent)."""
    rng = np.random.default_rng(seed)
    for _ in range(n_cases):
        Tn = int(rng.integers(1, 9))
        L = int(rng.integers(0, 4))
        blank = int(rng.integers(0, 4))
        seq = [int(v) for v in rng.choice([c for c in range(4) if c != blank], size=L)]
        lp = -rng.integers(0, 6, size=(Tn, 4)) / 8.0
        ext, skip = ext_of(seq, blank)
        yield lp[:, ext], skip, seq, lp, blank
