"""fp64 exact prefix search: the reference the CTC beam-search decoders (csrc/beam.cpp, csrc/beam.cu) are checked against.

Prefix search that keeps every prefix is exact: after the last frame each prefix's total is log P(l | x), the CTC forward
probability of that labelling summed over all its alignments.  Two facts make it a reference for a width-bounded beam:
  - When at every frame the number of prefixes with non-zero probability is at most the width, TF's beam never evicts a
    finite entry (a listed entry whose total went to -inf is the bottom and goes first), so its top entry is the most
    probable labelling and its total that labelling's log-probability.
  - When the beam prunes, an entry's total sums a subset of its labelling's alignments, so neg_log_prob >= -log P(out).
Nothing here restates TF's beam: no width, no visit order, no eviction.

Test infrastructure only (imported by tests/)."""
import itertools
import math

import numpy as np

NEG = float("-inf")
MAX_PREFIXES = 100_000
MUTANTS = (None, "repeat_from_total", "blank_only_score", "best_path")


def _lae(a, b):
    if a == NEG:
        return b
    if b == NEG:
        return a
    m = a if a > b else b
    return m + math.log1p(math.exp(-abs(a - b)))


def log_softmax(row):
    """fp64 log-softmax of one f32 frame; a NaN logit counts as -inf, and a frame with no finite normaliser is all -inf."""
    r = np.asarray(row, np.float64)
    r = np.where(np.isnan(r), NEG, r)
    mx = r.max()
    if not np.isfinite(mx):
        return np.full(r.shape, NEG)
    with np.errstate(divide="ignore"):
        return r - (mx + math.log(np.exp(r - mx).sum()))


def exact_prefix_search(x_n, length, mutant=None):
    """x_n [T, C] f32 logits of one utterance (blank C-1), its first `length` frames.  Returns ({labelling tuple: log P},
    the largest number of prefixes with non-zero probability over the frames, the empty prefix before frame 0 included).

    The textbook recursion, nothing pruned: per prefix (log p_blank, log p_label); a blank keeps the prefix, its last label
    repeated keeps it from p_label, a new label c extends it from the total -- from p_blank only when c repeats the last label.
    Controls (`mutant`), each wrong in one way: "repeat_from_total" extends a repeated label from the total too;
    "blank_only_score" reports p_blank alone as the score; "best_path" returns the collapsed most probable frame path (the
    greedy decode) with that path's log-probability."""
    assert mutant in MUTANTS, mutant
    x_n = np.asarray(x_n)
    C = x_n.shape[1]
    blank = C - 1
    lps = [log_softmax(x_n[t]) for t in range(length)]
    if mutant == "best_path":
        path = [int(np.argmax(lp)) for lp in lps]
        score = float(sum(lp[c] for lp, c in zip(lps, path)))
        lab = tuple(c for i, c in enumerate(path) if c != blank and (i == 0 or c != path[i - 1]))
        return {lab: score}, 1
    beams = {(): (0.0, NEG)}
    peak = 1
    for lp in lps:
        labels = [c for c in range(blank) if lp[c] > NEG]
        nxt = {}

        def add(pfx, pb, pl):
            ob, ol = nxt.get(pfx, (NEG, NEG))
            nxt[pfx] = (_lae(ob, pb), _lae(ol, pl))
        for pfx, (pb, pl) in beams.items():
            tot = _lae(pb, pl)
            if lp[blank] > NEG:
                add(pfx, tot + lp[blank], NEG)
            last = pfx[-1] if pfx else -1
            if last >= 0 and lp[last] > NEG and pl > NEG:
                add(pfx, NEG, pl + lp[last])
            for c in labels:
                src = (tot if mutant == "repeat_from_total" else pb) if c == last else tot
                if src > NEG:
                    add(pfx + (c,), NEG, src + lp[c])
        beams = {k: v for k, v in nxt.items() if v[0] > NEG or v[1] > NEG}
        peak = max(peak, len(beams))
        if len(beams) > MAX_PREFIXES:
            raise ValueError(f"exact_prefix_search: {len(beams)} prefixes, more than {MAX_PREFIXES}")
    if mutant == "blank_only_score":
        return {k: pb for k, (pb, pl) in beams.items()}, peak
    return {k: _lae(pb, pl) for k, (pb, pl) in beams.items()}, peak


def top_two(P):
    """(argmax labelling, its log P, the runner-up's log P or -inf); ties go to the smaller labelling so the result does not
    depend on dict order."""
    items = sorted(P.items(), key=lambda kv: (-kv[1], kv[0]))
    return items[0][0], items[0][1], items[1][1] if len(items) > 1 else NEG


def decided(lp1, lp2):
    """The top labelling is decided when the runner-up is more than 1e-9 * (1 + |log P1|) below it."""
    return lp1 - lp2 > 1e-9 * (1.0 + abs(lp1))


def expected(best, merge_repeated, strip):
    """The decoders' output rule on the decoded prefix: consecutive equal labels collapsed when merge_repeated is set, then
    `strip` dropped."""
    out, prev = [], None
    for l in best:
        if not (merge_repeated and l == prev) and l != strip:
            out.append(int(l))
        prev = l
    return out


def path_enumeration(x_n, length):
    """{labelling: log P} by summing every C^T frame path (small T and C only)."""
    x_n = np.asarray(x_n)
    C = x_n.shape[1]
    lps = [log_softmax(x_n[t]) for t in range(length)]
    P = {}
    for path in itertools.product(range(C), repeat=length):
        s = sum(lps[t][c] for t, c in enumerate(path))
        if s == NEG:
            continue
        lab = tuple(c for i, c in enumerate(path) if c != C - 1 and (i == 0 or c != path[i - 1]))
        P[lab] = _lae(P.get(lab, NEG), s)
    return P


# Every (C, T) that width 128 covers exhaustively on dense frames: (C-1)^0 + ... + (C-1)^T prefixes at most (T + 1 at C = 2).
DENSE_GRID = [(2, 127), (3, 6), (4, 4), (5, 3)] + [(c, 2) for c in range(6, 12)] + [(64, 1)]


def dense_case(C, T, N, seed):
    """[T, N, C] f32 dense random frames at scales 0.3, 1 and 3 (one per utterance, in turn) and ragged lengths: the first
    utterance full length, the others uniform in [0, T]."""
    rng = np.random.default_rng(seed)
    scale = np.array([0.3, 1.0, 3.0])[np.arange(N) % 3]
    x = (rng.standard_normal((T, N, C)) * scale[None, :, None]).astype(np.float32)
    il = rng.integers(0, T + 1, size=N).astype(np.int32)
    il[0] = T
    return x, il


def sparse_case(T, seed, C=64):
    """One [T, 1, C] f32 utterance, mostly blank-only frames (every label logit -inf): three or four frames offering two
    labels and the blank, one or two frames with a -inf blank, and a run of one label repeated over three frames."""
    rng = np.random.default_rng(seed)
    blank = C - 1
    x = np.full((T, C), NEG, np.float32)
    x[:, blank] = rng.standard_normal(T).astype(np.float32)
    frames = rng.permutation(T)
    k = int(rng.integers(3, 5))
    for t in frames[:k]:
        a, b = rng.choice(blank, size=2, replace=False)
        x[t, [a, b]] = rng.standard_normal(2) * 0.5
    for t in frames[k:k + int(rng.integers(1, 3))]:
        x[t, int(rng.integers(0, blank))] = rng.standard_normal()
        x[t, blank] = NEG
    t0 = int(rng.integers(0, T - 3))
    lab = int(rng.integers(0, blank))
    x[t0:t0 + 3, lab] = rng.standard_normal(3) * 0.5
    return x[:, None, :]


def sparse_batch(T, width, count, seed0=0):
    """The first `count` sparse_case utterances from seed0 on whose measured prefix count fits `width`, stacked to
    [T, count, 64]; returns (x, input_len, the seeds used)."""
    xs, seeds = [], []
    s = seed0
    while len(xs) < count:
        x = sparse_case(T, s)
        if exact_prefix_search(x[:, 0], T)[1] <= width:
            xs.append(x)
            seeds.append(s)
        s += 1
    return np.concatenate(xs, axis=1), np.full(count, T, np.int32), seeds


def references(x, il, mutant=None):
    """exact_prefix_search of every utterance of a [T, N, C] batch: a list of ({labelling: log P}, peak)."""
    return [exact_prefix_search(x[:, n], int(il[n]), mutant) for n in range(x.shape[1])]


def f32_neg(lp):
    return np.float32(-lp)


def within_one_ulp(a, b):
    """Equal, or the same sign and one f32 ulp apart (the rule of test_gpu_beam._within_one_ulp)."""
    a, b = np.float32(a), np.float32(b)
    return bool(a == b or (np.sign(a) == np.sign(b) and abs(int(a.view(np.int32)) - int(b.view(np.int32))) <= 1))


def check_exhaustive(lines, nlp, refs, merge_repeated, strip, stats):
    """One decode (labellings and neg_log_prob per utterance) of utterances whose beam was exhaustive against the exact
    search.  A decided line must give expected(argmax) and neg_log_prob within one f32 ulp of -log P(argmax); an undecided
    line (top two within 1e-9 relative) only the neg_log_prob of one of the two.  Adds to `stats` and returns the failures."""
    bad = []
    for n, (P, _) in enumerate(refs):
        best, l1, l2 = top_two(P)
        stats["lines"] += 1
        if decided(l1, l2):
            stats["decided"] += 1
            if list(lines[n]) != expected(best, merge_repeated, strip):
                stats["label_fail"] += 1
                bad.append(("label", n, list(lines[n]), expected(best, merge_repeated, strip)))
            if not within_one_ulp(nlp[n], f32_neg(l1)):
                stats["nlp_fail"] += 1
                bad.append(("neg_log_prob", n, float(nlp[n]), float(f32_neg(l1))))
        else:
            stats["undecided"] += 1
            if not (within_one_ulp(nlp[n], f32_neg(l1)) or within_one_ulp(nlp[n], f32_neg(l2))):
                stats["nlp_fail"] += 1
                bad.append(("neg_log_prob", n, float(nlp[n]), float(f32_neg(l1))))
    return bad


def new_stats():
    return dict(lines=0, decided=0, undecided=0, label_fail=0, nlp_fail=0)


def labelling_logp(x, il, lines):
    """log P(l | x) of one labelling per utterance (label ids, blank C-1) by the CTC forward DP in fp64: torch.ctc_loss on
    the fp64 log-softmax of the f32 logits.  Utterances of length 0 give 0 for the empty labelling."""
    import torch
    x = torch.as_tensor(np.asarray(x, np.float32)).double()
    T, N, C = x.shape
    lp = torch.log_softmax(x, 2)
    ll = torch.tensor([len(l) for l in lines], dtype=torch.long)
    tg = torch.tensor([v for l in lines for v in l] or [0], dtype=torch.long)
    il = torch.as_tensor(np.asarray(il, np.int64))
    out = np.zeros(N)
    live = (il > 0).nonzero()[:, 0]
    if len(live):
        off = np.r_[0, np.cumsum(ll.numpy())]
        sub_t = torch.cat([tg[off[n]:off[n + 1]] for n in live.tolist()] + [torch.zeros(0, dtype=torch.long)])
        cost = torch.nn.functional.ctc_loss(lp[:, live], sub_t, il[live], ll[live], blank=C - 1, reduction="none",
                                            zero_infinity=False)
        out[live.numpy()] = -cost.numpy()
    out[(il == 0).numpy()] = np.where(ll[(il == 0)].numpy() == 0, 0.0, NEG)
    return out


def lower_bound_slack(nlp, logp):
    """neg_log_prob minus f32(-log P(out)), in f32 ulps of the latter (>= -1 where the beam total understates P(out));
    relative slack alongside."""
    ref = np.array([f32_neg(v) for v in logp], np.float32)
    nlp = np.asarray(nlp, np.float32)
    ulp = np.spacing(np.abs(ref)).astype(np.float64)
    ulp = np.where(ulp > 0, ulp, np.spacing(np.float32(1e-38)))
    d = nlp.astype(np.float64) - ref.astype(np.float64)
    return d / ulp, d / np.maximum(np.abs(ref.astype(np.float64)), 1e-30)


def exhaustive_cases(N=24):
    """(name, x, input_len, references) for the dense grid and the sparse frames at T = 63, 255 and 1023."""
    out = []
    for C, T in DENSE_GRID:
        x, il = dense_case(C, T, N, seed=1000 * C + T)
        out.append((f"dense_C{C}_T{T}", x, il, references(x, il)))
    for T in (63, 255, 1023):
        x, il, _ = sparse_batch(T, 128, 6)
        out.append((f"sparse_T{T}", x, il, references(x, il)))
    return out


def pruned_cases(N=12):
    """(name, x, input_len) dense frames far beyond any width: C 3 ... 64 at T = 19 and 63."""
    return [(f"dense_C{C}_T{T}", *dense_case(C, T, N, seed=7 * C + T)) for C in (3, 17, 33, 64) for T in (19, 63)]


MODES = ((True, 0), (True, -1), (False, 0), (False, -1))


def run_exhaustive(decode, cases, widths=(128, 33, "peak", "peak-1")):
    """Decode every case at every width and output mode.  Lines whose measured prefix count fits the width are checked
    against the exact search (check_exhaustive); with merge_repeated=False, strip=-1 every line is also checked against the
    lower bound.  `decode(x, il, width, merge_repeated, strip)` -> (labellings, neg_log_prob).  "peak" decodes each line at
    its own measured prefix count, "peak-1" one below it (one eviction).  Returns (stats, failures, slack in ulps)."""
    st = new_stats()
    st.update(pruned=0, bound_fail=0)
    bad, slack = [], []
    for name, x, il, refs in cases:
        peak = np.array([p for _, p in refs])
        groups = []
        for w in widths:
            if w == "peak":
                groups += [(int(p), np.flatnonzero(peak == p)) for p in np.unique(peak)]
            elif w == "peak-1":
                groups += [(int(p) - 1, np.flatnonzero(peak == p)) for p in np.unique(peak) if p > 1]
            else:
                groups.append((w, np.arange(len(il))))
        for width, idx in groups:
            xs, ils = np.ascontiguousarray(x[:, idx]), il[idx]
            for merge, strip in MODES:
                lines, nlp = decode(xs, ils, width, merge, strip)
                ex = [k for k in range(len(idx)) if peak[idx[k]] <= width]
                for b in check_exhaustive([lines[k] for k in ex], [nlp[k] for k in ex], [refs[idx[k]] for k in ex], merge, strip, st):
                    bad.append((name, width, merge, strip) + b)
                if not merge and strip == -1:
                    st["pruned"] += len(idx) - len(ex)
                    b, s = check_lower_bound(xs, ils, lines, nlp, st)
                    bad += [(name, width) + e for e in b]
                    slack.append(s)
    return st, bad, np.concatenate(slack) if slack else np.zeros(0)


def check_lower_bound(x, il, lines, nlp, stats):
    """neg_log_prob >= f32(-log P(out)) less one ulp on every line of a merge_repeated=False, strip=-1 decode (the output is
    the decoded prefix itself).  Returns (failures, slack in ulps)."""
    lp = labelling_logp(x, il, lines)
    ulps, rel = lower_bound_slack(nlp, lp)
    stats["bound_checked"] = stats.get("bound_checked", 0) + len(lines)
    bad = [("lower_bound", n, list(lines[n]), float(nlp[n]), float(-lp[n])) for n in np.flatnonzero(~(ulps >= -1.0))]
    stats["bound_fail"] += len(bad)
    stats["min_rel_slack"] = min(stats.get("min_rel_slack", np.inf), float(rel.min()) if len(rel) else np.inf)
    return bad, ulps


def reference_decoder(mutant):
    """A decoder made of the exact search (or one of its controls): the argmax labelling and -f32 of its score; width
    ignored."""
    def decode(x, il, width, merge_repeated, strip):
        lines, nlp = [], []
        for P, _ in references(x, il, mutant):
            best, l1, _ = top_two(P)
            lines.append(expected(best, merge_repeated, strip))
            nlp.append(f32_neg(l1))
        return lines, np.array(nlp, np.float32)
    return decode
