"""References for lexicon-based reading (crnn_lexicon_candidates / crnn_ctc_lexicon_score).

levenshtein_dp      the plain row-by-row dynamic program, vectorised over (read, entry) pairs.
myers_distance      a restatement of the kernel's bit-parallel algorithm (the read as the pattern, 64-row words, the global
                    distance read on the pattern's last row), in Python integers.
candidates_ref      the header's candidate semantics on top of levenshtein_dp: (d, index) order, truncation, cand_total.
score_fp64          ln p(entry | line) in fp64 through ctc_refs' log2-space alpha recursion (the forward half of ctc_fp64), with
                    the analytic f32 bound of the kernel's arithmetic (score_allow).
select_ref          the best slot under the tie rule (highest finite score, lowest slot) and each line's top-two margin.

Test infrastructure only (imported by tests/)."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ctc_refs as R  # noqa: E402

C = 64
MASK = (1 << 64) - 1


# ------------------------------------------------------------------------------------------------------------- distances
def _match(a, b):
    """Ids equal and inside [0, 64): an id outside matches nothing, not even itself."""
    return (a == b) & (a >= 0) & (a < C)


def levenshtein_dp(reads, read_len, entries, entry_len):
    """Levenshtein distance of pairs: reads [P, A] and entries [P, B] int arrays (row p holds read_len[p] / entry_len[p] ids).
    The DP runs row by row over the read, every pair at once.  Returns [P] int64."""
    reads, entries = np.asarray(reads, np.int64), np.asarray(entries, np.int64)
    ra, rb = np.asarray(read_len, np.int64), np.asarray(entry_len, np.int64)
    P, B = entries.shape[0], entries.shape[1]
    prev = np.broadcast_to(np.arange(B + 1, dtype=np.int64), (P, B + 1)).copy()   # D[0][j] = j
    out = np.where(ra == 0, rb, 0)
    for i in range(1, reads.shape[1] + 1 if reads.ndim == 2 else 1):
        cur = np.empty_like(prev)
        cur[:, 0] = i
        sub = prev[:, :-1] + ~_match(reads[:, i - 1:i], entries)
        best = np.minimum(sub, prev[:, 1:] + 1)
        for j in range(1, B + 1):                                   # the insertion chain runs along the row
            cur[:, j] = np.minimum(best[:, j - 1], cur[:, j - 1] + 1)
        prev = cur
        done = ra == i
        out[done] = prev[done, rb[done]]
    return out


def levenshtein(a, b):
    """One pair (sequences of ints)."""
    A, B = max(len(a), 1), max(len(b), 1)
    ra = np.zeros((1, A), np.int64); ra[0, :len(a)] = a
    rb = np.zeros((1, B), np.int64); rb[0, :len(b)] = b
    return int(levenshtein_dp(ra, [len(a)], rb, [len(b)])[0])


def myers_distance(read, entry):
    """The kernel's lx_distance restated: Peq[c] per 64-row word of the read, per entry id one block step per word (hin = +1
    into word 0: the global distance), the score tracked at the read's last row."""
    m, n = len(read), len(entry)
    if m == 0:
        return n
    W = (m + 63) // 64
    peq = {}
    for i, c in enumerate(read):
        if 0 <= c < C:
            w = peq.setdefault(c, [0] * W)
            w[i // 64] |= 1 << (i % 64)
    pv, mv = [MASK] * W, [0] * W
    rl = (m - 1) & 63
    score = m
    for c in entry:
        eqs = peq.get(c, [0] * W) if 0 <= c < C else [0] * W
        hin = 1
        for b in range(W):
            eq = eqs[b]
            neg, pos = int(hin < 0), int(hin > 0)
            xv = eq | mv[b]
            eq |= neg
            xh = ((((eq & pv[b]) + pv[b]) & MASK) ^ pv[b]) | eq
            ph = (mv[b] | ~(xh | pv[b])) & MASK
            mh = pv[b] & xh
            if b == W - 1:
                score += ((ph >> rl) & 1) - ((mh >> rl) & 1)
            hin = (ph >> 63) - (mh >> 63)
            ph = ((ph << 1) | pos) & MASK
            mh = ((mh << 1) | neg) & MASK
            pv[b] = (mh | ~(xv | ph)) & MASK
            mv[b] = ph & xv
    return score


def pair_distances(reads, read_len, entries):
    """[N, K] distances of every read (rows of reads [N, M], read_len [N], clamped to [0, M]) to every entry (list of id
    sequences), by levenshtein_dp over all pairs."""
    reads = np.asarray(reads, np.int64)
    N, M = reads.shape
    rl = np.clip(np.asarray(read_len, np.int64), 0, M)
    K = len(entries)
    el = np.array([len(e) for e in entries], np.int64)
    E = np.zeros((K, max(int(el.max(initial=0)), 1)), np.int64)
    for k, e in enumerate(entries):
        E[k, :len(e)] = e
    out = np.empty((N, K), np.int64)
    rows = max(1, (1 << 22) // max(K, 1))
    for n0 in range(0, N, rows):
        nn = np.arange(n0, min(N, n0 + rows))
        ra = np.repeat(reads[nn] if M else np.zeros((len(nn), 1), np.int64), K, axis=0)
        out[nn] = levenshtein_dp(ra, np.repeat(rl[nn], K), np.tile(E, (len(nn), 1)), np.tile(el, len(nn))).reshape(len(nn), K)
    return out


def candidates_ref(dist, max_edit, max_candidates, valid=None):
    """From the [N, K] distances: cand, cand_dist [N, max_candidates] (ordered by (d, index), -1 past the count) and cand_total
    [N], with the header's semantics (max_edit < 0: no threshold).  valid [K]: entries that can be candidates at all."""
    N, K = dist.shape
    cand = np.full((N, max_candidates), -1, np.int32)
    cdist = np.full((N, max_candidates), -1, np.int32)
    total = np.zeros(N, np.int32)
    ok = np.ones(K, bool) if valid is None else np.asarray(valid, bool)
    for n in range(N):
        within = ok & ((dist[n] <= max_edit) if max_edit >= 0 else True)
        idx = np.flatnonzero(within)
        total[n] = len(idx)
        order = idx[np.lexsort((idx, dist[n, idx]))][:max_candidates]
        cand[n, :len(order)] = order
        cdist[n, :len(order)] = dist[n, order]
    return cand, cdist, total


# ------------------------------------------------------------------------------------------------------------- scores
def alpha_log2(lp2, ext, S, Tn, blank):
    """Forward half of ctc_refs.tables: lp2 [T, B, 64] log2-softmax (fp64), ext [B, Sm], S, Tn [B] -> log2 p [B] (-inf when no
    path)."""
    T, B, _ = lp2.shape
    live, skin, _ = R.transitions(ext, S, blank)
    e = torch.gather(lp2, 2, ext[None].expand(T, B, ext.shape[1])).masked_fill(~live[None], R.NEG)
    a = torch.full_like(e[0], R.NEG)
    a[:, :2] = e[0, :, :2]
    last = a.clone()
    for t in range(1, T):
        a = R.lse3(a, R.shift_up(a, 1), R.shift_up(a, 2).masked_fill(~skin, R.NEG)) + e[t]
        last = torch.where((Tn - 1 == t)[:, None], a, last)
    ar = torch.arange(B, device=lp2.device)
    a1 = last[ar, S - 1]
    a2 = torch.where(S >= 2, last[ar, (S - 2).clamp_min(0)], torch.full_like(a1, R.NEG))
    return torch.logaddexp2(a1, a2)


def score_fp64(x, input_len, entries, cand, blank=0, chunk=1 << 15):
    """ln p(entries[cand[n, j]] | x[:, n]) [N, J] fp64 (numpy), the header's special values included (-inf for empty slots and
    infeasible entries, NaN for invalid ones; L = 0 with T_n = 0 gives 0), and the analytic bound of the kernel's f32 result
    (score_allow).  x [T, N, 64] f32 torch tensor (the kernel's own logits); entries: id sequences; cand [N, J]."""
    T, N, _ = x.shape
    cand = np.asarray(cand, np.int64)
    J = cand.shape[1]
    dev = x.device
    xd = x.double()
    x2 = xd * R.LOG2E
    lse2 = torch.logsumexp(xd, 2) * R.LOG2E
    lp2 = x2 - lse2[..., None]
    Tn_all = np.clip(np.asarray(input_len, np.int64), 0, T)
    # per frame, the largest element bound of the stored log2-softmax row (ctc_refs.lp_allow)
    row_allow = R.lp_allow(x2, lse2[..., None], lp2).amax(2)                       # [T, N]
    cum_allow = torch.cat([torch.zeros(1, N, dtype=torch.float64, device=dev), torch.cumsum(row_allow, 0)]).cpu().numpy()
    out = np.full((N, J), -np.inf)
    allow = np.zeros((N, J))
    pairs = []
    for n in range(N):
        for j in range(J):
            k = int(cand[n, j])
            if k < 0:
                continue
            e = list(entries[k])
            if any(not 0 <= v < C or v == blank for v in e) or len(e) > 63:
                out[n, j] = np.nan
                continue
            Tn = int(Tn_all[n])
            reps = sum(e[i] == e[i - 1] for i in range(1, len(e)))
            if len(e) + reps > Tn:
                continue
            if Tn == 0:
                out[n, j] = 0.0
                continue
            pairs.append((n, j, e))
    for p0 in range(0, len(pairs), chunk):
        part = pairs[p0:p0 + chunk]
        nn = torch.tensor([p[0] for p in part], device=dev)
        Lm = max(len(p[2]) for p in part)
        ext = torch.full((len(part), 2 * Lm + 1), blank, dtype=torch.long, device=dev)
        for i, p in enumerate(part):
            if p[2]:
                ext[i, 1:2 * len(p[2]):2] = torch.tensor(p[2], device=dev)
        S = torch.tensor([2 * len(p[2]) + 1 for p in part], device=dev)
        Tn = torch.tensor([int(Tn_all[p[0]]) for p in part], device=dev)
        Tm = int(Tn.max())
        l2 = alpha_log2(lp2[:Tm, nn], ext, S, Tn, blank).cpu().numpy()
        for i, p in enumerate(part):
            n, j = p[0], p[1]
            out[n, j] = l2[i] * R.LN2
            allow[n, j] = score_allow(l2[i], int(Tn_all[n]), cum_allow[int(Tn_all[n]), n])
    return out, allow


def score_allow(log2p, Tn, emission_allow):
    """Analytic bound on |f32 score - fp64 score| (natural log).  The log-sum-exp recursion is 1-Lipschitz in the max norm, so
    the final error is at most the sum over frames of each step's own error: the stored emission's (ctc_refs.lp_allow, the
    largest of its row; emission_allow sums them over t < T_n) and one lse3 rounding (ctc_refs.alpha_step_allow with the
    alpha magnitudes bounded by |log2 p| + 8: a state carrying any weight has alpha >= log2 p - log2(S)), plus 32 U for the
    subtractions inside the sum; then the final lse3 and the conversion to natural log."""
    a = abs(log2p) + 8.0
    step = 2 * R.U * a + R.U * (a + 2) + R.APPROX + (R.APPROX + 4 * R.U) / R.LN2 + 32 * R.U
    return R.LN2 * (emission_allow + Tn * step) + 4 * R.U * abs(log2p) * R.LN2 + R.LN2 * (R.APPROX + 2 * R.U)


def select_ref(score, cand):
    """(best index [N] (-1 when no finite score), best slot [N], margin [N] = best finite score - second best finite score
    (inf when fewer than two)) under the tie rule: the highest finite score, the lowest slot on ties."""
    N, J = score.shape
    best = np.full(N, -1, np.int64)
    slot = np.full(N, -1, np.int64)
    margin = np.full(N, np.inf)
    for n in range(N):
        fin = np.flatnonzero(np.isfinite(score[n]))
        if not len(fin):
            continue
        v = score[n, fin]
        i = fin[int(np.argmax(v))]                       # argmax: the first (lowest slot) maximum
        slot[n], best[n] = i, cand[n, i]
        if len(fin) > 1:
            margin[n] = v.max() - np.sort(v)[-2]
    return best, slot, margin


# ------------------------------------------------------------------------------------------------------------- small cases
def enumerate_score(lp, entry, Tn, blank=0):
    """ln p(entry | frames) by enumerating every frame labelling of length Tn whose CTC collapse is `entry` (lp [T, C] natural
    log-softmax, small Tn and C only)."""
    import itertools
    Cn = lp.shape[1]
    tot = -np.inf
    for path in itertools.product(range(Cn), repeat=Tn):
        out, prev = [], None
        for c in path:
            if c != prev and c != blank:
                out.append(c)
            prev = c
        if out == list(entry):
            tot = np.logaddexp(tot, sum(lp[t, c] for t, c in enumerate(path)))
    return tot if Tn else (0.0 if not entry else -np.inf)


def distances_torch(reads, read_len, E, el, block=1 << 24):
    """levenshtein_dp on the GPU: reads [N, M] and E [K, B] (entries zero-padded) int tensors, read_len [N] (clamped to [0, M])
    and el [K] -> [N, K] int32 distances.  The same row-by-row DP (ids outside [0, 64) match nothing), in blocks of reads."""
    N, M = reads.shape
    K, B = E.shape
    dev = E.device
    rl = read_len.long().clamp(0, M)
    el = el.long()
    out = torch.empty((N, K), dtype=torch.int32, device=dev)
    inE = (E >= 0) & (E < C)
    rows = max(1, block // max(K * (B + 1), 1))
    base = torch.arange(B + 1, device=dev, dtype=torch.int16)
    for n0 in range(0, N, rows):
        nn = slice(n0, min(N, n0 + rows))
        r, l = reads[nn].long(), rl[nn]
        prev = base.expand(r.shape[0], K, B + 1).clone()
        res = torch.where(l[:, None] == 0, el[None].int(), torch.zeros((), dtype=torch.int32, device=dev)).clone()
        for i in range(1, int(l.max()) + 1 if r.shape[0] else 1):
            c = r[:, i - 1][:, None, None]
            miss = ~((E[None] == c) & inE[None])
            best = torch.minimum(prev[..., :-1] + miss.short(), prev[..., 1:] + 1)
            cur = torch.empty_like(prev)
            cur[..., 0] = i
            for j in range(1, B + 1):
                cur[..., j] = torch.minimum(best[..., j - 1], cur[..., j - 1] + 1)
            prev = cur
            done = l == i
            if done.any():
                res[done] = prev[done].gather(2, el[None, :, None].expand(int(done.sum()), K, 1))[..., 0].int()
        out[nn] = res
    return out


def candidates_torch(D, max_edit, max_candidates, valid=None):
    """candidates_ref on the GPU from [N, K] distances: keys d * K + index are distinct, so topk of the smallest is the
    (d, index) order."""
    N, K = D.shape
    d = D.long()
    within = torch.ones_like(d, dtype=torch.bool) if max_edit < 0 else d <= max_edit
    if valid is not None:
        within &= valid[None]
    big = torch.iinfo(torch.int64).max
    key = torch.where(within, d * K + torch.arange(K, device=D.device)[None], torch.full_like(d, big))
    k = min(max_candidates, K)
    v, _ = torch.topk(key, k, dim=1, largest=False, sorted=True)
    ok = v != big
    cand = torch.full((N, max_candidates), -1, dtype=torch.int32, device=D.device)
    dist = torch.full((N, max_candidates), -1, dtype=torch.int32, device=D.device)
    cand[:, :k] = torch.where(ok, v % K, -1).int()
    dist[:, :k] = torch.where(ok, v // K, -1).int()
    return cand, dist, within.sum(1).int()
