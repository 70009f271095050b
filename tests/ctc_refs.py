"""fp64 CTC reference for the kernels of csrc/ctc.cu, and the per-element checks built on it.

ctc_fp64 takes the kernel's own f32 logits and any blank, and computes in torch on the logits' device, batched over
utterances in chunks (the alpha / beta tables of a chunk stay near `budget` bytes) and looped over T, in log2 space as the
kernels are: the log2-softmax, alpha and beta, log2 p, y_tc and the posterior P_tc of each class (a label class summed over
its odd states, the blank over the even ones), the costs and the gradient grad_scale * (y - P) with the header's
semantics (include/crnn_ctc.h): an invalid utterance gives cost NaN and a zero gradient, an infeasible one cost 0 and a
zero gradient, frames past the length a zero gradient.

Each gradient element is checked against a bound that follows the kernels' arithmetic:
  - a class with no state in the utterance (P = 0): |g - grad_scale*y| <= grad_scale * y * eps, where eps (softmax_eps)
    holds the f32 roundings of x*log2e - lse, the normaliser's sum, the approximate ex2 / lg2 and the divide or multiply by
    the normaliser.  It is analytic and does not depend on T.
  - the label classes and the blank: grad_scale * ((y + P) * eps + c * P * R_n), R_n = 2^-24 * |log2 p_n| * sqrt(T_n).
    The recursions make errors relative to P: a log2-domain error d in alpha + beta - log2 p moves P by about P*ln2*d,
    and d adds up over the frames.  c is measured per kernel.
alpha_steps_isolated restates each row of ctc_long_kernel's stored alpha table from the GPU's own previous row and lp row.

Test infrastructure only (imported by tests/)."""
import math

import numpy as np
import torch
import torch.nn.functional as F

C = 64
U = 2.0 ** -24                     # half an f32 ulp, relative
LN2 = math.log(2.0)
LOG2E = 1.0 / LN2
# One allowance for an ex2.approx result (relative) and a lg2.approx result (absolute, log2 units).  It is an upper bound
# taken for the instructions, not a measurement of them.
APPROX = 2.0 ** -21
NEG = float("-inf")
# Largest c ctc_grad_posterior needed per kernel variant over every case that runs it (the frame limits at T = 130 ... 550,
# C3 at T = 63 for fast and long, long up to T = 2048, blanks 0 / 17 / 63), H100 80GB HBM3 (SXM, 700 W); the tests enforce
# 4.5x.  Per T it stays within a factor 1.7 (fast: 0.996 at T = 63, 0.59 at 550; long: 1.03 ... 1.11 from 131 to 2048), so
# sqrt(T_n) in R_n is the right scale.
MEASURED_POSTERIOR = {"fast": 0.996, "fast-me": 0.455, "tma": 0.841, "tma-me": 0.228, "generic1": 0.839, "generic2": 0.774,
                      "generic4": 0.870, "long": 1.11}


def draw_labels(rng, size, blank):
    """Label ids uniform over [0, 64) minus the blank (at blank 0 the same draws as rng.integers(1, 64))."""
    v = rng.integers(0, C - 1, size=size)
    return v + (v >= blank)


def layout(lab, ll, il, T, blank, max_label_len=None):
    """Per utterance (numpy): extended labels [N, 2*max(L)+1] (blank past S), S, the clamped length Tn, valid (label_len
    within max_label_len, every id in [0, 64) and not the blank) and feasible (valid, Tn > 0, L + repeats <= Tn)."""
    lab, ll = np.asarray(lab, np.int64), np.asarray(ll, np.int64)
    N = ll.size
    mll = int(ll.max(initial=0)) if max_label_len is None else int(max_label_len)
    off = np.r_[0, np.cumsum(np.maximum(ll, 0))]
    Tn = np.clip(np.asarray(il, np.int64), 0, T)
    ext = np.full((N, 2 * max(int(ll.max(initial=0)), 0) + 1), blank, np.int64)
    valid, feas = np.zeros(N, bool), np.zeros(N, bool)
    for n in range(N):
        L = int(ll[n])
        seq = lab[off[n]:off[n] + max(L, 0)]
        valid[n] = 0 <= L <= mll and not ((seq < 0) | (seq >= C) | (seq == blank)).any()
        if valid[n]:
            ext[n, 1:2 * L:2] = seq
            feas[n] = Tn[n] > 0 and L + int((seq[1:] == seq[:-1]).sum()) <= Tn[n]
    return dict(ext=ext, S=2 * np.maximum(ll, 0) + 1, Tn=Tn, valid=valid, feasible=feas)


def transitions(ext, S, blank):
    """ext [B, Sm] long, S [B] -> (live: s < S, skin: the skip s-2 -> s is allowed, skout: s -> s+2 is allowed)."""
    s = torch.arange(ext.shape[1], device=ext.device)
    live = s[None] < S[:, None]
    skin = (s[None] >= 2) & live & (ext != blank) & (ext != torch.roll(ext, 2, 1))
    skout = F.pad(skin[:, 2:], (0, 2), value=False)
    return live, skin, skout


def lse3(a, b, c):
    """log2(2^a + 2^b + 2^c) as the kernels form it (max, then the sum of three ex2 and one lg2); -inf when all are."""
    m = torch.maximum(torch.maximum(a, b), c)
    mm = torch.where(m == NEG, torch.zeros_like(m), m)
    return mm + torch.log2(torch.exp2(a - mm) + torch.exp2(b - mm) + torch.exp2(c - mm))


def shift_up(p, k):
    """p[..., s - k] (-inf below 0)."""
    return F.pad(p[..., :p.shape[-1] - k], (k, 0), value=NEG)


def shift_down(p, k):
    """p[..., s + k] (-inf past the end)."""
    return F.pad(p[..., k:], (0, k), value=NEG)


def tables(lp2, ext, S, Tn, blank):
    """lp2 [T, B, 64] log2-softmax, ext [B, Sm], S and Tn [B] -> emissions e, alpha and beta [T, B, Sm] in the dtype of
    lp2 (log2 units; -inf past S, beta -inf from Tn on)."""
    T, B, _ = lp2.shape
    live, skin, skout = transitions(ext, S, blank)
    e = torch.gather(lp2, 2, ext[None].expand(T, B, ext.shape[1])).masked_fill(~live[None], NEG)
    alpha = torch.full_like(e, NEG)
    alpha[0, :, :2] = e[0, :, :2]
    for t in range(1, T):
        p = alpha[t - 1]
        alpha[t] = lse3(p, shift_up(p, 1), shift_up(p, 2).masked_fill(~skin, NEG)) + e[t]
    beta = torch.full_like(e, NEG)
    s = torch.arange(ext.shape[1], device=ext.device)
    init_mask = live & (s[None] >= S[:, None] - 2)
    for t in range(T - 1, -1, -1):
        row = torch.where(init_mask, e[t], torch.full_like(e[t], NEG))
        if t < T - 1:
            p = beta[t + 1]
            rec = lse3(p, shift_down(p, 1), shift_down(p, 2).masked_fill(~skout, NEG)) + e[t]
            row = torch.where((t < Tn - 1)[:, None], rec, row)
        beta[t] = torch.where((t < Tn)[:, None], row, torch.full_like(row, NEG))
    return e, alpha, beta


def ctc_fp64(x, lab, ll, il, blank=0, grad_scale=1.0, max_label_len=None, budget=1 << 32, keep_tables=False):
    """x [T, N, 64] f32 torch tensor: the kernel's own logits.  Returns a dict of fp64 tensors on x's device:
    x2 = x*log2e, lse2 (log2 normaliser [T, N]), lp2 = x2 - lse2, y, P [T, N, 64], log2p [N] (NaN where not feasible),
    costs [N], grad [T, N, 64], and valid / feasible / Tn [N], inlab [N, 64] (the classes with a state: the labels and the
    blank), Rn [N]; with keep_tables, e / alpha / beta [T, N, Sm] (one chunk)."""
    T, N, _ = x.shape
    dev = x.device
    lay = layout(lab, ll, il, T, blank, max_label_len)
    xd = x.double()
    x2 = xd * LOG2E
    lse2 = torch.logsumexp(xd, 2) * LOG2E
    lp2 = x2 - lse2[..., None]
    y = torch.exp2(lp2)
    P = torch.zeros_like(y)
    log2p = torch.full((N,), float("nan"), dtype=torch.float64, device=dev)
    ext = torch.tensor(lay["ext"], device=dev)
    S = torch.tensor(lay["S"], device=dev)
    Tn = torch.tensor(lay["Tn"], device=dev)
    idx = np.flatnonzero(lay["feasible"])
    out = {}
    per = 5 * T * ext.shape[1] * 8
    B = len(idx) if keep_tables else max(1, budget // per)
    for i0 in range(0, len(idx), max(B, 1)):
        ii = torch.tensor(idx[i0:i0 + B], device=dev)
        Sm = int(S[ii].max())
        exc, Sc, Tc = ext[ii, :Sm], S[ii], Tn[ii]
        e, alpha, beta = tables(lp2[:, ii], exc, Sc, Tc, blank)
        last = alpha[Tc - 1, torch.arange(len(ii), device=dev)]
        a1 = last.gather(1, (Sc - 1)[:, None])[:, 0]
        a2 = torch.where(Sc >= 2, last.gather(1, (Sc - 2).clamp_min(0)[:, None])[:, 0], torch.full_like(a1, NEG))
        lp = torch.logaddexp2(a1, a2)
        log2p[ii] = lp
        w = torch.exp2(alpha + beta - e.masked_fill(e == NEG, 0.0) - lp[None, :, None])
        Pc = torch.zeros((T, len(ii), C), dtype=torch.float64, device=dev)
        Pc.scatter_add_(2, exc[None].expand(T, len(ii), Sm), w)
        P[:, ii] = Pc
        if keep_tables:
            out.update(e=e, alpha=alpha, beta=beta)
        del e, alpha, beta, w
    valid = torch.tensor(lay["valid"], device=dev)
    feas = torch.tensor(lay["feasible"], device=dev)
    costs = torch.where(feas, -log2p * LN2, torch.where(valid, 0.0, float("nan")).double())
    live = (torch.arange(T, device=dev)[:, None] < Tn[None]) & feas[None]
    grad = torch.where(live[..., None], grad_scale * (y - P), torch.zeros_like(y))
    inlab = torch.zeros((N, C), dtype=torch.bool, device=dev)
    inlab.scatter_(1, ext, True)                                   # the padding carries the blank
    Rn = U * log2p.abs() * Tn.double().sqrt()
    out.update(x2=x2, lse2=lse2, lp2=lp2, y=y, P=P, log2p=log2p, costs=costs, grad=grad, valid=valid, feasible=feas,
               Tn=Tn, inlab=inlab, Rn=Rn, ext=ext, S=S)
    return out


def lp_allow(x2, lse2, lp2):
    """Bound on a stored f32 log2-softmax element against fp64 (log2 units): the roundings of x*log2e (and of log2e
    itself), of the maximum and m + lg2(sum), and of x*log2e - lse; lg2.approx; the sum's ex2.approx and adds."""
    return U * (2 * x2.abs() + 2 * lse2.abs() + lp2.abs() + 12) + APPROX + (APPROX + 8 * U) / LN2


def softmax_eps(R):
    """Relative bound on the kernels' y = 2^(x*log2e - lse) [T, N, 64]: ln2 times the exponent's bound, the final ex2,
    and up to 24 f32 roundings of the normaliser's sum, the divide (__fdividef, 2 ulp) or multiply by it and the store."""
    return LN2 * lp_allow(R["x2"], R["lse2"][..., None], R["lp2"]) + APPROX + 32 * U


def check_grad(ck, kind, costs, grad, R, grad_scale, T=None):
    """The kernel's costs [N] and gradient [T, N, 64] against ctc_fp64's R: costs relative to |cost|; the two per-element
    gradient stages (ctc_grad_posterior's row per T, bound key ctc_grad_posterior/<kind>); the gradient's relative L2
    (ctc_grad/<kind>); exactly zero past each length, cost 0 / zero gradient where infeasible, NaN / zero where invalid."""
    T = grad.shape[0] if T is None else T
    feas, valid, Tn = R["feasible"], R["valid"], R["Tn"]
    ck.close(f"ctc_cost/{kind}", costs[feas], R["costs"][feas], R["costs"][feas].abs(), key=f"ctc_cost/{kind}")
    live = (torch.arange(grad.shape[0], device=grad.device)[:, None] < Tn[None]) & feas[None]
    eps = softmax_eps(R)
    soft = live[..., None] & ~R["inlab"][None]
    post = live[..., None] & R["inlab"][None]
    ck.close(f"ctc_grad_softmax/{kind}", grad, R["grad"], grad_scale * R["y"] * eps, mask=soft)
    ck.close_allow(f"ctc_grad_posterior/{kind}/T{T}", grad, R["grad"], grad_scale * R["P"] * R["Rn"][None, :, None],
                   grad_scale * (R["y"] + R["P"]) * eps, post, key=f"ctc_grad_posterior/{kind}", axes=("t", "n", "c"))
    ck.l2(f"ctc_grad/{kind}", grad[:, feas], R["grad"][:, feas])
    past = torch.arange(grad.shape[0], device=grad.device)[:, None] >= Tn[None]
    ck.exact(f"ctc_grad_past_len_zero/{kind}", grad[past], 0.0)
    ck.exact(f"ctc_infeasible_cost_zero/{kind}", costs[valid & ~feas], 0.0)
    ck.exact(f"ctc_infeasible_grad_zero/{kind}", grad[:, valid & ~feas], 0.0)
    ck.exact(f"ctc_invalid_cost_nan/{kind}", torch.isnan(costs[~valid]), True)
    ck.exact(f"ctc_invalid_grad_zero/{kind}", grad[:, ~valid], 0.0)
    ck._record(f"ctc_feasible/{kind}", 0.0, utterances=int(feas.sum()), T=T)


# ------------------------------------------------------------------------------------------- ctc_long_kernel's workspace
def long_stride(max_label_len):
    return (2 * max_label_len + 1 + 3) & ~3


def long_workspace_views(ws, T, N, max_label_len):
    """The caller's workspace (uint8 cuda tensor) as ctc_long_kernel lays it out: the pointer rounded up to 256 bytes,
    lp [N][T][64] then alpha [N][T][AS], both f32 log2 units."""
    off = (-ws.data_ptr()) % 256
    AS = long_stride(max_label_len)
    n_lp, n_al = N * T * C, N * T * AS
    f = ws[off:off + 4 * (n_lp + n_al)].view(torch.float32)
    return f[:n_lp].view(N, T, C), f[n_lp:].view(N, T, AS)


def alpha_steps_isolated(lp_gpu, al_gpu, ext, S, blank):
    """Each alpha row t >= 1 of the GPU's table restated in fp64 from the GPU's own row t-1 and its own lp row t:
    lp_gpu [B, T, 64], al_gpu [B, T, AS] (f32), ext [B, AS] (blank past S), S [B].  Returns (ref [B, T-1, AS] for rows
    1 .. T-1, m = the predecessors' maximum), -inf past S."""
    a = al_gpu.double()
    live, skin, _ = transitions(ext, S, blank)
    p = a[:, :-1]
    p1, p2 = shift_up(p, 1), shift_up(p, 2).masked_fill(~skin[:, None], NEG)
    m = torch.maximum(torch.maximum(p, p1), p2)
    e = torch.gather(lp_gpu[:, 1:].double(), 2, ext[:, None].expand(-1, a.shape[1] - 1, -1))
    ref = (torch.logaddexp2(torch.logaddexp2(p, p1), p2) + e).masked_fill(~live[:, None], NEG)
    return ref, m


def alpha_step_allow(ref, m):
    """Bound on one stored alpha element (log2 units): one f32 ulp of |alpha|, half an ulp of the predecessors' maximum
    (m + lg2(sum) rounds), lg2.approx, and the three ex2.approx and two adds of the sum (relative, over ln2)."""
    return 2 * U * ref.abs() + U * (m.abs() + 2) + APPROX + (APPROX + 4 * U) / LN2


def check_long_workspace(ck, kind, ws, x, costs, R, blank, max_label_len, budget=1 << 30):
    """ctc_long_kernel's stored tables after a call on logits x with workspace ws (costs: the call's), against R = ctc_fp64 of the same call:
    ctc_long_lp per element, ctc_long_alpha0 exactly, ctc_long_alpha_step per element teacher-forced (exactly -inf where
    every predecessor is and past S), ctc_long_cost_from_alpha from the GPU's own last row.  Feasible utterances only,
    rows t < T_n (the kernel writes no others)."""
    T, N, _ = x.shape
    lp_all, al_all = long_workspace_views(ws, T, N, max_label_len)
    AS = al_all.shape[2]
    dev = x.device
    ext = torch.full((N, AS), blank, dtype=torch.long, device=dev)
    ext[:, :R["ext"].shape[1]] = R["ext"][:, :AS]
    idx = torch.nonzero(R["feasible"]).flatten()
    B = max(1, budget // (6 * T * AS * 8))
    for i0 in range(0, len(idx), B):
        ii = idx[i0:i0 + B]
        Tn, S = R["Tn"][ii], R["S"][ii]
        rows = torch.arange(T, device=dev)[None] < Tn[:, None]                       # [B, T]
        lp_g = lp_all[ii]
        ck.close(f"ctc_long_lp/{kind}", lp_g, R["lp2"][:, ii].transpose(0, 1),
                 lp_allow(R["x2"][:, ii], R["lse2"][:, ii, None], R["lp2"][:, ii]).transpose(0, 1),
                 mask=rows[..., None].expand(-1, -1, C))
        lp_g = torch.where(rows[..., None], lp_g, torch.zeros_like(lp_g))              # rows past T_n hold no data
        al_g = al_all[ii]
        s = torch.arange(AS, device=dev)
        a0 = torch.where((s[None] < 2) & (s[None] < S[:, None]), lp_g[:, 0].gather(1, ext[ii]),
                         torch.full((len(ii), AS), NEG, device=dev))
        ck.exact(f"ctc_long_alpha0/{kind}", al_g[:, 0], a0)
        al_g = torch.where(rows[..., None], al_g, torch.full_like(al_g, NEG))
        ref, m = alpha_steps_isolated(lp_g, al_g, ext[ii], S, blank)
        g1 = al_g[:, 1:].double()
        step = rows[:, 1:, None].expand_as(ref)
        fin = step & torch.isfinite(ref)
        ck.close(f"ctc_long_alpha_step/{kind}", g1, ref, alpha_step_allow(ref, m), mask=fin)
        ck.exact(f"ctc_long_alpha_step_neg_inf/{kind}", g1[step & ~torch.isfinite(ref)], NEG)
        last = al_g[torch.arange(len(ii), device=dev), Tn - 1].double()
        a1 = last.gather(1, (S - 1)[:, None])[:, 0]
        a2 = torch.where(S >= 2, last.gather(1, (S - 2).clamp_min(0)[:, None])[:, 0], torch.full_like(a1, NEG))
        c_ref = -LN2 * torch.logaddexp2(a1, a2)
        mx = torch.maximum(a1, a2).abs()
        allow = 4 * U * c_ref.abs() + LN2 * (U * (mx + 2) + APPROX) + APPROX + 3 * U
        ck.close(f"ctc_long_cost_from_alpha/{kind}", costs[ii], c_ref, allow)
        del ref, m, g1



def bounds(kinds, post):
    """Bound table entries of the analytic stages (c = 1: the bound is the allowance itself) and of ctc_grad_posterior
    (post: kind -> enforced c)."""
    out = {f"{st}/{k}": (0, 1.0) for k in kinds for st in ("ctc_grad_softmax", "ctc_long_lp", "ctc_long_alpha_step",
                                                               "ctc_long_cost_from_alpha")}
    out.update({f"ctc_grad_posterior/{k}": (0, c) for k, c in post.items()})
    return out
