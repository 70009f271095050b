"""The fp64 CTC reference (tests/ctc_refs.py) and the per-element CTC checks built on it, no GPU needed.

Pins: ctc_fp64 equals fp64 torch.ctc_loss with autograd, path enumeration and oracle.ctc_loss_np to 1e-12 at blanks 0, 17
and 63, with id 0 inside the labels (a repeated pair of 0 where it is not the blank), and keeps the header's semantics.

An f32 emulation of the log2-space kernels (ctc_long_kernel's order: x*log2e - lse rows, alpha stored row by row, beta,
the posterior ex2(alpha + beta - e - log2 p), the class sums, grad_scale * (ex2(lp) - sum)) then passes the new stages at
T = 63 ... 2048 with one posterior constant c, and the workspace stages on its own stored lp and alpha tables.  Each
mutant of the emulation fails the stage that should see it:
  - beta allows the skip between two equal adjacent labels (the cost does not change): ctc_grad_posterior, while the flat
    per-element bounds the posterior stage replaced (4.5x the largest error measured on the H100 at T <= 550 and 2048)
    still pass it;
  - a class that occurs twice sums only its first state: ctc_grad_posterior;
  - one class outside the label takes the previous frame's normaliser: ctc_grad_softmax;
  - one alpha step reads the next frame's emission: ctc_long_alpha_step."""
import itertools
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ctc_refs as R  # noqa: E402
from stage_check import Checker  # noqa: E402

BLANKS = [0, 17, 63]
NEG = R.NEG
# A round figure above the largest c the emulation needs in ctc_grad_posterior over the soundness cases below (0.47 at
# T = 2048); enforced at 4.5x, as on the GPU.
EMU_C = 0.7
# The flat per-element gradient bounds (units of grad_scale) ctc_grad_softmax / ctc_grad_posterior replaced: 4.5x the
# largest error the H100 measured at T <= 550 (the fast kernel) and at T = 2048 (ctc_long_kernel).
FLAT = {550: 4.5 * 3.38e-3, 2048: 4.5 * 2.97e-2}


def _seqs(rng, Ls, blank):
    """Labels of the given lengths over [0, 64) minus the blank; from length 6 on a repeated pair, and where 0 is a
    label id, a repeated pair of 0."""
    out = []
    for L in Ls:
        seq = R.draw_labels(rng, L, blank)
        if L >= 6:
            seq[5] = seq[4]
            if blank != 0:
                seq[1] = seq[2] = 0
        out.append(seq)
    return out


def _batch(T, Ls, blank, seed, scale=2.0):
    rng = np.random.default_rng(seed)
    seqs = _seqs(rng, Ls, blank)
    lab = np.concatenate(seqs).astype(np.int64) if seqs else np.zeros(0, np.int64)
    ll = np.array(Ls, np.int64)
    il = np.array([T - 3 * i for i in range(len(Ls))], np.int64)
    x = torch.tensor(rng.standard_normal((T, len(Ls), 64)) * scale, dtype=torch.float32)
    return x, lab, ll, il


# --------------------------------------------------------------------------------------------------------------- pins
def _torch_ctc(x, lab, ll, il, blank):
    xd = x.double().requires_grad_(True)
    c = F.ctc_loss(torch.log_softmax(xd, 2), torch.tensor(lab), torch.tensor(il), torch.tensor(ll), blank=blank,
                   reduction="none")
    (g,) = torch.autograd.grad(c.sum(), xd)
    return c.detach(), g


@pytest.mark.parametrize("blank", BLANKS)
@pytest.mark.parametrize("T,Ls", [(63, [15, 6, 1, 0, 9]), (300, [64, 100, 20]), (700, [255, 40])])
def test_reference_equals_torch_ctc(T, Ls, blank):
    x, lab, ll, il = _batch(T, Ls, blank, seed=T + blank)
    if blank != 0:
        assert (lab == 0).any()
    out = R.ctc_fp64(x, lab, ll, il, blank=blank)
    c, g = _torch_ctc(x, lab, ll, il, blank)
    assert bool(out["feasible"].all())
    assert float((out["costs"] - c).abs().max()) <= 1e-12 * float(c.abs().max())
    # both sides round their fp64 log-space sums once per frame: 1e-12 per 63 frames
    assert float((out["grad"] - g).abs().max()) <= 1e-12 * max(1.0, T / 63)


@pytest.mark.parametrize("blank", BLANKS)
def test_reference_equals_the_oracle(blank):
    from oracle import crnn_oracle as O
    x, lab, ll, il = _batch(150, [30, 8, 0], blank, seed=blank)
    out = R.ctc_fp64(x, lab, ll, il, blank=blank)
    co, go = O.ctc_loss_np(x.double().numpy(), lab, ll, il, blank=blank)
    assert np.abs(out["costs"].numpy() - co).max() <= 1e-12 * np.abs(co).max()
    assert np.abs(out["grad"].numpy() - go).max() <= 1e-12 * 150 / 63


def _brute(x, seq, blank):
    """-ln p and d(-ln p)/dx of one utterance by enumerating every path over the label ids and the blank (paths through
    any other class give nothing)."""
    T = x.shape[0]
    lp = x - np.log(np.exp(x).sum(1, keepdims=True))
    p, occ = 0.0, np.zeros_like(x)
    for path in itertools.product(sorted(set(seq) | {blank}), repeat=T):
        out, prev = [], None
        for c in path:
            if c != prev and c != blank:
                out.append(c)
            prev = c
        if out == list(seq):
            q = math.exp(sum(lp[t, c] for t, c in enumerate(path)))
            p += q
            for t, c in enumerate(path):
                occ[t, c] += q
    return -math.log(p), np.exp(lp) - occ / p


@pytest.mark.parametrize("blank", BLANKS)
@pytest.mark.parametrize("seq,T", [([1], 1), ([0, 2], 3), ([0, 0], 3), ([2, 0, 2], 5), ([5, 5, 5], 6), ([1, 2, 3], 4)])
def test_reference_equals_path_enumeration(seq, T, blank):
    seq = [blank + 1 if v == blank else v for v in seq]
    if blank == 63:
        seq = [v % 63 for v in seq]
    x = torch.tensor(np.random.default_rng(len(seq) * 10 + T).standard_normal((T, 1, 64)) * 1.5, dtype=torch.float32)
    out = R.ctc_fp64(x, np.array(seq), [len(seq)], [T], blank=blank)
    cb, gb = _brute(x[:, 0].double().numpy(), seq, blank)
    assert abs(float(out["costs"][0]) - cb) <= 1e-12 * max(1.0, abs(cb))
    assert np.abs(out["grad"][:, 0].numpy() - gb).max() <= 1e-12


@pytest.mark.parametrize("blank", BLANKS)
def test_reference_semantics(blank):
    """A label equal to the blank and label_len > max_label_len: NaN, zero gradient; no frames and a label that does not
    fit: 0, zero gradient; frames past the length: zero; the posteriors of each frame sum to 1."""
    rng = np.random.default_rng(blank)
    T = 20
    x = torch.tensor(rng.standard_normal((T, 6, 64)), dtype=torch.float32)
    other = (blank + 5) % 64
    seqs = [[other] * 10, [other] * 11, [other, blank], [other], [other] * 3, [blank + 1 if blank < 63 else 0]]
    ll, il = [10, 11, 2, 1, 3, 1], [T, T, T, 0, T + 5, 7]
    out = R.ctc_fp64(x, np.concatenate(seqs), ll, il, blank=blank, max_label_len=10)
    c, g = out["costs"], out["grad"]
    assert float(c[0]) > 0 and bool(torch.isfinite(c[0]))                    # 10 repeats need 19 frames: fits in 20
    assert bool(torch.isnan(c[1])) and not g[:, 1].any()                      # label_len > max_label_len
    assert bool(torch.isnan(c[2])) and not g[:, 2].any()                      # the blank as a label id
    assert float(c[3]) == 0 and not g[:, 3].any()                             # no frames
    assert bool(torch.isfinite(c[4]))                                         # input_len clamped to T
    assert not g[7:, 5].any() and g[:7, 5].abs().max() > 0
    f = out["feasible"]
    assert float((out["P"][:, f].sum(2)[:7] - 1).abs().max()) < 1e-12


# ------------------------------------------------------------------------------------------------------- f32 emulation
MUTANTS = ("beta_skip_equal", "first_state_only", "wrong_normaliser", "alpha_wrong_emission")


def emulate(x, lab, ll, il, blank, scale, mll, mutant=None):
    """ctc_long_kernel's arithmetic in f32 (torch's exp2 / log2 in place of ex2 / lg2.approx).  Returns costs [N],
    gradient [T, N, 64] and a workspace (uint8) holding the stored lp and alpha tables in the kernel's layout."""
    T, N, _ = x.shape
    lay = R.layout(lab, ll, il, T, blank, mll)
    ext = torch.tensor(lay["ext"])
    S, Tn = torch.tensor(lay["S"]), torch.tensor(lay["Tn"])
    feas = torch.tensor(lay["feasible"])
    x0 = x * torch.tensor(R.LOG2E, dtype=torch.float32)
    m = x0.max(2).values
    lse = m + torch.log2(torch.exp2(x0 - m[..., None]).sum(2))
    lp = x0 - lse[..., None]
    ly = lp.clone()
    inlab = torch.zeros((N, 64), dtype=torch.bool).scatter_(1, ext, True)
    if mutant == "wrong_normaliser":              # the first class outside utterance 0's label, frames t >= 1
        c = int(torch.nonzero(~inlab[0])[0])
        ly[1:, 0, c] = x0[1:, 0, c] - lse[:-1, 0]
    live, skin, skout = R.transitions(ext, S, blank)
    if mutant == "beta_skip_equal":
        s = torch.arange(ext.shape[1])
        skout = F.pad(((s[None] >= 2) & live & (ext != blank))[:, 2:], (0, 2), value=False)
    e = torch.gather(lp, 2, ext[None].expand(T, N, ext.shape[1])).masked_fill(~live[None], NEG)
    alpha = torch.full_like(e, NEG)
    alpha[0, :, :2] = e[0, :, :2]
    for t in range(1, T):
        p = alpha[t - 1]
        et = e[t + 1] if mutant == "alpha_wrong_emission" and t == T // 2 else e[t]
        alpha[t] = R.lse3(p, R.shift_up(p, 1), R.shift_up(p, 2).masked_fill(~skin, NEG)) + et
    ar = torch.arange(N)
    last = alpha[(Tn - 1).clamp_min(0), ar]
    a1 = last.gather(1, (S - 1)[:, None])[:, 0]
    a2 = torch.where(S >= 2, last.gather(1, (S - 2).clamp_min(0)[:, None])[:, 0], torch.full_like(a1, NEG))
    ll2 = R.lse3(a1, a2, torch.full_like(a1, NEG))
    costs = torch.where(feas, -ll2 * torch.tensor(R.LN2, dtype=torch.float32),
                        torch.where(torch.tensor(lay["valid"]), 0.0, float("nan")))
    beta = torch.full_like(e, NEG)
    s = torch.arange(ext.shape[1])
    init = live & (s[None] >= S[:, None] - 2)
    for t in range(T - 1, -1, -1):
        row = torch.where(init, e[t], torch.full_like(e[t], NEG))
        if t < T - 1:
            p = beta[t + 1]
            rec = R.lse3(p, R.shift_down(p, 1), R.shift_down(p, 2).masked_fill(~skout, NEG)) + e[t]
            row = torch.where((t < Tn - 1)[:, None], rec, row)
        beta[t] = torch.where((t < Tn)[:, None], row, torch.full_like(row, NEG))
    w = torch.exp2(alpha + beta - e.masked_fill(e == NEG, 0.0) - ll2[None, :, None])
    w = torch.where(torch.isnan(w), torch.zeros_like(w), w)
    if mutant == "first_state_only":              # a class that occurs twice: only its first state is summed
        first = torch.ones_like(ext, dtype=torch.bool)
        for n in range(N):
            seen = set()
            for k in range(1, int(S[n]), 2):
                first[n, k] = int(ext[n, k]) not in seen
                seen.add(int(ext[n, k]))
        w = w * first[None]
    P = torch.zeros((T, N, 64), dtype=torch.float32).scatter_add_(2, ext[None].expand(T, N, ext.shape[1]), w)
    livet = (torch.arange(T)[:, None] < Tn[None]) & feas[None]
    grad = torch.where(livet[..., None], scale * (torch.exp2(ly) - P), torch.zeros_like(P))
    # the workspace: lp [N][T][64] and alpha [N][T][AS] from a 256-byte boundary, rows t < T_n of feasible utterances
    AS = R.long_stride(mll)
    ws = torch.zeros(4 * N * T * (64 + AS) + 256, dtype=torch.uint8)
    lp_w, al_w = R.long_workspace_views(ws, T, N, mll)
    lp_w.copy_(lp.transpose(0, 1))
    al_w.fill_(NEG)
    al_w[:, :, :alpha.shape[2]] = alpha.transpose(0, 1)
    return costs, grad, ws


def _check(kind, x, lab, ll, il, blank, scale, mll, mutant=None):
    costs, grad, ws = emulate(x, lab, ll, il, blank, scale, mll, mutant)
    ref = R.ctc_fp64(x, lab, ll, il, blank=blank, grad_scale=scale, max_label_len=mll)
    ck = Checker(kind, dict(R.bounds([kind], {kind: 4.5 * EMU_C}), **{f"ctc_cost/{kind}": (0, 1e-5)}),
                 l2_limit={f"ctc_grad/{kind}": 1.0})
    R.check_grad(ck, kind, costs, grad, ref, scale)
    R.check_long_workspace(ck, kind, ws, x, costs, ref, blank, mll)
    flat = float((grad - ref["grad"]).abs().max()) / scale
    return ck, {r["stage"].split("/")[0]: r for r in ck.rows}, flat


SOUND = [(63, [15, 15, 1, 0, 7]), (130, [63, 40]), (550, [15, 4, 9]), (1024, [100, 64]), (2048, [255, 15])]


@pytest.mark.parametrize("blank", BLANKS)
@pytest.mark.parametrize("T,Ls", SOUND)
def test_emulation_passes_the_new_stages(T, Ls, blank):
    x, lab, ll, il = _batch(T, Ls, blank, seed=T * 7 + blank)
    ck, rows, _ = _check("emu", x, lab, ll, il, blank, 1.0 / len(Ls), max(Ls))
    assert not ck.fail, "\n".join(ck.fail)
    post = rows["ctc_grad_posterior"]
    print(f"T={T} blank={blank}: posterior c needed {post['c_needed']:.3g}, softmax {rows['ctc_grad_softmax']['c_needed']:.3g}")


@pytest.mark.parametrize("mutant,stage", [("beta_skip_equal", "ctc_grad_posterior"), ("first_state_only", "ctc_grad_posterior"),
                                          ("wrong_normaliser", "ctc_grad_softmax"),
                                          ("alpha_wrong_emission", "ctc_long_alpha_step")])
@pytest.mark.parametrize("T", [550, 2048])
def test_each_mutant_fails_its_stage(mutant, stage, T):
    Ls, seed = ([15, 9, 6], T) if T == 550 else ([63, 15], T)
    if mutant == "beta_skip_equal":
        # how far the wrong paths move P depends on the draw: at these two the mutant stays inside the flat bound
        Ls, seed = ([15, 9, 6], 5) if T == 550 else ([127], 5)
    x, lab, ll, il = _batch(T, Ls, 17, seed=seed)
    ck, rows, flat = _check("emu", x, lab, ll, il, 17, 1.0 / len(Ls), max(Ls), mutant)
    failed = {f.split(":")[0].split("/")[0] for f in ck.fail}
    assert stage in failed, (mutant, ck.fail)
    if mutant == "beta_skip_equal":
        # the cost reads alpha only; the flat per-element bound these stages replaced does not see the mutant
        assert rows["ctc_cost"]["max_ratio"] <= 1.0
        assert flat <= FLAT[T], (flat, FLAT[T])
        print(f"T={T}: beta skip mutant at {flat / FLAT[T]:.3g} of the flat bound, "
              f"{rows['ctc_grad_posterior']['max_ratio']:.3g}x the posterior bound")
