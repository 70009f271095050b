"""The per-step BPTT checks (stage_refs.bptt_steps_isolated, test_gpu_stage_isolation.bptt_step_checks) on an f32
emulation of lstm_bwd_ks_kernel, no GPU needed.

The emulation restates the kernel's arithmetic (csrc/lstm_bwd.cuh): each rank's 128-deep partial product accumulated in f32
over its 8 k-steps of 16 and rounded to bf16 (round to nearest even), the 8 partials summed in f32 in rank order onto
d_out, the cell formulas in f32 in the kernel's operation order with dc carried in f32 from step to step, tanh off by the
PTX ISA's maximum relative error in a chosen direction, every dz stored as bf16.  Its operands are the GPU tests' own
parameter draw and batch, pushed through the oracle's fp64 forward (gates rounded to bf16 and the cell state to f32, as
the forward kernel saves them) and the logits backward of a seeded random d logits.

Soundness: the emulation passes the enforced bounds (test_gpu_stage_isolation.STAGE_BOUNDS) with tanh biased up, down
and with random signs.  Discrimination: each mutant of the emulation fails bptt_step_o or bptt_step_ijf.  Every report row
(build/bptt_steps_cpu_report.jsonl) also carries the ratio of the free-running dz_all check, which sees few of them."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_refs as S  # noqa: E402
import test_gpu_stage_isolation as B  # noqa: E402       the enforced bounds; importing the module needs no GPU
from oracle import crnn_oracle as O  # noqa: E402
from stage_check import Checker, ulp_bf16  # noqa: E402

REPORT = "bptt_steps_cpu_report.jsonl"
HID = S.HID


def _operands(N, W, widths, seed=5):
    """The BPTT's operands as the GPU would hold them for test_gpu_stage_isolation.py's draw of (N, W, widths)."""
    p = O.randomize_params(O.init_params(3, dtype=np.float32, logits_scale=10.0))
    p = {k: np.asarray(v, np.float64) for k, v in p.items()}
    data, _, _, tsl = O.synth_batch(N, W, seed=seed, widths=widths, min_len=1, max_len=4, dtype=np.float64)
    with torch.no_grad():
        _, acts = O.forward(O.to_torch(p), data, tsl, return_all=True)
    T, H2 = W // 4 - 1, W // 4
    a5 = torch.zeros((N, H2, 512), dtype=torch.float64)
    a5[:, :T] = acts["reshaped_layer"].detach()
    P = {k: torch.as_tensor(v) for k, v in p.items()}
    Wb = {k: S.bf16(v) for k, v in P.items() if k.endswith("weights")}
    wh = (Wb[O.LSTM_FW + "/weights"][512:], Wb[O.LSTM_BW + "/weights"][512:])
    xp = S.xproj_stage(a5, Wb[O.LSTM_FW + "/weights"][:512], Wb[O.LSTM_BW + "/weights"][:512], P[O.LSTM_FW + "/biases"],
                       P[O.LSTM_BW + "/biases"], tsl, T)["out"]
    rec = S.recurrence_stage(S.bf16(xp), wh[0], wh[1], tsl, T)
    lstm_out = S.bf16(rec["out"])
    dl = torch.randn((T, N, 64), generator=torch.Generator().manual_seed(17), dtype=torch.float64) * 0.05
    rows = S.bf16(S.dl_rows_stage(dl, H2)["dl_rows"])
    d_out = S.bf16(S.logits_bwd(lstm_out, rows, Wb["logits/weights"])["d_lstm_out"])
    return dict(N=N, T=T, H2=H2, lens=np.asarray(tsl), wh=wh, gates=S.bf16(rec["gates"]), c=S.f32(rec["c"]), d_out=d_out)


SHAPES = {"N5_W80": (5, 80, [80, 4, 8, 57, 33]), "N2_W256": (2, 256, [256, 201]), "N3_W16": (3, 16, [16, 4, 12])}


@pytest.fixture(scope="module", params=list(SHAPES))
def ops(request):
    return request.param, _operands(*SHAPES[request.param])


@pytest.fixture(scope="module")
def ops80():
    return _operands(*SHAPES["N5_W80"])


MUTANTS = {
    "carry_without_forget_gate": "the carry dc_{s+1} f_{s+1} without f",
    "forget_gate_of_wrong_step": "dc_s f_{s+1} carried instead of dc_s f_s",
    "dzf_with_c_s": "c_s in place of c_{s-1} in dz_f",
    "partial_of_one_rank_left_out": "rank 5's partial product not added",
    "partials_of_step_s_plus_2": "the other exchange buffer: dz of step s+2",
    "tanh_of_c_prev": "tanh(c_{s-1}) in place of tanh(c_s)",
    "backward_frame_off_by_one": "backward direction at frame len-s for rows with len < T",
    "wh_off_by_1pct": "W_h scaled by 1 + 0.01 U(-1, 1)",
}


def emulate(E, sign=1.0, mutant=None, seed=0):
    """lstm_bwd_ks_kernel's arithmetic in f32 (see the module docstring) -> dz_all [N, H2, 2048] (bf16 values, frame order,
    permuted gate columns).  sign: +1 / -1 (tanh too large / too small by D_TANH relative) or "random" (either, per
    element and step)."""
    N, T, H2, lens = E["N"], E["T"], E["H2"], E["lens"]
    L = S.clamp_lens(lens, T)
    gen = torch.Generator().manual_seed(seed)
    dz_all = torch.zeros((N, H2, 2048), dtype=torch.float64)
    ar = torch.arange(N)
    for d in range(2):
        wh = E["wh"][d]
        if mutant == "wh_off_by_1pct":
            wh = wh * (1 + 0.01 * (2 * torch.rand(wh.shape, generator=gen, dtype=torch.float64) - 1))
        whp = S.to_perm(wh).reshape(HID, 8, 8, 16)                     # [unit, rank, k-step, 16]
        z1 = torch.zeros((N, 1024), dtype=torch.float64)                # dz of step s+1 (permuted), and of step s+2
        z2 = torch.zeros_like(z1)
        dcr = torch.zeros((N, HID), dtype=torch.float32)
        f_prev = torch.zeros_like(dcr)
        for s in range(T - 1, -1, -1):
            act = torch.tensor([s < v for v in L])
            if d == 0:
                t = [s] * N
            else:
                t = [(v - s if (mutant == "backward_frame_off_by_one" and v < T) else v - 1 - s) if s < v else s for v in L]
            t = torch.tensor(t)
            rec = torch.zeros((N, HID), dtype=torch.float32)
            if s < T - 1:
                src = z2 if mutant == "partials_of_step_s_plus_2" else z1
                pk = torch.einsum("nrkx,urkx->nrku", src.reshape(N, 8, 8, 16), whp)
                part = torch.zeros((N, 8, HID), dtype=torch.float32)
                for k in range(8):                                      # f32 accumulation over the k-steps
                    part = (part.double() + pk[:, :, k]).float()
                for r in range(8):                                      # bf16 partials, f32 sum in rank order
                    if mutant == "partial_of_one_rank_left_out" and r == 5:
                        continue
                    rec = rec + part[:, r].to(torch.bfloat16).float()
            gi, gj, gf, go = E["gates"][d, :, s].float().unbind(-2)
            cc = E["c"][d, :, s].float()
            cp = E["c"][d, :, s - 1].float() if s > 0 else torch.zeros_like(cc)
            dh = E["d_out"][ar, t, d * HID:(d + 1) * HID].float()
            dht = dh + rec
            sg = (torch.randint(0, 2, cc.shape, generator=gen) * 2 - 1).double() if sign == "random" else sign
            th = torch.tanh((cp if mutant == "tanh_of_c_prev" else cc).double())
            tc = (th * (1 + sg * S.D_TANH)).float()
            dc = dcr + dht * go * (1 - tc * tc)
            dzo = dht * tc * go * (1 - go)
            dzi = dc * gj * gi * (1 - gi)
            dzj = dc * gi * (1 - gj * gj)
            dzf = dc * (cc if mutant == "dzf_with_c_s" else cp) * gf * (1 - gf)
            if mutant == "carry_without_forget_gate":
                dcr_new = dc
            elif mutant == "forget_gate_of_wrong_step":
                dcr_new = dc * f_prev
            else:
                dcr_new = dc * gf
            a = act[:, None]
            z = torch.where(a, torch.cat([dzi, dzj, dzf, dzo], -1), 0.0).to(torch.bfloat16).double()
            zp = S.to_perm(z)
            dz_all[ar, t, d * 1024:(d + 1) * 1024] = zp
            dcr = torch.where(a, dcr_new, dcr)
            f_prev = torch.where(a, gf, f_prev)
            z2, z1 = z1, zp
    return dz_all


def _check(case, E, dz):
    """The per-step checks and, for comparison, the free-running dz_all check (test_gpu_stage_isolation._backward_checks)."""
    ck = Checker(case, B.STAGE_BOUNDS, REPORT, ulp_bf16)
    T, lens = E["T"], E["lens"]
    bs = B.bptt_step_checks(ck, E["d_out"], E["gates"], E["c"], E["wh"], dz, lens, T)
    r = S.bptt_stage(E["d_out"], E["gates"], E["c"], E["wh"][0], E["wh"][1], lens, T, dz_in=dz)
    valid = torch.arange(E["H2"])[None, :] < torch.as_tensor(S.clamp_lens(lens, T))[:, None]
    ck.close_scaled("dz_all", dz, r["dz"], mask=valid[..., None].expand(r["dz"].shape))
    return ck, bs


@pytest.mark.parametrize("sign", [1.0, -1.0, "random"])
def test_f32_emulation_passes_the_step_bounds(ops, sign):
    """The kernel's arithmetic, tanh at either end of its error, stays within the enforced bounds of every step; the carry
    is recovered from the stored dz wherever a step has a successor, and some partials sit near a rounding midpoint."""
    name, E = ops
    ck, bs = _check(f"{name}/tanh_{sign}", E, emulate(E, sign, seed=1))
    rows = {r["stage"]: r for r in ck.rows}
    ck.report()
    assert not ck.fail, "\n".join(ck.fail)
    assert rows["bptt_step_ijf"]["carry_recovered"] > 0 or E["T"] == 1
    assert rows["bptt_step_o"]["near_midpoint_partials"] > 0


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_step_checks_fail_every_mutant(ops80, mutant):
    """Each mutant of the emulation fails bptt_step_o or bptt_step_ijf; the row records dz_all's ratio as well."""
    E = ops80
    ck, _ = _check(f"mutant/{mutant}", E, emulate(E, 1.0, mutant, seed=1))
    rows = {r["stage"]: r for r in ck.rows}
    ratios = {k: round(rows[k]["max_ratio"], 3) for k in ("bptt_step_o", "bptt_step_ijf", "dz_all")}
    ck._record("mutant_summary", 0.0, what=MUTANTS[mutant], **ratios)
    ck.report()
    assert max(ratios["bptt_step_o"], ratios["bptt_step_ijf"]) > 1.0, (mutant, ratios)


def test_carry_fallback_is_carried_and_counted(ops80):
    """Where both factors a carry could be recovered from are zero (i = 1 and |j| = 1 in bf16), the reference carries its
    own dc of the next step: forced here on one row's steps, the emulation still passes and the fallbacks are counted."""
    E = dict(ops80)
    g = E["gates"].clone()
    n, steps = 0, [3, 4, 5, 9]                       # a run of three and a single step, all with successors
    g[:, n, steps, 0] = 1.0
    g[:, n, steps, 1] = 1.0
    E["gates"] = g
    ck, bs = _check("carry_fallback", E, emulate(E, "random", seed=2))
    ck.report()
    assert not ck.fail, "\n".join(ck.fail)
    assert int(bs["fallback"].sum()) == 2 * len(steps) * HID
