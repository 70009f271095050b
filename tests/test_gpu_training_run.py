"""Every stage per element through a multi-step training run, and on workspaces and outputs filled with NaN before use.

The stage checks of test_gpu_stage_isolation.py run on a model whose parameters load_params just wrote, once, on a workspace
straight from torch.empty.  Training never runs in that state after its first step.  Here:

Training run (one model, one engine, set_training, set_solver; Adam, Momentum and RMSProp): five real steps -- forward, CTC
loss with grad_scale 1/N, backward, apply_gradients, as SolverWrapper runs them -- over batch shapes that change as
BucketSampler changes them (N130_W40 -> N5_W80 -> N3_W80 (same W, other N) -> N3_W160 -> N130_W40, the return allocating a
new workspace).  From step 2 on every step runs the full per-element forward and backward stage check (_check_step, the
existing STAGE_BOUNDS) against the parameters the solver just wrote, after asserting that the step changed the bf16 rounding
of at least MIN_SHARE of every weight tensor (else a stale bf16 operand cache would be invisible).  Every solver update is
checked per element against fp64 on the kernel's own inputs (test_gpu_solvers.py's convention, MEASURED below), the
simulated data-parallel call bit for bit against the single-device one, total_loss against mean(costs) + wd * 1/2 sum w^2 of
the parameters that step's forward ran with, and last_grad_norm against the fp64 norm of the finished gradient.  A control
shows the check sees a stale cache: parameters rewritten in place without crnn_model_params_changed fail it, and so does
W_h alone 1 % off, through the recurrence's and the BPTT's per-step checks.

NaN-filled buffers: a buffer filled with 0xFF bytes holds NaN as bf16, f32 and f64.  Before first use the engine's
workspace and every caller-owned output (logits, CTC costs / gradient / workspace, greedy and beam outputs, the beam arena)
are filled so; the checks must pass and every output must equal, bit for bit, the same call on zero-filled buffers (where
two zero-filled runs agree bit for bit; the weight gradients, summed with f32 atomics, must be NaN-free and within their
stage bounds).  Between steps the workspace is filled again at the same (N, W, pointer): the workspace's contents before a
forward must not matter (include/crnn_ctc.h).

No value the kernels read from the workspace or the outputs is used as an address, so a stray read shows up as NaN in a
checked value and cannot fault.  By reading the sources: the pool arg-max bytes am1 / am2 / am3 are compared with the
window position, never used as an index (unpool_relu_bwd_kernel, conv1_wgrad_tc); the LSTM and BPTT kernels index by
time_step_len (a caller input) and keep their h / dz exchange buffers written before read; the beam arena's indices are
written before they are read; the CTC workspace holds floats; line_width is clamped into the workspace
(launch_clamp_line_width) before any kernel reads it.

Rows go to build/training_run_report.jsonl, with the time and peak GPU memory of the batch-scale run."""
import os
import sys
import time

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_refs as S  # noqa: E402
import test_gpu_solvers as GS  # noqa: E402
import test_gpu_stage_isolation as B  # noqa: E402
import test_gpu_stage_isolation_batch as BB  # noqa: E402
from stage_check import Checker, ulp_bf16, widths_of  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = B.DEV
U = 2.0 ** -24
WD, CLIP = 1e-5, 10.0
REPORT = "training_run_report.jsonl"
# lr per solver: Adam's 1e-3 moves nearly every element by about one lr, far above a bf16 ulp of the ~2e-2 weights (86 to 100 %
# of every weight tensor change their bf16 value, measured).  Momentum's first update is lr times the clipped gradient: at the
# reference's LEARNING_RATE 0.01 it changed only 9.6 to 10.0 % of the LSTM and logits weights (measured), so it runs at 2e-2
# (15.5 % at least on the first step, 24.6 % from the second on).
# RMSProp's mean square starts at 1, so its first steps are plain gradient steps too: at 3e-2 it changes 20 to 68 %.
LR = {"Adam": 1e-3, "Momentum": 2e-2, "RMS": 3e-2}
MIN_SHARE = 0.10
# (N, W, widths): W changes as BucketSampler changes it, N changes at fixed W, and N130_W40 comes back at the end
RUN = [(130, 40, "cycle"), (5, 80, [80, 4, 8, 57, 33]), (3, 80, [80, 57, 12]), (3, 160, [160, 8, 97]), (130, 40, "cycle")]
BOUNDS = dict(B.STAGE_BOUNDS, **{k: v for k, v in BB.BOUNDS.items() if k.startswith("ctc_")},
              total_loss=(0, 64 * U), l2_loss=(0, 64 * U), grad_norm=(0, 1e-6))
L2_LIMIT = dict(B.L2_LIMIT, **{k: v for k, v in BB.L2_LIMIT.items() if k.startswith("ctc_")})
# Largest c (in u = 2^-24 of the term magnitudes, test_gpu_solvers.py's convention) per quantity over every update of
# test_training_run_checks_every_stage_and_update and test_training_run_at_batch_scale (slots carried over from real steps),
# H100 80GB HBM3 (SXM, 700 W); the enforced bound is 4.5x.
MEASURED = {"Adam": {"params": 4.87, "adam_m": 3.83, "adam_v": 7.37}, "Momentum": {"params": 2.25, "accum": 2.58},
            "RMS": {"params": 3.77, "ms": 0.78, "mom": 5.04}}
SOLVER_BOUND = {s: {k: 4.5 * v for k, v in d.items()} for s, d in MEASURED.items()}


def _checker(case, bounds=BOUNDS, l2=L2_LIMIT):
    return Checker(case, bounds, REPORT, ulp_bf16, l2)


def _model(solver, pn=None, compute_dtype="bf16", training=True):
    from lstm_ctc_ocr_b200 import engine
    from oracle import crnn_oracle as O
    pn = pn if pn is not None else O.randomize_params(O.init_params(3, dtype=np.float32, logits_scale=10.0))
    m = engine.CrnnModel(weight_decay=WD, device=DEV, compute_dtype=compute_dtype)
    m.load_params(pn)
    if training:
        m.set_training(True)
        m.set_solver(solver, momentum=0.9)
    return m, pn


def _batch(N, W, widths, seed=5):
    from oracle import crnn_oracle as O
    return O.synth_batch(N, W, seed=seed, widths=widths_of(N, W, widths), min_len=1, max_len=4)


def _params_now(m):
    return {k: m.tensor(k).cpu().numpy().copy() for k in m.table}


def _fill_ws(m, N, W, byte, lines=False):
    """The engine's workspace for (N, W) (allocated if needed, the pointer kept), every byte set to `byte`."""
    m._workspace(N, W, lines=lines)
    m._ws.fill_(byte)
    return m._ws.data_ptr()


def _poisoned(shape, dtype, byte=255):
    t = torch.empty(shape, dtype=dtype, device=DEV)
    t.view(torch.uint8).fill_(byte)
    return t


def _bits(t):
    """The raw bytes of a tensor, for bit-for-bit comparison (NaN equal to itself)."""
    return t.contiguous().view(torch.uint8)


def _same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(_bits(a), _bits(b))


def _finite(t):
    return bool(torch.isfinite(t.float()).all()) if t.dtype.is_floating_point else True


def _ctc_costs(ck_store):
    """A ctc callback for _check_step: the CTC gradient (grad_scale 1/N) checked against torch's fp64 CTC by
    test_gpu_stage_isolation_batch._ctc_grad (tests/ctc_refs.py), the costs of the same logits kept for the loss check."""
    def ctc(ck, logits, lab, ll, tsl):
        from lstm_ctc_ocr_b200 import engine
        t = lambda a: torch.tensor(a, device=DEV)
        costs, _ = engine.ctc_loss(logits, t(lab), t(ll), t(tsl), want_grad=False, max_label_len=int(ll.max()))
        ck_store["costs"] = costs.clone()
        return BB._ctc_grad(ck, logits, lab, ll, tsl)
    return ctc


def _bf16_shares(before, m):
    """Per weight tensor: the share of elements whose bf16 rounding the last update changed."""
    out = {}
    for k in m.table:
        if k.endswith("weights"):
            a = torch.as_tensor(before[k]).to(DEV).to(torch.bfloat16)
            b = m.tensor(k).to(torch.bfloat16)
            out[k] = float((a != b).float().mean())
    return out


def _loss_checks(ck, m, costs, pn):
    """total_loss of the costs against mean(costs) + wd * 1/2 sum w^2 over O.L2_NAMES of the parameters the forward ran with, in
    fp64; and total_loss of zero costs (the L2 term alone, m->sumsq) against its fp64 value."""
    from oracle import crnn_oracle as O
    wd = float(np.float32(WD))
    l2 = wd * 0.5 * sum(float((pn[k].astype(np.float64) ** 2).sum()) for k in O.L2_NAMES)
    c = costs.double()
    ok = torch.isfinite(c)
    assert bool(ok.all()), "CTC costs must be finite on feasible labels"
    ref = float(c.mean()) + l2
    got = float(m.total_loss(costs).item())
    ck.close("total_loss", np.array([got]), np.array([ref]), np.array([float(c.abs().mean()) + l2]))
    got0 = float(m.total_loss(torch.zeros_like(costs)).item())
    ck.close("l2_loss", np.array([got0]), np.array([l2]), np.array([l2]))


def _solver_update(ck, m, solver, lr, step, mask, worst, hp=None):
    """One apply_gradients on the backward's raw gradients, checked per element against fp64 on the kernel's own inputs, its
    simulated data-parallel twin bit for bit, and last_grad_norm against the fp64 norm of the finished gradient."""
    s = GS._state(m)
    raw = m.grads.clone()
    GS._call(m, solver, lr, CLIP, 1.0, 1.0, hp, step=step)
    single = GS._state(m)
    gn_gpu = m.last_grad_norm()
    GS._load_state(m, s)
    m.grads.copy_(raw * 2)
    GS._call(m, solver, lr, CLIP, 0.5, 2.0, hp, step=step)
    for k in single:
        assert torch.equal(single[k], getattr(m, k)), (solver, step, k, "data-parallel call differs")
    assert m.last_grad_norm(0.5) == gn_gpu
    kw = {"momentum": 0.9} if solver == "Momentum" else {"step": (hp or {}).get("step", step)} if solver == "Adam" else {}
    ref, gn = GS._reference(solver, s, GS._f64(raw), mask, WD, lr, CLIP, **kw)
    ck.close("grad_norm", np.array([gn_gpu]), np.array([gn]), np.array([gn]))
    for k, c in GS._c_needed(ref, m, solver).items():
        worst[k] = max(worst.get(k, 0.0), c)
    return gn


@pytest.mark.parametrize("solver", ["Adam", "Momentum", "RMS"])
def test_training_run_checks_every_stage_and_update(solver):
    m, pn = _model(solver)
    mask = GS._l2_mask(m)
    lr = LR[solver]
    fail, worst, shares, norms = [], {}, [], []
    cks = []
    for step, (N, W, widths) in enumerate(RUN, start=1):
        batch = _batch(N, W, widths, seed=5 + step)
        case = f"{solver}/step{step}_N{N}_W{W}"
        ck = _checker(case)
        store = {}
        before = _params_now(m)
        if step == 1:                      # the fresh model: test_gpu_stage_isolation.py's check
            _fwd_bwd(m, batch, _ctc_costs(store), ck)
        else:
            B._check_step(m, before, batch, case, dev=DEV, chunk=BB.CHUNK, ctc=_ctc_costs(store), ck=ck)
        _loss_checks(ck, m, store["costs"], before)
        norms.append(_solver_update(ck, m, solver, lr, step, mask, worst))
        sh = _bf16_shares(before, m)
        shares.append({k.split("/")[-3] if "lstm_cell" in k else k.split("/")[0]: round(v, 3) for k, v in sh.items()})
        low = {k: v for k, v in sh.items() if v < MIN_SHARE}
        assert not low, f"{case}: the update moved too few bf16 operands to show a stale cache: {low}"
        cks.append(ck)
    # the update of the last step feeds no check; one more forward / backward on the first shape checks those parameters too
    N, W, widths = RUN[1]
    ck = _checker(f"{solver}/after_step{len(RUN)}_N{N}_W{W}")
    B._check_step(m, _params_now(m), _batch(N, W, widths, seed=99), ck.case, dev=DEV, chunk=BB.CHUNK, ctc=_ctc_costs({}), ck=ck)
    cks.append(ck)
    ck = cks[0]
    ck._record("bf16_change_shares", 0.0, **{f"step{i + 1}": s for i, s in enumerate(shares)})
    ck._record("solver_c_needed", max(worst[k] / SOLVER_BOUND[solver][k] for k in worst), c_needed=worst,
               bound=SOLVER_BOUND[solver], grad_norms=norms)
    for c in cks:
        c.report()
        fail += c.fail
    assert not fail, "\n".join(fail)


def _perturb_in_place(m, rel=0.05, seed=3, names=None):
    """New f32 parameters written into m.params in place, without crnn_model_params_changed (the misuse include/crnn_ctc.h
    documents): every weight (or the tensors `names`, name -> row slice) scaled by 1 + rel * U(-1, 1)."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    for w in [m.params] if names is None else [m.tensor(k)[rows] for k, rows in names.items()]:
        w.mul_(1.0 + rel * (2.0 * torch.rand(w.shape, generator=gen, device=DEV) - 1.0))
    torch.cuda.synchronize()


# the stages that read a bf16 weight cache: the forward's (prepare_weights) and the backward's data gradients
# (prepare_weights_bwd), the recurrence's W_h (step_gates, step_c: each step on its own saved inputs) and the BPTT's
# (bptt_step_o, bptt_step_ijf).  conv1 reads the f32 weights and each bias is read as f32, so they follow the new values.
STALE_STAGES = ("conv2", "conv3_1", "conv3_2", "a4a_pre", "a4b_pre", "conv5", "xproj", "logits",
                "d_lstm_out", "d_a5", "d_a4b", "d_pre4a", "d_a3p", "d_pre31", "d_a2", "d_a1",
                "step_gates", "step_c", "bptt_step_o", "bptt_step_ijf")
# only the recurrent weights W_h of both directions, 1 % off: the forward's and the backward's per-step checks see it
STALE_WH = {B.FW + "/weights": slice(512, 768), B.BW + "/weights": slice(512, 768)}
STALE_WH_STAGES = ("step_c", "bptt_step_o")


def _stale_cache_control(tag, must_fail, rel, names=None):
    """After a forward and backward, parameters rewritten in place without crnn_model_params_changed leave the bf16 caches
    stale: the stage check must fail on every stage of `must_fail`, and pass again after params_changed."""
    from lstm_ctc_ocr_b200._lib import check
    m, pn = _model("Adam")
    N, W, widths = RUN[1]
    batch = _batch(N, W, widths)
    ck = _checker(f"{tag}/fresh")
    B._check_step(m, _params_now(m), batch, ck.case, dev=DEV, ck=ck)
    ck.assert_ok()
    _perturb_in_place(m, rel, names=names)
    ck = _checker(f"{tag}/in_place")
    B._check_step(m, _params_now(m), batch, ck.case, dev=DEV, ck=ck)
    ck.report()
    rows = {r["stage"]: r for r in ck.rows}
    passed = [s for s in must_fail if rows[s]["max_ratio"] <= 1.0]
    assert not passed, f"a stale bf16 cache went unnoticed in {passed}"
    check(m.lib.crnn_model_params_changed(m.handle))
    ck = _checker(f"{tag}/params_changed")
    B._check_step(m, _params_now(m), batch, ck.case, dev=DEV, ck=ck)
    ck.assert_ok()


def test_stage_check_sees_a_stale_weight_cache():
    """Control: every parameter 5 % off in place.  The check must fail on every conv stage that reads a cache, xproj,
    logits, the data gradients, and the recurrence's and the BPTT's per-step checks."""
    _stale_cache_control("stale", STALE_STAGES, 0.05)


def test_stage_check_sees_stale_recurrent_weights():
    """Control: only W_h of both LSTM directions 1 % off in place.  The recurrence's step_c and the BPTT's bptt_step_o must
    fail; the report's dz_all row shows how far the free-running BPTT check stays from noticing."""
    _stale_cache_control("stale_wh", STALE_WH_STAGES, 0.01, STALE_WH)


def test_training_run_at_batch_scale():
    """Adam, 512 x {256, 80, 160}: three steps, steps 2 and 3 checked per element with test_gpu_stage_isolation_batch.py's
    chunked fp64 references on the GPU and its bounds.  Records the time and the peak GPU memory."""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    m, pn = _model("Adam")
    mask = GS._l2_mask(m)
    worst, fail, cks = {}, [], []
    bounds = dict(BB.BOUNDS, total_loss=BOUNDS["total_loss"], l2_loss=BOUNDS["l2_loss"], grad_norm=BOUNDS["grad_norm"])
    for step, W in enumerate((256, 80, 160), start=1):
        N = 512
        case = f"batch/step{step}_N{N}_W{W}"
        ck = _checker(case, bounds, BB.L2_LIMIT)
        data, lab, ll, tsl = _batch(N, W, BB._widths(N, W), seed=40 + step)
        store = {}
        before = _params_now(m)
        if step == 1:
            _fwd_bwd(m, (data, lab, ll, tsl), _ctc_costs(store), ck)
        else:
            F_, _ = B._check_step(m, before, (data, lab, ll, tsl), case, dev=DEV, chunk=BB.CHUNK, ctc=_ctc_costs(store), ck=ck)
            del F_
        _loss_checks(ck, m, store["costs"], before)
        _solver_update(ck, m, "Adam", LR["Adam"], step, mask, worst)
        low = {k: v for k, v in _bf16_shares(before, m).items() if v < MIN_SHARE}
        assert not low, (case, low)
        cks.append(ck)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    cks[0]._record("peak_gpu_memory", peak / BB.PEAK_LIMIT, max_memory_allocated=peak, seconds=round(time.time() - t0, 1))
    cks[0]._record("solver_c_needed", max(worst[k] / SOLVER_BOUND["Adam"][k] for k in worst), c_needed=worst)
    for c in cks:
        c.report()
        fail += c.fail
    assert not fail, "\n".join(fail)


# ---- NaN-filled buffers ---------------------------------------------------------------------------------------------------------
def _dlogits(N, W):
    """_check_step's default backward input: the seeded random d logits."""
    gen = torch.Generator(device="cpu").manual_seed(17)
    return (torch.randn((W // 4 - 1, N, 64), generator=gen) * 0.05).float().to(DEV)


def _fwd_bwd(m, batch, ctc=None, ck=None):
    data, lab, ll, tsl = batch
    t = lambda a: torch.tensor(a, device=DEV)
    N, W = data.shape[0], data.shape[1]
    logits = m.forward(t(data), t(tsl))
    dl = _dlogits(N, W) if ctc is None else ctc(ck, logits, lab, ll, tsl)
    m.backward(t(data), t(tsl), dl)
    torch.cuda.synchronize()
    return logits


def _snapshot(m, N, W, logits, tsl, train=True):
    """Every quantity the last forward (and backward) left: the taps, the raw non-bf16 buffers, the logits and the gradients.
    The saved gates and cell states of the recurrence only where a step ran (t < len): the backward reads nothing else of
    them, and the rest of those buffers is never written."""
    out = {k: m.tap(k, N, W) for k in B.FWD_TAPS}
    out.update({"raw/" + k: m.tap_raw(k, N, W) for k in ("bn", "stats")})
    out["logits"] = logits.clone()
    if train:
        T = W // 4 - 1
        out.update({"raw/" + k: m.tap_raw(k, N, W) for k in ("am1", "am2", "am3")})
        L = torch.as_tensor(S.clamp_lens(tsl, T), device=DEV)
        act = (torch.arange(T, device=DEV)[None, :] < L[:, None])[None].expand(2, -1, -1)
        out["gates_steps"] = S.unpack_gates(m.tap("gates", N, W), N)[act]
        out["csave_steps"] = S.unpack_csave(m.tap_raw("csave", N, W), N)[act]
        out.update({k: m.tap(k, N, W) for k in B.BWD_TAPS})
        out.update({"grad/" + k: m.grad_tensor(k).clone() for k in m.table})
    torch.cuda.synchronize()
    return out


def _bit_identity(ck, poisoned, zero_a, zero_b):
    """Quantities two zero-filled runs reproduce bit for bit must come out the same from the NaN-filled run; the others, and
    every weight gradient (summed with f32 atomics, so two runs agree only by chance), must be NaN-free (their values are
    checked per element by the stage checks)."""
    repro = [k for k in zero_a if not k.startswith("grad/") and _same_bits(zero_a[k], zero_b[k])]
    other = [k for k in zero_a if k not in repro]
    diff = [k for k in repro if not _same_bits(poisoned[k], zero_a[k])]
    nan = [k for k in other if not _finite(poisoned[k])]
    ck._record("bit_identical_to_zero_filled", 0.0 if not diff else float("inf"), mismatches=len(diff), differ=diff[:12],
               reproducible=len(repro))
    ck._record("non_reproducible_finite", 0.0 if not nan else float("inf"), mismatches=len(nan), not_finite=nan[:12],
               atomics=other[:30])


def _zero_runs(m, batch, train=True):
    N, W = batch[0].shape[0], batch[0].shape[1]
    snaps = []
    for _ in range(2):
        _fill_ws(m, N, W, 0)
        lg = _fwd_bwd(m, batch) if train else _forward(m, batch, torch.zeros((W // 4 - 1, N, 64), device=DEV))
        snaps.append(_snapshot(m, N, W, lg, batch[3], train))
    return snaps


def _forward(m, batch, out):
    data, _, _, tsl = batch
    lg = m.forward(torch.tensor(data, device=DEV), torch.tensor(tsl, device=DEV), out=out)
    torch.cuda.synchronize()
    return lg


@pytest.mark.parametrize("N,W,widths,seed", B.STAGE_SHAPES)
def test_poisoned_workspace_before_first_use(N, W, widths, seed, request):
    """A training workspace filled with NaN before its first forward: every stage check passes and every output equals the
    zero-filled run's."""
    case = "first_use/" + request.node.callspec.id
    m, pn = _model("Adam")
    batch = _batch(N, W, widths, seed=seed)
    ck = _checker(case)
    _fill_ws(m, N, W, 255)
    F_, _ = B._check_step(m, pn, batch, case, dev=DEV, chunk=BB.CHUNK, ck=ck)
    poisoned = _snapshot(m, N, W, F_.logits, batch[3])
    za, zb = _zero_runs(m, batch)
    _bit_identity(ck, poisoned, za, zb)
    ck.assert_ok()


@pytest.mark.parametrize("solver", ["Adam", "RMS"])
@pytest.mark.parametrize("N,W,widths", [(130, 40, "cycle"), (3, 160, [160, 8, 97])], ids=["N130_W40", "N3_W160"])
def test_poisoned_workspace_between_steps(solver, N, W, widths):
    """Scratch contract: a step (forward, backward, solver update), then the workspace filled with NaN at the same (N, W,
    pointer), then the next step's forward and backward: every stage check passes and the outputs equal those of the same
    step on a zero-filled workspace."""
    m, pn = _model(solver)
    batch = _batch(N, W, widths)
    _fwd_bwd(m, batch)
    m.apply_gradients(LR[solver], 1, clip=CLIP)
    ptr = m._ws.data_ptr()
    assert _fill_ws(m, N, W, 255) == ptr
    case = f"between_steps/{solver}/N{N}_W{W}"
    ck = _checker(case)
    data, lab, ll, tsl = _batch(N, W, widths, seed=6)
    F_, _ = B._check_step(m, _params_now(m), (data, lab, ll, tsl), case, dev=DEV, chunk=BB.CHUNK, ck=ck)
    assert m._ws.data_ptr() == ptr
    poisoned = _snapshot(m, N, W, F_.logits, tsl)
    za, zb = _zero_runs(m, (data, lab, ll, tsl))
    _bit_identity(ck, poisoned, za, zb)
    ck.assert_ok()


@pytest.mark.parametrize("N,W,widths", [(130, 40, "cycle"), (3, 160, [160, 8, 97]), (512, 256, None)],
                         ids=["N130_W40", "N3_W160", "N512_W256"])
def test_poisoned_inference_plan(N, W, widths):
    """The inference plan (bench.py's forward) on a NaN-filled workspace and NaN-filled logits: every forward stage within its
    bound, the logits and every tap bit-identical to zero-filled buffers."""
    m, pn = _model(None, training=False)
    widths = BB._widths(N, W) if widths is None else widths
    batch = _batch(N, W, widths)
    _fill_ws(m, N, W, 255)
    out = _poisoned((W // 4 - 1, N, 64), torch.float32)
    lg = _forward(m, batch, out)
    G = {k: m.tap(k, N, W) for k in B.FWD_TAPS}
    Rr = {k: m.tap_raw(k, N, W) for k in ("bn", "stats")}
    ck = _checker(f"inference/N{N}_W{W}")
    F_ = B._Refs(pn, G, Rr, batch[0], batch[3], lg, N, W, DEV, BB.CHUNK)
    B._forward_checks(ck, F_, train=False)
    poisoned = _snapshot(m, N, W, lg, batch[3], train=False)
    za, zb = _zero_runs(m, batch, train=False)
    _bit_identity(ck, poisoned, za, zb)
    ck.assert_ok()


def test_poisoned_forward_lines():
    """Packed evaluation (forward_lines) on a NaN-filled workspace and logits: bit-identical to zero-filled buffers."""
    m, pn = _model(None, training=False)
    N, W = 6, 96
    lw = [96, 8, 40, 64, 12, 96]
    data, _, _, _ = _batch(N, W, lw)
    tsl = np.array([w // 4 - 1 for w in lw], np.int32)
    t = lambda a: torch.tensor(a, device=DEV)

    def run(byte):
        _fill_ws(m, N, W, byte, lines=True)
        out = _poisoned((W // 4 - 1, N, 64), torch.float32, byte)
        lg = m.forward_lines(t(data), t(np.array(lw, np.int32)), t(tsl), out=out)
        torch.cuda.synchronize()
        return lg.clone()
    p, a, b = run(255), run(0), run(0)
    assert _same_bits(a, b)
    assert _same_bits(p, a), "forward_lines on a NaN-filled workspace differs from the zero-filled run"


@pytest.mark.parametrize("dtype", ["fp8", "f32", "tf32"])
def test_poisoned_eval_paths(dtype):
    """fp8 calibration and forward, and the split-bf16 / tf32 forwards, on NaN-filled workspaces and logits: the fp8 scales and
    every logit bit-identical to zero-filled buffers."""
    m, pn = _model(None, compute_dtype=dtype, training=False)
    N, W = 130, 80
    batch = _batch(N, W, "cycle")
    t = lambda a: torch.tensor(a, device=DEV)

    def run(byte):
        if dtype == "fp8":
            _fill_ws(m, N, W, byte)
            m.calibrate_fp8(t(batch[0]), t(batch[3]))
            scales = m.fp8_scales()
        _fill_ws(m, N, W, byte)
        lg = _forward(m, batch, _poisoned((W // 4 - 1, N, 64), torch.float32, byte)).clone()
        return lg, (scales if dtype == "fp8" else None)
    p, a, b = run(255), run(0), run(0)
    assert _same_bits(a[0], b[0])
    assert _same_bits(p[0], a[0]), f"{dtype}: logits on a NaN-filled workspace differ from the zero-filled run"
    if dtype == "fp8":
        assert np.array_equal(p[1], a[1])


def _ctc_case(T, N, L, seed=0):
    """Logits, labels (1 .. L long; sample 0 holds an out-of-range id, sample 1 the blank, sample 2 does not fit its length) and
    input lengths (0, 1, T and in between)."""
    rng = np.random.default_rng(seed)
    logits = torch.tensor(rng.standard_normal((T, N, 64)).astype(np.float32) * 3, device=DEV)
    ll = rng.integers(1, L + 1, size=N).astype(np.int32)
    il = rng.integers(0, T + 1, size=N).astype(np.int32)
    il = np.maximum(il, np.minimum(2 * ll + 1, T)).astype(np.int32)
    il[3], il[4], il[5] = T, 1, 0
    ll[2], il[2] = min(L, T), max(0, min(L, T) // 2 - 1)
    lab = [rng.integers(1, 64, size=n).astype(np.int32) for n in ll]
    lab[0][0], lab[1][-1] = 64, 0
    return logits, np.concatenate(lab), ll, il


@pytest.mark.parametrize("T,N,L,ws", [(20, 40, 4, False), (500, 8, 10, False), (250, 16, 25, False), (120, 24, 60, False),
                                      (600, 8, 20, True), (90, 12, 100, True)],
                         ids=["T20_L4", "T500_L10", "T250_L25", "T120_L60", "ws_T600", "ws_L100"])
def test_poisoned_ctc_outputs(T, N, L, ws):
    """CTC loss with NaN-filled costs, gradient and workspace (the shared-memory kernels at four lengths, the workspace kernel
    for long frames and long labels): bit-identical to zero-filled outputs; invalid-label and infeasible samples and every
    frame past input_len have an exactly zero gradient."""
    from lstm_ctc_ocr_b200 import engine
    logits, lab, ll, il = _ctc_case(T, N, L)
    t = lambda a: torch.tensor(a, device=DEV)
    nbytes = engine.ctc_workspace_bytes(T, N, 64, int(ll.max()))
    assert (nbytes > 0) == ws

    def run(byte):
        costs = _poisoned((N,), torch.float32, byte)
        grad = _poisoned((T, N, 64), torch.float32, byte)
        w = _poisoned((nbytes,), torch.uint8, byte) if nbytes else None
        engine.ctc_loss(logits, t(lab), t(ll), t(il), want_grad=True, grad_scale=0.25, max_label_len=int(ll.max()), costs=costs,
                        grad=grad, workspace=w)
        torch.cuda.synchronize()
        return costs, grad
    (pc, pg), (ac, ag), (bc, bg) = run(255), run(0), run(0)
    assert _same_bits(ac, bc) and _same_bits(ag, bg)
    assert _same_bits(pc, ac) and _same_bits(pg, ag), "CTC outputs on NaN-filled buffers differ from the zero-filled run"
    assert bool(torch.isnan(pc[:2]).all()), "invalid label ids give cost NaN"
    assert float(pc[2]) == 0.0, "labels that do not fit their length give cost 0"
    assert bool((pg[:, :3] == 0).all()), "invalid and infeasible samples have a zero gradient"
    past = torch.arange(T, device=DEV)[:, None] >= t(il)[None, :].long()
    assert bool((pg[past] == 0).all())
    assert bool(torch.isfinite(pg).all()) and bool(torch.isfinite(pc[3:]).all())


def test_poisoned_decoder_outputs():
    """Greedy decoding and the device beam decoder into NaN-filled (0xFF) outputs and beam arena: bit-identical to zero-filled
    buffers, zero padded past each length."""
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200._lib import check
    T, N, C = 60, 40, 64
    logits, _, _, il = _ctc_case(T, N, 4, seed=2)
    d_il = torch.tensor(il, device=DEV)
    lib = engine._lib.load()
    nb = engine.beam_workspace_bytes(T, N, C, 16)

    def run(byte):
        out = _poisoned((N, T), torch.int32, byte)
        ol = _poisoned((N,), torch.int32, byte)
        check(lib.crnn_ctc_greedy(logits.data_ptr(), d_il.data_ptr(), T, N, C, engine.TF_BLANK, 0, out.data_ptr(), ol.data_ptr(),
                                  engine._stream()))
        bo = _poisoned((N, T), torch.int32, byte)
        bl = _poisoned((N,), torch.int32, byte)
        nlp = _poisoned((N,), torch.float32, byte)
        arena = _poisoned((nb,), torch.uint8, byte)
        check(lib.crnn_ctc_beam_search_device(logits.data_ptr(), d_il.data_ptr(), T, N, C, 16, 1, 0, bo.data_ptr(), bl.data_ptr(),
                                              nlp.data_ptr(), arena.data_ptr(), nb, engine._stream()))
        torch.cuda.synchronize()
        return out, ol, bo, bl, nlp
    p, a, b = run(255), run(0), run(0)
    for i, name in enumerate(("greedy_out", "greedy_len", "beam_out", "beam_len", "beam_nlp")):
        assert _same_bits(a[i], b[i]), name
        assert _same_bits(p[i], a[i]), f"{name} on NaN-filled buffers differs from the zero-filled run"
    for out, ol in ((p[0], p[1]), (p[2], p[3])):
        pad = torch.arange(T, device=DEV)[None, :] >= ol[:, None].long()
        assert bool((out[pad] == 0).all()) and bool((ol >= 0).all()) and bool((ol <= T).all())
