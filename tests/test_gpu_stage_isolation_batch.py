"""The stage checks of test_gpu_stage_isolation.py, with the same bounds, at the batch sizes the project runs.

Several code paths are only reached at large batches: split-K weight gradients whose chunks run hundreds of K-blocks (and a
short last chunk), persistent GEMMs taking many tile rounds per CTA, thousands of BatchNorm row-group partials per channel,
and more LSTM clusters than fit in one wave.  Here every forward and backward stage and all 24 gradient tensors are checked
per element at:
  c3          1024 x 256   the benchmarked forward and the training step
  b512_W*     512 x 80 / 160 / 256   the bucketed batches of BASELINE configs[3]
  two_waves   1160 x 160   10 row tiles (the last holding 8 rows): two waves of LSTM clusters, forward and BPTT
with lengths 0, 1 and T on every 128-row tile and random lengths in between.

The fp64 references are the same functions (tests/stage_refs.py), run on the GPU over chunks of CHUNK images: per-image
stages chunk by chunk, batch reductions (BatchNorm sums, weight and bias gradients, masked column sums) summed in fp64
over the chunks.  The recurrence and BPTT bounds scale with max|ref| of each chunk, which is at most the batch's.  On
sampled images (tile edges, the shortest and longest lengths) the same references also run on the CPU and must agree
with the GPU's to 1e-12 of acc.

At c3 the backward is driven by the real CTC gradient of the GPU's own logits (engine.ctc_loss with grad_scale 1/N, as
the training step runs it), checked against tests/ctc_refs.py's fp64 CTC: costs to 1e-4 relative, the gradient per element
(ctc_grad_softmax, ctc_grad_posterior), zero past each length.  Utterances whose labels do not fit their length have no
finite fp64 cost; there the kernel must give cost 0 and a zero gradient, and that gradient, unchanged, drives the
backward.  ctc_long_kernel runs once more on the same logits, its gradient and its stored tables checked too.  The inference plan (bench.py's) of a fresh model is checked stage by stage as well: conv1 .. conv3_2 equal to
the training plan's taps bit for bit, conv4_x within one bf16 ulp.

Rows go to build/stage_isolation_batch_report.jsonl, with the peak GPU memory of each case."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ctc_refs as CR  # noqa: E402
import stage_refs as S  # noqa: E402
import test_gpu_stage_isolation as B  # noqa: E402
from stage_check import Checker, ulp_bf16, widths_of  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = B.DEV
CHUNK = 128
PEAK_LIMIT = 30 * 2 ** 30          # bytes of GPU memory one case may hold (the H100s are shared)

# The small-shape bounds, except for the weight gradients whose split-K chunks grow long at these batches.  gemm_tn
# accumulates each chunk in f32 wgmma registers, and the tensor cores' f32 accumulation truncates: each of the 4 MMA
# k-steps of a 64-deep K-block can lose up to one ulp of the partial sum, at most 2^-23 * acc, always toward zero.  So the
# error grows linearly with the K-blocks of a chunk (pick_k_splits), and every worst element measured lies between 0 and
# the fp64 value.  At 1024 x 256 a chunk holds 256 K-blocks for W_x, 64 for W_h and 32 for the logits weights (worst case
# 4 * kb * 2^-23 = 1.2e-4, 3.1e-5, 1.5e-5), and hundreds to thousands for the conv wgrads; at the small shapes one to six.
# Largest c_needed and relative L2 per weight tensor over every case below, on H100 80GB HBM3 (runs at 400 and 700 W agree
# to a few percent) -- the small shapes need at most 5.2e-6 and 7.6e-6.  A tensor gets its own bound "wgrad/<name>", 4.5x its measurement (L2 at least
# the small-shape 1e-4), only where that exceeds the small-shape c = 2.5e-5; the rest keep the small-shape bound.
MEASURED_WGRAD = {
    "logits/weights": (1.01e-6, 6.04e-7), B.FW + "/weights": (3.03e-5, 1.52e-5), B.BW + "/weights": (2.51e-5, 1.59e-5),
    "conv5/weights": (8.85e-6, 5.21e-6), "conv4_2/weights": (1.28e-4, 1.36e-4), "conv4_1/weights": (1.31e-4, 5.05e-4),
    "conv3_2/weights": (6.02e-5, 1.58e-4), "conv3_1/weights": (5.54e-5, 1.40e-4), "conv2/weights": (3.05e-5, 7.83e-5),
    "conv1/weights": (4.74e-6, 7.56e-6),
}
WGRAD = {k: (4.5 * c, max(1e-4, 4.5 * l2)) for k, (c, l2) in MEASURED_WGRAD.items() if 4.5 * c > B.STAGE_BOUNDS["wgrad"][1]}
# plus the GPU references against the CPU ones, and the CTC stages of tests/ctc_refs.py (the default kernel and, at c3,
# ctc_long_kernel): the cost of test_gpu_parity.py relative to |cost| (1e-4), the gradient per element, its relative L2
# (measured 2.4e-5)
CTC_KINDS = {"fast": 1e-4, "long": 4.5 * 2.80e-6}
BOUNDS = dict(B.STAGE_BOUNDS, **{f"wgrad/{k}": (0, c) for k, (c, _) in WGRAD.items()}, ref_cpu=(0, 1e-12),
              **{f"ctc_cost/{k}": (0, c) for k, c in CTC_KINDS.items()},
              **CR.bounds(CTC_KINDS, {k: 4.5 * CR.MEASURED_POSTERIOR[k] for k in CTC_KINDS}))
L2_LIMIT = dict(B.L2_LIMIT, **{f"wgrad/{k}": l2 for k, (_, l2) in WGRAD.items()}, **{f"ctc_grad/{k}": 1.1e-4 for k in CTC_KINDS})

CASES = [
    pytest.param(1024, 256, id="c3"),
    pytest.param(512, 80, id="b512_W80"),
    pytest.param(512, 160, id="b512_W160"),
    pytest.param(512, 256, id="b512_W256"),
    pytest.param(1160, 160, id="two_waves"),
]


def _checker(case):
    return Checker(case, BOUNDS, "stage_isolation_batch_report.jsonl", ulp_bf16, L2_LIMIT)


def _widths(N, W, seed=11):
    """Even rows cycle through lengths T, 0, 1 and four in between (every 128-row tile holds each); odd rows random."""
    cyc = widths_of(N, W, "cycle")
    rnd = np.random.default_rng(seed).integers(1, W // 4 + 1, size=N) * 4
    return [cyc[i // 2] if i % 2 == 0 else int(rnd[i]) for i in range(N)]


def _ctc_grad(ck, logits, lab, ll, tsl, long_tables=False):
    """engine.ctc_loss on the GPU's logits (grad_scale 1/N) against ctc_refs.ctc_fp64; returns the backward's d logits.
    long_tables: also run ctc_long_kernel (CRNN_CTC_KERNEL=long) on the same logits, its gradient and its stored tables
    checked as well."""
    from lstm_ctc_ocr_b200 import engine
    T, N, _ = logits.shape
    t = lambda a: torch.tensor(a, device=DEV)
    m = int(ll.max())
    costs, grad = engine.ctc_loss(logits, t(lab), t(ll), t(tsl), want_grad=True, grad_scale=1.0 / N, max_label_len=m)
    ref = CR.ctc_fp64(logits, lab, ll, S.clamp_lens(tsl, T), grad_scale=1.0 / N, max_label_len=m)
    CR.check_grad(ck, "fast", costs, grad, ref, 1.0 / N)
    if long_tables:
        os.environ["CRNN_CTC_KERNEL"] = "long"
        try:
            ws = torch.empty(engine.ctc_workspace_bytes(T, N, 64, m), dtype=torch.uint8, device=DEV)
            c_l, g_l = engine.ctc_loss(logits, t(lab), t(ll), t(tsl), want_grad=True, grad_scale=1.0 / N, max_label_len=m,
                                       workspace=ws)
        finally:
            del os.environ["CRNN_CTC_KERNEL"]
        CR.check_grad(ck, "long", c_l, g_l, ref, 1.0 / N)
        CR.check_long_workspace(ck, "long", ws, logits, c_l, ref, 0, m)
        del ws, g_l
    del ref
    return grad


def _ctc_long_too(ck, logits, lab, ll, tsl):
    return _ctc_grad(ck, logits, lab, ll, tsl, long_tables=True)


def _ref_self_check(ck, F_):
    """The GPU's fp64 references against the same functions on the CPU, on sampled images."""
    N, T = F_.N, F_.T
    idx = sorted({0, 127, 128 % N, N - 1, (N - 1) // 128 * 128, int(np.argmin(F_.tsl)), int(np.argmax(F_.tsl))})
    out = {}
    for dev in (F_.dev, "cpu"):
        P = {k: v.to(dev) for k, v in F_.P.items()}
        Wb = {k: v.to(dev) for k, v in F_.Wb.items()}
        wh = (F_.wh[0].to(dev), F_.wh[1].to(dev))
        g = lambda k: F_.G[k][idx].to(dev, torch.float64)
        steps = lambda k: F_.G[k][:, idx].to(dev, torch.float64)
        lens = F_.tsl[idx]
        r = dict(conv1=S.conv1_stage(torch.as_tensor(F_.data[idx], dtype=torch.float64, device=dev), P["conv1/weights"],
                                     P["conv1/biases"]),
                 conv2=S.conv_relu_pool22_stage(g("conv1"), Wb["conv2/weights"], P["conv2/biases"]),
                 conv3_1=S.conv_relu_stage(g("conv2"), Wb["conv3_1/weights"], P["conv3_1/biases"]),
                 conv3_2=S.conv_relu_pool12_stage(g("conv3_1"), Wb["conv3_2/weights"], P["conv3_2/biases"]),
                 a4a_pre=S.conv_bias_stage(g("conv3_2"), Wb["conv4_1/weights"], P["conv4_1/biases"]),
                 conv5=S.conv5_stage(g("conv4_2"), Wb["conv5/weights"], P["conv5/biases"]),
                 xproj=S.xproj_stage(g("conv5"), Wb[B.FW + "/weights"][:512], Wb[B.BW + "/weights"][:512],
                                     P[B.FW + "/biases"], P[B.BW + "/biases"], lens, T),
                 logits=S.logits_stage(g("lstm_out"), Wb["logits/weights"], P["logits/biases"], T))
        rec = S.recurrence_stage(g("xproj"), wh[0], wh[1], lens, T)["out"]
        r["lstm_out"] = dict(out=rec, acc=rec.abs().max())
        dz = S.bptt_stage(g("d_lstm_out"), steps("gates_steps"), steps("csave_steps"), wh[0], wh[1], lens, T,
                          dz_in=g("dz_all"))["dz"]
        r["dz_all"] = dict(out=dz, acc=dz.abs().max())
        bs = S.bptt_steps_isolated(g("d_lstm_out"), steps("gates_steps"), steps("csave_steps"), wh[0], wh[1], g("dz_all"),
                                   lens, T)
        r["bptt_steps"] = dict(out=bs["dz"], acc=bs["acc"])
        r["bptt_steps_allow"] = dict(out=bs["allow"], acc=bs["allow"])
        del bs
        c = S.conv_bwd(g("d_pre2"), g("conv1"), Wb["conv2/weights"])
        r["d_a1"] = dict(out=c["dx"], acc=c["dx_acc"])
        r["conv2/weights"] = dict(out=c["dw"], acc=c["dw_acc"])
        out[dev] = r
    for k, cpu in out["cpu"].items():
        ck.close("ref_cpu/" + k, out[F_.dev][k]["out"].cpu(), cpu["out"], cpu["acc"], key="ref_cpu")


def _inference_plan_checks(ck, F_, N, W, chunk=CHUNK):
    """bench.py's plan: a fresh model in inference mode on the same batch, every forward stage against the references
    (over chunks of `chunk` images), and its front end against the training plan's taps."""
    from lstm_ctc_ocr_b200 import engine
    m = engine.CrnnModel(device=DEV)
    m.load_params(F_.pn)
    logits = m.forward(torch.tensor(F_.data, device=DEV), torch.tensor(F_.tsl, device=DEV))
    torch.cuda.synchronize()
    G = {k: m.tap(k, N, W) for k in B.FWD_TAPS}
    R = {k: m.tap_raw(k, N, W) for k in ("bn", "stats")}
    for k in ("conv1", "conv2", "conv3_1", "conv3_2"):
        ck.exact(f"{k}_equals_training_plan", G[k], F_.G[k])
    for k in ("conv4_1", "conv4_2"):
        a, b = G[k].double(), F_.G[k].double()
        ck._record(f"{k}_within_1ulp_of_training_plan", float(((a - b).abs() / ulp_bf16(torch.maximum(a.abs(), b.abs()))).max()))
    F_.G.clear()
    Fi = B._Refs(F_.pn, G, R, F_.data, F_.tsl, logits, N, W, F_.dev, chunk)
    B._forward_checks(ck, Fi, train=False)


def _peak(ck):
    peak = torch.cuda.max_memory_allocated()
    ck._record("peak_gpu_memory", peak / PEAK_LIMIT, max_memory_allocated=peak)


@pytest.mark.parametrize("N,W", CASES)
def test_every_stage_at_batch_scale(N, W, request):
    case = request.node.callspec.id
    torch.cuda.reset_peak_memory_stats()
    m, F_, ck = B._run_stage_checks(case, N, W, _widths(N, W), dev=DEV, chunk=CHUNK,
                                    ctc=_ctc_long_too if case == "c3" else None, ck=_checker(case))
    _ref_self_check(ck, F_)
    checkers = [ck]
    if case == "c3":
        del m
        for k in B.BWD_TAPS + ("gates_steps", "csave_steps", "conv5", "xproj", "lstm_out"):
            del F_.G[k]
        checkers.append(_checker("c3/inference"))
        _inference_plan_checks(checkers[1], F_, N, W)
    _peak(ck)
    fail = []
    for c in checkers:
        c.report()
        fail += c.fail
    assert not fail, "\n".join(fail)
