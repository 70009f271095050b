"""Every forward and backward stage of the bf16 path in isolation, against an fp64 restatement of that one operation.

Each stage's inputs are its OWN bf16 operands read back from the workspace (crnn_debug_tap / crnn_debug_tap_raw), so the
only legitimate differences from tests/stage_refs.py are the order of the f32 accumulation and the final rounding.  Error
does not compound from layer to layer, and a wrong element fails wherever it sits.  The whole-chain tests
(test_gpu_parity.py, test_gpu_shapes.py, test_gpu_training.py) pin the composition; these pin the kernels.  The shapes
here hold at most 130 images; test_gpu_stage_isolation_batch.py runs the same checks (_run_stage_checks, _forward_checks)
at the batch sizes the project runs, the inference plan included.

Per-element bounds (ratio = |gpu - ref| / bound must be <= 1):
  bf16 outputs:  ulp_bf16(|ref|) + c * acc      (acc: the same operation on |inputs| and |weights|)
  f32 outputs:   c * acc per element, and relative L2 <= 1e-4   (logits, weight / bias gradients)
The recurrence, its isolated steps and the free-running BPTT dz_all (bf16 h / dz exchange, approximate tanh / sigmoid, up
to 63 serial steps) use c * max|ref| of the tensor instead of acc.  Those c, and the c of the f32 outputs, are about 4x the
largest error measured over all shapes below on one H100 80GB HBM3 (SXM): the whole recurrence now holds lstm_out to
6.5e-3 of its max, where the whole-chain test allows 9e-2.  The bf16 stages measured at most 0.5 ulp, the final rounding
alone, so their bound stays at one ulp.  Every BPTT step is also checked on its own operands, the GPU's dz of the next
step among them (bptt_step_o, bptt_step_ijf; stage_refs.bptt_steps_isolated): ulp_bf16(|ref| + allow) + allow + c * acc
per element, where allow holds the kernel's roundings the reference does not restate (an exchanged bf16 partial near a
rounding midpoint, the bf16 dz the carried cell gradient is recovered from, tanh.approx) and c = 2^-19 the f32 arithmetic.
Every run appends the measured maxima to build/stage_isolation_report.jsonl, one line per stage and shape.

Ties: conv1 picks the first maximum on the f32 accumulators, the other pooled training epilogues on the bf16-rounded
values, and the pool3 backward re-derives the pair maximum from bf16-rounded BN outputs; the arg-max checks accept any
position within the bound of the maximum, and the pool3 reference routes by the same bf16 comparison."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_refs as S  # noqa: E402
from stage_check import SHAPES, ulp_bf16, widths_of  # noqa: E402
from stage_check import Checker as _Checker  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FW, BW = "logits/bidirectional_rnn/fw/lstm_cell", "logits/bidirectional_rnn/bw/lstm_cell"

# The per-step BPTT checks (bptt_step_checks): c covers only the f32 arithmetic between the exchange and the bf16 store,
# at most 20 roundings of 2^-24 of acc on any dz (the 8-term sum onto d_out, the cell formulas of lstm_bwd.cuh, and the
# f32 arithmetic behind the stored dz a carry is recovered from), so 2^-19.  On H100 80GB HBM3 (SXM, 700 W) every case of
# test_gpu_stage_isolation*.py, test_gpu_width_edges.py (T = 1 ... 255), test_gpu_training_run.py and
# test_gpu_dp_stages.py needed c = 0 -- the storage ulp and the allowances held every element; the largest ratio at this
# c is 0.988 (c3) -- so 4.5x the measurement would leave the f32 arithmetic no room at all; the analytic value stands
# instead.
BPTT_STEP_C = 2.0 ** -19

# stage -> (ulps of |ref|, c); c multiplies acc (bf16 / f32 outputs) or max|ref| (recurrence, free-running BPTT)
STAGE_BOUNDS = {
    "conv1": (1, 2 ** -15), "conv2": (1, 2 ** -16), "conv3_1": (1, 2 ** -16), "conv3_2": (1, 2 ** -16),
    "a4a_pre": (1, 2 ** -16), "conv4_1": (1, 2 ** -16), "a4b_pre": (1, 2 ** -16), "conv4_2": (1, 2 ** -16),
    "conv5": (1, 2 ** -16), "xproj": (1, 2 ** -16),
    "lstm_out": (1, 6.5e-3), "step_gates": (1, 4e-3), "step_c": (0, 3e-5), "step_h": (1, 4e-3),
    "logits": (0, 1e-6),
    "d_lstm_out": (1, 2 ** -16), "dz_all": (1, 7e-3), "bptt_step_o": (1, BPTT_STEP_C), "bptt_step_ijf": (1, BPTT_STEP_C),
    "d_a5": (1, 2 ** -16), "d_a4b": (1, 2 ** -16),
    "d_pre4b": (1, 2 ** -16), "d_pre4a": (1, 2 ** -16), "d_a3p": (1, 2 ** -16), "d_pre31": (1, 2 ** -16),
    "d_a2": (1, 2 ** -16), "d_a1": (1, 2 ** -16),
    "wgrad": (0, 2.5e-5), "bn41_affine": (0, 2.5e-5),
    # BatchNorm statistics: the f64 sums hold f32 partial sums over 32-row groups (c times sum|x| resp. sum x^2; measured
    # up to 1.9e-7); the f32 mean / invstd / scale / shift are bounded by c times their error scales from
    # stage_refs.bn_stats_stage (measured up to 2.2e-7)
    "bn_sums": (0, 1e-6), "bn_coef": (0, 3e-6),
}
# relative L2 limit of the f32 outputs.  conv4_1's gamma / beta gradients are sums over the bf16-STORED conv4_2 data
# gradient: where the f32 and the fp64 dgrad straddle a bf16 rounding boundary the stored value differs by one ulp, which
# happens to a sizeable share of the elements and leaves up to 3.1e-4 (measured) in these cancelling sums.
L2_LIMIT = {"bn41_affine": 1.2e-3}


def Checker(case):
    return _Checker(case, STAGE_BOUNDS, "stage_isolation_report.jsonl", ulp_bf16, L2_LIMIT)

def argmax_check(ck, stage, am, pre, pooled, c):
    """Pool window bytes: in range; where the pooled output is > 0 and the two largest fp64 window values are separated by
    more than the bf16 bound, the byte is the first fp64 arg-max; otherwise it points at a value within the bound of the max.
    Torch tensors on one device."""
    am = am.long()
    win = pre.shape[-1]
    bad_range = int((am >= win).sum())
    srt = pre.sort(-1).values
    mx, second = srt[..., -1], srt[..., -2]
    bound = ulp_bf16(mx) + c
    first = S.first_argmax(pre)
    chosen = torch.gather(pre, -1, am.clamp_max(win - 1)[..., None])[..., 0]
    live = pooled > 0
    clear = live & (mx - second > bound)
    wrong_clear = int((clear & (am != first)).sum())
    wrong_near = int((live & ~clear & (mx - chosen > bound)).sum())
    ck._record(stage, 0.0 if bad_range + wrong_clear + wrong_near == 0 else float("inf"), out_of_range=bad_range,
               wrong_clear=wrong_clear, wrong_near_tie=wrong_near, live=int(live.sum()))


def _setup(N, W, widths, seed=5, max_label=4):
    from lstm_ctc_ocr_b200 import engine
    from oracle import crnn_oracle as O
    pn = O.randomize_params(O.init_params(3, dtype=np.float32, logits_scale=10.0))
    data, lab, ll, tsl = O.synth_batch(N, W, seed=seed, widths=widths_of(N, W, widths), min_len=1, max_len=max_label)
    m = engine.CrnnModel(device=DEV)
    m.load_params(pn)
    return m, pn, data, lab, ll, tsl


FWD_TAPS = ("conv1", "conv2", "conv3_1", "conv3_2", "a4a_pre", "conv4_1", "a4b_pre", "conv4_2", "conv5", "xproj", "lstm_out")
BWD_TAPS = ("dl_rows", "d_lstm_out", "dz_all", "d_a5", "d_a4b", "d_pre4b", "d_pre4a", "d_a3p", "d_pre32", "d_pre31", "d_a2",
            "d_pre2", "d_a1")
EPS = float(np.float32(1e-3))


def _sum_into(tot, r):
    """Add one image chunk's batch reductions r (name -> tensor) into tot."""
    for k, v in r.items():
        tot[k] = tot[k] + v if k in tot else v


class _Refs:
    """The operands of one checked batch: the GPU's taps (f32 on the GPU, fp64 on `dev` one image chunk at a time), the
    parameters on `dev`, and the image chunks the references are evaluated over."""

    def __init__(self, pn, G, R, data, tsl, logits, N, W, dev, chunk):
        self.pn, self.G, self.data, self.logits, self.dev = pn, G, data, logits, dev
        self.R = {k: v.to(dev) for k, v in R.items()}
        self.N, self.T, self.H2 = N, W // 4 - 1, W // 4
        self.tsl = np.asarray(tsl)
        self.L = torch.as_tensor(S.clamp_lens(tsl, self.T), device=dev)
        self.P = {k: torch.as_tensor(np.asarray(v, np.float64)).to(dev) for k, v in pn.items()}
        self.Wb = {k: S.bf16(v) for k, v in self.P.items() if k.endswith("weights")}
        self.wh = (self.Wb[FW + "/weights"][512:], self.Wb[BW + "/weights"][512:])
        self.parts = [slice(i, min(i + (chunk or N), N)) for i in range(0, N, chunk or N)]

    def g(self, k, s):
        return self.G[k][s].to(self.dev, torch.float64)

    def steps(self, k, s):                     # unpacked saved gates / cell state [2, n, T, ...] of the images s
        return self.G[k][:, s].to(self.dev, torch.float64)

    def x(self, s):
        return torch.as_tensor(self.data[s], dtype=torch.float64, device=self.dev)

    def valid(self, s):                        # [n, H2]: frames t < len
        return torch.arange(self.H2, device=self.dev)[None, :] < self.L[s][:, None]


def _global_parts(p, v, world):
    """One rank's BatchNorm parts p (bn_sums() over its images) plus the other ranks' f64 sums v = [sum x | sum x^2]: the
    parts of the global batch of `world` equal shards.  The injected sums are operands, so their share of the error scale
    is their magnitude."""
    v = v.to(p["sum"].device)
    return dict(sum=p["sum"] + v[:512], sumsq=p["sumsq"] + v[512:], sum_acc=p["sum_acc"] + v[:512].abs(), cnt=p["cnt"] * world)


def _global_bwd_sums(s, v):
    """One rank's BatchNorm backward sums s (bn_bwd_sums() over its images) plus the other ranks' f64 [sum dy | sum dy*xhat]."""
    v = v.to(s["dbeta"].device)
    return dict(dbeta=s["dbeta"] + v[:512], dgamma=s["dgamma"] + v[512:], dbeta_acc=s["dbeta_acc"] + v[:512].abs(),
                dgamma_acc=s["dgamma_acc"] + v[512:].abs())


def _forward_checks(ck, F_, train=True, inject=None):
    """Every forward stage on its own inputs, image chunk by image chunk; the BatchNorm sums and coefficients from the sums
    over all chunks.  train: also the arg-max bytes and the isolated recurrence steps on the saved gates / cell state.
    inject: data parallelism emulated on one device, dict(world=w, fwd=[v41, v42], bwd=[v42, v41]) with the f64 sums the
    other ranks contributed to each exchange; the "stats" tap then holds the global sums and the coefficients are those of
    the global batch.  Returns this rank's BatchNorm partial sums of both layers' pre-activations."""
    P, Wb, T, dev = F_.P, F_.Wb, F_.T, F_.dev
    g, R = F_.g, F_.R
    bn = R["bn"].double()
    bnp = [{}, {}]
    for s in F_.parts:
        lens, Ls = F_.tsl[s], F_.L[s]
        r = S.conv1_stage(F_.x(s), P["conv1/weights"], P["conv1/biases"])
        ck.close("conv1", g("conv1", s), r["out"], r["acc"])
        if train:
            argmax_check(ck, "am1", R["am1"][s], S.windows22(r["pre"]), g("conv1", s), 2 ** -15 * r["acc"])
        r = S.conv_relu_pool22_stage(g("conv1", s), Wb["conv2/weights"], P["conv2/biases"])
        ck.close("conv2", g("conv2", s), r["out"], r["acc"])
        if train:
            argmax_check(ck, "am2", R["am2"][s], S.windows22(r["pre"]), g("conv2", s), 2 ** -16 * r["acc"])
        r = S.conv_relu_stage(g("conv2", s), Wb["conv3_1/weights"], P["conv3_1/biases"])
        ck.close("conv3_1", g("conv3_1", s), r["out"], r["acc"])
        r = S.conv_relu_pool12_stage(g("conv3_1", s), Wb["conv3_2/weights"], P["conv3_2/biases"])
        ck.close("conv3_2", g("conv3_2", s), r["out"], r["acc"])
        if train:
            argmax_check(ck, "am3", R["am3"][s], S.windows12(r["pre"]), g("conv3_2", s), 2 ** -16 * r["acc"])
        del r
        for li, (name, src, pre, out) in enumerate((("conv4_1", "conv3_2", "a4a_pre", "conv4_1"),
                                                    ("conv4_2", "conv4_1", "a4b_pre", "conv4_2"))):
            r = S.conv_bias_stage(g(src, s), Wb[f"{name}/weights"], P[f"{name}/biases"])
            ck.close(pre, g(pre, s), r["out"], r["acc"])
            _sum_into(bnp[li], S.bn_sums(g(pre, s)))
            if li == 0:
                r = S.bn_apply_relu_stage(g(pre, s), bn[0, 0], bn[0, 1])
            else:
                r = S.bn_apply_relu_pool_stage(g(pre, s), bn[1, 0], bn[1, 1])
            ck.close(out, g(out, s), r["out"], r["acc"] * 2 ** -8)        # one f32 fma, then the bf16 rounding: <= 1 ulp
        r = S.conv5_stage(g("conv4_2", s), Wb["conv5/weights"], P["conv5/biases"])
        ck.close("conv5", g("conv5", s)[:, :T], r["out"], r["acc"])
        r = S.xproj_stage(g("conv5", s), Wb[FW + "/weights"][:512], Wb[BW + "/weights"][:512], P[FW + "/biases"],
                          P[BW + "/biases"], lens, T)
        ck.close("xproj", g("xproj", s), r["out"], r["acc"])
        r = S.recurrence_stage(g("xproj", s), F_.wh[0], F_.wh[1], lens, T)
        valid = F_.valid(s)
        ck.exact("lstm_out_past_len_zero", g("lstm_out", s)[~valid], 0.0)
        ck.close_scaled("lstm_out", g("lstm_out", s), r["out"], mask=valid[..., None].expand(r["out"].shape))
        if train:
            gates, csave = F_.steps("gates_steps", s), F_.steps("csave_steps", s)
            iso = S.recurrence_steps_isolated(g("xproj", s), F_.wh[0], F_.wh[1], g("lstm_out", s), csave, lens, T)
            act2 = (torch.arange(T, device=dev)[None, :] < Ls[:, None])[None].expand(2, -1, -1)
            ck.close_scaled("step_gates", gates[act2], iso["gates"][act2])
            ck.close_scaled("step_c", csave[act2], iso["c"][act2])
            ck.close_scaled("step_h", S.step_h(g("lstm_out", s), lens, T)[act2], iso["h"][act2])
        r = S.logits_stage(g("lstm_out", s), Wb["logits/weights"], P["logits/biases"], T)
        lg = F_.logits[:, s].to(dev)
        ck.close("logits", lg, r["out"], r["acc"])
        past = torch.arange(T, device=dev)[:, None] >= Ls[None, :]
        ck.exact("logits_past_len_bias", lg[past], P["logits/biases"].float())
    stats = R["stats"]
    for li, name in enumerate(("conv4_1", "conv4_2")):
        p = bnp[li] if inject is None else _global_parts(bnp[li], inject["fwd"][li], inject["world"])
        st = S.bn_stats_stage(None, P[f"{name}/{name}/gamma"], P[f"{name}/{name}/beta"], EPS, parts=p)
        ck.close(f"{name}_stats", stats[li, 0], st["sum"], st["sum_acc"], key="bn_sums")
        ck.close(f"{name}_stats_sq", stats[li, 1], st["sumsq"], st["sumsq"], key="bn_sums")
        for j, k in enumerate(("scale", "shift", "mean", "invstd")):        # f32 roundings of f64 values of those sums
            ck.close(f"{name}_bn_{k}", bn[li, j], st[k], st["acc"][k], key="bn_coef")
    return bnp


STEP_AXES = ("dir", "row", "step", "gate", "unit")


def bptt_step_checks(ck, d_out, gates, csave, wh, dz_all, lens, T, origin=0):
    """Every BPTT step on its own operands (stage_refs.bptt_steps_isolated): the o column, the i / j / f columns, and dz_f of
    step 0 exactly zero (c_{-1} = 0).  The worst element's coordinates name the unit, whose rank is unit // 32."""
    bs = S.bptt_steps_isolated(d_out, gates, csave, wh[0], wh[1], dz_all, lens, T)
    act = bs["active"][..., None, None]
    o = slice(3, 4)
    kw = dict(axes=STEP_AXES, origin=(0, origin, 0, 0, 0))
    ck.close_allow("bptt_step_o", bs["gpu"][..., o, :], bs["dz"][..., o, :], bs["acc"][..., o, :], bs["allow"][..., o, :],
                   act, near_midpoint_partials=int(bs["near_midpoint"][bs["active"]].sum()), **kw)
    ck.close_allow("bptt_step_ijf", bs["gpu"][..., :3, :], bs["dz"][..., :3, :], bs["acc"][..., :3, :],
                   bs["allow"][..., :3, :], act, carry_recovered=int(bs["recovered"].sum()),
                   carry_fallbacks=int(bs["fallback"].sum()), **kw)
    if T > 0:
        ck.exact("bptt_step0_dzf_zero", bs["gpu"][:, :, 0, 2][bs["active"][:, :, 0]], 0.0)
    return bs


def _backward_checks(ck, F_, grad, dlogits, bnp, inject=None):
    """Every backward stage on its own inputs, image chunk by image chunk, and the 24 gradient tensors from the reference
    sums over all chunks.  The BatchNorm backwards need batch sums of their own input gradient first, so the chunks are
    walked three times: up to d_a4b (+ BN4_2's sums), d_pre4b (+ BN4_1's sums), the rest.  inject (see _forward_checks):
    the statistics and the data gradients of both BatchNorms are the global batch's, gamma / beta gradients this rank's
    own sums (the flat gradient buffer is summed over ranks afterwards).  Returns this rank's BatchNorm backward sums of
    conv4_2 and conv4_1."""
    P, Wb, T, H2 = F_.P, F_.Wb, F_.T, F_.H2
    g, R = F_.g, F_.R
    bn = R["bn"].double()
    if inject is not None:
        bnp = [_global_parts(p, v, inject["world"]) for p, v in zip(bnp, inject["fwd"])]
    glob = (lambda s, i: s) if inject is None else (lambda s, i: _global_bwd_sums(s, inject["bwd"][i]))
    st = [S.bn_batch(None, EPS, parts=p) for p in bnp]
    tot, s42, s41 = {}, {}, {}
    for s in F_.parts:
        lens = F_.tsl[s]
        dl = S.dl_rows_stage(dlogits[:, s].to(F_.dev, torch.float64), H2)
        ck.exact("dl_rows", g("dl_rows", s), S.bf16(dl["dl_rows"]))
        _sum_into(tot, {"logits/biases": dl["dbias"], "logits/biases_acc": dl["dbias_acc"]})
        r = S.logits_bwd(g("lstm_out", s), g("dl_rows", s), Wb["logits/weights"])
        _sum_into(tot, {"logits/weights": r["dw"], "logits/weights_acc": r["dw_acc"]})
        ck.close("d_lstm_out", g("d_lstm_out", s), r["d_lstm_out"], r["d_lstm_out_acc"])
        r = S.bptt_stage(g("d_lstm_out", s), F_.steps("gates_steps", s), F_.steps("csave_steps", s), F_.wh[0], F_.wh[1],
                         lens, T, dz_in=g("dz_all", s))
        valid = F_.valid(s)
        ck.exact("dz_all_past_len_zero", g("dz_all", s)[~valid], 0.0)
        ck.close_scaled("dz_all", g("dz_all", s), r["dz"], mask=valid[..., None].expand(r["dz"].shape))
        bptt_step_checks(ck, g("d_lstm_out", s), F_.steps("gates_steps", s), F_.steps("csave_steps", s), F_.wh,
                         g("dz_all", s), lens, T, origin=s.start)
        r = S.lstm_grads_stage(g("dz_all", s), g("conv5", s), g("lstm_out", s), Wb[FW + "/weights"][:512],
                               Wb[BW + "/weights"][:512], F_.wh[0], F_.wh[1])
        for d, scope in (("fw", FW), ("bw", BW)):
            _sum_into(tot, {scope + k: r[d + k] for k in ("/weights", "/weights_acc", "/biases", "/biases_acc")})
        ck.close("d_a5", g("d_a5", s), r["d_a5"], r["d_a5_acc"])
        r = S.conv5_bwd(g("d_a5", s), g("conv4_2", s), Wb["conv5/weights"])
        _sum_into(tot, {"conv5/weights": r["dw"], "conv5/weights_acc": r["dw_acc"], "conv5/biases": r["db"],
                        "conv5/biases_acc": r["db_acc"]})
        ck.close("d_a4b", g("d_a4b", s), r["dx"], r["dx_acc"])
        dyr = S.bn_relu_pool_route(g("d_a4b", s), g("a4b_pre", s), bn[1])
        _sum_into(s42, S.bn_bwd_sums(dyr, dyr.abs(), g("a4b_pre", s), st[1]))
    ck.close("conv4_2/gamma", grad["conv4_2/conv4_2/gamma"], s42["dgamma"], s42["dgamma_acc"], key="wgrad")
    ck.close("conv4_2/beta", grad["conv4_2/conv4_2/beta"], s42["dbeta"], s42["dbeta_acc"], key="wgrad")
    w42 = Wb["conv4_2/weights"]
    for s in F_.parts:
        r = S.bn_relu_pool_bwd_stage(g("d_a4b", s), g("a4b_pre", s), bn[1], P["conv4_2/conv4_2/gamma"], EPS, stats=st[1],
                                     sums=glob(s42, 0))
        ck.close("d_pre4b", g("d_pre4b", s), r["dx"], r["dx_acc"])
        r = S.conv_bwd(g("d_pre4b", s), g("conv4_1", s), w42)
        _sum_into(tot, {"conv4_2/weights": r["dw"], "conv4_2/weights_acc": r["dw_acc"]})
        d, d_acc = S.conv_relu_dgrad(g("d_pre4b", s), g("a4a_pre", s), bn[0], w42)
        _sum_into(s41, S.bn_bwd_sums(d, d_acc, g("a4a_pre", s), st[0]))
    ck.close("conv4_1/gamma", grad["conv4_1/conv4_1/gamma"], s41["dgamma"], s41["dgamma_acc"], key="bn41_affine")
    ck.close("conv4_1/beta", grad["conv4_1/conv4_1/beta"], s41["dbeta"], s41["dbeta_acc"], key="bn41_affine")
    for s in F_.parts:
        r = S.conv_bn_relu_bwd_stage(g("d_pre4b", s), g("a4a_pre", s), bn[0], P["conv4_1/conv4_1/gamma"], w42, EPS,
                                     stats=st[0], sums=glob(s41, 1))
        ck.close("d_pre4a", g("d_pre4a", s), r["dx"], r["dx_acc"])
        r = S.conv_bwd(g("d_pre4a", s), g("conv3_2", s), Wb["conv4_1/weights"])
        _sum_into(tot, {"conv4_1/weights": r["dw"], "conv4_1/weights_acc": r["dw_acc"]})
        ck.close("d_a3p", g("d_a3p", s), r["dx"], r["dx_acc"])
        ck.exact("d_pre32", g("d_pre32", s), S.unpool_stage(g("d_a3p", s), g("conv3_2", s), R["am3"][s].long(), 2))
        db, dba = S.masked_colsum(g("d_a3p", s), g("conv3_2", s))
        _sum_into(tot, {"conv3_2/biases": db, "conv3_2/biases_acc": dba})
        r = S.conv_bwd(g("d_pre32", s), g("conv3_1", s), Wb["conv3_2/weights"])
        _sum_into(tot, {"conv3_2/weights": r["dw"], "conv3_2/weights_acc": r["dw_acc"]})
        ck.close("d_pre31", g("d_pre31", s), r["dx"] * (g("conv3_1", s) > 0), r["dx_acc"])
        r = S.conv_bwd(g("d_pre31", s), g("conv2", s), Wb["conv3_1/weights"])
        _sum_into(tot, {"conv3_1/weights": r["dw"], "conv3_1/weights_acc": r["dw_acc"], "conv3_1/biases": r["db"],
                        "conv3_1/biases_acc": r["db_acc"]})
        ck.close("d_a2", g("d_a2", s), r["dx"], r["dx_acc"])
        ck.exact("d_pre2", g("d_pre2", s), S.unpool_stage(g("d_a2", s), g("conv2", s), R["am2"][s].long(), 4))
        db, dba = S.masked_colsum(g("d_a2", s), g("conv2", s))
        _sum_into(tot, {"conv2/biases": db, "conv2/biases_acc": dba})
        r = S.conv_bwd(g("d_pre2", s), g("conv1", s), Wb["conv2/weights"])
        _sum_into(tot, {"conv2/weights": r["dw"], "conv2/weights_acc": r["dw_acc"]})
        ck.close("d_a1", g("d_a1", s), r["dx"], r["dx_acc"])
        r = S.conv1_wgrad_stage(g("d_a1", s), g("conv1", s), R["am1"][s].long(), F_.x(s), P["conv1/weights"])
        _sum_into(tot, {"conv1/weights": r["dw"], "conv1/weights_acc": r["dw_acc"], "conv1/biases": r["db"],
                        "conv1/biases_acc": r["db_acc"]})
    for k in [k for k in tot if not k.endswith("_acc")]:                  # a tensor's own bound "wgrad/<name>" if any
        ck.close(k, grad[k], tot[k], tot[k + "_acc"], key=f"wgrad/{k}" if f"wgrad/{k}" in ck.bounds else "wgrad")
    ck.exact("conv4_2/biases_zero", grad["conv4_2/biases"], 0.0)
    ck.exact("conv4_1/biases_zero", grad["conv4_1/biases"], 0.0)
    return s42, s41


def _run_stage_checks(case, N, W, widths, dev="cpu", chunk=None, ctc=None, ck=None, max_label=4, seed=5):
    """The training-mode forward and backward of one batch on a fresh model, every stage checked on its own inputs.  dev:
    where the fp64 references run; chunk: images per reference evaluation (the whole batch by default).  ctc(ck, logits,
    lab, ll, tsl): returns the backward's d logits (default: a seeded random one).  max_label: label lengths are drawn from
    1 .. max_label.  seed: of the synthetic batch.  Returns the model, the operands (_Refs) and the checker (Checker(case)
    unless given), not yet asserted."""
    m, pn, data, lab, ll, tsl = _setup(N, W, widths, seed=seed, max_label=max_label)
    m.set_training(True)
    F_, ck = _check_step(m, pn, (data, lab, ll, tsl), case, dev, chunk, ctc, ck)
    return m, F_, ck


def _check_step(m, pn, batch, case, dev="cpu", chunk=None, ctc=None, ck=None):
    """The training-mode forward and backward of `batch` = (data, lab, ll, tsl) on a model in training mode in whatever state
    it is in (fresh, or parameters written by a solver step), every stage checked on its own inputs.  pn: the model's current
    f32 parameters ({name: array}, e.g. m.tensor(k) read back).  dev, chunk, ctc, ck as in _run_stage_checks.  Returns the
    operands (_Refs) and the checker, not yet asserted."""
    data, lab, ll, tsl = batch
    N, W = data.shape[0], data.shape[1]
    T = W // 4 - 1
    t = lambda a: torch.tensor(a, device=DEV)
    d_data, d_tsl = t(data), t(tsl)
    logits = m.forward(d_data, d_tsl)
    torch.cuda.synchronize()
    G = {k: m.tap(k, N, W) for k in FWD_TAPS}
    G["gates_steps"] = S.unpack_gates(m.tap("gates", N, W), N)
    R = {k: m.tap_raw(k, N, W) for k in ("bn", "stats", "am1", "am2", "am3")}
    G["csave_steps"] = S.unpack_csave(m.tap_raw("csave", N, W), N)
    ck = ck or Checker(case)
    if ctc is None:
        gen = torch.Generator(device="cpu").manual_seed(17)
        dlogits = (torch.randn((T, N, 64), generator=gen) * 0.05).float().to(DEV)
    else:
        dlogits = ctc(ck, logits, lab, ll, tsl)
    m.backward(d_data, d_tsl, dlogits)
    torch.cuda.synchronize()
    for k in BWD_TAPS:
        G[k] = m.tap(k, N, W)
    F_ = _Refs(pn, G, R, data, tsl, logits, N, W, dev, chunk)
    grad = {k: m.grad_tensor(k).to(dev, torch.float64) for k in m.table}
    bnp = _forward_checks(ck, F_)
    _backward_checks(ck, F_, grad, dlogits, bnp)
    return F_, ck


# SHAPES (shared with other modules) and two 128-row tiles of widths 8 .. 100: the LSTM recurrence's 8-CTA clusters exchange h
# over every step of both tiles, and the second tile's upper half has no valid row
STAGE_SHAPES = [pytest.param(*p.values, 5, id=p.id) for p in SHAPES] + [
    pytest.param(200, 100, [int(w) for w in np.random.default_rng(2).integers(8, 101, size=200)], 12, id="N200_W100")]


@pytest.mark.parametrize("N,W,widths,seed", STAGE_SHAPES)
def test_every_stage_against_fp64_on_its_own_inputs(N, W, widths, seed, request):
    _run_stage_checks(request.node.callspec.id, N, W, widths, seed=seed)[2].assert_ok()


@pytest.mark.parametrize("N,W,widths", [SHAPES[0], SHAPES[3], SHAPES[4]])
def test_training_forward_taps_match_inference(N, W, widths):
    """conv1 .. conv3_2 come before any atomics: the training variants (arg-max bytes) must write bit-identical values.
    conv4_1 and conv4_2 may differ by 1 bf16 ulp (order of the f64 atomics of the BatchNorm statistics).  The per-stage
    checks above run on training-mode plans; from conv5 on the kernels are the same in both modes.  The inference plan is
    checked stage by stage at 1024 x 256 in test_gpu_stage_isolation_batch.py, which also repeats this comparison there."""
    m, pn, data, _, _, tsl = _setup(N, W, widths)
    t = lambda a: torch.tensor(a, device=DEV)
    names = ("conv1", "conv2", "conv3_1", "conv3_2", "conv4_1", "conv4_2")
    m.forward(t(data), t(tsl))
    inf = {k: m.tap(k, N, W).cpu().numpy() for k in names}
    m.set_training(True)
    m.forward(t(data), t(tsl))
    trn = {k: m.tap(k, N, W).cpu().numpy() for k in names}
    for k in names[:4]:
        assert np.array_equal(inf[k], trn[k]), k
    for k in names[4:]:
        d = np.abs(inf[k] - trn[k])
        assert (d <= ulp_bf16(np.maximum(np.abs(inf[k]), np.abs(trn[k])))).all(), k


@pytest.mark.parametrize("N,W,widths", [SHAPES[0], pytest.param(8, 64, [64, 4, 8, 33, 64, 61, 12, 40], id="N8_W64")])
def test_chunked_front_end_is_bit_identical(N, W, widths):
    """forward_host(chunks=4) runs conv1 .. conv3_2 per image range (the img0 coordinate of conv1's output map): the front-end
    taps must equal the one-range forward bit for bit."""
    m, pn, data, _, _, tsl = _setup(N, W, widths)
    t = lambda a: torch.tensor(a, device=DEV)
    names = ("conv1", "conv2", "conv3_1", "conv3_2")
    m.forward(t(data), t(tsl))
    one = {k: m.tap(k, N, W).cpu().numpy() for k in names}
    host = torch.empty((N, W, 32), dtype=torch.float32, pin_memory=True)
    host.copy_(torch.as_tensor(data))
    m.forward_host(host.numpy(), t(tsl), chunks=4)
    torch.cuda.synchronize()
    for k in names:
        assert np.array_equal(m.tap(k, N, W).cpu().numpy(), one[k]), k
