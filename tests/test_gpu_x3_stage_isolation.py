"""Every stage of the f32-class forward paths (csrc/forward_x3.cu: compute_dtype 2 "f32" = split-bf16 operands, 3 "tf32"
= tf32 operands) in isolation, against an fp64 restatement of that one operation on its own operands.

Each stage's inputs are the exact operands the kernel consumed, read back byte for byte from the workspace
(crnn_debug_tap_raw): the [hi | lo] bf16 pairs of split mode, the tf32-rounded f32 values of tf32 mode, the f64 BatchNorm
sums and f32 coefficients, the f32 input projection.  Weights are split (`stage_refs.split`) or rounded (`tf32_rna`) the way
the weight kernels produce them.  A split stage's linear part is the split-operand product ah*wh + al*wh + ah*wl in fp64,
so what is left is the f32 accumulation order and the final storage rounding; error does not carry over from layer to
layer.  The whole-chain comparisons with the oracle (tests/test_gpu_x3.py) pin the composition.

Per-element bounds (ratio = |gpu - ref| / bound must be <= 1), acc = the same operation on absolute values:
  stored outputs:  the storage rounding + c * acc.  tf32 mode: half a tf32 ulp, 2^(floor(log2 |ref|) - 11).  Split mode:
                   a quarter of ulp_split = ulp_bf16(|ref|) * 2^-8, which is half an ulp of the lo half.  conv4_x: GEMM +
                   bias + BN apply with the GPU's own scale / shift (+ ReLU, + pool3), acc scaled by |scale|.
  f32 outputs:     c * acc, and relative L2 <= 1e-4 (xproj, logits).
  recurrence:      teacher-forced -- every step's gates from the GPU's own xproj row and its own h_{t-1} (read from
                   lstm_out), the cell state carried in fp64 -- h_t per step (+ the storage rounding) and the final c
                   against c * max|ref|.
  BatchNorm:       the f64 sums against the reference pre-activations of the whole batch (c * sum acc); the f32 coefficients
                   finalized from the workspace's own sums (c * their error scales, stage_refs.bn_stats_stage).
The c of each stage is 4.5x the largest error measured over all cases on one H100 80GB HBM3 (SXM), listed per stage in
MEASURED.  Every run writes its maxima (c_needed per stage and case) to build/x3_stage_isolation_report.jsonl.

Exact checks: lstm_out zero past each length, logits past each length equal to the bias, every stored split activation in
canonical form (|lo| <= ulp_bf16(hi)/2 and hi == bf16(hi + lo), except where lo is exactly that half ulp: the tie of
hi + lo may round either way), every stored tf32 activation with its low 13 mantissa bits zero."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_refs as S  # noqa: E402
from stage_check import SHAPES, Checker, ulp_bf16, ulp_split, ulp_tf32, widths_of  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FW, BW = "logits/bidirectional_rnn/fw/lstm_cell", "logits/bidirectional_rnn/bw/lstm_cell"
MODES = ["f32", "tf32"]
ACTS = ("conv1", "conv2", "conv3_1", "conv3_2", "conv4_1", "conv4_2", "conv5", "lstm_out")

# Largest c each stage needed (the error beyond its storage-ulp share, over acc or max|ref|), over every case of this file
# on one H100 80GB HBM3 (SXM): the c in BOUNDS below is 4.5x these, rounded up.  Re-measure from the report's c_needed.
MEASURED = {
    "f32": {"conv1": 1.01e-7, "conv2": 6.58e-7, "conv3_1": 7.08e-7, "conv3_2": 9.12e-7, "conv4_1": 1.0e-6,
            "conv4_2": 1.97e-6, "conv5": 1.15e-6, "xproj": 1.12e-6, "step_h": 1.28e-6, "cst": 4.82e-7,
            "logits": 9.58e-7, "bn_sums": 1.26e-6, "bn_coef": 2.07e-7},
    "tf32": {"conv1": 6.6e-8, "conv2": 2.63e-7, "conv3_1": 4.64e-7, "conv3_2": 5.2e-7, "conv4_1": 6.53e-7,
             "conv4_2": 1.26e-6, "conv5": 5.67e-7, "xproj": 4.95e-7, "step_h": 3.27e-7, "cst": 3.35e-7,
             "logits": 3.5e-7, "bn_sums": 8.49e-7, "bn_coef": 1.79e-7},
}
# mode -> stage -> (storage ulps, c); c multiplies acc, or max|ref| for the recurrence.  The storage share is the rounding
# alone: round-to-nearest errs by at most half a tf32 ulp, and by half an ulp of lo <= a quarter of ulp_split (|lo| <=
# ulp_bf16/2), so a truncating tf32 store fails the bound (tests/test_stage_refs_cpu.py).
BOUNDS = {
    "f32": {"conv1": (0.25, 4.6e-7), "conv2": (0.25, 3e-6), "conv3_1": (0.25, 3.2e-6), "conv3_2": (0.25, 4.2e-6),
            "conv4_1": (0.25, 4.5e-6), "conv4_2": (0.25, 8.9e-6), "conv5": (0.25, 5.2e-6), "xproj": (0, 5.1e-6),
            "step_h": (0.25, 5.8e-6), "cst": (0, 2.2e-6), "logits": (0, 4.4e-6),
            "bn_sums": (0, 5.7e-6), "bn_coef": (0, 9.4e-7)},
    "tf32": {"conv1": (0.5, 3e-7), "conv2": (0.5, 1.2e-6), "conv3_1": (0.5, 2.1e-6), "conv3_2": (0.5, 2.4e-6),
             "conv4_1": (0.5, 3e-6), "conv4_2": (0.5, 5.7e-6), "conv5": (0.5, 2.6e-6), "xproj": (0, 2.3e-6),
             "step_h": (0.5, 1.5e-6), "cst": (0, 1.6e-6), "logits": (0, 1.6e-6),
             "bn_sums": (0, 3.9e-6), "bn_coef": (0, 8.1e-7)},
}
STORAGE_ULP = {"f32": ulp_split, "tf32": ulp_tf32}

# the benchmarked configuration (BASELINE configs[1]): more tiles than SMs in every conv GEMM.  Its per-image stages are
# checked on a fixed sample of images (both 128-row tiles, their edges); conv4_x and the BatchNorm sums on the whole batch.
BENCH = pytest.param(256, 160, "cycle", id="N256_W160")
BENCH_SAMPLE = [0, 1, 127, 128, 200, 255]


def _params(seed):
    from oracle import crnn_oracle as O
    return O.randomize_params(O.init_params(seed, dtype=np.float32, logits_scale=10.0), seed=seed + 8)


def _model(mode, pn):
    from lstm_ctc_ocr_b200 import engine
    m = engine.CrnnModel(device=DEV, compute_dtype=mode)
    m.load_params(pn)
    return m


def _operand(raw, mode, name):
    """Raw tap -> the operand the next kernel reads: (hi, lo) fp64 pair (split) or the f32 value (tf32), tap shape."""
    if mode == "tf32":
        return raw.double()
    if name == "conv4_2":                                       # [N, H2, (hi, lo), 2 positions, 512]
        return raw[:, :, 0].double(), raw[:, :, 1].double()
    return raw[..., 0, :].double(), raw[..., 1, :].double()


def _weight(mode, w):
    return S.split(w) if mode == "f32" else S.tf32_rna(w)


def _canonical(ck, mode, name, raw):
    if mode == "tf32":
        bits = raw.contiguous().view(torch.int32)
        ck.exact(f"{name}_tf32_rounded", (bits & 0x1FFF).numpy(), 0)
        return
    hi, lo = _operand(raw, mode, name)
    half = ulp_bf16(hi.numpy()) / 2
    ok = np.abs(lo.numpy()) <= half
    ok &= (S.bf16(hi + lo) == hi).numpy() | (np.abs(lo.numpy()) == half)
    ok &= (hi.numpy() != 0) | (lo.numpy() == 0)
    ck.exact(f"{name}_canonical", ok, True)


def _run_stage_checks(case, mode, N, W, widths, m=None, pn=None, seed=5, sample=None):
    from oracle import crnn_oracle as O
    pn = pn if pn is not None else _params(3)
    m = m if m is not None else _model(mode, pn)
    data, lab, ll, tsl = O.synth_batch(N, W, seed=seed, widths=widths_of(N, W, widths), min_len=1, max_len=4)
    T, H2 = W // 4 - 1, W // 4
    t = lambda a: torch.tensor(a, device=DEV)
    logits = m.forward(t(data), t(tsl))
    torch.cuda.synchronize()
    raw = {k: m.tap_raw(k, N, W).cpu() for k in ACTS + ("bn", "stats", "cst")}
    xproj = m.tap("xproj", N, W).double().cpu()
    logits = logits.double().cpu()
    P = {k: torch.as_tensor(np.asarray(v, np.float64)) for k, v in pn.items()}
    Wt = {k: _weight(mode, v) for k, v in P.items() if k.endswith("weights")}
    img = list(range(N)) if sample is None else sample           # images of the per-image stages
    A = {k: _operand(raw[k], mode, k) for k in ACTS}
    Ai = {k: S.pair_map(lambda v: v[img], a) for k, a in A.items()}
    val = lambda k, sel=img: S.pair_value(A[k])[sel]
    eps = float(np.float32(1e-3))
    L = S.clamp_lens(tsl, T)
    Li = [L[n] for n in img]
    ck = Checker(f"{mode}/{case}", BOUNDS[mode], "x3_stage_isolation_report.jsonl", STORAGE_ULP[mode])
    for k in ACTS:
        _canonical(ck, mode, k, raw[k])

    # ---------------------------------------------------------------- conv front end (f32 FMAs, then split / tf32 GEMMs)
    x = torch.as_tensor(data, dtype=torch.float64)[img]
    r = S.conv1_stage(x, P["conv1/weights"], P["conv1/biases"])
    ck.close("conv1", val("conv1"), r["out"], r["acc"])
    r = S.conv_relu_pool22_stage(Ai["conv1"], Wt["conv2/weights"], P["conv2/biases"])
    ck.close("conv2", val("conv2"), r["out"], r["acc"])
    r = S.conv_relu_stage(Ai["conv2"], Wt["conv3_1/weights"], P["conv3_1/biases"])
    ck.close("conv3_1", val("conv3_1"), r["out"], r["acc"])
    r = S.conv_relu_pool12_stage(Ai["conv3_1"], Wt["conv3_2/weights"], P["conv3_2/biases"])
    ck.close("conv3_2", val("conv3_2"), r["out"], r["acc"])

    # ---------------------------------------------------------------- conv4_x: whole batch (batch statistics)
    bn = raw["bn"].double()
    stats = raw["stats"]
    for li, (name, src) in enumerate((("conv4_1", "conv3_2"), ("conv4_2", "conv4_1"))):
        pre = S.conv_bias_stage(A[src], Wt[f"{name}/weights"], P[f"{name}/biases"])
        flat, flat_acc = pre["out"].reshape(-1, 512), pre["acc"].reshape(-1, 512)
        ck.close(f"{name}_stats", stats[li, 0], flat.sum(0), flat_acc.sum(0), key="bn_sums")
        ck.close(f"{name}_stats_sq", stats[li, 1], (flat * flat).sum(0), (2 * flat.abs() * flat_acc).sum(0), key="bn_sums")
        # the coefficients from the workspace's own f64 sums (bn_finalize on its own inputs)
        st = S.bn_stats_stage(pre["out"], P[f"{name}/{name}/gamma"], P[f"{name}/{name}/beta"], eps,
                              sums=(stats[li, 0], stats[li, 1]))
        for j, k in enumerate(("scale", "shift", "mean", "invstd")):
            ck.close(f"{name}_bn_{k}", bn[li, j], st[k], st["acc"][k], key="bn_coef")
        sc, sh = bn[li, 0], bn[li, 1]
        acc = pre["acc"] * sc.abs() + sh.abs()
        if li == 0:
            r = S.bn_apply_relu_stage(pre["out"], sc, sh)
        else:
            r = S.bn_apply_relu_pool_stage(pre["out"], sc, sh, rnd=S.ident)
            acc = S.windows12(acc).max(-1).values
        ck.close(name, S.pair_value(A[name]), r["out"], acc)

    # ---------------------------------------------------------------- conv5, input projection, recurrence, logits
    r = S.conv5_stage(Ai["conv4_2"], Wt["conv5/weights"], P["conv5/biases"])
    ck.close("conv5", val("conv5")[:, :T], r["out"], r["acc"])
    # the [768, 1024] cell weights: rows 0..511 W_x, rows 512..767 W_h
    wx = tuple(S.pair_map(lambda v: v[:512], Wt[s + "/weights"]) for s in (FW, BW))
    wh = tuple(S.pair_map(lambda v: v[512:], Wt[s + "/weights"]) for s in (FW, BW))
    r = S.xproj_stage(Ai["conv5"], wx[0], wx[1], None, None, tsl, T, x3=True)
    ck.close("xproj", xproj[img], r["out"], r["acc"])
    iso = S.recurrence_steps_isolated(xproj[img], wh[0], wh[1], Ai["lstm_out"], None, Li, T,
                                      biases=(P[FW + "/biases"], P[BW + "/biases"]))
    lo_val = val("lstm_out")
    act = (torch.arange(T)[None, :] < torch.as_tensor(Li)[:, None]).numpy()
    act2 = np.broadcast_to(act[None], (2, len(img), T))
    h_gpu = torch.zeros_like(iso["h"])
    for d in range(2):
        for i in range(len(img)):
            for s in range(Li[i]):
                h_gpu[d, i, s] = lo_val[i, (Li[i] - 1 - s) if d else s, d * 256:(d + 1) * 256]
    ck.close_scaled("step_h", h_gpu.numpy()[act2], iso["h"].numpy()[act2])
    c_ref = torch.zeros((2, len(img), 256), dtype=torch.float64)
    for i in range(len(img)):
        if Li[i] > 0:
            c_ref[:, i] = iso["c"][:, i, Li[i] - 1]
    ck.close_scaled("cst", raw["cst"][:, img].double(), c_ref)
    valid = np.zeros((N, H2), bool)
    for n in range(N):
        valid[n, :L[n]] = True
    lo_raw = raw["lstm_out"].view(torch.int16 if mode == "f32" else torch.int32).numpy()
    ck.exact("lstm_out_past_len_zero", lo_raw[~valid], 0)
    r = S.logits_stage(Ai["lstm_out"], Wt["logits/weights"], P["logits/biases"], T)
    ck.close("logits", logits[:, img], r["out"], r["acc"])
    past = np.zeros((T, N), bool)
    for n in range(N):
        past[L[n]:, n] = True
    ck.exact("logits_past_len_bias", logits.numpy()[past], np.broadcast_to(np.float32(pn["logits/biases"]), (int(past.sum()), 64)))
    ck.assert_ok()
    return m


@pytest.mark.parametrize("N,W,widths", SHAPES + [BENCH])
@pytest.mark.parametrize("mode", MODES)
def test_every_x3_stage_against_fp64_on_its_own_operands(mode, N, W, widths, request):
    _run_stage_checks(request.node.callspec.id, mode, N, W, widths, sample=BENCH_SAMPLE if N == 256 else None)


@pytest.mark.parametrize("mode", MODES)
def test_weight_reload_rebuilds_the_operand_cache(mode):
    """The split / tf32 weight cache is rebuilt only when load_params marks it dirty: after a forward with one parameter
    set, a second set loaded into the same model must pass every stage check against the NEW weights."""
    m = _model(mode, _params(3))
    m.forward(torch.zeros((3, 100, 32), device=DEV), torch.tensor([100, 4, 61], dtype=torch.int32, device=DEV))
    pn = _params(7)
    m.load_params(pn)
    _run_stage_checks("reload_N3_W100", mode, 3, 100, [100, 4, 61], m=m, pn=pn)


@pytest.mark.parametrize("mode", MODES)
def test_plan_reuse_across_shapes(mode):
    """One model across shapes: build_plan re-lays out the workspace and rebuilds every activation tensor map; each shape
    must pass every stage check, including the return to the first shape."""
    pn = _params(3)
    m = _model(mode, pn)
    for i, (N, W, widths) in enumerate(((3, 100, [100, 4, 61]), (5, 24, [24, 4, 8, 12, 20]), (3, 100, [100, 4, 61]))):
        _run_stage_checks(f"reuse{i}_N{N}_W{W}", mode, N, W, widths, m=m, pn=pn, seed=5 + i)


@pytest.mark.parametrize("mode", MODES)
def test_taps_the_x3_path_does_not_have_fail(mode):
    from lstm_ctc_ocr_b200._lib import CrnnError
    m = _model(mode, _params(3))
    N, W = 2, 24
    m.forward(torch.zeros((N, W, 32), device=DEV), torch.tensor([24, 8], dtype=torch.int32, device=DEV))
    for k in ("am1", "am2", "am3", "csave", "dz_all", "nonsense"):
        with pytest.raises(CrnnError):
            m.tap_raw(k, N, W)
    for k in ("a4a_pre", "a4b_pre", "gates", "dl_rows", "d_a1"):
        with pytest.raises(CrnnError):
            m.tap(k, N, W)
