"""The fp8 forward (compute_dtype 4) checked per element wherever evaluation runs it.  Need the GPU.

tests/test_gpu_fp8.py checks every fp8 stage at W = 24 .. 256 and at C3.  Evaluation meets more than that: one line at a time
at that line's own width (W = 8 .. about 1000, T = 1 .. 250), packed batches of lines with per-line BatchNorm, shape changes on
every line, and weight reloads.  Code reached only there:
  - T = 1 in conv5's row-shift GEMM; H2 = 129 / 256 (the un-merged 4-box e4m3 tensor maps at large W); two LSTM row tiles
    at H2 = 256; the e4m3 pooled-store shuffle at every row alignment;
  - the LINES branches of the e4m3 producers (conv2_swap_kernel, frag_epilogue EPI_RELU / EPI_RELU_POOL12 / EPI_STATS,
    bn_apply_e4m3_kernel), the per-line statistics slots and coefficients;
  - a second wave of persistent tiles (1160 x 160);
  - the state an fp8 model keeps across calls: the e4m3 weight copies, colscale, the calibrated scales and the seven e4m3
    tensor maps rebuilt with the plan.
Every case runs tests/test_gpu_fp8.py's stage check (_stage_checks), or its packed counterpart below, over chunks of
128 * 256 / W images: the e4m3 producers within half an e4m3 ulp + c * acc and exactly 448 past the range, conv4_x and conv5
within half a bf16 ulp + c * acc, the BatchNorm applies exactly the e4m3 rounding of the f32 fma, the f64 statistics and f32
coefficients, and the stages after conv5 (the bf16 path's kernels, with its bounds; test_gpu_width_edges.LONG at T > 63).

Packed lines (test_gpu_packed_eval.SHAPES): each fp8 GEMM is restated over the packed taps.  Past each line the taps are zero,
so an ordinary SAME convolution of the packed tensor is each line's own zero-padded convolution at h < W_i / 4; the line mask
is then applied to the reference (tests/test_fp8_cpu.py shows this equals each line fed alone, and fails without the mask).

Measured on an H100 80GB HBM3 (SXM, 700 W power limit), largest c_needed over every case of this file, against the bound
each keeps (tests/test_gpu_fp8.py's, 4.5x its measurement at W <= 256, for the fp8 stages; the bf16 path's for the rest):
  conv2 9.23e-8 (W1024; 2.6e-8 at W <= 256) of 1.17e-7    conv3_1 1.35e-4 of 6.9e-4     conv3_2 1.60e-4 of 5.9e-4
  conv4_1 3.0e-4 of 1.3e-3                               conv4_2 4.51e-4 of 2.0e-3     conv5 3.43e-4 (two_waves) of 1.3e-3
  BatchNorm sums 1.6e-7 of 1e-6, coefficients 8.6e-7 of 3e-6, xproj 7.8e-8 of 1.5e-5, lstm_out 3.8e-4 of 6.5e-3,
  step_h 3.8e-6 of 4e-3, logits 2.3e-7 of 1e-6 (c * acc; the recurrence c * max|ref|)
Every stage holds at W = 1024 within the bound set at W <= 256, so no stage gets a wider one here.  Packed lines: every byte
of conv1 .. conv3_2 equals the line-alone run's and every conv4_x value is within one ulp (measured: all equal).  One line
at a time, the fp8 engine decodes all 67 evaluation lines as the bf16 engine does, greedy and beam (MEASURED_AGREEMENT, the
floor asserted).  Peak GPU memory: 4.70 GB at two_waves, 4.67 GB at W1024, against test_gpu_stage_isolation_batch.PEAK_LIMIT.
The inference plan keeps no cell state, so the recurrence's c is checked through h (tail_checks in tests/test_gpu_fp8.py).
Rows go to build/fp8_edges_report.jsonl."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_refs as S  # noqa: E402
import test_gpu_fp8 as F8  # noqa: E402
import test_gpu_packed_eval as PE  # noqa: E402
import test_gpu_stage_isolation as B  # noqa: E402
import test_gpu_stage_isolation_batch as BB  # noqa: E402
import test_gpu_width_edges as WE  # noqa: E402
from stage_check import Checker, ulp_bf16  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = F8.DEV
REPORT = "fp8_edges_report.jsonl"
# greedy / beam decodes of the 67 evaluation lines equal to the bf16 engine's, on an H100 80GB HBM3: the floor asserted
MEASURED_AGREEMENT = {"greedy": 67, "beam": 67}


def _long(W):
    return WE.LONG if W // 4 - 1 > 63 else None


# ------------------------------------------------------------------------------------------------ B. widths evaluation feeds
WIDTH_CASES = [pytest.param(p.values[0], p.values[1], None, id=p.id) for p in WE.CASES] + [
    pytest.param(2, 1024, [1024, 516], id="N2_W1024")]


@pytest.mark.parametrize("N,W,widths", WIDTH_CASES)
def test_fp8_stages_at_edge_widths(N, W, widths, request):
    """Every tile starts with lengths T, 1, 0 (test_gpu_width_edges._widths); each case calibrated on its own batch."""
    torch.cuda.reset_peak_memory_stats()
    F8._stage_checks(request.node.callspec.id, N, W, widths or WE._widths(N, W), chunk=WE._chunk(W), report=REPORT,
                     extra_bounds=_long(W), peak=True)


# ------------------------------------------------------------------------------------------------ C. batch scale
TWO_WAVES_SAMPLE = [0, 1, 2, 127, 128, 1023, 1024, 1151, 1152, 1153, 1159]


def test_fp8_stages_two_waves():
    """1160 x 160: ten LSTM row tiles (the last holding 8 rows) and a second wave of persistent GEMM tiles.  The per-image
    stages on images straddling the tile and wave boundaries, conv4_x and the BatchNorms on the whole batch."""
    torch.cuda.reset_peak_memory_stats()
    F8._stage_checks("two_waves", 1160, 160, BB._widths(1160, 160), sample=TWO_WAVES_SAMPLE, chunk=BB.CHUNK, report=REPORT,
                     peak=True)


# ------------------------------------------------------------------------------------------------ D. packed lines
def _line_mask(lw, idx, H, W, dims):
    """[n, H, 1, ...] True at positions inside their line (h < W_i * H / W) for the lines idx."""
    lim = torch.as_tensor(np.asarray(lw)[idx], device=DEV)[:, None] * H // W
    return (torch.arange(H, device=DEV)[None, :] < lim).view(len(idx), H, *([1] * (dims - 2)))


@pytest.mark.parametrize("shape", list(PE.SHAPES))
def test_fp8_every_stage_per_line(shape):
    """crnn_forward_lines on an fp8 model, every stage per line: masked bytes exactly zero, the fp8 GEMMs per element on the
    packed taps (reference masked by line), per-line statistics and coefficients against fp64 (count W_i), the per-line
    BatchNorm applies exactly, the tail stages, and each line against its own line-alone fp8 run with the same scales."""
    W, lw, data, tsl = PE._shape_lines(shape)
    N, T, H2 = len(lw), W // 4 - 1, W // 4
    pn = F8._params(3)
    m = F8._model(pn)
    d = F8._t
    m.calibrate_fp8(d(data), d(tsl))
    logits = m.forward_lines(d(data), d(lw), d(tsl))
    torch.cuda.synchronize()
    scales = m.tap_raw("fp8_scales", N, W).double()
    raw = {k: m.tap_raw(k, N, W) for k in F8.FP8_ACTS}
    stats = m.tap_raw("stats", N, W, lines=True)
    bn = m.tap_raw("bn", N, W, lines=True).double()
    G = {k: m.tap(k, N, W) for k in ("conv1", "a4a_pre", "a4b_pre", "conv5", "xproj", "lstm_out")}
    Wq, _, _ = F8._weights(m, N, W)
    P = {k: torch.as_tensor(np.asarray(v, np.float64), device=DEV) for k, v in pn.items()}
    ck8 = Checker(f"fp8_packed/{shape}", F8.BOUNDS, REPORT, F8.ulp_e4m3)
    ckb = Checker(f"fp8_packed_bf16/{shape}", dict(F8.BF16_BOUNDS, **(_long(W) or {})), REPORT, ulp_bf16)
    every = list(range(N))
    sample = every if N <= 130 else list(range(8)) + [int(v) for v in np.random.default_rng(1).choice(np.arange(8, N), 56,
                                                                                                       replace=False)]
    n = WE._chunk(W)
    parts = lambda idx: [idx[i:i + n] for i in range(0, len(idx), n)]  # noqa: E731
    q = lambda k, s: F8.decode(raw[k][s])                                # noqa: E731
    val = lambda k, s: q(k, s) * scales[F8.FP8_ACTS.index(k)]           # noqa: E731

    # masks: every stored byte / bf16 value at h >= W_i / 4 is exactly zero (conv1 at its own resolution)
    for k, t in list(raw.items()) + [(k, G[k].view(torch.int32)) for k in ("conv1", "a4a_pre", "a4b_pre")]:
        out = ~_line_mask(lw, every, t.shape[1], W, t.dim()).expand(t.shape)
        ck8.exact(f"masked_zero_{k}", t[out], 0)

    # the fp8 GEMMs and BatchNorm applies per element, each reference masked by line
    sat = {}
    for s in parts(sample):
        keep = _line_mask(lw, s, H2, W, 4).double()
        r = S.conv_relu_pool22_stage(G["conv1"][s].double(), S.bf16(P["conv2/weights"]), P["conv2/biases"])
        F8.e4m3_stage(ck8, sat, "conv2", q("conv2", s), r["out"] * keep, r["acc"], scales[0])
        r = S.conv_relu_stage(val("conv2", s), Wq["conv3_1"], P["conv3_1/biases"])
        F8.e4m3_stage(ck8, sat, "conv3_1", q("conv3_1", s), r["out"] * keep, r["acc"], scales[1])
        r = S.conv_relu_pool12_stage(val("conv3_1", s), Wq["conv3_2"], P["conv3_2/biases"])
        F8.e4m3_stage(ck8, sat, "conv3_2", q("conv3_2", s), r["out"] * keep, r["acc"], scales[2])
        for l, (k, src, pre) in enumerate((("conv4_1", "conv3_2", "a4a_pre"), ("conv4_2", "conv4_1", "a4b_pre"))):
            x = G[pre][s].double()
            r = S.conv_bias_stage(val(src, s), Wq[k], P[k + "/biases"])
            ckb.close(k, x, r["out"] * keep, r["acc"])
            # each line's own coefficients: e4m3 of the f32 fma, exactly, and zero past the line
            want, _ = F8.bn_apply_want(x, bn[l][s][:, 0, None, None, :], bn[l][s][:, 1, None, None, :], scales[3 + l], l == 1)
            ck8.exact(f"bn_apply_{k}", q(k, s), want * keep)
        r = S.conv5_stage(val("conv4_2", s), Wq["conv5"], P["conv5/biases"])
        ckb.close("conv5", G["conv5"][s][:, :T], r["out"], r["acc"])
        del r, x, want
    F8.tail_checks(ckb, P, G, logits, tsl, T, parts(sample))

    # per-line statistics against fp64 sums of each line's own pre-BN values; coefficients the fp64 finalize with count W_i
    for l, (k, pre) in enumerate((("conv4_1", "a4a_pre"), ("conv4_2", "a4b_pre"))):
        p = {"sum": [], "sumsq": [], "sum_acc": []}
        for s in parts(every):
            x = G[pre][s].double()
            p["sum"].append(x.sum((1, 2)))
            p["sumsq"].append((x * x).sum((1, 2)))
            p["sum_acc"].append(x.abs().sum((1, 2)))
        p = {a: torch.cat(v) for a, v in p.items()}
        p["cnt"] = torch.as_tensor(lw, device=DEV, dtype=torch.float64)[:, None]
        gamma, beta = P[f"{k}/{k}/gamma"], P[f"{k}/{k}/beta"]
        st = S.bn_stats_stage(None, gamma, beta, B.EPS, parts=p)
        ckb.close(f"{k}_stats", stats[l, :, 0], st["sum"], st["sum_acc"], key="bn_sums")
        ckb.close(f"{k}_stats_sq", stats[l, :, 1], st["sumsq"], st["sumsq"], key="bn_sums")
        st = S.bn_stats_stage(None, gamma, beta, B.EPS, sums=(stats[l, :, 0], stats[l, :, 1]), parts=p)
        for j, c in enumerate(("scale", "shift", "mean", "invstd")):
            ckb.close(f"{k}_bn_{c}", bn[l, :, j], st[c], st["acc"][c], key="bn_coef")

    # each line against its own line-alone fp8 run with the same scales: the front end bit for bit (it does not depend on
    # other lines), the bf16 pre-BN values within one bf16 ulp (the order of the f64 statistics atomics), their e4m3 BatchNorm
    # outputs within one e4m3 ulp
    exact_k = ("conv1", "conv2", "conv3_1", "conv3_2")
    mism = {k: 0 for k in exact_k + ("a4a_pre", "a4b_pre", "conv4_1", "conv4_2")}
    for i in sample:
        w = int(lw[i])
        m.forward(d(np.ascontiguousarray(data[i:i + 1, :w])), d(tsl[i:i + 1]))
        for k in mism:
            bf = k in ("conv1", "a4a_pre", "a4b_pre")
            a = (m.tap(k, 1, w) if bf else m.tap_raw(k, 1, w))[0]
            p = (G[k] if bf else raw[k])[i, :a.shape[0]]
            if k in exact_k:
                mism[k] += int(not torch.equal(a, p))
            elif bf:
                mism[k] += int(bool(((a.double() - p.double()).abs() > ulp_bf16(torch.maximum(a.abs(), p.abs()).double())).any()))
            else:
                a, p = F8.decode(a), F8.decode(p)
                mism[k] += int(bool(((a - p).abs() > F8.ulp_e4m3(torch.maximum(a.abs(), p.abs()))).any()))
    ck8._record("line_alone", 0.0 if not any(mism.values()) else float("inf"), lines=len(sample), **mism)
    fail = []
    for c in (ck8, ckb):
        c.report()
        fail += c.fail
    assert not fail, "\n".join(fail)


# ------------------------------------------------------------------------------------------------ E. state changes
def test_fp8_weight_reload_requantises():
    """A forward with one parameter set, then load_params of another: the forward is refused until recalibration; after it the
    e4m3 weights and scales are bit for bit the restatement of the NEW weights, and every stage passes against them."""
    from lstm_ctc_ocr_b200._lib import CrnnError
    from oracle import crnn_oracle as O
    m = F8._model(F8._params(3))
    data, _, _, tsl = O.synth_batch(3, 100, seed=2, widths=[100, 4, 61], min_len=1, max_len=3)
    m.calibrate_fp8(F8._t(data), F8._t(tsl))
    m.forward(F8._t(data), F8._t(tsl))
    old = m.tap_raw("fp8_w_conv4_2", 3, 100).clone()
    pn = F8._params(7)
    m.load_params(pn)
    with pytest.raises(CrnnError, match="calibration"):
        m.forward(F8._t(data), F8._t(tsl))
    F8._stage_checks("reload_N3_W100", 3, 100, [100, 4, 61], m=m, pn=pn, report=REPORT)
    assert not torch.equal(m.tap_raw("fp8_w_conv4_2", 3, 100), old)


@pytest.mark.parametrize("seq", [
    pytest.param(((3, 100, [100, 4, 61]), (5, 24, [24, 4, 8, 12, 20]), (3, 100, [100, 4, 61])), id="N3_W100-N5_W24"),
    pytest.param(((1, 1024, [1024]), (1, 8, [8]), (1, 1024, [1024])), id="N1_W1024-N1_W8"),
])
def test_fp8_plan_reuse_across_shapes(seq, request):
    """One model across shapes (the plan, its e4m3 tensor maps and the scales rebuilt at every step): every stage passes at
    every step, and the return to a shape gives the bits of its first visit."""
    pn = F8._params(3)
    m = F8._model(pn)
    ck = Checker(f"reuse/{request.node.callspec.id}", {}, REPORT)
    first = {}
    for i, (N, W, widths) in enumerate(seq):
        _, bits = F8._stage_checks(f"reuse{i}_N{N}_W{W}", N, W, widths, m=m, pn=pn, report=REPORT, chunk=WE._chunk(W),
                                   extra_bounds=_long(W))
        if (N, W) in first:
            for k, v in bits.items():
                ck.exact(f"return_N{N}_W{W}_{k}_bits", v.contiguous().view(torch.uint8), first[(N, W)][k])
        else:
            first[(N, W)] = {k: v.contiguous().view(torch.uint8).clone() for k, v in bits.items()}
    ck.assert_ok()


# ------------------------------------------------------------------------------------------------ F. one line at a time
def test_fp8_evaluation_one_line_at_a_time(monkeypatch):
    """Session.run(dense_decoded), one line per call, TEST.COMPUTE_DTYPE "fp8" (Session.assign calibrates), trained weights,
    over test_gpu_width_edges._eval_inputs (64 lines of W 396 - 944 and crops W = 8, 12, 12), greedy and beam: every decode
    equals the decode of the GPU's own logits (greedy: the oracle's greedy_decode; beam: the host decoder).  Agreement with the
    bf16 engine's decodes is reported and asserted at its measured floor."""
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.session import Session
    from oracle import crnn_oracle as O
    mk = WE._load("make_decode10k", "tests", "golden", "make_decode10k.py")
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    weights = mk.load_weights()
    inputs = WE._eval_inputs()
    ck = Checker("fp8_evaluation", {}, REPORT)
    dec = {}
    old = cfg.get("DECODER", "greedy")
    try:
        for dt in ("bf16", "fp8"):
            monkeypatch.setitem(cfg.TEST, "COMPUTE_DTYPE", dt)
            net = get_network("LSTM_test")
            f_logits, f_dense = Fetch(net, "logits"), Fetch(net, "dense_decoded")
            with Session(device=DEV) as sess:
                sess.assign(net, weights)
                eng = sess.engine_for(net)
                assert eng.compute_dtype == (4 if dt == "fp8" else 1)
                for decoder in ("greedy", "beam"):
                    cfg.DECODER = decoder
                    got_all, own_equal = [], 0
                    for data, tsl in inputs:
                        logits, dense = sess.run([f_logits, f_dense], feed_dict={net.data: data, net.time_step_len: tsl,
                                                                                 net.keep_prob: 1.0})
                        got = [int(v) for v in dense[0] if v != 0] if dense.size else []
                        if decoder == "greedy":
                            own = O.greedy_decode(logits, tsl)[0]
                        else:
                            hb, hbl, _ = engine.ctc_beam_search(logits, tsl, beam_width=100, merge_repeated=True)
                            own = [int(v) for v in hb[0, :hbl[0]] if v != 0]
                        own_equal += int(got == own)
                        got_all.append(got)
                    dec[(dt, decoder)] = got_all
                    ck._record(f"{dt}_{decoder}_own_decode", 0.0 if own_equal == len(inputs) else float("inf"),
                               lines=len(inputs), own_decode_equal=own_equal)
    finally:
        cfg.DECODER = old
    for decoder in ("greedy", "beam"):
        agree = sum(a == b for a, b in zip(dec[("fp8", decoder)], dec[("bf16", decoder)]))
        ck._record(f"fp8_equals_bf16_{decoder}", 0.0 if agree >= MEASURED_AGREEMENT[decoder] else float("inf"),
                   lines=len(inputs), agree=agree, floor=MEASURED_AGREEMENT[decoder])
    ck.assert_ok()
