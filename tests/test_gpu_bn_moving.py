"""Moving BatchNorm statistics on the GPU (include/crnn_ctc.h: crnn_model_bind_bn_moving, crnn_model_set_bn_statistics).

1. Tracking: a multi-step training run per solver over batch shapes that change as BucketSampler changes them.  After every
   step the moving buffer equals, bit for bit, the fp64 update (tests/bn_moving_refs.ema_update) of the f64 sums that step's
   forward normalised with (the "stats" tap), rounded once; a validation forward (training mode, no backward) leaves it
   unchanged; the loss equals bit for bit that of a model whose buffer is unbound, and the gradients agree to the rounding of
   their f32 atomics (which differs from run to run with or without tracking).
2. Data parallelism emulated on one GPU (test_gpu_dp_stages._Rank): the other rank's sums injected through the all-reduce
   callback and through peer memory; the update uses the global sums over count x world.
3. The fold: the bf16 W', the f32 b' and the fp8 colscale' equal the fp64 fold rounded once, exactly.
4. Every moving-mode stage per element against fp64 on its own operands: conv4_1 (EPI_RELU) and conv4_2 (EPI_RELU_POOL12)
   with the folded operands at Cout = 512 (two N tiles), bf16 and e4m3 outputs, and everything downstream, with the bounds
   conv3_1 / conv3_2 and the fp8 epilogues already hold (test_gpu_stage_isolation.STAGE_BOUNDS, test_gpu_fp8.BOUNDS).
5. Batch independence: an image's logits from a batch equal those of the same padded image alone; forward_lines equals each
   line alone.  Bit for bit: every row of every GEMM and recurrence tile is computed from that row's operands alone, in the
   same order, and nothing is reduced over the batch any more.
6. End to end through Session.run with cfg.TEST.BN_STATS = "moving".
7. Status codes, with the outputs untouched.

Workspaces and outputs are filled with NaN (0xFF bytes) before use, as in test_gpu_training_run.py."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bn_moving_refs as M  # noqa: E402
import stage_refs as S  # noqa: E402
import test_gpu_dp_stages as DS  # noqa: E402
import test_gpu_fp8 as G8  # noqa: E402
import test_gpu_stage_isolation as B  # noqa: E402
from stage_check import SHAPES, Checker, ulp_bf16, widths_of  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REPORT = "bn_moving_report.jsonl"
LR = {"Adam": 1e-3, "Momentum": 2e-2, "RMS": 3e-2}
RUN = [(130, 40, "cycle"), (5, 80, [80, 4, 8, 57, 33]), (3, 80, [80, 57, 12]), (3, 160, [160, 8, 97]), (130, 40, "cycle")]


def _t(a):
    return torch.tensor(a, device=DEV)


def _params(seed=3):
    from oracle import crnn_oracle as O
    return O.randomize_params(O.init_params(seed, dtype=np.float32, logits_scale=10.0))


def _moving(seed=7):
    """Moving statistics of the right order for the test weights, and gamma of mixed sign (set in _model)."""
    rng = np.random.default_rng(seed)
    mv = np.empty((2, 2, 512), np.float32)
    mv[:, 0] = rng.normal(0.0, 0.05, (2, 512))
    mv[:, 1] = rng.uniform(0.002, 0.02, (2, 512))
    return mv


def _with_negative_gamma(pn):
    p = dict(pn)
    for k in M.LAYERS:
        g = p[f"{k}/{k}/gamma"].copy()
        g[1::4] = -g[1::4]
        p[f"{k}/{k}/gamma"] = g
    return p


def _state(mv):
    from lstm_ctc_ocr_b200 import engine
    return {k: mv[i // 2, i % 2] for i, k in enumerate(engine.BN_MOVING_KEYS)}


def _model(pn, mv=None, dtype="bf16"):
    from lstm_ctc_ocr_b200 import engine
    m = engine.CrnnModel(device=DEV, compute_dtype=dtype)
    m.load_params(pn)
    if mv is not None:
        m.load_bn_moving(_state(mv))
        m.set_bn_statistics("moving")
    return m


def _nan_ws(m, N, W, lines=False):
    m._workspace(N, W, lines=lines)
    m._ws.fill_(255)


def _nan(shape, dtype=torch.float32):
    return torch.full(shape, 255, dtype=torch.uint8, device=DEV).view(dtype) if dtype == torch.uint8 else \
        torch.empty(shape, dtype=dtype, device=DEV).view(torch.uint8).fill_(255).view(dtype)


def _forward(m, data, tsl, lines=None):
    N, W = data.shape[:2]
    _nan_ws(m, N, W, lines=lines is not None)
    out = _nan((W // 4 - 1, N, 64))
    if lines is None:
        return m.forward(_t(data), _t(tsl), out=out)
    return m.forward_lines(_t(data), _t(lines), _t(tsl), out=out)


# ------------------------------------------------------------------------------------------------ 1. tracking
@pytest.mark.parametrize("solver", ["Adam", "Momentum", "RMS"])
def test_training_tracks_moving_statistics_bit_for_bit(solver):
    from lstm_ctc_ocr_b200 import engine
    from oracle import crnn_oracle as O
    pn = _params()
    a, b = _model(pn), _model(pn)
    engine.check(b.lib.crnn_model_bind_bn_moving(b.handle, None, 0.999))        # b does not track
    for m in (a, b):
        m.set_solver(solver)
        m.set_training(True)
    want = M.initial()
    assert np.array_equal(a.bn_moving.cpu().numpy(), want)
    for step, (N, W, widths) in enumerate(RUN):
        data, lab, ll, tsl = O.synth_batch(N, W, seed=step + 11, widths=widths_of(N, W, widths), min_len=1, max_len=4)
        res = []
        for m in (a, b):
            logits = _forward(m, data, tsl)
            stats = m.tap_raw("stats", N, W).cpu().numpy() if m is a else None
            costs, grad = engine.ctc_loss(logits, _t(lab), _t(ll), _t(tsl), want_grad=True, grad_scale=1.0 / N,
                                          max_label_len=int(ll.max()))
            loss = m.total_loss(costs)
            m.backward(_t(data), _t(tsl), grad)
            m.apply_gradients(LR[solver], step + 1)
            torch.cuda.synchronize()
            res.append((loss.clone(), m.grads.clone(), m.params.clone(), stats))
        (la, ga, pa, stats), (lb, gb, pb, _) = res
        # the forward and the loss are bit-identical; the weight gradients are sums of f32 atomics whose order differs from run
        # to run (test_gpu_training_run.py), so they agree to the rounding of those sums, and b continues from a's state
        assert torch.equal(la, lb), f"step {step}: tracking changed the loss"
        rel = float(torch.linalg.vector_norm(ga - gb) / torch.linalg.vector_norm(ga))
        assert rel <= 1e-5, f"step {step}: gradients differ by {rel:.3g} (relative L2)"
        b.params.copy_(a.params)
        b.adam_m.copy_(a.adam_m)
        b.adam_v.copy_(a.adam_v)
        engine.check(b.lib.crnn_model_params_changed(b.handle))
        want = M.ema_update(want, stats, N * (W // 4) * 4)
        got = a.bn_moving.cpu().numpy()
        assert np.array_equal(got, want), f"step {step}: {int((got != want).sum())} moving values differ"
        # a validation forward on the training-mode model (SolverWrapper._validate) does not move the statistics
        vd, _, _, vt = O.synth_batch(4, 64, seed=99, widths=[64, 40, 12, 64])
        _forward(a, vd, vt)
        torch.cuda.synchronize()
        assert np.array_equal(a.bn_moving.cpu().numpy(), want), f"step {step}: a forward without backward moved them"
    assert not np.array_equal(want, M.initial())


# ------------------------------------------------------------------------------------------------ 2. data parallelism
@pytest.mark.parametrize("peer", [False, True], ids=["callback", "peer"])
def test_data_parallel_update_uses_the_global_sums(peer):
    from oracle import crnn_oracle as O
    world, N, W = 2, 5, 80
    m = _model(_params())
    m.set_training(True)
    rk = DS._Rank(m, 0, world, peer=peer)
    rng = np.random.default_rng(5)
    other = {}
    for name in DS.NAMES:
        v = np.concatenate([rng.normal(0, 3.0, 512), rng.uniform(50.0, 90.0, 512)])      # [sum | sum of squares]
        other[name] = torch.tensor(v, dtype=torch.float64)
        if peer:
            rk.set_slots(name, {1: other[name]})
        else:
            rk.inject[name] = other[name].to(DEV)
    data, lab, ll, tsl = O.synth_batch(N, W, seed=3, widths=[80, 4, 8, 57, 33], min_len=1, max_len=4)
    _nan_ws(m, N, W)
    dlogits = torch.randn((W // 4 - 1, N, 64), device=DEV) * 1e-2
    rk.step(_t(data), _t(tsl), dlogits)
    stats = m.tap_raw("stats", N, W).cpu().numpy()
    local = np.stack([rk.local["F1"].cpu().numpy(), rk.local["F2"].cpu().numpy()]).reshape(2, 2, 512)
    inj = np.stack([other["F1"].numpy(), other["F2"].numpy()]).reshape(2, 2, 512)
    assert np.array_equal(stats, local + inj), "the stats tap does not hold the global sums"
    want = M.ema_update(M.initial(), stats, N * (W // 4) * 4 * world)
    assert np.array_equal(m.bn_moving.cpu().numpy(), want)


# ------------------------------------------------------------------------------------------------ 3 + 4. fold and stages
def _stage_checks(case, N, W, widths, dtype="bf16", sample=None, chunk=None, seed=5):
    """One moving-mode forward: the fold bit for bit, then every stage from conv4_1 on against fp64 on its own operands."""
    from oracle import crnn_oracle as O
    pn = _with_negative_gamma(G8._params(3) if dtype == "fp8" else _params())
    mv = _moving()
    m = _model(pn, mv, dtype)
    data, _, _, tsl = O.synth_batch(N, W, seed=seed, widths=widths_of(N, W, widths), min_len=1, max_len=4)
    if dtype == "fp8":
        _nan_ws(m, N, W)
        m.calibrate_fp8(_t(data), _t(tsl))
    logits = _forward(m, data, tsl)
    torch.cuda.synchronize()
    T = W // 4 - 1
    f = M.fold(pn, mv)
    P = {k: torch.as_tensor(np.asarray(v, np.float64), device=DEV) for k, v in pn.items()}
    # the bf16 outputs; on the fp8 path conv5 keeps test_gpu_fp8's bound (e4m3 operands, bf16 output)
    ck = Checker(f"{dtype}/{case}", dict(G8.BF16_BOUNDS if dtype == "fp8" else B.STAGE_BOUNDS), REPORT, ulp_bf16)
    # 3. the fold, exactly
    wt = {}
    for l, (k, K) in enumerate((("conv4_1", 2304), ("conv4_2", 4608))):
        got = m.tap_raw("moving_w_" + k, N, W).double()
        ref = f[k]["w"].reshape(K, 512).t().to(DEV)
        ck.exact(f"fold_w_{k}", got, ref)
        wt[k] = got.t().reshape(3, 3, K // 9, 512)                      # HWIO
    bias = m.tap_raw("moving_bias", N, W).double()
    ck.exact("fold_bias", bias.cpu().numpy(), np.stack([f[k]["b"] for k in M.LAYERS]))
    for name in ("a4a_pre", "a4b_pre"):
        with pytest.raises(Exception, match="INVALID_VALUE|moving statistics"):
            m.tap(name, N, W)
    for name in ("bn", "stats"):
        with pytest.raises(Exception, match="INVALID_VALUE|moving statistics"):
            m.tap_raw(name, N, W)
    img = list(range(N)) if sample is None else list(sample)
    n = chunk or N
    parts = lambda idx: [idx[i:i + n] for i in range(0, len(idx), n)]     # noqa: E731
    Gt = {k: m.tap(k, N, W) for k in ("conv5", "xproj", "lstm_out")}
    if dtype == "bf16":
        Gt.update({k: m.tap(k, N, W) for k in ("conv3_2", "conv4_1", "conv4_2")})
        for s in parts(list(range(N))):
            r = S.conv_relu_stage(Gt["conv3_2"][s].double(), wt["conv4_1"], bias[0])
            ck.close("conv4_1", Gt["conv4_1"][s], r["out"], r["acc"], key="conv3_1")
            r = S.conv_relu_pool12_stage(Gt["conv4_1"][s].double(), wt["conv4_2"], bias[1])
            ck.close("conv4_2", Gt["conv4_2"][s], r["out"], r["acc"], key="conv3_2")
            r = S.conv5_stage(Gt["conv4_2"][s].double(), S.bf16(P["conv5/weights"]), P["conv5/biases"])
            ck.close("conv5", Gt["conv5"][s][:, :T], r["out"], r["acc"])
        cks = [ck]
    else:
        # e4m3: colscale' exactly, then the e4m3 GEMMs on their own decoded operands with weights e4m3 x wscale x s
        cs = m.tap_raw("fp8_colscale", N, W).cpu().numpy()
        csm = m.tap_raw("fp8_colscale_moving", N, W).cpu().numpy()
        ck.exact("fold_colscale", csm, M.colscale_moving(cs, f["conv4_1"]["s"], f["conv4_2"]["s"]))
        scales = m.tap_raw("fp8_scales", N, W).double()
        raw = {k: m.tap_raw(k, N, W) for k in ("conv3_2", "conv4_1", "conv4_2")}
        Wq, _, _ = G8._weights(m, N, W)
        val = lambda k, s: G8.decode(raw[k][s]) * scales[G8.FP8_ACTS.index(k)]     # noqa: E731
        ck8 = Checker(f"fp8/{case}", G8.BOUNDS, REPORT, G8.ulp_e4m3)
        sat = {}
        s41 = torch.as_tensor(f["conv4_1"]["s"], device=DEV)
        s42 = torch.as_tensor(f["conv4_2"]["s"], device=DEV)
        for s in parts(list(range(N))):
            r = S.conv_relu_stage(val("conv3_2", s), Wq["conv4_1"] * s41, bias[0])
            G8.e4m3_stage(ck8, sat, "conv4_1", G8.decode(raw["conv4_1"][s]), r["out"], r["acc"], scales[3])
            r = S.conv_relu_pool12_stage(val("conv4_1", s), Wq["conv4_2"] * s42, bias[1])
            G8.e4m3_stage(ck8, sat, "conv4_2", G8.decode(raw["conv4_2"][s]), r["out"], r["acc"], scales[4])
            r = S.conv5_stage(val("conv4_2", s), Wq["conv5"], P["conv5/biases"])
            ck.close("conv5", Gt["conv5"][s][:, :T], r["out"], r["acc"])
        cks = [ck, ck8]
    G8.tail_checks(ck, P, Gt, logits, tsl, T, parts(img))
    fail = []
    for c in cks:
        c.report()
        fail += c.fail
    assert not fail, "\n".join(fail)
    return m, pn, mv


MOVING_SHAPES = SHAPES + [pytest.param(512, W, "cycle", id=f"N512_W{W}") for W in (80, 160, 256)] + [
    pytest.param(3, W, [W, W - 4, 8], id=f"N3_W{W}") for W in (8, 12, 16, 512, 516, 1024)]


@pytest.mark.parametrize("N,W,widths", MOVING_SHAPES)
@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
def test_moving_stages_per_element(dtype, N, W, widths, request):
    big = N >= 512
    _stage_checks(request.node.callspec.id, N, W, widths, dtype, sample=range(0, N, 37) if big else None, chunk=128 if big else None)


@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
def test_moving_stages_per_element_c3(dtype):
    _stage_checks("C3_N1024_W256", 1024, 256, "cycle", dtype, sample=range(0, 1024, 97), chunk=128)


# ------------------------------------------------------------------------------------------------ 5. batch independence
@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
def test_each_image_and_line_as_if_alone(dtype):
    from oracle import crnn_oracle as O
    pn = _with_negative_gamma(G8._params(3) if dtype == "fp8" else _params())
    m = _model(pn, _moving(), dtype)
    N, W = 6, 96
    widths = [96, 40, 8, 64, 92, 20]
    data, _, _, tsl = O.synth_batch(N, W, seed=4, widths=widths, min_len=1, max_len=4)
    if dtype == "fp8":
        _nan_ws(m, N, W)
        m.calibrate_fp8(_t(data), _t(tsl))
    whole = _forward(m, data, tsl).clone()
    for i in range(N):
        alone = _forward(m, data[i:i + 1], tsl[i:i + 1])
        assert torch.equal(whole[:, i], alone[:, 0]), f"image {i}: batched logits differ from the image alone"
    # packed lines: line i in columns [0, W_i) of its slot, zero beyond; each equal to that line fed alone at width W_i
    lw = np.asarray(widths, np.int32)
    packed = np.zeros_like(data)
    lt = np.minimum(tsl, lw // 4 - 1).astype(np.int32)
    for i in range(N):
        packed[i, :lw[i]] = data[i, :lw[i]]
    got = _forward(m, packed, lt, lines=lw).clone()
    for i in range(N):
        alone = _forward(m, np.ascontiguousarray(packed[i:i + 1, :lw[i]]), lt[i:i + 1])
        assert torch.equal(got[:lt[i], i], alone[:lt[i], 0]), f"line {i}: packed logits differ from the line alone"


def test_lines_workspace_holds_no_per_line_statistics():
    from lstm_ctc_ocr_b200 import _lib
    m = _model(_params())
    sizes = []
    for mode in ("batch", "moving"):
        m.set_bn_statistics(mode)
        nb = _lib.c_size_t()
        _lib.check(m.lib.crnn_lines_workspace_size(m.handle, 1024, 256, nb))
        sizes.append(nb.value)
    assert sizes[0] - sizes[1] >= 2 * 1024 * 2 * 512 * 8 + 2 * 1024 * 4 * 512 * 4


# ------------------------------------------------------------------------------------------------ 6. end to end
def test_session_decodes_with_moving_statistics(monkeypatch):
    """cfg.TEST.BN_STATS = "moving" through Session.run on packed lines of the trained fixture, greedy decode: equal to the
    decode of the fp64 moving-mode forward (tests/bn_moving_refs.forward) wherever its best-path margin exceeds 0.25.  The
    fixture's moving statistics are those of a batch-mode forward over the same rendered lines (f64 "stats" tap)."""
    import random
    import test_gpu_packed_eval as PE
    from lstm_ctc_ocr_b200 import session
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.test import decodeRes, pack_lines, prepare_line
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from oracle import crnn_oracle as O
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    pn = dict(PE._load("make_decode10k", "tests", "golden", "make_decode10k.py").load_weights())
    rng = random.Random(17)
    labels = [gen.gen_rand(rng, 4, 30) for _ in range(32)]
    lines = [prepare_line(gen.render_line(t, rng=rng)) for t in labels]
    data, lw, tsl = pack_lines(lines)
    N, W = data.shape[:2]
    # moving statistics: the batch statistics of a whole-batch forward over the lines
    m = _model(pn)
    _forward(m, data, tsl)
    st = m.tap_raw("stats", N, W).cpu().numpy()
    cnt = N * (W // 4) * 4
    mean = st[:, 0] / cnt
    mv = np.stack([mean, np.maximum(st[:, 1] / cnt - mean * mean, 0.0)], axis=1).astype(np.float32)
    po = O.to_torch({k: np.asarray(v, np.float64) for k, v in pn.items()})
    refs = [M.forward(po, data[i:i + 1, :lw[i]], tsl[i:i + 1], moving=mv).numpy() for i in range(N)]
    saved = (cfg.TEST.BN_STATS, cfg.TEST.COMPUTE_DTYPE)
    try:
        for dt in ("bf16", "fp8"):
            cfg.TEST.BN_STATS, cfg.TEST.COMPUTE_DTYPE = "moving", dt
            net = get_network("LSTM_test")
            with session.Session(device=DEV) as sess:
                with pytest.raises(KeyError, match="moving"):
                    sess.assign(net, pn)
                sess.assign(net, dict(pn, **_state(mv)))
                dense = sess.run(Fetch(net, "dense_decoded"), {net.data: data, net.line_width: lw, net.time_step_len: tsl,
                                                              net.keep_prob: 1.0})
            agree = clear = 0
            for i in range(N):
                ref = refs[i][:int(tsl[i])]
                top = np.sort(ref[:, 0], axis=-1)
                if (top[:, -1] - top[:, -2]).min() <= 0.25:
                    continue
                clear += 1
                want = O.greedy_decode(ref, tsl[i:i + 1])[0]
                got = [int(c) for c in dense[i] if c != 0]
                agree += int(got == want)
            assert clear > 0 and agree == clear, (dt, agree, clear)
            acc = sum("".join(decodeRes(dense[i])) == labels[i] for i in range(N)) / N
            print(f"moving-mode decode {dt}: {agree}/{clear} lines with a clear margin equal the fp64 decode; accuracy {acc:.3f}")
    finally:
        cfg.TEST.BN_STATS, cfg.TEST.COMPUTE_DTYPE = saved


# ------------------------------------------------------------------------------------------------ 7. status codes
def test_status_codes_leave_outputs_untouched():
    from lstm_ctc_ocr_b200 import _lib, engine
    from oracle import crnn_oracle as O
    N, W = 3, 48
    data, _, _, tsl = O.synth_batch(N, W, seed=2, widths=[48, 20, 8])
    pn = _params()
    d, tl = _t(data), _t(tsl)

    def code(fn, *a):
        return int(fn(*a))

    # training mode + moving: CRNN_INVALID_VALUE
    m = _model(pn)
    m.set_training(True)
    assert code(m.lib.crnn_model_set_bn_statistics, m.handle, 1) == 1
    m.set_training(False)
    # unbound buffer: the forward returns CRNN_NOT_BOUND and writes nothing
    assert code(m.lib.crnn_model_bind_bn_moving, m.handle, None, ctypes.c_float(0.999)) == 0
    assert code(m.lib.crnn_model_set_bn_statistics, m.handle, 1) == 0
    m.bn_statistics = "moving"
    out = _nan((W // 4 - 1, N, 64))
    before = out.clone()
    ws, nb = m._workspace(N, W)
    st = m.lib.crnn_forward(m.handle, d.data_ptr(), tl.data_ptr(), N, W, out.data_ptr(), ws, nb, 0)
    torch.cuda.synchronize()
    assert st == 3 and torch.equal(out.view(torch.int32), before.view(torch.int32))
    assert code(m.lib.crnn_model_bind_bn_moving, m.handle, m.bn_moving.data_ptr(), ctypes.c_float(1.5)) == 1
    # compute_dtype 2 / 3: CRNN_UNSUPPORTED
    for dt in ("f32", "tf32"):
        x = engine.CrnnModel(device=DEV, compute_dtype=dt)
        assert x.bn_moving is None
        assert code(x.lib.crnn_model_set_bn_statistics, x.handle, 1) == 4
        assert code(x.lib.crnn_model_bind_bn_moving, x.handle, None, ctypes.c_float(0.999)) == 4
        with pytest.raises(_lib.CrnnError):
            x.set_bn_statistics("moving")
    # fp8 calibrated in batch mode, then switched to moving: the scales are gone, the forward refuses and writes nothing
    f8 = _model(G8._params(3), dtype="fp8")
    _nan_ws(f8, N, W)
    f8.calibrate_fp8(_t(data), _t(tsl))
    f8.forward(_t(data), _t(tsl))
    f8.load_bn_moving(_state(_moving()))
    f8.calibrate_fp8(_t(data), _t(tsl))
    f8.set_bn_statistics("moving")
    out = _nan((W // 4 - 1, N, 64))
    ws, nb = f8._workspace(N, W)
    st = f8.lib.crnn_forward(f8.handle, d.data_ptr(), tl.data_ptr(), N, W, out.data_ptr(), ws, nb, 0)
    torch.cuda.synchronize()
    assert st == 1 and torch.equal(out.view(torch.int32), before.view(torch.int32))
    f8.calibrate_fp8(_t(data), _t(tsl))            # a moving-mode calibration makes it run
    f8.forward(_t(data), _t(tsl), out=out)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
