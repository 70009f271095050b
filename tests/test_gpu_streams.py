"""Every entry point on the caller's own streams: gated non-blocking compute and copy streams, a busy legacy stream, graph replay.

include/crnn_ctc.h promises that every call is asynchronous on the caller's stream, with no hidden host synchronisation, and
that the host buffers of crnn_forward_host / crnn_forward_pageable may be reused once the work queued on `copy_stream` has
completed.  Torch's default stream is the legacy NULL stream, which serialises with every blocking stream, so the rest of the
suite cannot see work issued to the wrong stream, a missing event between the copy and the compute stream, or a copy still
pending when the API says it is done.

The gated window (one run per case, deterministic by construction).  Reference: the call twice on the default stream; what the
two runs agree on bit for bit is the reproducible set (test_gpu_training_run._bit_identity's rule).  Window: the legacy stream is
gated for G0; on a fresh non-blocking stream s the inputs and outputs are filled with 0xFF, s is gated for G1, the real inputs are
copied in from device sources, the call is made on s and every output (model cases: every tap too) is cloned on s.  Work placed on
any other non-blocking stream without an event from s runs during G1 and reads the 0xFF inputs; work placed on the legacy stream
runs after G0 > 2 (G1 + the call's time), after the snapshots were taken.  Reproducible quantities must match bit for bit; the
model's stages go through the existing per-element checks against fp64 (test_gpu_stage_isolation.py's bounds), CTC through
tests/ctc_refs.py; then, after a device synchronise, the call again on s without gates (late writes that corrupt later calls).
0xFF goes only where every value is safe: f32 NaN, int32 -1 (lengths clamp to 0, label ids invalid, candidate slots empty), uint8
pixels 255; never the parameters or the lexicon CSR, and no poisoned value is used as an address (test_gpu_training_run.py).
A control issues crnn_ctc_greedy and crnn_ctc_loss on stream 0 inside the window: both must be reported as mismatches.

Host-buffer reuse: crnn_forward_host (chunks 1 and 4) and crnn_forward_pageable, f32 and uint8 feeds, compute_dtype 1 .. 4: the
compute stream is gated, the call made, copy_stream synchronised (what forward_host(wait_copy=True) does), and the host buffers
overwritten with 0xFF at once; the logits must equal the device-fed forward's bits.

Graph capture: after one call at the shape, the call captured on s (torch.cuda.graph, global mode), new inputs written into the
static buffers and replayed: the reproducible outputs equal a direct call on those inputs and differ from the capture-time ones.
"""
import os
import sys
import time

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ctc_refs as CR  # noqa: E402
import stage_refs as S  # noqa: E402
import test_gpu_stage_isolation as B  # noqa: E402
import test_gpu_stage_isolation_batch as BB  # noqa: E402
import test_gpu_training_run as TR  # noqa: E402
import test_gpu_ctc_long as CL  # noqa: E402
import test_gpu_u8_feed as U8  # noqa: E402
import test_gpu_width_edges as WE  # noqa: E402
from stage_check import Checker, ulp_bf16  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = B.DEV
G1_MS = 50.0
MODEL_SHAPES = [pytest.param(130, 40, "cycle", id="N130_W40"), pytest.param(3, 160, [160, 8, 97], id="N3_W160")]
_RATE = {}


def _cycles_per_ms():
    """torch.cuda._sleep's cycles per millisecond, measured once with CUDA events (no clock is assumed)."""
    if "r" not in _RATE:
        torch.cuda.synchronize()
        torch.cuda._sleep(1000000)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        torch.cuda._sleep(20000000)
        b.record()
        b.synchronize()
        _RATE["r"] = 20000000 / a.elapsed_time(b)
    return _RATE["r"]


def _gate(ms):
    """A bounded sleep kernel of `ms` milliseconds on the current stream."""
    assert 0 < ms < 1000
    torch.cuda._sleep(int(ms * _cycles_per_ms()))


def _t(a):
    return torch.tensor(np.asarray(a), device=DEV)


def _poison_(t):
    t.view(torch.uint8).fill_(255)


def _timed(call):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = call()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def _window(call, inputs=(), outputs=(), call_ms=0.0):
    """One gated run of call() on a fresh non-blocking stream (module docstring).  inputs: (device buffer, device source) pairs;
    outputs: caller-owned buffers filled with 0xFF first.  Returns (what call() returned, the stream)."""
    g0 = 2.0 * (G1_MS + call_ms) + 20.0
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    _gate(g0)                                   # the legacy stream: busy for G0
    with torch.cuda.stream(s):
        for d, _ in inputs:
            _poison_(d)
        for o in outputs:
            _poison_(o)
        _gate(G1_MS)
        for d, src in inputs:
            d.copy_(src)
        got = call()
    s.synchronize()
    torch.cuda.synchronize()
    return got, s


def _compare(a, b, got):
    """(reproducible keys that differ, keys two default-stream runs do not reproduce).  Keys under "full/" are operands of the
    stage checks only; the weight gradients ("grad/"), summed with f32 atomics, are never in the reproducible set."""
    keys = [k for k in a if not k.startswith("full/")]
    repro = [k for k in keys if not k.startswith("grad/") and TR._same_bits(a[k], b[k])]
    return [k for k in repro if not TR._same_bits(got[k], a[k])], [k for k in keys if k not in repro]


def _gated(name, call, inputs=(), outputs=(), check=None):
    """The reference pair, the window, the comparison and the late call; check(snapshot) runs the per-element checks on the
    window's own outputs.  Returns the window's snapshot."""
    for d, src in inputs:
        d.copy_(src)
    a, _ = _timed(call)
    b, ms = _timed(call)
    got, s = _window(call, inputs, outputs, ms)
    diff, other = _compare(a, b, got)
    nan = [k for k in other if not TR._finite(got[k])]
    assert not diff, f"{name}: on a gated side stream these differ from the default stream: {diff}"
    assert not nan, f"{name}: not finite on the side stream: {nan}"
    if check is not None:
        check(got)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        late = call()
    s.synchronize()
    diff, _ = _compare(a, b, late)
    assert not diff, f"{name}: a second call on the side stream differs (a late write corrupted state): {diff}"
    return got


# ---------------------------------------------------------------------------------------------------------- harness control
def _ctc_inputs(T, N, L, seed=0):
    logits, lab, ll, il = TR._ctc_case(T, N, L, seed=seed)
    return logits, _t(lab), _t(ll), _t(il), lab, ll, il


def test_harness_sees_work_on_the_legacy_stream():
    """crnn_ctc_greedy and crnn_ctc_loss issued with stream 0 inside the window: both are reported as mismatches."""
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200._lib import check
    lib = engine._lib.load()
    T, N, L = 60, 40, 4
    src, s_lab, s_ll, s_il, _, ll, _ = _ctc_inputs(T, N, L, seed=1)
    logits, il = torch.empty_like(src), torch.empty_like(s_il)
    out, ol = torch.empty((N, T), dtype=torch.int32, device=DEV), torch.empty(N, dtype=torch.int32, device=DEV)
    costs = torch.empty(N, dtype=torch.float32, device=DEV)

    def call():
        check(lib.crnn_ctc_greedy(logits.data_ptr(), il.data_ptr(), T, N, 64, engine.TF_BLANK, 0, out.data_ptr(), ol.data_ptr(), 0))
        check(lib.crnn_ctc_loss(logits.data_ptr(), 0, s_lab.data_ptr(), s_ll.data_ptr(), il.data_ptr(), T, N, 64, 0, int(ll.max()),
                                1.0, costs.data_ptr(), 0, 0, 0))
        return {"greedy_out": out.clone(), "greedy_len": ol.clone(), "ctc_costs": costs.clone()}
    for d, s in ((logits, src), (il, s_il)):
        d.copy_(s)
    a, _ = _timed(call)
    b, ms = _timed(call)
    got, _ = _window(call, [(logits, src), (il, s_il)], [out, ol, costs], ms)
    diff, _ = _compare(a, b, got)
    assert {"greedy_out", "greedy_len", "ctc_costs"} <= set(diff), f"the window missed work on the legacy stream: {diff}"


# ---------------------------------------------------------------------------------------------------------- model helpers
def _snap(m, N, W, logits, tsl, train=False, bwd=False):
    """TR._snapshot of the last forward (and backward), plus the full unpacked gates / cell states the stage checks read."""
    extra = {}
    if train and not bwd:
        extra.update({"raw/" + k: m.tap_raw(k, N, W) for k in ("am1", "am2", "am3")})
    if train:
        extra["full/gates_steps"] = S.unpack_gates(m.tap("gates", N, W), N)
        extra["full/csave_steps"] = S.unpack_csave(m.tap_raw("csave", N, W), N)
    out = TR._snapshot(m, N, W, logits, tsl, train=bwd)      # last: it ends in a device synchronise
    out.update(extra)
    return out


def _stage_checks(case, pn, data, tsl, snap, train, dlogits=None, table=None):
    """The existing per-element forward (and backward) stage checks on a snapshot taken on the side stream."""
    N, W = data.shape[0], data.shape[1]
    G = {k: snap[k] for k in B.FWD_TAPS}
    R = {k: snap["raw/" + k] for k in ("bn", "stats") + (("am1", "am2", "am3") if train else ())}
    if train:
        G["gates_steps"], G["csave_steps"] = snap["full/gates_steps"], snap["full/csave_steps"]
    ck = TR._checker("streams/" + case)
    F_ = B._Refs(pn, G, R, data, tsl, snap["logits"], N, W, DEV, BB.CHUNK)
    bnp = B._forward_checks(ck, F_, train=train)
    if dlogits is not None:
        for k in B.BWD_TAPS:
            G[k] = snap[k]
        grad = {k: snap["grad/" + k].to(DEV, torch.float64) for k in table}
        B._backward_checks(ck, F_, grad, dlogits, bnp)
    ck.assert_ok()


def _feed(N, W, widths, feed, seed=5):
    """(device-fed batch: f32 data or uint8 pixels, the f32 data the references read, labels, label_len, time_step_len)."""
    if feed == "u8":
        return U8._batch(N, W, widths, seed=seed)
    data, lab, ll, tsl = TR._batch(N, W, widths, seed=seed)
    return data, data, lab, ll, tsl


# ---------------------------------------------------------------------------------------------------------- bf16 model
@pytest.mark.parametrize("feed", ["f32", "u8"])
@pytest.mark.parametrize("N,W,widths", MODEL_SHAPES + [pytest.param(1024, 256, None, id="N1024_W256")])
def test_bf16_inference_forward_on_a_gated_stream(N, W, widths, feed):
    m, pn = TR._model(None, training=False)
    widths = BB._widths(N, W) if widths is None else widths
    fed, data, _, _, tsl = _feed(N, W, widths, feed)
    src, s_tsl = _t(fed), _t(tsl)
    d, d_tsl = torch.empty_like(src), torch.empty_like(s_tsl)
    out = torch.empty((W // 4 - 1, N, 64), dtype=torch.float32, device=DEV)

    def call():
        lg = m.forward(d, d_tsl, out=out)
        return _snap(m, N, W, lg, tsl)
    _gated(f"forward/{feed}", call, [(d, src), (d_tsl, s_tsl)], [out],
           check=lambda g: _stage_checks(f"inference/{feed}/N{N}_W{W}", pn, data, tsl, g, train=False))


@pytest.mark.parametrize("feed", ["f32", "u8"])
@pytest.mark.parametrize("N,W,widths", MODEL_SHAPES + [pytest.param(1024, 256, None, id="N1024_W256")])
def test_bf16_training_forward_ctc_backward_on_a_gated_stream(N, W, widths, feed):
    """The training forward, CTC (grad_scale 1/N) and crnn_backward / _u8, then crnn_total_loss, all on s; every forward and
    backward stage per element, the CTC gradient against fp64.  The 1024 x 256 shape runs the forward only."""
    from lstm_ctc_ocr_b200 import engine
    m, pn = TR._model("Adam")
    widths = BB._widths(N, W) if widths is None else widths
    fed, data, lab, ll, tsl = _feed(N, W, widths, feed)
    src, s_tsl, s_lab, s_ll = _t(fed), _t(tsl), _t(lab), _t(ll)
    d, d_tsl, d_lab, d_ll = (torch.empty_like(x) for x in (src, s_tsl, s_lab, s_ll))
    out = torch.empty((W // 4 - 1, N, 64), dtype=torch.float32, device=DEV)
    bwd = N < 1024

    def call():
        lg = m.forward(d, d_tsl, out=out)
        if not bwd:
            return _snap(m, N, W, lg, tsl, train=True)
        costs, grad = engine.ctc_loss(lg, d_lab, d_ll, d_tsl, want_grad=True, grad_scale=1.0 / N, max_label_len=int(ll.max()))
        m.backward(d, d_tsl, grad)
        extra = dict(ctc_costs=costs.clone(), ctc_grad=grad.clone(), total_loss=m.total_loss(costs).clone())
        snap = _snap(m, N, W, lg, tsl, train=True, bwd=True)
        snap.update(extra)
        return snap

    def check(g):
        dl = None
        if bwd:
            ck = TR._checker(f"streams/ctc/{feed}/N{N}_W{W}")
            ref = CR.ctc_fp64(g["logits"], lab, ll, S.clamp_lens(tsl, W // 4 - 1), grad_scale=1.0 / N, max_label_len=int(ll.max()))
            CR.check_grad(ck, "fast", g["ctc_costs"], g["ctc_grad"], ref, 1.0 / N)
            ck.assert_ok()
            dl = g["ctc_grad"]
        _stage_checks(f"training/{feed}/N{N}_W{W}", pn, data, tsl, g, train=True, dlogits=dl, table=m.table)
    _gated(f"training/{feed}", call, [(d, src), (d_tsl, s_tsl), (d_lab, s_lab), (d_ll, s_ll)], [out], check=check)


@pytest.mark.parametrize("solver", ["Adam", "Momentum", "RMS"])
def test_solver_step_from_a_restored_state_on_a_gated_stream(solver):
    """crnn_clip_{adam,momentum,rmsprop}_step after a real backward, from the same restored parameters and slots each time."""
    m, pn = TR._model(solver)
    N, W = 130, 40
    batch = TR._batch(N, W, "cycle")
    TR._fwd_bwd(m, batch)
    m.apply_gradients(TR.LR[solver], 1, clip=TR.CLIP)
    TR._fwd_bwd(m, batch)
    saved = {k: getattr(m, k).clone() for k in ("params", "adam_m", "adam_v")}
    s_grads = m.grads.clone()

    def call():
        for k, v in saved.items():
            getattr(m, k).copy_(v)
        m.apply_gradients(TR.LR[solver], 2, clip=TR.CLIP)
        return {k: getattr(m, k).clone() for k in saved}
    _gated(f"solver/{solver}", call, [(m.grads, s_grads)])


@pytest.mark.parametrize("feed", ["f32", "u8"])
@pytest.mark.parametrize("N,W,widths", MODEL_SHAPES)
def test_forward_lines_on_a_gated_stream(N, W, widths, feed):
    m, pn = TR._model(None, training=False)
    fed, data, _, _, _ = _feed(N, W, widths, feed)
    lw = np.array([max(8, w // 4 * 4) for w in B.widths_of(N, W, widths)], np.int32)
    tsl = (lw // 4 - 1).astype(np.int32)
    src, s_lw, s_tsl = _t(fed), _t(lw), _t(tsl)
    d, d_lw, d_tsl = torch.empty_like(src), torch.empty_like(s_lw), torch.empty_like(s_tsl)
    out = torch.empty((W // 4 - 1, N, 64), dtype=torch.float32, device=DEV)

    def call():
        lg = m.forward_lines(d, d_lw, d_tsl, out=out)
        return {"logits": lg.clone(), "raw/bn": m.tap_raw("bn", N, W, lines=True), "raw/stats": m.tap_raw("stats", N, W, lines=True)}
    _gated(f"forward_lines/{feed}", call, [(d, src), (d_lw, s_lw), (d_tsl, s_tsl)], [out])


def test_moving_statistics_forward_and_update_on_a_gated_stream():
    """Moving BatchNorm statistics: the evaluation forward folding them, and the update at the start of the backward."""
    m, pn = TR._model("Adam")
    N, W = 130, 40
    data, lab, ll, tsl = TR._batch(N, W, "cycle")
    TR._fwd_bwd(m, (data, lab, ll, tsl))
    saved = m.bn_moving.clone()
    src, s_tsl = _t(data), _t(tsl)
    d, d_tsl = torch.empty_like(src), torch.empty_like(s_tsl)
    dl = TR._dlogits(N, W)

    def train_call():
        m.bn_moving.copy_(saved)
        lg = m.forward(d, d_tsl)
        m.backward(d, d_tsl, dl)
        return {"logits": lg.clone(), "bn_moving": m.bn_moving.clone()}
    _gated("moving/update", train_call, [(d, src), (d_tsl, s_tsl)])
    m.set_training(False)
    m.set_bn_statistics("moving")

    def eval_call():
        lg = m.forward(d, d_tsl)
        return {"logits": lg.clone()}
    _gated("moving/forward", eval_call, [(d, src), (d_tsl, s_tsl)])


# ---------------------------------------------------------------------------------------------------------- fp8, f32-class
def test_fp8_model_created_on_a_side_stream_while_the_legacy_stream_is_busy():
    """An fp8 model created, loaded and calibrated (f32, then uint8) on s while the legacy stream is busy, then forward and
    forward_lines: its e4m3 weights and scales must survive everything creation queued."""
    from lstm_ctc_ocr_b200 import engine
    pn = TR._model(None, training=False)[1]
    N, W = 130, 40
    u, data, _, _, tsl = U8._batch(N, W, "cycle")
    lw = np.array([max(8, w // 4 * 4) for w in B.widths_of(N, W, "cycle")], np.int32)
    ins = [(_t(x), _t(x)) for x in (data, u, tsl, lw, (lw // 4 - 1).astype(np.int32))]
    for d, _ in ins:
        d.zero_()
    (d, _), (du, _), (d_tsl, _), (d_lw, _), (d_ltsl, _) = ins
    made = []

    def call():
        m = engine.CrnnModel(weight_decay=TR.WD, device=DEV, compute_dtype="fp8")
        m.load_params(pn)
        made.append(m)
        m.calibrate_fp8(d, d_tsl)
        lg = m.forward(d, d_tsl)
        ln = m.forward_lines(d, d_lw, d_ltsl)
        m.calibrate_fp8(du, d_tsl)
        lu = m.forward(du, d_tsl)
        return {"logits": lg.clone(), "lines": ln.clone(), "logits_u8": lu.clone(), "scales": m.tap_raw("fp8_scales", N, W)}

    def late():
        m = made[-1]
        return {"logits_u8": m.forward(du, d_tsl).clone(), "logits": m.forward(d, d_tsl).clone()}
    for x, src in ins:
        x.copy_(src)
    a, _ = _timed(call)
    b, ms = _timed(call)
    got, s = _window(call, ins, (), ms)
    diff, _ = _compare(a, b, got)
    assert not diff, f"fp8 creation on a side stream: differs from the default stream: {diff}"
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        again = late()
    s.synchronize()
    diff = [k for k in again if not TR._same_bits(again[k], a[k])]
    assert not diff, f"fp8 model created on a side stream: a later forward differs (creation wrote its block late): {diff}"


def test_fp8_set_scales_then_forward_on_a_gated_stream():
    m, pn = TR._model(None, compute_dtype="fp8", training=False)
    N, W = 130, 40
    data, _, _, tsl = TR._batch(N, W, "cycle")
    src, s_tsl = _t(data), _t(tsl)
    d, d_tsl = torch.empty_like(src), torch.empty_like(s_tsl)
    m.calibrate_fp8(src, s_tsl)
    scales = m.fp8_scales() * 2

    def call():
        m.set_fp8_scales(scales)
        return {"logits": m.forward(d, d_tsl).clone()}
    _gated("fp8/set_scales", call, [(d, src), (d_tsl, s_tsl)])


@pytest.mark.parametrize("dtype", ["f32", "tf32"])
@pytest.mark.parametrize("N,W,widths", MODEL_SHAPES)
def test_f32_class_forward_on_a_gated_stream(N, W, widths, dtype):
    m, pn = TR._model(None, compute_dtype=dtype, training=False)
    data, _, _, tsl = TR._batch(N, W, widths)
    src, s_tsl = _t(data), _t(tsl)
    d, d_tsl = torch.empty_like(src), torch.empty_like(s_tsl)
    out = torch.empty((W // 4 - 1, N, 64), dtype=torch.float32, device=DEV)

    def call():
        return {"logits": m.forward(d, d_tsl, out=out).clone(), "raw/cst": m.tap_raw("cst", N, W)}
    _gated(f"{dtype}/forward", call, [(d, src), (d_tsl, s_tsl)], [out])


# ---------------------------------------------------------------------------------------------------------- free functions
@pytest.mark.parametrize("T,N,L,ws", [(120, 24, 60, False), (600, 8, 100, True)], ids=["shared_T120_L60", "workspace_T600_L100"])
def test_ctc_loss_on_a_gated_stream(T, N, L, ws):
    from lstm_ctc_ocr_b200 import engine
    src, s_lab, s_ll, s_il, lab, ll, il = _ctc_inputs(T, N, L)
    x, d_il, d_lab, d_ll = (torch.empty_like(v) for v in (src, s_il, s_lab, s_ll))
    nbytes = engine.ctc_workspace_bytes(T, N, 64, int(ll.max()))
    assert (nbytes > 0) == ws
    costs, grad = torch.empty(N, device=DEV), torch.empty((T, N, 64), device=DEV)
    w = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=DEV)

    def call():
        engine.ctc_loss(x, d_lab, d_ll, d_il, want_grad=True, grad_scale=0.25, max_label_len=int(ll.max()), costs=costs, grad=grad,
                        workspace=w if nbytes else None)
        return {"costs": costs.clone(), "grad": grad.clone()}

    def check(g):
        # the bounds of the kernel at these frame counts: test_gpu_width_edges.py (shared memory), test_gpu_ctc_long.py (workspace)
        ck = (Checker(f"streams/ctc_loss/T{T}_L{L}", CL.BOUNDS, CL.REPORT, ulp_bf16, CL.L2) if ws
              else WE._checker(f"streams/ctc_loss/T{T}_L{L}", T))
        ref = CR.ctc_fp64(src, lab, ll, S.clamp_lens(il, T), grad_scale=0.25, max_label_len=int(ll.max()))
        CR.check_grad(ck, "long" if ws else "fast", g["costs"], g["grad"], ref, 0.25)
        ck.assert_ok()
    _gated(f"ctc_loss/{T}/{L}", call, [(x, src), (d_il, s_il), (d_lab, s_lab), (d_ll, s_ll)], [costs, grad] + ([w] if nbytes else []), check=check)


def test_decoders_on_a_gated_stream():
    """crnn_ctc_greedy and crnn_ctc_beam_search_device into caller-owned outputs and arena, all poisoned."""
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200._lib import check
    lib = engine._lib.load()
    T, N, BW = 60, 40, 16
    src, _, _, s_il, _, _, _ = _ctc_inputs(T, N, 4, seed=2)
    x, d_il = torch.empty_like(src), torch.empty_like(s_il)
    nb = engine.beam_workspace_bytes(T, N, 64, BW)
    arena = torch.empty(nb, dtype=torch.uint8, device=DEV)
    o, bo = (torch.empty((N, T), dtype=torch.int32, device=DEV) for _ in range(2))
    ol, bl = (torch.empty(N, dtype=torch.int32, device=DEV) for _ in range(2))
    nlp = torch.empty(N, dtype=torch.float32, device=DEV)

    def call():
        check(lib.crnn_ctc_greedy(x.data_ptr(), d_il.data_ptr(), T, N, 64, engine.TF_BLANK, 0, o.data_ptr(), ol.data_ptr(),
                                  engine._stream()))
        check(lib.crnn_ctc_beam_search_device(x.data_ptr(), d_il.data_ptr(), T, N, 64, BW, 1, 0, bo.data_ptr(), bl.data_ptr(),
                                              nlp.data_ptr(), arena.data_ptr(), nb, engine._stream()))
        return {"greedy_out": o.clone(), "greedy_len": ol.clone(), "beam_out": bo.clone(), "beam_len": bl.clone(),
                "beam_nlp": nlp.clone()}
    _gated("decoders", call, [(x, src), (d_il, s_il)], [o, ol, bo, bl, nlp, arena])


@pytest.mark.parametrize("dense", [False, True], ids=["flat", "dense"])
def test_ctc_align_on_a_gated_stream(dense):
    from lstm_ctc_ocr_b200 import engine
    T, N, L = 90, 24, 10
    src, s_lab, s_ll, s_il, lab, ll, _ = _ctc_inputs(T, N, L, seed=3)
    if dense:
        rows = np.zeros((N, L), np.int32)
        off = np.concatenate([[0], np.cumsum(ll)])
        for n in range(N):
            rows[n, :ll[n]] = lab[off[n]:off[n + 1]]
        s_lab = _t(rows)
    from lstm_ctc_ocr_b200._lib import check
    x, d_lab, d_ll, d_il = (torch.empty_like(v) for v in (src, s_lab, s_ll, s_il))
    nb = engine.ctc_align_workspace_bytes(T, N, 64, L)
    ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
    st, en = (torch.empty(s_lab.shape, dtype=torch.int32, device=DEV) for _ in range(2))
    pk, lp = torch.empty(s_lab.shape, dtype=torch.float32, device=DEV), torch.empty(N, dtype=torch.float32, device=DEV)
    stride = L if dense else 0

    def call():
        check(engine._lib.load().crnn_ctc_align(x.data_ptr(), d_lab.data_ptr(), stride, d_ll.data_ptr(), d_il.data_ptr(), T, N, 64, 0,
                                                L, st.data_ptr(), en.data_ptr(), pk.data_ptr(), lp.data_ptr(), ws.data_ptr(), nb,
                                                engine._stream()))
        return {"start": st.clone(), "end": en.clone(), "peak": pk.clone(), "path_logprob": lp.clone()}
    _gated(f"align/{'dense' if dense else 'flat'}", call, [(x, src), (d_lab, s_lab), (d_ll, s_ll), (d_il, s_il)],
           [st, en, pk, lp, ws])


def _lexicon_case(seed=4):
    from lstm_ctc_ocr_b200 import engine
    rng = np.random.default_rng(seed)
    words = [rng.integers(1, 63, size=int(rng.integers(1, 9))).tolist() for _ in range(3000)]
    lex = engine.Lexicon(words, device=DEV)
    T, N, M = 40, 32, 8
    reads = np.zeros((N, M), np.int32)
    rl = rng.integers(0, M + 1, size=N).astype(np.int32)
    for n in range(N):
        w = lex.entries[int(rng.integers(len(lex)))][:M]
        reads[n, :len(w)] = w
        rl[n] = len(w)
        if n % 3 == 0 and rl[n] > 1:
            reads[n, 0] = int(rng.integers(1, 63))
    logits = torch.tensor(rng.standard_normal((T, N, 64)).astype(np.float32) * 3, device=DEV)
    il = _t(rng.integers(0, T + 1, size=N).astype(np.int32))
    return lex, _t(reads), _t(rl), logits, il


def test_lexicon_on_a_gated_stream():
    """crnn_lexicon_candidates and crnn_ctc_lexicon_score into caller-owned outputs, all poisoned; the lexicon CSR never is."""
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200._lib import check
    lib = engine._lib.load()
    lex, s_reads, s_rl, s_x, s_il = _lexicon_case()
    reads, rl, x, il = (torch.empty_like(v) for v in (s_reads, s_rl, s_x, s_il))
    (N, M), T, J = reads.shape, x.shape[0], 32
    cand, dist, score = (torch.empty((N, J), dtype=dt, device=DEV) for dt in (torch.int32, torch.int32, torch.float32))
    total, best, bs = (torch.empty(N, dtype=dt, device=DEV) for dt in (torch.int32, torch.int32, torch.float32))

    def call():
        check(lib.crnn_lexicon_candidates(reads.data_ptr(), M, rl.data_ptr(), N, lex.ids.data_ptr(), lex.off.data_ptr(), len(lex),
                                          lex.max_entry_len, 3, J, cand.data_ptr(), dist.data_ptr(), total.data_ptr(), engine._stream()))
        check(lib.crnn_ctc_lexicon_score(x.data_ptr(), il.data_ptr(), T, N, 64, 0, lex.ids.data_ptr(), lex.off.data_ptr(),
                                         lex.max_entry_len, cand.data_ptr(), J, score.data_ptr(), best.data_ptr(), bs.data_ptr(),
                                         engine._stream()))
        return {"cand": cand.clone(), "dist": dist.clone(), "total": total.clone(), "score": score.clone(), "best": best.clone(),
                "best_score": bs.clone()}
    _gated("lexicon", call, [(reads, s_reads), (rl, s_rl), (x, s_x), (il, s_il)], [cand, dist, score, total, best, bs])


# ---------------------------------------------------------------------------------------------------------- host buffers
_EVAL = {}


def _eval_model(cd):
    """One evaluation model per compute_dtype (fp8 calibrated), shared by the host-buffer and graph cases."""
    if cd not in _EVAL:
        m, pn = TR._model(None, compute_dtype={1: "bf16", 2: "f32", 3: "tf32", 4: "fp8"}[cd], training=False)
        if cd == 4:
            data, _, _, tsl = TR._batch(128, 64, "cycle", seed=9)
            m.calibrate_fp8(_t(data), _t(tsl))
        _EVAL[cd] = m
    return _EVAL[cd]


def _host_batch(feed, N=128, W=64, seed=5):
    fed, _, _, _, tsl = _feed(N, W, "cycle", feed, seed=seed)
    return np.ascontiguousarray(fed), tsl


@pytest.mark.parametrize("how", ["host_chunks1", "host_chunks4", "pageable"])
@pytest.mark.parametrize("feed", ["f32", "u8"])
@pytest.mark.parametrize("cd", [1, 2, 3, 4])
def test_host_buffers_reusable_once_copy_stream_is_done(cd, feed, how):
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200._lib import check
    m = _eval_model(cd)
    fed, tsl = _host_batch(feed)
    N, W = fed.shape[0], fed.shape[1]
    d_tsl = _t(tsl)
    ref = m.forward(_t(fed), d_tsl).clone()
    dt = torch.uint8 if feed == "u8" else torch.float32
    pinned = torch.empty(fed.shape, dtype=dt, pin_memory=True)
    pinned.numpy()[...] = fed
    pageable = fed.copy()
    stage = torch.empty(fed.shape, dtype=dt, device=DEV)
    out = torch.empty((W // 4 - 1, N, 64), dtype=torch.float32, device=DEV)
    ws, nbytes = m._workspace(N, W)
    sfx = engine._feed_suffix(fed.dtype)
    s, cs = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        _gate(G1_MS)
        if how == "pageable":
            check(getattr(m.lib, "crnn_forward_pageable" + sfx)(m.handle, pageable.ctypes.data, pinned.data_ptr(), stage.data_ptr(),
                                                                d_tsl.data_ptr(), N, W, out.data_ptr(), ws, nbytes, 4, 4,
                                                                s.cuda_stream, cs.cuda_stream))
        else:
            check(getattr(m.lib, "crnn_forward_host" + sfx)(m.handle, pinned.data_ptr(), stage.data_ptr(), d_tsl.data_ptr(), N, W,
                                                            out.data_ptr(), ws, nbytes, 4 if how == "host_chunks4" else 1,
                                                            s.cuda_stream, cs.cuda_stream))
    cs.synchronize()                             # what the header names; forward_host(wait_copy=True) waits for exactly this
    pinned.numpy().view(np.uint8)[...] = 255
    pageable.view(np.uint8)[...] = 255
    torch.cuda.synchronize()
    bad = int((TR._bits(out) != TR._bits(ref)).any(-1).sum()) if out.shape == ref.shape else -1
    assert TR._same_bits(out, ref), (f"compute_dtype {cd} {feed} {how}: host buffers rewritten after copy_stream completed "
                                     f"changed the logits ({bad} mismatching logit rows of {out.shape[0] * out.shape[1]})")


@pytest.mark.parametrize("cd", [1, 2, 3, 4])
def test_pageable_back_to_back_reusing_the_staging(cd):
    """Two engine.forward_pageable calls through one page-locked staging, the second after only the event recorded on the returned
    copy stream (as Session.run waits), on a gated compute stream: each call's logits are those of its own batch."""
    m = _eval_model(cd)
    (b1, tsl), (b2, _) = _host_batch("f32", seed=5), _host_batch("f32", seed=6)
    d_tsl = _t(tsl)
    r1, r2 = m.forward(_t(b1), d_tsl).clone(), m.forward(_t(b2), d_tsl).clone()
    assert not TR._same_bits(r1, r2)
    pinned = torch.empty(b1.shape, dtype=torch.float32, pin_memory=True)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        _gate(G1_MS)
        o1, _, cst = m.forward_pageable(b1, pinned, d_tsl, chunks=4)
        ev = torch.cuda.Event()
        ev.record(cst)
        ev.synchronize()
        o2, _, _ = m.forward_pageable(b2, pinned, d_tsl, chunks=4)
    torch.cuda.synchronize()
    assert TR._same_bits(o1, r1), f"compute_dtype {cd}: the first call read the second call's batch from the reused staging"
    assert TR._same_bits(o2, r2)


# ---------------------------------------------------------------------------------------------------------- graph capture
def _graph(name, run, statics, old, new):
    """run() issues the call on the current stream and returns {name: output}.  statics: the input buffers; old / new: their
    values at capture time and at replay.  The replay of new inputs must equal a direct call on them (reproducible outputs) and
    differ from the capture-time result."""
    for d, v in zip(statics, old):
        d.copy_(v)
    run()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.graph(g, stream=s):
        outs = run()
    g.replay()
    torch.cuda.synchronize()
    at_capture = {k: v.clone() for k, v in outs.items()}
    for d, v in zip(statics, new):
        d.copy_(v)
    g.replay()
    torch.cuda.synchronize()
    replayed = {k: v.clone() for k, v in outs.items()}
    a = {k: v.clone() for k, v in run().items()}
    torch.cuda.synchronize()
    b = {k: v.clone() for k, v in run().items()}
    torch.cuda.synchronize()
    diff, other = _compare(a, b, replayed)
    assert not diff, f"{name}: graph replay differs from the direct call in {diff}"
    assert all(TR._finite(replayed[k]) for k in other), name
    assert any(not TR._same_bits(replayed[k], at_capture[k]) for k in replayed), f"{name}: the replay repeats the capture-time result"
    return replayed


@pytest.mark.parametrize("case", ["bf16_f32", "bf16_u8", "lines", "fp8", "f32", "tf32", "host_chunks4", "host_chunks4_f32",
                                  "host_chunks4_tf32", "host_chunks4_fp8"])
def test_inference_forwards_replay_from_a_graph(case):
    """host_chunks4*: crnn_forward_host with chunks 4; its copy_stream joins the capture through the copy handshake's events
    (the bf16 path's ranges, the one-range copy of the fp8 and f32-class paths)."""
    N, W = 128, 64
    cd = {"fp8": 4, "f32": 2, "tf32": 3}.get(case.replace("host_chunks4_", ""), 1)
    m = _eval_model(cd)
    feed = "u8" if case == "bf16_u8" else "f32"
    (f1, tsl), (f2, _) = _host_batch(feed, seed=5), _host_batch(feed, seed=7)
    d_tsl = _t(tsl)
    if case.startswith("host_chunks4"):
        pinned = torch.empty(f1.shape, dtype=torch.float32, pin_memory=True)
        hd = pinned.numpy()
        if getattr(m, "_copy_stream", None) is None:
            m._copy_stream = torch.cuda.Stream(device=m.device)
        out = torch.empty((W // 4 - 1, N, 64), dtype=torch.float32, device=DEV)

        def run():
            m.forward_host(hd, d_tsl, chunks=4, out=out, wait_copy=False)
            return {"logits": out}
        for v in (f1,):
            hd[...] = v
        run()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        with torch.cuda.graph(g, stream=s):
            run()
        g.replay()
        torch.cuda.synchronize()
        first = out.clone()
        hd[...] = f2
        g.replay()
        torch.cuda.synchronize()
        assert TR._same_bits(out, m.forward(_t(f2), d_tsl)) and TR._same_bits(first, m.forward(_t(f1), d_tsl))
        assert not TR._same_bits(out, first)
        return
    d = _t(f1)
    lw = _t(np.array(B.widths_of(N, W, "cycle"), np.int32) // 4 * 4)
    lw.clamp_(min=8)
    ltsl = (lw // 4 - 1).to(torch.int32)

    def run():
        if case == "lines":
            return {"logits": m.forward_lines(d, lw, ltsl)}
        return {"logits": m.forward(d, d_tsl)}
    _graph(case, run, [d], [_t(f1)], [_t(f2)])


def test_free_functions_replay_from_a_graph():
    """Both CTC kernels, greedy decoding, alignment and the two lexicon calls."""
    from lstm_ctc_ocr_b200 import engine
    for T, N, L in ((120, 24, 60), (600, 8, 100)):
        x, s_lab, s_ll, s_il, lab, ll, il = _ctc_inputs(T, N, L, seed=0)
        x2 = _ctc_inputs(T, N, L, seed=8)[0]
        d = x.clone()
        ws = "auto" if engine.ctc_workspace_bytes(T, N, 64, L) else None

        def run():
            c, g = engine.ctc_loss(d, s_lab, s_ll, s_il, want_grad=True, max_label_len=L, workspace=ws)
            st, en, pk, lp = engine.ctc_align(d, s_lab, s_ll, s_il, max_label_len=L)
            o, ol = engine.ctc_greedy(d, s_il)
            return {"costs": c, "grad": g, "start": st, "end": en, "peak": pk, "lp": lp, "greedy": o, "greedy_len": ol}
        _graph(f"ctc/T{T}", run, [d], [x], [x2])
    lex, reads, rl, x, il = _lexicon_case()
    _, reads2, rl2, x2, _ = _lexicon_case(seed=5)
    dr, drl, dx = reads.clone(), rl.clone(), x.clone()

    def run():
        cand, dist, total = engine.lexicon_candidates(dr, drl, lex, 3, 32)
        score, best, bs = engine.ctc_lexicon_score(dx, il, lex, cand)
        return {"cand": cand, "dist": dist, "total": total, "score": score, "best": best, "best_score": bs}
    _graph("lexicon", run, [dr, drl, dx], [reads, rl, x], [reads2, rl2, x2])


def test_training_step_and_solvers_replay_from_a_graph():
    """The training forward + CTC + backward, then each solver step from a restored state (the step number is baked in)."""
    from lstm_ctc_ocr_b200 import engine
    N, W = 130, 40
    m, pn = TR._model("Adam")
    b1, b2 = TR._batch(N, W, "cycle", seed=5), TR._batch(N, W, "cycle", seed=6)
    d, d_tsl, lab, ll = _t(b1[0]), _t(b1[3]), _t(b1[1]), _t(b1[2])
    L = int(max(b1[2].max(), b2[2].max()))

    def run():
        lg = m.forward(d, d_tsl)
        c, g = engine.ctc_loss(lg, lab, ll, d_tsl, want_grad=True, grad_scale=1.0 / N, max_label_len=L)
        m.backward(d, d_tsl, g)
        return {"logits": lg, "costs": c, "grad/all": m.grads}
    _graph("training", run, [d], [_t(b1[0])], [_t(b2[0])])
    for solver in ("Adam", "Momentum", "RMS"):
        m.set_solver(solver)
        saved = {k: getattr(m, k).clone() for k in ("params", "adam_m", "adam_v")}
        g1 = m.grads.clone()
        g2 = g1 * 0.5 + 1e-4

        def step():
            for k, v in saved.items():
                getattr(m, k).copy_(v)
            m.apply_gradients(TR.LR[solver], 3, clip=TR.CLIP)
            return {k: getattr(m, k) for k in saved}
        _graph(f"solver/{solver}", step, [m.grads], [g1], [g2])
        for k, v in saved.items():
            getattr(m, k).copy_(v)


# ---------------------------------------------------------------------------------------------------------- Session, data parallel
def _gated_host_run(run, call_ms):
    """run() on a fresh non-blocking stream gated for G1, the legacy stream gated for G0 (as _window, for calls that take host
    inputs and return host arrays)."""
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    _gate(2.0 * (G1_MS + call_ms) + 20.0)
    with torch.cuda.stream(s):
        _gate(G1_MS)
        out = run()
    s.synchronize()
    torch.cuda.synchronize()
    return out


def _host_bits_equal(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_host_bits_equal(a[k], b[k]) for k in a)
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def _repro_diff(a, b, got):
    """Positions (list indices) that two default-stream runs reproduce bit for bit and the side-stream run does not."""
    return [i for i in range(len(a)) if _host_bits_equal(a[i], b[i]) and not _host_bits_equal(got[i], a[i])]


@pytest.mark.parametrize("packed", [False, True], ids=["whole", "packed"])
@pytest.mark.parametrize("source", ["page_locked", "pageable"])
def test_session_evaluation_fetches_on_a_side_stream(source, packed, tmp_path):
    """Session.run inside torch.cuda.stream(s) on a gated s, the legacy stream busy: logits, greedy and beam dense_decoded,
    read_alignment, label_alignment and lexicon_decoded equal a default-stream Session's (whatever two of those reproduce)."""
    from lstm_ctc_ocr_b200 import synthetic
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg, get_encode_decode_dict
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.session import Session
    N, W = 256, 256                              # 8.4 MB: a pageable batch takes crnn_forward_pageable, a page-locked one forward_host
    widths = BB._widths(N, W)
    data, lab, ll, tsl = TR._batch(N, W, widths)
    lw = np.array([max(8, w // 4 * 4) for w in widths], np.int32)
    if packed:
        tsl = np.minimum(tsl, lw // 4 - 1).astype(np.int32)
    if source == "page_locked":
        buf = torch.empty(data.shape, dtype=torch.float32, pin_memory=True).numpy()
        buf[...] = data
        data = buf
    rng = np.random.default_rng(3)
    _, dec = get_encode_decode_dict()
    words = [rng.integers(1, 63, size=int(rng.integers(1, 6))).tolist() for _ in range(2000)]
    path = tmp_path / "words.txt"
    path.write_text("\n".join("".join(dec[v] for v in w) for w in words) + "\n", encoding="utf-8")
    net = get_network("LSTM_train")
    params = synthetic.init_params(3, logits_scale=10.0)
    feed = {net.data: data, net.time_step_len: tsl, net.labels: lab, net.labels_len: ll}
    if packed:
        feed[net.line_width] = lw
    fetch = [Fetch(net, k) for k in ("logits", "dense_decoded", "read_alignment", "label_alignment", "lexicon_decoded")]
    old = (cfg.DECODER, cfg.TEST.LEXICON)
    cfg.TEST.LEXICON = str(path)
    try:
        with Session(device=DEV) as sess:
            sess.assign(net, params)

            def run():
                cfg.DECODER = "greedy"
                out = sess.run(fetch, feed)
                cfg.DECODER = "beam"
                return out + [sess.run(Fetch(net, "dense_decoded"), feed)]
            a = run()
            t0 = time.perf_counter()
            b = run()
            ms = (time.perf_counter() - t0) * 1e3
            got = _gated_host_run(run, ms)
            diff = _repro_diff(a, b, got)
            assert not diff, f"Session.run on a side stream ({source}, {'packed' if packed else 'whole'}) differs in fetches {diff}"
            assert _host_bits_equal(a[0], b[0]), "two default-stream evaluations differ: nothing left to compare"
    finally:
        cfg.DECODER, cfg.TEST.LEXICON = old


def test_session_training_with_device_prefetch_on_a_side_stream():
    """Three training steps (loss, logits, train_op) with a PrefetchFeeder attached, inside torch.cuda.stream(s) on a gated s:
    every step's loss and logits bit for bit those of a default-stream Session wherever two default-stream runs agree bit for
    bit, and every loss finite."""
    from lstm_ctc_ocr_b200 import synthetic
    from lstm_ctc_ocr_b200.lib.lstm.train import TrainOp, Variable
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.session import Session
    net = get_network("LSTM_train")
    loss, _ = net.build_loss()
    arg_fn = lambda k: dict(k=k, batch_size=64, render=False, seed=21, rank=0, world=1, bucket=gen.BUCKETS[k % 3])

    def run(call_ms=None):
        """The three steps; with call_ms, gated as _gated_host_run gates (the feeder and the Session are set up first, ungated).
        Returns (fetches, the steps' wall time in ms)."""
        f = gen.PrefetchFeeder(arg_fn, num_workers=2, depth=3, max_width=256, batch_size=64, keep=2)
        out = []
        try:
            with Session(device=DEV) as sess:
                sess.assign(net, synthetic.init_params(3, logits_scale=10.0))
                sess.attach_feeder(f)
                op = TrainOp(net, Variable(1e-3), Variable(0))
                s = torch.cuda.Stream() if call_ms is not None else torch.cuda.current_stream()
                torch.cuda.synchronize()
                if call_ms is not None:
                    _gate(min(2.0 * (G1_MS + call_ms) + 20.0, 950.0))
                t0 = time.perf_counter()
                with torch.cuda.stream(s):
                    if call_ms is not None:
                        _gate(G1_MS)
                    for _ in range(3):
                        view, lab, ll, tsl = next(f)
                        feed = {net.data: view, net.labels: np.array(lab), net.time_step_len: np.array(tsl),
                                net.labels_len: np.array(ll), net.keep_prob: 1.0}
                        l, x, _ = sess.run([loss, Fetch(net, "logits"), op], feed_dict=feed)
                        out += [np.float32(l), x.copy()]
                s.synchronize()
                ms = (time.perf_counter() - t0) * 1e3
                torch.cuda.synchronize()
                hits = sess.ahead_hits
        finally:
            f.close()
        assert hits >= 2, hits
        return out, ms
    a, _ = run()
    b, ms = run()
    got, _ = run(ms)
    assert all(np.isfinite(got[i]) for i in (0, 2, 4))
    diff = _repro_diff(a, b, got)
    assert not diff, f"training on a side stream differs at fetch positions {diff} (loss, logits per step)"


class _Request(object):
    def __init__(self, case_id):
        self.node = type("node", (), {"callspec": type("callspec", (), {"id": case_id})()})()


def test_data_parallel_emulation_on_a_side_stream():
    """test_gpu_dp_stages.py's world-2 callback case (2 x 8, W 100) and its peer-mode rank 1 -- crnn_model_set_peers included --
    run whole inside torch.cuda.stream(s) on a non-blocking s, every stage checked per element on the taps read from s.  These
    cases synchronise the device between their stages, so they run ungated: misplaced work races rather than failing every
    time."""
    import test_gpu_dp_stages as DS
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        DS.test_world2_callback_every_stage_and_composition(8, 100, "cpu", None, _Request("2x8_W100_side_stream"))
        DS.test_world2_peer_rank1_every_stage()
    torch.cuda.synchronize()
