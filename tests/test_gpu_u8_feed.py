"""uint8 feed on the GPU: the crnn_*_u8 entry points and every Python layer above them against the f32 feed of the same pixels.

The input is seeded random bytes u in which every value 0..255 occurs (0 and 255 on each image's first row), and the f32 feed is
the host quotient u / 255 (include/crnn_ctc.h).  Each case runs the f32 feed twice and the u8 feed once and applies the rule of
test_gpu_training_run._bit_identity: what the two f32 runs reproduce bit for bit the u8 run must reproduce bit for bit; the rest
(the weight gradients, summed with f32 atomics) must be NaN-free and pass their existing per-element stage checks, run on the
u8 run's own operands with data = u / 255.  No new tolerance."""
import io
import os
import sys
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_packed_eval as PE  # noqa: E402
import test_gpu_stage_isolation as B  # noqa: E402
import test_gpu_stage_isolation_batch as BB  # noqa: E402
import test_gpu_training_run as TR  # noqa: E402
from stage_check import widths_of  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = B.DEV
F255 = np.float32(255)
_tr_batch = TR._batch                 # the training-run tests below patch TR._batch; the u8 batches are built from the original


def _pixels(N, W, widths, seed):
    """uint8 [N, W, 32]: random bytes inside each image's width, zero past it; every byte value occurs, 0 and 255 on row 0."""
    rng = np.random.default_rng(seed)
    u = rng.integers(0, 256, size=(N, W, 32), dtype=np.uint8)
    wd = np.asarray(widths_of(N, W, widths))
    u[np.arange(W)[None, :] >= wd[:, None]] = 0
    u[:, 0, 0], u[:, 0, 31] = 0, 255
    flat = u.reshape(-1)
    valid = np.nonzero((np.arange(W)[None, :, None] < wd[:, None, None]).repeat(32, axis=2).reshape(-1))[0]
    if valid.size >= 512:
        flat[valid[64:320]] = np.arange(256, dtype=np.uint8)
    return u


def _batch(N, W, widths, seed=5):
    """(u8 pixels, f32 quotient, labels, label_len, time_step_len)."""
    _, lab, ll, tsl = _tr_batch(N, W, widths, seed=seed)
    u = _pixels(N, W, widths, seed + 101)
    return u, u.astype(np.float32) / F255, lab, ll, tsl


class U8Model(object):
    """The engine, fed uint8: forward / backward get the bytes of a data tensor that holds u / 255 exactly.  Lets the stage
    checks (which hand the f32 tensor to the model and to the fp64 references) run on the u8 feed's own operands."""

    def __init__(self, m):
        self.__dict__["m"] = m
        self.__dict__["fed"] = 0

    @staticmethod
    def bytes_of(data):
        u = torch.round(data * 255.0).to(torch.uint8)
        # numpy's IEEE quotient (torch divides by a scalar through its reciprocal)
        assert np.array_equal(u.cpu().numpy().astype(np.float32) / F255, data.cpu().numpy()), "data is not a u / 255 tensor"
        return u

    def forward(self, data, tsl, out=None):
        self.__dict__["fed"] += 1
        return self.m.forward(self.bytes_of(data), tsl, out=out)

    def backward(self, data, tsl, dlogits):
        return self.m.backward(self.bytes_of(data), tsl, dlogits)

    def __getattr__(self, k):
        return getattr(self.m, k)

    def __setattr__(self, k, v):
        setattr(self.m, k, v)


def _taps(m, N, W):
    """Every crnn_debug_tap / _raw name the model's path offers after a forward, keyed tap/ and raw/."""
    from lstm_ctc_ocr_b200._lib import CrnnError
    names = list(B.FWD_TAPS) + ["xproj"]
    raws = ["bn", "stats", "cst", "conv1", "conv2", "conv3_1", "conv3_2", "conv4_1", "conv4_2", "conv5", "lstm_out", "fp8_scales"]
    out = {}
    for k in names:
        try:
            out["tap/" + k] = m.tap(k, N, W).clone()
        except CrnnError:
            pass
    for k in raws:
        try:
            out["raw/" + k] = m.tap_raw(k, N, W).clone()
        except CrnnError:
            pass
    torch.cuda.synchronize()
    return out


def _rule(case, u8, fa, fb):
    ck = TR._checker("u8_feed/" + case)
    TR._bit_identity(ck, u8, fa, fb)
    ck.assert_ok()
    return ck


def _forward_snaps(m, u, f, tsl):
    N, W = u.shape[0], u.shape[1]
    d_tsl = torch.tensor(tsl, device=DEV)
    snaps = []
    for data in (f, f, u):
        lg = m.forward(torch.tensor(data, device=DEV), d_tsl)
        s = _taps(m, N, W)
        s["logits"] = lg.clone()
        snaps.append(s)
    return snaps


FWD_SHAPES = [pytest.param(*p.values, id=p.id) for p in B.SHAPES] + [
    pytest.param(1160, 160, "cycle", id="N1160_W160"), pytest.param(1024, 256, "cycle", id="C3_N1024_W256"),
    pytest.param(1, 8, [8], id="N1_W8"), pytest.param(1, 12, [12], id="N1_W12"), pytest.param(1, 1024, [1024], id="N1_W1024")]


@pytest.mark.parametrize("dtype", ["bf16", "f32", "tf32", "fp8"])
@pytest.mark.parametrize("N,W,widths", FWD_SHAPES)
def test_forward_u8_matches_the_f32_feed(dtype, N, W, widths):
    from lstm_ctc_ocr_b200 import engine
    u, f, _, _, tsl = _batch(N, W, widths)
    _, pn = TR._model("Adam", training=False)
    m = engine.CrnnModel(weight_decay=TR.WD, device=DEV, compute_dtype=dtype)
    m.load_params(pn)
    if dtype == "fp8":          # both feeds run with the same scales
        m.calibrate_fp8(torch.tensor(f, device=DEV), torch.tensor(tsl, device=DEV))
    fa, fb, su = _forward_snaps(m, u, f, tsl)
    assert "logits" in su and len(su) > 3
    _rule(f"forward/{dtype}/N{N}_W{W}", su, fa, fb)


@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
def test_host_feed_paths_u8(dtype):
    """Device-fed, page-locked (chunks 1 and 4) and pageable (1 and 8 host threads) u8 feeds give the device-fed u8 run's bits,
    and the u8 staging holds the batch afterwards."""
    from lstm_ctc_ocr_b200 import engine
    N, W = 1024, 256
    u, f, _, _, tsl = _batch(N, W, "cycle")
    _, pn = TR._model("Adam", training=False)
    m = engine.CrnnModel(weight_decay=TR.WD, device=DEV, compute_dtype=dtype)
    m.load_params(pn)
    d_tsl = torch.tensor(tsl, device=DEV)
    if dtype == "fp8":
        m.calibrate_fp8(torch.tensor(f, device=DEV), d_tsl)
    ref = [m.forward(torch.tensor(u, device=DEV), d_tsl).clone() for _ in range(2)]
    ref_taps = _taps(m, N, W)
    assert TR._same_bits(ref[0], ref[1])
    pinned = torch.empty((N, W, 32), dtype=torch.uint8).pin_memory()
    pinned.numpy()[...] = u
    for chunks in (1, 4):
        stage_before = m._staging(N, W, np.uint8)
        stage_before.fill_(7)
        lg, stage = m.forward_host(pinned.numpy(), d_tsl, chunks=chunks)
        torch.cuda.synchronize()
        assert stage.dtype == torch.uint8 and torch.equal(stage.cpu(), torch.from_numpy(u)), chunks
        assert TR._same_bits(lg, ref[0]), f"page-locked chunks={chunks}"
        got = _taps(m, N, W)
        assert all(TR._same_bits(got[k], ref_taps[k]) for k in ref_taps), chunks
    pin8 = torch.empty(N * W * 32, dtype=torch.uint8).pin_memory()
    for threads in (1, 8):
        m._staging(N, W, np.uint8).fill_(7)
        lg, stage, cst = m.forward_pageable(np.ascontiguousarray(u), pin8, d_tsl, chunks=4, host_threads=threads)
        torch.cuda.synchronize()
        assert torch.equal(stage.cpu(), torch.from_numpy(u)), threads
        assert TR._same_bits(lg, ref[0]), f"pageable threads={threads}"


@pytest.mark.parametrize("dtype", ["bf16", "fp8"])
@pytest.mark.parametrize("stats", ["batch", "moving"])
def test_packed_lines_u8(dtype, stats):
    from lstm_ctc_ocr_b200 import engine
    rng = np.random.default_rng(9)
    N, W = 64, 400
    lw = (rng.integers(2, W // 4 + 1, size=N) * 4).astype(np.int32)
    lw[0], lw[1] = 8, W
    u = _pixels(N, W, lw.tolist(), 31)
    f = u.astype(np.float32) / F255
    for i in range(N):
        u[i, lw[i]:] = 255                         # bytes past each line's width are ignored
    tsl = (lw // 4 - 1).astype(np.int32)
    _, pn = TR._model("Adam", training=False)
    m = engine.CrnnModel(weight_decay=TR.WD, device=DEV, compute_dtype=dtype)
    m.load_params(pn)
    if stats == "moving":
        r = np.random.default_rng(4)
        m.load_bn_moving({k: (r.standard_normal(512) * 0.1 if "mean" in k else r.uniform(0.5, 2.0, 512)).astype(np.float32)
                          for k in engine.BN_MOVING_KEYS})
        m.set_bn_statistics("moving")
    d_lw, d_tsl = torch.tensor(lw, device=DEV), torch.tensor(tsl, device=DEV)
    if dtype == "fp8":
        m.calibrate_fp8(torch.tensor(f, device=DEV), d_tsl)
    snaps = []
    for data in (f, f, u):
        lg = m.forward_lines(torch.tensor(data, device=DEV), d_lw, d_tsl)
        s = {"logits": lg.clone()}
        s.update({"tap/" + k: m.tap(k, N, W).clone() for k in ("conv1", "conv2", "conv4_2", "lstm_out")})
        if stats == "batch":
            s.update({"raw/" + k: m.tap_raw(k, N, W, lines=True).clone() for k in ("bn", "stats")})
        snaps.append(s)
    _rule(f"lines/{dtype}/{stats}", snaps[2], snaps[0], snaps[1])


def test_calibrate_fp8_u8_gives_the_f32_scales():
    from lstm_ctc_ocr_b200 import engine
    u, f, _, _, tsl = _batch(256, 256, "cycle")
    _, pn = TR._model("Adam", training=False)
    m = engine.CrnnModel(weight_decay=TR.WD, device=DEV, compute_dtype="fp8")
    m.load_params(pn)
    d_tsl = torch.tensor(tsl, device=DEV)
    m.calibrate_fp8(torch.tensor(f, device=DEV), d_tsl)
    s_f = m.fp8_scales()
    m.set_fp8_scales(np.ones(5, np.float32))
    m.calibrate_fp8(torch.tensor(u, device=DEV), d_tsl)
    s_u = m.fp8_scales()
    assert s_f.tobytes() == s_u.tobytes(), (s_f, s_u)


@pytest.mark.parametrize("N,W,widths,seed", B.STAGE_SHAPES)
def test_training_forward_backward_u8(N, W, widths, seed, request):
    """Training forward, CTC gradient, backward_u8: every forward and backward stage and the 24 gradient tensors checked per
    element on the u8 run's operands (conv1's weight gradient against its 2.5e-5 acc bound), and the bit-identity rule against
    two f32 runs on zero-filled workspaces."""
    case = "train/" + request.node.callspec.id
    m, pn = TR._model("Adam")
    u, f, lab, ll, tsl = _batch(N, W, widths, seed=seed)
    ck = TR._checker("u8_feed/" + case)
    mu = U8Model(m)
    TR._fill_ws(m, N, W, 0)
    F_, _ = B._check_step(mu, pn, (f, lab, ll, tsl), case, dev=DEV, chunk=BB.CHUNK, ck=ck, ctc=TR._ctc_costs({}))
    assert mu.fed == 1
    fa, fb = TR._zero_runs(m, (f, lab, ll, tsl))                  # two f32 runs, seeded dlogits
    TR._fill_ws(m, N, W, 0)
    lg = TR._fwd_bwd(mu, (f, lab, ll, tsl))                       # the u8 run with the same dlogits
    TR._bit_identity(ck, TR._snapshot(m, N, W, lg, tsl), fa, fb)
    ck.assert_ok()


@pytest.mark.parametrize("solver", ["Adam", "Momentum", "RMS"])
def test_training_run_fed_u8(solver, monkeypatch):
    """test_gpu_training_run's five-step run per solver, every step fed uint8 (its per-step checks and bounds unchanged)."""
    calls = []

    def model(*a, **k):
        m, pn = _orig_model(*a, **k)
        calls.append(1)
        return U8Model(m), pn

    def batch(N, W, widths, seed=5):
        _, f, lab, ll, tsl = _batch(N, W, widths, seed=seed)
        return f, lab, ll, tsl

    _orig_model = TR._model
    monkeypatch.setattr(TR, "_model", model)
    monkeypatch.setattr(TR, "_batch", batch)
    TR.test_training_run_checks_every_stage_and_update(solver)
    assert calls


@pytest.mark.parametrize("solver", ["Adam", "RMS"])
def test_poisoned_workspace_between_steps_u8(solver, monkeypatch):
    """The NaN-filled-workspace runs of test_gpu_training_run, fed uint8: filled before the first forward and between steps."""
    def model(*a, **k):
        m, pn = _orig_model(*a, **k)
        return U8Model(m), pn

    def batch(N, W, widths, seed=5):
        _, f, lab, ll, tsl = _batch(N, W, widths, seed=seed)
        return f, lab, ll, tsl

    _orig_model = TR._model
    monkeypatch.setattr(TR, "_model", model)
    monkeypatch.setattr(TR, "_batch", batch)
    TR.test_poisoned_workspace_between_steps(solver, 130, 40, "cycle")
    m, pn = TR._model(solver)
    N, W = 130, 40
    b = batch(N, W, "cycle")
    ck = TR._checker(f"u8_feed/first_use/{solver}")
    TR._fill_ws(m.m, N, W, 255)
    F_, _ = B._check_step(m, pn, b, "first_use", dev=DEV, chunk=BB.CHUNK, ck=ck)
    ck.assert_ok()


# ---- Session.run ------------------------------------------------------------------------------------------------------------------
def _session_feeds(net, u, f, lab, ll, tsl):
    common = {net.labels: lab, net.labels_len: ll, net.time_step_len: tsl, net.keep_prob: 1.0}
    return {**common, net.data: f}, {**common, net.data_u8: u}


def _run_both(N, W, prep, train=False):
    """Three sessions on the same weights: f32, f32, u8 feeds of the same pixels.  prep(arr) -> the array to feed (its memory kind
    selects the feed path)."""
    from lstm_ctc_ocr_b200.lib.lstm.train import TrainOp, Variable
    from lstm_ctc_ocr_b200.lib.networks.LSTM_train import LSTM_train
    from lstm_ctc_ocr_b200.session import Session
    u, f, lab, ll, tsl = _batch(N, W, "cycle", seed=3)
    _, pn = TR._model("Adam", training=False)
    outs, paths, h2d = [], [], []
    for use_u8 in (False, False, True):
        net = LSTM_train()
        loss, dense = net.build_loss()
        with Session(device=DEV) as sess:
            sess.assign(net, pn)
            ff, fu = _session_feeds(net, u, f, lab, ll, tsl)
            feed = fu if use_u8 else ff
            key = net.data_u8 if use_u8 else net.data
            feed[key] = prep(feed[key])
            fetches = [loss, _fetch(net, "ctc_grad"), _fetch(net, "logits"), dense, _fetch(net, "layer:conv1")]
            if train:
                fetches.append(TrainOp(net, Variable(1e-3), Variable(0)))
            vals = sess.run(fetches, feed)
            paths.append(sess.last_feed_path)
            h2d.append(sess.h2d_bytes)
            o = {f"v{i}": torch.as_tensor(np.atleast_1d(np.asarray(v))) for i, v in enumerate(vals[:5])}
            if train:
                eng = sess.engine_for(net)
                o["params"] = eng.params.clone()
                o.update({"grad/" + k: eng.grad_tensor(k).clone() for k in eng.table})
            outs.append(o)
    return outs, paths, h2d, u


def _fetch(net, kind):
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    return Fetch(net, kind)


def _pinned_copy(a):
    t = torch.empty(a.shape, dtype=torch.from_numpy(np.asarray(a)).dtype).pin_memory()
    t.numpy()[...] = a
    return t.numpy()


@pytest.mark.parametrize("path", ["staged", "page-locked", "pageable"])
def test_session_run_data_u8(path):
    N, W = (64, 160) if path == "staged" else (1024, 256)
    prep = {"staged": np.ascontiguousarray, "page-locked": _pinned_copy, "pageable": lambda a: np.array(a, copy=True)}[path]
    outs, paths, h2d, u = _run_both(N, W, prep, train=(path != "pageable"))
    want = {"staged": "staged", "page-locked": "page-locked in place", "pageable": "staged"}[path]
    assert paths == [want] * 3, paths
    assert h2d[0] - h2d[2] == 3 * u.nbytes, h2d
    fa, fb, su = outs
    _rule(f"session/{path}", su, fa, fb)


def test_session_device_prefetch_u8():
    """A u8 PrefetchFeeder attached to the session: batches arrive through device prefetch (ahead_hits > 0) and give, step by
    step, the losses of two sessions fed the f32 quotient of the same bytes."""
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.LSTM_train import LSTM_train
    from lstm_ctc_ocr_b200.session import Session
    _, pn = TR._model("Adam", training=False)
    arg_fn = lambda k: dict(k=k, batch_size=256, render=False, seed=7, rank=0, world=1, width=160, dtype=np.uint8)  # noqa: E731
    feeder = gen.PrefetchFeeder(arg_fn, num_workers=0, depth=3, max_width=160, batch_size=256, keep=2)
    batches, got = [], []
    net = LSTM_train()
    loss, _ = net.build_loss()
    try:
        with Session(device=DEV) as sess:
            sess.assign(net, pn)
            sess.attach_feeder(feeder)
            for _ in range(4):
                data, lab, ll, tsl = next(feeder)
                assert data.dtype == np.uint8
                batches.append((data.copy(), lab, ll, tsl))
                got.append(np.float32(sess.run(loss, {net.data_u8: data, net.labels: lab, net.labels_len: ll, net.time_step_len: tsl})))
            assert sess.ahead_hits > 0 and "prefetch" in sess.last_feed_path
    finally:
        feeder.close()
    ref = []
    for _ in range(2):
        net = LSTM_train()
        loss, _ = net.build_loss()
        with Session(device=DEV) as sess:
            sess.assign(net, pn)
            ref.append([np.float32(sess.run(loss, {net.data: u.astype(np.float32) / F255, net.labels: lab, net.labels_len: ll,
                                                   net.time_step_len: tsl})) for u, lab, ll, tsl in batches])
    for a, b, c in zip(ref[0], ref[1], got):
        assert np.isfinite(c)
        if a.tobytes() == b.tobytes():
            assert c.tobytes() == a.tobytes(), (a, c)


def test_test_model_feed_dtype_uint8_same_decodes(tmp_path, monkeypatch):
    from lstm_ctc_ocr_b200.lib.lstm import test as T
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    mk = PE._load("make_decode10k", "tests", "golden", "make_decode10k.py")
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    PE._write_dir(str(tmp_path))
    weights = mk.load_weights()
    outs = {}
    old = cfg.FEED_DTYPE
    try:
        for fd in ("float32", "uint8"):
            cfg.FEED_DTYPE = fd
            net = get_network("LSTM_test")
            with Session(device=DEV) as sess:
                sess.assign(net, weights)
                sw = T.SolverWrapper(sess, net, None, str(tmp_path), None)
                buf = io.StringIO()
                with redirect_stdout(buf):
                    sw.test_model(sess, testDir=str(tmp_path), restore=False)
            outs[fd] = [ln for ln in buf.getvalue().splitlines() if "res:" in ln or ln.startswith("total acc")]
    finally:
        cfg.FEED_DTYPE = old
    assert outs["float32"] == outs["uint8"] and len(outs["uint8"]) > 60


# ---- status codes -----------------------------------------------------------------------------------------------------------------
def test_u8_status_codes_match_the_f32_twins():
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200._lib import c_size_t
    N, W = 4, 64
    u, f, _, _, tsl = _batch(N, W, "cycle")
    m, pn = TR._model("Adam", training=False)
    lib, h = m.lib, m.handle
    d_tsl = torch.tensor(tsl, device=DEV)
    du, df = torch.tensor(u, device=DEV), torch.tensor(f, device=DEV)
    ws, nbytes = m._workspace(N, W)
    out = torch.full((W // 4 - 1, N, 64), 7.0, device=DEV)
    s = lambda: engine._stream()  # noqa: E731

    def both(call):
        a, b = call(lib.crnn_forward, df.data_ptr()), call(lib.crnn_forward_u8, du.data_ptr())
        torch.cuda.synchronize()
        assert a == b != 0 and bool((out == 7.0).all()), (a, b)
        return a
    assert both(lambda fn, p: fn(h, 0, d_tsl.data_ptr(), N, W, out.data_ptr(), ws, nbytes, s())) == 1
    assert both(lambda fn, p: fn(h, p, d_tsl.data_ptr(), N, W - 2, out.data_ptr(), ws, nbytes, s())) == 1
    assert both(lambda fn, p: fn(h, p, d_tsl.data_ptr(), N, W, out.data_ptr(), ws, 1024, s())) == 5
    # misaligned uint8 data
    raw = torch.zeros(N * W * 32 + 4, dtype=torch.uint8, device=DEV)
    assert lib.crnn_forward_u8(h, raw.data_ptr() + 1, d_tsl.data_ptr(), N, W, out.data_ptr(), ws, nbytes, s()) == 1
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())
    # fp8 without scales
    m8 = engine.CrnnModel(weight_decay=TR.WD, device=DEV, compute_dtype="fp8")
    m8.load_params(pn)
    ws8, nb8 = m8._workspace(N, W)
    a = m8.lib.crnn_forward(m8.handle, df.data_ptr(), d_tsl.data_ptr(), N, W, out.data_ptr(), ws8, nb8, s())
    b = m8.lib.crnn_forward_u8(m8.handle, du.data_ptr(), d_tsl.data_ptr(), N, W, out.data_ptr(), ws8, nb8, s())
    assert a == b == 1 and bool((out == 7.0).all())
    # packed lines on a model in training mode
    m.set_training(True)
    lw = torch.full((N,), W, dtype=torch.int32, device=DEV)
    nbl = c_size_t()
    lib.crnn_lines_workspace_size(h, N, W, nbl)
    wsl = torch.empty(nbl.value + 1024, dtype=torch.uint8, device=DEV)
    p = (wsl.data_ptr() + 1023) // 1024 * 1024
    a = lib.crnn_forward_lines(h, df.data_ptr(), lw.data_ptr(), d_tsl.data_ptr(), N, W, out.data_ptr(), p, nbl.value, s())
    b = lib.crnn_forward_lines_u8(h, du.data_ptr(), lw.data_ptr(), d_tsl.data_ptr(), N, W, out.data_ptr(), p, nbl.value, s())
    assert a == b == 1 and bool((out == 7.0).all())
    # backward: misaligned pointer refused before the gradients are touched
    wst, nbt = m._workspace(N, W)
    m.forward(du, d_tsl)
    dl = TR._dlogits(N, W)
    m.grads.fill_(3.0)
    assert lib.crnn_backward_u8(h, raw.data_ptr() + 2, d_tsl.data_ptr(), dl.data_ptr(), N, W, wst, nbt, s()) == 1
    assert lib.crnn_backward(h, 0, d_tsl.data_ptr(), dl.data_ptr(), N, W, wst, nbt, s()) == \
        lib.crnn_backward_u8(h, 0, d_tsl.data_ptr(), dl.data_ptr(), N, W, wst, nbt, s()) == 1
    torch.cuda.synchronize()
    assert bool((m.grads == 3.0).all())
