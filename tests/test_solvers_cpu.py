"""The reference's Momentum and RMSProp solvers without a GPU: the fp64 restatements (tests/solver_refs.py) against TensorFlow's own
known answers, cfg.TRAIN.SOLVER dispatch as lib/lstm/train.py:74-76 does it, and the checkpoint slot keys / mismatch rule of
SolverWrapper.snapshot / restore on an engine whose buffers are CPU tensors.

Known answers [upstream-memory -- transcribed, not fetched: there is no network], TensorFlow 1.0.1:
  * tensorflow/python/training/momentum_test.py::MomentumOptimizerTest.testBasic: lr 2.0, momentum 0.9, var0 [1, 2] with grads
    [0.1, 0.1], var1 [3, 4] with grads [0.01, 0.01].  Step 1: var -= 2*g.  Step 2: every element moves a further (0.9*g + g)*2.
  * tensorflow/python/training/rmsprop_test.py (the no-momentum case): lr 2.0, decay 0.9, momentum 0.0, epsilon 1.0, same vars
    and grads.  Step 1: rms0 = 0.9*1.0 + 0.1*0.1^2 = 0.901 (rms1 = 0.90001) and var0 = 1 - 0.1*2/sqrt(0.901 + 1.0) -- the value
    that pins both the ones-initialised rms slot and epsilon INSIDE the square root (zeros or eps outside give other digits).
    Step 2: rms0 = 0.901*0.9 + 0.001, rms1 = 0.90001*0.9 + 1e-5, and each var moves a further g*2/sqrt(rms + 1.0)."""
import math
import os
import sys
import types
from collections import OrderedDict

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import solver_refs as R  # noqa: E402

LR = 2.0


def _kat_vars():
    t = lambda v: torch.tensor(v, dtype=torch.float64)
    params = OrderedDict(var0=t([1.0, 2.0]), var1=t([3.0, 4.0]))
    grads = OrderedDict(var0=t([0.1, 0.1]), var1=t([0.01, 0.01]))
    return params, grads


def _close(a, b):
    return np.abs(np.asarray(a, dtype=np.float64) - np.asarray(b, dtype=np.float64)).max() <= 1e-12


def test_momentum_reproduces_tensorflow_testBasic():
    params, grads = _kat_vars()
    slots = R.init_slots("Momentum", params)
    params, slots = R.apply("Momentum", params, grads, slots, 1, LR, momentum=0.9)
    assert _close(params["var0"], [1.0 - 0.1 * 2.0, 2.0 - 0.1 * 2.0])
    assert _close(params["var1"], [3.0 - 0.01 * 2.0, 4.0 - 0.01 * 2.0])
    assert _close(slots["accum"]["var0"], [0.1, 0.1]) and _close(slots["accum"]["var1"], [0.01, 0.01])
    params, slots = R.apply("Momentum", params, grads, slots, 2, LR, momentum=0.9)
    assert _close(params["var0"], [1.0 - 0.1 * 2.0 - (0.9 * 0.1 + 0.1) * 2.0, 2.0 - 0.1 * 2.0 - (0.9 * 0.1 + 0.1) * 2.0])
    assert _close(params["var1"], [3.0 - 0.01 * 2.0 - (0.9 * 0.01 + 0.01) * 2.0, 4.0 - 0.01 * 2.0 - (0.9 * 0.01 + 0.01) * 2.0])


def test_rmsprop_reproduces_tensorflow_known_answers():
    params, grads = _kat_vars()
    ms, mom = R.init_slots("RMS", params)["ms"], R.init_slots("RMS", params)["mom"]
    assert all(float(v.min()) == 1.0 for v in ms.values())          # TF's "rms" slot starts at ONE
    params, ms, mom = R.rmsprop_step(params, grads, ms, mom, LR, decay=0.9, momentum=0.0, epsilon=1.0)
    assert _close(ms["var0"], [0.901, 0.901]) and _close(ms["var1"], [0.90001, 0.90001])
    s0, s1 = 0.1 * 2.0 / math.sqrt(0.901 + 1.0), 0.01 * 2.0 / math.sqrt(0.90001 + 1.0)
    assert _close(params["var0"], [1.0 - s0, 2.0 - s0])
    assert _close(params["var1"], [3.0 - s1, 4.0 - s1])
    params, ms, mom = R.rmsprop_step(params, grads, ms, mom, LR, decay=0.9, momentum=0.0, epsilon=1.0)
    r0, r1 = 0.901 * 0.9 + 0.001, 0.90001 * 0.9 + 1e-5
    assert _close(ms["var0"], [r0, r0]) and _close(ms["var1"], [r1, r1])
    t0, t1 = 0.1 * 2.0 / math.sqrt(r0 + 1.0), 0.01 * 2.0 / math.sqrt(r1 + 1.0)
    assert _close(params["var0"], [1.0 - s0 - t0, 2.0 - s0 - t0])
    assert _close(params["var1"], [3.0 - s1 - t1, 4.0 - s1 - t1])


def test_rmsprop_known_answer_rejects_the_common_variants():
    """The step-1 vector tells TF's RMSProp apart from the Keras / PyTorch one (ms starting at 0, eps outside the root)."""
    g, lr, eps = 0.1, 2.0, 1.0
    tf = 1.0 - g * lr / math.sqrt(0.9 * 1.0 + 0.1 * g * g + eps)
    zeros_init = 1.0 - g * lr / math.sqrt(0.1 * g * g + eps)
    eps_outside = 1.0 - g * lr / (math.sqrt(0.9 * 1.0 + 0.1 * g * g) + eps)
    assert abs(tf - zeros_init) > 1e-3 and abs(tf - eps_outside) > 1e-3


def test_adam_train_step_is_the_oracle_train_step():
    """solver_refs.train_step(solver="Adam") gives what oracle.train_step gives (same loss, gradients, params and slots)."""
    from oracle import crnn_oracle as O
    pn = O.randomize_params(O.init_params(3, dtype=np.float64, logits_scale=10.0))
    batch = O.synth_batch(2, 24, seed=5)
    a = O.train_step(pn, batch, step=1, lr=1e-3)
    b = R.train_step(pn, batch, step=1, lr=1e-3, solver="Adam")
    assert a["loss"] == b["loss"] and a["grad_norm"] == b["grad_norm"]
    for k in pn:
        assert torch.equal(a["params"][k], b["params"][k])
        assert torch.equal(a["m"][k], b["slots"]["m"][k]) and torch.equal(a["v"][k], b["slots"]["v"][k])


# ---- cfg.TRAIN.SOLVER dispatch (train.py:74-76) -----------------------------------------------------------------------------------
@pytest.mark.parametrize("value,expected", [("Adam", "Adam"), ("RMS", "RMS"), ("Momentum", "Momentum"),
                                            ("SGD", "Momentum"), ("adam", "Momentum"), ("rms", "Momentum"), ("", "Momentum")])
def test_solver_config_dispatches_like_the_reference(value, expected):
    from lstm_ctc_ocr_b200.lib.lstm import train as T
    from lstm_ctc_ocr_b200.lib.lstm.config import AttrDict
    name, momentum = T.solver_from_cfg(AttrDict(SOLVER=value, MOMENTUM=0.75))
    assert name == expected and momentum == 0.75


def test_set_solver_override_on_the_command_line():
    from lstm_ctc_ocr_b200.lib.lstm import config as C, train as T
    old = dict(C.cfg.TRAIN)
    try:
        C.cfg_from_list(["TRAIN.SOLVER", "RMS"])
        assert T.solver_from_cfg(C.cfg.TRAIN)[0] == "RMS"
        C.cfg_from_list(["TRAIN.SOLVER", "Momentum", "TRAIN.MOMENTUM", "0.5"])
        assert T.solver_from_cfg(C.cfg.TRAIN) == ("Momentum", 0.5)
    finally:
        C.cfg.TRAIN.update(old)


# ---- engine solver state and checkpoints, with CPU tensors standing in for the device buffers -------------------------------------
class _FakeLib:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            return 0
        return fn


def _fake_engine(solver="Adam", momentum=0.9, training=True):
    from lstm_ctc_ocr_b200 import engine
    eng = engine.CrnnModel.__new__(engine.CrnnModel)
    eng.lib, eng.handle, eng.device = _FakeLib(), None, torch.device("cpu")
    eng.table = OrderedDict([("conv1/weights", (0, (3, 3, 1, 2))), ("logits/W", (18, (4, 2))), ("logits/b", (26, (2,)))])
    eng.total = 28
    eng.params = torch.arange(eng.total, dtype=torch.float32) * 0.25 - 3.0
    eng.grads = eng.adam_m = eng.adam_v = None
    eng.solver, eng.momentum = "Adam", 0.9
    if training:
        eng.grads = torch.zeros(eng.total)
        eng.adam_m, eng.adam_v = torch.zeros(eng.total), torch.zeros(eng.total)
    eng.set_solver(solver, momentum)
    return eng


class _FakeSess:
    def __init__(self, eng):
        self.eng = eng

    def engine_for(self, net):
        return self.eng


def _wrapper(eng, tmp_path):
    from lstm_ctc_ocr_b200.lib.lstm import train as T
    return T.SolverWrapper(_FakeSess(eng), object(), None, None, str(tmp_path), str(tmp_path))


@pytest.mark.parametrize("solver,m_fill,v_fill", [("Adam", 0.0, 0.0), ("Momentum", 0.0, 0.0), ("RMS", 0.0, 1.0)])
def test_set_solver_initialises_the_slots_as_tensorflow(solver, m_fill, v_fill):
    eng = _fake_engine()
    eng.adam_m.fill_(7.0); eng.adam_v.fill_(7.0)
    eng.set_solver(solver, 0.8)
    assert eng.solver == solver and eng.momentum == 0.8
    assert float(eng.adam_m.abs().max()) == m_fill and bool((eng.adam_v == v_fill).all())
    # slots allocated later (set_training) start from the same values
    late = _fake_engine(training=False)
    late.set_solver(solver)
    late.set_training(True)
    assert bool((late.adam_v == v_fill).all()) and float(late.adam_m.abs().max()) == 0.0


def test_unknown_solver_name_is_refused():
    from lstm_ctc_ocr_b200._lib import CrnnError
    with pytest.raises(CrnnError):
        _fake_engine().set_solver("Adagrad")


def test_apply_gradients_calls_the_entry_of_the_recorded_solver(monkeypatch):
    from lstm_ctc_ocr_b200 import engine
    monkeypatch.setattr(engine, "_stream", lambda: 0)
    want = {"Adam": ("crnn_clip_adam_step", (1e-3, 5.0, 7, 0.5, 2.0)),
            "Momentum": ("crnn_clip_momentum_step", (1e-3, 0.8, 5.0, 0.5, 2.0)),
            "RMS": ("crnn_clip_rmsprop_step", (1e-3, 0.9, 0.0, 1e-10, 5.0, 0.5, 2.0))}
    for solver, (name, args) in want.items():
        eng = _fake_engine(solver, momentum=0.8)
        eng.apply_gradients(1e-3, 7, clip=5.0, grad_mul=0.5, wd_mul=2.0)
        (called, got), = eng.lib.calls
        assert called == name and got[0] is None and got[-1] == 0
        assert np.allclose(np.float32(got[1:-1]), np.float32(args), rtol=0, atol=0), (solver, got)


@pytest.mark.parametrize("solver,keys", [("Adam", {"adam_m", "adam_v"}), ("Momentum", {"momentum"}), ("RMS", {"rms", "rms_momentum"})])
def test_snapshot_writes_the_solver_slot_keys_and_restore_reads_them_back(solver, keys, tmp_path):
    eng = _fake_engine(solver)
    rng = np.random.default_rng(1)
    eng.adam_m.copy_(torch.tensor(rng.standard_normal(eng.total), dtype=torch.float32))
    eng.adam_v.copy_(torch.tensor(rng.random(eng.total), dtype=torch.float32))
    path = _wrapper(eng, tmp_path).snapshot(_FakeSess(eng), 4)
    blob = np.load(path + ".npz")
    slot_keys = {f for f in blob.files if f.split("/", 1)[0] in {"adam_m", "adam_v", "momentum", "rms", "rms_momentum"}}
    assert slot_keys == {p + "/" + k for p in keys for k in eng.table}
    for prefix, buf in eng.solver_slots().items():
        off, shp = eng.table["logits/W"]
        assert np.array_equal(blob[prefix + "/logits/W"], buf[off:off + 8].view(*shp).numpy())
    if solver == "RMS":        # ms lives in adam_v, mom in adam_m
        assert np.array_equal(blob["rms/logits/b"], eng.adam_v[26:28].numpy())
        assert np.array_equal(blob["rms_momentum/logits/b"], eng.adam_m[26:28].numpy())
    fresh = _fake_engine(solver)
    _wrapper(fresh, tmp_path).restore(_FakeSess(fresh), path)
    assert torch.equal(fresh.params, eng.params)
    for prefix in keys:
        assert torch.equal(fresh.solver_slots()[prefix], eng.solver_slots()[prefix])


@pytest.mark.parametrize("solver", ["Adam", "Momentum", "RMS"])
def test_params_only_checkpoint_gives_fresh_slots(solver, tmp_path):
    eng = _fake_engine(solver)
    params_only = _fake_engine(solver, training=False)
    path = _wrapper(params_only, tmp_path).snapshot(_FakeSess(params_only), 0)
    assert not any("/" in f and f.split("/", 1)[0] in {"adam_m", "adam_v", "momentum", "rms", "rms_momentum"}
                   for f in np.load(path + ".npz").files)
    eng.adam_m.fill_(5.0); eng.adam_v.fill_(5.0)
    _wrapper(eng, tmp_path).restore(_FakeSess(eng), path)
    assert float(eng.adam_m.abs().max()) == 0.0
    assert bool((eng.adam_v == (1.0 if solver == "RMS" else 0.0)).all())


@pytest.mark.parametrize("saved,configured", [("Adam", "RMS"), ("Adam", "Momentum"), ("RMS", "Adam"), ("Momentum", "RMS"),
                                              ("RMS", "Momentum")])
def test_another_solvers_checkpoint_is_refused(saved, configured, tmp_path):
    from lstm_ctc_ocr_b200.lib.lstm import train as T
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    src = _fake_engine(saved)
    _wrapper(src, tmp_path).snapshot(_FakeSess(src), 9)
    eng = _fake_engine(configured)
    with pytest.raises(KeyError):
        _wrapper(eng, tmp_path).restore(_FakeSess(eng), os.path.join(str(tmp_path), "lstm_ctc_iter_10.ckpt"))
    # through the solver's resume path: the reference's "Check your pretrained" exception
    old = cfg.TRAIN.SOLVER
    cfg.TRAIN.SOLVER = configured
    try:
        eng = _fake_engine(saved)            # the engine last ran the other solver: _prepare switches it to the configured one
        eng._initialised = True
        sw = _wrapper(eng, tmp_path)
        with pytest.raises(Exception, match="Check your pretrained"):
            sw._prepare(_FakeSess(eng), True, T.Variable(1e-3), T.Variable(0))
        assert eng.solver == configured
    finally:
        cfg.TRAIN.SOLVER = old


def test_prepare_keeps_the_slots_of_an_unchanged_solver(tmp_path):
    """A second train_model on the same session continues with the slots it has (Adam's behaviour before Momentum / RMSProp)."""
    from lstm_ctc_ocr_b200.lib.lstm import train as T
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    old = (cfg.TRAIN.SOLVER, cfg.TRAIN.MOMENTUM)
    try:
        for solver in ("Adam", "Momentum", "RMS"):
            cfg.TRAIN.SOLVER, cfg.TRAIN.MOMENTUM = solver, 0.9
            eng = _fake_engine("Adam")
            eng._initialised = True
            sw = _wrapper(eng, tmp_path)
            sw._prepare(_FakeSess(eng), False, T.Variable(1e-3), T.Variable(0))
            assert eng.solver == solver and eng.momentum == 0.9
            eng.adam_m.fill_(3.0); eng.adam_v.fill_(4.0)
            sw._prepare(_FakeSess(eng), False, T.Variable(1e-3), T.Variable(0))
            assert bool((eng.adam_m == 3.0).all()) and bool((eng.adam_v == 4.0).all())
    finally:
        cfg.TRAIN.SOLVER, cfg.TRAIN.MOMENTUM = old


def test_c_entries_refuse_a_null_model_without_touching_the_device():
    """The new entry points exist in the library and validate before any CUDA call (runs on a machine without a GPU)."""
    from lstm_ctc_ocr_b200 import _lib
    L = _lib.load()
    assert L.crnn_version() >= 101
    assert L.crnn_clip_momentum_step(None, 1e-3, 0.9, 10.0, 1.0, 1.0, None) == 1
    assert L.crnn_clip_rmsprop_step(None, 1e-3, 0.9, 0.0, 1e-10, 10.0, 1.0, 1.0, None) == 1


@pytest.mark.parametrize("steps", [(1, 2, 3), (9998, 9999, 10000)])
def test_adam_restatement_equals_the_oracle_adam_step(steps):
    """solver_refs.adam_step (the per-element restatement the GPU Adam checks use) is the oracle's adam_step -- the formula of
    include/crnn_ctc.h, lr_t = lr*sqrt(1-b2^t)/(1-b1^t), theta -= lr_t*m/(sqrt(v)+1e-8) -- to 1e-12, with the bias correction
    far from 1 (steps 1 .. 3) and near it (9998 .. 10000), and its magnitudes bound every term."""
    from oracle import crnn_oracle as O
    rng = np.random.default_rng(4)
    shapes = OrderedDict(a=(64,), b=(7, 9))
    t = lambda a: torch.as_tensor(a, dtype=torch.float64)
    params = OrderedDict((k, t(rng.standard_normal(s) * 2e-2)) for k, s in shapes.items())
    p_o = OrderedDict((k, v.clone()) for k, v in params.items())
    m, v = R.init_slots("Adam", params)["m"], R.init_slots("Adam", params)["v"]
    m_o = OrderedDict((k, x.clone()) for k, x in m.items())
    v_o = OrderedDict((k, x.clone()) for k, x in v.items())
    for step in steps:
        grads = OrderedDict((k, t(rng.standard_normal(s) * 10.0 ** rng.uniform(-6, 0))) for k, s in shapes.items())
        params, m, v = R.adam_step(params, grads, m, v, step, 1e-3)
        p_o, m_o, v_o = O.adam_step(p_o, OrderedDict((k, g.clone()) for k, g in grads.items()), m_o, v_o, step, 1e-3)
        for k in shapes:
            for a, b in ((params[k], p_o[k]), (m[k], m_o[k]), (v[k], v_o[k])):
                assert float((a - b).abs().max()) <= 1e-12 * max(1.0, float(b.abs().max())), (step, k)
    # the f32 step size crnn_clip_adam_step passes: from the f32 lr, rounded to f32 once (two roundings of 2^-24 at most)
    for step in (1, 2, 1000, 10000):
        exact = 1e-3 * math.sqrt(1 - 0.999 ** step) / (1 - 0.9 ** step)
        assert R.adam_lr_t(1e-3, step, f32=False) == exact
        assert abs(R.adam_lr_t(1e-3, step) - exact) <= 2.0 ** -23 * exact
    # magnitudes: each holds |value| (and the f32 step of one element stays within a few units of it)
    g = np.array([1e-3, -2e-4, 0.0, 5.0])
    r = R.adam_update(np.array([0.02, -0.01, 0.0, 1.0]), g, np.array([1e-4, 1e-4, 0.0, -1.0]), np.array([1e-8, 0.0, 0.0, 1.0]),
                      R.adam_lr_t(1e-3, 3))
    for k, (val, mag) in r.items():
        assert (np.abs(val) <= mag + 1e-300).all(), k
