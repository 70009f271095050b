"""The reference's three solvers on the GPU (csrc/backward_kernels.cu clip_adam_kernel / clip_momentum_kernel / clip_rmsprop_kernel
behind crnn_clip_adam_step / crnn_clip_momentum_step / crnn_clip_rmsprop_step), against the fp64 restatements of tests/solver_refs.py, which
tests/test_solvers_cpu.py pins to TensorFlow's own known answers.

Per-element check of one update: the reference step is computed in fp64 from the kernel's own inputs (the f32 parameters, slots
and raw gradients read back just before the call), so the only differences are f32 rounding.  Each element's error is expressed
in units of u = 2^-24 times the sum of the magnitudes of the terms that make up that element (e.g. |p| + lr*(|accum*momentum| +
|g|) for a Momentum parameter): the largest such c over the whole 7 158 592-element buffer is MEASURED below, on one H100 80GB
HBM3 (SXM), and the enforced bound is 4.5x it."""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import solver_refs as R  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24

# Largest c (in u of the term magnitudes) per quantity over the three steps of test_update_matches_fp64_per_element, H100 80GB HBM3
# (SXM).  BOUND = 4.5x.
MEASURED = {"Momentum": {"params": 1.74, "accum": 1.95}, "RMS": {"params": 2.45, "ms": 0.67, "mom": 4.13},
            "Adam": {"params": 4.49, "adam_m": 2.85, "adam_v": 5.33}}
BOUND = {s: {k: 4.5 * v for k, v in d.items()} for s, d in MEASURED.items()}
# every run appends what it needed to build/solver_report.jsonl (re-measure from there)
REPORT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build", "solver_report.jsonl")


def _report(rec):
    os.makedirs(os.path.dirname(REPORT), exist_ok=True)
    with open(REPORT, "a") as f:
        f.write(json.dumps(rec) + "\n")


def _model(wd=1e-5):
    from lstm_ctc_ocr_b200 import engine
    from oracle import crnn_oracle as O
    pn = O.randomize_params(O.init_params(3, dtype=np.float32, logits_scale=10.0))
    m = engine.CrnnModel(weight_decay=wd, device=DEV)
    m.load_params(pn)
    m.set_training(True)
    return m


def _l2_mask(m):
    from oracle import crnn_oracle as O
    mask = np.zeros(m.total, dtype=bool)
    for k in O.L2_NAMES:
        off, shp = m.table[k]
        mask[off:off + int(np.prod(shp))] = True
    return mask


def _state(m):
    return {"params": m.params.clone(), "adam_m": m.adam_m.clone(), "adam_v": m.adam_v.clone()}


def _load_state(m, s):
    m.params.copy_(s["params"]); m.adam_m.copy_(s["adam_m"]); m.adam_v.copy_(s["adam_v"])


def _f64(t):
    return t.detach().cpu().numpy().astype(np.float64)


def _reference(solver, s, raw, mask, wd, lr, clip, momentum=0.9, decay=0.9, rms_momentum=0.0, eps=1e-10, step=1):
    """fp64 step from the f32 state `s`, the raw gradients and the f32 hyper-parameters the kernel receives: returns
    ({quantity: (value, magnitude of the terms that make it up)}, global norm).  Adam: `step` is the 1-based global step, the
    step size, b1, b2 and eps those crnn_clip_adam_step passes (solver_refs.adam_lr_t, f32 0.9 / 0.999 / 1e-8)."""
    f32 = lambda x: float(np.float32(x))
    wd, lr, clip, momentum, decay, rms_momentum, eps = (f32(x) for x in (wd, lr, clip, momentum, decay, rms_momentum, eps))
    p0 = _f64(s["params"])
    wdp = np.where(mask, wd * p0, 0.0)
    gf = raw + wdp
    gn = math.sqrt(float((gf * gf).sum()))
    scale = clip / max(gn, clip) if clip > 0 else 1.0
    g, g_mag = gf * scale, (np.abs(raw) + np.abs(wdp)) * scale
    if solver == "Adam":
        return R.adam_update(p0, g, _f64(s["adam_m"]), _f64(s["adam_v"]), R.adam_lr_t(lr, step), f32(R.ADAM_B1), f32(R.ADAM_B2),
                             f32(R.ADAM_EPS), g_mag=g_mag), gn
    if solver == "Momentum":
        a0 = _f64(s["adam_m"]) * momentum
        a = a0 + g
        a_mag = np.abs(a0) + g_mag
        return {"accum": (a, a_mag), "params": (p0 - lr * a, np.abs(p0) + lr * a_mag)}, gn
    ms0, mom0 = _f64(s["adam_v"]), _f64(s["adam_m"]) * rms_momentum
    ms = ms0 + (g * g - ms0) * (1.0 - decay)
    root = np.sqrt(ms + eps)
    mom = mom0 + lr * g / root
    mom_mag = np.abs(mom0) + lr * g_mag / root
    return {"ms": (ms, np.abs(ms0) + g_mag * g_mag), "mom": (mom, mom_mag), "params": (p0 - mom, np.abs(p0) + mom_mag)}, gn


def _c_needed(ref, m, solver):
    got = {"params": m.params, "accum": m.adam_m, "mom": m.adam_m, "ms": m.adam_v, "adam_m": m.adam_m, "adam_v": m.adam_v}
    out = {}
    for k, (val, mag) in ref.items():
        err = np.abs(_f64(got[k]) - val)
        out[k] = float((err / (U * np.maximum(mag, 1e-30))).max())
    return out


def _call(m, solver, lr, clip, grad_mul, wd_mul, hp, step=1):
    """One update: through apply_gradients with the reference's hyper-parameters at global step `step`, or straight through the
    C entry for `hp` (Adam: {"step": global step})."""
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200._lib import check
    if hp is None:
        m.apply_gradients(lr, step, clip=clip, grad_mul=grad_mul, wd_mul=wd_mul)
    elif solver == "Adam":
        check(m.lib.crnn_clip_adam_step(m.handle, lr, clip, hp["step"], grad_mul, wd_mul, engine._stream()))
    elif solver == "Momentum":
        check(m.lib.crnn_clip_momentum_step(m.handle, lr, hp["momentum"], clip, grad_mul, wd_mul, engine._stream()))
    else:
        check(m.lib.crnn_clip_rmsprop_step(m.handle, lr, hp["decay"], hp["rms_momentum"], hp["eps"], clip, grad_mul, wd_mul,
                                           engine._stream()))


# the third step of test_update_matches_fp64_per_element: through the C entry with other hyper-parameters (Adam: a global step
# whose bias correction is near 1)
THIRD_STEP = {"Adam": {"step": 10000}, "Momentum": {"momentum": 0.5}, "RMS": {"decay": 0.8, "rms_momentum": 0.5, "eps": 1e-3}}


@pytest.mark.parametrize("solver", ["Adam", "Momentum", "RMS"])
def test_update_matches_fp64_per_element(solver):
    """Whole buffer, weight decay on: step 1 clips (raw norm ~ 8e3), step 2 does not (norm ~ 2.7), lr changes between them, and a
    third step runs the C entry with other hyper-parameters (Adam at global step 10000, where the bias correction lr_t / lr is
    0.99998, against 0.316 at step 1 and 0.795 at step 1000 / Momentum 0.5 / RMSProp decay 0.8, momentum 0.5, epsilon 1e-3).  The simulated
    data-parallel call -- gradients x2, grad_mul 0.5, wd_mul 2, i.e. a SUM over two equal ranks -- equals the single-device
    call bit for bit."""
    wd, clip = 1e-5, 10.0
    m = _model(wd)
    m.set_solver(solver, momentum=0.9)
    mask = _l2_mask(m)
    rng = np.random.default_rng(7)
    steps = [(1e-3, 3.0, None), (4e-4, 1e-3, None), (2e-4, 1e-3, THIRD_STEP[solver])]
    worst = {}
    for i, (lr, gscale, hp) in enumerate(steps):
        raw = (rng.standard_normal(m.total) * gscale).astype(np.float32)
        s = _state(m)
        m.grads.copy_(torch.from_numpy(raw).to(DEV))
        _call(m, solver, lr, clip, 1.0, 1.0, hp, step=i + 1)
        single = _state(m)
        gn_gpu = m.last_grad_norm()
        _load_state(m, s)
        m.grads.copy_(torch.from_numpy(raw * 2).to(DEV))
        _call(m, solver, lr, clip, 0.5, 2.0, hp, step=i + 1)
        for k in single:
            assert torch.equal(single[k], getattr(m, k)), (solver, i, k)
        assert m.last_grad_norm(0.5) == gn_gpu
        kw = hp or ({"momentum": 0.9} if solver == "Momentum" else {"step": i + 1} if solver == "Adam" else {})
        ref, gn = _reference(solver, s, raw.astype(np.float64), mask, wd, lr, clip, **kw)
        assert (gn > clip) == (i == 0), gn
        assert abs(gn_gpu - gn) / gn < 1e-5, (gn_gpu, gn)
        for k, c in _c_needed(ref, m, solver).items():
            worst[k] = max(worst.get(k, 0.0), c)
    _report({"test": "per_element", "solver": solver, "c_needed": worst})
    for k, c in worst.items():
        assert c <= BOUND[solver][k], (solver, k, c, BOUND[solver][k])


def test_adam_through_apply_gradients_is_clip_adam_step_bit_for_bit():
    """Under the default solver, apply_gradients is today's Adam step: same parameters and slots, bit for bit."""
    m = _model()
    assert m.solver == "Adam"
    rng = np.random.default_rng(3)
    m.adam_m.copy_(torch.from_numpy(rng.standard_normal(m.total).astype(np.float32) * 1e-3).to(DEV))
    m.adam_v.copy_(torch.from_numpy(rng.random(m.total).astype(np.float32) * 1e-6).to(DEV))
    for step, gscale in ((3, 3.0), (4, 1e-3)):
        raw = torch.from_numpy((rng.standard_normal(m.total) * gscale).astype(np.float32)).to(DEV)
        s = _state(m)
        m.grads.copy_(raw)
        m.clip_adam_step(1e-3, step, clip=10.0)
        want = _state(m)
        _load_state(m, s)
        m.grads.copy_(raw)
        m.apply_gradients(1e-3, step, clip=10.0)
        for k in want:
            assert torch.equal(want[k], getattr(m, k)), (step, k)


def _setup_batch(N, W, widths, wd):
    from lstm_ctc_ocr_b200 import engine
    from oracle import crnn_oracle as O
    pn = O.randomize_params(O.init_params(3, dtype=np.float32, logits_scale=10.0))
    batch = O.synth_batch(N, W, seed=5, widths=widths)
    m = engine.CrnnModel(weight_decay=wd, device=DEV)
    m.load_params(pn)
    m.set_training(True)
    return m, pn, batch


def _gpu_grads(m, batch):
    from lstm_ctc_ocr_b200 import engine
    data, lab, ll, tsl = batch
    t = lambda a: torch.tensor(a, device=DEV)
    d_data, d_tsl = t(data), t(tsl)
    logits = m.forward(d_data, d_tsl)
    costs, grad = engine.ctc_loss(logits, t(lab), t(ll), d_tsl, want_grad=True, grad_scale=1.0 / data.shape[0], max_label_len=int(ll.max()))
    m.backward(d_data, d_tsl, grad)
    return costs


@pytest.mark.parametrize("solver", ["Momentum", "RMS"])
def test_three_training_steps_track_the_oracle(solver):
    """Forward, CTC, backward and the solver step three times, next to the fp64 oracle graph with the same solver (the bounds of
    the Adam version in test_gpu_training.py)."""
    wd, lr = 1e-5, 1e-3
    m, pn, batch = _setup_batch(8, 88, [88, 85, 60, 33, 88, 88, 70, 52], wd=wd)
    m.set_solver(solver, momentum=0.9)
    po = {k: v.astype(np.float64) for k, v in pn.items()}
    slots = None
    for step in (1, 2, 3):
        out = R.train_step(po, batch, slots, step=step, lr=lr, wd=wd, solver=solver, momentum=0.9)
        po = {k: v.numpy() for k, v in out["params"].items()}; slots = out["slots"]
        costs = _gpu_grads(m, batch)
        loss = float(m.total_loss(costs).item())
        m.apply_gradients(lr, step)
        assert abs(loss - out["loss"]) / out["loss"] < 1e-2, (step, loss, out["loss"])
        gn = m.last_grad_norm()
        assert abs(gn - out["grad_norm"]) / out["grad_norm"] < 0.08
    num = den_a = den_b = 0.0
    for k in m.table:
        da = m.tensor(k).cpu().numpy().astype(np.float64) - pn[k]
        db = po[k] - pn[k]
        num += (da * db).sum(); den_a += (da * da).sum(); den_b += (db * db).sum()
    assert num / math.sqrt(den_a * den_b) > 0.9


# lr per solver for the fixed-batch overfit: Adam's test uses 1e-3; Momentum runs at the reference's default LEARNING_RATE (0.01,
# lib/lstm/config.py), RMSProp, which normalises the step as Adam does, at Adam's 1e-3.
LEARN_LR = {"Momentum": 1e-2, "RMS": 1e-3}
SLOT_KEYS = {"Momentum": ("momentum",), "RMS": ("rms", "rms_momentum")}


@pytest.mark.parametrize("solver", ["Momentum", "RMS"])
def test_solver_loop_learns_snapshots_and_resumes(solver, tmp_path, capsys):
    """SolverWrapper.train_model with TRAIN.SOLVER = Momentum / RMS overfits one fixed batch like the Adam loop does; the snapshot
    holds the solver's slot keys; a restore gives back the saved arrays byte for byte; a resumed run continues the loss; an Adam
    checkpoint resumed under RMS (or Momentum) is refused."""
    from lstm_ctc_ocr_b200 import synthetic
    from lstm_ctc_ocr_b200.lib.lstm import train as T
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    keys = ("LEARNING_RATE", "DISPLAY", "SNAPSHOT_ITERS", "WEIGHT_DECAY", "SOLVER", "MOMENTUM")
    old = {k: cfg.TRAIN[k] for k in keys}
    cfg.TRAIN.LEARNING_RATE, cfg.TRAIN.DISPLAY, cfg.TRAIN.SNAPSHOT_ITERS, cfg.TRAIN.WEIGHT_DECAY = LEARN_LR[solver], 10, 20, 1e-5
    cfg.TRAIN.SOLVER, cfg.TRAIN.MOMENTUM = solver, 0.9
    try:
        data, lab, ll, tsl = synthetic.synth_batch(16, 88, seed=21, widths=[85] * 16)
        fixed = (list(data), lab.tolist(), ll.tolist(), tsl.tolist())

        def gen():
            while True:
                yield fixed
        net = get_network("LSTM_train")
        with Session(device=DEV) as sess:
            sw = T.SolverWrapper(sess, net, None, None, str(tmp_path), str(tmp_path))
            hist = sw.train_model(sess, 41, restore=False, train_gen=gen(), val_gen=gen())
            _report({"test": "learn", "solver": solver, "lr": LEARN_LR[solver], "first": hist[0], "last": hist[-1]})
            assert len(hist) == 40 and hist[-1] < 0.8 * hist[0], (hist[0], hist[-1])
            eng = sess.engine_for(net)
            assert eng.solver == solver
            ck = sw._latest_checkpoint()
            assert ck.endswith("lstm_ctc_iter_40.ckpt") and os.path.exists(ck + ".npz")
            blob = np.load(ck + ".npz")
            assert int(blob["global_step"]) == 39
            slot_files = {f for f in blob.files if "/" in f and f.split("/", 1)[0] in {"adam_m", "adam_v", "momentum", "rms", "rms_momentum"}}
            assert slot_files == {p + "/" + k for p in SLOT_KEYS[solver] for k in eng.table}
            sw.restore(sess, ck)
            now = sess.variables(net)
            for k in now:
                assert np.array_equal(blob[k], now[k])
            for prefix, buf in eng.solver_slots().items():
                for k, (off, shp) in eng.table.items():
                    got = buf[off:off + int(np.prod(shp))].view(*shp).cpu().numpy()
                    assert got.tobytes() == blob[prefix + "/" + k].tobytes(), (prefix, k)
            hist2 = sw.train_model(sess, 43, restore=True, train_gen=gen(), val_gen=gen())
            assert len(hist2) == 3 and hist2[0] < 0.9 * hist[0]
            # an Adam checkpoint (Adam slots only) resumed with this solver configured: refused, as TF's Saver would refuse it
            eng.set_solver("Adam")
            sw.snapshot(sess, 49)
            with pytest.raises(Exception, match="Check your pretrained"):
                sw.train_model(sess, 52, restore=True, train_gen=gen(), val_gen=gen())
        out = capsys.readouterr().out
        assert "iter: 10 / 41, total loss:" in out and "Wrote snapshot to:" in out
    finally:
        for k in keys:
            cfg.TRAIN[k] = old[k]


def test_bad_arguments_and_missing_slots_return_the_documented_codes():
    from lstm_ctc_ocr_b200 import engine
    INVALID, NOT_BOUND = 1, 3
    m = _model()
    m.grads.normal_()
    L, h, st = m.lib, m.handle, engine._stream()
    before = {k: getattr(m, k).clone() for k in ("params", "grads", "adam_m", "adam_v")}

    def untouched():
        torch.cuda.synchronize()
        return all(torch.equal(before[k], getattr(m, k)) for k in before)
    mom = lambda *a: L.crnn_clip_momentum_step(h, *a, st)
    rms = lambda *a: L.crnn_clip_rmsprop_step(h, *a, st)
    nan = float("nan")
    assert mom(1e-3, -0.1, 10.0, 1.0, 1.0) == INVALID
    assert mom(1e-3, nan, 10.0, 1.0, 1.0) == INVALID
    for decay, momentum, eps in ((-0.01, 0.0, 1e-10), (1.01, 0.0, 1e-10), (nan, 0.0, 1e-10), (0.9, -0.5, 1e-10), (0.9, 0.0, -1e-10)):
        assert rms(1e-3, decay, momentum, eps, 10.0, 1.0, 1.0) == INVALID, (decay, momentum, eps)
    assert untouched()
    # slots not bound
    L.crnn_model_bind(h, m.params.data_ptr(), m.grads.data_ptr(), None, None)
    assert mom(1e-3, 0.9, 10.0, 1.0, 1.0) == NOT_BOUND
    assert rms(1e-3, 0.9, 0.0, 1e-10, 10.0, 1.0, 1.0) == NOT_BOUND
    L.crnn_model_bind(h, m.params.data_ptr(), m.grads.data_ptr(), m.adam_m.data_ptr(), None)
    assert rms(1e-3, 0.9, 0.0, 1e-10, 10.0, 1.0, 1.0) == NOT_BOUND            # RMSProp's ms lives in adam_v
    assert untouched()
    # no crnn_model_set_training: buffers bound, but the gradient-norm scratch was never allocated
    fresh = engine.CrnnModel(weight_decay=1e-5, device=DEV)
    bufs = [torch.zeros_like(fresh.params) for _ in range(3)]
    L.crnn_model_bind(fresh.handle, fresh.params.data_ptr(), *(b.data_ptr() for b in bufs))
    assert L.crnn_clip_momentum_step(fresh.handle, 1e-3, 0.9, 10.0, 1.0, 1.0, st) == INVALID
    assert L.crnn_clip_rmsprop_step(fresh.handle, 1e-3, 0.9, 0.0, 1e-10, 10.0, 1.0, 1.0, st) == INVALID
    assert not bool(fresh.params.any())
    # Momentum needs adam_m only: with adam_v unbound it runs, and crnn_last_grad_norm reports its norm
    assert mom(1e-3, 0.9, 10.0, 1.0, 1.0) == 0
    assert not torch.equal(before["params"], m.params) and m.last_grad_norm() > 0
    assert torch.equal(before["adam_v"], m.adam_v)
    m._bind()


# ---- two GPUs (skipped with fewer) ---------------------------------------------------------------------------------------------
def _equiv_worker(rank, world, port, ret, solver):
    """Sharded batch + global-batch BatchNorm + bucketed gradient exchange + the solver step == the single-device step."""
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from lstm_ctc_ocr_b200 import engine, parallel, synthetic
    dev = torch.device("cuda", rank)
    params = synthetic.init_params(3, logits_scale=10.0)
    Ng, W = 32, 128
    data, lab, ll, tsl = synthetic.synth_batch(Ng, W, seed=31, widths=np.random.default_rng(1).integers(40, W + 1, size=Ng))
    tt = lambda a: torch.tensor(a, device=dev)

    def run(m, d, l, n, t):
        dd, dt = tt(d), tt(t)
        logits = m.forward(dd, dt)
        costs, grad = engine.ctc_loss(logits, tt(l), tt(n), dt, want_grad=True, grad_scale=1.0 / d.shape[0], max_label_len=int(n.max()))
        m.backward(dd, dt, grad)
        return logits, costs
    ref = engine.CrnnModel(weight_decay=1e-5, device=dev)
    ref.load_params(params); ref.set_solver(solver); ref.set_training(True)
    lg_ref, _ = run(ref, data, lab, ll, tsl)
    g_ref = ref.grads.clone()
    ref.apply_gradients(1e-3, 1)
    p_ref = ref.params.clone()
    m = engine.CrnnModel(weight_decay=1e-5, device=dev)
    m.load_params(params); m.set_solver(solver); m.set_training(True)
    dp = parallel.DataParallel(m, sync_bn=True, overlap=True, peer_memory=True)
    d, l, n, t = parallel.shard_batch(data, lab, ll, tsl, rank, world)
    for rep in range(3):
        lg, _ = run(m, d, l, n, t)
        dp.reduce_gradients()
        torch.cuda.synchronize()
    assert dp.peer_error() == 0
    per = Ng // world
    e_fwd = float((lg - lg_ref[:, rank * per:(rank + 1) * per]).abs().max() / lg_ref.abs().max())
    g = m.grads / world
    e_grad = float((g - g_ref).norm() / g_ref.norm())
    m.apply_gradients(1e-3, 1, grad_mul=1.0 / world, wd_mul=float(world))
    e_par = float((m.params - p_ref).abs().max())
    gathered = [torch.empty_like(m.params) for _ in range(world)]
    dist.all_gather(gathered, m.params)
    same = all(torch.equal(gathered[0], x) for x in gathered)
    slots = [torch.empty_like(m.adam_m) for _ in range(world)]
    dist.all_gather(slots, m.adam_m)
    same = same and all(torch.equal(slots[0], x) for x in slots)
    ret[rank] = (e_fwd, e_grad, e_par, same)
    dp.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("solver", ["Momentum", "RMS"])
def test_sharded_batch_equals_single_device_step(solver):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    mp.set_start_method("spawn", force=True)
    mgr = mp.Manager()
    ret = mgr.dict()
    port = 29900 + (os.getpid() % 1000) + (1 if solver == "RMS" else 0)
    procs = [mp.Process(target=_equiv_worker, args=(r, 2, port, ret, solver)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    for r in range(2):
        e_fwd, e_grad, e_par, same = ret[r]
        assert e_fwd < 2e-3 and e_grad < 2e-2 and e_par < 2e-3 and same, ret[r]
