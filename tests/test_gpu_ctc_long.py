"""The workspace CTC kernel (ctc_long_kernel): labels up to 639 and any number of frames, on the GPU.

Per element against tests/ctc_refs.py's fp64 CTC at blanks 0, 17 and 63: costs relative to |cost|, the gradient per element
(ctc_grad_softmax, ctc_grad_posterior) and the workspace's stored lp and alpha tables teacher-forced, at
L in {64, 100, 255, 639} x T in {131, 260, 551, 1024, 2048}, at N = 1 and at N larger than one wave of CTAs.  Each batch
holds lengths 0, 1, T and T+5, all-repeat labels that just fit and that do not, a bad id and label_len > max_label_len.
Also: CRNN_CTC_KERNEL=long at the shapes of test_gpu_width_edges.py::test_ctc_at_its_frame_limits, bit-identical results
with and without a workspace inside the shared-memory limits, run to run, and at 4-byte offsets, the one-byte-short
refusal, and long rendered lines end to end through warpctc.ctc, Session.run and SolverWrapper.train_model.  Two controls
show the new stages see what the flat per-element bound they replaced did not.  Every measured bound is 4.5x its
measurement on an H100 80GB HBM3 (SXM), recorded in MEASURED and ctc_refs.MEASURED_POSTERIOR.

Rows go to build/ctc_long_report.jsonl."""
import os
import random
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ctc_refs as R  # noqa: E402
from stage_check import Checker  # noqa: E402
from stage_check import ulp_bf16  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
REPORT = "ctc_long_report.jsonl"

# Largest c needed over every case of test_long_kernel_against_fp64 and test_forced_long_kernel_at_the_frame_limits,
# H100 80GB HBM3 (SXM): (cost relative to |cost|, the flat per-element gradient bound in units of grad_scale that
# ctc_grad_softmax / ctc_grad_posterior replaced, the gradient's relative L2).  Like the shared-memory kernels'
# (test_gpu_width_edges.py), the gradient's error grows with T: the log2-space recursions round at every step.
# Measured: cost 2.80e-6 (L = 255), gradient 2.97e-2 (L = 64, T = 2048), relative L2 8.57e-3; the forced shapes of
# test_ctc_at_its_frame_limits (T <= 550) need 1.05e-6, 4.07e-3 and 7.2e-4.
MEASURED = {"long": (2.80e-6, 2.97e-2, 8.57e-3)}
BOUNDS = dict({f"ctc_cost/{k}": (0, 4.5 * v[0]) for k, v in MEASURED.items()},
              **R.bounds(["long"], {"long": 4.5 * R.MEASURED_POSTERIOR["long"]}))
L2 = {f"ctc_grad/{k}": max(1e-4, 4.5 * v[2]) for k, v in MEASURED.items()}
BLANKS = [0, 17, 63]
# SolverWrapper.train_model on rendered 30-70 character lines, 300 steps of 32 lines at lr 1e-3: mean loss of the last 50
# steps over the first 50 (228.8 -> 207.9).  The test asks only that it falls.
MEASURED_TRAIN_RATIO = 0.909


def _t(a):
    return torch.tensor(np.asarray(a), device=DEV)


def _batch(T, m, N, seed, blank=0):
    """Rows (label, input length): the longest label at T (with a repeated pair of 0 where 0 is not the blank), lengths
    0 / 1 / T+5, an empty label, all-repeat labels that just fit (2m-1 frames) and that do not, the blank inside a label,
    label_len = m+1, then random rows up to N.  Label ids over [0, 64) minus the blank.  N = 1: the first row only.
    Returns logits, flat labels, label lengths, unclamped input lengths."""
    rng = np.random.default_rng(seed)
    lab = lambda n: R.draw_labels(rng, n, blank)
    rep = int(lab(1)[0])
    first = lab(m)
    if blank != 0:
        first[1] = first[2] = 0
    rows = [(first, T), (lab(1), 0), (lab(1), 1),
            (np.zeros(0, np.int64), T), (np.full(m, rep), min(T, 2 * m - 1)), (np.full(m, rep), min(T, 2 * m - 2)),
            (lab(m), T + 5), (np.r_[lab(m - 1), blank], T), (lab(m + 1), T)]
    while len(rows) < N:
        L = int(rng.integers(0, m + 1))
        rows.append((lab(L), int(rng.integers(1, T + 6))))
    rows = rows[:N]
    lab = np.concatenate([r[0] for r in rows]).astype(np.int32)
    ll = np.array([len(r[0]) for r in rows], np.int32)
    il = np.array([r[1] for r in rows], np.int32)
    x = (rng.standard_normal((T, N, 64)) * 2.0).astype(np.float32)
    return x, lab, ll, il


def _run(x, lab, ll, il, m, scale, workspace="auto", logits=None, grad=None, costs=None, blank=0):
    from lstm_ctc_ocr_b200 import engine
    lg = _t(x) if logits is None else logits
    grad = torch.empty_like(lg) if grad is None else grad
    costs, grad = engine.ctc_loss(lg, _t(lab), _t(ll), _t(il), blank=blank, want_grad=True, grad_scale=scale, max_label_len=m,
                                  costs=costs, grad=grad, workspace=workspace)
    torch.cuda.synchronize()
    return costs, grad


def _workspace(T, N, m):
    from lstm_ctc_ocr_b200 import engine
    return torch.empty(engine.ctc_workspace_bytes(T, N, 64, m), dtype=torch.uint8, device=DEV)


def run_and_check(ck, x, lab, ll, il, m, blank, kind="long"):
    """ctc_long_kernel on a workspace of its own at grad_scale 1/N: the costs and gradient against ctc_refs.ctc_fp64, then
    the workspace's stored lp and alpha tables teacher-forced (ctc_refs.check_long_workspace).  Returns (costs, grad, ref)."""
    N = x.shape[1]
    ws = _workspace(x.shape[0], N, m)
    lg = _t(x) if isinstance(x, np.ndarray) else x
    costs, grad = _run(None, lab, ll, il, m, 1.0 / N, workspace=ws, logits=lg, blank=blank)
    ref = R.ctc_fp64(lg, lab, ll, il, blank=blank, grad_scale=1.0 / N, max_label_len=m)
    R.check_grad(ck, kind, costs, grad, ref, 1.0 / N)
    R.check_long_workspace(ck, kind, ws, lg, costs, ref, blank, m)
    return costs, grad, ref


@pytest.mark.parametrize("blank", BLANKS)
@pytest.mark.parametrize("m", [64, 100, 255, 639])
def test_long_kernel_against_fp64(m, blank):
    """Every T of the grid at N = 1 and N = 300 (more than the CTAs of one wave: two 320-thread CTAs per SM at 96 registers)."""
    from lstm_ctc_ocr_b200 import engine
    ck = Checker(f"ctc_long_m{m}_b{blank}", BOUNDS, REPORT, ulp_bf16, L2)
    for T in (131, 260, 551, 1024, 2048):
        assert engine.ctc_workspace_bytes(T, 300, 64, m) > 0
        for N in (1, 300):
            x, lab, ll, il = _batch(T, m, N, seed=T + m + N + blank, blank=blank)
            run_and_check(ck, x, lab, ll, il, m, blank)
            torch.cuda.empty_cache()
    ck.assert_ok()


def test_forced_long_kernel_at_the_frame_limits(monkeypatch):
    """CRNN_CTC_KERNEL=long at the shapes test_ctc_at_its_frame_limits runs (its batches), at each blank of BLANKS: the
    same stages, one report case per blank."""
    import test_gpu_width_edges as WE
    monkeypatch.setenv("CRNN_CTC_KERNEL", "long")
    fail = []
    for blank in BLANKS:
        ck = Checker(f"ctc_long_forced_b{blank}", BOUNDS, REPORT, ulp_bf16, L2)
        for m in (4, 15, 31, 63):
            for T in WE._frame_limit_Ts(m):
                x, lab, ll, il = WE._ctc_batch(T, m, seed=T + m, blank=blank)
                run_and_check(ck, x, lab, ll, il, m, blank)
        ck.report()
        fail += [f"blank {blank}: {f}" for f in ck.fail]
    assert not fail, "\n".join(fail)


def test_controls_fail_the_new_stages_and_pass_the_flat_bound():
    """On the long kernel's own output at T = 2048: half of grad_scale * P moved onto the blank column, for the label-class
    elements with 1e-3 < P below the flat bound the per-element stages replaced, fails ctc_grad_posterior and passes that
    flat bound; 1e-3 added to one stored alpha entry fails ctc_long_alpha_step."""
    m, T, N, blank = 64, 2048, 4, 0
    x, lab, ll, il = _batch(T, m, N, seed=11, blank=blank)
    ck = Checker("ctc_long_control_clean", BOUNDS, REPORT, ulp_bf16, L2)
    costs, grad, ref = run_and_check(ck, x, lab, ll, il, m, blank)
    assert not ck.fail, ck.fail
    flat = 4.5 * MEASURED["long"][1] / N
    cls = ref["inlab"].clone()
    cls[:, blank] = False
    live = (torch.arange(T, device=DEV)[:, None] < ref["Tn"][None]) & ref["feasible"][None]
    sel = live[..., None] & cls[None] & (ref["P"] > 1e-3) & (ref["P"] / N < flat)
    assert int(sel.sum()) > 100
    bad = grad.clone()
    move = torch.where(sel, 0.5 * ref["P"] / N, torch.zeros_like(ref["P"]))
    move *= move.sum(2, keepdim=True) <= flat / 2             # frames whose blank moves by at most half the flat bound
    assert int((move > 0).sum()) > 100
    bad += move.float()                            # less posterior mass taken off the label classes ...
    bad[..., blank] -= move.sum(2).float()         # ... and as much more taken off the blank
    ck = Checker("ctc_long_control_moved", BOUNDS, REPORT, ulp_bf16, L2)
    R.check_grad(ck, "long", costs, bad, ref, 1.0 / N)
    ck.report()
    failed = {f.split(":")[0] for f in ck.fail}
    print("moved posterior mass fails:", ck.fail)
    assert f"ctc_grad_posterior/long/T{T}" in failed and not any(f.startswith("ctc_grad_softmax") for f in failed)
    assert float((bad.double() - ref["grad"]).abs().max()) <= flat
    # one stored alpha entry 1e-3 off
    ws = _workspace(T, N, m)
    costs, grad = _run(x, lab, ll, il, m, 1.0 / N, workspace=ws, blank=blank)
    _, al = R.long_workspace_views(ws, T, N, m)
    al[0, 8, 3] += 1e-3                            # an early frame: |alpha| ~ 50, where 1e-3 is ~2000 ulps
    ck = Checker("ctc_long_control_alpha", BOUNDS, REPORT, ulp_bf16, L2)
    R.check_long_workspace(ck, "long", ws, _t(x), costs, ref, blank, m)
    ck.report()
    assert {f.split(":")[0].split("/")[0] for f in ck.fail} == {"ctc_long_alpha_step"}, ck.fail


def test_workspace_changes_no_bits_inside_the_shared_memory_limits(monkeypatch):
    """Shapes a shared-memory kernel serves (each dispatch choice, aligned and 4 bytes off): a workspace, even a large one,
    leaves every bit as it is without one."""
    import test_gpu_width_edges as WE
    ws = torch.empty(64 << 20, dtype=torch.uint8, device=DEV)
    for m in (4, 15, 31, 63):
        for T in WE._frame_limit_Ts(m)[:2] + [WE.CEILING[m]]:
            x, lab, ll, il = WE._ctc_batch(T, m, seed=T + m)
            for env in ({}, {"CRNN_CTC_KERNEL": "tma"}, {"CRNN_CTC_KERNEL": "generic"}):
                monkeypatch.delenv("CRNN_CTC_KERNEL", raising=False)
                for k, v in env.items():
                    monkeypatch.setenv(k, v)
                if WE.kernel_for(T, m, env.get("CRNN_CTC_KERNEL", "fast")) is None:
                    continue
                c0, g0 = _run(x, lab, ll, il, m, 0.25, workspace=None)
                c1, g1 = _run(x, lab, ll, il, m, 0.25, workspace=ws)
                c2, g2 = _run(x, lab, ll, il, m, 0.25, workspace="auto")
                assert torch.equal(c0, c1) and torch.equal(g0, g1) and torch.equal(c0, c2) and torch.equal(g0, g2), (m, T, env)
            monkeypatch.delenv("CRNN_CTC_KERNEL", raising=False)
            if WE.kernel_for(T, m, aligned=False) is not None:
                buf = torch.empty(x.size + 4, device=DEV)
                lg = buf[1:1 + x.size].view(x.shape)
                lg.copy_(_t(x))
                c0, g0 = _run(x, lab, ll, il, m, 0.25, workspace=None, logits=lg)
                c1, g1 = _run(x, lab, ll, il, m, 0.25, workspace=ws, logits=lg)
                assert torch.equal(c0, c1) and torch.equal(g0, g1), (m, T, "misaligned")


def _same_bits(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))        # NaN costs compare equal bit for bit


def test_long_kernel_is_bit_identical_run_to_run_and_at_4_byte_offsets():
    m, T, N = 639, 2048, 300
    x, lab, ll, il = _batch(T, m, N, seed=7)
    c0, g0 = _run(x, lab, ll, il, m, 1.0 / N)
    c1, g1 = _run(x, lab, ll, il, m, 1.0 / N)
    assert _same_bits(c0, c1) and _same_bits(g0, g1)
    m, T, N = 100, 551, 40
    x, lab, ll, il = _batch(T, m, N, seed=8)
    c0, g0 = _run(x, lab, ll, il, m, 1.0 / N)
    buf = torch.empty(x.size + 4, device=DEV)
    lg = buf[1:1 + x.size].view(x.shape)
    lg.copy_(_t(x))
    assert lg.data_ptr() % 16 == 4
    c, g = _run(x, lab, ll, il, m, 1.0 / N, logits=lg)
    assert _same_bits(c, c0) and _same_bits(g, g0)
    gbuf = torch.empty(x.size + 4, device=DEV)
    c, g = _run(x, lab, ll, il, m, 1.0 / N, grad=gbuf[1:1 + x.size].view(x.shape))
    assert _same_bits(c, c0) and _same_bits(g, g0)
    # a caller's workspace at any byte offset
    from lstm_ctc_ocr_b200 import engine
    need = engine.ctc_workspace_bytes(T, N, 64, m)
    wbuf = torch.empty(need + 3, dtype=torch.uint8, device=DEV)
    c, g = _run(x, lab, ll, il, m, 1.0 / N, workspace=wbuf[3:])
    assert _same_bits(c, c0) and _same_bits(g, g0)
    # costs only
    costs, none = engine.ctc_loss(_t(x), _t(lab), _t(ll), _t(il), max_label_len=m, workspace="auto")
    torch.cuda.synchronize()
    assert none is None and _same_bits(costs, c0)


def test_a_workspace_one_byte_short_is_refused_and_leaves_the_outputs():
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200._lib import CrnnError
    for m, T in ((100, 260), (15, 600), (639, 131)):
        x, lab, ll, il = _batch(T, m, 12, seed=3)
        need = engine.ctc_workspace_bytes(T, 12, 64, m)
        for ws in (None, torch.empty(need - 1, dtype=torch.uint8, device=DEV)):
            costs = torch.full((12,), 1234.5, device=DEV)
            grad = torch.full(x.shape, -7.0, device=DEV)
            with pytest.raises(CrnnError, match=f"CRNN_UNSUPPORTED.*{need} bytes") as e:
                _run(x, lab, ll, il, m, 1.0, workspace=ws, grad=grad, costs=costs)
            if m <= 63:
                assert f"T = {T}" in str(e.value)
            assert bool((costs == 1234.5).all()) and bool((grad == -7.0).all())
        c, _ = _run(x, lab, ll, il, m, 1.0, workspace=torch.empty(need, dtype=torch.uint8, device=DEV))
        assert bool(torch.isfinite(c[0]))


# ------------------------------------------------------------------------------------------------------- end to end
def _long_lines(n, seed):
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    rng = random.Random(seed)
    labels = [gen.gen_rand(rng, 30, 70) for _ in range(n)]
    return gen.groupBatch([gen.render_line(t, rng=rng) for t in labels], labels)


def test_warpctc_and_session_on_rendered_long_lines():
    from lstm_ctc_ocr_b200 import synthetic, warpctc
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    assert gen.can_render()
    imgs, lab, ll, tsl = _long_lines(16, seed=4)
    data = np.array(imgs)
    assert max(ll) > 63 or data.shape[1] // 4 - 1 > 130
    # warpctc.ctc on logits of the real network
    net = get_network("LSTM_train")
    with Session(device=DEV) as sess:
        sess.assign(net, synthetic.init_params(3, logits_scale=4.0))
        from lstm_ctc_ocr_b200.lib.networks.network import Fetch
        loss, costs_op = net.build_loss()[0], Fetch(net, "ctc_costs")
        feed = {net.data: data, net.labels: np.array(lab, np.int32), net.time_step_len: np.array(tsl, np.int32),
                net.labels_len: np.array(ll, np.int32), net.keep_prob: 1.0}
        logits = sess.run(net.get_output("logits"), feed_dict=feed)
        T = logits.shape[0]
        x = torch.tensor(logits, device=DEV, requires_grad=True)
        c = warpctc.ctc(x, np.array(lab, np.int32), np.array(ll, np.int32), np.array(tsl, np.int32))
        c.sum().backward()
        ref = R.ctc_fp64(x.detach(), np.array(lab, np.int32), np.array(ll, np.int32), np.array(tsl, np.int32))
        assert bool(ref["feasible"].all())
        ck = Checker("warpctc_long_lines", BOUNDS, REPORT, ulp_bf16, L2)
        R.check_grad(ck, "long", c.detach(), x.grad, ref, 1.0)
        ck.assert_ok()
        with pytest.raises(ValueError, match="639"):
            warpctc.ctc(x.detach(), np.ones(640, np.int32), np.array([640] + [0] * (len(ll) - 1), np.int32),
                        np.full(len(ll), T, np.int32))
        # Session.run's loss and costs on the same feed: the same kernel on the same logits (train_op is exercised by
        # test_train_model_on_30_to_70_character_lines)
        lv, cv = sess.run([loss, costs_op], feed_dict=feed)
        assert np.array_equal(cv, c.detach().cpu().numpy())
        assert np.isfinite(lv) and float(lv) >= float(cv.mean())


def test_train_model_on_30_to_70_character_lines(tmp_path):
    """SolverWrapper.train_model with --set MIN_LEN 30 MAX_LEN 70 through the real feeder (gen.get_batch): every loss finite,
    the late mean below the early mean."""
    from lstm_ctc_ocr_b200.lib.lstm import train as TR
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    assert gen.can_render()
    keys = ("LEARNING_RATE", "DISPLAY", "SNAPSHOT_ITERS", "BATCH_SIZE")
    old = {k: cfg.TRAIN[k] for k in keys}
    old_len, old_val = (cfg.MIN_LEN, cfg.MAX_LEN), cfg.VAL.VAL_STEP
    cfg.TRAIN.LEARNING_RATE, cfg.TRAIN.DISPLAY, cfg.TRAIN.SNAPSHOT_ITERS, cfg.TRAIN.BATCH_SIZE = 1e-3, 100, 10 ** 9, 32
    cfg.MIN_LEN, cfg.MAX_LEN, cfg.VAL.VAL_STEP = 30, 70, 10 ** 9
    feeder = gen.get_batch(num_workers=12, batch_size=32, seed=77)
    try:
        assert feeder.max_width == gen.line_width_bound(70) > 256
        held = [_long_lines(8, seed=990)]
        net = get_network("LSTM_train")
        with Session(device=DEV) as sess:
            sw = TR.SolverWrapper(sess, net, None, None, str(tmp_path), str(tmp_path))
            hist = sw.train_model(sess, 301, restore=False, train_gen=feeder, val_gen=iter(held))
        hist = np.array(hist)
        assert len(hist) == 300 and np.isfinite(hist).all()
        ratio = float(hist[-50:].mean() / hist[:50].mean())
        print(f"train_model 30-70 chars: early {hist[:50].mean():.3f} late {hist[-50:].mean():.3f} ratio {ratio:.3f}")
        assert ratio < 1.0
    finally:
        feeder.close()
        for k in keys:
            cfg.TRAIN[k] = old[k]
        cfg.MIN_LEN, cfg.MAX_LEN = old_len
        cfg.VAL.VAL_STEP = old_val
