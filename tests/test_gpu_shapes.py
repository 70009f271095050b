"""Parity at the BENCHMARKED shapes (need the GPU).

VERDICT r1 weak #2 / ADVICE r1: the round-1 forward tests stopped at W <= 160 and the gradient tests at W in {88, 40, 100},
which never take the merged 128-position TMA boxes of the conv GEMMs (`mg2/mg3/mg4`: H1 % 8, H2 % 16, H2 % 32) nor the
64-position boxes of the weight-gradient GEMMs (`wm2/wm3/wm4`: H1 % 4, H2 % 8, H2 % 16) -- exactly the paths the 32x256
benchmark runs.  The cases below make every one of those flags true (and false) at least once:

      W    H1   H2   mg2 mg3 mg4   wm2 wm3 wm4
     256  128   64    1   1   1     1   1   1     BASELINE configs[2] / [3] / [4] width
     160   80   40    1   0   0     1   1   0     BASELINE configs[1] / [3] width
     128   64   32    1   1   1     1   1   1
      96   48   24    1   0   0     1   1   0
      80   40   20    1   0   0     1   0   0     BASELINE configs[3] width
      64   32   16    1   1   0     1   1   1

Every compared tensor's error is also appended to build/parity_report.jsonl (rel = max|a-b| / max|b|, l2 = relative L2)."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def rel_l2(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def report(test, **kv):
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    with open(os.path.join(ROOT, "build", "parity_report.jsonl"), "a") as f:
        f.write(json.dumps(dict(test=test, **kv)) + "\n")


# tolerances of the bf16-operand / f32-accumulate path against the fp64 oracle: max-abs error relative to max|reference|
# (every run appends the measured errors to build/parity_report.jsonl; lstm_out's bound is the max over 5 M elements of a
#  tanh-bounded tensor whose L2 error is about 1 %)
FWD_TOL = {"conv1": 4e-3, "conv2": 6e-3, "conv3_1": 6e-3, "conv3_2": 8e-3, "conv4_1": 2e-2, "conv4_2": 3.5e-2,
           "conv5": 2.5e-2, "lstm_out": 9e-2, "logits": 2.5e-2}
# ... and in relative L2 (the error averaged over the tensor)
FWD_TOL_L2 = {"conv1": 2.5e-3, "conv2": 3.5e-3, "conv3_1": 3.5e-3, "conv3_2": 4e-3, "conv4_1": 1.5e-2, "conv4_2": 2.2e-2,
              "conv5": 2.2e-2, "lstm_out": 1.6e-2, "logits": 1.6e-2}

SHAPES = [
    pytest.param(2, 256, [256, 201], id="c3_width_N2"),
    pytest.param(32, 256, None, id="c3_width_N32"),
    pytest.param(256, 160, None, id="c2_shape_N256_W160"),
    pytest.param(3, 128, [128, 100, 77], id="W128"),
    pytest.param(3, 96, [96, 95, 41], id="W96"),
    pytest.param(5, 80, [80, 77, 64, 33, 9], id="W80"),
    pytest.param(4, 64, [64, 61, 30, 64], id="W64"),
]


@pytest.mark.parametrize("N,W,widths", SHAPES)
def test_forward_layers_vs_oracle_at_benchmark_shapes(N, W, widths, request):
    """Every tap, the logits and the loss against the fp64 oracle at the benchmarked widths (32x256: configs[2]; 256x32x160:
    configs[1]; 80/160/256: configs[3]) -- the merged-box TMA paths of every conv GEMM."""
    from lstm_ctc_ocr_b200 import engine
    from oracle import crnn_oracle as O
    pn = O.randomize_params(O.init_params(3, dtype=np.float32, logits_scale=10.0))
    data, lab, ll, tsl = O.synth_batch(N, W, seed=5, widths=widths, min_len=1, max_len=6)
    m = engine.CrnnModel(device=DEV)
    m.load_params(pn)
    t = lambda a: torch.tensor(a, device=DEV)
    logits = m.forward(t(data), t(tsl))
    lo, acts = O.forward(O.to_torch(pn), data, tsl, return_all=True)
    T = W // 4 - 1
    got = {k: m.tap(k, N, W).cpu().numpy() for k in ("conv1", "conv2", "conv3_1", "conv3_2", "conv4_1", "conv4_2")}
    got["conv5"] = m.tap("conv5", N, W).cpu().numpy()[:, :T]
    got["lstm_out"] = m.tap("lstm_out", N, W).cpu().numpy()[:, :T]
    got["logits"] = logits.cpu().numpy()
    ref = {k: acts[k].permute(0, 2, 3, 1).numpy() for k in ("conv1", "conv2", "conv3_1", "conv3_2", "conv4_1", "conv4_2")}
    ref["conv5"] = acts["reshaped_layer"].numpy()
    ref["lstm_out"] = acts["lstm_out"].numpy()
    ref["logits"] = lo.numpy()
    errs = {k: (rel(got[k], ref[k]), rel_l2(got[k], ref[k])) for k in FWD_TOL}
    costs, _ = engine.ctc_loss(logits, t(lab), t(ll), t(tsl))
    co, _ = O.ctc_loss_np(lo.numpy(), lab, ll, tsl)
    loss_o = co.mean() + float(O.l2_reg(O.to_torch(pn), 1e-5))
    loss = float(m.total_loss(costs).item())
    report("forward", case=request.node.callspec.id, N=N, W=W, loss_rel=abs(loss - loss_o) / loss_o,
           **{k: {"rel": round(v[0], 6), "l2": round(v[1], 6)} for k, v in errs.items()})
    for k, (e, e2) in errs.items():
        assert e < FWD_TOL[k] and e2 < FWD_TOL_L2[k], (k, e, e2)
    assert abs(loss - loss_o) / loss_o < 5e-3


GRAD_SHAPES = [
    pytest.param(2, 256, [256, 201], id="c3_width"),
    pytest.param(3, 160, [160, 131, 160], id="c2_width"),
    pytest.param(3, 128, [128, 100, 77], id="W128"),
    pytest.param(3, 96, [96, 95, 41], id="W96"),
    pytest.param(4, 64, [64, 61, 30, 64], id="W64"),
]
# per-tensor gradient tolerance (relative L2 vs fp64 autograd).  bf16 activations AND bf16 gradient tensors between the
# layers: the error accumulates with depth from the logits to conv1; the bound is per layer group, cosine >= 0.99 everywhere.
def grad_tol(name):
    for key, tol in (("conv1/", 0.14), ("conv2/", 0.10), ("conv3_", 0.085), ("conv4_", 0.07), ("conv5/", 0.03),
                     ("lstm_cell", 0.05), ("logits/", 0.02)):
        if key in name:
            return tol
    return 0.10


GRAD_COS = 0.99


@pytest.mark.parametrize("N,W,widths", GRAD_SHAPES)
def test_gradients_vs_oracle_autograd_at_benchmark_widths(N, W, widths, request):
    """All 24 gradient tensors vs fp64 autograd at widths that take the merged dgrad boxes and the 64-position wgrad boxes."""
    from lstm_ctc_ocr_b200 import engine
    from oracle import crnn_oracle as O
    pn = O.randomize_params(O.init_params(3, dtype=np.float32, logits_scale=10.0))
    batch = O.synth_batch(N, W, seed=5, widths=widths)
    m = engine.CrnnModel(weight_decay=0.0, device=DEV)
    m.load_params(pn)
    m.set_training(True)
    out = O.train_step({k: v.astype(np.float64) for k, v in pn.items()}, batch, wd=0.0)
    data, lab, ll, tsl = batch
    t = lambda a: torch.tensor(a, device=DEV)
    d_data, d_tsl = t(data), t(tsl)
    logits = m.forward(d_data, d_tsl)
    costs, grad = engine.ctc_loss(logits, t(lab), t(ll), d_tsl, want_grad=True, grad_scale=1.0 / N, max_label_len=int(ll.max()))
    m.backward(d_data, d_tsl, grad)
    rows = {}
    bad = []
    for name in m.table:
        g = m.grad_tensor(name).cpu().numpy().astype(np.float64)
        go = out["grads"][name].numpy()
        if np.linalg.norm(go) < 1e-9:         # conv4_x biases: exactly cancelled by the batch-stat BN that follows
            # analytically zero: what the GPU holds is the bf16 rounding noise of the column sums of d(pre-BN) -- bounded against
            # the size of the same layer's beta gradient (the column sums before the BN-backward projection)
            scale = float(np.abs(out["grads"][name.replace("biases", name.split("/")[0] + "/beta")].numpy()).max())
            rows[name] = {"abs_max": round(float(np.abs(g).max()), 5), "beta_grad_max": round(scale, 4)}
            assert np.abs(g).max() < 0.05 * max(scale, 1.0), (name, float(np.abs(g).max()), scale)
            continue
        r = np.linalg.norm(g - go) / np.linalg.norm(go)
        c = float((g * go).sum() / (np.linalg.norm(g) * np.linalg.norm(go)))
        rows[name] = {"l2": round(float(r), 5), "cos": round(c, 6)}
        if not (c >= GRAD_COS and r <= grad_tol(name)):
            bad.append((name, r, c))
    report("gradients", case=request.node.callspec.id, N=N, W=W, tensors=rows)
    assert not bad, bad


def test_ctc_rejects_invalid_labels_per_sample():
    """SURVEY 8(b) / ADVICE r1 (ctc.cu:425,511): a label id >= C, < 0 or == blank makes THAT sample's cost NaN with an all-zero
    gradient row block; it is never used as an index (neighbouring samples are bit-identical to a clean run)."""
    from lstm_ctc_ocr_b200 import engine
    rng = np.random.default_rng(1)
    T, N = 24, 8
    x = torch.tensor(rng.standard_normal((T, N, 64)).astype(np.float32), device=DEV)
    ll = np.full(N, 4, np.int32); il = np.full(N, T, np.int32)
    lab = rng.integers(1, 63, size=4 * N).astype(np.int32)
    t = lambda a: torch.tensor(a, device=DEV)
    for which in ("fast", "tma", "generic"):
        if which != "fast":
            os.environ["CRNN_CTC_KERNEL"] = which
        try:
            c0, g0 = engine.ctc_loss(x, t(lab), t(ll), t(il), want_grad=True)
            bad = lab.copy()
            bad[4 * 2 + 1] = 64           # sample 2: id == C
            bad[4 * 5 + 3] = -7           # sample 5: negative
            bad[4 * 6 + 0] = 0            # sample 6: the blank itself
            bad[4 * 7 + 2] = 1 << 20      # sample 7: far out of range
            c1, g1 = engine.ctc_loss(x, t(bad), t(ll), t(il), want_grad=True)
            torch.cuda.synchronize()
        finally:
            os.environ.pop("CRNN_CTC_KERNEL", None)
        for n in range(N):
            if n in (2, 5, 6, 7):
                assert torch.isnan(c1[n]) and not g1[:, n].any()
            else:
                assert torch.equal(c1[n], c0[n]) and torch.equal(g1[:, n], g0[:, n])
    from lstm_ctc_ocr_b200 import warpctc
    with pytest.raises(ValueError):
        warpctc.ctc(x, bad, ll, il)                      # host arrays: validated before the launch
    with pytest.raises(ValueError):
        warpctc.ctc(x, lab[:-1], ll, il)                 # flat_labels shorter than sum(label_lengths)
    from lstm_ctc_ocr_b200._lib import CrnnError
    with pytest.raises(CrnnError):
        engine.ctc_loss(x, t(bad), t(ll), t(il), validate=True)


def test_learning_rate_step_and_resume_of_a_decayed_rate(tmp_path):
    """Row a15 (train.py:114-115): lr *= GAMMA every STEPSIZE iterations; the decayed rate is stored in the snapshot and
    restored on resume (train.py:96-106)."""
    from lstm_ctc_ocr_b200 import synthetic
    from lstm_ctc_ocr_b200.lib.lstm import train as T
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    keys = ("LEARNING_RATE", "DISPLAY", "SNAPSHOT_ITERS", "STEPSIZE", "GAMMA")
    old = {k: cfg.TRAIN[k] for k in keys}
    cfg.TRAIN.LEARNING_RATE, cfg.TRAIN.DISPLAY, cfg.TRAIN.SNAPSHOT_ITERS, cfg.TRAIN.STEPSIZE, cfg.TRAIN.GAMMA = 1e-3, 100, 7, 3, 0.5
    try:
        data, lab, ll, tsl = synthetic.synth_batch(8, 40, seed=21)
        fixed = (list(data), lab.tolist(), ll.tolist(), tsl.tolist())

        def gen():
            while True:
                yield fixed
        net = get_network("LSTM_train")
        with Session(device=DEV) as sess:
            sw = T.SolverWrapper(sess, net, None, None, str(tmp_path), str(tmp_path))
            sw.train_model(sess, 8, restore=False, train_gen=gen(), val_gen=gen())       # iterations 1..7: decays at 3 and 6
            assert abs(sw._lr.eval() - 1e-3 * 0.25) < 1e-12
            blob = np.load(sw._latest_checkpoint() + ".npz")                            # written at iter 6 ((6+1) % 7 == 0)
            assert abs(float(blob["lr"]) - 1e-3 * 0.25) < 1e-12
            sw.train_model(sess, 10, restore=True, train_gen=gen(), val_gen=gen())      # resumes at 7 with the decayed rate ...
            assert abs(sw._lr.eval() - 1e-3 * 0.125) < 1e-12                            # ... and decays once more at 9
    finally:
        for k in keys:
            cfg.TRAIN[k] = old[k]


def test_network_load_npy_dict(tmp_path):
    """Network.load (network.py:50-63): npy dict {scope: {var: array}} -> variables, `ignore_missing` semantics."""
    from lstm_ctc_ocr_b200 import synthetic
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    params = synthetic.init_params(9)
    nested = {}
    for k, v in params.items():
        scope, var = k.rsplit("/", 1)
        nested.setdefault(scope, {})[var] = v
    np.save(str(tmp_path / "w.npy"), nested, allow_pickle=True)
    net = get_network("LSTM_test")
    with Session(device=DEV) as sess:
        net.load(str(tmp_path / "w.npy"), sess)
        got = sess.variables(net)
        for k in params:
            assert np.array_equal(got[k], params[k]), k
        del nested["conv5"]
        np.save(str(tmp_path / "w2.npy"), nested, allow_pickle=True)
        with pytest.raises(KeyError):
            net.load(str(tmp_path / "w2.npy"), sess)
        net.load(str(tmp_path / "w2.npy"), sess, ignore_missing=True)


def test_session_feeds_from_the_page_locked_feeder_and_beam_decodes():
    """SURVEY 8(f)2 + 8(f)4 through the solver-facing call: batches from a PrefetchFeeder ring slot are DMA'd in place
    (crnn_forward_host, no staging copy), results equal the staged path; cfg.DECODER='beam' returns the reference's
    beam-search decode of the same logits (== the oracle's restatement)."""
    from lstm_ctc_ocr_b200 import synthetic
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    from oracle import crnn_oracle as O
    net = get_network("LSTM_train")
    loss, dense_decoded = net.build_loss()
    arg_fn = lambda k: dict(k=k, batch_size=64, render=True, seed=11, rank=0, world=1, bucket=gen.BUCKETS[k % 3])
    f = gen.PrefetchFeeder(arg_fn, num_workers=2, depth=3, max_width=256, batch_size=64)
    try:
        assert f.pinned
        with Session(device=DEV) as sess:
            sess.assign(net, synthetic.init_params(3, logits_scale=10.0))
            for k in range(4):
                view, lab, ll, tsl = next(f)
                feed = {net.data: view, net.labels: np.array(lab), net.time_step_len: np.array(tsl), net.labels_len: np.array(ll),
                        net.keep_prob: 1.0}
                l1, dec1, logits1 = sess.run([loss, dense_decoded, net.get_output("logits")], feed_dict=feed)
                assert sess.last_feed_path == "page-locked in place"
                feed[net.data] = np.array(view)                                     # pageable copy -> staged path
                l2, dec2 = sess.run([loss, dense_decoded], feed_dict=feed)
                assert sess.last_feed_path == "staged"
                assert abs(l1 - l2) <= 2e-3 * abs(l2) and dec1.shape[0] == 64
                if k == 0:
                    cfg.DECODER = "beam"
                    try:
                        decb = sess.run(dense_decoded, feed_dict=feed)
                    finally:
                        cfg.DECODER = "greedy"
                    ref = O.dense_decoded(O.beam_search_decode(logits1, np.array(tsl)))
                    # logits1 comes from the in-place run, decb from the staged run: BN-statistic atomics order may differ in
                    # the last bits, so compare per line and allow a handful of near-tie lines
                    same = sum([v for v in decb[i] if v] == [v for v in ref[i] if v] for i in range(64))
                    assert same >= 62, same
    finally:
        f.close()


def test_session_device_prefetch_overlaps_the_next_batch_and_changes_nothing():
    """Session.attach_feeder: the NEXT ring slot is copied host->device on a side stream while the current step runs; every step
    after the first finds its input resident, and losses / decodes equal those of a session fed without the prefetch."""
    from lstm_ctc_ocr_b200 import synthetic
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    net = get_network("LSTM_train")
    loss, dense_decoded = net.build_loss()
    arg_fn = lambda k: dict(k=k, batch_size=64, render=False, seed=21, rank=0, world=1, bucket=gen.BUCKETS[k % 3])
    results = {}
    for mode in ("plain", "prefetch"):
        f = gen.PrefetchFeeder(arg_fn, num_workers=2, depth=3, max_width=256, batch_size=64, keep=2)
        try:
            with Session(device=DEV) as sess:
                sess.assign(net, synthetic.init_params(3, logits_scale=10.0))
                if mode == "prefetch":
                    sess.attach_feeder(f)
                out = []
                for k in range(7):
                    view, lab, ll, tsl = next(f)
                    feed = {net.data: view, net.labels: np.array(lab), net.time_step_len: np.array(tsl), net.labels_len: np.array(ll),
                            net.keep_prob: 1.0}
                    l, dec = sess.run([loss, dense_decoded], feed_dict=feed)
                    out.append((float(l), dec.copy(), sess.last_feed_path))
                    if mode == "prefetch" and k == 3:
                        # a batch fed out of order (not the feeder's) must not pick up the staged copy
                        other = np.ascontiguousarray(view[::-1])
                        feed_o = dict(feed)
                        feed_o[net.data] = other
                        l_o = sess.run(loss, feed_dict=feed_o)
                        assert sess.last_feed_path == "staged" and np.isfinite(l_o)
                results[mode] = (out, sess.ahead_hits)
        finally:
            f.close()
    plain, pre = results["plain"][0], results["prefetch"][0]
    assert results["plain"][1] == 0
    assert results["prefetch"][1] >= 5, results["prefetch"][1]           # steps 1..3 and 5..6 (step 4's copy was dropped by the out-of-order run)
    assert all("device prefetch" in p[2] for p in pre[1:4])
    for a, b in zip(plain, pre):
        assert abs(a[0] - b[0]) <= 1e-3 * abs(a[0])                         # BN-statistic atomics may differ in the last bits
        assert a[1].shape == b[1].shape and (a[1] == b[1]).mean() > 0.99


def test_pageable_batches_go_through_the_host_copy_pool_and_change_nothing():
    """crnn_forward_pageable (what Session.run does with the reference's np.array(...)-per-step feeds, lib/lstm/train.py:119-125): the
    library's host threads move the batch into page-locked staging range by range; logits equal those of the resident-input forward
    bit for bit except for the order of the BN-statistic atomics, for 1 and for 4 ranges, at a size that does and one that does not
    split on tile boundaries."""
    from lstm_ctc_ocr_b200 import engine, synthetic
    m = engine.CrnnModel(device=DEV)
    m.load_params(synthetic.init_params(3, logits_scale=10.0))
    for N, W in ((64, 256), (6, 100)):
        data, _, _, tsl = synthetic.synth_batch(N, W, seed=9)
        d_tsl = torch.tensor(tsl, device=DEV)
        ref = m.forward(torch.tensor(data, device=DEV), d_tsl).clone()
        pin = torch.empty(data.size, dtype=torch.float32).pin_memory()
        for chunks, threads in ((1, 1), (4, 3), (4, 8)):
            pin.fill_(-7.0)
            src = np.array(data)                                            # fresh pageable copy, as the reference's solver builds
            out, d_data, cst = m.forward_pageable(src, pin, d_tsl, chunks=chunks, host_threads=threads)
            torch.cuda.synchronize()
            assert np.array_equal(pin[:data.size].numpy().reshape(data.shape), data)
            assert torch.equal(d_data.cpu(), torch.from_numpy(data))
            err = float((out - ref).abs().max() / ref.abs().max())
            assert err < 1e-3, (N, W, chunks, threads, err)
