"""Parity tests proper (need the GPU): every call goes through the C ABI of libcrnnctc.so via ctypes.

Stated tolerances for the bf16-operand / f32-accumulate path (north-star: 'within a stated fp tolerance'):
  * GEMM unit test vs f32 matmul of the same bf16 inputs ............ max-abs <= 2e-5 * K^0.5 relative to max|D|
  * CTC costs vs fp64 oracle (f32 kernel, ex2/lg2.approx) ........... rel 1e-4 ; CTC gradient abs 2e-4 (T<=63; 1e-3 at T=130)
  * greedy decode on identical logits ................................ identical sequences (bit-exact integers)
  * full forward logits vs fp64 oracle ............................... max-abs <= 3e-2 * max|logit|
  * total loss vs fp64 oracle ........................................ rel 5e-3
"""
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


@pytest.mark.parametrize("bn,M,Nc,K", [(64, 300, 64, 512), (64, 128, 128, 64), (128, 1000, 256, 576), (128, 77, 128, 1152),
                                       (256, 4096, 512, 2304), (256, 129, 256, 256), (256, 20000, 512, 4608)])
def test_tcgen05_gemm(bn, M, Nc, K):
    from lstm_ctc_ocr_b200 import engine
    g = torch.Generator().manual_seed(bn + M)
    A = (torch.randn(M, K, generator=g) * 0.5).to(torch.bfloat16).to(DEV)
    B = (torch.randn(Nc, K, generator=g) * 0.5).to(torch.bfloat16).to(DEV)
    D = engine.test_gemm_bf16(A, B, bn)
    ref = A.float() @ B.float().t()
    assert rel(D.cpu(), ref.cpu()) < 2e-5


def _ctc_case(T, N, lens, ilens, seed, scale=2.0, blank=0):
    """Label ids 1 .. 62, except that a blank other than 0 takes the place of the blank's own id: it becomes 0, and ids
    2, 3 become a repeated pair of 0."""
    from oracle import crnn_oracle as O
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((T, N, 64)) * scale).astype(np.float32)
    ll = np.asarray(lens, np.int32); il = np.asarray(ilens, np.int32)
    lab = rng.integers(1, 63, size=int(ll.sum())).astype(np.int32)
    if lab.size > 1:
        lab[1] = lab[0]                 # a repeated label
    if blank != 0:
        lab[lab == blank] = 0
        lab[2:4] = 0
    return x, lab, ll, il, O.ctc_loss_np(x, lab, ll, il, blank=blank)


@pytest.mark.parametrize("blank", [0, 17, 63])
@pytest.mark.parametrize("kernel", ["fast", "fast-me", "tma", "tma-me", "generic"])
@pytest.mark.parametrize("case", ["ragged", "edge", "two_warp", "many_frames", "long_ks2", "long_ks4"])
def test_ctc_loss_and_grad_vs_oracle(case, kernel, blank, monkeypatch):
    """ctc_fast_kernel (S <= 32, default: per-thread bulk row copies), ctc_tma_kernel (S <= 32: one tensor-map tile load/store per
    utterance) -- each with the log2-space recursion (default) and the mantissa/exponent recursion (`-me`) -- and the generic
    ctc_loss_kernel<KS> against the fp64 oracle; CRNN_CTC_KERNEL / CRNN_CTC_RECUR select them."""
    from lstm_ctc_ocr_b200 import engine
    if kernel != "fast" and case.startswith("long_ks"):
        pytest.skip("S > 32 always runs the generic kernel")
    monkeypatch.setenv("CRNN_CTC_KERNEL", kernel.split("-")[0])
    monkeypatch.setenv("CRNN_CTC_RECUR", "me" if kernel.endswith("-me") else "log")
    if case == "ragged":
        rng = np.random.default_rng(0)
        N, T = 37, 24
        lens = rng.integers(1, 8, size=N); ilens = rng.integers(14, T + 1, size=N)
    elif case == "edge":      # empty label, infeasible, T=1, input_len 0, full length
        T = 21
        lens = [0, 14, 1, 3, 6, 10]; ilens = [5, 10, 1, 0, 21, 21]
        N = len(lens)
    elif case == "two_warp":  # 16 < S <= 32: alpha and beta on separate warps, mixed with packed utterances
        T, N = 63, 7
        lens = [8, 15, 12, 9, 15, 3, 11]; ilens = [63, 63, 40, 20, 31, 63, 12]
    elif case == "many_frames":   # T > 64: every thread owns several frames
        T, N = 150, 4
        lens = [15, 6, 9, 1]; ilens = [150, 129, 64, 65]
    elif case == "long_ks2":
        T, N = 63, 5
        lens = [20, 31, 16, 25, 30]; ilens = [63, 63, 40, 60, 63]
    else:
        T, N = 130, 3
        lens = [40, 63, 33]; ilens = [130, 130, 100]
    x, lab, ll, il, (co, go) = _ctc_case(T, N, lens, ilens, seed=1, blank=blank)
    t = lambda a: torch.tensor(a, device=DEV)
    c, g = engine.ctc_loss(t(x), t(lab), t(ll), t(il), blank=blank, want_grad=True)
    c2, _ = engine.ctc_loss(t(x), t(lab), t(ll), t(il), blank=blank, want_grad=False)
    assert np.allclose(c.cpu().numpy(), co, rtol=1e-4, atol=1e-4)
    assert np.array_equal(c.cpu().numpy(), c2.cpu().numpy())
    # f32 ex2/lg2.approx recursion: error grows with the chain length (T=130 in the KS=4 case)
    assert np.abs(g.cpu().numpy() - go).max() < (2e-4 if T <= 63 else 1e-3)
    # frames past input_len carry exactly zero gradient; infeasible samples cost 0 with zero gradient
    for n in range(N):
        assert not g[int(il[n]):, n].any()
    if case == "edge":
        assert float(c[1]) == 0.0 and not g[:, 1].any()
    # the blank as a label id: that utterance alone gets cost NaN and a zero gradient
    n = int(np.flatnonzero(ll > 0)[0])
    bad = lab.copy()
    bad[int(ll[:n].sum())] = blank
    c3, g3 = engine.ctc_loss(t(x), t(bad), t(ll), t(il), blank=blank, want_grad=True)
    assert bool(torch.isnan(c3[n])) and not g3[:, n].any()
    keep = torch.arange(N, device=DEV) != n
    assert torch.equal(c3[keep], c[keep]) and torch.equal(g3[:, keep], g[:, keep])


def test_ctc_fast_kernel_extreme_logits_match_generic(monkeypatch):
    """Very peaked rows (scale 30: per-frame probabilities down to 2^-130) keep the log-space recursion finite; both kernels
    agree with the oracle and with each other.  Tolerance: the f32 log2-domain scores reach |a| ~ 4e3 here, where one ulp is
    2.4e-4, and the state posterior 2^(alpha+beta-e-ll) inherits a few ulps of that -- the same
    resolution limit warp-ctc's f32 log-space recursion has; at the working range (|logit| < 10) the bound is 3.6e-5."""
    from lstm_ctc_ocr_b200 import engine
    rng = np.random.default_rng(5)
    N, T = 64, 63
    lens = rng.integers(0, 16, size=N); ilens = rng.integers(32, T + 1, size=N)
    x, lab, ll, il, (co, go) = _ctc_case(T, N, lens, ilens, seed=9, scale=30.0)
    t = lambda a: torch.tensor(a, device=DEV)
    monkeypatch.setenv("CRNN_CTC_KERNEL", "generic")
    cg, gg = engine.ctc_loss(t(x), t(lab), t(ll), t(il), want_grad=True)
    for kern, recur in (("fast", "me"), ("fast", "log"), ("tma", "me")):
        monkeypatch.setenv("CRNN_CTC_KERNEL", kern)
        monkeypatch.setenv("CRNN_CTC_RECUR", recur)
        c, g = engine.ctc_loss(t(x), t(lab), t(ll), t(il), want_grad=True)
        assert torch.isfinite(c).all() and torch.isfinite(g).all(), (kern, recur)
        assert np.allclose(c.cpu().numpy(), co, rtol=2e-4, atol=1e-3), (kern, recur)
        assert np.allclose(c.cpu().numpy(), cg.cpu().numpy(), rtol=2e-4, atol=1e-3), (kern, recur)
        assert np.abs(g.cpu().numpy() - go).max() < 4e-3 and float((g - gg).abs().max()) < 4e-3, (kern, recur)


def test_ctc_grad_scale_and_rowsum_property_full_size():
    """C3-size property: d cost/d logits rows sum to 0 over classes (softmax minus a posterior), scaled by grad_scale."""
    from lstm_ctc_ocr_b200 import engine, synthetic
    T, N = 63, 1024
    _, lab, ll, tsl = synthetic.synth_batch(N, 256, seed=4)
    x = torch.randn(T, N, 64, device=DEV) * 3
    t = lambda a: torch.tensor(a, device=DEV)
    c, g = engine.ctc_loss(x, t(lab), t(ll), t(tsl), want_grad=True, grad_scale=1.0 / N)
    assert torch.isfinite(c).all() and (c > 0).all()
    assert float(g.sum(dim=2).abs().max()) < 1e-6
    c1, g1 = engine.ctc_loss(x, t(lab), t(ll), t(tsl), want_grad=True, grad_scale=1.0)
    assert torch.allclose(g1 / N, g, atol=1e-9)
    # against torch's own CTC on the GPU copy of the same logits (independent implementation)
    lp = torch.log_softmax(x.double(), 2).cpu()
    ref = torch.nn.functional.ctc_loss(lp, torch.tensor(lab, dtype=torch.long), torch.tensor(tsl, dtype=torch.long),
                                       torch.tensor(ll, dtype=torch.long), blank=0, reduction="none")
    assert np.allclose(c.cpu().numpy(), ref.numpy(), rtol=1e-4)


def test_greedy_decode_10k_lines_identical_to_oracle():
    """BASELINE config 4: greedy-decode label sequences identical on 10k synthetic lines, W in {80,160,256}."""
    from lstm_ctc_ocr_b200 import engine
    from oracle import crnn_oracle as O
    rng = np.random.default_rng(7)
    total = 0
    for W, n in ((80, 3400), (160, 3300), (256, 3300)):
        T = W // 4 - 1
        # peaked frames with blanks (0), decoder blanks (63), repeats, plus a noisy tail of flat frames
        path = rng.choice(64, size=(T, n), p=np.r_[0.25, np.full(62, 0.65 / 62), 0.10])
        rep = rng.random((T, n)) < 0.3
        for t in range(1, T):
            path[t] = np.where(rep[t], path[t - 1], path[t])
        x = rng.standard_normal((T, n, 64)).astype(np.float32)
        x[np.arange(T)[:, None], np.arange(n)[None, :], path] += 6.0
        x[:, : n // 50] = 0.0                                    # all-tie rows -> argmax index 0
        il = rng.integers(1, T + 1, size=n).astype(np.int32); il[:5] = [0, 1, T, T, 2]
        out, out_len = engine.ctc_greedy(torch.tensor(x, device=DEV), torch.tensor(il, device=DEV))
        out = out.cpu().numpy(); out_len = out_len.cpu().numpy()
        ref = O.greedy_decode(x, il)
        for i in range(n):
            assert out[i, :out_len[i]].tolist() == ref[i]
            assert not out[i, out_len[i]:].any()
        total += n
    assert total == 10000


def _load_golden():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(ROOT, "tests", "golden", "make_golden.py"))
    mg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mg)
    params, batch, digest = mg.inputs()
    g = np.load(os.path.join(ROOT, "tests", "golden", "crnn_n4_w88.npz"))
    assert str(g["digest"]) == digest
    return params, batch, g


def test_forward_loss_decode_vs_committed_golden():
    from lstm_ctc_ocr_b200 import engine
    params, (data, lab, ll, tsl), g = _load_golden()
    m = engine.CrnnModel(weight_decay=1e-5, device=DEV)
    m.load_params(params)
    t = lambda a: torch.tensor(a, device=DEV)
    logits = m.forward(t(data), t(tsl))
    assert rel(logits.cpu(), g["logits"]) < 3e-2
    costs, grad = engine.ctc_loss(logits, t(lab), t(ll), t(tsl), want_grad=True)
    assert np.allclose(costs.cpu().numpy(), g["costs"], rtol=1e-2)
    loss = float(m.total_loss(costs).item())
    assert abs(loss - float(g["loss"])) / float(g["loss"]) < 5e-3
    assert np.abs(grad.cpu().numpy() - g["ctc_grad"]).max() < 5e-2
    # per-layer statistics (mean, mean|x|, max|x|) within 2 %
    N, W = data.shape[0], data.shape[1]
    T = W // 4 - 1
    for name, tap in [("conv1", "conv1"), ("conv2", "conv2"), ("conv3_1", "conv3_1"), ("conv3_2", "conv3_2"),
                      ("conv4_1", "conv4_1"), ("conv4_2", "conv4_2"), ("reshaped_layer", "conv5"), ("lstm_out", "lstm_out")]:
        a = m.tap(tap, N, W).cpu().numpy()
        if tap in ("conv5", "lstm_out"):
            a = a[:, :T]
        st = g["stat_" + name]
        assert abs(np.abs(a).mean() - st[1]) <= 2e-2 * st[1], name
        assert abs(np.abs(a).max() - st[2]) <= 3e-2 * st[2], name
    # frames past each sample's length: LSTM output is zero, so logits equal the projection bias exactly
    b = params["logits/biases"]
    for n in range(N):
        assert np.array_equal(logits[int(tsl[n]):, n].cpu().numpy(), np.broadcast_to(b, (T - int(tsl[n]), 64)))


@pytest.mark.parametrize("N,W,widths", [(3, 100, None), (5, 24, [24, 20, 9, 24, 16]), (2, 160, [160, 131]), (130, 40, None)])
def test_forward_layers_vs_oracle(N, W, widths):
    """Every layer against the fp64 oracle (conv1_tc.cuh: im2col + split-bf16 wgmma; conv_swap.cuh: conv2 with channels on the
    MMA M side)."""
    from lstm_ctc_ocr_b200 import engine
    from oracle import crnn_oracle as O
    pn = O.randomize_params(O.init_params(3, dtype=np.float32, logits_scale=10.0))
    data, lab, ll, tsl = O.synth_batch(N, W, seed=5, widths=widths, min_len=1, max_len=3)
    m = engine.CrnnModel(device=DEV)
    m.load_params(pn)
    t = lambda a: torch.tensor(a, device=DEV)
    logits = m.forward(t(data), t(tsl))
    lo, acts = O.forward(O.to_torch(pn), data, tsl, return_all=True)
    T = W // 4 - 1
    tol = {"conv1": 5e-3, "conv2": 8e-3, "conv3_1": 8e-3, "conv3_2": 1e-2, "conv4_1": 2.5e-2, "conv4_2": 3.5e-2}
    for name, tl in tol.items():
        assert rel(m.tap(name, N, W).cpu(), acts[name].permute(0, 2, 3, 1).numpy()) < tl, name
    assert rel(m.tap("conv5", N, W).cpu().numpy()[:, :T], acts["reshaped_layer"].numpy()) < 3.5e-2
    assert rel(m.tap("lstm_out", N, W).cpu().numpy()[:, :T], acts["lstm_out"].numpy()) < 6e-2
    assert rel(logits.cpu(), lo.numpy()) < 3e-2
    costs, _ = engine.ctc_loss(logits, t(lab), t(ll), t(tsl))
    co, _ = O.ctc_loss_np(lo.numpy(), lab, ll, tsl)
    loss_o = co.mean() + float(O.l2_reg(O.to_torch(pn), 1e-5))
    assert abs(float(m.total_loss(costs).item()) - loss_o) / loss_o < 5e-3


@pytest.mark.parametrize("chunks", [1, 3, 4])
def test_forward_from_page_locked_host_memory_matches_device_forward(chunks):
    """crnn_forward_host (chunked H2D on a side stream overlapped with the conv front end) == crnn_forward on the same batch;
    chunks=3 does not split 64 images on tile-pair boundaries and must degenerate to one range."""
    from lstm_ctc_ocr_b200 import engine, synthetic
    N, W = 64, 64
    params = synthetic.init_params(3, logits_scale=10.0)
    data, _, _, tsl = synthetic.synth_batch(N, W, seed=21, widths=np.random.default_rng(3).integers(8, 65, size=N))
    m = engine.CrnnModel(device=DEV)
    m.load_params(params)
    d_tsl = torch.tensor(tsl, device=DEV)
    ref = m.forward(torch.tensor(data, device=DEV), d_tsl).clone()
    host = torch.from_numpy(data.copy()).pin_memory()
    for _ in range(2):                                   # second call re-uses the staging tensor while the first may be in flight
        logits, staged = m.forward_host(host.numpy(), d_tsl, chunks=chunks)
    torch.cuda.synchronize()
    assert torch.equal(staged.cpu(), torch.from_numpy(data))
    assert rel(logits.cpu().numpy(), ref.cpu().numpy()) < 2e-3      # BN-statistic atomics order is the only difference


def test_session_run_reads_like_the_reference_solver():
    """sess.run([loss, dense_decoded], feed_dict) as lib/lstm/train.py:121-130,160 does; decode == oracle greedy
    on samples whose per-frame top-2 margin is clear of bf16 noise."""
    from lstm_ctc_ocr_b200 import synthetic
    from lstm_ctc_ocr_b200.lib.lstm.utils.training import accuracy_calculation
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    from oracle import crnn_oracle as O
    net = get_network("LSTM_train")
    loss, dense_decoded = net.build_loss()
    params = synthetic.init_params(3, logits_scale=30.0)
    img, lab, ll, tsl = synthetic.synth_batch(16, 100, seed=8, widths=[100] * 8 + [77, 64, 52, 99, 100, 88, 96, 41])
    with Session(device=DEV) as sess:
        sess.assign(net, params)
        feed = {net.data: img, net.labels: lab, net.time_step_len: tsl, net.labels_len: ll, net.keep_prob: 0.5}
        ctc_loss, res = sess.run([loss, dense_decoded], feed_dict=feed)
        logits = sess.run(net.get_output("logits"), feed_dict=feed)
        assert sess.h2d_bytes == img.nbytes + tsl.nbytes and sess.d2h_bytes == logits.nbytes
    lo = O.forward(O.to_torch({k: v.astype(np.float64) for k, v in params.items()}), img, tsl).numpy()
    co, _ = O.ctc_loss_np(lo, lab, ll, tsl)
    # logits matrix scaled x30 here (peaked outputs for the decode check), which amplifies bf16 error in the loss too
    assert abs(ctc_loss - (co.mean() + float(O.l2_reg(O.to_torch(params), 1e-5)))) / co.mean() < 3e-2
    assert res.dtype == np.int32 and res.shape[0] == 16
    ref = O.greedy_decode(lo, tsl)
    # samples whose per-frame top-2 margin (oracle logits) exceeds twice the GPU-vs-oracle logit error decode identically
    srt = np.sort(lo, axis=2)
    margin = (srt[:, :, -1] - srt[:, :, -2])
    err = np.abs(logits - lo).max(axis=2)
    clear = [n for n in range(16) if tsl[n] > 0 and np.all(margin[:tsl[n], n] > 2 * err[:tsl[n], n].max())]
    for n in clear:
        assert [v for v in res[n] if v != 0] == ref[n]
    # decode of the GPU logits themselves is bit-identical to the oracle rule
    assert O.dense_decoded(O.greedy_decode(logits, tsl)).tolist() == res.tolist()
    org = [lab[s:s + l] for s, l in zip(np.cumsum(ll) - ll, ll)]
    assert 0.0 <= accuracy_calculation(org, res, isPrint=False) <= 1.0


def test_warpctc_drop_in_call_shape_and_autograd():
    from lstm_ctc_ocr_b200 import warpctc
    from oracle import crnn_oracle as O
    rng = np.random.default_rng(3)
    T, N = 20, 6
    x = (rng.standard_normal((T, N, 64))).astype(np.float32)
    ll = np.array([4, 5, 6, 4, 5, 6], np.int32); il = np.array([20, 19, 18, 20, 12, 20], np.int32)
    lab = rng.integers(1, 63, size=ll.sum()).astype(np.int32)
    co, go = O.ctc_loss_np(x, lab, ll, il)
    costs = warpctc.ctc(activations=x, flat_labels=lab, label_lengths=ll, input_lengths=il)     # numpy in -> numpy out
    assert isinstance(costs, np.ndarray) and np.allclose(costs, co, rtol=1e-4)
    xt = torch.tensor(x, device=DEV, requires_grad=True)
    c = warpctc.ctc(xt, lab, ll, il)
    (c * torch.arange(1, N + 1, device=DEV)).sum().backward()                                    # dloss[n] = n+1
    assert np.abs(xt.grad.cpu().numpy() - go * np.arange(1, N + 1)[None, :, None]).max() < 1e-3
    # blank_label = 63, with id 0 (a repeated pair of it) among the labels
    lab[2:4] = 0
    co, go = O.ctc_loss_np(x, lab, ll, il, blank=63)
    xt = torch.tensor(x, device=DEV, requires_grad=True)
    c = warpctc.ctc(xt, lab, ll, il, blank_label=63)
    (c * torch.arange(1, N + 1, device=DEV)).sum().backward()
    assert np.allclose(c.detach().cpu().numpy(), co, rtol=1e-4)
    assert np.abs(xt.grad.cpu().numpy() - go * np.arange(1, N + 1)[None, :, None]).max() < 1e-3


def test_full_size_c3_properties():
    """BASELINE config 3 shapes (batch 1024, 32x256): size-independent properties of the whole path."""
    from lstm_ctc_ocr_b200 import engine, synthetic
    N, W = 1024, 256
    T = W // 4 - 1
    params = synthetic.init_params(3, logits_scale=10.0)
    widths = np.r_[np.full(512, 256), np.random.default_rng(0).integers(8, 257, size=512)]
    data, lab, ll, tsl = synthetic.synth_batch(N, W, seed=6, widths=widths)
    m = engine.CrnnModel(device=DEV)
    m.load_params(params)
    t = lambda a: torch.tensor(a, device=DEV)
    logits = m.forward(t(data), t(tsl))
    assert torch.isfinite(logits).all()
    # (1) frames >= len are exactly the projection bias (zero LSTM output there)
    mask = torch.arange(T, device=DEV)[:, None] >= t(tsl)[None, :]
    assert torch.equal(logits[mask], t(params["logits/biases"]).expand(int(mask.sum()), 64))
    # (2) determinism: a second run on the same inputs is bit-identical except for BN-stat atomics order (f64) -> allow 1e-6
    logits2 = m.forward(t(data), t(tsl)).clone()
    assert float((logits2 - logits).abs().max()) <= 1e-3 * float(logits.abs().max())
    # (3) batch-permutation equivariance (BN statistics are permutation invariant)
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(1))
    lp = m.forward(t(data[perm.numpy()]), t(tsl[perm.numpy()]))
    assert float((lp - logits2[:, perm.to(DEV)]).abs().max()) <= 2e-2 * float(logits.abs().max())
    # (4) loss is finite and positive; greedy decode emits only ids 1..62, never more than len symbols
    costs, _ = engine.ctc_loss(lp, t(lab), t(ll), t(tsl[perm.numpy()]))
    assert torch.isfinite(costs).all()
    out, out_len = engine.ctc_greedy(logits2, t(tsl))
    assert int((out_len > t(tsl)).sum()) == 0
    assert int(out.max()) <= 62 and int(out.min()) >= 0
