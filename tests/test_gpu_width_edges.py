"""The widths evaluation feeds, and the CTC kernels at their frame limits.

Evaluation runs one line at a time at that line's own width (lib/lstm/test.py prepare_line: padded to a multiple of 4,
at least 8), so it runs N = 1 at T = W/4 - 1 from 1 (a crop 8 px wide) to 250 and more (a long line).  The other GPU
tests stay within W = 24 .. 256 (T = 5 .. 63).  Code paths reached only outside that range:
  - the recurrence's first fills and exchanges at T = 1, 2, 3 (no exchange at T = 1, one at T = 2, the first re-arm of a
    fill barrier at T = 3), and the BPTT's last step and mbarrier parities at T = 1 (no recurrent step at all);
  - the backward direction's reversed input-projection rows (the EPI_XPROJ epilogue) at H = W/4 = 128 (one sequence per
    128-row tile, the staged permutation) and at H = 129 and 256 (a sequence crosses tiles, the direct store);
  - 255 serial steps forward and backward;
  - the CTC kernels' shared-memory limits (tensor-map kernel T <= 256, the fast kernel, the generic kernels, and the
    ceiling beyond which the call fails), and the misaligned-pointer fall-back to the generic kernel;
  - greedy decode over several 32-frame chunks, and the device beam decoder over hundreds of frames.

The stage checks are those of test_gpu_stage_isolation.py with the fp64 references on the GPU, run over chunks of
128 * 256 / W images (positions, not images, set their memory).  Every stage keeps its small-shape bound (the weight
gradients the per-tensor bounds of test_gpu_stage_isolation_batch.py) except the CTC gradient at T > 63:
  - The free-running recurrence and BPTT (c * max|ref|) do not need more at T = 255.  Their error is the bf16 rounding of
    h (resp. dz) fed back every step, and the LSTM forgets: each step multiplies an earlier error by a forget gate below 1
    and a tanh' at most 1, so the worst element sees only the last few steps' roundings.  Measured 5.5e-4 and 2.7e-4 of
    max|ref| at T = 255 against 6.5e-3 and 7e-3 allowed (1.6e-3 at the small shapes, 6.6e-4 at 1024 x 256).
  - The CTC gradient's error does grow with T.  The log2-space alpha / beta recursions of the S <= 32 kernels and the
    generic kernel take one approximate ex2 / lg2 per state and step, so log alpha_t + log beta_t - log p carries a
    rounding error that adds up over the Tn steps, and the gradient alpha * beta / p inherits it as a relative error.  At
    T = 255 it reached 9.0e-4 * grad_scale, 4.5x the bound set at T <= 63 (test_gpu_parity.py).  The per-element stages
    of tests/ctc_refs.py scale with P * |log2 p| * sqrt(T_n) themselves; its relative L2 gets 4.5x the 1.49e-4 measured.
    The cost, a sum over the same path, stays at 1e-6 of |cost|.
Every enforced bound of this file is 4.5x its measurement on H100 80GB HBM3 (SXM).

Rows go to build/width_edges_report.jsonl, with the peak GPU memory of each stage-check case."""
import importlib.util
import os
import random
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_gpu_beam as GB  # noqa: E402
import test_gpu_lstm_halves as LH  # noqa: E402
import test_gpu_stage_isolation as B  # noqa: E402
import test_gpu_stage_isolation_batch as BB  # noqa: E402
import test_gpu_x3_stage_isolation as XS  # noqa: E402
import ctc_refs as R  # noqa: E402
from stage_check import Checker  # noqa: E402
from stage_check import ulp_bf16  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = B.DEV
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REPORT = "width_edges_report.jsonl"

# Largest c needed at T > 63 (W512, W516, W1024, N1_W1024, and the ring BPTT at W1024), H100 80GB HBM3 (SXM): stage ->
# (c, relative L2).  A stage whose 4.5 c exceeds its bound at T <= 63 gets 4.5 c (and L2 limit 4.5x) at T > 63.
# The CTC gradient's per-element stages (tests/ctc_refs.py) scale with T themselves; its relative L2 measured 1.49e-4.
MEASURED = {"lstm_out": (5.53e-4, None), "dz_all": (2.68e-4, None)}
LONG = {k: (BB.BOUNDS[k][0], 4.5 * c) for k, (c, _) in MEASURED.items() if 4.5 * c > BB.BOUNDS[k][1]}
LONG_L2 = {"ctc_grad/fast": max(BB.L2_LIMIT["ctc_grad/fast"], 4.5 * 1.49e-4)}

# id -> (N, W, CTC-driven backward with labels up to 15)
CASES = [
    pytest.param(5, 8, False, id="T1"),            # T = 1: no recurrent step forward or backward
    pytest.param(130, 12, True, id="T2"),          # T = 2: one exchange; two row tiles, H = 3
    pytest.param(3, 16, False, id="T3"),           # T = 3: the first re-arm of a fill barrier
    pytest.param(3, 512, False, id="W512"),        # H = 128: one sequence per tile, the permuted EPI_XPROJ store
    pytest.param(2, 516, False, id="W516"),        # H = 129: a sequence overhangs its tile by one row (direct store)
    pytest.param(130, 1024, True, id="W1024"),     # H = 256, two LSTM row tiles, 255 serial steps forward and BPTT
    pytest.param(1, 8, False, id="N1_W8"),         # the evaluation shapes exactly
    pytest.param(1, 1024, False, id="N1_W1024"),
]


def _checker(case, T):
    long = T > 63
    return Checker(case, dict(BB.BOUNDS, **(LONG if long else {})), REPORT, ulp_bf16,
                   dict(BB.L2_LIMIT, **(LONG_L2 if long else {})))


def _widths(N, W, seed=3):
    """Pixel widths: every 128-row tile starts with W, 8, 4 (lengths T, 1, 0); the other rows random multiples of 4."""
    w = np.random.default_rng(seed).integers(1, W // 4 + 1, size=N) * 4
    for t0 in range(0, N, 128):
        for j, v in enumerate((W, 8, 4)):
            if t0 + j < N:
                w[t0 + j] = v
    return [int(v) for v in w]


def _chunk(W):
    return max(1, 128 * 256 // W)


@pytest.mark.parametrize("N,W,ctc", CASES)
def test_every_stage_at_edge_widths(N, W, ctc, request):
    """Training forward + backward, every stage on its own inputs; then the inference plan of a fresh model on the same
    batch (its own epilogues: frag_epilogue, conv2_swap_kernel<false>, conv1_tc_kernel<false>), every forward stage
    against the references, conv1 .. conv3_2 bit-identical to the training plan and conv4_x within one bf16 ulp."""
    case, T = request.node.callspec.id, W // 4 - 1
    torch.cuda.reset_peak_memory_stats()
    m, F_, ck = B._run_stage_checks(case, N, W, _widths(N, W), dev=DEV, chunk=_chunk(W), ctc=BB._ctc_grad if ctc else None,
                                    ck=_checker(case, T), max_label=15 if ctc else 4)
    del m
    for k in B.BWD_TAPS + ("gates_steps", "csave_steps", "conv5", "xproj", "lstm_out"):
        del F_.G[k]
    ci = _checker(case + "/inference", T)
    BB._inference_plan_checks(ci, F_, N, W, _chunk(W))
    BB._peak(ck)
    fail = []
    for c in (ck, ci):
        c.report()
        fail += c.fail
    assert not fail, "\n".join(fail)


@pytest.mark.parametrize("W", [8, 12, 16, 1024])
def test_lstm_launches_and_training_bit_identical_at_edge_widths(W):
    """Inference and training, two launches each: bit-identical lstm_out, gates and cell state over 130 lines (two row
    tiles)."""
    LH.check_launches_and_training_bit_identical(130, W)


# ------------------------------------------------------------------------------------------------------------------- CTC
SMEM_LIMIT = 200 * 1024


def _alpha_stride(m):
    return (2 * m + 1) | 1


def _label_stride(m):
    return m | 1


def _tma_ok(T, m):
    rows = (T + 7) // 8 * 8
    return T <= 256 and 1024 + 2 * rows * 128 + 4 * T * (2 * _alpha_stride(m) + _label_stride(m) + 2) <= SMEM_LIMIT


def _fast_ok(T, m):
    return 4 * T * (68 + 2 * _alpha_stride(m) + _label_stride(m) + 2) <= SMEM_LIMIT


def _generic_ok(T, ks):
    return 4 * (T + 3 * T * 32 * ks + 4 * 4 * 64) <= SMEM_LIMIT


def kernel_for(T, m, choice="fast", aligned=True):
    """csrc/ctc.cu crnn_ctc_loss's dispatch, restated: the kernel a call runs, or None where it returns CRNN_UNSUPPORTED.
    choice: CRNN_CTC_KERNEL ("fast" is the default)."""
    S = 2 * m + 1
    if S <= 32 and aligned and choice == "tma" and _tma_ok(T, m):
        return "tma"
    if S <= 32 and aligned and choice != "generic" and _fast_ok(T, m):
        return "fast"
    ks = 1 if S <= 32 else 2 if S <= 64 else 4
    return f"generic{ks}" if _generic_ok(T, ks) else None


def _last(ok):
    return max(t for t in range(1, 2048) if ok(t))


CEILING = {m: _last(lambda t: kernel_for(t, m) is not None) for m in (4, 15, 31, 63)}
# the limits include/crnn_ctc.h documents
assert (_last(lambda t: _tma_ok(t, 15)), _last(lambda t: _fast_ok(t, 15)), _last(lambda t: _fast_ok(t, 4))) == (256, 348, 550)
assert [_last(lambda t: _generic_ok(t, ks)) for ks in (1, 2, 4)] == [517, 259, 130]
assert CEILING == {4: 550, 15: 517, 31: 259, 63: 130}

VARIANTS = {"fast": {}, "fast-me": {"CRNN_CTC_RECUR": "me"}, "tma": {"CRNN_CTC_KERNEL": "tma"},
            "tma-me": {"CRNN_CTC_KERNEL": "tma", "CRNN_CTC_RECUR": "me"}, "generic": {"CRNN_CTC_KERNEL": "generic"}}

# Largest c needed per kernel over every T of test_ctc_at_its_frame_limits (130 .. 550), H100 80GB HBM3 (SXM): (cost
# relative to |cost|, the flat per-element gradient bound in units of grad_scale that ctc_grad_softmax /
# ctc_grad_posterior replaced, the gradient's relative L2).  The gradient's error grows with T
# (see above); the "me" recursions (mantissa / exponent pairs, no transcendental on the chain) stay about 5x lower.
MEASURED_CTC = {"tma": (5.80e-7, 1.04e-3, 2.90e-4), "tma-me": (9.51e-8, 2.31e-4, 6.69e-5),
                "fast": (1.05e-6, 3.38e-3, 8.22e-4), "fast-me": (1.16e-7, 6.04e-4, 1.41e-4),
                "generic1": (1.05e-6, 3.39e-3, 7.00e-4), "generic2": (2.36e-7, 5.51e-4, 1.71e-4),
                "generic4": (3.07e-7, 2.54e-4, 9.54e-5)}
CTC_BOUNDS = dict({f"ctc_cost/{k}": (0, 4.5 * v[0]) for k, v in MEASURED_CTC.items()},
                  **R.bounds(MEASURED_CTC, {k: 4.5 * R.MEASURED_POSTERIOR[k] for k in MEASURED_CTC}))
CTC_L2 = {f"ctc_grad/{k}": max(1e-4, 4.5 * v[2]) for k, v in MEASURED_CTC.items()}


def _ctc_batch(T, m, seed, blank=0):
    """Lengths 0, 1, T (and one above T, which the kernel clamps), an empty label, all-repeat labels that just fit and
    that do not, and random utterances; label ids over [0, 64) minus the blank, a repeated pair of 0 in the first label
    where 0 is not the blank.  Returns logits, labels, label lengths, input lengths (unclamped)."""
    rng = np.random.default_rng(seed)
    rows = [(m, T), (1, 0), (1, 1), (0, T), ("rep", T), ("rep", min(T, 2 * m - 2)), ("rep", min(T, 2 * m - 1)),
            (m, T + 5)]
    rows += [(int(rng.integers(0, m + 1)), int(rng.integers(1, T + 1))) for _ in range(6)]
    lab, ll, il = [], [], []
    for i, (L, n) in enumerate(rows):
        if L == "rep":
            seq = [int(R.draw_labels(rng, 1, blank)[0])] * m
        else:
            seq = [int(v) for v in R.draw_labels(rng, L, blank)]
            if L >= 4:
                seq[2] = seq[1]                                   # a repeat inside a random label
            if i == 0 and blank != 0 and L >= 4:
                seq[1] = seq[2] = 0
        lab += seq; ll.append(len(seq)); il.append(n)
    N = len(rows)
    x = (rng.standard_normal((T, N, 64)) * 2.0).astype(np.float32)
    return x, np.array(lab, np.int32), np.array(ll, np.int32), np.array(il, np.int32)


def _ctc_run(x, lab, ll, il, m, scale, logits=None, grad=None, costs=None, blank=0):
    from lstm_ctc_ocr_b200 import engine
    t = lambda a: torch.tensor(a, device=DEV)
    lg = t(x) if logits is None else logits
    grad = torch.empty_like(lg) if grad is None else grad
    costs, grad = engine.ctc_loss(lg, t(lab), t(ll), t(il), blank=blank, want_grad=True, grad_scale=scale, max_label_len=m,
                                  costs=costs, grad=grad)
    torch.cuda.synchronize()
    return costs, grad


def _frame_limit_Ts(m):
    """Just below and just above every boundary the dispatch has at this max_label_len."""
    S = 2 * m + 1
    bounds = {CEILING[m]}
    if S <= 32:
        bounds |= {256, _last(lambda t: _fast_ok(t, m)), _last(lambda t: _generic_ok(t, 1))}
    return sorted({b for c in bounds for b in (c, c + 1) if b <= CEILING[m]})


@pytest.mark.parametrize("blank", [0, 17, 63])
@pytest.mark.parametrize("m", [4, 15, 31, 63])
def test_ctc_at_its_frame_limits(m, blank, monkeypatch):
    """Every kernel a call can run at T just below and above each dispatch boundary, against ctc_refs.ctc_fp64: costs
    relative to |cost|, the gradient per element (ctc_grad_softmax, ctc_grad_posterior) and its relative L2, exactly
    zero past each length; an infeasible utterance gives cost 0 and a zero gradient."""
    from lstm_ctc_ocr_b200._lib import CrnnError
    ck = Checker(f"ctc_m{m}_b{blank}", CTC_BOUNDS, REPORT, ulp_bf16, CTC_L2)
    for T in _frame_limit_Ts(m):
        x, lab, ll, il = _ctc_batch(T, m, seed=T + m + blank, blank=blank)
        N = x.shape[1]
        ref = R.ctc_fp64(torch.tensor(x, device=DEV), lab, ll, il, blank=blank, grad_scale=1.0 / N, max_label_len=m)
        done = set()
        for name, env in VARIANTS.items():
            if 2 * m + 1 > 32 and name != "fast":
                continue
            choice = env.get("CRNN_CTC_KERNEL", "fast")
            kind = kernel_for(T, m, choice)
            if kind in ("fast", "tma") and "CRNN_CTC_RECUR" in env:
                kind += "-me"
            if kind in done:
                continue
            done.add(kind)
            for k in ("CRNN_CTC_KERNEL", "CRNN_CTC_RECUR"):
                monkeypatch.delenv(k, raising=False)
            for k, v in env.items():
                monkeypatch.setenv(k, v)
            if kind is None:                       # forced generic past its limit
                with pytest.raises(CrnnError, match=f"CRNN_UNSUPPORTED.*T = {T}"):
                    _ctc_run(x, lab, ll, il, m, 1.0 / N, blank=blank)
                continue
            costs, grad = _ctc_run(x, lab, ll, il, m, 1.0 / N, blank=blank)
            R.check_grad(ck, kind, costs, grad, ref, 1.0 / N)
    ck.assert_ok()


@pytest.mark.parametrize("m", [4, 15, 31, 63])
def test_ctc_one_past_the_ceiling_fails_and_leaves_the_outputs(m, monkeypatch):
    """T = ceiling + 1: CrnnError with CRNN_UNSUPPORTED and a message naming T; costs and gradient keep their contents.
    Forced to the generic kernel, max_label_len 4 fails one past the generic limit (518) where the fast kernel still runs."""
    from lstm_ctc_ocr_b200._lib import CrnnError
    cases = [(CEILING[m] + 1, {})]
    if m == 4:
        cases.append((518, {"CRNN_CTC_KERNEL": "generic"}))
    for T, env in cases:
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        assert kernel_for(T, m, env.get("CRNN_CTC_KERNEL", "fast")) is None
        x, lab, ll, il = _ctc_batch(T, m, seed=1)
        costs = torch.full((x.shape[1],), 1234.5, device=DEV)
        grad = torch.full(x.shape, -7.0, device=DEV)
        with pytest.raises(CrnnError, match=f"CRNN_UNSUPPORTED.*T = {T}") as e:
            _ctc_run(x, lab, ll, il, m, 1.0, grad=grad, costs=costs)
        assert "bytes" in str(e.value)
        assert bool((costs == 1234.5).all()) and bool((grad == -7.0).all())


def test_ctc_misaligned_pointers_take_the_generic_kernel(monkeypatch):
    """Logits or a gradient 4 bytes off 16-byte alignment run the generic kernel: bit-identical to the aligned run forced
    to it.  Past the generic limit a misaligned call fails even where the fast kernel would run aligned."""
    from lstm_ctc_ocr_b200._lib import CrnnError
    m, T = 15, 300
    x, lab, ll, il = _ctc_batch(T, m, seed=5)
    N = x.shape[1]
    monkeypatch.setenv("CRNN_CTC_KERNEL", "generic")
    c_gen, g_gen = _ctc_run(x, lab, ll, il, m, 1.0 / N)
    monkeypatch.delenv("CRNN_CTC_KERNEL")
    c_fast, _ = _ctc_run(x, lab, ll, il, m, 1.0 / N)
    assert not torch.equal(c_fast, c_gen)                 # the two kernels round differently, so the comparison can tell
    buf = torch.empty(x.size + 4, device=DEV)
    lg = buf[1:1 + x.size].view(x.shape)
    lg.copy_(torch.tensor(x, device=DEV))
    assert lg.data_ptr() % 16 == 4
    c, g = _ctc_run(x, lab, ll, il, m, 1.0 / N, logits=lg)
    assert torch.equal(c, c_gen) and torch.equal(g, g_gen)
    gbuf = torch.empty(x.size + 4, device=DEV)
    c, g = _ctc_run(x, lab, ll, il, m, 1.0 / N, grad=gbuf[1:1 + x.size].view(x.shape))
    assert torch.equal(c, c_gen) and torch.equal(g, g_gen)
    T = 530                                               # max_label_len 4: fast up to 550, generic up to 517
    assert kernel_for(T, 4) == "fast" and kernel_for(T, 4, aligned=False) is None
    x, lab, ll, il = _ctc_batch(T, 4, seed=6)
    buf = torch.empty(x.size + 4, device=DEV)
    lg = buf[1:1 + x.size].view(x.shape)
    lg.copy_(torch.tensor(x, device=DEV))
    with pytest.raises(CrnnError, match=f"CRNN_UNSUPPORTED.*T = {T}"):
        _ctc_run(x, lab, ll, il, 4, 1.0, logits=lg)


# ---------------------------------------------------------------------------------------------------------------- decode
def _runs(T, N, rng):
    """Frames in runs of 1 .. 40 of one class (blank 63, the stripped 0, or a label), so that runs of repeats and of
    blanks straddle the 32-frame chunks; utterance 1 repeats one label across every chunk boundary (merged), utterance 2
    splits it with a blank on the boundary frame (emitted twice), utterance 3 has an all-equal frame (arg-max 0)."""
    x = rng.standard_normal((T, N, 64)).astype(np.float32)
    for n in range(N):
        t = 0
        while t < T:
            r = int(rng.integers(1, 41))
            c = [63, 0, int(rng.integers(1, 63))][int(rng.choice(3, p=[0.4, 0.1, 0.5]))]
            x[t:t + r, n, c] += 6.0
            t += r
    for t in range(31, T, 32):
        x[t - 1:t + 2, 1 % N] = 0.0
        x[t - 1:t + 2, 1 % N, 17] = 9.0
        if N > 2:
            x[t - 1:t + 2, 2] = 0.0
            x[t - 1, 2, 17] = x[t, 2, 63] = x[t + 1 if t + 1 < T else t, 2, 17] = 9.0
    if N > 3:
        x[T // 2, 3] = 0.5
    return x


@pytest.mark.parametrize("T", [1, 2, 31, 32, 33, 64, 65, 255, 1023])
def test_greedy_decode_over_many_chunks(T):
    from lstm_ctc_ocr_b200 import engine
    from oracle import crnn_oracle as O
    rng = np.random.default_rng(T)
    N = 9
    x = _runs(T, N, rng)
    il = np.array([T, T, T, T, 0, 1] + [int(v) for v in rng.integers(0, T + 1, size=N - 6)], np.int32)
    out, out_len = engine.ctc_greedy(torch.tensor(x, device=DEV), torch.tensor(il, device=DEV))
    out, out_len = out.cpu().numpy(), out_len.cpu().numpy()
    want = O.greedy_decode(x, il)
    for n in range(N):
        assert out[n, :out_len[n]].tolist() == want[n], (n, il[n])
        assert not out[n, out_len[n]:].any()
    buf = torch.empty(x.size + 4, device=DEV)               # logits 4 bytes off 16-byte alignment: the scalar-load kernel
    lg = buf[1:1 + x.size].view(x.shape)
    lg.copy_(torch.tensor(x, device=DEV))
    o2, l2 = engine.ctc_greedy(lg, torch.tensor(il, device=DEV))
    assert np.array_equal(o2.cpu().numpy(), out) and np.array_equal(l2.cpu().numpy(), out_len)


@pytest.mark.parametrize("T", [1, 2, 255, 511])
@pytest.mark.parametrize("kind", ["peaked", "soft"])
def test_device_beam_over_long_frames(T, kind):
    """Device labelling, zero padding and neg_log_prob equal the host decoder's (test_gpu_beam._both) at widths 1, 2,
    100 and 128."""
    rng = np.random.default_rng(T + (kind == "soft"))
    N = 6
    x = GB._peaked_lines(N, T, seed=T, margin=6.0 if kind == "peaked" else 2.0).astype(np.float32)
    il = np.array([T, 0, 1] + [int(v) for v in rng.integers(0, T + 1, size=N - 3)], np.int32)
    for bw in (1, 2, 100, 128):
        GB._both(x, il, beam_width=bw, merge_repeated=True)


@pytest.mark.parametrize("mode", XS.MODES)
@pytest.mark.parametrize("N,W,widths", [pytest.param(3, 8, [8, 8, 4], id="N3_W8"),
                                        pytest.param(2, 1024, [1024, 516], id="N2_W1024")])
def test_x3_stages_at_edge_widths(mode, N, W, widths, request):
    """The f32-class forward paths (split-bf16 and tf32 operands), every stage, with test_gpu_x3_stage_isolation's bounds."""
    XS._run_stage_checks(request.node.callspec.id, mode, N, W, widths)


# ------------------------------------------------------------------------------------------------------ evaluation
def _load(name, *path):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, *path))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _eval_inputs():
    """64 rendered lines of 30 - 70 characters (W about 400 - 1000) and crops 8, 9 and 12 px wide of a 32-high line
    (W = 8, 12, 12; lengths 1, 1, 2), each through prepare_line."""
    from PIL import Image
    from lstm_ctc_ocr_b200.lib.lstm.test import prepare_line
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    rng = random.Random(4242)
    imgs = [gen.render_line(gen.gen_rand(rng, 30, 70), rng=rng) for _ in range(64)]
    h32 = np.asarray(Image.fromarray(imgs[0]).resize((int(32 / imgs[0].shape[0] * imgs[0].shape[1]), 32), Image.BILINEAR),
                     dtype=np.uint8)
    imgs += [h32[:, 40:40 + w] for w in (8, 9, 12)]
    return [prepare_line(im) for im in imgs]


def test_evaluation_end_to_end_at_line_widths(monkeypatch):
    """Session.run(dense_decoded) one line at a time, trained weights (the decode-10k fixture's), greedy and beam.  Each
    decoder equals its own decode of the GPU's logits on every line (greedy: the oracle's greedy_decode; beam: the host
    decoder), and the oracle's decode of the oracle's logits on every line whose minimum top-2 margin exceeds
    test_gpu_decode10k.MARGIN; the others are reported."""
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.session import Session
    from oracle import crnn_oracle as O
    margin = _load("test_gpu_decode10k", "tests", "test_gpu_decode10k.py").MARGIN
    mk = _load("make_decode10k", "tests", "golden", "make_decode10k.py")
    monkeypatch.setenv("CRNN_FONT", "default")
    gen._FONT_CACHE.clear()
    weights = mk.load_weights()
    inputs = _eval_inputs()
    assert [(d.shape[1], int(t[0])) for d, t in inputs[-3:]] == [(8, 1), (12, 1), (12, 2)]
    assert min(d.shape[1] for d, _ in inputs[:64]) > 256
    p32 = O.to_torch({k: v.astype(np.float32) for k, v in weights.items()}, torch.float32)
    oracle = []
    for data, tsl in inputs:
        lo = O.forward(p32, data, tsl).numpy()
        srt = np.sort(lo[:, 0], axis=1)
        mg = float((srt[:, -1] - srt[:, -2])[:tsl[0]].min()) if tsl[0] > 0 else 99.0
        hb, hbl, _ = engine.ctc_beam_search(lo, tsl, beam_width=100, merge_repeated=True)
        oracle.append(dict(greedy=O.greedy_decode(lo, tsl)[0], beam=[int(v) for v in hb[0, :hbl[0]] if v != 0], margin=mg))
    net = get_network("LSTM_test")
    f_logits, f_dense = Fetch(net, "logits"), Fetch(net, "dense_decoded")
    ck = Checker("evaluation", {}, REPORT)
    old = cfg.get("DECODER", "greedy")
    try:
        with Session(device=DEV) as sess:
            sess.assign(net, weights)
            for decoder in ("greedy", "beam"):
                cfg.DECODER = decoder
                st = dict(lines=0, own_decode_equal=0, clear_margin_lines=0, clear_margin_identical=0, identical=0,
                          max_width=0)
                unclear = []
                for i, (data, tsl) in enumerate(inputs):
                    logits, dec = sess.run([f_logits, f_dense], feed_dict={net.data: data, net.time_step_len: tsl,
                                                                           net.keep_prob: 1.0})
                    got = [int(v) for v in dec[0] if v != 0] if dec.size else []
                    if decoder == "greedy":
                        own = O.greedy_decode(logits, tsl)[0]
                    else:
                        hb, hbl, _ = engine.ctc_beam_search(logits, tsl, beam_width=100, merge_repeated=True)
                        own = [int(v) for v in hb[0, :hbl[0]] if v != 0]
                    same = got == oracle[i][decoder]
                    clear = oracle[i]["margin"] > margin
                    st["lines"] += 1
                    st["own_decode_equal"] += int(got == own)
                    st["identical"] += int(same)
                    st["clear_margin_lines"] += int(clear)
                    st["clear_margin_identical"] += int(clear and same)
                    st["max_width"] = max(st["max_width"], int(data.shape[1]))
                    if not clear:
                        unclear.append(dict(line=i, W=int(data.shape[1]), margin=round(oracle[i]["margin"], 4), same=same))
                ok = st["own_decode_equal"] == st["lines"] and st["clear_margin_identical"] == st["clear_margin_lines"]
                ck._record(f"eval_{decoder}", 0.0 if ok else float("inf"), **st, below_margin=unclear)
    finally:
        cfg.DECODER = old
    ck.assert_ok()
