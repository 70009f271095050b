"""The workspace CTC path without a GPU: an fp64 restatement of ctc_long_kernel's algorithm, its workspace-size query, and
the feeder's ring-slot bound for long rendered lines.

The restatement follows the kernel step for step in fp64 natural-log space: log-softmax rows, the alpha rows, beta
recomputed row by row, each state's posterior alpha*beta/y/p against the alpha row, and the gradient y - (posterior sums per
class) with the kernel's fixed order: a class's states in label order, blank over its L+1 even states, each sum taken as 32
lane-strided partials then a fixed xor tree.  It must equal brute-force path enumeration on tiny cases and the oracle's CTC
and fp64 torch.ctc_loss with autograd at L = 64, 255 and 639 and T up to 2048."""
import itertools
import math
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

NEG = -np.inf


def _fixed_order_sum(W):
    """W [Tn, k] -> [Tn]: lane j sums columns j, j+32, ... in order; then the xor tree lane 0 ends with."""
    Tn, k = W.shape
    lanes = np.zeros((Tn, 32))
    for j in range(min(32, k)):
        for i in range(j, k, 32):
            lanes[:, j] += W[:, i]
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, np.arange(32) ^ o]
    return lanes[:, 0]


def ctc_long_ref(x, lab, ll, il, blank=0, max_label_len=None):
    """fp64 restatement of ctc_long_kernel: (costs [N], d costs[n] / d logits [T, N, C])."""
    x = np.asarray(x, np.float64)
    T, N, C = x.shape
    mll = int(max(ll)) if max_label_len is None else int(max_label_len)
    costs = np.zeros(N)
    grad = np.zeros_like(x)
    off = 0
    for n in range(N):
        L, Tn = int(ll[n]), max(0, min(int(il[n]), T))
        seq = np.asarray(lab[off:off + max(L, 0)], np.int64)
        off += max(L, 0)
        if L < 0 or L > mll or ((seq < 0) | (seq >= C) | (seq == blank)).any():
            costs[n] = np.nan
            continue
        rep = int((seq[1:] == seq[:-1]).sum()) if L > 1 else 0
        if Tn == 0 or L + rep > Tn:
            continue
        S = 2 * L + 1
        ext = np.full(S, blank, np.int64)
        ext[1::2] = seq
        xs = x[:Tn, n]
        m = xs.max(1, keepdims=True)
        lp = xs - (m + np.log(np.exp(xs - m).sum(1, keepdims=True)))
        e = lp[:, ext]
        skin = np.zeros(S, bool)
        skin[2:] = (ext[2:] != blank) & (ext[2:] != ext[:-2])
        skout = np.zeros(S, bool)
        skout[:-2] = (ext[2:] != blank) & (ext[2:] != ext[:-2])
        alpha = np.full((Tn, S), NEG)
        alpha[0, :min(2, S)] = e[0, :min(2, S)]
        for t in range(1, Tn):
            p = alpha[t - 1]
            v1 = np.concatenate(([NEG], p[:-1]))
            v2 = np.where(skin, np.concatenate(([NEG, NEG], p[:-2]))[:S], NEG)
            alpha[t] = np.logaddexp(np.logaddexp(p, v1), v2) + e[t]
        llk = np.logaddexp(alpha[-1, S - 1], alpha[-1, S - 2] if S > 1 else NEG)
        costs[n] = -llk
        if llk == NEG:
            continue
        beta = np.full((Tn, S), NEG)
        beta[-1, max(0, S - 2):] = e[-1, max(0, S - 2):]
        for t in range(Tn - 2, -1, -1):
            p = beta[t + 1]
            v1 = np.concatenate((p[1:], [NEG]))
            v2 = np.where(skout, np.concatenate((p[2:], [NEG, NEG]))[:S], NEG)
            beta[t] = np.logaddexp(np.logaddexp(p, v1), v2) + e[t]
        with np.errstate(invalid="ignore"):
            W = np.exp(alpha + beta - e - llk)                     # alpha*beta / y / p(l|x)
        W = np.nan_to_num(W, nan=0.0)
        g = np.exp(lp)
        g[:, blank] -= _fixed_order_sum(W[:, 0::2])
        for c in range(C):
            states = [s for s in range(1, S, 2) if ext[s] == c]   # label order
            if states:
                g[:, c] -= _fixed_order_sum(W[:, states])
        grad[:Tn, n] = g
    return costs, grad


def _brute(x, seq, blank=0):
    """-log p and its gradient by enumerating every path of a tiny case."""
    T, C = x.shape
    lp = x - np.log(np.exp(x).sum(1, keepdims=True))
    p, occ = 0.0, np.zeros((T, C))
    for path in itertools.product(range(C), repeat=T):
        out, prev = [], None
        for c in path:
            if c != prev and c != blank:
                out.append(c)
            prev = c
        if out == list(seq):
            q = math.exp(sum(lp[t, c] for t, c in enumerate(path)))
            p += q
            for t, c in enumerate(path):
                occ[t, c] += q
    return -math.log(p), np.exp(lp) - occ / p


@pytest.mark.parametrize("seq,T", [([1], 1), ([1, 2], 3), ([1, 1], 3), ([2, 1, 2], 5), ([3, 3, 3], 6), ([1, 2, 3], 4)])
def test_restatement_equals_path_enumeration(seq, T):
    rng = np.random.default_rng(len(seq) * 10 + T)
    x = rng.standard_normal((T, 1, 4)) * 1.5
    c, g = ctc_long_ref(x, seq, [len(seq)], [T])
    cb, gb = _brute(x[:, 0], seq)
    assert abs(c[0] - cb) < 1e-12 * max(1.0, abs(cb))
    assert np.abs(g[:, 0] - gb).max() < 1e-12


def _long_batch(L, T, seed, N=2):
    rng = np.random.default_rng(seed)
    lab, ll, il = [], [], []
    for i in range(N):
        seq = rng.integers(1, 64, size=L)
        seq[3] = seq[2]                                          # a repeat
        lab += seq.tolist(); ll.append(L); il.append(T - 7 * i)
    return (rng.standard_normal((T, N, 64)) * 2.0), np.array(lab), np.array(ll), np.array(il)


def _torch_ref(x, lab, ll, il):
    xd = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    c = F.ctc_loss(torch.log_softmax(xd, 2), torch.tensor(lab), torch.tensor(il), torch.tensor(ll), blank=0, reduction="none")
    (g,) = torch.autograd.grad(c.sum(), xd)
    return c.detach().numpy(), g.numpy()


@pytest.mark.parametrize("L,T", [(64, 200), (64, 2048), (255, 600), (255, 2048), (639, 1400), (639, 2048)])
def test_restatement_equals_torch_ctc(L, T):
    x, lab, ll, il = _long_batch(L, T, seed=L + T)
    c, g = ctc_long_ref(x, lab, ll, il)
    cr, gr = _torch_ref(x, lab, ll, il)
    assert np.abs(c - cr).max() <= 1e-9 * np.abs(cr).max()
    assert np.abs(g - gr).max() <= 1e-9


@pytest.mark.parametrize("L,T", [(64, 150), (255, 560), (639, 1300)])
def test_restatement_equals_the_oracle(L, T):
    from oracle import crnn_oracle as O
    x, lab, ll, il = _long_batch(L, T, seed=L, N=1)
    c, g = ctc_long_ref(x, lab, ll, il)
    co, go = O.ctc_loss_np(x, lab, ll, il, blank=0)
    assert abs(c[0] - co[0]) <= 1e-9 * abs(co[0])
    assert np.abs(g - go).max() <= 1e-9


def test_restatement_semantics():
    """Lengths 0 / past T, an infeasible all-repeat label, a bad id and label_len > max_label_len."""
    rng = np.random.default_rng(0)
    T = 20
    x = rng.standard_normal((T, 5, 64))
    lab = [5] * 10 + [5] * 11 + [1, 2] + [0, 3] + [4] * 3
    ll, il = [10, 11, 2, 2, 3], [T, T, 0, T, T + 5]
    c, g = ctc_long_ref(x, lab, ll, il, max_label_len=10)
    assert c[0] > 0 and np.isfinite(c[0])                        # 10 repeats need 19 frames: fits in 20
    assert np.isnan(c[1]) and not g[:, 1].any()                  # label_len > max_label_len
    assert c[2] == 0 and not g[:, 2].any()                       # no frames
    assert np.isnan(c[3]) and not g[:, 3].any()                  # the blank as a label id
    assert np.isfinite(c[4])                                     # input_len clamped to T
    c, g = ctc_long_ref(x[:, :1], [5] * 11, [11], [T])            # 11 repeats need 21 frames
    assert c[0] == 0 and not g.any()


# ------------------------------------------------------------------------------------------------------- size query
def _size(T, N, m, C=64):
    from lstm_ctc_ocr_b200 import _lib
    nbytes = _lib.c_size_t(0)
    st = _lib.load().crnn_ctc_workspace_size(T, N, C, m, nbytes)
    return st, nbytes.value


def _formula(T, N, m):
    return 4 * N * T * (64 + ((2 * m + 1 + 3) // 4) * 4) + 256


def test_ctc_workspace_size_is_zero_inside_the_shared_memory_limits(monkeypatch):
    monkeypatch.delenv("CRNN_CTC_KERNEL", raising=False)
    for m, limit in ((0, 517), (4, 517), (15, 517), (16, 259), (31, 259), (32, 130), (63, 130)):
        for T in (1, limit // 2, limit):
            for N in (1, 1024):
                assert _size(T, N, m) == (0, 0), (T, N, m)
        assert _size(limit + 1, 4, m) == (0, _formula(limit + 1, 4, m)), m
    for m in (64, 100, 255, 639):
        assert _size(1, 3, m) == (0, _formula(1, 3, m))


def test_ctc_workspace_size_is_monotone_beyond_them(monkeypatch):
    monkeypatch.delenv("CRNN_CTC_KERNEL", raising=False)
    base = _size(600, 64, 255)[1]
    for T, N, m in ((601, 64, 255), (600, 65, 255), (600, 64, 258), (2048, 64, 255), (600, 512, 255), (600, 64, 639)):
        assert _size(T, N, m)[1] > base, (T, N, m)
    for T in (131, 260, 551, 1024, 2047):
        assert _size(T, 8, 100)[1] < _size(T + 1, 8, 100)[1]
    for N in (1, 2, 63, 255):
        assert _size(300, N, 70)[1] < _size(300, N + 1, 70)[1]
    for m in (64, 70, 255, 600):
        assert _size(300, 8, m)[1] <= _size(300, 8, m + 1)[1] and _size(300, 8, m)[1] < _size(300, 8, m + 2)[1]


def test_ctc_workspace_size_refusals(monkeypatch):
    from lstm_ctc_ocr_b200 import _lib
    monkeypatch.delenv("CRNN_CTC_KERNEL", raising=False)
    assert _size(10, 4, 640)[0] == 4 and _size(1, 1, 10 ** 6)[0] == 4              # CRNN_UNSUPPORTED above 639
    assert _size(2 ** 30, 1, 639)[0] == 4                                          # per-utterance floats overflow an int
    assert _size(2 ** 21, 2 ** 31 - 1, 639)[0] == 4
    for T, N, m in ((0, 4, 4), (-1, 4, 4), (8, 0, 4), (8, 4, -1)):
        assert _size(T, N, m)[0] == 1, (T, N, m)                                   # CRNN_INVALID_VALUE
    assert _size(8, 4, 4, C=65)[0] == 4
    assert _lib.load().crnn_ctc_workspace_size(8, 4, 64, 4, None) == 1
    _size(10, 4, 700)
    assert b"639" in _lib.load().crnn_last_error()


def test_forced_long_kernel_sizes_every_shape(monkeypatch):
    monkeypatch.setenv("CRNN_CTC_KERNEL", "long")
    assert _size(63, 64, 15) == (0, _formula(63, 64, 15))
    assert _size(1, 1, 0) == (0, _formula(1, 1, 0))


def test_engine_workspace_helpers_need_no_gpu(monkeypatch):
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200._lib import CrnnError
    monkeypatch.delenv("CRNN_CTC_KERNEL", raising=False)
    assert engine.ctc_workspace_bytes(255, 64, 64, 70) == _formula(255, 64, 70)
    assert engine.ctc_workspace_bytes(130, 64, 64, 63) == 0
    assert engine.CTC_MAX_LABEL_LEN == 639
    with pytest.raises(CrnnError, match="CRNN_UNSUPPORTED"):
        engine.ctc_workspace_bytes(100, 4, 64, 640)


def test_reference_surfaces_reject_labels_past_639():
    from lstm_ctc_ocr_b200.session import Session
    T, N = 400, 2
    data = np.zeros((N, 4 * (T + 1), 32), np.float32)
    tsl = np.full(N, T, np.int32)
    ll = np.array([640, 1], np.int32)
    with pytest.raises(ValueError, match="639"):
        Session.validate_feed(data, tsl, np.ones(641, np.int32), ll)
    Session.validate_feed(data, tsl, np.ones(640, np.int32), np.array([639, 1], np.int32))


# ----------------------------------------------------------------------------------------------------- feeder slot
def test_feeder_slot_bound_covers_every_line_at_max_len_70(monkeypatch):
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    if not gen.can_render():
        pytest.skip("no scalable font for PIL on this machine")
    monkeypatch.setattr(cfg, "MIN_LEN", 30)
    monkeypatch.setattr(cfg, "MAX_LEN", 70)
    bound = gen.line_width_bound()
    assert bound % 4 == 0 and bound == gen.line_width_bound(70)
    assert gen.line_width_bound(6) <= 256                         # the default lines keep the 256 px slot
    widest = 0
    for seed in range(3000):
        rng = random.Random(seed)
        text = gen.gen_rand(rng, 60 if seed % 2 else 30, 70)
        img = gen.render_line(text, rng=rng)
        nw = int(cfg.IMG_HEIGHT / img.shape[0] * img.shape[1])
        widest = max(widest, int(math.ceil(nw / cfg.POOL_SCALE) * cfg.POOL_SCALE))
    assert widest <= bound, (widest, bound)
    # and it is reached: a line of MAX_LEN copies of the widest glyph fills the slot exactly
    font = gen._font(42)
    wide = max(cfg.CHARSET, key=lambda c: int(font.getlength(c)))
    img = gen.render_line(wide * 70, rng=random.Random(0))
    assert int(math.ceil(int(cfg.IMG_HEIGHT / img.shape[0] * img.shape[1]) / cfg.POOL_SCALE) * cfg.POOL_SCALE) == bound
    img_list, _, _, _ = gen.make_batch(0, batch_size=8, render=True, seed=5)
    assert img_list[0].shape[0] <= bound
