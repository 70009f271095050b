"""CPU oracle for the CRNN+CTC hot path of ilovin/lstm_ctc_ocr.

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl
reference`` legs may import it.  The product path (``lstm_ctc_ocr_b200``) never
imports anything under ``oracle/``.

PARITY UNPINNED against the reference itself: it ships no tests or golden
vectors, and its arithmetic lives in TensorFlow 1.0.1 and baidu warp-ctc,
neither of which is importable here (no wheels for Python 3.12, no network).
This file restates the *published* semantics of those ops at the reference's
own call sites.  What it IS pinned to (``tests/test_oracle.py``):
  * the known answers those two third-party projects hold in their own unit
    tests for the loss / decode call sites of network.py:653-657
    (``tests/golden/third_party_kats.py``: tf.nn.ctc_loss testBasic == warp-ctc
    options_test -- costs to the 6 published digits, all 60 gradient entries to
    1e-6; ctc_greedy_decoder; ctc_beam_search_decoder's beam_width-2 vector,
    which only TF's candidate ordering / eviction rule reproduces);
  * independent implementations for everything else (torch ``F.ctc_loss``,
    ``torch.nn.LSTM`` with permuted gates, ``F.batch_norm``, brute-force CTC
    path enumeration, fp64 finite differences through the whole graph).
  * TensorFlow's small known answers for the LSTM cell step (rnn_cell_test
    testBasicLSTMCell), conv2d NHWC x HWIO / max_pool (conv_ops_test,
    pooling_ops_test) and clip_by_global_norm (clip_ops_test): equations and
    layouts, not the network's sizes.
BatchNorm and Adam have no externally held vector.

Reference call sites restated (paths relative to the reference checkout):
  * topology / hyper-parameters ......... lib/networks/LSTM_train.py:22-38
  * conv -> bias -> BN -> ReLU order ..... lib/networks/network.py:160-191
  * max_pool ksize/stride mapping ....... lib/networks/network.py:343-350
  * reshape_squeeze_layer ............... lib/networks/network.py:361-368
  * bi_lstm + 512->64 projection ........ lib/networks/network.py:97-129
  * build_loss (CTC mean + L2, decode) .. lib/networks/network.py:647-664
  * l2_regularizer ...................... lib/networks/network.py:630-637
  * batch contract (lengths, padding) ... lib/lstm/utils/gen.py:41-67
  * constants / label map ............... lib/lstm/config.py:15-28,73-81
  * accuracy (sequence equality) ........ lib/lstm/utils/training.py:26-37
  * clip_by_global_norm + Adam .......... lib/lstm/train.py:73-83

Third-party semantics restated from the upstream projects' documented behaviour
(TensorFlow 1.0.1 ``LSTMCell`` / ``bidirectional_dynamic_rnn`` /
``contrib.layers.batch_norm`` / ``AdamOptimizer`` / ``ctc_greedy_decoder``;
warp-ctc ``compute_ctc_loss``): gate order i,j,f,o; forget_bias 1.0; ``[x,h]``
concat order; zero output and carried state past ``sequence_length``; backward
direction = reverse_sequence(len) before and after; BN population variance with
eps 1e-3; warp-ctc softmax with max subtraction, blank 0, cost = -log p(l|x),
zero gradient for frames >= input_length, infeasible alignments (L + repeats >
T) -> cost 0 and zero gradient; TF Adam with eps outside the bias correction.
"""
from __future__ import annotations

import math
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

# ---------------------------------------------------------------------------
# constants (lib/lstm/config.py:15-28)
# ---------------------------------------------------------------------------
CHARSET = "0123456789abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ"
NCLASSES = len(CHARSET) + 2          # config.py:23 -> 64
IMG_HEIGHT = 32                      # config.py:19
POOL_SCALE = 4                       # config.py:17
OFFSET_TIME_STEP = -1                # config.py:15
NUM_HID = 512                        # config.py:48 (split //2 per direction, network.py:104-105)
HID = NUM_HID // 2
BN_EPS = 1e-3                        # tf.contrib.layers.batch_norm default epsilon
CTC_BLANK = 0                        # warp-ctc blank_label default (network.py:653-654)
TF_BLANK = NCLASSES - 1              # tf.nn.ctc_*_decoder blank = num_classes-1 (network.py:656)

# (name, kh, kw, cin, cout, bn, relu, padding) -- LSTM_train.py:24-34
CONV_SPECS = [
    ("conv1",   3, 3,   1,  64, False, True,  "SAME"),
    ("conv2",   3, 3,  64, 128, False, True,  "SAME"),
    ("conv3_1", 3, 3, 128, 256, False, True,  "SAME"),
    ("conv3_2", 3, 3, 256, 256, False, True,  "SAME"),
    ("conv4_1", 3, 3, 256, 512, True,  True,  "SAME"),
    ("conv4_2", 3, 3, 512, 512, True,  True,  "SAME"),
    ("conv5",   2, 2, 512, 512, False, False, "VALID"),
]
# pools applied AFTER the named conv: (k_h, k_w) == (s_h, s_w), VALID  (LSTM_train.py:25,27,30,33)
POOL_AFTER = {"conv1": (2, 2), "conv2": (2, 2), "conv3_2": (1, 2), "conv4_2": (1, 2)}

LSTM_FW = "logits/bidirectional_rnn/fw/lstm_cell"
LSTM_BW = "logits/bidirectional_rnn/bw/lstm_cell"


def param_specs():
    """Ordered (tf_name, shape) of the 24 trainable tensors (SURVEY §8(a))."""
    specs = []
    for name, kh, kw, ci, co, bn, _relu, _pad in CONV_SPECS:
        specs.append((f"{name}/weights", (kh, kw, ci, co)))       # HWIO, network.py:171
        specs.append((f"{name}/biases", (co,)))                   # network.py:173
        if bn:                                                    # network.py:177-178 (scope nested)
            specs.append((f"{name}/{name}/beta", (co,)))
            specs.append((f"{name}/{name}/gamma", (co,)))
    for scope in (LSTM_FW, LSTM_BW):
        specs.append((f"{scope}/weights", (NUM_HID + HID, 4 * HID)))   # rows [x(512); h(256)]
        specs.append((f"{scope}/biases", (4 * HID,)))
    specs.append(("logits/weights", (NUM_HID, NCLASSES)))         # network.py:121
    specs.append(("logits/biases", (NCLASSES,)))                  # network.py:123
    return specs


L2_NAMES = [f"{s[0]}/weights" for s in CONV_SPECS] + ["logits/weights"]   # network.py:171,121


def init_params(seed=3, dtype=np.float64, logits_scale=1.0):
    """Reference initialisers (network.py:168-169,119-120; TF defaults for the LSTM).

    ``logits_scale`` > 1 multiplies the logits matrix to give *peaked* outputs for
    decode-equality tests (SURVEY §7.2 item 5)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    p = OrderedDict()
    for name, shape in param_specs():
        if name.endswith("/weights") and len(shape) == 4:          # xavier uniform
            kh, kw, ci, co = shape
            lim = math.sqrt(6.0 / (kh * kw * ci + kh * kw * co))
            v = rng.uniform(-lim, lim, size=shape)
        elif name.endswith("lstm_cell/weights"):                  # glorot uniform (TF default)
            lim = math.sqrt(6.0 / (shape[0] + shape[1]))
            v = rng.uniform(-lim, lim, size=shape)
        elif name == "logits/weights":                            # variance_scaling(0.01, FAN_AVG, normal)
            std = math.sqrt(1.3 * 0.01 / ((shape[0] + shape[1]) / 2.0))
            v = np.clip(rng.normal(0.0, std, size=shape), -2 * std, 2 * std) * logits_scale
        elif name.endswith("/gamma"):
            v = np.ones(shape)
        else:                                                     # biases, beta
            v = np.zeros(shape)
        p[name] = np.ascontiguousarray(v, dtype=dtype)
    return p


def randomize_params(p, seed=11, scale=0.1):
    """Perturb biases / BN affine so tests exercise them (they are 0/1 at init)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    q = OrderedDict()
    for k, v in p.items():
        if k.endswith("/biases") or k.endswith("/beta"):
            q[k] = (v + scale * rng.standard_normal(v.shape)).astype(v.dtype)
        elif k.endswith("/gamma"):
            q[k] = (v + scale * rng.standard_normal(v.shape)).astype(v.dtype)
        else:
            q[k] = v.copy()
    return q


def to_torch(p, dtype=torch.float64, requires_grad=False):
    out = OrderedDict()
    for k, v in p.items():
        t = torch.as_tensor(np.asarray(v)).to(dtype).clone()
        t.requires_grad_(requires_grad)
        out[k] = t
    return out


# ---------------------------------------------------------------------------
# synthetic batch with the data layer's contract (gen.py:41-67; SURVEY §8(d))
# ---------------------------------------------------------------------------
def synth_batch(N, W, seed=3, widths=None, min_len=4, max_len=6, dtype=np.float32):
    """data [N,W,32] in [0,1) with exact-zero right padding, flat labels 1..62,
    label_len U{min_len..max_len}, time_step_len = nw//4 - 1 (gen.py:54)."""
    assert W % POOL_SCALE == 0
    rng = np.random.Generator(np.random.PCG64(seed))
    if widths is None:
        widths = np.full((N,), W, dtype=np.int64)
    widths = np.asarray(widths, dtype=np.int64)
    data = rng.random((N, W, IMG_HEIGHT)).astype(dtype)
    col = np.arange(W)[None, :, None]
    data = np.where(col < widths[:, None, None], data, 0).astype(dtype)
    label_len = rng.integers(min_len, max_len + 1, size=N).astype(np.int32)
    labels = rng.integers(1, len(CHARSET) + 1, size=int(label_len.sum())).astype(np.int32)
    time_step_len = (widths // POOL_SCALE + OFFSET_TIME_STEP).astype(np.int32)
    return data, labels, label_len, time_step_len


# ---------------------------------------------------------------------------
# forward graph (LSTM_train.py:22-38)
# ---------------------------------------------------------------------------
def conv_single(x, w_hwio, b, bn=None, relu=True, padding="SAME"):
    """network.py:160-182: conv2d -> bias_add -> (batch_norm, batch stats) -> relu.
    ``x`` is NCHW with H = image width (time) axis, W = image height axis."""
    w = w_hwio.permute(3, 2, 0, 1)                                 # HWIO -> OIHW
    pad = (w.shape[2] // 2, w.shape[3] // 2) if padding == "SAME" else 0
    y = F.conv2d(x, w, b, stride=1, padding=pad)
    stats = None
    if bn is not None:
        beta, gamma = bn
        mean = y.mean(dim=(0, 2, 3))                              # moments over N,H,W incl. padded cols
        var = y.var(dim=(0, 2, 3), unbiased=False)
        stats = (mean, var)
        y = (y - mean[None, :, None, None]) / torch.sqrt(var[None, :, None, None] + BN_EPS)
        y = y * gamma[None, :, None, None] + beta[None, :, None, None]
    if relu:
        y = torch.relu(y)
    return y, stats


def lstm_cell(xt, c, h, w, b):
    """One step of tf.contrib.rnn.LSTMCell (no peepholes, no projection; identical to BasicLSTMCell): w [(in+H), 4H] with rows
    [x; h], gate columns i,j,f,o, forget_bias 1.0.  Pinned to TensorFlow's own known answer (rnn_cell_test.py::testBasicLSTMCell)
    in tests/test_oracle.py::test_third_party_known_answer_lstm_cell."""
    H = w.shape[1] // 4
    z = torch.cat([xt, h], dim=1) @ w + b                          # [x,h] concat order
    i, j, f, o = z.split(H, dim=1)                                # TF gate order i,j,f,o
    c_new = torch.sigmoid(f + 1.0) * c + torch.sigmoid(i) * torch.tanh(j)   # forget_bias=1.0
    h_new = torch.sigmoid(o) * torch.tanh(c_new)
    return c_new, h_new


def lstm_direction(x, seq_len, w, b, reverse):
    """One tf.contrib.rnn.LSTMCell(256) under dynamic_rnn(sequence_length)
    (network.py:104-107).  x [N,T,512]; returns [N,T,256] with zeros past len."""
    N, T, _ = x.shape
    H = w.shape[1] // 4
    h = x.new_zeros((N, H))
    c = x.new_zeros((N, H))
    out = [None] * T
    lens = torch.as_tensor(np.asarray(seq_len), dtype=torch.long)
    ar = torch.arange(N)
    for s in range(T):
        active = (s < lens)
        if reverse:      # reverse_sequence(len): step s consumes frame len-1-s
            t_idx = torch.where(active, lens - 1 - s, torch.full_like(lens, s))
        else:
            t_idx = torch.full_like(lens, s)
        xt = x[ar, t_idx]                                         # [N,512]
        c_new, h_new = lstm_cell(xt, c, h, w, b)
        m = active[:, None].to(x.dtype)
        c = m * c_new + (1 - m) * c                               # state carried past len
        h = m * h_new + (1 - m) * h
        out[s] = (m * h_new, t_idx, active)
    y = x.new_zeros((N, T, H))
    for s in range(T):
        o_s, t_idx, active = out[s]
        # un-reverse: value produced at step s belongs to frame t_idx (zeros past len)
        y = y.index_put((ar, t_idx), o_s, accumulate=True)
    return y


def forward(params, data, time_step_len, return_all=False):
    """data [N,W,32] -> logits [T,N,64] (time-major, network.py:126-128)."""
    p = params
    dt = next(iter(p.values())).dtype
    x = torch.as_tensor(np.asarray(data)).to(dt)[:, None, :, :]   # NCHW: H=width/time, W=height
    acts = OrderedDict()
    for name, kh, kw, ci, co, bn, relu, pad in CONV_SPECS:
        bnp = (p[f"{name}/{name}/beta"], p[f"{name}/{name}/gamma"]) if bn else None
        x, stats = conv_single(x, p[f"{name}/weights"], p[f"{name}/biases"], bnp, relu, pad)
        if stats is not None:
            acts[name + "/bn_stats"] = stats
        if name in POOL_AFTER:
            x = F.max_pool2d(x, POOL_AFTER[name], POOL_AFTER[name])
        acts[name] = x
    N = x.shape[0]
    feat = x.permute(0, 2, 3, 1).reshape(N, -1, NUM_HID)          # reshape_squeeze_layer: [N,T,512]
    acts["reshaped_layer"] = feat
    fw = lstm_direction(feat, time_step_len, p[f"{LSTM_FW}/weights"], p[f"{LSTM_FW}/biases"], False)
    bw = lstm_direction(feat, time_step_len, p[f"{LSTM_BW}/weights"], p[f"{LSTM_BW}/biases"], True)
    lstm_out = torch.cat([fw, bw], dim=2)                         # [N,T,512]
    acts["lstm_out"] = lstm_out
    logits = lstm_out.reshape(-1, NUM_HID) @ p["logits/weights"] + p["logits/biases"]
    logits = logits.reshape(N, -1, NCLASSES).permute(1, 0, 2).contiguous()
    acts["logits"] = logits
    return (logits, acts) if return_all else logits


# ---------------------------------------------------------------------------
# CTC (warp-ctc compute_ctc_loss restated; call site network.py:653-654)
# ---------------------------------------------------------------------------
def _logsumexp2(a, b):
    if a == -np.inf:
        return b
    if b == -np.inf:
        return a
    m = max(a, b)
    return m + math.log(math.exp(a - m) + math.exp(b - m))


def ctc_loss_np(logits, flat_labels, label_len, input_len, blank=CTC_BLANK, want_grad=True):
    """Explicit alpha/beta restatement in float64 numpy.

    logits [T,N,C] unnormalised.  Returns (costs [N], grad [T,N,C]) where
    grad = d costs[n] / d logits[:,n,:] (what warp-ctc stores as its 2nd output).

    Defined deviation in the deep tail [upstream-memory]: warp-ctc forms the softmax PROBABILITIES in float first and takes
    their log inside the recursion, so a class more than ~87-103 below its frame's maximum underflows to probability 0 and
    a labelling that needs it costs +inf (its tests/test_cpu.cpp::inf_test sets a label's activations to -1e30 and expects
    exactly that, with a NaN-free gradient).  This restatement -- and the product kernels -- stay in log space (log-softmax
    = x - logsumexp), where the same labelling gets its finite -log p (2e30 in that test's setting).  Identical wherever no
    needed probability underflows float, i.e. for any logits a trained model of this path produces."""
    x = np.asarray(logits, dtype=np.float64)
    T, N, C = x.shape
    flat_labels = np.asarray(flat_labels).astype(np.int64)
    label_len = np.asarray(label_len).astype(np.int64)
    input_len = np.asarray(input_len).astype(np.int64)
    costs = np.zeros((N,), dtype=np.float64)
    grad = np.zeros_like(x)
    off = 0
    for n in range(N):
        L = int(label_len[n]); Tn = int(input_len[n])
        lab = flat_labels[off:off + L]; off += L
        repeats = int(np.sum(lab[1:] == lab[:-1])) if L > 1 else 0
        if L + repeats > Tn:          # warp-ctc: "not right to return 0" but it does
            continue
        S = 2 * L + 1
        ext = np.full((S,), blank, dtype=np.int64); ext[1::2] = lab
        xs = x[:Tn, n, :]
        mx = xs.max(axis=1, keepdims=True)
        lse = mx[:, 0] + np.log(np.exp(xs - mx).sum(axis=1))
        logp = xs - lse[:, None]                                   # log softmax
        e = logp[:, ext]                                           # [Tn,S]
        alpha = np.full((Tn, S), -np.inf)
        alpha[0, 0] = e[0, 0]
        if S > 1:
            alpha[0, 1] = e[0, 1]
        for t in range(1, Tn):
            for s in range(S):
                a = alpha[t - 1, s]
                if s >= 1:
                    a = _logsumexp2(a, alpha[t - 1, s - 1])
                if s >= 2 and ext[s] != blank and ext[s] != ext[s - 2]:
                    a = _logsumexp2(a, alpha[t - 1, s - 2])
                alpha[t, s] = a + e[t, s] if a != -np.inf else -np.inf
        ll = _logsumexp2(alpha[Tn - 1, S - 1], alpha[Tn - 1, S - 2] if S > 1 else -np.inf)
        costs[n] = -ll
        if not want_grad:
            continue
        beta = np.full((Tn, S), -np.inf)                           # beta includes emission at t
        beta[Tn - 1, S - 1] = e[Tn - 1, S - 1]
        if S > 1:
            beta[Tn - 1, S - 2] = e[Tn - 1, S - 2]
        for t in range(Tn - 2, -1, -1):
            for s in range(S):
                b = beta[t + 1, s]
                if s + 1 < S:
                    b = _logsumexp2(b, beta[t + 1, s + 1])
                if s + 2 < S and ext[s + 2] != blank and ext[s + 2] != ext[s]:
                    b = _logsumexp2(b, beta[t + 1, s + 2])
                beta[t, s] = b + e[t, s] if b != -np.inf else -np.inf
        y = np.exp(logp)
        for t in range(Tn):
            acc = np.zeros((C,))
            for s in range(S):
                v = alpha[t, s] + beta[t, s]
                if v != -np.inf:
                    acc[ext[s]] += math.exp(v - e[t, s] - ll)      # alpha*beta/y / p(l|x)
            grad[t, n, :] = y[t] - acc
    return costs, grad


def ctc_loss_torch(logits, flat_labels, label_len, input_len, blank=CTC_BLANK):
    """Differentiable restatement (for autograd through the whole graph).
    Uses torch's CTC (same maths) but applies warp-ctc's infeasible -> 0 rule."""
    T, N, C = logits.shape
    lp = F.log_softmax(logits, dim=2)
    ll = torch.as_tensor(np.asarray(label_len), dtype=torch.long)
    il = torch.as_tensor(np.asarray(input_len), dtype=torch.long)
    fl = torch.as_tensor(np.asarray(flat_labels), dtype=torch.long)
    costs = F.ctc_loss(lp, fl, il, ll, blank=blank, reduction="none", zero_infinity=True)
    return costs


def greedy_decode(logits, input_len, tf_blank=TF_BLANK, strip=0):
    """North-star 'greedy' restatement of network.py:656-657 + training.py:32
    (SURVEY §8(c)): argmax per frame (lowest index on ties) for t < len; emit iff
    != tf_blank and != previous *raw* argmax; then drop ``strip`` (0)."""
    x = np.asarray(logits)
    T, N, C = x.shape
    out = []
    for n in range(N):
        prev = -1
        seq = []
        for t in range(int(input_len[n])):
            a = int(np.argmax(x[t, n]))
            if a != tf_blank and a != prev:
                seq.append(a)
            prev = a
        out.append([v for v in seq if v != strip])
    return out


class _Beam(object):
    """One prefix of TF's CTC beam search tree (ctc_beam_entry.h [upstream-memory]): log-probabilities of the prefix ending
    in blank / in its last label at the previous (`old`) and the current (`new`) frame."""
    __slots__ = ("parent", "label", "children", "old", "new")

    def __init__(self, parent, label):
        self.parent, self.label, self.children = parent, label, None
        self.old = [-np.inf, -np.inf, -np.inf]     # total, blank, label
        self.new = [-np.inf, -np.inf, -np.inf]

    def active(self):
        return self.new[0] > -np.inf

    def label_seq(self, merge_repeated):
        out, c, prev = [], self, -1
        seq = []
        while c.parent is not None:
            seq.append(c.label)
            c = c.parent
        for l in reversed(seq):
            if not merge_repeated or l != prev:
                out.append(l)
            prev = l
        return out


def beam_search_decode(logits, input_len, beam_width=100, merge_repeated=True, strip=0):
    """What the reference actually calls at network.py:656-657 / test.py:30:
    ``tf.nn.ctc_beam_search_decoder(logits, seq_len, merge_repeated=True)`` (beam_width 100, top_paths 1, blank = C-1)
    followed by the zero stripping of training.py:32.  [upstream-memory] restatement of TensorFlow 1.0's
    ``CTCBeamSearchDecoder::Step`` / ``TopPaths`` (core/util/ctc/ctc_beam_search.h): prefix beam search over log-softmax
    frames with per-prefix (blank, label) probabilities, candidates grown branch by branch in descending order against the
    running bottom of a beam_width-bounded top-N list, and -- the part that differs from greedy decoding even on peaked
    outputs -- ``merge_repeated=True`` collapsing consecutive equal labels of the DECODED sequence.  Test infrastructure
    only: it quantifies the defined deviation of the product's greedy decode (SURVEY 8(c)); nothing is pinned against TF."""
    x = np.asarray(logits, dtype=np.float64)
    T, N, C = x.shape
    blank = C - 1
    lse = lambda a, b: (max(a, b) + np.log1p(np.exp(-abs(a - b)))) if max(a, b) > -np.inf else -np.inf
    out = []
    for n in range(N):
        root = _Beam(None, -1)
        root.new = [0.0, 0.0, -np.inf]
        leaves = [root]
        for t in range(int(input_len[n])):
            row = x[t, n]
            # log-softmax in double with a SEQUENTIAL sum (not numpy's pairwise one): on frames with exactly tied scores the
            # decode depends on the last bit of the normaliser, and this is the arithmetic the product decoder states too
            mx = float(row.max())
            se = 0.0
            for v in row:
                se += math.exp(float(v) - mx)
            lp = row - (mx + math.log(se))
            branches = sorted(leaves, key=lambda b: -b.new[0])
            leaves = []
            for b in branches:
                b.old = list(b.new)
            for b in branches:
                if b.parent is not None:
                    if b.parent.active():
                        prev = b.parent.old[1] if b.label == b.parent.label else b.parent.old[0]
                        b.new[2] = lse(b.new[2], prev)
                    b.new[2] += lp[b.label]
                b.new[1] = b.old[0] + lp[blank]
                b.new[0] = lse(b.new[1], b.new[2])
                leaves.append(b)
            bottom = lambda: min(leaves, key=lambda e: e.new[0])

            state = {"bot": bottom().new[0]}              # total of the bottom, refreshed whenever the list changes

            def is_candidate(total):
                return total > -np.inf and (len(leaves) < beam_width or total > state["bot"])
            # CTCBeamSearchDecoder::Step's "grow new leaves" loop visits EVERY child of a candidate branch in class order, and
            # the visit order is observable: a branch that an insertion evicted earlier in this frame is still expanded when the
            # loop reaches it (its `old` survives the eviction) unless its parent's visit came first and rejected -- i.e. wiped
            # -- it.  Restated without the C-1 visits per branch: a child object exists only once it has entered the beam
            # (`children` is a dict), a child that never did has nothing to wipe, so the visit covers the classes that can still
            # enter (total above the bottom as of the start of the visit: the bottom only rises) plus every existing child.
            for b in branches:
                if not is_candidate(b.old[0]):
                    continue
                if b.children is None:
                    b.children = {}
                base = np.full(C - 1, b.old[0])
                if 0 <= b.label < C - 1:
                    base[b.label] = b.old[1]
                cand = base + lp[:C - 1]
                if len(leaves) < beam_width:
                    visit = range(C - 1)
                else:
                    visit = sorted(set(np.nonzero(cand > state["bot"])[0].tolist()) | set(b.children))
                for c in visit:
                    ch = b.children.get(c)
                    if ch is not None and ch.active():
                        continue
                    total = float(cand[c])
                    if is_candidate(total):
                        if ch is None:
                            ch = b.children[c] = _Beam(b, c)
                        ch.new = [total, -np.inf, total]
                        if len(leaves) == beam_width:
                            bt = bottom()
                            bt.new = [-np.inf, -np.inf, -np.inf]
                            leaves.remove(bt)
                        leaves.append(ch)
                        state["bot"] = bottom().new[0]
                    elif ch is not None:
                        ch.old = [-np.inf, -np.inf, -np.inf]
                        ch.new = [-np.inf, -np.inf, -np.inf]
        best = max(leaves, key=lambda e: e.new[0])
        out.append([v for v in best.label_seq(merge_repeated) if v != strip])
    return out


def dense_decoded(seqs, pad=0):
    """sparse_tensor_to_dense(default 0) (network.py:657) -> [N, maxlen] int32."""
    m = max([len(s) for s in seqs] + [0])
    d = np.full((len(seqs), m), pad, dtype=np.int32)
    for i, s in enumerate(seqs):
        d[i, :len(s)] = s
    return d


def accuracy_calculation(original_seq, decoded_seq, ignore_value=0):
    """training.py:26-37 (without the prints)."""
    if len(original_seq) != len(decoded_seq):
        return 0
    count = 0
    for org, dec in zip(original_seq, decoded_seq):
        if [l for l in org if l != ignore_value] == [j for j in dec if j != ignore_value]:
            count += 1
    return count * 1.0 / len(original_seq)


def l2_reg(params, wd):
    """network.py:630-637,660-662: sum_k wd * sum(w_k^2)/2 over conv kernels + logits W."""
    tot = 0.0
    for k in L2_NAMES:
        tot = tot + wd * 0.5 * (params[k] ** 2).sum()
    return tot


def build_loss(params, data, flat_labels, label_len, time_step_len, wd=1e-5):
    """network.py:647-664 -> (loss, ctc costs [N], logits, decoded lists)."""
    logits = forward(params, data, time_step_len)
    costs = ctc_loss_torch(logits, flat_labels, label_len, time_step_len)
    loss = costs.mean()
    if wd > 0:
        loss = loss + l2_reg(params, wd)
    dec = greedy_decode(logits.detach().numpy(), time_step_len)
    return loss, costs, logits, dec


# ---------------------------------------------------------------------------
# optimizer half of the solver (lib/lstm/train.py:73-83)
# ---------------------------------------------------------------------------
def clip_by_global_norm(grads, clip=10.0):
    gn = math.sqrt(sum(float((g.double() ** 2).sum()) for g in grads.values()))
    scale = clip / max(gn, clip)
    return OrderedDict((k, g * scale) for k, g in grads.items()), gn


def adam_step(params, grads, m, v, step, lr=1e-4, b1=0.9, b2=0.999, eps=1e-8):
    """TF AdamOptimizer: lr_t = lr*sqrt(1-b2^t)/(1-b1^t); theta -= lr_t*m/(sqrt(v)+eps)."""
    lr_t = lr * math.sqrt(1 - b2 ** step) / (1 - b1 ** step)
    for k in params:
        m[k] = b1 * m[k] + (1 - b1) * grads[k]
        v[k] = b2 * v[k] + (1 - b2) * grads[k] ** 2
        params[k] = params[k] - lr_t * m[k] / (torch.sqrt(v[k]) + eps)
    return params, m, v


def train_step(params_np, batch, m=None, v=None, step=1, lr=1e-4, wd=1e-5, clip=10.0, dtype=torch.float64):
    """One full solver iteration (train.py:129-130) via autograd on the restated graph."""
    data, labels, label_len, tsl = batch
    p = to_torch(params_np, dtype, requires_grad=True)
    loss, costs, logits, _ = build_loss(p, data, labels, label_len, tsl, wd)
    loss.backward()
    grads = OrderedDict((k, t.grad.detach().clone()) for k, t in p.items())
    clipped, gn = clip_by_global_norm(grads, clip)
    pd = OrderedDict((k, t.detach().clone()) for k, t in p.items())
    if m is None:
        m = OrderedDict((k, torch.zeros_like(t)) for k, t in pd.items())
        v = OrderedDict((k, torch.zeros_like(t)) for k, t in pd.items())
    pd, m, v = adam_step(pd, clipped, m, v, step, lr)
    return dict(loss=float(loss), costs=costs.detach().numpy(), logits=logits.detach().numpy(),
                grads=grads, grad_norm=gn, params=pd, m=m, v=v)


# ---------------------------------------------------------------------------
# fp32 unfused CPU baseline (BASELINE.md §3) -- the timed "reference port"
# ---------------------------------------------------------------------------
@torch.no_grad()
def fwd_ctc_fp32(params_t32, data, labels, label_len, tsl, wd=1e-5):
    logits = forward(params_t32, data, tsl)
    costs = ctc_loss_torch(logits, labels, label_len, tsl)
    loss = costs.mean() + l2_reg(params_t32, wd)
    return float(loss), logits
