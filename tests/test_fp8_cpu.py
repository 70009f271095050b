"""The fp8 path's arithmetic, restated without a GPU (compute_dtype 4, csrc/forward_fp8.cu):

- the e4m3 quantiser the kernels apply (cvt.rn.satfinite: round to nearest even, saturate to +-448, subnormals down to 2^-9)
  written out from its definition, bit-identical to x.clamp(-448, 448).to(torch.float8_e4m3fn) -- torch alone turns values
  above 448 into NaN, which the clamp removes;
- the power-of-two activation scale rule and the per-channel weight scale rule;
- the fp64 stage references of the GPU stage test (tests/stage_refs.py on quantised operands), chained from the oracle's conv1
  output through conv4_x, the BatchNorm applies into e4m3 and conv5's row-shift convolution, equal a direct fp64 evaluation
  of the same quantised graph."""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_refs as S  # noqa: E402
from test_gpu_fp8 import e4m3, scale_rule, weight_restatement  # noqa: E402


def e4m3_restated(x):
    """e4m3 of f32 values from the definition: |x| clamped to 448, quantum 2^(max(floor(log2 |x|), -6) - 3), ties to even."""
    x = np.asarray(x, np.float64)
    a = np.minimum(np.abs(x), 448.0)
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -6)))
    q = 2.0 ** (e - 3)
    r = np.round(a / q) * q                  # a / q is exact; np.round rounds half to even
    return np.where(np.isnan(x), np.nan, np.copysign(r, x))


def _bits(v):
    return torch.as_tensor(np.asarray(v, np.float32)).clamp(-448, 448).to(torch.float8_e4m3fn).view(torch.uint8).numpy()


def test_e4m3_quantiser_is_rne_with_saturation():
    rng = np.random.default_rng(0)
    grid = e4m3_restated(np.arange(-448, 449, 0.5 ** 9))              # includes every representable value
    specials = [0.0, -0.0, 2.0 ** -10, -(2.0 ** -10), 2.0 ** -9, 3 * 2.0 ** -11, 2.0 ** -6, 2.0 ** -6 * 0.96875, 448.0, 449.0,
                464.0, 465.0, 480.0, 1e30, -1e30, 240.0, 248.0, 232.0, 1.0 + 2 ** -4, 1.0 + 3 * 2 ** -4, 1.0 + 2 ** -4 + 2 ** -20]
    # ties: midpoints of every pair of neighbouring representable values, and one f32 ulp either side
    reps = np.unique(np.abs(grid))
    mids = (reps[1:] + reps[:-1]) / 2
    near = np.concatenate([mids, np.nextafter(mids.astype(np.float32), np.float32(np.inf)),
                           np.nextafter(mids.astype(np.float32), np.float32(0))])
    x = np.concatenate([specials, near, -near, rng.standard_normal(20000) * 10.0 ** rng.uniform(-4, 3, 20000)]).astype(np.float32)
    want = e4m3_restated(x)
    got = torch.as_tensor(_bits(x)).view(torch.float8_e4m3fn).double().numpy()
    assert np.array_equal(got, want), x[got != want][:10]
    # the cases named in the contract
    assert e4m3_restated(2.0 ** -10) == 0.0                            # the tie between 0 and the smallest subnormal goes to 0
    assert e4m3_restated(3 * 2.0 ** -11) == 2.0 ** -9
    assert e4m3_restated(1e30) == 448.0 and e4m3_restated(-1e30) == -448.0
    assert e4m3_restated(464.0) == 448.0                               # saturation, not a round-up to 480 (not e4m3fn)
    assert e4m3(torch.tensor([1e6, -1e6, 300.0])).tolist() == [448.0, -448.0, 288.0]


def test_activation_scale_rule():
    assert scale_rule(0.0) == 1.0 and scale_rule(float("inf")) == 1.0 and scale_rule(float("nan")) == 1.0
    assert scale_rule(448.0) == 1.0 and scale_rule(224.0) == 0.5 and scale_rule(np.nextafter(np.float32(448), np.float32(1e9))) == 2.0
    assert scale_rule(7 * 2.0 ** 6 * 2.0 ** -20) == 2.0 ** -20
    assert scale_rule(1e-38) == 2.0 ** -126                            # clamped: its reciprocal stays finite
    rng = np.random.default_rng(1)
    for a in (10.0 ** rng.uniform(-30, 30, 2000)).astype(np.float32):
        s = scale_rule(a)
        assert np.frexp(s)[0] == 0.5                                   # a power of two
        q = np.float32(a / np.float32(448.0))
        assert s / 2 < q <= s                                          # the smallest power of two at or above amax / 448
        assert a / s <= 448.0 * (1 + 2 ** -23)


def test_weight_scale_rule():
    rng = np.random.default_rng(2)
    w = (rng.standard_normal((3, 3, 16, 8)) * 0.05).astype(np.float32)
    w[..., 3] = 0.0                                                    # an all-zero channel gets scale 1
    q, s = weight_restatement(w)
    wk = w.reshape(-1, 8).T
    assert s[3] == 1.0 and not q[3].any()
    for co in (0, 1, 7):
        assert s[co] == np.float32(np.abs(wk[co]).max()) / np.float32(448.0)
        v = q[co].view(torch.float8_e4m3fn).double().numpy()
        assert np.abs(v).max() == 448.0                                # the channel's amax maps to the top of the range
        assert np.array_equal(v, e4m3_restated(np.float32(wk[co]) / np.float32(s[co])))


def _bn_direct(x, gamma, beta, eps):
    """tf.contrib.layers.batch_norm with batch statistics on NCHW fp64: (x - mean) / sqrt(var + eps) * gamma + beta."""
    mean = x.mean(dim=(0, 2, 3), keepdim=True)
    var = ((x - mean) ** 2).mean(dim=(0, 2, 3), keepdim=True)
    return (x - mean) / torch.sqrt(var + eps) * gamma[None, :, None, None] + beta[None, :, None, None]


def _direct_quantised_graph(a1, W, b, bn, s, eps):
    """The quantised graph conv2 .. conv5 written directly in NCHW fp64 (no stage_refs): e4m3 activations at the given scales,
    the e4m3 weights W (HWIO values), bf16 pre-BatchNorm outputs, batch-statistics BatchNorm, ReLU, the pools, conv5's 2x2
    VALID convolution over [N, H2, 2, 512]."""
    q = lambda x, sc: e4m3(x / sc) * sc                                 # noqa: E731
    conv = lambda x, k, pad=1: F.conv2d(x, W[k].permute(3, 2, 0, 1), b[k], padding=pad)  # noqa: E731
    x = a1.permute(0, 3, 1, 2)
    x = F.max_pool2d(torch.relu(conv(x, "conv2")), 2, 2)
    x = q(x, s[0])
    x = q(torch.relu(conv(x, "conv3_1")), s[1])
    x = q(F.max_pool2d(torch.relu(conv(x, "conv3_2")), (1, 2), (1, 2)), s[2])
    x = q(torch.relu(_bn_direct(S.bf16(conv(x, "conv4_1")), *bn["conv4_1"], eps)), s[3])
    x = torch.relu(_bn_direct(S.bf16(conv(x, "conv4_2")), *bn["conv4_2"], eps))
    x = q(F.max_pool2d(x, (1, 2), (1, 2)), s[4])                        # [N, 512, H2, 2]
    return conv(x, "conv5", 0)[:, :, :, 0].permute(0, 2, 1)              # [N, H2 - 1, 512]


def test_stage_references_chain_to_the_direct_quantised_graph():
    """conv2 .. conv5 through the stage references the GPU stage test uses, each output quantised as its producer does,
    against the same quantised graph evaluated directly."""
    from oracle import crnn_oracle as O
    pn = O.randomize_params(O.init_params(3, dtype=np.float32, logits_scale=10.0), seed=11)
    data, _, _, tsl = O.synth_batch(2, 24, seed=5, min_len=1, max_len=3)
    _, acts = O.forward(O.to_torch(pn), data, tsl, return_all=True)
    a1 = acts["conv1"].permute(0, 2, 3, 1).double()                     # the oracle's conv1 + pool1 output, NHWC
    P = {k: torch.as_tensor(np.asarray(v, np.float64)) for k, v in pn.items()}
    W = {"conv2": P["conv2/weights"]}
    for k in ("conv3_1", "conv3_2", "conv4_1", "conv4_2", "conv5"):
        q, sw = weight_restatement(pn[k + "/weights"])
        co, kh = q.shape[0], 2 if k == "conv5" else 3
        W[k] = (q.view(torch.float8_e4m3fn).double() * sw.double()[:, None]).reshape(co, kh, kh, -1).permute(1, 2, 3, 0)
    b = {k: P[k + "/biases"] for k in W}
    bn = {k: (P[f"{k}/{k}/gamma"], P[f"{k}/{k}/beta"]) for k in ("conv4_1", "conv4_2")}
    eps = float(np.float32(1e-3))
    # chained through the stage references, quantising each stage's output as the producer does; the activation scales come
    # from the rule applied to the chain's own amaxes
    s = []

    def quant(y):
        s.append(float(scale_rule(float(y.abs().max()))))
        return e4m3(y / s[-1]) * s[-1]
    a2 = quant(S.conv_relu_pool22_stage(a1, W["conv2"], b["conv2"])["out"])
    a3 = quant(S.conv_relu_stage(a2, W["conv3_1"], b["conv3_1"])["out"])
    a3p = quant(S.conv_relu_pool12_stage(a3, W["conv3_2"], b["conv3_2"])["out"])
    pre = S.bf16(S.conv_bias_stage(a3p, W["conv4_1"], b["conv4_1"])["out"])
    st = S.bn_stats_stage(pre, *bn["conv4_1"], eps)
    a4a = quant(S.bn_apply_relu_stage(pre, st["scale"], st["shift"])["out"])
    pre = S.bf16(S.conv_bias_stage(a4a, W["conv4_2"], b["conv4_2"])["out"])
    st = S.bn_stats_stage(pre, *bn["conv4_2"], eps)
    a4b = quant(S.bn_apply_relu_pool_stage(pre, st["scale"], st["shift"], rnd=S.ident)["out"])
    out = S.conv5_stage(a4b, W["conv5"], b["conv5"])["out"]
    direct = _direct_quantised_graph(a1, W, b, bn, s, eps)
    assert out.shape == direct.shape == (2, 5, 512)
    assert float((out - direct).abs().max()) <= 1e-9 * float(direct.abs().max())


# ---------------------------------------------------------------------------------------------------------- packed lines
PACKED_WIDTHS = [8, 12, 20, 36]


def _quantised_weights(seed=3):
    from oracle import crnn_oracle as O
    pn = O.randomize_params(O.init_params(seed, dtype=np.float32, logits_scale=10.0), seed=seed + 8)
    P = {k: torch.as_tensor(np.asarray(v, np.float64)) for k, v in pn.items()}
    W = {"conv2": S.bf16(P["conv2/weights"])}
    for k in ("conv3_1", "conv3_2", "conv4_1", "conv4_2", "conv5"):
        q, sw = weight_restatement(pn[k + "/weights"])
        co, kh = q.shape[0], 2 if k == "conv5" else 3
        W[k] = (q.view(torch.float8_e4m3fn).double() * sw.double()[:, None]).reshape(co, kh, kh, -1).permute(1, 2, 3, 0)
    b = {k: P[k + "/biases"] for k in W}
    bn = {k: (P[f"{k}/{k}/gamma"], P[f"{k}/{k}/beta"]) for k in ("conv4_1", "conv4_2")}
    return W, b, bn


def packed_fp8_reference(a1, lw, Wq, b, bn, scales=None, masks=True):
    """The fp8 graph conv2 .. conv5 over a packed batch as tests/test_gpu_fp8_edges.py restates it: each stage over the
    whole packed tensor through the stage references, then the line mask (zero at h >= W_i / 4) on the result; BatchNorm per
    line with count W_i.  a1 [N, H1, 16, 64] is zero at h >= W_i / 2.  scales None: each from the rule on its own amax.
    Returns the stage outputs (e4m3 values times their scale, bf16 pre-BN values, conv5) and the scales used."""
    N, H2 = a1.shape[0], a1.shape[1] // 2
    keep = torch.stack([torch.arange(H2) < (w // 4 if masks else H2) for w in lw]).double()[:, :, None, None]
    s = [] if scales is None else list(scales)
    out = {}

    def quant(name, i, y):
        if scales is None:
            s.append(float(scale_rule(float(y.abs().max()))))
        out[name] = e4m3(y * keep / s[i]) * s[i]
        return out[name]
    x = quant("conv2", 0, S.conv_relu_pool22_stage(a1, Wq["conv2"], b["conv2"])["out"])
    x = quant("conv3_1", 1, S.conv_relu_stage(x, Wq["conv3_1"], b["conv3_1"])["out"])
    x = quant("conv3_2", 2, S.conv_relu_pool12_stage(x, Wq["conv3_2"], b["conv3_2"])["out"])
    cnt = torch.tensor(lw, dtype=torch.float64)[:, None]
    for l, (k, pre) in enumerate((("conv4_1", "a4a_pre"), ("conv4_2", "a4b_pre"))):
        p = out[pre] = S.bf16(S.conv_bias_stage(x, Wq[k], b[k])["out"]) * keep
        st = S.bn_stats_stage(None, *bn[k], float(np.float32(1e-3)),
                              parts=dict(sum=p.sum((1, 2)), sumsq=(p * p).sum((1, 2)), sum_acc=p.abs().sum((1, 2)), cnt=cnt))
        sc, sh = st["scale"][:, None, None, :], st["shift"][:, None, None, :]
        y = S.bn_apply_relu_stage(p, sc, sh)["out"] if l == 0 else S.bn_apply_relu_pool_stage(p, sc, sh, rnd=S.ident)["out"]
        x = quant(k, 3 + l, y)
    out["conv5"] = S.conv5_stage(x, Wq["conv5"], b["conv5"])["out"]
    return out, s


def _packed_vs_alone(masks):
    """Worst relative difference, over every stage and line, between the packed reference and each line fed alone."""
    Wq, b, bn = _quantised_weights()
    W = max(PACKED_WIDTHS)
    rng = np.random.default_rng(4)
    a1 = torch.zeros((len(PACKED_WIDTHS), W // 2, 16, 64), dtype=torch.float64)
    for i, w in enumerate(PACKED_WIDTHS):
        a1[i, :w // 2] = torch.as_tensor(rng.random((w // 2, 16, 64)))
    packed, scales = packed_fp8_reference(a1, PACKED_WIDTHS, Wq, b, bn, masks=masks)
    worst = 0.0
    for i, w in enumerate(PACKED_WIDTHS):
        alone, _ = packed_fp8_reference(a1[i:i + 1, :w // 2], [w], Wq, b, bn, scales=scales)
        for k, a in alone.items():
            p = packed[k][i:i + 1, :a.shape[1]]
            worst = max(worst, float((p - a).abs().max()) / max(float(a.abs().max()), 1e-30))
    return worst


def test_packed_fp8_reference_equals_each_line_alone():
    """The shortcut of the GPU's packed-line check: a SAME convolution over the packed tensor (zero past each line), masked
    by line, is each line's own zero-padded convolution -- through e4m3 quantisation, per-line BatchNorm and conv5."""
    assert _packed_vs_alone(masks=True) <= 1e-12


def test_packed_fp8_reference_without_masks_differs():
    assert _packed_vs_alone(masks=False) > 1e-3
