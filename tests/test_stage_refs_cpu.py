"""CPU self-check of the per-stage fp64 references in tests/stage_refs.py (no GPU needed).

The stages are chained starting from the oracle's own fp64 activations, with identity rounding, through the workspace
layouts the GPU uses (permuted and reversed input projection, saved gates / cell state per 128-row tile, time-major logits,
frame rows of d logits).  The chain must reproduce crnn_oracle.forward(..., return_all=True) and the oracle's autograd
gradients to 1e-9 relative.  This pins the references, the gate permutation, the reversal, the window-index encoding and
the BatchNorm formulas before any GPU compares against them, so a wrong reference can neither hide a kernel bug nor
invent one."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stage_refs as S  # noqa: E402
from oracle import crnn_oracle as O  # noqa: E402

TOL = 1e-9
FW, BW = O.LSTM_FW, O.LSTM_BW


def rel(a, b):
    a = torch.as_tensor(a, dtype=torch.float64).detach()
    b = torch.as_tensor(b, dtype=torch.float64).detach()
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-30))


# the widths evaluation feeds beyond 3 x 24: T = 1 and 2 (a crop a few pixels wide; lengths 0, 1 and 2) and T = 128
# (W = 516, H = 129: the backward rows of the input projection cross a 128-row tile)
EDGE_CHAINS = [pytest.param((3, 8, [8, 8, 4]), id="N3_W8"), pytest.param((2, 12, [12, 9]), id="N2_W12"),
               pytest.param((1, 516, [516]), id="N1_W516")]


def _make_chain(N, W, widths):
    torch.manual_seed(0)
    p = O.randomize_params(O.init_params(3, dtype=np.float64, logits_scale=3.0), scale=0.3)
    data, lab, ll, tsl = O.synth_batch(N, W, seed=7, widths=widths, min_len=1, max_len=2, dtype=np.float64)
    pt = O.to_torch(p, requires_grad=True)
    logits, acts = O.forward(pt, data, tsl, return_all=True)
    loss = O.ctc_loss_torch(logits, lab, ll, tsl).mean()
    names = list(pt.keys())
    g = torch.autograd.grad(loss, [logits] + [pt[k] for k in names])
    dlogits = g[0].detach()
    grads = dict(zip(names, [t.detach() for t in g[1:]]))
    P = {k: v.detach() for k, v in pt.items()}
    A = {k: (S.nhwc(v.detach()) if isinstance(v, torch.Tensor) and v.dim() == 4 else v) for k, v in acts.items()}
    return dict(N=N, W=W, T=W // 4 - 1, H2=W // 4, tsl=tsl, data=torch.as_tensor(data), P=P, A=A, logits=logits.detach(),
                dlogits=dlogits, grads=grads)


@pytest.fixture(scope="module")
def chain():
    return _make_chain(3, 24, [24, 17, 4])


@pytest.fixture(scope="module", params=EDGE_CHAINS)
def edge_chain(request):
    return _make_chain(*request.param)


def _pad_rows(x, H2):
    out = x.new_zeros((x.shape[0], H2) + tuple(x.shape[2:]))
    out[:, :x.shape[1]] = x
    return out


def _forward_chain(c):
    P, A, T, H2, tsl = c["P"], c["A"], c["T"], c["H2"], c["tsl"]
    r = {}
    r["conv1"] = S.conv1_stage(c["data"], P["conv1/weights"], P["conv1/biases"])
    r["conv2"] = S.conv_relu_pool22_stage(A["conv1"], P["conv2/weights"], P["conv2/biases"])
    r["conv3_1"] = S.conv_relu_stage(A["conv2"], P["conv3_1/weights"], P["conv3_1/biases"])
    r["conv3_2"] = S.conv_relu_pool12_stage(A["conv3_1"], P["conv3_2/weights"], P["conv3_2/biases"])
    for name, src in (("conv4_1", "conv3_2"), ("conv4_2", "conv4_1")):
        pre = S.conv_bias_stage(A[src], P[f"{name}/weights"], P[f"{name}/biases"])["out"]
        st = S.bn_stats_stage(pre, P[f"{name}/{name}/gamma"], P[f"{name}/{name}/beta"], O.BN_EPS)
        if name == "conv4_1":
            ap = S.bn_apply_relu_stage(pre, st["scale"], st["shift"])
        else:
            ap = S.bn_apply_relu_pool_stage(pre, st["scale"], st["shift"], rnd=S.ident)
        r[name] = dict(pre=pre, st=st, out=ap["out"], bn=torch.stack([st["scale"], st["shift"], st["mean"], st["invstd"]]))
    r["conv5"] = S.conv5_stage(A["conv4_2"], P["conv5/weights"], P["conv5/biases"])
    a5 = _pad_rows(A["reshaped_layer"], H2)
    r["a5"] = a5
    r["xproj"] = S.xproj_stage(a5, P[f"{FW}/weights"][:512], P[f"{BW}/weights"][:512], P[f"{FW}/biases"], P[f"{BW}/biases"],
                               tsl, T, bias_rnd=S.ident)
    r["rec"] = S.recurrence_stage(r["xproj"]["out"], P[f"{FW}/weights"][512:], P[f"{BW}/weights"][512:], tsl, T, rnd=S.ident)
    r["logits"] = S.logits_stage(r["rec"]["out"], P["logits/weights"], P["logits/biases"], T)
    return r


def test_forward_stage_chain_reproduces_the_oracle(chain):
    _check_forward_chain(chain)


def test_forward_stage_chain_at_edge_widths(edge_chain):
    _check_forward_chain(edge_chain)


def _check_forward_chain(c):
    r = _forward_chain(c)
    A, T, H2 = c["A"], c["T"], c["H2"]
    for k in ("conv1", "conv2", "conv3_1", "conv3_2", "conv4_1", "conv4_2"):
        assert rel(r[k]["out"], A[k]) < TOL, k
    for k in ("conv4_1", "conv4_2"):
        mean, var = A[k + "/bn_stats"]
        assert rel(r[k]["st"]["mean"], mean.detach()) < TOL and rel(r[k]["st"]["var"], var.detach()) < TOL, k
    assert rel(r["conv5"]["out"], A["reshaped_layer"]) < TOL
    assert rel(r["rec"]["out"], _pad_rows(A["lstm_out"].detach(), H2)) < TOL
    assert rel(r["logits"]["out"], c["logits"]) < TOL
    # the per-step isolated recurrence, fed the chain's own h and c, reproduces every active step
    P, tsl = c["P"], c["tsl"]
    iso = S.recurrence_steps_isolated(r["xproj"]["out"], P[f"{FW}/weights"][512:], P[f"{BW}/weights"][512:], r["rec"]["out"],
                                      r["rec"]["c"], tsl, T)
    act = torch.arange(T)[None, :] < torch.as_tensor(S.clamp_lens(tsl, T))[:, None]
    for k in ("gates", "c"):
        assert rel(iso[k][:, act], r["rec"][k][:, act]) < TOL, k
    # the xproj layout: backward-direction rows reversed within each length, padding rows untouched
    L = S.clamp_lens(tsl, T)
    xp = r["xproj"]["out"]
    for n in range(c["N"]):
        for t in range(H2):
            src = (L[n] - 1 - t) if t < L[n] else t
            assert torch.equal(xp[n, t, 1024:], S.reverse_rows(xp, tsl, T)[n, src, 1024:])


def test_layout_helpers_round_trip():
    g = torch.randn(2, 130, 5, 4, 256, dtype=torch.float64)
    assert torch.equal(S.unpack_gates(S.pack_gates(g, 256), 130), g)
    c = torch.randn(2, 130, 5, 256, dtype=torch.float64)
    assert torch.equal(S.unpack_csave(S.pack_csave(c, 256), 130), c)
    z = torch.randn(7, 1024, dtype=torch.float64)
    assert torch.equal(S.from_perm(S.to_perm(z)), z)
    # lstm_perm: TF column g*256 + u -> (u/32)*128 + g*32 + u%32
    perm = S.gate_perm()
    assert int(perm[2 * 256 + 33]) == 1 * 128 + 2 * 32 + 1 and int(perm[255]) == 7 * 128 + 31


def test_backward_stage_chain_reproduces_oracle_gradients(chain):
    _check_backward_chain(chain)


def test_backward_stage_chain_at_edge_widths(edge_chain):
    _check_backward_chain(edge_chain)


def _check_backward_chain(c):
    r = _forward_chain(c)
    P, A, G, T, H2, tsl, eps = c["P"], c["A"], c["grads"], c["T"], c["H2"], c["tsl"], O.BN_EPS
    got = {}
    dl = S.dl_rows_stage(c["dlogits"], H2)
    got["logits/biases"] = dl["dbias"]
    lb = S.logits_bwd(r["rec"]["out"], dl["dl_rows"], P["logits/weights"])
    got["logits/weights"] = lb["dw"]
    bp = S.bptt_stage(lb["d_lstm_out"], r["rec"]["gates"], r["rec"]["c"], P[f"{FW}/weights"][512:], P[f"{BW}/weights"][512:],
                      tsl, T, rnd=S.ident)
    # the semi-isolated form (dz of the next step read back from dz_all) agrees with the self-fed one
    bp2 = S.bptt_stage(lb["d_lstm_out"], r["rec"]["gates"], r["rec"]["c"], P[f"{FW}/weights"][512:], P[f"{BW}/weights"][512:],
                       tsl, T, dz_in=bp["dz"])
    assert rel(bp2["dz"], bp["dz"]) < TOL
    lg = S.lstm_grads_stage(bp["dz"], r["a5"], r["rec"]["out"], P[f"{FW}/weights"][:512], P[f"{BW}/weights"][:512],
                            P[f"{FW}/weights"][512:], P[f"{BW}/weights"][512:])
    for d, scope in (("fw", FW), ("bw", BW)):
        got[f"{scope}/weights"] = lg[f"{d}/weights"]
        got[f"{scope}/biases"] = lg[f"{d}/biases"]
    c5 = S.conv5_bwd(lg["d_a5"], A["conv4_2"], P["conv5/weights"])
    got["conv5/weights"], got["conv5/biases"] = c5["dw"], c5["db"]
    d_a4b = c5["dx"]
    b42 = S.bn_relu_pool_bwd_stage(d_a4b, r["conv4_2"]["pre"], r["conv4_2"]["bn"], P["conv4_2/conv4_2/gamma"], eps,
                                   rnd=S.ident)
    got["conv4_2/conv4_2/gamma"], got["conv4_2/conv4_2/beta"] = b42["dgamma"], b42["dbeta"]
    got["conv4_2/weights"] = S.conv_bwd(b42["dx"], A["conv4_1"], P["conv4_2/weights"])["dw"]
    bn41 = r["conv4_1"]["bn"]
    b41 = S.conv_bn_relu_bwd_stage(b42["dx"], r["conv4_1"]["pre"], bn41, P["conv4_1/conv4_1/gamma"], P["conv4_2/weights"], eps,
                                   mask=(r["conv4_1"]["pre"] * bn41[0] + bn41[1] > 0).double(), rnd=S.ident)
    got["conv4_1/conv4_1/gamma"], got["conv4_1/conv4_1/beta"] = b41["dgamma"], b41["dbeta"]
    c41 = S.conv_bwd(b41["dx"], A["conv3_2"], P["conv4_1/weights"])
    got["conv4_1/weights"] = c41["dw"]
    d_pre32 = S.unpool_stage(c41["dx"], A["conv3_2"], r["conv3_2"]["am"], 2)
    got["conv3_2/biases"] = S.masked_colsum(c41["dx"], A["conv3_2"])[0]
    c32 = S.conv_bwd(d_pre32, A["conv3_1"], P["conv3_2/weights"])
    got["conv3_2/weights"] = c32["dw"]
    d_pre31 = c32["dx"] * (A["conv3_1"] > 0)
    c31 = S.conv_bwd(d_pre31, A["conv2"], P["conv3_1/weights"])
    got["conv3_1/weights"], got["conv3_1/biases"] = c31["dw"], c31["db"]
    d_pre2 = S.unpool_stage(c31["dx"], A["conv2"], r["conv2"]["am"], 4)
    got["conv2/biases"] = S.masked_colsum(c31["dx"], A["conv2"])[0]
    c2 = S.conv_bwd(d_pre2, A["conv1"], P["conv2/weights"])
    got["conv2/weights"] = c2["dw"]
    c1 = S.conv1_wgrad_stage(c2["dx"], A["conv1"], r["conv1"]["am"], c["data"], P["conv1/weights"])
    got["conv1/weights"], got["conv1/biases"] = c1["dw"], c1["db"]
    for k, v in got.items():
        assert rel(v, G[k]) < TOL, (k, rel(v, G[k]))
    # the biases in front of a batch-statistics BatchNorm have an analytically zero gradient (the kernels leave them at 0)
    for k in ("conv4_1/biases", "conv4_2/biases"):
        assert float(G[k].abs().max()) < 1e-12 * float(G[k.replace("biases", "weights")].abs().max()) + 1e-15
    assert len(got) == len(G) - 2


def test_bptt_steps_reproduce_the_chain(chain):
    _check_bptt_steps(chain)


def test_bptt_steps_at_edge_widths(edge_chain):
    _check_bptt_steps(edge_chain)


def _check_bptt_steps(c):
    """Fed the fp64 chain's own values (no rounding; dz from bptt_stage itself), every isolated BPTT step reproduces
    bptt_stage, and the dc recovered from each step's dz equals the chain's dc wherever a successor recovers it."""
    r = _forward_chain(c)
    P, T, H2, tsl = c["P"], c["T"], c["H2"], c["tsl"]
    wh = (P[f"{FW}/weights"][512:], P[f"{BW}/weights"][512:])
    d_out = S.logits_bwd(r["rec"]["out"], S.dl_rows_stage(c["dlogits"], H2)["dl_rows"], P["logits/weights"])["d_lstm_out"]
    bp = S.bptt_stage(d_out, r["rec"]["gates"], r["rec"]["c"], wh[0], wh[1], tsl, T, rnd=S.ident)
    bs = S.bptt_steps_isolated(d_out, r["rec"]["gates"], r["rec"]["c"], wh[0], wh[1], bp["dz"], tsl, T, rnd=S.ident)
    act = bs["active"]
    assert rel(bs["dz"][act], bs["gpu"][act]) < 1e-12
    assert rel(bs["dc"][act], bp["dc"][act]) < 1e-12
    rec = bs["recovered"][:, :, :-1]                   # the carry into step s recovered from step s+1
    assert int(bs["fallback"].sum()) == 0
    assert int(rec.sum()) == int(act[:, :, 1:].sum()) * S.HID
    if T > 1:
        assert rel(bs["dc_hat"][:, :, 1:][rec], bp["dc"][:, :, 1:][rec]) < 1e-12
    assert torch.equal(bs["dz"][:, :, 0, 2][act[:, :, 0]], torch.zeros_like(bs["dz"][:, :, 0, 2][act[:, :, 0]]))


# ---------------------------------------------------------------------------------------------------------- f32-class path
def _zero_pair(x):
    return (x, torch.zeros_like(x))


def test_x3_stage_chain_reproduces_the_oracle(chain):
    _check_x3_chain(chain)


def test_x3_stage_chain_at_edge_widths(edge_chain):
    _check_x3_chain(edge_chain)


def _check_x3_chain(c):
    """The f32-class layouts with lo = 0, wl = 0 and identity rounding: split-pair conv / GEMM stages, an input projection
    without bias in natural gate and frame order, the cell adding the bias and reading frame len-1-step backwards."""
    P, A, T, H2, tsl = c["P"], c["A"], c["T"], c["H2"], c["tsl"]
    Wp = {k: _zero_pair(v) for k, v in P.items() if k.endswith("weights")}
    for k, src, fn in (("conv2", "conv1", S.conv_relu_pool22_stage), ("conv3_1", "conv2", S.conv_relu_stage),
                       ("conv3_2", "conv3_1", S.conv_relu_pool12_stage)):
        assert rel(fn(_zero_pair(A[src]), Wp[f"{k}/weights"], P[f"{k}/biases"])["out"], A[k]) < TOL, k
    for name, src in (("conv4_1", "conv3_2"), ("conv4_2", "conv4_1")):
        pre = S.conv_bias_stage(_zero_pair(A[src]), Wp[f"{name}/weights"], P[f"{name}/biases"])["out"]
        st = S.bn_stats_stage(pre, P[f"{name}/{name}/gamma"], P[f"{name}/{name}/beta"], O.BN_EPS)
        fn = S.bn_apply_relu_stage if name == "conv4_1" else lambda x, a, b: S.bn_apply_relu_pool_stage(x, a, b, rnd=S.ident)
        assert rel(fn(pre, st["scale"], st["shift"])["out"], A[name]) < TOL, name
    assert rel(S.conv5_stage(_zero_pair(A["conv4_2"]), Wp["conv5/weights"], P["conv5/biases"])["out"], A["reshaped_layer"]) < TOL
    a5 = _pad_rows(A["reshaped_layer"], H2)
    wx = [S.pair_map(lambda v: v[:512], Wp[f"{s}/weights"]) for s in (FW, BW)]
    wh = [S.pair_map(lambda v: v[512:], Wp[f"{s}/weights"]) for s in (FW, BW)]
    biases = (P[f"{FW}/biases"], P[f"{BW}/biases"])
    xp = S.xproj_stage(_zero_pair(a5), wx[0], wx[1], None, None, tsl, T, x3=True)["out"]
    # natural layout: plain a5 W_x per direction, no bias, no permutation, no reversal
    assert rel(xp, torch.cat([a5 @ P[f"{s}/weights"][:512] for s in (FW, BW)], -1)) < TOL
    rec = S.recurrence_stage(xp, wh[0], wh[1], tsl, T, rnd=S.ident, biases=biases)
    assert rel(rec["out"], _pad_rows(A["lstm_out"].detach(), H2)) < TOL
    # the bf16-layout chain gives the same gates and cell states step for step
    ref = _forward_chain(c)["rec"]
    assert rel(rec["gates"], ref["gates"]) < TOL and rel(rec["c"], ref["c"]) < TOL
    assert rel(S.logits_stage(_zero_pair(rec["out"]), Wp["logits/weights"], P["logits/biases"], T)["out"], c["logits"]) < TOL
    # teacher-forced steps with the cell state carried in fp64 reproduce every active step's h and c
    iso = S.recurrence_steps_isolated(xp, wh[0], wh[1], _zero_pair(rec["out"]), None, tsl, T, biases=biases)
    act = torch.arange(T)[None, :] < torch.as_tensor(S.clamp_lens(tsl, T))[:, None]
    assert rel(iso["c"][:, act], rec["c"][:, act]) < TOL
    L = S.clamp_lens(tsl, T)
    for d in range(2):
        for n in range(c["N"]):
            for s in range(L[n]):
                t = (L[n] - 1 - s) if d else s
                assert rel(iso["h"][d, n, s], rec["out"][n, t, d * 256:(d + 1) * 256]) < TOL


def test_split_product_leaves_out_only_lo_times_lo():
    """A pair against a pair is ah*wh + al*wh + ah*wl = (ah+al)(wh+wl) - al*wl, for convolutions and matmuls alike."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 6, 4, 64, generator=g, dtype=torch.float64)
    w = torch.randn(3, 3, 64, 32, generator=g, dtype=torch.float64) * 0.1
    xs, ws = S.split(x), S.split(w)
    got = S.conv_bias_stage(xs, ws, None)["out"]
    want = S._conv(xs[0] + xs[1], ws[0] + ws[1]) - S._conv(xs[1], ws[1])
    assert rel(got, want) < 1e-12
    a = torch.randn(40, 512, generator=g, dtype=torch.float64)
    b = torch.randn(512, 96, generator=g, dtype=torch.float64)
    (ah, al), (bh, bl) = S.split(a), S.split(b)
    y, acc = S.bilinear(torch.matmul, (ah, al), (bh, bl))
    assert rel(y, (ah + al) @ (bh + bl) - al @ bl) < 1e-12
    assert rel(y, ah @ bh + al @ bh + ah @ bl) < 1e-12
    assert rel(acc, (ah.abs() + al.abs()) @ (bh.abs() + bl.abs())) < 1e-12


def test_dropped_term_size():
    """|lo| <= 2^-8 |x| (half a bf16 ulp), so one dropped al*wl is at most 2^-16 of |a||w| and about 2^-19 on average;
    summed over a K = 512 contraction with mixed signs it stays below 2^-18 of sum |a||w|."""
    g = torch.Generator().manual_seed(5)
    a = torch.randn(512, 512, generator=g, dtype=torch.float64).float().double()
    w = torch.randn(512, 256, generator=g, dtype=torch.float64).float().double()
    (ah, al), (wh, wl) = S.split(a), S.split(w)
    assert float((al.abs() / a.abs()).max()) <= 2.0 ** -8
    per = (al[:256, :256] * wl[:256]).abs() / (a[:256, :256] * w[:256]).abs()       # 65536 single products
    assert float(per.max()) <= 2.0 ** -16 and float(per.mean()) <= 2.0 ** -18
    assert float(((al @ wl).abs() / (a.abs() @ w.abs())).max()) <= 2.0 ** -18


def _bits(x):
    return [int(v) & 0xFFFFFFFF for v in torch.as_tensor(x, dtype=torch.float64).float().view(torch.int32)]


def test_split_bit_patterns():
    """hi = bf16 RNE(x), lo = bf16 RNE(x - hi): ties to even in both halves, signs, powers of two, exact bf16 values."""
    cases = [
        (1.0, 0x3F800000, 0x00000000),                                 # power of two: lo = 0
        (-0.375, 0xBEC00000, 0x00000000),                              # negative, exactly a bf16 value
        (1 + 2 ** -8, 0x3F800000, 0x3B800000),                         # tie, even hi below: lo = +2^-8
        (1 + 3 * 2 ** -8, 0x3F820000, 0xBB800000),                     # tie, even hi above: lo = -2^-8
        (-(1 + 2 ** -8), 0xBF800000, 0xBB800000),                      # negative tie
        (1 + 2 ** -9 + 2 ** -20, 0x3F800000, 0x3B000000),              # lo rounds away the 2^-20 bit
        (2.0 ** -30 * (1 + 2 ** -7 + 2 ** -12), 0x30810000, 0x2A800000),   # small exponents: lo = 2^-42
    ]
    for x, hi, lo in cases:
        h, l = S.split(torch.tensor([x], dtype=torch.float64))
        assert _bits(h) == [hi] and _bits(l) == [lo], (x, hex(_bits(h)[0]), hex(_bits(l)[0]))
        assert float(h + l) == float(np.float32(x)) or abs(float(h + l) - x) <= 2.0 ** -16 * abs(x)


def test_tf32_rna_bit_patterns():
    """Round to nearest with ties AWAY from zero on the 13 dropped mantissa bits (cvt.rna.tf32.f32)."""
    cases = [
        (1.0, 0x3F800000),
        (1 + 2 ** -11, 0x3F802000),                                     # tie -> away: 1 + 2^-10
        (1 + 3 * 2 ** -11, 0x3F804000),                                # tie -> away (not to even): 1 + 2^-9
        (-(1 + 2 ** -11), 0xBF802000),                                 # negative tie -> away from zero
        (1 + 2 ** -11 - 2 ** -23, 0x3F800000),                         # just below the tie -> down
        (2.0 - 2 ** -23, 0x40000000),                                  # carries into the exponent
        (-(2.0 ** -20), 0xB5800000),                                   # power of two, negative: unchanged
        (0.0, 0x00000000),
    ]
    for x, want in cases:
        got = _bits(S.tf32_rna(torch.tensor([x], dtype=torch.float64)))[0]
        assert got == want, (x, hex(got), hex(want))
        assert got & 0x1FFF == 0


def _truncate_tf32(x):
    """What a producer without cvt.rna would store: the low 13 mantissa bits cleared (round toward zero)."""
    return (x.float().contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32).double()


def _truncate_bf16(x):
    return (x.float().contiguous().view(torch.int32) & ~0xFFFF).view(torch.float32).double()


@pytest.mark.parametrize("mode", ["f32", "tf32"])
def test_x3_storage_checks_reject_a_truncating_store(mode):
    """The checks the f32-class stage isolation applies to a stored activation hold a round-to-nearest store of an f32 dot
    product (K = 2304, like conv3_2) and reject the same store with truncation in place of rounding.  tf32: the value
    bound (half a tf32 ulp + c * acc) fails, while the low 13 bits are zero either way.  Split: a truncated hi leaves a lo
    that still carries the value, so the value bound (a quarter of the lo-half ulp + c * acc) passes and the canonical-form
    check fails.  A split store that truncated only lo would err by less than 2^-16 of the value, below the stage's f32
    accumulation error c * acc, so no per-element check resolves it."""
    import test_gpu_x3_stage_isolation as X3           # the enforced checks; importing the module needs no GPU
    from stage_check import Checker
    g = torch.Generator().manual_seed(9)
    a = torch.randn(192, 2304, generator=g, dtype=torch.float64)
    w = torch.randn(2304, 128, generator=g, dtype=torch.float64) * 0.05
    ref, acc = a @ w, a.abs() @ w.abs()
    v = ref.float()                                     # an f32 accumulator off by at most 2^-24 |ref|
    if mode == "tf32":
        stores = {"rna": S.tf32_rna(v).float(), "truncated": _truncate_tf32(v).float()}
        value = {k: x.double() for k, x in stores.items()}
    else:
        hi_t = _truncate_bf16(v).float()
        stores = {"rna": torch.stack([t.to(torch.bfloat16) for t in S.split(v)], -2),
                  "truncated hi": torch.stack([hi_t.to(torch.bfloat16), (v - hi_t).to(torch.bfloat16)], -2)}
        value = {k: x[..., 0, :].double() + x[..., 1, :].double() for k, x in stores.items()}
    for name, raw in stores.items():
        ck = Checker(name, X3.BOUNDS[mode], ulp=X3.STORAGE_ULP[mode])
        ck.close("conv3_2", value[name], ref, acc)
        X3._canonical(ck, mode, "conv3_2", raw)
        if name == "rna":
            assert not ck.fail, ck.fail
        else:
            assert ck.fail, (name, ck.rows)
            assert ck.fail[0].startswith("conv3_2: " if mode == "tf32" else "conv3_2_canonical"), ck.fail


# ---------------------------------------------------------------------------------------------------------- batch scale
def test_vectorised_layout_helpers_equal_their_loops():
    """reverse_rows, step_h, gate_perm and first_argmax (device-agnostic, no per-row loops) equal plain loops."""
    g = torch.Generator().manual_seed(1)
    N, H2, T = 6, 9, 8
    lens = [8, 0, 1, 5, 12, 3]                        # 12 > T: clamped
    L = S.clamp_lens(lens, T)
    x = torch.randn(N, H2, 7, generator=g, dtype=torch.float64)
    want = x.clone()
    for n in range(N):
        if L[n] > 0:
            want[n, :L[n]] = x[n, :L[n]].flip(0)
    assert torch.equal(S.reverse_rows(x, lens, T), want)
    out = torch.randn(N, H2, 512, generator=g, dtype=torch.float64)
    h = S.step_h(out, lens, T)
    for d in range(2):
        for n in range(N):
            for s in range(L[n]):
                assert torch.equal(h[d, n, s], out[n, (L[n] - 1 - s) if d else s, d * 256:(d + 1) * 256])
    j = np.arange(1024)
    assert np.array_equal(S.gate_perm().numpy(), (j % 256 // 32) * 128 + j // 256 * 32 + j % 32)
    v = torch.randint(0, 3, (50, 4), generator=g).double()
    assert np.array_equal(S.first_argmax(v).numpy(), np.argmax(v.numpy(), -1))


def test_chunked_references_equal_the_whole_batch(chain):
    _check_chunked_references(chain)


def test_chunked_references_at_edge_widths(edge_chain):
    _check_chunked_references(edge_chain)


def _check_chunked_references(c):
    """Per-image stages over image chunks concatenate to the whole-batch result exactly; the batch reductions (BatchNorm
    sums and backward, weight and bias gradients, masked column sums) summed over chunks agree to 1e-12."""
    r = _forward_chain(c)
    P, A, T, H2, tsl, eps = c["P"], c["A"], c["T"], c["H2"], c["tsl"], O.BN_EPS
    cut = max(1, c["N"] - 1)                               # the last image on its own (one chunk when N = 1)
    parts = [slice(0, cut)] + ([slice(cut, c["N"])] if cut < c["N"] else [])
    cat = lambda f: {k: torch.cat([f(s)[k] for s in parts]) for k in f(parts[0]) if torch.is_tensor(f(parts[0])[k])}
    for k, v in cat(lambda s: S.conv_relu_pool22_stage(A["conv1"][s], P["conv2/weights"], P["conv2/biases"])).items():
        assert torch.equal(v, S.conv_relu_pool22_stage(A["conv1"], P["conv2/weights"], P["conv2/biases"])[k]), k
    xp = r["xproj"]["out"]
    rec = [S.recurrence_stage(xp[s], P[f"{FW}/weights"][512:], P[f"{BW}/weights"][512:], tsl[s], T) for s in parts]
    whole = S.recurrence_stage(xp, P[f"{FW}/weights"][512:], P[f"{BW}/weights"][512:], tsl, T)
    assert torch.equal(torch.cat([x["out"] for x in rec]), whole["out"])
    assert torch.equal(torch.cat([x["gates"] for x in rec], 1), whole["gates"])
    pre, bn = r["conv4_2"]["pre"], r["conv4_2"]["bn"]
    tot = {}
    for s in parts:
        for k, v in S.bn_sums(pre[s]).items():
            tot[k] = tot[k] + v if k in tot else v
    st = S.bn_stats_stage(None, P["conv4_2/conv4_2/gamma"], P["conv4_2/conv4_2/beta"], eps, parts=tot)
    st1 = S.bn_stats_stage(pre, P["conv4_2/conv4_2/gamma"], P["conv4_2/conv4_2/beta"], eps)
    for k in ("sum", "sumsq", "mean", "invstd", "scale", "shift"):
        assert rel(st[k], st1[k]) < 1e-12, k
    d = torch.randn(pre.shape[:2] + (2, pre.shape[3]), dtype=torch.float64)
    gamma = P["conv4_2/conv4_2/gamma"]
    stats = S.bn_batch(None, eps, parts=tot)
    sums = {}
    for s in parts:
        dyr = S.bn_relu_pool_route(d[s], pre[s], bn, rnd=S.ident)
        for k, v in S.bn_bwd_sums(dyr, dyr.abs(), pre[s], stats).items():
            sums[k] = sums[k] + v if k in sums else v
    whole = S.bn_relu_pool_bwd_stage(d, pre, bn, gamma, eps, rnd=S.ident)
    got = [S.bn_relu_pool_bwd_stage(d[s], pre[s], bn, gamma, eps, rnd=S.ident, stats=stats, sums=sums) for s in parts]
    assert rel(torch.cat([x["dx"] for x in got]), whole["dx"]) < 1e-12
    assert rel(torch.cat([x["dx_acc"] for x in got]), whole["dx_acc"]) < 1e-12
    for k in ("dgamma", "dbeta", "dgamma_acc", "dbeta_acc"):
        assert rel(got[0][k], whole[k]) < 1e-12, k
    dy = torch.randn(A["conv3_1"].shape, dtype=torch.float64)
    w = S.conv_bwd(dy, A["conv3_1"], P["conv3_2/weights"])
    ws = [S.conv_bwd(dy[s], A["conv3_1"][s], P["conv3_2/weights"]) for s in parts]
    assert torch.equal(torch.cat([x["dx"] for x in ws]), w["dx"])
    for k in ("dw", "dw_acc", "db", "db_acc"):
        assert rel(sum(x[k] for x in ws), w[k]) < 1e-12, k
    cs = [S.masked_colsum(dy[s], A["conv3_1"][s]) for s in parts]
    assert rel(sum(x[0] for x in cs), S.masked_colsum(dy, A["conv3_1"])[0]) < 1e-12


@pytest.fixture(scope="module")
def chain4():
    return _make_chain(4, 24, [24, 17, 4, 12])


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_references_with_injected_sums_equal_the_whole_batch(chain4, world):
    """The data-parallel rule the GPU stage checks use (test_gpu_stage_isolation._global_parts / _global_bwd_sums): each of
    `world` equal shards, its own BatchNorm sums plus the other shards' f64 sums injected, gives the whole batch's
    statistics and data gradients, and its gamma / beta gradients from its OWN sums add up over the shards to the whole
    batch's, all to 1e-12.  Taking gamma / beta from the global sums instead counts them `world` times."""
    import test_gpu_stage_isolation as B
    c = chain4
    r = _forward_chain(c)
    P, eps, N = c["P"], O.BN_EPS, c["N"]
    n = N // world
    shards = [slice(k * n, (k + 1) * n) for k in range(world)]
    others = lambda vs, k: sum(v for q, v in enumerate(vs) if q != k)
    gen = torch.Generator().manual_seed(3)
    w42 = P["conv4_2/weights"]
    for name in ("conv4_2", "conv4_1"):
        pre, bn = r[name]["pre"], r[name]["bn"]
        gamma, beta = P[f"{name}/{name}/gamma"], P[f"{name}/{name}/beta"]
        local = [S.bn_sums(pre[s]) for s in shards]
        fwd = [torch.cat([p["sum"], p["sumsq"]]) for p in local]
        whole_st = S.bn_stats_stage(pre, gamma, beta, eps)
        parts = [B._global_parts(local[k], others(fwd, k), world) for k in range(world)]
        for p in parts:
            st = S.bn_stats_stage(None, gamma, beta, eps, parts=p)
            for k in ("sum", "sumsq", "mean", "invstd", "scale", "shift"):
                assert rel(st[k], whole_st[k]) < 1e-12, (name, k)
        stats = S.bn_batch(pre, eps)
        if name == "conv4_2":
            d = torch.randn(pre.shape[:2] + (2, pre.shape[3]), dtype=torch.float64, generator=gen)
            stage = lambda s, **kw: S.bn_relu_pool_bwd_stage(d[s], pre[s], bn, gamma, eps, rnd=S.ident, **kw)
            dys = [S.bn_relu_pool_route(d[s], pre[s], bn, rnd=S.ident) for s in shards]
            dys = [(x, x.abs()) for x in dys]
        else:
            d = torch.randn(pre.shape, dtype=torch.float64, generator=gen)
            stage = lambda s, **kw: S.conv_bn_relu_bwd_stage(d[s], pre[s], bn, gamma, w42, eps, rnd=S.ident, **kw)
            dys = [S.conv_relu_dgrad(d[s], pre[s], bn, w42, rnd=S.ident) for s in shards]
        whole = stage(slice(None))
        st_k = [S.bn_batch(None, eps, parts=p) for p in parts]
        for k in range(world):
            assert rel(st_k[k]["mean"], stats["mean"]) < 1e-12 and rel(st_k[k]["invstd"], stats["invstd"]) < 1e-12
        ls = [S.bn_bwd_sums(dys[k][0], dys[k][1], pre[shards[k]], st_k[k]) for k in range(world)]
        bwd = [torch.cat([x["dbeta"], x["dgamma"]]) for x in ls]
        got = [stage(shards[k], stats=st_k[k], sums=B._global_bwd_sums(ls[k], others(bwd, k))) for k in range(world)]
        assert rel(torch.cat([x["dx"] for x in got]), whole["dx"]) < 1e-12, name
        for k in ("dgamma", "dbeta"):
            assert rel(sum(x[k] for x in ls), whole[k]) < 1e-12, (name, k)
            # the global sums in every shard's gamma / beta gradient: `world` times the whole batch's after the SUM
            assert rel(sum(x[k] for x in got), whole[k]) > 0.5, (name, k)
            assert rel(sum(x[k] for x in got), world * whole[k]) < 1e-12, (name, k)


def test_checker_rows_from_torch_equal_numpy():
    """Checker.close / close_scaled / exact give the same row from torch tensors as from numpy arrays, and a stage checked
    in image chunks merges into one row with the worst element, the maxima and the L2 of the whole."""
    from stage_check import Checker, ulp_bf16
    g = torch.Generator().manual_seed(2)
    ref = torch.randn(40, 33, generator=g, dtype=torch.float64) * 10 ** torch.randint(-3, 3, (40, 33), generator=g)
    gpu = S.bf16(ref * (1 + 2.0 ** -10 * torch.randn(40, 33, generator=g, dtype=torch.float64)))
    acc = ref.abs() + 0.1
    mask = torch.rand(40, 33, generator=g) > 0.3
    bounds = {"a": (1, 2 ** -12), "b": (0, 1e-3), "c": (1, 1e-3)}
    cks = {}
    for kind, cv in (("np", lambda t: t.numpy()), ("torch", lambda t: t)):
        ck = cks[kind] = Checker("x", bounds, ulp=ulp_bf16)
        ck.close("a", cv(gpu), cv(ref), cv(acc))
        ck.close("b", cv(gpu), cv(ref), cv(acc), mask=cv(mask))
        ck.close_scaled("c", cv(gpu), cv(ref), mask=cv(mask))
        ck.exact("e", cv(gpu), cv(ref))
    for a, b in zip(cks["np"].rows, cks["torch"].rows):          # the L2 norms may differ in the last bits
        for k in ("rel_l2", "_err_sq", "_ref_sq"):
            if k in a:
                va, vb = a.pop(k), b.pop(k)
                assert abs(va - vb) <= 1e-12 * abs(va), k
        assert a == b
    whole = Checker("x", bounds, ulp=ulp_bf16)
    whole.close("b", gpu, ref, acc)
    parts = Checker("x", bounds, ulp=ulp_bf16)
    for s in (slice(0, 7), slice(7, 40)):
        parts.close("b", gpu[s], ref[s], acc[s])
    (w,), (p,) = whole.rows, parts.rows
    for k in ("rel_l2", "_err_sq", "_ref_sq"):
        vp, vw = p.pop(k), w.pop(k)
        assert abs(vp - vw) <= 1e-12 * abs(vw), k
    assert p == w
    # a NaN in any chunk fails the merged row, whichever chunk comes after it
    bad = gpu.clone()
    bad[3, 5] = float("nan")
    for order in ((bad, gpu, gpu), (gpu, bad, gpu), (gpu, gpu, bad)):
        for use_torch in (True, False):
            ck = Checker("x", bounds, ulp=ulp_bf16)
            for g_ in order:
                args = (g_, ref, acc) if use_torch else (g_.numpy(), ref.numpy(), acc.numpy())
                ck.close("a", *args)
                ck.exact("e", *args[:2])
            (ra, re) = ck.rows
            assert np.isnan(ra["max_ratio"]) and np.isnan(ra["c_needed"]) and np.isnan(ra["max_abs_err"])
            assert np.isnan(ra["worst_gpu"]) and re["mismatches"] >= 1
            assert any(f.startswith("a: ") for f in ck.fail)
    # one stage name for two kinds of check is refused
    ck = Checker("x", bounds, ulp=ulp_bf16)
    ck.exact("a", gpu, gpu)
    with pytest.raises(AssertionError, match="different kinds"):
        ck.close("a", gpu, ref, acc)
