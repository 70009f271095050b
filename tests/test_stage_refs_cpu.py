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


@pytest.fixture(scope="module")
def chain():
    torch.manual_seed(0)
    N, W = 3, 24
    p = O.randomize_params(O.init_params(3, dtype=np.float64, logits_scale=3.0), scale=0.3)
    data, lab, ll, tsl = O.synth_batch(N, W, seed=7, widths=[24, 17, 4], min_len=1, max_len=2, dtype=np.float64)
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
    c = chain
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
    c = chain
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
    b42 = S.bn_relu_pool_bwd_stage(d_a4b, r["conv4_2"]["pre"], r["conv4_2"]["bn"], P["conv4_2/conv4_2/gamma"],
                                   P["conv4_2/conv4_2/beta"], eps, rnd=S.ident)
    got["conv4_2/conv4_2/gamma"], got["conv4_2/conv4_2/beta"] = b42["dgamma"], b42["dbeta"]
    got["conv4_2/weights"] = S.conv_bwd(b42["dx"], A["conv4_1"], P["conv4_2/weights"])["dw"]
    bn41 = r["conv4_1"]["bn"]
    b41 = S.conv_bn_relu_bwd_stage(b42["dx"], r["conv4_1"]["pre"], bn41, P["conv4_1/conv4_1/gamma"], P["conv4_1/conv4_1/beta"],
                                   P["conv4_2/weights"], eps, mask=(r["conv4_1"]["pre"] * bn41[0] + bn41[1] > 0).double(), rnd=S.ident)
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
