"""f32-class paths (crnn_config.compute_dtype = 2 "f32" and 3 "tf32", csrc/forward_x3.cu) against the fp64 oracle -- BASELINE
configs[1]: "1xH100 fp32 CRNN fwd + CTC loss, batch 256, 32x160".  Need the GPU.

Operands are split into bf16 hi + bf16 lo and multiplied as hi*hi + lo*hi + hi*lo on the wgmma pipe with f32 accumulation
(~2^-16 per operand), everything else is f32; stated tolerances (max-abs error relative to max|reference|):
    conv / LSTM taps 2e-4, logits 3e-4, |loss - oracle| / oracle 2e-4 (SURVEY 7.2(6) asks for <= 2e-3 of the fp32 config),
    greedy decode == oracle decode on >= 99.5 % of lines WITHOUT any margin filter.
"tf32": the same orchestration on tf32 wgmma operands (2^-11 per operand, rounded to nearest where produced); stated
tolerances: taps 4e-3, logits 2.5e-3, loss 5e-4 (SURVEY 7.2(6) asks for 2e-3), decode of the SOFT random-weight lines
>= 97 % unfiltered (the trained 10k-line fixture: tests/test_gpu_decode10k.py).  Each run appends its measured errors to
build/parity_report.jsonl.  These whole-chain bounds pin the composition; every single stage of both modes is checked per
element on its own operands in tests/test_gpu_x3_stage_isolation.py."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
TOL = {"f32": dict(tap=2e-4, logit=3e-4, loss=2e-4, decode=0.995),
       "tf32": dict(tap=4e-3, logit=2.5e-3, loss=5e-4, decode=0.97)}
MODES = ["f32", "tf32"]


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def report(test, **kv):
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    with open(os.path.join(ROOT, "build", "parity_report.jsonl"), "a") as f:
        f.write(json.dumps(dict(test=test, **kv)) + "\n")


@pytest.mark.parametrize("N,W,widths", [
    pytest.param(3, 100, None, id="c1_width"),
    pytest.param(2, 160, [160, 131], id="c2_width"),
    pytest.param(2, 256, [256, 201], id="c3_width"),
    pytest.param(5, 24, [24, 20, 9, 24, 16], id="W24_ragged"),
    pytest.param(4, 64, [64, 61, 30, 64], id="W64"),
    pytest.param(130, 40, None, id="N130_W40"),
])
@pytest.mark.parametrize("mode", MODES)
def test_f32_path_layers_vs_oracle(N, W, widths, mode, request):
    from lstm_ctc_ocr_b200 import engine
    from oracle import crnn_oracle as O
    pn = O.randomize_params(O.init_params(3, dtype=np.float32, logits_scale=10.0))
    data, lab, ll, tsl = O.synth_batch(N, W, seed=5, widths=widths, min_len=1, max_len=3)
    m = engine.CrnnModel(device=DEV, compute_dtype=mode)
    m.load_params(pn)
    t = lambda a: torch.tensor(a, device=DEV)
    logits = m.forward(t(data), t(tsl))
    lo, acts = O.forward(O.to_torch(pn), data, tsl, return_all=True)
    T = W // 4 - 1
    errs = {}
    for name in ("conv1", "conv2", "conv3_1", "conv3_2", "conv4_1", "conv4_2"):
        errs[name] = rel(m.tap(name, N, W).cpu(), acts[name].permute(0, 2, 3, 1).numpy())
    errs["conv5"] = rel(m.tap("conv5", N, W).cpu().numpy()[:, :T], acts["reshaped_layer"].numpy())
    errs["lstm_out"] = rel(m.tap("lstm_out", N, W).cpu().numpy()[:, :T], acts["lstm_out"].numpy())
    errs["logits"] = rel(logits.cpu(), lo.numpy())
    costs, _ = engine.ctc_loss(logits, t(lab), t(ll), t(tsl))
    co, _ = O.ctc_loss_np(lo.numpy(), lab, ll, tsl)
    loss_o = co.mean() + float(O.l2_reg(O.to_torch(pn), 1e-5))
    loss = float(m.total_loss(costs).item())
    report("forward_%s_path" % mode, case=request.node.callspec.id, N=N, W=W, loss_rel=abs(loss - loss_o) / loss_o,
           **{k: round(v, 8) for k, v in errs.items()})
    for k, e in errs.items():
        assert e < (TOL[mode]["logit"] if k == "logits" else TOL[mode]["tap"]), (k, e)
    assert abs(loss - loss_o) / loss_o < TOL[mode]["loss"]
    # frames past each sample's length: zero LSTM output, logits == projection bias exactly
    b = pn["logits/biases"]
    for n in range(N):
        if int(tsl[n]) < T:
            assert np.array_equal(logits[int(tsl[n]):, n].cpu().numpy(), np.broadcast_to(b, (T - int(tsl[n]), 64)))


@pytest.mark.parametrize("mode", MODES)
def test_f32_path_at_the_c2_configuration(mode):
    """BASELINE configs[1] as written: batch 256, 32x160, reference initialisers; logits and total loss vs the fp64 oracle."""
    from lstm_ctc_ocr_b200 import engine, synthetic
    from oracle import crnn_oracle as O
    N, W = 256, 160
    params = synthetic.init_params(3)
    data, lab, ll, tsl = synthetic.synth_batch(N, W, seed=3)
    m = engine.CrnnModel(weight_decay=1e-5, device=DEV, compute_dtype=mode)
    m.load_params(params)
    t = lambda a: torch.tensor(a, device=DEV)
    logits = m.forward(t(data), t(tsl))
    costs, grad = engine.ctc_loss(logits, t(lab), t(ll), t(tsl), want_grad=True, grad_scale=1.0 / N, max_label_len=int(ll.max()))
    loss = float(m.total_loss(costs).item())
    p64 = O.to_torch({k: v.astype(np.float64) for k, v in params.items()})
    lo = O.forward(p64, data.astype(np.float64), tsl).numpy()
    co, go = O.ctc_loss_np(lo, lab, ll, tsl)
    loss_o = float(co.mean() + float(O.l2_reg(p64, 1e-5)))
    e_logit = rel(logits.cpu(), lo)
    report("c2_%s_path" % mode, N=N, W=W, logits_rel=e_logit, loss=loss, loss_oracle=loss_o, loss_rel=abs(loss - loss_o) / loss_o,
           costs_rel_max=float(np.abs(costs.cpu().numpy() - co).max() / np.abs(co).max()),
           ctc_grad_abs_max=float(np.abs(grad.cpu().numpy() * N - go).max()))
    assert e_logit < TOL[mode]["logit"]
    assert abs(loss - loss_o) / loss_o < TOL[mode]["loss"]
    assert np.allclose(costs.cpu().numpy(), co, rtol=5e-4 if mode == "f32" else 5e-3)
    assert np.abs(grad.cpu().numpy() * N - go).max() < (1e-3 if mode == "f32" else 1e-2)


@pytest.mark.parametrize("mode", MODES)
def test_f32_path_decode_equals_oracle_without_margin_filter(mode):
    """Greedy decode through conv + BiLSTM on bucketed batches (W in {80,160,256}) vs the oracle's decode of the same weights:
    sequence equality on >= 99.5 % of ALL lines, no top-2-margin filter (the bf16 path needs one, VERDICT r1 weak #3)."""
    from lstm_ctc_ocr_b200 import engine, synthetic
    from oracle import crnn_oracle as O
    params = synthetic.init_params(3, logits_scale=30.0)
    p32 = O.to_torch({k: v.astype(np.float32) for k, v in params.items()}, torch.float32)
    m = engine.CrnnModel(device=DEV, compute_dtype=mode)
    m.load_params(params)
    total = same = 0
    for k, W in enumerate((80, 160, 256)):
        data, _, _, tsl = synthetic.synth_bucket_batch(96, W, seed=40 + k)
        logits = m.forward(torch.tensor(data, device=DEV), torch.tensor(tsl, device=DEV))
        out, out_len = engine.ctc_greedy(logits, torch.tensor(tsl, device=DEV))
        out, out_len = out.cpu().numpy(), out_len.cpu().numpy()
        ref = O.greedy_decode(O.forward(p32, data, tsl).numpy(), tsl)
        for n in range(len(ref)):
            total += 1
            same += int(out[n, :out_len[n]].tolist() == ref[n])
    report("decode_%s_path" % mode, lines=total, identical=same)
    assert same >= TOL[mode]["decode"] * total, (same, total)


@pytest.mark.parametrize("mode", MODES)
def test_f32_path_is_forward_only(mode):
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200._lib import CrnnError
    m = engine.CrnnModel(device=DEV, compute_dtype=mode)
    with pytest.raises(CrnnError):
        m.set_training(True)
