"""The workspace CTC kernel (long text lines) next to the training step it belongs to.  CUDA-event time per call of
engine.ctc_loss (loss + gradient, workspace "auto") at N in {64, 256, 512}, T in {250, 550, 1024, 2048}, max_label_len in
{70, 255, 639} (every label max_label_len long, or the longest that fits T), and of the bf16 forward + backward step at the
same N and W = 4 (T + 1), so the CTC share of a long-line training step is known.  A step whose workspace does not fit the
card is reported as not measured.  Prints the GPU's name and power limit, then one JSON line per shape.
Usage: python tools/ctc_long_bench.py [--quick]"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from lstm_ctc_ocr_b200 import engine, synthetic  # noqa: E402
from solver_bench import gpu_info  # noqa: E402


def _time(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def ctc_ms(N, T, m, reps):
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(N + T + m)
    L = min(m, (T - 1) // 2)                       # label and repeats fit T
    ll = np.full(N, L, np.int32)
    lab = rng.integers(1, 63, size=N * L).astype(np.int32)
    il = np.full(N, T, np.int32)
    x = torch.randn(T, N, 64, device=dev) * 2
    g = torch.empty_like(x)
    costs = torch.empty(N, device=dev)
    d_lab, d_ll, d_il = (torch.tensor(a, device=dev) for a in (lab, ll, il))

    def call():
        engine.ctc_loss(x, d_lab, d_ll, d_il, want_grad=True, grad_scale=1.0 / N, max_label_len=m, costs=costs, grad=g,
                        workspace="auto")
    ms = _time(call, reps)
    assert bool(torch.isfinite(costs).all())
    return ms, L, engine.ctc_workspace_bytes(T, N, 64, m)


def step_ms(model, N, T, reps):
    W = 4 * (T + 1)
    data = torch.rand(N, W, 32, device=model.device)
    tsl = torch.full((N,), T, dtype=torch.int32, device=model.device)
    dl = torch.randn(T, N, 64, device=model.device) * 1e-3

    def call():
        model.forward(data, tsl)
        model.backward(data, tsl, dl)
    try:
        return _time(call, reps, warmup=2)
    except (RuntimeError, engine.CrnnError) as e:
        return f"not measured ({type(e).__name__}: {str(e).splitlines()[0][:80]})"
    finally:
        model._ws = None
        model._ws_key = None
        torch.cuda.empty_cache()


def main(quick=False):
    print(json.dumps(gpu_info()))
    model = engine.CrnnModel(weight_decay=1e-5)
    model.load_params(synthetic.init_params(3))
    model.set_training(True)
    Ns, Ts, Ms = ((64,), (250, 2048), (70, 639)) if quick else ((64, 256, 512), (250, 550, 1024, 2048), (70, 255, 639))
    for N in Ns:
        for T in Ts:
            step = step_ms(model, N, T, reps=3 if T >= 1024 else 5)
            for m in Ms:
                ms, L, ws = ctc_ms(N, T, m, reps=5 if T >= 1024 else 10)
                row = {"N": N, "T": T, "W": 4 * (T + 1), "max_label_len": m, "label_len": L, "workspace_MB": round(ws / 2 ** 20, 1),
                       "ctc_ms": round(ms, 3)}
                if isinstance(step, float):
                    row.update(fwd_bwd_ms=round(step, 3), ctc_share=round(ms / (ms + step), 3))
                else:
                    row["fwd_bwd_ms"] = step
                print(json.dumps(row), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main(quick="--quick" in sys.argv)
