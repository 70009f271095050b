"""CTC forced alignment (crnn_ctc_align) against the CTC loss with its gradient (crnn_ctc_loss) and the greedy decode
(crnn_ctc_greedy), all on the same logits, at three shapes:
  c3       T = 63, N = 1024: the model's logits of a W = 256 batch and the batch's labels (4 - 6 ids)
  packed   T = 255, N = 64: one packed evaluation batch of 1024-px lines, labels of 30 - 70 ids
  long     T = 2048, N = 300, L = 639: the longest labels the kernels take
Each entry point is called through ctypes with preallocated outputs and workspaces (no Python allocation in the timed loop,
so the host does not bound the small shapes).  Times are CUDA events around `--iters` back-to-back calls after `--warmup`,
the median of `--reps` windows.  Prints one JSON
line with the card's name and power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = [v.strip() for v in out.split(",")]
        return dict(gpu=name, power_limit=power)
    except Exception as e:          # the numbers stay, the card is reported as unknown
        return dict(gpu=f"unknown ({e})", power_limit="unknown")


def timed(fn, iters, warmup, reps):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b) / iters)
    return float(np.median(ms))


def shapes(dev):
    from lstm_ctc_ocr_b200 import engine, synthetic
    out = {}
    m = engine.CrnnModel(weight_decay=1e-5, device=dev)
    m.load_params(synthetic.init_params(3, logits_scale=10.0))
    data, lab, ll, tsl = synthetic.synth_batch(1024, 256, seed=5)
    d_tsl = torch.tensor(tsl, device=dev)
    x = m.forward(torch.tensor(data, device=dev), d_tsl).clone()
    out["c3"] = (x, lab, ll, tsl)
    del m
    rng = np.random.default_rng(1)
    for name, T, N, lo, hi in (("packed", 255, 64, 30, 71), ("long", 2048, 300, 639, 640)):
        ll = rng.integers(lo, hi, size=N).astype(np.int32)
        lab = rng.integers(1, 63, size=int(ll.sum())).astype(np.int32)
        x = torch.tensor(rng.normal(0, 3.0, size=(T, N, 64)).astype(np.float32), device=dev)
        out[name] = (x, lab, ll, np.full(N, T, np.int32))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("align_bench needs a CUDA device (an H100); nothing is measured without one")
    from lstm_ctc_ocr_b200 import _lib, engine
    lib = _lib.load()
    dev = torch.device("cuda:0")
    res = dict(gpu_info(), iters=a.iters, reps=a.reps, shapes={})
    for name, (x, lab, ll, il) in shapes(dev).items():
        T, N, _ = x.shape
        mll = int(ll.max())
        d_lab, d_ll, d_il = (torch.tensor(v, device=dev) for v in (lab, ll, il))
        ctc_ws = engine._auto_ctc_workspace(T, N, 64, mll, dev)
        ctc_ws_ptr, ctc_ws_bytes = (0, 0) if ctc_ws is None else (ctc_ws.data_ptr(), ctc_ws.numel())
        al_ws = torch.empty(engine.ctc_align_workspace_bytes(T, N, 64, mll), dtype=torch.uint8, device=dev)
        grad = torch.empty_like(x)
        costs, lp = torch.empty(N, device=dev), torch.empty(N, device=dev)
        start, end = torch.empty_like(d_lab), torch.empty_like(d_lab)
        peak = torch.empty(d_lab.shape, device=dev)
        out, out_len = torch.empty((N, T), dtype=torch.int32, device=dev), torch.empty(N, dtype=torch.int32, device=dev)
        st = torch.cuda.current_stream().cuda_stream
        xp, lab_p, ll_p, il_p = x.data_ptr(), d_lab.data_ptr(), d_ll.data_ptr(), d_il.data_ptr()
        row = dict(T=T, N=N, max_label_len=mll)
        row["align_ms"] = timed(lambda: _lib.check(lib.crnn_ctc_align(xp, lab_p, 0, ll_p, il_p, T, N, 64, 0, mll, start.data_ptr(),
                                                                      end.data_ptr(), peak.data_ptr(), lp.data_ptr(), al_ws.data_ptr(),
                                                                      al_ws.numel(), st)), a.iters, a.warmup, a.reps)
        row["ctc_loss_grad_ms"] = timed(lambda: _lib.check(lib.crnn_ctc_loss(xp, grad.data_ptr(), lab_p, ll_p, il_p, T, N, 64, 0, mll,
                                                                             1.0, costs.data_ptr(), ctc_ws_ptr, ctc_ws_bytes, st)),
                                        a.iters, a.warmup, a.reps)
        row["greedy_ms"] = timed(lambda: _lib.check(lib.crnn_ctc_greedy(xp, il_p, T, N, 64, engine.TF_BLANK, 0, out.data_ptr(),
                                                                        out_len.data_ptr(), st)), a.iters, a.warmup, a.reps)
        row["align_over_loss"] = round(row["align_ms"] / row["ctc_loss_grad_ms"], 3)
        res["shapes"][name] = row
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
