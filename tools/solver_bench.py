"""Optimizer step alone: CrnnModel.apply_gradients for Adam, Momentum and RMSProp on the full 7 158 592-parameter training model,
CUDA-event time per call, the solvers alternating in blocks within one process.  Each call is two grid-stride passes over the flat
f32 buffers: the gradient finish (L2 term on the regularised tensors + global sum of squares) and the clip + update.

Bytes one call must move, from the shapes (4 bytes per element, n = 7 158 592, r = elements under the L2 term):
  finish pass       read grads (n), read params + write grads on the regularised tensors (2 r)
  Adam update       read g, p, m, v; write p, m, v        7 n
  Momentum update   read g, p, accum; write p, accum       5 n
  RMSProp update    read g, p, ms, mom; write p, ms, mom   7 n
Prints one JSON line per solver with the median time per call, the achieved bandwidth and its share of the H100 SXM data sheet's
3.35 TB/s, plus the GPU's name and power limit read in the same run.  Usage: python tools/solver_bench.py [calls_per_solver]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lstm_ctc_ocr_b200 import engine, synthetic  # noqa: E402

PEAK_BPS = 3.35e12
SOLVERS = ("Adam", "Momentum", "RMS")
UPDATE_STREAMS = {"Adam": 7, "Momentum": 5, "RMS": 7}
L2_TENSORS = [f"{c}/weights" for c in ("conv1", "conv2", "conv3_1", "conv3_2", "conv4_1", "conv4_2", "conv5")] + ["logits/weights"]


def gpu_info():
    idx = torch.cuda.current_device()
    info = {"gpu": torch.cuda.get_device_name(idx)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", str(idx)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in out.split(",")]
    except Exception as e:          # the query is informational: report what failed rather than guess
        info["power_limit"] = f"unavailable ({type(e).__name__})"
    return info


def main(calls=240, block=20, warmup=30):
    m = engine.CrnnModel(weight_decay=1e-5)
    m.load_params(synthetic.init_params(3))
    m.set_training(True)
    n = m.total
    reg = sum(int(np.prod(m.table[k][1])) for k in L2_TENSORS if k in m.table)
    assert len([k for k in L2_TENSORS if k in m.table]) == len(L2_TENSORS)
    finish_bytes = 4 * (n + 2 * reg)
    gen = torch.Generator(device=m.device).manual_seed(0)
    grads0 = torch.randn(n, device=m.device, generator=gen)
    times = {s: [] for s in SOLVERS}
    states = {}
    for s in SOLVERS:                                   # one slot state per solver, kept across its blocks
        m.set_solver(s, momentum=0.9)
        states[s] = (m.adam_m.clone(), m.adam_v.clone())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    step = {s: 0 for s in SOLVERS}

    def run(s, k):
        for _ in range(k):
            step[s] += 1
            m.apply_gradients(1e-4, step[s], clip=10.0)
    rounds = (calls + block - 1) // block
    for r in range(-1, rounds):
        for s in SOLVERS:
            m.solver = s
            m.adam_m.copy_(states[s][0]); m.adam_v.copy_(states[s][1])
            m.grads.copy_(grads0)
            torch.cuda.synchronize()
            if r < 0:
                run(s, warmup)
            else:
                e0.record()
                run(s, block)
                e1.record()
                torch.cuda.synchronize()
                times[s].append(e0.elapsed_time(e1) * 1e3 / block)
            states[s][0].copy_(m.adam_m); states[s][1].copy_(m.adam_v)
    info = gpu_info()
    adam_us = float(np.median(times["Adam"]))
    for s in SOLVERS:
        us = float(np.median(times[s]))
        nbytes = finish_bytes + UPDATE_STREAMS[s] * 4 * n
        print(json.dumps({"solver": s, "calls": len(times[s]) * block, "us_median": round(us, 2), "us_min": round(min(times[s]), 2),
                          "us_max": round(max(times[s]), 2), "bytes": nbytes, "finish_bytes": finish_bytes,
                          "update_bytes": UPDATE_STREAMS[s] * 4 * n, "GBps": round(nbytes / us / 1e3, 1),
                          "frac_of_3.35TBps": round(nbytes / us / 1e-6 / PEAK_BPS, 3), "vs_adam": round(us / adam_us, 3), **info}))


if __name__ == "__main__":
    main(calls=int(sys.argv[1]) if len(sys.argv) > 1 else 240)
