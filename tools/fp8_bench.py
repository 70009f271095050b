"""Forward + CTC loss at C3 (batch 1024 x 32x256) on the bf16 path and the fp8 path (compute_dtype 4), alternating in one call.

Prints one JSON line per round and precision (images/s over `--steps` timed steps after `--warmup`), then one summary line:
the per-stage times of crnn_profile_* for both precisions, each fp8 GEMM's TFLOP/s against the 1979 TFLOP/s dense FP8 data-sheet
figure, the card's name, power limit and max SM clock (read in the same call), and the max |fp8 - bf16| logit difference on
the same seeded input.  Needs the GPU.

    python tools/fp8_bench.py [--steps 20] [--warmup 5] [--rounds 3]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# FLOPs of the five e4m3 GEMMs at batch N, width W: (profile stage, output positions, Cout, K)
def fp8_gemm_flops(N, W):
    H2 = W // 4
    return {"conv3_1": 2.0 * N * H2 * 8 * 256 * 1152, "conv3_2_pool": 2.0 * N * H2 * 8 * 256 * 2304,
            "conv4_1_gemm": 2.0 * N * H2 * 4 * 512 * 2304, "conv4_2_gemm": 2.0 * N * H2 * 4 * 512 * 4608,
            "conv5": 2.0 * N * H2 * 512 * 2048}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001 -- the numbers are still worth printing without the card's settings
        return dict(gpu=torch.cuda.get_device_name(0), card_query_error=str(e))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--width", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_bench needs a CUDA device")
    from lstm_ctc_ocr_b200 import _lib, engine, synthetic
    N, W = args.batch, args.width
    dev = torch.device("cuda:0")
    params = synthetic.init_params(3)
    data, lab, ll, tsl = synthetic.synth_batch(N, W, seed=3)
    t = lambda a: torch.tensor(a, device=dev)  # noqa: E731
    d, tl, dlab, dll = t(data), t(tsl), t(lab), t(ll)
    models = {}
    for prec in ("bf16", "fp8"):
        m = engine.CrnnModel(device=dev, compute_dtype=prec)
        m.load_params(params)
        models[prec] = m
    models["fp8"].calibrate_fp8(d, tl)
    mll = int(ll.max())
    out = {p: torch.empty((W // 4 - 1, N, 64), dtype=torch.float32, device=dev) for p in models}

    def step(p):
        logits = models[p].forward(d, tl, out=out[p])
        engine.ctc_loss(logits, dlab, dll, tl, max_label_len=mll)

    for p in models:
        for _ in range(args.warmup):
            step(p)
    torch.cuda.synchronize()
    rate = {p: [] for p in models}
    for r in range(args.rounds):
        for p in models:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step(p)
            e1.record()
            e1.synchronize()
            ms = e0.elapsed_time(e1) / args.steps
            rate[p].append(N / (ms / 1e3))
            print(json.dumps(dict(round=r, precision=p, ms_per_step=round(ms, 4), images_per_s=round(N / (ms / 1e3), 1))), flush=True)

    # per-stage times of the forward (CUDA events between stages), a separate pass
    lib = _lib.load()
    names = [lib.crnn_profile_stage_name(i).decode() for i in range(lib.crnn_profile_num_stages())]
    stages = {}
    for p, m in models.items():
        _lib.check(lib.crnn_profile_begin(m.handle, args.steps))
        for _ in range(args.steps):
            step(p)
        buf = np.zeros((args.steps, len(names)), np.float32)
        nf = _lib.c_int()
        _lib.check(lib.crnn_profile_read(m.handle, buf.ctypes.data, nf))
        stages[p] = {n: round(float(v), 4) for n, v in zip(names, buf[:nf.value].mean(0))}
    flops = fp8_gemm_flops(N, W)
    tflops = {k: round(flops[k] / (stages["fp8"][k] * 1e-3) / 1e12, 1) for k in flops}
    tflops_bf16 = {k: round(flops[k] / (stages["bf16"][k] * 1e-3) / 1e12, 1) for k in flops}
    lb = models["bf16"].forward(d, tl)
    l8 = models["fp8"].forward(d, tl)
    torch.cuda.synchronize()
    summary = dict(config=f"C3 forward + CTC loss, batch {N} x 32x{W}", steps=args.steps, rounds=args.rounds,
                   images_per_s={p: [round(v, 1) for v in rate[p]] for p in rate},
                   speedup_median=round(float(np.median(rate["fp8"]) / np.median(rate["bf16"])), 3),
                   stage_ms=stages, fp8_gemm_tflops=tflops, bf16_same_gemms_tflops=tflops_bf16, fp8_peak_tflops=1979,
                   fp8_scales=[float(s) for s in models["fp8"].fp8_scales()],
                   max_abs_logit_diff_fp8_vs_bf16=float((l8 - lb).abs().max()), max_abs_logit_bf16=float(lb.abs().max()))
    summary.update(card())
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
