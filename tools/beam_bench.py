"""Beam-search decoder throughput: lines/s at the benchmark shape (T = 63 frames, 64 classes, beam width 100) on peaked, soft
and flat frames, for the host decoder (crnn_ctc_beam_search, csrc/beam.cpp) on this machine's cores and, with --device, for
the device decoder (crnn_ctc_beam_search_device, csrc/beam.cu; CUDA-event timing after a warm-up, several repeats) and on the
10 240 rendered lines of the decode-equality fixture (logits from the model with the fixture's trained weights).
Usage: python tools/beam_bench.py [N] [threads ...] [--device] [--repeats R]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lstm_ctc_ocr_b200 import engine  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def frames(kind, T, N, rng):
    if kind == "flat":
        return (rng.standard_normal((T, N, 64)) * 0.3).astype(np.float32)
    path = rng.choice(64, size=(T, N), p=np.r_[0.25, np.full(62, 0.65 / 62), 0.10])
    x = rng.standard_normal((T, N, 64)).astype(np.float32)
    x[np.arange(T)[:, None], np.arange(N)[None, :], path] += 10.0 if kind == "peaked" else 4.0
    return x


def _device_ms(x, il, repeats):
    """Median and minimum ms of one device decode call (CUDA events), after one warm-up call."""
    import torch
    engine.ctc_beam_search_device(x, il)
    torch.cuda.synchronize()
    ms = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        engine.ctc_beam_search_device(x, il)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), float(np.min(ms))


def _card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def _decode10k(repeats, nt):
    """Device and host decode of the fixture's 20 batches of logits (bf16 forward, trained weights)."""
    import importlib.util
    import torch
    spec = importlib.util.spec_from_file_location("make_decode10k", os.path.join(ROOT, "tests", "golden", "make_decode10k.py"))
    mk = importlib.util.module_from_spec(spec); spec.loader.exec_module(mk)
    fx = np.load(os.path.join(ROOT, "tests", "golden", "decode10k_oracle.npz"))
    s = mk.sampler()
    m = engine.CrnnModel(weight_decay=1e-5, device="cuda:0")
    m.load_params(mk.load_weights())
    batches = []
    for k in range(len(fx["crc"])):
        imgs, _, _, tsl = s.batch(k)
        d_tsl = torch.tensor(np.asarray(tsl, np.int32), device="cuda:0")
        batches.append((m.forward(torch.tensor(np.stack(imgs), device="cuda:0"), d_tsl).clone(), d_tsl))
    lines = sum(int(t.numel()) for _, t in batches)
    dev_ms = sum(_device_ms(x, t, repeats)[0] for x, t in batches)
    host = [(x.cpu().numpy(), t.cpu().numpy()) for x, t in batches]
    t0 = time.perf_counter()
    for x, t in host:
        engine.ctc_beam_search(x, t, num_threads=nt)
    host_s = time.perf_counter() - t0
    return {"lines": lines, "device_lines_per_s": round(lines / (dev_ms * 1e-3), 1),
            f"host_lines_per_s/{nt}t": round(lines / host_s, 1), "device_ms_total": round(dev_ms, 3)}


def main():
    args = sys.argv[1:]
    device = "--device" in args
    repeats = 5
    if "--repeats" in args:
        repeats = int(args[args.index("--repeats") + 1])
        del args[args.index("--repeats"):args.index("--repeats") + 2]
    args = [a for a in args if not a.startswith("--")]
    N = int(args[0]) if args else 1024
    ncpu = os.cpu_count() or 1
    threads = [int(a) for a in args[1:]] or sorted({1, min(8, ncpu), ncpu})
    T = 63
    rng = np.random.default_rng(0)
    il = np.full(N, T, np.int32)
    res = {"T": T, "C": 64, "beam_width": 100, "lines": N, "host_cpus": ncpu, "lines_per_s": {}}
    if device:
        import torch
        if not torch.cuda.is_available():
            raise SystemExit("--device needs a CUDA device")
        res["card"] = _card()
        res["device_ms_per_call"] = {}
        d_il = torch.tensor(il, device="cuda:0")
    for kind in ("peaked", "soft", "flat"):
        x = frames(kind, T, N, rng)
        engine.ctc_beam_search(x[:, :32], il[:32])                 # warm the allocator
        for nt in threads:
            t0 = time.perf_counter()
            engine.ctc_beam_search(x, il, num_threads=nt)
            res["lines_per_s"][f"{kind}/{nt}t"] = round(N / (time.perf_counter() - t0), 1)
        if device:
            med, best = _device_ms(torch.tensor(x, device="cuda:0"), d_il, repeats)
            res["lines_per_s"][f"{kind}/device"] = round(N / (med * 1e-3), 1)
            res["device_ms_per_call"][kind] = {"median": round(med, 3), "min": round(best, 3)}
    if device:
        res["decode10k"] = _decode10k(repeats, ncpu)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
