"""n-best beam decode cost at C3 (1024 lines, T = 63, C = 64, logits of the trained fixture weights, beam width 100): the
device decoder (crnn_ctc_beam_search_topk_device) at top_paths 1, 10 and 100 and the host decoder (crnn_ctc_beam_search_topk)
at 1 and 100, each timed against the single-best decoder on the same logits in the same run, the two calls alternating.
Device: CUDA events around each call, after a warm-up; host: wall clock over all cores.  Prints one JSON line of medians.
Usage: python tools/nbest_bench.py [--repeats R] [--host-repeats H]"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lstm_ctc_ocr_b200 import engine, synthetic  # noqa: E402


def _card():
    import torch
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def _c3_logits():
    import torch
    spec = importlib.util.spec_from_file_location("make_decode10k", os.path.join(ROOT, "tests", "golden", "make_decode10k.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    data, _, _, tsl = synthetic.synth_batch(1024, 256, seed=5)
    m = engine.CrnnModel(weight_decay=1e-5, device="cuda:0")
    m.load_params(mk.load_weights())
    d_tsl = torch.tensor(tsl, dtype=torch.int32, device="cuda:0")
    x = m.forward(torch.tensor(data, dtype=torch.float32, device="cuda:0"), d_tsl).clone()
    torch.cuda.synchronize()
    return x, d_tsl


def _event_ms(call):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    call()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def _wall_ms(call):
    t0 = time.perf_counter()
    call()
    return (time.perf_counter() - t0) * 1e3


def _pair(timer, single, topk, repeats):
    """Median ms of each call and the median of the per-repeat differences, the two calls alternating."""
    single(); topk()
    s, k = [], []
    for _ in range(repeats):
        s.append(timer(single))
        k.append(timer(topk))
    s, k = np.array(s), np.array(k)
    return {"single_ms": round(float(np.median(s)), 3), "topk_ms": round(float(np.median(k)), 3),
            "topk_minus_single_ms": round(float(np.median(k - s)), 3),
            "single_ms_range": [round(float(s.min()), 3), round(float(s.max()), 3)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=21)
    ap.add_argument("--host-repeats", type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("nbest_bench needs a CUDA device")
    x, d_tsl = _c3_logits()
    T, N, C = x.shape
    W = 100
    res = {"card": _card(), "T": T, "lines": N, "C": C, "beam_width": W, "repeats": a.repeats, "device": {}, "host": {}}
    for K in (1, 10, 100):
        res["device"][f"K{K}"] = _pair(_event_ms, lambda: engine.ctc_beam_search_device(x, d_tsl, beam_width=W),
                                       lambda: engine.ctc_beam_search_topk_device(x, d_tsl, beam_width=W, top_paths=K), a.repeats)
    xh, th = x.cpu().numpy(), d_tsl.cpu().numpy()
    res["host_cpus"] = os.cpu_count()
    for K in (1, 100):
        res["host"][f"K{K}"] = _pair(_wall_ms, lambda: engine.ctc_beam_search(xh, th, beam_width=W),
                                     lambda: engine.ctc_beam_search_topk(xh, th, beam_width=W, top_paths=K), a.host_repeats)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
