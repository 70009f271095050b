"""Evaluation throughput: one line per Session.run (the reference's lib/lstm/test.py loop) against packed batches.

Renders LINES text lines of 30 - 70 characters (W about 400 - 1000 px) with gen.render_line from a fixed seed and, on the same
lines and the decode-10k fixture's trained weights, reports
  - lines/s of test_model-style evaluation, one line per Session.run (prepare_line, run dense_decoded, decode);
  - lines/s of packed evaluation: lines grouped by width into batches of --batch, pack_lines, one Session.run each;
  - CUDA-event time of the packed forward + greedy decode alone (device tensors already resident), per batch and as lines/s.
The per-line and packed decodes are compared.  The card's name and power limit are read in the same run and printed.

    python tools/eval_bench.py [--lines 2048] [--batch 64]"""
import argparse
import importlib.util
import json
import os
import random
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception as e:        # the numbers are still printed; the card is then reported as unknown
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=2048)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20, help="timed repetitions of the device-only packed forward + decode")
    args = ap.parse_args()
    import torch
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.lstm.test import decodeRes, pack_lines, prepare_line
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.session import Session
    if not torch.cuda.is_available():
        raise SystemExit("eval_bench measures the GPU: no CUDA device")
    os.environ["CRNN_FONT"] = "default"
    gen._FONT_CACHE.clear()
    spec = importlib.util.spec_from_file_location("make_decode10k", os.path.join(ROOT, "tests", "golden", "make_decode10k.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    rng = random.Random(2024)
    lines = [prepare_line(gen.render_line(gen.gen_rand(rng, 30, 70), rng=rng)) for _ in range(args.lines)]
    widths = [d.shape[1] for d, _ in lines]
    net = get_network("LSTM_test")
    fetch = Fetch(net, "dense_decoded")
    with Session() as sess:
        sess.assign(net, mk.load_weights())
        eng = sess.engine_for(net)
        warm = lines[:8]
        for d, t in warm:                                         # module loads, first plans
            sess.run(fetch, {net.data: d, net.time_step_len: t})
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        per_line = []
        for d, t in lines:
            res = sess.run(fetch, {net.data: d, net.time_step_len: t})
            per_line.append("".join(decodeRes(res[0])))
        t_line = time.perf_counter() - t0

        order = sorted(range(len(lines)), key=lambda i: widths[i])
        batches = [order[i:i + args.batch] for i in range(0, len(order), args.batch)]
        packed = [pack_lines([lines[i] for i in b]) for b in batches]
        for (data, lw, tsl) in packed[:2]:
            sess.run(fetch, {net.data: data, net.line_width: lw, net.time_step_len: tsl})
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        got = {}
        for b in batches:
            data, lw, tsl = pack_lines([lines[i] for i in b])
            res = sess.run(fetch, {net.data: data, net.line_width: lw, net.time_step_len: tsl})
            for r, i in enumerate(b):
                got[i] = "".join(decodeRes(res[r]))
        t_packed = time.perf_counter() - t0
        same = sum(got[i] == per_line[i] for i in range(len(lines)))

        dev = [tuple(torch.tensor(a, device=sess.device) for a in p) for p in packed]
        for data, lw, tsl in dev:                                  # every batch shape once before timing
            engine.ctc_greedy(eng.forward_lines(data, lw, tsl), tsl)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            for data, lw, tsl in dev:
                engine.ctc_greedy(eng.forward_lines(data, lw, tsl), tsl)
        e1.record()
        torch.cuda.synchronize()
        ms_dev = e0.elapsed_time(e1) / args.reps
    name, limit = _card()
    pad = sum(p[0].shape[0] * p[0].shape[1] for p in packed) / sum(widths)
    out = dict(card=name, power_limit=limit, lines=len(lines), batch=args.batch, width_min=min(widths), width_max=max(widths),
               per_line_lines_per_s=round(len(lines) / t_line, 1), packed_lines_per_s=round(len(lines) / t_packed, 1),
               device_forward_decode_ms_per_pass=round(ms_dev, 3), device_lines_per_s=round(len(lines) / (ms_dev / 1e3), 1),
               padded_over_real_columns=round(pad, 4), decodes_equal=f"{same}/{len(lines)}")
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
