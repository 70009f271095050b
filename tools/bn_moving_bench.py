"""Evaluation with moving BatchNorm statistics against batch statistics, in one call, on one GPU.

For bf16 and fp8 models holding the decode-10k fixture's trained weights (moving statistics: the batch statistics of the
timed batch itself, so both modes normalise with similar values), alternating batch and moving mode round by round:
  - CUDA-event time of the C3 forward + CTC loss (N = 1024, 32 x 256, 63 frames) per call, median over rounds;
  - per-stage times of the forward (crnn_profile_*; bn4_1_apply / bn4_2_apply_pool3 read ~0 in moving mode: the BatchNorm is
    folded into the conv4_x GEMMs);
  - packed evaluation as tools/eval_bench.py times it on the device: forward_lines + greedy decode over rendered lines in
    batches of --batch, lines/s;
and the card's name and power limit, read in the same run.  One JSON line per (dtype, mode).

    python tools/bn_moving_bench.py [--rounds 5] [--steps 20] [--lines 1024] [--batch 64]"""
import argparse
import importlib.util
import json
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from eval_bench import _card  # noqa: E402

N, W = 1024, 256


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--lines", type=int, default=1024)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()
    import torch
    from lstm_ctc_ocr_b200 import _lib, engine, synthetic
    from lstm_ctc_ocr_b200.lib.lstm.test import pack_lines, prepare_line
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    if not torch.cuda.is_available():
        raise SystemExit("bn_moving_bench measures the GPU: no CUDA device")
    os.environ["CRNN_FONT"] = "default"
    gen._FONT_CACHE.clear()
    spec = importlib.util.spec_from_file_location("make_decode10k", os.path.join(ROOT, "tests", "golden", "make_decode10k.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    weights = mk.load_weights()
    dev = torch.device("cuda:0")
    data, lab, ll, tsl = synthetic.synth_batch(N, W, seed=5)
    d_data, d_lab, d_ll, d_tsl = (torch.tensor(a, device=dev) for a in (data, lab, ll, tsl))
    mll = int(ll.max())
    rng = random.Random(2024)
    lines = [prepare_line(gen.render_line(gen.gen_rand(rng, 30, 70), rng=rng)) for _ in range(args.lines)]
    order = sorted(range(len(lines)), key=lambda i: lines[i][0].shape[1])
    packed = [tuple(torch.tensor(a, device=dev) for a in pack_lines([lines[i] for i in order[b:b + args.batch]]))
              for b in range(0, len(order), args.batch)]
    lib = _lib.load()
    names = [lib.crnn_profile_stage_name(i).decode() for i in range(lib.crnn_profile_num_stages())]
    card, limit = _card()
    for dt in ("bf16", "fp8"):
        m = engine.CrnnModel(device=dev, compute_dtype=dt)
        m.load_params(weights)
        if dt == "fp8":
            m.calibrate_fp8(d_data, d_tsl)
        m.forward(d_data, d_tsl)                                    # batch statistics of the timed batch -> moving buffer
        st = m.tap_raw("stats", N, W).double().cpu().numpy()
        cnt = N * (W // 4) * 4
        mean = st[:, 0] / cnt
        var = np.maximum(st[:, 1] / cnt - mean * mean, 0.0)
        m.load_bn_moving({k: (mean, var)[i % 2][i // 2] for i, k in enumerate(engine.BN_MOVING_KEYS)})
        calib = {}
        res = {mode: dict(ms=[], stages=[], lines_s=[]) for mode in ("batch", "moving")}
        logits = {}
        for r in range(args.rounds):
            for mode in ("batch", "moving"):
                m.set_bn_statistics(mode)
                if dt == "fp8":
                    if mode not in calib:
                        m.calibrate_fp8(d_data, d_tsl)
                        calib[mode] = m.fp8_scales()
                    else:
                        m.set_fp8_scales(calib[mode])
                for _ in range(3):                                  # warm-up of this mode's plan and kernels
                    engine.ctc_loss(m.forward(d_data, d_tsl), d_lab, d_ll, d_tsl, max_label_len=mll)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    lg = m.forward(d_data, d_tsl)
                    engine.ctc_loss(lg, d_lab, d_ll, d_tsl, max_label_len=mll)
                e1.record()
                torch.cuda.synchronize()
                res[mode]["ms"].append(e0.elapsed_time(e1) / args.steps)
                logits[mode] = lg.clone()
                _lib.check(lib.crnn_profile_begin(m.handle, args.steps))
                for _ in range(args.steps):
                    m.forward(d_data, d_tsl)
                buf = np.zeros((args.steps, len(names)), np.float32)
                nf = _lib.c_int()
                _lib.check(lib.crnn_profile_read(m.handle, buf.ctypes.data, nf))
                res[mode]["stages"].append(np.median(buf[:nf.value], axis=0))
                for p in packed:                                    # every batch shape once
                    engine.ctc_greedy(m.forward_lines(p[0], p[1], p[2]), p[2])
                torch.cuda.synchronize()
                e0.record()
                for p in packed:
                    engine.ctc_greedy(m.forward_lines(p[0], p[1], p[2]), p[2])
                e1.record()
                torch.cuda.synchronize()
                res[mode]["lines_s"].append(len(lines) / (e0.elapsed_time(e1) / 1e3))
        diff = float((logits["batch"] - logits["moving"]).abs().max())
        for mode, v in res.items():
            out = dict(card=card, power_limit=limit, dtype=dt, bn_statistics=mode, N=N, W=W, rounds=args.rounds, steps=args.steps,
                       fwd_ctc_ms_median=round(float(np.median(v["ms"])), 4), fwd_ctc_ms_all=[round(x, 4) for x in v["ms"]],
                       stages_ms=dict(zip(names, [round(float(x), 4) for x in np.median(np.stack(v["stages"]), axis=0)])),
                       packed_lines=len(lines), packed_batch=args.batch,
                       packed_lines_per_s_median=round(float(np.median(v["lines_s"])), 1),
                       max_abs_logit_diff_batch_vs_moving=round(diff, 5))
            print(json.dumps(out), flush=True)
        del m
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
