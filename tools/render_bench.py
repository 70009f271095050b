"""Training lines rendered on the device (gen.DeviceLineRenderer) against the host renderer (render_line + groupBatch in producer
processes, PrefetchFeeder), over --rounds rounds:
  - device lines/s: the renderer's full batch (layout, integer-feed copy, compositing, resize), host loop included, for the
    default 4-6 character stream at batches 64 and 1024, buckets 80 / 160 / 256 at 512 and 1024, and MIN_LEN 30 / MAX_LEN 70;
    and the CUDA-event time of one batch's render beside the training step it feeds;
  - host lines/s per producer (make_batch in this process, uint8) and through a PrefetchFeeder of 12 and 16 producers;
  - train_model-style steps/s (Session.run([loss, train_op])) at batch 64 (4-6 characters) and at bucket 256 x 1024, each fed by
    device renders, by feeder renders (16 producers) and by cached synthetic batches.
The card's name and power limit are read in the same run; one JSON line is printed at the end.

    python tools/render_bench.py [--rounds 3] [--steps 60]"""
import argparse
import json
import os
import statistics
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
    except Exception as e:
        return f"unknown ({e})", "unknown"


def _spread(v):
    return dict(median=round(statistics.median(v), 2), min=round(min(v), 2), max=round(max(v), 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=60, help="timed training steps per configuration and round")
    ap.add_argument("--batches", type=int, default=20, help="timed device batches per configuration and round")
    ap.add_argument("--producers", default="12,16")
    args = ap.parse_args()
    import torch
    from lstm_ctc_ocr_b200 import synthetic
    from lstm_ctc_ocr_b200.lib.lstm import train as T
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    if not torch.cuda.is_available():
        raise SystemExit("render_bench needs a CUDA device: there is nothing to measure without one")
    dev = "cuda:0"
    card, limit = _card()
    res = {"card": card, "power_limit": limit}

    dev_cfgs = [("default", 64, None, None), ("default", 1024, None, None)] + \
               [(f"bucket{b}", n, b, None) for b in (80, 160, 256) for n in (512, 1024)] + [("len30_70", 1024, None, (30, 70))]

    def device_rate(n, bucket, lens):
        r = gen.DeviceLineRenderer(n, seed=11, bucket=bucket, lens=lens, device=dev)
        for _ in range(3):
            next(r)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.batches):
            next(r)
        torch.cuda.synchronize()
        return n * args.batches / (time.perf_counter() - t0)

    def render_ms(n, bucket, lens):
        """CUDA-event time of one batch's layout + compositing + resize on the current stream."""
        from lstm_ctc_ocr_b200 import engine
        r = gen.DeviceLineRenderer(n, seed=11, bucket=bucket, lens=lens, device=dev)
        lo, hi, nw_lo, nw_hi = r.min_len, r.max_len, r.nw_lo, r.nw_hi
        layout, feeds = engine.render_layout(5, lo, hi, nw_lo, nw_hi, r.atlas, N=n)
        W = int(feeds[3].item())
        out = torch.empty((n, W, 32), dtype=torch.uint8, device=dev)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(3):
            engine.render_layout(5, lo, hi, nw_lo, nw_hi, r.atlas, layout, feeds)
            engine.render_lines_u8(layout, hi, r.atlas, W, r.workspace, out)
        a.record()
        for _ in range(20):
            engine.render_layout(5, lo, hi, nw_lo, nw_hi, r.atlas, layout, feeds)
            engine.render_lines_u8(layout, hi, r.atlas, W, r.workspace, out)
        b.record()
        b.synchronize()
        return a.elapsed_time(b) / 20

    def host_rate(n, bucket, lens):
        t0 = time.perf_counter()
        k = 0
        while time.perf_counter() - t0 < 2.0:
            gen.make_batch(k, n, True, seed=11, bucket=bucket, lens=lens, dtype=np.uint8)
            k += 1
        return n * k / (time.perf_counter() - t0)

    def feeder_rate(n, workers, bucket=None):
        f = gen.get_batch(workers, batch_size=n, seed=11, bucket=bucket, dtype=np.uint8, max_width=256)
        try:
            for _ in range(workers):
                next(f)
            t0 = time.perf_counter()
            m = 3 * workers
            for _ in range(m):
                next(f)
            return n * m / (time.perf_counter() - t0)
        finally:
            f.close()

    def steps_per_s(source, n, bucket):
        net = get_network("LSTM_train")
        with Session(device=dev) as sess:
            sw = T.SolverWrapper(sess, net, None, None, "/tmp/render_bench_out", "/tmp/render_bench_log")
            sess.engine_for(net).load_params(synthetic.init_params(3))
            loss, _ = net.build_loss()
            train_op = T.TrainOp(net, T.Variable(1e-4), T.Variable(0))
            sw._prepare(sess, False, train_op.lr, train_op.global_step)
            closer = None
            if source == "device":
                it = gen.DeviceLineRenderer(n, seed=11, bucket=bucket, device=dev)
            elif source == "feeder":
                it = closer = gen.get_batch(16, batch_size=n, seed=11, bucket=bucket, dtype=np.uint8, max_width=256)
                sess.attach_feeder(it)
            else:
                fixed = [gen.make_batch(k, n, False, seed=11, bucket=bucket, dtype=np.uint8) for k in range(4)]
                fixed = [(np.stack(b[0]), b[1], b[2], b[3]) for b in fixed]
                it = (fixed[k % 4] for k in range(10 ** 9))
            try:
                for _ in range(10):
                    sess.run([loss, train_op], sw._feed(next(it), 0.5))
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    sess.run([loss, train_op], sw._feed(next(it), 0.5))
                torch.cuda.synchronize()
                return args.steps / (time.perf_counter() - t0)
            finally:
                if closer is not None:
                    closer.close()

    rounds = {}
    for rnd in range(args.rounds):
        cur = {}
        for name, n, b, lens in dev_cfgs:
            cur[f"device_lines_per_s/{name}/N{n}"] = device_rate(n, b, lens)
            cur[f"device_render_ms/{name}/N{n}"] = render_ms(n, b, lens)
        cur["host_lines_per_s_per_producer/default"] = host_rate(64, None, None)
        cur["host_lines_per_s_per_producer/bucket256"] = host_rate(512, 256, None)
        for w in (int(x) for x in args.producers.split(",")):
            cur[f"feeder_lines_per_s/default/{w}_producers"] = feeder_rate(64, w)
        for src in ("device", "feeder", "cached"):
            cur[f"steps_per_s/batch64/{src}"] = steps_per_s(src, 64, None)
            cur[f"steps_per_s/bucket256_N1024/{src}"] = steps_per_s(src, 1024, 256)
        for k, v in cur.items():
            rounds.setdefault(k, []).append(v)
        print(f"round {rnd}: " + json.dumps({k: round(v, 3) for k, v in cur.items()}), flush=True)
    res.update({k: _spread(v) for k, v in rounds.items()})
    for name in ("batch64", "bucket256_N1024"):
        step_ms = 1e3 / res[f"steps_per_s/{name}/cached"]["median"]
        key = "device_render_ms/default/N64" if name == "batch64" else "device_render_ms/bucket256/N1024"
        res[f"render_share_of_step/{name}"] = round(res[key]["median"] / step_ms, 4)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
