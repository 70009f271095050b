"""Native-size evaluation input: the device resize (crnn_resize_lines_u8, the `images` feed) against the host path (prepare_line,
Pillow's resize per line, + pack_lines).

Renders LINES text lines of 30 - 70 characters at their native 60 rows with gen.render_line from a fixed seed and, with the
decode-10k fixture's trained weights, reports per round:
  - CUDA-event time of the resize of a batch of 64 and of 256 lines (width-sorted, as test_model batches them), beside
    forward_lines + greedy decode of the same batch, and the resize's share of the two;
  - end-to-end lines/s over all LINES lines in memory, preparation included: prepare_line + pack_lines + Session.run (data_u8 feed)
    against Session.run with the `images` feed, batches of --batch;
  - test_model wall time on a directory of the LINES lines as PNG files: the host path (prepare_line per file, pack_lines, data_u8)
    against test_model itself (`images`).
Rounds alternate the two paths; the decodes of the two are compared.  The card's name and power limit are read in the same run.

    python tools/resize_bench.py [--lines 2048] [--batch 64] [--rounds 3]"""
import argparse
import contextlib
import importlib.util
import json
import os
import random
import statistics
import subprocess
import sys
import tempfile
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


def _spread(v):
    return dict(median=round(statistics.median(v), 4), min=round(min(v), 4), max=round(max(v), 4), runs=[round(x, 4) for x in v])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=2048)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=50, help="timed repetitions of each device-only measurement")
    args = ap.parse_args()
    import torch
    from PIL import Image
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.lstm import test as T
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.session import Session
    if not torch.cuda.is_available():
        raise SystemExit("resize_bench measures the GPU: no CUDA device")
    os.environ["CRNN_FONT"] = "default"
    gen._FONT_CACHE.clear()
    spec = importlib.util.spec_from_file_location("make_decode10k", os.path.join(ROOT, "tests", "golden", "make_decode10k.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    rng = random.Random(2024)
    texts = [gen.gen_rand(rng, 30, 70) for _ in range(args.lines)]
    images = [gen.render_line(t, rng=rng) for t in texts]
    widths = [T.line_size(*im.shape)[1] for im in images]
    order = sorted(range(len(images)), key=lambda i: widths[i])
    batches = [order[i:i + args.batch] for i in range(0, len(order), args.batch)]
    cfg.TEST.BATCH_SIZE = args.batch
    net = get_network("LSTM_test")
    fetch = Fetch(net, "dense_decoded")
    dev = torch.device("cuda:0")

    def device_batch(idx):
        ims = [images[i] for i in idx]
        sz = np.array([T.line_size(*im.shape) for im in ims], np.int32)
        nb = np.array([im.size for im in ims], np.int64)
        off = np.zeros(len(ims), np.int64)
        np.cumsum(nb[:-1], out=off[1:])
        t = lambda a: torch.tensor(np.ascontiguousarray(a), device=dev)  # noqa: E731
        src = t(np.concatenate([im.reshape(-1) for im in ims]))
        return (src, t(off), t([im.shape[0] for im in ims]).int(), t([im.shape[1] for im in ims]).int(), t(sz[:, 0]),
                int(sz[:, 1].max()), max(im.shape[0] for im in ims)), t(sz[:, 1]), t(sz[:, 2])

    def events(fn, reps):
        fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / reps * 1e3          # us per call

    def host_path(sess):
        got = {}
        for b in batches:
            data, lw, tsl = T.pack_lines([T.prepare_line(images[i], dtype=np.uint8) for i in b])
            res = sess.run(fetch, {net.data_u8: data, net.line_width: lw, net.time_step_len: tsl})
            for r, i in enumerate(b):
                got[i] = "".join(T.decodeRes(res[r]))
        return got

    def device_path(sess):
        got = {}
        for b in batches:
            res = sess.run(fetch, {net.images: [images[i] for i in b]})
            for r, i in enumerate(b):
                got[i] = "".join(T.decodeRes(res[r]))
        return got

    def host_test_model(sess, test_dir):
        files = sorted(os.listdir(test_dir))
        lines = [T.prepare_line(T.load_line_image(os.path.join(test_dir, f)), dtype=np.uint8) for f in files]
        order_ = sorted(range(len(files)), key=lambda i: lines[i][0].shape[1])
        for b0 in range(0, len(order_), args.batch):
            idx = order_[b0:b0 + args.batch]
            data, lw, tsl = T.pack_lines([lines[i] for i in idx])
            sess.run(fetch, {net.data_u8: data, net.line_width: lw, net.time_step_len: tsl})

    out = dict(lines=args.lines, batch=args.batch, rounds=args.rounds, width_min=min(widths), width_max=max(widths))
    with Session() as sess, tempfile.TemporaryDirectory() as tmp:
        sess.assign(net, mk.load_weights())
        eng = sess.engine_for(net)
        for i, (t, im) in enumerate(zip(texts, images)):
            Image.fromarray(im).save(os.path.join(tmp, f"{i:05d}_{t}.png"))
        sw = T.SolverWrapper.__new__(T.SolverWrapper)
        sw.net, sw.pretrained_model, sw.output_dir = net, None, tmp
        # device-only: the resize against forward_lines + greedy decode, per batch size (the middle batch of the width order)
        dev_rows = {}
        for bs in (64, 256):
            idx = order[len(order) // 2 - bs // 2: len(order) // 2 + bs // 2]
            rz, lw, tsl = device_batch(idx)
            rs = lambda: engine.resize_lines_u8(*rz)  # noqa: E731
            data = rs()
            fd = lambda: engine.ctc_greedy(eng.forward_lines(data, lw, tsl), tsl)  # noqa: E731
            rows = {"resize_us": [], "forward_decode_us": []}
            for _ in range(args.rounds):
                rows["resize_us"].append(events(rs, args.reps))
                rows["forward_decode_us"].append(events(fd, max(args.reps // 5, 5)))
            share = [a / b for a, b in zip(rows["resize_us"], rows["forward_decode_us"])]
            dev_rows[bs] = dict(W=int(data.shape[1]), src_bytes=int(rz[0].numel()), out_bytes=int(data.numel()),
                                resize_us=_spread(rows["resize_us"]), forward_decode_us=_spread(rows["forward_decode_us"]),
                                resize_share=_spread(share))
        out["device"] = dev_rows
        # end to end in memory, and test_model on the PNG directory; the two paths alternate within each round
        host_path(sess)
        device_path(sess)
        e2e = {"host": [], "device": []}
        tm = {"host": [], "device": []}
        same = None
        for _ in range(args.rounds):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            a = host_path(sess)
            e2e["host"].append(args.lines / (time.perf_counter() - t0))
            t0 = time.perf_counter()
            b = device_path(sess)
            e2e["device"].append(args.lines / (time.perf_counter() - t0))
            same = sum(a[i] == b[i] for i in range(args.lines))
            with open(os.devnull, "w") as null, contextlib.redirect_stdout(null):
                t0 = time.perf_counter()
                host_test_model(sess, tmp)
                tm["host"].append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                sw.test_model(sess, testDir=tmp, restore=False)
                tm["device"].append(time.perf_counter() - t0)
        out["e2e_lines_per_s"] = {k: _spread(v) for k, v in e2e.items()}
        out["e2e_speedup"] = _spread([d / h for h, d in zip(e2e["host"], e2e["device"])])
        out["test_model_s"] = {k: _spread(v) for k, v in tm.items()}
        out["decodes_equal"] = f"{same}/{args.lines}"
    name, limit = _card()
    out = dict(card=name, power_limit=limit, host_cpus=os.cpu_count(), **out)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
