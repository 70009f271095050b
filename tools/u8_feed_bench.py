"""f32 against uint8 feeds of the same C3 batches (1024 x 32x256) and of packed evaluation, alternated round by round.

Per round and feed dtype:
  - Session.run(loss) images/s: the PrefetchFeeder with device prefetch (built like bench.py's), a fresh pageable array per
    step, and the same buffer re-fed every step (page-locked in place after its second sighting);
  - device-resident forward + CTC (CUDA events) and the conv1 + pool1 stage time from crnn_profile;
  - Session.run([loss, train_op]) images/s with the feeder;
  - packed evaluation lines/s: 2048 rendered lines in batches of 64 through Session.run(dense_decoded), as tools/eval_bench.py
    times them, packed as f32 (data) or uint8 (data_u8).
The card's name, its power limit and the host CPU count are read in the same run.  One JSON line per (round, dtype) and a
summary line with the median of each row.

    python tools/u8_feed_bench.py [--rounds 3] [--steps 20]"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
N, W = 1024, 256


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in out.split(",")]
    except Exception as e:
        return [f"unknown ({e})", "unknown"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--lines", type=int, default=2048)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()
    import torch
    from lstm_ctc_ocr_b200 import engine, synthetic
    from lstm_ctc_ocr_b200.lib.lstm.test import pack_lines, prepare_line
    from lstm_ctc_ocr_b200.lib.lstm.train import TrainOp, Variable
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.LSTM_test import LSTM_test
    from lstm_ctc_ocr_b200.lib.networks.LSTM_train import LSTM_train
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.session import Session
    if not torch.cuda.is_available():
        raise SystemExit("u8_feed_bench measures the GPU: no CUDA device")
    os.environ["CRNN_FONT"] = "default"
    gen._FONT_CACHE.clear()
    params = synthetic.init_params(3, logits_scale=10.0)
    nwork = int(os.environ.get("CRNN_BENCH_FEED_WORKERS", "8"))
    rng = random.Random(2024)
    imgs = [gen.render_line(gen.gen_rand(rng, 30, 70), rng=rng) for _ in range(args.lines)]

    def sync():
        torch.cuda.synchronize()

    def rate(fn, n, per):
        sync()
        t0 = time.perf_counter()
        for i in range(n):
            fn(i)
        sync()
        return round(n * per / (time.perf_counter() - t0), 1)

    def one_round(dt):
        row = dict(dtype=np.dtype(dt).name)
        net = LSTM_train()
        loss, _ = net.build_loss()
        key = net.data_u8 if dt == np.uint8 else net.data
        arg_fn = lambda k: dict(k=k, batch_size=N, render=False, seed=3, rank=0, world=1, width=W, cache=4, dtype=dt)  # noqa: E731
        with Session() as sess:
            sess.assign(net, params)

            def run(data, lab, ll, tsl, fetches=loss):
                return sess.run(fetches, {key: data, net.labels: lab, net.labels_len: ll, net.time_step_len: tsl, net.keep_prob: 0.5})
            feeder = gen.PrefetchFeeder(arg_fn, num_workers=nwork, depth=4, max_width=W, batch_size=N, keep=2,
                                        warm=[arg_fn(k) for k in range(4)])
            try:
                sess.attach_feeder(feeder)
                step = lambda i: run(*next(feeder))  # noqa: E731
                for i in range(max(16, 8 * nwork)):
                    step(i)
                row["feeder_prefetch_img_s"] = rate(step, args.steps, N)
                row["feeder_path"] = sess.last_feed_path
                row["h2d_bytes"] = int(sess.h2d_bytes)
            finally:
                sess.attach_feeder(None)
                feeder.close()
            pool = [gen.make_batch(k, N, False, seed=3, width=W, dtype=dt) for k in range(2)]
            pool = [(np.ascontiguousarray(d), np.asarray(l, np.int32), np.asarray(ll, np.int32), np.asarray(t, np.int32))
                    for d, l, ll, t in pool]
            fresh = lambda i: run(np.array(pool[i % 2][0], copy=True), *pool[i % 2][1:])  # noqa: E731
            for i in range(3):
                fresh(i)
            row["pageable_fresh_img_s"] = rate(fresh, args.steps, N)
            refed = lambda i: run(*pool[0])  # noqa: E731
            for i in range(3):
                refed(i)
            row["refed_img_s"] = rate(refed, args.steps, N)
            row["refed_path"] = sess.last_feed_path
            # device-resident forward + CTC and the conv1 + pool1 stage
            eng = sess.engine_for(net)
            d = torch.tensor(pool[0][0], device=sess.device)
            lab, ll, tsl = (torch.tensor(a, device=sess.device) for a in pool[0][1:])
            mll = int(pool[0][2].max())

            def fwd(i):
                lg = eng.forward(d, tsl)
                engine.ctc_loss(lg, lab, ll, tsl, want_grad=True, grad_scale=1.0 / N, max_label_len=mll, workspace="auto")
            for i in range(3):
                fwd(i)
            row["resident_fwd_ctc_img_s"] = rate(fwd, args.steps, N)
            eng.lib.crnn_profile_begin(eng.handle, 10)
            for i in range(10):
                eng.forward(d, tsl)
            nst = eng.lib.crnn_profile_num_stages()
            ms = np.zeros((10, nst), np.float32)
            got = engine._lib.c_int()
            engine.check(eng.lib.crnn_profile_read(eng.handle, ms.ctypes.data, got))
            eng.lib.crnn_profile_begin(eng.handle, 0)
            names = [eng.lib.crnn_profile_stage_name(i).decode() for i in range(nst)]
            row["conv1_stage_ms"] = round(float(np.median(ms[:got.value, 0])), 4)
            row["conv1_stage_name"] = names[0]
            # training step with the feeder
            train = TrainOp(net, Variable(1e-4), Variable(0))
            feeder = gen.PrefetchFeeder(arg_fn, num_workers=nwork, depth=4, max_width=W, batch_size=N, keep=2,
                                        warm=[arg_fn(k) for k in range(4)])
            try:
                sess.attach_feeder(feeder)
                tstep = lambda i: run(*next(feeder), fetches=[loss, train])  # noqa: E731
                for i in range(max(8, 4 * nwork)):
                    tstep(i)
                row["train_feeder_img_s"] = rate(tstep, max(5, args.steps // 2), N)
            finally:
                sess.attach_feeder(None)
                feeder.close()
        # packed evaluation, as tools/eval_bench.py times it
        lines = [prepare_line(im, dtype=dt) for im in imgs]
        widths = [x.shape[1] for x, _ in lines]
        order = sorted(range(len(lines)), key=lambda i: widths[i])
        batches = [order[i:i + args.batch] for i in range(0, len(order), args.batch)]
        tnet = LSTM_test()
        fetch = Fetch(tnet, "dense_decoded")
        tkey = tnet.data_u8 if dt == np.uint8 else tnet.data
        with Session() as sess:
            sess.assign(tnet, params, ignore_missing=True)
            for b in batches[:2]:
                data, lw, ts = pack_lines([lines[i] for i in b])
                sess.run(fetch, {tkey: data, tnet.line_width: lw, tnet.time_step_len: ts})
            sync()
            t0 = time.perf_counter()
            for b in batches:
                data, lw, ts = pack_lines([lines[i] for i in b])
                sess.run(fetch, {tkey: data, tnet.line_width: lw, tnet.time_step_len: ts})
            row["packed_eval_lines_s"] = round(len(lines) / (time.perf_counter() - t0), 1)
        return row

    name, limit = _card()
    rows = []
    for r in range(args.rounds):
        for dt in (np.float32, np.uint8):
            row = dict(one_round(dt), round=r, card=name, power_limit=limit, host_cpus=os.cpu_count())
            rows.append(row)
            print(json.dumps(row), flush=True)
    summary = dict(card=name, power_limit=limit, host_cpus=os.cpu_count(), rounds=args.rounds)
    for dt in ("float32", "uint8"):
        rs = [r for r in rows if r["dtype"] == dt]
        for k, v in rs[0].items():
            if isinstance(v, float):
                vals = [r[k] for r in rs]
                summary[f"{dt}/{k}"] = [round(float(np.median(vals)), 4), round(float(min(vals)), 4), round(float(max(vals)), 4)]
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
