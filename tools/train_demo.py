"""End-to-end training demo on the GPU (VERDICT r1 "prove the training path learns").

Trains the CRNN from the reference initialisers with the reference-shaped solver (SolverWrapper.train_model) on FRESH
renders every step -- lines of MIN_LEN..MAX_LEN = 4..6 characters, batch 64, lr 1e-4 as lstm/lstm.yml sets them (reference
lib/lstm/utils/gen.py:69-110 draws a fresh captcha for every sample) -- fed by the page-locked PrefetchFeeder, and reports
  * the loss curve and the held-out exact-match accuracy (README.md:39-41 quotes > 95 %) every `eval_every` iterations,
  * agreement of the GPU greedy decode with the oracle's decode of the same weights on the held-out lines.
Writes build/train_demo_<tag>.json and (optionally) the trained parameters as build/trained_<tag>.npz.

    python tools/train_demo.py --iters 30000 --lr 1e-4 --batch 64 --seconds 240 --tag ref_cfg
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30000)
    ap.add_argument("--lr", type=float, default=1e-4)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=240.0, help="wall-clock budget of the training loop")
    ap.add_argument("--eval-every", type=int, default=2000)
    ap.add_argument("--eval-lines", type=int, default=1024)
    ap.add_argument("--workers", type=int, default=32)
    ap.add_argument("--bucketed", action="store_true", help="train on the W in {80,160,256} bucket stream instead of 4-6 character lines")
    ap.add_argument("--tag", default="ref_cfg")
    ap.add_argument("--save", action="store_true")
    ap.add_argument("--oracle-lines", type=int, default=256)
    args = ap.parse_args()

    import torch
    from lstm_ctc_ocr_b200.lib.lstm import train as T
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.lstm.utils.training import accuracy_calculation
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session

    cfg.TRAIN.LEARNING_RATE, cfg.TRAIN.DISPLAY, cfg.TRAIN.SNAPSHOT_ITERS, cfg.TRAIN.WEIGHT_DECAY = args.lr, 1000, 10 ** 9, 1e-5
    cfg.TRAIN.BATCH_SIZE, cfg.VAL.VAL_STEP, cfg.VAL.PRINT_NUM, cfg.TRAIN.STEPSIZE, cfg.TRAIN.GAMMA = args.batch, 10 ** 9, 0, 2000, 1.0
    assert gen.can_render(), "PIL cannot render 42-px glyphs on this box"
    B = args.batch
    if args.bucketed:
        arg_fn = lambda k: dict(k=k, batch_size=B, render=True, seed=1000, rank=0, world=1, bucket=gen.BUCKETS[k % 3])
        held_fn = lambda k: dict(k=k, batch_size=128, render=True, seed=900000, rank=0, world=1, bucket=gen.BUCKETS[k % 3])
    else:
        arg_fn = lambda k: dict(k=k, batch_size=B, render=True, seed=1000, rank=0, world=1)
        held_fn = lambda k: dict(k=k, batch_size=128, render=True, seed=900000, rank=0, world=1)
    held = [gen.make_batch(**held_fn(k)) for k in range(args.eval_lines // 128)]        # never seen in training (disjoint seeds)
    feeder = gen.PrefetchFeeder(arg_fn, num_workers=args.workers, depth=16, max_width=256, batch_size=B, keep=2)
    net = get_network("LSTM_train")
    out = {"iters_requested": args.iters, "batch": B, "lr": args.lr, "stream": "bucketed 80/160/256" if args.bucketed else "4-6 chars",
           "font": os.path.basename(gen._font_path() or "Pillow embedded default (scalable)"), "fresh_renders_every_step": True,
           "evals": []}
    try:
        with Session(device="cuda:0") as sess:
            sw = T.SolverWrapper(sess, net, None, None, "/tmp/train_demo_out", "/tmp/train_demo_log")
            loss_h, dec_h = net.build_loss()

            def evaluate():
                ok = tot = 0
                for (imgs, lab, ll, tsl) in held:
                    feed = {net.data: np.array(imgs), net.labels: np.array(lab), net.time_step_len: np.array(tsl),
                            net.labels_len: np.array(ll), net.keep_prob: 1.0}
                    res = sess.run(dec_h, feed_dict=feed)
                    org = sw.restoreLabel(lab, ll)
                    ok += accuracy_calculation(org, res, isPrint=False) * len(org); tot += len(org)
                return ok / tot

            # the solver loop is the reference's; run it in slices so that accuracy can be sampled along the way
            hist, done, t_start = [], 0, time.time()
            first = True
            while done < args.iters and time.time() - t_start < args.seconds:
                n = min(args.eval_every, args.iters - done)
                if first:
                    h = sw.train_model(sess, n + 1, restore=False, train_gen=feeder, val_gen=iter(held))
                    first = False
                else:
                    h = _continue(sw, sess, feeder, n)
                hist += h
                done += len(h)
                acc = evaluate()
                out["evals"].append({"iter": done, "seconds": round(time.time() - t_start, 1), "loss_mean_last_200": round(float(np.mean(hist[-200:])), 4),
                                     "heldout_accuracy": round(acc, 4)})
                print(out["evals"][-1], flush=True)
            torch.cuda.synchronize()
            out["iters"] = done
            out["train_seconds"] = round(time.time() - t_start, 1)
            out["loss_curve_mean_of_500"] = [round(float(np.mean(hist[i:i + 500])), 4) for i in range(0, len(hist), 500)]
            out["heldout_accuracy"] = out["evals"][-1]["heldout_accuracy"] if out["evals"] else None
            out["heldout_lines"] = args.eval_lines
            params = sess.variables(net)
            # ---- agreement with the oracle's decode on the trained weights (fp32 oracle: its own error is ~1e-6 of the logits)
            from oracle import crnn_oracle as O      # checker only
            p32 = O.to_torch({k: v.astype(np.float32) for k, v in params.items()}, torch.float32)
            agree = total = clear = 0
            worst = 0.0
            for (imgs, lab, ll, tsl) in held[:max(1, args.oracle_lines // 128)]:
                data = np.array(imgs)
                feed = {net.data: data, net.labels: np.array(lab), net.time_step_len: np.array(tsl), net.labels_len: np.array(ll), net.keep_prob: 1.0}
                res, logits_gpu = sess.run([dec_h, net.get_output("logits")], feed_dict=feed)
                lo = O.forward(p32, data, np.array(tsl)).numpy()         # BN uses batch statistics -> same batch composition
                ref = O.greedy_decode(lo, np.array(tsl))
                srt = np.sort(lo, axis=2)
                margin = srt[:, :, -1] - srt[:, :, -2]
                err = np.abs(logits_gpu - lo).max(axis=2)
                worst = max(worst, float(err.max() / np.abs(lo).max()))
                for n_ in range(len(ref)):
                    got = [int(v) for v in res[n_] if v != 0] if len(res) else []
                    total += 1
                    agree += int(got == ref[n_])
                    clear += int(np.all(margin[:tsl[n_], n_] > 2 * err[:tsl[n_], n_].max()))
            out.update(oracle_lines=total, decode_agreement_with_oracle=round(agree / total, 5), clear_margin_lines=clear,
                       max_logit_err_rel=round(worst, 5))
            if args.save:
                np.savez(os.path.join(ROOT, "build", f"trained_{args.tag}.npz"), **params)
    finally:
        feeder.close()
    print(json.dumps(out), flush=True)
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    json.dump(out, open(os.path.join(ROOT, "build", f"train_demo_{args.tag}.json"), "w"), indent=1)


def _continue(sw, sess, feeder, n):
    """n more iterations of the same solver state (the loop body of SolverWrapper.train_model, train.py:111-130)."""
    from lstm_ctc_ocr_b200.lib.lstm.train import TrainOp
    loss, _ = sw.net.build_loss()
    op = TrainOp(sw.net, sw._lr, sw._global_step, clip=10.0)
    hist = []
    for _ in range(n):
        v, _ = sess.run(fetches=[loss, op], feed_dict=sw._feed(next(feeder), 0.5))
        hist.append(float(v))
    return hist


if __name__ == "__main__":
    main()
