"""Generates the fixtures of the 10 000-line end-to-end decode-equality test (BASELINE configs[3]; VERDICT r1 next #2):

  tests/golden/trained_ref_cfg_bf16.npz   parameters trained on the GPU by tools/train_demo.py (reference configuration: fresh
                                          renders of 4-6 character lines, batch 64, lr 1e-4, 40 000 iterations; held-out exact
                                          match 100 % on 1024 lines), every value rounded to bf16 and stored as uint16 -- the
                                          oracle and the GPU path then start from bit-identical weights
  tests/golden/decode10k_oracle.npz       the ORACLE's greedy decode (fp32 restatement, oracle/crnn_oracle.py) of 10 240 rendered
                                          lines in 20 width-bucketed batches of 512 (W in {80,160,256}, lib/lstm/utils/gen.py
                                          BucketSampler, seed 77000, Pillow's embedded font), the ground-truth labels, every line's
                                          minimum top-2 logit margin, and a CRC of every rendered batch (so the GPU test can tell
                                          "the renderer produced different pixels here" from "the kernels decode differently")

    python tests/golden/make_decode10k.py build/trained_ref_cfg.npz        (~10 min on 8 cores)
"""
import os
import sys
import time
import zlib

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
HERE = os.path.dirname(os.path.abspath(__file__))
SEED, BATCH, NBATCH = 77000, 512, 20


def bf16_round(a):
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) >> 16                      # round to nearest even
    return u.astype(np.uint16)


def bf16_to_f32(u16):
    return (u16.astype(np.uint32) << 16).view(np.float32)


def load_weights(path=os.path.join(HERE, "trained_ref_cfg_bf16.npz")):
    z = np.load(path)
    return {k: bf16_to_f32(z[k]).reshape(z["shape/" + k]) for k in z.files if not k.startswith("shape/")}


def sampler():
    os.environ["CRNN_FONT"] = "default"                           # Pillow's embedded font: identical here and on the GPU box
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    gen._FONT_CACHE.clear()
    return gen.BucketSampler(batch_size=BATCH, render=True, seed=SEED, rank=0, world=1)


def batch_crc(data):
    return zlib.crc32(np.ascontiguousarray(data).tobytes()) & 0xFFFFFFFF


def main():
    src = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "build", "trained_ref_cfg.npz")
    P = dict(np.load(src))
    blob = {}
    for k, v in P.items():
        blob[k] = bf16_round(v).reshape(-1)
        blob["shape/" + k] = np.array(v.shape, np.int64)
    np.savez_compressed(os.path.join(HERE, "trained_ref_cfg_bf16.npz"), **blob)
    W = load_weights()
    from oracle import crnn_oracle as O
    p32 = O.to_torch({k: v.astype(np.float32) for k, v in W.items()}, torch.float32)
    s = sampler()
    dec_flat, dec_len, lab_flat, lab_len, margins, crcs, widths, tsls = [], [], [], [], [], [], [], []
    t0 = time.time()
    for k in range(NBATCH):
        imgs, lab, ll, tsl = s.batch(k)
        data = np.stack(imgs)
        tsl = np.asarray(tsl, np.int32)
        lo = O.forward(p32, data, tsl).numpy()
        dec = O.greedy_decode(lo, tsl)
        srt = np.sort(lo, axis=2)
        mg = srt[:, :, -1] - srt[:, :, -2]
        for n in range(BATCH):
            dec_flat += dec[n]; dec_len.append(len(dec[n]))
            margins.append(float(mg[:tsl[n], n].min()) if tsl[n] > 0 else 99.0)
        lab_flat += list(lab); lab_len += list(ll)
        crcs.append(batch_crc(data)); widths.append(data.shape[1]); tsls += tsl.tolist()
        acc = np.mean([dec[n] == list(lab[sum(ll[:n]):sum(ll[:n + 1])]) for n in range(BATCH)])
        print(f"batch {k} W={data.shape[1]} acc={acc:.4f} t={time.time() - t0:.0f}s", flush=True)
    np.savez_compressed(os.path.join(HERE, "decode10k_oracle.npz"), dec_flat=np.array(dec_flat, np.int8), dec_len=np.array(dec_len, np.int16),
                        lab_flat=np.array(lab_flat, np.int8), lab_len=np.array(lab_len, np.int16), min_margin=np.array(margins, np.float32),
                        crc=np.array(crcs, np.uint32), width=np.array(widths, np.int32), tsl=np.array(tsls, np.int16),
                        seed=np.array(SEED), batch=np.array(BATCH))
    print("done", time.time() - t0)


if __name__ == "__main__":
    main()
