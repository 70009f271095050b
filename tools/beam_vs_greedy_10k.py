"""Side statistic SURVEY 8(c) asks for: how often the reference's decoder (TF beam search, width 100, merge_repeated -- the product's
host-side crnn_ctc_beam_search) and the north-star's greedy decoder agree on the 10 240 rendered lines of the decode-equality
fixture, through the TRAINED weights of tests/golden/trained_ref_cfg_bf16.npz.  CPU only: logits come from the oracle's fp32
forward (the GPU path decodes these lines identically to it, tests/test_gpu_decode10k.py).  ~10 min on 8 cores.

    python tools/beam_vs_greedy_10k.py [n_batches]  ->  one JSON line on stdout"""
import importlib.util
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from oracle import crnn_oracle as O                     # tools/ is measurement infrastructure, like tests/
    from lstm_ctc_ocr_b200 import engine
    spec = importlib.util.spec_from_file_location("mk", os.path.join(ROOT, "tests", "golden", "make_decode10k.py"))
    mk = importlib.util.module_from_spec(spec); spec.loader.exec_module(mk)
    fx = np.load(os.path.join(ROOT, "tests", "golden", "decode10k_oracle.npz"))
    nb = int(sys.argv[1]) if len(sys.argv) > 1 else len(fx["crc"])
    p32 = O.to_torch({k: v.astype(np.float32) for k, v in mk.load_weights().items()}, torch.float32)
    s = mk.sampler()
    B = int(fx["batch"])
    st = dict(lines=0, beam_eq_greedy=0, greedy_correct=0, beam_correct=0, beam_nomerge_correct=0, beam_nomerge_eq_greedy=0,
              truth_has_double_letter=0, beam_wrong_only_because_a_double_letter_was_merged=0, crc_mismatch=0, beam_seconds=0.0)
    t0 = time.time()
    for k in range(nb):
        imgs, lab, ll, tsl = s.batch(k)
        data = np.stack(imgs); tsl = np.asarray(tsl, np.int32)
        st["crc_mismatch"] += int(mk.batch_crc(data) != int(fx["crc"][k]))
        lo = O.forward(p32, data, tsl).numpy()
        greedy = O.greedy_decode(lo, tsl)
        tb = time.time()
        out, ol, _ = engine.ctc_beam_search(lo, tsl, beam_width=100, merge_repeated=True, strip=0)
        st["beam_seconds"] += time.time() - tb
        out2, ol2, _ = engine.ctc_beam_search(lo, tsl, beam_width=100, merge_repeated=False, strip=0)
        off = np.concatenate([[0], np.cumsum(ll)])
        for n in range(B):
            truth = [int(v) for v in lab[off[n]:off[n + 1]]]
            beam = out[n, :ol[n]].tolist(); beam2 = out2[n, :ol2[n]].tolist()
            dbl = any(a == b for a, b in zip(truth, truth[1:]))
            merged_truth = [v for i, v in enumerate(truth) if i == 0 or v != truth[i - 1]]
            st["lines"] += 1
            st["beam_eq_greedy"] += int(beam == greedy[n]); st["beam_nomerge_eq_greedy"] += int(beam2 == greedy[n])
            st["greedy_correct"] += int(greedy[n] == truth); st["beam_correct"] += int(beam == truth); st["beam_nomerge_correct"] += int(beam2 == truth)
            st["truth_has_double_letter"] += int(dbl)
            st["beam_wrong_only_because_a_double_letter_was_merged"] += int(dbl and beam != truth and beam == merged_truth)
        print(f"batch {k} W={data.shape[1]} {st['lines']} lines, beam==greedy {st['beam_eq_greedy']}, t={time.time() - t0:.0f}s", flush=True)
    st["beam_lines_per_s_host"] = round(st["lines"] / max(st["beam_seconds"], 1e-9), 1)
    st["host_cpus"] = os.cpu_count()
    st["what"] = ("10 240 rendered lines (bucketed 512 x W in {80,160,256}) through the trained fixture weights; logits from the oracle's fp32 forward; "
                  "beam = crnn_ctc_beam_search width 100 (the reference's decoder, network.py:656: merge_repeated=True collapses repeated labels of the "
                  "DECODED sequence too), greedy = the north-star decoder; *_nomerge = the same beam search with merge_repeated=False")
    print(json.dumps(st))


if __name__ == "__main__":
    main()
