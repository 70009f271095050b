"""Lexicon-based reading: the candidate search (crnn_lexicon_candidates) and the candidates' CTC scores (crnn_ctc_lexicon_score)
against the forward pass of the same batch, with the trained fixture weights (tests/golden/trained_ref_cfg_bf16.npz):
  c3       T = 63, N = 1024: a W = 256 batch
  packed   T = 255, N = 64: a batch of 1024-px lines (packed evaluation's shape)
Reads are the greedy decode of the logits; lexicons are seeded random words of 2 - 15 ids, 1 000, 50 000 and 500 000 of them;
max_edit 3 (CRNN's delta) and -1 (no threshold), 64 candidates.  Each entry point is called through ctypes with preallocated
outputs; times are CUDA events around `--iters` back-to-back calls after `--warmup`, the median of `--reps` windows.  Prints one
JSON line with the card's name and power limit, read in the same run."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from align_bench import gpu_info, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lexicon_bench needs a CUDA device (an H100); nothing is measured without one")
    from lstm_ctc_ocr_b200 import _lib, engine, synthetic
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_decode10k", os.path.join(ROOT, "tests", "golden", "make_decode10k.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    lib = _lib.load()
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream().cuda_stream
    m = engine.CrnnModel(weight_decay=1e-5, device=dev)
    m.load_params(mk.load_weights())
    rng = np.random.default_rng(12)
    lexicons = {}
    for K in (1000, 50000, 500000):
        lexicons[K] = engine.Lexicon([rng.integers(1, 63, size=int(n)) for n in rng.integers(2, 16, size=K)], device=dev)
    res = dict(gpu_info(), iters=a.iters, reps=a.reps, shapes={})
    for name, N, W in (("c3", 1024, 256), ("packed", 64, 1024)):
        data, _, _, tsl = synthetic.synth_batch(N, W, seed=5)
        d_data, d_tsl = torch.tensor(data, device=dev), torch.tensor(tsl, device=dev)
        x = m.forward(d_data, d_tsl).clone()
        T = x.shape[0]
        o, ol = engine.ctc_greedy(x, d_tsl)
        reads = engine.dense_decoded(o, ol)
        if reads.shape[1] == 0:
            reads = torch.zeros((N, 1), dtype=torch.int32, device=dev)
        row = dict(T=T, N=N, mean_read_len=round(float(ol.float().mean()), 2), forward_ms=timed(lambda: m.forward(d_data, d_tsl),
                                                                                                 a.iters, a.warmup, a.reps), runs=[])
        J = 64
        cand, cdist, tot = (torch.empty((N, J), dtype=torch.int32, device=dev), torch.empty((N, J), dtype=torch.int32, device=dev),
                            torch.empty(N, dtype=torch.int32, device=dev))
        score = torch.empty((N, J), device=dev)
        best, bsc = torch.empty(N, dtype=torch.int32, device=dev), torch.empty(N, device=dev)
        for K, lex in lexicons.items():
            for delta in (3, -1):
                def cands():
                    _lib.check(lib.crnn_lexicon_candidates(reads.data_ptr(), reads.shape[1], ol.data_ptr(), N, lex.ids.data_ptr(),
                                                           lex.off.data_ptr(), len(lex), lex.max_entry_len, delta, J, cand.data_ptr(),
                                                           cdist.data_ptr(), tot.data_ptr(), st))

                def scores():
                    _lib.check(lib.crnn_ctc_lexicon_score(x.data_ptr(), d_tsl.data_ptr(), T, N, 64, 0, lex.ids.data_ptr(),
                                                          lex.off.data_ptr(), lex.max_entry_len, cand.data_ptr(), J, score.data_ptr(),
                                                          best.data_ptr(), bsc.data_ptr(), st))
                c_ms = timed(cands, a.iters, a.warmup, a.reps)
                s_ms = timed(scores, a.iters, a.warmup, a.reps)
                filled = float((cand >= 0).float().sum(1).mean())
                row["runs"].append(dict(K=K, max_edit=delta, candidates_ms=c_ms, score_ms=s_ms, mean_slots_filled=round(filled, 2),
                                        candidates_over_forward=round(c_ms / row["forward_ms"], 3),
                                        score_over_forward=round(s_ms / row["forward_ms"], 3)))
        res["shapes"][name] = row
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
