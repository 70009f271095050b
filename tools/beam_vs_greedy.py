"""Side statistic asked for by SURVEY 8(c): how often does the reference's decode (TF beam search, width 100, merge_repeated=True,
[upstream-memory] restatement in oracle/) agree with the greedy rule the product implements?  CPU only.
Usage: python tools/beam_vs_greedy.py [lines_per_setting]  -> one JSON line on stdout"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import crnn_oracle as O  # noqa: E402


def lines(n, T, seed, margin, p63):
    """Frames peaked (by `margin` logits) at a path of CTC blanks (0), letters, repeats and -- with probability p63 -- class 63."""
    rng = np.random.default_rng(seed)
    pr = np.r_[0.30, np.full(62, (0.70 - p63) / 62), p63]
    path = rng.choice(64, size=(T, n), p=pr)
    rep = rng.random((T, n)) < 0.3
    for t in range(1, T):
        path[t] = np.where(rep[t], path[t - 1], path[t])
    x = rng.standard_normal((T, n, 64))
    x[np.arange(T)[:, None], np.arange(n)[None, :], path] += margin
    return x


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 100
    res = []
    t0 = time.time()
    for margin, p63, what in ((6.0, 0.0, "peaked, class 63 never wins (a net trained with warp-ctc blank 0)"),
                              (6.0, 0.10, "peaked, class 63 wins 10 % of the frames"),
                              (2.0, 0.0, "soft frames (margin 2 logits), class 63 never wins")):
        agree = agree_nomerge = total = 0
        for T in (19, 39, 63):
            x = lines(n, T, seed=int(margin * 10) + T, margin=margin, p63=p63)
            il = np.full(n, T)
            g = O.greedy_decode(x, il)
            b = O.beam_search_decode(x, il, merge_repeated=True)
            bn = O.beam_search_decode(x, il, merge_repeated=False)
            agree += sum(a == c for a, c in zip(g, b))
            agree_nomerge += sum(a == c for a, c in zip(g, bn))
            total += n
        res.append({"frames": what, "margin_logits": margin, "p_class63": p63, "lines": total,
                    "greedy_equals_reference_beam_decode": agree / total,
                    "greedy_equals_beam_without_output_merge": agree_nomerge / total})
        print(res[-1], f"{time.time() - t0:.0f}s", flush=True)
    out = {"what": "greedy (product) vs TF beam search width 100 (reference, restated in oracle/crnn_oracle.py:beam_search_decode, "
                   "[upstream-memory], not pinned against TF); T in {19,39,63}, zeros stripped on both sides", "settings": res}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
