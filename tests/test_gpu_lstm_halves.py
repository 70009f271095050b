"""csrc/lstm.cuh lstm_mc_kernel: two independent 64-row half pipelines per CTA, the cell on the wgmma accumulator fragments.

Every launch must compute the same bits: the exchange buffers and mbarrier phases start over per launch, and the training
launch only adds stores of the saved state.  The batch shapes cover a lone sample, a
half tile, a tile plus a few rows (the second tile's upper half has no valid row but must still run and exchange every
step), and the benchmark batch; the lengths include 0, 1 and T.

A sample's recurrence reads only its own input-projection rows, so each comparison is made on the samples whose `xproj`
rows are bit-identical in the two runs (the BatchNorm statistics upstream are f64 atomics, whose order may change the last
bit of a conv4 output between runs).
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
W = 100
T = W // 4 - 1


def _batch(N, W=W):
    from oracle import crnn_oracle as O
    pn = O.randomize_params(O.init_params(3, dtype=np.float32, logits_scale=10.0))
    rng = np.random.default_rng(N)
    # width 4 -> length 0, width 8 -> length 1, width W -> length T, the rest in between
    widths = [[W, 4, 8][i] if i < 3 else int(rng.integers(4, W + 1)) for i in range(N)]
    data, _, _, tsl = O.synth_batch(N, W, seed=N + 7, widths=widths, min_len=1, max_len=4)
    return pn, data, tsl


def _per_sample(x, N):
    """[dir * tiles + tile][step][...][row 128][k] -> [dir][sample n][step][...][k]"""
    x = x.reshape(2, -1, *x.shape[1:])                        # [dir][tile][step][..., 128, k]
    x = np.moveaxis(x, -2, 2)                                 # [dir][tile][row][step][..., k]
    return x.reshape(2, -1, *x.shape[3:])[:, :N]


def _run(pn, data, tsl, training):
    from lstm_ctc_ocr_b200 import engine
    N, W = data.shape[:2]
    T = W // 4 - 1
    m = engine.CrnnModel(device=DEV)
    m.load_params(pn)
    m.set_training(training)
    t = lambda a: torch.tensor(a, device=DEV)
    runs = []
    for _ in range(2):                                        # the exchange buffers and mbarrier phases start over per launch
        m.forward(t(data), t(tsl))
        torch.cuda.synchronize()
        r = {k: m.tap(k, N, W).cpu().numpy()[:, :T] for k in ("xproj", "lstm_out")}       # frames 0 .. T-1
        if training:
            r["gates"] = _per_sample(m.tap("gates", N, W).cpu().numpy(), N)      # [dir][n][step][gate][unit/8][8]
            r["csave"] = _per_sample(m.tap_raw("csave", N, W).cpu().numpy(), N)  # [dir][n][step][unit/4][4]
        runs.append(r)
    del m
    return runs


def _same_rows(a, b):
    same = np.array([np.array_equal(a["xproj"][n], b["xproj"][n]) for n in range(a["xproj"].shape[0])])
    assert same.sum() >= max(1, (9 * len(same)) // 10), f"only {same.sum()} of {len(same)} samples with identical xproj"
    return same


def _assert_same(a, b, tsl, what):
    T = a["lstm_out"].shape[1]
    same = _same_rows(a, b)
    assert np.array_equal(a["lstm_out"][same], b["lstm_out"][same]), f"{what}: lstm_out"
    if "gates" in a and "gates" in b:
        # saved state is written for the valid steps only
        for n in np.nonzero(same)[0]:
            L = int(min(max(tsl[n], 0), T))
            for k in ("gates", "csave"):
                assert np.array_equal(a[k][:, n, :L], b[k][:, n, :L]), f"{what}: {k} of sample {n}"


def check_launches_and_training_bit_identical(N, W=W):
    """Inference and training, two launches each, on one batch of N lines of width W."""
    T = W // 4 - 1
    pn, data, tsl = _batch(N, W)
    inf = _run(pn, data, tsl, training=False)
    trn = _run(pn, data, tsl, training=True)
    _assert_same(inf[0], inf[1], tsl, "inference launch 2 vs 1")
    _assert_same(trn[0], trn[1], tsl, "training launch 2 vs 1")
    _assert_same(inf[0], trn[0], tsl, "training vs inference")
    # outputs past a sample's length are exactly zero, in both directions
    L = np.minimum(np.maximum(tsl, 0), T)
    past = np.arange(T)[None, :] >= L[:, None]
    assert not inf[0]["lstm_out"][past].any()


@pytest.mark.parametrize("N", [1, 63, 130, 200, 1024])
def test_launches_and_training_are_bit_identical(N):
    check_launches_and_training_bit_identical(N)
