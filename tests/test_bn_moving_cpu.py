"""Moving BatchNorm statistics without a GPU: the update pinned to TensorFlow's assign_moving_average, the fold against the
unfolded fp64 forward, the checkpoint keys and the configuration key."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bn_moving_refs as M  # noqa: E402


def test_update_reproduces_tf_assign_moving_average():
    """tf.contrib.layers.batch_norm(decay=0.999, zero_debias_moving_mean=False): moving -= (moving - value) * (1 - decay).
    Values worked by hand for a batch with mean 2 and population variance 0.25 (sum 8, sum of squares 17 over 4 positions)
    from TF's initial mean 0 / variance 1: after one step 0.002 and 0.99925, after two 0.003998 and 0.99850075."""
    st = np.zeros((2, 2, 512))
    st[:, 0], st[:, 1] = 8.0, 17.0
    m1 = M.ema_update(M.initial(), st, 4.0)
    m2 = M.ema_update(m1, st, 4.0)
    # the ABI's decay is an f32: 1 - 0.999f is 1.29e-5 (relative) below TF's f32(1 - 0.999), and so is each step's increment
    np.testing.assert_allclose(m1[:, 0], 0.002, rtol=1.5e-5)
    np.testing.assert_allclose(m1[:, 1], 0.99925, rtol=2e-7)
    np.testing.assert_allclose(m2[:, 0], 0.003998, rtol=1.5e-5)
    np.testing.assert_allclose(m2[:, 1], 0.99850075, rtol=2e-7)
    assert m1.dtype == np.float32


def test_update_uses_the_population_variance_and_clamps_it():
    st = np.zeros((2, 2, 512))
    st[:, 0], st[:, 1] = 3.0, 3.0 * 3.0 / 3.0 - 1e-12      # mean 1, sumsq/count - mean^2 slightly negative: clamped to 0
    m = M.ema_update(M.initial(), st, 3.0, decay=0.0)
    assert np.all(m[:, 0] == 1.0) and np.all(m[:, 1] == 0.0)


@pytest.mark.parametrize("seed", [1, 2])
def test_folded_forward_equals_the_unfolded_moving_forward(seed):
    """relu(gamma (conv + b - mean) / sqrt(var + eps) + beta) == relu(conv(x; W s) + (b - mean) s + beta), including channels
    with negative gamma (s < 0 flips the sign of the folded weights), to 1e-12 in fp64."""
    from oracle import crnn_oracle as O
    p = O.randomize_params(O.init_params(seed, dtype=np.float32, logits_scale=10.0), seed=seed + 4)
    rng = np.random.default_rng(seed)
    mv = np.empty((2, 2, 512), np.float32)
    mv[:, 0] = rng.normal(0, 0.3, (2, 512))
    mv[:, 1] = rng.uniform(0.05, 2.0, (2, 512))
    for k in M.LAYERS:
        g = p[f"{k}/{k}/gamma"].copy()
        g[::3] = -np.abs(g[::3]) - 0.1                      # every third channel negative
        p[f"{k}/{k}/gamma"] = g.astype(np.float32)
    pt = O.to_torch({k: v.astype(np.float64) for k, v in p.items()})
    data, _, _, tsl = O.synth_batch(2, 48, seed=seed, widths=[48, 29])
    a = M.forward(pt, data, tsl, moving=mv)
    b = M.forward(pt, data, tsl, moving=mv, folded=True)
    assert torch.isfinite(a).all()
    assert float((a - b).abs().max()) <= 1e-12 * max(1.0, float(a.abs().max()))
    # and the moving forward differs from the batch-statistics forward (the statistics are not the batch's)
    assert float((a - M.forward(pt, data, tsl)).abs().max()) > 1e-3


def test_fold_rounds_once():
    """W' is the bf16 nearest to the exact fp64 product W * s, b' the f32 nearest to (b - mean) s + beta."""
    from oracle import crnn_oracle as O
    p = O.randomize_params(O.init_params(3, dtype=np.float32))
    mv = M.initial()
    mv[:, 1] = 0.37
    f = M.fold(p, mv)
    for k in M.LAYERS:
        w, we = f[k]["w"], f[k]["w_exact"]
        ulp = torch.ldexp(torch.ones_like(we), torch.frexp(we)[1] - 8)      # bf16 spacing at |W s|
        assert float(((w - we).abs() / ulp).max()) <= 0.5
        assert torch.equal(w.float().to(torch.bfloat16).double(), w)         # representable in bf16


class _Eng:
    """The parts of engine.CrnnModel that restore_bn_moving uses."""

    def __init__(self, mode):
        self.bn_statistics = mode
        self.loaded = "untouched"

    def load_bn_moving(self, state=None):
        self.loaded = state


def test_checkpoint_keys_round_trip_and_old_checkpoints(tmp_path):
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.lstm.train import restore_bn_moving
    assert engine.BN_MOVING_KEYS == ("conv4_1/conv4_1/moving_mean", "conv4_1/conv4_1/moving_variance",
                                     "conv4_2/conv4_2/moving_mean", "conv4_2/conv4_2/moving_variance")
    rng = np.random.default_rng(0)
    blob = {k: rng.normal(size=512).astype(np.float32) for k in engine.BN_MOVING_KEYS}
    np.savez(tmp_path / "new.npz", x=np.zeros(1), **blob)
    np.savez(tmp_path / "old.npz", x=np.zeros(1))
    for mode in ("batch", "moving"):
        e = _Eng(mode)
        restore_bn_moving(e, np.load(tmp_path / "new.npz"))
        assert sorted(e.loaded) == sorted(engine.BN_MOVING_KEYS)
        assert all(np.array_equal(e.loaded[k], blob[k]) for k in blob)
    e = _Eng("batch")
    restore_bn_moving(e, np.load(tmp_path / "old.npz"))
    assert e.loaded is None                                      # TF's initial values: mean 0, variance 1
    e = _Eng("moving")
    with pytest.raises(KeyError) as ei:
        restore_bn_moving(e, np.load(tmp_path / "old.npz"))
    assert all(k in str(ei.value) for k in engine.BN_MOVING_KEYS)
    assert e.loaded == "untouched"


def test_config_key_merge_and_set(tmp_path):
    from lstm_ctc_ocr_b200.lib.lstm import config as C
    saved = C.cfg.TEST.BN_STATS
    try:
        assert saved == "batch"
        f = tmp_path / "c.yml"
        f.write_text("TEST:\n  BN_STATS: moving\n")
        C.cfg_from_file(str(f))
        assert C.cfg.TEST.BN_STATS == "moving"
        C.cfg_from_list(["TEST.BN_STATS", "batch"])
        assert C.cfg.TEST.BN_STATS == "batch"
        C.cfg_from_list(["TEST.BN_STATS", "moving"])
        assert C.cfg.TEST.BN_STATS == "moving"
        with pytest.raises(ValueError):
            f.write_text("TEST:\n  BN_STATS: 1\n")
            C.cfg_from_file(str(f))
    finally:
        C.cfg.TEST.BN_STATS = saved


def test_header_documents_the_entry_points():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    h = open(os.path.join(root, "include", "crnn_ctc.h")).read()
    assert "int     crnn_model_bind_bn_moving(crnn_model* m, float* moving, float decay);" in h
    assert "int     crnn_model_set_bn_statistics(crnn_model* m, int moving);" in h
