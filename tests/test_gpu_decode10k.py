"""10 240 rendered text lines, images -> conv -> BiLSTM -> greedy decode through `Session.run(dense_decoded)`, against the
ORACLE's decode of the same lines with the same (GPU-trained) weights -- BASELINE configs[3] ("variable-width bucketed batches
(W in {80,160,256}), batch 512, greedy-decode sequence equality vs ref") and the north-star's "greedy-decode sequence equality
on 10k synthetic lines".  Reference call sites: lib/networks/network.py:656-657 (decode -> dense, pad 0),
lib/lstm/utils/training.py:26-37 (strip 0, exact match).  Fixtures + generator: tests/golden/make_decode10k.py.

Stated bar: EVERY line whose minimum top-2 logit margin (oracle) exceeds MARGIN decodes identically; lines below it are reported,
not hidden: the unfiltered agreement must still be >= 99 % on the bf16 path and >= 99.9 % on the f32-class path."""
import importlib.util
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
MARGIN = 0.25          # logits; a few times the bf16 path's max |logit error| on these weights (max |logit| ~ 25)


def _mk():
    spec = importlib.util.spec_from_file_location("make_decode10k", os.path.join(ROOT, "tests", "golden", "make_decode10k.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    return mk


def run_decode10k(compute_dtype="bf16", device=DEV, max_batches=None):
    """Shared with bench.py's `decode_equality` field.  Returns the statistics dict."""
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    mk = _mk()
    fx = np.load(os.path.join(ROOT, "tests", "golden", "decode10k_oracle.npz"))
    weights = mk.load_weights()
    s = mk.sampler()
    B = int(fx["batch"])
    dec_off = np.concatenate([[0], np.cumsum(fx["dec_len"].astype(np.int64))])
    lab_off = np.concatenate([[0], np.cumsum(fx["lab_len"].astype(np.int64))])
    net = get_network("LSTM_test")
    _, dense_decoded = Fetches(net)
    stats = dict(lines=0, identical=0, clear_margin_lines=0, clear_margin_identical=0, correct_vs_truth=0, render_crc_mismatch=0,
                 per_width={})
    nb = len(fx["crc"]) if max_batches is None else min(max_batches, len(fx["crc"]))
    with Session(device=device) as sess:
        sess._engines[id(net)] = engine.CrnnModel(weight_decay=1e-5, device=device, compute_dtype=compute_dtype)
        sess.assign(net, weights)
        for k in range(nb):
            imgs, lab, ll, tsl = s.batch(k)
            data = np.stack(imgs)
            if mk.batch_crc(data) != int(fx["crc"][k]):
                stats["render_crc_mismatch"] += 1
            res = sess.run(dense_decoded, feed_dict={net.data: data, net.time_step_len: np.asarray(tsl, np.int32), net.keep_prob: 1.0})
            W = data.shape[1]
            pw = stats["per_width"].setdefault(str(W), dict(lines=0, identical=0))
            for n in range(B):
                g = k * B + n
                got = [int(v) for v in res[n] if v != 0] if res.size else []
                ref = fx["dec_flat"][dec_off[g]:dec_off[g + 1]].astype(np.int64).tolist()
                truth = fx["lab_flat"][lab_off[g]:lab_off[g + 1]].astype(np.int64).tolist()
                same = got == ref
                clear = float(fx["min_margin"][g]) > MARGIN
                stats["lines"] += 1; stats["identical"] += int(same); pw["lines"] += 1; pw["identical"] += int(same)
                stats["clear_margin_lines"] += int(clear); stats["clear_margin_identical"] += int(clear and same)
                stats["correct_vs_truth"] += int(got == truth)
    stats["filtered_out_by_margin"] = stats["lines"] - stats["clear_margin_lines"]
    stats["agreement_unfiltered"] = round(stats["identical"] / max(stats["lines"], 1), 5)
    stats["exact_match_accuracy"] = round(stats["correct_vs_truth"] / max(stats["lines"], 1), 5)
    stats["margin_threshold_logits"] = MARGIN
    stats["compute_dtype"] = compute_dtype
    return stats


def Fetches(net):
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    return Fetch(net, "logits"), Fetch(net, "dense_decoded")


@pytest.mark.parametrize("compute_dtype,min_agreement", [("bf16", 0.99), ("f32", 0.999), ("tf32", 0.995)])
def test_10k_rendered_lines_decode_equals_oracle(compute_dtype, min_agreement):
    if not os.path.exists(os.path.join(ROOT, "tests", "golden", "decode10k_oracle.npz")):
        pytest.skip("fixture missing: run tests/golden/make_decode10k.py")
    st = run_decode10k(compute_dtype)
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    with open(os.path.join(ROOT, "build", "parity_report.jsonl"), "a") as f:
        f.write(json.dumps(dict(test="decode10k", **st)) + "\n")
    assert st["render_crc_mismatch"] == 0, "the renderer produced different pixels than when the fixture was made"
    assert st["lines"] == 10240
    assert st["clear_margin_identical"] == st["clear_margin_lines"], st
    assert st["agreement_unfiltered"] >= min_agreement, st
    assert st["exact_match_accuracy"] >= 0.99, st
