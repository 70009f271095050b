"""The n-best beam-search decoder on the host (crnn_ctc_beam_search_topk, csrc/beam.cpp), without a GPU: against the fp64
exact prefix search where the beam is exhaustive, as a lower bound where it prunes, label for label against the Python
restatement of TF's CTCBeamSearchDecoder with top_paths (tests/nbest_refs.py), path 0 bit for bit the single-best decoder's,
and the surface around it: argument checks, padding, dense_decoded_topk, cfg.TEST.TOP_PATHS and test_model's output."""
import io
import os
import sys
from contextlib import redirect_stdout

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import beam_refs as BR  # noqa: E402
import nbest_refs as NR  # noqa: E402


def host_topk(x, il, width, K, merge_repeated=True, strip=0):
    from lstm_ctc_ocr_b200 import engine
    o, ol, lp, npaths = engine.ctc_beam_search_topk(x, il, beam_width=width, top_paths=K, merge_repeated=merge_repeated, strip=strip)
    return [[o[n, k, :ol[n, k]].tolist() for k in range(K)] for n in range(len(il))], lp, npaths


def oracle_topk(x, il, width, K, merge_repeated=True, strip=0):
    r = NR.beam_search_topk(x, il, width, K, merge_repeated, strip)
    paths = [[[] for _ in range(K)] for _ in r]
    lp = np.full((len(r), K), -np.inf, np.float32)
    for n, ps in enumerate(r):
        for k, (lab, v) in enumerate(ps):
            paths[n][k], lp[n, k] = lab, v
    return paths, lp, np.array([len(p) for p in r], np.int32)


@pytest.fixture(scope="module")
def cases():
    return NR.exhaustive_topk_cases()


def test_exact_topk_check_rejects_the_controls(cases):
    """The exact search itself passes the top-k check; each of beam_refs' wrong decoders fails it."""
    st, bad = NR.run_exhaustive_topk(NR.reference_topk_decoder(None), cases, widths=(128,), ks=(1, 7))
    assert not bad and st["lines"] > 0
    for mutant in BR.MUTANTS[1:]:
        _, bad = NR.run_exhaustive_topk(NR.reference_topk_decoder(mutant), cases, widths=(128,), ks=(1, 7))
        assert bad, mutant


def test_host_topk_is_the_k_most_probable_prefixes_where_exhaustive(cases):
    """Widths 128, 33 and each line's own prefix count; K 1, 2, 7 and the width; all four output modes."""
    st, bad = NR.run_exhaustive_topk(host_topk, cases)
    assert not bad, bad[:5]
    assert st["decided"] > 50_000, st


def test_oracle_topk_is_the_k_most_probable_prefixes_where_exhaustive(cases):
    dense = [c for c in cases if c[0].startswith("dense")]
    st, bad = NR.run_exhaustive_topk(oracle_topk, dense, widths=("peak",), ks=("width",))
    assert not bad, bad[:5]
    assert st["decided"] > 1000, st


def _pruned_and_blank_free_cases():
    out = [(name, x, il) for name, x, il in BR.pruned_cases()]
    x, il, _ = BR.sparse_batch(63, 128, 6)        # frames whose blank is impossible: runners-up can be lost below the width
    out.append(("sparse_T63", x, il))
    return out


@pytest.mark.parametrize("width", [2, 33, 128])
def test_host_topk_totals_are_lower_bounds_where_pruned(width):
    for name, x, il in _pruned_and_blank_free_cases():
        paths, lp, npaths = host_topk(x, il, width, width, merge_repeated=False, strip=-1)
        bad, slack = NR.check_lower_bound_topk(x, il, paths, lp, npaths)
        assert not bad, (name, width, bad[:3])
        assert len(slack) > 0


def _grid_cases():
    """Dense random lines (scales 0.3, 1, 3; ragged lengths including 0; a line with a NaN frame and one with a NaN logit) and
    sparse lines, C from 3 to 64, T in 1, 2, 19, 63."""
    rng = np.random.default_rng(11)
    for C in (3, 5, 17, 64):
        for T in (1, 2, 19, 63):
            x = (rng.standard_normal((T, 6, C)) * np.array([0.3, 1, 3, 1, 3, 0.3])[None, :, None]).astype(np.float32)
            il = rng.integers(0, T + 1, size=6).astype(np.int32)
            il[0], il[1] = T, 0
            x[rng.integers(0, T), 3] = np.nan
            x[rng.integers(0, T), 4, rng.integers(0, C)] = np.nan
            yield f"dense_C{C}_T{T}", x, il
    x, il, _ = BR.sparse_batch(63, 128, 3)
    yield "sparse_T63", x, il


@pytest.mark.parametrize("width", [1, 2, 33, 100, 128])
def test_host_topk_matches_the_restatement_and_path0_is_the_single_best_decode(width):
    from lstm_ctc_ocr_b200 import engine
    for name, x, il in _grid_cases():
        T = x.shape[0]
        if width >= 100 and T == 63 and x.shape[2] == 64 and not name.startswith("sparse"):
            slow_oracle = True                  # the Python restatement at full width and 64 classes: checked on the sparse lines
        else:
            slow_oracle = False
        for K in sorted({1, min(2, width), min(7, width), width}):
            for merge in (True, False):
                o, ol, lp, npaths = engine.ctc_beam_search_topk(x, il, beam_width=width, top_paths=K, merge_repeated=merge)
                so, sol, snlp = engine.ctc_beam_search(x, il, beam_width=width, merge_repeated=merge)
                assert np.array_equal(o[:, 0], so) and np.array_equal(ol[:, 0], sol), (name, width, K)
                assert np.array_equal((-lp[:, 0]).view(np.int32), snlp.view(np.int32)), (name, width, K)
                assert np.all((npaths >= 1) & (npaths <= K))
                assert np.all(lp[:, 1:] <= lp[:, :-1])
                if slow_oracle or (K > 7 and width > 33):
                    continue
                paths, rlp, rnp = oracle_topk(x, il, width, K, merge)
                got = [[o[n, k, :ol[n, k]].tolist() for k in range(K)] for n in range(len(il))]
                assert got == paths, (name, width, K, merge)
                assert np.array_equal(npaths, rnp)
                assert all(BR.within_one_ulp(a, b) for a, b in zip(lp.ravel(), rlp.ravel()))


def test_merged_prefixes_are_returned_separately():
    """"a blank a" and "a" are different prefixes; with merge_repeated both read as "a" and both are returned, each with its
    own exact probability."""
    x = np.log(np.array([[0.6, 0.1, 0.3], [0.2, 0.1, 0.7], [0.6, 0.1, 0.3]]))[:, None, :].astype(np.float32)
    il = np.array([3], np.int32)
    P, _ = BR.exact_prefix_search(x[:, 0], 3)
    paths, lp, npaths = host_topk(x, il, 100, 100, merge_repeated=True, strip=-1)
    raw, rlp, _ = host_topk(x, il, 100, 100, merge_repeated=False, strip=-1)
    k = npaths[0]
    assert k == len(P)
    assert np.array_equal(lp, rlp)
    idx = [i for i in range(k) if paths[0][i] == [0]]
    assert sorted(tuple(raw[0][i]) for i in idx) == [(0,), (0, 0)]
    for i in idx:
        assert BR.within_one_ulp(lp[0, i], np.float32(P[tuple(raw[0][i])]))


def test_num_paths_and_padding_past_the_listed_entries():
    from lstm_ctc_ocr_b200 import engine
    x = np.random.default_rng(0).standard_normal((4, 3, 3)).astype(np.float32)
    il = np.array([0, 1, 4], np.int32)
    o, ol, lp, npaths = engine.ctc_beam_search_topk(x, il, beam_width=8, top_paths=8)
    assert npaths[0] == 1 and ol[0, 0] == 0 and lp[0, 0] == 0.0          # only the empty prefix, log P = 0
    assert npaths[1] == 3                                                # the empty prefix, "0" and "1"
    for n in range(3):
        assert np.all(ol[n, npaths[n]:] == 0) and np.all(np.isneginf(lp[n, npaths[n]:]))
        assert not np.any(o[n, npaths[n]:])
    assert np.isclose(np.exp(lp[1, :3].astype(np.float64)).sum(), 1.0, atol=1e-6)


@pytest.mark.parametrize("K", [0, -1, 9])
def test_top_paths_outside_one_to_width_is_invalid(K):
    from lstm_ctc_ocr_b200 import _lib, engine
    x = np.zeros((4, 2, 5), np.float32)
    il = np.array([4, 2], np.int32)
    with pytest.raises(_lib.CrnnError, match="top_paths"):
        engine.ctc_beam_search_topk(x, il, beam_width=8, top_paths=K)
    out = np.zeros(2 * 4 * 16, np.int32); ol = np.zeros(32, np.int32)
    assert _lib.load().crnn_ctc_beam_search_topk(x.ctypes.data, il.ctypes.data, 4, 2, 5, 8, K, 1, 0, out.ctypes.data,
                                                 ol.ctypes.data, None, None, 1) == 1     # CRNN_INVALID_VALUE


def test_tensorflows_own_two_paths():
    """ctc_decoder_ops_test.py::testCTCDecoderBeamSearch decodes top_paths = 2 at beam_width 2 and pins both paths
    (tests/golden/third_party_kats.py): [1, 0] then [0, 1, 0]."""
    from golden import third_party_kats as K
    x, il = K.beam_case()
    paths, lp, npaths = host_topk(x.astype(np.float32), il, K.BEAM_WIDTH, 2, merge_repeated=True, strip=-1)
    assert paths[0] == K.BEAM_TOP_PATHS and npaths[0] == 2 and lp[0, 0] > lp[0, 1]
    assert oracle_topk(x, il, K.BEAM_WIDTH, 2, True, -1)[0][0] == K.BEAM_TOP_PATHS


def test_dense_decoded_topk_is_sparse_to_dense_per_path():
    from lstm_ctc_ocr_b200 import engine
    out = np.zeros((3, 2, 6), np.int32)
    out_len = np.array([[2, 0], [1, 3], [0, 0]], np.int32)
    out[0, 0, :2] = [4, 5]; out[1, 0, :1] = [7]; out[1, 1, :3] = [1, 2, 3]
    d = engine.dense_decoded_topk(out, out_len)
    assert len(d) == 2
    assert d[0].tolist() == [[4, 5], [7, 0], [0, 0]]
    assert d[1].tolist() == [[0, 0, 0], [1, 2, 3], [0, 0, 0]]


def test_top_paths_config_key():
    from lstm_ctc_ocr_b200.lib.lstm import config as C
    assert C.cfg.TEST.TOP_PATHS == 1
    try:
        C.cfg_from_list(["TEST.TOP_PATHS", "5"])
        assert C.cfg.TEST.TOP_PATHS == 5
    finally:
        C.cfg.TEST.TOP_PATHS = 1


class _Net:
    images = "images"
    keep_prob = "keep_prob"
    net = None

    def get_output(self, name):
        return self


class _Sess:
    """Session.run for test_model: the lines' reads from their file names, and for "beam_decoded" two paths per line."""

    def __init__(self, files):
        from lstm_ctc_ocr_b200.lib.lstm.config import get_encode_decode_dict
        self.enc = get_encode_decode_dict()[0]
        self.files = files
        self.fetched = []
        self.seen = 0

    def run(self, fetches, feed_dict):
        n = len(feed_dict["images"])
        names = self.files[self.seen:self.seen + n]          # one width: test_model keeps name order
        self.seen += n
        reads = [[self.enc[c] for c in f.split(".")[0].split("_")[1]] for f in names]
        L = max(len(r) for r in reads)
        dense = np.zeros((n, L), np.int32)
        for i, r in enumerate(reads):
            dense[i, :len(r)] = r
        flist = fetches if isinstance(fetches, list) else [fetches]
        self.fetched.append([f.kind for f in flist])
        out = []
        for f in flist:
            if f.kind == "dense_decoded":
                out.append(dense)
            elif f.kind == "beam_decoded":
                labels = np.zeros((n, 2, L), np.int32)
                labels[:, 0] = dense
                labels[:, 1, 0] = self.enc["z"]
                out.append({"labels": labels, "len": np.array([[len(r), 1] for r in reads], np.int32),
                            "log_prob": np.tile(np.log(np.array([0.75, 0.125], np.float32)), (n, 1)),
                            "num_paths": np.full(n, 2, np.int32)})
        return out if isinstance(fetches, list) else out[0]


def _test_model(tmp_path, K):
    from PIL import Image
    from lstm_ctc_ocr_b200.lib.lstm import test as T
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    files = ["0_ab1.png", "1_Zq.png", "2_x.png"]
    for f in files:
        Image.fromarray(np.zeros((32, 40), np.uint8)).save(tmp_path / f)
    sess = _Sess(files)
    cfg.TEST.TOP_PATHS = K
    try:
        buf = io.StringIO()
        with redirect_stdout(buf):
            correct, total = T.SolverWrapper(sess, _Net(), None, str(tmp_path), None).test_model(sess, testDir=str(tmp_path),
                                                                                               restore=False)
    finally:
        cfg.TEST.TOP_PATHS = 1
    lines = [ln for ln in buf.getvalue().splitlines() if "res:" in ln or ln.startswith("total acc")]
    return lines, sess.fetched, (correct, total)


def test_test_model_prints_todays_lines_with_one_path(tmp_path):
    lines, fetched, acc = _test_model(tmp_path, 1)
    assert fetched == [["dense_decoded"]]
    assert acc == (3, 3)
    assert lines == ["    res: ab1", "    res: Zq", "    res: x", "total acc:3/3=1.0000"]


def test_test_model_appends_the_n_best_reads(tmp_path):
    lines, fetched, acc = _test_model(tmp_path, 2)
    assert fetched == [["dense_decoded", "beam_decoded"]]
    assert acc == (3, 3)
    margin = float(np.log(np.float32(0.75)).astype(np.float64) - np.log(np.float32(0.125)).astype(np.float64))
    assert lines[0] == "    res: ab1, n-best: ab1 (0.7500), z (0.1250), margin: {:.4f}".format(margin)
    assert lines[-1] == "total acc:3/3=1.0000"
