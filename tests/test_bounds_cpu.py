"""Guarded host buffers (tests/bounds.py): the host entry points stay inside the memory they are given, and the helper sees
what it is meant to see.

Controls: a one-byte write just before a body and one just after it are reported with their offsets, and so is a read of one
element past an input that feeds an output; a clean call is not.  Then the host decoders (crnn_ctc_beam_search,
crnn_ctc_beam_search_topk) at widths 1, 33 and 128 with K = width, C = 2 and 64, lengths 0 and T, and crnn_host_copy at sizes
around its per-thread split, every output and input guarded."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bounds as BD  # noqa: E402


def _lib():
    from lstm_ctc_ocr_b200 import _lib as L
    return L.load()


# ------------------------------------------------------------------------------------------------ controls
def _poke(g, at):
    """Change the byte at body offset `at` (negative: in the front guard) to a value the guard does not hold there."""
    i = g.off + at
    g.raw[i] = (int(g.raw[i]) + 1) % 256
    return 0


@pytest.mark.parametrize("at,where", [(-1, "front guard written at body offsets [-1, -1], 1 bytes"),
                                      (0, None), (63, None),
                                      (64, "back guard written at body offsets [64, 64], 1 bytes")])
def test_one_byte_writes_around_the_body_are_reported(at, where):
    out = BD.output_of("out", (16,), torch.float32, device="cpu")
    found, _ = BD.run_case(lambda: _poke(out, at), [out], device="cpu")
    if where is None:
        assert found == [], found
    else:
        assert found and all(where in f for f in found), found
        assert all(f.startswith(f"run {r}: out: ") for r, f in enumerate(found)), found


@pytest.mark.parametrize("extra", [0, 1])
def test_a_read_past_an_input_that_feeds_an_output_is_reported(extra):
    x = BD.input_of("x", np.arange(1, 10, dtype=np.float32), device="cpu")
    out = BD.output_of("sum", (1,), torch.float32, device="cpu")

    def call():
        n = 9 + extra
        out.view()[0] = x.raw[x.off:x.off + 4 * n].view(torch.float32).sum()
        return 0
    found, last = BD.run_case(call, [x, out], device="cpu")
    if extra:
        assert found == ["sum: differs (4 bytes) when the input guards are poisoned instead of 0: a read past an input"], found
    else:
        assert found == [] and float(last["sum"][0]) == 45.0


def test_a_write_into_an_input_guard_is_reported():
    x = BD.input_of("x", np.zeros(4, np.int32), device="cpu")
    found, _ = BD.run_case(lambda: _poke(x, 16), [x], device="cpu")
    assert len(found) == 3 and all("x: back guard written at body offsets [16, 16], 1 bytes" in f for f in found), found


def test_a_clean_state_buffer_and_an_unreproducible_nan_output():
    s = BD.Guarded("s", 32, kind="state", device="cpu", dtype=torch.float32).set(np.ones(8, np.float32))
    out = BD.output_of("o", (2,), torch.float32, device="cpu")
    runs = iter(range(3))

    def call():
        r = next(runs)
        s.view().mul_(2.0)
        out.view()[:] = float("nan") if r == 2 else float(r)
        return 0
    found, _ = BD.run_case(call, [s, out], device="cpu")
    assert found == ["o: not reproducible and not finite"], found
    assert torch.equal(s.saved.view(torch.float32), torch.ones(8))


# ------------------------------------------------------------------------------------------------ host entry points
def _beam_case(T, N, C, seed):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((T, N, C)) * 3).astype(np.float32)
    il = rng.integers(0, T + 1, size=N).astype(np.int32)
    il[0], il[-1] = 0, T
    return x, il


@pytest.mark.parametrize("C", [2, 64])
@pytest.mark.parametrize("width", [1, 33, 128])
def test_host_beam_search_stays_inside_its_buffers(width, C):
    lib = _lib()
    T, N = 19, 5
    x, il = _beam_case(T, N, C, seed=width + C)
    d_x, d_il = BD.input_of("logits", x, device="cpu"), BD.input_of("input_len", il, device="cpu")
    out = BD.output_of("out", (N, T), torch.int32, device="cpu")
    ol = BD.output_of("out_len", (N,), torch.int32, device="cpu")
    nlp = BD.output_of("neg_log_prob", (N,), torch.float32, device="cpu")
    call = lambda: lib.crnn_ctc_beam_search(d_x.ptr, d_il.ptr, T, N, C, width, 1, 0, out.ptr, ol.ptr, nlp.ptr, 2)
    found, single = BD.run_case(call, [d_x, d_il, out, ol, nlp], device="cpu")
    assert found == [], found
    K = width
    outk = BD.output_of("out", (N, K, T), torch.int32, device="cpu")
    olk = BD.output_of("out_len", (N, K), torch.int32, device="cpu")
    lpk = BD.output_of("log_prob", (N, K), torch.float32, device="cpu")
    npk = BD.output_of("num_paths", (N,), torch.int32, device="cpu")
    call = lambda: lib.crnn_ctc_beam_search_topk(d_x.ptr, d_il.ptr, T, N, C, width, K, 1, 0, outk.ptr, olk.ptr, lpk.ptr, npk.ptr, 2)
    found, topk = BD.run_case(call, [d_x, d_il, outk, olk, lpk, npk], device="cpu")
    assert found == [], found
    # path 0 is the single-best decode: the guarded calls computed what they should
    assert torch.equal(topk["out"][:, 0], single["out"]) and torch.equal(topk["out_len"][:, 0], single["out_len"])
    assert int(single["out_len"][0]) == 0 and int(topk["num_paths"][0]) == 1


@pytest.mark.parametrize("nbytes", [0, 1, 4095, 4097, 1 << 20, (1 << 20) + 3])
@pytest.mark.parametrize("threads", [1, 4])
def test_host_copy_stays_inside_its_buffers(nbytes, threads):
    lib = _lib()
    src = BD.input_of("src", np.random.default_rng(nbytes).integers(0, 256, nbytes, dtype=np.uint8), device="cpu")
    dst = BD.output_of("dst", (nbytes,), torch.uint8, device="cpu", align=1)
    found, last = BD.run_case(lambda: lib.crnn_host_copy(dst.ptr, src.ptr, nbytes, threads), [src, dst], device="cpu")
    assert found == [], found
    assert torch.equal(last["dst"], src.view())
