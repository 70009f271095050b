"""The device beam-search decoder's host-side surface, without a GPU: the workspace query's argument checks and its growth
with the shapes, and no host fallback in engine.ctc_beam_search_device."""
import numpy as np
import pytest
import torch


def _size(T, N, C, bw):
    from lstm_ctc_ocr_b200 import _lib
    nbytes = _lib.c_size_t(0)
    st = _lib.load().crnn_ctc_beam_workspace_size(T, N, C, bw, nbytes)
    return st, nbytes.value


def test_beam_workspace_size_argument_checks():
    from lstm_ctc_ocr_b200 import _lib
    assert _size(63, 1024, 64, 100)[0] == 0
    assert _size(1, 1, 2, 1)[0] == 0 and _size(1, 1, 64, 128)[0] == 0
    for T, N in ((0, 4), (-1, 4), (8, 0), (8, -2)):
        assert _size(T, N, 64, 100)[0] == 1, (T, N)                      # CRNN_INVALID_VALUE
    for C, bw in ((1, 100), (65, 100), (64, 0), (64, 129), (64, -1)):
        assert _size(8, 4, C, bw)[0] == 4, (C, bw)                        # CRNN_UNSUPPORTED
    assert _size(2 ** 30, 2 ** 30, 64, 128)[0] == 4                       # the workspace would not fit a size_t / int index
    assert _lib.load().crnn_ctc_beam_workspace_size(8, 4, 64, 100, None) == 1
    assert len(_lib.load().crnn_last_error()) > 0


def test_beam_workspace_size_is_monotone_in_the_shapes():
    base = _size(63, 64, 64, 100)[1]
    assert base > 0
    for T, N, bw in ((64, 64, 100), (63, 65, 100), (63, 64, 101), (126, 64, 100), (63, 1024, 100), (63, 64, 128)):
        assert _size(T, N, 64, bw)[1] > base, (T, N, bw)
    for T in (1, 2, 10, 100, 1000):
        assert _size(T, 8, 64, 100)[1] < _size(T + 1, 8, 64, 100)[1]
    for N in (1, 2, 10, 100):
        assert _size(63, N, 64, 100)[1] < _size(63, N + 1, 64, 100)[1]
    for bw in (1, 2, 50, 127):
        assert _size(63, 8, 64, bw)[1] < _size(63, 8, 64, bw + 1)[1]


def test_device_beam_search_has_no_host_fallback():
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200._lib import CrnnError
    x = torch.zeros(4, 2, 64)
    il = torch.tensor([4, 1], dtype=torch.int32)
    with pytest.raises(CrnnError):
        engine.ctc_beam_search_device(x, il)
    with pytest.raises(CrnnError):
        engine.ctc_beam_search_device(np.zeros((4, 2, 64), np.float32), np.array([4, 1], np.int32))
