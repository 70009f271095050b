"""The device beam-search decoder (crnn_ctc_beam_search_device, csrc/beam.cu) against the fp64 exact prefix search of
tests/beam_refs.py directly, not through the host decoder: the cases of test_beam_exact_cpu.py (dense frames at every
(C, T) width 128 covers exhaustively, sparse frames up to T = 1023 at widths 128 and 33), the lower bound on pruned decodes
(including the trained fixture weights' logits at C3 against ctc_refs.ctc_fp64), decodes shown to compact the arena, and the
arena staying inside its workspace.  Counts go to build/beam_exact_report.jsonl."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import beam_refs as BR  # noqa: E402
import ctc_refs as R  # noqa: E402
import test_beam_exact_cpu as CPU  # noqa: E402
import test_gpu_beam as GB  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def device_decoder(x, il, width, merge_repeated, strip):
    from lstm_ctc_ocr_b200 import engine
    o, ol, nlp = engine.ctc_beam_search_device(torch.tensor(np.ascontiguousarray(x), device=DEV), torch.tensor(il, device=DEV),
                                               beam_width=width, merge_repeated=merge_repeated, strip=strip)
    o, ol = o.cpu().numpy(), ol.cpu().numpy()
    return [o[i, :ol[i]].tolist() for i in range(len(il))], nlp.cpu().numpy()


def test_device_decoder_equals_the_exact_search():
    """Widths 128, 33, each line's measured count and one below it; both merge modes, strip 0 and -1."""
    st, bad, slack = BR.run_exhaustive(device_decoder, BR.exhaustive_cases())
    CPU.report(test="device_exhaustive", min_slack_ulps=float(slack.min()), **st)
    assert not bad, bad[:5]
    assert st["decided"] > 0 and st["pruned"] > 0


def test_device_decoder_lower_bound_on_pruned_decodes():
    st = dict(bound_fail=0)
    bad = []
    for name, x, il in BR.pruned_cases():
        for width in (1, 2, 7, 31, 32, 33, 64, 65, 100, 127, 128):
            lines, nlp = device_decoder(x, il, width, False, -1)
            bad += [(name, width) + e for e in BR.check_lower_bound(x, il, lines, nlp, st)[0]]
    CPU.report(test="device_lower_bound", **st)
    assert not bad, bad[:5]


def test_device_decoder_lower_bound_on_trained_logits():
    """The trained fixture weights at C3 (T = 63, N = 1024), widths 100 and 128: neg_log_prob >= -log P(out), with P(out)
    from ctc_refs.ctc_fp64 on the GPU; the slack distribution is reported."""
    from lstm_ctc_ocr_b200 import engine, synthetic
    mk = GB._load("make_decode10k", "tests", "golden", "make_decode10k.py")
    data, _, _, tsl = synthetic.synth_batch(1024, 256, seed=5)
    m = engine.CrnnModel(weight_decay=1e-5, device=DEV)
    m.load_params(mk.load_weights())
    d_tsl = torch.tensor(tsl, dtype=torch.int32, device=DEV)
    x = m.forward(torch.tensor(data, dtype=torch.float32, device=DEV), d_tsl)
    torch.cuda.synchronize()
    for width in (100, 128):
        o, ol, nlp = engine.ctc_beam_search_device(x, d_tsl, beam_width=width, merge_repeated=False, strip=-1)
        o, ol, nlp = o.cpu().numpy(), ol.cpu().numpy(), nlp.cpu().numpy()
        lines = [o[i, :ol[i]] for i in range(len(ol))]
        ref = R.ctc_fp64(x, np.concatenate(lines + [np.zeros(0, np.int32)]), ol, tsl, blank=63, max_label_len=max(int(ol.max()), 1))
        assert bool(ref["feasible"].all())
        logp = -ref["costs"].cpu().numpy()
        ulps, rel = BR.lower_bound_slack(nlp, logp)
        CPU.report(test="device_lower_bound_trained_c3", width=width, lines=len(ol), min_slack_ulps=float(ulps.min()),
                   exact_lines=int((np.abs(ulps) <= 1).sum()), slack_rel_quantiles=[float(q) for q in np.quantile(rel, [0, 0.5, 0.9, 1])])
        assert (ulps >= -1).all(), (width, np.flatnonzero(ulps < -1)[:5])


def _oracle_entries(x, length, width):
    """_Beam objects oracle.beam_search_decode creates over the first `length` frames (the root included)."""
    from oracle import crnn_oracle as O
    count = [0]

    class Counting(O._Beam):
        __slots__ = ()

        def __init__(self, *a):
            count[0] += 1
            super().__init__(*a)
    orig = O._Beam
    O._Beam = Counting
    try:
        O.beam_search_decode(x, [length], beam_width=width)
    finally:
        O._Beam = orig
    return count[0]


def test_device_decoder_compacts_the_arena():
    """Flat frames (C = 64, T = 24 and 63, widths 100 and 128) on which the arena is compacted.  The oracle creates an entry
    exactly when a new child first enters the beam, as the kernel does until its first compaction, so the oracle's count
    after all frames but the last is the kernel's arena use before the last frame unless it compacted earlier; either way
    count + width * (C - 1) > 1 + width * (T + C), the kernel's trigger, shows a compaction.  Those decodes must equal the
    host's and satisfy the lower bound."""
    C = 64
    rows = []
    for T in (24, 63):
        rng = np.random.default_rng(T)
        x = rng.standard_normal((T, 4, C)).astype(np.float32)
        il = np.full(4, T, np.int32)
        for width in (100, 128):
            for n in range(4):
                count = _oracle_entries(x[:, n:n + 1], T - 1, width)
                assert count + width * (C - 1) > 1 + width * (T + C), (T, width, n, count)
                rows.append(dict(T=T, width=width, line=n, entries_before_last_frame=count, cap=1 + width * (T + C)))
            GB._both(x, il, beam_width=width, merge_repeated=True)
            GB._both(x, il, beam_width=width, merge_repeated=False, strip=-1)
            lines, nlp = device_decoder(x, il, width, False, -1)
            st = dict(bound_fail=0)
            assert not BR.check_lower_bound(x, il, lines, nlp, st)[0]
    CPU.report(test="device_compaction", cases=rows)


def test_device_decoder_stays_inside_its_workspace():
    """The workspace sized by crnn_ctc_beam_workspace_size, filled with 0xFF, followed by a 64 KiB guard of a pattern; the
    heaviest utterance (flat frames, full length) last, so its arena slab ends at the guard.  The guard is unchanged after
    the call and the outputs equal those of a zero-filled workspace."""
    from lstm_ctc_ocr_b200 import _lib, engine
    lib = _lib.load()
    T, N, C, width = 63, 8, 64, 128
    rng = np.random.default_rng(11)
    x = GB._peaked_lines(N, T, seed=11, margin=2.0).astype(np.float32)
    x[:, -1] = rng.standard_normal((T, C))
    il = rng.integers(0, T + 1, size=N).astype(np.int32)
    il[-1] = T
    d_x, d_il = torch.tensor(x, device=DEV), torch.tensor(il, device=DEV)
    need = engine.beam_workspace_bytes(T, N, C, width)
    guard = 64 * 1024
    pattern = torch.arange(guard, dtype=torch.int64, device=DEV).mul_(2654435761).remainder_(251).to(torch.uint8)
    outs = []
    for fill in (0x00, 0xFF):
        buf = torch.empty(need + guard, dtype=torch.uint8, device=DEV)
        buf[:need].fill_(fill)
        buf[need:].copy_(pattern)
        out = torch.empty((N, T), dtype=torch.int32, device=DEV)
        ol = torch.empty(N, dtype=torch.int32, device=DEV)
        nlp = torch.empty(N, dtype=torch.float32, device=DEV)
        st = lib.crnn_ctc_beam_search_device(d_x.data_ptr(), d_il.data_ptr(), T, N, C, width, 1, 0, out.data_ptr(), ol.data_ptr(),
                                             nlp.data_ptr(), buf.data_ptr(), need, torch.cuda.current_stream().cuda_stream)
        assert st == 0
        torch.cuda.synchronize()
        assert torch.equal(buf[need:], pattern), fill
        outs.append((out.cpu(), ol.cpu(), nlp.cpu()))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
