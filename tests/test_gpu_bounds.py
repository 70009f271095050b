"""Every entry point stays inside the memory it is given: writes inside each caller-owned buffer, reads inside each input.

Each buffer is guarded by tests/bounds.py: [front guard | body | back guard], the body exactly the size the header or the size
query gives, at the alignment the entry point requires (1024 bytes for model workspaces, 256 for render, 16 for the beam arena,
16 for f32 model data and logits, the element's size elsewhere), each guard at least 1 MiB (4 MiB next to model workspaces).
Outputs are poisoned with 0xFF before each call, guards hold a position-dependent pattern; inputs end at their back guard,
which holds 0 in two runs and 0xFF in a third.  After each run every guard must be intact; then what the two zero runs
reproduce bit for bit must be unchanged in the 0xFF run, and float outputs two runs do not reproduce (the weight gradients,
summed with f32 atomics) must be finite.  Every call goes through the C ABI with raw pointers (no engine slack).

  entry point                                    cases
  crnn_forward / _u8                             test_model_forward_and_backward: N 1 .. 1160, W 8 .. 1024, inference + training
  crnn_backward / _u8                            test_model_forward_and_backward (the CTC gradient of the forward as dlogits)
  crnn_ctc_loss                                  test_model_forward_and_backward, test_ctc_loss (fast, tma, each in log and me
                                                 recursion, generic 1 / 2 / 4, the workspace kernel at its exact size)
  crnn_model_bind / _bind_bn_moving              every model case (params, grads, slots and moving statistics guarded)
  crnn_clip_adam_step / _momentum / _rmsprop     test_solver_steps_and_total_loss
  crnn_total_loss                                test_solver_steps_and_total_loss
  crnn_forward_host / _pageable (+ _u8)          test_host_fed_forward: chunks 1 and 4
  crnn_forward_lines / _u8                       test_forward_lines: batch and moving statistics
  crnn_model_calibrate_fp8 (+ _u8)               test_fp8_and_f32_class_forwards: fp8 calibrate, forward, lines; compute_dtype 2, 3
  crnn_ctc_greedy                                test_greedy (aligned logits and 4 bytes off), test_greedy_control
  crnn_ctc_beam_search_device / _topk_device     test_device_beam: widths 1, 33, 128, K = width, C 2 and 64
  crnn_ctc_align                                 test_align: L 0, 64, 639, T 1 and 2048, the exact workspace
  crnn_lexicon_candidates, crnn_ctc_lexicon_score  test_lexicon: read strides 300 / 513 / 1024, K 1 and 50 000, T 768
  crnn_resize_lines_u8                           test_resize: max_h 1024, out_w 1 and W, a line ending at src's last byte
  crnn_render_layout, crnn_render_lines_u8       test_render: N 1 and 1024, bucketed and not, max_len 256, exact workspace
  crnn_ctc_beam_search, _topk, crnn_host_copy    tests/test_bounds_cpu.py (host memory)

The controls: test_greedy_control tells crnn_ctc_greedy N + 1 utterances with its buffers sized for N (the overrun stays inside
the guards); the back guards of out and out_len must be reported, and logits guards poisoned with frames peaked at class 5 must show
in the outputs.  Alignment:
every pointer the kernels access wider than its element (f32 data and data_staging, logits_out, dlogits, the bound params /
grads / slots) offset by 4 bytes, and the moving statistics by 2, returns CRNN_INVALID_VALUE on the host and leaves the outputs
untouched (test_misaligned_pointers_are_refused).  A short report goes to build/bounds_report.json (158 cases, 1101 guarded
buffers).  The file runs in 28 s (23 s of tests) on an H100 80GB HBM3 at a 700 W power limit."""
import ctypes
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bounds as BD  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WS_GUARD = 4 << 20
INVALID = 1
_REPORT = {"cases": 0, "buffers": 0, "entry_points": set()}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    with open(os.path.join(ROOT, "build", "bounds_report.json"), "w") as f:
        json.dump(dict(_REPORT, entry_points=sorted(_REPORT["entry_points"])), f, indent=1)


def _lib():
    from lstm_ctc_ocr_b200 import _lib as L
    return L.load()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _err():
    return _lib().crnn_last_error().decode()


def _case(entries, call, buffers):
    """One guarded case over `buffers`; `entries` names the entry points `call` runs."""
    found, last = BD.run_case(call, buffers, device=DEV)
    assert found == [], (entries, found, _err())
    _REPORT["cases"] += 1
    _REPORT["buffers"] += len(buffers)
    _REPORT["entry_points"].update(entries)
    return last


def _inp(name, a, align=16, poison=0xFF):
    return BD.input_of(name, a, device=DEV, align=align, poison=poison)


def _out(name, shape, dtype, align=16, compare=True, guard=BD.GUARD):
    return BD.output_of(name, shape, dtype, device=DEV, align=align, compare=compare, guard=guard)


def _ws(name, nbytes, align):
    return BD.Guarded(name, nbytes, kind="out", align=align, guard=WS_GUARD, device=DEV, compare=False)


def _size(fn, *args):
    b = ctypes.c_size_t()
    assert fn(*args, ctypes.byref(b)) == 0, _err()
    return int(b.value)


def _lens(N, T, rng):
    il = rng.integers(0, T + 1, size=N).astype(np.int32)
    il[0] = T
    if N > 1:
        il[1] = 0
    return il


def _labels(N, m, rng, blank=0, il=None):
    ll = rng.integers(0, m + 1, size=N).astype(np.int32)
    ll[0] = m
    if il is not None:
        ll = np.minimum(ll, np.maximum(il // 2, 0)).astype(np.int32)
        ll[0] = min(m, max(int(il[0]) // 2, 0))
    ids = [c for c in range(64) if c != blank]
    lab = rng.choice(ids, size=int(ll.sum())).astype(np.int32)
    return lab, ll


# ------------------------------------------------------------------------------------------------------------- decoders
@pytest.mark.parametrize("offset", [0, 4])
@pytest.mark.parametrize("T", [1, 33, 1023])
def test_greedy(T, offset):
    lib = _lib()
    N, C = 9, 64
    rng = np.random.default_rng(T)
    x = (rng.standard_normal((T, N, C)) * 3).astype(np.float32)
    lg = BD.Guarded("logits", x.nbytes, kind="in", align=16, offset=offset, device=DEV, dtype=torch.float32, shape=x.shape).set(x)
    il = _inp("input_len", _lens(N, T, rng))
    out, ol = _out("out", (N, T), torch.int32), _out("out_len", (N,), torch.int32)
    _case(["crnn_ctc_greedy"], lambda: lib.crnn_ctc_greedy(lg.ptr, il.ptr, T, N, C, 63, 0, out.ptr, ol.ptr, _st()), [lg, il, out, ol])


def test_greedy_control():
    """N + 1 utterances told, buffers sized for N: both back guards written, and the logits read past the input.  An all-0xFF
    (NaN) frame decodes like an all-zero one (class 0), so the logits' poison here is frames peaked at class 5."""
    import re
    lib = _lib()
    T, N, C = 33, 4, 64
    rng = np.random.default_rng(1)
    x = (rng.standard_normal((T, N, C)) * 3).astype(np.float32)
    row = np.zeros(C, np.float32)
    row[5] = 5.0
    peaked = torch.tensor(np.tile(row, BD.GUARD // (4 * C) + 1), device=DEV).view(torch.uint8)
    lg, il = _inp("logits", x, poison=peaked), _inp("input_len", np.full(N, T, np.int32))
    out, ol = _out("out", (N, T), torch.int32), _out("out_len", (N,), torch.int32)
    found, _ = BD.run_case(lambda: lib.crnn_ctc_greedy(lg.ptr, il.ptr, T, N + 1, C, 63, 0, out.ptr, ol.ptr, _st()), [lg, il, out, ol],
                           device=DEV)

    def span(name):
        hits = [re.search(name + r": back guard written at body offsets \[(\d+), (\d+)\]", f) for f in found]
        return [(int(h.group(1)), int(h.group(2))) for h in hits if h]
    assert span("out") and all(N * T * 4 <= a <= b < (N + 1) * T * 4 for a, b in span("out")), found
    assert span("out_len") and all(N * 4 <= a <= b < (N + 1) * 4 for a, b in span("out_len")), found
    assert any(f.startswith("out: differs") for f in found), found
    assert not any("front guard" in f or "logits:" in f or "input_len:" in f for f in found), found
    _REPORT["controls"] = found


@pytest.mark.parametrize("C", [2, 64])
@pytest.mark.parametrize("width", [1, 33, 128])
def test_device_beam(width, C):
    lib = _lib()
    T, N = 17, 5
    rng = np.random.default_rng(width * C)
    x = (rng.standard_normal((T, N, C)) * 3).astype(np.float32)
    lg, il = _inp("logits", x), _inp("input_len", _lens(N, T, rng))
    need = _size(lib.crnn_ctc_beam_workspace_size, T, N, C, width)
    ws = _ws("workspace", need, 16)
    out, ol, nlp = _out("out", (N, T), torch.int32), _out("out_len", (N,), torch.int32), _out("neg_log_prob", (N,), torch.float32)
    one = _case(["crnn_ctc_beam_search_device"],
                lambda: lib.crnn_ctc_beam_search_device(lg.ptr, il.ptr, T, N, C, width, 1, 0, out.ptr, ol.ptr, nlp.ptr, ws.ptr, need,
                                                        _st()), [lg, il, out, ol, nlp, ws])
    K = width
    outk, olk = _out("out", (N, K, T), torch.int32), _out("out_len", (N, K), torch.int32)
    lpk, npk = _out("log_prob", (N, K), torch.float32), _out("num_paths", (N,), torch.int32)
    top = _case(["crnn_ctc_beam_search_topk_device"],
                lambda: lib.crnn_ctc_beam_search_topk_device(lg.ptr, il.ptr, T, N, C, width, K, 1, 0, outk.ptr, olk.ptr, lpk.ptr,
                                                             npk.ptr, ws.ptr, need, _st()), [lg, il, outk, olk, lpk, npk, ws])
    assert torch.equal(top["out"][:, 0], one["out"]) and torch.equal(top["out_len"][:, 0], one["out_len"])


# ----------------------------------------------------------------------------------------------------------------- CTC
# (env, max_label_len, T): each kernel at T just below its ceiling (tests/test_gpu_width_edges.py's limits)
CTC_KERNELS = {"fast": ({}, 4, 550), "fast-me": ({"CRNN_CTC_RECUR": "me"}, 15, 348),
               "tma": ({"CRNN_CTC_KERNEL": "tma"}, 15, 256), "tma-me": ({"CRNN_CTC_KERNEL": "tma", "CRNN_CTC_RECUR": "me"}, 4, 256),
               "generic1": ({"CRNN_CTC_KERNEL": "generic"}, 15, 517), "generic2": ({}, 31, 259), "generic4": ({}, 63, 130),
               "workspace": ({}, 200, 600)}


def _ctc_buffers(x, lab, ll, il):
    return [_inp("logits", x, align=16), _inp("flat_labels", lab), _inp("label_len", ll), _inp("input_len", il)]


@pytest.mark.parametrize("blank", [0, 63])
@pytest.mark.parametrize("N", [1, 37])
@pytest.mark.parametrize("kernel", list(CTC_KERNELS))
def test_ctc_loss(kernel, N, blank, monkeypatch):
    lib = _lib()
    env, m, T = CTC_KERNELS[kernel]
    for k in ("CRNN_CTC_KERNEL", "CRNN_CTC_RECUR"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(T + N + blank)
    x = (rng.standard_normal((T, N, 64)) * 2).astype(np.float32)
    il = _lens(N, T, rng)
    lab, ll = _labels(N, m, rng, blank)
    ins = _ctc_buffers(x, lab, ll, il)
    # the size query is non-zero wherever a misaligned call would need the workspace (T = 550 here); aligned, only the
    # workspace kernel's case gets one
    need = _size(lib.crnn_ctc_workspace_size, T, N, 64, m) if kernel == "workspace" else 0
    assert need > 0 or kernel != "workspace"
    ws = _ws("workspace", max(need, 1), 16)
    costs, grad = _out("costs", (N,), torch.float32), _out("grad", (T, N, 64), torch.float32, align=16)
    _case(["crnn_ctc_loss"], lambda: lib.crnn_ctc_loss(ins[0].ptr, grad.ptr, ins[1].ptr, ins[2].ptr, ins[3].ptr, T, N, 64, blank, m,
                                                       1.0 / N, costs.ptr, ws.ptr if need else None, need, _st()),
          ins + [costs, grad, ws])


# ----------------------------------------------------------------------------------------------------------- alignment
@pytest.mark.parametrize("T", [1, 2048])
@pytest.mark.parametrize("L", [0, 64, 639])
def test_align(L, T):
    lib = _lib()
    N = 3
    rng = np.random.default_rng(L + T)
    x = (rng.standard_normal((T, N, 64)) * 2).astype(np.float32)
    il = _lens(N, T, rng)
    ll = np.array([L, L // 2, 0 if L else 0], np.int32)
    lab = rng.integers(1, 64, size=int(ll.sum())).astype(np.int32)
    need = _size(lib.crnn_ctc_align_workspace_size, T, N, 64, max(L, 1))
    for stride in (0, max(L, 1)):
        if stride:
            dense = np.zeros((N, stride), np.int32)
            o = 0
            for n in range(N):
                dense[n, :ll[n]] = lab[o:o + ll[n]]
                o += ll[n]
            labels, shape = dense, (N, stride)
        else:
            labels, shape = lab, (int(ll.sum()),)
        ins = [_inp("logits", x), _inp("labels", labels), _inp("label_len", ll), _inp("input_len", il)]
        ws = _ws("workspace", need, 1)
        s, e = _out("start", shape, torch.int32), _out("end", shape, torch.int32)
        pk, lp = _out("peak", shape, torch.float32), _out("path_logprob", (N,), torch.float32)
        _case(["crnn_ctc_align"], lambda: lib.crnn_ctc_align(ins[0].ptr, ins[1].ptr, stride, ins[2].ptr, ins[3].ptr, T, N, 64, 0, max(L, 1),
                                                             s.ptr, e.ptr, pk.ptr, lp.ptr, ws.ptr, need, _st()),
              ins + [s, e, pk, lp, ws])


# ------------------------------------------------------------------------------------------------------------- lexicon
def _lexicon(K, rng, max_len=24):
    lens = rng.integers(1, max_len + 1, size=K)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    return rng.integers(1, 64, size=int(off[-1])).astype(np.int32), off


@pytest.mark.parametrize("K", [1, 50000])
@pytest.mark.parametrize("stride", [300, 513, 1024])
def test_lexicon(stride, K):
    lib = _lib()
    N, T, mel = 4, 768, 24
    rng = np.random.default_rng(stride + K)
    ids, off = _lexicon(K, rng, mel)
    reads = rng.integers(0, 64, size=(N, stride)).astype(np.int32)
    rl = np.array([stride, 0, 7, int(off[1] - off[0])], np.int32)
    reads[3, :rl[3]] = ids[:rl[3]]
    ins = [_inp("reads", reads), _inp("read_len", rl), _inp("lex_ids", ids), _inp("lex_off", off)]
    x = (rng.standard_normal((T, N, 64)) * 2).astype(np.float32)
    lg, il = _inp("logits", x), _inp("input_len", _lens(N, T, rng))
    for mc, max_edit in ((1, 3), (256, -1)):
        cand, dist, tot = _out("cand", (N, mc), torch.int32), _out("cand_dist", (N, mc), torch.int32), _out("cand_total", (N,), torch.int32)
        last = _case(["crnn_lexicon_candidates"],
                     lambda: lib.crnn_lexicon_candidates(ins[0].ptr, stride, ins[1].ptr, N, ins[2].ptr, ins[3].ptr, K, mel, max_edit, mc,
                                                         cand.ptr, dist.ptr, tot.ptr, _st()), ins + [cand, dist, tot])
        cd = _inp("cand", last["cand"].cpu().numpy())
        sc, best, bs = _out("score", (N, mc), torch.float32), _out("best", (N,), torch.int32), _out("best_score", (N,), torch.float32)
        _case(["crnn_ctc_lexicon_score"],
              lambda: lib.crnn_ctc_lexicon_score(lg.ptr, il.ptr, T, N, 64, 0, ins[2].ptr, ins[3].ptr, mel, cd.ptr, mc, sc.ptr, best.ptr,
                                                 bs.ptr, _st()), [lg, il, ins[2], ins[3], cd, sc, best, bs])


# ------------------------------------------------------------------------------------------------------ resize, render
def test_resize():
    lib = _lib()
    W, max_h = 96, 1024
    rng = np.random.default_rng(2)
    lines = [(1024, 60, 1), (32, W, W), (100, 300, W), (7, 5, 1)]        # (h, w, out_w); the last one ends at src's last byte
    src = rng.integers(0, 256, size=sum(h * w for h, w, _ in lines)).astype(np.uint8)
    offs = np.concatenate([[0], np.cumsum([h * w for h, w, _ in lines])[:-1]]).astype(np.int64)
    N = len(lines)
    ins = [_inp("src", src), _inp("src_offset", offs), _inp("src_h", np.array([h for h, _, _ in lines], np.int32)),
           _inp("src_w", np.array([w for _, w, _ in lines], np.int32)), _inp("out_w", np.array([o for _, _, o in lines], np.int32))]
    out = _out("out", (N, W, 32), torch.uint8, align=4)
    _case(["crnn_resize_lines_u8"],
          lambda: lib.crnn_resize_lines_u8(*[g.ptr for g in ins], N, W, max_h, out.ptr, _st()), ins + [out])


@pytest.mark.parametrize("bucket", [None, 256])
@pytest.mark.parametrize("N", [1, 1024])
def test_render(N, bucket):
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    lib = _lib()
    atlas = engine.GlyphAtlas(gen._font(42), device=DEV)
    lo, hi, nw_lo, nw_hi = gen._render_range(bucket, None if bucket else (1, 256))
    glyphs, masks = _inp("glyphs", atlas.glyphs.cpu().numpy()), _inp("masks", atlas.masks.cpu().numpy())
    layout = _out("layout", (N, engine.render_record_ints(hi)), torch.int32)
    feeds = _out("feeds", (engine.render_feed_ints(N, hi),), torch.int32)
    last = _case(["crnn_render_layout"], lambda: lib.crnn_render_layout(77, N, lo, hi, nw_lo, nw_hi, glyphs.ptr, atlas.nglyphs, layout.ptr,
                                                                        feeds.ptr, _st()), [glyphs, layout, feeds])
    W = int(last["feeds"][3])
    lay = _inp("layout", last["layout"].cpu().numpy())
    need = _size(lib.crnn_render_workspace_size, N, hi, atlas.max_adv)
    ws, out = _ws("workspace", need, 256), _out("out", (N, W, 32), torch.uint8, align=4)
    _case(["crnn_render_lines_u8"], lambda: lib.crnn_render_lines_u8(lay.ptr, N, hi, glyphs.ptr, masks.ptr, atlas.max_adv, W, ws.ptr, need,
                                                                      out.ptr, _st()), [lay, glyphs, masks, ws, out])


# --------------------------------------------------------------------------------------------------------------- model
class Model:
    """A model handle whose params, grads, slots and moving statistics live in guarded buffers (bound through the C ABI)."""

    def __init__(self, dtype=1, training=False, seed=3):
        from lstm_ctc_ocr_b200 import engine, synthetic
        self.lib = _lib()
        self.e = engine.CrnnModel(device=DEV, compute_dtype=dtype)
        self.e.load_params(synthetic.init_params(seed, logits_scale=10.0))
        if training:
            self.e.set_training(True)
        self.h = self.e.handle
        n = self.e.total
        self.params = BD.Guarded("params", 4 * n, kind="state", device=DEV, dtype=torch.float32).set(self.e.params)
        self.slots = [BD.Guarded(k, 4 * n, kind="state", device=DEV, dtype=torch.float32) for k in ("grads", "adam_m", "adam_v")]
        for s, v in zip(self.slots, (0.0, 0.0, 1.0)):
            s.set(torch.full((n,), v, dtype=torch.float32, device=DEV))
        assert self.lib.crnn_model_bind(self.h, self.params.ptr, *[s.ptr for s in self.slots]) == 0, _err()
        self.moving = None
        if dtype in (1, 4):
            mv = np.stack([np.zeros((2, 512), np.float32), np.ones((2, 512), np.float32)], 1)
            mv[:, 0] += np.linspace(-0.1, 0.1, 512, dtype=np.float32)
            self.moving = BD.Guarded("bn_moving", mv.nbytes, kind="state", align=4, device=DEV, dtype=torch.float32).set(mv)
            assert self.lib.crnn_model_bind_bn_moving(self.h, self.moving.ptr, 0.9) == 0, _err()

    def bound(self):
        return [self.params] + ([self.moving] if self.moving is not None else [])

    def changed(self):
        """Every run re-derives the operand copies from the guarded params (a read past them would show)."""
        assert self.lib.crnn_model_params_changed(self.h) == 0
        return 0

    def ws(self, N, W, train=False, lines=False):
        if lines:
            need = _size(self.lib.crnn_lines_workspace_size, self.h, N, W)
        else:
            need = _size(self.lib.crnn_model_workspace_size, self.h, N, W, 1 if train else 0)
        return _ws("workspace", need, 1024), need


def _batch(N, W, u8, seed):
    rng = np.random.default_rng(seed)
    T = W // 4 - 1
    data = rng.integers(0, 256, size=(N, W, 32)).astype(np.uint8)
    if not u8:
        data = data.astype(np.float32) / np.float32(255)
    tsl = _lens(N, T, rng)
    return data, tsl, rng


def _seq(*calls):
    for c in calls:
        st = c()
        if st != 0:
            return st
    return 0


FWD_SHAPES = [(1, 8), (3, 12), (130, 40), (1160, 160), (3, 516), (1, 1024), (130, 516), (1160, 40)]


@pytest.mark.parametrize("u8", [False, True], ids=["f32", "u8"])
@pytest.mark.parametrize("N,W", FWD_SHAPES, ids=[f"N{n}_W{w}" for n, w in FWD_SHAPES])
def test_model_forward_and_backward(N, W, u8):
    """Inference forward, then a training forward, the CTC gradient of its logits (grad_scale 1/N) and the backward."""
    sfx = "_u8" if u8 else ""
    T = W // 4 - 1
    data, tsl, rng = _batch(N, W, u8, N + W)
    d, t = _inp("data", data, align=16 if not u8 else 4), _inp("time_step_len", tsl)
    m = Model()
    ws, need = m.ws(N, W)
    logits = _out("logits", (T, N, 64), torch.float32, align=16)
    fwd = getattr(m.lib, "crnn_forward" + sfx)
    _case(["crnn_forward" + sfx, "crnn_model_bind", "crnn_model_bind_bn_moving"],
          lambda: _seq(m.changed, lambda: fwd(m.h, d.ptr, t.ptr, N, W, logits.ptr, ws.ptr, need, _st())),
          [d, t, ws, logits] + m.bound())
    del m, ws
    m = Model(training=True)
    ws, need = m.ws(N, W, train=True)
    lab, ll = _labels(N, 4, rng, il=tsl)
    ctc = _ctc_buffers(np.zeros((T, N, 64), np.float32), lab, ll, tsl)[1:]
    costs, dl = _out("costs", (N,), torch.float32), _out("dlogits", (T, N, 64), torch.float32, align=16)
    grads = m.slots[0]
    grads.kind = "out"
    bwd = getattr(m.lib, "crnn_backward" + sfx)
    _case(["crnn_forward" + sfx, "crnn_backward" + sfx, "crnn_ctc_loss"],
          lambda: _seq(m.changed, lambda: fwd(m.h, d.ptr, t.ptr, N, W, logits.ptr, ws.ptr, need, _st()),
                       lambda: m.lib.crnn_ctc_loss(logits.ptr, dl.ptr, ctc[0].ptr, ctc[1].ptr, ctc[2].ptr, T, N, 64, 0, 4, 1.0 / N, costs.ptr,
                                                   None, 0, _st()),
                       lambda: bwd(m.h, d.ptr, t.ptr, dl.ptr, N, W, ws.ptr, need, _st())),
          [d, t, ws, logits, costs, dl, grads] + ctc + m.bound())


@pytest.mark.parametrize("solver", ["adam", "momentum", "rmsprop"])
def test_solver_steps_and_total_loss(solver):
    """One training step's gradient, then the solver step with params, grads and both slots guarded (each read and
    written), and crnn_total_loss's loss_out."""
    N, W = 130, 40
    T = W // 4 - 1
    data, tsl, rng = _batch(N, W, False, 9)
    m = Model(training=True)
    ws, need = m.ws(N, W, train=True)
    dt, tt = torch.tensor(data, device=DEV), torch.tensor(tsl, device=DEV)
    dl = (torch.randn((T, N, 64), generator=torch.Generator().manual_seed(1)) * 0.05).to(DEV)
    lg = torch.empty((T, N, 64), device=DEV)
    assert m.lib.crnn_forward(m.h, dt.data_ptr(), tt.data_ptr(), N, W, lg.data_ptr(), ws.ptr, need, _st()) == 0, _err()
    assert m.lib.crnn_backward(m.h, dt.data_ptr(), tt.data_ptr(), dl.data_ptr(), N, W, ws.ptr, need, _st()) == 0, _err()
    torch.cuda.synchronize()
    grads = m.slots[0]
    grads.set(grads.body.clone())
    step = {"adam": lambda: m.lib.crnn_clip_adam_step(m.h, 1e-3, 10.0, 1, 1.0, 1.0, _st()),
            "momentum": lambda: m.lib.crnn_clip_momentum_step(m.h, 1e-2, 0.9, 10.0, 1.0, 1.0, _st()),
            "rmsprop": lambda: m.lib.crnn_clip_rmsprop_step(m.h, 1e-2, 0.9, 0.0, 1e-10, 10.0, 1.0, 1.0, _st())}[solver]
    name = {"adam": "crnn_clip_adam_step", "momentum": "crnn_clip_momentum_step", "rmsprop": "crnn_clip_rmsprop_step"}[solver]
    _case([name], step, [m.params] + m.slots)
    costs = _inp("costs", rng.random(N).astype(np.float32))
    loss = _out("loss_out", (1,), torch.float32)
    _case(["crnn_total_loss"], lambda: _seq(m.changed, lambda: m.lib.crnn_total_loss(m.h, costs.ptr, N, loss.ptr, _st())),
          [costs, loss, m.params])


@pytest.mark.parametrize("u8", [False, True], ids=["f32", "u8"])
@pytest.mark.parametrize("chunks", [1, 4])
def test_host_fed_forward(chunks, u8):
    """crnn_forward_host (page-locked batch) and crnn_forward_pageable (the library's host threads fill the caller's
    page-locked staging): the host buffers and the device staging guarded."""
    sfx = "_u8" if u8 else ""
    N, W = 130, 160
    T = W // 4 - 1
    data, tsl, _ = _batch(N, W, u8, 4)
    dt = torch.uint8 if u8 else torch.float32
    t = _inp("time_step_len", tsl)
    m = Model()
    ws, need = m.ws(N, W)
    copy = torch.cuda.Stream()
    host = BD.Guarded("host_data", data.nbytes, kind="in", align=16, device="cpu", pinned=True, dtype=dt, shape=data.shape).set(data)
    stage = _out("data_staging", data.shape, dt, align=16)
    logits = _out("logits", (T, N, 64), torch.float32, align=16)
    fh = getattr(m.lib, "crnn_forward_host" + sfx)
    _case(["crnn_forward_host" + sfx],
          lambda: _seq(m.changed, lambda: fh(m.h, host.ptr, stage.ptr, t.ptr, N, W, logits.ptr, ws.ptr, need, chunks, _st(), copy.cuda_stream)),
          [host, stage, t, ws, logits] + m.bound())
    page = BD.Guarded("pageable_data", data.nbytes, kind="in", align=16, device="cpu", dtype=dt, shape=data.shape).set(data)
    pinned = BD.output_of("pinned_staging", data.shape, dt, device="cpu", align=16, pinned=True)
    fp = getattr(m.lib, "crnn_forward_pageable" + sfx)
    _case(["crnn_forward_pageable" + sfx],
          lambda: _seq(m.changed, lambda: fp(m.h, page.ptr, pinned.ptr, stage.ptr, t.ptr, N, W, logits.ptr, ws.ptr, need, chunks, 4, _st(),
                                             copy.cuda_stream)),
          [page, pinned, stage, t, ws, logits] + m.bound())


LINES_SHAPES = [(7, 1024), (130, 160), (1, 8)]


@pytest.mark.parametrize("moving", [0, 1], ids=["batch", "moving"])
@pytest.mark.parametrize("N,W", LINES_SHAPES, ids=[f"N{n}_W{w}" for n, w in LINES_SHAPES])
def test_forward_lines(N, W, moving):
    T = W // 4 - 1
    rng = np.random.default_rng(N + W)
    lw = (rng.integers(2, W // 4 + 1, size=N) * 4).astype(np.int32)
    lw[0] = W
    tsl = np.maximum(lw // 4 - 1, 0).astype(np.int32)
    tsl[-1] = 0
    m = Model()
    assert m.lib.crnn_model_set_bn_statistics(m.h, moving) == 0, _err()
    ws, need = m.ws(N, W, lines=True)
    w_, t_ = _inp("line_width", lw), _inp("time_step_len", tsl)
    logits = _out("logits", (T, N, 64), torch.float32, align=16)
    for u8 in (False, True):
        data, _, _ = _batch(N, W, u8, 7)
        d = _inp("data", data, align=16 if not u8 else 4)
        fn = m.lib.crnn_forward_lines_u8 if u8 else m.lib.crnn_forward_lines
        _case(["crnn_forward_lines" + ("_u8" if u8 else "")],
              lambda: _seq(m.changed, lambda: fn(m.h, d.ptr, w_.ptr, t_.ptr, N, W, logits.ptr, ws.ptr, need, _st())),
              [d, w_, t_, ws, logits] + m.bound())


@pytest.mark.parametrize("W", [8, 40, 516])
def test_fp8_and_f32_class_forwards(W):
    N = 3
    T = W // 4 - 1
    data, tsl, rng = _batch(N, W, False, W)
    d, d8, t = _inp("data", data, align=16), _inp("data", (data * 255).round().astype(np.uint8), align=4), _inp("time_step_len", tsl)
    logits = _out("logits", (T, N, 64), torch.float32, align=16)
    m = Model(dtype=4)
    ws, need = m.ws(N, W)
    _case(["crnn_model_calibrate_fp8_u8"], lambda: _seq(m.changed, lambda: m.lib.crnn_model_calibrate_fp8_u8(m.h, d8.ptr, t.ptr, N, W, ws.ptr,
                                                                                                          need, _st())),
          [d8, t, ws] + m.bound())
    calib = lambda: m.lib.crnn_model_calibrate_fp8(m.h, d.ptr, t.ptr, N, W, ws.ptr, need, _st())
    _case(["crnn_model_calibrate_fp8", "crnn_forward"],
          lambda: _seq(m.changed, calib, lambda: m.lib.crnn_forward(m.h, d.ptr, t.ptr, N, W, logits.ptr, ws.ptr, need, _st())),
          [d, t, ws, logits] + m.bound())
    lw = np.full(N, W, np.int32)
    lw[1:] = max(8, W // 2 // 4 * 4)
    lt = np.minimum(tsl, lw // 4 - 1).astype(np.int32)
    w_, t2 = _inp("line_width", lw), _inp("time_step_len", lt)
    wsl, needl = m.ws(N, W, lines=True)
    _case(["crnn_forward_lines"],
          lambda: _seq(m.changed, lambda: m.lib.crnn_model_calibrate_fp8(m.h, d.ptr, t.ptr, N, W, wsl.ptr, needl, _st()),
                       lambda: m.lib.crnn_forward_lines(m.h, d.ptr, w_.ptr, t2.ptr, N, W, logits.ptr, wsl.ptr, needl, _st())),
          [d, w_, t2, wsl, logits] + m.bound())
    del m, ws, wsl
    for dtype in (2, 3):
        m = Model(dtype=dtype)
        ws, need = m.ws(N, W)
        _case(["crnn_forward"], lambda: _seq(m.changed, lambda: m.lib.crnn_forward(m.h, d.ptr, t.ptr, N, W, logits.ptr, ws.ptr, need, _st())),
              [d, t, ws, logits] + m.bound())
        del m, ws


# ------------------------------------------------------------------------------------------------------- alignment rules
def _refused(call, outs, what):
    """`call` must return CRNN_INVALID_VALUE naming `what`, with every output body as it was."""
    before = [g.body.clone() for g in outs]
    torch.cuda.synchronize()
    st = call()
    torch.cuda.synchronize()
    assert st == INVALID and what in _err(), (st, _err(), what)
    assert all(torch.equal(g.body, b) for g, b in zip(outs, before)), what
    assert all(not g.problems() for g in outs), what


def _off(name, like, offset=4):
    """A device buffer shaped like `like`, `offset` bytes past a 16-byte aligned address."""
    return BD.Guarded(name, like.nbytes, kind="out", align=16, offset=offset, device=DEV, dtype=torch.uint8)


def test_misaligned_pointers_are_refused():
    lib = _lib()
    N, W = 3, 40
    T = W // 4 - 1
    data, tsl, _ = _batch(N, W, False, 1)
    d, t = _inp("data", data, align=16), _inp("time_step_len", tsl)
    d8 = _inp("data", (data * 255).astype(np.uint8), align=4)
    lw = _inp("line_width", np.full(N, W, np.int32))
    m = Model()
    ws, need = m.ws(N, W)
    wsl, needl = m.ws(N, W, lines=True)
    lg = _out("logits", (T, N, 64), torch.float32, align=16)
    lg_bad = _off("logits", lg.body)
    d_bad = _off("data", data)
    d_bad.body.copy_(d.body)
    outs = [lg, lg_bad, ws, wsl]
    st = _st()
    _refused(lambda: lib.crnn_forward(m.h, d_bad.ptr, t.ptr, N, W, lg.ptr, ws.ptr, need, st), outs, "forward: data must be 16-byte aligned")
    _refused(lambda: lib.crnn_forward(m.h, d.ptr, t.ptr, N, W, lg_bad.ptr, ws.ptr, need, st), outs,
             "forward: logits_out must be 16-byte aligned")
    _refused(lambda: lib.crnn_forward_u8(m.h, d8.ptr, t.ptr, N, W, lg_bad.ptr, ws.ptr, need, st), outs,
             "forward: logits_out must be 16-byte aligned")
    _refused(lambda: lib.crnn_forward_lines(m.h, d_bad.ptr, lw.ptr, t.ptr, N, W, lg.ptr, wsl.ptr, needl, st), outs,
             "forward: data must be 16-byte aligned")
    _refused(lambda: lib.crnn_forward_lines_u8(m.h, d8.ptr, lw.ptr, t.ptr, N, W, lg_bad.ptr, wsl.ptr, needl, st), outs,
             "forward: logits_out must be 16-byte aligned")
    host = BD.Guarded("host_data", data.nbytes, kind="in", align=16, device="cpu", pinned=True, dtype=torch.float32).set(data)
    copy = torch.cuda.Stream()
    stage_bad = _off("data_staging", data)
    for chunks in (1, 4):
        _refused(lambda: lib.crnn_forward_host(m.h, host.ptr, stage_bad.ptr, t.ptr, N, W, lg.ptr, ws.ptr, need, chunks, st,
                                               copy.cuda_stream), outs + [stage_bad], "forward: data_staging must be 16-byte aligned")
        _refused(lambda: lib.crnn_forward_pageable(m.h, host.ptr, host.ptr, stage_bad.ptr, t.ptr, N, W, lg.ptr, ws.ptr, need, chunks, 2, st,
                                                   copy.cuda_stream), outs + [stage_bad], "forward: data_staging must be 16-byte aligned")
    # uint8 host feeds: the f32 logits rule applies to them too
    h8 = BD.Guarded("host_data", data.size, kind="in", align=16, device="cpu", pinned=True).set((data * 255).astype(np.uint8))
    s8 = _out("data_staging", (data.size,), torch.uint8, align=16)
    _refused(lambda: lib.crnn_forward_host_u8(m.h, h8.ptr, s8.ptr, t.ptr, N, W, lg_bad.ptr, ws.ptr, need, 1, st, copy.cuda_stream),
             outs + [s8], "forward: logits_out must be 16-byte aligned")
    # the bind rules; a refused bind keeps the previous binding (the forward after it still runs)
    n = m.e.total
    p_bad = BD.Guarded("params", 4 * n, kind="out", align=16, offset=4, device=DEV)
    for k in range(4):
        ptrs = [m.params.ptr] + [s.ptr for s in m.slots]
        ptrs[k] = p_bad.ptr
        name = ("params", "grads", "adam_m", "adam_v")[k]
        _refused(lambda: lib.crnn_model_bind(m.h, *ptrs), [p_bad], f"model_bind: {name} must be 16-byte aligned")
    mv_bad = BD.Guarded("bn_moving", 4096, kind="out", align=16, offset=2, device=DEV)
    _refused(lambda: lib.crnn_model_bind_bn_moving(m.h, mv_bad.ptr, 0.9), [mv_bad], "bind_bn_moving: moving must be 4-byte aligned")
    assert lib.crnn_forward(m.h, d.ptr, t.ptr, N, W, lg.ptr, ws.ptr, need, st) == 0, _err()
    torch.cuda.synchronize()
    assert not m.params.problems() and not m.moving.problems()
    # fp8 calibration
    m8 = Model(dtype=4)
    _refused(lambda: lib.crnn_model_calibrate_fp8(m8.h, d_bad.ptr, t.ptr, N, W, ws.ptr, need, st), outs,
             "forward: data must be 16-byte aligned")
    # the backward: after a real training forward, data and dlogits
    mt = Model(training=True)
    wst, needt = mt.ws(N, W, train=True)
    assert lib.crnn_forward(mt.h, d.ptr, t.ptr, N, W, lg.ptr, wst.ptr, needt, st) == 0, _err()
    torch.cuda.synchronize()
    dl = _inp("dlogits", np.zeros((T, N, 64), np.float32), align=16)
    dl_bad = _off("dlogits", dl.body)
    dl_bad.body.zero_()
    grads = mt.slots[0]
    g0 = grads.body.clone()
    _refused(lambda: lib.crnn_backward(mt.h, d_bad.ptr, t.ptr, dl.ptr, N, W, wst.ptr, needt, st), [grads], "backward: data must be 16-byte aligned")
    _refused(lambda: lib.crnn_backward(mt.h, d.ptr, t.ptr, dl_bad.ptr, N, W, wst.ptr, needt, st), [grads],
             "backward: dlogits must be 16-byte aligned")
    _refused(lambda: lib.crnn_backward_u8(mt.h, d8.ptr, t.ptr, dl_bad.ptr, N, W, wst.ptr, needt, st), [grads],
             "backward: dlogits must be 16-byte aligned")
    assert torch.equal(grads.body, g0)
    _REPORT["entry_points"].update(["alignment: forward, forward_u8, forward_lines(_u8), forward_host(_u8), forward_pageable, "
                                    "calibrate_fp8, backward(_u8), model_bind, bind_bn_moving"])
