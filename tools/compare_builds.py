"""Outputs of two builds of the library on the same seeded inputs, each build run in a process of its own.

    python tools/compare_builds.py OLD_TREE NEW_TREE [--out DIR]

OLD_TREE and NEW_TREE are source trees with a built lstm_ctc_ocr_b200/libcrnnctc.so.  OLD runs three times and NEW twice, on
  train  1024 x 256, training mode: forward, backward with a seeded d logits, every gradient
  infer  1024 x 256, inference mode
  lines  64 x 256 packed lines (crnn_forward_lines), line widths 8 .. 256
  fp8    256 x 256 fp8 model (compute_dtype 4), calibrated on the batch itself, and its scales
and, at 256 x 256 in inference mode, every other way into the forward:
  u8                  uint8 pixels (crnn_forward_u8)
  host1, host4        page-locked host memory, one and four image ranges (crnn_forward_host)
  pageable            ordinary host memory in four ranges (crnn_forward_pageable)
  fp8_lines           packed lines on the fp8 model
  bf16_moving, fp8_moving, bf16_moving_lines, fp8_moving_lines
                      moving BatchNorm statistics, whole batch and packed lines (fp8: scales calibrated in moving mode)
Quantities computed before the first f64 BatchNorm atomics (conv1 .. conv3_2, the pool arg-max bytes, conv4_1's pre-BN
output) must be bit-identical between OLD and NEW.  Everything downstream may differ from OLD by no more than OLD differs from
itself between its runs (the order of the f64 BatchNorm atomics and of the f32 split-K / column-sum atomics of the weight
gradients changes the last bits from run to run).  Prints one JSON line; exit status 1 on a
violation.
"""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

BIT_EXACT = ("conv1", "conv2", "conv3_1", "conv3_2", "a4a_pre", "am1", "am2", "am3")


def _dump(tree, out):
    """Child process: run every case with the library of `tree`, write the outputs to `out` (torch.save)."""
    sys.path.insert(0, tree)
    from lstm_ctc_ocr_b200 import engine
    from oracle import crnn_oracle as O
    dev = torch.device("cuda:0")
    t = lambda a: torch.tensor(a, device=dev)
    pn = O.randomize_params(O.init_params(3, dtype=np.float32, logits_scale=10.0))
    res = {}

    def keep(key, x):
        x = x.detach()
        res[key] = x.to(torch.bfloat16).cpu() if x.dtype == torch.float32 and key.split("/")[1] in TAPS_BF16 else x.cpu()

    TAPS_BF16 = ("conv1", "conv2", "conv3_1", "conv3_2", "a4a_pre", "conv4_1", "a4b_pre", "conv4_2", "conv5", "xproj", "lstm_out",
                 "d_lstm_out", "d_a5", "d_pre4a", "d_a2", "d_a1")
    N, W = 1024, 256
    data, _, _, tsl = O.synth_batch(N, W, seed=11)
    for mode in ("train", "infer"):
        m = engine.CrnnModel(device=dev)
        m.load_params(pn)
        m.set_training(mode == "train")
        logits = m.forward(t(data), t(tsl))
        torch.cuda.synchronize()
        keep(f"{mode}/logits", logits)
        for k in ("conv1", "conv2", "conv3_1", "conv3_2", "a4a_pre", "conv4_1", "a4b_pre", "conv4_2", "conv5", "xproj", "lstm_out"):
            keep(f"{mode}/{k}", m.tap(k, N, W))
        for k in ("stats", "bn") + (("am1", "am2", "am3") if mode == "train" else ()):
            keep(f"{mode}/{k}", m.tap_raw(k, N, W))
        if mode == "train":
            gen = torch.Generator(device="cpu").manual_seed(17)
            dlogits = (torch.randn(logits.shape, generator=gen) * 0.05).float().to(dev)
            m.backward(t(data), t(tsl), dlogits)
            torch.cuda.synchronize()
            for k in ("d_lstm_out", "d_a5", "d_pre4a", "d_a2", "d_a1"):
                keep(f"{mode}/{k}", m.tap(k, N, W))
            for k in m.table:
                keep(f"{mode}/grad:{k}", m.grad_tensor(k))
        del m
        torch.cuda.empty_cache()
    # packed lines
    N = 64
    lw = np.random.default_rng(4).integers(2, W // 4 + 1, size=N).astype(np.int32) * 4
    data, _, _, tsl = O.synth_batch(N, W, seed=13, widths=[int(w) for w in lw])
    tsl = np.minimum(tsl, lw // 4 - 1).astype(np.int32)
    m = engine.CrnnModel(device=dev)
    m.load_params(pn)
    keep("lines/logits", m.forward_lines(t(data), t(lw), t(tsl)))
    for k in ("conv1", "conv2", "conv3_1", "conv3_2", "a4a_pre", "conv4_1", "conv4_2", "lstm_out"):
        keep(f"lines/{k}", m.tap(k, N, W))
    for k in ("stats", "bn"):
        keep(f"lines/{k}", m.tap_raw(k, N, W, lines=True))
    del m
    # fp8
    N = 256
    data, _, _, tsl = O.synth_batch(N, W, seed=14)
    m = engine.CrnnModel(device=dev, compute_dtype="fp8")
    m.load_params(pn)
    m.calibrate_fp8(t(data), t(tsl))
    keep("fp8/logits", m.forward(t(data), t(tsl)))
    keep("fp8/scales", torch.tensor(m.fp8_scales()))
    for k in ("conv1", "conv2", "conv3_1", "conv3_2", "a4a_pre", "conv4_1", "conv4_2", "lstm_out"):
        keep(f"fp8/{k}", m.tap(k, N, W))
    for k in ("stats", "bn"):
        keep(f"fp8/{k}", m.tap_raw(k, N, W))
    del m

    FWD = ("conv1", "conv2", "conv3_1", "conv3_2", "conv4_1", "conv4_2", "lstm_out")
    rng = np.random.default_rng(7)
    moving = {}
    for i, k in enumerate(engine.BN_MOVING_KEYS):       # [layer][mean, variance]
        moving[k] = rng.normal(0.0, 0.05, 512).astype(np.float32) if i % 2 == 0 else rng.uniform(0.002, 0.02, 512).astype(np.float32)

    def model(dtype="bf16", use_moving=False, cal=None):
        m = engine.CrnnModel(device=dev, compute_dtype=dtype)
        m.load_params(pn)
        if use_moving:
            m.load_bn_moving(moving)
            m.set_bn_statistics("moving")
        if cal is not None:
            m.calibrate_fp8(*cal)
            keep(f"{dtype}{'_moving' if use_moving else ''}_cal/scales", torch.tensor(m.fp8_scales()))
        return m

    def case(name, m, logits, N, W, taps=FWD + ("a4a_pre",), raw=("stats", "bn"), lines=False):
        torch.cuda.synchronize()
        keep(f"{name}/logits", logits)
        for k in taps:
            keep(f"{name}/{k}", m.tap(k, N, W))
        for k in raw:
            keep(f"{name}/{k}", m.tap_raw(k, N, W, lines=lines))

    N = 256
    data, _, _, tsl = O.synth_batch(N, W, seed=15)
    cal = (t(data), t(tsl))
    u8 = np.random.default_rng(15).integers(0, 256, size=data.shape, dtype=np.uint8)
    m = model()
    case("u8", m, m.forward(t(u8), t(tsl)), N, W)
    pin = torch.empty(data.shape, dtype=torch.float32).pin_memory()
    pin.numpy()[...] = data
    for chunks in (1, 4):
        m = model()
        case(f"host{chunks}", m, m.forward_host(pin.numpy(), t(tsl), chunks=chunks)[0], N, W)
    m = model()
    staging = torch.empty(data.size, dtype=torch.float32).pin_memory()
    case("pageable", m, m.forward_pageable(data.copy(), staging, t(tsl), chunks=4, host_threads=4)[0], N, W)
    lw = np.random.default_rng(5).integers(2, W // 4 + 1, size=N).astype(np.int32) * 4
    ldata, _, _, ltsl = O.synth_batch(N, W, seed=16, widths=[int(w) for w in lw])
    ltsl = np.minimum(ltsl, lw // 4 - 1).astype(np.int32)
    m = model("fp8", cal=cal)
    case("fp8_lines", m, m.forward_lines(t(ldata), t(lw), t(ltsl)), N, W, lines=True)
    for dtype in ("bf16", "fp8"):
        m = model(dtype, use_moving=True, cal=cal if dtype == "fp8" else None)
        case(f"{dtype}_moving", m, m.forward(t(data), t(tsl)), N, W, taps=FWD, raw=())
        case(f"{dtype}_moving_lines", m, m.forward_lines(t(ldata), t(lw), t(ltsl)), N, W, taps=FWD, raw=())
    del m
    torch.cuda.synchronize()
    torch.save(res, out)


def _maxdiff(a, b):
    if a.dtype == torch.uint8:
        return float((a != b).sum())
    return float((a - b).abs().max()) if a.numel() else 0.0


def main():
    if sys.argv[1] == "--dump":
        _dump(sys.argv[2], sys.argv[3])
        return 0
    old, new = os.path.abspath(sys.argv[1]), os.path.abspath(sys.argv[2])
    out_dir = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else tempfile.mkdtemp()
    runs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, tree in (("old0", old), ("new0", new), ("old1", old), ("new1", new), ("old2", old)):
            path = os.path.join(tmp, name + ".pt")
            subprocess.check_call([sys.executable, os.path.abspath(__file__), "--dump", tree, path], cwd=tree)
            runs[name] = torch.load(path)
            print(f"{name}: {len(runs[name])} quantities", flush=True)
    olds = [runs[f"old{i}"] for i in range(3)]
    news = [runs[f"new{i}"] for i in range(2)]
    report, bad = {}, []
    dev = torch.device("cuda:0")           # the taps of a 1024-image batch take minutes to compare on the host
    for k in sorted(olds[0]):
        exact = k.split("/")[1] in BIT_EXACT
        o = [(x[k].float() if x[k].dtype == torch.bfloat16 else x[k]).to(dev).contiguous() for x in olds]
        n = [(x[k].float() if x[k].dtype == torch.bfloat16 else x[k]).to(dev).contiguous() for x in news]
        ident = all(torch.equal(x.view(torch.uint8), o[0].view(torch.uint8)) for x in n)
        d_new = max(_maxdiff(a, b) for a in o for b in n)
        d_self = max(_maxdiff(o[i], o[j]) for i in range(3) for j in range(i + 1, 3))
        report[k] = {"bit_identical": ident, "maxdiff_new_vs_old": d_new, "maxdiff_old_vs_old": d_self}
        if (exact and not ident) or d_new > d_self:
            bad.append(k)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "compare_builds.json"), "w") as f:
        json.dump(report, f, indent=1)
    n_ident = sum(r["bit_identical"] for r in report.values())
    print(json.dumps({"quantities": len(report), "bit_identical": n_ident, "violations": bad}))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
