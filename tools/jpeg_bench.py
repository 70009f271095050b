"""JPEG text lines decoded on the device (crnn_jpeg_decode_gray_u8, the `images` feed's JPEG entries) against the host path.

Renders LINES text lines of 30 - 70 characters at their native 60 rows with gen.render_line from a fixed seed (resize_bench's
set) and saves them twice: as gray JPEG by cv2.imwrite (quality 95) and as 4:2:0 colour JPEG by Pillow (quality 75).  With the
decode-10k fixture's trained weights it reports, per set:
  - CUDA-event time of the device decode of the whole directory and of the middle width-sorted batches of 64 and 256 lines,
    bytes in and out, beside forward_lines + greedy decode of the same batch;
  - test_model wall time, this build (JPEG bytes fed, decoded on the device) against the host path (load_line_image per file,
    then the `images` feed of arrays), alternating within each round;
  - the device decodes compared with the host reader, and the reads of the two test_model paths.
It also times one file 60 x 65500 (the widest libjpeg writes) without restart markers, which a single thread decodes, and
the same file with a restart marker every 64 MCUs.  The card's name and power limit are
read in the same run.

With --stages it reports instead which kernel bounds the batch decode and how the decode of the batch of 64 changes with
restart markers (`stages`).

    python tools/jpeg_bench.py [--lines 2048] [--rounds 3] [--stages]"""
import argparse
import contextlib
import importlib.util
import io
import json
import os
import random
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from resize_bench import _card, _spread  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lines", type=int, default=2048)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20, help="timed repetitions of each device-only measurement")
    ap.add_argument("--stages", action="store_true", help="instead: which kernel bounds the batch decode (torch.profiler), and the "
                    "middle batch of 64 gray lines re-encoded with restart intervals of 1 .. 16 MCUs (CUDA events)")
    args = ap.parse_args()
    import cv2
    import torch
    from PIL import Image
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.lstm import test as T
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.session import Session
    if not torch.cuda.is_available():
        raise SystemExit("jpeg_bench measures the GPU: no CUDA device")
    os.environ["CRNN_FONT"] = "default"
    gen._FONT_CACHE.clear()
    spec = importlib.util.spec_from_file_location("make_decode10k", os.path.join(ROOT, "tests", "golden", "make_decode10k.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    rng = random.Random(2024)
    texts = [gen.gen_rand(rng, 30, 70) for _ in range(args.lines)]
    images = [gen.render_line(t, rng=rng) for t in texts]

    def pil_420(im):
        b = io.BytesIO()
        Image.fromarray(np.stack([im, im, im // 2 + 64], -1)).save(b, "JPEG", quality=75, subsampling=2)
        return b.getvalue()

    sets = {"cv2_gray_q95": [cv2.imencode(".jpg", im, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes() for im in images],
            "pil_420_q75": [pil_420(im) for im in images]}
    widths = [T.line_size(*im.shape)[1] for im in images]
    order = sorted(range(len(images)), key=lambda i: widths[i])
    cfg.TEST.BATCH_SIZE = 64
    net = get_network("LSTM_test")
    dev = torch.device("cuda:0")
    rule = T.gray_rule()

    def host_read(f):
        return cv2.imdecode(np.frombuffer(f, np.uint8), 0) if rule == 0 else np.asarray(Image.open(io.BytesIO(f)).convert("L"))

    def device_args(fs):
        hw = np.array([engine.jpeg_size(f) for f in fs], np.int64)
        flen = np.array([len(f) for f in fs], np.int64)
        foff = np.concatenate([[0], np.cumsum(flen)[:-1]]).astype(np.int64)
        ooff = np.concatenate([[0], np.cumsum(hw[:, 0] * hw[:, 1])[:-1]]).astype(np.int64)
        ws_offset, ws_bytes = engine.jpeg_plan(engine.jpeg_sof_records(fs), flen, rule)
        t = lambda a: torch.tensor(np.ascontiguousarray(a), device=dev)  # noqa: E731
        a = (t(np.frombuffer(b"".join(fs), np.uint8)), t(foff), t(flen), t(hw[:, 0].astype(np.int32)), t(hw[:, 1].astype(np.int32)),
             t(ooff), t(ws_offset))
        out = torch.empty(int((hw[:, 0] * hw[:, 1]).sum()), dtype=torch.uint8, device=dev)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        st = torch.empty(len(fs), dtype=torch.int32, device=dev)
        return (lambda: engine.decode_jpeg_gray(*a, rule, out=out, workspace=ws, status=st)), out, st, ooff, hw, int(flen.sum())

    def events(fn, reps):
        fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / reps * 1e3          # us per call

    def equal(fs, dout, ooff, hw):
        o = dout.cpu().numpy()
        return sum(np.array_equal(o[ooff[r]:ooff[r] + hw[r, 0] * hw[r, 1]].reshape(hw[r]), host_read(f)) for r, f in enumerate(fs))

    out = dict(lines=args.lines, rounds=args.rounds, rule=rule, width_min=min(widths), width_max=max(widths))
    if args.stages:
        out.update(stages(args, sets, images, order, device_args, events, equal))
        name, limit = _card()
        print(json.dumps(dict(card=name, power_limit=limit, **out)), flush=True)
        return
    with Session() as sess:
        sess.assign(net, mk.load_weights())
        eng = sess.engine_for(net)
        fetch = Fetch(net, "dense_decoded")
        for set_name, files in sets.items():
            res = dict(encoded_bytes=sum(len(f) for f in files), decoded_bytes=sum(im.size for im in images))
            rows = {}
            for name, idx in (("all", list(range(args.lines))), ("batch64", order[len(order) // 2 - 32: len(order) // 2 + 32]),
                              ("batch256", order[len(order) // 2 - 128: len(order) // 2 + 128])):
                fs = [files[i] for i in idx]
                fn, dout, st, ooff, hw, nin = device_args(fs)
                times = [events(fn, args.reps if name != "all" else max(args.reps // 4, 3)) for _ in range(args.rounds)]
                row = dict(files=len(idx), bytes_in=nin, bytes_out=int(dout.numel()), decode_us=_spread(times),
                           status_nonzero=int(st.cpu().numpy().astype(bool).sum()), equal_to_host=equal(fs, dout, ooff, hw))
                if name != "all":
                    ims = [images[i] for i in idx]
                    sz = np.array([T.line_size(*im.shape) for im in ims], np.int32)
                    nb = np.array([im.size for im in ims], np.int64)
                    off = np.concatenate([[0], np.cumsum(nb)[:-1]]).astype(np.int64)
                    t = lambda a: torch.tensor(np.ascontiguousarray(a), device=dev)  # noqa: E731
                    data = engine.resize_lines_u8(t(np.concatenate([im.reshape(-1) for im in ims])), t(off),
                                                  t([im.shape[0] for im in ims]).int(), t([im.shape[1] for im in ims]).int(),
                                                  t(sz[:, 0]), int(sz[:, 1].max()), max(im.shape[0] for im in ims))
                    lw, tsl = t(sz[:, 1]), t(sz[:, 2])
                    fd = lambda: engine.ctc_greedy(eng.forward_lines(data, lw, tsl), tsl)  # noqa: E731
                    row["forward_decode_us"] = _spread([events(fd, max(args.reps // 2, 5)) for _ in range(args.rounds)])
                rows[name] = row
            res["device"] = rows
            with tempfile.TemporaryDirectory() as tmp:
                for i, (t_, f) in enumerate(zip(texts, files)):
                    with open(os.path.join(tmp, f"{i:05d}_{t_}.jpg"), "wb") as fh:
                        fh.write(f)
                sw = T.SolverWrapper.__new__(T.SolverWrapper)
                sw.net, sw.pretrained_model, sw.output_dir = net, None, tmp

                def host_test_model():
                    names = sorted(os.listdir(tmp))
                    ims = [T.load_line_image(os.path.join(tmp, n)) for n in names]
                    order_ = sorted(range(len(names)), key=lambda i: T.line_size(*ims[i].shape)[1])
                    got = {}
                    for b0 in range(0, len(order_), 64):
                        idx = order_[b0:b0 + 64]
                        r_ = sess.run(fetch, {net.images: [ims[i] for i in idx]})
                        for r, i in enumerate(idx):
                            got[i] = "".join(T.decodeRes(r_[r]))
                    return [got[i] for i in range(len(names))]

                tm_dev, tm_host, reads_equal = [], [], None
                with open(os.devnull, "w") as null, contextlib.redirect_stdout(null):
                    sw.test_model(sess, testDir=tmp, restore=False)
                    host_test_model()
                for _ in range(args.rounds):
                    buf = io.StringIO()
                    with contextlib.redirect_stdout(buf):
                        t0 = time.perf_counter()
                        sw.test_model(sess, testDir=tmp, restore=False)
                        tm_dev.append(time.perf_counter() - t0)
                    with open(os.devnull, "w") as null, contextlib.redirect_stdout(null):
                        t0 = time.perf_counter()
                        host_reads = host_test_model()
                        tm_host.append(time.perf_counter() - t0)
                    dev_reads = [ln.split("res: ", 1)[1] for ln in buf.getvalue().splitlines() if ln.startswith("    res: ")]
                    reads_equal = f"{sum(x == y for x, y in zip(dev_reads, host_reads))}/{len(host_reads)}"
            res["test_model_s"] = {"device_jpeg": _spread(tm_dev), "host_path": _spread(tm_host)}
            res["test_model_reads_equal"] = reads_equal
            out[set_name] = res
        # the widest file the decoder takes, without restart markers: one thread decodes all of it
        wide = np.tile(np.concatenate(images[:8], 1), (1, 64))[:, :65500]
        f = cv2.imencode(".jpg", wide, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes()
        fn, dout, st, ooff, hw, nin = device_args([f])
        out["widest_60x65500_no_restart"] = dict(bytes_in=nin, decode_us=_spread([events(fn, 3) for _ in range(args.rounds)]),
                                                 equal_to_host=equal([f], dout, ooff, hw))
        fr = cv2.imencode(".jpg", wide, [cv2.IMWRITE_JPEG_QUALITY, 95, cv2.IMWRITE_JPEG_RST_INTERVAL, 64])[1].tobytes()
        fn, dout, st, ooff, hw, nin = device_args([fr])
        out["widest_60x65500_restart_64"] = dict(bytes_in=nin, decode_us=_spread([events(fn, 3) for _ in range(args.rounds)]),
                                                 equal_to_host=equal([fr], dout, ooff, hw))
    name, limit = _card()
    out = dict(card=name, power_limit=limit, host_cpus=os.cpu_count(), **out)
    print(json.dumps(out), flush=True)


def stages(args, sets, images, order, device_args, events, equal):
    """Per-kernel CUDA time of the middle batches' decode, from torch.profiler in a run of its own, and the middle batch of 64
    gray lines re-encoded by cv2 (quality 95) with a restart marker every 1, 4 or 16 MCUs: the entropy kernel decodes a file's
    restart segments on 32 lanes at once, so these times show how much of the decode is its serial Huffman walk."""
    import cv2
    import torch
    from torch.profiler import ProfilerActivity, profile
    res = {}
    for set_name, files in sets.items():
        for name, n in (("batch64", 32), ("batch256", 128)):
            fs = [files[i] for i in order[len(order) // 2 - n: len(order) // 2 + n]]
            fn = device_args(fs)[0]
            fn()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    fn()
                torch.cuda.synchronize()
            k = {}
            for e in prof.key_averages():
                if "jpeg_" in e.key:
                    k[e.key.split("jpeg_", 1)[1].split("(", 1)[0].split("<", 1)[0]] = round(e.device_time_total / args.reps, 1)
            res[f"{set_name}_{name}_kernel_us"] = k
    mid = order[len(order) // 2 - 32: len(order) // 2 + 32]
    for ri in (0, 16, 4, 1):
        fs = [cv2.imencode(".jpg", images[i], [cv2.IMWRITE_JPEG_QUALITY, 95, cv2.IMWRITE_JPEG_RST_INTERVAL, ri])[1].tobytes() for i in mid]
        fn, dout, st, ooff, hw, nin = device_args(fs)
        res[f"cv2_gray_q95_batch64_restart{ri}"] = dict(bytes_in=nin, decode_us=_spread([events(fn, args.reps) for _ in range(args.rounds)]),
                                                        equal_to_host=equal(fs, dout, ooff, hw))
    return res


if __name__ == "__main__":
    main()
