"""PNG text lines decoded on the device (crnn_png_decode_gray_u8, the `images` feed's PNG entries) against the host readers.

Renders LINES text lines of 30 - 70 characters at their native 60 rows with gen.render_line from a fixed seed (resize_bench's
set), saves them as 8-bit gray PNG with Pillow (as genImg does) and, with the decode-10k fixture's trained weights, reports per
round (the paths alternate within each round):
  - CUDA-event time of the device decode of the whole directory and of one width-sorted batch of 64 and of 256 lines, bytes in
    and out, beside forward_lines + greedy decode of the same batch;
  - host decode of the whole directory: cv2.imdecode per file on one thread, and on a pool of os.cpu_count() threads;
  - test_model wall time: this build (PNG bytes fed, decoded on the device) against the host path (load_line_image per file,
    then the `images` feed of arrays);
  - the decoded bytes of every path compared, and the reads of the two test_model paths;
  - which stage bounds the kernel: the batch of 64 re-encoded (tests/png_refs.py) with filter None or Paeth on every row and
    zlib level 0 (stored blocks: no Huffman decode) or 6, each variant's decode time beside Pillow's own files.
The card's name and power limit are read in the same run.

    python tools/png_bench.py [--lines 2048] [--rounds 3]"""
import argparse
import concurrent.futures
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
        raise SystemExit("png_bench measures the GPU: no CUDA device")
    os.environ["CRNN_FONT"] = "default"
    gen._FONT_CACHE.clear()
    spec = importlib.util.spec_from_file_location("make_decode10k", os.path.join(ROOT, "tests", "golden", "make_decode10k.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    rng = random.Random(2024)
    texts = [gen.gen_rand(rng, 30, 70) for _ in range(args.lines)]
    images = [gen.render_line(t, rng=rng) for t in texts]
    files = []
    for im in images:
        b = io.BytesIO()
        Image.fromarray(im).save(b, "PNG")
        files.append(b.getvalue())
    widths = [T.line_size(*im.shape)[1] for im in images]
    order = sorted(range(len(images)), key=lambda i: widths[i])
    cfg.TEST.BATCH_SIZE = 64
    net = get_network("LSTM_test")
    dev = torch.device("cuda:0")
    rule = T.gray_rule()

    def device_args(idx):
        fs = [files[i] for i in idx]
        hw = np.array([images[i].shape for i in idx], np.int64)
        flen = np.array([len(f) for f in fs], np.int64)
        foff = np.concatenate([[0], np.cumsum(flen)[:-1]]).astype(np.int64)
        ooff = np.concatenate([[0], np.cumsum(hw[:, 0] * hw[:, 1])[:-1]]).astype(np.int64)
        ws_offset, ws_bytes = engine.png_plan(np.stack([np.frombuffer(f, np.uint8, 13, 16) for f in fs]), flen)
        t = lambda a: torch.tensor(np.ascontiguousarray(a), device=dev)  # noqa: E731
        a = (t(np.frombuffer(b"".join(fs), np.uint8)), t(foff), t(flen), t(hw[:, 0].astype(np.int32)), t(hw[:, 1].astype(np.int32)),
             t(ooff), t(ws_offset))
        out = torch.empty(int((hw[:, 0] * hw[:, 1]).sum()), dtype=torch.uint8, device=dev)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        st = torch.empty(len(idx), dtype=torch.int32, device=dev)
        return (lambda: engine.decode_png_gray(*a, rule, out=out, workspace=ws, status=st)), out, st, ooff, int(flen.sum())

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

    def host_read(f):
        return cv2.imdecode(np.frombuffer(f, np.uint8), 0)

    out = dict(lines=args.lines, rounds=args.rounds, rule=rule, width_min=min(widths), width_max=max(widths),
               encoded_bytes=sum(len(f) for f in files), decoded_bytes=sum(im.size for im in images))
    with Session() as sess, tempfile.TemporaryDirectory() as tmp:
        sess.assign(net, mk.load_weights())
        eng = sess.engine_for(net)
        for i, (t, f) in enumerate(zip(texts, files)):
            with open(os.path.join(tmp, f"{i:05d}_{t}.png"), "wb") as fh:
                fh.write(f)
        sw = T.SolverWrapper.__new__(T.SolverWrapper)
        sw.net, sw.pretrained_model, sw.output_dir = net, None, tmp
        fetch = Fetch(net, "dense_decoded")

        def host_test_model():
            names = sorted(os.listdir(tmp))
            ims = [T.load_line_image(os.path.join(tmp, n)) for n in names]
            order_ = sorted(range(len(names)), key=lambda i: T.line_size(*ims[i].shape)[1])
            got = {}
            for b0 in range(0, len(order_), 64):
                idx = order_[b0:b0 + 64]
                res = sess.run(fetch, {net.images: [ims[i] for i in idx]})
                for r, i in enumerate(idx):
                    got[i] = "".join(T.decodeRes(res[r]))
            return [got[i] for i in range(len(names))]

        # device-only rows: the whole directory, and the middle width-sorted batches of 64 and 256 beside their forward + decode
        rows = {}
        for name, idx in (("all", list(range(args.lines))), ("batch64", order[len(order) // 2 - 32: len(order) // 2 + 32]),
                          ("batch256", order[len(order) // 2 - 128: len(order) // 2 + 128])):
            fn, dout, st, ooff, nin = device_args(idx)
            times = [events(fn, args.reps if name != "all" else max(args.reps // 4, 3)) for _ in range(args.rounds)]
            row = dict(files=len(idx), bytes_in=nin, bytes_out=int(dout.numel()), decode_us=_spread(times))
            o = dout.cpu().numpy()
            row["status_nonzero"] = int(st.cpu().numpy().astype(bool).sum())
            row["equal_to_cv2"] = sum(np.array_equal(o[ooff[r]:ooff[r] + images[i].size], host_read(files[i]).reshape(-1))
                                      for r, i in enumerate(idx))
            if name != "all":
                ims = [images[i] for i in idx]
                sz = np.array([T.line_size(*im.shape) for im in ims], np.int32)
                nb = np.array([im.size for im in ims], np.int64)
                off = np.concatenate([[0], np.cumsum(nb)[:-1]]).astype(np.int64)
                t = lambda a: torch.tensor(np.ascontiguousarray(a), device=dev)  # noqa: E731
                data = engine.resize_lines_u8(t(np.concatenate([im.reshape(-1) for im in ims])), t(off), t([im.shape[0] for im in ims]).int(),
                                              t([im.shape[1] for im in ims]).int(), t(sz[:, 0]), int(sz[:, 1].max()),
                                              max(im.shape[0] for im in ims))
                lw, tsl = t(sz[:, 1]), t(sz[:, 2])
                fd = lambda: engine.ctc_greedy(eng.forward_lines(data, lw, tsl), tsl)  # noqa: E731
                row["forward_decode_us"] = _spread([events(fd, max(args.reps // 2, 5)) for _ in range(args.rounds)])
            rows[name] = row
        out["device"] = rows
        # stage variants of the batch of 64: (filter, zlib level) -> decode time; None + 0 leaves the chunk walk, copies and
        # conversion, + 6 adds the Huffman decode, Paeth + 0 adds the serial unfilter
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import png_refs as PR
        mid = order[len(order) // 2 - 32: len(order) // 2 + 32]
        saved = {i: files[i] for i in mid}
        stages = {}
        for filt, level in ((0, 0), (0, 6), (4, 0), (4, 6)):
            for i in mid:
                files[i] = PR.write_png(images[i], 8, 0, filters=filt, level=level)
            fn, dout, st, ooff, nin = device_args(mid)
            fn()
            o = dout.cpu().numpy()
            stages[f"filter{filt}_zlib{level}"] = dict(
                bytes_in=nin, decode_us=_spread([events(fn, args.reps) for _ in range(args.rounds)]),
                equal_to_cv2=sum(np.array_equal(o[ooff[r]:ooff[r] + images[i].size], host_read(files[i]).reshape(-1))
                                 for r, i in enumerate(mid)),
                status_nonzero=int(st.cpu().numpy().astype(bool).sum()))
        for i, f in saved.items():
            files[i] = f
        out["stages_batch64"] = stages
        # host decode of the directory's bytes: one thread and a pool of os.cpu_count() threads; test_model both ways
        one, pool, tm_dev, tm_host = [], [], [], []
        reads_equal = None
        with concurrent.futures.ThreadPoolExecutor(os.cpu_count()) as ex:
            with open(os.devnull, "w") as null, contextlib.redirect_stdout(null):
                sw.test_model(sess, testDir=tmp, restore=False)
                host_test_model()
            for _ in range(args.rounds):
                t0 = time.perf_counter()
                a = [host_read(f) for f in files]
                one.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                b = list(ex.map(host_read, files))
                pool.append(time.perf_counter() - t0)
                assert all(np.array_equal(x, y) for x, y in zip(a, b))
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
        out["host_decode_s"] = {"one_thread": _spread(one), f"pool_{os.cpu_count()}_threads": _spread(pool)}
        out["test_model_s"] = {"device_png": _spread(tm_dev), "host_path": _spread(tm_host)}
        out["test_model_reads_equal"] = reads_equal
    name, limit = _card()
    out = dict(card=name, power_limit=limit, host_cpus=os.cpu_count(), **out)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
