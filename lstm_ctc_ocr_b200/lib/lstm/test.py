"""Evaluation solver with the reference's surface (lib/lstm/test.py): ``SolverWrapper.test_model(sess, testDir, restore)`` and
``test_net(network, imgdb, testDir, output_dir, log_dir, pretrained_model, restore)``.

Per file (test.py:57-88): read as gray, right-pad the width to a multiple of POOL_SCALE with 0, /255, transpose to
[1, W, 32], decode, map ids -> chars, exact match against the label encoded in the file name (``<idx>_<chars>.png``).
Deviation from the reference, per SURVEY §3.4: ``time_step_len`` is fed as W//4 - 1 (the data layer's convention,
gen.py:54), not the off-by-one W//4 of test.py:74 which exceeds the number of conv frames.

Lines are evaluated in packed batches of ``cfg.TEST.BATCH_SIZE`` (the ``images`` feed: each batch's lines travel at their native
size and crnn_resize_lines_u8 resizes and packs them on the device, byte for byte what ``prepare_line`` + ``pack_lines`` build on
the host): every line is still computed as if it were run alone, as the reference runs it -- its own BatchNorm statistics, zero
padding at its own right edge -- so the decodes are those of one line per run.  Files are grouped by padded width to cut padding;
the report keeps the reference's order (sorted names) and charges each file its batch's time (the resize included) divided by the
batch's lines.  ``cfg.FEED_DTYPE`` does not apply: the lines are fed as 8-bit pixels, which give the f32 feed's bits."""
import math
import os

import numpy as np

from ... import engine
from ...session import Session
from .config import cfg, get_encode_decode_dict
from .utils.timer import Timer


def gray_rule():
    """How a file becomes gray here: 0 when OpenCV imports (cv2.imread(path, 0), as the reference reads), 1 otherwise (Pillow's
    convert("L")).  load_line_image reads with it, and the device PNG decoder of the `images` feed follows it, so both give the
    same bytes."""
    try:
        import cv2  # noqa: F401
        return 0
    except Exception:
        return 1


def load_line_image(path):
    """uint8 gray HxW (cv2.imread(path, 0) in the reference; PIL here when cv2 is unavailable)."""
    if gray_rule() == 0:
        try:
            import cv2
            img = cv2.imread(path, 0)
            if img is not None:
                return img
        except Exception:
            pass
    from PIL import Image
    return np.asarray(Image.open(path).convert("L"), dtype=np.uint8)


def line_size(h, w):
    """The size rule of an evaluation line h rows x w columns: (nw, line_width, time_step_len) -- nw its width once resized to
    cfg.IMG_HEIGHT rows (the reference's int(32 / h * w) in Python's double arithmetic, at least 1; w itself when h is already 32),
    line_width its padded width (nw rounded up to a multiple of POOL_SCALE, at least 8) and time_step_len its conv frames
    (nw // 4 - 1, at least 0).  prepare_line and the `images` feed (crnn_resize_lines_u8) both take their sizes from here."""
    h, w = int(h), int(w)
    nw = w if h == cfg.IMG_HEIGHT else max(1, int(cfg.IMG_HEIGHT / h * w))
    width = max(8, int(math.ceil(nw / cfg.POOL_SCALE) * cfg.POOL_SCALE))
    return nw, width, max(nw // cfg.POOL_SCALE + cfg.OFFSET_TIME_STEP, 0)


def _line_entry(path):
    """A file's entry of the `images` feed: its bytes when they are a PNG of 1 .. engine.RESIZE_MAX_HEIGHT rows and 1 ..
    engine.PNG_MAX_WIDTH columns, or a baseline or extended-sequential JPEG (SOF0 / SOF1) of 1 .. engine.RESIZE_MAX_HEIGHT rows
    (read once, decoded on the device), otherwise load_line_image(path)."""
    try:
        with open(path, "rb") as f:
            data = f.read()
    except OSError:
        return load_line_image(path)
    size = engine.png_size(data)
    if size is not None and 1 <= size[0] <= engine.RESIZE_MAX_HEIGHT and 1 <= size[1] <= engine.PNG_MAX_WIDTH:
        return data
    sof = engine.jpeg_sof(data) if size is None else None
    if sof is not None and sof[0] in (0xC0, 0xC1):     # progressive and the other processes are read on the host
        h, w = engine.jpeg_size(data)
        if 1 <= h <= engine.RESIZE_MAX_HEIGHT and w >= 1:
            return data
    return load_line_image(path)


def _entry_size(entry):
    return (engine.png_size(entry) or engine.jpeg_size(entry)) if isinstance(entry, bytes) else entry.shape


def prepare_line(img, dtype=np.float32):
    """[H, W] uint8 -> ([1, Wpad, 32] f32, time_step_len) exactly as test.py:65-70 lays the tensor out, after Pillow's BILINEAR
    resize to 32 rows when H is not 32 (sizes from line_size).  ``dtype=np.uint8``: the same tensor as the 8-bit pixels, without
    the division (its f32 quotient by 255 is the f32 tensor bit for bit)."""
    nw, width, tsl = line_size(img.shape[0], img.shape[1])
    if img.shape[0] != cfg.IMG_HEIGHT:
        from PIL import Image
        img = np.asarray(Image.fromarray(img).resize((nw, cfg.IMG_HEIGHT), Image.BILINEAR), dtype=np.uint8)
    w = img.shape[1]
    if np.dtype(dtype) == np.uint8:
        pad = np.zeros((cfg.IMG_HEIGHT, width), np.uint8)
        pad[:, :w] = img
    else:
        pad = np.zeros((cfg.IMG_HEIGHT, width), np.float32)
        pad[:, :w] = img.astype(np.float32) / 255.0
    data = np.ascontiguousarray(pad.swapaxes(0, 1)).reshape(1, width, cfg.NUM_FEATURES)
    return data, np.array([tsl], np.int32)


def pack_lines(lines):
    """[(data [1, W_i, 32] f32, time_step_len [1] i32) as prepare_line returns them] -> (data [N, W, 32] f32 with line i in columns
    [0, W_i) of slot i and zero beyond, line_width [N] i32 = W_i, time_step_len [N] i32), W = max W_i: the feed of a packed run.
    Lines prepared as uint8 pack into a uint8 batch (the lines' dtype; all lines must share it)."""
    if not lines:
        raise ValueError("pack_lines: no lines")
    widths = []
    dtype = np.asarray(lines[0][0]).dtype
    for d, t in lines:
        d, t = np.asarray(d), np.asarray(t)
        if d.dtype != dtype:
            raise ValueError(f"pack_lines: lines of dtypes {dtype} and {d.dtype}")
        if d.ndim != 3 or d.shape[0] != 1 or d.shape[2] != cfg.NUM_FEATURES:
            raise ValueError(f"pack_lines: each line must be [1, W_i, {cfg.NUM_FEATURES}], got {d.shape}")
        w = d.shape[1]
        if w < 8 or w % cfg.POOL_SCALE:
            raise ValueError(f"pack_lines: line width {w} must be a multiple of {cfg.POOL_SCALE} and >= 8")
        if t.shape != (1,) or t[0] < 0 or t[0] > w // cfg.POOL_SCALE - 1:
            raise ValueError(f"pack_lines: time_step_len {t} must lie in [0, {w // cfg.POOL_SCALE - 1}] for a line {w} wide")
        widths.append(w)
    data = np.zeros((len(lines), max(widths), cfg.NUM_FEATURES), dtype)
    for i, (d, _) in enumerate(lines):
        data[i, :widths[i]] = d[0]
    tsl = np.array([int(np.asarray(t)[0]) for _, t in lines], np.int32)
    return data, np.array(widths, np.int32), tsl


def decodeRes(nums, ignore=0):
    _, decode_maps = get_encode_decode_dict()
    return [decode_maps[int(i)] for i in nums if i != ignore]


def nbest_text(nbest, r):
    """test_model's addition for line r of a "beam_decoded" fetch: ", n-best: <read> (<p>), ..." over its real paths, p =
    exp(log_prob), then ", margin: <log P1 - log P2>" when a second path exists."""
    k = int(nbest["num_paths"][r])
    lp = nbest["log_prob"][r].astype(np.float64)
    reads = ("{} ({:.4f})".format("".join(decodeRes(nbest["labels"][r, j, :nbest["len"][r, j]])), float(np.exp(lp[j])))
             for j in range(k))
    text = ", n-best: " + ", ".join(reads)
    if k > 1:
        text += ", margin: {:.4f}".format(float(lp[0] - lp[1]))
    return text


class SolverWrapper(object):
    def __init__(self, sess, network, imgdb, output_dir, logdir, pretrained_model=None):
        self.net = network
        self.imgdb = imgdb
        self.output_dir = output_dir
        self.pretrained_model = pretrained_model
        print("done")

    def test_model(self, sess, testDir=None, restore=True):
        dense_decoded = self.net.get_output("logits").net  # noqa: F841  (handle kept for symmetry with the reference)
        from ..networks.network import Fetch
        dense_decoded = Fetch(self.net, "dense_decoded")
        confidence = bool(cfg.TEST.get("CONFIDENCE", False))
        if confidence:      # the alignment's labels are dense_decoded's
            dense_decoded = Fetch(self.net, "read_alignment")
        lexicon = bool(cfg.TEST.get("LEXICON", ""))
        if lexicon:         # the lexicon read of each line next to its plain read
            dense_decoded = [dense_decoded, Fetch(self.net, "lexicon_decoded")]
        top_paths = int(cfg.TEST.get("TOP_PATHS", 1))
        if top_paths > 1:   # the n best beam reads after the read
            dense_decoded = (dense_decoded if lexicon else [dense_decoded]) + [Fetch(self.net, "beam_decoded")]
        if restore:
            from .train import SolverWrapper as TrainSolver
            ts = TrainSolver.__new__(TrainSolver)
            ts.net, ts.output_dir = self.net, self.output_dir
            path = self.pretrained_model or ts._latest_checkpoint()
            try:
                print("Restoring from {}...".format(path), end=" ")
                sess.engine_for(self.net)
                ts.restore(sess, path)
                print("done")
            except Exception:
                raise Exception("Check your pretrained {:s}".format(str(path)))
        files = sorted(os.listdir(testDir))
        # each line goes to the device at its native size and is resized there (the `images` feed), whatever cfg.FEED_DTYPE says:
        # a PNG or JPEG file as its bytes, decoded on the device, any other file as load_line_image's array
        images = [_line_entry(os.path.join(testDir, f)) for f in files]
        # batches of lines of similar padded width (stable sort: ties keep name order), so little of a batch is padding
        widths = [line_size(*_entry_size(im))[1] for im in images]
        order = sorted(range(len(files)), key=lambda i: widths[i])
        bs = max(1, int(cfg.TEST.BATCH_SIZE))
        timer = Timer()
        res_of, time_of, conf_of = {}, {}, {}
        for b0 in range(0, len(order), bs):
            idx = order[b0:b0 + bs]
            timer.tic()
            feed_dict = {self.net.images: [images[i] for i in idx], self.net.keep_prob: 1.0}
            try:
                dense = sess.run(fetches=dense_decoded, feed_dict=feed_dict)
            except engine.ImageDecodeError as e:   # files the device refused are read on the host, and the batch runs again
                for r in e.entries:
                    images[idx[r]] = load_line_image(os.path.join(testDir, files[idx[r]]))
                feed_dict[self.net.images] = [images[i] for i in idx]
                dense = sess.run(fetches=dense_decoded, feed_dict=feed_dict)
            dt = timer.toc(average=False) / len(idx)
            if top_paths > 1:
                *dense, nbest = dense
                dense = dense if lexicon else dense[0]
            if lexicon:
                dense, lex = dense
            if confidence:
                al, dense = dense, dense["labels"]
            for r, i in enumerate(idx):
                res_of[i] = "".join(decodeRes(dense[r]))
                time_of[i] = dt
                if lexicon:
                    plain, res_of[i] = res_of[i], "".join(decodeRes(lex["labels"][r]))
                    if plain != res_of[i]:
                        conf_of[i] = ", read: {}".format(plain)
                if confidence:
                    k = int((dense[r] != 0).sum())
                    conf_of[i] = conf_of.get(i, "") + ", conf: {:.4f}, peaks: [{}]".format(float(np.exp(np.float64(al["path_logprob"][r]))),
                                                                     " ".join("{:.3f}".format(float(p)) for p in al["peak"][r, :k]))
                if top_paths > 1:
                    conf_of[i] = conf_of.get(i, "") + nbest_text(nbest, r)
        total = correct = 0
        for i, file in enumerate(files):
            total += 1
            org = file.split(".")[0].split("_")[1]
            if org == res_of[i]:
                correct += 1
            print(file, end=" ")
            print("cost time: {:.3f},\n    res: {}{}".format(time_of[i], res_of[i], conf_of.get(i, "")))
        print("total acc:{}/{}={:.4f}".format(correct, total, correct / max(total, 1)))
        return correct, total


def test_net(network, imgdb, testDir, output_dir, log_dir, pretrained_model=None, restore=True):
    with Session() as sess:
        sw = SolverWrapper(sess, network, imgdb, output_dir, logdir=log_dir, pretrained_model=pretrained_model)
        print("Solving...")
        sw.test_model(sess, testDir=testDir, restore=restore)
        print("done solving")
