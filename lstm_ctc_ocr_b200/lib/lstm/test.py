"""Evaluation solver with the reference's surface (lib/lstm/test.py): ``SolverWrapper.test_model(sess, testDir, restore)`` and
``test_net(network, imgdb, testDir, output_dir, log_dir, pretrained_model, restore)``.

Per file (test.py:57-88): read as gray, right-pad the width to a multiple of POOL_SCALE with 0, /255, transpose to
[1, W, 32], decode, map ids -> chars, exact match against the label encoded in the file name (``<idx>_<chars>.png``).
Deviation from the reference, per SURVEY §3.4: ``time_step_len`` is fed as W//4 - 1 (the data layer's convention,
gen.py:54), not the off-by-one W//4 of test.py:74 which exceeds the number of conv frames.

Lines are evaluated in packed batches of ``cfg.TEST.BATCH_SIZE`` (``pack_lines`` + the ``line_width`` feed): every line is still
computed as if it were run alone, as the reference runs it -- its own BatchNorm statistics, zero padding at its own right edge --
so the decodes are those of one line per run.  Files are grouped by width to cut padding; the report keeps the reference's
order (sorted names) and charges each file its batch's time divided by the batch's lines."""
import math
import os

import numpy as np

from ...session import Session
from .config import cfg, get_encode_decode_dict
from .utils.gen import feed_dtype
from .utils.timer import Timer


def load_line_image(path):
    """uint8 gray HxW (cv2.imread(path, 0) in the reference; PIL here when cv2 is unavailable)."""
    try:
        import cv2
        img = cv2.imread(path, 0)
        if img is not None:
            return img
    except Exception:
        pass
    from PIL import Image
    return np.asarray(Image.open(path).convert("L"), dtype=np.uint8)


def prepare_line(img, dtype=np.float32):
    """[H=32, W] uint8 -> ([1, Wpad, 32] f32, time_step_len) exactly as test.py:65-70 lays the tensor out.  ``dtype=np.uint8``:
    the same tensor as the 8-bit pixels, without the division (its f32 quotient by 255 is the f32 tensor bit for bit)."""
    if img.shape[0] != cfg.IMG_HEIGHT:
        from PIL import Image
        nw = max(1, int(cfg.IMG_HEIGHT / img.shape[0] * img.shape[1]))
        img = np.asarray(Image.fromarray(img).resize((nw, cfg.IMG_HEIGHT), Image.BILINEAR), dtype=np.uint8)
    w = img.shape[1]
    width = max(8, int(math.ceil(w / cfg.POOL_SCALE) * cfg.POOL_SCALE))
    if np.dtype(dtype) == np.uint8:
        pad = np.zeros((cfg.IMG_HEIGHT, width), np.uint8)
        pad[:, :w] = img
    else:
        pad = np.zeros((cfg.IMG_HEIGHT, width), np.float32)
        pad[:, :w] = img.astype(np.float32) / 255.0
    data = np.ascontiguousarray(pad.swapaxes(0, 1)).reshape(1, width, cfg.NUM_FEATURES)
    return data, np.array([max(w // cfg.POOL_SCALE + cfg.OFFSET_TIME_STEP, 0)], np.int32)


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
        dtype = feed_dtype(cfg.FEED_DTYPE)       # "uint8": lines stay 8-bit pixels and are fed through data_u8
        lines = [prepare_line(load_line_image(os.path.join(testDir, f)), dtype=dtype) for f in files]
        # batches of lines of similar width (stable sort: ties keep name order), so little of a batch is padding
        order = sorted(range(len(files)), key=lambda i: lines[i][0].shape[1])
        bs = max(1, int(cfg.TEST.BATCH_SIZE))
        timer = Timer()
        res_of, time_of, conf_of = {}, {}, {}
        for b0 in range(0, len(order), bs):
            idx = order[b0:b0 + bs]
            timer.tic()
            data, lw, tsl = pack_lines([lines[i] for i in idx])
            feed_dict = {(self.net.data_u8 if dtype == np.uint8 else self.net.data): data, self.net.line_width: lw, self.net.time_step_len: tsl, self.net.keep_prob: 1.0}
            dense = sess.run(fetches=dense_decoded, feed_dict=feed_dict)
            dt = timer.toc(average=False) / len(idx)
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
