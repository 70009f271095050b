"""Pillow's 8-bit BILINEAR resize restated in numpy, the reference crnn_resize_lines_u8 is checked against.

For one axis, in_size -> out_size, PB = 22 (Pillow's Resample.c: precompute_coeffs, normalize_coeffs_8bpc and the 8bpc passes):
    scale = in / out;  fs = max(scale, 1);  support = fs;  ss = 1 / fs;  ksize = 2 * ceil(support) + 1
    center = (xx + 0.5) * scale
    xmin = max(0, (int)(center - support + 0.5));  n = min(in, (int)(center + support + 0.5)) - xmin
    w[x] = max(0, 1 - |(x + xmin - center + 0.5) * ss|) for x < n;  ww = sum of w in index order;  w[x] /= ww when ww != 0
    k[x] = (int)(w[x] * 2^PB + 0.5)   (w[x] * 2^PB - 0.5 for a negative weight; the bilinear filter has none)
    out[xx] = clamp((2^(PB-1) + sum_x src[xmin + x] * k[x]) >> PB, 0, 255)
The horizontal pass runs first, on every row; the vertical pass on its u8 result; a pass whose size is unchanged is skipped.  A
source more than 100 times taller than wide (h > 100 w) takes the passes the other way round, vertical first, as Pillow 12.2 does
(found by sweeping h against w: the boundary is exactly h = 100 w + 1, whatever the target size).
numpy's float64 ufuncs round each operation (no contraction), so the weights are Pillow's.  The weight sum is accumulated column by
column in index order: np.sum's pairwise summation would reorder it.  The integer sums are exact in any order."""
import numpy as np

PB = 22


def axis_coeffs(in_size, out_size):
    """(xmin [out] int64, k [out, ksize] int64): the integer taps of every output position, zero past each window."""
    scale = float(in_size) / float(out_size)
    fs = max(scale, 1.0)
    support = fs
    ss = 1.0 / fs
    ksize = int(np.ceil(support)) * 2 + 1
    center = (np.arange(out_size, dtype=np.float64) + 0.5) * scale
    xmin = np.maximum(np.trunc(center - support + 0.5), 0).astype(np.int64)
    xmax = np.minimum(np.trunc(center + support + 0.5).astype(np.int64), in_size)
    n = xmax - xmin
    x = np.arange(ksize, dtype=np.int64)[None, :]
    t = np.abs(((x + xmin[:, None]).astype(np.float64) - center[:, None] + 0.5) * ss)
    w = np.where((x < n[:, None]) & (t < 1.0), 1.0 - t, 0.0)
    ww = np.zeros(out_size, np.float64)
    for j in range(ksize):                       # in index order, as Pillow adds them
        ww = ww + w[:, j]
    w = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    k = np.where(w < 0, np.trunc(w * (1 << PB) - 0.5), np.trunc(w * (1 << PB) + 0.5)).astype(np.int64)
    return xmin, k


def _pass(img, out_size, axis):
    """One axis of `img` (uint8 2-D) resampled to out_size along `axis` (1: horizontal, 0: vertical)."""
    a = img if axis == 1 else img.T
    in_size = a.shape[1]
    xmin, k = axis_coeffs(in_size, out_size)
    ksize = k.shape[1]
    idx = np.minimum(xmin[:, None] + np.arange(ksize)[None, :], in_size - 1)    # taps past a window have k = 0
    acc = np.full((a.shape[0], out_size), 1 << (PB - 1), np.int64)
    src = a.astype(np.int64)
    for j in range(ksize):
        acc += src[:, idx[:, j]] * k[:, j][None, :]
    out = np.clip(acc >> PB, 0, 255).astype(np.uint8)
    return out if axis == 1 else np.ascontiguousarray(out.T)


def resize_bilinear(img, out_w, out_h):
    """Image.fromarray(img).resize((out_w, out_h), Image.BILINEAR) for a uint8 gray img [h, w]."""
    img = np.asarray(img, np.uint8)
    h, w = img.shape
    if out_w != w and out_h != h and h > 100 * w:
        return np.ascontiguousarray(_pass(_pass(img, out_h, 0), out_w, 1))
    if out_w != w:
        img = _pass(img, out_w, 1)
    if out_h != h:
        img = _pass(img, out_h, 0)
    return np.ascontiguousarray(img)


def pack_slot(img, W, line_size):
    """Slot of one native-size line in the [N, W, 32] uint8 batch crnn_resize_lines_u8 writes: the resized line transposed into
    columns [0, out_w), zero from there to W.  line_size: lib.lstm.test.line_size."""
    nw, _, _ = line_size(*img.shape)
    r = resize_bilinear(img, nw, 32)
    slot = np.zeros((W, 32), np.uint8)
    slot[:nw] = r.T
    return slot
