"""uint8 feed without a GPU: the pixel quotient, the data layer's dtype switch, the feeder, the FEED_DTYPE key and the data_u8
placeholder.  The device side of the same contract is tests/test_gpu_u8_feed.py."""
import numpy as np
import pytest


def test_quotient_is_the_ieee_division_and_not_a_reciprocal_multiply():
    """x = (float)u / 255.0f for all 256 bytes is numpy's u.astype(f32) / f32(255) and the f64 quotient rounded once to f32 --
    the value every f32 feed of the project holds.  A bare multiply by the f32 reciprocal (or __fdividef) is cheaper but is a
    different number on 126 of the 256 bytes, so conv1 would see other operands than the f32 feed gives it: it is not used
    without the correction checked below."""
    u = np.arange(256, dtype=np.uint8)
    q = u.astype(np.float32) / np.float32(255)
    assert q.dtype == np.float32
    assert np.array_equal(q, (u.astype(np.float64) / 255.0).astype(np.float32))          # correctly rounded
    py = u.astype(np.float32) / 255.                                      # prepare_line's spelling: the same f32 division
    assert py.dtype == np.float32 and np.array_equal(py, q)
    recip = u.astype(np.float32) * np.float32(1.0 / 255.0)
    assert int((recip != q).sum()) == 126
    assert q[0] == 0.0 and q[255] == 1.0


def _round_f32(x):
    """An exact rational rounded once to the nearest f32 (ties to even)."""
    from fractions import Fraction
    c = np.float32(float(x))
    best = None
    for v in (np.nextafter(c, np.float32(-np.inf)), c, np.nextafter(c, np.float32(np.inf))):
        d = abs(Fraction(float(v)) - x)
        if best is None or d < best[0] or (d == best[0] and int(np.float32(v).view(np.int32)) & 1 == 0):
            best = (d, np.float32(v))
    return best[1]


def test_device_quotient_is_exact_for_every_byte():
    """The kernels form the quotient as q0 = u * r, q = fma(fma(-q0, 255, u), r, q0) with r = f32(1/255) (u8_pixel in
    csrc/common.cuh): each operation emulated here in exact arithmetic and rounded once, as the device's __fmul_rn / __fmaf_rn
    round.  It equals u.astype(f32) / f32(255) for all 256 bytes, where q0 alone misses 126."""
    from fractions import Fraction as Fr
    r = np.float32(1) / np.float32(255)
    for u in range(256):
        q0 = _round_f32(Fr(u) * Fr(float(r)))
        res = _round_f32(Fr(u) - Fr(float(q0)) * 255)
        q = _round_f32(Fr(float(res)) * Fr(float(r)) + Fr(float(q0)))
        assert q == np.float32(u) / np.float32(255), u


def _renders(n, seed):
    import random
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    rng = random.Random(seed)
    labels = [gen.gen_rand(rng) for _ in range(n)]
    return [gen.render_line(t, rng=rng) for t in labels], labels


def test_group_batch_u8_over_255_is_the_f32_batch_bit_for_bit():
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    imgs, labels = _renders(9, 17)
    assert all(im.dtype == np.uint8 for im in imgs)
    for pad_to in (None, 256):
        f = gen.groupBatch(imgs, labels, pad_to=pad_to)
        u = gen.groupBatch(imgs, labels, pad_to=pad_to, dtype=np.uint8)
        assert f[1:] == u[1:]
        for a, b in zip(f[0], u[0]):
            assert b.dtype == np.uint8 and a.dtype == np.float32 and a.shape == b.shape
            assert np.array_equal((b.astype(np.float32) / np.float32(255)).view(np.int32), a.view(np.int32))   # padding included
    with pytest.raises(ValueError):
        gen.groupBatch([imgs[0].astype(np.float32)], labels[:1], dtype=np.uint8)
    with pytest.raises(ValueError):
        gen.groupBatch(imgs, labels, dtype=np.float16)


def test_prepare_and_pack_lines_u8_over_255_are_the_f32_feed():
    from lstm_ctc_ocr_b200.lib.lstm import test as T
    imgs, _ = _renders(7, 23)
    tall = np.repeat(imgs[0], 2, axis=0)                          # a 64-row line: prepare_line resizes it to height 32
    lines_f = [T.prepare_line(im) for im in imgs + [tall]]
    lines_u = [T.prepare_line(im, dtype=np.uint8) for im in imgs + [tall]]
    for (df, tf), (du, tu) in zip(lines_f, lines_u):
        assert du.dtype == np.uint8 and np.array_equal(tf, tu)
        assert np.array_equal((du.astype(np.float32) / np.float32(255)).view(np.int32), df.view(np.int32))
    pf, lwf, tsf = T.pack_lines(lines_f)
    pu, lwu, tsu = T.pack_lines(lines_u)
    assert pu.dtype == np.uint8 and np.array_equal(lwf, lwu) and np.array_equal(tsf, tsu)
    assert np.array_equal((pu.astype(np.float32) / np.float32(255)).view(np.int32), pf.view(np.int32))
    with pytest.raises(ValueError):
        T.pack_lines([lines_f[0], lines_u[1]])


@pytest.mark.parametrize("render", [True, False])
def test_bucket_sampler_passes_the_dtype_through(render):
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    f = gen.BucketSampler(batch_size=6, render=render, seed=5, rank=0, world=1)
    u = gen.BucketSampler(batch_size=6, render=render, seed=5, rank=0, world=1, dtype=np.uint8)
    for k in range(3):
        a, b = f.batch(k), u.batch(k)
        assert a[1:] == b[1:]
        for x, y in zip(a[0], b[0]):
            assert y.dtype == np.uint8 and y.shape == x.shape == (f.bucket_of(k), 32)
            if render:
                assert np.array_equal((y.astype(np.float32) / np.float32(255)).view(np.int32), x.view(np.int32))
            else:                                                 # the synthetic stream has no 8-bit source: its pixels are rounded
                assert np.array_equal(y, np.rint(x * np.float32(255)).astype(np.uint8))


def test_u8_prefetch_feeder_delivers_the_stream_in_order():
    """As test_prefetch_feeder_delivers_the_stream_in_order, with uint8 batches: slots a quarter of the f32 size, views uint8."""
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    arg_fn = lambda k: dict(k=k, batch_size=6, render=True, seed=11, rank=0, world=1, bucket=gen.BUCKETS[k % 3], dtype=np.uint8)
    ref = [gen.make_batch(**arg_fn(k)) for k in range(7)]
    for workers in (0, 2):
        f = gen.PrefetchFeeder(arg_fn, num_workers=workers, depth=3, max_width=256, batch_size=6)
        try:
            assert f.slot_bytes == 6 * 256 * 32
            held = []
            for k in range(7):
                view, lab, ll, tsl = next(f)
                assert view.dtype == np.uint8 and view.shape == (6, gen.BUCKETS[k % 3], 32) and view.flags.c_contiguous
                assert np.array_equal(view, np.stack(ref[k][0]))
                for got, want in zip((lab, ll, tsl), ref[k][1:]):
                    assert isinstance(got, np.ndarray) and got.dtype == np.int32 and got.tolist() == list(want)
                held.append((k, view))
                for kk, v in held[-3:]:
                    assert np.array_equal(v, np.stack(ref[kk][0]))
        finally:
            f.close()
    it = gen.get_batch(num_workers=2, batch_size=5, render=True, seed=11, dtype=np.uint8)
    try:
        imgs, flat, lens, steps = next(it)
        assert len(imgs) == 5 and imgs[0].dtype == np.uint8 and len(flat) == sum(lens)
    finally:
        if hasattr(it, "close"):
            it.close()


def test_feed_dtype_config_key(tmp_path):
    from lstm_ctc_ocr_b200.lib.lstm import config as C
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    saved = C.cfg.FEED_DTYPE
    try:
        assert saved == "float32" and gen.feed_dtype(saved) == np.float32
        f = tmp_path / "c.yml"
        f.write_text("FEED_DTYPE: uint8\n")
        C.cfg_from_file(str(f))
        assert C.cfg.FEED_DTYPE == "uint8" and gen.feed_dtype(C.cfg.FEED_DTYPE) == np.uint8
        C.cfg_from_list(["FEED_DTYPE", "float32"])
        assert C.cfg.FEED_DTYPE == "float32"
        C.cfg_from_list(["FEED_DTYPE", "uint8"])
        assert C.cfg.FEED_DTYPE == "uint8"
        with pytest.raises(ValueError):
            f.write_text("FEED_DTYPE: 8\n")
            C.cfg_from_file(str(f))
        for bad in ("float16", "int8", "u8"):
            with pytest.raises(ValueError):
                gen.feed_dtype(bad)
    finally:
        C.cfg.FEED_DTYPE = saved


def test_networks_declare_data_u8_and_refuse_both_feeds():
    from lstm_ctc_ocr_b200.lib.networks.LSTM_test import LSTM_test
    from lstm_ctc_ocr_b200.lib.networks.LSTM_train import LSTM_train
    from lstm_ctc_ocr_b200.session import Session
    for cls in (LSTM_train, LSTM_test):
        net = cls()
        ph = net.data_u8
        assert ph is net.data_u8 and ph.name == "data_u8" and ph.dtype == "uint8" and ph.shape == [None, None, 32]
        assert net.data.dtype == "float32"
    u = np.arange(2 * 8 * 32, dtype=np.int64).reshape(2, 8, 32) % 256
    got = Session._data_feed({"data_u8": u})
    assert got.dtype == np.uint8 and np.array_equal(got, u)
    got = Session._data_feed({"data": u.astype(np.uint8)})              # data keeps its meaning: the values 0..255 as f32
    assert got.dtype == np.float32 and np.array_equal(got, u.astype(np.float32))
    with pytest.raises(ValueError):
        Session._data_feed({"data": u.astype(np.float32), "data_u8": u.astype(np.uint8)})
