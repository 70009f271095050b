"""Device line renderer (csrc/render.cu) on the GPU:
  1. Layout: crnn_render_layout equals gen.philox_layout exactly (default stream, buckets 80/160/256, lines of 30-70 characters,
     N = 1, 64, 1024, ranks 0..7 of world 8).
  2. Pixels: outputs and workspace filled with 0xA5 first; the batch equals groupBatch(render_layout(...), uint8, pad_to) byte
     for byte, padding included, with equal labels, lengths and time steps.
  3. Determinism and streams: the same bits on every run and on a gated non-blocking stream behind a busy default stream;
     status codes leave the outputs untouched; an unreachable bucket raises through its status flag.
  4. Feed: Session.run fed the device tensor computes bit for bit what the same bytes fed as a host data_u8 array compute.
  5. Learning: train_model with cfg.RENDER = "device" learns to read, with no producer processes."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _atlas():
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    return engine.GlyphAtlas(gen._font(42), device=DEV)


def _device_layout(atlas, N, seed, bucket=None, lens=None):
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    lo, hi, nw_lo, nw_hi = gen._render_range(bucket, lens)
    layout = torch.full((N, engine.render_record_ints(hi)), -0x5A5A5A5B, dtype=torch.int32, device=DEV)
    feeds = torch.full((engine.render_feed_ints(N, hi),), -0x5A5A5A5B, dtype=torch.int32, device=DEV)
    engine.render_layout(seed, lo, hi, nw_lo, nw_hi, atlas, layout, feeds)
    torch.cuda.synchronize()
    return layout, feeds


def _assert_layout_equal(d, h):
    assert d["status"] == h["status"] == 0
    for k in ("len", "bg", "x0", "canvas_w", "nw", "tsl", "attempt", "chars", "x", "y", "fill"):
        assert np.array_equal(d[k], h[k]), k
    off = np.concatenate([[0], np.cumsum(h["len"])[:-1]])
    assert np.array_equal(d["label_off"], off)
    assert np.array_equal(d["label_len"], h["len"]) and np.array_equal(d["time_steps"], h["tsl"])
    live = np.arange(h["max_len"])[None, :] < h["len"][:, None]
    assert np.array_equal(d["labels"], h["chars"][live])
    assert d["max_nw"] == h["nw"].max()


LAYOUT_CASES = ([pytest.param(N, None, None, 0, 1, id=f"default_N{N}") for N in (1, 64, 1024)]
                + [pytest.param(N, b, None, 0, 1, id=f"bucket{b}_N{N}") for b in (80, 160, 256) for N in (1, 64, 1024)]
                + [pytest.param(N, None, (30, 70), 0, 1, id=f"len30_70_N{N}") for N in (1, 64, 1024)]
                + [pytest.param(64, b, None, r, 8, id=f"rank{r}_of_8_bucket{b}") for r in range(8) for b in (None, 256)])


@pytest.mark.parametrize("N,bucket,lens,rank,world", LAYOUT_CASES)
def test_layout_equals_the_host_stream(N, bucket, lens, rank, world):
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    atlas = _atlas()
    for k in (0, 5):
        seed = gen.batch_seed(k, 1234, rank, world)
        d = engine.render_layout_dict(*_device_layout(atlas, N, seed, bucket, lens))
        _assert_layout_equal(d, gen.philox_layout(N, seed, bucket=bucket, lens=lens))
        want_W = bucket if bucket else max(8, -(-int(d["max_nw"]) // 4) * 4)
        assert d["W"] == want_W


def _device_batch(atlas, N, seed, bucket=None, lens=None):
    from lstm_ctc_ocr_b200 import engine
    layout, feeds = _device_layout(atlas, N, seed, bucket, lens)
    d = engine.render_layout_dict(layout, feeds)
    ws = torch.full((engine.render_workspace_bytes(N, d["max_len"], atlas.max_adv),), 0xA5, dtype=torch.uint8, device=DEV)
    out = torch.full((N, d["W"], 32), 0xA5, dtype=torch.uint8, device=DEV)
    engine.render_lines_u8(layout, d["max_len"], atlas, d["W"], ws, out)
    torch.cuda.synchronize()
    return out.cpu().numpy(), d


PIXEL_CASES = [pytest.param(64, None, None, id="default_N64"), pytest.param(1024, None, None, id="default_N1024"),
               pytest.param(1, None, None, id="default_N1")] + \
              [pytest.param(256, b, None, id=f"bucket{b}_N256") for b in (80, 160, 256)] + \
              [pytest.param(64, None, (30, 70), id="len30_70_N64")]


@pytest.mark.parametrize("N,bucket,lens", PIXEL_CASES)
def test_pixels_equal_pils_batch_byte_for_byte(N, bucket, lens):
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    atlas = _atlas()
    seed = gen.batch_seed(3, 777)
    got, d = _device_batch(atlas, N, seed, bucket, lens)
    lay = gen.philox_layout(N, seed, bucket=bucket, lens=lens)
    imgs, lab, ll, tsl = gen.render_layout(lay, pad_to=bucket)
    want = np.stack(imgs)
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = np.flatnonzero((got != want).reshape(N, -1).any(1))
    assert bad.size == 0, f"lines {bad[:10].tolist()} differ ({bad.size} of {N})"
    assert np.array_equal(d["labels"], lab) and np.array_equal(d["label_len"], ll) and np.array_equal(d["time_steps"], tsl)


@pytest.mark.parametrize("bucket,lens", [(None, None), (256, None), (None, (30, 70))])
def test_renderer_batches_equal_the_host_restatement(bucket, lens):
    """DeviceLineRenderer's batches k = 0, 1, 2 (the pipelined path: layout one batch ahead on its own stream) against the host
    restatement of the same batch seeds, and the same bits from a second renderer."""
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    r1 = gen.DeviceLineRenderer(48, seed=55, rank=1, world=2, bucket=bucket, lens=lens, device=DEV)
    r2 = gen.get_batch(0, batch_size=48, seed=55, rank=1, world=2, bucket=bucket, on_device=True, device=DEV) if lens is None else \
        gen.DeviceLineRenderer(48, seed=55, rank=1, world=2, bucket=bucket, lens=lens, device=DEV)
    for k in range(3):
        x, lab, ll, tsl = next(r1)
        y = next(r2)
        assert x.dtype == torch.uint8 and x.is_cuda and x.is_contiguous()
        assert lab.dtype == ll.dtype == tsl.dtype == np.int32
        lay = gen.philox_layout(48, gen.batch_seed(k, 55, 1, 2), bucket=bucket, lens=lens)
        imgs, hl, hll, htsl = gen.render_layout(lay, pad_to=bucket)
        xa = x.cpu().numpy()
        assert np.array_equal(xa, np.stack(imgs)), k
        assert np.array_equal(lab, hl) and np.array_equal(ll, hll) and np.array_equal(tsl, htsl)
        assert np.array_equal(xa, y[0].cpu().numpy()) and np.array_equal(lab, y[1])


def test_same_bits_on_a_gated_stream_behind_a_busy_default_stream():
    import test_gpu_streams as SG
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    atlas = _atlas()
    N, seed = 256, gen.batch_seed(9, 31)
    lo, hi, nw_lo, nw_hi = gen._render_range(None, (8, 20))
    layout = torch.empty((N, engine.render_record_ints(hi)), dtype=torch.int32, device=DEV)
    feeds = torch.empty((engine.render_feed_ints(N, hi),), dtype=torch.int32, device=DEV)
    ws = torch.empty((engine.render_workspace_bytes(N, hi, atlas.max_adv),), dtype=torch.uint8, device=DEV)
    engine.render_layout(seed, lo, hi, nw_lo, nw_hi, atlas, layout, feeds)
    W, total = int(feeds[3].item()), int(feeds[2].item())
    out = torch.empty((N, W, 32), dtype=torch.uint8, device=DEV)

    def call():
        engine.render_layout(seed, lo, hi, nw_lo, nw_hi, atlas, layout, feeds)
        engine.render_lines_u8(layout, hi, atlas, W, ws, out)
        return {"out": out.clone(), "feeds": feeds[:4 + 2 * N + total].clone()}      # past the labels: unspecified
    got = SG._gated("render", call, [], [layout, feeds, ws, out])
    lay = gen.philox_layout(N, seed, lens=(8, 20))
    assert np.array_equal(got["out"].cpu().numpy(), np.stack(gen.render_layout(lay)[0]))


def test_status_codes_leave_the_outputs_untouched():
    from lstm_ctc_ocr_b200 import _lib, engine
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    lib = _lib.load()
    atlas = _atlas()
    N, L = 8, 6
    layout, feeds = _device_layout(atlas, N, 5)
    lay_before, feeds_before = layout.clone(), feeds.clone()
    ws_bytes = engine.render_workspace_bytes(N, L, atlas.max_adv)
    ws = torch.full((ws_bytes,), 0xA5, dtype=torch.uint8, device=DEV)
    out = torch.full((N, 88, 32), 0xA5, dtype=torch.uint8, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    p = lambda t: t.data_ptr()  # noqa: E731
    g, m = p(atlas.glyphs), p(atlas.masks)
    assert lib.crnn_render_layout(5, N, 4, L, 0, 0, g, 63, p(layout), p(feeds), st) == 1
    assert lib.crnn_render_layout(5, N, 4, 257, 0, 0, g, 62, p(layout), p(feeds), st) == 4
    assert lib.crnn_render_layout(5, N, 4, L, 80, 80, g, 62, p(layout), p(feeds), st) == 1
    assert lib.crnn_render_layout(5, 0, 4, L, 0, 0, g, 62, p(layout), p(feeds), st) == 1
    assert lib.crnn_render_lines_u8(p(layout), N, L, g, m, atlas.max_adv, 86, p(ws), ws_bytes, p(out), st) == 1
    assert lib.crnn_render_lines_u8(p(layout), N, L, g, m, atlas.max_adv, 88, p(ws), ws_bytes, p(out) + 1, st) == 1
    assert lib.crnn_render_lines_u8(p(layout), N, L, g, m, atlas.max_adv, 88, p(ws), ws_bytes - 1, p(out), st) == 5
    assert lib.crnn_render_lines_u8(p(layout), N, L, g, m, atlas.max_adv, 88, 0, ws_bytes, p(out), st) == 1
    assert lib.crnn_render_lines_u8(p(layout), N, 300, g, m, atlas.max_adv, 88, p(ws), ws_bytes, p(out), st) == 4
    torch.cuda.synchronize()
    assert torch.equal(layout, lay_before) and torch.equal(feeds, feeds_before)
    assert (out == 0xA5).all() and (ws == 0xA5).all()


def test_unreachable_bucket_is_an_error_not_a_line():
    """Lines of 30-40 characters never fit the 80-px bucket: the layout reports every line through its status word, and the
    renderer raises naming the bucket."""
    from lstm_ctc_ocr_b200 import engine
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    atlas = _atlas()
    N = 16
    layout = torch.empty((N, engine.render_record_ints(40)), dtype=torch.int32, device=DEV)
    feeds = torch.empty((engine.render_feed_ints(N, 40),), dtype=torch.int32, device=DEV)
    engine.render_layout(3, 30, 40, 0, 80, atlas, layout, feeds)
    d = engine.render_layout_dict(layout, feeds)
    assert d["status"] == N and (d["attempt"] == gen.RENDER_MAX_ATTEMPTS - 1).all()
    h = gen.philox_layout(N, 3, lens=(30, 40))
    assert h["status"] == 0                                        # the same lengths without the bucket are fine
    old = dict(gen.BUCKET_CHARS)
    gen.BUCKET_CHARS[80] = (30, 40)
    try:
        assert gen.philox_layout(N, 3, bucket=80)["status"] == N
        r = gen.DeviceLineRenderer(N, seed=3, bucket=80, device=DEV)
        with pytest.raises(ValueError, match="bucket 80"):
            next(r)
    finally:
        gen.BUCKET_CHARS.clear()
        gen.BUCKET_CHARS.update(old)


def _train_net():
    from lstm_ctc_ocr_b200 import synthetic
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    net = get_network("LSTM_train")
    sess = Session(device=DEV)
    sess.engine_for(net).load_params(synthetic.init_params(3))
    return net, sess


def test_session_takes_the_device_batch_in_place():
    """Logits, costs, CTC gradient, loss and a training step's loss: bit for bit those of the same bytes fed as a host data_u8
    array; the weight gradients of the step (summed with f32 atomics, so not bit-reproducible run to run on either feed) to
    within reordering.  h2d_bytes counts only the integer feeds."""
    from lstm_ctc_ocr_b200.lib.lstm import train as T
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    r = gen.DeviceLineRenderer(64, seed=8, device=DEV)
    x, lab, ll, tsl = next(r)
    host = x.cpu().numpy()
    res = {}
    for name, data in (("device", x), ("host", host)):
        net, sess = _train_net()
        with sess:
            loss, dec = net.build_loss()
            feed = {net.data_u8: data, net.labels: lab, net.labels_len: ll, net.time_step_len: tsl, net.keep_prob: 1.0}
            fl = [Fetch(net, "logits"), Fetch(net, "ctc_costs"), loss, dec, Fetch(net, "ctc_grad")]
            out = sess.run(fl, feed)
            h2d = sess.h2d_bytes
            train_op = T.TrainOp(net, T.Variable(1e-3), T.Variable(0))
            sess.engine_for(net).set_solver("Adam", 0.9)
            step_loss, _ = sess.run([loss, train_op], feed)
            eng = sess.engine_for(net)
            res[name] = dict(logits=out[0], costs=out[1], loss=out[2], dec=out[3], ctc_grad=out[4], step_loss=step_loss, h2d=h2d,
                             grads={k: eng.grad_tensor(k).cpu().numpy() for k in eng.table})
    a, b = res["device"], res["host"]
    for k in ("logits", "costs", "dec", "ctc_grad"):
        assert np.array_equal(a[k], b[k]), k
    assert np.float32(a["loss"]).tobytes() == np.float32(b["loss"]).tobytes()
    assert np.float32(a["step_loss"]).tobytes() == np.float32(b["step_loss"]).tobytes()
    for k, g in b["grads"].items():
        assert np.linalg.norm(a["grads"][k] - g) <= 1e-4 * np.linalg.norm(g) + 1e-7, k
    assert a["h2d"] == tsl.nbytes + lab.nbytes + ll.nbytes
    assert b["h2d"] == host.nbytes + tsl.nbytes + lab.nbytes + ll.nbytes


def test_session_refuses_device_batches_it_cannot_take():
    from lstm_ctc_ocr_b200 import synthetic
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.networks.network import Fetch
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    net = get_network("LSTM_test")
    r = gen.DeviceLineRenderer(4, seed=8, device=DEV)
    x, lab, ll, tsl = next(r)
    with Session(device=DEV) as sess:
        sess.assign(net, synthetic.init_params(3))
        f = Fetch(net, "logits")
        with pytest.raises(ValueError, match="line_width"):
            sess.run(f, {net.data_u8: x, net.time_step_len: tsl, net.line_width: np.full(4, x.shape[1], np.int32)})
        with pytest.raises(ValueError, match="uint8"):
            sess.run(f, {net.data_u8: x.float(), net.time_step_len: tsl})
        with pytest.raises(ValueError, match="uint8"):
            sess.run(f, {net.data_u8: x[:, ::2], net.time_step_len: tsl})


def test_training_on_device_renders_learns_to_read():
    """train_model with cfg.RENDER = "device" (no producer processes) reaches the bar of
    test_gpu_training.py::test_training_on_fresh_renders_learns_to_read on the same host-rendered held-out lines."""
    from lstm_ctc_ocr_b200.lib.lstm import train as T
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    from lstm_ctc_ocr_b200.lib.lstm.utils.training import accuracy_calculation
    from lstm_ctc_ocr_b200.lib.networks.factory import get_network
    from lstm_ctc_ocr_b200.session import Session
    assert gen.can_render()
    keys = ("LEARNING_RATE", "DISPLAY", "SNAPSHOT_ITERS", "WEIGHT_DECAY", "BATCH_SIZE", "STEPSIZE", "GAMMA")
    old = {k: cfg.TRAIN[k] for k in keys}
    old_val, old_render, old_seed = cfg.VAL.VAL_STEP, cfg.RENDER, cfg.RNG_SEED
    cfg.TRAIN.LEARNING_RATE, cfg.TRAIN.DISPLAY, cfg.TRAIN.SNAPSHOT_ITERS, cfg.TRAIN.WEIGHT_DECAY = 1e-4, 2000, 10 ** 9, 1e-5
    cfg.TRAIN.BATCH_SIZE, cfg.TRAIN.STEPSIZE, cfg.TRAIN.GAMMA, cfg.VAL.VAL_STEP = 64, 2000, 1.0, 10 ** 9
    cfg.RENDER, cfg.RNG_SEED = "device", 1000
    held = [gen.make_batch(k, 128, True, seed=900000) for k in range(4)]                   # disjoint seeds: never seen in training
    try:
        net = get_network("LSTM_train")
        with Session(device=DEV) as sess:
            sw = T.SolverWrapper(sess, net, None, None, "/tmp/crnn_learn_dev_out", "/tmp/crnn_learn_dev_log")
            hist = sw.train_model(sess, 4001, restore=False)
            assert len(hist) == 4000 and np.mean(hist[-200:]) < 0.15 * np.mean(hist[:200]), (np.mean(hist[:200]), np.mean(hist[-200:]))
            _, dec_h = net.build_loss()
            ok = tot = 0
            for (imgs, lab, ll, tsl) in held:
                res = sess.run(dec_h, feed_dict={net.data: np.array(imgs), net.labels: np.array(lab), net.time_step_len: np.array(tsl),
                                                 net.labels_len: np.array(ll), net.keep_prob: 1.0})
                org = sw.restoreLabel(lab, ll)
                ok += accuracy_calculation(org, res, isPrint=False) * len(org); tot += len(org)
        assert ok / tot >= 0.85, ok / tot
    finally:
        for k in keys:
            cfg.TRAIN[k] = old[k]
        cfg.VAL.VAL_STEP, cfg.RENDER, cfg.RNG_SEED = old_val, old_render, old_seed
