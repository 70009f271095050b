"""Device line renderer, host side (no GPU): the numpy Philox4x64-10 against numpy's own, the layout stream's ranges and
uniformity, the numpy compositing restatement against Pillow's draw_bitmap, the host restatement against render_line, the atlas
builder's refusal, argument checks and the ABI table."""
import os
import random
import re

import numpy as np
import pytest

from render_refs import atlas_mask, blend_glyph, composite_line

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gen():
    from lstm_ctc_ocr_b200.lib.lstm.utils import gen
    return gen


def _fonts():
    """The embedded scalable font, and a TrueType file when the machine has one."""
    gen = _gen()
    from PIL import ImageFont
    fonts = [("embedded", gen.embedded_font(42))]
    for p in ("/usr/share/fonts/truetype/dejavu/DejaVuSans-Bold.ttf", "/usr/share/fonts/truetype/dejavu/DejaVuSans.ttf",
              os.path.join(ROOT, "fonts", "Ubuntu-M.ttf")):
        if os.path.exists(p):
            fonts.append((os.path.basename(p), ImageFont.truetype(p, 42)))
            break
    return fonts


def test_philox_matches_numpy_philox():
    gen = _gen()
    rng = np.random.default_rng(1)
    for t in range(200):
        key = (int(rng.integers(0, 2 ** 63)) * 2 + t % 2, gen.RENDER_KEY1 if t % 3 else int(rng.integers(0, 2 ** 63)))
        ctr = [int(v) for v in rng.integers(0, 2 ** 63, 4, dtype=np.int64)]
        if t % 4 == 0:
            ctr = [t, t % 7, t % 5, 0]                     # the renderer's (line, attempt, block, 0) counters
        if t == 1:
            ctr = [2 ** 64 - 1, 5, 0, 0]                  # a carry into the second word
        c_int = sum(v << (64 * k) for k, v in enumerate(ctr))
        ref = np.random.Philox(key=key[0] + (key[1] << 64), counter=(c_int - 1) % 2 ** 256).random_raw(4)
        got = gen.philox4x64(np.array(ctr, np.uint64), key)
        assert np.array_equal(got, ref), (key, ctr)
    # vectorised over a batch of counters
    ctr = np.stack([np.arange(64), np.zeros(64), np.arange(64) % 3, np.zeros(64)], axis=1).astype(np.uint64)
    got = gen.philox4x64(ctr, (9, gen.RENDER_KEY1))
    for i in range(64):
        c_int = i + ((i % 3) << 128)
        assert np.array_equal(got[i], np.random.Philox(key=9 + (gen.RENDER_KEY1 << 64), counter=c_int - 1 if c_int else 2 ** 256 - 1)
                              .random_raw(4))


def test_integer_draw_is_the_high_word_of_the_product():
    gen = _gen()
    u = np.array([0, 1, 2 ** 63, 2 ** 64 - 1, 0x123456789ABCDEF0], np.uint64)
    for a, b in ((0, 61), (180, 255), (-2, 3), (2, 12)):
        want = [a + ((int(x) * (b - a + 1)) >> 64) for x in u]
        assert gen._draw(u, a, b).tolist() == want


@pytest.mark.parametrize("bucket,lens", [(None, None), (None, (30, 70)), (80, None), (160, None), (256, None)])
def test_layout_values_in_range(bucket, lens):
    gen = _gen()
    lay = gen.philox_layout(2000, 12345, bucket=bucket, lens=lens)
    lo, hi, nw_lo, nw_hi = gen._render_range(bucket, lens)
    assert lay["status"] == 0
    assert lay["len"].min() >= lo and lay["len"].max() <= hi
    assert lay["bg"].min() >= 180 and lay["bg"].max() <= 255 and lay["x0"].min() >= 2 and lay["x0"].max() <= 12
    live = np.arange(lay["max_len"])[None, :] < lay["len"][:, None]
    assert lay["chars"][live].min() >= 1 and lay["chars"][live].max() <= 62 and (lay["chars"][~live] == 0).all()
    for k, a, b in (("y", 0, 10), ("fill", 0, 90), ("dx", -2, 3)):
        assert lay[k][live].min() >= a and lay[k][live].max() <= b
    adv = gen._glyph_adv(gen._font(42), gen.cfg.CHARSET)
    assert np.array_equal(lay["canvas_w"], np.where(live, adv[np.maximum(lay["chars"] - 1, 0)], 0).sum(1) + 28)
    assert np.array_equal(lay["nw"], [int(32 / 60 * w) for w in lay["canvas_w"]])
    assert np.array_equal(lay["tsl"], lay["nw"] // 4 - 1)
    if nw_hi:
        assert lay["nw"].min() > nw_lo and lay["nw"].max() <= nw_hi


def test_layout_stream_is_uniform():
    """Fixed-seed chi-square on 10^5 lines: length, characters, background, x0, y, fill and dx."""
    from scipy.stats import chisquare
    gen = _gen()
    lay = gen.philox_layout(100000, 777, lens=(4, 6))
    live = np.arange(lay["max_len"])[None, :] < lay["len"][:, None]
    for name, v, a, b in (("len", lay["len"], 4, 6), ("bg", lay["bg"], 180, 255), ("x0", lay["x0"], 2, 12),
                          ("chars", lay["chars"][live], 1, 62), ("y", lay["y"][live], 0, 10), ("fill", lay["fill"][live], 0, 90),
                          ("dx", lay["dx"][live], -2, 3)):
        counts = np.bincount(v - a, minlength=b - a + 1)
        assert counts.size == b - a + 1
        p = chisquare(counts).pvalue
        assert p > 1e-4, (name, p)


def test_seeds_and_lines_draw_distinct_streams():
    gen = _gen()
    a = gen.philox_layout(256, gen.batch_seed(0, 5, 0, 8))
    b = gen.philox_layout(256, gen.batch_seed(0, 5, 1, 8))
    assert not np.array_equal(a["chars"], b["chars"])
    assert len({tuple(r) for r in a["chars"]}) > 250


@pytest.mark.parametrize("name,font", _fonts())
def test_numpy_compositing_matches_draw_bitmap(name, font):
    """Random placements of every glyph, clipped at all four edges, overlapping, at the extreme fills and backgrounds."""
    from PIL import Image, ImageDraw
    gen = _gen()
    g = gen._glyphs(font)
    if not g["fast"]:
        pytest.skip(f"{name}: the cached glyph path is off for this font")
    glyphs, masks = gen.glyph_atlas(font)
    rng = np.random.default_rng(7)
    for t in range(300):
        W = int(rng.integers(20, 200))
        bg = (180, 255, int(rng.integers(180, 256)))[t % 3]
        img = Image.new("L", (W, 60), color=bg)
        d = ImageDraw.Draw(img)
        ref = np.full((60, W), bg, np.uint8)
        for k in range(int(rng.integers(1, 6))):
            c = (t * 5 + k) % 62 if t < 30 else int(rng.integers(0, 62))
            m, ox, oy = atlas_mask(glyphs, masks, c)
            fill = (0, 90, int(rng.integers(0, 91)))[k % 3]
            sx = int(rng.integers(-m.shape[1] - 3, W + 3))
            sy = int(rng.integers(-m.shape[0] - 3, 64)) if t % 2 else int(rng.integers(0, 11)) + oy
            mask, off = g["mask"][gen.cfg.CHARSET[c]]
            d.draw.draw_bitmap((sx, sy), mask, d.draw.draw_ink(fill))
            blend_glyph(ref, m, sx, sy, fill)
        assert np.array_equal(np.asarray(img), ref), (name, t)


def test_host_layouts_compose_as_pil_draws_them():
    gen = _gen()
    font = gen._font(42)
    glyphs, masks = gen.glyph_atlas(font)
    lay = gen.philox_layout(40, 99, lens=(4, 12))
    for i in range(40):
        assert np.array_equal(composite_line(lay, i, glyphs, masks), gen.draw_layout_line(lay, i, font)), i


def test_render_layout_of_render_lines_layout_is_render_line():
    """The layout render_line draws (its rng calls restated into a layout dict) gives render_line's image through render_layout."""
    gen = _gen()
    font = gen._font(42)
    adv = dict(zip(gen.cfg.CHARSET, gen._glyph_adv(font, gen.cfg.CHARSET)))
    for seed in range(12):
        text = gen.gen_rand(random.Random(seed), 3, 9)
        img = gen.render_line(text, rng=random.Random(1000 + seed))
        r = random.Random(1000 + seed)
        bg, x0 = r.randint(180, 255), r.randint(2, 12)
        x, xs, ys, fills = x0, [], [], []
        for ch in text:
            ys.append(r.randint(0, 10)); fills.append(r.randint(0, 90)); xs.append(x)
            x += adv[ch] + r.randint(-2, 3)
        lay = {"len": np.array([len(text)]), "bg": np.array([bg]), "canvas_w": np.array([sum(adv[c] for c in text) + 28]),
               "chars": np.array([[gen.cfg.CHARSET.index(c) + 1 for c in text]]), "x": np.array([xs]), "y": np.array([ys]),
               "fill": np.array([fills])}
        assert np.array_equal(gen.draw_layout_line(lay, 0, font), img), seed
        imgs, lab, ll, tsl = gen.render_layout(lay, font)
        want = gen.groupBatch([img], [text], dtype=np.uint8)
        assert np.array_equal(imgs[0], want[0][0]) and lab == want[1] and ll == want[2] and tsl == want[3]


def test_atlas_refuses_a_font_whose_glyph_path_is_off():
    from PIL import ImageFont
    gen = _gen()
    font = ImageFont.load_default(41)
    g = gen._glyphs(font)
    g["fast"] = False
    try:
        with pytest.raises(ValueError, match="glyph"):
            gen.glyph_atlas(font)
        from lstm_ctc_ocr_b200 import engine
        with pytest.raises(ValueError):
            engine.GlyphAtlas(font, device="cpu")
    finally:
        gen._GLYPHS.pop(id(font), None)


def test_atlas_rows_hold_each_glyphs_mask():
    gen = _gen()
    font = gen._font(42)
    glyphs, masks = gen.glyph_atlas(font)
    assert glyphs.shape == (62, 8) and glyphs.dtype == np.int32
    for c, ch in enumerate(gen.cfg.CHARSET):
        mask, (ox, oy) = font.getmask2(ch, "L", anchor="la", start=(0.0, 0.0))
        w, h = mask.size
        m, gox, goy = atlas_mask(glyphs, masks, c)
        assert (gox, goy) == (ox, oy) and m.shape == (h, w) and glyphs[c, 0] == int(font.getlength(ch))
        assert all(int(m[y, x]) == mask.getpixel((x, y)) for y in range(0, h, 3) for x in range(0, w, 3))


def test_bucket_and_length_arguments_are_checked():
    gen = _gen()
    with pytest.raises(ValueError, match="bucket"):
        gen._render_range(100, None)
    from lstm_ctc_ocr_b200.lib.lstm.train import render_on_device
    assert render_on_device("device") and not render_on_device("host")
    with pytest.raises(ValueError, match="RENDER"):
        render_on_device("gpu")


def test_render_config_key_takes_set_overrides():
    from lstm_ctc_ocr_b200.lib.lstm.config import cfg, cfg_from_list
    assert cfg.RENDER == "host"
    try:
        cfg_from_list(["RENDER", "device"])
        assert cfg.RENDER == "device"
    finally:
        cfg.RENDER = "host"


def test_header_ctypes_and_binding_table_agree_on_the_render_entries():
    from lstm_ctc_ocr_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "crnn_ctc.h")).read(), flags=re.S)
    for name, nargs in (("crnn_render_layout", 11), ("crnn_render_workspace_size", 4), ("crnn_render_lines_u8", 11)):
        m = re.search(r"\bint\s+" + name + r"\s*\(([^;]*)\)\s*;", src)
        assert m, name
        assert len([p for p in m.group(1).split(",") if p.strip()]) == nargs
        assert len(_lib.SIGNATURES[name][1]) == nargs
        assert hasattr(_lib.load(), name)


def test_status_codes_without_touching_the_device():
    """Argument checks come before any launch: null pointers, bad shapes and unsupported limits return without a CUDA call."""
    import ctypes
    from lstm_ctc_ocr_b200 import _lib
    lib = _lib.load()
    p = 256                                                 # never dereferenced: every call below fails its checks first
    assert lib.crnn_render_layout(1, 4, 4, 6, 0, 0, 0, 62, p, p, None) == 1
    assert lib.crnn_render_layout(1, 0, 4, 6, 0, 0, p, 62, p, p, None) == 1
    assert lib.crnn_render_layout(1, 4, 0, 6, 0, 0, p, 62, p, p, None) == 1
    assert lib.crnn_render_layout(1, 4, 7, 6, 0, 0, p, 62, p, p, None) == 1
    assert lib.crnn_render_layout(1, 4, 4, 257, 0, 0, p, 62, p, p, None) == 4
    assert "257" in lib.crnn_last_error().decode()
    assert lib.crnn_render_layout(1, 4, 4, 6, 0, 0, p, 63, p, p, None) == 1
    assert lib.crnn_render_layout(1, 4, 4, 6, 80, 80, p, 62, p, p, None) == 1
    assert lib.crnn_render_layout(1, 4, 4, 6, 0, 82, p, 62, p, p, None) == 1
    n = ctypes.c_size_t()
    assert lib.crnn_render_workspace_size(0, 6, 40, n) == 1
    assert lib.crnn_render_workspace_size(4, 257, 40, n) == 4
    assert lib.crnn_render_workspace_size(4, 6, 40, None) == 1
    assert lib.crnn_render_workspace_size(4, 6, 40, n) == 0 and n.value >= 4 * 60 * (6 * 40 + 28)
    big = n.value
    assert lib.crnn_render_lines_u8(0, 4, 6, p, p, 40, 88, p, big, p, None) == 1
    assert lib.crnn_render_lines_u8(p, 4, 6, p, p, 40, 86, p, big, p, None) == 1
    assert lib.crnn_render_lines_u8(p, 4, 6, p, p, 40, 4, p, big, p, None) == 1
    assert lib.crnn_render_lines_u8(p, 4, 6, p, p, 40, 88, p, big, p + 2, None) == 1
    assert lib.crnn_render_lines_u8(p, 4, 6, p, p, 40, 88, p + 16, big, p, None) == 1
    assert lib.crnn_render_lines_u8(p, 4, 257, p, p, 40, 88, p, big, p, None) == 4
    assert lib.crnn_render_lines_u8(p, 4, 6, p, p, 40, 88, p, big - 1, p, None) == 5


def test_device_entry_points_fail_loudly_without_a_gpu():
    import torch
    from lstm_ctc_ocr_b200 import CrnnError, engine
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(CrnnError):
        engine.render_lines_u8(torch.zeros((4, engine.render_record_ints(6)), dtype=torch.int32), 6, None, 88)
