"""numpy restatement of the device renderer's compositing (csrc/render.cu render_composite_kernel): a glyph mask blended into a
gray canvas as Pillow's fill_mask_L (ImagingFill2, behind ImageDraw's draw_bitmap) blends it, clipped to the canvas."""
import numpy as np


def div255(v):
    v = np.asarray(v, np.int64) + 128
    return ((v >> 8) + v) >> 8


def blend_glyph(canvas, mask, sx, sy, fill):
    """Blend `mask` (h x w uint8) into `canvas` (rows x cols uint8, in place) with its top-left corner at column sx, row sy:
    out = DIV255(out * (255 - m) + fill * m) on the pixels the mask and the canvas share."""
    H, W = canvas.shape
    h, w = mask.shape
    r0, r1 = max(sy, 0), min(sy + h, H)
    c0, c1 = max(sx, 0), min(sx + w, W)
    if r0 >= r1 or c0 >= c1:
        return canvas
    m = mask[r0 - sy:r1 - sy, c0 - sx:c1 - sx].astype(np.int64)
    out = canvas[r0:r1, c0:c1].astype(np.int64)
    canvas[r0:r1, c0:c1] = div255(out * (255 - m) + int(fill) * m).astype(np.uint8)
    return canvas


def atlas_mask(glyphs, masks, c):
    """Charset index c's mask from gen.glyph_atlas's arrays, as an h x w array, and its (ox, oy)."""
    adv, w, h, ox, oy, off = (int(v) for v in glyphs[c, :6])
    return masks[off:off + w * h].reshape(h, w), ox, oy


def composite_line(layout, i, glyphs, masks):
    """Line i of a layout (gen.philox_layout's dict) composited in numpy from the atlas arrays: the 60-row canvas."""
    canvas = np.full((60, int(layout["canvas_w"][i])), int(layout["bg"][i]), np.uint8)
    for j in range(int(layout["len"][i])):
        m, ox, oy = atlas_mask(glyphs, masks, int(layout["chars"][i, j]) - 1)
        blend_glyph(canvas, m, int(layout["x"][i, j]) + ox, int(layout["y"][i, j]) + oy, int(layout["fill"][i, j]))
    return canvas
