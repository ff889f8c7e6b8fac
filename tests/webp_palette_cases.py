"""Few-colour test images of the lossless WebP palette tests (test_webp_palette_host.py, test_webp_palette_gpu.py)."""
import numpy as np


def coloured(h, w, k, seed, alpha="opaque"):
    """h x w RGBA of exactly min(k, h * w) distinct colours.  alpha: 'opaque', 'translucent' (random alpha) or 'hidden' (half the
    colours fully transparent, each with its own RGB)"""
    rng = np.random.default_rng(seed)
    cols = rng.integers(0, 256, (k, 4), dtype=np.uint8)
    if alpha == "opaque":
        cols[:, 3] = 255
    elif alpha == "hidden":
        cols[::2, 3] = 0
        cols[1::2, 3] = 255
    while len(np.unique(cols.view(np.uint32))) < k:
        cols[:, :3] = rng.integers(0, 256, (k, 3), dtype=np.uint8)
    idx = rng.integers(0, k, h * w)
    if h * w >= k:
        idx[:k] = rng.permutation(k)
    return cols[idx].reshape(h, w, 4)


def two_colour_bitmap(h, w):
    yy, xx = np.mgrid[:h, :w]
    on = ((xx // 7 + yy // 5) % 3 == 0) | (np.hypot(xx - w / 2, yy - h / 2) < min(h, w) / 3)
    img = np.zeros((h, w, 4), np.uint8)
    img[on] = (20, 20, 30, 255)
    img[~on] = (250, 245, 240, 255)
    return img


def sprite_sheet(h, w, seed=4):
    """16 colours (one transparent) in 16 x 16 sprites drawn at random over a transparent sheet"""
    rng = np.random.default_rng(seed)
    cols = np.concatenate([rng.integers(0, 256, (15, 4), dtype=np.uint8), np.zeros((1, 4), np.uint8)])
    cols[:15, 3] = 255
    sprites = rng.integers(0, 16, (6, 16, 16))
    img = np.zeros((h, w, 4), np.uint8)
    for y in range(0, h - 15, 16):
        for x in range(0, w - 15, 16):
            img[y:y + 16, x:x + 16] = cols[sprites[rng.integers(0, 6)]]
    return img
