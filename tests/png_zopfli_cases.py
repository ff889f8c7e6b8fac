"""Seeded inputs for the PNG `--zopfli` tests: images (photograph, flat art, text, noise, one pixel wide) as raw rows, their filtered
streams, and streams at the segment and slice boundaries."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SEG, SLICE = 32768, 8 << 20


def photo(w, h, seed=0):
    from tools.synth import synth_rgb
    return synth_rgb(w, h, seed)


def flat(w, h, seed=1):
    """few-colour rectangles and ellipses on white"""
    from PIL import Image, ImageDraw
    rng = np.random.default_rng(seed)
    im = Image.new("RGB", (w, h), (255, 255, 255))
    d = ImageDraw.Draw(im)
    for _ in range(24):
        x0, y0 = int(rng.integers(0, w)), int(rng.integers(0, h))
        x1, y1 = x0 + int(rng.integers(4, max(5, w // 3))), y0 + int(rng.integers(4, max(5, h // 3)))
        col = tuple(int(c) for c in rng.choice([0, 64, 128, 200, 255], 3))
        (d.rectangle if rng.random() < 0.5 else d.ellipse)([x0, y0, x1, y1], fill=col)
    return np.asarray(im)


def text(w, h, seed=2):
    """lines of words in Pillow's built-in default font"""
    from PIL import Image, ImageDraw
    rng = np.random.default_rng(seed)
    words = ["lorem", "ipsum", "dolor", "sit", "amet", "pixel", "kernel", "deflate", "parse", "0123", "cost", "segment"]
    im = Image.new("RGB", (w, h), (250, 250, 250))
    d = ImageDraw.Draw(im)
    for y in range(2, h - 10, 12):
        d.text((4, y), " ".join(rng.choice(words, 12)), fill=(0, 0, 0))
    return np.asarray(im)


def noise(w, h, seed=3):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)


def images(scale=1):
    """name -> uint8 [h, w, 3]"""
    return {"photo": photo(64 * scale, 48 * scale), "flat": flat(96 * scale, 64 * scale), "text": text(160 * scale, 40 * scale),
            "noise": noise(40 * scale, 30 * scale), "one_wide": photo(1, 200 * scale)[:, :1]}


def filtered(img, strategy=0):
    """the image's rows filtered by the oracle with one strategy -> (stream, bpp, stride)"""
    from oracle import oracle as O
    h, w, c = img.shape
    raw = np.ascontiguousarray(img).reshape(h, w * c)
    return O.png_filter(raw, c, strategy).reshape(-1), c, w * c + 1


def boundary_stream(n, seed=4):
    """n bytes with repeats at short and long range (so matches meet the segment end), filter distance 3, stride 301"""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 16, 4096, dtype=np.uint8)
    reps = np.tile(base, n // base.size + 1)[:n].copy()
    flip = rng.random(n) < 0.05
    reps[flip] = rng.integers(0, 256, int(flip.sum()), dtype=np.uint8)
    return reps, 3, 301
