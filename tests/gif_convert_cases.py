"""Rules of the GIF conversions restated in numpy for the tests: the canvas a converted source becomes (alpha 0 -> clear, any other
alpha -> opaque), frame 0 of a GIF source as the image crate reads it (built on gifutil's independent parser), and GIF sources
whose frame 0 covers transparency, offsets, local and global tables, interlacing and every minimum code size."""
import numpy as np

import gif_cases
import gifutil


def canvas(rgba):
    """uint8 [h, w, 4] -> the GIF canvas [h, w, 4]: all zero where alpha is 0, else (R, G, B, 255)"""
    rgba = np.asarray(rgba, np.uint8)
    out = rgba.copy()
    out[..., 3] = 255
    out[rgba[..., 3] == 0] = 0
    return np.ascontiguousarray(out)


def twin(rgba, q):
    """the file a conversion to GIF must write: the GIF leg's twin on the one-frame canvas, delay 0, no loop count"""
    from oracle import gif as G
    return G.gif_encode(canvas(rgba)[None], [0], -1, q)


def first_frame(data):
    """frame 0 of a GIF -> uint8 [H, W, 4]: inside its rectangle the palette colour with alpha 0 for the transparent index and
    255 otherwise, all zero outside"""
    info = gifutil.parse(data)
    f = info["frames"][0]
    out = np.zeros((info["height"], info["width"], 4), np.uint8)
    rgb = f["table"][f["indices"]]
    alpha = np.full(f["indices"].shape, 255, np.uint8)
    if f["transparent"] is not None:
        alpha[f["indices"] == f["transparent"]] = 0
    out[f["y"]:f["y"] + f["h"], f["x"]:f["x"] + f["w"]] = np.concatenate([rgb, alpha[..., None]], axis=2)
    return out


def sources():
    """[(name, GIF bytes)]: the GIF leg's test files plus frames 0 that are small, offset, transparent over a non-black colour,
    interlaced with a local table, or opaque"""
    rng = np.random.default_rng(7)
    gct = [(200, 100, 50), (1, 2, 3), (250, 250, 250), (0, 0, 0)]
    out = list(gif_cases.cases())
    out.append(("offset_transparent_global", gif_cases.raw_gif(23, 17, [
        dict(x=5, y=3, idx=rng.integers(0, 4, (9, 11)).astype(np.uint8), transparent=0, m=2),
        dict(x=0, y=0, idx=rng.integers(0, 4, (17, 23)).astype(np.uint8))], gct=gct, loop=0)))
    out.append(("interlaced_local", gif_cases.raw_gif(19, 21, [
        dict(x=2, y=1, idx=rng.integers(0, 16, (19, 13)).astype(np.uint8), table=[tuple(int(v) for v in c) for c in rng.integers(0, 256, (16, 3))],
             transparent=9, interlace=True, m=4)], gct=gct)))
    out.append(("opaque_global", gif_cases.raw_gif(31, 9, [dict(x=0, y=0, idx=rng.integers(0, 4, (9, 31)).astype(np.uint8), m=3)], gct=gct)))
    return out
