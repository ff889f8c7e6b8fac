"""Seeded GIF test files, written by Pillow or by hand, shared by the GIF tests: stills and animations that cover disposal 0-3, global and
local colour tables, transparency, interlacing, frames smaller than the screen at odd offsets, minimum code sizes 2-8 and
streams long enough to fill the LZW dictionary.  `golden/g1_head.gif` is the first two frames of caesium-clt's animated sample
`samples/level_1_0/level_2_0/level_3_0/g1.gif` (689x459, gifski output), cut at block boundaries and closed with the trailer."""
import io
import os

import numpy as np
from PIL import Image

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _pal_image(idx, colours):
    im = Image.fromarray(np.ascontiguousarray(idx, np.uint8), "P")
    pal = np.zeros((256, 3), np.uint8)
    pal[:len(colours)] = colours
    im.putpalette(pal.reshape(-1).tolist())
    return im


def _save(frames, **kw):
    buf = io.BytesIO()
    if len(frames) == 1:
        frames[0].save(buf, "GIF", **kw)
    else:
        frames[0].save(buf, "GIF", save_all=True, append_images=frames[1:], **kw)
    return buf.getvalue()


def still(bits, w=37, h=29, seed=0, interlace=False):
    """a still of 2^bits colours (minimum code size max(2, bits))"""
    rng = np.random.default_rng(seed)
    n = 1 << bits
    colours = rng.integers(0, 256, (n, 3))
    idx = (np.add.outer(np.arange(h) // 3, np.arange(w) // 2) + rng.integers(0, 2, (h, w))) % n
    if bits == 8 or interlace:
        return _save([_pal_image(idx, colours)], interlace=interlace, optimize=False)
    # Pillow always codes at minimum code size 8: the smaller sizes come from the hand-written container
    return raw_gif(w, h, [dict(x=0, y=0, idx=idx.astype(np.uint8), table=[tuple(int(v) for v in c) for c in colours], m=max(2, bits))])


def noise(w=160, h=120, seed=1):
    """256 random colours of random pixels: the dictionary fills many times"""
    rng = np.random.default_rng(seed)
    return _save([_pal_image(rng.integers(0, 256, (h, w)), rng.integers(0, 256, (256, 3)))], optimize=False)


def animation(disposal, w=48, h=40, n=5, seed=2, transparency=True, interlace=True, loop=0):
    """frames with a moving square over a textured background, each frame its own palette (local tables)"""
    rng = np.random.default_rng(seed)
    frames = []
    for k in range(n):
        colours = rng.integers(0, 256, (16, 3))
        idx = (np.add.outer(np.arange(h) // 4, np.arange(w) // 4) + k) % 15 + 1
        if transparency:
            idx[(k * 3) % h:(k * 3) % h + 9, :7] = 0
        idx[5 + k:15 + k, 7 + 3 * k:19 + 3 * k] = 15
        frames.append(_pal_image(idx, colours))
    kw = dict(duration=[30 + 10 * k for k in range(n)], loop=loop, disposal=disposal, interlace=interlace, optimize=False)
    if transparency:
        kw["transparency"] = 0
    return _save(frames, **kw)


def repeated(w=30, h=20):
    """an animation with a repeated frame (it is dropped and its delay moves to the previous frame)"""
    a = _pal_image(np.add.outer(np.arange(h), np.arange(w)) % 4, [(255, 0, 0), (0, 255, 0), (0, 0, 255), (9, 9, 9)])
    b = _pal_image((np.add.outer(np.arange(h), np.arange(w)) + 1) % 4, [(255, 0, 0), (0, 255, 0), (0, 0, 255), (9, 9, 9)])
    return _save([a, a.copy(), b, b.copy(), a], duration=[100, 200, 300, 400, 500], loop=3, optimize=False)


def raw_gif(w, h, frames, gct=None, loop=None):
    """hand-written container: frames = [dict(x, y, w, h, table (list of RGB) or None, idx uint8 [h, w], disposal, delay,
    transparent, interlace, m)] with a plain LZW stream (CLEAR + literals) per frame"""
    out = bytearray(b"GIF89a" + bytes([w & 255, w >> 8, h & 255, h >> 8]))
    if gct is not None:
        s = max(0, (len(gct) - 1).bit_length() - 1)
        out += bytes([0x80 | s, 0, 0])
        t = list(gct) + [(0, 0, 0)] * ((2 << s) - len(gct))
        out += bytes(c for rgb in t for c in rgb)
    else:
        out += bytes([0, 0, 0])
    if loop is not None:
        out += b"\x21\xff\x0bNETSCAPE2.0\x03\x01" + bytes([loop & 255, loop >> 8, 0])
    for f in frames:
        t = f.get("transparent")
        out += bytes([0x21, 0xF9, 4, f.get("disposal", 0) << 2 | (t is not None), f.get("delay", 0) & 255, f.get("delay", 0) >> 8, t or 0, 0])
        fh, fw = f["idx"].shape
        flags = 0x40 if f.get("interlace") else 0
        tab = f.get("table")
        if tab is not None:
            s = max(0, (len(tab) - 1).bit_length() - 1)
            flags |= 0x80 | s
        out += bytes([0x2C, f["x"] & 255, f["x"] >> 8, f["y"] & 255, f["y"] >> 8, fw & 255, fw >> 8, fh & 255, fh >> 8, flags])
        if tab is not None:
            t2 = list(tab) + [(0, 0, 0)] * ((2 << s) - len(tab))
            out += bytes(c for rgb in t2 for c in rgb)
        rows = list(range(fh))
        if f.get("interlace"):
            rows = list(range(0, fh, 8)) + list(range(4, fh, 8)) + list(range(2, fh, 4)) + list(range(1, fh, 2))
        seq = np.concatenate([f["idx"][r] for r in rows]) if fh else np.zeros(0, np.uint8)
        m = f.get("m", 8)
        out += bytes([m]) + literal_lzw(seq, m)
    return bytes(out + b"\x3b")


def literal_lzw(seq, m):
    """a valid LZW stream of literals only (CLEAR before the width would grow), sub-blocked"""
    clear, w = 1 << m, m + 1
    bits, nbits, codes = 0, 0, [clear]
    run = 0
    for v in seq:
        if run == (1 << w) - clear - 3:
            codes.append(clear)
            run = 0
        codes.append(int(v))
        run += 1
    codes.append(clear + 1)
    data = bytearray()
    for c in codes:
        bits |= c << nbits
        nbits += w
        while nbits >= 8:
            data.append(bits & 255)
            bits >>= 8
            nbits -= 8
    if nbits:
        data.append(bits & 255)
    out = bytearray()
    for i in range(0, len(data), 255):
        out += bytes([len(data[i:i + 255])]) + data[i:i + 255]
    return bytes(out + b"\x00")


def disposal_mix():
    """disposal 0-3 in one file, frames at odd offsets, a global table and one local table, transparency and interlacing"""
    rng = np.random.default_rng(5)
    gct = [tuple(int(c) for c in rng.integers(0, 256, 3)) for _ in range(8)]
    W, H = 33, 27
    fr = [dict(x=0, y=0, idx=rng.integers(0, 8, (H, W)).astype(np.uint8), disposal=1, delay=7)]
    fr.append(dict(x=3, y=5, idx=rng.integers(0, 8, (9, 11)).astype(np.uint8), disposal=2, delay=9, transparent=3, interlace=True))
    fr.append(dict(x=17, y=1, idx=rng.integers(0, 4, (13, 7)).astype(np.uint8), disposal=3, delay=11, table=[(1, 2, 3), (250, 9, 9), (9, 250, 9), (9, 9, 250)], m=2))
    fr.append(dict(x=1, y=20, idx=rng.integers(0, 8, (6, 31)).astype(np.uint8), disposal=0, delay=13, transparent=0))
    fr.append(dict(x=30, y=24, idx=rng.integers(0, 8, (3, 3)).astype(np.uint8), disposal=2, delay=0))
    fr.append(dict(x=0, y=0, idx=np.zeros((1, 1), np.uint8), disposal=1, delay=5, transparent=0))
    return raw_gif(W, H, fr, gct=gct, loop=2)


def cases():
    """[(name, bytes)]"""
    out = [("still_m%d" % max(2, b), still(b, seed=b)) for b in range(1, 9)]
    out += [("still_interlaced", still(5, w=41, h=35, interlace=True)), ("noise", noise())]
    out += [("anim_disposal%d" % d, animation(d)) for d in range(4)]
    out += [("anim_opaque", animation(1, transparency=False, interlace=False, loop=7)), ("repeated", repeated()), ("disposal_mix", disposal_mix())]
    with open(os.path.join(GOLDEN, "g1_head.gif"), "rb") as f:
        out.append(("g1", f.read()))
    return out
