"""Seeded animated WebP fixtures (nothing is committed): animations written by Pillow, RIFF files assembled by hand from Pillow's
still VP8 / VP8L payloads to reach every compositing rule, and corrupt variants of the hand-built files.  Also an independent
reader of the container that decodes each frame with Pillow, for the twin."""
import io
import struct

import numpy as np
from PIL import Image

NO_BLEND, DISPOSE_BG = 2, 1


def _chunks(data, start=12, end=None):
    end = len(data) if end is None else end
    out, i = [], start
    while i + 8 <= end:
        tag, size = data[i:i + 4], struct.unpack("<I", data[i + 4:i + 8])[0]
        out.append((tag, data[i + 8:i + 8 + size]))
        i += 8 + size + (size & 1)
    return out


def _chunk(tag, payload):
    return tag + struct.pack("<I", len(payload)) + payload + (b"\0" if len(payload) & 1 else b"")


def rgba_image(rng, w, h, alpha="mixed"):
    px = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    # smooth parts too, so the lossy coder has something to keep
    px[: h // 2, :, :3] = (np.arange(w)[None, :, None] * 7 + np.arange(h // 2)[:, None, None] * 3 + np.array([0, 60, 120])) % 256
    if alpha == "opaque":
        px[..., 3] = 255
    elif alpha == "mixed":
        px[..., 3] = rng.choice(np.array([0, 255, 1, 128, 254, 77], np.uint8), (h, w))
    return px


def still_payload(rgba, lossless, quality=80):
    """the image sub-chunks (ALPH + 'VP8 ', or VP8L) of Pillow's still WebP of rgba, as bytes"""
    im = Image.fromarray(np.ascontiguousarray(rgba), "RGBA")
    if not lossless and (rgba[..., 3] == 255).all():
        im = im.convert("RGB")
    b = io.BytesIO()
    im.save(b, "WEBP", lossless=lossless, quality=quality, exact=True, method=4)
    parts = [(t, p) for t, p in _chunks(b.getvalue()) if t in (b"ALPH", b"VP8 ", b"VP8L")]
    return b"".join(_chunk(t, p) for t, p in parts)


def assemble(width, height, frames, loop=0, bg=b"\x00\x00\x00\x00", alpha_flag=True):
    """frames: [(x, y, w, h, duration, flags, image sub-chunks)] -> an animated WebP file"""
    body = _chunk(b"VP8X", bytes([0x02 | (0x10 if alpha_flag else 0), 0, 0, 0]) + (width - 1).to_bytes(3, "little") + (height - 1).to_bytes(3, "little"))
    body += _chunk(b"ANIM", bytes(bg) + struct.pack("<H", loop))
    for x, y, w, h, dur, flags, sub in frames:
        head = (x // 2).to_bytes(3, "little") + (y // 2).to_bytes(3, "little") + (w - 1).to_bytes(3, "little") + (h - 1).to_bytes(3, "little")
        body += _chunk(b"ANMF", head + int(dur).to_bytes(3, "little") + bytes([flags]) + sub)
    return b"RIFF" + struct.pack("<I", 4 + len(body)) + b"WEBP" + body


def read_frames(data):
    """independent reader: -> (W, H, loop, bg, [(x, y, flags, has_alpha, rgba [h, w, 4], duration)]), each frame decoded by Pillow
    from a still file made of its sub-chunks"""
    top = _chunks(data, 12, 8 + struct.unpack("<I", data[4:8])[0])
    vp8x = dict(top)[b"VP8X"]
    W, H = 1 + int.from_bytes(vp8x[4:7], "little"), 1 + int.from_bytes(vp8x[7:10], "little")
    anim = dict(top)[b"ANIM"]
    out = []
    for tag, p in top:
        if tag != b"ANMF":
            continue
        x, y = 2 * int.from_bytes(p[0:3], "little"), 2 * int.from_bytes(p[3:6], "little")
        dur, flags = int.from_bytes(p[12:15], "little"), p[15] & 3
        sub = [(t, q) for t, q in _chunks(p, 16) if t in (b"ALPH", b"VP8 ", b"VP8L")]
        tags = [t for t, _ in sub]
        if b"VP8L" in tags:
            has_alpha = bool((int.from_bytes(dict(sub)[b"VP8L"][1:5], "little") >> 28) & 1)
            w = 1 + (int.from_bytes(dict(sub)[b"VP8L"][1:5], "little") & 0x3FFF)
            h = 1 + ((int.from_bytes(dict(sub)[b"VP8L"][1:5], "little") >> 14) & 0x3FFF)
            still = b"WEBP" + _chunk(b"VP8L", dict(sub)[b"VP8L"])
        else:
            v = dict(sub)[b"VP8 "]
            w, h = int.from_bytes(v[6:8], "little") & 0x3FFF, int.from_bytes(v[8:10], "little") & 0x3FFF
            has_alpha = b"ALPH" in tags
            x8 = _chunk(b"VP8X", bytes([0x10 if has_alpha else 0, 0, 0, 0]) + (w - 1).to_bytes(3, "little") + (h - 1).to_bytes(3, "little"))
            still = b"WEBP" + x8 + b"".join(_chunk(t, q) for t, q in sub)
        still = b"RIFF" + struct.pack("<I", len(still)) + still
        rgba = np.asarray(Image.open(io.BytesIO(still)).convert("RGBA"))
        out.append((x, y, flags, has_alpha, rgba, dur))
    return W, H, int.from_bytes(anim[4:6], "little"), bytes(anim[:4]), out


def pillow_frames(data):
    """Pillow's composited frames (WebPAnimDecoder) as RGBA, and their durations"""
    im = Image.open(io.BytesIO(data))
    canv, durs = [], []
    for k in range(im.n_frames):
        im.seek(k)
        canv.append(np.asarray(im.convert("RGBA")))
        durs.append(im.info.get("duration", 0))
    return np.stack(canv), durs


def pillow_cases(seed=7):
    """animations written by Pillow: lossy and lossless, with and without alpha, with moving sub-rectangles and repeats"""
    rng = np.random.default_rng(seed)
    out = {}
    for lossless in (False, True):
        for alpha in ("opaque", "mixed"):
            base = rgba_image(rng, 48, 36, alpha)
            ims = []
            for k in range(6):
                f = base.copy()
                f[5 + k:15 + k, 4 + 3 * k:20 + 3 * k] = rgba_image(rng, 16, 10, alpha)
                if k == 3:
                    f = ims[-1]
                ims.append(f)
            pil = [Image.fromarray(f, "RGBA") if alpha != "opaque" else Image.fromarray(f[..., :3].copy(), "RGB") for f in ims]
            b = io.BytesIO()
            pil[0].save(b, "WEBP", save_all=True, append_images=pil[1:], duration=[40, 0, 70, 70, 100, 33], loop=3, lossless=lossless,
                        quality=75, exact=True, kmin=2, kmax=4)
            out[f"pillow_{'lossless' if lossless else 'lossy'}_{alpha}"] = b.getvalue()
    return out


def hand_cases(seed=11):
    """hand-assembled files covering every compositing rule"""
    rng = np.random.default_rng(seed)
    out = {}
    W, H = 40, 30
    full = lambda alpha="mixed", lossless=True: still_payload(rgba_image(rng, W, H, alpha), lossless)
    part = lambda w, h, alpha="mixed", lossless=True: still_payload(rgba_image(rng, w, h, alpha), lossless)
    # every blend x dispose pair on the middle frame, with a blending frame after it that overlaps it
    for blend in (0, 1):
        for dispose in (0, 1):
            flags = (0 if blend else NO_BLEND) | (DISPOSE_BG if dispose else 0)
            out[f"pair_b{blend}_d{dispose}"] = assemble(W, H, [
                (0, 0, W, H, 50, 0, full("opaque")),
                (4, 6, 20, 12, 60, flags, part(20, 12)),
                (10, 2, 22, 22, 70, 0, part(22, 22)),
                (0, 0, 16, 16, 80, flags, part(16, 16, lossless=False)),
            ])
    # overlapping and edge-touching rectangles, lossy frames with and without ALPH
    out["edges"] = assemble(W, H, [
        (0, 0, W, H, 10, 0, full("mixed", lossless=False)),
        (W - 8, H - 6, 8, 6, 20, 0, part(8, 6, lossless=False)),
        (0, H - 4, W, 4, 30, DISPOSE_BG, part(W, 4)),
        (W - 2, 0, 2, H, 40, 0, part(2, H, "opaque", lossless=False)),
        (2, 2, W - 2, H - 2, 50, 0, part(W - 2, H - 2)),
    ])
    # keyframes: a full opaque blend frame; a full no-blend frame with alpha; after a full frame disposed to background; after a
    # keyframe disposed to background; and a full blend frame with alpha, which is not one
    out["key_full_opaque"] = assemble(W, H, [(0, 0, W, H, 10, 0, full()), (0, 0, W, H, 10, 0, full("opaque", lossless=False)), (6, 6, 10, 10, 10, 0, part(10, 10))])
    out["key_full_noblend"] = assemble(W, H, [(0, 0, W, H, 10, 0, full()), (0, 0, W, H, 10, NO_BLEND, full()), (6, 6, 10, 10, 10, 0, part(10, 10))])
    out["key_after_full_dispose"] = assemble(W, H, [(0, 0, W, H, 10, DISPOSE_BG, full()), (4, 4, 12, 12, 10, DISPOSE_BG, part(12, 12)),
                                                    (8, 8, 20, 20, 10, 0, part(20, 20)), (0, 0, 10, 10, 10, 0, part(10, 10))])
    out["not_key_full_blend"] = assemble(W, H, [(0, 0, W, H, 10, 0, full()), (0, 0, W, H, 10, 0, full()), (2, 2, 6, 6, 10, DISPOSE_BG, part(6, 6)),
                                                (0, 0, 8, 8, 10, 0, part(8, 8))])
    # odd canvas, 1x1 frames, the background colour (not painted) and the largest loop count
    out["odd_1x1"] = assemble(17, 13, [(4, 2, 1, 1, 5, 0, part(1, 1)), (16, 12, 1, 1, 5, 0, part(1, 1, "opaque", lossless=False)),
                                       (0, 0, 17, 13, 5, DISPOSE_BG, still_payload(rgba_image(rng, 17, 13), True)), (2, 2, 1, 1, 5, 0, part(1, 1))],
                              loop=65535, bg=b"\x10\x20\x30\x40")
    out["one_pixel_canvas"] = assemble(1, 1, [(0, 0, 1, 1, 7, 0, part(1, 1)), (0, 0, 1, 1, 9, 0, part(1, 1))])
    # repeated canvases and durations at both ends of the 24-bit range
    a, b = full("opaque"), part(8, 8, "opaque")
    out["repeats_durations"] = assemble(W, H, [(0, 0, W, H, 0, 0, a), (0, 0, W, H, (1 << 24) - 1, 0, a), (0, 0, W, H, (1 << 24) - 2, 0, a),
                                               (4, 4, 8, 8, 0, 0, b), (4, 4, 8, 8, 0, 0, b), (4, 4, 8, 8, 12, 0, b)], loop=0)
    return out


def corrupt_cases(seed=13):
    """(name, bytes) of damaged hand-built files, each of which must answer code 4"""
    rng = np.random.default_rng(seed)
    px = still_payload(rgba_image(rng, 8, 6), True)
    good = assemble(16, 12, [(0, 0, 8, 6, 10, 0, px), (8, 6, 8, 6, 10, 0, px)])
    out = [
        ("outside", assemble(16, 12, [(0, 0, 8, 6, 10, 0, px), (10, 6, 8, 6, 10, 0, px)])),
        ("size_mismatch", assemble(16, 12, [(0, 0, 8, 6, 10, 0, px), (0, 0, 9, 6, 10, 0, px)])),
        ("canvas_too_wide", assemble(16384, 12, [(0, 0, 8, 6, 10, 0, px)])),
        ("no_frames", assemble(16, 12, [])),
        ("riff_too_long", good[:4] + struct.pack("<I", len(good)) + good[8:]),
    ]
    for cut in (20, 30, 45, 60, len(good) - 40, len(good) - 3):
        out.append((f"truncated_{cut}", good[:4] + struct.pack("<I", cut - 8) + good[8:cut]))
    # ANMF that claims more than the file holds
    i = good.index(b"ANMF")
    out.append(("anmf_overrun", good[:i + 4] + struct.pack("<I", 10 ** 6) + good[i + 8:]))
    return good, out
