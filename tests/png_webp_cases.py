"""PNG sources for the lossless WebP conversion tests: every colour type x legal bit depth, with and without tRNS, framed with
pngutil.frame_png (filter byte 0, random bits in the padding of sub-byte rows), and a numpy restatement of the pixels the conversion
must code (the lossy PNG -> WebP conversion's rule: palette lookup with black past PLTE, sub-byte greys scaled v * 255 / (2^bd - 1),
16-bit samples by their high byte, tRNS colour keys compared at full precision)."""
import zlib

import numpy as np

from pngutil import chunk, frame_png

CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}


def row_bytes(w, ct, bd):
    return (w * CHANNELS[ct] * bd + 7) // 8


def samples(raw, w, ct, bd):
    """un-filtered rows uint8 [h, row_bytes] -> full-precision samples int64 [h, w, channels]"""
    raw = np.asarray(raw, np.uint8)
    h, nc = raw.shape[0], CHANNELS[ct]
    if bd == 16:
        b = raw[:, :2 * w * nc].astype(np.int64)
        s = b[:, 0::2] << 8 | b[:, 1::2]
    elif bd == 8:
        s = raw[:, :w * nc].astype(np.int64)
    else:
        bits = np.unpackbits(raw, axis=1)[:, :w * nc * bd].reshape(h, w * nc, bd).astype(np.int64)
        s = (bits << np.arange(bd - 1, -1, -1)).sum(axis=2)
    return s.reshape(h, w, nc)


def expected_rgba(raw, w, ct, bd, plte=b"", trns=b""):
    """the RGBA uint8 [h, w, 4] the conversion codes for these rows"""
    s = samples(raw, w, ct, bd)
    eight = (s >> 8) if bd == 16 else (s * 255 // ((1 << bd) - 1)) if bd < 8 else s
    h = s.shape[0]
    out = np.full((h, w, 4), 255, np.int64)
    if ct == 3:
        pal = np.zeros((256, 4), np.int64); pal[:, 3] = 255
        p = np.frombuffer(plte, np.uint8).reshape(-1, 3)
        pal[:len(p), :3] = p
        t = np.frombuffer(trns, np.uint8)
        pal[:len(t), 3] = t
        out = pal[s[..., 0]]
    elif ct == 0:
        out[..., :3] = eight[..., :1]
        if len(trns) >= 2:
            out[..., 3] = np.where(s[..., 0] == (trns[0] << 8 | trns[1]), 0, 255)
    elif ct == 2:
        out[..., :3] = eight
        if len(trns) >= 6:
            key = np.array([trns[0] << 8 | trns[1], trns[2] << 8 | trns[3], trns[4] << 8 | trns[5]])
            out[..., 3] = np.where((s == key).all(axis=2), 0, 255)
    elif ct == 4:
        out[..., :3] = eight[..., :1]; out[..., 3] = eight[..., 1]
    else:
        out = eight
    return out.astype(np.uint8)


def make_case(w, h, ct, bd, seed=0, trns=None, plte_len=None):
    """(file bytes, raw rows, plte, trns): random samples; trns='key' takes the first pixel's value as the colour key, 'partial'
    gives the first palette entries soft alphas; plte_len shorter than 2^bd leaves indices past PLTE"""
    rng = np.random.default_rng(seed)
    rb = row_bytes(w, ct, bd)
    raw = rng.integers(0, 256, (h, rb), dtype=np.uint8)
    if ct in (0, 2) and bd == 8 and trns == "key":      # a few repeats of the first pixel, so that the key hits more than once
        nc = CHANNELS[ct]
        for y, x in ((h // 2, w // 2), (h - 1, w - 1)):
            raw[y, x * nc:(x + 1) * nc] = raw[0, :nc]
    plte, t = b"", b""
    extra = b""
    if ct == 3:
        n = plte_len if plte_len is not None else 1 << bd
        plte = rng.integers(0, 256, 3 * n, dtype=np.uint8).tobytes()
        extra += chunk(b"PLTE", plte)
        if trns == "partial":
            t = bytes([0, 128, 255, 7][:max(1, min(4, n - 1))])
    elif trns == "key":
        s = samples(raw[:1], 1, ct, bd)[0, 0]
        t = b"".join(int(v).to_bytes(2, "big") for v in s)
    if t:
        extra += chunk(b"tRNS", t)
    filt = np.concatenate([np.zeros((h, 1), np.uint8), raw], axis=1)
    data = frame_png(w, h, bd, ct, zlib.compress(filt.tobytes(), 6), extra)
    return data, raw, plte, t


def cases():
    """(id, w, h, ct, bd, trns, plte_len) for every colour type x depth and tRNS form, at odd and degenerate sizes"""
    out = []
    for ct, depths in DEPTHS.items():
        for bd in depths:
            forms = [None]
            if ct in (0, 2):
                forms.append("key")
            if ct == 3:
                forms += ["partial", "short"]
            for form in forms:
                for (w, h) in ((13, 7), (1, 1), (1, 9), (11, 1)):
                    plte_len = max(1, (1 << bd) - 3) if form == "short" else None
                    out.append((f"ct{ct}_bd{bd}_{form or 'plain'}_{w}x{h}", w, h, ct, bd, "partial" if form == "short" else form, plte_len))
    return out
