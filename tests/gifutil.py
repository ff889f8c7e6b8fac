"""An independent pure-Python GIF reader for the tests: container, LZW, interlace, gif-dispose compositing (the canvas starts
clear; disposal 2 clears the frame's rectangle, disposal 3 restores the canvas from before the frame), delays and loop count.
Canvases are uint8 [h, w, 4] with alpha 0 or 255 and clear pixels all zero."""
import numpy as np


class GifError(ValueError):
    pass


def _blocks(d, pos):
    out = bytearray()
    while True:
        if pos >= len(d):
            raise GifError("truncated sub-blocks")
        n = d[pos]
        pos += 1
        if n == 0:
            return bytes(out), pos
        if pos + n > len(d):
            raise GifError("truncated sub-block")
        out += d[pos:pos + n]
        pos += n


def lzw_decode(data, m, npix):
    """GIF LZW image data (sub-blocks joined) -> npix indices (bytes); extra codes after the last pixel are ignored."""
    clear, eoi = 1 << m, (1 << m) + 1
    table = [bytes([i]) for i in range(clear)] + [b"", b""]
    w, prev, out = m + 1, None, bytearray()
    acc, nacc, pos = 0, 0, 0
    while len(out) < npix:
        while nacc < w and pos < len(data):
            acc |= data[pos] << nacc
            nacc += 8
            pos += 1
        if nacc < w:
            break
        code = acc & ((1 << w) - 1)
        acc >>= w
        nacc -= w
        if code == clear:
            table = table[:clear + 2]
            w, prev = m + 1, None
            continue
        if code == eoi:
            break
        if prev is None:
            if code >= clear:
                raise GifError("bad first code")
            out += table[code]
            prev = table[code]
            continue
        if code < len(table):
            cur = table[code]
        elif code == len(table) and len(table) < 4096:
            cur = prev + prev[:1]
        else:
            raise GifError("code past the dictionary")
        out += cur
        if len(table) < 4096:
            table.append(prev + cur[:1])
            if len(table) == (1 << w) and w < 12:
                w += 1
        prev = cur
    if len(out) < npix:
        raise GifError("image data too short")
    return bytes(out[:npix])


def _rows(h, interlaced):
    if not interlaced:
        return list(range(h))
    return list(range(0, h, 8)) + list(range(4, h, 8)) + list(range(2, h, 4)) + list(range(1, h, 2))


def parse(data):
    """-> dict(width, height, loop (None when absent), frames=[dict(x, y, w, h, disposal, delay, transparent, interlaced,
    table uint8 [n, 3], min_code_size, indices uint8 [h, w])])"""
    d = bytes(data)
    if len(d) < 13 or d[:6] not in (b"GIF87a", b"GIF89a"):
        raise GifError("not a GIF")
    W, H, flags = d[6] | d[7] << 8, d[8] | d[9] << 8, d[10]
    pos, gct = 13, None
    if flags & 0x80:
        n = 2 << (flags & 7)
        if pos + 3 * n > len(d):
            raise GifError("truncated global table")
        gct = np.frombuffer(d[pos:pos + 3 * n], np.uint8).reshape(n, 3)
        pos += 3 * n
    res = dict(width=W, height=H, loop=None, frames=[])
    gce = None
    while True:
        if pos >= len(d):
            raise GifError("no trailer")
        b = d[pos]
        pos += 1
        if b == 0x3B:
            return res
        if b == 0x21:
            if pos >= len(d):
                raise GifError("truncated extension")
            label = d[pos]
            pos += 1
            body, pos2 = _blocks(d, pos)
            if label == 0xF9:
                if d[pos] < 4:
                    raise GifError("short graphic control extension")
                f = body[0]
                gce = dict(disposal=(f >> 2) & 7, delay=body[1] | body[2] << 8, transparent=body[3] if f & 1 else None)
            elif label == 0xFF and d[pos] == 11 and body[:11] == b"NETSCAPE2.0" and d[pos + 12] == 3 and body[11] == 1:
                res["loop"] = body[12] | body[13] << 8
            pos = pos2
        elif b == 0x2C:
            if pos + 9 > len(d):
                raise GifError("truncated descriptor")
            x, y, w, h = (d[pos + k] | d[pos + k + 1] << 8 for k in (0, 2, 4, 6))
            f = d[pos + 8]
            pos += 9
            table = gct
            if f & 0x80:
                n = 2 << (f & 7)
                if pos + 3 * n > len(d):
                    raise GifError("truncated local table")
                table = np.frombuffer(d[pos:pos + 3 * n], np.uint8).reshape(n, 3)
                pos += 3 * n
            if table is None:
                raise GifError("no colour table")
            if pos >= len(d):
                raise GifError("truncated image data")
            m = d[pos]
            if not 2 <= m <= 8:
                raise GifError("minimum code size out of range")
            data, pos = _blocks(d, pos + 1)
            idx = np.frombuffer(lzw_decode(data, m, w * h), np.uint8).reshape(h, w)
            if idx.size and int(idx.max()) >= len(table):
                raise GifError("index past the colour table")
            rows = _rows(h, bool(f & 0x40))
            ordered = np.zeros_like(idx)
            for k, r in enumerate(rows):
                ordered[r] = idx[k]
            g = gce or dict(disposal=0, delay=0, transparent=None)
            res["frames"].append(dict(x=x, y=y, w=w, h=h, disposal=g["disposal"], delay=g["delay"], transparent=g["transparent"],
                                      interlaced=bool(f & 0x40), table=table, min_code_size=m, indices=ordered))
            gce = None
        else:
            raise GifError("unknown block")


def composite(info):
    """-> (list of (canvas uint8 [H, W, 4], delay), loop or None)"""
    W, H = info["width"], info["height"]
    canvas = np.zeros((H, W, 4), np.uint8)
    out, prev, saved = [], None, None
    for fr in info["frames"]:
        if prev is not None:
            if prev["disposal"] == 2:
                canvas[prev["y"]:prev["y"] + prev["h"], prev["x"]:prev["x"] + prev["w"]] = 0
            elif prev["disposal"] == 3 and saved is not None:
                canvas = saved
        saved = canvas.copy() if fr["disposal"] == 3 else None
        x, y, w, h = fr["x"], fr["y"], fr["w"], fr["h"]
        if x + w > W or y + h > H:
            raise GifError("frame past the logical screen")
        rgba = np.concatenate([fr["table"][fr["indices"]], np.full((h, w, 1), 255, np.uint8)], axis=2)
        draw = np.ones((h, w), bool) if fr["transparent"] is None else fr["indices"] != fr["transparent"]
        region = canvas[y:y + h, x:x + w]
        region[draw] = rgba[draw]
        out.append((canvas.copy(), fr["delay"]))
        prev = fr
    return out, info["loop"]


def decode(data):
    """-> (list of (canvas, delay), loop or None)"""
    return composite(parse(data))
