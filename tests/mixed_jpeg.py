"""Same-shaped baseline JPEG files that differ in everything but their shape, for the megabatch tests (not a fixture: imported by
the test modules).

A megabatch (b200_compress_batch) and the resident pipe run K images of one shape through one launch sequence, and a CUDA graph
replays that sequence while only counts, high-water sizes and buffer addresses stay the same.  Everything else is per image: the
Huffman tables and selectors the decoder stages, the dequantisation tables chosen through each image's own tq map, the component
ids, quantisation precision and marker segments the file assembly copies.  variants() builds, from one picture, files that share
width, height and sampling factors and differ in exactly those things:

- most are header rewrites of a Pillow (libjpeg-turbo) file -- table ids, selectors, component ids, table precision, segment order
  and merging, fill bytes, APPn segments, trailing bytes -- so the entropy-coded data is the original's;
- some are fresh Pillow encodes (other qualities, optimised Huffman tables, custom quantisation tables and tq maps);
- some are coded here by encode_scan(): quantisation tables above 255 (the original's tables scaled, the coefficients divided
  to match), Huffman tables the device decoder's lookup pool cannot hold, and a periodic stream the device decoder cannot
  synchronise within its round budget.

Every variant is pinned to libjpeg-turbo by the test module test_megabatch_mixed_host.py: its native YCbCr decode through Pillow
must equal the oracle's, and a header rewrite must decode exactly like the file it came from.  So a test that compares the
product with the oracle on these files cannot agree with a mis-read header."""
import functools
import io
import os
import sys
from dataclasses import dataclass

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

W, H = 322, 199
ZZ = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
               35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])
SOF0, SOF1, DHT, DQT, SOS = 0xC0, 0xC1, 0xC4, 0xDB, 0xDA


# ---- a parsed single-scan baseline file ------------------------------------------------------------------------------------------
@dataclass
class Parsed:
    apps: list                  # [(marker, payload)] APPn / COM in file order
    dqt: list                   # [(pq, tq, 64 values in zigzag order)]
    dht: list                   # [(tc, th, bits[1..16], vals)]
    sof: int                    # SOF marker (0xC0 / 0xC1)
    comps: list                 # [(cid, h, v, tq)]
    sel: list                   # [(cid, td, ta)] in scan order
    ecs: bytes
    tail: bytes = b"\xff\xd9"
    width: int = W
    height: int = H


def parse(data):
    """A baseline single-scan file -> Parsed (the entropy-coded segment ends at the first marker that is not RSTn)."""
    assert data[:2] == b"\xff\xd8"
    p = Parsed([], [], [], 0, [], [], b"")
    i = 2
    while True:
        while data[i + 1] == 0xFF:
            i += 1
        assert data[i] == 0xFF
        m, n = data[i + 1], int.from_bytes(data[i + 2:i + 4], "big")
        seg = data[i + 4:i + 2 + n]
        i += 2 + n
        if m == DQT:
            k = 0
            while k < len(seg):
                pq, tq = seg[k] >> 4, seg[k] & 15
                w = 2 if pq else 1
                vals = [int.from_bytes(seg[k + 1 + w * z:k + 1 + w * z + w], "big") for z in range(64)]
                p.dqt.append((pq, tq, vals)); k += 1 + 64 * w
        elif m == DHT:
            k = 0
            while k < len(seg):
                bits = list(seg[k + 1:k + 17]); nv = sum(bits)
                p.dht.append((seg[k] >> 4, seg[k] & 15, bits, list(seg[k + 17:k + 17 + nv]))); k += 17 + nv
        elif m in (SOF0, SOF1):
            p.sof, p.height, p.width = m, int.from_bytes(seg[1:3], "big"), int.from_bytes(seg[3:5], "big")
            p.comps = [(seg[6 + 3 * c], seg[7 + 3 * c] >> 4, seg[7 + 3 * c] & 15, seg[8 + 3 * c]) for c in range(seg[5])]
        elif m == SOS:
            p.sel = [(seg[1 + 2 * k], seg[2 + 2 * k] >> 4, seg[2 + 2 * k] & 15) for k in range(seg[0])]
            j = i
            while not (data[j] == 0xFF and data[j + 1] != 0 and not 0xD0 <= data[j + 1] <= 0xD7):
                j += 1
            p.ecs, p.tail = data[i:j], data[j:]
            return p
        else:
            p.apps.append((m, seg))


def _seg(m, payload, fill=0):
    return b"\xff" * fill + bytes([0xFF, m]) + (len(payload) + 2).to_bytes(2, "big") + bytes(payload)


def dqt_payload(tables):
    out = bytearray()
    for pq, tq, vals in tables:
        out.append((pq << 4) | tq)
        for v in vals:
            out += v.to_bytes(2, "big") if pq else bytes([v])
    return bytes(out)


def dht_payload(tables):
    out = bytearray()
    for tc, th, bits, vals in tables:
        out.append((tc << 4) | th); out += bytes(bits) + bytes(vals)
    return bytes(out)


def build(p, dqt_merged=False, dht_merged=False, dqt_after_sof=False, dht_before_sof=False, fill=0):
    """Parsed -> file.  The default layout is libjpeg's (one DQT / DHT segment per table, DQT before SOF, DHT after it), so
    build(parse(f)) == f for a Pillow file.  `fill` 0xFF bytes go in front of every marker of the header."""
    dqt = [_seg(DQT, dqt_payload(p.dqt), fill)] if dqt_merged else [_seg(DQT, dqt_payload([t]), fill) for t in p.dqt]
    dht = [_seg(DHT, dht_payload(p.dht), fill)] if dht_merged else [_seg(DHT, dht_payload([t]), fill) for t in p.dht]
    sof = bytearray([8]) + p.height.to_bytes(2, "big") + p.width.to_bytes(2, "big") + bytes([len(p.comps)])
    for cid, h, v, tq in p.comps:
        sof += bytes([cid, (h << 4) | v, tq])
    sos = bytearray([len(p.sel)])
    for cid, td, ta in p.sel:
        sos += bytes([cid, (td << 4) | ta])
    sos += bytes([0, 63, 0])
    out = b"\xff\xd8" + b"".join(_seg(m, s, fill) for m, s in p.apps)
    out += b"".join(dht if dht_before_sof else []) + b"".join([] if dqt_after_sof else dqt)
    out += _seg(p.sof, sof, fill) + b"".join(dqt if dqt_after_sof else []) + b"".join([] if dht_before_sof else dht)
    return out + _seg(SOS, sos, fill) + p.ecs + p.tail


def rewrite(data, fn, **layout):
    p = parse(data)
    fn(p)
    return build(p, **layout)


# ---- a baseline encoder with caller-chosen Huffman tables --------------------------------------------------------------------------
def _codes(bits, vals):
    """Canonical Huffman codes (ITU T.81 Annex C): symbol -> (code, length)."""
    out, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            out[vals[k]] = (code, length); code += 1; k += 1
        code <<= 1
    return out


def _nbits(v):
    return int(abs(int(v))).bit_length()


def encode_scan(coefs, comps, tables):
    """One interleaved baseline scan.  coefs[c]: [bh, bw, 64] natural order, whole MCUs (the oracle's layout); comps[c] = (h, v);
    tables[c] = (dc (bits, vals), ac (bits, vals)).  Returns the stuffed entropy-coded bytes."""
    dcc = [_codes(*t[0]) for t in tables]
    acc = [_codes(*t[1]) for t in tables]
    zz = [np.ascontiguousarray(c.reshape(-1, 64)[:, ZZ]).reshape(c.shape) for c in coefs]
    single = len(coefs) == 1
    mcuy, mcux = (zz[0].shape[0], zz[0].shape[1]) if single else (zz[0].shape[0] // comps[0][1], zz[0].shape[1] // comps[0][0])
    out, pred = [], [0] * len(coefs)

    def put(code, length):
        out.append(format(code, "0%db" % length))

    def put_value(v, s):
        if s:
            put(v if v >= 0 else v + (1 << s) - 1, s)
    for my in range(mcuy):
        for mx in range(mcux):
            for c, (h, v) in enumerate([(1, 1)] if single else comps):
                for by in range(v):
                    for bx in range(h):
                        blk = zz[c][my * v + by, mx * h + bx].tolist()
                        d = blk[0] - pred[c]; pred[c] = blk[0]
                        s = _nbits(d); put(*dcc[c][s]); put_value(d, s)
                        run = 0
                        for k in range(1, 64):
                            a = blk[k]
                            if a == 0:
                                run += 1
                                continue
                            while run > 15:
                                put(*acc[c][0xF0]); run -= 16
                            s = _nbits(a); put(*acc[c][(run << 4) | s]); put_value(a, s); run = 0
                        if run:
                            put(*acc[c][0x00])
    s = "".join(out)
    s += "1" * (-len(s) % 8)
    raw = int(s, 2).to_bytes(len(s) // 8, "big") if s else b""
    return raw.replace(b"\xff", b"\xff\x00")


# ---- sources -------------------------------------------------------------------------------------------------------------------------
KINDS = ("420", "444", "grey")
PIL_SUB = {"420": "4:2:0", "444": "4:4:4"}


@functools.lru_cache(maxsize=None)
def _pixels(kind):
    from PIL import Image
    from tools.synth import synth_rgb
    im = Image.fromarray(synth_rgb(W, H, 31), "RGB")
    return im.convert("L") if kind == "grey" else im


def pillow(kind, **kw):
    b = io.BytesIO()
    kw.setdefault("quality", 75)
    if kind != "grey":
        kw.setdefault("subsampling", PIL_SUB[kind])
    _pixels(kind).save(b, "JPEG", **kw)
    return b.getvalue()


def _custom_table(seed, lo, hi):
    rng = np.random.default_rng(seed)
    base = np.add.outer(np.arange(8), np.arange(8)).reshape(64)            # grows with frequency, like the Annex K tables
    return [int(v) for v in np.clip(lo + base * (hi - lo) // 14 + rng.integers(0, 4, 64), 1, 255)]


def _icc_segment():
    body = b"ICC_PROFILE\x00\x01\x01" + bytes(range(256)) * 2       # chunk 1 of 1; content need not be a real profile
    return (0xE2, body)


def _exif_segment():
    tiff = b"MM\x00\x2a\x00\x00\x00\x08\x00\x01\x01\x12\x00\x03\x00\x00\x00\x01\x00\x06\x00\x00\x00\x00\x00\x00"
    return (0xE1, b"Exif\x00\x00" + tiff)


def _set_density(p, units, x, y):
    for k, (m, s) in enumerate(p.apps):
        if m == 0xE0 and s[:5] == b"JFIF\x00":
            p.apps[k] = (m, s[:7] + bytes([units]) + x.to_bytes(2, "big") + y.to_bytes(2, "big") + s[12:])


def _renumber_huff(p, ids):
    """Huffman table id t becomes ids[t] (DHT and SOS alike)."""
    p.dht = [(tc, ids[th], bits, vals) for tc, th, bits, vals in p.dht]
    p.sel = [(cid, ids[td], ids[ta]) for cid, td, ta in p.sel]


def _renumber_quant(p, ids):
    p.dqt = [(pq, ids[tq], vals) for pq, tq, vals in p.dqt]
    p.comps = [(cid, h, v, ids[tq]) for cid, h, v, tq in p.comps]


def _set_cids(p, cids):
    m = {old: new for (old, _, _, _), new in zip(p.comps, cids)}
    p.comps = [(m[cid], h, v, tq) for cid, h, v, tq in p.comps]
    p.sel = [(m[cid], td, ta) for cid, td, ta in p.sel]


def _own(kind, coefs, dqt, tables, sof=SOF1, sel=None):
    """A file coded by encode_scan() over the header of the kind's Pillow file, with the given quantisation and Huffman tables."""
    p = parse(pillow(kind))
    p.sof, p.dqt = sof, dqt
    comps = [(h, v) for _, h, v, _ in p.comps]
    sel = sel or [(i, i) for i in range(len(p.comps))]                  # (td, ta) per component
    p.sel = [(cid, td, ta) for (cid, _, _, _), (td, ta) in zip(p.comps, sel)]
    p.dht = []
    for c, (td, ta) in enumerate(sel):
        if all(t[:2] != (0, td) for t in p.dht):
            p.dht.append((0, td) + tuple(tables[c][0]))
        if all(t[:2] != (1, ta) for t in p.dht):
            p.dht.append((1, ta) + tuple(tables[c][1]))
    p.ecs = encode_scan(coefs, comps, tables)
    return build(p)


def _annex_k(kind):
    """The Annex K (dc, ac) tables of each component of the kind's Pillow file."""
    p = parse(pillow(kind))
    get = {(tc, th): (bits, vals) for tc, th, bits, vals in p.dht}
    return [(get[(0, td)], get[(1, ta)]) for _, td, ta in p.sel]


def _scaled_tables(kind, k):
    """The kind's q75 file with every quantisation table multiplied by k (k = 7: luma up to 427, chroma up to 350, Pq = 1) and
    every coefficient divided by k, rounded: dequantised values stay near the original's, far below 2^15."""
    from oracle import oracle as O
    src = pillow(kind)
    j = O.Jpeg(src)
    coefs = []
    for c in range(j.ncomp):
        a = j.coef(c).astype(np.int32)
        coefs.append((np.sign(a) * ((np.abs(a) + k // 2) // k)).astype(np.int16))
    dqt = [(1, tq, [v * k for v in vals]) for _, tq, vals in parse(src).dqt]
    return _own(kind, coefs, dqt, _annex_k(kind))


# code-length profiles that need many second-level lookup entries (a 9-bit prefix with codes up to 16 bits below it costs 128):
# the AC profile of test_gpudec.py's adversarial tables (368 entries), and a DC profile of 16 symbols that costs 260
ADVERSARIAL_AC = {1: 1, 10: 24, 11: 48, 12: 60, 13: 40, 14: 30, 15: 20, 16: 33}
ADVERSARIAL_DC = {1: 1, 10: 1, 11: 4, 12: 2, 13: 3, 14: 1, 15: 1, 16: 3}


def _refused_tables(kind):
    """Every component codes with its own pair of adversarial tables (Td/Ta 0, 1, 2 under SOF1): six of them need 1884 entries
    of the device decoder's second-level pool, which holds 1536, so the device refuses the table set and the host decodes."""
    from oracle import oracle as O
    src = pillow(kind)
    j = O.Jpeg(src)
    tables = []
    for c in range(j.ncomp):
        rng = np.random.default_rng(c)                               # each component's symbols on different codes
        dc = ([ADVERSARIAL_DC.get(l, 0) for l in range(1, 17)], [int(v) for v in rng.permutation(16)])
        ac = ([ADVERSARIAL_AC.get(l, 0) for l in range(1, 17)], [int(v) for v in rng.permutation(256)])
        tables.append((dc, ac))
    return _own(kind, [j.coef(c) for c in range(j.ncomp)], parse(src).dqt, tables)


def _periodic(kind):
    """A stream with period one MCU that never synchronises by itself: every block holds the same 40 +-1 AC coefficients and DC
    difference 0, so a decoder started at a wrong bit keeps its wrong phase, and the device decoder's rounds can only correct one
    subsequence after the other (over 100 of them here, against a budget of 24 rounds): the image goes to the host decoder."""
    from oracle import oracle as O
    j = O.Jpeg(pillow(kind))
    coefs = []
    for c in range(j.ncomp):
        a = np.zeros_like(j.coef(c))
        a[..., ZZ[1:41]] = np.where(np.arange(40) % 3 == 0, -1, 1)
        coefs.append(a)
    return _own(kind, coefs, parse(pillow(kind)).dqt, _annex_k(kind), sof=SOF0, sel=[(0, 0)] + [(1, 1)] * (j.ncomp - 1))


@dataclass
class Variant:
    name: str
    data: bytes
    origin: bytes = None            # the file this one is a header rewrite of: both must decode alike
    pipe: bool = True               # the resident pipe accepts it (a device-decodable file, walked on the host)
    settles: bool = True            # the device decoder settles it (else the image goes to the host decoder)


@functools.lru_cache(maxsize=None)
def variants(kind):
    """The variants of one picture, all W x H with the kind's sampling factors."""
    grey = kind == "grey"
    base = pillow(kind)
    ncomp = 1 if grey else 3
    out = [Variant("annex_k_q75", base)]
    for q in (50, 92):
        out.append(Variant(f"q{q}", pillow(kind, quality=q)))
    out.append(Variant("q100_long_codes", pillow(kind, quality=100)))
    out.append(Variant("optimised_q30", pillow(kind, quality=30, optimize=True)))
    out.append(Variant("optimised_q95", pillow(kind, quality=95, optimize=True)))
    t0, t1, t2 = _custom_table(1, 3, 60), _custom_table(2, 9, 120), _custom_table(3, 5, 200)
    out.append(Variant("custom_qtables", pillow(kind, qtables=[t0] if grey else [t0, t1])))
    if not grey:
        out.append(Variant("one_qtable_tq000", pillow(kind, qtables=[t1])))
        out.append(Variant("three_qtables_tq012", pillow(kind, qtables=[t0, t1, t2])))

    def rw(name, fn=lambda p: None, **layout):
        out.append(Variant(name, rewrite(base, fn, **layout), origin=base))

    rw("unused_extra_qtable", lambda p: p.dqt.append((0, 3, _custom_table(4, 1, 255))))
    rw("qtables_16bit_sof1", lambda p: (setattr(p, "dqt", [(1, tq, v) for _, tq, v in p.dqt]), setattr(p, "sof", SOF1)))
    out.append(Variant("qtables_above_255_sof1", _scaled_tables(kind, 7)))
    rw("qtable_ids_swapped", lambda p: _renumber_quant(p, {0: 1, 1: 0}))
    rw("qtable_ids_2_3", lambda p: _renumber_quant(p, {0: 3, 1: 2}))
    rw("huff_selectors_swapped", lambda p: _renumber_huff(p, {0: 1, 1: 0}))
    rw("huff_ids_2_3_sof1", lambda p: (_renumber_huff(p, {0: 2, 1: 3}), setattr(p, "sof", SOF1)))
    rw("component_ids_0_1_2", lambda p: _set_cids(p, [0, 1, 2][:ncomp]))
    rw("component_ids_odd", lambda p: _set_cids(p, [200, 7, 99][:ncomp]))
    rw("no_jfif", lambda p: setattr(p, "apps", [a for a in p.apps if a[0] != 0xE0]))
    rw("jfif_300dpi", lambda p: _set_density(p, 1, 300, 300))
    rw("jfif_aspect_3_2", lambda p: _set_density(p, 0, 3, 2))
    rw("exif_and_icc", lambda p: p.apps.extend([_exif_segment(), _icc_segment()]))
    rw("tables_merged", dqt_merged=True, dht_merged=True)
    rw("tables_moved_across_sof", dqt_after_sof=True, dht_before_sof=True)
    rw("tables_merged_and_moved", dqt_merged=True, dht_merged=True, dqt_after_sof=True, dht_before_sof=True)
    rw("fill_bytes_before_markers", fill=3)
    rw("trailing_garbage", lambda p: setattr(p, "tail", p.tail + bytes(np.random.default_rng(5).integers(0, 0xFF, 300, dtype=np.uint8))))
    # a multi-picture camera file: the host walk stops at the first EOI; a megabatch, which takes the segment to end at the file's
    # last EOI, meets the second picture's markers inside it and hands the file to the host decoder
    rw("second_jpeg_appended", lambda p: setattr(p, "tail", p.tail + pillow("grey", quality=40)))
    # the host walk meets 0xFF fill in front of EOI and hands the file to the host decoder: not for the resident pipe
    out.append(Variant("fill_bytes_before_eoi", rewrite(base, lambda p: setattr(p, "tail", b"\xff\xff" + p.tail)), origin=base, pipe=False))
    if not grey:                # (one component has too few tables to overflow the pool, and its periodic stream settles at once)
        out.append(Variant("huff_tables_refused", _refused_tables(kind), settles=False))
        out.append(Variant("periodic_stream", _periodic(kind), settles=False))
    return tuple(out)
