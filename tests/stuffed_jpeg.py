"""Valid baseline JPEGs whose entropy-coded segments are dense in stuffed bytes (0xFF 0x00 pairs).

Photographic scans hold a stuffed pair in roughly every hundredth byte.  Here every coefficient is +-(2^k - 1): a positive value's
magnitude bits are a run of ones, and the rare long symbols of an optimised Huffman table are runs of ones too, so a large share of
the bytes comes out 0xFF and gets a stuffed zero behind it.  k and the signs are seeded per coefficient so that the stream is not
periodic (a periodic stream need not self-synchronise, and then the device decoder rightly hands it to the host).  The layout is
that of a Pillow file of the shape; the host encoder (L.jpeg_encode_coefficients, sequential) writes the file."""
import io

import numpy as np
from PIL import Image

SUBSAMPLING = {"420": "4:2:0", "444": "4:4:4", "422": "4:2:2", "grey": None}


def pillow_layout(L, kind, w, h):
    rgb = np.zeros((h, w, 3), np.uint8)
    b = io.BytesIO()
    if kind == "grey":
        Image.fromarray(rgb[:, :, 0], "L").save(b, "JPEG", quality=95)
    else:
        Image.fromarray(rgb, "RGB").save(b, "JPEG", quality=95, subsampling=SUBSAMPLING[kind])
    return L.jpeg_decode_coefficients(b.getvalue())


def dense_coefficients(lay, seed, ac_per_block=(24, 63), last_extra=0):
    """coefficients of `lay` (zigzag, block after block): DC +-(2^k - 1), k <= 10, and a seeded number of AC coefficients +-(2^k - 1),
    k <= 10, mostly positive, at seeded zigzag positions.  last_extra changes the last block only (to move the scan's length)."""
    rng = np.random.default_rng(seed)
    nblk = lay.total_coefs // 64
    co = np.zeros((nblk, 64), np.int16)

    def runs(shape, kmax, p_neg):
        k = rng.integers(1, kmax + 1, shape)
        return (((1 << k) - 1) * np.where(rng.random(shape) < p_neg, -1, 1)).astype(np.int16)

    co[:, 0] = runs(nblk, 10, 0.5)
    n_ac = rng.integers(ac_per_block[0], ac_per_block[1] + 1, nblk)
    vals = runs((nblk, 63), 10, 0.15)
    keep = rng.random((nblk, 63)).argsort(axis=1) < n_ac[:, None]      # n_ac seeded positions per block
    co[:, 1:] = np.where(keep, vals, 0)
    if last_extra:
        co[-1, 1:] = 0
        co[-1, 1:1 + last_extra % 63] = 1
    return co.reshape(-1)


def dense_jpeg(L, kind, w, h, seed, **kw):
    """(file bytes, layout, coefficients) of a dense baseline file"""
    lay, _ = pillow_layout(L, kind, w, h)
    co = dense_coefficients(lay, seed, **kw)
    return L.jpeg_encode_coefficients(lay, co, False), lay, co


def real_blocks(lay, co):
    """the blocks inside the image (rbw x rbh per component): a re-encoder writes the MCU padding blocks as it likes (libjpeg: zero
    AC, the DC of the block before)"""
    out = []
    for c in range(lay.ncomp):
        blk = co[lay.comp_offset[c]:lay.comp_offset[c] + lay.bw[c] * lay.bh[c] * 64].reshape(lay.bh[c], lay.bw[c], 64)
        out.append(blk[:lay.rbh[c], :lay.rbw[c]])
    return out


def same_coefficients(L, data, lay, co):
    """the file `data` holds the coefficients co (of layout lay) in every block inside the image"""
    lay2, co2 = L.jpeg_decode_coefficients(data)
    a, b = real_blocks(lay, co), real_blocks(lay2, co2)
    return len(a) == len(b) and all(x.shape == y.shape and np.array_equal(x, y) for x, y in zip(a, b))


def scan_bounds(data):
    """(first byte of the entropy-coded segment, position of the EOI that ends it)"""
    sos = data.index(b"\xff\xda")
    return sos + 2 + int.from_bytes(data[sos + 2:sos + 4], "big"), data.rindex(b"\xff\xd9")


def stuffing_density(data):
    """share of the entropy-coded segment's bytes that are stuffed pairs"""
    s, e = scan_bounds(data)
    seg = data[s:e]
    return 2 * seg.count(b"\xff\x00") / max(len(seg), 1)


def with_fill(data, n):
    """n fill bytes 0xFF in front of the EOI (T.81 B.1.1.2: any marker may be preceded by fill bytes)"""
    e = data.rindex(b"\xff\xd9")
    return data[:e] + b"\xff" * n + data[e:]


def with_trailer(data, junk=b"\x00\xff\xd9garbage\xff\x00\xff"):
    """bytes after the EOI"""
    return data + junk


SHAPES = [(w, h) for w, h in ((1, 1), (17, 9), (355, 237), (640, 480))]
KINDS = ["420", "444", "422", "grey"]


def dense_corpus(L):
    """name -> (file, layout, coefficients): every kind at every shape, and 4:2:0 355x237 files whose last block is varied until
    the scan lengths have covered all 16 residues mod 16"""
    out = {}
    for kind in KINDS:
        for i, (w, h) in enumerate(SHAPES):
            out[f"{kind}_{w}x{h}"] = dense_jpeg(L, kind, w, h, 1000 + 10 * KINDS.index(kind) + i)
    seen = set()
    for extra in range(1, 400):
        if len(seen) == 16:
            break
        data, lay, co = dense_jpeg(L, "420", 355, 237, 77, last_extra=extra)
        s, e = scan_bounds(data)
        r = (e - s) % 16
        if r not in seen:
            seen.add(r)
            out[f"420_355x237_len_mod16_{r}"] = (data, lay, co)
    return out
