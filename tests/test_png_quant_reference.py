"""The lossy PNG quantiser against pq_reference.py, a plain restatement of the rules in png_quant_core.h's header comment that
shares no code with the header, its scalar twin (oracle/png_quant_oracle.c) or the device.

CPU: the reference equals the twin on a corpus that reaches premultiplication rounding, clamped targets, nearest-entry ties and the
256 / 257 distinct-value boundary, and both pass check_dither (every index re-derived as the exhaustive nearest entry of its target).
GPU: the device equals the reference bit for bit on that corpus, across the shapes where the dither wavefront changes behaviour
(one row, one column, widths around the 32-pixel steps and the 64-entry ring, heights around the 32-row groups), on targets spread
over about 20,000 candidate-grid cells and on palettes with entries on cell edges, at the exact-path boundary with colliding hash
slots, and in a batch; and equals the twin at large shapes."""
import functools

import numpy as np
import pytest

import pq_reference as R
from oracle.png_quant import png_quantize as twin_quantize
from pngutil import pil_pixels, pil_png, synth

QUALITIES = [0, 1, 40, 80, 93, 94, 100]


def opaque(rgb):
    return np.concatenate([rgb, np.full(rgb.shape[:2] + (1,), 255, np.uint8)], 2)


def gradient(h=40, w=72):
    y, x = np.mgrid[0:h, 0:w]
    return np.stack([x * 255 // (w - 1), y * 255 // (h - 1), (x + 2 * y) % 256, 255 - (x * y) % 64], -1).astype(np.uint8)


def alpha_ramp(h=36, w=49):
    """every alpha the premultiplication rounds differently at (0, 1, 2, 127, 128, 254, 255), one per column, under noise"""
    img = synth(h, w, 4, seed=21, kind="noise")
    img[:, :, 3] = np.array([0, 1, 2, 127, 128, 254, 255], np.uint8)[np.arange(w) % 7]
    return img


def saturated(h=40, w=48):
    """channels within 4 of 0 or 255, so the diffused error pushes targets past the ends and the clamp decides them"""
    rng = np.random.default_rng(22)
    v = rng.integers(0, 4, (h, w, 3))
    return opaque(np.where(rng.integers(0, 2, (h, w, 3)) == 1, 255 - v, v).astype(np.uint8))


def premul_ties(h=32, w=40):
    """alpha 1, 2, 17 and 34 under random colour: hundreds of source values premultiply to few coordinates on a coarse lattice, so
    at q = 100 dozens of targets sit at equal distance from two entries and the tie rule decides the index"""
    rng = np.random.default_rng(23)
    img = rng.integers(0, 256, (h, w, 4)).astype(np.uint8)
    img[:, :, 3] = np.array([1, 2, 17, 34], np.uint8)[rng.integers(0, 4, (h, w))]
    return img


def distinct_values(n, h=24, w=30):
    """exactly n distinct values (transparent ones among them), the k-th first at pixel k, the rest cycling"""
    k = np.arange(n)
    vals = np.stack([k & 255, (k * 7 + 3) & 255, (k >> 3) * 13 & 255, np.where(k % 5 == 0, 0, 255 - (k % 3) * 60)], -1)
    return vals[np.arange(h * w) % n].reshape(h, w, 4).astype(np.uint8)


def photo_hole():
    img = opaque(synth(48, 64, 3, seed=0))
    img[20:26, 30:37] = (200, 30, 90, 0)
    return img


CORPUS = {
    "photo": lambda: opaque(synth(48, 64, 3, seed=0)),
    "photo_hole": photo_hole,
    "soft_alpha": lambda: synth(40, 52, 4, seed=3),
    "flat": lambda: opaque(synth(40, 56, 3, seed=1, kind="flat")),
    "noise": lambda: synth(32, 40, 4, seed=5, kind="noise"),
    "gradient": gradient,
    "alpha_ramp": alpha_ramp,
    "saturated": saturated,
    "premul_ties": premul_ties,
    "distinct_255": lambda: distinct_values(255),
    "distinct_256": lambda: distinct_values(256),
    "distinct_257": lambda: distinct_values(257),
}


@functools.lru_cache(maxsize=None)
def reference(case, q):
    return R.png_quantize_ref(CORPUS[case](), q)


def assert_same(img, got, want, what):
    """palette and indices equal; else the first differing pixel, with its reference target"""
    gp, gi = got
    wp, wi = want
    assert np.array_equal(gp, wp), f"{what}: palettes differ ({len(gp)} vs {len(wp)} entries)"
    bad = np.argwhere(gi != wi)
    if len(bad):
        y, x = bad[0]
        res = R.check_dither(img, wp, wi)
        tgt = tuple(res[0][y, x]) if res else "exact path"
        pytest.fail(f"{what}: {len(bad)} indices differ, first at (x={x}, y={y}): {gi[y, x]} vs {wi[y, x]}, target {tgt}")


# ---- CPU: the reference, the twin and the definition ------------------------------------------------------------------------------

def test_target_mse_table_is_the_formula():
    """2000 * ((100 - q) / 100)^3 rounded, and 0 from q = 94 up"""
    import os
    import re
    with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "caesium-clt_b200", "csrc", "png_quant_core.h")) as f:
        body = re.search(r"pq_target_mse\[101\] = \{([^}]*)\}", f.read()).group(1)
    assert [int(v) for v in body.replace("\n", " ").split(",")] == R.TARGET_MSE
    assert R.TARGET_MSE[93] > 0 and R.TARGET_MSE[94] == 0


@pytest.mark.parametrize("q", QUALITIES)
@pytest.mark.parametrize("case", sorted(CORPUS))
def test_reference_equals_the_twin(case, q):
    img = CORPUS[case]()
    want = reference(case, q)
    assert_same(img, twin_quantize(img, q), want, "twin")
    R.check_dither(img, *want)


def test_corpus_reaches_its_edges():
    """the corpus exercises what it is there for: the clamp, the tie rule, every alpha class, and both sides of 256 values"""
    sat = R.check_dither(saturated(), *reference("saturated", 1))
    assert sat[1] > 100
    ti = CORPUS["premul_ties"]()
    assert R.ties(ti, reference("premul_ties", 100)[0], R.check_dither(ti, *reference("premul_ties", 100))[0]) > 10
    assert R.ties(CORPUS["photo"](), reference("photo", 80)[0], R.check_dither(CORPUS["photo"](), *reference("photo", 80))[0]) > 10
    assert len(reference("distinct_256", 40)[0]) == 256 and R.check_dither(distinct_values(256), *reference("distinct_256", 40)) is None
    assert R.check_dither(distinct_values(257), *reference("distinct_257", 40)) is not None
    p = R.premultiply(alpha_ramp())
    assert set(np.unique(p[:, :, 3])) == {0, 1, 2, 127, 128, 254, 255}


def test_check_dither_rejects_a_wrong_index():
    """check_dither is a real check: moving one pixel to its second-nearest entry is caught, at that pixel"""
    img = CORPUS["photo"]()
    pal, idx = reference("photo", 40)
    tgt, _ = R.check_dither(img, pal, idx)
    coords = np.array([R.entry_coords(tuple(int(v) for v in e)) for e in pal])
    d = ((coords - tgt[10, 17]) ** 2).sum(1)
    bad = idx.copy()
    bad[10, 17] = np.argsort(d, kind="stable")[1]
    with pytest.raises(AssertionError, match=r"pixel \(17, 10\)"):
        R.check_dither(img, pal, bad)


def test_reference_rounding_rules():
    """the rules written out: premultiplication rounds to nearest (c * a % 255 == 127 rounds down, 128 up); a palette entry is the
    rounded mean (halves up), un-premultiplied with rounding; the incoming dither error rounds half away from zero"""
    assert R.premultiply(np.array([127, 1, 128, 1], np.uint8))[0] == 0            # 127 / 255 < 1/2
    assert R.premultiply(np.array([128, 1, 0, 1], np.uint8))[0] == 1              # 128 / 255 > 1/2
    assert R.entry_rgba([3, 0, 0, 8], 2) == (128, 0, 0, 4)                         # mean 1.5 -> 2 at alpha 4: 127.5 -> 128
    assert R.entry_rgba([1, 0, 0, 6], 2) == (85, 0, 0, 3)                          # 0.5 -> 1 at alpha 3: 255 / 3
    # a grey 8 halfway between entries 0 and 16 goes to the lower index, and its error of +-8 reaches the next pixel as
    # 7 * 8 / 16 = 3.5, rounded away from zero
    idx, tgt = R.dither(opaque(np.array([[[8] * 3, [0] * 3]], np.uint8)), [(0, 0, 0, 255), (16, 16, 16, 255)])
    assert idx.tolist() == [[0, 0]] and tuple(tgt[0, 1]) == (4, 4, 4, 255)
    idx, tgt = R.dither(opaque(np.array([[[8] * 3, [20] * 3]], np.uint8)), [(16, 16, 16, 255), (0, 0, 0, 255)])
    assert idx.tolist() == [[0, 0]] and tuple(tgt[0, 1]) == (16, 16, 16, 255)


# ---- GPU: the device against the reference ----------------------------------------------------------------------------------------

def noise_with_hole(h, w, seed):
    img = synth(h, w, 4, seed=seed, kind="noise")
    img[:, :, 3] |= 1                                               # the hole is the only transparent area
    img[h // 3: h // 3 + max(1, h // 4), w // 2: w // 2 + max(1, w // 5), 3] = 0
    return img


SWEEP_H = [1, 2, 31, 32, 33, 63, 64, 65, 97]
SWEEP_W = [1, 2, 3, 31, 32, 33, 63, 64, 65, 127, 129]
# shapes of more than 256 pixels with one row or column, or one dimension just past a 32-step: the sweep above reaches these
# only with at most 256 distinct values (the exact path)
LONG = [(1, 300), (1, 1000), (1, 4097), (300, 1), (2, 257), (3, 131), (129, 2), (257, 3), (33, 1025)]


@pytest.mark.gpu
@pytest.mark.parametrize("q", QUALITIES)
@pytest.mark.parametrize("case", sorted(CORPUS))
def test_device_equals_the_reference(L, case, q):
    img = CORPUS[case]()
    assert_same(img, L.png_quantize(img, q), reference(case, q), "device")


@pytest.mark.gpu
@pytest.mark.parametrize("h", SWEEP_H)
def test_device_shape_sweep(L, h):
    for w in SWEEP_W:
        img = noise_with_hole(h, w, seed=h * 1000 + w)
        assert_same(img, L.png_quantize(img, 40), R.png_quantize_ref(img, 40), f"{w}x{h}")


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", LONG)
def test_device_long_shapes(L, h, w):
    img = noise_with_hole(h, w, seed=h * 7 + w)
    assert_same(img, L.png_quantize(img, 40), R.png_quantize_ref(img, 40), f"{w}x{h}")


def grid_source():
    """256 x 256 pixels whose premultiplied values run through every combination of four 4-bit cell coordinates, each colour nibble
    capped at the alpha nibble (a premultiplied colour never exceeds alpha), at a random position inside the cell"""
    rng = np.random.default_rng(31)
    y, x = np.mgrid[0:256, 0:256]
    nib = np.stack([y >> 4, y & 15, x >> 4, x & 15], -1)
    nib[..., :3] = np.minimum(nib[..., :3], nib[..., 3:])
    pm = nib * 16 + rng.integers(0, 16, (256, 256, 4))
    pm[..., 3] = np.maximum(pm[..., 3], 1)
    pm[..., :3] = np.minimum(pm[..., :3], pm[..., 3:])
    # the least straight colour c with round(c * a / 255) >= pm; that rounding climbs in steps of at most one, so it equals pm
    c = np.maximum(0, -(-((2 * pm[..., :3] - 1) * 255) // (2 * pm[..., 3:])))
    img = np.concatenate([c, pm[..., 3:]], -1).astype(np.uint8)
    assert np.array_equal(R.premultiply(img), pm)
    return img


def edge_source(seed):
    """a few colours on candidate-cell edges (0, 15, 16, 239, 240, 255) in blocks, plus a sparse scatter of random values: the
    palette gets entries exactly on the edges and the scatter's error walks targets across them"""
    rng = np.random.default_rng(seed)
    edges = np.array([0, 15, 16, 239, 240, 255])
    cols = np.concatenate([edges[rng.integers(0, 6, (6, 3))], np.full((6, 1), 255)], 1)
    # translucent white premultiplies to (a, a, a, a): entries on the edges in alpha too
    cols = np.r_[cols, [[255, 255, 255, a] for a in (15, 16, 239, 240)]]
    img = cols[(np.arange(96)[:, None] // 12 + np.arange(128)[None, :] // 16) % 10]
    m = rng.random((96, 128)) < 0.06
    img[m] = rng.integers(0, 256, (int(m.sum()), 4))
    return img.astype(np.uint8)


@pytest.mark.gpu
@pytest.mark.parametrize("q", [1, 40, 100])
def test_device_grid_coverage(L, q):
    img = grid_source()
    want = R.png_quantize_ref(img, q)
    tgt, _ = R.check_dither(img, *want)
    t = tgt.reshape(-1, 4) >> 4
    # Targets are premultiplied values plus diffused error, so a colour above alpha needs large error; the source visits about
    # 19,600 to 19,900 of the 65,536 cells (about 18,500 have no colour nibble above the alpha nibble), not all of them.
    visited = set((t[:, 0] << 12 | t[:, 1] << 8 | t[:, 2] << 4 | t[:, 3]).tolist())
    assert len(visited) > 19000
    assert_same(img, L.png_quantize(img, q), want, f"grid q={q}")


@pytest.mark.gpu
@pytest.mark.parametrize("q", [1, 40, 100])
@pytest.mark.parametrize("seed", [41, 42, 43])
def test_device_entries_on_cell_edges(L, seed, q):
    img = edge_source(seed)
    want = R.png_quantize_ref(img, q)
    assert_same(img, L.png_quantize(img, q), want, f"edges seed={seed} q={q}")


def colliding_values():
    """257 distinct RGBA values whose slots in the device's distinct-value set ((v * 2654435761 mod 2^32) >> 22 of 1024) are 1023
    and 0, so they form one probe chain that wraps; 40 of them fully transparent with different colours"""
    rng = np.random.default_rng(51)

    def pick(lo, hi, n):
        v = rng.integers(lo, hi, 1 << 22, dtype=np.uint64)
        s = ((v * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)) >> np.uint64(22)
        v = np.unique(v[(s == 1023) | (s == 0)])
        assert len(v) >= n
        return v[:n]

    vals = np.r_[pick(1 << 24, 1 << 32, 217), pick(0, 1 << 24, 40)]        # alpha >= 1, then alpha 0
    rng.shuffle(vals)
    return np.stack([(vals >> np.uint64(8 * c)) & np.uint64(255) for c in range(4)], -1).astype(np.uint8)


def boundary_image(n, where, h=40, w=37):
    """h x w pixels of the first 256 colliding values cycling; n == 257 adds the 257th at pixel 0 or at the last pixel only"""
    vals = colliding_values()
    img = vals[np.arange(h * w) % 256].reshape(h, w, 4).copy()
    if n == 257:
        img.reshape(-1, 4)[0 if where == "first" else -1] = vals[256]
    return img


@pytest.mark.gpu
def test_exact_path_at_256_colliding_values(L, lossy):
    img = boundary_image(256, None)
    assert len(np.unique(img.reshape(-1, 4), axis=0)) == 256
    pal, idx = L.png_quantize(img, 40)
    assert_same(img, (pal, idx), R.png_quantize_ref(img, 40), "256 values")
    assert np.array_equal(pal[idx], img)
    p = L.default_params()
    p.png_optimize, p.png_quality = 0, 40
    assert np.array_equal(np.asarray(pil_pixels(lossy.compress_in_memory(pil_png(img), p)).convert("RGBA")), img)


@pytest.mark.gpu
@pytest.mark.parametrize("where", ["first", "last"])
def test_quantised_at_257_colliding_values(L, where):
    img = boundary_image(257, where)
    assert len(np.unique(img.reshape(-1, 4), axis=0)) == 257
    for q in (40, 100):
        want = R.png_quantize_ref(img, q)
        R.check_dither(img, *want)
        assert_same(img, L.png_quantize(img, q), want, f"257 values, the last one at the {where} pixel, q={q}")


@pytest.fixture
def lossy(L):
    assert L.set_png_lossy(True) == 0
    yield L
    L.set_png_lossy(False)


@pytest.mark.gpu
def test_batch_of_mixed_shapes(lossy):
    L = lossy
    shapes = [(1, 300), (300, 1), (33, 65), (64, 64), (2, 129), (97, 31), (40, 52), (17, 200)]
    imgs = []
    for i in range(16):
        h, w = shapes[i % len(shapes)]
        imgs.append(noise_with_hole(h, w, 60 + i) if i % 2 else opaque(synth(h, w, 3, seed=60 + i)))
    p = L.default_params()
    p.png_optimize, p.png_quality = 0, 70
    res = L.compress_batch([pil_png(im) for im in imgs], p, n_threads=8)
    for i, (im, (data, code, msg)) in enumerate(zip(imgs, res)):
        assert code == 0, msg
        pal, idx = R.png_quantize_ref(im, 70)
        assert np.array_equal(np.asarray(pil_pixels(data).convert("RGBA")), pal[idx]), f"batch item {i} ({im.shape[1]}x{im.shape[0]})"


# ---- GPU: the device against the twin at large shapes -----------------------------------------------------------------------------

def big_photo_hole():
    img = opaque(synth(3072, 4096, 3, seed=71))
    img[1000:1400, 2000:2600, 3] = 0
    return img


LARGE = {
    "4096x3072_hole_q40": (big_photo_hole, 40),
    "65535x3_q40": (lambda: opaque(synth(3, 65535, 3, seed=72)), 40),
    "3x20000_q40": (lambda: noise_with_hole(20000, 3, 73), 40),
    "2000x1500_q1": (lambda: opaque(synth(1500, 2000, 3, seed=74)), 1),
    "2000x1500_q80": (lambda: synth(1500, 2000, 4, seed=75), 80),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(LARGE))
def test_device_equals_the_twin_at_large_shapes(L, case):
    make, q = LARGE[case]
    img = make()
    got, want = L.png_quantize(img, q), twin_quantize(img, q)
    assert np.array_equal(got[0], want[0]), f"{case}: palettes differ"
    bad = np.argwhere(got[1] != want[1])
    assert not len(bad), f"{case}: {len(bad)} indices differ, first at (x={bad[0][1]}, y={bad[0][0]})"
