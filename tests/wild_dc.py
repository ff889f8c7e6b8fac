"""Baseline JPEG files whose running DC leaves int16, and a plain restatement of how the deferred-DC path rebuilds it, for the
deferred-DC tests (not a fixture: imported by the test modules).

A lossy megabatch and the resident pipe decode with GpuDecoder::Item::defer_dc: each decoded block keeps its DC DIFFERENCE, the
decoder leaves an int32 inclusive prefix sum of the differences over the whole batch (component-major within each image, images
one after the other), and the transform kernels rebuild the DC of block (bx, by) in put_dc as sum[slot] - sum[first - 1],
truncated to int16, with slot and first from GpuDecoder::dc_sums.  libjpeg-turbo instead keeps one running DC per component in
an int and stores (JCOEF) of it.  The two agree modulo 2^16 only if the slot, the component offsets and the wrap are all right.

wild_jpeg() codes any geometry of jpeg_geometry.GEOMETRIES with jpeg_geometry's picture as AC content and caller-chosen DC
differences (categories up to 15, which libjpeg-turbo decodes: its DC table may hold symbols 0..15), one interleaved scan, no
restart interval, so the device decoder takes it.  Every file is pinned to libjpeg-turbo by test_deferred_dc_wrap_host.py: its
native decode through Pillow (libjpeg_c_native) must equal the oracle's.  reference_dc() is the DC of every block by the JPEG
spec's MCU walk; deferred_dc() is put_dc and dc_sums restated over a batch.  The host tests check one against the other and both against the host decoder."""
import functools
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import jpeg_geometry as G          # noqa: E402
import mixed_jpeg as M             # noqa: E402

# DC table: symbols (categories) 0..15, all five bits long (sixteen four-bit codes would include the all-ones code)
WILD_DC_TABLE = ([0, 0, 0, 0, 16] + [0] * 11, list(range(16)))
# the grey image whose running DC climbs to about +-2^30 in +-32767 steps: 181 x 181 = 32761 blocks
CLIMB_SIZE = (1448, 1448)


def _int16(v):
    return (int(v) + 32768) % 65536 - 32768


def _int32(v):
    return (int(v) + 2 ** 31) % 2 ** 32 - 2 ** 31


class Declared(tuple):
    """One component's factors ((hs, vs),) laid out as declared -- hs x vs blocks per MCU, bw = mcux * hs, so rbw < bw and rbw != mcux
    -- where the readers give a grey file one block per MCU.  The layout of a non-interleaved scan of a subsampled component: no
    file the device decoder takes has it, so only the restatement meets it (dc_sums must still use rbw for such a scan)."""


def components(w, h, factors):
    """Per component (hs, vs, rbw, rbh, bw, bh) as the readers lay it out, and (ns, mcux, mcuy)."""
    if isinstance(factors, Declared):
        (hs, vs), = factors
        mcux, mcuy = -(-w // (8 * hs)), -(-h // (8 * vs))
        return [(hs, vs, -(-w // 8), -(-h // 8), mcux * hs, mcuy * vs)], (1, mcux, mcuy)
    geo, (_, _, mcux, mcuy) = G.geometry(w, h, factors)
    return [(hs, vs, rbw, rbh, bw, bh) for hs, vs, _, _, rbw, rbh, bw, bh in geo], (len(geo), mcux, mcuy)


def scan_order(w, h, factors):
    """The blocks in the order the scan codes them, as (component, bx, by) in the component's bw x bh grid (ITU T.81 A.2): a
    single-component scan is a raster over the real blocks rbw x rbh; an interleaved scan walks the MCUs in raster order and,
    inside each, every component's hs x vs blocks in raster order, MCU padding blocks included."""
    comps, (ns, mcux, mcuy) = components(w, h, factors)
    if ns == 1:
        _, _, rbw, rbh, _, _ = comps[0]
        return [(0, bx, by) for by in range(rbh) for bx in range(rbw)]
    return [(c, mx * hs + u, my * vs + v) for my in range(mcuy) for mx in range(mcux)
            for c, (hs, vs, _, _, _, _) in enumerate(comps) for v in range(vs) for u in range(hs)]


def block_counts(w, h, factors):
    """Blocks the scan codes for each component (the length of its DC difference sequence)."""
    n = [0] * len(components(w, h, factors)[0])
    for c, _, _ in scan_order(w, h, factors):
        n[c] += 1
    return n


def reference_dc(w, h, factors, diffs):
    """The DC of every block as libjpeg-turbo keeps it: per component an unbounded running sum of its differences in scan order,
    stored as int16.  -> per component [bh, bw] int16 (blocks the scan does not code stay 0)."""
    comps, _ = components(w, h, factors)
    out = [np.zeros((bh, bw), np.int16) for _, _, _, _, bw, bh in comps]
    pred, k = [0] * len(comps), [0] * len(comps)
    for c, bx, by in scan_order(w, h, factors):
        pred[c] += int(diffs[c][k[c]]); k[c] += 1
        out[c][by, bx] = _int16(pred[c])
    return out


# ---- put_dc and dc_sums restated ---------------------------------------------------------------------------------------------
def dc_array_index(w, h, factors):
    """Where the decoder's write pass stores each block's DC difference (gd::Walk dc_base / dc_step, as dc_slot_index): in scan
    order, the index in the image's component-major array -- component c's blocks from its offset on, hs * vs per MCU."""
    comps, (ns, mcux, mcuy) = components(w, h, factors)
    if ns == 1:
        return list(range(len(scan_order(w, h, factors))))
    start, base = 0, []
    for hs, vs, _, _, _, _ in comps:
        base.append(start)
        start += mcux * mcuy * hs * vs
    out = []
    for c, bx, by in scan_order(w, h, factors):
        hs, vs = comps[c][:2]
        out.append(base[c] + ((by // vs) * mcux + bx // hs) * hs * vs + (by % vs) * hs + bx % hs)
    return out


def dc_sums(w, h, factors, single_mcux=None):
    """GpuDecoder::dc_sums for each component: (offset of its first block in the image's DC array, hs, vs, mcux).  A single-component
    scan is one block per MCU, rbw of them per row.  single_mcux: what a single-component scan takes as blocks per row instead
    of rbw (a test of the restatement's own reach: see test_slot_restatement_tells_mutants_apart)."""
    comps, (ns, mcux, mcuy) = components(w, h, factors)
    out, start = [], 0
    for hs, vs, rbw, _, _, _ in comps:
        if ns == 1:
            hs = vs = 1
        out.append((start, hs, vs, (rbw if single_mcux is None else single_mcux) if ns == 1 else mcux))
        start += mcux * mcuy * hs * vs
    return out


def put_dc_slot(bx, by, hs, vs, mcux):
    """put_dc's slot of block (bx, by) of a component, relative to its first block."""
    mx, my = bx // hs, by // vs
    return (my * mcux + mx) * (hs * vs) + (by - my * vs) * hs + (bx - mx * hs)


def batch_prefix_sum(members):
    """members: [(w, h, factors, diffs)] -> (the decoder's int32 inclusive prefix sum over the batch, with int32 wrap; each
    member's first index in it; the same sum unbounded, to show where it leaves int32)."""
    arrays, firsts, n = [], [], 0
    for w, h, factors, diffs in members:
        idx = dc_array_index(w, h, factors)
        a = np.zeros(len(idx), np.int64)
        k = [0] * len(diffs)
        for (c, _, _), i in zip(scan_order(w, h, factors), idx):
            a[i] = int(diffs[c][k[c]]); k[c] += 1
        arrays.append(a); firsts.append(n); n += len(a)
    exact = np.cumsum(np.concatenate(arrays)) if arrays else np.zeros(0, np.int64)
    wrapped = ((exact + 2 ** 31) % 2 ** 32 - 2 ** 31).astype(np.int64)
    return wrapped, firsts, exact


def deferred_dc(members, swap_hv=False, no_prev=False, no_trunc=False, single_mcux=None):
    """put_dc over a batch: per member, per component, [bh, bw] of the DC the transform kernels rebuild at every block of the
    grid the scan codes.  The flags restate the mutations the tests must catch (int64 results where no_trunc is set)."""
    wrapped, firsts, _ = batch_prefix_sum(members)
    out = []
    for (w, h, factors, _), first in zip(members, firsts):
        comps, (ns, _, _) = components(w, h, factors)
        per = []
        for (_, _, rbw, rbh, bw, bh), (start, hs, vs, mcux) in zip(comps, dc_sums(w, h, factors, single_mcux)):
            b = first + start
            prev = 0 if (b == 0 or no_prev) else int(wrapped[b - 1])
            gw, gh = (rbw, rbh) if ns == 1 else (bw, bh)
            a = np.zeros((bh, bw), np.int64 if no_trunc else np.int16)
            for by in range(gh):
                for bx in range(gw):
                    slot = put_dc_slot(bx, by, vs, hs, mcux) if swap_hv else put_dc_slot(bx, by, hs, vs, mcux)
                    i = b + slot
                    v = _int32(int(wrapped[i]) - prev) if 0 <= i < len(wrapped) else 1 << 20
                    a[by, bx] = v if no_trunc else _int16(v)
            per.append(a)
        out.append(per)
    return out


# ---- DC difference patterns ------------------------------------------------------------------------------------------------------
def wild_diffs(n, seed):
    """n DC differences of every category 0..15, uniformly: the running DC crosses +-32767 / -32768 over and over, and every 97th
    block is steered to land exactly on 32767, -32768 or 0 (mod 2^16)."""
    rng = np.random.default_rng(seed)
    cat = rng.integers(0, 16, n)
    lo = np.where(cat > 0, 1 << np.maximum(cat - 1, 0), 0)             # category s: magnitudes 2^(s-1) .. 2^s - 1
    mag = lo + rng.integers(0, 1 << 15, n) % np.maximum(lo, 1)
    d = (mag * rng.choice([-1, 1], n)).astype(np.int64)
    run, targets = 0, (32767, -32768, 0)
    for k in range(n):
        if k % 97 == 96:
            t = targets[(k // 97) % 3]
            step = (t - run) % 65536
            step = step - 65536 if step > 32767 else step
            if step != -32768:                    # -32768 has no category (16): land on the next steering block instead
                d[k] = step
        run += int(d[k])
    return d


def pattern_diffs(w, h, factors, pattern, seed=0):
    """Per component DC differences for `pattern`: "wild" (wild_diffs, another seed per component) or "climb<k>" (k every block,
    k signed: "climb+32767" climbs by the largest difference there is)."""
    out = []
    for c, n in enumerate(block_counts(w, h, factors)):
        if pattern == "wild":
            out.append(wild_diffs(n, seed * 1009 + c))
        elif pattern.startswith("climb"):
            out.append(np.full(n, int(pattern[5:]), np.int64))
        else:
            raise ValueError(pattern)
    return out


# Batches of CLIMB_SIZE grey files whose batch-wide prefix sum passes +2^31 (-2^31) inside the third member, while every member's
# own running DC stays within +-1.08e9: each member's steps differ, so every member has its own dc_prev.
WRAP_BATCHES = {"up": ("climb+32767", "climb+32765", "climb+32766"), "down": ("climb-32767", "climb-32765", "climb-32766")}


def _dht_tables(data):
    """(dc, ac) Huffman tables per component of a baseline file, in frame order."""
    p = M.parse(data)
    get = {(tc, th): (bits, vals) for tc, th, bits, vals in p.dht}
    return p, [(get[(0, td)], get[(1, ta)]) for _, td, ta in p.sel]


@functools.lru_cache(maxsize=None)
def wild_jpeg(w, h, factors, pattern, seed=0):
    """A w x h baseline file at `factors` (jpeg_geometry.GEOMETRIES) with jpeg_geometry's picture (seed) as AC content and the DC
    differences of pattern_diffs(), coded by mixed_jpeg.encode_scan; the DC table is WILD_DC_TABLE for every component.  (Pinned to libjpeg-turbo by the host test module.)"""
    factors = tuple(tuple(f) for f in factors)
    base = G.make_jpeg(w, h, factors, False, seed)
    coefs, _ = G._coefficients(w, h, factors, seed, 75)
    p, tables = _dht_tables(base)
    diffs = pattern_diffs(w, h, factors, pattern, seed)
    tables = [(WILD_DC_TABLE, ac) for _, ac in tables]
    p.sel = [(cid, 0, ta) for cid, _, ta in p.sel]
    p.dht = [(0, 0) + WILD_DC_TABLE] + [t for t in p.dht if t[0] == 1]
    comps = [(hs, vs) for hs, vs, _, _, _, _ in components(w, h, factors)[0]]
    # encode_scan codes each DC as the difference from the previous block's: give every block its unbounded running DC (int64),
    # and the differences it codes are exactly `diffs`
    coefs = [c.astype(np.int64) for c in coefs]
    run, k = [0] * len(coefs), [0] * len(coefs)
    for c, bx, by in scan_order(w, h, factors):
        run[c] += int(diffs[c][k[c]]); k[c] += 1
        coefs[c][by, bx, 0] = run[c]
    p.ecs = M.encode_scan(coefs, comps, tables)
    return M.build(p)


_C_DECODE = """import pickle, sys
sys.path.insert(0, {tests!r})
import jpeg_geometry as G
pickle.dump([G.libjpeg_native(d) for d in pickle.load(sys.stdin.buffer)], sys.stdout.buffer)
"""


def libjpeg_c_native(datas):
    """libjpeg-turbo's native decode (through Pillow) of each file with its SIMD code switched off (JSIMD_FORCENONE, read once per
    process: so in a child).  Its SIMD inverse DCT works in 16-bit lanes and differs from its own C jidctint.c once a dequantised
    DC leaves the range an 8-bit baseline stream can reach (category 11); the C path is the definition the oracle and the
    product follow, so the wild files are pinned to that."""
    import pickle
    import subprocess
    r = subprocess.run([sys.executable, "-c", _C_DECODE.format(tests=os.path.join(ROOT, "tests"))], input=pickle.dumps(list(datas)),
                       capture_output=True, env=dict(os.environ, JSIMD_FORCENONE="1"))
    assert r.returncode == 0, r.stderr.decode()[-2000:]
    return pickle.loads(r.stdout)
