"""The deferred DC of lossy megabatches (tests/wild_dc.py), on the CPU: files whose running DC leaves int16, pinned to libjpeg-turbo;
a plain MCU walk of their DC against the host decoder and the oracle; and put_dc's slot formula with dc_sums' component offsets,
restated in Python, against that walk at every geometry and size, in batches whose prefix sum leaves int32.
test_deferred_dc_wrap_gpu.py runs the same files through the device."""
import numpy as np
import pytest

import jpeg_geometry as G
import wild_dc as W

CASES = [(name, w, h) for name, f in G.GEOMETRIES.items() for (w, h) in G.sizes_for(f)]
GREY = G.GEOMETRIES["grey22"]
# single-component scans laid out at their declared factors (rbw < bw, rbw != mcux): the restatement's reach beyond the files
DECLARED = [(W.Declared(((hs, vs),)), w, h) for hs, vs in ((2, 2), (4, 1), (1, 3)) for (w, h) in G.SMALL_SIZES + [(263, 77)]]


def _all_files():
    out = [(f"{name} {w}x{h} wild", W.wild_jpeg(w, h, G.GEOMETRIES[name], "wild", 1)) for name, w, h in CASES]
    out += [(f"climb {p}", W.wild_jpeg(*W.CLIMB_SIZE, GREY, p)) for ps in W.WRAP_BATCHES.values() for p in ps]
    return out


def _members(factors, w, h, patterns):
    return [(w, h, factors, W.pattern_diffs(w, h, factors, p, s)) for p, s in patterns]


def test_wild_files_are_pinned_to_libjpeg_turbo(O):
    """libjpeg-turbo decodes every wild file (category-15 DC differences and all) exactly as the oracle does.  Its C inverse DCT
    is the reference: the SIMD one, which works in 16-bit lanes, is only asked not to refuse the files."""
    files = _all_files()
    for (what, d), ref in zip(files, W.libjpeg_c_native([d for _, d in files])):
        got = O.Jpeg(d).decode_native()
        assert ref.shape == got.shape and np.array_equal(ref, got), what
        assert not G.libjpeg_refuses(d), what


def test_wild_dc_crosses_every_int16_edge():
    """The wild differences reach category 15, the running DC leaves int16 both ways and lands on 32767, -32768 and 0; the climbs
    end near +-2^30 without leaving int32."""
    for name, w, h in CASES:
        n = W.block_counts(w, h, G.GEOMETRIES[name])[0]
        if n < 400:
            continue
        d = W.wild_diffs(n, 1)
        run = np.cumsum(d)
        assert max(int(abs(x)).bit_length() for x in d) == 15, name
        wraps = np.diff((run + 32768) // 65536)               # +1: the int16 DC passed 32767 upwards; -1: -32768 downwards
        assert (wraps > 0).sum() >= 5 and (wraps < 0).sum() >= 5, name
        lands = set(((run + 32768) % 65536 - 32768).tolist())
        assert {32767, -32768, 0} <= lands, name
    for ps in W.WRAP_BATCHES.values():
        for p in ps:
            run = np.cumsum(W.pattern_diffs(*W.CLIMB_SIZE, GREY, p)[0])
            assert 0.99 * 2 ** 30 < abs(int(run[-1])) < 2 ** 31, p


@pytest.mark.parametrize("name,w,h", CASES)
def test_reference_dc_equals_host_decoder_and_oracle(L, O, name, w, h):
    """reference_dc() against the DC of every block the host decoder (JpegReader) and the oracle decode, both per component."""
    f = G.GEOMETRIES[name]
    for pattern, data in (("wild", W.wild_jpeg(w, h, f, "wild", 1)), (None, G.make_jpeg(w, h, f, False))):
        lay, co = L.jpeg_decode_coefficients(data)
        if pattern:
            want = W.reference_dc(w, h, f, W.pattern_diffs(w, h, f, pattern, 1))
        else:
            want = [O.Jpeg(data).coef(c)[..., 0] for c in range(lay.ncomp)]
        j = O.Jpeg(data)
        for c in range(lay.ncomp):
            n = lay.bw[c] * lay.bh[c] * 64
            dc = co[lay.comp_offset[c]:lay.comp_offset[c] + n].reshape(lay.bh[c], lay.bw[c], 64)[..., 0]
            assert np.array_equal(dc, want[c]), (pattern, c)
            assert np.array_equal(j.coef(c)[..., 0], want[c]), (pattern, c)


def test_reference_dc_of_the_climbs(L):
    for ps in W.WRAP_BATCHES.values():
        for p in ps:
            data = W.wild_jpeg(*W.CLIMB_SIZE, GREY, p)
            lay, co = L.jpeg_decode_coefficients(data)
            want = W.reference_dc(*W.CLIMB_SIZE, GREY, W.pattern_diffs(*W.CLIMB_SIZE, GREY, p))[0]
            assert np.array_equal(co.reshape(lay.bh[0], lay.bw[0], 64)[..., 0], want), p


@pytest.mark.parametrize("name,w,h", CASES + [(None, w, h) for _, w, h in DECLARED])
def test_slot_restatement_equals_reference(name, w, h):
    """put_dc + dc_sums over a three-member batch (wild, climb, wild: every member its own dc_prev) give reference_dc() at every
    block of every component, MCU padding blocks included."""
    factors = G.GEOMETRIES[name] if name else None
    for f in ([factors] if name else [d for d, dw, dh in DECLARED if (dw, dh) == (w, h)]):
        members = _members(f, w, h, [("wild", 1), ("climb+32767", 0), ("wild", 2)])
        for (mw, mh, mf, diffs), got in zip(members, W.deferred_dc(members)):
            want = W.reference_dc(mw, mh, mf, diffs)
            for c in range(len(want)):
                assert np.array_equal(got[c], want[c]), (f, c)


@pytest.mark.parametrize("direction", list(W.WRAP_BATCHES))
def test_batch_prefix_sum_leaves_int32(direction):
    """The wrap batches: the batch-wide sum passes +2^31 (-2^31) inside the third member, each member's own running DC stays within
    int32, and the restatement, which wraps the sum as the int32 scan does, still gives every block's DC."""
    members = _members(GREY, *W.CLIMB_SIZE, [(p, 0) for p in W.WRAP_BATCHES[direction]])
    _, firsts, exact = W.batch_prefix_sum(members)
    sign = 1 if direction == "up" else -1
    assert sign * exact[firsts[2] - 1] < 2 ** 31 <= sign * exact[-1]
    for _, _, _, diffs in members:
        assert np.abs(np.cumsum(diffs[0])).max() < 2 ** 31
    for (w, h, f, diffs), got in zip(members, W.deferred_dc(members)):
        assert np.array_equal(got[0], W.reference_dc(w, h, f, diffs)[0])


def test_slot_restatement_tells_mutants_apart():
    """The comparison above is sharp enough to see each way put_dc / dc_sums could go wrong: swapped hs / vs, no dc_prev
    subtraction, mcux instead of rbw for a single-component scan, no int16 truncation."""
    def differs(members, **mutation):
        got = W.deferred_dc(members, **mutation)
        return any(not np.array_equal(g[c], W.reference_dc(w, h, f, d)[c]) for (w, h, f, d), g in zip(members, got) for c in range(len(g)))
    for name in ("y12", "y41", "c21", "c12", "y32"):
        members = _members(G.GEOMETRIES[name], 67, 45, [("wild", 1), ("wild", 2)])
        assert not differs(members)
        assert differs(members, swap_hv=True), name
        assert differs(members, no_prev=True), name
        assert differs(members, no_trunc=True), name
    for f, w, h in DECLARED:
        if w > 16 and f[0][0] > 1:                   # (1 x v: mcux == rbw, the two readings agree)
            members = _members(f, w, h, [("wild", 1)])
            mcux = W.components(w, h, f)[1][1]
            assert not differs(members) and differs(members, single_mcux=mcux), (f, w, h)
