"""The same-shape JPEG variants of mixed_jpeg.py, on the CPU: every one is pinned to libjpeg-turbo, the device decoder's verdict on
each (decoded, refused, not settled) is pinned through its serial emulation, and the host transcode (entropy mode 0) gives the
oracle's file for every one of them.  The GPU half, test_megabatch_mixed_gpu.py, runs the same files through megabatches and the
resident pipe."""
import ctypes as C

import numpy as np
import pytest

from jpeg_geometry import libjpeg_native
from mixed_jpeg import KINDS, build, parse, variants
from test_gpudec import emul  # noqa: F401  (fixture: the serial emulation of the device decoder, tests/emul/gpudec_emul.cpp)

SUBSEQ_BITS, ROUNDS = 2048, 24          # GpuDecoder's defaults (jpeg_gpudec.h)


@pytest.mark.parametrize("kind", KINDS)
def test_variants_share_one_shape_and_decode_like_libjpeg(O, kind):
    vs = variants(kind)
    assert len({v.name for v in vs}) == len(vs)
    assert len({v.data for v in vs}) == len(vs)
    j0 = O.Jpeg(vs[0].data)
    shape = lambda j: (j.s.width, j.s.height, j.ncomp, tuple(j.s.hs[:j.ncomp]), tuple(j.s.vs[:j.ncomp]))
    for v in vs:
        j = O.Jpeg(v.data)
        assert shape(j) == shape(j0), v.name
        assert not j.s.progressive and j.s.restart_interval == 0 and j.s.nscans == 1, v.name
        ref = libjpeg_native(v.data)
        assert np.array_equal(j.decode_native(), ref), f"{v.name}: oracle decode differs from libjpeg-turbo"
        if v.origin is not None:
            assert np.array_equal(ref, libjpeg_native(v.origin)), f"{v.name}: the rewrite decodes unlike its source"


@pytest.mark.parametrize("kind", KINDS)
def test_variants_differ_where_they_claim_to(O, kind):
    """The headers really carry what the names say (a rewrite that silently did nothing would test nothing)."""
    vs = {v.name: O.Jpeg(v.data) for v in variants(kind)}
    n = vs["annex_k_q75"].ncomp
    tq = lambda name: tuple(vs[name].s.tq[:n])
    cid = lambda name: tuple(vs[name].s.cid[:n])
    assert cid("component_ids_0_1_2") == (0, 1, 2)[:n] and cid("component_ids_odd") == (200, 7, 99)[:n]
    assert tq("qtable_ids_2_3") == (3, 2, 2)[:n] and tq("qtable_ids_swapped") == (1, 0, 0)[:n]
    assert vs["qtables_above_255_sof1"].qtable(0).max() > 255
    if n == 3:
        assert tq("one_qtable_tq000") == (0, 0, 0) and tq("three_qtables_tq012") == (0, 1, 2)
        q = vs["three_qtables_tq012"]
        assert not np.array_equal(q.qtable(1), q.qtable(2))
        assert vs["qtables_above_255_sof1"].qtable(1).max() > 255
    data = {v.name: v.data for v in variants(kind)}
    assert build(parse(data["annex_k_q75"])) == data["annex_k_q75"]          # the rewrites start from the Pillow file itself
    assert b"\xff\xc1" in data["qtables_16bit_sof1"] and b"\xff\xc1" in data["huff_ids_2_3_sof1"]
    assert b"JFIF" not in data["no_jfif"] and b"Exif\x00\x00" in data["exif_and_icc"] and b"ICC_PROFILE" in data["exif_and_icc"]
    assert data["second_jpeg_appended"].count(b"\xff\xd8") == 2


@pytest.mark.parametrize("kind", KINDS)
def test_device_decoder_verdicts(L, emul, kind):
    """The serial emulation of the device decoder at its default subsequence size and round budget: every variant decodes to the
    host decoder's coefficients, except those it must hand to the host -- the Huffman tables that overflow its lookup pool
    (refused), the periodic stream (not settled within the budget) and 0xFF fill in front of EOI (not a device scan).  These are
    the counts the GPU tests expect."""
    for v in variants(kind):
        lay, ref = L.jpeg_decode_coefficients(v.data)
        out = np.zeros(lay.total_coefs, np.int16)
        rounds = C.c_int(0)
        rc = emul.emul_gpu_decode(v.data, C.c_size_t(len(v.data)), SUBSEQ_BITS, ROUNDS, out.ctypes.data_as(C.c_void_p), C.c_longlong(out.size), C.byref(rounds))
        want = 10 if not v.pipe else 12 if v.name == "huff_tables_refused" else 11 if not v.settles else 0
        assert rc == want, (v.name, rc)
        if rc == 0:
            assert np.array_equal(out, ref), v.name
        if v.name == "periodic_stream":           # it settles, one subsequence per round: far beyond the budget
            rc = emul.emul_gpu_decode(v.data, C.c_size_t(len(v.data)), SUBSEQ_BITS, 100000, out.ctypes.data_as(C.c_void_p), C.c_longlong(out.size), C.byref(rounds))
            assert rc == 0 and rounds.value > 4 * ROUNDS and np.array_equal(out, ref)


@pytest.mark.parametrize("prog", [True, False])
@pytest.mark.parametrize("kind", KINDS)
def test_host_transcode_equals_oracle(L, O, kind, prog):
    """--lossless on the host coders: the oracle's file for every variant, the source's JFIF version and density kept as
    jpeg_copy_critical_parameters keeps them."""
    p = L.default_params()
    p.jpeg_optimize, p.jpeg_progressive = 1, int(prog)
    L.set_entropy_mode(0)
    try:
        for v in variants(kind):
            try:
                want = O.jpeg_lossless(v.data, O.params(80, 0, prog))
            except O.OracleError:
                with pytest.raises(L.B200Error):
                    L.compress_in_memory(v.data, p)
                continue
            assert L.compress_in_memory(v.data, p) == want, v.name
    finally:
        L.set_entropy_mode(3)
