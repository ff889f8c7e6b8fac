"""JPEG sampling geometries beyond what Pillow writes (tests/jpeg_geometry.py), on the CPU: the oracle and libjpeg-turbo, the host
decoder, the device decoder's and encoder's kernel bodies run serially (tests/emul), and the 4:1:1 forward path against a numpy
restatement of libjpeg's downsampler.  Files with more than 10 blocks in an interleaved MCU are corrupt input everywhere."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import jpeg_geometry as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL_DIR = os.path.join(ROOT, "tests", "emul")
ZZ = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
               35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])
CASES = [(name, w, h) for name, f in G.GEOMETRIES.items() for (w, h) in G.sizes_for(f)]


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(EMUL_DIR, "libgpudec_emul.so")
    srcs = [os.path.join(EMUL_DIR, "gpudec_emul.cpp"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_host.cpp"),
            os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_gpudec_core.h"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_gpuenc_core.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-msse2", "-Wno-unknown-pragmas", "-o", so, srcs[0], srcs[1]])
    return C.CDLL(so)


@pytest.fixture(scope="module")
def enc_emul():
    so = os.path.join(EMUL_DIR, "libgpuenc_emul.so")
    srcs = [os.path.join(EMUL_DIR, "gpuenc_emul.cpp"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_host.cpp"),
            os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_gpuenc_core.h"), os.path.join(ROOT, "caesium-clt_b200", "csrc", "jpeg_gpuenc_plan.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-msse2", "-o", so, srcs[0], srcs[1]])
    return C.CDLL(so)


def emul_decode(emul, data, total_coefs, subseq):
    out = np.zeros(total_coefs, dtype=np.int16)
    r = C.c_int(0)
    rc = emul.emul_gpu_decode(data, C.c_size_t(len(data)), subseq, 256, out.ctypes.data_as(C.c_void_p), C.c_longlong(out.size), C.byref(r))
    return rc, out


def emul_transcode(enc_emul, data, prog):
    outp, outl = C.c_void_p(), C.c_size_t()
    rc = enc_emul.emul_gpu_transcode(data, C.c_size_t(len(data)), prog, C.byref(outp), C.byref(outl))
    assert rc == 0, rc
    return C.string_at(outp, outl.value)


def host_transcode(L, data, prog):
    p = L.default_params()
    p.jpeg_optimize, p.jpeg_progressive = 1, int(prog)
    return L.compress_in_memory(data, p)


@pytest.mark.parametrize("name,w,h", CASES)
def test_oracle_host_decoder_and_kernel_emulations(L, O, emul, enc_emul, name, w, h):
    """At every geometry and size, baseline and progressive: the oracle's decode equals libjpeg-turbo's (make_jpeg pins it), the
    host decoder's coefficients equal the oracle's for every component, the device decoder's kernel bodies equal the host decoder
    at two subsequence sizes, and the device encoder's transcode in the input's geometry equals the host transcode and the oracle."""
    f = G.GEOMETRIES[name]
    for prog in (False, True):
        data = G.make_jpeg(w, h, f, prog)
        o = O.Jpeg(data)
        lay, co = L.jpeg_decode_coefficients(data)
        assert (lay.ncomp, lay.width, lay.height) == (o.ncomp, w, h)
        for c in range(lay.ncomp):
            assert np.array_equal(L.component_view(lay, co, c), o.coef(c)[:, :, ZZ]), (prog, c)
        if not prog:
            for subseq in (128, 1024):
                rc, out = emul_decode(emul, data, lay.total_coefs, subseq)
                assert rc == 0 and np.array_equal(out, co), (subseq, rc)
        for oprog in (0, 1):
            got = emul_transcode(enc_emul, data, oprog)
            assert got == host_transcode(L, data, oprog)
            assert got == O.jpeg_lossless(data, O.params(80, 0, bool(oprog)))


def _int_downsample_411(plane, rbw, rbh):
    """jcsample.c int_downsample for h_expand = 4, v_expand = 1, with jcsample.c expand_right_edge and jcprepct.c's bottom
    edge replication: each output sample is (sum of 4 + 2) / 4 over the edge-extended row."""
    H, W = plane.shape
    ext = np.pad(plane.astype(np.int32), ((0, rbh * 8 - H), (0, rbw * 8 * 4 - W)), mode="edge")
    return ((ext.reshape(rbh * 8, rbw * 8, 4).sum(axis=2) + 2) // 4).astype(np.uint8)


@pytest.mark.parametrize("w,h", [(1, 1), (2, 3), (17, 9), (67, 45), (130, 61), (257, 8)])
def test_411_forward_path_restated(O, w, h):
    """libjpeg-turbo cannot be asked for 4:1:1 through Pillow: the oracle's forward path at 4:1:1 against the downsampler restated
    in numpy, then the oracle's FDCT + quantiser per block."""
    from tools.synth import synth_rgb
    planes = O.rgb_to_ycc(np.ascontiguousarray(synth_rgb(w, h, w + h).transpose(2, 0, 1)))
    for q in (75, 30):
        j = O.forward(planes, O.params(q, 411, False))
        assert [(j.s.hs[c], j.s.vs[c]) for c in range(3)] == [(4, 1), (1, 1), (1, 1)]
        for c in range(3):
            rbw, rbh = j.s.rbw[c], j.s.rbh[c]
            if c == 0:
                ds = np.pad(planes[0], ((0, rbh * 8 - h), (0, rbw * 8 - w)), mode="edge")
            else:
                ds = _int_downsample_411(planes[c], rbw, rbh)
            qt = O.quant_table(q, 0 if c == 0 else 1)
            got = j.coef(c)
            for by in range(rbh):
                for bx in range(rbw):
                    want = O.fdct_quant(ds[by * 8:by * 8 + 8, bx * 8:bx * 8 + 8], qt)[1].reshape(64)
                    assert np.array_equal(got[by, bx], want), (q, c, by, bx)


@pytest.mark.parametrize("name", sorted(G.OVERSIZED))
def test_oversized_mcu_is_refused(L, O, emul, name):
    """More than 10 blocks in an interleaved MCU (libjpeg's JERR_BAD_MCU_SIZE; make_jpeg asserts libjpeg-turbo refuses the file):
    the oracle's reader, the host decoder and the device decoder's eligibility check refuse it, baseline and progressive."""
    f = G.OVERSIZED[name]
    for prog in (False, True):
        data = G.make_jpeg(67, 45, f, prog)
        with pytest.raises(O.OracleError, match="MCU"):
            O.Jpeg(data)
        with pytest.raises(L.B200Error) as e:
            L.jpeg_decode_coefficients(data)
        assert e.value.code == L.ERR_CORRUPT_INPUT and "MCU" in str(e.value)
        rc, _ = emul_decode(emul, data, 1 << 20, 1024)
        assert rc == 10
        with pytest.raises(L.B200Error) as e:
            host_transcode(L, data, prog)
        assert e.value.code == L.ERR_CORRUPT_INPUT


def test_fractional_ratio_is_unsupported_before_any_device_work(L, O):
    """Y 3x1 with Cb 2x1 has no integral upsampling ratio (libjpeg: JERR_FRACT_SAMPLE_NOT_IMPL; make_jpeg asserts libjpeg-turbo
    refuses it).  Every leg that decodes to samples answers 3 straight after the header, so also on a machine without a device;
    the coefficient-domain transcode has no upsampling and still equals the oracle's."""
    data = G.make_jpeg(67, 45, G.FRACTIONAL, False)
    calls = [lambda: L.compress_in_memory(data, L.default_params()),
             lambda: L.compress_in_memory(data, _resize_params(L, 40, 0)),
             lambda: L.convert_in_memory(data, L.default_params(), 3),
             lambda: L.compress_to_size_in_memory(data, L.default_params(), len(data) // 2)]
    for call in calls:
        with pytest.raises(L.B200Error) as e:
            call()
        assert e.value.code == L.ERR_UNSUPPORTED and "fractional" in str(e.value)
    for prog in (0, 1):
        assert host_transcode(L, data, prog) == O.jpeg_lossless(data, O.params(80, 0, bool(prog)))


def _resize_params(L, w, h):
    p = L.default_params()
    p.width, p.height = w, h
    return p


def test_one_block_mcus_stay_legal(L, O):
    """The limit is on interleaved MCUs: a single-component file with 4x4 factors in its header has one block per MCU, and a
    progressive file at the 10-block limit (Y 4x2 + 1 + 1, whose interleaved DC scan holds 10) decodes everywhere."""
    for f, prog in (([(4, 4)], False), ([(4, 4)], True), (G.GEOMETRIES["y42"], True), (G.GEOMETRIES["y42"], False)):
        data = G.make_jpeg(67, 45, tuple(map(tuple, f)), prog)        # decodes in libjpeg-turbo, equal to the oracle
        lay, co = L.jpeg_decode_coefficients(data)
        o = O.Jpeg(data)
        for c in range(lay.ncomp):
            assert np.array_equal(L.component_view(lay, co, c), o.coef(c)[:, :, ZZ])
