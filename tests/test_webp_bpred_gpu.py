"""GPU parity tests of lossy WebP with 4x4 intra prediction (B_PRED): k_vp8_encode_bpred + the device token pass + the host writer,
through the C-ABI, against the scalar twin (oracle/webp_bpred_oracle.c), byte for byte; the switch off keeps today's bytes; a large
frame under 8 concurrent calls keeps its bytes (the trail-by-two wavefront under load); the host token walk agrees with the device's;
a frame whose first partition would overflow falls back to the 16x16-only bytes."""
import os
import subprocess
import sys
import threading
import ctypes as C

import numpy as np
import pytest

from pngutil import pil_png, synth
from webputil import decode_like_libwebp, pil_decode

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FMT_WEBP = 3


@pytest.fixture(scope="module")
def OB(O):
    from oracle import webp_bpred
    return webp_bpred


@pytest.fixture
def bpred_on(L):
    assert L.set_webp_bpred(1) == 0
    yield
    assert L.set_webp_bpred(0) == 0


def planar(img):
    return np.ascontiguousarray(img.transpose(2, 0, 1))


def vp8_chunk(data):
    i = 12
    while i + 8 <= len(data):
        n = int.from_bytes(data[i + 4:i + 8], "little")
        if data[i:i + 4] == b"VP8 ":
            return data[i + 8:i + 8 + n]
        i += 8 + n + (n & 1)
    raise AssertionError("no VP8 chunk")


@pytest.mark.parametrize("h,w,q,kind", [(64, 64, 75, "photo"), (37, 53, 50, "photo"), (1, 1, 80, "flat"), (16, 16, 10, "noise"),
                                        (300, 16, 60, "photo"), (17, 300, 90, "noise"), (200, 300, 100, "photo"), (129, 65, 85, "noise"),
                                        (240, 320, 30, "flat"), (33, 17, 0, "photo")])
def test_stage_output_and_file_match_the_twin(L, OB, h, w, q, kind):
    img = planar(synth(h, w, 3, seed=h + w + q, kind=kind))
    data, levels, modes, bmodes = L.webp_encode_rgb_bpred(img, q, want_stage=True)
    st = OB.webp_bpred_stages(img, q)
    assert np.array_equal(modes, st["modes"]) and np.array_equal(bmodes, st["bmodes"]) and np.array_equal(levels, st["levels"])
    assert data == st["file"]
    assert np.array_equal(pil_decode(data), decode_like_libwebp(st["Y"], st["U"], st["V"], w, h))


def test_png_to_webp_with_and_without_resize_and_alpha(L, O, OB, bpred_on):
    rgb = synth(90, 120, 3, seed=4)
    p = L.default_params(); p.webp_quality = 80
    assert L.convert_in_memory(pil_png(rgb), p, FMT_WEBP) == OB.webp_bpred_encode(planar(rgb), 80)
    rgba = np.concatenate([rgb, synth(90, 120, 1, seed=9)], axis=2)
    out = L.convert_in_memory(pil_png(rgba), p, FMT_WEBP)
    assert out[12:16] == b"VP8X" and vp8_chunk(out) == vp8_chunk(OB.webp_bpred_encode(planar(rgb), 80))
    p.width = 77
    nw, nh = O.compute_dimensions(120, 90, 77, 0)
    want = OB.webp_bpred_encode(np.stack([O.resize_plane(np.ascontiguousarray(rgb[:, :, c]), nw, nh) for c in range(3)]), 80)
    assert L.convert_in_memory(pil_png(rgb), p, FMT_WEBP) == want


def _jpeg_rgb(O, data, nw=None, nh=None):
    ycc = O.Jpeg(data).decode_native()
    rgb = O.ycc_to_rgb(ycc) if ycc.shape[0] == 3 else np.repeat(ycc, 3, axis=0)
    if nw is not None and (nw, nh) != (rgb.shape[2], rgb.shape[1]):
        rgb = np.stack([O.resize_plane(rgb[c], nw, nh) for c in range(3)])
    return rgb


@pytest.mark.parametrize("name,tw,th", [("in_420_base_355x237.jpg", 0, 0), ("in_444_base_355x237.jpg", 0, 0), ("in_420_base_640x480.jpg", 177, 99)])
def test_jpeg_to_webp(L, O, OB, golden, bpred_on, name, tw, th):
    data = golden(name)
    p = L.default_params(); p.webp_quality = 70; p.width, p.height = tw, th
    out = L.convert_in_memory(data, p, FMT_WEBP)
    rgb = _jpeg_rgb(O, data)
    if tw or th:
        nw, nh = O.compute_dimensions(rgb.shape[2], rgb.shape[1], tw, th)
        rgb = _jpeg_rgb(O, data, nw, nh)
    assert out == OB.webp_bpred_encode(rgb, 70)


def test_webp_recompression(L, O, OB, bpred_on):
    src, _ = O.webp_encode(planar(synth(120, 160, 3, seed=3)), 100)
    p = L.default_params(); p.webp_quality = 60
    out = L.compress_in_memory(src, p)
    assert out == OB.webp_bpred_encode(planar(L.webp_decode(src)), 60)


def test_switch_off_keeps_todays_bytes(L, O):
    assert L.set_webp_bpred(0) == 0
    img = planar(synth(100, 130, 3, seed=7))
    p = L.default_params(); p.webp_quality = 75
    assert L.webp_encode_rgb(img, 75) == O.webp_encode(img, 75)[0]
    assert L.convert_in_memory(pil_png(img.transpose(1, 2, 0)), p, FMT_WEBP) == O.webp_encode(img, 75)[0]


def test_large_frame_under_concurrency(L, OB, bpred_on):
    img = planar(synth(1536, 2048, 3, seed=11, kind="photo"))
    want = OB.webp_bpred_encode(img, 75)
    outs = [None] * 8
    def run(i):
        outs[i] = L.webp_encode_rgb_bpred(img, 75)
    ts = [threading.Thread(target=run, args=(i,)) for i in range(8)]
    for t in ts: t.start()
    for t in ts: t.join()
    assert all(o == want for o in outs)


def test_host_token_walk_gives_the_same_bytes(L, tmp_path):
    img = planar(synth(200, 300, 3, seed=5, kind="noise"))
    np.save(tmp_path / "img.npy", img)
    code = ("import sys, numpy as np; sys.path.insert(0, %r); import __graft_entry__ as G; L = G._pkg(); "
            "sys.stdout.buffer.write(L.webp_encode_rgb_bpred(np.load(%r), 65))") % (ROOT, str(tmp_path / "img.npy"))
    env = dict(os.environ, B200_WEBP_TOKENS="host")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr.decode()
    assert r.stdout == L.webp_encode_rgb_bpred(img, 65)


def test_first_partition_overflow_falls_back_to_the_16x16_bytes(L, OB, bpred_on):
    """8192x4096 noise at q 100: every macroblock takes B_PRED, and their sub-block modes alone pass the 2^19-byte first partition (the
    twin reports the overflow on the same frame); the device then codes the frame 16x16-only, byte for byte the switch-off file"""
    rng = np.random.default_rng(0)
    img = rng.integers(0, 256, (3, 4096, 8192), dtype=np.uint8)
    assert OB.webp_bpred_stages(img, 100, allow_overflow=True)["overflow"]
    on = L.webp_encode_rgb(img, 100)
    forced, _, modes, bmodes = L.webp_encode_rgb_bpred(img, 100, want_stage=True)
    assert not (modes[:, 0] == 4).any() and np.array_equal(bmodes, np.repeat(modes[:, :1], 16, axis=1))
    only_bmodes, outp, outl = np.zeros_like(bmodes), C.POINTER(C.c_uint8)(), C.c_size_t()      # sub-block modes asked for without the modes
    assert L.lib().b200_webp_encode_rgb_bpred(img.ctypes.data_as(C.c_void_p), 8192, 4096, 100, C.byref(outp), C.byref(outl), None, None,
                                              only_bmodes.ctypes.data_as(C.c_void_p)).code == 0
    L.lib().b200_free(outp)
    assert np.array_equal(only_bmodes, bmodes)
    assert L.set_webp_bpred(0) == 0
    assert on == forced == L.webp_encode_rgb(img, 100)


def test_gif_to_webp(L, OB, bpred_on):
    import gif_cases
    from gif_convert_cases import first_frame
    assert L.set_gif_convert(1) == 0
    try:
        for name, data in gif_cases.cases():
            if name not in ("still_m8", "anim_opaque", "g1", "disposal_mix"):
                continue
            f0 = first_frame(data)
            p = L.default_params(); p.webp_quality = 75
            out = L.convert_in_memory(data, p, FMT_WEBP)
            frame = OB.webp_bpred_encode(planar(np.ascontiguousarray(f0[..., :3])), 75)
            if (f0[..., 3] == 0).any():
                assert out[12:16] == b"VP8X" and vp8_chunk(out) == vp8_chunk(frame), name
            else:
                assert out == frame, name
    finally:
        L.set_gif_convert(0)


def test_animated_webp_lossy_frames(L, OB, bpred_on):
    import webp_anim_cases as wc
    from oracle import webp_anim as OW
    assert L.set_webp_anim(1) == 0
    try:
        cases = wc.pillow_cases()
        for name in sorted(cases)[:3]:
            data = cases[name]
            p = L.default_params(); p.webp_quality = 75
            out = L.compress_in_memory(data, p)
            canv, durs, _, _ = L.webp_anim_decode(data)
            tf = OW.frames(canv, durs)
            top = wc._chunks(out)
            anmf = [pl for tag, pl in top if tag == b"ANMF"]
            assert len(anmf) == len(tf)
            for (k, (x, y, w, h), _), pl in zip(tf, anmf):
                sub = dict(wc._chunks(pl, 16))
                rgb = planar(np.ascontiguousarray(canv[k, y:y + h, x:x + w, :3]))
                assert sub[b"VP8 "] == vp8_chunk(OB.webp_bpred_encode(rgb, 75)), name
    finally:
        L.set_webp_anim(0)


def test_max_size_answer_is_the_twin_at_the_landed_quality(L, OB, bpred_on):
    with open(os.path.join(ROOT, "tests", "golden", "reference_samples", "w0.webp"), "rb") as f:
        data = f.read()
    rgb = planar(pil_decode(data))
    for frac in (2, 4):
        target = len(data) // frac
        p = L.default_params(); p.webp_quality = 80
        out = L.compress_to_size_in_memory(data, p, target)
        assert len(out) <= target and out == OB.webp_bpred_encode(rgb, int(p.webp_quality)), (frac, p.webp_quality)
