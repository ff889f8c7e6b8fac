"""The animated WebP leg on the device: the container, frame rectangles, flags and durations against the oracle twin's frame rule
over the host decoder's canvases; every frame's payload against the still encoders on the twin's cropped rectangle; lossless output
decoded by Pillow against the source canvases (the device compositor end to end); lossy output as Pillow shows it; batches and
concurrent calls against single calls; and the refusals that stay with the switch on."""
import io
import os
import subprocess
import sys
import struct
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
from PIL import Image

import webp_anim_cases as wc
from oracle import webp_anim as OW

pytestmark = pytest.mark.gpu

CASES = {**wc.pillow_cases(), **wc.hand_cases()}
IDS = sorted(CASES)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def on(L):
    assert L.lib().b200_init_device(0) == 0
    L.set_webp_anim(1)
    yield L
    L.set_webp_anim(0)


def params(L, lossless, quality=75):
    p = L.default_params()
    p.webp_lossless, p.webp_quality = int(lossless), quality
    return p


def parse(out):
    """-> (VP8X flags, W, H, ANIM payload, [(rect, duration, flags byte, [(tag, payload)])])"""
    assert out[:4] == b"RIFF" and out[8:12] == b"WEBP" and struct.unpack("<I", out[4:8])[0] == len(out) - 8
    top = wc._chunks(out)
    assert [t for t, _ in top[:2]] == [b"VP8X", b"ANIM"] and all(t == b"ANMF" for t, _ in top[2:])
    x8 = top[0][1]
    frames = []
    for _, p in top[2:]:
        rect = (2 * int.from_bytes(p[0:3], "little"), 2 * int.from_bytes(p[3:6], "little"), 1 + int.from_bytes(p[6:9], "little"),
                1 + int.from_bytes(p[9:12], "little"))
        frames.append((rect, int.from_bytes(p[12:15], "little"), p[15], wc._chunks(p, 16)))
    return x8[0], 1 + int.from_bytes(x8[4:7], "little"), 1 + int.from_bytes(x8[7:10], "little"), top[1][1], frames


def twin(L, data):
    canv, durs, loop, bg = L.webp_anim_decode(data)
    return canv, OW.frames(canv, durs), loop, bg


def check_container(L, data, out):
    canv, tf, loop, bg = twin(L, data)
    flags, W, H, anim, frames = parse(out)
    kept = np.stack([canv[k] for k, _, _ in tf])
    assert (W, H) == (canv.shape[2], canv.shape[1])
    assert flags == 0x02 | (0x10 if (kept[..., 3] < 255).any() else 0)
    assert anim == bg + struct.pack("<H", loop)
    assert [(f[0], f[1], f[2]) for f in frames] == [(r, d, 2) for _, r, d in tf]
    return canv, tf, frames


def still_lossless(rgba):
    b = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(rgba), "RGBA").save(b, "WEBP", lossless=True, exact=True)
    return b.getvalue()


@pytest.mark.parametrize("name", IDS)
def test_lossless_matches_twin_and_source(on, name):
    L, data = on, CASES[name]
    out = L.compress_in_memory(data, params(L, True))
    canv, tf, frames = check_container(L, data, out)
    # each frame is what the still lossless encoder makes of the twin's cropped rectangle
    for (k, (x, y, w, h), _), (_, _, _, sub) in zip(tf, frames):
        ref = L.compress_in_memory(still_lossless(canv[k, y:y + h, x:x + w]), params(L, True))
        assert sub == [t for t in wc._chunks(ref) if t[0] == b"VP8L"]
    # decoded by Pillow, the output shows every kept canvas exactly
    pc, pd = wc.pillow_frames(out)
    assert np.array_equal(pc, np.stack([canv[k] for k, _, _ in tf]))
    assert pd == [d for _, _, d in tf]


@pytest.mark.parametrize("name", IDS)
def test_lossy_frames_match_the_still_encoder(on, name):
    L, data = on, CASES[name]
    out = L.compress_in_memory(data, params(L, False, 75))
    canv, tf, frames = check_container(L, data, out)
    for (k, (x, y, w, h), _), (_, _, _, sub) in zip(tf, frames):
        ref = L.compress_in_memory(still_lossless(canv[k, y:y + h, x:x + w]), params(L, False, 75))
        assert sub == [t for t in wc._chunks(ref) if t[0] in (b"ALPH", b"VP8 ")]
    im = Image.open(io.BytesIO(out))
    assert im.n_frames == len(tf) and im.info.get("loop") == twin(L, data)[2]
    pc, pd = wc.pillow_frames(out)
    assert pd == [d for _, _, d in tf]


def test_batch_and_threads_give_single_call_bytes(on):
    L = on
    names = IDS[:8]
    for lossless in (False, True):
        p = params(L, lossless)
        single = [L.compress_in_memory(CASES[n], p) for n in names]
        assert [r[0] for r in L.compress_batch([CASES[n] for n in names], p)] == single
        with ThreadPoolExecutor(8) as ex:
            assert list(ex.map(lambda n: L.compress_in_memory(CASES[n], p), names * 3)) == single * 3


def test_larger_animation(on):
    L = on
    rng = np.random.default_rng(3)
    base = wc.rgba_image(rng, 480, 270, "opaque")
    ims = []
    for k in range(12):
        f = base.copy()
        f[20 + 5 * k:80 + 5 * k, 30 + 9 * k:150 + 9 * k] = wc.rgba_image(rng, 120, 60, "mixed")
        ims.append(Image.fromarray(f, "RGBA"))
    b = io.BytesIO()
    ims[0].save(b, "WEBP", save_all=True, append_images=ims[1:], duration=40, loop=0, lossless=True, exact=True)
    data = b.getvalue()
    out = L.compress_in_memory(data, params(L, True))
    canv, tf, _ = check_container(L, data, out)
    assert np.array_equal(wc.pillow_frames(out)[0], np.stack([canv[k] for k, _, _ in tf]))


def test_refusals_with_the_switch_on(on):
    L, data = on, CASES["pillow_lossy_mixed"]
    p = params(L, False)
    p.height = 10
    with pytest.raises(L.B200Error) as e:
        L.compress_in_memory(data, p)
    assert e.value.code == 3
    with pytest.raises(L.B200Error) as e:
        L.compress_to_size_in_memory(data, params(L, False), len(data) // 2)
    assert e.value.code == 3
    for fmt in (L.FMT_JPEG, L.FMT_PNG, L.FMT_GIF):
        with pytest.raises(L.B200Error) as e:
            L.convert_in_memory(data, params(L, False), fmt)
        assert e.value.code == 3


def test_environment_switch(on):
    L, data = on, CASES["edges"]
    want = L.compress_in_memory(data, params(L, False)).hex()
    code = ("import sys; sys.path.insert(0, %r); import __graft_entry__ as g; L = g._pkg(); p = L.default_params(); p.webp_quality = 75; "
            "sys.stdout.write(L.compress_in_memory(bytes.fromhex(%r), p).hex())") % (ROOT, data.hex())
    env = dict(os.environ, B200_WEBP_ANIM="gpu")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr
    assert r.stdout == want
