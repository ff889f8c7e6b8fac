"""The animated WebP leg on the CPU: the host decoder hook (b200_webp_anim_decode) against Pillow's WebPAnimDecoder and against the
oracle twin fed by an independent reader, refusals of corrupt and mutated files, and the answers of the calls with the switch off
(and, for the refusals that do not depend on it, on)."""
import numpy as np
import pytest

import webp_anim_cases as wc
from oracle import webp_anim as OW

CASES = {**wc.pillow_cases(), **wc.hand_cases()}
IDS = sorted(CASES)
ANIM_MSG = "animated WebP is outside the GPU path (route to caesium::compress_in_memory) [3]"


@pytest.mark.parametrize("name", IDS)
def test_hook_equals_pillow_and_oracle(L, name):
    data = CASES[name]
    canv, durs, loop, bg = L.webp_anim_decode(data)
    pc, pd = wc.pillow_frames(data)
    assert np.array_equal(canv, pc)
    assert durs == pd
    W, H, rloop, rbg, frames = wc.read_frames(data)
    assert (canv.shape[2], canv.shape[1], loop, bg) == (W, H, rloop, rbg)
    assert durs == [f[5] for f in frames]
    assert np.array_equal(canv, OW.compose(W, H, [f[:5] for f in frames]))


def test_cases_reach_every_rule():
    # blend x dispose pairs, the background bytes kept, loop counts at both ends, durations at the top of the range
    assert {n for n in CASES if n.startswith("pair_")} == {f"pair_b{b}_d{d}" for b in (0, 1) for d in (0, 1)}
    _, _, loop, bg, _ = wc.read_frames(CASES["odd_1x1"])
    assert (loop, bg) == (65535, b"\x10\x20\x30\x40")
    assert max(f[5] for f in wc.read_frames(CASES["repeats_durations"])[4]) == (1 << 24) - 1


def test_background_colour_is_not_painted(L):
    canv = L.webp_anim_decode(CASES["odd_1x1"])[0]
    assert (canv[0].reshape(-1, 4) == 0).all(axis=1).sum() == 17 * 13 - 1


def test_oracle_frame_rule():
    canv, durs = wc.pillow_frames(CASES["repeats_durations"])
    out = OW.frames(canv, durs)
    # the three equal full canvases merge into one frame whose duration saturates; so do the three equal 8x8 updates
    assert [k for k, _, _ in out] == [0, 3]
    assert out[0][2] == (1 << 24) - 1 and out[1][2] == 12
    assert out[0][1] == (0, 0, 40, 30)
    x, y, w, h = out[1][1]
    assert x % 2 == 0 and y % 2 == 0 and x <= 4 and y <= 4 and x + w <= 12 and y + h <= 12


@pytest.mark.parametrize("name", [n for n, _ in wc.corrupt_cases()[1]])
def test_corrupt_files_answer_code_4(L, name):
    data = dict(wc.corrupt_cases()[1])[name]
    with pytest.raises(L.B200Error) as e:
        L.webp_anim_decode(data)
    assert e.value.code == 4


def test_mutated_files_never_crash(L):
    good, _ = wc.corrupt_cases()
    rng = np.random.default_rng(5)
    codes = set()
    for it in range(600):
        d = bytearray(good)
        mode = it % 3
        if mode == 0:
            for _ in range(1 + it % 5):
                d[int(rng.integers(12, len(d)))] = int(rng.integers(0, 256))
        elif mode == 1:
            d = d[: int(rng.integers(1, len(d)))]
        else:
            i = int(rng.integers(12, len(d)))
            d[i:i] = bytes(rng.integers(0, 256, int(rng.integers(1, 30)), dtype=np.uint8))
        try:
            L.webp_anim_decode(bytes(d))
            codes.add(0)
        except L.B200Error as e:
            codes.add(e.code)
    assert codes <= {0, 4}


@pytest.fixture
def switch(L):
    yield L.set_webp_anim
    L.set_webp_anim(0)


def test_switch_values(L, switch):
    assert switch(2) == 1 and switch(-1) == 1          # B200_ERR_INVALID_ARGUMENT
    assert switch(1) == 0 and switch(0) == 0


def _answer(fn):
    try:
        fn()
    except Exception as e:  # B200Error
        return e.code, str(e)
    return 0, ""


def test_switch_off_answers_as_before(L, switch):
    switch(0)
    data = CASES["pillow_lossy_mixed"]
    p = L.default_params()
    assert _answer(lambda: L.compress_in_memory(data, p)) == (3, ANIM_MSG)
    p.webp_lossless = 1
    assert _answer(lambda: L.compress_in_memory(data, p)) == (3, ANIM_MSG)
    assert L.compress_batch([data, data], L.default_params()) == [(None, 3, ANIM_MSG)] * 2
    assert _answer(lambda: L.webp_decode(data))[0] == 3


@pytest.mark.parametrize("on", [0, 1])
def test_refusals_either_way(L, switch, on):
    switch(on)
    data = CASES["pillow_lossless_mixed"]
    p = L.default_params()
    p.width = 20
    want = 3 if on else (3, ANIM_MSG)
    got = _answer(lambda: L.compress_in_memory(data, p))
    assert (got[0] if on else got) == want
    p = L.default_params()
    assert _answer(lambda: L.compress_to_size_in_memory(data, p, len(data) // 2)) == (3, ANIM_MSG)
    for fmt in (L.FMT_JPEG, L.FMT_PNG, L.FMT_GIF):
        assert _answer(lambda: L.convert_in_memory(data, p, fmt))[0] == 3
    assert _answer(lambda: L.webp_decode(data))[0] == 3
    assert _answer(lambda: L.webp_decode_rgba(data))[0] == 3


def test_switch_on_refuses_corrupt_before_any_device(L, switch):
    switch(1)
    for name, data in wc.corrupt_cases()[1]:
        assert _answer(lambda: L.compress_in_memory(data, L.default_params()))[0] == 4, name
