"""GIF on the device (b200_set_gif): with the switch off every GIF call answers code 3 as before; with it on, the device file
equals the oracle twin's byte for byte at q = 1, 50, 80 and 100, the LZW coder alone equals the twin around segment boundaries and
on several megabytes, and batches and concurrent calls give the single-call bytes."""
import threading

import numpy as np
import pytest

import gif_cases
import gifutil
from oracle import gif as G

pytestmark = pytest.mark.gpu

FMT_JPEG, FMT_PNG, FMT_GIF, FMT_WEBP = 0, 1, 2, 3
GIF_SEG = 16384
CASES = gif_cases.cases()
IDS = [n for n, _ in CASES]


@pytest.fixture
def gif(L):
    assert L.set_gif(True) == 0
    yield L
    L.set_gif(False)


def params(L, q):
    p = L.default_params()
    p.gif_quality = q
    return p


def twin(data, q):
    frames, loop = gifutil.decode(data)
    return G.gif_encode(np.stack([c for c, _ in frames]), [d for _, d in frames], -1 if loop is None else loop, q)


def test_switch_off_answers_unsupported(L):
    assert L.set_gif(False) == 0
    data = dict(CASES)["anim_disposal2"]
    with pytest.raises(L.B200Error) as e:
        L.compress_in_memory(data, params(L, 80))
    assert e.value.code == L.ERR_UNSUPPORTED
    res = L.compress_batch([data, data], params(L, 80))
    assert [r[1] for r in res] == [L.ERR_UNSUPPORTED] * 2
    assert L.lib().b200_set_gif(2) == L.ERR_INVALID_ARGUMENT


def test_refusals_stay_with_the_switch_on(gif):
    L = gif
    data = dict(CASES)["anim_disposal1"]
    p = params(L, 80)
    p.width = 10
    for call in (lambda: L.compress_in_memory(data, p), lambda: L.compress_to_size_in_memory(data, params(L, 80), 100),
                 lambda: L.convert_in_memory(data, params(L, 80), FMT_PNG), lambda: L.convert_in_memory(data, params(L, 80), FMT_WEBP)):
        with pytest.raises(L.B200Error) as e:
            call()
        assert e.value.code == L.ERR_UNSUPPORTED
    past = gif_cases.raw_gif(6, 2, [dict(x=3, y=0, idx=np.zeros((2, 4), np.uint8), table=[(0, 0, 0), (1, 1, 1)], m=2)])
    with pytest.raises(L.B200Error) as e:
        L.compress_in_memory(past, params(L, 80))
    assert e.value.code == L.ERR_UNSUPPORTED
    with pytest.raises(L.B200Error) as e:
        L.compress_in_memory(data[:len(data) // 2], params(L, 80))
    assert e.value.code == L.ERR_CORRUPT_INPUT


@pytest.mark.parametrize("q", [1, 50, 80, 100])
@pytest.mark.parametrize("name,data", CASES, ids=IDS)
def test_device_equals_twin(gif, name, data, q):
    out = gif.compress_in_memory(data, params(gif, q))
    assert out == twin(data, q), (name, q)


@pytest.mark.parametrize("m", [2, 5, 8])
def test_lzw_hook_equals_twin(L, m):
    rng = np.random.default_rng(m)
    for n in (1, GIF_SEG - 1, GIF_SEG, GIF_SEG + 1, 3 * GIF_SEG, 6 << 20):
        idx = rng.integers(0, 1 << m, n).astype(np.uint8)
        if n == 6 << 20:
            idx[: n // 2] = np.repeat(idx[: n // 64], 32)[: n // 2]          # long runs as well as noise
        out = L.gif_lzw(idx, m)
        assert out == G.gif_lzw(idx, m), (m, n)
        if n <= 3 * GIF_SEG:
            body, _ = gifutil._blocks(out, 0)
            assert gifutil.lzw_decode(body, m, n) == idx.tobytes()


def test_mixed_batch_and_concurrent_calls_equal_single_calls(gif, golden):
    L = gif
    p = params(L, 60)
    p.png_optimize = 1                                          # lossless PNG: the lossy PNG switch stays off
    gifs = [d for n, d in CASES if n in ("g1", "disposal_mix", "anim_disposal3", "noise")]
    single = [L.compress_in_memory(d, p) for d in gifs]
    jpeg = golden("in_420_base_640x480.jpg")
    png = golden("reference_samples/p2.png")
    mixed = [gifs[0], jpeg, gifs[1], png, gifs[2], gifs[3]]
    res = L.compress_batch(mixed, p, n_threads=4)
    assert all(r[1] == 0 for r in res)
    assert [res[i][0] for i in (0, 2, 4, 5)] == single
    assert res[1][0] == L.compress_in_memory(jpeg, p) and res[3][0] == L.compress_in_memory(png, p)
    got = [None] * 8

    def run(k):
        got[k] = L.compress_in_memory(gifs[k % 4], p)
    th = [threading.Thread(target=run, args=(k,)) for k in range(8)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert got == single + single
