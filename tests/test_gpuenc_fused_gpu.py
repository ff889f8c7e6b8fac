"""GPU test of the device encoder's single-pass emission of single-component scans (k_geb_emit's per-thread slots, k_ge_place):
a dense image at quality 100, whose units overflow their 256-bit slot and are coded a second time straight to their place, goes
through the resident pipe and b200_compress_batch and must equal the host encoder byte for byte -- lossy and lossless, progressive
and sequential, colour and grey."""
import io

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _dense_jpeg(w, h, mode, seed):
    """a gradient under +-24 of noise: nearly every AC coefficient is non-zero at quality 100"""
    from PIL import Image
    rng = np.random.default_rng(seed)
    shape = (h, w, 3) if mode == "RGB" else (h, w)
    base = np.add.outer(np.arange(h), np.arange(w)) * 200 // (h + w) + 28
    px = (base.reshape(h, w, *([1] if mode == "RGB" else [])) + rng.integers(-24, 25, size=shape)).clip(0, 255).astype(np.uint8)
    img = Image.fromarray(px, mode)
    buf = io.BytesIO()
    img.save(buf, "JPEG", quality=100, subsampling=0 if mode == "RGB" else -1)
    return buf.getvalue()


def _params(L, prog, lossless):
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive, p.jpeg_optimize = 100, 420, int(prog), int(lossless)
    return p


@pytest.mark.parametrize("lossless", [0, 1])
@pytest.mark.parametrize("prog", [1, 0])
def test_dense_units_overflow_slots(L, prog, lossless):
    import torch
    assert L.lib().b200_init_device(0) == 0
    datas = [_dense_jpeg(520, 264, "RGB", s) for s in range(3)] + [_dense_jpeg(520, 264, "L", 9)]
    p = _params(L, prog, lossless)
    L.set_entropy_mode(0)
    try:
        want = [L.compress_in_memory(d, p) for d in datas]
    finally:
        L.set_entropy_mode(1)
    for d, w, (out, code, msg) in zip(datas, want, L.compress_batch(datas, p, n_threads=2)):
        assert code == 0, msg
        assert out == w
    st = torch.cuda.Stream()
    pipe = L.JpegPipe(datas[:3], p, group=3)
    try:
        pipe.run(st.cuda_stream)
        torch.cuda.synchronize()
        pipe.finish()
        for i in range(3):
            assert pipe.fetch(i) == want[i], i
    finally:
        pipe.close()
