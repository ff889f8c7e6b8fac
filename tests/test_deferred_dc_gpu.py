"""Lossy megabatches and the resident pipe skip the decoder's DC scatter: the decoded blocks keep their DC differences and the
transform kernels (k_fused_same, k_idct_plane) add the per-component prefix sums themselves (GpuDecoder::Item::defer_dc).

Run with -m gpu: lossy outputs against the oracle at every sampling geometry the suite uses, at both output samplings, with
dense then sparse inputs through the same slot, with trellis quantisation, with a megabatch member that goes to the host
decoder, and through the resident pipe.  --lossless keeps the scatter and is covered by test_gpudec_write_gpu.py."""
import pytest

import test_gpudec_damaged as D
from test_gpudec_write_gpu import pair

SHAPES = [("420", 355, 237), ("444", 355, 237), ("422", 355, 237), ("grey", 355, 237), ("grey22", 355, 237), ("420", 640, 480), ("420", 17, 9)]


def _lossy(L, O, ss, q=80):
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive = q, ss, 1
    return p, O.params(q, ss, True)


def _check_megabatches(L, O, layout, w, h, trellis):
    from oracle import jpeg_trellis as T
    L.set_entropy_mode(3)
    assert L.set_jpeg_trellis(1 if trellis else 0) == 0
    try:
        dense, sparse = pair(layout, w, h)
        for ss in (0, 420):
            p, op = _lossy(L, O, ss)
            want = {d: (T.jpeg_lossy if trellis else O.jpeg_lossy)(d, op) for d in (dense, sparse)}
            for d in (dense, sparse, dense):
                for out, code, msg in L.compress_batch([d] * 3, p, n_threads=1):
                    assert code == 0 and out == want[d], (layout, w, h, ss, trellis, d is dense, msg)
    finally:
        assert L.set_jpeg_trellis(0) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("layout,w,h", SHAPES)
def test_megabatch_lossy_matches_oracle(L, O, layout, w, h):
    _check_megabatches(L, O, layout, w, h, False)


@pytest.mark.gpu
@pytest.mark.parametrize("layout,w,h", [("420", 131, 77), ("444", 67, 45)])
def test_megabatch_lossy_trellis_matches_oracle(L, O, layout, w, h):
    _check_megabatches(L, O, layout, w, h, True)


@pytest.mark.gpu
def test_megabatch_with_a_member_on_the_host_decoder(L, O, golden):
    """A damaged member is decoded on the host and transformed on its own; the others take the deferred DC."""
    L.set_entropy_mode(3)
    data = golden("in_420_base_640x480.jpg")
    start, end = D.scan_bounds(data)
    bad = data[:start + (end - start) // 2] + b"\xff\xd9"             # the scan ends halfway: the device flags it, the host pads
    p, op = _lossy(L, O, 420)
    batch = [data, bad, data, data]
    for d, (out, code, msg) in zip(batch, L.compress_batch(batch, p, n_threads=1)):
        assert code == 0 and out == O.jpeg_lossy(d, op), msg


@pytest.mark.gpu
@pytest.mark.parametrize("layout,w,h", [("420", 640, 480), ("444", 355, 237), ("422", 355, 237), ("grey22", 355, 237)])
def test_resident_pipe_lossy_matches_oracle(L, O, layout, w, h):
    import torch
    assert L.lib().b200_init_device(0) == 0
    dense, sparse = pair(layout, w, h)
    p, op = _lossy(L, O, 420)
    want = {d: O.jpeg_lossy(d, op) for d in (dense, sparse)}
    st = torch.cuda.Stream()
    work = [dense] * 2 + [sparse] * 2
    pipe = L.JpegPipe(work, p, group=2)
    try:
        for _ in range(2):
            pipe.run(st.cuda_stream)
        torch.cuda.synchronize()
        _, not_settled, _ = pipe.finish()
        assert not_settled == 0
        for i, d in enumerate(work):
            assert pipe.fetch(i) == want[d], i
    finally:
        pipe.close()
