"""Throughput probe: b200_compress_batch over synthetic 4K JPEGs with different host thread counts (B200_TRACE=1 for
the per-stage wall-clock breakdown printed at shutdown).  Two timings per setting: the C-ABI call with its outputs left
in the library's malloc'ed buffers (what a Rust/C host sees), and the same call followed by the ctypes copy of every output
into a Python bytes object (binding overhead, not part of the product).
usage: python tools/throughput.py [threads,threads,...] [n_images]"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402

if __name__ == "__main__":
    threads_list = [int(x) for x in (sys.argv[1] if len(sys.argv) > 1 else "8,16,32").split(",")]
    n_images = int(sys.argv[2]) if len(sys.argv) > 2 else 128
    datas = bench.make_inputs(8, 0)
    if os.environ.get("TOOL_TORCH"):                       # let torch create the CUDA context first, as bench.py does
        import torch
        torch.cuda.init(); torch.zeros(1, device="cuda")
    L = bench.load_pkg()
    L.lib().b200_init_device(0)
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive = 80, 420, 1
    work = [datas[i % len(datas)] for i in range(n_images)]
    bi = L.BatchInputs(work)
    L.compress_batch(work[:48], p, 48, copy=False)          # warm the per-image slots
    for _ in range(2):
        L.compress_batch((work * 4)[:256], p, 32, copy=False)   # and every megabatch worker's slot (buffers are allocated on first use)
    reps = int(os.environ.get("REPS", "4"))
    for th in threads_list:
        for copy in (False, True):
            for rep in range(reps if not copy else 1):      # the first repetition still grows malloc arenas / page-faults fresh output buffers
                c0 = os.times()
                t0 = time.perf_counter()
                res = L.compress_batch(bi, p, th, copy=copy)
                dt = time.perf_counter() - t0
                c1 = os.times()
                assert all(r[1] == 0 for r in res)
                cpu = (c1.user - c0.user + c1.system - c0.system) / dt
                print(f"threads={th:3d} {'+python copy' if copy else 'C-ABI only  '} rep {rep}: {n_images / dt:8.1f} img/s  {n_images * bench.MP_PER_IMAGE / dt:9.1f} MP/s   host CPU busy: {cpu:5.1f} cores "
                      f"(user {(c1.user - c0.user) / dt:.1f}, sys {(c1.system - c0.system) / dt:.1f})", flush=True)
    L.lib().b200_shutdown()
