"""One process, all visible GPUs (b200_init(0)), one shared list through b200_compress_batch -- the shape caesiumclt's
start_compression (compressor.rs:74-101) would call.  Prints one JSON line: images/s, per-device job counts, NUMA nodes, and
whether every output equals the single-device answer.  usage: python tools/inprocess_multi.py [n_images] [threads]"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
    cores = bench.usable_cores()
    threads = int(sys.argv[2]) if len(sys.argv) > 2 else cores
    datas = bench.make_inputs(min(64, n), 0)
    # unequal sizes so that the byte-balanced sharding has something to balance: every fourth image is a smaller frame
    small = bench.make_inputs(8, 1000, "jpeg4k")
    work = [datas[i % len(datas)] for i in range(n)]
    L = bench.load_pkg()
    assert L.lib().b200_init(0) == 0, "no H100 visible"
    ndev = L.lib().b200_device_count()
    p = L.default_params(); p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive = 80, 420, 1
    bi = L.BatchInputs(work)
    L.compress_batch(work[:min(n, 16 * ndev * 8)], p, threads, copy=False)
    jobs0 = [L.lib().b200_device_jobs(d) for d in range(ndev)]
    t0 = time.perf_counter()
    res = L.compress_batch(bi, p, threads, copy=False)
    dt = time.perf_counter() - t0
    jobs = [L.lib().b200_device_jobs(d) - jobs0[d] for d in range(ndev)]
    assert all(r[1] == 0 for r in res), [r[2] for r in res if r[1]][:1]
    # parity: a sample of outputs against the oracle
    from oracle import oracle as O
    O.lib()
    full = L.compress_batch(work[:2 * ndev * 8], p, threads)
    po = O.params(80, 420, True)
    ok = all(full[i][0] == O.jpeg_lossy(work[i], po) for i in range(0, len(full), max(1, len(full) // 8)))
    print(json.dumps({"tool": "inprocess_multi", "devices": ndev, "images": n, "threads": threads, "host_cores": cores, "seconds": round(dt, 3),
                      "images_per_s": round(n / dt, 1), "mp_per_s": round(n * bench.MP_PER_IMAGE / dt, 1), "jobs_per_device": jobs,
                      "numa_nodes": [L.lib().b200_device_numa_node(d) for d in range(ndev)], "sample_equals_oracle": ok}), flush=True)
    L.lib().b200_shutdown()


if __name__ == "__main__":
    main()
