"""Cost and effect of trellis quantisation (b200_set_jpeg_trellis) on the configs[1] workload: 3840x2160 q90 4:2:0 synthetic JPEGs
re-encoded at -q 80 4:2:0 progressive through the device-resident pipe (b200_jpeg_pipe_*), switch off and on alternating in one
process.  Reports GP/s of each setting (CUDA events around pipe runs), the k_jpeg_trellis row of the per-kernel table, total
output bytes per setting, and the card's name and power limit read in the same call.  GPU machine only.
usage: python tools/jpeg_trellis_probe.py [--batch 128] [--group 8] [--unique 16] [--rounds 3] [--steps 5] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--group", type=int, default=8)
    ap.add_argument("--unique", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from __graft_entry__ import _pkg
    from tools.synth import synth_jpeg
    L = _pkg()
    assert L.lib().b200_init_device(0) == 0, "no H100 visible"
    uniq = [synth_jpeg(3840, 2160, i) for i in range(a.unique)]
    datas = [uniq[i % len(uniq)] for i in range(a.batch)]
    p = L.default_params()
    p.jpeg_quality, p.jpeg_chroma_subsampling, p.jpeg_progressive = 80, 420, 1
    pipes = {}
    for on in (0, 1):
        assert L.set_jpeg_trellis(on) == 0
        pipes[on] = L.JpegPipe(datas, p, group=a.group)          # the pipe reads the switch at create
    L.set_jpeg_trellis(0)
    stream = torch.cuda.current_stream()
    res = {0: [], 1: []}
    try:
        for on in (0, 1):                                         # warm-up
            pipes[on].run(stream.cuda_stream); pipes[on].finish()
        for _ in range(a.rounds):
            for on in (0, 1):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(a.steps):
                    pipes[on].run(stream.cuda_stream)
                e1.record(stream)
                sizes, bad, _ = pipes[on].finish()
                assert bad == 0
                ms = e0.elapsed_time(e1) / a.steps
                res[on].append({"ms_per_step": round(ms, 3), "gpix_per_s": round(a.batch * 3840 * 2160 / ms / 1e6, 2), "bytes": int(sum(sizes))})
        kt = pipes[1].kernel_times(iters=3)
    finally:
        for pp in pipes.values():
            pp.close()
    best = {on: min(r["ms_per_step"] for r in res[on]) for on in (0, 1)}
    out = {"card": card(), "workload": f"{a.batch} x 3840x2160 q90 4:2:0 synthetic ({a.unique} unique) -> q80 4:2:0 progressive, resident pipe, group {a.group}",
           "off": res[0], "on": res[1],
           "best_ms_per_step": {"off": best[0], "on": best[1]}, "trellis_cost_ms_per_step": round(best[1] - best[0], 3),
           "bytes": {"off": res[0][-1]["bytes"], "on": res[1][-1]["bytes"], "ratio_on_over_off": round(res[1][-1]["bytes"] / res[0][-1]["bytes"], 4)},
           "k_jpeg_trellis": {"ms_per_launch": kt["k_jpeg_trellis"][0], "launches_per_megabatch": kt["k_jpeg_trellis"][1],
                              "megabatches_per_step": (a.batch + a.group - 1) // a.group}}
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
