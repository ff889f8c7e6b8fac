"""Sharding of an image list over ranks (one process per GPU) -- the multi-GPU shape of caesiumclt's data-parallel map
over files (caesium-clt's src/compressor.rs:74-101).  Images are independent, so there is no collective on the data
path: each rank takes its shard, and results are put back in input order (par_iter().collect() semantics).  The only
exchange is the one-time broadcast of the quantisation tables (a handshake, not a bandwidth operation)."""


def shard_indices(sizes, world_size, rank, policy="lpt"):
    """Indices this rank processes.  "lpt": greedy longest-processing-time on byte sizes (balanced work for mixed
    inputs); "rr": round robin (homogeneous synthetic sets).  Deterministic, identical on every rank."""
    n = len(sizes)
    if world_size <= 1:
        return list(range(n))
    if policy == "rr":
        return list(range(rank, n, world_size))
    order = sorted(range(n), key=lambda i: (-int(sizes[i]), i))
    load = [0] * world_size
    owner = [0] * n
    for i in order:
        r = min(range(world_size), key=lambda k: (load[k], k))
        owner[i] = r
        load[r] += int(sizes[i])
    return [i for i in range(n) if owner[i] == rank]


def merge_in_input_order(n, shards, results):
    """shards[r] = indices of rank r, results[r] = that rank's outputs in the same order -> list of n in input order."""
    out = [None] * n
    for idx, res in zip(shards, results):
        for i, v in zip(idx, res):
            out[i] = v
    return out


def broadcast_quant_table(table_u16, dist, src=0, device=None):
    """Rank `src` sends its 64-entry table (NCCL on GPUs, gloo in the CPU tests); every rank returns what it received."""
    import numpy as np
    import torch
    t = torch.tensor(np.asarray(table_u16, dtype=np.int32), device=device)
    if dist is not None and dist.is_initialized() and dist.get_world_size() > 1:
        dist.broadcast(t, src)
    return t.cpu().numpy().astype(np.uint16)
