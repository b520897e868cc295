"""Multi-GPU plumbing: one process per GPU (torchrun), clips sharded across ranks, ONE
broadcast of the packed weights at init and no collective on the hot path.

The reference has no distributed code at all; its multi-GPU recipe is N independent CLI
processes racing over a file list (reference README.md:53-56, cli.py:178-184).  Here rank 0
reads and packs the checkpoint and every other rank receives the packed blob through one
``torch.distributed.broadcast`` (NCCL over NVLink on the GPU box, gloo in the CPU tests).
"""
from __future__ import annotations

import os

import numpy as np
import torch
import torch.distributed as dist


def env_rank_world():
    return int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))


def init_from_env(backend: str | None = None):
    """Initialise the default process group from torchrun's environment (no-op for 1 rank)."""
    rank, world, local = env_rank_world()
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, world, local


def shard_indices(n_items: int, rank: int, world: int) -> list[int]:
    """Round-robin shard of clip indices (clips are independent; BASELINE config 3)."""
    return list(range(rank, n_items, world))


def shard_by_cost(costs, world: int) -> list[list[int]]:
    """Greedy longest-first balancing by chunk count for ragged clip lengths (config 5):
    returns, per rank, the item indices it owns."""
    order = sorted(range(len(costs)), key=lambda i: -costs[i])
    load = [0] * world
    out = [[] for _ in range(world)]
    for i in order:
        r = min(range(world), key=lambda k: load[k])
        out[r].append(i)
        load[r] += costs[i]
    return [sorted(o) for o in out]


def broadcast_packed(packed: dict | None, hparams: dict | None, device, src: int = 0):
    """Broadcast (hparams, packed parameters) from ``src`` to every rank: the index travels as
    a small object list, the weights as ONE flat fp32 tensor (81 MB for final0)."""
    from .weights import blob_from_packed, packed_from_blob

    if not dist.is_initialized() or dist.get_world_size() == 1:
        return packed, hparams
    rank = dist.get_rank()
    meta = [None]
    if rank == src:
        blob, names, sizes = blob_from_packed(packed)
        meta = [(names, sizes, hparams)]
    dist.broadcast_object_list(meta, src=src)
    names, sizes, hparams = meta[0]
    total = int(sum(sizes))
    dev = torch.device(device)
    if rank == src:
        t = torch.from_numpy(blob).to(dev)
    else:
        t = torch.empty(total, dtype=torch.float32, device=dev)
    dist.broadcast(t, src=src)
    if rank == src:
        return packed, hparams
    return packed_from_blob(t.cpu().numpy(), names, sizes), hparams


def load_model_distributed(checkpoint_path, device, float16=False, wave_chunks=None, max_chunk_size=1500):
    """load_model for torchrun jobs: rank 0 loads + packs, one broadcast, every rank uploads.  The RoPE tables of
    max_chunk_size rows travel in the blob, and every rank's model takes its maximum chunk length from them."""
    from .inference import BeatThisB200, check_max_chunk_size, load_checkpoint
    from .utils import replace_state_dict_key
    from .weights import filter_hparams, pack_parameters

    max_chunk_size = check_max_chunk_size(max_chunk_size)
    rank = dist.get_rank() if dist.is_initialized() else 0
    packed, hparams = None, None
    if rank == 0:
        ckpt = load_checkpoint(checkpoint_path, "cpu")
        hparams = filter_hparams(ckpt["hyper_parameters"])
        packed = pack_parameters(replace_state_dict_key(dict(ckpt["state_dict"]), "model.", ""), hparams,
                                 rope_positions=max_chunk_size)
    packed, hparams = broadcast_packed(packed, hparams, device)
    return BeatThisB200(hparams, packed, device, float16, wave_chunks)


def gather_results(local_results: dict, world: int):
    """Collect per-rank {clip index: result} dicts on every rank (tiny: timestamps only)."""
    if not dist.is_initialized() or world == 1:
        return local_results
    out = [None] * world
    dist.all_gather_object(out, local_results)
    merged = {}
    for d in out:
        merged.update(d)
    return merged
