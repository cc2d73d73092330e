"""Pair-sharded multi-GPU matching (SURVEY.md §8e).

Image pairs are independent, so the path shards with no data-path collective: one process per GPU
(torchrun), rank r takes a contiguous block of pairs, every rank holds a full replica of the
23.7 MB weights.  The only communication is the final gather of fixed-size match indices / scores
(``all_gather`` over NCCL on GPUs, gloo in the CPU tests).  The reference has no distributed code at
all (SURVEY.md §2a); this module is the multi-GPU deployment story for BASELINE config 5.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist


def _parse_cpulist(text: str) -> List[int]:
    cpus: List[int] = []
    for part in text.strip().split(","):
        if not part:
            continue
        lo, _, hi = part.partition("-")
        cpus.extend(range(int(lo), int(hi or lo) + 1))
    return cpus


def gpu_numa_node(device_index: int) -> Optional[int]:
    """NUMA node of a GPU from sysfs (``/sys/bus/pci/devices/<bdf>/numa_node``), or None when it cannot be told."""
    try:
        pr = torch.cuda.get_device_properties(device_index)
        bdf = f"{pr.pci_domain_id:04x}:{pr.pci_bus_id:02x}:{pr.pci_device_id:02x}.0"
        with open(f"/sys/bus/pci/devices/{bdf}/numa_node") as f:
            node = int(f.read().strip())
        return node if node >= 0 else None
    except Exception:
        return None


def bind_to_gpu_numa_node(device_index: int) -> dict:
    """Pin the calling process to the CPUs of the NUMA node its GPU hangs off (one process per GPU).

    Pinned host buffers allocated AFTER this call are first-touched on that node, so the H2D / D2H copies of the
    streaming path (``pipeline.match_stream``) do not cross the inter-socket link, and the threads that enqueue the
    kernels run next to the GPU.  Without it the end-to-end throughput of a multi-rank job depends on where the
    scheduler happened to place each rank (round 1: 0.62 of the resident rate at 2 ranks).  Returns what was done;
    never raises (containers without sysfs topology simply stay unpinned)."""
    info = {"device": device_index, "numa_node": None, "cpus": None, "bound": False}
    node = gpu_numa_node(device_index)
    if node is None:
        return info
    info["numa_node"] = node
    try:
        with open(f"/sys/devices/system/node/node{node}/cpulist") as f:
            cpus = set(_parse_cpulist(f.read()))
        allowed = set(os.sched_getaffinity(0))
        use = sorted(cpus & allowed)
        if use:
            os.sched_setaffinity(0, use)
            info["cpus"] = len(use)
            info["bound"] = True
    except Exception:
        pass
    return info


def shard_range(total: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous block [lo, hi) of `total` pairs owned by `rank`; sizes differ by at most one."""
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def gather_matches(local: Dict[str, torch.Tensor], total: int, group=None) -> Dict[str, torch.Tensor]:
    """All-gather the per-rank ``matches0`` [P_r, M] / ``matching_scores0`` (and the image1 side) into
    [total, ...] tensors in pair order.  Indices travel as int32 and are widened back to int64.
    Ragged shards (total % world != 0) are padded to the largest shard for the collective."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    sizes = [shard_range(total, r, world)[1] - shard_range(total, r, world)[0] for r in range(world)]
    pmax = max(sizes)
    out: Dict[str, torch.Tensor] = {}
    for key in ("matches0", "matches1", "matching_scores0", "matching_scores1"):
        t = local[key]
        wire = t.to(torch.int32) if t.dtype == torch.int64 else t
        if wire.shape[0] < pmax:
            pad = torch.zeros(pmax - wire.shape[0], *wire.shape[1:], dtype=wire.dtype, device=wire.device)
            wire = torch.cat([wire, pad], 0)
        buf = [torch.empty_like(wire) for _ in range(world)]
        dist.all_gather(buf, wire.contiguous(), group=group)
        full = torch.cat([b[: sizes[r]] for r, b in enumerate(buf)], 0)
        out[key] = full.to(torch.int64) if t.dtype == torch.int64 else full
    del rank
    return out


def match_sharded(matcher, data: dict, batch: int = 32, group=None) -> Dict[str, torch.Tensor]:
    """Match `total` pairs given on every rank as CPU tensors: each rank runs its shard through
    `matcher` (on its own GPU) in batches of `batch` pairs, then the results are gathered."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    total = data["image0"]["keypoints"].shape[0]
    lo, hi = shard_range(total, rank, world)
    dev = next(matcher.parameters()).device
    parts: List[Dict[str, torch.Tensor]] = []
    for b0 in range(lo, hi, batch):
        b1 = min(hi, b0 + batch)
        chunk = {k: {kk: vv[b0:b1].to(dev, non_blocking=True) for kk, vv in v.items()} for k, v in data.items()}
        o = matcher(chunk)
        parts.append({k: o[k] for k in ("matches0", "matches1", "matching_scores0", "matching_scores1")})
    m, n = data["image0"]["keypoints"].shape[1], data["image1"]["keypoints"].shape[1]
    if parts:
        local = {k: torch.cat([p[k] for p in parts], 0) for k in parts[0]}
    else:
        local = {
            "matches0": torch.empty(0, m, dtype=torch.int64, device=dev),
            "matches1": torch.empty(0, n, dtype=torch.int64, device=dev),
            "matching_scores0": torch.empty(0, m, dtype=torch.float32, device=dev),
            "matching_scores1": torch.empty(0, n, dtype=torch.float32, device=dev),
        }
    return gather_matches(local, total, group)
