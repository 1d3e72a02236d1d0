"""Multi-GPU: shard independent messages over the ranks of one node, all-gather the digest table.

Files / map inputs / 8 MiB blocks / multipart parts carry no cross-message state, so the path shards with
no data-path collective; the only exchange is the fixed-width digest table (48 B per message:
SHA-256 || MD5), all-gathered once over NCCL (NVLink / NVSwitch) -- or gloo in the CPU tests.
One process per GPU (torchrun); every rank ends up with the full table in the caller's message order.
"""
from __future__ import annotations

import numpy as np

from ._backend import get_context
from ._lib import MD5, SHA256, TRIM_ZEROS
from .batch import DigestTable


def gpu_node_cpus(device: int) -> set[int] | None:
    """CPUs of the NUMA node CUDA device ``device`` hangs off (sysfs), or None when that cannot be told."""
    import os

    try:
        import torch

        p = torch.cuda.get_device_properties(device)
        bdf = f"{p.pci_domain_id:04x}:{p.pci_bus_id:02x}:{p.pci_device_id:02x}.0"
        with open(f"/sys/bus/pci/devices/{bdf}/numa_node") as f:
            node = int(f.read().strip())
        if node < 0:
            return None
        with open(f"/sys/devices/system/node/node{node}/cpulist") as f:
            text = f.read().strip()
    except Exception:
        return None
    cpus: set[int] = set()
    for part in text.split(","):
        a, _, b = part.partition("-")
        cpus.update(range(int(a), int(b or a) + 1))
    cpus &= os.sched_getaffinity(0)
    return cpus or None


def bind_process_to_gpu_node(device: int) -> bool:
    """One process per GPU: run this process (and every thread it starts later) on the CPUs next to its GPU, so that
    the payloads it allocates, the pinned staging ring and the packer threads all sit in the memory the GPU's DMA
    engine reads from.  torchrun does not do this; without it 8 ranks packing pageable payloads push most bytes
    across the socket interconnect.  Returns whether it bound."""
    import os

    cpus = gpu_node_cpus(device)
    if not cpus:
        return False
    try:
        os.sched_setaffinity(0, cpus)
        return True
    except OSError:
        return False


def shard_assignment(lengths, world: int) -> list[np.ndarray]:
    """Byte-balanced partition of message indices over ``world`` ranks: sort by length (longest first) and
    deal in boustrophedon order (0..w-1, w-1..0, ...), the vectorisable cousin of LPT list scheduling.
    Returns one ascending index array per rank.  Deterministic, so every rank computes the same plan."""
    lengths = np.asarray(lengths, dtype=np.uint64)
    n = lengths.size
    order = np.argsort(-lengths.astype(np.int64), kind="stable")
    pos = np.arange(n)
    lap, col = pos // world, pos % world
    owner_sorted = np.where(lap % 2 == 0, col, world - 1 - col)
    owner = np.empty(n, np.int64)
    owner[order] = owner_sorted
    return [np.flatnonzero(owner == r) for r in range(world)]


def all_gather_table(local, counts: list[int], group=None, device=None, to_host: bool = True):
    """All-gather per-rank uint8[count_r, W] tables (padded to the largest count) -> list of per-rank tables.
    ``local`` may be a numpy array (copied to the device once) or a CUDA tensor that is already there -- a table that
    the hash call wrote into device memory never visits the host before the exchange.  ``to_host=False`` returns
    device tensors (views of one gathered buffer) instead of numpy arrays."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group)
    width = int(local.shape[1])
    cap = max(max(counts), 1)
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend(group) == "nccl" else torch.device("cpu")
    rows = int(local.shape[0])
    if isinstance(local, torch.Tensor) and local.device == torch.device(device) and rows == cap and local.is_contiguous():
        send = local  # already padded and in place
    else:
        send = torch.zeros((cap, width), dtype=torch.uint8, device=device)
        if rows:
            src = local if isinstance(local, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(local))
            send[:rows] = src.to(device)
    recv = torch.empty((world * cap, width), dtype=torch.uint8, device=device)
    dist.all_gather_into_tensor(recv, send, group=group)
    if not to_host:
        g = recv.view(world, cap, width)
        return [g[r, : counts[r]] for r in range(world)]
    host = recv.cpu().numpy().reshape(world, cap, width)
    return [host[r, : counts[r]] for r in range(world)]


def hash_table_sharded(base, offsets, lengths, *, sha256: bool = True, md5: bool = True, trim_zeros: bool = False,
                       group=None, ctx=None) -> DigestTable:
    """Every rank passes the SAME (offsets, lengths) description of the whole message set and a ``base`` in
    which at least its own shard is readable; each rank hashes only its shard on its own GPU, then the
    48-byte rows (+ 8-byte hashed length) are all-gathered and un-permuted into message order.
    Over NCCL the shard's table is written by the hash call straight into device memory (the outputs of
    b200h_hash_batch_host may be device pointers), gathered there, and copied to the host once, whole."""
    import torch.distributed as dist

    offsets = np.asarray(offsets, dtype=np.uint64)
    lengths = np.asarray(lengths, dtype=np.uint64)
    n = offsets.size
    flags = (SHA256 if sha256 else 0) | (MD5 if md5 else 0) | (TRIM_ZEROS if trim_zeros else 0)
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        s, m, t = (ctx or get_context()).hash_batch_host(base, offsets, lengths, flags)
        return DigestTable(s, m, t)
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    plan = shard_assignment(lengths, world)
    mine = plan[rank]
    counts = [p.size for p in plan]
    context = ctx or get_context()
    if dist.get_backend(group) == "nccl":
        import torch

        dev = torch.device("cuda", context.device)
        cap = max(max(counts), 1)
        # one buffer per rank, column blocks: sha[cap,32] | md5[cap,16] | hashed_len[cap] -- 56 bytes per row
        rows = torch.zeros(cap * 56, dtype=torch.uint8, device=dev)
        p = rows.data_ptr()
        context.hash_batch_host(base, offsets[mine], lengths[mine], flags, out_sha=p if sha256 else 0,
                                out_md5=p + 32 * cap if md5 else 0, out_trimmed=p + 48 * cap)
        recv = torch.empty(world * cap * 56, dtype=torch.uint8, device=dev)
        dist.all_gather_into_tensor(recv, rows, group=group)
        host = recv.cpu().numpy().reshape(world, cap * 56)  # the only device->host copy: the whole job's table
        sha_full = np.zeros((n, 32), np.uint8) if sha256 else None
        md5_full = np.zeros((n, 16), np.uint8) if md5 else None
        len_full = np.zeros(n, np.uint64)
        for r in range(world):
            c = counts[r]
            if sha256:
                sha_full[plan[r]] = host[r, : 32 * cap].reshape(cap, 32)[:c]
            if md5:
                md5_full[plan[r]] = host[r, 32 * cap : 48 * cap].reshape(cap, 16)[:c]
            len_full[plan[r]] = host[r, 48 * cap :].view("<u8")[:c]
        return DigestTable(sha_full, md5_full, len_full)
    s, m, t = context.hash_batch_host(base, offsets[mine], lengths[mine], flags)
    row = np.zeros((mine.size, 56), np.uint8)
    if s is not None:
        row[:, :32] = s
    if m is not None:
        row[:, 32:48] = m
    row[:, 48:56] = np.ascontiguousarray(t, dtype="<u8").view(np.uint8).reshape(-1, 8)
    tables = all_gather_table(row, counts, group=group)
    full = np.zeros((n, 56), np.uint8)
    for r in range(world):
        full[plan[r]] = tables[r]
    return DigestTable(
        np.ascontiguousarray(full[:, :32]) if sha256 else None,
        np.ascontiguousarray(full[:, 32:48]) if md5 else None,
        np.ascontiguousarray(full[:, 48:56]).view("<u8").reshape(-1).astype(np.uint64),
    )
