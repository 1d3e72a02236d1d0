"""tools/j1_matrix.py -- BASELINE.json configs C3 / C4 / C5 on 1/2/4/8 GPUs with the reference's CPU path beside them.

  torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 tools/j1_matrix.py [c3] [c4] [c5] [cpu]

Every rank generates its share of the synthetic bytes in HBM (counter-based generator, same stream on every
machine), and for each configuration reports
  kernel   HBM-resident: b200h_hash_batch_device (+ the NCCL all-gather of the 56-byte rows), CUDA events, max over ranks
  e2e      the same messages from PAGEABLE host memory through b200h_hash_batch_host (pack + H2D + kernels + D2H),
           wall clock between barriers, max over ranks (bounded to <= E2E_CAP bytes per rank, stated per row)
  cpu      (rank 0, only with the `cpu` argument, meant for the 1-GPU run) the reference's own functions loaded
           through oracle/ref_shim.py on the same bytes -- single thread, ThreadPoolExecutor() default workers
           min(32, ncpu+4), workers = ncpu, and for volumefs2 blocks FileUploadSpec2.from_fileobj under
           Semaphore(cpu_count) -- as BASELINE.md section 3 prescribes, on a bounded prefix (stated per row).
C3 is STRONG scaling (the 100 GiB / 1 Mi-file tree is split over the ranks by sharding.shard_assignment), C5 is weak
(8 GiB per GPU per point), C4 is one 10 GiB stream on one GPU.  One JSON line per row on stdout (rank 0) and appended
to j1_out/j1_n<N>.jsonl.  Environment: J1_C3_GIB (100), J1_C3_FILES (1048576), J1_C5_BYTES (8 GiB), J1_C5_KMAX (10),
J1_C4_GIB (10), J1_E2E_CAP (12.5 GiB), J1_CPU_PREFIX (8 GiB)."""
import asyncio
import io
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist

from modal_client_b200 import _lib, sharding

GiB = float(1 << 30)
rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
which = [a for a in sys.argv[1:]] or ["c3", "c4", "c5"]
WITH_CPU = "cpu" in which
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
if world > 1:
    sharding.bind_process_to_gpu_node(local)
    dist.init_process_group("nccl", device_id=dev)
ctx = _lib.Context(local, pinned_bytes=512 << 20, device_bytes=8 << 30)
st = torch.cuda.Stream(device=dev)
torch.cuda.set_stream(st)
PEAK = 3350.0  # GB/s, NVIDIA H100 SXM data sheet
try:
    PEAK = float(json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:
    pass
E2E_CAP = int(float(os.environ.get("J1_E2E_CAP", 12.5)) * GiB)
CPU_PREFIX = int(float(os.environ.get("J1_CPU_PREFIX", 8)) * GiB)
BOTH = _lib.SHA256 | _lib.MD5
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "j1_out", f"j1_n{world}.jsonl")
os.makedirs(os.path.dirname(OUT), exist_ok=True)


def emit(row: dict):
    if rank == 0:
        line = json.dumps(row)
        print(line, flush=True)
        with open(OUT, "a") as f:
            f.write(line + "\n")


def barrier():
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()


def allmax(x: float) -> float:
    t = torch.tensor([x], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def allsum(x: float) -> float:
    t = torch.tensor([x], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return float(t.item())


def allgather_floats(x: float) -> list:
    t = torch.tensor([x], dtype=torch.float64, device=dev)
    if world == 1:
        return [x]
    out = [torch.zeros_like(t) for _ in range(world)]
    dist.all_gather(out, t)
    return [round(float(o.item()), 3) for o in out]


def gpu_row(name, data, offs, lens, flags, reps=2, gather=True, warm=True, e2e=True, **extra):
    """Kernel-only (HBM-resident) and e2e (pageable host) timing of one message set on every rank."""
    offs = np.ascontiguousarray(offs, np.uint64)
    lens = np.ascontiguousarray(lens, np.uint64)
    n = len(lens)
    d_off = torch.from_numpy(offs.astype(np.int64)).to(dev)
    d_len = torch.from_numpy(lens.astype(np.int64)).to(dev)
    counts = [n]
    if world > 1:
        c = torch.tensor([n], device=dev)
        allc = [torch.zeros_like(c) for _ in range(world)]
        dist.all_gather(allc, c)
        counts = [int(x.item()) for x in allc]
    cap = max(max(counts), 1)
    rows = torch.zeros(cap * 56, dtype=torch.uint8, device=dev)  # sha[cap,32] | md5[cap,16] | trimmed[cap] as one buffer
    sha_p, md5_p, tr_p = rows.data_ptr(), rows.data_ptr() + 32 * cap, rows.data_ptr() + 48 * cap
    recv = torch.empty(world * cap * 56, dtype=torch.uint8, device=dev) if world > 1 and gather else None
    trim = bool(flags & _lib.TRIM_ZEROS)

    h0, h1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def step():
        # lengths are known on the host -> the call only enqueues (trim mode: the planner's count is read back)
        h0.record(st)
        ctx.hash_batch_device(data.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), n, flags,
                              sha_p if flags & _lib.SHA256 else 0, md5_p if flags & _lib.MD5 else 0, tr_p, st.cuda_stream,
                              h_lengths=None if trim else lens)
        h1.record(st)  # this rank's own makespan ends here; the all-gather then waits for the slowest rank
        if recv is not None:
            dist.all_gather_into_tensor(recv, rows)

    if warm:
        step()
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(reps):
        step()
    e1.record(st)
    barrier()
    my_ms = e0.elapsed_time(e1) / reps
    ms = allmax(my_ms)
    per_rank_ms = allgather_floats(my_ms)
    per_rank_hash_ms = allgather_floats(h0.elapsed_time(h1))  # last pass, hash only (before the gather)
    my_bytes = float(lens.astype(np.float64).sum())
    total = allsum(my_bytes)
    outliers = ctx.last_outlier_count
    digest_dev = rows.cpu().numpy()

    # ---- e2e from pageable host memory on a bounded prefix of this rank's messages
    csum = np.cumsum(lens.astype(np.float64))
    k = int(np.searchsorted(csum, E2E_CAP, side="right"))
    k = (max(1, min(n, k)) if n else 0) if e2e else 0
    e2e_gibs = e2e_bytes_total = None
    same = True
    if k:
        span_lo, span_hi = int(offs[:k].min()), int((offs[:k] + lens[:k]).max())
        host = data[span_lo:span_hi].cpu().numpy()  # pageable
        ho = offs[:k] - np.uint64(span_lo)
        ctx.hash_batch_host(host[: min(host.size, 1 << 20)], [0], [min(host.size, 1 << 20)], BOTH)  # page in the path
        barrier()
        t0 = time.perf_counter()
        s, m, t = ctx.hash_batch_host(host, ho, lens[:k], flags)
        barrier()
        dt = allmax(time.perf_counter() - t0)
        e2e_bytes_total = allsum(float(lens[:k].astype(np.float64).sum()))
        e2e_gibs = e2e_bytes_total / GiB / dt
        if s is not None:
            same &= bool(np.array_equal(s, digest_dev[: 32 * cap].reshape(cap, 32)[:k]))
        if m is not None:
            same &= bool(np.array_equal(m, digest_dev[32 * cap : 48 * cap].reshape(cap, 16)[:k]))
        same &= bool(np.array_equal(t, digest_dev[48 * cap :].view("<u8")[:k]))
        del host
    gbps = total / 1e9 / (ms / 1e3)
    emit({"config": name, "n_gpus": world, "messages_total": int(allsum(n)), "bytes_total": int(total),
          "kernel_ms": round(ms, 3), "kernel_GiBps": round(total / GiB / (ms / 1e3), 2), "kernel_GBps": round(gbps, 1),
          "hbm_frac_per_gpu": round(gbps / world / PEAK, 4), "per_rank_ms": per_rank_ms, "per_rank_hash_ms": per_rank_hash_ms,
          "e2e_GiBps": round(e2e_gibs, 2) if e2e_gibs else None,
          "e2e_bytes": int(e2e_bytes_total) if e2e_bytes_total else None, "e2e_equals_kernel_digests": same,
          "outliers_on_rank0": outliers, "flags": flags, **extra})
    return digest_dev, cap


# ------------------------------------------------------------------------------------------------- CPU side

_ref = None


def ref():
    global _ref
    if _ref is None:
        from oracle import ref_shim

        _ref = ref_shim.load()
    return _ref


def cpu_host():
    import ssl

    model, sha_ni = "unknown", False
    try:
        for line in open("/proc/cpuinfo"):
            if line.startswith("model name") and model == "unknown":
                model = line.split(":", 1)[1].strip()
            elif line.startswith("flags"):
                sha_ni = " sha_ni" in line
                break
    except OSError:
        pass
    return {"logical_cpus": os.cpu_count(), "cpu_model": model, "sha_ni": sha_ni, "openssl": ssl.OPENSSL_VERSION}


def cpu_pool(fn, items, workers):
    from concurrent.futures import ThreadPoolExecutor

    t0 = time.perf_counter()
    with ThreadPoolExecutor(max_workers=workers) as ex:
        out = list(ex.map(fn, items))
    return time.perf_counter() - t0, out


def cpu_fused_rows(name, blobs, check=None, serial_cap=1 << 30, **extra):
    """get_upload_hashes(bytes) per message: one thread (bounded), ThreadPoolExecutor default size, workers = ncpu."""
    h = ref()[0]
    ncpu = os.cpu_count() or 1
    nbytes = sum(len(b) for b in blobs)
    acc, k = 0, 0
    for b in blobs:
        if acc >= serial_cap and k:
            break
        acc += len(b)
        k += 1
    t0 = time.perf_counter()
    for b in blobs[:k]:
        h.get_upload_hashes(b)
    serial = acc / GiB / (time.perf_counter() - t0)
    d_def, out = cpu_pool(h.get_upload_hashes, blobs, min(32, ncpu + 4))
    d_all, _ = cpu_pool(h.get_upload_hashes, blobs, ncpu)
    ok = None
    if check is not None:
        ok = all(bytes.fromhex(o.sha256_hex()) == check[0][i].tobytes() and bytes.fromhex(o.md5_hex()) == check[1][i].tobytes()
                 for i, o in enumerate(out))
    emit({"config": name, "side": "cpu", "what": "reference get_upload_hashes(bytes) per message (SHA-256+MD5)",
          "sample_bytes": nbytes, "messages": len(blobs), "single_thread_GiBps": round(serial, 3),
          "single_thread_sample_bytes": acc, f"pool_default_{min(32, ncpu + 4)}_GiBps": round(nbytes / GiB / d_def, 3),
          f"pool_ncpu_{ncpu}_GiBps": round(nbytes / GiB / d_all, 3), "digests_equal_gpu": ok, "host": cpu_host(), **extra})


def cpu_v2_rows(name, blobs, check=None, **extra):
    """volumefs2: the reference's FileUploadSpec2.from_fileobj -> _gather_blocks -> _gather_block (two reads + SHA-256
    per block) via asyncio.to_thread under Semaphore(cpu_count), all files gathered concurrently (volume.py:1358,1381)."""
    from pathlib import PurePosixPath

    b = ref()[1]

    async def run():
        sem = asyncio.Semaphore(os.cpu_count() or 1)
        t0 = time.perf_counter()
        specs = await asyncio.gather(*[b.FileUploadSpec2.from_fileobj(io.BytesIO(x), PurePosixPath(f"f{i}"), sem, 0o644)
                                       for i, x in enumerate(blobs)])
        return time.perf_counter() - t0, specs

    dt, specs = asyncio.run(run())
    nbytes = sum(len(x) for x in blobs)
    ok = None
    if check is not None:
        flat = [blk for s in specs for blk in s.blocks]
        ok = len(flat) == len(check[0]) and all(blk.contents_sha256 == check[0][i].tobytes() and blk.end - blk.start == int(check[1][i])
                                               for i, blk in enumerate(flat))
    emit({"config": name, "side": "cpu", "what": "reference FileUploadSpec2.from_fileobj (_gather_block: trim scan + SHA-256, "
          f"Semaphore({os.cpu_count()}), asyncio.to_thread default executor)", "sample_bytes": nbytes, "files": len(blobs),
          "GiBps": round(nbytes / GiB / dt, 3), "digests_equal_gpu": ok, "host": cpu_host(), **extra})


def host_blobs(data, offs, lens, cap_bytes):
    """Python bytes objects of the first messages (<= cap_bytes) of this rank, copied out of HBM."""
    csum = np.cumsum(lens.astype(np.float64))
    k = max(1, int(np.searchsorted(csum, cap_bytes, side="right")))
    k = min(k, len(lens))
    lo, hi = int(offs[:k].min()), int((offs[:k] + lens[:k]).max())
    host = data[lo:hi].cpu().numpy()
    return [host[int(o) - lo : int(o) - lo + int(l)].tobytes() for o, l in zip(offs[:k], lens[:k])], k


# ------------------------------------------------------------------------------------------------------ C3

if "c3" in which:
    total_gib = float(os.environ.get("J1_C3_GIB", 100))
    nfiles = int(os.environ.get("J1_C3_FILES", 1 << 20))
    rng = np.random.default_rng(0)
    sizes = np.clip(rng.lognormal(np.log(102400) - 1.5**2 / 2, 1.5, nfiles), 1, 1 << 30)
    sizes = np.maximum(1, (sizes * (total_gib * 2**30 / sizes.sum())).astype(np.int64))
    mine = sharding.shard_assignment(sizes, world)[rank]
    my_sizes = sizes[mine].astype(np.uint64)
    offs = np.concatenate([[0], np.cumsum((my_sizes + np.uint64(15)) & ~np.uint64(15))]).astype(np.uint64)
    nbytes = int(offs[-1])
    offs = offs[:-1]
    data = torch.empty(nbytes + 64, dtype=torch.uint8, device=dev)
    ctx.fill_synth_device(data.data_ptr(), (nbytes + 64) & ~7, 0xC3 + rank)
    info = {"files_total": nfiles, "tree_GiB": total_gib, "largest_file": int(sizes.max()), "scaling": "strong",
            "shard_bytes_rank0": int(my_sizes.sum())}
    dig, cap = gpu_row("C3-v1 whole-file SHA-256+MD5 (100 GiB / 1 Mi files, log-normal)", data, offs, my_sizes, BOTH, **info)
    if WITH_CPU and rank == 0:
        blobs, k = host_blobs(data, offs, my_sizes, CPU_PREFIX)
        cpu_fused_rows("C3-v1 whole-file SHA-256+MD5 (100 GiB / 1 Mi files, log-normal)", blobs,
                       check=(dig[: 32 * cap].reshape(cap, 32), dig[32 * cap : 48 * cap].reshape(cap, 16)),
                       sample=f"first {k} files of rank 0's shard")
    B = 8 << 20
    nblk = ((my_sizes + np.uint64(B - 1)) // np.uint64(B)).astype(np.int64)
    first = np.cumsum(nblk) - nblk
    within = np.arange(int(nblk.sum())) - np.repeat(first, nblk)
    boff = (np.repeat(offs, nblk) + (within * B).astype(np.uint64)).astype(np.uint64)
    blen = np.minimum(np.uint64(B), np.repeat(my_sizes, nblk) - (within * B).astype(np.uint64)).astype(np.uint64)
    dig, cap = gpu_row("C3-v2 zero-trimmed <= 8 MiB blocks SHA-256 (same tree)", data, boff, blen, _lib.SHA256 | _lib.TRIM_ZEROS,
                       blocks_rank0=int(nblk.sum()), **info)
    if WITH_CPU and rank == 0:
        blobs, k = host_blobs(data, offs, my_sizes, CPU_PREFIX)
        nb = int(nblk[:k].sum())
        cpu_v2_rows("C3-v2 zero-trimmed <= 8 MiB blocks SHA-256 (same tree)", blobs,
                    check=(dig[: 32 * cap].reshape(cap, 32)[:nb], dig[48 * cap :].view("<u8")[:nb]),
                    sample=f"first {k} files of rank 0's shard")
        del blobs
    del data
    torch.cuda.empty_cache()

# ------------------------------------------------------------------------------------------------------ C5

if "c5" in which:
    CAP = int(os.environ.get("J1_C5_BYTES", 8 << 30))
    data = torch.empty(CAP + 64, dtype=torch.uint8, device=dev)
    ctx.fill_synth_device(data.data_ptr(), CAP + 64, 0xC5 + rank)
    for k in range(0, int(os.environ.get("J1_C5_KMAX", 10)) + 1):
        size = 4096 * 4**k
        n = max(1, CAP // size)
        offs, lens = np.arange(n, dtype=np.uint64) * np.uint64(size), np.full(n, size, np.uint64)
        name = f"C5 size={size} ({n} messages = {n * size / GiB:.0f} GiB per GPU)"
        long_chains = size >= (1 << 28)  # chain-bound points take 4..60 s per pass: one pass, e2e on the 1-GPU run only
        dig, cap = gpu_row(name, data, offs, lens, BOTH, reps=1 if size >= (1 << 24) else 2, warm=not long_chains,
                           e2e=(not long_chains) or (world == 1 and size < (1 << 30)), size=size, scaling="weak")
        if WITH_CPU and rank == 0:
            cpu_cap = min(CAP, CPU_PREFIX if size < (1 << 28) else CAP, 200_000 * size)
            blobs, kk = host_blobs(data, offs, lens, cpu_cap)
            cpu_fused_rows(name, blobs, check=(dig[: 32 * cap].reshape(cap, 32), dig[32 * cap : 48 * cap].reshape(cap, 16)),
                           serial_cap=1 << 30, size=size, sample=f"first {kk} messages")
            del blobs
    del data
    torch.cuda.empty_cache()

# ------------------------------------------------------------------------------------------------------ C4

if "c4" in which and world == 1:
    G = int(float(os.environ.get("J1_C4_GIB", 10)) * GiB)
    data = torch.empty(G + 64, dtype=torch.uint8, device=dev)
    ctx.fill_synth_device(data.data_ptr(), G + 64, 0xC4)
    # make it look like a tar of a build context: some blank and half-blank 8 MiB regions
    B = 8 << 20
    nb = G // B
    for i in range(0, nb, 16):
        data[i * B : (i + 1) * B].zero_()
    for i in range(5, nb, 16):
        data[i * B + (3 << 20) : (i + 1) * B].zero_()
    torch.cuda.synchronize()
    offs, lens = np.arange(nb, dtype=np.uint64) * np.uint64(B), np.full(nb, B, np.uint64)
    dig2, cap2 = gpu_row(f"C4(ii) {nb} x 8 MiB blocks: zero-trim scan + SHA-256 ({G / GiB:.0f} GiB stream)", data, offs, lens,
                         _lib.SHA256 | _lib.TRIM_ZEROS)
    P = 64 << 20
    npart = G // P
    poffs, plens = np.arange(npart, dtype=np.uint64) * np.uint64(P), np.full(npart, P, np.uint64)
    dig3, cap3 = gpu_row(f"C4(iii) {npart} x 64 MiB multipart parts MD5 ({G / GiB:.0f} GiB stream)", data, poffs, plens, _lib.MD5)
    dig1, cap1 = gpu_row(f"C4(i) ONE {G / GiB:.0f} GiB message SHA-256+MD5 (a single serial chain)", data, np.array([0], np.uint64),
                         np.array([G], np.uint64), BOTH, reps=1, warm=False, e2e=False)
    if WITH_CPU:
        h, b, _ = ref()
        host = data[:G].cpu().numpy()
        whole = host.tobytes()
        del host
        cpu_v2_rows(f"C4(ii) {nb} x 8 MiB blocks: zero-trim scan + SHA-256 ({G / GiB:.0f} GiB stream)", [whole],
                    check=(dig2[: 32 * cap2].reshape(cap2, 32), dig2[48 * cap2 :].view("<u8")), sample="the whole stream")
        import hashlib

        parts = [memoryview(whole)[i * P : (i + 1) * P] for i in range(npart)]
        ncpu = os.cpu_count() or 1
        d_def, out = cpu_pool(lambda p: hashlib.md5(p).digest(), parts, min(32, ncpu + 4))
        ok = all(o == dig3[32 * cap3 : 48 * cap3].reshape(cap3, 16)[i].tobytes() for i, o in enumerate(out))
        emit({"config": f"C4(iii) {npart} x 64 MiB multipart parts MD5 ({G / GiB:.0f} GiB stream)", "side": "cpu",
              "what": f"hashlib.md5 per part in ThreadPoolExecutor({min(32, ncpu + 4)}) (the per-part MD5 that "
                      "BytesIOSegmentPayload folds on executor threads while parts upload concurrently)",
              "sample_bytes": G, "GiBps": round(G / GiB / d_def, 3), "digests_equal_gpu": ok, "host": cpu_host()})
        sample = min(G, 2 << 30)
        t0 = time.perf_counter()
        one = h.get_upload_hashes(io.BytesIO(whole[:sample]))
        dt = time.perf_counter() - t0
        t0 = time.perf_counter()
        full = h.get_upload_hashes(io.BytesIO(whole))
        dt_full = time.perf_counter() - t0
        ok = bytes.fromhex(full.sha256_hex()) == dig1[:32].tobytes() and bytes.fromhex(full.md5_hex()) == dig1[32 * cap1 : 32 * cap1 + 16].tobytes()
        emit({"config": f"C4(i) ONE {G / GiB:.0f} GiB message SHA-256+MD5 (a single serial chain)", "side": "cpu",
              "what": "reference get_upload_hashes(BinaryIO), one thread, 64 KiB reads", "sample_bytes": G,
              "GiBps": round(G / GiB / dt_full, 3), "first_2GiB_GiBps": round(sample / GiB / dt, 3), "digests_equal_gpu": ok,
              "host": cpu_host()})

ctx.close()
if world > 1:
    dist.destroy_process_group()
