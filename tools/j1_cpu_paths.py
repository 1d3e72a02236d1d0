"""tools/j1_cpu_paths.py -- the reference's CPU path for the configurations whose source is a FILE, driven the way the
reference drives it (from_path on real files; tools/j1_matrix.py's BytesIO stand-in makes the reference copy the whole
buffer for every block: `BytesIO(buffer)` in FileUploadSpec2.from_fileobj, py/modal/_utils/blob_utils.py:580-584):
  C4   one 10 GiB stream in /dev/shm: (ii) FileUploadSpec2.from_path (trim scan + SHA-256 per 8 MiB block, Semaphore(ncpu)),
       (iii) hashlib.md5 per 64 MiB part on a thread pool, (i) get_upload_hashes(open(path)) on one thread
  C3-v2  the first ~8 GiB of the 100 GiB / 1 Mi-file tree as files in /dev/shm, FileUploadSpec2.from_path for all of them
The bytes are the ones tools/j1_matrix.py hashes on the GPU (same generator, same seeds); the block / part digests are
compared with a GPU pass over the same files (b200h_hash_files).  Appends rows to j1_out/r2_j1_cpu_paths.jsonl."""
import asyncio
import hashlib
import json
import os
import shutil
import sys
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path, PurePosixPath

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from modal_client_b200 import _lib
from oracle import ref_shim

GiB = float(1 << 30)
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "j1_out", "r2_j1_cpu_paths.jsonl")
ref_hash, ref_blob, _ = ref_shim.load()
ctx = _lib.Context(0)
dev = torch.device("cuda:0")
ncpu = os.cpu_count() or 1
root = "/dev/shm/b200h_j1_cpu"
shutil.rmtree(root, ignore_errors=True)
os.makedirs(root)


def emit(row):
    import ssl

    row["host"] = {"logical_cpus": ncpu, "openssl": ssl.OPENSSL_VERSION}
    line = json.dumps(row)
    print(line, flush=True)
    with open(OUT, "a") as f:
        f.write(line + "\n")


async def v2_specs(paths):
    sem = asyncio.Semaphore(ncpu)
    t0 = time.perf_counter()
    specs = await asyncio.gather(*[ref_blob.FileUploadSpec2.from_path(Path(p), PurePosixPath(os.path.basename(p)), sem) for p in paths])
    return time.perf_counter() - t0, specs


which = sys.argv[1:] or ["c4", "c3"]
if "c4" in which:
    G = int(float(os.environ.get("J1_C4_GIB", 10)) * GiB)
    B, P = 8 << 20, 64 << 20
    data = torch.empty(G + 64, dtype=torch.uint8, device=dev)
    ctx.fill_synth_device(data.data_ptr(), G + 64, 0xC4)
    nb = G // B
    for i in range(0, nb, 16):
        data[i * B : (i + 1) * B].zero_()
    for i in range(5, nb, 16):
        data[i * B + (3 << 20) : (i + 1) * B].zero_()
    path = os.path.join(root, "stream.bin")
    data[:G].cpu().numpy().tofile(path)
    del data
    torch.cuda.empty_cache()
    sizes, _ = ctx.stat_files([path])
    g_sha, _, g_trim = ctx.hash_files([path], sizes, B, _lib.SHA256 | _lib.TRIM_ZEROS)
    _, g_md5, _ = ctx.hash_files([path], sizes, P, _lib.MD5)
    dt, specs = asyncio.run(v2_specs([path]))
    blocks = specs[0].blocks
    ok = len(blocks) == len(g_sha) and all(b.contents_sha256 == g_sha[i].tobytes() and b.end - b.start == int(g_trim[i]) for i, b in enumerate(blocks))
    emit({"config": f"C4(ii) {nb} x 8 MiB blocks: zero-trim scan + SHA-256 ({G / GiB:.0f} GiB stream)", "side": "cpu",
          "what": f"reference FileUploadSpec2.from_path on the stream as a file in /dev/shm (_gather_block: trim scan + SHA-256, Semaphore({ncpu}), asyncio.to_thread default executor)",
          "sample_bytes": G, "GiBps": round(G / GiB / dt, 3), "digests_equal_gpu": bool(ok)})
    fd = os.open(path, os.O_RDONLY)
    nparts = G // P

    def part_md5(i):
        return hashlib.md5(os.pread(fd, P, i * P)).digest()

    for workers in (min(32, ncpu + 4), ncpu):
        t0 = time.perf_counter()
        with ThreadPoolExecutor(max_workers=workers) as ex:
            out = list(ex.map(part_md5, range(nparts)))
        dt = time.perf_counter() - t0
        ok = all(o == g_md5[i].tobytes() for i, o in enumerate(out))
        emit({"config": f"C4(iii) {nparts} x 64 MiB multipart parts MD5 ({G / GiB:.0f} GiB stream)", "side": "cpu",
              "what": f"hashlib.md5 per part (pread from /dev/shm) in ThreadPoolExecutor({workers}): the per-part MD5 that BytesIOSegmentPayload folds on executor threads while parts upload concurrently",
              "sample_bytes": G, "GiBps": round(G / GiB / dt, 3), "digests_equal_gpu": bool(ok)})
    os.close(fd)
    t0 = time.perf_counter()
    with open(path, "rb") as fp:
        full = ref_hash.get_upload_hashes(fp)
    dt = time.perf_counter() - t0
    emit({"config": f"C4(i) ONE {G / GiB:.0f} GiB message SHA-256+MD5 (a single serial chain)", "side": "cpu",
          "what": "reference get_upload_hashes(BinaryIO) on the stream as a file in /dev/shm, one thread, 64 KiB reads",
          "sample_bytes": G, "GiBps": round(G / GiB / dt, 3), "digests_equal_gpu": None, "sha256_hex": full.sha256_hex(),
          "note": "the GPU digest of this 151 s chain is not recomputed here; >= 4 GiB single messages are pinned by tests/test_gpu_round2.py"})
    os.remove(path)

if "c3" in which:
    from modal_client_b200 import sharding  # noqa: F401  (same tree as tools/j1_matrix.py)

    nfiles, total_gib = int(os.environ.get("J1_C3_FILES", 1 << 20)), float(os.environ.get("J1_C3_GIB", 100))
    rng = np.random.default_rng(0)
    sizes = np.clip(rng.lognormal(np.log(102400) - 1.5**2 / 2, 1.5, nfiles), 1, 1 << 30)
    sizes = np.maximum(1, (sizes * (total_gib * 2**30 / sizes.sum())).astype(np.int64)).astype(np.uint64)
    prefix = int(float(os.environ.get("J1_CPU_PREFIX", 8)) * GiB)
    k = int(np.searchsorted(np.cumsum(sizes.astype(np.float64)), prefix, side="right"))
    my = sizes[:k]
    offs = np.concatenate([[0], np.cumsum((my + np.uint64(15)) & ~np.uint64(15))]).astype(np.uint64)
    nbytes = int(offs[-1])
    data = torch.empty(nbytes + 64, dtype=torch.uint8, device=dev)
    ctx.fill_synth_device(data.data_ptr(), (nbytes + 64) & ~7, 0xC3)
    host = data.cpu().numpy()
    del data
    d = os.path.join(root, "tree")
    os.makedirs(d)
    paths = []
    for i in range(k):
        p = os.path.join(d, f"f{i:06d}")
        host[int(offs[i]) : int(offs[i]) + int(my[i])].tofile(p)
        paths.append(p)
    del host
    st_sizes, _ = ctx.stat_files(paths)
    g_sha, _, g_trim = ctx.hash_files(paths, st_sizes, 8 << 20, _lib.SHA256 | _lib.TRIM_ZEROS)
    dt, specs = asyncio.run(v2_specs(paths))
    flat = [b for s in specs for b in s.blocks]
    ok = len(flat) == len(g_sha) and all(b.contents_sha256 == g_sha[i].tobytes() and b.end - b.start == int(g_trim[i]) for i, b in enumerate(flat))
    nb = float(my.astype(np.float64).sum())
    emit({"config": "C3-v2 zero-trimmed <= 8 MiB blocks SHA-256 (same tree)", "side": "cpu",
          "what": f"reference FileUploadSpec2.from_path over real files in /dev/shm (_gather_block: trim scan + SHA-256, Semaphore({ncpu}), asyncio.to_thread default executor)",
          "sample": f"first {k} files of the tree", "sample_bytes": int(nb), "files": k, "GiBps": round(nb / GiB / dt, 3), "digests_equal_gpu": bool(ok)})
shutil.rmtree(root, ignore_errors=True)
ctx.close()
