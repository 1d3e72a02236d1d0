"""tools/device_put_bench.py -- the second half of uploading a checkpoint that lives in GPU memory: getting the bytes
of the blocks the server reports missing off the device, and the whole volumefs2 upload around it.

The seeded bf16 state dict of the block benches (safetensors_blocks_bench.state_dict: about 4 GiB in about 300
tensors; DPB_GIB sets the size) as DeviceFile.safetensors and as DeviceFile.torch_save, every block missing.  Arms,
alternating, DPB_REPS (5) runs each, median and range:

  y   yardstick: ONE cudaMemcpyAsync of as many bytes as the trimmed blocks hold, from one aligned device buffer into
      the same page-locked buffer (the most the copy engine gives); CUDA events
  s   stage_ranges of all trimmed blocks (one b200h_copy_ranges_to_host call, stage_ranges_kernel storing straight
      into the page-locked buffer): CUDA events around the call on the file's stream, so the host's table building is
      inside; GB/s and share of y
  r   the read side of the unstaged upload alone: every block through reopen() + 256 KiB reads from 128 threads, as
      the PUT path issues them; host clock
  u0  the whole VolumeUploadContextManager2 upload against an in-process fake servicer and aiohttp block server
      (VolumePutFiles2 answers the missing blocks, PUT /block/{token} stores by SHA-256), unstaged; host clock from
      __aexit__ entry to its return.  The server hashes every body on the same event loop, in both arms.
  u1  the same with device_staging_bytes = twice the file (one wave); also the time from __aexit__ entry to
      device_released

After s the staged bytes are hashed on the host and compared with the block table; after u0 / u1 the server's blocks
are.  The card name and power limit are read in the same run.  Needs a GPU: nothing here falls back.
One JSON line per file kind and arm; also written to $DPB_OUT/device_put_bench.json when set."""
import asyncio
import hashlib
import json
import os
import sys
import time
import types
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch
from aiohttp import web

from modal_client_b200 import DeviceFile, _backend, _lib, blob_utils, stage_ranges, volume
from safetensors_blocks_bench import gpu_info, state_dict

GIB = float(os.environ.get("DPB_GIB", 4))
REPS = int(os.environ.get("DPB_REPS", 5))
ARMS = os.environ.get("DPB_ARMS", "y,s,r,u0,u1").split(",")
BS = blob_utils.BLOCK_SIZE
CHUNK, THREADS = 256 << 10, 128


class Servicer:
    """VolumePutFiles2 as the volume server answers it: blocks without a valid put_response are missing."""

    def __init__(self):
        self.blocks, self.host, self.files = {}, None, {}

    async def VolumePutFiles2(self, req):
        missing = []
        for fi, f in enumerate(req.files):
            for bi, b in enumerate(f.blocks):
                bid = b.contents_sha256.hex()
                if not (b.put_response == b"put:" + bid.encode() and bid in self.blocks):
                    missing.append(types.SimpleNamespace(file_index=fi, block_index=bi, put_url=f"{self.host}/block/{bid}"))
        if not missing:
            self.files.update({f.path: [b.contents_sha256 for b in f.blocks] for f in req.files})
        return types.SimpleNamespace(missing_blocks=missing)


async def upload(make_file, budget):
    """One upload against a fresh server -> (seconds in __aexit__, seconds to device_released, digests that arrived)."""
    srv = Servicer()

    async def put_block(request):
        body = await request.read()
        bid = hashlib.sha256(body).hexdigest()
        srv.blocks[bid] = len(body)
        return web.Response(text=f"put:{bid}")

    app = web.Application(client_max_size=BS + 1024)
    app.add_routes([web.put("/block/{token}", put_block)])
    runner = web.AppRunner(app)
    await runner.setup()
    site = web.TCPSite(runner, "127.0.0.1", 0)
    await site.start()
    srv.host = f"http://127.0.0.1:{site._server.sockets[0].getsockname()[1]}"
    try:
        f = make_file()
        torch.cuda.synchronize()
        batch = volume.VolumeUploadContextManager2("vo-bench", types.SimpleNamespace(stub=srv), device_staging_bytes=budget)
        await batch.__aenter__()
        batch.put_file(f, "/ckpt/model")
        released = []

        async def watch(t0):
            await batch.device_released.wait()
            released.append(time.perf_counter() - t0)

        t0 = time.perf_counter()
        watcher = asyncio.ensure_future(watch(t0))
        await batch.__aexit__(None, None, None)
        wall = time.perf_counter() - t0
        await watcher
        return wall, released[0], dict(srv.blocks)
    finally:
        await runner.cleanup()
        await blob_utils.ClientSessionRegistry.close_session()


def main():
    if not torch.cuda.is_available():
        raise SystemExit("device_put_bench needs a GPU")
    ctx = _lib.Context(0)
    _backend.set_context(ctx)
    sd = state_dict(ctx, int(GIB * (1 << 30)))
    kinds = {"safetensors": lambda: DeviceFile.safetensors(sd), "torch_save": lambda: DeviceFile.torch_save(sd)}
    info = gpu_info()
    lines = []
    pool = ThreadPoolExecutor(THREADS)
    for kind, make in kinds.items():
        f = make()
        sha, _, trimmed = f.hash_parts(BS, _lib.SHA256 | _lib.TRIM_ZEROS)
        ranges = [(0, i * BS, int(t)) for i, t in enumerate(trimmed)]
        offsets, at = [], 0
        for _, _, n in ranges:
            offsets.append(at)
            at += -(-n // 128) * 128
        nbytes = int(trimmed.sum())
        table = {sha[i].tobytes().hex(): int(trimmed[i]) for i in range(len(ranges))}
        dst = ctx.host_alloc(max(at, 1))
        host_t = torch.from_numpy(dst)
        assert host_t.is_pinned()
        aligned = torch.empty(nbytes, dtype=torch.uint8, device="cuda:0")
        ctx.fill_synth_device(aligned.data_ptr(), nbytes // 8 * 8, seed=5)
        stream = f._src.stream

        def timed(enqueue):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record(stream)
            enqueue()
            e1.record(stream)
            e1.synchronize()
            return e0.elapsed_time(e1) / 1e3

        def arm_y():
            def go():
                with torch.cuda.stream(stream):
                    host_t[:nbytes].copy_(aligned, non_blocking=True)
            return {"s": timed(go)}

        def arm_s():
            return {"s": timed(lambda: stage_ranges([f], ranges, dst, offsets))}

        def read_block(r):
            _, off, n = r
            with f.reopen() as rd:
                rd.seek(off)
                got = 0
                while got < n:
                    got += len(rd.read(min(CHUNK, n - got)))

        def arm_r():
            t0 = time.perf_counter()
            list(pool.map(read_block, ranges))
            return {"s": time.perf_counter() - t0}

        def arm_u(budget):
            wall, rel, blocks = asyncio.run(upload(make, budget))
            assert blocks == table, "the server's blocks differ from the block table"
            return {"s": wall, "released_s": rel}

        arms = {"y": arm_y, "s": arm_s, "r": arm_r, "u0": lambda: arm_u(None),
                "u1": lambda: arm_u(2 * (at + BS))}
        arms = {k: v for k, v in arms.items() if k in ARMS}
        for k, fn in arms.items():  # warm-up of every arm
            fn()
            print(f"# {kind}: arm {k} warmed up", file=sys.stderr, flush=True)
        if "s" in arms:  # what arm s staged, against the block table
            dst[:] = 0
            stage_ranges([f], ranges, dst, offsets).wait()
            for i, (o, (_, _, n)) in enumerate(zip(offsets, ranges)):
                assert hashlib.sha256(dst[o : o + n]).digest() == sha[i].tobytes(), f"block {i} of {kind} differs"
        runs = {k: [] for k in arms}
        for _ in range(REPS):
            for k, fn in arms.items():
                runs[k].append(fn())
                print(f"# {kind}: arm {k} {runs[k][-1]}", file=sys.stderr, flush=True)
        med = lambda xs: sorted(xs)[len(xs) // 2]  # noqa: E731
        y = med([r["s"] for r in runs["y"]]) if "y" in runs else None
        for k, rs in runs.items():
            t = sorted(r["s"] for r in rs)
            rec = {"tool": "device_put_bench", "file": kind, "arm": k, "bytes": nbytes, "file_bytes": f.nbytes,
                   "blocks": len(ranges), "segments": len(f._src.segments), "reps": REPS, "s_median": med(t),
                   "s_min": t[0], "s_max": t[-1], "gb_per_s_median": nbytes / med(t) / 1e9, **info}
            if k == "s" and y:
                rec["share_of_y"] = y / med(t)
            if k == "u1":
                rel = sorted(r["released_s"] for r in rs)
                rec.update({"released_s_median": med(rel), "released_s_min": rel[0], "released_s_max": rel[-1]})
            lines.append(json.dumps(rec))
            print(lines[-1], flush=True)
        del aligned, host_t
        ctx.host_free(dst)
    out = os.environ.get("DPB_OUT")
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "device_put_bench.json"), "w") as fh:
            fh.write("\n".join(lines) + "\n")
    pool.shutdown()
    ctx.close()


if __name__ == "__main__":
    main()
