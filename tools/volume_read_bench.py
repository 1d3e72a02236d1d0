"""tools/volume_read_bench.py -- reading a checkpoint from a volume back into GPU memory.

(a) kernel: a seeded safetensors-shaped state dict (VRB_GIB, default 2 GiB: four large bf16 matrices plus hundreds of
    small norms and biases) as DeviceFile.safetensors; every 8 MiB block of the file, from one page-locked buffer
    (block k at offset k * BLOCK_SIZE, as read_file_into_device lays a wave out), written with ONE
    b200h_copy_ranges_from_host call, against ONE cudaMemcpyAsync of as many bytes from one aligned page-locked buffer
    into one device buffer.  CUDA events, VRB_REPS (5) runs each, alternating, best and median; GB/s and the share of
    the copy engine's figure.  The tensors are checked against the source afterwards.
(b) end to end over LOOPBACK (an in-process aiohttp block server on 127.0.0.1: it measures the client, not a network):
    a VRB_E2E_GIB (1 GiB) safetensors file uploaded once, then read_safetensors against the reference's route
    (read_file_into_fileobj into BytesIO, safetensors.torch.load, .to("cuda") per tensor), alternating, VRB_E2E_REPS
    (2) runs each; host clock from call to a synchronised result, and the peak growth of the process's resident set
    during the call (sampled every 2 ms).  The results are compared tensor by tensor.
(c) the same for a torch.save training checkpoint of VRB_E2E_GIB, uploaded once with DeviceFile.torch_save: a state
    dict shaped as in (b) plus an Adam state dict (``exp_avg`` / ``exp_avg_sq`` of the small tensors, CPU ``step``
    tensors), read with read_torch_save against read_file_into_fileobj into BytesIO + torch.load(map_location="cuda"),
    alternating, timed and compared bitwise as in (b).  Then the CRC launch alone (one crc32_device call over the loaded
    storages, CUDA events, best of VRB_REPS) against the load_ranges time of arm (a), when it ran.

(d) slices for tensor parallelism, rank VRB_RANK (3) of 8 of a Llama-shaped bf16 layer stack (hidden 2048, kv 512,
    intermediate 5632): q, k, v, gate and up sliced on dim 0, o and down on dim 1, the norms whole.
    kernel: one 128 MiB wave laid out as _load_in_waves lays it out (16 blocks of the file in consecutive 8 MiB slots,
    the data region starting at 8 mod 16 as safetensors headers leave it), its boxes planned as read_safetensors_slices
    plans them, written into one packed device buffer by (1) ONE load_boxes call, (2) one cudaMemcpy2DAsync per box
    from the same page-locked buffer (ctypes on libcudart), (3) load_ranges of the whole wave into scratch HBM and
    .contiguous() slices of every tensor, against (4) one cudaMemcpyAsync of the selected byte count.  CUDA events,
    VRB_REPS runs each, alternating, best and median, and the host's time inside each call; the three results are
    compared bitwise.  The same for a selection that enumerates its outer dimension (rows 4..11, columns 2048..3071 of
    every expert of a [511, 16, 8192] stack: 511 boxes in the wave).  Then arm (a)'s workload
    as 1-row boxes (load_boxes) next to load_ranges.
    end to end over loopback: a VRB_E2E_GIB (1 GiB) stack uploaded once; for every rank 0..7, read_safetensors_slices
    against read_safetensors followed by .contiguous() slices, alternating: host clock, the bytes GET from the server,
    the peak HBM growth (torch.cuda.max_memory_allocated) and resident-set growth, and a bitwise comparison.

(e) loading converted to another dtype (F32 <-> BF16).
    kernel: a VRB_GIB (2 GiB) image of F32 (then of BF16) in one page-locked buffer, as 1-row boxes of one 8 MiB block
    each, the data region starting at 0 and at 8 mod 16 (a safetensors data region starts at either): (1) ONE
    load_cast_boxes call (F32 -> BF16, BF16 -> F32), (2) ONE load_boxes call of the same source bytes, unconverted, and
    (3) the unfused route: that load_boxes call into scratch HBM followed by torch's .to() into the result.  CUDA
    events, VRB_REPS runs each, alternating, best and median; GB/s of source bytes and the share of load_boxes' rate.
    The converted results are compared bitwise with torch's cast.
    end to end over loopback: a VRB_E2E_GIB (1 GiB) F32 Llama-shaped file uploaded once; read_safetensors(dtype=
    torch.bfloat16) against read_safetensors followed by .to(torch.bfloat16), alternating, VRB_E2E_REPS (2) runs each:
    host clock, peak HBM growth (torch.cuda.max_memory_allocated) and a bitwise comparison.  The same for rank
    VRB_RANK's TP slices: read_safetensors_slices(dtype=torch.bfloat16) against the slices followed by .to().

(f) loading FP8 weights dequantized with 128 x 128 block scales (F8_E4M3 with F32 ``_scale_inv``, to BF16).
    kernel: one 128 MiB wave (16 blocks of 8 MiB, the data region at 8 mod 16) of a [R, 7168] E4M3 weight as 1-row
    boxes of one block each: (1) ONE load_scaled_boxes call against (2) ONE load_boxes call of the same FP8 bytes.
    CUDA events, VRB_REPS runs each, alternating, best and median; the cost of dequantizing over a plain copy.  The
    result is compared bitwise with torch's CUDA dequantization.
    end to end over loopback: a seeded, Qwen3/DeepSeek-shaped FP8 stack of VRB_FP8_GIB (2.5) GB exported with
    safetensors_shards in 1 GB shards and uploaded once; read_safetensors_sharded(dtype=torch.bfloat16,
    scales=fp8_scales(...)) against read_safetensors_sharded followed by per-weight torch dequantization (what
    DeepSeek's fp8_cast_bf16.py does), alternating, VRB_FP8_REPS (3) runs each: host clock, peak HBM growth
    (torch.cuda.max_memory_allocated) and a bitwise comparison.

VRB_ARMS (default "abcd") picks the arms; "e" and "f" are run only when named.

The card name and power limit are read in the same run.  Needs a GPU: nothing here falls back.
One JSON line per arm; also written to $VRB_OUT/volume_read_bench.json when set."""
import asyncio
import json
import os
import statistics
import sys
import threading
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from modal_client_b200 import DeviceFile, _backend, _lib, blob_utils, load_ranges, volume
from tests.volume_read_server import running_volume_server

GiB, MiB = 1 << 30, 1 << 20


def gpu_info() -> dict:
    import subprocess

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in q.split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def state_dict(total: int, seed: int = 0) -> dict:
    """Four large bf16 matrices holding most of ``total`` bytes, plus 400 small norms / biases of odd sizes."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    sd = {}
    for i in range(400):
        n = 1000 + 37 * i
        sd[f"layers.{i}.norm.weight"] = torch.randn(n, device="cuda", generator=g).to(torch.bfloat16)
        if i % 2:
            sd[f"layers.{i}.bias"] = torch.randn(n + 3, device="cuda", generator=g)
    left = total - sum(t.numel() * t.element_size() for t in sd.values())
    cols = 8192
    for i in range(4):
        rows = left // 4 // 2 // cols
        sd[f"mat.{i}.weight"] = torch.randn(rows, cols, device="cuda", generator=g).to(torch.bfloat16)
    return sd


def events_ms(fn) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def kernel_arm(ctx, info, out):
    BS = blob_utils.BLOCK_SIZE
    sd = state_dict(int(float(os.environ.get("VRB_GIB", "2")) * GiB))
    f = DeviceFile.safetensors(sd)
    n = f.nbytes
    ranges = [(0, o, min(BS, n - o)) for o in range(0, n, BS)]
    offsets = [o for _, o, _ in ranges]
    src = ctx.host_alloc(n)
    try:
        src[:] = torch.randint(0, 256, (n,), dtype=torch.uint8).numpy()
        yard_src = torch.from_numpy(src.copy()).pin_memory()
        yard_dst = torch.empty(n, dtype=torch.uint8, device="cuda")
        times = {"load_ranges": [], "memcpy": []}
        load = lambda: load_ranges([f], ranges, src, offsets, ctx=ctx)  # noqa: E731
        load().wait()
        yard_dst.copy_(yard_src, non_blocking=True)
        for _ in range(int(os.environ.get("VRB_REPS", "5"))):
            times["load_ranges"].append(events_ms(load))
            times["memcpy"].append(events_ms(lambda: yard_dst.copy_(yard_src, non_blocking=True)))
        torch.cuda.synchronize()
        image = b"".join(s.cpu().numpy().tobytes() for s in f._src.segments)
        ok = image == src.tobytes()
        best = {k: min(v) for k, v in times.items()}
        for arm, v in times.items():
            out.append({"arm": f"kernel.{arm}", "bytes": n, "ranges": len(ranges), "tensors": len(sd),
                        "best_ms": round(best[arm], 3), "median_ms": round(statistics.median(v), 3),
                        "range_ms": [round(min(v), 3), round(max(v), 3)], "GB_s": round(n / best[arm] / 1e6, 2),
                        "share_of_memcpy": round(best["memcpy"] / best[arm], 3), "bytes_equal": ok, **info})
            print(json.dumps(out[-1]), flush=True)
    finally:
        torch.cuda.synchronize()
        ctx.host_free(src)


class PeakRss:
    """Peak growth of the resident set while the block runs (sampled)."""

    def __enter__(self):
        self.base = self.peak = self._rss()
        self.stop = threading.Event()
        self.t = threading.Thread(target=self._run, daemon=True)
        self.t.start()
        return self

    @staticmethod
    def _rss() -> int:
        with open("/proc/self/statm") as fh:
            return int(fh.read().split()[1]) * os.sysconf("SC_PAGE_SIZE")

    def _run(self):
        while not self.stop.wait(0.002):
            self.peak = max(self.peak, self._rss())

    def __exit__(self, *exc):
        self.stop.set()
        self.t.join()
        self.peak = max(self.peak, self._rss())
        self.growth = self.peak - self.base


async def e2e_arm(info, out):
    import io

    from safetensors.torch import load as st_load

    sd = state_dict(int(float(os.environ.get("VRB_E2E_GIB", "1")) * GiB), seed=1)
    async with running_volume_server(blob_utils.BLOCK_SIZE) as (stub, _):
        client = types.SimpleNamespace(stub=stub)
        batch = volume.VolumeUploadContextManager2("vo-b", client)
        async with batch:
            batch.put_file(DeviceFile.safetensors(sd), "/m.safetensors")
        size = len(stub.volume_files["/m.safetensors"][0])

        async def ours():
            got = await volume.read_safetensors(client, "vo-b", "/m.safetensors")
            torch.cuda.synchronize()
            return got

        async def reference_route():
            buf = io.BytesIO()
            await volume.read_file_into_fileobj(client, "vo-b", "/m.safetensors", buf)
            host = st_load(buf.getvalue())
            del buf
            got = {k: v.to("cuda") for k, v in host.items()}
            torch.cuda.synchronize()
            return got

        res = {"read_safetensors": [], "fileobj_load_to_cuda": []}
        for _ in range(int(os.environ.get("VRB_E2E_REPS", "2"))):
            for arm, fn in (("read_safetensors", ours), ("fileobj_load_to_cuda", reference_route)):
                with PeakRss() as rss:
                    t0 = time.perf_counter()
                    got = await fn()
                    dt = time.perf_counter() - t0
                equal = sorted(got) == sorted(sd) and all(torch.equal(got[k].view(torch.uint8), sd[k].view(torch.uint8)) for k in sd)
                del got
                res[arm].append((dt, rss.growth, equal))
        for arm, v in res.items():
            ts = [t for t, _, _ in v]
            out.append({"arm": f"e2e_loopback.{arm}", "bytes": size, "median_s": round(statistics.median(ts), 3),
                        "range_s": [round(min(ts), 3), round(max(ts), 3)],
                        "peak_rss_growth_GB": round(max(g for _, g, _ in v) / 1e9, 3),
                        "tensors_equal": all(e for _, _, e in v), **info})
            print(json.dumps(out[-1]), flush=True)


def training_checkpoint(total: int, seed: int = 2) -> dict:
    """``state_dict(total)`` as the model, and the Adam state of its small tensors after one step."""
    sd = state_dict(total, seed)
    small = [k for k in sd if not k.startswith("mat.")]
    params = [torch.nn.Parameter(sd[k].float()) for k in small]
    opt = torch.optim.Adam(params, lr=1e-3)
    for p in params:
        p.grad = torch.ones_like(p)
    opt.step()
    return {"model": sd, "optim": opt.state_dict(), "step": 1}


def _flat(obj, at=""):
    if isinstance(obj, torch.Tensor):
        yield at, obj
    elif isinstance(obj, dict):
        for k, v in obj.items():
            yield from _flat(v, f"{at}/{k}")
    elif isinstance(obj, (list, tuple)):
        for i, v in enumerate(obj):
            yield from _flat(v, f"{at}/{i}")


def _bitwise_equal(a, b) -> bool:
    fa, fb = list(_flat(a)), list(_flat(b))
    return [k for k, _ in fa] == [k for k, _ in fb] and all(
        x.device == y.device and x.dtype == y.dtype and x.shape == y.shape and x.stride() == y.stride() and
        torch.equal(x.reshape(-1).view(torch.uint8), y.reshape(-1).view(torch.uint8)) for (_, x), (_, y) in zip(fa, fb))


async def torch_save_arm(ctx, info, out):
    import io

    ckpt = training_checkpoint(int(float(os.environ.get("VRB_E2E_GIB", "1")) * GiB))
    async with running_volume_server(blob_utils.BLOCK_SIZE) as (stub, _):
        client = types.SimpleNamespace(stub=stub)
        batch = volume.VolumeUploadContextManager2("vo-b", client)
        async with batch:
            batch.put_file(DeviceFile.torch_save(ckpt), "/ckpt.pt")
        size = len(stub.volume_files["/ckpt.pt"][0])
        want = torch.load(io.BytesIO(stub.volume_files["/ckpt.pt"][0]), map_location="cuda")

        async def ours():
            got = await volume.read_torch_save(client, "vo-b", "/ckpt.pt")
            torch.cuda.synchronize()
            return got

        async def reference_route():
            buf = io.BytesIO()
            await volume.read_file_into_fileobj(client, "vo-b", "/ckpt.pt", buf)
            buf.seek(0)
            got = torch.load(buf, map_location="cuda")
            del buf
            torch.cuda.synchronize()
            return got

        res = {"read_torch_save": [], "fileobj_torch_load_cuda": []}
        for _ in range(int(os.environ.get("VRB_E2E_REPS", "2"))):
            for arm, fn in (("read_torch_save", ours), ("fileobj_torch_load_cuda", reference_route)):
                with PeakRss() as rss:
                    t0 = time.perf_counter()
                    got = await fn()
                    dt = time.perf_counter() - t0
                equal = _bitwise_equal(got, want)
                if arm == "read_torch_save":
                    kept = got
                del got
                res[arm].append((dt, rss.growth, equal))
        for arm, v in res.items():
            ts = [t for t, _, _ in v]
            out.append({"arm": f"torch_save_loopback.{arm}", "bytes": size, "median_s": round(statistics.median(ts), 3),
                        "range_s": [round(min(ts), 3), round(max(ts), 3)],
                        "peak_rss_growth_GB": round(max(g for _, g, _ in v) / 1e9, 3),
                        "bitwise_equal_to_torch_load": all(e for _, _, e in v), **info})
            print(json.dumps(out[-1]), flush=True)
    storages = {t.untyped_storage().data_ptr(): t.untyped_storage() for _, t in _flat(kept) if t.untyped_storage().nbytes()}
    ptrs, lens = list(storages), [st.nbytes() for st in storages.values()]
    crc = torch.empty(len(ptrs), dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream or 1
    launch = lambda: ctx.crc32_device(ptrs, lens, crc.data_ptr(), stream)  # noqa: E731
    launch()
    ms = [events_ms(launch) for _ in range(int(os.environ.get("VRB_REPS", "5")))]
    load = next((o for o in out if o["arm"] == "kernel.load_ranges"), None)
    row = {"arm": "torch_save.crc32_device", "storages": len(ptrs), "bytes": sum(lens), "best_ms": round(min(ms), 3),
           "median_ms": round(statistics.median(ms), 3), "GB_s": round(sum(lens) / min(ms) / 1e6, 2)}
    if load is not None:  # load_ranges of arm (a) scaled to these bytes
        row["share_of_load_ranges_at_arm_a_rate"] = round(min(ms) / (sum(lens) / (load["GB_s"] * 1e6)), 4)
    out.append({**row, **info})
    print(json.dumps(out[-1]), flush=True)


LLAMA = {"q_proj": (2048, 2048), "k_proj": (512, 2048), "v_proj": (512, 2048), "o_proj": (2048, 2048),
         "gate_proj": (5632, 2048), "up_proj": (5632, 2048), "down_proj": (2048, 5632), "input_layernorm": (2048,),
         "post_attention_layernorm": (2048,)}


def llama_shapes(total: int) -> dict:
    per = sum(2 * (s[0] * (s[1] if len(s) > 1 else 1)) for s in LLAMA.values())
    return {f"layers.{i}.{k}.weight": s for i in range(max(1, total // per)) for k, s in LLAMA.items()}


def tp_index(name: str, shape, rank: int, ranks: int = 8):
    if len(shape) == 1:
        return ...
    d = 1 if ("o_proj" in name or "down_proj" in name) else 0
    n = shape[d] // ranks
    return (slice(None),) * d + (slice(rank * n, (rank + 1) * n),)


def slices_kernel_arm(ctx, info, out):
    """The TP slices of a Llama stack (few boxes per wave), then a selection that enumerates its outer dimension: rows
    4..11 and columns 2048..3071 of every expert of a [511, 16, 8192] stack, 511 boxes in one wave."""
    rank = int(os.environ.get("VRB_RANK", "3"))
    wave = 16 * blob_utils.BLOCK_SIZE
    box_workload(ctx, info, out, "slices_kernel", llama_shapes(2 * wave), lambda n, s: tp_index(n, s, rank))
    box_workload(ctx, info, out, "slices_kernel_many_boxes", {"experts.weight": (511, 16, 8192)},
                 lambda n, s: (slice(None), slice(4, 12), slice(2048, 3072)))
    one_row_boxes_arm(ctx, info, out)


def box_workload(ctx, info, out, label: str, shapes: dict, index_of):
    import ctypes

    from modal_client_b200 import load_boxes

    BS, rank = blob_utils.BLOCK_SIZE, int(os.environ.get("VRB_RANK", "3"))
    wave = 16 * BS
    data0 = 8 + 8 * 126  # the data region starts at 8 mod 16
    # the file's tensors in data order; the wave holds file bytes [0, wave) in consecutive slots
    runs, tensors, at, dest = [], [], data0, 0
    for name, shape in shapes.items():
        nbytes = 2 * int(np.prod(shape))
        if at >= wave:
            break
        bounds, kept = volume._slice_bounds(name, shape, index_of(name, shape))
        result = [hi - lo for (lo, hi), k in zip(bounds, kept) if k]
        first = len(runs)
        for run in volume._slice_runs(shape, bounds, 2, at):
            runs.append((run, dest))
            dest += run[1] * run[3]
        tensors.append((name, shape, at, nbytes, bounds, first, len(runs)))
        at += nbytes
    boxes = [(0, *b) for run, d in runs for b in volume._clip_run(run, d, 0, wave, 0)]
    selected = sum(b[2] * b[3] for b in boxes)
    # the sliced results of tensors wholly inside the wave (the comparison of route (3) needs whole tensors)
    whole = [t for t in tensors if t[2] + t[3] <= wave]
    src = ctx.host_alloc(wave)
    try:
        src[:] = torch.randint(0, 256, (wave,), dtype=torch.uint8).numpy()
        dst = {k: torch.zeros(dest, dtype=torch.uint8, device="cuda") for k in ("load_boxes", "memcpy2d", "slice")}
        scratch = torch.empty(wave, dtype=torch.uint8, device="cuda")
        ceiling_dst = torch.empty(selected, dtype=torch.uint8, device="cuda")
        ceiling_src = torch.from_numpy(src[:selected].copy()).pin_memory()
        cudart = ctypes.CDLL("libcudart.so.12")
        cudart.cudaMemcpy2DAsync.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t,
                                             ctypes.c_size_t, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p]
        f = DeviceFile(dst["load_boxes"])
        base, out_ptr = src.ctypes.data, dst["memcpy2d"].data_ptr()
        stream = torch.cuda.current_stream().cuda_stream

        def memcpy2d():
            for _, off, w, r, at, pitch in boxes:
                rc = cudart.cudaMemcpy2DAsync(out_ptr + off, w, base + at, pitch, w, r, 1, stream)
                assert rc == 0, rc

        def slice_route():
            load_ranges([DeviceFile(scratch)], [(0, 0, wave)], src, [0], ctx=ctx)
            for name, shape, at, nbytes, bounds, first, last in whole:
                if first == last:
                    continue
                t = scratch[at : at + nbytes].view(torch.bfloat16).view(shape)
                part = t[tuple(slice(lo, hi) for lo, hi in bounds)]
                d0 = runs[first][1]
                dst["slice"][d0 : d0 + part.numel() * 2].view(torch.bfloat16).view(part.shape).copy_(part)

        cands = {"load_boxes": lambda: load_boxes([f], boxes, src, ctx=ctx), "memcpy2d_per_box": memcpy2d,
                 "load_ranges_then_slice": slice_route,
                 "memcpy_ceiling": lambda: ceiling_dst.copy_(ceiling_src, non_blocking=True)}
        for fn in cands.values():
            fn()
        times, enqueue = {k: [] for k in cands}, {k: [] for k in cands}

        def host_timed(k, fn):
            def run():
                t0 = time.perf_counter()
                fn()
                enqueue[k].append((time.perf_counter() - t0) * 1e3)
            return run

        for _ in range(int(os.environ.get("VRB_REPS", "5"))):
            for k, fn in cands.items():
                times[k].append(events_ms(host_timed(k, fn)))
        torch.cuda.synchronize()
        whole_end = runs[whole[-1][6] - 1][1] + runs[whole[-1][6] - 1][0][1] * runs[whole[-1][6] - 1][0][3]
        equal = {"memcpy2d_equal": torch.equal(dst["load_boxes"], dst["memcpy2d"]),
                 "slice_equal_on_whole_tensors": torch.equal(dst["load_boxes"][:whole_end], dst["slice"][:whole_end])}
        best = {k: min(v) for k, v in times.items()}
        for k, v in times.items():
            out.append({"arm": f"{label}.{k}", "selected_bytes": selected, "wave_bytes": wave, "boxes": len(boxes),
                        "tensors": len(tensors), "rank": rank, "best_ms": round(best[k], 3),
                        "median_ms": round(statistics.median(v), 3), "GB_s": round(selected / best[k] / 1e6, 2),
                        "host_call_median_ms": round(statistics.median(enqueue[k]), 3),
                        "share_of_ceiling": round(best["memcpy_ceiling"] / best[k], 3), **equal, **info})
            print(json.dumps(out[-1]), flush=True)
    finally:
        torch.cuda.synchronize()
        ctx.host_free(src)


def one_row_boxes_arm(ctx, info, out):
    """Arm (a)'s workload (every block of a safetensors image at its slot) as 1-row boxes, next to load_ranges."""
    from modal_client_b200 import load_boxes

    BS = blob_utils.BLOCK_SIZE
    sd = state_dict(int(float(os.environ.get("VRB_GIB", "2")) * GiB))
    f = DeviceFile.safetensors(sd)
    n = f.nbytes
    ranges = [(0, o, min(BS, n - o)) for o in range(0, n, BS)]
    boxes = [(0, o, m, 1, o, m) for _, o, m in ranges]
    src = ctx.host_alloc(n)
    try:
        src[:] = torch.randint(0, 256, (n,), dtype=torch.uint8).numpy()
        cands = {"load_ranges": lambda: load_ranges([f], ranges, src, [o for _, o, _ in ranges], ctx=ctx),
                 "load_boxes_1_row": lambda: load_boxes([f], boxes, src, ctx=ctx)}
        for fn in cands.values():
            fn()
        times = {k: [] for k in cands}
        for _ in range(int(os.environ.get("VRB_REPS", "5"))):
            for k, fn in cands.items():
                times[k].append(events_ms(fn))
        torch.cuda.synchronize()
        ok = b"".join(s.cpu().numpy().tobytes() for s in f._src.segments) == src.tobytes()
        for k, v in times.items():
            out.append({"arm": f"arm_a_workload.{k}", "bytes": n, "ranges": len(ranges), "best_ms": round(min(v), 3),
                        "median_ms": round(statistics.median(v), 3), "GB_s": round(n / min(v) / 1e6, 2),
                        "bytes_equal": ok, **info})
            print(json.dumps(out[-1]), flush=True)
    finally:
        torch.cuda.synchronize()
        ctx.host_free(src)
    del sd, f


async def slices_e2e_arm(info, out):
    BS = blob_utils.BLOCK_SIZE
    total = int(float(os.environ.get("VRB_E2E_GIB", "1")) * GiB)
    g = torch.Generator(device="cuda").manual_seed(7)
    sd = {k: torch.randn(s, device="cuda", generator=g).to(torch.bfloat16) for k, s in llama_shapes(total).items()}
    size = sum(t.numel() * 2 for t in sd.values())
    got_bytes = [0]
    real_fetch = volume._fetch_block

    async def counting_fetch(url, buf, want, semaphore):
        got_bytes[0] += want
        await real_fetch(url, buf, want, semaphore)

    volume._fetch_block = counting_fetch
    rows = {"slices": [], "full_then_slice": []}
    try:
        async with running_volume_server(BS) as (stub, _):
            client = types.SimpleNamespace(stub=stub)
            async with volume.VolumeUploadContextManager2("vo-b", client) as batch:
                batch.put_file(DeviceFile.safetensors(sd), "/tp.safetensors")
            del sd
            _, info_hdr = await volume.read_safetensors_header(client, "vo-b", "/tp.safetensors")
            for rank in range(8):
                select = {k: tp_index(k, s, rank) for k, (_, s) in info_hdr.items()}
                results = {}
                order = ("slices", "full_then_slice") if rank % 2 == 0 else ("full_then_slice", "slices")
                for route in order:
                    torch.cuda.synchronize()
                    got_bytes[0] = 0
                    hbm = torch.cuda.memory_allocated()
                    torch.cuda.reset_peak_memory_stats()
                    with PeakRss() as rss:
                        t0 = time.perf_counter()
                        if route == "slices":
                            res = await volume.read_safetensors_slices(client, "vo-b", "/tp.safetensors", select)
                        else:
                            full = await volume.read_safetensors(client, "vo-b", "/tp.safetensors")
                            res = {k: full[k][i].contiguous() for k, i in select.items()}
                            del full
                        torch.cuda.synchronize()
                        dt = time.perf_counter() - t0
                    results[route] = res
                    rows[route].append((dt, got_bytes[0], torch.cuda.max_memory_allocated() - hbm, rss.growth))
                equal = all(torch.equal(results["slices"][k].view(torch.int16),
                                        results["full_then_slice"][k].view(torch.int16)) for k in select)
                rows["slices"][-1] += (equal,)
                rows["full_then_slice"][-1] += (equal,)
                del results
    finally:
        volume._fetch_block = real_fetch
    for route, v in rows.items():
        ts = [x[0] for x in v]
        out.append({"arm": f"slices_loopback.{route}", "file_bytes": size, "ranks": 8, "median_s": round(statistics.median(ts), 3),
                    "range_s": [round(min(ts), 3), round(max(ts), 3)],
                    "bytes_get_per_rank": [x[1] for x in v], "peak_hbm_growth_GB": round(max(x[2] for x in v) / 1e9, 3),
                    "peak_rss_growth_GB": round(max(x[3] for x in v) / 1e9, 3),
                    "bitwise_equal": all(x[4] for x in v), **info})
        print(json.dumps(out[-1]), flush=True)


def cast_kernel_arm(ctx, info, out):
    from modal_client_b200 import load_boxes, load_cast_boxes

    BS = blob_utils.BLOCK_SIZE
    n = int(float(os.environ.get("VRB_GIB", "2")) * GiB) // BS * BS
    src = ctx.host_alloc(n + 16)
    try:
        torch.from_numpy(src).random_(0, 256)
        for stored, target in ((torch.float32, torch.bfloat16), (torch.bfloat16, torch.float32)):
            ss, ds = stored.itemsize, target.itemsize
            plain = torch.empty(n, dtype=torch.uint8, device="cuda")  # the unconverted bytes / the unfused scratch
            conv = torch.empty(n // ss, dtype=target, device="cuda")
            fp, fc = DeviceFile(plain), DeviceFile(conv)
            for phase in (0, 8):
                # one 1-row box per 8 MiB block slot; the data region starts at `phase`
                blocks = [(max(phase, o), o + BS - max(phase, o)) for o in range(0, n, BS)]
                plain_boxes = [(0, a - phase, m, 1, a, m) for a, m in blocks]
                cast_boxes = [(0, (a - phase) // ss * ds, m, 1, a, m, stored, target) for a, m in blocks]
                nbytes = sum(m for _, m in blocks)
                view, head = plain[: nbytes].view(stored), conv[: nbytes // ss]

                def unfused():
                    load_boxes([fp], plain_boxes, src, ctx=ctx)
                    head.copy_(view)

                cands = {"load_cast_boxes": lambda: load_cast_boxes([fc], cast_boxes, src, ctx=ctx),
                         "load_boxes": lambda: load_boxes([fp], plain_boxes, src, ctx=ctx),
                         "load_boxes_then_to": unfused}
                for fn in cands.values():
                    fn()
                times = {k: [] for k in cands}
                for _ in range(int(os.environ.get("VRB_REPS", "5"))):
                    for k, fn in cands.items():
                        times[k].append(events_ms(fn))
                load_cast_boxes([fc], cast_boxes, src, ctx=ctx)
                load_boxes([fp], plain_boxes, src, ctx=ctx)
                torch.cuda.synchronize()
                iv = torch.int16 if ds == 2 else torch.int32
                equal = torch.equal(conv[: nbytes // ss].view(iv), view.to(target).view(iv))
                best = {k: min(v) for k, v in times.items()}
                for k, v in times.items():
                    out.append({"arm": f"cast_kernel.{stored}_to_{target}.phase{phase}.{k}", "source_bytes": nbytes,
                                "boxes": len(blocks), "best_ms": round(best[k], 3),
                                "median_ms": round(statistics.median(v), 3), "GB_s": round(nbytes / best[k] / 1e6, 2),
                                "share_of_load_boxes": round(best["load_boxes"] / best[k], 3), "bitwise_equal": equal,
                                **info})
                    print(json.dumps(out[-1]), flush=True)
            del fp, fc, plain, conv, view, head
    finally:
        torch.cuda.synchronize()
        ctx.host_free(src)


async def cast_e2e_arm(info, out):
    BS = blob_utils.BLOCK_SIZE
    total = int(float(os.environ.get("VRB_E2E_GIB", "1")) * GiB)
    rank = int(os.environ.get("VRB_RANK", "3"))
    g = torch.Generator(device="cuda").manual_seed(8)
    sd = {k: torch.randn(s, device="cuda", generator=g) for k, s in llama_shapes(total // 2).items()}  # F32
    size = sum(t.numel() * 4 for t in sd.values())
    bf16 = torch.bfloat16
    rows = {}
    async with running_volume_server(BS) as (stub, _):
        client = types.SimpleNamespace(stub=stub)
        async with volume.VolumeUploadContextManager2("vo-e", client) as batch:
            batch.put_file(DeviceFile.safetensors(sd), "/f32.safetensors")
        shapes = {k: tuple(t.shape) for k, t in sd.items()}
        del sd
        select = {k: tp_index(k, s, rank) for k, s in shapes.items()}

        async def read(converted: bool, sliced: bool):
            if sliced:
                if converted:
                    return await volume.read_safetensors_slices(client, "vo-e", "/f32.safetensors", select, dtype=bf16)
                res = await volume.read_safetensors_slices(client, "vo-e", "/f32.safetensors", select)
            else:
                if converted:
                    return await volume.read_safetensors(client, "vo-e", "/f32.safetensors", dtype=bf16)
                res = await volume.read_safetensors(client, "vo-e", "/f32.safetensors")
            out_ = {}
            for k in list(res):
                out_[k] = res.pop(k).to(bf16)
            return out_

        for sliced in (False, True):
            label = "slices_rank" if sliced else "full"
            for rep in range(int(os.environ.get("VRB_E2E_REPS", "2"))):
                results = {}
                order = (True, False) if rep % 2 == 0 else (False, True)
                for converted in order:
                    route = f"{label}.{'dtype_bf16' if converted else 'read_then_to_bf16'}"
                    torch.cuda.synchronize()
                    hbm = torch.cuda.memory_allocated()
                    torch.cuda.reset_peak_memory_stats()
                    t0 = time.perf_counter()
                    res = await read(converted, sliced)
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                    rows.setdefault(route, []).append((dt, torch.cuda.max_memory_allocated() - hbm))
                    results[converted] = res
                equal = all(torch.equal(results[True][k].view(torch.int16), results[False][k].view(torch.int16))
                            for k in results[True])
                for converted in order:
                    route = f"{label}.{'dtype_bf16' if converted else 'read_then_to_bf16'}"
                    rows[route][-1] += (equal,)
                del results
    for route, v in rows.items():
        ts = [x[0] for x in v]
        out.append({"arm": f"cast_loopback.{route}", "file_bytes": size, "rank": rank if "slices" in route else None,
                    "median_s": round(statistics.median(ts), 3), "range_s": [round(min(ts), 3), round(max(ts), 3)],
                    "peak_hbm_growth_GB": round(max(x[1] for x in v) / 1e9, 3),
                    "bitwise_equal": all(x[2] for x in v), **info})
        print(json.dumps(out[-1]), flush=True)


def _dequant_bf16(w, s):
    """torch's CUDA dequantization of an E4M3 weight with 128 x 128 block scales, to bfloat16."""
    R, C = w.shape
    full = s.repeat_interleave(128, 0)[:R].repeat_interleave(128, 1)[:, :C]
    return (w.float() * full).to(torch.bfloat16)


def fp8_kernel_arm(ctx, info, out):
    from modal_client_b200 import load_boxes, load_scaled_boxes

    BS, C, phase = blob_utils.BLOCK_SIZE, 7168, 8
    n = 16 * BS
    R = (n - phase) // C
    g = torch.Generator(device="cuda").manual_seed(9)
    w = (torch.randn(R, C, generator=g, device="cuda") * 50).to(torch.float8_e4m3fn)
    s = torch.rand(-(-R // 128), C // 128, generator=g, device="cuda") * 1e-3
    src = ctx.host_alloc(n + 16)
    try:
        src[phase : phase + R * C] = w.view(torch.uint8).reshape(-1).cpu().numpy()
        nbytes = R * C
        blocks = [(max(phase, o), min(o + BS, phase + nbytes) - max(phase, o)) for o in range(0, n, BS)]
        blocks = [(a, m) for a, m in blocks if m > 0]
        plain = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        res = torch.empty(R, C, dtype=torch.bfloat16, device="cuda")
        fp, fr = DeviceFile(plain), DeviceFile(res)
        plain_boxes = [(0, a - phase, m, 1, a, m) for a, m in blocks]
        scaled_boxes = [(0, (a - phase) * 2, m, 1, a, m, torch.float8_e4m3fn, torch.bfloat16, s, a - phase, R, C, 128, 128)
                        for a, m in blocks]
        cands = {"load_scaled_boxes": lambda: load_scaled_boxes([fr], scaled_boxes, src, ctx=ctx),
                 "load_boxes": lambda: load_boxes([fp], plain_boxes, src, ctx=ctx)}
        for fn in cands.values():
            fn()
        times = {k: [] for k in cands}
        for _ in range(int(os.environ.get("VRB_REPS", "5"))):
            for k, fn in cands.items():
                times[k].append(events_ms(fn))
        torch.cuda.synchronize()
        equal = torch.equal(res.view(torch.int16), _dequant_bf16(w, s).view(torch.int16)) and \
            torch.equal(plain, w.view(torch.uint8).reshape(-1))
        best = {k: min(v) for k, v in times.items()}
        for k, v in times.items():
            out.append({"arm": f"fp8_kernel.e4m3_to_bf16.{k}", "source_bytes": nbytes, "boxes": len(blocks),
                        "best_ms": round(best[k], 3), "median_ms": round(statistics.median(v), 3),
                        "GB_s": round(nbytes / best[k] / 1e6, 2),
                        "share_of_load_boxes": round(best["load_boxes"] / best[k], 3), "bitwise_equal": equal, **info})
            print(json.dumps(out[-1]), flush=True)
        del fp, fr, plain, res
    finally:
        torch.cuda.synchronize()
        ctx.host_free(src)


def fp8_stack(total: int, h: int = 4096, m: int = 12288) -> dict:
    """Qwen3/DeepSeek-shaped E4M3 layers (q, kv_a with 576 rows, o, gate, up, down) with F32 128 x 128
    ``weight_scale_inv`` tensors and BF16 norms, about ``total`` bytes."""
    shapes = {"self_attn.q_proj": (h, h), "self_attn.kv_a_proj": (576, h), "self_attn.o_proj": (h, h),
              "mlp.gate_proj": (m, h), "mlp.up_proj": (m, h), "mlp.down_proj": (h, m)}
    per = sum(r * c for r, c in shapes.values())
    g = torch.Generator(device="cuda").manual_seed(10)
    sd = {}
    for i in range(max(1, total // per)):
        p = f"model.layers.{i}."
        for k, (r, c) in shapes.items():
            sd[p + k + ".weight"] = (torch.randn(r, c, generator=g, device="cuda") * 50).to(torch.float8_e4m3fn)
            sd[p + k + ".weight_scale_inv"] = torch.rand(-(-r // 128), -(-c // 128), generator=g, device="cuda") * 1e-3
        sd[p + "input_layernorm.weight"] = torch.randn(h, generator=g, device="cuda").to(torch.bfloat16)
    return sd


async def fp8_e2e_arm(info, out):
    from modal_client_b200 import device_file

    BS = blob_utils.BLOCK_SIZE
    sd = fp8_stack(int(float(os.environ.get("VRB_FP8_GIB", "2.5")) * 1e9))
    size = sum(t.numel() * t.element_size() for t in sd.values())
    index = "/fp8/model.safetensors.index.json"
    rows = {}
    async with running_volume_server(BS) as (stub, _):
        client = types.SimpleNamespace(stub=stub)
        shards = device_file.safetensors_shards(sd, max_shard_size="1GB")
        nshards = len(shards.files)
        async with volume.VolumeUploadContextManager2("vo-f", client) as batch:
            shards.put(batch, "/fp8")
        del shards, sd
        _, where = await volume.read_safetensors_index(client, "vo-f", index)
        scales = volume.fp8_scales(where)

        async def read(fused: bool):
            if fused:
                return await volume.read_safetensors_sharded(client, "vo-f", index, dtype=torch.bfloat16,
                                                             scales=scales)
            res = await volume.read_safetensors_sharded(client, "vo-f", index)
            for w, sc in scales.items():
                res[w] = _dequant_bf16(res[w], res.pop(sc))
            return res

        for rep in range(int(os.environ.get("VRB_FP8_REPS", "3"))):
            results = {}
            order = (True, False) if rep % 2 == 0 else (False, True)
            for fused in order:
                route = "dtype_bf16_scales" if fused else "read_then_torch_dequant"
                torch.cuda.synchronize()
                hbm = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                t0 = time.perf_counter()
                res = await read(fused)
                torch.cuda.synchronize()
                rows.setdefault(route, []).append([time.perf_counter() - t0,
                                                   torch.cuda.max_memory_allocated() - hbm])
                results[fused] = res
            equal = sorted(results[True]) == sorted(results[False]) and all(
                torch.equal(results[True][k].view(torch.int16), results[False][k].view(torch.int16))
                for k in results[True])
            for route in rows:
                rows[route][-1].append(equal)
            del results
    for route, v in rows.items():
        ts = [x[0] for x in v]
        out.append({"arm": f"fp8_loopback.{route}", "file_bytes": size, "shards": nshards,
                    "median_s": round(statistics.median(ts), 3), "range_s": [round(min(ts), 3), round(max(ts), 3)],
                    "peak_hbm_growth_GB": round(max(x[1] for x in v) / 1e9, 3),
                    "bitwise_equal": all(x[2] for x in v), **info})
        print(json.dumps(out[-1]), flush=True)


def main():
    if not torch.cuda.is_available():
        raise SystemExit("volume_read_bench needs a GPU")
    info = gpu_info()
    ctx = _lib.Context(0, pinned_bytes=64 << 20, device_bytes=512 << 20)
    _backend.set_context(ctx)
    out, arms = [], os.environ.get("VRB_ARMS", "abcd")
    if "a" in arms:
        kernel_arm(ctx, info, out)
    if "b" in arms:
        asyncio.run(e2e_arm(info, out))
    if "c" in arms:
        asyncio.run(torch_save_arm(ctx, info, out))
    if "d" in arms:
        slices_kernel_arm(ctx, info, out)
        asyncio.run(slices_e2e_arm(info, out))
    if "e" in arms:
        cast_kernel_arm(ctx, info, out)
        asyncio.run(cast_e2e_arm(info, out))
    if "f" in arms:
        fp8_kernel_arm(ctx, info, out)
        asyncio.run(fp8_e2e_arm(info, out))
    if os.environ.get("VRB_OUT"):
        os.makedirs(os.environ["VRB_OUT"], exist_ok=True)
        with open(os.path.join(os.environ["VRB_OUT"], "volume_read_bench.json"), "w") as fh:
            json.dump(out, fh, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
