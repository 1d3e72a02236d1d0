"""tools/fp8_load_bench.py -- loading a bf16 checkpoint from a volume as block-scaled FP8:
``read_safetensors_sharded(..., fp8=names)``, which quantizes the weights in the staging waves, against reading the
bf16 checkpoint and quantizing every weight with torch's ``per_block_cast_to_fp8``, and against reading the
pre-quantized FP8 file.

The workload is the Llama-shaped bf16 stack of tools/fp8_export_bench.py (hidden 4096, MLP 11008, F8L_LAYERS layers,
10 by default: 4.05 GB); every 2-D weight is quantized in 128 x 128 blocks, the norms stay bf16.  Both checkpoints are
uploaded once to the in-process loopback volume server (tests/volume_read_server.py) in 2 GB shards.  Arms, after one
warm-up of each, alternating, F8L_REPS (3) runs each, median and range, with the peak growth of torch's HBM allocations
over the call:

  a  ``read_safetensors_sharded(bf16 index, fp8=names)``
  b  ``read_safetensors_sharded(bf16 index)`` then ``per_block_cast_to_fp8`` of every weight (the bf16 image and the
     results in HBM together)
  c  ``read_safetensors_sharded(fp8 index)`` of the pre-quantized export of the same tensors

The outputs of (a) and (b) are compared bitwise, and (c) must equal them too.  A kernel arm times, with CUDA events,
one wave's worth of the stack (the four attention weights of a layer, 128 MiB, the default staging half) staged in
page-locked memory: the quantizing calls (``load_fp8_amax_boxes`` then ``load_quant_boxes`` with one band per weight)
against one ``load_cast_boxes`` bf16 -> f16 over the same boxes.  The card name and power limit are read in the same
run.  Needs a GPU: nothing here falls back.  One JSON line per arm; also written to $F8L_OUT/fp8_load_bench.json when
set."""
import asyncio
import json
import os
import statistics
import sys
import time
import types

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from device_cast_upload_bench import events, summary  # noqa: E402
from fp8_export_bench import llama_stack, per_block_cast_to_fp8  # noqa: E402
from modal_client_b200 import (DeviceFile, _backend, blob_utils, device_file, load_cast_boxes,  # noqa: E402
                               load_fp8_amax_boxes, load_quant_boxes, volume)
from safetensors_blocks_bench import gpu_info  # noqa: E402
from tests.volume_read_server import running_volume_server  # noqa: E402

LAYERS = int(os.environ.get("F8L_LAYERS", 10))
REPS = int(os.environ.get("F8L_REPS", 3))
KREPS = 20


def _equal(a: dict, b: dict) -> bool:
    return sorted(a) == sorted(b) and all(
        a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and torch.equal(a[k].view(torch.uint8),
                                                                            b[k].view(torch.uint8)) for k in a)


def kernel_arm(ctx, sd, info) -> dict:
    names = [f"layers.0.{n}.weight" for n in ("q", "k", "v", "o")]
    ws = [sd[n] for n in names]
    total = sum(w.numel() * 2 for w in ws)
    buf = ctx.host_alloc(total)
    try:
        offs, at = [], 0
        for w in ws:
            buf[at : at + w.numel() * 2] = w.contiguous().view(torch.uint8).reshape(-1).cpu().numpy()
            offs.append(at)
            at += w.numel() * 2
        q = [torch.empty(w.shape, dtype=torch.float8_e4m3fn, device="cuda") for w in ws]
        h = [torch.empty(w.shape, dtype=torch.float16, device="cuda") for w in ws]
        grids = [(-(-w.shape[0] // 128), -(-w.shape[1] // 128)) for w in ws]
        amax = [torch.empty(g[0] * g[1], dtype=torch.float32, device="cuda") for g in grids]
        scales = [torch.empty(g, dtype=torch.float32, device="cuda") for g in grids]
        fq = DeviceFile._over(DeviceFile._Source(q, device_file.BOUNCE_BYTES))
        fh = DeviceFile._over(DeviceFile._Source(h, device_file.BOUNCE_BYTES))
        qboxes, hboxes, d = [], [], 0
        for w, o, a in zip(ws, offs, amax):
            n = w.numel()
            qboxes.append((0, d, n * 2, 1, o, n * 2, torch.bfloat16, a, 0, w.shape[0], w.shape[1], 128, 128))
            hboxes.append((0, d * 2, n * 2, 1, o, n * 2, torch.bfloat16, torch.float16))
            d += n
        bands = [(a, s.view(-1), 0, a.numel()) for a, s in zip(amax, scales)]

        def quant():
            def run():
                for a in amax:
                    a.zero_()
                load_fp8_amax_boxes([fq], qboxes, buf, ctx=ctx)
                load_quant_boxes([fq], qboxes, bands, buf, ctx=ctx)
            return events(run)[0]

        def cast():
            return events(lambda: load_cast_boxes([fh], hboxes, buf, ctx=ctx))[0]

        quant(), cast()
        times = {"quant": [], "cast": []}
        for _ in range(KREPS):
            times["quant"].append(quant())
            times["cast"].append(cast())
        for w, got, s in zip(ws, q, scales):
            wq, ws_ = per_block_cast_to_fp8(w)
            assert torch.equal(got.view(torch.uint8), wq.view(torch.uint8)) and torch.equal(s, ws_)
        med = {k: statistics.median(v) for k, v in times.items()}
        return {"arm": "kernel, one 128 MiB wave", **{k: summary(v) for k, v in times.items()}, "source_bytes": total,
                "quant_gbs": round(total / med["quant"] / 1e6, 2), "cast_gbs": round(total / med["cast"] / 1e6, 2),
                "quant_over_cast": round(med["quant"] / med["cast"], 3), "outputs_equal": True, **info}
    finally:
        ctx.host_free(buf)


async def e2e_arm(sd, info) -> dict:
    names = [n for n, t in sd.items() if t.dim() == 2]
    async with running_volume_server(blob_utils.BLOCK_SIZE) as (stub, _):
        client = types.SimpleNamespace(stub=stub)
        for where, kw in (("/bf16", {}), ("/fp8", {"fp8": names})):
            shards = device_file.safetensors_shards(sd, max_shard_size="2GB", **kw)
            async with volume.VolumeUploadContextManager2("vo-bench", client) as batch:
                shards.put(batch, where)
            del shards

        async def a():
            return await volume.read_safetensors_sharded(client, "vo-bench", "/bf16/model.safetensors.index.json",
                                                         fp8=names)

        async def b():
            got = await volume.read_safetensors_sharded(client, "vo-bench", "/bf16/model.safetensors.index.json")
            out = {}
            for n, t in got.items():
                if n in names:
                    out[n], out[n + "_scale_inv"] = per_block_cast_to_fp8(t)
                else:
                    out[n] = t
            return out

        async def c():
            return await volume.read_safetensors_sharded(client, "vo-bench", "/fp8/model.safetensors.index.json")

        async def timed(fn):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            t0 = time.perf_counter()
            out = await fn()
            torch.cuda.synchronize()
            return time.perf_counter() - t0, (torch.cuda.max_memory_allocated() - base) / 2**30, out

        arms = {"a_fp8_on_load": a, "b_bf16_then_torch": b, "c_prequantized": c}
        res = {k: {"s": [], "hbm_gib": []} for k in arms}
        for fn in arms.values():  # warm-up
            await timed(fn)
        for _ in range(REPS):
            outs = {}
            for k, fn in arms.items():
                s, g, outs[k] = await timed(fn)
                res[k]["s"].append(s)
                res[k]["hbm_gib"].append(g)
            assert _equal(outs["a_fp8_on_load"], outs["b_bf16_then_torch"])
            assert _equal(outs["a_fp8_on_load"], outs["c_prequantized"])
            del outs
        return {"arm": "e2e loopback read", "reps": REPS, "bf16_bytes": sum(t.numel() * 2 for t in sd.values()),
                **{k: {"median_s": round(statistics.median(v["s"]), 3), "min_s": round(min(v["s"]), 3),
                       "max_s": round(max(v["s"]), 3), "peak_hbm_growth_gib": round(max(v["hbm_gib"]), 3)}
                   for k, v in res.items()}, "a_equals_b_bitwise": True, "a_equals_c_bitwise": True, **info}


def main():
    info = gpu_info()
    ctx = _backend.get_context()
    sd = llama_stack(LAYERS)
    lines = []
    for arm in (lambda: kernel_arm(ctx, sd, info), lambda: asyncio.run(e2e_arm(sd, info))):
        lines.append(json.dumps({"layers": LAYERS, **arm()}))
        print(lines[-1], flush=True)
    if os.environ.get("F8L_OUT"):
        os.makedirs(os.environ["F8L_OUT"], exist_ok=True)
        with open(os.path.join(os.environ["F8L_OUT"], "fp8_load_bench.json"), "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
