"""tools/sharded_checkpoint_bench.py -- a checkpoint in the Hugging Face Hub's sharded layout, to and from a volume over
the loopback test server (tests/volume_read_server.py), one wave loop and one batch against the per-shard routes.

Workload: a Llama-shaped stack (hidden 4096, MLP 11008, SCB_LAYERS layers, 10 by default, plus a 32000-row embedding:
about 4.3 GB in bf16) in 1 GB shards (``max_shard_size="1GB"``).  Arms, after one warm-up of each route, alternating,
SCB_REPS (5) runs each, median and range of wall time:

  load    ``read_safetensors_sharded`` of the index against ``read_safetensors_index`` followed by a loop of
          ``read_safetensors`` over the shards (which reads each header again), 256 MiB of staging each; bytes downloaded, VolumeGetFile2 calls and the peak growth
          of torch's HBM allocations over the results; results compared bitwise
  export  from the same stack in F32: ``safetensors_shards(sd, max_shard_size="1GB", dtype=torch.bfloat16).put`` on
          one volumefs2 batch against ``.to(torch.bfloat16)``, the split of ``huggingface_hub`` and a
          ``DeviceFile.safetensors`` per shard plus the index on one batch; 1 GiB of ``device_staging_bytes``, a fresh
          server per run; peak HBM growth; the stored files compared

``SCB_ARMS`` (``load,export``) picks the arms.  The card name and power limit are read in the same run.  Needs a GPU: nothing here falls back.  One JSON line per
route; also written to $SCB_OUT/sharded_checkpoint_bench.json when set."""
import asyncio
import io
import json
import os
import statistics
import sys
import time
import types

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from modal_client_b200 import DeviceFile, blob_utils, device_file, volume  # noqa: E402
from safetensors_blocks_bench import gpu_info  # noqa: E402
from tests.volume_read_server import running_volume_server  # noqa: E402

ARMS = os.environ.get("SCB_ARMS", "load,export").split(",")
LAYERS = int(os.environ.get("SCB_LAYERS", 10))
REPS = int(os.environ.get("SCB_REPS", 5))
BS = blob_utils.BLOCK_SIZE
INDEX = "/ckpt/model.safetensors.index.json"


def llama(dtype) -> dict:
    g = torch.Generator(device="cuda").manual_seed(3)
    h, m = 4096, 11008
    r = lambda *s: (torch.randn(*s, generator=g, device="cuda") * 0.02).to(dtype)  # noqa: E731
    sd = {"model.embed_tokens.weight": r(32000, h)}
    for i in range(LAYERS):
        p = f"model.layers.{i}."
        for k in "qkvo":
            sd[p + f"self_attn.{k}_proj.weight"] = r(h, h)
        sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"] = r(m, h), r(m, h)
        sd[p + "mlp.down_proj.weight"] = r(h, m)
        sd[p + "input_layernorm.weight"], sd[p + "post_attention_layernorm.weight"] = r(h), r(h)
    sd["model.norm.weight"] = r(h)
    sd["lm_head.weight"] = r(32000, h)
    return sd


def spread(xs):
    return {"median_s": round(statistics.median(xs), 3), "range_s": [round(min(xs), 3), round(max(xs), 3)]}


def bitwise_equal(a: dict, b: dict) -> bool:
    return a.keys() == b.keys() and all(torch.equal(a[k].view(torch.int16), b[k].view(torch.int16)) for k in a)


async def load_arm(info, out):
    sd = llama(torch.bfloat16)
    shards = device_file.safetensors_shards(sd, max_shard_size="1GB")
    image = sum(f.nbytes for f in shards.files.values())
    got_bytes = [0]
    real_fetch = volume._fetch_block

    async def counting_fetch(url, buf, want, semaphore):
        got_bytes[0] += want
        await real_fetch(url, buf, want, semaphore)

    async def per_shard(client):  # the index and its shards' headers, then read_safetensors shard by shard
        _, where = await volume.read_safetensors_index(client, "vo-b", INDEX)
        res = {}
        for path in dict.fromkeys(p for p, _, _ in where.values()):
            res.update(await volume.read_safetensors(client, "vo-b", path))
        return res

    routes = {"one_wave_loop": lambda c: volume.read_safetensors_sharded(c, "vo-b", INDEX), "per_shard": per_shard}
    rows = {k: [] for k in routes}
    volume._fetch_block = counting_fetch
    try:
        async with running_volume_server(BS) as (stub, _):
            client = types.SimpleNamespace(stub=stub)
            async with volume.VolumeUploadContextManager2("vo-b", client) as batch:
                shards.put(batch, "/ckpt")
            del shards
            for rep in range(REPS + 1):
                results = {}
                for name in (("one_wave_loop", "per_shard") if rep % 2 == 0 else ("per_shard", "one_wave_loop")):
                    torch.cuda.synchronize()
                    got_bytes[0], calls = 0, len(stub.get_file_calls)
                    hbm = torch.cuda.memory_allocated()
                    torch.cuda.reset_peak_memory_stats()
                    t0 = time.perf_counter()
                    res = await routes[name](client)
                    torch.cuda.synchronize()
                    dt = time.perf_counter() - t0
                    held = sum(t.numel() * t.element_size() for t in res.values())
                    if rep:  # rep 0 warms both routes up
                        rows[name].append((dt, got_bytes[0], len(stub.get_file_calls) - calls,
                                           torch.cuda.max_memory_allocated() - hbm - held))
                    results[name] = res
                equal = bitwise_equal(results["one_wave_loop"], results["per_shard"]) and \
                    bitwise_equal(results["one_wave_loop"], {k: sd[k] for k in results["per_shard"]})
                del results
                assert equal, "the two routes read different tensors"
    finally:
        volume._fetch_block = real_fetch
    for name, v in rows.items():
        out.append({"arm": f"load.{name}", "image_bytes": image, "reps": REPS, **spread([x[0] for x in v]),
                    "bytes_get": sorted({x[1] for x in v}), "get_file2_calls": sorted({x[2] for x in v}),
                    "peak_hbm_growth_over_results_MB": round(max(x[3] for x in v) / 1e6, 3), "bitwise_equal": True,
                    **info})
        print(json.dumps(out[-1]), flush=True)


async def export_once(make):
    """``make(batch)`` queues the files: (seconds from building the files to the batch's end, peak HBM growth, stored files) on a fresh server."""
    async with running_volume_server(BS) as (stub, _):
        client = types.SimpleNamespace(stub=stub)
        torch.cuda.synchronize()
        hbm = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        batch = volume.VolumeUploadContextManager2("vo-b", client, device_staging_bytes=1 << 30)
        async with batch:
            make(batch)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        return dt, torch.cuda.max_memory_allocated() - hbm, {p: v[0] for p, v in stub.volume_files.items()}


def export_arm(info, out):
    from huggingface_hub import split_torch_state_dict_into_shards

    sd = llama(torch.float32)

    def shards_route(batch):
        device_file.safetensors_shards(sd, max_shard_size="1GB", dtype=torch.bfloat16).put(batch, "/ckpt")

    def manual_route(batch):
        pre = {k: v.to(torch.bfloat16) for k, v in sd.items()}
        split = split_torch_state_dict_into_shards(pre, max_shard_size="1GB")
        files = {f"/ckpt/{n}": DeviceFile.safetensors({k: pre[k] for k in names}, {"format": "pt"})
                 for n, names in split.filename_to_tensors.items()}
        index = {"metadata": split.metadata, "weight_map": split.tensor_to_filename}
        files["/ckpt/model.safetensors.index.json"] = io.BytesIO(json.dumps(index, indent=2).encode())
        for path, f in files.items():
            batch.put_file(f, path)

    routes = {"safetensors_shards": shards_route, "to_then_per_shard": manual_route}
    rows = {k: [] for k in routes}
    for rep in range(REPS + 1):
        stored = {}
        for name in (("safetensors_shards", "to_then_per_shard") if rep % 2 == 0 else
                     ("to_then_per_shard", "safetensors_shards")):
            dt, growth, stored[name] = asyncio.run(export_once(routes[name]))
            if rep:
                rows[name].append((dt, growth))
        assert stored["safetensors_shards"] == stored["to_then_per_shard"], "the routes stored different files"
        image = sum(len(v) for v in stored["safetensors_shards"].values())
        del stored
    for name, v in rows.items():
        out.append({"arm": f"export.{name}", "stored_bytes": image, "reps": REPS, **spread([x[0] for x in v]),
                    "peak_hbm_growth_GB": round(max(x[1] for x in v) / 1e9, 3), "files_equal": True, **info})
        print(json.dumps(out[-1]), flush=True)


def main():
    if not torch.cuda.is_available():
        raise SystemExit("sharded_checkpoint_bench needs a GPU")
    info = gpu_info()
    out = []
    if "load" in ARMS:
        asyncio.run(load_arm(info, out))
        torch.cuda.empty_cache()
    if "export" in ARMS:
        export_arm(info, out)
    if os.environ.get("SCB_OUT"):
        os.makedirs(os.environ["SCB_OUT"], exist_ok=True)
        with open(os.path.join(os.environ["SCB_OUT"], "sharded_checkpoint_bench.json"), "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
