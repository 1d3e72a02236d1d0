"""tools/device_cast_upload_bench.py -- exporting an F32 checkpoint in GPU memory as a bf16 safetensors file:
``DeviceFile.safetensors(sd, dtype=torch.bfloat16)``, which converts on the device as blocks are hashed and staged,
against ``{k: v.to(torch.bfloat16)}`` followed by ``DeviceFile.safetensors``, which holds the converted copy in HBM.

The workload is a Llama-shaped F32 stack (hidden 4096, MLP 11008, DCU_LAYERS layers, 5 by default: about 4 GiB).
Arms, after one warm-up of each, alternating, DCU_REPS (7) runs each, median and range:

  1  hashing: the file's 8 MiB blocks, SHA-256 + TRIM_ZEROS (``hash_parts``), CUDA events; the pre-converted route
     reported with and without its ``.to()``
  2  staging: ``stage_ranges`` of every block of the file into one page-locked buffer (``b200h_copy_cast_ranges``
     against ``b200h_copy_ranges_to_host`` of the pre-converted file), CUDA events, GB/s of image bytes
  3  end to end over loopback: the volumefs2 upload with device_staging_bytes = 1 GiB against an in-process fake
     server (device_put_bench.upload), host clock, plus the peak growth of torch's HBM allocations from building the
     file to the end of the upload (the ``.to()`` copy counted for the pre-converted route)

The outputs of the two routes are compared bitwise in every arm (digest tables, staged bytes, blocks the server got).
The card name and power limit are read in the same run.  Needs a GPU: nothing here falls back.
One JSON line per arm; also written to $DCU_OUT/device_cast_upload_bench.json when set."""
import asyncio
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from device_put_bench import upload  # noqa: E402
from modal_client_b200 import DeviceFile, _backend, _lib, blob_utils, stage_ranges  # noqa: E402
from safetensors_blocks_bench import gpu_info  # noqa: E402

LAYERS = int(os.environ.get("DCU_LAYERS", 5))
REPS = int(os.environ.get("DCU_REPS", 7))
BS = blob_utils.BLOCK_SIZE
FLAGS = _lib.SHA256 | _lib.TRIM_ZEROS


def llama_stack(layers: int) -> dict:
    g = torch.Generator(device="cuda").manual_seed(3)
    h, m = 4096, 11008
    sd = {}
    for i in range(layers):
        for name, shape in (("q", (h, h)), ("k", (h, h)), ("v", (h, h)), ("o", (h, h)), ("gate", (m, h)),
                            ("up", (m, h)), ("down", (h, m)), ("attn_norm", (h,)), ("mlp_norm", (h,))):
            sd[f"layers.{i}.{name}.weight"] = torch.randn(shape, generator=g, device="cuda") * 0.02
    sd["norm.weight"] = torch.ones(h, device="cuda")
    return sd


def events(fn, stream=None):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    out = fn()
    b.record(stream)
    b.synchronize()
    return a.elapsed_time(b), out


def summary(ms):
    return {"median_ms": round(statistics.median(ms), 3), "min_ms": round(min(ms), 3), "max_ms": round(max(ms), 3)}


def main():
    info = gpu_info()
    ctx = _backend.get_context()
    sd = llama_stack(LAYERS)
    f32_bytes = sum(t.numel() * 4 for t in sd.values())
    to_bf16 = lambda: {k: v.to(torch.bfloat16) for k, v in sd.items()}  # noqa: E731
    cast = DeviceFile.safetensors(sd, dtype=torch.bfloat16)
    pre_sd = to_bf16()
    pre = DeviceFile.safetensors(pre_sd)
    image = cast.nbytes
    assert image == pre.nbytes
    out = []

    # 1. hashing
    def hash_cast():
        return events(lambda: cast.hash_parts(BS, FLAGS), cast._src.stream)

    def hash_pre():
        return events(lambda: pre.hash_parts(BS, FLAGS), pre._src.stream)

    def hash_pre_with_to():
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        d = DeviceFile.safetensors(to_bf16())
        t = d.hash_parts(BS, FLAGS)
        b.record(torch.cuda.current_stream())
        b.synchronize()
        return a.elapsed_time(b), t

    for fn in (hash_cast, hash_pre, hash_pre_with_to):
        fn()
    times = {"cast": [], "pre": [], "pre_with_to": []}
    for _ in range(REPS):
        for k, fn in (("cast", hash_cast), ("pre", hash_pre), ("pre_with_to", hash_pre_with_to)):
            ms, table = fn()
            times[k].append(ms)
            if k == "cast":
                ref = table
            else:
                assert all(np.array_equal(x, y) for x, y in zip(ref, table) if x is not None), k
    med = {k: statistics.median(v) for k, v in times.items()}
    out.append({"arm": "1 hash", **{k: summary(v) for k, v in times.items()}, "image_bytes": image,
                "cast_over_pre": round(med["cast"] / med["pre"], 3),
                "cast_gbs": round(image / med["cast"] / 1e6, 2), "pre_gbs": round(image / med["pre"] / 1e6, 2),
                "outputs_equal": True, **info})

    # 2. staging every block
    _, _, trimmed = pre.hash_parts(BS, FLAGS)
    ranges = [(0, i * BS, int(t)) for i, t in enumerate(trimmed)]
    offsets, at = [], 0
    for _, _, n in ranges:
        offsets.append(at)
        at += -(-n // 16) * 16
    dst = ctx.host_alloc(at)
    staged_bytes = sum(n for _, _, n in ranges)
    try:
        def stage(f):
            return events(lambda: stage_ranges([f], ranges, dst, offsets).wait(), f._src.stream)[0]

        stage(cast), stage(pre)
        st = {"cast": [], "pre": []}
        for _ in range(REPS):
            st["cast"].append(stage(cast))
            got = dst.copy()
            st["pre"].append(stage(pre))
            assert np.array_equal(got, dst)
        med = {k: statistics.median(v) for k, v in st.items()}
        out.append({"arm": "2 stage", **{k: summary(v) for k, v in st.items()}, "staged_bytes": staged_bytes,
                    "cast_gbs": round(staged_bytes / med["cast"] / 1e6, 2),
                    "pre_gbs": round(staged_bytes / med["pre"] / 1e6, 2),
                    "cast_share_of_pre": round(med["pre"] / med["cast"], 3), "outputs_equal": True, **info})
    finally:
        ctx.host_free(dst)
    del pre, pre_sd

    # 3. end to end over loopback, with staging
    budget = 1 << 30

    def run(make):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        wall, released, blocks = asyncio.run(upload(make, budget))
        torch.cuda.synchronize()
        return wall, (torch.cuda.max_memory_allocated() - base) / 2**30, blocks

    routes = {"cast": lambda: DeviceFile.safetensors(sd, dtype=torch.bfloat16),
              "pre": lambda: DeviceFile.safetensors(to_bf16())}
    e2e = {k: {"s": [], "hbm_gib": []} for k in routes}
    blocks = {}
    for _ in range(3):
        for k, make in routes.items():
            wall, grew, got = run(make)
            e2e[k]["s"].append(wall)
            e2e[k]["hbm_gib"].append(grew)
            assert blocks.setdefault("ref", got) == got, k
    out.append({"arm": "3 upload", "reps": 3, "staging_bytes": budget,
                **{k: {"median_s": round(statistics.median(v["s"]), 3), "min_s": round(min(v["s"]), 3),
                       "max_s": round(max(v["s"]), 3), "peak_hbm_growth_gib": round(max(v["hbm_gib"]), 3)}
                   for k, v in e2e.items()}, "blocks_equal": True, **info})
    lines = [json.dumps({"f32_bytes": f32_bytes, "layers": LAYERS, "reps": REPS, **r}) for r in out]
    print("\n".join(lines))
    if os.environ.get("DCU_OUT"):
        os.makedirs(os.environ["DCU_OUT"], exist_ok=True)
        with open(os.path.join(os.environ["DCU_OUT"], "device_cast_upload_bench.json"), "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
