"""tools/fp8_export_bench.py -- exporting a bf16 checkpoint in GPU memory as a block-scaled FP8 safetensors file:
``DeviceFile.safetensors(sd, fp8=names)``, which computes the scales with one call and quantizes on the device as blocks
are hashed and staged, against torch's ``per_block_cast_to_fp8`` per weight followed by ``DeviceFile.safetensors`` of
the quantized dict, which holds the FP8 weights (and, while it runs, F32 temporaries) in HBM.

The workload is a Llama-shaped bf16 stack (hidden 4096, MLP 11008, F8B_LAYERS layers, 10 by default: about 4 GiB);
every 2-D weight is quantized in 128 x 128 blocks, the norms stay bf16.  Arms, after one warm-up of each, alternating,
F8B_REPS (7) runs each, median and range:

  a  scales: one ``b200h_fp8_block_scales`` call for every weight against torch's per_block_cast_to_fp8 of every weight
     (which also quantizes), CUDA events on the current stream; the scales are compared bitwise
  b  hashing: the file's 8 MiB blocks, SHA-256 + TRIM_ZEROS (``hash_parts``), CUDA events, against hashing the
     pre-quantized file, and that route with its torch quantization included
  c  staging: ``stage_ranges`` of every block of the file into one page-locked buffer (``b200h_copy_scaled_ranges``)
     against the same of a float16 export of the stack (``b200h_copy_cast_ranges``), GB/s of source bytes and of image
     bytes
  d  end to end over loopback: the volumefs2 upload with device_staging_bytes = 1 GiB against an in-process fake
     server (device_put_bench.upload), host clock, with the peak growth of torch's HBM allocations from building the
     file to the end of the upload (the quantized copy counted for the pre-quantized route)

The outputs of the routes are compared bitwise in every arm.  The card name and power limit are read in the same run.
Needs a GPU: nothing here falls back.  One JSON line per arm; also written to $F8B_OUT/fp8_export_bench.json when set."""
import asyncio
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from device_cast_upload_bench import events, summary  # noqa: E402
from device_put_bench import upload  # noqa: E402
from modal_client_b200 import DeviceFile, _backend, _lib, blob_utils, stage_ranges  # noqa: E402
from safetensors_blocks_bench import gpu_info  # noqa: E402

LAYERS = int(os.environ.get("F8B_LAYERS", 10))
REPS = int(os.environ.get("F8B_REPS", 7))
BS = blob_utils.BLOCK_SIZE
FLAGS = _lib.SHA256 | _lib.TRIM_ZEROS
BLOCK = (128, 128)


def llama_stack(layers: int) -> dict:
    g = torch.Generator(device="cuda").manual_seed(3)
    h, m = 4096, 11008
    sd = {}
    for i in range(layers):
        for name, shape in (("q", (h, h)), ("k", (h, h)), ("v", (h, h)), ("o", (h, h)), ("gate", (m, h)),
                            ("up", (m, h)), ("down", (h, m)), ("attn_norm", (h,)), ("mlp_norm", (h,))):
            sd[f"layers.{i}.{name}.weight"] = (torch.randn(shape, generator=g, device="cuda") * 0.02).to(torch.bfloat16)
    sd["norm.weight"] = torch.ones(h, device="cuda", dtype=torch.bfloat16)
    return sd


def per_block_cast_to_fp8(w):
    """The widely copied form (DeepGEMM's tests): q and the F32 scale of every 128 x 128 block."""
    R, C = w.shape
    gR, gC = -(-R // BLOCK[0]), -(-C // BLOCK[1])
    padded = w.new_zeros(gR * BLOCK[0], gC * BLOCK[1])
    padded[:R, :C] = w
    v = padded.view(gR, BLOCK[0], gC, BLOCK[1])
    amax = v.abs().float().amax(dim=(1, 3), keepdim=True).clamp(1e-4)
    q = (v * (448.0 / amax)).to(torch.float8_e4m3fn).view(gR * BLOCK[0], gC * BLOCK[1])[:R, :C].contiguous()
    return q, (amax / 448.0).view(gR, gC)


def main():
    info = gpu_info()
    ctx = _backend.get_context()
    sd = llama_stack(LAYERS)
    names = [n for n, t in sd.items() if t.dim() == 2]
    src_bytes = sum(t.numel() * 2 for t in sd.values())

    def quantized():
        out = {}
        for n, t in sd.items():
            if n in names:
                out[n], out[n + "_scale_inv"] = per_block_cast_to_fp8(t)
            else:
                out[n] = t
        return out

    f = DeviceFile.safetensors(sd, fp8=names)
    pre_sd = quantized()
    pre = DeviceFile.safetensors(pre_sd)
    image = f.nbytes
    assert image == pre.nbytes
    out = []

    # a. scales
    def scales_ours():
        return events(lambda: DeviceFile._fp8_scales(sd, {n: n + "_scale_inv" for n in names}, BLOCK, ctx))

    def scales_torch():
        return events(lambda: {n: per_block_cast_to_fp8(sd[n])[1] for n in names})

    scales_ours(), scales_torch()
    times = {"ours": [], "torch": []}
    for _ in range(REPS):
        ms, (got, _) = scales_ours()
        times["ours"].append(ms)
        ms, want = scales_torch()
        times["torch"].append(ms)
        assert all(torch.equal(got[n][0].view(torch.int32), want[n].view(torch.int32)) for n in names)
    med = {k: statistics.median(v) for k, v in times.items()}
    out.append({"arm": "a scales", **{k: summary(v) for k, v in times.items()}, "weights": len(names),
                "source_bytes": src_bytes, "ours_gbs": round(src_bytes / med["ours"] / 1e6, 2),
                "torch_over_ours": round(med["torch"] / med["ours"], 2), "outputs_equal": True, **info})

    # b. hashing
    def hash_fp8():
        return events(lambda: f.hash_parts(BS, FLAGS), f._src.stream)

    def hash_pre():
        return events(lambda: pre.hash_parts(BS, FLAGS), pre._src.stream)

    def hash_pre_with_quantization():
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        d = DeviceFile.safetensors(quantized())
        t = d.hash_parts(BS, FLAGS)
        b.record(torch.cuda.current_stream())
        b.synchronize()
        return a.elapsed_time(b), t

    for fn in (hash_fp8, hash_pre, hash_pre_with_quantization):
        fn()
    times = {"fp8": [], "pre": [], "pre_with_quantization": []}
    for _ in range(REPS):
        for k, fn in (("fp8", hash_fp8), ("pre", hash_pre), ("pre_with_quantization", hash_pre_with_quantization)):
            ms, table = fn()
            times[k].append(ms)
            if k == "fp8":
                ref = table
            else:
                assert all(np.array_equal(x, y) for x, y in zip(ref, table) if x is not None), k
    med = {k: statistics.median(v) for k, v in times.items()}
    out.append({"arm": "b hash", **{k: summary(v) for k, v in times.items()}, "image_bytes": image,
                "fp8_over_pre": round(med["fp8"] / med["pre"], 3),
                "fp8_over_pre_with_quantization": round(med["fp8"] / med["pre_with_quantization"], 3),
                "fp8_image_gbs": round(image / med["fp8"] / 1e6, 2), "outputs_equal": True, **info})

    # c. staging every block, against a converting (bf16 -> f16) export of the same stack
    half = DeviceFile.safetensors(sd, dtype=torch.float16)
    rates = {}
    st = {"fp8": [], "cast_f16": []}
    plans = {}
    for k, d in (("fp8", f), ("cast_f16", half)):
        _, _, trimmed = d.hash_parts(BS, FLAGS)
        ranges = [(0, i * BS, int(t)) for i, t in enumerate(trimmed)]
        offsets, at = [], 0
        for _, _, n in ranges:
            offsets.append(at)
            at += -(-n // 16) * 16
        plans[k] = (d, ranges, offsets, at)
    dst = ctx.host_alloc(max(p[3] for p in plans.values()))
    try:
        def stage(k):
            d, ranges, offsets, _ = plans[k]
            return events(lambda: stage_ranges([d], ranges, dst, offsets).wait(), d._src.stream)[0]

        stage("fp8"), stage("cast_f16")
        for _ in range(REPS):
            for k in st:
                st[k].append(stage(k))
        for k in st:
            n = sum(x for _, _, x in plans[k][1])
            rates[k] = {"image_gbs": round(n / statistics.median(st[k]) / 1e6, 2),
                        "source_gbs": round(src_bytes / statistics.median(st[k]) / 1e6, 2)}
        _, ranges, offsets, used = plans["fp8"]  # the pre-quantized file has the same blocks
        stage_ranges([pre], ranges, dst, offsets).wait()
        ref = dst[:used].copy()
        stage("fp8")
        assert np.array_equal(ref, dst[:used])
    finally:
        ctx.host_free(dst)
    out.append({"arm": "c stage", **{k: summary(v) for k, v in st.items()}, **rates, "outputs_equal": True, **info})
    del pre, pre_sd, half

    # d. end to end over loopback, with staging
    budget = 1 << 30

    def run(make):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        wall, released, blocks = asyncio.run(upload(make, budget))
        torch.cuda.synchronize()
        return wall, (torch.cuda.max_memory_allocated() - base) / 2**30, blocks

    routes = {"fp8": lambda: DeviceFile.safetensors(sd, fp8=names),
              "pre": lambda: DeviceFile.safetensors(quantized())}
    e2e = {k: {"s": [], "hbm_gib": []} for k in routes}
    blocks = {}
    for _ in range(3):
        for k, make in routes.items():
            wall, grew, got = run(make)
            e2e[k]["s"].append(wall)
            e2e[k]["hbm_gib"].append(grew)
            assert blocks.setdefault("ref", got) == got, k
    out.append({"arm": "d upload", "reps": 3, "staging_bytes": budget,
                **{k: {"median_s": round(statistics.median(v["s"]), 3), "min_s": round(min(v["s"]), 3),
                       "max_s": round(max(v["s"]), 3), "peak_hbm_growth_gib": round(max(v["hbm_gib"]), 3)}
                   for k, v in e2e.items()}, "blocks_equal": True, **info})
    lines = [json.dumps({"bf16_bytes": src_bytes, "layers": LAYERS, "reps": REPS, **r}) for r in out]
    print("\n".join(lines))
    if os.environ.get("F8B_OUT"):
        os.makedirs(os.environ["F8B_OUT"], exist_ok=True)
        with open(os.path.join(os.environ["F8B_OUT"], "fp8_export_bench.json"), "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
