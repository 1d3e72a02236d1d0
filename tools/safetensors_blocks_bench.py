"""tools/safetensors_blocks_bench.py -- volumefs2 block tables (8 MiB blocks, zero trim + SHA-256) of a state dict that
lives in GPU memory, uploaded as one safetensors file or as one file per tensor.

A seeded bf16 state dict of about 4 GiB in about 300 tensors (8 KiB norms to 256 MiB matrices; STB_GIB sets the size),
filled with fill_synth_device, some with zero tails.  Arms, alternating, STB_REPS (5) runs each, host clock from the
call to the block table on the host (every arm ends in a synchronisation):

  a  segmented     DeviceFile.safetensors(sd) -> FileUploadSpec2 blocks: ONE b200h_hash_segment_parts_device call;
                   the blocks that straddle tensors are gathered into a wave slot, the others hashed in place
  a0 aligned       the same image bytes in one 16-byte-aligned buffer -> DeviceFile(buf) blocks (the same entry with one
                   segment): a against a0 is the cost of in-place parts that start unaligned plus the gather
  b  cat           torch.cat of the header and every tensor's bytes into one buffer -> DeviceFile(buf) blocks
  c  host          safetensors.torch.save on the host -> FileUploadSpec2.from_fileobj(BytesIO)
  d1 files/call    the tensors as separate files in one v2 batch, one library call per file (from_fileobj each)
  d2 files/batch   the same files, one library call for all (blob_utils.device_file_specs2)

Per arm: median / min / max seconds, the peak extra HBM PyTorch saw (max_memory_allocated delta; the library's wave
slots are its own cudaMalloc and are reported apart), the gathered parts and waves, and whether its block table equals
arm c's (a / a0 / b / c) or the per-file tables (d1 / d2).  The card name and power limit are read in the same run.
One JSON line per arm; also written to $STB_OUT/safetensors_blocks_bench.json when set."""
import asyncio
import json
import os
import random
import subprocess
import sys
import time
from io import BytesIO
from pathlib import PurePosixPath

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from safetensors.torch import save

from modal_client_b200 import DeviceFile, _backend, _lib, blob_utils, device_file

GIB = float(os.environ.get("STB_GIB", 4))
REPS = int(os.environ.get("STB_REPS", 5))
BS = blob_utils.BLOCK_SIZE
FLAGS = _lib.SHA256 | _lib.TRIM_ZEROS


def gpu_info() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in (q.stdout.strip().split(",") + ["?", "?", "?"])[:3])
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock, "torch_device": torch.cuda.get_device_name(0)}


def state_dict(ctx, total: int) -> dict:
    """Up to ~total bytes of bf16 tensors: per layer two norms and three biases of about 8 KiB, four attention and
    three MLP matrices, then a 256 MiB embedding and a final norm: about 300 tensors from 8 KiB to 256 MiB."""
    rng = random.Random(7)
    sizes = []
    layer = 0
    while sum(n for _, n in sizes) < total - (256 << 20) and len(sizes) < 288:
        for kind, n in (("input_norm", 8 << 10), ("post_norm", 8 << 10), ("q_bias", 8 << 10), ("k_bias", 8 << 10),
                        ("v_bias", 8 << 10), ("q", 16 << 20), ("k", 4 << 20), ("v", 4 << 20), ("o", 16 << 20),
                        ("gate", 36 << 20), ("up", 36 << 20), ("down", 36 << 20)):
            sizes.append((f"model.layers.{layer}.{kind}.weight", n + 2 * rng.randrange(0, 1000)))
        layer += 1
    sizes.append(("model.embed_tokens.weight", max(8 << 10, min(256 << 20, total - sum(n for _, n in sizes)))))
    sizes.append(("model.norm.weight", 8 << 10))
    sd = {}
    for i, (name, n) in enumerate(sizes):
        t = torch.empty(n // 2, dtype=torch.bfloat16, device="cuda:0")
        ctx.fill_synth_device(t.data_ptr(), n // 8 * 8, seed=1000 + i)
        if i % 4 == 0:
            t.view(torch.uint8)[n - rng.randrange(2, n // 2) :] = 0
        sd[name] = t
    torch.cuda.synchronize()
    return sd


def blocks(fp) -> list:
    spec = asyncio.run(blob_utils.FileUploadSpec2.from_fileobj(fp, PurePosixPath("/ckpt/model.safetensors"),
                                                               asyncio.Semaphore(1), 0o644))
    return [(b.start, b.end, b.contents_sha256) for b in spec.blocks]


def main():
    ctx = _lib.Context(0)
    _backend.set_context(ctx)
    sd = state_dict(ctx, int(GIB * (1 << 30)))
    header, ordered = device_file.safetensors_layout(sd)
    seg_lens = [len(header)] + [t.numel() * t.element_size() for _, t in ordered]
    nbytes = sum(seg_lens)
    seg, wave, nwaves = _lib.segment_parts_preview(seg_lens, [0, len(seg_lens)], BS, 4 << 30)
    gathered = int((seg == _lib.GATHERED).sum())
    aligned = torch.empty(nbytes, dtype=torch.uint8, device="cuda:0")
    aligned[: len(header)] = torch.frombuffer(bytearray(header), dtype=torch.uint8).cuda()
    at = len(header)
    for _, t in ordered:
        n = t.numel() * t.element_size()
        aligned[at : at + n] = t.reshape(-1).view(torch.uint8)
        at += n
    torch.cuda.synchronize()
    names = list(sd)
    items = lambda: [(DeviceFile(sd[k]), PurePosixPath(f"/ckpt/{k}"), 0o644) for k in names]  # noqa: E731

    def arm_a():
        return blocks(DeviceFile.safetensors(sd))

    def arm_a0():
        return blocks(DeviceFile(aligned))

    def arm_b():
        head = torch.frombuffer(bytearray(header), dtype=torch.uint8).cuda()
        buf = torch.cat([head] + [t.reshape(-1).view(torch.uint8) for _, t in ordered])
        return blocks(DeviceFile(buf))

    def arm_c():
        return blocks(BytesIO(save({k: v.cpu() for k, v in sd.items()})))

    def arm_d1():
        sem = asyncio.Semaphore(1)
        return [[(b.start, b.end, b.contents_sha256) for b in
                 asyncio.run(blob_utils.FileUploadSpec2.from_fileobj(f, p, sem, m)).blocks] for f, p, m in items()]

    def arm_d2():
        return [[(b.start, b.end, b.contents_sha256) for b in s.blocks]
                for s in asyncio.run(blob_utils.device_file_specs2(items()))]

    arms = {"a": arm_a, "a0": arm_a0, "b": arm_b, "c": arm_c, "d1": arm_d1, "d2": arm_d2}
    tables = {k: fn() for k, fn in arms.items()}  # warm-up of every shape, and the tables compared
    same = {k: tables[k] == (tables["c"] if k in ("a", "a0", "b", "c") else tables["d1"]) for k in arms}
    wall = {k: [] for k in arms}
    hbm = {k: 0 for k in arms}
    for _ in range(REPS):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            t0 = time.perf_counter()
            fn()
            wall[k].append(time.perf_counter() - t0)
            hbm[k] = max(hbm[k], torch.cuda.max_memory_allocated() - base)
    info = gpu_info()
    lines = []
    for k in arms:
        w = sorted(wall[k])
        rec = {"tool": "safetensors_blocks_bench", "arm": k, "bytes": nbytes, "tensors": len(sd), "blocks": seg.size,
               "reps": REPS, "wall_s_median": w[len(w) // 2], "wall_s_min": w[0], "wall_s_max": w[-1],
               "peak_extra_hbm_torch_bytes": hbm[k], "table_equal": same[k], **info}
        if k == "a":
            rec.update({"gathered_parts": gathered, "waves": nwaves,
                        "staged_bytes": int(sum((min(BS, nbytes - i * BS) + 15) // 16 * 16
                                                for i in range(seg.size) if seg[i] == _lib.GATHERED))})
        lines.append(json.dumps(rec))
    out = os.environ.get("STB_OUT")
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "safetensors_blocks_bench.json"), "w") as fh:
            fh.write("\n".join(lines) + "\n")
    print("\n".join(lines))
    ctx.close()


if __name__ == "__main__":
    main()
