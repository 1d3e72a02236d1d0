"""tools/torch_save_blocks_bench.py -- volumefs2 block tables (8 MiB blocks, zero trim + SHA-256) of a state dict that
lives in GPU memory, uploaded as one torch.save file, and the CRC-32 kernel that makes that possible.

The state dict is tools/safetensors_blocks_bench.py's: seeded bf16, about 4 GiB in about 300 tensors (TSB_GIB sets
the size).  Arms, alternating, TSB_REPS (5) runs each, host clock from the call to the block table on the host (every
arm ends in a synchronisation):

  a  torch_save    DeviceFile.torch_save(sd) -> FileUploadSpec2 blocks: one b200h_crc32_device call over every
                   storage (plus one for the serialization id), then one b200h_hash_segment_parts_device call
  c  host          torch.save to BytesIO on the host -> FileUploadSpec2.from_fileobj(BytesIO)
  s  safetensors   DeviceFile.safetensors(sd) -> blocks, for comparison

Per arm: median / min / max seconds, the peak extra HBM PyTorch saw, and whether the table equals arm c's (a)
or the table of the safetensors image hashed on the host (s).  Then the CRC launch alone: b200h_crc32_device over
every storage, CUDA events around TSB_CRC_REPS (20) back-to-back launches after a warm-up; bytes CRC'd per second
and that as a share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).  The card name and power limit are read
in the same run.  One JSON line per arm and one for the kernel; also written to $TSB_OUT/torch_save_blocks_bench.json
when set."""
import asyncio
import json
import os
import sys
import time
from io import BytesIO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch
from safetensors.torch import save as st_save

from modal_client_b200 import DeviceFile, _backend, _lib
from safetensors_blocks_bench import blocks, gpu_info, state_dict

GIB = float(os.environ.get("TSB_GIB", 4))
REPS = int(os.environ.get("TSB_REPS", 5))
CRC_REPS = int(os.environ.get("TSB_CRC_REPS", 20))
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def main():
    ctx = _lib.Context(0)
    _backend.set_context(ctx)
    sd = state_dict(ctx, int(GIB * (1 << 30)))
    nbytes = sum(t.numel() * t.element_size() for t in sd.values())

    def arm_a():
        return blocks(DeviceFile.torch_save(sd))

    def arm_c():
        buf = BytesIO()
        torch.save(sd, buf)
        return blocks(BytesIO(buf.getvalue()))

    def arm_s():
        return blocks(DeviceFile.safetensors(sd))

    arms = {"a": arm_a, "c": arm_c, "s": arm_s}
    tables = {k: fn() for k, fn in arms.items()}  # warm-up of every shape, and the tables compared
    st_host = blocks(BytesIO(st_save({k: v.cpu() for k, v in sd.items()})))
    same = {"a": tables["a"] == tables["c"], "c": True, "s": tables["s"] == st_host}
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

    # the CRC launch alone: every storage of the state dict, as DeviceFile.torch_save passes them
    ptrs = [t.untyped_storage().data_ptr() for t in sd.values()]
    lens = [t.untyped_storage().nbytes() for t in sd.values()]
    out = torch.empty(len(lens), dtype=torch.int32, device="cuda:0")
    stream = torch.cuda.current_stream().cuda_stream or 1  # 1: cudaStreamLegacy (NULL would be the library's stream)
    for _ in range(3):
        ctx.crc32_device(ptrs, lens, out.data_ptr(), stream)
    launches = ctx.launch_count
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(CRC_REPS):
        ctx.crc32_device(ptrs, lens, out.data_ptr(), stream)
    e1.record()
    e1.synchronize()
    per_call = e0.elapsed_time(e1) / 1e3 / CRC_REPS
    info = gpu_info()
    lines = []
    for k in arms:
        w = sorted(wall[k])
        lines.append(json.dumps({"tool": "torch_save_blocks_bench", "arm": k, "bytes": nbytes, "tensors": len(sd),
                                 "blocks": len(tables[k]), "reps": REPS, "wall_s_median": w[len(w) // 2],
                                 "wall_s_min": w[0], "wall_s_max": w[-1], "peak_extra_hbm_torch_bytes": hbm[k],
                                 "table_equal": same[k], **info}))
    lines.append(json.dumps({"tool": "torch_save_blocks_bench", "arm": "crc32_kernel", "bytes": sum(lens),
                             "ranges": len(lens), "launches_per_call": (ctx.launch_count - launches) / CRC_REPS,
                             "reps": CRC_REPS, "s_per_call": per_call, "bytes_per_s": sum(lens) / per_call,
                             "share_of_hbm_datasheet": sum(lens) / per_call / HBM_BYTES_PER_S, **info}))
    out_dir = os.environ.get("TSB_OUT")
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "torch_save_blocks_bench.json"), "w") as fh:
            fh.write("\n".join(lines) + "\n")
    print("\n".join(lines))
    ctx.close()


if __name__ == "__main__":
    main()
