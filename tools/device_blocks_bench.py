"""tools/device_blocks_bench.py -- volumefs2 block hashing (8 MiB blocks, zero trim + SHA-256) of one large CUDA tensor:

  device   DeviceFile(t).hash_parts(BLOCK_SIZE, SHA256 | TRIM_ZEROS): one b200h_hash_segment_parts_device call (one
           segment, every block in place) where the tensor lives; only the (trimmed length, SHA-256) table comes to
           the host
  host     what a caller had to do before DeviceFile: t.cpu(), then the blocks of that host image the way
           FileUploadSpec2.from_fileobj builds them (b200h_hash_fixed_parts, which stages the bytes back to the GPU)

The two routes alternate, REPS times each, on the same tensor (default 4 GiB: DEVBLK_GIB).  Both are timed on the host
clock from the call to the block table being on the host, which ends in a synchronisation; the device route is also
timed with CUDA events on its stream.  The block tables of the two routes are compared.  One JSON line per route with
the card name and power limit read in the same run; also written to $DEVBLK_OUT/device_blocks_bench.json when set."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from modal_client_b200 import DeviceFile, _backend, _lib, blob_utils

GIB = int(os.environ.get("DEVBLK_GIB", 4))
REPS = int(os.environ.get("DEVBLK_REPS", 5))
BS = blob_utils.BLOCK_SIZE
FLAGS = _lib.SHA256 | _lib.TRIM_ZEROS


def gpu_info() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in (q.stdout.strip().split(",") + ["?", "?", "?"])[:3])
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock, "torch_device": torch.cuda.get_device_name(0)}


def main():
    ctx = _lib.Context(0)
    _backend.set_context(ctx)
    n = GIB << 30
    t = torch.empty(n, dtype=torch.uint8, device="cuda:0")
    ctx.fill_synth_device(t.data_ptr(), n, seed=2024)
    torch.cuda.synchronize()
    for i in range(n // BS):  # a checkpoint-like mix: zero tails of every length, some all-zero blocks
        tail = [0, 0, 0, 4096, BS // 3, BS - 1, BS, 17][i % 8]
        if tail:
            t[(i + 1) * BS - tail : (i + 1) * BS] = 0
    torch.cuda.synchronize()
    f = DeviceFile(t)

    def device_route():
        sha, _, trimmed = f.hash_parts(BS, FLAGS)
        return sha, trimmed

    def host_route():
        view = t.cpu().numpy()
        sha, _, trimmed, _ = ctx.hash_fixed_parts(view, BS, FLAGS)
        return sha, trimmed

    # warm-up of both shapes, and the same block table from both routes
    ds, dt = device_route()
    hs, ht = host_route()
    assert np.array_equal(ds, hs) and np.array_equal(dt, ht), "device and host block tables differ"
    wall = {"device": [], "host": []}
    dev_ms = []
    stream = f._src.stream
    for _ in range(REPS):
        for route, fn in (("device", device_route), ("host", host_route)):
            if route == "device":
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
            t0 = time.perf_counter()
            fn()
            wall[route].append(time.perf_counter() - t0)
            if route == "device":
                e1.record(stream)
                e1.synchronize()
                dev_ms.append(e0.elapsed_time(e1))
    info = gpu_info()
    lines = []
    for route in ("device", "host"):
        w = sorted(wall[route])
        rec = {"tool": "device_blocks_bench", "route": route, "bytes": n, "blocks": n // BS, "reps": REPS,
               "wall_s_median": w[len(w) // 2], "wall_s_min": w[0], "wall_s_max": w[-1],
               "wall_gbs_median": n / w[len(w) // 2] / 1e9, **info}
        if route == "device":
            d = sorted(dev_ms)
            rec.update({"device_ms_median": d[len(d) // 2], "device_ms_min": d[0], "device_ms_max": d[-1],
                        "device_gbs_median": n / (d[len(d) // 2] / 1e3) / 1e9})
        lines.append(json.dumps(rec))
    out = os.environ.get("DEVBLK_OUT")
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "device_blocks_bench.json"), "w") as fh:
            fh.write("\n".join(lines) + "\n")
    print("\n".join(lines))
    ctx.close()


if __name__ == "__main__":
    main()
