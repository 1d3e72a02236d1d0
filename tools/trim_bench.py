"""tools/trim_bench.py -- the zero-trim scan alone (trim_probe_kernel + trim_wide_kernel) on the shapes that matter:
  blank   1 280 x 8 MiB all-zero blocks (C4(ii)'s worst case: every byte must be read to prove the block is blank)
  half    1 280 x 8 MiB blocks, 3 MiB of data then zeros
  dense   1 280 x 8 MiB blocks of random bytes (the probe settles each one with a single 2 KiB step)
  tree    131 072 files, log-normal sizes (one rank's share of C3), random bytes
Times the TRIM_ZEROS | SHA256 batch and, separately, the hash of the trimmed lengths alone, so that
trim time = difference; prints achieved read bandwidth of the scan against the measured HBM peak.
Under ncu (--set full, -k regex:trim) the same script gives dram__bytes_read for the two kernels."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from modal_client_b200 import _lib

ctx = _lib.Context(0)
dev = torch.device("cuda:0")
st = torch.cuda.Stream()
torch.cuda.set_stream(st)
B = 8 << 20
NB = int(os.environ.get("TRIM_BLOCKS", 1280))
reps = int(os.environ.get("TRIM_REPS", 5))
PEAK = 3350.0  # GB/s, NVIDIA H100 SXM data sheet
try:
    PEAK = float(json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:
    pass
which = sys.argv[1:] or ["blank", "half", "dense", "tree"]


def timed(fn):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(reps):
        fn()
    e1.record(st)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def run(name, data, offs, lens):
    n = len(lens)
    d_off = torch.from_numpy(np.asarray(offs, np.int64)).to(dev)
    d_len = torch.from_numpy(np.asarray(lens, np.int64)).to(dev)
    sha = torch.empty((n, 32), dtype=torch.uint8, device=dev)
    tr = torch.empty(n, dtype=torch.int64, device=dev)
    flags = _lib.SHA256 | _lib.TRIM_ZEROS | _lib.NO_OUTLIERS
    both = timed(lambda: ctx.hash_batch_device(data.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), n, flags, sha.data_ptr(), 0,
                                               tr.data_ptr(), st.cuda_stream))
    trimmed = tr.cpu().numpy()
    hash_only = timed(lambda: ctx.hash_batch_device(data.data_ptr(), d_off.data_ptr(), tr.data_ptr(), n, _lib.SHA256 | _lib.NO_OUTLIERS,
                                                    sha.data_ptr(), 0, 0, st.cuda_stream))
    scanned = float((np.asarray(lens, np.float64) - trimmed).sum())  # bytes the scan had to read: the zero tails
    trim_ms = max(both - hash_only, 1e-6)
    print(json.dumps({"case": name, "messages": n, "bytes": int(np.asarray(lens, np.float64).sum()), "zero_tail_bytes": int(scanned),
                      "trim_plus_hash_ms": round(both, 4), "hash_only_ms": round(hash_only, 4), "trim_ms": round(trim_ms, 4),
                      "scan_GBps": round(scanned / 1e6 / trim_ms, 1), "scan_frac_of_hbm_peak": round(scanned / 1e6 / trim_ms / PEAK, 4),
                      "hbm_peak_GBps": PEAK}), flush=True)


total = NB * B
data = torch.empty(total + 64, dtype=torch.uint8, device=dev)
offs, lens = np.arange(NB) * B, np.full(NB, B)
if "blank" in which:
    data.zero_()
    torch.cuda.synchronize()
    run(f"blank: {NB} x 8 MiB all-zero blocks", data, offs, lens)
if "half" in which:
    ctx.fill_synth_device(data.data_ptr(), total, 7)
    v = data[:total].view(NB, B)
    v[:, 3 << 20 :] = 0
    v[:, (3 << 20) - 1] = 1
    torch.cuda.synchronize()
    run(f"half: {NB} x 8 MiB blocks, 3 MiB data + 5 MiB zeros", data, offs, lens)
if "dense" in which:
    ctx.fill_synth_device(data.data_ptr(), total, 8)
    data[:total].view(NB, B)[:, -1] = 1
    torch.cuda.synchronize()
    run(f"dense: {NB} x 8 MiB random blocks", data, offs, lens)
if "tree" in which:
    ctx.fill_synth_device(data.data_ptr(), total, 9)
    rng = np.random.default_rng(0)
    n = 131072
    sizes = np.clip(rng.lognormal(np.log(102400) - 1.5**2 / 2, 1.5, n), 1, 1 << 30)
    sizes = np.minimum(np.maximum(1, (sizes * (0.95 * total / sizes.sum())).astype(np.int64)), B)
    o = np.concatenate([[0], np.cumsum((sizes + 15) & ~15)])[:-1]
    run("tree: 131 072 log-normal files (blocks <= 8 MiB), random bytes", data, o, sizes)
ctx.close()
