"""tools/lane_ab.py -- same-call A/B of lane-kernel builds: kbench.py (per digest set) and bench.py, alternating.

usage: python tools/lane_ab.py --variant NAME=SPEC [--variant NAME=SPEC ...] [--kbench-runs 5] [--bench-runs 3] [--flags 3,1,2]
                               [--build-dir DIR] [--build-only] [--json FILE]

A SPEC is either a path to a built libb200hash.so (e.g. a build of another commit) or a list of -D defines (possibly
empty) that the library is built with from this tree's sources, e.g. `head=` and `parent=/tmp/parent/libb200hash.so`,
or `trial=-DTRIAL_FORM` for a form under study put behind an `#if` in the source.
Every build goes to --build-dir (default: a temporary directory), never into the tree, and is loaded through B200H_LIB.
Rounds alternate the variants (the order flips every round, so a drift of the card's clock over the call does not
favour one of them).  Each result line gives the median and min-max next to the card's name, power limit, median SM
clock and the throttle reasons seen while that measurement ran.  The first bench.py run of every variant dumps its
digest table; the tables must be byte-identical across variants.
"""
from __future__ import annotations

import argparse
import json
import os
import shlex
import statistics
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "modal_client_b200", "csrc")
SRCS = ["b200hash_kernels.cu", "b200hash_dedupe.cu", "b200hash_crc32.cu", "b200hash_stage.cu", "b200hash_api.cu",
        "b200blob_host.cpp", "b200pack_copy.cpp"]  # the sources of modal_client_b200/csrc/Makefile
NVFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC,-Wall,-mavx2",
           "-Xptxas", "-v"]  # the flags of modal_client_b200/csrc/Makefile
FLAG_NAMES = {3: "sha256+md5", 1: "sha256", 2: "md5"}


def build(name: str, spec: str, build_dir: str) -> str:
    if spec.endswith(".so"):
        return os.path.abspath(spec)
    out_dir = os.path.join(build_dir, name)
    os.makedirs(out_dir, exist_ok=True)
    out = os.path.join(out_dir, "libb200hash.so")
    cmd = [os.environ.get("NVCC", "nvcc")] + NVFLAGS + shlex.split(spec) + ["-shared", "-o", out] + SRCS + ["-lpthread", "-ldl"]
    r = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    with open(os.path.join(out_dir, "build.log"), "w") as f:
        f.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
    if r.returncode:
        raise SystemExit(f"building {name} ({spec!r}) failed:\n{r.stderr[-4000:]}")
    return out


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True)
    name, _, plim = q.stdout.strip().partition(",")
    return {"card": name.strip() or None, "power_limit_w": plim.strip() or None}


def run_sampled(cmd: list, env: dict) -> tuple[str, dict]:
    """Run one measurement while nvidia-smi samples the SM clock and throttle reasons every 200 ms."""
    from bench import ClockSampler

    sampler = ClockSampler(0)
    sampler.start()
    try:
        r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True)
    finally:
        rows = sampler.halt()
    clocks = ClockSampler.summarize(rows, sampler.proc is not None)
    # the process spends most of its time importing torch and filling the input at idle clocks: the busy clock is
    # the median over the samples taken while the card drew more than half its peak draw of this run
    busy = []
    for row in rows:
        try:
            busy.append((float(row[3]), float(row[1])))
        except (IndexError, ValueError):
            continue
    peak = max((w for w, _ in busy), default=0.0)
    clocks["sm_mhz"] = statistics.median([mhz for w, mhz in busy if w > peak / 2]) if busy else None
    if r.returncode:
        raise SystemExit(f"{' '.join(cmd)} failed ({r.returncode}):\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}")
    return r.stdout, clocks


def kbench(lib: str, flags: int) -> tuple[float, dict]:
    out, clocks = run_sampled([sys.executable, "tools/kbench.py", "100000", "262144", "5", str(flags)],
                              dict(os.environ, B200H_LIB=lib))
    line = [ln for ln in out.splitlines() if "lane kernel" in ln][-1]
    return float(line.split("lane kernel")[1].split("ms")[0]), clocks


def bench(lib: str, dump: str | None) -> tuple[dict, dict]:
    cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", "5", "--warmup", "3"]
    if dump:
        cmd += ["--dump-outputs", dump]
    out, clocks = run_sampled(cmd, dict(os.environ, B200H_LIB=lib))
    return json.loads([ln for ln in out.splitlines() if ln.startswith("{")][-1]), clocks


def summary(xs: list) -> str:
    return f"median {statistics.median(xs):.3f} (min {min(xs):.3f}, max {max(xs):.3f}, n={len(xs)})"


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--variant", action="append", metavar="NAME=SPEC", required=True)
    ap.add_argument("--kbench-runs", type=int, default=5)
    ap.add_argument("--bench-runs", type=int, default=3)
    ap.add_argument("--flags", default="3,1,2", help="kbench digest sets: 3=sha256+md5, 1=sha256, 2=md5")
    ap.add_argument("--build-dir", default=None)
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--json", default=None, help="also write every sample to this file")
    args = ap.parse_args()
    variants = dict(v.split("=", 1) for v in args.variant)
    build_dir = os.path.abspath(args.build_dir or tempfile.mkdtemp(prefix="lane_ab_"))
    with ThreadPoolExecutor(max_workers=len(variants)) as ex:
        libs = dict(zip(variants, ex.map(lambda kv: build(kv[0], kv[1], build_dir), variants.items())))
    for name, lib in libs.items():
        print(f"{name}: {variants[name]!r} -> {lib}", flush=True)
    if args.build_only:
        return
    sys.path.insert(0, ROOT)
    flags = [int(f) for f in args.flags.split(",") if f]
    dump_root = tempfile.mkdtemp(prefix="lane_ab_dump_")
    samples: dict = {name: {"kbench": {f: [] for f in flags}, "bench": []} for name in libs}
    names = list(libs)
    for rnd in range(max(args.kbench_runs, args.bench_runs)):
        for name in (names if rnd % 2 == 0 else names[::-1]):
            lib, c = libs[name], card()
            if rnd < args.kbench_runs:
                for f in flags:
                    ms, clocks = kbench(lib, f)
                    samples[name]["kbench"][f].append(ms)
                    print(f"round {rnd} {name:>12} kbench {FLAG_NAMES[f]:>10}: lane kernel {ms:.3f} ms | {c['card']}, "
                          f"{c['power_limit_w']} W limit, SM {clocks.get('sm_mhz')} MHz, reasons {clocks.get('reasons')}",
                          flush=True)
            if rnd < args.bench_runs:
                res, clocks = bench(lib, os.path.join(dump_root, name) if rnd == 0 else None)
                samples[name]["bench"].append(res)
                print(f"round {rnd} {name:>12} bench.py: value {res['value']} GiB/s, kernel "
                      f"{res['roofline']['kernel_avg_ms']} ms, launches {res['gpu_launches']}, host syncs "
                      f"{res['config']['host_syncs_in_timed_region']}, parity: {res['parity']} | {c['card']}, "
                      f"{c['power_limit_w']} W limit, SM {clocks.get('sm_mhz')} MHz, reasons {clocks.get('reasons')}",
                      flush=True)
    c = card()
    print(f"\n== summary ({c['card']}, power limit {c['power_limit_w']} W)")
    for name in names:
        for f in flags:
            xs = samples[name]["kbench"][f]
            if xs:
                print(f"{name:>12} kbench {FLAG_NAMES[f]:>10} lane kernel ms: {summary(xs)}")
        vals = [r["value"] for r in samples[name]["bench"]]
        if vals:
            print(f"{name:>12} bench.py value GiB/s: {summary(vals)}")
    if args.bench_runs:
        import numpy as np

        ref = names[0]
        for name in names[1:]:
            same = all(np.array_equal(np.load(os.path.join(dump_root, ref, fn)), np.load(os.path.join(dump_root, name, fn)))
                       for fn in ("sha256.npy", "md5.npy"))
            print(f"digest tables {ref} vs {name}: {'identical' if same else 'DIFFERENT'}")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"card": c, "variants": variants, "samples": samples}, fh, indent=1)


if __name__ == "__main__":
    main()
