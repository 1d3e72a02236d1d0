"""tools/j1_table.py -- merge the JSON lines of tools/j1_matrix.py (one file per GPU count) into the markdown table the
round-2 review asked for: per configuration GPU kernel GiB/s, GPU e2e GiB/s, fraction of the HBM roofline per GPU, the
reference's CPU path beside it.    python tools/j1_table.py j1_n1.jsonl j1_n2.jsonl ..."""
import json
import sys
from collections import OrderedDict


def short(cfg: str) -> str:
    return cfg.split(" (")[0] if cfg.startswith("C5") else cfg


gpu = OrderedDict()  # config -> {n_gpus: row}
cpu = OrderedDict()  # config -> row
for path in sys.argv[1:]:
    for line in open(path):
        line = line.strip()
        if not line.startswith("{"):
            continue
        r = json.loads(line)
        key = short(r["config"])
        if r.get("side") == "cpu":
            cpu[key] = r
        else:
            gpu.setdefault(key, {})[r["n_gpus"]] = r


def cpu_cell(r):
    if r is None:
        return "—"
    parts = []
    for k, v in r.items():
        if k == "single_thread_GiBps":
            parts.append(f"1 thread {v}")
        elif k.startswith("pool_default_"):
            parts.append(f"pool({k.split('_')[2]}) {v}")
        elif k.startswith("pool_ncpu_"):
            parts.append(f"pool({k.split('_')[2]}) {v}")
        elif k == "GiBps":
            parts.append(f"{v}")
        elif k == "first_2GiB_GiBps":
            parts.append(f"(first 2 GiB: {v})")
    eq = r.get("digests_equal_gpu")
    return "; ".join(parts) + (" ✓" if eq else (" ✗" if eq is False else ""))


ns = sorted({n for rows in gpu.values() for n in rows})
print("| config | " + " | ".join(f"{n} GPU kernel GiB/s (HBM frac/GPU) · e2e GiB/s" for n in ns) + " | reference CPU path, GiB/s |")
print("|---|" + "---|" * (len(ns) + 1))
for key, rows in gpu.items():
    cells = []
    for n in ns:
        r = rows.get(n)
        if r is None:
            cells.append("—")
            continue
        e2e = r.get("e2e_GiBps")
        e2e_s = "—" if e2e is None else f"{e2e}"
        if e2e is not None and r.get("e2e_bytes") and r["e2e_bytes"] < 0.99 * r["bytes_total"]:
            e2e_s += f" (on {r['e2e_bytes'] / 2**30:.1f} GiB)"
        cells.append(f"**{r['kernel_GiBps']}** ({r['hbm_frac_per_gpu']}) · {e2e_s}")
    print(f"| {key} | " + " | ".join(cells) + f" | {cpu_cell(cpu.get(key))} |")
print()
host = next((r.get("host") for r in cpu.values() if r.get("host")), None)
if host:
    print(f"CPU host: {host['logical_cpus']} logical CPUs, {host['cpu_model']}, sha_ni={host['sha_ni']}, {host['openssl']}.")
for key, r in cpu.items():
    print(f"- CPU `{key}`: {r['what']}; sample {r.get('sample', '')} ({r['sample_bytes'] / 2**30:.2f} GiB)"
          + (f"; one thread on {r['single_thread_sample_bytes'] / 2**30:.2f} GiB" if 'single_thread_sample_bytes' in r else ""))
for key, rows in gpu.items():
    r = rows[max(rows)]
    if "largest_file" in r:
        print(f"- GPU `{key}`: largest file {r['largest_file']} B; per-rank hash makespan (ms, before the gather) at {max(rows)} GPUs: {r.get('per_rank_hash_ms', r['per_rank_ms'])}; "
              f"messages on the chain kernel (rank 0): {r['outliers_on_rank0']}")
