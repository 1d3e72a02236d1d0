"""tools/lane_sass_score.py -- rank equivalent forms of the dense fused lane kernel's block body from their SASS (CPU only).

usage: python tools/lane_sass_score.py --variant NAME=SPEC [--variant NAME=SPEC ...] [--build-dir DIR] [--jobs 4]
                                      [--json FILE]

A SPEC is what tools/lane_ab.py takes: a path to a built libb200hash.so (e.g. a build of another commit, or of this tree
with the form under study edited in) or a list of -D defines (possibly empty) built from this tree's sources with
lane_ab.py's flags.  For each variant it prints, for the per-block body of lane_hash_kernel<true,true,false> (the block
extraction of tests/test_lane_mix_cpu.py):
  body     instructions in the body;  alu: SHF + LOP3 + LEA + PRMT (the ALU pipe);  lea: LEA.HI;  imad / viadd;
  regs     registers and spill bytes (stores + loads) of the kernel, from ptxas -v;  local: LDL/STL in the body;
  vreads   vector-register source reads: every R operand of an instruction (memory addresses included) except RZ,
           minus reuse-cache hits (the same register in the same operand slot as a .reuse operand of the instruction
           before); uniform registers, predicates and immediates are not counted;
  vdist    the same, but a register read twice by one instruction (SHF.W / LEA.HI with lo == hi) counts once;
  bank3    instructions whose three vector source reads left after reuse hits are three distinct registers in one bank.
ASSUMPTION: bank = register index mod 2 (two banks, as published for Volta by microbenchmarks; NVIDIA does not document
the Hopper register file).  tools/ubench.cu's read-cost modes measure whether these costs are real.  The table is for
cutting the list of candidates before they are timed, not for predicting which is fastest.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
from collections import Counter
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from lane_ab import build  # noqa: E402  (same sources and flags as the timed builds)
from tests.test_lane_mix_cpu import _INSN, FUSED_DENSE, _block_body, _cuobjdump, _opcode  # noqa: E402

_REG = re.compile(r"^-?\|?R(\d+)\|?(\.reuse)?")
_MEMREG = re.compile(r"\bR(\d+)\b")


def fused_sass(lib: str) -> list:
    """[(address, instruction)] of the dense fused lane kernel in lib."""
    out = subprocess.run([_cuobjdump(), "-sass", lib], capture_output=True, text=True, check=True).stdout
    code, on = [], False
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            on = m.group(1).startswith(FUSED_DENSE)
            continue
        m = _INSN.search(line)
        if m and on:
            code.append((int(m.group(1), 16), m.group(2)))
    return code


def source_slots(ins: str) -> list:
    """[(slot, register index, reuse flag)] of the vector-register sources of one SASS instruction."""
    body = re.sub(r"^@!?U?P\w+\s+", "", ins)
    op, _, rest = body.partition(" ")
    ops = [o.strip() for o in rest.split(",")] if rest else []
    srcs = ops if op.startswith(("ST", "RED", "BRA", "EXIT", "BAR")) else ops[1:]
    slots = []
    for k, o in enumerate(srcs):
        if o.startswith("["):  # address operand: its registers are read
            slots += [(k, int(r), False) for r in _MEMREG.findall(o.replace("RZ", ""))]
            continue
        m = _REG.match(o)
        if m:
            slots.append((k, int(m.group(1)), bool(m.group(2))))
    return slots


def score_body(body: list) -> dict:
    ops = Counter(_opcode(i).split(".")[0] for i in body)
    vreads = vdist = bank3 = 0
    prev_reuse: set = set()
    for ins in body:
        slots = source_slots(ins)
        live = [(k, r) for k, r, _ in slots if (k, r) not in prev_reuse]  # reuse-cache hits read no bank
        vreads += len(live)
        regs = sorted({r for _, r in live})
        vdist += len(regs)
        if len(regs) == 3 and len({r % 2 for r in regs}) == 1:
            bank3 += 1
        prev_reuse = {(k, r) for k, r, reuse in slots if reuse}
    return {
        "body": len(body), "alu": ops["SHF"] + ops["LOP3"] + ops["LEA"] + ops["PRMT"], "lea": ops["LEA"],
        "imad": ops["IMAD"], "viadd": ops["VIADD"], "local": sum(_opcode(i).startswith(("LDL", "STL")) for i in body),
        "vreads": vreads, "vdist": vdist, "bank3": bank3,
    }


def ptxas_info(lib: str) -> dict:
    """registers and spill bytes of the dense fused kernel, from the ptxas -v output of lib's build: build.log next to
    lib (a lane_ab.py build) or in the csrc/ beside it (the Makefile's)."""
    d = os.path.dirname(lib)
    log = next((p for p in (os.path.join(d, "build.log"), os.path.join(d, "csrc", "build.log")) if os.path.exists(p)), None)
    if log is None:
        raise SystemExit(f"no build.log for {lib}")
    lines = open(log).read().splitlines()
    for i, ln in enumerate(lines):
        if "Function properties for " + FUSED_DENSE in ln:
            spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", lines[i + 1])
            regs = next(re.search(r"Used (\d+) registers", l) for l in lines[i + 1:] if "Used" in l)
            return {"regs": int(regs.group(1)), "spill": int(spill.group(1)) + int(spill.group(2))}
    raise SystemExit(f"no ptxas entry for {FUSED_DENSE} in {log}")


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--variant", action="append", metavar="NAME=SPEC", required=True)
    ap.add_argument("--build-dir", default=None)
    ap.add_argument("--jobs", type=int, default=4)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if _cuobjdump() is None:
        raise SystemExit("cuobjdump not found")
    variants = dict(v.split("=", 1) for v in args.variant)
    build_dir = os.path.abspath(args.build_dir or tempfile.mkdtemp(prefix="lane_score_"))
    with ThreadPoolExecutor(max_workers=args.jobs) as ex:
        libs = dict(zip(variants, ex.map(lambda kv: build(kv[0], kv[1], build_dir), variants.items())))
    rows = {}
    for name, lib in libs.items():
        rows[name] = {**score_body(_block_body(fused_sass(lib))),
                      **ptxas_info(lib)}
    cols = ["body", "alu", "lea", "imad", "viadd", "regs", "spill", "local", "vreads", "vdist", "bank3"]
    print("bank = register index mod 2 is an assumption (see the module docstring)")
    print(f"{'variant':>14} " + " ".join(f"{c:>6}" for c in cols) + "  defines")
    for name, r in rows.items():
        print(f"{name:>14} " + " ".join(f"{r[c]:>6}" for c in cols) + f"  {variants[name]}")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"variants": variants, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
