"""CPU: the per-block body of the dense fused SHA-256 + MD5 lane kernel, read from the built library's SASS.

On H100 that kernel issues at the rate an SMSP sustains for a mix of ALU-pipe and FMA-pipe integer instructions
(DESIGN.md 5.1), so its time per block follows the number of instructions in the body.  A toolkit that stops fusing a
rotate with its add into LEA.HI, or a change that adds instructions there or starts spilling inside it, costs throughput
without failing any digest test; this catches all three.  (The stack frame is used only by the padding-block and
quantum set-up paths.)"""
import os
import re
import shutil
import subprocess
from collections import Counter

import pytest

from modal_client_b200 import _lib

FUSED_DENSE = "_ZN5b200h16lane_hash_kernelILb1ELb1ELb0E"
# per 64-byte block with CUDA 12.9: 545 SHF + 416 LOP3 + 192 LEA.HI + 16 PRMT on the ALU pipe, 671 IMAD on the FMA
# pipe, 10 others.  Each LEA.HI is a rotate fused with its add (add_rotl): without them the body is 2 042.
BODY_MAX = 1850
ALU_MAX = 1169

_INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
_BRA = re.compile(r"\bBRA\b[^;]*?0x([0-9a-f]+)\s*$")


def _cuobjdump():
    for cand in (shutil.which("cuobjdump"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")):
        if cand and os.path.exists(cand):
            return cand
    return None


def _kernel_sass(prefix: str) -> list:
    """[(address, instruction)] of the one kernel whose mangled name starts with prefix."""
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libb200hash.so not built")
    out = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    code, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = code.setdefault(m.group(1), []) if m.group(1).startswith(prefix) else None
            continue
        m = _INSN.search(line)
        if m and cur is not None:
            cur.append((int(m.group(1), 16), m.group(2)))
    assert len(code) == 1, sorted(code)
    return next(iter(code.values()))


def _block_body(code: list) -> list:
    """The largest basic block: the unrolled compression of one 64-byte block, run once per block."""
    targets = {int(m.group(1), 16) for _, ins in code for m in [_BRA.search(ins)] if m}
    blocks, cur = [], []
    for addr, ins in code:
        if addr in targets and cur:
            blocks.append(cur)
            cur = []
        cur.append(ins)
        if re.search(r"\b(BRA|EXIT|RET)\b", ins):
            blocks.append(cur)
            cur = []
    blocks.append(cur)
    return max(blocks, key=len)


def _opcode(ins: str) -> str:
    return re.sub(r"^@!?U?P\w+\s+", "", ins).split()[0]


@pytest.fixture(scope="module")
def fused_body():
    return _block_body(_kernel_sass(FUSED_DENSE))


def test_block_body_instruction_count(fused_body):
    ops = Counter(_opcode(i).split(".")[0] for i in fused_body)
    assert len(fused_body) <= BODY_MAX, ops
    # the adds that are not fused with a rotate stay IMADs on the FMA pipe: the ALU pipe carries no more than before
    assert ops["LEA"] >= 192 and ops["SHF"] + ops["LOP3"] + ops["LEA"] + ops["PRMT"] <= ALU_MAX, ops


def test_no_local_memory_in_block_body(fused_body):
    local = [i for i in fused_body if _opcode(i).startswith(("LDL", "STL"))]
    assert not local, local
