"""CPU: the source operands of the dense fused lane kernel's per-block body, read from the built library's SASS.

Every add of that body but the round-constant ones is `addf` = IMAD x, one, y.  On H100 an IMAD that reads three
vector registers issues slower next to the ALU-pipe LOP3s and SHFs than one that reads `one` from a uniform register
(tools/ubench.cu modes 7 and 25, DESIGN.md 5.1).  ptxas keeps `one` in a uniform register only while no IMAD of the
kernel has an immediate addend, so the 128 round-constant adds (SHA-256's W + K, MD5's x + T) are plain adds, which it
issues as VIADD (sha_round / md5_step).  A toolkit or a source change that puts `one` back in a vector register, or
turns those adds into ALU-pipe IADD3s, costs throughput without failing any digest test; this catches both."""
import re
from collections import Counter

import pytest

from tests.test_lane_mix_cpu import FUSED_DENSE, _block_body, _kernel_sass, _opcode

# per 64-byte block with CUDA 12.9: 528 IMAD R, R, UR, R (the adds); 128 VIADD R, R, imm (the round-constant adds) + 1
# of the loop; 15 other IMAD forms.  The parent layout, 656 IMAD + 1 VIADD, had 528 three-vector-register IMADs.
UNIFORM_ADDS_MIN = 528
CONST_ADDS_MIN = 128
FMA_MAX = 672  # IMAD + VIADD: the constant adds moved between FMA-pipe forms, none went to the ALU pipe

_VREG = re.compile(r"-?R\d+(\.reuse)?$")


def _sources(ins: str) -> list:
    return [o.strip() for o in re.sub(r"^@!?U?P\w+\s+", "", ins).split(None, 1)[1].split(",")[1:]]


@pytest.fixture(scope="module")
def fused_body():
    return _block_body(_kernel_sass(FUSED_DENSE))


def test_adds_read_one_from_a_uniform_register(fused_body):
    imads = [i for i in fused_body if _opcode(i).split(".")[0] == "IMAD"]
    three_vreg = [i for i in imads if sum(bool(_VREG.match(s)) for s in _sources(i)) == 3]
    assert not three_vreg, (len(three_vreg), three_vreg[:4])
    uniform = [i for i in imads if any(re.match(r"UR\d+$", s) for s in _sources(i))]
    assert len(uniform) >= UNIFORM_ADDS_MIN, (len(uniform), len(imads))


def test_constant_adds_are_viadd(fused_body):
    ops = Counter(_opcode(i).split(".")[0] for i in fused_body)
    # VIADD issues next to SHF / LOP3 at 0.73-0.88 warp-instructions per cycle per SMSP, above the ALU pipe's 0.5
    # (tools/ubench.cu modes 26, 27): it is not an ALU-pipe instruction
    assert ops["VIADD"] >= CONST_ADDS_MIN and ops["IMAD"] + ops["VIADD"] <= FMA_MAX, ops
