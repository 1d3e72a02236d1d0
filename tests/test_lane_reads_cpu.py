"""CPU: the vector register-file reads of the dense fused lane kernel's per-block body, read from the built library's SASS.

That body's instruction count is at its floor (1 168 ALU-pipe instructions are the minimum, DESIGN.md 5.1), and the
kernel issues well under the ALU pipe's rate: what is left to win or lose is in how ptxas schedules and allocates the
same instructions, which sets how many source operands are read from the vector register file rather than the operand
reuse cache.  A toolkit or a source change that reads more, spills inside the body, or gives back a LEA.HI
rotate+add costs throughput without failing any digest test; this catches each.  The counts are
tools/lane_sass_score.py's, with CUDA 12.9."""
import os
import sys
from collections import Counter

import pytest

from tests.test_lane_mix_cpu import FUSED_DENSE, _block_body, _kernel_sass, _opcode

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
from lane_sass_score import score_body  # noqa: E402

# per 64-byte block, the body as built: 3 854 vector reads at 3 CTAs per SM with SHA-256's LOP3 operands in the order
# (b, c, a) and MD5 steps first; the form before (4 CTAs, 128 registers) read 3 882 and ran 3.1 % slower (DESIGN.md 5.1)
VREADS_MAX = 3860
ALU = 1169  # 545 SHF + 416 LOP3 + 192 LEA.HI + 16 PRMT
LEA_HI = 192


@pytest.fixture(scope="module")
def fused_body():
    return _block_body(_kernel_sass(FUSED_DENSE))


def test_vector_register_reads_per_block(fused_body):
    s = score_body(fused_body)
    assert s["vreads"] <= VREADS_MAX, s


def test_no_local_memory_in_block_body(fused_body):
    assert score_body(fused_body)["local"] == 0


def test_alu_pipe_and_lea_hi_counts(fused_body):
    ops = Counter(_opcode(i) for i in fused_body)
    s = score_body(fused_body)
    assert s["alu"] == ALU and ops["LEA.HI"] == LEA_HI, (s, ops["LEA.HI"])
