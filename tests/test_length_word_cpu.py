"""CPU: the routing and the oracle that tests/test_length_word_gpu.py relies on.

The GPU tests assert their path at run time; this pins, without a GPU, that the message shapes they use take that path
on an H100 SXM (132 SMs): every message of the chain batch routed to the chain kernel, none of the lane batch, and that
their lane batch mixes high words inside warps.  It also checks the prefix-sharing oracle and the stream schedule."""
import hashlib

import numpy as np
import pytest

from modal_client_b200 import _lib
from tests import test_length_word_gpu as lw
from tests.test_plan_cpu import restated

SMS = 132
SHA, MD5, BOTH, NO_OUT = _lib.SHA256, _lib.MD5, _lib.SHA256 | _lib.MD5, _lib.NO_OUTLIERS


def _lens(pairs) -> np.ndarray:
    return np.array([ln for _, ln in pairs], np.uint64)


def test_message_set_brackets_the_high_word():
    bits = {d: (lw.HI + d) << 3 for d in lw.DS}
    assert [b >> 32 for b in bits.values()] == [0, 0, 0] + [1] * 8
    assert bits[-8] & 0xFFFFFFFF == 0xFFFFFFC0 and bits[0] == 1 << 32
    tails = [(lw.HI + d) & 63 for d in lw.DS if d >= 0]
    assert any(t < 56 for t in tails) and any(t >= 56 for t in tails)  # one padding block and two
    assert {s & 15 for s in lw.STARTS} == {0, 1, 7, 15}
    for s, ln in lw.ZERO_TAIL:
        assert lw.Z - s >= lw.HI and lw.Z < s + ln <= lw.BUF
    assert all(s + ln < lw.Z for s, ln in lw.M)


@pytest.mark.parametrize("flags", [SHA, MD5, BOTH])
def test_chain_batch_routes_every_message_to_the_chain_kernel(flags):
    n = 2 * SMS + 7
    pairs = lw._cycled(lw.ALL, n)
    trimmed = [(s, lw.Z - s if (s, ln) in lw.ZERO_TAIL else ln) for s, ln in pairs]
    for p in (pairs, trimmed):
        assert _lib.plan_preview(_lens(p), flags, SMS) == restated(_lens(p), flags, SMS) == (n, 0)
        assert _lib.plan_preview(_lens(p), flags | NO_OUT, SMS) == (0, 0)
    assert n > 2 * SMS  # more messages than SMs twice over: several message groups per chain CTA


@pytest.mark.parametrize("flags", [SHA, MD5, BOTH])
def test_lane_batch_stays_on_the_lane_kernel(flags):
    n = 8 * SMS + len(lw.M)
    pairs = lw._cycled(lw.M, n)
    assert 4 * SMS < n <= 128 * SMS  # sparse launch shape, several lanes per warp
    assert _lib.plan_preview(_lens(pairs), flags | NO_OUT, SMS) == (0, 0)
    # without NO_OUTLIERS too: more long messages than chain slots, so none is moved and none queued apart
    assert _lib.plan_preview(_lens(pairs), flags, SMS) == restated(_lens(pairs), flags, SMS) == (0, 0)


def test_lane_batch_mixes_high_words_inside_warps():
    n = 8 * SMS + len(lw.M)
    pairs = lw._cycled(lw.M, n)
    assert {lw.plan_bucket(ln) for _, ln in pairs} == {lw.plan_bucket(lw.HI - 72), lw.plan_bucket(lw.HI)}
    assert {lw.bit_count_high(ln) for _, ln in pairs if lw.plan_bucket(ln) == lw.plan_bucket(lw.HI)} == {0, 1}
    assert lw.warps_mixing_high_words(pairs, 3) >= n // 30
    assert lw.warps_mixing_high_words([(0, 1 << 20)] * 30, 3) == 0


def test_prefix_digests_equal_hashlib():
    rng = np.random.default_rng(5)
    buf = rng.integers(0, 256, 5000, dtype=np.uint8)
    for start in (0, 1, 7, 15, 333):
        lengths = [0, 1, 55, 56, 64, 119, 120, 4000, 64, 1]  # unsorted, repeated, empty
        got = lw.prefix_digests(buf, start, lengths)
        assert sorted(got) == sorted(set(lengths))
        for ln, (s, m) in got.items():
            raw = buf[start : start + ln].tobytes()
            assert s == hashlib.sha256(raw).digest() and m == hashlib.md5(raw).digest()


def test_trimmed_length():
    buf = np.zeros(3 << 20, np.uint8)
    buf[[5, 100, (2 << 20) + 9]] = 1
    assert lw.trimmed_length(buf, 0, 3 << 20) == (2 << 20) + 10
    assert lw.trimmed_length(buf, 6, (2 << 20)) == 95
    assert lw.trimmed_length(buf, 101, 50) == 0


def test_stream_schedule_reaches_every_checkpoint():
    updates = list(lw.stream_pieces())
    offs = np.array([o for o, _, _ in updates])
    lens = np.array([ln for _, ln, _ in updates])
    assert offs[0] == 0 and np.array_equal(offs[1:], (offs + lens)[:-1]) and lens.min() >= 1
    assert [o + ln for o, ln, cp in updates if cp] == list(lw.CHECKPOINTS)
    assert all(o // lw.CHUNK == (o + ln - 1) // lw.CHUNK for o, ln, _ in updates)  # no update spans two chunks
    assert len(set(lens.tolist())) > 10  # uneven
    for total in lw.CHECKPOINTS:
        assert lw.finishes_on_chain(total) == (total % lw.STREAM_CAP >= 65_472)
    assert lw.bit_count_high(lw.CHECKPOINTS[-2]) == 8  # prior_bytes >= 2^32 when the digest runs
