"""The planner's routing policy, checked on the CPU.

``b200h_plan_preview`` runs the library's host-side planner (``plan_outliers_host``: the code that sizes the chain /
long-queue launches without reading the device planner's answer back; on the GPU
``tests/test_gpu_round2.py::test_host_outlier_plan_equals_device_plan`` pins it to the device kernels).  Here it is
compared with a plain-Python restatement of the rules as DESIGN.md 5.3 / 5.4 states them, on random batches and on the
scenarios the design quotes."""
import numpy as np
import pytest

from modal_client_b200 import _lib

SMS = 132  # H100 SXM
MIN_BLOCKS, RATIO, MAX_CHAIN_CAP, LONG_RING = 1024, 21000, 1184, 32768


def _bucket(length: int) -> int:
    nb = (length >> 6) + 1
    if nb < 16:
        return nb
    e = nb.bit_length() - 1
    return min(16 + (e - 4) * 8 + ((nb >> (e - 3)) & 7), 511)


def _bucket_floor(b: int) -> int:
    if b < 16:
        return b
    e, mant = (b - 16) // 8 + 4, (b - 16) % 8
    return (8 + mant) << (e - 3)


def restated(lengths, flags=_lib.SHA256 | _lib.MD5, sms=SMS):
    """(n_chain, n_long) by the rules of DESIGN.md 5.3 / 5.4, on bucket lower bounds like the device planner."""
    lengths = [int(x) for x in lengths]
    n = len(lengths)
    if n == 0:
        return 0, 0
    max_chain = 0 if flags & _lib.NO_OUTLIERS else min(4 * sms, MAX_CHAIN_CAP)
    long_cap = min(sms * 4 * 32, LONG_RING)
    ratio8 = 3 if (flags & 3) == 3 else 4
    total = sum((x >> 6) + 1 for x in lengths)
    longest = max(lengths)
    if (longest >> 6) + 1 < MIN_BLOCKS:
        return 0, 0
    thr1 = max(total // RATIO, MIN_BLOCKS)                     # rule (1): outlasts the batch on saturated lanes
    thr = max(thr1, _bucket_floor(_bucket(longest)) // 8 * ratio8)  # rule (2): longer than ratio8/8 of the longest
    floors = [_bucket_floor(_bucket(x)) for x in lengths]
    count1 = sum(f >= thr1 for f in floors)
    chosen = [f for f in floors if f >= thr]
    count, chain_blocks = len(chosen), sum(chosen)
    c = 0                                                       # rule (3): all of them or none
    if max_chain and 0 < count <= max_chain:
        if count <= sms * 3 // 4 or count == n or total - min(chain_blocks, total) <= total // 4:
            c = count
    n_long = max(count1 - c, 0)
    if n_long == 0 or n_long > long_cap or n_long == n - c:
        n_long = 0
    return c, n_long


SCENARIOS = [
    # (lengths, flags, expected (n_chain, n_long) -- as DESIGN.md states them)
    ("bench: 100 000 x 256 KiB", [262144] * 100_000, 3, (0, 0)),
    ("C5: 128 x 64 MiB -> nothing but long messages, all on chains", [64 << 20] * 128, 3, (128, 0)),
    ("C4(ii): 1 024 x 8 MiB equal blocks -> more than 4 per SM: none", [8 << 20] * 1024, 1, (0, 0)),
    ("2 048 x 4 MiB -> none (moving a part only costs interference)", [4 << 20] * 2048, 3, (0, 0)),
    ("C3-v1 shard: one 59.75 MB file among 131 071 of 100 KB", [59_753_768] + [100_000] * 131_071, 3, (1, 0)),
    ("one 1 GiB message", [1 << 30], 3, (1, 0)),
    ("short messages only", [4096] * 5000, 3, (0, 0)),
    ("outliers switched off", [59_753_768] + [100_000] * 1000, 3 | _lib.NO_OUTLIERS, (0, None)),
]


@pytest.mark.parametrize("name,lengths,flags,expect", SCENARIOS, ids=[s[0] for s in SCENARIOS])
def test_documented_routing_scenarios(name, lengths, flags, expect):
    got = _lib.plan_preview(lengths, flags, SMS)
    assert got == restated(lengths, flags)
    assert got[0] == expect[0] and (expect[1] is None or got[1] == expect[1])


def test_c3v2_share_routes_its_8mib_blocks_and_queues_the_1_to_4_mib_ones():
    """One rank's share of C3-v2: 93 blocks of 8 MiB among 131 002 smaller ones, 1 339 of
    them between 1 and 4 MiB: the 8 MiB blocks get an SM each (93 <= 3/4 of the SMs), the 1-4 MiB blocks form the long
    lane queue, the rest is the ordinary queue."""
    rng = np.random.default_rng(11)
    small = rng.integers(1_000, 180_000, 131_002 - 1_339)  # ~12 GiB in all: rule (1) starts at ~0.7 MB
    mid = rng.integers(1 << 20, 4 << 20, 1_339)
    lengths = np.concatenate([[8 << 20] * 93, mid, small]).astype(np.uint64)
    rng.shuffle(lengths)
    n_chain, n_long = _lib.plan_preview(lengths, _lib.SHA256, SMS)
    assert (n_chain, n_long) == restated(lengths, _lib.SHA256)
    assert n_chain == 93 and n_long == 1_339


def test_plan_preview_equals_the_restated_rules_on_random_batches():
    rng = np.random.default_rng(2)
    for case in range(300):
        n = int(rng.integers(1, 3000))
        kind = case % 5
        if kind == 0:  # heavy tail
            lengths = np.exp(rng.normal(11, 2.2, n)).astype(np.uint64)
        elif kind == 1:  # equal long messages
            lengths = np.full(n, int(rng.integers(1 << 16, 1 << 24)), np.uint64)
        elif kind == 2:  # a few outliers among small ones
            lengths = rng.integers(0, 200_000, n).astype(np.uint64)
            k = int(rng.integers(1, 200))
            lengths[:k] = rng.integers(4 << 20, 64 << 20, min(k, n))[: min(k, n)]
        elif kind == 3:  # two size classes
            lengths = np.where(rng.random(n) < 0.3, 6 << 20, 1 << 20).astype(np.uint64)
        else:  # tiny
            lengths = rng.integers(0, 5000, n).astype(np.uint64)
        for flags in (3, 1, 2):
            sms = int(rng.choice([148, 132, 16]))
            assert _lib.plan_preview(lengths, flags, sms) == restated(lengths, flags, sms), (case, flags, sms)


def test_plan_preview_rejects_bad_arguments():
    with pytest.raises(_lib.B200HashError):
        _lib.plan_preview([1, 2, 3], flags=0)
    with pytest.raises(_lib.B200HashError):
        _lib.plan_preview([1, 2, 3], sm_count=0)
    assert _lib.plan_preview([]) == (0, 0)
