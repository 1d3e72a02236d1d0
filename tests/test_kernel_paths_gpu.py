"""GPU: every kernel path the dispatcher can take, each checked against the oracle.

Most batches elsewhere in the suite reach the lane kernel only in its simplest regime.  Every test here first asserts
that it reached the path it names, from the message count against the SM count, the host planner's preview
(``plan_preview``), the outlier count and the number of kernel launches.  Then it compares every digest row bit for bit
with oracle.c_oracle (hashlib for streams), trimmed lengths included.

launch_lane_hash (csrc/b200hash_kernels.cu) runs a lane batch of n messages on a device with S SMs as follows:

  n <= 4 S            sparse instantiation, one live lane per warp
  4 S < n <= 128 S    sparse, several live lanes per warp: the SHA-256-only pair gather and the MD5-only octet gather
                      fetch granules for live, misaligned partner lanes
  128 S < n           dense instantiation, full warps
  n > resident lanes  at a quantum boundary a lane saves its message's chaining state (hs, hm, prior, done) and puts
                      the message back on the queue, and another lane resumes it later

The lane kernel's 36 KiB of shared memory allow at most 6 CTAs of 128 threads per SM, whatever its register count.
So n >= 2 x 768 x S messages, each longer than one quantum, are sure to rotate through the queue.
"""
import asyncio
import base64
import hashlib
import io
import os
import subprocess
import sys

import numpy as np
import pytest

from modal_client_b200 import _lib
from modal_client_b200.synth import synth_bytes
from oracle import c_oracle

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHA, MD5, TRIM = _lib.SHA256, _lib.MD5, _lib.TRIM_ZEROS
BOTH = SHA | MD5
LANE_FLAGS = (SHA, MD5, BOTH, SHA | TRIM, BOTH | TRIM)
FULL_BLOCKS = (0, 1, 2, 31, 32, 33, 63, 64, 65, 97)
# tail residues: the padding block in the message's last quantum or the next one; one padding block or two
RESIDUES = (0, 1, 55, 56, 57, 63)
LANES_PER_SM_MAX = 6 * 128  # lane CTAs per SM allowed by shared memory x threads per CTA
QUANTUM = 32                # default blocks per time slice (B200H_QUANTUM)
CHAIN_MIN_BLOCKS = 1024     # kChainMinBlocks: a single message this long is routed to the chain kernel


def _sm_count() -> int:
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _new_context() -> _lib.Context:
    return _lib.Context(0, pinned_bytes=16 << 20, device_bytes=64 << 20)


@pytest.fixture(scope="module")
def ctx():
    c = _new_context()
    yield c
    c.close()


def _lengths(n: int, rng, blocks=FULL_BLOCKS, lo: int = 0, hi: int = 160) -> np.ndarray:
    """n lengths.  The first len(blocks) x len(RESIDUES) messages take every (full blocks, tail residue) pair once; after
    that, even messages cycle through ``blocks``, odd ones draw from [lo, hi], and residues are drawn from RESIDUES."""
    i = np.arange(n)
    b = np.asarray(blocks, np.int64)
    r = np.asarray(RESIDUES, np.int64)
    nb = np.where(i % 2 == 0, b[(i // 2) % b.size], rng.integers(lo, hi + 1, n))
    res = r[rng.integers(0, r.size, n)]
    k = min(n, b.size * r.size)
    nb[:k] = b[np.arange(k) // r.size]
    res[:k] = r[np.arange(k) % r.size]
    return (nb * 64 + res).astype(np.uint64)


class _Layout:
    """n messages in one CUDA tensor.  Message i starts at a 16-aligned cursor plus a misalignment 0..15 drawn
    independently of its length: the planner orders messages by length, so this is what mixes misalignments inside
    a warp.  ``zero_every`` = k zeroes a tail of every k-th message (1 byte, part of a block, a block, all of it), which
    only TRIM_ZEROS sees.  The host copy feeds the oracle."""

    def __init__(self, ctx, lens, seed: int, zero_every: int = 0):
        import torch

        rng = np.random.default_rng(seed)
        self.lens = np.asarray(lens, np.uint64)
        n = self.lens.size
        self.mis = rng.integers(0, 16, n).astype(np.uint64)
        span = (self.mis + self.lens + np.uint64(15)) & ~np.uint64(15)
        cursor = np.concatenate([[0], np.cumsum(span)]).astype(np.uint64)
        self.offs = cursor[:-1] + self.mis
        total = int(cursor[-1]) + 64
        self.data = torch.empty(total, dtype=torch.uint8, device="cuda:0")
        ctx.fill_synth_device(self.data.data_ptr(), total, seed)
        torch.cuda.synchronize()
        self.host = self.data.cpu().numpy()
        if zero_every:
            for k, i in enumerate(range(0, n, zero_every)):
                ln = int(self.lens[i])
                z = min(ln, (1, 63, 64, 200, ln)[k % 5])
                end = int(self.offs[i]) + ln
                self.host[end - z : end] = 0
            self.data.copy_(torch.from_numpy(self.host))
        self.d_off = torch.from_numpy(self.offs.astype(np.int64)).to(self.data.device)
        self.d_len = torch.from_numpy(self.lens.astype(np.int64)).to(self.data.device)
        self._want = {}

    def oracle(self, trim: bool):
        """(sha[n,32], md5[n,16], end[n]) of the whole layout: both digests in one pass, once per trim setting."""
        if trim not in self._want:
            self._want[trim] = c_oracle.hash_batch(self.host, self.offs, self.lens, trim=trim)
        return self._want[trim]

    def seen_lengths(self, flags: int) -> np.ndarray:
        """The lengths the planner sees: the trimmed ones under TRIM_ZEROS."""
        return self.oracle(True)[2] if flags & TRIM else self.lens

    def hash(self, ctx, flags: int):
        """Hash the layout through b200h_hash_batch_device_hl -> (sha | None, md5 | None, trimmed, launches made)."""
        import torch

        n = self.lens.size
        dev = self.data.device
        sha = torch.empty((n, 32), dtype=torch.uint8, device=dev) if flags & SHA else None
        md5 = torch.empty((n, 16), dtype=torch.uint8, device=dev) if flags & MD5 else None
        trimmed = torch.empty(n, dtype=torch.int64, device=dev)
        l0 = ctx.launch_count
        ctx.hash_batch_device(self.data.data_ptr(), self.d_off.data_ptr(), self.d_len.data_ptr(), n, flags,
                              0 if sha is None else sha.data_ptr(), 0 if md5 is None else md5.data_ptr(),
                              trimmed.data_ptr(), torch.cuda.current_stream().cuda_stream, h_lengths=self.lens)
        torch.cuda.synchronize()
        launches = ctx.launch_count - l0
        return (None if sha is None else sha.cpu().numpy(), None if md5 is None else md5.cpu().numpy(),
                trimmed.cpu().numpy().astype(np.uint64), launches)

    def check(self, flags: int, sha, md5, trimmed):
        s, m, e = self.oracle(bool(flags & TRIM))
        assert np.array_equal(trimmed, e if flags & TRIM else self.lens), f"flags {flags}: trimmed lengths differ"
        for name, got, want in (("sha256", sha, s), ("md5", md5, m)):
            if got is None:
                continue
            bad = np.flatnonzero((got != want).any(axis=1))
            rows = ", ".join(f"#{i} {int(e[i]) >> 6} blocks + {int(e[i]) & 63} B at misalignment {int(self.mis[i])}"
                             for i in bad[:8])
            assert bad.size == 0, f"flags {flags}: {bad.size} of {len(e)} {name} rows differ from the oracle: {rows}"


def _run_lane_only(ctx, lay: _Layout, flags: int, sm: int):
    """Hash ``lay`` with ``flags`` after asserting that one short-queue lane launch does all the work: no outliers and no
    long lane queue in the preview, none routed by the call, and launches = trim (2) + plan (3) + one lane launch."""
    assert _lib.plan_preview(lay.seen_lengths(flags), flags & BOTH, sm) == (0, 0)
    sha, md5, trimmed, launches = lay.hash(ctx, flags)
    assert ctx.last_outlier_count == 0
    assert launches == (2 if flags & TRIM else 0) + 3 + 1, launches
    lay.check(flags, sha, md5, trimmed)


# ------------------------------------------------------------------------------------------- lane-kernel regimes


def _regime_n(regime: str, sm: int) -> int:
    n = {"sparse_one_lane_per_warp": 4 * sm, "sparse_lanes_share_warps": 68 * sm + 24, "dense_full_warps": 227 * sm + 36}[regime]
    if regime == "sparse_one_lane_per_warp":
        assert n <= 4 * sm  # one warp per message
    elif regime == "sparse_lanes_share_warps":
        assert 4 * sm < n <= 128 * sm and -(-n // (4 * sm)) >= 2  # 4 S warps, >= 2 live lanes each
    else:
        assert 128 * sm < n < 2 * LANES_PER_SM_MAX * sm  # more than 4 S full warps, below the rotation bound
    return n


@pytest.mark.parametrize(
    "regime,no_sparse",
    [
        ("sparse_one_lane_per_warp", False),
        ("sparse_lanes_share_warps", False),
        ("dense_full_warps", False),
        # B200H_NO_SPARSE is read at every launch: the dense instantiations with fewer than 32 live lanes per warp
        ("sparse_one_lane_per_warp", True),
        ("sparse_lanes_share_warps", True),
    ],
)
def test_lane_regimes_match_oracle(ctx, monkeypatch, regime, no_sparse):
    if no_sparse:
        monkeypatch.setenv("B200H_NO_SPARSE", "1")
    else:
        monkeypatch.delenv("B200H_NO_SPARSE", raising=False)
    sm = _sm_count()
    n = _regime_n(regime, sm)
    lay = _Layout(ctx, _lengths(n, np.random.default_rng(n)), seed=n, zero_every=7)
    for flags in LANE_FLAGS:
        _run_lane_only(ctx, lay, flags, sm)


def test_dense_lanes_rotate_messages_through_the_queue(ctx):
    """More messages than lanes can ever be resident, each longer than one quantum: every message is saved to its
    ChainState and resumed by another lane at least once, with mixed misalignments and every tail residue."""
    sm = _sm_count()
    n = 2 * LANES_PER_SM_MAX * sm
    lens = _lengths(n, np.random.default_rng(7), blocks=(33, 63, 64, 65, 97), lo=33, hi=100)
    assert int((lens >> np.uint64(6)).min()) > QUANTUM
    lay = _Layout(ctx, lens, seed=70, zero_every=8)
    for flags in LANE_FLAGS:
        _run_lane_only(ctx, lay, flags, sm)


def test_long_lane_queue_with_single_digests(ctx):
    """Chain kernel + lane-packed long queue + short queue for SHA-256 alone and MD5 alone, from device memory with
    misaligned starts (the host entry points pack every message 16-byte aligned)."""
    sm = _sm_count()
    lens = np.array([8 << 20] * 3 + [(1 << 20) + 64 * i for i in range(100)] + [3000 + (i % 977) for i in range(20000)],
                    np.uint64)
    lay = _Layout(ctx, lens, seed=71)
    assert len(set(lay.mis[:103].tolist())) > 8
    for flags in (SHA, MD5):
        assert _lib.plan_preview(lens, flags, sm) == (3, 100)
        sha, md5, trimmed, launches = lay.hash(ctx, flags)
        assert ctx.last_outlier_count == 3
        assert launches == 3 + 1 + 2  # plan, chain, lane launches for the short and the long queue
        lay.check(flags, sha, md5, trimmed)


# ------------------------------------------------------------------------------- paths that need a fresh process


def _run_child(call: str, env: dict, timeout: int = 600) -> str:
    """Run ``tests.test_kernel_paths_gpu.<call>`` in a fresh interpreter with ``env`` added (settings the library
    caches per process); fail with the child's output unless it exits with 0."""
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    cmd += ["-c", f"import tests.test_kernel_paths_gpu as t; t.{call}"]
    r = subprocess.run(cmd, cwd=ROOT, env=dict(os.environ, **env), capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, f"{call} with {env} exited with {r.returncode}\n{r.stdout[-4000:]}\n{r.stderr[-8000:]}"
    return r.stdout


def _odd_quantum_child():
    """Child of test_odd_quanta: the rotation regime with short messages (3..20 blocks) under B200H_QUANTUM."""
    q = int(os.environ["B200H_QUANTUM"])
    sm = _sm_count()
    c = _new_context()
    n = 2 * LANES_PER_SM_MAX * sm
    lens = _lengths(n, np.random.default_rng(q), blocks=(3, 4, 5, 6, 7, 19, 20), lo=3, hi=20)
    assert int((lens >> np.uint64(6)).min()) >= q
    lay = _Layout(c, lens, seed=80 + q, zero_every=8)
    for flags in LANE_FLAGS:
        _run_lane_only(c, lay, flags, sm)
    c.close()
    print(f"quantum {q}: {n} messages ok")


@pytest.mark.parametrize("quantum", [1, 3])
def test_odd_quanta(quantum):
    """With an odd quantum a time slice ends in a one-block chunk inside a message and the next one starts at an odd
    block; the default of 32 never does either.  The quantum is cached on the first launch, hence a fresh process."""
    out = _run_child("_odd_quantum_child()", {"B200H_QUANTUM": str(quantum)})
    assert f"quantum {quantum}:" in out


def _eight_group_child():
    """Child of test_eight_group_chain_kernel: 4 S < N <= 8 S outliers of 64 KiB + e, routed with B200H_CHAIN_GROUPS=8."""
    assert os.environ["B200H_CHAIN_GROUPS"] == "8"
    sm = _sm_count()
    c = _new_context()
    big_n = 5 * sm + 7
    assert 4 * sm < big_n <= 8 * sm  # more than the default 4 groups per CTA hold
    rng = np.random.default_rng(81)
    # every tail residue at several block counts, the 32-block tile boundaries, then random lengths
    extra = [64 * k + r for k in (0, 1, 31, 32, 33, 63, 64, 65, 97) for r in RESIDUES] + [2047, 2048, 2049, 4095, 4096, 4097]
    extra += rng.integers(0, 8000, big_n - len(extra)).tolist()
    lens = (65536 + np.array(extra, np.int64)).astype(np.uint64)
    lay = _Layout(c, lens, seed=82)
    assert set(lay.mis.tolist()) == set(range(16))
    for flags in (SHA, MD5, BOTH, BOTH | TRIM):
        sha, md5, trimmed, launches = lay.hash(c, flags)
        assert c.last_outlier_count == big_n, c.last_outlier_count  # the routing is decided with the 8-group cap
        assert launches == (2 if flags & TRIM else 0) + 3 + 1  # plan, one chain launch, no lane launch
        lay.check(flags, sha, md5, trimmed)
    c.close()
    print(f"eight groups: {big_n} outliers on {sm} SMs ok")


def test_eight_group_chain_kernel():
    """The chain-kernel instantiations with eight message groups per CTA run only when more than 4 x SMs outliers are
    routed, which needs B200H_CHAIN_GROUPS=8.  The library keeps that setting process-wide from the first context on,
    so it is tried in a fresh process."""
    out = _run_child("_eight_group_child()", {"B200H_CHAIN_GROUPS": "8"})
    assert "eight groups:" in out


# ------------------------------------------------------------------------------------------------------- streams

STREAM_SETTINGS = {
    "chain_4mib_absorbs": {},
    "chain_64kib_absorbs": {"B200H_STREAM_BUF": "65536"},
    "lane_64kib_absorbs": {"B200H_CHAIN": "0", "B200H_STREAM_BUF": "65536"},
}


@pytest.mark.parametrize("setting", list(STREAM_SETTINGS))
def test_digest_streams_of_every_digest_selection(monkeypatch, setting):
    """SHA-256 alone, MD5 alone and both, one after another on one context (each new stream reuses the pooled buffer of
    the one closed before it, with other flags).  Irregular pieces, totals that are exact multiples of the absorb size
    (the digest then resumes a zero-byte message), a reset mid-stream, and digests() against hashlib after every
    update.  Each absorb goes to the chain kernel, or to the lane kernel with B200H_CHAIN=0."""
    env = STREAM_SETTINGS[setting]
    for k in ("B200H_CHAIN", "B200H_STREAM_BUF"):
        if k in env:
            monkeypatch.setenv(k, env[k])
        else:
            monkeypatch.delenv(k, raising=False)
    cap = int(env.get("B200H_STREAM_BUF", 4 << 20))
    chain = env.get("B200H_CHAIN") != "0"
    pieces = [0, 1, 63, 64, cap - 1, 1, cap, 3 * cap + 5, 17]
    pieces.append(6 * cap - sum(pieces))  # total 6 x cap
    pieces.append(70_000)  # with 4 MiB absorbs the digest of this fill goes to the chain kernel as well
    src = synth_bytes(90, cap + 127 + sum(pieces))
    c = _new_context()
    try:
        for flags in (SHA, MD5, BOTH):
            st = c.stream(flags)
            pos, total = 0, 0
            hs, hm = hashlib.sha256(), hashlib.md5()
            for i, k in enumerate(pieces[:5] + ["reset"] + pieces):
                if k == "reset":
                    st.reset()
                    total, hs, hm = 0, hashlib.sha256(), hashlib.md5()
                    continue
                chunk = src[pos : pos + k]
                pos += k
                st.update(chunk)
                hs.update(chunk)
                hm.update(chunk)
                if (total + k) // cap > total // cap:  # this update absorbed at least one whole buffer
                    assert c.last_outlier_count == (1 if chain else 0), (flags, i)
                total += k
                fill = total % cap
                s, m = st.digests()
                assert s == (hs.digest() if flags & SHA else None), (flags, i, total)
                assert m == (hm.digest() if flags & MD5 else None), (flags, i, total)
                assert c.last_outlier_count == (1 if chain and (fill >> 6) + 1 >= CHAIN_MIN_BLOCKS else 0), (flags, i)
            assert total == 6 * cap + 70_000
            st.close()
    finally:
        c.close()


def test_production_single_digest_callers(gpu_backend):
    """hash_utils over a BinaryIO (SHA-256 alone, MD5 alone, both) and the MD5 BytesIOSegmentPayload computes on the
    device when no digest was supplied: default 4 MiB absorbs on the chain kernel."""
    from modal_client_b200 import hash_utils
    from modal_client_b200.bytes_io_segment_payload import BytesIOSegmentPayload

    data = synth_bytes(91, (9 << 20) + 3)
    b64 = lambda raw: base64.b64encode(raw).decode("ascii")  # noqa: E731
    assert hash_utils.get_md5_base64(io.BytesIO(data)) == b64(hashlib.md5(data).digest())
    assert hash_utils.get_sha256_hex(io.BytesIO(data)) == hashlib.sha256(data).hexdigest()
    up = hash_utils.get_upload_hashes(io.BytesIO(data))
    assert up.md5_base64 == b64(hashlib.md5(data).digest()) and up.sha256_base64 == b64(hashlib.sha256(data).digest())
    assert gpu_backend.last_outlier_count == 1  # the last 1 MiB + 3 bytes were digested on the chain kernel too

    class Sink:
        def __init__(self):
            self.data = bytearray()

        async def write(self, chunk):
            self.data += chunk

    start, length = 12345, 6 << 20
    pl = BytesIOSegmentPayload(io.BytesIO(data), segment_start=start, segment_length=length, chunk_size=(1 << 20) + 7)
    sink = Sink()
    asyncio.run(pl.write_with_length(sink, None))
    assert bytes(sink.data) == data[start : start + length] and pl.remaining_bytes() == 0
    assert pl.md5_checksum().hexdigest() == hashlib.md5(data[start : start + length]).hexdigest()
    pl.reset_state()
