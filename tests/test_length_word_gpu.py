"""GPU: the high word of the 64-bit bit count in every final block, against hashlib.

SHA-256 and MD5 end every message with its length in bits as a 64-bit word; its high half is non-zero once a message
reaches 2^29 bytes (512 MiB).  Two kernels write that word, each in its own code: ``chain_hash_kernel`` (warp 0 puts
it into the padding tile the MD5 warp reads, the SHA-256 expander substitutes its own big-endian words) and
``lane_hash_kernel`` (``bits_hi`` passed to every ``compress<>`` body: sparse fused, sparse SHA-256, MD5 alone, dense
fused, dense SHA-256).  A wrong high word gives wrong digests for large messages only, so each test here hashes
messages of 2^29 + d bytes whose final block the kernel under test writes:

  chain kernel, batch    ``hash_batch_device`` over 2 S + 7 long messages: all routed to the chain kernel, several
                         message groups per CTA, each group with its own high word
  chain kernel, callers  ``hash_batch_host`` / ``hash_files`` / ``get_file_upload_specs`` with the library's default
                         staging (4 GiB wave slots: a 512 MiB message is hashed whole, not segmented)
  lane kernel            ``NO_OUTLIERS`` batches of 4 S < n <= 128 S messages: sparse (several live lanes per warp),
                         MD5 alone, and the dense bodies with ``B200H_NO_SPARSE``
  streams                ``DigestStream`` past 2^29 and 2^32 bytes absorbed, finished on the chain or the lane kernel

Every test first asserts the path it reaches (planner preview, outlier count, launch count), then compares every row
bit for bit, trimmed lengths included.  The oracle hashes each start once up to its shortest message and extends that
state in ascending length order, taking a ``copy()`` digest at every length (``prefix_digests``).
"""
import base64
import hashlib
import io
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from modal_client_b200 import _lib
from modal_client_b200.synth import synth_array

pytestmark = pytest.mark.gpu

SHA, MD5, TRIM, NO_OUT = _lib.SHA256, _lib.MD5, _lib.TRIM_ZEROS, _lib.NO_OUTLIERS
BOTH = SHA | MD5
CHAIN_MIN_BLOCKS = 1024  # kChainMinBlocks: a single message this long is routed to the chain kernel

HI = 1 << 29                    # first length whose bit count needs the high word
BUF = HI + (8 << 20)            # the shared device buffer
Z = HI + (4 << 20)              # the buffer is zero from here to its end
STARTS = (0, 1, 7, 15)          # misalignments of the message starts
# 2^29 + d: bit count 0xFFFFFDC0 / 0xFFFFFFC0 / 0xFFFFFFF8 (high word 0), exactly 2^32 (d = 0), then both padding
# shapes (tail < 56 bytes: one padding block, >= 56: two) on either side of a block edge, and a longer tail
DS = (-72, -8, -1, 0, 1, 55, 56, 57, 63, 64, 64 * 33 + 55)
M = tuple((s, HI + d) for s in STARTS for d in DS)
# messages that run into the zero region: under TRIM_ZEROS they trim to Z - start (>= 2^29) after a wide zero scan
ZERO_TAIL = tuple((s, end - s) for s, end in zip(STARTS, (BUF, Z + 1, Z + 127, Z + (2 << 20) + 5)))
ALL = M + ZERO_TAIL


def prefix_digests(buf, start: int, lengths) -> dict:
    """{L: (sha256, md5) of buf[start : start + L]} for every L in ``lengths``: one pass per algorithm, the lengths
    taken in ascending order, each digest from a ``copy()`` of the running state."""
    mv = memoryview(buf).cast("B")
    hs, hm = hashlib.sha256(), hashlib.md5()
    out, pos = {}, 0
    for ln in sorted({int(x) for x in lengths}):
        chunk = mv[start + pos : start + ln]
        hs.update(chunk)
        hm.update(chunk)
        pos = ln
        out[ln] = (hs.copy().digest(), hm.copy().digest())
    return out


def trimmed_length(buf: np.ndarray, start: int, length: int) -> int:
    """Length of buf[start : start + length] without its trailing zero bytes."""
    end, step = start + length, 1 << 20
    while end > start:
        lo = max(start, end - step)
        nz = np.flatnonzero(buf[lo:end])
        if nz.size:
            return lo + int(nz[-1]) + 1 - start
        end = lo
    return 0


def bit_count_high(length: int, prior: int = 0) -> int:
    return ((prior + length) << 3) >> 32


def plan_bucket(length: int) -> int:
    """The planner's queue bucket of a message (plan_bucket in csrc/b200hash_kernels.cu)."""
    nb = (length >> 6) + 1
    if nb < 16:
        return nb
    e = nb.bit_length() - 1
    return min(16 + (e - 4) * 8 + ((nb >> (e - 3)) & 7), 511)


def warps_mixing_high_words(pairs, lanes_per_warp: int) -> int:
    """Warps whose lanes see both high words 0 and 1, if each bucket's queue keeps the batch order and every warp takes
    ``lanes_per_warp`` consecutive entries of one bucket."""
    mixed = 0
    for b in sorted({plan_bucket(ln) for _, ln in pairs}):
        hi = [bit_count_high(ln) for _, ln in pairs if plan_bucket(ln) == b]
        mixed += sum(len(set(hi[i : i + lanes_per_warp])) > 1 for i in range(0, len(hi), lanes_per_warp))
    return mixed


def _sm_count() -> int:
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


class _Data:
    """The shared buffer on the device and on the host, and every digest and trimmed length the tests compare with."""

    def __init__(self):
        import torch

        ctx = _lib.Context(0, pinned_bytes=16 << 20, device_bytes=64 << 20)
        try:
            self.dev = torch.empty(BUF, dtype=torch.uint8, device="cuda:0")
            ctx.fill_synth_device(self.dev.data_ptr(), BUF, 29)
            torch.cuda.synchronize()
        finally:
            ctx.close()
        self.dev[Z:] = 0
        self.host = self.dev.cpu().numpy()
        self.trimmed = {(s, ln): trimmed_length(self.host, s, ln) for s, ln in ALL}
        for s, ln in ZERO_TAIL:
            assert HI <= self.trimmed[(s, ln)] <= Z - s
        want = {s: [] for s in STARTS}
        for (s, ln), t in self.trimmed.items():
            want[s] += [ln, t]
        with ThreadPoolExecutor(len(STARTS)) as ex:  # hashlib drops the GIL over large buffers
            per_start = dict(zip(STARTS, ex.map(lambda s: prefix_digests(self.host, s, want[s]), STARTS)))
        self.digests = {(s, ln): per_start[s][ln] for s, lens in want.items() for ln in lens}

    def expect(self, pairs, flags: int):
        """(sha[n, 32], md5[n, 16], lengths[n]) that ``flags`` must produce for these (start, length) messages."""
        ends = [self.trimmed[p] if flags & TRIM else p[1] for p in pairs]
        rows = [self.digests[(s, e)] for (s, _), e in zip(pairs, ends)]
        sha = np.frombuffer(b"".join(r[0] for r in rows), np.uint8).reshape(-1, 32)
        md5 = np.frombuffer(b"".join(r[1] for r in rows), np.uint8).reshape(-1, 16)
        return sha, md5, np.array(ends, np.uint64)


@pytest.fixture(scope="module")
def data():
    return _Data()


def _check_rows(pairs, flags: int, got, want, what: str):
    sha, md5, ends = got
    w_sha, w_md5, w_ends = want
    assert np.array_equal(ends, w_ends), f"{what}: lengths differ from the oracle"
    for name, g, w in (("sha256", sha, w_sha), ("md5", md5, w_md5)):
        if g is None:
            continue
        bad = np.flatnonzero((g != w).any(axis=1))
        rows = ", ".join(f"#{i} start {pairs[i][0]} 2^29{int(w_ends[i]) - HI:+d} B (high word {bit_count_high(int(w_ends[i]))})"
                         for i in bad[:8])
        assert bad.size == 0, f"{what}: {bad.size} of {len(pairs)} {name} rows differ from the oracle: {rows}"


def _hash_device(ctx, data: _Data, pairs, flags: int):
    """``pairs`` through b200h_hash_batch_device_hl -> ((sha | None, md5 | None, lengths), launches made)."""
    import torch

    n = len(pairs)
    offs = np.array([s for s, _ in pairs], np.uint64)
    lens = np.array([ln for _, ln in pairs], np.uint64)
    d_off = torch.from_numpy(offs.astype(np.int64)).cuda()
    d_len = torch.from_numpy(lens.astype(np.int64)).cuda()
    sha = torch.empty((n, 32), dtype=torch.uint8, device="cuda") if flags & SHA else None
    md5 = torch.empty((n, 16), dtype=torch.uint8, device="cuda") if flags & MD5 else None
    trimmed = torch.empty(n, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    l0 = ctx.launch_count
    ctx.hash_batch_device(data.dev.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), n, flags,
                          0 if sha is None else sha.data_ptr(), 0 if md5 is None else md5.data_ptr(), trimmed.data_ptr(),
                          torch.cuda.current_stream().cuda_stream, h_lengths=lens)
    torch.cuda.synchronize()
    launches = ctx.launch_count - l0
    return (None if sha is None else sha.cpu().numpy(), None if md5 is None else md5.cpu().numpy(),
            trimmed.cpu().numpy().astype(np.uint64)), launches


def _cycled(pairs, n: int):
    return [pairs[i % len(pairs)] for i in range(n)]


# ---------------------------------------------------------------------------------------------- chain kernel


@pytest.mark.parametrize("flags", [SHA, MD5, BOTH, BOTH | TRIM], ids=["sha256", "md5", "both", "both_trim"])
def test_chain_kernel_final_blocks_batch_route(data, flags):
    """2 S + 7 messages of 2^29 + d bytes, all routed to the chain kernel: more than one message group per chain CTA,
    groups with high words 0 and 1 side by side, misaligned starts, and (TRIM) zero tails scanned off."""
    sm = _sm_count()
    n = 2 * sm + 7
    pairs = _cycled(ALL, n)
    lens = np.array([ln for _, ln in pairs], np.uint64)
    seen = np.array([data.trimmed[p] for p in pairs], np.uint64) if flags & TRIM else lens
    assert _lib.plan_preview(seen, flags & BOTH, sm) == (n, 0)
    ctx = _lib.Context(0, pinned_bytes=16 << 20, device_bytes=64 << 20)
    try:
        got, launches = _hash_device(ctx, data, pairs, flags)
        assert ctx.last_outlier_count == n
        assert launches == (2 if flags & TRIM else 0) + 3 + 1, launches  # trim, plan, one chain launch, no lane launch
    finally:
        ctx.close()
    _check_rows(pairs, flags, got, data.expect(pairs, flags), f"chain batch, flags {flags}")


def test_chain_kernel_final_blocks_production_route(data, tmp_path, monkeypatch):
    """The library's default staging (8 GiB of device memory: 4 GiB wave slots), so a message of 512 MiB and more is
    hashed whole on the chain kernel, final block included: ``hash_batch_host`` from pageable and from page-locked
    memory, ``hash_files`` (mounts, volumefs1 uploads), and ``get_file_upload_specs``, the batched route of
    ``Volume.batch_upload`` and ``Mount``."""
    from modal_client_b200 import _backend, blob_utils

    pairs = [(0, HI - 8), (1, HI), (7, HI + 57), (15, HI + 64 * 33 + 55), (1, HI + 56)]
    offs = np.array([s for s, _ in pairs], np.uint64)
    lens = np.array([ln for _, ln in pairs], np.uint64)
    want = data.expect(pairs, BOTH)
    files = [(tmp_path / "a.bin", (7, HI + 57)), (tmp_path / "b.bin", (0, HI - 8))]
    for path, (s, ln) in files:
        with open(path, "wb") as f:
            f.write(memoryview(data.host)[s : s + ln])
    ctx = _lib.Context(0)
    try:
        got = ctx.hash_batch_host(data.host, offs, lens, BOTH)
        assert ctx.last_outlier_count == len(pairs)  # one wave, every message whole on the chain kernel
        _check_rows(pairs, BOTH, got, want, "hash_batch_host, pageable")

        pinned = ctx.host_alloc(BUF)
        try:
            pinned[:] = data.host
            got = ctx.hash_batch_host(pinned, offs, lens, BOTH)
            assert ctx.last_outlier_count == len(pairs)
            _check_rows(pairs, BOTH, got, want, "hash_batch_host, page-locked")
        finally:
            ctx.host_free(pinned)

        fpairs = [p for _, p in files]
        got = ctx.hash_files([str(p) for p, _ in files], [ln for _, ln in fpairs], 0, BOTH)
        assert ctx.last_outlier_count == len(files)
        _check_rows(fpairs, BOTH, got, data.expect(fpairs, BOTH), "hash_files")

        monkeypatch.setattr(_backend, "_override", ctx)
        (spec,) = blob_utils.get_file_upload_specs([(files[0][0], "big.bin", None)])
        assert ctx.last_outlier_count == 1
        sha, md5 = data.digests[files[0][1]]
        assert spec.size == HI + 57 and spec.use_blob
        assert spec.sha256_hex == sha.hex()
        assert spec.size <= blob_utils.MULTIPART_UPLOAD_THRESHOLD and spec.md5_hex == md5.hex()
    finally:
        monkeypatch.undo()
        ctx.close()


# ----------------------------------------------------------------------------------------------- lane kernel

LANE_CASES = {
    # id: (flags, B200H_NO_SPARSE)
    "sparse_sha256": (SHA, False),
    "md5": (MD5, False),
    "sparse_fused": (BOTH, False),
    "dense_sha256": (SHA, True),
    "dense_fused": (BOTH, True),
}


@pytest.mark.parametrize("case", list(LANE_CASES))
def test_lane_final_blocks(data, monkeypatch, case):
    """8 S + 44 messages cycled from the 44 (start, length) pairs of M, kept on the lane kernel (NO_OUTLIERS): the sparse
    launch shape (4 S warps of up to three live lanes) on the sparse bodies, MD5 alone, or (B200H_NO_SPARSE, read at every
    launch) the dense bodies.  Every length but 2^29 - 72 falls into one planner bucket, in which the queue keeps runs of
    32 consecutive batch entries in batch order (the plan kernel's warp-aggregated scatter), and a warp's lanes take
    consecutive queue entries.  So warps hold neighbouring pairs of M, whose high words are 0 (d = -8, -1) and 1
    (d >= 0) side by side: a body that took one lane's high word for the whole warp would give wrong digests."""
    flags, no_sparse = LANE_CASES[case]
    if no_sparse:
        monkeypatch.setenv("B200H_NO_SPARSE", "1")
    else:
        monkeypatch.delenv("B200H_NO_SPARSE", raising=False)
    sm = _sm_count()
    n = 8 * sm + len(M)
    assert 4 * sm < n <= 128 * sm and -(-n // (4 * sm)) == 3  # sparse launch shape: 4 S warps of up to 3 lanes
    pairs = _cycled(M, n)
    assert warps_mixing_high_words(pairs, 3) >= n // 30
    lens = np.array([ln for _, ln in pairs], np.uint64)
    assert _lib.plan_preview(lens, flags | NO_OUT, sm) == (0, 0)
    ctx = _lib.Context(0, pinned_bytes=16 << 20, device_bytes=64 << 20)
    try:
        got, launches = _hash_device(ctx, data, pairs, flags | NO_OUT)
        assert ctx.last_outlier_count == 0
        assert launches == 3 + 1, launches  # plan, one lane launch
    finally:
        ctx.close()
    _check_rows(pairs, flags, got, data.expect(pairs, flags), f"lane batch {case}")


# ---------------------------------------------------------------------------------------------------- streams

STREAM_CAP = 4 << 20  # default bytes per absorb (B200H_STREAM_BUF)
# digests() at these totals: 4 MiB - 8 B in the buffer (chain), exactly 2^32 bits (the digest resumes a zero-byte
# message on a lane), 57 B (lane), 70 000 B (chain), 2^32 - 1 B (chain, high word 7), then prior_bytes with a non-zero
# high half: 1 B (lane) and 70 056 B (chain)
CHECKPOINTS = (HI - 8, HI, HI + 57, HI + 70_000, (1 << 32) - 1, (1 << 32) + 1, (1 << 32) + 70_056)
CHUNK = 64 << 20  # the synthetic bytes are generated this much at a time
PIECES = (1, 4093, STREAM_CAP + 3, 65_536, (7 << 20) - 1, 123_457, 64, (3 << 20) + 1001, 55, 15 << 20)  # update sizes


def stream_pieces(checkpoints=CHECKPOINTS, chunk: int = CHUNK, pieces=PIECES):
    """(offset, length, is_checkpoint) of every update of the stream tests: the sizes of ``pieces`` in turn, cut at every
    chunk edge and every checkpoint, up to the last checkpoint."""
    total, i = 0, 0
    cps = list(checkpoints)
    while cps:
        ln = min(pieces[i % len(pieces)], cps[0] - total, chunk - total % chunk)
        i += 1
        yield total, ln, total + ln == cps[0]
        total += ln
        if total == cps[0]:
            cps.pop(0)


def finishes_on_chain(total: int, cap: int = STREAM_CAP) -> bool:
    """Whether digests() after ``total`` bytes hands its final message (what is left in the buffer) to the chain
    kernel: that message is a single one of at least kChainMinBlocks blocks."""
    return ((total % cap) >> 6) + 1 >= CHAIN_MIN_BLOCKS


def _feed_stream(ctx, flags: int, seed: int) -> list:
    """One stream of ``flags`` on ``ctx`` over stream_pieces(); at every checkpoint digests() is compared with hashlib
    and the kernel that finished it is checked.  -> the checkpoints reached."""
    st = ctx.stream(flags)
    hs, hm = hashlib.sha256(), hashlib.md5()
    reached, chunk, chunk_at = [], None, -1
    try:
        for off, ln, cp in stream_pieces():
            if off // CHUNK != chunk_at:
                chunk_at = off // CHUNK
                chunk = synth_array(seed, CHUNK, chunk_at * CHUNK)
            piece = chunk[off % CHUNK : off % CHUNK + ln]
            st.update(piece)
            if flags & SHA:
                hs.update(piece)
            if flags & MD5:
                hm.update(piece)
            if not cp:
                continue
            total = off + ln
            s, m = st.digests()
            chain = finishes_on_chain(total)
            assert ctx.last_outlier_count == int(chain), (flags, total)
            assert s == (hs.digest() if flags & SHA else None), f"flags {flags}: sha256 after {total} B ({'chain' if chain else 'lane'})"
            assert m == (hm.digest() if flags & MD5 else None), f"flags {flags}: md5 after {total} B ({'chain' if chain else 'lane'})"
            reached.append(total)
    finally:
        st.close()
    return reached


def test_streams_past_4gib(monkeypatch):
    """SHA-256 alone, MD5 alone and both, each on a context of its own (so that ``last_outlier_count`` belongs to its
    thread), fed the same ~4 GiB of synthetic bytes concurrently, uneven update sizes: digests() against hashlib after
    2^29 and 2^32 bytes, finished on the chain kernel (>= 64 KiB in the buffer) or on a lane."""
    for k in ("B200H_CHAIN", "B200H_STREAM_BUF", "B200H_NO_SPARSE"):  # fixed before the threads start, never toggled
        monkeypatch.delenv(k, raising=False)
    assert [finishes_on_chain(t) for t in CHECKPOINTS] == [True, False, False, True, True, False, True]
    ctxs = [_lib.Context(0, pinned_bytes=16 << 20, device_bytes=64 << 20) for _ in range(3)]
    try:
        with ThreadPoolExecutor(3) as ex:
            futs = [ex.submit(_feed_stream, c, f, 93) for c, f in zip(ctxs, (SHA, MD5, BOTH))]
            reached = [f.result() for f in futs]
    finally:
        for c in ctxs:
            c.close()
    assert reached == [list(CHECKPOINTS)] * 3


def test_md5_base64_of_a_512mib_stream(data, gpu_backend):
    """hash_utils.get_md5_base64 over a BytesIO of 2^29 + 57 bytes (get_md5_base64 / BytesIOSegmentPayload on an
    object of 512 MiB or more): 4 MiB absorbs on the chain kernel, then the last 57 bytes on the MD5-only lane body
    with high word 1."""
    from modal_client_b200 import hash_utils

    s, ln = 1, HI + 57
    assert not finishes_on_chain(ln) and bit_count_high(ln) == 1
    got = hash_utils.get_md5_base64(io.BytesIO(data.host[s : s + ln].tobytes()))
    assert gpu_backend.last_outlier_count == 0
    assert got == base64.b64encode(data.digests[(s, ln)][1]).decode("ascii")
