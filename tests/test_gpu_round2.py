"""GPU: parity and behaviour of the round-2 native work -- host-side outlier plan (no read-back), wide zero-trim
scan, combining queue for concurrent small callers, concurrent digest streams, device-resident outputs, >= 4 GiB
single messages.  Everything goes through the C ABI and is checked against the oracle / hashlib."""
import hashlib
import os
import threading

import numpy as np
import pytest

from modal_client_b200 import _lib
from modal_client_b200.synth import synth_array, synth_bytes
from oracle import c_oracle

pytestmark = pytest.mark.gpu

BOTH = _lib.SHA256 | _lib.MD5


@pytest.fixture(scope="module")
def ctx():
    os.environ["B200H_VERIFY_PLAN"] = "1"  # every host-side outlier count is cross-checked against the device's
    c = _lib.Context(0, pinned_bytes=64 << 20, device_bytes=512 << 20)
    os.environ.pop("B200H_VERIFY_PLAN")
    yield c
    c.close()


@pytest.fixture(scope="module")
def plain_ctx():
    c = _lib.Context(0, pinned_bytes=64 << 20, device_bytes=512 << 20)
    yield c
    c.close()


def _layout(lens, gap=7, lead=0):
    lens = np.asarray(lens, np.uint64)
    offs = (np.concatenate([[0], np.cumsum(lens + np.uint64(gap))])[:-1] + lead).astype(np.uint64)
    return offs, lens


# ------------------------------------------------------------------------------------- outlier plan on the host


def test_host_outlier_plan_equals_device_plan(ctx):
    """plan_outliers_host (used instead of reading qctl[3] back) must select exactly what plan_scan_kernel selects;
    with B200H_VERIFY_PLAN=1 the library fails the call on any disagreement.  Digests are checked as well."""
    rng = np.random.default_rng(42)
    shapes = [
        [3 << 20] + [5000] * 3000,
        [3 << 20, (3 << 20) - 4097, 1 << 20] + [70_000] * 500,
        [1 << 20] * 40,
        [100_000] * 2000,
        [80 * 1024] * 700,
        [2 << 20], [100], [0], [65536], [65535], [65536 - 64],
        [1 << 16] * 528, [1 << 16] * 529,                # either side of the chain cap (4 per SM on 132 SMs)
        [3 << 20] * 344 + [1 << 20] * 995,               # more outlier candidates than 3/4 of the SMs in a mixed batch: none routed
        [16 << 20] * 200 + [100] * 10,                   # ... unless next to nothing is left for the lanes
        [8 << 20] * 3 + [1 << 20] * 200 + [3000] * 20000,  # chain + long lane queue + short lane queue
        list(rng.integers(0, 300_000, 900)) + [9 << 20],
        list((rng.lognormal(10, 2.0, 1500)).astype(np.int64) % (6 << 20)),
    ]
    for lens in shapes:
        offs, lens = _layout(lens)
        buf = synth_array(31, int(offs[-1] + lens[-1]) + 8)
        sha, md5, _ = ctx.hash_batch_host(buf, offs, lens, BOTH)
        s, m, _ = c_oracle.hash_batch(buf, offs, lens)
        assert np.array_equal(sha, s) and np.array_equal(md5, m)


def test_long_lane_messages_get_their_own_packed_launch(ctx):
    """Mixed batch: 3 outliers (chain kernel), 100 long messages below half of the longest (they stay on lanes but in
    their own queue: a second, lane-packed launch), 20 000 short ones.  Host plan == device plan (B200H_VERIFY_PLAN),
    digests exact, and the launch list shows both lane launches."""
    offs, lens = _layout([8 << 20] * 3 + [(1 << 20) + 64 * i for i in range(100)] + [3000 + (i % 977) for i in range(20000)])  # one staging wave
    buf = synth_array(36, int(offs[-1] + lens[-1]) + 8)
    l0 = ctx.launch_count
    sha, md5, _ = ctx.hash_batch_host(buf, offs, lens, BOTH)
    assert ctx.last_outlier_count == 3
    assert ctx.launch_count - l0 == 3 + 1 + 2  # plan x3, chain, lane (short), lane (long)
    s, m, _ = c_oracle.hash_batch(buf, offs, lens)
    assert np.array_equal(sha, s) and np.array_equal(md5, m)
    # outlier routing off: the long queue then holds the 8 MiB messages too
    l0 = ctx.launch_count
    sha, md5, _ = ctx.hash_batch_host(buf, offs, lens, BOTH | _lib.NO_OUTLIERS)
    assert ctx.last_outlier_count == 0 and ctx.launch_count - l0 == 3 + 2
    assert np.array_equal(sha, s) and np.array_equal(md5, m)


def test_device_batch_only_enqueues_with_host_lengths_or_no_outliers(plain_ctx):
    import torch

    ctx = plain_ctx
    dev = torch.device("cuda:0")
    lens = np.array([3 << 20] + [40_000] * 2000, np.uint64)  # one outlier
    offs = (np.arange(lens.size, dtype=np.uint64) * np.uint64(3 << 20))[: lens.size]
    offs = np.concatenate([[0], np.cumsum(lens)])[:-1].astype(np.uint64)
    total = int(lens.sum())
    data = torch.empty(total, dtype=torch.uint8, device=dev)
    ctx.fill_synth_device(data.data_ptr(), total, seed=5)
    d_off = torch.from_numpy(offs.astype(np.int64)).to(dev)
    d_len = torch.from_numpy(lens.astype(np.int64)).to(dev)
    outs = []
    st = torch.cuda.current_stream().cuda_stream
    syncs0 = ctx.plan_sync_count
    for kw, flags in (({"h_lengths": lens}, BOTH), ({}, BOTH | _lib.NO_OUTLIERS)):
        sha = torch.empty((lens.size, 32), dtype=torch.uint8, device=dev)
        md5 = torch.empty((lens.size, 16), dtype=torch.uint8, device=dev)
        ctx.hash_batch_device(data.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), lens.size, flags, sha.data_ptr(),
                              md5.data_ptr(), 0, st, **kw)
        outs.append((sha, md5))
    assert ctx.plan_sync_count == syncs0, "the call read the outlier count back although it did not have to"
    assert ctx.last_outlier_count == 0  # the NO_OUTLIERS batch
    sha = torch.empty((lens.size, 32), dtype=torch.uint8, device=dev)
    md5 = torch.empty((lens.size, 16), dtype=torch.uint8, device=dev)
    ctx.hash_batch_device(data.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), lens.size, BOTH, sha.data_ptr(),
                          md5.data_ptr(), 0, st)
    assert ctx.plan_sync_count == syncs0 + 1 and ctx.last_outlier_count == 1
    torch.cuda.synchronize()
    host = data.cpu().numpy()
    s, m, _ = c_oracle.hash_batch(host, offs, lens)
    for a, b in outs + [(sha, md5)]:
        assert np.array_equal(a.cpu().numpy(), s) and np.array_equal(b.cpu().numpy(), m)


def test_host_batch_writes_device_outputs(plain_ctx):
    """sha/md5/trimmed outputs of b200h_hash_batch_host may be DEVICE memory (the table a rank all-gathers next)."""
    import torch

    ctx = plain_ctx
    offs, lens = _layout([0, 1, 64, 4096, 300_001, 65536])
    buf = synth_array(33, int(offs[-1] + lens[-1]) + 8)
    dev = torch.device("cuda:0")
    tab = torch.zeros(lens.size * 48, dtype=torch.uint8, device=dev)
    trimmed = torch.zeros(lens.size, dtype=torch.int64, device=dev)
    r = ctx.hash_batch_host(buf, offs, lens, BOTH, out_sha=tab.data_ptr(), out_md5=tab.data_ptr() + 32 * lens.size,
                            out_trimmed=trimmed.data_ptr())
    assert r == (None, None, None)
    s, m, _ = c_oracle.hash_batch(buf, offs, lens)
    t = tab.cpu().numpy()
    assert np.array_equal(t[: 32 * lens.size].reshape(-1, 32), s)
    assert np.array_equal(t[32 * lens.size :].reshape(-1, 16), m)
    assert np.array_equal(trimmed.cpu().numpy().astype(np.uint64), lens)


def test_sparse_selection_from_pinned_memory_is_gathered(plain_ctx):
    """One rank's interleaved shard of a page-locked buffer: only the selected messages may be copied (the wave
    buffers here are far too small to hold the span with its gaps, which the old direct path would have DMA'd)."""
    ctx = plain_ctx
    n, size = 512, 1 << 20
    pinned = ctx.host_alloc(n * size)
    try:
        pinned[:] = synth_array(34, n * size)
        sel = np.arange(3, n, 8)
        offs = (sel * size).astype(np.uint64)
        lens = np.full(sel.size, size - 5, np.uint64)
        sha, md5, _ = ctx.hash_batch_host(pinned, offs, lens, BOTH)
        s, m, _ = c_oracle.hash_batch(pinned, offs, lens)
        assert np.array_equal(sha, s) and np.array_equal(md5, m)
    finally:
        ctx.host_free(pinned)


# --------------------------------------------------------------------------------------------------- wide trim


def test_trim_long_zero_runs_take_the_wide_scan(ctx):
    """Messages whose zero tail is far longer than the probe warp settles (16 KiB): blank blocks, a lone non-zero
    byte at every kind of position (chunk borders, unaligned head, first byte), unaligned starts and ends."""
    rng = np.random.default_rng(3)
    C = 512 * 1024
    sizes = [8 << 20, (8 << 20) - 3, 3 * C, 3 * C + 17, C + 16384, 2 * C, 300_000, 262144 + 16384 + 2048, 5 << 20, 1 << 20]
    cases = []
    for sz in sizes:
        for last in (None, 0, 1, 15, 16, 17, C - 1, C, C + 1, sz - C - 1, sz - C, sz - C + 1, sz - 16385 - 2048, sz // 2,
                     sz - 20000, int(rng.integers(0, sz))):
            if last is None or 0 <= last < sz:
                cases.append((sz, last))
    lens = np.array([c[0] for c in cases], np.uint64)
    offs, lens = _layout(lens, gap=13, lead=5)
    buf = np.zeros(int(offs[-1] + lens[-1]) + 32, np.uint8)
    for (sz, last), o in zip(cases, offs):
        if last is not None:
            # random bytes up to and including `last` for some, a lone byte for others
            if last % 3 == 0:
                buf[int(o) + last] = 0x5A
            else:
                seg = synth_array(1000 + last % 97, last + 1).copy()
                seg[-1] |= 1
                buf[int(o) : int(o) + last + 1] = seg
    sha, md5, trimmed = ctx.hash_batch_host(buf, offs, lens, BOTH | _lib.TRIM_ZEROS)
    s, m, e = c_oracle.hash_batch(buf, offs, lens, trim=True)
    want = np.array([0 if c[1] is None else c[1] + 1 for c in cases], np.uint64)
    assert np.array_equal(e, want)
    assert np.array_equal(trimmed, e)
    assert np.array_equal(sha, s) and np.array_equal(md5, m)


def test_trim_blank_blocks_fixed_parts(ctx):
    """volumefs2 shape: a 40 MiB stream of 8 MiB blocks -- blank, half blank, full -- through b200h_hash_fixed_parts."""
    bs = 8 << 20
    data = np.zeros(5 * bs - 12345, np.uint8)
    data[bs : bs + (3 << 20)] = synth_array(8, 3 << 20) | 1       # block 1: 3 MiB of data then zeros
    data[3 * bs : 4 * bs] = synth_array(9, bs) | 1                # block 3: full
    data[4 * bs + 100] = 7                                        # block 4 (short): one byte near its start
    sha, _, trimmed, _ = ctx.hash_fixed_parts(data, bs, _lib.SHA256 | _lib.TRIM_ZEROS)
    assert list(map(int, trimmed)) == [0, 3 << 20, 0, bs, 101]
    for i, t in enumerate(trimmed):
        assert sha[i].tobytes() == hashlib.sha256(data[i * bs : i * bs + int(t)]).digest()


# --------------------------------------------------------------------------------------------- combining queue


def test_concurrent_single_message_callers_share_batches(plain_ctx):
    """16 threads x 40 one-message calls, plus a second context hammered at the same time: every caller gets its own
    digests, and the combining queue turns the calls into far fewer GPU batches."""
    ctx = plain_ctx
    ctx2 = _lib.Context(0, pinned_bytes=8 << 20, device_bytes=64 << 20)
    payloads = [synth_bytes(500 + i, 1 + (i * 7919) % 200_000) for i in range(64)]
    want = [(hashlib.sha256(p).digest(), hashlib.md5(p).digest()) for p in payloads]
    errors = []
    g0, r0 = ctx.combine_stats()
    launches0 = ctx.launch_count

    def worker(tid, c):
        try:
            for k in range(40):
                i = (tid * 13 + k * 5) % len(payloads)
                flags = BOTH if (tid + k) % 3 else _lib.SHA256
                sha, md5, _ = c.hash_buffers([payloads[i]], flags)
                assert sha[0].tobytes() == want[i][0]
                if flags & _lib.MD5:
                    assert md5[0].tobytes() == want[i][1]
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))

    threads = [threading.Thread(target=worker, args=(t, ctx if t < 16 else ctx2)) for t in range(24)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    ctx2.close()
    assert not errors, errors[:3]
    g, r = ctx.combine_stats()
    assert r - r0 == 16 * 40
    assert (g - g0) * 4 <= r - r0, f"{r - r0} calls were served by {g - g0} GPU batches"
    assert ctx.launch_count - launches0 <= 8 * (g - g0)


def test_concurrent_streams_and_batches(plain_ctx):
    """8 digest streams fed from 8 threads (each on its own CUDA stream) while the main thread runs host batches:
    the thread-safety the ABI promises (promoted from tools/stress.py)."""
    ctx = plain_ctx
    datas = [synth_bytes(700 + i, (5 << 20) + 4099 * i + 1) for i in range(8)]
    want = [(hashlib.sha256(d).digest(), hashlib.md5(d).digest()) for d in datas]
    errors = []

    def feed(i):
        try:
            st = ctx.stream(BOTH)
            pos, step = 0, 1 + 65536 * (i + 1)
            while pos < len(datas[i]):
                st.update(datas[i][pos : pos + step])
                pos += step
                if i == 3 and pos < (2 << 20):  # digest() is non-destructive, mid-stream too
                    s, _ = st.digests()
                    assert s == hashlib.sha256(datas[i][:pos]).digest()
            assert st.digests() == want[i]
            st.reset()
            st.update(b"abc")
            assert st.digests()[0] == hashlib.sha256(b"abc").digest()
            st.close()
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))

    threads = [threading.Thread(target=feed, args=(i,)) for i in range(8)]
    for t in threads:
        t.start()
    offs, lens = _layout([100_000] * 300)
    buf = synth_array(35, int(offs[-1] + lens[-1]) + 8)
    s, m, _ = c_oracle.hash_batch(buf, offs, lens)
    for _ in range(5):
        sha, md5, _ = ctx.hash_batch_host(buf, offs, lens, BOTH)
        assert np.array_equal(sha, s) and np.array_equal(md5, m)
    for t in threads:
        t.join()
    assert not errors, errors[:3]


# ------------------------------------------------------------------------------------------- >= 4 GiB messages


def test_single_message_of_4gib_plus_1(plain_ctx):
    """One message whose LENGTH (not just its offset) needs more than 32 bits: 4 GiB + 1 B through the host entry
    point (segmented over the staging waves, chaining state on the device), against hashlib."""
    n = (4 << 30) + 1
    data = synth_array(77, n)
    sha, md5, trimmed = plain_ctx.hash_batch_host(data, [0], [n], BOTH)
    assert int(trimmed[0]) == n
    assert sha[0].tobytes() == hashlib.sha256(data).digest()
    assert md5[0].tobytes() == hashlib.md5(data).digest()


# ------------------------------------------------------------------------------------- hex columns (B200H_HEX_OUT)


def test_hex_columns_formatted_on_the_device(plain_ctx, tmp_path):
    """The digest columns as lowercase ASCII hex (the text MountFile.sha256_hex / FileUploadSpec.md5_hex carry), from
    the host entry point, the file reader and the device entry point."""
    import torch

    ctx = plain_ctx
    offs, lens = _layout([0, 1, 55, 64, 4096, 300_001, 65536, 200_000])
    buf = synth_array(41, int(offs[-1] + lens[-1]) + 8)
    want_sha = [hashlib.sha256(buf[int(o) : int(o + n)]).hexdigest() for o, n in zip(offs, lens)]
    want_md5 = [hashlib.md5(buf[int(o) : int(o + n)]).hexdigest() for o, n in zip(offs, lens)]
    sha, md5, _ = ctx.hash_batch_host(buf, offs, lens, BOTH | _lib.HEX_OUT)
    assert sha.shape == (len(lens), 64) and md5.shape == (len(lens), 32)
    assert [r.tobytes().decode() for r in sha] == want_sha and [r.tobytes().decode() for r in md5] == want_md5
    sha, md5, _ = ctx.hash_batch_host(buf, offs, lens, _lib.SHA256 | _lib.HEX_OUT)
    assert md5 is None and [r.tobytes().decode() for r in sha] == want_sha
    paths = []
    for i, (o, n) in enumerate(zip(offs, lens)):
        p = tmp_path / f"f{i}"
        buf[int(o) : int(o + n)].tofile(p)
        paths.append(str(p))
    sizes, _ = ctx.stat_files(paths)
    sha, md5, _ = ctx.hash_files(paths, sizes, 0, BOTH | _lib.HEX_OUT)
    assert [r.tobytes().decode() for r in sha] == want_sha and [r.tobytes().decode() for r in md5] == want_md5
    dev = torch.device("cuda:0")
    d = torch.from_numpy(buf).to(dev)
    d_off = torch.from_numpy(offs.astype(np.int64)).to(dev)
    d_len = torch.from_numpy(lens.astype(np.int64)).to(dev)
    h_sha = torch.zeros((len(lens), 64), dtype=torch.uint8, device=dev)
    h_md5 = torch.zeros((len(lens), 32), dtype=torch.uint8, device=dev)
    ctx.hash_batch_device(d.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), len(lens), BOTH | _lib.HEX_OUT, h_sha.data_ptr(),
                          h_md5.data_ptr(), 0, torch.cuda.current_stream().cuda_stream, h_lengths=lens)
    torch.cuda.synchronize()
    assert [bytes(r).decode() for r in h_sha.cpu().numpy()] == want_sha
    assert [bytes(r).decode() for r in h_md5.cpu().numpy()] == want_md5


def test_small_lane_grid_next_to_chain_ctas_loses_nothing(plain_ctx):
    """Regression (round 2): a handful of long parts on the chain kernel plus ONE short message on a one-CTA lane launch --
    the multipart shape 5 x 1 MiB + 123 B.  A lane CTA must never step aside for a chain CTA unless other lane CTAs are
    guaranteed to exist; repeated because CTA placement is not deterministic."""
    offs, lens = _layout([1 << 20] * 5 + [123])
    buf = synth_array(37, int(offs[-1] + lens[-1]) + 8)
    s, m, _ = c_oracle.hash_batch(buf, offs, lens)
    for flags in (BOTH, _lib.MD5, _lib.SHA256):
        for _ in range(15):
            sha, md5, _ = plain_ctx.hash_batch_host(buf, offs, lens, flags)
            assert sha is None or np.array_equal(sha, s)
            assert md5 is None or np.array_equal(md5, m)
