"""GPU: b200h_copy_ranges_to_host is byte-exact for every source phase, segment shape and range edge, writes nothing
outside its destinations, launches one kernel per call and only enqueues; staged views of DeviceFile.safetensors /
DeviceFile.torch_save blocks equal the serialised images; a staged volumefs2 upload lets the tensors go at
``device_released``."""
import asyncio
import hashlib
import io
import types

import numpy as np
import pytest

from modal_client_b200 import DeviceFile, _lib, blob_utils, stage_ranges, volume
from tests.test_device_file_cpu import _volume_server

pytestmark = pytest.mark.gpu

MiB = 1 << 20
SENTINEL = 0xC3


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0, pinned_bytes=64 << 20, device_bytes=512 << 20)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pinned(ctx):
    buf = ctx.host_alloc(192 * MiB)
    yield buf
    ctx.host_free(buf)


def _random_bytes(n, seed):
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, 256, (max(n, 1),), dtype=torch.uint8, device="cuda", generator=g)[:n]


def _layout(lens, gap=128):
    """128-byte aligned destinations with ``gap`` untouched bytes between them and at both ends."""
    offsets, at = [], gap
    for n in lens:
        offsets.append(at)
        at += -(-n // 128) * 128 + gap
    return offsets, at


def _copy_and_check(ctx, pinned, segs, first, ranges, images, stream=0):
    """One call; every range equals the slice of its file's host image, every other byte of the buffer is untouched."""
    import torch

    offsets, total = _layout([n for _, _, n in ranges])
    assert total <= pinned.size
    dst = pinned[:total]
    dst[:] = SENTINEL
    launches, syncs = ctx.launch_count, ctx.plan_sync_count
    ctx.copy_ranges_to_host([s.data_ptr() if s.numel() else 0 for s in segs], [s.numel() for s in segs], first, ranges,
                            dst, offsets, stream)
    assert ctx.launch_count - launches == (1 if any(n for _, _, n in ranges) else 0)
    assert ctx.plan_sync_count == syncs
    torch.cuda.synchronize()
    untouched = np.ones(total, bool)
    for (f, off, n), at in zip(ranges, offsets):
        assert np.array_equal(dst[at : at + n], images[f][off : off + n]), (f, off, n)
        untouched[at : at + n] = False
    assert (dst[untouched] == SENTINEL).all()


SEG_LENS = [0, 1, 15, 16, 17, 63, 64, 65, 4095, 4096, 4097, MiB - 1, MiB, MiB + 1, 9 * MiB]


@pytest.mark.parametrize("phase", range(16))
def test_every_source_phase_and_segment_length(ctx, pinned, phase):
    """One file per segment length, each segment starting ``phase`` bytes behind a 256-byte boundary; the whole file
    and a range with odd edges of each."""
    pool = _random_bytes(sum(-(-(n + 16) // 256) * 256 for n in SEG_LENS) + 256, 100 + phase)
    segs, at = [], 0
    for n in SEG_LENS:
        segs.append(pool[at + phase : at + phase + n])
        at += -(-(n + 16) // 256) * 256
    images = [s.cpu().numpy() for s in segs]
    ranges = [(f, 0, n) for f, n in enumerate(SEG_LENS)]
    ranges += [(f, min(3, n), max(0, n - 8)) for f, n in enumerate(SEG_LENS)]
    _copy_and_check(ctx, pinned, segs, list(range(len(segs) + 1)), ranges, images)


def test_ranges_start_and_end_at_every_residue(ctx, pinned):
    seg = _random_bytes(70_000, 7)[5:]
    image = seg.cpu().numpy()
    ranges = [(0, 1000 + a, 66_000 + b - a) for a in range(16) for b in range(16)]
    _copy_and_check(ctx, pinned, [seg], [0, 1], ranges, [image])


def test_ranges_over_hundreds_of_tiny_segments_and_empty_ones(ctx, pinned):
    rng = np.random.default_rng(3)
    pool = _random_bytes(1 << 20, 11)
    segs, at = [], 0
    for i in range(900):
        n = 0 if i % 7 == 3 else int(rng.integers(1, 40)) if i % 50 else 70_000
        start = at + int(rng.integers(0, 16))
        segs.append(pool[start : start + n])
        at = start + n
    image = np.concatenate([s.cpu().numpy() for s in segs])
    size = image.size
    ranges = [(0, 0, size), (0, 17, size - 40), (0, size - 1, 1), (0, size, 0), (0, 5, 0)]
    ranges += [(0, int(o), int(n)) for o, n in zip(rng.integers(0, size - 9000, 40), rng.integers(1, 9000, 40))]
    _copy_and_check(ctx, pinned, segs, [0, len(segs)], ranges, [image])
    _copy_and_check(ctx, pinned, segs, [0, len(segs)], [(0, 9, 0), (0, size, 0)], [image])  # all empty: no launch


def test_ten_thousand_ranges_in_one_call(ctx, pinned):
    rng = np.random.default_rng(5)
    a, b = _random_bytes(6 * MiB, 21)[3:], _random_bytes(MiB, 22)[9:]
    segs = [a[: 2 * MiB], a[2 * MiB :], b]
    images = [a.cpu().numpy(), b.cpu().numpy()]
    ranges = []
    for _ in range(10_000):
        f = int(rng.integers(0, 2))
        n = int(rng.integers(0, 3000))
        ranges.append((f, int(rng.integers(0, images[f].size - n)), n))
    _copy_and_check(ctx, pinned, segs, [0, 2, 3], ranges, images)


def test_one_range_larger_than_4gib(ctx):
    import torch

    n = (4 << 30) + 12_345
    if torch.cuda.mem_get_info(0)[0] < n + (2 << 30):
        pytest.skip("not enough free device memory")
    try:
        dst = ctx.host_alloc(n + 256)
    except _lib.B200HashError:
        pytest.skip("not enough page-lockable host memory")
    try:
        src = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
        ctx.fill_synth_device(src.data_ptr(), (n + 16) // 8 * 8, seed=77, stream=1)
        seg = src[7 : 7 + n]
        dst[:128], dst[128 + n :] = SENTINEL, SENTINEL
        ctx.copy_ranges_to_host([seg.data_ptr()], [n], [0, 1], [(0, 0, n)], dst, [128], 1)
        torch.cuda.synchronize()
        assert (dst[:128] == SENTINEL).all() and (dst[128 + n :] == SENTINEL).all()
        for lo in (0, (4 << 30) - 5 * MiB, n - 3 * MiB):  # the start, across 2^32, the end
            hi = min(n, lo + 8 * MiB)
            assert np.array_equal(dst[128 + lo : 128 + hi], seg[lo:hi].cpu().numpy()), lo
    finally:
        ctx.host_free(dst)


def test_the_call_is_stream_ordered(ctx, pinned):
    """A kernel queued before the call on the same stream rewrites the source: the copy sees what it wrote."""
    import torch

    stream = torch.cuda.Stream()
    src = torch.zeros(32 * MiB + 5, dtype=torch.uint8, device="cuda")
    fresh = _random_bytes(32 * MiB + 5, 31)
    busy = torch.empty(64 * MiB, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    dst = pinned[: 33 * MiB]
    dst[:] = SENTINEL
    with torch.cuda.stream(stream):
        for _ in range(20):
            busy.normal_()  # keeps the stream busy while the host enqueues what follows
        src.copy_(fresh)
        ctx.copy_ranges_to_host([src.data_ptr()], [src.numel()], [0, 1], [(0, 3, src.numel() - 3)], dst, [256],
                                stream.cuda_stream)
    stream.synchronize()
    assert np.array_equal(dst[256 : 256 + src.numel() - 3], fresh[3:].cpu().numpy())


def test_bad_arguments_are_rejected_before_anything_is_enqueued(ctx, pinned):
    import torch

    seg = _random_bytes(4096, 41)
    host = torch.empty(4096, dtype=torch.uint8)
    pageable = np.zeros(8192, np.uint8)
    ok = dict(ptrs=[seg.data_ptr()], lens=[4096], first=[0, 1], ranges=[(0, 0, 100), (0, 200, 100)], dst=pinned,
              offsets=[0, 128])
    cases = {
        "foreign segment": dict(ptrs=[host.data_ptr()]),
        "NULL segment": dict(ptrs=[0]),
        "segment whose address range wraps": dict(lens=[2**64 - seg.data_ptr() + 16]),
        "pageable destination": dict(dst=pageable[-pageable.ctypes.data % 16 :][:4096]),
        "misaligned destination": dict(offsets=[0, 136]),
        "overlapping destinations": dict(offsets=[0, 96]),
        "destination out of bounds": dict(offsets=[0, pinned.size - 64]),
        "range past the end of its file": dict(ranges=[(0, 0, 100), (0, 4000, 97)]),
        "range of a file that does not exist": dict(ranges=[(1, 0, 1), (0, 0, 1)]),
        "file table that does not cover the segments": dict(first=[0, 0]),
    }
    pinned[:256] = SENTINEL
    for name, change in cases.items():
        a = {**ok, **change}
        launches = ctx.launch_count
        with pytest.raises(_lib.B200HashError, match=r"\(-1\)"):
            ctx.copy_ranges_to_host(a["ptrs"], a["lens"], a["first"], a["ranges"], a["dst"], a["offsets"])
        assert ctx.launch_count == launches, name
    torch.cuda.synchronize()
    assert (pinned[:256] == SENTINEL).all()
    ctx.copy_ranges_to_host(ok["ptrs"], ok["lens"], ok["first"], ok["ranges"], ok["dst"], ok["offsets"])
    torch.cuda.synchronize()
    assert np.array_equal(pinned[128:228], seg[200:300].cpu().numpy())


# ------------------------------------------------------------------------------------------- device files


def _state_dict(total, seed=0):
    """bf16 / f32 / u8 tensors of mixed sizes (odd byte counts included) adding up to about ``total`` bytes."""
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    sd, left, i = {}, total, 0
    sizes = [total // 3, total // 5, 12 * MiB + 6, 9 * MiB, 3 * MiB + 2, 70_001, 4099, 513, 64, 7, 1]
    while left > 0:
        n = min(left, sizes[i % len(sizes)])
        raw = torch.randint(0, 256, (n + 4,), dtype=torch.uint8, device="cuda", generator=g)
        if i % 3 == 0:
            raw[n // 2 :] = 0  # zero tails: trimmed blocks, blank blocks in the large tensors
        sd[f"t{i}"] = raw[: n // 2 * 2].view(torch.bfloat16) if i % 4 == 0 else \
            raw[: n // 4 * 4].view(torch.float32) if i % 4 == 1 else raw[:n]
        left -= n
        i += 1
    return sd


@pytest.mark.parametrize("kind", ["safetensors", "torch_save"])
def test_staged_blocks_of_a_device_file_equal_the_serialised_image(gpu_backend, kind):
    import torch
    from safetensors.torch import save

    sd = _state_dict(70 * MiB, seed=1)
    if kind == "safetensors":
        f, image = DeviceFile.safetensors(sd), save({k: v.cpu() for k, v in sd.items()})
    else:
        buf = io.BytesIO()
        torch.save(sd, buf)
        f, image = DeviceFile.torch_save(sd), buf.getvalue()
    assert f.nbytes == len(image)
    BS = blob_utils.BLOCK_SIZE
    _, _, trimmed = f.hash_parts(BS, _lib.SHA256 | _lib.TRIM_ZEROS)
    ranges = [(0, i * BS, int(t)) for i, t in enumerate(trimmed)]
    offsets, total = _layout([n for _, _, n in ranges])
    dst = gpu_backend.host_alloc(total)
    try:
        dst[:] = SENTINEL
        launches = gpu_backend.launch_count
        staged = stage_ranges([f], ranges, dst, offsets)
        staged.wait()
        assert gpu_backend.launch_count == launches + 1
        for i, (_, off, n) in enumerate(ranges):
            assert staged.view(i) == image[off : off + n], i
            assert image[off + n : off + BS].count(0) == len(image[off + n : off + BS])
        assert f.bytes_to_host == int(trimmed.sum())
        gaps = np.ones(total, bool)
        for at, (_, _, n) in zip(offsets, ranges):
            gaps[at : at + n] = False
        assert (dst[gaps] == SENTINEL).all()
    finally:
        gpu_backend.host_free(dst)


@pytest.mark.parametrize("budget_mib", [48, 1200])
def test_staged_upload_of_a_1gib_state_dict_releases_the_tensors_early(gpu_backend, budget_mib):
    """The tensors are overwritten as soon as ``device_released`` is set; what the server ends up with still hashes to
    the digests declared before."""
    import torch

    sd = _state_dict(1 << 30, seed=2)
    BS = blob_utils.BLOCK_SIZE

    async def run():
        async with _volume_server(BS) as (stub, _):
            f = DeviceFile.safetensors(sd)
            spec = (await blob_utils.device_file_specs2([(f, "/ckpt/m.safetensors", 0o644)]))[0]
            batch = volume.VolumeUploadContextManager2("vo-g", types.SimpleNamespace(stub=stub),
                                                       device_staging_bytes=budget_mib * MiB, put_concurrency=8)

            async def clobber():
                await batch.device_released.wait()
                for t in sd.values():
                    t.view(torch.uint8).fill_(0x5A)
                torch.cuda.synchronize()
                return stub.block_puts

            task = asyncio.ensure_future(clobber())
            async with batch:
                batch.put_file(f, "/ckpt/m.safetensors")
            puts_at_release = await task
            distinct = {b.contents_sha256: b.end - b.start for b in spec.blocks}
            assert stub.block_puts == len(distinct)
            assert puts_at_release < stub.block_puts  # the tensors were free while PUTs were still outstanding
            assert f.bytes_to_host == sum(distinct.values())
            for digest, n in distinct.items():
                body = stub.blocks[digest.hex()]
                assert len(body) == n and hashlib.sha256(body).digest() == digest
            data = stub.volume_files["/ckpt/m.safetensors"][0]
            assert len(data) == f.nbytes

    asyncio.run(run())
