"""``stage_ranges`` and the staged missing-block round of the volumefs2 uploader, on the CPU: the C ABI of
``b200h_copy_ranges_to_host``, the host logic of ``stage_ranges`` over host-memory device files, and the upload against
the fake volume server, with a context that does the copy with ``ctypes`` moves and records its calls."""
import asyncio
import contextlib
import ctypes
import hashlib
import io
import os
import re
import types

import numpy as np
import pytest
import torch
from aiohttp import web
from safetensors.torch import save as st_save

from modal_client_b200 import _lib, blob_utils, stage_ranges, volume
from modal_client_b200.synth import synth_bytes
from tests.blob_server import running_blob_server
from tests.test_device_file_cpu import FakeDeviceContext, HostDeviceFile, _ContentAddressedStub, _HostSegments

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class StagingContext(FakeDeviceContext):
    """Plus ``copy_ranges_to_host`` (host addresses on both sides, the argument rules of the entry point) and
    ``host_alloc`` / ``host_free`` over ordinary memory."""

    def __init__(self):
        super().__init__()
        self.live_buffers = 0

    def host_alloc(self, nbytes):
        self.live_buffers += 1
        self.calls.append(("host_alloc", nbytes))
        return np.full(nbytes, 0xEE, np.uint8)

    def host_free(self, arr):
        self.live_buffers -= 1

    def copy_ranges_to_host(self, seg_ptrs, seg_lens, file_first_seg, ranges, dst, dst_offsets, stream=0):
        self.calls.append(("copy_ranges_to_host", len(ranges), sum(n for _, _, n in ranges)))
        spans = sorted((at, at + n) for at, (_, _, n) in zip(dst_offsets, ranges) if n)
        assert all(at % 16 == 0 for at in dst_offsets) and all(hi <= dst.size for _, hi in spans)
        assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))
        for (f, off, n), at in zip(ranges, dst_offsets):
            for p, into, k in range_pieces(seg_ptrs, seg_lens, file_first_seg, f, off, n):
                ctypes.memmove(dst.ctypes.data + at + into, p, k)


def range_pieces(seg_ptrs, seg_lens, file_first_seg, f, off, n):
    """(address, offset into the range, bytes) of every segment piece of range ``(f, off, n)``, which must lie inside
    its file."""
    segs = list(zip(seg_ptrs[file_first_seg[f] : file_first_seg[f + 1]],
                    seg_lens[file_first_seg[f] : file_first_seg[f + 1]]))
    assert off + n <= sum(ln for _, ln in segs)
    pieces, start = [], 0
    for p, ln in segs:
        lo, hi = max(off, start), min(off + n, start + ln)
        if lo < hi:
            pieces.append((int(p) + lo - start, lo - off, hi - lo))
        start += ln
    return pieces


class _StagedHostSegments(_HostSegments):
    marks = 0

    def _mark(self):
        type(self).marks += 1
        return lambda: None


class StagedHostDeviceFile(HostDeviceFile):
    _Source = _StagedHostSegments


def segments_file(chunks):
    return StagedHostDeviceFile._over(_StagedHostSegments(
        [torch.frombuffer(bytearray(c), dtype=torch.uint8) if c else torch.empty(0, dtype=torch.uint8) for c in chunks],
        1 << 20))


@pytest.fixture
def staging_backend(monkeypatch):
    from modal_client_b200 import _backend

    ctx = StagingContext()
    monkeypatch.setattr(_backend, "_override", ctx)
    return ctx


def copies(ctx):
    return [c for c in ctx.calls if c[0] == "copy_ranges_to_host"]


# ------------------------------------------------------------------------------------------------ C ABI


def test_copy_ranges_to_host_is_declared_exported_and_rejects_a_null_context():
    header = open(os.path.join(ROOT, "include", "b200hash.h")).read()
    assert re.search(r"\bint b200h_copy_ranges_to_host\(b200h_ctx\* ctx, const b200h_segment\* segs,", header)
    assert "typedef struct b200h_file_range" in header
    assert "b200h_copy_ranges_to_host" in _lib.ABI_SYMBOLS
    L = _lib.load_library()
    assert hasattr(L, "b200h_copy_ranges_to_host")
    first = (ctypes.c_uint64 * 1)(0)
    assert L.b200h_copy_ranges_to_host(None, None, 0, first, 0, None, 0, None, 0, None, None) == -1  # B200H_E_INVALID


# ------------------------------------------------------------------------------------------ stage_ranges


def test_stage_ranges_views_equal_the_image(staging_backend):
    chunks = [synth_bytes(1, 100), b"", b"", synth_bytes(2, 1), synth_bytes(3, 4097), b"", synth_bytes(4, 33)]
    chunks += [synth_bytes(10 + i, 1 + i % 5) for i in range(40)]
    f, g = segments_file(chunks), segments_file([synth_bytes(7, 5000)])
    images = [b"".join(chunks), synth_bytes(7, 5000)]
    n0 = len(images[0])
    ranges = [(0, 5, 50),  # inside one segment
              (0, 90, 4200),  # across many, over the empty ones
              (0, 100, 1),  # exactly the one-byte segment behind two empty ones
              (0, 17, 0), (0, n0, 0),  # zero-length, also at the very end
              (0, 0, n0),  # the whole file
              (0, 4231, n0 - 4231),  # the tiny segments
              (1, 0, 5000), (1, 4999, 1), (0, 1, 15)]  # a second file in the same call
    offsets, at = [], 128
    for _, _, n in ranges:
        offsets.append(at)
        at += -(-n // 128) * 128 + 128
    dst = np.full(at, 0xA5, np.uint8)
    marks = _StagedHostSegments.marks
    staged = stage_ranges([f, g], ranges, dst, offsets)
    staged.wait()
    staged.wait()
    assert copies(staging_backend) == [("copy_ranges_to_host", len(ranges), sum(n for _, _, n in ranges))]
    assert _StagedHostSegments.marks == marks + 1
    covered = np.zeros(at, bool)
    for i, ((fi, off, n), o) in enumerate(zip(ranges, offsets)):
        assert bytes(staged.view(i)) == images[fi][off : off + n], i
        assert staged.view(i).nbytes == n
        if n:
            assert np.shares_memory(np.frombuffer(staged.view(i), np.uint8), dst)
        covered[o : o + n] = True
    assert (dst[~covered] == 0xA5).all()
    assert f.bytes_to_host == sum(n for fi, _, n in ranges if fi == 0)
    assert g.bytes_to_host == sum(n for fi, _, n in ranges if fi == 1)
    with pytest.raises(ValueError):
        stage_ranges([f], [(0, 0, 1)], dst, [])
    stage_ranges([], [], dst, []).wait()  # no files: nothing to do, no call
    assert len(copies(staging_backend)) == 1


# ------------------------------------------------------------------------------------------------ uploads


def _state_dict():
    g = torch.Generator().manual_seed(5)
    sd = {f"l{i}.w": torch.randint(-100, 100, (n,), generator=g, dtype=torch.int16)
          for i, n in enumerate([3000, 1, 700, 5000, 12, 2048, 2048, 9000])}
    sd["blank"] = torch.zeros(6000, dtype=torch.int16)  # blank blocks
    sd["l3.w"][-1500:] = 0  # trailing zeros inside a block
    sd["l5.w"][:] = 7
    sd["l6.w"][:] = 7  # duplicate content
    sd["dup.a"] = torch.full((8192,), 3, dtype=torch.int16)  # whole duplicate blocks
    return sd


def _images():
    sd = _state_dict()
    buf = io.BytesIO()
    torch.save(sd, buf)
    return {"safetensors": (lambda ctx: StagedHostDeviceFile.safetensors(sd, ctx=ctx), st_save(sd)),
            "torch_save": (lambda ctx: StagedHostDeviceFile.torch_save(sd, ctx=ctx), buf.getvalue())}


@contextlib.asynccontextmanager
async def _recording_server(BS, fail_first=0):
    """The contract of ``_volume_server``, plus a log of every request and ``fail_first`` PUTs answered 500."""
    log, state = [], {"fail": fail_first}

    class Stub(_ContentAddressedStub):
        async def VolumePutFiles2(self, req):
            out = await super().VolumePutFiles2(req)
            log.append(("rpc", sorted((m.file_index, m.block_index) for m in out.missing_blocks)))
            return out

    async with running_blob_server() as (host, store):
        stub = Stub(host, store, BS)
        stub.block_puts = 0

        async def put_block(request):
            body = await request.read()
            if state["fail"]:
                state["fail"] -= 1
                log.append(("put-failed", hashlib.sha256(body).hexdigest()))
                return web.Response(status=500, text="try again")
            bid = hashlib.sha256(body).hexdigest()
            log.append(("put", bid))
            for hook in state.get("on_put", []):
                hook()
            stub.blocks[bid] = body
            stub.block_puts += 1
            return web.Response(text=f"test-put-response:{bid}")

        app = web.Application(client_max_size=1 << 26)
        app.add_routes([web.put("/block/{token}", put_block)])
        runner = web.AppRunner(app)
        await runner.setup()
        site = web.TCPSite(runner, "127.0.0.1", 0)
        await site.start()
        stub.host = f"http://127.0.0.1:{site._server.sockets[0].getsockname()[1]}"
        try:
            yield stub, log, state
        finally:
            await runner.cleanup()
            await blob_utils.ClientSessionRegistry.close_session()


def _normal(log):
    """The request sequence up to the order of the PUTs inside one round (they run concurrently)."""
    out, puts = [], []
    for kind, what in log:
        if kind == "rpc":
            out += [sorted(puts), ("rpc", what)]
            puts = []
        else:
            puts.append((kind, what))
    return out + [sorted(puts)]


async def _upload(stub, make, budget, path="/ckpt/model", **kw):
    f = make(blob_utils.get_context())
    batch = volume.VolumeUploadContextManager2("vo-s", types.SimpleNamespace(stub=stub), device_staging_bytes=budget, **kw)
    async with batch:
        batch.put_file(f, path)
    return f, batch


@pytest.mark.parametrize("kind", ["safetensors", "torch_save"])
def test_staged_upload_equals_the_unstaged_upload(staging_backend, monkeypatch, kind):
    BS = 4096
    monkeypatch.setattr(blob_utils, "BLOCK_SIZE", BS)
    make, image = _images()[kind]
    nblocks = -(-len(image) // BS)
    trimmed = [len(image[i * BS : (i + 1) * BS].rstrip(b"\0")) for i in range(nblocks)]
    distinct = {}
    for i in range(nblocks):
        distinct.setdefault(hashlib.sha256(image[i * BS : i * BS + trimmed[i]]).digest(), trimmed[i])
    assert len(distinct) < nblocks and 0 in trimmed and any(0 < t < BS for t in trimmed[:-1])

    async def run(budget):
        async with _recording_server(BS) as (stub, log, _):
            f, batch = await _upload(stub, make, budget)
            assert stub.volume_files["/ckpt/model"][0] == image
            assert batch.device_released.is_set() and staging_backend.live_buffers == 0
            return dict(stub.blocks), _normal(log), f.bytes_to_host

    want = asyncio.run(run(None))
    assert copies(staging_backend) == []  # no budget, no staging call
    assert want[2] == sum(distinct.values())

    def expected_waves(half):
        waves, used = 0, None
        for n in distinct.values():  # missing blocks arrive in file order, first occurrences only
            if used is None or used + n > half:
                waves, used = waves + 1, 0
            used += -(-n // 128) * 128
        return waves

    for budget in (2 * BS, 3 * BS, 2 * len(image) + 4 * BS):
        staging_backend.calls.clear()
        got = asyncio.run(run(budget))
        assert got == want
        half = budget // 2 // 128 * 128
        assert len(copies(staging_backend)) == expected_waves(half)  # one device call per wave
        assert sum(c[2] for c in copies(staging_backend)) == sum(distinct.values())
        assert [c for c in staging_backend.calls if c[0] == "host_alloc"] == [("host_alloc", 2 * half)]
    assert expected_waves(BS) > expected_waves(3 * BS // 2 // 128 * 128) > 1
    assert len(copies(staging_backend)) == 1  # a budget above the file: one copy after the block table


def test_device_released_before_the_last_put_and_at_once_when_nothing_is_missing(staging_backend, monkeypatch):
    BS = 4096
    monkeypatch.setattr(blob_utils, "BLOCK_SIZE", BS)
    make, image = _images()["safetensors"]

    async def run():
        async with _recording_server(BS) as (stub, log, state):
            seen = []
            f = make(staging_backend)
            batch = volume.VolumeUploadContextManager2("vo-s", types.SimpleNamespace(stub=stub),
                                                       device_staging_bytes=4 * len(image))
            state["on_put"] = [lambda: seen.append(batch.device_released.is_set())]
            assert not batch.device_released.is_set()
            async with batch:
                batch.put_file(f, "/a")
            assert seen and all(seen)  # released before the FIRST PUT is served: the one wave holds every block
            # the same file again: nothing is missing, nothing is staged, no buffer is taken
            staging_backend.calls.clear()
            puts = stub.block_puts
            again = volume.VolumeUploadContextManager2("vo-s", types.SimpleNamespace(stub=stub), force=True,
                                                       device_staging_bytes=4 * len(image))
            async with again:
                again.put_file(f, "/a")
            assert again.device_released.is_set() and stub.block_puts == puts
            assert [c for c in staging_backend.calls if c[0] in ("copy_ranges_to_host", "host_alloc")] == []

    asyncio.run(run())


def test_staged_mixed_batch(staging_backend, monkeypatch, tmp_path):
    BS = 4096
    monkeypatch.setattr(blob_utils, "BLOCK_SIZE", BS)
    kinds = _images()
    on_disk, in_memory = synth_bytes(41, 3 * BS + 17), synth_bytes(42, 2 * BS)
    (tmp_path / "p.bin").write_bytes(on_disk)

    async def run(budget):
        async with _recording_server(BS) as (stub, log, _):
            batch = volume.VolumeUploadContextManager2("vo-m", types.SimpleNamespace(stub=stub),
                                                       device_staging_bytes=budget)
            async with batch:
                batch.put_file(tmp_path / "p.bin", "/p")
                batch.put_file(kinds["safetensors"][0](staging_backend), "/st")
                batch.put_file(io.BytesIO(in_memory), "/mem")
                batch.put_file(kinds["torch_save"][0](staging_backend), "/pt")
            files = {k: v[0] for k, v in stub.volume_files.items()}
            assert files == {"/p": on_disk, "/st": kinds["safetensors"][1], "/mem": in_memory, "/pt": kinds["torch_save"][1]}
            return dict(stub.blocks), _normal(log)

    want = asyncio.run(run(None))
    staging_backend.calls.clear()
    assert asyncio.run(run(6 * BS)) == want
    calls = copies(staging_backend)
    assert len(calls) > 1 and staging_backend.live_buffers == 0


def test_a_failed_put_is_retried_from_the_staged_bytes(staging_backend, monkeypatch):
    BS = 4096
    monkeypatch.setattr(blob_utils, "BLOCK_SIZE", BS)
    make, image = _images()["torch_save"]
    naps = []

    async def no_sleep(t):
        naps.append(t)

    async def run():
        async with _recording_server(BS, fail_first=2) as (stub, log, _):
            monkeypatch.setattr("modal_client_b200.async_utils.asyncio.sleep", no_sleep)
            progress = []
            f, _ = await _upload(stub, make, 4 * len(image), put_concurrency=1,
                                 progress_cb=lambda **kw: progress.append(kw) or 1)
            assert stub.volume_files["/ckpt/model"][0] == image
            assert [k for k, _ in log].count("put-failed") == 2
            failed = [w for k, w in log if k == "put-failed"]
            assert failed[0] == failed[1] and ("put", failed[0]) in log  # the same block, three times, then accepted
            assert len(copies(staging_backend)) == 1  # read from the device once
            assert sum(kw.get("advance", 0) for kw in progress) == f.bytes_to_host
            assert any(kw.get("advance", 0) < 0 for kw in progress)

    asyncio.run(run())
    assert [t for t in naps if t] == [0.5, 1.0]  # the two back-offs of the retried PUT


def test_blocks_still_missing_after_release_raise_without_another_put(staging_backend, monkeypatch):
    BS = 4096
    monkeypatch.setattr(blob_utils, "BLOCK_SIZE", BS)
    make, image = _images()["safetensors"]

    async def run():
        async with _recording_server(BS) as (stub, log, _):
            real = stub.VolumePutFiles2

            async def forgetful(req):  # a server that never accepts block 1
                for f in req.files:
                    f.blocks[1].put_response = None
                    stub.blocks.pop(f.blocks[1].contents_sha256.hex(), None)
                return await real(req)

            stub.VolumePutFiles2 = forgetful
            with pytest.raises(RuntimeError, match="Did not succeed"):
                await _upload(stub, make, 4 * len(image))
            kinds = [k for k, _ in log]
            assert kinds.count("rpc") == 2 and kinds[-1] == "rpc"  # nothing is PUT after the second answer
            assert len(copies(staging_backend)) == 1 and staging_backend.live_buffers == 0

    asyncio.run(run())


def test_a_budget_below_two_blocks_is_refused(monkeypatch):
    monkeypatch.setattr(blob_utils, "BLOCK_SIZE", 4096)
    with pytest.raises(ValueError, match="two blocks"):
        volume.VolumeUploadContextManager2("vo", None, device_staging_bytes=8191)
    volume.VolumeUploadContextManager2("vo", None, device_staging_bytes=8192)
    m = volume._AbstractVolumeUploadContextManager.resolve(volume.VOLUME_FS_VERSION_V2, "vo", None,
                                                           device_staging_bytes=8192)
    assert m._device_staging_bytes == 8192
    assert isinstance(volume._AbstractVolumeUploadContextManager.resolve(volume.VOLUME_FS_VERSION_V1, "vo", None,
                                                                         device_staging_bytes=8192),
                      volume.VolumeUploadContextManager)
