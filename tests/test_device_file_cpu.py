"""DeviceFile and the volumefs2 device path, on the CPU: the file-object semantics, the block table built from one
``hash_segment_parts_device`` call, and the upload rounds, with the oracle-backed context and CPU tensors standing in
for GPU memory.  The fake context, fixture and host-memory source here serve the other device-file CPU tests too."""
import asyncio
import contextlib
import ctypes
import hashlib
import io
import random
import types
import zlib
from pathlib import PurePosixPath

import numpy as np
import pytest
import torch
from aiohttp import web

from modal_client_b200 import DeviceFile, _lib, blob_utils, device_file, volume
from modal_client_b200.synth import materialize, synth_bytes
from oracle import c_oracle
from tests.blob_server import running_blob_server
from tests.fake_backend import FakeContext
from tests.test_volume_upload import FakeVolumeStub, _add_block_route


class FakeDeviceContext(FakeContext):
    """The oracle-backed context plus stand-ins for ``Context.hash_segment_parts_device`` and ``crc32_device``.
    Segment, range and output addresses are HOST addresses (CPU tensors standing in for device memory), so the host
    logic around the calls runs on the CPU.  The split is checked by the library's own preview, the digests come from
    the oracle and the CRCs from zlib."""

    def hash_segment_parts_device(self, seg_ptrs, seg_lens, file_first_seg, part_len, flags, d_sha=0, d_md5=0,
                                  d_trimmed=0, stream=0):
        self.calls.append(("hash_segment_parts_device", len(file_first_seg) - 1, part_len, flags))
        seg, _, _ = _lib.segment_parts_preview(seg_lens, file_first_seg, part_len, 1 << 30)  # raises like the entry
        images = [b"".join(ctypes.string_at(int(p), int(n)) if n else b"" for p, n in
                           zip(seg_ptrs[file_first_seg[f] : file_first_seg[f + 1]],
                               seg_lens[file_first_seg[f] : file_first_seg[f + 1]]))
                  for f in range(len(file_first_seg) - 1)]
        data = np.frombuffer(b"".join(images) or b"\0", np.uint8)
        starts, lens, at = [], [], 0
        for img in images:
            for o in range(0, len(img), part_len):
                starts.append(at + o)
                lens.append(min(part_len, len(img) - o))
            at += len(img)
        assert len(starts) == len(seg)
        s, m, e = c_oracle.hash_batch(data, np.array(starts, np.uint64), np.array(lens, np.uint64),
                                      sha=bool(flags & _lib.SHA256), md5=bool(flags & _lib.MD5),
                                      trim=bool(flags & _lib.TRIM_ZEROS))
        for addr, table in ((d_sha, s), (d_md5, m), (d_trimmed, e)):
            if addr and table is not None and len(table):
                ctypes.memmove(addr, np.ascontiguousarray(table).tobytes(), table.nbytes)
        return len(starts)

    def crc32_device(self, ptrs, lens, d_out, stream=0):
        self.calls.append(("crc32_device", len(lens)))
        crcs = np.array([zlib.crc32(ctypes.string_at(int(p), int(n))) if n else 0 for p, n in zip(ptrs, lens)],
                        np.uint32)
        if len(crcs):
            ctypes.memmove(d_out, crcs.tobytes(), crcs.nbytes)


@pytest.fixture
def fake_device_backend(monkeypatch):
    """The host layer routed to FakeDeviceContext (like the ``fake_backend`` fixture for FakeContext)."""
    from modal_client_b200 import _backend

    ctx = FakeDeviceContext()
    monkeypatch.setattr(_backend, "_override", ctx)
    return ctx


class _HostSegments(device_file._TensorBytes):
    """Segments in CPU tensors: only the stream, the pinned and device buffers, the wait and the uploads change."""

    device_type = "cpu"

    def __init__(self, tensors, bounce_bytes):
        self._attach(tensors, bounce_bytes)
        self.stream_handle = 0

    def _on_stream(self):
        return contextlib.nullcontext()

    def _new_bounce(self, n):
        return torch.empty(n, dtype=torch.uint8)

    def _wait(self):
        pass

    @classmethod
    def _to_device(cls, data, ctx):
        return torch.frombuffer(bytearray(data), dtype=torch.uint8)

    @classmethod
    def _pinned(cls, n):
        return torch.empty(n, dtype=torch.uint8)

    @classmethod
    def _empty(cls, n, ctx):
        return torch.empty(n, dtype=torch.uint8)

    @classmethod
    def _current_stream(cls, ctx):
        return 0


class HostDeviceFile(DeviceFile):
    _Source = _HostSegments


def host_segments_file(chunks, bounce_bytes=1 << 20) -> DeviceFile:
    """A DeviceFile whose "device" bytes are CPU tensors holding ``chunks``, one segment each."""
    return DeviceFile._over(_HostSegments([torch.frombuffer(bytearray(c), dtype=torch.uint8) if c else
                                           torch.empty(0, dtype=torch.uint8) for c in chunks], bounce_bytes))


def host_device_file(data: bytes, bounce_bytes: int = 1 << 20) -> DeviceFile:
    """A DeviceFile whose "device" bytes are one CPU tensor holding ``data``."""
    return host_segments_file([data], bounce_bytes)


# ------------------------------------------------------------------------------------------------ C ABI


def test_fixed_parts_device_is_exported_and_rejects_a_null_context():
    L = _lib.load_library()
    assert hasattr(L, "b200h_hash_fixed_parts_device")
    assert "b200h_hash_fixed_parts_device" in _lib.ABI_SYMBOLS
    got = ctypes.c_uint64(12345)
    for part_len in (0, 8 << 20):
        rc = L.b200h_hash_fixed_parts_device(None, None, 100, part_len, _lib.SHA256 | _lib.TRIM_ZEROS, None, None, None,
                                             None, ctypes.byref(got), None)
        assert rc == -1  # B200H_E_INVALID
        assert got.value == 12345  # nothing written


# ------------------------------------------------------------------------------------------- DeviceFile


def test_device_file_reads_like_bytesio_through_any_seek_read_sequence():
    data = synth_bytes(11, 300_001)
    rng = random.Random(5)
    for bounce in (1, 4096, 1 << 20):
        f, ref = host_device_file(data, bounce_bytes=bounce if bounce > 1 else 7), io.BytesIO(data)
        assert f.readable() and f.seekable() and not f.writable()
        for _ in range(60):
            op = rng.randrange(5)
            if op == 0:
                whence = rng.choice([0, 1, 2])
                off = rng.randrange(-1000, len(data) + 1000) if whence else rng.randrange(0, len(data) + 1000)
                if whence == 1:
                    off = max(off, -ref.tell())
                elif whence == 2:
                    off = max(off, -len(data))
                assert f.seek(off, whence) == ref.seek(off, whence)
            elif op == 1:
                n = rng.choice([0, 1, 63, 4096, 70_000, -1])
                assert f.read(n) == ref.read(n)
            elif op == 2:
                buf_a = bytearray(rng.randrange(0, 50_000))
                buf_b = bytearray(len(buf_a))
                assert f.readinto(buf_a) == ref.readinto(buf_b) and buf_a == buf_b
            elif op == 3:
                assert f.read() == ref.read()
            assert f.tell() == ref.tell()
    f = host_device_file(data)
    assert f.seek(0, io.SEEK_END) == len(data) and f.read(10) == b"" and f.readall() == b""
    f.seek(0)
    assert f.readall() == data and f.bytes_to_host == len(data)


def test_device_file_io_contract():
    f = host_device_file(b"abc")
    with pytest.raises(OSError):
        f.fileno()
    with pytest.raises(ValueError):
        f.seek(-1)
    r = f.reopen()  # own position, shared counter
    assert r.read(2) == b"ab" and f.tell() == 0 and f.read() == b"abc"
    assert f.bytes_to_host == 5
    r.close()
    with pytest.raises(ValueError):
        r.read()
    assert f.read(1) == b""  # the original stays open
    with host_device_file(b"") as e:
        assert e.read() == b"" and e.seek(0, io.SEEK_END) == 0


def test_device_file_rejects_host_tensors():
    with pytest.raises(ValueError, match="CUDA"):
        DeviceFile(torch.zeros(16, dtype=torch.float16))
    with pytest.raises(ValueError, match="CUDA"):
        DeviceFile(torch.zeros(4, 4).t())


# -------------------------------------------------------------------------------------- FileUploadSpec2


def test_spec2_from_device_file_equals_spec2_from_bytesio(fake_device_backend, golden, monkeypatch):
    for c in golden("blocks.json")["spec2"]:
        data = materialize(c["input"])
        if len(data) > 20_000_000:
            continue  # keep the CPU suite quick (the GPU suite covers it)
        sem = asyncio.Semaphore(1)
        f = host_device_file(data)
        with monkeypatch.context() as mp:
            for k, v in c["patch"].items():
                mp.setattr(blob_utils, k, v)
            dev = asyncio.run(blob_utils.FileUploadSpec2.from_fileobj(f, PurePosixPath(c["path"]), sem, 0o644))
            host = asyncio.run(blob_utils.FileUploadSpec2.from_fileobj(io.BytesIO(data), PurePosixPath(c["path"]), sem,
                                                                       0o644))
        assert [[b.start, b.end, b.contents_sha256.hex()] for b in dev.blocks] == c["blocks"]
        assert (dev.blocks, dev.size, dev.mode, dev.path) == (host.blocks, host.size, host.mode, host.path)
        assert f.bytes_to_host == 0  # only the digest table was fetched
        with dev.source() as rd:
            assert rd.read() == data
    assert ("hash_segment_parts_device", 1, blob_utils.BLOCK_SIZE, _lib.SHA256 | _lib.TRIM_ZEROS) in \
        fake_device_backend.calls


def test_spec2_device_file_block_edges(fake_device_backend, monkeypatch):
    """Trailing zeros that end exactly at a block edge, all-zero blocks, a one-byte tail, the empty file."""
    BS = 4096
    monkeypatch.setattr(blob_utils, "BLOCK_SIZE", BS)
    cases = [b"", b"x", b"a" + bytes(BS - 1), b"a" * (BS - 5) + bytes(5) + b"b" * BS, bytes(2 * BS) + b"z",
             (b"a" + bytes(BS - 1)) * 2 + b"cdef", synth_bytes(3, 3 * BS + 4711)]
    for data in cases:
        spec = asyncio.run(blob_utils.FileUploadSpec2.from_fileobj(host_device_file(data), PurePosixPath("/x"),
                                                                   asyncio.Semaphore(1), 0o600))
        assert spec.size == len(data) and len(spec.blocks) == -(-len(data) // BS)
        for i, b in enumerate(spec.blocks):
            block = data[i * BS : (i + 1) * BS]
            assert (b.start, b.end) == (i * BS, i * BS + len(block.rstrip(b"\0")))
            assert b.contents_sha256 == hashlib.sha256(data[b.start : b.end]).digest()


# ----------------------------------------------------------------------------------------------- uploads


class _ContentAddressedStub(FakeVolumeStub):
    """The volumefs2 fake, plus what a real server does across batches: a block whose content it already holds is not
    reported missing again (the base fake only accepts blocks that carry this batch's put_response)."""

    async def VolumePutFiles2(self, req):
        for f in req.files:
            for b in f.blocks:
                bid = b.contents_sha256.hex()
                if b.put_response is None and bid in self.blocks:
                    b.put_response = b"test-put-response:" + bid.encode()
        return await super().VolumePutFiles2(req)


@contextlib.asynccontextmanager
async def _volume_server(BS):
    holder = {}
    async with running_blob_server() as (host, store):
        stub = _ContentAddressedStub(host, store, BS)
        stub.block_puts = 0
        holder["stub"] = stub
        app = web.Application(client_max_size=1 << 26)
        app.add_routes([web.put("/block/{token}", _add_block_route(store, holder, BS))])
        runner = web.AppRunner(app)
        await runner.setup()
        site = web.TCPSite(runner, "127.0.0.1", 0)
        await site.start()
        stub.host = f"http://127.0.0.1:{site._server.sockets[0].getsockname()[1]}"
        try:
            yield stub, store
        finally:
            await runner.cleanup()
            await blob_utils.ClientSessionRegistry.close_session()


def _trimmed_total(data: bytes, BS: int, blocks=None) -> int:
    idx = range(-(-len(data) // BS)) if blocks is None else blocks
    return sum(len(data[i * BS : (i + 1) * BS].rstrip(b"\0")) for i in idx)


def test_v2_put_file_device_file_puts_only_missing_blocks(fake_device_backend, monkeypatch):
    BS = 4096
    monkeypatch.setattr(blob_utils, "BLOCK_SIZE", BS)
    data = bytearray(synth_bytes(21, 9 * BS + 100))
    data[2 * BS - 300 : 2 * BS] = bytes(300)  # trailing zeros at a block edge
    data[5 * BS : 6 * BS] = bytes(BS)  # an all-zero block
    data = bytes(data)

    async def run():
        async with _volume_server(BS) as (stub, _):
            client = types.SimpleNamespace(stub=stub)
            f = host_device_file(data, bounce_bytes=1000)
            async with volume.VolumeUploadContextManager2("vo-d", client) as batch:
                batch.put_file(f, "/d/weights.bin", mode=0o600)
            assert stub.volume_files["/d/weights.bin"][0] == data and stub.volume_files["/d/weights.bin"][1] == 0o600
            first_puts = stub.block_puts
            assert first_puts == len({hashlib.sha256(data[i * BS : (i + 1) * BS].rstrip(b"\0")).digest()
                                      for i in range(10)})
            assert f.bytes_to_host == _trimmed_total(data, BS)  # exactly the trimmed bytes of the PUT blocks
            # the same source again: the server knows every block, nothing is PUT or copied
            async with volume.VolumeUploadContextManager2("vo-d", client, force=True) as batch:
                batch.put_file(f, "/d/weights.bin")
            assert stub.block_puts == first_puts and f.bytes_to_host == _trimmed_total(data, BS)
            # one block changed: only that block travels
            changed = bytearray(data)
            changed[7 * BS + 5] ^= 0xFF
            g = host_device_file(bytes(changed))
            async with volume.VolumeUploadContextManager2("vo-d", client, force=True) as batch:
                batch.put_file(g, "/d/weights.bin")
            assert stub.block_puts == first_puts + 1
            assert g.bytes_to_host == _trimmed_total(bytes(changed), BS, [7])
            assert stub.volume_files["/d/weights.bin"][0] == bytes(changed)

    asyncio.run(run())


@pytest.mark.parametrize("size", [0, 100, 5000, 12_000_017])
def test_v1_put_file_reads_a_device_file_through_the_stream_path(fake_device_backend, monkeypatch, size):
    """volumefs1 needs whole-object digests: it reads the DeviceFile like any stream (inline, single PUT, multipart)."""
    monkeypatch.setattr(blob_utils, "LARGE_FILE_LIMIT", 4000)
    data = bytearray(synth_bytes(31, size))
    if size > 1000:
        data[-700:] = bytes(700)
    data = bytes(data)

    async def run():
        async with running_blob_server() as (host, store):
            stub = FakeVolumeStub(host, store, 8 << 20)
            client = types.SimpleNamespace(stub=stub)
            async with volume.VolumeUploadContextManager("vo-1", client) as batch:
                batch.put_file(host_device_file(data, bounce_bytes=1 << 16), "/d/x")
            got, _, sha = stub.volume_files["/d/x"]
            assert got == data and sha == hashlib.sha256(data).hexdigest()
            await blob_utils.ClientSessionRegistry.close_session()

    asyncio.run(run())
