"""Reading volumefs2 files back, on the CPU: the C ABI of ``b200h_copy_ranges_from_host``, ``read_file`` /
``read_file_into_fileobj`` against the fake read server, ``read_file_into_device`` over host-memory device files with a
context whose ``copy_ranges_from_host`` does ``ctypes`` moves and checks the entry's argument rules, and
``read_safetensors`` against ``safetensors.torch.load``."""
import asyncio
import contextlib
import ctypes
import io
import json
import os
import re
import types

import numpy as np
import pytest
import torch
from safetensors.torch import load as st_load
from safetensors.torch import save as st_save

from modal_client_b200 import _lib, blob_utils, volume
from modal_client_b200.exception import ExecutionError
from modal_client_b200.synth import synth_bytes
from tests.test_device_file_cpu import HostDeviceFile, _HostSegments
from tests.test_stage_ranges_cpu import StagingContext, range_pieces
from tests.volume_read_server import running_volume_server

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BS = 4096


class ReadContext(StagingContext):
    """Plus ``copy_ranges_from_host`` over host addresses, asserting the argument rules of the entry point, and a log
    of which staging bytes each copy read (to check that no half is refilled before its copy was waited for)."""

    def copy_ranges_from_host(self, seg_ptrs, seg_lens, file_first_seg, ranges, src, src_offsets, stream=0):
        self.calls.append(("copy_ranges_from_host", len(ranges), sum(n for _, _, n in ranges)))
        assert all(at % 16 == 0 for at in src_offsets)
        assert all(at + n <= src.size for (_, _, n), at in zip(ranges, src_offsets))
        written = []
        for (f, off, n), at in zip(ranges, src_offsets):
            for p, into, k in range_pieces(seg_ptrs, seg_lens, file_first_seg, f, off, n):
                written.append((p, p + k))
                ctypes.memmove(p, src.ctypes.data + at + into, k)
        written.sort()
        assert all(a[1] <= b[0] for a, b in zip(written, written[1:])), "two ranges write the same device bytes"


class _LoadHostSegments(_HostSegments):
    """Host-memory segments that also take the ordering steps of ``load_ranges`` and log when a copy is waited for."""

    log: list = []

    def _after_current(self):
        pass

    def _publish(self):
        log = type(self).log
        k = len([e for e in log if e[0] == "copy"])
        log.append(("copy", k))
        return lambda: log.append(("wait", k))

    @classmethod
    def _new_tensor(cls, shape, dtype, ctx):
        return torch.empty(shape, dtype=dtype)


class LoadHostDeviceFile(HostDeviceFile):
    _Source = _LoadHostSegments


def host_file(n: int, fill: int = 0xEE):
    return LoadHostDeviceFile._over(_LoadHostSegments([torch.full((n,), fill, dtype=torch.uint8)], 1 << 20))


@pytest.fixture
def read_backend(monkeypatch):
    from modal_client_b200 import _backend

    ctx = ReadContext()
    monkeypatch.setattr(_backend, "_override", ctx)
    monkeypatch.setattr(blob_utils, "BLOCK_SIZE", BS)
    monkeypatch.setattr(volume, "DeviceFile", LoadHostDeviceFile)
    _LoadHostSegments.log = []
    return ctx


@pytest.fixture
def no_sleep(monkeypatch):
    naps = []

    async def nap(t):
        naps.append(t)

    monkeypatch.setattr("modal_client_b200.async_utils.asyncio.sleep", nap)
    return naps


@contextlib.asynccontextmanager
async def volume_with(files: dict):
    """The read server with ``files`` (path -> bytes) uploaded through VolumeUploadContextManager2."""
    async with running_volume_server(BS) as (stub, faults):
        client = types.SimpleNamespace(stub=stub)
        async with volume.VolumeUploadContextManager2("vo-r", client) as batch:
            for path, data in files.items():
                batch.put_file(io.BytesIO(data), path)
        yield client, stub, faults


def loads(ctx):
    return [c for c in ctx.calls if c[0] == "copy_ranges_from_host"]


def _trimmed_data() -> bytes:
    data = bytearray(synth_bytes(5, 7 * BS + 123))
    data[BS - 300 : BS] = bytes(300)  # trailing zeros at a block edge: stored trimmed, served zero-padded
    data[3 * BS : 4 * BS] = bytes(BS)  # an all-zero block
    data[-50:] = bytes(50)
    return bytes(data)


# ------------------------------------------------------------------------------------------------ C ABI


def test_copy_ranges_from_host_is_declared_exported_and_rejects_a_null_context():
    header = open(os.path.join(ROOT, "include", "b200hash.h")).read()
    assert re.search(r"\bint b200h_copy_ranges_from_host\(b200h_ctx\* ctx, const b200h_segment\* segs,", header)
    assert "_read_file_into_fileobj" in header.split("b200h_copy_ranges_from_host")[0].rsplit("*/", 2)[-2]
    assert "b200h_copy_ranges_from_host" in _lib.ABI_SYMBOLS
    L = _lib.load_library()
    assert hasattr(L, "b200h_copy_ranges_from_host")
    first = (ctypes.c_uint64 * 1)(0)
    assert L.b200h_copy_ranges_from_host(None, None, 0, first, 0, None, 0, None, 0, None, None) == -1  # B200H_E_INVALID


# ------------------------------------------------------------------------------------------- host reads


def test_read_file_and_read_file_into_fileobj_round_trip(read_backend):
    files = {"/t/trimmed": _trimmed_data(), "/t/empty": b"", "/t/one": b"x", "/t/exact": synth_bytes(6, 2 * BS)}

    async def run():
        async with volume_with(files) as (client, _, _):
            for path, data in files.items():
                bodies = [b async for b in volume.read_file(client, "vo-r", path)]
                assert b"".join(bodies) == data, path
                assert all(len(b) == BS for b in bodies[:-1])
                buf = io.BytesIO(b"prefix")
                buf.seek(6)
                progress = []
                n = await volume.read_file_into_fileobj(client, "vo-r", path, buf,
                                                        progress_cb=lambda **kw: progress.append(kw), concurrency=3)
                assert n == len(data) and buf.getvalue() == b"prefix" + data and buf.tell() == 6 + len(data)
                assert sum(kw["advance"] for kw in progress) == len(data)

    asyncio.run(run())


def test_host_reads_of_a_missing_path_and_failing_gets(read_backend, no_sleep):
    data = _trimmed_data()

    async def run():
        async with volume_with({"/f": data}) as (client, stub, faults):
            with pytest.raises(FileNotFoundError):
                [b async for b in volume.read_file(client, "vo-r", "/nope")]
            with pytest.raises(FileNotFoundError):
                await volume.read_file_into_fileobj(client, "vo-r", "/nope", io.BytesIO())
            faults["statuses"] = [500, 503]  # two failed GETs, then success: retried
            assert b"".join([b async for b in volume.read_file(client, "vo-r", "/f")]) == data
            faults["statuses"] = [500]
            buf = io.BytesIO()
            assert await volume.read_file_into_fileobj(client, "vo-r", "/f", buf) == len(data)
            assert buf.getvalue() == data
            stub.token_version["/f"] = "error-404"  # every GET of the file: 404
            with pytest.raises(ExecutionError, match="404"):
                [b async for b in volume.read_file(client, "vo-r", "/f")]
            with pytest.raises(ExecutionError, match="404"):
                await volume.read_file_into_fileobj(client, "vo-r", "/f", io.BytesIO())

    asyncio.run(run())
    assert [t for t in no_sleep if t][:3] == [0.1, 0.1, 0.1]  # the three failed GETs each waited the first back-off


# ------------------------------------------------------------------------------ read_file_into_device


@pytest.mark.parametrize("start", [0, 1, BS - 1, BS, 2 * BS + 17])
def test_read_file_into_device_in_many_waves(read_backend, start):
    data = _trimmed_data()

    async def run():
        async with volume_with({"/f": data}) as (client, stub, faults):
            for staging in (2 * BS, 5 * BS + 100, 64 * BS):
                read_backend.calls.clear()
                _LoadHostSegments.log = []
                dst = host_file(len(data) - start - 5)
                n = await volume.read_file_into_device(client, "vo-r", "/f", dst, start=start, staging_bytes=staging,
                                                       concurrency=2)
                assert n == dst.nbytes and dst._src.segments[0].numpy().tobytes() == data[start : start + n]
                per_half = staging // 2 // BS
                nblocks = (start + n - 1) // BS - start // BS + 1
                assert len(loads(read_backend)) == -(-nblocks // per_half)  # one device call per wave
                assert [c for c in read_backend.calls if c[0] == "host_alloc"] == [("host_alloc", 2 * per_half * BS)]
                assert read_backend.live_buffers == 0
                # wave k + 2 refills the half of wave k: only after wave k's copy was waited for
                log = _LoadHostSegments.log
                for k in range(2, len(loads(read_backend))):
                    assert log.index(("wait", k - 2)) < log.index(("copy", k)), (k, log)
            assert stub.get_file_calls[-1].start == start and stub.get_file_calls[-1].len == len(data) - start - 5

    asyncio.run(run())


def test_read_file_into_device_into_a_segmented_file(read_backend):
    data = _trimmed_data()
    cuts = [0, 1, 1, 17, 4000, 4096, 9000, 9001, len(data)]
    segs = [torch.full((b - a,), 0xEE, dtype=torch.uint8) for a, b in zip(cuts, cuts[1:])]
    dst = LoadHostDeviceFile._over(_LoadHostSegments(segs, 1 << 20))

    async def run():
        async with volume_with({"/f": data}) as (client, _, _):
            assert await volume.read_file_into_device(client, "vo-r", "/f", dst, staging_bytes=3 * BS) == len(data)

    asyncio.run(run())
    assert b"".join(s.numpy().tobytes() for s in segs) == data


def test_read_file_into_device_refuses_before_any_get(read_backend):
    data = _trimmed_data()

    async def run():
        async with volume_with({"/f": data}) as (client, stub, faults):
            with pytest.raises(ValueError, match="two blocks"):
                await volume.read_file_into_device(client, "vo-r", "/f", host_file(10), staging_bytes=2 * BS - 1)
            with pytest.raises(ValueError, match="beyond the end"):
                await volume.read_file_into_device(client, "vo-r", "/f", host_file(len(data) - 9), start=10)
            with pytest.raises(FileNotFoundError):
                await volume.read_file_into_device(client, "vo-r", "/nope", host_file(10))
            real = stub.VolumeGetFile2

            async def lying(req):
                out = await real(req)
                out.get_urls = out.get_urls[:-1]
                return out

            stub.VolumeGetFile2 = lying
            with pytest.raises(ExecutionError, match="blocks"):
                await volume.read_file_into_device(client, "vo-r", "/f", host_file(len(data)))
            assert faults["gets"] == 0 and read_backend.live_buffers == 0
            assert await volume.read_file_into_device(client, "vo-r", "/f", host_file(0)) == 0

    asyncio.run(run())


def test_a_short_body_raises_and_frees_the_staging_buffer(read_backend, no_sleep):
    data = _trimmed_data()

    async def run():
        async with volume_with({"/f": data}) as (client, _, faults):
            faults["short"] = True
            dst = host_file(len(data))
            with pytest.raises(ExecutionError, match="slice has"):
                await volume.read_file_into_device(client, "vo-r", "/f", dst, staging_bytes=2 * BS)
            assert read_backend.live_buffers == 0
            assert faults["gets"] >= 5  # the block was retried
            faults["short"] = False
            faults["statuses"] = [500]  # a retried block restarts in its slot
            assert await volume.read_file_into_device(client, "vo-r", "/f", dst, staging_bytes=2 * BS) == len(data)
            assert dst._src.segments[0].numpy().tobytes() == data

    asyncio.run(run())


# ------------------------------------------------------------------------------------- read_safetensors


def _mixed_state_dict():
    g = torch.Generator().manual_seed(3)
    sd = {
        "w.bf16": torch.randn(37, 29, generator=g).to(torch.bfloat16),
        "w.f32": torch.randn(1000, generator=g),
        "w.fp8": torch.randn(55, 3, generator=g).to(torch.float8_e4m3fn),
        "mask": torch.rand(77, generator=g) > 0.5,
        "scalar": torch.tensor(3.5, dtype=torch.float64),
        "empty": torch.zeros(0, 5, dtype=torch.float16),
        "empty2": torch.zeros(0, dtype=torch.int32),
        "ids": torch.randint(-(1 << 40), 1 << 40, (300,), generator=g, dtype=torch.int64),
        "big": torch.randn(3 * BS, generator=g),
    }
    sd["big"][BS : 2 * BS] = 0  # blank blocks inside a tensor
    return sd


def _assert_same(got: dict, want: dict):
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, k
        assert torch.equal(got[k].view(-1).view(torch.uint8) if got[k].numel() else got[k],
                           want[k].reshape(-1).view(torch.uint8) if want[k].numel() else want[k]), k


def test_read_safetensors_equals_safetensors_load(read_backend):
    sd = _mixed_state_dict()
    images = {"/st/save": st_save(sd, metadata={"format": "pt", "step": "7"}),
              "/st/device": LoadHostDeviceFile.safetensors(sd, metadata={"m": "1"}).readall(),
              "/st/none": st_save({}), "/st/zeros_only": st_save({"e": torch.zeros(0)})}

    async def run():
        async with volume_with(images) as (client, _, _):
            for path, image in images.items():
                got = await volume.read_safetensors(client, "vo-r", path, staging_bytes=2 * BS)
                _assert_same(got, st_load(image))

    asyncio.run(run())


def _image(header, data: bytes = b"", length=None) -> bytes:
    text = header if isinstance(header, bytes) else json.dumps(header).encode()
    return (len(text) if length is None else length).to_bytes(8, "little") + text + data


def test_read_safetensors_rejects_malformed_headers(read_backend):
    ok = {"a": {"dtype": "F32", "shape": [2], "data_offsets": [0, 8]}}
    bad = {
        "/short": (b"abc", "too short"),
        "/huge": (_image(b"{}", length=100_000_001), "larger than"),
        "/past_end": (_image(b"{}", length=50), "does not fit"),
        "/not_json": (_image(b"{nope", bytes(8)), "JSON"),
        "/not_object": (_image([1, 2], bytes(8)), "JSON object"),
        "/bad_meta": (_image({"__metadata__": {"k": 1}, **ok}, bytes(8)), "__metadata__"),
        "/dtype": (_image({"a": {"dtype": "Q7", "shape": [2], "data_offsets": [0, 8]}}, bytes(8)), "dtype"),
        "/size": (_image({"a": {"dtype": "F32", "shape": [3], "data_offsets": [0, 8]}}, bytes(8)), "need 12"),
        "/hole": (_image({"a": {"dtype": "F32", "shape": [2], "data_offsets": [4, 12]}}, bytes(12)), "starts at 4"),
        "/overlap": (_image({**ok, "b": {"dtype": "F32", "shape": [1], "data_offsets": [4, 8]}}, bytes(8)), "starts at 4"),
        "/tail": (_image(ok, bytes(12)), "cover 8 bytes of a 12"),
        "/keys": (_image({"a": {"dtype": "F32", "shape": [2]}}, bytes(8)), "exactly"),
        "/shape": (_image({"a": {"dtype": "F32", "shape": [-2], "data_offsets": [0, 8]}}, bytes(8)), "malformed"),
        "/f4_odd": (_image({"a": {"dtype": "F4", "shape": [3], "data_offsets": [0, 1]}}, bytes(1)), "F4"),
    }

    async def run():
        async with volume_with({p: img for p, (img, _) in bad.items()}) as (client, _, _):
            for path, (image, match) in bad.items():
                allocated = len([c for c in read_backend.calls if c[0] == "copy_ranges_from_host"])
                with pytest.raises(ValueError, match=match):
                    await volume.read_safetensors(client, "vo-r", path)
                assert len(loads(read_backend)) == allocated, path

    asyncio.run(run())


def test_read_safetensors_into_fills_in_place_and_reports_mismatches(read_backend):
    sd = _mixed_state_dict()
    image = st_save(sd)

    async def run():
        async with volume_with({"/m": image}) as (client, stub, faults):
            into = {k: torch.full_like(v, 0) if v.dtype != torch.bool else torch.zeros_like(v) for k, v in sd.items()}
            ptrs = {k: v.data_ptr() for k, v in into.items()}
            got = await volume.read_safetensors(client, "vo-r", "/m", into=into)
            assert all(got[k] is into[k] and into[k].data_ptr() == ptrs[k] for k in sd)
            _assert_same(got, st_load(image))
            gets = faults["gets"]
            wrong = dict(into)
            del wrong["mask"]
            wrong["extra"] = torch.zeros(1)
            wrong["w.f32"] = torch.zeros(999)
            wrong["w.bf16"] = torch.zeros(37, 29)
            wrong["ids"] = torch.zeros(600, dtype=torch.int64)[::2]
            big = torch.zeros(2 * 3 * BS)
            wrong["big"], wrong["scalar"] = big[: 3 * BS], big[8:10].view(torch.float64).reshape(())
            with pytest.raises(ValueError) as err:
                await volume.read_safetensors(client, "vo-r", "/m", into=wrong)
            msg = str(err.value)
            for part in ("'mask' is in the file", "'extra' is in into", "'w.f32'", "'w.bf16'", "contiguous", "overlap"):
                assert part in msg, (part, msg)
            assert faults["gets"] == gets + 2  # only the header's two small reads went out before the refusal

    asyncio.run(run())
