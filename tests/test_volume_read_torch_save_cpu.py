"""``volume.read_torch_save`` on the CPU: checkpoints read back from the fake volume server into host-memory "device"
storages, against ``torch.load(..., map_location="cpu")``, with the zlib-backed ``crc32_device`` of the fake context and
a 4 KiB block size, so that storages straddle block and wave edges at the two-block staging minimum."""
import asyncio
import io
import pickle
import zipfile

import pytest
import torch
from torch.utils.serialization import config

from modal_client_b200 import volume
from modal_client_b200.exception import ExecutionError
from tests.test_torch_save_cpu import CASES, _adam_state, saved
from tests.test_volume_read_cpu import (  # noqa: F401 (read_backend, no_sleep: fixtures)
    BS, LoadHostDeviceFile, loads, no_sleep, read_backend, volume_with)

STAGING = 2 * BS


def _assert_same(got, want, path="obj"):
    """Same structure, types, dtypes, shapes, strides and bytes; tensors sharing a storage in ``want`` share one in
    ``got``."""
    shared_want, shared_got = {}, {}

    def walk(g, w, at):
        assert type(g) is type(w), at
        if isinstance(w, torch.Tensor):
            assert (g.dtype, g.shape, g.stride(), g.storage_offset()) == (w.dtype, w.shape, w.stride(),
                                                                          w.storage_offset()), at
            assert g.untyped_storage().nbytes() == w.untyped_storage().nbytes(), at
            assert bytes(g.untyped_storage()) == bytes(w.untyped_storage()), at
            if w.untyped_storage().nbytes():
                shared_want.setdefault(w.untyped_storage().data_ptr(), set()).add(at)
                shared_got.setdefault(g.untyped_storage().data_ptr(), set()).add(at)
        elif isinstance(w, dict):
            assert list(g) == list(w), at
            for k in w:
                walk(g[k], w[k], f"{at}[{k!r}]")
        elif isinstance(w, (list, tuple)):
            assert len(g) == len(w), at
            for i, (a, b) in enumerate(zip(g, w)):
                walk(a, b, f"{at}[{i}]")
        else:
            assert g == w, at

    walk(got, want, path)
    assert sorted(map(sorted, shared_got.values())) == sorted(map(sorted, shared_want.values()))


def _read(client, path, **kw):
    return volume.read_torch_save(client, "vo-r", path, staging_bytes=kw.pop("staging_bytes", STAGING), **kw)


def crcs(ctx):
    return [c for c in ctx.calls if c[0] == "crc32_device"]


@pytest.mark.parametrize("name", list(CASES))
def test_equals_torch_load(read_backend, name):
    obj = CASES[name]
    images = {"/host.pt": saved(obj), "/device.pt": LoadHostDeviceFile.torch_save(obj).read()}
    assert images["/host.pt"] == images["/device.pt"]

    async def run():
        async with volume_with(images) as (client, _, _):
            for path, image in images.items():
                got = await _read(client, path)
                _assert_same(got, torch.load(io.BytesIO(image), map_location="cpu", weights_only=True))
                assert read_backend.live_buffers == 0

    asyncio.run(run())


def test_a_file_saved_to_a_path_has_another_prefix(read_backend, tmp_path):
    obj = _adam_state()
    torch.save(obj, tmp_path / "last_step.pt")
    image = (tmp_path / "last_step.pt").read_bytes()
    assert zipfile.ZipFile(io.BytesIO(image)).namelist()[0].startswith("last_step/")

    async def run():
        async with volume_with({"/ckpt/last.pt": image}) as (client, _, _):
            _assert_same(await _read(client, "/ckpt/last.pt"), torch.load(io.BytesIO(image), map_location="cpu"))

    asyncio.run(run())


def _many(n=300):
    return {f"w{i}": torch.arange(i % 37 + (i % 5) * 100, dtype=torch.float32) + i for i in range(n)}


@pytest.mark.parametrize("crc", [True, False])
def test_request_and_call_counts_of_a_300_storage_checkpoint(read_backend, monkeypatch, crc):
    monkeypatch.setattr(config.save, "compute_crc32", crc)
    obj = _many()
    image = saved(obj)
    assert all((i.CRC != 0) == crc for i in zipfile.ZipFile(io.BytesIO(image)).infolist() if i.file_size)

    async def run():
        async with volume_with({"/m.pt": image}) as (client, stub, _):
            for staging in (STAGING, 5 * BS, 64 * BS):
                stub.get_file_calls.clear()
                read_backend.calls.clear()
                got = await _read(client, "/m.pt", staging_bytes=staging)
                _assert_same(got, torch.load(io.BytesIO(image), map_location="cpu"))
                assert len(stub.get_file_calls) <= 5
                nblocks = _nblocks(stub.get_file_calls[-1])  # the data region's call
                assert len(loads(read_backend)) == -(-nblocks // (staging // 2 // BS))  # one load per wave
                assert len(crcs(read_backend)) == (1 if crc else 0)
                assert read_backend.live_buffers == 0

    asyncio.run(run())


@pytest.mark.parametrize("n", [1056, 1063, 1070, 1112])
def test_a_central_directory_longer_than_the_end_read(read_backend, n):
    """Some central directory entry lies on the edge of the first read of the file's end, whichever n it is."""
    obj = {f"w{i}": torch.ones(1) for i in range(n)}
    image = saved(obj)
    cd_off = int.from_bytes(image[image.rfind(b"PK\x05\x06") + 16 :][:4], "little")
    assert cd_off < len(image) - volume._ZIP_TAIL

    async def run():
        async with volume_with({"/m.pt": image}) as (client, stub, _):
            _assert_same(await _read(client, "/m.pt", staging_bytes=64 * BS), torch.load(io.BytesIO(image)))
            assert len(stub.get_file_calls) <= 5

    asyncio.run(run())


def test_the_records_after_the_data_are_checked(read_backend):
    image = saved({"w": torch.arange(3000, dtype=torch.float32)})
    info = zipfile.ZipFile(io.BytesIO(image)).getinfo("archive/.data/serialization_id")
    at = info.header_offset + 30 + len(info.filename) + int.from_bytes(image[info.header_offset + 28 :][:2], "little")
    assert image[at : at + 40].isdigit()
    bad = bytearray(image)
    bad[at + 3] = ord("0") + (bad[at + 3] - ord("0") + 1) % 10

    async def run():
        async with volume_with({"/m.pt": bytes(bad)}) as (client, _, faults):
            with pytest.raises(ExecutionError, match=r"archive/.data/serialization_id \(stored"):
                await _read(client, "/m.pt")
            assert not loads(read_backend)

    asyncio.run(run())


def _rezipped(image: bytes, *, compress=False, extra=None, align_off=0) -> bytes:
    """The records of ``image`` rewritten by Python's zipfile (no data descriptors, no alignment padding)."""
    src = zipfile.ZipFile(io.BytesIO(image))
    out = io.BytesIO()
    out.write(b"\0" * align_off)
    with zipfile.ZipFile(out, "a" if align_off else "w",
                         zipfile.ZIP_DEFLATED if compress else zipfile.ZIP_STORED) as z:
        for info in src.infolist():
            z.writestr(info.filename, src.read(info.filename))
        for name, data in (extra or {}).items():
            z.writestr(name, data)
    return out.getvalue()


def _with_record(image: bytes, name: str, data: bytes) -> bytes:
    """``image`` with the record ``<prefix>/name`` replaced by ``data`` (same length), through torch's own writer."""
    src = zipfile.ZipFile(io.BytesIO(image))
    prefix = src.namelist()[0].split("/", 1)[0]
    out = io.BytesIO()
    w = torch._C.PyTorchFileWriter(out)
    for n in src.namelist():
        rel = n[len(prefix) + 1 :]
        if rel in ("version", ".data/serialization_id") and rel != name:
            continue  # the writer adds both
        body = data if rel == name else src.read(n)
        w.write_record(rel, body, len(body))
    w.write_end_of_file()
    return out.getvalue()


class _Evil:
    def __reduce__(self):
        return (print, ("never",))


def test_rejections_come_before_any_get_of_the_data_region(read_backend):
    sd = {"w": torch.arange(3000, dtype=torch.float32), "b": torch.ones(7)}
    image = saved(sd)
    legacy = io.BytesIO()
    torch.save(sd, legacy, _use_new_zipfile_serialization=False)
    evil = saved({"w": torch.ones(3), "evil": _Evil()})
    pkl = zipfile.ZipFile(io.BytesIO(image)).read("archive/data.pkl")
    bad = {
        "/legacy.pt": (legacy.getvalue(), ValueError, "not a torch.save zip"),
        "/plain": (b"hello" * 1000, ValueError, "not a torch.save zip"),
        "/script.pt": (_rezipped(image, extra={"archive/constants.pkl": b"x"}), ValueError, "TorchScript"),
        "/deflated.pt": (_rezipped(image, compress=True), ValueError, "uncompressed"),
        "/big_endian.pt": (_with_record(image, "byteorder", b"big"), ValueError, "byteorder"),
        "/unaligned.pt": (_rezipped(image), ValueError, "16-byte aligned"),
        "/size.pt": (_with_record(image, "data/1", bytes(8)), ValueError, "28 bytes, its record holds 8"),
        "/missing.pt": (_with_record(image, "data.pkl", pkl.replace(b"X\x01\x00\x00\x001", b"X\x01\x00\x00\x007")),
                        ValueError, "has no record"),
        "/evil.pt": (evil, pickle.UnpicklingError, "print"),
        "/future.pt": (_with_record(image, "version", b"99\n"), ValueError, "version 99"),
    }
    assert b"X\x01\x00\x00\x001" in pkl

    async def run():
        async with volume_with({p: img for p, (img, _, _) in bad.items()}) as (client, stub, faults):
            for path, (_, exc, match) in bad.items():
                faults["gets"] = 0
                before = len(stub.get_file_calls)
                with pytest.raises(exc, match=match):
                    await _read(client, path)
                calls = stub.get_file_calls[before:]
                # the size probe, then host reads of the structure only: every GET was one of theirs
                assert 2 <= len(calls) <= 4 and calls[0].len == 1, path
                assert faults["gets"] == sum(_nblocks(c) for c in calls[1:]), path
                assert not [c for c in read_backend.calls if c[0] == "host_alloc"], path
            with pytest.raises(FileNotFoundError):
                await _read(client, "/nope")
            got = await volume.read_torch_save(client, "vo-r", "/evil.pt", weights_only=False, staging_bytes=STAGING)
            assert isinstance(got["evil"], type(None)) and torch.equal(got["w"], torch.ones(3))

    asyncio.run(run())


def _nblocks(call) -> int:
    return (call.start + call.len - 1) // BS - call.start // BS + 1


def _flip(image: bytes, at: int) -> bytes:
    b = bytearray(image)
    b[at] ^= 0x40
    return bytes(b)


def test_corruption_is_found(read_backend, monkeypatch):
    sd = {"a": torch.arange(5000, dtype=torch.float32), "b": torch.arange(3 * BS, dtype=torch.int16)}
    image = saved(sd)
    z = zipfile.ZipFile(io.BytesIO(image))
    info = {i.filename: i for i in z.infolist()}

    def data_at(name):
        i = info[name]
        return i.header_offset + 30 + len(i.filename.encode()) + int.from_bytes(
            image[i.header_offset + 28 : i.header_offset + 30], "little")

    with monkeypatch.context() as m:
        m.setattr(config.save, "compute_crc32", False)
        image_nocrc = saved(sd)
    renamed = image.replace(b"archive/data/1", b"archive/data/9", 1)  # the local header only (it comes first)
    assert renamed.count(b"archive/data/9") == 1
    files = {
        "/storage.pt": _flip(image, data_at("archive/data/1") + 2 * BS + 5),
        "/pkl.pt": _flip(image, data_at("archive/data.pkl") + 3),
        "/renamed.pt": renamed,
        "/nocrc.pt": _flip(image_nocrc, data_at("archive/data/1") + 2 * BS + 5),
    }

    async def read(path):
        async with volume_with({path: files[path]}) as (client, _, _):  # one file per server: equal sizes
            return await _read(client, path)

    with pytest.raises(ExecutionError, match=r"archive/data/1 \(stored [0-9a-f]{8}, computed") as err:
        asyncio.run(read("/storage.pt"))
    assert "data/0" not in str(err.value) and read_backend.live_buffers == 0
    read_backend.calls.clear()
    with pytest.raises(ExecutionError, match="archive/data.pkl"):
        asyncio.run(read("/pkl.pt"))
    assert not loads(read_backend)
    with pytest.raises(ValueError, match="local header of 'archive/data/1'"):
        asyncio.run(read("/renamed.pt"))
    assert read_backend.live_buffers == 0
    got = asyncio.run(read("/nocrc.pt"))
    assert not torch.equal(got["b"], sd["b"])  # no CRC to check: the flipped byte is loaded
    _assert_same(got, torch.load(io.BytesIO(files["/nocrc.pt"])))


def test_the_staging_buffer_is_freed_when_a_data_get_fails(read_backend, no_sleep):
    image = saved(_many(40))

    async def run():
        async with volume_with({"/m.pt": image}) as (client, stub, _):
            await _read(client, "/m.pt")
            structure = len(stub.get_file_calls) - 1  # the calls before the data region's
            stub.get_file_calls.clear()
            real = stub.VolumeGetFile2

            async def failing_data(req):
                if len(stub.get_file_calls) == structure:
                    stub.token_version["/m.pt"] = "error-500"
                return await real(req)

            stub.VolumeGetFile2 = failing_data
            with pytest.raises(ExecutionError, match="500"):
                await _read(client, "/m.pt")
            assert [c[0] for c in read_backend.calls].count("host_alloc") == 2 and read_backend.live_buffers == 0

    asyncio.run(run())
