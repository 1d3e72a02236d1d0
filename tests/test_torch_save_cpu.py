"""``DeviceFile.torch_save`` on the CPU: the image against ``torch.save(obj, BytesIO())`` byte for byte, reads, round
trips and the volumefs2 path, with CPU tensors standing in for GPU memory and ``zlib.crc32`` standing in for
``b200h_crc32_device``."""
import asyncio
import ctypes
import io
import pickle
import random
import types
import zipfile
from pathlib import PurePosixPath

import numpy as np
import pytest
import torch
from torch.utils.serialization import config

from modal_client_b200 import _lib, blob_utils, device_file, volume
from modal_client_b200.synth import synth_bytes
from tests.test_device_file_cpu import (  # noqa: F401 (fake_device_backend: a fixture)
    FakeDeviceContext, HostDeviceFile, _trimmed_total, _volume_server, fake_device_backend, host_segments_file)

safetensors_torch = pytest.importorskip("safetensors.torch")


def saved(obj) -> bytes:
    b = io.BytesIO()
    torch.save(obj, b)
    return b.getvalue()


# every dtype torch.save stores (quantized dtypes aside)
SAVE_DTYPES = [getattr(torch, n) for n in (
    "bool", "uint8", "int8", "int16", "uint16", "int32", "uint32", "int64", "uint64", "float16", "bfloat16", "float32",
    "float64", "complex32", "complex64", "complex128", "float8_e4m3fn", "float8_e5m2", "float8_e4m3fnuz",
    "float8_e5m2fnuz", "float8_e8m0fnu", "float4_e2m1fn_x2", "bits8", "bits16") if hasattr(torch, n)]


def _rand(rng: random.Random, dtype, shape):
    numel = int(np.prod(shape)) if shape else 1
    esize = torch.empty(0, dtype=dtype).element_size()
    raw = torch.tensor(list(rng.randbytes(numel * esize)), dtype=torch.uint8)
    return raw.view(dtype).reshape(shape)


def _state_dict(seed: int, n: int) -> dict:
    rng = random.Random(seed)
    return {f"layer.{i}.w": _rand(rng, rng.choice(SAVE_DTYPES), rng.choice([(), (0,), (1,), (7,), (4, 5), (2, 3, 9),
                                                                              (rng.randrange(1, 3000),)]))
            for i in range(n)}


def _adam_state() -> dict:
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(8, 16), torch.nn.ReLU(), torch.nn.Linear(16, 3))
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    for _ in range(2):
        model(torch.randn(4, 8)).sum().backward()
        opt.step()
    return {"model": model.state_dict(), "optim": opt.state_dict(), "step": 2}


def _cases():
    base = torch.arange(64, dtype=torch.float32)
    m = torch.arange(30.0).reshape(5, 6)
    yield "dtypes", _state_dict(1, len(SAVE_DTYPES) * 2)
    yield "every_dtype_once", {str(dt): _rand(random.Random(2), dt, (3,)) for dt in SAVE_DTYPES}
    yield "empty_and_0d", {"e": torch.zeros(0), "e2": torch.zeros(3, 0, dtype=torch.int8), "s": torch.tensor(3.5),
                           "i": torch.tensor(7)}
    yield "views", {"off": base[10:20], "t": m.t(), "strided": m[:, ::2], "row": m[3]}
    yield "shared", {"a": base[:40], "b": base[40:], "c": base[10:20], "d": base.view(8, 8)}
    yield "many_storages", {f"k{i}": torch.full((i + 1,), float(i)) for i in range(23)}
    yield "nested", {"cfg": {"lr": 0.1, "name": "run-7", "sizes": [1, 2, 3]}, "tensors": [torch.ones(3), (torch.eye(2),)],
                     "n": 12, "s": "text"}
    yield "adam", _adam_state()
    yield "no_tensors", {"a": 1, "b": [2, "three"]}
    yield "bare_tensor", torch.arange(1000, dtype=torch.int16)
    yield "dtypes_seed5", _state_dict(5, 40)


CASES = dict(_cases())


@pytest.mark.parametrize("name", list(CASES))
def test_image_equals_torch_save(name):
    obj = CASES[name]
    want = saved(obj)
    ctx = FakeDeviceContext()
    f = HostDeviceFile.torch_save(obj, ctx=ctx, bounce_bytes=random.Random(name).choice([1, 7, 100, 1 << 20]))
    assert f.nbytes == len(want)
    got = f.read()
    assert got == want
    assert f.bytes_to_host == len(got)
    names = zipfile.ZipFile(io.BytesIO(got)).namelist()
    assert all(n.startswith("archive/") for n in names)
    crc_calls = [c for c in ctx.calls if c[0] == "crc32_device"]
    has_storages = any(n.startswith("archive/data/") for n in names)
    assert len(crc_calls) == (2 if has_storages else 0)  # the storages, then the serialization id


def test_keys_ten_and_up_follow_nine():
    sd = {f"k{i}": torch.full((2,), float(i)) for i in range(12)}
    names = zipfile.ZipFile(io.BytesIO(HostDeviceFile.torch_save(sd, ctx=FakeDeviceContext()).read())).namelist()
    data = [n for n in names if n.startswith("archive/data/")]
    assert data == [f"archive/data/{i}" for i in range(12)]


def test_without_crc32_the_skeleton_is_the_file(monkeypatch):
    monkeypatch.setattr(config.save, "compute_crc32", False)
    obj = _adam_state()
    want = saved(obj)
    ctx = FakeDeviceContext()
    f = HostDeviceFile.torch_save(obj, ctx=ctx)
    assert f.read() == want
    assert not [c for c in ctx.calls if c[0] == "crc32_device"]
    assert all(i.CRC == 0 for i in zipfile.ZipFile(io.BytesIO(want)).infolist())


def test_storage_keys_pickler_pickles_like_pickle():
    for obj in (CASES["nested"], CASES["adam"], CASES["shared"]):
        keys = device_file._StorageKeys()
        b = io.BytesIO()
        torch.save(obj, b, pickle_module=keys)
        plain = io.BytesIO()
        torch.save(obj, plain, pickle_module=pickle)
        assert b.getvalue() == plain.getvalue() == saved(obj)
        assert list(keys.keys) == [str(i) for i in range(len(keys.keys))]


def test_random_reads_across_segment_edges():
    rng = random.Random(3)
    obj = {"sd": _state_dict(9, 30), "opt": _adam_state()}
    want = saved(obj)
    for bounce in (1, 5, 64, 4096):
        f, ref = HostDeviceFile.torch_save(obj, ctx=FakeDeviceContext(), bounce_bytes=bounce), io.BytesIO(want)
        for _ in range(150):
            op = rng.randrange(3)
            if op == 0:
                off = rng.randrange(0, len(want) + 50)
                assert f.seek(off) == ref.seek(off)
            elif op == 1:
                n = rng.choice([0, 1, 3, 8, 100, 999, -1])
                assert f.read(n) == ref.read(n)
            else:
                a = bytearray(rng.randrange(0, 2000))
                b = bytearray(len(a))
                assert f.readinto(a) == ref.readinto(b) and a == b
            assert f.tell() == ref.tell()
    assert f.reopen().read() == want


def test_torch_load_round_trip():
    obj = _adam_state()
    obj["views"] = CASES["views"]
    back = torch.load(io.BytesIO(HostDeviceFile.torch_save(obj, ctx=FakeDeviceContext()).read()), weights_only=True)
    for k, t in obj["model"].items():
        assert torch.equal(back["model"][k], t)
    assert back["optim"]["param_groups"] == obj["optim"]["param_groups"]
    for i, st in obj["optim"]["state"].items():
        for k, v in st.items():
            assert torch.equal(back["optim"]["state"][i][k], v)
    assert back["step"] == 2
    for k, t in obj["views"].items():
        assert torch.equal(back["views"][k], t) and back["views"][k].stride() == t.stride()


def test_rejections_name_the_device():
    with pytest.raises(ValueError, match="meta"):
        HostDeviceFile.torch_save({"w": torch.zeros(4, device="meta")}, ctx=FakeDeviceContext())


def test_layout_check_rejects_a_compressed_archive():
    b = io.BytesIO()
    with zipfile.ZipFile(b, "w", zipfile.ZIP_DEFLATED) as z:
        z.writestr("archive/data.pkl", b"x" * 1000)
    image = b.getvalue()
    with pytest.raises(ValueError, match="uncompressed"):
        device_file._parse_zip(device_file._Skeleton([(0, bytearray(image))]), len(image))


def test_crc_entry_is_exported_and_rejects_a_null_context():
    L = _lib.load_library()
    assert hasattr(L, "b200h_crc32_device") and "b200h_crc32_device" in _lib.ABI_SYMBOLS
    ranges = (ctypes.c_uint64 * 4)(0, 0, 0, 0)
    out = (ctypes.c_uint32 * 2)(7, 7)
    for n in (0, 2):
        assert L.b200h_crc32_device(None, ranges, n, out, None) == -1  # B200H_E_INVALID
    assert list(out) == [7, 7]


# ------------------------------------------------------------------------------------------------ volumefs2


def _edge_checkpoints(BS: int):
    u8 = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8) if b else torch.zeros(0, dtype=torch.uint8)  # noqa: E731
    yield {}
    yield {"big": u8(synth_bytes(1, 3 * BS + 77)), "z": u8(bytes(2 * BS)), "tail": u8(b"q")}
    yield {f"n{i:03d}": u8(synth_bytes(i, 1 + i % 13) + bytes(i % 5)) for i in range(40)}
    yield _adam_state()
    yield _state_dict(11, 30)


def test_spec2_of_torch_save_file_equals_spec2_of_bytesio(fake_device_backend, monkeypatch):
    BS = 4096
    monkeypatch.setattr(blob_utils, "BLOCK_SIZE", BS)
    for obj in _edge_checkpoints(BS):
        image = saved(obj)
        f = HostDeviceFile.torch_save(obj, ctx=fake_device_backend)
        sem = asyncio.Semaphore(1)
        dev = asyncio.run(blob_utils.FileUploadSpec2.from_fileobj(f, PurePosixPath("/c.pt"), sem, 0o644))
        host = asyncio.run(blob_utils.FileUploadSpec2.from_fileobj(io.BytesIO(image), PurePosixPath("/c.pt"), sem,
                                                                   0o644))
        assert (dev.blocks, dev.size, dev.mode, dev.path) == (host.blocks, host.size, host.mode, host.path)
        assert f.bytes_to_host == 0
        with dev.source() as rd:
            assert rd.read() == image


def test_batch_of_torch_save_safetensors_and_plain_makes_one_call(fake_device_backend, monkeypatch):
    BS = 4096
    monkeypatch.setattr(blob_utils, "BLOCK_SIZE", BS)
    ckpt = _adam_state()
    sd = {"w": torch.frombuffer(bytearray(synth_bytes(4, 3 * BS + 5)), dtype=torch.uint8), "b": torch.ones(7)}
    plain = synth_bytes(6, 2 * BS + 1)
    files = [HostDeviceFile.torch_save(ckpt, ctx=fake_device_backend),
             HostDeviceFile.safetensors(sd, ctx=fake_device_backend), host_segments_file([plain])]
    datas = [saved(ckpt), safetensors_torch.save(sd), plain]
    items = [(f, PurePosixPath(f"/f{i}"), 0o600) for i, f in enumerate(files)]
    fake_device_backend.calls.clear()
    specs = asyncio.run(blob_utils.device_file_specs2(items))
    assert [c[0] for c in fake_device_backend.calls if c[0].startswith("hash_")] == ["hash_segment_parts_device"]
    for spec, data, (f, remote, _) in zip(specs, datas, items):
        want = asyncio.run(blob_utils.FileUploadSpec2.from_fileobj(io.BytesIO(data), remote, asyncio.Semaphore(1),
                                                                   0o600))
        assert (spec.blocks, spec.size) == (want.blocks, want.size)
        assert f.bytes_to_host == 0


def test_v2_round_puts_only_missing_blocks_of_a_torch_save_file(fake_device_backend, monkeypatch):
    BS = 4096
    monkeypatch.setattr(blob_utils, "BLOCK_SIZE", BS)
    ckpt = _adam_state()
    ckpt["big"] = torch.frombuffer(bytearray(synth_bytes(5, 5 * BS + 11)), dtype=torch.uint8)
    ckpt["zeros"] = torch.zeros(3 * BS, dtype=torch.uint8)
    image = saved(ckpt)
    nblocks = -(-len(image) // BS)

    async def run():
        async with _volume_server(BS) as (stub, _):
            client = types.SimpleNamespace(stub=stub)
            f = HostDeviceFile.torch_save(ckpt, ctx=fake_device_backend, bounce_bytes=1000)
            async with volume.VolumeUploadContextManager2("vo-t", client) as batch:
                batch.put_file(io.BytesIO(b"plain"), "/p")
                batch.put_file(f, "/ckpt/last.pt")
            assert stub.volume_files["/ckpt/last.pt"][0] == image
            assert f.bytes_to_host == _trimmed_total(image, BS)
            # one byte of one storage changes: its block, the CRC fields and the id change, nothing else
            ckpt["big"][7] ^= 0xFF
            image2 = saved(ckpt)
            changed = [i for i in range(nblocks) if image2[i * BS : (i + 1) * BS] != image[i * BS : (i + 1) * BS]]
            g = HostDeviceFile.torch_save(ckpt, ctx=fake_device_backend)
            before = stub.block_puts
            async with volume.VolumeUploadContextManager2("vo-t", client, force=True) as batch:
                batch.put_file(g, "/ckpt/last.pt")
            assert stub.block_puts == before + len(changed) and 1 <= len(changed) < nblocks
            assert g.bytes_to_host == _trimmed_total(image2, BS, changed)
            assert stub.volume_files["/ckpt/last.pt"][0] == image2

    asyncio.run(run())
