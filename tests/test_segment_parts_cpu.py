"""Files made of many device buffers, on the CPU: the safetensors image of ``DeviceFile.safetensors`` against the
safetensors library, the part / wave split of b200h_segment_parts_preview against a plain restatement, and the
volumefs2 path with one ``hash_segment_parts_device`` call per batch, with CPU tensors standing in for GPU memory and
the oracle standing in for the GPU."""
import asyncio
import ctypes
import hashlib
import io
import json
import random
import types
from pathlib import PurePosixPath

import numpy as np
import pytest
import torch

safetensors_torch = pytest.importorskip("safetensors.torch")

from modal_client_b200 import DeviceFile, _lib, blob_utils, device_file, volume  # noqa: E402
from modal_client_b200.synth import synth_bytes  # noqa: E402
from tests.blob_server import running_blob_server  # noqa: E402
from tests.test_device_file_cpu import (  # noqa: E402,F401 (fake_device_backend: a fixture)
    FakeDeviceContext, HostDeviceFile, _trimmed_total, _volume_server, fake_device_backend, host_segments_file)
from tests.test_volume_upload import FakeVolumeStub  # noqa: E402

GATHERED = int(_lib.GATHERED)


# every dtype safetensors.torch.save stores, as this torch spells it
ST_DTYPES = [getattr(torch, n) for n in ("bool", "uint8", "int8", "int16", "uint16", "int32", "uint32", "int64",
                                          "uint64", "float16", "bfloat16", "float32", "float64", "complex64",
                                          "float8_e4m3fn", "float8_e5m2", "float8_e8m0fnu", "float4_e2m1fn_x2")
             if hasattr(torch, n)]
NOT_LOADABLE = {getattr(torch, n) for n in ("float8_e8m0fnu", "float4_e2m1fn_x2") if hasattr(torch, n)}
NAMES = ["w", "bias", "layer.0.attn.q_proj.weight", "ß", "层.权重", "emb😀", "a\"b\\c", "tab\tnl\n", "Z", "z", "_",
         "model.norm"]


def _rand_tensor(rng: random.Random, dtype, shape):
    numel = int(np.prod(shape)) if shape else 1
    esize = torch.empty(0, dtype=dtype).element_size()
    raw = torch.tensor(list(rng.randbytes(numel * esize)), dtype=torch.uint8)
    if rng.random() < 0.3 and raw.numel():
        raw[rng.randrange(raw.numel()):] = 0  # zero tails: trimming happens across tensor edges
    return raw.view(dtype).reshape(shape)


def _rand_state_dict(rng: random.Random, n: int) -> dict:
    d = {}
    while len(d) < n:
        name = rng.choice(NAMES) + (str(len(d)) if rng.random() < 0.7 else "")
        shape = rng.choice([(), (0,), (3, 0), (1,), (7,), (4, 5), (2, 3, 9), (rng.randrange(1, 300),)])
        d[name] = _rand_tensor(rng, rng.choice(ST_DTYPES), shape)
    return d


def _bytes_of(t: torch.Tensor) -> bytes:
    return bytes(t.reshape(-1).view(torch.uint8).numpy().tobytes())


# ------------------------------------------------------------------------------------------------ C ABI


def test_segment_entries_are_exported_and_reject_a_null_context():
    L = _lib.load_library()
    for s in ("b200h_hash_segment_parts_device", "b200h_segment_parts_preview"):
        assert hasattr(L, s) and s in _lib.ABI_SYMBOLS
    got = ctypes.c_uint64(12345)
    segs = (ctypes.c_uint64 * 4)(0, 0, 0, 0)
    first = (ctypes.c_uint64 * 2)(0, 2)
    for part_len in (0, 8 << 20):
        rc = L.b200h_hash_segment_parts_device(None, segs, 2, first, 1, part_len, _lib.SHA256 | _lib.TRIM_ZEROS, None,
                                               None, None, ctypes.byref(got), None)
        assert rc == -1  # B200H_E_INVALID
        assert got.value == 12345  # nothing written


# ---------------------------------------------------------------------------------------------- splitting


def restated_split(seg_lens, first, part_len, wave_bytes):
    """What the header promises, restated: parts per file, in place iff inside one segment, waves over contiguous
    rows, a new wave at the gathered part that would overflow the staged bytes (16-byte granules)."""
    seg, wave = [], []
    w, used = 0, 0
    for f in range(len(first) - 1):
        lens = seg_lens[first[f] : first[f + 1]]
        starts = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64) if lens else np.zeros(1, np.int64)
        size = int(starts[-1])
        for o in range(0, size, part_len):
            end = min(size, o + part_len)
            holders = [k for k in range(len(lens)) if starts[k] <= o < starts[k + 1]]
            k = holders[0]
            if end <= starts[k + 1]:
                seg.append(first[f] + k)
            else:
                seg.append(GATHERED)
                need = (end - o + 15) // 16 * 16
                if used and used + need > wave_bytes:
                    w, used = w + 1, 0
                used += need
            wave.append(w)
    return seg, wave, (w + 1 if seg else 0)


def _random_layout(rng: random.Random, part_len: int):
    nfiles = rng.randrange(0, 6)
    seg_lens, first = [], [0]
    for _ in range(nfiles):
        for _ in range(rng.randrange(0, 9)):
            seg_lens.append(rng.choice([0, 0, 1, 15, 16, 17, part_len - 1, part_len, part_len + 1, 3 * part_len,
                                        rng.randrange(1, 4 * part_len)]))
        first.append(len(seg_lens))
    return seg_lens, first


def test_preview_equals_the_restated_split():
    rng = random.Random(7)
    for trial in range(400):
        part_len = rng.choice([1, 7, 16, 64, 1000])
        seg_lens, first = _random_layout(rng, part_len)
        total = sum(seg_lens)
        for wave_bytes in (1, 16, part_len, 3 * part_len + 5, 16 * (total + 1) + 16):
            seg, wave, nwaves = _lib.segment_parts_preview(seg_lens, first, part_len, wave_bytes)
            want_seg, want_wave, want_n = restated_split(seg_lens, first, part_len, wave_bytes)
            assert seg.tolist() == want_seg and wave.tolist() == want_wave and nwaves == want_n, (seg_lens, first,
                                                                                                  part_len, wave_bytes)


def test_preview_edge_layouts():
    # segments ending exactly on part edges: every part in place, one wave
    seg, wave, n = _lib.segment_parts_preview([64, 128, 0, 64], [0, 4], 64, 1 << 20)
    assert seg.tolist() == [0, 1, 1, 3] and wave.tolist() == [0] * 4 and n == 1
    # one part over three segments (and an empty one between them)
    seg, _, n = _lib.segment_parts_preview([10, 0, 20, 30], [0, 4], 64, 1 << 20)
    assert seg.tolist() == [GATHERED] and n == 1
    # zero-byte files have no parts; a file of empty segments neither
    seg, wave, n = _lib.segment_parts_preview([0, 0, 5], [0, 0, 2, 2, 3], 4, 1 << 20)
    assert seg.tolist() == [2, 2] and n == 1
    seg, wave, n = _lib.segment_parts_preview([], [0, 0], 4, 1 << 20)
    assert seg.size == 0 and n == 0
    # wave caps: one gathered part per wave up to all of them in one
    lens = [5, 5] * 6
    first = [0, 2, 4, 6, 8, 10, 12]
    for cap, waves in ((1, 6), (16, 6), (32, 3), (48, 2), (96, 1), (1 << 30, 1)):
        seg, wave, n = _lib.segment_parts_preview(lens, first, 10, cap)
        assert (seg == GATHERED).all() and n == waves and wave.tolist() == [i * waves // 6 for i in range(6)]


@pytest.mark.parametrize("args", [
    ([1, 2], [1, 2], 4, 64),     # file_first_seg does not start at 0
    ([1, 2], [0, 1], 4, 64),     # ... does not end at nsegs
    ([1, 2], [0, 2, 1, 2], 4, 64),  # ... decreases
    ([1, 2], [0, 2], 0, 64),     # part_len 0
    ([1, 2], [0, 2], 4, 0),      # wave_bytes 0
])
def test_preview_rejects_bad_arguments(args):
    with pytest.raises(_lib.B200HashError):
        _lib.segment_parts_preview(*args)


# ------------------------------------------------------------------------------------------- safetensors


@pytest.mark.parametrize("seed", range(12))
def test_safetensors_image_equals_the_library(seed):
    rng = random.Random(seed)
    sd = _rand_state_dict(rng, rng.choice([0, 1, 2, 5, 17, 64]))
    for metadata in (None, {}, {"format": "pt"}, {"ß": "ü \"q\"", "a": "1", "B": ""}):
        want = safetensors_torch.save(sd, metadata)
        f = HostDeviceFile.safetensors(sd, metadata, ctx=FakeDeviceContext(), bounce_bytes=rng.choice([1, 7, 100]))
        got = f.read()
        if not sd and metadata == {}:
            # safetensors 0.7.0 writes the invalid header '{},"__metadata__":{}}' here; ours is the JSON it means
            assert got == b'\x18' + bytes(7) + b'{"__metadata__":{}}     '
        elif metadata is None or len(metadata) <= 1:
            assert got == want
        else:  # the library writes several metadata entries in no fixed order: same header, same data
            n = int.from_bytes(want[:8], "little")
            assert got[:8] == want[:8] and got[8 + n :] == want[8 + n :]
            assert json.loads(got[8 : 8 + n]) == json.loads(want[8 : 8 + n])
        if any(t.dtype in NOT_LOADABLE for t in sd.values()):
            continue  # the library writes these dtypes but cannot read them back
        back = safetensors_torch.load(got)
        assert back.keys() == sd.keys()
        for k, t in sd.items():
            assert back[k].dtype == t.dtype and back[k].shape == t.shape and _bytes_of(back[k]) == _bytes_of(t)
        assert f.bytes_to_host == len(got)


def test_safetensors_random_reads_across_segment_edges():
    rng = random.Random(3)
    sd = _rand_state_dict(rng, 40)
    want = safetensors_torch.save(sd)
    for bounce in (1, 5, 64, 4096):
        f, ref = HostDeviceFile.safetensors(sd, ctx=FakeDeviceContext(), bounce_bytes=bounce), io.BytesIO(want)
        for _ in range(150):
            op = rng.randrange(3)
            if op == 0:
                off = rng.randrange(0, len(want) + 50)
                assert f.seek(off) == ref.seek(off)
            elif op == 1:
                n = rng.choice([0, 1, 3, 8, 100, 999, -1])
                assert f.read(n) == ref.read(n)
            else:
                a, b = bytearray(rng.randrange(0, 2000)), None
                b = bytearray(len(a))
                assert f.readinto(a) == ref.readinto(b) and a == b
            assert f.tell() == ref.tell()
    r = f.reopen()
    assert r.read() == want and r.nbytes == len(want)


def test_safetensors_dtype_order_and_header():
    """The data order is dtype rank (descending), then name; the header is padded with spaces to a multiple of 8."""
    sd = {f"t_{str(dt).split('.')[-1]}": _rand_tensor(random.Random(1), dt, (2,)) for dt in ST_DTYPES}
    want = safetensors_torch.save(sd)
    header, ordered = device_file.safetensors_layout(sd)
    n = int.from_bytes(want[:8], "little")
    assert header == want[: 8 + n] and len(header) % 8 == 0
    lib_order = [k for k in json.loads(want[8 : 8 + n])]
    assert [k for k, _ in ordered] == lib_order
    assert device_file.safetensors_layout({})[0] == safetensors_torch.save({})  # b"{}" padded to 8 bytes


def test_safetensors_shared_storage_is_read_twice():
    base = _rand_tensor(random.Random(2), torch.float32, (64,))
    sd = {"a": base[:40], "b": base[40:], "c": base[10:20]}
    f = HostDeviceFile.safetensors(sd, ctx=FakeDeviceContext())
    back = safetensors_torch.load(f.read())
    assert all(_bytes_of(back[k]) == _bytes_of(sd[k]) for k in sd)
    disjoint = {"a": base[:40], "b": base[40:]}
    assert HostDeviceFile.safetensors(disjoint, ctx=FakeDeviceContext()).read() == safetensors_torch.save(disjoint)


def test_safetensors_rejections_name_what_is_wrong():
    ctx = FakeDeviceContext()
    ok = torch.zeros(4)
    with pytest.raises(ValueError, match="'w'.*CUDA"):
        DeviceFile.safetensors({"w": ok})  # a CPU tensor where GPU memory is expected
    with pytest.raises(ValueError, match="'nc'.*contiguous"):
        HostDeviceFile.safetensors({"x": ok, "nc": torch.zeros(4, 4).t()}, ctx=ctx)
    with pytest.raises(ValueError, match="cuda:3"):
        HostDeviceFile.safetensors({"x": ok}, ctx=types.SimpleNamespace(device=3))
    with pytest.raises(ValueError, match="7"):
        HostDeviceFile.safetensors({7: ok}, ctx=ctx)
    with pytest.raises(ValueError, match="'k'"):
        HostDeviceFile.safetensors({"x": ok}, {"k": 1}, ctx=ctx)
    with pytest.raises(ValueError, match="'c'.*complex128"):
        HostDeviceFile.safetensors({"x": ok, "c": torch.zeros(2, dtype=torch.complex128)}, ctx=ctx)
    with pytest.raises(ValueError, match="__metadata__"):
        HostDeviceFile.safetensors({"__metadata__": ok}, ctx=ctx)
    with pytest.raises(ValueError, match="'x'"):
        HostDeviceFile.safetensors({"x": [1, 2]}, ctx=ctx)


# ------------------------------------------------------------------------------------------------ specs


def _edge_state_dicts(BS: int):
    """blocks.json-style edges: trailing zeros ending on a block edge, all-zero blocks, one-byte tails, many tiny
    tensors inside one block, a tensor spanning several blocks, empty and 0-d tensors."""
    u8 = lambda b: torch.frombuffer(bytearray(b), dtype=torch.uint8) if b else torch.zeros(0, dtype=torch.uint8)  # noqa: E731
    yield {}
    yield {"x": u8(b"a")}
    yield {"big": u8(synth_bytes(1, 3 * BS + 77)), "z": u8(bytes(2 * BS)), "tail": u8(b"q")}
    yield {f"n{i:03d}": u8(synth_bytes(i, 1 + i % 13) + bytes(i % 5)) for i in range(300)}
    yield {"a": u8(b"a" * (BS - 5) + bytes(5)), "b": u8(bytes(BS)), "c": torch.zeros(()), "d": torch.zeros(0, 4),
           "e": u8(synth_bytes(9, BS // 2))}
    rng = random.Random(11)
    yield _rand_state_dict(rng, 50)


def test_spec2_of_safetensors_file_equals_spec2_of_bytesio(fake_device_backend, monkeypatch):
    BS = 4096
    monkeypatch.setattr(blob_utils, "BLOCK_SIZE", BS)
    for sd in _edge_state_dicts(BS):
        image = safetensors_torch.save(sd)
        f = HostDeviceFile.safetensors(sd, ctx=fake_device_backend)
        sem = asyncio.Semaphore(1)
        dev = asyncio.run(blob_utils.FileUploadSpec2.from_fileobj(f, PurePosixPath("/m.safetensors"), sem, 0o644))
        host = asyncio.run(blob_utils.FileUploadSpec2.from_fileobj(io.BytesIO(image), PurePosixPath("/m.safetensors"),
                                                                   sem, 0o644))
        assert (dev.blocks, dev.size, dev.mode, dev.path) == (host.blocks, host.size, host.mode, host.path)
        assert f.bytes_to_host == 0  # only the digest table was fetched
        with dev.source() as rd:
            assert rd.read() == image
    assert ("hash_segment_parts_device", 1, BS, _lib.SHA256 | _lib.TRIM_ZEROS) in fake_device_backend.calls


def test_batch_of_device_files_makes_one_call(fake_device_backend, monkeypatch):
    BS = 4096
    monkeypatch.setattr(blob_utils, "BLOCK_SIZE", BS)
    sds = list(_edge_state_dicts(BS))
    images = [safetensors_torch.save(sd) for sd in sds]
    plain = [synth_bytes(40 + i, n) for i, n in enumerate((0, 1, BS, 3 * BS + 1))]
    for k in (1, 2, 5, len(sds) + len(plain)):
        files = [HostDeviceFile.safetensors(sd, ctx=fake_device_backend) for sd in sds]
        files += [host_segments_file([p]) for p in plain]
        datas = images + plain
        items = [(f, PurePosixPath(f"/f{i}"), 0o600) for i, f in enumerate(files[:k])]
        fake_device_backend.calls.clear()
        specs = asyncio.run(blob_utils.device_file_specs2(items))
        dev_calls = [c for c in fake_device_backend.calls if c[0].startswith("hash_")]
        assert len(dev_calls) == (1 if any(len(d) for d in datas[:k]) else 0)
        for spec, data, (f, remote, _) in zip(specs, datas, items):
            want = asyncio.run(blob_utils.FileUploadSpec2.from_fileobj(io.BytesIO(data), remote, asyncio.Semaphore(1),
                                                                       0o600))
            assert (spec.blocks, spec.size, spec.mode, spec.path) == (want.blocks, want.size, want.mode, want.path)
            assert f.bytes_to_host == 0


def test_v2_round_puts_only_missing_blocks_of_a_safetensors_file(fake_device_backend, monkeypatch):
    BS = 4096
    monkeypatch.setattr(blob_utils, "BLOCK_SIZE", BS)
    sd = _rand_state_dict(random.Random(21), 40)
    sd["zeros"] = torch.zeros(3 * BS, dtype=torch.uint8)
    sd["big"] = torch.frombuffer(bytearray(synth_bytes(5, 5 * BS + 11)), dtype=torch.uint8)
    image = safetensors_torch.save(sd)
    nblocks = -(-len(image) // BS)

    async def run():
        async with _volume_server(BS) as (stub, _):
            client = types.SimpleNamespace(stub=stub)
            f = HostDeviceFile.safetensors(sd, ctx=fake_device_backend, bounce_bytes=1000)
            extra = host_segments_file([b"x" * 100, synth_bytes(2, 2 * BS)])
            async with volume.VolumeUploadContextManager2("vo-s", client) as batch:
                batch.put_file(io.BytesIO(b"plain"), "/p")
                batch.put_file(f, "/ckpt/model.safetensors")
                batch.put_file(extra, "/ckpt/extra.bin")
            assert stub.volume_files["/ckpt/model.safetensors"][0] == image
            assert stub.volume_files["/ckpt/extra.bin"][0] == b"x" * 100 + synth_bytes(2, 2 * BS)
            assert stub.volume_files["/p"][0] == b"plain"
            assert f.bytes_to_host == _trimmed_total(image, BS)
            assert sum(c[0] == "hash_segment_parts_device" for c in fake_device_backend.calls) == 1
            # one tensor changes: only the blocks holding its bytes travel again
            sd["big"][7] ^= 0xFF
            image2 = safetensors_torch.save(sd)
            changed = [i for i in range(nblocks) if image2[i * BS : (i + 1) * BS] != image[i * BS : (i + 1) * BS]]
            g = HostDeviceFile.safetensors(sd, ctx=fake_device_backend)
            before = stub.block_puts
            async with volume.VolumeUploadContextManager2("vo-s", client, force=True) as batch:
                batch.put_file(g, "/ckpt/model.safetensors")
            assert stub.block_puts == before + len(changed) and len(changed) == 1
            assert g.bytes_to_host == _trimmed_total(image2, BS, changed)
            assert stub.volume_files["/ckpt/model.safetensors"][0] == image2

    asyncio.run(run())


def test_v1_put_file_of_a_safetensors_file(fake_device_backend, monkeypatch):
    monkeypatch.setattr(blob_utils, "LARGE_FILE_LIMIT", 4000)
    sd = _rand_state_dict(random.Random(8), 30)
    sd["w"] = torch.frombuffer(bytearray(synth_bytes(3, 20_000)), dtype=torch.uint8)
    image = safetensors_torch.save(sd)

    async def run():
        async with running_blob_server() as (host, store):
            stub = FakeVolumeStub(host, store, 8 << 20)
            client = types.SimpleNamespace(stub=stub)
            async with volume.VolumeUploadContextManager("vo-1", client) as batch:
                batch.put_file(HostDeviceFile.safetensors(sd, ctx=fake_device_backend, bounce_bytes=1 << 12), "/m")
            got, _, sha = stub.volume_files["/m"]
            assert got == image and sha == hashlib.sha256(image).hexdigest()
            await blob_utils.ClientSessionRegistry.close_session()

    asyncio.run(run())
