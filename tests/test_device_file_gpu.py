"""GPU: b200h_hash_fixed_parts_device is bit-exact against the host entry and the oracle; DeviceFile reads back the
tensor's bytes; a 1 GiB tensor uploads through volumefs2 with only the missing blocks' trimmed bytes crossing to the
host."""
import asyncio
import hashlib
import io
import random
import types
from pathlib import PurePosixPath

import numpy as np
import pytest

from modal_client_b200 import DeviceFile, _lib, blob_utils, volume
from modal_client_b200.synth import materialize, synth_array
from oracle import c_oracle
from tests.test_device_file_cpu import _volume_server

pytestmark = pytest.mark.gpu

MiB8 = 8 << 20


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0, pinned_bytes=64 << 20, device_bytes=512 << 20)
    yield c
    c.close()


def _buffer(n: int, seed: int) -> np.ndarray:
    """Synthetic bytes with zero runs where trimming matters: a zero tail before the first 8 MiB edge, an all-zero
    stretch, and a zero tail at the end."""
    a = synth_array(seed, n).copy()
    for lo, hi in ((MiB8 - 5000, MiB8), (MiB8 + 100, 2 * MiB8 + 100), (n - 3000, n), (n - 70, n - 3)):
        a[max(0, min(lo, n)) : max(0, min(hi, n))] = 0
    return a


def _device_parts(ctx, d, nbytes, part_len, flags, want_etag, stream=0):
    import torch

    n = -(-nbytes // part_len)
    dev = torch.device("cuda", 0)
    sha = torch.empty((n, 32), dtype=torch.uint8, device=dev)
    md5 = torch.empty((n, 16), dtype=torch.uint8, device=dev)
    trim = torch.empty(n, dtype=torch.int64, device=dev)
    etag = torch.empty(16, dtype=torch.uint8, device=dev)
    got = ctx.hash_fixed_parts_device(d, nbytes, part_len, flags, sha.data_ptr() if n else 0,
                                      md5.data_ptr() if n else 0, trim.data_ptr() if n else 0,
                                      etag.data_ptr() if want_etag else 0, stream)
    assert got == n
    torch.cuda.synchronize()
    return (sha.cpu().numpy() if flags & _lib.SHA256 else None, md5.cpu().numpy() if flags & _lib.MD5 else None,
            trim.cpu().numpy().astype(np.uint64), etag.cpu().numpy().tobytes() if want_etag else None)


LENGTHS = [0, 1, MiB8 - 1, MiB8, MiB8 + 1, 3 * MiB8 + 4711]
PART_LENS = [1, 64, MiB8, 100_003]  # 100_003: not a multiple of 64


@pytest.mark.parametrize("nbytes", LENGTHS)
@pytest.mark.parametrize("part_len", PART_LENS)
def test_fixed_parts_device_matches_host_entry_and_oracle(ctx, nbytes, part_len):
    import torch

    if part_len == 1 and nbytes > 1:
        nbytes = 4097  # one message per byte: ~10^7 one-byte parts would only time the oracle
    host = _buffer(nbytes, 900 + nbytes % 97)
    odd = torch.empty(nbytes + 1, dtype=torch.uint8, device="cuda:0")  # odd[1:]: an unaligned device address
    if nbytes:
        odd[1:] = torch.from_numpy(host).to("cuda:0")
    aligned = odd[1:].clone()
    starts = np.arange(0, nbytes, part_len, dtype=np.uint64)
    lens = np.minimum(part_len, nbytes - starts).astype(np.uint64)
    for trim in (False, True):
        want_s, want_m, want_e = c_oracle.hash_batch(host, starts, lens, trim=trim)
        for sel in (_lib.SHA256, _lib.MD5, _lib.SHA256 | _lib.MD5):
            flags = sel | (_lib.TRIM_ZEROS if trim else 0)
            etag = bool(sel & _lib.MD5)
            host_entry = ctx.hash_fixed_parts(host, part_len, flags, want_etag=etag)
            for base in (aligned.data_ptr(), odd.data_ptr() + 1):
                got = _device_parts(ctx, base, nbytes, part_len, flags, etag)
                for a, b in zip(got, host_entry):
                    assert (a is None and b is None) or np.array_equal(np.asarray(a), np.asarray(b))
                s, m, e, t = got
                assert np.array_equal(e, want_e)
                if sel & _lib.SHA256:
                    assert np.array_equal(s, want_s)
                if sel & _lib.MD5:
                    assert np.array_equal(m, want_m)
                    assert t == c_oracle.md5(want_m.tobytes() if len(want_m) else b"")


def test_fixed_parts_device_blank_block_fixture_and_argument_checks(ctx, golden):
    import torch

    case = golden("blocks.json")["spec2"][0]  # (b"a" + b"\0" * (8 MiB - 1)) * 2 + b"cdef"
    data = materialize(case["input"])
    assert data == (b"a" + bytes(MiB8 - 1)) * 2 + b"cdef"
    d = torch.frombuffer(bytearray(data), dtype=torch.uint8).to("cuda:0")
    s, _, e, _ = _device_parts(ctx, d.data_ptr(), len(data), MiB8, _lib.SHA256 | _lib.TRIM_ZEROS, False)
    assert [[i * MiB8, i * MiB8 + int(e[i]), s[i].tobytes().hex()] for i in range(len(e))] == case["blocks"]
    out = torch.empty(64, dtype=torch.uint8, device="cuda:0")
    with pytest.raises(_lib.B200HashError, match="part_len"):
        ctx.hash_fixed_parts_device(d.data_ptr(), len(data), 0, _lib.SHA256, out.data_ptr())
    with pytest.raises(_lib.B200HashError, match="aligned"):
        ctx.hash_fixed_parts_device(d.data_ptr(), 100, 64, _lib.SHA256, out.data_ptr() + 4)
    with pytest.raises(_lib.B200HashError, match="HEX"):
        ctx.hash_fixed_parts_device(d.data_ptr(), 100, 64, _lib.SHA256 | _lib.HEX_OUT, out.data_ptr())
    with pytest.raises(_lib.B200HashError, match="etag"):
        ctx.hash_fixed_parts_device(d.data_ptr(), 100, 64, _lib.SHA256, out.data_ptr(), 0, 0, out.data_ptr() + 32)
    host = np.zeros(4096, np.uint8)
    launches = ctx.launch_count
    with pytest.raises(_lib.B200HashError, match=r"\(-1\)"):  # host memory: rejected before anything is enqueued
        ctx.hash_fixed_parts_device(host.ctypes.data, 100, 64, _lib.SHA256, out.data_ptr())
    assert ctx.launch_count == launches


def test_fixed_parts_device_synchronises_only_where_the_header_says(ctx):
    """Without B200H_TRIM_ZEROS (ETag included) and with TRIM_ZEROS | NO_OUTLIERS the call only enqueues; TRIM_ZEROS
    with outlier routing may read the planner's count back once."""
    import torch

    n = 5 * MiB8 + 99
    d = torch.empty(n, dtype=torch.uint8, device="cuda:0")
    ctx.fill_synth_device(d.data_ptr(), n, seed=5)
    torch.cuda.synchronize()
    for flags, etag, may in ((_lib.SHA256 | _lib.MD5, True, 0), (_lib.SHA256, False, 0),
                             (_lib.SHA256 | _lib.TRIM_ZEROS | _lib.NO_OUTLIERS, False, 0),
                             (_lib.MD5 | _lib.TRIM_ZEROS | _lib.NO_OUTLIERS, True, 0),
                             (_lib.SHA256 | _lib.TRIM_ZEROS, False, 1)):
        before = ctx.plan_sync_count
        _device_parts(ctx, d.data_ptr(), n, MiB8, flags, etag)
        assert ctx.plan_sync_count - before <= may, flags


# ------------------------------------------------------------------------------------------- DeviceFile


@pytest.mark.parametrize("dtype", ["float16", "bfloat16", "uint8"])
def test_device_file_reads_back_the_tensor_bytes(gpu_backend, dtype):
    import torch

    g = torch.Generator(device="cuda:0").manual_seed(3)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):  # produced on another stream: reads must wait for it
        t = torch.randn((1234, 777), generator=g, device="cuda:0").to(getattr(torch, dtype)) if dtype != "uint8" else \
            torch.randint(0, 256, (5_000_011,), generator=g, device="cuda:0", dtype=torch.uint8)
        f = DeviceFile(t, bounce_bytes=1 << 16)
    first = f.read()  # no synchronisation before this read: the DeviceFile orders itself after `side`
    torch.cuda.synchronize()
    want = t.reshape(-1).view(torch.uint8).cpu().numpy().tobytes()
    assert first == want and f.bytes_to_host == len(want)
    f.seek(0)
    ref = io.BytesIO(want)
    rng = random.Random(7)
    for _ in range(200):
        op = rng.randrange(4)
        if op == 0:
            pos = rng.randrange(0, len(want) + 100)
            assert f.seek(pos) == ref.seek(pos)
        elif op == 1:
            n = rng.choice([0, 1, 15, 65536, 65537, 300_000, -1])
            assert f.read(n) == ref.read(n)
        elif op == 2:
            a = bytearray(rng.randrange(1, 200_000))
            b = bytearray(len(a))
            assert f.readinto(a) == ref.readinto(b) and a == b
        else:
            back = -rng.randrange(0, 5000)
            assert f.seek(back, io.SEEK_END) == ref.seek(back, io.SEEK_END)
        assert f.tell() == ref.tell()
    f.seek(0)
    assert f.read() == want
    with pytest.raises(OSError):
        f.fileno()


def test_device_file_rejects_non_contiguous_and_host_tensors(gpu_backend):
    import torch

    with pytest.raises(ValueError, match="contiguous"):
        DeviceFile(torch.zeros((64, 64), device="cuda:0").t())
    with pytest.raises(ValueError, match="CUDA"):
        DeviceFile(torch.zeros(64))


def test_spec2_from_device_file_matches_golden_blocks(gpu_backend, golden, monkeypatch):
    import torch

    for c in golden("blocks.json")["spec2"]:
        data = materialize(c["input"])
        t = torch.frombuffer(bytearray(data), dtype=torch.uint8).to("cuda:0") if data else \
            torch.empty(0, dtype=torch.uint8, device="cuda:0")
        f = DeviceFile(t)
        with monkeypatch.context() as mp:
            for k, v in c["patch"].items():
                mp.setattr(blob_utils, k, v)
            spec = asyncio.run(blob_utils.FileUploadSpec2.from_fileobj(f, PurePosixPath(c["path"]), asyncio.Semaphore(1),
                                                                       0o644))
        assert [[b.start, b.end, b.contents_sha256.hex()] for b in spec.blocks] == c["blocks"]
        assert spec.size == c["size"] and f.bytes_to_host == 0


# ----------------------------------------------------------------------------------------------- upload


def test_v2_put_file_of_a_1gib_tensor(gpu_backend):
    import torch

    n = 1 << 30
    t = torch.empty(n // 2, dtype=torch.float16, device="cuda:0")
    gpu_backend.fill_synth_device(t.data_ptr(), n, seed=41)
    torch.cuda.synchronize()
    u8 = t.view(torch.uint8)
    for i in range(n // MiB8):  # zero-filled tails of every length class, whole zero blocks, untouched blocks
        tail = [0, 1, 63, 64, 4096, MiB8 // 2, MiB8 - 1, MiB8][i % 8]
        if tail:
            u8[(i + 1) * MiB8 - tail : (i + 1) * MiB8] = 0
    host_bytes = u8.cpu().numpy().tobytes()
    seen = []

    async def run():
        async with _volume_server(MiB8) as (stub, _):
            record = stub.VolumePutFiles2

            async def recording(req):
                resp = await record(req)
                seen.append(([[(b.contents_sha256, b.put_response) for b in f.blocks] for f in req.files],
                             list(resp.missing_blocks)))
                return resp

            stub.VolumePutFiles2 = recording
            client = types.SimpleNamespace(stub=stub)
            f = DeviceFile(t)
            async with volume.VolumeUploadContextManager2("vo-g", client) as batch:
                batch.put_file(f, "/ckpt/shard0")
            dev_blocks = [d for d, _ in seen[0][0][0]]
            first_missing = seen[0][1]
            # what the host path produces on the same bytes
            host_spec = await blob_utils.FileUploadSpec2.from_fileobj(io.BytesIO(host_bytes), PurePosixPath("/ckpt/shard0"),
                                                                      asyncio.Semaphore(1), 0o644)
            assert dev_blocks == [b.contents_sha256 for b in host_spec.blocks]
            distinct = {}
            for mb in first_missing:
                b = host_spec.blocks[mb.block_index]
                distinct.setdefault(b.contents_sha256, b.end - b.start)
            assert f.bytes_to_host == sum(distinct.values())
            got = stub.volume_files["/ckpt/shard0"][0]
            assert len(got) == n and hashlib.sha256(got).digest() == hashlib.sha256(host_bytes).digest()
            before_puts, before_bytes = stub.block_puts, f.bytes_to_host
            seen.clear()
            async with volume.VolumeUploadContextManager2("vo-g", client, force=True) as batch:
                batch.put_file(f, "/ckpt/shard0")
            assert stub.block_puts == before_puts and f.bytes_to_host == before_bytes
            assert not seen[0][1]  # nothing reported missing the second time

    asyncio.run(run())
