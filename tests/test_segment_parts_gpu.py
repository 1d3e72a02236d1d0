"""GPU: b200h_hash_segment_parts_device is bit-exact against the oracle over the concatenated bytes and against
b200h_hash_fixed_parts_device over a torch.cat copy, for every alignment and in several waves; it synchronises only
where the header says and rejects foreign pointers on the host; DeviceFile.safetensors reads back the library's image
and uploads a ~1 GiB state dict through volumefs2; a batch of device files costs one library call."""
import asyncio
import io
import random
import types
from pathlib import PurePosixPath

import numpy as np
import pytest

from modal_client_b200 import DeviceFile, _lib, blob_utils, volume
from oracle import c_oracle
from tests.test_device_file_cpu import _volume_server

pytestmark = pytest.mark.gpu

MiB = 1 << 20
SEG_LENS = [0, 1, 15, 16, 17, 63, 64, 65, 4095, 4096, 4097, MiB - 1, MiB + 1, 9 * MiB]
FLAGS = [_lib.SHA256, _lib.MD5, _lib.SHA256 | _lib.MD5, _lib.SHA256 | _lib.TRIM_ZEROS]


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0, pinned_bytes=64 << 20, device_bytes=512 << 20)
    yield c
    c.close()


def _layout(rng: random.Random, nfiles: int):
    """Segment lengths per file (every length class, empty files, several segments per file), shuffled."""
    files = []
    for _ in range(nfiles):
        files.append([rng.choice(SEG_LENS) for _ in range(rng.randrange(0, 7))])
    files[rng.randrange(nfiles)] = list(SEG_LENS)  # all of them in one file
    return files


def _place(ctx, files, seed: int, misalign):
    """One large device tensor holding every segment at a chosen start mod 16, with zero runs straddling segment
    edges and some all-zero segments.  -> (big tensor, segment addresses, segment lengths, file_first_seg, host bytes
    of every file)."""
    import torch

    rng = random.Random(seed)
    lens = [n for f in files for n in f]
    starts, at = [], 0
    for n in lens:
        at = (at + 15) // 16 * 16 + misalign(rng)
        starts.append(at)
        at += n
    big = torch.empty(at + 64, dtype=torch.uint8, device="cuda:0")
    ctx.fill_synth_device(big.data_ptr(), big.numel() // 8 * 8, seed)
    host = big.cpu().numpy().copy()
    for k, (s, n) in enumerate(zip(starts, lens)):
        r = rng.random()
        if r < 0.2:
            host[s : s + n] = 0  # an all-zero segment
        elif r < 0.5 and n:
            host[s + rng.randrange(n) : s + n] = 0  # a zero tail running into the next segment's zero head
            if k + 1 < len(lens):
                nxt = starts[k + 1]
                host[nxt : nxt + rng.randrange(lens[k + 1] + 1)] = 0
    big.copy_(torch.from_numpy(host))
    ptrs = [big.data_ptr() + s for s in starts]
    first = np.concatenate([[0], np.cumsum([len(f) for f in files])]).astype(np.uint64)
    images, k = [], 0
    for f in files:
        images.append(b"".join(host[starts[k + j] : starts[k + j] + n].tobytes() for j, n in enumerate(f)))
        k += len(f)
    return big, ptrs, lens, first, images


def _segment_rows(ctx, ptrs, lens, first, part_len, flags, nrows):
    import torch

    dev = torch.device("cuda", 0)
    sha = torch.empty((nrows, 32), dtype=torch.uint8, device=dev)
    md5 = torch.empty((nrows, 16), dtype=torch.uint8, device=dev)
    trim = torch.empty(nrows, dtype=torch.int64, device=dev)
    got = ctx.hash_segment_parts_device(ptrs, lens, first, part_len, flags, sha.data_ptr() if nrows else 0,
                                        md5.data_ptr() if nrows else 0, trim.data_ptr() if nrows else 0)
    assert got == nrows
    torch.cuda.synchronize()
    return (sha.cpu().numpy() if flags & _lib.SHA256 else None, md5.cpu().numpy() if flags & _lib.MD5 else None,
            trim.cpu().numpy().astype(np.uint64))


def _oracle_rows(images, part_len, flags):
    data = np.frombuffer(b"".join(images) or b"\0", np.uint8)
    starts, lens, at = [], [], 0
    for img in images:
        for o in range(0, len(img), part_len):
            starts.append(at + o)
            lens.append(min(part_len, len(img) - o))
        at += len(img)
    return c_oracle.hash_batch(data, np.array(starts, np.uint64), np.array(lens, np.uint64),
                               sha=bool(flags & _lib.SHA256), md5=bool(flags & _lib.MD5),
                               trim=bool(flags & _lib.TRIM_ZEROS))


def _check(got, want, flags):
    if flags & _lib.SHA256:
        assert np.array_equal(got[0], want[0])
    if flags & _lib.MD5:
        assert np.array_equal(got[1], want[1])
    assert np.array_equal(got[2], want[2])


@pytest.mark.parametrize("part_len", [64, 1000, 4096, 8 * MiB])
@pytest.mark.parametrize("flags", FLAGS)
def test_segment_parts_match_oracle_and_fixed_parts_of_a_copy(ctx, part_len, flags):
    import torch

    for seed, misalign in ((1, lambda r: 0), (2, lambda r: r.randrange(16)), (3, lambda r: 1)):
        files = _layout(random.Random(seed), 4)
        big, ptrs, lens, first, images = _place(ctx, files, seed, misalign)
        nrows = sum(-(-len(i) // part_len) for i in images)
        got = _segment_rows(ctx, ptrs, lens, first, part_len, flags, nrows)
        _check(got, _oracle_rows(images, part_len, flags), flags)
        # the same rows from b200h_hash_fixed_parts_device over one contiguous copy of every file
        row = 0
        for f, img in enumerate(images):
            if not img:
                continue
            copy = torch.frombuffer(bytearray(img), dtype=torch.uint8).cuda()
            n = -(-len(img) // part_len)
            sha = torch.empty((n, 32), dtype=torch.uint8, device="cuda:0")
            md5 = torch.empty((n, 16), dtype=torch.uint8, device="cuda:0")
            trim = torch.empty(n, dtype=torch.int64, device="cuda:0")
            ctx.hash_fixed_parts_device(copy.data_ptr(), len(img), part_len, flags, sha.data_ptr(), md5.data_ptr(),
                                        trim.data_ptr())
            torch.cuda.synchronize()
            if flags & _lib.SHA256:
                assert np.array_equal(sha.cpu().numpy(), got[0][row : row + n])
            if flags & _lib.MD5:
                assert np.array_equal(md5.cpu().numpy(), got[1][row : row + n])
            assert np.array_equal(trim.cpu().numpy().astype(np.uint64), got[2][row : row + n])
            row += n
        del big


def test_segment_parts_in_several_waves():
    """A context whose wave slots hold 1 MiB: the gathered parts need at least three waves and the rows still match."""
    c = _lib.Context(0, pinned_bytes=16 << 20, device_bytes=2 * MiB)
    try:
        rng = random.Random(5)
        files = [[rng.choice([4095, 4097, 65, 100_000, 300_001]) for _ in range(60)] for _ in range(3)]
        big, ptrs, lens, first, images = _place(c, files, 5, lambda r: r.randrange(16))
        part_len = 256 << 10
        seg, wave, nwaves = _lib.segment_parts_preview(lens, first, part_len, MiB)
        assert nwaves >= 3 and (seg == _lib.GATHERED).sum() >= 8
        for flags in (_lib.SHA256 | _lib.MD5, _lib.SHA256 | _lib.TRIM_ZEROS):
            got = _segment_rows(c, ptrs, lens, first, part_len, flags, seg.size)
            _check(got, _oracle_rows(images, part_len, flags), flags)
    finally:
        c.close()


def test_segment_parts_synchronise_only_where_the_header_says(ctx):
    files = [[4097, 9 * MiB, 17], [MiB + 1, 0, 63]]
    big, ptrs, lens, first, images = _place(ctx, files, 9, lambda r: 3)
    part_len = 2 * MiB
    _, _, nwaves = _lib.segment_parts_preview(lens, first, part_len, 256 * MiB)
    nrows = sum(-(-len(i) // part_len) for i in images)
    for flags, extra in ((_lib.SHA256 | _lib.MD5, 0), (_lib.SHA256 | _lib.TRIM_ZEROS | _lib.NO_OUTLIERS, 0),
                         (_lib.SHA256 | _lib.TRIM_ZEROS, nwaves)):
        before = ctx.plan_sync_count
        got = _segment_rows(ctx, ptrs, lens, first, part_len, flags, nrows)
        assert ctx.plan_sync_count == before + extra
        _check(got, _oracle_rows(images, part_len, flags), flags)


def test_segment_parts_reject_foreign_pointers_before_launching(ctx):
    import torch

    host = np.zeros(4096, np.uint8)
    dev = torch.zeros(4096, dtype=torch.uint8, device="cuda:0")
    cases = [([dev.data_ptr(), host.ctypes.data], [4096, 4096]),  # host memory
             ([host.ctypes.data, dev.data_ptr()], [16, 4096]),
             ([dev.data_ptr(), 0], [10, 5]),                       # NULL with bytes behind it
             ([dev.data_ptr()], [2**64 - dev.data_ptr() + 16])]    # an address range that wraps
    if torch.cuda.device_count() > 1:  # another device's memory
        other = torch.zeros(64, dtype=torch.uint8, device="cuda:1")
        cases.append(([dev.data_ptr(), other.data_ptr()], [64, 64]))
    launches = ctx.launch_count
    for ptrs, lens in cases:
        with pytest.raises(_lib.B200HashError, match=r"\(-1\)"):
            ctx.hash_segment_parts_device(ptrs, lens, [0, len(ptrs)], 64, _lib.SHA256, 0, 0, 0)
    assert ctx.launch_count == launches
    with pytest.raises(_lib.B200HashError, match=r"\(-1\)"):
        ctx.hash_segment_parts_device([dev.data_ptr()], [10], [0, 2], 64, _lib.SHA256)  # file_first_seg past nsegs


@pytest.mark.parametrize("seed", [0, 1])
def test_safetensors_reads_back_the_library_image(gpu_backend, seed):
    import torch
    from safetensors.torch import save

    rng = random.Random(seed)
    dtypes = [torch.bfloat16, torch.float16, torch.float32, torch.int64, torch.uint8, torch.bool, torch.float8_e4m3fn]
    sd = {}
    for i in range(40):
        dt = rng.choice(dtypes)
        shape = rng.choice([(), (0,), (1,), (17,), (33, 65), (rng.randrange(1, 5000),)])
        raw = torch.randint(0, 256, (int(np.prod(shape)) * torch.empty(0, dtype=dt).element_size(),),
                            dtype=torch.uint8, device="cuda:0")
        sd[f"layers.{i}.{rng.choice(['w', 'b', 'norm'])}"] = raw.view(dt).reshape(shape)
    want = save({k: v.cpu() for k, v in sd.items()}, {"format": "pt"})
    f = DeviceFile.safetensors(sd, {"format": "pt"}, bounce_bytes=rng.choice([4096, 1 << 20]))
    assert f.read() == want and f.nbytes == len(want)
    sha, _, trimmed = f.hash_parts(MiB // 4, _lib.SHA256)
    assert np.array_equal(sha, _oracle_rows([want], MiB // 4, _lib.SHA256)[0])


def test_v2_put_of_a_1gib_state_dict(gpu_backend):
    import torch
    from safetensors.torch import save

    MiB8 = blob_utils.BLOCK_SIZE
    rng = random.Random(17)
    sizes = [rng.choice([4 << 10, 64 << 10, MiB, 3 * MiB + 2]) for _ in range(180)]
    sizes += [64 * MiB] * (((1 << 30) - sum(sizes)) // (64 * MiB))  # big matrices fill up to ~1 GiB
    sd = {}
    for i, n in enumerate(sizes):
        t = torch.empty(n // 2, dtype=torch.bfloat16, device="cuda:0")
        gpu_backend.fill_synth_device(t.data_ptr(), n // 8 * 8, seed=100 + i)
        if i % 3 == 0:
            t.view(torch.uint8)[n - rng.randrange(1, n) :] = 0  # a zero tail
        sd[f"model.layers.{i}.weight"] = t
    torch.cuda.synchronize()
    image = save({k: v.cpu() for k, v in sd.items()})
    assert 900 * MiB < len(image) < 1100 * MiB and 190 <= len(sd) <= 210
    seen = []

    async def run():
        async with _volume_server(MiB8) as (stub, _):
            record = stub.VolumePutFiles2

            async def recording(req):
                resp = await record(req)
                seen.append(list(resp.missing_blocks))
                return resp

            stub.VolumePutFiles2 = recording
            client = types.SimpleNamespace(stub=stub)
            f = DeviceFile.safetensors(sd)
            async with volume.VolumeUploadContextManager2("vo-g", client) as batch:
                batch.put_file(f, "/ckpt/model.safetensors")
            assert stub.volume_files["/ckpt/model.safetensors"][0] == image
            host_spec = await blob_utils.FileUploadSpec2.from_fileobj(io.BytesIO(image), PurePosixPath("/x"),
                                                                      asyncio.Semaphore(1), 0o644)
            distinct = {}
            for mb in seen[0]:
                b = host_spec.blocks[mb.block_index]
                distinct.setdefault(b.contents_sha256, b.end - b.start)
            assert f.bytes_to_host == sum(distinct.values())

    asyncio.run(run())


def test_batch_of_50_device_files_is_one_library_call(gpu_backend, monkeypatch):
    import torch

    calls = []
    for name in ("hash_segment_parts_device", "hash_fixed_parts_device"):
        real = getattr(_lib.Context, name)

        def counted(self, *a, _real=real, _name=name, **k):
            calls.append(_name)
            return _real(self, *a, **k)

        monkeypatch.setattr(_lib.Context, name, counted)
    rng = random.Random(23)
    tensors = []
    for i in range(50):
        n = rng.choice([0, 1, 4097, MiB, 9 * MiB, 17 * MiB + 5])
        t = torch.zeros(n, dtype=torch.uint8, device="cuda:0")
        if n >= 8:
            gpu_backend.fill_synth_device(t.data_ptr(), n // 8 * 8, seed=i)
        tensors.append(t)
    items = [(DeviceFile(t), PurePosixPath(f"/t/{i}"), 0o644) for i, t in enumerate(tensors)]
    specs = asyncio.run(blob_utils.device_file_specs2(items))
    assert calls == ["hash_segment_parts_device"]
    calls.clear()
    one_by_one = [asyncio.run(blob_utils.FileUploadSpec2.from_fileobj(f, p, asyncio.Semaphore(1), m)) for f, p, m in items]
    assert len(calls) == sum(1 for t in tensors if t.numel())
    for a, b in zip(specs, one_by_one):
        assert (a.blocks, a.size, a.mode, a.path) == (b.blocks, b.size, b.mode, b.path)
