"""GPU: b200h_crc32_device against zlib.crc32 over every small length and alignment, chunk edges, many ranges and one
range past 4 GiB, with its launch count and pointer checks; DeviceFile.torch_save of CUDA checkpoints byte for byte
against torch.save (ZIP64 included), ordered after the current stream, with no bytes to the host, bounded extra HBM,
two synchronisations, and a ~1 GiB upload through volumefs2."""
import asyncio
import io
import random
import types
import warnings
import zlib
from pathlib import PurePosixPath

import numpy as np
import pytest

from modal_client_b200 import DeviceFile, _lib, blob_utils, device_file, volume
from tests.test_device_file_cpu import _volume_server

pytestmark = pytest.mark.gpu

MiB = 1 << 20
LEGACY = 1  # cudaStreamLegacy: PyTorch's default stream (a NULL stream is the library context's own stream)
CHUNK = 16 << 10  # kCrcChunkBytes
PIECE = CHUNK // 32


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0, pinned_bytes=64 << 20, device_bytes=256 << 20)
    yield c
    c.close()


def _device_crcs(ctx, big, ranges):
    import torch

    out = torch.full((max(len(ranges), 1),), -1, dtype=torch.int32, device="cuda:0")
    ctx.crc32_device([big.data_ptr() + s if n else 0 for s, n in ranges], [n for _, n in ranges], out.data_ptr(),
                     torch.cuda.current_stream().cuda_stream or LEGACY)
    return out.cpu().numpy().view(np.uint32)[: len(ranges)].tolist()


def _random_buffer(ctx, nbytes: int, seed: int):
    import torch

    big = torch.empty(nbytes + 64, dtype=torch.uint8, device="cuda:0")
    ctx.fill_synth_device(big.data_ptr(), big.numel() // 8 * 8, seed, stream=LEGACY)
    return big, big.cpu().numpy().tobytes()


def test_crc32_every_short_length_at_every_misalignment(ctx):
    ranges, at = [], 0
    for n in range(301):
        for mis in range(16):
            at = (at + 15) // 16 * 16 + mis
            ranges.append((at, n))
            at += n
    big, host = _random_buffer(ctx, at, 1)
    got = _device_crcs(ctx, big, ranges)
    assert got == [zlib.crc32(host[s : s + n]) for s, n in ranges]


def test_crc32_at_chunk_and_piece_edges(ctx):
    lens = sorted({k * u + d for u in (PIECE, CHUNK) for k in (1, 2, 3, 31, 32, 33, 64) for d in (-1, 0, 1)})
    ranges, at = [], 0
    for i, n in enumerate(lens):
        at = (at + 15) // 16 * 16 + i % 16
        ranges.append((at, n))
        at += n
    big, host = _random_buffer(ctx, at, 2)
    assert _device_crcs(ctx, big, ranges) == [zlib.crc32(host[s : s + n]) for s, n in ranges]
    for s, n in ranges[::7]:  # one range per call as well
        assert _device_crcs(ctx, big, [(s, n)]) == [zlib.crc32(host[s : s + n])]


def test_crc32_ten_thousand_mixed_ranges_in_one_call(ctx):
    rng = random.Random(3)
    ranges, at = [], 0
    for _ in range(10_000):
        n = rng.choice([0, 0, 1, 7, 40, rng.randrange(1, 600), rng.randrange(1, 70_000), CHUNK, CHUNK + 1])
        at += rng.randrange(0, 40)
        ranges.append((at, n))
        at += n
    ranges[5000] = (7, 3 * MiB + 5)  # one large range overlapping others
    big, host = _random_buffer(ctx, at + 4 * MiB, 4)
    launches = ctx.launch_count
    got = _device_crcs(ctx, big, ranges)
    assert ctx.launch_count == launches + 1
    assert got == [zlib.crc32(host[s : s + n]) for s, n in ranges]


def test_crc32_of_one_range_past_4gib(ctx):
    import torch

    n = (4 << 30) + 12_345
    big = torch.empty(n + 3, dtype=torch.uint8, device="cuda:0")
    ctx.fill_synth_device(big.data_ptr(), (n + 3) // 8 * 8, 9, stream=LEGACY)
    got = _device_crcs(ctx, big, [(3, n), (0, 5)])
    want, step = 0, 256 * MiB
    for a in range(3, n + 3, step):
        want = zlib.crc32(big[a : min(a + step, n + 3)].cpu().numpy().tobytes(), want)
    assert got == [want, zlib.crc32(big[:5].cpu().numpy().tobytes())]
    del big
    torch.cuda.empty_cache()


def test_crc32_empty_ranges_and_launch_counts(ctx):
    big, host = _random_buffer(ctx, 1 << 16, 5)
    launches = ctx.launch_count
    assert _device_crcs(ctx, big, [(0, 0), (5, 0), (9, 0)]) == [0, 0, 0]
    assert ctx.launch_count == launches  # nothing to checksum: no launch
    for k in (1, 300):
        ranges = [(i * 37 % 60_000, (i * 101) % 4000 + 1) for i in range(k)]
        launches = ctx.launch_count
        assert _device_crcs(ctx, big, ranges) == [zlib.crc32(host[s : s + n]) for s, n in ranges]
        assert ctx.launch_count == launches + 1


def test_crc32_rejects_foreign_pointers_before_launching(ctx):
    import torch

    host = np.zeros(4096, np.uint8)
    dev = torch.zeros(4096, dtype=torch.uint8, device="cuda:0")
    out = torch.full((2,), 7, dtype=torch.int32, device="cuda:0")
    launches = ctx.launch_count
    for ptrs, lens, o in (([dev.data_ptr(), host.ctypes.data], [4096, 16], out.data_ptr()),  # host memory
                          ([dev.data_ptr(), 0], [10, 5], out.data_ptr()),                    # NULL with bytes
                          ([dev.data_ptr(), dev.data_ptr()], [10, 5], host.ctypes.data),     # host output
                          ([dev.data_ptr(), dev.data_ptr()], [10, 5], out.data_ptr() + 2)):  # misaligned output
        with pytest.raises(_lib.B200HashError, match=r"\(-1\)"):
            ctx.crc32_device(ptrs, lens, o)
    torch.cuda.synchronize()
    assert ctx.launch_count == launches and out.tolist() == [7, 7]


# -------------------------------------------------------------------------------------------- torch_save


def _saved(obj) -> bytes:
    import torch

    b = io.BytesIO()
    torch.save(obj, b)
    return b.getvalue()


def _bf16_state_dict(ctx, layers: int, hidden: int, seed: int) -> dict:
    import torch

    sd = {"embed.weight": torch.empty(4 * hidden, hidden, dtype=torch.bfloat16, device="cuda:0")}
    for i in range(layers):
        for name, shape in (("attn.qkv.weight", (3 * hidden, hidden)), ("attn.o.weight", (hidden, hidden)),
                            ("mlp.up.weight", (4 * hidden, hidden)), ("mlp.down.weight", (hidden, 4 * hidden)),
                            ("norm.weight", (hidden,))):
            sd[f"layers.{i}.{name}"] = torch.empty(shape, dtype=torch.bfloat16, device="cuda:0")
    for k, t in enumerate(sd.values()):
        ctx.fill_synth_device(t.data_ptr(), t.numel() * 2 // 8 * 8, seed + k, stream=LEGACY)
    return sd


def _training_checkpoint():
    import torch

    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(64, 256), torch.nn.GELU(), torch.nn.Linear(256, 10)).cuda()
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    for _ in range(3):
        model(torch.randn(8, 64, device="cuda")).square().mean().backward()
        opt.step()
    ckpt = {"model": model.state_dict(), "optim": opt.state_dict(), "step": 3}
    assert all(s["step"].device.type == "cpu" for s in ckpt["optim"]["state"].values())  # CPU step tensors
    return ckpt


def test_torch_save_images_equal_torch_save(gpu_backend):
    import torch

    base = torch.arange(4096, dtype=torch.float32, device="cuda:0")
    m = torch.randn(33, 65, device="cuda:0")
    cases = {
        "bf16_model": _bf16_state_dict(gpu_backend, 4, 256, 10),
        "training": _training_checkpoint(),
        "shared_and_offset": {"a": base[:1000], "b": base[1000:], "c": base[17:40], "t": m.t(), "cols": m[:, 3::5],
                              "empty": torch.zeros(0, device="cuda:0"), "zero_d": torch.tensor(2.0, device="cuda:0"),
                              "cpu": torch.arange(10)},
    }
    for name, obj in cases.items():
        torch.cuda.synchronize()
        want = _saved(obj)
        f = DeviceFile.torch_save(obj, bounce_bytes=random.Random(name).choice([4096, MiB]))
        assert f.nbytes == len(want), name
        assert f.read() == want, name
        back = torch.load(io.BytesIO(want), weights_only=True)
        assert back.keys() == obj.keys()


def test_torch_save_of_an_image_past_4gib_uses_zip64(gpu_backend):
    import torch

    big = torch.empty((4 << 30) + 4099, dtype=torch.uint8, device="cuda:0")
    gpu_backend.fill_synth_device(big.data_ptr(), big.numel() // 8 * 8, 21, stream=LEGACY)
    obj = {"big": big, "small": torch.ones(5, device="cuda:0"), "step": torch.tensor(7)}
    torch.cuda.synchronize()
    want = _saved(obj)
    assert len(want) > 4 << 30
    f = DeviceFile.torch_save(obj)
    assert f.nbytes == len(want)
    step = 512 * MiB
    for a in range(0, len(want), step):
        assert f.read(step) == want[a : a + step], a
    del want, f, big
    torch.cuda.empty_cache()


def test_torch_save_hashes_what_the_current_stream_wrote(gpu_backend):
    import torch

    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        t = torch.empty(64 * MiB, dtype=torch.uint8, device="cuda:0")
        u = torch.empty(3 * MiB + 5, dtype=torch.int8, device="cuda:0")
        torch.cuda._sleep(50_000_000)  # the writes land well after construction returns
        t.fill_(0x5A)
        u.copy_(torch.arange(u.numel(), device="cuda:0").to(torch.int8))
        f = DeviceFile.torch_save({"t": t, "u": u})
    torch.cuda.synchronize()
    assert f.read() == _saved({"t": t, "u": u})


def test_torch_save_syncs_twice_stays_in_hbm_and_copies_nothing_back(gpu_backend):
    import torch

    ckpt = _training_checkpoint()
    ckpt["model_bf16"] = _bf16_state_dict(gpu_backend, 2, 512, 40)
    torch.cuda.synchronize()
    skeleton = device_file.torch_save_layout(ckpt)[0]
    skel_bytes = sum(len(p) for _, p in skeleton.pieces)
    staged = sum(s["step"].untyped_storage().nbytes() for s in ckpt["optim"]["state"].values())
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            f = DeviceFile.torch_save(ckpt)
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    syncs = [w for w in caught if "synchroniz" in str(w.message)]
    assert len(syncs) == 2, [str(w.message) for w in caught]
    extra = torch.cuda.max_memory_allocated() - before
    assert extra <= skel_bytes + staged + 64 * 1024, (extra, skel_bytes, staged)
    sha, _, trimmed = f.hash_parts(blob_utils.BLOCK_SIZE, _lib.SHA256 | _lib.TRIM_ZEROS)
    assert f.bytes_to_host == 0 and len(trimmed) == -(-f.nbytes // blob_utils.BLOCK_SIZE)


def test_v2_put_of_a_1gib_checkpoint(gpu_backend):
    import torch

    MiB8 = blob_utils.BLOCK_SIZE
    ckpt = _training_checkpoint()
    sd = {}
    rng = random.Random(17)
    sizes = [rng.choice([4 << 10, 64 << 10, MiB, 3 * MiB + 2]) for _ in range(120)]
    sizes += [64 * MiB] * (((1 << 30) - sum(sizes)) // (64 * MiB))
    for i, n in enumerate(sizes):
        t = torch.empty(n // 2, dtype=torch.bfloat16, device="cuda:0")
        gpu_backend.fill_synth_device(t.data_ptr(), n // 8 * 8, seed=300 + i, stream=LEGACY)
        if i % 3 == 0:
            t.view(torch.uint8)[n - rng.randrange(1, n) :] = 0  # a zero tail
        sd[f"model.layers.{i}.weight"] = t
    ckpt["model_big"] = sd
    torch.cuda.synchronize()
    image = _saved(ckpt)
    assert 900 * MiB < len(image) < 1100 * MiB
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
            f = DeviceFile.torch_save(ckpt)
            async with volume.VolumeUploadContextManager2("vo-g", client) as batch:
                batch.put_file(f, "/ckpt/step3.pt")
            assert stub.volume_files["/ckpt/step3.pt"][0] == image
            host_spec = await blob_utils.FileUploadSpec2.from_fileobj(io.BytesIO(image), PurePosixPath("/x"),
                                                                      asyncio.Semaphore(1), 0o644)
            dev_spec = await blob_utils.FileUploadSpec2.from_fileobj(DeviceFile.torch_save(ckpt), PurePosixPath("/x"),
                                                                     asyncio.Semaphore(1), 0o644)
            assert dev_spec.blocks == host_spec.blocks
            distinct = {}
            for mb in seen[0]:
                b = host_spec.blocks[mb.block_index]
                distinct.setdefault(b.contents_sha256, b.end - b.start)
            assert f.bytes_to_host == sum(distinct.values())

    asyncio.run(run())
