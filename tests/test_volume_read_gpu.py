"""GPU: b200h_copy_ranges_from_host is byte-exact for every source residue and destination phase, over tiny and empty
segments and 10 000 ranges, writes nothing outside its destinations, launches one kernel per call, only enqueues and
rejects bad arguments before enqueueing; safetensors and torch.save files round-trip through the fake volume into
CUDA tensors."""
import asyncio
import io
import types

import numpy as np
import pytest

from modal_client_b200 import DeviceFile, _lib, blob_utils, load_ranges, volume
from tests.volume_read_server import running_volume_server

pytestmark = pytest.mark.gpu

MiB = 1 << 20
CANARY = 0x5C


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0, pinned_bytes=64 << 20, device_bytes=512 << 20)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pinned(ctx):
    buf = ctx.host_alloc(96 * MiB)
    yield buf
    ctx.host_free(buf)


def _load_and_check(ctx, pinned, segs, first, ranges, stream=0):
    """One call from random source bytes at 16-aligned offsets; every range's device bytes equal its source, every
    other byte of every segment keeps its canary."""
    import torch

    rng = np.random.default_rng(len(ranges))
    offsets, at = [], 16 * int(rng.integers(0, 8))
    for _, _, n in ranges:
        offsets.append(at)
        at += -(-n // 16) * 16 + 16 * int(rng.integers(0, 3))
    assert at <= pinned.size
    pinned[:at] = rng.integers(0, 256, at, dtype=np.uint8)
    for s in segs:
        s.fill_(CANARY)
    images = []
    for f in range(len(first) - 1):
        images.append(np.concatenate([np.full(s.numel(), CANARY, np.uint8) for s in segs[first[f] : first[f + 1]]]
                                     or [np.zeros(0, np.uint8)]))
    for (f, off, n), o in zip(ranges, offsets):
        images[f][off : off + n] = pinned[o : o + n]
    torch.cuda.synchronize()
    launches = ctx.launch_count
    ctx.copy_ranges_from_host([s.data_ptr() if s.numel() else 0 for s in segs], [s.numel() for s in segs], first,
                              ranges, pinned[:at], offsets, stream)
    assert ctx.launch_count - launches == (1 if any(n for _, _, n in ranges) else 0)
    torch.cuda.synchronize()
    for f in range(len(first) - 1):
        got = np.concatenate([s.cpu().numpy() for s in segs[first[f] : first[f + 1]]] or [np.zeros(0, np.uint8)])
        assert np.array_equal(got, images[f]), f


def _pool(n):
    import torch

    return torch.empty(n, dtype=torch.uint8, device="cuda")


@pytest.mark.parametrize("phase", range(16))
def test_every_source_residue_and_destination_phase(ctx, pinned, phase):
    """Segments starting ``phase`` bytes past a 256-byte boundary; ranges whose source and destination residues take
    every combination (a source offset is a multiple of 16, so the file offset sets the difference)."""
    lens = [1, 15, 16, 17, 63, 4095, 4097, 70_001, 3 * MiB + 5]
    pool = _pool(sum(-(-(n + 16) // 256) * 256 for n in lens) + 256)
    segs, at = [], 0
    for n in lens:
        segs.append(pool[at + phase : at + phase + n])
        at += -(-(n + 16) // 256) * 256
    _load_and_check(ctx, pinned, segs, list(range(len(segs) + 1)), [(f, 0, n) for f, n in enumerate(lens)])
    _load_and_check(ctx, pinned, segs, list(range(len(segs) + 1)), [(f, n // 3, n // 2) for f, n in enumerate(lens)])
    big = pool[phase : phase + 600_000]
    # file offset residue d (with the 16-aligned sources: every source / destination phase pair) x length residue e
    ranges = [(0, 2048 * (16 * d + e) + d, 1000 + e) for d in range(16) for e in range(16)]
    _load_and_check(ctx, pinned, [big], [0, 1], ranges)


def test_ranges_over_hundreds_of_tiny_segments_and_empty_ones(ctx, pinned):
    rng = np.random.default_rng(3)
    pool = _pool(MiB)
    segs, at = [], 0
    for i in range(900):
        n = 0 if i % 7 == 3 else int(rng.integers(1, 40)) if i % 50 else 70_000
        start = at + int(rng.integers(0, 16))
        segs.append(pool[start : start + n])
        at = start + n
    size = sum(s.numel() for s in segs)
    cuts = sorted(set(int(x) for x in rng.integers(0, size, 60)) | {0, size})
    ranges = [(0, a, b - a) for a, b in zip(cuts, cuts[1:])]  # disjoint ranges tiling the file
    _load_and_check(ctx, pinned, segs, [0, len(segs)], ranges)
    _load_and_check(ctx, pinned, segs, [0, len(segs)], [(0, 9, 0), (0, size, 0)])  # all empty: no launch


def test_ten_thousand_ranges_in_one_call(ctx, pinned):
    rng = np.random.default_rng(5)
    a, b = _pool(6 * MiB)[3:], _pool(MiB)[9:]
    segs = [a[: 2 * MiB], a[2 * MiB :], b]
    ranges = []
    for f, size in ((0, a.numel()), (1, b.numel())):
        cuts = np.unique(np.concatenate([[0, size], rng.integers(0, size, 6000)]))
        ranges += [(f, int(x), int(y - x)) for x, y in zip(cuts, cuts[1:])]
    order = rng.permutation(len(ranges))[:10_000]
    _load_and_check(ctx, pinned, segs, [0, 2, 3], [ranges[i] for i in order])


def test_the_call_is_stream_ordered(ctx, pinned):
    """Work queued before the call on the same stream overwrites the destination; the copy lands after it."""
    import torch

    stream = torch.cuda.Stream()
    dst = _pool(32 * MiB + 5)
    busy = torch.empty(64 * MiB, dtype=torch.float32, device="cuda")
    pinned[: 33 * MiB] = np.random.default_rng(9).integers(0, 256, 33 * MiB, dtype=np.uint8)
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        for _ in range(20):
            busy.normal_()
        dst.fill_(1)
        ctx.copy_ranges_from_host([dst.data_ptr()], [dst.numel()], [0, 1], [(0, 3, dst.numel() - 3)], pinned[: 33 * MiB],
                                  [256], stream.cuda_stream)
    stream.synchronize()
    got = dst.cpu().numpy()
    assert got[:3].tolist() == [1, 1, 1] and np.array_equal(got[3:], pinned[256 : 256 + dst.numel() - 3])


def test_bad_arguments_are_rejected_before_anything_is_enqueued(ctx, pinned):
    import torch

    seg = _pool(4096)
    seg.fill_(CANARY)
    host = torch.empty(4096, dtype=torch.uint8)
    pageable = np.zeros(8192, np.uint8)
    ok = dict(ptrs=[seg.data_ptr()], lens=[4096], first=[0, 1], ranges=[(0, 0, 100), (0, 200, 100)], src=pinned,
              offsets=[0, 128])
    cases = {
        "host segment": dict(ptrs=[host.data_ptr()]),
        "NULL segment": dict(ptrs=[0]),
        "segment whose address range wraps": dict(lens=[2**64 - seg.data_ptr() + 16]),
        "overlapping destinations": dict(ranges=[(0, 0, 100), (0, 99, 100)]),
        "the same tensor in two files": dict(ptrs=[seg.data_ptr()] * 2, lens=[4096] * 2, first=[0, 1, 2],
                                             ranges=[(0, 0, 100), (1, 50, 10)]),
        "misaligned source": dict(offsets=[0, 136]),
        "source out of bounds": dict(offsets=[0, pinned.size - 64]),
        "source not page-locked": dict(src=pageable[-pageable.ctypes.data % 16 :][:4096]),
        "range past the end of its file": dict(ranges=[(0, 0, 100), (0, 4000, 97)]),
        "range of a file that does not exist": dict(ranges=[(1, 0, 1), (0, 0, 1)]),
    }
    for name, change in cases.items():
        a = {**ok, **change}
        launches = ctx.launch_count
        with pytest.raises(_lib.B200HashError, match=r"\(-1\)"):
            ctx.copy_ranges_from_host(a["ptrs"], a["lens"], a["first"], a["ranges"], a["src"], a["offsets"])
        assert ctx.launch_count == launches, name
    torch.cuda.synchronize()
    assert (seg.cpu().numpy() == CANARY).all()


# ----------------------------------------------------------------------------------------- volume reads


def _state_dict(total, seed=0):
    """bf16 / f32 / u8 / bool tensors of mixed sizes adding up to about ``total`` bytes, a 0-d and a zero-size one."""
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    sd, left, i = {}, total, 0
    sizes = [total // 3, total // 5, 12 * MiB + 6, 9 * MiB, 3 * MiB + 2, 70_001, 4099, 513, 64, 7, 1]
    while left > 0:
        n = min(left, sizes[i % len(sizes)])
        raw = torch.randint(0, 256, (n + 4,), dtype=torch.uint8, device="cuda", generator=g)
        if i % 3 == 0:
            raw[n // 2 :] = 0
        sd[f"t{i}"] = raw[: n // 2 * 2].view(torch.bfloat16) if i % 4 == 0 else \
            raw[: n // 4 * 4].view(torch.float32) if i % 4 == 1 else raw[:n] if i % 4 == 2 else raw[:n] > 127
        left -= n
        i += 1
    sd["scalar"] = torch.tensor(2.5, device="cuda")
    sd["none"] = torch.zeros(0, 3, dtype=torch.float16, device="cuda")
    return sd


async def _upload(stub, f, path):
    batch = volume.VolumeUploadContextManager2("vo-g", types.SimpleNamespace(stub=stub))
    async with batch:
        batch.put_file(f, path)


def _equal(got, want):
    import torch

    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k].device.type == "cuda" and got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, k
        assert torch.equal(got[k].reshape(-1).view(torch.uint8), want[k].reshape(-1).view(torch.uint8)), k  # NaNs


def test_safetensors_round_trip_and_into(gpu_backend):
    import torch

    sd = _state_dict(40 * MiB, seed=1)
    BS = blob_utils.BLOCK_SIZE

    async def run():
        async with running_volume_server(BS) as (stub, _):
            client = types.SimpleNamespace(stub=stub)
            await _upload(stub, DeviceFile.safetensors(sd, metadata={"format": "pt"}), "/m.safetensors")
            _equal(await volume.read_safetensors(client, "vo-g", "/m.safetensors"), sd)
            model = torch.nn.Sequential(torch.nn.Linear(300, 200), torch.nn.LayerNorm(200), torch.nn.Linear(200, 7))
            model = model.to("cuda", torch.bfloat16)
            want = {k: torch.randn_like(v) for k, v in model.state_dict().items()}
            await _upload(stub, DeviceFile.safetensors(want), "/model.safetensors")
            params = dict(model.named_parameters())
            ptrs = {k: p.data_ptr() for k, p in params.items()}
            with torch.no_grad():
                got = await volume.read_safetensors(client, "vo-g", "/model.safetensors",
                                                    into={k: p.data for k, p in params.items()})
            assert {k: p.data_ptr() for k, p in params.items()} == ptrs
            _equal({k: p.data for k, p in params.items()}, want)
            assert all(got[k].data_ptr() == ptrs[k] for k in want)

    asyncio.run(run())


def test_a_1gib_state_dict_in_many_waves(gpu_backend):
    sd = _state_dict(1 << 30, seed=2)

    async def run():
        async with running_volume_server(blob_utils.BLOCK_SIZE) as (stub, _):
            client = types.SimpleNamespace(stub=stub)
            await _upload(stub, DeviceFile.safetensors(sd), "/big.safetensors")
            launches = gpu_backend.launch_count
            got = await volume.read_safetensors(client, "vo-g", "/big.safetensors", staging_bytes=64 * MiB)
            assert gpu_backend.launch_count - launches >= (1 << 30) // (32 * MiB)  # one load per wave of 4 blocks
            _equal(got, sd)

    asyncio.run(run())


def test_torch_save_file_into_a_uint8_tensor(gpu_backend):
    import torch

    obj = {"sd": _state_dict(20 * MiB, seed=3), "step": 7, "note": "x"}
    buf = io.BytesIO()
    torch.save(obj, buf)
    image = buf.getvalue()

    async def run():
        async with running_volume_server(blob_utils.BLOCK_SIZE) as (stub, _):
            client = types.SimpleNamespace(stub=stub)
            await _upload(stub, DeviceFile.torch_save(obj), "/ckpt.pt")
            dst = torch.full((len(image),), 0xEE, dtype=torch.uint8, device="cuda")
            n = await volume.read_file_into_device(client, "vo-g", "/ckpt.pt", DeviceFile(dst), staging_bytes=16 * MiB)
            assert n == len(image)
            host = dst.cpu()  # ordered after the copy on the current stream
            assert host.numpy().tobytes() == image
            back = torch.load(io.BytesIO(host.numpy().tobytes()), map_location="cuda")
            assert back["step"] == 7 and back["note"] == "x"
            _equal(back["sd"], obj["sd"])
            # a start that is not on a block edge
            tail = torch.empty(len(image) - 12_345, dtype=torch.uint8, device="cuda")
            await volume.read_file_into_device(client, "vo-g", "/ckpt.pt", DeviceFile(tail), start=12_345)
            assert tail.cpu().numpy().tobytes() == image[12_345:]

    asyncio.run(run())


def test_load_ranges_orders_after_earlier_reads(gpu_backend):
    """A kernel queued on the current stream reads the tensor before load_ranges; it sees the old bytes, and work
    queued after the call sees the new ones, without a host synchronisation in between."""
    import torch

    t = torch.full((512 * MiB,), 3, dtype=torch.uint8, device="cuda")  # ~10 ms over PCIe: a missing wait would show
    busy = torch.empty(64 * MiB, dtype=torch.float32, device="cuda")
    src = gpu_backend.host_alloc(512 * MiB)
    try:
        src[:] = 9
        f = DeviceFile(t)
        for _ in range(20):
            busy.normal_()
        before = t.sum(dtype=torch.int64)
        loaded = load_ranges([f], [(0, 0, t.numel())], src, [0])
        after = t.sum(dtype=torch.int64)
        loaded.wait()
        assert int(before) == 3 * t.numel() and int(after) == 9 * t.numel()
    finally:
        torch.cuda.synchronize()
        gpu_backend.host_free(src)
