"""GPU: ``volume.read_torch_save`` loads torch.save checkpoints from the fake volume into CUDA storages equal to
``torch.load(..., map_location="cuda")``, in many waves, beyond 4 GiB (ZIP64), with the CRC-32s checked on the device
and the result ordered on the caller's current stream."""
import asyncio
import io
import types

import pytest

from modal_client_b200 import DeviceFile, blob_utils, volume
from modal_client_b200.exception import ExecutionError
from tests.test_volume_read_gpu import _state_dict, _upload
from tests.volume_read_server import running_volume_server

pytestmark = pytest.mark.gpu

MiB, GiB = 1 << 20, 1 << 30


def _contiguous_state_dict(total: int, seed: int) -> dict:
    """``_state_dict`` with every tensor over a storage of its own size: a typed view of a storage that is not a whole
    number of its elements is refused by ``torch.load``."""
    return {k: v.clone() for k, v in _state_dict(total, seed=seed).items()}


def _saved(obj) -> bytes:
    import torch

    buf = io.BytesIO()
    torch.save(obj, buf)
    return buf.getvalue()


def _training_checkpoint(total: int, seed: int) -> dict:
    import torch

    sd = _contiguous_state_dict(total, seed)
    model = torch.nn.Sequential(torch.nn.Linear(64, 128), torch.nn.LayerNorm(128), torch.nn.Linear(128, 10)).cuda()
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    model(torch.randn(8, 64, device="cuda")).sum().backward()
    opt.step()
    sd.update({f"net.{k}": v for k, v in model.state_dict().items()})
    sd["net.0.weight.T"] = sd["net.0.weight"].t()  # a view sharing a storage
    return {"model": sd, "optim": opt.state_dict(), "step": 7, "note": "x"}


def _tensors(obj, at=""):
    import torch

    if isinstance(obj, torch.Tensor):
        yield at, obj
    elif isinstance(obj, dict):
        for k, v in obj.items():
            yield from _tensors(v, f"{at}/{k}")
    elif isinstance(obj, (list, tuple)):
        for i, v in enumerate(obj):
            yield from _tensors(v, f"{at}/{i}")


def _same(got, want, device):
    """Bitwise equal, same structure, every tensor on ``device``, storages shared exactly where ``want``'s are."""
    import torch

    g, w = list(_tensors(got)), list(_tensors(want))
    assert [k for k, _ in g] == [k for k, _ in w]
    for (k, a), (_, b) in zip(g, w):
        assert a.device == device == b.device, k
        assert (a.dtype, a.shape, a.stride(), a.storage_offset()) == (b.dtype, b.shape, b.stride(), b.storage_offset()), k
        assert torch.equal(a.reshape(-1).view(torch.uint8), b.reshape(-1).view(torch.uint8)), k
    groups = lambda ts: sorted(sorted(k for k, t in ts if t.untyped_storage().data_ptr() == p)  # noqa: E731
                               for p in {t.untyped_storage().data_ptr() for _, t in ts if t.untyped_storage().nbytes()})
    assert groups(g) == groups(w)


def _strip(obj):
    """``obj`` without its tensors (for comparing the rest)."""
    import torch

    if isinstance(obj, torch.Tensor):
        return None
    if isinstance(obj, dict):
        return {k: _strip(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(_strip(v) for v in obj)
    return obj


def test_a_training_checkpoint_equals_torch_load(gpu_backend):
    import torch

    ckpt = _training_checkpoint(40 * MiB, seed=4)
    image = _saved(ckpt)
    assert any(t.device.type == "cpu" for _, t in _tensors(ckpt["optim"]))  # Adam's step
    device = torch.device(f"cuda:{gpu_backend.device}")

    async def run():
        async with running_volume_server(blob_utils.BLOCK_SIZE) as (stub, _):
            client = types.SimpleNamespace(stub=stub)
            await _upload(stub, DeviceFile.torch_save(ckpt), "/dev.pt")
            await _upload(stub, io.BytesIO(image), "/host.pt")
            assert stub.volume_files["/dev.pt"][0] == image
            want = torch.load(io.BytesIO(image), map_location="cuda")
            for path in ("/dev.pt", "/host.pt"):
                got = await volume.read_torch_save(client, "vo-g", path, staging_bytes=16 * MiB)
                _same(got, want, device)
                assert _strip(got) == _strip(want) and got["step"] == 7 and got["note"] == "x"

    asyncio.run(run())


def test_a_1gib_checkpoint_in_many_waves_takes_only_its_storages(gpu_backend):
    import torch

    sd = _contiguous_state_dict(GiB, 5)

    async def run():
        async with running_volume_server(blob_utils.BLOCK_SIZE) as (stub, _):
            client = types.SimpleNamespace(stub=stub)
            await _upload(stub, DeviceFile.torch_save(sd), "/big.pt")
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            launches = gpu_backend.launch_count
            got = await volume.read_torch_save(client, "vo-g", "/big.pt", staging_bytes=64 * MiB)
            torch.cuda.synchronize()
            growth = torch.cuda.max_memory_allocated() - base
            span = stub.get_file_calls[-1]  # the data region's call
            BS = blob_utils.BLOCK_SIZE
            waves = -(-((span.start + span.len - 1) // BS - span.start // BS + 1) // 4)  # 4 block slots per half
            assert waves >= (GiB - 32 * MiB) // (32 * MiB)
            assert gpu_backend.launch_count - launches == waves + 1  # one load per wave, then the CRC launch
            storages = {t.untyped_storage().data_ptr(): t.untyped_storage().nbytes() for t in got.values()}
            held = torch.cuda.memory_allocated() - base  # the storages, as the caching allocator rounds their blocks
            assert held <= sum(storages.values()) + 2 * MiB * len(storages), (held, sum(storages.values()))
            assert growth <= held + MiB, (growth, held)  # nothing transient beyond the CRC output
            _same(got, sd, torch.device(f"cuda:{gpu_backend.device}"))

    asyncio.run(run())


def test_a_zip64_checkpoint_over_4gib(gpu_backend):
    import torch

    big = torch.zeros((4 << 30) + 3 * MiB + 5, dtype=torch.uint8, device="cuda")  # trimmed blocks: cheap to store
    big[: 2 * MiB] = torch.randint(0, 256, (2 * MiB,), dtype=torch.uint8, device="cuda")
    big[-MiB:] = 7
    obj = {"big": big, "after": torch.arange(1000, dtype=torch.float32, device="cuda"),
           "cpu_after": torch.tensor([1.5, 2.5])}

    async def run():
        async with running_volume_server(blob_utils.BLOCK_SIZE) as (stub, _):
            client = types.SimpleNamespace(stub=stub)
            await _upload(stub, DeviceFile.torch_save(obj), "/z64.pt")
            got = await volume.read_torch_save(client, "vo-g", "/z64.pt", staging_bytes=64 * MiB)
            assert torch.equal(got["big"], big) and torch.equal(got["after"], obj["after"])
            assert got["cpu_after"].device.type == "cuda" and torch.equal(got["cpu_after"].cpu(), obj["cpu_after"])
            assert len(stub.volume_files["/z64.pt"][0]) > 1 << 32  # the last local headers lie beyond 4 GiB

    asyncio.run(run())


def test_a_flipped_byte_is_found_unless_crcs_are_off(gpu_backend, monkeypatch):
    import torch
    from torch.utils.serialization import config

    sd = {"a": torch.arange(3 * MiB, dtype=torch.float32, device="cuda"), "b": torch.ones(1000, device="cuda")}
    images = {"/crc.pt": bytearray(_saved(sd))}
    with monkeypatch.context() as m:
        m.setattr(config.save, "compute_crc32", False)
        images["/nocrc.pt"] = bytearray(_saved(sd))
    for image in images.values():
        at = image.find(b"archive/data/0") + 100_000  # inside storage 0's bytes
        image[at] ^= 1

    async def run():
        async with running_volume_server(blob_utils.BLOCK_SIZE) as (stub, _):
            client = types.SimpleNamespace(stub=stub)
            for path, image in images.items():
                await _upload(stub, io.BytesIO(bytes(image)), path)
            with pytest.raises(ExecutionError, match=r"archive/data/0 \(stored"):
                await volume.read_torch_save(client, "vo-g", "/crc.pt")
            got = await volume.read_torch_save(client, "vo-g", "/nocrc.pt")
            want = torch.load(io.BytesIO(bytes(images["/nocrc.pt"])), map_location="cuda")
            assert not torch.equal(got["a"], sd["a"]) and torch.equal(got["a"], want["a"])

    asyncio.run(run())


def test_work_on_a_side_stream_after_the_call_sees_the_values(gpu_backend):
    import torch

    sd = {"w": torch.randn(64 * MiB // 4, device="cuda"), "v": torch.randn(7, device="cuda")}
    want = {k: float(v.double().sum()) for k, v in sd.items()}
    stream = torch.cuda.Stream()

    async def run():
        async with running_volume_server(blob_utils.BLOCK_SIZE) as (stub, _):
            client = types.SimpleNamespace(stub=stub)
            await _upload(stub, DeviceFile.torch_save(sd), "/s.pt")
            torch.cuda.synchronize()
            with torch.cuda.stream(stream):
                got = await volume.read_torch_save(client, "vo-g", "/s.pt", staging_bytes=16 * MiB)
                sums = {k: v.double().sum() for k, v in got.items()}  # enqueued on the side stream, no sync between
            stream.synchronize()
            assert {k: float(s) for k, s in sums.items()} == want

    asyncio.run(run())
