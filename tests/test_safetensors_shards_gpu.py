"""GPU: a ~2 GiB Llama-shaped checkpoint exported in the Hugging Face Hub's sharded layout with
``DeviceFile.safetensors_shards(..., max_shard_size="512MB")`` -- in bf16, and from F32 with ``dtype=torch.bfloat16``
-- uploaded over the loopback server with and without ``device_staging_bytes``, stored byte for byte as
``huggingface_hub.save_torch_state_dict`` writes it, and read back with ``volume.read_safetensors_sharded`` bitwise
equal, whole and as rank 3 of 8's tensor-parallel slices, with HBM growing by no more than the results plus 8 MiB."""
import asyncio
import os
import types

import pytest

from modal_client_b200 import blob_utils, device_file, volume
from tests.volume_read_server import running_volume_server

pytestmark = pytest.mark.gpu

MiB = 1 << 20
INDEX = "/ckpt/model.safetensors.index.json"


def llama(dtype, layers=5, h=4096, m=11008, vocab=32000):
    """About 2.3 GB in bf16: embedding (tied to lm_head), attention and MLP matrices, norms."""
    import torch

    g = torch.Generator(device="cuda").manual_seed(5)
    r = lambda *s: (torch.randn(*s, generator=g, device="cuda") * 0.02).to(dtype)  # noqa: E731
    sd = {"model.embed_tokens.weight": r(vocab, h)}
    for i in range(layers):
        p = f"model.layers.{i}."
        for k in "qkvo":
            sd[p + f"self_attn.{k}_proj.weight"] = r(h, h)
        sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"] = r(m, h), r(m, h)
        sd[p + "mlp.down_proj.weight"] = r(h, m)
        sd[p + "input_layernorm.weight"], sd[p + "post_attention_layernorm.weight"] = r(h), r(h)
    sd["model.norm.weight"] = r(h)
    sd["lm_head.weight"] = sd["model.embed_tokens.weight"]
    return sd


def tp_index(name: str, shape, rank: int = 3, ranks: int = 8):
    """Rank ``rank`` of ``ranks``: column-parallel rows, row-parallel columns, vocabulary rows; norms whole."""
    if len(shape) == 1:
        return ...
    if name.endswith(("o_proj.weight", "down_proj.weight")):
        n = shape[1] // ranks
        return (slice(None), slice(rank * n, (rank + 1) * n))
    n = shape[0] // ranks
    return (slice(rank * n, (rank + 1) * n),)


def hub_files(sd, d) -> dict:
    """{file name: bytes} of ``huggingface_hub.save_torch_state_dict`` of a host copy of ``sd`` that keeps its ties."""
    from huggingface_hub import save_torch_state_dict

    memo = {}
    host = {k: memo.setdefault(v.data_ptr(), v.cpu()) for k, v in sd.items()}
    d.mkdir()
    save_torch_state_dict(host, str(d), max_shard_size="512MB")
    return {name: (d / name).read_bytes() for name in sorted(os.listdir(d))}


def _same_bits(a, b):
    import torch

    iv = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(iv), b.contiguous().view(iv))


async def _grown(call):
    """(result, peak growth of torch's HBM allocations during ``call``, bytes of the result's tensors)."""
    import torch

    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = await call()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base, sum(t.numel() * t.element_size() for t in out.values())


def _check_round_trip(make_shards, sd, want_files, budget):
    import torch

    async def run():
        async with running_volume_server(blob_utils.BLOCK_SIZE) as (stub, _):
            client = types.SimpleNamespace(stub=stub)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            shards = make_shards()
            assert len(shards.files) >= 4 and shards.index is not None
            batch = volume.VolumeUploadContextManager2("vo-g", client, device_staging_bytes=budget)
            async with batch:
                shards.put(batch, "/ckpt")
            torch.cuda.synchronize()
            upload_growth = torch.cuda.max_memory_allocated() - base
            stored = {p[len("/ckpt/"):]: v[0] for p, v in stub.volume_files.items()}
            assert sorted(stored) == sorted(want_files)
            for name, data in want_files.items():
                assert stored[name] == data, name
            del stored, shards
            assert upload_growth <= 8 * MiB, upload_growth  # headers and digest tables only
            got, growth, results = await _grown(lambda: volume.read_safetensors_sharded(client, "vo-g", INDEX))
            assert growth <= results + 8 * MiB, (growth, results)
            kept = {k for k in sd if k != "model.embed_tokens.weight"}  # the Hub keeps lm_head of the tied pair
            assert set(got) == kept
            for k in kept:
                assert _same_bits(got[k], sd[k]), k
            del got
            _, where = await volume.read_safetensors_index(client, "vo-g", INDEX)
            select = {k: tp_index(k, shape) for k, (_, _, shape) in where.items()}
            got, growth, results = await _grown(lambda: volume.read_safetensors_sharded(client, "vo-g", INDEX,
                                                                                        select=select))
            assert growth <= results + 8 * MiB, (growth, results)
            for k, i in select.items():
                assert _same_bits(got[k], sd[k][i].contiguous()), k

    asyncio.run(run())


@pytest.mark.parametrize("budget", [None, 256 * MiB])
def test_a_2gib_bf16_checkpoint_round_trips_in_the_hubs_sharded_layout(gpu_backend, tmp_path, budget):
    import torch

    sd = llama(torch.bfloat16)
    want = hub_files(sd, tmp_path / "hub")
    _check_round_trip(lambda: device_file.safetensors_shards(sd, max_shard_size="512MB"), sd, want, budget)


def test_an_f32_checkpoint_exports_as_the_hubs_bf16_shards(gpu_backend, tmp_path):
    import torch

    sd32 = llama(torch.float32)
    sd16 = {}
    for k, v in sd32.items():  # converted once per storage: the tie stays a tie
        sd16[k] = next((sd16[j] for j in sd16 if sd32[j] is v), None)
        if sd16[k] is None:
            sd16[k] = v.to(torch.bfloat16)
    want = hub_files(sd16, tmp_path / "hub")
    _check_round_trip(lambda: device_file.safetensors_shards(sd32, max_shard_size="512MB", dtype=torch.bfloat16),
                      sd16, want, 256 * MiB)
