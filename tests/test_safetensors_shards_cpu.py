"""Sharded safetensors checkpoints (the Hugging Face Hub layout: ``model-0000k-of-0000n.safetensors`` plus
``model.safetensors.index.json``) on the CPU: ``DeviceFile.safetensors_shards`` against the files
``huggingface_hub.save_torch_state_dict`` writes, its refusals, an upload of every shard through one volumefs2 batch,
and ``volume.read_safetensors_index`` / ``read_safetensors_sharded`` against ``safetensors.torch.load`` of the Hub's
files, with the requests and copies they make, over host-memory device files and the fake read server."""
import asyncio
import json
import os
import random
import types

import pytest
import torch
from huggingface_hub import save_torch_state_dict
from safetensors.torch import load as st_load

from modal_client_b200 import device_file, volume
from tests import test_device_file_cast_cpu as upload_cast
from tests import test_volume_read_cast_cpu as read_cast
from tests.test_device_file_cast_cpu import CastHostDeviceFile, _CastHostSegments
from tests.test_volume_read_cpu import BS, read_backend, volume_with  # noqa: F401
from tests.test_volume_read_slices_cpu import _same
from tests.volume_read_server import running_volume_server

BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32


class ShardContext(upload_cast.CastContext, read_cast.CastContext):
    """The hash and staging entries of an upload (converting ones included) and the box copies of a read."""


@pytest.fixture
def backend(monkeypatch, read_backend):  # noqa: F811
    from modal_client_b200 import _backend

    ctx = ShardContext()
    monkeypatch.setattr(_backend, "_override", ctx)
    return ctx


def hub_files(sd, tmp_path, **kw) -> dict:
    """{file name: bytes} of what the Hub writes for ``sd``."""
    d = tmp_path / f"hub{len(os.listdir(tmp_path))}"
    d.mkdir()
    save_torch_state_dict(dict(sd), str(d), **kw)
    return {name: (d / name).read_bytes() for name in sorted(os.listdir(d))}


def our_files(shards) -> dict:
    out = {}
    for name, f in shards.files.items():
        f.seek(0)
        out[name] = f.read()
    if shards.index is not None:
        out[shards.index[0]] = shards.index[1]
    return out


def _parsed(image: bytes):
    n = int.from_bytes(image[:8], "little")
    return json.loads(image[8 : 8 + n]), image[8 + n :]


def assert_same_files(ours: dict, hub: dict):
    """Byte for byte, but for a file whose header has several metadata entries (the library writes them in no fixed
    order): its header as parsed and every data byte."""
    assert sorted(ours) == sorted(hub)
    for name, data in hub.items():
        if name.endswith(".json") or len(_parsed(data)[0].get("__metadata__", {})) <= 1:
            assert ours[name] == data, name
        else:
            assert _parsed(ours[name]) == _parsed(data), name


def llama(layers=3, hidden=64, inter=160, vocab=300, seed=0, dtype=BF16, tied=True):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g).to(dtype)  # noqa: E731
    sd = {"model.embed_tokens.weight": r(vocab, hidden)}
    for i in range(layers):
        p = f"model.layers.{i}."
        for k in ("q", "k", "v", "o"):
            sd[p + f"self_attn.{k}_proj.weight"] = r(hidden, hidden)
        for k, shape in (("gate", (inter, hidden)), ("up", (inter, hidden)), ("down", (hidden, inter))):
            sd[p + f"mlp.{k}_proj.weight"] = r(*shape)
        sd[p + "input_layernorm.weight"] = r(hidden)
        sd[p + "post_attention_layernorm.weight"] = r(hidden)
    sd["model.norm.weight"] = r(hidden)
    sd["lm_head.weight"] = sd["model.embed_tokens.weight"] if tied else r(vocab, hidden)
    return sd


def odd_dict(seed=1):
    """Mixed dtypes, zero-size and 0-d tensors, and a tensor larger than small limits."""
    g = torch.Generator().manual_seed(seed)
    sd = {"big.f32": torch.randn(3000, generator=g), "a.i64": torch.arange(50), "s.bf16": torch.tensor(1.5, dtype=BF16),
          "z.f32": torch.zeros(0, 5), "m.bool": torch.rand(33, generator=g) > 0.5, "h.f16": torch.randn(7, 9).half(),
          "z2.i8": torch.zeros(0, dtype=torch.int8), "u.u8": torch.arange(200, dtype=torch.uint8),
          "w.f64": torch.randn(40, generator=g, dtype=torch.float64), "s.i32": torch.tensor(7, dtype=torch.int32)}
    sd["tail.f32"] = torch.randn(500, generator=g)
    return sd


def tie_preserving_to(sd, dtype):
    """``{k: v.to(dtype)}`` with every storage converted once, so names that share a storage still share one (what
    ``model.to(dtype).state_dict()`` gives for tied weights)."""
    memo, out = {}, {}
    for k, v in sd.items():
        if v.dtype not in (F32, F16, BF16) or v.dtype == dtype:
            out[k] = v
            continue
        key = v.untyped_storage().data_ptr()
        if key not in memo or not key:
            memo[key] = torch.empty(0, dtype=v.dtype).set_(v.untyped_storage()).to(dtype)
        out[k] = memo[key].as_strided(v.shape, v.stride(), v.storage_offset())
    return out


# ----------------------------------------------------------------------------------------------- export


EXPORT_CASES = [
    ("one shard", lambda: llama(), dict()),
    ("two shards", lambda: llama(layers=2), dict(max_shard_size=100_000)),
    ("many shards", lambda: llama(layers=4, tied=False), dict(max_shard_size="30KB")),
    ("a tensor over the limit", lambda: odd_dict(), dict(max_shard_size=3000)),
    ("zero-size and 0-d, one file", lambda: odd_dict(), dict()),
    ("pattern and metadata, sharded", lambda: llama(layers=2), dict(max_shard_size="0.05MB",
                                                                  filename_pattern="weights{suffix}.st",
                                                                  metadata={"format": "pt", "note": "x"})),
    ("pattern and metadata, one file", lambda: llama(layers=1), dict(filename_pattern="w{suffix}.safetensors",
                                                                    metadata={"note": "x", "b": "y"})),
    ("tied, discard the embedding", lambda: llama(layers=2), dict(max_shard_size=50_000,
                                                                 shared_tensors_to_discard=["model.embed_tokens.weight"])),
    ("int limit of 1", lambda: odd_dict(2), dict(max_shard_size=1)),
]


@pytest.mark.parametrize("case", EXPORT_CASES, ids=[c[0] for c in EXPORT_CASES])
def test_export_equals_the_hubs_files(backend, tmp_path, case):
    _, make, kw = case
    sd = make()
    shards = CastHostDeviceFile.safetensors_shards(sd, **kw)
    assert_same_files(our_files(shards), hub_files(sd, tmp_path, **kw))
    assert list(shards.files) == sorted(shards.files)


def test_tied_weights_are_written_once_and_recorded(backend, tmp_path):
    sd = llama(layers=2)
    shards = CastHostDeviceFile.safetensors_shards(sd, max_shard_size=40_000)
    index = json.loads(shards.index[1])
    assert "model.embed_tokens.weight" not in index["weight_map"]  # the first covering name is kept: lm_head
    assert index["metadata"]["model.embed_tokens.weight"] == "lm_head.weight"
    assert len(shards.files) > 2
    # a view the whole storage covers is removed too; the segments are the tensors where they are
    sd["extra.view"] = sd["model.norm.weight"].view(8, 8)
    shards = CastHostDeviceFile.safetensors_shards(sd, max_shard_size=40_000)
    assert_same_files(our_files(shards), hub_files(sd, tmp_path, max_shard_size=40_000))
    ptrs = {s.data_ptr() for f in shards.files.values() for s in f._src.segments[1:]}
    assert sd["model.layers.1.mlp.up_proj.weight"].data_ptr() in ptrs


@pytest.mark.parametrize("seed", range(4))
def test_random_dicts_and_limits_equal_the_hub(backend, tmp_path, seed):
    rng = random.Random(seed)
    sd = upload_cast.random_dict(seed, n=20)
    for k in list(sd)[:3]:
        sd[k + ".tied"] = sd[k]
    limit = rng.choice([1, 100, 5000, "0.02MB", 10**9])
    kw = dict(max_shard_size=limit, metadata={"seed": str(seed)} if seed % 2 else None)
    assert_same_files(our_files(CastHostDeviceFile.safetensors_shards(sd, **kw)), hub_files(sd, tmp_path, **kw))


@pytest.mark.parametrize("kw", [dict(max_shard_size="60KB"), dict(), dict(max_shard_size=1, metadata={"k": "v"})])
def test_dtype_equals_the_hubs_save_of_the_converted_dict(backend, tmp_path, kw):
    sd = llama(layers=3, dtype=F32)
    sd["step"] = torch.arange(5)
    sd["h.f16"] = torch.randn(10, 10).half()
    for dtype in (BF16, {"model.norm.weight": F16, "model.layers.0.mlp.up_proj.weight": BF16}):
        shards = CastHostDeviceFile.safetensors_shards(sd, dtype=dtype, **kw)
        if isinstance(dtype, dict):
            pre = {k: v.to(dtype[k]) if k in dtype else v for k, v in sd.items()}
        else:
            pre = tie_preserving_to(sd, dtype)
        assert_same_files(our_files(shards), hub_files(pre, tmp_path, **kw))
        assert any(f._src.casts for f in shards.files.values())


def test_an_empty_dict_writes_nothing_as_the_hub(backend, tmp_path):
    shards = CastHostDeviceFile.safetensors_shards({})
    assert shards.files == {} and shards.index is None and hub_files({}, tmp_path) == {}


def test_every_refusal_comes_in_one_error_before_any_device_copy(backend):
    base = torch.arange(40, dtype=F32)
    sd = {"t": torch.ones(4, 6).t(), "part": base[:10], "part2": base[20:], "ok": torch.ones(3),
          "d": torch.ones(2, dtype=torch.float64), "meta": torch.ones(3, device="meta")}
    before = _CastHostSegments.to_device
    with pytest.raises(ValueError) as e:
        CastHostDeviceFile.safetensors_shards(sd, filename_pattern="model.safetensors", max_shard_size="5XB")
    msg = str(e.value)
    for part in ("filename_pattern 'model.safetensors' needs", "Unit 'XB' not supported",
                 "safetensors_shards['t'] needs a contiguous tensor", "safetensors_shards['meta'] needs a CUDA tensor",
                 "no name covers the whole storage of 'part'", "no name covers the whole storage of 'part2'"):
        assert part in msg, (part, msg)
    with pytest.raises(ValueError) as e:
        CastHostDeviceFile.safetensors_shards({"ok": torch.ones(3), "d": torch.ones(2, dtype=torch.float64),
                                               "i": torch.ones(2, dtype=torch.int32)}, dtype={"i": BF16, "no": F16})
    assert "'i' is I32; only F32" in str(e.value) and "'no' is in dtype but not" in str(e.value)
    with pytest.raises(ValueError, match="F64, which does not convert"):
        CastHostDeviceFile.safetensors_shards({"d": torch.ones(2, dtype=torch.float64)}, dtype=BF16)
    tied = torch.ones(4)
    with pytest.raises(ValueError, match="share a storage but convert to different dtypes"):
        CastHostDeviceFile.safetensors_shards({"a": tied, "b": tied}, dtype={"a": BF16})
    with pytest.raises(ValueError, match="reserved"):
        CastHostDeviceFile.safetensors_shards({"__metadata__": torch.ones(1)})
    with pytest.raises(ValueError, match="metadata entries must be str"):
        CastHostDeviceFile.safetensors_shards({"a": torch.ones(1)}, metadata={"a": 1})
    assert _CastHostSegments.to_device == before and not backend.calls


def test_parse_size_to_int_is_the_hubs():
    from huggingface_hub.serialization._base import parse_size_to_int as hub

    for s in ["5GB", "5gb", " 1.5 MB ", "100KB", "2TB", "0.05MB", 1234]:
        assert device_file.parse_size_to_int(s) == (hub(s) if isinstance(s, str) else s)
    for s in ["5", "5PB", "xMB"]:
        with pytest.raises(ValueError):
            device_file.parse_size_to_int(s)


# ----------------------------------------------------------------------------------------------- upload


@pytest.mark.parametrize("budget", [None, 3 * BS])
def test_put_uploads_every_shard_and_the_index_with_one_device_hash_call(backend, tmp_path, monkeypatch, budget):
    monkeypatch.setattr(volume, "DeviceFile", device_file.DeviceFile)  # the uploader's test: any DeviceFile subclass
    sd = llama(layers=3, dtype=F32)
    kw = dict(max_shard_size="40KB")
    shards = CastHostDeviceFile.safetensors_shards(sd, dtype=BF16, **kw)
    assert len(shards.files) >= 3
    want = hub_files(tie_preserving_to(sd, BF16), tmp_path, **kw)

    async def run():
        async with running_volume_server(BS) as (stub, _):
            batch = volume.VolumeUploadContextManager2("vo-s", types.SimpleNamespace(stub=stub),
                                                       device_staging_bytes=budget)
            async with batch:
                shards.put(batch, "/ckpt")
            assert batch.device_released.is_set()
            return {p: v[0] for p, v in stub.volume_files.items()}

    stored = asyncio.run(run())
    assert stored == {f"/ckpt/{name}": data for name, data in want.items()}
    hashes = [c for c in backend.calls if c[0].endswith("_device")]  # the index is hashed on the host's path
    assert hashes == [("hash_cast_segment_parts_device", len(shards.files), BS, hashes[0][3])]
    stages = [c for c in backend.calls if c[0] in ("copy_cast_ranges", "copy_ranges_to_host")]
    assert stages and (budget is None or all(c[0] == "copy_cast_ranges" for c in stages))


# ------------------------------------------------------------------------------------------------- read


@pytest.fixture
def waves(monkeypatch):
    """Per wave: (the file of every block, the copy entries it called, every block's offset in its file's range)."""
    out = []
    real = volume._load_in_waves

    async def spy(slices, load, *args):
        def counted(wave, at, buf, ctx):
            before = len(ctx.calls)
            loaded = load(wave, at, buf, ctx)
            out.append(([s[3] for s in wave], [c[0] for c in ctx.calls[before:]], [s[1] for s in wave]))
            return loaded

        await real(slices, counted, *args)

    monkeypatch.setattr(volume, "_load_in_waves", spy)
    return out


def _hub_volume(sd, tmp_path, root="/ckpt", **kw):
    files = hub_files(sd, tmp_path, **kw)
    return files, {f"{root}/{name}": data for name, data in files.items()}


def _merged(files: dict) -> dict:
    out = {}
    for name in sorted(files):
        if not name.endswith(".json"):
            out.update(st_load(files[name]))
    return out


def test_sharded_reads_equal_loading_the_hubs_files(backend, tmp_path, waves):
    sd = llama(layers=3, dtype=F32, tied=False)
    sd["step"] = torch.arange(7)
    sd["z"] = torch.zeros(0, 3)
    files, on_volume = _hub_volume(sd, tmp_path, max_shard_size="30KB")
    full = _merged(files)
    rnd = random.Random(3)

    async def run():
        async with volume_with(on_volume) as (client, _, _):
            index = "/ckpt/model.safetensors.index.json"
            meta, where = await volume.read_safetensors_index(client, "vo-r", index)
            assert meta == json.loads(files["model.safetensors.index.json"])["metadata"]
            assert sorted(where) == sorted(full)
            for name, (path, dt, shape) in where.items():
                assert path == "/ckpt/" + json.loads(files["model.safetensors.index.json"])["weight_map"][name]
                assert (dt, shape) == (full[name].dtype, tuple(full[name].shape))
            got = await volume.read_safetensors_sharded(client, "vo-r", index, staging_bytes=2 * BS)
            assert list(got) == list(where)  # shard order, then data order
            for k, t in full.items():
                _same(got[k], t, k)
            for dtype in (BF16, F16):
                got = await volume.read_safetensors_sharded(client, "vo-r", index, dtype=dtype, staging_bytes=4 * BS)
                for k, t in full.items():
                    _same(got[k], read_cast._cast(t, dtype), (dtype, k))
            into = {k: torch.full(t.shape, 7, dtype=BF16 if t.is_floating_point() else t.dtype) for k, t in full.items()}
            got = await volume.read_safetensors_sharded(client, "vo-r", index, into=into, dtype=BF16)
            assert all(got[k] is into[k] for k in full)
            for k, t in full.items():
                _same(into[k], read_cast._cast(t, BF16), k)
            for rank in range(3):
                select = {k: read_cast._valid_index(t, rnd) for k, t in full.items() if rnd.random() < 0.6}
                for dtype in (None, F16):
                    got = await volume.read_safetensors_sharded(client, "vo-r", index, select=select, dtype=dtype,
                                                                staging_bytes=2 * BS)
                    assert list(got) == list(select)
                    for k, i in select.items():
                        _same(got[k], read_cast._cast(full[k][i], dtype) if dtype else full[k][i], (rank, k, i))

    asyncio.run(run())
    assert any(len(set(shards)) > 1 for shards, _, _ in waves)  # waves that mix shards


@pytest.fixture
def data_gets(monkeypatch):
    """The URL of every block GET made inside the wave loop, one list per sharded read."""
    out, live = [], []
    real_fetch, real_waves = volume._fetch_block, volume._load_in_waves

    async def fetch(url, buf, want, semaphore):
        if live:
            out[-1].append(url)
        await real_fetch(url, buf, want, semaphore)

    async def waves(*args):
        out.append([])
        live.append(1)
        try:
            await real_waves(*args)
        finally:
            live.pop()

    monkeypatch.setattr(volume, "_fetch_block", fetch)
    monkeypatch.setattr(volume, "_load_in_waves", waves)
    return out


def _blocks(header_len: int, spans) -> set:
    """The blocks that hold a byte of ``spans`` -- (data offset, length) each -- of a safetensors file."""
    return {(8 + header_len + lo + i) // BS for lo, n in spans for i in (0, n - 1) if n} | \
        {b for lo, n in spans if n for b in range((8 + header_len + lo) // BS, (8 + header_len + lo + n - 1) // BS + 1)}


def test_requests_one_data_call_per_touched_shard_each_block_once_two_copies_per_wave(backend, tmp_path, monkeypatch,
                                                                                      waves, data_gets):
    sd = llama(layers=4, hidden=64, dtype=F32, tied=False)
    files, on_volume = _hub_volume(sd, tmp_path, max_shard_size="50KB")
    shard_names = sorted(n for n in files if not n.endswith(".json"))
    assert len(shard_names) >= 4
    full = _merged(files)
    weight_map = json.loads(files["model.safetensors.index.json"])["weight_map"]
    header = {}
    for name in shard_names:
        n = int.from_bytes(files[name][:8], "little")
        header[name] = (n, json.loads(files[name][8 : 8 + n]))
    cases = [(None, None), (None, BF16),
             ({"model.layers.0.mlp.up_proj.weight": (slice(40, 80),),
               "model.layers.3.self_attn.q_proj.weight": (slice(None), slice(16, 32))}, None),
             ({"model.layers.0.mlp.up_proj.weight": (slice(40, 80),), "model.norm.weight": ...}, BF16)]

    ranges = []  # (path, start) of every _block_slices call
    real = volume._block_slices

    async def spy(client, volume_id, path, start, n):
        ranges.append((path, start))
        return await real(client, volume_id, path, start, n)

    monkeypatch.setattr(volume, "_block_slices", spy)

    async def run():
        async with volume_with(on_volume) as (client, stub, _):
            for select, dtype in cases:
                calls, nw = len(stub.get_file_calls), len(waves)
                got = await volume.read_safetensors_sharded(client, "vo-r", "/ckpt/model.safetensors.index.json",
                                                            select=select, dtype=dtype, staging_bytes=8 * BS)
                for k in got:
                    want = full[k] if select is None else full[k][select[k]]
                    _same(got[k], read_cast._cast(want, dtype) if dtype else want, k)
                reqs = [(r.path, r.start, r.len) for r in stub.get_file_calls[calls:]]
                names = select or full
                touched = sorted({weight_map[k] for k in names})
                # the index (one call), then three per shard header, then one data call per touched shard
                assert reqs[0] == ("/ckpt/model.safetensors.index.json", 0, 0)
                assert sorted(p for p, _, _ in reqs[1 : 1 + 3 * len(shard_names)]) == \
                    sorted(f"/ckpt/{s}" for s in shard_names * 3)
                data = reqs[1 + 3 * len(shard_names) :]
                assert sorted(p for p, _, _ in data) == [f"/ckpt/{s}" for s in touched]
                # every touched block once, no other
                per_wave = waves[nw:]
                want_blocks = set()
                for s in touched:
                    n, h = header[s]
                    spans = []
                    for k in names:
                        if weight_map[k] != s:
                            continue
                        lo, hi = h[k]["data_offsets"]
                        if select is None or select[k] is ...:
                            spans.append((lo, hi - lo))
                        else:  # a row range (dim 0) or a column range (dim 1) of a 2-d F32 matrix
                            rows, cols = h[k]["shape"]
                            r = range(rows)[select[k][0]]
                            c = range(cols)[select[k][1]] if len(select[k]) > 1 else range(cols)
                            spans += [(lo + (i * cols + c.start) * 4, len(c) * 4) for i in r]
                    want_blocks |= {(f"/ckpt/{s}", b) for b in _blocks(n, spans)}
                live = ranges[-len(data) :]  # the data calls, in the order of the files of the wave loop
                got_blocks = [(live[i][0], (live[i][1] + off) // BS) for shards_of_wave, _, offs in per_wave
                              for i, off in zip(shards_of_wave, offs)]
                assert len(got_blocks) == len(set(got_blocks)) == len(data_gets[-1])
                assert set(got_blocks) == want_blocks, (select, dtype)
                for _, entries, _ in per_wave:
                    assert entries.count("copy_boxes_from_host") <= 1
                    assert entries.count("copy_cast_boxes_from_host") <= 1
                    assert "copy_ranges_from_host" not in entries
                if select is None:
                    assert any(len(set(s)) > 1 for s, _, _ in per_wave)  # waves that mix shards

    asyncio.run(run())


def test_every_index_inconsistency_is_rejected_before_any_data_get(backend, tmp_path):
    sd = llama(layers=2, tied=False)
    files, on_volume = _hub_volume(sd, tmp_path, max_shard_size="20KB")
    index = json.loads(files["model.safetensors.index.json"])
    shards = sorted(set(index["weight_map"].values()))
    wm = index["weight_map"]
    moved = dict(wm, **{"model.norm.weight": shards[0] if wm["model.norm.weight"] != shards[0] else shards[1]})
    missing = dict(wm, **{"ghost.weight": shards[0]})
    crowded = next(k for k, f in wm.items() if sum(g == f for g in wm.values()) > 1)
    dropped = {k: v for k, v in wm.items() if k != crowded}
    twice = {"/ckpt/dup.safetensors": files[wm["lm_head.weight"]]}
    both = dict(wm, **{"dup": "dup.safetensors"})
    cases = [
        (moved, {}, ["holds 'model.norm.weight', which weight_map maps to",
                     "weight_map maps 'model.norm.weight' to"]),
        (missing, {}, ["weight_map maps 'ghost.weight' to"]),
        (dropped, {}, [f"holds {crowded!r}, which weight_map does not name"]),
        (both, twice, ["'lm_head.weight' is in both", "weight_map maps 'dup' to dup.safetensors"]),
        (dict(wm, x="/abs.safetensors"), {}, ["'/abs.safetensors'"]),
        (dict(wm, x="../up.safetensors"), {}, ["'../up.safetensors'"]),
    ]

    async def run():
        extra = {f"/ckpt/bad{i}.json": json.dumps({"metadata": {}, "weight_map": m}).encode()
                 for i, (m, _, _) in enumerate(cases)}
        extra.update({p: d for _, more, _ in cases for p, d in more.items()})
        extra["/ckpt/notjson.json"] = b"{nope"
        async with volume_with({**on_volume, **extra}) as (client, stub, faults):
            for i, (_, _, parts) in enumerate(cases):
                for call in (volume.read_safetensors_index, volume.read_safetensors_sharded):
                    calls = len(stub.get_file_calls)
                    with pytest.raises(ValueError) as err:
                        await call(client, "vo-r", f"/ckpt/bad{i}.json")
                    for part in parts:
                        assert part in str(err.value), (part, str(err.value))
                    # only the index and header reads: no call covers a data region
                    assert all(r.len in (0, 8) or r.start == 8 for r in stub.get_file_calls[calls:])
            with pytest.raises(ValueError, match="not a valid JSON index"):
                await volume.read_safetensors_index(client, "vo-r", "/ckpt/notjson.json")
            with pytest.raises(ValueError, match="no tensors named 'nope'"):
                await volume.read_safetensors_sharded(client, "vo-r", "/ckpt/model.safetensors.index.json",
                                                      select={"nope": 0})

    asyncio.run(run())


def test_single_file_reads_make_the_same_requests_as_before(backend, tmp_path, waves):
    """``read_safetensors`` with ``dtype`` and ``read_safetensors_slices`` go through the same planner with one file:
    one data call, every wave's boxes against file 0."""
    sd = llama(layers=1, dtype=F32)
    files, on_volume = _hub_volume(sd, tmp_path)

    async def run():
        async with volume_with(on_volume) as (client, stub, _):
            calls = len(stub.get_file_calls)
            await volume.read_safetensors(client, "vo-r", "/ckpt/model.safetensors", dtype=BF16, staging_bytes=2 * BS)
            assert len(stub.get_file_calls) - calls == 4
            assert all(set(s) == {0} for s, _, _ in waves)
            boxes = [b for c in backend.calls if c[0] == "copy_cast_boxes_from_host" for b in c[1]]
            assert boxes and all(b[0] == 0 for b in boxes)

    asyncio.run(run())
