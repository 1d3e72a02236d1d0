"""Slices of safetensors tensors read from a volume, on the CPU: the C ABI of ``b200h_copy_boxes_from_host``,
``read_safetensors_header`` and ``read_safetensors_slices`` against the fake read server, over host-memory device files
with a context whose ``copy_boxes_from_host`` does the moves with ``ctypes`` and asserts the entry's argument rules.
Results are compared with ``safetensors.torch.load(data)[name][index]`` and ``safe_open(...).get_slice(name)[index]``."""
import asyncio
import ctypes
import json
import os
import random
import re

import numpy as np
import pytest
import torch
from safetensors import safe_open
from safetensors.torch import load as st_load
from safetensors.torch import save as st_save

from modal_client_b200 import _lib, device_file, volume
from modal_client_b200.exception import ExecutionError
from tests.test_stage_ranges_cpu import range_pieces
from tests.test_volume_read_cpu import BS, ReadContext, _LoadHostSegments, no_sleep, read_backend, volume_with  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class BoxContext(ReadContext):
    """Plus ``copy_boxes_from_host``: the entry's argument rules asserted, the rows moved with ``ctypes``, and a log of
    the boxes of every call."""

    def copy_boxes_from_host(self, seg_ptrs, seg_lens, file_first_seg, boxes, src, stream=0):
        self.calls.append(("copy_boxes_from_host", [tuple(b) for b in boxes]))
        written = []
        for f, off, width, rows, at, pitch in boxes:
            assert f < len(file_first_seg) - 1
            if width * rows == 0:
                continue
            assert rows == 1 or pitch >= width
            assert at + (rows - 1) * pitch + width <= src.size
            for p, into, k in range_pieces(seg_ptrs, seg_lens, file_first_seg, f, off, rows * width):
                written.append((p, p + k))
                r0, r1 = into // width, (into + k - 1) // width
                for r in range(r0, r1 + 1):
                    lo, hi = max(into, r * width), min(into + k, (r + 1) * width)
                    ctypes.memmove(p + lo - into, src.ctypes.data + at + r * pitch + lo - r * width, hi - lo)
        written.sort()
        assert all(a[1] <= b[0] for a, b in zip(written, written[1:])), "two boxes write the same device bytes"


@pytest.fixture
def box_backend(monkeypatch, read_backend):
    from modal_client_b200 import _backend

    ctx = BoxContext()
    monkeypatch.setattr(_backend, "_override", ctx)
    return ctx


def box_calls(ctx):
    return [c[1] for c in ctx.calls if c[0] == "copy_boxes_from_host"]


def _st_bytes(t: torch.Tensor) -> bytes:
    if not t.numel():
        return b""
    flat = torch.empty(t.numel(), dtype=t.dtype)
    flat.copy_(t.reshape(-1))
    return flat.view(torch.uint8).numpy().tobytes()


def _same(got: torch.Tensor, want: torch.Tensor, what=""):
    assert got.dtype == want.dtype and tuple(got.shape) == tuple(want.shape), (what, got.shape, want.shape)
    assert got.is_contiguous(), what
    assert _st_bytes(got) == _st_bytes(want), what


# ------------------------------------------------------------------------------------------------ C ABI


def test_copy_boxes_from_host_is_declared_exported_and_rejects_a_null_context():
    header = open(os.path.join(ROOT, "include", "b200hash.h")).read()
    assert re.search(r"\bint b200h_copy_boxes_from_host\(b200h_ctx\* ctx, const b200h_segment\* segs,", header)
    assert re.search(r"typedef struct b200h_box \{", header)
    comment = header.split("int b200h_copy_boxes_from_host")[0].rsplit("/*", 1)[-1]
    assert "Replaces: _read_file_into_fileobj (py/modal/volume.py:923-1000)" in comment and "get_slice" in comment
    assert "b200h_copy_boxes_from_host" in _lib.ABI_SYMBOLS
    L = _lib.load_library()
    assert hasattr(L, "b200h_copy_boxes_from_host")
    first = (ctypes.c_uint64 * 1)(0)
    assert L.b200h_copy_boxes_from_host(None, None, 0, first, 0, None, 0, None, 0, None) == -1  # B200H_E_INVALID


# ------------------------------------------------------------------------------------------------ header


def _dtypes():
    return [getattr(torch, name) for name, _ in device_file._ST_TAGS
            if hasattr(torch, name) and name not in ("float4_e2m1fn_x2", "float8_e8m0fnu")]


def _tensor(shape, dtype, g):
    raw = torch.randint(0, 256, (int(np.prod(shape)) * dtype.itemsize,), generator=g, dtype=torch.uint8)
    if dtype == torch.bool:
        return (raw[: int(np.prod(shape))] & 1).bool().reshape(shape)
    return raw.view(dtype).reshape(shape)


def test_read_safetensors_header_equals_safe_open(box_backend, tmp_path):
    g = torch.Generator().manual_seed(1)
    sd = {f"t{i}.{str(dt).split('.')[-1]}": _tensor((3, i + 1), dt, g) for i, dt in enumerate(_dtypes())}
    sd["scalar"], sd["empty"] = torch.tensor(2.5), torch.zeros(0, 4)
    image = st_save(sd, metadata={"format": "pt", "x": "y"})
    (tmp_path / "m").write_bytes(image)

    async def run():
        async with volume_with({"/m": image, "/n": st_save({"a": torch.ones(2)})}) as (client, stub, _):
            calls = len(stub.get_file_calls)
            meta, info = await volume.read_safetensors_header(client, "vo-r", "/m")
            assert len(stub.get_file_calls) == calls + 3
            with safe_open(str(tmp_path / "m"), "pt") as f:
                assert meta == f.metadata()
                assert sorted(info) == sorted(f.keys())
                for k in f.keys():
                    t = f.get_tensor(k)
                    assert info[k] == (t.dtype, tuple(t.shape)), k
            n = int.from_bytes(image[:8], "little")
            offsets = {k: v["data_offsets"] for k, v in json.loads(image[8 : 8 + n]).items() if k != "__metadata__"}
            assert list(info) == sorted(offsets, key=lambda k: offsets[k])  # data order
            assert (await volume.read_safetensors_header(client, "vo-r", "/n"))[0] is None
            with pytest.raises(FileNotFoundError):
                await volume.read_safetensors_header(client, "vo-r", "/missing")

    asyncio.run(run())


# ------------------------------------------------------------------------------------------ slice parity


def _random_index(shape, rnd: random.Random):
    def one(d):
        if rnd.random() < 0.3 and d:
            return rnd.randrange(-d, d)
        lo = rnd.choice([None, rnd.randint(-d - 3, d + 3)])
        hi = rnd.choice([None, rnd.randint(-d - 3, d + 3)])
        return slice(lo, hi, rnd.choice([None, 1]))

    items = [one(d) for d in shape[: rnd.randint(0, len(shape))]]
    if rnd.random() < 0.3:
        items.insert(rnd.randint(0, len(items)), Ellipsis)
        if len(shape) > len(items) - 1 and rnd.random() < 0.5:
            items.append(one(shape[-1]))
    if len([x for x in items if x is not Ellipsis]) > len(shape):
        items = items[: len(shape)]
    return items[0] if len(items) == 1 and rnd.random() < 0.5 else tuple(items)


def test_slices_equal_torch_and_safe_open_for_every_dtype_index_and_phase(box_backend, tmp_path):
    g = torch.Generator().manual_seed(2)
    rnd = random.Random(5)
    base = {}
    for i, dt in enumerate(_dtypes()):
        base[f"m{i}"] = _tensor((23 + i, 37 + 3 * i), dt, g)  # spans blocks: 4096-byte blocks
    base["cube"] = _tensor((5, 17, 61), torch.float32, g)
    base["row"] = _tensor((3 * BS + 5,), torch.int16, g)
    base["scalar"] = torch.tensor(7.25, dtype=torch.float64)
    plain = st_save(base)
    n = int.from_bytes(plain[:8], "little")
    header = plain[8 : 8 + n].rstrip(b" ")
    images = {}
    for pad in range(16):  # header lengths that give every data phase mod 16
        text = header + b" " * pad
        images[f"/p{pad}"] = len(text).to_bytes(8, "little") + text + plain[8 + n :]
    assert {(8 + int.from_bytes(im[:8], "little")) % 16 for im in images.values()} == set(range(16))

    async def run():
        async with volume_with(images) as (client, _, _):
            for path, image in images.items():
                (tmp_path / "f").write_bytes(image)
                full = st_load(image)
                select = {}
                for name, t in full.items():
                    select[name] = _random_index(tuple(t.shape), rnd)
                got = await volume.read_safetensors_slices(client, "vo-r", path, select, staging_bytes=4 * BS)
                assert list(got) == list(select)
                with safe_open(str(tmp_path / "f"), "pt") as f:
                    for name, index in select.items():
                        _same(got[name], full[name][index], (path, name, index))
                        if full[name].dim():
                            _same(got[name], f.get_slice(name)[index], (path, name, index))

    asyncio.run(run())


def test_slices_of_0d_and_empty_results(box_backend):
    sd = {"s": torch.tensor(3.0), "m": torch.arange(64 * 40, dtype=torch.float32).reshape(64, 40)}
    image = st_save(sd)

    async def run():
        async with volume_with({"/m": image}) as (client, stub, faults):
            got = await volume.read_safetensors_slices(client, "vo-r", "/m", {"s": (), "m": (5, ...)})
            _same(got["s"], sd["s"]), _same(got["m"], sd["m"][5])
            got = await volume.read_safetensors_slices(client, "vo-r", "/m", {"s": ..., "m": (slice(3, 3),)})
            _same(got["s"], sd["s"]), _same(got["m"], sd["m"][3:3])
            calls, gets = len(stub.get_file_calls), faults["gets"]
            got = await volume.read_safetensors_slices(client, "vo-r", "/m", {"m": (slice(9, 2), slice(None))})
            _same(got["m"], sd["m"][9:2])
            assert len(stub.get_file_calls) == calls + 3 and faults["gets"] == gets + 2  # the header only
            calls = len(stub.get_file_calls)
            assert await volume.read_safetensors_slices(client, "vo-r", "/m", {}) == {}
            assert len(stub.get_file_calls) == calls + 3

    asyncio.run(run())


# ------------------------------------------------------------------------------------------- downloads


def _expected_blocks(image: bytes, select: dict) -> set:
    """Blocks holding a selected element's bytes, from element offsets (independent of the planner)."""
    n = int.from_bytes(image[:8], "little")
    full = st_load(image)
    meta = json.loads(image[8 : 8 + n])
    out = set()
    for name, index in select.items():
        t = full[name]
        flat = torch.arange(t.numel()).reshape(t.shape)[index].reshape(-1)
        start = 8 + n + meta[name]["data_offsets"][0]
        for e in flat.tolist():
            for b in range(start + e * t.element_size(), start + (e + 1) * t.element_size()):
                out.add(b // BS)
    return out


def test_exactly_the_touched_blocks_are_fetched_once(box_backend, monkeypatch):
    g = torch.Generator().manual_seed(4)
    sd = {"a": _tensor((40, 300), torch.bfloat16, g), "b": _tensor((6, 9, 700), torch.float32, g),
          "c": _tensor((3000,), torch.int8, g), "d": _tensor((200, 50), torch.float16, g)}
    image = st_save(sd)
    cases = [{"b": (slice(None), slice(2, 4))}, {"a": (slice(10, 20),), "d": (slice(None), slice(5, 9))},
             {"b": (slice(1, 5), 3, slice(100, 120))}, {"c": slice(1000, 1001)}, {"a": -1, "c": ...}]
    fetched = []
    real = volume._fetch_block

    async def spy(url, out, want, semaphore):
        fetched.append(url)
        await real(url, out, want, semaphore)

    monkeypatch.setattr(volume, "_fetch_block", spy)

    async def run():
        async with volume_with({"/m": image}) as (client, stub, _):
            for select in cases:
                calls = len(stub.get_file_calls)
                fetched.clear()
                got = await volume.read_safetensors_slices(client, "vo-r", "/m", select, staging_bytes=2 * BS)
                for name, index in select.items():
                    _same(got[name], sd[name][index], (select, name))
                reqs = stub.get_file_calls[calls:]
                assert len(reqs) == 4, select
                data = reqs[3]
                data_fetches = fetched[2:]  # the header's two small reads come first
                assert len(data_fetches) == len(set(data_fetches))
                want = _expected_blocks(image, select)
                assert data.start == min(want) * BS
                # the URL of block k of the data call carries its slice; map fetched URLs back to block indices
                resp = await stub.VolumeGetFile2(data)
                index_of = {u: data.start // BS + k for k, u in enumerate(resp.get_urls)}
                blocks = [index_of[u] for u in data_fetches]
                assert len(blocks) == len(set(blocks)) and set(blocks) == want, select

    asyncio.run(run())


# ------------------------------------------------------------------------------------------- box splits


def test_boxes_split_at_wave_edges_and_skipped_blocks(box_backend):
    g = torch.Generator().manual_seed(6)
    sd = {"w": _tensor((64, 96), torch.float32, g),  # 384-byte rows: 64 rows over 6 blocks
          "x": _tensor((4, 8, 300), torch.bfloat16, g)}  # [E, R, C]: 4800-byte pitch over dim 0 > BS
    image = st_save(sd)
    _LoadHostSegments.log = []

    async def run():
        async with volume_with({"/m": image}) as (client, _, _):
            for index in [(slice(None), slice(10, 30)), (slice(7, 50),), (slice(None), 5)]:
                before = len(box_calls(box_backend))
                got = await volume.read_safetensors_slices(client, "vo-r", "/m", {"w": index}, staging_bytes=2 * BS)
                _same(got["w"], sd["w"][index])
                calls = box_calls(box_backend)[before:]
                assert len(calls) >= 2  # one block per half: many waves
                assert all(len(c) <= 3 for c in calls), calls  # a 2-D tensor: at most 3 boxes per wave
                rows = [b for c in calls for b in c]
                if index == (slice(None), slice(10, 30)):  # 80-byte rows, some cut at a wave edge
                    assert any(r[3] == 1 and r[2] < 80 for r in rows)
            got = await volume.read_safetensors_slices(client, "vo-r", "/m", {"x": (slice(None), slice(2, 3))},
                                                       staging_bytes=2 * BS)
            _same(got["x"], sd["x"][:, 2:3])
        log = _LoadHostSegments.log
        copies = [e for e in log if e[0] == "copy"]
        assert len(copies) > 4
        for _, k in copies:  # a half is refilled only after its previous copy was waited for
            if k >= 2:
                assert log.index(("wait", k - 2)) < log.index(("copy", k))

    asyncio.run(run())


def test_a_row_straddling_a_wave_edge_is_cut_into_two_boxes(box_backend):
    sd = {"w": torch.arange(10 * 1000, dtype=torch.int32).reshape(10, 1000)}  # 4000-byte rows over 4096-byte blocks
    image = st_save(sd)

    async def run():
        async with volume_with({"/m": image}) as (client, _, _):
            got = await volume.read_safetensors_slices(client, "vo-r", "/m", {"w": (slice(2, 9), slice(1, 999))},
                                                       staging_bytes=2 * BS)
            _same(got["w"], sd["w"][2:9, 1:999])
            calls = box_calls(box_backend)
            assert all(len(c) <= 3 for c in calls)
            dests = sorted((b[1], b[1] + b[2] * b[3]) for c in calls for b in c)
            assert dests[0][0] == 0 and dests[-1][1] == 7 * 998 * 4
            assert all(a[1] == b[0] for a, b in zip(dests, dests[1:]))  # the boxes tile the result
            assert any(b[3] == 1 and b[2] < 998 * 4 for c in calls for b in c)  # a cut row

    asyncio.run(run())


# --------------------------------------------------------------------------------------------- into=


def test_into_fills_in_place_and_lists_every_mismatch(box_backend):
    g = torch.Generator().manual_seed(8)
    sd = {"a": _tensor((30, 70), torch.float32, g), "b": _tensor((50,), torch.int64, g), "c": torch.tensor(1.5),
          "d": torch.ones(3)}  # in the file, not selected
    image = st_save(sd)
    select = {"a": (slice(None), slice(10, 20)), "b": slice(5, 45), "c": ()}

    async def run():
        async with volume_with({"/m": image}) as (client, _, faults):
            into = {"a": torch.zeros(30, 10), "b": torch.zeros(40, dtype=torch.int64), "c": torch.tensor(0.0)}
            ptrs = {k: v.data_ptr() for k, v in into.items()}
            got = await volume.read_safetensors_slices(client, "vo-r", "/m", select, into=into)
            for k in select:
                assert got[k] is into[k] and into[k].data_ptr() == ptrs[k]
                _same(got[k], sd[k][select[k]])
            gets = faults["gets"]
            big = torch.zeros(400)
            wrong = {"a": torch.zeros(10, 30).t(), "b": big[:40].view(torch.int64)[:20], "x": torch.zeros(1)}
            wrong["b"], wrong["d"] = torch.zeros(40, dtype=torch.int32), torch.zeros(3)
            with pytest.raises(ValueError) as err:
                await volume.read_safetensors_slices(client, "vo-r", "/m", select, into=wrong)
            msg = str(err.value)
            for part in ("read_safetensors_slices(into=...)", "'c' is selected but not in into",
                         "'x' is in into but not selected", "'d' is in into but not selected",
                         "'b': the slice is torch.int64 [40]",
                         "contiguous"):
                assert part in msg, (part, msg)
            overlap = {"a": big[:300].reshape(30, 10), "b": big[200:280].view(torch.int64), "c": torch.tensor(0.0)}
            with pytest.raises(ValueError, match="overlap"):
                await volume.read_safetensors_slices(client, "vo-r", "/m", select, into=overlap)
            assert faults["gets"] == gets + 4  # only the header's reads

    asyncio.run(run())


# ------------------------------------------------------------------------------------------- rejections


def test_rejected_indices_and_names_raise_before_any_data_get(box_backend, no_sleep):  # noqa: F811
    sd = {"m": torch.zeros(6, 8), "v": torch.zeros(5)}
    image = st_save(sd)
    bad = [(None, TypeError), ([1, 2], TypeError), (torch.tensor([1]), TypeError), (True, TypeError),
           ((slice(None), None), TypeError), (slice(0, 4, 2), ValueError), (slice(None, None, -1), ValueError),
           (6, IndexError), (-7, IndexError), ((0, 0, 0), IndexError), ((..., 0, ...), IndexError),
           ((slice(1.5, 3),), TypeError)]

    async def run():
        async with volume_with({"/m": image}) as (client, stub, faults):
            for index, exc in bad:
                gets = faults["gets"]
                with pytest.raises(exc):
                    await volume.read_safetensors_slices(client, "vo-r", "/m", {"m": index})
                assert faults["gets"] == gets + 2, index  # the header's two reads
                if exc is IndexError and Ellipsis not in (index if isinstance(index, tuple) else ()):  # as torch
                    with pytest.raises(IndexError):
                        sd["m"][index]
            with pytest.raises(ValueError) as err:
                await volume.read_safetensors_slices(client, "vo-r", "/m", {"m": 0, "nope": 1, "v": 0, "zz": ...})
            assert "'nope'" in str(err.value) and "'zz'" in str(err.value)
            with pytest.raises(FileNotFoundError):
                await volume.read_safetensors_slices(client, "vo-r", "/missing", {"m": 0})
            faults["short"] = True
            with pytest.raises(ExecutionError):
                await volume.read_safetensors_slices(client, "vo-r", "/m", {"m": 0})

    asyncio.run(run())


# ------------------------------------------------------------------------------------ nothing else changes


def test_read_safetensors_makes_the_same_requests(box_backend):
    g = torch.Generator().manual_seed(9)
    sd = {"a": _tensor((30, 700), torch.float32, g), "b": _tensor((11,), torch.int8, g)}
    image = st_save(sd)

    async def run():
        async with volume_with({"/m": image}) as (client, stub, _):
            calls = len(stub.get_file_calls)
            got = await volume.read_safetensors(client, "vo-r", "/m", staging_bytes=2 * BS)
            for k in sd:
                _same(got[k], sd[k])
            n = int.from_bytes(image[:8], "little")
            reqs = [(r.start, r.len) for r in stub.get_file_calls[calls:]]
            assert reqs == [(0, 8), (0, 8), (8, n), (8 + n, len(image) - 8 - n)]
            assert not box_calls(box_backend)

    asyncio.run(run())
