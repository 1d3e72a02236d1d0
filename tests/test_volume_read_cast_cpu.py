"""Safetensors tensors read from a volume and converted to bfloat16, float16 or float32 as they land, on the CPU: the C
ABI of ``b200h_copy_cast_boxes_from_host``, and ``read_safetensors`` / ``read_safetensors_slices`` with ``dtype=``
against the fake read server, over host-memory device files with a context whose ``copy_cast_boxes_from_host`` asserts
the entry's argument rules and converts with torch on the host.  Results are compared with
``safetensors.torch.load(data)[name][index].to(dtype)``."""
import asyncio
import ctypes
import json
import os
import random
import re

import numpy as np
import pytest
import torch
from safetensors.torch import load as st_load
from safetensors.torch import save as st_save

from modal_client_b200 import _lib, device_file, volume
from tests.test_stage_ranges_cpu import range_pieces
from tests.test_volume_read_cpu import BS, _LoadHostSegments, no_sleep, read_backend, volume_with  # noqa: F401
from tests.test_volume_read_slices_cpu import BoxContext, _random_index, _same, _tensor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
_BY_CODE = {_lib.DT_F32: F32, _lib.DT_F16: F16, _lib.DT_BF16: BF16}


class CastContext(BoxContext):
    """Plus ``copy_cast_boxes_from_host``: every argument rule of the entry asserted, the elements converted with
    torch's ``.to()`` on the host, and a log of the boxes of every call."""

    def copy_cast_boxes_from_host(self, seg_ptrs, seg_lens, file_first_seg, boxes, src, stream=0):
        self.calls.append(("copy_cast_boxes_from_host", [tuple(b) for b in boxes]))
        written = []
        for f, off, width, rows, at, pitch, st, dt in boxes:
            assert st in _BY_CODE and dt in _BY_CODE and st != dt
            sd, dd = _BY_CODE[st], _BY_CODE[dt]
            ss, ds = sd.itemsize, dd.itemsize
            assert f < len(file_first_seg) - 1
            assert width % ss == 0 and pitch % ss == 0
            assert (src.ctypes.data + at) % ss == 0, "a row's source is not element-aligned"
            if width * rows == 0:
                continue
            assert rows == 1 or pitch >= width
            assert at + (rows - 1) * pitch + width <= src.size
            n = rows * width // ss * ds
            pieces = range_pieces(seg_ptrs, seg_lens, file_first_seg, f, off, n)
            assert len(pieces) == 1, "a cast box's destination crosses a segment edge"
            p = pieces[0][0]
            assert p % ds == 0, "a cast box's destination is not element-aligned"
            rows_bytes = b"".join(src[at + r * pitch : at + r * pitch + width].tobytes() for r in range(rows))
            out = torch.frombuffer(bytearray(rows_bytes), dtype=sd).to(dd).view(torch.uint8).numpy().tobytes()
            assert len(out) == n
            ctypes.memmove(p, out, n)
            written.append((p, p + n))
        written.sort()
        assert all(a[1] <= b[0] for a, b in zip(written, written[1:])), "two boxes write the same device bytes"


@pytest.fixture
def cast_backend(monkeypatch, read_backend):  # noqa: F811
    from modal_client_b200 import _backend

    ctx = CastContext()
    monkeypatch.setattr(_backend, "_override", ctx)
    return ctx


@pytest.fixture
def waves(monkeypatch):
    """The entry points each wave's copy called, one list per wave."""
    out = []
    real = volume._load_in_waves

    async def spy(slices, load, *args):
        def counted(wave, at, buf, ctx):
            before = len(ctx.calls)
            loaded = load(wave, at, buf, ctx)
            out.append([c[0] for c in ctx.calls[before:]])
            return loaded

        await real(slices, counted, *args)

    monkeypatch.setattr(volume, "_load_in_waves", spy)
    return out


@pytest.fixture
def fetched(monkeypatch):
    """The URL of every block GET, in order."""
    urls = []
    real = volume._fetch_block

    async def spy(url, out, want, semaphore):
        urls.append(url)
        await real(url, out, want, semaphore)

    monkeypatch.setattr(volume, "_fetch_block", spy)
    return urls


def _float(shape, dtype, g):
    """Random bit patterns without NaNs: torch's CPU casts keep or drop NaN payloads depending on the loop that
    converts (the GPU tests compare NaN bits with the device's cast)."""
    t = _tensor(shape, dtype, g)
    return t.masked_fill(t.isnan(), 0.0)


def _mixed(seed: int):
    g = torch.Generator().manual_seed(seed)
    return {"w.f32": _float((37, 211), F32, g), "h.bf16": _float((1001,), BF16, g), "e.f16": _float((13, 77), F16, g),
            "ids.i64": _tensor((333,), torch.int64, g), "mask": _tensor((17,), torch.bool, g),
            "odd.f32": _float((5, 3, 7), F32, g), "s.f16": torch.tensor(1.5, dtype=F16), "z.f32": torch.zeros(0, 5)}


def _cast(t: torch.Tensor, dtype):
    return t.to(dtype) if t.dtype in (F32, F16, BF16) else t


def _valid_index(t: torch.Tensor, rnd: random.Random):
    """A random index that torch accepts for ``t``."""
    while True:
        index = _random_index(tuple(t.shape), rnd)
        try:
            t[index]
            return index
        except IndexError:
            pass


def _padded(image: bytes, pad: int) -> bytes:
    """``image`` with ``pad`` more spaces in its header: its data region moves by ``pad`` bytes."""
    n = int.from_bytes(image[:8], "little")
    text = image[8 : 8 + n] + b" " * pad
    return len(text).to_bytes(8, "little") + text + image[8 + n :]


# ------------------------------------------------------------------------------------------------ C ABI


def test_copy_cast_boxes_from_host_is_declared_exported_and_rejects_a_null_context():
    header = open(os.path.join(ROOT, "include", "b200hash.h")).read()
    assert re.search(r"\bint b200h_copy_cast_boxes_from_host\(b200h_ctx\* ctx, const b200h_segment\* segs,", header)
    assert re.search(r"typedef struct b200h_cast_box \{\s*b200h_box box;\s*uint64_t src_type, dst_type;", header)
    for name, code in (("F32", _lib.DT_F32), ("F16", _lib.DT_F16), ("BF16", _lib.DT_BF16)):
        assert re.search(rf"#define B200H_DT_{name} {code}u\b", header)
    comment = header.split("int b200h_copy_cast_boxes_from_host")[0].rsplit("/*", 1)[-1]
    assert "Replaces: _read_file_into_fileobj (py/modal/volume.py:923-1000)" in comment and ".to(dtype)" in comment
    assert "b200h_copy_cast_boxes_from_host" in _lib.ABI_SYMBOLS
    L = _lib.load_library()
    assert hasattr(L, "b200h_copy_cast_boxes_from_host")
    first = (ctypes.c_uint64 * 1)(0)
    assert L.b200h_copy_cast_boxes_from_host(None, None, 0, first, 0, None, 0, None, 0, None) == -1  # B200H_E_INVALID
    import modal_client_b200

    assert modal_client_b200.load_cast_boxes is device_file.load_cast_boxes
    assert "load_cast_boxes" in device_file.__all__


def test_load_cast_boxes_rejects_malformed_boxes():
    with pytest.raises(ValueError, match="a box is"):
        device_file.load_cast_boxes([], [(0, 0, 4, 1, 0, 4, F32)], np.zeros(16, np.uint8), ctx=object())
    with pytest.raises(ValueError, match="converts between"):
        device_file.load_cast_boxes([], [(0, 0, 8, 1, 0, 8, torch.float64, BF16)], np.zeros(16, np.uint8), ctx=object())


# ------------------------------------------------------------------------------------ the alignment premise


def test_safetensors_save_puts_every_tensor_at_a_multiple_of_its_element_size():
    rnd = random.Random(11)
    g = torch.Generator().manual_seed(11)
    dtypes = [torch.float64, F32, F16, BF16, torch.int64, torch.int32, torch.int16, torch.int8, torch.uint8,
              torch.bool, torch.float8_e4m3fn, torch.float8_e5m2]
    for _ in range(60):
        sd = {}
        for i in range(rnd.randint(1, 12)):
            name = "".join(rnd.choice("abcdefgh._") for _ in range(rnd.randint(1, 40))) + str(i)
            shape = tuple(rnd.randint(0, 9) for _ in range(rnd.randint(0, 3)))
            sd[name] = _tensor(shape, rnd.choice(dtypes), g)
        meta = {"k" * rnd.randint(0, 9): "v" * rnd.randint(0, 33)} if rnd.random() < 0.5 else None
        image = st_save(sd, metadata=meta)
        n = int.from_bytes(image[:8], "little")
        header = json.loads(image[8 : 8 + n])
        for name, t in sd.items():
            assert (8 + n + header[name]["data_offsets"][0]) % t.element_size() == 0, (name, t.dtype)


# -------------------------------------------------------------------------------------------------- parity


@pytest.mark.parametrize("pad", [0, 8])  # a safetensors data region starts at 0 or 8 mod 16
def test_read_safetensors_converts_every_float_tensor_as_to_does(cast_backend, pad):
    image = _padded(st_save(_mixed(1)), pad)
    full = st_load(image)

    async def run():
        async with volume_with({"/m": image}) as (client, _, _):
            for dtype in (BF16, F16, F32):
                got = await volume.read_safetensors(client, "vo-r", "/m", dtype=dtype, staging_bytes=2 * BS)
                assert sorted(got) == sorted(full)
                for name, t in full.items():
                    _same(got[name], _cast(t, dtype), (dtype, name))
            mapping = {"w.f32": BF16, "h.bf16": F32, "e.f16": F16, "odd.f32": F16}
            got = await volume.read_safetensors(client, "vo-r", "/m", dtype=mapping, staging_bytes=4 * BS)
            for name, t in full.items():
                _same(got[name], t.to(mapping[name]) if name in mapping else t, name)

    asyncio.run(run())


@pytest.mark.parametrize("pad", [0, 8])
def test_read_safetensors_slices_converts_every_slice_as_to_does(cast_backend, pad):
    rnd = random.Random(3 + pad)
    image = _padded(st_save(_mixed(2)), pad)
    full = st_load(image)

    async def run():
        async with volume_with({"/m": image}) as (client, _, _):
            for k in range(12):
                dtype = (BF16, F16, F32)[k % 3]
                select = {name: _valid_index(t, rnd) for name, t in full.items()}
                form = dtype if k % 2 else {name: dtype for name, t in full.items() if t.dtype in (F32, F16, BF16)}
                got = await volume.read_safetensors_slices(client, "vo-r", "/m", select, dtype=form,
                                                           staging_bytes=2 * BS)
                for name, index in select.items():
                    _same(got[name], _cast(full[name][index], dtype), (dtype, name, index))

    asyncio.run(run())


# ---------------------------------------------------------------------------------------- requests and calls


def test_converted_reads_make_the_unconverted_requests_and_two_calls_at_most_per_wave(cast_backend, waves, fetched):
    g = torch.Generator().manual_seed(4)
    # F32 tensors across many 4096-byte blocks, one block per half: both kinds of wave edge (half 0 -> 1, 1 -> 0)
    sd = {"a": _float((40, 300), F32, g), "b": _float((3001,), BF16, g), "c": _tensor((700,), torch.int32, g),
          "d": _float((6, 9, 70), F16, g)}
    image = st_save(sd)
    full = st_load(image)
    cases = [(None, BF16), ({"a": (slice(None), slice(2, 40)), "d": (slice(1, 5), 3)}, {"a": BF16, "d": F32}),
             ({"a": (slice(5, 35),), "b": slice(100, 2900), "c": ...}, F16)]

    async def run():
        async with volume_with({"/m": image}) as (client, stub, _):
            for select, dtype in cases:
                for form in (None, dtype):
                    calls, nfetched, nwaves = len(stub.get_file_calls), len(fetched), len(waves)
                    if select is None:
                        got = await volume.read_safetensors(client, "vo-r", "/m", dtype=form, staging_bytes=2 * BS)
                        want = {k: _cast(t, form) if form else t for k, t in full.items()}
                    else:
                        got = await volume.read_safetensors_slices(client, "vo-r", "/m", select, dtype=form,
                                                                   staging_bytes=2 * BS)
                        targets = form if isinstance(form, dict) else {k: form for k in select} if form else {}
                        want = {k: _cast(full[k][i], targets[k]) if k in targets else full[k][i]
                                for k, i in select.items()}
                    for k, t in want.items():
                        _same(got[k], t, (select, form, k))
                    reqs = [(r.start, r.len) for r in stub.get_file_calls[calls:]]
                    gets = fetched[nfetched:]
                    if form is None:
                        plain_reqs, plain_gets = reqs, gets
                        continue
                    assert reqs == plain_reqs and gets == plain_gets, (select, form)
                    per_wave = waves[nwaves:]
                    assert len(per_wave) >= 3, per_wave  # both halves, and back to the first
                    for calls_of_wave in per_wave:
                        assert calls_of_wave.count("copy_boxes_from_host") <= 1, per_wave
                        assert calls_of_wave.count("copy_cast_boxes_from_host") <= 1, per_wave
                        assert "copy_ranges_from_host" not in calls_of_wave
                    if select is None or "c" in select:  # int32 "c" meets converted tensors inside a block
                        assert any(len(c) == 2 for c in per_wave)
                    assert all("copy_cast_boxes_from_host" in c for c in per_wave if len(c) == 2)

    asyncio.run(run())


def test_a_cast_box_is_cut_at_wave_edges_and_skipped_blocks(cast_backend):
    sd = {"w": torch.randn(64, 300, generator=torch.Generator().manual_seed(5))}  # 1200-byte F32 rows
    image = st_save(sd)

    async def run():
        async with volume_with({"/m": image}) as (client, _, _):
            for index in [(slice(None), slice(10, 290)), (slice(3, 60),), (slice(None), 7)]:
                before = len(cast_backend.calls)
                got = await volume.read_safetensors_slices(client, "vo-r", "/m", {"w": index}, dtype=BF16,
                                                           staging_bytes=2 * BS)
                _same(got["w"], sd["w"][index].to(BF16))
                boxes = [b for c in cast_backend.calls[before:] if c[0] == "copy_cast_boxes_from_host" for b in c[1]]
                assert not [c for c in cast_backend.calls[before:] if c[0] == "copy_boxes_from_host"]
                dests = sorted((b[1], b[1] + b[2] * b[3] // 2) for b in boxes)  # F32 -> BF16: half the bytes
                assert dests[0][0] == 0 and dests[-1][1] == got["w"].numel() * 2
                assert all(a[1] == b[0] for a, b in zip(dests, dests[1:]))  # the boxes tile the result
                if index == (slice(None), slice(10, 290)):
                    assert any(b[3] == 1 and b[2] < 280 * 4 for b in boxes)  # a row cut at a block edge

    asyncio.run(run())


def test_a_dtype_that_converts_nothing_makes_exactly_the_calls_without_it(cast_backend, fetched):
    g = torch.Generator().manual_seed(6)
    sd = {"a": _tensor((30, 500), BF16, g), "b": _tensor((77,), torch.int64, g), "c": _tensor((9, 9), BF16, g)}
    image = st_save(sd)

    async def run():
        async with volume_with({"/m": image}) as (client, stub, _):
            logs = []
            for kw in ({}, {"dtype": BF16}, {"dtype": {"a": BF16}}):
                for sliced in (False, True):
                    calls, nfetched, nctx = len(stub.get_file_calls), len(fetched), len(cast_backend.calls)
                    if sliced:
                        got = await volume.read_safetensors_slices(client, "vo-r", "/m", {"a": (slice(3, 9),), "b": 5},
                                                                   staging_bytes=2 * BS, **kw)
                        _same(got["a"], sd["a"][3:9])
                    else:
                        got = await volume.read_safetensors(client, "vo-r", "/m", staging_bytes=2 * BS, **kw)
                        _same(got["a"], sd["a"])
                    logs.append((sliced, [(r.start, r.len) for r in stub.get_file_calls[calls:]], fetched[nfetched:],
                                 cast_backend.calls[nctx:]))
            for sliced in (False, True):
                same = [log[1:] for log in logs if log[0] == sliced]
                assert same[0] == same[1] == same[2]
                assert not any(c[0] == "copy_cast_boxes_from_host" for c in same[0][2])

    asyncio.run(run())


# ------------------------------------------------------------------------------------------- rejections


def test_every_rejection_names_every_offender_before_any_data_get(cast_backend):
    g = torch.Generator().manual_seed(7)
    sd = {"a": _tensor((8, 8), F32, g), "d": _tensor((5,), torch.float64, g), "e": _tensor((3,), torch.float8_e4m3fn, g),
          "i": _tensor((4,), torch.int32, g), "h": _tensor((6,), F16, g)}
    image = st_save(sd)
    n = int.from_bytes(image[:8], "little")
    a_at = 8 + n + 1 + json.loads(image[8 : 8 + n])["a"]["data_offsets"][0]
    misaligned = _padded(image, 1)  # every tensor one byte off: F32, F16, F64 and I32 starts are misaligned
    cases = [
        ("/m", BF16, None, ["'d' is F64", "'e' is F8_E4M3"]),
        ("/m", torch.float64, None, ["torch.float64 is not a supported target"]),
        ("/m", torch.int8, None, ["torch.int8 is not a supported target"]),
        ("/m", "bfloat16", None, ["bfloat16 is not a supported target"]),
        ("/m", {"a": BF16, "nope": F16, "zz": F32}, None, ["'nope' is in dtype but not", "'zz' is in dtype but not"]),
        ("/m", {"a": torch.float64, "h": torch.int16}, None, ["'a': torch.float64 is not", "'h': torch.int16 is not"]),
        ("/m", {"i": BF16, "d": F32}, None, ["'i' is I32; only F32, F16 and BF16", "'d' is F64"]),
        ("/x", {"a": BF16, "h": F32, "i": BF16}, None, [f"'a' starts at file offset {a_at}, not a multiple of its "
                                                       "element size 4", "'h' starts at file offset", "'i' is I32"]),
        ("/m", {"a": BF16, "h": F32}, {"a": 0, "i": 1}, ["'h' is in dtype but not selected"]),
    ]

    async def run():
        async with volume_with({"/m": image, "/x": misaligned}) as (client, stub, faults):
            for path, dtype, select, parts in cases:
                for sliced in ((False, True) if select is None else (True,)):
                    calls, gets = len(stub.get_file_calls), faults["gets"]
                    with pytest.raises(ValueError) as err:
                        if sliced:
                            await volume.read_safetensors_slices(client, "vo-r", path, select or {k: ... for k in sd},
                                                                 dtype=dtype)
                        else:
                            await volume.read_safetensors(client, "vo-r", path, dtype=dtype)
                    for part in parts:
                        assert part in str(err.value), (part, str(err.value))
                    assert len(stub.get_file_calls) == calls + 3 and faults["gets"] == gets + 2  # the header only
            # the misaligned file still loads unconverted, and converts what is aligned (U8 and the F16 pair at odd)
            got = await volume.read_safetensors(client, "vo-r", "/x")
            _same(got["a"], sd["a"])

    asyncio.run(run())


def test_into_messages_say_what_the_file_holds_and_what_it_converts_to(cast_backend):
    g = torch.Generator().manual_seed(8)
    sd = {"a": _float((30, 70), F32, g), "b": _tensor((50,), torch.int64, g), "c": _float((9,), BF16, g)}
    image = st_save(sd)
    full = st_load(image)

    async def run():
        async with volume_with({"/m": image}) as (client, _, faults):
            into = {"a": torch.zeros(30, 70, dtype=BF16), "b": torch.zeros(50, dtype=torch.int64), "c": torch.zeros(9, dtype=BF16)}
            got = await volume.read_safetensors(client, "vo-r", "/m", into=into, dtype=BF16)
            for k in sd:
                assert got[k] is into[k]
                _same(got[k], _cast(full[k], BF16), k)
            sl = {"a": torch.zeros(30, 10, dtype=F16), "c": torch.zeros(4, dtype=F32)}
            got = await volume.read_safetensors_slices(client, "vo-r", "/m", {"a": (slice(None), slice(5, 15)),
                                                                             "c": slice(2, 6)},
                                                       into=sl, dtype={"a": F16, "c": F32})
            _same(got["a"], full["a"][:, 5:15].to(F16)), _same(got["c"], full["c"][2:6].to(F32))
            gets = faults["gets"]
            wrong = {"a": torch.zeros(30, 70), "b": torch.zeros(50, dtype=torch.int64), "c": torch.zeros(9, dtype=F16)}
            with pytest.raises(ValueError) as err:
                await volume.read_safetensors(client, "vo-r", "/m", into=wrong, dtype=BF16)
            msg = str(err.value)
            assert "'a': the file holds torch.float32 [30, 70], converted to torch.bfloat16, into has torch.float32" in msg
            assert "'c': the file holds torch.bfloat16 [9], into has torch.float16 [9]" in msg  # BF16 stays BF16
            with pytest.raises(ValueError) as err:
                await volume.read_safetensors(client, "vo-r", "/m", into=wrong)
            assert "'a': the file holds" not in str(err.value) or "converted" not in str(err.value)
            assert "'c': the file holds torch.bfloat16 [9], into has torch.float16 [9]" in str(err.value)
            with pytest.raises(ValueError) as err:
                await volume.read_safetensors_slices(client, "vo-r", "/m", {"a": 0}, into={"a": torch.zeros(70)},
                                                     dtype=F16)
            assert "'a': the slice is torch.float32 [70], converted to torch.float16, into has torch.float32 [70]" in \
                str(err.value)
            assert faults["gets"] == gets + 6  # only the headers' reads

    asyncio.run(run())
