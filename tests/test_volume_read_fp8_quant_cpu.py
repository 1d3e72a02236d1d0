"""F32 / F16 / BF16 safetensors weights read from a volume and quantized to block-scaled FP8 E4M3 as they land, on the
CPU: the C ABI of ``b200h_fp8_amax_boxes_from_host`` and ``b200h_copy_quant_boxes_from_host``, and
``read_safetensors`` / ``read_safetensors_sharded`` with ``fp8=`` against the fake read server, over host-memory device
files with a context that emulates both entries with the integer reference of ``tests/test_fp8_quant_reference_cpu.py``
(asserting their argument rules).  Results are compared with ``reference_block_scales`` / ``reference_quant`` of the
whole weight."""
import asyncio
import ctypes
import json
import math
import os
import re

import numpy as np
import pytest
import torch
from safetensors.torch import save as st_save

from modal_client_b200 import _lib, device_file, volume
from tests.test_fp8_quant_reference_cpu import (F32_INF, FLOOR, INV_448, _widen_abs, f32_mul, reference_block_scales,
                                                reference_multiplier, reference_quant)
from tests.test_stage_ranges_cpu import range_pieces
from tests.test_volume_read_cast_cpu import _BY_CODE, _float
from tests.test_volume_read_cpu import BS, _LoadHostSegments, read_backend, volume_with  # noqa: F401
from tests.test_volume_read_fp8_cpu import ScaledContext

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16, F16, F32, E4M3 = torch.bfloat16, torch.float16, torch.float32, torch.float8_e4m3fn


def _u32(ptr: int, n: int) -> np.ndarray:
    return np.ctypeslib.as_array((ctypes.c_uint32 * n).from_address(ptr)) if n else np.zeros(0, np.uint32)


class QuantContext(ScaledContext):
    """Plus ``fp8_amax_boxes_from_host`` and ``copy_quant_boxes_from_host``: every argument rule of the entries
    asserted, a max-reduced over the bits of |x| and the elements quantized with the integer reference, and a log of
    the boxes of every call."""

    def _quant_elements(self, seg_ptrs, seg_lens, file_first_seg, boxes, src):
        """Per non-empty box: (destination address, element bits, src dtype, a array, block index of each element)."""
        out, written = [], []
        self.src_base = src.ctypes.data
        for f, off, width, rows, at, pitch, st, dt, ap, count, first, R, C, br, bc in boxes:
            assert st in _BY_CODE and dt == _lib.DT_F8E4M3
            assert R >= 1 and C >= 1 and br >= 1 and bc >= 1 and math.ceil(R / br) * math.ceil(C / bc) <= count
            assert ap % 4 == 0 and ap
            assert f < len(file_first_seg) - 1
            sd = _BY_CODE[st]
            ss = sd.itemsize
            assert width % ss == 0 and pitch % ss == 0
            assert (src.ctypes.data + at) % ss == 0, "a row's source is not element-aligned"
            if width * rows == 0:
                continue
            assert rows == 1 or pitch >= width
            assert at + (rows - 1) * pitch + width <= src.size
            assert first + ((rows - 1) * pitch + width) // ss <= R * C
            n = rows * width // ss
            pieces = range_pieces(seg_ptrs, seg_lens, file_first_seg, f, off, n)
            assert len(pieces) == 1, "a quantizing box's destination crosses a segment edge"
            raw = b"".join(src[at + r * pitch : at + r * pitch + width].tobytes() for r in range(rows))
            bits = torch.frombuffer(bytearray(raw), dtype=sd).view(torch.int16 if ss == 2 else torch.int32)
            bits = bits.to(torch.int64) & ((1 << (8 * ss)) - 1)
            e = torch.tensor([first + (r * pitch + c) // ss for r in range(rows) for c in range(0, width, ss)])
            brc, bcc = min(br, R), min(bc, C)
            key = (e // C // brc) * math.ceil(C / bcc) + (e % C) // bcc
            out.append((pieces[0][0], bits, sd, _u32(ap, count), key))
            written.append((pieces[0][0], pieces[0][0] + n))
        written.sort()
        assert all(a[1] <= b[0] for a, b in zip(written, written[1:])), "two boxes write the same device bytes"
        return out

    def fp8_amax_boxes_from_host(self, seg_ptrs, seg_lens, file_first_seg, boxes, src, stream=0):
        self.calls.append(("fp8_amax_boxes_from_host", [tuple(b) for b in boxes]))
        for _, bits, sd, a, key in self._quant_elements(seg_ptrs, seg_lens, file_first_seg, boxes, src):
            np.maximum.at(a, key.numpy(), _widen_abs(bits, sd).numpy().astype(np.uint32))

    def copy_quant_boxes_from_host(self, seg_ptrs, seg_lens, file_first_seg, boxes, bands, src, stream=0):
        self.calls.append(("copy_quant_boxes_from_host", [tuple(b) for b in boxes], [tuple(b) for b in bands]))
        elements = self._quant_elements(seg_ptrs, seg_lens, file_first_seg, boxes, src)
        for ap, sp, count in bands:
            assert count >= 1 and ap % 4 == 0 and sp % 4 == 0
            a, s = _u32(ap, count), _u32(sp, count)
            top = torch.from_numpy(a.astype(np.int64))
            fin = torch.where(top > F32_INF, top, torch.clamp(top, min=FLOOR))
            a[:] = fin.numpy().astype(np.uint32)
            s[:] = f32_mul(fin, torch.full_like(fin, INV_448)).numpy().astype(np.uint32)
        for p, bits, sd, a, key in elements:
            m = reference_multiplier(torch.from_numpy(a.astype(np.int64))[key])
            q = reference_quant(bits, sd, m).to(torch.uint8).numpy().tobytes()
            ctypes.memmove(p, q, len(q))


@pytest.fixture
def quant_backend(monkeypatch, read_backend):  # noqa: F811
    from modal_client_b200 import _backend

    ctx = QuantContext()
    monkeypatch.setattr(_backend, "_override", ctx)
    return ctx


def reference(w: torch.Tensor, block):
    """(E4M3 tensor, F32 scale tensor) of weight w in ``block``: the integer reference over the whole weight."""
    R, C = w.shape
    ss = w.element_size()
    bits = w.contiguous().view(torch.int16 if ss == 2 else torch.int32).to(torch.int64) & ((1 << (8 * ss)) - 1)
    a, s = reference_block_scales(bits.reshape(-1), w.dtype, R, C, block)
    br, bc = min(block[0] or R, R), min(block[1] or C, C)
    full = a.repeat_interleave(br, 0)[:R].repeat_interleave(bc, 1)[:, :C]
    q = reference_quant(bits.reshape(R, C), w.dtype, reference_multiplier(full))
    return q.to(torch.uint8).view(E4M3), s.to(torch.int32).view(torch.float32)


def _same_bits(got: dict, want: dict):
    assert list(got) == list(want)
    for k in want:
        assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, k
        assert torch.equal(got[k].contiguous().view(torch.uint8), want[k].contiguous().view(torch.uint8)), k


def _weights(seed: int):
    """A Llama-shaped state dict: F32, F16 and BF16 weights with sides that are not multiples of 128 (and a column
    count that leaves rows at odd phases), with NaN, inf, -0 and all-zero blocks planted; a norm and a bias."""
    g = torch.Generator().manual_seed(seed)
    sd = {"embed": _float((37, 20), BF16, g)}
    for k, (dt, R, C) in enumerate(((BF16, 300, 259), (F16, 200, 131), (F32, 130, 141), (BF16, 129, 3))):
        w = _float((R, C), dt, g)
        if k == 0:
            w[0, 0], w[140, 200], w[260:, :128] = float("nan"), float("-inf"), 0.0
            w[5, 7] = -0.0
        sd[f"layers.{k}.proj.weight"] = w
        sd[f"layers.{k}.norm"] = _float((C,), F32, g)
    return sd


NAMES = [f"layers.{k}.proj.weight" for k in range(4)]
BLOCKS = {"b128": (128, 128), "chan": (1, None), "tensor": (None, None), "b64x96": (64, 96)}


def _in_data_order(data: bytes, sd: dict) -> dict:
    n = int.from_bytes(data[:8], "little")
    _, entries = volume._safetensors_entries(data[8 : 8 + n], len(data) - 8 - n)
    return {e[0]: sd[e[0]] for e in entries}


def _want(sd, names, block, dtype=None, suffix="_scale_inv", data=None):
    out = {}
    for n, t in (_in_data_order(data, sd) if data is not None else sd).items():
        if n in names:
            out[n], out[n + suffix] = reference(t, block)
        else:
            out[n] = t.to(dtype) if dtype is not None and t.dtype in (F32, F16, BF16) else t
    return out


def _run(coro):
    return asyncio.run(coro)


# ------------------------------------------------------------------------------------------------ C ABI


def test_quant_box_entries_are_declared_exported_and_reject_a_null_context():
    header = open(os.path.join(ROOT, "include", "b200hash.h")).read()
    assert re.search(r"\bint b200h_fp8_amax_boxes_from_host\(b200h_ctx\* ctx, const b200h_segment\* segs,", header)
    assert re.search(r"\bint b200h_copy_quant_boxes_from_host\(b200h_ctx\* ctx, const b200h_segment\* segs,", header)
    struct = header.split("typedef struct b200h_quant_box {")[1].split("}")[0]
    # the 15 eight-byte words _lib passes: the cast box (8), then these 7 in this order
    assert re.findall(r"(\w+)[,;]", struct) == ["cast", "d_amax", "scale_count", "first_elem", "rows_total", "cols",
                                                "block_rows", "block_cols"]
    band = header.split("typedef struct b200h_fp8_band {")[1].split("}")[0]
    assert re.findall(r"(\w+)[,;]", band) == ["d_amax", "d_scales", "count"]
    for name in ("b200h_fp8_amax_boxes_from_host", "b200h_copy_quant_boxes_from_host"):
        assert name in _lib.ABI_SYMBOLS
    L = _lib.load_library()
    first = (ctypes.c_uint64 * 1)(0)
    assert L.b200h_fp8_amax_boxes_from_host(None, None, 0, first, 0, None, 0, None, 0, None) == -1
    assert L.b200h_copy_quant_boxes_from_host(None, None, 0, first, 0, None, 0, None, 0, None, 0, None) == -1
    import modal_client_b200

    for name in ("load_fp8_amax_boxes", "load_quant_boxes"):
        assert getattr(modal_client_b200, name) is getattr(device_file, name)
        assert name in device_file.__all__


def test_quant_box_wrappers_reject_malformed_boxes_and_bands():
    a = torch.zeros(4)
    src = np.zeros(16, np.uint8)
    with pytest.raises(ValueError, match="a box is"):
        device_file.load_fp8_amax_boxes([], [(0, 0, 4, 1, 0, 4, BF16, a)], src, ctx=object())
    good = (0, 0, 4, 1, 0, 4, BF16, a, 0, 1, 2, 128, 128)
    for k, bad, msg in ((6, E4M3, "quantizing boxes take"), (6, torch.float64, "quantizing boxes take"),
                        (7, torch.zeros(4, dtype=torch.int32), "amax"), (7, torch.zeros(4, 2).t(), "amax"),
                        (7, "a", "amax")):
        box = list(good)
        box[k] = bad
        for call in (lambda b: device_file.load_fp8_amax_boxes([], [b], src, ctx=object()),
                     lambda b: device_file.load_quant_boxes([], [b], [], src, ctx=object())):
            with pytest.raises(ValueError, match=msg):
                call(tuple(box))
    for band, msg in (((a, a, 0), "a band is"), ((a, torch.zeros(4, dtype=F16), 0, 1), "scales"),
                      ((a, a, 3, 2), "reaches past"), ((a, a, -1, 1), "reaches past")):
        with pytest.raises(ValueError, match=msg):
            device_file.load_quant_boxes([], [good], [band], src, ctx=object())


# ------------------------------------------------------------------------------------------------ reads


@pytest.mark.parametrize("block", list(BLOCKS.values()), ids=list(BLOCKS))
def test_read_safetensors_fp8_equals_the_integer_reference(quant_backend, block):
    sd = _weights(1)
    data = st_save(sd)

    async def go():
        async with volume_with({"m.safetensors": data}) as (client, _, _):
            return await volume.read_safetensors(client, "vo-r", "m.safetensors", fp8=NAMES, scale_block=block,
                                                 dtype=BF16, staging_bytes=96 * BS)

    _same_bits(_run(go()), _want(sd, NAMES, block, BF16, data=data))


@pytest.mark.parametrize("extra", [0, 1, 3])
@pytest.mark.parametrize("block", [(128, 128), (64, 96), (1, None)], ids=["b128", "b64x96", "chan"])
def test_bands_that_straddle_waves_and_both_halves_stay_exact(quant_backend, block, extra):
    """With a few blocks of staging (a band's blocks, less one, plus ``extra`` per half), bands start in one wave and
    end in the next, in either half."""
    g = torch.Generator().manual_seed(7)
    sd = {"pad": _float((5,), BF16, g), "w": _float((600, 70), BF16, g), "v": _float((300, 33), F32, g),
          "u": _float((390, 17), F16, g)}
    band = max(min(block[0] or 10**9, t.shape[0]) * t.shape[1] * t.element_size() for n, t in sd.items() if n != "pad")
    staging = 2 * (band // BS + 1 + extra)
    data = st_save(sd)
    carried = []
    real = volume._load_in_waves

    async def spy(slices, load, *args):
        def counted(*a):
            got = load(*a)
            carried.append(isinstance(got, tuple))
            return got

        await real(slices, counted, *args)

    volume._load_in_waves = spy
    try:
        async def go():
            async with volume_with({"m.safetensors": data}) as (client, _, _):
                return await volume.read_safetensors(client, "vo-r", "m.safetensors", fp8=["w", "v", "u"],
                                                     scale_block=block, staging_bytes=staging * BS)

        got = _run(go())
    finally:
        volume._load_in_waves = real
    _same_bits(got, _want(sd, ["w", "v", "u"], block, data=data))
    assert any(carried) and len(carried) >= 4


def test_sharded_fp8_equals_the_reference_and_fetches_the_plain_blocks_once(quant_backend, monkeypatch):
    sd = _weights(3)
    names = list(sd)
    files = {"m-1.safetensors": st_save({n: sd[n] for n in names[:5]}),
             "m-2.safetensors": st_save({n: sd[n] for n in names[5:]})}
    index = {"metadata": {}, "weight_map": {n: "m-1.safetensors" if i < 5 else "m-2.safetensors"
                                            for i, n in enumerate(names)}}
    files["m.safetensors.index.json"] = json.dumps(index).encode()
    fetched = []
    real = volume._load_in_waves

    async def spy(slices, load, *args):
        fetched.append(sorted((i, off) for _, off, _, i in slices))
        await real(slices, load, *args)

    monkeypatch.setattr(volume, "_load_in_waves", spy)

    async def go(**kw):
        async with volume_with(files) as (client, _, _):
            return await volume.read_safetensors_sharded(client, "vo-r", "m.safetensors.index.json",
                                                         staging_bytes=40 * BS, **kw)

    got = _run(go(fp8=NAMES, dtype=F32))
    plain = _run(go(dtype=F32))
    want = {}
    for f in ("m-1.safetensors", "m-2.safetensors"):
        part = {n: sd[n] for n, s in index["weight_map"].items() if s == f}
        want.update(_want(part, NAMES, (128, 128), F32, data=files[f]))
    _same_bits(got, want)
    assert set(plain) | {n + "_scale_inv" for n in NAMES} == set(got)
    assert len(fetched) == 2 and fetched[0] == fetched[1] and len(set(fetched[0])) == len(fetched[0])


def test_each_wave_makes_a_fixed_number_of_calls_and_the_scales_follow_their_weights(quant_backend, monkeypatch):
    sd = _weights(4)
    data = st_save(sd)
    waves = []
    real = volume._load_in_waves

    async def spy(slices, load, *args):
        def counted(wave, at, buf, ctx):
            before = len(ctx.calls)
            got = load(wave, at, buf, ctx)
            waves.append([c[0] for c in ctx.calls[before:]])
            return got

        await real(slices, counted, *args)

    monkeypatch.setattr(volume, "_load_in_waves", spy)

    async def go():
        async with volume_with({"m.safetensors": data}) as (client, _, _):
            return await volume.read_safetensors(client, "vo-r", "m.safetensors", fp8=NAMES, dtype=F16,
                                                 staging_bytes=40 * BS)

    got = _run(go())
    assert len(waves) > 3
    for w in waves:
        assert len(w) == len(set(w)) <= 4
        assert set(w) <= {"copy_boxes_from_host", "copy_cast_boxes_from_host", "fp8_amax_boxes_from_host",
                          "copy_quant_boxes_from_host"}
    keys = list(got)
    for n in NAMES:
        assert keys[keys.index(n) + 1] == n + "_scale_inv"


def test_a_half_read_by_a_carried_band_is_refilled_only_after_that_copy(quant_backend, monkeypatch):
    """Every block GET into a staging slot comes after the wait for every earlier copy that read that slot."""
    g = torch.Generator().manual_seed(5)
    sd = {"a": _float((3,), BF16, g), "w": _float((900, 50), BF16, g), "v": _float((197, 41), F32, g)}
    data = st_save(sd)
    log = _LoadHostSegments.log
    real_fetch = volume._fetch_block

    async def fetch(url, out, want, semaphore):
        log.append(("fill", out.ctypes.data, out.ctypes.data + want))
        await real_fetch(url, out, want, semaphore)

    monkeypatch.setattr(volume, "_fetch_block", fetch)

    async def go():
        async with volume_with({"m.safetensors": data}) as (client, _, _):
            return await volume.read_safetensors(client, "vo-r", "m.safetensors", fp8=["w", "v"],
                                                 staging_bytes=12 * BS)

    got = _run(go())
    _same_bits(got, _want(sd, ["w", "v"], (128, 128), data=data))
    kinds = ("copy_boxes_from_host", "copy_cast_boxes_from_host", "fp8_amax_boxes_from_host",
             "copy_quant_boxes_from_host")
    calls = [c for c in quant_backend.calls if c[0] in kinds]
    copies = [e for e in log if e[0] == "copy"]
    assert len(copies) == len(calls)
    # the staging bytes each copy read: boxes are (file, offset, width, rows, src_offset, src_pitch, ...)
    base = quant_backend.src_base
    reads = [[(b[4], b[4] + (b[3] - 1) * b[5] + b[2]) for b in c[1]] for c in calls]
    waited, read_by = -1, []  # every copy is on one stream: the wait for copy k is a wait for every copy before it
    for e in log:
        if e[0] == "copy":
            read_by.append(e[1])
        elif e[0] == "wait":
            waited = max(waited, e[1])
        elif e[0] == "fill" and read_by:
            for k in read_by:
                if k <= waited:
                    continue
                for lo, hi in reads[k]:
                    assert not (e[1] < base + hi and base + lo < e[2]), f"slot refilled before copy {k} was waited for"
    assert any(c[0] == "copy_quant_boxes_from_host" and any(b[4] for b in c[1]) for c in calls)


def test_every_refusal_comes_in_one_error_before_any_data_get(quant_backend, monkeypatch):
    g = torch.Generator().manual_seed(6)
    sd = {"w": _float((300, 400), BF16, g), "v": _float((4, 4, 4), F32, g), "i": torch.arange(6, dtype=torch.int32),
          "e": torch.zeros((0, 5), dtype=F16), "w_scale_inv": torch.ones(3, 4), "x": _float((8, 8), F16, g),
          "f8": torch.zeros((4, 4), dtype=E4M3)}
    data = st_save(sd)
    runs = []

    async def no_runs(*a, **k):
        runs.append(a)

    monkeypatch.setattr(volume, "_load_runs", no_runs)

    async def go(path="m.safetensors", **kw):
        async with volume_with({"m.safetensors": data}) as (client, _, _):
            return await volume.read_safetensors(client, "vo-r", path, **kw)

    with pytest.raises(ValueError) as exc:
        _run(go(fp8=["w", "v", "i", "e", "nope", "x", "x", "f8"], dtype={"x": F32}, staging_bytes=4 * BS))
    msg = str(exc.value)
    for part in ("'w_scale_inv', is already a tensor", "'v' has shape [4, 4, 4]", "'i' has shape [6]", "'e' has shape [0, 5]",
                 "'nope' is in fp8 but not in the file", "'x' is in fp8 twice", "'x' is in both fp8 and dtype",
                 "'f8' is F8_E4M3", "'w': one band of 128 rows"):
        assert part in msg, part
    assert "staging_bytes=" in msg.split("'w': one band")[1]
    with pytest.raises(ValueError, match="fp8 cannot be combined with scales"):
        _run(go(fp8=["x"], scales={"f8": "w_scale_inv"}, dtype=BF16))
    with pytest.raises(ValueError, match="must be an iterable"):
        _run(go(fp8=3))
    with pytest.raises(ValueError, match="scale_block"):
        _run(go(fp8=["x"], scale_block=(0, 4)))
    with pytest.raises(ValueError, match="read_safetensors\\(into=...\\)"):
        _run(go(fp8=["x"], into={"x": torch.empty(8, 8, dtype=E4M3)}))
    with pytest.raises(ValueError) as exc:  # an fp8 problem and an into= mismatch, in one error
        _run(go(fp8=["nope", "x"], into={"x": torch.empty(8, 8, dtype=F16)}))
    msg = str(exc.value)
    for part in ("'nope' is in fp8 but not in the file", "read_safetensors(into=...)", "'x': the file holds",
                 "'x_scale_inv' is in the file but not in into"):
        assert part in msg, part
    assert runs == []
    with pytest.raises(TypeError):
        _run(volume.read_safetensors_slices(None, "vo-r", "m.safetensors", {"x": ...}, fp8=["x"]))


def test_sharded_fp8_refuses_select(quant_backend):
    sd = {"x": _float((8, 8), F16, torch.Generator().manual_seed(1))}
    files = {"a.safetensors": st_save(sd),
             "i.json": json.dumps({"weight_map": {"x": "a.safetensors"}}).encode()}

    async def go():
        async with volume_with(files) as (client, _, _):
            return await volume.read_safetensors_sharded(client, "vo-r", "i.json", fp8=["x"], select={"x": ...})

    with pytest.raises(ValueError, match="fp8 does not take select="):
        _run(go())


def test_into_fills_fp8_weights_and_scales_in_place(quant_backend):
    sd = _weights(8)
    data = st_save(sd)
    want = _want(sd, NAMES, (1, None), data=data)
    into = {n: torch.empty_like(t) for n, t in want.items()}

    async def go():
        async with volume_with({"m.safetensors": data}) as (client, _, _):
            return await volume.read_safetensors(client, "vo-r", "m.safetensors", fp8=NAMES, scale_block=(1, None),
                                                 into=into, scale_suffix="_scale_inv")

    got = _run(go())
    _same_bits(got, want)
    assert all(got[n] is into[n] for n in want)


def test_without_fp8_the_calls_are_those_of_today(quant_backend):
    sd = _weights(9)
    data = st_save(sd)

    async def go(**kw):
        async with volume_with({"m.safetensors": data}) as (client, _, _):
            before = len(quant_backend.calls)
            out = await volume.read_safetensors(client, "vo-r", "m.safetensors", staging_bytes=8 * BS, **kw)
            return out, quant_backend.calls[before:]

    for kw in ({}, {"dtype": BF16}):
        a, calls_a = _run(go(**kw))
        b, calls_b = _run(go(fp8=None, **kw))
        _same_bits(a, b)
        assert calls_a == calls_b
        assert not any(c[0] in ("fp8_amax_boxes_from_host", "copy_quant_boxes_from_host") for c in calls_a)
