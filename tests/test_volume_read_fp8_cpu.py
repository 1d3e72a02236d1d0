"""FP8 safetensors weights read from a volume and dequantized with their block scales as they land, on the CPU: the C
ABI of ``b200h_copy_scaled_boxes_from_host``, ``fp8_scales``, and ``read_safetensors`` / ``read_safetensors_slices`` /
``read_safetensors_sharded`` with ``scales=`` against the fake read server, over host-memory device files with a
context whose ``copy_scaled_boxes_from_host`` asserts the entry's argument rules and dequantizes with torch on the host.
Results are compared with torch's CPU dequantization of the full tensor, ``(W.float() * S_expanded).to(dtype)``."""
import asyncio
import ctypes
import json
import math
import os
import re

import numpy as np
import pytest
import torch
from safetensors.torch import load as st_load
from safetensors.torch import save as st_save

from modal_client_b200 import _lib, device_file, volume
from tests.test_stage_ranges_cpu import range_pieces
from tests.test_volume_read_cast_cpu import _BY_CODE, CastContext, _float, _padded
from tests.test_volume_read_cpu import BS, read_backend, volume_with  # noqa: F401
from tests.test_volume_read_slices_cpu import _same, _tensor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
_FP8 = {_lib.DT_F8E4M3: E4M3, _lib.DT_F8E5M2: E5M2}


def dequant(w: torch.Tensor, s: torch.Tensor, block, dtype) -> torch.Tensor:
    """The reference: ``(W.float() * S_expanded).to(dtype)``, ``block`` entries None for the whole dimension."""
    R, C = w.shape
    br, bc = (R if block[0] is None else block[0]), (C if block[1] is None else block[1])
    sr, sc = (1 if block[0] is None else -(-R // br)), (1 if block[1] is None else -(-C // bc))
    full = s.float().reshape(sr, sc).repeat_interleave(max(br, 1), 0)[:R].repeat_interleave(max(bc, 1), 1)[:, :C]
    return (w.float() * full).to(dtype)


class ScaledContext(CastContext):
    """Plus ``copy_scaled_boxes_from_host``: every argument rule of the entry asserted, the elements dequantized with
    torch on the host, and a log of the boxes of every call."""

    def copy_scaled_boxes_from_host(self, seg_ptrs, seg_lens, file_first_seg, boxes, src, stream=0):
        self.calls.append(("copy_scaled_boxes_from_host", [tuple(b) for b in boxes]))
        written = []
        for f, off, width, rows, at, pitch, st, dt, sp, stype, count, first, R, C, br, bc in boxes:
            assert st in _FP8 and dt in _BY_CODE and stype in _BY_CODE
            assert br >= 1 and bc >= 1 and math.ceil(R / br) * math.ceil(C / bc) <= count
            assert f < len(file_first_seg) - 1
            if width * rows == 0:
                continue
            assert rows == 1 or pitch >= width
            assert at + (rows - 1) * pitch + width <= src.size
            assert first + (rows - 1) * pitch + width <= R * C
            ds = _BY_CODE[dt].itemsize
            n = rows * width * ds
            pieces = range_pieces(seg_ptrs, seg_lens, file_first_seg, f, off, n)
            assert len(pieces) == 1, "a scaled box's destination crosses a segment edge"
            p = pieces[0][0]
            assert p % ds == 0
            raw = b"".join(src[at + r * pitch : at + r * pitch + width].tobytes() for r in range(rows))
            q = torch.frombuffer(bytearray(raw), dtype=_FP8[st]).float()
            es = _BY_CODE[stype].itemsize
            scales = torch.frombuffer(bytearray(ctypes.string_at(sp, count * es)), dtype=_BY_CODE[stype]).float()
            e = torch.tensor([first + r * pitch + c for r in range(rows) for c in range(width)], dtype=torch.int64)
            i, j = e // C, e % C
            out = (q * scales[(i // br) * math.ceil(C / bc) + j // bc]).to(_BY_CODE[dt])
            ctypes.memmove(p, out.view(torch.uint8).numpy().tobytes(), n)
            written.append((p, p + n))
        written.sort()
        assert all(a[1] <= b[0] for a, b in zip(written, written[1:])), "two boxes write the same device bytes"


@pytest.fixture
def fp8_backend(monkeypatch, read_backend):  # noqa: F811
    from modal_client_b200 import _backend

    ctx = ScaledContext()
    monkeypatch.setattr(_backend, "_override", ctx)
    return ctx


@pytest.fixture
def passes(monkeypatch):
    """Per ``_load_runs`` pass: the data calls ((path, start)), the blocks it fetched ({(path, block)}) and the entry
    points each of its waves called."""
    out = []
    real_slices, real_waves = volume._block_slices, volume._load_in_waves
    pending = []

    async def slices_spy(client, volume_id, path, start, n):
        pending.append((path, start))
        return await real_slices(client, volume_id, path, start, n)

    async def waves_spy(slices, load, *args):
        files = pending[len(pending) - 1 - max(i for *_, i in slices) :]  # the data calls come last
        pending.clear()
        blocks = [(files[i][0], (files[i][1] + off) // BS) for _, off, _, i in slices]
        rec = {"files": files, "blocks": blocks, "waves": []}
        out.append(rec)

        def counted(wave, at, buf, ctx):
            before = len(ctx.calls)
            loaded = load(wave, at, buf, ctx)
            rec["waves"].append([c[0] for c in ctx.calls[before:]])
            return loaded

        await real_waves(slices, counted, *args)

    monkeypatch.setattr(volume, "_block_slices", slices_spy)
    monkeypatch.setattr(volume, "_load_in_waves", waves_spy)
    return out


def _fp8(shape, dtype, g):
    """Random FP8 bit patterns without NaNs (torch's CPU casts and the device differ only in NaN bits)."""
    t = _tensor(shape, dtype, g)
    bits = t.view(torch.uint8)
    return torch.where(t.float().isnan(), torch.zeros_like(bits), bits).view(dtype)


def _scale(shape, dtype, g):
    return (torch.rand(shape, generator=g) * 2.0 ** torch.randint(-12, 4, shape, generator=g).float()).to(dtype)


BLOCKS = {"b128": (128, 128), "chan": (1, None), "tensor": (None, None), "b64x32": (64, 32)}


def _checkpoint(seed: int):
    """A DeepSeek-shaped state dict: FP8 weights whose sides are not multiples of 128, with scales for every block
    form, F32 and BF16 scales, E4M3 and E5M2, plus a norm and a bias.  -> (state dict, {weight: (scale, block)})"""
    g = torch.Generator().manual_seed(seed)
    sd, meta = {}, {}
    for k, (name, block) in enumerate(BLOCKS.items()):
        for fmt, sdt in ((E4M3, F32), (E5M2, BF16)):
            R, C = 300 - 37 * k, 200 + 11 * k
            w = f"layers.{name}.{str(fmt).split('_')[-1]}.weight"
            sd[w] = _fp8((R, C), fmt, g)
            sr = 1 if block[0] is None else -(-R // block[0])
            sc = 1 if block[1] is None else -(-C // block[1])
            shape = (sr, sc) if block != (None, None) else ()
            if block == (1, None):
                shape = (sr,)
            sd[w + "_scale_inv"] = _scale(shape, sdt, g)
            meta[w] = (w + "_scale_inv", block)
    sd["norm.weight"] = _float((300,), BF16, g)
    sd["bias"] = _float((77,), F32, g)
    return sd, meta


def _want(full, meta, block, dtype, names=None):
    out = {}
    for name, t in full.items():
        if name.endswith("_scale_inv") or (names is not None and name not in names):
            continue
        if name in meta:
            out[name] = dequant(t, full[meta[name][0]], block, dtype)
        else:
            out[name] = t.to(dtype) if t.dtype in (F32, F16, BF16) else t
    return out


# ------------------------------------------------------------------------------------------------ C ABI


def test_copy_scaled_boxes_from_host_is_declared_exported_and_rejects_a_null_context():
    header = open(os.path.join(ROOT, "include", "b200hash.h")).read()
    assert re.search(r"\bint b200h_copy_scaled_boxes_from_host\(b200h_ctx\* ctx, const b200h_segment\* segs,", header)
    assert re.search(r"typedef struct b200h_scaled_box \{\s*b200h_cast_box cast;\s*const void\* d_scales;", header)
    assert re.search(rf"#define B200H_DT_F8E4M3 {_lib.DT_F8E4M3}u\b", header)
    assert re.search(rf"#define B200H_DT_F8E5M2 {_lib.DT_F8E5M2}u\b", header)
    struct = header.split("typedef struct b200h_scaled_box {")[1].split("}")[0]
    # the 16 eight-byte words _lib passes: the cast box (8), then these 8 in this order
    fields = re.findall(r"(\w+)[,;]", struct)
    assert fields == ["cast", "d_scales", "scale_type", "scale_count", "first_elem", "rows_total", "cols", "block_rows",
                      "block_cols"]
    assert "b200h_copy_scaled_boxes_from_host" in _lib.ABI_SYMBOLS
    L = _lib.load_library()
    first = (ctypes.c_uint64 * 1)(0)
    assert L.b200h_copy_scaled_boxes_from_host(None, None, 0, first, 0, None, 0, None, 0, None) == -1
    import modal_client_b200

    assert modal_client_b200.load_scaled_boxes is device_file.load_scaled_boxes
    assert "load_scaled_boxes" in device_file.__all__


def test_load_scaled_boxes_rejects_malformed_boxes():
    s = torch.ones(4)
    with pytest.raises(ValueError, match="a box is"):
        device_file.load_scaled_boxes([], [(0, 0, 4, 1, 0, 4, E4M3, BF16)], np.zeros(16, np.uint8), ctx=object())
    good = (0, 0, 4, 1, 0, 4, E4M3, BF16, s, 0, 1, 4, 128, 128)
    for k, bad, msg in ((6, F16, "dequantizes"), (7, torch.float64, "converts to"), (8, torch.ones(4, dtype=torch.int32), "scales"),
                        (8, torch.ones(4, 2).t(), "scales"), (8, "s", "scales")):
        box = list(good)
        box[k] = bad
        with pytest.raises(ValueError, match=msg):
            device_file.load_scaled_boxes([], [tuple(box)], np.zeros(16, np.uint8), ctx=object())


def test_fp8_scales_pairs_every_name_with_its_suffixed_twin():
    names = ["a.weight", "a.weight_scale_inv", "b.weight", "c.weight_scale_inv", "d.weight", "d.weight_scale",
             "e.weight_scale_inv_scale_inv", "e.weight_scale_inv"]
    assert volume.fp8_scales(names) == {"a.weight": "a.weight_scale_inv",
                                        "e.weight_scale_inv": "e.weight_scale_inv_scale_inv"}
    assert volume.fp8_scales({n: None for n in names}, suffix="_scale") == {"d.weight": "d.weight_scale"}
    assert list(volume.fp8_scales(reversed(names))) == ["e.weight_scale_inv", "a.weight"]
    assert volume.fp8_scales([]) == {}


# -------------------------------------------------------------------------------------------------- parity


@pytest.mark.parametrize("pad", [0, 8])
@pytest.mark.parametrize("block", list(BLOCKS))
def test_read_safetensors_dequantizes_every_weight_as_torch_does(fp8_backend, passes, block, pad):
    sd, meta = _checkpoint(1)
    # keep the weights whose scales fit this block; the others are left out of the file
    sd = {k: v for k, v in sd.items() if not k.startswith("layers.") or f".{block}." in k}
    image = _padded(st_save(sd), pad)
    full = st_load(image)
    scales = volume.fp8_scales(full)
    assert len(scales) == 2

    async def run():
        async with volume_with({"/m": image}) as (client, _, _):
            for dtype in (BF16, F16, F32):
                got = await volume.read_safetensors(client, "vo-r", "/m", dtype=dtype, scales=scales,
                                                    scale_block=BLOCKS[block], staging_bytes=2 * BS)
                want = _want(full, meta, BLOCKS[block], dtype)
                assert sorted(got) == sorted(want)  # scales consumed
                for name, t in want.items():
                    _same(got[name], t, (dtype, name))
            mapping = {w: (BF16, F32)[k] for k, w in enumerate(scales)}
            got = await volume.read_safetensors(client, "vo-r", "/m", dtype=mapping, scales=scales,
                                                scale_block=BLOCKS[block], staging_bytes=4 * BS)
            for w, dt in mapping.items():
                _same(got[w], dequant(full[w], full[scales[w]], BLOCKS[block], dt), w)
            _same(got["norm.weight"], full["norm.weight"])  # not in the mapping: as stored

    asyncio.run(run())


@pytest.mark.parametrize("block", list(BLOCKS))
def test_tp_slices_equal_the_slices_of_the_dequantized_weight(fp8_backend, block):
    sd, meta = _checkpoint(2)
    sd = {k: v for k, v in sd.items() if not k.startswith("layers.") or f".{block}." in k}
    image = st_save(sd)
    full = st_load(image)
    scales = volume.fp8_scales(full)

    async def run():
        async with volume_with({"/m": image}) as (client, _, _):
            for index in [(slice(3, 131),), (slice(None), slice(17, 163)), (slice(129, 257), slice(1, 130)), 5,
                          (slice(None), 131), (slice(250, None),), (slice(0, 0),), ...]:
                select = {w: index for w in scales}
                select["bias"] = slice(3, 40)
                got = await volume.read_safetensors_slices(client, "vo-r", "/m", select, dtype=BF16, scales=scales,
                                                           scale_block=BLOCKS[block], staging_bytes=2 * BS)
                assert list(got) == list(select)
                for w in scales:
                    _same(got[w], dequant(full[w], full[scales[w]], BLOCKS[block], BF16)[index], (w, index))
                _same(got["bias"], full["bias"][3:40].to(BF16))

    asyncio.run(run())


def _sharded(sd: dict, split):
    """Files of a sharded checkpoint: shard k holds the names ``split`` maps to k."""
    files, weight_map = {}, {}
    for k in sorted(set(split.values())):
        name = f"model-{k + 1:05d}-of-{len(set(split.values())):05d}.safetensors"
        files[f"/ckpt/{name}"] = st_save({n: t for n, t in sd.items() if split[n] == k})
        weight_map.update({n: name for n in sd if split[n] == k})
    files["/ckpt/model.safetensors.index.json"] = json.dumps({"metadata": {}, "weight_map": weight_map}).encode()
    return files


def test_sharded_reads_take_a_scale_from_another_shard(fp8_backend, passes):
    sd, meta = _checkpoint(3)
    names = list(sd)
    # every scale in a different shard from its weight; the second shard holds some weights and the first's scales
    split = {n: (names.index(n) // 2) % 2 if not n.endswith("_scale_inv") else 1 - (names.index(n[:-10]) // 2) % 2
             for n in names}
    files = _sharded(sd, split)
    index = "/ckpt/model.safetensors.index.json"

    async def run():
        async with volume_with(files) as (client, _, _):
            _, tensors = await volume.read_safetensors_index(client, "vo-r", index)
            scales = volume.fp8_scales(tensors)
            assert len(scales) == 8 and all(tensors[w][0] != tensors[s][0] for w, s in scales.items())
            by_block = {}
            for w in scales:
                by_block.setdefault(meta[w][1], []).append(w)
            for block, ws in by_block.items():
                sub = {w: scales[w] for w in ws}
                select = {w: (slice(7, 290), slice(3, 199)) for w in ws}
                got = await volume.read_safetensors_sharded(client, "vo-r", index, select=select, dtype=F16,
                                                            scales=sub, scale_block=block, staging_bytes=2 * BS)
                for w in ws:
                    _same(got[w], dequant(sd[w], sd[sub[w]], block, F16)[7:290, 3:199], (block, w))
            # whole: only the (128, 128) weights have scales of that block; the rest stay out of scales and select
            ws = by_block[(128, 128)]
            keep = {n: ... for n in tensors if n not in scales.values() and (n not in scales or n in ws)}
            got = await volume.read_safetensors_sharded(client, "vo-r", index, select=keep, dtype=BF16,
                                                        scales={w: scales[w] for w in ws}, staging_bytes=2 * BS)
            for w in ws:
                _same(got[w], dequant(sd[w], sd[scales[w]], (128, 128), BF16), w)
            _same(got["norm.weight"], sd["norm.weight"])
            _same(got["bias"], sd["bias"].to(BF16))
            # both passes: the scales' shards, then the weights' shards; each pass its blocks once
            p1, p2 = passes[-2], passes[-1]
            assert {p for p, _ in p1["files"]} == {"/ckpt/" + tensors[scales[w]][0].split("/")[-1] for w in ws}
            assert len(p1["blocks"]) == len(set(p1["blocks"])) and len(p2["blocks"]) == len(set(p2["blocks"]))

    asyncio.run(run())


def test_into_is_filled_in_place(fp8_backend):
    sd, meta = _checkpoint(4)
    sd = {k: v for k, v in sd.items() if not k.startswith("layers.") or ".b128." in k}
    image = st_save(sd)
    full = st_load(image)
    scales = volume.fp8_scales(full)

    async def run():
        async with volume_with({"/m": image}) as (client, _, faults):
            want = _want(full, meta, (128, 128), BF16)
            into = {k: torch.zeros_like(t) for k, t in want.items()}
            got = await volume.read_safetensors(client, "vo-r", "/m", into=into, dtype=BF16, scales=scales)
            for k in want:
                assert got[k] is into[k]
                _same(got[k], want[k], k)
            w = next(iter(scales))
            sl = {w: torch.zeros(100, 20, dtype=F32)}
            got = await volume.read_safetensors_slices(client, "vo-r", "/m", {w: (slice(100, 200), slice(120, 140))},
                                                       into=sl, dtype=F32, scales={w: scales[w]})
            _same(got[w], dequant(full[w], full[scales[w]], (128, 128), F32)[100:200, 120:140])
            gets = faults["gets"]
            with pytest.raises(ValueError) as err:
                await volume.read_safetensors_slices(client, "vo-r", "/m", {w: 0}, into={w: torch.zeros(3)},
                                                     dtype=F16, scales={w: scales[w]})
            assert f"'{w}': the slice is {full[w].dtype} [{full[w].shape[1]}], converted to torch.float16, " \
                   "into has torch.float32 [3]" in str(err.value)
            bad = dict(into, **{scales[w]: torch.zeros(3, 2)})
            with pytest.raises(ValueError, match="is in into, but scales are consumed"):
                await volume.read_safetensors(client, "vo-r", "/m", into=bad, dtype=BF16, scales=scales)
            assert faults["gets"] == gets + 4  # only the headers' reads

    asyncio.run(run())


# ---------------------------------------------------------------------------------------- requests and calls


def _blocks_of(spans):
    return {b for lo, n in spans if n for b in range(lo // BS, (lo + n - 1) // BS + 1)}


def test_both_passes_fetch_exactly_their_blocks_with_three_calls_at_most_per_wave(fp8_backend, passes):
    g = torch.Generator().manual_seed(5)
    sd = {"w1": _fp8((300, 250), E4M3, g), "w1_scale_inv": _scale((3, 2), F32, g),
          "w2": _fp8((130, 500), E5M2, g), "w2_scale_inv": _scale((2, 4), BF16, g),
          "b": _float((1001,), F32, g), "c": _tensor((700,), torch.int32, g), "n": _float((3000,), BF16, g)}
    image = st_save(sd)
    full = st_load(image)
    n = int.from_bytes(image[:8], "little")
    header = json.loads(image[8 : 8 + n])
    at = {k: (8 + n + v["data_offsets"][0], v["data_offsets"][1] - v["data_offsets"][0]) for k, v in header.items()
          if k != "__metadata__"}
    scales = volume.fp8_scales(full)

    async def run():
        async with volume_with({"/m": image}) as (client, stub, _):
            calls = len(stub.get_file_calls)
            got = await volume.read_safetensors(client, "vo-r", "/m", dtype=BF16, scales=scales, staging_bytes=2 * BS)
            for k, t in _want(full, {w: (s, (128, 128)) for w, s in scales.items()}, (128, 128), BF16).items():
                _same(got[k], t, k)
            p1, p2 = passes[-2:]
            reqs = [(r.start, r.len) for r in stub.get_file_calls[calls:]]
            assert len(reqs) == 3 + 2  # the header, then one data call per pass
            sc = [at[s] for s in scales.values()]
            rest = [v for k, v in at.items() if k not in scales.values()]
            assert reqs[3][0] == min(lo for lo, _ in sc) and reqs[4][0] == min(lo for lo, _ in rest)
            assert sorted(b for _, b in p1["blocks"]) == sorted(_blocks_of(sc))
            assert sorted(b for _, b in p2["blocks"]) == sorted(_blocks_of(rest))
            assert p1["waves"] and all(w == ["copy_boxes_from_host"] for w in p1["waves"])
            assert len(p2["waves"]) >= 3
            for w in p2["waves"]:
                for entry in ("copy_boxes_from_host", "copy_cast_boxes_from_host", "copy_scaled_boxes_from_host"):
                    assert w.count(entry) <= 1, p2["waves"]
            assert any(len(w) == 3 for w in p2["waves"]) or any("copy_scaled_boxes_from_host" in w for w in p2["waves"])
            # a slice fetches only the blocks its rows touch, and the whole scale
            calls = len(stub.get_file_calls)
            got = await volume.read_safetensors_slices(client, "vo-r", "/m", {"w1": (slice(None), slice(100, 140))},
                                                       dtype=F32, scales={"w1": "w1_scale_inv"}, staging_bytes=2 * BS)
            _same(got["w1"], dequant(full["w1"], full["w1_scale_inv"], (128, 128), F32)[:, 100:140])
            lo = at["w1"][0]
            assert sorted(b for _, b in passes[-2]["blocks"]) == sorted(_blocks_of([at["w1_scale_inv"]]))
            assert sorted(b for _, b in passes[-1]["blocks"]) == sorted(
                _blocks_of([(lo + r * 250 + 100, 40) for r in range(300)]))

    asyncio.run(run())


def test_without_scales_the_requests_and_calls_are_those_of_today(fp8_backend, passes):
    g = torch.Generator().manual_seed(6)
    sd = {"a": _float((30, 500), F32, g), "b": _tensor((77,), torch.int64, g), "c": _tensor((9, 9), BF16, g)}
    image = st_save(sd)

    async def run():
        async with volume_with({"/m": image}) as (client, stub, _):
            logs = []
            for kw in ({"dtype": BF16}, {"dtype": BF16, "scales": None}, {"dtype": BF16, "scales": {}}):
                for sliced in (False, True):
                    calls, nctx, npass = len(stub.get_file_calls), len(fp8_backend.calls), len(passes)
                    if sliced:
                        await volume.read_safetensors_slices(client, "vo-r", "/m", {"a": (slice(3, 9),), "b": 5},
                                                             staging_bytes=2 * BS, **kw)
                    else:
                        await volume.read_safetensors(client, "vo-r", "/m", staging_bytes=2 * BS, **kw)
                    logs.append((sliced, [(r.start, r.len) for r in stub.get_file_calls[calls:]],
                                 fp8_backend.calls[nctx:], passes[npass:]))
            for sliced in (False, True):
                same = [log[1:] for log in logs if log[0] == sliced]
                assert same[0] == same[1] == same[2]
                assert len(same[0][2]) == 1
                assert not any(c[0] == "copy_scaled_boxes_from_host" for c in same[0][1])

    asyncio.run(run())


# ------------------------------------------------------------------------------------------- rejections


def test_every_rejection_names_every_offender_before_any_data_get(fp8_backend):
    g = torch.Generator().manual_seed(7)
    sd = {"w": _fp8((300, 200), E4M3, g), "w_scale_inv": _scale((3, 2), F32, g),
          "v": _fp8((10, 20), E5M2, g), "v_scale_inv": _scale((1, 1), F32, g),
          "flat": _fp8((400,), E4M3, g), "flat_scale_inv": _scale((4,), F32, g),
          "bf": _float((8, 8), BF16, g), "bf_scale_inv": _scale((1, 1), F32, g),
          "i8s": _tensor((1, 1), torch.int8, g), "e": _fp8((3,), E4M3, g)}
    image = st_save(sd)
    W = {"w": "w_scale_inv"}
    cases = [
        (None, {}, W, (128, 128), ["scales needs dtype="]),
        (BF16, {}, W, (128, 0), ["scale_block (128, 0) is not a pair"]),
        (BF16, {}, W, (128,), ["scale_block (128,) is not a pair"]),
        (BF16, {}, W, (True, 128), ["is not a pair"]),
        (BF16, {}, {"nope": "w_scale_inv", "w": "gone"}, (128, 128),
         ["weight 'nope' is not in the file", "scale 'gone' of 'w' is not in the file"]),
        (BF16, {}, {"bf": "bf_scale_inv", "flat": "flat_scale_inv"}, (128, 128),
         ["weight 'bf' is BF16, not F8_E4M3", "weight 'flat' has shape [400], not 2-D"]),
        (BF16, {}, {"w": "e", "v": "i8s"}, (128, 128), ["scale 'e' is F8_E4M3, not F32", "scale 'i8s' is I8"]),
        (BF16, {}, W, (64, 64), ["scale 'w_scale_inv' has shape [3, 2]; weight 'w' of shape [300, 200] in blocks "
                                 "(64, 64) needs [5, 4]"]),
        (BF16, {}, {"w": "v", "v": "v_scale_inv"}, (128, 128), ["'v' is both a weight and a scale"]),
        ({"v": BF16, "v_scale_inv": F32}, {}, {"w": "w_scale_inv", "v": "v_scale_inv"}, (128, 128),
         ["'v_scale_inv' is a scale, which is consumed, but dtype names it", "weight 'w' has no target in dtype"]),
        (torch.int8, {}, W, (128, 128), ["weight 'w': torch.int8 is not a supported target"]),
        ({"w": torch.float64}, {}, W, (128, 128), ["weight 'w': torch.float64 is not a supported target"]),
        (BF16, {"w": 0, "w_scale_inv": ...}, W, (128, 128), ["scale 'w_scale_inv' is selected"]),
        (BF16, {"bf": ...}, W, (128, 128), ["weight 'w' is not selected"]),
        (BF16, None, {"v": "v_scale_inv"}, (128, 128), ["'w' is F8_E4M3, which does not convert"]),  # no scale: refused
    ]

    async def run():
        async with volume_with({"/m": image}) as (client, stub, faults):
            for dtype, select, scales, block, parts in cases:
                for sliced in ((False, True) if not select else (True,)):
                    calls, gets = len(stub.get_file_calls), faults["gets"]
                    with pytest.raises(ValueError) as err:
                        if sliced:
                            sel = select or {k: ... for k in sd if k not in scales.values()}
                            await volume.read_safetensors_slices(client, "vo-r", "/m", sel, dtype=dtype, scales=scales,
                                                                 scale_block=block)
                        else:
                            await volume.read_safetensors(client, "vo-r", "/m", dtype=dtype, scales=scales,
                                                          scale_block=block)
                    for part in parts:
                        assert part in str(err.value), (part, str(err.value))
                    assert len(stub.get_file_calls) == calls + 3 and faults["gets"] == gets + 2  # the header only

    asyncio.run(run())
