"""``DeviceFile.safetensors(..., dtype=)`` on the CPU: the C ABI of the cast entry points, the converted image against
``safetensors.torch.save`` of the ``.to()`` dict, reads at any position, the part split of
``b200h_cast_segment_parts_preview``, and the volumefs2 upload rounds against the upload of the pre-converted dict.
The context converts with torch's CPU ``.to()``; the library's own previews check every argument rule."""
import asyncio
import ctypes
import hashlib
import os
import random
import re
import types

import numpy as np
import pytest
import torch
from safetensors.torch import save as st_save

from modal_client_b200 import _lib, blob_utils, volume
from modal_client_b200.device_file import cast_dtypes
from oracle import c_oracle
from tests.test_stage_ranges_cpu import (StagedHostDeviceFile, StagingContext, _normal, _recording_server,
                                         _StagedHostSegments)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
BY_CODE = {code: dt for dt, code in cast_dtypes().items()}


def cast_images(seg_ptrs, seg_lens, src_types, dst_types, file_first_seg):
    """The image of every file: each segment's host bytes, converted by torch's CPU ``.to()`` where it converts."""
    segs = []
    for p, n, st, dt in zip(seg_ptrs, seg_lens, src_types, dst_types):
        raw = ctypes.string_at(int(p), int(n)) if n else b""
        if st != dt:
            t = torch.frombuffer(bytearray(raw), dtype=torch.uint8).view(BY_CODE[st]) if n else \
                torch.empty(0, dtype=BY_CODE[st])
            raw = t.to(BY_CODE[dt]).view(torch.uint8).numpy().tobytes()
        segs.append(raw)
    return [b"".join(segs[file_first_seg[f] : file_first_seg[f + 1]]) for f in range(len(file_first_seg) - 1)]


class CastContext(StagingContext):
    """Plus ``hash_cast_segment_parts_device`` and ``copy_cast_ranges`` over host addresses.  Both check their
    segments through ``b200h_cast_segment_parts_preview`` (which raises like the entry points) and convert with
    torch's CPU ``.to()``."""

    def hash_cast_segment_parts_device(self, seg_ptrs, seg_lens, src_types, dst_types, file_first_seg, part_len, flags,
                                       d_sha=0, d_md5=0, d_trimmed=0, stream=0):
        self.calls.append(("hash_cast_segment_parts_device", len(file_first_seg) - 1, part_len, flags))
        seg, _, _ = _lib.cast_segment_parts_preview(seg_lens, src_types, dst_types, file_first_seg, part_len, 1 << 30)
        images = cast_images(seg_ptrs, seg_lens, src_types, dst_types, file_first_seg)
        data = np.frombuffer(b"".join(images) or b"\0", np.uint8)
        starts, lens, at = [], [], 0
        for img in images:
            for o in range(0, len(img), part_len):
                starts.append(at + o)
                lens.append(min(part_len, len(img) - o))
            at += len(img)
        assert len(starts) == len(seg)
        s, m, e = c_oracle.hash_batch(data, np.array(starts, np.uint64), np.array(lens, np.uint64),
                                      sha=bool(flags & _lib.SHA256), md5=bool(flags & _lib.MD5),
                                      trim=bool(flags & _lib.TRIM_ZEROS))
        for addr, table in ((d_sha, s), (d_md5, m), (d_trimmed, e)):
            if addr and table is not None and len(table):
                ctypes.memmove(addr, np.ascontiguousarray(table).tobytes(), table.nbytes)
        return len(starts)

    def copy_cast_ranges(self, seg_ptrs, seg_lens, src_types, dst_types, file_first_seg, ranges, dst, dst_offsets,
                         stream=0):
        self.calls.append(("copy_cast_ranges", len(ranges), sum(n for _, _, n in ranges)))
        _lib.cast_segment_parts_preview(seg_lens, src_types, dst_types, file_first_seg, 1 << 20, 1 << 30)
        spans = sorted((at, at + n) for at, (_, _, n) in zip(dst_offsets, ranges) if n)
        assert all(at % 16 == 0 for at in dst_offsets) and all(hi <= dst.size for _, hi in spans)
        assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))
        images = cast_images(seg_ptrs, seg_lens, src_types, dst_types, file_first_seg)
        for (f, off, n), at in zip(ranges, dst_offsets):
            assert off + n <= len(images[f])
            dst[at : at + n] = np.frombuffer(images[f][off : off + n], np.uint8)


class _CastHostSegments(_StagedHostSegments):
    to_device = 0  # header copies to the "device"

    def __init__(self, tensors, bounce_bytes, casts=None, ctx=None):
        self._attach(tensors, bounce_bytes, casts, ctx)
        self.stream_handle = 0

    @classmethod
    def _to_device(cls, data, ctx):
        cls.to_device += 1
        return super()._to_device(data, ctx)


class CastHostDeviceFile(StagedHostDeviceFile):
    _Source = _CastHostSegments


@pytest.fixture
def cast_backend(monkeypatch):
    from modal_client_b200 import _backend

    ctx = CastContext()
    monkeypatch.setattr(_backend, "_override", ctx)
    return ctx


def random_dict(seed, n=12, big=False):
    """Tensors of every dtype safetensors stores, floats of the three convertible types most often."""
    g = torch.Generator().manual_seed(seed)
    rng = random.Random(seed)
    kinds = [F32, F32, F32, F16, BF16, torch.int64, torch.int8, torch.bool, torch.float64, torch.uint8, torch.int32]
    sd = {}
    for i in range(n):
        dt = rng.choice(kinds)
        shape = rng.choice([(), (0,), (1,), (3, 5), (rng.randrange(1, 4000),), (7, rng.randrange(1, 300))])
        if big and i == 0:
            dt, shape = F32, (50_000,)
        if dt.is_floating_point:
            t = (torch.randn(shape, generator=g, dtype=torch.float64) * 10 ** rng.randrange(-6, 6)).to(dt)
        elif dt == torch.bool:
            t = torch.randint(0, 2, shape, generator=g).bool()
        else:
            t = torch.randint(-100 if dt.is_signed else 0, 100, shape, generator=g, dtype=dt)
        sd[f"t{rng.randrange(1000)}.{i}"] = t
    return sd


def converted(sd, dtype):
    """{k: v.to(target)} as ``dtype`` asks (one dtype for every F32 / F16 / BF16 tensor, or a mapping)."""
    if isinstance(dtype, dict):
        return {k: v.to(dtype[k]) if k in dtype else v for k, v in sd.items()}
    return {k: v.to(dtype) if v.dtype in (F32, F16, BF16) else v for k, v in sd.items()}


def image(f) -> bytes:
    f.seek(0)
    return f.read()


# ------------------------------------------------------------------------------------------------ C ABI


def test_cast_entry_points_are_declared_exported_and_reject_a_null_context():
    header = open(os.path.join(ROOT, "include", "b200hash.h")).read()
    for name in ("b200h_copy_cast_ranges", "b200h_hash_cast_segment_parts_device", "b200h_cast_segment_parts_preview"):
        assert name in _lib.ABI_SYMBOLS and hasattr(_lib.load_library(), name)
        assert re.search(rf"\bint {name}\(", header)
    L = _lib.load_library()
    first = (ctypes.c_uint64 * 1)(0)
    got = ctypes.c_uint64(777)
    assert L.b200h_copy_cast_ranges(None, None, 0, first, 0, None, 0, None, 0, None, None) == -1
    assert L.b200h_hash_cast_segment_parts_device(None, None, 0, first, 0, 8, _lib.SHA256, None, None, None,
                                                  ctypes.byref(got), None) == -1
    assert got.value == 777


def test_cast_segment_struct_layout_matches_the_binding():
    class CastSegment(ctypes.Structure):  # b200h_cast_segment as include/b200hash.h declares it
        _fields_ = [("d_ptr", ctypes.c_void_p), ("len", ctypes.c_uint64), ("src_type", ctypes.c_uint64),
                    ("dst_type", ctypes.c_uint64)]

    assert ctypes.sizeof(CastSegment) == 32
    header = open(os.path.join(ROOT, "include", "b200hash.h")).read()
    body = re.search(r"typedef struct b200h_cast_segment \{(.*?)\} b200h_cast_segment;", header, re.S).group(1)
    assert [ln.split("/*")[0].strip() for ln in body.strip().splitlines()] == \
        ["const void* d_ptr;", "uint64_t len;", "uint64_t src_type, dst_type;"]
    segs = _lib._cast_segments([0x1000, 0x2000], [8, 6], [_lib.DT_F32, 0], [_lib.DT_BF16, 0])
    assert segs.dtype == np.uint64 and segs.shape == (2, 4) and segs.flags.c_contiguous
    raw = (CastSegment * 2).from_buffer_copy(segs.tobytes())
    assert [(r.d_ptr, r.len, r.src_type, r.dst_type) for r in raw] == [(0x1000, 8, 1, 3), (0x2000, 6, 0, 0)]
    assert (_lib.DT_F32, _lib.DT_F16, _lib.DT_BF16) == (1, 2, 3)
    assert all(f"#define B200H_DT_{n} {v}u" in header for n, v in (("F32", 1), ("F16", 2), ("BF16", 3)))


def test_preview_rejects_every_broken_cast_rule():
    ok = dict(seg_lens=[8, 40], src_types=[0, _lib.DT_F32], dst_types=[0, _lib.DT_BF16], file_first_seg=[0, 2])
    _lib.cast_segment_parts_preview(**ok, part_len=16, wave_bytes=1 << 20)
    bad = [dict(ok, seg_lens=[8, 42]),  # not whole source elements
           dict(ok, src_types=[0, 7]),  # unknown source type
           dict(ok, dst_types=[0, 9]),  # unknown destination type
           dict(ok, src_types=[5, _lib.DT_F32], dst_types=[5, _lib.DT_BF16]),  # equal, but not a type
           dict(ok, seg_lens=[6, 40], dst_types=[0, _lib.DT_F32], src_types=[0, _lib.DT_BF16]),  # image at 6 % 4
           dict(ok, file_first_seg=[0, 3])]
    for b in bad:
        with pytest.raises(_lib.B200HashError):
            _lib.cast_segment_parts_preview(**b, part_len=16, wave_bytes=1 << 20)


# ------------------------------------------------------------------------------------------- the image


@pytest.mark.parametrize("seed", range(6))
def test_converted_image_equals_safetensors_save_of_the_converted_dict(cast_backend, seed):
    sd = random_dict(seed)
    floats = [k for k, v in sd.items() if v.dtype in (F32, F16, BF16)]
    meta = {"format": "pt"} if seed % 2 else None  # one entry: the library orders several in no fixed way
    rng = random.Random(seed)
    dtypes = [BF16, F16, F32, {k: rng.choice([BF16, F16, F32]) for k in floats if rng.random() < 0.7}]
    for dtype in dtypes:
        if not isinstance(dtype, dict) and any(v.dtype == torch.float64 for v in sd.values()):
            with pytest.raises(ValueError, match="F64, which does not convert"):
                CastHostDeviceFile.safetensors(sd, meta, dtype=dtype)
            continue
        f = CastHostDeviceFile.safetensors(sd, meta, dtype=dtype)
        want = st_save(converted(sd, dtype), meta)
        assert f.nbytes == len(want) and image(f) == want
        assert f.bytes_to_host == len(want)


def test_targets_reorder_the_data_and_unconverted_tensors_stay_in_place(cast_backend):
    sd = {"a": torch.arange(10, dtype=F32), "b": torch.arange(6, dtype=torch.int16), "c": torch.ones(3, dtype=BF16),
          "d": torch.arange(5, dtype=torch.int64)}
    f = CastHostDeviceFile.safetensors(sd, dtype={"a": F16, "c": F32})
    assert image(f) == st_save(converted(sd, {"a": F16, "c": F32}))
    names = [n for n in re.findall(rb'"(\w)":\{"dtype"', image(f))]
    assert names == [b"d", b"c", b"a", b"b"]  # I64, then F32 (was BF16), then F16 (was F32) with I16 by name
    src = f._src
    assert [c for c in src.casts] == [(0, 0), (0, 0), (_lib.DT_BF16, _lib.DT_F32), (_lib.DT_F32, _lib.DT_F16), (0, 0)]
    # every segment is a tensor where it is: no copy, no conversion in memory
    assert [s.data_ptr() for s in src.segments[1:]] == [sd[n].data_ptr() for n in "dcab"]
    g = CastHostDeviceFile.safetensors(sd, dtype=BF16)
    assert image(g) == st_save(converted(sd, BF16))
    at = 1 + [n for n, _ in sorted(sd.items(), key=lambda kv: (kv[1].dtype != torch.int64, kv[1].dtype == torch.int16,
                                                               kv[0]))].index("c")  # I64, then the BF16s, then I16
    assert g._src.segments[at].data_ptr() == sd["c"].data_ptr() and g._src.casts[at] == (0, 0)  # already BF16


def test_dtype_none_or_converting_nothing_is_todays_file(cast_backend):
    sd = random_dict(3)
    for dtype in (None, {}, {k: v.dtype for k, v in sd.items() if v.dtype in (F32, F16, BF16)}):
        f, g = CastHostDeviceFile.safetensors(sd, dtype=dtype), StagedHostDeviceFile.safetensors(sd)
        assert f._src.casts is None and [s.data_ptr() for s in f._src.segments[1:]] == \
            [s.data_ptr() for s in g._src.segments[1:]]
        assert image(f) == image(g) == st_save(sd)
    assert not [c for c in cast_backend.calls if "cast" in c[0]]


def test_reads_at_random_positions_cross_segment_and_element_edges(cast_backend):
    sd = random_dict(11, n=16, big=True)
    sd = {k: v for k, v in sd.items() if v.dtype != torch.float64}
    want = st_save(converted(sd, BF16))
    rng = random.Random(4)
    for bounce in (16, 1000, 1 << 20):
        f = CastHostDeviceFile.safetensors(sd, dtype=BF16, bounce_bytes=bounce)
        for _ in range(60):
            pos = rng.randrange(0, len(want) + 10)
            n = rng.choice([1, 2, 3, 15, 16, 17, rng.randrange(1, 5000), rng.randrange(1, 120_000)])
            f.seek(pos)
            assert f.read(n) == want[pos : pos + n]
        calls = [c for c in cast_backend.calls if c[0] == "copy_cast_ranges"]
        assert calls and all(c[1] == 1 and c[2] <= bounce for c in calls)  # one range per bounce fill
        cast_backend.calls.clear()


def test_every_rejection_comes_in_one_error_before_any_device_copy(cast_backend):
    sd = {"w": torch.ones(4, dtype=F32), "d": torch.ones(4, dtype=torch.float64), "i": torch.ones(2, dtype=torch.int32)}
    before = _CastHostSegments.to_device
    with pytest.raises(ValueError) as e:
        CastHostDeviceFile.safetensors(sd, dtype=BF16)
    assert "'d' is F64, which does not convert" in str(e.value)
    with pytest.raises(ValueError) as e:
        CastHostDeviceFile.safetensors(sd, dtype={"nope": BF16, "i": BF16, "w": torch.float64, "d": F16})
    msg = str(e.value)
    assert all(s in msg for s in ("'nope' is in dtype but not", "'i' is I32; only F32, F16 and BF16 tensors convert",
                                  "'w': torch.float64 is not a supported target", "'d' is F64; only F32"))
    for dtype in (torch.int8, torch.float64, "bf16"):
        with pytest.raises(ValueError, match="is not a supported target"):
            CastHostDeviceFile.safetensors(sd, dtype=dtype)
    with pytest.raises(ValueError, match="reserved"):
        CastHostDeviceFile.safetensors({"__metadata__": torch.ones(2)}, dtype=BF16)
    with pytest.raises(ValueError, match="CUDA"):
        from modal_client_b200 import DeviceFile
        DeviceFile.safetensors({"w": torch.ones(4)}, dtype=BF16)
    assert _CastHostSegments.to_device == before
    assert not cast_backend.calls


# ---------------------------------------------------------------------------------------------- the split


def restated_split(lens, casts, ffs, part_len, wave_cap):
    """(segment or GATHERED per part, wave per part, waves): the parts of every image, in place only inside one
    segment that converts nothing; gathered parts padded to 16 fill waves of wave_cap."""
    size = {1: 4, 2: 2, 3: 2}
    img = [n // size[s] * size[d] if s != d else n for n, (s, d) in zip(lens, casts)]
    segs, waves, used, w = [], [], None, 0
    for f in range(len(ffs) - 1):
        starts, at = [], 0
        for s in range(ffs[f], ffs[f + 1]):
            starts.append((at, at + img[s], s))
            at += img[s]
        for o in range(0, at, part_len):
            e = min(o + part_len, at)
            hit = [s for lo, hi, s in starts if lo < e and hi > o]
            if len(hit) == 1 and casts[hit[0]][0] == casts[hit[0]][1]:
                segs.append(hit[0])
            else:
                need = -(-(e - o) // 16) * 16
                if used is not None and used and used + need > wave_cap:
                    w, used = w + 1, 0
                used = (used or 0) + need
                segs.append(_lib.GATHERED)
            waves.append(w)
    return segs, waves, w + 1 if segs else 0


@pytest.mark.parametrize("seed", range(5))
def test_preview_split_matches_the_restatement(seed):
    rng = random.Random(seed)
    pairs = [(0, 0), (1, 3), (1, 2), (3, 1), (2, 3), (3, 2), (2, 1), (1, 1)]
    lens, casts, ffs = [], [], [0]
    for f in range(rng.randrange(1, 5)):
        at = 0
        for _ in range(rng.randrange(0, 9)):
            st, dt = rng.choice(pairs)
            size = {1: 4, 2: 2, 3: 2}
            if st != dt and at % size[dt]:
                st, dt = 0, 0
            n = rng.choice([0, 4, 8, 64, 100, 4096, rng.randrange(0, 20_000)])
            if st != dt:
                n -= n % size[st]
            lens.append(n)
            casts.append((st, dt))
            at += n // size[st] * size[dt] if st != dt else n
        ffs.append(len(lens))
    for part_len, cap in ((64, 256), (1000, 4096), (4096, 1 << 20), (7, 64)):
        seg, wave, nw = _lib.cast_segment_parts_preview(lens, [s for s, _ in casts], [d for _, d in casts], ffs,
                                                        part_len, cap)
        want = restated_split(lens, casts, ffs, part_len, cap)
        assert (list(map(int, seg)), list(map(int, wave)), nw) == (want[0], want[1], want[2])


def test_preview_has_three_waves_with_a_small_cap_and_no_cast_equals_the_plain_preview():
    lens = [8, 4000, 4000, 100]
    seg, wave, nw = _lib.cast_segment_parts_preview(lens, [0, 1, 3, 0], [0, 3, 1, 0], [0, 4], 512, 1024)
    assert nw >= 3 and int(seg[0]) == _lib.GATHERED  # the header's part reaches into the converting segment
    plain = _lib.segment_parts_preview(lens, [0, 4], 512, 1024)
    same = _lib.cast_segment_parts_preview(lens, [0] * 4, [0] * 4, [0, 4], 512, 1024)
    assert all(np.array_equal(a, b) for a, b in zip(plain[:2], same[:2])) and plain[2] == same[2]


# ------------------------------------------------------------------------------------------------ uploads


def _bf16_dict():
    g = torch.Generator().manual_seed(9)
    sd = {f"layers.{i}.w": torch.randn(n, generator=g) for i, n in enumerate([3000, 1, 700, 5000, 12, 2048, 9000])}
    sd["layers.2.w"][-300:] = 0  # trailing zeros
    sd["blank"] = torch.zeros(6000)  # blank blocks
    sd["dup.a"] = torch.full((8192,), 3.0)  # whole duplicate blocks
    sd["dup.b"] = torch.full((8192,), 3.0)
    sd["step"] = torch.arange(500, dtype=torch.int64)
    sd["emb"] = torch.randn(3000, generator=g).to(BF16)  # already in the target dtype
    return sd


async def _upload_all(stub, files, budget):
    batch = volume.VolumeUploadContextManager2("vo-c", types.SimpleNamespace(stub=stub), device_staging_bytes=budget)
    async with batch:
        for i, f in enumerate(files):
            batch.put_file(f, f"/ckpt/{i}")
    return batch


@pytest.mark.parametrize("budget", [None, 8192, 3 * 4096, 1 << 22])
def test_upload_equals_the_upload_of_the_preconverted_dict(cast_backend, monkeypatch, budget, tmp_path):
    """Blocks, bytes and request sequence; a batch that mixes a converting file, an unconverted device file and a
    host file."""
    BS = 4096
    monkeypatch.setattr(blob_utils, "BLOCK_SIZE", BS)
    sd = _bf16_dict()
    other = {"x": torch.arange(3000, dtype=torch.int32), "y": torch.randn(777)}
    host = tmp_path / "host.bin"
    host.write_bytes(st_save({"z": torch.arange(5000, dtype=torch.int16)}))

    def files(pre):
        conv = StagedHostDeviceFile.safetensors(converted(sd, BF16)) if pre else CastHostDeviceFile.safetensors(sd, dtype=BF16)
        return [conv, StagedHostDeviceFile.safetensors(other), str(host)]

    async def run(pre):
        cast_backend.calls.clear()
        async with _recording_server(BS) as (stub, log, _):
            fs = files(pre)
            await _upload_all(stub, fs, budget)
            kinds = [c[0] for c in cast_backend.calls if c[0] != "host_alloc"]
            return (dict(stub.blocks), {p: v[0] for p, v in stub.volume_files.items()}, _normal(log),
                    [f.bytes_to_host for f in fs[:2]]), kinds

    want, plain_calls = asyncio.run(run(True))
    got, cast_calls = asyncio.run(run(False))
    assert got == want
    assert want[1]["/ckpt/0"] == st_save(converted(sd, BF16))
    # every device call of the pre-converted upload, one per round, is made by its cast twin when the files it covers
    # convert (a staging wave of only the unconverted file stays plain); without a staging budget the missing blocks
    # are read through the bounce buffer, one copy_cast_ranges per fill
    plain = {"hash_cast_segment_parts_device": "hash_segment_parts_device", "copy_cast_ranges": "copy_ranges_to_host"}
    assert "hash_cast_segment_parts_device" in cast_calls and "copy_cast_ranges" in cast_calls
    if budget is None:
        assert [plain.get(k, k) for k in cast_calls if k != "copy_cast_ranges"] == plain_calls
    else:
        assert [plain.get(k, k) for k in cast_calls] == plain_calls


def test_spec2_of_a_converting_file_equals_the_preconverted_spec(cast_backend, monkeypatch):
    from pathlib import PurePosixPath

    BS = 4096
    monkeypatch.setattr(blob_utils, "BLOCK_SIZE", BS)
    sd = _bf16_dict()
    sem = asyncio.Semaphore(1)
    f = CastHostDeviceFile.safetensors(sd, dtype=F16)
    g = StagedHostDeviceFile.safetensors(converted(sd, F16))
    a = asyncio.run(blob_utils.FileUploadSpec2.from_fileobj(f, PurePosixPath("/m"), sem, 0o644))
    b = asyncio.run(blob_utils.FileUploadSpec2.from_fileobj(g, PurePosixPath("/m"), sem, 0o644))
    assert (a.blocks, a.size) == (b.blocks, b.size)
    assert f.bytes_to_host == 0
    data = st_save(converted(sd, F16))
    assert [blk.contents_sha256 for blk in a.blocks] == \
        [hashlib.sha256(data[i : i + BS].rstrip(b"\0")).digest() for i in range(0, len(data), BS)]
