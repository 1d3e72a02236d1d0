"""``DeviceFile.safetensors(..., fp8=...)`` and ``safetensors_shards(..., fp8=...)`` on the CPU: the C ABI of the FP8
entries, a torch CPU model of the quantization checked against ``per_block_cast_to_fp8``, the file against
``safetensors.torch.save`` of the quantized dict, the part split of ``b200h_scaled_segment_parts_preview``, the upload
rounds, the Hub's sharded layout, the round trip through ``read_safetensors(..., scales=...)`` and every refusal.  The
context quantizes with the model; the library's own preview checks every argument rule."""
import asyncio
import ctypes
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
from tests import test_device_file_cast_cpu as upload_cast
from tests import test_volume_read_fp8_cpu as read_fp8
from tests.test_device_file_cast_cpu import CastContext, _CastHostSegments, _upload_all, cast_images
from tests.test_safetensors_shards_cpu import assert_same_files, hub_files, our_files
from tests.test_stage_ranges_cpu import StagedHostDeviceFile, _normal, _recording_server
from tests.test_volume_read_cpu import BS, read_backend, volume_with  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16, F16, F32, E4M3 = torch.bfloat16, torch.float16, torch.float32, torch.float8_e4m3fn
BY_CODE = {code: dt for dt, code in cast_dtypes().items()}
INV_448 = torch.tensor(1 / 448, dtype=F32)  # RN(1 / 448)


def fp8_block_reference(w, block=(128, 128)):
    """per_block_cast_to_fp8 (DeepGEMM's tests), generalised to edge blocks and None dimensions."""
    R, C = w.shape
    bR, bC = (R if block[0] is None else block[0]), (C if block[1] is None else block[1])
    gR, gC = -(-R // bR), -(-C // bC)
    padded = w.new_zeros(gR * bR, gC * bC)
    padded[:R, :C] = w
    v = padded.view(gR, bR, gC, bC)
    amax = v.abs().float().amax(dim=(1, 3), keepdim=True).clamp(1e-4)
    q = (v * (448.0 / amax)).to(E4M3).view(gR * bR, gC * bC)[:R, :C].contiguous()
    return q, (amax / 448.0).view(gR, gC)


def _expand(x, block, shape):
    R, C = shape
    return x.repeat_interleave(block[0], 0)[:R].repeat_interleave(block[1], 1)[:, :C]


def model_amax(w, block):
    """a of every block: the integer max of the |x| bits widened to F32 (a NaN wins), then the 1e-4 floor."""
    R, C = w.shape
    br, bc = min(block[0], R), min(block[1], C)
    gR, gC = -(-R // br), -(-C // bc)
    bits = w.float().abs().view(torch.int32).to(torch.int64)
    padded = torch.zeros(gR * br, gC * bc, dtype=torch.int64)
    padded[:R, :C] = bits
    top = padded.view(gR, br, gC, bc).amax(dim=(1, 3)).to(torch.int32).view(F32)
    return torch.where(torch.isnan(top), top, torch.clamp(top, min=1e-4))


def model_scale(a):
    """s = a * RN(1 / 448): ATen's CUDA true division by a CPU scalar multiplies by its reciprocal."""
    return a * INV_448


def model_q(w, a, block):
    """q = E4M3(RN(float(x) * m)) with m = RN(RN(1 / a) * 448)."""
    m = torch.reciprocal(a) * 448.0
    return (w.float() * _expand(m, block, w.shape)).to(E4M3)


def _tensor_at(ptr, nbytes, dtype):
    return torch.frombuffer(bytearray(ctypes.string_at(int(ptr), int(nbytes))), dtype=torch.uint8).view(dtype)


def scaled_images(seg_ptrs, seg_lens, src_types, dst_types, scales, file_first_seg):
    """The image of every file: cast_images, with quantizing segments replaced by the model's q."""
    plain_dst = [0 if d == _lib.DT_F8E4M3 else d for d in dst_types]
    plain_src = [0 if d == _lib.DT_F8E4M3 else s for s, d in zip(src_types, dst_types)]
    segs = [cast_images([p], [n], [s], [d], [0, 1])[0]
            for p, n, s, d in zip(seg_ptrs, seg_lens, plain_src, plain_dst)]
    for k, (p, n, st, dt, sc) in enumerate(zip(seg_ptrs, seg_lens, src_types, dst_types, scales)):
        if dt == _lib.DT_F8E4M3 and st != dt:
            amax_ptr, count, R, C, br, bc = map(int, sc)
            w = _tensor_at(p, n, BY_CODE[st]).view(R, C)
            a = _tensor_at(amax_ptr, count * 4, F32)
            br, bc = min(br, R), min(bc, C)
            a = a[: -(-R // br) * -(-C // bc)].view(-(-R // br), -(-C // bc))
            segs[k] = model_q(w, a, (br, bc)).view(torch.uint8).numpy().tobytes()
    return [b"".join(segs[file_first_seg[f] : file_first_seg[f + 1]]) for f in range(len(file_first_seg) - 1)]


class Fp8Context(CastContext, read_fp8.ScaledContext):
    """Plus ``fp8_block_scales``, ``hash_scaled_segment_parts_device`` and ``copy_scaled_ranges`` over host addresses,
    quantizing with the model; the scaled entries check their segments through ``b200h_scaled_segment_parts_preview``."""

    def fp8_block_scales(self, jobs, stream=0):
        self.calls.append(("fp8_block_scales", len(jobs)))
        for src, st, R, C, br, bc, s_ptr, a_ptr in jobs:
            w = _tensor_at(src, R * C * BY_CODE[st].itemsize, BY_CODE[st]).view(R, C)
            a = model_amax(w, (br, bc))
            s = model_scale(a)
            ctypes.memmove(a_ptr, a.numpy().tobytes(), a.numel() * 4)
            ctypes.memmove(s_ptr, s.numpy().tobytes(), s.numel() * 4)

    def hash_scaled_segment_parts_device(self, seg_ptrs, seg_lens, src_types, dst_types, scales, file_first_seg,
                                         part_len, flags, d_sha=0, d_md5=0, d_trimmed=0, stream=0):
        self.calls.append(("hash_scaled_segment_parts_device", len(file_first_seg) - 1, part_len, flags))
        _lib.scaled_segment_parts_preview(seg_lens, src_types, dst_types, scales, file_first_seg, part_len, 1 << 30)
        images = scaled_images(seg_ptrs, seg_lens, src_types, dst_types, scales, file_first_seg)
        return self._hash_images(images, part_len, flags, d_sha, d_md5, d_trimmed)

    def _hash_images(self, images, part_len, flags, d_sha, d_md5, d_trimmed):
        from oracle import c_oracle

        data = np.frombuffer(b"".join(images) or b"\0", np.uint8)
        starts, lens, at = [], [], 0
        for img in images:
            for o in range(0, len(img), part_len):
                starts.append(at + o)
                lens.append(min(part_len, len(img) - o))
            at += len(img)
        s, m, e = c_oracle.hash_batch(data, np.array(starts, np.uint64), np.array(lens, np.uint64),
                                      sha=bool(flags & _lib.SHA256), md5=bool(flags & _lib.MD5),
                                      trim=bool(flags & _lib.TRIM_ZEROS))
        for addr, table in ((d_sha, s), (d_md5, m), (d_trimmed, e)):
            if addr and table is not None and len(table):
                ctypes.memmove(addr, np.ascontiguousarray(table).tobytes(), table.nbytes)
        return len(starts)

    def copy_scaled_ranges(self, seg_ptrs, seg_lens, src_types, dst_types, scales, file_first_seg, ranges, dst,
                           dst_offsets, stream=0):
        self.calls.append(("copy_scaled_ranges", len(ranges), sum(n for _, _, n in ranges)))
        _lib.scaled_segment_parts_preview(seg_lens, src_types, dst_types, scales, file_first_seg, 1 << 20, 1 << 30)
        assert all(at % 16 == 0 for at in dst_offsets)
        images = scaled_images(seg_ptrs, seg_lens, src_types, dst_types, scales, file_first_seg)
        for (f, off, n), at in zip(ranges, dst_offsets):
            assert off + n <= len(images[f])
            dst[at : at + n] = np.frombuffer(images[f][off : off + n], np.uint8)


class _Fp8HostSegments(_CastHostSegments):
    def __init__(self, tensors, bounce_bytes, casts=None, ctx=None, scales=None):
        self._attach(tensors, bounce_bytes, casts, ctx, scales)
        self.stream_handle = 0

    @classmethod
    def _new_tensor(cls, shape, dtype, ctx):
        return torch.empty(shape, dtype=dtype)


class Fp8HostDeviceFile(StagedHostDeviceFile):
    _Source = _Fp8HostSegments


@pytest.fixture
def fp8_backend(monkeypatch, read_backend):  # noqa: F811
    from modal_client_b200 import _backend

    ctx = Fp8Context()
    monkeypatch.setattr(_backend, "_override", ctx)
    return ctx


def ref_dict(sd, fp8, block=(128, 128), suffix="_scale_inv", dtype=None):
    """The caller's dict, every fp8 weight replaced by the model's q and its scale inserted right after it, the others
    converted by ``dtype``."""
    out = {}
    for n, t in sd.items():
        if n in fp8:
            blk = tuple(min(b or d, d) for b, d in zip(block, t.shape))
            a = model_amax(t, blk)
            out[n], out[n + suffix] = model_q(t, a, blk), model_scale(a)
        elif isinstance(dtype, dict) and n in dtype:
            out[n] = t.to(dtype[n])
        elif dtype is not None and not isinstance(dtype, dict) and t.dtype in (F32, F16, BF16):
            out[n] = t.to(dtype)
        else:
            out[n] = t
    return out


def stack(seed, dtype=BF16):
    g = torch.Generator().manual_seed(seed)
    sd = {"embed": torch.randn(50, 24, generator=g).to(dtype)}
    for i, (R, C) in enumerate([(130, 136), (97, 131), (256, 256), (33, 300), (130, 17), (1, 1)]):
        sd[f"l{i}.w"] = (torch.randn(R, C, generator=g) * 3).to(dtype)
        sd[f"l{i}.norm"] = torch.ones(C, dtype=dtype)
    sd["l2.w"][:128, :128] = 0
    sd["l3.w"][5, 7] = float("inf")
    sd["l4.w"][3, 3] = float("nan")
    sd["steps"] = torch.arange(11)
    return sd


def image(f) -> bytes:
    f.seek(0)
    return f.read()


# ------------------------------------------------------------------------------------------------ C ABI


def test_fp8_entry_points_are_declared_exported_and_reject_a_null_context():
    header = open(os.path.join(ROOT, "include", "b200hash.h")).read()
    for name in ("b200h_fp8_block_scales", "b200h_copy_scaled_ranges", "b200h_hash_scaled_segment_parts_device",
                 "b200h_scaled_segment_parts_preview"):
        assert name in _lib.ABI_SYMBOLS and hasattr(_lib.load_library(), name)
        assert re.search(rf"\bint {name}\(", header)
    L = _lib.load_library()
    first = (ctypes.c_uint64 * 1)(0)
    got = ctypes.c_uint64(777)
    assert L.b200h_fp8_block_scales(None, None, 0, None) == -1
    assert L.b200h_copy_scaled_ranges(None, None, 0, first, 0, None, 0, None, 0, None, None) == -1
    assert L.b200h_hash_scaled_segment_parts_device(None, None, 0, first, 0, 8, _lib.SHA256, None, None, None,
                                                    ctypes.byref(got), None) == -1
    assert got.value == 777


def test_struct_layouts_match_the_binding():
    header = open(os.path.join(ROOT, "include", "b200hash.h")).read()
    body = re.search(r"typedef struct b200h_scaled_segment \{(.*?)\} b200h_scaled_segment;", header, re.S).group(1)
    assert [ln.split("/*")[0].strip() for ln in body.strip().splitlines()] == \
        ["b200h_cast_segment cast;", "const float* d_amax;", "uint64_t scale_count;", "uint64_t rows, cols;",
         "uint64_t block_rows, block_cols;"]
    body = re.search(r"typedef struct b200h_fp8_scale_job \{(.*?)\} b200h_fp8_scale_job;", header, re.S).group(1)
    assert [ln.split("/*")[0].strip() for ln in body.strip().splitlines()] == \
        ["const void* d_src;", "uint64_t src_type;", "uint64_t rows, cols;", "uint64_t block_rows, block_cols;",
         "float* d_scales;", "float* d_amax;"]
    segs = _lib._scaled_segments([0x1000], [8], [_lib.DT_F32], [_lib.DT_F8E4M3], [(0x2000, 4, 1, 2, 128, 128)])
    assert segs.shape == (1, 10) and segs.tolist() == [[0x1000, 8, 1, 4, 0x2000, 4, 1, 2, 128, 128]]


def _preview(**kw):
    args = dict(seg_lens=[8, 24 * 2], src_types=[0, _lib.DT_BF16], dst_types=[0, _lib.DT_F8E4M3],
                scales=[(0,) * 6, (0, 1, 4, 6, 128, 128)], file_first_seg=[0, 2], part_len=16, wave_bytes=1 << 20)
    args.update(kw)
    return _lib.scaled_segment_parts_preview(**args)


def test_preview_rejects_every_broken_quantizing_rule_and_the_cast_entries_refuse_fp8():
    _preview()
    bad = [dict(src_types=[0, _lib.DT_F8E5M2]),  # an FP8 source
           dict(dst_types=[0, _lib.DT_F8E5M2]),  # E5M2 is not a target
           dict(seg_lens=[8, 46]),  # len != R * C * ss
           dict(scales=[(0,) * 6, (0, 1, 4, 6, 0, 128)]),  # block rows 0
           dict(scales=[(0,) * 6, (0, 1, 4, 6, 128, 0)]),  # block cols 0
           dict(scales=[(0,) * 6, (0, 3, 4, 6, 2, 2)]),  # 2 x 3 blocks, 3 scales
           dict(file_first_seg=[0, 3])]
    for b in bad:
        with pytest.raises(_lib.B200HashError):
            _preview(**b)
    _preview(scales=[(0,) * 6, (0, 6, 4, 6, 2, 2)])
    with pytest.raises(_lib.B200HashError):  # the cast entries keep refusing the FP8 codes
        _lib.cast_segment_parts_preview([8, 48], [0, _lib.DT_BF16], [0, _lib.DT_F8E4M3], [0, 2], 16, 1 << 20)


def test_preview_gathers_every_part_that_touches_a_quantizing_segment():
    lens = [4096, 2 * 64 * 64, 4096, 4 * 100 * 10]
    scales = [(0,) * 6, (0, 1, 64, 64, 128, 128), (0,) * 6, (0, 1, 100, 10, 128, 128)]
    seg, wave, nw = _lib.scaled_segment_parts_preview(lens, [0, _lib.DT_BF16, 0, _lib.DT_F32],
                                                      [0, _lib.DT_F8E4M3, 0, _lib.DT_F8E4M3], scales, [0, 4], 1024,
                                                      2048)
    image = [(0, 4096, 0), (4096, 8192, 1), (8192, 12288, 2), (12288, 13288, 3)]
    want = []
    for o in range(0, 13288, 1024):
        hit = [s for lo, hi, s in image if lo < min(o + 1024, 13288) and hi > o]
        want.append(hit[0] if len(hit) == 1 and hit[0] in (0, 2) else _lib.GATHERED)
    assert list(map(int, seg)) == want and nw == 3  # 2 KiB per wave: two gathered 1 KiB parts each
    assert list(map(int, wave)) == [0] * 6 + [1] * 6 + [2]


# ------------------------------------------------------------------------------------------------ the model


@pytest.mark.parametrize("block", [(128, 128), (64, 32), (1, None), (None, None), (7, 5)])
@pytest.mark.parametrize("dtype", [F32, F16, BF16])
def test_the_model_is_per_block_cast_to_fp8_but_for_the_scale_division(block, dtype):
    sd = stack(3, dtype)
    for n, w in sd.items():
        if w.dim() != 2:
            continue
        blk = tuple(min(b or d, d) for b, d in zip(block, w.shape))
        q, s = fp8_block_reference(w, block)
        a = model_amax(w, blk)
        assert torch.equal(model_q(w, a, blk).view(torch.uint8), q.view(torch.uint8)), n
        # the reference's own clamped amax, before its division
        R, C = w.shape
        gR, gC = -(-R // blk[0]), -(-C // blk[1])
        padded = w.new_zeros(gR * blk[0], gC * blk[1])
        padded[:R, :C] = w
        ref_a = padded.view(gR, blk[0], gC, blk[1]).abs().float().amax(dim=(1, 3)).clamp(1e-4)
        assert torch.equal(a.view(torch.int32), ref_a.view(torch.int32)) or (torch.isnan(a).any() and
                                                                              torch.equal(a.isnan(), ref_a.isnan()))
        # the CPU divides by 448; on CUDA the division by a CPU scalar multiplies by RN(1 / 448) (checked on the GPU)
        assert torch.allclose(s, model_scale(a), rtol=2 ** -23, atol=0, equal_nan=True)


# ------------------------------------------------------------------------------------------------ the file


@pytest.mark.parametrize("block", [(128, 128), (64, 32), (1, None), (None, None)])
@pytest.mark.parametrize("dtype", [F32, F16, BF16])
def test_file_bytes_equal_safetensors_save_of_the_quantized_dict(fp8_backend, block, dtype):
    sd = stack(1, dtype)
    fp8 = [n for n in sd if n.endswith(".w")]
    f = Fp8HostDeviceFile.safetensors(sd, {"format": "pt"}, fp8=fp8, scale_block=block)
    want = st_save(ref_dict(sd, fp8, block), {"format": "pt"})
    assert f.nbytes == len(want) and image(f) == want
    assert [c for c in fp8_backend.calls if c[0] == "fp8_block_scales"] == [("fp8_block_scales", len(fp8))]
    rng = random.Random(block[0] or 0)
    g = Fp8HostDeviceFile.safetensors(sd, {"format": "pt"}, fp8=fp8, scale_block=block, bounce_bytes=1000)
    for _ in range(60):
        pos, n = rng.randrange(len(want) + 5), rng.choice([1, 15, 16, 17, rng.randrange(1, 5000)])
        g.seek(pos)
        assert g.read(n) == want[pos : pos + n]


def test_dtype_mixes_and_the_quantized_weights_stay_in_place(fp8_backend):
    sd = stack(2, F32)
    fp8 = ["l0.w", "l2.w", "l5.w"]
    for dtype in (BF16, {"embed": F16, "l1.w": BF16}):
        f = Fp8HostDeviceFile.safetensors(sd, fp8=fp8, dtype=dtype, scale_block=(1, None), scale_suffix="_scale")
        assert image(f) == st_save(ref_dict(sd, fp8, (1, None), "_scale", dtype))
        src = f._src
        for n in fp8:
            k = [t.data_ptr() for t in src.tensors].index(sd[n].data_ptr())
            assert src.casts[k] == (_lib.DT_F32, _lib.DT_F8E4M3) and src.scales[k][2:4] == tuple(sd[n].shape)


def test_fp8_none_makes_todays_calls(fp8_backend):
    sd = stack(4, F32)
    for dtype in (None, BF16):
        a = Fp8HostDeviceFile.safetensors(sd, dtype=dtype)
        b = upload_cast.CastHostDeviceFile.safetensors(sd, dtype=dtype)
        calls = list(fp8_backend.calls)
        assert image(a) == image(b)
        assert a._src.scales is None
        assert not [c for c in calls if "scale" in c[0] or "fp8" in c[0]]
    assert not [c for c in fp8_backend.calls if "scale" in c[0] or "fp8" in c[0]]


def test_every_refusal_comes_in_one_error_before_any_device_copy(fp8_backend):
    g = torch.Generator().manual_seed(0)
    w = torch.randn(4, 4, generator=g)
    sd = {"w": w, "tied": w.view(16), "v": torch.randn(3), "e": torch.zeros(0, 3), "i": torch.ones(2, 2, dtype=torch.int32),
          "d": torch.randn(3, 3, dtype=torch.float64), "x": torch.randn(2, 2), "x_scale_inv": torch.ones(1),
          "y": torch.randn(2, 2)}
    before = _Fp8HostSegments.to_device
    with pytest.raises(ValueError) as e:
        Fp8HostDeviceFile.safetensors(sd, fp8=["w", "nope", "v", "e", "i", "d", "x", "y", "y"], dtype={"y": BF16})
    msg = str(e.value)
    for part in ("'nope' is in fp8 but not in the tensors", "'v' is not a non-empty 2-D tensor",
                 "'e' is not a non-empty 2-D tensor", "'i' is torch.int32; only float32",
                 "'d' is torch.float64; only float32", "'x_scale_inv', is already a tensor name",
                 "'w' shares its storage with 'tied'", "'y' is in fp8 twice", "'y' is in both fp8 and dtype"):
        assert part in msg, part
    for block in ((0, 128), (128,), (128, 1.5), "128", (True, 1)):
        with pytest.raises(ValueError, match="scale_block"):
            Fp8HostDeviceFile.safetensors({"x": torch.ones(2, 2)}, fp8=["x"], scale_block=block)
    with pytest.raises(ValueError, match="scale_suffix"):
        Fp8HostDeviceFile.safetensors({"x": torch.ones(2, 2)}, fp8=["x"], scale_suffix=None)
    with pytest.raises(ValueError, match="iterable"):
        Fp8HostDeviceFile.safetensors({"x": torch.ones(2, 2)}, fp8="x")
    with pytest.raises(ValueError, match="safetensors_shards.*'nope' is in fp8"):
        Fp8HostDeviceFile.safetensors_shards({"x": torch.ones(2, 2)}, fp8=["nope"])
    assert _Fp8HostSegments.to_device == before
    assert not [c for c in fp8_backend.calls if c[0] != "host_alloc"]


# ------------------------------------------------------------------------------------------------ uploads


@pytest.mark.parametrize("budget", [None, 8192, 1 << 22])
def test_upload_equals_the_upload_of_the_prequantized_dict(fp8_backend, monkeypatch, budget):
    monkeypatch.setattr(blob_utils, "BLOCK_SIZE", 4096)
    sd = stack(5, BF16)
    fp8 = [n for n in sd if n.endswith(".w")]
    other = {"x": torch.arange(3000, dtype=torch.int32)}

    async def run(pre):
        fp8_backend.calls.clear()
        async with _recording_server(4096) as (stub, log, _):
            f = StagedHostDeviceFile.safetensors(ref_dict(sd, fp8)) if pre else \
                Fp8HostDeviceFile.safetensors(sd, fp8=fp8)
            fs = [f, StagedHostDeviceFile.safetensors(other)]
            await _upload_all(stub, fs, budget)
            kinds = [c[0] for c in fp8_backend.calls if c[0] not in ("host_alloc", "fp8_block_scales")]
            return (dict(stub.blocks), {p: v[0] for p, v in stub.volume_files.items()}, _normal(log),
                    [f.bytes_to_host for f in fs]), kinds

    want, plain_calls = asyncio.run(run(True))
    got, fp8_calls = asyncio.run(run(False))
    assert got == want and want[1]["/ckpt/0"] == st_save(ref_dict(sd, fp8))
    plain = {"hash_scaled_segment_parts_device": "hash_segment_parts_device", "copy_scaled_ranges": "copy_ranges_to_host"}
    assert fp8_calls.count("hash_scaled_segment_parts_device") == 1  # one hash call for the batch
    copies = ("copy_scaled_ranges", "copy_ranges_to_host")
    assert [plain.get(k, k) for k in fp8_calls if k not in copies] == [k for k in plain_calls if k not in copies]


# ------------------------------------------------------------------------------------------------ shards


@pytest.mark.parametrize("max_size", [130 * 136, 6000, "5GB"])
def test_shards_equal_the_hubs_save_of_the_quantized_dict(fp8_backend, tmp_path, max_size):
    sd = stack(6, BF16)
    fp8 = [n for n in sd if n.endswith(".w")]
    shards = Fp8HostDeviceFile.safetensors_shards(sd, fp8=fp8, max_shard_size=max_size)
    ref = ref_dict(sd, fp8)
    assert_same_files(our_files(shards), hub_files(ref, tmp_path, max_shard_size=max_size))
    assert [c for c in fp8_backend.calls if c[0] == "fp8_block_scales"] == [("fp8_block_scales", len(fp8))]
    if max_size == 130 * 136:  # l0.w fills a shard: its scale opens the next one
        import json

        wm = json.loads(shards.index[1])["weight_map"]
        assert wm["l0.w"] != wm["l0.w_scale_inv"]


# ------------------------------------------------------------------------------------------------ round trip


@pytest.mark.parametrize("sharded", [False, True])
def test_round_trip_through_read_safetensors_with_scales(fp8_backend, tmp_path, sharded):
    sd = stack(7, BF16)
    fp8 = [n for n in sd if n.endswith(".w") and n != "l4.w"]  # l4.w holds a NaN
    ref = ref_dict(sd, fp8)
    files = (dict(our_files(Fp8HostDeviceFile.safetensors_shards(sd, fp8=fp8, max_shard_size=20_000))) if sharded
             else {"model.safetensors": image(Fp8HostDeviceFile.safetensors(sd, fp8=fp8))})

    async def go():
        async with volume_with(files) as (client, _, _):
            scales = volume.fp8_scales(list(ref))
            if sharded:
                return await volume.read_safetensors_sharded(client, "vo-r", "model.safetensors.index.json",
                                                             dtype=BF16, scales=scales)
            return await volume.read_safetensors(client, "vo-r", "model.safetensors", dtype=BF16, scales=scales)

    got = asyncio.run(go())
    for n in fp8:
        s = _expand(ref[n + "_scale_inv"], (128, 128), sd[n].shape)
        assert torch.equal(got[n].view(torch.int16), (ref[n].float() * s).to(BF16).view(torch.int16)), n
