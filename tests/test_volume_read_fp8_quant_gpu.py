"""GPU: F32 / F16 / BF16 weights quantized to block-scaled FP8 E4M3 on the way from page-locked host memory into device
files (``b200h_fp8_amax_boxes_from_host``, ``b200h_copy_quant_boxes_from_host``; ``fp8_amax_boxes_kernel``,
``fp8_finalize_kernel``, ``load_quant_boxes_kernel``), checked bit for bit against the integer reference of
``tests/test_fp8_quant_reference_cpu.py`` run on the device.

Through the entries directly: every F16 and BF16 pattern under every structured amax, the structured and random F32
sets (each element its own block, a given as it is), boxes at every element-aligned source phase and destination
phase, NaN / inf / signed-zero / all-zero / edge blocks through the amax, the finalisation and the copy, and one band's
amax split over two calls.  End to end over the loopback volume server: a ~1 GB Llama-shaped bf16 stack read with
``read_safetensors_sharded(fp8=names)`` equals, as a dict and bit for bit, the FP8 export of the same tensors read
back, and ``fp8_block_reference``, with HBM growing by no more than the results (as the caching allocator rounds them), the amax array and 8 MiB;
F32 and F16 sources, per-channel and per-tensor scales and ``into=`` too."""
import asyncio
import types

import numpy as np
import pytest

from modal_client_b200 import _lib, blob_utils, device_file, volume
from tests.test_device_file_fp8_gpu import fp8_block_reference
from tests.test_fp8_quant_reference_cpu import (random_f32_rows, reference_block_scales, reference_multiplier,
                                                reference_quant, sixteen_bit_pairs, structured_f32_pairs)
from tests.volume_read_server import running_volume_server

pytestmark = pytest.mark.gpu

MiB = 1 << 20
SENTINEL = 0xC3


def _t():
    import torch

    return torch


def _code(dt):
    torch = _t()
    return {torch.float32: _lib.DT_F32, torch.float16: _lib.DT_F16, torch.bfloat16: _lib.DT_BF16}[dt]


def _bits(t):
    """Element bit patterns of a CUDA tensor as int64 (unsigned)."""
    torch = _t()
    ss = t.element_size()
    v = t.contiguous().view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[ss]).to(torch.int64)
    return v & ((1 << (8 * ss)) - 1)


def _current():
    return _t().cuda.current_stream().cuda_stream or 1


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0, pinned_bytes=64 << 20, device_bytes=512 << 20)
    yield c
    c.close()


def _stage(ctx, x, phase: int):
    """A page-locked buffer holding x's bytes from byte ``phase`` (16-byte aligned base)."""
    raw = x.contiguous().view(_t().uint8).reshape(-1).cpu().numpy()
    buf = ctx.host_alloc(raw.size + phase + 64)
    buf[:] = 0
    buf[phase : phase + raw.size] = raw
    return buf


def _quantize(ctx, x, block, phase=0, dphase=0, split=None, given_a=None):
    """Weight x (CUDA, R x C) through the entries from a staging buffer at ``phase``: the amax (one call, or two
    split at element ``split``), then one copy with one band over every block, into a sentinel-padded destination at
    byte ``dphase``.  ``given_a``: no amax call and no band, the copy uses these a bits as they are.
    -> (q codes int64, s bits int64, a bits int64)"""
    torch = _t()
    R, C = x.shape
    ss = x.element_size()
    br, bc = min(block[0] or R, R), min(block[1] or C, C)
    n = -(-R // br) * -(-C // bc)
    buf = _stage(ctx, x, phase)
    out = torch.full((R * C + dphase + 32,), SENTINEL, dtype=torch.uint8, device="cuda")
    amax = torch.zeros(n, dtype=torch.float32, device="cuda")
    if given_a is not None:
        amax.copy_(given_a.to(torch.int32).view(torch.float32))
    scales = torch.full((n,), -1.0, dtype=torch.float32, device="cuda")
    seg = ([out.data_ptr()], [out.numel()], [0, 1])

    def box(e0, e1):
        return (0, dphase + e0, (e1 - e0) * ss, 1, phase + e0 * ss, (e1 - e0) * ss, _code(x.dtype), _lib.DT_F8E4M3,
                amax.data_ptr(), n, e0, R, C, block[0] or R, block[1] or C)

    whole = [box(0, R * C)]
    torch.cuda.synchronize()
    launches = ctx.launch_count
    if given_a is None:
        parts = [whole] if split is None else [[box(0, split)], [box(split, R * C)]]
        for p in parts:
            ctx.fp8_amax_boxes_from_host(*seg, p, buf, _current())
    bands = [] if given_a is not None else [(amax.data_ptr(), scales.data_ptr(), n)]
    ctx.copy_quant_boxes_from_host(*seg, whole, bands, buf, _current())
    torch.cuda.synchronize()
    assert ctx.launch_count - launches == (0 if given_a is not None else len(parts) + 1) + 1
    o = out.cpu()
    assert (o[:dphase] == SENTINEL).all() and (o[dphase + R * C :] == SENTINEL).all()
    ctx.host_free(buf)
    return (_bits(out[dphase : dphase + R * C]).reshape(R, C), _bits(scales), _bits(amax))


def _expect(x, block):
    """(q, s) of the integer reference on the device."""
    torch = _t()
    R, C = x.shape
    a, s = reference_block_scales(_bits(x).reshape(-1), x.dtype, R, C, block)
    br, bc = min(block[0] or R, R), min(block[1] or C, C)
    full = a.repeat_interleave(br, 0)[:R].repeat_interleave(bc, 1)[:, :C]
    return reference_quant(_bits(x).reshape(R, C), x.dtype, reference_multiplier(full)), s.reshape(-1), a.reshape(-1)


def _given(ctx, x_bits, src, a_bits, C=64):
    """Elements with their own a (block (1, 1)), through the copy alone; compared with reference_quant."""
    torch = _t()
    n = x_bits.numel()
    pad = (-n) % C
    x_bits = torch.cat([x_bits, torch.zeros(pad, dtype=torch.int64, device="cuda")])
    a_bits = torch.cat([a_bits, torch.full((pad,), 0x3F800000, dtype=torch.int64, device="cuda")])
    iv = torch.int32 if src == torch.float32 else torch.int16
    x = x_bits.to(torch.int32 if iv == torch.int32 else torch.int64).to(iv).view(src).reshape(-1, C)
    q, _, _ = _quantize(ctx, x, (1, 1), phase=6 if src != torch.float32 else 4, dphase=3, given_a=a_bits)
    want = reference_quant(x_bits, src, reference_multiplier(a_bits)).reshape(q.shape)
    bad = (q != want).nonzero()
    assert bad.numel() == 0, (bad[:5].tolist(), q.reshape(-1)[:8].tolist())


# ----------------------------------------------------------------------------------------- direct value sets


@pytest.mark.parametrize("src", ["float16", "bfloat16"])
def test_every_16_bit_pattern_under_every_structured_amax(ctx, src):
    torch = _t()
    dt = getattr(torch, src)
    x, a = sixteen_bit_pairs(dt, device="cuda")
    _given(ctx, x, dt, a)


def test_structured_and_random_f32_sets(ctx):
    torch = _t()
    x, a = structured_f32_pairs()
    _given(ctx, x.cuda(), torch.float32, a.cuda())
    x, a = random_f32_rows(1 << 20, 11, device="cuda")
    _given(ctx, x, torch.float32, a)


# ----------------------------------------------------------------------------------------- layouts and blocks


def _weight(R, C, dt, seed):
    torch = _t()
    g = torch.Generator(device="cuda").manual_seed(seed)
    w = (torch.randn(R, C, generator=g, device="cuda") * torch.exp2(torch.randint(-20, 20, (R, 1), generator=g,
                                                                                  device="cuda").float())).to(dt)
    return w


def _check(ctx, x, block, **kw):
    q, s, _ = _quantize(ctx, x, block, **kw)
    wq, ws, _ = _expect(x, block)
    assert torch_equal(q, wq) and torch_equal(s, ws), (block, kw)


def torch_equal(a, b):
    return bool(_t().equal(a, b))


@pytest.mark.parametrize("dtype", ["bfloat16", "float16", "float32"])
def test_every_source_and_destination_phase(ctx, dtype):
    torch = _t()
    dt = getattr(torch, dtype)
    ss = dt.itemsize
    x = _weight(67, 300, dt, 1)
    for phase in range(0, 16, ss):
        for dphase in (0, 1, 7, 15):
            _check(ctx, x, (128, 128), phase=phase, dphase=dphase)
    # rows that start at every phase inside the weight: an odd column count
    _check(ctx, _weight(131, 77, dt, 2), (64, 96), phase=ss, dphase=5)


@pytest.mark.parametrize("dtype", ["bfloat16", "float16", "float32"])
def test_nan_inf_signed_zero_zero_and_edge_blocks(ctx, dtype):
    torch = _t()
    dt = getattr(torch, dtype)
    x = _weight(300, 259, dt, 3)
    x[0, 0] = float("nan")
    x[130, 140] = float("inf")
    x[131, 10] = float("-inf")
    x[200:256, 0:128] = 0.0
    x[200, 5] = -0.0
    x[299, 258] = float("nan")
    x[257:, 256:] = -0.0
    for block in ((128, 128), (1, None), (None, None), (64, 96), (300, 1)):
        _check(ctx, x, block, phase=0 if dt == torch.float32 else 2)


def test_one_bands_amax_split_over_two_calls_equals_one_call(ctx):
    torch = _t()
    for dt, block in ((torch.bfloat16, (128, 128)), (torch.float32, (None, None)), (torch.float16, (64, 96))):
        x = _weight(200, 333, dt, 4)
        one = _quantize(ctx, x, block)
        for split in (1, 333 * 64 + 17, 200 * 333 - 5):
            two = _quantize(ctx, x, block, split=split)
            assert all(torch.equal(u, v) for u, v in zip(one, two)), split


def test_pitched_boxes_take_the_hull_path_in_both_kernels(ctx):
    """Two boxes of rows > 1 whose pitch (the weight's row) exceeds their width by 16 bytes or more (hull != 0): the
    left and right column ranges of a weight staged whole, each written packed; the cursors re-seek at every box row."""
    torch = _t()
    for dt, block, (R, C, w0), phase in ((torch.bfloat16, (128, 128), (300, 259, 130), 6),
                                         (torch.float32, (64, 96), (131, 200, 97), 12),
                                         (torch.float16, (1, None), (50, 333, 40), 2)):
        ss = dt.itemsize
        x = _weight(R, C, dt, 6)
        R_, C_ = block[0] or R, block[1] or C
        n = -(-R // min(R_, R)) * -(-C // min(C_, C))
        buf = _stage(ctx, x, phase)
        out = torch.full((R * C + 5 + 32,), SENTINEL, dtype=torch.uint8, device="cuda")
        amax = torch.zeros(n, dtype=torch.float32, device="cuda")
        scales = torch.zeros(n, dtype=torch.float32, device="cuda")
        seg = ([out.data_ptr()], [out.numel()], [0, 1])
        boxes = [(0, 5, w0 * ss, R, phase, C * ss, _code(dt), _lib.DT_F8E4M3, amax.data_ptr(), n, 0, R, C, R_, C_),
                 (0, 5 + R * w0, (C - w0) * ss, R, phase + w0 * ss, C * ss, _code(dt), _lib.DT_F8E4M3, amax.data_ptr(),
                  n, w0, R, C, R_, C_)]
        ctx.fp8_amax_boxes_from_host(*seg, boxes[1:], buf, _current())
        ctx.fp8_amax_boxes_from_host(*seg, boxes[:1], buf, _current())
        ctx.copy_quant_boxes_from_host(*seg, boxes, [(amax.data_ptr(), scales.data_ptr(), n)], buf, _current())
        torch.cuda.synchronize()
        q, s, _ = _expect(x, block)
        got = _bits(out)
        assert torch.equal(got[5 : 5 + R * w0].reshape(R, w0), q[:, :w0]), dt
        assert torch.equal(got[5 + R * w0 : 5 + R * C].reshape(R, C - w0), q[:, w0:]), dt
        assert torch.equal(_bits(scales), s), dt
        assert (got[:5] == SENTINEL).all() and (got[5 + R * C :] == SENTINEL).all()
        ctx.host_free(buf)


def test_bad_arguments_are_refused_before_anything_is_enqueued(ctx):
    torch = _t()
    x = _weight(16, 16, torch.bfloat16, 5)
    buf = _stage(ctx, x, 0)
    out = torch.full((256,), SENTINEL, dtype=torch.uint8, device="cuda")
    amax = torch.zeros(1, dtype=torch.float32, device="cuda")
    seg = ([out.data_ptr()], [out.numel()], [0, 1])
    good = [0, 0, 512, 1, 0, 512, _lib.DT_BF16, _lib.DT_F8E4M3, amax.data_ptr(), 1, 0, 16, 16, 128, 128]
    host_a = np.zeros(4, np.float32)
    for k, v, what in ((6, _lib.DT_F8E4M3, "an FP8 source"), (7, _lib.DT_BF16, "a non-E4M3 target"),
                       (13, 0, "a zero block"), (9, 0, "too few scales"), (8, amax.data_ptr() + 2, "unaligned a"),
                       (8, host_a.ctypes.data, "a in host memory"), (11, 15, "past R * C"), (2, 511, "odd width"),
                       (1, 250, "past the file")):
        b = list(good)
        b[k] = v
        launches = ctx.launch_count
        for call in (lambda: ctx.fp8_amax_boxes_from_host(*seg, [tuple(b)], buf, _current()),
                     lambda: ctx.copy_quant_boxes_from_host(*seg, [tuple(b)], [], buf, _current())):
            with pytest.raises(_lib.B200HashError):
                call()
        assert ctx.launch_count == launches, what
    for band, what in (((amax.data_ptr(), amax.data_ptr(), 0), "an empty band"),
                       ((amax.data_ptr() + 1, amax.data_ptr(), 1), "unaligned"),
                       ((host_a.ctypes.data, amax.data_ptr(), 1), "a in host memory")):
        launches = ctx.launch_count
        with pytest.raises(_lib.B200HashError):
            ctx.copy_quant_boxes_from_host(*seg, [tuple(good)], [band], buf, _current())
        assert ctx.launch_count == launches, what
    torch.cuda.synchronize()
    assert (out == SENTINEL).all() and (amax == 0).all()
    ctx.host_free(buf)


# --------------------------------------------------------------------------------------------- end to end


def _stack(layers=11, h=2048, kv=320, m=5632):
    """About 1 GB of bf16: Llama-shaped projections (the KV sides not multiples of 128) and norms."""
    torch = _t()
    g = torch.Generator(device="cuda").manual_seed(9)
    sd = {"model.embed_tokens.weight": torch.randn(1000, h, generator=g, device="cuda").to(torch.bfloat16)}
    for i in range(layers):
        p = f"model.layers.{i}."
        shapes = {"self_attn.q_proj": (h, h), "self_attn.k_proj": (kv, h), "self_attn.v_proj": (kv, h),
                  "self_attn.o_proj": (h, h), "mlp.gate_proj": (m, h), "mlp.up_proj": (m, h),
                  "mlp.down_proj": (h, m)}
        for k, (R, C) in shapes.items():
            sd[p + k + ".weight"] = (torch.randn(R, C, generator=g, device="cuda") * 0.02).to(torch.bfloat16)
        sd[p + "input_layernorm.weight"] = torch.randn(h, generator=g, device="cuda").to(torch.bfloat16)
    return sd


async def _grown(fn):
    torch = _t()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = await fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


def _held(n: int) -> int:
    """The most HBM torch's caching allocator counts for an n-byte tensor: a request over 1 MiB takes a block of up to
    n rounded up to 2 MiB (a remainder of 1 MiB or less is not split off: 11 534 336 bytes take 12 MiB), a smaller one
    n rounded up to 512 bytes."""
    return -(-n // (2 * MiB)) * 2 * MiB if n > MiB else -(-n // 512) * 512


def _same(got: dict, want: dict):
    torch = _t()
    assert sorted(got) == sorted(want)
    for k, v in want.items():
        assert got[k].dtype == v.dtype and got[k].shape == v.shape, k
        assert torch.equal(got[k].view(torch.uint8), v.view(torch.uint8)), k


def test_a_1gb_bf16_stack_reads_back_quantized_as_its_fp8_export(gpu_backend):
    torch = _t()
    sd = _stack()
    names = [k for k in sd if k.endswith("proj.weight")]

    async def run():
        async with running_volume_server(blob_utils.BLOCK_SIZE) as (stub, _):
            client = types.SimpleNamespace(stub=stub)
            for where, kw in (("/bf16", {}), ("/fp8", {"fp8": names})):
                shards = device_file.safetensors_shards(sd, max_shard_size="300MB", **kw)
                assert len(shards.files) >= (2 if kw else 3)  # the FP8 image is about half the bf16 one
                async with volume.VolumeUploadContextManager2("vo-g", client) as batch:
                    shards.put(batch, where)
                del shards
            want = await volume.read_safetensors_sharded(client, "vo-g", "/fp8/model.safetensors.index.json")
            for staging in (256 << 20, 4 * blob_utils.BLOCK_SIZE):
                got, growth = await _grown(lambda: volume.read_safetensors_sharded(
                    client, "vo-g", "/bf16/model.safetensors.index.json", fp8=names, staging_bytes=staging))
                _same(got, want)
                keys = list(got)
                assert all(keys[keys.index(n) + 1] == n + "_scale_inv" for n in names)
                results = sum(_held(t.numel() * t.element_size()) for t in got.values())
                amax = sum(got[n + "_scale_inv"].numel() * 4 for n in names)
                assert growth <= results + amax + 8 * MiB, (growth, results, amax)
                del got
            for n in names[:7]:
                q, s = fp8_block_reference(sd[n])
                assert torch.equal(want[n].view(torch.uint8), q.view(torch.uint8)), n
                assert torch.equal(want[n + "_scale_inv"], s), n

    asyncio.run(run())


def test_f32_and_f16_sources_channel_and_tensor_scales_and_into(gpu_backend):
    torch = _t()
    g = torch.Generator(device="cuda").manual_seed(10)
    sd = {"a.weight": (torch.randn(1000, 1536, generator=g, device="cuda")).to(torch.float16),
          "b.weight": torch.randn(320, 2048, generator=g, device="cuda"),
          "c.weight": (torch.randn(777, 1000, generator=g, device="cuda") * 1e3).to(torch.bfloat16),
          "norm": torch.randn(2048, generator=g, device="cuda")}
    names = ["a.weight", "b.weight", "c.weight"]

    async def run():
        async with running_volume_server(blob_utils.BLOCK_SIZE) as (stub, _):
            client = types.SimpleNamespace(stub=stub)
            shards = device_file.safetensors_shards(sd, max_shard_size="1MB")
            async with volume.VolumeUploadContextManager2("vo-g", client) as batch:
                shards.put(batch, "/src")
            for block in ((1, None), (None, None), (128, 128)):
                exp = device_file.safetensors_shards(sd, max_shard_size="1MB", fp8=names, scale_block=block,
                                                     scale_suffix="_scale")
                where = f"/fp8-{block[0]}-{block[1]}"
                async with volume.VolumeUploadContextManager2("vo-g", client) as batch:
                    exp.put(batch, where)
                cast = {"norm": torch.float16} if block == (1, None) else None
                want = await volume.read_safetensors_sharded(client, "vo-g", where + "/model.safetensors.index.json",
                                                             dtype=cast)
                kw = dict(fp8=names, scale_block=block, scale_suffix="_scale", dtype=cast)
                got = await volume.read_safetensors_sharded(client, "vo-g", "/src/model.safetensors.index.json", **kw)
                _same(got, want)
                into = {k: torch.empty_like(v) for k, v in want.items()}
                got = await volume.read_safetensors_sharded(client, "vo-g", "/src/model.safetensors.index.json",
                                                            into=into, **kw)
                assert all(got[k] is into[k] for k in into)
                _same(got, want)
                for n in names:
                    q, s = fp8_block_reference(sd[n], block)
                    assert torch.equal(got[n].view(torch.uint8), q.view(torch.uint8)), (n, block)
                    assert torch.equal(got[n + "_scale"], s), (n, block)

    asyncio.run(run())
