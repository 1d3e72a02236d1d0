"""FP8 export on the H100: ``b200h_fp8_block_scales`` and the quantizing copies against torch on CUDA running the
widely copied ``per_block_cast_to_fp8`` form, every F32 pattern up to 448 and every F16 / BF16 pattern through the
quantizing store, the kernel's word paths, the hash tables against the pre-quantized file, and an upload of a
Llama-shaped stack that reads back bit for bit."""
import asyncio
import random
import types

import numpy as np
import pytest

from modal_client_b200 import DeviceFile, _lib, blob_utils, stage_ranges, volume
from tests.volume_read_server import running_volume_server

pytestmark = pytest.mark.gpu

MiB, GiB = 1 << 20, 1 << 30
SENTINEL = 0xC3


def fp8_block_reference(w, block=(128, 128)):
    """q, s of a 2-D float32 / float16 / bfloat16 CUDA tensor (numel > 0): per_block_cast_to_fp8 as DeepGEMM's tests
    write it, with edge blocks padded by zeros and None meaning the whole dimension."""
    import torch

    R, C = w.shape
    bR, bC = (R if block[0] is None else block[0]), (C if block[1] is None else block[1])
    gR, gC = -(-R // bR), -(-C // bC)
    padded = w.new_zeros(gR * bR, gC * bC)
    padded[:R, :C] = w
    v = padded.view(gR, bR, gC, bC)
    amax = v.abs().float().amax(dim=(1, 3), keepdim=True).clamp(1e-4)
    q = (v * (448.0 / amax)).to(torch.float8_e4m3fn).view(gR * bR, gC * bC)[:R, :C].contiguous()
    return q, (amax / 448.0).view(gR, gC)


def _codes():
    import torch

    return {torch.float32: _lib.DT_F32, torch.float16: _lib.DT_F16, torch.bfloat16: _lib.DT_BF16}


def _current():
    import torch

    return torch.cuda.current_stream().cuda_stream or 1


def _bits(t):
    import torch

    return t.contiguous().view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0, pinned_bytes=64 << 20, device_bytes=512 << 20)
    yield c
    c.close()


def _scales(ctx, weights, block):
    """(s, a) of every weight through one fp8_block_scales call."""
    import torch

    grids = [(-(-w.shape[0] // (block[0] or w.shape[0])), -(-w.shape[1] // (block[1] or w.shape[1]))) for w in weights]
    amax = torch.full((sum(a * b for a, b in grids),), 1.5, dtype=torch.float32, device="cuda")  # not zeros: the call
    out, jobs, at = [], [], 0
    for w, (g0, g1) in zip(weights, grids):
        s = torch.empty((g0, g1), dtype=torch.float32, device="cuda")
        a = amax[at : at + g0 * g1].view(g0, g1)
        jobs.append((w.data_ptr(), _codes()[w.dtype], w.shape[0], w.shape[1], block[0] or w.shape[0],
                     block[1] or w.shape[1], s.data_ptr(), a.data_ptr()))
        out.append((s, a))
        at += g0 * g1
    ctx.fp8_block_scales(jobs, _current())
    torch.cuda.synchronize()
    return out


def _weights(seed, dtype):
    """Weights of odd shapes with NaN, inf and all-zero blocks among them."""
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for R, C in [(1, 1), (3, 17), (129, 257), (300, 1000), (256, 128), (77, 4099), (5000, 3)]:
        w = (torch.randn(R, C, device="cuda", generator=g) * 10 ** (seed % 5 - 2)).to(dtype)
        out.append(w)
    w = torch.randn(300, 300, device="cuda", generator=g).to(dtype)
    w[:128, :128] = 0  # an all-zero block
    w[5, 200] = float("nan")
    w[200, 5] = float("inf")
    w[250, 250] = -float("inf")
    w[140, 140] = 1e-30 if dtype != torch.float16 else 0
    out.append(w)
    return out


@pytest.mark.parametrize("block", [(128, 128), (64, 32), (1, None), (None, None), (7, 5), (1, 1)])
@pytest.mark.parametrize("dtype", ["float32", "float16", "bfloat16"])
def test_scales_equal_torch_for_every_block_form(ctx, block, dtype):
    import torch

    ws = _weights(len(dtype) + 7 * (block[0] or 0), getattr(torch, dtype))
    for w, (s, a) in zip(ws, _scales(ctx, ws, block)):
        _, s_ref = fp8_block_reference(w, block)
        assert torch.equal(_bits(s), _bits(s_ref)), (w.shape, block)
        assert not torch.isnan(a).any() or torch.isnan(w).any()


def test_a_per_tensor_scale_over_2_27_elements(ctx):
    import torch

    w = torch.randn(1 << 14, 1 << 13, device="cuda", dtype=torch.bfloat16)
    w[12345, 678] = 1000.0
    (s, _), = _scales(ctx, [w], (None, None))
    _, s_ref = fp8_block_reference(w, (None, None))
    assert torch.equal(_bits(s), _bits(s_ref))


def _quantize(ctx, w, a, block):
    """q of weight w with clamped amax values a (one F32 per block) through one copy_scaled_ranges call into device
    memory; -> q as uint8."""
    import torch

    R, C = w.shape
    n = R * C
    dst = torch.full((n + 256,), SENTINEL, dtype=torch.uint8, device="cuda")
    ctx.copy_scaled_ranges([w.data_ptr()], [n * w.element_size()], [_codes()[w.dtype]], [_lib.DT_F8E4M3],
                           [(a.data_ptr(), a.numel(), R, C, block[0], block[1])], [0, 1], [(0, 0, n)], dst, [128],
                           _current())
    torch.cuda.synchronize()
    assert (dst[:128] == SENTINEL).all() and (dst[128 + n :] == SENTINEL).all()
    return dst[128 : 128 + n]


def _torch_q(w, a, block):
    """torch's q on CUDA for clamped amax values a: (x * (448 / a_expanded)).to(e4m3)."""
    import torch

    R, C = w.shape
    m = (448.0 / a).repeat_interleave(block[0], 0)[:R].repeat_interleave(block[1], 1)[:, :C]
    return (w * m).to(torch.float8_e4m3fn).view(torch.uint8).reshape(-1)


def test_every_f32_pattern_up_to_448_quantizes_as_torch_does_with_m_1(ctx):
    import torch

    top = 0x43E00000  # 448.0
    chunk = 1 << 27
    C = 1 << 12
    a = torch.full((chunk // C, 1), 448.0, dtype=torch.float32, device="cuda")
    for sign in (0, 1 << 31):
        for lo in range(0, top + 1, chunk):
            bits = torch.arange(lo, lo + chunk, dtype=torch.int64, device="cuda").clamp_(max=top) | sign
            w = bits.to(torch.int32).view(torch.float32).view(-1, C)
            assert torch.equal(_quantize(ctx, w, a, (1, C)), _torch_q(w, a, (1, C)))
            assert torch.equal(_torch_q(w, a, (1, C)), w.reshape(-1).to(torch.float8_e4m3fn).view(torch.uint8))


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_every_16_bit_pattern_quantizes_as_torch_does_under_several_amax_values(ctx, dtype):
    import torch

    dt = getattr(torch, dtype)
    every = torch.arange(-(1 << 15), 1 << 15, dtype=torch.int32, device="cuda").to(torch.int16).view(dt)
    for amax in (448.0, 1.0, 0.5, 3.0, 1e-4, 1000.0, 65504.0, 1e30, 0.013, float("inf"), float("nan")):
        if amax != amax:  # a block holding a NaN: every pattern
            x = every
        elif amax == float("inf"):  # a block holding an infinity: every pattern but the NaNs
            x = every[~torch.isnan(every)]
        else:  # the patterns a block of this amax can hold
            x = every[every.float().abs() <= amax]
        n = x.numel() - x.numel() % 64
        w = x[:n].view(-1, 64)
        a = torch.full((w.shape[0], 1), amax, dtype=torch.float32, device="cuda")
        assert torch.equal(_quantize(ctx, w, a, (1, 64)), _torch_q(w, a, (1, 64))), amax


# ------------------------------------------------------------------------------------------------ the file


def _ref_dict(sd, fp8, block, suffix="_scale_inv", dtype=None):
    """The caller's dict with every fp8 weight replaced by q and its scale inserted right after it, the others
    converted by ``dtype`` -- on the CPU, for safetensors.torch.save."""
    out = {}
    for n, t in sd.items():
        if n in fp8:
            q, s = fp8_block_reference(t, block)
            out[n], out[n + suffix] = q.cpu(), s.cpu()
        elif dtype is not None and t.is_floating_point() and t.dtype != dtype:
            out[n] = t.to(dtype).cpu()
        else:
            out[n] = t.cpu()
    return out


def _phased(t, k):
    """t's values in a tensor whose data starts k elements into a fresh allocation (source phase k * itemsize)."""
    import torch

    buf = torch.empty(t.numel() + k, dtype=t.dtype, device="cuda")
    v = buf[k : k + t.numel()].view(t.shape)
    v.copy_(t)
    return v


def _stack(seed, dtype, phases=True):
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    sd = {"embed": torch.randn(333, 40, device="cuda", generator=g).to(dtype)}
    for i, (R, C) in enumerate([(200, 136), (97, 131), (256, 256), (33, 1000), (130, 17)]):
        w = (torch.randn(R, C, device="cuda", generator=g) * 3).to(dtype)
        sd[f"l{i}.w"] = _phased(w, (i * 3 + seed) % (16 // w.element_size())) if phases else w
        sd[f"l{i}.norm"] = torch.ones(C, device="cuda", dtype=dtype)
    sd["l2.w"][:128, :128] = 0
    sd["steps"] = torch.arange(11, device="cuda")
    return sd


@pytest.mark.parametrize("block", [(128, 128), (64, 32), (1, None), (None, None), (7, 5)])
@pytest.mark.parametrize("dtype", ["float32", "float16", "bfloat16"])
def test_file_bytes_equal_safetensors_save_of_the_quantized_dict(ctx, block, dtype):
    import torch
    from safetensors.torch import save

    dt = getattr(torch, dtype)
    for phase in range(16 // dt.itemsize):
        sd = _stack(phase, dt)
        fp8 = [n for n in sd if n.endswith(".w")]
        f = DeviceFile.safetensors(sd, {"format": "pt"}, fp8=fp8, scale_block=block, ctx=ctx)
        want = save(_ref_dict(sd, fp8, block), {"format": "pt"})
        assert f.nbytes == len(want)
        assert f.read() == want
        rng = random.Random(phase)
        for _ in range(40):  # reads at any image byte, through the bounce buffer
            pos, n = rng.randrange(len(want)), rng.choice([1, 15, 16, 17, 33, rng.randrange(1, 5000)])
            f.seek(pos)
            assert f.read(n) == want[pos : pos + n]


def test_dtype_and_scale_suffix_mix_and_device_and_pinned_ranges_keep_their_sentinels(ctx):
    import torch
    from safetensors.torch import save

    sd = _stack(3, torch.float32)
    fp8 = ["l0.w", "l3.w", "l4.w"]
    f = DeviceFile.safetensors(sd, fp8=fp8, scale_block=(1, None), scale_suffix="_scale", dtype=torch.bfloat16, ctx=ctx)
    want = np.frombuffer(save(_ref_dict(sd, fp8, (1, None), "_scale", torch.bfloat16)), np.uint8)
    assert f.nbytes == want.size
    rng = random.Random(5)
    ranges = [(0, 0, want.size)] + [(0, o, rng.randrange(0, min(9000, want.size - o)))
                                    for o in (rng.randrange(want.size) for _ in range(200))]
    offsets, at = [], 128
    for _, _, n in ranges:
        offsets.append(at)
        at += -(-n // 128) * 128 + 128
    pinned = ctx.host_alloc(at)
    try:
        for dst in (pinned, torch.full((at,), SENTINEL, dtype=torch.uint8, device="cuda")):
            if isinstance(dst, np.ndarray):
                dst[:] = SENTINEL
            stage_ranges([f], ranges, dst, offsets, ctx=ctx).wait()
            got = dst if isinstance(dst, np.ndarray) else dst.cpu().numpy()
            clean = np.ones(at, bool)
            for (_, o, n), p in zip(ranges, offsets):
                assert np.array_equal(got[p : p + n], want[o : o + n]), (o, n)
                clean[p : p + n] = False
            assert (got[clean] == SENTINEL).all()
    finally:
        ctx.host_free(pinned)


@pytest.mark.parametrize("part_len", [4096 + 3, MiB])
def test_hash_tables_equal_those_of_the_prequantized_file(part_len):
    import torch

    small = _lib.Context(0, pinned_bytes=16 << 20, device_bytes=24 << 20)
    try:
        g = torch.Generator(device="cuda").manual_seed(part_len)
        sd = {f"w{i}": torch.randn(1000 + i, 2048 + 7 * i, device="cuda", generator=g).to(torch.bfloat16)
              for i in range(12)}
        sd["bias"] = torch.randn(5000, device="cuda")
        fp8 = [n for n in sd if n.startswith("w")]
        f = DeviceFile.safetensors(sd, fp8=fp8, ctx=small)
        pre = {k: v.cuda() for k, v in _ref_dict(sd, fp8, (128, 128)).items()}
        h = DeviceFile.safetensors(pre, ctx=small)
        for flags in (_lib.SHA256 | _lib.MD5, _lib.SHA256 | _lib.TRIM_ZEROS):
            a, b = f.hash_parts(part_len, flags, ctx=small), h.hash_parts(part_len, flags, ctx=small)
            assert all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(a, b))
    finally:
        small.close()


def test_construction_launches_two_kernels_and_one_memset_whatever_the_weights(ctx):
    import torch
    from torch.profiler import ProfilerActivity, profile

    sd = {f"w{i}": torch.randn(64 + i, 300, device="cuda") for i in range(40)}
    torch.cuda.synchronize()
    launches = ctx.launch_count
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        DeviceFile.safetensors(sd, fp8=list(sd), ctx=ctx)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type.name == "CUDA"]
    memsets = [n for n in names if "Memset" in n]
    kernels = [n for n in names if "Memset" not in n and "Memcpy" not in n]
    assert len(memsets) == 1 and len(kernels) == 2, names
    assert any("fp8_amax_kernel" in n for n in kernels) and any("fp8_finalize_kernel" in n for n in kernels)
    assert ctx.launch_count - launches == 2


# ------------------------------------------------------------------------------------------------ end to end


def _llama(total, dtype):
    """A Llama-shaped bf16 stack of about ``total`` bytes: embeddings, per layer q/k/v/o and gate/up/down, norms."""
    import torch

    g = torch.Generator(device="cuda").manual_seed(1)
    H, F, V = 2048, 5632, 32000
    sd = {"model.embed_tokens.weight": torch.randn(V, H, device="cuda", generator=g).to(dtype)}
    i = 0
    while sum(t.numel() * t.element_size() for t in sd.values()) < total:
        p = f"model.layers.{i}."
        for n, shape in (("self_attn.q_proj", (H, H)), ("self_attn.k_proj", (H // 4, H)), ("self_attn.v_proj", (H // 4, H)),
                         ("self_attn.o_proj", (H, H)), ("mlp.gate_proj", (F, H)), ("mlp.up_proj", (F, H)),
                         ("mlp.down_proj", (H, F))):
            sd[p + n + ".weight"] = (torch.randn(*shape, device="cuda", generator=g) * 0.02).to(dtype)
        sd[p + "input_layernorm.weight"] = torch.ones(H, device="cuda", dtype=dtype)
        i += 1
    return sd


@pytest.mark.parametrize("budget_mib", [None, 256])
def test_a_2gib_llama_stack_exports_as_fp8_and_reads_back_bit_for_bit(gpu_backend, budget_mib):
    import torch
    from safetensors.torch import save

    sd = _llama(2 * GiB, torch.bfloat16)
    fp8 = [n for n, t in sd.items() if t.dim() == 2 and "embed" not in n]
    grid = sum(-(-sd[n].shape[0] // 128) * -(-sd[n].shape[1] // 128) for n in fp8)
    budget = budget_mib * MiB if budget_mib else None
    ref = _ref_dict(sd, fp8, (128, 128))

    async def go():
        async with running_volume_server(blob_utils.BLOCK_SIZE) as (stub, _):
            client = types.SimpleNamespace(stub=stub)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            f = DeviceFile.safetensors(sd, fp8=fp8)
            batch = volume.VolumeUploadContextManager2("vo-f", client, device_staging_bytes=budget)
            async with batch:
                batch.put_file(f, "/m.safetensors")
            torch.cuda.synchronize()
            growth = torch.cuda.max_memory_allocated() - base
            back = await volume.read_safetensors(client, "vo-f", "/m.safetensors")
            deq = await volume.read_safetensors(client, "vo-f", "/m.safetensors", dtype=torch.bfloat16,
                                                scales=volume.fp8_scales(list(ref)))
            return growth, back, deq, f.nbytes

    growth, back, deq, nbytes = asyncio.run(go())
    assert nbytes == len(save(ref))
    assert growth <= 2 * grid * 4 + 8 * MiB, growth  # the scales, the amax values, the tables and wave work
    assert set(back) == set(ref)
    for k, v in ref.items():
        assert torch.equal(_bits(back[k].cpu()), _bits(v)), k
    for n in fp8:
        s = ref[n + "_scale_inv"].cuda().repeat_interleave(128, 0)[: sd[n].shape[0]].repeat_interleave(128, 1)[:, : sd[n].shape[1]]
        assert torch.equal(_bits(deq[n]), _bits((back[n].float() * s).to(torch.bfloat16))), n


def test_a_sharded_fp8_export_equals_the_hub_layout_of_the_quantized_dict(gpu_backend):
    import json
    import tempfile

    import torch
    from safetensors.torch import load_file

    sd = _stack(1, torch.bfloat16, phases=False)
    fp8 = [n for n in sd if n.endswith(".w")]
    # l0.w (200 x 136 elements, one byte each) fills a shard of its own, so its scale opens the next one
    shards = DeviceFile.safetensors_shards(sd, fp8=fp8, max_shard_size=200 * 136)
    ref = _ref_dict(sd, fp8, (128, 128))
    assert shards.index is not None
    weight_map = json.loads(shards.index[1])["weight_map"]
    assert set(weight_map) == set(ref)
    assert any(weight_map[n] != weight_map[n + "_scale_inv"] for n in fp8)  # a scale in another shard
    with tempfile.TemporaryDirectory() as d:
        for name, f in shards.files.items():
            p = f"{d}/{name}"
            open(p, "wb").write(f.read())
            for k, v in load_file(p).items():
                assert weight_map[k] == name and torch.equal(_bits(v), _bits(ref[k])), k
