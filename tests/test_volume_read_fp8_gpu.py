"""GPU: FP8 weights dequantized with their block scales on the way from page-locked host memory into device files
(``b200h_copy_scaled_boxes_from_host``, ``load_scaled_boxes_kernel``), checked bit for bit against torch's CUDA
expression ``(W.float() * S.float().repeat_interleave(bR, 0)[:R].repeat_interleave(bC, 1)[:, :C]).to(T)``.

Every FP8 pattern of both formats meets a scale set (signed zeros, every power of two from 2^-149 to 2^127 with both
signs, so products go subnormal and overflow, +-inf, NaN, random scales) into all three targets; a subset does so
with F16 and BF16 scales.  Layouts force each path of the store step: the ring fast path at every source and
destination phase, words across block-column and tensor-row edges, the element loop, 64 KiB tile seams, 1 000-row
boxes and 10 000 boxes in one call, with sentinels around every destination, one launch per call and stream order.
Every rejected argument is refused before anything is enqueued.  End to end, a ~1 GB FP8 stack exported with
``safetensors_shards`` is read back over the loopback server with ``scales=`` whole and as rank 3 of 8's slices, with
HBM growing by no more than the results, the scales and 8 MiB.  A NaN element or product gives the NaN of
``NAN_POLICY``."""
import asyncio
import math
import types

import numpy as np
import pytest

from modal_client_b200 import _lib, blob_utils, device_file, volume
from tests.volume_read_server import running_volume_server

pytestmark = pytest.mark.gpu

MiB = 1 << 20
SENTINEL = 0xC3
# the NaN every NaN element or product gives, per target (bits): the NaN of the paired conversion intrinsics for 16-bit
# targets and of FMUL for F32
NAN_POLICY = {_lib.DT_F32: 0x7FFFFFFF, _lib.DT_F16: 0x7FFF, _lib.DT_BF16: 0x7FFF}


def _t():
    import torch

    return torch


def _dt(code):
    torch = _t()
    return {_lib.DT_F32: torch.float32, _lib.DT_F16: torch.float16, _lib.DT_BF16: torch.bfloat16,
            _lib.DT_F8E4M3: torch.float8_e4m3fn, _lib.DT_F8E5M2: torch.float8_e5m2}[code]


def _iv(code):
    torch = _t()
    return torch.int32 if code == _lib.DT_F32 else torch.int16


TARGETS = [_lib.DT_BF16, _lib.DT_F16, _lib.DT_F32]
FORMATS = [_lib.DT_F8E4M3, _lib.DT_F8E5M2]


def reference(w, s, block, tc):
    """torch's CUDA dequantization of the FP8 CUDA tensor w (R x C) with scales s, blocks ``block`` (None: whole)."""
    R, C = w.shape
    br, bc = block[0] or R, block[1] or C
    full = s.float().reshape(-(-R // br), -(-C // bc)).repeat_interleave(br, 0)[:R].repeat_interleave(bc, 1)[:, :C]
    return (w.float() * full).to(_dt(tc))


def _current():
    return _t().cuda.current_stream().cuda_stream or 1


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0, pinned_bytes=64 << 20, device_bytes=512 << 20)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pinned(ctx):
    buf = ctx.host_alloc(256 * MiB)
    yield buf
    _t().cuda.synchronize()
    ctx.host_free(buf)


def same_or_policy(got, want, tc, where=""):
    """got == want bit for bit where want is not NaN; got is NAN_POLICY's NaN where want is NaN."""
    torch = _t()
    nan = want.isnan()
    g, w = got.view(_iv(tc)), want.view(_iv(tc))
    bad = (g != w) & ~nan
    if bad.any():
        k = int(bad.nonzero()[0])
        raise AssertionError(f"{where}: {int(bad.sum())} elements differ, first at {k}: got {int(g[k]) & 0xFFFFFFFF:#x}, "
                             f"torch {int(w[k]) & 0xFFFFFFFF:#x}")
    nan_bits = (g[nan].to(torch.int64) & ((1 << (8 * got.element_size())) - 1))
    assert (nan_bits == NAN_POLICY[tc]).all(), (where, sorted({hex(int(x)) for x in nan_bits.unique()[:8]}))


def call(ctx, pinned, boxes, out_bytes, stream=None):
    """ONE copy_scaled_boxes_from_host call into a fresh device buffer of ``out_bytes`` (sentinel-filled); -> it."""
    torch = _t()
    out = torch.full((out_bytes,), SENTINEL, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    launches = ctx.launch_count
    ctx.copy_scaled_boxes_from_host([out.data_ptr()], [out.numel()], [0, 1], boxes, pinned, stream or _current())
    torch.cuda.synchronize()
    assert ctx.launch_count == launches + (1 if any(b[2] * b[3] for b in boxes) else 0)
    return out


def box(off, width, rows, src_off, pitch, fc, tc, s, sc, first, R, C, block):
    """A box tuple of ``_lib.Context.copy_scaled_boxes_from_host``."""
    br, bc = block[0] or R, block[1] or C
    return (0, off, width, rows, src_off, pitch, fc, tc, s.data_ptr(), sc, s.numel(), first, R, C, br, bc)


def stage(pinned, at, w):
    """The FP8 CUDA tensor w's bytes to pinned[at:]."""
    raw = w.view(_t().uint8).reshape(-1).cpu().numpy()
    pinned[at : at + raw.size] = raw
    return raw.size


def scale_set(g):
    torch = _t()
    p2 = [2.0 ** e for e in range(-149, 128)]
    vals = [0.0, -0.0] + p2 + [-x for x in p2] + [math.inf, -math.inf, math.nan, 448.0, 1 / 448.0, 3.0 * 2 ** -140]
    rnd = (torch.rand(64, generator=g) * 2 - 1) * 2.0 ** torch.randint(-30, 30, (64,), generator=g).float()
    return torch.cat([torch.tensor(vals, dtype=torch.float32), rnd]).cuda()


# --------------------------------------------------------------------------------------------- values


@pytest.mark.parametrize("fc", FORMATS)
def test_every_fp8_pattern_times_the_scale_set_into_every_target(ctx, pinned, fc):
    """Row i of W holds all 256 patterns; its per-channel scale is scale i of the set.  F32 scales into all three
    targets; F16 and BF16 scales (the set rounded to them) into BF16 and F32."""
    torch = _t()
    g = torch.Generator().manual_seed(1)
    s32 = scale_set(g)
    R, C = s32.numel(), 256
    w = torch.arange(256, dtype=torch.uint8, device="cuda").repeat(R, 1).view(_dt(fc))
    n = stage(pinned, 0, w)
    cases = [(_lib.DT_F32, t) for t in TARGETS] + [(sc, t) for sc in (_lib.DT_F16, _lib.DT_BF16)
                                                   for t in (_lib.DT_BF16, _lib.DT_F32)]
    for sc, tc in cases:
        s = s32.to(_dt(sc))
        ds = _dt(tc).itemsize
        # one run (the fast path at phase 0), and again at source phase 5 with a 2-element destination phase
        for sp, dq in ((0, 0), (5, 2)):
            stage(pinned, sp, w)
            out = call(ctx, pinned, [box(dq * ds, n, 1, sp, n, fc, tc, s, sc, 0, R, C, (1, None))], (n + 8) * ds)
            want = reference(w, s, (1, None), tc).reshape(-1)
            same_or_policy(out[dq * ds : (dq + n) * ds].view(_dt(tc)), want, tc, (fc, sc, tc, sp))
            assert (out[: dq * ds] == SENTINEL).all() and (out[(dq + n) * ds :] == SENTINEL).all()


def test_nan_policy_of_every_nan_input(ctx, pinned):
    """A NaN element (every NaN pattern of both formats) times a finite scale, and a finite element times a NaN
    scale, give NAN_POLICY's NaN in every target."""
    torch = _t()
    for fc in FORMATS:
        pats = torch.arange(256, dtype=torch.uint8, device="cuda")
        nan_pats = pats[pats.view(_dt(fc)).float().isnan()]
        w = torch.cat([nan_pats, torch.full((8,), 0x38, dtype=torch.uint8, device="cuda")]).view(_dt(fc))[None]
        C = w.shape[1]
        n = stage(pinned, 0, w)
        for tc in TARGETS:
            for sv in (1.5, math.nan):
                s = torch.tensor([sv], device="cuda")
                out = call(ctx, pinned, [box(0, n, 1, 0, n, fc, tc, s, _lib.DT_F32, 0, 1, C, (None, None))],
                           n * _dt(tc).itemsize)
                got = out.view(_iv(tc)).to(torch.int64) & ((1 << (8 * _dt(tc).itemsize)) - 1)
                want_nan = torch.ones(C, dtype=torch.bool, device="cuda") if sv != sv else \
                    torch.arange(C, device="cuda") < nan_pats.numel()
                assert (got[want_nan] == NAN_POLICY[tc]).all(), (fc, tc, sv, got[want_nan].unique())
                assert not out.view(_dt(tc))[~want_nan].isnan().any()


# --------------------------------------------------------------------------------------------- paths


def _random_fp8(shape, fc, g):
    torch = _t()
    return torch.randint(0, 256, shape, generator=g, dtype=torch.uint8).cuda().view(_dt(fc))


@pytest.mark.parametrize("tc", TARGETS)
def test_ring_path_at_every_source_and_destination_phase(ctx, pinned, tc):
    """One row of 1000 elements, starting at column 3 of row 5 of a 300 x 1003 weight in 128 x 128 blocks, staged at
    source phases 0..15 and written at every destination element phase."""
    torch = _t()
    g = torch.Generator().manual_seed(2)
    ds = _dt(tc).itemsize
    for fc in FORMATS:
        R, C = 300, 1003
        w = _random_fp8((R, C), fc, g)
        s = (torch.rand(3, 8, generator=g) * 4 - 2).cuda()
        want = reference(w, s, (128, 128), tc)[5, 3:]
        row = w[5, 3:].contiguous()
        for sp in range(16):
            n = stage(pinned, 4096 + sp, row)
            for dq in range(16 // ds):
                out = call(ctx, pinned, [box(dq * ds, n, 1, 4096 + sp, n, fc, tc, s, _lib.DT_F32, 5 * C + 3, R, C,
                                             (128, 128))], (n + 16) * ds)
                same_or_policy(out[dq * ds : (dq + n) * ds].view(_dt(tc)), want, tc, (fc, sp, dq))
                assert (out[: dq * ds] == SENTINEL).all() and (out[(dq + n) * ds :] == SENTINEL).all()


@pytest.mark.parametrize("tc", TARGETS)
def test_words_across_block_and_row_edges_and_the_element_loop(ctx, pinned, tc):
    """Column slices of a 257 x 300 weight (rows staged at the weight's pitch) with odd bounds, in blocks (128, 128),
    (64, 32), (1, None) and (None, None): words cross block-column edges; narrow slices (1..9 columns) and box ends go
    through the element loop; runs of whole rows cross tensor-row edges inside a word."""
    torch = _t()
    g = torch.Generator().manual_seed(3)
    ds = _dt(tc).itemsize
    R, C = 257, 300
    for fc in FORMATS:
        w = _random_fp8((R, C), fc, g)
        n = stage(pinned, 7, w)
        for block in ((128, 128), (64, 32), (1, None), (None, None)):
            sr, sc = -(-R // (block[0] or R)), -(-C // (block[1] or C))
            s = ((torch.rand(sr, sc, generator=g) * 4 - 2) * 2.0 ** torch.randint(-8, 8, (sr, sc), generator=g)).cuda()
            ref = reference(w, s, block, tc)
            for r0, r1, c0, c1 in ((0, R, 0, C), (3, 250, 31, 161), (1, 200, 127, 130), (0, R, 64, 65),
                                   (9, 17, 5, 14), (100, 101, 0, C), (2, 255, 33, 41)):
                rows, width = r1 - r0, c1 - c0
                out = call(ctx, pinned, [box(ds, width, rows, 7 + r0 * C + c0, C, fc, tc, s, _lib.DT_F32,
                                             r0 * C + c0, R, C, block)], (rows * width + 2) * ds)
                got = out[ds : ds + rows * width * ds].view(_dt(tc))
                same_or_policy(got, ref[r0:r1, c0:c1].reshape(-1), tc, (fc, block, r0, r1, c0, c1))
                assert (out[:ds] == SENTINEL).all() and (out[ds + rows * width * ds :] == SENTINEL).all()
            # a run of rows 10 .. 20, whole: words cross tensor-row edges
            out = call(ctx, pinned, [box(0, 10 * C, 1, 7 + 10 * C, 10 * C, fc, tc, s, _lib.DT_F32, 10 * C, R, C,
                                         block)], 10 * C * ds)
            same_or_policy(out.view(_dt(tc)), ref[10:20].reshape(-1), tc, (fc, block, "run"))
            assert n == R * C


def test_tile_seams_long_boxes_and_ten_thousand_boxes_in_one_call(ctx, pinned):
    """A 1000-row box of 3001-element rows (many 64 KiB tiles, seams at every phase) and 10 000 small boxes of one
    weight in one call, with F16 scales."""
    torch = _t()
    g = torch.Generator().manual_seed(4)
    R, C = 1200, 3011
    w = _random_fp8((R, C), _lib.DT_F8E4M3, g)
    n = stage(pinned, 3, w)
    s = (torch.rand(10, 24, generator=g) * 2).to(torch.float16).cuda()
    for tc in TARGETS:
        ds = _dt(tc).itemsize
        ref = reference(w, s, (128, 128), tc)
        out = call(ctx, pinned, [box(ds, 3001, 1000, 3 + 150 * C + 5, C, _lib.DT_F8E4M3, tc, s, _lib.DT_F16,
                                     150 * C + 5, R, C, (128, 128))], (3001 * 1000 + 2) * ds)
        same_or_policy(out[ds : ds + 3001 * 1000 * ds].view(_dt(tc)), ref[150:1150, 5:3006].reshape(-1), tc, "long")
        assert (out[:ds] == SENTINEL).all() and (out[ds + 3001 * 1000 * ds :] == SENTINEL).all()
    tc, ds = _lib.DT_BF16, 2
    ref = reference(w, s, (128, 128), tc)
    rng = np.random.default_rng(5)
    boxes, want, at = [], [], 0
    for k in range(10_000):
        r0, c0 = int(rng.integers(0, R - 3)), int(rng.integers(0, C - 40))
        rows, width = int(rng.integers(1, 4)), int(rng.integers(1, 40))
        boxes.append(box(at * ds, width, rows, 3 + r0 * C + c0, C, _lib.DT_F8E4M3, tc, s, _lib.DT_F16, r0 * C + c0,
                         R, C, (128, 128)))
        want.append((at, ref[r0 : r0 + rows, c0 : c0 + width].reshape(-1)))
        at += rows * width + int(rng.integers(0, 3))
    out = call(ctx, pinned, boxes, (at + 8) * ds)
    got = out[: at * ds].view(torch.bfloat16)
    clean = torch.ones(at, dtype=torch.bool, device="cuda")
    for a, wv in want:
        clean[a : a + wv.numel()] = False
    same_or_policy(torch.cat([got[a : a + wv.numel()] for a, wv in want]), torch.cat([wv for _, wv in want]), tc,
                   "10000 boxes")
    assert (out[: at * ds].view(torch.int16)[clean] == (SENTINEL | SENTINEL << 8) - 65536).all()
    assert n == R * C


def test_stream_order(ctx, pinned):
    """On a side stream, the copy sees the scales a kernel wrote before it on that stream, and its bytes are there
    for the next kernel on that stream."""
    torch = _t()
    g = torch.Generator().manual_seed(6)
    R, C = 256, 4096
    w = _random_fp8((R, C), _lib.DT_F8E4M3, g)
    n = stage(pinned, 0, w)
    side = torch.cuda.Stream()
    s = torch.zeros(2, 32, device="cuda")
    out = torch.full((n * 4,), SENTINEL, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(20_000_000)
        s.fill_(0.5)
        ctx.copy_scaled_boxes_from_host([out.data_ptr()], [out.numel()], [0, 1],
                                        [box(0, n, 1, 0, n, _lib.DT_F8E4M3, _lib.DT_F32, s, _lib.DT_F32, 0, R, C,
                                             (128, 128))], pinned, side.cuda_stream)
        total = out.view(torch.float32).nan_to_num(0.0).sum()
    side.synchronize()
    want = reference(w, s, (128, 128), _lib.DT_F32).reshape(-1)
    same_or_policy(out.view(torch.float32), want, _lib.DT_F32, "stream")
    assert float(total) == float(want.nan_to_num(0.0).sum())


# --------------------------------------------------------------------------------------------- rejections


def test_every_rejected_argument_is_refused_before_anything_is_enqueued(ctx, pinned):
    torch = _t()
    R, C = 300, 200
    s = torch.ones(3, 2, device="cuda")
    out = torch.full((R * C * 4,), SENTINEL, dtype=torch.uint8, device="cuda")
    good = box(0, C, R, 0, C, _lib.DT_F8E4M3, _lib.DT_BF16, s, _lib.DT_F32, 0, R, C, (128, 128))
    host_s = torch.ones(6)
    odd = torch.ones(7, device="cuda")
    other = torch.ones(6, dtype=torch.float16, device="cuda")
    bad = {
        "src_type F32": {6: _lib.DT_F32}, "src_type 9": {6: 9}, "dst_type F8": {7: _lib.DT_F8E5M2}, "dst_type 0": {7: 0},
        "scale_type F8": {9: _lib.DT_F8E4M3}, "block_rows 0": {14: 0}, "block_cols 0": {15: 0},
        "too few scales": {10: 5}, "scale count for smaller blocks": {14: 64},
        "past R * C": {11: 1}, "rows past R": {3: R + 1, 12: R}, "huge R * C overflow": {11: 2 ** 63, 12: 2 ** 40},
        "NULL scales": {8: 0}, "host scales": {8: host_s.data_ptr()}, "misaligned scales": {8: odd.data_ptr() + 2},
        "F16 scales misaligned": {8: other.data_ptr() + 1, 9: _lib.DT_F16},
        "destination past the file": {1: R * C * 3}, "source past h_src": {4: pinned.size - 10},
    }
    torch.cuda.synchronize()
    for what, change in bad.items():
        b = list(good)
        for k, v in change.items():
            b[k] = v
        launches = ctx.launch_count
        with pytest.raises(_lib.B200HashError):
            ctx.copy_scaled_boxes_from_host([out.data_ptr()], [out.numel()], [0, 1], [tuple(b)], pinned, _current())
        assert ctx.launch_count == launches, what
    torch.cuda.synchronize()
    assert (out == SENTINEL).all()
    # the converting entries keep refusing the FP8 codes
    for fc in FORMATS:
        for cast in ((0, 0, 16, 1, 0, 16, fc, _lib.DT_BF16), (0, 0, 16, 1, 0, 16, _lib.DT_F32, fc)):
            with pytest.raises(_lib.B200HashError, match="unknown element type"):
                ctx.copy_cast_boxes_from_host([out.data_ptr()], [out.numel()], [0, 1], [cast], pinned, _current())
        with pytest.raises(_lib.B200HashError):
            ctx.copy_cast_ranges([out.data_ptr()], [64], [fc], [_lib.DT_BF16], [0, 1], [(0, 0, 16)], out, [0])
    # an empty box launches nothing
    call(ctx, pinned, [box(0, 0, 5, 0, C, _lib.DT_F8E4M3, _lib.DT_BF16, s, _lib.DT_F32, 0, R, C, (128, 128))], 16)


# --------------------------------------------------------------------------------------------- end to end


def _fp8_stack(layers=5, h=4096, m=12288):
    """About 1 GB: DeepSeek/Qwen3-shaped E4M3 projections (sides not all multiples of 128 for the KV pair) with F32
    128 x 128 ``_scale_inv`` tensors, and BF16 norms."""
    torch = _t()
    g = torch.Generator(device="cuda").manual_seed(7)
    sd = {}
    for i in range(layers):
        p = f"model.layers.{i}."
        shapes = {"self_attn.q_proj": (h, h), "self_attn.kv_a_proj": (576, h), "self_attn.o_proj": (h, h),
                  "mlp.gate_proj": (m, h), "mlp.up_proj": (m, h), "mlp.down_proj": (h, m)}
        for k, (R, C) in shapes.items():
            sd[p + k + ".weight"] = (torch.randn(R, C, generator=g, device="cuda") * 50).to(torch.float8_e4m3fn)
            sd[p + k + ".weight_scale_inv"] = torch.rand(-(-R // 128), -(-C // 128), generator=g, device="cuda") * 1e-3
        sd[p + "input_layernorm.weight"] = torch.randn(h, generator=g, device="cuda").to(torch.bfloat16)
    return sd


def test_a_1gb_fp8_stack_reads_back_dequantized_whole_and_as_tp_slices(gpu_backend):
    torch = _t()
    sd = _fp8_stack()
    scales = volume.fp8_scales(sd)
    want = {k: (reference(v, sd[scales[k]], (128, 128), _lib.DT_BF16) if k in scales else v) for k, v in sd.items()
            if k not in scales.values()}

    def tp(name, shape, rank=3, ranks=8):
        if len(shape) == 1:
            return ...
        if name.endswith(("o_proj.weight", "down_proj.weight")):
            n = shape[1] // ranks
            return (slice(None), slice(rank * n + 1, (rank + 1) * n + 3))  # odd bounds across block edges
        n = shape[0] // ranks
        return (slice(rank * n + 5, (rank + 1) * n),)

    async def grown(fn):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = await fn()
        torch.cuda.synchronize()
        return out, torch.cuda.max_memory_allocated() - base

    async def run():
        async with running_volume_server(blob_utils.BLOCK_SIZE) as (stub, _):
            client = types.SimpleNamespace(stub=stub)
            shards = device_file.safetensors_shards(sd, max_shard_size="300MB")
            assert len(shards.files) >= 3
            async with volume.VolumeUploadContextManager2("vo-g", client) as batch:
                shards.put(batch, "/ckpt")
            del shards
            index = "/ckpt/model.safetensors.index.json"
            _, where = await volume.read_safetensors_index(client, "vo-g", index)
            assert volume.fp8_scales(where) == scales
            scale_bytes = sum(sd[s].numel() * 4 for s in scales.values())
            got, growth = await grown(lambda: volume.read_safetensors_sharded(
                client, "vo-g", index, dtype=torch.bfloat16, scales=scales))
            results = sum(t.numel() * t.element_size() for t in got.values())
            assert growth <= results + scale_bytes + 8 * MiB, (growth, results, scale_bytes)
            assert sorted(got) == sorted(want)
            for k, v in want.items():
                assert torch.equal(got[k].view(torch.int16 if v.element_size() == 2 else torch.uint8),
                                   v.view(torch.int16 if v.element_size() == 2 else torch.uint8)), k
            del got
            select = {k: tp(k, where[k][2]) for k in want}
            got, growth = await grown(lambda: volume.read_safetensors_sharded(
                client, "vo-g", index, select=select, dtype=torch.bfloat16, scales=scales))
            results = sum(t.numel() * t.element_size() for t in got.values())
            assert growth <= results + scale_bytes + 8 * MiB, (growth, results, scale_bytes)
            for k, i in select.items():
                assert torch.equal(got[k].view(torch.int16), want[k][i].contiguous().view(torch.int16)), k

    asyncio.run(run())
