"""GPU: b200h_copy_cast_ranges equals torch's CUDA ``.to()`` bit for bit for every pair of F32 / F16 / BF16, every
16-bit pattern, F32 specials and 2^24 random patterns, at every range residue, into host and device memory, writing
nothing outside its destinations; b200h_hash_cast_segment_parts_device equals the plain entry over the pre-converted
dict; ``DeviceFile.safetensors(sd, dtype=torch.bfloat16)`` uploads what the pre-converted dict uploads, reads back
bitwise equal to ``.to()``, and allocates no converted copy in HBM."""
import asyncio
import hashlib
import types

import numpy as np
import pytest

from modal_client_b200 import DeviceFile, _lib, blob_utils, volume
from tests.volume_read_server import running_volume_server

pytestmark = pytest.mark.gpu

MiB, GiB = 1 << 20, 1 << 30
SENTINEL = 0xC3
PAIRS = [(a, b) for a in (1, 2, 3) for b in (1, 2, 3) if a != b]


def _dt(code):
    import torch

    return {_lib.DT_F32: torch.float32, _lib.DT_F16: torch.float16, _lib.DT_BF16: torch.bfloat16}[code]


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0, pinned_bytes=64 << 20, device_bytes=512 << 20)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pinned(ctx):
    buf = ctx.host_alloc(160 * MiB)
    yield buf
    ctx.host_free(buf)


def _patterns(code, n_random=1 << 24):
    """Source elements of type ``code`` on the device: every 16-bit pattern, or for F32 the specials, subnormals,
    rounding ties of both narrow types, NaNs with payloads, and ``n_random`` random patterns."""
    import torch

    if code != _lib.DT_F32:
        return torch.arange(-(1 << 15), 1 << 15, dtype=torch.int32, device="cuda").to(torch.int16).view(_dt(code))
    special = [0, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FBFFFFF, 0xFFFFFFFF,
               0x00000001, 0x807FFFFF, 0x00800000, 0x7F7FFFFF, 0xFF7FFFFF, 0x33800000, 0x387FC000, 0x477FF000,
               0x477FE000, 0x47800000]
    ties = []
    for hi in range(0, 1 << 16, 97):  # BF16 ties (low half 0x8000, even and odd kept halves) and near-ties
        ties += [(hi << 16) | 0x8000, (hi << 16) | 0x7FFF, (hi << 16) | 0x8001]
    for e in range(103, 143):  # F16 ties around every exponent F16 reaches, subnormals included
        for m in (0x1000, 0x3000, 0x0FFF, 0x1001):
            ties += [(e << 23) | m, (1 << 31) | (e << 23) | m]
    fixed = torch.tensor(np.array(special + ties, np.uint32).view(np.int32), device="cuda")
    g = torch.Generator(device="cuda").manual_seed(7)
    rnd = torch.randint(-(1 << 31), 1 << 31, (n_random,), dtype=torch.int64, device="cuda", generator=g).to(torch.int32)
    return torch.cat([fixed, rnd]).view(torch.float32)


def _expected(segs, casts):
    """The file image: every segment's bytes, converted by torch's CUDA ``.to()`` where it converts."""
    import torch

    parts = []
    for t, (st, dt) in zip(segs, casts):
        parts.append(t.view(_dt(st)).to(_dt(dt)).view(torch.uint8) if st != dt else t.view(torch.uint8))
    return torch.cat(parts) if parts else torch.empty(0, dtype=torch.uint8, device="cuda")


def _current():
    """torch's current stream as the library takes it (the legacy default stream is 1: NULL is the context's own)."""
    import torch

    return torch.cuda.current_stream().cuda_stream or 1


def _copy(ctx, segs, casts, ranges, dst, offsets, stream=None):
    """One call, ordered after the work torch enqueued on its current stream (the sources, the sentinel fill)."""
    ctx.copy_cast_ranges([t.data_ptr() if t.numel() else 0 for t in segs],
                         [t.numel() * t.element_size() for t in segs], [c[0] for c in casts], [c[1] for c in casts],
                         [0, len(segs)], ranges, dst, offsets, stream or _current())


def _layout(lens, gap=128):
    offsets, at = [], gap
    for n in lens:
        offsets.append(at)
        at += -(-n // 128) * 128 + gap
    return offsets, at


def _check(ctx, pinned, segs, casts, ranges, where):
    """One call into a host or device buffer filled with the sentinel; ranges equal the image, the rest untouched."""
    import torch

    image = _expected(segs, casts).cpu().numpy()
    offsets, total = _layout([n for _, _, n in ranges])
    if where == "host":
        dst = pinned[:total]
        dst[:] = SENTINEL
    else:
        dst = torch.full((total,), SENTINEL, dtype=torch.uint8, device="cuda")
    launches = ctx.launch_count
    _copy(ctx, segs, casts, ranges, dst, offsets)
    torch.cuda.synchronize()
    assert ctx.launch_count == launches + (1 if any(n for _, _, n in ranges) else 0)
    got = dst if where == "host" else dst.cpu().numpy()
    clean = np.ones(total, bool)
    for (_, off, n), at in zip(ranges, offsets):
        assert np.array_equal(got[at : at + n], image[off : off + n]), (off, n)
        clean[at : at + n] = False
    assert (got[clean] == SENTINEL).all()


@pytest.mark.parametrize("where", ["host", "device"])
@pytest.mark.parametrize("pair", PAIRS)
def test_every_bit_pattern_converts_as_torch_does(ctx, pinned, pair, where):
    import torch

    st, dt = pair
    src = _patterns(st, n_random=(1 << 24) if where == "device" else 1 << 16)
    want = src.to(_dt(dt)).view(torch.uint8)
    if where == "device":
        dst = torch.full((want.numel() + 256,), SENTINEL, dtype=torch.uint8, device="cuda")
        _copy(ctx, [src], [pair], [(0, 0, want.numel())], dst, [128])
        torch.cuda.synchronize()
        assert torch.equal(dst[128:-128], want)
        assert (dst[:128] == SENTINEL).all() and (dst[-128:] == SENTINEL).all()
    else:
        n = want.numel()
        dst = pinned[: n + 256]
        dst[:] = SENTINEL
        _copy(ctx, [src], [pair], [(0, 0, n)], dst, [128])
        torch.cuda.synchronize()
        assert np.array_equal(dst[128 : 128 + n], want.cpu().numpy())
        assert (dst[:128] == SENTINEL).all() and (dst[128 + n :] == SENTINEL).all()


@pytest.mark.parametrize("where", ["host", "device"])
def test_ranges_at_every_residue_across_segments_and_elements(ctx, pinned, where):
    """A header-like plain segment, then converting segments of every pair and of lengths 0 .. 9 MiB, views at
    every source phase; ranges that start at every residue mod 16, mid-element included, and end anywhere."""
    import torch

    g = torch.Generator(device="cuda").manual_seed(3)
    pool = torch.randint(0, 256, (40 * MiB,), dtype=torch.uint8, device="cuda", generator=g)
    pool.view(torch.int32)[::97] = 0x7FC00001  # some NaNs
    segs, casts, at, base = [pool[7:7 + 88]], [(0, 0)], 88, 4096
    sizes = [0, 4, 8, 12, 16, 20, 64, 100, 4096, 65536 + 44, MiB + 36, 9 * MiB]
    for i, n in enumerate(sizes):
        st, dt = PAIRS[i % len(PAIRS)]
        ss, ds = _dt(st).itemsize, _dt(dt).itemsize
        if at % ds:  # keep the image offset a multiple of the destination size with a plain filler
            segs.append(pool[base : base + (ds - at % ds)])
            casts.append((0, 0))
            at += ds - at % ds
            base += 64
        base = -(-base // 16) * 16
        phase = (i * ss) % 16  # source address phase (a multiple of the element size)
        n -= n % ss
        segs.append(pool[base + phase : base + phase + n])
        casts.append((st, dt))
        at += n // ss * ds
        base += n + 4096
        segs.append(pool[base + i : base + i + 3 + i])  # plain bytes between converting segments
        casts.append((0, 0))
        at += 3 + i
        base += 64
    total = at
    rng = np.random.default_rng(1)
    ranges = [(0, 0, total), (0, total - 1, 1), (0, 5, 0)]
    ranges += [(0, r, int(rng.integers(1, 300))) for r in range(16)]
    ranges += [(0, int(o), int(min(total - o, rng.integers(1, 3 * MiB)))) for o in rng.integers(0, total - 1, 40)]
    _check(ctx, pinned, segs, casts, ranges, where)


def test_ten_thousand_ranges_in_one_call(ctx, pinned):
    import torch

    src = _patterns(_lib.DT_F32, n_random=1 << 20)
    segs = [src[:300_000], src[300_000:300_001], src[400_000:900_000].view(torch.uint8)[:1001]]
    casts = [(_lib.DT_F32, _lib.DT_BF16), (_lib.DT_F32, _lib.DT_F16), (0, 0)]
    total = 300_000 * 2 + 2 + 1001
    rng = np.random.default_rng(2)
    starts = rng.integers(0, total - 1, 10_000)
    ranges = [(0, int(s), int(min(total - s, rng.integers(0, 200)))) for s in starts]
    _check(ctx, pinned, segs, casts, ranges, "host")


def test_one_range_whose_source_span_is_over_4gib(ctx):
    import torch

    n = (4 * GiB + 64 * MiB) // 4
    src = torch.empty(n, dtype=torch.float32, device="cuda")
    src.view(torch.int32).random_(generator=torch.Generator(device="cuda").manual_seed(5))
    want = src.to(torch.bfloat16).view(torch.uint8)
    dst = torch.full((want.numel() + 32,), SENTINEL, dtype=torch.uint8, device="cuda")
    _copy(ctx, [src[1:]], [(_lib.DT_F32, _lib.DT_BF16)], [(0, 6, want.numel() - 8)], dst, [16])
    torch.cuda.synchronize()
    assert torch.equal(dst[16 : 16 + want.numel() - 8], want[8:])
    assert (dst[:16] == SENTINEL).all() and (dst[16 + want.numel() - 8 :] == SENTINEL).all()


def test_the_call_is_stream_ordered_and_launches_once(ctx):
    import torch

    src = torch.zeros(32 * MiB, dtype=torch.float32, device="cuda")
    dst = torch.zeros(16 * MiB * 4, dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(4):
            src.add_(1.5)  # the copy must see all of them
        launches = ctx.launch_count
        _copy(ctx, [src], [(_lib.DT_F32, _lib.DT_F16)], [(0, 0, 64 * MiB)], dst, [0], stream=s.cuda_stream)
        _copy(ctx, [src], [(_lib.DT_F32, _lib.DT_F16)], [(0, 0, 0), (0, 7, 0)], dst, [0, 16], stream=s.cuda_stream)
    s.synchronize()
    assert ctx.launch_count == launches + 1
    assert torch.equal(dst.view(torch.float16), torch.full((32 * MiB,), 6.0, dtype=torch.float16, device="cuda"))


def test_bad_arguments_are_rejected_before_anything_is_enqueued(ctx, pinned):
    import torch

    seg = torch.arange(1024, dtype=torch.float32, device="cuda")
    f32, bf16 = _lib.DT_F32, _lib.DT_BF16
    ok = dict(ptrs=[seg.data_ptr()], lens=[4096], st=[f32], dt=[bf16], first=[0, 1], ranges=[(0, 0, 100)],
              dst=pinned[:4096], offsets=[0])
    bad = {
        "misaligned pointer": dict(ok, ptrs=[seg.data_ptr() + 2], lens=[4092]),
        "length not whole elements": dict(ok, lens=[4094]),
        "image at an odd offset": dict(ok, ptrs=[seg.data_ptr(), seg.data_ptr()], lens=[3, 4092], st=[0, f32],
                                       dt=[0, f32 + 1], first=[0, 2]),
        "unknown source type": dict(ok, st=[9]),
        "unknown destination type": dict(ok, dt=[0]),
        "equal but unknown": dict(ok, st=[6], dt=[6]),
        "range past the image": dict(ok, ranges=[(0, 2000, 100)]),
        "offset not a multiple of 16": dict(ok, offsets=[8]),
        "overlapping destinations": dict(ok, ranges=[(0, 0, 32), (0, 64, 32)], offsets=[0, 16]),
        "foreign pointer": dict(ok, ptrs=[pinned.ctypes.data]),
        "pageable destination": dict(ok, dst=np.zeros(4096, np.uint8)),
    }
    torch.cuda.synchronize()
    pinned[:4096] = SENTINEL
    for name, a in bad.items():
        launches = ctx.launch_count
        with pytest.raises(_lib.B200HashError):
            ctx.copy_cast_ranges(a["ptrs"], a["lens"], a["st"], a["dt"], a["first"], a["ranges"], a["dst"],
                                 a["offsets"])
        assert ctx.launch_count == launches, name
    torch.cuda.synchronize()
    assert (pinned[:4096] == SENTINEL).all()


# ------------------------------------------------------------------------------------------------- hashing


def _mixed_dict(total, seed):
    """F32 weights (some with zero tails and blank stretches), I64 and BF16 tensors, odd sizes included."""
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    sd, left, i = {}, total, 0
    sizes = [total // 3, total // 7, 9 * MiB + 12, 3 * MiB + 4, 70_004, 4100, 516, 64, 8, 4]
    while left > 0:
        n = min(left, sizes[i % len(sizes)])
        t = torch.randn(n // 4, generator=g, device="cuda")
        if i % 3 == 0:
            t[t.numel() // 2 :] = 0
        if i % 5 == 4:
            t = torch.randint(-1000, 1000, (max(1, n // 8),), generator=g, device="cuda")
        elif i % 5 == 3:
            t = t.to(torch.bfloat16)
        sd[f"layer.{i}.w"] = t
        left -= n
        i += 1
    return sd


def _table(ctx, f, part_len, flags, cast):
    import torch

    src = f._src
    ptrs = [s.data_ptr() if s.numel() else 0 for s in src.segments]
    lens = [s.numel() for s in src.segments]
    n = -(-src.nbytes // part_len)
    sha = torch.zeros((n, 32), dtype=torch.uint8, device="cuda")
    md5 = torch.zeros((n, 16), dtype=torch.uint8, device="cuda")
    trim = torch.zeros(n, dtype=torch.int64, device="cuda")
    o_sha, o_md5 = (sha.data_ptr() if flags & _lib.SHA256 else 0), (md5.data_ptr() if flags & _lib.MD5 else 0)
    if cast:
        casts = src.casts or [(0, 0)] * len(ptrs)
        got = ctx.hash_cast_segment_parts_device(ptrs, lens, [c[0] for c in casts], [c[1] for c in casts],
                                                 [0, len(ptrs)], part_len, flags, o_sha, o_md5, trim.data_ptr(),
                                                 _current())
    else:
        got = ctx.hash_segment_parts_device(ptrs, lens, [0, len(ptrs)], part_len, flags, o_sha, o_md5, trim.data_ptr(),
                                            _current())
    assert got == n
    torch.cuda.synchronize()
    return sha.cpu().numpy(), md5.cpu().numpy(), trim.cpu().numpy()


@pytest.mark.parametrize("part_len", [4096 + 3, MiB, 8 * MiB])
def test_hash_equals_the_plain_entry_over_the_preconverted_dict_and_hashlib(part_len):
    import torch
    from safetensors.torch import save

    small = _lib.Context(0, pinned_bytes=16 << 20, device_bytes=24 << 20)  # 12 MiB wave slots: several waves
    try:
        sd = _mixed_dict(96 * MiB, seed=part_len % 7)
        pre = {k: v.to(torch.bfloat16) if v.dtype == torch.float32 else v for k, v in sd.items()}
        f = DeviceFile.safetensors(sd, dtype=torch.bfloat16, ctx=small)
        g = DeviceFile.safetensors(pre, ctx=small)
        image = save({k: v.cpu() for k, v in pre.items()})
        assert f.nbytes == g.nbytes == len(image)
        lens = [s.numel() for s in f._src.segments]
        casts = f._src.casts
        _, _, nwaves = _lib.cast_segment_parts_preview(lens, [c[0] for c in casts], [c[1] for c in casts],
                                                       [0, len(lens)], part_len, 12 * MiB)
        assert nwaves >= 3
        for flags in (_lib.SHA256, _lib.MD5, _lib.SHA256 | _lib.MD5, _lib.SHA256 | _lib.TRIM_ZEROS,
                      _lib.SHA256 | _lib.MD5 | _lib.TRIM_ZEROS | _lib.NO_OUTLIERS):
            syncs, launches = small.plan_sync_count, small.launch_count
            a = _table(small, f, part_len, flags, cast=True)
            # the rule of the plain entry: one read-back per wave with TRIM_ZEROS and outlier routing, none otherwise
            trims = flags & _lib.TRIM_ZEROS and not flags & _lib.NO_OUTLIERS
            assert small.plan_sync_count - syncs == (nwaves if trims else 0), flags
            b = _table(small, g, part_len, flags, cast=False)
            assert all(np.array_equal(x, y) for x, y in zip(a, b)), flags
            assert small.launch_count > launches
            for i in range(0, -(-len(image) // part_len), max(1, len(image) // part_len // 9)):
                part = image[i * part_len : (i + 1) * part_len]
                if flags & _lib.TRIM_ZEROS:
                    part = part.rstrip(b"\0")
                    assert int(a[2][i]) == len(part)
                if flags & _lib.SHA256:
                    assert a[0][i].tobytes() == hashlib.sha256(part).digest(), (flags, i)
                if flags & _lib.MD5:
                    assert a[1][i].tobytes() == hashlib.md5(part).digest(), (flags, i)
    finally:
        small.close()


# ------------------------------------------------------------------------------------------------ end to end


def _same_bits(a, b):
    import torch

    iv = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(iv), b.contiguous().view(iv))


@pytest.mark.parametrize("budget_mib", [None, 256])
def test_a_1gib_f32_state_dict_uploads_as_bf16_without_a_converted_copy(gpu_backend, budget_mib):
    import torch

    sd = _mixed_dict(GiB, seed=11)
    want = {k: v.to(torch.bfloat16) if v.dtype == torch.float32 else v for k, v in sd.items()}
    BS = blob_utils.BLOCK_SIZE
    budget = budget_mib * MiB if budget_mib else None

    async def upload(make):
        async with running_volume_server(BS) as (stub, _):
            rounds = []
            put = stub.VolumePutFiles2

            async def logged(req):
                out = await put(req)
                rounds.append(sorted((m.file_index, m.block_index) for m in out.missing_blocks))
                return out

            stub.VolumePutFiles2 = logged
            client = types.SimpleNamespace(stub=stub)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            f = make()
            batch = volume.VolumeUploadContextManager2("vo-e", client, device_staging_bytes=budget)
            async with batch:
                batch.put_file(f, "/m.safetensors")
            torch.cuda.synchronize()
            growth = torch.cuda.max_memory_allocated() - base
            back = await volume.read_safetensors(client, "vo-e", "/m.safetensors")
            return rounds, dict(stub.blocks), growth, back, f.bytes_to_host

    pre = asyncio.run(upload(lambda: DeviceFile.safetensors(want)))
    got = asyncio.run(upload(lambda: DeviceFile.safetensors(sd, dtype=torch.bfloat16)))
    assert got[0] == pre[0] and got[1].keys() == pre[1].keys() and got[4] == pre[4]
    assert all(got[1][k] == pre[1][k] for k in pre[1])
    assert got[2] <= 8 * MiB, got[2]  # the header and the digest tables; the .to() copy alone is 0.5 GiB
    assert set(got[3]) == set(want)
    for k in want:
        assert _same_bits(got[3][k], want[k]), k
