"""GPU: b200h_copy_cast_boxes_from_host against torch's CUDA ``.to()`` on the same device, compared bit for bit through
integer views: every F16 and BF16 bit pattern through the four conversions from 16-bit sources, every F32 bit pattern
to BF16 and to F16; every element-aligned source phase against every element-aligned destination phase, widths of 1 to
300 elements and past a 64 KiB tile, 1 to 1000 rows, pitches equal to and above the width, 10 000 boxes in one call
and a source span over 4 GiB; nothing is written outside the boxes, one kernel per call (none for empty boxes), the
copy is stream-ordered and bad arguments are rejected before anything is enqueued.  End to end, a ~1 GiB F32 state
dict with BF16, F16 and I64 tensors, read with ``dtype=``, equals ``read_safetensors`` followed by ``.to()``, with the
unconverted call's requests, at most two launches per wave and no HBM beyond the results; every tensor-parallel rank's
converted slices, on dim 0 and on dim 1, concatenate to the converted full tensors."""
import asyncio
import types

import numpy as np
import pytest

from modal_client_b200 import DeviceFile, _lib, blob_utils, load_cast_boxes, volume
from tests.test_volume_read_slices_gpu import tp_select
from tests.volume_read_server import running_volume_server

pytestmark = pytest.mark.gpu

MiB, GiB = 1 << 20, 1 << 30
CANARY = 0x5C
PAIRS = [(s, d) for s in ("float32", "float16", "bfloat16") for d in ("float32", "float16", "bfloat16") if s != d]
CODE = {"float32": _lib.DT_F32, "float16": _lib.DT_F16, "bfloat16": _lib.DT_BF16}
SIZE = {"float32": 4, "float16": 2, "bfloat16": 2}
INT = {4: "int32", 2: "int16"}


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0, pinned_bytes=64 << 20, device_bytes=512 << 20)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pinned(ctx):
    buf = ctx.host_alloc(96 * MiB)
    yield buf
    ctx.host_free(buf)


def _pool(n):
    import torch

    return torch.empty(n, dtype=torch.uint8, device="cuda")


def _torch(name):
    import torch

    return getattr(torch, name)


def _cast_on_device(raw: np.ndarray, src: str, dst: str) -> np.ndarray:
    """The bytes of torch's CUDA ``.to(dst)`` of the ``src`` elements in ``raw``."""
    import torch

    if not raw.size:
        return raw
    t = torch.from_numpy(raw.copy()).cuda().view(_torch(src)).to(_torch(dst))
    return t.view(torch.uint8).cpu().numpy()


def _rows(box):
    """numpy indices of the source bytes of ``box`` in packed order."""
    _, _, w, rows, at, pitch = box[:6]
    return (at + np.arange(rows, dtype=np.int64)[:, None] * pitch + np.arange(w, dtype=np.int64)[None, :]).reshape(-1)


def _cast_boxes_and_check(ctx, src, segs, first, boxes, stream=0, fill=True):
    """One call; every box's device bytes equal torch's CUDA cast of its rows of ``src``, every other byte of every
    segment keeps its canary."""
    import torch

    if fill:
        used = max((b[4] + (b[3] - 1) * b[5] + b[2] for b in boxes if b[2] * b[3]), default=0)
        src[:used] = np.random.default_rng(len(boxes)).integers(0, 256, used, dtype=np.uint8)
    for s in segs:
        s.fill_(CANARY)
    images = []
    for f in range(len(first) - 1):
        images.append(np.concatenate([np.full(s.numel(), CANARY, np.uint8) for s in segs[first[f] : first[f + 1]]]
                                     or [np.zeros(0, np.uint8)]))
    by_pair = {}
    for b in boxes:
        if b[2] * b[3]:
            by_pair.setdefault((b[6], b[7]), []).append(b)
    for (s, d), bs in by_pair.items():  # one device cast per pair
        out = _cast_on_device(np.concatenate([src[_rows(b)] for b in bs]), s, d)
        at = 0
        for b in bs:
            n = b[2] * b[3] // SIZE[s] * SIZE[d]
            images[b[0]][b[1] : b[1] + n] = out[at : at + n]
            at += n
    torch.cuda.synchronize()
    launches = ctx.launch_count
    ctx.copy_cast_boxes_from_host([s.data_ptr() if s.numel() else 0 for s in segs], [s.numel() for s in segs], first,
                                  [b[:6] + (CODE[b[6]], CODE[b[7]]) for b in boxes], src, stream)
    assert ctx.launch_count - launches == (1 if any(b[2] * b[3] for b in boxes) else 0)
    torch.cuda.synchronize()
    for f in range(len(first) - 1):
        got = np.concatenate([s.cpu().numpy() for s in segs[first[f] : first[f + 1]]] or [np.zeros(0, np.uint8)])
        bad = np.flatnonzero(got != images[f])
        assert not bad.size, (f, bad[:10], got[bad[:10]], images[f][bad[:10]])


# ------------------------------------------------------------------------------------------ every value


def test_every_16_bit_pattern_through_the_four_conversions_from_16_bit_sources(ctx, pinned):
    import torch

    patterns = np.arange(1 << 16, dtype=np.uint16)
    for src, dst in [p for p in PAIRS if p[0] != "float32"]:
        s, d = SIZE[src], SIZE[dst]
        phase = 6  # an element-aligned source that is not 16-byte aligned
        pinned[phase : phase + (2 << 16)] = patterns.view(np.uint8)
        out = torch.full(((1 << 16) * d + 16,), CANARY, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()  # the copy runs on the context's stream
        ctx.copy_cast_boxes_from_host([out.data_ptr()], [out.numel()], [0, 1],
                                      [(0, 0, (1 << 16) * s, 1, phase, (1 << 16) * s, CODE[src], CODE[dst])], pinned)
        want = torch.from_numpy(patterns.view(np.int16).copy()).cuda().view(_torch(src)).to(_torch(dst))
        torch.cuda.synchronize()
        got = out[: (1 << 16) * d].view(getattr(torch, INT[d]))
        assert torch.equal(got, want.view(getattr(torch, INT[d]))), (src, dst)
        assert (out[(1 << 16) * d :] == CANARY).all()


def test_every_f32_bit_pattern_to_bf16_and_to_f16(ctx):
    import torch

    n = 1 << 26  # 256 MiB of F32 per chunk, 64 chunks
    buf = ctx.host_alloc(4 * n + 64)
    try:
        base = np.arange(n, dtype=np.uint32)
        outs = {d: torch.empty(2 * n, dtype=torch.uint8, device="cuda") for d in ("bfloat16", "float16")}
        idx = torch.arange(n, dtype=torch.int64, device="cuda")
        for k in range(64):
            phase = 4 * (k % 4)  # every F32 phase of a 16-byte word
            view = buf[phase : phase + 4 * n].view(np.uint32)
            np.add(base, np.uint32(k * n), out=view)
            for d, out in outs.items():
                ctx.copy_cast_boxes_from_host([out.data_ptr()], [out.numel()], [0, 1],
                                              [(0, 0, 4 * n, 1, phase, 4 * n, _lib.DT_F32, CODE[d])], buf)
            torch.cuda.synchronize()
            bits = idx + k * n
            bits = torch.where(bits >= 1 << 31, bits - (1 << 32), bits).to(torch.int32).view(torch.float32)
            for d, out in outs.items():
                want = bits.to(_torch(d)).view(torch.int16)
                got = out.view(torch.int16)
                if not torch.equal(got, want):
                    bad = torch.nonzero(got != want)[:8].flatten()
                    raise AssertionError((d, k, (bad + k * n).tolist(), got[bad].tolist(), want[bad].tolist()))
            torch.cuda.synchronize()  # the buffer is refilled next
    finally:
        torch.cuda.synchronize()
        ctx.host_free(buf)


# ---------------------------------------------------------------------------------------------- layout


@pytest.mark.parametrize("src,dst", PAIRS)
def test_every_source_phase_against_every_destination_phase(ctx, pinned, src, dst):
    """Boxes of every element-aligned source phase and every element-aligned destination phase (the segment itself
    starts at every such phase too), with pitches equal to the width, less than 16 bytes above it and more, then
    widths of 1 to 300 elements and three past 64 KiB, each a few rows."""
    s, d = SIZE[src], SIZE[dst]
    for seg_phase in range(0, 16, d):
        pool = _pool(24 * MiB + 256)
        seg = pool[seg_phase : seg_phase + 24 * MiB]
        boxes, dd, ss = [], 0, 0
        for sp in range(0, 16, s):
            for dq in range(0, 16, d):
                for w, rows, gap in ((37, 3, 0), (37, 3, 3), (37, 3, 11), (5, 9, 2), (1, 7, 1), (100, 2, 75)):
                    dd = -(-dd // 16) * 16 + dq + 16
                    ss = -(-ss // 16) * 16 + sp
                    boxes.append((0, dd, w * s, rows, ss, (w + gap) * s, src, dst))
                    dd += w * rows * d
                    ss += ((rows - 1) * (w + gap) + w) * s
        rng = np.random.default_rng(seg_phase)
        for w in list(range(1, 301)) + [16 * 1024, 16 * 1024 + 3, 50_001]:
            rows = int(rng.integers(1, 5))
            gap = int(rng.choice([0, rng.integers(1, 4), rng.integers(4, 1000)]))
            dd += int(rng.integers(0, 20)) * d
            ss += int(rng.integers(0, 20)) * s
            boxes.append((0, dd, w * s, rows, ss, (w + gap) * s, src, dst))
            dd += w * rows * d
            ss += ((rows - 1) * (w + gap) + w) * s
        assert dd <= seg.numel() and ss <= pinned.size
        _cast_boxes_and_check(ctx, pinned, [seg], [0, 1], boxes)


def test_rows_up_to_a_thousand_and_boxes_in_many_segments(ctx, pinned):
    rng = np.random.default_rng(3)
    segs, boxes, ss = [], [], 0
    for src, dst in PAIRS:
        s, d = SIZE[src], SIZE[dst]
        for rows in (1, 2, 3, 7, 31, 100, 999, 1000):
            for w in (1, 2, 3, 4, 5, 8, 9, 33, 100):
                gap = int(rng.choice([0, 1, 3, 4, 5, 300]))
                ss += s * int(rng.integers(0, 8))
                n = w * rows * d
                seg = _pool(n + 64)[d : d + n + int(rng.integers(0, 3)) * d]  # the box fills its segment or not
                boxes.append((len(segs), 0, w * s, rows, ss, (w + gap) * s, src, dst))
                segs.append(seg)
                ss += ((rows - 1) * (w + gap) + w) * s
    assert ss <= pinned.size
    first = list(range(len(segs) + 1))
    _cast_boxes_and_check(ctx, pinned, segs, first, boxes)
    # one file of all the segments: each box inside one of them
    offsets = np.concatenate([[0], np.cumsum([s.numel() for s in segs])[:-1]]).tolist()
    _cast_boxes_and_check(ctx, pinned, segs, [0, len(segs)], [(0, o) + b[2:] for b, o in zip(boxes, offsets)])


def test_ten_thousand_boxes_in_one_call(ctx, pinned):
    rng = np.random.default_rng(10)
    boxes, dd, ss = [], 0, 0
    for i in range(10_000):
        src, dst = PAIRS[i % len(PAIRS)]
        s, d = SIZE[src], SIZE[dst]
        w, rows = int(rng.integers(1, 60)), int(rng.integers(1, 5))
        gap = int(rng.choice([0, rng.integers(1, 4), rng.integers(4, 100)]))
        dd = -(-dd // d) * d
        ss = -(-ss // s) * s
        back = s * int(rng.integers(0, min(ss // s, 12) + 1))  # sources may overlap
        boxes.append((0, dd, w * s, rows, ss - back, (w + gap) * s, src, dst))
        dd += w * rows * d
        ss += ((rows - 1) * (w + gap) + w) * s
    _cast_boxes_and_check(ctx, pinned, [_pool(dd + 16)], [0, 1], boxes)


def test_one_box_whose_source_spans_more_than_4_gib(ctx):
    import torch

    pitch = 2 * GiB + 12
    big = ctx.host_alloc(2 * pitch + MiB + 64)
    try:
        box = (0, 16, MiB, 3, 20, pitch, "float32", "bfloat16")
        rng = np.random.default_rng(11)
        for r in range(3):
            big[4 + r * pitch : 36 + r * pitch + MiB] = rng.integers(0, 256, MiB + 32, dtype=np.uint8)
        _cast_boxes_and_check(ctx, big, [_pool(3 * MiB // 2 + 64)], [0, 1], [box], fill=False)
    finally:
        torch.cuda.synchronize()
        ctx.host_free(big)


def test_empty_boxes_launch_nothing_and_the_call_is_stream_ordered(ctx, pinned):
    import torch

    seg = _pool(4096)
    launches = ctx.launch_count
    ctx.copy_cast_boxes_from_host([seg.data_ptr()], [4096], [0, 1], [(0, 0, 0, 9, 0, 0, 1, 3), (0, 4, 8, 0, 4, 8, 1, 3)],
                                  pinned)
    ctx.copy_cast_boxes_from_host([seg.data_ptr()], [4096], [0, 1], [], pinned)
    assert ctx.launch_count == launches
    stream = torch.cuda.Stream()
    dst = _pool(16 * MiB + 8)
    busy = torch.empty(64 * MiB, dtype=torch.float32, device="cuda")
    pinned[: 65 * MiB] = np.random.default_rng(9).integers(0, 256, 65 * MiB, dtype=np.uint8)
    torch.cuda.synchronize()
    rows, w = 16 * MiB // 2048, 4096
    box = (0, 2, w, rows, 260, 2 * w, "float32", "bfloat16")
    with torch.cuda.stream(stream):
        for _ in range(20):
            busy.normal_()
        dst.fill_(1)
        ctx.copy_cast_boxes_from_host([dst.data_ptr()], [dst.numel()], [0, 1],
                                      [box[:6] + (_lib.DT_F32, _lib.DT_BF16)], pinned, stream.cuda_stream)
    stream.synchronize()
    got = dst.cpu().numpy()
    want = _cast_on_device(pinned[_rows(box)], "float32", "bfloat16")
    assert got[:2].tolist() == [1, 1] and np.array_equal(got[2 : 2 + want.size], want)
    assert (got[2 + want.size :] == 1).all()


def test_bad_arguments_are_rejected_before_anything_is_enqueued(ctx, pinned):
    import torch

    pool = _pool(8192 + 16)
    seg = pool[:4096]
    seg2 = pool[4096:8192]
    pool.fill_(CANARY)
    host = torch.empty(4096, dtype=torch.uint8)
    pageable = np.zeros(8192, np.uint8)
    F32, F16, BF16 = _lib.DT_F32, _lib.DT_F16, _lib.DT_BF16
    ok = dict(ptrs=[seg.data_ptr()], lens=[4096], first=[0, 1],
              boxes=[(0, 0, 40, 10, 0, 40, F32, BF16), (0, 800, 8, 3, 4, 12, BF16, F32)], src=pinned[:4096])
    cases = {
        "host segment": dict(ptrs=[host.data_ptr()]),
        "NULL segment": dict(ptrs=[0]),
        "file that does not exist": dict(boxes=[(1, 0, 4, 1, 0, 4, F32, F16)]),
        "misaligned source element": dict(boxes=[(0, 0, 8, 1, 2, 8, F32, BF16)]),
        "misaligned source row of a buffer at an odd phase": dict(src=pinned[1:4097],
                                                                  boxes=[(0, 0, 8, 1, 0, 8, F16, F32)]),
        "misaligned destination": dict(boxes=[(0, 1, 8, 1, 0, 8, F32, BF16)]),
        "misaligned widened destination": dict(boxes=[(0, 2, 8, 1, 0, 8, F16, F32)]),
        "width not a multiple of the element size": dict(boxes=[(0, 0, 6, 1, 0, 6, F32, BF16)]),
        "pitch not a multiple of the element size": dict(boxes=[(0, 0, 8, 2, 0, 10, F32, BF16)]),
        "destination across a segment edge": dict(ptrs=[seg.data_ptr(), seg2.data_ptr()], lens=[4096, 4096],
                                                  first=[0, 2], boxes=[(0, 4094, 8, 1, 0, 8, F32, BF16)]),
        "equal types": dict(boxes=[(0, 0, 8, 1, 0, 8, BF16, BF16)]),
        "unknown source type": dict(boxes=[(0, 0, 8, 1, 0, 8, 0, BF16)]),
        "unknown destination type": dict(boxes=[(0, 0, 8, 1, 0, 8, F32, 4)]),
        "destination past the end of its file": dict(boxes=[(0, 4000, 100, 1, 0, 100, F16, F32)]),
        "rows * width overflows": dict(boxes=[(0, 0, 1 << 33, 1 << 33, 0, 1 << 33, F32, F16)]),
        "widened size overflows": dict(boxes=[(0, 0, 2**63 + 2, 1, 0, 2**63 + 2, F16, F32)]),
        "offset + destination overflows": dict(boxes=[(0, 2**64 - 8, 16, 1, 0, 16, F32, F16)]),
        "source past h_src_bytes": dict(boxes=[(0, 0, 40, 10, 4000, 40, F32, F16)]),
        "source offset overflows": dict(boxes=[(0, 0, 16, 1, 2**64 - 8, 16, F32, F16)]),
        "overlapping destinations": dict(boxes=[(0, 0, 40, 10, 0, 40, F32, BF16), (0, 198, 4, 1, 0, 4, F32, BF16)]),
        "source not page-locked": dict(src=pageable[:4096]),
    }
    for name, change in cases.items():
        a = {**ok, **change}
        launches = ctx.launch_count
        with pytest.raises(_lib.B200HashError, match=r"\(-1\)"):
            ctx.copy_cast_boxes_from_host(a["ptrs"], a["lens"], a["first"], a["boxes"], a["src"])
        assert ctx.launch_count == launches, name
    torch.cuda.synchronize()
    assert (pool.cpu().numpy() == CANARY).all()


def test_load_cast_boxes_orders_after_earlier_reads(gpu_backend):
    """As load_boxes: a kernel queued before the call sees the old values, work queued after it the new ones."""
    import torch

    t = torch.full((64 * MiB,), 3, dtype=torch.bfloat16, device="cuda")
    busy = torch.empty(64 * MiB, dtype=torch.float32, device="cuda")
    src = gpu_backend.host_alloc(256 * MiB + 4096)
    try:
        src.view(np.float32)[:] = 9.0
        f = DeviceFile(t)
        for _ in range(20):
            busy.normal_()
        before = t.sum(dtype=torch.float64)
        loaded = load_cast_boxes([f], [(0, 0, 4096, t.numel() // 1024, 8, 4096, torch.float32, torch.bfloat16)], src)
        after = t.sum(dtype=torch.float64)
        loaded.wait()
        assert float(before) == 3 * t.numel() and float(after) == 9 * t.numel()
    finally:
        torch.cuda.synchronize()
        gpu_backend.host_free(src)


# ----------------------------------------------------------------------------------------- end to end


def mixed_state_dict(total: int, seed: int = 0):
    """A Llama-shaped F32 layer stack of about ``total`` bytes (hidden 1024, intermediate 2816), plus BF16, F16 and
    I64 tensors of odd lengths and an F32 tensor of special values (NaNs with payloads, infinities, subnormals, values
    that overflow F16)."""
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    H, I = 1024, 2816
    shapes = {"q_proj": (H, H), "k_proj": (H // 4, H), "o_proj": (H, H), "gate_proj": (I, H), "down_proj": (H, I)}
    per = sum(int(np.prod(s)) * 4 for s in shapes.values())
    sd = {}
    for i in range(max(1, total // per)):
        for name, shape in shapes.items():
            sd[f"layers.{i}.{name}.weight"] = torch.randn(shape, device="cuda", generator=g)
        sd[f"layers.{i}.norm.weight"] = torch.randn(H + 3, device="cuda", generator=g).to(torch.bfloat16)
        sd[f"layers.{i}.bias"] = torch.randn(2 * H + 1, device="cuda", generator=g).to(torch.float16)
        sd[f"layers.{i}.ids"] = torch.randint(-2**40, 2**40, (333,), device="cuda", generator=g)
    special = torch.randint(-2**31, 2**31 - 1, (1 << 20,), device="cuda", generator=g, dtype=torch.int64)
    sd["special"] = special.to(torch.int32).view(torch.float32) * 1  # NaNs, infinities, subnormals and all
    sd["special"][:8] = torch.tensor([65520.0, 65519.0, -1e-45, 3.4e38, float("inf"), -0.0, 1e-40, 2.0**-24],
                                     device="cuda")
    return sd


def _same_bits(a, b):
    import torch

    assert a.dtype == b.dtype and a.shape == b.shape
    iv = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]
    return torch.equal(a.contiguous().view(iv), b.contiguous().view(iv))


def test_a_1gib_f32_state_dict_read_as_bf16_and_every_tp_rank(gpu_backend):
    import torch

    sd_ref = [mixed_state_dict(GiB)]
    BS = blob_utils.BLOCK_SIZE
    staging = 64 * MiB

    def waves(nblocks):
        return -(-nblocks // (staging // 2 // BS))

    async def run():
        async with running_volume_server(BS) as (stub, faults):
            client = types.SimpleNamespace(stub=stub)
            batch = volume.VolumeUploadContextManager2("vo-c", client)
            async with batch:
                batch.put_file(DeviceFile.safetensors(sd_ref[0]), "/m.safetensors")
            del batch
            calls, gets = len(stub.get_file_calls), faults["gets"]
            full = await volume.read_safetensors(client, "vo-c", "/m.safetensors", staging_bytes=staging)
            plain_reqs = [(r.start, r.len) for r in stub.get_file_calls[calls:]]
            plain_gets = faults["gets"] - gets
            for k, t in full.items():
                assert _same_bits(t, sd_ref[0][k]), k
            sd_ref.clear()
            nblocks = plain_gets - 2
            mapping = {k: (torch.float16 if "bias" in k or "special" in k else torch.bfloat16)
                       for k, t in full.items() if t.dtype == torch.float32 and "gate" not in k}
            mapping.update({k: torch.float32 for k, t in full.items() if t.dtype == torch.bfloat16})
            for form in (torch.bfloat16, torch.float16, torch.float32, mapping):
                targets = form if isinstance(form, dict) else {k: form for k, t in full.items() if t.is_floating_point()}
                want = {k: t.to(targets[k]) if k in targets else t for k, t in full.items()}
                for into in (False, True):
                    given = {k: torch.empty_like(t) for k, t in want.items()} if into else None
                    calls, gets = len(stub.get_file_calls), faults["gets"]
                    torch.cuda.synchronize()
                    base = torch.cuda.memory_allocated()
                    torch.cuda.reset_peak_memory_stats()
                    launches = gpu_backend.launch_count
                    got = await volume.read_safetensors(client, "vo-c", "/m.safetensors", dtype=form, into=given,
                                                        staging_bytes=staging)
                    torch.cuda.synchronize()
                    assert gpu_backend.launch_count - launches <= 2 * waves(nblocks)
                    result = sum(t.numel() * t.element_size() for t in got.values())
                    # torch allocates the results and nothing else (slack: the caching allocator's rounding)
                    assert torch.cuda.max_memory_allocated() - base <= (0 if into else result) + 16 * MiB, form
                    assert [(r.start, r.len) for r in stub.get_file_calls[calls:]] == plain_reqs
                    assert faults["gets"] - gets == plain_gets
                    assert list(got) == list(full)
                    for k in want:
                        assert _same_bits(got[k], want[k]), (form, into, k)
                        if into:
                            assert got[k] is given[k]
                    del got, given
            shapes = {k: tuple(t.shape) for k, t in full.items() if "layers" in k and t.dim() == 2}
            conv = {k: full[k].to(torch.bfloat16) for k in shapes}
            for dim in (0, 1):
                parts = []
                for rank in range(8):
                    select = tp_select(shapes, rank, dim=dim)
                    got = await volume.read_safetensors_slices(client, "vo-c", "/m.safetensors", select,
                                                               dtype=torch.bfloat16, staging_bytes=staging)
                    parts.append(got)
                for name, t in conv.items():
                    assert _same_bits(torch.cat([p[name] for p in parts], dim=dim), t), (dim, name)
                del parts

    asyncio.run(run())
