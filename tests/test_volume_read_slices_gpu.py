"""GPU: b200h_copy_boxes_from_host is byte-exact against numpy for widths 1..300 and past 64 KiB, every source phase
against every destination phase, pitches equal to and above the width, 1..1000 rows, boxes across the segment edges
of a multi-segment file, 10 000 boxes in one call and a source span over 4 GiB; it writes nothing outside its boxes,
launches one kernel per call (none for empty boxes), is stream-ordered and rejects bad arguments before enqueueing.
End to end, every tensor-parallel rank's slices of a ~1 GiB bf16 state dict, on dim 0 and on dim 1, concatenate to
what read_safetensors returns, with the predicted GETs and the HBM torch allocates bounded by the results."""
import asyncio
import json
import types

import numpy as np
import pytest

from modal_client_b200 import DeviceFile, _lib, blob_utils, load_boxes, volume
from modal_client_b200.device_file import safetensors_layout
from tests.volume_read_server import running_volume_server

pytestmark = pytest.mark.gpu

MiB, GiB = 1 << 20, 1 << 30
CANARY = 0x5C


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


def _rows(box):
    """numpy indices of the source bytes of ``box`` in packed order."""
    _, _, w, rows, at, pitch = box
    return (at + np.arange(rows, dtype=np.int64)[:, None] * pitch + np.arange(w, dtype=np.int64)[None, :]).reshape(-1)


def _boxes_and_check(ctx, src, segs, first, boxes, stream=0, fill=True):
    """One call; every box's device bytes equal its rows of ``src``, every other byte of every segment keeps its
    canary."""
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
    for b in boxes:
        if b[2] * b[3]:
            images[b[0]][b[1] : b[1] + b[2] * b[3]] = src[_rows(b)]
    torch.cuda.synchronize()
    launches = ctx.launch_count
    ctx.copy_boxes_from_host([s.data_ptr() if s.numel() else 0 for s in segs], [s.numel() for s in segs], first, boxes,
                             src, stream)
    assert ctx.launch_count - launches == (1 if any(b[2] * b[3] for b in boxes) else 0)
    torch.cuda.synchronize()
    for f in range(len(first) - 1):
        got = np.concatenate([s.cpu().numpy() for s in segs[first[f] : first[f + 1]]] or [np.zeros(0, np.uint8)])
        bad = np.flatnonzero(got != images[f])
        assert not bad.size, (f, bad[:10], got[bad[:10]], images[f][bad[:10]])


@pytest.mark.parametrize("dst_phase", range(16))
def test_every_source_phase_against_every_destination_phase(ctx, pinned, dst_phase):
    """Per call: one destination phase (the segment starts that far past a 256-byte boundary); boxes of every source
    phase and every packed-destination phase, with pitches equal to the width, less than 16 bytes above it and more,
    then widths 1..300 and three past 64 KiB, each a few rows."""
    pool = _pool(64 * MiB + 256)
    seg = pool[dst_phase : dst_phase + 64 * MiB]
    boxes, d, s = [], 0, 0
    for sp in range(16):
        for dq in range(16):
            for w, rows, gap in ((37, 3, 0), (37, 3, 13), (37, 3, 43), (5, 9, 11), (100, 2, 300)):
                d = -(-d // 16) * 16 + dq + 16
                s = -(-s // 16) * 16 + sp
                boxes.append((0, d, w, rows, s, w + gap))
                d += w * rows
                s += (rows - 1) * (w + gap) + w
    rng = np.random.default_rng(dst_phase)
    for w in list(range(1, 301)) + [64 * 1024, 64 * 1024 + 13, 200_001]:
        rows = int(rng.integers(1, 6))
        gap = int(rng.choice([0, rng.integers(1, 16), rng.integers(16, 5000)]))
        d += int(rng.integers(0, 40))
        s += int(rng.integers(0, 40))
        boxes.append((0, d, w, rows, s, w + gap))
        d += w * rows
        s += (rows - 1) * (w + gap) + w
    assert d <= seg.numel() and s <= pinned.size
    _boxes_and_check(ctx, pinned, [seg], [0, 1], boxes)


def test_rows_up_to_a_thousand(ctx, pinned):
    boxes, d, s = [], 0, 3
    for rows in (1, 2, 3, 7, 31, 100, 999, 1000):
        for w in (1, 2, 5, 15, 16, 17, 33, 100, 257):
            for gap in (0, 1, 15, 16, 17, 4096 - w % 7):
                boxes.append((0, d, w, rows, s, w + gap))
                d += w * rows + 5
                s += (rows - 1) * (w + gap) + w + 3
    seg = _pool(d + 64)
    assert s <= pinned.size
    _boxes_and_check(ctx, pinned, [seg], [0, 1], boxes)


def test_boxes_across_the_segment_edges_of_a_multi_segment_file(ctx, pinned):
    import torch

    lens = [1, 7, 0, 16, 100, 4095, 3, 70_001, 17, 0, 300_000, 5, 64 * 1024 + 1, 2]
    pool = _pool(sum(-(-(n + 16) // 256) * 256 for n in lens) + 256)
    segs, at = [], 0
    for i, n in enumerate(lens):
        segs.append(pool[at + i % 16 : at + i % 16 + n])
        at += -(-(n + 16) // 256) * 256
    other = torch.empty(1000, dtype=torch.uint8, device="cuda")
    size = sum(lens)
    rng = np.random.default_rng(4)
    boxes, d, s = [], 0, 0
    while True:
        w, rows = int(rng.integers(1, 400)), int(rng.integers(1, 40))
        if d + w * rows > size:
            break
        gap = int(rng.choice([0, rng.integers(1, 16), rng.integers(16, 3000)]))
        boxes.append((0, d, w, rows, s, w + gap))
        d += w * rows + int(rng.integers(0, 20))
        s += (rows - 1) * (w + gap) + w + int(rng.integers(0, 20))
    boxes.append((1, 10, 30, 30, 7, 33))
    boxes.append((0, 0, 0, 5, 0, 0))  # empty
    _boxes_and_check(ctx, pinned, segs + [other], [0, len(segs), len(segs) + 1], boxes)


def test_ten_thousand_boxes_in_one_call(ctx, pinned):
    rng = np.random.default_rng(10)
    boxes, d, s = [], 0, 0
    for _ in range(10_000):
        w, rows = int(rng.integers(1, 200)), int(rng.integers(1, 5))
        gap = int(rng.choice([0, rng.integers(1, 16), rng.integers(16, 500)]))
        boxes.append((0, d, w, rows, s - int(rng.integers(0, min(s, 50) + 1)), w + gap))  # sources may overlap
        d += w * rows
        s += (rows - 1) * (w + gap) + w
    _boxes_and_check(ctx, pinned, [_pool(d)], [0, 1], boxes)


def test_one_box_whose_source_spans_more_than_4_gib(ctx):
    import torch

    pitch = 2 * GiB + 7
    big = ctx.host_alloc(2 * pitch + MiB + 64)
    try:
        box = (0, 16, MiB, 3, 21, pitch)
        rng = np.random.default_rng(11)
        for r in range(3):
            big[5 + r * pitch : 37 + r * pitch + MiB] = rng.integers(0, 256, MiB + 32, dtype=np.uint8)
        _boxes_and_check(ctx, big, [_pool(3 * MiB + 64)], [0, 1], [box], fill=False)
    finally:
        torch.cuda.synchronize()
        ctx.host_free(big)


@pytest.mark.parametrize("phase", [1, 3, 8, 15])
def test_a_source_buffer_at_any_phase(ctx, pinned, phase):
    """h_src a view into page-locked memory that starts `phase` bytes past a 16-byte boundary: byte-exact as at 0."""
    src = pinned[phase : phase + 8 * MiB]
    assert src.ctypes.data % 16 == phase
    boxes, d, s = [], 0, 0
    for w, rows, gap in ((1, 40, 0), (7, 30, 9), (37, 20, 3), (100, 9, 400), (4096, 5, 0), (70_001, 3, 17)):
        for sp in range(16):
            s = -(-s // 16) * 16 + sp
            boxes.append((0, d, w, rows, s, w + gap))
            d += w * rows + 3
            s += (rows - 1) * (w + gap) + w
    boxes.append((0, d, 16, 1, src.size - 16, 16))  # the source's last bytes
    d += 16
    assert s <= src.size
    _boxes_and_check(ctx, src, [_pool(d + 64)[5 : 5 + d]], [0, 1], boxes)


def test_empty_boxes_launch_nothing_and_the_call_is_stream_ordered(ctx, pinned):
    import torch

    seg = _pool(4096)
    launches = ctx.launch_count
    ctx.copy_boxes_from_host([seg.data_ptr()], [4096], [0, 1], [(0, 0, 0, 9, 0, 0), (0, 5, 9, 0, 3, 1)], pinned)
    ctx.copy_boxes_from_host([seg.data_ptr()], [4096], [0, 1], [], pinned)
    assert ctx.launch_count == launches
    stream = torch.cuda.Stream()
    dst = _pool(32 * MiB + 5)
    busy = torch.empty(64 * MiB, dtype=torch.float32, device="cuda")
    pinned[: 65 * MiB] = np.random.default_rng(9).integers(0, 256, 65 * MiB, dtype=np.uint8)
    torch.cuda.synchronize()
    rows, w = (32 * MiB + 2) // 4096, 4096
    with torch.cuda.stream(stream):
        for _ in range(20):
            busy.normal_()
        dst.fill_(1)
        ctx.copy_boxes_from_host([dst.data_ptr()], [dst.numel()], [0, 1], [(0, 3, w, rows, 257, 2 * w)], pinned,
                                 stream.cuda_stream)
    stream.synchronize()
    got = dst.cpu().numpy()
    want = pinned[_rows((0, 3, w, rows, 257, 2 * w))]
    assert got[:3].tolist() == [1, 1, 1] and np.array_equal(got[3 : 3 + rows * w], want)
    assert (got[3 + rows * w :] == 1).all()


def test_bad_arguments_are_rejected_before_anything_is_enqueued(ctx, pinned):
    import torch

    seg = _pool(4096)
    seg.fill_(CANARY)
    host = torch.empty(4096, dtype=torch.uint8)
    pageable = np.zeros(8192, np.uint8)
    ok = dict(ptrs=[seg.data_ptr()], lens=[4096], first=[0, 1], boxes=[(0, 0, 10, 10, 0, 10), (0, 200, 7, 3, 1, 9)],
              src=pinned[:4096])
    cases = {
        "host segment": dict(ptrs=[host.data_ptr()]),
        "NULL segment": dict(ptrs=[0]),
        "segment whose address range wraps": dict(lens=[2**64 - seg.data_ptr() + 16]),
        "file_first_seg not ending at nsegs": dict(first=[0, 2]),
        "file that does not exist": dict(boxes=[(1, 0, 1, 1, 0, 1)]),
        "destination past the end of its file": dict(boxes=[(0, 4000, 10, 10, 0, 10)]),
        "rows * width overflows": dict(boxes=[(0, 0, 1 << 33, 1 << 33, 0, 1 << 33)]),
        "offset + rows * width overflows": dict(boxes=[(0, 2**64 - 8, 4, 4, 0, 4)]),
        "pitch below the width": dict(boxes=[(0, 0, 10, 2, 0, 9)]),
        "source past h_src_bytes": dict(boxes=[(0, 0, 10, 10, 4000, 10)]),
        "source pitch overflows": dict(boxes=[(0, 0, 1, 3, 0, 2**63)]),
        "source offset overflows": dict(boxes=[(0, 0, 16, 1, 2**64 - 8, 16)]),
        "overlapping destinations": dict(boxes=[(0, 0, 10, 10, 0, 10), (0, 99, 1, 1, 0, 1)]),
        "the same tensor in two files": dict(ptrs=[seg.data_ptr()] * 2, lens=[4096] * 2, first=[0, 1, 2],
                                             boxes=[(0, 0, 100, 1, 0, 100), (1, 50, 10, 1, 0, 10)]),
        "source not page-locked": dict(src=pageable[:4096]),
    }
    for name, change in cases.items():
        a = {**ok, **change}
        launches = ctx.launch_count
        with pytest.raises(_lib.B200HashError, match=r"\(-1\)"):
            ctx.copy_boxes_from_host(a["ptrs"], a["lens"], a["first"], a["boxes"], a["src"])
        assert ctx.launch_count == launches, name
    torch.cuda.synchronize()
    assert (seg.cpu().numpy() == CANARY).all()


def test_load_boxes_orders_after_earlier_reads(gpu_backend):
    """As load_ranges: a kernel queued before the call sees the old bytes, work queued after it the new ones."""
    import torch

    t = torch.full((256 * MiB,), 3, dtype=torch.uint8, device="cuda")
    busy = torch.empty(64 * MiB, dtype=torch.float32, device="cuda")
    src = gpu_backend.host_alloc(512 * MiB + 4096)
    try:
        src[:] = 9
        f = DeviceFile(t)
        for _ in range(20):
            busy.normal_()
        before = t.sum(dtype=torch.int64)
        loaded = load_boxes([f], [(0, 0, 4096, t.numel() // 4096, 5, 8192)], src)
        after = t.sum(dtype=torch.int64)
        loaded.wait()
        assert int(before) == 3 * t.numel() and int(after) == 9 * t.numel()
    finally:
        torch.cuda.synchronize()
        gpu_backend.host_free(src)


# ----------------------------------------------------------------------------------------- end to end


def llama_layers(total: int, seed: int = 0, device="cuda"):
    """A Llama-shaped bf16 layer stack of about ``total`` bytes (hidden 2048, kv 512, intermediate 5632)."""
    import torch

    g = torch.Generator(device=device).manual_seed(seed)
    H, KV, I = 2048, 512, 5632
    shapes = {"q_proj": (H, H), "k_proj": (KV, H), "v_proj": (KV, H), "o_proj": (H, H), "gate_proj": (I, H),
              "up_proj": (I, H), "down_proj": (H, I), "input_layernorm": (H,), "post_attention_layernorm": (H,)}
    per = sum(int(np.prod(s)) * 2 for s in shapes.values())
    sd = {}
    for i in range(max(1, total // per)):
        for name, shape in shapes.items():
            sd[f"layers.{i}.{name}.weight"] = torch.randn(shape, device=device, generator=g).to(torch.bfloat16)
    return sd


def tp_select(names_shapes, rank: int, ranks: int = 8, dim: int | None = None):
    """Rank ``rank``'s slices: q/k/v/gate/up on dim 0, o/down on dim 1, norms whole (or every matrix on ``dim``)."""
    out = {}
    for name, shape in names_shapes.items():
        if len(shape) == 1:
            out[name] = ...
            continue
        d = dim if dim is not None else (1 if ("o_proj" in name or "down_proj" in name) else 0)
        n = shape[d] // ranks
        out[name] = (slice(None),) * d + (slice(rank * n, (rank + 1) * n),)
    return out


def test_every_tp_rank_of_a_1gib_state_dict(gpu_backend):
    import torch

    sd = llama_layers(GiB)
    header, order = safetensors_layout(sd)
    meta = json.loads(header[8:])
    BS = blob_utils.BLOCK_SIZE

    def predicted_blocks(select):
        out = set()
        for name, index in select.items():
            start = len(header) + meta[name]["data_offsets"][0]
            shape = sd[name].shape
            if index is ...:
                out.update(range(start // BS, (start + sd[name].numel() * 2 - 1) // BS + 1))
                continue
            d, sl = len(index) - 1, index[-1]
            if d == 0:
                lo, hi = start + sl.start * shape[1] * 2, start + sl.stop * shape[1] * 2
                out.update(range(lo // BS, (hi - 1) // BS + 1))
            else:
                s = start + np.arange(shape[0], dtype=np.int64) * shape[1] * 2 + sl.start * 2
                e = s + (sl.stop - sl.start) * 2 - 1
                for a, b in zip((s // BS).tolist(), (e // BS).tolist()):
                    out.update(range(a, b + 1))
        return out

    async def run():
        async with running_volume_server(BS) as (stub, faults):
            client = types.SimpleNamespace(stub=stub)
            batch = volume.VolumeUploadContextManager2("vo-g", client)
            async with batch:
                batch.put_file(DeviceFile.safetensors(sd), "/m.safetensors")
            full = await volume.read_safetensors(client, "vo-g", "/m.safetensors")
            _, info = await volume.read_safetensors_header(client, "vo-g", "/m.safetensors")
            shapes = {k: s for k, (_, s) in info.items()}
            for dim in (0, 1, None):
                parts = []
                for rank in range(8):
                    select = tp_select(shapes, rank, dim=dim)
                    gets = faults["gets"]
                    torch.cuda.synchronize()
                    base = torch.cuda.memory_allocated()
                    torch.cuda.reset_peak_memory_stats()
                    got = await volume.read_safetensors_slices(client, "vo-g", "/m.safetensors", select,
                                                               staging_bytes=64 * MiB)
                    torch.cuda.synchronize()
                    result = sum(t.numel() * t.element_size() for t in got.values())
                    # what torch allocates: the results, and no whole tensor or span of the file on the way.  The
                    # slack is the caching allocator's rounding of ~100 result tensors; the copy's tables come from
                    # cudaMallocAsync, which this count does not see
                    assert torch.cuda.max_memory_allocated() - base <= result + 4 * MiB, (dim, rank)
                    assert faults["gets"] - gets == 2 + len(predicted_blocks(select)), (dim, rank)
                    assert list(got) == list(select)
                    parts.append(got)
                for name, t in full.items():
                    if t.dim() == 1:
                        assert all(torch.equal(p[name].view(torch.int16), t.view(torch.int16)) for p in parts)
                        continue
                    d = dim if dim is not None else (1 if ("o_proj" in name or "down_proj" in name) else 0)
                    cat = torch.cat([p[name] for p in parts], dim=d)
                    assert torch.equal(cat.view(torch.int16), t.view(torch.int16)), (dim, name)
                del parts

    asyncio.run(run())
