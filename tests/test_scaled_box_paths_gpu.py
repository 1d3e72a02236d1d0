"""GPU: ``load_scaled_boxes_kernel`` (b200hash_stage.cu) against the integer-exact ``reference_dequant`` of
tests/test_fp8_reference_cpu.py, through every branch of its store step and every state of its scale cursor.

The value sets: every FP8 pattern of both formats times every F16 and every BF16 scale, and times the structured F32
scales of ``structured_f32_scales`` (F32 ties, double-rounding pairs, F16 and F32 edges) plus 2^16 random F32
patterns, into all three targets.  Each set goes through three layouts:
  * the fast path of ``scaled_words_out`` (one run of 256-wide rows, one scale per row), at source phase 0 and at a
    phase that takes its two-word branch ``sh + 16 / ds > 16``;
  * a scale reload at every element of ``scale_next`` (the transposed tensor, one scale per column);
  * the element loop (the ``else`` branch: boxes narrower than a destination word, so every word spans box rows and
    seeks the cursor again).
The cursor (``scale_seek`` / ``scale_next`` / ``scale_load``) meets rows narrower than a word, blocks from 1 to above
the dimension and 2^64 - 1 (clamped by the host), source pitches other than C (box rows start mid-row and cross row
edges), coordinates past 2^32 and tensors of up to ~2^62 elements, 64 KiB tile seams inside 3-column blocks, and one
call that mixes formats, targets and scale types with scales at addresses 2 mod 4 and 4 mod 16.

Every result must equal the reference where it is not a NaN and be ``NAN_POLICY``'s NaN where the reference gives a
NaN; the layouts of one value set must give identical bits.  Destinations are surrounded by sentinel bytes that must
survive, and each call makes one launch."""
import numpy as np
import pytest

from modal_client_b200 import _lib
from tests.test_fp8_reference_cpu import NAN, random_f32_scales, reference_dequant, structured_f32_scales
from tests.test_volume_read_fp8_gpu import SENTINEL, box, call, same_or_policy, stage

pytestmark = pytest.mark.gpu

MiB = 1 << 20
F32, F16, BF16, E4M3, E5M2 = _lib.DT_F32, _lib.DT_F16, _lib.DT_BF16, _lib.DT_F8E4M3, _lib.DT_F8E5M2
TARGETS, FORMATS, SCALES = [BF16, F16, F32], [E4M3, E5M2], [F32, F16, BF16]
NAME = {F32: "f32", F16: "f16", BF16: "bf16", E4M3: "e4m3", E5M2: "e5m2"}
SIZE = {F32: 4, F16: 2, BF16: 2}
CHUNK = 1 << 23  # pairs per reference_dequant call on the device: its int64 temporaries stay under 2 GiB


def _t():
    import torch

    return torch


def _dt(code):
    torch = _t()
    return {F32: torch.float32, F16: torch.float16, BF16: torch.bfloat16, E4M3: torch.float8_e4m3fn,
            E5M2: torch.float8_e5m2}[code]


def _iv(code):
    torch = _t()
    return torch.int32 if code == F32 else torch.int16


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0, pinned_bytes=64 << 20, device_bytes=512 << 20)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pinned(ctx):
    buf = ctx.host_alloc(96 * MiB)
    yield buf
    _t().cuda.synchronize()
    ctx.host_free(buf)


def expected(w_bits, fc, s_bits, sc, tc):
    """reference_dequant on the device, as a tc tensor (a quiet NaN where the reference gives its NaN marker)."""
    torch = _t()
    out = torch.empty(w_bits.numel(), dtype=torch.int64, device="cuda")
    for lo in range(0, w_bits.numel(), CHUNK):
        out[lo : lo + CHUNK] = reference_dequant(w_bits[lo : lo + CHUNK], _dt(fc), s_bits[lo : lo + CHUNK], _dt(sc),
                                                 _dt(tc))
    w = 8 * SIZE[tc]
    out = torch.where(out == NAN, torch.full_like(out, (0x7FC00000 if tc == F32 else 0x7FC0 if tc == BF16 else 0x7E00)),
                      out)
    return torch.where(out >= 1 << (w - 1), out - (1 << w), out).to(_iv(tc)).view(_dt(tc))


def scale_tensor(bits, sc):
    """A CUDA tensor of type sc with these bit patterns (int64, any shape)."""
    torch = _t()
    w = 8 * SIZE[sc]
    b = bits.to(torch.int64) & ((1 << w) - 1)
    return torch.where(b >= 1 << (w - 1), b - (1 << w), b).to(_iv(sc)).cuda().view(_dt(sc))


def _bits(s):
    """The zero-extended bit patterns (int64) of a CUDA float tensor."""
    torch = _t()
    return s.view(torch.int32 if s.element_size() == 4 else torch.int16).to(torch.int64) & \
        ((1 << (8 * s.element_size())) - 1)


# --------------------------------------------------------------------------------------------- every value, 3 layouts


def _value_sets():
    return [(sc, fc) for sc in SCALES for fc in FORMATS]


@pytest.mark.parametrize("sc,fc", _value_sets(), ids=[f"{NAME[s]}-scales-{NAME[f]}" for s, f in _value_sets()])
def test_every_fp8_pattern_times_every_scale_through_the_fast_path_the_reload_and_the_element_loop(ctx, pinned, sc, fc):
    """Row i of W (R x 256) holds all 256 patterns and has scale i: every F16 or BF16 pattern, or the structured and
    random F32 scales.  The same pairs go through (a) the fast path, one run with block (1, None), at source phases 0
    and 13 (F32 target) or 9 (16-bit target), both of which take the two-word branch; (b) W^T (256 x R) with block
    (None, 1), so that every element reloads its scale; (c) W read by two interleaved boxes of width 2 (F32 target)
    or 4 (16-bit target) at pitch twice the width, so that every destination word spans box rows (the element loop; a
    pitch equal to the width would be merged into one run by the host)."""
    torch = _t()
    if sc == F32:
        sbits = torch.from_numpy(np.concatenate([structured_f32_scales(), random_f32_scales()]).astype(np.int64))
    else:
        sbits = torch.arange(1 << 16, dtype=torch.int64)
    s = scale_tensor(sbits, sc)
    R, C = s.numel(), 256
    n = R * C
    w = torch.arange(256, dtype=torch.uint8, device="cuda").repeat(R, 1)
    wt = w.t().contiguous()
    w_bits = w.reshape(-1).to(torch.int64)
    s_bits = _bits(s).repeat_interleave(C)
    for tc in TARGETS:
        ds = SIZE[tc]
        want = expected(w_bits, fc, s_bits, sc, tc)
        got = {}
        for sp in (0, 13 if tc == F32 else 9):
            stage(pinned, sp, w.view(_dt(fc)))
            out = call(ctx, pinned, [box(0, n, 1, sp, n, fc, tc, s, sc, 0, R, C, (1, None))], n * ds + 16)
            assert (out[n * ds :] == SENTINEL).all()
            got[f"fast path, source phase {sp}"] = out[: n * ds].view(_dt(tc))
        stage(pinned, 0, wt.view(_dt(fc)))
        out = call(ctx, pinned, [box(0, n, 1, 0, n, fc, tc, s, sc, 0, C, R, (None, 1))], n * ds + 16)
        assert (out[n * ds :] == SENTINEL).all()
        got["a reload at every element"] = out[: n * ds].view(_dt(tc)).reshape(C, R).t().reshape(-1)
        stage(pinned, 0, w.view(_dt(fc)))
        wd = 16 // ds // 2
        rows = n // (2 * wd)
        out = call(ctx, pinned, [box(0, wd, rows, 0, 2 * wd, fc, tc, s, sc, 0, R, C, (1, None)),
                                 box(n // 2 * ds, wd, rows, wd, 2 * wd, fc, tc, s, sc, wd, R, C, (1, None))],
                   n * ds + 16)
        assert (out[n * ds :] == SENTINEL).all()
        got["the element loop"] = out[: n * ds].view(_dt(tc)).reshape(2, rows, wd).transpose(0, 1).reshape(-1)
        first = None
        for path, g in got.items():
            same_or_policy(g, want, tc, (NAME[sc], NAME[fc], NAME[tc], path))
            if first is None:
                first = g.view(_iv(tc))
            assert torch.equal(g.view(_iv(tc)), first), path


# --------------------------------------------------------------------------------------------- boxes of any layout


class Tensor:
    """An R x C FP8 tensor in blocks (br, bc) with its scales: ``src`` is where element 0 would be staged."""

    def __init__(self, R, C, block, fc, sc, scales, src):
        self.R, self.C, self.block, self.fc, self.sc, self.s, self.src = R, C, block, fc, sc, scales, src
        self.br, self.bc = min(block[0] or R, R), min(block[1] or C, C)

    def scale_index(self, e):
        """The flat form: the scale of tensor element e (row-major) is (e / C / br) * ceil(C / bc) + (e mod C) / bc."""
        return e // self.C // self.br * (-(-self.C // self.bc)) + e % self.C // self.bc


def scales_for(R, C, block, sc, g):
    """Random finite scales of type sc, one per block, with exponents spread over +-20 binades."""
    torch = _t()
    br, bc = min(block[0] or R, R), min(block[1] or C, C)
    n = -(-R // br) * -(-C // bc)
    v = (torch.rand(n, generator=g) * 4 - 2) * 2.0 ** torch.randint(-20, 20, (n,), generator=g).float()
    return v.to(_dt(sc)).cuda()


def run_boxes(ctx, pinned, boxes, segments=1, where=""):
    """boxes: (tensor, first, rows, width, pitch, tc); box k reads element first + r * pitch + c of its tensor from
    pinned[tensor.src + first + r * pitch + c].  ONE call: destinations packed in order, each at its own phase with a
    16-byte sentinel gap before it, over ``segments`` segments of one file.  Checks every box against the reference
    and every gap and tail for sentinels."""
    torch = _t()
    per = -(-len(boxes) // segments)
    groups = [boxes[i : i + per] for i in range(0, len(boxes), per)]
    tuples, spans, seg_lens, at = [], [], [], 0
    for gi, group in enumerate(groups):
        base = at
        for k, (t, first, rows, width, pitch, tc) in enumerate(group):
            ds = SIZE[tc]
            at = -(-(at + 16) // 16) * 16 + (k % (16 // ds)) * ds
            tuples.append(box(at, width, rows, t.src + first, pitch, t.fc, tc, t.s, t.sc, first, t.R, t.C, t.block))
            spans.append((at, rows * width * ds))
            at += rows * width * ds
        at = -(-(at + 16) // 16) * 16
        seg_lens.append(at - base)
    segs = [torch.full((m,), SENTINEL, dtype=torch.uint8, device="cuda") for m in seg_lens]
    torch.cuda.synchronize()
    launches = ctx.launch_count
    ctx.copy_scaled_boxes_from_host([x.data_ptr() for x in segs], seg_lens, [0, len(segs)], tuples, pinned,
                                    torch.cuda.current_stream().cuda_stream or 1)
    torch.cuda.synchronize()
    assert ctx.launch_count == launches + 1
    image = torch.cat(segs)
    clean = torch.ones(image.numel(), dtype=torch.bool, device="cuda")
    for (t, first, rows, width, pitch, tc), (a, nb) in zip(boxes, spans):
        rc = (torch.arange(rows, device="cuda")[:, None] * pitch + torch.arange(width, device="cuda")[None, :]).reshape(-1)
        lo, hi = t.src + first, t.src + first + (rows - 1) * pitch + width
        raw = torch.from_numpy(pinned[lo:hi].copy()).cuda().to(torch.int64)
        e = first + rc
        want = expected(raw[rc], t.fc, _bits(t.s)[t.scale_index(e)], t.sc, tc)
        same_or_policy(image[a : a + nb].view(_dt(tc)), want, tc, (where, t.R, t.C, t.block, first, rows, width, pitch,
                                                                   NAME[t.fc], NAME[tc], NAME[t.sc]))
        clean[a : a + nb] = False
    assert (image[clean] == SENTINEL).all(), where


def _random_bytes(pinned, at, n, g):
    torch = _t()
    pinned[at : at + n] = torch.randint(0, 256, (n,), generator=g, dtype=torch.uint8).numpy()


BLOCK_SIZES = [1, 2, 3, 5, 7, 16, 128, "above", 2**64 - 1]


def _blocks(R, C):
    """(br, bc) pairs: every size as bc with br cycling through them, and every size as br with bc cycling."""
    size = lambda v, dim: dim + 3 if v == "above" else v  # noqa: E731
    n = len(BLOCK_SIZES)
    pairs = [(BLOCK_SIZES[(k * 4 + 1) % n], BLOCK_SIZES[k]) for k in range(n)]
    pairs += [(BLOCK_SIZES[k], BLOCK_SIZES[(k * 2 + 3) % n]) for k in range(n)]
    return [(size(a, R), size(b, C)) for a, b in pairs]


@pytest.mark.parametrize("C", [1, 2, 3, 5, 7, 8, 9, 15, 16, 17, 33])
def test_scale_cursor_across_narrow_rows_small_blocks_and_clamped_blocks(ctx, pinned, C):
    """A 41 x C tensor (rows narrower than a destination word for C < 16 / ds, so one word crosses several tensor rows
    and block rows; block columns narrower than a word, so one word reloads its scale several times) in 18 blocks
    (br, bc) from 1 to above the dimension and 2^64 - 1, read as one whole-tensor run and as column slices at odd
    bounds; every format, target and scale type, one call per target."""
    torch = _t()
    g = torch.Generator().manual_seed(100 + C)
    R = 41
    _random_bytes(pinned, 5, R * C, g)
    slices = sorted({(c0, c1) for c0, c1 in ((1, C - 1), (C // 3, C), (0, (C + 1) // 2), (C - 1, C))
                     if 0 <= c0 < c1 <= C and (c0, c1) != (0, C)})
    for tc in TARGETS:
        boxes = []
        for k, block in enumerate(_blocks(R, C)):
            fc, sc = FORMATS[k % 2], SCALES[k % 3]
            t = Tensor(R, C, block, fc, sc, scales_for(R, C, block, sc, g), 5)
            boxes.append((t, 0, 1, R * C, R * C, tc))
            boxes += [(t, c0, R, c1 - c0, C, tc) for c0, c1 in slices]
        run_boxes(ctx, pinned, boxes, where=("C", C, NAME[tc]))


@pytest.mark.parametrize("C", [1, 3, 8, 17, 33, 300])
def test_source_pitches_other_than_the_row_length(ctx, pinned, C):
    """Pitches C + 1, C + 3, 2C and 3C - 1 (element first + r * pitch + c): box rows start mid-row and cross tensor-row
    and block edges.  Widths 1, C and pitch - 1; first elements 0 and 3."""
    torch = _t()
    g = torch.Generator().manual_seed(200 + C)
    R = 37
    _random_bytes(pinned, 11, R * C, g)
    for tc in TARGETS:
        boxes = []
        for k, pitch in enumerate((C + 1, C + 3, 2 * C, 3 * C - 1)):
            if pitch < 2:
                continue
            block = [(3, 2), (1, 5), (7, None), (2, 1)][k]
            fc, sc = FORMATS[k % 2], SCALES[(k + C) % 3]
            t = Tensor(R, C, block, fc, sc, scales_for(R, C, block, sc, g), 11)
            for width in sorted({1, C, pitch - 1}):
                for first in (0, 3):
                    if first + width > R * C:
                        continue
                    rows = (R * C - first - width) // pitch + 1
                    boxes.append((t, first, rows, width, pitch, tc))
        run_boxes(ctx, pinned, boxes, where=("pitch", C, NAME[tc]))


def test_coordinates_past_2_to_the_32_and_tensors_near_2_to_the_62(ctx, pinned):
    """Only the boxes' bytes are staged.  R * C >= 2^40 with rows longer than 2^32 (300 x (2^33 + 7)) and shorter
    (2^20 + 3 x 2^20 + 5), and (2^31 - 1) x (2^31 + 11), about 2^62 elements: first elements past 2^32, box rows across
    block-column and tensor-row edges there, multi-row boxes at small pitches, and boxes ending at element R * C - 1."""
    torch = _t()
    g = torch.Generator().manual_seed(300)
    shapes = [(300, 2**33 + 7, (7, 2**31 + 1)), (2**20 + 3, 2**20 + 5, (1000, 999)),
              ((1 << 31) - 1, (1 << 31) + 11, ((1 << 24) + 1, (1 << 24) - 3))]
    at = 0
    boxes = []
    for k, (R, C, block) in enumerate(shapes):
        br, bc = block
        n = R * C
        assert n >= 1 << 40
        row = -(-(1 << 32) // C) + 5  # a row whose first element lies past 2^32
        edge = -(-row // br) * br  # and a row that starts a block row, past it
        layouts = [
            (row * C + 3 * bc - 50, 1, 200, 200),  # across a block-column edge
            (edge * C - 33, 1, 100, 100),  # across a tensor-row edge that is also a block-row edge
            (row * C + 2 * bc - 7, 4, 31, 1000),  # 4 rows at pitch 1000, across a block-column edge
            (n - 77, 1, 77, 77),  # ends at element R * C - 1
            (n - 1 - 2 * 513 - 40 + 1, 3, 40, 513),  # 3 rows, the last ending at element R * C - 1
            (n - 1, 1, 1, 1),
        ]
        for j, (first, rows, width, pitch) in enumerate(layouts):
            assert first >= 1 << 32 and first + (rows - 1) * pitch + width <= n
            fc, sc = FORMATS[(k + j) % 2], SCALES[(k + j) % 3]
            span = (rows - 1) * pitch + width
            at = -(-at // 16) * 16 + 16 + j  # every source phase from 0 to 5
            _random_bytes(pinned, at, span, g)
            t = Tensor(R, C, block, fc, sc, scales_for(R, C, block, sc, g), at - first)
            boxes += [(t, first, rows, width, pitch, tc) for tc in TARGETS]
            at += span
    run_boxes(ctx, pinned, boxes, where="large")


def test_one_call_mixing_formats_targets_and_scale_types(ctx, pinned):
    """One box per (format, target, scale type), each with its own tensor, shape, block and scales; F16 / BF16 scales
    at addresses 2 mod 4 and F32 scales at 4 mod 16; destinations in three segments of one file."""
    torch = _t()
    g = torch.Generator().manual_seed(400)
    rng = np.random.default_rng(400)
    store = torch.empty(8 * MiB, dtype=torch.uint8, device="cuda")
    sat, at, boxes = 0, 0, []
    for fc in FORMATS:
        for tc in TARGETS:
            for sc in SCALES:
                R, C = int(rng.integers(20, 300)), int(rng.integers(1, 300))
                block = (int(rng.choice([1, 3, 16, 128, R + 1])), int(rng.choice([1, 2, 7, 32, 128, C])))
                s = scales_for(R, C, block, sc, g)
                nb = s.numel() * SIZE[sc]
                sat = -(-sat // 16) * 16 + 16 + (4 if sc == F32 else 2)
                placed = store[sat : sat + nb].view(_dt(sc))
                placed.copy_(s)
                assert placed.data_ptr() % (16 if sc == F32 else 4) == (4 if sc == F32 else 2)
                sat += nb
                at = -(-at // 16) * 16 + 16 + int(rng.integers(0, 16))
                _random_bytes(pinned, at, R * C, g)
                t = Tensor(R, C, block, fc, sc, placed, at)
                r0, c0 = int(rng.integers(0, R // 2)), int(rng.integers(0, C))
                r1, c1 = int(rng.integers(r0 + 1, R + 1)), int(rng.integers(c0 + 1, C + 1))
                boxes.append((t, r0 * C + c0, r1 - r0, c1 - c0, C, tc))
                at += R * C
    run_boxes(ctx, pinned, boxes, segments=3, where="mixed")


def test_tile_seams_inside_three_column_blocks(ctx, pinned):
    """Rows of 70 001 elements (more than 64 KiB, so tile seams fall at every phase inside rows) in blocks (2, 3):
    a whole-tensor run and a box of rows 1 .. 4 columns 5 .. 69 995, at source phase 3."""
    torch = _t()
    g = torch.Generator().manual_seed(500)
    R, C = 5, 70_001
    _random_bytes(pinned, 3, R * C, g)
    for fc in FORMATS:
        boxes = []
        for tc in TARGETS:
            for sc in (F32, BF16):
                t = Tensor(R, C, (2, 3), fc, sc, scales_for(R, C, (2, 3), sc, g), 3)
                boxes += [(t, 0, 1, R * C, R * C, tc), (t, C + 5, 4, C - 10, C, tc)]
        run_boxes(ctx, pinned, boxes, where=("seams", NAME[fc]))
