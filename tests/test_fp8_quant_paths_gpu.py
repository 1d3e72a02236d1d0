"""GPU: the FP8 export kernels (b200hash_stage.cu) against the integer-exact reference of
tests/test_fp8_quant_reference_cpu.py, through every branch of the quantizing store and the amax reduction.

``stage_scaled_ranges_kernel`` (``copy_scaled_ranges``, ``hash_scaled_segment_parts_device``) gets a passed straight
in, one block per row, and quantizes these value sets:
  * every F16 and BF16 pattern with |x| <= a, for every structured a (the multiplier's hard cases, the 1e-4 floor and
    its neighbours, powers of two, 448, 65504, a in (2^126, FLT_MAX] whose reciprocal is an F32 subnormal, inf, NaNs);
  * the structured F32 set (x solved so that RN(x * m) lands on every E4M3 tie and 1 ulp either side, on double
    rounding pairs, on [448, 464) and on +-2^-10) plus 2^24 random patterns under their rows' own amax;
  * every finite F32 pattern under a = FLT_MAX, and every F32 pattern in a's top binade for some structured a.
Each set goes through these layouts, which must all give the reference's bits:
  * ``quant_load_word`` at every source phase (0, 4, 8, 12 for F32; 0 .. 14 for the 16-bit types);
  * a reload of m at every element of ``quant_next`` (the transposed weight with block (None, 1));
  * ``scaled_image_word``: quantizing segments of 1 to 15 elements, and words across a quantizing piece and a plain or
    converting piece;
  * ``scaled_image_byte``: ranges of 1 to 15 bytes (tail bytes only);
  * ranges that start at odd element offsets inside a segment (``quant_seek`` mid-row).
The cursor meets C from 1 to 33 in blocks from 1 to C + 1 and 2^64 - 1 columns and 1, 2, 3, R and R + 1 rows, each
block with its own a at least 2x from its neighbours'; ranges past element 2^32 of an 8 GiB weight; ``fp8_amax_kernel``
meets maxima planted at every tile corner of blocks whose tiles have neighbours; the scale call meets NaN payloads,
sNaNs, infinities, the floor, signed zeros, subnormals, and one call that mixes types, block forms, source phases and
d_amax arrays out of order.  Destinations are surrounded by sentinel bytes, in device memory and in page-locked memory,
and every call makes the launches the header promises."""
import hashlib

import numpy as np
import pytest

from modal_client_b200 import _lib
from tests.test_fp8_quant_reference_cpu import (E4M3_MAX, E4M3_NAN, F32_INF, F32_NAN, FLOOR, FLT_MAX,
                                                 random_f32_rows, reference_block_scales, reference_multiplier,
                                                 reference_quant, sixteen_bit_pairs, structured_amax,
                                                 structured_f32_pairs)

pytestmark = pytest.mark.gpu

DEV = "cuda"
MiB = 1 << 20
SENTINEL = 0xC3
CHUNK = 1 << 22  # elements per reference call on the device: its int64 temporaries stay well under 2 GiB
WHOLE = 2**64 - 1  # a block size over the whole dimension (the host clamps it)
F32, F16, BF16, E4M3 = _lib.DT_F32, _lib.DT_F16, _lib.DT_BF16, _lib.DT_F8E4M3
SIZE = {F32: 4, F16: 2, BF16: 2}
NAME = {F32: "f32", F16: "f16", BF16: "bf16"}
CODES = [F32, F16, BF16]


def _t():
    import torch

    return torch


def _dt(code):
    torch = _t()
    return {F32: torch.float32, F16: torch.float16, BF16: torch.bfloat16}[code]


def _current():
    torch = _t()
    return (torch.cuda.current_stream().cuda_stream or 1) if DEV == "cuda" else 0


def _sync():
    if DEV == "cuda":
        _t().cuda.synchronize()


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0, pinned_bytes=64 << 20, device_bytes=512 << 20)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pinned(ctx):
    buf = ctx.host_alloc(64 * MiB)
    yield buf
    _sync()
    ctx.host_free(buf)


def as_tensor(bits, code):
    """A tensor of type ``code`` with these bit patterns (int64, low bits), on their device."""
    torch = _t()
    w = 8 * SIZE[code]
    b = bits.to(torch.int64) & ((1 << w) - 1)
    return torch.where(b >= 1 << (w - 1), b - (1 << w), b).to(torch.int32 if w == 32 else torch.int16).view(_dt(code))


def bits_of(t):
    """The zero-extended bit patterns (int64) of a float tensor."""
    torch = _t()
    w = 8 * t.element_size()
    return t.view(torch.int32 if w == 32 else torch.int16).to(torch.int64) & ((1 << w) - 1)


def expected_q(x_bits, code, m_bits):
    """reference_quant on the device in chunks, as uint8 (m_bits may be an expanded view)."""
    torch = _t()
    out = torch.empty(x_bits.numel(), dtype=torch.uint8, device=x_bits.device)
    for lo in range(0, x_bits.numel(), CHUNK):
        out[lo : lo + CHUNK] = reference_quant(x_bits[lo : lo + CHUNK], _dt(code), m_bits[lo : lo + CHUNK]).to(torch.uint8)
    return out


def check(got, want, where):
    torch = _t()
    bad = got != want
    if bool(bad.any()):
        k = int(bad.nonzero()[0])
        raise AssertionError(f"{where}: {int(bad.sum())} of {want.numel()} codes differ, first at {k}: got "
                             f"{int(got[k]):#04x}, reference {int(want[k]):#04x}")
    assert got.numel() == want.numel() and got.dtype == torch.uint8


def quant_seg(t, code, amax, R, C, block, count=None):
    """A b200h_scaled_segment row (ptr, len, src, dst, amax, count, R, C, br, bc) of the R x C weight ``t``."""
    return [t.data_ptr(), R * C * SIZE[code], code, E4M3, amax.data_ptr(), count or amax.numel(), R, C, block[0],
            block[1]]


def plain_seg(ptr, n, src=0, dst=0):
    return [ptr, n, src, dst, 0, 0, 0, 0, 0, 0]


def _index(offs, lens):
    """Destination byte indices of ranges placed at offs with lengths lens (int64 tensors), in range order."""
    torch = _t()
    total = int(lens.sum())
    base = torch.repeat_interleave(offs - (torch.cumsum(lens, 0) - lens), lens)
    return base + torch.arange(total, device=offs.device)


def copy(ctx, segs, ranges, pinned=None):
    """ONE copy_scaled_ranges call: ranges (image offset, length) of the one file made of ``segs`` (rows of
    ``quant_seg`` / ``plain_seg``), each at its own 16-aligned destination after at least 16 sentinel bytes, in
    page-locked memory when ``pinned`` is given, else in device memory.  Checks that the call made one launch and that
    every byte outside the destinations kept its sentinel; -> the ranges' bytes, in order (uint8 on DEV)."""
    torch = _t()
    segs = np.asarray(segs, dtype=np.uint64).reshape(-1, 10)
    rg = np.asarray(ranges, dtype=np.int64).reshape(-1, 2)
    padded = -(-rg[:, 1] // 16) * 16 + 16
    offs = 16 + np.cumsum(padded) - padded
    at = int(offs[-1] + padded[-1]) if len(rg) else 16
    if pinned is not None:
        assert at <= pinned.size
        dst = pinned[:at]
        dst[:] = SENTINEL
    else:
        dst = torch.full((at,), SENTINEL, dtype=torch.uint8, device=DEV)
    _sync()
    before = ctx.launch_count
    ctx.copy_scaled_ranges(segs[:, 0], segs[:, 1], segs[:, 2], segs[:, 3], segs[:, 4:], [0, len(segs)],
                           np.column_stack([np.zeros(len(rg), np.int64), rg]), dst, offs, _current())
    _sync()
    assert ctx.launch_count == before + (1 if rg[:, 1].any() else 0)
    img = torch.from_numpy(dst.copy()).to(DEV) if pinned is not None else dst
    idx = _index(torch.from_numpy(offs).to(DEV), torch.from_numpy(rg[:, 1].copy()).to(DEV))
    clean = torch.ones(at, dtype=torch.bool, device=DEV)
    clean[idx] = False
    assert bool((img[clean] == SENTINEL).all()), "a byte outside the destinations was written"
    return img[idx]


def cover(n, lens):
    """Consecutive ranges (offset, length) over [0, n) with lengths taken from ``lens`` in turn (the last one cut)."""
    lens = np.asarray(lens, np.int64)
    reps = -(-n // max(int(lens.sum()), 1)) + 1
    cs = np.cumsum(np.tile(lens, reps))
    ends = np.concatenate([cs[cs < n], [n]])
    starts = np.concatenate([[0], ends[:-1]])
    return np.column_stack([starts, ends - starts])


# --------------------------------------------------------------------------------------------- every value, 5 layouts


def _rows(x_bits, a_bits, W):
    """The pairs laid out as rows of W elements under one a each: every run of equal a padded with +0 to whole rows;
    -> (x_bits, a per row)."""
    torch = _t()
    vals, counts = torch.unique_consecutive(a_bits, return_counts=True)
    rows = -(-counts // W)
    starts = torch.cumsum(rows, 0) - rows
    x = torch.zeros(int(rows.sum()) * W, dtype=torch.int64, device=x_bits.device)
    within = torch.arange(x_bits.numel(), device=x_bits.device) - torch.repeat_interleave(torch.cumsum(counts, 0) -
                                                                                          counts, counts)
    x[torch.repeat_interleave(starts * W, counts) + within] = x_bits
    return x, torch.repeat_interleave(vals, rows)


def layouts(ctx, pinned, x_bits, code, a_rows, W, where, element_limit=None):
    """x (R x W, row i under a_rows[i]) through every layout; the element-by-element layouts take the first
    ``element_limit`` elements (whole rows), all of them when None."""
    torch = _t()
    ss = SIZE[code]
    n = x_bits.numel()
    R = n // W
    assert R * W == n and a_rows.numel() == R
    x = as_tensor(x_bits, code)
    a = as_tensor(a_rows, F32)
    want = expected_q(x_bits, code, reference_multiplier(a_rows).repeat_interleave(W))
    for k in range(16 // ss):  # quant_load_word at source phase k * ss
        buf = torch.empty(n + 16 // ss, dtype=x.dtype, device=DEV)
        v = buf[k : k + n]
        v.copy_(x)
        to_pinned = k == 1 and n + 64 <= pinned.size
        got = copy(ctx, [quant_seg(v, code, a, R, W, (1, WHOLE))], [(0, n)], pinned if to_pinned else None)
        check(got, want, (where, "quant_load_word, source phase", k * ss, "page-locked" if to_pinned else "device"))
        del buf, v
    xt = x.view(R, W).t().contiguous()  # W x R, one block per column: m reloads at every element
    got = copy(ctx, [quant_seg(xt, code, a, W, R, (WHOLE, 1))], [(0, n)])
    check(got.view(W, R).t().reshape(-1), want, (where, "a reload at every element"))
    del xt
    m = n if element_limit is None else min(n, element_limit // W * W)
    element_paths(ctx, pinned, x[:m], code, a_rows[: m // W], W, want[:m], where)


def element_paths(ctx, pinned, x, code, a_rows, W, want, where):
    torch = _t()
    ss = SIZE[code]
    n = x.numel()
    R = n // W
    rng = np.random.default_rng(n + code)
    # scaled_image_word: every element its own 1 x L weight (L = 1 .. 15) in blocks (1, 1) under its row's a
    a_el = as_tensor(a_rows.repeat_interleave(W), F32)
    rg = cover(n, np.arange(1, 16))
    segs = np.zeros((len(rg), 10), np.uint64)
    segs[:, 0] = x.data_ptr() + rg[:, 0] * ss
    segs[:, 1] = rg[:, 1] * ss
    segs[:, 2], segs[:, 3] = code, E4M3
    segs[:, 4] = a_el.data_ptr() + rg[:, 0] * 4
    segs[:, 5], segs[:, 6], segs[:, 7], segs[:, 8], segs[:, 9] = rg[:, 1], 1, rg[:, 1], 1, 1
    check(copy(ctx, segs, [(0, n)]), want, (where, "scaled_image_word: quantizing segments of 1 to 15 elements"))
    # scaled_image_word across pieces: 1 .. 3 rows of quantizing weight, then 1 .. 15 plain bytes, or F32 values that
    # convert to BF16 exactly (after one plain byte when the image offset is odd)
    a = as_tensor(a_rows, F32)
    junk = torch.randint(0, 256, (4096,), dtype=torch.uint8, device=DEV)
    conv_bits = torch.randint(0, 1 << 16, (4096,), dtype=torch.int64, device=DEV) & 0xBFFF  # finite BF16 patterns
    conv_src = as_tensor(conv_bits << 16, F32)
    conv_img = as_tensor(conv_bits, BF16).view(torch.uint8)
    segs, parts, r, at = [], [], 0, 0
    while r < R:
        k = min(R - r, int(rng.integers(1, 4)))
        segs.append(quant_seg(x[r * W :], code, a[r:], k, W, (1, WHOLE), count=k))
        parts.append(want[r * W : (r + k) * W])
        at += k * W
        r += k
        if rng.integers(2) or at % 2:
            j, nb = int(rng.integers(0, 4000)), (1 if rng.integers(2) and at % 2 else int(rng.integers(1, 16)))
            segs.append(plain_seg(junk.data_ptr() + j, nb))
            parts.append(junk[j : j + nb])
            at += nb
        if at % 2 == 0 and rng.integers(2):
            j, ne = int(rng.integers(0, 4000)), int(rng.integers(1, 8))
            segs.append(plain_seg(conv_src.data_ptr() + 4 * j, 4 * ne, F32, BF16))
            parts.append(conv_img[2 * j : 2 * (j + ne)])
            at += 2 * ne
    image = torch.cat(parts)
    check(copy(ctx, segs, [(0, at)]), image, (where, "scaled_image_word: words across quantizing and other pieces"))
    one = [quant_seg(x, code, a, R, W, (1, WHOLE))]
    # scaled_image_byte: ranges of 1 to 15 bytes, into page-locked memory (in pieces that fit)
    rg = cover(n, rng.integers(1, 16, 4096))
    per = (pinned.size // 32) - 16
    for lo in range(0, len(rg), per):
        part = rg[lo : lo + per]
        got = copy(ctx, one, part, pinned)
        check(got, want[int(part[0, 0]) : int(part[-1].sum())], (where, "scaled_image_byte: ranges of 1 to 15 bytes"))
    # quant_seek mid-row: ranges that start at odd element offsets (one byte, then even lengths)
    rg = np.concatenate([[[0, 1]], cover(n - 1, 2 * rng.integers(9, 2000, 512)) + [1, 0]])
    check(copy(ctx, one, rg), want, (where, "ranges at odd element offsets"))


@pytest.mark.parametrize("code", [F16, BF16], ids=["f16", "bf16"])
def test_every_16_bit_pattern_under_every_structured_amax_through_every_layout(ctx, pinned, code):
    """57 structured a (infinity and NaN among them), each with every pattern it admits."""
    x, a = sixteen_bit_pairs(_dt(code), device=DEV)
    x, a_rows = _rows(x, a, 64)
    layouts(ctx, pinned, x, code, a_rows, 64, NAME[code])


def test_structured_and_random_f32_sets_through_every_layout(ctx, pinned):
    x, a = structured_f32_pairs()
    x, a_rows = _rows(x.to(DEV), a.to(DEV), 64)
    layouts(ctx, pinned, x, F32, a_rows, 64, "structured f32")
    x, a = random_f32_rows(1 << 24, seed=11, device=DEV)
    layouts(ctx, pinned, x, F32, a[::64].contiguous(), 64, "random f32", element_limit=1 << 20)


def test_every_finite_f32_pattern_under_flt_max(ctx, pinned):
    """m = RN(RN(1 / FLT_MAX) * 448), with RN(1 / FLT_MAX) = 2^-128 an F32 subnormal: a flushed reciprocal would give
    zeros.  Chunks of 2^27 patterns, rows of 4096; the element-by-element layouts take 2^16 of each chunk."""
    torch = _t()
    W, n = 4096, 1 << 27
    for sign in (0, 1 << 31):
        for lo in range(0, F32_INF, n):
            x = (torch.arange(lo, lo + n, dtype=torch.int64, device=DEV).clamp_(max=FLT_MAX)) | sign
            a_rows = torch.full((n // W,), FLT_MAX, dtype=torch.int64, device=DEV)
            layouts(ctx, pinned, x, F32, a_rows, W, ("f32 under FLT_MAX", hex(lo | sign)), element_limit=1 << 16)


TOP_BINADE = [0x40400000, 0x43E00000, FLOOR + 1, 0x477FE000, 0x7F400000, FLT_MAX]


def test_every_f32_pattern_in_the_top_binade_of_a(ctx, pinned):
    """x from a's binade floor up to a, both signs, for a of both rounding directions of m and a > 2^126."""
    torch = _t()
    extra = [a for a in structured_amax() if a < F32_INF and a not in TOP_BINADE]
    for a in TOP_BINADE + extra[:2]:
        lo = a & 0x7F800000
        pos = torch.arange(lo, a + 1, dtype=torch.int64, device=DEV)
        x = torch.cat([pos, pos | (1 << 31)])
        x, a_rows = _rows(x, torch.full_like(x, a), 4096)
        layouts(ctx, pinned, x, F32, a_rows, 4096, ("top binade of", hex(a)), element_limit=1 << 18)


# --------------------------------------------------------------------------------------------- the scale cursor


def _neighbour_amax(gR, gC, rng):
    """a per block (int64 F32 bits, row-major): 2^e * [1, 2) with even e in -8 .. 8, different from the a of every
    block a cursor could confuse it with (left, up, the diagonals above, and the last block of this and the previous
    block row, which a row wrap passes), so that those a are at least 2x apart."""
    e = np.zeros((gR, gC), np.int64)
    for i in range(gR):
        for j in range(gC):
            near = [(i, j - 1), (i - 1, j), (i - 1, j - 1), (i - 1, j + 1), (i, 0), (i - 1, gC - 1)]
            taken = {int(e[p]) for p in near if 0 <= p[0] and 0 <= p[1] < gC and (p[0] < i or p[1] < j)}
            e[i, j] = rng.choice([v for v in range(-8, 9, 2) if v not in taken])
    v = np.ldexp(1 + rng.random((gR, gC)), e).astype(np.float32)
    return _t().from_numpy(v.reshape(-1).view(np.int32).astype(np.int64))


@pytest.mark.parametrize("C", range(1, 34))
def test_scale_cursor_across_block_edges_and_row_wraps(ctx, pinned, C):
    """A 7 x C weight in blocks of 1 .. C + 1 and 2^64 - 1 columns by 1, 2, 3, 7 and 8 rows, one segment each, all in
    one file per source type: the whole image as one range into device memory, and consecutive ranges of 1 to 40 bytes
    (seeks at every element, tail bytes, words across segments) into page-locked memory."""
    torch = _t()
    R = 7
    rng = np.random.default_rng(C)
    g = torch.Generator().manual_seed(C)
    for code in CODES:
        segs, want, keep = [], [], []
        for bc in list(range(1, C + 2)) + [WHOLE]:
            for br in (1, 2, 3, R, R + 1):
                bre, bce = min(br, R), min(bc, C)
                gR, gC = -(-R // bre), -(-C // bce)
                a_bits = _neighbour_amax(gR, gC, rng)
                e = torch.arange(R * C)
                blk = (e // C // bre) * gC + e % C // bce
                u = torch.rand(R * C, generator=g) * 2 - 1
                x = (u * as_tensor(a_bits, F32)[blk]).to(_dt(code)).to(DEV)
                amax = as_tensor(a_bits, F32).to(DEV)
                keep += [x, amax]
                segs.append(quant_seg(x, code, amax, R, C, (br, bc)))
                want.append(expected_q(bits_of(x), code, reference_multiplier(a_bits.to(DEV))[blk.to(DEV)]))
        want = torch.cat(want)
        n = want.numel()
        check(copy(ctx, segs, [(0, n)]), want, ("C", C, NAME[code], "one range"))
        check(copy(ctx, segs, cover(n, rng.integers(1, 41, 997)), pinned), want, ("C", C, NAME[code], "short ranges"))


# --------------------------------------------------------------------------------------------- past 2^32


def _scales(ctx, jobs):
    """ONE fp8_block_scales call over jobs (2-D tensor, code, block); checks its two launches; -> [(a_bits, s_bits)]."""
    torch = _t()
    out, rows = [], []
    for w, code, (br, bc) in jobs:
        R, C = w.shape
        g = -(-R // min(br, R)) * -(-C // min(bc, C))
        a = torch.empty(g, dtype=torch.float32, device=DEV)
        s = torch.empty(g, dtype=torch.float32, device=DEV)
        out.append((a, s))
        rows.append((w.data_ptr(), code, R, C, br, bc, s.data_ptr(), a.data_ptr()))
    _sync()
    before = ctx.launch_count
    ctx.fp8_block_scales(rows, _current())
    _sync()
    assert ctx.launch_count == before + 2
    return [(bits_of(a), bits_of(s)) for a, s in out]


def test_ranges_past_element_2_to_the_32_and_a_per_tensor_amax_there(ctx):
    """One BF16 weight of (2^16 + 1) x 2^16 = 2^32 + 2^16 elements (8 GiB), freed at the end."""
    torch = _t()
    R, C = (1 << 16) + 1, 1 << 16
    n, T = R * C, 1 << 32
    w = torch.empty(n, dtype=torch.bfloat16, device=DEV)
    try:
        w.uniform_(-1, 1)
        gR, gC = -(-R // 128), C // 128
        a_bits = bits_of(torch.rand(gR * gC, device=DEV) * 3 + 1)
        amax = as_tensor(a_bits, F32)
        ranges = [(T - 40, 100), (T, 33), (T + 5, 1000), (T - 5000, 20000), (n - 77, 77), (n - 1, 1)]
        got = copy(ctx, [quant_seg(w, BF16, amax, R, C, (128, 128))], ranges)
        e = torch.cat([torch.arange(o, o + k, device=DEV) for o, k in ranges])
        blk = (e // C // 128) * gC + e % C // 128
        check(got, expected_q(bits_of(w[e]), BF16, reference_multiplier(a_bits)[blk]), "ranges past 2^32")
        for at in (T, n - 1):
            w[at] = 100.0
            (a, s), = _scales(ctx, [(w.view(R, C), BF16, (WHOLE, WHOLE))])
            top = max(int((w[lo : lo + (1 << 28)].view(torch.int16) & 0x7FFF).max()) for lo in range(0, n, 1 << 28))
            ra, rs = reference_block_scales(torch.tensor([top], device=DEV), _dt(BF16), 1, 1, (1, 1))
            assert top == 0x42C8 and int(a[0]) == int(ra) and int(s[0]) == int(rs), (at, hex(int(a[0])))
            w[at] = 0.5
    finally:
        del w
        torch.cuda.empty_cache()


# --------------------------------------------------------------------------------------------- amax tile seams

SEAMS = [((300, 64), (700, 158)), ((40, 5000), (100, 12000)), ((3, 4097), (8, 8294)), ((16385, 1), (40000, 3))]


def _corners(size, sub):
    return sorted({o for s in range(0, size, sub) for o in (s, min(s + sub, size) - 1)})


@pytest.mark.parametrize("block,shape", SEAMS, ids=[f"{b[0]}x{b[1]}" for b, _ in SEAMS])
def test_amax_tile_seams_with_neighbour_blocks(ctx, block, shape):
    """Tiles of at most 4096 columns and 16384 elements (kScaleTileCols / kScaleTileElems): blocks of more rows or
    columns than one tile holds, at least two full blocks and a partial one in each direction (so whole tiles of the
    edge blocks are skipped).  Every block's max is planted at one tile corner offset at a time (the block's last
    element among them; a partial block takes its own last row / column), so that the neighbour's max lies just across
    every seam; the maxima rise with the block index, then fall, so that reading past a seam changes some a."""
    torch = _t()
    R, C = shape
    br, bc = block
    sub_cols = min(bc, 4096)
    sub_rows = min(br, max(1, 16384 // sub_cols))
    gR, gC = -(-R // br), -(-C // bc)
    assert R // br >= 2 and R % br and (C // bc >= 2 and C % bc or bc == 1)
    bi = torch.arange(gR, device=DEV)[:, None].expand(gR, gC)
    bj = torch.arange(gC, device=DEV)[None, :].expand(gR, gC)
    last_r, last_c = torch.clamp((bi + 1) * br, max=R) - 1, torch.clamp((bj + 1) * bc, max=C) - 1
    for code in CODES:
        g = torch.Generator(device=DEV).manual_seed(code)
        base = (torch.rand(R, C, device=DEV, generator=g) - 0.5).to(_dt(code))
        for ro in _corners(br, sub_rows):
            for co in _corners(bc, sub_cols):
                r, c = torch.minimum(bi * br + ro, last_r), torch.minimum(bj * bc + co, last_c)
                for order in (1, -1):
                    w = base.clone()
                    k = torch.arange(gR * gC, device=DEV).view(gR, gC)
                    w[r, c] = (2 + (k if order > 0 else gR * gC - 1 - k)).to(w.dtype)
                    (a, s), = _scales(ctx, [(w, code, block)])
                    ra, rs = reference_block_scales(bits_of(w), _dt(code), R, C, block)
                    where = (NAME[code], block, ro, co, order)
                    assert torch.equal(a, ra.reshape(-1)), (where, a.tolist(), ra.reshape(-1).tolist())
                    assert torch.equal(s, rs.reshape(-1)), where


# --------------------------------------------------------------------------------------------- the scale call's edges

# (patterns of one block) per source type: NaN payloads, sNaNs and negative NaNs; NaN beside infinity; around the floor;
# signed zeros; subnormals; infinities beside finite values of both signs
EDGES = {
    F32: [[0x7F800001, 0x3F800000], [0x7FC00000, 0xBF800000], [0x7FFFFFFF], [0xFF800001, 0x40000000], [0xFFC12345],
          [0x7FA00000, 0x7F800000, 0xFF800000], [FLOOR - 1, 0xB8D1B715], [FLOOR, 0x80000000], [FLOOR + 1, 0x38000000],
          [0x80000000], [0x00000001, 0x807FFFFF, 0x00400000], [0x7F800000, 0xBFC00000, 0x3F000000],
          [0xFF800000, 0xC2C80000, 0x00000001]],
    F16: [[0x7C01, 0x3C00], [0x7E00, 0xBC00], [0xFC01], [0x7FFF, 0x7C00], [0xFE00, 0xFC00, 0x4000], [0x068D, 0x868D],
          [0x068E], [0x068F, 0x8001], [0x8000], [0x0001, 0x83FF, 0x0200], [0x7C00, 0xBE00, 0x3800],
          [0xFC00, 0xD640, 0x0001]],
    BF16: [[0x7F81, 0x3F80], [0xFF81, 0xBF80], [0x7FC0], [0x7FA5, 0x7F80, 0xFF80], [0xFFFF], [0x38D1, 0xB8D1],
           [0x38D2], [0x8000], [0x0001, 0x807F, 0x0040], [0x7F80, 0xBFC0, 0x3F00], [0xFF80, 0xC2C8, 0x0001]],
}


@pytest.mark.parametrize("code", CODES, ids=[NAME[c] for c in CODES])
def test_scale_call_edges_and_their_codes(ctx, code):
    """One block of 4 x 16 per case, its patterns repeated over it: a bit for bit (NaN payloads included), s the
    canonical NaN F32_NAN for a NaN a, every q of a NaN block 0x7F, and in a block with an infinity (m = 0) the finite
    negative elements 0x80, the positive ones 0x00 and the infinities (inf * 0) 0x7F."""
    torch = _t()
    cases = EDGES[code]
    w_bits = torch.cat([torch.tensor(c, dtype=torch.int64).repeat(64)[:64].view(4, 16) for c in cases], 1).to(DEV)
    w = as_tensor(w_bits, code)
    R, C = 4, 16 * len(cases)
    (a, s), = _scales(ctx, [(w, code, (4, 16))])
    ra, rs = reference_block_scales(w_bits, _dt(code), R, C, (4, 16))
    assert torch.equal(a, ra.reshape(-1)), [(hex(int(x)), hex(int(y))) for x, y in zip(a, ra.reshape(-1))]
    assert torch.equal(s, rs.reshape(-1)), [hex(int(x)) for x in s]
    nan = a > F32_INF
    assert bool((s[nan] == F32_NAN).all()) and int(nan.sum()) >= 5
    amax = as_tensor(a, F32)  # held until the copy is done
    got = copy(ctx, [quant_seg(w, code, amax, R, C, (4, 16))], [(0, R * C)]).view(R, C)
    m = reference_multiplier(a)[torch.arange(C, device=DEV) // 16].expand(R, C).reshape(-1)
    check(got.reshape(-1), expected_q(w_bits.reshape(-1), code, m), ("edges", NAME[code]))
    for k, blk in enumerate(got.view(R, len(cases), 16).transpose(0, 1)):
        x = w_bits[:, 16 * k : 16 * (k + 1)]
        if nan[k]:
            assert bool((blk == E4M3_NAN).all()), (NAME[code], k)
        elif int(a[k]) == F32_INF:
            xf = as_tensor(x, code).float()
            assert bool((blk[xf.isinf()] == E4M3_NAN).all())
            assert bool((blk[(xf < 0) & xf.isfinite()] == 0x80).all()) and bool((blk[(xf >= 0) & xf.isfinite()] == 0).all())


def test_one_scale_call_mixing_types_block_forms_phases_and_scattered_amax_arrays(ctx):
    """Nine jobs (three per source type, at source phases of 1 and 3 elements, blocks (128, 128), (7, 5), (1, None),
    (None, 3), ...), whose d_amax arrays lie in reverse order with sentinel gaps, except two that lie back to back.
    The call makes two launches; every array is cleared before the reduction (the sentinel, 0x5A5A5A5A, exceeds the
    bits of every finite |x| here, so an array left uncleared gives a wrong a) and no gap is touched; a and s equal the
    reference.  The memsets are not counted here: torch's profiler, used a second time in one process, was seen to
    record 2 of 8 of them."""
    torch = _t()
    g = torch.Generator(device=DEV).manual_seed(8)
    forms = [(128, 128), (7, 5), (1, WHOLE), (WHOLE, 3), (WHOLE, WHOLE), (16, 1), (3, 4097), (50, 50), (1, 1)]
    shapes = [(300, 257), (33, 17), (5, 9000), (1000, 7), (64, 64), (77, 3), (9, 8200), (120, 99), (3, 5)]
    jobs, srcs = [], []
    for k, ((R, C), block) in enumerate(zip(shapes, forms)):
        code = CODES[k % 3]
        ph = 1 + 2 * (k % 2)
        buf = torch.empty(R * C + ph, dtype=_dt(code), device=DEV)
        w = buf[ph:].view(R, C)
        w.copy_((torch.randn(R, C, device=DEV, generator=g) * 10 ** (k % 5 - 2)).to(w.dtype))
        if k == 4:
            w[3, 3] = float("nan")
        srcs.append(buf)
        jobs.append((w, code, block))
    counts = [-(-R // min(b[0], R)) * -(-C // min(b[1], C)) for (R, C), b in zip(shapes, forms)]
    store = torch.full((sum(counts) + 5 * len(counts) + 5,), 0x5A5A5A5A, dtype=torch.int32, device=DEV)
    at, place = 5, {}
    for k in reversed(range(len(jobs))):  # the last job first; jobs 3 and 4 back to back
        place[k] = at
        at += counts[k] + (0 if k == 4 else 5)
    scales = [torch.empty(c, dtype=torch.float32, device=DEV) for c in counts]
    rows = [(w.data_ptr(), code, w.shape[0], w.shape[1], b[0], b[1], scales[k].data_ptr(),
             store[place[k] :].data_ptr()) for k, (w, code, b) in enumerate(jobs)]
    _sync()
    before = ctx.launch_count
    ctx.fp8_block_scales(rows, _current())
    _sync()
    assert ctx.launch_count == before + 2
    clean = torch.ones(store.numel(), dtype=torch.bool, device=DEV)
    for k, (w, code, block) in enumerate(jobs):
        a = store[place[k] : place[k] + counts[k]].view(torch.float32)
        clean[place[k] : place[k] + counts[k]] = False
        ra, rs = reference_block_scales(bits_of(w.contiguous()), _dt(code), w.shape[0], w.shape[1], block)
        assert torch.equal(bits_of(a), ra.reshape(-1)) and torch.equal(bits_of(scales[k]), rs.reshape(-1)), k
    assert bool((store[clean] == 0x5A5A5A5A).all())


# --------------------------------------------------------------------------------------------- the hash entry


@pytest.mark.parametrize("part_len", [4099, MiB])
def test_hash_entry_digests_equal_hashlib_of_the_reference_image(ctx, part_len):
    """Three files in one call: one mixing quantizing (all three source types), converting and plain segments; one
    whose image ends in 0x00 bytes quantized from non-zero sources; one whose image ends in 0x80 (negative values
    that quantize to -0), which TRIM_ZEROS must keep."""
    torch = _t()
    from tests.test_cast_reference_cpu import reference_cast

    g = torch.Generator(device=DEV).manual_seed(part_len)
    segs, images, ffs, keep = [], [], [0], []

    def quant(w, code, block, tail=None):
        R, C = w.shape
        if tail is not None:
            w.view(-1)[-tail[0] :] = tail[1]
        a, _ = reference_block_scales(bits_of(w), _dt(code), R, C, block)
        amax = as_tensor(a.reshape(-1), F32)
        keep.extend([w, amax])
        segs.append(quant_seg(w, code, amax, R, C, block))
        blk = (torch.arange(R * C, device=DEV) // C // min(block[0], R)) * a.shape[1] + \
            torch.arange(R * C, device=DEV) % C // min(block[1], C)
        images.append(expected_q(bits_of(w).reshape(-1), code, reference_multiplier(a.reshape(-1))[blk]))

    quant(torch.randn(300, 1000, device=DEV, generator=g).to(torch.bfloat16), BF16, (128, 128))
    conv = torch.randn(5001, device=DEV, generator=g)
    keep.append(conv)
    segs.append(plain_seg(conv.data_ptr(), 4 * 5001, F32, BF16))
    images.append(as_tensor(reference_cast(bits_of(conv), torch.float32, torch.bfloat16), BF16).view(torch.uint8))
    raw = torch.randint(0, 256, (12345,), dtype=torch.uint8, device=DEV, generator=g)
    keep.append(raw)
    segs.append(plain_seg(raw.data_ptr(), raw.numel()))
    images.append(raw)
    quant(torch.randn(77, 4099, device=DEV, generator=g) * 1e3, F32, (WHOLE, 64))
    quant(torch.randn(129, 257, device=DEV, generator=g).to(torch.float16), F16, (1, WHOLE))
    ffs.append(len(segs))
    quant(torch.randn(64, 333, device=DEV, generator=g), F32, (16, 16), tail=(5000, 1e-7))
    ffs.append(len(segs))
    quant(torch.randn(64, 333, device=DEV, generator=g).to(torch.bfloat16), BF16, (16, 16), tail=(5000, -1e-7))
    ffs.append(len(segs))
    files = [torch.cat(images[ffs[f] : ffs[f + 1]]).cpu().numpy().tobytes() for f in range(3)]
    assert files[1].endswith(b"\0" * 4000) and files[2].endswith(b"\x80" * 4000)
    seg = np.asarray(segs, dtype=np.uint64)
    parts = [(f, o, min(part_len, len(files[f]) - o)) for f in range(3) for o in range(0, len(files[f]), part_len)]
    for flags in (_lib.SHA256 | _lib.MD5, _lib.SHA256 | _lib.MD5 | _lib.TRIM_ZEROS):
        sha = torch.zeros((len(parts), 32), dtype=torch.uint8, device=DEV)
        md5 = torch.zeros((len(parts), 16), dtype=torch.uint8, device=DEV)
        ends = torch.zeros(len(parts), dtype=torch.int64, device=DEV)
        got = ctx.hash_scaled_segment_parts_device(seg[:, 0], seg[:, 1], seg[:, 2], seg[:, 3], seg[:, 4:], ffs,
                                                   part_len, flags, sha.data_ptr(), md5.data_ptr(), ends.data_ptr(),
                                                   _current())
        _sync()
        assert got == len(parts)
        sha, md5, ends = sha.cpu().numpy(), md5.cpu().numpy(), ends.cpu().tolist()
        for i, (f, o, k) in enumerate(parts):
            body = files[f][o : o + k]
            if flags & _lib.TRIM_ZEROS:
                body = body.rstrip(b"\0")
                assert ends[i] == len(body), (f, o)
            assert sha[i].tobytes() == hashlib.sha256(body).digest(), (flags, f, o)
            assert md5[i].tobytes() == hashlib.md5(body).digest(), (flags, f, o)
        if flags & _lib.TRIM_ZEROS:
            last = [max(i for i, p in enumerate(parts) if p[0] == f) for f in (1, 2)]
            assert ends[last[0]] < parts[last[0]][2] and ends[last[1]] == parts[last[1]][2]


# --------------------------------------------------------------------------------------------- a caller's a


@pytest.mark.parametrize("code", CODES, ids=[NAME[c] for c in CODES])
def test_a_caller_amax_below_the_block_max_saturates(ctx, code):
    """The C ABI quantizes with whatever a it is given.  With a = 1 (m = 448) over values up to +-1000 and +-inf,
    every product of magnitude 448 or more gives 0x7E / 0xFE (satfinite; c10 would give NaN past 464), and +-inf * 448
    gives +-448; NaNs give 0x7F."""
    torch = _t()
    g = torch.Generator(device=DEV).manual_seed(code)
    w = ((torch.rand(16, 256, device=DEV, generator=g) * 2 - 1) * 1000).to(_dt(code))
    w[:, :4] = torch.tensor([float("inf"), -float("inf"), float("nan"), -1.0], device=DEV).to(w.dtype)
    a_bits = torch.full((16,), 0x3F800000, dtype=torch.int64, device=DEV)
    amax = as_tensor(a_bits, F32)
    got = copy(ctx, [quant_seg(w, code, amax, 16, 256, (1, WHOLE))], [(0, w.numel())]).view(16, 256)
    want = expected_q(bits_of(w).reshape(-1), code, reference_multiplier(a_bits).repeat_interleave(256)).view(16, 256)
    check(got.reshape(-1), want.reshape(-1), ("caller a", NAME[code]))
    wf = w.float()
    assert bool((got[wf * 448 >= 448] == E4M3_MAX).all()) and bool((got[wf * 448 <= -448] == 0x80 | E4M3_MAX).all())
    assert bool((got[:, 0] == E4M3_MAX).all()) and bool((got[:, 1] == 0xFE).all()) and bool((got[:, 2] == E4M3_NAN).all())
    assert int((wf.abs() * 448 >= 464).sum()) > 1000  # the region where c10 gives NaN
