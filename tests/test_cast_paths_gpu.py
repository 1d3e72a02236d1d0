"""GPU: every F32 / F16 / BF16 bit pattern through every code path of the two converting copy kernels of
b200hash_stage.cu, against the integer-exact ``reference_cast`` of tests/test_cast_reference_cpu.py.

The value sets: all 65 536 patterns of F16 and of BF16; for F32 the structured set of ``structured_f32`` (every
exponent with the mantissas around every rounding tie, F16 subnormal boundaries, the F16 overflow edge, signed zeros,
infinities, NaNs) plus 2^24 random patterns; and every one of the 2^32 F32 patterns through one element-by-element path
of each kernel (the ``test_every_f32_pattern_*`` sweeps, 256 MiB of F32 at a time).

Every test checks two things for every element, through byte-exact comparison with one expected image:
  (a) non-NaN inputs give exactly ``reference_cast``'s bits, and NaN inputs give a NaN;
  (b) every path gives the bits of the fast path -- stage_ranges_kernel's ``cast_load_word`` at source phase 0 -- for
      the same input, so NaNs too come out the same whichever path a word takes.
The expected image is the fast path's output after it has been checked against (a) (``_fast``), so (b) pins the one
NaN policy of ``NAN_POLICY`` (checked in ``test_nan_policy_of_the_fast_path``) on every path.

Each test names the branch of b200hash_stage.cu its layout forces, so that a change that moves a branch has to move the
test with it.  Destinations are surrounded by sentinel bytes that must survive."""
import hashlib

import numpy as np
import pytest

from modal_client_b200 import DeviceFile, _lib
from tests.test_cast_reference_cpu import NAN, is_nan_bits, reference_cast, structured_f32

pytestmark = pytest.mark.gpu

MiB = 1 << 20
SENTINEL = 0xC3
F32, F16, BF16 = _lib.DT_F32, _lib.DT_F16, _lib.DT_BF16
PAIRS = [(s, d) for s in (F32, F16, BF16) for d in (F32, F16, BF16) if s != d]
NAME = {F32: "f32", F16: "f16", BF16: "bf16"}
IDS = [f"{NAME[s]}-{NAME[d]}" for s, d in PAIRS]
SIZE = {F32: 4, F16: 2, BF16: 2}
CHECK_CHUNK = 1 << 23  # elements per reference_cast call on the device: its int64 temporaries stay under 1 GiB

# The NaN bits the fast path gives (and so every path) for a NaN input with bits x, as measured on an H100 (sm_90a):
# the destination's canonical NaN, sign and payload dropped, except BF16 -> F32, whose exact widening keeps every bit
# (x << 16: sign, payload and a clear quiet bit alike).
NAN_POLICY = {
    (F32, F16): lambda x: 0x7FFF + 0 * x,
    (F32, BF16): lambda x: 0x7FFF + 0 * x,
    (F16, F32): lambda x: 0x7FFFFFFF + 0 * x,
    (F16, BF16): lambda x: 0x7FFF + 0 * x,
    (BF16, F32): lambda x: x << 16,
    (BF16, F16): lambda x: 0x7FFF + 0 * x,
}


def _torch(code):
    import torch

    return {F32: torch.float32, F16: torch.float16, BF16: torch.bfloat16}[code]


def _int(code):
    import torch

    return torch.int32 if code == F32 else torch.int16


def _bits(x, code):
    """The zero-extended bit patterns (int64) of the elements in the integer or float tensor x of type code."""
    import torch

    return x.view(_int(code)).to(torch.int64) & ((1 << (8 * SIZE[code])) - 1)


def _current():
    import torch

    return torch.cuda.current_stream().cuda_stream or 1


@pytest.fixture(scope="module")
def ctx():
    c = _lib.Context(0, pinned_bytes=64 << 20, device_bytes=512 << 20)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pinned(ctx):
    buf = ctx.host_alloc(640 * MiB)
    yield buf
    import torch

    torch.cuda.synchronize()
    ctx.host_free(buf)


_values, _images = {}, {}


def values(st):
    """The value set of source type st, on the device, a multiple of 16 elements."""
    import torch

    if st not in _values:
        if st != F32:
            v = torch.arange(-(1 << 15), 1 << 15, dtype=torch.int32, device="cuda").to(torch.int16)
        else:
            g = torch.Generator(device="cuda").manual_seed(24)
            fixed = torch.from_numpy(structured_f32().view(np.int32)).cuda()
            rnd = torch.randint(-(1 << 31), 1 << 31, (1 << 24,), dtype=torch.int64, device="cuda", generator=g)
            v = torch.cat([fixed, rnd.to(torch.int32)])
            v = torch.cat([v, v[: -v.numel() % 16]]) if v.numel() % 16 else v
        _values[st] = v.view(_torch(st))
    return _values[st]


def _copy(ctx, ptrs, lens, sts, dts, ranges, dst, offsets):
    ctx.copy_cast_ranges(ptrs, lens, sts, dts, [0, len(lens)], ranges, dst, offsets, _current())


def check_against_reference(src_bits, got_bits, st, dt):
    """(a): got equals reference_cast where the input is not a NaN, and is a NaN where it is."""
    import torch

    for lo in range(0, src_bits.numel(), CHECK_CHUNK):
        x, y = src_bits[lo : lo + CHECK_CHUNK], got_bits[lo : lo + CHECK_CHUNK]
        ref = reference_cast(x, _torch(st), _torch(dt))
        nan = ref == NAN
        assert torch.equal(nan, is_nan_bits(x, _torch(st)))
        bad = torch.nonzero((~nan & (y != ref)) | (nan & ~is_nan_bits(y, _torch(dt)))).flatten()[:8]
        assert not bad.numel(), (NAME[st], NAME[dt], [hex(v) for v in x[bad].tolist()],
                                 [hex(v) for v in y[bad].tolist()], [hex(v) for v in ref[bad].tolist()])


def _fast(ctx, src, st, dt):
    """The fast path's image of src (one range over one 256-byte aligned segment from image offset 0: every word takes
    cast_load_word at source phase 0), into device memory, checked against the reference."""
    import torch

    n = src.numel() * SIZE[dt]
    out = torch.full((n + 256,), SENTINEL, dtype=torch.uint8, device="cuda")
    _copy(ctx, [src.data_ptr()], [src.numel() * SIZE[st]], [st], [dt], [(0, 0, n)], out, [128])
    torch.cuda.synchronize()
    assert (out[:128] == SENTINEL).all() and (out[-128:] == SENTINEL).all()
    image = out[128:-128]
    check_against_reference(_bits(src, st), _bits(image, dt), st, dt)
    return image


def image(ctx, pair):
    """The expected image of values(pair[0]) converted to pair[1] (uint8, device)."""
    if pair not in _images:
        _images[pair] = _fast(ctx, values(pair[0]), *pair)
    return _images[pair]


def _mismatch(got, want, where):
    import torch

    bad = torch.nonzero(got != want).flatten()[:8]
    return where, bad.tolist(), got[bad].tolist(), want[bad].tolist()


def stage_and_check(ctx, pinned, segs, ranges, want, where):
    """One copy_cast_ranges call of ``ranges`` (int64 [n, 2] of (image offset, length) in the file of the segments
    ``segs`` = (ptrs, lens, src types, dst types)) into host or device memory, each range at its own 16-byte aligned
    destination with at least 16 sentinel bytes after it; every range's bytes equal ``want[offset : offset + length]``
    (``want``: the file's expected image, uint8 on the device) and every other byte keeps the sentinel."""
    import torch

    ranges = np.asarray(ranges, np.int64).reshape(-1, 2)
    lens = ranges[:, 1]
    room = (lens + 15) // 16 * 16 + 16
    offs = 128 + np.concatenate([[0], np.cumsum(room)[:-1]])
    total = int(offs[-1] + room[-1] + 128)
    if where == "host":
        assert total <= pinned.size
        dst = pinned[:total]
        dst[:] = SENTINEL
    else:
        dst = torch.full((total,), SENTINEL, dtype=torch.uint8, device="cuda")
    launches = ctx.launch_count
    rg = np.zeros((len(ranges), 3), np.int64)
    rg[:, 1:] = ranges
    _copy(ctx, *segs, rg, dst, offs)
    torch.cuda.synchronize()
    assert ctx.launch_count == launches + 1
    got = torch.from_numpy(dst).cuda() if where == "host" else dst
    clean = torch.ones(total, dtype=torch.bool, device="cuda")
    if len(ranges) <= 64:
        for (o, n), at in zip(ranges.tolist(), offs.tolist()):
            assert torch.equal(got[at : at + n], want[o : o + n]), _mismatch(got[at : at + n], want[o : o + n], o)
            clean[at : at + n] = False
    else:
        L = torch.from_numpy(lens).cuda()
        rid = torch.repeat_interleave(torch.arange(len(lens), device="cuda"), L)
        within = torch.arange(int(lens.sum()), device="cuda") - torch.repeat_interleave(torch.cumsum(L, 0) - L, L)
        at = torch.from_numpy(offs).cuda()[rid] + within
        src = torch.from_numpy(ranges[:, 0]).cuda()[rid] + within
        assert torch.equal(got[at], want[src]), _mismatch(got[at], want[src], "bytes")
        clean[at] = False
    assert (got[clean] == SENTINEL).all()
    torch.cuda.synchronize()


def boxes_and_check(ctx, pinned, out, boxes, want):
    """One copy_cast_boxes_from_host call of ``boxes`` (source offsets into ``pinned``) into the device buffer ``out``
    (filled with the sentinel first); the bytes [offset, offset + len(w)) of ``out`` equal w for every (offset, w) in
    ``want``, every other byte keeps the sentinel."""
    import torch

    out.fill_(SENTINEL)
    launches = ctx.launch_count
    ctx.copy_cast_boxes_from_host([out.data_ptr()], [out.numel()], [0, 1], boxes, pinned, _current())
    torch.cuda.synchronize()
    assert ctx.launch_count == launches + 1
    clean = torch.ones(out.numel(), dtype=torch.bool, device="cuda")
    for o, w in want:
        assert torch.equal(out[o : o + w.numel()], w), _mismatch(out[o : o + w.numel()], w, o)
        clean[o : o + w.numel()] = False
    assert (out[clean] == SENTINEL).all()
    torch.cuda.synchronize()


def _raw(st):
    """values(st) as host bytes (numpy uint8)."""
    import torch

    return values(st).view(torch.uint8).cpu().numpy()


# ------------------------------------------------------------------------------------------------ the fast path


@pytest.mark.parametrize("pair", PAIRS, ids=IDS)
def test_nan_policy_of_the_fast_path(ctx, pair):
    """(a) for the fast path itself, and the NaN bits it gives for every NaN of the value set: NAN_POLICY."""
    import torch

    st, dt = pair
    img = image(ctx, pair)
    x, y = _bits(values(st), st), _bits(img, dt)
    nan = is_nan_bits(x, _torch(st))
    assert nan.sum() > 100
    want = NAN_POLICY[pair](x[nan])
    bad = torch.nonzero(y[nan] != want).flatten()[:8]
    assert not bad.numel(), (NAME[st], NAME[dt], [(hex(a), hex(b)) for a, b in zip(x[nan][bad].tolist(),
                                                                                 y[nan][bad].tolist())])
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------ stage_ranges_kernel


WHERE = ["host", "device"]


@pytest.mark.parametrize("where", WHERE)
@pytest.mark.parametrize("pair", PAIRS, ids=IDS)
def test_stage_cast_load_word_at_every_source_phase(ctx, pinned, pair, where):
    """cast_load_word at every element-aligned source phase: the value set is copied to a segment at each phase 0 ..
    15 (step: the source element size), and each segment's image is one range from its first byte.  Every word then
    has ``left >= 16`` and ``((in + p.phase) & (ds - 1)) == 0`` (the image starts every word on an element, phase 0),
    so stage_ranges_kernel takes cast_load_word for it, with ``sh`` = the segment's phase (narrowing, F16 <-> BF16)
    or alternately that phase and that phase + 8 (widening: both sides of its ``sh > 8`` split)."""
    import torch

    st, dt = pair
    src, want = values(st), image(ctx, pair)
    nb = src.numel() * SIZE[st]
    phases = list(range(0, 16, SIZE[st]))
    pool = torch.empty(len(phases) * (nb + 256), dtype=torch.uint8, device="cuda")
    ptrs = []
    for i, p in enumerate(phases):
        at = i * (nb + 256) + p
        pool[at : at + nb] = src.view(torch.uint8)
        ptrs.append(pool.data_ptr() + at)
    L = want.numel()
    segs = (ptrs, [nb] * len(phases), [st] * len(phases), [dt] * len(phases))
    stage_and_check(ctx, pinned, segs, [(i * L, L) for i in range(len(phases))], want.repeat(len(phases)), where)


@pytest.mark.parametrize("where", WHERE)
@pytest.mark.parametrize("pair", PAIRS, ids=IDS)
def test_stage_image_word_mid_element(ctx, pinned, pair, where):
    """image_word for words that start inside an element: ranges of the value set's image from image offsets 1, 2
    and 3 that are not a multiple of the destination size (1 and 3 for 16-bit destinations; 1, 2 and 3 for F32 ones).
    Every word of such a range has ``((in + p.phase) & (ds - 1)) != 0``, so it is built by image_word, byte by byte
    through image_byte and cast_one; the range's last bytes are tail bytes."""
    st, dt = pair
    src, want = values(st), image(ctx, pair)
    segs = ([src.data_ptr()], [src.numel() * SIZE[st]], [st], [dt])
    starts = [o for o in (1, 2, 3) if o % SIZE[dt]]
    stage_and_check(ctx, pinned, segs, [(o, want.numel() - o) for o in starts], want, where)


@pytest.mark.parametrize("where", WHERE)
@pytest.mark.parametrize("pair", PAIRS, ids=IDS)
def test_stage_image_word_across_pieces(ctx, pinned, pair, where):
    """image_word for words across pieces: the value set split into converting segments of 1 .. 7 elements (1 .. 3
    when the destination is F32, so that no piece holds 16 image bytes), with plain segments of 1 .. 5 bytes between
    them (two when one would leave the next converting segment's image off a multiple of its element size).  No piece
    then has ``left >= 16``, so every word of the one range over the whole file is assembled by image_word, walking
    the pieces.  For F32 sources the random part of the set is cut to 2^20 patterns here: every segment costs the
    library two pointer lookups when the call is checked."""
    import torch

    st, dt = pair
    ss, ds = SIZE[st], SIZE[dt]
    src, want = values(st), image(ctx, pair)
    n = src.numel() if st != F32 else src.numel() - (1 << 24) + (1 << 20)
    rng = np.random.default_rng(st * 10 + dt)
    per = rng.integers(1, (7 if ds == 2 else 3) + 1, n)
    per = per[np.cumsum(per) <= n]
    per = np.append(per, n - per.sum()) if per.sum() < n else per
    first = np.concatenate([[0], np.cumsum(per)[:-1]])
    g1 = rng.integers(1, 6, len(per))
    g2 = (-g1) % ds
    plain = torch.randint(0, 256, (8 * MiB,), dtype=torch.uint8, device="cuda")
    pofs = rng.integers(0, plain.numel() - 16, (len(per), 2))
    k = len(per)
    ptrs = np.stack([src.data_ptr() + first * ss, plain.data_ptr() + pofs[:, 0], plain.data_ptr() + pofs[:, 1]], 1)
    lens = np.stack([per * ss, g1, g2], 1)
    sts = np.tile([st, 0, 0], (k, 1))
    dts = np.tile([dt, 0, 0], (k, 1))
    # the expected image: per segment, its bytes in `bank` = want || plain
    starts = np.stack([first * ds, want.numel() + pofs[:, 0], want.numel() + pofs[:, 1]], 1)
    ilens = np.stack([per * ds, g1, g2], 1)
    keep = (lens > 0).reshape(-1)
    ptrs, lens, sts, dts = (a.reshape(-1)[keep] for a in (ptrs, lens, sts, dts))
    starts, ilens = starts.reshape(-1)[keep], ilens.reshape(-1)[keep]
    bank = torch.cat([want, plain])
    IL = torch.from_numpy(ilens).cuda()
    within = torch.arange(int(ilens.sum()), device="cuda") - torch.repeat_interleave(torch.cumsum(IL, 0) - IL, IL)
    file_image = bank[torch.repeat_interleave(torch.from_numpy(starts).cuda(), IL) + within]
    del within
    stage_and_check(ctx, pinned, (ptrs, lens, sts, dts), [(0, file_image.numel())], file_image, where)


@pytest.mark.parametrize("where", WHERE)
@pytest.mark.parametrize("pair", PAIRS, ids=IDS)
def test_stage_tail_bytes(ctx, pinned, pair, where):
    """The tail bytes: the value set's image cut into consecutive ranges of 1 .. 15 bytes, so every range is one tile
    with ``tile.len & 15`` bytes and no whole word, and every byte of the image is stored by the ``threadIdx.x <
    tail`` branch (image_byte of the piece find_piece returns), starting at every residue of an element."""
    st, dt = pair
    src, want = values(st), image(ctx, pair)
    rng = np.random.default_rng(dt * 10 + st)
    n = want.numel()
    lens = rng.integers(1, 16, n // 4)
    lens = lens[np.cumsum(lens) <= n]
    lens = np.append(lens, n - lens.sum()) if lens.sum() < n else lens
    assert lens.max() < 16
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]])
    segs = ([src.data_ptr()], [src.numel() * SIZE[st]], [st], [dt])
    stage_and_check(ctx, pinned, segs, np.stack([offs, lens], 1), want, where)


# -------------------------------------------------------------------------------------------- load_boxes_kernel


@pytest.mark.parametrize("pair", PAIRS, ids=IDS)
def test_box_ring_path_at_every_source_and_destination_phase(ctx, pinned, pair):
    """The ring path of cast_words_out: the value set as a one-row box from every element-aligned source phase into
    every element-aligned destination phase.  A one-row box is one run, so every word whose 16 bytes lie in the box
    has ``c + 16 / ds <= welems`` and is built from the ring with shift_bytes at ``sh`` = (source address & 15) and
    cast_word; the words at the box's ends and at the seams of its 64 KiB tiles take the element loop."""
    import torch

    st, dt = pair
    ss, ds = SIZE[st], SIZE[dt]
    raw, want = _raw(st), image(ctx, pair)
    L = want.numel()
    dphases = list(range(0, 16, ds))
    out = torch.empty(len(dphases) * (L + 256), dtype=torch.uint8, device="cuda")
    for sp in range(0, 16, ss):
        pinned[sp : sp + raw.size] = raw
        boxes = [(0, i * (L + 256) + 128 + dq, raw.size, 1, sp, raw.size, st, dt) for i, dq in enumerate(dphases)]
        boxes_and_check(ctx, pinned, out, boxes, [(b[1], want) for b in boxes])


def _rows_box(ctx, pinned, pair, w, pitch, sp, dq):
    """The value set as rows of w elements, ``pitch`` source bytes apart, from source phase sp, into one device buffer
    from destination byte 128 + dq; the elements that do not fill a row are one more box of one row."""
    import torch

    st, dt = pair
    ss, ds = SIZE[st], SIZE[dt]
    raw, want = _raw(st), image(ctx, pair)
    n = raw.size // ss
    rows, rest = n // w, n % w
    span = sp + rows * pitch + rest * ss
    assert span <= pinned.size
    pinned[:span] = 0xA5  # the bytes between rows: never to be converted
    pinned[sp : sp + rows * pitch].reshape(rows, pitch)[:, : w * ss] = raw[: rows * w * ss].reshape(rows, w * ss)
    pinned[sp + rows * pitch : span] = raw[rows * w * ss :]
    out = torch.empty(want.numel() + 256 + dq, dtype=torch.uint8, device="cuda")
    boxes = [(0, 128 + dq, w * ss, rows, sp, pitch, st, dt)]
    if rest:
        boxes.append((0, 128 + dq + rows * w * ds, rest * ss, 1, sp + rows * pitch, rest * ss, st, dt))
    boxes_and_check(ctx, pinned, out, boxes, [(128 + dq, want)])


@pytest.mark.parametrize("pair", PAIRS, ids=IDS)
def test_box_element_loop(ctx, pinned, pair):
    """The element loop of cast_words_out: the value set as rows of one element with ``pitch = width + ss`` (rows
    whose hulls touch: ``hull == 0``) and ``pitch = width + 16`` (a hull per row), then rows of 2 .. 16 / ds - 1
    elements.  A row never fills a destination word, ``c + 16 / ds <= welems`` never holds, so every word is built
    element by element, across rows."""
    st, dt = pair
    ss, ds = SIZE[st], SIZE[dt]
    layouts = [(1, 2 * ss), (1, ss + 16)] + [(w, (w + 1) * ss) for w in range(2, 16 // ds)]
    for i, (w, pitch) in enumerate(layouts):
        _rows_box(ctx, pinned, pair, w, pitch, sp=(i * ss) % 16, dq=(i * ds) % 16)


@pytest.mark.parametrize("pair", PAIRS, ids=IDS)
def test_box_tile_seams(ctx, pinned, pair):
    """The seams of a box's 64 KiB tiles: rows of 3001 elements (no row count fits a tile's 4096 virtual words), with
    a hull per row (``pitch - width >= 16``) and with touching hulls, from a source phase other than 0 into a
    destination phase other than 0.  A tile's first and last destination words hold elements of both tiles; each tile
    stores its own through the element loop, and every other word of the box takes the ring path."""
    st, dt = pair
    ss, ds = SIZE[st], SIZE[dt]
    for pitch in (3001 * ss + 48, 3001 * ss + ss):
        _rows_box(ctx, pinned, pair, 3001, pitch, sp=16 - ss, dq=ds)


# ------------------------------------------------------------------------------------ every F32 pattern, twice


def _f32_chunks():
    import torch

    n = 1 << 26  # 256 MiB of F32 at a time
    idx = torch.arange(n, dtype=torch.int64, device="cuda")
    for k in range(1 << 32 >> 26):
        bits = idx + k * n
        yield k, n, torch.where(bits >= 1 << 31, bits - (1 << 32), bits).to(torch.int32)


def test_every_f32_pattern_through_image_word(ctx):
    """Every F32 pattern to BF16 and to F16 through stage_ranges_kernel's image_word: each chunk's image is read from
    image offset 1, so every word starts inside an element (``((in + p.phase) & (ds - 1)) != 0``).  Its bytes equal
    the fast path's (the chunk's image from offset 0, cast_load_word at phase 0), which is checked against the
    reference."""
    import torch

    for k, n, bits in _f32_chunks():
        src = bits.view(torch.float32)
        for dt in (BF16, F16):
            fast = _fast(ctx, src, F32, dt)
            out = torch.full((2 * n + 256,), SENTINEL, dtype=torch.uint8, device="cuda")
            _copy(ctx, [src.data_ptr()], [4 * n], [F32], [dt], [(0, 1, 2 * n - 1)], out, [128])
            torch.cuda.synchronize()
            assert torch.equal(out[128 : 128 + 2 * n - 1], fast[1:]), _mismatch(out[128 : 128 + 2 * n - 1], fast[1:], k)
            assert (out[:128] == SENTINEL).all() and (out[128 + 2 * n - 1 :] == SENTINEL).all()
            del fast, out
    torch.cuda.synchronize()


def test_every_f32_pattern_through_the_box_element_loop(ctx, pinned):
    """Every F32 pattern to BF16 and to F16 through load_boxes_kernel's element loop: rows of 4 elements, 20 bytes
    apart, from source phase 4, so that no row fills a destination word (``c + 16 / ds <= welems`` never holds).  The
    result equals the fast path's image of the same chunk, which is checked against the reference."""
    import torch

    rows_view = pinned[4 : 4 + (1 << 24) * 20].view(np.uint32).reshape(1 << 24, 5)
    out = torch.empty((1 << 27) + 256, dtype=torch.uint8, device="cuda")
    base = np.arange(1 << 26, dtype=np.uint32).reshape(1 << 24, 4)
    for k, n, bits in _f32_chunks():
        np.add(base, np.uint32(k * n), out=rows_view[:, :4])
        rows_view[:, 4] = 0x7FC0FFEE
        src = bits.view(torch.float32)
        for dt in (BF16, F16):
            fast = _fast(ctx, src, F32, dt)
            boxes_and_check(ctx, pinned, out, [(0, 128, 16, 1 << 24, 4, 20, F32, dt)], [(128, fast)])
            del fast
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ end to end


def _file(ctx):
    """A file of an 8-byte plain header and the value set of every pair, each converting: its segments and image."""
    import torch

    head = torch.arange(8, dtype=torch.uint8, device="cuda") + 0x40
    segs = ([head.data_ptr()], [8], [0], [0])
    parts = [head]
    for pair in PAIRS:
        src = values(pair[0])
        for a, b in zip(segs, (src.data_ptr(), src.numel() * SIZE[pair[0]], *pair)):
            a.append(b)
        parts.append(image(ctx, pair))
    return head, segs, torch.cat(parts)


def test_hash_of_the_converted_file_at_a_part_length_of_4099(ctx):
    """b200h_hash_cast_segment_parts_device with parts of 4096 + 3 bytes over a file of every value set: the parts in
    converting segments are gathered by stage_ranges_kernel from ranges that start at every residue, mid-element
    included; every part's SHA-256 and MD5 equal hashlib's over the expected image."""
    import torch

    head, segs, want = _file(ctx)
    data = want.cpu().numpy().tobytes()
    part = 4096 + 3
    n = -(-len(data) // part)
    sha = torch.zeros((n, 32), dtype=torch.uint8, device="cuda")
    md5 = torch.zeros((n, 16), dtype=torch.uint8, device="cuda")
    trim = torch.zeros(n, dtype=torch.int64, device="cuda")
    got = ctx.hash_cast_segment_parts_device(*segs, [0, len(segs[0])], part, _lib.SHA256 | _lib.MD5, sha.data_ptr(),
                                             md5.data_ptr(), trim.data_ptr(), _current())
    assert got == n
    torch.cuda.synchronize()
    sha, md5 = sha.cpu().numpy(), md5.cpu().numpy()
    for i in range(n):
        p = data[i * part : (i + 1) * part]
        assert sha[i].tobytes() == hashlib.sha256(p).digest(), i
        assert md5[i].tobytes() == hashlib.md5(p).digest(), i
    torch.cuda.synchronize()


def test_read_back_of_a_converted_safetensors_file_at_odd_offsets(ctx):
    """``DeviceFile.safetensors(sd, dtype={...}).read()`` of a file holding every value set, converted to each other
    type, from odd offsets in reads of odd lengths through a bounce buffer of 1 MiB + 5 bytes: every bounce read is a
    copy_cast_ranges range that starts and ends mid-element.  The bytes equal ``safetensors.torch.save`` of the
    expected images."""
    import torch
    from safetensors.torch import save

    sd, targets, want = {}, {}, {}
    for st, dt in PAIRS:
        name = f"{NAME[st]}_as_{NAME[dt]}"
        sd[name], targets[name] = values(st), _torch(dt)
        want[name] = image(ctx, (st, dt)).view(_torch(dt)).cpu()
    data = save(want)
    f = DeviceFile.safetensors(sd, dtype=targets, ctx=ctx, bounce_bytes=MiB + 5)
    assert f.nbytes == len(data)
    rng = np.random.default_rng(5)
    pos = 1
    while pos < len(data):
        n = int(rng.integers(1, 3 * MiB)) | 1
        f.seek(pos)
        got = f.read(n)
        assert got == data[pos : pos + n], pos
        pos += n + int(rng.integers(0, 4096)) * 2 + 1
    f.seek(0)
    assert f.read() == data
    torch.cuda.synchronize()
