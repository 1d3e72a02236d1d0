"""tools/sanitize_cases.py -- small batches that drive every kernel through its synchronisation-heavy paths, sized
for compute-sanitizer (memcheck / racecheck / synccheck slow kernels down 10-100x):
  lane kernel  more messages than resident lanes (time slicing: states saved/restored, ring re-queue with volatile
               spin-waits and cross-warp atomics), unaligned starts, every tail shape
  chain kernel TMA tile ring + mbarrier hand-offs between the expander / SHA-256 / MD5 warps, 3 long messages
  trim kernels probe + wide scan (atomicMax across CTAs, work counter), blank and half-blank blocks
  dedupe       hash-table insert/resolve with CAS
  streams      absorb/digest on a private CUDA stream
  stage        stage_ranges_kernel: ranges of segmented device files into page-locked host memory: every source
               phase, segments that start at the first and end at the last byte of their allocation (the aligned-hull
               loads), ranges across tiny and empty segments, partial last words
  boxes        load_boxes_kernel: rows at every source phase into a file of exact-size allocations, boxes across
               segment seams, the last box ending at the last byte of the file and of the page-locked source
  cast boxes   load_boxes_kernel converting: every conversion between F32, F16 and BF16, boxes that end at the last
               byte of their exact-size destination allocation and of the page-locked source, every element phase, rows
               that cross destination words, 1-element rows
  cast ranges  stage_ranges_kernel with converting pieces: every conversion, segments that are exact-size allocations,
               ranges at odd image offsets into page-locked host memory and into device memory
  gather       gather_segments_kernel (b200h_hash_segment_parts_device): segments that are exact-size allocations,
               parts that straddle them at every relative phase, and parts hashed in place
  scaled boxes load_scaled_boxes_kernel: FP8 boxes of every format, target and scale type, each scale tensor an
               exact-size allocation with partial last blocks; the last box reads the last element, source byte and
               scale, checked against the integer-exact reference of tests/test_fp8_reference_cpu.py
  fp8 export   fp8_amax_kernel / fp8_finalize_kernel (b200h_fp8_block_scales) and stage_scaled_ranges_kernel: weights
               of every source type that are exact-size allocations at every element phase, partial last blocks, the
               atomicMax of many CTAs into one per-tensor scale, blocks that span two amax tiles beside neighbour
               blocks; ranges at every image offset into page-locked host memory and device memory, checked against
               the integer-exact reference of tests/test_fp8_quant_reference_cpu.py
Digests are compared with hashlib, so a sanitizer run is also a parity run.
  compute-sanitizer --tool memcheck  python tools/sanitize_cases.py
  compute-sanitizer --tool racecheck python tools/sanitize_cases.py"""
import hashlib
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from modal_client_b200 import _lib
from modal_client_b200.synth import synth_array

BOTH = _lib.SHA256 | _lib.MD5
ctx = _lib.Context(0, pinned_bytes=8 << 20, device_bytes=64 << 20)


def check(buf, offs, lens, sha, md5, idx):
    for i in idx:
        m = buf[int(offs[i]) : int(offs[i] + lens[i])].tobytes()
        assert sha is None or sha[i].tobytes() == hashlib.sha256(m).digest(), i
        assert md5 is None or md5[i].tobytes() == hashlib.md5(m).digest(), i


# 1. lane kernel with time slicing: 120 000 short messages (> 94 720 resident lanes) + mixed tails, unaligned
n = int(os.environ.get("SAN_N", 120_000))
rng = np.random.default_rng(1)
lens = rng.integers(0, 200, n).astype(np.uint64)
lens[:64] = np.arange(64) * 3
lens[64:72] = [4096, 5000, 70_000, 64, 128, 55, 56, 119]
offs = (np.concatenate([[0], np.cumsum(lens + np.uint64(1))])[:-1] + np.uint64(3)).astype(np.uint64)
buf = synth_array(1, int(offs[-1] + lens[-1]) + 8)
sha, md5, _ = ctx.hash_batch_host(buf, offs, lens, BOTH)
check(buf, offs, lens, sha, md5, list(range(0, 80)) + list(range(80, n, 997)))
print("lane kernel (time-sliced) ok", flush=True)

# 2. chain kernel: three outliers among small messages, aligned and unaligned, all flag sets
lens = np.array([200_000, 150_001, 131_072 + 55] + [300] * 400, np.uint64)
offs = (np.concatenate([[0], np.cumsum(lens + np.uint64(5))])[:-1] + np.uint64(16)).astype(np.uint64)
buf = synth_array(2, int(offs[-1] + lens[-1]) + 8)
for flags in (BOTH, _lib.SHA256, _lib.MD5):
    sha, md5, _ = ctx.hash_batch_host(buf, offs, lens, flags)
    assert ctx.last_outlier_count == 3, ctx.last_outlier_count
    check(buf, offs, lens, sha, md5, [0, 1, 2, 3, 402])
print("chain kernel ok", flush=True)

# 3. trim: blank / half-blank / dense blocks of 1 MiB, one with a lone byte deep inside
B = 1 << 20
blk = np.zeros(6 * B + 77, np.uint8)
blk[B : B + 300_000] = synth_array(3, 300_000) | 1
blk[3 * B : 4 * B] = synth_array(4, B) | 1
blk[4 * B + 12345] = 9
blk[5 * B + 5 : 5 * B + 70] = 1
sha, _, trimmed, _ = ctx.hash_fixed_parts(blk, B, _lib.SHA256 | _lib.TRIM_ZEROS)
want = [0, 300_000, 0, B, 12346, 70, 0]
assert list(map(int, trimmed)) == want, list(map(int, trimmed))
for i, t in enumerate(want):
    assert sha[i].tobytes() == hashlib.sha256(blk[i * B : i * B + t]).digest()
print("trim kernels ok", flush=True)

# 4. dedupe
keys = np.frombuffer(b"".join(hashlib.sha256(bytes([i % 50])).digest() for i in range(5000)), np.uint8).reshape(-1, 32)
first, nd = ctx.dedupe(keys)
assert nd == 50 and all(int(first[i]) == i % 50 for i in range(5000))
print("dedupe ok", flush=True)

# 5. stream on its own CUDA stream (small buffer so that several absorbs happen)
os.environ["B200H_STREAM_BUF"] = "65536"
c2 = _lib.Context(0, pinned_bytes=1 << 20, device_bytes=4 << 20)
s = c2.stream(BOTH)
data = synth_array(5, 300_007).tobytes()
for i in range(0, len(data), 50_000):
    s.update(data[i : i + 50_000])
assert s.digests() == (hashlib.sha256(data).digest(), hashlib.md5(data).digest())
s.close()
c2.close()
print("stream ok", flush=True)

# 6. stage_ranges_kernel: segments cut out of exact-size allocations at every phase, ranges with odd edges
import torch

pool = [torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda") for n in (70_001, 4097, 33, 1, 300_007)]
segs = [pool[0], pool[1][5:], pool[2][:-3], pool[3], pool[1][:0], pool[4][9:]] + [pool[4][i * 7 : i * 7 + 1 + i % 9] for i in range(64)]
segs += [pool[0][ph : 5000 + 2 * ph] for ph in range(16)]
image = np.concatenate([t.cpu().numpy() for t in segs])
ranges = [(0, 0, image.size), (0, 3, image.size - 8), (0, image.size - 1, 1), (0, 7, 0)]
ranges += [(0, 70_001 - 9 + a, 4097 + 40 + a) for a in range(16)]
offsets, at = [], 128
for _, _, n in ranges:
    offsets.append(at)
    at += -(-n // 128) * 128 + 128
dst = ctx.host_alloc(at)
dst[:] = 0xC3
ctx.copy_ranges_to_host([t.data_ptr() if t.numel() else 0 for t in segs], [t.numel() for t in segs], [0, len(segs)], ranges,
                        dst, offsets, 1)
torch.cuda.synchronize()
clean = np.ones(at, bool)
for (_, off, n), o in zip(ranges, offsets):
    assert np.array_equal(dst[o : o + n], image[off : off + n]), (off, n)
    clean[o : o + n] = False
assert (dst[clean] == 0xC3).all()
ctx.host_free(dst)
print("stage ranges ok", flush=True)

# 7. load_boxes_kernel, the bytes as they are: one file of exact-size allocations, every other box across the seam of
#    two of them; rows at every source phase, with rows that touch, narrow gaps, wide gaps and a box of two tiles; the
#    last box ends at the file's last byte and reads the source's last bytes
src = ctx.host_alloc(1 << 20)
src[:] = synth_array(8, 1 << 20)
shapes = ((1, 9, 0), (3, 7, 1), (37, 5, 2), (9000, 2, 5), (17, 4, 0), (5, 6, 27), (40, 3, 40), (70_001, 1, 0))
boxes, at, d = [], 0, 0
for ph in range(16):
    w, rows, gap = shapes[ph % len(shapes)]
    at = -(-at // 16) * 16 + ph
    boxes.append((0, d, w, rows, at, w + gap))
    at += (rows - 1) * (w + gap) + w
    d += w * rows
f, o, w, rows, _, pitch = boxes[-1]
boxes[-1] = (f, o, w, rows, src.size - (rows - 1) * pitch - w, pitch)
cuts = [0] + [o + w * rows // 2 for _, o, w, rows, _, _ in boxes[1::2]] + [d]
segs = [torch.zeros(b - a, dtype=torch.uint8, device="cuda") for a, b in zip(cuts, cuts[1:])]
ctx.copy_boxes_from_host([t.data_ptr() for t in segs], [t.numel() for t in segs], [0, len(segs)], boxes, src, 1)
torch.cuda.synchronize()
want = np.concatenate([src[a + r * pitch : a + r * pitch + w] for _, _, w, rows, a, pitch in boxes for r in range(rows)])
assert np.array_equal(torch.cat(segs).cpu().numpy(), want)
ctx.host_free(src)
print("boxes ok", flush=True)

# 8. load_boxes_kernel converting: each box fills an exact-size allocation; the last box reads the source's last bytes
names = {_lib.DT_F32: torch.float32, _lib.DT_F16: torch.float16, _lib.DT_BF16: torch.bfloat16}
src = ctx.host_alloc(1 << 20)
src[:] = synth_array(7, 1 << 20)
boxes, outs, at = [], [], 0
for st, dt in [(a, b) for a in names for b in names if a != b]:
    ss, ds = names[st].itemsize, names[dt].itemsize
    for w, rows, gap, ph in ((1, 9, 0, 0), (3, 7, 1, 1), (37, 5, 2, 2), (9000, 2, 5, 3), (8, 1, 0, 0)):
        at = -(-at // 16) * 16 + ph * ss
        outs.append(torch.empty(w * rows * ds, dtype=torch.uint8, device="cuda"))
        boxes.append((len(outs) - 1, 0, w * ss, rows, at, (w + gap) * ss, st, dt))
        at += ((rows - 1) * (w + gap) + w) * ss
boxes[-1] = boxes[-1][:4] + (src.size - 8 * names[boxes[-1][6]].itemsize,) + boxes[-1][5:]
ctx.copy_cast_boxes_from_host([t.data_ptr() for t in outs], [t.numel() for t in outs], list(range(len(outs) + 1)),
                              boxes, src)
torch.cuda.synchronize()
for (f, _, w, rows, a, pitch, st, dt), t in zip(boxes, outs):
    rows_ = np.concatenate([src[a + r * pitch : a + r * pitch + w] for r in range(rows)])
    want = torch.from_numpy(rows_).cuda().view(names[st]).to(names[dt]).view(torch.uint8)
    assert torch.equal(t, want), (st, dt, w, rows)
ctx.host_free(src)
print("cast boxes ok", flush=True)

# 9. stage_ranges_kernel with converting pieces: every conversion, each segment an exact-size allocation (its first
#    and last bytes are those of the allocation), plain bytes between them, ranges at odd image offsets into host and
#    device memory
segs, casts, at = [], [], 0
for st, dt in [(a, b) for a in names for b in names if a != b] + [(0, 0)]:
    ss, ds = (names[st].itemsize, names[dt].itemsize) if st else (1, 1)
    if at % ds:
        segs.append(torch.randint(0, 256, (ds - at % ds,), dtype=torch.uint8, device="cuda"))
        casts.append((0, 0))
        at += ds - at % ds
    n = 4099 * ss if st else 37
    segs.append(torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda"))
    casts.append((st, dt))
    at += n // ss * ds
image = torch.cat([t.view(names[st]).to(names[dt]).view(torch.uint8) if st else t
                   for t, (st, dt) in zip(segs, casts)]).cpu().numpy()
ranges = [(0, 0, image.size), (0, 1, image.size - 2), (0, image.size - 3, 3), (0, 8199, 5000)]
offsets, at = [], 128
for _, _, n in ranges:
    offsets.append(at)
    at += -(-n // 128) * 128 + 128
args = ([t.data_ptr() for t in segs], [t.numel() for t in segs], [c[0] for c in casts], [c[1] for c in casts],
        [0, len(segs)], ranges)
host = ctx.host_alloc(at)
dev = torch.empty(at, dtype=torch.uint8, device="cuda")
for dst in (host, dev):
    ctx.copy_cast_ranges(*args, dst, offsets, 1)  # after the fills on torch's (legacy) default stream
    torch.cuda.synchronize()
    got = dst if dst is host else dst.cpu().numpy()
    for (_, off, n), o in zip(ranges, offsets):
        assert np.array_equal(got[o : o + n], image[off : off + n]), (off, n)
ctx.host_free(host)
print("cast ranges ok", flush=True)

# 10. gather_segments_kernel (b200h_hash_segment_parts_device): each segment an exact-size allocation, parts that
#     straddle segments at every relative phase of source and wave slot, and parts hashed in place in the long segments
sizes = [1, 15, 16, 17, 0, 33, 255, 4097, 70_001, 3, 5000, 64, 9] + [1 + i * 37 % 97 for i in range(48)]
files = [[torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda") for n in f] for f in (sizes, sizes[::-1])]
segs = [t for f in files for t in f]
images = [b"".join(t.cpu().numpy().tobytes() for t in f) for f in files]
for part_len in (64, 1000, 4096):
    nrows = sum(-(-len(img) // part_len) for img in images)
    sha = torch.empty((nrows, 32), dtype=torch.uint8, device="cuda")
    md5 = torch.empty((nrows, 16), dtype=torch.uint8, device="cuda")
    assert ctx.hash_segment_parts_device([t.data_ptr() if t.numel() else 0 for t in segs], [t.numel() for t in segs],
                                         [0, len(sizes), len(segs)], part_len, BOTH, sha.data_ptr(),
                                         md5.data_ptr()) == nrows
    torch.cuda.synchronize()
    sha, md5, row = sha.cpu().numpy(), md5.cpu().numpy(), 0
    for img in images:
        for o in range(0, len(img), part_len):
            m = img[o : o + part_len]
            assert sha[row].tobytes() == hashlib.sha256(m).digest(), (part_len, row)
            assert md5[row].tobytes() == hashlib.md5(m).digest(), (part_len, row)
            row += 1
print("segment parts gather ok", flush=True)

# 11. load_scaled_boxes_kernel: FP8 boxes dequantized with block scales, for every format x target x scale type; each
#     scale tensor an exact-size allocation of ceil(R / br) * ceil(C / bc) elements whose last block is partial in both
#     dimensions, each destination an exact-size allocation; the boxes take the fast path, the element loop and rows
#     across tensor-row edges; the last box reads its tensor's last element, the source's last byte and the last scale
from tests.test_cast_reference_cpu import is_nan_bits
from tests.test_fp8_reference_cpu import NAN, reference_dequant

names[_lib.DT_F8E4M3], names[_lib.DT_F8E5M2] = torch.float8_e4m3fn, torch.float8_e5m2
src = ctx.host_alloc(1 << 20)
src[:] = synth_array(11, 1 << 20)
g = torch.Generator().manual_seed(11)
combos = [(fc, tc, sc) for fc in (_lib.DT_F8E4M3, _lib.DT_F8E5M2) for tc in (_lib.DT_BF16, _lib.DT_F16, _lib.DT_F32)
          for sc in (_lib.DT_F32, _lib.DT_F16, _lib.DT_BF16)]
boxes, outs, meta, at = [], [], [], 0
for k, (fc, tc, sc) in enumerate(combos):
    br, bc = 8, 5 + k % 4
    R, C = 37 + 2 * k, bc * (9 + k) + 1 + k % 3  # partial last blocks: R % br and C % bc are not 0
    assert R % br and C % bc
    nscales = -(-R // br) * -(-C // bc)
    scales = ((torch.rand(nscales, generator=g) * 4 - 2) * 2.0 ** torch.randint(-10, 10, (nscales,), generator=g)).to(
        names[sc]).cuda()
    first, rows, width, pitch = [(0, 1, R * C, R * C), (C + 1, R - 2, C - 3, C), (5, R - 1, 3, C + 1),
                                 (C - 7, 4, 20, 2 * C)][k % 4]
    if k == len(combos) - 1:  # the last box ends at the tensor's last element, which is the source's last byte
        first, rows, width, pitch = R * C - 1 - 2 * (C + 2) - 30 + 1, 3, 30, C + 2
        at = src.size - R * C
    at = -(-at // 16) * 16 + k % 16 if k < len(combos) - 1 else at
    outs.append(torch.empty(rows * width * names[tc].itemsize, dtype=torch.uint8, device="cuda"))
    boxes.append((len(outs) - 1, 0, width, rows, at + first, pitch, fc, tc, scales.data_ptr(), sc, nscales, first, R,
                  C, br, bc))
    meta.append((at, scales, R, C, br, bc))
    at += R * C
assert boxes[-1][4] + (boxes[-1][3] - 1) * boxes[-1][5] + boxes[-1][2] == src.size
ctx.copy_scaled_boxes_from_host([t.data_ptr() for t in outs], [t.numel() for t in outs], list(range(len(outs) + 1)),
                                boxes, src)
torch.cuda.synchronize()
for (_, _, width, rows, s_at, pitch, fc, tc, _, sc, _, first, R, C, br, bc), (at, scales, *_), t in zip(boxes, meta,
                                                                                                      outs):
    e = first + (torch.arange(rows)[:, None] * pitch + torch.arange(width)[None, :]).reshape(-1)
    w_bits = torch.from_numpy(src[at : at + R * C].copy()).to(torch.int64)[e]
    s_bits = scales.cpu().view(torch.int32 if sc == _lib.DT_F32 else torch.int16).to(torch.int64)
    ref = reference_dequant(w_bits, names[fc], s_bits[e // C // br * -(-C // bc) + e % C // bc], names[sc], names[tc])
    got = t.cpu().view(torch.int32 if tc == _lib.DT_F32 else torch.int16).to(torch.int64) & \
        ((1 << (8 * names[tc].itemsize)) - 1)
    nan = ref == NAN
    assert torch.equal(got[~nan], ref[~nan]) and bool(is_nan_bits(got[nan], names[tc]).all()), (fc, tc, sc, R, C)
ctx.host_free(src)
print("scaled boxes ok", flush=True)

# 12. FP8 export: the scale call and the quantizing copies over exact-size allocations, one block form (3, 4097) whose
#     blocks span two amax tiles and have neighbours in both directions; checked against the integer-exact reference
from safetensors.torch import save as st_save  # noqa: E402

from modal_client_b200 import DeviceFile, stage_ranges  # noqa: E402
from tests.test_fp8_quant_reference_cpu import reference_block_scales, reference_multiplier, reference_quant  # noqa: E402

sd, fp8 = {}, []
for k, (dt, shape) in enumerate([(torch.float32, (37, 29)), (torch.float16, (130, 141)), (torch.bfloat16, (5, 1001)),
                                 (torch.bfloat16, (1 << 10, 1 << 9)), (torch.float32, (8, 8300))]):
    sd[f"w{k}"] = torch.randn(*shape, generator=g).to(dt).cuda()  # its own allocation, sized exactly
    fp8.append(f"w{k}")
sd["norm"] = torch.ones(29, dtype=torch.float32).cuda()
for block in ((128, 128), (7, 5), (None, None), (3, 4097)):
    f = DeviceFile.safetensors(sd, fp8=fp8, scale_block=block, ctx=ctx)
    ref = {}
    for n, t in sd.items():
        if n not in fp8:
            ref[n] = t.cpu()
            continue
        R, C = t.shape
        bR, bC = min(block[0] or R, R), min(block[1] or C, C)
        bits = t.cpu().view(torch.int32 if t.dtype == torch.float32 else torch.int16).to(torch.int64).reshape(-1)
        bits &= (1 << (8 * t.element_size())) - 1
        a, s = reference_block_scales(bits, t.dtype, R, C, (bR, bC))
        e = torch.arange(R * C)
        q = reference_quant(bits, t.dtype, reference_multiplier(a.reshape(-1))[e // C // bR * a.shape[1] + e % C // bC])
        ref[n] = q.to(torch.uint8).view(torch.float8_e4m3fn).view(R, C)
        ref[n + "_scale_inv"] = s.to(torch.int32).view(torch.float32)
    want = np.frombuffer(st_save(ref), np.uint8)
    assert f.nbytes == want.size
    ranges = [(0, 0, want.size)] + [(0, o, min(777, want.size - o)) for o in range(1, want.size, want.size // 37)]
    offsets = [sum(-(-n // 16) * 16 for _, _, n in ranges[:i]) for i in range(len(ranges))]
    total = offsets[-1] + -(-ranges[-1][2] // 16) * 16
    pinned = ctx.host_alloc(total)
    device = torch.empty(total, dtype=torch.uint8, device="cuda")
    for dst in (pinned, device):
        stage_ranges([f], ranges, dst, offsets, ctx=ctx).wait()
        got = dst if isinstance(dst, np.ndarray) else dst.cpu().numpy()
        for (_, o, n), at in zip(ranges, offsets):
            assert np.array_equal(got[at : at + n], want[o : o + n]), (block, o, n)
    ctx.host_free(pinned)
print("fp8 export ok", flush=True)
ctx.close()
print("ALL OK")
