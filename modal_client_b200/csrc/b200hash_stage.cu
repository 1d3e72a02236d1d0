// b200hash_stage.cu -- copy byte ranges of segmented device files to one destination buffer with full-width stores:
// the blocks of a checkpoint in HBM that a volume server reports missing, on their way to page-locked host memory;
// and back (load_ranges_kernel, below): downloaded blocks from page-locked host memory into the tensors of a file.
//
//   stage_ranges_kernel  persistent CTAs take destination tiles (kStageTileBytes of one range's destination, the last
//                        tile of a range may be shorter); every thread produces whole, 16-byte aligned destination
//                        words.  The work is organised by DESTINATION because the destination is on the far side of
//                        PCIe, where a store narrower than 16 bytes costs as much as a full one: source and destination
//                        phases differ almost always (safetensors data starts at 8 + header length, a torch.save
//                        storage where the zip puts it, and a block made of several tensors changes phase at every
//                        tensor edge), so a copy at the widest access on which both sides agree, as
//                        gather_segments_kernel does between HBM buffers, would degrade to byte stores here.  The
//                        kernel is at the end of the file: its pieces may also convert elements, with the conversion
//                        helpers of load_boxes_kernel.
//
// A range is cut by the host into pieces (range intersected with one segment, never empty), listed in destination
// order; a tile names the slice of the piece list it draws from.
//   * a tile that lies in one piece that converts nothing is copied with no lookups (stage_one_piece);
//   * a destination word that lies inside one such piece is built from the two aligned 16-byte source words around it
//     and a byte shift by (source address & 15): one load when the phases agree, two otherwise;
//   * a word that crosses pieces is assembled byte by byte and still stored as one word;
//   * only the bytes behind a range's last whole word are stored singly (the destination beyond the range is not the
//     kernel's to write).
// Loads never leave the 16-byte aligned hull of a piece: the aligned words that hold a piece's first and last byte.
// Those words lie in the same allocation granule as the bytes themselves (device allocations are at least 256-byte
// aligned and sized in multiples of that), which the lane kernel's misaligned-start reads rely on as well.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200hash.h"
#include "b200hash_kernels.cuh"

namespace b200h {
namespace {

constexpr int kStageThreads = 256;
constexpr int kStageCtasPerSm = 4;

// bytes [sh, sh + 16) of the 32 bytes lo || hi (sh < 16)
__device__ __forceinline__ uint4 shift_bytes(uint4 lo, uint4 hi, uint32_t sh) {
    const uint32_t k = sh >> 2, b = (sh & 3u) * 8u;
    const uint32_t v0 = k == 0 ? lo.x : k == 1 ? lo.y : k == 2 ? lo.z : lo.w;
    const uint32_t v1 = k == 0 ? lo.y : k == 1 ? lo.z : k == 2 ? lo.w : hi.x;
    const uint32_t v2 = k == 0 ? lo.z : k == 1 ? lo.w : k == 2 ? hi.x : hi.y;
    const uint32_t v3 = k == 0 ? lo.w : k == 1 ? hi.x : k == 2 ? hi.y : hi.z;
    const uint32_t v4 = k == 0 ? hi.x : k == 1 ? hi.y : k == 2 ? hi.z : hi.w;
    return make_uint4(__funnelshift_r(v0, v1, b), __funnelshift_r(v1, v2, b), __funnelshift_r(v2, v3, b),
                      __funnelshift_r(v3, v4, b));
}

// the 16 bytes at src (all of them inside one piece), whatever its alignment
__device__ __forceinline__ uint4 load_word(const uint8_t* src) {
    const uint32_t sh = (uint32_t)((uintptr_t)src & 15u);
    const uint4* a = reinterpret_cast<const uint4*>(src - sh);
    const uint4 lo = __ldg(a);
    return sh ? shift_bytes(lo, __ldg(a + 1), sh) : lo;
}

// the piece of pc[lo .. n) that holds destination offset d (the pieces of a range tile its destination without gaps)
__device__ __forceinline__ uint32_t find_piece(const CastPiece* __restrict__ pc, uint32_t lo, uint32_t n, uint64_t d) {
    uint32_t hi = n - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (pc[mid].r.host <= d) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// A tile whose bytes all come, as they are, from one piece at `src`: one phase, no lookups.
__device__ __forceinline__ void stage_one_piece(const uint8_t* src, uint8_t* out, uint32_t words, uint32_t tail) {
    const uint32_t sh = (uint32_t)((uintptr_t)src & 15u);
    const uint4* a = reinterpret_cast<const uint4*>(src - sh);
    uint4* o = reinterpret_cast<uint4*>(out);
    uint32_t w = threadIdx.x;
    if (sh == 0) {
        for (; w + 3 * kStageThreads < words; w += 4 * kStageThreads) {
            uint4 v[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) v[i] = __ldg(a + w + i * kStageThreads);
#pragma unroll
            for (int i = 0; i < 4; ++i) o[w + i * kStageThreads] = v[i];
        }
        for (; w < words; w += kStageThreads) o[w] = __ldg(a + w);
    } else {
        for (; w + 3 * kStageThreads < words; w += 4 * kStageThreads) {
            uint4 lo[4], hi[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                lo[i] = __ldg(a + w + i * kStageThreads);
                hi[i] = __ldg(a + w + i * kStageThreads + 1);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) o[w + i * kStageThreads] = shift_bytes(lo[i], hi[i], sh);
        }
        for (; w < words; w += kStageThreads) o[w] = shift_bytes(__ldg(a + w), __ldg(a + w + 1), sh);
    }
    if (threadIdx.x < tail) out[(uint64_t)words * 16 + threadIdx.x] = src[(uint64_t)words * 16 + threadIdx.x];
}

// ---- the inverse direction: page-locked host memory -> segmented device files
//
//   load_ranges_kernel   persistent CTAs whose warps take source tiles (kStageTileBytes of one range's source, the
//                        last tile of a range may be shorter).  The work is organised by SOURCE because the source is
//                        now on the far side of PCIe: every source byte crosses it exactly once, as part of one aligned
//                        16-byte load issued by one lane (a warp's 32 lanes read 512 consecutive bytes per load).  A
//                        repeated read of mapped host memory is never relied on to hit a cache.
//
// Lane k of a chunk holds source word w = (the tile's first word) + 32 * chunk + k and builds, for every piece, the
// aligned destination word whose last source byte lies in word w: with r = (piece device address - piece source
// offset) & 15, that word takes the 16 source bytes [16w - r, 16w + 16 - r), i.e. bytes 16 - r .. 15 of word w - 1
// (from lane k - 1 through __shfl_up_sync, or carried over from the previous chunk's lane 31) and bytes 0 .. 15 - r of
// word w, joined with shift_bytes.  Every source byte belongs to exactly one such word per piece.  The word is stored
// whole when all 16 bytes lie inside the piece; only at a piece's edges, and at a tile's first word, whose word w - 1
// was read by the warp that has the tile before (it stores those bytes as the extra lane one past its last word), is
// it stored in narrower parts.  Device bytes outside the pieces are never written.  Loads stay inside the 16-byte
// aligned hull of the tile's source bytes, which lies in the same page-locked allocation as the bytes themselves.

constexpr int kLoadChunks = 4;  // 32-word chunks in flight per warp

// bytes [lo, hi) of v (0 <= lo < hi <= 16) to the 16-byte aligned `out`
__device__ __forceinline__ void store_bytes(uint8_t* out, uint4 v, uint32_t lo, uint32_t hi) {
    if (lo == 0 && hi == 16) {
        *reinterpret_cast<uint4*>(out) = v;
        return;
    }
    for (uint32_t j = lo; j < hi; ++j) {
        const uint32_t k = j >> 2, x = k == 0 ? v.x : k == 1 ? v.y : k == 2 ? v.z : v.w;
        out[j] = (uint8_t)(x >> (8 * (j & 3)));
    }
}

__device__ __forceinline__ uint4 shfl_up_word(uint4 v) {
    return make_uint4(__shfl_up_sync(0xffffffffu, v.x, 1), __shfl_up_sync(0xffffffffu, v.y, 1),
                      __shfl_up_sync(0xffffffffu, v.z, 1), __shfl_up_sync(0xffffffffu, v.w, 1));
}

__device__ __forceinline__ uint4 shfl_last_word(uint4 v) {
    return make_uint4(__shfl_sync(0xffffffffu, v.x, 31), __shfl_sync(0xffffffffu, v.y, 31),
                      __shfl_sync(0xffffffffu, v.z, 31), __shfl_sync(0xffffffffu, v.w, 31));
}

// The destination words of source word w (see above) for pieces pc[p .. n).  Source offsets are relative to the
// tile's first byte `ts` (a tile is at most 64 KiB): base = 16 * (w - the tile's first word); only source bytes in
// [lo, hi), the words this lane holds, are stored.  p is the lane's cursor: pieces that end before anything word w
// could take are skipped.
__device__ __forceinline__ void load_word_out(const RangePiece* __restrict__ pc, uint32_t& p, uint32_t n, uint64_t ts,
                                              int32_t base, uint4 prev, uint4 cur, int32_t lo, int32_t hi) {
    const uint64_t at = ts + (uint32_t)base;
    while (p < n && pc[p].host + pc[p].len + 15 <= at) ++p;
    for (uint32_t q = p; q < n && pc[q].host < at + 16; ++q) {
        const RangePiece piece = pc[q];
        const uint32_t r = (uint32_t)(piece.dev - piece.host) & 15u;
        const int32_t s0 = base - (int32_t)r;
        // the piece clipped to [base - 16, base + 16): it may begin in an earlier tile or end in a later one
        const int32_t from = piece.host + 16 <= at ? base - 16 : (int32_t)(piece.host - ts);
        const int32_t to = piece.host + piece.len >= at + 16 ? base + 16 : (int32_t)(piece.host + piece.len - ts);
        const int32_t a = max(max(s0, from), lo), b = min(min(s0 + 16, to), hi);
        if (a >= b) continue;
        store_bytes(reinterpret_cast<uint8_t*>(piece.dev + (ts - piece.host) + (uint64_t)(int64_t)s0),
                    r ? shift_bytes(prev, cur, 16 - r) : cur, (uint32_t)(a - s0), (uint32_t)(b - s0));
    }
}

__global__ void __launch_bounds__(kStageThreads, kStageCtasPerSm)
    load_ranges_kernel(const RangeTile* __restrict__ tiles, uint64_t ntiles, const RangePiece* __restrict__ pieces,
                       const uint8_t* __restrict__ src) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint4* words = reinterpret_cast<const uint4*>(src);
    const uint4 zero = make_uint4(0, 0, 0, 0);
    const uint64_t nwarps = (uint64_t)gridDim.x * (kStageThreads / 32);
    for (uint64_t t = (uint64_t)blockIdx.x * (kStageThreads / 32) + (threadIdx.x >> 5); t < ntiles; t += nwarps) {
        const RangeTile tile = tiles[t];
        const RangePiece* __restrict__ pc = pieces + tile.first_piece;
        const uint4* tw = words + (tile.host >> 4);
        const int32_t nw = (int32_t)((tile.len + 15) >> 4);
        uint32_t p = 0;
        uint4 carry = zero;
        // the tile's words [0, nw) are loaded; lane nw loads nothing and stores what word nw - 1 gives the destination
        // words that begin there and end in the next tile's first word
        for (int32_t c = 0; c <= nw; c += 32 * kLoadChunks) {
            uint4 v[kLoadChunks];
#pragma unroll
            for (int i = 0; i < kLoadChunks; ++i) {
                const int32_t w = c + i * 32 + (int32_t)lane;
                v[i] = w < nw ? __ldg(tw + w) : zero;
            }
#pragma unroll
            for (int i = 0; i < kLoadChunks; ++i) {
                const int32_t w = c + i * 32 + (int32_t)lane;
                uint4 prev = shfl_up_word(v[i]);
                if (lane == 0) prev = carry;
                carry = shfl_last_word(v[i]);
                if (w <= nw)
                    load_word_out(pc, p, tile.npieces, tile.host, w * 16, prev, v[i], w > 0 ? w * 16 - 16 : 0,
                                  w < nw ? w * 16 + 16 : w * 16);
            }
        }
    }
}

// ---- boxes: rows of a page-locked host buffer, `pitch` bytes apart, packed into segmented device files
//
//   load_boxes_kernel    persistent CTAs whose warps take tiles of a box's virtual source words (CastTile), tile t on
//                        CTA t % gridDim.x so that a call with few tiles still spreads over every SM.  Lane k of a
//                        chunk loads virtual word 128 * chunk + 32 * i + k (i < kLoadChunks) with one aligned 16-byte
//                        load, so every source byte that lands crosses PCIe once and no load leaves its row's hull (the
//                        bytes between rows are read only inside the hull words, or, when rows are less than 16 bytes
//                        apart, because every such byte lies in one).  The loads run two chunks ahead in registers,
//                        so they are in flight while the warp stores the current chunk; a chunk goes to the warp's
//                        ring in shared memory (two chunks) when its turn comes.
//                        The warp stores every destination word whose last byte's source has arrived: an aligned
//                        device word of one piece, built from two ring words and shift_bytes when its 16 bytes are one
//                        run of one row, byte by byte from the ring otherwise (a word across rows; narrow rows).  A
//                        destination word's bytes come from at most 33 consecutive virtual words, so the previous
//                        chunk is still in the ring.  Words are stored whole except at the run's ends, at piece edges
//                        and at the seam of two tiles, where each tile stores the bytes its words hold.

constexpr uint32_t kBoxChunk = 32 * kLoadChunks;  // virtual words loaded per warp and step
constexpr uint32_t kBoxRing = 2 * kBoxChunk;
// 64-bit row arithmetic needs more than the 64 registers of 4 CTAs per SM; 16 warps of 2 KiB loads each per SM still
// keep far more in flight than PCIe's bandwidth-delay product
constexpr int kBoxCtasPerSm = 2;

// The virtual word of source byte s, which lies in row r of the box.
__device__ __forceinline__ uint64_t box_virtual(const BoxTile& b, uint64_t r, uint64_t s) {
    return b.hull ? r * b.hull + (s >> 4) - ((b.src + r * b.pitch) >> 4) : (s >> 4) - (b.src >> 4);
}

// Lane `lane`'s words of the chunk that starts at virtual word b.v0 + c (zero where a row's last slot is empty).
__device__ __forceinline__ void box_load_chunk(const BoxTile& b, const uint4* words, uint32_t c, uint32_t lane,
                                               uint4 (&v)[kLoadChunks]) {
#pragma unroll
    for (int i = 0; i < kLoadChunks; ++i) {
        const uint32_t j = c + i * 32 + lane;
        v[i] = make_uint4(0, 0, 0, 0);
        if (j < b.nv) {
            const uint64_t g = b.v0 + j;
            if (b.hull) {
                const uint64_t r = g / b.hull, s = b.src + r * b.pitch, x = (s >> 4) + g % b.hull;
                if (x <= (s + b.width - 1) >> 4) v[i] = __ldg(words + x);
            } else {
                v[i] = __ldg(words + (b.src >> 4) + g);
            }
        }
    }
}

// Destination words of piece `pc` whose bytes (clipped to the piece and to [b.dlo, b.dhi)) end in [from, upto).
// Word bounds are compared as device addresses: a piece's first word may begin before its packed offset 0.
__device__ __forceinline__ void box_words_out(const BoxTile& b, const RangePiece pc, const uint4* ring, uint64_t from,
                                              uint64_t upto, uint32_t lane) {
    const uint64_t qlo = max(pc.host, b.dlo), qhi = min(pc.host + pc.len, b.dhi);
    const uint64_t lo = max(from, qlo), hi = min(upto, qhi);
    if (lo >= hi) return;
    const uint64_t base = pc.dev - pc.host;  // device address of packed byte d: base + d (mod 2^64)
    const uint64_t qa = base + qlo, qe = base + qhi, ha = base + hi;
    // a word whose bytes go on past `hi` waits for the next step
    const uint64_t w1 = hi < qhi ? ha >> 4 : ((ha - 1) >> 4) + 1;
    for (uint64_t w = ((base + lo) >> 4) + lane; w < w1; w += 32) {
        const uint64_t ws = w * 16, aa = max(ws, qa), ea = min(ws + 16, qe);
        const uint32_t jlo = (uint32_t)(aa - ws), jhi = (uint32_t)(ea - ws);
        const uint64_t a = aa - base;
        uint64_t r = a / b.width, c = a % b.width;
        uint4 v;
        if (jhi - jlo == 16 && c + 16 <= b.width) {
            const uint64_t s = b.src + r * b.pitch + c;
            const uint32_t slot = (uint32_t)(box_virtual(b, r, s) - b.v0), sh = (uint32_t)s & 15u;
            const uint4 w0 = ring[slot % kBoxRing];
            v = sh ? shift_bytes(w0, ring[(slot + 1) % kBoxRing], sh) : w0;
        } else {
            uint64_t x[2] = {0, 0};
#pragma unroll 1
            for (uint32_t j = jlo; j < jhi; ++j) {
                const uint64_t s = b.src + r * b.pitch + c;
                const uint8_t* word =
                    reinterpret_cast<const uint8_t*>(ring + (uint32_t)(box_virtual(b, r, s) - b.v0) % kBoxRing);
                const uint64_t byte = (uint64_t)word[s & 15u] << (8 * (j & 7));
                if (j < 8) x[0] |= byte;
                else x[1] |= byte;
                if (++c == b.width) c = 0, ++r;
            }
            v = make_uint4((uint32_t)x[0], (uint32_t)(x[0] >> 32), (uint32_t)x[1], (uint32_t)(x[1] >> 32));
        }
        store_bytes(reinterpret_cast<uint8_t*>(ws), v, jlo, jhi);
    }
}

// One warp's pass over tile b: the loads run two chunks ahead in registers, a chunk goes to the warp's ring when its
// turn comes, and out(from, upto) stores the packed destination bytes [from, upto) (in source bytes) whose source has
// arrived.  The ring's other half still holds the chunk before, which a destination word may need.
template <class Out>
__device__ __forceinline__ void box_tile_steps(const BoxTile& b, const uint4* words, uint4* ring, uint32_t lane,
                                               Out&& out) {
    uint64_t from = b.dlo;
    uint4 v[kLoadChunks], u[kLoadChunks];  // chunks c and c + 1, loaded
    box_load_chunk(b, words, 0, lane, v);
    box_load_chunk(b, words, kBoxChunk, lane, u);
    for (uint32_t c = 0; c < b.nv; c += kBoxChunk) {
        // the ring's other half holds chunk c - 1, which this step's words may still need
#pragma unroll
        for (int i = 0; i < kLoadChunks; ++i) {
            ring[(c + i * 32 + lane) % kBoxRing] = v[i];
            v[i] = u[i];
        }
        __syncwarp();
        box_load_chunk(b, words, c + 2 * kBoxChunk, lane, u);
        const uint64_t upto = c + kBoxChunk >= b.nv ? b.dhi : box_dest_at(b, b.v0 + c + kBoxChunk);
        out(from, upto);
        __syncwarp();
        from = upto;
    }
}

// ---- boxes whose elements change type on the way (F32, F16, BF16; b200h_copy_cast_boxes_from_host)
//
// The same tiles, loads and ring, with a destination word built from elements instead of bytes.  Every element of a
// box lies whole in one aligned source word (rows start at a multiple of the element size), and the box's destination
// is one piece at a multiple of the destination element size, so every destination word holds whole elements.  A word
// of 16 / ds elements takes 16 / ds * ss source bytes: 32 when narrowing F32 (two or three ring words), 16 between F16
// and BF16 (one or two), 8 when widening (one or two).  When they are one run of one row they come from the ring with
// shift_bytes; otherwise (a word across rows, a box's ends) element by element.  The conversion then takes pairs of
// elements with the paired sm_90 intrinsics.

constexpr uint32_t kDtF32 = B200H_DT_F32, kDtF16 = B200H_DT_F16;

__device__ __forceinline__ uint32_t dt_bytes(uint32_t t) { return t == kDtF32 ? 4u : 2u; }

// two 16-bit elements (F16 or BF16), widened exactly
__device__ __forceinline__ float2 widen_pair(uint32_t x, uint32_t t) {
    if (t == kDtF16) {
        __half2 h;
        memcpy(&h, &x, 4);
        return __half22float2(h);
    }
    __nv_bfloat162 h;
    memcpy(&h, &x, 4);
    return __bfloat1622float2(h);
}

// two floats rounded to nearest even, as F16 or BF16
__device__ __forceinline__ uint32_t narrow_pair(float a, float b, uint32_t t) {
    uint32_t x;
    if (t == kDtF16) {
        const __half2 h = __float22half2_rn(make_float2(a, b));
        memcpy(&x, &h, 4);
    } else {
        const __nv_bfloat162 h = __float22bfloat162_rn(make_float2(a, b));
        memcpy(&x, &h, 4);
    }
    return x;
}

// The destination word of the source bytes lo || hi (32 of them from F32, 16 between F16 and BF16, 8 widening).
__device__ __forceinline__ uint4 cast_word(uint4 lo, uint4 hi, uint32_t st, uint32_t dt) {
    if (st == kDtF32)
        return make_uint4(narrow_pair(__uint_as_float(lo.x), __uint_as_float(lo.y), dt),
                          narrow_pair(__uint_as_float(lo.z), __uint_as_float(lo.w), dt),
                          narrow_pair(__uint_as_float(hi.x), __uint_as_float(hi.y), dt),
                          narrow_pair(__uint_as_float(hi.z), __uint_as_float(hi.w), dt));
    if (dt == kDtF32) {
        const float2 a = widen_pair(lo.x, st), b = widen_pair(lo.y, st);
        return make_uint4(__float_as_uint(a.x), __float_as_uint(a.y), __float_as_uint(b.x), __float_as_uint(b.y));
    }
    const float2 a = widen_pair(lo.x, st), b = widen_pair(lo.y, st), c = widen_pair(lo.z, st), d = widen_pair(lo.w, st);
    return make_uint4(narrow_pair(a.x, a.y, dt), narrow_pair(b.x, b.y, dt), narrow_pair(c.x, c.y, dt),
                      narrow_pair(d.x, d.y, dt));
}

// Destination words of the box (one piece at device address `dev`) whose elements have packed source bytes in
// [from, upto) (clipped to [b.dlo, b.dhi)) and whose last element's source lies before `upto`.
__device__ __forceinline__ void cast_words_out(const BoxTile& b, uint32_t st, uint32_t dt, uint64_t dev,
                                               const uint4* ring, uint64_t from, uint64_t upto, uint32_t lane) {
    const uint32_t ss = dt_bytes(st), ds = dt_bytes(dt);
    const uint64_t qhi = b.dhi / ss * ds, lo = from / ss * ds, hi = upto / ss * ds;
    if (lo >= hi) return;
    const uint64_t qa = dev + b.dlo / ss * ds, qe = dev + qhi, ha = dev + hi, welems = b.width / ss;
    // a word whose elements go on past `hi` waits for the next step
    const uint64_t w1 = hi < qhi ? ha >> 4 : ((ha - 1) >> 4) + 1;
    for (uint64_t w = ((dev + lo) >> 4) + lane; w < w1; w += 32) {
        const uint64_t ws = w * 16, aa = max(ws, qa), ea = min(ws + 16, qe);
        const uint32_t jlo = (uint32_t)(aa - ws), jhi = (uint32_t)(ea - ws);
        const uint64_t e = (aa - dev) / ds;  // the word's first element, counted in the box's packed run
        uint64_t r = e / welems, c = e % welems;
        uint4 s0, s1 = make_uint4(0, 0, 0, 0);
        if (jhi - jlo == 16 && c + 16 / ds <= welems) {
            const uint64_t s = b.src + r * b.pitch + c * ss;
            const uint32_t slot = (uint32_t)(box_virtual(b, r, s) - b.v0), sh = (uint32_t)s & 15u;
            const uint4 w0 = ring[slot % kBoxRing];
            if (ss * 16 / ds == 32) {
                const uint4 n1 = ring[(slot + 1) % kBoxRing];
                s0 = sh ? shift_bytes(w0, n1, sh) : w0;
                s1 = sh ? shift_bytes(n1, ring[(slot + 2) % kBoxRing], sh) : n1;
            } else if (ss == ds) {
                s0 = sh ? shift_bytes(w0, ring[(slot + 1) % kBoxRing], sh) : w0;
            } else {
                s0 = sh > 8 ? shift_bytes(w0, ring[(slot + 1) % kBoxRing], sh) : shift_bytes(w0, w0, sh);
            }
        } else {
            uint64_t x[4] = {0, 0, 0, 0};  // the source bytes, element k at byte k * ss
#pragma unroll 1
            for (uint32_t j = jlo; j < jhi; j += ds) {
                const uint64_t s = b.src + r * b.pitch + c * ss;
                const uint8_t* word =
                    reinterpret_cast<const uint8_t*>(ring + (uint32_t)(box_virtual(b, r, s) - b.v0) % kBoxRing);
                const uint32_t p = j / ds * ss;
                const uint64_t val = (ss == 4 ? (uint64_t)*reinterpret_cast<const uint32_t*>(word + (s & 15u))
                                              : (uint64_t)*reinterpret_cast<const uint16_t*>(word + (s & 15u)))
                                     << (8 * (p & 7));
                if (p < 8) x[0] |= val;
                else if (p < 16) x[1] |= val;
                else if (p < 24) x[2] |= val;
                else x[3] |= val;
                if (++c == welems) c = 0, ++r;
            }
            s0 = make_uint4((uint32_t)x[0], (uint32_t)(x[0] >> 32), (uint32_t)x[1], (uint32_t)(x[1] >> 32));
            s1 = make_uint4((uint32_t)x[2], (uint32_t)(x[2] >> 32), (uint32_t)x[3], (uint32_t)(x[3] >> 32));
        }
        store_bytes(reinterpret_cast<uint8_t*>(ws), cast_word(s0, s1, st, dt), jlo, jhi);
    }
}

// Every box, converting or not: the type pair is per tile, so the branch is warp-uniform.  A tile that converts
// nothing (equal types; 0 and 0 for b200h_copy_boxes_from_host) stores bytes through every piece it uses, so its box
// may span segments; a converting tile's box is one piece.
__global__ void __launch_bounds__(kStageThreads, kBoxCtasPerSm)
    load_boxes_kernel(const CastTile* __restrict__ tiles, uint64_t ntiles, const RangePiece* __restrict__ pieces,
                      const uint8_t* __restrict__ src) {
    __shared__ uint4 rings[kStageThreads / 32][kBoxRing];
    const uint32_t lane = threadIdx.x & 31u;
    uint4* ring = rings[threadIdx.x >> 5];
    const uint4* words = reinterpret_cast<const uint4*>(src);
    const uint64_t nwarps = (uint64_t)gridDim.x * (kStageThreads / 32);
    for (uint64_t t = (uint64_t)(threadIdx.x >> 5) * gridDim.x + blockIdx.x; t < ntiles; t += nwarps) {
        const CastTile ct = tiles[t];
        const BoxTile& b = ct.box;
        const RangePiece* __restrict__ pc = pieces + b.first_piece;
        if (ct.src_type == ct.dst_type) {
            box_tile_steps(b, words, ring, lane, [&](uint64_t from, uint64_t upto) {
                for (uint32_t q = 0; q < b.npieces; ++q) box_words_out(b, pc[q], ring, from, upto, lane);
            });
        } else {
            const uint64_t dev = pc->dev;
            box_tile_steps(b, words, ring, lane, [&](uint64_t from, uint64_t upto) {
                cast_words_out(b, ct.src_type, ct.dst_type, dev, ring, from, upto, lane);
            });
        }
    }
}

// ---- boxes of FP8 elements dequantized on the way (b200h_copy_scaled_boxes_from_host)
//
//   load_scaled_boxes_kernel  the tiles, loads and ring of load_boxes_kernel, with another store step.  A destination
//                        word of 16 / ds elements takes 16 / ds source bytes (8 for a 16-bit target, 4 for F32): from
//                        one ring word, or two and shift_bytes, when they are one run of one row; element by element
//                        otherwise (a word across rows, a box's ends).  Every element is decoded exactly (FP8 -> F16
//                        -> F32, both exact), multiplied by its scale (widened exactly) with one round-to-nearest
//                        multiply that keeps subnormals, and rounded once to the target: bit for bit torch's
//                        (W.float() * S_expanded).to(T) on CUDA.  The tensor coordinates (i, j) of a word's first
//                        element are computed once per word (again where a box row ends inside the word), then
//                        stepped one element at a time; a scale is loaded when (i, j) crosses a block-column edge or a
//                        row's end.  Its own kernel, so that load_boxes_kernel's code stays as it is.

constexpr uint32_t kDtF8E4M3 = B200H_DT_F8E4M3;

// Where the next element of a word lies in the tensor, and its scale.
struct ScaleCursor {
    uint64_t i, j, jend;  // the element's coordinates; the column where its scale block (or the row) ends
    float s;
};

// the scale of element (q.i, q.j), and the end of its block column
__device__ __forceinline__ void scale_load(const ScaledTile& t, ScaleCursor& q) {
    const uint64_t jb = q.j / t.block_cols, k = q.i / t.block_rows * t.scale_cols + jb;
    q.jend = min((jb + 1) * t.block_cols, t.cols);
    if (t.scale_type == kDtF32) {
        q.s = __ldg(reinterpret_cast<const float*>(t.scales) + k);
    } else {
        const unsigned short x = __ldg(reinterpret_cast<const unsigned short*>(t.scales) + k);
        q.s = t.scale_type == kDtF16 ? __half2float(__ushort_as_half(x)) : __bfloat162float(__ushort_as_bfloat16(x));
    }
}

// the cursor at tensor element e (its row-major index)
__device__ __forceinline__ void scale_seek(const ScaledTile& t, uint64_t e, ScaleCursor& q) {
    q.i = e / t.cols;
    q.j = e - q.i * t.cols;
    scale_load(t, q);
}

// the scale of the cursor's element; the cursor moves on to the tensor's next element
__device__ __forceinline__ float scale_next(const ScaledTile& t, ScaleCursor& q) {
    if (q.j == q.jend) {
        if (q.j == t.cols) q.j = 0, ++q.i;
        scale_load(t, q);
    }
    ++q.j;
    return q.s;
}

// the two FP8 elements of the low 16 bits of x (type t), exactly as floats
__device__ __forceinline__ float2 fp8_pair(uint32_t x, uint32_t t) {
    const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(x & 0xffffu),
                                                     t == kDtF8E4M3 ? __NV_E4M3 : __NV_E5M2);
    return __half22float2(__half2(h));
}

// Destination words of the box (one piece at device address `dev`) whose elements have packed source bytes in
// [from, upto) (clipped to [b.dlo, b.dhi)) and whose last element's source lies before `upto`.
__device__ __forceinline__ void scaled_words_out(const ScaledTile& t, uint64_t dev, const uint4* ring, uint64_t from,
                                                 uint64_t upto, uint32_t lane) {
    const BoxTile& b = t.cast.box;
    const uint32_t st = t.cast.src_type, dt = t.cast.dst_type, ds = dt_bytes(dt);
    const uint64_t qhi = b.dhi * ds, lo = from * ds, hi = upto * ds;
    if (lo >= hi) return;
    const uint64_t qa = dev + b.dlo * ds, qe = dev + qhi, ha = dev + hi;
    // a word whose elements go on past `hi` waits for the next step
    const uint64_t w1 = hi < qhi ? ha >> 4 : ((ha - 1) >> 4) + 1;
    for (uint64_t w = ((dev + lo) >> 4) + lane; w < w1; w += 32) {
        const uint64_t ws = w * 16, aa = max(ws, qa), ea = min(ws + 16, qe);
        const uint32_t jlo = (uint32_t)(aa - ws), jhi = (uint32_t)(ea - ws);
        const uint64_t e = (aa - dev) / ds;  // the word's first element, counted in the box's packed run
        uint64_t r = e / b.width, c = e % b.width;
        ScaleCursor q;
        uint4 v;
        if (jhi - jlo == 16 && c + 16 / ds <= b.width) {
            const uint64_t s = b.src + r * b.pitch + c;
            const uint32_t slot = (uint32_t)(box_virtual(b, r, s) - b.v0), sh = (uint32_t)s & 15u;
            const uint4 w0 = ring[slot % kBoxRing];
            const uint4 x = sh + 16 / ds > 16 ? shift_bytes(w0, ring[(slot + 1) % kBoxRing], sh) : shift_bytes(w0, w0, sh);
            scale_seek(t, t.first_elem + r * b.pitch + c, q);
            const float2 p0 = fp8_pair(x.x, st), p1 = fp8_pair(x.x >> 16, st);
            const float s0 = scale_next(t, q), s1 = scale_next(t, q), s2 = scale_next(t, q), s3 = scale_next(t, q);
            const float a0 = __fmul_rn(p0.x, s0), a1 = __fmul_rn(p0.y, s1), a2 = __fmul_rn(p1.x, s2),
                        a3 = __fmul_rn(p1.y, s3);
            if (ds == 4) {
                v = make_uint4(__float_as_uint(a0), __float_as_uint(a1), __float_as_uint(a2), __float_as_uint(a3));
            } else {
                const float2 p2 = fp8_pair(x.y, st), p3 = fp8_pair(x.y >> 16, st);
                const float s4 = scale_next(t, q), s5 = scale_next(t, q), s6 = scale_next(t, q), s7 = scale_next(t, q);
                v = make_uint4(narrow_pair(a0, a1, dt), narrow_pair(a2, a3, dt),
                               narrow_pair(__fmul_rn(p2.x, s4), __fmul_rn(p2.y, s5), dt),
                               narrow_pair(__fmul_rn(p3.x, s6), __fmul_rn(p3.y, s7), dt));
            }
        } else {
            uint64_t x[2] = {0, 0};  // the results, element k at byte k * ds
            bool seek = true;
#pragma unroll 1
            for (uint32_t j = jlo; j < jhi; j += ds) {
                const uint64_t s = b.src + r * b.pitch + c;
                const uint8_t* word =
                    reinterpret_cast<const uint8_t*>(ring + (uint32_t)(box_virtual(b, r, s) - b.v0) % kBoxRing);
                if (seek) scale_seek(t, t.first_elem + r * b.pitch + c, q), seek = false;
                const float a = __fmul_rn(fp8_pair(word[s & 15u], st).x, scale_next(t, q));
                const uint64_t val = (ds == 4 ? (uint64_t)__float_as_uint(a) : (uint64_t)(narrow_pair(a, 0.f, dt) & 0xffffu))
                                     << (8 * (j & 7));
                if (j < 8) x[0] |= val;
                else x[1] |= val;
                if (++c == b.width) c = 0, ++r, seek = true;
            }
            v = make_uint4((uint32_t)x[0], (uint32_t)(x[0] >> 32), (uint32_t)x[1], (uint32_t)(x[1] >> 32));
        }
        store_bytes(reinterpret_cast<uint8_t*>(ws), v, jlo, jhi);
    }
}

__global__ void __launch_bounds__(kStageThreads, kBoxCtasPerSm)
    load_scaled_boxes_kernel(const ScaledTile* __restrict__ tiles, uint64_t ntiles,
                             const RangePiece* __restrict__ pieces, const uint8_t* __restrict__ src) {
    __shared__ uint4 rings[kStageThreads / 32][kBoxRing];
    const uint32_t lane = threadIdx.x & 31u;
    uint4* ring = rings[threadIdx.x >> 5];
    const uint4* words = reinterpret_cast<const uint4*>(src);
    const uint64_t nwarps = (uint64_t)gridDim.x * (kStageThreads / 32);
    for (uint64_t k = (uint64_t)(threadIdx.x >> 5) * gridDim.x + blockIdx.x; k < ntiles; k += nwarps) {
        const ScaledTile t = tiles[k];
        const uint64_t dev = pieces[t.cast.box.first_piece].dev;
        box_tile_steps(t.cast.box, words, ring, lane, [&](uint64_t from, uint64_t upto) {
            scaled_words_out(t, dev, ring, from, upto, lane);
        });
    }
}

// ---- stage_ranges_kernel, whose pieces may change type on the way out (b200h_copy_cast_ranges, and the wave-slot
//      gather of b200h_hash_cast_segment_parts_device)
//
// A converting piece's image is its source elements converted, element k at image byte k * ds; a range may start at
// any image byte, so a piece records the element that holds its first byte and that byte's place in it (`phase`).
//   * a destination word inside one converting piece whose first byte starts an element takes its 16 / ds * ss source
//     bytes with aligned 16-byte loads inside the piece's 16-byte hull (two or three narrowing F32, one or two between
//     F16 and BF16, one widening unless the 8 bytes cross a word), joined with shift_bytes and converted by cast_word;
//   * any other word that is not inside one piece that converts nothing (across pieces, or holding part of an element)
//     is assembled element by element, one byte at a time, and still stored as one word.
// A single element converts through the paired intrinsics too (the other half of the pair unused), so every path gives
// the same bits.

// one element of type st (in the low bits of x) as type dt
__device__ __forceinline__ uint32_t cast_one(uint32_t x, uint32_t st, uint32_t dt) {
    if (st == kDtF32) return narrow_pair(__uint_as_float(x), 0.f, dt) & 0xffffu;
    const float2 f = widen_pair(x & 0xffffu, st);
    return dt == kDtF32 ? __float_as_uint(f.x) : narrow_pair(f.x, 0.f, dt) & 0xffffu;
}

// byte d (a destination offset inside piece p) of the piece's image
__device__ __forceinline__ uint32_t image_byte(const CastPiece& p, uint64_t d) {
    const uint8_t* s = reinterpret_cast<const uint8_t*>(p.r.dev);
    if (p.src_type == p.dst_type) return s[d - p.r.host];
    const uint32_t ss = dt_bytes(p.src_type), ds = dt_bytes(p.dst_type);
    const uint64_t rel = d - p.r.host + p.phase, e = ds == 4 ? rel >> 2 : rel >> 1;
    const uint32_t x = ss == 4 ? *reinterpret_cast<const uint32_t*>(s + e * 4)
                               : (uint32_t)*reinterpret_cast<const uint16_t*>(s + e * 2);
    return (cast_one(x, p.src_type, p.dst_type) >> (8 * (uint32_t)(rel & (ds - 1)))) & 0xffu;
}

// the destination word at d, byte by byte from pieces pc[i ..] (pc[i] holds d; the word lies in the range)
__device__ __forceinline__ uint4 image_word(const CastPiece* __restrict__ pc, uint32_t i, uint64_t d) {
    uint64_t x[2] = {0, 0};
    uint64_t end = pc[i].r.host + pc[i].r.len;
#pragma unroll 1
    for (uint32_t j = 0; j < 16; ++j) {
        while (d + j >= end) {
            ++i;
            end = pc[i].r.host + pc[i].r.len;
        }
        const uint64_t b = (uint64_t)image_byte(pc[i], d + j) << (8 * (j & 7));
        if (j < 8) x[0] |= b;
        else x[1] |= b;
    }
    return make_uint4((uint32_t)x[0], (uint32_t)(x[0] >> 32), (uint32_t)x[1], (uint32_t)(x[1] >> 32));
}

// the destination word of the 16 / ds elements at s (a multiple of ss), inside one converting piece
__device__ __forceinline__ uint4 cast_load_word(const uint8_t* s, uint32_t st, uint32_t dt) {
    const uint32_t sh = (uint32_t)((uintptr_t)s & 15u);
    const uint4* a = reinterpret_cast<const uint4*>(s - sh);
    const uint4 w0 = __ldg(a);
    uint4 lo, hi = make_uint4(0, 0, 0, 0);
    if (st == kDtF32) {  // 32 source bytes
        const uint4 w1 = __ldg(a + 1);
        lo = sh ? shift_bytes(w0, w1, sh) : w0;
        hi = sh ? shift_bytes(w1, __ldg(a + 2), sh) : w1;
    } else if (dt != kDtF32) {  // 16
        lo = sh ? shift_bytes(w0, __ldg(a + 1), sh) : w0;
    } else {  // 8
        lo = sh > 8 ? shift_bytes(w0, __ldg(a + 1), sh) : shift_bytes(w0, w0, sh);
    }
    return cast_word(lo, hi, st, dt);
}

__global__ void __launch_bounds__(kStageThreads, kStageCtasPerSm)
    stage_ranges_kernel(const RangeTile* __restrict__ tiles, uint64_t ntiles, const CastPiece* __restrict__ pieces,
                        uint8_t* __restrict__ dst) {
    for (uint64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const RangeTile tile = tiles[t];
        const CastPiece* __restrict__ pc = pieces + tile.first_piece;
        uint8_t* out = dst + tile.host;
        const uint32_t words = tile.len >> 4, tail = tile.len & 15u;
        if (tile.npieces == 1 && pc->src_type == pc->dst_type) {
            stage_one_piece(reinterpret_cast<const uint8_t*>(pc->r.dev) + (tile.host - pc->r.host), out, words, tail);
            continue;
        }
        uint32_t cur = 0;
        for (uint32_t w = threadIdx.x; w < words; w += kStageThreads) {
            const uint64_t d = tile.host + (uint64_t)w * 16;
            if (d >= pc[cur].r.host + pc[cur].r.len) cur = find_piece(pc, cur + 1, tile.npieces, d);
            const CastPiece p = pc[cur];
            const uint64_t in = d - p.r.host, left = p.r.len - in;
            const uint8_t* s = reinterpret_cast<const uint8_t*>(p.r.dev);
            uint4 v;
            if (left >= 16 && p.src_type == p.dst_type) {
                v = load_word(s + in);
            } else if (left >= 16 && ((in + p.phase) & (dt_bytes(p.dst_type) - 1)) == 0) {
                const uint64_t e = (in + p.phase) / dt_bytes(p.dst_type);
                v = cast_load_word(s + e * dt_bytes(p.src_type), p.src_type, p.dst_type);
            } else {
                v = image_word(pc, cur, d);
            }
            *reinterpret_cast<uint4*>(dst + d) = v;
        }
        if (threadIdx.x < tail) {
            const uint64_t d = tile.host + (uint64_t)words * 16 + threadIdx.x;
            dst[d] = (uint8_t)image_byte(pc[find_piece(pc, 0, tile.npieces, d)], d);
        }
    }
}

}  // namespace

int launch_load_boxes(const CastTile* tiles, uint64_t ntiles, const RangePiece* pieces, const void* src, cudaStream_t st) {
    if (!ntiles) return 0;
    const uint64_t cap = (uint64_t)device_sm_count() * kBoxCtasPerSm;
    load_boxes_kernel<<<(int)(ntiles < cap ? ntiles : cap), kStageThreads, 0, st>>>(tiles, ntiles, pieces,
                                                                                   static_cast<const uint8_t*>(src));
    return 1;
}

int launch_load_scaled_boxes(const ScaledTile* tiles, uint64_t ntiles, const RangePiece* pieces, const void* src,
                             cudaStream_t st) {
    if (!ntiles) return 0;
    const uint64_t cap = (uint64_t)device_sm_count() * kBoxCtasPerSm;
    load_scaled_boxes_kernel<<<(int)(ntiles < cap ? ntiles : cap), kStageThreads, 0, st>>>(
        tiles, ntiles, pieces, static_cast<const uint8_t*>(src));
    return 1;
}

int launch_load_ranges(const RangeTile* tiles, uint64_t ntiles, const RangePiece* pieces, const void* src, cudaStream_t st) {
    if (!ntiles) return 0;
    const uint64_t per_cta = kStageThreads / 32, ctas = (ntiles + per_cta - 1) / per_cta;
    const uint64_t cap = (uint64_t)device_sm_count() * kStageCtasPerSm;
    load_ranges_kernel<<<(int)(ctas < cap ? ctas : cap), kStageThreads, 0, st>>>(tiles, ntiles, pieces,
                                                                                static_cast<const uint8_t*>(src));
    return 1;
}

int launch_stage_ranges(const RangeTile* tiles, uint64_t ntiles, const CastPiece* pieces, void* dst, cudaStream_t st) {
    if (!ntiles) return 0;
    const uint64_t cap = (uint64_t)device_sm_count() * kStageCtasPerSm;
    stage_ranges_kernel<<<(int)(ntiles < cap ? ntiles : cap), kStageThreads, 0, st>>>(tiles, ntiles, pieces,
                                                                                      static_cast<uint8_t*>(dst));
    return 1;
}

}  // namespace b200h
