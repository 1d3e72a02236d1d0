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

// ---- stage_scaled_ranges_kernel: stage_ranges_kernel whose pieces may also quantize to FP8 E4M3 on the way out
//      (b200h_copy_scaled_ranges, and the wave-slot gather of b200h_hash_scaled_segment_parts_device)
//
// A quantizing piece's image has one byte per element, so every image byte starts an element and a destination word
// inside the piece is 16 elements: 32 source bytes from a 16-bit source, 64 from F32, taken with aligned 16-byte loads
// inside the piece's hull and shift_bytes.  Element e = (i, j) of the weight is multiplied by its block's
// m = RN(RN(1 / a) * 448) with one round-to-nearest multiply that keeps subnormals and converted with the sm_90 paired
// E4M3 conversion (round to nearest even; satfinite, which no element reaches: |x * m| rounds to at most 448, and a NaN
// product gives 0x7F either way).  (i, j) is computed once per word, then stepped one element at a time; m is reloaded
// only where j crosses a block-column edge or a row's end.  Words across pieces and tail bytes go element by element.
// Its own kernel, so that stage_ranges_kernel's code stays as it is.

constexpr float kE4M3Max = 448.0f;

// The element of a quantizing piece that the cursor stands on, and its block's multiplier.
struct QuantCursor {
    uint64_t i, j, jend;  // the element's coordinates; the column where its block column (or the row) ends
    float m;
};

__device__ __forceinline__ void quant_load(const PieceScale& q, QuantCursor& c) {
    const uint64_t jb = c.j / q.block_cols;
    c.jend = min((jb + 1) * q.block_cols, q.cols);
    const float a = __ldg(reinterpret_cast<const float*>(q.amax) + c.i / q.block_rows * q.scale_cols + jb);
    c.m = __fmul_rn(__frcp_rn(a), kE4M3Max);
}

// the cursor at element e of the weight (its row-major index)
__device__ __forceinline__ void quant_seek(const PieceScale& q, uint64_t e, QuantCursor& c) {
    c.i = e / q.cols;
    c.j = e - c.i * q.cols;
    quant_load(q, c);
}

// the multiplier of the cursor's element; the cursor moves on to the weight's next element
__device__ __forceinline__ float quant_next(const PieceScale& q, QuantCursor& c) {
    if (c.j == c.jend) {
        if (c.j == q.cols) c.j = 0, ++c.i;
        quant_load(q, c);
    }
    ++c.j;
    return c.m;
}

// one element of type st (F32, F16 or BF16; in the low bits of x), exactly as a float
__device__ __forceinline__ float widen_one(uint32_t x, uint32_t st) {
    return st == kDtF32 ? __uint_as_float(x) : widen_pair(x & 0xffffu, st).x;
}

// two products as E4M3, the first in the low byte
__device__ __forceinline__ uint32_t e4m3_pair(float a, float b) {
    return (uint32_t)__nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
}

// the destination word of the 16 elements at s (a multiple of ss, inside one quantizing piece), whose first is element e
__device__ __forceinline__ uint4 quant_load_word(const uint8_t* s, uint32_t st, const PieceScale& q, uint64_t e) {
    const uint32_t sh = (uint32_t)((uintptr_t)s & 15u);
    const uint4* a = reinterpret_cast<const uint4*>(s - sh);
    float x[16];
    if (st == kDtF32) {  // 64 source bytes
        uint4 w[5];
        w[0] = __ldg(a);
#pragma unroll
        for (int k = 1; k < 4; ++k) w[k] = __ldg(a + k);
        w[4] = sh ? __ldg(a + 4) : w[3];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint4 v = sh ? shift_bytes(w[k], w[k + 1], sh) : w[k];
            x[4 * k] = __uint_as_float(v.x), x[4 * k + 1] = __uint_as_float(v.y);
            x[4 * k + 2] = __uint_as_float(v.z), x[4 * k + 3] = __uint_as_float(v.w);
        }
    } else {  // 32
        const uint4 w0 = __ldg(a), w1 = __ldg(a + 1), w2 = sh ? __ldg(a + 2) : w1;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const uint4 v = sh ? shift_bytes(k ? w1 : w0, k ? w2 : w1, sh) : (k ? w1 : w0);
            const float2 p0 = widen_pair(v.x, st), p1 = widen_pair(v.y, st), p2 = widen_pair(v.z, st),
                         p3 = widen_pair(v.w, st);
            x[8 * k] = p0.x, x[8 * k + 1] = p0.y, x[8 * k + 2] = p1.x, x[8 * k + 3] = p1.y;
            x[8 * k + 4] = p2.x, x[8 * k + 5] = p2.y, x[8 * k + 6] = p3.x, x[8 * k + 7] = p3.y;
        }
    }
    QuantCursor c;
    quant_seek(q, e, c);
    uint32_t out[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float y0 = __fmul_rn(x[4 * k], quant_next(q, c)), y1 = __fmul_rn(x[4 * k + 1], quant_next(q, c));
        const float y2 = __fmul_rn(x[4 * k + 2], quant_next(q, c)), y3 = __fmul_rn(x[4 * k + 3], quant_next(q, c));
        out[k] = e4m3_pair(y0, y1) | e4m3_pair(y2, y3) << 16;
    }
    return make_uint4(out[0], out[1], out[2], out[3]);
}

// byte d (a destination offset inside piece p, whose scales are q) of the piece's image
__device__ __forceinline__ uint32_t scaled_image_byte(const CastPiece& p, const PieceScale& q, uint64_t d) {
    if (p.dst_type != kDtF8E4M3) return image_byte(p, d);
    const uint64_t in = d - p.r.host;
    const uint8_t* s = reinterpret_cast<const uint8_t*>(p.r.dev);
    const uint32_t x = p.src_type == kDtF32 ? *reinterpret_cast<const uint32_t*>(s + in * 4)
                                            : (uint32_t)*reinterpret_cast<const uint16_t*>(s + in * 2);
    QuantCursor c;
    quant_seek(q, q.first_elem + in, c);
    return e4m3_pair(__fmul_rn(widen_one(x, p.src_type), c.m), 0.f) & 0xffu;
}

// the destination word at d, byte by byte from pieces pc[i ..] (pc[i] holds d; the word lies in the range)
__device__ __forceinline__ uint4 scaled_image_word(const CastPiece* __restrict__ pc, const PieceScale* __restrict__ ps,
                                                   uint32_t i, uint64_t d) {
    uint64_t x[2] = {0, 0};
    uint64_t end = pc[i].r.host + pc[i].r.len;
#pragma unroll 1
    for (uint32_t j = 0; j < 16; ++j) {
        while (d + j >= end) {
            ++i;
            end = pc[i].r.host + pc[i].r.len;
        }
        const uint64_t b = (uint64_t)scaled_image_byte(pc[i], ps[i], d + j) << (8 * (j & 7));
        if (j < 8) x[0] |= b;
        else x[1] |= b;
    }
    return make_uint4((uint32_t)x[0], (uint32_t)(x[0] >> 32), (uint32_t)x[1], (uint32_t)(x[1] >> 32));
}

__global__ void __launch_bounds__(kStageThreads, kStageCtasPerSm)
    stage_scaled_ranges_kernel(const RangeTile* __restrict__ tiles, uint64_t ntiles,
                               const CastPiece* __restrict__ pieces, const PieceScale* __restrict__ scales,
                               uint8_t* __restrict__ dst) {
    for (uint64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const RangeTile tile = tiles[t];
        const CastPiece* __restrict__ pc = pieces + tile.first_piece;
        const PieceScale* __restrict__ ps = scales + tile.first_piece;
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
            } else if (left >= 16 && p.dst_type == kDtF8E4M3) {
                const PieceScale q = ps[cur];
                v = quant_load_word(s + in * dt_bytes(p.src_type), p.src_type, q, q.first_elem + in);
            } else if (left >= 16 && ((in + p.phase) & (dt_bytes(p.dst_type) - 1)) == 0) {
                const uint64_t e = (in + p.phase) / dt_bytes(p.dst_type);
                v = cast_load_word(s + e * dt_bytes(p.src_type), p.src_type, p.dst_type);
            } else {
                v = scaled_image_word(pc, ps, cur, d);
            }
            *reinterpret_cast<uint4*>(dst + d) = v;
        }
        if (threadIdx.x < tail) {
            const uint64_t d = tile.host + (uint64_t)words * 16 + threadIdx.x;
            const uint32_t k = find_piece(pc, 0, tile.npieces, d);
            dst[d] = (uint8_t)scaled_image_byte(pc[k], ps[k], d);
        }
    }
}

// ---- FP8 block scales (b200h_fp8_block_scales)
//
//   fp8_amax_kernel      persistent CTAs take tiles (up to sub_rows x sub_cols elements of one block of one job); warp
//                        w takes the tile's rows w, w + 8, ..., its lanes the columns.  |x| is widened to F32 and its
//                        bits max-reduced as integers (for non-negative floats the integer order is the float order,
//                        and a NaN's bits exceed every other value's), per warp, then per CTA, then one atomicMax per
//                        CTA into the block's amax word.
//   fp8_finalize_kernel  a = amax is NaN ? amax : max(amax, 1e-4f) in place, s = a * RN(1 / 448): the F32 arithmetic of
//                        torch's clamp and its CUDA division by a CPU scalar (a multiplication by its reciprocal).

constexpr int kScaleThreads = 256;
constexpr float kAmaxFloor = 1e-4f;
constexpr float kInvE4M3Max = 1.0f / 448.0f;

__device__ __forceinline__ uint32_t abs_bits(const uint8_t* src, uint64_t e, uint32_t st) {
    if (st == kDtF32) return __ldg(reinterpret_cast<const uint32_t*>(src) + e) & 0x7fffffffu;
    const uint32_t x = __ldg(reinterpret_cast<const unsigned short*>(src) + e);
    return __float_as_uint(widen_one(x, st)) & 0x7fffffffu;
}

__global__ void __launch_bounds__(kScaleThreads)
    fp8_amax_kernel(const ScaleJob* __restrict__ jobs, uint32_t njobs, uint64_t ntiles) {
    __shared__ uint32_t red[kScaleThreads / 32];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    for (uint64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        uint32_t lo = 0, hi = njobs - 1;
        while (lo < hi) {
            const uint32_t mid = (lo + hi + 1) >> 1;
            if (jobs[mid].first_tile <= t) lo = mid;
            else hi = mid - 1;
        }
        const ScaleJob& J = jobs[lo];
        const uint64_t u = t - J.first_tile, blk = u / J.tiles_per_block, in = u % J.tiles_per_block;
        const uint64_t bi = blk / J.scale_cols, bj = blk % J.scale_cols;
        const uint64_t si = in / J.tile_cols, sj = in % J.tile_cols;
        const uint64_t r0 = bi * J.block_rows + si * J.sub_rows, c0 = bj * J.block_cols + sj * J.sub_cols;
        const uint64_t r1 = min(min(r0 + J.sub_rows, (bi + 1) * J.block_rows), J.rows);
        const uint64_t c1 = min(min(c0 + J.sub_cols, (bj + 1) * J.block_cols), J.cols);
        if (r0 >= r1 || c0 >= c1) continue;  // a tile past an edge block's end (the whole CTA skips it)
        const uint8_t* src = reinterpret_cast<const uint8_t*>(J.src);
        const uint32_t st = J.src_type, w = (uint32_t)(c1 - c0);
        uint32_t m = 0;
        for (uint64_t r = r0 + warp; r < r1; r += kScaleThreads / 32) {
            const uint64_t base = r * J.cols + c0;
#pragma unroll 4
            for (uint32_t c = lane; c < w; c += 32) m = max(m, abs_bits(src, base + c, st));
        }
#pragma unroll
        for (int k = 16; k; k >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, k));
        if (lane == 0) red[warp] = m;
        __syncthreads();
        if (threadIdx.x == 0) {
#pragma unroll
            for (int k = 1; k < kScaleThreads / 32; ++k) m = max(m, red[k]);
            atomicMax(reinterpret_cast<unsigned int*>(J.amax) + (blk), m);
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kScaleThreads)
    fp8_finalize_kernel(const ScaleJob* __restrict__ jobs, uint32_t njobs, uint64_t nblocks) {
    for (uint64_t k = (uint64_t)blockIdx.x * kScaleThreads + threadIdx.x; k < nblocks;
         k += (uint64_t)gridDim.x * kScaleThreads) {
        uint32_t lo = 0, hi = njobs - 1;
        while (lo < hi) {
            const uint32_t mid = (lo + hi + 1) >> 1;
            if (jobs[mid].first_block <= k) lo = mid;
            else hi = mid - 1;
        }
        const uint64_t b = k - jobs[lo].first_block;
        float* amax = reinterpret_cast<float*>(jobs[lo].amax) + b;
        const float x = *amax, a = isnan(x) ? x : fmaxf(x, kAmaxFloor);
        *amax = a;
        reinterpret_cast<float*>(jobs[lo].scales)[b] = __fmul_rn(a, kInvE4M3Max);
    }
}

// ---- boxes of F32 / F16 / BF16 elements quantized to E4M3 on the way in (b200h_fp8_amax_boxes_from_host,
//      b200h_copy_quant_boxes_from_host)
//
//   fp8_amax_boxes_kernel   the tiles, loads and ring of load_boxes_kernel; no device stores but the amax.  At each
//                           step lane k takes the k-th 32nd of the elements whose source has arrived, contiguous, and
//                           max-reduces the bits of |x| widened to F32 (as fp8_amax_kernel does) per block, following
//                           the block with a cursor; where its elements leave a block it flushes with one atomicMax.
//                           Its last block's value then goes through a warp reduction over the lanes that end in the
//                           same block, and one lane per such run issues the atomicMax.
//   load_quant_boxes_kernel the same tiles and ring with the store step of the cast boxes: a destination word is 16 E4M3
//                           elements, 32 or 64 source bytes (three or five ring words with shift_bytes) when they are
//                           one run of one row, element by element otherwise.  The multiplier and conversion are those
//                           of stage_scaled_ranges_kernel (quant_seek / quant_next: m = RN(RN(1 / a) * 448), reloaded
//                           only where j crosses a block-column edge or a row's end; FMUL without .FTZ; satfinite).
// The a they read was finalized (fp8_finalize_kernel, launched by b200h_copy_quant_boxes_from_host before the copy).

// Bits of |x| of the element of type st at byte `at` of a ring word, widened to F32.
__device__ __forceinline__ uint32_t ring_abs_bits(const uint8_t* word, uint32_t at, uint32_t st) {
    const uint32_t x = st == kDtF32 ? *reinterpret_cast<const uint32_t*>(word + at)
                                    : (uint32_t)*reinterpret_cast<const uint16_t*>(word + at);
    return __float_as_uint(widen_one(x, st)) & 0x7fffffffu;
}

// The amax of the box's elements whose packed source bytes lie in [from, upto) (clipped to [b.dlo, b.dhi)).
__device__ __forceinline__ void amax_words_out(const BoxTile& b, uint32_t st, const PieceScale& q, const uint4* ring,
                                               uint64_t from, uint64_t upto, uint32_t lane) {
    const uint32_t ss = dt_bytes(st);
    const uint64_t lo = max(from, b.dlo) / ss, hi = min(upto, b.dhi) / ss, welems = b.width / ss;
    const uint64_t per = hi > lo ? (hi - lo + 31) / 32 : 0;
    const uint64_t e0 = min(lo + lane * per, hi), e1 = min(e0 + per, hi);
    float* amax = reinterpret_cast<float*>(q.amax);
    uint64_t key = ~0ull;
    uint32_t m = 0;
    if (e0 < e1) {
        uint64_t r = e0 / welems, c = e0 % welems;
        QuantCursor cur;
        bool seek = true;
#pragma unroll 1
        for (uint64_t e = e0; e < e1; ++e) {
            bool load = seek;
            if (seek) {  // the element's coordinates, once per lane and again where a box row ends
                const uint64_t te = q.first_elem + r * (b.pitch / ss) + c;
                cur.i = te / q.cols;
                cur.j = te - cur.i * q.cols;
                seek = false;
            } else if (cur.j == cur.jend) {
                if (cur.j == q.cols) cur.j = 0, ++cur.i;
                load = true;
            }
            if (load) {
                const uint64_t jb = cur.j / q.block_cols, k = cur.i / q.block_rows * q.scale_cols + jb;
                cur.jend = min((jb + 1) * q.block_cols, q.cols);
                if (k != key) {
                    if (key != ~0ull) atomicMax(reinterpret_cast<unsigned int*>(amax) + key, m);
                    key = k, m = 0;
                }
            }
            const uint64_t s = b.src + r * b.pitch + c * ss;
            const uint8_t* word =
                reinterpret_cast<const uint8_t*>(ring + (uint32_t)(box_virtual(b, r, s) - b.v0) % kBoxRing);
            m = max(m, ring_abs_bits(word, (uint32_t)s & 15u, st));
            ++cur.j;
            if (++c == welems) c = 0, ++r, seek = true;
        }
    }
    // lanes that end in one block: a segmented max, every merged value from a lane of the same key
#pragma unroll
    for (int k = 1; k < 32; k <<= 1) {
        const uint32_t om = __shfl_down_sync(0xffffffffu, m, k);
        const uint64_t ok = __shfl_down_sync(0xffffffffu, key, k);
        if (lane + k < 32 && ok == key) m = max(m, om);
    }
    const uint64_t before = __shfl_up_sync(0xffffffffu, key, 1);
    if (key != ~0ull && (lane == 0 || before != key)) atomicMax(reinterpret_cast<unsigned int*>(amax) + key, m);
}

__global__ void __launch_bounds__(kStageThreads, kBoxCtasPerSm)
    fp8_amax_boxes_kernel(const QuantTile* __restrict__ tiles, uint64_t ntiles, const uint8_t* __restrict__ src) {
    __shared__ uint4 rings[kStageThreads / 32][kBoxRing];
    const uint32_t lane = threadIdx.x & 31u;
    uint4* ring = rings[threadIdx.x >> 5];
    const uint4* words = reinterpret_cast<const uint4*>(src);
    const uint64_t nwarps = (uint64_t)gridDim.x * (kStageThreads / 32);
    for (uint64_t k = (uint64_t)(threadIdx.x >> 5) * gridDim.x + blockIdx.x; k < ntiles; k += nwarps) {
        const QuantTile t = tiles[k];
        box_tile_steps(t.cast.box, words, ring, lane, [&](uint64_t from, uint64_t upto) {
            amax_words_out(t.cast.box, t.cast.src_type, t.q, ring, from, upto, lane);
        });
    }
}

// Destination words of the box (one piece at device address `dev`, one byte per element) whose elements have packed
// source bytes in [from, upto) (clipped to [b.dlo, b.dhi)) and whose last element's source lies before `upto`.
__device__ __forceinline__ void quant_words_out(const BoxTile& b, uint32_t st, const PieceScale& q, uint64_t dev,
                                                const uint4* ring, uint64_t from, uint64_t upto, uint32_t lane) {
    const uint32_t ss = dt_bytes(st);
    const uint64_t qhi = b.dhi / ss, lo = from / ss, hi = upto / ss;
    if (lo >= hi) return;
    const uint64_t qa = dev + b.dlo / ss, qe = dev + qhi, ha = dev + hi, welems = b.width / ss;
    // a word whose elements go on past `hi` waits for the next step
    const uint64_t w1 = hi < qhi ? ha >> 4 : ((ha - 1) >> 4) + 1;
    for (uint64_t w = ((dev + lo) >> 4) + lane; w < w1; w += 32) {
        const uint64_t ws = w * 16, aa = max(ws, qa), ea = min(ws + 16, qe);
        const uint32_t jlo = (uint32_t)(aa - ws), jhi = (uint32_t)(ea - ws);
        const uint64_t e = aa - dev;  // the word's first element, counted in the box's packed run
        uint64_t r = e / welems, c = e % welems;
        QuantCursor cur;
        uint4 v;
        if (jhi - jlo == 16 && c + 16 <= welems) {
            const uint64_t s = b.src + r * b.pitch + c * ss;
            const uint32_t slot = (uint32_t)(box_virtual(b, r, s) - b.v0), sh = (uint32_t)s & 15u;
            float x[16];
            if (st == kDtF32) {  // 64 source bytes
                uint4 wd[5];
#pragma unroll
                for (int k = 0; k < 4; ++k) wd[k] = ring[(slot + k) % kBoxRing];
                wd[4] = sh ? ring[(slot + 4) % kBoxRing] : wd[3];
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const uint4 u = sh ? shift_bytes(wd[k], wd[k + 1], sh) : wd[k];
                    x[4 * k] = __uint_as_float(u.x), x[4 * k + 1] = __uint_as_float(u.y);
                    x[4 * k + 2] = __uint_as_float(u.z), x[4 * k + 3] = __uint_as_float(u.w);
                }
            } else {  // 32
                const uint4 w0 = ring[slot % kBoxRing], w1 = ring[(slot + 1) % kBoxRing];
                const uint4 w2 = sh ? ring[(slot + 2) % kBoxRing] : w1;
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                    const uint4 u = sh ? shift_bytes(k ? w1 : w0, k ? w2 : w1, sh) : (k ? w1 : w0);
                    const float2 p0 = widen_pair(u.x, st), p1 = widen_pair(u.y, st), p2 = widen_pair(u.z, st),
                                 p3 = widen_pair(u.w, st);
                    x[8 * k] = p0.x, x[8 * k + 1] = p0.y, x[8 * k + 2] = p1.x, x[8 * k + 3] = p1.y;
                    x[8 * k + 4] = p2.x, x[8 * k + 5] = p2.y, x[8 * k + 6] = p3.x, x[8 * k + 7] = p3.y;
                }
            }
            quant_seek(q, q.first_elem + r * (b.pitch / ss) + c, cur);
            uint32_t out[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float y0 = __fmul_rn(x[4 * k], quant_next(q, cur)), y1 = __fmul_rn(x[4 * k + 1], quant_next(q, cur));
                const float y2 = __fmul_rn(x[4 * k + 2], quant_next(q, cur)),
                            y3 = __fmul_rn(x[4 * k + 3], quant_next(q, cur));
                out[k] = e4m3_pair(y0, y1) | e4m3_pair(y2, y3) << 16;
            }
            v = make_uint4(out[0], out[1], out[2], out[3]);
        } else {
            uint64_t y[2] = {0, 0};  // the codes, element k at byte k
            bool seek = true;
#pragma unroll 1
            for (uint32_t j = jlo; j < jhi; ++j) {
                const uint64_t s = b.src + r * b.pitch + c * ss;
                const uint8_t* word =
                    reinterpret_cast<const uint8_t*>(ring + (uint32_t)(box_virtual(b, r, s) - b.v0) % kBoxRing);
                const uint32_t x = ss == 4 ? *reinterpret_cast<const uint32_t*>(word + (s & 15u))
                                           : (uint32_t)*reinterpret_cast<const uint16_t*>(word + (s & 15u));
                if (seek) quant_seek(q, q.first_elem + r * (b.pitch / ss) + c, cur), seek = false;
                const uint64_t code = e4m3_pair(__fmul_rn(widen_one(x, st), quant_next(q, cur)), 0.f) & 0xffu;
                if (j < 8) y[0] |= code << (8 * j);
                else y[1] |= code << (8 * (j - 8));
                if (++c == welems) c = 0, ++r, seek = true;
            }
            v = make_uint4((uint32_t)y[0], (uint32_t)(y[0] >> 32), (uint32_t)y[1], (uint32_t)(y[1] >> 32));
        }
        store_bytes(reinterpret_cast<uint8_t*>(ws), v, jlo, jhi);
    }
}

__global__ void __launch_bounds__(kStageThreads, kBoxCtasPerSm)
    load_quant_boxes_kernel(const QuantTile* __restrict__ tiles, uint64_t ntiles, const RangePiece* __restrict__ pieces,
                            const uint8_t* __restrict__ src) {
    __shared__ uint4 rings[kStageThreads / 32][kBoxRing];
    const uint32_t lane = threadIdx.x & 31u;
    uint4* ring = rings[threadIdx.x >> 5];
    const uint4* words = reinterpret_cast<const uint4*>(src);
    const uint64_t nwarps = (uint64_t)gridDim.x * (kStageThreads / 32);
    for (uint64_t k = (uint64_t)(threadIdx.x >> 5) * gridDim.x + blockIdx.x; k < ntiles; k += nwarps) {
        const QuantTile t = tiles[k];
        const uint64_t dev = pieces[t.cast.box.first_piece].dev;
        box_tile_steps(t.cast.box, words, ring, lane, [&](uint64_t from, uint64_t upto) {
            quant_words_out(t.cast.box, t.cast.src_type, t.q, dev, ring, from, upto, lane);
        });
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

int launch_stage_scaled_ranges(const RangeTile* tiles, uint64_t ntiles, const CastPiece* pieces,
                               const PieceScale* scales, void* dst, cudaStream_t st) {
    if (!ntiles) return 0;
    const uint64_t cap = (uint64_t)device_sm_count() * kStageCtasPerSm;
    stage_scaled_ranges_kernel<<<(int)(ntiles < cap ? ntiles : cap), kStageThreads, 0, st>>>(
        tiles, ntiles, pieces, scales, static_cast<uint8_t*>(dst));
    return 1;
}

int launch_fp8_block_scales(const ScaleJob* jobs, uint32_t njobs, uint64_t ntiles, uint64_t nblocks, cudaStream_t st) {
    if (!njobs) return 0;
    const uint64_t cap = (uint64_t)device_sm_count() * 8;
    fp8_amax_kernel<<<(int)(ntiles < cap ? ntiles : cap), kScaleThreads, 0, st>>>(jobs, njobs, ntiles);
    const uint64_t ctas = (nblocks + kScaleThreads - 1) / kScaleThreads;
    fp8_finalize_kernel<<<(int)(ctas < cap ? ctas : cap), kScaleThreads, 0, st>>>(jobs, njobs, nblocks);
    return 2;
}

int launch_fp8_finalize(const ScaleJob* jobs, uint32_t njobs, uint64_t nblocks, cudaStream_t st) {
    if (!nblocks) return 0;
    const uint64_t cap = (uint64_t)device_sm_count() * 8, ctas = (nblocks + kScaleThreads - 1) / kScaleThreads;
    fp8_finalize_kernel<<<(int)(ctas < cap ? ctas : cap), kScaleThreads, 0, st>>>(jobs, njobs, nblocks);
    return 1;
}

int launch_fp8_amax_boxes(const QuantTile* tiles, uint64_t ntiles, const void* src, cudaStream_t st) {
    if (!ntiles) return 0;
    const uint64_t cap = (uint64_t)device_sm_count() * kBoxCtasPerSm;
    fp8_amax_boxes_kernel<<<(int)(ntiles < cap ? ntiles : cap), kStageThreads, 0, st>>>(
        tiles, ntiles, static_cast<const uint8_t*>(src));
    return 1;
}

int launch_load_quant_boxes(const QuantTile* tiles, uint64_t ntiles, const RangePiece* pieces, const void* src,
                            cudaStream_t st) {
    if (!ntiles) return 0;
    const uint64_t cap = (uint64_t)device_sm_count() * kBoxCtasPerSm;
    load_quant_boxes_kernel<<<(int)(ntiles < cap ? ntiles : cap), kStageThreads, 0, st>>>(
        tiles, ntiles, pieces, static_cast<const uint8_t*>(src));
    return 1;
}

}  // namespace b200h
