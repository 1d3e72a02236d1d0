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
//                        gather_segments_kernel does between HBM buffers, would degrade to byte stores here.
//
// A range is cut by the host into pieces (range intersected with one segment, never empty), listed in destination
// order; a tile names the slice of the piece list it draws from.
//   * a destination word that lies inside one piece is built from the two aligned 16-byte source words around it and a
//     byte shift by (source address & 15): one load when the phases agree, two otherwise;
//   * a word that crosses pieces is assembled byte by byte and still stored as one word;
//   * only the bytes behind a range's last whole word are stored singly (the destination beyond the range is not the
//     kernel's to write).
// Loads never leave the 16-byte aligned hull of a piece: the aligned words that hold a piece's first and last byte.
// Those words lie in the same allocation granule as the bytes themselves (device allocations are at least 256-byte
// aligned and sized in multiples of that), which the lane kernel's misaligned-start reads rely on as well.
#include <cuda_runtime.h>
#include <stdint.h>

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
__device__ __forceinline__ uint32_t find_piece(const RangePiece* __restrict__ pc, uint32_t lo, uint32_t n, uint64_t d) {
    uint32_t hi = n - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (pc[mid].host <= d) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(kStageThreads, kStageCtasPerSm)
    stage_ranges_kernel(const RangeTile* __restrict__ tiles, uint64_t ntiles, const RangePiece* __restrict__ pieces,
                        uint8_t* __restrict__ dst) {
    for (uint64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const RangeTile tile = tiles[t];
        const RangePiece* __restrict__ pc = pieces + tile.first_piece;
        uint8_t* out = dst + tile.host;
        const uint32_t words = tile.len >> 4, tail = tile.len & 15u;
        if (tile.npieces == 1) {
            // the whole tile comes from one segment: one phase, no lookups
            const uint8_t* src = reinterpret_cast<const uint8_t*>(pc->dev) + (tile.host - pc->host);
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
            continue;
        }
        uint32_t cur = 0;
        for (uint32_t w = threadIdx.x; w < words; w += kStageThreads) {
            const uint64_t d = tile.host + (uint64_t)w * 16;
            if (d >= pc[cur].host + pc[cur].len) cur = find_piece(pc, cur + 1, tile.npieces, d);
            const uint64_t in = d - pc[cur].host, left = pc[cur].len - in;
            uint4 v;
            if (left >= 16) {
                v = load_word(reinterpret_cast<const uint8_t*>(pc[cur].dev) + in);
            } else {
                uint32_t r[4] = {0, 0, 0, 0};
                uint32_t i = cur;
                uint64_t end = pc[i].host + pc[i].len;
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    while (d + j >= end) {
                        ++i;
                        end = pc[i].host + pc[i].len;
                    }
                    r[j >> 2] |= (uint32_t)reinterpret_cast<const uint8_t*>(pc[i].dev)[d + j - pc[i].host] << (8 * (j & 3));
                }
                v = make_uint4(r[0], r[1], r[2], r[3]);
            }
            *reinterpret_cast<uint4*>(dst + d) = v;
        }
        if (threadIdx.x < tail) {
            const uint64_t d = tile.host + (uint64_t)words * 16 + threadIdx.x;
            const uint32_t i = find_piece(pc, 0, tile.npieces, d);
            dst[d] = reinterpret_cast<const uint8_t*>(pc[i].dev)[d - pc[i].host];
        }
    }
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

}  // namespace

int launch_load_ranges(const RangeTile* tiles, uint64_t ntiles, const RangePiece* pieces, const void* src, cudaStream_t st) {
    if (!ntiles) return 0;
    const uint64_t per_cta = kStageThreads / 32, ctas = (ntiles + per_cta - 1) / per_cta;
    const uint64_t cap = (uint64_t)device_sm_count() * kStageCtasPerSm;
    load_ranges_kernel<<<(int)(ctas < cap ? ctas : cap), kStageThreads, 0, st>>>(tiles, ntiles, pieces,
                                                                                static_cast<const uint8_t*>(src));
    return 1;
}

int launch_stage_ranges(const RangeTile* tiles, uint64_t ntiles, const RangePiece* pieces, void* dst, cudaStream_t st) {
    if (!ntiles) return 0;
    const uint64_t cap = (uint64_t)device_sm_count() * kStageCtasPerSm;
    stage_ranges_kernel<<<(int)(ntiles < cap ? ntiles : cap), kStageThreads, 0, st>>>(tiles, ntiles, pieces,
                                                                                      static_cast<uint8_t*>(dst));
    return 1;
}

}  // namespace b200h
