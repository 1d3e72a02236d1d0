// b200hash_stage.cu -- copy byte ranges of segmented device files to one destination buffer with full-width stores:
// the blocks of a checkpoint in HBM that a volume server reports missing, on their way to page-locked host memory.
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
__device__ __forceinline__ uint32_t find_piece(const StagePiece* __restrict__ pc, uint32_t lo, uint32_t n, uint64_t d) {
    uint32_t hi = n - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (pc[mid].dst <= d) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(kStageThreads, kStageCtasPerSm)
    stage_ranges_kernel(const StageTile* __restrict__ tiles, uint64_t ntiles, const StagePiece* __restrict__ pieces,
                        uint8_t* __restrict__ dst) {
    for (uint64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const StageTile tile = tiles[t];
        const StagePiece* __restrict__ pc = pieces + tile.first_piece;
        uint8_t* out = dst + tile.dst;
        const uint32_t words = tile.len >> 4, tail = tile.len & 15u;
        if (tile.npieces == 1) {
            // the whole tile comes from one segment: one phase, no lookups
            const uint8_t* src = reinterpret_cast<const uint8_t*>(pc->src) + (tile.dst - pc->dst);
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
            const uint64_t d = tile.dst + (uint64_t)w * 16;
            if (d >= pc[cur].dst + pc[cur].len) cur = find_piece(pc, cur + 1, tile.npieces, d);
            const uint64_t in = d - pc[cur].dst, left = pc[cur].len - in;
            uint4 v;
            if (left >= 16) {
                v = load_word(reinterpret_cast<const uint8_t*>(pc[cur].src) + in);
            } else {
                uint32_t r[4] = {0, 0, 0, 0};
                uint32_t i = cur;
                uint64_t end = pc[i].dst + pc[i].len;
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    while (d + j >= end) {
                        ++i;
                        end = pc[i].dst + pc[i].len;
                    }
                    r[j >> 2] |= (uint32_t)reinterpret_cast<const uint8_t*>(pc[i].src)[d + j - pc[i].dst] << (8 * (j & 3));
                }
                v = make_uint4(r[0], r[1], r[2], r[3]);
            }
            *reinterpret_cast<uint4*>(dst + d) = v;
        }
        if (threadIdx.x < tail) {
            const uint64_t d = tile.dst + (uint64_t)words * 16 + threadIdx.x;
            const uint32_t i = find_piece(pc, 0, tile.npieces, d);
            dst[d] = reinterpret_cast<const uint8_t*>(pc[i].src)[d - pc[i].dst];
        }
    }
}

}  // namespace

int launch_stage_ranges(const StageTile* tiles, uint64_t ntiles, const StagePiece* pieces, void* dst, cudaStream_t st) {
    if (!ntiles) return 0;
    const uint64_t cap = (uint64_t)device_sm_count() * kStageCtasPerSm;
    stage_ranges_kernel<<<(int)(ntiles < cap ? ntiles : cap), kStageThreads, 0, st>>>(tiles, ntiles, pieces,
                                                                                      static_cast<uint8_t*>(dst));
    return 1;
}

}  // namespace b200h
