// b200hash_crc32.cu -- CRC-32 (zlib / IEEE 802.3: reflected polynomial 0xEDB88320, initial value and final XOR
// 0xFFFFFFFF) of many device ranges in one launch: the per-record checksums of a torch.save zip archive.
//
//   crc32_chunks_kernel  one persistent CTA per SM (1024 threads); every warp takes an equal run of 16 KiB chunks of
//                        the concatenated ranges and every lane a 512-byte piece of each chunk (slicing-by-4 over
//                        16-byte loads, the tables replicated 32 times in shared memory so that no lookup conflicts);
//                        the lane and chunk results are combined by multiplying with x^(8n) mod P (DESIGN.md 5.11).
//
// CRC-32 is affine over GF(2): with raw(D) the register after D starting from 0,
//   crc(A || B) register = raw(B) ^ raw(A) * x^(8|B|) mod P,
// so any piece of a message can be checksummed on its own and shifted into place afterwards.
#include <cuda_runtime.h>
#include <stdint.h>

#include "b200hash_kernels.cuh"

namespace b200h {
namespace {

constexpr uint32_t kPoly = 0xEDB88320u;
constexpr int kCrcThreads = 1024;
constexpr int kCrcWarps = kCrcThreads / 32;
constexpr uint64_t kPiece = kCrcChunkBytes / 32;  // bytes per lane and chunk
constexpr int kTableWords = 4 * 256 * 32;         // four slicing tables, every entry once per bank
constexpr int kPowTerms = 68;                     // x^(2^k) for k < 68: any x^(8n) with n < 2^64

// a(x) * b(x) mod P(x) in the reflected representation (bit 31 = x^0), as zlib's multmodp; branch-free
__host__ __device__ constexpr uint32_t mulmodp(uint32_t a, uint32_t b) {
    uint32_t p = 0;
    for (int i = 0; i < 32; ++i) {
        p ^= b & (0u - ((a >> (31 - i)) & 1u));
        b = (b >> 1) ^ (kPoly & (0u - (b & 1u)));
    }
    return p;
}

struct PowTable {
    uint32_t v[kPowTerms];  // x^(2^k) mod P
};
constexpr PowTable make_pow_table() {
    PowTable t{};
    t.v[0] = 0x40000000u;  // x^1
    for (int k = 1; k < kPowTerms; ++k) t.v[k] = mulmodp(t.v[k - 1], t.v[k - 1]);
    return t;
}

struct SliceTables {
    uint32_t t[4][256];  // t[0]: the byte table; t[k][b] = t[k-1][b] shifted through one more zero byte
};
constexpr SliceTables make_slice_tables() {
    SliceTables s{};
    for (uint32_t b = 0; b < 256; ++b) {
        uint32_t c = b;
        for (int i = 0; i < 8; ++i) c = (c >> 1) ^ (kPoly & (0u - (c & 1u)));
        s.t[0][b] = c;
    }
    for (int k = 1; k < 4; ++k)
        for (int b = 0; b < 256; ++b) s.t[k][b] = (s.t[k - 1][b] >> 8) ^ s.t[0][s.t[k - 1][b] & 255u];
    return s;
}

constexpr PowTable kPowHost = make_pow_table();
__constant__ PowTable kPowDev = make_pow_table();
__constant__ SliceTables kSliceDev = make_slice_tables();

// x^(8n) mod P
__host__ __device__ inline uint32_t x8nmodp(uint64_t n, const uint32_t* pw) {
    uint32_t p = 0x80000000u;  // x^0
    for (int k = 3; n; n >>= 1, ++k)
        if (n & 1) p = mulmodp(pw[k], p);
    return p;
}

// T points at this lane's replica: entry b of table k is T[(k * 256 + b) * 32]
__device__ __forceinline__ uint32_t crc_byte(uint32_t c, uint32_t byte, const uint32_t* T) {
    return (c >> 8) ^ T[((c ^ byte) & 255u) << 5];
}
__device__ __forceinline__ uint32_t crc_word(uint32_t c, uint32_t w, const uint32_t* T) {
    c ^= w;
    return T[(3 * 256 + (c & 255u)) << 5] ^ T[(2 * 256 + ((c >> 8) & 255u)) << 5] ^ T[(256 + ((c >> 16) & 255u)) << 5] ^
           T[(c >> 24) << 5];
}
__device__ __forceinline__ uint32_t crc_vec(uint32_t c, uint4 v, const uint32_t* T) {
    c = crc_word(c, v.x, T);
    c = crc_word(c, v.y, T);
    c = crc_word(c, v.z, T);
    return crc_word(c, v.w, T);
}

// register c run over p[0..n) (any alignment; 16-byte loads for the aligned middle)
__device__ __forceinline__ uint32_t crc_update(uint32_t c, const uint8_t* p, uint64_t n, const uint32_t* T) {
    while (n && ((uintptr_t)p & 15u)) {
        c = crc_byte(c, *p++, T);
        --n;
    }
    const uint4* v = reinterpret_cast<const uint4*>(p);
    uint64_t nv = n >> 4;
    for (; nv >= 4; nv -= 4, v += 4) {
        const uint4 a = __ldg(v), b = __ldg(v + 1), d = __ldg(v + 2), e = __ldg(v + 3);
        c = crc_vec(c, a, T);
        c = crc_vec(c, b, T);
        c = crc_vec(c, d, T);
        c = crc_vec(c, e, T);
    }
    for (; nv; --nv, ++v) c = crc_vec(c, __ldg(v), T);
    p = reinterpret_cast<const uint8_t*>(v);
    for (n &= 15; n; --n) c = crc_byte(c, *p++, T);
    return c;
}

// Chunks are cut from the END of every range (so only a range's first chunk may be short) and numbered range-major:
// range r owns chunks [first[r], first[r + 1]).  Warp w of the grid takes chunks [G w / W, G (w + 1) / W).  Within a
// chunk, lane l takes the l-th of its 32 pieces of kPiece bytes, also cut from the chunk's end, and keeps one register
// across the warp's chunks of a range (Horner: the next piece of the same lane starts kCrcChunkBytes - kPiece bytes
// after this one ends).  When the warp leaves a range, every lane shifts its register by the bytes behind its piece in
// the chunk, the warp XORs them, lane 0 shifts that by the bytes behind the chunk in the range and XORs it into out[r],
// which the host initialised with the range's length term (the 0xFFFFFFFF start register shifted through L bytes,
// XORed with 0xFFFFFFFF).
__global__ void __launch_bounds__(kCrcThreads, 1)
    crc32_chunks_kernel(const CrcRange* __restrict__ ranges, const uint64_t* __restrict__ first, uint64_t n,
                        uint64_t nchunks, uint32_t* __restrict__ out) {
    extern __shared__ uint32_t s_tab[];  // [4][256][32]
    __shared__ uint32_t s_lane_shift[32];
    for (int i = threadIdx.x; i < kTableWords; i += kCrcThreads) s_tab[i] = (&kSliceDev.t[0][0])[i >> 5];
    if (threadIdx.x < 32) s_lane_shift[threadIdx.x] = x8nmodp((31 - threadIdx.x) * kPiece, kPowDev.v);
    __syncthreads();

    const int lane = threadIdx.x & 31;
    const uint32_t* T = s_tab + lane;
    const uint64_t nw = (uint64_t)gridDim.x * kCrcWarps, w = (uint64_t)blockIdx.x * kCrcWarps + (threadIdx.x >> 5);
    uint64_t g = nchunks * w / nw;
    const uint64_t g_end = nchunks * (w + 1) / nw;
    if (g >= g_end) return;
    // the range that holds chunk g: the last r with first[r] <= g (empty ranges own no chunk)
    uint64_t lo = 0, hi = n - 1;
    while (lo < hi) {
        const uint64_t mid = (lo + hi + 1) >> 1;
        if (first[mid] <= g) lo = mid;
        else hi = mid - 1;
    }
    uint64_t r = lo, r_end = first[r + 1];
    const uint8_t* base = reinterpret_cast<const uint8_t*>(ranges[r].ptr);
    uint64_t len = ranges[r].len;
    const uint32_t step = x8nmodp(kCrcChunkBytes - kPiece, kPowDev.v);
    uint32_t acc = 0;
    while (true) {
        const uint64_t q = r_end - 1 - g;  // chunks behind this one in the range
        const int64_t piece_end = (int64_t)(len - q * kCrcChunkBytes) - (int64_t)((31 - lane) * kPiece);
        const int64_t piece_start = piece_end - (int64_t)kPiece > 0 ? piece_end - (int64_t)kPiece : 0;
        acc = mulmodp(acc, step);
        if (piece_end > 0) acc = crc_update(acc, base + piece_start, (uint64_t)(piece_end - piece_start), T);
        ++g;
        if (g == g_end || g == r_end) {
            uint32_t v = mulmodp(acc, s_lane_shift[lane]);
#pragma unroll
            for (int o = 16; o; o >>= 1) v ^= __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0) {
                if (q) v = mulmodp(v, x8nmodp(q * kCrcChunkBytes, kPowDev.v));
                atomicXor(out + r, v);
            }
            if (g == g_end) break;
            acc = 0;
            do {
                r_end = first[++r + 1];
            } while (r_end <= g);
            base = reinterpret_cast<const uint8_t*>(ranges[r].ptr);
            len = ranges[r].len;
        }
    }
}

}  // namespace

uint32_t crc32_length_term(uint64_t len) { return mulmodp(x8nmodp(len, kPowHost.v), 0xFFFFFFFFu) ^ 0xFFFFFFFFu; }

int launch_crc32(const CrcRange* ranges, const uint64_t* first, uint64_t n, uint64_t nchunks, uint32_t* out,
                 cudaStream_t st) {
    if (!nchunks) return 0;
    const size_t smem = kTableWords * sizeof(uint32_t);
    cudaFuncSetAttribute(crc32_chunks_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const uint64_t want = (nchunks + kCrcWarps - 1) / kCrcWarps;
    const int grid = (int)(want < (uint64_t)device_sm_count() ? want : (uint64_t)device_sm_count());
    crc32_chunks_kernel<<<grid, kCrcThreads, smem, st>>>(ranges, first, n, nchunks, out);
    return 1;
}

}  // namespace b200h
