// b200hash_dedupe.cu -- first-occurrence index of every row of a digest table (the step right after the hash path).
//
// The reference dedupes content-addressed uploads with a Python set / dict keyed by the hex digest, one file at
// a time on the event loop (py/modal/mount.py:498,518-534 `accounted_hashes`; the volumefs1 uploader relies on
// the server for it, py/modal/volume.py:1288-1333).  Here the digest table is already in HBM, so the same
// answer -- first[i] = min{ j : key_j == key_i } -- is computed there for the whole batch.
//
//   dedupe_insert_kernel   one thread per row; open-addressing table (linear probing, power-of-two capacity
//                          >= 2n) keyed by the first 8 bytes of the digest (already uniformly distributed; a
//                          splitmix finaliser is applied anyway so that any fixed-width keys work).  A slot is
//                          claimed with atomicCAS on `rep` (the row that owns it); later rows compare their FULL
//                          key against the owner's key bytes (exact, not probabilistic) and atomicMin their
//                          index into `mn`.  The row's slot is left in first[i].
//   dedupe_resolve_kernel  first[i] = mn[slot_i]; rows with first[i] == i are counted (warp-aggregated).
//
// Both kernels are bound by random 32-byte sector accesses to L2/HBM (the table for n <= ~8M rows is L2 resident):
// algorithmic traffic = n * key_bytes read + 4n written.
#include "b200hash_kernels.cuh"

#include <algorithm>

namespace b200h {

namespace {

constexpr uint32_t kEmptySlot = 0xffffffffu;

__device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x ^= x >> 30;
    x *= 0xbf58476d1ce4e5b9ull;
    x ^= x >> 27;
    x *= 0x94d049bb133111ebull;
    x ^= x >> 31;
    return x;
}

// KW = key width in 32-bit words (8 for SHA-256 rows, 4 for MD5 rows); rows are 4-byte aligned.
template <int KW>
__device__ __forceinline__ bool same_key(const uint32_t* __restrict__ a, const uint32_t (&k)[KW]) {
    uint32_t diff = 0;
#pragma unroll
    for (int w = 0; w < KW; ++w) diff |= __ldg(a + w) ^ k[w];
    return diff == 0;
}

template <int KW>
__global__ void __launch_bounds__(256)
dedupe_insert_kernel(const uint32_t* __restrict__ keys, uint32_t n, uint32_t* __restrict__ rep,
                     uint32_t* __restrict__ mn, uint32_t mask, uint32_t* __restrict__ first) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        uint32_t k[KW];
        const uint32_t* row = keys + (size_t)i * KW;
#pragma unroll
        for (int w = 0; w < KW; ++w) k[w] = __ldg(row + w);
        uint32_t h = (uint32_t)mix64(((uint64_t)k[1] << 32) | k[0]) & mask;
        for (;;) {
            uint32_t r = rep[h];
            if (r == kEmptySlot) r = atomicCAS(&rep[h], kEmptySlot, i);
            if (r == kEmptySlot || r == i || same_key<KW>(keys + (size_t)r * KW, k)) {
                atomicMin(&mn[h], i);
                first[i] = h;
                break;
            }
            h = (h + 1) & mask;
        }
    }
}

__global__ void __launch_bounds__(256)
dedupe_resolve_kernel(uint32_t n, const uint32_t* __restrict__ mn, uint32_t* __restrict__ first,
                      unsigned long long* __restrict__ ndistinct) {
    for (uint32_t base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {
        const uint32_t i = base + threadIdx.x;
        bool is_first = false;
        if (i < n) {
            const uint32_t f = mn[first[i]];
            first[i] = f;
            is_first = f == i;
        }
        const uint32_t m = __ballot_sync(0xffffffffu, is_first);
        if (ndistinct && (threadIdx.x & 31) == 0 && m) atomicAdd(ndistinct, (unsigned long long)__popc(m));
    }
}

}  // namespace

uint32_t dedupe_table_capacity(uint64_t n) {
    uint64_t c = 1024;
    while (c < 2 * n) c <<= 1;
    return (uint32_t)c;
}

// table: 2 * dedupe_table_capacity(n) uint32 words (rep | mn); d_first: n words; d_ndistinct may be null.
int launch_dedupe(const void* d_keys, uint64_t n, uint32_t key_bytes, uint32_t* table, uint32_t* d_first,
                  unsigned long long* d_ndistinct, cudaStream_t st) {
    const uint32_t cap = dedupe_table_capacity(n);
    cudaMemsetAsync(table, 0xff, (size_t)cap * 2 * sizeof(uint32_t), st);
    if (d_ndistinct) cudaMemsetAsync(d_ndistinct, 0, sizeof(unsigned long long), st);
    if (n == 0) return 0;
    const int threads = 256;
    const int blocks = (int)std::min<uint64_t>((n + threads - 1) / threads, (uint64_t)device_sm_count() * 8);
    const uint32_t* k = static_cast<const uint32_t*>(d_keys);
    if (key_bytes == 32)
        dedupe_insert_kernel<8><<<blocks, threads, 0, st>>>(k, (uint32_t)n, table, table + cap, cap - 1, d_first);
    else
        dedupe_insert_kernel<4><<<blocks, threads, 0, st>>>(k, (uint32_t)n, table, table + cap, cap - 1, d_first);
    dedupe_resolve_kernel<<<blocks, threads, 0, st>>>((uint32_t)n, table + cap, d_first, d_ndistinct);
    return 2;
}

}  // namespace b200h
