// tools/chainbench.cu -- what can ONE warp do for ONE chain?  Cycles per 64-byte block of a lone warp running
//   (a) SHA-256 rounds only, W+K rows read from shared memory (the schedule expanded elsewhere),
//   (b) full SHA-256 (schedule + rounds), (c) MD5, (d) fused SHA-256 + MD5 (the lane kernel's compress<>),
// message words read from shared memory.  One CTA, NW warps (one per SMSP when NW <= 4).
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tools/chainbench tools/chainbench.cu
#include <cstdio>
#include "../modal_client_b200/csrc/b200hash_kernels.cu"

namespace b200h {

// round variants for the lone-warp chain: fewer instructions matter more than pipe placement at 0.5 instr/clk
#define CH_RND_FMA(a, b, c, d, e, f, g, h, WK)                                                        \
    {                                                                                                 \
        const uint32_t t1 = addf(addf(addf(h, WK, one), lop3<0xCA>(e, f, g), one), SHA_S1(e), one);   \
        const uint32_t t2 = addf(SHA_S0(a), lop3<0xE8>(a, b, c), one);                                \
        d = addf(d, t1, one);                                                                         \
        h = addf(t1, t2, one);                                                                        \
    }
#define CH_RND_PLAIN(a, b, c, d, e, f, g, h, WK)                                      \
    {                                                                                 \
        const uint32_t t1 = h + WK + lop3<0xCA>(e, f, g) + SHA_S1(e);                 \
        d += t1;                                                                      \
        h = t1 + SHA_S0(a) + lop3<0xE8>(a, b, c);                                     \
    }
#define CH_RND_DPRE(a, b, c, d, e, f, g, h, WK)                                       \
    {                                                                                 \
        const uint32_t hwk = addf(h, WK, one);                                        \
        const uint32_t dh = addf(d, hwk, one);                                        \
        const uint32_t cs = lop3<0xCA>(e, f, g) + SHA_S1(e);                          \
        d = addf(dh, cs, one);                                                        \
        h = hwk + cs + SHA_S0(a) + lop3<0xE8>(a, b, c);                               \
    }

// MD5 block for the lone-warp chain, step written so that ptxas fuses rotate+add into LEA.HI (VAR 1) or with the
// shipped MD5_STEP_MIX form (VAR 0): latency, not instruction count, bounds this chain.
template <int VAR>
__device__ __forceinline__ void md5_block_xt(uint32_t (&hm)[4], const uint32_t (&xt)[64], uint32_t one) {
    // xt[i] = M[g(i)] + T[i] prepared by another warp (like W+K for SHA-256)
    constexpr int S[4][4] = {{7, 12, 17, 22}, {5, 9, 14, 20}, {4, 11, 16, 23}, {6, 10, 15, 21}};
    uint32_t v[4] = {hm[0], hm[1], hm[2], hm[3]};  // a b c d
#pragma unroll
    for (int i = 0; i < 64; ++i) {
        const int r = i >> 4;
        // roles rotate: step i updates v[(4 - i) & 3] using the other three in order
        uint32_t& a = v[(64 - i) & 3];
        const uint32_t b = v[(65 - i) & 3], c = v[(66 - i) & 3], d = v[(67 - i) & 3];
        const uint32_t fn = r == 0 ? lop3<0xCA>(b, c, d) : r == 1 ? lop3<0xE4>(b, c, d) : r == 2 ? lop3<0x96>(b, c, d) : lop3<0x39>(b, c, d);
        if (VAR == 1) {
            a = b + rotl(a + fn + xt[i], S[r][i & 3]);                    // IADD3 + LEA.HI
        } else {
            a = addf(b, rotl(a + fn + xt[i], S[r][i & 3]), one);          // IADD3 + SHF + IMAD
        }
    }
    hm[0] += v[0]; hm[1] += v[1]; hm[2] += v[2]; hm[3] += v[3];
}

template <int MODE>
__global__ void __launch_bounds__(128) chain_bench(uint32_t* out, long long* cyc, int nblocks, uint32_t one, uint32_t seed) {
    __shared__ __align__(16) uint32_t rows[32][68];  // 32 blocks of 64 W+K words (or 16 message words), padded
    for (int i = threadIdx.x; i < 32 * 68; i += blockDim.x) (&rows[0][0])[i] = seed * 2654435761u + i * 40503u;
    __syncthreads();
    uint32_t hs[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
    uint32_t hm[4] = {0x67452301u, 0xefcdab89u, 0x98badcfeu, 0x10325476u};
    const long long t0 = clock64();
#pragma unroll 1
    for (int b = 0; b < nblocks; ++b) {
        const uint4* row = reinterpret_cast<const uint4*>(rows[b & 31]);
        if (MODE == 7 || MODE == 8) {
            uint32_t xt[64];
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const uint4 v = row[i];
                xt[4 * i] = v.x; xt[4 * i + 1] = v.y; xt[4 * i + 2] = v.z; xt[4 * i + 3] = v.w;
            }
            md5_block_xt<MODE == 7 ? 1 : 0>(hm, xt, one);
        } else if (MODE == 0 || (MODE >= 4 && MODE <= 6)) {
            uint32_t k[64];
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const uint4 v = row[i];
                k[4 * i] = v.x; k[4 * i + 1] = v.y; k[4 * i + 2] = v.z; k[4 * i + 3] = v.w;
            }
            uint32_t a = hs[0], bb = hs[1], c = hs[2], d = hs[3], e = hs[4], f = hs[5], g = hs[6], h = hs[7];
#define R8(RND)                                                                              \
    _Pragma("unroll") for (int i = 0; i < 64; i += 8) {                                      \
        RND(a, bb, c, d, e, f, g, h, k[i]);     RND(h, a, bb, c, d, e, f, g, k[i + 1]);      \
        RND(g, h, a, bb, c, d, e, f, k[i + 2]); RND(f, g, h, a, bb, c, d, e, k[i + 3]);      \
        RND(e, f, g, h, a, bb, c, d, k[i + 4]); RND(d, e, f, g, h, a, bb, c, k[i + 5]);      \
        RND(c, d, e, f, g, h, a, bb, k[i + 6]); RND(bb, c, d, e, f, g, h, a, k[i + 7]);      \
    }
            if (MODE == 0) { R8(CH_RND_FMA) }
            if (MODE == 4) { R8(CH_RND) }
            if (MODE == 5) { R8(CH_RND_PLAIN) }
            if (MODE == 6) { R8(CH_RND_DPRE) }
            hs[0] += a; hs[1] += bb; hs[2] += c; hs[3] += d; hs[4] += e; hs[5] += f; hs[6] += g; hs[7] += h;
        } else {
            uint32_t x[16];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const uint4 v = row[i];
                x[4 * i] = v.x; x[4 * i + 1] = v.y; x[4 * i + 2] = v.z; x[4 * i + 3] = v.w;
            }
            if (MODE == 9) md5_chain_block(hm, x, one);
            if (MODE == 1) compress<true, false>(hs, hm, x, false, 0u, 0u, one);
            if (MODE == 2) compress<false, true>(hs, hm, x, false, 0u, 0u, one);
            if (MODE == 3) compress<true, true>(hs, hm, x, false, 0u, 0u, one);
            if (MODE == 10) compress<true, true, true>(hs, hm, x, false, 0u, 0u, one);
            if (MODE == 11) compress<true, false, true>(hs, hm, x, false, 0u, 0u, one);
        }
    }
    const long long t1 = clock64();
    uint32_t s = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) s ^= hs[i];
#pragma unroll
    for (int i = 0; i < 4; ++i) s ^= hm[i];
    out[threadIdx.x] = s;
    if (threadIdx.x == 0) *cyc = t1 - t0;
}

}  // namespace b200h

template <int MODE>
static void run(const char* name, int warps) {
    uint32_t* out;
    long long* cyc;
    cudaMalloc(&out, 4096);
    cudaMalloc(&cyc, 8);
    const int nb = 4096;
    for (int rep = 0; rep < 2; ++rep) b200h::chain_bench<MODE><<<1, 32 * warps>>>(out, cyc, nb, 1u, 7u);
    cudaDeviceSynchronize();
    long long c = 0;
    cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
    cudaError_t e = cudaGetLastError();
    const double cpb = (double)c / nb;
    int khz = 0;  // the SM clock the cycle count is converted at (the device's maximum)
    cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
    printf("%-34s warps=%d  %8.1f cycles/block  -> %6.1f MB/s per chain at %.3f GHz  (%s)\n", name, warps, cpb,
           64.0 * (khz / 1e3) / cpb, khz / 1e6, cudaGetErrorString(e));
    cudaFree(out);
    cudaFree(cyc);
}

int main() {
    run<4>("rounds only (shipped: 2 IADD3)", 1);
    run<5>("rounds only, plain C adds", 1);
    run<6>("rounds only, d pre-added", 1);
    run<7>("MD5 from M+T rows, IADD3 + LEA.HI", 1);
    run<8>("MD5 from M+T rows, IADD3 + SHF + IMAD", 1);
    run<9>("MD5 md5_chain_block (shipped)", 1);
    run<10>("fused, sparse instantiation (plain adds)", 1);
    run<11>("SHA-256 full, sparse instantiation", 1);
    for (int w : {1, 4}) {
        run<0>("rounds only, all adds IMAD", w);
        run<1>("SHA-256 full (schedule + rounds)", w);
        run<2>("MD5", w);
        run<3>("fused SHA-256 + MD5", w);
    }
    return 0;
}
