// b200hash_kernels.cu -- hand-written sm_90a (H100) kernels for the blob-ingest / content-hash path.
//
// Replaces the hashlib calls of the reference (py/modal/_utils/hash_utils.py:14-101,
// blob_utils.py:640-705 and :216-219, bytes_io_segment_payload.py:58,102) with batched device
// kernels.  See DESIGN.md for the data layout and the roofline of each kernel.
//
//   lane_hash_kernel   one message per lane; fused SHA-256 + MD5 over a single read of the bytes.
//                      Persistent warps pull messages from a device-side work queue and time-slice them
//                      (32-block quanta) so n messages share the resident lanes evenly.  Each lane gathers
//                      its own 128-byte chunks with cp.async (LDGSTS) into a private, conflict-free
//                      shared-memory slot, double buffered, and runs both compression functions interleaved
//                      in registers.  Bound: INT32 issue (ALU pipe for SHF/LOP3/PRMT, FMA pipe for the adds).
//   chain_hash_kernel  outlier path: CTA per long message, TMA bulk tiles (UBLKCP) + mbarrier ring, 32-lane
//                      schedule expansion, SHA-256 rounds and MD5 on separate warps: one chain at the one-warp
//                      issue limit (0.5 instr/clk over 1 056 instead of 2 108 instructions per block), ~2x a lane.
//   trim_kernel        warp per message reverse scan for the last non-zero byte (HBM bound).
//   plan kernels       bucket messages by block count (longest first) straight into the work queue.
//   fill_synth_kernel  counter-based synthetic bytes (bench/test data; same stream as synth.py).
#include "b200hash_kernels.cuh"

#include <cstdlib>

namespace b200h {

// ---------------------------------------------------------------------------------- PTX helpers

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
// 1-D TMA bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP).
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
// Ampere-style per-thread async copy (SASS: LDGSTS): 16 bytes global -> shared, L1 bypassed.
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

template <int IMM>
__device__ __forceinline__ uint32_t lop3(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t d;
    asm("lop3.b32 %0, %1, %2, %3, %4;" : "=r"(d) : "r"(a), "r"(b), "r"(c), "n"(IMM));
    return d;
}
// a + b issued as IMAD (a * one + b) so that the add runs on the FMA pipe instead of the ALU pipe, which
// SHF/LOP3/PRMT already saturate.  `one` is a kernel argument (== 1) so ptxas cannot fold the multiply.
__device__ __forceinline__ uint32_t addf(uint32_t a, uint32_t b, uint32_t one) {
    uint32_t d;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(one), "r"(b));
    return d;
}
// acc + rotl(u, k) as one plain add of a funnel shift: ptxas fuses the two into a single ALU-pipe LEA.HI
// (acc + ((u:u) << k) >> 32), so the add leaves the FMA pipe without a rotate being added to the ALU pipe.
template <int K>
__device__ __forceinline__ uint32_t add_rotl(uint32_t acc, uint32_t u) {
    return acc + __funnelshift_l(u, u, K);
}
__device__ __forceinline__ uint32_t rotr(uint32_t x, int n) { return __funnelshift_r(x, x, n); }
__device__ __forceinline__ uint32_t rotl(uint32_t x, int n) { return __funnelshift_l(x, x, n); }
__device__ __forceinline__ uint32_t bswap(uint32_t x) { return __byte_perm(x, 0, 0x0123); }

// ---------------------------------------------------------------------- compression functions
// SHA-256: FIPS 180-4 section 6.2.2; MD5: RFC 1321 section 3.4.  Boolean functions are single LOP3s:
//   Ch(e,f,g)=e?f:g (0xCA)  Maj (0xE8)  xor3 (0x96)  MD5 F=b?c:d (0xCA)  G=d?b:c (0xE4)  H=b^c^d (0x96)  I=c^(b|~d) (0x39)

#define SHA_S0(x) lop3<0x96>(rotr(x, 2), rotr(x, 13), rotr(x, 22))
#define SHA_S1(x) lop3<0x96>(rotr(x, 6), rotr(x, 11), rotr(x, 25))
#define SHA_s0(x) lop3<0x96>(rotr(x, 7), rotr(x, 18), (x) >> 3)
#define SHA_s1(x) lop3<0x96>(rotr(x, 17), rotr(x, 19), (x) >> 10)
constexpr int kMd5F = 0xCA, kMd5G = 0xE4, kMd5H = 0x96, kMd5I = 0x39;

// lop3<IMM>(a, b, c) issued with its operands in the order (b, c, a), the truth table permuted to match
__host__ __device__ constexpr int lut_bca(int imm) {
    int lut = 0;
    for (int j = 0; j < 8; ++j) lut |= ((imm >> (((j & 1) << 2) | (j >> 1))) & 1) << j;
    return lut;
}
static_assert(lut_bca(0xCA) == 0xE4 && lut_bca(0xE8) == 0xE8 && lut_bca(0x96) == 0x96, "lop3 operand order");
template <int IMM>
__device__ __forceinline__ uint32_t lop3_bca(uint32_t a, uint32_t b, uint32_t c) {
    return lop3<lut_bca(IMM)>(b, c, a);
}
__device__ __forceinline__ void rotw(uint32_t x, uint32_t mul, uint32_t& lo, uint32_t& hi) {
    uint64_t d;
    asm("mul.wide.u32 %0, %1, %2;" : "=l"(d) : "r"(x), "r"(mul));
    lo = (uint32_t)d;
    hi = (uint32_t)(d >> 32);
}

// The forms of the lane kernel's compression body, one per kind of batch; compress<> picks one per instantiation.
// Dense batches put many warps on every SMSP, and the ALU pipe, which SHF/LOP3/PRMT already load, sets the pace: their
// adds run as IMAD on the FMA pipe (addf).  Sparse batches (<= 4 warps per SM) leave every warp alone on its SMSP, where
// it issues one instruction per two cycles whatever the pipe: their adds are plain C, which ptxas fuses into IADD3 / LEA
// (~15 % fewer instructions per block).
enum class Body {
    kDenseFused,  // SHA-256 + MD5, dense
    kDenseSha,    // SHA-256 alone, dense
    kMd5,         // MD5 alone, dense or not
    kSparse,      // SHA-256 + MD5 or SHA-256 alone, sparse
};

// One SHA-256 round on rotating register names: d += T1, h = T1 + T2.
template <Body B>
__device__ __forceinline__ void sha_round(uint32_t a, uint32_t b, uint32_t c, uint32_t& d, uint32_t e, uint32_t f,
                                          uint32_t g, uint32_t& h, uint32_t K, uint32_t W, uint32_t one) {
    if constexpr (B == Body::kDenseFused) {
        // This kernel issues at the rate its vector register reads allow, well under both pipes' rates, so fewer
        // instructions win (DESIGN.md 5.1).  Factored out, the outer rotate of Sigma1 / Sigma0 ends in an add --
        // Sigma1(e) = rotr6(e ^ rotr5 e ^ rotr19 e) goes into T1, Sigma0(a) = rotr2(a ^ rotr11 a ^ rotr20 a) onto Maj --
        // and each such pair is one LEA.HI (add_rotl) in place of SHF + IMAD: 1 instruction less, ALU pipe unchanged.
        // Multiplies do not pay here: IMAD.HI issues at half the rate of IMAD or SHF on H100 (tools/ubench.cu).
        // W + K is a plain add, which ptxas issues as VIADD R, R, imm.  Any IMAD with an immediate addend makes ptxas keep
        // `one` in a vector register for every addf, so each of the other 528 adds of a block would read three vector
        // registers; this way they read `one` from a uniform register (IMAD R, R, UR, R).  VIADD stays off the ALU pipe:
        // it issues next to SHF and LOP3 above that pipe's rate (tools/ubench.cu).
        // Every LOP3 of SHA-256 (here and in sha_sched) takes its operands in the order (b, c, a).  With 3 CTAs per SM
        // and the MD5 steps ahead of the SHA-256 rounds (compress), that made the lane kernel 3.1 % faster than order
        // (a, b, c) at 4 CTAs, H100 at 700 W (tools/lane_sass_score.py, DESIGN.md 5.1, 6).
        uint32_t t1 = addf(addf(h, W + K, one), lop3_bca<0xCA>(e, f, g), one);
        t1 = add_rotl<26>(t1, lop3_bca<0x96>(e, rotr(e, 5), rotr(e, 19)));
        const uint32_t t2 = add_rotl<30>(lop3_bca<0xE8>(a, b, c), lop3_bca<0x96>(a, rotr(a, 11), rotr(a, 20)));
        d = addf(d, t1, one);
        h = addf(t1, t2, one);
    } else if constexpr (B == Body::kDenseSha) {
        // Without MD5 the ALU pipe carries 1040 of the 1640 instructions per block while the FMA pipe idles, so the
        // outer rotate of Sigma1 / Sigma0 is a widening multiply x * 2^(32-n) -> {x << (32-n), x >> n}; the halves have
        // disjoint bits, so both are simply added into the round sum (one SHF less, one IMAD.WIDE + one IMAD more).
        uint32_t t1 = addf(addf(h, addf(W, K, one), one), lop3<0xCA>(e, f, g), one);
        uint32_t lo, hi;
        rotw(lop3<0x96>(e, rotr(e, 5), rotr(e, 19)), 1u << 26, lo, hi);
        t1 = addf(addf(t1, lo, one), hi, one);
        rotw(lop3<0x96>(a, rotr(a, 11), rotr(a, 20)), 1u << 30, lo, hi);
        const uint32_t t2 = addf(addf(lo, hi, one), lop3<0xE8>(a, b, c), one);
        d = addf(d, t1, one);
        h = addf(t1, t2, one);
    } else {
        static_assert(B == Body::kSparse, "no SHA-256 round in this body");
        const uint32_t t1 = h + (W + K) + lop3<0xCA>(e, f, g) + SHA_S1(e);
        const uint32_t t2 = SHA_S0(a) + lop3<0xE8>(a, b, c);
        d = d + t1;
        h = t1 + t2;
    }
}

// Message schedule in place: w[i & 15] becomes W[i] for i >= 16, with the adds and LOP3 operand order of sha_round.
// W[i-16], W[i-7], W[i-15], W[i-2] are read in the order they are added: another order changes the SASS ptxas emits.
template <Body B>
__device__ __forceinline__ void sha_sched(uint32_t (&w)[16], int i, uint32_t one) {
    const uint32_t w16 = w[i & 15], w7 = w[(i - 7) & 15], w15 = w[(i - 15) & 15], w2 = w[(i - 2) & 15];
    if constexpr (B == Body::kDenseFused)
        w[i & 15] = addf(addf(addf(w16, w7, one), lop3_bca<0x96>(rotr(w15, 7), rotr(w15, 18), w15 >> 3), one),
                         lop3_bca<0x96>(rotr(w2, 17), rotr(w2, 19), w2 >> 10), one);
    else if constexpr (B == Body::kDenseSha)
        w[i & 15] = addf(addf(addf(w16, w7, one), SHA_s0(w15), one), SHA_s1(w2), one);
    else
        w[i & 15] = w16 + w7 + SHA_s0(w15) + SHA_s1(w2);
}

// One MD5 step: a = b + rotl(a + FN(b, c, d) + x[k] + T, S).
template <Body B, int FN, int S>
__device__ __forceinline__ void md5_step(uint32_t& a, uint32_t b, uint32_t c, uint32_t d, uint32_t xk, uint32_t T,
                                         uint32_t one) {
    if constexpr (B == Body::kDenseFused) {
        // as in sha_round: the last add fused with the rotate into one LEA.HI (64 per block), x + T a VIADD
        const uint32_t t = addf(addf(a, xk + T, one), lop3<FN>(b, c, d), one);
        a = add_rotl<S>(b, t);
    } else if constexpr (B == Body::kMd5) {
        // MD5 alone: the FMA pipe is the bottleneck (4 IMAD vs 2 ALU ops per step), so the 3-input sum goes back to
        // the ALU pipe as one IADD3: per step ALU = LOP3 + IADD3 + SHF, FMA = (x + T) and (+ b).
        const uint32_t xt = addf(xk, T, one);
        a = addf(b, rotl(a + lop3<FN>(b, c, d) + xt, S), one);
    } else {
        static_assert(B == Body::kSparse, "no MD5 step in this body");
        a = b + rotl(a + (xk + T) + lop3<FN>(b, c, d), S);
    }
}

// The two hashes are independent dependency chains over the same 16 words, so their rounds are
// interleaved at source level (4 SHA rounds : 4 MD5 steps) to give every warp two chains of ILP.
template <bool DO_SHA, bool DO_MD5, bool SPARSE = false>
__device__ __forceinline__ void compress(uint32_t (&hs)[8], uint32_t (&hm)[4], const uint32_t (&x)[16],
                                         bool is_last, uint32_t bits_lo, uint32_t bits_hi, uint32_t one) {
    //   instantiation <DO_SHA, DO_MD5, SPARSE>   SHA-256 round         MD5 step                   quad order
    //   dense fused    <1, 1, 0>  kDenseFused    LEA.HI Sigma rotates  LEA.HI rotate-add          MD5 first
    //   dense SHA-256  <1, 0, 0>  kDenseSha      IMAD.WIDE rotates     -                          -
    //   MD5 only       <0, 1, 0>  kMd5           -                     IADD3 sum, IMAD x+T and +b -
    //   sparse fused   <1, 1, 1>  kSparse        plain adds            plain adds                 SHA-256 first
    //   sparse SHA-256 <1, 0, 1>  kSparse        plain adds            -                          -
    // Every body expands the four schedule words of a quad of SHA-256 rounds ahead of its first round.
    static_assert(DO_SHA || !SPARSE, "MD5 alone has no sparse body");
    constexpr Body kBody = SPARSE ? Body::kSparse : !DO_SHA ? Body::kMd5 : DO_MD5 ? Body::kDenseFused : Body::kDenseSha;
    uint32_t w[16];
    uint32_t m14 = x[14], m15 = x[15];
    if (DO_SHA) {
#pragma unroll
        for (int i = 0; i < 16; ++i) w[i] = bswap(x[i]);
        if (is_last) {
            w[14] = bits_hi;
            w[15] = bits_lo;
        }
    }
    if (DO_MD5 && is_last) {
        m14 = bits_lo;
        m15 = bits_hi;
    }
    uint32_t a = hs[0], b = hs[1], c = hs[2], d = hs[3], e = hs[4], f = hs[5], g = hs[6], h = hs[7];
    uint32_t A = hm[0], B = hm[1], C = hm[2], D = hm[3];

#define SHA4(i, k0, k1, k2, k3)                                               \
    if constexpr (DO_SHA) {                                                   \
        if ((i) >= 16) {                                                      \
            sha_sched<kBody>(w, (i), one);                                    \
            sha_sched<kBody>(w, (i) + 1, one);                                \
            sha_sched<kBody>(w, (i) + 2, one);                                \
            sha_sched<kBody>(w, (i) + 3, one);                                \
        }                                                                     \
        if (((i)&7) == 0) {                                                   \
            sha_round<kBody>(a, b, c, d, e, f, g, h, k0, w[(i)&15], one);     \
            sha_round<kBody>(h, a, b, c, d, e, f, g, k1, w[((i) + 1) & 15], one); \
            sha_round<kBody>(g, h, a, b, c, d, e, f, k2, w[((i) + 2) & 15], one); \
            sha_round<kBody>(f, g, h, a, b, c, d, e, k3, w[((i) + 3) & 15], one); \
        } else {                                                              \
            sha_round<kBody>(e, f, g, h, a, b, c, d, k0, w[(i)&15], one);     \
            sha_round<kBody>(d, e, f, g, h, a, b, c, k1, w[((i) + 1) & 15], one); \
            sha_round<kBody>(c, d, e, f, g, h, a, b, k2, w[((i) + 2) & 15], one); \
            sha_round<kBody>(b, c, d, e, f, g, h, a, k3, w[((i) + 3) & 15], one); \
        }                                                                     \
    }
#define MD4(FN, x0, x1, x2, x3, s0, s1, s2, s3, t0, t1, t2, t3) \
    if constexpr (DO_MD5) {                                     \
        md5_step<kBody, FN, s0>(A, B, C, D, x0, t0, one);       \
        md5_step<kBody, FN, s1>(D, A, B, C, x1, t1, one);       \
        md5_step<kBody, FN, s2>(C, D, A, B, x2, t2, one);       \
        md5_step<kBody, FN, s3>(B, C, D, A, x3, t3, one);       \
    }
#define QUAD(i, k0, k1, k2, k3, FN, x0, x1, x2, x3, s0, s1, s2, s3, t0, t1, t2, t3)      \
    if constexpr (kBody == Body::kDenseFused) {                                        \
        MD4(FN, x0, x1, x2, x3, s0, s1, s2, s3, t0, t1, t2, t3) SHA4(i, k0, k1, k2, k3) \
    } else {                                                                           \
        SHA4(i, k0, k1, k2, k3) MD4(FN, x0, x1, x2, x3, s0, s1, s2, s3, t0, t1, t2, t3) \
    }

    QUAD(0, 0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, kMd5F, x[0], x[1], x[2], x[3], 7, 12, 17, 22, 0xd76aa478u, 0xe8c7b756u, 0x242070dbu, 0xc1bdceeeu)
    QUAD(4, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u, kMd5F, x[4], x[5], x[6], x[7], 7, 12, 17, 22, 0xf57c0fafu, 0x4787c62au, 0xa8304613u, 0xfd469501u)
    QUAD(8, 0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, kMd5F, x[8], x[9], x[10], x[11], 7, 12, 17, 22, 0x698098d8u, 0x8b44f7afu, 0xffff5bb1u, 0x895cd7beu)
    QUAD(12, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u, kMd5F, x[12], x[13], m14, m15, 7, 12, 17, 22, 0x6b901122u, 0xfd987193u, 0xa679438eu, 0x49b40821u)
    QUAD(16, 0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, kMd5G, x[1], x[6], x[11], x[0], 5, 9, 14, 20, 0xf61e2562u, 0xc040b340u, 0x265e5a51u, 0xe9b6c7aau)
    QUAD(20, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau, kMd5G, x[5], x[10], m15, x[4], 5, 9, 14, 20, 0xd62f105du, 0x02441453u, 0xd8a1e681u, 0xe7d3fbc8u)
    QUAD(24, 0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, kMd5G, x[9], m14, x[3], x[8], 5, 9, 14, 20, 0x21e1cde6u, 0xc33707d6u, 0xf4d50d87u, 0x455a14edu)
    QUAD(28, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u, kMd5G, x[13], x[2], x[7], x[12], 5, 9, 14, 20, 0xa9e3e905u, 0xfcefa3f8u, 0x676f02d9u, 0x8d2a4c8au)
    QUAD(32, 0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, kMd5H, x[5], x[8], x[11], m14, 4, 11, 16, 23, 0xfffa3942u, 0x8771f681u, 0x6d9d6122u, 0xfde5380cu)
    QUAD(36, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u, kMd5H, x[1], x[4], x[7], x[10], 4, 11, 16, 23, 0xa4beea44u, 0x4bdecfa9u, 0xf6bb4b60u, 0xbebfbc70u)
    QUAD(40, 0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, kMd5H, x[13], x[0], x[3], x[6], 4, 11, 16, 23, 0x289b7ec6u, 0xeaa127fau, 0xd4ef3085u, 0x04881d05u)
    QUAD(44, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u, kMd5H, x[9], x[12], m15, x[2], 4, 11, 16, 23, 0xd9d4d039u, 0xe6db99e5u, 0x1fa27cf8u, 0xc4ac5665u)
    QUAD(48, 0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, kMd5I, x[0], x[7], m14, x[5], 6, 10, 15, 21, 0xf4292244u, 0x432aff97u, 0xab9423a7u, 0xfc93a039u)
    QUAD(52, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u, kMd5I, x[12], x[3], x[10], x[1], 6, 10, 15, 21, 0x655b59c3u, 0x8f0ccc92u, 0xffeff47du, 0x85845dd1u)
    QUAD(56, 0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, kMd5I, x[8], m15, x[6], x[13], 6, 10, 15, 21, 0x6fa87e4fu, 0xfe2ce6e0u, 0xa3014314u, 0x4e0811a1u)
    QUAD(60, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u, kMd5I, x[4], x[11], x[2], x[9], 6, 10, 15, 21, 0xf7537e82u, 0xbd3af235u, 0x2ad7d2bbu, 0xeb86d391u)
#undef SHA4
#undef MD4
#undef QUAD

    if (DO_SHA) {
        hs[0] += a; hs[1] += b; hs[2] += c; hs[3] += d;
        hs[4] += e; hs[5] += f; hs[6] += g; hs[7] += h;
    }
    if (DO_MD5) {
        hm[0] += A; hm[1] += B; hm[2] += C; hm[3] += D;
    }
}

// ------------------------------------------------------------------------------ lane_hash_kernel

// CTAs per SM each lane-kernel instantiation is compiled for.  H100 (100 000 x 256 KiB, kernel time): SHA-256 alone
// gains 5 % at 4 CTAs (128 registers) over 5 (96).  The fused SHA-256 + MD5 kernel with LEA.HI rotate+adds and a uniform
// `one` runs 7 % faster at 4 CTAs, where it needs no spill, than at 5 (96 registers, 88 bytes of spill): 36.14 -> 33.70
// ms on an H100 80GB HBM3 at a 700 W power limit (DESIGN.md 6).  So the instantiations that compute SHA-256 get 4,
// except the dense fused one: at 3 CTAs (up to 168 registers; ptxas takes 158) its body reads fewer vector registers and
// it ran 2.2 % faster than at 4 (128 registers) on an H100 at 700 W, and 3.1 % faster with its LOP3 operand order and
// MD5-first quads (sha_round, DESIGN.md 6).  MD5 alone, at 96 registers either way, keeps 5.
template <bool DO_SHA, bool DO_MD5, bool SPARSE>
__host__ __device__ constexpr int lane_ctas_per_sm() {
    return !DO_SHA ? 5 : (DO_MD5 && !SPARSE) ? 3 : 4;
}
constexpr int kLaneThreads = 128;  // 4 warps; every warp runs an independent TMA/mbarrier ring
constexpr int kLaneWarps = kLaneThreads / 32;
constexpr int kBPC = 2;     // 64-byte blocks per chunk (one bulk copy)
constexpr int kStages = 2;  // chunks in flight per lane
constexpr int kSlot = kBPC * 64 + 16;  // +16: holds the misaligned-start granule and de-conflicts LDS.128
constexpr int kWarpSmem = kStages * 32 * kSlot;
constexpr int kLaneSmem = kLaneWarps * kWarpSmem;

__device__ __forceinline__ uint64_t warp_max_u64(uint64_t v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        uint64_t t = __shfl_xor_sync(0xffffffffu, v, o);
        v = t > v ? t : v;
    }
    return v;
}

// Work queue shared by all persistent warps: a power-of-two ring of message ids in plan order (longest
// first).  qctl[0] = entries available (signed), qctl[1] = head ticket, qctl[2] = tail ticket.
// A FRESH entry starts from the IV; a re-queued entry resumes from its ChainState in st[].
constexpr uint32_t kFresh = 0x80000000u;
constexpr uint32_t kEmpty = 0xffffffffu;

__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void st_volatile_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.volatile.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Persistent, time-sliced scheduling.  Every lane owns at most one message at a time and advances it by
// one quantum (<= `quantum` 64-byte blocks, plus the padding blocks when the message ends).  At each quantum
// boundary a warp whose lanes still hold unfinished messages puts them back on the queue *if other messages
// are waiting* and pops the next ones, so n messages share S < n lanes evenly (no wave quantisation) and
// mixed sizes balance like longest-first list scheduling.  Digest chaining state travels through st[].
// SPARSE: instantiation for batches that leave every warp alone on its SMSP (<= 4 warps per SM): such a warp is
// bound by its own issue rate (one instruction per two cycles), so the adds are left to ptxas (IADD3 / LEA fusion,
// ~15 % fewer instructions per block) instead of being spread over the FMA pipe.
template <bool DO_SHA, bool DO_MD5, bool SPARSE>
__global__ void __launch_bounds__(kLaneThreads, lane_ctas_per_sm<DO_SHA, DO_MD5, SPARSE>())
lane_hash_kernel(const uint8_t* __restrict__ base, const uint64_t* __restrict__ off, const uint64_t* __restrict__ len,
                 uint32_t* __restrict__ ring, uint32_t ring_mask, int* __restrict__ qctl, const int* __restrict__ ctl,
                 uint32_t flags, int lanes_per_warp, uint32_t quantum, uint8_t* __restrict__ sha_out,
                 uint8_t* __restrict__ md5_out, ChainState* __restrict__ st, uint32_t one) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int lane = threadIdx.x & 31;
    const int wib = threadIdx.x >> 5;
    const uint32_t lt_mask = (1u << lane) - 1u;
    uint8_t* ring_smem = smem + wib * kWarpSmem;
    constexpr bool kOctetGather = !DO_SHA && kBPC == 2;
    constexpr bool kPairGather = !(DO_SHA && DO_MD5) && !kOctetGather;
    const bool final = !(flags & F_NO_FINAL);
    const bool lane_on = lane < lanes_per_warp;
    if (flags & F_YIELD_CHAIN_SMS) {
        // This SM hosts a chain CTA that carries one of the batch's longest messages: the chain's round warp issues at
        // most one instruction every two cycles and every lane warp next to it on the SMSP takes slots away from the
        // one chain that sets the makespan.
        // The queue makes leaving free: whatever this CTA would have hashed is pulled by the CTAs on the other SMs.
        // The chain kernel is launched just before this one, on a high-priority stream, with at most one CTA per SM
        // on at most 3/4 of the SMs: its CTAs are resident within microseconds.  Wait for them (bounded: if they are
        // not all there after kYieldWaitNs we simply go ahead and share), then leave if this SM is taken.  Leaving
        // happens here only, before a single message has been taken, so nothing can be stranded.
        uint32_t smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        const uint32_t* q = reinterpret_cast<const uint32_t*>(ctl);
        const uint32_t expected = ld_volatile_u32(q + kChainExpectedWord);
        if (expected) {
            const unsigned long long t0 = globaltimer_ns();
            while (ld_volatile_u32(q + kChainStartedWord) < expected && globaltimer_ns() - t0 < kYieldWaitNs) {
            }
        }
        if (smid < (uint32_t)kSmFlagWords && ld_volatile_u32(q + kSmFlagsAfterQctl + smid) != 0u) return;
    }

    // ---- per-lane message context
    bool has = false;
    uint32_t mi = 0;
    const uint8_t* p = base;
    uint64_t L = 0, nfull = 0, done = 0, prior = 0;
    uint32_t hs[8], hm[4];

    for (;;) {
        // ------------------------------------------------------------ rotate: give waiting messages a turn
        int waiting = 0;
        if (lane == 0) waiting = *reinterpret_cast<volatile int*>(&qctl[0]);
        waiting = __shfl_sync(0xffffffffu, waiting, 0);
        const uint32_t has_mask = __ballot_sync(0xffffffffu, has);
        if (waiting > 0 && has_mask) {
            if (has) {
                uint4* sp = reinterpret_cast<uint4*>(&st[mi]);
                __stcg(sp + 0, make_uint4(hs[0], hs[1], hs[2], hs[3]));
                __stcg(sp + 1, make_uint4(hs[4], hs[5], hs[6], hs[7]));
                __stcg(sp + 2, make_uint4(hm[0], hm[1], hm[2], hm[3]));
                __stcg(sp + 3, make_uint4((uint32_t)prior, (uint32_t)(prior >> 32), (uint32_t)done, (uint32_t)(done >> 32)));
                __threadfence();
            }
            const int k = __popc(has_mask);
            uint32_t t0 = 0;
            if (lane == 0) t0 = atomicAdd(reinterpret_cast<unsigned int*>(&qctl[2]), (unsigned int)k);
            t0 = __shfl_sync(0xffffffffu, t0, 0);
            if (has) {
                uint32_t* slot = ring + ((t0 + __popc(has_mask & lt_mask)) & ring_mask);
                while (ld_volatile_u32(slot) != kEmpty) {
                }
                st_volatile_u32(slot, mi);
                __threadfence();
            }
            __syncwarp();
            if (lane == 0) atomicAdd(&qctl[0], k);
            has = false;
        }
        // ------------------------------------------------------------ acquire
        const uint32_t need_mask = __ballot_sync(0xffffffffu, lane_on && !has);
        if (need_mask) {
            const int need = __popc(need_mask);
            int got = 0;
            uint32_t h0 = 0;
            if (lane == 0) {
                const int old = atomicSub(&qctl[0], need);
                got = old >= need ? need : (old > 0 ? old : 0);
                if (got < need) atomicAdd(&qctl[0], need - got);
                if (got) h0 = atomicAdd(reinterpret_cast<unsigned int*>(&qctl[1]), (unsigned int)got);
            }
            got = __shfl_sync(0xffffffffu, got, 0);
            h0 = __shfl_sync(0xffffffffu, h0, 0);
            if (lane_on && !has && __popc(need_mask & lt_mask) < got) {
                uint32_t* slot = ring + ((h0 + __popc(need_mask & lt_mask)) & ring_mask);
                uint32_t e;
                while ((e = ld_volatile_u32(slot)) == kEmpty) {
                }
                st_volatile_u32(slot, kEmpty);
                mi = e & ~kFresh;
                has = true;
                p = base + off[mi];
                L = len[mi];
                nfull = L >> 6;
                if (e & kFresh) {
                    hs[0] = 0x6a09e667u; hs[1] = 0xbb67ae85u; hs[2] = 0x3c6ef372u; hs[3] = 0xa54ff53au;
                    hs[4] = 0x510e527fu; hs[5] = 0x9b05688cu; hs[6] = 0x1f83d9abu; hs[7] = 0x5be0cd19u;
                    hm[0] = 0x67452301u; hm[1] = 0xefcdab89u; hm[2] = 0x98badcfeu; hm[3] = 0x10325476u;
                    done = 0;
                    prior = 0;
                } else {
                    __threadfence();
                    const uint4* sp = reinterpret_cast<const uint4*>(&st[mi]);
                    const uint4 q0 = __ldcg(sp + 0), q1 = __ldcg(sp + 1), q2 = __ldcg(sp + 2), q3 = __ldcg(sp + 3);
                    hs[0] = q0.x; hs[1] = q0.y; hs[2] = q0.z; hs[3] = q0.w;
                    hs[4] = q1.x; hs[5] = q1.y; hs[6] = q1.z; hs[7] = q1.w;
                    hm[0] = q2.x; hm[1] = q2.y; hm[2] = q2.z; hm[3] = q2.w;
                    prior = (uint64_t)q3.x | ((uint64_t)q3.y << 32);
                    done = (uint64_t)q3.z | ((uint64_t)q3.w << 32);
                }
            }
        }
        if (!__any_sync(0xffffffffu, has)) break;

        // ------------------------------------------------------------ one quantum
        const uint32_t r = final ? (uint32_t)(L & 63) : 0u;
        uint32_t qblocks = 0, ntail = 0;
        if (has) {
            const uint64_t rem = nfull - done;
            qblocks = rem < quantum ? (uint32_t)rem : quantum;
            if (final && done + qblocks == nfull) ntail = r < 56 ? 1u : 2u;
        }
        const uint32_t nsteps = qblocks + ntail;
        const uint64_t bits = (prior + L) << 3;
        const uint32_t bits_lo = (uint32_t)bits, bits_hi = (uint32_t)(bits >> 32);
        const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 15u);
        const uint8_t* src = p - mis + (done << 6);  // 16B-aligned source of this quantum's first block
        const bool warp_aligned = __all_sync(0xffffffffu, mis == 0);
        const uint32_t nchunks = (qblocks + kBPC - 1) / kBPC;
        const uint32_t max_outer = (__reduce_max_sync(0xffffffffu, nsteps) + kBPC - 1) / kBPC;

        // Each lane gathers its own chunk with 16-byte cp.async (LDGSTS) into its private slot; one commit
        // group per chunk, so wait_group<kStages-1> means "my chunk c has landed".  No cross-lane sync.
        // Lane pairs gather each other's chunks: in one LDGSTS instruction lanes 2k and 2k+1 fetch the two
        // 16-byte halves of the SAME 32-byte sector (of message 2k first, then of message 2k+1), so the LSU
        // coalesces them into one sector request; a lane fetching only its own 16-byte pieces asks L2 for every
        // sector twice (ncu: lts sectors = 2.5x the payload in the MD5-only kernel).  Copies written by the
        // partner are tracked by the partner's commit group, hence the __syncwarp after wait_group below.
        // Measured (100000 x 256 KiB): MD5-only +4.8 %, SHA-only +6 %, fused -2.7 % (already issue-bound, the extra
        // shuffles cost more than the L2 relief gives) -> enabled for the single-digest instantiations only.
        auto issue = [&](uint32_t c) {
            if constexpr (kOctetGather) {
                // Eight lanes fetch the eight 16-byte pieces of ONE message's 128-byte chunk in the same LDGSTS, four
                // messages per instruction: every instruction is 4 full-line requests instead of 32 sector requests
                // (the MD5-only kernel ran at 79 % l1tex throughput with per-lane gathers).
                uint32_t pieces = 0, dst = 0;
                const uint8_t* g = src;
                if (c < nchunks) {
                    const uint32_t rem = qblocks - c * kBPC;
                    pieces = (rem < (uint32_t)kBPC ? rem : (uint32_t)kBPC) * 4u + (mis ? 1u : 0u);
                    dst = smem_u32(ring_smem + ((c % kStages) * 32 + lane) * kSlot);
                    g = src + c * (kBPC * 64);
                }
                const uint64_t g64 = reinterpret_cast<uint64_t>(g);
                const uint32_t k = lane & 7u;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int from = 4 * i + (lane >> 3);
                    const uint64_t og = __shfl_sync(0xffffffffu, g64, from);
                    const uint32_t on = __shfl_sync(0xffffffffu, pieces, from);
                    const uint32_t od = __shfl_sync(0xffffffffu, dst, from);
                    if (k < on) cp_async16(od + 16u * k, reinterpret_cast<const uint8_t*>(og) + 16u * k);
                }
                if (pieces > 8) cp_async16(dst + 128u, g + 128);  // the extra granule of a misaligned start
                cp_async_commit();
            } else if constexpr (kPairGather) {
                uint32_t pieces = 0, dst = 0;
                const uint8_t* g = src;
                if (c < nchunks) {
                    const uint32_t rem = qblocks - c * kBPC;
                    pieces = (rem < (uint32_t)kBPC ? rem : (uint32_t)kBPC) * 4u + (mis ? 1u : 0u);
                    dst = smem_u32(ring_smem + ((c % kStages) * 32 + lane) * kSlot);
                    g = src + c * (kBPC * 64);
                }
                const uint32_t odd = lane & 1u;
                const uint64_t g64 = reinterpret_cast<uint64_t>(g);
                const uint64_t pg64 = __shfl_xor_sync(0xffffffffu, g64, 1);
                const uint32_t ppieces = __shfl_xor_sync(0xffffffffu, pieces, 1);
                const uint32_t pdst = __shfl_xor_sync(0xffffffffu, dst, 1);
                // message of the even lane (A), then message of the odd lane (B)
                const uint64_t ga = odd ? pg64 : g64, gb = odd ? g64 : pg64;
                const uint32_t na = odd ? ppieces : pieces, nb = odd ? pieces : ppieces;
                const uint32_t da = odd ? pdst : dst, db = odd ? dst : pdst;
                // start at an even 16-byte granule of the source so that a pair shares a 32-byte sector
                const int pa = (int)((ga >> 4) & 1u), pb = (int)((gb >> 4) & 1u);
#pragma unroll
                for (int i = 0; i < (kBPC * 4 + 1 + 2) / 2; ++i) {
                    const int k = 2 * i + (int)odd - pa;
                    if (k >= 0 && (uint32_t)k < na) cp_async16(da + 16u * k, reinterpret_cast<const uint8_t*>(ga) + 16 * k);
                }
#pragma unroll
                for (int i = 0; i < (kBPC * 4 + 1 + 2) / 2; ++i) {
                    const int k = 2 * i + (int)odd - pb;
                    if (k >= 0 && (uint32_t)k < nb) cp_async16(db + 16u * k, reinterpret_cast<const uint8_t*>(gb) + 16 * k);
                }
                cp_async_commit();
            } else {
                if (c < nchunks) {
                    const uint32_t rem = qblocks - c * kBPC;
                    const uint32_t pieces = (rem < (uint32_t)kBPC ? rem : (uint32_t)kBPC) * 4u + (mis ? 1u : 0u);
                    const uint32_t dst = smem_u32(ring_smem + ((c % kStages) * 32 + lane) * kSlot);
                    const uint8_t* g = src + c * (kBPC * 64);
                    if (pieces == kBPC * 4) {
                        // a full, aligned chunk (every chunk of an aligned message but its last): 8 copies at immediate
                        // offsets from one address pair instead of a predicated address pair per piece
#pragma unroll
                        for (uint32_t k = 0; k < kBPC * 4; ++k) cp_async16(dst + 16 * k, g + 16 * k);
                    } else {
#pragma unroll
                        for (uint32_t k = 0; k < kBPC * 4 + 1; ++k)
                            if (k < pieces) cp_async16(dst + 16 * k, g + 16 * k);
                    }
                }
                cp_async_commit();
            }
        };

#pragma unroll
        for (int s = 0; s < kStages; ++s) issue(s);

        for (uint32_t c = 0; c < max_outer; ++c) {
            const uint32_t sidx = c % kStages;
            cp_async_wait<kStages - 1>();
            if constexpr (kPairGather || kOctetGather) __syncwarp();  // my chunk was partly copied by other lanes
            const uint8_t* slot = ring_smem + (sidx * 32 + lane) * kSlot;
#pragma unroll 1
            for (int j = 0; j < kBPC; ++j) {
                const uint32_t step = c * kBPC + j;
                if (step < nsteps) {
                    uint32_t x[16];
                    if (step < qblocks) {
                        const uint8_t* blk = slot + j * 64;
                        if (warp_aligned) {
                            const uint4* q = reinterpret_cast<const uint4*>(blk);
#pragma unroll
                            for (int k = 0; k < 4; ++k) {
                                uint4 v = q[k];
                                x[4 * k] = v.x; x[4 * k + 1] = v.y; x[4 * k + 2] = v.z; x[4 * k + 3] = v.w;
                            }
                        } else {
                            const uint32_t* wp = reinterpret_cast<const uint32_t*>(blk + (mis & ~3u));
                            const uint32_t sh = (mis & 3u) * 8u;
                            uint32_t y[17];
#pragma unroll
                            for (int k = 0; k < 17; ++k) y[k] = wp[k];
#pragma unroll
                            for (int k = 0; k < 16; ++k) x[k] = __funnelshift_r(y[k], y[k + 1], sh);
                        }
                    } else if (step == qblocks) {
                        // first padding block: the r leftover bytes straight from global (aligned 32-bit words,
                        // only words that contain a message byte), then 0x80 and zero fill.
                        const uint8_t* g = p + (nfull << 6);
                        const uint32_t gm = (uint32_t)(reinterpret_cast<uintptr_t>(g) & 3u);
                        const uint32_t* gw = reinterpret_cast<const uint32_t*>(g - gm);
                        const uint32_t span = r ? gm + r : 0u;  // bytes from gw to the end of the message
                        uint32_t y[17];
#pragma unroll
                        for (int k = 0; k < 17; ++k) y[k] = (4u * k < span) ? __ldg(gw + k) : 0u;
#pragma unroll
                        for (int k = 0; k < 16; ++k) {
                            uint32_t v = __funnelshift_r(y[k], y[k + 1], gm * 8u);
                            const int have = (int)r - 4 * k;  // message bytes in this word
                            if (have <= 0) v = 0;
                            else if (have < 4) v &= (1u << (8 * have)) - 1u;
                            if (have >= 0 && have < 4) v |= 0x80u << (8 * have);
                            x[k] = v;
                        }
                    } else {
#pragma unroll
                        for (int k = 0; k < 16; ++k) x[k] = 0u;
                    }
                    const bool is_last = ntail && (step + 1 == nsteps);
                    compress<DO_SHA, DO_MD5, SPARSE>(hs, hm, x, is_last, bits_lo, bits_hi, one);
                }
            }
            issue(c + kStages);  // refill the slot just consumed (an empty group when nothing is left)
        }
        cp_async_wait<0>();
        if constexpr (kPairGather || kOctetGather) __syncwarp();

        // ------------------------------------------------------------ retire finished messages
        if (has) {
            done += qblocks;
            if (done == nfull) {
                if (final) {
                    if (DO_SHA && sha_out) {
                        uint4* o = reinterpret_cast<uint4*>(sha_out + 32ull * mi);
                        o[0] = make_uint4(bswap(hs[0]), bswap(hs[1]), bswap(hs[2]), bswap(hs[3]));
                        o[1] = make_uint4(bswap(hs[4]), bswap(hs[5]), bswap(hs[6]), bswap(hs[7]));
                    }
                    if (DO_MD5 && md5_out)
                        *reinterpret_cast<uint4*>(md5_out + 16ull * mi) = make_uint4(hm[0], hm[1], hm[2], hm[3]);
                } else {
                    // continuation segment: hand the chaining state back to the caller
                    uint4* sp = reinterpret_cast<uint4*>(&st[mi]);
                    const uint64_t np = prior + L;
                    sp[0] = make_uint4(hs[0], hs[1], hs[2], hs[3]);
                    sp[1] = make_uint4(hs[4], hs[5], hs[6], hs[7]);
                    sp[2] = make_uint4(hm[0], hm[1], hm[2], hm[3]);
                    sp[3] = make_uint4((uint32_t)np, (uint32_t)(np >> 32), 0u, 0u);
                }
                has = false;
            }
        }
    }
}

// ------------------------------------------------------------------------------ chain_hash_kernel
// One CTA per SM (its shared-memory request is more than half an SM's, so placement cannot double CTAs up); a CTA
// hosts up to kChainGroups long messages, each served by a group of three specialised warps on tiles of 32 blocks
// (2 KiB).  Within a group:
//   warp 0  producer/expander: one elected lane streams the message into a 4-deep shared-memory tile ring
//           with 1-D TMA bulk copies (cp.async.bulk -> UBLKCP, mbarrier complete_tx); then all 32 lanes
//           expand the SHA-256 message schedule of the tile's 32 blocks in parallel (lane = block) and store
//           W[t]+K[t] rows for the chain warp.  The padding block(s) are synthesised into a final tile.
//   warp 1  SHA-256 chain: one lane runs the 64 rounds per block straight from the W+K rows.
//   warp 2  MD5 chain: one lane runs the 64 steps per block straight from the raw tile.
// The warps of a group hand tiles over through mbarriers only.  Entry e of the chain list is served by group
// e / gridDim.x of CTA e % gridDim.x: up to gridDim.x outliers get an SM each, and with warp w of a CTA on SMSP
// w % 4 the twelve warps of a full CTA put exactly one expander, one SHA-256 and one MD5 warp on every SMSP.

constexpr int kChainGroups = 4;     // messages per CTA by default (one expander, one SHA-256 and one MD5 warp per SMSP)
constexpr int kChainGroupsMax = 8;  // B200H_CHAIN_GROUPS=8: twice that per SMSP; off by default
constexpr int kChainGroupThreads = 96;
constexpr int kTileBlocks = 32;
constexpr int kTileData = kTileBlocks * 64;
constexpr int kTileStride = kTileData + 32;  // + the misaligned leading granule; keeps 16-byte alignment
constexpr int kNT = 4;                        // raw tile ring depth
constexpr int kWkRow = 64 * 4 + 16;           // 272 B: conflict-free STS.128 across lanes
constexpr int kWkBuf = kTileBlocks * kWkRow;
constexpr int kNW = 2;                        // W+K ring depth
constexpr int kChainGroupSmem = (kNT * kTileStride + kNW * kWkBuf + (2 * kNT + 2 * kNW) * 8 + 127) & ~127;
constexpr int kChainSmemMin = 116 * 1024;  // > 227 KB / 2: never two chain CTAs on one SM
constexpr int chain_smem_bytes(int groups) {
    return groups * kChainGroupSmem > kChainSmemMin ? groups * kChainGroupSmem : kChainSmemMin;
}
static int g_chain_groups = kChainGroups;  // set once by configure_kernels() from B200H_CHAIN_GROUPS

__constant__ uint32_t kShaKAll[64] = {
    0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u,
    0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u,
    0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau,
    0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u,
    0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
    0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u,
    0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u,
    0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u};

__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

// 16 little-endian message words of the 64-byte block at `blk + toff` (toff = 0..15 bytes of misalignment)
__device__ __forceinline__ void load_block_words(const uint8_t* blk, uint32_t toff, uint32_t (&x)[16]) {
    if (toff == 0) {
        const uint4* q = reinterpret_cast<const uint4*>(blk);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint4 v = q[k];
            x[4 * k] = v.x; x[4 * k + 1] = v.y; x[4 * k + 2] = v.z; x[4 * k + 3] = v.w;
        }
    } else {
        const uint32_t* wp = reinterpret_cast<const uint32_t*>(blk + (toff & ~3u));
        const uint32_t sh = (toff & 3u) * 8u;
        uint32_t y[17];
#pragma unroll
        for (int k = 0; k < 17; ++k) y[k] = wp[k];
#pragma unroll
        for (int k = 0; k < 16; ++k) x[k] = __funnelshift_r(y[k], y[k + 1], sh);
    }
}

// One SHA-256 round for the chain warp.  A lone warp issues at most one instruction every two cycles whatever
// the pipe, so what counts here is the instruction count: the two three-input sums are IADD3s (14 instructions
// per round instead of 16 with two-input IMAD adds: 2 049 -> 1 769 cycles per block, tools/chainbench.cu).
#define CH_RND(a, b, c, d, e, f, g, h, WK)                                            \
    {                                                                                 \
        const uint32_t hwk = addf(h, WK, one);                                        \
        const uint32_t t1 = hwk + lop3<0xCA>(e, f, g) + SHA_S1(e);                    \
        d = addf(d, t1, one);                                                         \
        h = t1 + SHA_S0(a) + lop3<0xE8>(a, b, c);                                     \
    }

// MD5 block for the chain warp.  One chain on one warp is bound by the dependent-instruction latency of a step
// (b -> F -> sum -> rotate -> + b), not by issue slots, so the step is written for the shortest dependency chain:
// (x + T) off the critical path, one IADD3, and rotate+add left to ptxas as a single LEA.HI (tools/chainbench.cu
// measures the cycles per block).
// T[i] = floor(2^32 * |sin(i + 1)|) (RFC 1321); a switch so that the unrolled steps get immediates, not
// constant-bank loads whose latency a lone warp cannot hide.
__device__ __forceinline__ constexpr uint32_t md5_T(int i) {
    switch (i) {
        case 0: return 0xd76aa478u;
        case 1: return 0xe8c7b756u;
        case 2: return 0x242070dbu;
        case 3: return 0xc1bdceeeu;
        case 4: return 0xf57c0fafu;
        case 5: return 0x4787c62au;
        case 6: return 0xa8304613u;
        case 7: return 0xfd469501u;
        case 8: return 0x698098d8u;
        case 9: return 0x8b44f7afu;
        case 10: return 0xffff5bb1u;
        case 11: return 0x895cd7beu;
        case 12: return 0x6b901122u;
        case 13: return 0xfd987193u;
        case 14: return 0xa679438eu;
        case 15: return 0x49b40821u;
        case 16: return 0xf61e2562u;
        case 17: return 0xc040b340u;
        case 18: return 0x265e5a51u;
        case 19: return 0xe9b6c7aau;
        case 20: return 0xd62f105du;
        case 21: return 0x02441453u;
        case 22: return 0xd8a1e681u;
        case 23: return 0xe7d3fbc8u;
        case 24: return 0x21e1cde6u;
        case 25: return 0xc33707d6u;
        case 26: return 0xf4d50d87u;
        case 27: return 0x455a14edu;
        case 28: return 0xa9e3e905u;
        case 29: return 0xfcefa3f8u;
        case 30: return 0x676f02d9u;
        case 31: return 0x8d2a4c8au;
        case 32: return 0xfffa3942u;
        case 33: return 0x8771f681u;
        case 34: return 0x6d9d6122u;
        case 35: return 0xfde5380cu;
        case 36: return 0xa4beea44u;
        case 37: return 0x4bdecfa9u;
        case 38: return 0xf6bb4b60u;
        case 39: return 0xbebfbc70u;
        case 40: return 0x289b7ec6u;
        case 41: return 0xeaa127fau;
        case 42: return 0xd4ef3085u;
        case 43: return 0x04881d05u;
        case 44: return 0xd9d4d039u;
        case 45: return 0xe6db99e5u;
        case 46: return 0x1fa27cf8u;
        case 47: return 0xc4ac5665u;
        case 48: return 0xf4292244u;
        case 49: return 0x432aff97u;
        case 50: return 0xab9423a7u;
        case 51: return 0xfc93a039u;
        case 52: return 0x655b59c3u;
        case 53: return 0x8f0ccc92u;
        case 54: return 0xffeff47du;
        case 55: return 0x85845dd1u;
        case 56: return 0x6fa87e4fu;
        case 57: return 0xfe2ce6e0u;
        case 58: return 0xa3014314u;
        case 59: return 0x4e0811a1u;
        case 60: return 0xf7537e82u;
        case 61: return 0xbd3af235u;
        case 62: return 0x2ad7d2bbu;
        default: return 0xeb86d391u;
    }
}

__device__ __forceinline__ void md5_chain_block(uint32_t (&hm)[4], const uint32_t (&x)[16], uint32_t one) {
    uint32_t v[4] = {hm[0], hm[1], hm[2], hm[3]};  // A B C D; step i writes v[(64 - i) & 3] (RFC 1321 role rotation)
#pragma unroll
    for (int i = 0; i < 64; ++i) {
        const int r = i >> 4;
        const int g = r == 0 ? i : r == 1 ? (5 * i + 1) & 15 : r == 2 ? (3 * i + 5) & 15 : (7 * i) & 15;
        const int sh = r == 0 ? (i & 3) * 5 + 7                                   // 7 12 17 22
                              : r == 1 ? ((i & 3) == 0 ? 5 : (i & 3) == 1 ? 9 : (i & 3) == 2 ? 14 : 20)
                                       : r == 2 ? ((i & 3) == 0 ? 4 : (i & 3) == 1 ? 11 : (i & 3) == 2 ? 16 : 23)
                                                : ((i & 3) == 0 ? 6 : (i & 3) == 1 ? 10 : (i & 3) == 2 ? 15 : 21);
        uint32_t& a = v[(64 - i) & 3];
        const uint32_t b = v[(65 - i) & 3], c = v[(66 - i) & 3], d = v[(67 - i) & 3];
        const uint32_t fn = r == 0 ? lop3<0xCA>(b, c, d) : r == 1 ? lop3<0xE4>(b, c, d)
                                   : r == 2 ? lop3<0x96>(b, c, d) : lop3<0x39>(b, c, d);
        // x + T as a multiply-add by the run-time 1: ptxas cannot re-associate through it (with a plain add it
        // folds T into IADD3(F, T, x) and appends "+ a", one more dependent instruction per step)
        const uint32_t xt = addf(x[g], md5_T(i), one);
        a = b + rotl(a + fn + xt, sh);
    }
    hm[0] += v[0]; hm[1] += v[1]; hm[2] += v[2]; hm[3] += v[3];
}

template <bool DO_SHA, bool DO_MD5, int GROUPS>  // GROUPS only sets the launch bound (threads = 96 x GROUPS)
__global__ void __launch_bounds__(kChainGroupThreads * GROUPS)
chain_hash_kernel(const uint8_t* __restrict__ base, const uint64_t* __restrict__ off, const uint64_t* __restrict__ len,
                  const uint32_t* __restrict__ chain_list, const int* __restrict__ qctl, uint32_t flags,
                  uint8_t* __restrict__ sha_out, uint8_t* __restrict__ md5_out, ChainState* __restrict__ st,
                  int resume, uint32_t one) {
    const uint32_t n_chain = (uint32_t)qctl[3];
    if (blockIdx.x >= n_chain) return;  // entry e lives in CTA e % gridDim.x: this CTA has none
    if (threadIdx.x == 0) {  // tell lane CTAs that this SM is taken (F_YIELD_CHAIN_SMS), then that this CTA is resident
        uint32_t smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        uint32_t* q = const_cast<uint32_t*>(reinterpret_cast<const uint32_t*>(qctl));
        if (smid < (uint32_t)kSmFlagWords) st_volatile_u32(q + kSmFlagsAfterQctl + smid, 1u);
        __threadfence();
        atomicAdd(q + kChainStartedWord, 1u);
    }
    extern __shared__ __align__(128) uint8_t smem_all[];
    const int lane = threadIdx.x & 31;
    const int grp = (threadIdx.x >> 5) / 3;   // which of the CTA's messages
    const int warp = (threadIdx.x >> 5) % 3;  // role within the group
    uint8_t* smem = smem_all + grp * kChainGroupSmem;
    uint8_t* tiles = smem;
    uint8_t* wkbuf = smem + kNT * kTileStride;
    const uint32_t bars = smem_u32(smem + kNT * kTileStride + kNW * kWkBuf);
    const uint32_t tile_full = bars, tile_free = bars + 8 * kNT, wk_full = bars + 16 * kNT, wk_free = bars + 16 * kNT + 8 * kNW;
    if (warp == 0 && lane == 0) {
        for (int i = 0; i < kNT; ++i) {
            mbar_init(tile_full + 8 * i, 1);
            mbar_init(tile_free + 8 * i, (DO_SHA ? 1 : 0) + (DO_MD5 ? 1 : 0));
        }
        for (int i = 0; i < kNW; ++i) {
            mbar_init(wk_full + 8 * i, 1);
            mbar_init(wk_free + 8 * i, 1);
        }
        fence_mbar_init();
        fence_proxy_async();
    }
    __syncthreads();
    const uint32_t ent = blockIdx.x + gridDim.x * (uint32_t)grp;
    if (ent >= n_chain) return;  // this group has no message (its warps are done; the others never wait for them)

    const uint32_t mi = chain_list[ent];
    const uint8_t* p = base + off[mi];
    const uint64_t L = len[mi];
    const bool final = !(flags & F_NO_FINAL);
    uint64_t prior = 0;
    if (resume) prior = st[mi].prior_bytes;
    const uint64_t nfull = L >> 6;
    const uint32_t r = final ? (uint32_t)(L & 63) : 0u;
    const uint32_t ntail = final ? (r < 56 ? 1u : 2u) : 0u;
    const uint64_t t_data = (nfull + kTileBlocks - 1) / kTileBlocks;  // tiles streamed by TMA
    const uint64_t t_all = t_data + (ntail ? 1 : 0);                  // + the synthesised padding tile
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 15u);
    const uint8_t* p0 = p - mis;
    const uint64_t bits = (prior + L) << 3;
    const uint32_t bits_lo = (uint32_t)bits, bits_hi = (uint32_t)(bits >> 32);
    auto blocks_in = [&](uint64_t t) -> uint32_t {
        if (t < t_data) {
            const uint64_t rem = nfull - t * kTileBlocks;
            return rem < (uint64_t)kTileBlocks ? (uint32_t)rem : (uint32_t)kTileBlocks;
        }
        return ntail;
    };

    if (warp == 0) {
        // ------------------------------------------------------------------ producer / schedule expander
        auto issue = [&](uint64_t t) {
            const uint32_t slot = (uint32_t)(t % kNT);
            mbar_wait(tile_free + 8 * slot, (uint32_t)(((t / kNT) & 1) ^ 1));
            uint8_t* tile = tiles + slot * kTileStride;
            if (t < t_data) {
                if (lane == 0) {
                    const uint32_t bytes = blocks_in(t) * 64u + (mis ? 16u : 0u);
                    mbar_arrive_expect_tx(tile_full + 8 * slot, bytes);
                    bulk_g2s(smem_u32(tile), p0 + t * kTileData, bytes, tile_full + 8 * slot);
                }
            } else {
                // padding tile: r leftover bytes, 0x80, zeros, 64-bit length (MD5 layout; the SHA expander
                // substitutes its own big-endian length words)
                reinterpret_cast<uint32_t*>(tile)[lane] = 0u;
                __syncwarp();
                const uint8_t* g = p + (nfull << 6);
                for (uint32_t i = lane; i < r; i += 32) tile[i] = g[i];
                if (lane == 0) {
                    tile[r] = 0x80;
                    uint32_t* lenw = reinterpret_cast<uint32_t*>(tile + (ntail - 1) * 64 + 56);
                    lenw[0] = bits_lo;
                    lenw[1] = bits_hi;
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(tile_full + 8 * slot);
            }
        };
        for (uint64_t t = 0; t < t_all && t < (uint64_t)(kNT - 1); ++t) issue(t);
        for (uint64_t t = 0; t < t_all; ++t) {
            if (t + kNT - 1 < t_all) issue(t + kNT - 1);
            if (DO_SHA) {
                const uint32_t slot = (uint32_t)(t % kNT), ws = (uint32_t)(t % kNW);
                const uint32_t nb = blocks_in(t);
                const uint32_t toff = t < t_data ? mis : 0u;
                mbar_wait(tile_full + 8 * slot, (uint32_t)((t / kNT) & 1));
                uint32_t x[16];
                if ((uint32_t)lane < nb) load_block_words(tiles + slot * kTileStride + lane * 64, toff, x);
                __syncwarp();
                if (lane == 0) mbar_arrive(tile_free + 8 * slot);
                mbar_wait(wk_free + 8 * ws, (uint32_t)(((t / kNW) & 1) ^ 1));
                if ((uint32_t)lane < nb) {
                    uint32_t w[16];
#pragma unroll
                    for (int i = 0; i < 16; ++i) w[i] = bswap(x[i]);
                    if (t >= t_data && (uint32_t)lane == ntail - 1) {
                        w[14] = bits_hi;
                        w[15] = bits_lo;
                    }
                    uint4* row = reinterpret_cast<uint4*>(wkbuf + ws * kWkBuf + lane * kWkRow);
#pragma unroll
                    for (int i = 0; i < 64; i += 4) {
                        uint32_t o[4];
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const int tt = i + j;
                            if (tt >= 16)
                                w[tt & 15] = w[tt & 15] + SHA_s1(w[(tt - 2) & 15]) + w[(tt - 7) & 15] + SHA_s0(w[(tt - 15) & 15]);
                            o[j] = w[tt & 15] + kShaKAll[tt];
                        }
                        row[i / 4] = make_uint4(o[0], o[1], o[2], o[3]);
                    }
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(wk_full + 8 * ws);
            }
        }
    } else if (warp == 1) {
        // ------------------------------------------------------------------------------- SHA-256 chain
        if (!DO_SHA) return;
        uint32_t hs[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au,
                          0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
        if (resume && lane == 0) {
#pragma unroll
            for (int i = 0; i < 8; ++i) hs[i] = st[mi].sha[i];
        }
        for (uint64_t t = 0; t < t_all; ++t) {
            const uint32_t ws = (uint32_t)(t % kNW);
            const uint32_t nb = blocks_in(t);
            mbar_wait(wk_full + 8 * ws, (uint32_t)((t / kNW) & 1));
            if (lane == 0) {
#pragma unroll 1
                for (uint32_t bidx = 0; bidx < nb; ++bidx) {
                    const uint4* row = reinterpret_cast<const uint4*>(wkbuf + ws * kWkBuf + bidx * kWkRow);
                    uint32_t k[64];
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        const uint4 v = row[i];
                        k[4 * i] = v.x; k[4 * i + 1] = v.y; k[4 * i + 2] = v.z; k[4 * i + 3] = v.w;
                    }
                    uint32_t a = hs[0], b = hs[1], c = hs[2], d = hs[3], e = hs[4], f = hs[5], g = hs[6], h = hs[7];
#pragma unroll
                    for (int i = 0; i < 64; i += 8) {
                        CH_RND(a, b, c, d, e, f, g, h, k[i]);
                        CH_RND(h, a, b, c, d, e, f, g, k[i + 1]);
                        CH_RND(g, h, a, b, c, d, e, f, k[i + 2]);
                        CH_RND(f, g, h, a, b, c, d, e, k[i + 3]);
                        CH_RND(e, f, g, h, a, b, c, d, k[i + 4]);
                        CH_RND(d, e, f, g, h, a, b, c, k[i + 5]);
                        CH_RND(c, d, e, f, g, h, a, b, k[i + 6]);
                        CH_RND(b, c, d, e, f, g, h, a, k[i + 7]);
                    }
                    hs[0] += a; hs[1] += b; hs[2] += c; hs[3] += d;
                    hs[4] += e; hs[5] += f; hs[6] += g; hs[7] += h;
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(wk_free + 8 * ws);
        }
        if (lane == 0) {
            if (final) {
                if (sha_out) {
                    uint4* o = reinterpret_cast<uint4*>(sha_out + 32ull * mi);
                    o[0] = make_uint4(bswap(hs[0]), bswap(hs[1]), bswap(hs[2]), bswap(hs[3]));
                    o[1] = make_uint4(bswap(hs[4]), bswap(hs[5]), bswap(hs[6]), bswap(hs[7]));
                }
            } else if (st) {
#pragma unroll
                for (int i = 0; i < 8; ++i) st[mi].sha[i] = hs[i];
                st[mi].prior_bytes = prior + L;
                st[mi].reserved = 0;
            }
        }
    } else {
        // ----------------------------------------------------------------------------------- MD5 chain
        if (!DO_MD5) return;
        uint32_t hm[4] = {0x67452301u, 0xefcdab89u, 0x98badcfeu, 0x10325476u};
        if (resume && lane == 0) {
#pragma unroll
            for (int i = 0; i < 4; ++i) hm[i] = st[mi].md5[i];
        }
        for (uint64_t t = 0; t < t_all; ++t) {
            const uint32_t slot = (uint32_t)(t % kNT);
            const uint32_t nb = blocks_in(t);
            const uint32_t toff = t < t_data ? mis : 0u;
            mbar_wait(tile_full + 8 * slot, (uint32_t)((t / kNT) & 1));
            if (lane == 0) {
#pragma unroll 1
                for (uint32_t bidx = 0; bidx < nb; ++bidx) {
                    uint32_t x[16];
                    load_block_words(tiles + slot * kTileStride + bidx * 64, toff, x);
                    md5_chain_block(hm, x, one);
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(tile_free + 8 * slot);
        }
        if (lane == 0) {
            if (final) {
                if (md5_out) *reinterpret_cast<uint4*>(md5_out + 16ull * mi) = make_uint4(hm[0], hm[1], hm[2], hm[3]);
            } else if (st) {
#pragma unroll
                for (int i = 0; i < 4; ++i) st[mi].md5[i] = hm[i];
                if (!DO_SHA) {
                    st[mi].prior_bytes = prior + L;
                    st[mi].reserved = 0;
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------ trim kernels
// Reference semantics (blob_utils.py:667-705): index just past the last non-zero byte, 0 when the
// message is empty or all zero.  Two kernels:
//   trim_probe_kernel  one warp per message scanning backwards from the end, 2 KiB (4 x 16 B per lane) per step.
//                      Most messages end in a non-zero byte and are settled by the first step, so the common case
//                      reads <= 2 KiB per message.  A message that is still all zero after kTrimProbeSteps steps
//                      with >= kTrimWideMin bytes left is handed to the wide scan: its remaining range is cut into
//                      kTrimChunk-byte work items (nearest the end first) appended to a device-side list.
//   trim_wide_kernel   persistent CTAs pull those items from a counter; a CTA scans its chunk backwards 32 KiB per
//                      step (256 threads x 8 x 16 B in flight), publishes what it finds with atomicMax on
//                      trimmed[m] and gives up as soon as a later chunk of the same message has found a byte.
//                      Long zero runs (blank volumefs2 blocks, sparse files) are therefore read by every SM at once
//                      -- this is the one HBM-bound kernel on the path -- instead of by one warp walking 2 KiB per
//                      dependent step (~1 280 warps x 2 KiB in flight for 1 280 blank 8 MiB blocks).

constexpr int kTrimProbeSteps = 8;              // 16 KiB settled by the probe warp before a message goes wide
constexpr uint64_t kTrimWideMin = 256 * 1024;   // shorter remainders stay on the probe warp
constexpr uint64_t kTrimChunk = 512 * 1024;     // bytes per wide work item (multiple of the 32 KiB step)
constexpr int kTrimWideThreads = 256;
constexpr int kTrimWideLoads = 8;               // 16-byte loads in flight per thread
constexpr int kTrimWideCtasPerSm = 4;           // 64 registers per thread; 4 x 32 KiB in flight per SM
constexpr uint64_t kTrimWideStep = (uint64_t)kTrimWideThreads * kTrimWideLoads * 16;

// 1 + index (within the message, `pos` = index of the granule's first byte) of the last non-zero byte of a 16-byte
// granule, 0 if it is all zero
__device__ __forceinline__ uint64_t granule_last_nonzero(const uint4& v, uint64_t pos) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint64_t best = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q)
        if (w[q]) best = pos + 4 * q + (4 - (__clz(w[q]) >> 3));
    return best;
}

__global__ void __launch_bounds__(256)
trim_probe_kernel(const uint8_t* __restrict__ base, const uint64_t* __restrict__ off, const uint64_t* __restrict__ len,
                  uint64_t n, uint64_t* __restrict__ trimmed, unsigned long long* __restrict__ wctl,
                  TrimWideEntry* __restrict__ wlist) {
    const int lane = threadIdx.x & 31;
    const uint64_t warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t m = (((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5); m < n; m += warps) {
        const uint8_t* p = base + off[m];
        uint64_t end = len[m];
        uint64_t found = 0;  // 1 + index of last non-zero byte
        // unaligned tail bytes first so the bulk of the scan runs on 16B-aligned granules
        const uint64_t a_end = (reinterpret_cast<uintptr_t>(p) + end) & 15u;  // bytes past the last aligned boundary
        uint64_t tail = a_end < end ? a_end : end;
        {
            uint32_t hit = 0;
            if ((uint64_t)lane < tail && p[end - 1 - lane] != 0) hit = 1;  // lane 0 = last byte
            const uint32_t mask = __ballot_sync(0xffffffffu, hit);
            if (mask) found = end - (uint64_t)(__ffs(mask) - 1);
            end -= tail;
        }
        int steps = 0;
        bool wide = false;
        while (!found && end >= 16) {
            if (steps == kTrimProbeSteps && end >= kTrimWideMin) {
                wide = true;
                break;
            }
            ++steps;
            // granules [end-16*(k+1), end-16*k) for k = lane + 32*u, u = 0..3 (nearest the end first)
            uint4 v[4];
            uint64_t pos[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const uint64_t k = (uint64_t)lane + 32u * u;
                const bool ok = 16 * (k + 1) <= end;  // p + end is 16B-aligned here
                pos[u] = ok ? end - 16 * (k + 1) : 0;
                v[u] = ok ? __ldcs(reinterpret_cast<const uint4*>(p + pos[u])) : make_uint4(0, 0, 0, 0);
            }
            uint64_t best = 0;
#pragma unroll
            for (int u = 3; u >= 0; --u) {
                const uint64_t cand = granule_last_nonzero(v[u], pos[u]);
                best = cand > best ? cand : best;
            }
            best = warp_max_u64(best);
            if (best) found = best;
            const uint64_t whole = end & ~15ull;
            end -= whole < 2048 ? whole : 2048;
        }
        if (wide) {
            // [0, end) is still unknown and p + end is 16-byte aligned: cut it into chunks, nearest the end first.
            // One 64-bit atomic reserves the list slot (high word) and the item range (low word) together, so the
            // list is sorted by first item and the wide kernel can binary-search it.
            if (lane == 0) {
                const uint64_t k = (end + kTrimChunk - 1) / kTrimChunk;
                const unsigned long long old = atomicAdd(&wctl[0], (1ull << 32) | (unsigned long long)k);
                TrimWideEntry e;
                e.msg = m;
                e.end = end;
                e.first_item = (uint32_t)old;
                e.items = (uint32_t)k;
                wlist[old >> 32] = e;
                trimmed[m] = 0;  // the answer if everything left is zero; raised by atomicMax in the wide kernel
            }
            continue;
        }
        if (!found && end > 0 && end < 16) {
            // fewer than 16 bytes remain at the (unaligned) head of the message
            uint32_t hit = 0;
            if ((uint64_t)lane < end && p[end - 1 - lane] != 0) hit = 1;
            const uint32_t mask = __ballot_sync(0xffffffffu, hit);
            if (mask) found = end - (uint64_t)(__ffs(mask) - 1);
        }
        if (lane == 0) trimmed[m] = found;
    }
}

__device__ __forceinline__ unsigned long long ld_volatile_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

__global__ void __launch_bounds__(kTrimWideThreads, kTrimWideCtasPerSm)
trim_wide_kernel(const uint8_t* __restrict__ base, const uint64_t* __restrict__ off, uint64_t* __restrict__ trimmed,
                 unsigned long long* __restrict__ wctl, const TrimWideEntry* __restrict__ wlist) {
    __shared__ uint32_t sh_item;
    __shared__ uint64_t sh_best[kTrimWideThreads / 32];
    const unsigned long long ctl = wctl[0];  // written by the probe kernel (earlier in the stream)
    const uint32_t total = (uint32_t)ctl, entries = (uint32_t)(ctl >> 32);
    if (!total) return;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    unsigned long long* best_of = reinterpret_cast<unsigned long long*>(trimmed);
    for (;;) {
        __syncthreads();  // sh_item / sh_best of the previous item are no longer read
        if (tid == 0) sh_item = (uint32_t)atomicAdd(&wctl[1], 1ull);
        __syncthreads();
        const uint32_t item = sh_item;
        if (item >= total) return;
        // entry with the largest first_item <= item
        uint32_t lo = 0, hi = entries;
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (wlist[mid].first_item <= item) lo = mid;
            else hi = mid;
        }
        const TrimWideEntry e = wlist[lo];
        const uint64_t j = item - e.first_item;              // 0 = the chunk nearest the end
        const uint64_t c_hi = e.end - j * kTrimChunk;         // p + c_hi is 16-byte aligned
        const uint64_t c_lo = c_hi > kTrimChunk ? c_hi - kTrimChunk : 0;
        const uint8_t* p = base + off[e.msg];
        // aligned part of the chunk: [a_lo, c_hi); the < 16 unaligned head bytes [0, a_lo) exist only when c_lo == 0
        // p + c_hi is aligned, so p & 15 == (-c_hi) & 15 and the bytes before the first aligned address number c_hi & 15
        const uint64_t head = c_lo ? 0 : (c_hi & 15u);
        const uint64_t a_lo = c_lo + head;
        uint64_t cur = c_hi;
        uint64_t found = 0;
        bool superseded = false;
        while (cur > a_lo) {
            uint4 v[kTrimWideLoads];
            uint64_t pos[kTrimWideLoads];
#pragma unroll
            for (int u = 0; u < kTrimWideLoads; ++u) {
                const uint64_t k = (uint64_t)tid + (uint64_t)kTrimWideThreads * u;
                const bool ok = cur >= a_lo + 16 * (k + 1);
                pos[u] = ok ? cur - 16 * (k + 1) : 0;
                v[u] = ok ? __ldcs(reinterpret_cast<const uint4*>(p + pos[u])) : make_uint4(0, 0, 0, 0);
            }
            uint64_t best = 0;
#pragma unroll
            for (int u = 0; u < kTrimWideLoads; ++u) {
                const uint64_t cand = granule_last_nonzero(v[u], pos[u]);
                best = cand > best ? cand : best;
            }
            // a later chunk of this message already holds a non-zero byte: nothing in here can matter
            const bool stale = tid == 0 && ld_volatile_u64(&best_of[e.msg]) > c_hi;
            const int flags = __syncthreads_or((best ? 1 : 0) | (stale ? 2 : 0));
            if (flags & 2) {
                superseded = true;
                break;
            }
            if (flags & 1) {
                best = warp_max_u64(best);
                if (lane == 0) sh_best[wid] = best;
                __syncthreads();
                if (tid == 0) {
                    uint64_t b = 0;
                    for (int w = 0; w < kTrimWideThreads / 32; ++w) b = sh_best[w] > b ? sh_best[w] : b;
                    found = b;
                }
                break;
            }
            const uint64_t span = cur - a_lo;
            cur -= span < kTrimWideStep ? span : kTrimWideStep;
        }
        if (tid == 0) {
            if (!found && !superseded && head) {
                // the unaligned first bytes of the message
                for (uint64_t i = head; i > 0; --i)
                    if (p[i - 1]) {
                        found = i;
                        break;
                    }
            }
            if (found) atomicMax(&best_of[e.msg], (unsigned long long)found);
        }
    }
}

// ------------------------------------------------------------------------------------ plan kernels
// Bucket key: exact block count below 16, then 8 sub-buckets per power of two (<= 12.5 % spread inside
// a bucket, so lanes of a warp run nearly equal trip counts).  Buckets are laid out longest first.

__host__ __device__ __forceinline__ int plan_log2_u64(uint64_t v) {  // floor(log2 v), v > 0
#ifdef __CUDA_ARCH__
    return 63 - __clzll((long long)v);
#else
    return 63 - __builtin_clzll(v);
#endif
}

__host__ __device__ __forceinline__ uint32_t plan_bucket(uint64_t len) {
    const uint64_t nb = (len >> 6) + 1;
    if (nb < 16) return (uint32_t)nb;
    const int e = plan_log2_u64(nb);
    const uint32_t b = 16u + (uint32_t)(e - 4) * 8u + (uint32_t)((nb >> (e - 3)) & 7u);
    return b < (uint32_t)kPlanBuckets ? b : (uint32_t)kPlanBuckets - 1;
}

// smallest block count that maps to bucket b (inverse of plan_bucket)
__host__ __device__ __forceinline__ uint64_t plan_bucket_min_blocks(uint32_t b) {
    if (b < 16) return b;
    const uint32_t e = (b - 16) / 8 + 4, mant = (b - 16) % 8;
    if (e - 3 >= 60) return ~0ull;  // buckets no 64-bit length can reach: saturate instead of wrapping around
    return (uint64_t)(8 + mant) << (e - 3);
}

// Rule (3) of the chain selection, shared by the planner kernel and its host mirror.
//   count          messages that satisfy rules (1) and (2)
//   chain_blocks   lower bound of their 64-byte blocks (bucket lower bounds x bucket counts; buckets are 12.5 % wide)
// Chain CTAs and lane CTAs that share an SM slow each other down badly (one rank's share of C3-v2 with
// its 1..4 MiB blocks on chains spread over every SM took more than twice as long as with all of them on lanes).  So:
//   * up to 3/4 of the SMs' worth of outliers get an SM each, which the lane kernel then leaves alone (F_YIELD_CHAIN_SMS);
//   * more than that only when (almost) nothing is left for the lanes -- a batch of equally long messages, where the
//     chain kernel runs by itself at up to max_chain chains (4 per SM);
//   * otherwise none.
__host__ __device__ __forceinline__ uint32_t plan_chain_count(uint32_t count, unsigned long long chain_blocks,
                                                             unsigned long long total_blocks, uint32_t n, uint32_t max_chain,
                                                             uint32_t sm_count) {
    if (count == 0 || count > max_chain) return 0u;  // all of them or none
    if (count <= sm_count * 3 / 4) return count;
    if (count == n) return count;
    const unsigned long long rest = total_blocks > chain_blocks ? total_blocks - chain_blocks : 0ull;
    return rest <= total_blocks / 4 ? count : 0u;
}

// The LONG lane messages: those that satisfy rule (1) -- each would still be running on its lane after the rest of the
// batch is done -- but stay on lanes (not routed to chains).  In one launch the time slicing scatters them one per warp
// over the whole grid, and the tail then runs ~2 000 warps with a single live lane each (one rank's share of C3-v2: its
// 1..4 MiB blocks alone, lane-packed, take about half the time of the whole mixed launch).  So they get
// their own queue and a second, lane-packed launch behind the short ones.  count1 = messages satisfying rule (1).
__host__ __device__ __forceinline__ uint32_t plan_long_count(uint32_t count1, uint32_t chain, uint32_t n, uint32_t long_cap) {
    const uint32_t nl = count1 > chain ? count1 - chain : 0u;
    if (nl == 0 || nl > long_cap) return 0u;     // too many to be lane-packed one wave deep: one launch as before
    if (nl == n - chain) return 0u;              // nothing but long messages on the lanes: a single (packed) launch anyway
    return nl;
}

// Host mirror of plan_hist_kernel + plan_scan_kernel's chain selection: how many of these messages the planner will
// hand to the chain kernel.  Same integer arithmetic on the same lengths, so the answer is the device's; callers
// that hold the lengths on the host use it to size the chain launch WITHOUT reading qctl[3] back (no stream
// synchronisation inside an enqueue).  B200H_VERIFY_PLAN=1 makes the API cross-check it against the device.
uint32_t plan_outliers_host(const uint64_t* len, uint64_t n, uint32_t max_chain, uint32_t sm_count, uint32_t long_cap,
                            uint32_t ratio8, uint32_t* n_long_out) {
    *n_long_out = 0;
    if (!n) return 0;
    uint64_t longest = 0;
    unsigned long long total = 0;
    for (uint64_t i = 0; i < n; ++i) {
        longest = len[i] > longest ? len[i] : longest;
        total += (len[i] >> 6) + 1;
    }
    if ((longest >> 6) + 1 < kChainMinBlocks) return 0;  // nothing can reach rule (1)
    unsigned long long thr = total / kChainRatio;
    if (thr < kChainMinBlocks) thr = kChainMinBlocks;
    const unsigned long long thr1 = thr;  // rule (1) alone
    const uint32_t top = plan_bucket(longest);
    const unsigned long long half = plan_bucket_min_blocks(top) / 8 * ratio8;
    if (thr < half) thr = half;
    // messages in buckets whose lower bound reaches thr (bucket lower bounds are monotone in the bucket index)
    uint64_t count = 0, count1 = 0;
    unsigned long long chain_blocks = 0;
    for (uint64_t i = 0; i < n; ++i) {
        const uint64_t lb = plan_bucket_min_blocks(plan_bucket(len[i]));
        if (lb >= thr1) ++count1;
        if (lb >= thr) {
            ++count;
            chain_blocks += lb;
        }
    }
    const uint32_t c = (max_chain && count <= max_chain)
                           ? plan_chain_count((uint32_t)count, chain_blocks, total, (uint32_t)n, max_chain, sm_count) : 0u;
    *n_long_out = plan_long_count((uint32_t)count1, c, (uint32_t)n, long_cap);
    return c;
}

__global__ void plan_hist_kernel(const uint64_t* __restrict__ len, uint64_t n, uint32_t* __restrict__ hist,
                                 unsigned long long* __restrict__ total_blocks) {
    __shared__ uint32_t sh[kPlanBuckets];
    __shared__ unsigned long long sh_total;
    for (int i = threadIdx.x; i < kPlanBuckets; i += blockDim.x) sh[i] = 0;
    if (threadIdx.x == 0) sh_total = 0;
    __syncthreads();
    unsigned long long mine = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t l = len[i];
        mine += (l >> 6) + 1;
        atomicAdd(&sh[plan_bucket(l)], 1u);
    }
    atomicAdd(&sh_total, mine);
    __syncthreads();
    for (int i = threadIdx.x; i < kPlanBuckets; i += blockDim.x)
        if (sh[i]) atomicAdd(&hist[i], sh[i]);
    if (threadIdx.x == 0 && sh_total) atomicAdd(total_blocks, sh_total);
}

// hist[0..B) counts -> cursor[0..B) start positions, longest bucket first; also decides how many of the
// longest messages leave the lane queue for the chain kernel.  Single CTA of kPlanBuckets threads.
//
// Chain selection.  One chain on the chain kernel runs ~2x faster than on a lane (the
// one-warp issue limit of 0.5 instr/clk applied to 1 056 instead of 2 108 instructions per block), but a chain CTA
// serves ONE message with three warps where a lane-kernel warp serves 32, and the two kernels slow each other
// down while they share SMSPs.  So only true outliers go there -- the messages that would still be running on
// their lane after everything else has finished:
//   (1) longer than the whole batch takes on the saturated lane kernel (block count > total_blocks / kChainRatio)
//       and long enough for the tile pipeline to pay off (kChainMinBlocks);
//   (2) longer than half the longest message (anything shorter finishes on a lane before the longest one
//       finishes on the chain kernel);
//   (3) and only if ALL such messages fit (count <= max_chain, one CTA per SM): routing a part of a set of
//       equally long messages leaves the makespan where it was and costs the interference (2048 x 4 MiB with one
//       SM's worth of them moved over took twice as long).
// qctl = {lane entries available, head, tail, chain count}.
__global__ void plan_scan_kernel(const uint32_t* __restrict__ hist, uint32_t* __restrict__ cursor, int* __restrict__ qctl,
                                 const unsigned long long* __restrict__ total_blocks, uint32_t n, uint32_t max_chain,
                                 uint32_t sm_count, uint32_t long_cap, uint32_t ratio8) {
    __shared__ uint32_t sh[kPlanBuckets];
    __shared__ uint32_t sh_chain, sh_top, sh_count1;
    __shared__ unsigned long long sh_chain_blocks;
    const int t = threadIdx.x;
    if (t == 0) {
        sh_chain = 0;
        sh_top = 0;
        sh_chain_blocks = 0;
        sh_count1 = 0;
    }
    const int rev = kPlanBuckets - 1 - t;  // position in longest-first order
    sh[t] = hist[rev];
    __syncthreads();
    for (int o = 1; o < kPlanBuckets; o <<= 1) {
        uint32_t v = t >= o ? sh[t - o] : 0u;
        __syncthreads();
        sh[t] += v;
        __syncthreads();
    }
    cursor[rev] = sh[t] - hist[rev];  // exclusive
    unsigned long long thr = *total_blocks / kChainRatio;
    if (thr < kChainMinBlocks) thr = kChainMinBlocks;
    {   // rule (1) alone: everything at least this long is a "long" message (chain or long lane queue)
        const bool mine1 = plan_bucket_min_blocks((uint32_t)rev) >= thr;
        const bool next1 = rev > 0 && plan_bucket_min_blocks((uint32_t)rev - 1) >= thr;
        if (mine1 && !next1) atomicMax(&sh_count1, sh[t]);
    }
    // longest non-empty bucket -> rule (2); buckets are 12.5 % wide, compare on their lower bounds
    if (hist[rev]) atomicMax(&sh_top, (uint32_t)rev);
    __syncthreads();
    // rule (2): "longer than ratio8/8 of the longest" -- what stays on a lane must finish there before the longest
    // message finishes on its chain: lane speed / chain speed is about 3/8 for the fused digests and 4/8 for SHA-256 /
    // MD5 alone (the one-warp issue limit applied to each kernel's instruction count per block).
    const unsigned long long half = plan_bucket_min_blocks(sh_top) / 8 * ratio8;
    if (thr < half) thr = half;
    const bool mine = plan_bucket_min_blocks((uint32_t)rev) >= thr;
    const bool next = rev > 0 && plan_bucket_min_blocks((uint32_t)rev - 1) >= thr;
    if (mine && !next) atomicMax(&sh_chain, sh[t]);  // inclusive count of everything at least this long
    if (mine && hist[rev]) atomicAdd(&sh_chain_blocks, (unsigned long long)hist[rev] * plan_bucket_min_blocks((uint32_t)rev));
    __syncthreads();
    if (t == 0) {
        const uint32_t c = max_chain ? plan_chain_count(sh_chain, sh_chain_blocks, *total_blocks, n, max_chain, sm_count) : 0u;
        const uint32_t nl = plan_long_count(sh_count1, c, n, long_cap);
        qctl[0] = (int)(n - c - nl);  // lane-queue entries available (the short messages)
        qctl[1] = 0;                  // head ticket
        qctl[2] = (int)(n - c - nl);  // tail ticket
        qctl[3] = (int)c;             // messages handed to the chain kernel
        int* ql = qctl + kLongQctlAfterQctl;  // the long lane messages: their own queue
        ql[0] = (int)nl;
        ql[1] = 0;
        ql[2] = (int)nl;
        ql[3] = (int)nl;
        // qctl[4..5] hold total_blocks; [6] = chain CTAs the lane kernel may wait for, [7] = chain CTAs that started
        qctl[kChainExpectedWord] = (int)(c <= sm_count * 3 / 4 ? c : 0u);
        qctl[kChainStartedWord] = 0;
    }
}

__global__ void plan_scatter_kernel(const uint64_t* __restrict__ len, uint64_t n, uint32_t* __restrict__ cursor,
                                    uint32_t* __restrict__ ring, uint32_t* __restrict__ ring_long,
                                    uint32_t* __restrict__ chain_list, const int* __restrict__ qctl, uint32_t tag) {
    const uint32_t nchain = (uint32_t)qctl[3];
    const uint32_t nlong = (uint32_t)qctl[kLongQctlAfterQctl + 3];
    // warp-aggregated atomics: lanes hitting the same bucket share one atomicAdd
    for (uint64_t i0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) & ~31ull; i0 < n;
         i0 += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t i = i0 + (threadIdx.x & 31);
        const bool ok = i < n;
        const uint32_t b = ok ? plan_bucket(len[i]) : 0xffffffffu;
        const uint32_t peers = __match_any_sync(0xffffffffu, b);
        const int leader = __ffs(peers) - 1;
        uint32_t basepos = 0;
        if (ok && (threadIdx.x & 31) == leader) basepos = atomicAdd(&cursor[b], (uint32_t)__popc(peers));
        basepos = __shfl_sync(0xffffffffu, basepos, leader);
        if (ok) {
            const uint32_t pos = basepos + __popc(peers & ((1u << (threadIdx.x & 31)) - 1u));
            if (pos < nchain) chain_list[pos] = (uint32_t)i;
            else if (pos < nchain + nlong) ring_long[pos - nchain] = (uint32_t)i | tag;
            else ring[pos - nchain - nlong] = (uint32_t)i | tag;
        }
    }
}

// ------------------------------------------------------------------------------- utility kernels

__device__ __forceinline__ uint64_t mix64(uint64_t z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// dst[0..nbytes) = bytes [start, start+nbytes) of synthetic stream `seed` (see modal_client_b200/synth.py).
// dst must be 8-byte aligned and start a multiple of 8; the last partial word is written bytewise.
__global__ void fill_synth_kernel(uint8_t* __restrict__ dst, uint64_t nbytes, uint64_t seed_mul, uint64_t word0) {
    const uint64_t nwords = nbytes >> 3;
    uint64_t* d64 = reinterpret_cast<uint64_t*>(dst);
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= nwords;
         i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t v = mix64(seed_mul + word0 + i);
        if (i < nwords) {
            d64[i] = v;
        } else {
            for (uint64_t b = 0; b < (nbytes & 7); ++b) dst[8 * nwords + b] = (uint8_t)(v >> (8 * b));
        }
    }
}

// Lowercase hex of a byte table (the wire form of MountFile.sha256_hex / md5_hex, modal_proto/api.proto:2582-2587):
// one thread turns 4 digest bytes into 8 ASCII characters, so a whole digest column leaves the device already in
// the form the RPC rows carry.  nbytes is a multiple of 16 (whole rows).
__global__ void hex_rows_kernel(const uint32_t* __restrict__ in, uint64_t nwords, uint2* __restrict__ out) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nwords; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t w = in[i];  // bytes b0..b3 little-endian
        uint32_t o[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            uint32_t acc = 0;
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const uint32_t b = (w >> (16 * h + 8 * k)) & 0xffu;
                const uint32_t hi = b >> 4, lo = b & 15u;
                const uint32_t ch = (hi < 10 ? hi + 48u : hi + 87u), cl = (lo < 10 ? lo + 48u : lo + 87u);
                acc |= (ch | (cl << 8)) << (16 * k);
            }
            o[h] = acc;
        }
        out[i] = make_uint2(o[0], o[1]);
    }
}

static int g_sm_count = 132;  // set from the device by configure_kernels()

int device_sm_count() { return g_sm_count; }

int launch_hex_rows(const uint8_t* in, uint64_t nbytes, uint8_t* out, cudaStream_t st) {
    if (!nbytes) return 0;
    const uint64_t nwords = nbytes / 4;
    uint64_t g = (nwords + 255) / 256;
    if (g > (uint64_t)g_sm_count * 16) g = (uint64_t)g_sm_count * 16;
    hex_rows_kernel<<<(int)g, 256, 0, st>>>(reinterpret_cast<const uint32_t*>(in), nwords, reinterpret_cast<uint2*>(out));
    return 1;
}

// One tile of gather_segments_kernel: dst[0..len) = src[0..len), V-wide where both pointers agree mod sizeof(V).
// The bytes before dst's first V boundary and after the last whole V go one at a time.
template <typename V>
__device__ __forceinline__ void copy_tile(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, uint32_t len) {
    constexpr uint32_t W = sizeof(V);
    const uint32_t head = min(len, (uint32_t)((W - ((uintptr_t)dst & (W - 1))) & (W - 1)));
    const uint32_t nv = (len - head) / W;
    for (uint32_t i = threadIdx.x; i < head; i += blockDim.x) dst[i] = src[i];
    const V* sv = reinterpret_cast<const V*>(src + head);
    V* dv = reinterpret_cast<V*>(dst + head);
    for (uint32_t i = threadIdx.x; i < nv; i += blockDim.x) dv[i] = sv[i];
    for (uint32_t i = head + nv * W + threadIdx.x; i < len; i += blockDim.x) dst[i] = src[i];
}

// Copies the pieces of the parts that straddle segments into a wave slot (b200h_hash_segment_parts_device): one CTA
// per tile at a time.  The widest access both addresses allow: 16 bytes when source and destination agree mod 16
// (the destination of a part's first piece always is 16-byte aligned), down to single bytes.
__global__ void __launch_bounds__(256) gather_segments_kernel(const GatherTile* __restrict__ tiles, uint64_t ntiles) {
    for (uint64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const GatherTile g = tiles[t];
        const uint8_t* src = reinterpret_cast<const uint8_t*>(g.src);
        uint8_t* dst = reinterpret_cast<uint8_t*>(g.dst);
        const uint32_t len = (uint32_t)g.len;
        const uint32_t phase = (uint32_t)(g.src ^ g.dst);
        if (!(phase & 15u)) copy_tile<uint4>(src, dst, len);
        else if (!(phase & 7u)) copy_tile<uint2>(src, dst, len);
        else if (!(phase & 3u)) copy_tile<uint32_t>(src, dst, len);
        else if (!(phase & 1u)) copy_tile<uint16_t>(src, dst, len);
        else copy_tile<uint8_t>(src, dst, len);
    }
}

int launch_gather_segments(const GatherTile* tiles, uint64_t ntiles, cudaStream_t st) {
    if (!ntiles) return 0;
    const uint64_t g = ntiles < (uint64_t)g_sm_count * 16 ? ntiles : (uint64_t)g_sm_count * 16;
    gather_segments_kernel<<<(int)g, 256, 0, st>>>(tiles, ntiles);
    return 1;
}

// --------------------------------------------------------------------------------- launch wrappers

static int grid_for(uint64_t n, int threads, int cap) {
    uint64_t g = (n + threads - 1) / threads;
    if (g < 1) g = 1;
    return (int)(g > (uint64_t)cap ? (uint64_t)cap : g);
}

int launch_trim(const uint8_t* base, const uint64_t* off, const uint64_t* len, uint64_t n, uint64_t* trimmed,
                unsigned long long* wctl, TrimWideEntry* wlist, cudaStream_t st) {
    if (!n) return 0;
    cudaMemsetAsync(wctl, 0, 2 * sizeof(unsigned long long), st);
    trim_probe_kernel<<<grid_for(n * 32, 256, g_sm_count * 8), 256, 0, st>>>(base, off, len, n, trimmed, wctl, wlist);
    trim_wide_kernel<<<g_sm_count * kTrimWideCtasPerSm, kTrimWideThreads, 0, st>>>(base, off, trimmed, wctl, wlist);
    return 2;
}


// [sha+md5, sha, md5]; configure_kernels() replaces them with the occupancy the compiled kernels reach
static int g_lane_ctas_per_sm[3] = {lane_ctas_per_sm<true, true, false>(), lane_ctas_per_sm<true, false, false>(),
                                    lane_ctas_per_sm<false, true, false>()};

// most long messages a second, lane-packed launch takes: one wave of lanes at one warp per SMSP
uint32_t plan_long_cap() {
    const uint32_t cap = (uint32_t)g_sm_count * 4u * 32u;
    return cap < kLongRingCapacity ? cap : kLongRingCapacity;
}

uint32_t ring_capacity(uint64_t n) {
    uint32_t cap = 32;
    while (cap < n) cap <<= 1;
    return cap;
}

// Builds the work lists: chain_list[0..c) = the c longest outlier messages (see plan_scan_kernel) for the chain
// kernel; ring[0..n-c) = the rest, bucketed longest-first (tagged FRESH unless the batch resumes from
// caller-provided chaining states), ring[n-c..cap) = EMPTY; qctl = {n-c, 0, n-c, c}.
int launch_plan(const uint64_t* len, uint64_t n, uint32_t* ring, uint32_t* ring_long, uint32_t* chain_list, uint32_t* scratch,
                bool fresh, uint32_t max_chain, uint32_t ratio8, cudaStream_t st) {
    const uint32_t sm_count = (uint32_t)g_sm_count;
    if (!n) return 0;
    uint32_t* hist = scratch;
    uint32_t* cursor = scratch + kPlanBuckets;
    int* qctl = plan_qctl(scratch);
    unsigned long long* total = reinterpret_cast<unsigned long long*>(scratch + 2 * kPlanBuckets + 4);
    cudaMemsetAsync(hist, 0, sizeof(uint32_t) * kPlanBuckets, st);
    cudaMemsetAsync(reinterpret_cast<uint32_t*>(qctl) + kSmFlagsAfterQctl, 0, sizeof(uint32_t) * kSmFlagWords, st);
    cudaMemsetAsync(total, 0, sizeof(unsigned long long), st);
    cudaMemsetAsync(ring, 0xff, sizeof(uint32_t) * ring_capacity(n), st);
    if (ring_long) cudaMemsetAsync(ring_long, 0xff, sizeof(uint32_t) * kLongRingCapacity, st);
    plan_hist_kernel<<<grid_for(n, 256, g_sm_count * 4), 256, 0, st>>>(len, n, hist, total);
    plan_scan_kernel<<<1, kPlanBuckets, 0, st>>>(hist, cursor, qctl, total, (uint32_t)n, max_chain, sm_count,
                                                 ring_long ? plan_long_cap() : 0u, ratio8);
    plan_scatter_kernel<<<grid_for(n, 256, g_sm_count * 4), 256, 0, st>>>(len, n, cursor, ring, ring_long, chain_list, qctl,
                                                                fresh ? kFresh : 0u);
    return 3;
}

// One CTA per chain-list entry; the grid is sized for the cap and surplus CTAs exit at once (the count lives
// on the device, in qctl[3]).
int launch_chain_hash(const uint8_t* base, const uint64_t* off, const uint64_t* len, const uint32_t* chain_list,
                      const int* qctl, uint32_t flags, uint8_t* sha_out, uint8_t* md5_out, ChainState* state,
                      bool resume, uint32_t n_chain, cudaStream_t st) {
    const bool s = flags & F_SHA256, m = flags & F_MD5;
    // n_chain live entries (read back from the planner): entry e -> CTA e % grid, group e / grid; one CTA per SM
    const uint32_t live = n_chain < kMaxChain ? n_chain : kMaxChain;
    const int grid = (int)(live < (uint32_t)g_sm_count ? live : (uint32_t)g_sm_count);
    if (grid <= 0) return 0;
    const int groups = (int)((live + grid - 1) / grid) <= kChainGroups ? kChainGroups : kChainGroupsMax;
    const int threads = kChainGroupThreads * groups, smem = chain_smem_bytes(groups);
#define CHAIN_LAUNCH(S_, M_)                                                                                          \
    do {                                                                                                              \
        if (groups == kChainGroups)                                                                                   \
            chain_hash_kernel<S_, M_, kChainGroups><<<grid, threads, smem, st>>>(base, off, len, chain_list, qctl, flags, \
                                                                                 sha_out, md5_out, state, resume, 1u);  \
        else                                                                                                          \
            chain_hash_kernel<S_, M_, kChainGroupsMax><<<grid, threads, smem, st>>>(base, off, len, chain_list, qctl,  \
                                                                                    flags, sha_out, md5_out, state,   \
                                                                                    resume, 1u);                      \
    } while (0)
    if (s && m) CHAIN_LAUNCH(true, true);
    else if (s) CHAIN_LAUNCH(true, false);
    else if (m) CHAIN_LAUNCH(false, true);
#undef CHAIN_LAUNCH
    else
        return 0;
    return 1;
}

template <bool S, bool M, bool SP>
static void launch_lane_t(int grid, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint32_t* ring,
                          uint32_t ring_mask, int* qctl, const int* ctl, uint32_t flags, int lpw, uint32_t quantum,
                          uint8_t* sha_out, uint8_t* md5_out, ChainState* state, cudaStream_t st) {
    lane_hash_kernel<S, M, SP><<<grid, kLaneThreads, kLaneSmem, st>>>(base, off, len, ring, ring_mask, qctl, ctl, flags, lpw,
                                                                quantum, sha_out, md5_out, state, 1u);
}

// Persistent launch: at most one resident wave of CTAs; lanes pull messages from the queue until it drains.
// When the batch has fewer messages than resident lanes, messages are spread one-per-warp first
// (lanes_per_warp < 32) so that every chain gets its own issue slots.
int launch_lane_hash(const uint8_t* base, const uint64_t* off, const uint64_t* len, uint32_t* ring, uint32_t ring_entries,
                     int* qctl, const int* ctl, uint64_t n, uint32_t flags, uint8_t* sha_out, uint8_t* md5_out,
                     ChainState* state, cudaStream_t st) {
    if (!n) return 0;
    // Lane packing.  A warp costs the same issue slots whether 1 or 32 of its lanes carry a message, and
    // one warp alone on an SMSP is latency-bound (~0.27 IPC; measured), so: fill lanes first, but never use
    // fewer warps than there are SMSPs (4 per SM) and never more than fit resident.
    const bool want_sha = flags & F_SHA256, want_md5 = flags & F_MD5;
    const int variant = want_sha ? (want_md5 ? 0 : 1) : 2;
    const uint64_t resident_warps = (uint64_t)g_sm_count * g_lane_ctas_per_sm[variant] * kLaneWarps;
    const uint64_t min_warps = (uint64_t)g_sm_count * 4;
    uint64_t warps = (n + 31) / 32;
    if (warps < min_warps) warps = n < min_warps ? n : min_warps;
    if (warps > resident_warps) warps = resident_warps;
    int lpw = (int)((n + warps - 1) / warps);
    if (lpw > 32) lpw = 32;
    const int grid = (int)((warps + kLaneWarps - 1) / kLaneWarps);
    // Leaving chain SMs is only safe when the grid fills every SM (a full resident wave): then CTAs on the chain-free
    // SMs are guaranteed to exist and pull the work.  A small grid (a handful of CTAs, or one per SM) could land entirely
    // on chain SMs and strand its messages -- a lone 123-byte multipart tail next to five 1 MiB parts did exactly that.
    if (warps < resident_warps) flags &= ~F_YIELD_CHAIN_SMS;
    const uint32_t mask = ring_entries - 1;
    static const uint32_t quantum = [] {
        const char* e = getenv("B200H_QUANTUM");  // tuning knob (blocks per time slice)
        const long v = e ? atol(e) : 0;
        return (uint32_t)(v > 0 ? v : 32);
    }();
    const bool s = flags & F_SHA256, m = flags & F_MD5;
    // every warp alone on its SMSP -> the minimum-instruction instantiation (SHA-256 kernels; MD5 alone is latency bound)
    const bool sparse = warps <= min_warps && getenv("B200H_NO_SPARSE") == nullptr;
#define LANE_ARGS grid, base, off, len, ring, mask, qctl, ctl, flags, lpw, quantum, sha_out, md5_out, state, st
    if (s && m) {
        if (sparse) launch_lane_t<true, true, true>(LANE_ARGS);
        else launch_lane_t<true, true, false>(LANE_ARGS);
    } else if (s) {
        if (sparse) launch_lane_t<true, false, true>(LANE_ARGS);
        else launch_lane_t<true, false, false>(LANE_ARGS);
    } else if (m) {
        launch_lane_t<false, true, false>(LANE_ARGS);
    }
#undef LANE_ARGS
    else return 0;
    return 1;
}

int launch_fill_synth(uint8_t* dst, uint64_t nbytes, uint64_t seed, uint64_t start, cudaStream_t st) {
    if (!nbytes) return 0;
    fill_synth_kernel<<<grid_for((nbytes >> 3) + 1, 256, g_sm_count * 16), 256, 0, st>>>(dst, nbytes, seed * 0xD1342543DE82EF95ull,
                                                                                 start >> 3);
    return 1;
}

int chain_groups_per_cta() { return g_chain_groups; }

cudaError_t configure_kernels() {
    cudaError_t e;
    if (const char* g = getenv("B200H_CHAIN_GROUPS")) g_chain_groups = atoi(g) >= kChainGroupsMax ? kChainGroupsMax : kChainGroups;
    const void* lane_kernels[5] = {(const void*)lane_hash_kernel<true, true, false>, (const void*)lane_hash_kernel<true, false, false>,
                                   (const void*)lane_hash_kernel<false, true, false>, (const void*)lane_hash_kernel<true, true, true>,
                                   (const void*)lane_hash_kernel<true, false, true>};
    for (const void* k : lane_kernels) {
        e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kLaneSmem);
        if (e != cudaSuccess) return e;
    }
    const void* chain_kernels[6] = {
        (const void*)chain_hash_kernel<true, true, kChainGroups>, (const void*)chain_hash_kernel<true, false, kChainGroups>,
        (const void*)chain_hash_kernel<false, true, kChainGroups>, (const void*)chain_hash_kernel<true, true, kChainGroupsMax>,
        (const void*)chain_hash_kernel<true, false, kChainGroupsMax>, (const void*)chain_hash_kernel<false, true, kChainGroupsMax>};
    for (int i = 0; i < 6; ++i) {
        e = cudaFuncSetAttribute(chain_kernels[i], cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 chain_smem_bytes(i < 3 ? kChainGroups : kChainGroupsMax));
        if (e != cudaSuccess) return e;
    }
    int dev = 0, sms = 0, ctas = 0;
    e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return e;
    if (sms > 0) g_sm_count = sms;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, lane_hash_kernel<true, true, false>, kLaneThreads, kLaneSmem);
    if (e != cudaSuccess) return e;
    if (ctas > 0) g_lane_ctas_per_sm[0] = ctas;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, lane_hash_kernel<true, false, false>, kLaneThreads, kLaneSmem);
    if (e != cudaSuccess) return e;
    if (ctas > 0) g_lane_ctas_per_sm[1] = ctas;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, lane_hash_kernel<false, true, false>, kLaneThreads, kLaneSmem);
    if (e != cudaSuccess) return e;
    if (ctas > 0) g_lane_ctas_per_sm[2] = ctas;
    return cudaSuccess;
}

const char* kernel_build_info() {
    return "b200hash kernels: sm_90a, lane_hash(persistent, time-sliced q=32, cp.async ring 2x128B per lane), " __DATE__;
}

}  // namespace b200h
