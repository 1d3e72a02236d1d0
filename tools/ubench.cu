// tools/ubench.cu -- issue-rate microbenchmarks for the INT32 instruction forms the hash kernel uses.
// Each test runs 8 independent accumulators per thread (no dependency stalls), 16 warps/SM... and reports
// warp-instructions per cycle per SMSP.   nvcc -arch=sm_90a -o ubench ubench.cu
#include <cstdio>
#include <cuda_runtime.h>
#include <stdint.h>

#define ITER 4096
#ifndef ACC
#define ACC 8
#endif

template <int MODE>
__global__ void k(uint32_t* out, uint32_t one, uint32_t seed, long long* cyc) {
    uint32_t a[ACC];
#pragma unroll
    for (int i = 0; i < ACC; ++i) a[i] = seed + threadIdx.x * 7 + i;
    const uint32_t uone = one;  // stays warp-uniform: ptxas reads it from a uniform register (IMAD R, R, UR, R)
#ifdef VEC
    // per-thread operands: ptxas must keep them in vector registers (the hash kernel's operands all are).  Every
    // accumulator has its own b and c, so consecutive instructions read distinct registers and the operand reuse cache
    // cannot serve them, as in the hash kernel (555 of its 4 717 vector source operands per block carry .reuse).
    uint32_t bv[ACC], cv[ACC];
#pragma unroll
    for (int i = 0; i < ACC; ++i) {
        bv[i] = (seed ^ 0x9e3779b9u) + threadIdx.x * 0x01000193u + i * 0x3c6ef372u;
        cv[i] = seed * 3 + 1 + (threadIdx.x << 7) + i * 0x7f4a7c15u;
    }
#define B(i) bv[i]
#define C(i) cv[i]
    if (seed == 0x7fffffffu) one += threadIdx.x;  // never true at run time, but keeps `one` in a vector register
#else
    uint32_t b = seed ^ 0x9e3779b9u, c = seed * 3 + 1;
#define B(i) b
#define C(i) c
#endif
    uint32_t w[ACC];
    float fa[ACC], fb = __uint_as_float(0x3f800001u + (seed & 1)), fc = 1e-9f;
#ifdef VEC
    fb += (float)(threadIdx.x >> 11); fc *= (float)(1 + (threadIdx.x >> 12));
#endif
#pragma unroll
    for (int i = 0; i < ACC; ++i) { w[i] = 0; fa[i] = (float)(seed + i); }
    long long t0 = clock64();
#pragma unroll 1
    for (int it = 0; it < ITER; ++it) {
#pragma unroll
        for (int i = 0; i < ACC; ++i) {
            if (MODE == 0) asm volatile("add.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(B(i)));                          // IADD
            if (MODE == 1) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(one), "r"(B(i)));         // IMAD R,R,R
            if (MODE == 2) asm volatile("mad.lo.u32 %0, %0, 3, %1;" : "+r"(a[i]) : "r"(B(i)));                    // IMAD R,imm,R
            if (MODE == 3) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(B(i)), "r"(C(i)));       // LOP3
            if (MODE == 4) asm volatile("shf.r.wrap.b32 %0, %0, %0, 7;" : "+r"(a[i]));                         // SHF
            if (MODE == 5) asm volatile("{ .reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2; }" : "+r"(a[i]) : "r"(B(i)), "r"(C(i))); // IADD3
            if (MODE == 6) {  // alternate ALU (LOP3) and IMAD imm
                if (i & 1) asm volatile("mad.lo.u32 %0, %0, 3, %1;" : "+r"(a[i]) : "r"(B(i)));
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(B(i)), "r"(C(i)));
            }
            if (MODE == 7) {  // alternate ALU (LOP3) and IMAD R,R,R
                if (i & 1) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(one), "r"(B(i)));
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(B(i)), "r"(C(i)));
            }
            if (MODE == 8) {  // alternate SHF and IADD (both ALU)
                if (i & 1) asm volatile("add.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(B(i)));
                else asm volatile("shf.r.wrap.b32 %0, %0, %0, 7;" : "+r"(a[i]));
            }
            if (MODE == 9) asm volatile("mad.lo.u32 %0, %0, 1, %1;" : "+r"(a[i]) : "r"(B(i)));                    // what does ptxas do with *1
            if (MODE == 10) asm volatile("mad.lo.u32 %0, %1, %0, %2;" : "+r"(a[i]) : "r"(one), "r"(B(i)));
            if (MODE == 11) {  // IMAD.WIDE R, R, imm, RZ: rotate by multiply (lo/hi halves kept live by one LOP3 per 4)
                uint64_t d; asm volatile("mul.wide.u32 %0, %1, 0x4000000;" : "=l"(d) : "r"(a[i]));
                a[i] = (uint32_t)d; w[i] = (uint32_t)(d >> 32);
            }
            if (MODE == 12) {  // alternate LOP3 and IMAD.WIDE
                if (i & 1) { uint64_t d; asm volatile("mul.wide.u32 %0, %1, 0x4000000;" : "=l"(d) : "r"(a[i])); a[i] = (uint32_t)d; w[i] = (uint32_t)(d >> 32); }
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(B(i)), "r"(C(i)));
            }
            if (MODE == 13) {  // 2 ALU : 1 FMA
                if (i % 3 == 2) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(one), "r"(B(i)));
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(B(i)), "r"(C(i)));
            }
            if (MODE == 14) {  // 1 ALU : 2 FMA
                if (i % 3 != 2) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(one), "r"(B(i)));
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(B(i)), "r"(C(i)));
            }
            if (MODE == 15) asm volatile("mul.hi.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(B(i)));                     // IMAD.HI
            if (MODE == 16) {  // the hash mix: 7 ALU (4 SHF + 3 LOP3) : 5 IMAD over 12 slots
                const int j = i % 12;
                if (j == 1 || j == 3 || j == 6 || j == 8 || j == 10) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(one), "r"(B(i)));
                else if (j & 1) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(B(i)), "r"(C(i)));
                else asm volatile("shf.r.wrap.b32 %0, %0, %0, 7;" : "+r"(a[i]));
            }
            if (MODE == 17) {  // FFMA (fma heavy+lite) alternating with LOP3: is the cap an INT-FMA cap or a dispatch cap?
                if (i & 1) asm volatile("fma.rn.f32 %0, %0, %1, %2;" : "+f"(fa[i]) : "f"(fb), "f"(fc));
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(B(i)), "r"(C(i)));
            }
            if (MODE == 19) {  // LOP3 + two-input add (ptxas: VIADD / IMAD.IADD)
                if (i & 1) asm volatile("add.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(B(i)));
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(B(i)), "r"(C(i)));
            }
            if (MODE == 20) {  // the hash mix with two-input adds instead of IMAD
                const int j = i % 12;
                if (j == 1 || j == 3 || j == 6 || j == 8 || j == 10) asm volatile("add.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(B(i)));
                else if (j & 1) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(B(i)), "r"(C(i)));
                else asm volatile("shf.r.wrap.b32 %0, %0, %0, 7;" : "+r"(a[i]));
            }
            if (MODE == 18) asm volatile("fma.rn.f32 %0, %0, %1, %2;" : "+f"(fa[i]) : "f"(fb), "f"(fc));      // FFMA alone
            // acc + rotl(u, 26) on the FMA pipe: multiplier one << 26 (a run-time value), 32-bit accumulator b
            if (MODE == 21) asm volatile("mad.hi.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(one << 26), "r"(B(i)));  // IMAD.HI R,UR,R
            if (MODE == 22) asm volatile("{ .reg .u32 t; mad.hi.u32 t, %0, %1, %2; mad.lo.u32 %0, %0, %1, t; }"
                                         : "+r"(a[i]) : "r"(one << 26), "r"(B(i)));                            // IMAD.HI + IMAD
            if (MODE == 23) {  // alternate LOP3 and IMAD.HI R,UR,R
                if (i & 1) asm volatile("mad.hi.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(one << 26), "r"(B(i)));
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(B(i)), "r"(C(i)));
            }
            if (MODE == 24) asm volatile("mul.hi.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(one << 26));               // IMAD.HI R,UR,RZ
            // the fused lane kernel's add forms (B200H_UNIFORM_ONE): x * one + y with `one` in a vector or a uniform
            // register, and x + constant as VIADD or as IMAD with the constant in the C slot
            if (MODE == 25) {  // alternate LOP3 and IMAD R,R,UR,R
                if (i & 1) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(uone), "r"(B(i)));
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(B(i)), "r"(C(i)));
            }
            if (MODE == 26) {  // alternate LOP3 and VIADD R,R,imm
                if (i & 1) asm volatile("add.u32 %0, %0, 0x5a827999;" : "+r"(a[i]));
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(B(i)), "r"(C(i)));
            }
            if (MODE == 27) {  // alternate SHF and VIADD R,R,imm
                if (i & 1) asm volatile("add.u32 %0, %0, 0x5a827999;" : "+r"(a[i]));
                else asm volatile("shf.r.wrap.b32 %0, %0, %0, 7;" : "+r"(a[i]));
            }
            if (MODE == 28) asm volatile("add.u32 %0, %0, 0x5a827999;" : "+r"(a[i]));                          // VIADD alone
            if (MODE == 29 || MODE == 30 || MODE == 31) {  // the hash mix, 7 ALU : 5 adds, adds as IMAD R,R,UR,R
                const int j = i % 12;
                if (j == 10 && MODE == 30) asm volatile("add.u32 %0, %0, 0x5a827999;" : "+r"(a[i]));  // 1 in 5 a VIADD imm
                else if (j == 10 && MODE == 31) asm volatile("mad.lo.u32 %0, %0, %1, 0x5a827999;" : "+r"(a[i]) : "r"(one));  // or an IMAD R,R,imm
                else if (j == 1 || j == 3 || j == 6 || j == 8 || j == 10) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(uone), "r"(B(i)));
                else if (j & 1) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(B(i)), "r"(C(i)));
                else asm volatile("shf.r.wrap.b32 %0, %0, %0, 7;" : "+r"(a[i]));
            }
            if (MODE == 32) {  // alternate LOP3 and IMAD R,R,imm (one vector-register multiplier, constant addend)
                if (i & 1) asm volatile("mad.lo.u32 %0, %0, %1, 0x5a827999;" : "+r"(a[i]) : "r"(one));
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(B(i)), "r"(C(i)));
            }
            // the read costs tools/lane_sass_score.py assumes (modes 33-37, 40); mode 4 is SHF.W with hi == lo.  Register banks
            // cannot be set from PTX: ptxas allocates (and splits 64-bit pairs) freely, so no mode pins a LOP3's sources to one bank
            if (MODE == 33) asm volatile("shf.r.wrap.b32 %0, %0, %1, 7;" : "+r"(a[i]) : "r"(B(i)));            // SHF.W lo != hi
            // acc + rotl: ptxas fuses a plain add of a funnel shift into LEA.HI d, lo, acc, hi (as add_rotl does)
            if (MODE == 34) a[i] = B(i) + __funnelshift_l(a[i], a[i], 5);                                     // LEA.HI (u, u)
            if (MODE == 35) a[i] = B(i) + __funnelshift_l(C(i), a[i], 5);                                     // LEA.HI (u, v)
            if (MODE == 36) {  // alternate LOP3 and LEA.HI (u, u): at most 0.5 if LEA.HI is on the ALU pipe
                if (i & 1) a[i] = B(i) + __funnelshift_l(a[i], a[i], 5);
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(B(i)), "r"(C(i)));
            }
            if (MODE == 37) {  // alternate IMAD R,R,UR,R and LEA.HI (u, u)
                if (i & 1) a[i] = B(i) + __funnelshift_l(a[i], a[i], 5);
                else asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(uone), "r"(B(i)));
            }
            if (MODE == 40) {  // LOP3 alone, 8 per accumulator and loop trip: the loop's own instructions count 8x less
#pragma unroll
                for (int r = 0; r < 8; ++r) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(B(i)), "r"(C(i)));
            }
        }
    }
    long long t1 = clock64();
    uint32_t s = 0;
#pragma unroll
    for (int i = 0; i < ACC; ++i) s ^= a[i] ^ w[i] ^ __float_as_uint(fa[i]);
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}

template <int MODE>
void run(const char* name, int warps_per_smsp) {
    uint32_t* out;
    long long* cyc;
    int threads = 128 * warps_per_smsp;  // one CTA per SM, warps spread over the 4 SMSPs
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    cudaMalloc(&out, (size_t)sms * threads * 4);
    cudaMalloc(&cyc, 8);
    k<MODE><<<sms, threads>>>(out, 1, 12345, cyc);
    cudaDeviceSynchronize();
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    cudaEventRecord(e0);
    k<MODE><<<sms, threads>>>(out, 1, 12345, cyc);
    cudaEventRecord(e1);
    cudaDeviceSynchronize();
    long long c;
    cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    double inst = (double)ITER * ACC * warps_per_smsp * (MODE == 22 ? 2 : MODE == 40 ? 8 : 1);  // warp-instructions per SMSP
    printf("%-28s warps/SMSP=%d  cycles=%lld  IPC/SMSP=%.3f  (%.3f ms)\n", name, warps_per_smsp, c, inst / c, ms);
    cudaFree(out);
    cudaFree(cyc);
}

static void read_modes() {
    // the read costs of the fused lane kernel's body (modes 33-37, 40); it runs 4 warps per SMSP, 3 at 3 CTAs per SM
    for (int w : {3, 4}) {
        run<4>("SHF.W hi == lo", w); run<33>("SHF.W hi != lo", w);
        run<34>("LEA.HI (u, u)", w); run<35>("LEA.HI (u, v)", w);
        run<36>("LOP3 + LEA.HI alt", w); run<37>("IMAD R,R,UR,R + LEA.HI alt", w);
        run<3>("LOP3", w); run<40>("LOP3 x8 per loop trip", w);
    }
}

int main(int argc, char** argv) {
    (void)argv;
    read_modes();
    if (argc > 1) return 0;  // `ubench reads`: only the read-cost modes
    // one warp per SMSP: what a single instruction stream with plenty of ILP can issue
    run<0>("IADD R,R,R", 1); run<1>("IMAD R,R,R(one),R", 1); run<3>("LOP3", 1); run<4>("SHF.W", 1);
    run<6>("LOP3 + IMAD imm alt", 1); run<8>("SHF + IADD alt", 1);
    run<0>("IADD R,R,R", 2); run<3>("LOP3", 2); run<6>("LOP3 + IMAD imm alt", 2);
    for (int w : {4, 8}) {
        if (w == 4) {
            run<0>("IADD R,R,R", 4); run<1>("IMAD R,R,R(one),R", 4); run<2>("IMAD R,R,imm3,R", 4); run<3>("LOP3", 4);
            run<4>("SHF.W", 4); run<5>("IADD3 (2 adds)", 4); run<6>("LOP3 + IMAD imm alt", 4); run<7>("LOP3 + IMAD RRR alt", 4);
            run<8>("SHF + IADD alt", 4); run<9>("mad *1 (ptxas choice)", 4); run<10>("IMAD one,R,R", 4);
        } else {
            run<0>("IADD R,R,R", 8); run<1>("IMAD R,R,R(one),R", 8); run<2>("IMAD R,R,imm3,R", 8); run<3>("LOP3", 8);
            run<4>("SHF.W", 8); run<5>("IADD3 (2 adds)", 8); run<6>("LOP3 + IMAD imm alt", 8); run<7>("LOP3 + IMAD RRR alt", 8);
            run<8>("SHF + IADD alt", 8); run<9>("mad *1 (ptxas choice)", 8); run<10>("IMAD one,R,R", 8);
        }
    }
    for (int w : {5, 8}) {
        if (w == 5) { run<19>("LOP3 + add2 alt", 5); run<20>("hash mix 7 ALU : 5 add2", 5); run<8>("SHF + add2 alt", 5); run<0>("add2 alone", 5); run<16>("hash mix 7 ALU : 5 IMAD", 5); run<7>("LOP3 + IMAD RRR alt", 5); run<17>("LOP3 + FFMA alt", 5);}
        if (w == 8) { run<19>("LOP3 + add2 alt", 8); run<20>("hash mix 7 ALU : 5 add2", 8); }
    }
    for (int w : {4, 5, 8}) {
        if (w == 4) { run<11>("IMAD.WIDE imm", 4); run<12>("LOP3 + IMAD.WIDE alt", 4); run<13>("2 LOP3 : 1 IMAD", 4); run<14>("1 LOP3 : 2 IMAD", 4); run<15>("IMAD.HI", 4); run<16>("hash mix 7 ALU : 5 IMAD", 4); run<17>("LOP3 + FFMA alt", 4); run<18>("FFMA RRR", 4); }
        if (w == 5) { run<7>("LOP3 + IMAD RRR alt", 5); run<12>("LOP3 + IMAD.WIDE alt", 5); run<13>("2 LOP3 : 1 IMAD", 5); run<16>("hash mix 7 ALU : 5 IMAD", 5); }
        if (w == 8) { run<11>("IMAD.WIDE imm", 8); run<12>("LOP3 + IMAD.WIDE alt", 8); run<13>("2 LOP3 : 1 IMAD", 8); run<14>("1 LOP3 : 2 IMAD", 8); run<15>("IMAD.HI", 8); run<16>("hash mix 7 ALU : 5 IMAD", 8); run<17>("LOP3 + FFMA alt", 8); run<18>("FFMA RRR", 8); }
    }
    // acc + rotl(u, k) = mad.lo(u, 2^k, mad.hi(u, 2^k, acc)): the forms alone and against the ALU pipe
    for (int w : {1, 4, 5, 8}) {
        run<21>("IMAD.HI R,UR,R (acc)", w); run<24>("IMAD.HI R,UR,RZ", w); run<22>("IMAD.HI + IMAD pair", w);
        run<23>("LOP3 + IMAD.HI alt", w); run<1>("IMAD R,R,R(one),R", w); run<7>("LOP3 + IMAD RRR alt", w);
    }
    // the fused lane kernel's add forms (modes 25-32); it runs 5 warps per SMSP
    for (int w : {4, 5, 8}) {
        run<3>("LOP3", w); run<4>("SHF.W", w); run<28>("VIADD imm", w);
        run<7>("LOP3 + IMAD R,R,R alt", w); run<25>("LOP3 + IMAD R,R,UR,R alt", w); run<32>("LOP3 + IMAD R,R,imm alt", w);
        run<26>("LOP3 + VIADD imm alt", w); run<27>("SHF + VIADD imm alt", w);
        run<16>("mix 7:5 IMAD R,R,R", w); run<29>("mix 7:5 IMAD R,R,UR", w); run<30>("mix 7:5 UR, 1/5 VIADD", w);
        run<31>("mix 7:5 UR, 1/5 IMAD imm", w);
    }
    return 0;
}
