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
#ifdef VEC
    // per-thread operands: ptxas must keep them in vector registers (the hash kernel's operands all are)
    uint32_t b = (seed ^ 0x9e3779b9u) + threadIdx.x * 0x01000193u, c = seed * 3 + 1 + (threadIdx.x << 7);
    if (seed == 0x7fffffffu) one += threadIdx.x;  // never true at run time, but keeps `one` in a vector register
#else
    uint32_t b = seed ^ 0x9e3779b9u, c = seed * 3 + 1;
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
            if (MODE == 0) asm volatile("add.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(b));                          // IADD
            if (MODE == 1) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(one), "r"(b));         // IMAD R,R,R
            if (MODE == 2) asm volatile("mad.lo.u32 %0, %0, 3, %1;" : "+r"(a[i]) : "r"(b));                    // IMAD R,imm,R
            if (MODE == 3) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(b), "r"(c));       // LOP3
            if (MODE == 4) asm volatile("shf.r.wrap.b32 %0, %0, %0, 7;" : "+r"(a[i]));                         // SHF
            if (MODE == 5) asm volatile("{ .reg .u32 t; add.u32 t, %0, %1; add.u32 %0, t, %2; }" : "+r"(a[i]) : "r"(b), "r"(c)); // IADD3
            if (MODE == 6) {  // alternate ALU (LOP3) and IMAD imm
                if (i & 1) asm volatile("mad.lo.u32 %0, %0, 3, %1;" : "+r"(a[i]) : "r"(b));
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(b), "r"(c));
            }
            if (MODE == 7) {  // alternate ALU (LOP3) and IMAD R,R,R
                if (i & 1) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(one), "r"(b));
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(b), "r"(c));
            }
            if (MODE == 8) {  // alternate SHF and IADD (both ALU)
                if (i & 1) asm volatile("add.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(b));
                else asm volatile("shf.r.wrap.b32 %0, %0, %0, 7;" : "+r"(a[i]));
            }
            if (MODE == 9) asm volatile("mad.lo.u32 %0, %0, 1, %1;" : "+r"(a[i]) : "r"(b));                    // what does ptxas do with *1
            if (MODE == 10) asm volatile("mad.lo.u32 %0, %1, %0, %2;" : "+r"(a[i]) : "r"(one), "r"(b));
            if (MODE == 11) {  // IMAD.WIDE R, R, imm, RZ: rotate by multiply (lo/hi halves kept live by one LOP3 per 4)
                uint64_t d; asm volatile("mul.wide.u32 %0, %1, 0x4000000;" : "=l"(d) : "r"(a[i]));
                a[i] = (uint32_t)d; w[i] = (uint32_t)(d >> 32);
            }
            if (MODE == 12) {  // alternate LOP3 and IMAD.WIDE
                if (i & 1) { uint64_t d; asm volatile("mul.wide.u32 %0, %1, 0x4000000;" : "=l"(d) : "r"(a[i])); a[i] = (uint32_t)d; w[i] = (uint32_t)(d >> 32); }
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(b), "r"(c));
            }
            if (MODE == 13) {  // 2 ALU : 1 FMA
                if (i % 3 == 2) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(one), "r"(b));
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(b), "r"(c));
            }
            if (MODE == 14) {  // 1 ALU : 2 FMA
                if (i % 3 != 2) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(one), "r"(b));
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(b), "r"(c));
            }
            if (MODE == 15) asm volatile("mul.hi.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(b));                     // IMAD.HI
            if (MODE == 16) {  // the hash mix: 7 ALU (4 SHF + 3 LOP3) : 5 IMAD over 12 slots
                const int j = i % 12;
                if (j == 1 || j == 3 || j == 6 || j == 8 || j == 10) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(one), "r"(b));
                else if (j & 1) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(b), "r"(c));
                else asm volatile("shf.r.wrap.b32 %0, %0, %0, 7;" : "+r"(a[i]));
            }
            if (MODE == 17) {  // FFMA (fma heavy+lite) alternating with LOP3: is the cap an INT-FMA cap or a dispatch cap?
                if (i & 1) asm volatile("fma.rn.f32 %0, %0, %1, %2;" : "+f"(fa[i]) : "f"(fb), "f"(fc));
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(b), "r"(c));
            }
            if (MODE == 19) {  // LOP3 + two-input add (ptxas: VIADD / IMAD.IADD)
                if (i & 1) asm volatile("add.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(b));
                else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(b), "r"(c));
            }
            if (MODE == 20) {  // the hash mix with two-input adds instead of IMAD
                const int j = i % 12;
                if (j == 1 || j == 3 || j == 6 || j == 8 || j == 10) asm volatile("add.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(b));
                else if (j & 1) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(b), "r"(c));
                else asm volatile("shf.r.wrap.b32 %0, %0, %0, 7;" : "+r"(a[i]));
            }
            if (MODE == 18) asm volatile("fma.rn.f32 %0, %0, %1, %2;" : "+f"(fa[i]) : "f"(fb), "f"(fc));      // FFMA alone
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
    double inst = (double)ITER * ACC * warps_per_smsp;  // warp-instructions per SMSP
    printf("%-28s warps/SMSP=%d  cycles=%lld  IPC/SMSP=%.3f  (%.3f ms)\n", name, warps_per_smsp, c, inst / c, ms);
    cudaFree(out);
    cudaFree(cyc);
}

int main() {
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
    return 0;
}
