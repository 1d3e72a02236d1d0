// tools/outlier_bench.cu -- one (or a few) long messages through the launch wrappers directly: lane kernel vs
// chain kernel, with the planner's routing decision printed.  Includes the kernel translation unit.
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tools/outlier_bench tools/outlier_bench.cu
#include <cstdio>
#include <vector>
#include "../modal_client_b200/csrc/b200hash_kernels.cu"

using namespace b200h;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)

int main(int argc, char** argv) {
    const uint64_t n = argc > 1 ? atoll(argv[1]) : 1;
    const uint64_t size = argc > 2 ? atoll(argv[2]) : (16ull << 20);
    const uint64_t nsmall = argc > 3 ? atoll(argv[3]) : 0;  // extra 100 KiB messages sharing the batch
    const uint32_t cap = argc > 4 ? (uint32_t)atoi(argv[4]) : 528u;  // chain CTAs available to the planner
    const uint64_t ssz = 100 * 1024;
    CK(configure_kernels());
    const uint64_t N = n + nsmall;
    const uint64_t total = n * size + nsmall * ssz;
    uint8_t* d_base; CK(cudaMalloc(&d_base, total + 64));
    cudaStream_t st, st2; CK(cudaStreamCreate(&st)); CK(cudaStreamCreate(&st2));
    launch_fill_synth(d_base, total, 5, 0, st);
    std::vector<uint64_t> off(N), len(N);
    uint64_t pos = 0;
    for (uint64_t i = 0; i < N; ++i) { off[i] = pos; len[i] = i < n ? size : ssz; pos += len[i]; }
    uint64_t *d_off, *d_len; CK(cudaMalloc(&d_off, N * 8)); CK(cudaMalloc(&d_len, N * 8));
    CK(cudaMemcpy(d_off, off.data(), N * 8, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_len, len.data(), N * 8, cudaMemcpyHostToDevice));
    uint32_t *ring, *scratch; CK(cudaMalloc(&ring, ring_capacity(N) * 4)); CK(cudaMalloc(&scratch, (kPlanScratchWords + kMaxChain) * 4));
    uint32_t* chain_list = scratch + kPlanScratchWords;
    int* qctl = plan_qctl(scratch);
    ChainState* states; CK(cudaMalloc(&states, N * sizeof(ChainState)));
    uint8_t *sha[2], *md5[2];
    for (int k = 0; k < 2; ++k) { CK(cudaMalloc(&sha[k], N * 32)); CK(cudaMalloc(&md5[k], N * 16)); CK(cudaMemset(sha[k], 0, N * 32)); CK(cudaMemset(md5[k], 0, N * 16)); }
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    const uint32_t flag_sets[3] = {F_SHA256 | F_MD5, F_SHA256, F_MD5};
    for (uint32_t flags : flag_sets) {
        float ms[2] = {0, 0};
        int hq[4];
        for (int mode = 0; mode < 2; ++mode) {  // 0 = lane only, 1 = outliers to the chain kernel
            for (int rep = 0; rep < 2; ++rep) {
                launch_plan(d_len, N, ring, chain_list, scratch, true, mode ? cap : 0u, st);
                CK(cudaMemcpyAsync(hq, qctl, 16, cudaMemcpyDeviceToHost, st));
                CK(cudaStreamSynchronize(st));
                cudaEventRecord(e0, st);
                if (mode && hq[3] > 0) launch_chain_hash(d_base, d_off, d_len, chain_list, qctl, flags, sha[mode], md5[mode], states, false, (uint32_t)hq[3], st2);
                launch_lane_hash(d_base, d_off, d_len, ring, qctl, N, flags, sha[mode], md5[mode], states, st);
                CK(cudaStreamSynchronize(st2));
                cudaEventRecord(e1, st);
                CK(cudaStreamSynchronize(st));
                cudaEventElapsedTime(&ms[mode], e0, e1);
            }
            printf("flags=%u mode=%s qctl={avail %d, head %d, tail %d, chain %d}  %.3f ms  (%.1f MB/s per long message)\n", flags,
                   mode ? "chain" : "lane ", hq[0], hq[1], hq[2], hq[3], ms[mode], size / ms[mode] / 1e3);
        }
        std::vector<uint8_t> a(N * 32), b(N * 32), c(N * 16), d(N * 16);
        cudaMemcpy(a.data(), sha[0], N * 32, cudaMemcpyDeviceToHost); cudaMemcpy(b.data(), sha[1], N * 32, cudaMemcpyDeviceToHost);
        cudaMemcpy(c.data(), md5[0], N * 16, cudaMemcpyDeviceToHost); cudaMemcpy(d.data(), md5[1], N * 16, cudaMemcpyDeviceToHost);
        printf("   digests equal: sha %s md5 %s\n", (!(flags & F_SHA256) || a == b) ? "yes" : "NO", (!(flags & F_MD5) || c == d) ? "yes" : "NO");
    }
    return 0;
}
