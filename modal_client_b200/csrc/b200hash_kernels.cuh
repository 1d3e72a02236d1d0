// b200hash_kernels.cuh -- device-side declarations shared by the kernel and host translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200h {

// Per-message chaining state for streamed / segmented messages (64 B, 16-byte aligned).
struct alignas(16) ChainState {
    uint32_t sha[8];
    uint32_t md5[4];
    uint64_t prior_bytes;  // bytes already absorbed before this segment
    uint64_t reserved;
};

enum : uint32_t {
    F_SHA256 = 1u,
    F_MD5 = 2u,
    F_TRIM = 4u,      // hash the zero-trimmed prefix of every message, report trimmed length
    F_NO_FINAL = 8u,  // continuation segment: len % 64 == 0, no padding, write ChainState back
    F_YIELD_CHAIN_SMS = 16u,  // lane kernel: a CTA that lands on an SM hosting a live chain CTA exits at once
};

constexpr int kPlanBuckets = 512;
constexpr unsigned long long kChainMinBlocks = 1024;  // 64 KiB: shorter messages never go to the chain kernel
constexpr unsigned long long kChainRatio = 21000;     // H100: lane kernel ~540 GB/s fused vs ~26 MB/s for one lane
constexpr uint32_t kMaxChain = 1184;                  // chain-list capacity (entries)
constexpr int kSmFlagWords = 256;  // one word per SM: set by a chain CTA that serves a message (see F_YIELD_CHAIN_SMS)
// hist, cursor, qctl[4], total_blocks (u64), chain words[2], qctl_long[8], sm_flags[kSmFlagWords]
constexpr int kPlanScratchWords = 2 * kPlanBuckets + 16 + kSmFlagWords;
constexpr uint32_t kLongRingCapacity = 32768;  // entries of the long-message ring (>= 4 x SMs x 32 lanes, power of two)

// Launch wrappers (defined in b200hash_kernels.cu).  All asynchronous on `st`.
// Every wrapper returns the number of kernels it launched (for gpu_launches accounting).
// One entry per message the trim probe hands to the wide scan: bytes [0, end) of message `msg` are still unknown,
// cut into `items` chunks (nearest the end first) numbered from `first_item`.
struct TrimWideEntry {
    uint64_t msg;
    uint64_t end;
    uint32_t first_item;
    uint32_t items;
};
// wctl: 2 x u64 control block {entries << 32 | items, next item}; wlist: n entries.
int launch_trim(const uint8_t* base, const uint64_t* off, const uint64_t* len, uint64_t n, uint64_t* trimmed,
                unsigned long long* wctl, TrimWideEntry* wlist, cudaStream_t st);
// The planner's outlier count for these lengths, computed on the host (mirror of plan_scan_kernel's selection).
uint32_t plan_outliers_host(const uint64_t* len, uint64_t n, uint32_t max_chain, uint32_t sm_count, uint32_t long_cap,
                            uint32_t ratio8, uint32_t* n_long_out);
uint32_t plan_long_cap();  // most messages the long lane queue takes (0 is passed instead when a batch has no such queue)
uint32_t ring_capacity(uint64_t n);  // power of two >= max(n, 32): entries of the work-queue ring
// scratch layout (uint32 words): hist[kPlanBuckets] | cursor[kPlanBuckets] | qctl[4] | total_blocks (u64) | pad
inline int* plan_qctl(uint32_t* scratch) { return reinterpret_cast<int*>(scratch + 2 * kPlanBuckets); }
// the per-SM flags live 8 words behind qctl (device code reaches them through the qctl pointer it already has)
constexpr int kSmFlagsAfterQctl = 16;
// second queue control block {available, head, tail, count}: the LONG lane messages (see launch_plan)
constexpr int kLongQctlAfterQctl = 8;
inline int* plan_qctl_long(uint32_t* scratch) { return plan_qctl(scratch) + kLongQctlAfterQctl; }
constexpr int kPlanReadbackInts = 12;  // qctl[0..3], total, chain words, qctl_long[0..3]: what the API reads back
constexpr int kChainExpectedWord = 6;  // qctl[6]: chain CTAs the lane kernel's CTAs wait for before they look at the flags
constexpr int kChainStartedWord = 7;   // qctl[7]: chain CTAs that have set their flag
constexpr unsigned long long kYieldWaitNs = 200000;  // bound of that wait (0.2 ms; the chain CTAs are there in microseconds)
// Builds three work lists from the lengths: chain_list (outliers, see plan_scan_kernel), ring_long (the lane messages
// that would outlast the rest of the batch on a saturated lane kernel: hashed by a second, lane-packed launch once the
// short ones are done) and ring (everything else, longest first).
int launch_plan(const uint64_t* len, uint64_t n, uint32_t* ring /*ring_capacity(n)*/, uint32_t* ring_long /*kLongRingCapacity*/,
                uint32_t* chain_list /*kMaxChain*/, uint32_t* scratch /*kPlanScratchWords*/, bool fresh, uint32_t max_chain,
                uint32_t ratio8 /*rule (2): outliers are longer than ratio8/8 of the longest message*/, cudaStream_t st);
inline uint32_t plan_ratio8(uint32_t kflags) { return ((kflags & F_SHA256) && (kflags & F_MD5)) ? 3u : 4u; }
int launch_chain_hash(const uint8_t* base, const uint64_t* off, const uint64_t* len, const uint32_t* chain_list,
                      const int* qctl, uint32_t flags, uint8_t* sha_out, uint8_t* md5_out, ChainState* state,
                      bool resume, uint32_t n_chain /*live entries, as read back from qctl[3]*/, cudaStream_t st);
// n = messages in THIS queue (sizes the grid and the lane packing); ring_entries = capacity of `ring` (power of two);
// ctl = the batch's primary control block (chain words and SM flags live behind it), qctl = this queue's own.
int launch_lane_hash(const uint8_t* base, const uint64_t* off, const uint64_t* len, uint32_t* ring, uint32_t ring_entries,
                     int* qctl, const int* ctl, uint64_t n, uint32_t flags, uint8_t* sha_out, uint8_t* md5_out,
                     ChainState* state /*indexed by message id: caller states (F_NO_FINAL / resume) or scratch*/,
                     cudaStream_t st);
// first-occurrence dedupe of a digest table (b200hash_dedupe.cu)
uint32_t dedupe_table_capacity(uint64_t n);  // slots; the table buffer holds 2x that many uint32 words
int launch_dedupe(const void* d_keys, uint64_t n, uint32_t key_bytes, uint32_t* table, uint32_t* d_first,
                  unsigned long long* d_ndistinct, cudaStream_t st);
int launch_fill_synth(uint8_t* dst, uint64_t nbytes, uint64_t seed, uint64_t start, cudaStream_t st);
// out[2*nbytes] = lowercase ASCII hex of in[nbytes] (nbytes a multiple of 4, both 8-byte aligned)
int launch_hex_rows(const uint8_t* in, uint64_t nbytes, uint8_t* out, cudaStream_t st);

int chain_groups_per_cta();        // long messages one chain CTA can host (one CTA per SM)
int device_sm_count();             // SMs of the current device (as seen by configure_kernels)
cudaError_t configure_kernels();  // one-time cudaFuncSetAttribute calls for the current device
const char* kernel_build_info();

}  // namespace b200h
