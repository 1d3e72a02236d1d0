// b200hash_api.cu -- host side of libb200hash.so: the C ABI declared in include/b200hash.h.
//
// Owns the per-device context (streams, pinned staging ring, HBM wave buffers, grow-only scratch),
// turns host batches into double-buffered waves (pack -> cudaMemcpyAsync -> trim/plan/lane_hash) and
// implements the streaming (hashlib-object shaped) interface on top of the chaining-state kernel mode.
// No CPU hashing exists in this library: without a CUDA device every entry point fails.
#include <cuda_runtime.h>
#include <stdint.h>

#include <fcntl.h>
#include <immintrin.h>
#include <pthread.h>
#include <sched.h>
#include <sys/stat.h>
#include <unistd.h>

#include <nvtx3/nvToolsExt.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cctype>
#include <cerrno>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <vector>

#include "../../include/b200hash.h"
#include "b200hash_kernels.cuh"
#include "b200pack_team.h"

using namespace b200h;

static const uint32_t kShaIv[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au,
                                   0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
static const uint32_t kMd5Iv[4] = {0x67452301u, 0xefcdab89u, 0x98badcfeu, 0x10325476u};

namespace {

thread_local std::string g_create_error;

// NVTX range around every C-ABI entry point (visible in nsys / ncu --nvtx; a no-op without an injected tool)
struct NvtxRange {
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
    NvtxRange(const NvtxRange&) = delete;
    NvtxRange& operator=(const NvtxRange&) = delete;
};
#define B200H_RANGE(name) NvtxRange nvtx_range__(name)

// One caller's small b200h_hash_batch_host request while it waits to be merged with its neighbours'.
struct CombineReq {
    const uint8_t* base;
    const uint64_t* off;
    const uint64_t* len;
    uint64_t n;
    uint32_t flags;
    uint8_t* sha;
    uint8_t* md5;
    uint64_t* trim;
    int rc = 0;
    bool done = false;
};

// Combining queue for concurrent small requests (the reference's ThreadPool / to_thread callers each hash ONE
// file, block or payload per call: py/modal/volume.py:1209-1216, blob_utils.py:622-645).  The first caller in
// becomes the leader; while it waits for the context (the GPU is busy with the previous group) the others join
// its group; the leader then issues ONE batch for all of them and hands every caller its own digests.
struct Combiner {
    std::mutex m;
    std::condition_variable cv_done, cv_more;
    std::vector<CombineReq*> pending[2];  // [B200H_TRIM_ZEROS?]: trimming changes what a message means, never mixed
    bool leader[2] = {false, false};
    bool recent_multi = false;  // the last group had company: worth waiting a moment for the next one to fill
    uint64_t groups = 0, requests = 0;
};
constexpr uint64_t kCombineMaxN = 1024;     // requests with more messages fill the GPU on their own
constexpr size_t kCombineFull = 64;          // stop waiting for company at this many callers
constexpr int kCombineWaitUs = 200;

struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
};

struct Wave {
    uint64_t i0, i1;    // message index range [i0, i1)
    uint64_t src_lo;    // direct mode: host offset (relative to base) of the first byte copied
    uint64_t bytes;     // bytes occupying the device wave buffer
    // A message larger than one wave slot is hashed as consecutive segments of itself (one wave each), the
    // chaining state travelling through a device-resident ChainState: seg != 0, message i0, bytes
    // [seg_start, seg_start + bytes) of it.
    int seg = 0;        // 0 = ordinary wave, 1 = first/middle segment, 2 = last segment
    bool seg_first = false;
    uint64_t seg_start = 0;
};

}  // namespace

struct b200h_ctx {
    int device = 0;
    std::mutex mu;
    std::string err;
    cudaStream_t s_copy = nullptr, s_comp = nullptr, s_chain = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    // Outlier path: the warp-specialised chain kernel (TMA tile ring + mbarriers; schedule expansion, SHA-256 rounds
    // and MD5 on three warps of one CTA) runs ONE chain about twice as fast as a lane does,
    // at up to 4 CTAs per SM.  The planner (plan_scan_kernel) hands it only true outliers and only when all of
    // them fit in chain_cap CTAs; everything else stays on the lane kernel.  B200H_CHAIN=0 disables it, =N sets the cap.
    bool chain_enabled = true;
    // One chain CTA per SM, each hosting up to chain_groups_per_cta() messages (set from the SM count at create).
    uint32_t chain_cap = 528;
    uint32_t sm_count = 132;
    // B200H_YIELD_CHAIN_SMS=1: CTAs of a full-grid lane launch leave the SMs that host chain CTAs.  Off by default:
    // on one rank's share of C3 the long pole was the lane tail, not the chains -- and it must never be applied to a
    // small grid (see launch_lane_hash).
    bool yield_chain_sms = false;
    int* h_plan = nullptr;        // pinned: the planner's control block {avail, head, tail, outliers} of the last batch
    uint32_t last_outliers = 0;
    bool verify_plan = false;     // B200H_VERIFY_PLAN=1: cross-check the host-side outlier count against the device's
    uint64_t plan_syncs = 0;      // enqueues that had to read the outlier count back (stream synchronisation)
    Combiner combiner;
    bool combine_enabled = true;  // B200H_COMBINE=0 turns the combining queue off
    struct StreamBuf {            // resources of a b200h_stream, pooled per context (allocation costs ~1 ms)
        uint8_t* h = nullptr;     // pinned host accumulation buffer
        uint8_t* d = nullptr;     // device block: states | meta | out | plan scratch | ring | data
        cudaStream_t st = nullptr;
        cudaEvent_t ev = nullptr;
    };
    std::vector<StreamBuf> stream_pool;
    size_t stream_cap = size_t(4) << 20;  // bytes absorbed per kernel launch (B200H_STREAM_BUF)
    cudaEvent_t ev_copied[2] = {nullptr, nullptr};    // H2D of a wave slot finished
    cudaEvent_t ev_consumed[2] = {nullptr, nullptr};  // kernels reading a wave slot finished
    cudaEvent_t ev_pin[2] = {nullptr, nullptr};       // H2D out of a pinned slot finished
    cudaEvent_t ev_scratch = nullptr;                 // last use of the shared scratch buffers
    bool scratch_used = false;
    cudaEvent_t ev_dedupe = nullptr;                  // last use of the dedupe table
    bool dedupe_used = false;
    uint8_t* pin[2] = {nullptr, nullptr};
    size_t pin_cap = 0;  // per slot
    uint8_t* dwave[2] = {nullptr, nullptr};
    size_t dwave_cap = 0;  // per slot
    size_t dwave_want = 0;
    DevBuf d_off, d_len, d_order, d_order_long, d_trim, d_sha, d_md5, d_scratch, d_small, d_states, d_dedupe, d_keys, d_trimctl, d_hex;
    DevBuf d_parts;  // part table of b200h_hash_segment_parts_device: absolute addresses | lengths | gather tiles
                     // (b200h_hash_fixed_parts_device: the ETag message {offset, length} after the lengths)
    uint64_t* h_meta = nullptr;  // pinned: offsets then lengths
    size_t h_meta_cap = 0;       // in uint64 elements
    uint64_t launches = 0;
    bool profiling = false;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof_events;
    double prof_ms = 0.0;
    uint64_t prof_n = 0;
    int pack_threads = 1;
    int io_threads = 1;
    PackTeam team;  // the packer / reader threads (used under `mu` only)
    // CPUs of the NUMA node the GPU hangs off (empty set: unknown / single node / B200H_NUMA=0).  The packer and
    // reader threads are pinned there: the staging ring lives in that node's memory and the DMA engine reads it from
    // there, so a packer on the other socket would push every byte across the socket interconnect twice.
    cpu_set_t node_cpus;
    bool node_cpus_valid = false;
};

struct b200h_stream {
    b200h_ctx* ctx = nullptr;
    uint32_t flags = 0;
    b200h_ctx::StreamBuf res;
    uint8_t* hbuf = nullptr;  // = res.h: pinned host accumulation buffer (cap bytes, multiple of 64)
    size_t cap = 0;
    size_t fill = 0;
    bool h2d_pending = false;      // res.ev marks the end of the last copy out of hbuf
    uint8_t* d_buf = nullptr;      // device copy of hbuf
    ChainState* d_state = nullptr; // [0] running state, [1] scratch copy for digest()
    uint64_t* d_meta = nullptr;    // off, len
    uint8_t* d_out = nullptr;      // 32 + 16
    uint32_t* d_plan = nullptr;    // this stream's own planner scratch + ring: its launches never wait for other batches
    uint32_t* d_ring = nullptr;
    uint64_t total = 0;
};

namespace {

void stream_res_destroy(b200h_ctx::StreamBuf& r);  // defined with the streaming entry points

// "0-31,64-95" -> cpu_set_t
bool parse_cpulist(const char* s, cpu_set_t* out) {
    CPU_ZERO(out);
    int n = 0;
    while (*s && *s != '\n') {
        char* end = nullptr;
        long a = strtol(s, &end, 10);
        if (end == s) return false;
        long b = a;
        if (*end == '-') {
            s = end + 1;
            b = strtol(s, &end, 10);
            if (end == s) return false;
        }
        for (long c = a; c <= b && c < CPU_SETSIZE; ++c) {
            CPU_SET((int)c, out);
            ++n;
        }
        s = *end == ',' ? end + 1 : end;
    }
    return n > 0;
}

// CPUs local to CUDA device `device` (sysfs: the PCI function's numa_node -> that node's cpulist)
bool gpu_node_cpus(int device, cpu_set_t* out) {
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    for (char* c = bus; *c; ++c) *c = (char)tolower(*c);
    char path[128], buf[4096];
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE* f = fopen(path, "r");
    if (!f) return false;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    if (node < 0) return false;
    snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
    f = fopen(path, "r");
    if (!f) return false;
    const bool got = fgets(buf, sizeof buf, f) != nullptr;
    fclose(f);
    if (!got || !parse_cpulist(buf, out)) return false;
    // keep only CPUs this process may run on (cgroup / taskset); if none is left, give up
    cpu_set_t allowed;
    if (sched_getaffinity(0, sizeof allowed, &allowed) == 0) {
        cpu_set_t both;
        CPU_AND(&both, out, &allowed);
        if (CPU_COUNT(&both) == 0) return false;
        // a process already confined to a subset keeps its own mask
        *out = both;
    }
    return true;
}

int fail(b200h_ctx* ctx, int code, const std::string& msg) {
    if (ctx) ctx->err = msg;
    else g_create_error = msg;
    return code;
}

#define CU_TRY(ctx, call)                                                                                   \
    do {                                                                                                    \
        cudaError_t e__ = (call);                                                                           \
        if (e__ != cudaSuccess) {                                                                           \
            char b__[512];                                                                                  \
            snprintf(b__, sizeof b__, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
            cudaGetLastError();                                                                             \
            return fail(ctx, e__ == cudaErrorMemoryAllocation ? B200H_E_NOMEM : B200H_E_CUDA, b__);         \
        }                                                                                                   \
    } while (0)

int ensure_dev(b200h_ctx* ctx, DevBuf& b, size_t bytes) {
    if (bytes <= b.cap) return 0;
    size_t want = std::max(bytes, b.cap + b.cap / 2);
    want = (want + 255) & ~size_t(255);
    if (b.p) {
        CU_TRY(ctx, cudaDeviceSynchronize());
        CU_TRY(ctx, cudaFree(b.p));
        b.p = nullptr;
        b.cap = 0;
    }
    CU_TRY(ctx, cudaMalloc(&b.p, want));
    b.cap = want;
    return 0;
}

int ensure_wave(b200h_ctx* ctx, size_t bytes) {
    if (bytes <= ctx->dwave_cap) return 0;
    // grow geometrically towards the configured wave size; beyond it only as far as one message needs
    size_t want = std::max(bytes, std::min(ctx->dwave_want, std::max<size_t>(2 * ctx->dwave_cap, size_t(64) << 20)));
    want = (want + 255) & ~size_t(255);
    CU_TRY(ctx, cudaDeviceSynchronize());
    for (int s = 0; s < 2; ++s) {
        if (ctx->dwave[s]) CU_TRY(ctx, cudaFree(ctx->dwave[s]));
        ctx->dwave[s] = nullptr;
    }
    ctx->dwave_cap = 0;
    for (int s = 0; s < 2; ++s) CU_TRY(ctx, cudaMalloc(&ctx->dwave[s], want));
    ctx->dwave_cap = want;
    return 0;
}

int ensure_meta(b200h_ctx* ctx, size_t elems) {
    if (elems <= ctx->h_meta_cap) return 0;
    if (ctx->h_meta) CU_TRY(ctx, cudaFreeHost(ctx->h_meta));
    ctx->h_meta = nullptr;
    ctx->h_meta_cap = 0;
    size_t want = std::max(elems, size_t(1) << 16);
    CU_TRY(ctx, cudaHostAlloc(&ctx->h_meta, want * sizeof(uint64_t), cudaHostAllocDefault));
    ctx->h_meta_cap = want;
    return 0;
}

int prof_begin(b200h_ctx* ctx, cudaStream_t st, cudaEvent_t* a, cudaEvent_t* b) {
    *a = *b = nullptr;
    if (!ctx->profiling) return 0;
    CU_TRY(ctx, cudaEventCreate(a));
    CU_TRY(ctx, cudaEventCreate(b));
    CU_TRY(ctx, cudaEventRecord(*a, st));
    return 0;
}
int prof_end(b200h_ctx* ctx, cudaStream_t st, cudaEvent_t a, cudaEvent_t b) {
    if (!a) return 0;
    CU_TRY(ctx, cudaEventRecord(b, st));
    ctx->prof_events.emplace_back(a, b);
    return 0;
}

constexpr uint32_t kFlagNoFinal = 0x80000000u;  // internal: continuation segment (no padding, state written back)

// Enqueue trim -> plan -> lane_hash for n device-resident messages on `st`.  ctx->mu must be held.
// h_len (may be NULL) = the same lengths on the host.  With them the outlier routing is decided here without reading
// anything back, so the call only enqueues; without them (and without B200H_NO_OUTLIERS) the planner's count is
// read back after the ~12 us plan kernels, which synchronises `st` once.
int enqueue_device_batch(b200h_ctx* ctx, const uint8_t* d_base, const uint64_t* d_off, const uint64_t* d_len,
                         uint64_t n, uint32_t flags, uint8_t* d_sha, uint8_t* d_md5, uint64_t* d_trim_out,
                         ChainState* d_state, cudaStream_t st, const uint64_t* h_len = nullptr,
                         uint32_t* own_scratch = nullptr, uint32_t* own_ring = nullptr) {
    if (n == 0) return 0;
    if (n > 0xffffffffull) return fail(ctx, B200H_E_INVALID, "batch larger than 2^32-1 messages");
    uint32_t kflags = 0;
    if (flags & B200H_SHA256) kflags |= F_SHA256;
    if (flags & B200H_MD5) kflags |= F_MD5;
    if (flags & kFlagNoFinal) kflags |= F_NO_FINAL;
    if (!(kflags & (F_SHA256 | F_MD5))) return fail(ctx, B200H_E_INVALID, "flags select neither SHA256 nor MD5");

    // own_scratch / own_ring: planner scratch and queue ring private to the caller (a b200h_stream): the batch then
    // shares nothing with other batches of the context and runs concurrently with them on its own CUDA stream.
    const bool shared_scratch = own_scratch == nullptr;
    if (shared_scratch && ctx->scratch_used) CU_TRY(ctx, cudaStreamWaitEvent(st, ctx->ev_scratch, 0));
    const uint64_t* len_used = d_len;
    if (flags & B200H_TRIM_ZEROS) {
        uint64_t* tbuf = d_trim_out;
        if (!tbuf) {
            if (int rc = ensure_dev(ctx, ctx->d_trim, n * sizeof(uint64_t))) return rc;
            tbuf = (uint64_t*)ctx->d_trim.p;
        }
        if (int rc = ensure_dev(ctx, ctx->d_trimctl, 16 + n * sizeof(TrimWideEntry))) return rc;
        ctx->launches += launch_trim(d_base, d_off, d_len, n, tbuf, (unsigned long long*)ctx->d_trimctl.p,
                                     (TrimWideEntry*)((uint8_t*)ctx->d_trimctl.p + 16), st);
        len_used = tbuf;
        h_len = nullptr;  // the lengths that matter now exist on the device only
    } else if (d_trim_out) {
        CU_TRY(ctx, cudaMemcpyAsync(d_trim_out, d_len, n * sizeof(uint64_t), cudaMemcpyDeviceToDevice, st));
    }
    // work queue (ring + control block) and chaining-state scratch for the persistent lane kernel
    if (n >= 0x7fffffffull) return fail(ctx, B200H_E_INVALID, "batch larger than 2^31-2 messages");
    if (shared_scratch) {
        if (int rc = ensure_dev(ctx, ctx->d_order, (size_t)ring_capacity(n) * sizeof(uint32_t))) return rc;
        if (int rc = ensure_dev(ctx, ctx->d_order_long, (size_t)kLongRingCapacity * sizeof(uint32_t))) return rc;
        if (int rc = ensure_dev(ctx, ctx->d_scratch, (kPlanScratchWords + kMaxChain) * sizeof(uint32_t))) return rc;
    }
    uint32_t* ring = shared_scratch ? (uint32_t*)ctx->d_order.p : own_ring;
    // the long lane messages get a queue of their own (a private single-message batch never has any)
    // (nor does a B200H_NO_OUTLIERS batch whose lengths the host does not hold: that flag promises "only enqueues",
    // and sizing the second launch would need the planner's answer)
    uint32_t* ring_long = (shared_scratch && !((flags & B200H_NO_OUTLIERS) && !h_len)) ? (uint32_t*)ctx->d_order_long.p : nullptr;
    const uint32_t long_cap = ring_long ? plan_long_cap() : 0u;
    uint32_t* scratch = shared_scratch ? (uint32_t*)ctx->d_scratch.p : own_scratch;
    uint32_t* chain_list = scratch + kPlanScratchWords;
    int* qctl = plan_qctl(scratch);
    ChainState* states = d_state;
    if (!states) {
        if (int rc = ensure_dev(ctx, ctx->d_states, n * sizeof(ChainState))) return rc;
        states = (ChainState*)ctx->d_states.p;
    }
    const bool resume = d_state != nullptr;
    const bool chain_on = ctx->chain_enabled && !(flags & B200H_NO_OUTLIERS);
    const uint32_t max_chain = chain_on ? ctx->chain_cap : 0u;
    const uint32_t ratio8 = plan_ratio8(kflags);
    ctx->launches += launch_plan(len_used, n, ring, ring_long, chain_list, scratch, /*fresh=*/!resume, max_chain, ratio8, st);
    int* qctl_long = qctl + kLongQctlAfterQctl;
    // How many outliers did the planner pick?  The count is read back (16 bytes, one stream synchronisation after
    // the ~12 us plan kernels) because a chain kernel launched "just in case" is not free: its CTAs ask for half an
    // SM's shared memory and, idle or not, skew where the lane kernel's CTAs land.
    // So: lengths known on the host -> the same selection is computed here (plan_outliers_host); otherwise read back.
    // The same goes for the long lane queue (its launch is sized on the host as well).  A batch too small to have
    // either (nothing reaches kChainMinBlocks) needs no answer at all -- but only the host can know that.
    uint32_t n_chain = 0, n_long = 0;
    if (chain_on || long_cap) {
        const bool mirrored = h_len != nullptr;
        if (mirrored) n_chain = plan_outliers_host(h_len, n, max_chain, ctx->sm_count, long_cap, ratio8, &n_long);
        if (!mirrored || ctx->verify_plan) {
            CU_TRY(ctx, cudaMemcpyAsync(ctx->h_plan, qctl, kPlanReadbackInts * sizeof(int), cudaMemcpyDeviceToHost, st));
            CU_TRY(ctx, cudaStreamSynchronize(st));
            ctx->plan_syncs += 1;
            const uint32_t d_chain = (uint32_t)ctx->h_plan[3], d_long = (uint32_t)ctx->h_plan[kLongQctlAfterQctl + 3];
            if (mirrored && (n_chain != d_chain || n_long != d_long)) {
                char b[160];
                snprintf(b, sizeof b, "plan mismatch: host chain %u long %u, device chain %u long %u", n_chain, n_long, d_chain, d_long);
                return fail(ctx, B200H_E_STATE, b);
            }
            n_chain = d_chain;
            n_long = d_long;
        }
    }
    ctx->last_outliers = n_chain;
    if (n_chain && !shared_scratch) {
        // a private single-message batch: the chain kernel IS the batch, no side stream needed
        ctx->launches += launch_chain_hash(d_base, d_off, len_used, chain_list, qctl, kflags, d_sha, d_md5, states,
                                           resume, n_chain, st);
    } else if (n_chain) {
        // the outliers set the makespan: their CTAs go first (high-priority stream), one per SM
        CU_TRY(ctx, cudaEventRecord(ctx->ev_fork, st));
        CU_TRY(ctx, cudaStreamWaitEvent(ctx->s_chain, ctx->ev_fork, 0));
        ctx->launches += launch_chain_hash(d_base, d_off, len_used, chain_list, qctl, kflags, d_sha, d_md5, states,
                                           resume, n_chain, ctx->s_chain);
        CU_TRY(ctx, cudaEventRecord(ctx->ev_join, ctx->s_chain));
    }
    cudaEvent_t pa, pb;
    if (int rc = prof_begin(ctx, st, &pa, &pb)) return rc;
    // Lane CTAs leave the SMs that host a live chain CTA to the chains (they set the makespan) -- as long as enough SMs
    // stay chain-free for the lane work (chain CTAs sit on at most n_chain SMs, one each).
    const uint32_t lane_flags = (n_chain && n_chain <= ctx->sm_count * 3 / 4 && ctx->yield_chain_sms) ? (kflags | F_YIELD_CHAIN_SMS) : kflags;
    // the short messages (dense, time-sliced), then -- same stream -- the long ones, lane-packed at one warp per SMSP
    const uint64_t n_short = n - n_chain - n_long;
    if (n_short)
        ctx->launches += launch_lane_hash(d_base, d_off, len_used, ring, ring_capacity(n), qctl, qctl, n_short, lane_flags,
                                          d_sha, d_md5, states, st);
    if (n_long)
        ctx->launches += launch_lane_hash(d_base, d_off, len_used, ring_long, kLongRingCapacity, qctl_long, qctl, n_long,
                                          lane_flags, d_sha, d_md5, states, st);
    if (int rc = prof_end(ctx, st, pa, pb)) return rc;
    if (n_chain && shared_scratch) CU_TRY(ctx, cudaStreamWaitEvent(st, ctx->ev_join, 0));
    CU_TRY(ctx, cudaGetLastError());
    if (shared_scratch) {
        CU_TRY(ctx, cudaEventRecord(ctx->ev_scratch, st));
        ctx->scratch_used = true;
    }
    return 0;
}

// memcpy into the pinned staging ring with non-temporal stores (b200pack_copy.cpp: widest store the CPU has).
static inline void stream_copy(uint8_t* dst, const uint8_t* src, size_t n) { b200h_stream_copy(dst, src, n); }

// Copy the packed byte range [lo, hi) of a staged wave into dst (= pinned slot, dst[0] <-> packed byte lo).
// doff[] are the packed offsets (ascending) of messages i0..i1 inside the wave.
// Where the bytes of message i come from: host memory (base + off[i]) or a file (paths[file_of[i]] at byte
// offset off[i]).  File reads go straight into the pinned staging ring with pread -- no intermediate copy.
struct Source {
    const uint8_t* base = nullptr;
    const uint64_t* off = nullptr;
    const char* const* paths = nullptr;
    const uint64_t* file_of = nullptr;
    std::atomic<int>* io_errno = nullptr;  // first I/O failure (errno, or -1 for a short read)
    std::atomic<uint64_t>* io_file = nullptr;
};

// Copy the packed byte range [lo, hi) of a staged wave into dst (= pinned slot, dst[0] <-> packed byte lo).
// doff[] are the packed offsets (ascending) of messages i0..i1 inside the wave.
void pack_range(const Source& src, const uint64_t* len, const uint64_t* doff, uint64_t i0, uint64_t i1, uint64_t lo,
                uint64_t hi, uint8_t* dst) {
    // first message whose packed end is beyond lo
    uint64_t a = i0, b = i1;
    while (a < b) {
        const uint64_t m = (a + b) / 2;
        if (doff[m] + len[m] <= lo) a = m + 1;
        else b = m;
    }
    int fd = -1;
    uint64_t fd_file = ~0ull;
    for (uint64_t i = a; i < i1 && doff[i] < hi; ++i) {
        const uint64_t s = std::max(doff[i], lo), e = std::min(doff[i] + len[i], hi);
        if (e <= s) continue;
        if (!src.paths) {
            stream_copy(dst + (s - lo), src.base + src.off[i] + (s - doff[i]), (size_t)(e - s));
            continue;
        }
        if (src.io_errno->load(std::memory_order_relaxed)) break;
        const uint64_t f = src.file_of[i];
        if (f != fd_file) {
            if (fd >= 0) close(fd);
            fd = open(src.paths[f], O_RDONLY | O_CLOEXEC);
            fd_file = f;
        }
        int err = fd < 0 ? errno : 0;
        uint64_t got = 0;
        const uint64_t want = e - s, at = src.off[i] + (s - doff[i]);
        while (!err && got < want) {
            const ssize_t r = pread(fd, dst + (s - lo) + got, (size_t)(want - got), (off_t)(at + got));
            if (r < 0) {
                if (errno == EINTR) continue;
                err = errno;
            } else if (r == 0) {
                err = -1;  // the file is shorter than the size the caller passed
            } else {
                got += (uint64_t)r;
            }
        }
        if (err) {
            int expected = 0;
            if (src.io_errno->compare_exchange_strong(expected, err)) src.io_file->store(f);
            break;
        }
    }
    if (fd >= 0) close(fd);
}

// Fill dst with the packed byte range [lo, hi) using up to `threads` threads.  The range is cut into grains (>= 1 MiB,
// about eight per thread) that the threads take from a shared counter: with a static split the slot is only as fast as
// its slowest thread, and the packers share their cores with the DMA set-up, Python threads, a second context's team
// and, under torchrun, the other ranks' teams.  (Build machine, a shared 8-core VM, scattered 256 KiB sources into
// 256 MiB slots, best of three runs: two teams of 8 threads at once 44.6 -> 48.1 GiB/s, two teams of 16 39.6 -> 43.6,
// two teams of 4 53.0 -> 55.5; a lone team of 8 swung between 12 and 24 GiB/s with the static split and 17 and 41 with
// grains while a neighbour was busy.)  The threads are the context's PackTeam; the calling thread works too.
void pack_parallel(PackTeam& team, int threads, const Source& src, const uint64_t* len, const uint64_t* doff, uint64_t i0,
                   uint64_t i1, uint64_t lo, uint64_t hi, uint8_t* dst, const cpu_set_t* cpus = nullptr) {
    const uint64_t bytes = hi - lo;
    // memory sources: one thread per >= 4 MiB; file sources: syscalls dominate small files, so also split by count
    uint64_t want = bytes / (4u << 20);
    if (src.paths) want = std::max<uint64_t>(want, (i1 - i0) / 64);
    const int t = (int)std::min<uint64_t>((uint64_t)threads, want);
    if (t <= 1) {
        pack_range(src, len, doff, i0, i1, lo, hi, dst);
        return;
    }
    const uint64_t grain = std::max<uint64_t>(uint64_t(1) << 20, (bytes / ((uint64_t)t * 8) + 4095) & ~uint64_t(4095));
    const uint64_t grains = (bytes + grain - 1) / grain;
    std::atomic<uint64_t> next{0};
    auto work = [&] {
        for (;;) {
            const uint64_t g = next.fetch_add(1, std::memory_order_relaxed);
            if (g >= grains) return;
            const uint64_t a = lo + g * grain, b = std::min(hi, a + grain);
            pack_range(src, len, doff, i0, i1, a, b, dst + (a - lo));
        }
    };
    team.run(t, cpus, work);
}

int hash_batch_host_impl(b200h_ctx* ctx, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint64_t n,
                         uint32_t flags, uint8_t* sha_out, uint8_t* md5_out, uint64_t* trim_out, uint8_t* etag_out,
                         const char* const* paths = nullptr, const uint64_t* file_of = nullptr) {
    if (n == 0) return 0;
    std::atomic<int> io_errno{0};
    std::atomic<uint64_t> io_file{0};
    Source src;
    src.base = base;
    src.off = off;
    src.paths = paths;
    src.file_of = file_of;
    src.io_errno = &io_errno;
    src.io_file = &io_file;
    if (!off || !len) return fail(ctx, B200H_E_INVALID, "offsets/lengths must not be NULL");
    if (!(flags & (B200H_SHA256 | B200H_MD5))) return fail(ctx, B200H_E_INVALID, "flags select neither SHA256 nor MD5");
    if (etag_out && !(flags & B200H_MD5)) return fail(ctx, B200H_E_INVALID, "etag requires B200H_MD5");
    CU_TRY(ctx, cudaSetDevice(ctx->device));

    // Page-locked source?  Then DMA straight from the caller's memory, no staging copy.
    // (Only when the messages cover most of the span they sit in: a wave DMAs its whole [min offset, max end) span,
    // so a sparse selection -- one rank's interleaved shard of a shared buffer -- would copy the gaps too; those
    // are gathered through the staging ring like pageable memory.)
    bool direct = false;
    if (base && !paths) {
        cudaPointerAttributes at;
        if (cudaPointerGetAttributes(&at, base) == cudaSuccess) direct = (at.type == cudaMemoryTypeHost);
        else cudaGetLastError();
        if (direct) {
            uint64_t lo = ~0ull, hi = 0, payload = 0;
            for (uint64_t i = 0; i < n; ++i) {
                lo = std::min(lo, off[i]);
                hi = std::max(hi, off[i] + len[i]);
                payload += len[i];
            }
            if (hi - lo > payload + payload / 4 + (uint64_t(16) << 20)) direct = false;
        }
    }

    if (int rc = ensure_meta(ctx, 2 * n)) return rc;
    uint64_t* doff = ctx->h_meta;      // device-relative offsets
    uint64_t* hlen = ctx->h_meta + n;  // lengths (pinned copy)
    memcpy(hlen, len, n * sizeof(uint64_t));

    // ---- carve the batch into waves that fit one HBM wave slot
    size_t cap = std::max(ctx->dwave_cap, ctx->dwave_want);
    const uint64_t seg_cap = cap & ~uint64_t(63);
    std::vector<Wave> waves;
    {
        uint64_t i = 0;
        while (i < n) {
            Wave w{i, i, 0, 0};
            if (len[i] + 16 > cap) {
                // oversized message: consecutive 64-byte-aligned segments, one wave each
                if (flags & B200H_TRIM_ZEROS)
                    return fail(ctx, B200H_E_INVALID, "B200H_TRIM_ZEROS is not supported for a message larger than one staging wave");
                for (uint64_t s0 = 0; s0 < len[i]; s0 += seg_cap) {
                    Wave sw{i, i + 1, 0, std::min<uint64_t>(seg_cap, len[i] - s0)};
                    sw.seg = (s0 + seg_cap >= len[i]) ? 2 : 1;
                    sw.seg_first = s0 == 0;
                    sw.seg_start = s0;
                    waves.push_back(sw);
                }
                doff[i] = 0;
                i += 1;
                continue;
            }
            if (direct) {
                uint64_t lo = off[i], hi = off[i] + len[i];
                uint64_t j = i + 1;
                for (; j < n; ++j) {
                    if (len[j] + 16 > cap) break;  // oversized: gets its own segment waves
                    const uint64_t nlo = std::min(lo, off[j]), nhi = std::max(hi, off[j] + len[j]);
                    if (nhi - (nlo & ~15ull) > cap) break;
                    lo = nlo;
                    hi = nhi;
                }
                w.i1 = j;
                w.src_lo = lo & ~15ull;  // keep the 16-byte phase of every message
                w.bytes = hi - w.src_lo;
                for (uint64_t k = i; k < j; ++k) doff[k] = off[k] - w.src_lo;
            } else {
                uint64_t used = 0;
                uint64_t j = i;
                for (; j < n; ++j) {
                    const uint64_t need = (len[j] + 15) & ~15ull;
                    if (len[j] + 16 > cap) break;  // oversized: gets its own segment waves
                    if (j > i && used + need > cap) break;
                    doff[j] = used;
                    used += need;
                }
                w.i1 = j;
                w.bytes = used;
            }
            waves.push_back(w);
            i = w.i1;
        }
    }
    size_t need_wave = 16;
    for (auto& w : waves) need_wave = std::max<size_t>(need_wave, w.bytes);
    if (int rc = ensure_wave(ctx, need_wave)) return rc;

    if (int rc = ensure_dev(ctx, ctx->d_off, n * sizeof(uint64_t))) return rc;
    if (int rc = ensure_dev(ctx, ctx->d_len, n * sizeof(uint64_t))) return rc;
    if (int rc = ensure_dev(ctx, ctx->d_trim, n * sizeof(uint64_t))) return rc;
    if (flags & B200H_SHA256)
        if (int rc = ensure_dev(ctx, ctx->d_sha, n * 32)) return rc;
    if (flags & B200H_MD5)
        if (int rc = ensure_dev(ctx, ctx->d_md5, n * 16 + 16)) return rc;
    uint64_t* d_off = (uint64_t*)ctx->d_off.p;
    uint64_t* d_len = (uint64_t*)ctx->d_len.p;
    uint64_t* d_trim = (uint64_t*)ctx->d_trim.p;
    uint8_t* d_sha = (flags & B200H_SHA256) ? (uint8_t*)ctx->d_sha.p : nullptr;
    uint8_t* d_md5 = (flags & B200H_MD5) ? (uint8_t*)ctx->d_md5.p : nullptr;

    CU_TRY(ctx, cudaMemcpyAsync(d_off, doff, n * sizeof(uint64_t), cudaMemcpyHostToDevice, ctx->s_comp));
    CU_TRY(ctx, cudaMemcpyAsync(d_len, hlen, n * sizeof(uint64_t), cudaMemcpyHostToDevice, ctx->s_comp));

    if (int rc = ensure_dev(ctx, ctx->d_small, 256)) return rc;
    uint64_t* d_segmeta = (uint64_t*)((uint8_t*)ctx->d_small.p + 64);
    ChainState* d_segstate = (ChainState*)((uint8_t*)ctx->d_small.p + 128);

    bool pin_used[2] = {false, false};
    int pin_slot = 0;
    for (size_t wi = 0; wi < waves.size(); ++wi) {
        const Wave& w = waves[wi];
        const int slot = (int)(wi & 1);
        // the slot's last reader: an earlier wave of this batch, or b200h_hash_segment_parts_device on another stream
        CU_TRY(ctx, cudaStreamWaitEvent(ctx->s_copy, ctx->ev_consumed[slot], 0));
        // a segment wave is message w.i0 restricted to [seg_start, seg_start + bytes), placed at device offset 0
        const uint64_t seg_off1 = w.seg ? off[w.i0] + w.seg_start : 0, seg_len1 = w.bytes, seg_doff1 = 0;
        const uint64_t seg_file1 = (w.seg && file_of) ? file_of[w.i0] : 0;
        Source seg_src = src;
        seg_src.off = &seg_off1;
        seg_src.file_of = file_of ? &seg_file1 : nullptr;
        if (direct) {
            const uint8_t* from = w.seg ? base + off[w.i0] + w.seg_start : base + w.src_lo;
            if (w.bytes) CU_TRY(ctx, cudaMemcpyAsync(ctx->dwave[slot], from, w.bytes, cudaMemcpyHostToDevice, ctx->s_copy));
        } else {
            for (uint64_t lo = 0; lo < w.bytes; lo += ctx->pin_cap) {
                const uint64_t hi = std::min<uint64_t>(w.bytes, lo + ctx->pin_cap);
                if (pin_used[pin_slot]) CU_TRY(ctx, cudaEventSynchronize(ctx->ev_pin[pin_slot]));
                const cpu_set_t* cpus = ctx->node_cpus_valid ? &ctx->node_cpus : nullptr;
                if (w.seg)
                    pack_parallel(ctx->team, paths ? ctx->io_threads : ctx->pack_threads, seg_src, &seg_len1, &seg_doff1, 0, 1, lo, hi,
                                  ctx->pin[pin_slot], cpus);
                else
                    pack_parallel(ctx->team, paths ? ctx->io_threads : ctx->pack_threads, src, len, doff, w.i0, w.i1, lo, hi,
                                  ctx->pin[pin_slot], cpus);
                if (io_errno.load()) {
                    const int e = io_errno.load();
                    CU_TRY(ctx, cudaDeviceSynchronize());
                    return fail(ctx, B200H_E_IO,
                                std::string("reading ") + paths[io_file.load()] + ": " +
                                    (e == -1 ? "file is shorter than the size passed in" : strerror(e)));
                }
                CU_TRY(ctx, cudaMemcpyAsync(ctx->dwave[slot] + lo, ctx->pin[pin_slot], hi - lo, cudaMemcpyHostToDevice,
                                            ctx->s_copy));
                CU_TRY(ctx, cudaEventRecord(ctx->ev_pin[pin_slot], ctx->s_copy));
                pin_used[pin_slot] = true;
                pin_slot ^= 1;
            }
        }
        CU_TRY(ctx, cudaEventRecord(ctx->ev_copied[slot], ctx->s_copy));
        CU_TRY(ctx, cudaStreamWaitEvent(ctx->s_comp, ctx->ev_copied[slot], 0));
        const uint64_t cnt = w.i1 - w.i0;
        if (w.seg) {
            if (w.seg_first) {
                ChainState iv;
                memcpy(iv.sha, kShaIv, sizeof kShaIv);
                memcpy(iv.md5, kMd5Iv, sizeof kMd5Iv);
                iv.prior_bytes = 0;
                iv.reserved = 0;
                CU_TRY(ctx, cudaMemcpyAsync(d_segstate, &iv, sizeof iv, cudaMemcpyHostToDevice, ctx->s_comp));
            }
            const uint64_t meta[2] = {0, w.bytes};
            CU_TRY(ctx, cudaMemcpyAsync(d_segmeta, meta, sizeof meta, cudaMemcpyHostToDevice, ctx->s_comp));
            const uint32_t f = (flags & (3u | B200H_NO_OUTLIERS)) | (w.seg == 2 ? 0u : kFlagNoFinal);
            const uint64_t seg_bytes = w.bytes;
            if (int rc = enqueue_device_batch(ctx, ctx->dwave[slot], d_segmeta, d_segmeta + 1, 1, f,
                                              d_sha ? d_sha + 32 * w.i0 : nullptr, d_md5 ? d_md5 + 16 * w.i0 : nullptr,
                                              nullptr, d_segstate, ctx->s_comp, &seg_bytes))
                return rc;
            if (w.seg == 2)
                CU_TRY(ctx, cudaMemcpyAsync(d_trim + w.i0, d_len + w.i0, sizeof(uint64_t), cudaMemcpyDeviceToDevice, ctx->s_comp));
            CU_TRY(ctx, cudaEventRecord(ctx->ev_consumed[slot], ctx->s_comp));
            continue;
        }
        if (int rc = enqueue_device_batch(ctx, ctx->dwave[slot], d_off + w.i0, d_len + w.i0, cnt, flags,
                                          d_sha ? d_sha + 32 * w.i0 : nullptr, d_md5 ? d_md5 + 16 * w.i0 : nullptr,
                                          d_trim + w.i0, nullptr, ctx->s_comp, len + w.i0))
            return rc;
        CU_TRY(ctx, cudaEventRecord(ctx->ev_consumed[slot], ctx->s_comp));
    }

    uint8_t* d_etag = nullptr;
    if (etag_out) {
        // MD5 over the concatenated raw part digests, still on the device (blob_utils.py:216-219)
        if (int rc = ensure_dev(ctx, ctx->d_small, 64)) return rc;
        uint64_t meta[2] = {0, n * 16};
        uint64_t* d_meta = (uint64_t*)ctx->d_small.p;
        d_etag = (uint8_t*)ctx->d_small.p + 32;
        CU_TRY(ctx, cudaMemcpyAsync(d_meta, meta, sizeof meta, cudaMemcpyHostToDevice, ctx->s_comp));
        if (int rc = enqueue_device_batch(ctx, d_md5, d_meta, d_meta + 1, 1, B200H_MD5, nullptr, d_etag, nullptr,
                                          nullptr, ctx->s_comp, &meta[1]))
            return rc;
    }
    // The output arrays may live in host OR device memory (cudaMemcpyDefault): a caller that goes on to all-gather
    // the table over NCCL passes device buffers and the digests never visit the host.
    if (flags & B200H_HEX_OUT) {
        // the digest columns leave the device as lowercase ASCII hex (64 / 32 characters per row)
        const bool want_sha = sha_out && d_sha, want_md5 = md5_out && d_md5;
        if (int rc = ensure_dev(ctx, ctx->d_hex, n * 96 + 64)) return rc;
        uint8_t* hex_sha = (uint8_t*)ctx->d_hex.p;
        uint8_t* hex_md5 = hex_sha + n * 64;
        if (want_sha) {
            ctx->launches += launch_hex_rows(d_sha, n * 32, hex_sha, ctx->s_comp);
            CU_TRY(ctx, cudaMemcpyAsync(sha_out, hex_sha, n * 64, cudaMemcpyDefault, ctx->s_comp));
        }
        if (want_md5) {
            ctx->launches += launch_hex_rows(d_md5, n * 16, hex_md5, ctx->s_comp);
            CU_TRY(ctx, cudaMemcpyAsync(md5_out, hex_md5, n * 32, cudaMemcpyDefault, ctx->s_comp));
        }
        CU_TRY(ctx, cudaGetLastError());
    } else {
        if (sha_out && d_sha) CU_TRY(ctx, cudaMemcpyAsync(sha_out, d_sha, n * 32, cudaMemcpyDefault, ctx->s_comp));
        if (md5_out && d_md5) CU_TRY(ctx, cudaMemcpyAsync(md5_out, d_md5, n * 16, cudaMemcpyDefault, ctx->s_comp));
    }
    if (trim_out) CU_TRY(ctx, cudaMemcpyAsync(trim_out, d_trim, n * sizeof(uint64_t), cudaMemcpyDefault, ctx->s_comp));
    if (etag_out) CU_TRY(ctx, cudaMemcpyAsync(etag_out, d_etag, 16, cudaMemcpyDefault, ctx->s_comp));
    CU_TRY(ctx, cudaStreamSynchronize(ctx->s_comp));
    return 0;
}

constexpr uint32_t kPublicFlags = 7u | B200H_NO_OUTLIERS | B200H_HEX_OUT;

// The fixed-size part layout shared by b200h_hash_fixed_parts, b200h_hash_fixed_parts_device and
// b200h_hash_files(part_len > 0): part i of a `len`-byte object starts at i * part_len and holds
// min(part_len, len - i * part_len) bytes, so only the last part may be short and an empty object has no parts.
// Appends the parts to off / ln and returns how many there are.  part_len must be > 0.
uint64_t split_fixed_parts(uint64_t len, uint64_t part_len, std::vector<uint64_t>& off, std::vector<uint64_t>& ln) {
    const uint64_t nparts = len / part_len + (len % part_len != 0);
    off.reserve(off.size() + nparts);
    ln.reserve(ln.size() + nparts);
    for (uint64_t o = 0; o < len; o += part_len) {
        off.push_back(o);
        ln.push_back(std::min(part_len, len - o));
    }
    return nparts;
}

// The file table of the segmented entry points: file f is the concatenation of segments
// [file_first_seg[f], file_first_seg[f + 1]), segment s holding seg_lens[s] bytes (both arrays the caller's).
struct FileTable {
    const uint64_t* seg_lens;
    const uint64_t* file_first_seg;
    std::vector<uint64_t> seg_start;  // offset of every segment in its file
    std::vector<uint64_t> size;       // bytes of every file
};

// Checks the table and fills `t`; returns 0, or B200H_E_INVALID with the reason in `err` (no context needed, so
// b200h_segment_parts_preview runs it without a GPU).
int file_table(const uint64_t* seg_lens, uint64_t nsegs, const uint64_t* file_first_seg, uint64_t nfiles, FileTable& t,
               std::string& err) {
    if (nsegs && !seg_lens) return err = "segments must not be NULL", B200H_E_INVALID;
    if (!file_first_seg) return err = "file_first_seg must not be NULL (it has nfiles + 1 entries)", B200H_E_INVALID;
    if (file_first_seg[0] != 0) return err = "file_first_seg[0] must be 0", B200H_E_INVALID;
    if (file_first_seg[nfiles] != nsegs) return err = "file_first_seg[nfiles] must equal nsegs", B200H_E_INVALID;
    for (uint64_t f = 0; f < nfiles; ++f)
        if (file_first_seg[f + 1] < file_first_seg[f]) return err = "file_first_seg must not decrease", B200H_E_INVALID;
    t.seg_lens = seg_lens;
    t.file_first_seg = file_first_seg;
    t.seg_start.assign(nsegs, 0);
    t.size.assign(nfiles, 0);
    for (uint64_t f = 0; f < nfiles; ++f)
        for (uint64_t s = file_first_seg[f]; s < file_first_seg[f + 1]; ++s) {
            if (t.size[f] + seg_lens[s] < t.size[f]) return err = "a file is larger than 2^64 - 1 bytes", B200H_E_INVALID;
            t.seg_start[s] = t.size[f];
            t.size[f] += seg_lens[s];
        }
    return 0;
}

// Calls piece(segment, offset in the segment, n) for every segment that holds some of the bytes
// [offset, offset + len) of file `file`, in file order; empty segments yield no piece.  len > 0, inside the file.
template <class Piece>
void file_pieces(const FileTable& t, uint64_t file, uint64_t offset, uint64_t len, Piece&& piece) {
    const uint64_t* start = t.seg_start.data();
    // the last segment of the file that starts at or before the first byte (it is not empty: offset < the file's size)
    uint64_t s = std::upper_bound(start + t.file_first_seg[file], start + t.file_first_seg[file + 1], offset) - start - 1;
    for (uint64_t done = 0; done < len; ++s) {
        const uint64_t in = offset + done - start[s];
        if (in >= t.seg_lens[s]) continue;  // an empty segment
        const uint64_t n = std::min(t.seg_lens[s] - in, len - done);
        piece(s, in, n);
        done += n;
    }
}

// Bytes of one element of a B200H_DT_* type; 0 for an unknown code.
static uint64_t dt_bytes(uint64_t t) {
    return t == B200H_DT_F32 ? 4 : t == B200H_DT_F16 || t == B200H_DT_BF16 ? 2 : 0;
}

// Bytes of one image element of a segment's destination type: dt_bytes, or 1 for B200H_DT_F8E4M3 (scaled segments).
static uint64_t image_bytes(uint64_t t) { return t == B200H_DT_F8E4M3 ? 1 : dt_bytes(t); }

static bool converts(const b200h_cast_segment& c) { return c.src_type != c.dst_type; }
static const b200h_cast_segment kNoSegment{};  // what the cast entries pass as their segments when nsegs == 0
static const b200h_scaled_segment kNoScaled{};  // and the scaled entries

// The file table of cast segments (file_table over their image lengths, which `seg_lens` receives) and their source
// ranges as plain segments in `plain` (for segments_on_device).  Checks every rule of a cast segment: known type codes
// (equal codes are 0 or a B200H_DT_* code), a converting segment's length and, with check_ptrs, its address multiples
// of the source element size, and its image offset in its file a multiple of the destination element size.  With
// fp8_ok (scaled segments), B200H_DT_F8E4M3 is a destination type of one byte per element.
static int cast_file_table(const b200h_cast_segment* segs, uint64_t nsegs, const uint64_t* file_first_seg,
                           uint64_t nfiles, bool check_ptrs, std::vector<uint64_t>& seg_lens,
                           std::vector<b200h_segment>& plain, FileTable& t, std::string& err, bool fp8_ok = false) {
    if (nsegs && !segs) return err = "segments must not be NULL", B200H_E_INVALID;
    seg_lens.assign(nsegs, 0);
    plain.assign(nsegs, b200h_segment{nullptr, 0});
    for (uint64_t s = 0; s < nsegs; ++s) {
        const b200h_cast_segment& c = segs[s];
        const std::string name = "segment " + std::to_string(s);
        const uint64_t ss = dt_bytes(c.src_type),
                       ds = fp8_ok && c.dst_type == B200H_DT_F8E4M3 ? 1 : dt_bytes(c.dst_type);
        plain[s] = {c.d_ptr, c.len};
        seg_lens[s] = c.len;
        if (!converts(c)) {
            if (c.src_type && !ss) return err = name + ": unknown element type", B200H_E_INVALID;
            continue;
        }
        if (!ss || !ds) return err = name + ": unknown element type", B200H_E_INVALID;
        if (c.len % ss) return err = name + ": its length is not a multiple of the source element size", B200H_E_INVALID;
        if (check_ptrs && (uintptr_t)c.d_ptr % ss)
            return err = name + ": its address is not a multiple of the source element size", B200H_E_INVALID;
        if (c.len / ss > ~0ull / ds) return err = name + ": its image is larger than 2^64 - 1 bytes", B200H_E_INVALID;
        seg_lens[s] = c.len / ss * ds;
    }
    if (int rc = file_table(segs ? seg_lens.data() : nullptr, nsegs, file_first_seg, nfiles, t, err)) return rc;
    for (uint64_t s = 0; s < nsegs; ++s)
        if (converts(segs[s]) && t.seg_start[s] % image_bytes(segs[s].dst_type))
            return err = "segment " + std::to_string(s) + ": its image starts at file offset " +
                         std::to_string(t.seg_start[s]) + ", not a multiple of the destination element size",
                   B200H_E_INVALID;
    return 0;
}

// The casts of scaled segments (what cast_file_table checks, with fp8_ok), after the rules of a quantizing segment
// (dst_type B200H_DT_F8E4M3) that need no device: its source type, len == R * C * ss, block sizes >= 1, the scale count,
// and with check_ptrs d_amax 4-byte aligned and not NULL.
static int scaled_casts(const b200h_scaled_segment* segs, uint64_t nsegs, bool check_ptrs,
                        std::vector<b200h_cast_segment>& casts, std::string& err) {
    if (nsegs && !segs) return err = "segments must not be NULL", B200H_E_INVALID;
    casts.resize(nsegs);
    for (uint64_t s = 0; s < nsegs; ++s) {
        const b200h_scaled_segment& x = segs[s];
        casts[s] = x.cast;
        if (x.cast.dst_type != B200H_DT_F8E4M3 || !converts(x.cast)) continue;
        const std::string name = "segment " + std::to_string(s);
        const uint64_t ss = dt_bytes(x.cast.src_type);
        if (!ss) return err = name + ": only F32, F16 and BF16 sources quantize", B200H_E_INVALID;
        if (!x.block_rows || !x.block_cols) return err = name + ": block sizes must be >= 1", B200H_E_INVALID;
        if ((unsigned __int128)x.rows * x.cols * ss != x.cast.len)
            return err = name + ": len is not R * C * (source element size)", B200H_E_INVALID;
        const unsigned __int128 nscales = (unsigned __int128)(x.rows / x.block_rows + (x.rows % x.block_rows != 0)) *
                                          (x.cols / x.block_cols + (x.cols % x.block_cols != 0));
        if (nscales > x.scale_count)
            return err = name + ": scale_count is less than ceil(R / block_rows) * ceil(C / block_cols)", B200H_E_INVALID;
        if (check_ptrs && (!x.d_amax || (uintptr_t)x.d_amax % 4))
            return err = name + ": d_amax is NULL or not 4-byte aligned", B200H_E_INVALID;
    }
    return 0;
}

constexpr uint64_t kInPlace = ~0ull;

// Where every part of a segmented batch is hashed: b200h_segment_parts_preview reports it, and
// b200h_hash_segment_parts_device builds its tables from it.  The parts of every file of the table are cut by
// split_fixed_parts and listed file-major.  A part that lies inside one segment is hashed where it is; a part that spans
// two or more segments is gathered into a wave slot at the next multiple of 16.  Waves are contiguous ranges of parts:
// a new wave starts at the gathered part that would take the current wave's staging beyond wave_cap (a wave always
// takes its first gathered part, so a part larger than wave_cap gets a wave of its own).  Parts without a gathered part
// between them share a wave.
struct SegmentParts {
    std::vector<uint64_t> file;      // the file of every part
    std::vector<uint64_t> off, len;  // part i: bytes [off[i], off[i] + len[i]) of its file
    std::vector<uint64_t> seg;       // the segment holding the part's first byte
    std::vector<uint64_t> seg_off;   // offset of that byte inside the segment
    std::vector<uint64_t> stage;     // offset of a gathered part in its wave slot; kInPlace for an in-place part
    std::vector<uint32_t> wave;      // the wave of every part
    std::vector<uint64_t> wave_first;  // first part of every wave, then nparts
    std::vector<uint64_t> wave_bytes;  // staged bytes of every wave
};

// Fills `p`; returns 0, or B200H_E_INVALID with the reason in `err`.  With `casts` (the segments of
// b200h_hash_cast_segment_parts_device), a part is hashed in place only when its segment converts nothing.
int layout_segment_parts(const FileTable& t, uint64_t part_len, uint64_t wave_cap, SegmentParts& p, std::string& err,
                         const b200h_cast_segment* casts = nullptr) {
    if (part_len == 0) return err = "part_len must be > 0", B200H_E_INVALID;
    if (wave_cap == 0) return err = "wave_bytes must be > 0", B200H_E_INVALID;
    for (uint64_t f = 0; f < t.size.size(); ++f) {
        const size_t first = p.off.size();
        split_fixed_parts(t.size[f], part_len, p.off, p.len);
        for (size_t i = first; i < p.off.size(); ++i) {
            uint64_t npieces = 0;
            file_pieces(t, f, p.off[i], p.len[i], [&](uint64_t s, uint64_t in, uint64_t) {
                if (npieces++) return;
                p.seg.push_back(s);
                p.seg_off.push_back(in);
            });
            p.file.push_back(f);
            p.stage.push_back(npieces == 1 && !(casts && converts(casts[p.seg.back()])) ? kInPlace : 0);
        }
    }
    const uint64_t nparts = p.off.size();
    p.wave.resize(nparts);
    uint64_t used = 0;
    for (uint64_t i = 0; i < nparts; ++i) {
        if (i == 0) {
            p.wave_first.push_back(0);
            p.wave_bytes.push_back(0);
        }
        if (p.stage[i] != kInPlace) {
            const uint64_t need = (p.len[i] + 15) & ~15ull;
            if (used && used + need > wave_cap) {
                p.wave_first.push_back(i);
                p.wave_bytes.push_back(0);
                used = 0;
            }
            p.stage[i] = used;
            used += need;
            p.wave_bytes.back() = used;
        }
        p.wave[i] = (uint32_t)(p.wave_first.size() - 1);
    }
    p.wave_first.push_back(nparts);
    return 0;
}

// A pointer that is not memory of ctx's device would fault the kernels, so every device range an entry point takes is
// checked before anything is enqueued: its first and last byte (the allocation in between is the caller's promise).
// Needs cudaSetDevice(ctx->device).
bool device_range_ok(b200h_ctx* ctx, const void* ptr, uint64_t len) {
    if (!len) return true;
    for (const uint8_t* q : {(const uint8_t*)ptr, (const uint8_t*)ptr + (len - 1)}) {
        cudaPointerAttributes at;
        const bool ok = cudaPointerGetAttributes(&at, q) == cudaSuccess &&
                        (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) && at.device == ctx->device;
        cudaGetLastError();
        if (!ok) return false;
    }
    return true;
}

// Every segment an entry point takes, checked before anything is enqueued: not NULL when it has bytes, not wrapping the
// address space, and device_range_ok.  `noun` names a segment in the message.  Needs cudaSetDevice(ctx->device).
int segments_on_device(b200h_ctx* ctx, const b200h_segment* segs, uint64_t n, const char* noun) {
    for (uint64_t i = 0; i < n; ++i) {
        const uintptr_t p = (uintptr_t)segs[i].d_ptr;
        std::string fault;
        if (segs[i].len && !p) fault = " is NULL";
        else if (p + segs[i].len < p) fault = " wraps the address space";
        else if (!device_range_ok(ctx, segs[i].d_ptr, segs[i].len))
            fault = " is not device memory on cuda:" + std::to_string(ctx->device);
        if (!fault.empty()) return fail(ctx, B200H_E_INVALID, noun + (" " + std::to_string(i)) + fault);
    }
    return 0;
}

// The amax arrays of the quantizing segments among segs[0 .. n), checked as segments_on_device checks segments.
static int scales_on_device(b200h_ctx* ctx, const b200h_scaled_segment* segs, uint64_t n) {
    for (uint64_t i = 0; i < n; ++i) {
        const b200h_scaled_segment& x = segs[i];
        if (x.cast.dst_type != B200H_DT_F8E4M3 || !converts(x.cast)) continue;
        if (x.scale_count > ~0ull / 4 || (uintptr_t)x.d_amax + x.scale_count * 4 < (uintptr_t)x.d_amax ||
            !device_range_ok(ctx, x.d_amax, x.scale_count * 4))
            return fail(ctx, B200H_E_INVALID, "segment " + std::to_string(i) + ": its scale_count values at d_amax "
                                              "are not device memory of cuda:" + std::to_string(ctx->device));
    }
    return 0;
}

// The file table of segs[0 .. nsegs) (see file_table); `seg_lens` receives their lengths and backs t.seg_lens.
int segment_file_table(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs, const uint64_t* file_first_seg,
                       uint64_t nfiles, std::vector<uint64_t>& seg_lens, FileTable& t) {
    seg_lens.resize(segs ? nsegs : 0);
    for (uint64_t s = 0; s < seg_lens.size(); ++s) seg_lens[s] = segs[s].len;
    std::string err;
    if (int rc = file_table(segs ? seg_lens.data() : nullptr, nsegs, file_first_seg, nfiles, t, err))
        return fail(ctx, rc, err);
    return 0;
}

// Uploads the tables a, b and c (in that order; c may be empty) into one stream-ordered allocation on `st`, runs
// launch(device a, device b, device c) and frees the allocation behind it: no synchronisation, and no scratch shared
// with other streams' calls.
template <class A, class B, class C, class Launch>
int launch_with_tables(b200h_ctx* ctx, cudaStream_t st, const std::vector<A>& a, const std::vector<B>& b,
                       const std::vector<C>& c, Launch&& launch) {
    const size_t a_bytes = a.size() * sizeof(A), b_bytes = b.size() * sizeof(B), c_bytes = c.size() * sizeof(C);
    void* d_table = nullptr;
    CU_TRY(ctx, cudaMallocAsync(&d_table, a_bytes + b_bytes + c_bytes, st));
    A* d_a = (A*)d_table;
    B* d_b = (B*)((uint8_t*)d_table + a_bytes);
    C* d_c = (C*)((uint8_t*)d_table + a_bytes + b_bytes);
    CU_TRY(ctx, cudaMemcpyAsync(d_a, a.data(), a_bytes, cudaMemcpyHostToDevice, st));
    CU_TRY(ctx, cudaMemcpyAsync(d_b, b.data(), b_bytes, cudaMemcpyHostToDevice, st));
    if (c_bytes) CU_TRY(ctx, cudaMemcpyAsync(d_c, c.data(), c_bytes, cudaMemcpyHostToDevice, st));
    ctx->launches += launch(d_a, d_b, d_c);
    CU_TRY(ctx, cudaGetLastError());
    CU_TRY(ctx, cudaFreeAsync(d_table, st));
    return 0;
}

// launch_with_tables with two tables: launch(device a, device b).
template <class A, class B, class Launch>
int launch_with_tables(b200h_ctx* ctx, cudaStream_t st, const std::vector<A>& a, const std::vector<B>& b,
                       Launch&& launch) {
    return launch_with_tables(ctx, st, a, b, std::vector<uint8_t>{},
                              [&](const A* d_a, const B* d_b, const uint8_t*) { return launch(d_a, d_b); });
}

// The piece of segment s (bytes [in, in + n) of its image) that lands at destination offset `at`: `segs` are the
// source ranges, `casts` (may be NULL) the segments' types.
static CastPiece cast_piece(const b200h_segment* segs, const b200h_cast_segment* casts, uint64_t s, uint64_t in,
                            uint64_t n, uint64_t at) {
    const uint64_t dev = (uint64_t)(uintptr_t)segs[s].d_ptr;
    if (!casts || !converts(casts[s])) return {{dev + in, at, n}, 0, 0, 0, 0};
    const uint64_t ss = dt_bytes(casts[s].src_type), ds = image_bytes(casts[s].dst_type);
    return {{dev + in / ds * ss, at, n}, (uint32_t)casts[s].src_type, (uint32_t)casts[s].dst_type, (uint32_t)(in % ds), 0};
}

// The block scales of the piece of scaled segment s that starts at image byte `in` (zero unless it quantizes).
static PieceScale piece_scale(const b200h_scaled_segment& x, uint64_t in) {
    if (x.cast.dst_type != B200H_DT_F8E4M3 || !converts(x.cast)) return {};
    const uint64_t br = std::min(x.block_rows, x.rows), bc = std::min(x.block_cols, x.cols);
    return {(uint64_t)(uintptr_t)x.d_amax, in, x.cols, br, bc, x.cols / bc + (x.cols % bc != 0)};
}

// Appends the pieces of bytes [offset, offset + len) of file `file` (len > 0) landing at destination offset `at`, in
// file order, and the tiles of their destination bytes (kStageTileBytes each, the last one shorter), which use them.
// With `scaled` (whose casts are `casts`), every piece's block scales go to `scales` as well.
static void range_tables(const FileTable& t, const b200h_segment* segs, const b200h_cast_segment* casts, uint64_t file,
                         uint64_t offset, uint64_t len, uint64_t at, std::vector<CastPiece>& pieces,
                         std::vector<RangeTile>& tiles, const b200h_scaled_segment* scaled = nullptr,
                         std::vector<PieceScale>* scales = nullptr) {
    const size_t first = pieces.size();
    uint64_t h = at;
    file_pieces(t, file, offset, len, [&](uint64_t s, uint64_t in, uint64_t n) {
        pieces.push_back(cast_piece(segs, casts, s, in, n, h));
        if (scaled) scales->push_back(piece_scale(scaled[s], in));
        h += n;
    });
    size_t p = first;
    for (uint64_t o = 0; o < len; o += kStageTileBytes) {
        const uint64_t n = std::min(kStageTileBytes, len - o), d = at + o;
        while (pieces[p].r.host + pieces[p].r.len <= d) ++p;
        size_t q = p;
        while (q + 1 < pieces.size() && pieces[q + 1].r.host < d + n) ++q;
        tiles.push_back({d, (uint32_t)n, (uint32_t)(q - p + 1), (uint64_t)p});
    }
}

// b200h_hash_segment_parts_device with ctx->mu held, on stream `st`.  d_etag_msg != NULL (b200h_hash_fixed_parts_device):
// two more words, the ETag message {0, nparts * 16}, ride the part-table upload, even when there are no parts, and
// *d_etag_msg points at them.  With `casts` (b200h_hash_cast_segment_parts_device; segs is then NULL), the files are
// the cast segments' images, and the parts that are not hashed in place are gathered by stage_ranges_kernel.  With
// `scaled` (b200h_hash_scaled_segment_parts_device; `casts` are then their casts), by stage_scaled_ranges_kernel.
int hash_segment_parts_locked(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs, const uint64_t* file_first_seg,
                              uint64_t nfiles, uint64_t part_len, uint32_t flags, void* d_sha256, void* d_md5,
                              uint64_t* d_trimmed_len, uint64_t* nparts_out, cudaStream_t st, const uint64_t** d_etag_msg,
                              const b200h_cast_segment* casts = nullptr, const b200h_scaled_segment* scaled = nullptr) {
    if (flags & B200H_HEX_OUT) return fail(ctx, B200H_E_INVALID, "B200H_HEX_OUT is not supported for device parts");
    if (((uintptr_t)d_sha256 | (uintptr_t)d_md5) & 15u)
        return fail(ctx, B200H_E_INVALID, "digest outputs must be 16-byte aligned");
    std::vector<uint64_t> seg_lens;
    std::vector<b200h_segment> plain;
    FileTable t;
    std::string err;
    if (casts) {
        if (int rc = cast_file_table(casts, nsegs, file_first_seg, nfiles, true, seg_lens, plain, t, err, scaled))
            return fail(ctx, rc, err);
        segs = plain.data();
    } else if (int rc = segment_file_table(ctx, segs, nsegs, file_first_seg, nfiles, seg_lens, t)) {
        return rc;
    }
    // before the layout, whose part list the segments' lengths size
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    if (int rc = segments_on_device(ctx, segs, nsegs, "segment")) return rc;
    if (scaled)
        if (int rc = scales_on_device(ctx, scaled, nsegs)) return rc;
    SegmentParts p;
    if (int rc = layout_segment_parts(t, part_len, std::max(ctx->dwave_cap, ctx->dwave_want), p, err, casts))
        return fail(ctx, rc, err);
    const uint64_t nparts = p.off.size();
    if (nparts && !(flags & (B200H_SHA256 | B200H_MD5)))
        return fail(ctx, B200H_E_INVALID, "flags select neither SHA256 nor MD5");
    if (nparts_out) *nparts_out = nparts;
    if (nparts == 0 && !d_etag_msg) return 0;
    uint64_t stage_max = 0;
    for (uint64_t b : p.wave_bytes) stage_max = std::max(stage_max, b);
    if (stage_max)
        if (int rc = ensure_wave(ctx, stage_max)) return rc;

    // device table: part addresses | part lengths | [ETag message] | gather tiles (after the gather, every part is an
    // absolute address)
    const size_t nwaves = p.wave_bytes.size();
    std::vector<uint64_t> table(2 * nparts);
    if (d_etag_msg) table.insert(table.end(), {0, nparts * 16});
    std::vector<uint64_t> wave_tiles(nwaves + 1, 0);  // tiles of wave w: [wave_tiles[w], wave_tiles[w + 1])
    std::vector<GatherTile> tiles;
    // with casts: the tables of every wave's stage_ranges_kernel launch (destination offsets in the wave's slot)
    std::vector<std::vector<CastPiece>> cast_pieces(casts ? nwaves : 0);
    std::vector<std::vector<RangeTile>> cast_tiles(casts ? nwaves : 0);
    std::vector<std::vector<PieceScale>> piece_scales(scaled ? nwaves : 0);
    for (size_t w = 0; w < nwaves; ++w) {
        uint8_t* slot = ctx->dwave[w & 1];
        for (uint64_t i = p.wave_first[w]; i < p.wave_first[w + 1]; ++i) {
            table[nparts + i] = p.len[i];
            if (p.stage[i] == kInPlace) {
                table[i] = (uint64_t)(uintptr_t)segs[p.seg[i]].d_ptr + p.seg_off[i];
                continue;
            }
            table[i] = (uint64_t)(uintptr_t)(slot + p.stage[i]);
            if (casts) {
                range_tables(t, segs, casts, p.file[i], p.off[i], p.len[i], p.stage[i], cast_pieces[w], cast_tiles[w],
                             scaled, scaled ? &piece_scales[w] : nullptr);
                continue;
            }
            uint64_t at = table[i];
            file_pieces(t, p.file[i], p.off[i], p.len[i], [&](uint64_t s, uint64_t in, uint64_t n) {
                for (uint64_t k = 0; k < n; k += kGatherTileBytes)
                    tiles.push_back({(uint64_t)(uintptr_t)segs[s].d_ptr + in + k, at + k,
                                     std::min(kGatherTileBytes, n - k)});
                at += n;
            });
        }
        wave_tiles[w + 1] = tiles.size();
    }
    const size_t table_bytes = table.size() * sizeof(uint64_t), tiles_bytes = tiles.size() * sizeof(GatherTile);
    // The table is context scratch like the planner's: it is rewritten only after the last batch that read it.
    if (ctx->scratch_used) CU_TRY(ctx, cudaStreamWaitEvent(st, ctx->ev_scratch, 0));
    if (int rc = ensure_dev(ctx, ctx->d_parts, table_bytes + tiles_bytes)) return rc;
    uint64_t* d_table = (uint64_t*)ctx->d_parts.p;
    GatherTile* d_tiles = (GatherTile*)(d_table + table.size());
    CU_TRY(ctx, cudaMemcpyAsync(d_table, table.data(), table_bytes, cudaMemcpyHostToDevice, st));
    if (tiles_bytes) CU_TRY(ctx, cudaMemcpyAsync(d_tiles, tiles.data(), tiles_bytes, cudaMemcpyHostToDevice, st));
    if (d_etag_msg) *d_etag_msg = d_table + 2 * nparts;
    uint8_t* o_sha = (flags & B200H_SHA256) ? (uint8_t*)d_sha256 : nullptr;
    uint8_t* o_md5 = (flags & B200H_MD5) ? (uint8_t*)d_md5 : nullptr;
    for (size_t w = 0; w < nwaves; ++w) {
        const uint64_t i0 = p.wave_first[w], cnt = p.wave_first[w + 1] - i0;
        const int slot = (int)(w & 1);
        const bool staged = casts ? !cast_tiles[w].empty() : wave_tiles[w + 1] > wave_tiles[w];
        if (staged) {
            // the slot is shared with the *_host entry points and the previous waves: wait for its last reader
            CU_TRY(ctx, cudaStreamWaitEvent(st, ctx->ev_consumed[slot], 0));
            if (scaled) {
                if (int rc = launch_with_tables(ctx, st, cast_tiles[w], cast_pieces[w], piece_scales[w],
                                                [&](const RangeTile* d_ct, const CastPiece* d_cp, const PieceScale* d_ps) {
                                                    return launch_stage_scaled_ranges(d_ct, cast_tiles[w].size(), d_cp,
                                                                                      d_ps, ctx->dwave[slot], st);
                                                }))
                    return rc;
            } else if (casts) {
                if (int rc = launch_with_tables(ctx, st, cast_tiles[w], cast_pieces[w],
                                                [&](const RangeTile* d_ct, const CastPiece* d_cp) {
                                                    return launch_stage_ranges(d_ct, cast_tiles[w].size(), d_cp,
                                                                               ctx->dwave[slot], st);
                                                }))
                    return rc;
            } else {
                ctx->launches += launch_gather_segments(d_tiles + wave_tiles[w], wave_tiles[w + 1] - wave_tiles[w], st);
                CU_TRY(ctx, cudaGetLastError());
            }
        }
        if (int rc = enqueue_device_batch(ctx, nullptr, d_table + i0, d_table + nparts + i0, cnt, flags & kPublicFlags,
                                          o_sha ? o_sha + 32 * i0 : nullptr, o_md5 ? o_md5 + 16 * i0 : nullptr,
                                          d_trimmed_len ? d_trimmed_len + i0 : nullptr, nullptr, st, p.len.data() + i0))
            return rc;
        if (staged) CU_TRY(ctx, cudaEventRecord(ctx->ev_consumed[slot], st));
    }
    return 0;
}

// A small request from one of possibly many concurrent callers: merge it with whatever else arrives while the context
// is busy, run ONE batch, hand every caller its rows.  (See Combiner.)
int combined_hash_batch_host(b200h_ctx* ctx, const uint8_t* base, const uint64_t* off, const uint64_t* len, uint64_t n,
                             uint32_t flags, uint8_t* sha_out, uint8_t* md5_out, uint64_t* trim_out) {
    Combiner& cb = ctx->combiner;
    CombineReq r{base, off, len, n, flags, sha_out, md5_out, trim_out};
    const int k = (flags & B200H_TRIM_ZEROS) ? 1 : 0;
    std::unique_lock<std::mutex> cl(cb.m);
    cb.pending[k].push_back(&r);
    if (cb.leader[k]) {  // somebody is already collecting this group: ride along
        cb.cv_more.notify_one();
        cb.cv_done.wait(cl, [&] { return r.done; });
        return r.rc;
    }
    cb.leader[k] = true;
    if (cb.recent_multi && cb.pending[k].size() < kCombineFull)  // concurrent callers were seen a moment ago
        cb.cv_more.wait_for(cl, std::chrono::microseconds(kCombineWaitUs), [&] { return cb.pending[k].size() >= kCombineFull; });
    cl.unlock();
    std::unique_lock<std::mutex> gl(ctx->mu);  // while the previous group occupies the GPU, callers keep joining this one
    cl.lock();
    std::vector<CombineReq*> grp;
    grp.swap(cb.pending[k]);
    cb.leader[k] = false;
    cb.recent_multi = grp.size() > 1;
    cb.groups += 1;
    cb.requests += grp.size();
    cl.unlock();

    int rc = 0;
    if (grp.size() == 1) {
        rc = hash_batch_host_impl(ctx, base, off, len, n, flags, sha_out, md5_out, trim_out, nullptr);
        gl.unlock();
    } else {
        uint64_t total = 0;
        uint32_t uflags = 0;
        for (CombineReq* q : grp) {
            total += q->n;
            uflags |= q->flags;
        }
        std::vector<uint64_t> aoff(total), alen(total), ttrim(total);
        std::vector<uint8_t> tsha((uflags & B200H_SHA256) ? total * 32 : 0), tmd5((uflags & B200H_MD5) ? total * 16 : 0);
        uint64_t at = 0;
        for (CombineReq* q : grp)
            for (uint64_t i = 0; i < q->n; ++i, ++at) {
                aoff[at] = (uint64_t)(uintptr_t)q->base + q->off[i];  // absolute addresses, base = NULL
                alen[at] = q->len[i];
            }
        rc = total ? hash_batch_host_impl(ctx, nullptr, aoff.data(), alen.data(), total, uflags,
                                          tsha.empty() ? nullptr : tsha.data(), tmd5.empty() ? nullptr : tmd5.data(),
                                          ttrim.data(), nullptr)
                   : 0;
        gl.unlock();
        at = 0;
        for (CombineReq* q : grp) {
            if (!rc) {
                if (q->sha && (q->flags & B200H_SHA256)) memcpy(q->sha, tsha.data() + at * 32, q->n * 32);
                if (q->md5 && (q->flags & B200H_MD5)) memcpy(q->md5, tmd5.data() + at * 16, q->n * 16);
                if (q->trim) memcpy(q->trim, ttrim.data() + at, q->n * sizeof(uint64_t));
            }
            at += q->n;
        }
    }
    cl.lock();
    for (CombineReq* q : grp) {
        q->rc = rc;
        q->done = true;
    }
    cb.cv_done.notify_all();
    return rc;
}

}  // namespace

// =============================================================================================== C ABI

extern "C" {

const char* b200h_version(void) { return kernel_build_info(); }

int b200h_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

const char* b200h_last_error(b200h_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

int b200h_create(int device, size_t pinned_bytes, size_t device_bytes, b200h_ctx** out) {
    if (!out) return fail(nullptr, B200H_E_INVALID, "out is NULL");
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(nullptr, B200H_E_CUDA,
                    std::string("no usable CUDA device (libb200hash has no CPU fallback): ") + cudaGetErrorString(e));
    }
    if (device < 0 || device >= ndev) return fail(nullptr, B200H_E_INVALID, "device index out of range");
    b200h_ctx* ctx = new (std::nothrow) b200h_ctx();
    if (!ctx) return fail(nullptr, B200H_E_NOMEM, "out of host memory");
    ctx->device = device;
    auto bail = [&](int rc) {
        g_create_error = ctx->err;
        b200h_destroy(ctx);
        return rc;
    };
#define CU_INIT(call)                                                                              \
    do {                                                                                           \
        cudaError_t e__ = (call);                                                                  \
        if (e__ != cudaSuccess) {                                                                  \
            ctx->err = std::string(#call " failed: ") + cudaGetErrorString(e__);                   \
            cudaGetLastError();                                                                    \
            return bail(e__ == cudaErrorMemoryAllocation ? B200H_E_NOMEM : B200H_E_CUDA);          \
        }                                                                                          \
    } while (0)
    CU_INIT(cudaSetDevice(device));
    cudaDeviceProp prop;
    CU_INIT(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {  // sm_90a code loads on compute capability 9.0 and nothing else
        ctx->err = "device is not an H100-class GPU (compute capability 9.0; kernels are built for sm_90a only)";
        return bail(B200H_E_CUDA);
    }
    CU_INIT(configure_kernels());
    ctx->chain_cap = (uint32_t)std::min<long>((long)prop.multiProcessorCount * chain_groups_per_cta(), (long)kMaxChain);
    ctx->sm_count = (uint32_t)prop.multiProcessorCount;
    if (const char* e = getenv("B200H_YIELD_CHAIN_SMS")) ctx->yield_chain_sms = atoi(e) != 0;
    CU_INIT(cudaStreamCreateWithFlags(&ctx->s_copy, cudaStreamNonBlocking));
    CU_INIT(cudaStreamCreateWithFlags(&ctx->s_comp, cudaStreamNonBlocking));
    {
        int lo = 0, hi = 0;
        CU_INIT(cudaDeviceGetStreamPriorityRange(&lo, &hi));
        CU_INIT(cudaStreamCreateWithPriority(&ctx->s_chain, cudaStreamNonBlocking, hi));
    }
    CU_INIT(cudaHostAlloc(&ctx->h_plan, 64, cudaHostAllocDefault));
    CU_INIT(cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
    CU_INIT(cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming));
    if (const char* e = getenv("B200H_CHAIN")) {  // tuning knob: 0 disables the outlier path, N >= 2 sets the CTA cap
        const long v = atol(e);
        ctx->chain_enabled = v > 0;
        if (v > 1) ctx->chain_cap = (uint32_t)std::min<long>(v, (long)ctx->chain_cap);  // never above groups x SMs
    }
    for (int s = 0; s < 2; ++s) {
        CU_INIT(cudaEventCreateWithFlags(&ctx->ev_copied[s], cudaEventDisableTiming));
        CU_INIT(cudaEventCreateWithFlags(&ctx->ev_consumed[s], cudaEventDisableTiming));
        CU_INIT(cudaEventCreateWithFlags(&ctx->ev_pin[s], cudaEventDisableTiming));
    }
    CU_INIT(cudaEventCreateWithFlags(&ctx->ev_scratch, cudaEventDisableTiming));
    CU_INIT(cudaEventCreateWithFlags(&ctx->ev_dedupe, cudaEventDisableTiming));
    if (pinned_bytes == 0) pinned_bytes = size_t(512) << 20;
    if (device_bytes == 0) device_bytes = size_t(8) << 30;
    ctx->pin_cap = std::max<size_t>((pinned_bytes / 2) & ~size_t(4095), 1 << 20);
    ctx->dwave_want = std::max<size_t>((device_bytes / 2) & ~size_t(255), 1 << 20);
    for (int s = 0; s < 2; ++s) CU_INIT(cudaHostAlloc(&ctx->pin[s], ctx->pin_cap, cudaHostAllocDefault));
    unsigned hc = std::thread::hardware_concurrency();
    {
        const char* e = getenv("B200H_NUMA");
        if (!(e && atoi(e) == 0)) ctx->node_cpus_valid = gpu_node_cpus(device, &ctx->node_cpus);
    }
    // One process per GPU shares the host with its siblings.  The packers run on the GPU's NUMA node, so what a rank
    // may use is that node's CPUs divided by the ranks whose GPUs hang off the same node (LOCAL_WORLD_SIZE ranks spread
    // over the nodes), and a caller that keeps two batches in flight (the map pump) runs two packer teams at once:
    // 8 ranks x 2 x 16 packers were 256 threads on 128 CPUs in an early 8-GPU run of the pump.
    unsigned share = ctx->node_cpus_valid ? (unsigned)CPU_COUNT(&ctx->node_cpus) : hc;
    if (const char* e = getenv("LOCAL_WORLD_SIZE")) {
        const int lw = atoi(e);
        if (lw > 1) {
            unsigned nodes = 0;
            if (ctx->node_cpus_valid) {
                for (int k = 0; k < 64; ++k) {
                    char path[64];
                    snprintf(path, sizeof path, "/sys/devices/system/node/node%d", k);
                    if (access(path, F_OK) == 0) ++nodes;
                }
            }
            const unsigned per_node = nodes ? ((unsigned)lw + nodes - 1) / nodes : (unsigned)lw;
            share = std::max(4u, share / std::max(1u, per_node));
        }
    }
    ctx->pack_threads = (int)std::min(16u, std::max(2u, share / 2));  // 16: best of 8..64 on a two-socket host
    if (const char* e = getenv("B200H_PACK_THREADS")) ctx->pack_threads = std::max(1, atoi(e));
    ctx->io_threads = (int)std::min(16u, std::max(1u, share));  // measured: 16 > 32 > 64 > 128 (kernel-side contention)
    if (const char* e = getenv("B200H_IO_THREADS")) ctx->io_threads = std::max(1, atoi(e));
    if (const char* e = getenv("B200H_VERIFY_PLAN")) ctx->verify_plan = atoi(e) != 0;
    if (const char* e = getenv("B200H_COMBINE")) ctx->combine_enabled = atoi(e) != 0;
    if (const char* e = getenv("B200H_STREAM_BUF")) {
        const long long v = atoll(e);
        if (v >= 65536) ctx->stream_cap = (size_t)v & ~size_t(63);
    }
#undef CU_INIT
    *out = ctx;
    return 0;
}

void b200h_destroy(b200h_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    for (auto& pr : ctx->prof_events) {
        cudaEventDestroy(pr.first);
        cudaEventDestroy(pr.second);
    }
    for (DevBuf* b : {&ctx->d_off, &ctx->d_len, &ctx->d_order, &ctx->d_trim, &ctx->d_sha, &ctx->d_md5, &ctx->d_scratch,
                      &ctx->d_small, &ctx->d_states, &ctx->d_dedupe, &ctx->d_keys, &ctx->d_trimctl, &ctx->d_hex, &ctx->d_order_long,
                      &ctx->d_parts})
        if (b->p) cudaFree(b->p);
    for (auto& r : ctx->stream_pool) stream_res_destroy(r);
    ctx->stream_pool.clear();
    for (int s = 0; s < 2; ++s) {
        if (ctx->dwave[s]) cudaFree(ctx->dwave[s]);
        if (ctx->pin[s]) cudaFreeHost(ctx->pin[s]);
        if (ctx->ev_copied[s]) cudaEventDestroy(ctx->ev_copied[s]);
        if (ctx->ev_consumed[s]) cudaEventDestroy(ctx->ev_consumed[s]);
        if (ctx->ev_pin[s]) cudaEventDestroy(ctx->ev_pin[s]);
    }
    if (ctx->ev_scratch) cudaEventDestroy(ctx->ev_scratch);
    if (ctx->ev_dedupe) cudaEventDestroy(ctx->ev_dedupe);
    if (ctx->h_meta) cudaFreeHost(ctx->h_meta);
    if (ctx->h_plan) cudaFreeHost(ctx->h_plan);
    if (ctx->s_copy) cudaStreamDestroy(ctx->s_copy);
    if (ctx->s_comp) cudaStreamDestroy(ctx->s_comp);
    if (ctx->s_chain) cudaStreamDestroy(ctx->s_chain);
    if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
    if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
    cudaGetLastError();
    delete ctx;
}

void* b200h_host_alloc(b200h_ctx* ctx, size_t bytes) {
    if (!ctx) return nullptr;
    std::lock_guard<std::mutex> lk(ctx->mu);
    void* p = nullptr;
    if (cudaSetDevice(ctx->device) != cudaSuccess || cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocPortable) != cudaSuccess) {
        ctx->err = std::string("cudaHostAlloc failed: ") + cudaGetErrorString(cudaGetLastError());
        return nullptr;
    }
    return p;
}

void b200h_host_free(b200h_ctx* ctx, void* p) {
    if (!ctx || !p) return;
    std::lock_guard<std::mutex> lk(ctx->mu);
    cudaFreeHost(p);
    cudaGetLastError();
}

int b200h_hash_batch_host(b200h_ctx* ctx, const uint8_t* base, const uint64_t* offsets, const uint64_t* lengths,
                          uint64_t n, uint32_t flags, uint8_t* sha256_out, uint8_t* md5_out,
                          uint64_t* trimmed_len_out) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_hash_batch_host");
    if (n && n <= kCombineMaxN && ctx->combine_enabled && offsets && lengths && (flags & (B200H_SHA256 | B200H_MD5)) &&
        !(flags & B200H_HEX_OUT))
        return combined_hash_batch_host(ctx, base, offsets, lengths, n, flags & kPublicFlags, sha256_out, md5_out,
                                        trimmed_len_out);
    std::lock_guard<std::mutex> lk(ctx->mu);
    return hash_batch_host_impl(ctx, base, offsets, lengths, n, flags & kPublicFlags, sha256_out, md5_out,
                                trimmed_len_out, nullptr);
}

int b200h_hash_batch_device_hl(b200h_ctx* ctx, const void* d_base, const uint64_t* d_offsets, const uint64_t* d_lengths,
                               const uint64_t* h_lengths, uint64_t n, uint32_t flags, void* d_sha256, void* d_md5,
                               uint64_t* d_trimmed_len, void* cuda_stream) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_hash_batch_device");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (n && (!d_offsets || !d_lengths)) return fail(ctx, B200H_E_INVALID, "offsets/lengths must not be NULL");
    if (((uintptr_t)d_sha256 | (uintptr_t)d_md5) & 15u)
        return fail(ctx, B200H_E_INVALID, "digest outputs must be 16-byte aligned");
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->s_comp;
    uint8_t* o_sha = (flags & B200H_SHA256) ? (uint8_t*)d_sha256 : nullptr;
    uint8_t* o_md5 = (flags & B200H_MD5) ? (uint8_t*)d_md5 : nullptr;
    if (!(flags & B200H_HEX_OUT) || !n)
        return enqueue_device_batch(ctx, (const uint8_t*)d_base, d_offsets, d_lengths, n, flags & kPublicFlags, o_sha, o_md5,
                                    d_trimmed_len, nullptr, st, h_lengths);
    // hex columns: the kernels write raw rows into library scratch, hex_rows_kernel expands them into the caller's
    // (twice as wide) buffers, all on `st`
    if (ctx->scratch_used) CU_TRY(ctx, cudaStreamWaitEvent(st, ctx->ev_scratch, 0));
    if (int rc = ensure_dev(ctx, ctx->d_hex, n * 48 + 64)) return rc;
    uint8_t* raw_sha = (uint8_t*)ctx->d_hex.p;
    uint8_t* raw_md5 = raw_sha + n * 32;
    if (int rc = enqueue_device_batch(ctx, (const uint8_t*)d_base, d_offsets, d_lengths, n, flags & kPublicFlags,
                                      o_sha ? raw_sha : nullptr, o_md5 ? raw_md5 : nullptr, d_trimmed_len, nullptr, st, h_lengths))
        return rc;
    if (o_sha) ctx->launches += launch_hex_rows(raw_sha, n * 32, o_sha, st);
    if (o_md5) ctx->launches += launch_hex_rows(raw_md5, n * 16, o_md5, st);
    CU_TRY(ctx, cudaGetLastError());
    CU_TRY(ctx, cudaEventRecord(ctx->ev_scratch, st));  // d_hex is shared scratch like the planner's
    return 0;
}

int b200h_hash_batch_device(b200h_ctx* ctx, const void* d_base, const uint64_t* d_offsets, const uint64_t* d_lengths,
                            uint64_t n, uint32_t flags, void* d_sha256, void* d_md5, uint64_t* d_trimmed_len,
                            void* cuda_stream) {
    return b200h_hash_batch_device_hl(ctx, d_base, d_offsets, d_lengths, nullptr, n, flags, d_sha256, d_md5,
                                      d_trimmed_len, cuda_stream);
}

int b200h_hash_fixed_parts(b200h_ctx* ctx, const uint8_t* base, uint64_t len, uint64_t part_len, uint32_t flags,
                           uint8_t* sha256_out, uint8_t* md5_out, uint64_t* trimmed_len_out, uint8_t etag_md5_out[16],
                           uint64_t* nparts_out) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_hash_fixed_parts");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (part_len == 0) return fail(ctx, B200H_E_INVALID, "part_len must be > 0");
    std::vector<uint64_t> off, ln;
    const uint64_t nparts = split_fixed_parts(len, part_len, off, ln);
    if (nparts_out) *nparts_out = nparts;
    if (nparts == 0) {
        if (etag_md5_out) {
            // md5 of the empty concatenation: hash one empty message
            uint64_t z = 0;
            return hash_batch_host_impl(ctx, base ? base : (const uint8_t*)&z, &z, &z, 1, B200H_MD5, nullptr,
                                        etag_md5_out, nullptr, nullptr);
        }
        return 0;
    }
    return hash_batch_host_impl(ctx, base, off.data(), ln.data(), nparts, flags & kPublicFlags, sha256_out, md5_out,
                                trimmed_len_out, etag_md5_out);
}

int b200h_hash_fixed_parts_device(b200h_ctx* ctx, const void* d_base, uint64_t len, uint64_t part_len, uint32_t flags,
                                  void* d_sha256, void* d_md5, uint64_t* d_trimmed_len, void* d_etag_md5,
                                  uint64_t* nparts_out, void* cuda_stream) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_hash_fixed_parts_device");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (part_len == 0) return fail(ctx, B200H_E_INVALID, "part_len must be > 0");
    const uint64_t nparts = len / part_len + (len % part_len != 0);
    if (d_etag_md5 && !(flags & B200H_MD5)) return fail(ctx, B200H_E_INVALID, "etag requires B200H_MD5");
    if (d_etag_md5 && nparts && !d_md5) return fail(ctx, B200H_E_INVALID, "etag requires the part MD5 output d_md5");
    if ((uintptr_t)d_etag_md5 & 15u) return fail(ctx, B200H_E_INVALID, "digest outputs must be 16-byte aligned");
    if (len && !d_base) return fail(ctx, B200H_E_INVALID, "d_base must not be NULL");
    // the one-segment case of b200h_hash_segment_parts_device: every part is hashed where it is
    const b200h_segment seg = {d_base, len};
    const uint64_t file_first_seg[2] = {0, 1};
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->s_comp;
    const uint64_t* d_etag_msg = nullptr;
    if (int rc = hash_segment_parts_locked(ctx, &seg, 1, file_first_seg, 1, part_len, flags, d_sha256, d_md5, d_trimmed_len,
                                           nparts_out, st, d_etag_md5 ? &d_etag_msg : nullptr))
        return rc;
    if (d_etag_md5) {
        // MD5 over the concatenated raw part MD5s, on the device like the host entry's (an empty object: md5(""))
        const uint64_t etag_len = nparts * 16;
        const uint8_t* etag_src = nparts ? (const uint8_t*)d_md5 : (const uint8_t*)d_etag_msg;
        if (int rc = enqueue_device_batch(ctx, etag_src, d_etag_msg, d_etag_msg + 1, 1, B200H_MD5, nullptr,
                                          (uint8_t*)d_etag_md5, nullptr, nullptr, st, &etag_len))
            return rc;
    }
    return 0;
}

int b200h_hash_segment_parts_device(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs, const uint64_t* file_first_seg,
                                    uint64_t nfiles, uint64_t part_len, uint32_t flags, void* d_sha256, void* d_md5,
                                    uint64_t* d_trimmed_len, uint64_t* nparts_out, void* cuda_stream) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_hash_segment_parts_device");
    std::lock_guard<std::mutex> lk(ctx->mu);
    return hash_segment_parts_locked(ctx, segs, nsegs, file_first_seg, nfiles, part_len, flags, d_sha256, d_md5,
                                     d_trimmed_len, nparts_out, cuda_stream ? (cudaStream_t)cuda_stream : ctx->s_comp,
                                     nullptr);
}

int b200h_hash_cast_segment_parts_device(b200h_ctx* ctx, const b200h_cast_segment* segs, uint64_t nsegs,
                                         const uint64_t* file_first_seg, uint64_t nfiles, uint64_t part_len,
                                         uint32_t flags, void* d_sha256, void* d_md5, uint64_t* d_trimmed_len,
                                         uint64_t* nparts_out, void* cuda_stream) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_hash_cast_segment_parts_device");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (nsegs && !segs) return fail(ctx, B200H_E_INVALID, "segments must not be NULL");
    return hash_segment_parts_locked(ctx, nullptr, nsegs, file_first_seg, nfiles, part_len, flags, d_sha256, d_md5,
                                     d_trimmed_len, nparts_out, cuda_stream ? (cudaStream_t)cuda_stream : ctx->s_comp,
                                     nullptr, segs ? segs : &kNoSegment);
}

int b200h_hash_scaled_segment_parts_device(b200h_ctx* ctx, const b200h_scaled_segment* segs, uint64_t nsegs,
                                           const uint64_t* file_first_seg, uint64_t nfiles, uint64_t part_len,
                                           uint32_t flags, void* d_sha256, void* d_md5, uint64_t* d_trimmed_len,
                                           uint64_t* nparts_out, void* cuda_stream) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_hash_scaled_segment_parts_device");
    std::lock_guard<std::mutex> lk(ctx->mu);
    std::vector<b200h_cast_segment> casts;
    std::string err;
    if (int rc = scaled_casts(segs, nsegs, true, casts, err)) return fail(ctx, rc, err);
    return hash_segment_parts_locked(ctx, nullptr, nsegs, file_first_seg, nfiles, part_len, flags, d_sha256, d_md5,
                                     d_trimmed_len, nparts_out, cuda_stream ? (cudaStream_t)cuda_stream : ctx->s_comp,
                                     nullptr, nsegs ? casts.data() : &kNoSegment, nsegs ? segs : &kNoScaled);
}

int b200h_crc32_device(b200h_ctx* ctx, const b200h_segment* ranges, uint64_t n, uint32_t* d_crc_out, void* cuda_stream) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_crc32_device");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (n && !ranges) return fail(ctx, B200H_E_INVALID, "ranges must not be NULL");
    if (n && !d_crc_out) return fail(ctx, B200H_E_INVALID, "d_crc_out must not be NULL");
    if ((uintptr_t)d_crc_out & 3u) return fail(ctx, B200H_E_INVALID, "d_crc_out must be 4-byte aligned");
    if (n == 0) return 0;
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    if (int rc = segments_on_device(ctx, ranges, n, "range")) return rc;
    if (!device_range_ok(ctx, d_crc_out, n * sizeof(uint32_t)))
        return fail(ctx, B200H_E_INVALID, "d_crc_out is not device memory on cuda:" + std::to_string(ctx->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->s_comp;
    // device table: ranges | chunk prefix (n + 1); the output starts as every range's length term
    std::vector<CrcRange> rs(n);
    std::vector<uint64_t> first(n + 1, 0);
    std::vector<uint32_t> init(n);
    for (uint64_t i = 0; i < n; ++i) {
        rs[i] = {(uint64_t)(uintptr_t)ranges[i].d_ptr, ranges[i].len};
        first[i + 1] = first[i] + (ranges[i].len + kCrcChunkBytes - 1) / kCrcChunkBytes;
        init[i] = crc32_length_term(ranges[i].len);
    }
    CU_TRY(ctx, cudaMemcpyAsync(d_crc_out, init.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    if (first[n] == 0) return 0;
    return launch_with_tables(ctx, st, rs, first, [&](const CrcRange* d_ranges, const uint64_t* d_first) {
        return launch_crc32(d_ranges, d_first, n, first[n], d_crc_out, st);
    });
}

// The device's address of [h, h + bytes), or NULL unless it is page-locked host memory ctx's device can reach
// (pageable memory would fault the kernels).  Needs cudaSetDevice(ctx->device).
static void* pinned_device_pointer(b200h_ctx* ctx, const void* h, uint64_t bytes) {
    void* d = nullptr;
    for (const uint8_t* q : {(const uint8_t*)h, (const uint8_t*)h + (bytes ? bytes - 1 : 0)}) {
        cudaPointerAttributes at;
        const bool ok = cudaPointerGetAttributes(&at, q) == cudaSuccess && at.type == cudaMemoryTypeHost &&
                        cudaHostGetDevicePointer(&d, const_cast<void*>(h), 0) == cudaSuccess && d;
        cudaGetLastError();
        if (!ok) return nullptr;
    }
    return d;
}

// b200h_copy_ranges_to_host (to_host) and b200h_copy_ranges_from_host: range i of the segmented files and bytes
// [host_offsets[i], host_offsets[i] + len) of the page-locked buffer `host` are copied one way or the other.
// b200h_copy_cast_ranges (casts != NULL, segs NULL, to_host): the files are the cast segments' images, and `host` is
// page-locked host memory or memory of ctx's device.
// b200h_copy_scaled_ranges: `scaled` as well, whose casts are `casts`.
static int copy_ranges(b200h_ctx* ctx, bool to_host, const b200h_segment* segs, uint64_t nsegs,
                       const uint64_t* file_first_seg, uint64_t nfiles, const b200h_file_range* ranges, uint64_t nranges,
                       const void* host, uint64_t host_bytes, const uint64_t* host_offsets, void* cuda_stream,
                       const b200h_cast_segment* casts = nullptr, const b200h_scaled_segment* scaled = nullptr) {
    const std::string buf = casts ? "dst" : to_host ? "h_dst" : "h_src", offsets = to_host ? "dst_offsets" : "src_offsets",
                      noun = to_host ? "destination" : "source";
    std::vector<uint64_t> seg_lens;
    std::vector<b200h_segment> plain;
    FileTable t;
    if (casts) {
        std::string err;
        if (int rc = cast_file_table(casts, nsegs, file_first_seg, nfiles, true, seg_lens, plain, t, err, scaled))
            return fail(ctx, rc, err);
        segs = plain.data();
    } else if (int rc = segment_file_table(ctx, segs, nsegs, file_first_seg, nfiles, seg_lens, t)) {
        return rc;
    }
    if (nranges && (!ranges || !host_offsets))
        return fail(ctx, B200H_E_INVALID, "ranges and " + offsets + " must not be NULL");
    if (nranges && !host) return fail(ctx, B200H_E_INVALID, buf + " must not be NULL");
    if ((uintptr_t)host & 15u) return fail(ctx, B200H_E_INVALID, buf + " must be 16-byte aligned");
    std::vector<uint64_t> order;  // the non-empty ranges
    for (uint64_t i = 0; i < nranges; ++i) {
        const b200h_file_range& r = ranges[i];
        const std::string name = "range " + std::to_string(i);
        if (r.file >= nfiles) return fail(ctx, B200H_E_INVALID, name + " names a file that does not exist");
        if (r.offset > t.size[r.file] || r.len > t.size[r.file] - r.offset)
            return fail(ctx, B200H_E_INVALID, name + " reaches past the end of its file");
        if (host_offsets[i] & 15u)
            return fail(ctx, B200H_E_INVALID, name + ": its " + noun + " offset is not a multiple of 16");
        if (host_offsets[i] > host_bytes || r.len > host_bytes - host_offsets[i])
            return fail(ctx, B200H_E_INVALID, name + ": its " + noun + " reaches past " + buf + "_bytes");
        if (r.len) order.push_back(i);
    }
    if (to_host) {  // no host byte may be written twice
        std::sort(order.begin(), order.end(), [&](uint64_t a, uint64_t b) { return host_offsets[a] < host_offsets[b]; });
        for (size_t k = 1; k < order.size(); ++k)
            if (host_offsets[order[k - 1]] + ranges[order[k - 1]].len > host_offsets[order[k]])
                return fail(ctx, B200H_E_INVALID, "the destinations of ranges " + std::to_string(order[k - 1]) + " and " +
                                                      std::to_string(order[k]) + " overlap");
    }
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    if (int rc = segments_on_device(ctx, segs, nsegs, "segment")) return rc;
    if (scaled)
        if (int rc = scales_on_device(ctx, scaled, nsegs)) return rc;
    if (nranges == 0) return 0;
    void* d_host = casts && device_range_ok(ctx, host, host_bytes) ? const_cast<void*>(host)
                                                                   : pinned_device_pointer(ctx, host, host_bytes);
    if (!d_host)
        return fail(ctx, B200H_E_INVALID,
                    buf + (casts ? " is neither device memory on cuda:" + std::to_string(ctx->device) +
                                       " nor page-locked host memory it can reach"
                                 : " is not page-locked host memory reachable from cuda:" +
                                       std::to_string(ctx->device)));
    if (order.empty()) return 0;

    // pieces (range x segment, in file order within a range) and the tiles of host bytes that use them
    std::vector<CastPiece> pieces;
    std::vector<RangeTile> tiles;
    std::vector<PieceScale> scales;
    std::vector<uint64_t> range_of;  // per piece: the range it belongs to (for the overlap message)
    for (uint64_t i = 0; i < nranges; ++i) {
        const b200h_file_range& r = ranges[i];
        if (!r.len) continue;
        range_tables(t, segs, casts, r.file, r.offset, r.len, host_offsets[i], pieces, tiles, scaled, &scales);
        range_of.resize(pieces.size(), i);
    }
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->s_comp;
    if (scaled)
        return launch_with_tables(ctx, st, tiles, pieces, scales,
                                  [&](const RangeTile* d_tiles, const CastPiece* d_pieces, const PieceScale* d_scales) {
                                      return launch_stage_scaled_ranges(d_tiles, tiles.size(), d_pieces, d_scales,
                                                                        d_host, st);
                                  });
    if (to_host)
        return launch_with_tables(ctx, st, tiles, pieces, [&](const RangeTile* d_tiles, const CastPiece* d_pieces) {
            return launch_stage_ranges(d_tiles, tiles.size(), d_pieces, d_host, st);
        });
    std::vector<RangePiece> bytes(pieces.size());
    for (size_t k = 0; k < pieces.size(); ++k) bytes[k] = pieces[k].r;
    // no device byte may be written twice: two files, or two segments of one file, may share a tensor
    std::vector<size_t> by_dev(bytes.size());
    for (size_t k = 0; k < by_dev.size(); ++k) by_dev[k] = k;
    std::sort(by_dev.begin(), by_dev.end(), [&](size_t a, size_t b) { return bytes[a].dev < bytes[b].dev; });
    for (size_t k = 1; k < by_dev.size(); ++k)
        if (bytes[by_dev[k - 1]].dev + bytes[by_dev[k - 1]].len > bytes[by_dev[k]].dev)
            return fail(ctx, B200H_E_INVALID, "ranges " + std::to_string(range_of[by_dev[k - 1]]) + " and " +
                                                  std::to_string(range_of[by_dev[k]]) + " write the same device bytes");
    return launch_with_tables(ctx, st, tiles, bytes, [&](const RangeTile* d_tiles, const RangePiece* d_pieces) {
        return launch_load_ranges(d_tiles, tiles.size(), d_pieces, d_host, st);
    });
}

int b200h_copy_ranges_to_host(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs, const uint64_t* file_first_seg,
                              uint64_t nfiles, const b200h_file_range* ranges, uint64_t nranges, void* h_dst,
                              uint64_t h_dst_bytes, const uint64_t* dst_offsets, void* cuda_stream) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_copy_ranges_to_host");
    std::lock_guard<std::mutex> lk(ctx->mu);
    return copy_ranges(ctx, true, segs, nsegs, file_first_seg, nfiles, ranges, nranges, h_dst, h_dst_bytes, dst_offsets,
                       cuda_stream);
}

int b200h_copy_ranges_from_host(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs, const uint64_t* file_first_seg,
                                uint64_t nfiles, const b200h_file_range* ranges, uint64_t nranges, const void* h_src,
                                uint64_t h_src_bytes, const uint64_t* src_offsets, void* cuda_stream) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_copy_ranges_from_host");
    std::lock_guard<std::mutex> lk(ctx->mu);
    return copy_ranges(ctx, false, segs, nsegs, file_first_seg, nfiles, ranges, nranges, h_src, h_src_bytes, src_offsets,
                       cuda_stream);
}

int b200h_copy_cast_ranges(b200h_ctx* ctx, const b200h_cast_segment* segs, uint64_t nsegs, const uint64_t* file_first_seg,
                           uint64_t nfiles, const b200h_file_range* ranges, uint64_t nranges, void* dst,
                           uint64_t dst_bytes, const uint64_t* dst_offsets, void* cuda_stream) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_copy_cast_ranges");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (nsegs && !segs) return fail(ctx, B200H_E_INVALID, "segments must not be NULL");
    return copy_ranges(ctx, true, nullptr, nsegs, file_first_seg, nfiles, ranges, nranges, dst, dst_bytes, dst_offsets,
                       cuda_stream, segs ? segs : &kNoSegment);
}

int b200h_copy_scaled_ranges(b200h_ctx* ctx, const b200h_scaled_segment* segs, uint64_t nsegs,
                             const uint64_t* file_first_seg, uint64_t nfiles, const b200h_file_range* ranges,
                             uint64_t nranges, void* dst, uint64_t dst_bytes, const uint64_t* dst_offsets,
                             void* cuda_stream) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_copy_scaled_ranges");
    std::lock_guard<std::mutex> lk(ctx->mu);
    std::vector<b200h_cast_segment> casts;
    std::string err;
    if (int rc = scaled_casts(segs, nsegs, true, casts, err)) return fail(ctx, rc, err);
    return copy_ranges(ctx, true, nullptr, nsegs, file_first_seg, nfiles, ranges, nranges, dst, dst_bytes, dst_offsets,
                       cuda_stream, nsegs ? casts.data() : &kNoSegment, nsegs ? segs : &kNoScaled);
}

// b200h_fp8_block_scales: the jobs' tiles.  A tile is up to kScaleTileElems elements of one block: at most
// kScaleTileCols of its columns, and as many of its rows as fill the rest.
constexpr uint64_t kScaleTileElems = 16384, kScaleTileCols = 4096;

int b200h_fp8_block_scales(b200h_ctx* ctx, const b200h_fp8_scale_job* jobs, uint64_t njobs, void* cuda_stream) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_fp8_block_scales");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (njobs && !jobs) return fail(ctx, B200H_E_INVALID, "jobs must not be NULL");
    if (njobs > 0xffffffffull) return fail(ctx, B200H_E_INVALID, "too many jobs");
    std::vector<ScaleJob> table(njobs);
    std::vector<std::pair<uintptr_t, uint64_t>> amax;  // (address, bytes) of every job's a
    uint64_t ntiles = 0, nblocks = 0;
    for (uint64_t i = 0; i < njobs; ++i) {
        const b200h_fp8_scale_job& x = jobs[i];
        const std::string name = "job " + std::to_string(i);
        const uint64_t ss = dt_bytes(x.src_type);
        if (!ss) return fail(ctx, B200H_E_INVALID, name + ": src_type is not F32, F16 or BF16");
        if (!x.rows || !x.cols) return fail(ctx, B200H_E_INVALID, name + ": R and C must be >= 1");
        if (!x.block_rows || !x.block_cols) return fail(ctx, B200H_E_INVALID, name + ": block sizes must be >= 1");
        if ((unsigned __int128)x.rows * x.cols * ss > ~0ull) return fail(ctx, B200H_E_INVALID, name + ": R * C overflows");
        if (!x.d_src || (uintptr_t)x.d_src % ss)
            return fail(ctx, B200H_E_INVALID, name + ": d_src is NULL or not aligned to its element size");
        if (!x.d_scales || !x.d_amax || ((uintptr_t)x.d_scales | (uintptr_t)x.d_amax) % 4)
            return fail(ctx, B200H_E_INVALID, name + ": d_scales and d_amax must be 4-byte aligned, not NULL");
        ScaleJob& J = table[i];
        J.src = (uint64_t)(uintptr_t)x.d_src;
        J.rows = x.rows;
        J.cols = x.cols;
        J.block_rows = std::min(x.block_rows, x.rows);
        J.block_cols = std::min(x.block_cols, x.cols);
        J.scale_cols = J.cols / J.block_cols + (J.cols % J.block_cols != 0);
        J.sub_cols = std::min(J.block_cols, kScaleTileCols);
        J.sub_rows = std::min(J.block_rows, std::max<uint64_t>(1, kScaleTileElems / J.sub_cols));
        J.tile_cols = J.block_cols / J.sub_cols + (J.block_cols % J.sub_cols != 0);
        J.tiles_per_block = (J.block_rows / J.sub_rows + (J.block_rows % J.sub_rows != 0)) * J.tile_cols;
        const uint64_t count = (J.rows / J.block_rows + (J.rows % J.block_rows != 0)) * J.scale_cols;
        J.first_tile = ntiles;
        J.first_block = nblocks;
        J.scales = (uint64_t)(uintptr_t)x.d_scales;
        J.amax = (uint64_t)(uintptr_t)x.d_amax;
        J.src_type = (uint32_t)x.src_type;
        ntiles += count * J.tiles_per_block;
        nblocks += count;
        amax.push_back({J.amax, count * 4});
    }
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    for (uint64_t i = 0; i < njobs; ++i) {
        const b200h_fp8_scale_job& x = jobs[i];
        const uint64_t count = amax[i].second / 4;
        if (!device_range_ok(ctx, x.d_src, x.rows * x.cols * dt_bytes(x.src_type)) ||
            !device_range_ok(ctx, x.d_scales, count * 4) || !device_range_ok(ctx, x.d_amax, count * 4))
            return fail(ctx, B200H_E_INVALID, "job " + std::to_string(i) + ": d_src, d_scales or d_amax is not device "
                                              "memory of cuda:" + std::to_string(ctx->device));
    }
    // a starts as zeros: one memset per contiguous run of the jobs' a arrays
    std::sort(amax.begin(), amax.end());
    std::vector<std::pair<uintptr_t, uint64_t>> runs;
    for (const auto& r : amax) {
        if (!runs.empty() && runs.back().first + runs.back().second > r.first)
            return fail(ctx, B200H_E_INVALID, "the d_amax arrays of two jobs overlap");
        if (!runs.empty() && runs.back().first + runs.back().second == r.first) runs.back().second += r.second;
        else runs.push_back(r);
    }
    if (njobs == 0) return 0;
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->s_comp;
    for (const auto& r : runs) CU_TRY(ctx, cudaMemsetAsync((void*)r.first, 0, r.second, st));
    return launch_with_tables(ctx, st, table, std::vector<uint8_t>{}, [&](const ScaleJob* d_jobs, const uint8_t*) {
        return launch_fp8_block_scales(d_jobs, (uint32_t)njobs, ntiles, nblocks, st);
    });
}

static bool is_fp8(uint64_t t) { return t == B200H_DT_F8E4M3 || t == B200H_DT_F8E5M2; }

// Bytes of one element of a box's type code: dt_bytes, or 1 for code 0 (the bytes as they are) and the FP8 codes.
static uint64_t box_elem_bytes(uint64_t t) { return t && !is_fp8(t) ? dt_bytes(t) : 1; }

static uint64_t ceil_div(uint64_t a, uint64_t b) { return a / b + (a % b != 0); }

// The rules of a scaled box that need no device: its types, block sizes, the scale count and the tensor bounds.
static std::string scaled_box_fault(const b200h_scaled_box& x) {
    const b200h_box& b = x.cast.box;
    if (!is_fp8(x.cast.src_type)) return ": src_type is not an FP8 type";
    if (!dt_bytes(x.cast.dst_type)) return ": dst_type is not F32, F16 or BF16";
    if (!dt_bytes(x.scale_type)) return ": scale_type is not F32, F16 or BF16";
    if (!x.block_rows || !x.block_cols) return ": block sizes must be >= 1";
    const unsigned __int128 nscales =
        (unsigned __int128)ceil_div(x.rows_total, x.block_rows) * ceil_div(x.cols, x.block_cols);
    if (nscales > x.scale_count) return ": scale_count is less than ceil(R / block_rows) * ceil(C / block_cols)";
    if (!x.d_scales) return ": d_scales is NULL";
    if ((uintptr_t)x.d_scales % dt_bytes(x.scale_type)) return ": d_scales is not aligned to its element size";
    if (b.rows && b.width) {  // first_elem + (rows - 1) * src_pitch + width <= R * C
        const unsigned __int128 end =
            (unsigned __int128)x.first_elem + (unsigned __int128)(b.rows - 1) * b.src_pitch + b.width;
        if (end > (unsigned __int128)x.rows_total * x.cols) return ": it reaches past element R * C of its tensor";
    }
    return "";
}

// The rules of a quantizing box that need no device: its types, block sizes, the scale count, a's alignment and the
// weight's bounds.
static std::string quant_box_fault(const b200h_quant_box& x) {
    const b200h_box& b = x.cast.box;
    const uint64_t ss = dt_bytes(x.cast.src_type);
    if (!ss) return ": src_type is not F32, F16 or BF16";
    if (x.cast.dst_type != B200H_DT_F8E4M3) return ": dst_type is not B200H_DT_F8E4M3";
    if (!x.rows_total || !x.cols) return ": R and C must be >= 1";
    if (!x.block_rows || !x.block_cols) return ": block sizes must be >= 1";
    const unsigned __int128 nscales =
        (unsigned __int128)ceil_div(x.rows_total, x.block_rows) * ceil_div(x.cols, x.block_cols);
    if (nscales > x.scale_count) return ": scale_count is less than ceil(R / block_rows) * ceil(C / block_cols)";
    if (!x.d_amax || (uintptr_t)x.d_amax % 4) return ": d_amax is NULL or not 4-byte aligned";
    if (b.rows && b.width) {  // first_elem + ((rows - 1) * src_pitch + width) / ss <= R * C
        const unsigned __int128 end =
            (unsigned __int128)x.first_elem + ((unsigned __int128)(b.rows - 1) * b.src_pitch + b.width) / ss;
        if (end > (unsigned __int128)x.rows_total * x.cols) return ": it reaches past element R * C of its weight";
    }
    return "";
}

// The quantizing entries' own arguments: box i's weight and a (boxes[i] == quant.boxes[i].cast), the bands
// b200h_copy_quant_boxes_from_host finalizes before its copy, and amax: b200h_fp8_amax_boxes_from_host.
struct QuantArgs {
    const b200h_quant_box* boxes;
    const b200h_fp8_band* bands;
    uint64_t nbands;
    bool amax;
};

// b200h_copy_boxes_from_host (cast == false; every box has type code 0 on both sides),
// b200h_copy_cast_boxes_from_host and b200h_copy_scaled_boxes_from_host (`scaled`: box i's scales, boxes[i] ==
// scaled[i].cast): box i of h_src to its packed destination run, its elements converted when its types differ.
// With `quant`, the amax of the boxes (quant->amax) or the bands' finalisation and the quantizing copy.
static int copy_boxes(b200h_ctx* ctx, bool cast, const b200h_segment* segs, uint64_t nsegs,
                      const uint64_t* file_first_seg, uint64_t nfiles, const b200h_cast_box* boxes, uint64_t nboxes,
                      const void* h_src, uint64_t h_src_bytes, void* cuda_stream,
                      const b200h_scaled_box* scaled = nullptr, const QuantArgs* quant = nullptr) {
    std::vector<uint64_t> seg_lens;
    FileTable t;
    if (int rc = segment_file_table(ctx, segs, nsegs, file_first_seg, nfiles, seg_lens, t)) return rc;
    if (nboxes && !boxes) return fail(ctx, B200H_E_INVALID, "boxes must not be NULL");
    if (nboxes && !h_src) return fail(ctx, B200H_E_INVALID, "h_src must not be NULL");
    bool any = false;
    for (uint64_t i = 0; i < nboxes; ++i) {
        const b200h_box& b = boxes[i].box;
        const std::string name = "box " + std::to_string(i);
        const uint64_t ss = box_elem_bytes(boxes[i].src_type), ds = box_elem_bytes(boxes[i].dst_type);
        if (scaled || quant) {
            const std::string fault = scaled ? scaled_box_fault(scaled[i]) : quant_box_fault(quant->boxes[i]);
            if (!fault.empty()) return fail(ctx, B200H_E_INVALID, name + fault);
        } else if (cast) {
            if (!dt_bytes(boxes[i].src_type) || !dt_bytes(boxes[i].dst_type))
                return fail(ctx, B200H_E_INVALID, name + ": unknown element type");
        }
        if (cast) {
            if (boxes[i].src_type == boxes[i].dst_type)
                return fail(ctx, B200H_E_INVALID, name + ": src_type and dst_type are the same");
            if (b.width % ss || b.src_pitch % ss)
                return fail(ctx, B200H_E_INVALID,
                            name + ": width and src_pitch must be multiples of the source element size");
            if (((uintptr_t)h_src + b.src_offset) % ss)
                return fail(ctx, B200H_E_INVALID,
                            name + ": its rows do not start at a multiple of the source element size");
        }
        if (b.file >= nfiles) return fail(ctx, B200H_E_INVALID, name + " names a file that does not exist");
        if (b.width && b.rows > ~0ull / b.width) return fail(ctx, B200H_E_INVALID, name + ": rows * width overflows");
        const uint64_t n = b.rows * b.width;
        if (n / ss > ~0ull / ds) return fail(ctx, B200H_E_INVALID, name + ": its destination size overflows");
        const uint64_t nd = n / ss * ds;  // destination bytes
        if (b.offset > t.size[b.file] || nd > t.size[b.file] - b.offset)
            return fail(ctx, B200H_E_INVALID, name + " reaches past the end of its file");
        if (b.rows > 1 && b.src_pitch < b.width) return fail(ctx, B200H_E_INVALID, name + ": src_pitch is less than width");
        if (!n) continue;
        // src_offset + (rows - 1) * src_pitch + width <= h_src_bytes, without overflow
        const bool fits = (b.rows == 1 || b.src_pitch <= h_src_bytes / (b.rows - 1)) &&
                          b.width <= h_src_bytes - (b.rows - 1) * b.src_pitch &&
                          b.src_offset <= h_src_bytes - (b.rows - 1) * b.src_pitch - b.width;
        if (!fits) return fail(ctx, B200H_E_INVALID, name + ": its source reaches past h_src_bytes");
        if (cast) {  // one segment, so that every destination word holds whole elements
            uint64_t npieces = 0, dev = 0;
            file_pieces(t, b.file, b.offset, nd, [&](uint64_t s, uint64_t in, uint64_t) {
                if (!npieces++) dev = (uint64_t)(uintptr_t)segs[s].d_ptr + in;
            });
            if (npieces != 1) return fail(ctx, B200H_E_INVALID, name + ": its destination crosses a segment edge");
            if (dev % ds)
                return fail(ctx, B200H_E_INVALID,
                            name + ": its destination is not at a multiple of the destination element size");
        }
        any = true;
    }
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    if (int rc = segments_on_device(ctx, segs, nsegs, "segment")) return rc;
    if (scaled) {  // every box's scales in device memory of ctx's device (boxes of one tensor share them: checked once)
        std::vector<std::pair<uintptr_t, uint64_t>> seen;
        for (uint64_t i = 0; i < nboxes; ++i) {
            const b200h_scaled_box& x = scaled[i];
            const std::pair<uintptr_t, uint64_t> at{(uintptr_t)x.d_scales, x.scale_count};
            if (std::find(seen.end() - std::min<size_t>(seen.size(), 8), seen.end(), at) != seen.end()) continue;
            const uint64_t es = dt_bytes(x.scale_type);
            if (x.scale_count > ~0ull / es || at.first + x.scale_count * es < at.first ||
                !device_range_ok(ctx, x.d_scales, x.scale_count * es))
                return fail(ctx, B200H_E_INVALID, "box " + std::to_string(i) + ": its scale_count scales at d_scales "
                                                  "are not device memory of cuda:" + std::to_string(ctx->device));
            seen.push_back(at);
        }
    }
    std::vector<ScaleJob> jobs;  // the bands to finalize (first_block, amax and scales)
    uint64_t nblocks = 0;
    if (quant) {  // every box's a, and every band's a and s, in device memory of ctx's device
        std::vector<std::pair<uintptr_t, uint64_t>> seen;
        for (uint64_t i = 0; i < nboxes; ++i) {
            const b200h_quant_box& x = quant->boxes[i];
            const std::pair<uintptr_t, uint64_t> at{(uintptr_t)x.d_amax, x.scale_count};
            if (std::find(seen.end() - std::min<size_t>(seen.size(), 8), seen.end(), at) != seen.end()) continue;
            if (x.scale_count > ~0ull / 4 || at.first + x.scale_count * 4 < at.first ||
                !device_range_ok(ctx, x.d_amax, x.scale_count * 4))
                return fail(ctx, B200H_E_INVALID, "box " + std::to_string(i) + ": its scale_count values at d_amax "
                                                  "are not device memory of cuda:" + std::to_string(ctx->device));
            seen.push_back(at);
        }
        if (quant->nbands && !quant->bands) return fail(ctx, B200H_E_INVALID, "bands must not be NULL");
        if (quant->nbands > 0xffffffffull) return fail(ctx, B200H_E_INVALID, "too many bands");
        for (uint64_t i = 0; i < quant->nbands; ++i) {
            const b200h_fp8_band& x = quant->bands[i];
            const std::string name = "band " + std::to_string(i);
            if (!x.count) return fail(ctx, B200H_E_INVALID, name + ": count must be >= 1");
            if (!x.d_amax || !x.d_scales || ((uintptr_t)x.d_amax | (uintptr_t)x.d_scales) % 4)
                return fail(ctx, B200H_E_INVALID, name + ": d_amax and d_scales must be 4-byte aligned, not NULL");
            if (x.count > ~0ull / 4 || (uintptr_t)x.d_amax + x.count * 4 < (uintptr_t)x.d_amax ||
                (uintptr_t)x.d_scales + x.count * 4 < (uintptr_t)x.d_scales ||
                !device_range_ok(ctx, x.d_amax, x.count * 4) || !device_range_ok(ctx, x.d_scales, x.count * 4))
                return fail(ctx, B200H_E_INVALID, name + ": d_amax or d_scales is not device memory of cuda:" +
                                                      std::to_string(ctx->device));
            ScaleJob J{};
            J.first_block = nblocks;
            J.amax = (uint64_t)(uintptr_t)x.d_amax;
            J.scales = (uint64_t)(uintptr_t)x.d_scales;
            jobs.push_back(J);
            nblocks += x.count;
        }
    }
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->s_comp;
    auto finalize = [&]() -> int {  // the bands' a and s, before the copy that reads a
        if (jobs.empty()) return 0;
        return launch_with_tables(ctx, st, jobs, std::vector<uint8_t>{}, [&](const ScaleJob* d_jobs, const uint8_t*) {
            return launch_fp8_finalize(d_jobs, (uint32_t)jobs.size(), nblocks, st);
        });
    };
    if (nboxes == 0) return finalize();
    void* d_host = pinned_device_pointer(ctx, h_src, h_src_bytes);
    if (!d_host)
        return fail(ctx, B200H_E_INVALID,
                    "h_src is not page-locked host memory reachable from cuda:" + std::to_string(ctx->device));
    if (!any) return finalize();

    // h_src may sit at any phase (a view into page-locked memory): the kernel reads aligned words from the aligned-down
    // base, so every source offset in the tables is taken from there.  The words it reads hold selected bytes, so they
    // lie in the same page-locked pages as the bytes themselves.
    const uint64_t phase = (uintptr_t)d_host & 15u;
    // pieces (box x segment, in destination order within a box; `host` = offset in the box's packed run) and the tiles
    // of every box's virtual source words (see BoxTile): neither grows with the rows
    std::vector<RangePiece> pieces;
    std::vector<CastTile> tiles;
    std::vector<uint64_t> box_of;   // per piece: the box it belongs to (for the overlap message)
    std::vector<uint64_t> tile_of;  // per tile: its box (for the scaled tiles)
    for (uint64_t i = 0; i < nboxes; ++i) {
        const b200h_box& bx = boxes[i].box;
        const uint64_t ss = box_elem_bytes(boxes[i].src_type), ds = box_elem_bytes(boxes[i].dst_type);
        const uint64_t n = bx.rows * bx.width;
        if (!n) continue;
        CastTile ct{{}, (uint32_t)boxes[i].src_type, (uint32_t)boxes[i].dst_type};
        BoxTile& b = ct.box;
        const bool run = bx.rows == 1 || bx.src_pitch == bx.width;  // one contiguous source run
        b.src = bx.src_offset + phase;
        b.width = run ? n : bx.width;
        b.rows = run ? 1 : bx.rows;
        b.pitch = run ? n : bx.src_pitch;
        b.hull = b.pitch - b.width < 16 ? 0 : ((b.width + 14) >> 4) + 1;
        const uint64_t last = b.src + (b.rows - 1) * b.pitch;  // the last row's first source byte
        const uint64_t nv = b.hull ? (b.rows - 1) * b.hull + ((last + b.width - 1) >> 4) - (last >> 4) + 1
                                   : ((last + b.width - 1) >> 4) - (b.src >> 4) + 1;
        const size_t first = pieces.size();
        uint64_t at = 0;
        file_pieces(t, bx.file, bx.offset, n / ss * ds, [&](uint64_t s, uint64_t in, uint64_t len) {
            pieces.push_back({(uint64_t)(uintptr_t)segs[s].d_ptr + in, at, len});
            box_of.push_back(i);
            at += len;
        });
        size_t p = first;
        for (uint64_t v0 = 0; v0 < nv; v0 += kStageTileBytes / 16) {
            b.v0 = v0;
            b.nv = (uint32_t)std::min(kStageTileBytes / 16, nv - v0);
            b.dlo = box_dest_at(b, v0);
            b.dhi = v0 + b.nv == nv ? n : box_dest_at(b, v0 + b.nv);
            // the pieces that hold the tile's destination bytes (dlo and dhi count source bytes)
            while (pieces[p].host + pieces[p].len <= b.dlo / ss * ds) ++p;
            size_t q = p;
            while (q + 1 < pieces.size() && pieces[q + 1].host < b.dhi / ss * ds) ++q;
            b.first_piece = p;
            b.npieces = (uint32_t)(q - p + 1);
            tiles.push_back(ct);
            tile_of.push_back(i);
        }
    }
    // no device byte may be written twice: two files, or two segments of one file, may share a tensor
    std::vector<size_t> by_dev(pieces.size());
    for (size_t k = 0; k < by_dev.size(); ++k) by_dev[k] = k;
    std::sort(by_dev.begin(), by_dev.end(), [&](size_t a, size_t b) { return pieces[a].dev < pieces[b].dev; });
    for (size_t k = 1; k < by_dev.size(); ++k)
        if (pieces[by_dev[k - 1]].dev + pieces[by_dev[k - 1]].len > pieces[by_dev[k]].dev)
            return fail(ctx, B200H_E_INVALID, "boxes " + std::to_string(box_of[by_dev[k - 1]]) + " and " +
                                                  std::to_string(box_of[by_dev[k]]) + " write the same device bytes");
    const void* d_src = (const uint8_t*)d_host - phase;
    if (quant) {
        std::vector<QuantTile> qt(tiles.size());
        for (size_t k = 0; k < tiles.size(); ++k) {
            const b200h_quant_box& x = quant->boxes[tile_of[k]];
            const uint64_t bc = std::min(x.block_cols, x.cols), br = std::min(x.block_rows, x.rows_total);
            qt[k] = {tiles[k], {(uint64_t)(uintptr_t)x.d_amax, x.first_elem, x.cols, br, bc, ceil_div(x.cols, bc)}};
        }
        if (quant->amax)
            return launch_with_tables(ctx, st, qt, std::vector<uint8_t>{}, [&](const QuantTile* d_tiles, const uint8_t*) {
                return launch_fp8_amax_boxes(d_tiles, qt.size(), d_src, st);
            });
        if (int rc = finalize()) return rc;
        return launch_with_tables(ctx, st, qt, pieces, [&](const QuantTile* d_tiles, const RangePiece* d_pieces) {
            return launch_load_quant_boxes(d_tiles, qt.size(), d_pieces, d_src, st);
        });
    }
    if (scaled) {
        std::vector<ScaledTile> sc(tiles.size());
        for (size_t k = 0; k < tiles.size(); ++k) {
            const b200h_scaled_box& x = scaled[tile_of[k]];
            // a block over the whole dimension (or more) is the dimension, so that no block edge lies past it
            const uint64_t bc = std::min(x.block_cols, x.cols), br = std::min(x.block_rows, x.rows_total);
            sc[k] = {tiles[k], (uint64_t)(uintptr_t)x.d_scales, x.first_elem, x.cols, br, bc, ceil_div(x.cols, bc),
                     (uint32_t)x.scale_type, 0};
        }
        return launch_with_tables(ctx, st, sc, pieces, [&](const ScaledTile* d_tiles, const RangePiece* d_pieces) {
            return launch_load_scaled_boxes(d_tiles, sc.size(), d_pieces, d_src, st);
        });
    }
    return launch_with_tables(ctx, st, tiles, pieces, [&](const CastTile* d_tiles, const RangePiece* d_pieces) {
        return launch_load_boxes(d_tiles, tiles.size(), d_pieces, d_src, st);
    });
}

int b200h_copy_boxes_from_host(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs, const uint64_t* file_first_seg,
                               uint64_t nfiles, const b200h_box* boxes, uint64_t nboxes, const void* h_src,
                               uint64_t h_src_bytes, void* cuda_stream) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_copy_boxes_from_host");
    std::lock_guard<std::mutex> lk(ctx->mu);
    std::vector<b200h_cast_box> casts(boxes ? nboxes : 0);  // type code 0 on both sides: the bytes as they are
    for (uint64_t i = 0; i < casts.size(); ++i) casts[i].box = boxes[i];
    return copy_boxes(ctx, false, segs, nsegs, file_first_seg, nfiles, boxes ? casts.data() : nullptr, nboxes, h_src,
                      h_src_bytes, cuda_stream);
}

int b200h_copy_cast_boxes_from_host(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs,
                                    const uint64_t* file_first_seg, uint64_t nfiles, const b200h_cast_box* boxes,
                                    uint64_t nboxes, const void* h_src, uint64_t h_src_bytes, void* cuda_stream) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_copy_cast_boxes_from_host");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (nboxes && !boxes) return fail(ctx, B200H_E_INVALID, "boxes must not be NULL");
    return copy_boxes(ctx, true, segs, nsegs, file_first_seg, nfiles, boxes, nboxes, h_src, h_src_bytes, cuda_stream);
}

int b200h_copy_scaled_boxes_from_host(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs,
                                      const uint64_t* file_first_seg, uint64_t nfiles, const b200h_scaled_box* boxes,
                                      uint64_t nboxes, const void* h_src, uint64_t h_src_bytes, void* cuda_stream) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_copy_scaled_boxes_from_host");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (nboxes && !boxes) return fail(ctx, B200H_E_INVALID, "boxes must not be NULL");
    std::vector<b200h_cast_box> casts(boxes ? nboxes : 0);
    for (uint64_t i = 0; i < casts.size(); ++i) casts[i] = boxes[i].cast;
    return copy_boxes(ctx, true, segs, nsegs, file_first_seg, nfiles, boxes ? casts.data() : nullptr, nboxes, h_src,
                      h_src_bytes, cuda_stream, boxes);
}

// b200h_fp8_amax_boxes_from_host (bands == nullptr) and b200h_copy_quant_boxes_from_host.
static int quant_boxes(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs, const uint64_t* file_first_seg,
                       uint64_t nfiles, const b200h_quant_box* boxes, uint64_t nboxes, const b200h_fp8_band* bands,
                       uint64_t nbands, bool amax, const void* h_src, uint64_t h_src_bytes, void* cuda_stream) {
    if (nboxes && !boxes) return fail(ctx, B200H_E_INVALID, "boxes must not be NULL");
    std::vector<b200h_cast_box> casts(boxes ? nboxes : 0);
    for (uint64_t i = 0; i < casts.size(); ++i) casts[i] = boxes[i].cast;
    const QuantArgs q{boxes, bands, nbands, amax};
    return copy_boxes(ctx, true, segs, nsegs, file_first_seg, nfiles, boxes ? casts.data() : nullptr, nboxes, h_src,
                      h_src_bytes, cuda_stream, nullptr, &q);
}

int b200h_fp8_amax_boxes_from_host(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs,
                                   const uint64_t* file_first_seg, uint64_t nfiles, const b200h_quant_box* boxes,
                                   uint64_t nboxes, const void* h_src, uint64_t h_src_bytes, void* cuda_stream) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_fp8_amax_boxes_from_host");
    std::lock_guard<std::mutex> lk(ctx->mu);
    return quant_boxes(ctx, segs, nsegs, file_first_seg, nfiles, boxes, nboxes, nullptr, 0, true, h_src, h_src_bytes,
                       cuda_stream);
}

int b200h_copy_quant_boxes_from_host(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs,
                                     const uint64_t* file_first_seg, uint64_t nfiles, const b200h_quant_box* boxes,
                                     uint64_t nboxes, const b200h_fp8_band* bands, uint64_t nbands, const void* h_src,
                                     uint64_t h_src_bytes, void* cuda_stream) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_copy_quant_boxes_from_host");
    std::lock_guard<std::mutex> lk(ctx->mu);
    return quant_boxes(ctx, segs, nsegs, file_first_seg, nfiles, boxes, nboxes, bands, nbands, false, h_src,
                       h_src_bytes, cuda_stream);
}

// ---------------------------------------------------------------------------------------------- files

int b200h_stat_files(b200h_ctx* ctx, const char* const* paths, uint64_t n, uint64_t* sizes_out, uint32_t* modes_out) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_stat_files");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (n && (!paths || !sizes_out)) return fail(ctx, B200H_E_INVALID, "paths/sizes_out must not be NULL");
    std::atomic<int> err{0};
    std::atomic<uint64_t> bad{0};
    const int t = (int)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)ctx->io_threads, n / 256));
    auto work = [&](uint64_t a, uint64_t b) {
        for (uint64_t i = a; i < b && !err.load(std::memory_order_relaxed); ++i) {
            struct stat sb;
            if (stat(paths[i], &sb) != 0 || !S_ISREG(sb.st_mode)) {
                int expected = 0;
                if (err.compare_exchange_strong(expected, errno ? errno : EINVAL)) bad.store(i);
                return;
            }
            sizes_out[i] = (uint64_t)sb.st_size;
            if (modes_out) modes_out[i] = (uint32_t)(sb.st_mode & 07777);
        }
    };
    if (t <= 1) {
        work(0, n);
    } else {
        std::vector<std::thread> th;
        for (int k = 0; k < t; ++k) th.emplace_back(work, n * k / t, n * (k + 1) / t);
        for (auto& x : th) x.join();
    }
    if (err.load()) return fail(ctx, B200H_E_IO, std::string("stat ") + paths[bad.load()] + ": " + strerror(err.load()));
    return 0;
}

int b200h_hash_files(b200h_ctx* ctx, const char* const* paths, uint64_t n, const uint64_t* sizes, uint64_t part_len,
                     uint32_t flags, uint8_t* sha256_out, uint8_t* md5_out, uint64_t* trimmed_len_out) {
    if (!ctx) return B200H_E_INVALID;
    B200H_RANGE("b200h_hash_files");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (n && (!paths || !sizes)) return fail(ctx, B200H_E_INVALID, "paths/sizes must not be NULL");
    // message list: one per file (part_len == 0) or one per part_len-sized part, file-major
    std::vector<uint64_t> off, len, file_of;
    for (uint64_t f = 0; f < n; ++f) {
        if (part_len == 0) {
            off.push_back(0);
            len.push_back(sizes[f]);
            file_of.push_back(f);
        } else {
            file_of.resize(file_of.size() + split_fixed_parts(sizes[f], part_len, off, len), f);
        }
    }
    if (off.empty()) return 0;
    return hash_batch_host_impl(ctx, nullptr, off.data(), len.data(), off.size(), flags & kPublicFlags, sha256_out,
                                md5_out, trimmed_len_out, nullptr, paths, file_of.data());
}

// ------------------------------------------------------------------------------------------ streaming
// A b200h_stream owns a CUDA stream, a pinned accumulation buffer and a device block that holds everything its
// launches touch (chaining state, planner scratch, queue ring, data), so several streams of one context -- the
// reference hashes files from ThreadPool / to_thread workers, one hashlib object each -- advance concurrently on the
// GPU, one chain per stream.  update() only copies into the pinned buffer; every `cap` bytes one absorb is enqueued
// (H2D + plan + chain kernel) and update() returns without waiting for it: the next absorb's bytes are gathered
// while the GPU works on this one.  The host knows every length, so nothing is read back.

extern "C++" {
namespace {

constexpr size_t kStreamStateBytes = 2 * sizeof(ChainState);  // [0] running, [1] scratch copy for digest()
constexpr size_t kStreamMetaOff = kStreamStateBytes;          // 2 x u64
constexpr size_t kStreamOutOff = kStreamMetaOff + 64;         // 32 + 16
constexpr size_t kStreamPlanOff = kStreamOutOff + 64;         // planner scratch + chain list
constexpr size_t kStreamPlanBytes = (kPlanScratchWords + kMaxChain) * sizeof(uint32_t);
constexpr size_t kStreamRingOff = (kStreamPlanOff + kStreamPlanBytes + 127) & ~size_t(127);
constexpr size_t kStreamRingBytes = 32 * sizeof(uint32_t);    // ring_capacity(1)
constexpr size_t kStreamDataOff = (kStreamRingOff + kStreamRingBytes + 255) & ~size_t(255);

int stream_res_acquire(b200h_ctx* ctx, b200h_ctx::StreamBuf* out) {
    if (!ctx->stream_pool.empty()) {
        *out = ctx->stream_pool.back();
        ctx->stream_pool.pop_back();
        return 0;
    }
    b200h_ctx::StreamBuf r;
    cudaError_t e = cudaHostAlloc(&r.h, ctx->stream_cap + 128, cudaHostAllocDefault);  // + pinned {offset, length} slots and digests
    if (e == cudaSuccess) e = cudaMalloc(&r.d, kStreamDataOff + ctx->stream_cap + 64);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&r.st, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&r.ev, cudaEventDisableTiming);
    if (e != cudaSuccess) {
        cudaGetLastError();
        if (r.h) cudaFreeHost(r.h);
        if (r.d) cudaFree(r.d);
        if (r.st) cudaStreamDestroy(r.st);
        if (r.ev) cudaEventDestroy(r.ev);
        return fail(ctx, B200H_E_NOMEM, std::string("stream allocation failed: ") + cudaGetErrorString(e));
    }
    *out = r;
    return 0;
}

void stream_res_destroy(b200h_ctx::StreamBuf& r) {
    if (r.st) cudaStreamSynchronize(r.st);
    if (r.h) cudaFreeHost(r.h);
    if (r.d) cudaFree(r.d);
    if (r.st) cudaStreamDestroy(r.st);
    if (r.ev) cudaEventDestroy(r.ev);
    cudaGetLastError();
    r = b200h_ctx::StreamBuf();
}

int stream_write_iv(b200h_stream* s) {
    b200h_ctx* ctx = s->ctx;
    ChainState init;
    memcpy(init.sha, kShaIv, sizeof kShaIv);
    memcpy(init.md5, kMd5Iv, sizeof kMd5Iv);
    init.prior_bytes = 0;
    init.reserved = 0;
    // {0, cap}: offset and length of every absorb, device-resident for the life of the stream (no per-absorb copy)
    uint64_t* h_meta = reinterpret_cast<uint64_t*>(s->hbuf + s->cap);
    h_meta[0] = 0;
    h_meta[1] = s->cap;
    CU_TRY(ctx, cudaMemcpyAsync(s->d_state, &init, sizeof init, cudaMemcpyHostToDevice, s->res.st));
    CU_TRY(ctx, cudaMemcpyAsync(s->d_meta, h_meta, 2 * sizeof(uint64_t), cudaMemcpyHostToDevice, s->res.st));
    CU_TRY(ctx, cudaStreamSynchronize(s->res.st));  // also drains whatever the stream still had in flight
    s->h2d_pending = false;
    s->fill = 0;
    s->total = 0;
    return 0;
}

// hbuf may be rewritten once the last copy out of it has finished (waits outside the context lock)
int stream_wait_hbuf(b200h_stream* s) {
    if (s->h2d_pending) {
        CU_TRY(s->ctx, cudaEventSynchronize(s->res.ev));
        s->h2d_pending = false;
    }
    return 0;
}

// enqueue: absorb the first `nbytes` (multiple of 64) of hbuf into the running state.  ctx->mu must be held.
int stream_absorb(b200h_stream* s, size_t nbytes) {
    b200h_ctx* ctx = s->ctx;
    if (nbytes != s->cap) return fail(ctx, B200H_E_STATE, "stream absorbs whole buffers only");
    const uint64_t hlen = nbytes;
    cudaStream_t st = s->res.st;
    CU_TRY(ctx, cudaMemcpyAsync(s->d_buf, s->hbuf, nbytes, cudaMemcpyHostToDevice, st));  // pinned: truly asynchronous
    CU_TRY(ctx, cudaEventRecord(s->res.ev, st));
    s->h2d_pending = true;
    return enqueue_device_batch(ctx, s->d_buf, s->d_meta, s->d_meta + 1, 1, (s->flags & 3u) | kFlagNoFinal, nullptr,
                                nullptr, nullptr, s->d_state, st, &hlen, s->d_plan, s->d_ring);
}

}  // namespace
}  // extern "C++"

int b200h_stream_new(b200h_ctx* ctx, uint32_t flags, b200h_stream** out) {
    if (!ctx || !out) return B200H_E_INVALID;
    B200H_RANGE("b200h_stream_new");
    std::lock_guard<std::mutex> lk(ctx->mu);
    *out = nullptr;
    if (!(flags & (B200H_SHA256 | B200H_MD5))) return fail(ctx, B200H_E_INVALID, "flags select neither SHA256 nor MD5");
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    b200h_stream* s = new (std::nothrow) b200h_stream();
    if (!s) return fail(ctx, B200H_E_NOMEM, "out of host memory");
    s->ctx = ctx;
    s->flags = flags & 3u;
    s->cap = ctx->stream_cap;
    if (int rc = stream_res_acquire(ctx, &s->res)) {
        delete s;
        return rc;
    }
    uint8_t* blk = s->res.d;
    s->hbuf = s->res.h;
    s->d_state = (ChainState*)blk;
    s->d_meta = (uint64_t*)(blk + kStreamMetaOff);
    s->d_out = blk + kStreamOutOff;
    s->d_plan = (uint32_t*)(blk + kStreamPlanOff);
    s->d_ring = (uint32_t*)(blk + kStreamRingOff);
    s->d_buf = blk + kStreamDataOff;
    if (int rc = stream_write_iv(s)) {
        stream_res_destroy(s->res);
        delete s;
        return rc;
    }
    *out = s;
    return 0;
}

int b200h_stream_update(b200h_stream* s, const uint8_t* data, uint64_t len) {
    if (!s) return B200H_E_INVALID;
    B200H_RANGE("b200h_stream_update");
    b200h_ctx* ctx = s->ctx;
    if (len && !data) {
        std::lock_guard<std::mutex> lk(ctx->mu);
        return fail(ctx, B200H_E_INVALID, "data is NULL");
    }
    if (cudaSetDevice(ctx->device) != cudaSuccess) {
        std::lock_guard<std::mutex> lk(ctx->mu);
        CU_TRY(ctx, cudaSetDevice(ctx->device));
    }
    s->total += len;
    while (len) {
        if (s->fill == 0)
            if (int rc = stream_wait_hbuf(s)) return rc;
        const size_t take = (size_t)std::min<uint64_t>(len, s->cap - s->fill);
        memcpy(s->hbuf + s->fill, data, take);
        s->fill += take;
        data += take;
        len -= take;
        if (s->fill == s->cap) {
            std::lock_guard<std::mutex> lk(ctx->mu);  // enqueue only: microseconds
            if (int rc = stream_absorb(s, s->cap)) return rc;
            s->fill = 0;
        }
    }
    return 0;
}

int b200h_stream_digest(b200h_stream* s, uint8_t sha256_out[32], uint8_t md5_out[16]) {
    if (!s) return B200H_E_INVALID;
    B200H_RANGE("b200h_stream_digest");
    b200h_ctx* ctx = s->ctx;
    cudaStream_t st = s->res.st;
    uint8_t* host = s->hbuf + s->cap + 64;  // pinned: the copy below only enqueues
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        CU_TRY(ctx, cudaSetDevice(ctx->device));
        // finalise on a scratch copy of the state so that further updates remain possible
        uint64_t* h_meta = reinterpret_cast<uint64_t*>(s->hbuf + s->cap) + 2;  // pinned slot of the digest launch
        h_meta[0] = 0;
        h_meta[1] = s->fill;
        const uint64_t hlen = s->fill;
        CU_TRY(ctx, cudaMemcpyAsync(s->d_state + 1, s->d_state, sizeof(ChainState), cudaMemcpyDeviceToDevice, st));
        if (s->fill) CU_TRY(ctx, cudaMemcpyAsync(s->d_buf, s->hbuf, s->fill, cudaMemcpyHostToDevice, st));
        CU_TRY(ctx, cudaMemcpyAsync(s->d_meta + 2, h_meta, 2 * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
        if (int rc = enqueue_device_batch(ctx, s->d_buf, s->d_meta + 2, s->d_meta + 3, 1, s->flags, s->d_out, s->d_out + 32,
                                          nullptr, s->d_state + 1, st, &hlen, s->d_plan, s->d_ring))
            return rc;
        CU_TRY(ctx, cudaMemcpyAsync(host, s->d_out, 48, cudaMemcpyDeviceToHost, st));
    }
    CU_TRY(ctx, cudaStreamSynchronize(st));  // outside the lock: other streams keep enqueueing meanwhile
    s->h2d_pending = false;
    if (sha256_out && (s->flags & B200H_SHA256)) memcpy(sha256_out, host, 32);
    if (md5_out && (s->flags & B200H_MD5)) memcpy(md5_out, host + 32, 16);
    return 0;
}

int b200h_stream_reset(b200h_stream* s) {
    if (!s) return B200H_E_INVALID;
    std::lock_guard<std::mutex> lk(s->ctx->mu);
    CU_TRY(s->ctx, cudaSetDevice(s->ctx->device));
    return stream_write_iv(s);
}

void b200h_stream_free(b200h_stream* s) {
    if (!s) return;
    cudaSetDevice(s->ctx->device);
    cudaStreamSynchronize(s->res.st);
    cudaGetLastError();
    {
        std::lock_guard<std::mutex> lk(s->ctx->mu);
        if (s->ctx->stream_pool.size() < 64) s->ctx->stream_pool.push_back(s->res);
        else stream_res_destroy(s->res);
    }
    delete s;
}

// ---- dedupe of the digest table ------------------------------------------------------------------

static int dedupe_args_ok(b200h_ctx* ctx, uint64_t n, uint32_t key_bytes) {
    if (!ctx) return B200H_E_INVALID;
    if (key_bytes != 32 && key_bytes != 16) return fail(ctx, B200H_E_INVALID, "key_bytes must be 32 (SHA-256) or 16 (MD5)");
    if (n >= 0x7fffffffull) return fail(ctx, B200H_E_INVALID, "table larger than 2^31-2 rows");
    return 0;
}

int b200h_dedupe_device(b200h_ctx* ctx, const void* d_keys, uint64_t n, uint32_t key_bytes, uint32_t* d_first,
                        uint64_t* d_ndistinct, void* cuda_stream) {
    if (int rc = dedupe_args_ok(ctx, n, key_bytes)) return rc;
    if (n && (!d_keys || !d_first)) return fail(ctx, B200H_E_INVALID, "null device pointer");
    if ((reinterpret_cast<uintptr_t>(d_keys) & 3) != 0) return fail(ctx, B200H_E_INVALID, "d_keys must be 4-byte aligned");
    std::lock_guard<std::mutex> lk(ctx->mu);
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->s_comp;
    if (int rc = ensure_dev(ctx, ctx->d_dedupe, (size_t)dedupe_table_capacity(n) * 2 * sizeof(uint32_t))) return rc;
    if (ctx->dedupe_used) CU_TRY(ctx, cudaStreamWaitEvent(st, ctx->ev_dedupe, 0));  // table shared across streams
    ctx->launches += launch_dedupe(d_keys, n, key_bytes, (uint32_t*)ctx->d_dedupe.p, d_first,
                                   reinterpret_cast<unsigned long long*>(d_ndistinct), st);
    CU_TRY(ctx, cudaGetLastError());
    CU_TRY(ctx, cudaEventRecord(ctx->ev_dedupe, st));
    ctx->dedupe_used = true;
    return 0;
}

int b200h_dedupe_host(b200h_ctx* ctx, const uint8_t* keys, uint64_t n, uint32_t key_bytes, uint32_t* first_out,
                      uint64_t* ndistinct_out) {
    if (int rc = dedupe_args_ok(ctx, n, key_bytes)) return rc;
    if (n && (!keys || !first_out)) return fail(ctx, B200H_E_INVALID, "null pointer");
    if (n == 0) {
        if (ndistinct_out) *ndistinct_out = 0;
        return 0;
    }
    std::lock_guard<std::mutex> lk(ctx->mu);
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->s_comp;
    // device layout: keys | first[n] | ndistinct (8-byte aligned)
    const size_t kb = (size_t)n * key_bytes, fb = ((size_t)n * 4 + 7) & ~size_t(7);
    if (int rc = ensure_dev(ctx, ctx->d_keys, kb + fb + 8)) return rc;
    if (int rc = ensure_dev(ctx, ctx->d_dedupe, (size_t)dedupe_table_capacity(n) * 2 * sizeof(uint32_t))) return rc;
    uint8_t* d = (uint8_t*)ctx->d_keys.p;
    uint32_t* d_first = (uint32_t*)(d + kb);
    unsigned long long* d_cnt = (unsigned long long*)(d + kb + fb);
    if (ctx->dedupe_used) CU_TRY(ctx, cudaStreamWaitEvent(st, ctx->ev_dedupe, 0));
    CU_TRY(ctx, cudaMemcpyAsync(d, keys, kb, cudaMemcpyHostToDevice, st));
    ctx->launches += launch_dedupe(d, n, key_bytes, (uint32_t*)ctx->d_dedupe.p, d_first, d_cnt, st);
    CU_TRY(ctx, cudaGetLastError());
    CU_TRY(ctx, cudaMemcpyAsync(first_out, d_first, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    unsigned long long cnt = 0;
    CU_TRY(ctx, cudaMemcpyAsync(&cnt, d_cnt, 8, cudaMemcpyDeviceToHost, st));
    CU_TRY(ctx, cudaStreamSynchronize(st));
    if (ndistinct_out) *ndistinct_out = cnt;
    return 0;
}

// ------------------------------------------------------------------------------------------ utilities

int b200h_fill_synth_device(b200h_ctx* ctx, void* d_dst, uint64_t nbytes, uint64_t seed, uint64_t start,
                            void* cuda_stream) {
    if (!ctx) return B200H_E_INVALID;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (((uintptr_t)d_dst & 7u) || (start & 7u)) return fail(ctx, B200H_E_INVALID, "dst/start must be 8-byte aligned");
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : ctx->s_comp;
    ctx->launches += launch_fill_synth((uint8_t*)d_dst, nbytes, seed, start, st);
    CU_TRY(ctx, cudaGetLastError());
    return 0;
}

int b200h_pack_preview(const uint8_t* base, const uint64_t* offsets, const uint64_t* lengths, uint64_t n, uint8_t* dst,
                       uint64_t dst_bytes, uint64_t slot_bytes, int threads, uint64_t* packed_offsets_out) {
    if ((!offsets || !lengths) && n) return B200H_E_INVALID;
    if (!dst || threads < 1 || slot_bytes < 4096) return B200H_E_INVALID;
    // the layout a staged wave gets in hash_batch_host_impl: every message at the next multiple of 16
    std::vector<uint64_t> doff(n ? n : 1);
    uint64_t used = 0;
    for (uint64_t i = 0; i < n; ++i) {
        doff[i] = used;
        used += (lengths[i] + 15) & ~15ull;
    }
    if (used > dst_bytes) return B200H_E_INVALID;
    Source src;
    src.base = base;
    src.off = offsets;
    // ... filled slot by slot, as the pinned ring is, by a team that outlives the call like a context's does (one per
    // calling thread here: a context's team is protected by the context mutex, this one by being thread-local)
    static thread_local PackTeam team;
    for (uint64_t lo = 0; lo < used; lo += slot_bytes)
        pack_parallel(team, threads, src, lengths, doff.data(), 0, n, lo, std::min(used, lo + slot_bytes), dst + lo);
    if (packed_offsets_out)
        for (uint64_t i = 0; i < n; ++i) packed_offsets_out[i] = doff[i];
    return 0;
}

int b200h_plan_preview(const uint64_t* lengths, uint64_t n, uint32_t flags, uint32_t sm_count, uint32_t* n_chain_out,
                       uint32_t* n_long_out) {
    if ((!lengths && n) || !sm_count || !(flags & (B200H_SHA256 | B200H_MD5)) || n >= 0x7fffffffull) return B200H_E_INVALID;
    // the same arguments enqueue_device_batch passes for a context on such a device with the default settings
    const uint32_t max_chain = (flags & B200H_NO_OUTLIERS) ? 0u : std::min<uint32_t>(sm_count * 4u, kMaxChain);
    const uint32_t long_cap = std::min<uint32_t>(sm_count * 4u * 32u, kLongRingCapacity);
    uint32_t n_long = 0;
    const uint32_t n_chain = plan_outliers_host(lengths, n, max_chain, sm_count, long_cap, plan_ratio8(flags & 3u), &n_long);
    if (n_chain_out) *n_chain_out = n_chain;
    if (n_long_out) *n_long_out = n_long;
    return 0;
}

// The outputs of the two previews.
static void report_segment_parts(const SegmentParts& p, uint64_t* nparts_out, uint64_t* nwaves_out, uint64_t* seg_out,
                                 uint32_t* wave_out, uint64_t out_cap) {
    const uint64_t nparts = p.off.size();
    if (nparts_out) *nparts_out = nparts;
    if (nwaves_out) *nwaves_out = p.wave_bytes.size();
    for (uint64_t i = 0; i < std::min(nparts, out_cap); ++i) {
        if (seg_out) seg_out[i] = p.stage[i] == kInPlace ? p.seg[i] : kInPlace;
        if (wave_out) wave_out[i] = p.wave[i];
    }
}

int b200h_segment_parts_preview(const uint64_t* seg_lens, uint64_t nsegs, const uint64_t* file_first_seg, uint64_t nfiles,
                                uint64_t part_len, uint64_t wave_bytes, uint64_t* nparts_out, uint64_t* nwaves_out,
                                uint64_t* seg_out, uint32_t* wave_out, uint64_t out_cap) {
    FileTable t;
    SegmentParts p;
    std::string err;
    if (int rc = file_table(seg_lens, nsegs, file_first_seg, nfiles, t, err)) return rc;
    if (int rc = layout_segment_parts(t, part_len, wave_bytes, p, err)) return rc;
    report_segment_parts(p, nparts_out, nwaves_out, seg_out, wave_out, out_cap);
    return 0;
}

int b200h_cast_segment_parts_preview(const b200h_cast_segment* segs, uint64_t nsegs, const uint64_t* file_first_seg,
                                     uint64_t nfiles, uint64_t part_len, uint64_t wave_bytes, uint64_t* nparts_out,
                                     uint64_t* nwaves_out, uint64_t* seg_out, uint32_t* wave_out, uint64_t out_cap) {
    std::vector<uint64_t> seg_lens;
    std::vector<b200h_segment> plain;
    FileTable t;
    SegmentParts p;
    std::string err;
    if (int rc = cast_file_table(segs, nsegs, file_first_seg, nfiles, false, seg_lens, plain, t, err)) return rc;
    if (int rc = layout_segment_parts(t, part_len, wave_bytes, p, err, segs ? segs : &kNoSegment)) return rc;
    report_segment_parts(p, nparts_out, nwaves_out, seg_out, wave_out, out_cap);
    return 0;
}

int b200h_scaled_segment_parts_preview(const b200h_scaled_segment* segs, uint64_t nsegs, const uint64_t* file_first_seg,
                                       uint64_t nfiles, uint64_t part_len, uint64_t wave_bytes, uint64_t* nparts_out,
                                       uint64_t* nwaves_out, uint64_t* seg_out, uint32_t* wave_out, uint64_t out_cap) {
    std::vector<b200h_cast_segment> casts;
    std::vector<uint64_t> seg_lens;
    std::vector<b200h_segment> plain;
    FileTable t;
    SegmentParts p;
    std::string err;
    if (int rc = scaled_casts(segs, nsegs, false, casts, err)) return rc;
    const b200h_cast_segment* cs = nsegs ? casts.data() : &kNoSegment;
    if (int rc = cast_file_table(nsegs ? cs : nullptr, nsegs, file_first_seg, nfiles, false, seg_lens, plain, t, err, true))
        return rc;
    if (int rc = layout_segment_parts(t, part_len, wave_bytes, p, err, cs)) return rc;
    report_segment_parts(p, nparts_out, nwaves_out, seg_out, wave_out, out_cap);
    return 0;
}

int b200h_last_outlier_count(b200h_ctx* ctx, uint32_t* count_out) {
    if (!ctx || !count_out) return B200H_E_INVALID;
    std::lock_guard<std::mutex> lk(ctx->mu);
    *count_out = ctx->last_outliers;
    return 0;
}

int b200h_combine_stats(b200h_ctx* ctx, uint64_t* groups_out, uint64_t* requests_out) {
    if (!ctx) return B200H_E_INVALID;
    std::lock_guard<std::mutex> lk(ctx->combiner.m);
    if (groups_out) *groups_out = ctx->combiner.groups;
    if (requests_out) *requests_out = ctx->combiner.requests;
    return 0;
}

uint64_t b200h_plan_sync_count(b200h_ctx* ctx) {
    if (!ctx) return 0;
    std::lock_guard<std::mutex> lk(ctx->mu);
    return ctx->plan_syncs;
}

uint64_t b200h_launch_count(b200h_ctx* ctx) {
    if (!ctx) return 0;
    std::lock_guard<std::mutex> lk(ctx->mu);
    return ctx->launches;
}

int b200h_profile_enable(b200h_ctx* ctx, int on) {
    if (!ctx) return B200H_E_INVALID;
    std::lock_guard<std::mutex> lk(ctx->mu);
    ctx->profiling = on != 0;
    return 0;
}

int b200h_profile_read(b200h_ctx* ctx, double* ms, uint64_t* launches) {
    if (!ctx) return B200H_E_INVALID;
    std::lock_guard<std::mutex> lk(ctx->mu);
    CU_TRY(ctx, cudaSetDevice(ctx->device));
    for (auto& pr : ctx->prof_events) {
        CU_TRY(ctx, cudaEventSynchronize(pr.second));
        float t = 0.f;
        CU_TRY(ctx, cudaEventElapsedTime(&t, pr.first, pr.second));
        ctx->prof_ms += t;
        ctx->prof_n += 1;
        cudaEventDestroy(pr.first);
        cudaEventDestroy(pr.second);
    }
    ctx->prof_events.clear();
    if (ms) *ms = ctx->prof_ms;
    if (launches) *launches = ctx->prof_n;
    ctx->prof_ms = 0.0;
    ctx->prof_n = 0;
    return 0;
}

}  // extern "C"
