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
// One piece of device memory to copy: absolute addresses, len <= kGatherTileBytes.
struct GatherTile {
    uint64_t src, dst, len;
};
constexpr uint64_t kGatherTileBytes = 64 << 10;
// Every tile's copy, in one launch (any alignment of src and dst).
int launch_gather_segments(const GatherTile* tiles, uint64_t ntiles, cudaStream_t st);

// CRC-32 of device ranges (b200hash_crc32.cu).  A range of L bytes is ceil(L / kCrcChunkBytes) chunks, cut from its end.
struct CrcRange {
    uint64_t ptr, len;
};
constexpr uint64_t kCrcChunkBytes = 16 << 10;
// first[n + 1]: range r owns chunks [first[r], first[r + 1]), nchunks = first[n].  out[r] must hold
// crc32_length_term(len_r) before the launch; the kernel XORs the bytes' contribution into it.  Launches nothing when
// nchunks == 0; returns the number of kernels launched.
int launch_crc32(const CrcRange* ranges, const uint64_t* first, uint64_t n, uint64_t nchunks, uint32_t* out,
                 cudaStream_t st);
// zlib.crc32 of `len` zero-contribution bytes: the 0xFFFFFFFF start register shifted through len bytes, XOR 0xFFFFFFFF
// (host arithmetic on CRC values; no data involved)
uint32_t crc32_length_term(uint64_t len);

// Ranges of segmented device files copied to or from one host buffer (b200hash_stage.cu; a copy out of the device may
// also go to a device buffer, which `host` offsets then count in).  A piece is the part of a range that lies in one
// segment (len > 0); the pieces of a range are listed in file order and cover its bytes of the host buffer without
// gaps.  A tile is up to kStageTileBytes of one range's bytes of the host buffer, starting at a multiple of 16; it uses
// pieces [first_piece, first_piece + npieces), every piece that holds one of its bytes.
struct RangePiece {
    uint64_t dev, host, len;  // device address; byte offset in the host buffer
};
struct RangeTile {
    uint64_t host;  // byte offset in the host buffer
    uint32_t len, npieces;
    uint64_t first_piece;
};
constexpr uint64_t kStageTileBytes = 64 << 10;
// Every tile's copy host -> device, in one launch (none when ntiles == 0); `src` is 16-byte aligned memory the device
// can load from.
int launch_load_ranges(const RangeTile* tiles, uint64_t ntiles, const RangePiece* pieces, const void* src, cudaStream_t st);
// A piece of a range copied out of the device, whose segment may convert its elements on the way.  src_type ==
// dst_type: `r` as in RangePiece, the bytes as they are, phase 0.  Otherwise the piece's bytes are its segment's image
// (the source elements converted, the B200H_DT_* codes of b200hash.h): r.dev is the source address of the element that
// holds the piece's first image byte, which is byte `phase` of that element's converted value; r.host and r.len count
// image bytes.
struct CastPiece {
    RangePiece r;
    uint32_t src_type, dst_type, phase, pad;
};
// Every tile's copy of the pieces' images, in one launch (none when ntiles == 0); `dst` is 16-byte aligned memory the
// device can store to (page-locked host memory or device memory).
int launch_stage_ranges(const RangeTile* tiles, uint64_t ntiles, const CastPiece* pieces, void* dst, cudaStream_t st);

// Boxes of a host buffer copied into segmented device files (load_boxes_kernel, b200hash_stage.cu).  A box is `rows`
// rows of `width` bytes, row r at byte src + r * pitch of the host buffer, packed into one destination run.  Its source
// is read as a stream of aligned 16-byte "virtual" words: when pitch - width < 16 the rows' hulls touch and every word
// of the box's source span is read once (hull == 0: virtual word v is word (src >> 4) + v); otherwise the hulls are
// disjoint and row r owns the `hull` virtual words r * hull + k, holding words ((src + r * pitch) >> 4) + k, the last
// one empty when the row's phase needs one word less.  A tile is up to kStageTileBytes / 16 consecutive virtual words of
// one box; it writes the packed destination bytes [dlo, dhi) whose source lies in its words, through the pieces
// [first_piece, first_piece + npieces) of the box's destination (RangePiece; `host` is the piece's offset in the run).
struct BoxTile {
    uint64_t src, pitch, width, rows, hull;  // the box (rows == 1 or pitch >= width); src from the aligned base
    uint64_t v0;                             // first virtual word
    uint64_t dlo, dhi;                       // packed destination bytes written
    uint64_t first_piece;
    uint32_t nv, npieces;  // virtual words; pieces
};
// The first packed destination byte of the box whose source lies in virtual word v or later (rows * width if none).
__host__ __device__ inline uint64_t box_dest_at(const BoxTile& b, uint64_t v) {
    if (b.hull) {
        const uint64_t r = v / b.hull, k = v % b.hull;
        if (r >= b.rows) return b.rows * b.width;
        const uint64_t s = b.src + r * b.pitch, x = (s >> 4) + k;
        if (x > ((s + b.width - 1) >> 4)) return (r + 1) * b.width;
        return r * b.width + (x * 16 > s ? x * 16 - s : 0);
    }
    if (v == 0) return 0;
    const uint64_t t = ((b.src >> 4) + v) * 16 - b.src, r = t / b.pitch, c = t % b.pitch;
    if (r >= b.rows) return b.rows * b.width;
    return c >= b.width ? (r + 1) * b.width : r * b.width + c;
}
// A tile of a box with its source and destination element types.  Equal types (0 and 0 for a plain box): the bytes as
// they are, `box` as above.  Otherwise two different B200H_DT_* codes of b200hash.h, and the box's elements change type:
// `box` counts source bytes (dlo and dhi included, which are multiples of the source element size), its destination is
// one piece (it lies in one segment) at a device address that is a multiple of the destination element size, and packed
// source byte p of the box lands at destination byte p / (source size) * (destination size).
struct CastTile {
    BoxTile box;
    uint32_t src_type, dst_type;
};
// Every tile's copy host -> device, in one launch (none when ntiles == 0); `src` is 16-byte aligned memory the device can
// load from (the tiles' source offsets count from it).
int launch_load_boxes(const CastTile* tiles, uint64_t ntiles, const RangePiece* pieces, const void* src, cudaStream_t st);
// A tile of a box of FP8 elements (cast.src_type B200H_DT_F8E4M3 or B200H_DT_F8E5M2) dequantized on the way: `cast` as
// above with one-byte source elements, and element (i, j) of the R x C tensor the box is cut from multiplied by scale
// (i / block_rows) * scale_cols + j / block_cols of `scales` (type scale_type, device memory) before it is rounded to
// cast.dst_type.  The tensor element of packed source byte p (counted from the box's first source byte, box.src) is
// first_elem + (row of p) * box.pitch + (column of p): the box's rows are rows of the tensor's row-major storage.
struct ScaledTile {
    CastTile cast;
    uint64_t scales;
    uint64_t first_elem, cols, block_rows, block_cols, scale_cols;
    uint32_t scale_type, pad;
};
// Every tile's copy host -> device, in one launch (load_scaled_boxes_kernel; none when ntiles == 0).
int launch_load_scaled_boxes(const ScaledTile* tiles, uint64_t ntiles, const RangePiece* pieces, const void* src,
                             cudaStream_t st);

// The block scales of a quantizing piece (a CastPiece with dst_type B200H_DT_F8E4M3, whose image has one byte per
// element and phase 0): image byte k of the piece is element first_elem + k of the R x C weight, whose block
// (i / block_rows, j / block_cols) has its clamped amax at amax[(i / block_rows) * scale_cols + j / block_cols].  Block
// sizes are clamped to the dimensions.  Unused (zero) for the other pieces.
struct PieceScale {
    uint64_t amax;
    uint64_t first_elem, cols, block_rows, block_cols, scale_cols;
};
// Every tile's copy of the pieces' images, quantizing pieces included (stage_scaled_ranges_kernel); scales[k] goes with
// pieces[k].
int launch_stage_scaled_ranges(const RangeTile* tiles, uint64_t ntiles, const CastPiece* pieces,
                               const PieceScale* scales, void* dst, cudaStream_t st);

// One weight of b200h_fp8_block_scales, split into tiles: a tile is up to sub_rows x sub_cols elements of one block
// (tiles_per_block of them per block, tile_cols across its columns); the job's tiles are numbered from first_tile and its
// blocks from first_block (a flat numbering over every job of the call).
struct ScaleJob {
    uint64_t src;
    uint64_t rows, cols, block_rows, block_cols, scale_cols;  // block sizes clamped to the dimensions
    uint64_t sub_rows, sub_cols, tile_cols, tiles_per_block;
    uint64_t first_tile, first_block;
    uint64_t scales, amax;  // F32 outputs; amax starts as zeros and receives the bits of max |x| first
    uint32_t src_type, pad;
};
// The amax reduction and the finalisation of a and s (two launches; amax must be zero before them).
int launch_fp8_block_scales(const ScaleJob* jobs, uint32_t njobs, uint64_t ntiles, uint64_t nblocks, cudaStream_t st);
// The finalisation alone (fp8_finalize_kernel; one launch, none when nblocks == 0): of the jobs only first_block, amax
// and scales are read.
int launch_fp8_finalize(const ScaleJob* jobs, uint32_t njobs, uint64_t nblocks, cudaStream_t st);

// A tile of a box of F32 / F16 / BF16 elements quantized to E4M3 on the way in: `cast` as for CastTile (dst_type
// B200H_DT_F8E4M3, one destination byte per element), and q as for a quantizing piece, with q.first_elem the weight's
// element of the box's first source byte; the element of packed source byte p (row r, column c of the box) is
// q.first_elem + r * box.pitch / ss + c / ss.  q.amax holds the weight's a.
struct QuantTile {
    CastTile cast;
    PieceScale q;
};
// The amax of every tile's elements into q.amax (atomicMax over the bits of |x|; fp8_amax_boxes_kernel), and the
// quantizing copy (load_quant_boxes_kernel) that reads the finalized a: one launch each, none when ntiles == 0.
int launch_fp8_amax_boxes(const QuantTile* tiles, uint64_t ntiles, const void* src, cudaStream_t st);
int launch_load_quant_boxes(const QuantTile* tiles, uint64_t ntiles, const RangePiece* pieces, const void* src,
                            cudaStream_t st);

int chain_groups_per_cta();        // long messages one chain CTA can host (one CTA per SM)
int device_sm_count();             // SMs of the current device (as seen by configure_kernels)
cudaError_t configure_kernels();  // one-time cudaFuncSetAttribute calls for the current device
const char* kernel_build_info();

}  // namespace b200h
