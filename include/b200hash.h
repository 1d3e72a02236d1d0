/*
 * b200hash.h -- C ABI of libb200hash.so: batched SHA-256 + MD5 content hashing on NVIDIA H100 (sm_90a).
 *
 * The reference (modal-labs/modal-client) has no FFI for this path: its seam is a set of Python
 * module-level functions that call hashlib.  Each entry point below names the reference call site(s)
 * it replaces (paths relative to the reference root).  INTEGRATION.md shows the ctypes stub a
 * maintainer would add to py/modal/_utils/hash_utils.py / blob_utils.py, and the cgo stub for go/blob.go.
 *
 * Conventions
 *   - every function returning int returns 0 on success and a negative B200H_E_* code on failure;
 *     b200h_last_error(ctx) gives a message (owned by the library, valid until the next call on ctx);
 *   - no exceptions cross the boundary; the caller owns every buffer it passes;
 *   - a context is bound to one CUDA device; batch calls on one context are serialised internally
 *     (thread-safe, re-entrant across contexts); the caller's GIL is never needed.  Concurrent SMALL
 *     b200h_hash_batch_host calls (<= 1024 messages each) are merged into one GPU batch by a combining queue
 *     (the first caller in leads, the others ride along and get their own rows back), and every b200h_stream
 *     runs on its own CUDA stream, so the reference's thread-pool callers overlap on the GPU;
 *   - there is NO CPU fallback: without a usable CUDA device b200h_create fails with B200H_E_CUDA.
 *   - digests are raw bytes: SHA-256 = 32 bytes (big-endian words, FIPS 180-4), MD5 = 16 bytes (RFC 1321).
 */
#ifndef B200HASH_H
#define B200HASH_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200H_SHA256 1u     /* compute SHA-256 */
#define B200H_MD5 2u        /* compute MD5 */
#define B200H_TRIM_ZEROS 4u /* hash the prefix up to the last non-zero byte (volumefs2 blocks) */
#define B200H_HEX_OUT 32u /* the digest outputs receive lowercase ASCII hex (64 chars per SHA-256 row, 32 per MD5
                             row; buffers twice as wide) formatted on the device: the column MountFile.sha256_hex /
                             FileUploadSpec.md5_hex carry (modal_proto/api.proto:2582-2587), straight from the table */
#define B200H_NO_OUTLIERS 16u /* keep every message on the lane kernel (no outlier routing): with it
                                 b200h_hash_batch_device never reads anything back, i.e. only enqueues */

#define B200H_OK 0
#define B200H_E_INVALID (-1) /* bad argument */
#define B200H_E_CUDA (-2)    /* CUDA runtime / driver error (no device, launch failure, ...) */
#define B200H_E_NOMEM (-3)   /* host or device allocation failed */
#define B200H_E_STATE (-4)   /* object used in the wrong state (e.g. update after final) */
#define B200H_E_IO (-5)      /* a file could not be opened / read (b200h_stat_files, b200h_hash_files) */

typedef struct b200h_ctx b200h_ctx;
typedef struct b200h_stream b200h_stream;

/* ---- lifecycle ------------------------------------------------------------------------------- */

/* Bind a context to CUDA device `device`.  pinned_bytes / device_bytes size the host staging ring and
 * the HBM staging buffers used by the *_host entry points (0 = defaults: 512 MiB pinned, 8 GiB HBM,
 * both split in two for double buffering).  A message larger than one HBM wave slot is hashed in
 * consecutive segments with the chaining state kept on the device, so message size is not limited by them. */
int b200h_create(int device, size_t pinned_bytes, size_t device_bytes, b200h_ctx** out);
void b200h_destroy(b200h_ctx* ctx);
/* ctx may be NULL: returns the message of the last failed b200h_create on this thread. */
const char* b200h_last_error(b200h_ctx* ctx);
const char* b200h_version(void);
int b200h_device_count(void);

/* Page-locked host memory the *_host entry points can DMA from directly (no staging copy). */
void* b200h_host_alloc(b200h_ctx* ctx, size_t bytes);
void b200h_host_free(b200h_ctx* ctx, void* p);
/* The staging copy the *_host entry points use to fill their pinned ring: memcpy with non-temporal stores, widest
 * store the CPU has (AVX-512 / AVX2 / plain; picked once at run time, B200H_COPY_ISA caps the choice).  Exported for
 * callers that fill page-locked memory from b200h_host_alloc themselves (a serializer writing its output where the
 * DMA engine can take it) and for the CPU tests.  Needs no context and no GPU.  The reference has no counterpart. */
void b200h_stream_copy(void* dst, const void* src, size_t n);
const char* b200h_stream_copy_isa(void); /* "avx512" | "avx2" | "plain": what b200h_stream_copy runs on this CPU */

/* ---- batch hashing ---------------------------------------------------------------------------- */

/* Hash n independent messages that live in HOST memory; message i is base[offsets[i] .. +lengths[i]).
 * (base may be NULL with absolute addresses in offsets[].)  Outputs (each may be NULL): sha256_out[n*32],
 * md5_out[n*16], trimmed_len_out[n] (length actually hashed; == lengths[i] unless B200H_TRIM_ZEROS).
 * Stages through pinned memory to HBM with cudaMemcpyAsync in double-buffered waves; blocks until the
 * digests are in the output arrays.  The output arrays may be host or device memory (copied with
 * cudaMemcpyDefault): a caller that all-gathers the table over NCCL next passes device buffers.
 * Replaces: hashlib in hash_utils.get_upload_hashes (py/modal/_utils/hash_utils.py:68-101) as called per
 * payload from blob_utils.py:345 (map pump) and per file from blob_utils.py:459-474 (FileUploadSpec);
 * with B200H_TRIM_ZEROS: _find_end_of_block + _hash_range_sha256 (blob_utils.py:640-705);
 * md5.Sum/sha256.Sum256 in go/blob.go:51-52. */
int b200h_hash_batch_host(b200h_ctx* ctx, const uint8_t* base, const uint64_t* offsets, const uint64_t* lengths,
                          uint64_t n, uint32_t flags, uint8_t* sha256_out, uint8_t* md5_out,
                          uint64_t* trimmed_len_out);

/* Same, but every pointer is a DEVICE pointer on ctx's device and the call only enqueues work on
 * `cuda_stream` (a cudaStream_t; NULL = the context's compute stream).  d_sha256/d_md5 must be 16-byte
 * aligned.  This is the HBM-resident path the roofline is quoted on.
 * Outlier routing (a few very long messages go to the chain kernel, whose launch is sized on the host) needs the
 * planner's count.  Three ways, in order of preference:
 *   b200h_hash_batch_device_hl  the caller also holds the lengths on the host (h_lengths[n] == d_lengths[n]): the
 *                               library computes the same selection there; the call ONLY ENQUEUES;
 *   flags | B200H_NO_OUTLIERS   no outlier routing for this batch (right for many similar messages); ONLY ENQUEUES;
 *   neither                     the count is read back after the ~12 us planning kernels: one synchronisation of
 *                               `cuda_stream` per call (also whenever B200H_TRIM_ZEROS is set and outliers are on:
 *                               the lengths that matter then exist on the device only). */
int b200h_hash_batch_device(b200h_ctx* ctx, const void* d_base, const uint64_t* d_offsets, const uint64_t* d_lengths,
                            uint64_t n, uint32_t flags, void* d_sha256, void* d_md5, uint64_t* d_trimmed_len,
                            void* cuda_stream);
int b200h_hash_batch_device_hl(b200h_ctx* ctx, const void* d_base, const uint64_t* d_offsets, const uint64_t* d_lengths,
                               const uint64_t* h_lengths, uint64_t n, uint32_t flags, void* d_sha256, void* d_md5,
                               uint64_t* d_trimmed_len, void* cuda_stream);

/* Split one host buffer into ceil(len/part_len) fixed-size parts and hash each (the last may be short).
 * etag_md5_out (may be NULL) = MD5 over the concatenated raw part MD5s, computed on the device
 * (requires B200H_MD5).  Returns the number of parts through *nparts_out.
 * Replaces: the per-8MiB-block loop of _gather_blocks (blob_utils.py:622-645, with B200H_TRIM_ZEROS) and
 * the per-part MD5 + md5(concat) ETag of perform_multipart_upload (blob_utils.py:194-219,
 * bytes_io_segment_payload.py:58,102). */
int b200h_hash_fixed_parts(b200h_ctx* ctx, const uint8_t* base, uint64_t len, uint64_t part_len, uint32_t flags,
                           uint8_t* sha256_out, uint8_t* md5_out, uint64_t* trimmed_len_out,
                           uint8_t etag_md5_out[16], uint64_t* nparts_out);

/* Same split, but the buffer [d_base, d_base + len) and every output are DEVICE memory on ctx's device, and the work is
 * only enqueued on `cuda_stream` (a cudaStream_t; NULL = the context's compute stream).  The parts are cut by the same
 * code as b200h_hash_fixed_parts and b200h_hash_files(part_len > 0).  Outputs (each may be NULL): d_sha256[nparts*32],
 * d_md5[nparts*16] (both 16-byte aligned), d_trimmed_len[nparts] (== the part length unless B200H_TRIM_ZEROS),
 * d_etag_md5[16] (16-byte aligned; MD5 over the concatenated raw part MD5s, md5("") for len == 0; requires B200H_MD5,
 * and d_md5 when len > 0).  *nparts_out = ceil(len / part_len), returned on the host.  No B200H_HEX_OUT here.
 * The part lengths are known on the host, so outliers are routed there (as b200h_hash_batch_device_hl does) and the
 * call ONLY ENQUEUES -- except with B200H_TRIM_ZEROS and outlier routing on: the lengths that matter are then the
 * trimmed ones, which exist on the device only, and the planner's count is read back (one synchronisation of
 * `cuda_stream`, counted by b200h_plan_sync_count).  B200H_TRIM_ZEROS | B200H_NO_OUTLIERS only enqueues.
 * The part table (16 bytes per part) travels to the device with the work.
 * This is the one-segment case of b200h_hash_segment_parts_device (segment {d_base, len}; every part is hashed where
 * it is), plus the ETag.  A d_base range whose first or last byte is not device memory on ctx's device is
 * B200H_E_INVALID, rejected before anything is enqueued.
 * Replaces: the per-8MiB-block loop of _gather_blocks (blob_utils.py:622-645) for a buffer that already lives in HBM,
 * which the reference would first copy to host memory. */
int b200h_hash_fixed_parts_device(b200h_ctx* ctx, const void* d_base, uint64_t len, uint64_t part_len, uint32_t flags,
                                  void* d_sha256, void* d_md5, uint64_t* d_trimmed_len, void* d_etag_md5,
                                  uint64_t* nparts_out, void* cuda_stream);

/* One piece of a segmented device file: len bytes at d_ptr (device memory on ctx's device; may be NULL if len == 0). */
typedef struct b200h_segment {
    const void* d_ptr;
    uint64_t len;
} b200h_segment;

/* The same split over nfiles virtual files that live in device memory as many buffers: file f is the concatenation of
 * segs[file_first_seg[f] .. file_first_seg[f+1]) (segs and file_first_seg[nfiles + 1] are host arrays;
 * file_first_seg[0] == 0, it never decreases and file_first_seg[nfiles] == nsegs).  Every file is cut into
 * ceil(size / part_len) parts exactly as b200h_hash_fixed_parts_device cuts one buffer; rows are flattened file-major
 * (like b200h_hash_files), so the parts of all files form ONE batch.  Empty segments and zero-byte files (no rows) are
 * allowed.  Flags: B200H_SHA256 / B200H_MD5 / B200H_TRIM_ZEROS / B200H_NO_OUTLIERS; no B200H_HEX_OUT, no ETag.
 * Outputs as in b200h_hash_fixed_parts_device (d_sha256 / d_md5 16-byte aligned, each may be NULL);
 * *nparts_out = the total row count, returned on the host.
 * A part that lies inside one segment is hashed where it is (its start need not be aligned).  A part that spans
 * segments is first copied into one of the context's HBM wave slots (device_bytes / 2 each, the buffers the *_host
 * entry points stage through) by one gather kernel launch.  When those parts do not fit one slot, the call is split
 * into waves over contiguous ranges of rows, each costing about one more part's hash time; b200h_segment_parts_preview
 * shows the split.  Every non-empty segment's first and last byte must be device memory on ctx's device
 * (cudaPointerGetAttributes); a NULL or foreign pointer is B200H_E_INVALID, and every argument is checked before any
 * work is enqueued.
 * The call ONLY ENQUEUES on `cuda_stream` -- except with B200H_TRIM_ZEROS and outlier routing on, where the planner's
 * count is read back once per wave (synchronising `cuda_stream`, counted by b200h_plan_sync_count);
 * B200H_TRIM_ZEROS | B200H_NO_OUTLIERS only enqueues.  Growing the wave slots or the part table allocates, which
 * synchronises the device.
 * Replaces: the per-8MiB-block loop of _gather_blocks (blob_utils.py:622-645) for a file that lives in HBM as many
 * buffers (a safetensors image of a state dict), which the reference would serialise in host memory first -- and, with
 * nfiles > 1, the one-file-at-a-time spec building of the volumefs2 uploader (py/modal/volume.py:1380-1390). */
int b200h_hash_segment_parts_device(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs, const uint64_t* file_first_seg,
                                    uint64_t nfiles, uint64_t part_len, uint32_t flags, void* d_sha256, void* d_md5,
                                    uint64_t* d_trimmed_len, uint64_t* nparts_out, void* cuda_stream);

/* CRC-32 of n device ranges: d_crc_out[i] (a DEVICE array of n uint32, 4-byte aligned) = zlib.crc32 of
 * ranges[i].len bytes at ranges[i].d_ptr (IEEE polynomial, reflected, initial value and final XOR 0xFFFFFFFF): the
 * checksum a zip archive stores for every record, such as those of a torch.save file.  Any start alignment, any length
 * (0 gives 0).  `ranges` is a host array; every non-empty range's first and last byte, and the first and last byte of
 * d_crc_out, must be device memory on ctx's device (cudaPointerGetAttributes): a NULL or foreign pointer is
 * B200H_E_INVALID, and every argument is checked before any work is enqueued.
 * The work is spread by bytes, not by ranges: every range is cut into 16 KiB chunks and the grid's warps take equal runs
 * of them, so one huge range occupies the whole GPU and many small ranges share warps.  One kernel launch
 * (crc32_chunks_kernel) per call whatever n is, none when every range is empty.  The host writes each range's length
 * term to d_crc_out first (CRC arithmetic on the lengths; the library never hashes bytes on the CPU) and the kernel
 * XORs the bytes' contribution into it.  The call ONLY ENQUEUES on `cuda_stream` (NULL = the context's compute stream):
 * its small range table lives in a stream-ordered allocation (cudaMallocAsync / cudaFreeAsync), so it never
 * synchronises.
 * Replaces: the CRC-32 torch.save computes on the host over every storage after copying it there
 * (torch/serialization.py _save -> PyTorchStreamWriter::writeRecord), for a checkpoint that lives in HBM. */
int b200h_crc32_device(b200h_ctx* ctx, const b200h_segment* ranges, uint64_t n, uint32_t* d_crc_out, void* cuda_stream);

/* len bytes at offset `offset` of file `file` of a segmented batch. */
typedef struct b200h_file_range {
    uint64_t file, offset, len;
} b200h_file_range;

/* Copy byte ranges of files that live in device memory as many buffers into page-locked HOST memory: range i lands at
 * h_dst + dst_offsets[i].  The files are described exactly as for b200h_hash_segment_parts_device (segs,
 * file_first_seg: host arrays, file-major).  A range may lie inside one segment or cross any number of them, empty
 * ones included; len == 0 copies nothing.  `ranges` and `dst_offsets` are host arrays.
 * h_dst is what b200h_host_alloc returns (16-byte aligned).  The caller owns its layout: every dst_offsets[i] must be a
 * multiple of 16 and the destinations must lie inside h_dst_bytes without overlapping; no packing rule is imposed.
 * Every argument is checked before any work is enqueued, B200H_E_INVALID otherwise: the rules of the segment-parts
 * entry for segs / file_first_seg (every non-empty segment's first and last byte device memory on ctx's device),
 * file < nfiles, offset + len within the file, h_dst page-locked host memory the context's device can reach
 * (cudaPointerGetAttributes), destination offsets aligned, in bounds and disjoint.
 * ONE kernel launch (stage_ranges_kernel) per call whatever the number of ranges and segments, none when every range
 * is empty.  The kernel stores straight into h_dst, and every store is a full aligned 16-byte word whatever the phase
 * of the source bytes, except the bytes behind a range's last whole word; bytes of h_dst outside the destinations are
 * not written.  The call ONLY ENQUEUES on `cuda_stream` (NULL = the context's compute stream): its tables live in a
 * stream-ordered allocation as b200h_crc32_device's do, so it never synchronises; h_dst holds the bytes once the work
 * enqueued on the stream has completed (cudaStreamSynchronize, or an event recorded after the call).
 * Replaces: the per-chunk reads of _put_missing_blocks (py/modal/volume.py:1500-1574) for a file that lives in HBM,
 * which the reference would have in host memory already. */
int b200h_copy_ranges_to_host(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs, const uint64_t* file_first_seg,
                              uint64_t nfiles, const b200h_file_range* ranges, uint64_t nranges, void* h_dst,
                              uint64_t h_dst_bytes, const uint64_t* dst_offsets, void* cuda_stream);

/* The inverse of b200h_copy_ranges_to_host: the bytes at h_src + src_offsets[i] are written to range i of files that
 * live in device memory as many buffers, described as there (segs, file_first_seg, b200h_file_range; host arrays).
 * h_src is what b200h_host_alloc returns (16-byte aligned); every src_offsets[i] must be a multiple of 16 and every
 * source must lie inside h_src_bytes (sources may overlap).
 * Every argument is checked before any work is enqueued, B200H_E_INVALID otherwise: the rules of the to-host entry for
 * segs / file_first_seg / ranges, h_src page-locked host memory the context's device can reach
 * (cudaPointerGetAttributes), source offsets aligned and in bounds, and no device byte written by two ranges (checked on
 * the resolved device addresses: two files, or two segments of one file, may share a tensor).
 * ONE kernel launch (load_ranges_kernel) per call whatever the number of ranges and segments, none when every range is
 * empty.  The kernel reads h_src straight over PCIe, every source byte once, in aligned 16-byte loads that stay inside
 * the 16-byte hull of the sources; device stores are full aligned 16-byte words except at the edges of a segment's part
 * of a range and at one word per 64 KiB of source.  Device bytes of the segments outside every range are not written.
 * The call ONLY ENQUEUES on `cuda_stream` (NULL = the context's compute stream), as the to-host entry does: h_src must
 * stay unchanged, and the device bytes are there, once the work enqueued on the stream has completed.
 * Replaces: _read_file_into_fileobj (py/modal/volume.py:923-1000) writing a downloaded file into host memory, from
 * which a checkpoint would then be copied to the device tensor by tensor. */
int b200h_copy_ranges_from_host(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs, const uint64_t* file_first_seg,
                                uint64_t nfiles, const b200h_file_range* ranges, uint64_t nranges, const void* h_src,
                                uint64_t h_src_bytes, const uint64_t* src_offsets, void* cuda_stream);

/* A box of a host buffer: `rows` rows of `width` bytes, row r at h_src + src_offset + r * src_pitch (any byte phase),
 * written packed to bytes [offset, offset + rows * width) of file `file` of a segmented batch. */
typedef struct b200h_box {
    uint64_t file, offset;
    uint64_t width, rows;
    uint64_t src_offset, src_pitch;
} b200h_box;

/* Like b200h_copy_ranges_from_host, for strided sources: box i of h_src is written packed to its destination run of
 * files that live in device memory as many buffers, described as there (segs, file_first_seg; host arrays).  A box's
 * run may cross any number of segments; rows * width == 0 copies nothing.  `boxes` is a host array.  Neither h_src
 * nor the sources need any alignment (h_src may be a view into what b200h_host_alloc returns), and sources may overlap.
 * Every argument is checked before any work is enqueued, B200H_E_INVALID otherwise: the rules of the segment-parts entry
 * for segs / file_first_seg, file < nfiles, the destination inside its file and the last source byte inside
 * h_src_bytes (both without overflow), src_pitch >= width when rows > 1, h_src page-locked host memory the context's
 * device can reach (cudaPointerGetAttributes), and no device byte written by two boxes (checked on the resolved device
 * addresses).
 * ONE kernel launch (load_boxes_kernel) per call, none when every box is empty; the tables it uploads grow with the
 * boxes and their 64 KiB tiles of source words, never with the rows, which the kernel expands.  It reads h_src straight
 * over PCIe, every source byte that lands once, in aligned 16-byte loads inside the 16-byte hull of its row; bytes
 * between rows are read only inside those words.  Device stores are full aligned 16-byte words except at the ends of a
 * box's run, at segment edges and at one word per 64 KiB tile.  Device bytes outside every box are not written.
 * The call ONLY ENQUEUES on `cuda_stream` (NULL = the context's compute stream), as the range entries do: h_src must
 * stay unchanged, and the device bytes are there, once the work enqueued on the stream has completed.
 * Replaces: _read_file_into_fileobj (py/modal/volume.py:923-1000) followed by the host-side get_slice of the
 * safetensors library and a per-tensor .to("cuda"), to give each tensor-parallel rank its slice of a checkpoint. */
int b200h_copy_boxes_from_host(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs, const uint64_t* file_first_seg,
                               uint64_t nfiles, const b200h_box* boxes, uint64_t nboxes, const void* h_src,
                               uint64_t h_src_bytes, void* cuda_stream);

/* Element types of b200h_cast_box (IEEE binary32, IEEE binary16, bfloat16; all little-endian). */
#define B200H_DT_F32 1u
#define B200H_DT_F16 2u
#define B200H_DT_BF16 3u

/* A box whose elements change type on the way: `box` as in b200h_box, except that `width` and `src_pitch` count SOURCE
 * bytes, and its rows * width / (source element size) elements are written packed, as `dst_type`, to bytes
 * [offset, offset + rows * width / (source element size) * (destination element size)) of file `file`. */
typedef struct b200h_cast_box {
    b200h_box box;
    uint64_t src_type, dst_type; /* B200H_DT_* */
} b200h_cast_box;

/* b200h_copy_boxes_from_host with a conversion: every element of box i of h_src, of type src_type, is converted to
 * dst_type and written packed to the box's destination run.  Narrowing rounds to nearest even, exactly as the CUDA
 * intrinsics __float2bfloat16 (F32 -> BF16) and __float2half (F32 -> F16) do, NaN bit patterns included; F16 <-> BF16
 * widens to F32 exactly and rounds once; widening is exact.
 * Every argument is checked before any work is enqueued, B200H_E_INVALID otherwise: every rule of
 * b200h_copy_boxes_from_host (the destination measured in destination bytes), and further: src_type and dst_type are
 * two different B200H_DT_* codes; width and src_pitch are multiples of the source element size; every row's source
 * address is a multiple of the source element size; and each box's destination lies in ONE segment, at a device
 * address that is a multiple of the destination element size.  (Every file written by safetensors.torch.save meets the
 * alignment rules: the header is padded to a multiple of 8 and tensors are laid out by decreasing element size, so
 * every tensor starts at a multiple of its element size.)
 * ONE kernel launch (load_boxes_kernel, the kernel of b200h_copy_boxes_from_host) per call, none when every box is
 * empty, with tables that grow as those of b200h_copy_boxes_from_host.  Every source word that holds a selected byte
 * crosses PCIe once, in an aligned 16-byte load inside its row's hull; device stores are full aligned 16-byte words
 * except at the ends of a box's run and at one word per 64 KiB tile of source words.  Device bytes outside every box
 * are not written.
 * The call ONLY ENQUEUES on `cuda_stream` (NULL = the context's compute stream), as the range entries do.
 * Replaces: _read_file_into_fileobj (py/modal/volume.py:923-1000) followed by safetensors.torch.load and a per-tensor
 * .to(dtype), which holds the stored image and its converted copy at once, to load a checkpoint in a compute dtype. */
int b200h_copy_cast_boxes_from_host(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs,
                                    const uint64_t* file_first_seg, uint64_t nfiles, const b200h_cast_box* boxes,
                                    uint64_t nboxes, const void* h_src, uint64_t h_src_bytes, void* cuda_stream);

/* FP8 element types (OCP 8-bit floats: E4M3 with no infinities, as torch.float8_e4m3fn; E5M2, as torch.float8_e5m2).
 * Only b200h_copy_scaled_boxes_from_host takes them; the other entries refuse them as unknown types. */
#define B200H_DT_F8E4M3 4u
#define B200H_DT_F8E5M2 5u

/* A box of FP8 elements dequantized on the way: `cast` as in b200h_cast_box, with src_type B200H_DT_F8E4M3 or
 * B200H_DT_F8E5M2 (so width and src_pitch count elements as well as bytes) and dst_type B200H_DT_F32, F16 or BF16.
 * The box is cut from the R x C row-major tensor W (rows_total = R, cols = C): element c of its row r is W's element
 * first_elem + r * src_pitch + c, i.e. (that / C, that % C).  Its scales are scale_count elements of scale_type
 * (B200H_DT_F32, F16 or BF16) at d_scales, device memory of the context's device, ceil(R / block_rows) x
 * ceil(C / block_cols) of them in row-major order: element (i, j) of W uses scale (i / block_rows) *
 * ceil(C / block_cols) + j / block_cols.  A block size of R or more (C or more) is one block over the dimension. */
typedef struct b200h_scaled_box {
    b200h_cast_box cast;
    const void* d_scales;
    uint64_t scale_type, scale_count;
    uint64_t first_elem;
    uint64_t rows_total, cols;
    uint64_t block_rows, block_cols;
} b200h_scaled_box;

/* b200h_copy_cast_boxes_from_host for FP8 boxes with block scales: every element of box i is decoded exactly, multiplied
 * in F32 by its scale (widened exactly), rounding to nearest even with subnormals kept, and the product rounded once
 * to dst_type (no second rounding for F32): bit for bit what torch computes on CUDA as
 * (W.float() * S.float().repeat_interleave(block_rows, 0)[:R].repeat_interleave(block_cols, 1)[:, :C]).to(dst).
 * A NaN element or product gives a NaN (0x7FFF for a 16-bit target, 0x7FFFFFFF for F32).
 * Every argument is checked before any work is enqueued, B200H_E_INVALID otherwise: every rule of
 * b200h_copy_cast_boxes_from_host, with src_type an FP8 code, and further: block_rows and block_cols >= 1;
 * ceil(R / block_rows) * ceil(C / block_cols) <= scale_count; every element a box touches lies below R * C (both computed
 * without overflow); scale_type a known code; d_scales aligned to its element size, and its scale_count elements device
 * memory of the context's device (cudaPointerGetAttributes).
 * ONE kernel launch (load_scaled_boxes_kernel) per call, none when every box is empty, with tables that grow as those of
 * b200h_copy_boxes_from_host (never with the rows).  Source words cross PCIe once, as for the cast entry; scales are
 * read from device memory.  The call ONLY ENQUEUES on `cuda_stream` (NULL = the context's compute stream).
 * Replaces: loading an FP8 checkpoint and its scales, then w.float() * expanded_scale per weight in torch (DeepSeek's
 * fp8_cast_bf16.py), which holds the FP8 image, the results and F32 temporaries in HBM together. */
int b200h_copy_scaled_boxes_from_host(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs,
                                      const uint64_t* file_first_seg, uint64_t nfiles, const b200h_scaled_box* boxes,
                                      uint64_t nboxes, const void* h_src, uint64_t h_src_bytes, void* cuda_stream);

/* A segment of a file whose elements may change type on the way out: len SOURCE bytes at d_ptr (device memory on ctx's
 * device).  src_type == dst_type: the bytes as they are (0 or a B200H_DT_* code).  Otherwise two different B200H_DT_*
 * codes, and the segment contributes its len / (source element size) elements converted to dst_type, packed:
 * len / ss * ds bytes of its file's image. */
typedef struct b200h_cast_segment {
    const void* d_ptr;
    uint64_t len;                /* source bytes */
    uint64_t src_type, dst_type; /* equal: the bytes as they are; else two different B200H_DT_* codes */
} b200h_cast_segment;

/* b200h_copy_ranges_to_host over files made of cast segments: range i (a b200h_file_range of the file's IMAGE, any start
 * byte, mid-element included) of the converted images lands at dst + dst_offsets[i].  Conversion is that of
 * b200h_copy_cast_boxes_from_host: exactly torch's CUDA .to(), NaN bit patterns included.
 * Every argument is checked before anything is enqueued, B200H_E_INVALID otherwise: the rules of
 * b200h_copy_ranges_to_host (file table, ranges within their files, dst_offsets multiples of 16, destinations in bounds
 * and disjoint, segments device memory on ctx's device), and for a converting segment: d_ptr and len multiples of the
 * source element size, and its image offset in its file a multiple of the destination element size (every file written
 * by safetensors.torch.save meets this).  dst is 16-byte aligned page-locked host memory the device can reach, or
 * memory of ctx's device (cudaPointerGetAttributes).
 * ONE kernel launch (stage_ranges_kernel) per call, none when every range is empty; its tables live in a
 * stream-ordered allocation, so the call ONLY ENQUEUES on `cuda_stream` (NULL = the context's compute stream).  Every
 * store is a full aligned 16-byte word except the bytes behind a range's last whole word; bytes of dst outside the
 * destinations are not written.
 * Replaces: safetensors.torch.save({k: v.to(dtype)}) followed by the reads of _put_missing_blocks
 * (py/modal/volume.py:1500-1574), which holds the converted copy of every tensor in memory at once. */
int b200h_copy_cast_ranges(b200h_ctx* ctx, const b200h_cast_segment* segs, uint64_t nsegs, const uint64_t* file_first_seg,
                           uint64_t nfiles, const b200h_file_range* ranges, uint64_t nranges, void* dst,
                           uint64_t dst_bytes, const uint64_t* dst_offsets, void* cuda_stream);

/* b200h_hash_segment_parts_device over files made of cast segments (the rules of b200h_copy_cast_ranges for them): the
 * parts are cut from the converted images, with the same rows, flags, outputs and synchronisation rules.  A part is
 * hashed in place only when it lies in one segment that converts nothing; every other part is gathered into a wave
 * slot by stage_ranges_kernel (one launch per wave), so the converted bytes never exist in HBM outside the wave
 * slots.  b200h_cast_segment_parts_preview shows the split. */
int b200h_hash_cast_segment_parts_device(b200h_ctx* ctx, const b200h_cast_segment* segs, uint64_t nsegs,
                                         const uint64_t* file_first_seg, uint64_t nfiles, uint64_t part_len,
                                         uint32_t flags, void* d_sha256, void* d_md5, uint64_t* d_trimmed_len,
                                         uint64_t* nparts_out, void* cuda_stream);

/* ---- FP8 export: block scales and quantizing copies ---------------------------------------------------------------
 *
 * A 2-D weight W (R x C, row-major, F32 / F16 / BF16) is quantized to B200H_DT_F8E4M3 per block of block_rows x
 * block_cols elements (edge blocks are smaller; a block size of R or more, C or more, is the whole dimension), as the
 * widely copied per_block_cast_to_fp8 does it on CUDA in torch:
 *   a = NaN if the block holds a NaN, else max(amax |x|, 1e-4f)     (the clamped amax; torch's clamp propagates NaN)
 *   s = a * RN(1 / 448)                                               (the F32 scale stored next to the weight)
 *   m = RN(RN(1 / a) * 448)                                           (the multiplier: from a, never from s)
 *   q = E4M3(RN(float(x) * m))                                        (round to nearest even, subnormals kept)
 * A block holding an infinity has s = inf and m = 0: its finite elements give +-0, its infinities (inf * 0) NaN.
 * NaN bits: a NaN a is the block's largest |x| pattern widened to F32 (an F32 or BF16 payload kept, signalling ones
 * included; every F16 NaN widens to 0x7FFFFFFF), and its s is 0x7FFFFFFF.  Every NaN product gives q = 0x7F, whatever
 * the sign of the NaN.
 * The conversion saturates (satfinite): with a block's own a no product reaches 448 by more than rounding, but the
 * quantizing copies take the a they are given, and with an a below the block's max every product of magnitude 448 or
 * more gives 0x7E / 0xFE (+-448), +-inf * m (m > 0) included; torch's conversion gives NaN from 464 on instead. */

/* One weight of b200h_fp8_block_scales.  s and a hold ceil(R / block_rows) x ceil(C / block_cols) F32 values each,
 * row-major: d_scales receives s (the weight's scale tensor), d_amax receives a (kept for the quantizing copies). */
typedef struct b200h_fp8_scale_job {
    const void* d_src;
    uint64_t src_type; /* B200H_DT_F32, F16 or BF16 */
    uint64_t rows, cols;
    uint64_t block_rows, block_cols;
    float* d_scales;
    float* d_amax;
} b200h_fp8_scale_job;

/* s and a of every job (see above), computed on the device.  The amax is an integer max over the bits of |x| widened
 * to F32 (monotone for non-negative floats, and a NaN wins), reduced per warp and CTA, with one atomicMax per CTA per
 * block, so a per-channel or per-tensor block is spread over many CTAs.  Any R, C and block sizes; d_src need only be
 * aligned to its element size.
 * Every argument is checked before anything is enqueued, B200H_E_INVALID otherwise: a known src_type, R and C >= 1, block
 * sizes >= 1, d_src aligned to its element size and its R * C elements device memory of ctx's device, d_scales and d_amax
 * 4-byte aligned device memory of ctx's device, and no two jobs' d_amax arrays overlapping.
 * Enqueues on `cuda_stream` (NULL = the context's compute stream), whatever njobs is: one cudaMemsetAsync per
 * contiguous run of the jobs' d_amax arrays (one when they lie back to back), then two kernel launches (the amax
 * reduction, then the finalisation of a and s); it never synchronises.
 * Replaces: per_block_cast_to_fp8's padding, abs, amax and division in torch per weight, which allocates F32
 * temporaries of 4x the weight. */
int b200h_fp8_block_scales(b200h_ctx* ctx, const b200h_fp8_scale_job* jobs, uint64_t njobs, void* cuda_stream);

/* A segment of a file that may quantize: `cast` as in b200h_cast_segment, or, with cast.dst_type B200H_DT_F8E4M3, the
 * R x C weight at cast.d_ptr (cast.src_type F32, F16 or BF16, cast.len == R * C * its element size) quantized with the
 * clamped amax values a at d_amax (scale_count F32 values, ceil(R / block_rows) x ceil(C / block_cols) of them used,
 * row-major; what b200h_fp8_block_scales left there): the segment's image is the R * C one-byte elements q. */
typedef struct b200h_scaled_segment {
    b200h_cast_segment cast;
    const float* d_amax;
    uint64_t scale_count;
    uint64_t rows, cols;
    uint64_t block_rows, block_cols;
} b200h_scaled_segment;

/* b200h_copy_cast_ranges over files made of scaled segments: quantizing segments give q (see above), the others what
 * they give there.  Every rule of b200h_copy_cast_ranges applies to the cast segments, and for a quantizing segment:
 * src_type F32, F16 or BF16; len == R * C * its element size; block sizes >= 1; scale_count >= ceil(R / block_rows) *
 * ceil(C / block_cols); d_amax 4-byte aligned device memory of ctx's device.  Everything is checked before anything is
 * enqueued (B200H_E_INVALID).  ONE kernel launch (stage_scaled_ranges_kernel) per call, none when every range is empty;
 * only enqueues, as b200h_copy_cast_ranges.  The cast entries keep refusing the FP8 codes.
 * Replaces: safetensors.torch.save of the quantized dict followed by the reads of _put_missing_blocks
 * (py/modal/volume.py:1500-1574), which holds a quantized copy of every weight in memory at once. */
int b200h_copy_scaled_ranges(b200h_ctx* ctx, const b200h_scaled_segment* segs, uint64_t nsegs,
                             const uint64_t* file_first_seg, uint64_t nfiles, const b200h_file_range* ranges,
                             uint64_t nranges, void* dst, uint64_t dst_bytes, const uint64_t* dst_offsets,
                             void* cuda_stream);

/* b200h_hash_cast_segment_parts_device over files made of scaled segments (the rules of b200h_copy_scaled_ranges for
 * them): a part that touches a quantizing or converting segment is gathered into a wave slot by
 * stage_scaled_ranges_kernel (one launch per wave), so the quantized bytes never exist in HBM outside the wave slots. */
int b200h_hash_scaled_segment_parts_device(b200h_ctx* ctx, const b200h_scaled_segment* segs, uint64_t nsegs,
                                           const uint64_t* file_first_seg, uint64_t nfiles, uint64_t part_len,
                                           uint32_t flags, void* d_sha256, void* d_md5, uint64_t* d_trimmed_len,
                                           uint64_t* nparts_out, void* cuda_stream);

/* ---- FP8 load: weights quantized as they arrive from page-locked host memory ---------------------------------------
 *
 * The numerical contract is the export's (above): a, s, m and q bit for bit as b200h_fp8_block_scales and the
 * quantizing copies give them.  A block's s depends on every element of the block, so a weight that arrives in pieces
 * is quantized in two calls per piece of staging: b200h_fp8_amax_boxes_from_host reduces the amax of the elements that
 * have arrived into a, and once every element of a block row (a "band") has arrived, b200h_copy_quant_boxes_from_host
 * finalizes the band's a and s and writes its E4M3 codes. */

/* A box of F32 / F16 / BF16 elements quantized to E4M3: `cast` as in b200h_cast_box with cast.src_type B200H_DT_F32,
 * F16 or BF16 and cast.dst_type B200H_DT_F8E4M3 (one destination byte per element).  The box is cut from the R x C
 * row-major weight W (rows_total = R, cols = C): the element at source byte c of its row r is W's element first_elem +
 * (r * src_pitch + c) / (source element size).  d_amax holds W's a: scale_count F32 values, ceil(R / block_rows) x
 * ceil(C / block_cols) of them used, row-major (a block size of R or more, C or more, is the whole dimension). */
typedef struct b200h_quant_box {
    b200h_cast_box cast;
    float* d_amax;
    uint64_t scale_count;
    uint64_t first_elem;
    uint64_t rows_total, cols;
    uint64_t block_rows, block_cols;
} b200h_quant_box;

/* count consecutive blocks to finalize: d_amax[k] = NaN ? d_amax[k] : max(d_amax[k], 1e-4f) in place, and
 * d_scales[k] = d_amax[k] * RN(1 / 448), for k < count (fp8_finalize_kernel's rules). */
typedef struct b200h_fp8_band {
    float* d_amax;
    float* d_scales;
    uint64_t count;
} b200h_fp8_band;

/* The amax of every element of box i of h_src, max-reduced into its block's d_amax value: an integer max over the bits
 * of |x| widened to F32, exactly as b200h_fp8_block_scales reduces it.  The max is order-independent, so the elements
 * of a block may arrive over any number of calls (d_amax starts as zeros; the caller clears it).  Nothing but d_amax is
 * written; the destinations in segs are checked, not written, so that the amax and the copy take the same boxes.
 * Every argument is checked before anything is enqueued, B200H_E_INVALID otherwise: every rule of
 * b200h_copy_cast_boxes_from_host (destinations measured in one byte per element), and further: src_type F32, F16 or
 * BF16 and dst_type B200H_DT_F8E4M3; block sizes >= 1; scale_count >= ceil(R / block_rows) * ceil(C / block_cols);
 * every element a box touches below R * C (both without overflow); d_amax 4-byte aligned, and its scale_count values
 * device memory of the context's device.
 * ONE kernel launch (fp8_amax_boxes_kernel) per call, none when every box is empty; within the call source words cross
 * PCIe once, in the loads of b200h_copy_boxes_from_host.  The copy of the same boxes (b200h_copy_quant_boxes_from_host)
 * reads them again: quantizing on load takes every source byte across PCIe twice, once for the amax and once for the
 * codes.  Only enqueues on `cuda_stream` (NULL = the context's compute stream). */
int b200h_fp8_amax_boxes_from_host(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs,
                                   const uint64_t* file_first_seg, uint64_t nfiles, const b200h_quant_box* boxes,
                                   uint64_t nboxes, const void* h_src, uint64_t h_src_bytes, void* cuda_stream);

/* The bands' a and s finalized (b200h_fp8_band), then every element x of box i of h_src written to its destination as
 * q = E4M3(RN(float(x) * m)), m = RN(RN(1 / a) * 448) from its block's finalized a: what the FP8 export stores for the
 * weight, once every element of the boxes' blocks has gone through b200h_fp8_amax_boxes_from_host and been finalized
 * (by this call or an earlier one).
 * Every argument is checked before anything is enqueued, B200H_E_INVALID otherwise: every rule of
 * b200h_fp8_amax_boxes_from_host for segs and boxes, and for every band: count >= 1, d_amax and d_scales not NULL,
 * 4-byte aligned, their count values device memory of the context's device (both without overflow).
 * Enqueues on `cuda_stream` (NULL = the context's compute stream): one launch (fp8_finalize_kernel) when nbands > 0, then
 * one (load_quant_boxes_kernel) when a box is not empty; it never synchronises.
 * Replaces: loading a bfloat16 checkpoint into HBM and quantizing it per weight in torch (per_block_cast_to_fp8), which
 * holds the whole bfloat16 image and F32 temporaries of 4x a weight in HBM besides the FP8 results. */
int b200h_copy_quant_boxes_from_host(b200h_ctx* ctx, const b200h_segment* segs, uint64_t nsegs,
                                     const uint64_t* file_first_seg, uint64_t nfiles, const b200h_quant_box* boxes,
                                     uint64_t nboxes, const b200h_fp8_band* bands, uint64_t nbands, const void* h_src,
                                     uint64_t h_src_bytes, void* cuda_stream);

/* ---- files (native reader pool; no Python I/O, no mmap) ------------------------------------------ */

/* Sizes (and permission bits, may be NULL) of n regular files, stat'ed by the library's I/O threads.
 * Replaces the per-file seek-to-end / os.stat of _get_file_upload_spec (blob_utils.py:455-457,494). */
int b200h_stat_files(b200h_ctx* ctx, const char* const* paths, uint64_t n, uint64_t* sizes_out, uint32_t* modes_out);

/* Hash the contents of n files.  The library's reader threads pread() them straight into the pinned staging
 * ring; waves are hashed while the next ones are being read.  sizes[] = what b200h_stat_files returned (a file
 * that turns out shorter is B200H_E_IO).
 *   part_len == 0: one message per file -> n rows (get_file_upload_spec_from_path over a tree:
 *                  py/modal/volume.py:1209-1216, py/modal/mount.py:467-485, blob_utils.py:490-501)
 *   part_len  > 0: every file is split into ceil(size/part_len) parts, rows flattened file-major; with
 *                  B200H_TRIM_ZEROS these are the volumefs2 blocks (blob_utils.py:622-645). */
int b200h_hash_files(b200h_ctx* ctx, const char* const* paths, uint64_t n, const uint64_t* sizes, uint64_t part_len,
                     uint32_t flags, uint8_t* sha256_out, uint8_t* md5_out, uint64_t* trimmed_len_out);

/* ---- streaming single message (hashlib-object shaped) ------------------------------------------- */

/* Incremental digest of ONE message fed in arbitrary pieces with bounded memory; the chaining state
 * stays on the device between updates.  A single message is a serial Merkle-Damgard chain, so this is
 * latency-bound by construction (one GPU thread's speed per stream) -- use the batch entry points for throughput.
 * update() gathers into a pinned buffer and enqueues one absorb per 4 MiB (B200H_STREAM_BUF) without waiting
 * for it; every stream has its own CUDA stream and scratch, so N streams fed from N threads advance concurrently.
 * One stream object must not be used from two threads at once (like a hashlib object).
 * Replaces: hashlib objects in hash_utils._update over a BinaryIO (hash_utils.py:18-29) and
 * BytesIOSegmentPayload._md5_checksum (bytes_io_segment_payload.py:58,102,79-80). */
int b200h_stream_new(b200h_ctx* ctx, uint32_t flags, b200h_stream** out);
int b200h_stream_update(b200h_stream* s, const uint8_t* data, uint64_t len);
/* Non-destructive: may be called repeatedly and interleaved with further updates (like hashlib.digest()). */
int b200h_stream_digest(b200h_stream* s, uint8_t sha256_out[32], uint8_t md5_out[16]);
int b200h_stream_reset(b200h_stream* s);
void b200h_stream_free(b200h_stream* s);

/* ---- dedupe of the digest table (the step right after the path) ---------------------------------- */

/* For n fixed-width keys (key_bytes = 32: SHA-256 rows, 16: MD5 rows) compute first[i] = the smallest j with
 * key_j == key_i (so first[i] == i marks the first occurrence of a content) and the number of distinct keys.
 * Exact (full-key comparison), deterministic, computed on the device over a hash table in HBM.
 * Replaces: the `accounted_hashes` set of _Mount._load_mount (py/modal/mount.py:498,518-534), which dedupes one
 * file at a time on the event loop, and the per-file MountPutFile existence round trips the volumefs1 uploader
 * spends on duplicates inside one batch (py/modal/volume.py:1288-1296).
 * _host: keys / first_out are host arrays, blocks until done.  _device: every pointer is a device pointer
 * (d_keys 4-byte aligned, d_ndistinct may be NULL), work is only enqueued on cuda_stream (NULL = ctx's stream). */
int b200h_dedupe_host(b200h_ctx* ctx, const uint8_t* keys, uint64_t n, uint32_t key_bytes, uint32_t* first_out,
                      uint64_t* ndistinct_out);
int b200h_dedupe_device(b200h_ctx* ctx, const void* d_keys, uint64_t n, uint32_t key_bytes, uint32_t* d_first,
                        uint64_t* d_ndistinct, void* cuda_stream);

/* ---- utilities ---------------------------------------------------------------------------------- */

/* Counter-based synthetic bytes on the device (bench / test data): d_dst[0..nbytes) = bytes
 * [start, start+nbytes) of stream `seed`; d_dst 8-byte aligned, start a multiple of 8. */
int b200h_fill_synth_device(b200h_ctx* ctx, void* d_dst, uint64_t nbytes, uint64_t seed, uint64_t start,
                            void* cuda_stream);
/* How many messages of the most recent batch the planner handed to the outlier path (chain kernel: one CTA per
 * long message) instead of the lane kernel.  Diagnostic. */
int b200h_last_outlier_count(b200h_ctx* ctx, uint32_t* count_out);
/* The staging step of b200h_hash_batch_host on its own: gather n messages (base may be NULL with absolute addresses in
 * offsets[]) into dst the way a wave is laid out in HBM -- message i at the next multiple of 16, offsets returned
 * through packed_offsets_out -- with the library's packer team of `threads` threads working slot_bytes at a time (the
 * size of a pinned slot).  dst needs sum((len + 15) & ~15) bytes.  No context, no GPU: for the CPU tests of the packer
 * and for measuring a host's packing rate (tools/packbench.py).  Diagnostic. */
int b200h_pack_preview(const uint8_t* base, const uint64_t* offsets, const uint64_t* lengths, uint64_t n, uint8_t* dst,
                       uint64_t dst_bytes, uint64_t slot_bytes, int threads, uint64_t* packed_offsets_out);
/* What the planner decides for a batch with these message lengths on a device with sm_count SMs (default settings):
 * how many messages go to the chain kernel (true outliers, DESIGN.md 5.4) and how many form the long lane queue
 * (second, lane-packed launch, DESIGN.md 5.3).  Pure host arithmetic -- the same code that sizes the launches of
 * b200h_hash_batch_host / _device_hl without reading the device planner's answer back -- so it needs neither a
 * context nor a GPU.  flags: B200H_SHA256 / B200H_MD5 / B200H_NO_OUTLIERS.  Diagnostic. */
int b200h_plan_preview(const uint64_t* lengths, uint64_t n, uint32_t flags, uint32_t sm_count, uint32_t* n_chain_out,
                       uint32_t* n_long_out);
/* How b200h_hash_segment_parts_device splits files made of segments of these lengths, for wave slots of wave_bytes
 * bytes: the row count, the wave count, and for each of the first out_cap rows (seg_out / wave_out may be NULL) the
 * segment the part is hashed in place in (UINT64_MAX: the part spans segments and is gathered) and its wave.  The
 * same code builds the device entry's tables; no context, no GPU.  Argument rules as there (wave_bytes > 0). */
int b200h_segment_parts_preview(const uint64_t* seg_lens, uint64_t nsegs, const uint64_t* file_first_seg, uint64_t nfiles,
                                uint64_t part_len, uint64_t wave_bytes, uint64_t* nparts_out, uint64_t* nwaves_out,
                                uint64_t* seg_out, uint32_t* wave_out, uint64_t out_cap);
/* The same for b200h_hash_cast_segment_parts_device: segments as b200h_cast_segment (their pointers unused, every other
 * rule checked); a part is in place only in a segment that converts nothing. */
int b200h_cast_segment_parts_preview(const b200h_cast_segment* segs, uint64_t nsegs, const uint64_t* file_first_seg,
                                     uint64_t nfiles, uint64_t part_len, uint64_t wave_bytes, uint64_t* nparts_out,
                                     uint64_t* nwaves_out, uint64_t* seg_out, uint32_t* wave_out, uint64_t out_cap);
/* The same for b200h_hash_scaled_segment_parts_device: segments as b200h_scaled_segment (their pointers unused, every
 * other rule checked). */
int b200h_scaled_segment_parts_preview(const b200h_scaled_segment* segs, uint64_t nsegs, const uint64_t* file_first_seg,
                                       uint64_t nfiles, uint64_t part_len, uint64_t wave_bytes, uint64_t* nparts_out,
                                       uint64_t* nwaves_out, uint64_t* seg_out, uint32_t* wave_out, uint64_t out_cap);
/* Kernels launched by this context so far (all kinds). */
uint64_t b200h_launch_count(b200h_ctx* ctx);
/* Combining queue of b200h_hash_batch_host: GPU batches issued for, and caller requests served by, the small-request
 * path so far (requests / groups = how many concurrent callers shared a batch on average). */
int b200h_combine_stats(b200h_ctx* ctx, uint64_t* groups_out, uint64_t* requests_out);
/* Enqueues that had to synchronise their stream to read the planner's outlier count back (see
 * b200h_hash_batch_device); 0 for a caller that passes host lengths or B200H_NO_OUTLIERS. */
uint64_t b200h_plan_sync_count(b200h_ctx* ctx);
/* When enabled, every lane_hash launch is bracketed by CUDA events on its stream;
 * b200h_profile_read synchronises and returns the accumulated device time and launch count, then clears. */
int b200h_profile_enable(b200h_ctx* ctx, int on);
int b200h_profile_read(b200h_ctx* ctx, double* hash_kernel_ms, uint64_t* hash_kernel_launches);

#ifdef __cplusplus
}
#endif
#endif /* B200HASH_H */
