/*
 * nvrx_snap.h -- C ABI of libnvrx_snap.so, the H100 (sm_90a) checkpoint-snapshot engine.
 *
 * This is the drop-in boundary *below* the NVRx Python API.  The reference has no FFI for this path
 * (it is pure Python on top of PyTorch), so every entry point below names the reference code it
 * replaces; paths are relative to /root/reference/src/nvidia_resiliency_ext/checkpointing/.
 *
 * Conventions
 *   - plain C types only: pointers, sizes, ints.  Streams/events are passed as void* holding a
 *     cudaStream_t / cudaEvent_t (identical to the driver CUstream / CUevent, so handles coming
 *     from torch.cuda.Stream.cuda_stream can be passed directly).
 *   - every function returns an int status: 0 = NVRX_OK, 1..999 = a cudaError_t value,
 *     >= 1000 = one of the NVRX_E_* codes.  Nothing throws.  nvrx_strerror() decodes.
 *   - the caller owns every data buffer; a plan owns only its descriptor tables.
 *   - a plan is thread-compatible (one thread at a time); there is no global mutable state.
 *   - every call may pass its own stream.  A call that re-uploads a plan's descriptor tables (after update_ptrs, or a
 *     change between sharded and plain packing) orders that upload after the plan's earlier kernel launches on the
 *     device, whatever streams they ran on; the host does not wait.  A launch still queued on one stream therefore
 *     packs or scatters the tensors the plan pointed at when it was issued.  Destroying a plan waits for its last launch.
 *
 * Packed ("staging") layout produced by a plan -- the oracle (oracle/snapshot_oracle.py) restates it:
 *   segment i (tensor i in TensorAwareStateDict flattening order, basic_state_dict.py:34-41,112-120)
 *   starts at  off[i] = round_up(off[i-1] + packed_nbytes[i-1], align),  off[0] = 0
 *   packed_nbytes[i] = nbytes[i]            (bit copy)
 *                    = nbytes[i] / 2        (NVRX_SEG_NARROW_F32_BF16: fp32 -> bf16, RNE, NaN -> 0x7FFF)
 *   total = round_up(off[n-1] + packed_nbytes[n-1], align).  Gap bytes are never written.
 */
#ifndef NVRX_SNAP_H_
#define NVRX_SNAP_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NVRX_ABI_VERSION 9

enum {
    NVRX_OK = 0,
    NVRX_E_INVALID = 1000,  /* bad argument (null pointer, bad size, odd narrow length, ...) */
    NVRX_E_NOMEM = 1001,    /* host allocation failed */
    NVRX_E_STATE = 1002,    /* call not valid in the object's current state */
    NVRX_E_SYS = 1003,      /* an OS call (shm_open, mmap, ftruncate, pwrite ...) failed; see errno */
    NVRX_E_NODRIVER = 1004  /* a driver entry point could not be resolved */
};

/* per-segment flags */
#define NVRX_SEG_NARROW_F32_BF16 0x1u /* pack: fp32 -> bf16; scatter: bf16 -> fp32 (exact widen) */

/* kernel variants (nvrx_plan_set_variant); AUTO picks the measured-fastest for the plan's shape */
enum {
    NVRX_VARIANT_AUTO = 0,
    NVRX_VARIANT_LDG = 1, /* LDG.128 -> registers -> STG.128, warp-shuffle realign for ragged tiles */
    NVRX_VARIANT_TMA = 2  /* cp.async.bulk global->smem->global mbarrier ring + LDG ragged warps    */
};

typedef struct nvrx_plan nvrx_plan;
typedef struct nvrx_hostbuf nvrx_hostbuf;

/* ---- misc ---------------------------------------------------------------------------------- */
int nvrx_abi_version(void);
const char* nvrx_strerror(int status);
/* SM count / L2 bytes / device name of `device`; any out pointer may be NULL. */
int nvrx_device_info(int device, int* sm_count, uint64_t* l2_bytes, char* name, int name_len);

/* ---- plan: the flattened tensor table -> tile work-list ------------------------------------
 * Replaces the per-tensor loops of utils.py:85-99 (preload_tensors) and
 * local/basic_state_dict.py:162-187 (copy_tensors_to_cpu / restore_tensor_device): instead of N
 * independent `tensor.to(...)` calls the N (pointer, nbytes) pairs are compiled once into a tile
 * list that one kernel walks.  The plan is cached by the Python shim per state-dict structure
 * (the idea of async_ckpt/filesystem_async.py:81-116).
 *   n          number of segments (tensors); 0 is allowed
 *   ptrs[i]    device address of tensor i (contiguous bytes); may be unaligned; NULL iff nbytes 0
 *   nbytes[i]  source byte length of tensor i
 *   flags[i]   NVRX_SEG_* (NULL = all zero); NARROW requires nbytes % 4 == 0 and ptr % 4 == 0
 *   align      staging alignment of each segment start; power of two >= 16 (0 = default 512)
 *   tile_bytes work granule in source bytes; power of two in [4096, 65536] (0 = default)
 *   device     CUDA device ordinal that owns the tensors and the descriptor tables
 */
int nvrx_plan_create(int64_t n, const void* const* ptrs, const uint64_t* nbytes, const uint32_t* flags,
                     uint64_t align, uint32_t tile_bytes, int device, nvrx_plan** out);
/* Same, with caller-chosen staging offsets (16-byte aligned, ascending, non-overlapping) instead of the round_up rule:
 * lets the packed image coincide with the payload region of a checkpoint container (zero-copy persistence). */
int nvrx_plan_create_at(int64_t n, const void* const* ptrs, const uint64_t* nbytes, const uint32_t* flags,
                        const uint64_t* staging_offsets, uint64_t align, uint32_t tile_bytes, int device, nvrx_plan** out);
int nvrx_plan_destroy(nvrx_plan* plan);
/* total staging bytes / number of tiles (bulk + ragged) / algorithmic HBM bytes of one pack launch
 * (source bytes read + packed bytes written; SURVEY.md 8(d): 2*S, or 1.5*S_in with narrowing). */
int nvrx_plan_info(const nvrx_plan* plan, uint64_t* staging_bytes, uint64_t* n_tiles,
                   uint64_t* algorithmic_bytes);
/* off[i], packed_nbytes[i] for all n segments (either may be NULL). */
int nvrx_plan_layout(const nvrx_plan* plan, uint64_t* offsets, uint64_t* packed_nbytes);
/* Re-point the plan at a new set of tensors with identical sizes/flags (e.g. scatter destinations on
 * restore, or re-allocated parameters).  Alignment classes may change; the tile list is rebuilt. */
int nvrx_plan_update_ptrs(nvrx_plan* plan, const void* const* ptrs);
/* Re-point segments [seg_lo, seg_lo + n) at ptrs[0, n) while the snapshot ranges before them may still be in flight.  Only
 * the changed entries are uploaded, from their own region of the pinned mirror, by the next upload (the next launch on the
 * plan), which waits on the host only for an earlier upload of the same entries -- not for the disjoint ranges uploaded
 * earlier in the same snapshot.  A pointer that changes its 16-byte alignment class would change the tile list:
 * NVRX_E_STATE, nothing is changed, and the caller re-points the whole plan with nvrx_plan_update_ptrs instead. */
int nvrx_plan_update_ptrs_range(nvrx_plan* plan, int64_t seg_lo, int64_t n, const void* const* ptrs);
int nvrx_plan_set_variant(nvrx_plan* plan, int variant);
/* Introspection (tests, tooling): the tile work-list a launch would walk -- tiles [0, *n_bulk) are the TMA-eligible ones,
 * the rest ragged; up to `capacity` entries are written to seg/nbytes/off (any may be NULL).  `shard_bytes` != 0 shows
 * the list as nvrx_pack_sharded would build it (tiles never straddle a shard boundary).  No CUDA call is made: the
 * planner (create / layout / update_ptrs / tiles) works on a machine without a GPU. */
int nvrx_plan_tiles(const nvrx_plan* plan, uint64_t shard_bytes, uint32_t* n_bulk, uint32_t* n_tiles, uint32_t* seg,
                    uint32_t* nbytes, uint64_t* off, uint64_t capacity);
/* Upload descriptor tables if dirty (otherwise done lazily by the first pack/scatter). */
int nvrx_plan_commit(nvrx_plan* plan, void* stream);

/* ---- the hot path ---------------------------------------------------------------------------
 * nvrx_pack    tensors -> staging   ONE kernel launch on `stream`  (replaces utils.py:92-96,
 *              basic_state_dict.py:171-174 hot loop #1; group_utils.py:360-373 sender side)
 * nvrx_scatter staging -> tensors   ONE kernel launch on `stream`  (replaces
 *              basic_state_dict.py:184-187 hot loop #4; group_utils.py:442-448 receiver side)
 * `staging` must be 512-byte aligned device memory of at least staging_bytes. */
int nvrx_pack(nvrx_plan* plan, void* staging, void* stream);
int nvrx_scatter(nvrx_plan* plan, const void* staging, void* stream);

/* Fused pack + sharded replica exchange (the all-to-all layout: every member keeps 1/n of every other member's
 * snapshot; replaces strategies.py:88-140 / group_utils.py:342-375 for that layout): the packed byte range is cut into
 * `n_peers` contiguous shards of `shard_bytes` (multiple of 512); shard j = [j*shard_bytes, (j+1)*shard_bytes) is stored
 * at peer_bases[j] + slot_offset (peer-mapped device memory reached with NVLink P2P stores).  If `staging` is not NULL
 * the kernel additionally keeps the full packed copy there (own snapshot), reading the source tensors only once. */
int nvrx_pack_sharded(nvrx_plan* plan, void* staging, void* const* peer_bases, int n_peers, uint64_t shard_bytes,
                      uint64_t slot_offset, void* stream);

/* Walk order of nvrx_pack_sharded: start with the tiles of shard `first_shard` and wrap around (default 0).  Members of
 * a clique pass different values (rank r starts at the shard owned by r+1) so that at any moment they store into
 * different destination GPUs instead of all into the same one. */
int nvrx_plan_set_shard_rotation(nvrx_plan* plan, uint32_t first_shard);

/* Fused pack + all-gather (reference-identical full replication, strategies.py:88-140): every packed byte is
 * written to ALL `n_peers` buffers at peer_bases[j] + slot_offset + position.  The source tensors are read from
 * HBM once; remote copies travel as NVLink P2P stores issued by the same kernel (TMA bulk stores from the one
 * shared-memory slot, or STG.128 on the ragged path).  Callers order it between two clique barriers. */
int nvrx_pack_broadcast(nvrx_plan* plan, void* const* peer_bases, int n_peers, uint64_t slot_offset, void* stream);

/* ---- parity of erasure-coded local checkpoints ---------------------------------------------------
 * dst[0, bytes) = srcs[0] ^ srcs[1] ^ ... ^ srcs[n-1] over [0, bytes); with clear_srcs != 0 every source range is zero
 * afterwards.  One launch on `stream` (on the current device).  Device pointers 16-byte aligned, bytes % 16 == 0,
 * 1 <= n <= 64, dst must not overlap any source; otherwise NVRX_E_INVALID.  bytes may exceed 2^32; bytes == 0 launches
 * nothing.  Algorithmic HBM bytes: (n + 1) * bytes, (2n + 1) * bytes with clearing. */
int nvrx_xor_reduce(void* dst, void* const* srcs, int n, uint64_t bytes, int clear_srcs, void* stream);
/* dsts[d][0, bytes) = XOR over s of coef[d*n_src + s] * srcs[s][0, bytes) in GF(2^8) with the polynomial
 * x^8+x^4+x^3+x^2+1 (0x11d): the Reed-Solomon parity of a clique that keeps m >= 2 parity fragments, and its decode.
 * 1 <= n_dst <= 4, 1 <= n_src <= 64; device pointers 16-byte aligned, bytes % 16 == 0, no destination overlaps a source
 * or another destination; otherwise NVRX_E_INVALID and nothing is launched.  clear_srcs != 0: every source range is
 * zero afterwards.  Every source is read once per launch whatever the number of destinations; a coefficient 0 skips the
 * source for that row, 1 is a plain XOR.  One launch on `stream` (on the current device); bytes may exceed 2^32;
 * bytes == 0 launches nothing.  Algorithmic HBM bytes: (n_src + n_dst) * bytes, (2 n_src + n_dst) * bytes with
 * clearing. */
int nvrx_gf_combine(void* const* dsts, int n_dst, void* const* srcs, int n_src, const uint8_t* coef, uint64_t bytes,
                    int clear_srcs, void* stream);

/* ---- drain: device staging -> pinned host on a side stream ------------------------------------
 * Replaces the device-wide torch.cuda.synchronize() stall of async_ckpt/torch_ckpt.py:50,
 * local/ckpt_managers/base_manager.py:306-309 and async_ckpt/core.py:345.
 * Copies `bytes` in `chunk_bytes` pieces (0 = one piece) with cudaMemcpyAsync on `stream`; after piece k
 * lands, the 64-bit word at `progress` (pinned/registered host memory, may be NULL) is set to
 * base_value + bytes_done by a stream-ordered write, so a CPU-only process mapping the same shared
 * memory can follow the drain without touching CUDA.  If `done_event` != NULL it is recorded at the end. */
int nvrx_drain(void* host_dst, const void* staging, uint64_t bytes, uint64_t chunk_bytes,
               volatile uint64_t* progress, uint64_t base_value, void* stream, void* done_event);
/* Pipelined pack + drain, the whole snapshot in one call: the packed range is cut into `chunk_bytes` chunks; chunk c is
 * copied to `host_dst` on `drain_stream` as soon as the pack sub-launch (on `pack_stream`, tiles in staging order) that
 * covers it has finished, so the D2H starts ~100 us after the call instead of after the full pack.
 * `progress`/`base_value` as in nvrx_drain.  `packed_event` (optional) is recorded on pack_stream after the last
 * sub-launch -- the training stream is free from there; `done_event` (optional) on drain_stream after the last copy. */
int nvrx_snapshot(nvrx_plan* plan, void* staging, void* host_dst, uint64_t chunk_bytes, volatile uint64_t* progress,
                  uint64_t base_value, void* pack_stream, void* drain_stream, void* packed_event, void* done_event);
/* nvrx_snapshot of the staging range of segments [seg_lo, seg_hi) alone: from off[seg_lo] (0 when seg_lo == 0) to
 * off[seg_hi] (staging_bytes when seg_hi == n), cut into chunks and pack groups from the range's start by the same rule.
 * Calls for consecutive ranges on the same streams make one snapshot whose first range can be launched while the tensors
 * of the later ones are still being checked; nvrx_snapshot is the call for [0, n).  The progress word counts absolute
 * staging bytes (base_value + end of each chunk), so it rises across the ranges. */
int nvrx_snapshot_range(nvrx_plan* plan, int64_t seg_lo, int64_t seg_hi, void* staging, void* host_dst, uint64_t chunk_bytes,
                        volatile uint64_t* progress, uint64_t base_value, void* pack_stream, void* drain_stream,
                        void* packed_event, void* done_event);
/* Kernel launches of the last snapshot on this plan: the pack runs as a few sub-launches over geometrically growing
 * groups of copy chunks (1, 4, 16, ... chunks; NVRX_B200_PACK_GROWTH), 4 for a 16 GB snapshot with 256 MiB chunks.  A
 * range starting at segment 0 sets the count, a later range adds its own. */
int nvrx_plan_last_launches(const nvrx_plan* plan, uint32_t* launches);
/* ---- staging-free snapshot: live tensors -> pinned slot, no device staging buffer -------------------------------------
 * The reference's preload_tensors (utils.py:85-99) copies every tensor to the host on the training stream and then
 * synchronises the device.  Here the copies run on a side stream behind an event of the training stream and read the live
 * tensors; the caller must not write them until the done event (the "fence").
 *
 * nvrx_direct_schedule (no CUDA call) splits a layout of n segments (tensor-side nbytes, NVRX_SEG_* flags and slot
 * offsets, ascending) into the segments one small pack kernel writes -- every narrowed segment and every non-empty segment
 * below `small_bytes` -- and the ones the copy engines move, one cudaMemcpyAsync each, in offset order:
 *   in_kernel[i]       1 for a kernel segment, else 0 (empty segments are neither: no byte to move)
 *   progress_after[i]  for a copied segment, the slot offset the progress word reports (minus base_value) after its copy:
 *                      the end of segment i when the copies since the previous report (this one included) move at least
 *                      `chunk_bytes`; 0 = no report.  Kernel and empty segments always get 0.
 * NVRX_E_INVALID on NULL arrays, offsets that are not ascending and disjoint, or an odd narrowed length. */
int nvrx_direct_schedule(int64_t n, const uint64_t* nbytes, const uint32_t* flags, const uint64_t* offsets,
                         uint64_t small_bytes, uint64_t chunk_bytes, uint8_t* in_kernel, uint64_t* progress_after);
/* Enqueue one staging-free snapshot on `stream` (the engine's side stream), behind `start_event` (recorded on the training
 * stream; may be NULL):
 *   1. `kernel_plan` (may be NULL): a plan over the kernel segments alone, created with their slot offsets
 *      (nvrx_plan_create_at), packed by the LDG walker with a grid of a few CTAs straight into the mapped device address of
 *      `host_dst` (registered with cudaHostRegisterMapped).  One launch, none when the plan has no tiles.
 *   2. n_copies cudaMemcpyAsync D2H, src[i] -> host_dst + dst_offsets[i], nbytes[i] bytes, offsets ascending; after copy i
 *      a stream-ordered write sets *progress = base_value + progress_after[i] when that is not 0 (nvrx_direct_schedule).
 *   3. *progress = base_value + total_bytes, then `done_event` (optional) is recorded.
 * The kernel runs before every copy in stream order, so the progress word never reports a byte that has not landed.
 * `done_event` is the end of every read of the source tensors.  NVRX_E_INVALID on a range past total_bytes, offsets
 * that are not ascending, progress values that fall or lie past the end of their copy's group, or a kernel plan
 * larger than total_bytes. */
int nvrx_snapshot_direct(nvrx_plan* kernel_plan, int64_t n_copies, const void* const* src, const uint64_t* dst_offsets,
                         const uint64_t* nbytes, const uint64_t* progress_after, void* host_dst, uint64_t total_bytes,
                         volatile uint64_t* progress, uint64_t base_value, int device, void* start_event, void* stream,
                         void* done_event);
/* Mirror for restore: pinned host -> device staging (H2D), optional event. */
int nvrx_fill(void* staging, const void* host_src, uint64_t bytes, uint64_t chunk_bytes, void* stream,
              void* done_event);

/* Restore pipeline, file -> device staging without a snapshot-sized host buffer: `threads` readers pread() the n extents
 * (file_offs[i], nbytes[i]) of `fd` into a process-wide ring of `ring_slots` pinned chunks of `chunk_bytes` (allocated on
 * first use per device; 0 / <2 = defaults 64 MiB x 4) at the staging positions stg_offs[i] (ascending, disjoint), and the
 * calling thread copies every chunk to `staging` on `stream` as soon as its reads have landed, so the file read and the H2D
 * overlap.  Returns when the last chunk's copy has left the ring; follow with nvrx_scatter on the same stream.
 * Replaces the reference's torch.load + N x tensor.to("cuda") (local_manager.py:91-105, basic_state_dict.py:184-187). */
int nvrx_fill_from_fd(void* staging, uint64_t staging_bytes, int fd, int64_t n, const uint64_t* stg_offs,
                      const uint64_t* nbytes, const uint64_t* file_offs, uint64_t chunk_bytes, int ring_slots, int threads,
                      int device, void* stream);

/* ---- box scatter: resharded torch.distributed.checkpoint loads --------------------------------
 * Replaces the per-item tail of torch's FileSystemReader.read_data (torch/distributed/checkpoint/filesystem.py:897-915:
 * torch.load of the whole saved chunk, narrow_tensor_by_index, target.copy_() into a possibly non-contiguous view).  Each
 * of the n boxes is an N-d sub-box of a saved chunk that already sits in device staging, written into an N-d sub-box of
 * its destination; ONE kernel walks all of them.
 *   elem_bytes[i]   element size of box i: 1, 2, 4, 8 or 16
 *   ndim[i]         dims of box i, 0..NVRX_BOX_MAXDIM; sizes / strides of box i follow those of box i-1 in the flat arrays
 *   sizes[]         extents (>= 0)
 *   src_offs[i]     staging byte offset of element (0, ..., 0) of box i
 *   src_strides[]   staging strides in ELEMENTS (as torch reports them, >= 0)
 *   dst_ptrs[i]     device address of element (0, ..., 0) of the destination view of box i (NULL iff the box is empty)
 *   dst_strides[]   destination strides in elements (>= 0; 0 only on dims of size 1)
 *   staging_bytes   every source byte must lie below it
 *   tile_bytes      work granule (0 = default 32 KiB; power of two in [4096, 65536])
 * The planner drops size-1 dims, merges dims that are contiguous on both sides and, when the innermost dim is contiguous
 * on both sides, copies whole "runs" with the vector copy of nvrx_scatter; otherwise it moves one element per thread.  A
 * tile is (box, first row, rows, byte range): descriptors grow with boxes + tiles, not with rows.  No CUDA call is made
 * by create / create_cast / info / tiles / box / box_cast. */
#define NVRX_BOX_MAXDIM 8
typedef struct nvrx_boxplan nvrx_boxplan;
int nvrx_boxplan_create(int64_t n, const uint32_t* elem_bytes, const int32_t* ndim, const int64_t* sizes,
                        const uint64_t* src_offs, const int64_t* src_strides, const void* const* dst_ptrs,
                        const int64_t* dst_strides, uint64_t staging_bytes, uint32_t tile_bytes, int device,
                        nvrx_boxplan** out);
int nvrx_boxplan_destroy(nvrx_boxplan* plan);
/* nvrx_boxplan_create, converting between fp32, bf16 and fp16 on the way (loading a checkpoint into a model of another dtype).  cast[i] is
 * one NVRX_CAST_* code per box (cast == NULL or cast[i] == 0: bit copy, exactly as nvrx_boxplan_create plans it).  For a
 * converting box elem_bytes[i] is the SOURCE element size and must match the code, src_offs[i] (bytes) must be a multiple
 * of it and dst_ptrs[i] a multiple of the destination element size; src_strides count source elements, dst_strides
 * destination elements.  Otherwise NVRX_E_INVALID (as for an unknown code).  Narrowing rounds to nearest even, keeps
 * subnormals, sends overflow to +-inf and writes NaN as 0x7FFF; widening is exact (bf16 <-> fp16 goes through fp32).  The
 * converting boxes' tiles follow all copy tiles. */
#define NVRX_CAST_NONE 0u
#define NVRX_CAST_F32_BF16 1u
#define NVRX_CAST_F32_F16 2u
#define NVRX_CAST_BF16_F32 3u
#define NVRX_CAST_F16_F32 4u
#define NVRX_CAST_BF16_F16 5u
#define NVRX_CAST_F16_BF16 6u
int nvrx_boxplan_create_cast(int64_t n, const uint32_t* elem_bytes, const int32_t* ndim, const int64_t* sizes,
                             const uint64_t* src_offs, const int64_t* src_strides, const void* const* dst_ptrs,
                             const int64_t* dst_strides, const uint32_t* cast, uint64_t staging_bytes, uint32_t tile_bytes,
                             int device, nvrx_boxplan** out);
/* tiles of one nvrx_box_scatter / algorithmic HBM bytes of it: (es + ed) x numel per box, es / ed the source / destination
 * element sizes (2 x the bytes moved for a bit copy) */
int nvrx_boxplan_info(const nvrx_boxplan* plan, uint64_t* n_tiles, uint64_t* algorithmic_bytes);
/* Introspection (tests, tooling), like nvrx_plan_tiles: tile t covers rows [row[t], row[t] + nrows[t]) of box box[t]; with
 * one row it covers bytes [byte_off[t], byte_off[t] + nbytes[t]) of it, with several the whole rows.  Up to `capacity`
 * entries are written (any array may be NULL).  For a converting box byte_off / nbytes (and row_bytes below) count SOURCE
 * bytes, multiples of es; the destination bytes are byte_off / es * ed and nbytes / es * ed. */
int nvrx_boxplan_tiles(const nvrx_boxplan* plan, uint64_t* n_tiles, uint32_t* box, uint64_t* row, uint64_t* nrows,
                       uint64_t* byte_off, uint32_t* nbytes, uint64_t capacity);
/* The row geometry the planner made of box i: row r (mixed radix over sizes[0..n_outer), outermost first) is the
 * row_bytes bytes at staging offset src_off + sum idx_d * src_stride[d] and at device address dst + sum idx_d * dst_stride[d]
 * (byte strides; for a converting box row_bytes and src_stride in source bytes, dst_stride in destination bytes).  Arrays
 * hold NVRX_BOX_MAXDIM entries. */
int nvrx_boxplan_box(const nvrx_boxplan* plan, int64_t i, uint64_t* row_bytes, uint32_t* n_outer, uint64_t* sizes,
                     int64_t* src_stride, int64_t* dst_stride, uint64_t* src_off, uint64_t* dst);
/* The NVRX_CAST_* code of box i and its destination element size (the source size for a bit copy); either may be NULL. */
int nvrx_boxplan_box_cast(const nvrx_boxplan* plan, int64_t i, uint32_t* cast, uint32_t* dst_elem_bytes);
/* Upload the descriptor tables on `stream` (otherwise done by the first nvrx_box_scatter), e.g. to time the kernel alone. */
int nvrx_boxplan_commit(nvrx_boxplan* plan, void* stream);
/* staging -> destination views on `stream` (grids sized from the SM count): ONE kernel launch over the copy tiles, then
 * one over the converting tiles; a plan without converting boxes makes exactly one launch.  With converting boxes
 * `staging` must be 4-byte aligned; the vector body of a converting run needs the staging and destination addresses of
 * an element to sit at the same position in their vectors (see DESIGN.md), anything else runs element by element. */
int nvrx_box_scatter(nvrx_boxplan* plan, const void* staging, void* stream);

/* ---- device staging / stream helpers (so callers need no CUDA binding of their own) ---------- */
int nvrx_dev_alloc(int device, uint64_t bytes, void** out); /* cudaMalloc, zero-filled, IPC-capable */
int nvrx_dev_free(int device, void* ptr);
int nvrx_stream_create(int device, int high_priority, void** out);
int nvrx_stream_destroy(void* stream);
int nvrx_event_create(int device, int timing, void** out);
int nvrx_event_destroy(void* event);
int nvrx_event_record(void* event, void* stream);
int nvrx_stream_wait_event(void* stream, void* event);
int nvrx_event_query(void* event, int* done); /* done = 1 when complete */
int nvrx_event_sync(void* event);
int nvrx_event_elapsed_ms(void* start, void* stop, float* ms);
int nvrx_stream_sync(void* stream);
/* CUDA IPC for the fused exchange: 64-byte opaque handle. */
int nvrx_ipc_export(void* dev_ptr, uint8_t handle_out[64]);
int nvrx_ipc_import(int device, const uint8_t handle[64], void** out);
int nvrx_ipc_close(int device, void* imported);
/* Stream-ordered 64-bit flag write / wait on device-visible memory (peer or registered host). */
int nvrx_stream_write_u64(void* stream, void* addr, uint64_t value);
int nvrx_stream_wait_u64_geq(void* stream, void* addr, uint64_t value);

/* ---- host snapshot buffers --------------------------------------------------------------------
 * Replaces the N per-tensor pinned allocations made by Tensor.to("cpu", non_blocking=True)
 * (utils.py:94) and the full extra host copy torch.multiprocessing makes when CPU tensors cross the
 * mp.Queue to the persistent worker (async_ckpt/core.py:541): ONE persistent POSIX shared-memory
 * mapping, page-locked with cudaHostRegister, that the writer process maps by name.
 *   shm_name   "/name" for shm_open, or NULL for an anonymous MAP_SHARED mapping (fork-inheritable)
 *   bytes      payload capacity (a 4096-byte header page precedes the payload inside the mapping; the page begins with a
 *              ZIP local file header of an empty record, so that a slot packed in checkpoint-container geometry can be
 *              published as a torch.load-able file by a hard link, and holds the progress word at byte 192)
 *   prefault_threads  >0: touch pages with that many threads before pinning
 *   pin        0: map only (CPU-only process / no GPU), 1: cudaHostRegister for `device`
 */
int nvrx_hostbuf_create(const char* shm_name, uint64_t bytes, int prefault_threads, int pin, int device,
                        nvrx_hostbuf** out);
/* Map an existing named buffer in another process (never pins, never touches CUDA). */
int nvrx_hostbuf_open(const char* shm_name, nvrx_hostbuf** out);
int nvrx_hostbuf_destroy(nvrx_hostbuf* hb, int unlink_name);
void* nvrx_hostbuf_data(nvrx_hostbuf* hb);                  /* payload base (4096-aligned) */
uint64_t nvrx_hostbuf_capacity(const nvrx_hostbuf* hb);     /* payload bytes */
volatile uint64_t* nvrx_hostbuf_progress(nvrx_hostbuf* hb); /* header word the drain advances */
/* Block (sleeping, no CUDA) until *progress >= value or timeout_ms elapses (-1 = forever).
 * Returns NVRX_OK, or NVRX_E_STATE on timeout. */
int nvrx_hostbuf_wait(nvrx_hostbuf* hb, uint64_t value, int64_t timeout_ms);
/* Write [offset, offset+bytes) of the payload to `fd` at file offset `file_off` with `threads`
 * parallel pwrite() workers (persistence of the drained buffer; replaces the single-threaded
 * pickle+write of local/ckpt_managers/local_manager.py:117-122 for the payload part). */
int nvrx_hostbuf_write_fd(nvrx_hostbuf* hb, uint64_t offset, uint64_t bytes, int fd, uint64_t file_off,
                          int threads);
/* Vectored form: n extents (payload offset, length, file offset) written by one pool of `threads` pwrite() workers.
 * This is how a drained snapshot is persisted: torch.save lays out the container with its data records skipped
 * (torch.serialization.skip_data) and the extents fill them in in parallel. */
int nvrx_hostbuf_writev_fd(nvrx_hostbuf* hb, int64_t n, const uint64_t* offsets, const uint64_t* nbytes,
                           const uint64_t* file_offs, int fd, int threads);
/* Restore-side mirror: copy n host ranges (e.g. tensors of a loaded / mmapped checkpoint file) into the payload at
 * dst_offsets with `threads` memcpy workers, so ONE H2D + ONE scatter kernel can follow (replaces the N pageable
 * per-tensor H2D copies of local/basic_state_dict.py:184-187). */
int nvrx_hostbuf_gather(nvrx_hostbuf* hb, int64_t n, const void* const* srcs, const uint64_t* nbytes,
                        const uint64_t* dst_offsets, int threads);
/* Restore-side alternative to gather when the tensors come from a file: n file ranges -> payload offsets with `threads`
 * pread workers (no page-by-page faulting of an mmap of the file). */
int nvrx_hostbuf_readv_fd(nvrx_hostbuf* hb, int64_t n, const uint64_t* offsets, const uint64_t* nbytes, const uint64_t* file_offs,
                          int fd, int threads);
/* crc32 (zlib polynomial) of a payload range computed with `threads` workers and combined. */
int nvrx_hostbuf_crc32(nvrx_hostbuf* hb, uint64_t offset, uint64_t bytes, int threads, uint32_t* out);
/* The same for n extents in one call (checksums of all records of a checkpoint container): out[i] = crc32 of
 * [offsets[i], offsets[i] + nbytes[i]).  The sums use carry-less-multiply folding where the CPU has PCLMULQDQ. */
int nvrx_hostbuf_crc32v(nvrx_hostbuf* hb, int64_t n, const uint64_t* offsets, const uint64_t* nbytes, int threads,
                        uint32_t* out);

/* ---- CRC-32 of packed extents on the GPU ----------------------------------------------------------------------------
 * Replaces the CPU checksum pass of the reference's writer: `torch.save` (async_ckpt/torch_ckpt.py:36-41,
 * local/ckpt_managers/local_manager.py:117-122) runs miniz' crc32 over every tensor record on one core.  Here a kernel reads
 * the packed device buffer once more (HBM-bound integer work, one coalesced 16-byte load per lane) and emits one 32-bit
 * partial value per 64 KiB chunk; the values travel to the host with the snapshot and a CPU-only step chains them into the
 * zlib-compatible crc32 of every extent (== tensor record).  See csrc/crc_kernels.cuh for the arithmetic.
 *   offsets[i], nbytes[i]   extent i inside the buffer (those that start 16-byte aligned are summed on the GPU, whole
 *                           512-byte rows only; the remaining bytes are read from the host copy by nvrx_crc_finish)
 */
typedef struct nvrx_crc nvrx_crc;
int nvrx_crc_create(int64_t n, const uint64_t* offsets, const uint64_t* nbytes, int device, nvrx_crc** out); /* no CUDA call */
int nvrx_crc_destroy(nvrx_crc* c);
int nvrx_crc_info(const nvrx_crc* c, uint64_t* n_values); /* partial values one run produces */
/* Launch on `stream`: partial values of the buffer at dev_base, their D2H copy into host_values (pinned, n_values words)
 * and then -- optional -- a copy of `ready_value` into *host_ready (pinned), all stream-ordered: a CPU-only process that
 * sees *host_ready == ready_value may read the values.  The buffer must stay unchanged until that point of the stream. */
int nvrx_crc_run(nvrx_crc* c, const void* dev_base, uint32_t* host_values, uint64_t* host_ready, uint64_t ready_value,
                 void* stream);
/* CPU only (writer process): chain the partial values and the host copy of the left-over bytes (host_base = host copy of
 * the buffer, same offsets) into out_crcs[i] = crc32 of extent i.  NVRX_E_INVALID if n_values does not match the extents. */
int nvrx_crc_finish(int64_t n, const uint64_t* offsets, const uint64_t* nbytes, const uint32_t* values, uint64_t n_values,
                    const void* host_base, uint32_t* out_crcs);
/* The 4x256-word operator table "feed `which` zero bytes" (4, 16, 512; 0 = one full chunk) -- tooling and tests. */
int nvrx_crc_operator(uint32_t which, uint32_t* out_1024_words);

/* ---- CRC-32 of extents at any offset and of any length, entirely on the device ----------------------------------------
 * Verifies what a torch.distributed.checkpoint load put in HBM against the CRC-32 field of each storage record's ZIP
 * directory entry (torch's writer fills it in; torch.load and FileSystemReader.read_data never check it).  The reference has
 * no counterpart: its loads do not verify anything.  Unlike nvrx_crc_*, no host code reads payload bytes: the 16-byte
 * aligned body of every extent goes through the same chunk kernel (whole 512-byte rows, 64 KiB chunks) and a second small
 * kernel, one warp per extent, sums the head (< 16 bytes before the first 16-byte boundary) and the tail (< 512 bytes after
 * the last whole row) and folds everything into the extent's crc32.  See csrc/crc_kernels.cuh.
 *   offsets[i], nbytes[i]   extent i inside the buffer; any offset, any length (0 included); NVRX_E_INVALID on NULL arrays
 *                           or offset + length overflow.  No CUDA call. */
typedef struct nvrx_crcx nvrx_crcx;
int nvrx_crcx_create(int64_t n, const uint64_t* offsets, const uint64_t* nbytes, int device, nvrx_crcx** out);
int nvrx_crcx_destroy(nvrx_crcx* c);
/* body chunks one run sums / kernel launches one run makes (1 with only sub-row extents, 2 otherwise, 0 when n == 0);
 * either pointer may be NULL.  No CUDA call. */
int nvrx_crcx_info(const nvrx_crcx* c, uint64_t* n_chunks, uint32_t* launches);
/* Upload the descriptors on `stream` (otherwise done by the first run), e.g. to time the kernels alone. */
int nvrx_crcx_commit(nvrx_crcx* c, void* stream);
/* Enqueue on `stream`: when the stream reaches the end of this work, host_crcs[i] (pinned, n words; nothing past them is
 * written) == zlib.crc32 of extent i of the buffer at dev_base (device memory, 16-byte aligned).  The buffer must stay
 * unchanged until then.  The first run uploads the descriptors (stream-ordered). */
int nvrx_crcx_run(nvrx_crcx* c, const void* dev_base, uint32_t* host_crcs, void* stream);
/* zlib's crc32_combine: crc32(A | B) from crc32(A), crc32(B) and len(B) (any length below 2^64).  Returns the CRC, not a
 * status; host only, no CUDA call.  Chains the parts of a record that was split over several staging batches. */
uint32_t nvrx_crc32_combine(uint32_t crc_a, uint32_t crc_b, uint64_t len_b);

#ifdef __cplusplus
}
#endif
#endif /* NVRX_SNAP_H_ */
