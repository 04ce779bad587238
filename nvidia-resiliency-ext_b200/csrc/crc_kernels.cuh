// crc_kernels.cuh -- zlib-compatible CRC-32 of extents of a packed device buffer, computed on the GPU so that checkpoint
// records carry valid checksums without a CPU pass over the payload (the reference's writer spends most of its time in
// exactly that pass: torch.save -> miniz crc32, single-threaded; SURVEY.md 8a "Where time goes today").
//
// Arithmetic (reflected polynomial 0xEDB88320).  Let Z(n) be the linear map "feed n zero bytes" on a 32-bit CRC state.
// Feeding a little-endian word w from state s gives Z(4)(s ^ w), hence for a message of words w_0..w_{N-1}
//     state = Z(4N)(init)  ^  XOR_k Z(4(N-k))(w_k)                                            (1)
// The second term ("value" of the message) does not depend on init, so pieces can be computed independently and chained
// on the host:  state' = Z(len)(state) ^ value.
//
// A warp computes the value of one chunk of R rows x 512 bytes.  Lane l owns bytes [16l, 16l+16) of every row (one
// coalesced 16-byte load per lane and row) and keeps one running value per word column c = 4l+j:
//     t_c <- Z(512)(t_c) ^ w          so that after the last row   t_c = XOR_m Z(512(R-1-m))(w_{c+128m})
// By (1) the chunk value is XOR_c Z(4(128-c))(t_c), i.e. the word-CRC of the sequence t_0..t_127 from state 0:
// every lane folds its four columns with Z(4), then the 32 lane values (16 bytes apart) are chained with Z(16).
// Z(n) is applied with 4 lookups in a 4x256 table (one per state byte) held in shared memory.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define NVRX_HD __host__ __device__ __forceinline__
#else
#define NVRX_HD inline
#endif

namespace nvrx {

constexpr uint32_t kCrcRowBytes = 512;     // one warp-wide 16-byte load
constexpr uint32_t kCrcChunkRows = 128;    // rows per chunk -> 64 KiB per partial value
constexpr uint32_t kCrcOpWords = 4 * 256;  // words of one Z(n) operator table

struct CrcChunk {
    uint64_t off;   // byte offset of the first row inside the buffer (16-byte aligned)
    uint32_t rows;  // 1..kCrcChunkRows
    uint32_t ext;   // extent the chunk belongs to
};

// Z(n)(s) through the operator table `op` (op[j*256 + b] = Z(n)(b << 8j)).
NVRX_HD uint32_t crc_apply(const uint32_t* op, uint32_t s) {
    return op[s & 0xffu] ^ op[256 + ((s >> 8) & 0xffu)] ^ op[512 + ((s >> 16) & 0xffu)] ^ op[768 + (s >> 24)];
}

// The same map through a table replicated per lane: entry e of lane l lives at op32[e * 32 + l], i.e. always in shared-memory
// bank l -- 32 lanes looking up 32 unrelated entries never collide (a single copy serves random indices with ~3-way bank
// conflicts, which is what bounds the plain kernel).
NVRX_HD uint32_t crc_apply_lane(const uint32_t* op32, uint32_t lane, uint32_t s) {
    return op32[((s & 0xffu) << 5) + lane] ^ op32[((256u + ((s >> 8) & 0xffu)) << 5) + lane] ^
           op32[((512u + ((s >> 16) & 0xffu)) << 5) + lane] ^ op32[((768u + (s >> 24)) << 5) + lane];
}

NVRX_HD void crc_row_step_lane(const uint32_t* z512x32, uint32_t lane, uint32_t t[4], uint32_t w0, uint32_t w1, uint32_t w2,
                               uint32_t w3) {
    t[0] = crc_apply_lane(z512x32, lane, t[0]) ^ w0;
    t[1] = crc_apply_lane(z512x32, lane, t[1]) ^ w1;
    t[2] = crc_apply_lane(z512x32, lane, t[2]) ^ w2;
    t[3] = crc_apply_lane(z512x32, lane, t[3]) ^ w3;
}

// One row step of a lane: four column values advance by one row each.
NVRX_HD void crc_row_step(const uint32_t* z512, uint32_t t[4], uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {
    t[0] = crc_apply(z512, t[0]) ^ w0;
    t[1] = crc_apply(z512, t[1]) ^ w1;
    t[2] = crc_apply(z512, t[2]) ^ w2;
    t[3] = crc_apply(z512, t[3]) ^ w3;
}

// Fold a lane's four column values (4 bytes apart) into one value for its 16-byte slot.
NVRX_HD uint32_t crc_fold_lane(const uint32_t* z4, const uint32_t t[4]) {
    uint32_t u = crc_apply(z4, t[0]);
    u = crc_apply(z4, u ^ t[1]);
    u = crc_apply(z4, u ^ t[2]);
    return crc_apply(z4, u ^ t[3]);
}

// Chain step over lane values that sit 16 bytes apart: s <- Z(16)(s) ^ u.
NVRX_HD uint32_t crc_chain_lane(const uint32_t* z16, uint32_t s, uint32_t u) { return crc_apply(z16, s) ^ u; }

// ---- extents at any offset and of any length (nvrx_crcx_*) ----------------------------------------------------------
// An extent [off, off + len) of a 16-byte aligned buffer splits into
//     head  [off, a)                  a = min(round_up(off, 16), off + len): fewer than 16 bytes, summed byte by byte
//     body  [a, a + 512 * rows)       whole rows, in chunks of kCrcChunkRows rows: the values crc_chunks_private<> makes
//     tail  [a + 512 * rows, end)     fewer than 512 bytes, starting 16-byte aligned: 16 bytes per lane, like a short row
// and its crc32 is ~(Z(tail)(Z(body)(head state) ^ body value) ^ tail value), the head state fed from 0xFFFFFFFF.
// Z(n) for any n is applied through the tables Z(2^k), k = 0..63 (pow2 + k * kCrcOpWords): one lookup round per set bit.
constexpr uint32_t kCrcPow2Tables = 64;

struct CrcxExtent {
    uint64_t off;    // byte offset inside the buffer (any alignment)
    uint64_t len;    // bytes (0 allowed)
    uint64_t first;  // index of the extent's first body chunk value
};

NVRX_HD void crcx_split(uint64_t off, uint64_t len, uint32_t* head, uint64_t* rows, uint32_t* tail) {
    const uint64_t h = (16u - (off & 15u)) & 15u;
    *head = static_cast<uint32_t>(h < len ? h : len);
    const uint64_t rest = len - *head;
    *rows = rest / kCrcRowBytes;
    *tail = static_cast<uint32_t>(rest % kCrcRowBytes);
}

// body chunks of an extent with `rows` whole rows, and the rows of its last chunk
NVRX_HD uint64_t crcx_chunks(uint64_t rows) { return (rows + kCrcChunkRows - 1) / kCrcChunkRows; }
NVRX_HD uint32_t crcx_chunk_rows(uint64_t rows, uint64_t c) {
    const uint64_t left = rows - c * kCrcChunkRows;
    return static_cast<uint32_t>(left < kCrcChunkRows ? left : kCrcChunkRows);
}

// Z(n)(s) for any n (zlib's crc32_combine: crc(A | B) = Z(len B)(crc A) ^ crc B).
NVRX_HD uint32_t crc_zeros(const uint32_t* pow2, uint32_t s, uint64_t n) {
    for (uint32_t k = 0; n; ++k, n >>= 1)
        if (n & 1u) s = crc_apply(pow2 + k * kCrcOpWords, s);
    return s;
}

// Feed n bytes into state s one at a time (z1 = Z(1): its first 256 words are the classic byte table).
NVRX_HD uint32_t crc_feed_bytes(const uint32_t* z1, uint32_t s, const uint8_t* p, uint32_t n) {
    for (uint32_t k = 0; k < n; ++k) s = z1[(s ^ p[k]) & 0xffu] ^ (s >> 8);
    return s;
}

// Lane `lane` of 32 folds the contiguous block of chunk values [begin, end) it owns: value and byte count of the block.
NVRX_HD void crcx_lane_block(uint64_t n_chunks, uint32_t lane, uint64_t* begin, uint64_t* end) {
    const uint64_t q = (n_chunks + 31u) / 32u;
    const uint64_t b = lane * q;
    *begin = b < n_chunks ? b : n_chunks;
    *end = b + q < n_chunks ? b + q : n_chunks;
}
NVRX_HD uint32_t crcx_fold_block(const uint32_t* pow2, const uint32_t* vals, uint64_t rows, uint64_t begin, uint64_t end,
                                 uint64_t* bytes) {
    uint32_t u = 0;
    uint64_t nb = 0;
    for (uint64_t c = begin; c < end; ++c) {
        const uint64_t cb = static_cast<uint64_t>(crcx_chunk_rows(rows, c)) * kCrcRowBytes;
        u = crc_zeros(pow2, u, cb) ^ vals[c];
        nb += cb;
    }
    *bytes = nb;
    return u;
}

// Lane `lane`'s share of a tail of `tail` bytes at p: bytes [16 lane, 16 lane + 16) of it, value from state 0.
NVRX_HD uint32_t crcx_tail_lane(const uint32_t* z1, const uint8_t* p, uint32_t tail, uint32_t lane, uint32_t* n) {
    const uint32_t b = 16u * lane;
    *n = b < tail ? (tail - b < 16u ? tail - b : 16u) : 0u;
    return crc_feed_bytes(z1, 0u, p + b, *n);
}

// The extent's crc32 from its head state and the body and tail values.
NVRX_HD uint32_t crcx_finish(const uint32_t* pow2, uint32_t head_state, uint64_t rows, uint32_t body, uint32_t tail_bytes,
                             uint32_t tail) {
    const uint32_t s = crc_zeros(pow2, head_state, rows * kCrcRowBytes) ^ body;
    return ~(crc_zeros(pow2, s, tail_bytes) ^ tail);
}

#if defined(__CUDACC__)

// tables: [Z512 | Z4 | Z16], kCrcOpWords each, in global memory; copied to shared memory once per CTA.
template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
crc_chunks(const uint8_t* __restrict__ base, const CrcChunk* __restrict__ chunks, uint32_t n_chunks,
           const uint32_t* __restrict__ tables, uint32_t* __restrict__ out, unsigned long long* ready_word,
           unsigned long long ready_value) {
    // the word is copied to the host AFTER the values (stream order), telling a CPU-only reader they are complete
    if (blockIdx.x == 0 && threadIdx.x == 0) *ready_word = ready_value;
    __shared__ uint32_t s_op[3 * kCrcOpWords];
    for (uint32_t i = threadIdx.x; i < 3 * kCrcOpWords; i += WARPS * 32) s_op[i] = tables[i];
    __syncthreads();
    const uint32_t* z512 = s_op;
    const uint32_t* z4 = s_op + kCrcOpWords;
    const uint32_t* z16 = s_op + 2 * kCrcOpWords;
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t warp = blockIdx.x * WARPS + (threadIdx.x >> 5);
    const uint32_t n_warps = gridDim.x * WARPS;
    for (uint32_t c = warp; c < n_chunks; c += n_warps) {
        const CrcChunk ch = chunks[c];
        const uint4* p = reinterpret_cast<const uint4*>(base + ch.off) + lane;  // row stride = 32 uint4
        uint32_t t[4] = {0u, 0u, 0u, 0u};
        uint32_t r = 0;
        for (; r + 4 <= ch.rows; r += 4) {  // four loads in flight per lane before the dependent lookups
            const uint4 a = __ldg(p + (r + 0) * 32), b = __ldg(p + (r + 1) * 32);
            const uint4 d = __ldg(p + (r + 2) * 32), e = __ldg(p + (r + 3) * 32);
            crc_row_step(z512, t, a.x, a.y, a.z, a.w);
            crc_row_step(z512, t, b.x, b.y, b.z, b.w);
            crc_row_step(z512, t, d.x, d.y, d.z, d.w);
            crc_row_step(z512, t, e.x, e.y, e.z, e.w);
        }
        for (; r < ch.rows; ++r) {
            const uint4 a = __ldg(p + r * 32);
            crc_row_step(z512, t, a.x, a.y, a.z, a.w);
        }
        const uint32_t u = crc_fold_lane(z4, t);
        uint32_t s = 0;
#pragma unroll
        for (int l = 0; l < 32; ++l) s = crc_chain_lane(z16, s, __shfl_sync(0xffffffffu, u, l));
        if (lane == 0) out[c] = s;
    }
}

// Same algorithm with the hot operator Z(512) replicated per lane in 128 KiB of dynamic shared memory (one CTA per SM).
// With conflict-free lookups the kernel is bound by the LDG stream, i.e. by HBM, instead of by shared-memory replays.
constexpr uint32_t kCrcPrivateSmemBytes = kCrcOpWords * 32 * sizeof(uint32_t);

template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32, 1)
crc_chunks_private(const uint8_t* __restrict__ base, const CrcChunk* __restrict__ chunks, uint32_t n_chunks,
                   const uint32_t* __restrict__ tables, uint32_t* __restrict__ out, unsigned long long* ready_word,
                   unsigned long long ready_value) {
    extern __shared__ uint32_t s_z512x32[];  // [entry][lane]
    __shared__ uint32_t s_small[2 * kCrcOpWords];  // Z4 | Z16, single copies (used 4 + 32 times per chunk)
    if (blockIdx.x == 0 && threadIdx.x == 0) *ready_word = ready_value;
    for (uint32_t i = threadIdx.x; i < kCrcOpWords * 32; i += WARPS * 32) s_z512x32[i] = tables[i >> 5];
    for (uint32_t i = threadIdx.x; i < 2 * kCrcOpWords; i += WARPS * 32) s_small[i] = tables[kCrcOpWords + i];
    __syncthreads();
    const uint32_t* z4 = s_small;
    const uint32_t* z16 = s_small + kCrcOpWords;
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t warp = blockIdx.x * WARPS + (threadIdx.x >> 5);
    const uint32_t n_warps = gridDim.x * WARPS;
    for (uint32_t c = warp; c < n_chunks; c += n_warps) {
        const CrcChunk ch = chunks[c];
        const uint4* p = reinterpret_cast<const uint4*>(base + ch.off) + lane;
        uint32_t t[4] = {0u, 0u, 0u, 0u};
        uint32_t r = 0;
        for (; r + 4 <= ch.rows; r += 4) {
            const uint4 a = __ldg(p + (r + 0) * 32), b = __ldg(p + (r + 1) * 32);
            const uint4 d = __ldg(p + (r + 2) * 32), e = __ldg(p + (r + 3) * 32);
            crc_row_step_lane(s_z512x32, lane, t, a.x, a.y, a.z, a.w);
            crc_row_step_lane(s_z512x32, lane, t, b.x, b.y, b.z, b.w);
            crc_row_step_lane(s_z512x32, lane, t, d.x, d.y, d.z, d.w);
            crc_row_step_lane(s_z512x32, lane, t, e.x, e.y, e.z, e.w);
        }
        for (; r < ch.rows; ++r) {
            const uint4 a = __ldg(p + r * 32);
            crc_row_step_lane(s_z512x32, lane, t, a.x, a.y, a.z, a.w);
        }
        const uint32_t u = crc_fold_lane(z4, t);
        uint32_t s = 0;
#pragma unroll
        for (int l = 0; l < 32; ++l) s = crc_chain_lane(z16, s, __shfl_sync(0xffffffffu, u, l));
        if (lane == 0) out[c] = s;
    }
}

// Second pass of nvrx_crcx_run: one warp per extent folds the body chunk values crc_chunks_private<> left in `vals` (a
// contiguous block per lane, then the 32 block values chained), sums the head and the tail from `base` and writes the
// extent's crc32 to out[i].  pow2: the tables Z(2^k), read through L1 (a few hundred lookups per extent).
template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
crcx_fold(const uint8_t* __restrict__ base, const CrcxExtent* __restrict__ ext, uint32_t n,
          const uint32_t* __restrict__ vals, const uint32_t* __restrict__ pow2, uint32_t* __restrict__ out) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t warp = blockIdx.x * WARPS + (threadIdx.x >> 5);
    const uint32_t n_warps = gridDim.x * WARPS;
    for (uint32_t i = warp; i < n; i += n_warps) {
        const CrcxExtent e = ext[i];
        uint32_t head, tail;
        uint64_t rows;
        crcx_split(e.off, e.len, &head, &rows, &tail);
        uint64_t b, en, nb;
        crcx_lane_block(crcx_chunks(rows), lane, &b, &en);
        const uint32_t u = crcx_fold_block(pow2, vals + e.first, rows, b, en, &nb);
        uint32_t tn;
        const uint32_t w = crcx_tail_lane(pow2, base + e.off + head + rows * kCrcRowBytes, tail, lane, &tn);
        uint32_t body = 0, tv = 0;
        for (int l = 0; l < 32; ++l) {  // every lane chains all 32 (uniform control flow); lane 0 stores
            body = crc_zeros(pow2, body, __shfl_sync(0xffffffffu, nb, l)) ^ __shfl_sync(0xffffffffu, u, l);
            tv = crc_zeros(pow2, tv, __shfl_sync(0xffffffffu, tn, l)) ^ __shfl_sync(0xffffffffu, w, l);
        }
        if (lane == 0) {
            const uint32_t hs = crc_feed_bytes(pow2, 0xffffffffu, base + e.off, head);
            out[i] = crcx_finish(pow2, hs, rows, body, tail, tv);
        }
    }
}

#endif  // __CUDACC__

}  // namespace nvrx
