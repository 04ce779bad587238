// TEST INFRASTRUCTURE ONLY -- runs the arithmetic of nvrx_crcx_run (csrc/crc_kernels.cuh) on the host.
//
// The device functions are __host__ __device__; compiled here for the CPU, they are driven by loops that stand in for the
// 32 lanes of a warp: the body chunks row by row as crc_chunks_private<> walks them, then the fold crcx_fold<> makes of
// one extent (a contiguous block of chunk values per lane, the tail 16 bytes per lane, the head byte by byte).
// tests/test_dcp_verify_cpu.py compiles it with g++ and compares the results with zlib.  Nothing in the product links it.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "crc_kernels.cuh"

namespace {

std::vector<uint32_t> make_pow2() {  // Z(2^k), k = 0..63, by repeated squaring of Z(1)
    std::vector<uint32_t> t(static_cast<size_t>(nvrx::kCrcPow2Tables) * nvrx::kCrcOpWords);
    for (uint32_t j = 0; j < 4; ++j)
        for (uint32_t b = 0; b < 256; ++b) {
            const uint32_t s = b << (8 * j);
            uint32_t c = s & 0xffu;
            for (int k = 0; k < 8; ++k) c = (c & 1u) ? (c >> 1) ^ 0xEDB88320u : c >> 1;
            t[j * 256 + b] = c ^ (s >> 8);
        }
    for (uint32_t k = 1; k < nvrx::kCrcPow2Tables; ++k) {
        const uint32_t* prev = t.data() + (k - 1) * nvrx::kCrcOpWords;
        for (uint32_t i = 0; i < nvrx::kCrcOpWords; ++i) t[k * nvrx::kCrcOpWords + i] = nvrx::crc_apply(prev, prev[i]);
    }
    return t;
}

const std::vector<uint32_t>& pow2() {
    static const std::vector<uint32_t> t = make_pow2();
    return t;
}

}  // namespace

extern "C" void crcx_lanes_pow2(uint32_t* out) { memcpy(out, pow2().data(), pow2().size() * sizeof(uint32_t)); }

// crc32 of [off, off + len) of `base` (offsets count from a 16-byte aligned origin), the way the two kernels compute it.
extern "C" uint32_t crcx_lanes_extent(const uint8_t* base, uint64_t off, uint64_t len) {
    const uint32_t* p2 = pow2().data();
    const uint32_t *z4 = p2 + 2 * nvrx::kCrcOpWords, *z16 = p2 + 4 * nvrx::kCrcOpWords, *z512 = p2 + 9 * nvrx::kCrcOpWords;
    uint32_t head, tail;
    uint64_t rows;
    nvrx::crcx_split(off, len, &head, &rows, &tail);
    // body: one value per chunk of up to kCrcChunkRows rows, lane by lane as crc_chunks_private<> computes it
    const uint64_t n_chunks = nvrx::crcx_chunks(rows);
    std::vector<uint32_t> vals(n_chunks);
    for (uint64_t c = 0; c < n_chunks; ++c) {
        const uint8_t* chunk = base + off + head + c * nvrx::kCrcChunkRows * nvrx::kCrcRowBytes;
        uint32_t t[32][4];
        memset(t, 0, sizeof(t));
        for (uint32_t r = 0, nr = nvrx::crcx_chunk_rows(rows, c); r < nr; ++r)
            for (uint32_t lane = 0; lane < 32; ++lane) {
                uint32_t w[4];
                memcpy(w, chunk + static_cast<uint64_t>(r) * nvrx::kCrcRowBytes + lane * 16, 16);
                nvrx::crc_row_step(z512, t[lane], w[0], w[1], w[2], w[3]);
            }
        uint32_t s = 0;
        for (uint32_t lane = 0; lane < 32; ++lane) s = nvrx::crc_chain_lane(z16, s, nvrx::crc_fold_lane(z4, t[lane]));
        vals[c] = s;
    }
    // the fold of crcx_fold<>: per-lane blocks and tail slices, chained in lane order
    uint32_t u[32], w[32], tn[32];
    uint64_t nb[32];
    const uint8_t* tp = base + off + head + rows * nvrx::kCrcRowBytes;
    for (uint32_t lane = 0; lane < 32; ++lane) {
        uint64_t b, e;
        nvrx::crcx_lane_block(n_chunks, lane, &b, &e);
        u[lane] = nvrx::crcx_fold_block(p2, vals.data(), rows, b, e, &nb[lane]);
        w[lane] = nvrx::crcx_tail_lane(p2, tp, tail, lane, &tn[lane]);
    }
    uint32_t body = 0, tv = 0;
    for (uint32_t l = 0; l < 32; ++l) {
        body = nvrx::crc_zeros(p2, body, nb[l]) ^ u[l];
        tv = nvrx::crc_zeros(p2, tv, tn[l]) ^ w[l];
    }
    const uint32_t hs = nvrx::crc_feed_bytes(p2, 0xffffffffu, base + off, head);
    return nvrx::crcx_finish(p2, hs, rows, body, tail, tv);
}
