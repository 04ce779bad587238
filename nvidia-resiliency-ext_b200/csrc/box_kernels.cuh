// box_kernels.cuh -- sm_90a device code of the box scatter: N-d sub-boxes of saved checkpoint chunks (already in device
// staging) -> N-d sub-boxes of destination tensors, for resharded torch.distributed.checkpoint loads.
//
// A box is described once (BoxDesc); the work-list holds tiles of (box, first row, rows, byte range) and the walker
// derives every row's two addresses by mixed-radix index arithmetic, so descriptor bytes grow with boxes + tiles and not
// with rows (a column-resharded 16 GB load has millions of rows).
//
// Three tile shapes, one walker (LDG only; see DESIGN.md for why there is no TMA variant):
//   one row, a byte range of it   : the whole CTA runs copy_bytes (LDG.128 / SHFL-funnel realignment / head peel)
//   several rows of >= 32 bytes   : one warp per row, copy_bytes with the warp as the thread group
//   several rows of < 32 bytes    : one thread per row (element-wise path: transposed chunk or target view)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "snap_kernels.cuh"

namespace nvrx {

constexpr int kBoxMaxDim = 8;

struct __align__(16) BoxDesc {
    uint64_t src;        // staging byte offset of row 0
    uint64_t dst;        // device address of row 0
    uint64_t row_bytes;  // contiguous bytes per row on both sides
    uint32_t n_outer;    // dims that enumerate rows (outermost first)
    uint32_t pad;
    uint64_t size[kBoxMaxDim];
    int64_t sstr[kBoxMaxDim];  // byte strides
    int64_t dstr[kBoxMaxDim];
};

struct __align__(16) BoxTile {
    uint64_t row;       // first row
    uint64_t nrows;     // rows covered (1: a byte range of one row)
    uint64_t byte_off;  // nrows == 1: first byte inside the row
    uint32_t box;
    uint32_t nbytes;    // nrows == 1: bytes covered
};

constexpr int kBoxThreads = 256;
constexpr uint64_t kBoxWarpRow = 32;  // rows at least this long get a warp each

__device__ __forceinline__ void box_row_addr(const BoxDesc& b, uint64_t r, uint8_t* staging, const uint8_t*& s, uint8_t*& d) {
    int64_t so = 0, dof = 0;
    for (int k = static_cast<int>(b.n_outer) - 1; k >= 0; --k) {
        const uint64_t n = b.size[k];
        const uint64_t q = r / n;
        const int64_t i = static_cast<int64_t>(r - q * n);
        so += i * b.sstr[k];
        dof += i * b.dstr[k];
        r = q;
    }
    s = staging + b.src + so;
    d = reinterpret_cast<uint8_t*>(b.dst) + dof;
}

// a short row (< 32 bytes) by one thread, in the widest access both addresses and the length allow
__device__ __forceinline__ void copy_short(uint8_t* d, const uint8_t* s, uint32_t n) {
    const uint32_t al = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(d) | reinterpret_cast<uintptr_t>(s)) | n;
    if ((al & 15u) == 0) {
        for (uint32_t i = 0; i < n; i += 16) *reinterpret_cast<int4*>(d + i) = *reinterpret_cast<const int4*>(s + i);
    } else if ((al & 7u) == 0) {
        for (uint32_t i = 0; i < n; i += 8) *reinterpret_cast<uint64_t*>(d + i) = *reinterpret_cast<const uint64_t*>(s + i);
    } else if ((al & 3u) == 0) {
        for (uint32_t i = 0; i < n; i += 4) *reinterpret_cast<uint32_t*>(d + i) = *reinterpret_cast<const uint32_t*>(s + i);
    } else if ((al & 1u) == 0) {
        for (uint32_t i = 0; i < n; i += 2) *reinterpret_cast<uint16_t*>(d + i) = *reinterpret_cast<const uint16_t*>(s + i);
    } else {
        for (uint32_t i = 0; i < n; ++i) d[i] = s[i];
    }
}

// grid = SMs x resident CTAs, CTA b takes tiles b, b+G, b+2G, ...
__global__ void __launch_bounds__(kBoxThreads, 4)
walk_box(const BoxDesc* __restrict__ boxes, const BoxTile* __restrict__ tiles, uint32_t ntiles, uint8_t* staging) {
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    constexpr uint32_t nwarp = kBoxThreads / 32;
    for (uint32_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const BoxTile td = tiles[t];
        const BoxDesc& b = boxes[td.box];
        const uint64_t row_bytes = b.row_bytes;
        if (td.nrows == 1) {
            const uint8_t* s;
            uint8_t* d;
            box_row_addr(b, td.row, staging, s, d);
            copy_bytes<kLdgUnroll>(d + td.byte_off, s + td.byte_off, td.nbytes, tid, kBoxThreads);
        } else if (row_bytes >= kBoxWarpRow) {
            for (uint64_t r = warp; r < td.nrows; r += nwarp) {
                const uint8_t* s;
                uint8_t* d;
                box_row_addr(b, td.row + r, staging, s, d);
                copy_bytes<2>(d, s, static_cast<uint32_t>(row_bytes), lane, 32);
            }
        } else {
            for (uint64_t r = tid; r < td.nrows; r += kBoxThreads) {
                const uint8_t* s;
                uint8_t* d;
                box_row_addr(b, td.row + r, staging, s, d);
                copy_short(d, s, static_cast<uint32_t>(row_bytes));
            }
        }
    }
}

}  // namespace nvrx
