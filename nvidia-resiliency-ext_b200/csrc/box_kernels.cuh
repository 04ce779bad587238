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
//
// Boxes that convert fp32 / bf16 / fp16 into another of the three (a checkpoint loaded into a model of another dtype) have
// tiles of their own after the copy tiles, walked by walk_box_cast with the same three shapes; walk_box never sees them.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "snap_kernels.cuh"

namespace nvrx {

constexpr int kBoxMaxDim = 8;

// dtype conversion of a box (NVRX_CAST_* in nvrx_snap.h); 0 = bit copy
enum : uint32_t {
    kCastNone = 0,
    kCastF32Bf16 = 1,
    kCastF32F16 = 2,
    kCastBf16F32 = 3,
    kCastF16F32 = 4,
    kCastBf16F16 = 5,
    kCastF16Bf16 = 6,
    kCastCount = 7
};

struct __align__(16) BoxDesc {
    uint64_t src;        // staging byte offset of row 0
    uint64_t dst;        // device address of row 0
    uint64_t row_bytes;  // contiguous bytes per row on both sides (converting box: source bytes)
    uint32_t n_outer;    // dims that enumerate rows (outermost first)
    uint32_t cast;       // kCast*; walk_box only sees boxes with kCastNone
    uint64_t size[kBoxMaxDim];
    int64_t sstr[kBoxMaxDim];  // byte strides
    int64_t dstr[kBoxMaxDim];
};

struct __align__(16) BoxTile {
    uint64_t row;       // first row
    uint64_t nrows;     // rows covered (1: a byte range of one row)
    uint64_t byte_off;  // nrows == 1: first byte inside the row (converting box: source bytes)
    uint32_t box;
    uint32_t nbytes;    // nrows == 1: bytes covered (converting box: source bytes)
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

// ------------------------------------------------------------------------------------------------
// converting walker: the same tiles and row geometry, fp32 / bf16 / fp16 -> another of the three.
// Narrowing rounds to nearest even (cvt.rn, no .ftz: subnormals kept, overflow -> inf, NaN -> 0x7FFF); widening is exact.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float f32_of_f16(uint32_t h) {
    float f;
    asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"(static_cast<uint16_t>(h)));
    return f;
}
__device__ __forceinline__ uint16_t cvt_f16(float f) {
    uint16_t r;
    asm("cvt.rn.f16.f32 %0, %1;" : "=h"(r) : "f"(f));
    return r;
}
// fp32 pair -> packed f16x2, lo in the low half
__device__ __forceinline__ uint32_t cvt_f16x2(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}
__device__ __forceinline__ int4 ld_vec(const int4* p) { return ld_stream(p); }
__device__ __forceinline__ int2 ld_vec(const int2* p) { return ld_stream64(p); }
__device__ __forceinline__ void st_vec(int4* p, const int4& v) { st_stream(p, v); }
__device__ __forceinline__ void st_vec(int2* p, const int2& v) { st_stream64(p, v); }

// One conversion: S / D source and destination element, V elements per vector (16 B on the wider side), one() per
// element, vec() per vector.
template <uint32_t C>
struct CastOp;
template <>
struct CastOp<kCastF32Bf16> {
    using S = uint32_t;
    using D = uint16_t;
    using SV = int4;
    using DV = int2;
    static constexpr uint32_t V = 4;
    __device__ static D one(S s) { return cvt_bf16(s); }
    __device__ static DV vec(const SV& v) { return make_int2(cvt_bf16x2(v.x, v.y), cvt_bf16x2(v.z, v.w)); }
};
template <>
struct CastOp<kCastF32F16> {
    using S = uint32_t;
    using D = uint16_t;
    using SV = int4;
    using DV = int2;
    static constexpr uint32_t V = 4;
    __device__ static D one(S s) { return cvt_f16(__uint_as_float(s)); }
    __device__ static DV vec(const SV& v) {
        return make_int2(cvt_f16x2(__int_as_float(v.x), __int_as_float(v.y)), cvt_f16x2(__int_as_float(v.z), __int_as_float(v.w)));
    }
};
template <>
struct CastOp<kCastBf16F32> {
    using S = uint16_t;
    using D = uint32_t;
    using SV = int2;
    using DV = int4;
    static constexpr uint32_t V = 4;
    __device__ static D one(S s) { return static_cast<uint32_t>(s) << 16; }
    __device__ static DV vec(const SV& v) {
        const uint32_t x = v.x, y = v.y;
        return make_int4(x << 16, x & 0xffff0000u, y << 16, y & 0xffff0000u);
    }
};
template <>
struct CastOp<kCastF16F32> {
    using S = uint16_t;
    using D = uint32_t;
    using SV = int2;
    using DV = int4;
    static constexpr uint32_t V = 4;
    __device__ static D one(S s) { return __float_as_uint(f32_of_f16(s)); }
    __device__ static DV vec(const SV& v) {
        const uint32_t x = v.x, y = v.y;
        return make_int4(__float_as_int(f32_of_f16(x & 0xffffu)), __float_as_int(f32_of_f16(x >> 16)),
                         __float_as_int(f32_of_f16(y & 0xffffu)), __float_as_int(f32_of_f16(y >> 16)));
    }
};
template <>
struct CastOp<kCastBf16F16> {  // bf16 -> fp32 (exact) -> fp16 (RNE)
    using S = uint16_t;
    using D = uint16_t;
    using SV = int4;
    using DV = int4;
    static constexpr uint32_t V = 8;
    __device__ static uint32_t two(uint32_t w) { return cvt_f16x2(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u)); }
    __device__ static D one(S s) { return cvt_f16(__uint_as_float(static_cast<uint32_t>(s) << 16)); }
    __device__ static DV vec(const SV& v) { return make_int4(two(v.x), two(v.y), two(v.z), two(v.w)); }
};
template <>
struct CastOp<kCastF16Bf16> {  // fp16 -> fp32 (exact) -> bf16 (RNE)
    using S = uint16_t;
    using D = uint16_t;
    using SV = int4;
    using DV = int4;
    static constexpr uint32_t V = 8;
    __device__ static uint32_t two(uint32_t w) {
        return cvt_bf16x2(__float_as_uint(f32_of_f16(w & 0xffffu)), __float_as_uint(f32_of_f16(w >> 16)));
    }
    __device__ static D one(S s) { return cvt_bf16(__float_as_uint(f32_of_f16(s))); }
    __device__ static DV vec(const SV& v) { return make_int4(two(v.x), two(v.y), two(v.z), two(v.w)); }
};

// n elements of one run by a group of `nthr` threads: element head up to the destination's vector boundary, then, if the
// source is vector-aligned at that element, the vector body (one source vector -> one destination vector per thread,
// lane-contiguous on both sides), then the element tail.  Otherwise every remaining element is an element load: still
// lane-contiguous and coalesced, no realignment needed.
template <uint32_t C, int UNROLL>
__device__ __forceinline__ void cast_run(uint8_t* dst, const uint8_t* src, uint32_t n, uint32_t tid, uint32_t nthr) {
    using Op = CastOp<C>;
    using S = typename Op::S;
    using D = typename Op::D;
    using SV = typename Op::SV;
    using DV = typename Op::DV;
    constexpr uint32_t V = Op::V;
    const S* s = reinterpret_cast<const S*>(src);
    D* d = reinterpret_cast<D*>(dst);
    uint32_t head = (V - static_cast<uint32_t>(reinterpret_cast<uintptr_t>(d) / sizeof(D)) % V) % V;
    if (head > n) head = n;
    for (uint32_t i = tid; i < head; i += nthr) d[i] = Op::one(__ldg(s + i));
    uint32_t done = head;
    if ((reinterpret_cast<uintptr_t>(s + head) & (V * sizeof(S) - 1)) == 0) {
        const uint32_t nvec = (n - head) / V;
        const SV* sv = reinterpret_cast<const SV*>(s + head);
        DV* dv = reinterpret_cast<DV*>(d + head);
        uint32_t i = tid;
        for (; i + (UNROLL - 1) * nthr < nvec; i += UNROLL * nthr) {
            SV v[UNROLL];
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) v[u] = ld_vec(sv + i + u * nthr);
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) st_vec(dv + i + u * nthr, Op::vec(v[u]));
        }
        for (; i < nvec; i += nthr) st_vec(dv + i, Op::vec(ld_vec(sv + i)));
        done += nvec * V;
    }
    for (uint32_t i = done + tid; i < n; i += nthr) d[i] = Op::one(__ldg(s + i));
}

// one tile of a converting box; the three tile shapes of walk_box, byte ranges and row_bytes in source bytes
template <uint32_t C>
__device__ __forceinline__ void cast_tile(const BoxDesc& b, const BoxTile& td, uint8_t* staging, uint32_t tid) {
    using Op = CastOp<C>;
    constexpr uint32_t es = sizeof(typename Op::S), ed = sizeof(typename Op::D);
    const uint32_t lane = tid & 31u, warp = tid >> 5;
    constexpr uint32_t nwarp = kBoxThreads / 32;
    const uint64_t row_bytes = b.row_bytes;
    if (td.nrows == 1) {
        const uint8_t* s;
        uint8_t* d;
        box_row_addr(b, td.row, staging, s, d);
        cast_run<C, kLdgUnroll>(d + td.byte_off / es * ed, s + td.byte_off, td.nbytes / es, tid, kBoxThreads);
    } else if (row_bytes >= kBoxWarpRow) {
        for (uint64_t r = warp; r < td.nrows; r += nwarp) {
            const uint8_t* s;
            uint8_t* d;
            box_row_addr(b, td.row + r, staging, s, d);
            cast_run<C, 2>(d, s, static_cast<uint32_t>(row_bytes / es), lane, 32);
        }
    } else {
        const uint32_t n = static_cast<uint32_t>(row_bytes / es);
        for (uint64_t r = tid; r < td.nrows; r += kBoxThreads) {
            const uint8_t* s;
            uint8_t* d;
            box_row_addr(b, td.row + r, staging, s, d);
            const typename Op::S* s_el = reinterpret_cast<const typename Op::S*>(s);
            typename Op::D* d_el = reinterpret_cast<typename Op::D*>(d);
            for (uint32_t j = 0; j < n; ++j) d_el[j] = Op::one(__ldg(s_el + j));
        }
    }
}

// converting tiles only (the planner puts them after the copy tiles); the code is per box, so the switch is uniform per
// tile.  Same grid rule as walk_box.
__global__ void __launch_bounds__(kBoxThreads, 4)
walk_box_cast(const BoxDesc* __restrict__ boxes, const BoxTile* __restrict__ tiles, uint32_t ntiles, uint8_t* staging) {
    for (uint32_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const BoxTile td = tiles[t];
        const BoxDesc& b = boxes[td.box];
        switch (b.cast) {
            case kCastF32Bf16: cast_tile<kCastF32Bf16>(b, td, staging, threadIdx.x); break;
            case kCastF32F16: cast_tile<kCastF32F16>(b, td, staging, threadIdx.x); break;
            case kCastBf16F32: cast_tile<kCastBf16F32>(b, td, staging, threadIdx.x); break;
            case kCastF16F32: cast_tile<kCastF16F32>(b, td, staging, threadIdx.x); break;
            case kCastBf16F16: cast_tile<kCastBf16F16>(b, td, staging, threadIdx.x); break;
            case kCastF16Bf16: cast_tile<kCastF16Bf16>(b, td, staging, threadIdx.x); break;
            default: break;
        }
    }
}

}  // namespace nvrx
