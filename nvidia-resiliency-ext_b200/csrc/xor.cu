// xor.cu -- nvrx_xor_reduce: byte-wise XOR of n equally long device ranges into one, the parity of an erasure-coded local
// checkpoint (include/nvrx_snap.h).  HBM-bound: (n + 1) x bytes of traffic, (2n + 1) x bytes when the sources are cleared.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "nvrx_snap.h"
#include "snap_kernels.cuh"

namespace {

constexpr int kXorMaxSrcs = 64;
constexpr int kXorThreads = 256;
constexpr int kXorUnroll = 4;
constexpr int kXorCtasPerSm = 3;  // 78-80 registers per thread, no spills (ptxas); capped at 64 for 4 CTAs/SM it spills

struct XorSrcs {
    const int4* p[kXorMaxSrcs];
};

// Sources that the kernel also zeroes are read with coherent loads: a non-coherent (ld.global.nc) load is not ordered
// with the same thread's later store to the same address, which may land first and make the load return the zero.
__device__ __forceinline__ int4 ld_src_cleared(const int4* p) {
    int4 r;
    asm volatile("ld.global.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p)
                 : "memory");
    return r;
}

template <bool CLEAR>
__device__ __forceinline__ int4 ld_src(const int4* p) {
    return CLEAR ? ld_src_cleared(p) : nvrx::ld_stream(p);
}

// Grid-stride over 16-byte vectors, kXorUnroll vectors in flight per thread and source.  Every vector is read and (with
// CLEAR) zeroed by the one thread that owns it, read first.
template <bool CLEAR>
__global__ void __launch_bounds__(kXorThreads, kXorCtasPerSm) xor_reduce(int4* __restrict__ dst, const __grid_constant__ XorSrcs srcs, int n,
                                                           uint64_t nvec) {
    const uint64_t nthr = static_cast<uint64_t>(gridDim.x) * kXorThreads;
    uint64_t i = static_cast<uint64_t>(blockIdx.x) * kXorThreads + threadIdx.x;
    const int4 zero = make_int4(0, 0, 0, 0);
    for (; i + (kXorUnroll - 1) * nthr < nvec; i += kXorUnroll * nthr) {
        int4 acc[kXorUnroll];
#pragma unroll
        for (int u = 0; u < kXorUnroll; ++u) acc[u] = ld_src<CLEAR>(srcs.p[0] + i + u * nthr);
        if (CLEAR) {
#pragma unroll
            for (int u = 0; u < kXorUnroll; ++u) nvrx::st_stream(const_cast<int4*>(srcs.p[0]) + i + u * nthr, zero);
        }
        for (int s = 1; s < n; ++s) {
            int4 v[kXorUnroll];
#pragma unroll
            for (int u = 0; u < kXorUnroll; ++u) v[u] = ld_src<CLEAR>(srcs.p[s] + i + u * nthr);
#pragma unroll
            for (int u = 0; u < kXorUnroll; ++u) {
                acc[u].x ^= v[u].x;
                acc[u].y ^= v[u].y;
                acc[u].z ^= v[u].z;
                acc[u].w ^= v[u].w;
            }
            if (CLEAR) {
#pragma unroll
                for (int u = 0; u < kXorUnroll; ++u) nvrx::st_stream(const_cast<int4*>(srcs.p[s]) + i + u * nthr, zero);
            }
        }
#pragma unroll
        for (int u = 0; u < kXorUnroll; ++u) nvrx::st_stream(dst + i + u * nthr, acc[u]);
    }
    for (; i < nvec; i += nthr) {
        int4 acc = ld_src<CLEAR>(srcs.p[0] + i);
        if (CLEAR) nvrx::st_stream(const_cast<int4*>(srcs.p[0]) + i, zero);
        for (int s = 1; s < n; ++s) {
            const int4 v = ld_src<CLEAR>(srcs.p[s] + i);
            acc.x ^= v.x;
            acc.y ^= v.y;
            acc.z ^= v.z;
            acc.w ^= v.w;
            if (CLEAR) nvrx::st_stream(const_cast<int4*>(srcs.p[s]) + i, zero);
        }
        nvrx::st_stream(dst + i, acc);
    }
}

inline bool overlaps(uintptr_t a, uintptr_t b, uint64_t bytes) { return a < b + bytes && b < a + bytes; }

}  // namespace

extern "C" int nvrx_xor_reduce(void* dst, void* const* srcs, int n, uint64_t bytes, int clear_srcs, void* stream) {
    if (!dst || !srcs || n < 1 || n > kXorMaxSrcs || (bytes & 15u)) return NVRX_E_INVALID;
    const uintptr_t d = reinterpret_cast<uintptr_t>(dst);
    if (d & 15u) return NVRX_E_INVALID;
    XorSrcs s;
    for (int j = 0; j < n; ++j) {
        const uintptr_t p = reinterpret_cast<uintptr_t>(srcs[j]);
        if (!p || (p & 15u) || overlaps(p, d, bytes)) return NVRX_E_INVALID;
        s.p[j] = reinterpret_cast<const int4*>(p);
    }
    for (int j = n; j < kXorMaxSrcs; ++j) s.p[j] = nullptr;
    const uint64_t nvec = bytes >> 4;
    if (nvec == 0) return NVRX_OK;
    int dev = 0, sms = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return static_cast<int>(e);
    // one resident wave: kXorCtasPerSm CTAs per SM, fewer when the range is small
    const uint64_t want = (nvec + kXorThreads - 1) / kXorThreads;
    const uint32_t grid = static_cast<uint32_t>(std::max<uint64_t>(1, std::min<uint64_t>(want, static_cast<uint64_t>(sms) * kXorCtasPerSm)));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (clear_srcs) xor_reduce<true><<<grid, kXorThreads, 0, st>>>(static_cast<int4*>(dst), s, n, nvec);
    else xor_reduce<false><<<grid, kXorThreads, 0, st>>>(static_cast<int4*>(dst), s, n, nvec);
    e = cudaGetLastError();
    return e == cudaSuccess ? NVRX_OK : static_cast<int>(e);
}
