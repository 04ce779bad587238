// xor.cu -- nvrx_xor_reduce: byte-wise XOR of n equally long device ranges into one, the parity of an erasure-coded local
// checkpoint (include/nvrx_snap.h).  HBM-bound: (n + 1) x bytes of traffic, (2n + 1) x bytes when the sources are cleared.
// nvrx_gf_combine: up to 4 GF(2^8) linear combinations of up to 64 ranges in one pass, the Reed-Solomon parity (and its
// decode) when a clique keeps more than one parity fragment.
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

// ---- GF(2^8) combine ----------------------------------------------------------------------------------------------
constexpr int kGfMaxDsts = 4;
constexpr int kGfMaxSrcs = 64;
constexpr int kGfThreads = 256;
constexpr int kGfUnroll = 4;
constexpr int kGfTabWords = 6;  // per coefficient: 2 + 2 PRMT table words, 2 splat words

struct GfArgs {
    const int4* src[kGfMaxSrcs];
    int4* dst[kGfMaxDsts];
    uint8_t coef[kGfMaxDsts * kGfMaxSrcs];  // row-major [d][s], n_src columns used
    int n_src;
};

__device__ __forceinline__ uint32_t gf_mul_slow(uint32_t a, uint32_t b) {  // shift and reduce by 0x11d (table build only)
    uint32_t r = 0;
    for (int i = 0; i < 8; ++i) {
        if (b & 1u) r ^= a;
        b >>= 1;
        a = (a << 1) ^ ((a & 0x80u) ? 0x11du : 0u);
    }
    return r & 0xffu;
}

__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {  // PTX semantics: selector bit 3 = sign mode
    uint32_t d;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
    return d;
}

// Table words of coefficient c: t[0..1] = c*{0..7}, t[2..3] = c*{0x00,0x10,..,0x70}, t[4] = splat(c*0x08), t[5] = splat(c*0x80).
// GF multiplication is linear over XOR, so c*b = c*(b&7) ^ c*(b&0x70) ^ c*(b&8) ^ c*(b&0x80): two 8-entry PRMT lookups
// (one PRMT covers 8 table bytes) and two byte masks instead of 16-entry tables, whose bit 3 would need a second PRMT
// and a select per nibble.
__device__ __forceinline__ uint32_t gf_table_word(uint32_t c, int w) {
    if (w >= 4) return gf_mul_slow(c, w == 4 ? 0x08u : 0x80u) * 0x01010101u;
    const uint32_t base = (w & 1) * 4, shift = (w >> 1) * 4;
    uint32_t r = 0;
    for (uint32_t j = 0; j < 4; ++j) r |= gf_mul_slow(c, (base + j) << shift) << (8 * j);
    return r;
}

// Per source word, shared by every coefficient applied to it: the PRMT selectors of bits 0-2 and 4-6 of each byte, and
// 0x00/0xff byte masks of bits 3 and 7 (PRMT sign mode replicates a byte's bit 7).  The selectors are built from the word
// with bytes 1 and 2 swapped, which makes the cheap nibble compaction below come out in natural byte order.
struct GfSel {
    uint32_t lo, hi, m3, m7;
};

__device__ __forceinline__ GfSel gf_sel(uint32_t x) {
    const uint32_t xs = prmt(x, 0u, 0x3120u);
    GfSel s;
    s.lo = (xs & 0x0707u) | ((xs >> 12) & 0x7070u);
    s.hi = ((xs >> 4) & 0x0707u) | ((xs >> 16) & 0x7070u);
    s.m3 = prmt(x << 4, 0u, 0xBA98u);
    s.m7 = prmt(x, 0u, 0xBA98u);
    return s;
}

__device__ __forceinline__ uint32_t gf_mul_word(const GfSel& s, const uint32_t* t) {
    return prmt(t[0], t[1], s.lo) ^ prmt(t[2], t[3], s.hi) ^ (s.m3 & t[4]) ^ (s.m7 & t[5]);
}

__device__ __forceinline__ void xor4(int4& a, const int4& b) {
    a.x ^= b.x;
    a.y ^= b.y;
    a.z ^= b.z;
    a.w ^= b.w;
}

template <int U>
__device__ __forceinline__ void gf_madd(int4 (&acc)[U], const int4 (&v)[U], const uint32_t* t) {
#pragma unroll
    for (int u = 0; u < U; ++u) {
        acc[u].x ^= gf_mul_word(gf_sel(v[u].x), t);
        acc[u].y ^= gf_mul_word(gf_sel(v[u].y), t);
        acc[u].z ^= gf_mul_word(gf_sel(v[u].z), t);
        acc[u].w ^= gf_mul_word(gf_sel(v[u].w), t);
    }
}

// ND destinations (a template parameter, so the accumulators stay in registers).  The coefficient of (d, s) is uniform
// across the grid: 0 skips, 1 is a plain XOR, anything else goes through the shared-memory tables.  Loop shape and
// load/clear rules as in xor_reduce.
template <int ND, bool CLEAR>
__global__ void __launch_bounds__(kGfThreads, ND <= 2 ? 3 : 2) gf_combine(const __grid_constant__ GfArgs a, uint64_t nvec) {
    __shared__ uint32_t tab[kGfMaxDsts * kGfMaxSrcs * kGfTabWords];
    const int ns = a.n_src;
    for (int e = threadIdx.x; e < ND * ns * kGfTabWords; e += kGfThreads) {
        const int ds = e / kGfTabWords;
        tab[e] = gf_table_word(a.coef[(ds / ns) * kGfMaxSrcs + ds % ns], e % kGfTabWords);
    }
    __syncthreads();
    const uint64_t nthr = static_cast<uint64_t>(gridDim.x) * kGfThreads;
    uint64_t i = static_cast<uint64_t>(blockIdx.x) * kGfThreads + threadIdx.x;
    const int4 zero = make_int4(0, 0, 0, 0);
    for (; i + (kGfUnroll - 1) * nthr < nvec; i += kGfUnroll * nthr) {
        int4 acc[ND][kGfUnroll];
#pragma unroll
        for (int d = 0; d < ND; ++d)
#pragma unroll
            for (int u = 0; u < kGfUnroll; ++u) acc[d][u] = zero;
        for (int s = 0; s < ns; ++s) {
            int4 v[kGfUnroll];
#pragma unroll
            for (int u = 0; u < kGfUnroll; ++u) v[u] = ld_src<CLEAR>(a.src[s] + i + u * nthr);
            if (CLEAR) {
#pragma unroll
                for (int u = 0; u < kGfUnroll; ++u) nvrx::st_stream(const_cast<int4*>(a.src[s]) + i + u * nthr, zero);
            }
#pragma unroll
            for (int d = 0; d < ND; ++d) {
                const uint32_t c = a.coef[d * kGfMaxSrcs + s];
                if (c == 1u) {
#pragma unroll
                    for (int u = 0; u < kGfUnroll; ++u) xor4(acc[d][u], v[u]);
                } else if (c != 0u) {
                    const uint32_t* t = tab + (d * ns + s) * kGfTabWords;
                    uint32_t tw[kGfTabWords];
#pragma unroll
                    for (int w = 0; w < kGfTabWords; ++w) tw[w] = t[w];
                    gf_madd(acc[d], v, tw);
                }
            }
        }
#pragma unroll
        for (int d = 0; d < ND; ++d)
#pragma unroll
            for (int u = 0; u < kGfUnroll; ++u) nvrx::st_stream(a.dst[d] + i + u * nthr, acc[d][u]);
    }
    for (; i < nvec; i += nthr) {
        int4 acc[ND][1];
#pragma unroll
        for (int d = 0; d < ND; ++d) acc[d][0] = zero;
        for (int s = 0; s < ns; ++s) {
            int4 v[1] = {ld_src<CLEAR>(a.src[s] + i)};
            if (CLEAR) nvrx::st_stream(const_cast<int4*>(a.src[s]) + i, zero);
#pragma unroll
            for (int d = 0; d < ND; ++d) {
                const uint32_t c = a.coef[d * kGfMaxSrcs + s];
                if (c == 1u) {
                    xor4(acc[d][0], v[0]);
                } else if (c != 0u) {
                    const uint32_t* t = tab + (d * ns + s) * kGfTabWords;
                    uint32_t tw[kGfTabWords];
#pragma unroll
                    for (int w = 0; w < kGfTabWords; ++w) tw[w] = t[w];
                    gf_madd(acc[d], v, tw);
                }
            }
        }
#pragma unroll
        for (int d = 0; d < ND; ++d) nvrx::st_stream(a.dst[d] + i, acc[d][0]);
    }
}

template <int ND, bool CLEAR>
cudaError_t launch_gf(const GfArgs& a, uint64_t nvec, int sms, cudaStream_t st) {
    constexpr int per_sm = ND <= 2 ? 3 : 2;
    const uint64_t want = (nvec + kGfThreads - 1) / kGfThreads;
    const uint32_t grid = static_cast<uint32_t>(std::max<uint64_t>(1, std::min<uint64_t>(want, static_cast<uint64_t>(sms) * per_sm)));
    gf_combine<ND, CLEAR><<<grid, kGfThreads, 0, st>>>(a, nvec);
    return cudaGetLastError();
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

extern "C" int nvrx_gf_combine(void* const* dsts, int n_dst, void* const* srcs, int n_src, const uint8_t* coef, uint64_t bytes,
                               int clear_srcs, void* stream) {
    if (!dsts || !srcs || !coef || n_dst < 1 || n_dst > kGfMaxDsts || n_src < 1 || n_src > kGfMaxSrcs || (bytes & 15u))
        return NVRX_E_INVALID;
    GfArgs a;
    a.n_src = n_src;
    for (int d = 0; d < kGfMaxDsts; ++d) a.dst[d] = nullptr;
    for (int s = 0; s < kGfMaxSrcs; ++s) a.src[s] = nullptr;
    for (int e = 0; e < kGfMaxDsts * kGfMaxSrcs; ++e) a.coef[e] = 0;
    for (int d = 0; d < n_dst; ++d) {
        const uintptr_t p = reinterpret_cast<uintptr_t>(dsts[d]);
        if (!p || (p & 15u)) return NVRX_E_INVALID;
        for (int e = 0; e < d; ++e)
            if (overlaps(p, reinterpret_cast<uintptr_t>(a.dst[e]), bytes)) return NVRX_E_INVALID;
        a.dst[d] = reinterpret_cast<int4*>(p);
        for (int s = 0; s < n_src; ++s) a.coef[d * kGfMaxSrcs + s] = coef[d * n_src + s];
    }
    for (int s = 0; s < n_src; ++s) {
        const uintptr_t p = reinterpret_cast<uintptr_t>(srcs[s]);
        if (!p || (p & 15u)) return NVRX_E_INVALID;
        for (int d = 0; d < n_dst; ++d)
            if (overlaps(p, reinterpret_cast<uintptr_t>(a.dst[d]), bytes)) return NVRX_E_INVALID;
        a.src[s] = reinterpret_cast<const int4*>(p);
    }
    const uint64_t nvec = bytes >> 4;
    if (nvec == 0) return NVRX_OK;
    int dev = 0, sms = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return static_cast<int>(e);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (n_dst * 2 + (clear_srcs ? 1 : 0)) {
        case 2: e = launch_gf<1, false>(a, nvec, sms, st); break;
        case 3: e = launch_gf<1, true>(a, nvec, sms, st); break;
        case 4: e = launch_gf<2, false>(a, nvec, sms, st); break;
        case 5: e = launch_gf<2, true>(a, nvec, sms, st); break;
        case 6: e = launch_gf<3, false>(a, nvec, sms, st); break;
        case 7: e = launch_gf<3, true>(a, nvec, sms, st); break;
        case 8: e = launch_gf<4, false>(a, nvec, sms, st); break;
        default: e = launch_gf<4, true>(a, nvec, sms, st); break;
    }
    return e == cudaSuccess ? NVRX_OK : static_cast<int>(e);
}
