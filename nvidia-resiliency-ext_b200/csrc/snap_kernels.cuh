// snap_kernels.cuh -- sm_90a device code of the snapshot engine: the tile walkers that pack a flattened
// TensorAwareStateDict into one staging buffer and scatter it back.
//
// Pure data movement (no tensor cores): the roofline is HBM bandwidth, algorithmic traffic 2*S bytes per
// S snapshot bytes (1.5*S_in when narrowing fp32->bf16), see DESIGN.md.
//
// Two walkers over the same descriptor tables:
//   walk_ldg  : every CTA takes tiles round-robin; LDG.128 (L1 no-allocate) -> registers -> STG.128,
//               4 vectors in flight per thread; sources/destinations that are not mutually 16-byte aligned
//               go through the warp-shuffle funnel (aligned LDG.128, SHFL the neighbour lane's vector,
//               funnel-shift by the byte misalignment) so HBM still only sees full-width accesses.
//   walk_tma  : warp 0 / lane 0 drives a cp.async.bulk ring (global -> smem mbarrier::complete_tx,
//               smem -> global bulk_group), i.e. the SM's TMA unit moves the aligned body of every tensor
//               without touching the LSU or the register file; warps 1..3 run the LDG/funnel code on the
//               ragged tiles (unaligned tensors, <16 B tails, scalar optimizer steps, narrowed segments).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nvrx {

struct __align__(16) SegDesc {  // one per tensor (32 B)
    uint64_t ptr;      // tensor device address
    uint64_t stg_off;  // byte offset of the packed segment in the staging buffer
    uint64_t nbytes;   // tensor-side byte length
    uint32_t flags;    // NVRX_SEG_*
    uint32_t pad;
};

struct __align__(16) TileDesc {  // one per work granule (16 B)
    uint32_t seg;     // index into SegDesc table
    uint32_t nbytes;  // tensor-side bytes covered by this tile
    uint64_t off;     // tensor-side byte offset inside the segment
};

// Destinations of the fused pack+exchange.  Sharded: staging position p lives in
// bases[p / shard_bytes] + slot_off + p % shard_bytes.
// n_peers == 0 -> single local buffer.  mode kPeerShard: position p goes to ONE peer (all-to-all layout);
// mode kPeerBroadcast: every byte is written to ALL bases at slot_off + p (pack fused with an all-gather:
// the source is read from HBM once and stored over NVLink P2P to each clique member's exchange buffer).
struct PeerMap {
    uint8_t* bases[16];
    uint64_t shard_bytes;
    uint64_t slot_off;
    int n_peers;
    int mode;
    int own;  // kPeerShard only: additionally keep a full copy in the local staging buffer
};
constexpr int kPeerShard = 1;
constexpr int kPeerBroadcast = 2;

constexpr uint32_t kSegNarrow = 0x1u;
constexpr int kDirPack = 0;
constexpr int kDirScatter = 1;

// ------------------------------------------------------------------------------------------------
// memory access primitives
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int4 ld_stream(const int4* p) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ void st_stream(int4* p, const int4& v) {
    asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y),
                 "r"(v.z), "r"(v.w)
                 : "memory");
}
__device__ __forceinline__ int2 ld_stream64(const int2* p) {
    int2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.s32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
__device__ __forceinline__ void st_stream64(int2* p, const int2& v) {
    asm volatile("st.global.L1::no_allocate.v2.s32 [%0], {%1,%2};" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
}
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// fp32 pair -> packed bf16x2 (round-to-nearest-even, NaN -> 0x7FFF), lo in the low half
__device__ __forceinline__ uint32_t cvt_bf16x2(uint32_t lo_f32_bits, uint32_t hi_f32_bits) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(__uint_as_float(hi_f32_bits)), "f"(__uint_as_float(lo_f32_bits)));
    return r;
}
__device__ __forceinline__ uint16_t cvt_bf16(uint32_t f32_bits) {
    uint16_t r;
    asm("cvt.rn.bf16.f32 %0, %1;" : "=h"(r) : "f"(__uint_as_float(f32_bits)));
    return r;
}

// ------------------------------------------------------------------------------------------------
// bit copy of n bytes by a group of `nthr` threads (nthr % 32 == 0, tid in [0,nthr)).
// dst/src may have any alignment.  All global traffic of the body is 16-byte vectors.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int4 funnel16(const int4& a, const int4& b, uint32_t ws, uint32_t bs) {
    // bytes [4*ws + bs/8, +16) of the 32-byte window {a,b}; ws, bs are warp-uniform
    uint32_t w0, w1, w2, w3, w4;
    switch (ws) {
        case 0: w0 = a.x; w1 = a.y; w2 = a.z; w3 = a.w; w4 = b.x; break;
        case 1: w0 = a.y; w1 = a.z; w2 = a.w; w3 = b.x; w4 = b.y; break;
        case 2: w0 = a.z; w1 = a.w; w2 = b.x; w3 = b.y; w4 = b.z; break;
        default: w0 = a.w; w1 = b.x; w2 = b.y; w3 = b.z; w4 = b.w; break;
    }
    int4 o;
    o.x = __funnelshift_r(w0, w1, bs);
    o.y = __funnelshift_r(w1, w2, bs);
    o.z = __funnelshift_r(w2, w3, bs);
    o.w = __funnelshift_r(w3, w4, bs);
    return o;
}

template <int UNROLL>
__device__ __forceinline__ void copy_bytes(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, uint32_t n,
                                           uint32_t tid, uint32_t nthr) {
    // (1) head: bring dst to a 16-byte boundary
    uint32_t head = (16u - (static_cast<uint32_t>(reinterpret_cast<uintptr_t>(dst)) & 15u)) & 15u;
    if (head > n) head = n;
    if (tid < head) dst[tid] = src[tid];
    dst += head;
    src += head;
    n -= head;
    if (n == 0) return;

    const uint32_t a = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(src)) & 15u;
    uint32_t done;  // bytes handled by the vector body
    if (a == 0) {
        // (2a) mutually aligned: straight vector copy, UNROLL loads in flight per thread
        const uint32_t nvec = n >> 4;
        const int4* s4 = reinterpret_cast<const int4*>(src);
        int4* d4 = reinterpret_cast<int4*>(dst);
        uint32_t i = tid;
        for (; i + (UNROLL - 1) * nthr < nvec; i += UNROLL * nthr) {
            int4 v[UNROLL];
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) v[u] = ld_stream(s4 + i + u * nthr);
#pragma unroll
            for (int u = 0; u < UNROLL; ++u) st_stream(d4 + i + u * nthr, v[u]);
        }
        for (; i < nvec; i += nthr) st_stream(d4 + i, ld_stream(s4 + i));
        done = nvec << 4;
    } else {
        // (2b) ragged source: aligned vectors sa[q] start `a` bytes before src; output vector p is the
        // 16 bytes at offset a inside {sa[p], sa[p+1]}.  Lane l owns sa[p]; sa[p+1] comes from lane l+1 by
        // SHFL, lane 31's from one extra load done by lane 0.  Only vectors fully inside [src-a, src+n)
        // are touched, the rest (< 32 B) goes to the byte tail.
        const int nv = static_cast<int>((n + a) >> 4) - 1;  // outputs p in [0,nv) need sa[0..nv]
        if (nv > 0) {
            const int4* sa = reinterpret_cast<const int4*>(src - a);
            int4* d4 = reinterpret_cast<int4*>(dst);
            const uint32_t ws = a >> 2, bs = (a & 3u) * 8u;
            const uint32_t lane = tid & 31u, warp = tid >> 5, nwarp = nthr >> 5;
            for (int base = warp * 32; base < nv; base += nwarp * 32) {
                const int p = base + lane;
                int4 v = make_int4(0, 0, 0, 0), e = make_int4(0, 0, 0, 0);
                if (p <= nv) v = ld_stream(sa + p);
                if (lane == 0 && base + 32 <= nv) e = ld_stream(sa + base + 32);
                int4 nx;
                nx.x = __shfl_down_sync(0xffffffffu, v.x, 1);
                nx.y = __shfl_down_sync(0xffffffffu, v.y, 1);
                nx.z = __shfl_down_sync(0xffffffffu, v.z, 1);
                nx.w = __shfl_down_sync(0xffffffffu, v.w, 1);
                e.x = __shfl_sync(0xffffffffu, e.x, 0);
                e.y = __shfl_sync(0xffffffffu, e.y, 0);
                e.z = __shfl_sync(0xffffffffu, e.z, 0);
                e.w = __shfl_sync(0xffffffffu, e.w, 0);
                if (lane == 31) nx = e;
                if (p < nv) st_stream(d4 + p, funnel16(v, nx, ws, bs));
            }
            done = static_cast<uint32_t>(nv) << 4;
        } else {
            done = 0;
        }
    }
    // (3) byte tail (< 32 B)
    const uint32_t tail = n - done;
    for (uint32_t i = tid; i < tail; i += nthr) dst[done + i] = src[done + i];
}

// fp32 -> bf16 narrowing copy: n = source bytes (multiple of 4), dst receives n/2 bytes.
// Lane-contiguous on both sides: each thread turns ONE 16-byte vector (4 floats) into ONE 8-byte vector, so a warp
// reads 512 contiguous bytes and writes 256 contiguous bytes per instruction (every 32-byte sector fully used; the
// 2 x LDG.128 -> 1 x STG.128 per-thread shape strides lanes by 32 B and touches every sector twice).
template <int UNROLL>
__device__ __forceinline__ void narrow_bytes(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, uint32_t n,
                                             uint32_t tid, uint32_t nthr) {
    const uint32_t nelem = n >> 2;
    uint32_t done = 0;  // elements handled by the vector body
    if (((reinterpret_cast<uintptr_t>(src) & 15u) | (reinterpret_cast<uintptr_t>(dst) & 7u)) == 0) {
        const uint32_t nvec = nelem >> 2;  // 4 floats (int4) -> 4 bf16 (int2)
        const int4* s4 = reinterpret_cast<const int4*>(src);
        int2* d2 = reinterpret_cast<int2*>(dst);
        constexpr int U = 2 * UNROLL;
        uint32_t i = tid;
        for (; i + (U - 1) * nthr < nvec; i += U * nthr) {
            int4 v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) v[u] = ld_stream(s4 + i + u * nthr);
#pragma unroll
            for (int u = 0; u < U; ++u) {
                int2 o;
                o.x = cvt_bf16x2(v[u].x, v[u].y);
                o.y = cvt_bf16x2(v[u].z, v[u].w);
                st_stream64(d2 + i + u * nthr, o);
            }
        }
        for (; i < nvec; i += nthr) {
            const int4 v = ld_stream(s4 + i);
            int2 o;
            o.x = cvt_bf16x2(v.x, v.y);
            o.y = cvt_bf16x2(v.z, v.w);
            st_stream64(d2 + i, o);
        }
        done = nvec << 2;
    }
    const uint32_t* s32 = reinterpret_cast<const uint32_t*>(src);
    uint16_t* d16 = reinterpret_cast<uint16_t*>(dst);
    for (uint32_t i = done + tid; i < nelem; i += nthr) d16[i] = cvt_bf16(__ldg(s32 + i));
}

// bf16 -> fp32 widening copy (exact): n = destination bytes (multiple of 4), src holds n/2 bytes.
// Mirror shape: ONE 8-byte load (4 bf16) -> ONE 16-byte store per thread, lane-contiguous on both sides.
template <int UNROLL>
__device__ __forceinline__ void widen_bytes(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, uint32_t n,
                                            uint32_t tid, uint32_t nthr) {
    const uint32_t nelem = n >> 2;
    uint32_t done = 0;
    if (((reinterpret_cast<uintptr_t>(src) & 7u) | (reinterpret_cast<uintptr_t>(dst) & 15u)) == 0) {
        const uint32_t nvec = nelem >> 2;
        const int2* s2 = reinterpret_cast<const int2*>(src);
        int4* d4 = reinterpret_cast<int4*>(dst);
        constexpr int U = 2 * UNROLL;
        uint32_t i = tid;
        for (; i + (U - 1) * nthr < nvec; i += U * nthr) {
            int2 v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) v[u] = ld_stream64(s2 + i + u * nthr);
#pragma unroll
            for (int u = 0; u < U; ++u) {
                int4 o;
                o.x = v[u].x << 16;
                o.y = v[u].x & 0xffff0000u;
                o.z = v[u].y << 16;
                o.w = v[u].y & 0xffff0000u;
                st_stream(d4 + i + u * nthr, o);
            }
        }
        for (; i < nvec; i += nthr) {
            const int2 v = ld_stream64(s2 + i);
            int4 o;
            o.x = v.x << 16;
            o.y = v.x & 0xffff0000u;
            o.z = v.y << 16;
            o.w = v.y & 0xffff0000u;
            st_stream(d4 + i, o);
        }
        done = nvec << 2;
    }
    const uint16_t* s16 = reinterpret_cast<const uint16_t*>(src);
    uint32_t* d32 = reinterpret_cast<uint32_t*>(dst);
    for (uint32_t i = done + tid; i < nelem; i += nthr) d32[i] = static_cast<uint32_t>(__ldg(s16 + i)) << 16;
}

// staging address of packed position `pos`
__device__ __forceinline__ uint8_t* stg_addr(uint8_t* staging, const PeerMap& pm, uint64_t pos, int copy = 0) {
    if (pm.n_peers == 0) return staging + pos;
    if (pm.mode == kPeerBroadcast) return pm.bases[copy] + pm.slot_off + pos;
    if (pm.own && copy == 0) return staging + pos;
    const uint64_t j = pos / pm.shard_bytes;
    return pm.bases[j] + pm.slot_off + (pos - j * pm.shard_bytes);
}
__device__ __forceinline__ int n_copies(const PeerMap& pm) {
    if (pm.n_peers == 0) return 1;
    return pm.mode == kPeerBroadcast ? pm.n_peers : (pm.own ? 2 : 1);
}

// one tile, executed by a thread group
template <int DIR, int UNROLL>
__device__ __forceinline__ void run_tile(const SegDesc& sd, const TileDesc& td, uint8_t* staging, const PeerMap& pm,
                                         uint32_t tid, uint32_t nthr) {
    uint8_t* ten = reinterpret_cast<uint8_t*>(sd.ptr) + td.off;
    const int copies = (DIR == kDirPack) ? n_copies(pm) : 1;  // broadcast re-reads the tile from L2, HBM sees it once
    for (int c = 0; c < copies; ++c) {
        if (sd.flags & kSegNarrow) {
            uint8_t* stg = stg_addr(staging, pm, sd.stg_off + (td.off >> 1), c);
            if (DIR == kDirPack) narrow_bytes<UNROLL>(stg, ten, td.nbytes, tid, nthr);
            else widen_bytes<UNROLL>(ten, stg, td.nbytes, tid, nthr);
        } else {
            uint8_t* stg = stg_addr(staging, pm, sd.stg_off + td.off, c);
            if (DIR == kDirPack) copy_bytes<UNROLL>(stg, ten, td.nbytes, tid, nthr);
            else copy_bytes<UNROLL>(ten, stg, td.nbytes, tid, nthr);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// walker 1: all-LSU.  grid = SMs x resident CTAs, CTA b takes tiles b, b+G, b+2G, ...
// The next tile's descriptors are fetched before the current tile is copied.
// ------------------------------------------------------------------------------------------------
constexpr int kLdgThreads = 256;
constexpr int kLdgUnroll = 4;

// A launch covers two index ranges of the tile table (the bulk and the ragged tiles of one staging chunk).
struct TileSpan {
    const TileDesc* a;
    const TileDesc* b;
    uint32_t na, nb;
    __device__ __forceinline__ TileDesc at(uint32_t t) const { return t < na ? a[t] : b[t - na]; }
    __device__ __forceinline__ uint32_t size() const { return na + nb; }
};

template <int DIR>
__global__ void __launch_bounds__(kLdgThreads, 4)
walk_ldg(const SegDesc* __restrict__ segs, const TileSpan span, uint8_t* staging, const __grid_constant__ PeerMap pm) {
    const uint32_t ntiles = span.size();
    uint32_t t = blockIdx.x;
    if (t >= ntiles) return;
    TileDesc td = span.at(t);
    SegDesc sd = segs[td.seg];
    while (true) {
        const uint32_t tn = t + gridDim.x;
        TileDesc td_n;
        SegDesc sd_n;
        const bool more = tn < ntiles;
        if (more) {
            td_n = span.at(tn);
            sd_n = segs[td_n.seg];
        }
        run_tile<DIR, kLdgUnroll>(sd, td, staging, pm, threadIdx.x, kLdgThreads);
        if (!more) break;
        t = tn;
        td = td_n;
        sd = sd_n;
    }
}

// ------------------------------------------------------------------------------------------------
// walker 2: TMA bulk-copy ring + ragged warps.
//   span.a[0, na) : bulk tiles -- both sides 16-B aligned, nbytes % 16 == 0, nbytes <= stage_bytes, bit copy
//   span.b[0, nb) : ragged tiles -- everything else
// ------------------------------------------------------------------------------------------------
constexpr int kTmaThreads = 128;

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t"
        "}" ::"r"(bar),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t smem_dst, const void* gsrc, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_dst),
                 "l"(gsrc), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gdst, uint32_t smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_src), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// STAGES smem slots of stage_bytes; LOADS tiles of global->smem kept in flight; up to STAGES-LOADS
// smem->global stores may still be reading their slot.
template <int DIR, int STAGES, int LOADS>
__global__ void __launch_bounds__(kTmaThreads, 1)
walk_tma(const SegDesc* __restrict__ segs, const TileSpan span, uint8_t* staging, uint32_t stage_bytes,
         const __grid_constant__ PeerMap pm) {
    const TileDesc* __restrict__ tiles = span.a;
    const uint32_t nbulk = span.na;
    static_assert(LOADS >= 1 && LOADS < STAGES, "need at least one slot for stores in flight");
    extern __shared__ __align__(1024) uint8_t ring[];
    __shared__ __align__(8) uint64_t full[STAGES];

    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;

    if (warp == 0) {
        if (lane != 0) return;
        // ---- the TMA engine thread ----
        for (int s = 0; s < STAGES; ++s) mbar_init(smem_u32(&full[s]), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");

        const uint32_t first = blockIdx.x, stride = gridDim.x;
        if (first >= nbulk) return;
        const uint32_t n_my = (nbulk - first + stride - 1) / stride;
        const uint32_t ring_base = smem_u32(ring);

        auto issue_load = [&](uint32_t i) {
            const TileDesc td = tiles[first + i * stride];
            const SegDesc sd = segs[td.seg];
            const uint32_t s = i % STAGES;
            const uint8_t* g = (DIR == kDirPack) ? reinterpret_cast<const uint8_t*>(sd.ptr) + td.off
                                                 : stg_addr(staging, pm, sd.stg_off + td.off);
            const uint32_t bar = smem_u32(&full[s]);
            mbar_expect_tx(bar, td.nbytes);
            bulk_g2s(ring_base + s * stage_bytes, g, td.nbytes, bar);
        };

        const uint32_t pre = n_my < static_cast<uint32_t>(LOADS) ? n_my : static_cast<uint32_t>(LOADS);
        for (uint32_t i = 0; i < pre; ++i) issue_load(i);

        for (uint32_t i = 0; i < n_my; ++i) {
            const TileDesc td = tiles[first + i * stride];
            const SegDesc sd = segs[td.seg];
            const uint32_t s = i % STAGES;
            mbar_wait(smem_u32(&full[s]), (i / STAGES) & 1u);
            if (DIR == kDirPack) {
                // one smem slot feeds every destination (own buffer + NVLink peers); one bulk group per tile
                const int copies = n_copies(pm);
                for (int c = 0; c < copies; ++c)
                    bulk_s2g(stg_addr(staging, pm, sd.stg_off + td.off, c), ring_base + s * stage_bytes, td.nbytes);
            } else {
                bulk_s2g(reinterpret_cast<uint8_t*>(sd.ptr) + td.off, ring_base + s * stage_bytes, td.nbytes);
            }
            bulk_commit();
            if (i + LOADS < n_my) {
                // slot (i+LOADS)%STAGES was last read by the store of tile i+LOADS-STAGES
                bulk_wait_read<STAGES - LOADS>();
                issue_load(i + LOADS);
            }
        }
        bulk_wait_all();
        return;
    }

    // ---- ragged warps: one warp per tile ----
    const uint32_t nrag = span.nb;
    const uint32_t nw = (kTmaThreads / 32) - 1;
    for (uint32_t r = blockIdx.x * nw + (warp - 1); r < nrag; r += gridDim.x * nw) {
        const TileDesc td = span.b[r];
        const SegDesc sd = segs[td.seg];
        run_tile<DIR, 4>(sd, td, staging, pm, lane, 32);
    }
}

}  // namespace nvrx
