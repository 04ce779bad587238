// snap_api.cu -- planner + C ABI of libnvrx_snap.so (see include/nvrx_snap.h for the contract and the
// reference file:line each entry point replaces).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <new>
#include <vector>

#include "nvrx_snap.h"
#include "snap_kernels.cuh"

using nvrx::PeerMap;
using nvrx::SegDesc;
using nvrx::TileDesc;
using nvrx::TileSpan;

#define NVRX_CUDA(expr)                                   \
    do {                                                  \
        cudaError_t e__ = (expr);                         \
        if (e__ != cudaSuccess) return static_cast<int>(e__); \
    } while (0)

namespace {

constexpr uint64_t kDefaultAlign = 512;
constexpr uint32_t kDefaultTile = 32768;
constexpr uint32_t kMinBulkBytes = 1024;  // smaller aligned pieces are cheaper on the ragged warps

inline uint64_t round_up(uint64_t v, uint64_t a) { return (v + a - 1) / a * a; }
inline bool is_pow2(uint64_t v) { return v && !(v & (v - 1)); }

struct DeviceGuard {
    int prev = -1;
    bool ok = false;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) == cudaSuccess) {
            ok = (prev == dev) || cudaSetDevice(dev) == cudaSuccess;
            if (prev == dev) prev = -1;
        }
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

}  // namespace

struct nvrx_plan {
    int device = 0;
    int sm_count = 0;
    int64_t n = 0;
    uint64_t align = kDefaultAlign;
    uint32_t tile_bytes = kDefaultTile;
    int variant = NVRX_VARIANT_AUTO;
    bool any_narrow = false;

    std::vector<uint64_t> ptrs, nbytes, off, packed;
    std::vector<uint32_t> flags;
    uint64_t staging_bytes = 0;
    uint64_t algo_bytes = 0;

    // sharding of the packed range for the fused exchange (0 = none); the walk starts at shard `first_shard`
    uint64_t shard_bytes = 0;
    uint32_t first_shard = 0;

    // descriptor tables.  The planner itself never touches CUDA (so its logic is testable without a GPU): host
    // vectors are authoritative, the pinned upload mirror and the device copy are created by the first upload.
    std::vector<SegDesc> h_segs;
    std::vector<TileDesc> h_tiles;  // [0,n_bulk) bulk, [n_bulk,n_tiles) ragged
    SegDesc* pin_segs = nullptr;
    TileDesc* pin_tiles = nullptr;
    SegDesc* d_segs = nullptr;
    TileDesc* d_tiles = nullptr;
    size_t segs_cap = 0, tiles_cap = 0;  // capacity (entries) of the pinned / device mirrors
    uint32_t n_bulk = 0, n_tiles = 0;
    bool segs_dirty = true, tiles_dirty = true;
    std::vector<cudaEvent_t> chunk_events;  // pack -> drain hand-off of the pipelined snapshot
    cudaEvent_t upload_done = nullptr;      // last H2D of the descriptor mirrors (they are reused)
    uint32_t last_launches = 0;             // kernel launches of the last nvrx_snapshot (its pack groups)
};

namespace {

// Build the tile list: tiles[0,n_bulk) are TMA-eligible, the rest ragged.  Both are emitted in segment
// order so that neighbouring CTAs touch neighbouring DRAM pages.
int build_tiles(nvrx_plan* p) {
    std::vector<TileDesc> bulk, ragged;
    const uint32_t T = p->tile_bytes;
    size_t est = 0;
    for (int64_t i = 0; i < p->n; ++i) est += static_cast<size_t>(p->nbytes[i] / T + 2);
    bulk.reserve(est);
    for (int64_t i = 0; i < p->n; ++i) {
        const uint64_t nb = p->nbytes[i];
        if (nb == 0) continue;
        const bool narrow = (p->flags[i] & NVRX_SEG_NARROW_F32_BF16) != 0;
        const bool ptr_al = (p->ptrs[i] & 15u) == 0;
        const uint64_t scale = narrow ? 2 : 1;  // tensor bytes per staging byte
        uint64_t o = 0;
        while (o < nb) {
            uint64_t len = std::min<uint64_t>(T, nb - o);
            if (p->shard_bytes) {
                // never let a tile straddle a shard boundary of the packed range
                const uint64_t pos = p->off[i] + o / scale;
                const uint64_t room = (p->shard_bytes - pos % p->shard_bytes) * scale;
                len = std::min(len, room);
            }
            TileDesc td;
            td.seg = static_cast<uint32_t>(i);
            td.off = o;
            if (!narrow && ptr_al && len >= kMinBulkBytes) {
                const uint32_t body = static_cast<uint32_t>(len & ~uint64_t(15));
                td.nbytes = body;
                bulk.push_back(td);
                if (len > body) {
                    td.off = o + body;
                    td.nbytes = static_cast<uint32_t>(len - body);
                    ragged.push_back(td);
                }
            } else {
                td.nbytes = static_cast<uint32_t>(len);
                ragged.push_back(td);
            }
            o += len;
        }
    }
    const size_t total = bulk.size() + ragged.size();
    if (total > 0xffffffffull) return NVRX_E_INVALID;
    if (p->shard_bytes) {
        auto pos_of = [&](const TileDesc& t) {
            const bool nr = (p->flags[t.seg] & NVRX_SEG_NARROW_F32_BF16) != 0;
            return p->off[t.seg] + (nr ? t.off / 2 : t.off);
        };
        const char* env = getenv("NVRX_B200_SHARD_INTERLEAVE");
        const bool interleave = !(env && env[0] == '0');
        if (interleave) {
            // Destination-major balance for the fused pack + all-to-all: list position q holds a tile of shard
            // (first_shard + q) mod n_shards.  CTAs take list positions b, b+G, b+2G, ..., so at every moment the CTAs of
            // this GPU are spread evenly over ALL destination GPUs (each peer gets 1/n of this GPU's NVLink egress, and
            // receives 1/n from each of its n senders) -- no destination sees more than one GPU's worth of ingress, whatever
            // the relative progress of the ranks.  Walking the shards one after the other made every rank store into the
            // same one or two peers at a time (incast).
            auto weave = [&](std::vector<TileDesc>& v) {
                if (v.empty()) return;
                const uint64_t n_shards = (p->staging_bytes + p->shard_bytes - 1) / p->shard_bytes;
                if (n_shards < 2) return;
                std::vector<size_t> begin(n_shards + 1, v.size());  // v is sorted by staging position
                size_t i = 0;
                for (uint64_t sh = 0; sh < n_shards; ++sh) {
                    while (i < v.size() && pos_of(v[i]) / p->shard_bytes < sh) ++i;
                    begin[sh] = i;
                }
                begin[n_shards] = v.size();
                for (uint64_t sh = n_shards; sh-- > 0;) begin[sh] = std::min(begin[sh], begin[sh + 1]);
                std::vector<TileDesc> out;
                out.reserve(v.size());
                std::vector<size_t> cur(begin.begin(), begin.end() - 1);
                size_t left = v.size();
                uint64_t sh = p->first_shard % n_shards;
                while (left) {
                    if (cur[sh] < begin[sh + 1]) {
                        out.push_back(v[cur[sh]++]);
                        --left;
                    }
                    sh = (sh + 1 == n_shards) ? 0 : sh + 1;
                }
                v.swap(out);
            };
            weave(bulk);
            weave(ragged);
        } else if (p->first_shard) {
            // Sequential walk, rotated so that it starts with the tiles of shard `first_shard` and wraps around: with a
            // different starting shard on every rank the ranks of a clique store into distinct peers as long as they stay
            // in step (kept for the A/B measurement, NVRX_B200_SHARD_INTERLEAVE=0).
            const uint64_t start = static_cast<uint64_t>(p->first_shard) * p->shard_bytes;
            auto rot = [&](std::vector<TileDesc>& v) {
                auto it = std::partition_point(v.begin(), v.end(), [&](const TileDesc& t) { return pos_of(t) < start; });
                std::rotate(v.begin(), it, v.end());
            };
            rot(bulk);
            rot(ragged);
        }
    }
    p->h_tiles.clear();
    p->h_tiles.reserve(total);
    p->h_tiles.insert(p->h_tiles.end(), bulk.begin(), bulk.end());
    p->h_tiles.insert(p->h_tiles.end(), ragged.begin(), ragged.end());
    p->n_bulk = static_cast<uint32_t>(bulk.size());
    p->n_tiles = static_cast<uint32_t>(total);
    p->tiles_dirty = true;
    return NVRX_OK;
}

void fill_segs(nvrx_plan* p) {
    p->h_segs.resize(static_cast<size_t>(p->n));
    for (int64_t i = 0; i < p->n; ++i) {
        SegDesc& s = p->h_segs[i];
        s.ptr = p->ptrs[i];
        s.stg_off = p->off[i];
        s.nbytes = p->nbytes[i];
        s.flags = p->flags[i];
        s.pad = 0;
    }
    p->segs_dirty = true;
}

int upload(nvrx_plan* p, cudaStream_t st) {
    if (p->sm_count == 0) NVRX_CUDA(cudaDeviceGetAttribute(&p->sm_count, cudaDevAttrMultiProcessorCount, p->device));
    if (!(p->segs_dirty && p->n > 0) && !(p->tiles_dirty && p->n_tiles > 0)) {
        p->segs_dirty = p->tiles_dirty = false;
        return NVRX_OK;
    }
    // the pinned mirrors are about to be rewritten: an earlier upload must have finished reading them
    if (p->upload_done) NVRX_CUDA(cudaEventSynchronize(p->upload_done));
    else NVRX_CUDA(cudaEventCreateWithFlags(&p->upload_done, cudaEventDisableTiming));
    if (p->segs_dirty && p->n > 0) {
        const size_t n = static_cast<size_t>(p->n);
        if (n > p->segs_cap) {
            if (p->pin_segs) cudaFreeHost(p->pin_segs);
            if (p->d_segs) cudaFree(p->d_segs);
            p->pin_segs = nullptr;
            p->d_segs = nullptr;
            p->segs_cap = 0;
            NVRX_CUDA(cudaMallocHost(reinterpret_cast<void**>(&p->pin_segs), n * sizeof(SegDesc)));
            NVRX_CUDA(cudaMalloc(reinterpret_cast<void**>(&p->d_segs), n * sizeof(SegDesc)));
            p->segs_cap = n;
        }
        memcpy(p->pin_segs, p->h_segs.data(), n * sizeof(SegDesc));
        NVRX_CUDA(cudaMemcpyAsync(p->d_segs, p->pin_segs, n * sizeof(SegDesc), cudaMemcpyHostToDevice, st));
    }
    p->segs_dirty = false;
    if (p->tiles_dirty && p->n_tiles > 0) {
        const size_t n = p->n_tiles;
        if (n > p->tiles_cap) {
            const size_t cap = std::max<size_t>(n + n / 8, 64);
            if (p->pin_tiles) cudaFreeHost(p->pin_tiles);
            if (p->d_tiles) cudaFree(p->d_tiles);
            p->pin_tiles = nullptr;
            p->d_tiles = nullptr;
            p->tiles_cap = 0;
            NVRX_CUDA(cudaMallocHost(reinterpret_cast<void**>(&p->pin_tiles), cap * sizeof(TileDesc)));
            NVRX_CUDA(cudaMalloc(reinterpret_cast<void**>(&p->d_tiles), cap * sizeof(TileDesc)));
            p->tiles_cap = cap;
        }
        memcpy(p->pin_tiles, p->h_tiles.data(), n * sizeof(TileDesc));
        NVRX_CUDA(cudaMemcpyAsync(p->d_tiles, p->pin_tiles, n * sizeof(TileDesc), cudaMemcpyHostToDevice, st));
    }
    p->tiles_dirty = false;
    NVRX_CUDA(cudaEventRecord(p->upload_done, st));
    return NVRX_OK;
}

// ring geometry of the TMA walker: STAGES smem slots of tile_bytes, LOADS tiles of loads in flight.
// The deepest ring that fits the 227 KB of shared memory is chosen unless NVRX_B200_TMA_STAGES overrides it.
constexpr size_t kSmemBudget = 200 * 1024;

int pick_stages(uint32_t tile_bytes) {
    // default: 32 KiB x 4 stages x 1 CTA/SM (128 KiB of the 227 KiB an H100 block may have); tools/gpu_selftest.py sweeps
    // the alternatives (16 KiB x 6 x 2 CTAs/SM, 64 KiB x 3) on the card at hand.
    static const int kChoices[] = {12, 8, 6, 4, 3};
    int want = tile_bytes >= 65536 ? 3 : tile_bytes >= 32768 ? 4 : tile_bytes >= 16384 ? 6 : 12;
    if (const char* env = getenv("NVRX_B200_TMA_STAGES")) want = atoi(env);
    for (int c : kChoices) {
        if (static_cast<size_t>(c) * tile_bytes > kSmemBudget) continue;
        if (c <= want) return c;
    }
    return 3;
}

template <int DIR, int STAGES, int LOADS>
int launch_tma(nvrx_plan* p, const TileSpan& span, uint8_t* staging, const PeerMap& pm, cudaStream_t st) {
    const size_t smem = static_cast<size_t>(STAGES) * p->tile_bytes;
    auto kern = nvrx::walk_tma<DIR, STAGES, LOADS>;
    NVRX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    uint32_t per_sm = static_cast<uint32_t>(std::max<size_t>(1, std::min<size_t>(4, (220 * 1024) / (smem + 2048))));
    if (const char* env = getenv("NVRX_B200_TMA_CTAS_PER_SM")) per_sm = std::max(1, atoi(env));
    uint32_t grid = static_cast<uint32_t>(p->sm_count) * per_sm;
    const uint32_t need = std::max<uint32_t>(span.na, (span.nb + 2) / 3);
    grid = std::max<uint32_t>(1, std::min(grid, need));
    kern<<<grid, nvrx::kTmaThreads, smem, st>>>(p->d_segs, span, staging, p->tile_bytes, pm);
    NVRX_CUDA(cudaGetLastError());
    return NVRX_OK;
}

template <int DIR>
int launch_span(nvrx_plan* p, const TileSpan& span, uint8_t* staging, const PeerMap& pm, cudaStream_t st) {
    if (span.na + span.nb == 0) return NVRX_OK;
    int variant = p->variant;
    if (variant == NVRX_VARIANT_AUTO) variant = (p->any_narrow || p->n_bulk == 0) ? NVRX_VARIANT_LDG : NVRX_VARIANT_TMA;
    if (variant == NVRX_VARIANT_TMA) {
        switch (pick_stages(p->tile_bytes)) {
            case 12: return launch_tma<DIR, 12, 8>(p, span, staging, pm, st);
            case 8: return launch_tma<DIR, 8, 6>(p, span, staging, pm, st);
            case 6: return launch_tma<DIR, 6, 4>(p, span, staging, pm, st);
            case 4: return launch_tma<DIR, 4, 3>(p, span, staging, pm, st);
            default: return launch_tma<DIR, 3, 2>(p, span, staging, pm, st);
        }
    }
    uint32_t per_sm = 8;  // grid of 8 CTAs per SM (tools/gpu_selftest.py sweeps it)
    if (const char* env = getenv("NVRX_B200_LDG_CTAS_PER_SM")) per_sm = std::max(1, atoi(env));
    uint32_t grid = static_cast<uint32_t>(p->sm_count) * per_sm;
    grid = std::max<uint32_t>(1, std::min(grid, span.na + span.nb));
    nvrx::walk_ldg<DIR><<<grid, nvrx::kLdgThreads, 0, st>>>(p->d_segs, span, staging, pm);
    NVRX_CUDA(cudaGetLastError());
    return NVRX_OK;
}

TileSpan whole_span(const nvrx_plan* p) {
    TileSpan s;
    s.a = p->d_tiles;
    s.na = p->n_bulk;
    s.b = p->d_tiles + p->n_bulk;
    s.nb = p->n_tiles - p->n_bulk;
    return s;
}

template <int DIR>
int launch(nvrx_plan* p, uint8_t* staging, const PeerMap& pm, cudaStream_t st) {
    return launch_span<DIR>(p, whole_span(p), staging, pm, st);
}

// staging position of a tile (bulk and ragged lists are each sorted by it: tiles are emitted in segment order)
inline uint64_t tile_pos(const nvrx_plan* p, const TileDesc& t) {
    const bool narrow = (p->flags[t.seg] & NVRX_SEG_NARROW_F32_BF16) != 0;
    return p->off[t.seg] + (narrow ? t.off / 2 : t.off);
}

// first index in tiles[lo, hi) whose staging position is >= pos
uint32_t lower_tile(const nvrx_plan* p, uint32_t lo, uint32_t hi, uint64_t pos) {
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (tile_pos(p, p->h_tiles[mid]) < pos) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

}  // namespace

extern "C" {

int nvrx_abi_version(void) { return NVRX_ABI_VERSION; }

const char* nvrx_strerror(int status) {
    switch (status) {
        case NVRX_OK: return "ok";
        case NVRX_E_INVALID: return "nvrx: invalid argument";
        case NVRX_E_NOMEM: return "nvrx: out of host memory";
        case NVRX_E_STATE: return "nvrx: invalid state or timeout";
        case NVRX_E_SYS: return "nvrx: operating-system call failed";
        case NVRX_E_NODRIVER: return "nvrx: CUDA driver entry point unavailable";
        default: break;
    }
    if (status > 0 && status < 1000) return cudaGetErrorString(static_cast<cudaError_t>(status));
    return "nvrx: unknown status";
}

int nvrx_device_info(int device, int* sm_count, uint64_t* l2_bytes, char* name, int name_len) {
    cudaDeviceProp prop;
    NVRX_CUDA(cudaGetDeviceProperties(&prop, device));
    if (sm_count) *sm_count = prop.multiProcessorCount;
    if (l2_bytes) *l2_bytes = static_cast<uint64_t>(prop.l2CacheSize);
    if (name && name_len > 0) {
        strncpy(name, prop.name, static_cast<size_t>(name_len) - 1);
        name[name_len - 1] = 0;
    }
    return NVRX_OK;
}

int nvrx_plan_create(int64_t n, const void* const* ptrs, const uint64_t* nbytes, const uint32_t* flags, uint64_t align,
                     uint32_t tile_bytes, int device, nvrx_plan** out) {
    return nvrx_plan_create_at(n, ptrs, nbytes, flags, nullptr, align, tile_bytes, device, out);
}

int nvrx_plan_create_at(int64_t n, const void* const* ptrs, const uint64_t* nbytes, const uint32_t* flags,
                        const uint64_t* staging_offsets, uint64_t align, uint32_t tile_bytes, int device, nvrx_plan** out) {
    if (!out || n < 0 || (n > 0 && (!ptrs || !nbytes))) return NVRX_E_INVALID;
    if (staging_offsets) {
        // caller-chosen layout (e.g. the record offsets of a checkpoint container): 16-byte aligned, ascending, disjoint
        uint64_t prev_end = 0;
        for (int64_t i = 0; i < n; ++i) {
            const bool nr = flags && (flags[i] & NVRX_SEG_NARROW_F32_BF16);
            if ((staging_offsets[i] & 15u) || staging_offsets[i] < prev_end) return NVRX_E_INVALID;
            prev_end = staging_offsets[i] + (nr ? nbytes[i] / 2 : nbytes[i]);
        }
    }
    if (align == 0) align = kDefaultAlign;
    if (tile_bytes == 0) tile_bytes = kDefaultTile;
    if (!is_pow2(align) || align < 16) return NVRX_E_INVALID;
    if (!is_pow2(tile_bytes) || tile_bytes < 4096 || tile_bytes > 65536) return NVRX_E_INVALID;
    for (int64_t i = 0; i < n; ++i) {
        const uint32_t f = flags ? flags[i] : 0;
        if (nbytes[i] && !ptrs[i]) return NVRX_E_INVALID;
        if (f & ~NVRX_SEG_NARROW_F32_BF16) return NVRX_E_INVALID;
        if ((f & NVRX_SEG_NARROW_F32_BF16) && ((nbytes[i] & 3u) || (reinterpret_cast<uintptr_t>(ptrs[i]) & 3u)))
            return NVRX_E_INVALID;
    }
    nvrx_plan* p = new (std::nothrow) nvrx_plan();
    if (!p) return NVRX_E_NOMEM;
    try {  // the ABI never throws: container growth failures become NVRX_E_NOMEM
    p->device = device;
    p->n = n;
    p->align = align;
    p->tile_bytes = tile_bytes;
    p->ptrs.resize(n);
    p->nbytes.assign(nbytes, nbytes + n);
    p->flags.resize(n);
    p->off.resize(n);
    p->packed.resize(n);
    uint64_t cur = 0, src_total = 0, packed_total = 0;
    for (int64_t i = 0; i < n; ++i) {
        p->ptrs[i] = reinterpret_cast<uint64_t>(ptrs[i]);
        p->flags[i] = flags ? flags[i] : 0;
        const bool narrow = (p->flags[i] & NVRX_SEG_NARROW_F32_BF16) != 0;
        p->any_narrow |= narrow;
        p->packed[i] = narrow ? p->nbytes[i] / 2 : p->nbytes[i];
        cur = staging_offsets ? staging_offsets[i] : round_up(cur, align);
        p->off[i] = cur;
        cur += p->packed[i];
        src_total += p->nbytes[i];
        packed_total += p->packed[i];
    }
    p->staging_bytes = round_up(cur, align);
    p->algo_bytes = src_total + packed_total;

    fill_segs(p);
    int rc = build_tiles(p);
    if (rc) {
        nvrx_plan_destroy(p);
        return rc;
    }
    } catch (const std::bad_alloc&) {
        nvrx_plan_destroy(p);
        return NVRX_E_NOMEM;
    }
    *out = p;
    return NVRX_OK;
}

int nvrx_plan_destroy(nvrx_plan* p) {
    if (!p) return NVRX_OK;
    if (p->pin_segs || p->pin_tiles || p->d_segs || p->d_tiles || !p->chunk_events.empty() || p->upload_done) {
        DeviceGuard guard(p->device);
        if (p->upload_done) cudaEventDestroy(p->upload_done);
        if (p->pin_segs) cudaFreeHost(p->pin_segs);
        if (p->pin_tiles) cudaFreeHost(p->pin_tiles);
        if (p->d_segs) cudaFree(p->d_segs);
        if (p->d_tiles) cudaFree(p->d_tiles);
    }
    for (cudaEvent_t ev : p->chunk_events) cudaEventDestroy(ev);
    delete p;
    return NVRX_OK;
}

int nvrx_plan_info(const nvrx_plan* p, uint64_t* staging_bytes, uint64_t* n_tiles, uint64_t* algorithmic_bytes) {
    if (!p) return NVRX_E_INVALID;
    if (staging_bytes) *staging_bytes = p->staging_bytes;
    if (n_tiles) *n_tiles = p->n_tiles;
    if (algorithmic_bytes) *algorithmic_bytes = p->algo_bytes;
    return NVRX_OK;
}

int nvrx_plan_layout(const nvrx_plan* p, uint64_t* offsets, uint64_t* packed_nbytes) {
    if (!p) return NVRX_E_INVALID;
    for (int64_t i = 0; i < p->n; ++i) {
        if (offsets) offsets[i] = p->off[i];
        if (packed_nbytes) packed_nbytes[i] = p->packed[i];
    }
    return NVRX_OK;
}

int nvrx_plan_update_ptrs(nvrx_plan* p, const void* const* ptrs) {
    if (!p || (p->n > 0 && !ptrs)) return NVRX_E_INVALID;
    bool same_class = true;
    for (int64_t i = 0; i < p->n; ++i) {
        const uint64_t np = reinterpret_cast<uint64_t>(ptrs[i]);
        if (p->nbytes[i] && !np) return NVRX_E_INVALID;
        if ((p->flags[i] & NVRX_SEG_NARROW_F32_BF16) && (np & 3u)) return NVRX_E_INVALID;
        if (((np ^ p->ptrs[i]) & 15u) != 0) same_class = false;
    }
    for (int64_t i = 0; i < p->n; ++i) p->ptrs[i] = reinterpret_cast<uint64_t>(ptrs[i]);
    try {
        fill_segs(p);
        if (!same_class) return build_tiles(p);
    } catch (const std::bad_alloc&) {
        return NVRX_E_NOMEM;
    }
    return NVRX_OK;
}

int nvrx_plan_set_shard_rotation(nvrx_plan* p, uint32_t first_shard) {
    if (!p) return NVRX_E_INVALID;
    if (p->first_shard != first_shard) {
        p->first_shard = first_shard;
        if (p->shard_bytes) return build_tiles(p);
    }
    return NVRX_OK;
}

int nvrx_plan_tiles(const nvrx_plan* p, uint64_t shard_bytes, uint32_t* n_bulk, uint32_t* n_tiles, uint32_t* seg, uint32_t* nbytes,
                    uint64_t* off, uint64_t capacity) {
    if (!p) return NVRX_E_INVALID;
    const nvrx_plan* src = p;
    nvrx_plan tmp;
    if (shard_bytes != p->shard_bytes) {  // what-if view with another sharding (does not modify the plan)
        tmp.n = p->n;
        tmp.tile_bytes = p->tile_bytes;
        tmp.ptrs = p->ptrs;
        tmp.nbytes = p->nbytes;
        tmp.off = p->off;
        tmp.flags = p->flags;
        tmp.staging_bytes = p->staging_bytes;
        tmp.shard_bytes = shard_bytes;
        tmp.first_shard = p->first_shard;
        int rc = build_tiles(&tmp);
        if (rc) return rc;
        src = &tmp;
    }
    if (n_bulk) *n_bulk = src->n_bulk;
    if (n_tiles) *n_tiles = src->n_tiles;
    for (uint64_t i = 0; i < src->n_tiles && i < capacity; ++i) {
        if (seg) seg[i] = src->h_tiles[i].seg;
        if (nbytes) nbytes[i] = src->h_tiles[i].nbytes;
        if (off) off[i] = src->h_tiles[i].off;
    }
    return NVRX_OK;
}

int nvrx_plan_set_variant(nvrx_plan* p, int variant) {
    if (!p || variant < NVRX_VARIANT_AUTO || variant > NVRX_VARIANT_TMA) return NVRX_E_INVALID;
    p->variant = variant;
    return NVRX_OK;
}

int nvrx_plan_commit(nvrx_plan* p, void* stream) {
    if (!p) return NVRX_E_INVALID;
    DeviceGuard guard(p->device);
    return upload(p, static_cast<cudaStream_t>(stream));
}

int nvrx_pack(nvrx_plan* p, void* staging, void* stream) {
    if (!p || (!staging && p->staging_bytes)) return NVRX_E_INVALID;
    if (reinterpret_cast<uintptr_t>(staging) & 511u) return NVRX_E_INVALID;
    DeviceGuard guard(p->device);
    if (p->shard_bytes) {
        p->shard_bytes = 0;
        int rc = build_tiles(p);
        if (rc) return rc;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = upload(p, st);
    if (rc) return rc;
    PeerMap pm;
    memset(&pm, 0, sizeof(pm));
    return launch<nvrx::kDirPack>(p, static_cast<uint8_t*>(staging), pm, st);
}

int nvrx_scatter(nvrx_plan* p, const void* staging, void* stream) {
    if (!p || (!staging && p->staging_bytes)) return NVRX_E_INVALID;
    if (reinterpret_cast<uintptr_t>(staging) & 511u) return NVRX_E_INVALID;
    DeviceGuard guard(p->device);
    if (p->shard_bytes) {
        p->shard_bytes = 0;
        int rc = build_tiles(p);
        if (rc) return rc;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = upload(p, st);
    if (rc) return rc;
    PeerMap pm;
    memset(&pm, 0, sizeof(pm));
    return launch<nvrx::kDirScatter>(p, const_cast<uint8_t*>(static_cast<const uint8_t*>(staging)), pm, st);
}

int nvrx_pack_sharded(nvrx_plan* p, void* staging, void* const* peer_bases, int n_peers, uint64_t shard_bytes,
                      uint64_t slot_offset, void* stream) {
    if (!p || !peer_bases || n_peers < 1 || n_peers > 16) return NVRX_E_INVALID;
    if (reinterpret_cast<uintptr_t>(staging) & 511u) return NVRX_E_INVALID;
    if (shard_bytes == 0 || (shard_bytes & 511u) || (slot_offset & 511u)) return NVRX_E_INVALID;
    if (shard_bytes * static_cast<uint64_t>(n_peers) < p->staging_bytes) return NVRX_E_INVALID;
    DeviceGuard guard(p->device);
    if (p->shard_bytes != shard_bytes) {
        p->shard_bytes = shard_bytes;
        int rc = build_tiles(p);
        if (rc) return rc;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = upload(p, st);
    if (rc) return rc;
    PeerMap pm;
    memset(&pm, 0, sizeof(pm));
    pm.n_peers = n_peers;
    pm.mode = nvrx::kPeerShard;
    pm.own = staging != nullptr;
    pm.shard_bytes = shard_bytes;
    pm.slot_off = slot_offset;
    for (int j = 0; j < n_peers; ++j) {
        if (!peer_bases[j] || (reinterpret_cast<uintptr_t>(peer_bases[j]) & 511u)) return NVRX_E_INVALID;
        pm.bases[j] = static_cast<uint8_t*>(peer_bases[j]);
    }
    return launch<nvrx::kDirPack>(p, static_cast<uint8_t*>(staging), pm, st);
}

int nvrx_snapshot(nvrx_plan* p, void* staging, void* host_dst, uint64_t chunk_bytes, volatile uint64_t* progress,
                  uint64_t base_value, void* pack_stream, void* drain_stream, void* packed_event, void* done_event) {
    if (!p || (p->staging_bytes && (!staging || !host_dst))) return NVRX_E_INVALID;
    if (reinterpret_cast<uintptr_t>(staging) & 511u) return NVRX_E_INVALID;
    DeviceGuard guard(p->device);
    if (p->shard_bytes) {
        p->shard_bytes = 0;
        int rc = build_tiles(p);
        if (rc) return rc;
    }
    cudaStream_t ps = static_cast<cudaStream_t>(pack_stream), ds = static_cast<cudaStream_t>(drain_stream);
    int rc = upload(p, ps);
    if (rc) return rc;
    const uint64_t total = p->staging_bytes;
    if (chunk_bytes == 0 || chunk_bytes > total) chunk_bytes = total ? total : 1;
    chunk_bytes = round_up(chunk_bytes, 512);
    uint64_t n_chunks = total ? (total + chunk_bytes - 1) / chunk_bytes : 0;
    if (n_chunks > 256) {  // keep the number of launches bounded
        chunk_bytes = round_up((total + 255) / 256, 512);
        n_chunks = (total + chunk_bytes - 1) / chunk_bytes;
    }
    while (p->chunk_events.size() < n_chunks) {
        cudaEvent_t ev;
        NVRX_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        p->chunk_events.push_back(ev);
    }
    void* prog_dev = nullptr;
    if (progress) NVRX_CUDA(cudaHostGetDevicePointer(&prog_dev, const_cast<uint64_t*>(progress), 0));
    PeerMap pm;
    memset(&pm, 0, sizeof(pm));
    // Pack sub-launches cover GROUPS of copy chunks that grow geometrically (1, g, g^2, ... chunks; g = 4 by default,
    // NVRX_B200_PACK_GROWTH, 1 = one launch per chunk): the pack runs ~55x faster than the PCIe copy, so the copy of group
    // k (which must wait for that group's launch) never waits on the pack of group k+1 as long as g < 55, and a 16 GB
    // snapshot needs 4 launches instead of 60 -- no launch gaps and CTA tails on the training stream.  The copies themselves
    // stay `chunk_bytes` long (granularity of the progress word the writer follows).
    uint64_t growth = 4;
    if (const char* env = getenv("NVRX_B200_PACK_GROWTH")) growth = std::max<long long>(1, atoll(env));
    uint32_t b_lo = 0, r_lo = p->n_bulk;
    uint64_t c = 0, group = 1, n_groups = 0;
    while (c < n_chunks) {
        const uint64_t g_end = std::min(n_chunks, c + group);
        const uint64_t end_pos = std::min(total, g_end * chunk_bytes);
        // group = every tile that STARTS before end_pos and was not launched yet; a tile reaching into the next group
        // is complete before that group's event, which is what that group's copies wait for
        const uint32_t b_hi = (g_end == n_chunks) ? p->n_bulk : lower_tile(p, b_lo, p->n_bulk, end_pos);
        const uint32_t r_hi = (g_end == n_chunks) ? p->n_tiles : lower_tile(p, r_lo, p->n_tiles, end_pos);
        TileSpan span;
        span.a = p->d_tiles + b_lo;
        span.na = b_hi - b_lo;
        span.b = p->d_tiles + r_lo;
        span.nb = r_hi - r_lo;
        rc = launch_span<nvrx::kDirPack>(p, span, static_cast<uint8_t*>(staging), pm, ps);
        if (rc) return rc;
        b_lo = b_hi;
        r_lo = r_hi;
        NVRX_CUDA(cudaEventRecord(p->chunk_events[n_groups], ps));
        NVRX_CUDA(cudaStreamWaitEvent(ds, p->chunk_events[n_groups], 0));
        ++n_groups;
        for (; c < g_end; ++c) {
            const uint64_t begin = c * chunk_bytes, stop = std::min(total, (c + 1) * chunk_bytes);
            NVRX_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(host_dst) + begin, static_cast<const uint8_t*>(staging) + begin,
                                      stop - begin, cudaMemcpyDeviceToHost, ds));
            if (prog_dev) {
                rc = nvrx_stream_write_u64(ds, prog_dev, base_value + stop);
                if (rc) return rc;
            }
        }
        group *= growth;
    }
    p->last_launches = static_cast<uint32_t>(n_groups);
    if (n_chunks == 0 && prog_dev) {
        rc = nvrx_stream_write_u64(ds, prog_dev, base_value);
        if (rc) return rc;
    }
    if (packed_event) NVRX_CUDA(cudaEventRecord(static_cast<cudaEvent_t>(packed_event), ps));
    if (done_event) NVRX_CUDA(cudaEventRecord(static_cast<cudaEvent_t>(done_event), ds));
    return NVRX_OK;
}

int nvrx_plan_last_launches(const nvrx_plan* p, uint32_t* launches) {
    if (!p || !launches) return NVRX_E_INVALID;
    *launches = p->last_launches;
    return NVRX_OK;
}

int nvrx_pack_broadcast(nvrx_plan* p, void* const* peer_bases, int n_peers, uint64_t slot_offset, void* stream) {
    if (!p || !peer_bases || n_peers < 1 || n_peers > 16) return NVRX_E_INVALID;
    if (slot_offset & 511u) return NVRX_E_INVALID;
    DeviceGuard guard(p->device);
    if (p->shard_bytes) {
        p->shard_bytes = 0;
        int rc = build_tiles(p);
        if (rc) return rc;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = upload(p, st);
    if (rc) return rc;
    PeerMap pm;
    memset(&pm, 0, sizeof(pm));
    pm.n_peers = n_peers;
    pm.mode = nvrx::kPeerBroadcast;
    pm.slot_off = slot_offset;
    for (int j = 0; j < n_peers; ++j) {
        if (!peer_bases[j] || (reinterpret_cast<uintptr_t>(peer_bases[j]) & 511u)) return NVRX_E_INVALID;
        pm.bases[j] = static_cast<uint8_t*>(peer_bases[j]);
    }
    return launch<nvrx::kDirPack>(p, nullptr, pm, st);
}

}  // extern "C"
