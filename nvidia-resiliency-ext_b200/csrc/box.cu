// box.cu -- planner + C ABI of the box scatter (include/nvrx_snap.h, "box scatter"): resharded
// torch.distributed.checkpoint loads, saved-chunk sub-boxes in device staging -> destination sub-boxes.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <new>
#include <vector>

#include "box_kernels.cuh"
#include "nvrx_snap.h"

using nvrx::BoxDesc;
using nvrx::BoxTile;

#define NVRX_CUDA(expr)                                       \
    do {                                                      \
        cudaError_t e__ = (expr);                             \
        if (e__ != cudaSuccess) return static_cast<int>(e__); \
    } while (0)

static_assert(NVRX_BOX_MAXDIM == nvrx::kBoxMaxDim, "header and kernel disagree on the dim limit");

struct nvrx_boxplan {
    int device = 0;
    int sm_count = 0;
    uint64_t algo_bytes = 0;
    std::vector<BoxDesc> boxes;  // host copies are authoritative; the device mirrors are made by commit / the first launch
    std::vector<BoxTile> tiles;  // [0, n_copy_tiles): bit copies (walk_box); the rest convert (walk_box_cast)
    size_t n_copy_tiles = 0;
    std::vector<uint32_t> dst_elem;  // destination element size of each box (introspection only)
    BoxDesc* d_boxes = nullptr;
    BoxTile* d_tiles = nullptr;
    bool uploaded = false;
};

namespace {

constexpr uint32_t kDefaultBoxTile = 32768;

inline bool is_pow2(uint64_t v) { return v && !(v & (v - 1)); }

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) == cudaSuccess && prev != dev) cudaSetDevice(dev);
        else prev = -1;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

// element sizes (source, destination) of each cast code; index 0 (bit copy) takes the box's own size
constexpr uint32_t kCastElem[nvrx::kCastCount][2] = {{0, 0}, {4, 2}, {4, 2}, {2, 4}, {2, 4}, {2, 2}, {2, 2}};
static_assert(NVRX_CAST_F32_BF16 == nvrx::kCastF32Bf16 && NVRX_CAST_F32_F16 == nvrx::kCastF32F16 &&
                  NVRX_CAST_BF16_F32 == nvrx::kCastBf16F32 && NVRX_CAST_F16_F32 == nvrx::kCastF16F32 &&
                  NVRX_CAST_BF16_F16 == nvrx::kCastBf16F16 && NVRX_CAST_F16_BF16 == nvrx::kCastF16Bf16,
              "header and kernel disagree on the cast codes");

// One box -> its canonical row geometry (BoxDesc) and its element count; NVRX_E_INVALID on malformed input.  es / ed are
// the source / destination element sizes (equal for a bit copy): source offsets, row_bytes and source strides come out in
// source bytes, destination strides in destination bytes.
int canonical_box(uint32_t es, uint32_t ed, int32_t nd, const int64_t* sizes, uint64_t src_off, const int64_t* sst,
                  const void* dst, const int64_t* dstr, uint64_t staging_bytes, BoxDesc* out, uint64_t* numel_out) {
    if (nd < 0 || nd > NVRX_BOX_MAXDIM) return NVRX_E_INVALID;
    if (!(es == 1 || es == 2 || es == 4 || es == 8 || es == 16)) return NVRX_E_INVALID;
    uint64_t numel = 1;
    for (int k = 0; k < nd; ++k) {
        if (sizes[k] < 0 || sst[k] < 0 || dstr[k] < 0) return NVRX_E_INVALID;
        if (sizes[k] > 1 && dstr[k] == 0) return NVRX_E_INVALID;  // two elements of the destination would share a byte
        numel *= static_cast<uint64_t>(sizes[k]);
    }
    memset(out, 0, sizeof(*out));
    *numel_out = 0;
    if (numel == 0) return NVRX_OK;  // empty box: no tiles (row_bytes stays 0)
    if (!dst) return NVRX_E_INVALID;
    // last source byte (all strides >= 0: the element at the far corner)
    uint64_t last = src_off + es;
    for (int k = 0; k < nd; ++k) last += static_cast<uint64_t>(sizes[k] - 1) * static_cast<uint64_t>(sst[k]) * es;
    if (last > staging_bytes || last < src_off) return NVRX_E_INVALID;
    // drop size-1 dims, then merge neighbours that are contiguous on both sides
    uint64_t sz[NVRX_BOX_MAXDIM];
    int64_t ss[NVRX_BOX_MAXDIM], ds[NVRX_BOX_MAXDIM];
    int m = 0;
    for (int k = 0; k < nd; ++k) {
        if (sizes[k] == 1) continue;
        const uint64_t n = static_cast<uint64_t>(sizes[k]);
        if (m > 0 && ss[m - 1] == sst[k] * static_cast<int64_t>(n) && ds[m - 1] == dstr[k] * static_cast<int64_t>(n)) {
            sz[m - 1] *= n;
            ss[m - 1] = sst[k];
            ds[m - 1] = dstr[k];
            continue;
        }
        sz[m] = n;
        ss[m] = sst[k];
        ds[m] = dstr[k];
        ++m;
    }
    out->src = src_off;
    out->dst = reinterpret_cast<uint64_t>(dst);
    if (m > 0 && ss[m - 1] == 1 && ds[m - 1] == 1) {
        out->row_bytes = sz[m - 1] * es;  // a run: the innermost dim is contiguous on both sides
        --m;
    } else {
        out->row_bytes = es;  // element-wise
    }
    out->n_outer = static_cast<uint32_t>(m);
    for (int k = 0; k < m; ++k) {
        out->size[k] = sz[k];
        out->sstr[k] = ss[k] * static_cast<int64_t>(es);
        out->dstr[k] = ds[k] * static_cast<int64_t>(ed);
    }
    *numel_out = numel;
    return NVRX_OK;
}

// Tiles of ~tile_bytes on the wider side (source bytes tile_bytes / max(es, ed) * es, a multiple of es; tile_bytes itself
// for a bit copy): a row longer than half a tile is cut into byte ranges, shorter rows are grouped.
void box_tiles(const BoxDesc& b, uint32_t index, uint32_t tile_bytes, uint32_t es, uint32_t ed, std::vector<BoxTile>& tiles) {
    if (b.row_bytes == 0) return;
    tile_bytes = tile_bytes / std::max(es, ed) * es;
    uint64_t rows = 1;
    for (uint32_t k = 0; k < b.n_outer; ++k) rows *= b.size[k];
    BoxTile t;
    t.box = index;
    if (b.row_bytes * 2 > tile_bytes) {
        for (uint64_t r = 0; r < rows; ++r) {
            for (uint64_t o = 0; o < b.row_bytes; o += tile_bytes) {
                t.row = r;
                t.nrows = 1;
                t.byte_off = o;
                t.nbytes = static_cast<uint32_t>(std::min<uint64_t>(tile_bytes, b.row_bytes - o));
                tiles.push_back(t);
            }
        }
        return;
    }
    const uint64_t per = tile_bytes / b.row_bytes;
    for (uint64_t r = 0; r < rows; r += per) {
        t.row = r;
        t.nrows = std::min(per, rows - r);
        t.byte_off = 0;
        t.nbytes = static_cast<uint32_t>(b.row_bytes);
        tiles.push_back(t);
    }
}

int boxplan_create(int64_t n, const uint32_t* elem_bytes, const int32_t* ndim, const int64_t* sizes, const uint64_t* src_offs,
                   const int64_t* src_strides, const void* const* dst_ptrs, const int64_t* dst_strides, const uint32_t* cast,
                   uint64_t staging_bytes, uint32_t tile_bytes, int device, nvrx_boxplan** out) {
    if (!out || n < 0 || (n > 0 && (!elem_bytes || !ndim || !src_offs || !dst_ptrs))) return NVRX_E_INVALID;
    if (n > 0xffffffffll) return NVRX_E_INVALID;
    if (tile_bytes == 0) tile_bytes = kDefaultBoxTile;
    if (!is_pow2(tile_bytes) || tile_bytes < 4096 || tile_bytes > 65536) return NVRX_E_INVALID;
    int64_t total_dims = 0;
    for (int64_t i = 0; i < n; ++i) {
        if (ndim[i] < 0 || ndim[i] > NVRX_BOX_MAXDIM) return NVRX_E_INVALID;
        total_dims += ndim[i];
    }
    if (total_dims > 0 && (!sizes || !src_strides || !dst_strides)) return NVRX_E_INVALID;
    nvrx_boxplan* p = new (std::nothrow) nvrx_boxplan();
    if (!p) return NVRX_E_NOMEM;
    try {  // the ABI never throws: container growth failures become NVRX_E_NOMEM
        p->device = device;
        p->boxes.resize(static_cast<size_t>(n));
        p->dst_elem.resize(static_cast<size_t>(n));
        std::vector<BoxTile> cast_tiles;
        int64_t d0 = 0;
        for (int64_t i = 0; i < n; ++i) {
            const uint32_t code = cast ? cast[i] : 0u;
            uint32_t es = elem_bytes[i], ed = es;
            int rc = NVRX_OK;
            if (code >= nvrx::kCastCount) {
                rc = NVRX_E_INVALID;
            } else if (code != 0) {
                ed = kCastElem[code][1];
                if (es != kCastElem[code][0] || src_offs[i] % es != 0 || reinterpret_cast<uintptr_t>(dst_ptrs[i]) % ed != 0)
                    rc = NVRX_E_INVALID;
            }
            uint64_t numel = 0;
            if (rc == NVRX_OK)
                rc = canonical_box(es, ed, ndim[i], sizes + d0, src_offs[i], src_strides + d0, dst_ptrs[i], dst_strides + d0,
                                   staging_bytes, &p->boxes[i], &numel);
            if (rc) {
                delete p;
                return rc;
            }
            p->boxes[i].cast = code;
            p->dst_elem[i] = ed;
            p->algo_bytes += numel * (es + ed);
            d0 += ndim[i];
            box_tiles(p->boxes[i], static_cast<uint32_t>(i), tile_bytes, es, ed, code ? cast_tiles : p->tiles);
        }
        p->n_copy_tiles = p->tiles.size();
        p->tiles.insert(p->tiles.end(), cast_tiles.begin(), cast_tiles.end());
        if (p->tiles.size() > 0xffffffffull) {
            delete p;
            return NVRX_E_INVALID;
        }
    } catch (const std::bad_alloc&) {
        delete p;
        return NVRX_E_NOMEM;
    }
    *out = p;
    return NVRX_OK;
}

}  // namespace

extern "C" {

int nvrx_boxplan_create(int64_t n, const uint32_t* elem_bytes, const int32_t* ndim, const int64_t* sizes,
                        const uint64_t* src_offs, const int64_t* src_strides, const void* const* dst_ptrs,
                        const int64_t* dst_strides, uint64_t staging_bytes, uint32_t tile_bytes, int device,
                        nvrx_boxplan** out) {
    return boxplan_create(n, elem_bytes, ndim, sizes, src_offs, src_strides, dst_ptrs, dst_strides, nullptr, staging_bytes,
                          tile_bytes, device, out);
}

int nvrx_boxplan_create_cast(int64_t n, const uint32_t* elem_bytes, const int32_t* ndim, const int64_t* sizes,
                             const uint64_t* src_offs, const int64_t* src_strides, const void* const* dst_ptrs,
                             const int64_t* dst_strides, const uint32_t* cast, uint64_t staging_bytes, uint32_t tile_bytes,
                             int device, nvrx_boxplan** out) {
    return boxplan_create(n, elem_bytes, ndim, sizes, src_offs, src_strides, dst_ptrs, dst_strides, cast, staging_bytes,
                          tile_bytes, device, out);
}

int nvrx_boxplan_destroy(nvrx_boxplan* p) {
    if (!p) return NVRX_OK;
    if (p->d_boxes || p->d_tiles) {
        DeviceGuard guard(p->device);
        if (p->d_boxes) cudaFree(p->d_boxes);
        if (p->d_tiles) cudaFree(p->d_tiles);
    }
    delete p;
    return NVRX_OK;
}

int nvrx_boxplan_info(const nvrx_boxplan* p, uint64_t* n_tiles, uint64_t* algorithmic_bytes) {
    if (!p) return NVRX_E_INVALID;
    if (n_tiles) *n_tiles = p->tiles.size();
    if (algorithmic_bytes) *algorithmic_bytes = p->algo_bytes;
    return NVRX_OK;
}

int nvrx_boxplan_tiles(const nvrx_boxplan* p, uint64_t* n_tiles, uint32_t* box, uint64_t* row, uint64_t* nrows,
                       uint64_t* byte_off, uint32_t* nbytes, uint64_t capacity) {
    if (!p) return NVRX_E_INVALID;
    if (n_tiles) *n_tiles = p->tiles.size();
    for (uint64_t i = 0; i < p->tiles.size() && i < capacity; ++i) {
        const BoxTile& t = p->tiles[i];
        if (box) box[i] = t.box;
        if (row) row[i] = t.row;
        if (nrows) nrows[i] = t.nrows;
        if (byte_off) byte_off[i] = t.byte_off;
        if (nbytes) nbytes[i] = t.nbytes;
    }
    return NVRX_OK;
}

int nvrx_boxplan_box(const nvrx_boxplan* p, int64_t i, uint64_t* row_bytes, uint32_t* n_outer, uint64_t* sizes,
                     int64_t* src_stride, int64_t* dst_stride, uint64_t* src_off, uint64_t* dst) {
    if (!p || i < 0 || static_cast<uint64_t>(i) >= p->boxes.size()) return NVRX_E_INVALID;
    const BoxDesc& b = p->boxes[static_cast<size_t>(i)];
    if (row_bytes) *row_bytes = b.row_bytes;
    if (n_outer) *n_outer = b.n_outer;
    for (int k = 0; k < NVRX_BOX_MAXDIM; ++k) {
        if (sizes) sizes[k] = b.size[k];
        if (src_stride) src_stride[k] = b.sstr[k];
        if (dst_stride) dst_stride[k] = b.dstr[k];
    }
    if (src_off) *src_off = b.src;
    if (dst) *dst = b.dst;
    return NVRX_OK;
}

int nvrx_boxplan_box_cast(const nvrx_boxplan* p, int64_t i, uint32_t* cast, uint32_t* dst_elem_bytes) {
    if (!p || i < 0 || static_cast<uint64_t>(i) >= p->boxes.size()) return NVRX_E_INVALID;
    const BoxDesc& b = p->boxes[static_cast<size_t>(i)];
    if (cast) *cast = b.cast;
    if (dst_elem_bytes) *dst_elem_bytes = p->dst_elem[static_cast<size_t>(i)];
    return NVRX_OK;
}

namespace {

int box_upload(nvrx_boxplan* p, cudaStream_t st) {
    if (!p->uploaded && !p->tiles.empty()) {
        // a plan is used for one launch (one batch of a load): plain stream-ordered copies of the two tables
        if (p->sm_count == 0) NVRX_CUDA(cudaDeviceGetAttribute(&p->sm_count, cudaDevAttrMultiProcessorCount, p->device));
        const size_t bb = p->boxes.size() * sizeof(BoxDesc), tb = p->tiles.size() * sizeof(BoxTile);
        NVRX_CUDA(cudaMalloc(reinterpret_cast<void**>(&p->d_boxes), bb));
        NVRX_CUDA(cudaMalloc(reinterpret_cast<void**>(&p->d_tiles), tb));
        NVRX_CUDA(cudaMemcpyAsync(p->d_boxes, p->boxes.data(), bb, cudaMemcpyHostToDevice, st));
        NVRX_CUDA(cudaMemcpyAsync(p->d_tiles, p->tiles.data(), tb, cudaMemcpyHostToDevice, st));
        p->uploaded = true;
    }
    return NVRX_OK;
}

}  // namespace

int nvrx_boxplan_commit(nvrx_boxplan* p, void* stream) {
    if (!p) return NVRX_E_INVALID;
    DeviceGuard guard(p->device);
    return box_upload(p, static_cast<cudaStream_t>(stream));
}

int nvrx_box_scatter(nvrx_boxplan* p, const void* staging, void* stream) {
    if (!p) return NVRX_E_INVALID;
    if (p->tiles.empty()) return NVRX_OK;
    if (!staging) return NVRX_E_INVALID;
    const uint32_t ncopy = static_cast<uint32_t>(p->n_copy_tiles);
    const uint32_t ncast = static_cast<uint32_t>(p->tiles.size() - p->n_copy_tiles);
    if (ncast && reinterpret_cast<uintptr_t>(staging) % 4 != 0) return NVRX_E_INVALID;  // source elements must be aligned
    DeviceGuard guard(p->device);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = box_upload(p, st);
    if (rc) return rc;
    uint8_t* stg = const_cast<uint8_t*>(static_cast<const uint8_t*>(staging));
    const uint32_t max_grid = static_cast<uint32_t>(p->sm_count) * 8;  // 8 resident CTAs of 256 threads per SM
    if (ncopy) {
        const uint32_t grid = std::max<uint32_t>(1, std::min(max_grid, ncopy));
        nvrx::walk_box<<<grid, nvrx::kBoxThreads, 0, st>>>(p->d_boxes, p->d_tiles, ncopy, stg);
        NVRX_CUDA(cudaGetLastError());
    }
    if (ncast) {
        const uint32_t grid = std::max<uint32_t>(1, std::min(max_grid, ncast));
        nvrx::walk_box_cast<<<grid, nvrx::kBoxThreads, 0, st>>>(p->d_boxes, p->d_tiles + ncopy, ncast, stg);
        NVRX_CUDA(cudaGetLastError());
    }
    return NVRX_OK;
}

}  // extern "C"
