// crc.cu -- host side of the GPU CRC-32 (tables, chunk enumeration, C ABI) and the CPU-only chaining of the partial values.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <new>
#include <vector>

#include "crc_kernels.cuh"
#include "nvrx_snap.h"

using nvrx::CrcChunk;
using nvrx::kCrcChunkRows;
using nvrx::kCrcOpWords;
using nvrx::kCrcRowBytes;

#define NVRX_CUDA(expr)                                       \
    do {                                                      \
        cudaError_t e__ = (expr);                             \
        if (e__ != cudaSuccess) return static_cast<int>(e__); \
    } while (0)

namespace {

// ---- operator tables ------------------------------------------------------------------------------------------------
struct Ops {
    uint32_t byte_tab[256];        // Z(1) restricted to the low byte: the classic table
    uint32_t z1[kCrcOpWords];      // Z(1) as a full operator
    uint32_t z4[kCrcOpWords], z16[kCrcOpWords], z512[kCrcOpWords];
    uint32_t zchunk[kCrcOpWords];  // Z(kCrcChunkRows * 512): chains full chunks on the host
};

void compose(const uint32_t* a, const uint32_t* b, uint32_t* out) {  // out = a o b
    uint32_t tmp[kCrcOpWords];
    for (uint32_t i = 0; i < kCrcOpWords; ++i) tmp[i] = nvrx::crc_apply(a, b[i]);
    memcpy(out, tmp, sizeof(tmp));
}

const Ops& ops() {
    static Ops o;
    static std::once_flag once;
    std::call_once(once, [] {
        for (uint32_t i = 0; i < 256; ++i) {
            uint32_t c = i;
            for (int k = 0; k < 8; ++k) c = (c & 1u) ? (c >> 1) ^ 0xEDB88320u : c >> 1;
            o.byte_tab[i] = c;
        }
        for (uint32_t j = 0; j < 4; ++j)
            for (uint32_t b = 0; b < 256; ++b) {
                const uint32_t s = b << (8 * j);
                o.z1[j * 256 + b] = o.byte_tab[s & 0xffu] ^ (s >> 8);
            }
        uint32_t cur[kCrcOpWords];
        memcpy(cur, o.z1, sizeof(cur));
        for (uint32_t n = 1; n < kCrcChunkRows * kCrcRowBytes;) {  // repeated squaring: Z(2n) = Z(n) o Z(n)
            compose(cur, cur, cur);
            n *= 2;
            if (n == 4) memcpy(o.z4, cur, sizeof(cur));
            if (n == 16) memcpy(o.z16, cur, sizeof(cur));
            if (n == kCrcRowBytes) memcpy(o.z512, cur, sizeof(cur));
            if (n == kCrcChunkRows * kCrcRowBytes) memcpy(o.zchunk, cur, sizeof(cur));
        }
    });
    return o;
}
static_assert((kCrcRowBytes & (kCrcRowBytes - 1)) == 0 && (kCrcChunkRows & (kCrcChunkRows - 1)) == 0, "powers of two");

// ---- chunk enumeration (shared by the device run and the host finish: both must see the same list) --------------------
// Extent i contributes its whole rows of 512 bytes, kCrcChunkRows at a time, when it starts 16-byte aligned; the bytes
// after the last whole row (and unaligned extents as a whole) are left to the host.
template <typename F>
void for_each_chunk(int64_t n, const uint64_t* offsets, const uint64_t* nbytes, F&& f) {
    for (int64_t i = 0; i < n; ++i) {
        if (offsets[i] & 15u) continue;
        uint64_t rows = nbytes[i] / kCrcRowBytes, off = offsets[i];
        while (rows) {
            const uint32_t take = static_cast<uint32_t>(rows < kCrcChunkRows ? rows : kCrcChunkRows);
            f(CrcChunk{off, take, static_cast<uint32_t>(i)});
            off += static_cast<uint64_t>(take) * kCrcRowBytes;
            rows -= take;
        }
    }
}

uint32_t feed_bytes(const Ops& o, uint32_t s, const uint8_t* p, uint64_t n) {
    for (uint64_t k = 0; k < n; ++k) s = o.byte_tab[(s ^ p[k]) & 0xffu] ^ (s >> 8);
    return s;
}

// ---- per-device copy of [Z512 | Z4 | Z16] ---------------------------------------------------------------------------
std::mutex g_dev_lock;
uint32_t* g_dev_tables[64] = {nullptr};

int device_tables(int device, uint32_t** out) {
    if (device < 0 || device >= 64) return NVRX_E_INVALID;
    std::lock_guard<std::mutex> lk(g_dev_lock);
    if (!g_dev_tables[device]) {
        const Ops& o = ops();
        uint32_t* d = nullptr;
        NVRX_CUDA(cudaMalloc(&d, 3 * sizeof(o.z4)));
        cudaError_t e = cudaMemcpy(d, o.z512, sizeof(o.z512), cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemcpy(d + kCrcOpWords, o.z4, sizeof(o.z4), cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemcpy(d + 2 * kCrcOpWords, o.z16, sizeof(o.z16), cudaMemcpyHostToDevice);
        if (e != cudaSuccess) {
            cudaFree(d);
            return static_cast<int>(e);
        }
        g_dev_tables[device] = d;
    }
    *out = g_dev_tables[device];
    return NVRX_OK;
}

}  // namespace

struct nvrx_crc {
    int device = 0;
    int sm_count = 0;
    std::vector<CrcChunk> chunks;
    CrcChunk* d_chunks = nullptr;  // uploaded by the first run
    uint32_t* d_vals = nullptr;    // n values, then (8-byte aligned) the 64-bit ready word
    size_t ready_index = 0;        // index (in 32-bit words) of the ready word inside d_vals
};

int nvrx_crc_create(int64_t n, const uint64_t* offsets, const uint64_t* nbytes, int device, nvrx_crc** out) {
    if (!out || n < 0 || (n > 0 && (!offsets || !nbytes))) return NVRX_E_INVALID;
    nvrx_crc* c = new (std::nothrow) nvrx_crc();
    if (!c) return NVRX_E_NOMEM;
    c->device = device;
    try {
        for_each_chunk(n, offsets, nbytes, [&](const CrcChunk& ch) { c->chunks.push_back(ch); });
    } catch (const std::bad_alloc&) {
        delete c;
        return NVRX_E_NOMEM;
    }
    if (c->chunks.size() > 0xffffffffull) {
        delete c;
        return NVRX_E_INVALID;
    }
    *out = c;
    return NVRX_OK;
}

int nvrx_crc_destroy(nvrx_crc* c) {
    if (!c) return NVRX_OK;
    if (c->d_chunks || c->d_vals) {
        int prev = -1;
        cudaGetDevice(&prev);
        if (prev != c->device) cudaSetDevice(c->device);
        if (c->d_chunks) cudaFree(c->d_chunks);
        if (c->d_vals) cudaFree(c->d_vals);
        if (prev >= 0 && prev != c->device) cudaSetDevice(prev);
    }
    delete c;
    return NVRX_OK;
}

int nvrx_crc_info(const nvrx_crc* c, uint64_t* n_values) {
    if (!c || !n_values) return NVRX_E_INVALID;
    *n_values = c->chunks.size();
    return NVRX_OK;
}

int nvrx_crc_run(nvrx_crc* c, const void* dev_base, uint32_t* host_values, uint64_t* host_ready, uint64_t ready_value,
                 void* stream) {
    if (!c || (!c->chunks.empty() && (!dev_base || !host_values))) return NVRX_E_INVALID;
    if (c->chunks.empty() && !host_ready) return NVRX_OK;
    int prev = -1;
    NVRX_CUDA(cudaGetDevice(&prev));
    if (prev != c->device) NVRX_CUDA(cudaSetDevice(c->device));
    struct Restore {
        int prev, dev;
        ~Restore() {
            if (prev >= 0 && prev != dev) cudaSetDevice(prev);
        }
    } restore{prev, c->device};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t n = c->chunks.size();
    if (!c->d_chunks) {
        NVRX_CUDA(cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, c->device));
        c->ready_index = (n + 1) & ~static_cast<size_t>(1);
        NVRX_CUDA(cudaMalloc(&c->d_chunks, (n ? n : 1) * sizeof(CrcChunk)));
        NVRX_CUDA(cudaMalloc(&c->d_vals, (c->ready_index + 2) * sizeof(uint32_t)));
        // one-time, synchronous: the list is pageable host memory and must be on the device before the first launch
        if (n) NVRX_CUDA(cudaMemcpy(c->d_chunks, c->chunks.data(), n * sizeof(CrcChunk), cudaMemcpyHostToDevice));
    }
    uint32_t* tables = nullptr;
    int rc = device_tables(c->device, &tables);
    if (rc) return rc;
    unsigned long long* d_ready = reinterpret_cast<unsigned long long*>(c->d_vals + c->ready_index);
    const uint8_t* src = static_cast<const uint8_t*>(dev_base);
    const char* variant = getenv("NVRX_B200_CRC_VARIANT");  // "shared": one copy of the tables per CTA (A/B measurements)
    if (variant && !strcmp(variant, "shared")) {
        constexpr int kWarps = 8;
        const uint64_t want = (n + kWarps - 1) / kWarps;
        const uint64_t cap = static_cast<uint64_t>(c->sm_count) * 4;
        const uint32_t grid = static_cast<uint32_t>(want < cap ? want : cap);
        nvrx::crc_chunks<kWarps><<<grid ? grid : 1, kWarps * 32, 0, st>>>(src, c->d_chunks, static_cast<uint32_t>(n), tables,
                                                                           c->d_vals, d_ready,
                                                                           static_cast<unsigned long long>(ready_value));
    } else {
        // default: Z(512) replicated per lane in 128 KiB of shared memory, one 32-warp CTA per SM
        constexpr int kWarps = 32;
        // per device (function attributes live in the device's context); a few microseconds, so simply set it every time
        NVRX_CUDA(cudaFuncSetAttribute(nvrx::crc_chunks_private<kWarps>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(nvrx::kCrcPrivateSmemBytes)));
        const uint64_t want = (n + kWarps - 1) / kWarps;
        const uint32_t grid = static_cast<uint32_t>(want < static_cast<uint64_t>(c->sm_count) ? want : c->sm_count);
        nvrx::crc_chunks_private<kWarps><<<grid ? grid : 1, kWarps * 32, nvrx::kCrcPrivateSmemBytes, st>>>(
            src, c->d_chunks, static_cast<uint32_t>(n), tables, c->d_vals, d_ready, static_cast<unsigned long long>(ready_value));
    }
    NVRX_CUDA(cudaGetLastError());
    if (n) NVRX_CUDA(cudaMemcpyAsync(host_values, c->d_vals, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    if (host_ready) NVRX_CUDA(cudaMemcpyAsync(host_ready, d_ready, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    return NVRX_OK;
}

int nvrx_crc_finish(int64_t n, const uint64_t* offsets, const uint64_t* nbytes, const uint32_t* values, uint64_t n_values,
                    const void* host_base, uint32_t* out_crcs) {
    if (n < 0 || (n > 0 && (!offsets || !nbytes || !out_crcs || !host_base)) || (n_values > 0 && !values)) return NVRX_E_INVALID;
    const Ops& o = ops();
    const uint8_t* base = static_cast<const uint8_t*>(host_base);
    std::vector<uint32_t> state(static_cast<size_t>(n), 0xffffffffu);
    std::vector<uint64_t> done(static_cast<size_t>(n), 0);  // bytes of extent i already covered by chunk values
    uint64_t k = 0;
    bool short_list = false;
    for_each_chunk(n, offsets, nbytes, [&](const CrcChunk& ch) {
        if (k >= n_values) {
            short_list = true;
            return;
        }
        uint32_t s = state[ch.ext];
        if (ch.rows == kCrcChunkRows) {
            s = nvrx::crc_apply(o.zchunk, s);
        } else {
            for (uint32_t r = 0; r < ch.rows; ++r) s = nvrx::crc_apply(o.z512, s);
        }
        state[ch.ext] = s ^ values[k++];
        done[ch.ext] += static_cast<uint64_t>(ch.rows) * kCrcRowBytes;
    });
    if (short_list || k != n_values) return NVRX_E_INVALID;
    for (int64_t i = 0; i < n; ++i) {
        const uint32_t s = feed_bytes(o, state[i], base + offsets[i] + done[i], nbytes[i] - done[i]);
        out_crcs[i] = ~s;
    }
    return NVRX_OK;
}

// ---- extents at any offset and of any length, summed entirely on the device ------------------------------------------
using nvrx::CrcxExtent;
using nvrx::kCrcPow2Tables;

namespace {

// Z(2^k), k = 0..63, back to back: host copy (nvrx_crc32_combine) and one device copy per device (the fold kernel)
const uint32_t* pow2_tables() {
    static std::vector<uint32_t> t;
    static std::once_flag once;
    std::call_once(once, [] {
        t.resize(static_cast<size_t>(kCrcPow2Tables) * kCrcOpWords);
        memcpy(t.data(), ops().z1, sizeof(ops().z1));
        for (uint32_t k = 1; k < kCrcPow2Tables; ++k) {
            const uint32_t* prev = t.data() + (k - 1) * kCrcOpWords;
            compose(prev, prev, t.data() + k * kCrcOpWords);
        }
    });
    return t.data();
}

uint32_t* g_dev_pow2[64] = {nullptr};

int device_pow2_tables(int device, uint32_t** out) {
    if (device < 0 || device >= 64) return NVRX_E_INVALID;
    std::lock_guard<std::mutex> lk(g_dev_lock);
    if (!g_dev_pow2[device]) {
        const size_t bytes = static_cast<size_t>(kCrcPow2Tables) * kCrcOpWords * sizeof(uint32_t);
        uint32_t* d = nullptr;
        NVRX_CUDA(cudaMalloc(&d, bytes));
        const cudaError_t e = cudaMemcpy(d, pow2_tables(), bytes, cudaMemcpyHostToDevice);
        if (e != cudaSuccess) {
            cudaFree(d);
            return static_cast<int>(e);
        }
        g_dev_pow2[device] = d;
    }
    *out = g_dev_pow2[device];
    return NVRX_OK;
}

}  // namespace

struct nvrx_crcx {
    int device = 0;
    int sm_count = 0;
    std::vector<CrcxExtent> ext;
    std::vector<CrcChunk> chunks;  // body chunks of all extents, extent by extent (ext[i].first indexes them)
    uint8_t* d_mem = nullptr;      // [extents | chunks | chunk values | ready word | crcs], uploaded by the first run
    size_t chunks_at = 0, vals_at = 0, ready_at = 0, out_at = 0;
};

int nvrx_crcx_create(int64_t n, const uint64_t* offsets, const uint64_t* nbytes, int device, nvrx_crcx** out) {
    if (!out || n < 0 || n > 0xffffffffll || (n > 0 && (!offsets || !nbytes))) return NVRX_E_INVALID;
    for (int64_t i = 0; i < n; ++i)
        if (offsets[i] + nbytes[i] < offsets[i]) return NVRX_E_INVALID;
    nvrx_crcx* c = new (std::nothrow) nvrx_crcx();
    if (!c) return NVRX_E_NOMEM;
    c->device = device;
    try {
        c->ext.resize(static_cast<size_t>(n));
        for (int64_t i = 0; i < n; ++i) {
            uint32_t head, tail;
            uint64_t rows;
            nvrx::crcx_split(offsets[i], nbytes[i], &head, &rows, &tail);
            c->ext[i] = CrcxExtent{offsets[i], nbytes[i], c->chunks.size()};
            uint64_t off = offsets[i] + head;
            for (uint64_t k = 0, m = nvrx::crcx_chunks(rows); k < m; ++k) {
                const uint32_t r = nvrx::crcx_chunk_rows(rows, k);
                c->chunks.push_back(CrcChunk{off, r, static_cast<uint32_t>(i)});
                off += static_cast<uint64_t>(r) * kCrcRowBytes;
            }
        }
    } catch (const std::bad_alloc&) {
        delete c;
        return NVRX_E_NOMEM;
    }
    if (c->chunks.size() > 0xffffffffull) {
        delete c;
        return NVRX_E_INVALID;
    }
    *out = c;
    return NVRX_OK;
}

int nvrx_crcx_destroy(nvrx_crcx* c) {
    if (!c) return NVRX_OK;
    if (c->d_mem) {
        int prev = -1;
        cudaGetDevice(&prev);
        if (prev != c->device) cudaSetDevice(c->device);
        cudaFree(c->d_mem);
        if (prev >= 0 && prev != c->device) cudaSetDevice(prev);
    }
    delete c;
    return NVRX_OK;
}

int nvrx_crcx_info(const nvrx_crcx* c, uint64_t* n_chunks, uint32_t* launches) {
    if (!c) return NVRX_E_INVALID;
    if (n_chunks) *n_chunks = c->chunks.size();
    if (launches) *launches = (c->chunks.empty() ? 0u : 1u) + (c->ext.empty() ? 0u : 1u);
    return NVRX_OK;
}

namespace {

struct CrcxDevice {  // makes c->device current for the lifetime of the object
    int prev = -1, dev = 0;
    int enter(int d) {
        dev = d;
        NVRX_CUDA(cudaGetDevice(&prev));
        if (prev != dev) NVRX_CUDA(cudaSetDevice(dev));
        return NVRX_OK;
    }
    ~CrcxDevice() {
        if (prev >= 0 && prev != dev) cudaSetDevice(prev);
    }
};

int crcx_upload(nvrx_crcx* c, cudaStream_t st) {
    const size_t n = c->ext.size(), nc = c->chunks.size();
    if (!c->d_mem && n) {
        NVRX_CUDA(cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, c->device));
        const auto up16 = [](size_t v) { return (v + 15) & ~static_cast<size_t>(15); };
        c->chunks_at = up16(n * sizeof(CrcxExtent));
        c->vals_at = up16(c->chunks_at + nc * sizeof(CrcChunk));
        c->ready_at = up16(c->vals_at + nc * sizeof(uint32_t));
        c->out_at = c->ready_at + 16;
        NVRX_CUDA(cudaMalloc(&c->d_mem, c->out_at + n * sizeof(uint32_t)));
        // stream-ordered from pageable memory: the runtime stages the descriptors before this call returns
        NVRX_CUDA(cudaMemcpyAsync(c->d_mem, c->ext.data(), n * sizeof(CrcxExtent), cudaMemcpyHostToDevice, st));
        if (nc)
            NVRX_CUDA(cudaMemcpyAsync(c->d_mem + c->chunks_at, c->chunks.data(), nc * sizeof(CrcChunk), cudaMemcpyHostToDevice, st));
    }
    return NVRX_OK;
}

}  // namespace

int nvrx_crcx_commit(nvrx_crcx* c, void* stream) {
    if (!c) return NVRX_E_INVALID;
    CrcxDevice guard;
    int rc = guard.enter(c->device);
    if (rc) return rc;
    return crcx_upload(c, static_cast<cudaStream_t>(stream));
}

int nvrx_crcx_run(nvrx_crcx* c, const void* dev_base, uint32_t* host_crcs, void* stream) {
    if (!c) return NVRX_E_INVALID;
    const size_t n = c->ext.size(), nc = c->chunks.size();
    if (!n) return NVRX_OK;
    if (!host_crcs || !dev_base || (reinterpret_cast<uintptr_t>(dev_base) & 15u)) return NVRX_E_INVALID;
    CrcxDevice guard;
    int rc = guard.enter(c->device);
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    rc = crcx_upload(c, st);
    if (rc) return rc;
    uint32_t *tables = nullptr, *pow2 = nullptr;
    rc = device_tables(c->device, &tables);
    if (!rc) rc = device_pow2_tables(c->device, &pow2);
    if (rc) return rc;
    const uint8_t* src = static_cast<const uint8_t*>(dev_base);
    uint32_t* vals = reinterpret_cast<uint32_t*>(c->d_mem + c->vals_at);
    uint32_t* crcs = reinterpret_cast<uint32_t*>(c->d_mem + c->out_at);
    if (nc) {  // the bodies: the restore / snapshot checksum kernel, unchanged (its ready word goes to a scratch word)
        constexpr int kWarps = 32;
        NVRX_CUDA(cudaFuncSetAttribute(nvrx::crc_chunks_private<kWarps>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(nvrx::kCrcPrivateSmemBytes)));
        const uint64_t want = (nc + kWarps - 1) / kWarps;
        const uint32_t grid = static_cast<uint32_t>(want < static_cast<uint64_t>(c->sm_count) ? want : c->sm_count);
        nvrx::crc_chunks_private<kWarps><<<grid, kWarps * 32, nvrx::kCrcPrivateSmemBytes, st>>>(
            src, reinterpret_cast<const CrcChunk*>(c->d_mem + c->chunks_at), static_cast<uint32_t>(nc), tables, vals,
            reinterpret_cast<unsigned long long*>(c->d_mem + c->ready_at), 0ull);
        NVRX_CUDA(cudaGetLastError());
    }
    {
        constexpr int kWarps = 8;
        const uint64_t want = (n + kWarps - 1) / kWarps;
        const uint64_t cap = static_cast<uint64_t>(c->sm_count) * 8;
        const uint32_t grid = static_cast<uint32_t>(want < cap ? want : cap);
        nvrx::crcx_fold<kWarps><<<grid, kWarps * 32, 0, st>>>(src, reinterpret_cast<const CrcxExtent*>(c->d_mem),
                                                              static_cast<uint32_t>(n), vals, pow2, crcs);
        NVRX_CUDA(cudaGetLastError());
    }
    NVRX_CUDA(cudaMemcpyAsync(host_crcs, crcs, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    return NVRX_OK;
}

uint32_t nvrx_crc32_combine(uint32_t crc_a, uint32_t crc_b, uint64_t len_b) {
    return nvrx::crc_zeros(pow2_tables(), crc_a, len_b) ^ crc_b;
}

// Operator tables for tooling and tests: which = 4, 16, 512 -> Z(which); 0 -> Z(chunk bytes).  `out` holds 1024 words.
int nvrx_crc_operator(uint32_t which, uint32_t* out) {
    if (!out) return NVRX_E_INVALID;
    const Ops& o = ops();
    const uint32_t* src = which == 4 ? o.z4 : which == 16 ? o.z16 : which == kCrcRowBytes ? o.z512 : which == 0 ? o.zchunk : nullptr;
    if (!src) return NVRX_E_INVALID;
    memcpy(out, src, sizeof(o.z4));
    return NVRX_OK;
}
