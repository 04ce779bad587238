// restore_pipe.cu -- the host half of a restore as a pipeline: checkpoint file -> small pinned ring -> device staging.
//
// Mirror of nvrx_snapshot for the way back (reference: local/ckpt_managers/local_manager.py:91-105 `torch.load` reads the
// whole file through one thread into pageable memory, local/basic_state_dict.py:184-187 then issues one blocking H2D per
// tensor).  Here `threads` readers pread() the file ranges of the tensors straight into a ring of pinned chunks (no page
// faults on the source, no 16 GB slot to create and page-lock in a freshly restarted process) and the calling thread
// sends every chunk to the device with cudaMemcpyAsync as soon as its reads have landed, so the file read (page cache ->
// pinned) and the H2D overlap chunk by chunk.  Throughput = min(read rate of the pool, PCIe H2D).  The scatter kernel that
// follows (nvrx_scatter) reads only segment bytes, so the padding between segments is neither read nor defined.
#include <cuda_runtime.h>
#include <errno.h>
#include <sched.h>
#include <stdint.h>
#include <stdlib.h>
#include <time.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <mutex>
#include <new>
#include <thread>
#include <vector>

#include <sys/mman.h>

#include "nvrx_snap.h"
#include "host_numa.h"

#define NVRX_CUDA(expr)                                       \
    do {                                                      \
        cudaError_t e__ = (expr);                             \
        if (e__ != cudaSuccess) return static_cast<int>(e__); \
    } while (0)

namespace {

struct Ring {  // one per device, kept for the life of the process (page-locking is the expensive part)
    uint8_t* base = nullptr;
    bool have_cpus = false;  // CPUs of the NUMA node the GPU hangs off: readers run there, the ring was first touched there
    cpu_set_t cpus;
    uint64_t chunk = 0;
    int slots = 0;
    std::vector<cudaEvent_t> sent;  // H2D of the chunk that last used the slot
};
std::mutex g_ring_lock;
Ring g_rings[64];

int ring_for(int device, uint64_t chunk, int slots, Ring** out) {
    if (device < 0 || device >= 64) return NVRX_E_INVALID;
    Ring& r = g_rings[device];
    if (r.base && (r.chunk != chunk || r.slots != slots)) {
        for (cudaEvent_t ev : r.sent) cudaEventDestroy(ev);
        r.sent.clear();
        cudaHostUnregister(r.base);
        munmap(r.base, r.chunk * static_cast<uint64_t>(r.slots));
        r.base = nullptr;
    }
    if (!r.base) {
        // anonymous pages first touched from the CPUs next to the GPU (so the reads land in, and the H2D leaves from, the DRAM
        // behind the GPU's PCIe root port), then page-locked -- the same placement the snapshot slots get (hostbuf.cu)
        const uint64_t bytes = chunk * static_cast<uint64_t>(slots);
        void* p = mmap(nullptr, bytes, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
        if (p == MAP_FAILED) return NVRX_E_NOMEM;
        // writer processes are forked later: a private mapping would turn copy-on-write at fork(), the readers' pread() would
        // then land in fresh pages while the DMA mapping still points at the old ones (the H2D sends stale bytes).  No child
        // uses the ring, so it is not inherited at all.
        if (madvise(p, bytes, MADV_DONTFORK) != 0) {
            munmap(p, bytes);
            return NVRX_E_SYS;
        }
        r.have_cpus = !getenv("NVRX_B200_NO_NUMA") && nvrx::numa_cpus_of_device(device, &r.cpus);
        {
            uint8_t* b = static_cast<uint8_t*>(p);
            const bool bind = r.have_cpus;
            const cpu_set_t cpus = r.cpus;
            std::thread toucher([=] {
                if (bind) sched_setaffinity(0, sizeof(cpu_set_t), &cpus);
                for (uint64_t o = 0; o < bytes; o += 4096) b[o] = 0;
            });
            toucher.join();
        }
        cudaError_t e = cudaHostRegister(p, bytes, cudaHostRegisterPortable);
        if (e != cudaSuccess) {
            munmap(p, bytes);
            return static_cast<int>(e);
        }
        r.base = static_cast<uint8_t*>(p);
        r.chunk = chunk;
        r.slots = slots;
        for (int s = 0; s < slots; ++s) {
            cudaEvent_t ev;
            NVRX_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
            r.sent.push_back(ev);
        }
    }
    *out = &r;
    return NVRX_OK;
}

struct Piece {
    uint64_t file_off;
    uint64_t ring_off;  // inside the chunk's ring slot
    uint32_t len;
    uint32_t chunk;
};

inline void nap_us(long us) {
    struct timespec ts = {0, us * 1000};
    nanosleep(&ts, nullptr);
}

}  // namespace

extern "C" {

int nvrx_fill_from_fd(void* staging, uint64_t staging_bytes, int fd, int64_t n, const uint64_t* stg_offs,
                      const uint64_t* nbytes, const uint64_t* file_offs, uint64_t chunk_bytes, int ring_slots, int threads,
                      int device, void* stream) {
    if (fd < 0 || n < 0 || (n > 0 && (!stg_offs || !nbytes || !file_offs)) || (staging_bytes && !staging)) return NVRX_E_INVALID;
    if (chunk_bytes == 0) chunk_bytes = 64ull << 20;
    chunk_bytes = (chunk_bytes + 4095) / 4096 * 4096;
    if (ring_slots < 2) ring_slots = 4;
    if (threads < 1) threads = 1;
    uint64_t prev_end = 0;
    for (int64_t i = 0; i < n; ++i) {  // ascending, disjoint, inside staging
        if (stg_offs[i] < prev_end || nbytes[i] > staging_bytes || stg_offs[i] > staging_bytes - nbytes[i]) return NVRX_E_INVALID;
        prev_end = stg_offs[i] + nbytes[i];
    }
    if (prev_end == 0) return NVRX_OK;
    const uint64_t n_chunks = (prev_end + chunk_bytes - 1) / chunk_bytes;
    if (n_chunks > 0xffffffffull) return NVRX_E_INVALID;

    std::vector<Piece> pieces;
    std::vector<uint32_t> first_of_chunk, pieces_in_chunk;
    std::vector<uint64_t> chunk_lo, chunk_hi;  // byte range of the chunk that holds segment data (what the H2D sends)
    try {
        first_of_chunk.assign(n_chunks + 1, 0);
        pieces_in_chunk.assign(n_chunks, 0);
        chunk_lo.assign(n_chunks, UINT64_MAX);
        chunk_hi.assign(n_chunks, 0);
        const uint64_t grain = 4ull << 20;
        for (int64_t i = 0; i < n; ++i) {
            uint64_t o = 0;
            while (o < nbytes[i]) {
                const uint64_t pos = stg_offs[i] + o;
                const uint64_t c = pos / chunk_bytes;
                const uint64_t room = (c + 1) * chunk_bytes - pos;
                const uint64_t len = std::min<uint64_t>({grain, room, nbytes[i] - o});
                Piece p;
                p.file_off = file_offs[i] + o;
                p.ring_off = pos - c * chunk_bytes;
                p.len = static_cast<uint32_t>(len);
                p.chunk = static_cast<uint32_t>(c);
                pieces.push_back(p);  // extents ascend in staging order -> pieces ascend by chunk
                ++pieces_in_chunk[c];
                chunk_lo[c] = std::min(chunk_lo[c], pos);
                chunk_hi[c] = std::max(chunk_hi[c], pos + len);
                o += len;
            }
        }
        for (uint64_t c = 0; c < n_chunks; ++c) first_of_chunk[c + 1] = first_of_chunk[c] + pieces_in_chunk[c];
    } catch (const std::bad_alloc&) {
        return NVRX_E_NOMEM;
    }

    int prev_dev = -1;
    cudaGetDevice(&prev_dev);
    if (prev_dev != device) NVRX_CUDA(cudaSetDevice(device));
    std::lock_guard<std::mutex> guard(g_ring_lock);
    Ring* ring = nullptr;
    int rc = ring_for(device, chunk_bytes, ring_slots, &ring);
    if (rc) {
        if (prev_dev >= 0 && prev_dev != device) cudaSetDevice(prev_dev);
        return rc;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);

    std::vector<std::atomic<uint32_t>> remaining(n_chunks);
    for (uint64_t c = 0; c < n_chunks; ++c) remaining[c].store(pieces_in_chunk[c], std::memory_order_relaxed);
    std::atomic<uint64_t> next{0};
    std::atomic<uint64_t> readable{static_cast<uint64_t>(ring_slots)};  // chunks [0, readable) may be read into the ring
    std::atomic<int> err{0};
    const uint64_t total_pieces = pieces.size();

    auto reader = [&] {
        if (ring->have_cpus) sched_setaffinity(0, sizeof(cpu_set_t), &ring->cpus);  // this thread only; it ends with the call
        while (!err.load(std::memory_order_relaxed)) {
            const uint64_t i = next.fetch_add(1);
            if (i >= total_pieces) break;
            const Piece& p = pieces[i];
            uint32_t spins = 0;
            while (p.chunk >= readable.load(std::memory_order_acquire)) {  // the slot still feeds an earlier chunk's H2D
                if (err.load(std::memory_order_relaxed)) return;
                if (++spins > 200) nap_us(20);
            }
            uint8_t* dst = ring->base + (p.chunk % ring->slots) * ring->chunk + p.ring_off;
            uint64_t done = 0;
            while (done < p.len) {
                ssize_t r = pread(fd, dst + done, p.len - done, static_cast<off_t>(p.file_off + done));
                if (r < 0 && errno == EINTR) continue;
                if (r <= 0) {  // error, or the file is shorter than the caller said
                    err.store(r < 0 && errno ? errno : EIO);
                    return;
                }
                done += static_cast<uint64_t>(r);
            }
            remaining[p.chunk].fetch_sub(1, std::memory_order_release);
        }
    };
    const int nthreads = static_cast<int>(std::min<uint64_t>(static_cast<uint64_t>(threads), total_pieces));
    std::vector<std::thread> pool;
    for (int t = 0; t < nthreads; ++t) pool.emplace_back(reader);

    // the coordinator: chunk c goes to the device when its reads are in; its slot is free again when that copy is done
    uint64_t sent = 0, freed = 0;
    cudaError_t cerr = cudaSuccess;
    while (sent < n_chunks && !err.load() && cerr == cudaSuccess) {
        bool progressed = false;
        if (remaining[sent].load(std::memory_order_acquire) == 0) {
            if (pieces_in_chunk[sent]) {
                const uint64_t lo = chunk_lo[sent], hi = chunk_hi[sent];
                const uint8_t* src = ring->base + (sent % ring->slots) * ring->chunk + (lo - sent * chunk_bytes);
                cerr = cudaMemcpyAsync(static_cast<uint8_t*>(staging) + lo, src, hi - lo, cudaMemcpyHostToDevice, st);
            }
            if (cerr == cudaSuccess) cerr = cudaEventRecord(ring->sent[sent % ring->slots], st);
            ++sent;
            progressed = true;
        }
        while (freed < sent && cerr == cudaSuccess) {
            cudaError_t q = cudaEventQuery(ring->sent[freed % ring->slots]);
            if (q == cudaErrorNotReady) break;
            if (q != cudaSuccess) {
                cerr = q;
                break;
            }
            ++freed;
            readable.store(freed + ring->slots, std::memory_order_release);
            progressed = true;
        }
        if (!progressed) nap_us(20);
    }
    if (cerr != cudaSuccess) err.store(EIO);
    for (auto& th : pool) th.join();
    // the ring is reused by the next call: its last copies must have left it
    if (cerr == cudaSuccess && sent) cerr = cudaEventSynchronize(ring->sent[(sent - 1) % ring->slots]);
    if (prev_dev >= 0 && prev_dev != device) cudaSetDevice(prev_dev);
    if (cerr != cudaSuccess) return static_cast<int>(cerr);
    if (err.load()) {
        errno = err.load();
        return NVRX_E_SYS;
    }
    return NVRX_OK;
}

}  // extern "C"
