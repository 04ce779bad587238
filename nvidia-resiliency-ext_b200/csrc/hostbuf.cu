// hostbuf.cu -- host snapshot buffers of the C ABI: one POSIX shared-memory mapping per snapshot slot,
// page-locked for DMA, followed by CPU-only processes through a progress word in its header page.
//
// Layout of the shm object:  [ header page, 4096 B ][ payload, capacity B ]
// The header page starts with a ZIP local file header (see write_slot_prefix) and carries the Header struct at byte 128.
#include <cuda_runtime.h>
#include <ctype.h>
#include <errno.h>
#include <fcntl.h>
#include <sched.h>
#include <stdio.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <time.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <new>
#include <string>
#include <thread>
#include <vector>

#include "nvrx_snap.h"
#include "host_numa.h"

extern "C" size_t nvrx_crc32_fold(uint32_t* crc, const uint8_t* p, size_t n);  // crc32_fold.cpp (not part of the ABI)

namespace {

constexpr uint64_t kHeaderBytes = 4096;
constexpr uint64_t kMagic = 0x4e56525842323030ull;  // "NVRXB200"

struct Header {
    uint64_t magic;
    uint64_t capacity;
    uint8_t pad0[48];
    volatile uint64_t progress;  // own cache line: advanced by stream-ordered GPU writes
    uint8_t pad1[56];
};
static_assert(sizeof(Header) == 128, "header layout");
constexpr uint64_t kHeaderOff = 128;  // where the Header struct sits inside the header page

inline Header* header_of(uint8_t* map) { return reinterpret_cast<Header*>(map + kHeaderOff); }

void put16(uint8_t* p, uint16_t v) {
    p[0] = static_cast<uint8_t>(v);
    p[1] = static_cast<uint8_t>(v >> 8);
}
void put32(uint8_t* p, uint32_t v) {
    put16(p, static_cast<uint16_t>(v));
    put16(p + 2, static_cast<uint16_t>(v >> 16));
}

// The header page doubles as a ZIP local file header: an empty stored record named ".nvrx_slot" whose *extra field* spans
// the rest of the page (and so contains the Header struct).  A slot whose payload was packed in checkpoint-container
// geometry (checkpointing/b200/ptzip.py) can then be published as a torch.load-able file by writing the container's tail and
// adding a hard link to the shm object -- torch.load insists on "PK\3\4" as the first four bytes of a checkpoint.  The
// record is not listed in any central directory; readers that walk local headers see a zero-length file.
void write_slot_prefix(uint8_t* page) {
    static const char name[] = ".nvrx_slot";
    const uint16_t name_len = static_cast<uint16_t>(sizeof(name) - 1);
    const uint16_t extra_len = static_cast<uint16_t>(kHeaderBytes - 30 - name_len);
    put32(page + 0, 0x04034b50u);  // local file header signature
    put16(page + 4, 20);           // version needed
    put16(page + 6, 0);            // flags
    put16(page + 8, 0);            // method: stored
    put16(page + 10, 0);           // time
    put16(page + 12, 0x21);        // date 1980-01-01
    put32(page + 14, 0);           // crc32 of no bytes
    put32(page + 18, 0);           // compressed size
    put32(page + 22, 0);           // uncompressed size
    put16(page + 26, name_len);
    put16(page + 28, extra_len);
    memcpy(page + 30, name, name_len);
    put16(page + 30 + name_len, 0x4246);  // "FB": the extra-field id PyTorch uses for alignment padding
    put16(page + 32 + name_len, static_cast<uint16_t>(extra_len - 4));
    static_assert(30 + sizeof(name) - 1 + 4 <= kHeaderOff, "zip prefix must end before the Header struct");
}

void prefault(uint8_t* base, uint64_t bytes, int threads, const cpu_set_t* cpus) {
    if (threads < 1) threads = 1;
    const uint64_t page = 4096;
    const uint64_t per = ((bytes / threads) + page - 1) / page * page;
    std::vector<std::thread> pool;
    for (int t = 0; t < threads; ++t) {
        const uint64_t lo = std::min<uint64_t>(bytes, per * t), hi = std::min<uint64_t>(bytes, per * (t + 1));
        if (lo >= hi) break;
        pool.emplace_back([=] {
            if (cpus) sched_setaffinity(0, sizeof(cpu_set_t), cpus);  // this thread only; it exits after touching
            for (uint64_t o = lo; o < hi; o += page) base[o] = 0;
        });
    }
    for (auto& th : pool) th.join();
}

// ---- crc32 (reflected polynomial 0xEDB88320, zlib-compatible), slice-by-8 -------------------------
uint32_t g_tab[8][256];
std::atomic<int> g_tab_ready{0};

void crc_init() {
    if (g_tab_ready.load(std::memory_order_acquire)) return;
    static std::atomic<int> lock{0};
    int expected = 0;
    if (lock.compare_exchange_strong(expected, 1)) {
        for (uint32_t i = 0; i < 256; ++i) {
            uint32_t c = i;
            for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ 0xEDB88320u : c >> 1;
            g_tab[0][i] = c;
        }
        for (uint32_t i = 0; i < 256; ++i)
            for (int s = 1; s < 8; ++s) g_tab[s][i] = (g_tab[s - 1][i] >> 8) ^ g_tab[0][g_tab[s - 1][i] & 0xff];
        g_tab_ready.store(1, std::memory_order_release);
    } else {
        while (!g_tab_ready.load(std::memory_order_acquire)) {
        }
    }
}

uint32_t crc_update(uint32_t crc, const uint8_t* p, uint64_t n) {
    crc = ~crc;
    {  // carry-less-multiply folding for the bulk (crc32_fold.cpp); the table loop below takes what is left (< 64 B + tail)
        const size_t took = nvrx_crc32_fold(&crc, p, static_cast<size_t>(n));
        p += took;
        n -= took;
    }
    while (n && (reinterpret_cast<uintptr_t>(p) & 7u)) {
        crc = (crc >> 8) ^ g_tab[0][(crc ^ *p++) & 0xff];
        --n;
    }
    while (n >= 8) {
        uint64_t v;
        memcpy(&v, p, 8);
        v ^= crc;
        crc = g_tab[7][v & 0xff] ^ g_tab[6][(v >> 8) & 0xff] ^ g_tab[5][(v >> 16) & 0xff] ^ g_tab[4][(v >> 24) & 0xff] ^
              g_tab[3][(v >> 32) & 0xff] ^ g_tab[2][(v >> 40) & 0xff] ^ g_tab[1][(v >> 48) & 0xff] ^ g_tab[0][v >> 56];
        p += 8;
        n -= 8;
    }
    while (n--) crc = (crc >> 8) ^ g_tab[0][(crc ^ *p++) & 0xff];
    return ~crc;
}

// crc(A||B) from crc(A), crc(B), len(B): multiply crc(A) by x^(8*lenB) in GF(2)[x]/P via square-and-multiply
// on 32x32 bit matrices.
uint32_t mat_times(const uint32_t* mat, uint32_t vec) {
    uint32_t sum = 0;
    for (int i = 0; vec; ++i, vec >>= 1)
        if (vec & 1) sum ^= mat[i];
    return sum;
}
void mat_square(uint32_t* sq, const uint32_t* mat) {
    for (int i = 0; i < 32; ++i) sq[i] = mat_times(mat, mat[i]);
}
uint32_t crc_combine(uint32_t crc1, uint32_t crc2, uint64_t len2) {
    if (len2 == 0) return crc1;
    uint32_t even[32], odd[32];
    odd[0] = 0xEDB88320u;  // operator for one zero bit
    uint32_t row = 1;
    for (int i = 1; i < 32; ++i) {
        odd[i] = row;
        row <<= 1;
    }
    mat_square(even, odd);  // two zero bits
    mat_square(odd, even);  // four zero bits
    do {
        mat_square(even, odd);  // first pass: one zero byte
        if (len2 & 1) crc1 = mat_times(even, crc1);
        len2 >>= 1;
        if (!len2) break;
        mat_square(odd, even);
        if (len2 & 1) crc1 = mat_times(odd, crc1);
        len2 >>= 1;
    } while (len2);
    return crc1 ^ crc2;
}

}  // namespace

struct nvrx_hostbuf {
    uint8_t* map = nullptr;  // header page + payload
    uint64_t map_bytes = 0;
    uint64_t capacity = 0;
    bool pinned = false;
    bool owner = false;
    int device = 0;
    std::string name;
};

extern "C" {

int nvrx_hostbuf_create(const char* shm_name, uint64_t bytes, int prefault_threads, int pin, int device,
                        nvrx_hostbuf** out) {
    if (!out) return NVRX_E_INVALID;
    const uint64_t cap = (bytes + 4095) / 4096 * 4096;
    const uint64_t total = kHeaderBytes + std::max<uint64_t>(cap, 4096);
    void* m = MAP_FAILED;
    if (shm_name && shm_name[0]) {
        int fd = shm_open(shm_name, O_CREAT | O_EXCL | O_RDWR, 0600);
        if (fd < 0) return NVRX_E_SYS;
        if (ftruncate(fd, static_cast<off_t>(total)) != 0) {
            close(fd);
            shm_unlink(shm_name);
            return NVRX_E_SYS;
        }
        m = mmap(nullptr, total, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
        close(fd);
        if (m == MAP_FAILED) {
            shm_unlink(shm_name);
            return NVRX_E_SYS;
        }
    } else {
        m = mmap(nullptr, total, PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
        if (m == MAP_FAILED) return NVRX_E_SYS;
    }
    nvrx_hostbuf* hb = new (std::nothrow) nvrx_hostbuf();
    if (!hb) {
        munmap(m, total);
        if (shm_name && shm_name[0]) shm_unlink(shm_name);
        return NVRX_E_NOMEM;
    }
    hb->map = static_cast<uint8_t*>(m);
    hb->map_bytes = total;
    hb->capacity = total - kHeaderBytes;
    hb->owner = true;
    hb->device = device;
    if (shm_name) hb->name = shm_name;
    if (prefault_threads > 0) {
        cpu_set_t cpus;
        const bool local = pin && !getenv("NVRX_B200_NO_NUMA") && nvrx::numa_cpus_of_device(device, &cpus);
        prefault(hb->map, total, prefault_threads, local ? &cpus : nullptr);
    }
    write_slot_prefix(hb->map);
    Header* h = header_of(hb->map);
    h->magic = kMagic;
    h->capacity = hb->capacity;
    h->progress = 0;
    if (pin) {
        int prev = -1;
        cudaGetDevice(&prev);
        if (prev != device) cudaSetDevice(device);
        cudaError_t e = cudaHostRegister(hb->map, total, cudaHostRegisterPortable | cudaHostRegisterMapped);
        if (prev >= 0 && prev != device) cudaSetDevice(prev);
        if (e != cudaSuccess) {
            nvrx_hostbuf_destroy(hb, 1);
            return static_cast<int>(e);
        }
        hb->pinned = true;
    }
    *out = hb;
    return NVRX_OK;
}

int nvrx_hostbuf_open(const char* shm_name, nvrx_hostbuf** out) {
    if (!out || !shm_name || !shm_name[0]) return NVRX_E_INVALID;
    int fd = shm_open(shm_name, O_RDWR, 0600);
    if (fd < 0) return NVRX_E_SYS;
    struct stat st;
    if (fstat(fd, &st) != 0 || static_cast<uint64_t>(st.st_size) < kHeaderBytes + 4096) {
        close(fd);
        return NVRX_E_SYS;
    }
    const uint64_t total = static_cast<uint64_t>(st.st_size);
    void* m = mmap(nullptr, total, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    close(fd);
    if (m == MAP_FAILED) return NVRX_E_SYS;
    const Header* h = header_of(static_cast<uint8_t*>(m));
    if (h->magic != kMagic || h->capacity != total - kHeaderBytes) {
        munmap(m, total);
        return NVRX_E_STATE;
    }
    nvrx_hostbuf* hb = new (std::nothrow) nvrx_hostbuf();
    if (!hb) {
        munmap(m, total);
        return NVRX_E_NOMEM;
    }
    hb->map = static_cast<uint8_t*>(m);
    hb->map_bytes = total;
    hb->capacity = total - kHeaderBytes;
    hb->name = shm_name;
    *out = hb;
    return NVRX_OK;
}

int nvrx_hostbuf_destroy(nvrx_hostbuf* hb, int unlink_name) {
    if (!hb) return NVRX_OK;
    int rc = NVRX_OK;
    if (hb->pinned) {
        cudaError_t e = cudaHostUnregister(hb->map);
        if (e != cudaSuccess) rc = static_cast<int>(e);
    }
    if (hb->map) munmap(hb->map, hb->map_bytes);
    if (unlink_name && !hb->name.empty()) shm_unlink(hb->name.c_str());
    delete hb;
    return rc;
}

void* nvrx_hostbuf_data(nvrx_hostbuf* hb) { return hb ? hb->map + kHeaderBytes : nullptr; }

uint64_t nvrx_hostbuf_capacity(const nvrx_hostbuf* hb) { return hb ? hb->capacity : 0; }

volatile uint64_t* nvrx_hostbuf_progress(nvrx_hostbuf* hb) {
    return hb ? &header_of(hb->map)->progress : nullptr;
}

int nvrx_hostbuf_wait(nvrx_hostbuf* hb, uint64_t value, int64_t timeout_ms) {
    if (!hb) return NVRX_E_INVALID;
    volatile uint64_t* prog = nvrx_hostbuf_progress(hb);
    struct timespec t0;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    uint64_t spins = 0;
    while (true) {
        if (__atomic_load_n(prog, __ATOMIC_ACQUIRE) >= value) return NVRX_OK;
        if (++spins > 2000) {
            struct timespec nap = {0, 200000};  // 0.2 ms
            nanosleep(&nap, nullptr);
        }
        if (timeout_ms >= 0 && (spins & 63) == 0) {
            struct timespec t1;
            clock_gettime(CLOCK_MONOTONIC, &t1);
            const int64_t ms = (t1.tv_sec - t0.tv_sec) * 1000 + (t1.tv_nsec - t0.tv_nsec) / 1000000;
            if (ms > timeout_ms) return NVRX_E_STATE;
        }
    }
}

int nvrx_hostbuf_writev_fd(nvrx_hostbuf* hb, int64_t n, const uint64_t* offsets, const uint64_t* nbytes, const uint64_t* file_offs,
                           int fd, int threads) {
    if (!hb || fd < 0 || n < 0 || (n > 0 && (!offsets || !nbytes || !file_offs))) return NVRX_E_INVALID;
    for (int64_t i = 0; i < n; ++i)
        if (offsets[i] > hb->capacity || nbytes[i] > hb->capacity - offsets[i]) return NVRX_E_INVALID;
    if (threads < 1) threads = 1;
    const uint8_t* base = hb->map + kHeaderBytes;
    const uint64_t grain = 8ull << 20;
    // work items: (extent, piece) pairs handed out through one atomic cursor over the piece prefix sums
    std::vector<uint64_t> first_piece(static_cast<size_t>(n) + 1, 0);
    for (int64_t i = 0; i < n; ++i) first_piece[i + 1] = first_piece[i] + (nbytes[i] + grain - 1) / grain;
    const uint64_t total_pieces = first_piece[n];
    if (total_pieces == 0) return NVRX_OK;
    // Preferred path: map the destination range and memcpy into it.  pwrite() on tmpfs takes the inode lock, so N
    // writers to ONE file serialise (measured 3.6 GB/s with 16 threads); page faults on a shared mapping do not.
    uint64_t lo = UINT64_MAX, hi = 0;
    for (int64_t i = 0; i < n; ++i) {
        if (!nbytes[i]) continue;
        lo = std::min(lo, file_offs[i]);
        hi = std::max(hi, file_offs[i] + nbytes[i]);
    }
    const uint64_t map_lo = lo & ~uint64_t(4095);
    uint8_t* mapped = nullptr;
    bool may_map = !getenv("NVRX_B200_WRITE_PWRITE");
    if (!getenv("NVRX_B200_NO_FALLOCATE")) {
        // Allocate the destination range up front.  (1) A store into a mapping of a sparse file that the file system cannot
        // back (ENOSPC on the local SSD, tmpfs size limit, cgroup memory limit) is a SIGBUS that kills the writer with no
        // message; posix_fallocate reports the same condition as an errno.  (2) One in-kernel allocation pass is cheaper than
        // one page fault per 4 KiB from 16 threads (measurably faster for a fresh 16 GB /dev/shm file).
        const int rc = posix_fallocate(fd, static_cast<off_t>(map_lo), static_cast<off_t>(hi - map_lo));
        if (rc == EOPNOTSUPP || rc == EINVAL || rc == ENOSYS) {
            may_map = false;  // cannot pre-allocate here: use pwrite, whose errors are errnos as well
        } else if (rc != 0) {
            errno = rc;
            return NVRX_E_SYS;
        }
    }
    if (may_map) {
        void* m = mmap(nullptr, hi - map_lo, PROT_READ | PROT_WRITE, MAP_SHARED, fd, static_cast<off_t>(map_lo));
        if (m != MAP_FAILED) mapped = static_cast<uint8_t*>(m);
    }
    std::atomic<uint64_t> next{0};
    std::atomic<int> err{0};
    auto worker = [&] {
        int64_t ext = 0;
        while (!err.load(std::memory_order_relaxed)) {
            const uint64_t piece = next.fetch_add(1);
            if (piece >= total_pieces) break;
            while (first_piece[ext + 1] <= piece) ++ext;  // pieces are handed out in increasing order per thread
            const uint64_t o = (piece - first_piece[ext]) * grain;
            uint64_t len = std::min<uint64_t>(grain, nbytes[ext] - o), done = 0;
            if (mapped) {
                memcpy(mapped + (file_offs[ext] - map_lo) + o, base + offsets[ext] + o, len);
                continue;
            }
            while (done < len) {
                ssize_t w = pwrite(fd, base + offsets[ext] + o + done, len - done, static_cast<off_t>(file_offs[ext] + o + done));
                if (w < 0) {
                    if (errno == EINTR) continue;
                    err.store(errno ? errno : EIO);
                    return;
                }
                done += static_cast<uint64_t>(w);
            }
        }
    };
    const int nthreads = static_cast<int>(std::min<uint64_t>(static_cast<uint64_t>(threads), total_pieces));
    std::vector<std::thread> pool;
    for (int t = 1; t < nthreads; ++t) pool.emplace_back(worker);
    worker();
    for (auto& th : pool) th.join();
    if (mapped) munmap(mapped, hi - map_lo);
    if (err.load()) {
        errno = err.load();
        return NVRX_E_SYS;
    }
    return NVRX_OK;
}

int nvrx_hostbuf_write_fd(nvrx_hostbuf* hb, uint64_t offset, uint64_t bytes, int fd, uint64_t file_off, int threads) {
    return nvrx_hostbuf_writev_fd(hb, 1, &offset, &bytes, &file_off, fd, threads);
}

// Mirror of writev_fd for restore: file ranges -> payload with `threads` pread workers.  Reading through the page cache copies
// without faulting the source in page by page, which is what bounds a memcpy from an mmap of the checkpoint file.
int nvrx_hostbuf_readv_fd(nvrx_hostbuf* hb, int64_t n, const uint64_t* offsets, const uint64_t* nbytes, const uint64_t* file_offs,
                          int fd, int threads) {
    if (!hb || fd < 0 || n < 0 || (n > 0 && (!offsets || !nbytes || !file_offs))) return NVRX_E_INVALID;
    for (int64_t i = 0; i < n; ++i)
        if (offsets[i] > hb->capacity || nbytes[i] > hb->capacity - offsets[i]) return NVRX_E_INVALID;
    if (threads < 1) threads = 1;
    uint8_t* base = hb->map + kHeaderBytes;
    const uint64_t grain = 8ull << 20;
    std::vector<uint64_t> first_piece(static_cast<size_t>(n) + 1, 0);
    for (int64_t i = 0; i < n; ++i) first_piece[i + 1] = first_piece[i] + (nbytes[i] + grain - 1) / grain;
    const uint64_t total_pieces = first_piece[n];
    if (total_pieces == 0) return NVRX_OK;
    std::atomic<uint64_t> next{0};
    std::atomic<int> err{0};
    auto worker = [&] {
        int64_t ext = 0;
        while (!err.load(std::memory_order_relaxed)) {
            const uint64_t piece = next.fetch_add(1);
            if (piece >= total_pieces) break;
            while (first_piece[ext + 1] <= piece) ++ext;
            const uint64_t o = (piece - first_piece[ext]) * grain;
            const uint64_t len = std::min<uint64_t>(grain, nbytes[ext] - o);
            uint64_t done = 0;
            while (done < len) {
                ssize_t r = pread(fd, base + offsets[ext] + o + done, len - done, static_cast<off_t>(file_offs[ext] + o + done));
                if (r < 0 && errno == EINTR) continue;
                if (r <= 0) {  // error, or the file is shorter than the caller said
                    err.store(r < 0 && errno ? errno : EIO);
                    return;
                }
                done += static_cast<uint64_t>(r);
            }
        }
    };
    const int nthreads = static_cast<int>(std::min<uint64_t>(static_cast<uint64_t>(threads), total_pieces));
    std::vector<std::thread> pool;
    for (int t = 1; t < nthreads; ++t) pool.emplace_back(worker);
    worker();
    for (auto& th : pool) th.join();
    if (err.load()) {
        errno = err.load();
        return NVRX_E_SYS;
    }
    return NVRX_OK;
}

int nvrx_hostbuf_gather(nvrx_hostbuf* hb, int64_t n, const void* const* srcs, const uint64_t* nbytes, const uint64_t* dst_offsets,
                        int threads) {
    if (!hb || n < 0 || (n > 0 && (!srcs || !nbytes || !dst_offsets))) return NVRX_E_INVALID;
    for (int64_t i = 0; i < n; ++i) {
        if (dst_offsets[i] > hb->capacity || nbytes[i] > hb->capacity - dst_offsets[i]) return NVRX_E_INVALID;
        if (nbytes[i] && !srcs[i]) return NVRX_E_INVALID;
    }
    if (threads < 1) threads = 1;
    uint8_t* base = hb->map + kHeaderBytes;
    const uint64_t grain = 4ull << 20;
    std::vector<uint64_t> first_piece(static_cast<size_t>(n) + 1, 0);
    for (int64_t i = 0; i < n; ++i) first_piece[i + 1] = first_piece[i] + (nbytes[i] + grain - 1) / grain;
    const uint64_t total_pieces = first_piece[n];
    if (total_pieces == 0) return NVRX_OK;
    std::atomic<uint64_t> next{0};
    auto worker = [&] {
        int64_t ext = 0;
        while (true) {
            const uint64_t piece = next.fetch_add(1);
            if (piece >= total_pieces) break;
            while (first_piece[ext + 1] <= piece) ++ext;
            const uint64_t o = (piece - first_piece[ext]) * grain;
            const uint64_t len = std::min<uint64_t>(grain, nbytes[ext] - o);
            memcpy(base + dst_offsets[ext] + o, static_cast<const uint8_t*>(srcs[ext]) + o, len);
        }
    };
    const int nthreads = static_cast<int>(std::min<uint64_t>(static_cast<uint64_t>(threads), total_pieces));
    std::vector<std::thread> pool;
    for (int t = 1; t < nthreads; ++t) pool.emplace_back(worker);
    worker();
    for (auto& th : pool) th.join();
    return NVRX_OK;
}

int nvrx_hostbuf_crc32(nvrx_hostbuf* hb, uint64_t offset, uint64_t bytes, int threads, uint32_t* out) {
    if (!hb || !out || offset > hb->capacity || bytes > hb->capacity - offset) return NVRX_E_INVALID;
    crc_init();
    const uint8_t* base = hb->map + kHeaderBytes + offset;
    if (threads < 1) threads = 1;
    const uint64_t min_part = 1ull << 20;
    uint64_t parts = std::min<uint64_t>(static_cast<uint64_t>(threads), std::max<uint64_t>(1, bytes / min_part));
    const uint64_t per = (bytes + parts - 1) / parts;
    std::vector<uint32_t> crcs(parts, 0);
    std::vector<uint64_t> lens(parts, 0);
    std::vector<std::thread> pool;
    for (uint64_t t = 0; t < parts; ++t) {
        const uint64_t lo = std::min(bytes, per * t), hi = std::min(bytes, per * (t + 1));
        lens[t] = hi - lo;
        auto job = [&, t, lo, hi] { crcs[t] = crc_update(0, base + lo, hi - lo); };
        if (t + 1 < parts) pool.emplace_back(job);
        else job();
    }
    for (auto& th : pool) th.join();
    uint32_t crc = crcs[0];
    for (uint64_t t = 1; t < parts; ++t) crc = crc_combine(crc, crcs[t], lens[t]);
    *out = crc;
    return NVRX_OK;
}

// crc32 of n extents of the payload at once: pieces of 4 MiB are summed by `threads` workers (across and inside extents) and
// chained per extent -- one call for the ~1500 records of a checkpoint instead of one thread pool per record.
int nvrx_hostbuf_crc32v(nvrx_hostbuf* hb, int64_t n, const uint64_t* offsets, const uint64_t* nbytes, int threads, uint32_t* out) {
    if (!hb || n < 0 || (n > 0 && (!offsets || !nbytes || !out))) return NVRX_E_INVALID;
    for (int64_t i = 0; i < n; ++i)
        if (offsets[i] > hb->capacity || nbytes[i] > hb->capacity - offsets[i]) return NVRX_E_INVALID;
    if (n == 0) return NVRX_OK;
    crc_init();
    if (threads < 1) threads = 1;
    const uint8_t* base = hb->map + kHeaderBytes;
    const uint64_t grain = 4ull << 20;
    std::vector<uint64_t> first_piece;
    std::vector<uint32_t> part;
    try {
        first_piece.assign(static_cast<size_t>(n) + 1, 0);
        for (int64_t i = 0; i < n; ++i) first_piece[i + 1] = first_piece[i] + (nbytes[i] + grain - 1) / grain;
        part.assign(first_piece[n], 0);
    } catch (const std::bad_alloc&) {
        return NVRX_E_NOMEM;
    }
    const uint64_t total_pieces = first_piece[n];
    std::atomic<uint64_t> next{0};
    auto worker = [&] {
        int64_t ext = 0;
        while (true) {
            const uint64_t piece = next.fetch_add(1);
            if (piece >= total_pieces) break;
            while (first_piece[ext + 1] <= piece) ++ext;
            const uint64_t o = (piece - first_piece[ext]) * grain;
            part[piece] = crc_update(0, base + offsets[ext] + o, std::min<uint64_t>(grain, nbytes[ext] - o));
        }
    };
    const int nthreads = static_cast<int>(std::min<uint64_t>(static_cast<uint64_t>(threads), std::max<uint64_t>(total_pieces, 1)));
    std::vector<std::thread> pool;
    for (int t = 1; t < nthreads; ++t) pool.emplace_back(worker);
    worker();
    for (auto& th : pool) th.join();
    for (int64_t i = 0; i < n; ++i) {
        uint32_t crc = 0;
        for (uint64_t pc = first_piece[i]; pc < first_piece[i + 1]; ++pc) {
            const uint64_t o = (pc - first_piece[i]) * grain;
            const uint64_t len = std::min<uint64_t>(grain, nbytes[i] - o);
            crc = (pc == first_piece[i]) ? part[pc] : crc_combine(crc, part[pc], len);
        }
        out[i] = crc;
    }
    return NVRX_OK;
}

}  // extern "C"
