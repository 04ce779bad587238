// snap_runtime.cu -- stream/event/IPC helpers and the drain (device staging -> pinned host) of the C ABI.
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "nvrx_snap.h"

#define NVRX_CUDA(expr)                                       \
    do {                                                      \
        cudaError_t e__ = (expr);                             \
        if (e__ != cudaSuccess) return static_cast<int>(e__); \
    } while (0)

namespace {

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

// Driver entry points are resolved through the runtime so the library has no link-time dependency on
// libcuda.so.1 and still loads (and exports every symbol) on a machine without a driver.
typedef CUresult (*write64_fn)(CUstream, CUdeviceptr, cuuint64_t, unsigned int);
typedef CUresult (*wait64_fn)(CUstream, CUdeviceptr, cuuint64_t, unsigned int);

int resolve(const char* name, void** fn) {
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint(name, fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess) return static_cast<int>(e);
    if (qres != cudaDriverEntryPointSuccess || !*fn) return NVRX_E_NODRIVER;
    return NVRX_OK;
}

int driver_write64(cudaStream_t st, void* dev_addr, uint64_t value) {
    static write64_fn fn = nullptr;
    if (!fn) {
        void* f = nullptr;
        int rc = resolve("cuStreamWriteValue64", &f);
        if (rc) return rc;
        fn = reinterpret_cast<write64_fn>(f);
    }
    CUresult r = fn(st, reinterpret_cast<CUdeviceptr>(dev_addr), value, CU_STREAM_WRITE_VALUE_DEFAULT);
    return r == CUDA_SUCCESS ? NVRX_OK : static_cast<int>(cudaErrorUnknown);
}

int driver_wait64_geq(cudaStream_t st, void* dev_addr, uint64_t value) {
    static wait64_fn fn = nullptr;
    if (!fn) {
        void* f = nullptr;
        int rc = resolve("cuStreamWaitValue64", &f);
        if (rc) return rc;
        fn = reinterpret_cast<wait64_fn>(f);
    }
    CUresult r = fn(st, reinterpret_cast<CUdeviceptr>(dev_addr), value, CU_STREAM_WAIT_VALUE_GEQ);
    return r == CUDA_SUCCESS ? NVRX_OK : static_cast<int>(cudaErrorUnknown);
}

}  // namespace

extern "C" {

int nvrx_dev_alloc(int device, uint64_t bytes, void** out) {
    if (!out) return NVRX_E_INVALID;
    DeviceGuard guard(device);
    if (!guard.ok) return static_cast<int>(cudaErrorInvalidDevice);
    void* p = nullptr;
    NVRX_CUDA(cudaMalloc(&p, bytes ? bytes : 512));
    // The fill is over on return.  cudaMemset would only queue it on the legacy default stream, which the engine's
    // non-blocking streams do not wait for: a reduce into a parity buffer allocated mid-save raced with its zero-fill.
    cudaStream_t st = nullptr;
    cudaError_t e = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaMemsetAsync(p, 0, bytes ? bytes : 512, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (st) cudaStreamDestroy(st);
    if (e != cudaSuccess) {
        cudaFree(p);
        return static_cast<int>(e);
    }
    *out = p;
    return NVRX_OK;
}

int nvrx_dev_free(int device, void* ptr) {
    if (!ptr) return NVRX_OK;
    DeviceGuard guard(device);
    NVRX_CUDA(cudaFree(ptr));
    return NVRX_OK;
}

int nvrx_stream_create(int device, int high_priority, void** out) {
    if (!out) return NVRX_E_INVALID;
    DeviceGuard guard(device);
    if (!guard.ok) return static_cast<int>(cudaErrorInvalidDevice);
    int lo = 0, hi = 0;
    NVRX_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    cudaStream_t st;
    NVRX_CUDA(cudaStreamCreateWithPriority(&st, cudaStreamNonBlocking, high_priority ? hi : lo));
    *out = st;
    return NVRX_OK;
}

int nvrx_stream_destroy(void* stream) {
    if (!stream) return NVRX_OK;
    NVRX_CUDA(cudaStreamDestroy(static_cast<cudaStream_t>(stream)));
    return NVRX_OK;
}

int nvrx_event_create(int device, int timing, void** out) {
    if (!out) return NVRX_E_INVALID;
    DeviceGuard guard(device);
    if (!guard.ok) return static_cast<int>(cudaErrorInvalidDevice);
    cudaEvent_t ev;
    NVRX_CUDA(cudaEventCreateWithFlags(&ev, timing ? cudaEventDefault : cudaEventDisableTiming));
    *out = ev;
    return NVRX_OK;
}

int nvrx_event_destroy(void* event) {
    if (!event) return NVRX_OK;
    NVRX_CUDA(cudaEventDestroy(static_cast<cudaEvent_t>(event)));
    return NVRX_OK;
}

int nvrx_event_record(void* event, void* stream) {
    if (!event) return NVRX_E_INVALID;
    NVRX_CUDA(cudaEventRecord(static_cast<cudaEvent_t>(event), static_cast<cudaStream_t>(stream)));
    return NVRX_OK;
}

int nvrx_stream_wait_event(void* stream, void* event) {
    if (!event) return NVRX_E_INVALID;
    NVRX_CUDA(cudaStreamWaitEvent(static_cast<cudaStream_t>(stream), static_cast<cudaEvent_t>(event), 0));
    return NVRX_OK;
}

int nvrx_event_query(void* event, int* done) {
    if (!event || !done) return NVRX_E_INVALID;
    cudaError_t e = cudaEventQuery(static_cast<cudaEvent_t>(event));
    if (e == cudaSuccess) {
        *done = 1;
        return NVRX_OK;
    }
    if (e == cudaErrorNotReady) {
        *done = 0;
        return NVRX_OK;
    }
    return static_cast<int>(e);
}

int nvrx_event_sync(void* event) {
    if (!event) return NVRX_E_INVALID;
    NVRX_CUDA(cudaEventSynchronize(static_cast<cudaEvent_t>(event)));
    return NVRX_OK;
}

int nvrx_event_elapsed_ms(void* start, void* stop, float* ms) {
    if (!start || !stop || !ms) return NVRX_E_INVALID;
    NVRX_CUDA(cudaEventElapsedTime(ms, static_cast<cudaEvent_t>(start), static_cast<cudaEvent_t>(stop)));
    return NVRX_OK;
}

int nvrx_stream_sync(void* stream) {
    NVRX_CUDA(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
    return NVRX_OK;
}

int nvrx_ipc_export(void* dev_ptr, uint8_t handle_out[64]) {
    if (!dev_ptr || !handle_out) return NVRX_E_INVALID;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "ipc handle size");
    cudaIpcMemHandle_t h;
    NVRX_CUDA(cudaIpcGetMemHandle(&h, dev_ptr));
    memcpy(handle_out, &h, 64);
    return NVRX_OK;
}

int nvrx_ipc_import(int device, const uint8_t handle[64], void** out) {
    if (!handle || !out) return NVRX_E_INVALID;
    DeviceGuard guard(device);
    if (!guard.ok) return static_cast<int>(cudaErrorInvalidDevice);
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    void* p = nullptr;
    NVRX_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    *out = p;
    return NVRX_OK;
}

int nvrx_ipc_close(int device, void* imported) {
    if (!imported) return NVRX_OK;
    DeviceGuard guard(device);
    NVRX_CUDA(cudaIpcCloseMemHandle(imported));
    return NVRX_OK;
}

int nvrx_stream_write_u64(void* stream, void* addr, uint64_t value) {
    if (!addr) return NVRX_E_INVALID;
    return driver_write64(static_cast<cudaStream_t>(stream), addr, value);
}

int nvrx_stream_wait_u64_geq(void* stream, void* addr, uint64_t value) {
    if (!addr) return NVRX_E_INVALID;
    return driver_wait64_geq(static_cast<cudaStream_t>(stream), addr, value);
}

int nvrx_drain(void* host_dst, const void* staging, uint64_t bytes, uint64_t chunk_bytes, volatile uint64_t* progress,
               uint64_t base_value, void* stream, void* done_event) {
    if (bytes && (!host_dst || !staging)) return NVRX_E_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (chunk_bytes == 0 || chunk_bytes > bytes) chunk_bytes = bytes;
    void* prog_dev = nullptr;
    if (progress) {
        // registered (or cudaHostAlloc'ed) host memory: get the address the GPU writes through
        NVRX_CUDA(cudaHostGetDevicePointer(&prog_dev, const_cast<uint64_t*>(progress), 0));
    }
    uint64_t done = 0;
    while (done < bytes) {
        const uint64_t len = (bytes - done < chunk_bytes) ? bytes - done : chunk_bytes;
        NVRX_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(host_dst) + done, static_cast<const uint8_t*>(staging) + done, len,
                                  cudaMemcpyDeviceToHost, st));
        done += len;
        if (prog_dev) {
            int rc = driver_write64(st, prog_dev, base_value + done);
            if (rc) return rc;
        }
    }
    if (bytes == 0 && prog_dev) {
        int rc = driver_write64(st, prog_dev, base_value);
        if (rc) return rc;
    }
    if (done_event) NVRX_CUDA(cudaEventRecord(static_cast<cudaEvent_t>(done_event), st));
    return NVRX_OK;
}

int nvrx_fill(void* staging, const void* host_src, uint64_t bytes, uint64_t chunk_bytes, void* stream, void* done_event) {
    if (bytes && (!host_src || !staging)) return NVRX_E_INVALID;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (chunk_bytes == 0 || chunk_bytes > bytes) chunk_bytes = bytes;
    uint64_t done = 0;
    while (done < bytes) {
        const uint64_t len = (bytes - done < chunk_bytes) ? bytes - done : chunk_bytes;
        NVRX_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(staging) + done, static_cast<const uint8_t*>(host_src) + done, len,
                                  cudaMemcpyHostToDevice, st));
        done += len;
    }
    if (done_event) NVRX_CUDA(cudaEventRecord(static_cast<cudaEvent_t>(done_event), st));
    return NVRX_OK;
}

}  // extern "C"
