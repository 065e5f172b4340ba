// Shared host-side plumbing of libcpb200: handle, scratch workspace, error reporting.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/cpb200.h"

// A device allocation of the handle, grown on demand by cp_buffer_reserve.
struct cp_buffer {
    void *ptr;
    size_t bytes;
};

// Makes `buf` hold at least `need` bytes.  A larger block replaces the old one (cudaFree synchronises the device, so no
// kernel in flight still uses it), with need / slack_div bytes of slack, rounded up to 1 MiB.  `what` starts the error
// message.
int cp_buffer_reserve(cp_buffer &buf, size_t need, size_t slack_div, const char *what);

// The Cholesky factor kept between cp_ls_factor / cp_ls_solve and cp_ls_resolve (ls.cu).  It has its own allocation
// because every entry point reuses the scratch `ws`.
struct cp_kept_factor {
    cp_buffer buf;
    int K, Kfull;  // K == 0: the handle holds no factor
    int64_t N;
    int rows;      // rows of L stored in `buf` (K, or K + n when right-hand sides rode along)
};

// cp_create zero-initialises every field (new cp_handle_s()) and sets device and num_sms.
struct cp_handle_s {
    int device;
    int num_sms;
    cp_buffer ws;      // scratch
    void *tmap_encode; // cuTensorMapEncodeTiled entry point (resolved lazily)
    // look-ahead of the blocked Cholesky (ls.cu): low-priority side stream + fork/join events, created lazily
    cudaStream_t side;   // urgent look-ahead: the updates the chain will need within the next few panels
    cudaStream_t bulk;   // the rest of every pair's trailing update (long kernels with slack): never ahead of `side` work
    cudaEvent_t ev_panel, ev_side, ev_bulk;
    cp_kept_factor fac;
    // second scratch: temporaries of an entry point that calls another one (cp_ls_residual -> cp_gram), which
    // carves its own scratch out of `ws`
    cp_buffer aux;
    // cp_gram_profile: CUDA events around the tensor-core GEMM kernel of cp_gram (bench.py's roofline of that kernel)
    bool gram_profile;
    cudaEvent_t ev_gram0, ev_gram1;
    // tensor-core (split-precision) bulk products of the least-squares solver (gemm_tc.cu): on/off per handle
    // (cp_ls_tensor_cores) and one operand buffer per stream the solver issues work on (caller's, side, bulk)
    bool ls_tc;
    cp_buffer tcbuf[3];
};

// Entry points run on the handle's device whatever the caller's current device is (restored on return).
struct cp_device_guard {
    int prev;
    bool ok;
    explicit cp_device_guard(int dev) : prev(-1), ok(true) {
        int cur = -1;
        ok = cudaGetDevice(&cur) == cudaSuccess;
        if (ok && cur != dev) {
            ok = cudaSetDevice(dev) == cudaSuccess;
            if (ok) prev = cur;
        }
    }
    ~cp_device_guard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};
#define CP_DEVICE_GUARD(h)                                                             \
    cp_device_guard guard__((h)->device);                                              \
    if (!guard__.ok) CP_FAIL(CP_ERR_CUDA, "cannot switch to device %d of the handle", (h)->device)

// cudaFuncSetAttribute is per DEVICE: one flag per device ordinal for every kernel that opts into large shared memory
constexpr int CP_MAX_DEVICES = 64;
struct cp_per_device_flag {
    bool done[CP_MAX_DEVICES] = {};
    bool *slot() {
        int cur = 0;
        cudaGetDevice(&cur);
        return &done[cur >= 0 && cur < CP_MAX_DEVICES ? cur : 0];
    }
};

extern thread_local char cp_err_buf[512];

#define CP_FAIL(code, ...)                                  \
    do {                                                    \
        snprintf(cp_err_buf, sizeof(cp_err_buf), __VA_ARGS__); \
        return (code);                                      \
    } while (0)

#define CP_CUDA(call)                                                                         \
    do {                                                                                      \
        cudaError_t e__ = (call);                                                             \
        if (e__ != cudaSuccess)                                                               \
            CP_FAIL(CP_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
    } while (0)

// every kernel launch of the library goes through one of these two, so the counter is exact
#include <atomic>
extern std::atomic<unsigned long long> cp_launch_counter;
#define CP_CHECK_LAUNCH()                                             \
    do {                                                              \
        cp_launch_counter.fetch_add(1, std::memory_order_relaxed);    \
        CP_CUDA(cudaGetLastError());                                  \
    } while (0)
#define CP_GEMM_LAUNCH(call)                                          \
    do {                                                              \
        cp_launch_counter.fetch_add(1, std::memory_order_relaxed);    \
        CP_CUDA((call));                                              \
    } while (0)

#define CP_REQUIRE(cond, ...)                         \
    do {                                              \
        if (!(cond)) CP_FAIL(CP_ERR_INVALID, __VA_ARGS__); \
    } while (0)

// Returns scratch of at least `bytes` (256-byte aligned); grows (synchronising) if needed.
int cp_ws_reserve(cp_handle_t h, size_t bytes, void **out);
int cp_aux_reserve(cp_handle_t h, size_t bytes, void **out);

static inline size_t cp_align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
static inline int cp_cdiv(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }
static inline bool cp_aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

// Carves aligned sub-buffers out of one reservation.
struct cp_carver {
    char *base;
    size_t off;
    explicit cp_carver(void *b) : base((char *)b), off(0) {}
    template <typename T>
    T *take(size_t count) {
        T *p = (T *)(base + off);
        off += cp_align_up(count * sizeof(T), 256);
        return p;
    }
    static size_t need(size_t count, size_t elt) { return cp_align_up(count * elt, 256); }
};
