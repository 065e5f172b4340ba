// libcpb200: handle lifetime, version, error string.
#include "common.cuh"

thread_local char cp_err_buf[512] = "";
std::atomic<unsigned long long> cp_launch_counter{0};

extern "C" int64_t cp_launch_count(void) { return (int64_t)cp_launch_counter.load(std::memory_order_relaxed); }

extern "C" int cp_version(void) { return 200; }  // 0.2.0

extern "C" const char *cp_last_error(void) { return cp_err_buf; }

extern "C" int cp_create(cp_handle_t *out, int device) {
    CP_REQUIRE(out != nullptr, "cp_create: out is NULL");
    int ndev = 0;
    CP_CUDA(cudaGetDeviceCount(&ndev));
    CP_REQUIRE(device >= 0 && device < ndev, "cp_create: device %d out of range (%d visible)", device, ndev);
    cudaDeviceProp prop;
    CP_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        CP_FAIL(CP_ERR_CUDA, "cp_create: device %d is sm_%d%d; libcpb200 is built for sm_90a only", device,
                prop.major, prop.minor);
    cp_handle_s *h = new cp_handle_s();
    h->device = device;
    h->num_sms = prop.multiProcessorCount;
    *out = h;
    return CP_OK;
}

extern "C" int cp_destroy(cp_handle_t h) {
    if (!h) return CP_OK;
    cp_buffer *bufs[] = {&h->ws, &h->aux, &h->fac.buf, &h->tcbuf[0], &h->tcbuf[1], &h->tcbuf[2]};
    bool held = h->side || h->ev_gram0;
    for (cp_buffer *b : bufs) held = held || b->ptr;
    if (held) {
        int cur = 0;
        cudaGetDevice(&cur);
        cudaSetDevice(h->device);
        for (cp_buffer *b : bufs)
            if (b->ptr) cudaFree(b->ptr);
        if (h->ev_gram0) {
            cudaEventDestroy(h->ev_gram0);
            cudaEventDestroy(h->ev_gram1);
        }
        if (h->side) {
            cudaStreamDestroy(h->side);
            cudaStreamDestroy(h->bulk);
            cudaEventDestroy(h->ev_panel);
            cudaEventDestroy(h->ev_side);
            cudaEventDestroy(h->ev_bulk);
        }
        cudaSetDevice(cur);
    }
    delete h;
    return CP_OK;
}

extern "C" int cp_gram_profile(cp_handle_t h, int enable) {
    CP_REQUIRE(h != nullptr, "cp_gram_profile: NULL handle");
    CP_DEVICE_GUARD(h);
    if (enable && !h->ev_gram0) {
        CP_CUDA(cudaEventCreate(&h->ev_gram0));
        CP_CUDA(cudaEventCreate(&h->ev_gram1));
    }
    h->gram_profile = enable != 0;
    return CP_OK;
}

extern "C" int cp_ls_tensor_cores(cp_handle_t h, int enable) {
    CP_REQUIRE(h != nullptr, "cp_ls_tensor_cores: NULL handle");
    h->ls_tc = enable != 0;
    return CP_OK;
}

extern "C" int cp_gram_kernel_ms(cp_handle_t h, float *ms) {
    CP_REQUIRE(h != nullptr && ms != nullptr, "cp_gram_kernel_ms: NULL argument");
    CP_REQUIRE(h->gram_profile && h->ev_gram0, "cp_gram_kernel_ms: profiling is off (cp_gram_profile)");
    CP_DEVICE_GUARD(h);
    CP_CUDA(cudaEventSynchronize(h->ev_gram1));
    CP_CUDA(cudaEventElapsedTime(ms, h->ev_gram0, h->ev_gram1));
    return CP_OK;
}

extern "C" int64_t cp_workspace_bytes(cp_handle_t h) { return h ? (int64_t)h->ws.bytes : 0; }

int cp_buffer_reserve(cp_buffer &buf, size_t need, size_t slack_div, const char *what) {
    if (need <= buf.bytes) return CP_OK;
    if (buf.ptr) CP_CUDA(cudaFree(buf.ptr));
    buf = {};
    const size_t want = cp_align_up(need + need / slack_div, (size_t)1 << 20);
    cudaError_t e = cudaMalloc(&buf.ptr, want);
    if (e != cudaSuccess) {
        cudaGetLastError();
        CP_FAIL(CP_ERR_WORKSPACE, "%s of %zu bytes failed: %s", what, want, cudaGetErrorString(e));
    }
    buf.bytes = want;
    return CP_OK;
}

int cp_ws_reserve(cp_handle_t h, size_t bytes, void **out) {
    int rc = cp_buffer_reserve(h->ws, bytes, 8, "workspace allocation");
    if (rc) return rc;
    *out = h->ws.ptr;
    return CP_OK;
}

int cp_aux_reserve(cp_handle_t h, size_t bytes, void **out) {
    int rc = cp_buffer_reserve(h->aux, bytes, 8, "auxiliary workspace allocation");
    if (rc) return rc;
    *out = h->aux.ptr;
    return CP_OK;
}
