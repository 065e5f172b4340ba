// Grid size and pipeline depth of the NHWC host-map reader (csrc/gather_host.cu): conv3_2 and conv4_2 of VGG-16 at
// N = 5000, fp32 and bf16 maps in pinned host memory, every (CTAs, stages) pair timed with CUDA events, the pairs
// alternating over repetitions.  Every output is checked against the first configuration's, bit for bit.
//   make -C channel-pruning_b200/csrc
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o /tmp/host_nhwc_ctas profiles/host_nhwc_ctas.cu \
//        -Lchannel-pruning_b200 -lcpb200 -Xlinker -rpath=$PWD/channel-pruning_b200
//   /tmp/host_nhwc_ctas
#include <algorithm>
#include <random>
#include <vector>

#include "../channel-pruning_b200/csrc/gather_host.cu"

#define CK(x)                                                                            \
    do {                                                                                 \
        cudaError_t e_ = (x);                                                            \
        if (e_ != cudaSuccess) {                                                         \
            fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_));   \
            exit(1);                                                                     \
        }                                                                                \
    } while (0)

struct Layer {
    const char *name;
    int c, H;
};

template <int NS, typename T>
static float run(const T *map, const HostGeom &g0, int64_t rows, const int32_t *rx, const int32_t *ry, float *X,
                 int64_t ldx, int ncta, int launches) {
    HostGeom g;
    if (!host_geom(g, map, (int)sizeof(T), g0.B, g0.P, g0.c, 1, g0.H, g0.W, nullptr, g0.w, NS)) exit(2);
    cudaEvent_t a, b;
    CK(cudaEventCreate(&a));
    CK(cudaEventCreate(&b));
    CK(cudaEventRecord(a));
    for (int i = 0; i < launches; ++i) launch_host<NS>(map, g, rows, rx, ry, 1, X, ldx, ncta, 0);
    CK(cudaGetLastError());
    CK(cudaEventRecord(b));
    CK(cudaEventSynchronize(b));
    float ms;
    CK(cudaEventElapsedTime(&ms, a, b));
    CK(cudaEventDestroy(a));
    CK(cudaEventDestroy(b));
    return ms / launches;
}

template <typename T>
static void sweep(const Layer &L, const char *dt, int reps, int launches) {
    const int N = 5000, B = 10, P = 10, k = 3, pad = 1, stride = 1, nb = N / (B * P), nimg = nb * B;
    const size_t nel = (size_t)nimg * L.H * L.H * L.c;
    T *map;
    CK(cudaMallocHost(&map, nel * sizeof(T)));
    std::mt19937 rng(7);
    std::normal_distribution<float> nd;
    for (size_t i = 0; i < nel; ++i) map[i] = (T)nd(rng);
    std::vector<int32_t> hx(nb * P), hy(nb * P);
    std::uniform_int_distribution<int> pd(0, L.H - 1);
    for (auto &v : hx) v = pd(rng);
    for (auto &v : hy) v = pd(rng);
    int32_t *rx, *ry;
    float *X, *X0;
    const int64_t K = (int64_t)L.c * k * k;
    CK(cudaMalloc(&rx, hx.size() * 4));
    CK(cudaMalloc(&ry, hy.size() * 4));
    CK(cudaMemcpy(rx, hx.data(), hx.size() * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(ry, hy.data(), hy.size() * 4, cudaMemcpyHostToDevice));
    CK(cudaMalloc(&X, N * K * 4));
    CK(cudaMalloc(&X0, N * K * 4));
    HostGeom g0;
    const cp_window w{1, k, k, 0, pad, pad, 1, stride, stride, 1, 1, 1};
    host_geom(g0, map, (int)sizeof(T), B, P, L.c, 1, L.H, L.H, nullptr, w, 2);
    const int ctas[] = {16, 32, 48, 64, 96, 132};
    const int stages[] = {1, 2, 3};
    std::vector<std::vector<float>> t(18);
    run<2>(map, g0, N, rx, ry, X0, K, 64, 1);
    for (int rep = 0; rep < reps; ++rep) {
        int ci = 0;
        for (int nc : ctas)
            for (int ns : stages) {
                CK(cudaMemset(X, 0xff, N * K * 4));
                const float ms = ns == 1   ? run<1>(map, g0, N, rx, ry, X, K, nc, launches)
                                 : ns == 2 ? run<2>(map, g0, N, rx, ry, X, K, nc, launches)
                                           : run<3>(map, g0, N, rx, ry, X, K, nc, launches);
                t[ci++].push_back(ms);
                if (rep == 0) {
                    std::vector<float> a(N * K), b(N * K);
                    CK(cudaMemcpy(a.data(), X, N * K * 4, cudaMemcpyDeviceToHost));
                    CK(cudaMemcpy(b.data(), X0, N * K * 4, cudaMemcpyDeviceToHost));
                    if (memcmp(a.data(), b.data(), N * K * 4)) {
                        printf("MISMATCH %s %s ctas %d stages %d\n", L.name, dt, nc, ns);
                        exit(3);
                    }
                }
            }
    }
    // window bytes: the in-bounds taps of every window, c elements each
    double wbytes = 0;
    for (int i = 0; i < nb * P; ++i) {
        int taps = 0;
        for (int py = 0; py < k; ++py)
            for (int px = 0; px < k; ++px) {
                const int yy = hx[i] - pad + py, xx = hy[i] - pad + px;
                taps += yy >= 0 && yy < L.H && xx >= 0 && xx < L.H;
            }
        wbytes += (double)taps * L.c * sizeof(T) * B;
    }
    printf("%s %s (c %d, H %d, k 3, N %d): %.0f MB of window bytes; ms per gather, median of %d x %d launches\n",
           L.name, dt, L.c, L.H, N, wbytes / 1e6, reps, launches);
    int ci = 0;
    for (int nc : ctas) {
        printf("  %4d CTAs:", nc);
        for (int ns : stages) {
            auto &v = t[ci++];
            std::sort(v.begin(), v.end());
            const float med = v[v.size() / 2];
            printf("   %d stage%s %7.3f ms (%5.1f GB/s, spread %.3f)", ns, ns > 1 ? "s" : " ", med,
                   wbytes / (med / 1e3) / 1e9, v.back() - v.front());
        }
        printf("\n");
    }
    fflush(stdout);
    CK(cudaFreeHost(map));
    CK(cudaFree(rx));
    CK(cudaFree(ry));
    CK(cudaFree(X));
    CK(cudaFree(X0));
}

int main(int argc, char **argv) {
    const int reps = argc > 1 ? atoi(argv[1]) : 5, launches = argc > 2 ? atoi(argv[2]) : 5;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    printf("device: %s, %d SMs\n", prop.name, prop.multiProcessorCount);
    const Layer layers[] = {{"conv3_2", 256, 56}, {"conv4_2", 512, 28}};
    for (const Layer &L : layers) {
        sweep<float>(L, "fp32", reps, launches);
        sweep<__nv_bfloat16>(L, "bf16", reps, launches);
    }
    return 0;
}
