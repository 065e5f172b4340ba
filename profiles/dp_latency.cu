// Microbenchmark: latency of dependent fp64 operations on one warp (clock64 around an unrolled dependent chain),
// the numbers that bound the serial recurrence of the LASSO coordinate descent (lasso.cu) and the pivot chain of
// the Cholesky panel (ls.cu).   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o dp_latency dp_latency.cu
#include <cstdio>
#include <cuda_runtime.h>

template <int OP>
__global__ void chain(double *out, long long *cyc, double a, double b, int reps) {
    double x = a;
    long long t0 = clock64();
    for (int r = 0; r < reps; ++r) {
#pragma unroll
        for (int i = 0; i < 64; ++i) {
            if (OP == 0) x = __fma_rn(x, b, a);
            if (OP == 1) x = __dadd_rn(x, b);
            if (OP == 2) x = __dmul_rn(x, b);
            if (OP == 3) { x = __dadd_rn(__dmul_rn(x, b), a); }                   // mul + add
            if (OP == 4) { double q0 = __dmul_rn(x, b); double rr = __fma_rn(-q0, a, x); x = __fma_rn(rr, b, q0); }  // markstein
            if (OP == 5) x = __shfl_sync(0xffffffffu, x, (threadIdx.x + 1) & 31);
            if (OP == 6) x = fmax(x, b) + a;                                      // dsetp/sel + add
            if (OP == 7) { float f = (float)x; f = rsqrtf(f); x = (double)f + a; }  // cvt + mufu + cvt + add
            if (OP == 8) x = (x > b) ? __dadd_rn(x, a) : __dadd_rn(-x, b);        // compare-select
            if (OP == 9) x = __ddiv_rn(x, b);
            if (OP == 10) x = sqrt(x) + a;
        }
    }
    long long t1 = clock64();
    if (threadIdx.x == 0) { out[OP] = x; cyc[OP] = t1 - t0; }
}

__global__ void smem_pingpong(long long *cyc, int reps) {
    // warp 0 writes a flag, warp 1 polls it and answers: round-trip of a shared-memory hand-off between two warps
    __shared__ volatile int f0, f1;
    if (threadIdx.x == 0) { f0 = 0; f1 = 0; }
    __syncthreads();
    const int w = threadIdx.x >> 5;
    long long t0 = clock64();
    for (int r = 1; r <= reps; ++r) {
        if (w == 0) { if ((threadIdx.x & 31) == 0) f0 = r; while (f1 != r) {} }
        else { while (f0 != r) {} if ((threadIdx.x & 31) == 0) f1 = r; }
    }
    long long t1 = clock64();
    if (threadIdx.x == 0) cyc[0] = t1 - t0;
}

int main() {
    double *out; long long *cyc;
    cudaMalloc(&out, 16 * sizeof(double)); cudaMalloc(&cyc, 16 * sizeof(long long));
    const int reps = 200;
    const char *names[] = {"DFMA", "DADD", "DMUL", "DMUL+DADD", "markstein(3)", "SHFL.64(2x32)", "DMNMX+DADD", "F2F+MUFU.RSQ+F2F+DADD",
                           "DSETP/sel+DADD", "DDIV", "DSQRT+DADD"};
#define RUN(OP) chain<OP><<<1, 32>>>(out, cyc, 1.0000001, 0.9999999, reps);
    for (int pass = 0; pass < 2; ++pass) { RUN(0) RUN(1) RUN(2) RUN(3) RUN(4) RUN(5) RUN(6) RUN(7) RUN(8) RUN(9) RUN(10) }
    cudaDeviceSynchronize();
    long long h[16];
    cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
    for (int i = 0; i < 11; ++i) printf("%-24s %7.1f cycles per chained group\n", names[i], (double)h[i] / (reps * 64.0));
    smem_pingpong<<<1, 64>>>(cyc, 2000);
    cudaDeviceSynchronize();
    cudaMemcpy(h, cyc, sizeof(long long), cudaMemcpyDeviceToHost);
    printf("%-24s %7.1f cycles per round trip (two hand-offs)\n", "smem flag ping-pong", (double)h[0] / 2000.0);
    printf("cuda status: %s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
