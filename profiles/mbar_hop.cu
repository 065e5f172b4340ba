// Microbenchmark: what does one intra-CTA hand-shake hop cost on sm_90a?
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o profiles/mbar_hop profiles/mbar_hop.cu && profiles/mbar_hop
//
// One CTA, NW "worker" warps and one single-thread "issuer" (the shape of a producer <-> consumer stage ring).
// Per round: every worker warp signals the issuer (fan-in), the issuer answers (fan-out); ROUNDS rounds, clock64
// around the loop, result = cycles per round (= two hops).  DEPTH > 1 lets the workers run ahead by DEPTH rounds
// (a ring of DEPTH barriers), which is what a multi-stage pipeline relies on to hide the hop latency.
//
// Primitives:  0 mbarrier + try_wait (all lanes probe)     1 mbarrier + test_wait (all lanes probe)
//              2 mbarrier + try_wait (lane 0 probes, __syncwarp fan-out)
//              3 shared-memory counters (st.release / ld.acquire polling)
//              4 named barriers (bar.arrive / bar.sync), fan-in and fan-out
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

constexpr int MAXD = 8;

__device__ __forceinline__ uint32_t s32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mb_init(uint32_t b, uint32_t n) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(b), "r"(n)); }
__device__ __forceinline__ void mb_arrive(uint32_t b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(b) : "memory"); }
template <bool TEST>
__device__ __forceinline__ void mb_wait(uint32_t b, uint32_t parity) {
    uint32_t done = 0;
    while (!done) {
        if (TEST)
            asm volatile("{\n\t.reg .pred p;\n\tmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                         : "=r"(done) : "r"(b), "r"(parity) : "memory");
        else
            asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                         : "=r"(done) : "r"(b), "r"(parity) : "memory");
    }
}

template <int PRIM>
__global__ void hop_kernel(int nw, int rounds, int depth, long long *out) {
    __shared__ __align__(8) unsigned long long bars[2 * MAXD];  // [0..D) workers -> issuer, [D..2D) issuer -> workers
    __shared__ volatile unsigned int cnt_up[MAXD], cnt_dn[MAXD];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const bool issuer = warp == nw;  // highest warp id
    if (threadIdx.x == 0) {
        for (int d = 0; d < depth; ++d) {
            mb_init(s32(&bars[d]), nw);      // one arrival per worker warp
            mb_init(s32(&bars[depth + d]), 1);
            cnt_up[d] = 0;
            cnt_dn[d] = 0;
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    long long t0 = clock64();
    if (issuer) {
        if (PRIM == 4 || lane == 0) {
            for (int r = 0; r < rounds; ++r) {
                const int d = r % depth;
                const uint32_t ph = (r / depth) & 1;
                if (PRIM <= 2) {
                    mb_wait<PRIM == 1>(s32(&bars[d]), ph);
                    mb_arrive(s32(&bars[depth + d]));
                } else if (PRIM == 3) {
                    const unsigned int want = (unsigned int)(r / depth + 1) * nw;
                    while (cnt_up[d] < want) { }
                    __threadfence_block();
                    cnt_dn[d] = r / depth + 1;
                } else {  // named barriers 1+d (up) and 1+MAXD+d (down); whole issuer warp participates
                    asm volatile("bar.sync %0, %1;" ::"r"(1 + d), "r"(32 * (nw + 1)) : "memory");
                    asm volatile("bar.arrive %0, %1;" ::"r"(1 + MAXD / 2 + d), "r"(32 * (nw + 1)) : "memory");
                }
            }
        }
    } else {
        for (int r = 0; r < rounds; ++r) {
            const int d = r % depth;
            const uint32_t ph = (r / depth) & 1;
            // wait until the issuer has answered round r - depth (ring slot free), then signal round r
            if (r >= depth) {
                const uint32_t php = ((r - depth) / depth) & 1;
                if (PRIM == 0) mb_wait<false>(s32(&bars[depth + d]), php);
                else if (PRIM == 1) mb_wait<true>(s32(&bars[depth + d]), php);
                else if (PRIM == 2) { if (lane == 0) mb_wait<false>(s32(&bars[depth + d]), php); __syncwarp(); }
                else if (PRIM == 3) { while (cnt_dn[d] < (unsigned int)((r - depth) / depth + 1)) { } __threadfence_block(); }
                else asm volatile("bar.sync %0, %1;" ::"r"(1 + MAXD / 2 + d), "r"(32 * (nw + 1)) : "memory");
            }
            (void)ph;
            if (PRIM <= 2) { __syncwarp(); if (lane == 0) mb_arrive(s32(&bars[d])); }
            else if (PRIM == 3) { __syncwarp(); if (lane == 0) { __threadfence_block(); atomicAdd((unsigned int *)&cnt_up[d], 1u); } }
            else asm volatile("bar.arrive %0, %1;" ::"r"(1 + d), "r"(32 * (nw + 1)) : "memory");
        }
    }
    long long t1 = clock64();
    if (threadIdx.x == 0) out[0] = t1 - t0;
    __syncthreads();
}

template <int PRIM>
static void run(const char *name, int nw, int depth) {
    long long *d_out, h = 0;
    cudaMalloc(&d_out, sizeof(long long));
    const int rounds = 20000;
    hop_kernel<PRIM><<<1, 32 * (nw + 1)>>>(nw, rounds, depth, d_out);
    hop_kernel<PRIM><<<1, 32 * (nw + 1)>>>(nw, rounds, depth, d_out);
    cudaError_t e = cudaDeviceSynchronize();
    cudaMemcpy(&h, d_out, sizeof(h), cudaMemcpyDeviceToHost);
    printf("%-52s workers %2d depth %d : %7.1f cycles / round%s\n", name, nw, depth, (double)h / rounds,
           e == cudaSuccess ? "" : "  (CUDA ERROR)");
    cudaFree(d_out);
}

int main() {
    for (int nw : {1, 8}) {
        for (int depth : {1, 3}) {
            run<0>("mbarrier, try_wait, all lanes probe", nw, depth);
            run<1>("mbarrier, test_wait, all lanes probe", nw, depth);
            run<2>("mbarrier, try_wait, lane 0 probes + __syncwarp", nw, depth);
            run<3>("shared-memory counters (poll)", nw, depth);
            if (depth <= MAXD / 2) run<4>("named barriers (bar.arrive / bar.sync)", nw, depth);
        }
    }
    return 0;
}
