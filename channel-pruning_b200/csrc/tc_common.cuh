// Shared device / host helpers of the Hopper tensor-core kernels that run on split-fp16 operands (gram_tc2.cu,
// gemm_tc.cu): mbarrier / TMA / wgmma PTX wrappers, the TMA -> wgmma pipeline of one 128 x 128 output tile, and the
// tensor-map encoder for K-major fp16 operand matrices (64-element = 128-byte swizzled boxes).
//
// Pipeline: warp 8 = TMA producer (per 64-element stage: A hi/lo, B hi/lo, 128 rows x 128 B each; diagonal tiles take A
// out of the B tile); warps 0-7 = two consumer warpgroups of 64 x 128 outputs (hi'hi + hi'lo + lo'hi, m64n128k16).  The
// tensor core truncates when it adds into its fp32 accumulator, and that bias shows in means of the products (the
// intercept of a least-squares refit), so an accumulator takes one stage (12 adds) and is then added into fp32 register
// sums with round-to-nearest.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include "common.cuh"

namespace cptc {

constexpr int KS = 64;                      // reduction elements per stage = one 128-byte swizzled row of fp16
constexpr int TILE = 128;                   // output tile edge: rows of A x rows of B
constexpr int OP_TILE = TILE * 128;         // bytes of one 128-row operand tile (hi or lo)
constexpr int STAGE_BYTES = 4 * OP_TILE;    // A hi, A lo, B hi, B lo
constexpr int STAGES = 3;
constexpr int SUB_STAGES = 1;               // stages per accumulator run (64 reduction elements)
constexpr int NCONS_WARPS = 8;              // two consumer warpgroups
constexpr int NTHREADS = 32 * (NCONS_WARPS + 1);
constexpr int W_TMA = NCONS_WARPS;
constexpr int OFF_BAR = STAGES * STAGE_BYTES;
constexpr int SMEM_BYTES = OFF_BAR + 2 * STAGES * 8 + 1024;  // + alignment slack
constexpr int FRAG = 64;                    // fp32 accumulator registers per consumer thread (64 x 128 per warpgroup)

// ------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// bounded wait: a protocol bug traps (CUDA error) after ~2 s instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done = 0;
    uint64_t t0 = 0;
    for (uint32_t spin = 0; !done; ++spin) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(bar), "r"(parity)
            : "memory");
        if (!done && (spin & 63) == 63) {
            uint64_t t;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
            if (t0 == 0) t0 = t;
            else if (t - t0 > 2000000000ull) __trap();
        }
    }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1)
        : "memory");
}
// K-major SWIZZLE_128B operand tile: rows of 128 B, 8-row groups 1024 B apart (wgmma matrix descriptor: start >> 4,
// leading byte offset 1 (unused for swizzled K-major), stride byte offset 1024 >> 4 at 32, layout 1 = 128B swizzle at 62)
__device__ __forceinline__ uint64_t wgmma_desc_k_sw128(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// d (64 x 128 fp32 fragment of the warpgroup) = A (64 x 16) B' (16 x 128) + (acc ? d : 0), both operands K-major in
// shared memory
#define CP_F8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                 "+f"(d[i + 6]), "+f"(d[i + 7])
__device__ __forceinline__ void wgmma_f16_m64n128(float (&d)[FRAG], uint64_t adesc, uint64_t bdesc, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}"
        : CP_F8(0), CP_F8(8), CP_F8(16), CP_F8(24), CP_F8(32), CP_F8(40), CP_F8(48), CP_F8(56)
        : "l"(adesc), "l"(bdesc), "r"(acc)
        : "memory");
}
#undef CP_F8

// Fragment element e of a consumer thread -> (row, column) of its warpgroup's 64 x 128 block: pairs of adjacent columns
__device__ __forceinline__ int frag_row(int e) { return ((threadIdx.x & 127) >> 5) * 16 + ((threadIdx.x & 31) >> 2) + 8 * ((e >> 1) & 1); }
__device__ __forceinline__ int frag_col(int e) { return (e >> 2) * 8 + (threadIdx.x & 3) * 2 + (e & 1); }

// ------------------------------------------------------------------ the pipeline
__device__ __forceinline__ uint32_t bar_full(uint32_t sbase, int s) { return sbase + OFF_BAR + 8 * s; }
__device__ __forceinline__ uint32_t bar_empty(uint32_t sbase, int s) { return sbase + OFF_BAR + 8 * (STAGES + s); }

__device__ __forceinline__ void pipe_init(uint32_t sbase) {
    if (threadIdx.x == 32 * W_TMA) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(bar_full(sbase, s), 1);
            mbar_init(bar_empty(sbase, s), NCONS_WARPS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
}

// Producer (one thread): nst stages of reduction elements r0 + 64 st of operand rows rowA / rowB (hi) and
// rowA + loA / rowB + loB (lo).  g counts the stages issued by this thread so far.
__device__ __forceinline__ void pipe_produce(uint32_t sbase, uint32_t &g, const CUtensorMap *mapA, const CUtensorMap *mapB,
                                             int rowA, int loA, int rowB, int loB, int64_t r0, int nst, bool diag) {
    for (int st = 0; st < nst; ++st, ++g) {
        const int s = g % STAGES;
        mbar_wait(bar_empty(sbase, s), ((g / STAGES) & 1) ^ 1);
        const uint32_t dst = sbase + s * STAGE_BYTES, full = bar_full(sbase, s);
        const int r = (int)(r0 + (int64_t)st * KS);
        mbar_arrive_expect_tx(full, diag ? 2 * OP_TILE : STAGE_BYTES);
        if (!diag) {
            tma_load_2d(dst, mapA, full, r, rowA);
            tma_load_2d(dst + OP_TILE, mapA, full, r, loA + rowA);
        }
        tma_load_2d(dst + 2 * OP_TILE, mapB, full, r, rowB);
        tma_load_2d(dst + 3 * OP_TILE, mapB, full, r, loB + rowB);
    }
}

// Consumer warpgroup wg: sum = this warpgroup's 64 x 128 block of hi'hi + hi'lo + lo'hi over nst stages, fp32 runs of
// SUB_STAGES stages added with round-to-nearest.  g counts the stages consumed so far (same sequence as the producer).
__device__ __forceinline__ void pipe_consume(uint32_t sbase, uint32_t &g, int wg, int nst, bool diag, float (&sum)[FRAG]) {
    float acc[FRAG];
#pragma unroll
    for (int e = 0; e < FRAG; ++e) sum[e] = acc[e] = 0.f;
    const int lane = threadIdx.x & 31;
    for (int st0 = 0; st0 < nst; st0 += SUB_STAGES) {
        const int st1 = st0 + SUB_STAGES < nst ? st0 + SUB_STAGES : nst;
        for (int st = st0; st < st1; ++st) {
            const int s = (g + (st - st0)) % STAGES;
            mbar_wait(bar_full(sbase, s), ((g + (st - st0)) / STAGES) & 1);
            const uint32_t stage = sbase + s * STAGE_BYTES;
            const uint32_t b_hi = stage + 2 * OP_TILE, b_lo = stage + 3 * OP_TILE;
            const uint32_t a_off = (uint32_t)wg * 64 * 128;  // this warpgroup's 64 A rows
            const uint32_t a_hi = (diag ? b_hi : stage) + a_off, a_lo = (diag ? b_lo : stage + OP_TILE) + a_off;
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < KS / 16; ++ks) {
                const uint32_t off = ks * 32;  // 16 fp16 = 32 bytes along K inside the 128-byte swizzled row
                const uint32_t first = (st == st0 && ks == 0) ? 0u : 1u;
                wgmma_f16_m64n128(acc, wgmma_desc_k_sw128(a_hi + off), wgmma_desc_k_sw128(b_hi + off), first);
                wgmma_f16_m64n128(acc, wgmma_desc_k_sw128(a_hi + off), wgmma_desc_k_sw128(b_lo + off), 1u);
                wgmma_f16_m64n128(acc, wgmma_desc_k_sw128(a_lo + off), wgmma_desc_k_sw128(b_hi + off), 1u);
            }
            wgmma_commit();
        }
        wgmma_wait_all();
        __syncwarp();
        if (lane == 0)
            for (int st = st0; st < st1; ++st) mbar_arrive(bar_empty(sbase, (g + (st - st0)) % STAGES));
        g += st1 - st0;
#pragma unroll
        for (int e = 0; e < FRAG; ++e) sum[e] = __fadd_rn(sum[e], acc[e]);
    }
}


typedef CUresult (*encode_fn_t)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline int make_map16(cp_handle_t h, CUtensorMap *map, const __half *base, int64_t inner, int64_t rows, int box_rows) {
    if (!h->tmap_encode) {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        CP_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
        if (!fn || qres != cudaDriverEntryPointSuccess) CP_FAIL(CP_ERR_CUDA, "cuTensorMapEncodeTiled not available");
        h->tmap_encode = fn;
    }
    const cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)inner * 2};
    const cuuint32_t box[2] = {(cuuint32_t)KS, (cuuint32_t)box_rows};
    const cuuint32_t estr[2] = {1, 1};
    CUresult r = ((encode_fn_t)h->tmap_encode)(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void *)base, dims, strides, box,
                                               estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) CP_FAIL(CP_ERR_CUDA, "cuTensorMapEncodeTiled (fp16 operands) failed (%d)", (int)r);
    return CP_OK;
}


}  // namespace cptc
