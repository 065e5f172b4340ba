// fp64 GEMM on the tensor cores in 22-bit split precision -- the bulk products of the least-squares solver when the
// statistics themselves came from the tensor cores (ls.cu: Cholesky trailing updates, forward substitutions).
//
//   C[m, nn] = alpha * sum_r A[m, r] * B[nn, r] + beta * C[m, nn]        A: M x R, B: Nn x R, C: M x Nn, all fp64,
//                                                                        reduction index contiguous in A and B
//
// The reference solves its least squares in float64 LAPACK (lib/decompose.py:665-666).  In the tensor-core mode the
// normal equations already carry the 4e-7 of the split-precision Gram (gram_tc2.cu) and every solve is followed by a
// refinement step from the data; the FP64 pipe, not accuracy, is what bounds the 13-layer step (~7.6e11 fp64 flop).
// This kernel takes the GEMM-shaped bulk of those flops to wgmma:
//
//   prep   row scale 2^e (power of two, exact: max|row| * 2^e in [2^9, 2^10)), v = fl32(x 2^e) = hi + lo with
//          hi = fp16_rn(v), lo = fp16_rn(v - hi) -- 22 mantissa bits of every operand entry, K-major rows, zero padded
//   gemm   hi'hi + hi'lo + lo'hi on wgmma (128 x 128 tiles), the TMA -> wgmma pipeline of tc_common.cuh: fp32
//          accumulation in registers in runs of 64 reduction elements, added with round-to-nearest
//   epilogue  C = beta C + alpha 2^-(eA_i + eB_j) acc, read-modify-write in fp64 straight from the accumulator
//             fragments (pairs of adjacent columns: 16-byte accesses)
//
// Error per product sum: <= ~2.4e-7 * sum_r |a||b| (the dropped lo'lo term and the fp32 accumulation), i.e. relative to
// sqrt(C_ii C_jj) for the symmetric updates of a Cholesky factorisation, summed over all updates (sum_k L_ik^2 = G_ii).
// Bound: the read-modify-write of C (16 bytes per 2R flop) for R <= 512, then the tensor pipe.
#include <cuda.h>
#include <cuda_fp16.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace {

using namespace cptc;

struct GtParams {
    double *C;
    int64_t ldc;
    const double *invA, *invB;  // 2^-e per operand row
    double alpha, beta;
    int M, Nn;
    int nst;       // stages = padded reduction / 64
    int tm, tn;    // 128-row tiles of A / B
    int lower;     // only tiles with ti >= tj
    int ntiles;
    int same;      // B operand rows are the first rows of the A operand (symmetric update): diagonal tiles share A and B
    int rowsA;     // operand rows of the A matrix (hi part); its lo part follows
    int rowsB;
};

struct GtItem {
    int ti, tj;
    bool diag;
};
__device__ __forceinline__ GtItem gt_decode(const GtParams &P, int w) {
    GtItem it;
    if (P.lower) {  // column-tile major: for tj, row tiles ti = tj .. tm-1
        int tj = 0, l = w;
        while (l >= P.tm - tj) { l -= P.tm - tj; ++tj; }
        it.tj = tj;
        it.ti = tj + l;
    } else {
        it.ti = w / P.tn;
        it.tj = w - it.ti * P.tn;
    }
    it.diag = P.same && it.ti == it.tj;
    return it;
}

__global__ void __launch_bounds__(NTHREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const GtParams P) {
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_dyn + 1023) & ~(uintptr_t)1023);
    const uint32_t sbase = smem_u32(smem);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    pipe_init(sbase);
    uint32_t g = 0;
    if (warp == W_TMA) {
        if (lane == 0)
            for (int w = blockIdx.x; w < P.ntiles; w += gridDim.x) {
                const GtItem it = gt_decode(P, w);
                pipe_produce(sbase, g, &mapA, &mapB, it.ti * TILE, P.rowsA, it.tj * TILE, P.rowsB, 0, P.nst, it.diag);
            }
        return;
    }
    const int wg = warp >> 2;
    const bool vec = ((reinterpret_cast<uintptr_t>(P.C) & 15) == 0) && ((P.ldc & 1) == 0);
    for (int w = blockIdx.x; w < P.ntiles; w += gridDim.x) {
        const GtItem it = gt_decode(P, w);
        float sum[FRAG];
        pipe_consume(sbase, g, wg, P.nst, it.diag, sum);
        const int ibase = it.ti * TILE + wg * 64, jbase = it.tj * TILE;
#pragma unroll
        for (int e = 0; e < FRAG; e += 2) {
            const int i = ibase + frag_row(e), j = jbase + frag_col(e);  // this thread's columns j, j + 1
            if (i >= P.M || j >= P.Nn) continue;
            const bool two = j + 1 < P.Nn;
            double *dst = P.C + (int64_t)i * P.ldc + j;
            double2 cv = make_double2(0.0, 0.0);
            if (P.beta != 0.0) {
                if (vec && two) cv = *reinterpret_cast<const double2 *>(dst);
                else { cv.x = dst[0]; if (two) cv.y = dst[1]; }
            }
            const double ai = P.alpha * __ldg(P.invA + i);
            cv.x = P.beta * cv.x + ai * __ldg(P.invB + j) * (double)sum[e];
            cv.y = P.beta * cv.y + ai * (two ? __ldg(P.invB + j + 1) : 0.0) * (double)sum[e + 1];
            if (vec && two) *reinterpret_cast<double2 *>(dst) = cv;
            else { dst[0] = cv.x; if (two) dst[1] = cv.y; }
        }
    }
}

// ------------------------------------------------------------------ operand preparation
// warp = one operand row: row maximum -> power-of-two scale -> hi / lo fp16, zero padding to (rows_pad x Rp)
__global__ void __launch_bounds__(256)
gemm_tc_prep(const double *__restrict__ P, int64_t ld, int rows, int R, int rows_pad, int Rp, __half *__restrict__ Ohi,
             __half *__restrict__ Olo, double *__restrict__ inv) {
    const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= rows_pad) return;
    __half *oh = Ohi + (size_t)row * Rp, *ol = Olo + (size_t)row * Rp;
    if (row >= rows) {
        for (int k = lane; k < Rp; k += 32) { oh[k] = __float2half_rn(0.f); ol[k] = __float2half_rn(0.f); }
        if (lane == 0) inv[row] = 0.0;
        return;
    }
    const double *src = P + (int64_t)row * ld;
    double mx = 0.0;
    for (int k = lane; k < R; k += 32) mx = fmax(mx, fabs(src[k]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    int e = 0;
    if (mx > 0.0 && isfinite(mx)) {
        e = 9 - ilogb(mx);
        e = e > 900 ? 900 : (e < -900 ? -900 : e);
    }
    const double sc = ldexp(1.0, e);
    for (int k = lane; k < Rp; k += 32) {
        float v = 0.f;
        if (k < R) v = (float)(src[k] * sc);
        const __half h = __float2half_rn(v);
        oh[k] = h;
        ol[k] = __float2half_rn(__fsub_rn(v, __half2float(h)));
    }
    if (lane == 0) inv[row] = ldexp(1.0, -e);
}

// ------------------------------------------------------------------ operand preparation, transposed source
// operand row nn, reduction index r  <-  P[r * ld + nn]   (the factor's block row in the backward substitution)
// pass 1: per-column maximum -> power-of-two scale; pass 2: 32 x 32 tiles through shared memory.
__global__ void __launch_bounds__(256)
gemm_tc_colmax(const double *__restrict__ P, int64_t ld, int ncols, int R, int rows_pad, double *__restrict__ scale,
               double *__restrict__ inv) {
    // CTA = 32 columns x 8 row lanes (the loads of a lane are independent: 8 in flight per thread)
    __shared__ double red[8][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int nn = blockIdx.x * 32 + tx;
    double mx = 0.0;
    if (nn < ncols) {
#pragma unroll 8
        for (int r = ty; r < R; r += 8) mx = fmax(mx, fabs(P[(int64_t)r * ld + nn]));
    }
    red[ty][tx] = mx;
    __syncthreads();
    if (ty == 0 && nn < rows_pad) {
#pragma unroll
        for (int k = 1; k < 8; ++k) mx = fmax(mx, red[k][tx]);
        int e = 0;
        if (mx > 0.0 && isfinite(mx)) {
            e = 9 - ilogb(mx);
            e = e > 900 ? 900 : (e < -900 ? -900 : e);
        }
        scale[nn] = nn < ncols ? ldexp(1.0, e) : 0.0;
        inv[nn] = nn < ncols ? ldexp(1.0, -e) : 0.0;
    }
}
__global__ void __launch_bounds__(256)
gemm_tc_prep_t(const double *__restrict__ P, int64_t ld, int ncols, int R, int Rp, const double *__restrict__ scale,
               __half *__restrict__ Ohi, __half *__restrict__ Olo) {
    __shared__ float tile[32][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int nn0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    const int nn = nn0 + tx;
    const double sc = scale[nn];  // 0 for padding rows
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int r = r0 + ty + 8 * k;
        float v = 0.f;
        if (r < R && nn < ncols) v = (float)(P[(int64_t)r * ld + nn] * sc);
        tile[ty + 8 * k][tx] = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int row = nn0 + ty + 8 * k;  // operand row
        const float v = tile[tx][ty + 8 * k];
        const __half h = __float2half_rn(v);
        const size_t o = (size_t)row * Rp + r0 + tx;
        Ohi[o] = h;
        Olo[o] = __float2half_rn(__fsub_rn(v, __half2float(h)));
    }
}

}  // namespace

// slot: which of the handle's operand buffers to use -- one per stream the solver issues work on (calls on one stream
// are ordered, so a buffer is never rewritten under a kernel that still reads it)
// b_nc: the B operand is stored reduction-major, b(nn, r) = B[r * ldb + nn]
int cp_gemm_tc_f64(cp_handle_t h, int slot, const double *A, int64_t lda, const double *B, int64_t ldb, double *C, int64_t ldc,
                   int M, int Nn, int R, double alpha, double beta, int lower, cudaStream_t stream, int max_ctas,
                   int b_nc) {
    if (M <= 0 || Nn <= 0) return CP_OK;
    CP_REQUIRE(slot >= 0 && slot < 3 && R > 0, "cp_gemm_tc_f64: bad slot / R");
    const bool same = (!b_nc && A == B && lda == ldb && Nn <= M);
    const int Rp = cp_cdiv(R, KS) * KS;
    const int rowsA = cp_cdiv(M, TILE) * TILE, rowsB = same ? rowsA : cp_cdiv(Nn, TILE) * TILE;
    const size_t needA = 2 * (size_t)rowsA * Rp * sizeof(__half), needB = same ? 0 : 2 * (size_t)rowsB * Rp * sizeof(__half);
    const size_t need = cp_align_up(needA, 256) + cp_align_up(needB, 256) + cp_align_up((size_t)(rowsA + 2 * rowsB) * 8, 256);
    int rc = cp_buffer_reserve(h->tcbuf[slot], need, 4, "tensor-core GEMM operand buffer");
    if (rc) return rc;
    cp_carver cv(h->tcbuf[slot].ptr);
    __half *opA = cv.take<__half>(2 * (size_t)rowsA * Rp);
    __half *opB = same ? opA : cv.take<__half>(2 * (size_t)rowsB * Rp);
    double *invA = cv.take<double>(rowsA + 2 * rowsB);
    double *invB = same ? invA : invA + rowsA;
    double *scaleB = invA + rowsA + rowsB;  // transposed source only

    gemm_tc_prep<<<rowsA / 8, 256, 0, stream>>>(A, lda, M, R, rowsA, Rp, opA, opA + (size_t)rowsA * Rp, invA);
    CP_CHECK_LAUNCH();
    if (b_nc) {
        gemm_tc_colmax<<<rowsB / 32, 256, 0, stream>>>(B, ldb, Nn, R, rowsB, scaleB, invB);
        CP_CHECK_LAUNCH();
        gemm_tc_prep_t<<<dim3(rowsB / 32, Rp / 32), 256, 0, stream>>>(B, ldb, Nn, R, Rp, scaleB, opB, opB + (size_t)rowsB * Rp);
        CP_CHECK_LAUNCH();
    } else if (!same) {
        gemm_tc_prep<<<rowsB / 8, 256, 0, stream>>>(B, ldb, Nn, R, rowsB, Rp, opB, opB + (size_t)rowsB * Rp, invB);
        CP_CHECK_LAUNCH();
    }
    CUtensorMap mapA, mapB;
    rc = make_map16(h, &mapA, opA, Rp, 2 * (int64_t)rowsA, TILE);
    if (rc) return rc;
    rc = make_map16(h, &mapB, opB, Rp, 2 * (int64_t)rowsB, TILE);
    if (rc) return rc;
    GtParams P{};
    P.C = C; P.ldc = ldc; P.invA = invA; P.invB = invB; P.alpha = alpha; P.beta = beta; P.M = M; P.Nn = Nn;
    P.nst = Rp / KS; P.tm = cp_cdiv(M, TILE); P.tn = cp_cdiv(Nn, TILE); P.lower = lower ? 1 : 0;
    P.ntiles = lower ? P.tn * P.tm - P.tn * (P.tn - 1) / 2 : P.tm * P.tn;
    P.same = same ? 1 : 0; P.rowsA = rowsA; P.rowsB = rowsB;
    static cp_per_device_flag configured;
    if (bool *done = configured.slot(); !*done) {
        CP_CUDA(cudaFuncSetAttribute(gemm_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
        *done = true;
    }
    int grid = h->num_sms;
    if (max_ctas > 0 && max_ctas < grid) grid = max_ctas;
    if (P.ntiles < grid) grid = P.ntiles;
    gemm_tc_kernel<<<grid, NTHREADS, SMEM_BYTES, stream>>>(mapA, mapB, P);
    CP_CHECK_LAUNCH();
    return CP_OK;
}

extern "C" int cp_gemm_tc_split(cp_handle_t h, int M, int Nn, int R, double alpha, const double *A, int64_t lda,
                                const double *B, int64_t ldb, double beta, double *C, int64_t ldc, int lower,
                                cp_stream_t stream) {
    CP_REQUIRE(h && A && B && C, "cp_gemm_tc_split: NULL argument");
    CP_REQUIRE(M >= 0 && Nn >= 0 && R > 0 && R <= 1024 && lda >= R && ldb >= ((lower & 2) ? Nn : R) && ldc >= Nn,
               "cp_gemm_tc_split: bad shape");
    CP_REQUIRE(!(lower & 1) || M >= Nn, "cp_gemm_tc_split: lower tiles need M >= Nn");
    CP_DEVICE_GUARD(h);
    return cp_gemm_tc_f64(h, 0, A, lda, B, ldb, C, ldc, M, Nn, R, alpha, beta, lower & 1, (cudaStream_t)stream, 0, (lower >> 1) & 1);
}
