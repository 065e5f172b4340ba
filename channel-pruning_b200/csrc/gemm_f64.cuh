// fp64-accumulate tile GEMM used wherever the path needs products that are exact with
// respect to the reference's float64 arithmetic (Gram of fp32 data widened to fp64,
// Cholesky trailing updates, triangular solves through inverted diagonal blocks).
//
//   C[m, nn] (op)= sum_{r = r_begin}^{r_end-1}  a(m, r) * b(nn, r)
//
//   a(m, r) = A_MC ? A[rowidx(r) * lda + m] : A[m * lda + r]      (TA = float | double)
//   b(nn,r) = B_NC ? B[rowidx(r) * ldb + nn] - bias[nn] : B[nn * ldb + r]
//
// CTA tile 128 x 128, 256 threads, reduction staged 16 deep through double-buffered shared
// memory with register prefetch of the next stage.  Two inner loops over the same staged tiles:
//   DMMA (default)  mma.sync.m8n8k4.f64: warp tile 64 x 32 (8 x 4 MMA tiles, 64 accumulators per lane),
//                   12 conflict-free LDS.64 per 32 MMAs (the staged leading dimension is 4 mod 16 doubles)
//   DFMA            8 x 8 register micro-tile per thread (interleaved 2-wide, LDS.128)
// CPB200_GEMM=dfma selects the second (A/B measurements: profiles/gemm_bench.py).  Bound: FP64 pipe.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdlib>

namespace cpgemm {

constexpr int BM = 128, BN = 128, BK = 16, NT = 256;
constexpr int LDS_ = BM + 4;  // padded leading dimension of a staged tile (doubles): 4 mod 16 (DMMA fragment loads)
constexpr size_t SMEM_BYTES = 2ull /*buffers*/ * 2 /*A,B*/ * BK * LDS_ * sizeof(double);

enum TileMode { TILES_ALL = 0, TILES_UPPER_SYM = 1, TILES_LOWER = 2 };

struct Args {
    const void *A;
    int64_t lda;
    const void *B;
    int64_t ldb;
    double *C;
    int64_t ldc;
    int64_t c_split_stride;  // elements between split partials (nsplit > 1)
    int M, Nn;
    int64_t R;
    const int32_t *rowidx;  // optional gather on the reduction index (A_MC / B_NC operands only)
    const float *b_bias;    // optional, B_NC only
    int nsplit;
    int64_t r_per_split;    // multiple of BK
    double alpha, beta;     // nsplit == 1: C = alpha*acc + beta*C ; nsplit > 1: partial = acc
    int tile_mode;
    int a_vec, b_vec;       // 16-byte vector loads allowed (alignment checked by the host)
    int max_ctas;           // > 0: at most that many CTAs walk the tiles (leaves SMs free for latency-bound kernels of
                            // other streams: a resident 128 x 128 x 256 tile holds its SM for a long time)
};

template <typename T>
__device__ __forceinline__ double to_f64(T v) { return (double)v; }

// Loads 8 consecutive elements (contiguous direction) starting at p[0], valid count `nvalid` (0..8).
template <typename T>
__device__ __forceinline__ void load8(const T *p, int nvalid, bool vec, double out[8]) {
    if (nvalid >= 8 && vec) {
        if constexpr (sizeof(T) == 4) {
            const float4 v0 = __ldg(reinterpret_cast<const float4 *>(p));
            const float4 v1 = __ldg(reinterpret_cast<const float4 *>(p) + 1);
            out[0] = v0.x; out[1] = v0.y; out[2] = v0.z; out[3] = v0.w;
            out[4] = v1.x; out[5] = v1.y; out[6] = v1.z; out[7] = v1.w;
        } else {
            const double2 *q = reinterpret_cast<const double2 *>(p);
            const double2 v0 = __ldg(q), v1 = __ldg(q + 1), v2 = __ldg(q + 2), v3 = __ldg(q + 3);
            out[0] = v0.x; out[1] = v0.y; out[2] = v1.x; out[3] = v1.y;
            out[4] = v2.x; out[5] = v2.y; out[6] = v3.x; out[7] = v3.y;
        }
    } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) out[i] = (i < nvalid) ? to_f64(__ldg(p + i)) : 0.0;
    }
}

// Operand whose tile dimension (m or nn) is contiguous in memory: element (x, r) = P[rowidx(r)*ld + x].
// thread t fetches r = t/16, x = (t%16)*8 .. +8
template <typename T>
__device__ __forceinline__ void fetch_xcontig(const T *P, int64_t ld, const int32_t *rowidx, int x0, int xlim,
                                              int64_t r0, int64_t rlim, bool vec, const float *bias,
                                              double out[8]) {
    const int t = threadIdx.x;
    const int64_t r = r0 + (t >> 4);
    const int x = x0 + (t & 15) * 8;
    int nvalid = xlim - x;
    nvalid = nvalid < 0 ? 0 : (nvalid > 8 ? 8 : nvalid);
    if (r >= rlim) nvalid = 0;
    if (nvalid == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) out[i] = 0.0;
        return;
    }
    const int64_t row = rowidx ? (int64_t)__ldg(rowidx + r) : r;
    load8(P + row * ld + x, nvalid, vec, out);
    if (bias) {
#pragma unroll
        for (int i = 0; i < 8; ++i)
            if (i < nvalid) out[i] -= (double)__ldg(bias + x + i);
    }
}
__device__ __forceinline__ void stage_xcontig(double *S, const double v[8]) {
    const int t = threadIdx.x;
    double *d = S + (t >> 4) * LDS_ + (t & 15) * 8;
#pragma unroll
    for (int i = 0; i < 8; i += 2) *reinterpret_cast<double2 *>(d + i) = make_double2(v[i], v[i + 1]);
}

// Operand whose reduction dimension is contiguous: element (x, r) = P[x*ld + r].
// thread t fetches x = t/2, r = (t%2)*8 .. +8
template <typename T>
__device__ __forceinline__ void fetch_rcontig(const T *P, int64_t ld, int x0, int xlim, int64_t r0, int64_t rlim,
                                              bool vec, double out[8]) {
    const int t = threadIdx.x;
    const int x = x0 + (t >> 1);
    const int64_t r = r0 + (t & 1) * 8;
    int64_t nv = rlim - r;
    int nvalid = nv < 0 ? 0 : (nv > 8 ? 8 : (int)nv);
    if (x >= xlim) nvalid = 0;
    if (nvalid == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) out[i] = 0.0;
        return;
    }
    load8(P + (int64_t)x * ld + r, nvalid, vec, out);
}
__device__ __forceinline__ void stage_rcontig(double *S, const double v[8]) {
    const int t = threadIdx.x;
    double *d = S + ((t & 1) * 8) * LDS_ + (t >> 1);
#pragma unroll
    for (int i = 0; i < 8; ++i) d[i * LDS_] = v[i];
}

__device__ __forceinline__ int num_tiles_dev(int tm, int tn, int mode) {
    if (mode == 1) return tn * (tn + 1) / 2;
    if (mode == 2) return tn * tm - tn * (tn - 1) / 2;
    return tm * tn;
}

__device__ __forceinline__ void dmma884(double &c0, double &c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                 : "+d"(c0), "+d"(c1)
                 : "d"(a), "d"(b));
}

template <typename TA, typename TB, bool A_MC, bool B_NC, bool DMMA>
__global__ void __launch_bounds__(NT, 1) gemm_kernel(const Args g) {
    extern __shared__ __align__(16) double smem[];
    // stage buffer b: A tile at smem + b*2*BK*LDS_, B tile right after it
    auto As = [&](int b) { return smem + (size_t)b * 2 * BK * LDS_; };
    auto Bs = [&](int b) { return smem + (size_t)b * 2 * BK * LDS_ + BK * LDS_; };

    // ---- tile decode (a capped grid walks the tiles with a stride)
    const int tiles_m = (g.M + BM - 1) / BM, tiles_n = (g.Nn + BN - 1) / BN;
    const int ntiles = num_tiles_dev(tiles_m, tiles_n, g.tile_mode);
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int lane = threadIdx.x & 31, wm = threadIdx.x >> 7, wn = (threadIdx.x >> 5) & 3;  // DMMA: 2 x 4 warps
    const TA *A = reinterpret_cast<const TA *>(g.A);
    const TB *B = reinterpret_cast<const TB *>(g.B);
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    int l = tile, ti, tj;
    if (g.tile_mode == TILES_UPPER_SYM) {
        ti = 0;
        while (l >= tiles_n - ti) { l -= tiles_n - ti; ++ti; }
        tj = ti + l;
    } else if (g.tile_mode == TILES_LOWER) {
        // column-tile major: for tj, row tiles ti = tj .. tiles_m-1
        tj = 0;
        while (l >= tiles_m - tj) { l -= tiles_m - tj; ++tj; }
        ti = tj + l;
    } else {
        ti = l / tiles_n;
        tj = l - ti * tiles_n;
    }
    const int split = blockIdx.y;
    const int m0 = ti * BM, n0 = tj * BN;
    const int64_t r_begin = (int64_t)split * g.r_per_split;
    int64_t r_end = r_begin + g.r_per_split;
    if (r_end > g.R) r_end = g.R;

    double acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.0;

    double ra[8], rb[8];

    auto fetch = [&](int64_t r0) {
        if constexpr (A_MC) fetch_xcontig<TA>(A, g.lda, g.rowidx, m0, g.M, r0, r_end, g.a_vec, nullptr, ra);
        else fetch_rcontig<TA>(A, g.lda, m0, g.M, r0, r_end, g.a_vec, ra);
        if constexpr (B_NC) fetch_xcontig<TB>(B, g.ldb, g.rowidx, n0, g.Nn, r0, r_end, g.b_vec, g.b_bias, rb);
        else fetch_rcontig<TB>(B, g.ldb, n0, g.Nn, r0, r_end, g.b_vec, rb);
    };
    auto stage = [&](int buf) {
        if constexpr (A_MC) stage_xcontig(As(buf), ra); else stage_rcontig(As(buf), ra);
        if constexpr (B_NC) stage_xcontig(Bs(buf), rb); else stage_rcontig(Bs(buf), rb);
    };

    int buf = 0;
    if (r_begin < r_end) {
        fetch(r_begin);
        stage(0);
    }
    __syncthreads();
    for (int64_t r0 = r_begin; r0 < r_end; r0 += BK) {
        const bool has_next = r0 + BK < r_end;
        if (has_next) fetch(r0 + BK);
        const double *a_s = As(buf), *b_s = Bs(buf);
        if constexpr (DMMA) {
            // acc[i][2j + e]: rows wm*64 + 8i + (lane >> 2), columns wn*32 + 8j + 2 (lane & 3) + e
            const double *ap = a_s + (lane & 3) * LDS_ + wm * 64 + (lane >> 2);
            const double *bp = b_s + (lane & 3) * LDS_ + wn * 32 + (lane >> 2);
#pragma unroll
            for (int k4 = 0; k4 < BK; k4 += 4) {
                double af[8], bf[4];
#pragma unroll
                for (int i = 0; i < 8; ++i) af[i] = ap[k4 * LDS_ + 8 * i];
#pragma unroll
                for (int j = 0; j < 4; ++j) bf[j] = bp[k4 * LDS_ + 8 * j];
#pragma unroll
                for (int i = 0; i < 8; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) dmma884(acc[i][2 * j], acc[i][2 * j + 1], af[i], bf[j]);
            }
        } else {
#pragma unroll
            for (int kk = 0; kk < BK; ++kk) {
                double a[8], b[8];
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const double2 av = *reinterpret_cast<const double2 *>(a_s + kk * LDS_ + q * 32 + ty * 2);
                    const double2 bv = *reinterpret_cast<const double2 *>(b_s + kk * LDS_ + q * 32 + tx * 2);
                    a[2 * q] = av.x; a[2 * q + 1] = av.y;
                    b[2 * q] = bv.x; b[2 * q + 1] = bv.y;
                }
#pragma unroll
                for (int i = 0; i < 8; ++i)
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
            }
        }
        if (has_next) stage(buf ^ 1);
        __syncthreads();
        buf ^= 1;
    }

    // ---- epilogue: two tile rows at a time, all their C values LOADED before any is stored (beta != 0): the
    // read-modify-write of a 128 x 128 tile is 64 values per thread, and one load -> fma -> store chain per value
    // would expose the memory latency 64 times (rank-128 trailing updates spent as long here as in the k loop)
    double *C = g.C + (g.nsplit > 1 ? (int64_t)split * g.c_split_stride : 0);
    const bool partial = g.nsplit > 1;
    const bool rmw = !partial && g.beta != 0.0;
    const bool cvec = ((reinterpret_cast<uintptr_t>(C) & 15) == 0) && (g.ldc % 2 == 0);
    // element (i, 2q + e') of the thread's accumulators sits at tile row erow(i), tile column ecol(q) + e'
    auto erow = [&](int i) { return DMMA ? wm * 64 + 8 * i + (lane >> 2) : (i >> 1) * 32 + ty * 2 + (i & 1); };
    auto ecol = [&](int q) { return DMMA ? wn * 32 + 8 * q + 2 * (lane & 3) : q * 32 + tx * 2; };
#pragma unroll
    for (int ip = 0; ip < 4; ++ip) {
        double old[2][8];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int m = m0 + erow(2 * ip + e);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int nn = n0 + ecol(q);
                old[e][2 * q] = old[e][2 * q + 1] = 0.0;
                if (rmw && m < g.M) {
                    const double *p = C + (int64_t)m * g.ldc + nn;
                    if (cvec && nn + 1 < g.Nn) {
                        const double2 v = *reinterpret_cast<const double2 *>(p);
                        old[e][2 * q] = v.x;
                        old[e][2 * q + 1] = v.y;
                    } else {
                        if (nn < g.Nn) old[e][2 * q] = p[0];
                        if (nn + 1 < g.Nn) old[e][2 * q + 1] = p[1];
                    }
                }
            }
        }
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int i = 2 * ip + e;
            const int m = m0 + erow(i);
            if (m >= g.M) continue;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int nn = n0 + ecol(q);
                double v0 = acc[i][2 * q], v1 = acc[i][2 * q + 1];
                if (!partial) {
                    v0 *= g.alpha;
                    v1 *= g.alpha;
                    if (rmw) {
                        v0 = fma(g.beta, old[e][2 * q], v0);
                        v1 = fma(g.beta, old[e][2 * q + 1], v1);
                    }
                }
                double *p = C + (int64_t)m * g.ldc + nn;
                if (cvec && nn + 1 < g.Nn) {
                    *reinterpret_cast<double2 *>(p) = make_double2(v0, v1);
                } else {
                    if (nn < g.Nn) p[0] = v0;
                    if (nn + 1 < g.Nn) p[1] = v1;
                }
            }
        }
    }
    }  // tile loop (the k loop ends with a __syncthreads: the staging buffers are free again)
}

inline int num_tiles(int M, int Nn, int mode) {
    const int tm = (M + BM - 1) / BM, tn = (Nn + BN - 1) / BN;
    if (mode == TILES_UPPER_SYM) return tn * (tn + 1) / 2;          // requires M == Nn
    if (mode == TILES_LOWER) return tn * tm - tn * (tn - 1) / 2;    // requires tm >= tn
    return tm * tn;
}

inline bool use_dmma() {
    static const bool on = [] {
        const char *e = getenv("CPB200_GEMM");
        return !(e && (e[0] == 'd' || e[0] == 'D') && (e[1] == 'f' || e[1] == 'F'));  // "dfma" switches the MMA loop off
    }();
    return on;
}

template <typename TA, typename TB, bool A_MC, bool B_NC, bool DMMA>
inline cudaError_t launch_impl(const Args &g, cudaStream_t stream) {
    auto kern = gemm_kernel<TA, TB, A_MC, B_NC, DMMA>;
    static bool configured[64] = {};  // per instantiation and per device (the attribute is per device)
    int dev = 0;
    cudaGetDevice(&dev);
    bool &done = configured[dev >= 0 && dev < 64 ? dev : 0];
    if (!done) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES);
        if (e != cudaSuccess) return e;
        done = true;
    }
    dim3 grid((unsigned)num_tiles(g.M, g.Nn, g.tile_mode), (unsigned)(g.nsplit > 1 ? g.nsplit : 1));
    if (grid.x == 0) return cudaSuccess;
    if (g.max_ctas > 0 && grid.x > (unsigned)g.max_ctas) grid.x = (unsigned)g.max_ctas;
    kern<<<grid, NT, SMEM_BYTES, stream>>>(g);
    return cudaGetLastError();
}

template <typename TA, typename TB, bool A_MC, bool B_NC>
inline cudaError_t launch(const Args &g, cudaStream_t stream) {
    return use_dmma() ? launch_impl<TA, TB, A_MC, B_NC, true>(g, stream) : launch_impl<TA, TB, A_MC, B_NC, false>(g, stream);
}

}  // namespace cpgemm
