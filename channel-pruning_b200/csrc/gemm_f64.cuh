// fp64-accumulate tile GEMMs, used wherever the path needs products that are exact with respect to the reference's
// float64 arithmetic (Gram of fp32 data widened to fp64, Cholesky trailing updates, triangular solves through
// inverted diagonal blocks, substitutions).  Both kernels run mma.sync.m8n8k4.f64 (DMMA) on 2 x 4 warps.
//
//   C[m, nn] (op)= sum_r a(m, r) * b(nn, r)
//
// gemm_kernel<TA, TB, A_MC, B_NC>: register-staged, 128 x 128 tiles, for operands that need work on the way in
//   a(m, r)  = A_MC ? A[rowidx(r) * lda + m] : A[m * lda + r]                  (TA = float | double)
//   b(nn, r) = B_NC ? B[rowidx(r) * ldb + nn] - bias[nn] : B[nn * ldb + r]
//   Global -> registers (fp32 widened, rows gathered, bias subtracted) -> double-buffered shared memory, reduction
//   staged 16 deep with register prefetch of the next stage; warp tile 64 x 32 (64 accumulators per lane), 12
//   conflict-free LDS.64 per 32 MMAs (the staged leading dimension is 4 mod 16 doubles).  Optional split of the
//   reduction into fp64 partials.
//
// gemm_async_kernel<T, B_NC>: cp.async-staged, T x T tiles (T = 128 for throughput, 64 for latency: everything on a
//   dependency chain), for plain fp64 operands
//   a(m, r)  = A[m * lda + r]
//   b(nn, r) = B_NC ? B[r * ldb + nn] : B[nn * ldb + r]
//   For fp64 operands the register detour costs 16 conflicting STS per thread and stage and exposes the global latency
//   once per 16-deep stage.  Here 16-byte cp.async copies land the tiles in shared memory directly, NS stages deep, in
//   the layout the MMA fragments want:
//     r-contiguous operand  ->  [tile row][k]   leading dimension BK + 4 doubles  (4 mod 16: the m8n8k4 fragment
//     x-contiguous operand  ->  [k][tile col]   leading dimension T + 4 doubles    loads of a half-warp hit 16 banks)
//   Tails (rows beyond the matrix, reduction not a multiple of the stage) are zero-filled by the copy itself (src-size
//   operand).  Requires 16-byte aligned operands and even leading dimensions (aligned()).
//
// launch() takes the async kernel whenever the operands allow it, the register-staged one otherwise.  Bound: FP64 pipe.
// product() puts launch() behind the split-reduction policy of cp_gram's fp64 products and of cp_gemm_f64.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "common.cuh"

namespace cpgemm {

constexpr int BK = 16, NT = 256;

// Tile sets of a launch over the tiles_m x tiles_n tiles of C:
//   TILES_ALL        every tile, row-tile major
//   TILES_UPPER_SYM  tiles j >= i of a square C (requires M == Nn)
//   TILES_LOWER      tiles i >= j, column-tile major: for tj, row tiles ti = tj .. tiles_m-1 (requires tiles_m >= tiles_n)
enum TileMode { TILES_ALL = 0, TILES_UPPER_SYM = 1, TILES_LOWER = 2 };

// SYM = false: a kernel that never walks TILES_UPPER_SYM (gemm_async_kernel) carries no code for it
// tiles of the set on a grid of tiles_m x tiles_n
template <bool SYM = true>
__host__ __device__ __forceinline__ int tile_count(int tiles_m, int tiles_n, int mode) {
    if (SYM && mode == TILES_UPPER_SYM) return tiles_n * (tiles_n + 1) / 2;
    if (mode == TILES_LOWER) return tiles_n * tiles_m - tiles_n * (tiles_n - 1) / 2;
    return tiles_m * tiles_n;
}
// tiles of the set for an M x Nn product on T x T tiles
inline int num_tiles(int M, int Nn, int mode, int T) { return tile_count((M + T - 1) / T, (Nn + T - 1) / T, mode); }

// tile index l of the set -> tile row ti, tile column tj
template <bool SYM = true>
__device__ __forceinline__ void tile_coords(int l, int tiles_m, int tiles_n, int mode, int &ti, int &tj) {
    if (SYM && mode == TILES_UPPER_SYM) {
        ti = 0;
        while (l >= tiles_n - ti) { l -= tiles_n - ti; ++ti; }
        tj = ti + l;
    } else if (mode == TILES_LOWER) {
        tj = 0;
        while (l >= tiles_m - tj) { l -= tiles_m - tj; ++tj; }
        ti = tj + l;
    } else {
        ti = l / tiles_n;
        tj = l - ti * tiles_n;
    }
}

__device__ __forceinline__ void dmma884(double &c0, double &c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                 : "+d"(c0), "+d"(c1)
                 : "d"(a), "d"(b));
}

// ---------------------------------------------------------------- register-staged kernel
constexpr int BM = 128, BN = 128;
constexpr int LDS_ = BM + 4;  // padded leading dimension of a staged tile (doubles): 4 mod 16 (DMMA fragment loads)
constexpr size_t SMEM_BYTES = 2ull /*buffers*/ * 2 /*A,B*/ * BK * LDS_ * sizeof(double);

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

template <typename TA, typename TB, bool A_MC, bool B_NC>
__global__ void __launch_bounds__(NT, 1) gemm_kernel(const Args g) {
    extern __shared__ __align__(16) double smem[];
    // stage buffer b: A tile at smem + b*2*BK*LDS_, B tile right after it
    auto As = [&](int b) { return smem + (size_t)b * 2 * BK * LDS_; };
    auto Bs = [&](int b) { return smem + (size_t)b * 2 * BK * LDS_ + BK * LDS_; };

    const int tiles_m = (g.M + BM - 1) / BM, tiles_n = (g.Nn + BN - 1) / BN;
    const int ntiles = tile_count(tiles_m, tiles_n, g.tile_mode);
    const int lane = threadIdx.x & 31, wm = threadIdx.x >> 7, wn = (threadIdx.x >> 5) & 3;  // 2 x 4 warps
    const TA *A = reinterpret_cast<const TA *>(g.A);
    const TB *B = reinterpret_cast<const TB *>(g.B);
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    int ti, tj;
    tile_coords(tile, tiles_m, tiles_n, g.tile_mode, ti, tj);
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
    auto erow = [&](int i) { return wm * 64 + 8 * i + (lane >> 2); };
    auto ecol = [&](int q) { return wn * 32 + 8 * q + 2 * (lane & 3); };
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

// ---------------------------------------------------------------- cp.async-staged kernel
constexpr int LDK = BK + 4;  // [row][k] tiles

struct AsyncArgs {
    const double *A;
    int64_t lda;
    const double *B;
    int64_t ldb;
    double *C;
    int64_t ldc;
    int M, Nn, R;
    double alpha, beta;
    int tile_mode;  // TILES_ALL or TILES_LOWER
    int max_ctas;   // > 0: at most that many CTAs walk the tiles (leaves SMs free for latency-bound kernels of other
                    // streams: a resident 128 x 128 x 256 tile holds its SM for a long time)
};

template <int T>
struct Cfg {
    static constexpr int NS = T == 128 ? 4 : 3;                 // stages
    static constexpr int LDX = T + 4;                           // [k][col] tiles
    static constexpr int A_ELEMS = T * LDK;                     // doubles per A stage
    static constexpr int B_ELEMS_RC = T * LDK, B_ELEMS_XC = BK * LDX;
    static constexpr int WM = T / 2, WN = T / 4;                // warp tile
    static constexpr int MI = WM / 8, NJ = WN / 8;              // MMA tiles per warp
};

__device__ __forceinline__ void cp_async16(void *smem, const void *gmem, int src_bytes) {
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// r-contiguous operand: T rows x BK doubles = T * 8 chunks of 16 bytes
template <int T>
__device__ __forceinline__ void load_rc(double *S, const double *P, int64_t ld, int x0, int xlim, int r0, int rlim) {
#pragma unroll
    for (int q = threadIdx.x; q < T * 8; q += NT) {
        const int row = q >> 3, ch = q & 7;
        const int x = x0 + row, r = r0 + ch * 2;
        int bytes = 0;
        if (x < xlim && r < rlim) bytes = (rlim - r >= 2) ? 16 : 8;
        const double *src = bytes ? P + (int64_t)x * ld + r : P;
        cp_async16(S + row * LDK + ch * 2, src, bytes);
    }
}
// x-contiguous operand: BK rows (k) x T doubles = BK * T / 2 chunks
template <int T>
__device__ __forceinline__ void load_xc(double *S, const double *P, int64_t ld, int x0, int xlim, int r0, int rlim) {
    constexpr int CPR = T / 2;  // chunks per k-row
#pragma unroll
    for (int q = threadIdx.x; q < BK * CPR; q += NT) {
        const int kr = q / CPR, ch = q - kr * CPR;
        const int r = r0 + kr, x = x0 + ch * 2;
        int bytes = 0;
        if (r < rlim && x < xlim) bytes = (xlim - x >= 2) ? 16 : 8;
        const double *src = bytes ? P + (int64_t)r * ld + x : P;
        cp_async16(S + kr * Cfg<T>::LDX + ch * 2, src, bytes);
    }
}

template <int T, bool B_NC>
__global__ void __launch_bounds__(NT, T == 128 ? 1 : 2) gemm_async_kernel(const AsyncArgs g) {
    using C_ = Cfg<T>;
    extern __shared__ __align__(16) double sm_async[];
    constexpr int B_ELEMS = B_NC ? C_::B_ELEMS_XC : C_::B_ELEMS_RC;
    constexpr int STAGE = C_::A_ELEMS + B_ELEMS;
    const int lane = threadIdx.x & 31, wm = threadIdx.x >> 7, wn = (threadIdx.x >> 5) & 3;
    const int tiles_m = (g.M + T - 1) / T, tiles_n = (g.Nn + T - 1) / T;
    const int ntiles = tile_count<false>(tiles_m, tiles_n, g.tile_mode);
    const int nk = (g.R + BK - 1) / BK;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        int ti, tj;
        tile_coords<false>(tile, tiles_m, tiles_n, g.tile_mode, ti, tj);
        const int m0 = ti * T, n0 = tj * T;
        auto issue = [&](int kb) {
            if (kb < nk) {
                double *S = sm_async + (size_t)(kb % C_::NS) * STAGE;
                load_rc<T>(S, g.A, g.lda, m0, g.M, kb * BK, g.R);
                if constexpr (B_NC) load_xc<T>(S + C_::A_ELEMS, g.B, g.ldb, n0, g.Nn, kb * BK, g.R);
                else load_rc<T>(S + C_::A_ELEMS, g.B, g.ldb, n0, g.Nn, kb * BK, g.R);
            }
            cp_commit();  // one group per slot, empty or not: the wait below counts groups
        };
        double acc[C_::MI][2 * C_::NJ];
#pragma unroll
        for (int i = 0; i < C_::MI; ++i)
#pragma unroll
            for (int j = 0; j < 2 * C_::NJ; ++j) acc[i][j] = 0.0;
#pragma unroll
        for (int s = 0; s < C_::NS - 1; ++s) issue(s);
        for (int kb = 0; kb < nk; ++kb) {
            cp_wait<C_::NS - 2>();   // this thread's copies of stage kb have landed ...
            __syncthreads();         // ... and everybody's; everybody is also done with the slot refilled next
            issue(kb + C_::NS - 1);
            const double *a_s = sm_async + (size_t)(kb % C_::NS) * STAGE;
            const double *b_s = a_s + C_::A_ELEMS;
            const double *ap = a_s + (wm * C_::WM + (lane >> 2)) * LDK + (lane & 3);
#pragma unroll
            for (int k4 = 0; k4 < BK; k4 += 4) {
                double af[C_::MI], bf[C_::NJ];
#pragma unroll
                for (int i = 0; i < C_::MI; ++i) af[i] = ap[8 * i * LDK + k4];
#pragma unroll
                for (int j = 0; j < C_::NJ; ++j) {
                    if constexpr (B_NC) bf[j] = b_s[(k4 + (lane & 3)) * C_::LDX + wn * C_::WN + 8 * j + (lane >> 2)];
                    else bf[j] = b_s[(wn * C_::WN + 8 * j + (lane >> 2)) * LDK + k4 + (lane & 3)];
                }
#pragma unroll
                for (int i = 0; i < C_::MI; ++i)
#pragma unroll
                    for (int j = 0; j < C_::NJ; ++j) dmma884(acc[i][2 * j], acc[i][2 * j + 1], af[i], bf[j]);
            }
        }
        cp_wait<0>();
        __syncthreads();  // the next tile's prologue refills the slots
        // ---- epilogue: acc[i][2j + e] -> row m0 + wm*WM + 8i + (lane >> 2), column n0 + wn*WN + 8j + 2 (lane & 3) + e;
        // every old C value of a group of rows is loaded before any is stored (one memory latency per group)
        const bool rmw = g.beta != 0.0;
        const bool cvec = ((reinterpret_cast<uintptr_t>(g.C) & 15) == 0) && (g.ldc % 2 == 0);
        constexpr int GRP = C_::MI >= 4 ? 4 : C_::MI;
#pragma unroll
        for (int ig = 0; ig < C_::MI; ig += GRP) {
            double old[GRP][2 * C_::NJ];
#pragma unroll
            for (int u = 0; u < GRP; ++u) {
                const int m = m0 + wm * C_::WM + 8 * (ig + u) + (lane >> 2);
#pragma unroll
                for (int j = 0; j < C_::NJ; ++j) {
                    const int nn = n0 + wn * C_::WN + 8 * j + 2 * (lane & 3);
                    old[u][2 * j] = old[u][2 * j + 1] = 0.0;
                    if (rmw && m < g.M) {
                        const double *p = g.C + (int64_t)m * g.ldc + nn;
                        if (cvec && nn + 1 < g.Nn) {
                            const double2 v = *reinterpret_cast<const double2 *>(p);
                            old[u][2 * j] = v.x;
                            old[u][2 * j + 1] = v.y;
                        } else {
                            if (nn < g.Nn) old[u][2 * j] = p[0];
                            if (nn + 1 < g.Nn) old[u][2 * j + 1] = p[1];
                        }
                    }
                }
            }
#pragma unroll
            for (int u = 0; u < GRP; ++u) {
                const int m = m0 + wm * C_::WM + 8 * (ig + u) + (lane >> 2);
                if (m >= g.M) continue;
#pragma unroll
                for (int j = 0; j < C_::NJ; ++j) {
                    const int nn = n0 + wn * C_::WN + 8 * j + 2 * (lane & 3);
                    double v0 = acc[ig + u][2 * j] * g.alpha, v1 = acc[ig + u][2 * j + 1] * g.alpha;
                    if (rmw) {
                        v0 = fma(g.beta, old[u][2 * j], v0);
                        v1 = fma(g.beta, old[u][2 * j + 1], v1);
                    }
                    double *p = g.C + (int64_t)m * g.ldc + nn;
                    if (cvec && nn + 1 < g.Nn) {
                        *reinterpret_cast<double2 *>(p) = make_double2(v0, v1);
                    } else {
                        if (nn < g.Nn) p[0] = v0;
                        if (nn + 1 < g.Nn) p[1] = v1;
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------- launches
// the cp.async copies need 16-byte aligned operands and rows of whole 16-byte chunks
inline bool aligned(const AsyncArgs &g) {
    return cp_aligned16(g.A) && cp_aligned16(g.B) && (g.lda % 2 == 0) && (g.ldb % 2 == 0);
}

template <int T, bool B_NC>
inline cudaError_t launch_async(const AsyncArgs &g, cudaStream_t stream) {
    using C_ = Cfg<T>;
    if (g.tile_mode == TILES_UPPER_SYM) return cudaErrorInvalidValue;
    if (g.M <= 0 || g.Nn <= 0) return cudaSuccess;
    constexpr size_t smem = (size_t)C_::NS * (C_::A_ELEMS + (B_NC ? C_::B_ELEMS_XC : C_::B_ELEMS_RC)) * sizeof(double);
    auto kern = gemm_async_kernel<T, B_NC>;
    static cp_per_device_flag configured;  // per instantiation
    if (bool *done = configured.slot(); !*done) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        *done = true;
    }
    unsigned grid = (unsigned)num_tiles(g.M, g.Nn, g.tile_mode, T);
    if (g.max_ctas > 0 && grid > (unsigned)g.max_ctas) grid = (unsigned)g.max_ctas;
    kern<<<grid, NT, smem, stream>>>(g);
    return cudaGetLastError();
}

// C (op)= a b' in the operand layouts of gemm_kernel<TA, TB, A_MC, B_NC>: on gemm_async_kernel<tile, B_NC> (tile = 64
// or 128) when the operands are plain aligned fp64 (no widening, no gather, no bias, no split, no symmetric tile set),
// otherwise on gemm_kernel
template <typename TA, typename TB, bool A_MC, bool B_NC>
inline cudaError_t launch(const Args &g, cudaStream_t stream, int tile = 128) {
    if constexpr (std::is_same_v<TA, double> && std::is_same_v<TB, double> && !A_MC) {
        const AsyncArgs a{(const double *)g.A, g.lda, (const double *)g.B, g.ldb, g.C, g.ldc, g.M, g.Nn, (int)g.R,
                          g.alpha, g.beta, g.tile_mode, 0};
        if (g.nsplit == 1 && !g.rowidx && !g.b_bias && g.R > 0 && g.R <= INT32_MAX && g.tile_mode != TILES_UPPER_SYM &&
            aligned(a))
            return tile == 128 ? launch_async<128, B_NC>(a, stream) : launch_async<64, B_NC>(a, stream);
    }
    auto kern = gemm_kernel<TA, TB, A_MC, B_NC>;
    static cp_per_device_flag configured;  // per instantiation
    if (bool *done = configured.slot(); !*done) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES);
        if (e != cudaSuccess) return e;
        *done = true;
    }
    dim3 grid((unsigned)num_tiles(g.M, g.Nn, g.tile_mode, BM), (unsigned)(g.nsplit > 1 ? g.nsplit : 1));
    if (grid.x == 0) return cudaSuccess;
    kern<<<grid, NT, SMEM_BYTES, stream>>>(g);
    return cudaGetLastError();
}

// ---------------------------------------------------------------- products on the handle
// C[i, j] = alpha * (sum of the nsplit M x Nn partials, in split order) + beta * C[i, j]; C is not read when beta == 0.
// SYM: upper tiles only, the lower ones come from mirror_upper_tiles.
template <bool SYM>
__global__ void reduce_splits(const double *__restrict__ part, int nsplit, double *__restrict__ C, int M, int Nn,
                              int64_t ldc, double alpha, double beta) {
    const int64_t total = (int64_t)M * Nn;
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    const int i = (int)(e / Nn), j = (int)(e - (int64_t)i * Nn);
    if (SYM && (i / BM) > (j / BN)) return;
    double s = 0.0;
    for (int k = 0; k < nsplit; ++k) s += part[k * total + e];
    double v = alpha * s;
    if (beta != 0.0) v = fma(beta, C[(int64_t)i * ldc + j], v);
    C[(int64_t)i * ldc + j] = v;
}

// C[j, i] = C[i, j] for every element of the strictly-upper T x T tiles, through a padded shared-memory tile so that
// both the reads and the writes are coalesced.
template <int T>
__global__ void __launch_bounds__(256)
mirror_upper_tiles(double *__restrict__ C, int M, int64_t ldc) {
    __shared__ double t[32][33];
    const int bx = blockIdx.x, by = blockIdx.y;  // 32x32 sub-tile (row block by, column block bx)
    if ((by * 32) / T >= (bx * 32) / T) return;  // only strictly-upper T-tiles
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int r = ty; r < 32; r += 8) {
        const int i = by * 32 + r, j = bx * 32 + tx;
        if (i < M && j < M) t[r][tx] = C[(int64_t)i * ldc + j];
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
        const int j = bx * 32 + r, i = by * 32 + tx;
        if (i < M && j < M) C[(int64_t)j * ldc + i] = t[tx][r];
    }
}

// C = alpha a b' + beta C, for the operands, shape, row gather, bias, alpha, beta, tile set, C and ldc set in g.
// Products whose tiles do not fill 2 x SMs, over at least min_split_r reduction rows, split the reduction over CTAs
// (at least 64 rows per split, a multiple of BK) into fp64 partials in the handle's scratch, summed in a fixed order
// (deterministic, no atomics).  TILES_UPPER_SYM fills the lower tiles from the upper ones.  R = 0 gives C = beta C.
template <typename TA, typename TB, bool A_MC, bool B_NC>
int product(cp_handle_t h, Args g, int64_t min_split_r, cudaStream_t stream) {
    g.a_vec = cp_aligned16(g.A) && (g.lda % (16 / sizeof(TA)) == 0);
    g.b_vec = cp_aligned16(g.B) && (g.ldb % (16 / sizeof(TB)) == 0);
    const int tiles = num_tiles(g.M, g.Nn, g.tile_mode, BM);
    const int target = 2 * h->num_sms;
    int nsplit = 1;
    int64_t rps = g.R;
    if (tiles < target && g.R > 0 && g.R >= min_split_r) {
        nsplit = (target + tiles - 1) / tiles;
        const int64_t max_by_rows = (g.R + 4 * BK - 1) / (4 * BK);
        if (nsplit > max_by_rows) nsplit = (int)max_by_rows;
        rps = (g.R + nsplit - 1) / nsplit;
        rps = (rps + BK - 1) / BK * BK;
        nsplit = (int)((g.R + rps - 1) / rps);
    }
    double *const C = g.C;
    const int64_t ldc = g.ldc;
    const bool sym = g.tile_mode == TILES_UPPER_SYM;
    if (nsplit == 1) {
        g.nsplit = 1;
        g.r_per_split = g.R;
        // fewer 128 x 128 tiles than SMs: 64 x 64 tiles if the cp.async kernel takes the product
        CP_GEMM_LAUNCH((launch<TA, TB, A_MC, B_NC>(g, stream, tiles >= h->num_sms ? 128 : 64)));
    } else {
        void *ws = nullptr;
        int rc = cp_ws_reserve(h, (size_t)nsplit * g.M * g.Nn * sizeof(double), &ws);
        if (rc) return rc;
        g.nsplit = nsplit;
        g.r_per_split = rps;
        g.C = (double *)ws; g.ldc = g.Nn; g.c_split_stride = (int64_t)g.M * g.Nn;
        CP_GEMM_LAUNCH((launch<TA, TB, A_MC, B_NC>(g, stream)));
        const unsigned blocks = (unsigned)cp_cdiv((int64_t)g.M * g.Nn, 256);
        if (sym) reduce_splits<true><<<blocks, 256, 0, stream>>>(g.C, nsplit, C, g.M, g.Nn, ldc, g.alpha, g.beta);
        else reduce_splits<false><<<blocks, 256, 0, stream>>>(g.C, nsplit, C, g.M, g.Nn, ldc, g.alpha, g.beta);
        CP_CHECK_LAUNCH();
    }
    if (sym && g.M > BM) {
        const int nb32 = (g.M + 31) / 32;
        mirror_upper_tiles<BM><<<dim3(nb32, nb32), 256, 0, stream>>>(C, g.M, ldc);
        CP_CHECK_LAUNCH();
    }
    return CP_OK;
}

// scale * column sums (and optionally scale * sums of squares) of X[rows] - bias, fp64 accumulation in a fixed
// summation order: each CTA owns 32 columns, 8 row lanes, then a serial 8-way add.
template <typename T>
__global__ void __launch_bounds__(256)
colsum_kernel(const T *__restrict__ X, int64_t ld, int ncols, const int32_t *__restrict__ rows, int64_t nrows,
              const float *__restrict__ bias, double scale, double *__restrict__ sum_out,
              double *__restrict__ sumsq_out) {
    __shared__ double s1[8][33], s2[8][33];
    const int cx = threadIdx.x & 31, rg = threadIdx.x >> 5;
    const int col = blockIdx.x * 32 + cx;
    double a = 0.0, q = 0.0;
    if (col < ncols) {
        const double b = bias ? (double)bias[col] : 0.0;
        for (int64_t r = rg; r < nrows; r += 8) {
            const int64_t row = rows ? (int64_t)rows[r] : r;
            const double v = (double)__ldg(X + row * ld + col) - b;
            a += v;
            q = fma(v, v, q);
        }
    }
    s1[rg][cx] = a;
    s2[rg][cx] = q;
    __syncthreads();
    if (rg == 0 && col < ncols) {
        double ta = 0.0, tq = 0.0;
#pragma unroll
        for (int k = 0; k < 8; ++k) { ta += s1[k][cx]; tq += s2[k][cx]; }
        if (sum_out) sum_out[col] = ta * scale;
        if (sumsq_out) sumsq_out[col] = tq * scale;
    }
}

}  // namespace cpgemm
