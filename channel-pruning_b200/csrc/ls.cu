// Least-squares reconstruction of the surviving weights.
//
//   cp_ls_solve       <- fc_kernel / LinearRegression(fit_intercept=True).fit
//                        (reference lib/decompose.py:622-623, 636-669): centred normal
//                        equations on the principal sub-block of the Gram matrix.
//   cp_ls_solve_dual  <- the same call when N-1 < K' (gelsd's minimum-norm answer),
//                        through the dual (row) normal equations.
//   cp_ls_factor / cp_ls_resolve
//                     <- nonlinear_fc (lib/decompose.py:671-685): 50 refits against the SAME X --
//                        factor the centred Gram once, then one forward/backward substitution per refit.
//
// All of them run one routine: right-looking blocked Cholesky with 128-wide panels.
//   * the diagonal block of a panel is factored AND inverted by ONE CTA entirely in shared
//     memory (potrf128: 32-wide sub-panels; the 32 x 32 pivot blocks are factored by a single
//     warp in registers with shuffles -- the only truly serial part, ~100 ns per pivot);
//   * the rows below are multiplied by the inverted block (a GEMM, not a triangular solve);
//   * the trailing update is split three ways: the next panel's columns stay on the caller's
//     stream (small 64 x 64 tiles: few flops, many CTAs, short latency), the panel after that
//     and the rest run on a low-priority side stream underneath the next panel's factorisation.
//   * right-hand sides ride along as extra ROWS of the matrix, so the forward substitution
//     happens inside the panel steps; the backward substitution reuses the inverted blocks.
// The factor goes to a second array (L), the trailing matrix is updated in place (M): no step
// reads and writes the same tile, whatever the tile shape.
// Bound: the dependency chain of ~K'/128 x (potrf128 + 2 small GEMMs) for the factorisation,
// the FP64 pipe for the far updates (K'^3/3 flop).
#include "common.cuh"
#include "gemm_f64.cuh"

int cp_gemm_tc_f64(cp_handle_t h, int slot, const double *A, int64_t lda, const double *B, int64_t ldb, double *C,
                   int64_t ldc, int M, int Nn, int R, double alpha, double beta, int lower, cudaStream_t stream,
                   int max_ctas, int b_nc);

namespace {

constexpr int PB = 128;          // panel width
constexpr int GB = 512;          // group of four panels: the substitutions run on inverted GB x GB diagonal blocks
constexpr int SB = 32;           // sub-block factored by one warp
constexpr int NSB = PB / SB;     // 4
constexpr int LDA_S = PB + 1;    // padded leading dimension of the shared-memory panel
constexpr int LDX_S = SB + 1;
constexpr int P128_T = 512;
constexpr size_t P128_SMEM =
    (size_t)(PB * LDA_S + 2 * NSB * SB * LDX_S + 3 * SB * LDX_S + 3 * PB + 2 * SB) * sizeof(double);

// ---------------------------------------------------------------- assemble
// centred right-hand side t at column sj:  Bxy[sj, t] - sx_sj sy_t / N
__device__ __forceinline__ double centred_rhs(const double *__restrict__ Bxy, const double *__restrict__ sx,
                                              const double *__restrict__ sy, double invN, int n, int sj, int t) {
    return Bxy[(int64_t)sj * n + t] - sx[sj] * sy[t] * invN;
}

// M rows 0..Ks-1    : G[sel_i, sel_j] - sx_i sx_j / N   (lower triangle only)
// M rows Ks..Ks+n-1 : Bxy[sel_j, t]   - sx_j sy_t / N   (right-hand sides, transposed)
__global__ void __launch_bounds__(256)
ls_assemble(const double *__restrict__ G, const double *__restrict__ Bxy, const double *__restrict__ sx,
            const double *__restrict__ sy, double invN, int K, int n, const int32_t *__restrict__ sel, int Ks,
            double *__restrict__ M, int64_t ld, double *__restrict__ diag0) {
    const int j = blockIdx.x * 256 + threadIdx.x;
    const int i = blockIdx.y;
    if (j >= Ks) return;
    const int sj = sel ? sel[j] : j;
    if (i < Ks) {
        if (j > i) return;
        const int si = sel ? sel[i] : i;
        const double v = G[(int64_t)si * K + sj] - sx[si] * sx[sj] * invN;
        M[(int64_t)i * ld + j] = v;
        if (i == j) diag0[i] = v;
    } else if (Bxy) {
        M[(int64_t)i * ld + j] = centred_rhs(Bxy, sx, sy, invN, n, sj, i - Ks);
    }
}

// ---------------------------------------------------------------- 128 x 128 diagonal block: L and L^-1
// 1/sqrt(d): hardware fp64 seed (MUFU.RSQ64H, ~2^-22) + ONE third-order correction  y += y e (1/2 + 3/8 e),
// e = 1 - d y^2: four dependent fp64 operations (32 cycles) where two Newton steps on an fp32 seed cost six plus
// two conversions -- this sits on the serial pivot chain of the factorisation.
__device__ __forceinline__ double rsqrt_fast(double d) {
    double y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(d));
    const double t = d * y;
    const double e = fma(-t, y, 1.0);
    const double p = fma(0.375, e, 0.5);
    const double ye = y * e;
    return fma(ye, p, y);
}

__device__ __forceinline__ void atomic_min_pos(double *addr, double v) {  // v > 0: bit patterns order like the values
    atomicMin(reinterpret_cast<unsigned long long *>(addr), (unsigned long long)__double_as_longlong(v));
}

// One warp factors the 32 x 32 block at (k0, k0) of the shared-memory panel.  Lane i owns row i in registers.
// Per pivot the serial chain is: pivot broadcast (one shuffle) -> 1/sqrt -> scale -> the NEXT pivot (lane k+1
// updates its own diagonal entry from its own column entry: no communication) -> broadcast.  The rank-1 update of the
// other entries needs column k of all lanes: published through a double-buffered shared-memory column (one store per
// lane, broadcast LDS.128 reads) -- 32 - k shuffles per pivot had been 3/4 of this routine's time.
__device__ __forceinline__ void potrf32_warp(double *As, int k0, const double *thr_s, double *rinv_s, int32_t *info,
                                             int jglob, int lane, double &ratio_min, const double *inv0_s, double *cb) {
    double a[SB];
#pragma unroll
    for (int j = 0; j < SB; ++j) a[j] = (j <= lane) ? As[(k0 + lane) * LDA_S + k0 + j] : 0.0;
    const double thr = thr_s[k0 + lane];
    double myrs = 1.0;
    double dk = __shfl_sync(0xffffffffu, a[0], 0);
#pragma unroll
    for (int k = 0; k < SB; ++k) {
        const double tk = __shfl_sync(0xffffffffu, thr, k);
        if (lane == k) {  // the pivot as met, before a failed one is replaced: a NaN or negative pivot counts as 0
            const double i0 = inv0_s[k0 + k];
            if (i0 >= 0.0) ratio_min = fmin(ratio_min, dk > 0.0 ? dk * i0 : 0.0);
        }
        // pivot must stay above 1e-12 of the original diagonal entry: the squared form of the
        // sigma < 1e-6 sigma_max cut-off LinearRegression applies (sklearn _base.py:752-753, cond=tol=1e-6)
        if (!(dk > tk)) {
            if (lane == 0) atomicCAS(info, 0, jglob + k0 + k + 1);
            dk = 1.0;
        }
        const double rs = rsqrt_fast(dk);
        double l = (lane > k) ? a[k] * rs : 0.0;
        if (lane == k) {
            l = dk * rs;
            myrs = rs;
        }
        a[k] = l;
        if (k + 1 < SB) {
            // the next pivot, from lane k+1's own entries (bit-identical to its general update below)
            const double dn = fma(-l, l, a[k + 1]);
            const double dnext = __shfl_sync(0xffffffffu, dn, k + 1);
            double *col = cb + (k & 1) * SB;
            col[lane] = l;
            __syncwarp();
#pragma unroll
            for (int jj = (k + 1) & ~1; jj < SB; jj += 2) {
                const double2 v = *reinterpret_cast<const double2 *>(col + jj);
                if (jj >= k + 1) a[jj] = fma(-l, v.x, a[jj]);  // entries right of the diagonal (j > lane) are never read
                a[jj + 1] = fma(-l, v.y, a[jj + 1]);
            }
            dk = dnext;
        }
    }
#pragma unroll
    for (int j = 0; j < SB; ++j)
        if (j <= lane) As[(k0 + lane) * LDA_S + k0 + j] = a[j];
    rinv_s[k0 + lane] = myrs;
}

// out[r * dr + c * dc] = sign * sum_terms sum_q A_t[r * sa_t + q] * B_t[c * sb_t + q]   (32 x 32 blocks)
struct MmTerm {
    const double *A;
    int sa;
    const double *B;
    int sb;
};
struct MmTask {
    double *dst;
    int dr, dc;
    double sign;
    int nterm;
    MmTerm t[3];
};
// acc += one warp's 16 x 16 block of A B' over 32 reduction elements, as 2 x 2 m8n8k4 tiles (acc[u][v]: A rows
// 8u to 8u+7, B rows 8v to 8v+7).  pa, pb: the lane's first fragment elements (row lane / 4, element lane % 4); sa8,
// sb8: the distance of eight rows of A and of B.  Fragment loads: A[r][q], B[c][q] with q contiguous.
__device__ __forceinline__ void dmma_block16(double (&acc)[2][2][2], const double *pa, int sa8, const double *pb,
                                             int sb8) {
#pragma unroll
    for (int q = 0; q < SB; q += 4) {
        const double a0 = pa[q], a1 = pa[sa8 + q], b0 = pb[q], b1 = pb[sb8 + q];
        cpgemm::dmma884(acc[0][0][0], acc[0][0][1], a0, b0);
        cpgemm::dmma884(acc[0][1][0], acc[0][1][1], a0, b1);
        cpgemm::dmma884(acc[1][0][0], acc[1][0][1], a1, b0);
        cpgemm::dmma884(acc[1][1][0], acc[1][1][1], a1, b1);
    }
}

// Block products on the FP64 tensor path: four warps per task, one 16 x 16 quadrant each, so the twelve warps of a
// three-task phase sit on all four schedulers (rather than a 2 x 4 register micro-tile per thread on 128 threads per
// task).
__device__ __forceinline__ void run_tasks_mma(const MmTask *tasks, int ntask) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp >= ntask * 4) return;
    const MmTask &tk = tasks[warp >> 2];
    const int r0 = ((warp >> 1) & 1) * 16, c0 = (warp & 1) * 16;
    const int fr = lane >> 2, fk = lane & 3;
    double acc[2][2][2];
#pragma unroll
    for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int v = 0; v < 2; ++v) acc[u][v][0] = acc[u][v][1] = 0.0;
    for (int w = 0; w < tk.nterm; ++w)
        dmma_block16(acc, tk.t[w].A + (r0 + fr) * tk.t[w].sa + fk, 8 * tk.t[w].sa,
                     tk.t[w].B + (c0 + fr) * tk.t[w].sb + fk, 8 * tk.t[w].sb);
#pragma unroll
    for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int v = 0; v < 2; ++v)
#pragma unroll
            for (int e = 0; e < 2; ++e)
                tk.dst[(r0 + 8 * u + fr) * tk.dr + (c0 + 8 * v + 2 * fk + e) * tk.dc] = tk.sign * acc[u][v][e];
}

#ifdef CP_TIMING
__device__ long long cp_ls_chain[2 * 64];  // %globaltimer (ns) at entry / exit of potrf128, per panel of the last factorisation
__device__ __forceinline__ long long ls_globaltimer() {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#define LS_CHAIN(i)                                                                      \
    do {                                                                                 \
        if (threadIdx.x == 64 && j0 / PB < 64) cp_ls_chain[2 * (j0 / PB) + (i)] = ls_globaltimer(); \
    } while (0)
__device__ long long cp_ls_times[32];
// every lane of warp 0 stores the same stamp (no divergence before the warp-synchronous pivot routine)
#define LS_STAMP(i)                                            \
    do {                                                       \
        if (threadIdx.x < 32 && j0 == 0) cp_ls_times[i] = clock64(); \
        __syncwarp();                                          \
    } while (0)
#else
#define LS_STAMP(i)
#define LS_CHAIN(i)
#endif

// A: the (updated) diagonal block in the trailing matrix; Lout: where the factor goes; Linv: 128 x 128
// row-major with leading dimension ldi (zero above the diagonal).  nb < 128 (last panel) is padded with the identity.
__global__ void __launch_bounds__(P128_T, 1)
potrf128(const double *__restrict__ A, int64_t lda, int nb, double *__restrict__ Lout, int64_t ldl,
         double *__restrict__ Linv, int64_t ldi, int32_t *__restrict__ info, double *__restrict__ ratio_out, int j0,
         const double *__restrict__ diag0) {
    extern __shared__ __align__(16) double psm[];
    double *As = psm;                             // [128][129]  lower: L ; strictly-upper blocks: (L^-1)^T
    double *Xd = As + PB * LDA_S;                 // [4][32][33] inverses of the diagonal sub-blocks
    double *Xdt = Xd + NSB * SB * LDX_S;          // the same, transposed
    double *Tt = Xdt + NSB * SB * LDX_S;          // [3][32][33] temporaries of the block inversion (transposed)
    double *rinv = Tt + 3 * SB * LDX_S;           // [128] 1 / L[k][k]
    double *thr = rinv + PB;                      // [128] pivot thresholds
    double *inv0 = thr + PB;                      // [128] 1 / original diagonal (0: not positive; -1: padding)
    double *cb = inv0 + PB;                       // [2][32] column of the pivot step, published to the whole warp
    __shared__ MmTask tasks[3];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    LS_CHAIN(0);
    LS_STAMP(0);
    // (eight loads in flight per thread: this CTA is alone on the chain, nothing else hides the memory latency)
#pragma unroll 8
    for (int e = tid; e < PB * PB; e += P128_T) {
        const int i = e >> 7, j = e & (PB - 1);
        double v = 0.0;
        if (i < nb && j <= i) v = __ldg(A + (int64_t)i * lda + j);
        else if (i >= nb && i == j) v = 1.0;
        As[i * LDA_S + j] = v;
    }
    if (tid < PB) {
        const double d0 = tid < nb ? diag0[j0 + tid] : 0.0;
        thr[tid] = tid < nb ? 1e-12 * d0 : 0.0;
        inv0[tid] = tid >= nb ? -1.0 : (d0 > 0.0 ? 1.0 / d0 : 0.0);  // an all-zero column meets the ratio 0
    }
    __syncthreads();

    double ratio_min = 1e300;
    LS_STAMP(1);
    for (int sp = 0; sp < NSB; ++sp) {
        const int k0 = sp * SB;
        LS_STAMP(2 + 4 * sp);
        if (warp == 0) potrf32_warp(As, k0, thr, rinv, info, j0, lane, ratio_min, inv0, cb);
        __syncthreads();
        LS_STAMP(3 + 4 * sp);
        const int r0 = k0 + SB, T = PB - r0;
        if (T == 0) break;
        // rows below the pivot block:  x * L32' = a  (one thread per row, right-looking over the 32 columns)
        if (tid < T) {
            double a[SB];
            double *row = As + (r0 + tid) * LDA_S + k0;
#pragma unroll
            for (int j = 0; j < SB; ++j) a[j] = row[j];
#pragma unroll
            for (int k = 0; k < SB; ++k) {
                const double x = a[k] * rinv[k0 + k];
                a[k] = x;
#pragma unroll
                for (int j = k + 1; j < SB; ++j) a[j] = fma(-x, As[(k0 + j) * LDA_S + k0 + k], a[j]);
            }
#pragma unroll
            for (int j = 0; j < SB; ++j) row[j] = a[j];
        }
        __syncthreads();
        LS_STAMP(4 + 4 * sp);
        // trailing block -= P P'  on the FP64 tensor path: one warp per 16 x 16 block of the lower triangle
        {
            const int nb16 = T >> 4, nblk = nb16 * (nb16 + 1) / 2;
            const int fr = lane >> 2, fk = lane & 3;
            for (int blk = warp; blk < nblk; blk += P128_T / 32) {
                int bj = 0, l = blk;
                while (l >= nb16 - bj) { l -= nb16 - bj; ++bj; }
                const int bi = bj + l;
                double acc[2][2][2];
#pragma unroll
                for (int u = 0; u < 2; ++u)
#pragma unroll
                    for (int v = 0; v < 2; ++v) acc[u][v][0] = acc[u][v][1] = 0.0;
                dmma_block16(acc, As + (r0 + 16 * bi + fr) * LDA_S + k0 + fk, 8 * LDA_S,
                             As + (r0 + 16 * bj + fr) * LDA_S + k0 + fk, 8 * LDA_S);
#pragma unroll
                for (int u = 0; u < 2; ++u)
#pragma unroll
                    for (int v = 0; v < 2; ++v)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int ri = r0 + 16 * bi + 8 * u + fr, cj = r0 + 16 * bj + 8 * v + 2 * fk + e;
                            if (ri >= cj) As[ri * LDA_S + cj] -= acc[u][v][e];
                        }
            }
        }
        __syncthreads();
        LS_STAMP(5 + 4 * sp);
    }
    LS_STAMP(18);
    if (warp == 0) {
#pragma unroll
        for (int off = 16; off; off >>= 1) ratio_min = fmin(ratio_min, __shfl_xor_sync(0xffffffffu, ratio_min, off));
        if (lane == 0 && ratio_min < 1e299 && ratio_out) atomic_min_pos(ratio_out, ratio_min > 0.0 ? ratio_min : 1e-300);
    }
    // ---- the factor leaves now (coalesced rows); the shared copy stays for the inversion
#pragma unroll 8
    for (int e = tid; e < PB * PB; e += P128_T) {
        const int i = e >> 7, j = e & (PB - 1);
        if (i < nb && j <= i) Lout[(int64_t)i * ldl + j] = As[i * LDA_S + j];
    }
    LS_STAMP(19);
    // ---- inverse of the four 32 x 32 diagonal sub-blocks: lane c solves L x = e_c
    if (warp < NSB) {
        const int b = warp, c = lane;
        const double *Lb = As + (b * SB) * LDA_S + b * SB;
        double x[SB];
#pragma unroll
        for (int i = 0; i < SB; ++i) x[i] = (i == c) ? 1.0 : 0.0;
#pragma unroll
        for (int j = 0; j < SB; ++j) {  // right-looking: the updates of one step are independent of each other
            const double xj = x[j] * rinv[b * SB + j];
            x[j] = xj;
#pragma unroll
            for (int i = j + 1; i < SB; ++i) x[i] = fma(-Lb[i * LDA_S + j], xj, x[i]);
        }
#pragma unroll
        for (int i = 0; i < SB; ++i) {
            Xd[(b * SB + i) * LDX_S + c] = x[i];
            Xdt[(b * SB + c) * LDX_S + i] = x[i];
        }
    }
    __syncthreads();
    LS_STAMP(20);
    // ---- off-diagonal blocks of X = L^-1, sub-diagonal by sub-diagonal:
    //      X_ij = -X_ii * sum_{k=j}^{i-1} L_ik X_kj ;  X_ij (i > j) is kept TRANSPOSED in the upper block (j, i) of As
    auto Lblk = [&](int i, int k) { return As + (i * SB) * LDA_S + k * SB; };        // L_ik[r][q]   stride LDA_S
    auto XoffT = [&](int k, int j) { return As + (j * SB) * LDA_S + k * SB; };       // X_kj[q][c] at [c][q], stride LDA_S
    for (int d = 1; d < NSB; ++d) {
        const int ntask = NSB - d;
        if (tid < ntask) {
            const int j = tid, i = j + d;
            MmTask t;
            t.dst = Tt + tid * SB * LDX_S;
            t.dr = 1; t.dc = LDX_S; t.sign = 1.0; t.nterm = d;
            for (int u = 0; u < d; ++u) {
                const int k = j + u;
                t.t[u].A = Lblk(i, k); t.t[u].sa = LDA_S;
                if (k == j) { t.t[u].B = Xdt + (j * SB) * LDX_S; t.t[u].sb = LDX_S; }
                else { t.t[u].B = XoffT(k, j); t.t[u].sb = LDA_S; }
            }
            tasks[tid] = t;
        }
        __syncthreads();
        run_tasks_mma(tasks, ntask);
        __syncthreads();
        if (tid < ntask) {
            const int j = tid, i = j + d;
            MmTask t;
            t.dst = XoffT(i, j);
            t.dr = 1; t.dc = LDA_S; t.sign = -1.0; t.nterm = 1;
            t.t[0].A = Xd + (i * SB) * LDX_S; t.t[0].sa = LDX_S;
            t.t[0].B = Tt + tid * SB * LDX_S; t.t[0].sb = LDX_S;
            tasks[tid] = t;
        }
        __syncthreads();
        run_tasks_mma(tasks, ntask);
        __syncthreads();
    }
    LS_STAMP(21);
#pragma unroll 8
    for (int e = tid; e < PB * PB; e += P128_T) {
        const int i = e >> 7, j = e & (PB - 1);
        double v = 0.0;
        if (j <= i) v = ((i >> 5) == (j >> 5)) ? Xd[((i >> 5) * SB + (i & 31)) * LDX_S + (j & 31)] : As[j * LDA_S + i];
        Linv[(int64_t)i * ldi + j] = v;
    }
    LS_STAMP(22);
    LS_CHAIN(1);
}

#ifdef CP_TIMING
}  // namespace
extern "C" int cp_debug_ls_times(long long *host_out) {  // clock64 stamps of the first panel of the last factorisation
    return (int)cudaMemcpyFromSymbol(host_out, cp_ls_times, sizeof(long long) * 32);
}
extern "C" int cp_debug_ls_chain(long long *host_out) {  // entry / exit times (ns) of every panel factorisation
    return (int)cudaMemcpyFromSymbol(host_out, cp_ls_chain, sizeof(long long) * 128);
}
namespace {
#endif

__global__ void __launch_bounds__(256)
ls_output(const double *__restrict__ Wt, int64_t ld, const double *__restrict__ sx, const double *__restrict__ sy,
          const int32_t *__restrict__ sel, int Ks, double invN, double *__restrict__ W_out,
          double *__restrict__ b_out, int accumulate) {
    __shared__ double red[256];
    const int t = blockIdx.x;
    const double *src = Wt + (int64_t)t * ld;
    double s = 0.0;
    for (int i = threadIdx.x; i < Ks; i += 256) {
        const double w = src[i];
        W_out[(int64_t)t * Ks + i] = accumulate ? W_out[(int64_t)t * Ks + i] + w : w;
        s = fma(sx[sel ? sel[i] : i], w, s);
    }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const double v = (sy[t] - red[0]) * invN;
        b_out[t] = accumulate ? b_out[t] + v : v;
    }
}

// C = alpha * a b' + beta C on the solver's fp64 operands:  a(m, r) = A[m * lda + r],
// b(nn, r) = B_NC ? B[r * ldb + nn] : B[nn * ldb + r].
// tc: the product may take the tensor cores.  With the handle's tensor-core mode on, products wide enough to fill the
// 128 x 128 tiles of the split-precision kernel (gemm_tc.cu) run there, on one operand buffer per stream of the solver.
// Everything else runs on gemm_async_kernel with tile x tile tiles (128: throughput; 64: latency, everything on the
// dependency chain).  The operands never need the register-staged kernel: every matrix here is carved 256-byte aligned
// (cp_carver, h->fac), every leading dimension is ld_for(K) or GB, and every column offset a multiple of 128.
template <bool B_NC>
int dgemm(cp_handle_t h, bool tc, int tile, int tile_mode, int max_ctas, const double *A, int64_t lda, const double *B,
          int64_t ldb, double *C, int64_t ldc, int M, int Nn, int R, double alpha, double beta, cudaStream_t stream) {
    using namespace cpgemm;
    if (tc && h->ls_tc && R >= 128 && R <= 1024 && Nn >= 192 && M >= 256 &&
        (tile_mode == TILES_ALL || tile_mode == TILES_LOWER)) {
        const int slot = stream == h->side ? 1 : (stream == h->bulk ? 2 : 0);
        return cp_gemm_tc_f64(h, slot, A, lda, B, ldb, C, ldc, M, Nn, R, alpha, beta, tile_mode == TILES_LOWER, stream,
                              max_ctas, B_NC);
    }
    const AsyncArgs g{A, lda, B, ldb, C, ldc, M, Nn, R, alpha, beta, tile_mode, max_ctas};
    CP_REQUIRE(aligned(g), "least-squares GEMM: operand not 16-byte aligned (A %p lda %lld, B %p ldb %lld)", (const void *)A,
               (long long)lda, (const void *)B, (long long)ldb);
    if (M <= 0 || Nn <= 0) return CP_OK;
    if (tile == 128) CP_GEMM_LAUNCH((launch_async<128, B_NC>(g, stream)));
    else CP_GEMM_LAUNCH((launch_async<64, B_NC>(g, stream)));
    return CP_OK;
}

// The look-ahead stream runs one priority level below the stream of the first solve on this handle (a handle serves one
// stream in the layer pipeline): behind its own chain, ahead of cheaper problems' work.
int ensure_side(cp_handle_t h, cudaStream_t stream) {
    if (!h->side) {
        int lo = 0, hi = 0, p = 0;
        CP_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));  // lo: numerically greatest = least urgent
        if (cudaStreamGetPriority(stream, &p) != cudaSuccess) {
            (void)cudaGetLastError();
            p = lo;
        }
        p = p + 1 > lo ? lo : p + 1;
        CP_CUDA(cudaStreamCreateWithPriority(&h->side, cudaStreamNonBlocking, p));
        CP_CUDA(cudaStreamCreateWithPriority(&h->bulk, cudaStreamNonBlocking, lo));
        CP_CUDA(cudaEventCreateWithFlags(&h->ev_bulk, cudaEventDisableTiming));
        CP_CUDA(cudaEventCreateWithFlags(&h->ev_panel, cudaEventDisableTiming));
        CP_CUDA(cudaEventCreateWithFlags(&h->ev_side, cudaEventDisableTiming));
    }
    return CP_OK;
}

}  // namespace

static inline int ngroups(int Kd) { return (Kd + GB - 1) / GB; }
static inline size_t xinv_elems(int Kd) { return (size_t)ngroups(Kd) * GB * GB; }

// X21 = -X22 * L21 * X11 inside one group block X (GB x GB, leading dimension GB): rows/cols [a0, a1) and [a1, a2)
// of the group hold the already inverted diagonal parts X11 and X22; L21 = the factor's rows a1..a2, columns a0..a1.
static int merge_inverse(cp_handle_t h, double *X, const double *L21, int64_t ld, int a0, int a1, int a2, double *T,
                         cudaStream_t stream) {
    using namespace cpgemm;
    const int h1 = a1 - a0, h2 = a2 - a1;
    if (h1 <= 0 || h2 <= 0) return CP_OK;
    // T = L21 * X11        (h2 x h1, inner h1)
    int rc = dgemm<true>(h, false, 64, TILES_ALL, 0, L21, ld, X + (int64_t)a0 * GB + a0, GB, T, GB, h2, h1, h1, 1.0, 0.0,
                         stream);
    if (rc) return rc;
    // X21 = -X22 * T       (h2 x h1, inner h2)
    return dgemm<true>(h, false, 64, TILES_ALL, 0, X + (int64_t)a1 * GB + a1, GB, T, GB, X + (int64_t)a1 * GB + a0, GB, h2,
                       h1, h2, -1.0, 0.0, stream);
}

// Factorisation.  M: (Kd + nrhs) x Kd (leading dimension ld): rows 0..Kd-1 an SPD matrix (lower part used, destroyed),
// rows Kd.. transposed right-hand sides (destroyed).  L (same shape, same ld) receives the factor in rows 0..Kd-1
// and the forward-substituted right-hand sides  (L^-1 Rhs)'  in rows Kd.. .  Xinv: ceil(Kd/512) blocks of 512 x 512
// that end up holding the INVERSES of the 512-wide diagonal blocks of L (the 128-wide ones come out of potrf128; they
// are merged pairwise, X21 = -X22 L21 X11, on the side stream while the factorisation proceeds); Tm: scratch of the
// same size.  The substitutions then take ceil(Kd/512) steps instead of ceil(Kd/128).
// Status: info receives the first failed pivot (1-based, 0: none), ratio the smallest pivot / original diagonal ratio,
// copied to stat_out (when not NULL) once the factorisation is complete.
// tc: the pair updates (near, near2, rest) may take the tensor cores (not in the dual path, whatever the handle's mode).
static int chol_factor(cp_handle_t h, bool tc, double *M, double *L, int64_t ld, int Kd, int nrhs, double *Xinv,
                       double *Tm, const double *diag0, int32_t *info, double *ratio, double *stat_out,
                       cudaStream_t stream) {
    using namespace cpgemm;
    const int Ktot = Kd + nrhs;
    int rc = ensure_side(h, stream);
    if (rc) return rc;
    static cp_per_device_flag potrf_configured;
    if (bool *done = potrf_configured.slot(); !*done) {
        CP_CUDA(cudaFuncSetAttribute(potrf128, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)P128_SMEM));
        *done = true;
    }
    CP_CUDA(cudaMemsetAsync(info, 0, sizeof(int32_t), stream));
    CP_CUDA(cudaMemsetAsync(ratio, 0x7f, sizeof(double), stream));  // 1.4e306: "no pivot seen yet"
    CP_CUDA(cudaMemsetAsync(Xinv, 0, xinv_elems(Kd) * sizeof(double), stream));
    // Trailing updates.  Panels are paired (e, o = e + 1).  What the chain needs next stays small and immediate:
    //   crit(p)   : block column p+1, inner dimension 128, on the caller's stream, 64 x 64 tiles
    //   far_a(e)  : block column e+2 (needed by crit(o)), side stream
    // everything else is applied once per PAIR with inner dimension 256 -- half the read-modify-write traffic of
    // the trailing matrix per flop (a rank-128 update moves 8 bytes per 8 flop: memory bound on a 37 TF/s pipe):
    //   near(e,o) : block columns e+3, e+4 (the next pair's crit / far_a targets), side stream, then an event
    //   near2(e,o): block columns e+5, e+6 (the next pair's near targets), side stream
    //   rest(e,o) : block columns >= e+7, BULK stream, capped grid
    // The side stream is a FIFO the chain waits on: with the bulk update in it, far_a of the next pair queued behind a
    // ~250 us kernel and every second panel stalled (in-kernel chain timeline: 219 us instead of 30 us between panels).
    // Every update of a block column by different panels is ordered (same stream, or through ev_side / ev_panel /
    // ev_bulk): near2(e,o) and rest(e-2,o-2) touch the same columns, so the side stream waits for the previous pair's
    // bulk update there -- five panels after that update was issued.
    bool side_pending = false, bulk_pending = false;
    int ip = 0;
    for (int j0 = 0; j0 < Kd; j0 += PB, ++ip) {
        const int nb = Kd - j0 < PB ? Kd - j0 : PB;
        const int j1 = j0 + nb;
        const int g0 = j0 / GB * GB, og = (j0 - g0) / PB;   // group origin, panel index inside the group
        double *Xg = Xinv + (size_t)(j0 / GB) * GB * GB;
        double *Lp = Xg + (int64_t)(j0 - g0) * GB + (j0 - g0);
        potrf128<<<1, P128_T, P128_SMEM, stream>>>(M + (int64_t)j0 * ld + j0, ld, nb, L + (int64_t)j0 * ld + j0, ld, Lp, GB,
                                                   info, ratio, j0, diag0);
        CP_CHECK_LAUNCH();
        const int below = Ktot - j1;
        if (below > 0) {
            // block column of the factor: rows below * L_d^-T  (right-hand-side rows included)
            rc = dgemm<false>(h, false, 64, TILES_ALL, 0, M + (int64_t)j1 * ld + j0, ld, Lp, GB, L + (int64_t)j1 * ld + j0,
                              ld, below, nb, nb, 1.0, 0.0, stream);
            if (rc) return rc;
        }
        const int ncols = Kd - j1;
        const int w2 = ncols < PB ? ncols : PB;            // block column p+1
        const bool more = ncols > w2;                      // block columns beyond p+1 exist
        const bool last_in_group = (og == GB / PB - 1) || j1 >= Kd;
        const bool merges = (og & 1) || last_in_group;     // this panel completes a pair and / or its group
        if (more || merges) {
            CP_CUDA(cudaEventRecord(h->ev_panel, stream));  // block column j0..j1 of L and its inverse are final
            CP_CUDA(cudaStreamWaitEvent(h->side, h->ev_panel, 0));
        }
        if (merges) {  // inverse blocks of the group, off the critical path
            double *Tg = Tm + (size_t)(j0 / GB) * GB * GB;
            const int ge = (j1 - g0);  // columns of the group factored so far
            if (og & 1) {              // pair (og-1, og): [a0, a0+128) and [a0+128, ge)
                const int a0 = (og - 1) * PB;
                rc = merge_inverse(h, Xg, L + (int64_t)(g0 + a0 + PB) * ld + g0 + a0, ld, a0, a0 + PB, ge, Tg, h->side);
                if (rc) return rc;
            }
            if (last_in_group && ge > 2 * PB) {  // halves [0, 256) and [256, ge)
                rc = merge_inverse(h, Xg, L + (int64_t)(g0 + 2 * PB) * ld + g0, ld, 0, 2 * PB, ge, Tg, h->side);
                if (rc) return rc;
            }
        }
        if (ncols <= 0) break;
        const bool odd = (ip & 1) != 0;
        if (side_pending) {  // far_a(e) before crit(o); near(e-2, e-1) before crit(e)
            CP_CUDA(cudaStreamWaitEvent(stream, h->ev_side, 0));
            side_pending = false;
        }
        const double *Pn = L + (int64_t)j1 * ld + j0;
        rc = dgemm<false>(h, false, 64, TILES_LOWER, 0, Pn, ld, Pn, ld, M + (int64_t)j1 * ld + j1, ld, Ktot - j1, w2, nb,
                          -1.0, 1.0, stream);
        if (rc) return rc;
        if (!more) continue;
        const int j2 = j1 + w2;
        if (!odd) {
            const int w3 = Kd - j2 < PB ? Kd - j2 : PB;
            const double *Pf = L + (int64_t)j2 * ld + j0;
            rc = dgemm<false>(h, tc, 128, TILES_LOWER, 0, Pf, ld, Pf, ld, M + (int64_t)j2 * ld + j2, ld, Ktot - j2, w3, nb,
                              -1.0, 1.0, h->side);
            if (rc) return rc;
            CP_CUDA(cudaEventRecord(h->ev_side, h->side));
            side_pending = true;
        } else {
            // pair (e, o): columns [j0 - PB, j1) of L, inner dimension PB + nb; targets: block columns >= o + 2 = j2
            const int je = j0 - PB, R2 = PB + nb;
            const int wn = Kd - j2 < 2 * PB ? Kd - j2 : 2 * PB;  // near: the next pair's two block columns
            const double *Pq = L + (int64_t)j2 * ld + je;
            rc = dgemm<false>(h, tc, 128, TILES_LOWER, 0, Pq, ld, Pq, ld, M + (int64_t)j2 * ld + j2, ld, Ktot - j2, wn, R2,
                              -1.0, 1.0, h->side);
            if (rc) return rc;
            CP_CUDA(cudaEventRecord(h->ev_side, h->side));
            side_pending = true;
            const int j4 = j2 + wn;
            if (Kd - j4 > 0) {
                if (bulk_pending) {  // rest(e-2, o-2) updates these columns too
                    CP_CUDA(cudaStreamWaitEvent(h->side, h->ev_bulk, 0));
                    bulk_pending = false;
                }
                const int wm = Kd - j4 < 2 * PB ? Kd - j4 : 2 * PB;
                const double *P4 = L + (int64_t)j4 * ld + je;
                rc = dgemm<false>(h, tc, 128, TILES_LOWER, 0, P4, ld, P4, ld, M + (int64_t)j4 * ld + j4, ld, Ktot - j4, wm,
                                  R2, -1.0, 1.0, h->side);
                if (rc) return rc;
                const int j6 = j4 + wm;
                if (Kd - j6 > 0) {
                    // the bulk of the trailing update has slack; its long-running tiles must not take every SM either,
                    // or the chain's small kernels queue behind them: two thirds of the SMs
                    CP_CUDA(cudaStreamWaitEvent(h->bulk, h->ev_panel, 0));
                    const double *Pr = L + (int64_t)j6 * ld + je;
                    rc = dgemm<false>(h, tc, 128, TILES_LOWER, h->num_sms * 2 / 3, Pr, ld, Pr, ld, M + (int64_t)j6 * ld + j6,
                                      ld, Ktot - j6, Kd - j6, R2, -1.0, 1.0, h->bulk);
                    if (rc) return rc;
                    CP_CUDA(cudaEventRecord(h->ev_bulk, h->bulk));
                    bulk_pending = true;
                }
            }
        }
    }
    // whatever the side streams still hold (last merges, last bulk update: its targets were all consumed by later
    // updates on the side stream, but the scratch must not be reused under it) is ordered before the next user
    CP_CUDA(cudaEventRecord(h->ev_side, h->side));
    CP_CUDA(cudaStreamWaitEvent(stream, h->ev_side, 0));
    CP_CUDA(cudaEventRecord(h->ev_bulk, h->bulk));
    CP_CUDA(cudaStreamWaitEvent(stream, h->ev_bulk, 0));
    if (stat_out) CP_CUDA(cudaMemcpyAsync(stat_out, ratio, sizeof(double), cudaMemcpyDeviceToDevice, stream));
    return CP_OK;
}

// The bulk update of a substitution step, C (n x Nn) -= A (n x R) b' (b as in dgemm).  tc: it may take the tensor cores.
// Few right-hand sides: 128 x 128 tiles would leave most SMs idle on a 512-deep product, 64 x 64 tiles fill them.
// Tensor-core mode: split-precision tiles (n >= 256 right-hand sides, a few column tiles) beat the fp64 pipe.
template <bool B_NC>
static int subst_update(cp_handle_t h, bool tc, const double *A, int64_t lda, const double *B, int64_t ldb, double *C,
                        int64_t ldc, int n, int Nn, int R, cudaStream_t stream) {
    using namespace cpgemm;
    const bool use_tc = tc && h->ls_tc && n >= 256 && Nn >= 512;
    const int tile = use_tc || num_tiles(n, Nn, TILES_ALL, BM) >= 2 * h->num_sms ? 128 : 64;
    return dgemm<B_NC>(h, use_tc, tile, TILES_ALL, 0, A, lda, B, ldb, C, ldc, n, Nn, R, -1.0, 1.0, stream);
}

// Forward substitution of further right-hand sides: Zt (n x Kd, ld) is destroyed, F (n x Kd, ld) receives (L^-1 Rhs)'.
static int chol_forward(cp_handle_t h, const double *L, int64_t ld, int Kd, const double *Xinv, double *Zt, double *F,
                        int64_t ldz, int n, cudaStream_t stream) {
    using namespace cpgemm;
    for (int g0 = 0; g0 < Kd; g0 += GB) {
        const int gs = Kd - g0 < GB ? Kd - g0 : GB;
        const int g1 = g0 + gs;
        const double *Xg = Xinv + (size_t)(g0 / GB) * GB * GB;
        // F_g = Zt_g * Xinv_g'   (C[t, i] = sum_r Zt[t, g0 + r] * Xinv_g[i, r])
        int rc = dgemm<false>(h, false, 64, TILES_ALL, 0, Zt + g0, ldz, Xg, GB, F + g0, ldz, n, gs, gs, 1.0, 0.0, stream);
        if (rc) return rc;
        if (Kd - g1 > 0) {  // Zt[:, g1:] -= F_g * L[g1:, g0:g1]'
            rc = subst_update<false>(h, true, F + g0, ldz, L + (int64_t)g1 * ld + g0, ld, Zt + g1, ldz, n, Kd - g1, gs,
                                     stream);
            if (rc) return rc;
        }
    }
    return CP_OK;
}

// Backward substitution: F (n x Kd, ldf; destroyed) holds (L^-1 Rhs)'; Wt (n x Kd, ldw) receives (SPD^-1 Rhs)'.
// tc: the bulk products may take the tensor cores (not in the dual path, whatever the handle's mode).
static int chol_backward(cp_handle_t h, bool tc, const double *L, int64_t ld, int Kd, const double *Xinv, double *F,
                         int64_t ldf, double *Wt, int64_t ldw, int n, cudaStream_t stream) {
    using namespace cpgemm;
    for (int g = ngroups(Kd) - 1; g >= 0; --g) {
        const int g0 = g * GB;
        const int gs = Kd - g0 < GB ? Kd - g0 : GB;
        const double *Xg = Xinv + (size_t)g * GB * GB;
        // Wt_g = F_g * Xinv_g   (C[t, i] = sum_r F[t, g0 + r] * Xinv_g[r, i])
        int rc = dgemm<true>(h, false, 64, TILES_ALL, 0, F + g0, ldf, Xg, GB, Wt + g0, ldw, n, gs, gs, 1.0, 0.0, stream);
        if (rc) return rc;
        if (g0 > 0) {  // F[:, 0:g0] -= Wt_g * L[g0:g0+gs, 0:g0]
            rc = subst_update<true>(h, tc, Wt + g0, ldw, L + (int64_t)g0 * ld, ld, F, ldf, n, g0, gs, stream);
            if (rc) return rc;
        }
    }
    return CP_OK;
}

static inline int64_t ld_for(int K) { return (K + 7) / 8 * 8; }

// The kept factor (h->fac) lives in the handle's own allocation, not in the shared scratch: it must survive the calls
// that follow a solve (refinement against the same factor, cp_ls_resolve), and every other entry point reuses the
// scratch.  Layout: L (rows x ld_for(Kd)), the inverted 512-wide diagonal blocks, their scratch, the pivot ratio.
struct FacParts {
    double *L, *Linv, *Tm, *ratio;
};
static size_t fac_bytes(size_t rows, int Kd) {
    return cp_carver::need(rows * ld_for(Kd), 8) + 2 * cp_carver::need(xinv_elems(Kd), 8) + cp_carver::need(1, 8);
}
static FacParts fac_carve(void *base, size_t rows, int Kd) {
    cp_carver fc(base);
    FacParts p;
    p.L = fc.take<double>(rows * ld_for(Kd));
    p.Linv = fc.take<double>(xinv_elems(Kd));
    p.Tm = fc.take<double>(xinv_elems(Kd));
    p.ratio = fc.take<double>(1);
    return p;
}

// Assembles the centred Gram of the selected columns, with the n right-hand sides of Bxy as rows under it when Bxy is
// given, factors it into the kept factor and records that on the handle, for cp_ls_resolve or the rest of
// cp_ls_solve.  A call that fails leaves the handle without a factor.  Wt: n x ld_for(Ksel) of scratch for the caller.
static int factor_and_keep(cp_handle_t h, const double *G, const double *Bxy, const double *sx, const double *sy,
                           int64_t N, int K, int n, const int32_t *sel_cols, int Ksel, int32_t *info_out,
                           double *stat_out, cudaStream_t stream, FacParts *fac, double **Wt) {
    h->fac.K = 0;
    const int64_t ld = ld_for(Ksel);
    const size_t rows = (size_t)(Ksel + n);
    int rc = cp_buffer_reserve(h->fac.buf, fac_bytes(rows, Ksel), 8, "factor allocation");
    if (rc) return rc;
    *fac = fac_carve(h->fac.buf.ptr, rows, Ksel);
    void *ws = nullptr;
    rc = cp_ws_reserve(h, cp_carver::need(rows * ld, 8) + cp_carver::need((size_t)n * ld, 8) + cp_carver::need(Ksel, 8),
                       &ws);
    if (rc) return rc;
    cp_carver cv(ws);
    double *M = cv.take<double>(rows * ld);
    *Wt = cv.take<double>((size_t)n * ld);
    double *diag0 = cv.take<double>(Ksel);
    ls_assemble<<<dim3(cp_cdiv(Ksel, 256), Ksel + n), 256, 0, stream>>>(G, Bxy, sx, sy, 1.0 / (double)N, K, n, sel_cols,
                                                                       Ksel, M, ld, diag0);
    CP_CHECK_LAUNCH();
    rc = chol_factor(h, true, M, fac->L, ld, Ksel, n, fac->Linv, fac->Tm, diag0, info_out, fac->ratio, stat_out, stream);
    if (rc) return rc;
    h->fac.K = Ksel;
    h->fac.Kfull = K;
    h->fac.N = N;
    h->fac.rows = Ksel + n;
    return CP_OK;
}

extern "C" int cp_ls_solve(cp_handle_t h, const double *G, const double *Bxy, const double *sx, const double *sy,
                           int64_t N, int K, int n, const int32_t *sel_cols, int Ksel, double *W_out, double *b_out,
                           int32_t *info_out, double *stat_out, cp_stream_t stream_) {
    CP_REQUIRE(h && G && Bxy && sx && sy && W_out && b_out && info_out, "cp_ls_solve: NULL argument");
    CP_REQUIRE(K > 0 && n > 0 && Ksel > 0 && Ksel <= K && N > 0, "cp_ls_solve: bad shape");
    CP_REQUIRE(sel_cols || Ksel == K, "cp_ls_solve: sel_cols may be NULL only when every column is used");
    CP_REQUIRE(N - 1 >= Ksel, "cp_ls_solve: N-1=%lld < K'=%d: centred Gram is singular, use cp_ls_solve_dual",
               (long long)(N - 1), Ksel);
    CP_DEVICE_GUARD(h);
    cudaStream_t stream = (cudaStream_t)stream_;
    FacParts f;
    double *Wt = nullptr;
    int rc = factor_and_keep(h, G, Bxy, sx, sy, N, K, n, sel_cols, Ksel, info_out, stat_out, stream, &f, &Wt);
    if (rc) return rc;
    const int64_t ld = ld_for(Ksel);
    rc = chol_backward(h, true, f.L, ld, Ksel, f.Linv, f.L + (int64_t)Ksel * ld, ld, Wt, ld, n, stream);
    if (rc) return rc;
    ls_output<<<n, 256, 0, stream>>>(Wt, ld, sx, sy, sel_cols, Ksel, 1.0 / (double)N, W_out, b_out, 0);
    CP_CHECK_LAUNCH();
    return CP_OK;
}

// ---------------------------------------------------------------- factor once, solve many (nonlinear_fc)
extern "C" int cp_ls_factor(cp_handle_t h, const double *G, const double *sx, int64_t N, int K,
                            const int32_t *sel_cols, int Ksel, int32_t *info_out, double *stat_out,
                            cp_stream_t stream_) {
    CP_REQUIRE(h && G && sx && info_out, "cp_ls_factor: NULL argument");
    CP_REQUIRE(K > 0 && Ksel > 0 && Ksel <= K && N > 0, "cp_ls_factor: bad shape");
    CP_REQUIRE(sel_cols || Ksel == K, "cp_ls_factor: sel_cols may be NULL only when every column is used");
    CP_REQUIRE(N - 1 >= Ksel, "cp_ls_factor: N-1=%lld < K'=%d: centred Gram is singular", (long long)(N - 1), Ksel);
    CP_DEVICE_GUARD(h);
    FacParts f;
    double *Wt = nullptr;
    return factor_and_keep(h, G, nullptr, sx, nullptr, N, K, 0, sel_cols, Ksel, info_out, stat_out,
                           (cudaStream_t)stream_, &f, &Wt);
}

namespace {
// rows of the right-hand sides, transposed and centred: Zt[t, j] = Bxy[sel_j, t] - sx[sel_j] sy[t] / N
__global__ void __launch_bounds__(256)
rhs_assemble(const double *__restrict__ Bxy, const double *__restrict__ sx, const double *__restrict__ sy, double invN,
             int n, const int32_t *__restrict__ sel, int Ks, double *__restrict__ Zt, int64_t ld) {
    const int j = blockIdx.x * 256 + threadIdx.x;
    const int t = blockIdx.y;
    if (j >= Ks) return;
    Zt[(int64_t)t * ld + j] = centred_rhs(Bxy, sx, sy, invN, n, sel ? sel[j] : j, t);
}
}  // namespace

extern "C" int cp_ls_resolve(cp_handle_t h, const double *Bxy, const double *sx, const double *sy, int n,
                             const int32_t *sel_cols, double *W_out, double *b_out, int accumulate,
                             cp_stream_t stream_) {
    CP_REQUIRE(h && Bxy && sx && sy && W_out && b_out, "cp_ls_resolve: NULL argument");
    CP_REQUIRE(h->fac.K > 0, "cp_ls_resolve: no factor on this handle (call cp_ls_factor first)");
    CP_REQUIRE(n > 0, "cp_ls_resolve: bad shape");
    CP_REQUIRE(sel_cols || h->fac.K == h->fac.Kfull, "cp_ls_resolve: sel_cols needed (the factor used a column subset)");
    CP_DEVICE_GUARD(h);
    cudaStream_t stream = (cudaStream_t)stream_;
    const int Ksel = h->fac.K;
    const int64_t ld = ld_for(Ksel);
    const FacParts f = fac_carve(h->fac.buf.ptr, h->fac.rows, Ksel);
    void *ws = nullptr;
    int rc = cp_ws_reserve(h, 3 * cp_carver::need((size_t)n * ld, 8), &ws);
    if (rc) return rc;
    cp_carver cv(ws);
    double *Zt = cv.take<double>((size_t)n * ld);
    double *F = cv.take<double>((size_t)n * ld);
    double *Wt = cv.take<double>((size_t)n * ld);
    const double invN = 1.0 / (double)h->fac.N;
    rhs_assemble<<<dim3(cp_cdiv(Ksel, 256), n), 256, 0, stream>>>(Bxy, sx, sy, invN, n, sel_cols, Ksel, Zt, ld);
    CP_CHECK_LAUNCH();
    rc = chol_forward(h, f.L, ld, Ksel, f.Linv, Zt, F, ld, n, stream);
    if (rc) return rc;
    rc = chol_backward(h, true, f.L, ld, Ksel, f.Linv, F, ld, Wt, ld, n, stream);
    if (rc) return rc;
    ls_output<<<n, 256, 0, stream>>>(Wt, ld, sx, sy, sel_cols, Ksel, invN, W_out, b_out, accumulate);
    CP_CHECK_LAUNCH();
    return CP_OK;
}

// ---------------------------------------------------------------- residual of a solve (iterative refinement)
namespace {
// Wf (n x K, zero for unselected columns) <- W (n x Ksel)
__global__ void __launch_bounds__(256)
scatter_cols(const double *__restrict__ W, int Ks, const int32_t *__restrict__ sel, double *__restrict__ Wf, int K) {
    const int j = blockIdx.x * 256 + threadIdx.x;
    const int t = blockIdx.y;
    if (j < Ks) Wf[(int64_t)t * K + (sel ? sel[j] : j)] = W[(int64_t)t * Ks + j];
}
// Xt[k, r] = X[r, k]   (fp32, 32 x 32 tiles through shared memory: both sides coalesced)
__global__ void __launch_bounds__(256)
transpose_f32(const float *__restrict__ X, int64_t ldx, int64_t N, int K, float *__restrict__ Xt, int64_t ldt) {
    __shared__ float tile[32][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int64_t r0 = (int64_t)blockIdx.x * 32;
    const int k0 = blockIdx.y * 32;
    for (int q = ty; q < 32; q += 8)
        if (r0 + q < N && k0 + tx < K) tile[q][tx] = X[(r0 + q) * ldx + k0 + tx];
    __syncthreads();
    for (int q = ty; q < 32; q += 8)
        if (k0 + q < K && r0 + tx < N) Xt[(int64_t)(k0 + q) * ldt + r0 + tx] = tile[tx][q];
}
// WfT[sel_j, t] = (float) W[t, j]   (K x n fp32, zero rows for unselected columns)
__global__ void __launch_bounds__(256)
scatter_cols_t(const double *__restrict__ W, int Ks, const int32_t *__restrict__ sel, float *__restrict__ WfT, int n) {
    const int t = blockIdx.x * 256 + threadIdx.x;
    const int j = blockIdx.y;
    if (t < n) WfT[(int64_t)(sel ? sel[j] : j) * n + t] = (float)W[(int64_t)t * Ks + j];
}
// R[r, t] = float( (Y[r, t] - y_bias[t] - b[t]) - sum_k part_k[r, t] )
template <typename T>
__global__ void __launch_bounds__(256)
residual_finish(const T *__restrict__ Y, int64_t ldy, const float *__restrict__ y_bias, const double *__restrict__ b,
                const double *__restrict__ part, int64_t split_stride, int nsplit, int64_t N, int n, float *__restrict__ R,
                int64_t ldr) {
    const int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (e >= N * n) return;
    const int64_t r = e / n;
    const int t = (int)(e - r * n);
    double acc = 0.0;
    for (int k = 0; k < nsplit; ++k) acc += part[(int64_t)k * split_stride + e];
    const double y0 = (double)Y[r * ldy + t] - ((y_bias ? (double)y_bias[t] : 0.0) + b[t]);
    R[r * ldr + t] = (float)(y0 - acc);
}
}  // namespace

extern "C" int cp_ls_residual(cp_handle_t h, const float *X, int64_t N, int K, int64_t ldx, const void *Yraw, int y_dtype,
                              int n, int64_t ldy, const float *y_bias, const int32_t *sel_cols, int Ksel, const double *W,
                              const double *b, float *R_out, int64_t ldr, int mode, cp_stream_t stream_) {
    using namespace cpgemm;
    CP_REQUIRE(h && X && Yraw && W && b && R_out, "cp_ls_residual: NULL argument");
    CP_REQUIRE(N > 0 && K > 0 && n > 0 && Ksel > 0 && Ksel <= K && ldx >= K && ldy >= n && ldr >= n, "cp_ls_residual: bad shape");
    CP_REQUIRE(sel_cols || Ksel == K, "cp_ls_residual: sel_cols may be NULL only when every column is used");
    CP_REQUIRE(y_dtype == CP_F32 || y_dtype == CP_F64, "cp_ls_residual: unknown y_dtype %d", y_dtype);
    CP_REQUIRE(mode == CP_GRAM_FP64 || mode == CP_GRAM_3XTF32, "cp_ls_residual: unknown mode %d", mode);
    CP_DEVICE_GUARD(h);
    cudaStream_t stream = (cudaStream_t)stream_;
    if (mode == CP_GRAM_3XTF32 && N % 4 == 0 && N >= 128 && K >= 64 && n % 4 == 0) {
        // Tensor-core variant: X Wf' = (X')'(Wf') is a product of the cp_gram shape (reduction over the ROWS of both
        // operands) once X is transposed: split precision on the tensor cores instead of 2 N K n flops on the FP64 pipe.  Its
        // ~4e-7 relative error in the prediction perturbs the correction ~sqrt(N) times less than the same relative
        // error in the Gram matrix did (the residual error is uncorrelated noise, not a structured change of G).
        const int64_t ldt = N;
        void *aux = nullptr;
        int rc = cp_aux_reserve(h, cp_carver::need((size_t)K * ldt, 4) + cp_carver::need((size_t)K * n, 4) +
                                       cp_carver::need((size_t)N * n, 8), &aux);
        if (rc) return rc;
        cp_carver cv(aux);
        float *Xt = cv.take<float>((size_t)K * ldt);
        float *WfT = cv.take<float>((size_t)K * n);
        double *P = cv.take<double>((size_t)N * n);
        transpose_f32<<<dim3(cp_cdiv(N, 32), cp_cdiv(K, 32)), 256, 0, stream>>>(X, ldx, N, K, Xt, ldt);
        CP_CHECK_LAUNCH();
        CP_CUDA(cudaMemsetAsync(WfT, 0, (size_t)K * n * sizeof(float), stream));
        scatter_cols_t<<<dim3(cp_cdiv(n, 256), Ksel), 256, 0, stream>>>(W, Ksel, sel_cols, WfT, n);
        CP_CHECK_LAUNCH();
        rc = cp_gram(h, Xt, K, (int)N, ldt, WfT, CP_F32, n, n, nullptr, nullptr, 0, nullptr, P, nullptr, nullptr, nullptr,
                     CP_GRAM_3XTF32, stream_);
        if (rc) return rc;
        const int64_t count = N * (int64_t)n;
        const unsigned nblk = (unsigned)((count + 255) / 256);
        if (y_dtype == CP_F32)
            residual_finish<float><<<nblk, 256, 0, stream>>>((const float *)Yraw, ldy, y_bias, b, P, 0, 1, N, n, R_out, ldr);
        else
            residual_finish<double><<<nblk, 256, 0, stream>>>((const double *)Yraw, ldy, y_bias, b, P, 0, 1, N, n, R_out, ldr);
        CP_CHECK_LAUNCH();
        return CP_OK;
    }
    const int64_t ldw = ld_for(K);
    // X Wf' in fp64 (exact products of fp32 data with the fp64 weights): 128 x 128 tiles, reduction split so that the
    // tile count fills whole waves of the SMs (5000 x 512 is 160 tiles on 132 SMs: two waves for 1.2 waves of work)
    const int tiles = num_tiles((int)N, n, TILES_ALL, BM);
    int nsplit = 1;
    double best = 1e30;
    for (int ns = 1; ns <= 6; ++ns) {
        if (K / ns < 8 * BK) break;
        const double cost = (double)cp_cdiv((int64_t)tiles * ns, h->num_sms) / ns + 0.02 * ns;  // waves of 1/ns length
        if (cost < best) {
            best = cost;
            nsplit = ns;
        }
    }
    int64_t rps = (K + nsplit - 1) / nsplit;
    rps = (rps + BK - 1) / BK * BK;
    nsplit = (int)((K + rps - 1) / rps);
    void *ws = nullptr;
    int rc = cp_ws_reserve(h, cp_carver::need((size_t)n * ldw, 8) + cp_carver::need((size_t)nsplit * N * n, 8), &ws);
    if (rc) return rc;
    cp_carver cv(ws);
    double *Wf = cv.take<double>((size_t)n * ldw);
    double *part = cv.take<double>((size_t)nsplit * N * n);
    CP_CUDA(cudaMemsetAsync(Wf, 0, (size_t)n * ldw * sizeof(double), stream));
    scatter_cols<<<dim3(cp_cdiv(Ksel, 256), n), 256, 0, stream>>>(W, Ksel, sel_cols, Wf, (int)ldw);
    CP_CHECK_LAUNCH();
    Args g{};
    g.A = X; g.lda = ldx; g.B = Wf; g.ldb = ldw; g.C = part; g.ldc = n;
    g.c_split_stride = N * (int64_t)n;
    g.M = (int)N; g.Nn = n; g.R = K;
    g.nsplit = nsplit > 1 ? nsplit : 1;
    g.r_per_split = nsplit > 1 ? rps : K;
    g.alpha = 1.0; g.beta = 0.0; g.tile_mode = TILES_ALL;
    g.a_vec = cp_aligned16(X) && (ldx % 4 == 0);
    g.b_vec = cp_aligned16(Wf) && (ldw % 2 == 0);
    CP_GEMM_LAUNCH((launch<float, double, false, false>(g, stream)));
    const int64_t count = N * (int64_t)n;
    const unsigned nblk = (unsigned)((count + 255) / 256);
    if (y_dtype == CP_F32)
        residual_finish<float><<<nblk, 256, 0, stream>>>((const float *)Yraw, ldy, y_bias, b, part, g.c_split_stride, g.nsplit,
                                                        N, n, R_out, ldr);
    else
        residual_finish<double><<<nblk, 256, 0, stream>>>((const double *)Yraw, ldy, y_bias, b, part, g.c_split_stride,
                                                         g.nsplit, N, n, R_out, ldr);
    CP_CHECK_LAUNCH();
    return CP_OK;
}

// ---------------------------------------------------------------- dual (minimum-norm) path
namespace {

// column means of the selected columns of X (fp64, fixed order) and of Y - bias
template <typename T>
__global__ void __launch_bounds__(256)
colmean_sel(const T *__restrict__ X, int64_t ld, const int32_t *__restrict__ sel, int ncols, int64_t N,
            const float *__restrict__ bias, double *__restrict__ mean_out) {
    __shared__ double s1[8][33];
    const int cx = threadIdx.x & 31, rg = threadIdx.x >> 5;
    const int j = blockIdx.x * 32 + cx;
    double a = 0.0;
    if (j < ncols) {
        const int col = sel ? sel[j] : j;
        const double b = bias ? (double)bias[col] : 0.0;
        for (int64_t r = rg; r < N; r += 8) a += (double)__ldg(X + r * ld + col) - b;
    }
    s1[rg][cx] = a;
    __syncthreads();
    if (rg == 0 && j < ncols) {
        double t = 0.0;
#pragma unroll
        for (int k = 0; k < 8; ++k) t += s1[k][cx];
        mean_out[j] = t / (double)N;
    }
}

// Xc[r, j] = X[r, sel_j] - mean_j    (N x Ks fp64, ld)
__global__ void __launch_bounds__(256)
center_sel(const float *__restrict__ X, int64_t ldx, const int32_t *__restrict__ sel, int Ks,
           const double *__restrict__ mean, double *__restrict__ Xc, int64_t ld) {
    const int j = blockIdx.x * 256 + threadIdx.x;
    const int64_t r = blockIdx.y;
    if (j < Ks) Xc[r * ld + j] = (double)__ldg(X + r * ldx + (sel ? sel[j] : j)) - mean[j];
}

// rows N..N+n-1 of the augmented matrix: Yc' (n x N):  M[N + t, r] = Y[r, t] - bias_t - ymean_t
template <typename T>
__global__ void __launch_bounds__(256)
dual_rhs(const T *__restrict__ Y, int64_t ldy, const float *__restrict__ bias, const double *__restrict__ ymean,
         int64_t N, int n, double *__restrict__ M, int64_t ld) {
    const int64_t r = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int t = blockIdx.y;
    if (r < N) M[(N + t) * ld + r] = (double)__ldg(Y + r * ldy + t) - (bias ? (double)bias[t] : 0.0) - ymean[t];
}

__global__ void add_const_lower(double *__restrict__ M, int64_t ld, int N, double v, double *__restrict__ diag0) {
    const int j = blockIdx.x * 256 + threadIdx.x;
    const int i = blockIdx.y;
    if (j < N && j <= i) {
        const double x = M[(int64_t)i * ld + j] + v;
        M[(int64_t)i * ld + j] = x;
        if (i == j) diag0[i] = x;
    }
}

}  // namespace

extern "C" int cp_ls_solve_dual(cp_handle_t h, const float *X, int64_t N, int K, int64_t ldx, const void *Yraw,
                                int y_dtype, int n, int64_t ldy, const float *y_bias, const int32_t *sel_cols, int Ksel,
                                double *W_out, double *b_out, int32_t *info_out, double *stat_out, cp_stream_t stream_) {
    using namespace cpgemm;
    CP_REQUIRE(h && X && Yraw && W_out && b_out && info_out, "cp_ls_solve_dual: NULL argument");
    CP_REQUIRE(N > 1 && N < (1 << 15) && K > 0 && n > 0 && Ksel > 0 && Ksel <= K && ldx >= K && ldy >= n,
               "cp_ls_solve_dual: bad shape (N must be < 32768)");
    CP_REQUIRE(sel_cols || Ksel == K, "cp_ls_solve_dual: sel_cols may be NULL only when every column is used");
    CP_REQUIRE(y_dtype == CP_F32 || y_dtype == CP_F64, "cp_ls_solve_dual: unknown y_dtype %d", y_dtype);
    CP_DEVICE_GUARD(h);
    cudaStream_t stream = (cudaStream_t)stream_;
    const int Ni = (int)N;
    const int64_t ldc = ld_for(Ksel);  // Xc
    const int64_t ldm = ld_for(Ni);    // dual system
    const size_t nM = (size_t)(Ni + n) * ldm;
    const size_t need = cp_carver::need((size_t)Ni * ldc, 8) + 2 * cp_carver::need(nM, 8) +
                        2 * cp_carver::need(xinv_elems(Ni), 8) + cp_carver::need((size_t)n * ldm, 8) +
                        cp_carver::need((size_t)n * ldc, 8) + cp_carver::need(Ksel, 8) + cp_carver::need(n, 8) +
                        cp_carver::need(Ni, 8) + cp_carver::need(1, 8);
    void *ws = nullptr;
    int rc = cp_ws_reserve(h, need, &ws);
    if (rc) return rc;
    cp_carver cv(ws);
    double *Xc = cv.take<double>((size_t)Ni * ldc);
    double *M = cv.take<double>(nM);
    double *L = cv.take<double>(nM);
    double *Linv = cv.take<double>(xinv_elems(Ni));
    double *Tm = cv.take<double>(xinv_elems(Ni));
    double *At = cv.take<double>((size_t)n * ldm);
    double *Wt = cv.take<double>((size_t)n * ldc);
    double *xmean = cv.take<double>(Ksel);
    double *ymean = cv.take<double>(n);
    double *diag0 = cv.take<double>(Ni);
    double *ratio = cv.take<double>(1);
    colmean_sel<float><<<cp_cdiv(Ksel, 32), 256, 0, stream>>>(X, ldx, sel_cols, Ksel, N, nullptr, xmean);
    CP_CHECK_LAUNCH();
    if (y_dtype == CP_F32)
        colmean_sel<float><<<cp_cdiv(n, 32), 256, 0, stream>>>((const float *)Yraw, ldy, nullptr, n, N, y_bias, ymean);
    else
        colmean_sel<double><<<cp_cdiv(n, 32), 256, 0, stream>>>((const double *)Yraw, ldy, nullptr, n, N, y_bias, ymean);
    CP_CHECK_LAUNCH();
    center_sel<<<dim3(cp_cdiv(Ksel, 256), Ni), 256, 0, stream>>>(X, ldx, sel_cols, Ksel, xmean, Xc, ldc);
    CP_CHECK_LAUNCH();
    // H = Xc Xc' (lower tiles) + 1/N
    rc = dgemm<false>(h, false, 128, TILES_LOWER, 0, Xc, ldc, Xc, ldc, M, ldm, Ni, Ni, Ksel, 1.0, 0.0, stream);
    if (rc) return rc;
    add_const_lower<<<dim3(cp_cdiv(Ni, 256), Ni), 256, 0, stream>>>(M, ldm, Ni, 1.0 / (double)N, diag0);
    CP_CHECK_LAUNCH();
    if (y_dtype == CP_F32)
        dual_rhs<float><<<dim3(cp_cdiv(Ni, 256), n), 256, 0, stream>>>((const float *)Yraw, ldy, y_bias, ymean, N, n, M, ldm);
    else
        dual_rhs<double><<<dim3(cp_cdiv(Ni, 256), n), 256, 0, stream>>>((const double *)Yraw, ldy, y_bias, ymean, N, n, M, ldm);
    CP_CHECK_LAUNCH();
    rc = chol_factor(h, false, M, L, ldm, Ni, n, Linv, Tm, diag0, info_out, ratio, stat_out, stream);
    if (rc) return rc;
    rc = chol_backward(h, false, L, ldm, Ni, Linv, L + (int64_t)Ni * ldm, ldm, At, ldm, n, stream);
    if (rc) return rc;
    // Wt = At * Xc   (C[t, i] = sum_r At[t, r] * Xc[r, i])
    rc = dgemm<true>(h, false, 128, TILES_ALL, 0, At, ldm, Xc, ldc, Wt, ldc, n, Ksel, Ni, 1.0, 0.0, stream);
    if (rc) return rc;
    ls_output<<<n, 256, 0, stream>>>(Wt, ldc, xmean, ymean, nullptr, Ksel, 1.0, W_out, b_out, 0);
    CP_CHECK_LAUNCH();
    return CP_OK;
}
