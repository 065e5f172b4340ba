// Dense fp64 building blocks of the 3C companions of the pruning path (SURVEY.md 8a-a8 / 8f):
//
//   cp_gemm_f64      <- every np.dot / np.tensordot of VH_decompose, nonlinear_fc and ITQ_decompose
//                       (reference lib/decompose.py:85-147, 163-319, 671-685) and reg.predict (:680)
//   cp_svd_jacobi    <- scipy.linalg.svd(x, full_matrices=False, lapack_driver='gesvd') (decompose.py:154-156)
//                       and, through the eigen-decomposition of a symmetric matrix, scipy.linalg.pinv (:149-152)
//   cp_solve_relu    <- solve_relu (decompose.py:51-59) and the identical block of ITQ_decompose (:231-240),
//                       fused with the bias add of reg.predict and with the column means of the result
//   cp_colstats_f64  <- ndarray.mean(0) (decompose.py:180, 242)
//
// The SVD is a one-sided (Hestenes) Jacobi: column pairs of F are orthogonalised by plane rotations in a
// round-robin order; one CTA per pair, all n/2 pairs of a step are disjoint, one launch per step.  Everything the
// reference takes SVDs of on this path is small (VH: (c k) x (n k) <= 1536 x 1536; ITQ: reduced to n x n, n <= 512,
// because X = G M has the right singular vectors of the n x n matrix L_S' M with G'G = L_S L_S') so the kernel keeps
// both columns of a pair in shared memory.  Jacobi is also the most accurate dense SVD (high relative accuracy).
#include "common.cuh"
#include "gemm_f64.cuh"

namespace {

// ---------------------------------------------------------------- one-sided Jacobi
// pair i of step s in the round-robin ("circle") ordering of npad (even) players
__device__ __forceinline__ void rr_pair(int s, int i, int npad, int &p, int &q) {
    const int m1 = npad - 1;
    if (i == 0) {
        p = s;
        q = m1;
    } else {
        p = (s + i) % m1;
        q = (s - i + m1) % m1;
    }
    if (p > q) {
        const int t = p;
        p = q;
        q = t;
    }
}

__device__ __forceinline__ double block_sum(double v, double *red) {  // 256 threads
#pragma unroll
    for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w];
    return t;
}

__global__ void __launch_bounds__(256)
jacobi_step(double *__restrict__ Ft, int m, int64_t ldf, double *__restrict__ Wt, int n, int64_t ldw, int step, int npad,
            double tol, unsigned int *__restrict__ counter, const double *__restrict__ frob2) {
    extern __shared__ __align__(16) double js[];  // [2][m]
    __shared__ double red[8];
    int p, q;
    rr_pair(step, blockIdx.x, npad, p, q);
    if (q >= n) return;  // phantom column of an odd n
    double *fp = Ft + (int64_t)p * ldf, *fq = Ft + (int64_t)q * ldf;
    double *sp = js, *sq = js + m;
    double a = 0.0, b = 0.0, g = 0.0;
    for (int e = threadIdx.x; e < m; e += 256) {
        const double x = fp[e], y = fq[e];
        sp[e] = x;
        sq[e] = y;
        a = fma(x, x, a);
        b = fma(y, y, b);
        g = fma(x, y, g);
    }
    a = block_sum(a, red);
    b = block_sum(b, red);
    g = block_sum(g, red);
    if (!(fabs(g) > tol * sqrt(a * b))) return;  // already orthogonal (also covers zero columns)
    // columns at the rounding-noise level of the matrix (rank-deficient input: |f|^2 < (1e-15 |F|_F)^2) are null
    // vectors already; rotating noise against noise would never converge
    const double floor2 = 1e-30 * frob2[0];
    if (a <= floor2 || b <= floor2) return;
    const double zeta = (b - a) / (2.0 * g);
    const double t = copysign(1.0, zeta) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
    const double c = rsqrt(1.0 + t * t), s = c * t;
    for (int e = threadIdx.x; e < m; e += 256) {
        const double x = sp[e], y = sq[e];
        fp[e] = c * x - s * y;
        fq[e] = s * x + c * y;
    }
    double *wp = Wt + (int64_t)p * ldw, *wq = Wt + (int64_t)q * ldw;
    for (int e = threadIdx.x; e < n; e += 256) {
        const double x = wp[e], y = wq[e];
        wp[e] = c * x - s * y;
        wq[e] = s * x + c * y;
    }
    if (threadIdx.x == 0) atomicAdd(counter, 1u);
}

// sum of squares of the whole matrix (one CTA; the matrices are small)
__global__ void __launch_bounds__(256)
frob2_kernel(const double *__restrict__ Ft, int m, int64_t ldf, int n, double *__restrict__ out) {
    __shared__ double red[8];
    double a = 0.0;
    for (int r = 0; r < n; ++r)
        for (int e = threadIdx.x; e < m; e += 256) {
            const double v = Ft[(int64_t)r * ldf + e];
            a = fma(v, v, a);
        }
    a = block_sum(a, red);
    if (threadIdx.x == 0) out[0] = a;
}

__global__ void set_identity(double *__restrict__ W, int n, int64_t ld) {
    const int j = blockIdx.x * 256 + threadIdx.x, i = blockIdx.y;
    if (j < n) W[(int64_t)i * ld + j] = (i == j) ? 1.0 : 0.0;
}

// sigma[j] = |row j|; row j /= sigma[j] (left singular vector) when normalise != 0
__global__ void __launch_bounds__(256)
row_norms(double *__restrict__ Ft, int m, int64_t ldf, double *__restrict__ sigma, int normalise) {
    __shared__ double red[8];
    double *f = Ft + (int64_t)blockIdx.x * ldf;
    double a = 0.0;
    for (int e = threadIdx.x; e < m; e += 256) a = fma(f[e], f[e], a);
    a = block_sum(a, red);
    const double sg = sqrt(a);
    if (threadIdx.x == 0) sigma[blockIdx.x] = sg;
    if (normalise && sg > 0.0) {
        const double inv = 1.0 / sg;
        for (int e = threadIdx.x; e < m; e += 256) f[e] *= inv;
    }
}

// ---------------------------------------------------------------- elementwise / column statistics
// RU = RUraw + b (+ add_mean); U = solve_relu(RU, Z, lambda) (decompose.py:51-59).
__global__ void __launch_bounds__(256)
solve_relu_kernel(const double *__restrict__ RUraw, int64_t ldr, const double *__restrict__ bias, const double *__restrict__ Z,
                  int64_t ldz, double lambda, double *__restrict__ U, int64_t ldu, int64_t N, int n) {
    // one CTA per 32 columns x 64-row band: coalesced rows
    const int cx = threadIdx.x & 31, rg = threadIdx.x >> 5;
    const int j = blockIdx.x * 32 + cx;
    const int64_t r0 = (int64_t)blockIdx.y * 64;
    if (j < n) {
        const double bj = bias ? bias[j] : 0.0;
        for (int64_t r = r0 + rg; r < r0 + 64 && r < N; r += 8) {
            // every operation rounded separately, in numpy's evaluation order (decompose.py:52-58): no FMA contraction
            const double ru = bias ? __dadd_rn(RUraw[r * ldr + j], bj) : RUraw[r * ldr + j];
            const double z = Z[r * ldz + j];
            const double u0 = fmin(ru, 0.0);
            const double d0 = __dadd_rn(u0, -ru);
            const double cost0 = __dadd_rn(__dmul_rn(z, z), __dmul_rn(lambda, __dmul_rn(d0, d0)));
            const double u1 = fmax(__ddiv_rn(__dadd_rn(__dmul_rn(lambda, ru), z), __dadd_rn(lambda, 1.0)), 0.0);
            const double d1 = __dadd_rn(u1, -z), d2 = __dadd_rn(u1, -ru);
            const double cost1 = __dadd_rn(__dmul_rn(d1, d1), __dmul_rn(lambda, __dmul_rn(d2, d2)));
            const double u = (cost0 <= cost1) ? u0 : u1;
            U[r * ldu + j] = u;
        }
    }
}

// X[r, j] = (X[r, j] - shift[j]) in place, or into Out
__global__ void __launch_bounds__(256)
shift_cols(const double *__restrict__ X, int64_t ldx, const double *__restrict__ shift, double *__restrict__ Out,
           int64_t ldo, int64_t N, int n) {
    const int j = blockIdx.x * 256 + threadIdx.x;
    if (j >= n) return;
    for (int64_t r = blockIdx.y; r < N; r += gridDim.y) Out[r * ldo + j] = X[r * ldx + j] - shift[j];
}

}  // namespace

extern "C" int cp_gemm_f64(cp_handle_t h, int a_mc, int b_nc, int M, int Nn, int64_t R, double alpha, const double *A,
                           int64_t lda, const double *B, int64_t ldb, double beta, double *C, int64_t ldc,
                           cp_stream_t stream_) {
    CP_REQUIRE(h && A && B && C, "cp_gemm_f64: NULL argument");
    CP_REQUIRE(M > 0 && Nn > 0 && R >= 0 && ldc >= Nn, "cp_gemm_f64: bad shape");
    CP_REQUIRE(lda >= (a_mc ? M : R) && ldb >= (b_nc ? Nn : R), "cp_gemm_f64: leading dimension too small");
    CP_DEVICE_GUARD(h);
    cudaStream_t stream = (cudaStream_t)stream_;
    using cpgemm::product;
    cpgemm::Args g{};
    g.A = A; g.lda = lda; g.B = B; g.ldb = ldb; g.C = C; g.ldc = ldc;
    g.M = M; g.Nn = Nn; g.R = R;
    g.alpha = alpha; g.beta = beta;
    g.tile_mode = cpgemm::TILES_ALL;
    const int64_t min_split_r = 8 * cpgemm::BK;  // reductions shorter than 8 stages run unsplit
    if (a_mc && b_nc) return product<double, double, true, true>(h, g, min_split_r, stream);
    if (a_mc) return product<double, double, true, false>(h, g, min_split_r, stream);
    if (b_nc) return product<double, double, false, true>(h, g, min_split_r, stream);
    return product<double, double, false, false>(h, g, min_split_r, stream);
}

extern "C" int cp_svd_jacobi(cp_handle_t h, double *Ft, int m, int n, int64_t ldf, double *Wt, int64_t ldw, double *sigma,
                             int normalise_left, double tol, int max_sweeps, int32_t *sweeps_out, cp_stream_t stream_) {
    CP_REQUIRE(h && Ft && Wt && sigma, "cp_svd_jacobi: NULL argument");
    CP_REQUIRE(m > 0 && n > 0 && ldf >= m && ldw >= n && max_sweeps > 0, "cp_svd_jacobi: bad shape");
    CP_REQUIRE((size_t)m * 2 * sizeof(double) <= 200 * 1024, "cp_svd_jacobi: m=%d too large for the shared-memory pair buffer", m);
    CP_DEVICE_GUARD(h);
    cudaStream_t stream = (cudaStream_t)stream_;
    const size_t smem = (size_t)2 * m * sizeof(double);
    if (smem > 48 * 1024) {
        static cp_per_device_flag configured;
        if (bool *done = configured.slot(); !*done) {
            CP_CUDA(cudaFuncSetAttribute(jacobi_step, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
            *done = true;
        }
    }
    void *ws = nullptr;
    int rc = cp_ws_reserve(h, 256, &ws);
    if (rc) return rc;
    unsigned int *counter = (unsigned int *)ws;
    double *frob2 = (double *)ws + 8;
    frob2_kernel<<<1, 256, 0, stream>>>(Ft, m, ldf, n, frob2);
    CP_CHECK_LAUNCH();
    set_identity<<<dim3(cp_cdiv(n, 256), n), 256, 0, stream>>>(Wt, n, ldw);
    CP_CHECK_LAUNCH();
    const int npad = n + (n & 1);
    int sweeps = 0;
    for (; sweeps < max_sweeps; ++sweeps) {
        CP_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned int), stream));
        if (npad >= 2) {
            for (int s = 0; s < npad - 1; ++s) {
                jacobi_step<<<npad / 2, 256, smem, stream>>>(Ft, m, ldf, Wt, n, ldw, s, npad, tol, counter, frob2);
                CP_CHECK_LAUNCH();
            }
        }
        unsigned int rotated = 0;  // the sweep count is data dependent: this routine synchronises once per sweep
        CP_CUDA(cudaMemcpyAsync(&rotated, counter, sizeof(unsigned int), cudaMemcpyDeviceToHost, stream));
        CP_CUDA(cudaStreamSynchronize(stream));
        if (rotated == 0) break;
    }
    row_norms<<<n, 256, 0, stream>>>(Ft, m, ldf, sigma, normalise_left);
    CP_CHECK_LAUNCH();
    if (sweeps_out) *sweeps_out = sweeps;
    return CP_OK;
}

extern "C" int cp_solve_relu(cp_handle_t h, const double *RUraw, int64_t ldr, const double *bias, const double *Z, int64_t ldz,
                             double lambda, double *U, int64_t ldu, int64_t N, int n, double *colmean_out,
                             cp_stream_t stream_) {
    CP_REQUIRE(h && RUraw && Z && U, "cp_solve_relu: NULL argument");
    CP_REQUIRE(N > 0 && n > 0 && ldr >= n && ldz >= n && ldu >= n, "cp_solve_relu: bad shape");
    CP_DEVICE_GUARD(h);
    cudaStream_t stream = (cudaStream_t)stream_;
    solve_relu_kernel<<<dim3(cp_cdiv(n, 32), cp_cdiv(N, 64)), 256, 0, stream>>>(RUraw, ldr, bias, Z, ldz, lambda, U, ldu, N, n);
    CP_CHECK_LAUNCH();
    if (colmean_out) {  // fixed-order column means
        cpgemm::colsum_kernel<double><<<cp_cdiv(n, 32), 256, 0, stream>>>(U, ldu, n, nullptr, N, nullptr, 1.0 / (double)N,
                                                                          colmean_out, nullptr);
        CP_CHECK_LAUNCH();
    }
    return CP_OK;
}

extern "C" int cp_colstats_f64(cp_handle_t h, const double *X, int64_t ldx, int64_t N, int n, double scale, double *colsum_out,
                               double *centred_out, int64_t ldo, cp_stream_t stream_) {
    CP_REQUIRE(h && X && colsum_out, "cp_colstats_f64: NULL argument");
    CP_REQUIRE(N > 0 && n > 0 && ldx >= n, "cp_colstats_f64: bad shape");
    CP_DEVICE_GUARD(h);
    cudaStream_t stream = (cudaStream_t)stream_;
    cpgemm::colsum_kernel<double><<<cp_cdiv(n, 32), 256, 0, stream>>>(X, ldx, n, nullptr, N, nullptr, scale, colsum_out, nullptr);
    CP_CHECK_LAUNCH();
    if (centred_out) {  // centred_out = X - colsum_out (meaningful with scale = 1/N: the column means)
        CP_REQUIRE(ldo >= n, "cp_colstats_f64: ldo < n");
        shift_cols<<<dim3(cp_cdiv(n, 256), (unsigned)(N < 32768 ? N : 32768)), 256, 0, stream>>>(X, ldx, colsum_out, centred_out, ldo, N, n);
        CP_CHECK_LAUNCH();
    }
    return CP_OK;
}
