// cp_gram: tall-skinny sufficient statistics  G = X'X, Bxy = X'Y, column sums, sum(Y^2).
//
// Replaces the O(N K^2) passes of LinearRegression.fit (reference lib/decompose.py:665-666)
// and of the LASSO design matrix (lib/decompose.py:428-434,457); see SURVEY.md 7.1.
//
// CP_GRAM_FP64: fp32 inputs widened to fp64 in registers, fp64 accumulation on DMMA
// (cpgemm::gemm_kernel).  Every product of two fp32 values is exact in fp64, so the
// only rounding is the fp64 accumulation -- the same arithmetic class as the
// reference's float64 numpy path.  Small K does not fill the SMs with output tiles,
// so the reduction (row) dimension is split across CTAs into fp64 partials that a
// second kernel sums in a fixed order (deterministic, no atomics).
#include <stdlib.h>

#include "common.cuh"
#include "gemm_f64.cuh"


int cp_gram_tc2(cp_handle_t h, const float *X, int64_t N, int K, int64_t ldx, const void *Yraw, int y_dtype, int n, int64_t ldy,
                const float *y_bias, const int32_t *rows, int nrows, double *G, double *Bxy, double *sx,
                double *sy, double *yy, cudaStream_t stream);

int cp_gram_fp64_products(cp_handle_t h, const float *X, int64_t N, int K, int64_t ldx, const void *Yraw, int y_dtype,
                          int n, int64_t ldy, const float *y_bias, const int32_t *rows, int nrows, double *G,
                          double *Bxy, double *sx, double *sy, double *yy, cudaStream_t stream);

namespace {

// sums partials over splits in order; symmetric mode mirrors the upper tile region.
__global__ void reduce_partials(const double *__restrict__ part, int64_t split_stride, int nsplit,
                                double *__restrict__ C, int M, int Nn, int64_t ldc, int sym) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)M * Nn) return;
    const int i = (int)(e / Nn), j = (int)(e - (int64_t)i * Nn);
    if (sym && (i / cpgemm::BM) > (j / cpgemm::BN)) return;  // lower tiles come from the mirror
    double s = 0.0;
    for (int k = 0; k < nsplit; ++k) s += part[(int64_t)k * split_stride + (int64_t)i * ldc + j];
    C[(int64_t)i * ldc + j] = s;
}

// C[j, i] = C[i, j] for every element of the strictly-upper 128x128 tiles, through a padded
// shared-memory tile so that both the reads and the writes are coalesced.
__global__ void __launch_bounds__(256)
mirror_upper_tiles(double *__restrict__ C, int M, int64_t ldc) {
    __shared__ double t[32][33];
    const int bx = blockIdx.x, by = blockIdx.y;  // 32x32 sub-tile (row block by, column block bx)
    if ((by * 32) / cpgemm::BM >= (bx * 32) / cpgemm::BN) return;  // only strictly-upper 128-tiles
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

// column sums (and optionally sums of squares) of an fp32 matrix, fp64 accumulation,
// fixed summation order: each CTA owns 32 columns, 8 row lanes, then a serial 8-way add.
template <typename T>
__global__ void __launch_bounds__(256)
colsum_kernel(const T *__restrict__ X, int64_t ld, int ncols, const int32_t *__restrict__ rows, int64_t nrows,
              const float *__restrict__ bias, double *__restrict__ sum_out, double *__restrict__ sumsq_out) {
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
        if (sum_out) sum_out[col] = ta;
        if (sumsq_out) sumsq_out[col] = tq;
    }
}

__global__ void serial_sum(const double *__restrict__ v, int n, double *__restrict__ out) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        double s = 0.0;
        for (int i = 0; i < n; ++i) s += v[i];
        *out = s;
    }
}

inline bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace

// C = A' B over (optionally gathered) rows, via split-R partials when the tile count is small.
template <typename TB>
static int gram_product(cp_handle_t h, const float *A, int64_t lda, int M, const TB *B, int64_t ldb, int Nn,
                        const float *b_bias, const int32_t *rows, int64_t R, double *C, bool sym,
                        cudaStream_t stream) {
    using namespace cpgemm;
    Args g{};
    g.A = A; g.lda = lda; g.B = B; g.ldb = ldb;
    g.M = M; g.Nn = Nn; g.R = R;
    g.rowidx = rows; g.b_bias = b_bias;
    g.alpha = 1.0; g.beta = 0.0;
    g.tile_mode = sym ? TILES_UPPER_SYM : TILES_ALL;
    g.a_vec = aligned16(A) && (lda % 4 == 0);
    g.b_vec = aligned16(B) && (ldb % (16 / sizeof(TB)) == 0);
    const int tiles = num_tiles(M, Nn, g.tile_mode, BM);
    const int target = 2 * h->num_sms;
    int nsplit = 1;
    if (tiles < target) {
        nsplit = (target + tiles - 1) / tiles;
        const int64_t max_by_rows = (R + 4 * BK - 1) / (4 * BK);  // at least 64 rows per split
        if (nsplit > max_by_rows) nsplit = (int)max_by_rows;
        const size_t per = (size_t)M * Nn * sizeof(double);
        const size_t cap = (size_t)256 << 20;
        if ((size_t)nsplit * per > cap) nsplit = (int)(cap / per);
        if (nsplit < 1) nsplit = 1;
    }
    int64_t rps = (R + nsplit - 1) / nsplit;
    rps = (rps + BK - 1) / BK * BK;
    nsplit = (int)((R + rps - 1) / rps);
    if (nsplit < 1) nsplit = 1;
    g.nsplit = nsplit;
    g.r_per_split = rps;
    if (nsplit == 1) {
        g.C = C; g.ldc = Nn; g.c_split_stride = 0;
        g.r_per_split = R > 0 ? R : 1;
        CP_GEMM_LAUNCH((launch<float, TB, true, true>(g, stream)));
    } else {
        void *ws = nullptr;
        int rc = cp_ws_reserve(h, (size_t)nsplit * M * Nn * sizeof(double), &ws);
        if (rc) return rc;
        g.C = (double *)ws; g.ldc = Nn; g.c_split_stride = (int64_t)M * Nn;
        CP_GEMM_LAUNCH((launch<float, TB, true, true>(g, stream)));
        const int64_t total = (int64_t)M * Nn;
        reduce_partials<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>((const double *)ws, g.c_split_stride,
                                                                           nsplit, C, M, Nn, Nn, sym ? 1 : 0);
        CP_CHECK_LAUNCH();
    }
    if (sym && M > BM) {
        const int nb32 = (M + 31) / 32;
        mirror_upper_tiles<<<dim3(nb32, nb32), 256, 0, stream>>>(C, M, Nn);
        CP_CHECK_LAUNCH();
    }
    return CP_OK;
}

extern "C" int cp_gram(cp_handle_t h, const float *X, int64_t N, int K, int64_t ldx, const void *Yraw, int y_dtype,
                       int n, int64_t ldy, const float *y_bias, const int32_t *rows, int nrows, double *G, double *Bxy,
                       double *sx, double *sy, double *yy, int mode, cp_stream_t stream_) {
    CP_REQUIRE(h && (X || N == 0), "cp_gram: NULL handle or X");
    CP_REQUIRE(N >= 0 && K > 0 && ldx >= K, "cp_gram: bad X shape (N=%lld K=%d ldx=%lld)", (long long)N, K, (long long)ldx);
    CP_REQUIRE((Bxy == nullptr && sy == nullptr && yy == nullptr) || (Yraw != nullptr && n > 0 && ldy >= n),
               "cp_gram: Y outputs requested without a valid Y");
    CP_REQUIRE(rows == nullptr || nrows >= 0, "cp_gram: bad nrows");
    CP_REQUIRE(y_dtype == CP_F32 || y_dtype == CP_F64, "cp_gram: unknown y_dtype %d", y_dtype);
    CP_REQUIRE(mode == CP_GRAM_FP64 || mode == CP_GRAM_3XTF32, "cp_gram: unknown mode %d", mode);
    cudaStream_t stream = (cudaStream_t)stream_;
    const int64_t R = rows ? (int64_t)nrows : N;

    if (R == 0) {  // empty input: all statistics are zero
        if (G) CP_CUDA(cudaMemsetAsync(G, 0, sizeof(double) * (size_t)K * K, stream));
        if (Bxy) CP_CUDA(cudaMemsetAsync(Bxy, 0, sizeof(double) * (size_t)K * n, stream));
        if (sx) CP_CUDA(cudaMemsetAsync(sx, 0, sizeof(double) * (size_t)K, stream));
        if (sy) CP_CUDA(cudaMemsetAsync(sy, 0, sizeof(double) * (size_t)n, stream));
        if (yy) CP_CUDA(cudaMemsetAsync(yy, 0, sizeof(double), stream));
        return CP_OK;
    }
    if (mode == CP_GRAM_3XTF32) {  // falls back to the fp64 products when TMA alignment rules are not met
        return cp_gram_tc2(h, X, N, K, ldx, Yraw, y_dtype, n, ldy, y_bias, rows, nrows, G, Bxy, sx, sy, yy, stream);
    }
    return cp_gram_fp64_products(h, X, N, K, ldx, Yraw, y_dtype, n, ldy, y_bias, rows, nrows, G, Bxy, sx, sy, yy, stream);
}

int cp_gram_fp64_products(cp_handle_t h, const float *X, int64_t N, int K, int64_t ldx, const void *Yraw, int y_dtype,
                          int n, int64_t ldy, const float *y_bias, const int32_t *rows, int nrows, double *G,
                          double *Bxy, double *sx, double *sy, double *yy, cudaStream_t stream) {
    const int64_t R = rows ? (int64_t)nrows : N;
    if (G) {
        int rc = gram_product<float>(h, X, ldx, K, X, ldx, K, nullptr, rows, R, G, true, stream);
        if (rc) return rc;
    }
    if (Bxy) {
        int rc = y_dtype == CP_F32
                     ? gram_product<float>(h, X, ldx, K, (const float *)Yraw, ldy, n, y_bias, rows, R, Bxy, false, stream)
                     : gram_product<double>(h, X, ldx, K, (const double *)Yraw, ldy, n, y_bias, rows, R, Bxy, false, stream);
        if (rc) return rc;
    }
    if (sx) {
        colsum_kernel<float><<<cp_cdiv(K, 32), 256, 0, stream>>>(X, ldx, K, rows, R, nullptr, sx, nullptr);
        CP_CHECK_LAUNCH();
    }
    if (sy || yy) {
        double *sq = nullptr;
        if (yy) {
            void *ws = nullptr;  // NB: shares the handle scratch with the split partials above; stream order keeps it safe
            int rc = cp_ws_reserve(h, (size_t)n * sizeof(double), &ws);
            if (rc) return rc;
            sq = (double *)ws;
        }
        if (y_dtype == CP_F32)
            colsum_kernel<float><<<cp_cdiv(n, 32), 256, 0, stream>>>((const float *)Yraw, ldy, n, rows, R, y_bias, sy, sq);
        else
            colsum_kernel<double><<<cp_cdiv(n, 32), 256, 0, stream>>>((const double *)Yraw, ldy, n, rows, R, y_bias, sy, sq);
        CP_CHECK_LAUNCH();
        if (yy) {
            serial_sum<<<1, 32, 0, stream>>>(sq, n, yy);
            CP_CHECK_LAUNCH();
        }
    }
    return CP_OK;
}
