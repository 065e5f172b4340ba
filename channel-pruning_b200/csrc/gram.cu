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

__global__ void serial_sum(const double *__restrict__ v, int n, double *__restrict__ out) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        double s = 0.0;
        for (int i = 0; i < n; ++i) s += v[i];
        *out = s;
    }
}

}  // namespace

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
    using cpgemm::colsum_kernel;
    using cpgemm::product;
    const int64_t R = rows ? (int64_t)nrows : N;
    // C = X' B over the (optionally gathered) rows; every reduction length may split
    cpgemm::Args g{};
    g.A = X; g.lda = ldx; g.M = K; g.R = R; g.rowidx = rows;
    g.alpha = 1.0; g.beta = 0.0;
    if (G) {
        g.B = X; g.ldb = ldx; g.Nn = K; g.C = G; g.ldc = K;
        g.tile_mode = cpgemm::TILES_UPPER_SYM;
        int rc = product<float, float, true, true>(h, g, 0, stream);
        if (rc) return rc;
    }
    if (Bxy) {
        g.B = Yraw; g.ldb = ldy; g.Nn = n; g.b_bias = y_bias; g.C = Bxy; g.ldc = n;
        g.tile_mode = cpgemm::TILES_ALL;
        int rc = y_dtype == CP_F32 ? product<float, float, true, true>(h, g, 0, stream)
                                   : product<float, double, true, true>(h, g, 0, stream);
        if (rc) return rc;
    }
    if (sx) {
        colsum_kernel<float><<<cp_cdiv(K, 32), 256, 0, stream>>>(X, ldx, K, rows, R, nullptr, 1.0, sx, nullptr);
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
            colsum_kernel<float><<<cp_cdiv(n, 32), 256, 0, stream>>>((const float *)Yraw, ldy, n, rows, R, y_bias, 1.0, sy, sq);
        else
            colsum_kernel<double><<<cp_cdiv(n, 32), 256, 0, stream>>>((const double *)Yraw, ldy, n, rows, R, y_bias, 1.0, sy, sq);
        CP_CHECK_LAUNCH();
        if (yy) {
            serial_sum<<<1, 32, 0, stream>>>(sq, n, yy);
            CP_CHECK_LAUNCH();
        }
    }
    return CP_OK;
}
