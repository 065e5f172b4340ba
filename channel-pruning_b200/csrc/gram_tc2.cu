// cp_gram, tensor-core mode (CP_GRAM_3XTF32 in the header): split-fp16 operands prepared once, a persistent
// TMA -> wgmma pipeline with no conversion work on the critical path.
//
//   G = X'X (K x K),  Bxy = X'(Y - b) (K x n)      X: N x K fp32 row-major, N ~ 5e3..1e5, K = c*k*k
//
// The reference does this arithmetic in float64 on the CPU (numpy matmul / LAPACK inside LinearRegression.fit,
// lib/decompose.py:665-666, and the LASSO design products lib/decompose.py:428-457).  The tensor cores have no fp64
// MMA at this rate, so the products are taken in three fp16 MMAs of a 22-bit hi/lo split:
//
//   prep   xs = fl32(x - s_col)             s = fp32 column mean (removes the rank-one mean component)
//          v  = xs * 2^e_col                power-of-two column scale (exact): max|v| in [2^9, 2^10)
//          v  = hi + lo                     hi = fp16_rn(v), lo = fp16_rn(v - hi): 22 mantissa bits kept -- the
//                                           same split precision as tf32 (10 explicit bits each), but fp16 MMAs
//                                           run at twice the tf32 rate and the operands are half as wide
//          written TRANSPOSED (operand row = column of X, reduction index contiguous, zero padded) so that the
//          GEMM reads plain K-major SWIZZLE_128B tiles with TMA; the same pass produces the fp64 column sums
//          and sums of squares of xs (fixed summation order)
//   gemm   P += hi'hi + hi'lo + lo'hi       three wgmma chains (m64n128k16) per k-step, fp32 accumulation in
//          registers in runs of 64 rows, each run added into fp32 register sums with round-to-nearest
//          (tc_common.cuh)
//   reduce fp64 sum of the row splits, exact rescale by 2^-(e_i + e_j), shift undone exactly
//          (G = P + s T' + T s' + N s s',  T = column sums of xs in fp64), diagonal from the fp64 squares,
//          lower triangle written in the same pass.
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdlib.h>

#include "common.cuh"
#include "tc_common.cuh"

int cp_gram_fp64_products(cp_handle_t h, const float *X, int64_t N, int K, int64_t ldx, const void *Yraw, int y_dtype,
                          int n, int64_t ldy, const float *y_bias, const int32_t *rows, int nrows, double *G,
                          double *Bxy, double *sx, double *sy, double *yy, cudaStream_t stream);
bool cp_gram_tc_eligible(const float *X, int64_t N, int K, int64_t ldx, const void *Yraw, int y_dtype, int n, int64_t ldy,
                         const int32_t *rows, bool wantB);

namespace {

using namespace cptc;

constexpr int TN = TILE;                    // output tile: 128 rows of G (or of X'Y) x 128 columns
constexpr int RS = 32;                      // row splits of the statistics passes (partials combined in fixed order)
constexpr int PT = 64;                      // prep tile: 64 rows x 64 columns

struct Tc2Params {
    float *partial;      // [nsplit][ntiles][128][128]
    int64_t Np;          // padded row count (multiple of 64) = inner extent of the operand matrix
    int rows_per_split;  // multiple of 64
    int nsplit;
    int tiles_sym;       // number of 128 x 128 tiles covering the upper triangle of G (0 when G is not requested)
    int tk;              // ceil(K / 128): row tiles
    int tjx;             // ceil(K / 128): column tiles inside X
    int tjy0;            // first column tile of the Y region (= Kp / 128)
    int tnb;             // column tiles of the Y region
    int ntiles;
    int mtot;            // operand rows of one half (hi); the lo half starts at row mtot
};

// tile index -> (ti, tj): the tiles of the upper triangle first (row ti: tj = ti .. tjx-1), then X'Y
__host__ __device__ __forceinline__ void decode_tile(int l, int tiles_sym, int tjx, int tjy0, int tnb, int &ti, int &tj) {
    if (l < tiles_sym) {
        ti = 0;
        while (l >= tjx - ti) { l -= tjx - ti; ++ti; }
        tj = ti + l;
    } else {
        l -= tiles_sym;
        ti = l / tnb;
        tj = tjy0 + (l - ti * tnb);
    }
}

// item -> (tile, split) -> (ti, tj)
struct Item {
    int tile, split, ti, tj, nst;
    int64_t r_begin;
    bool diag;  // ti == tj inside X: the A rows are the B rows
};
__device__ __forceinline__ Item decode_item(const Tc2Params &P, int w) {
    Item it;
    it.split = w / P.ntiles;
    it.tile = w - it.split * P.ntiles;
    decode_tile(it.tile, P.tiles_sym, P.tjx, P.tjy0, P.tnb, it.ti, it.tj);
    it.diag = it.tile < P.tiles_sym && it.ti == it.tj;
    it.r_begin = (int64_t)it.split * P.rows_per_split;
    int64_t r_end = it.r_begin + P.rows_per_split;
    if (r_end > P.Np) r_end = P.Np;
    it.nst = (int)((r_end - it.r_begin) / KS);
    return it;
}

// ------------------------------------------------------------------ the GEMM
// Persistent grid (one CTA per SM), static round-robin over (output tile, row split) items; the TMA -> wgmma pipeline
// of tc_common.cuh, one fp32 partial tile per item.
// Bound: L2 -> SM operand traffic (64 KB per 3 x 128 x 128 x 64 products), then the tensor pipe.
__global__ void __launch_bounds__(NTHREADS, 1)
gram_tc2_kernel(const __grid_constant__ CUtensorMap mapA, const Tc2Params P) {
    extern __shared__ unsigned char smem_dyn[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_dyn + 1023) & ~(uintptr_t)1023);
    const uint32_t sbase = smem_u32(smem);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nitems = P.ntiles * P.nsplit;
    pipe_init(sbase);
    uint32_t g = 0;
    if (warp == W_TMA) {
        if (lane == 0)
            for (int w = blockIdx.x; w < nitems; w += gridDim.x) {
                const Item it = decode_item(P, w);
                pipe_produce(sbase, g, &mapA, &mapA, it.ti * TILE, P.mtot, it.tj * TILE, P.mtot, it.r_begin, it.nst, it.diag);
            }
        return;
    }
    const int wg = warp >> 2;
    for (int w = blockIdx.x; w < nitems; w += gridDim.x) {
        const Item it = decode_item(P, w);
        float sum[FRAG];
        pipe_consume(sbase, g, wg, it.nst, it.diag, sum);
        float *dst = P.partial + ((size_t)it.split * P.ntiles + it.tile) * (size_t)(TILE * TN) + (size_t)(wg * 64) * TN;
#pragma unroll
        for (int e = 0; e < FRAG; e += 2)
            *reinterpret_cast<float2 *>(dst + (size_t)frag_row(e) * TN + frag_col(e)) = make_float2(sum[e], sum[e + 1]);
    }
}

// ------------------------------------------------------------------ operand space
// Operand row o of the GEMM: o < Kp -> column o of X (zero row when o >= K); o >= Kp -> column o - Kp of Y.
// Kp and the Y extent are multiples of 128, so no strip of the kernels below straddles the two matrices.
struct Cols {
    const float *X, *Y;
    int64_t ldx, ldy;
    int K, n, Kp;
};
struct ColRef {
    const float *base;
    int64_t ld;
    int col, ncols;
};
__device__ __forceinline__ ColRef col_ref(const Cols &C, int o) {
    ColRef r;
    if (o < C.Kp) { r.base = C.X; r.ld = C.ldx; r.col = o; r.ncols = C.K; }
    else { r.base = C.Y; r.ld = C.ldy; r.col = o - C.Kp; r.ncols = C.n; }
    return r;
}

// ------------------------------------------------------------------ statistics pass 1: column sums and max |x|
// CTA = 128 operand rows (32 float4 lanes) x 8 row lanes over one row split; fixed summation order.
__global__ void __launch_bounds__(256)
colstat_part(const Cols C, int64_t nrows, int mtot, double *__restrict__ part, float *__restrict__ part_max) {
    __shared__ double s1[8][132];
    __shared__ float s2[8][132];
    const int cq = threadIdx.x & 31, rg = threadIdx.x >> 5;
    const int o0 = blockIdx.x * 128 + cq * 4;
    const ColRef cr = col_ref(C, o0);
    const int64_t per = (nrows + RS - 1) / RS;
    const int64_t r0 = (int64_t)blockIdx.y * per;
    const int64_t r1 = r0 + per < nrows ? r0 + per : nrows;
    double a[4] = {0, 0, 0, 0};
    float mx[4] = {0, 0, 0, 0};
    if (cr.col + 3 < cr.ncols) {
#pragma unroll 4
        for (int64_t r = r0 + rg; r < r1; r += 8) {
            const float4 v = __ldg(reinterpret_cast<const float4 *>(cr.base + r * cr.ld + cr.col));
            a[0] += (double)v.x; a[1] += (double)v.y; a[2] += (double)v.z; a[3] += (double)v.w;
            mx[0] = fmaxf(mx[0], fabsf(v.x)); mx[1] = fmaxf(mx[1], fabsf(v.y));
            mx[2] = fmaxf(mx[2], fabsf(v.z)); mx[3] = fmaxf(mx[3], fabsf(v.w));
        }
    } else if (cr.col < cr.ncols) {
        for (int64_t r = r0 + rg; r < r1; r += 8)
            for (int c = 0; c < 4 && cr.col + c < cr.ncols; ++c) {
                const float v = __ldg(cr.base + r * cr.ld + cr.col + c);
                a[c] += (double)v;
                mx[c] = fmaxf(mx[c], fabsf(v));
            }
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) { s1[rg][cq * 4 + c] = a[c]; s2[rg][cq * 4 + c] = mx[c]; }
    __syncthreads();
    if (threadIdx.x < 128) {
        double t = 0.0;
        float m2 = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) { t += s1[k][threadIdx.x]; m2 = fmaxf(m2, s2[k][threadIdx.x]); }
        part[(size_t)blockIdx.y * mtot + blockIdx.x * 128 + threadIdx.x] = t;
        part_max[(size_t)blockIdx.y * mtot + blockIdx.x * 128 + threadIdx.x] = m2;
    }
}

// shift[o] = fl32(mean), scale[o] = 2^e with 2 * max|x| * 2^e in [2^9, 2^10), inv[o] = 2^-e (fp64).
// e comes from max|x| itself (2 max|x| overflows fp32 from 2^127 on) and is clamped to the exponents of normal fp32
// powers of two; only columns with max|x| < 2^-119 reach the clamp, and they keep |v| < 2^10.
__global__ void __launch_bounds__(128)
colstat_finish(const double *__restrict__ part, const float *__restrict__ part_max, int mtot, double invN,
               float *__restrict__ shift, float *__restrict__ scale, double *__restrict__ inv) {
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= mtot) return;
    double v[RS];
    float m[RS];
#pragma unroll
    for (int r = 0; r < RS; ++r) { v[r] = part[(size_t)r * mtot + o]; m[r] = part_max[(size_t)r * mtot + o]; }
    double t = 0.0;
    float mx = 0.f;
#pragma unroll
    for (int r = 0; r < RS; ++r) { t += v[r]; mx = fmaxf(mx, m[r]); }
    shift[o] = (float)(t * invN);
    int e = 0;  // |x - mean| <= 2 max|x|
    if (mx > 0.f && isfinite(mx)) {
        e = 8 - ilogbf(mx);
        e = e > 127 ? 127 : (e < -126 ? -126 : e);
    }
    scale[o] = ldexpf(1.f, e);
    inv[o] = ldexp(1.0, -e);
}

// ------------------------------------------------------------------ operand preparation (+ statistics pass 2)
// One CTA = a strip of 64 operand rows x the 64-row tiles of one row split.  Reads the data once (coalesced along the
// columns), writes the hi and lo operand rows (coalesced along the reduction index) through a swizzled shared-memory
// tile, and accumulates the fp64 column sums / sums of squares of xs in a fixed order.
__global__ void __launch_bounds__(256)
tc2_prep(const Cols C, int64_t nrows, int64_t Np, int tiles_per_split, int mtot, const float *__restrict__ shift,
         const float *__restrict__ scale, __half *__restrict__ Ohi, __half *__restrict__ Olo, double *__restrict__ part,
         double *__restrict__ part_sq) {
    __shared__ __align__(16) unsigned char tile_hi[PT * 128], tile_lo[PT * 128];
    __shared__ double red[16][PT + 1];
    const int t = threadIdx.x, jq = t & 15, rg = t >> 4;
    const int o0 = blockIdx.x * PT;       // first operand row of the strip
    const ColRef cr = col_ref(C, o0);
    const float *__restrict__ X = cr.base;
    const int64_t ld = cr.ld;
    const int ncols = cr.ncols;
    const int cj = cr.col + jq * 4;
    const bool vec = (cj + 3 < ncols);
    float sh[4], sc[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        sh[c] = cj + c < ncols ? shift[o0 + jq * 4 + c] : 0.f;
        sc[c] = cj + c < ncols ? scale[o0 + jq * 4 + c] : 0.f;
    }
    double a[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0};
    const int64_t ntile = Np / PT;
    const int64_t tb = (int64_t)blockIdx.y * tiles_per_split;
    int64_t te = tb + tiles_per_split;
    if (te > ntile) te = ntile;

    float4 cur[4], nxt[4];
    auto load = [&](int64_t tile, float4(&v)[4]) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int64_t r = tile * PT + rg * 4 + i;
            float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r < nrows) {
                const float *p = X + r * ld + cj;
                if (vec) x = __ldg(reinterpret_cast<const float4 *>(p));
                else {
                    if (cj + 0 < ncols) x.x = __ldg(p + 0);
                    if (cj + 1 < ncols) x.y = __ldg(p + 1);
                    if (cj + 2 < ncols) x.z = __ldg(p + 2);
                }
            }
            v[i] = x;
        }
    };
#pragma unroll
    for (int i = 0; i < 4; ++i) cur[i] = nxt[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (tb < te) load(tb, cur);
    for (int64_t tile = tb; tile < te; ++tile) {
        if (tile + 1 < te) load(tile + 1, nxt);
        // split: thread owns rows rg*4 .. rg*4+3 of the tile and 4 columns
        __half hi[4][4], lo[4][4];  // [column][row]
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const bool live = tile * PT + rg * 4 + i < nrows;
            const float xv[4] = {cur[i].x, cur[i].y, cur[i].z, cur[i].w};
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const float xs = (live && cj + c < ncols) ? __fsub_rn(xv[c], sh[c]) : 0.f;
                const double x64 = (double)xs;
                a[c] += x64;
                q[c] = fma(x64, x64, q[c]);
                const float v = __fmul_rn(xs, sc[c]);
                const __half h = __float2half_rn(v);
                hi[c][i] = h;
                lo[c][i] = __float2half_rn(__fsub_rn(v, __half2float(h)));
            }
        }
        // operand row j of the strip: 64 reduction values = 8 chunks of 16 B; chunk index swizzled by j >> 2
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int j = jq * 4 + c;
            const uint32_t off = (uint32_t)j * 128u + (uint32_t)(((rg >> 1) ^ (jq & 7)) << 4) + (uint32_t)((rg & 1) << 3);
            uint2 ph, pl;
            ph.x = (uint32_t)__half_as_ushort(hi[c][0]) | ((uint32_t)__half_as_ushort(hi[c][1]) << 16);
            ph.y = (uint32_t)__half_as_ushort(hi[c][2]) | ((uint32_t)__half_as_ushort(hi[c][3]) << 16);
            pl.x = (uint32_t)__half_as_ushort(lo[c][0]) | ((uint32_t)__half_as_ushort(lo[c][1]) << 16);
            pl.y = (uint32_t)__half_as_ushort(lo[c][2]) | ((uint32_t)__half_as_ushort(lo[c][3]) << 16);
            *reinterpret_cast<uint2 *>(tile_hi + off) = ph;
            *reinterpret_cast<uint2 *>(tile_lo + off) = pl;
        }
        __syncthreads();
#pragma unroll
        for (int it = 0; it < 2; ++it) {
            const int j = (t >> 3) + 32 * it, ch = t & 7;
            const uint32_t off = (uint32_t)j * 128u + (uint32_t)((ch ^ ((j >> 2) & 7)) << 4);
            const size_t o = (size_t)(o0 + j) * (size_t)Np + (size_t)tile * PT + (size_t)ch * 8;
            *reinterpret_cast<uint4 *>(Ohi + o) = *reinterpret_cast<const uint4 *>(tile_hi + off);
            *reinterpret_cast<uint4 *>(Olo + o) = *reinterpret_cast<const uint4 *>(tile_lo + off);
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < 4; ++i) cur[i] = nxt[i];
    }
    // column statistics of the strip: 16 row groups summed in a fixed order
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
        for (int c = 0; c < 4; ++c) red[rg][jq * 4 + c] = pass ? q[c] : a[c];
        __syncthreads();
        if (t < PT) {
            double s = 0.0;
#pragma unroll
            for (int k = 0; k < 16; ++k) s += red[k][t];
            (pass ? part_sq : part)[(size_t)blockIdx.y * mtot + o0 + t] = s;
        }
        __syncthreads();
    }
}

// T[o] = sum of the split partials (fixed order), SQ likewise; the caller's column sums:
// out[col] = T + N * ((double)shift - bias)   (sx for the X part, sy for the Y part)
__global__ void __launch_bounds__(128)
tc2_stat_finish(const double *__restrict__ part, const double *__restrict__ part_sq, int nsplit_used, int mtot, Cols C,
                const float *__restrict__ shift, const float *__restrict__ y_bias, double Nd, double *__restrict__ T,
                double *__restrict__ SQ, double *__restrict__ sx, double *__restrict__ sy) {
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= mtot) return;
    double v[RS], w[RS];
#pragma unroll
    for (int r = 0; r < RS; ++r) {
        v[r] = r < nsplit_used ? part[(size_t)r * mtot + o] : 0.0;
        w[r] = r < nsplit_used ? part_sq[(size_t)r * mtot + o] : 0.0;
    }
    double t = 0.0, t2 = 0.0;
#pragma unroll
    for (int r = 0; r < RS; ++r) { t += v[r]; t2 += w[r]; }
    T[o] = t;
    SQ[o] = t2;
    if (o < C.Kp) {
        if (sx && o < C.K) sx[o] = t + Nd * (double)shift[o];
    } else if (sy && o - C.Kp < C.n) {
        const int j = o - C.Kp;
        sy[j] = t + Nd * ((double)shift[o] - (y_bias ? (double)y_bias[j] : 0.0));
    }
}

// ------------------------------------------------------------------ reduction of the row splits
// CTA = 32 rows x 128 columns of a tile; thread = 4 consecutive columns x 4 rows (float4 loads of every split's partial,
// all issued before the first use).
//   C[i,j] = inv_i inv_j sum_s P_s[i,j] + uA_i TB_j + TA_i uB_j + N uA_i uB_j,   u = (double)shift32 - bias.
// G tiles: the diagonal tile reads the upper element for both (i,j) and (j,i) (the tensor core produced them with
// different rounding; G must be bitwise symmetric), tiles above it are also written transposed (the lower triangle of G)
// through shared memory.
__global__ void __launch_bounds__(256)
reduce_tc2(const float *__restrict__ partial, int nsplit, int ntiles, int tiles_sym, int tjx, int tjy0, int tnb, int Kp,
           const float *__restrict__ shift, const double *__restrict__ inv, const double *__restrict__ T,
           const double *__restrict__ SQ, const float *__restrict__ y_bias, double Nd, int K, int n,
           double *__restrict__ G, double *__restrict__ Bxy) {
    constexpr int TR = TILE;
    __shared__ double tr[32][129];
    int ti, tj;
    const bool sym = (int)blockIdx.x < tiles_sym;
    decode_tile(blockIdx.x, tiles_sym, tjx, tjy0, tnb, ti, tj);
    const int rowbase = ti * TR, colbase = tj * TN;  // colbase in operand space
    const int sr = blockIdx.y, i0 = rowbase + sr * 32;
    if (i0 >= K) return;
    const int Nn = sym ? K : n;
    const int coff = sym ? 0 : Kp;  // operand index of column 0 of C
    const int oj0 = colbase + blockIdx.z * 128, j0 = oj0 - coff;
    if (j0 >= Nn) return;
    const int rb128 = i0 >> 7, cb128 = j0 >> 7;
    if (sym && cb128 < rb128) return;
    const bool dblock = sym && cb128 == rb128, upper = sym && cb128 > rb128;
    const size_t tile_elems = (size_t)TR * TN, split_stride = (size_t)ntiles * tile_elems;
    const float *p0 = partial + (size_t)blockIdx.x * tile_elems;
    double *__restrict__ Cm = sym ? G : Bxy;
    const int64_t ldc = sym ? K : n;
    const int cq = threadIdx.x & 31, rl = threadIdx.x >> 5;
    const int jc = j0 + cq * 4, ojc = oj0 + cq * 4;  // first of this thread's 4 columns
    const int ec0 = blockIdx.z * 128 + cq * 4;        // ... inside the tile

    double sv[4][4];
    if (!dblock) {
        double d[4][4];
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
            for (int e = 0; e < 4; ++e) d[p][e] = 0.0;
        for (int c = 0; c < nsplit; ++c) {
            float4 v[4];
#pragma unroll
            for (int p = 0; p < 4; ++p)
                v[p] = __ldg(reinterpret_cast<const float4 *>(p0 + (size_t)c * split_stride +
                                                              (size_t)(sr * 32 + rl + 8 * p) * TN + ec0));
#pragma unroll
            for (int p = 0; p < 4; ++p) {
                d[p][0] += (double)v[p].x; d[p][1] += (double)v[p].y; d[p][2] += (double)v[p].z; d[p][3] += (double)v[p].w;
            }
        }
        double invj[4], ubj[4], Tj[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const bool ok = jc + e < Nn;
            invj[e] = ok ? inv[ojc + e] : 0.0;
            Tj[e] = ok ? T[ojc + e] : 0.0;
            ubj[e] = ok ? (double)shift[ojc + e] - ((!sym && y_bias) ? (double)y_bias[jc + e] : 0.0) : 0.0;
        }
        const bool vec2 = ((ldc & 1) == 0) && (jc + 3 < Nn) && ((reinterpret_cast<uintptr_t>(Cm) & 15) == 0);
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const int i = i0 + rl + 8 * p;
            if (i < K) {
                const double invi = inv[i], ua = (double)shift[i], Ti = T[i];
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    sv[p][e] = d[p][e] * (invi * invj[e]) + (ua * Tj[e] + Ti * ubj[e] + Nd * ua * ubj[e]);
                double *dst = Cm + (int64_t)i * ldc + jc;
                if (vec2) {
                    *reinterpret_cast<double2 *>(dst) = make_double2(sv[p][0], sv[p][1]);
                    *reinterpret_cast<double2 *>(dst + 2) = make_double2(sv[p][2], sv[p][3]);
                } else {
#pragma unroll
                    for (int e = 0; e < 4; ++e)
                        if (jc + e < Nn) dst[e] = sv[p][e];
                }
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) sv[p][e] = 0.0;
            }
        }
    } else {
        // diagonal 128-block: element-wise, (i > j) reads the mirrored element
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const int lr = rl + 8 * p, i = i0 + lr;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int j = jc + e;
                double s = 0.0;
                if (i < K && j < K) {
                    int er = sr * 32 + lr, ec = ec0 + e;
                    if (i > j) {
                        const int nr = (colbase + ec) - rowbase, nc = (rowbase + er) - colbase;
                        er = nr;
                        ec = nc;
                    }
                    for (int c = 0; c < nsplit; ++c) s += (double)p0[(size_t)c * split_stride + (size_t)er * TN + ec];
                    s *= inv[i] * inv[j];
                    if (i == j) s = SQ[i];
                    const double ua = (double)shift[i], ub = (double)shift[j];
                    s += ua * T[j] + T[i] * ub + Nd * ua * ub;
                    G[(int64_t)i * K + j] = s;
                }
                sv[p][e] = s;
            }
        }
    }
    if (upper) {  // the transposed copy: G[j][i] for the 32 x 128 strip (CTA-uniform condition)
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
            for (int e = 0; e < 4; ++e) tr[rl + 8 * p][cq * 4 + e] = sv[p][e];
        __syncthreads();
        const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll 4
        for (int k = 0; k < 16; ++k) {
            const int col = w * 16 + k;
            const int j = j0 + col, i = i0 + lane;
            if (i < K && j < K) G[(int64_t)j * K + i] = tr[lane][col];
        }
    }
}

}  // namespace

bool cp_gram_tc_eligible(const float *X, int64_t N, int K, int64_t ldx, const void *Yraw, int y_dtype, int n, int64_t ldy,
                         const int32_t *rows, bool wantB) {
    if (rows != nullptr || N < 64 || K < 64) return false;
    if ((((uintptr_t)X) & 15) || (ldx % 4)) return false;  // 16-byte vector loads of the statistics / preparation passes
    if (wantB && (y_dtype != CP_F32 || (((uintptr_t)Yraw) & 15) || (ldy % 4) || n < 1)) return false;
    return true;
}

int cp_gram_tc2(cp_handle_t h, const float *X, int64_t N, int K, int64_t ldx, const void *Yraw, int y_dtype, int n,
                int64_t ldy, const float *y_bias, const int32_t *rows, int nrows, double *G, double *Bxy, double *sx,
                double *sy, double *yy, cudaStream_t stream) {
    const bool wantB = Bxy != nullptr;
    if (yy != nullptr || !cp_gram_tc_eligible(X, N, K, ldx, Yraw, y_dtype, n, ldy, rows, wantB || sy != nullptr))
        return cp_gram_fp64_products(h, X, N, K, ldx, Yraw, y_dtype, n, ldy, y_bias, rows, nrows, G, Bxy, sx, sy, yy, stream);
    if (sy != nullptr && !wantB)  // column sums of Y alone: nothing for the tensor cores to do
        return cp_gram_fp64_products(h, X, N, K, ldx, Yraw, y_dtype, n, ldy, y_bias, rows, nrows, G, Bxy, sx, sy, yy, stream);
    const int tjx = cp_cdiv(K, TN), tk = tjx;
    const int Kp = tjx * TN;
    const int tnb = wantB ? cp_cdiv(n, TN) : 0;
    const int np_ = tnb * TN;
    const int mtot = Kp + np_;
    int tiles_sym = 0;
    if (G)
        tiles_sym = tk * (tk + 1) / 2;
    const int ntiles = tiles_sym + tk * tnb;
    const int64_t Np = cp_cdiv(N, KS) * (int64_t)KS;
    const int units = h->num_sms;  // CTAs working concurrently

    // Row splits.  An item (tile x split) costs its stages (~1.2 us each) plus a small hand-over; items run
    // round-robin on the persistent grid; every split adds one fp32 partial per tile (written, then read by the
    // reduction).  A split is a multiple of the accumulator run and at most 4096 rows (the fp32 register sums
    // stay below 4e-7 of the partial sum whatever N is).
    constexpr int64_t SUB = SUB_STAGES * KS, MAX_SPLIT_ROWS = 4096;
    const int ns_min = (int)cp_cdiv(N, MAX_SPLIT_ROWS);
    int nsplit = ns_min, rps = (int)(cp_cdiv(cp_cdiv(N, ns_min), SUB) * SUB);
    if (ntiles > 0) {
        double best = 1e300;
        const int max_ns = (int)cp_cdiv(N, SUB);
        for (int ns = ns_min; ns <= max_ns && ns < ns_min + 32; ++ns) {
            const int64_t r = cp_cdiv(cp_cdiv(N, ns), SUB) * SUB;
            const int ns_eff = (int)cp_cdiv(N, r);
            const double rounds = (double)cp_cdiv((int64_t)ntiles * ns_eff, units);
            const double cost = rounds * (1.2 * (double)(r / KS) + 1.0) +
                                (double)ns_eff * (2.0 * ntiles * TILE * TN * 4.0 / 3.0e6);  // HBM bytes per us
            if (cost < best * 0.98) {
                best = cost;
                nsplit = ns_eff;
                rps = (int)r;
            }
        }
    }

    const size_t part_elems = (size_t)nsplit * ntiles * TILE * TN;
    const size_t op_elems = 2 * (size_t)mtot * (size_t)Np;  // hi rows, then lo rows
    const size_t need = cp_carver::need(part_elems, 4) + cp_carver::need(op_elems, 2) + 3 * cp_carver::need(mtot, 8) +
                        2 * cp_carver::need((size_t)RS * mtot, 8) + cp_carver::need((size_t)RS * mtot, 4) +
                        2 * cp_carver::need(mtot, 4);
    void *ws = nullptr;
    int rc = cp_ws_reserve(h, need, &ws);
    if (rc) return rc;
    cp_carver cv(ws);
    float *partial = cv.take<float>(part_elems);
    __half *ops = cv.take<__half>(op_elems);
    double *T = cv.take<double>(mtot), *SQ = cv.take<double>(mtot), *inv = cv.take<double>(mtot);
    double *cpart = cv.take<double>((size_t)RS * mtot), *cpart_sq = cv.take<double>((size_t)RS * mtot);
    float *cpart_max = cv.take<float>((size_t)RS * mtot);
    float *shift = cv.take<float>(mtot), *scale = cv.take<float>(mtot);
    const double invN = 1.0 / (double)N, Nd = (double)N;
    __half *Ohi = ops, *Olo = ops + (size_t)mtot * (size_t)Np;
    const int64_t ntile_rows = Np / PT;
    const int tiles_per_split = cp_cdiv(ntile_rows, RS);
    const int splits_used = cp_cdiv(ntile_rows, tiles_per_split);
    Cols C{X, (const float *)Yraw, ldx, ldy, K, wantB ? n : 0, Kp};

    colstat_part<<<dim3(mtot / 128, RS), 256, 0, stream>>>(C, N, mtot, cpart, cpart_max);
    CP_CHECK_LAUNCH();
    colstat_finish<<<cp_cdiv(mtot, 128), 128, 0, stream>>>(cpart, cpart_max, mtot, invN, shift, scale, inv);
    CP_CHECK_LAUNCH();
    tc2_prep<<<dim3(mtot / PT, splits_used), 256, 0, stream>>>(C, N, Np, tiles_per_split, mtot, shift, scale, Ohi, Olo, cpart,
                                                               cpart_sq);
    CP_CHECK_LAUNCH();
    tc2_stat_finish<<<cp_cdiv(mtot, 128), 128, 0, stream>>>(cpart, cpart_sq, splits_used, mtot, C, shift, y_bias, Nd, T, SQ, sx,
                                                            wantB ? sy : nullptr);
    CP_CHECK_LAUNCH();
    if (ntiles > 0) {
        CUtensorMap mapA;
        rc = make_map16(h, &mapA, ops, Np, 2 * (int64_t)mtot, TILE);
        if (rc) return rc;
        Tc2Params P{};
        P.partial = partial; P.Np = Np; P.rows_per_split = rps; P.nsplit = nsplit; P.tiles_sym = tiles_sym; P.tk = tk;
        P.tjx = tjx; P.tjy0 = Kp / TN; P.tnb = tnb; P.ntiles = ntiles; P.mtot = mtot;
        const int nitems = ntiles * nsplit;
        const bool prof = h->gram_profile;
        if (prof) CP_CUDA(cudaEventRecord(h->ev_gram0, stream));
        static cp_per_device_flag configured;
        if (bool *done = configured.slot(); !*done) {
            CP_CUDA(cudaFuncSetAttribute(gram_tc2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
            *done = true;
        }
        const int grid = nitems < units ? nitems : units;
        gram_tc2_kernel<<<grid, NTHREADS, SMEM_BYTES, stream>>>(mapA, P);
        CP_CHECK_LAUNCH();
        if (prof) CP_CUDA(cudaEventRecord(h->ev_gram1, stream));
        reduce_tc2<<<dim3(ntiles, TILE / 32, TN / 128), 256, 0, stream>>>(partial, nsplit, ntiles, tiles_sym, tjx, P.tjy0, tnb, Kp,
                                                                         shift, inv, T, SQ, y_bias, Nd, K, n, G, Bxy);
        CP_CHECK_LAUNCH();
    }
    return CP_OK;
}
