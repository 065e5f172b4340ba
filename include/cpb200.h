/*
 * cpb200 -- C ABI of the H100-native channel-pruning solver (libcpb200.so).
 *
 * The reference (ethanhe42/channel-pruning) has no FFI of its own for this path:
 * the hot path is Python calling numpy / scikit-learn / scipy (SURVEY.md 8b).  Each
 * entry point below replaces one piece of that Python/third-party arithmetic; the
 * reference location it stands in for is cited per function.  The host side that
 * mirrors the reference's Python interface (lib/decompose.py, lib/net.py) lives in
 * channel-pruning_b200/lib/ and binds these symbols with cffi (ABI mode).
 *
 * Conventions
 *   - plain C: raw device pointers, sizes, a cudaStream_t passed as void*.
 *   - every call is asynchronous and stream-ordered on `stream`; nothing
 *     synchronises unless stated.  Outputs live in caller-owned device memory.
 *   - the handle owns only scratch workspace (grown on demand) and is bound to one
 *     device; one handle per process/GPU; a handle must not be used from two
 *     streams concurrently (use one handle per stream).
 *   - return value: CP_OK (0), <0 invalid argument, >0 CUDA / numerical failure;
 *     cp_last_error() returns a thread-local message for the last failure.
 *   - column order of a patch matrix X (N x K, K = c*k*k) is the reference's
 *     (c, kh, kw): column = a*k*k + p  (lib/net.py:1702 rollaxis -> (N,c,k,k)).
 *   - row order of gathered matrices is the reference's (batch, point, image):
 *     row = (batch*P + point)*B + image  (lib/net.py:509-513, 640).
 */
#ifndef CPB200_H
#define CPB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct cp_handle_s *cp_handle_t;
typedef void *cp_stream_t; /* cudaStream_t */

enum {
    CP_OK = 0,
    CP_ERR_INVALID = -1,
    CP_ERR_CUDA = 1,
    CP_ERR_NOT_SPD = 2,
    CP_ERR_WORKSPACE = 3
};

/* feature-map layouts accepted by the gather kernels */
enum { CP_LAYOUT_NCHW = 0, CP_LAYOUT_NHWC = 1 };

/* element types.  Y operand of cp_gram and the solvers: CP_F32 or CP_F64 (a caller of the Python-level
 * decompose.dictionary may hand over float64 targets, which are then used exactly).  Feature map of the gathers
 * (cp_patch_gather_typed / cp_point_gather_typed): CP_F32, CP_BF16 or CP_F16 -- what a 16-bit forward pass
 * (autocast, channels_last) produces; the gathered X and Y are fp32 either way, widened exactly. */
enum { CP_F32 = 0, CP_F64 = 1, CP_BF16 = 2, CP_F16 = 3 };

/* arithmetic of cp_gram */
enum {
    CP_GRAM_FP64 = 0,  /* fp32 inputs widened to fp64, DMMA accumulate (exact products) */
    CP_GRAM_3XTF32 = 1 /* tensor cores (wgmma), three products of a 22-bit hi/lo operand split, fp32 register
                          accumulation per 64-row run, fp64 reduction over the runs.  The split is into two fp16
                          halves of the shifted and power-of-two scaled data (the same split precision as tf32 at
                          twice the rate; csrc/gram_tc2.cu); the name of the constant is kept for source
                          compatibility. */
};

int cp_version(void);
const char *cp_last_error(void);

int cp_create(cp_handle_t *out, int device);
int cp_destroy(cp_handle_t h);
/* number of CUDA kernels this library has launched in the process so far (diagnostics; bench.py
 * reports the per-step difference as gpu_launches) */
int64_t cp_launch_count(void);
/* bytes of scratch currently owned by the handle (diagnostics) */
int64_t cp_workspace_bytes(cp_handle_t h);
/* Diagnostics for the roofline of the tensor-core Gram kernel: with profiling enabled, cp_gram (mode CP_GRAM_3XTF32)
 * records CUDA events on its stream right before and after the tensor-core GEMM launch; cp_gram_kernel_ms waits for the
 * second event and returns the elapsed time of that launch alone (bench.py divides the algorithmic flops by it). */
int cp_gram_profile(cp_handle_t h, int enable);
/* Arithmetic of the bulk products inside the following cp_ls_solve / cp_ls_factor / cp_ls_resolve calls on this handle
 * (the solver behind LinearRegression.fit, lib/decompose.py:665-666).  0 (default): fp64 (DMMA).  1: Cholesky
 * trailing updates and forward substitutions with >= 256 columns run on the tensor cores in 22-bit split precision
 * (csrc/gemm_tc.cu) -- meant for statistics that came from cp_gram's tensor-core mode and are followed by a
 * refinement step (cp_ls_residual + cp_ls_resolve); the panel factorisations, the panel solves and the pivot-ratio
 * statistic stay fp64.  cp_ls_solve_dual is always fp64, whatever this mode. */
int cp_ls_tensor_cores(cp_handle_t h, int enable);
int cp_gram_kernel_ms(cp_handle_t h, float *ms);

/*
 * Sparse-point im2col -- replaces Net.extract_XY (lib/net.py:534-684, w1=None
 * branch) plus the relu of Net.dictionary_kernel (lib/net.py:1720) when relu != 0.
 *
 *   fmap   : nbatch*B images, layout NCHW (B,c,H,W) or NHWC (B,H,W,c), fp32 (cp_patch_gather) or fmap_dtype
 *            CP_F32 | CP_BF16 | CP_F16 (cp_patch_gather_typed; CP_F64 and other codes return CP_ERR_INVALID).
 *            16-bit values are widened exactly to fp32 and the relu is applied after widening, so X is bit for
 *            bit the X of the fp32 map holding the widened values.  Device memory, or -- NCHW or NHWC --
 *            page-locked host memory mapped under UVA (cudaHostAlloc / pinned torch tensor): the kernel then
 *            reads the sampled windows in place over PCIe with a small persistent grid (the reference keeps
 *            its feature maps in host RAM; only the windows have to cross).  An NHWC host map is read as
 *            whole contiguous window rows, with 16-byte loads when c * element size is a multiple of 16
 *            bytes and the map is 16-byte aligned (csrc/gather_host.cu).
 *            NHWC in device memory with c >= 16, c % 4 == 0 (fp32) or c % 8 == 0 (bf16 / fp16: the 16-byte
 *            stride rule of TMA), and 16-byte aligned fmap / X_out / ldx takes the TMA path
 *            (csrc/gather_tma.cu): one 4-D tensor-map request per k x k x c window, padding taps zero-filled
 *            by the copy engine, the patch row leaves as one bulk store -- 74 % of the HBM copy rate at conv4_x
 *            (NCHW: 24 %; k-float runs cannot be fetched at sector efficiency).  Other NHWC device maps take the
 *            SIMT kernel.  NHWC maps off the TMA path (host or device) accept kernel_size <= 9; a larger one
 *            returns CP_ERR_INVALID.  Results are bit-identical.
 *   randx  : nbatch*P sampled output rows   (points_dict[(batch, Y, "randx")])
 *   randy  : nbatch*P sampled output cols
 *   window : rows [stride*x - pad, +k), cols [stride*y - pad, +k) of the bottom
 *            blob, zero outside (net.py:564-589, 631-632).
 *   X_out  : (nbatch*P*B) x (c*k*k) fp32, leading dimension ldx (elements),
 *            column = a*k*k + py*k + px.
 * cp_patch_gather and cp_patch_gather_typed take the reference's square, odd, undilated window (lib/net.py:534-684;
 * an even k returns CP_ERR_INVALID) and are cp_patch_gather_conv with kh = kw = k, one pad, one stride, dilation 1.
 */
int cp_patch_gather(cp_handle_t h, const float *fmap, int nbatch, int B, int c, int H, int W, int layout,
                    const int32_t *randx, const int32_t *randy, int P, int k, int pad, int stride, int relu,
                    float *X_out, int64_t ldx, cp_stream_t stream);
int cp_patch_gather_typed(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int c, int H, int W,
                          int layout, const int32_t *randx, const int32_t *randy, int P, int k, int pad, int stride,
                          int relu, float *X_out, int64_t ldx, cp_stream_t stream);
/*
 * Patch gather for any torch.nn.Conv2d with groups == 1: rectangular kernels, per-axis padding and stride, dilation.
 * Output point (x, y) reads the taps
 *     (stride_h*x - pad_h + dil_h*i, stride_w*y - pad_w + dil_w*j),  i < kh, j < kw,
 * zero outside the map, into column a*kh*kw + i*kw + j (the order of F.unfold and of W.reshape(n, -1)).  Only the
 * top / left padding enters the window origin; the bottom / right padding only sets the output size, which the
 * sampled points already respect -- so padding='same' with an even kernel is one pad per axis too.  The other
 * arguments are those of cp_patch_gather_typed; ldx >= c*kh*kw.  kh, kw, stride < 1, dilation < 1 or pad < 0 return
 * CP_ERR_INVALID before any device work.
 * Paths, as for the square window: NHWC in device memory takes the TMA kernel when its 16-byte rules hold, both
 * dilations are <= 8, both window spans (k-1)*dil+1 are <= 256 and kh, kw <= 16; other NHWC device maps take the
 * SIMT kernel (kh*kw <= 95); NHWC maps in pinned host memory take the in-place reader (kh*kw <= 81); NCHW maps take
 * the SIMT kernel with any window.  A window beyond a path's bound returns CP_ERR_INVALID.  The two bounds are the
 * contract of the 2-D entries (cp_patch_gather, _typed, _conv), kept from their square windows: the kernels are those
 * of cp_patch_gather_conv3d, which takes larger windows.  Square, odd, undilated windows give the bits of
 * cp_patch_gather_typed.
 */
int cp_patch_gather_conv(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int c, int H, int W,
                         int layout, const int32_t *randx, const int32_t *randy, int P, int kh, int kw, int pad_h,
                         int pad_w, int stride_h, int stride_w, int dil_h, int dil_w, int relu, float *X_out,
                         int64_t ldx, cp_stream_t stream);

/*
 * Patch gather for torch.nn.Conv3d (groups == 1): 3-D maps of video and volumetric networks.
 *   fmap   : nbatch*B images, layout CP_LAYOUT_NCHW meaning NCDHW (B,c,D,H,W) or CP_LAYOUT_NHWC meaning NDHWC
 *            (B,D,H,W,c, channels_last_3d); fmap_dtype CP_F32 | CP_BF16 | CP_F16, widened exactly; device memory or
 *            page-locked host memory (read in place), as for the 2-D gathers.
 *   randt, randx, randy : nbatch*P sampled output points (t, x, y), t < To, x < Ho, y < Wo.
 * Output point (t, x, y) reads the taps
 *     (stride_t*t - pad_t + dil_t*u,  stride_h*x - pad_h + dil_h*i,  stride_w*y - pad_w + dil_w*j),
 * u < kt, i < kh, j < kw, zero outside the map, into column a*kt*kh*kw + (u*kh + i)*kw + j (the order of
 * Conv3d.weight.reshape(n, -1)); relu as in cp_patch_gather_conv.  X_out: (nbatch*P*B) x (c*kt*kh*kw) fp32, ldx >=
 * c*kt*kh*kw.  Before any device work, CP_ERR_INVALID for: an extent, stride or dilation < 1, a padding < 0, more
 * than 4096 taps, or an empty output map ((in + 2 pad - dil (k - 1) - 1) / stride + 1 < 1 on an axis).
 * Paths: NDHWC in device memory takes the TMA kernel (5-D tensor map, one request per window and channel box) under
 * the rules of the 2-D TMA path (16-byte rules, c >= 16, every extent <= 16, dilations <= 8, spans <= 256); NDHWC in
 * pinned host memory the in-place reader (kt*kh*kw <= 343, else CP_ERR_INVALID); other NDHWC device maps the SIMT
 * kernel; NCDHW maps the SIMT kernel.  Results are bit-identical across paths.
 */
int cp_patch_gather_conv3d(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int c, int D, int H,
                           int W, int layout, const int32_t *randt, const int32_t *randx, const int32_t *randy, int P,
                           int kt, int kh, int kw, int pad_t, int pad_h, int pad_w, int stride_t, int stride_h,
                           int stride_w, int dil_t, int dil_h, int dil_w, int relu, float *X_out, int64_t ldx,
                           cp_stream_t stream);

/*
 * Patch gathers for torch.nn.ConvTranspose2d / ConvTranspose3d (groups == 1): the up-convolutions of U-Net and
 * 3-D U-Net decoders, FCN heads, DCGAN-style generators.
 *   fmap   : the transposed convolution's INPUT map, nbatch*B images of c x H x W (3-D: c x D x H x W), layout, dtype
 *            and memory (device or pinned host, read in place) as for cp_patch_gather_conv / _conv3d.
 *   randx, randy (3-D: randt, randx, randy) : nbatch*P sampled points of its OUTPUT map.
 *   kh, kw, pad, stride, dil : the arguments of nn.ConvTranspose2d (kernel_size, padding, stride, dilation) per axis.
 * Output point (x, y) reads, for tap (i, j), the input pixel
 *     h = (x + pad_h - dil_h*i) / stride_h,   w = (y + pad_w - dil_w*j) / stride_w
 * when both divisions are exact and 0 <= h < H, 0 <= w < W, otherwise 0 (3-D: the depth axis likewise), into column
 * a*kh*kw + i*kw + j (3-D: a*kt*kh*kw + (u*kh + i)*kw + j), the conv gathers' order.  So
 * X_out @ weight.transpose(0, 1).reshape(n, -1).T is the transposed convolution's output at the points, minus its bias.
 * output_padding only sets the output map's size, which the sampled points already respect: it is no argument.
 * relu as in cp_patch_gather_conv.  X_out: (nbatch*P*B) x (c*kh*kw) (3-D: c*kt*kh*kw) fp32, leading dimension ldx.
 * Before any device work, CP_ERR_INVALID with a message for: an unknown dtype or layout, a NULL pointer, a bad shape,
 * an extent, stride or dilation < 1, a padding < 0, more than 4096 taps, ldx below c*kh*kw (c*kt*kh*kw).  Every tap is
 * range-checked, so no window is refused for leaving the output map empty.
 * Paths (csrc/gather_tr.cu), bit-identical: channels first one CTA per output row; channels last per (row, channel
 * tile) with the touched pixels' channels staged in shared memory; pinned host maps read in place by the same kernels
 * with a small persistent grid.
 */
int cp_patch_gather_conv_transpose(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int c, int H,
                                   int W, int layout, const int32_t *randx, const int32_t *randy, int P, int kh,
                                   int kw, int pad_h, int pad_w, int stride_h, int stride_w, int dil_h, int dil_w,
                                   int relu, float *X_out, int64_t ldx, cp_stream_t stream);
int cp_patch_gather_conv_transpose3d(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int c, int D,
                                     int H, int W, int layout, const int32_t *randt, const int32_t *randx,
                                     const int32_t *randy, int P, int kt, int kh, int kw, int pad_t, int pad_h,
                                     int pad_w, int stride_t, int stride_h, int stride_w, int dil_t, int dil_h,
                                     int dil_w, int relu, float *X_out, int64_t ldx, cp_stream_t stream);

/*
 * Point gather -- replaces the gather of Net.extract_features (lib/net.py:509-519):
 *   Y_out[(batch*P+point)*B + image, j] = fmap[batch*B+image, j, randx, randy].
 * fp32 out (the reference widens to fp64; the bias of lib/net.py:1707 is applied
 * exactly, in fp64, inside cp_gram via y_bias).  The map: fp32 (cp_point_gather), or fmap_dtype CP_F32 | CP_BF16 |
 * CP_F16 (cp_point_gather_typed), widened exactly.
 */
int cp_point_gather(cp_handle_t h, const float *fmap, int nbatch, int B, int n, int H, int W, int layout,
                    const int32_t *randx, const int32_t *randy, int P, float *Y_out, int64_t ldy,
                    cp_stream_t stream);
int cp_point_gather_typed(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int n, int H, int W,
                          int layout, const int32_t *randx, const int32_t *randy, int P, float *Y_out, int64_t ldy,
                          cp_stream_t stream);
/* The same for the output map of a Conv3d consumer, (B,n,D,H,W) (CP_LAYOUT_NCHW: NCDHW) or (B,D,H,W,n)
 * (CP_LAYOUT_NHWC: NDHWC):  Y_out[(batch*P+point)*B + image, j] = fmap[batch*B+image, j, randt, randx, randy].
 * An empty map (n, D, H or W < 1) returns CP_ERR_INVALID. */
int cp_point_gather3d(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int n, int D, int H, int W,
                      int layout, const int32_t *randt, const int32_t *randx, const int32_t *randy, int P,
                      float *Y_out, int64_t ldy, cp_stream_t stream);

/*
 * Tall-skinny Gram / cross products -- replaces the O(N K^2) arithmetic inside
 * LinearRegression.fit (lib/decompose.py:665-666) and the Z / Lasso.fit data passes
 * (lib/decompose.py:428-434,457) by sufficient statistics (SURVEY.md 7.1):
 *
 *   G   = X' X  (K x K, full symmetric, row-major fp64)          [may be NULL]
 *   Bxy = X' Y  (K x n, row-major fp64), Y = fp64(Yraw) - y_bias [may be NULL]
 *   sx  = 1' X  (K),  sy = 1' Y (n),  yy = sum(Y**2) (1 double)  [each may be NULL]
 *
 *   X : N x K fp32, leading dimension ldx.   Yraw : N x n (y_dtype CP_F32 | CP_F64), leading dimension ldy.
 *   y_bias : n fp32 or NULL.
 *   rows : nrows int32 row indices (repetitions allowed -- the reference samples
 *          with replacement, lib/decompose.py:425) or NULL for all N rows.
 */
int cp_gram(cp_handle_t h, const float *X, int64_t N, int K, int64_t ldx, const void *Yraw, int y_dtype, int n,
            int64_t ldy, const float *y_bias, const int32_t *rows, int nrows, double *G, double *Bxy,
            double *sx, double *sy, double *yy, int mode, cp_stream_t stream);

/*
 * LASSO sufficient statistics in channel space -- replaces the construction of
 * Z (lib/decompose.py:428-434) and sklearn's centring of (Z, reY):
 *   Q[a,b] = sum_{p,q} Gs[(a,p),(b,q)] * WW[(a,p),(b,q)] - m zbar_a zbar_b
 *   qv[a]  = sum_{p,j} W2[j,(a,p)] * Bs[(a,p),j]          - m zbar_a ybar
 *   yn2    = yy_s - m ybar^2,       m = S*n
 * Gs/Bs/sxs/sys/yys : cp_gram over the S sampled rows;  WW/sw : cp_gram of W2
 * viewed as an (n x c*k2) matrix.  Outputs: Q (c x ldq, ldq even >= c, padding column
 * zeroed so that rows are 16-byte aligned for cp_lasso_select), qv (c), yn2 (1), fp64.
 */
int cp_lasso_build(cp_handle_t h, const double *Gs, const double *Bs, const double *sxs, const double *sys,
                   const double *yys, const double *WW, const double *sw, const float *W2, int c, int k2,
                   int n, int S, double *Q, int ldq, double *qv, double *yn2, cp_stream_t stream);

/*
 * Channel selection -- replaces the alpha search of decompose.dictionary
 * (lib/decompose.py:489-525) including every Lasso.fit it performs
 * (sklearn _cd_fast.enet_coordinate_descent: random coordinate order from a 32-bit
 * xorshift seeded per fit, warm start, tol / duality-gap stopping rule, gap-safe
 * screening), evaluated in Gram arithmetic, fp64, in ONE launch (one warp: the search is a
 * serial dependency chain).  Q: c x ldq row-major, ldq even, base 16-byte aligned, any
 * padding column zero; it need not be bitwise symmetric (cp_lasso_build's is not): the update
 * of coordinate j reads row j, as the model oracle/cd_oracle.c:cp_enet_cd_gram does.
 *
 *   right0        : cfgs.alpha on entry (lib/decompose.py:491)
 *   rank, lbound, rbound : target count and acceptance window (:492-501)
 *   seeds         : max_probes uint32, the values rng.randint(0, 2**31-1) would
 *                   return for successive fits (host draws them)
 *   out_idxs      : c bytes (coef != 0)          out_coef : c doubles
 *   out_scalars   : [alpha, n_probes, status, nnz]  (status 0 ok, 1 probe cap hit)
 *   out_probe_log : max_probes x 4 doubles (alpha, nnz, n_iter, gap)
 */
int cp_lasso_select(cp_handle_t h, const double *Q, int ldq, const double *qv, const double *yn2, int c, double m,
                    int rank, double lbound, double rbound, double right0, double tol, int max_iter,
                    const uint32_t *seeds, int max_probes, uint8_t *out_idxs, double *out_coef,
                    double *out_scalars, double *out_probe_log, cp_stream_t stream);

/*
 * Data-form coordinate descent (benchmark kernel; SURVEY.md 8b/8d "LASSO data-form CD: 4 m c bytes per sweep") --
 * the algorithm sklearn runs for the reference's Lasso.fit(Z, reY) (lib/decompose.py:428-457), on the MATERIALISED
 * design matrix instead of its Gram matrix.  The product path never forms Z (cp_lasso_build + cp_lasso_select).
 *
 * cp_lasso_dataform_build: Z (m = S*n rows, c columns, fp32, COLUMN major, leading dimension ldz) and y (m, fp64):
 *   Z[a*ldz + s*n + t] = sum_p X[samples[s], a*k2 + p] * W2[t, a*k2 + p],   y[s*n + t] = Y[samples[s], t] - y_bias[t]
 *   (lib/decompose.py:428-437).
 * cp_lasso_cd_dataform: ONE Lasso.fit at `alpha` (l1_reg = alpha*m), warm start from / result in w (c, fp64):
 *   enet_coordinate_descent with selection='random' (32-bit xorshift from `seed`), tol / duality-gap stopping rule,
 *   no screening; centring of Z and y implicit.  Coordinates are processed 8 at a time with exact sequential
 *   semantics (see csrc/lasso_df.cu); Z is streamed from HBM once per sweep.
 *   out_scalars: [n_iter, gap, tol*|yc|^2, sweeps, gap checks].  Cooperative launch: synchronises `stream` once
 *   before the launch (one scalar read-back).
 */
int cp_lasso_dataform_build(cp_handle_t h, const float *X, int64_t N, int K, int64_t ldx, const float *W2, int n, int c,
                            int k2, const int32_t *samples, int S, const void *Yraw, int y_dtype, int64_t ldy,
                            const float *y_bias, float *Z_out, int64_t ldz, double *y_out, cp_stream_t stream);
int cp_lasso_cd_dataform(cp_handle_t h, const float *Z, int64_t ldz, const double *y, int m, int c, double alpha,
                         double tol, int max_iter, uint32_t seed, double *w, double *out_scalars, cp_stream_t stream);

/*
 * Least-squares reconstruction on the surviving channels -- replaces fc_kernel /
 * LinearRegression(fit_intercept=True).fit (lib/decompose.py:622-623, 665-669) by
 * the centred normal equations on the principal sub-block of G:
 *   Gc = G[sel,sel] - sx sx'/N,  Bc = Bxy[sel,:] - sx sy'/N,  Gc W = Bc  (blocked Cholesky)
 *   b  = (sy - sx' W)/N
 * sel_cols : Ksel int32 column indices (device), ascending; NULL = all K columns (Ksel == K).
 * W_out : n x Ksel fp64 row-major (== coef_, i.e. newW2.reshape(n, c', k, k));
 * b_out : n fp64.  info_out : 1 int32 (0 ok, j>0: pivot j fell below 1e-12 of its original diagonal entry --
 * the squared form of the sigma < 1e-6 sigma_max cut-off of LinearRegression, sklearn _base.py:752-753).
 * stat_out : NULL or 1 double: the smallest pivot / original-diagonal ratio met (1 - R^2 of the most collinear
 * column given its predecessors) -- the caller's conditioning signal for choosing the Gram arithmetic.  A failed
 * pivot enters with its own ratio (<= 1e-12; a NaN or non-positive pivot, or an all-zero column, as 1e-300).
 * Requires N - 1 >= Ksel (otherwise use cp_ls_solve_dual).
 */
int cp_ls_solve(cp_handle_t h, const double *G, const double *Bxy, const double *sx, const double *sy,
                int64_t N, int K, int n, const int32_t *sel_cols, int Ksel, double *W_out, double *b_out,
                int32_t *info_out, double *stat_out, cp_stream_t stream);

/*
 * Minimum-norm least squares for N - 1 < Ksel (what gelsd returns for the
 * rank-deficient case, lib/decompose.py:665-666 at small N): dual normal
 * equations  (Xc Xc' + (1/N) 1 1') A = Yc,  W = Xc' A.
 * X : N x K fp32 (ldx);  Yraw/y_bias as in cp_gram.
 */
int cp_ls_solve_dual(cp_handle_t h, const float *X, int64_t N, int K, int64_t ldx, const void *Yraw, int y_dtype,
                     int n, int64_t ldy, const float *y_bias, const int32_t *sel_cols, int Ksel, double *W_out,
                     double *b_out, int32_t *info_out, double *stat_out, cp_stream_t stream);

/*
 * Factor once, refit many -- replaces the loop of nonlinear_fc (lib/decompose.py:671-685): 50 calls of
 * fc_kernel(X, U, ret_reg=True) with the SAME X and changing targets U.  cp_ls_factor keeps the Cholesky factor
 * of the centred Gram of the selected columns inside the handle (until the next cp_ls_factor on that handle);
 * cp_ls_resolve solves for new targets given their cross products Bxy = X'U (K x n) and column sums sy = 1'U:
 *   W_out (n x Ksel), b_out (n)  as in cp_ls_solve.  sx / sel_cols must be the ones given to cp_ls_factor.
 * cp_ls_solve leaves its factor on the handle too, so cp_ls_resolve can refine that very solve:
 * accumulate != 0 ADDS the solution to W_out / b_out (one step of iterative refinement when Bxy / sy are the cross
 * products and column sums of the residual, see cp_ls_residual).
 */
int cp_ls_factor(cp_handle_t h, const double *G, const double *sx, int64_t N, int K, const int32_t *sel_cols,
                 int Ksel, int32_t *info_out, double *stat_out, cp_stream_t stream);
int cp_ls_resolve(cp_handle_t h, const double *Bxy, const double *sx, const double *sy, int n,
                  const int32_t *sel_cols, double *W_out, double *b_out, int accumulate, cp_stream_t stream);

/*
 * Residual of a least-squares solve, from the DATA (not from the Gram statistics).  mode CP_GRAM_FP64: exact products
 * of the fp32 features with the fp64 weights, fp64 accumulation; mode CP_GRAM_3XTF32: the prediction X W' on the
 * tensor cores (X transposed once, then a product of the cp_gram shape).  Rounded to fp32 on output --
 *   R_out[r, t] = (Y[r, t] - y_bias[t]) - sum_j X[r, sel_j] W[t, j] - b[t]           (N x n, leading dimension ldr)
 * With statistics from the tensor-core Gram (~4e-7 relative), refitting this residual against the same factor
 * (cp_gram of (X, R) + cp_ls_resolve(accumulate = 1)) removes the error the statistics put into W and b: one step of
 * iterative refinement, the reference's LinearRegression.fit (lib/decompose.py:665-666) being the fixed point.
 */
int cp_ls_residual(cp_handle_t h, const float *X, int64_t N, int K, int64_t ldx, const void *Yraw, int y_dtype, int n,
                   int64_t ldy, const float *y_bias, const int32_t *sel_cols, int Ksel, const double *W, const double *b,
                   float *R_out, int64_t ldr, int mode, cp_stream_t stream);

/*
 * The split-precision tensor-core product the solver uses for its bulk updates when cp_ls_tensor_cores is on
 * (csrc/gemm_tc.cu), exposed for tests and measurements: the fp64 matrix products inside LinearRegression.fit's
 * solve (lib/decompose.py:665-666), evaluated with 22 mantissa bits per operand entry on wgmma.
 *   C[m, nn] = alpha * sum_r A[m * lda + r] * B[nn * ldb + r] + beta * C[m * ldc + nn]      (fp64 in, fp64 out)
 * lower bit 0: only the 128 x 128 tiles with row tile >= column tile are touched (M >= Nn); bit 1: B is stored
 * reduction-major, b(nn, r) = B[r * ldb + nn] (the factor's block row in the backward substitution).  R <= 1024.
 */
int cp_gemm_tc_split(cp_handle_t h, int M, int Nn, int R, double alpha, const double *A, int64_t lda, const double *B,
                     int64_t ldb, double beta, double *C, int64_t ldc, int lower, cp_stream_t stream);

/*
 * ---- dense fp64 building blocks of the 3C companions (VH_decompose, nonlinear_fc, ITQ_decompose) ----
 *
 * General product -- replaces the np.dot / np.tensordot / np.matmul calls of lib/decompose.py:85-147, 163-319,
 * 671-685 and reg.predict (:680):
 *   C[m, nn] = alpha * sum_r a(m, r) * b(nn, r) + beta * C[m, nn]          (all fp64, row-major)
 *   a(m, r)  = a_mc ? A[r * lda + m] : A[m * lda + r]
 *   b(nn, r) = b_nc ? B[r * ldb + nn] : B[nn * ldb + r]
 * Tall-skinny shapes (long reduction, few output tiles) are split over CTAs and summed in a fixed order.
 * R = 0 gives C = beta * C (A and B are not read).
 */
int cp_gemm_f64(cp_handle_t h, int a_mc, int b_nc, int M, int Nn, int64_t R, double alpha, const double *A,
                int64_t lda, const double *B, int64_t ldb, double beta, double *C, int64_t ldc, cp_stream_t stream);

/*
 * Singular value decomposition -- replaces scipy.linalg.svd(x, full_matrices=False, lapack_driver='gesvd')
 * (lib/decompose.py:154-156) by a one-sided Jacobi (column pairs orthogonalised in round-robin order, one CTA per
 * pair).  F is m x n, handed over TRANSPOSED: Ft is n rows of length m (row j = column j of F), leading dimension ldf.
 * On return   row j of Ft = sigma_j * u_j  (u_j itself when normalise_left != 0),  row j of Wt (n x n) = the right
 * singular vector v_j,  sigma[j] = sigma_j  -- UNSORTED (the caller orders them; gesvd returns descending order).
 * tol: rotation threshold on |f_p . f_q| / (|f_p| |f_q|) (about sqrt(m) * 2.2e-16).  The number of sweeps is data
 * dependent: this routine synchronises `stream` once per sweep.  m <= 12800.
 */
int cp_svd_jacobi(cp_handle_t h, double *Ft, int m, int n, int64_t ldf, double *Wt, int64_t ldw, double *sigma,
                  int normalise_left, double tol, int max_sweeps, int32_t *sweeps_out, cp_stream_t stream);

/*
 * ReLU-aware target update -- replaces solve_relu (lib/decompose.py:51-59) and the identical block of ITQ_decompose
 * (:231-240), fused with the bias add of the prediction:  RU = RUraw + bias (bias may be NULL);
 *   U = argmin_u (relu(u) - Z)^2 + lambda (u - RU)^2   elementwise (N x n);  colmean_out (n, may be NULL) = U.mean(0).
 */
int cp_solve_relu(cp_handle_t h, const double *RUraw, int64_t ldr, const double *bias, const double *Z, int64_t ldz,
                  double lambda, double *U, int64_t ldu, int64_t N, int n, double *colmean_out, cp_stream_t stream);

/*
 * Column statistics -- replaces ndarray.mean(0) and the centring `Y - Y_mean` (lib/decompose.py:180-182, 242-244):
 *   colsum_out[j] = scale * sum_r X[r, j];   centred_out (may be NULL) = X - colsum_out (use scale = 1/N).
 */
int cp_colstats_f64(cp_handle_t h, const double *X, int64_t ldx, int64_t N, int n, double scale, double *colsum_out,
                    double *centred_out, int64_t ldo, cp_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* CPB200_H */
