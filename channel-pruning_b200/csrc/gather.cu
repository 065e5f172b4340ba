// Sparse-point gathers: the "im2col" of the pruning path.
//
//   cp_patch_gather  <- Net.extract_XY          (reference lib/net.py:534-684) + relu (:1720)
//   cp_point_gather  <- Net.extract_features    (reference lib/net.py:509-519)
//
// Both are pure data movement (HBM bound).  Row r of the output is
// (batch, point, image) = ((r / B) / P, (r / B) % P, r % B), the reference's order.
//
// NCHW path: one CTA per output row; consecutive threads write consecutive columns
// (a*k*k + py*k + px), so stores are fully coalesced; the loads are the sparse part
// (k floats per (channel,row) segment) and are served through L1/L2 at sector
// granularity -- that over-fetch is inherent to reading k-wide windows out of NCHW.
// NHWC path: a window row is k*c contiguous floats; the CTA stages the k*k x c tile
// in shared memory with coalesced loads (channel fastest) and writes it back
// transposed to (c, k*k) column order, again coalesced.  NHWC maps in HBM mostly take the TMA kernel (gather_tma.cu),
// NHWC maps in pinned host memory the in-place reader of gather_host.cu.
// Window: any nn.Conv2d window with groups == 1 (cp_window, cp_patch_gather_conv): kh x kw taps, per-axis pad and
// stride, dilation; the k notation below is the reference's square, undilated case.
// Element type of the map: fp32, bf16 or fp16 (template parameter T, fmap_types.cuh).  X and Y are fp32 in every
// case; the ReLU is applied to the widened value with the fp32 kernel's expression, so -0, inf and NaN come out as the
// fp32 kernel gives them for the widened map.
#include "common.cuh"
#include "fmap_types.cuh"

namespace {

// KS > 0: a square, undilated KS x KS window known at compile time (1 and 3); KS = 0: any window of g
template <int KS, typename T>
__global__ void __launch_bounds__(256)
patch_gather_nchw(const T *__restrict__ fmap, const int32_t *__restrict__ randx,
                  const int32_t *__restrict__ randy, float *__restrict__ X, int64_t ldx, int64_t rows, int B, int c,
                  int H, int W, int P, cp_window g, int relu) {
    const int kw = KS > 0 ? KS : g.kw;
    const int dil_h = KS > 0 ? 1 : g.dil_h, dil_w = KS > 0 ? 1 : g.dil_w;
    const int k2 = KS > 0 ? KS * KS : g.kh * g.kw;
    const int K = c * k2;
    // one CTA per output row when the map is in HBM; a small persistent grid strides over the rows when the
    // map is read in place from pinned host memory (PCIe-bound: more CTAs only block SMs other layers need)
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        const int img_in_batch = (int)(r % B);
        const int64_t bp = r / B;  // batch*P + point
        const int batch = (int)(bp / P);
        const int y0 = g.stride_h * randx[bp] - g.pad_h;  // window origin, rows   (net.py: feat[:,:,x,y], x indexes H)
        const int x0 = g.stride_w * randy[bp] - g.pad_w;  // window origin, cols
        const T *src = fmap + ((int64_t)batch * B + img_in_batch) * c * H * W;
        float *dst = X + r * ldx;
#pragma unroll 4
        for (int col = threadIdx.x; col < K; col += blockDim.x) {
            const int a = col / k2;
            const int p = col - a * k2;
            const int py = p / kw;
            const int px = p - py * kw;
            const int yy = y0 + py * dil_h, xx = x0 + px * dil_w;
            float v = 0.f;
            if (yy >= 0 && yy < H && xx >= 0 && xx < W) v = cp_widen(__ldg(src + ((int64_t)a * H + yy) * W + xx));
            if (relu) v = fmaxf(v, 0.f);
            dst[col] = v;
        }
    }
}

constexpr int64_t CP_HOST_GATHER_CTAS = 64;  // grid of the in-place (zero-copy) reader

// NHWC: tile = kh*kw spatial taps x CT channels staged through shared memory.
constexpr int NHWC_CT = 128;  // channels per tile

template <typename T>
__global__ void __launch_bounds__(256)
patch_gather_nhwc(const T *__restrict__ fmap, const int32_t *__restrict__ randx,
                  const int32_t *__restrict__ randy, float *__restrict__ X, int64_t ldx, int B, int c, int H,
                  int W, int P, cp_window g, int relu) {
    extern __shared__ float tile[];  // [k2][NHWC_CT + 1]
    const int k2 = g.kh * g.kw;
    const int64_t r = blockIdx.x;
    const int a0 = blockIdx.y * NHWC_CT;
    const int ct = min(NHWC_CT, c - a0);
    const int img_in_batch = (int)(r % B);
    const int64_t bp = r / B;
    const int batch = (int)(bp / P);
    const int y0 = g.stride_h * randx[bp] - g.pad_h;
    const int x0 = g.stride_w * randy[bp] - g.pad_w;
    const T *src = fmap + ((int64_t)batch * B + img_in_batch) * H * W * c;
    for (int e = threadIdx.x; e < k2 * ct; e += blockDim.x) {
        const int p = e / ct;
        const int a = e - p * ct;
        const int py = p / g.kw, px = p - py * g.kw;
        const int yy = y0 + py * g.dil_h, xx = x0 + px * g.dil_w;
        float v = 0.f;
        if (yy >= 0 && yy < H && xx >= 0 && xx < W) v = cp_widen(__ldg(src + ((int64_t)yy * W + xx) * c + a0 + a));
        if (relu) v = fmaxf(v, 0.f);
        tile[p * (NHWC_CT + 1) + a] = v;
    }
    __syncthreads();
    float *dst = X + r * ldx + (int64_t)a0 * k2;
    for (int e = threadIdx.x; e < k2 * ct; e += blockDim.x) {
        const int a = e / k2;
        const int p = e - a * k2;
        dst[e] = tile[p * (NHWC_CT + 1) + a];
    }
}

template <typename T>
__global__ void __launch_bounds__(256)
point_gather(const T *__restrict__ fmap, const int32_t *__restrict__ randx,
             const int32_t *__restrict__ randy, float *__restrict__ Y, int64_t ldy, int B, int n, int H, int W,
             int P, int nhwc) {
    const int64_t r = blockIdx.x;
    const int img_in_batch = (int)(r % B);
    const int64_t bp = r / B;
    const int batch = (int)(bp / P);
    const int yy = randx[bp], xx = randy[bp];
    const T *src = fmap + ((int64_t)batch * B + img_in_batch) * n * H * W;
    float *dst = Y + r * ldy;
    if (nhwc) {
        const T *s = src + ((int64_t)yy * W + xx) * n;
        for (int j = threadIdx.x; j < n; j += blockDim.x) dst[j] = cp_widen(__ldg(s + j));
    } else {
        const T *s = src + (int64_t)yy * W + xx;
        for (int j = threadIdx.x; j < n; j += blockDim.x) dst[j] = cp_widen(__ldg(s + (int64_t)j * H * W));
    }
}

}  // namespace

// gather_tma.cu
bool cp_gather_tma_eligible(const void *fmap, int esize, int c, const cp_window &g, float *X_out, int64_t ldx);
int cp_patch_gather_tma(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int c, int H, int W,
                        const int32_t *randx, const int32_t *randy, int P, const cp_window &g, int relu,
                        float *X_out, int64_t ldx, cudaStream_t stream);
// gather_host.cu
int cp_patch_gather_nhwc_host(const void *fmap, int fmap_dtype, int nbatch, int B, int c, int H, int W,
                              const int32_t *randx, const int32_t *randy, int P, const cp_window &g, int relu,
                              float *X_out, int64_t ldx, cudaStream_t stream);

template <typename T>
static void launch_patch_gather_simt(const T *fmap, int layout, bool host_src, int64_t rows,
                                     int B, int c, int H, int W, const int32_t *randx, const int32_t *randy, int P,
                                     const cp_window &g, int relu, float *X_out, int64_t ldx, cudaStream_t stream) {
    if (layout == CP_LAYOUT_NCHW) {
        const int64_t ncta = host_src ? (rows < CP_HOST_GATHER_CTAS ? rows : CP_HOST_GATHER_CTAS) : rows;
        dim3 grid((unsigned)ncta);
        const bool square = g.kh == g.kw && g.dil_h == 1 && g.dil_w == 1;
        if (square && g.kh == 3)
            patch_gather_nchw<3><<<grid, 256, 0, stream>>>(fmap, randx, randy, X_out, ldx, rows, B, c, H, W, P, g, relu);
        else if (square && g.kh == 1)
            patch_gather_nchw<1><<<grid, 256, 0, stream>>>(fmap, randx, randy, X_out, ldx, rows, B, c, H, W, P, g, relu);
        else
            patch_gather_nchw<0><<<grid, 256, 0, stream>>>(fmap, randx, randy, X_out, ldx, rows, B, c, H, W, P, g, relu);
    } else {
        const size_t smem = (size_t)g.kh * g.kw * (NHWC_CT + 1) * sizeof(float);
        dim3 grid((unsigned)rows, (unsigned)cp_cdiv(c, NHWC_CT));
        patch_gather_nhwc<<<grid, 256, smem, stream>>>(fmap, randx, randy, X_out, ldx, B, c, H, W, P, g, relu);
    }
}

// Largest window (kh * kw taps) of the NHWC reader of pinned host maps: the k <= 9 of the square windows.  Its
// channel chunks would still fit a stage beyond it, but no layer it was measured on needs more.
constexpr int CP_HOST_NHWC_MAX_TAPS = 81;

extern "C" int cp_patch_gather_conv(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int c, int H,
                                    int W, int layout, const int32_t *randx, const int32_t *randy, int P, int kh,
                                    int kw, int pad_h, int pad_w, int stride_h, int stride_w, int dil_h, int dil_w,
                                    int relu, float *X_out, int64_t ldx, cp_stream_t stream_) {
    const int esize = cp_fmap_esize(fmap_dtype);
    CP_REQUIRE(esize, "cp_patch_gather: feature-map dtype %d is not CP_F32, CP_BF16 or CP_F16", fmap_dtype);
    CP_REQUIRE(h && fmap && randx && randy && X_out, "cp_patch_gather: NULL argument");
    CP_REQUIRE(nbatch >= 0 && B > 0 && c > 0 && H > 0 && W > 0 && P > 0, "cp_patch_gather: bad shape");
    CP_REQUIRE(kh >= 1 && kw >= 1, "cp_patch_gather: kernel_size %dx%d: both extents must be >= 1", kh, kw);
    CP_REQUIRE(stride_h >= 1 && stride_w >= 1, "cp_patch_gather: stride (%d, %d) must be >= 1", stride_h, stride_w);
    CP_REQUIRE(dil_h >= 1 && dil_w >= 1, "cp_patch_gather: dilation (%d, %d) must be >= 1", dil_h, dil_w);
    CP_REQUIRE(pad_h >= 0 && pad_w >= 0, "cp_patch_gather: padding (%d, %d) must be >= 0", pad_h, pad_w);
    CP_REQUIRE(kh <= 4096 / kw, "cp_patch_gather: kernel_size %dx%d has more than 4096 taps", kh, kw);
    CP_REQUIRE(ldx >= (int64_t)c * kh * kw, "cp_patch_gather: ldx %lld < c*kh*kw", (long long)ldx);
    CP_REQUIRE(layout == CP_LAYOUT_NCHW || layout == CP_LAYOUT_NHWC, "cp_patch_gather: unknown layout %d", layout);
    const cp_window g{kh, kw, pad_h, pad_w, stride_h, stride_w, dil_h, dil_w};
    cudaStream_t stream = (cudaStream_t)stream_;
    const int64_t rows = (int64_t)nbatch * P * B;
    if (rows == 0) return CP_OK;
    CP_REQUIRE(rows < (1ll << 31), "cp_patch_gather: too many rows");
    bool host_src = false;
    if (layout == CP_LAYOUT_NCHW) {
        // map in (pinned, UVA-mapped) host memory?  then the kernel is a PCIe reader: keep its footprint small
        cudaPointerAttributes pa;
        host_src = cudaPointerGetAttributes(&pa, fmap) == cudaSuccess && pa.type == cudaMemoryTypeHost;
        (void)cudaGetLastError();
    } else if (cp_gather_tma_eligible(fmap, esize, c, g, X_out, ldx)) {
        // NHWC map in HBM: whole windows by TMA, rows out by bulk store (gather_tma.cu)
        return cp_patch_gather_tma(h, fmap, fmap_dtype, nbatch, B, c, H, W, randx, randy, P, g, relu, X_out, ldx,
                                   stream);
    } else {
        // NHWC map in pinned host memory: whole window rows as 16-byte reads over PCIe (gather_host.cu)
        cudaPointerAttributes pa;
        const bool host_nhwc = cudaPointerGetAttributes(&pa, fmap) == cudaSuccess && pa.type == cudaMemoryTypeHost;
        (void)cudaGetLastError();
        if (host_nhwc) {
            CP_REQUIRE(kh * kw <= CP_HOST_NHWC_MAX_TAPS,
                       "cp_patch_gather: kernel_size %dx%d too large for the NHWC host reader (kh*kw <= %d)", kh, kw,
                       CP_HOST_NHWC_MAX_TAPS);
            return cp_patch_gather_nhwc_host(fmap, fmap_dtype, nbatch, B, c, H, W, randx, randy, P, g, relu, X_out,
                                             ldx, stream);
        }
        const size_t smem = (size_t)kh * kw * (NHWC_CT + 1) * sizeof(float);
        CP_REQUIRE(smem <= 48 * 1024, "cp_patch_gather: kernel_size %dx%d too large for the NHWC tile", kh, kw);
    }
    if (fmap_dtype == CP_F32)
        launch_patch_gather_simt((const float *)fmap, layout, host_src, rows, B, c, H, W, randx, randy, P, g, relu,
                                 X_out, ldx, stream);
    else if (fmap_dtype == CP_BF16)
        launch_patch_gather_simt((const __nv_bfloat16 *)fmap, layout, host_src, rows, B, c, H, W, randx, randy, P, g,
                                 relu, X_out, ldx, stream);
    else
        launch_patch_gather_simt((const __half *)fmap, layout, host_src, rows, B, c, H, W, randx, randy, P, g, relu,
                                 X_out, ldx, stream);
    CP_CHECK_LAUNCH();
    return CP_OK;
}

extern "C" int cp_patch_gather_typed(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int c, int H,
                                     int W, int layout, const int32_t *randx, const int32_t *randy, int P, int k,
                                     int pad, int stride, int relu, float *X_out, int64_t ldx, cp_stream_t stream_) {
    CP_REQUIRE(k >= 1 && (k & 1) == 1, "cp_patch_gather: kernel_size must be odd (reference net.py:604-605), got %d", k);
    return cp_patch_gather_conv(h, fmap, fmap_dtype, nbatch, B, c, H, W, layout, randx, randy, P, k, k, pad, pad,
                                stride, stride, 1, 1, relu, X_out, ldx, stream_);
}

extern "C" int cp_patch_gather(cp_handle_t h, const float *fmap, int nbatch, int B, int c, int H, int W,
                               int layout, const int32_t *randx, const int32_t *randy, int P, int k, int pad,
                               int stride, int relu, float *X_out, int64_t ldx, cp_stream_t stream_) {
    return cp_patch_gather_typed(h, fmap, CP_F32, nbatch, B, c, H, W, layout, randx, randy, P, k, pad, stride, relu,
                                 X_out, ldx, stream_);
}

extern "C" int cp_point_gather_typed(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int n, int H,
                                     int W, int layout, const int32_t *randx, const int32_t *randy, int P,
                                     float *Y_out, int64_t ldy, cp_stream_t stream_) {
    CP_REQUIRE(cp_fmap_esize(fmap_dtype), "cp_point_gather: feature-map dtype %d is not CP_F32, CP_BF16 or CP_F16",
               fmap_dtype);
    CP_REQUIRE(h && fmap && randx && randy && Y_out, "cp_point_gather: NULL argument");
    CP_REQUIRE(nbatch >= 0 && B > 0 && n > 0 && H > 0 && W > 0 && P > 0, "cp_point_gather: bad shape");
    CP_REQUIRE(ldy >= n, "cp_point_gather: ldy < n");
    CP_REQUIRE(layout == CP_LAYOUT_NCHW || layout == CP_LAYOUT_NHWC, "cp_point_gather: unknown layout %d", layout);
    const int64_t rows = (int64_t)nbatch * P * B;
    if (rows == 0) return CP_OK;
    CP_REQUIRE(rows < (1ll << 31), "cp_point_gather: too many rows");
    const cudaStream_t stream = (cudaStream_t)stream_;
    const int nhwc = layout == CP_LAYOUT_NHWC;
    if (fmap_dtype == CP_F32)
        point_gather<<<(unsigned)rows, 256, 0, stream>>>((const float *)fmap, randx, randy, Y_out, ldy, B, n, H, W, P, nhwc);
    else if (fmap_dtype == CP_BF16)
        point_gather<<<(unsigned)rows, 256, 0, stream>>>((const __nv_bfloat16 *)fmap, randx, randy, Y_out, ldy, B, n, H,
                                                         W, P, nhwc);
    else
        point_gather<<<(unsigned)rows, 256, 0, stream>>>((const __half *)fmap, randx, randy, Y_out, ldy, B, n, H, W, P,
                                                         nhwc);
    CP_CHECK_LAUNCH();
    return CP_OK;
}

extern "C" int cp_point_gather(cp_handle_t h, const float *fmap, int nbatch, int B, int n, int H, int W,
                               int layout, const int32_t *randx, const int32_t *randy, int P, float *Y_out,
                               int64_t ldy, cp_stream_t stream_) {
    return cp_point_gather_typed(h, fmap, CP_F32, nbatch, B, n, H, W, layout, randx, randy, P, Y_out, ldy, stream_);
}
