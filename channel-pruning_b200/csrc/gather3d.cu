// Sparse-point gathers of 3-D feature maps: the im2col of Conv3d consumers (video backbones, volumetric segmentation
// networks), with the semantics of torch.nn.Conv3d (groups == 1, cp_window3).
//
//   cp_patch_gather_conv3d   X (rows, c*kt*kh*kw) of the windows at the sampled output points (t, x, y)
//   cp_point_gather3d        Y (rows, n) of the consumer's output map at the same points
//
// Row r is (batch, point, image) = ((r / B) / P, (r / B) % P, r % B), as in the 2-D gathers (gather.cu); column
// a*kt*kh*kw + (u*kh + i)*kw + j.  Paths, as for 2-D maps:
//   NCDHW, HBM or pinned host     patch_gather_ncdhw: one CTA per row (a small persistent grid for a host map),
//                                 consecutive threads on consecutive columns
//   NDHWC, HBM, TMA rules hold    gather_tma.cu (5-D tensor map)
//   NDHWC, pinned host            gather_host.cu (contiguous window rows by 16-byte cp.async)
//   NDHWC, HBM, otherwise         patch_gather_ndhwc: a kt*kh*kw x CT tile through shared memory
// 16-bit maps are widened exactly (cp_widen) and the ReLU applied after widening, so X is the X of fmap.float().
#include "common.cuh"
#include "fmap_types.cuh"

namespace {

constexpr int64_t CP_HOST_GATHER3D_CTAS = 64;  // grid of the in-place NCDHW reader (that of the NCHW reader)
constexpr int NDHWC_TILE_FLOATS = 12 * 1024;   // shared-memory tile of the NDHWC SIMT kernel: 48 KB

template <typename T>
__global__ void __launch_bounds__(256)
patch_gather_ncdhw(const T *__restrict__ fmap, const int32_t *__restrict__ randt, const int32_t *__restrict__ randx,
                   const int32_t *__restrict__ randy, float *__restrict__ X, int64_t ldx, int64_t rows, int B, int c,
                   int D, int H, int W, int P, cp_window3 g, int relu) {
    const int khw = g.kh * g.kw, k3 = g.kt * khw;
    const int K = c * k3;
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        const int img_in_batch = (int)(r % B);
        const int64_t bp = r / B;
        const int batch = (int)(bp / P);
        const int t0 = g.stride_t * randt[bp] - g.pad_t;
        const int y0 = g.stride_h * randx[bp] - g.pad_h;
        const int x0 = g.stride_w * randy[bp] - g.pad_w;
        const T *src = fmap + ((int64_t)batch * B + img_in_batch) * c * D * H * W;
        float *dst = X + r * ldx;
#pragma unroll 4
        for (int col = threadIdx.x; col < K; col += blockDim.x) {
            const int a = col / k3;
            const int p = col - a * k3;
            const int pu = p / khw, q = p - pu * khw;
            const int py = q / g.kw, px = q - py * g.kw;
            const int tt = t0 + pu * g.dil_t, yy = y0 + py * g.dil_h, xx = x0 + px * g.dil_w;
            float v = 0.f;
            if (tt >= 0 && tt < D && yy >= 0 && yy < H && xx >= 0 && xx < W)
                v = cp_widen(__ldg(src + (((int64_t)a * D + tt) * H + yy) * W + xx));
            if (relu) v = fmaxf(v, 0.f);
            dst[col] = v;
        }
    }
}

// grid (rows, channel tiles); the tile is [k3][ct + 1] floats, ct channels (ct + 1: the transposed read is
// conflict-free)
template <typename T>
__global__ void __launch_bounds__(256)
patch_gather_ndhwc(const T *__restrict__ fmap, const int32_t *__restrict__ randt, const int32_t *__restrict__ randx,
                   const int32_t *__restrict__ randy, float *__restrict__ X, int64_t ldx, int B, int c, int D, int H,
                   int W, int P, cp_window3 g, int ct_tile, int relu) {
    extern __shared__ float tile3[];
    const int khw = g.kh * g.kw, k3 = g.kt * khw;
    const int64_t r = blockIdx.x;
    const int a0 = blockIdx.y * ct_tile;
    const int ct = min(ct_tile, c - a0);
    const int img_in_batch = (int)(r % B);
    const int64_t bp = r / B;
    const int batch = (int)(bp / P);
    const int t0 = g.stride_t * randt[bp] - g.pad_t;
    const int y0 = g.stride_h * randx[bp] - g.pad_h;
    const int x0 = g.stride_w * randy[bp] - g.pad_w;
    const T *src = fmap + ((int64_t)batch * B + img_in_batch) * D * H * W * c;
    for (int e = threadIdx.x; e < k3 * ct; e += blockDim.x) {
        const int p = e / ct;
        const int a = e - p * ct;
        const int pu = p / khw, q = p - pu * khw;
        const int py = q / g.kw, px = q - py * g.kw;
        const int tt = t0 + pu * g.dil_t, yy = y0 + py * g.dil_h, xx = x0 + px * g.dil_w;
        float v = 0.f;
        if (tt >= 0 && tt < D && yy >= 0 && yy < H && xx >= 0 && xx < W)
            v = cp_widen(__ldg(src + (((int64_t)tt * H + yy) * W + xx) * c + a0 + a));
        if (relu) v = fmaxf(v, 0.f);
        tile3[p * (ct_tile + 1) + a] = v;
    }
    __syncthreads();
    float *dst = X + r * ldx + (int64_t)a0 * k3;
    for (int e = threadIdx.x; e < k3 * ct; e += blockDim.x) {
        const int a = e / k3;
        const int p = e - a * k3;
        dst[e] = tile3[p * (ct_tile + 1) + a];
    }
}

template <typename T>
__global__ void __launch_bounds__(256)
point_gather3d(const T *__restrict__ fmap, const int32_t *__restrict__ randt, const int32_t *__restrict__ randx,
               const int32_t *__restrict__ randy, float *__restrict__ Y, int64_t ldy, int B, int n, int D, int H,
               int W, int P, int ndhwc) {
    const int64_t r = blockIdx.x;
    const int img_in_batch = (int)(r % B);
    const int64_t bp = r / B;
    const int batch = (int)(bp / P);
    const int64_t pix = ((int64_t)randt[bp] * H + randx[bp]) * W + randy[bp];
    const int64_t plane = (int64_t)D * H * W;
    const T *src = fmap + ((int64_t)batch * B + img_in_batch) * n * plane;
    float *dst = Y + r * ldy;
    if (ndhwc) {
        const T *s = src + pix * n;
        for (int j = threadIdx.x; j < n; j += blockDim.x) dst[j] = cp_widen(__ldg(s + j));
    } else {
        const T *s = src + pix;
        for (int j = threadIdx.x; j < n; j += blockDim.x) dst[j] = cp_widen(__ldg(s + (int64_t)j * plane));
    }
}

template <typename T>
void launch_ncdhw(const void *fmap, bool host_src, int64_t rows, int B, int c, int D, int H, int W,
                  const int32_t *randt, const int32_t *randx, const int32_t *randy, int P, const cp_window3 &g,
                  int relu, float *X_out, int64_t ldx, cudaStream_t stream) {
    const int64_t ncta = host_src ? (rows < CP_HOST_GATHER3D_CTAS ? rows : CP_HOST_GATHER3D_CTAS) : rows;
    patch_gather_ncdhw<<<(unsigned)ncta, 256, 0, stream>>>((const T *)fmap, randt, randx, randy, X_out, ldx, rows, B,
                                                            c, D, H, W, P, g, relu);
}

template <typename T>
void launch_ndhwc(const void *fmap, int64_t rows, int B, int c, int D, int H, int W, const int32_t *randt,
                  const int32_t *randx, const int32_t *randy, int P, const cp_window3 &g, int ct_tile, int relu,
                  float *X_out, int64_t ldx, cudaStream_t stream) {
    const int k3 = g.kt * g.kh * g.kw;
    const size_t smem = (size_t)k3 * (ct_tile + 1) * sizeof(float);
    dim3 grid((unsigned)rows, (unsigned)cp_cdiv(c, ct_tile));
    patch_gather_ndhwc<<<grid, 256, smem, stream>>>((const T *)fmap, randt, randx, randy, X_out, ldx, B, c, D, H, W, P,
                                                     g, ct_tile, relu);
}

}  // namespace

// gather_tma.cu
bool cp_gather_tma3d_eligible(const void *fmap, int esize, int c, const cp_window3 &g, float *X_out, int64_t ldx);
int cp_patch_gather_tma3d(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int c, int D, int H,
                          int W, const int32_t *randt, const int32_t *randx, const int32_t *randy, int P,
                          const cp_window3 &g, int relu, float *X_out, int64_t ldx, cudaStream_t stream);
// gather_host.cu
int cp_patch_gather_ndhwc_host(const void *fmap, int fmap_dtype, int nbatch, int B, int c, int D, int H, int W,
                               const int32_t *randt, const int32_t *randx, const int32_t *randy, int P,
                               const cp_window3 &w, int relu, float *X_out, int64_t ldx, cudaStream_t stream);

// Largest window (kt * kh * kw taps) of every 3-D path; the NDHWC SIMT tile then holds at least 2 channels
constexpr int CP_GATHER3D_MAX_TAPS = 4096;
// Largest window of the NDHWC reader of pinned host maps: 7 x 7 x 7 (a 3 x 7 x 7 stem is 147)
constexpr int CP_HOST_NDHWC_MAX_TAPS = 343;

static bool cp_is_host_memory(const void *p) {
    cudaPointerAttributes pa;
    const bool host = cudaPointerGetAttributes(&pa, p) == cudaSuccess && pa.type == cudaMemoryTypeHost;
    (void)cudaGetLastError();
    return host;
}

extern "C" int cp_patch_gather_conv3d(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int c,
                                      int D, int H, int W, int layout, const int32_t *randt, const int32_t *randx,
                                      const int32_t *randy, int P, int kt, int kh, int kw, int pad_t, int pad_h,
                                      int pad_w, int stride_t, int stride_h, int stride_w, int dil_t, int dil_h,
                                      int dil_w, int relu, float *X_out, int64_t ldx, cp_stream_t stream_) {
    const int esize = cp_fmap_esize(fmap_dtype);
    CP_REQUIRE(esize, "cp_patch_gather_conv3d: feature-map dtype %d is not CP_F32, CP_BF16 or CP_F16", fmap_dtype);
    CP_REQUIRE(h && fmap && randt && randx && randy && X_out, "cp_patch_gather_conv3d: NULL argument");
    CP_REQUIRE(nbatch >= 0 && B > 0 && c > 0 && D > 0 && H > 0 && W > 0 && P > 0, "cp_patch_gather_conv3d: bad shape");
    CP_REQUIRE(kt >= 1 && kh >= 1 && kw >= 1, "cp_patch_gather_conv3d: kernel_size %dx%dx%d: every extent must be >= 1",
               kt, kh, kw);
    CP_REQUIRE(stride_t >= 1 && stride_h >= 1 && stride_w >= 1,
               "cp_patch_gather_conv3d: stride (%d, %d, %d) must be >= 1", stride_t, stride_h, stride_w);
    CP_REQUIRE(dil_t >= 1 && dil_h >= 1 && dil_w >= 1, "cp_patch_gather_conv3d: dilation (%d, %d, %d) must be >= 1",
               dil_t, dil_h, dil_w);
    CP_REQUIRE(pad_t >= 0 && pad_h >= 0 && pad_w >= 0, "cp_patch_gather_conv3d: padding (%d, %d, %d) must be >= 0",
               pad_t, pad_h, pad_w);
    CP_REQUIRE(kh <= CP_GATHER3D_MAX_TAPS / kw && kt <= CP_GATHER3D_MAX_TAPS / (kh * kw),
               "cp_patch_gather_conv3d: kernel_size %dx%dx%d has more than %d taps", kt, kh, kw, CP_GATHER3D_MAX_TAPS);
    // the output map of nn.Conv3d, (in + 2 pad - dil (k - 1) - 1) / stride + 1 per axis, must not be empty
    CP_REQUIRE((int64_t)D + 2ll * pad_t >= (int64_t)dil_t * (kt - 1) + 1 &&
                   (int64_t)H + 2ll * pad_h >= (int64_t)dil_h * (kh - 1) + 1 &&
                   (int64_t)W + 2ll * pad_w >= (int64_t)dil_w * (kw - 1) + 1,
               "cp_patch_gather_conv3d: empty output map (the dilated window exceeds the padded %dx%dx%d map)", D, H, W);
    const int k3 = kt * kh * kw;
    CP_REQUIRE(ldx >= (int64_t)c * k3, "cp_patch_gather_conv3d: ldx %lld < c*kt*kh*kw", (long long)ldx);
    CP_REQUIRE(layout == CP_LAYOUT_NCHW || layout == CP_LAYOUT_NHWC, "cp_patch_gather_conv3d: unknown layout %d",
               layout);
    const cp_window3 g{kt, kh, kw, pad_t, pad_h, pad_w, stride_t, stride_h, stride_w, dil_t, dil_h, dil_w};
    cudaStream_t stream = (cudaStream_t)stream_;
    const int64_t rows = (int64_t)nbatch * P * B;
    if (rows == 0) return CP_OK;
    CP_REQUIRE(rows < (1ll << 31), "cp_patch_gather_conv3d: too many rows");
    if (layout == CP_LAYOUT_NCHW) {
        const bool host_src = cp_is_host_memory(fmap);
        if (fmap_dtype == CP_F32)
            launch_ncdhw<float>(fmap, host_src, rows, B, c, D, H, W, randt, randx, randy, P, g, relu, X_out, ldx,
                                stream);
        else if (fmap_dtype == CP_BF16)
            launch_ncdhw<__nv_bfloat16>(fmap, host_src, rows, B, c, D, H, W, randt, randx, randy, P, g, relu, X_out,
                                        ldx, stream);
        else
            launch_ncdhw<__half>(fmap, host_src, rows, B, c, D, H, W, randt, randx, randy, P, g, relu, X_out, ldx,
                                 stream);
        CP_CHECK_LAUNCH();
        return CP_OK;
    }
    if (cp_gather_tma3d_eligible(fmap, esize, c, g, X_out, ldx))
        return cp_patch_gather_tma3d(h, fmap, fmap_dtype, nbatch, B, c, D, H, W, randt, randx, randy, P, g, relu,
                                     X_out, ldx, stream);
    if (cp_is_host_memory(fmap)) {
        CP_REQUIRE(k3 <= CP_HOST_NDHWC_MAX_TAPS,
                   "cp_patch_gather_conv3d: kernel_size %dx%dx%d too large for the NDHWC host reader (kt*kh*kw <= %d)",
                   kt, kh, kw, CP_HOST_NDHWC_MAX_TAPS);
        return cp_patch_gather_ndhwc_host(fmap, fmap_dtype, nbatch, B, c, D, H, W, randt, randx, randy, P, g, relu,
                                          X_out, ldx, stream);
    }
    // channels per tile: up to 128, fewer for large windows so the tile stays within 48 KB
    int ct_tile = NDHWC_TILE_FLOATS / k3 - 1;
    ct_tile = ct_tile > 128 ? 128 : ct_tile;
    if (fmap_dtype == CP_F32)
        launch_ndhwc<float>(fmap, rows, B, c, D, H, W, randt, randx, randy, P, g, ct_tile, relu, X_out, ldx, stream);
    else if (fmap_dtype == CP_BF16)
        launch_ndhwc<__nv_bfloat16>(fmap, rows, B, c, D, H, W, randt, randx, randy, P, g, ct_tile, relu, X_out, ldx,
                                    stream);
    else
        launch_ndhwc<__half>(fmap, rows, B, c, D, H, W, randt, randx, randy, P, g, ct_tile, relu, X_out, ldx, stream);
    CP_CHECK_LAUNCH();
    return CP_OK;
}

extern "C" int cp_point_gather3d(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int n, int D,
                                 int H, int W, int layout, const int32_t *randt, const int32_t *randx,
                                 const int32_t *randy, int P, float *Y_out, int64_t ldy, cp_stream_t stream_) {
    CP_REQUIRE(cp_fmap_esize(fmap_dtype), "cp_point_gather3d: feature-map dtype %d is not CP_F32, CP_BF16 or CP_F16",
               fmap_dtype);
    CP_REQUIRE(h && fmap && randt && randx && randy && Y_out, "cp_point_gather3d: NULL argument");
    CP_REQUIRE(nbatch >= 0 && B > 0 && P > 0, "cp_point_gather3d: bad shape");
    CP_REQUIRE(n > 0 && D > 0 && H > 0 && W > 0, "cp_point_gather3d: empty output map (%d x %d x %d x %d)", n, D, H, W);
    CP_REQUIRE(ldy >= n, "cp_point_gather3d: ldy < n");
    CP_REQUIRE(layout == CP_LAYOUT_NCHW || layout == CP_LAYOUT_NHWC, "cp_point_gather3d: unknown layout %d", layout);
    const int64_t rows = (int64_t)nbatch * P * B;
    if (rows == 0) return CP_OK;
    CP_REQUIRE(rows < (1ll << 31), "cp_point_gather3d: too many rows");
    const cudaStream_t stream = (cudaStream_t)stream_;
    const int ndhwc = layout == CP_LAYOUT_NHWC;
    if (fmap_dtype == CP_F32)
        point_gather3d<<<(unsigned)rows, 256, 0, stream>>>((const float *)fmap, randt, randx, randy, Y_out, ldy, B, n,
                                                           D, H, W, P, ndhwc);
    else if (fmap_dtype == CP_BF16)
        point_gather3d<<<(unsigned)rows, 256, 0, stream>>>((const __nv_bfloat16 *)fmap, randt, randx, randy, Y_out, ldy,
                                                           B, n, D, H, W, P, ndhwc);
    else
        point_gather3d<<<(unsigned)rows, 256, 0, stream>>>((const __half *)fmap, randt, randx, randy, Y_out, ldy, B, n,
                                                           D, H, W, P, ndhwc);
    CP_CHECK_LAUNCH();
    return CP_OK;
}
