// Sparse-point gathers: the "im2col" of the pruning path.
//
//   cp_patch_gather  <- Net.extract_XY          (reference lib/net.py:534-684) + relu (:1720)
//   cp_point_gather  <- Net.extract_features    (reference lib/net.py:509-519)
//
// Both are pure data movement (HBM bound).  Row r of the output is
// (batch, point, image) = ((r / B) / P, (r / B) % P, r % B), the reference's order.
//
// One implementation serves 2-D (Conv2d) and 3-D (Conv3d) maps: a 2-D map is the one-frame 3-D map (D = 1, kt = 1,
// t = 0, cp_window), which its entries pass with randt = NULL; each path has one body, whose DEPTH = false
// instantiation compiles the depth arithmetic out, under one kernel name per rank.  Paths:
//   channels first (NCHW / NCDHW), HBM or pinned host   patch_gather_nchw / _ncdhw: one CTA per output row (a small
//       persistent grid for a host map); consecutive threads write consecutive columns, so stores are fully
//       coalesced; the loads are the sparse part (kw elements per (channel, tap row) segment), served through L1/L2
//       at sector granularity -- that over-fetch is inherent to reading kw-wide windows out of a channels-first map
//   channels last (NHWC / NDHWC), HBM, TMA rules hold   gather_tma.cu
//   channels last, pinned host                          gather_host.cu (contiguous window rows by 16-byte cp.async)
//   channels last, HBM, otherwise                       patch_gather_nhwc / _ndhwc: the CTA stages a taps x channels tile in
//       shared memory with coalesced loads (channel fastest) and writes it back transposed to (c, taps) column order,
//       again coalesced
// Element type of the map: fp32, bf16 or fp16 (template parameter T, fmap_types.cuh).  X and Y are fp32 in every
// case; the ReLU is applied to the widened value with the fp32 kernel's expression, so -0, inf and NaN come out as the
// fp32 kernel gives them for the widened map.
// cp_patch_gather_act runs each path's XFORM = true instantiation: the consumer's input transform (cp_xform_apply,
// fmap_types.cuh: a folded BatchNorm and an activation) on every in-map tap, +0 on the others.  The XFORM = false
// instantiations are the relu-flag kernels of the other entries, unchanged.
#include "common.cuh"
#include "fmap_types.cuh"

namespace {

// KS > 0: a square, undilated KS x KS 2-D window known at compile time (1 and 3); KS = 0: any window of g.
// XFORM: the input transform xf on in-map taps (cp_patch_gather_act); otherwise the relu flag.
template <int KS, bool DEPTH, bool XFORM, typename T>
__device__ __forceinline__ void cfirst_body(const T *__restrict__ fmap, const int32_t *__restrict__ randt,
                                            const int32_t *__restrict__ randx,
                                            const int32_t *__restrict__ randy, float *__restrict__ X, int64_t ldx,
                                            int64_t rows, int B, int c, int D, int H, int W, int P, const cp_window &g,
                                            int relu, const cp_xform &xf) {
    const int k = KS > 0 ? KS * KS : (DEPTH ? g.kt : 1) * g.kh * g.kw;  // taps
    const int K = c * k;
    // one CTA per output row when the map is in HBM; a small persistent grid strides over the rows when the
    // map is read in place from pinned host memory (PCIe-bound: more CTAs only block SMs other layers need)
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        const int img_in_batch = (int)(r % B);
        const int64_t bp = r / B;  // batch*P + point
        const int batch = (int)(bp / P);
        const int t0 = DEPTH ? g.stride_t * randt[bp] - g.pad_t : 0;
        const int y0 = g.stride_h * randx[bp] - g.pad_h;  // window origin, rows   (net.py: feat[:,:,x,y], x indexes H)
        const int x0 = g.stride_w * randy[bp] - g.pad_w;  // window origin, cols
        const T *src = fmap + ((int64_t)batch * B + img_in_batch) * c * (DEPTH ? D : 1) * H * W;
        float *dst = X + r * ldx;
#pragma unroll 4
        for (int col = threadIdx.x; col < K; col += blockDim.x) {
            const int a = col / k;
            int tt, yy, xx;
            float v = 0.f;
            if (cp_window_tap<DEPTH, KS>(g, col - a * k, t0, y0, x0, D, H, W, tt, yy, xx)) {
                v = cp_widen(__ldg(src + (DEPTH ? (((int64_t)a * D + tt) * H + yy) * W : ((int64_t)a * H + yy) * W) + xx));
                if (XFORM) v = cp_xform_apply(xf, v, a);
            }
            if (!XFORM && relu) v = fmaxf(v, 0.f);
            dst[col] = v;
        }
    }
}

// The kernels by name, one per rank (profiles and tests tell the paths apart by it): the 2-D entry passes D = 1 and
// no randt to the DEPTH = false body
#define CP_CFIRST_PARAMS                                                                                              \
    const T *__restrict__ fmap, const int32_t *__restrict__ randt, const int32_t *__restrict__ randx,                  \
        const int32_t *__restrict__ randy, float *__restrict__ X, int64_t ldx, int64_t rows, int B, int c, int D, int H, \
        int W, int P, cp_window g, int relu, cp_xform xf
template <int KS, typename T, bool XFORM = false>
__global__ void __launch_bounds__(256) patch_gather_nchw(CP_CFIRST_PARAMS) {
    cfirst_body<KS, false, XFORM>(fmap, nullptr, randx, randy, X, ldx, rows, B, c, 1, H, W, P, g, relu, xf);
}
template <typename T, bool XFORM = false>
__global__ void __launch_bounds__(256) patch_gather_ncdhw(CP_CFIRST_PARAMS) {
    cfirst_body<0, true, XFORM>(fmap, randt, randx, randy, X, ldx, rows, B, c, D, H, W, P, g, relu, xf);
}

constexpr int64_t CP_HOST_GATHER_CTAS = 64;  // grid of the in-place (zero-copy) channels-first reader
constexpr int CLAST_TILE_FLOATS = 12 * 1024;  // shared-memory tile of the channels-last SIMT kernels: 48 KB

// grid (rows, channel tiles); the tile is [taps][ct_tile + 1] floats, ct_tile channels (ct_tile + 1: the transposed
// read is conflict-free)
template <bool DEPTH, bool XFORM, typename T>
__device__ __forceinline__ void clast_body(const T *__restrict__ fmap, const int32_t *__restrict__ randt,
                                           const int32_t *__restrict__ randx, const int32_t *__restrict__ randy,
                                           float *__restrict__ X, int64_t ldx, int B, int c, int D, int H, int W, int P,
                                           const cp_window &g, int ct_tile, int relu, const cp_xform &xf) {
    extern __shared__ float tile[];
    const int k = (DEPTH ? g.kt : 1) * g.kh * g.kw;
    const int64_t r = blockIdx.x;
    const int a0 = blockIdx.y * ct_tile;
    const int ct = min(ct_tile, c - a0);
    const int img_in_batch = (int)(r % B);
    const int64_t bp = r / B;
    const int batch = (int)(bp / P);
    const int t0 = DEPTH ? g.stride_t * randt[bp] - g.pad_t : 0;
    const int y0 = g.stride_h * randx[bp] - g.pad_h;
    const int x0 = g.stride_w * randy[bp] - g.pad_w;
    const T *src = fmap + ((int64_t)batch * B + img_in_batch) * D * H * W * c;
    for (int e = threadIdx.x; e < k * ct; e += blockDim.x) {
        const int p = e / ct;
        const int a = e - p * ct;
        int tt, yy, xx;
        float v = 0.f;
        if (cp_window_tap<DEPTH>(g, p, t0, y0, x0, D, H, W, tt, yy, xx)) {
            v = cp_widen(__ldg(src + cp_pixel<DEPTH>(tt, yy, xx, H, W) * c + a0 + a));
            if (XFORM) v = cp_xform_apply(xf, v, a0 + a);
        }
        if (!XFORM && relu) v = fmaxf(v, 0.f);
        tile[p * (ct_tile + 1) + a] = v;
    }
    __syncthreads();
    float *dst = X + r * ldx + (int64_t)a0 * k;
    for (int e = threadIdx.x; e < k * ct; e += blockDim.x) {
        const int a = e / k;
        const int p = e - a * k;
        dst[e] = tile[p * (ct_tile + 1) + a];
    }
}

#define CP_CLAST_PARAMS                                                                                               \
    const T *__restrict__ fmap, const int32_t *__restrict__ randt, const int32_t *__restrict__ randx,                  \
        const int32_t *__restrict__ randy, float *__restrict__ X, int64_t ldx, int B, int c, int D, int H, int W, int P, \
        cp_window g, int ct_tile, int relu, cp_xform xf
template <typename T, bool XFORM = false>
__global__ void __launch_bounds__(256) patch_gather_nhwc(CP_CLAST_PARAMS) {
    clast_body<false, XFORM>(fmap, nullptr, randx, randy, X, ldx, B, c, 1, H, W, P, g, ct_tile, relu, xf);
}
template <typename T, bool XFORM = false>
__global__ void __launch_bounds__(256) patch_gather_ndhwc(CP_CLAST_PARAMS) {
    clast_body<true, XFORM>(fmap, randt, randx, randy, X, ldx, B, c, D, H, W, P, g, ct_tile, relu, xf);
}

// randt NULL: a 2-D map (t = 0)
template <typename T>
__global__ void __launch_bounds__(256)
point_gather(const T *__restrict__ fmap, const int32_t *__restrict__ randt, const int32_t *__restrict__ randx,
             const int32_t *__restrict__ randy, float *__restrict__ Y, int64_t ldy, int B, int n, int D, int H, int W,
             int P, int clast) {
    const int64_t r = blockIdx.x;
    const int img_in_batch = (int)(r % B);
    const int64_t bp = r / B;
    const int batch = (int)(bp / P);
    const int64_t pix = ((int64_t)(randt ? randt[bp] : 0) * H + randx[bp]) * W + randy[bp];
    const int64_t plane = (int64_t)D * H * W;
    const T *src = fmap + ((int64_t)batch * B + img_in_batch) * n * plane;
    float *dst = Y + r * ldy;
    if (clast) {
        const T *s = src + pix * n;
        for (int j = threadIdx.x; j < n; j += blockDim.x) dst[j] = cp_widen(__ldg(s + j));
    } else {
        const T *s = src + pix;
        for (int j = threadIdx.x; j < n; j += blockDim.x) dst[j] = cp_widen(__ldg(s + (int64_t)j * plane));
    }
}

}  // namespace

// gather_tma.cu: whether the TMA path takes a channels-last map in device memory, and the gather by it
bool cp_gather_tma_applies(const cp_patch_args &a);
int cp_patch_gather_tma(cp_handle_t h, const cp_patch_args &a);
// gather_host.cu: the in-place reader of channels-last maps in pinned host memory
int cp_patch_gather_host(const cp_patch_args &a);
// gather_tr.cu: the gathers of transposed convolutions, every layout, from HBM or (host_src) pinned host memory
int cp_patch_gather_tr(const cp_patch_args &a, bool host_src);

template <typename T, bool XFORM>
static void launch_patch_gather_simt(const cp_patch_args &a, bool host_src) {
    const cp_window &g = a.g;
    const T *fmap = (const T *)a.fmap;
    const int64_t rows = a.rows();
    const bool depth = a.randt != nullptr;
    if (a.layout == CP_LAYOUT_NCHW) {
        const int64_t ncta = host_src ? (rows < CP_HOST_GATHER_CTAS ? rows : CP_HOST_GATHER_CTAS) : rows;
        const bool square = !depth && g.kh == g.kw && g.dil_h == 1 && g.dil_w == 1;
        auto kern = depth                   ? patch_gather_ncdhw<T, XFORM>
                    : square && g.kh == 3 ? patch_gather_nchw<3, T, XFORM>
                    : square && g.kh == 1 ? patch_gather_nchw<1, T, XFORM>
                                          : patch_gather_nchw<0, T, XFORM>;
        kern<<<(unsigned)ncta, 256, 0, a.stream>>>(fmap, a.randt, a.randx, a.randy, a.X, a.ldx, rows, a.B, a.c, a.D,
                                                   a.H, a.W, a.P, g, a.relu, a.xf);
    } else {
        // channels per tile: up to 128, fewer for windows over 95 taps so the tile stays within 48 KB
        const int k = g.kt * g.kh * g.kw;
        const int ct_tile = CLAST_TILE_FLOATS / k - 1 > 128 ? 128 : CLAST_TILE_FLOATS / k - 1;
        const size_t smem = (size_t)k * (ct_tile + 1) * sizeof(float);
        dim3 grid((unsigned)rows, (unsigned)cp_cdiv(a.c, ct_tile));
        auto kern = depth ? patch_gather_ndhwc<T, XFORM> : patch_gather_nhwc<T, XFORM>;
        kern<<<grid, 256, smem, a.stream>>>(fmap, a.randt, a.randx, a.randy, a.X, a.ldx, a.B, a.c, a.D, a.H, a.W, a.P,
                                            g, ct_tile, a.relu, a.xf);
    }
}

// The bounds of an entry point (cpb200.h).  Every entry takes at most CP_GATHER_MAX_TAPS taps.
constexpr int CP_GATHER_MAX_TAPS = 4096;
struct cp_gather_limits {
    const char *name;
    bool d3;             // kt x kh x kw windows and randt; otherwise kh x kw windows on D = 1 maps, randt NULL
    int max_simt_taps;   // channels-last SIMT kernel in HBM; 0: no bound of its own
    int max_host_taps;   // channels-last reader of pinned host maps
    bool refuse_empty;   // refuse a window that leaves the output map empty
    bool transposed;     // a transposed convolution's window (gather_tr.cu): every tap is range-checked
};
// The 2-D entries keep the bounds of their square-window origins: the SIMT tile of 128 channels in 48 KB (95 taps)
// and the host reader's k <= 9.  Its channel chunks, and the adaptive SIMT tile, would fit larger windows.
static const cp_gather_limits CP_GATHER_2D = {"cp_patch_gather", false, 95, 81, false};
// The 3-D entry: the host reader up to 7 x 7 x 7 (a 3 x 7 x 7 stem is 147)
static const cp_gather_limits CP_GATHER_3D = {"cp_patch_gather_conv3d", true, 0, 343, true};
// The transposed entries: no bound of a path's own, and no empty output map (output_padding only sets its size)
static const cp_gather_limits CP_GATHER_TR_2D = {"cp_patch_gather_conv_transpose", false, 0, 0, false, true};
static const cp_gather_limits CP_GATHER_TR_3D = {"cp_patch_gather_conv_transpose3d", true, 0, 0, false, true};

// Per-axis values as the entry prints them: "h<sep>w" (2-D) or "t<sep>h<sep>w" (3-D)
static const char *cp_axes(char (&buf)[64], bool d3, const char *sep, int t, int h, int w) {
    if (d3)
        snprintf(buf, sizeof buf, "%d%s%d%s%d", t, sep, h, sep, w);
    else
        snprintf(buf, sizeof buf, "%d%s%d", h, sep, w);
    return buf;
}

// Argument checks of a patch gather, in the order every entry makes them; no CUDA call
static int cp_check_patch_gather(const cp_gather_limits &L, cp_handle_t h, const cp_patch_args &a) {
    const cp_window &g = a.g;
    const char *nm = L.name;
    char s[64];
    CP_REQUIRE(cp_fmap_esize(a.dtype), "%s: feature-map dtype %d is not CP_F32, CP_BF16 or CP_F16", nm, a.dtype);
    CP_REQUIRE(h && a.fmap && (a.randt || !L.d3) && a.randx && a.randy && a.X, "%s: NULL argument", nm);
    CP_REQUIRE(a.nbatch >= 0 && a.B > 0 && a.c > 0 && a.D > 0 && a.H > 0 && a.W > 0 && a.P > 0, "%s: bad shape", nm);
    CP_REQUIRE(g.kt >= 1 && g.kh >= 1 && g.kw >= 1, "%s: kernel_size %s: %s must be >= 1", nm,
               cp_axes(s, L.d3, "x", g.kt, g.kh, g.kw), L.d3 ? "every extent" : "both extents");
    CP_REQUIRE(g.stride_t >= 1 && g.stride_h >= 1 && g.stride_w >= 1, "%s: stride (%s) must be >= 1", nm,
               cp_axes(s, L.d3, ", ", g.stride_t, g.stride_h, g.stride_w));
    CP_REQUIRE(g.dil_t >= 1 && g.dil_h >= 1 && g.dil_w >= 1, "%s: dilation (%s) must be >= 1", nm,
               cp_axes(s, L.d3, ", ", g.dil_t, g.dil_h, g.dil_w));
    CP_REQUIRE(g.pad_t >= 0 && g.pad_h >= 0 && g.pad_w >= 0, "%s: padding (%s) must be >= 0", nm,
               cp_axes(s, L.d3, ", ", g.pad_t, g.pad_h, g.pad_w));
    CP_REQUIRE(g.kh <= CP_GATHER_MAX_TAPS / g.kw && g.kt <= CP_GATHER_MAX_TAPS / (g.kh * g.kw),
               "%s: kernel_size %s has more than %d taps", nm, cp_axes(s, L.d3, "x", g.kt, g.kh, g.kw),
               CP_GATHER_MAX_TAPS);
    // the output map of nn.Conv3d, (in + 2 pad - dil (k - 1) - 1) / stride + 1 per axis, must not be empty
    CP_REQUIRE(!L.refuse_empty || ((int64_t)a.D + 2ll * g.pad_t >= (int64_t)g.dil_t * (g.kt - 1) + 1 &&
                                   (int64_t)a.H + 2ll * g.pad_h >= (int64_t)g.dil_h * (g.kh - 1) + 1 &&
                                   (int64_t)a.W + 2ll * g.pad_w >= (int64_t)g.dil_w * (g.kw - 1) + 1),
               "%s: empty output map (the dilated window exceeds the padded %s map)", nm,
               cp_axes(s, L.d3, "x", a.D, a.H, a.W));
    CP_REQUIRE(a.ldx >= (int64_t)a.c * g.kt * g.kh * g.kw, "%s: ldx %lld < %s", nm, (long long)a.ldx,
               L.d3 ? "c*kt*kh*kw" : "c*kh*kw");
    CP_REQUIRE(a.layout == CP_LAYOUT_NCHW || a.layout == CP_LAYOUT_NHWC, "%s: unknown layout %d", nm, a.layout);
    return CP_OK;
}

// Checks, picks the path and launches
static int cp_patch_gather_any(const cp_gather_limits &L, cp_handle_t h, const cp_patch_args &a) {
    if (int rc = cp_check_patch_gather(L, h, a)) return rc;
    const int64_t rows = a.rows();
    if (rows == 0) return CP_OK;
    CP_REQUIRE(rows < (1ll << 31), "%s: too many rows", L.name);
    const cp_window &g = a.g;
    const int taps = g.kt * g.kh * g.kw;
    char s[64];
    // map in (pinned, UVA-mapped) host memory?  then the kernel is a PCIe reader: keep its footprint small
    const cp_mem_kind kind = cp_pointer_kind(a.fmap);
    if (L.transposed) return cp_patch_gather_tr(a, kind == CP_MEM_HOST);
    if (a.layout == CP_LAYOUT_NHWC) {
        // channels-last map in HBM: whole windows by TMA, rows out by bulk store (gather_tma.cu)
        if (kind == CP_MEM_DEVICE && cp_gather_tma_applies(a)) return cp_patch_gather_tma(h, a);
        // channels-last map in pinned host memory: whole window rows as 16-byte reads over PCIe (gather_host.cu)
        if (kind == CP_MEM_HOST) {
            CP_REQUIRE(taps <= L.max_host_taps, "%s: kernel_size %s too large for the %s host reader (%s <= %d)",
                       L.name, cp_axes(s, L.d3, "x", g.kt, g.kh, g.kw), L.d3 ? "NDHWC" : "NHWC",
                       L.d3 ? "kt*kh*kw" : "kh*kw", L.max_host_taps);
            return cp_patch_gather_host(a);
        }
        CP_REQUIRE(!L.max_simt_taps || taps <= L.max_simt_taps, "%s: kernel_size %s too large for the NHWC tile",
                   L.name, cp_axes(s, L.d3, "x", g.kt, g.kh, g.kw));
    }
    cp_with_fmap_type(a.dtype, [&](auto z) {
        if (a.fused)
            launch_patch_gather_simt<decltype(z), true>(a, kind == CP_MEM_HOST);
        else
            launch_patch_gather_simt<decltype(z), false>(a, kind == CP_MEM_HOST);
    });
    CP_CHECK_LAUNCH();
    return CP_OK;
}

extern "C" int cp_patch_gather_conv(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int c, int H,
                                    int W, int layout, const int32_t *randx, const int32_t *randy, int P, int kh,
                                    int kw, int pad_h, int pad_w, int stride_h, int stride_w, int dil_h, int dil_w,
                                    int relu, float *X_out, int64_t ldx, cp_stream_t stream) {
    const cp_window g{1, kh, kw, 0, pad_h, pad_w, 1, stride_h, stride_w, 1, dil_h, dil_w};
    return cp_patch_gather_any(CP_GATHER_2D, h,
                               {CP_GATHER_2D.name, fmap, fmap_dtype, layout, nbatch, B, c, 1, H, W, P, nullptr, randx,
                                randy, g, relu, X_out, ldx, (cudaStream_t)stream});
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

extern "C" int cp_patch_gather_conv3d(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int c,
                                      int D, int H, int W, int layout, const int32_t *randt, const int32_t *randx,
                                      const int32_t *randy, int P, int kt, int kh, int kw, int pad_t, int pad_h,
                                      int pad_w, int stride_t, int stride_h, int stride_w, int dil_t, int dil_h,
                                      int dil_w, int relu, float *X_out, int64_t ldx, cp_stream_t stream) {
    const cp_window g{kt, kh, kw, pad_t, pad_h, pad_w, stride_t, stride_h, stride_w, dil_t, dil_h, dil_w};
    return cp_patch_gather_any(CP_GATHER_3D, h,
                               {CP_GATHER_3D.name, fmap, fmap_dtype, layout, nbatch, B, c, D, H, W, P, randt, randx,
                                randy, g, relu, X_out, ldx, (cudaStream_t)stream});
}

extern "C" int cp_patch_gather_conv_transpose(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B,
                                              int c, int H, int W, int layout, const int32_t *randx,
                                              const int32_t *randy, int P, int kh, int kw, int pad_h, int pad_w,
                                              int stride_h, int stride_w, int dil_h, int dil_w, int relu,
                                              float *X_out, int64_t ldx, cp_stream_t stream) {
    const cp_window g{1, kh, kw, 0, pad_h, pad_w, 1, stride_h, stride_w, 1, dil_h, dil_w};
    return cp_patch_gather_any(CP_GATHER_TR_2D, h,
                               {CP_GATHER_TR_2D.name, fmap, fmap_dtype, layout, nbatch, B, c, 1, H, W, P, nullptr,
                                randx, randy, g, relu, X_out, ldx, (cudaStream_t)stream});
}

extern "C" int cp_patch_gather_conv_transpose3d(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B,
                                                int c, int D, int H, int W, int layout, const int32_t *randt,
                                                const int32_t *randx, const int32_t *randy, int P, int kt, int kh,
                                                int kw, int pad_t, int pad_h, int pad_w, int stride_t, int stride_h,
                                                int stride_w, int dil_t, int dil_h, int dil_w, int relu, float *X_out,
                                                int64_t ldx, cp_stream_t stream) {
    const cp_window g{kt, kh, kw, pad_t, pad_h, pad_w, stride_t, stride_h, stride_w, dil_t, dil_h, dil_w};
    return cp_patch_gather_any(CP_GATHER_TR_3D, h,
                               {CP_GATHER_TR_3D.name, fmap, fmap_dtype, layout, nbatch, B, c, D, H, W, P, randt, randx,
                                randy, g, relu, X_out, ldx, (cudaStream_t)stream});
}

extern "C" int cp_patch_gather_act(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int c, int D,
                                   int H, int W, int layout, const int32_t *randt, const int32_t *randx,
                                   const int32_t *randy, int P, int kt, int kh, int kw, int pad_t, int pad_h,
                                   int pad_w, int stride_t, int stride_h, int stride_w, int dil_t, int dil_h,
                                   int dil_w, int transposed, int act, float act_param, const float *in_scale,
                                   const float *in_shift, float *X_out, int64_t ldx, cp_stream_t stream) {
    const char *nm = "cp_patch_gather_act";
    const bool d3 = randt != nullptr;
    const cp_gather_limits &L0 = transposed ? (d3 ? CP_GATHER_TR_3D : CP_GATHER_TR_2D) : (d3 ? CP_GATHER_3D : CP_GATHER_2D);
    CP_REQUIRE(act >= CP_ACT_IDENTITY && act <= CP_ACT_SILU, "%s: unknown act %d", nm, act);
    CP_REQUIRE(isfinite(act_param), "%s: act_param must be finite", nm);
    CP_REQUIRE(d3 || (D == 1 && kt == 1 && pad_t == 0 && stride_t == 1 && dil_t == 1),
               "%s: a 2-D gather (randt NULL) takes D = 1, kt = 1, pad_t = 0, stride_t = dil_t = 1", nm);
    CP_REQUIRE(!in_scale || cp_pointer_kind(in_scale) == CP_MEM_DEVICE, "%s: in_scale is not in device memory", nm);
    CP_REQUIRE(!in_shift || cp_pointer_kind(in_shift) == CP_MEM_DEVICE, "%s: in_shift is not in device memory", nm);
    cp_gather_limits L = L0;
    L.name = nm;
    cp_patch_args a{nm, fmap, fmap_dtype, layout, nbatch, B, c, D, H, W, P, randt, randx, randy,
                    cp_window{kt, kh, kw, pad_t, pad_h, pad_w, stride_t, stride_h, stride_w, dil_t, dil_h, dil_w},
                    0, X_out, ldx, (cudaStream_t)stream};
    a.fused = true;
    a.xf = cp_xform{act, act_param, in_scale, in_shift};
    return cp_patch_gather_any(L, h, a);
}

// d3: the 3-D entry (randt required, D from the caller); otherwise D = 1 and randt NULL
static int cp_point_gather_any(const char *nm, bool d3, cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch,
                               int B, int n, int D, int H, int W, int layout, const int32_t *randt,
                               const int32_t *randx, const int32_t *randy, int P, float *Y_out, int64_t ldy,
                               cp_stream_t stream_) {
    CP_REQUIRE(cp_fmap_esize(fmap_dtype), "%s: feature-map dtype %d is not CP_F32, CP_BF16 or CP_F16", nm, fmap_dtype);
    CP_REQUIRE(h && fmap && (randt || !d3) && randx && randy && Y_out, "%s: NULL argument", nm);
    CP_REQUIRE(nbatch >= 0 && B > 0 && P > 0 && (d3 || (n > 0 && H > 0 && W > 0)), "%s: bad shape", nm);
    CP_REQUIRE(n > 0 && D > 0 && H > 0 && W > 0, "%s: empty output map (%d x %d x %d x %d)", nm, n, D, H, W);
    CP_REQUIRE(ldy >= n, "%s: ldy < n", nm);
    CP_REQUIRE(layout == CP_LAYOUT_NCHW || layout == CP_LAYOUT_NHWC, "%s: unknown layout %d", nm, layout);
    const int64_t rows = (int64_t)nbatch * P * B;
    if (rows == 0) return CP_OK;
    CP_REQUIRE(rows < (1ll << 31), "%s: too many rows", nm);
    const cudaStream_t stream = (cudaStream_t)stream_;
    const int clast = layout == CP_LAYOUT_NHWC;
    cp_with_fmap_type(fmap_dtype, [&](auto z) {
        using T = decltype(z);
        point_gather<<<(unsigned)rows, 256, 0, stream>>>((const T *)fmap, randt, randx, randy, Y_out, ldy, B, n, D, H,
                                                         W, P, clast);
    });
    CP_CHECK_LAUNCH();
    return CP_OK;
}

extern "C" int cp_point_gather_typed(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int n, int H,
                                     int W, int layout, const int32_t *randx, const int32_t *randy, int P,
                                     float *Y_out, int64_t ldy, cp_stream_t stream_) {
    return cp_point_gather_any("cp_point_gather", false, h, fmap, fmap_dtype, nbatch, B, n, 1, H, W, layout, nullptr,
                               randx, randy, P, Y_out, ldy, stream_);
}

extern "C" int cp_point_gather(cp_handle_t h, const float *fmap, int nbatch, int B, int n, int H, int W,
                               int layout, const int32_t *randx, const int32_t *randy, int P, float *Y_out,
                               int64_t ldy, cp_stream_t stream_) {
    return cp_point_gather_typed(h, fmap, CP_F32, nbatch, B, n, H, W, layout, randx, randy, P, Y_out, ldy, stream_);
}

extern "C" int cp_point_gather3d(cp_handle_t h, const void *fmap, int fmap_dtype, int nbatch, int B, int n, int D,
                                 int H, int W, int layout, const int32_t *randt, const int32_t *randx,
                                 const int32_t *randy, int P, float *Y_out, int64_t ldy, cp_stream_t stream_) {
    return cp_point_gather_any("cp_point_gather3d", true, h, fmap, fmap_dtype, nbatch, B, n, D, H, W, layout, randt,
                               randx, randy, P, Y_out, ldy, stream_);
}
