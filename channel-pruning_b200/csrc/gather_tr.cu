// Patch gathers of transposed convolutions (nn.ConvTranspose2d / ConvTranspose3d, groups == 1): the up-convolutions of
// U-Net and 3-D U-Net decoders, FCN heads and DCGAN-style generators.  fmap is the transposed convolution's INPUT map,
// the sampled points lie in its OUTPUT map.
//
// Per axis, tap i of output coordinate x reads input coordinate h = (x + pad - dil*i) / stride when the division is
// exact and 0 <= h < n; otherwise the entry is zero.  With g = gcd(stride, dil) the valid taps are i = i0 (mod
// stride/g), consecutive ones dil/g input rows apart, and none at all when x + pad is not a multiple of g: each row
// therefore touches at most ceil(k / (stride/g)) input coordinates per axis (one for the k = stride up-convolutions).
// The columns are in the conv gathers' order a*kt*kh*kw + (u*kh + i)*kw + j, so X @ weight.transpose(0, 1)
// .reshape(n, -1).T is the transposed convolution's output (minus its bias) at the sampled points.
//
// Each row's valid taps are found from its phase (tr_taps: first valid tap, count, step), never by testing every tap.
// Paths, one body each, compiled with (NCDHW / NDHWC) and without (NCHW / NHWC, D = 1, randt NULL) the depth axis:
//   channels first   patch_gather_tr_nchw / _ncdhw: one CTA per output row builds the row's tap -> pixel table in
//       shared memory, then consecutive threads write consecutive columns, zero columns included (coalesced stores)
//   channels last    patch_gather_tr_nhwc / _ndhwc: a unit is (output row, channel tile); the c channels of each touched
//       pixel are read with coalesced (16-byte where aligned) loads, staged in shared memory and written transposed
//       to (c, taps) order
// A map in pinned host memory is read in place by the same kernel with a small persistent grid (PCIe-bound: more CTAs
// only block SMs that other layers need).  The values are widened exactly and the ReLU is applied with the expression
// of the conv gathers (gather.cu), so -0, inf and NaN come out as the conv gathers give them; the XFORM = true kernels
// apply cp_patch_gather_act's input transform to the valid taps instead, and leave the invalid ones +0.
#include "common.cuh"
#include "fmap_types.cuh"

namespace {

// Valid taps of one axis for output coordinate x: taps first, first + period, ... (count of them), reading input
// coordinates in0, in0 - step, ...  count = 0: no tap of this axis is valid (x + pad off the gcd grid, or out of range).
struct tr_axis {
    int first, count, period, in0, step;
};

__device__ __forceinline__ tr_axis tr_taps(int x, int pad, int s, int d, int k, int n) {
    tr_axis r{0, 0, 1, 0, 0};
    const int num = x + pad;  // >= 0: x >= 0, pad >= 0
    int g = s, b = d;
    while (b) {
        const int t = g % b;
        g = b, b = t;
    }
    if (num % g) return r;
    const int period = s / g;
    // the tap of the phase: d*i0 = num (mod s), 0 <= i0 < period (d/g is invertible modulo period)
    int i0 = 0;
    while ((num - d * i0) % s) ++i0;
    // input coordinate < n:  num - d*i <= s*(n - 1)  <=>  i >= ceil((num - s*(n - 1)) / d)
    const int over = num - s * (n - 1);
    const int lo = over > 0 ? (over + d - 1) / d : 0;
    const int first = i0 + (lo > i0 ? (lo - i0 + period - 1) / period * period : 0);
    // input coordinate >= 0 (a negative numerator is never divided):  i <= num / d
    const int last = min(k - 1, num / d);
    if (first > last) return r;
    r.first = first, r.count = (last - first) / period + 1, r.period = period;
    r.in0 = (num - d * first) / s, r.step = d / g;
    return r;
}

// The valid taps of a row: per axis (t, h, w), and how many there are in all
struct tr_row {
    tr_axis t, h, w;
    int nv;
};

template <bool DEPTH>
__device__ __forceinline__ tr_row tr_row_taps(const cp_window &g, int tp, int xp, int yp, int D, int H, int W) {
    tr_row q;
    q.t = DEPTH ? tr_taps(tp, g.pad_t, g.stride_t, g.dil_t, g.kt, D) : tr_axis{0, 1, 1, 0, 0};
    q.h = tr_taps(xp, g.pad_h, g.stride_h, g.dil_h, g.kh, H);
    q.w = tr_taps(yp, g.pad_w, g.stride_w, g.dil_w, g.kw, W);
    q.nv = q.t.count * q.h.count * q.w.count;
    return q;
}

// Valid tap v (< q.nv) of a row: its column offset p within a channel's taps and its pixel in the D x H x W map
template <bool DEPTH>
__device__ __forceinline__ void tr_valid_tap(const tr_row &q, const cp_window &g, int v, int H, int W, int &p,
                                             int64_t &pix) {
    const int mw = v % q.w.count;
    const int mh = (v / q.w.count) % q.h.count;
    const int mt = DEPTH ? v / (q.w.count * q.h.count) : 0;
    const int u = q.t.first + mt * q.t.period, i = q.h.first + mh * q.h.period, j = q.w.first + mw * q.w.period;
    p = (u * g.kh + i) * g.kw + j;
    pix = cp_pixel<DEPTH>(q.t.in0 - mt * q.t.step, q.h.in0 - mh * q.h.step, q.w.in0 - mw * q.w.step, H, W);
}

// Channels first: grid-stride over the rows (grid = rows in HBM, a small persistent grid for a pinned host map).
// Shared: k pixel offsets, -1 for an invalid tap.
template <bool DEPTH, bool XFORM, typename T>
__device__ __forceinline__ void tr_cfirst_body(const T *__restrict__ fmap, const int32_t *__restrict__ randt,
                                               const int32_t *__restrict__ randx, const int32_t *__restrict__ randy,
                                               float *__restrict__ X, int64_t ldx, int64_t rows, int B, int c, int D,
                                               int H, int W, int P, const cp_window &g, int relu,
                                               const cp_xform &xf) {
    extern __shared__ int64_t tap_pix[];
    const int k = (DEPTH ? g.kt : 1) * g.kh * g.kw;
    const int K = c * k;
    const int64_t plane = (int64_t)(DEPTH ? D : 1) * H * W;
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        const int64_t bp = r / B;
        const int img = (int)(bp / P) * B + (int)(r % B);
        const tr_row q = tr_row_taps<DEPTH>(g, DEPTH ? randt[bp] : 0, randx[bp], randy[bp], D, H, W);
        for (int p = threadIdx.x; p < k; p += blockDim.x) tap_pix[p] = -1;
        __syncthreads();
        for (int v = threadIdx.x; v < q.nv; v += blockDim.x) {
            int p;
            int64_t pix;
            tr_valid_tap<DEPTH>(q, g, v, H, W, p, pix);
            tap_pix[p] = pix;
        }
        __syncthreads();
        const T *src = fmap + (int64_t)img * c * plane;
        float *dst = X + r * ldx;
#pragma unroll 4
        for (int col = threadIdx.x; col < K; col += blockDim.x) {
            const int a = col / k;
            const int64_t pix = tap_pix[col - a * k];
            float v = 0.f;
            if (pix >= 0) {
                v = cp_widen(__ldg(src + a * plane + pix));
                if (XFORM) v = cp_xform_apply(xf, v, a);
            }
            if (!XFORM && relu) v = fmaxf(v, 0.f);
            dst[col] = v;
        }
        __syncthreads();  // the table is rebuilt for the next row
    }
}

#define CP_TR_CFIRST_PARAMS                                                                                           \
    const T *__restrict__ fmap, const int32_t *__restrict__ randt, const int32_t *__restrict__ randx,                  \
        const int32_t *__restrict__ randy, float *__restrict__ X, int64_t ldx, int64_t rows, int B, int c, int D, int H, \
        int W, int P, cp_window g, int relu, cp_xform xf
template <typename T, bool XFORM = false>
__global__ void __launch_bounds__(256) patch_gather_tr_nchw(CP_TR_CFIRST_PARAMS) {
    tr_cfirst_body<false, XFORM>(fmap, nullptr, randx, randy, X, ldx, rows, B, c, 1, H, W, P, g, relu, xf);
}
template <typename T, bool XFORM = false>
__global__ void __launch_bounds__(256) patch_gather_tr_ncdhw(CP_TR_CFIRST_PARAMS) {
    tr_cfirst_body<true, XFORM>(fmap, randt, randx, randy, X, ldx, rows, B, c, D, H, W, P, g, relu, xf);
}

// Channels last: grid-stride over the units (output row, channel tile of ct_tile channels).  Shared: k slots (index of
// tap p among the row's valid taps, -1 when invalid), then the tile [nvmax][ct_tile + 1] of the valid taps' channels
// (widened, ReLU applied; ct_tile + 1: the transposed read is conflict-free).  VE > 1: 16-byte loads of VE elements
// (the launcher's rules: c and ct_tile multiples of VE, 16-byte aligned map).
template <bool DEPTH, int VE, bool XFORM, typename T>
__device__ __forceinline__ void tr_clast_body(const T *__restrict__ fmap, const int32_t *__restrict__ randt,
                                              const int32_t *__restrict__ randx, const int32_t *__restrict__ randy,
                                              float *__restrict__ X, int64_t ldx, int64_t units, int ntile, int B,
                                              int c, int D, int H, int W, int P, const cp_window &g, int ct_tile,
                                              int tile_off, int relu, const cp_xform &xf) {
    extern __shared__ __align__(16) unsigned char tr_smem[];
    int *slot = reinterpret_cast<int *>(tr_smem);
    float *tile = reinterpret_cast<float *>(tr_smem + tile_off);
    const int k = (DEPTH ? g.kt : 1) * g.kh * g.kw;
    const int ld = ct_tile + 1;
    for (int64_t u = blockIdx.x; u < units; u += gridDim.x) {
        const int64_t r = u / ntile;
        const int a0 = (int)(u - r * ntile) * ct_tile;
        const int ct = min(ct_tile, c - a0);
        const int64_t bp = r / B;
        const int img = (int)(bp / P) * B + (int)(r % B);
        const tr_row q = tr_row_taps<DEPTH>(g, DEPTH ? randt[bp] : 0, randx[bp], randy[bp], D, H, W);
        for (int p = threadIdx.x; p < k; p += blockDim.x) slot[p] = -1;
        __syncthreads();
        const T *src = fmap + (int64_t)img * (DEPTH ? D : 1) * H * W * c + a0;
        const int nvec = ct / VE;
        for (int e = threadIdx.x; e < q.nv * nvec; e += blockDim.x) {
            const int v = e / nvec, jv = e - v * nvec;
            int p;
            int64_t pix;
            tr_valid_tap<DEPTH>(q, g, v, H, W, p, pix);
            if (jv == 0) slot[p] = v;
            float *t = tile + v * ld + jv * VE;
            if (VE > 1) {
                union {
                    uint4 q4;
                    T e[VE];
                } w;
                w.q4 = __ldg(reinterpret_cast<const uint4 *>(src + pix * c) + jv);
#pragma unroll
                for (int m = 0; m < VE; ++m) {
                    float x = cp_widen(w.e[m]);
                    if (XFORM) x = cp_xform_apply(xf, x, a0 + jv * VE + m);
                    else if (relu) x = fmaxf(x, 0.f);
                    t[m] = x;
                }
            } else {
                float x = cp_widen(__ldg(src + pix * c + jv));
                if (XFORM) x = cp_xform_apply(xf, x, a0 + jv);
                else if (relu) x = fmaxf(x, 0.f);
                t[0] = x;
            }
        }
        __syncthreads();
        float *dst = X + r * ldx + (int64_t)a0 * k;
        for (int e = threadIdx.x; e < k * ct; e += blockDim.x) {
            const int a = e / k;
            const int s = slot[e - a * k];
            dst[e] = s >= 0 ? tile[s * ld + a] : 0.f;  // the ReLU of a zero tap is +0; the transform skips it
        }
        __syncthreads();  // slots and tile are rebuilt for the next unit
    }
}

#define CP_TR_CLAST_PARAMS                                                                                            \
    const T *__restrict__ fmap, const int32_t *__restrict__ randt, const int32_t *__restrict__ randx,                  \
        const int32_t *__restrict__ randy, float *__restrict__ X, int64_t ldx, int64_t units, int ntile, int B, int c,   \
        int D, int H, int W, int P, cp_window g, int ct_tile, int tile_off, int relu, cp_xform xf
template <int VE, typename T, bool XFORM = false>
__global__ void __launch_bounds__(256) patch_gather_tr_nhwc(CP_TR_CLAST_PARAMS) {
    tr_clast_body<false, VE, XFORM>(fmap, nullptr, randx, randy, X, ldx, units, ntile, B, c, 1, H, W, P, g, ct_tile,
                                    tile_off, relu, xf);
}
template <int VE, typename T, bool XFORM = false>
__global__ void __launch_bounds__(256) patch_gather_tr_ndhwc(CP_TR_CLAST_PARAMS) {
    tr_clast_body<true, VE, XFORM>(fmap, randt, randx, randy, X, ldx, units, ntile, B, c, D, H, W, P, g, ct_tile,
                                   tile_off, relu, xf);
}

// Grids of the in-place readers of pinned host maps: those of the conv gathers' channels-first and channels-last
// host readers (gather.cu, gather_host.cu)
constexpr int64_t TR_HOST_CFIRST_CTAS = 64;
constexpr int64_t TR_HOST_CLAST_CTAS = 32;
constexpr int TR_TILE_FLOATS = 12 * 1024;  // shared memory of the channels-last kernel: 48 KB, slots included

// Most valid taps a row of one axis can have: ceil(k / (stride / gcd(stride, dil)))
int tr_max_taps(int k, int s, int d) {
    int g = s, b = d;
    while (b) {
        const int t = g % b;
        g = b, b = t;
    }
    const int period = s / g;
    return (k + period - 1) / period;
}

template <typename T, bool XFORM>
void launch_tr(const cp_patch_args &a, bool host_src) {
    const cp_window &g = a.g;
    const T *fmap = (const T *)a.fmap;
    const int64_t rows = a.rows();
    const bool depth = a.randt != nullptr;
    const int k = g.kt * g.kh * g.kw;
    const int64_t grid_max = 0x7fffffff;
    if (a.layout == CP_LAYOUT_NCHW) {
        const int64_t grid = host_src ? std::min(rows, TR_HOST_CFIRST_CTAS) : rows;
        auto kern = depth ? patch_gather_tr_ncdhw<T, XFORM> : patch_gather_tr_nchw<T, XFORM>;
        kern<<<(unsigned)grid, 256, (size_t)k * sizeof(int64_t), a.stream>>>(
            fmap, a.randt, a.randx, a.randy, a.X, a.ldx, rows, a.B, a.c, a.D, a.H, a.W, a.P, g, a.relu, a.xf);
        return;
    }
    const int nvmax = tr_max_taps(g.kt, g.stride_t, g.dil_t) * tr_max_taps(g.kh, g.stride_h, g.dil_h) *
                      tr_max_taps(g.kw, g.stride_w, g.dil_w);
    const int tile_off = (k * (int)sizeof(int) + 15) / 16 * 16;
    // channels per tile: all c when the valid taps and the slots fit 48 KB (>= 1 channel for k <= 4096).  A unit of
    // few valid taps writes k2 columns per staged element, so a whole row per unit keeps a CTA from being mostly
    // set-up: on an H100 80GB HBM3 at 700 W, 128-channel tiles ran the k = s = 2, c = 1024 U-Net layer (fp32) in
    // 0.28 ms, whole rows in 0.08 ms
    int ct_tile = std::min(a.c, (TR_TILE_FLOATS - tile_off / 4) / nvmax - 1);
    constexpr int VE = 16 / sizeof(T);
    const bool vec = (a.c * sizeof(T)) % 16 == 0 && ((uintptr_t)a.fmap & 15) == 0 && ct_tile >= VE;
    if (vec) ct_tile -= ct_tile % VE;
    const int ntile = cp_cdiv(a.c, ct_tile);
    const int64_t units = rows * ntile;
    const int64_t grid = std::min(host_src ? TR_HOST_CLAST_CTAS : grid_max, units);
    const size_t smem = (size_t)tile_off + (size_t)nvmax * (ct_tile + 1) * sizeof(float);
    auto kern = vec ? (depth ? patch_gather_tr_ndhwc<VE, T, XFORM> : patch_gather_tr_nhwc<VE, T, XFORM>)
                    : (depth ? patch_gather_tr_ndhwc<1, T, XFORM> : patch_gather_tr_nhwc<1, T, XFORM>);
    kern<<<(unsigned)grid, 256, smem, a.stream>>>(fmap, a.randt, a.randx, a.randy, a.X, a.ldx, units, ntile, a.B, a.c,
                                                  a.D, a.H, a.W, a.P, g, ct_tile, tile_off, a.relu, a.xf);
}

}  // namespace

// gather.cu's entries call this once the arguments passed its checks (rows > 0); host_src: the map lies in pinned
// host memory
int cp_patch_gather_tr(const cp_patch_args &a, bool host_src) {
    cp_with_fmap_type(a.dtype, [&](auto z) {
        if (a.fused)
            launch_tr<decltype(z), true>(a, host_src);
        else
            launch_tr<decltype(z), false>(a, host_src);
    });
    CP_CHECK_LAUNCH();
    return CP_OK;
}
