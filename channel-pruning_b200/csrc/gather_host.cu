// In-place reader of channels-last (NHWC / NDHWC) feature maps in pinned host memory: the patch gather of the
// host-resident input path for maps a channels_last forward hands over (layout CP_LAYOUT_NHWC, map in page-locked host
// memory mapped under UVA).
//
// Over PCIe a gather costs read requests, not bytes.  In NHWC the in-bounds taps of an undilated window row are one
// contiguous run of (taps x c) elements (a dilated row: kw runs of c elements), so the reader fetches each run as
// 16-byte vectors, consecutive threads on consecutive addresses: every 128-byte line of the run is requested once and
// nearly all of its bytes are used (NCHW: c*kh runs of kw elements per window).
// A work unit is one (output row, channel chunk).  Its kh*kw x ct sub-window (cp_window) is copied by cp.async into a
// shared-memory stage; while one unit is widened, transposed to the (c, kh*kw) column order and stored, the copies of
// the next NS - 1 units of the CTA are in flight.  Chunks keep a stage within NHWC_HOST_SMEM / NS bytes whatever c and
// kh*kw <= 81 (a c = 2048, 3 x 3 fp32 window is 72 KB).  A small persistent grid strides over the units: the zero-copy gathers run beside other
// layers' searches and Grams, which need the SMs.
// Maps whose channel stride or base address is not a multiple of 16 bytes (c = 3, 5, 12 in fp32; odd c in 16 bit)
// take plain element loads into the same stages: correct for every c, not tuned.
// The output is bit for bit that of the HBM NHWC kernels: zero outside the map, cp_widen, then fmaxf for the ReLU
// (XFORM = true: the input transform of cp_patch_gather_act instead).
// NDHWC maps (Conv3d windows, DEPTH = true) take kt*kh*kw taps per unit: each (u, i) row of an undilated window is
// again one contiguous run of kw*c elements.
#include "common.cuh"
#include "fmap_types.cuh"

namespace {

constexpr int NHWC_HOST_SMEM = 48 * 1024;  // shared memory of a CTA (all stages)
constexpr int NHWC_HOST_PAD = 16;          // bytes after each tap of a stage: keeps 16-byte alignment, spreads banks

struct HostGeom {
    const int32_t *randt;  // NULL: a 2-D map (D = 1, t = 0)
    int B, P, c, D, H, W;
    cp_window w;
    int ct;       // channels per chunk (the last chunk may be shorter)
    int nchunk;   // chunks per window
    int tap;      // bytes per tap in a stage: ct * esize + NHWC_HOST_PAD
    int stage;    // bytes per stage
    int vec;      // 16-byte copies (c * esize % 16 == 0, 16-byte aligned map)
};

__device__ __forceinline__ void nh_cp_async16(void *smem, const void *gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)),
                 "l"(gmem) : "memory");
}

// Starts the copy of unit u into `stage`: 16-byte cp.async requests, or (vec == 0) plain element loads.
template <bool DEPTH, typename T>
__device__ __forceinline__ void host_fetch(const T *__restrict__ fmap, const int32_t *__restrict__ randx,
                                           const int32_t *__restrict__ randy, const HostGeom &g, int64_t u,
                                           unsigned char *stage) {
    const int64_t r = u / g.nchunk;
    const int a0 = (int)(u - r * g.nchunk) * g.ct;
    const int ct = min(g.ct, g.c - a0);
    const int k = (DEPTH ? g.w.kt : 1) * g.w.kh * g.w.kw;
    const int64_t bp = r / g.B;
    const int img = (int)(bp / g.P) * g.B + (int)(r % g.B);
    const int t0 = DEPTH ? g.w.stride_t * g.randt[bp] - g.w.pad_t : 0;
    const int y0 = g.w.stride_h * randx[bp] - g.w.pad_h;
    const int x0 = g.w.stride_w * randy[bp] - g.w.pad_w;
    const T *src = fmap + (int64_t)img * (DEPTH ? g.D : 1) * g.H * g.W * g.c + a0;
    int tt, yy, xx;
    if (g.vec) {
        constexpr int VE = 16 / sizeof(T);  // elements per copy
        const int nv = ct / VE;
        for (int e = threadIdx.x; e < k * nv; e += blockDim.x) {
            const int p = e / nv, j = e - p * nv;
            if (cp_window_tap<DEPTH>(g.w, p, t0, y0, x0, g.D, g.H, g.W, tt, yy, xx))
                nh_cp_async16(stage + p * g.tap + j * 16, src + cp_pixel<DEPTH>(tt, yy, xx, g.H, g.W) * g.c + j * VE);
        }
    } else {
        for (int e = threadIdx.x; e < k * ct; e += blockDim.x) {
            const int p = e / ct, a = e - p * ct;
            if (cp_window_tap<DEPTH>(g.w, p, t0, y0, x0, g.D, g.H, g.W, tt, yy, xx))
                reinterpret_cast<T *>(stage + p * g.tap)[a] = __ldg(src + cp_pixel<DEPTH>(tt, yy, xx, g.H, g.W) * g.c + a);
        }
    }
}

// Writes unit u from its stage: column a*taps + p of the chunk, zero for taps outside the map.  XFORM: the input
// transform xf on in-map taps; otherwise the relu flag.
template <bool DEPTH, bool XFORM, typename T>
__device__ __forceinline__ void host_store(const int32_t *__restrict__ randx, const int32_t *__restrict__ randy,
                                           float *__restrict__ X, int64_t ldx, const HostGeom &g, int64_t u,
                                           const unsigned char *stage, int relu, const cp_xform &xf) {
    const int64_t r = u / g.nchunk;
    const int a0 = (int)(u - r * g.nchunk) * g.ct;
    const int ct = min(g.ct, g.c - a0);
    const int k = (DEPTH ? g.w.kt : 1) * g.w.kh * g.w.kw;
    const int64_t bp = r / g.B;
    const int t0 = DEPTH ? g.w.stride_t * g.randt[bp] - g.w.pad_t : 0;
    const int y0 = g.w.stride_h * randx[bp] - g.w.pad_h;
    const int x0 = g.w.stride_w * randy[bp] - g.w.pad_w;
    float *dst = X + r * ldx + (int64_t)a0 * k;
    int tt, yy, xx;
    for (int e = threadIdx.x; e < k * ct; e += blockDim.x) {
        const int a = e / k, p = e - a * k;
        float v = 0.f;
        if (cp_window_tap<DEPTH>(g.w, p, t0, y0, x0, g.D, g.H, g.W, tt, yy, xx)) {
            v = cp_widen(reinterpret_cast<const T *>(stage + p * g.tap)[a]);
            if (XFORM) v = cp_xform_apply(xf, v, a0 + a);
        }
        if (!XFORM && relu) v = fmaxf(v, 0.f);
        dst[e] = v;
    }
}

// NS stages: unit u + i * gridDim.x is copied into stage (it + i) % NS while unit u is stored.
template <int NS, bool DEPTH, bool XFORM, typename T>
__device__ __forceinline__ void host_reader_body(const T *__restrict__ fmap, const int32_t *__restrict__ randx,
                                                 const int32_t *__restrict__ randy, float *__restrict__ X, int64_t ldx,
                                                 int64_t units, const HostGeom &g, int relu, const cp_xform &xf) {
    extern __shared__ __align__(16) unsigned char nh_smem[];
    const int64_t step = gridDim.x;
#pragma unroll
    for (int i = 0; i < NS - 1; ++i) {
        const int64_t ui = blockIdx.x + i * step;
        if (ui < units) host_fetch<DEPTH>(fmap, randx, randy, g, ui, nh_smem + i * g.stage);
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    int it = 0;
    for (int64_t u = blockIdx.x; u < units; u += step, ++it) {
        const int64_t un = u + (NS - 1) * step;
        if (un < units) host_fetch<DEPTH>(fmap, randx, randy, g, un, nh_smem + ((it + NS - 1) % NS) * g.stage);
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group %0;" ::"n"(NS - 1) : "memory");  // unit u's copies have landed
        __syncthreads();
        host_store<DEPTH, XFORM, T>(randx, randy, X, ldx, g, u, nh_smem + (it % NS) * g.stage, relu, xf);
        __syncthreads();  // the stage is refilled NS - 1 units later
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// The reader by name, one per rank (profiles and tests tell the paths apart by it, and the element type by the last
// template argument)
template <int NS, bool XFORM, typename T>
__global__ void __launch_bounds__(256)
patch_gather_nhwc_host(const T *__restrict__ fmap, const int32_t *__restrict__ randx,
                       const int32_t *__restrict__ randy, float *__restrict__ X, int64_t ldx, int64_t units,
                       HostGeom g, int relu, cp_xform xf) {
    host_reader_body<NS, false, XFORM>(fmap, randx, randy, X, ldx, units, g, relu, xf);
}
template <int NS, bool XFORM, typename T>
__global__ void __launch_bounds__(256)
patch_gather_ndhwc_host(const T *__restrict__ fmap, const int32_t *__restrict__ randx,
                        const int32_t *__restrict__ randy, float *__restrict__ X, int64_t ldx, int64_t units,
                        HostGeom g, int relu, cp_xform xf) {
    host_reader_body<NS, true, XFORM>(fmap, randx, randy, X, ldx, units, g, relu, xf);
}

}  // namespace

// Geometry, channel chunk and stage sizes of the reader for NS = ns stages.  Returns false when one copy per tap does
// not fit a stage (never for the kh*kw <= 81 that cp_patch_gather_conv, or the kt*kh*kw <= 343 that
// cp_patch_gather_conv3d, lets through).
static bool host_geom(HostGeom &g, const void *fmap, int esize, int B, int P, int c, int D, int H, int W,
                      const int32_t *randt, const cp_window &w, int ns) {
    g.randt = randt, g.B = B, g.P = P, g.c = c, g.D = D, g.H = H, g.W = W, g.w = w;
    const int k = w.kt * w.kh * w.kw;
    g.vec = (c * esize) % 16 == 0 && ((uintptr_t)fmap & 15) == 0;
    const int ve = g.vec ? 16 / esize : 1;
    int ctmax = (NHWC_HOST_SMEM / ns / k - NHWC_HOST_PAD) / esize;
    ctmax -= ctmax % ve;
    if (ctmax < ve) return false;
    g.nchunk = cp_cdiv(c, ctmax);
    g.ct = cp_cdiv(cp_cdiv(c, g.nchunk), ve) * ve;  // balanced chunks, whole 16-byte copies
    g.nchunk = cp_cdiv(c, g.ct);
    g.tap = g.ct * esize + NHWC_HOST_PAD;
    g.stage = k * g.tap;
    return true;
}

template <int NS, bool XFORM, typename T>
static void launch_host(const T *fmap, const HostGeom &g, int64_t rows, const int32_t *randx, const int32_t *randy,
                        int relu, const cp_xform &xf, float *X_out, int64_t ldx, int ncta, cudaStream_t stream) {
    const int64_t units = rows * g.nchunk;
    const unsigned grid = (unsigned)(units < ncta ? units : ncta);
    auto kern = g.randt ? patch_gather_ndhwc_host<NS, XFORM, T> : patch_gather_nhwc_host<NS, XFORM, T>;
    kern<<<grid, 256, (size_t)NS * g.stage, stream>>>(fmap, randx, randy, X_out, ldx, units, g, relu, xf);
}

// Grid and pipeline depth of the reader (profiles/host_nhwc_ctas.cu; H100 80GB HBM3 SXM, 700 W; DESIGN.md section 3).
// The link bounds it: conv3_2 / conv4_2 at N = 5000 read 23-27 GB/s of window bytes with 16 to 132 CTAs.  With two
// stages 32 CTAs are within the spread of 64 and 132 in fp32 and bf16 and leave the other SMs to the layers that
// search and factor meanwhile; with one stage (no copy in flight while a unit is stored) 16 CTAs lose 30 % in bf16.
constexpr int CP_HOST_NHWC_GATHER_CTAS = 32;
constexpr int CP_HOST_NHWC_STAGES = 2;

int cp_patch_gather_host(const cp_patch_args &a) {
    HostGeom g;
    CP_REQUIRE(host_geom(g, a.fmap, cp_fmap_esize(a.dtype), a.B, a.P, a.c, a.D, a.H, a.W, a.randt, a.g,
                         CP_HOST_NHWC_STAGES),
               "%s: kernel_size %dx%dx%d too large for the channels-last host reader", a.name, a.g.kt, a.g.kh, a.g.kw);
    cp_with_fmap_type(a.dtype, [&](auto z) {
        using T = decltype(z);
        auto launch = a.fused ? launch_host<CP_HOST_NHWC_STAGES, true, T> : launch_host<CP_HOST_NHWC_STAGES, false, T>;
        launch((const T *)a.fmap, g, a.rows(), a.randx, a.randy, a.relu, a.xf, a.X, a.ldx, CP_HOST_NHWC_GATHER_CTAS,
               a.stream);
    });
    CP_CHECK_LAUNCH();
    return CP_OK;
}
