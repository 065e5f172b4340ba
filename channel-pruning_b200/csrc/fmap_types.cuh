// Element types of the feature maps the gathers read (CP_F32, CP_BF16, CP_F16).  The gathered matrices X and Y are
// fp32 whatever the map holds: cp_widen converts exactly (every bf16 and fp16 value, fp16 subnormals included, is an
// fp32 value), so a 16-bit map gathers to the bits the fp32 map of the same values gives.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/cpb200.h"

__device__ __forceinline__ float cp_widen(float v) { return v; }
__device__ __forceinline__ float cp_widen(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float cp_widen(__half v) { return __half2float(v); }

// bytes per map element; 0 for a type the gathers do not read (CP_F64, unknown codes)
static inline int cp_fmap_esize(int fmap_dtype) {
    return fmap_dtype == CP_F32 ? 4 : (fmap_dtype == CP_BF16 || fmap_dtype == CP_F16) ? 2 : 0;
}

// f(T()) with T the element type of fmap_dtype: float, __nv_bfloat16 or __half (a code cp_fmap_esize accepts)
template <typename F>
static inline auto cp_with_fmap_type(int fmap_dtype, F &&f) {
    if (fmap_dtype == CP_BF16) return f(__nv_bfloat16());
    if (fmap_dtype == CP_F16) return f(__half());
    return f(float());
}

// Where a map lies: device memory, page-locked host memory mapped under UVA, or neither (pageable, managed, unknown)
enum cp_mem_kind { CP_MEM_DEVICE, CP_MEM_HOST, CP_MEM_OTHER };
static inline cp_mem_kind cp_pointer_kind(const void *p) {
    cudaPointerAttributes pa;
    cp_mem_kind kind = CP_MEM_OTHER;
    if (cudaPointerGetAttributes(&pa, p) == cudaSuccess)
        kind = pa.type == cudaMemoryTypeDevice ? CP_MEM_DEVICE : pa.type == cudaMemoryTypeHost ? CP_MEM_HOST : CP_MEM_OTHER;
    (void)cudaGetLastError();
    return kind;
}

// Window of a patch gather, with the semantics of PyTorch's Conv3d (groups == 1): output point (t, x, y) reads the taps
// (stride_t*t - pad_t + dil_t*u, stride_h*x - pad_h + dil_h*i, stride_w*y - pad_w + dil_w*j), u < kt, i < kh, j < kw,
// zero outside the map, into column a*kt*kh*kw + (u*kh + i)*kw + j (the order of Conv3d.weight.reshape(n, -1)).  Only
// the front / top / left padding enters: the other side's only sets the output size.  A Conv2d window is the one-frame
// case kt = 1, pad_t = 0, stride_t = dil_t = 1 on a map of depth D = 1 with t = 0 (column a*kh*kw + i*kw + j, the order
// of F.unfold); the reference's layers are its square, undilated case (kh = kw = k, one pad, one stride, dilation 1).
struct cp_window {
    int kt, kh, kw, pad_t, pad_h, pad_w, stride_t, stride_h, stride_w, dil_t, dil_h, dil_w;
};

// The input transform of a consumer (cp_patch_gather_act): an activation act (CP_ACT_*, slope: LeakyReLU's negative
// slope) after an optional per-channel affine (scale[a], shift[a]), the producer's eval-mode BatchNorm folded; either
// pointer may be NULL (scale 1, shift 0).
struct cp_xform {
    int act;
    float slope;
    const float *scale, *shift;
};

// The transform of an in-map tap on (global) channel a, v the widened value.  Each operation is rounded in fp32 (no
// FMA contraction); without an affine no arithmetic touches v, so -0 stays -0 under the identity.  Taps outside the
// map are never passed here: they are +0 whatever the transform (the consumer's zero padding pads its
// post-activation input).  SiLU is v / (1 + expf(-v)) with the accurate expf; below -64, where expf(-v) heads for
// overflow, the same value as (v e) e with e = expf(v / 2), which keeps the result within 4 ulp down to the
// subnormals.
__device__ __forceinline__ float cp_xform_apply(const cp_xform &f, float v, int a) {
    if (f.scale) v = __fmul_rn(v, __ldg(f.scale + a));
    if (f.shift) v = __fadd_rn(v, __ldg(f.shift + a));
    switch (f.act) {
        case CP_ACT_RELU: return fmaxf(v, 0.f);
        case CP_ACT_RELU6: return fminf(fmaxf(v, 0.f), 6.f);
        case CP_ACT_LEAKY_RELU: return v > 0.f ? v : __fmul_rn(v, f.slope);
        case CP_ACT_HARDSWISH: return __fdiv_rn(__fmul_rn(v, fminf(fmaxf(__fadd_rn(v, 3.f), 0.f), 6.f)), 6.f);
        case CP_ACT_SILU:
            if (v < -64.f) {
                const float e = expf(0.5f * v);
                return __fmul_rn(__fmul_rn(v, e), e);
            }
            return __fdiv_rn(v, __fadd_rn(1.f, expf(-v)));
        default: return v;  // CP_ACT_IDENTITY
    }
}

// One patch gather as an entry point hands it to a path (gather.cu, gather_host.cu, gather_tma.cu): nbatch*B images
// of c x D x H x W, channels first (CP_LAYOUT_NCHW) or last (CP_LAYOUT_NHWC); randt NULL for a 2-D map (D = 1, t = 0).
struct cp_patch_args {
    const char *name;  // the entry point, which the messages name
    const void *fmap;
    int dtype, layout, nbatch, B, c, D, H, W, P;
    const int32_t *randt, *randx, *randy;
    cp_window g;
    int relu;
    float *X;
    int64_t ldx;
    cudaStream_t stream;
    // cp_patch_gather_act: the input transform, applied by the paths' XFORM = true kernels (relu then unused)
    bool fused = false;
    cp_xform xf = {};
    int64_t rows() const { return (int64_t)nbatch * P * B; }
};

// Tap p of window g from the window origin (t0, y0, x0): its coordinates (tt, yy, xx) and whether they lie inside the
// D x H x W map.  DEPTH = false: a 2-D window (kt = 1, t0 = 0, tt = 0), the depth arithmetic compiled out.  KS > 0: a
// square, undilated KS x KS 2-D window known at compile time.
template <bool DEPTH, int KS = 0>
__device__ __forceinline__ bool cp_window_tap(const cp_window &g, int p, int t0, int y0, int x0, int D, int H, int W,
                                              int &tt, int &yy, int &xx) {
    static_assert(KS == 0 || !DEPTH, "compile-time windows are 2-D");
    const int kw = KS > 0 ? KS : g.kw, khw = KS > 0 ? KS * KS : g.kh * g.kw;
    const int dil_h = KS > 0 ? 1 : g.dil_h, dil_w = KS > 0 ? 1 : g.dil_w;
    int t = 0, q = p;
    if (DEPTH) {
        const int pu = p / khw;
        q = p - pu * khw;
        t = t0 + pu * g.dil_t;
    }
    const int py = q / kw, px = q - py * kw;
    const int y = y0 + py * dil_h, x = x0 + px * dil_w;
    tt = t, yy = y, xx = x;
    return (!DEPTH || (t >= 0 && t < D)) && y >= 0 && y < H && x >= 0 && x < W;
}

// Pixel (tt*H + yy)*W + xx of a D x H x W map (DEPTH = false: yy*W + xx)
template <bool DEPTH>
__device__ __forceinline__ int64_t cp_pixel(int tt, int yy, int xx, int H, int W) {
    return DEPTH ? ((int64_t)tt * H + yy) * W + xx : (int64_t)yy * W + xx;
}
