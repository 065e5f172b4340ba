// Element types of the feature maps the gathers read (CP_F32, CP_BF16, CP_F16).  The gathered matrices X and Y are
// fp32 whatever the map holds: cp_widen converts exactly (every bf16 and fp16 value, fp16 subnormals included, is an
// fp32 value), so a 16-bit map gathers to the bits the fp32 map of the same values gives.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "../../include/cpb200.h"

__device__ __forceinline__ float cp_widen(float v) { return v; }
__device__ __forceinline__ float cp_widen(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float cp_widen(__half v) { return __half2float(v); }

// bytes per map element; 0 for a type the gathers do not read (CP_F64, unknown codes)
static inline int cp_fmap_esize(int fmap_dtype) {
    return fmap_dtype == CP_F32 ? 4 : (fmap_dtype == CP_BF16 || fmap_dtype == CP_F16) ? 2 : 0;
}

// Window of a patch gather, with the semantics of PyTorch's Conv2d: output point (x, y) reads the taps
// (stride_h*x - pad_h + dil_h*i, stride_w*y - pad_w + dil_w*j), i < kh, j < kw, zero outside the map, into column
// a*kh*kw + i*kw + j.  Only the top / left padding enters: the bottom / right padding only sets the output size.
// The reference's layers are the square, undilated case (kh = kw = k, one pad, one stride, dilation 1).
struct cp_window {
    int kh, kw, pad_h, pad_w, stride_h, stride_w, dil_h, dil_w;
};

// Window of a 3-D patch gather (torch.nn.Conv3d, groups == 1): output point (t, x, y) reads the taps
// (stride_t*t - pad_t + dil_t*u, stride_h*x - pad_h + dil_h*i, stride_w*y - pad_w + dil_w*j), u < kt, i < kh, j < kw,
// zero outside the map, into column a*kt*kh*kw + (u*kh + i)*kw + j (the order of Conv3d.weight.reshape(n, -1)).
struct cp_window3 {
    int kt, kh, kw, pad_t, pad_h, pad_w, stride_t, stride_h, stride_w, dil_t, dil_h, dil_w;
};
