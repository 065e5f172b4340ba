// Sparse-point im2col on channels-last (NHWC / NDHWC) feature maps, TMA in / TMA out -- the HBM-roofline path of the
// patch gathers
// (replaces Net.extract_XY, reference lib/net.py:534-684, + the relu of lib/net.py:1720).
//
// One sampled output point needs a kh x kw x c window of the bottom blob (cp_window).  In NHWC that window is kh runs
// of kw*c contiguous floats (6 KB at c = 512, 3 x 3): a 4-D tensor map over (c, W, H, image) with box
// (c_box, (kw-1)*dil_w+1, (kh-1)*dil_h+1, 1) and traversal strides (1, dil_w, dil_h, 1) lets ONE cp.async.bulk.tensor
// request fetch it -- the copy engine delivers ceil(box / stride) = kw x kh taps per channel, so a dilated window lands
// as densely as an undilated one -- zero-filling the taps that fall into the padding (out-of-range coordinates,
// net.py:631-632), and the finished patch row (K = c kh kw contiguous floats of X) leaves through a bulk
// shared->global copy.  Persistent CTAs (as many per SM as shared memory allows: the latency of one row -- TMA flight, two CTA-wide
// hand-offs, the transposition -- is hidden by the other CTAs of the SM) each keep a ring of windows in flight:
//     producer warp     the 32 lanes prefetch the sampled coordinates of the next 32 rows (one global-load latency per
//                       32 rows instead of per row); one lane arms the mbarrier and issues the TMA loads (ring of NS stages)
//     128 consumers     [tap][channel] -> [channel][tap] (the reference's column order a*kh*kw + p) with the ReLU folded
//                       in, conflict-free both ways when kh*kw is odd (lanes walk channels, the tap stride is kh*kw)
//     one consumer      bulk store of the row, two rows in flight
// Bytes: the window is read once and the row written once -- 8 N K bytes, the algorithmic figure of SURVEY.md 8(d).
// Bound: HBM.
// bf16 / fp16 maps (template parameter T): the tensor map has the 16-bit data type, the window stage holds 16-bit
// elements (half the bytes), and the consumers widen exactly while transposing; the row stays fp32.  6 N K bytes.
// The 16-byte rules of TMA (global strides, box rows) then need c % 8 == 0.
// NDHWC maps (Conv3d windows) take the same kernel body (ND = 5) over a 5-D tensor map (c, W, H, D, image): box
// (c_box, (kw-1)*dil_w+1, (kh-1)*dil_h+1, (kt-1)*dil_t+1, 1), traversal strides (1, dil_w, dil_h, dil_t, 1),
// one cp.async.bulk.tensor.5d request per box delivering kt x kh x kw taps per channel.  A 3 x 3 x 3 window is three
// times a 3 x 3 one, so there a work unit is one channel box of a row rather than the whole row: the stage and the
// output segment (c_box kt kh kw contiguous floats of X) keep the size of the 2-D conv4_x rows.
#include <cuda.h>

#include "common.cuh"
#include "fmap_types.cuh"

namespace {

constexpr int GT_CONS = 128;             // consumer threads
constexpr int GT_THREADS = GT_CONS + 32; // + producer warp
constexpr int GT_OUT = 2;                // output rows in flight

struct GtParams {
    const int32_t *randx, *randy;
    float *X;
    int64_t ldx, rows;
    int B, P, c, k2, pad_h, pad_w, stride_h, stride_w, relu, cbox, nbox, nstage;
    int box_f, stage_f, out_f;  // strides in map elements (box, stage) and floats (out); 128-byte multiples each
    // 5-D maps only: a unit is one channel group of a row -- rows counts units (rows of X x ngrp), c the channels of a
    // unit (one box), and unit u writes columns [(u % ngrp) c k2, +c k2) of row u / ngrp
    const int32_t *randt;
    int stride_t, pad_t, ngrp;
};
// The parameters of the XFORM kernels: + the window and the map extents (which taps lie in the map), and the input
// transform
struct GtXParams : GtParams {
    cp_window g;
    int D, H, W;
    cp_xform xf;
};
template <bool XFORM>
using GtArgs = std::conditional_t<XFORM, GtXParams, GtParams>;

__device__ __forceinline__ uint32_t g_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void g_mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void g_mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void g_mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void g_mbar_wait(uint32_t bar, uint32_t parity) {  // bounded: a protocol bug traps
    uint32_t done = 0;
    for (uint32_t spin = 0; !done; ++spin) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(bar), "r"(parity)
            : "memory");
        if (spin > (1u << 26)) __trap();
    }
}
__device__ __forceinline__ void g_tma_load_4d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void g_tma_load_5d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1, int c2, int c3,
                                              int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
        : "memory");
}
__device__ __forceinline__ void g_bulk_store(void *gdst, uint32_t ssrc, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(ssrc), "r"(bytes) : "memory");
}
__device__ __forceinline__ void g_cons_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(GT_CONS) : "memory"); }

// ND: 4 (NHWC map, whole rows) or 5 (NDHWC map, units of one channel box).  XFORM: the input transform P.xf
// (cp_patch_gather_act).  The copy engine's zero fill is then not enough -- the transform of a zero is not zero once
// there is a shift -- so the producer hands each stage's window origin and channel offset to the consumers, which
// find the row's in-map taps (cp_window_tap; a bit mask for the first 32) and write +0 for the others.
template <typename T, int K2, int ND, bool XFORM>
__device__ __forceinline__ void gt_body(const CUtensorMap &map, const GtArgs<XFORM> &P) {
    extern __shared__ __align__(128) unsigned char gsm_raw[];
    const int k2 = K2 > 0 ? K2 : P.k2, K = P.c * k2;
    const uint32_t stage_bytes = (uint32_t)K * (uint32_t)sizeof(T), row_bytes = (uint32_t)K * 4u;
    // layout: [nstage][K] input windows ([box][tap][c_box], type T), [GT_OUT][K] fp32 output rows, mbarriers
    unsigned char *base = (unsigned char *)(((uintptr_t)gsm_raw + 127) & ~(uintptr_t)127);
    T *in = reinterpret_cast<T *>(base);
    float *out = reinterpret_cast<float *>(in + (size_t)P.nstage * P.stage_f);
    uint64_t *bars = reinterpret_cast<uint64_t *>(out + (size_t)GT_OUT * P.out_f);  // full[nstage], empty[nstage]
    // XFORM: (t0, y0, x0, channel offset) of the unit in each stage, within the 256 bytes gt_plan adds
    int *origin = reinterpret_cast<int *>(bars + 2 * P.nstage);
    const int tid = threadIdx.x;
    const uint32_t bar0 = g_smem_u32(bars);
    auto full = [&](int s) { return bar0 + 8u * (uint32_t)s; };
    auto empty = [&](int s) { return bar0 + 8u * (uint32_t)(P.nstage + s); };
    if (tid == 0) {
        for (int s = 0; s < P.nstage; ++s) {
            g_mbar_init(full(s), 1);
            g_mbar_init(empty(s), 1);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int64_t first = blockIdx.x, step = gridDim.x;
    if (tid >= GT_CONS) {
        // ---------------- producer warp
        const int lane = tid & 31;
        int it = 0;
        for (int64_t rb = first; rb < P.rows; rb += 32 * step) {
            // lane l looks up the window of row rb + l * step
            const int64_t u = rb + (int64_t)lane * step;
            int x0 = 0, y0 = 0, img = 0, t0 = 0, ch0 = 0;
            if (u < P.rows) {
                int64_t r = u;
                if constexpr (ND == 5) {
                    r = u / P.ngrp;
                    ch0 = (int)(u - r * P.ngrp) * P.c;
                }
                const int img_in_batch = (int)(r % P.B);
                const int64_t bp = r / P.B;  // batch * P + point
                const int batch = (int)(bp / P.P);
                y0 = P.stride_h * P.randx[bp] - P.pad_h;  // window origin, rows  (feat[:,:,x,y]: x indexes H)
                x0 = P.stride_w * P.randy[bp] - P.pad_w;
                if constexpr (ND == 5) t0 = P.stride_t * P.randt[bp] - P.pad_t;
                img = batch * P.B + img_in_batch;
            }
            const int64_t left = (P.rows - rb + step - 1) / step;
            const int nb = left < 32 ? (int)left : 32;
            for (int j = 0; j < nb; ++j, ++it) {
                const int xs = __shfl_sync(0xffffffffu, x0, j), ys = __shfl_sync(0xffffffffu, y0, j);
                const int is = __shfl_sync(0xffffffffu, img, j);
                int ts = 0, cs = 0;
                if constexpr (ND == 5) {
                    ts = __shfl_sync(0xffffffffu, t0, j);
                    cs = __shfl_sync(0xffffffffu, ch0, j);
                }
                if (lane == 0) {
                    const int s = it % P.nstage;
                    const uint32_t ph = (uint32_t)((it / P.nstage) & 1);
                    if (it >= P.nstage) g_mbar_wait(empty(s), ph ^ 1);  // the consumers have released the stage
                    if constexpr (XFORM) {  // published by the arrive below (release), read after the wait (acquire)
                        int *o = origin + 4 * s;
                        o[0] = ts, o[1] = ys, o[2] = xs, o[3] = cs;
                    }
                    g_mbar_expect_tx(full(s), stage_bytes);
                    const uint32_t dst = g_smem_u32(in + (size_t)s * P.stage_f);
                    for (int b = 0; b < P.nbox; ++b) {
                        const uint32_t db = dst + (uint32_t)b * (uint32_t)P.box_f * (uint32_t)sizeof(T);
                        if constexpr (ND == 5)
                            g_tma_load_5d(db, &map, full(s), cs + b * P.cbox, xs, ys, ts, is);
                        else
                            g_tma_load_4d(db, &map, full(s), b * P.cbox, xs, ys, is);
                    }
                }
                __syncwarp();
            }
        }
        return;
    }
    // ---------------- consumers
    int it = 0;
    for (int64_t r = first; r < P.rows; r += step, ++it) {
        const int s = it % P.nstage, o = it % GT_OUT;
        const uint32_t ph = (uint32_t)((it / P.nstage) & 1);
        g_mbar_wait(full(s), ph);
        if (tid == 0 && it >= GT_OUT) asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(GT_OUT - 1) : "memory");
        g_cons_barrier();  // out[o] is no longer being read by the store of row it - GT_OUT
        const T *src = in + (size_t)s * P.stage_f;
        float *dst = out + (size_t)o * P.out_f;
        int t0 = 0, y0 = 0, x0 = 0, cs = 0;
        uint32_t inmap = 0;  // bit p: tap p < 32 lies in the map
        if constexpr (XFORM) {
            const int *og = origin + 4 * s;
            t0 = og[0], y0 = og[1], x0 = og[2], cs = og[3];
            const int nb = k2 < 32 ? k2 : 32;
            for (int p = 0; p < nb; ++p) {
                int tt, yy, xx;
                inmap |= (uint32_t)cp_window_tap<ND == 5>(P.g, p, t0, y0, x0, P.D, P.H, P.W, tt, yy, xx) << p;
            }
        }
        // XFORM: the value of tap p of channel a (within the unit) as it is stored (Q: P, a GtXParams)
        auto xput = [&](const auto &Q, float v, int p, int a) {
            int tt, yy, xx;
            const bool in = p < 32 ? (inmap >> p) & 1u
                                   : cp_window_tap<ND == 5>(Q.g, p, t0, y0, x0, Q.D, Q.H, Q.W, tt, yy, xx);
            return in ? cp_xform_apply(Q.xf, v, cs + a) : 0.f;
        };
        for (int a = tid; a < P.c; a += GT_CONS) {
            const int b = a / P.cbox, al = a - b * P.cbox;
            const T *sp = src + (size_t)b * P.box_f + al;
            float *dp = dst + (size_t)a * k2;
            if constexpr (XFORM) {
                // one tap at a time: the transform's division and expf leave no registers for a batch of loads
                for (int p = 0; p < k2; ++p) dp[p] = xput(P, cp_widen(sp[(size_t)p * P.cbox]), p, a);
            } else if (K2 > 0) {
                // loads of a slab batched ahead of its stores; a 3 x 3 x 3 window goes by 3 x 3 slabs (registers)
                constexpr int KS = K2 > 9 && K2 % 9 == 0 ? 9 : (K2 > 0 ? K2 : 1);
#pragma unroll
                for (int p0 = 0; p0 < K2; p0 += KS) {
                    float v[KS];
#pragma unroll
                    for (int p = 0; p < KS; ++p) v[p] = cp_widen(sp[(p0 + p) * P.cbox]);
#pragma unroll
                    for (int p = 0; p < KS; ++p) dp[p0 + p] = P.relu ? fmaxf(v[p], 0.f) : v[p];
                }
            } else {
                for (int p = 0; p < k2; ++p) {
                    float v = cp_widen(sp[(size_t)p * P.cbox]);
                    if (P.relu) v = fmaxf(v, 0.f);
                    dp[p] = v;
                }
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the bulk store
        g_cons_barrier();
        if (tid == 0) {
            g_mbar_arrive(empty(s));  // every consumer has finished reading in[s]
            float *xr = P.X + r * P.ldx;
            if constexpr (ND == 5) {
                const int64_t row = r / P.ngrp;
                xr = P.X + row * P.ldx + (r - row * P.ngrp) * (int64_t)K;
            }
            g_bulk_store(xr, g_smem_u32(dst), row_bytes);
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
    }
    if (tid == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // shared memory must outlive the reads
}

// The kernel by name, one per rank of the tensor map (profiles and tests tell the paths apart by it); T: map element
// type; K2: taps known at compile time (gt_launch) or 0
template <typename T, int K2, bool XFORM = false>
__global__ void __launch_bounds__(GT_THREADS)
patch_gather_nhwc_tma(const __grid_constant__ CUtensorMap map, const GtArgs<XFORM> P) {
    gt_body<T, K2, 4, XFORM>(map, P);
}
template <typename T, int K2, bool XFORM = false>
__global__ void __launch_bounds__(GT_THREADS)
patch_gather_ndhwc_tma(const __grid_constant__ CUtensorMap map, const GtArgs<XFORM> P) {
    gt_body<T, K2, 5, XFORM>(map, P);
}

inline size_t gt_round128(size_t b) { return (b + 127) & ~(size_t)127; }

// Elements one tiled TMA request delivers to shared memory: ceil(boxDim[i] / elementStrides[i]) per dimension (the
// rule of the cuTensorMapEncodeTiled documentation)
inline size_t gt_box_elems(const cuuint32_t *box, const cuuint32_t *estr, int rank) {
    size_t n = 1;
    for (int i = 0; i < rank; ++i) n *= (box[i] + estr[i] - 1) / estr[i];
    return n;
}

typedef CUresult (*encode_fn_t)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

}  // namespace

template <bool XFORM>
using gt_kernel_t = void (*)(const CUtensorMap, const GtArgs<XFORM>);

template <int ND, typename T, int K2, bool XFORM>
static gt_kernel_t<XFORM> gt_kernel() {
    if constexpr (ND == 4)
        return patch_gather_nhwc_tma<T, K2, XFORM>;
    else
        return patch_gather_ndhwc_tma<T, K2, XFORM>;
}

template <bool XFORM>
static int gt_run(cp_handle_t h, gt_kernel_t<XFORM> kern, cp_per_device_flag &configured, const CUtensorMap &map,
                  const GtArgs<XFORM> &Pm, size_t smem, int per_sm, cudaStream_t stream) {
    if (bool *done = configured.slot(); !*done) {
        CP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
        *done = true;
    }
    int64_t grid = (int64_t)h->num_sms * per_sm;
    if (grid > Pm.rows) grid = Pm.rows;
    kern<<<(unsigned)grid, GT_THREADS, smem, stream>>>(map, Pm);
    CP_CHECK_LAUNCH();
    return CP_OK;
}

// One instantiation per (rank, element type, taps): 1 x 1 and 3 x 3 windows of either rank, 5 x 5 of 2-D maps and
// 3 x 3 x 3 of 3-D maps at compile time (a dilated window takes the instantiation of its tap count), the rest K2 = 0
template <int ND, typename T, bool XFORM>
static int gt_launch(cp_handle_t h, const CUtensorMap &map, const GtArgs<XFORM> &Pm, size_t smem, int per_sm,
                     cudaStream_t stream) {
    constexpr int KBIG = ND == 4 ? 25 : 27;
    const int k2 = Pm.k2;
    auto kern = k2 == 9 ? gt_kernel<ND, T, 9, XFORM>() : k2 == 1 ? gt_kernel<ND, T, 1, XFORM>()
              : k2 == KBIG ? gt_kernel<ND, T, KBIG, XFORM>() : gt_kernel<ND, T, 0, XFORM>();
    static cp_per_device_flag configured[4];  // one set per (rank, element type, XFORM): per instantiation of gt_launch
    const int which = k2 == 9 ? 0 : k2 == 1 ? 1 : k2 == KBIG ? 2 : 3;
    return gt_run<XFORM>(h, kern, configured[which], map, Pm, smem, per_sm, stream);
}

// CTAs per SM and input stages for a window stage of `row` bytes and output rows of `out_b` bytes: as many CTAs as fit
// with >= 2 input stages each (up to 4), then the stages fill what is left.
// conv4_x (c = 512, k = 3): fp32 stage 18 KB, row 18 KB -> 2 CTAs x 3 stages; 16-bit stage 9 KB, row 18 KB ->
// 3 CTAs x 3 stages (the fp32 output rows then take most of the budget)
static void gt_ring(size_t row, size_t out_b, int &per_sm, int &nstage) {
    const size_t budget = 216 * 1024;
    per_sm = (int)(budget / (2 * row + GT_OUT * out_b + 1024));
    per_sm = per_sm < 1 ? 1 : (per_sm > 4 ? 4 : per_sm);
    nstage = (int)((budget / per_sm - 1024 - GT_OUT * out_b) / row);
    if (nstage > 6) nstage = 6;
}

static int gt_encode_fn(cp_handle_t h) {
    if (!h->tmap_encode) {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        CP_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
        if (!fn || qres != cudaDriverEntryPointSuccess) CP_FAIL(CP_ERR_CUDA, "cuTensorMapEncodeTiled not available");
        h->tmap_encode = fn;
    }
    return CP_OK;
}

static CUtensorMapDataType gt_dtype(int fmap_dtype) {
    return fmap_dtype == CP_BF16  ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
           : fmap_dtype == CP_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                  : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
}

// Bytes of one work unit's output segment the 3-D path aims at: the fp32 row of the 2-D path at conv4_x (c = 512,
// 3 x 3), which that path moves at its best rate.  A 3 x 3 x 3 window at c >= 128 is split into 128-channel units.
constexpr size_t GT3_UNIT_BYTES = 18 * 1024;

// Channels per TMA box: the largest divisor d of c in [16, 256] with whole 16-byte box rows (TMA) whose fp32 output
// segment d * taps * 4 is at most seg_max bytes; the smallest such divisor when none is; 0 when c has none
static int gt_cbox(int c, int esize, int taps, size_t seg_max) {
    int last = 0;
    for (int d = 256; d >= 16; d -= 16 / esize) {
        if (c % d) continue;
        if ((size_t)d * taps * 4 <= seg_max) return d;
        last = d;
    }
    return last;
}

// Traversal strides of a tensor map are at most 8 and box extents at most 256 (cuTensorMapEncodeTiled)
constexpr int GT_MAX_DIL = 8, GT_MAX_SPAN = 256;

// How a channels-last map goes through the kernel.  2-D maps: a rank-4 tensor map, a work unit is a whole row of X
// (nbox = c / cbox boxes, gt_cbox's largest box).  3-D maps: a rank-5 tensor map, a work unit is one box of a row
// (ngrp = c / cbox units per row), the box sized by GT3_UNIT_BYTES.
struct GtPlan {
    int rank, taps, cbox, uc, nbox, ngrp;  // uc: channels per unit
    size_t box_b, row, out_b;             // bytes of a box and of a unit's window stage (type T) and output (fp32)
    int per_sm, nstage;
    size_t smem;
};

// false when the TMA path does not take the window: the 16-byte rules, an extent over 16, a dilation over 8, a span
// over 256, no channel box, or no room for two input stages in one CTA
static bool gt_plan(GtPlan &pl, int esize, int c, const cp_window &g, bool depth) {
    if (c % (16 / esize) || c < 16 || g.kt > 16 || g.kh > 16 || g.kw > 16) return false;
    if (g.dil_t > GT_MAX_DIL || g.dil_h > GT_MAX_DIL || g.dil_w > GT_MAX_DIL) return false;
    if ((g.kt - 1) * g.dil_t + 1 > GT_MAX_SPAN || (g.kh - 1) * g.dil_h + 1 > GT_MAX_SPAN ||
        (g.kw - 1) * g.dil_w + 1 > GT_MAX_SPAN)
        return false;
    pl.rank = depth ? 5 : 4;
    pl.taps = g.kt * g.kh * g.kw;
    pl.cbox = gt_cbox(c, esize, pl.taps, depth ? GT3_UNIT_BYTES : SIZE_MAX);
    if (!pl.cbox) return false;
    pl.uc = depth ? pl.cbox : c;
    pl.nbox = pl.uc / pl.cbox;
    pl.ngrp = c / pl.uc;
    pl.box_b = gt_round128((size_t)pl.cbox * pl.taps * esize);
    pl.row = pl.box_b * pl.nbox;
    pl.out_b = gt_round128((size_t)pl.uc * pl.taps * 4);
    // for fp32 the stage is never smaller than the output
    if (2 * pl.row + GT_OUT * (pl.row > pl.out_b ? pl.row : pl.out_b) + 1024 > 200 * 1024) return false;
    gt_ring(pl.row, pl.out_b, pl.per_sm, pl.nstage);
    // + 256: the 128-byte alignment of the base, and the XFORM kernels' stage origins (16 bytes per stage, nstage <= 6)
    pl.smem = (size_t)pl.nstage * pl.row + GT_OUT * pl.out_b + 2 * pl.nstage * 8 + 256;
    return true;
}

// The tensor map over (c, W, H, image) or (c, W, H, D, image).  The box spans the dilated window,
// (cbox, (kw-1)*dil_w+1, (kh-1)*dil_h+1[, (kt-1)*dil_t+1], 1); the traversal strides (1, dil_w, dil_h[, dil_t], 1)
// pick its taps, which land densely.
static int gt_encode(cp_handle_t h, CUtensorMap &map, const cp_patch_args &a, const GtPlan &pl) {
    const cp_window &g = a.g;
    const int esize = cp_fmap_esize(a.dtype), n = pl.rank;
    cuuint64_t dims[5] = {(cuuint64_t)a.c, (cuuint64_t)a.W, (cuuint64_t)a.H, (cuuint64_t)a.D,
                          (cuuint64_t)a.nbatch * a.B};
    if (n == 4) dims[3] = dims[4];  // no depth axis
    cuuint64_t strides[4] = {(cuuint64_t)a.c * esize};
    for (int i = 1; i < n - 1; ++i) strides[i] = strides[i - 1] * dims[i];
    const cuuint32_t box[5] = {(cuuint32_t)pl.cbox, (cuuint32_t)((g.kw - 1) * g.dil_w + 1),
                               (cuuint32_t)((g.kh - 1) * g.dil_h + 1), (cuuint32_t)((g.kt - 1) * g.dil_t + 1), 1};
    const cuuint32_t estr[5] = {1, (cuuint32_t)g.dil_w, (cuuint32_t)g.dil_h, (cuuint32_t)g.dil_t, 1};
    CUresult cr = ((encode_fn_t)h->tmap_encode)(&map, gt_dtype(a.dtype), n, (void *)a.fmap, dims, strides, box, estr,
                                                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                                CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) CP_FAIL(CP_ERR_CUDA, "cuTensorMapEncodeTiled (%d-D feature map) failed (%d)", n, (int)cr);
    // Elements the copy engine delivers per box, hence what expect_tx must announce (the kernel arms cbox * taps per
    // box): ceil(box[i] / estr[i]) per dimension (gt_box_elems)
    if (gt_box_elems(box, estr, n) != (size_t)pl.cbox * pl.taps)
        CP_FAIL(CP_ERR_CUDA, "%s: TMA box delivers %zu elements, the window has %zu", a.name, gt_box_elems(box, estr, n),
                (size_t)pl.cbox * pl.taps);
    return CP_OK;
}

// true when the TMA path takes a channels-last map that lies in device memory: 16-byte aligned fmap, X_out and ldx,
// and a plan (gt_plan); the caller takes the SIMT kernel otherwise
bool cp_gather_tma_applies(const cp_patch_args &a) {
    if (((uintptr_t)a.fmap & 15) || ((uintptr_t)a.X & 15) || (a.ldx % 4)) return false;
    GtPlan pl;
    return gt_plan(pl, cp_fmap_esize(a.dtype), a.c, a.g, a.randt != nullptr);
}

int cp_patch_gather_tma(cp_handle_t h, const cp_patch_args &a) {
    const int esize = cp_fmap_esize(a.dtype);
    GtPlan pl;
    if (!gt_plan(pl, esize, a.c, a.g, a.randt != nullptr))
        CP_FAIL(CP_ERR_INVALID, "%s: the window does not fit the TMA path", a.name);
    if (int rc = gt_encode_fn(h)) return rc;
    CUtensorMap map;
    if (int rc = gt_encode(h, map, a, pl)) return rc;
    const cp_window &g = a.g;
    GtXParams Pm{};
    Pm.randx = a.randx; Pm.randy = a.randy; Pm.randt = a.randt; Pm.X = a.X; Pm.ldx = a.ldx;
    Pm.ngrp = pl.ngrp;
    Pm.rows = a.rows() * pl.ngrp;  // work units
    Pm.B = a.B; Pm.P = a.P; Pm.c = pl.uc; Pm.k2 = pl.taps; Pm.relu = a.relu;
    Pm.pad_t = g.pad_t; Pm.pad_h = g.pad_h; Pm.pad_w = g.pad_w;
    Pm.stride_t = g.stride_t; Pm.stride_h = g.stride_h; Pm.stride_w = g.stride_w;
    Pm.cbox = pl.cbox; Pm.nbox = pl.nbox; Pm.nstage = pl.nstage;
    Pm.box_f = (int)(pl.box_b / esize); Pm.stage_f = (int)(pl.row / esize); Pm.out_f = (int)(pl.out_b / 4);
    Pm.g = g; Pm.D = a.D; Pm.H = a.H; Pm.W = a.W; Pm.xf = a.xf;
    return cp_with_fmap_type(a.dtype, [&](auto z) {
        using T = decltype(z);
        if (a.fused)
            return pl.rank == 5 ? gt_launch<5, T, true>(h, map, Pm, pl.smem, pl.per_sm, a.stream)
                                : gt_launch<4, T, true>(h, map, Pm, pl.smem, pl.per_sm, a.stream);
        return pl.rank == 5 ? gt_launch<5, T, false>(h, map, Pm, pl.smem, pl.per_sm, a.stream)
                            : gt_launch<4, T, false>(h, map, Pm, pl.smem, pl.per_sm, a.stream);
    });
}
