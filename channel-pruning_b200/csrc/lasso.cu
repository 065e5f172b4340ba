// LASSO channel selection on the device.
//
//   cp_lasso_build   <- construction of Z and sklearn's centring (reference
//                       lib/decompose.py:428-437, sklearn _pre_fit), in channel space
//   cp_lasso_select  <- the alpha search of decompose.dictionary (lib/decompose.py:489-525)
//                       with every Lasso.fit inside it (sklearn 1.9.0
//                       _cd_fast.pyx enet_coordinate_descent, selection='random',
//                       warm_start=True, tol=1e-4, gap-safe screening)
//
// The executable specification of cp_lasso_select is oracle/cd_oracle.c:cp_enet_cd_gram
// (same control flow as sklearn's data-form solver, evaluated on Q = Zc'Zc, q = Zc'yc,
// |yc|^2).  The kernel reproduces that model BIT FOR BIT: every floating-point operation
// the model rounds separately is issued with an explicit *_rn intrinsic (no FMA
// contraction), the gap reductions run in the model's "warp order", the division is
// correctly rounded, and the random coordinate order comes from the same 32-bit xorshift.
//
// Coordinate descent is one long serial dependency chain (each coordinate update needs the
// previous one), so the search is latency bound and is organised as ONE warp-specialised CTA
// per problem (7 warps), every warp doing only what must be on its own critical path:
//   chain warp     the serial recurrence only: x = Qw[j] (as published by the pair-update warps
//                  LAG steps ago) + the last LAG deltas applied locally, soft threshold,
//                  correctly rounded division (pre-computed reciprocal + one Markstein step),
//                  publish delta
//   4 update warps own interleaved pairs of Qw (in registers during a sweep), apply  Qw += delta * Q[j,:]
//                  (DMUL / DADD), stream the rows of Q from L2 into a register ring several steps ahead, and
//                  publish the Qw entry the chain warp will need LAG+1 steps later
//   packager warp  per-step operands of the chain (q_j, Q_jj, 1/Q_jj, the LAG entries
//                  Q[j_s][j_{s-i}]) gathered 32 steps at a time, lane-parallel
//   sequencer warp the xorshift stream of the NEXT sweep (it does not depend on the active set)
// Hand-offs are release/acquire counters in shared memory (bounded spins: a protocol bug traps
// instead of hanging); CTA barriers only at sweep boundaries.
#include <type_traits>

#include "common.cuh"

namespace {

// ------------------------------------------------------------------ build
__global__ void __launch_bounds__(256)
lasso_build_Q(const double *__restrict__ Gs, const double *__restrict__ WW, const double *__restrict__ sxs,
              const double *__restrict__ sw, int c, int k2, double m, double *__restrict__ Q, int ldq) {
    const int b = blockIdx.x * 16 + (threadIdx.x & 15);
    const int a = blockIdx.y * 16 + (threadIdx.x >> 4);
    if (a >= c || b >= ldq) return;
    if (b >= c) {  // padding column (keeps rows 16-byte aligned for the selection kernel)
        Q[(int64_t)a * ldq + b] = 0.0;
        return;
    }
    const int64_t K = (int64_t)c * k2;
    double s = 0.0, za = 0.0, zb = 0.0;
    for (int p = 0; p < k2; ++p) {
        const double *g = Gs + ((int64_t)a * k2 + p) * K + (int64_t)b * k2;
        const double *w = WW + ((int64_t)a * k2 + p) * K + (int64_t)b * k2;
        for (int q = 0; q < k2; ++q) s = fma(g[q], w[q], s);
        za = fma(sxs[a * k2 + p], sw[a * k2 + p], za);
        zb = fma(sxs[b * k2 + p], sw[b * k2 + p], zb);
    }
    Q[(int64_t)a * ldq + b] = s - za * zb / m;  // - m * zbar_a * zbar_b
}

// qv[a] = sum_{p,j} W2[j,(a,p)] * Bs[(a,p), j] - m zbar_a ybar ;  block per channel, fixed-shape tree.
__global__ void __launch_bounds__(128)
lasso_build_q(const float *__restrict__ W2, const double *__restrict__ Bs, const double *__restrict__ sxs,
              const double *__restrict__ sw, const double *__restrict__ sys, const double *__restrict__ yys, int c,
              int k2, int n, double m, double *__restrict__ qv, double *__restrict__ yn2) {
    __shared__ double red[128];
    const int a = blockIdx.x;
    const int64_t K = (int64_t)c * k2;
    double s = 0.0;
    for (int e = threadIdx.x; e < k2 * n; e += 128) {
        const int p = e / n, j = e - p * n;
        s = fma((double)W2[(int64_t)j * K + a * k2 + p], Bs[((int64_t)a * k2 + p) * n + j], s);
    }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int w = 64; w > 0; w >>= 1) {
        if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        double za = 0.0;
        for (int p = 0; p < k2; ++p) za = fma(sxs[a * k2 + p], sw[a * k2 + p], za);
        double ysum = 0.0;
        for (int j = 0; j < n; ++j) ysum += sys[j];
        qv[a] = red[0] - za * ysum / m;  // - m * (za/m) * (ysum/m)
        if (a == 0) *yn2 = *yys - ysum * ysum / m;
    }
}

// ------------------------------------------------------------------ select
struct SelectParams {
    const double *Q;
    int ldq;
    const double *qv, *yn2;
    int c;
    double m;
    int rank;
    double lbound, rbound, right0, tol;
    int max_iter;
    const uint32_t *seeds;
    int max_probes;
    uint8_t *out_idxs;
    double *out_coef, *out_scalars, *out_probe_log;
};

constexpr int MAXC = 2048;   // largest channel count (shared-memory bound)
// Deltas the chain warp applies itself (slack of the update warps).  The unrolled chain / update blocks are laid out for
// LAG = 4: the delta ring is static across 16-step blocks and the publish targets sit inside two 16-byte index loads.
constexpr int LAG = 4;
constexpr int NBULK = 4;     // pair-update warps
// Role of a warp inside a sweep.  The chain warp sits on warp CHAIN_W: with 7 warps on 4 scheduler partitions, warp 3
// is the only one that has a partition to itself (0/4, 1/5, 2/6 share), so the serial recurrence never competes for
// issue slots with a polling warp.  Roles of the others, in warp order: NBULK update warps, packager, sequencer.
constexpr int CHAIN_W = 3;
// Polling back-off (ns) of the warps that wait for the chain: a tight LDS polling loop of five warps keeps the
// shared-memory pipe busy and lengthens every shared-memory access of the chain warp.
constexpr int POLL_SLEEP_NS = 32;
constexpr int WS_THREADS = 32 * (3 + NBULK);
__device__ __forceinline__ int role_of(int warp) {  // -1 chain, 0..NBULK-1 update, NBULK packager, NBULK+1 sequencer
    return warp == CHAIN_W ? -1 : (warp < CHAIN_W ? warp : warp - 1);
}
__device__ __forceinline__ void poll_backoff() { __nanosleep(POLL_SLEEP_NS); }
constexpr int QR = 64;       // rings of per-step scalars (steps in flight << QR)

__device__ __forceinline__ uint32_t xorshift_step(uint32_t s) {  // sklearn/utils/_random.pxd:20-34 (state update)
    if (s == 0) s = 1;
    s ^= s << 13;
    s ^= s >> 17;
    s ^= s << 5;
    return s;
}
// a % d for 32-bit a through a pre-computed M = floor(2^64 / d) + 1 (Lemire's fastmod; exact)
__device__ __forceinline__ uint32_t fastmod(uint32_t a, uint64_t M, uint32_t d) {
    return (uint32_t)__umul64hi(M * (uint64_t)a, (uint64_t)d);
}

__device__ __forceinline__ void st_release(int *p, int v) {
    asm volatile("st.release.cta.shared.b32 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(p)), "r"(v) : "memory");
}
__device__ __forceinline__ int ld_acquire(const int *p) {
    int v;
    asm volatile("ld.acquire.cta.shared.b32 %0, [%1];" : "=r"(v) : "r"((uint32_t)__cvta_generic_to_shared(p)) : "memory");
    return v;
}
// bounded spin: a protocol bug traps (CUDA error) instead of hanging the GPU
__device__ __forceinline__ void wait_ge(const int *p, int target) {
    for (uint32_t spin = 0; ld_acquire(p) < target; ++spin)
        if (spin > (1u << 26)) __trap();
}
// ring-reuse positions: published with st_release after a __syncwarp, so that the reads of the slots they free are
// ordered before the waiter's overwrite
__device__ __forceinline__ void wait_ge_backoff(const int *p, int target) {
    for (uint32_t spin = 0; ld_acquire(p) < target; ++spin) {
        if (spin > (1u << 26)) __trap();
        poll_backoff();
    }
}
// Tagged 16-byte records {value, check}: ONE st.shared.v2.f64 / ld.shared.v2.f64 each, no fence on the serial chain.
// A vector access is not single-copy atomic, so check = value bits XOR a mix of the tag: a read that combines halves of
// two records fails the check (unless both held the same value) and is repeated.
__device__ __forceinline__ long long tag_mix(uint32_t tag) {
    return (long long)(((uint64_t)tag * 0x9E3779B97F4A7C15ull) | 1ull);
}
__device__ __forceinline__ bool tag_ok(double v, double t, uint32_t tag) {
    return (__double_as_longlong(v) ^ __double_as_longlong(t)) == tag_mix(tag);
}
__device__ __forceinline__ void put_tagged(uint32_t slot_saddr, double v, uint32_t tag) {
    asm volatile("st.volatile.shared.v2.f64 [%0], {%1, %2};" ::"r"(slot_saddr), "d"(v),
                 "d"(__longlong_as_double(__double_as_longlong(v) ^ tag_mix(tag)))
                 : "memory");
}
__device__ __forceinline__ double get_tagged(uint32_t slot_saddr, uint32_t tag) {
    double v, t;
    for (uint32_t spin = 0;; ++spin) {
        asm volatile("ld.volatile.shared.v2.f64 {%0, %1}, [%2];" : "=d"(v), "=d"(t) : "r"(slot_saddr) : "memory");
        if (tag_ok(v, t, tag)) break;
        if (spin > (1u << 26)) __trap();
    }
    return v;
}

// waiting variant for the warps that trail the chain: backs off between polls
__device__ __forceinline__ double wait_tagged(uint32_t slot_saddr, uint32_t tag) {
    double v, t;
    for (uint32_t spin = 0;; ++spin) {
        asm volatile("ld.volatile.shared.v2.f64 {%0, %1}, [%2];" : "=d"(v), "=d"(t) : "r"(slot_saddr) : "memory");
        if (tag_ok(v, t, tag)) break;
        if (spin > (1u << 24)) __trap();
        poll_backoff();
    }
    return v;
}
// the same record read WITHOUT waiting for the tag: the caller checks it later (after the latency has been hidden)
__device__ __forceinline__ void peek_tagged(uint32_t slot_saddr, double &v, double &t) {
    asm volatile("ld.volatile.shared.v2.f64 {%0, %1}, [%2];" : "=d"(v), "=d"(t) : "r"(slot_saddr) : "memory");
}

__device__ __forceinline__ double warp_sum_butterfly(double v) {  // model: p[l] + p[l ^ off], off = 16..1
#pragma unroll
    for (int off = 16; off; off >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, off));
    return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int off = 16; off; off >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, off));
    return v;
}

// correctly rounded num / d given rc = RN(1/d):  q0 = RN(num*rc), r = num - q0*d (exact), q = RN(q0 + r*rc)
__device__ __forceinline__ double div_markstein(double num, double d, double rc) {
    const double q0 = __dmul_rn(num, rc);
    const double r = __fma_rn(-q0, d, num);
    return __fma_rn(r, rc, q0);
}

#ifdef CP_TIMING
constexpr int TSTEPS = 384;
__device__ long long cp_lasso_times[TSTEPS * 8];  // per step: chain {top, fetched, confirmed, published}, update warp {poll, got, pub, end}
#define CH_STAMP(s, i)                                                                   \
    do {                                                                                 \
        if (rec && lane == 0 && (s) < TSTEPS) cp_lasso_times[(s) * 8 + (i)] = clock64(); \
    } while (0)
#else
#define CH_STAMP(s, i)
#endif

struct Ctl {  // CTA-wide scalars
    int chain_pos, bulk_pos[NBULK], pk_pos;
    int n_active, nnz, pad;
    double gap, dual_norm, w_max, d_w_max;
};

template <int NPB>  // pairs per update lane; padded channel count CP = 2 * 32 * NBULK * NPB
__global__ void __launch_bounds__(WS_THREADS, 1) lasso_select_kernel(const SelectParams P) {
    constexpr int BL = 32 * NBULK;  // update lanes
    constexpr int CP = 2 * BL * NPB;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int c = P.c, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    double *w = reinterpret_cast<double *>(smem_raw);  // [CP]
    double *Qw = w + CP;
    double *qv = Qw + CP;
    double *dg = qv + CP;
    double *pk = dg + CP;                   // [QR][8]: q, Qjj, 1/Qjj, r1 .. r5
    double *dq = pk + QR * 8;               // [QR][2] published {delta, tag}
    double *xq = dq + QR * 2;               // [QR][2] published {Qw entry, tag}
    uint32_t *active = reinterpret_cast<uint32_t *>(xq + QR * 2);
    uint32_t *jz = active + CP;             // coordinate sequence of the sweep / eviction list of the screening
    uint32_t *raw = jz + CP;                // [2][CP] xorshift states (this sweep / next sweep)
    uint8_t *excluded = reinterpret_cast<uint8_t *>(raw + 2 * CP);
    __shared__ Ctl ctl;

    const double *__restrict__ Q = P.Q;
    const int ldq = P.ldq;
    const double yn2 = *P.yn2;
    for (int e = tid; e < CP; e += WS_THREADS) {
        w[e] = 0.0;
        Qw[e] = 0.0;
        const bool in = e < c;
        qv[e] = in ? P.qv[e] : 0.0;
        dg[e] = in ? Q[(int64_t)e * ldq + e] : 0.0;
        active[e] = e;
        excluded[e] = 0;
    }
    for (int e = tid; e < QR * 4; e += WS_THREADS) dq[e] = 0.0;  // dq and xq: no tag matches {0, 0}
    __syncthreads();
    uint32_t sweep_no = 1;  // tags are (sweep_no << 12) | (step + 1): unique over the whole launch (< 2^20 sweeps)

    const double tolS = __dmul_rn(P.tol, yn2);
    int probe = 0, status = 0;

    // ================= helpers that run on warp 0 alone (between sweeps) =================
    // Qw += a * Q[j,:], row fetched directly (rare path: screening evictions)
    auto axpy_row_direct = [&](uint32_t j, double a) {
        const double *src = Q + (int64_t)j * ldq;
        for (int e = 2 * lane; e < c; e += 64) {
            const double2 r = *reinterpret_cast<const double2 *>(src + e);
            double2 v = *reinterpret_cast<double2 *>(Qw + e);
            v.x = __dadd_rn(v.x, __dmul_rn(a, r.x));
            v.y = __dadd_rn(v.y, __dmul_rn(a, r.y));
            *reinterpret_cast<double2 *>(Qw + e) = v;
        }
    };
    // gap_enet_gram + dual_gap_formulation_A (beta = 0) in warp order
    auto gap_check = [&](double l1) {
        double a1 = 0.0, a2 = 0.0, a3 = 0.0, dn = 0.0;
        for (int i = lane; i < c; i += 32) {
            const double wi = w[i];
            a1 = __dadd_rn(a1, __dmul_rn(wi, qv[i]));
            a2 = __dadd_rn(a2, __dmul_rn(wi, Qw[i]));
            a3 = __dadd_rn(a3, fabs(wi));
            dn = fmax(dn, fabs(__dadd_rn(qv[i], -Qw[i])));
        }
        const double q_dot_w = warp_sum_butterfly(a1);
        const double wQw = warp_sum_butterfly(a2);
        const double l1n = warp_sum_butterfly(a3);
        dn = warp_max(dn);
        const double R_norm2 = __dadd_rn(__dadd_rn(yn2, wQw), -__dmul_rn(2.0, q_dot_w));
        const double Ry = __dadd_rn(yn2, -q_dot_w);
        const double primal = __dadd_rn(__dmul_rn(0.5, R_norm2), __dmul_rn(l1, l1n));
        const double scale = dn > l1 ? __ddiv_rn(l1, dn) : 1.0;
        const double dual = __dadd_rn(__dmul_rn(__dmul_rn(-0.5, __dmul_rn(scale, scale)), R_norm2), __dmul_rn(scale, Ry));
        if (lane == 0) {
            ctl.gap = __dadd_rn(primal, -dual);
            ctl.dual_norm = dn;
        }
        __syncwarp();
    };
    // gap-safe screening: keep j iff (1 - |XtA_j / max(l1, dn)|) / sqrt(Q_jj) <= sqrt(2|gap|) / l1
    auto screen = [&](bool first, double l1, double gap, double dual_norm) {
        const double radius = __ddiv_rn(sqrt(__dmul_rn(2.0, fabs(gap))), l1);
        const double den = l1 > dual_norm ? l1 : dual_norm;
        int na = 0, nz = 0;
        for (int base = 0; base < c; base += 32) {
            const int j = base + lane;
            bool keep = false, evict_nonzero = false;
            if (j < c) {
                if (first && dg[j] == 0.0) {
                    w[j] = 0.0;  // zero column
                    excluded[j] = 1;
                } else if (!first && excluded[j]) {
                    // stays excluded
                } else {
                    const double th = __ddiv_rn(__dadd_rn(qv[j], -Qw[j]), den);
                    const double d_j = __ddiv_rn(__dadd_rn(1.0, -fabs(th)), sqrt(dg[j]));
                    keep = d_j <= radius;
                    if (!keep) {
                        evict_nonzero = w[j] != 0.0;
                        excluded[j] = 1;
                    } else excluded[j] = 0;
                }
            }
            const uint32_t mk = __ballot_sync(0xffffffffu, keep);
            const uint32_t mz = __ballot_sync(0xffffffffu, evict_nonzero);
            const uint32_t lt = (1u << lane) - 1u;
            if (keep) active[na + __popc(mk & lt)] = j;
            if (evict_nonzero) jz[nz + __popc(mz & lt)] = j;
            na += __popc(mk);
            nz += __popc(mz);
        }
        __syncwarp();
        for (int z = 0; z < nz; ++z) {  // Qw -= w[j] * Q[j,:], ascending j like the model
            const uint32_t j = jz[z];
            axpy_row_direct(j, -w[j]);
            __syncwarp();
        }
        for (int z = lane; z < nz; z += 32) w[jz[z]] = 0.0;
        if (lane == 0) ctl.n_active = na;
        __syncwarp();
    };

    // ================= one sweep over the active set, all warps =================
    // soft-threshold update of one coordinate from the current x = Qw[j]
    auto cd_update = [&](double qj, double Qjj, double rj, double x, double w_j, double l1, double &delta, double &aw,
                         double &w_new) {
        const double tmp = __dadd_rn(__dadd_rn(qj, -x), __dmul_rn(w_j, Qjj));
        const double mag = __dadd_rn(fabs(tmp), -l1);
        // fsign(tmp) * fmax(|tmp| - l1, 0) / Qjj  (Qjj > 0): signed zero when thresholded away
        const double wn = mag > 0.0 ? div_markstein(copysign(mag, tmp), Qjj, rj) : (tmp < 0.0 ? -0.0 : 0.0);
        // model: "if Qjj == 0: continue" -- cannot trigger here: the first screening of every fit removes
        // zero-diagonal columns from the active set, and only active coordinates are visited
        w_new = wn;
        delta = __dadd_rn(wn, -w_j);
        aw = fabs(wn);
    };
    auto sweep = [&](int n_active, bool fresh, uint32_t seed, int cur, double l1) {
        uint32_t *raw_cur = raw + cur * CP, *raw_nxt = raw + (cur ^ 1) * CP;
        if (fresh) {  // first sweep of a fit: the stream restarts from this fit's seed
            if (role_of(warp) == NBULK + 1 && lane == 0) {
                uint32_t st = seed;
                for (int f = 0; f < n_active; ++f) {
                    st = xorshift_step(st);
                    raw_cur[f] = st;
                }
            }
            __syncthreads();
        }
        {
            const uint64_t M = ~0ull / (uint32_t)n_active + 1ull;
            for (int f = tid; f < n_active; f += WS_THREADS)
                jz[f] = active[fastmod(raw_cur[f] & 0x7fffffffu, M, (uint32_t)n_active)];
            if (tid == 0) {
                ctl.chain_pos = 0;
                ctl.pk_pos = 0;
#pragma unroll
                for (int b = 0; b < NBULK; ++b) ctl.bulk_pos[b] = 0;
            }
        }
        __syncthreads();
        const uint32_t tag0 = sweep_no << 12;
#ifdef CP_TIMING
        const bool rec = (probe == 0 && sweep_no == 3);
#endif
        const uint32_t dq_s = (uint32_t)__cvta_generic_to_shared(dq), xq_s = (uint32_t)__cvta_generic_to_shared(xq);
        const int role = role_of(warp);
        if (role < 0) {
            // -------- chain warp: the serial recurrence and nothing else.  One warp alone hides no latency (every
            // dependent instruction costs its full pipeline depth), so the loop is organised for the fewest
            // instructions per step: blocks of 16 steps fully unrolled, two operand sets used alternately (no
            // register rotation), ring addresses and tags that are compile-time offsets from a per-block base, the
            // last LAG deltas in a ring indexed by the step number (LAG divides 16), hand-shake bookkeeping once
            // per block.  The operands of step s+1 (coordinate, packaged scalars, w[j], the published Qw entry) are
            // fetched BEFORE the dependent arithmetic of step s.
            double D[LAG];  // D[s % LAG] = delta of step s
#pragma unroll
            for (int i = 0; i < LAG; ++i) D[i] = 0.0;
            double w_max = 0.0, d_w_max = 0.0;
            uint32_t J[2];
            double P[2][8];  // q, Qjj, 1/Qjj, r1..r5
            double WJ[2], XV[2], XT[2];
            const uint32_t w_s = (uint32_t)__cvta_generic_to_shared(w);
            auto fetch = [&](int set, int s, int slot) {  // slot = s & (QR - 1)
                const uint32_t jv = jz[s];
                J[set] = jv;
                const double2 *rec = reinterpret_cast<const double2 *>(pk + slot * 8);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const double2 v = rec[q];
                    P[set][2 * q] = v.x;
                    P[set][2 * q + 1] = v.y;
                }
                WJ[set] = w[jv];
                // Qw[j] as of update s-LAG-1, published by the owning update lane (tag checked at use)
                peek_tagged(xq_s + (uint32_t)slot * 16u, XV[set], XT[set]);
            };
            auto block_sync = [&](int s0) {  // before any step of s0 .. s0+15 or the fetch of s0+16
                wait_ge(&ctl.pk_pos, s0 + 17 < n_active ? s0 + 17 : n_active);
                // operands of steps <= s0 are in registers: their slots may be reused
                __syncwarp();
                if (lane == 0) st_release(&ctl.chain_pos, s0);
                if (s0 >= 32) {  // nobody may fall more than ~32 steps behind (ring reuse)
#pragma unroll
                    for (int b = 0; b < NBULK; ++b) wait_ge_backoff(&ctl.bulk_pos[b], s0 - 24);
                }
            };
            auto run_block = [&](auto guarded, int s0) {
                constexpr bool GUARD = decltype(guarded)::value;
                const int sb = s0 & (QR - 1);
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const int s = s0 + i;
                    if (GUARD && s >= n_active) break;
                    const int cur = i & 1, nxt = cur ^ 1;
                    CH_STAMP(s, 0);
                    const bool has_next = (GUARD || i == 15) ? (s + 1 < n_active) : true;
                    if (has_next) fetch(nxt, s + 1, i == 15 ? ((sb + 16) & (QR - 1)) : sb + i + 1);
                    asm volatile("" ::: "memory");  // the loads above stay above the arithmetic below
                    CH_STAMP(s, 1);
                    const uint32_t tag = tag0 + (uint32_t)(s + 1);
                    const uint32_t j = J[cur];
                    double xv = XV[cur];
                    if (!tag_ok(XV[cur], XT[cur], tag)) xv = get_tagged(xq_s + (uint32_t)(sb + i) * 16u, tag);
                    // the lanes leave the spin above independently; w[] below is written by every lane and read back
                    // by every lane one step later, so a lane must not run ahead of one still storing an older w[j]
                    __syncwarp();
                    CH_STAMP(s, 2);
                    double x = xv;
#pragma unroll
                    for (int k = LAG; k >= 1; --k)  // oldest delta first: delta_{s-k} * Q[j_s][j_{s-k}]
                        x = __dadd_rn(x, __dmul_rn(D[(i + 16 * LAG - k) % LAG], P[cur][2 + k]));
                    double delta, aw, w_new;
                    cd_update(P[cur][0], P[cur][1], P[cur][2], x, WJ[cur], l1, delta, aw, w_new);
                    w[j] = w_new;  // every lane stores the same value: no intra-warp ordering needed
                    if (lane == 0) put_tagged(dq_s + (uint32_t)(sb + i) * 16u, delta, tag);
                    CH_STAMP(s, 3);
                    d_w_max = fmax(d_w_max, fabs(delta));
                    w_max = fmax(w_max, aw);
                    D[i % LAG] = delta;
                    if (has_next && J[nxt] == j) WJ[nxt] = w_new;  // same coordinate twice in a row: prefetched w[j] stale
                }
            };
            (void)w_s;
            block_sync(0);
            fetch(0, 0, 0);
            for (int s0 = 0; s0 < n_active; s0 += 16) {
                if (s0) block_sync(s0);
                if (s0 + 16 <= n_active) run_block(std::false_type{}, s0);
                else run_block(std::true_type{}, s0);
            }
            if (lane == 0) {
                ctl.w_max = w_max;
                ctl.d_w_max = d_w_max;
            }
        } else if (role < NBULK) {
            // -------- pair-update warps: this lane's NPB pairs of Qw live in REGISTERS for the whole sweep (loaded from /
            // written back to shared memory at its ends); the pairs of row t are in registers before delta_t arrives
            const int b = role, bt = b * 32 + lane;
            const double *Qmine = Q + 2 * bt;                  // this lane's first pair of any row
            // The rows of Q go straight from L2 into a REGISTER ring, DEPTH steps ahead (ld.global.nc, no shared-memory
            // staging: a cp.async ring cost a commit, a wait and a shared-memory read per step on a warp that hides no
            // latency).  Blocks of DEPTH steps are fully unrolled, so ring slots, record slots and the publish targets
            // are compile-time offsets; the coordinates a block needs arrive in 16-byte index loads.
            constexpr int DEPTH = NPB <= 2 ? 8 : 4;
            double2 qw[NPB], rr[DEPTH][NPB];
#pragma unroll
            for (int sp = 0; sp < NPB; ++sp) qw[sp] = *reinterpret_cast<const double2 *>(Qw + 2 * BL * sp + 2 * bt);
            auto fetch_row = [&](uint32_t j, int slot) {
                const double *src = Qmine + (uint32_t)(j * (uint32_t)ldq);  // c * ldq < 2^31
#pragma unroll
                for (int sp = 0; sp < NPB; ++sp) {
                    double2 v = make_double2(0.0, 0.0);
                    if (2 * BL * sp + 2 * bt < c) v = __ldg(reinterpret_cast<const double2 *>(src + 2 * BL * sp));
                    rr[slot][sp] = v;
                }
            };
            // entry js of Qw if this lane owns it (element 2*BL*sp + 2*bt + h)
            auto publish = [&](uint32_t js, int step) {
                const int ob = (int)((js >> 1) & (BL - 1));
                if ((ob >> 5) == b) {  // warp-uniform: only the owning warp looks for the owning lane
                    if ((ob & 31) == lane) {
                        const int spj = (int)(js >> 1) / BL;
                        double v = 0.0;
#pragma unroll
                        for (int sp = 0; sp < NPB; ++sp)
                            if (sp == spj) v = (js & 1) ? qw[sp].y : qw[sp].x;
                        put_tagged(xq_s + (uint32_t)(step & (QR - 1)) * 16u, v, tag0 + (uint32_t)(step + 1));
                    }
                }
            };
#pragma unroll
            for (int d = 0; d < DEPTH; ++d)
                if (d < n_active) fetch_row(jz[d], d);
            for (int s = 0; s <= LAG && s < n_active; ++s) publish(jz[s], s);  // entries the chain needs before any update
            static_assert(QR % DEPTH == 0 && LAG + 1 <= 8, "block layout of the update warps");
            auto run_block = [&](auto guarded, int t0) {
                constexpr bool GUARD = decltype(guarded)::value;
                const int sb = t0 & (QR - 1);
                // coordinates: rows t0+DEPTH .. t0+2*DEPTH-1 to fetch, entries t0+LAG+1 .. t0+LAG+DEPTH to publish
                uint32_t jr[DEPTH], jp[DEPTH + 8];
#pragma unroll
                for (int q = 0; q < DEPTH / 4; ++q) {
                    const uint4 v = *reinterpret_cast<const uint4 *>(jz + t0 + DEPTH + 4 * q);  // (beyond n_active: unused)
                    jr[4 * q] = v.x; jr[4 * q + 1] = v.y; jr[4 * q + 2] = v.z; jr[4 * q + 3] = v.w;
                }
#pragma unroll
                for (int q = 0; q < (DEPTH + 8) / 4; ++q) {
                    const uint4 v = *reinterpret_cast<const uint4 *>(jz + t0 + 4 * q);  // jz[t0 .. t0+DEPTH+7]
                    jp[4 * q] = v.x; jp[4 * q + 1] = v.y; jp[4 * q + 2] = v.z; jp[4 * q + 3] = v.w;
                }
#pragma unroll
                for (int u = 0; u < DEPTH; ++u) {
                    const int t = t0 + u;
                    if (GUARD && t >= n_active) break;
#ifdef CP_TIMING
                    if (rec && b == 0 && lane == 0 && t < TSTEPS) cp_lasso_times[t * 8 + 4] = clock64();
#endif
                    const double delta = wait_tagged(dq_s + (uint32_t)(sb + u) * 16u, tag0 + (uint32_t)(t + 1));
#ifdef CP_TIMING
                    if (rec && b == 0 && lane == 0 && t < TSTEPS) cp_lasso_times[t * 8 + 5] = clock64();
#endif
                    if (delta != 0.0) {
#pragma unroll
                        for (int sp = 0; sp < NPB; ++sp) {
                            qw[sp].x = __dadd_rn(qw[sp].x, __dmul_rn(delta, rr[u][sp].x));
                            qw[sp].y = __dadd_rn(qw[sp].y, __dmul_rn(delta, rr[u][sp].y));
                        }
                    }
                    const int sp1 = t + LAG + 1;  // the chain step that starts from Qw after THIS update
                    if (sp1 < n_active) publish(jp[u + LAG + 1], sp1);
#ifdef CP_TIMING
                    if (rec && b == 0 && lane == 0 && t < TSTEPS) cp_lasso_times[t * 8 + 6] = clock64();
#endif
                    if (t + DEPTH < n_active) fetch_row(jr[u], u);  // row t is consumed: its ring slot takes row t+DEPTH
#ifdef CP_TIMING
                    if (rec && b == 0 && lane == 0 && t < TSTEPS) cp_lasso_times[t * 8 + 7] = clock64();
#endif
                }
                if (DEPTH == 8 || (t0 & 4)) {
                    __syncwarp();
                    if (lane == 0) st_release(&ctl.bulk_pos[b], t0 + DEPTH);
                }
            };
            for (int t0 = 0; t0 < n_active; t0 += DEPTH) {
                if (t0 + DEPTH <= n_active) run_block(std::false_type{}, t0);
                else run_block(std::true_type{}, t0);
            }
#pragma unroll
            for (int sp = 0; sp < NPB; ++sp) *reinterpret_cast<double2 *>(Qw + 2 * BL * sp + 2 * bt) = qw[sp];
        } else if (role == NBULK) {
            // -------- packager: operands of 32 chain steps at a time
            for (int base = 0; base < n_active; base += 32) {
                if (base >= QR) wait_ge_backoff(&ctl.chain_pos, base - 32);  // slots of batch base-64 are free
                const int s = base + lane;
                if (s < n_active) {
                    const uint32_t j = jz[s];
                    const double d = dg[j];
                    const double *qrow = Q + (int64_t)j * ldq;
                    double rr[5];
#pragma unroll
                    for (int i = 1; i <= 5; ++i) rr[i - 1] = (i <= LAG && s >= i) ? __ldg(qrow + jz[s - i]) : 0.0;
                    double *o = pk + (s & (QR - 1)) * 8;
                    *reinterpret_cast<double2 *>(o) = make_double2(qv[j], d);
                    *reinterpret_cast<double2 *>(o + 2) = make_double2(d != 0.0 ? __drcp_rn(d) : 0.0, rr[0]);
                    *reinterpret_cast<double2 *>(o + 4) = make_double2(rr[1], rr[2]);
                    *reinterpret_cast<double2 *>(o + 6) = make_double2(rr[3], rr[4]);
                }
                __syncwarp();
                if (lane == 0) st_release(&ctl.pk_pos, base + 32 < n_active ? base + 32 : n_active);
            }
        } else {
            // -------- sequencer: xorshift states of the next sweep (independent of the active set)
            if (lane == 0) {
                uint32_t st = raw_cur[n_active - 1];
                for (int f = 0; f < n_active; ++f) {
                    st = xorshift_step(st);
                    raw_nxt[f] = st;
                }
            }
        }
        ++sweep_no;
        __syncthreads();
    };

    // ---- one Lasso.fit (warm start) at l1 = alpha*m; returns nnz (uniform across the CTA)
    auto solve = [&](double alpha_user) -> int {
        const double l1 = __dmul_rn(alpha_user, P.m);
        const uint32_t seed = P.seeds[probe];
        int n_active = c, n_iter_ret = 0;
        if (warp == 0) gap_check(l1);
        __syncthreads();
        double gap = ctl.gap, dual_norm = ctl.dual_norm;
        if (!(gap <= tolS)) {
            if (warp == 0) screen(true, l1, gap, dual_norm);
            __syncthreads();
            n_active = ctl.n_active;
            bool broke = false, fresh = true;
            int cur = 0, n_iter = 0;
            for (n_iter = 0; n_iter < P.max_iter; ++n_iter) {
                double w_max = 0.0, d_w_max = 0.0;
                if (n_active > 0) {
                    sweep(n_active, fresh, seed, cur, l1);
                    fresh = false;
                    cur ^= 1;
                    w_max = ctl.w_max;
                    d_w_max = ctl.d_w_max;
                }
                if (w_max == 0.0 || __ddiv_rn(d_w_max, w_max) <= P.tol || n_iter == P.max_iter - 1) {
                    __syncthreads();  // everyone has read ctl.w_max before warp 0 moves on
                    if (warp == 0) gap_check(l1);
                    __syncthreads();
                    gap = ctl.gap;
                    dual_norm = ctl.dual_norm;
                    if (gap <= tolS) { broke = true; break; }
                    if (warp == 0) screen(false, l1, gap, dual_norm);
                    __syncthreads();
                    n_active = ctl.n_active;
                }
            }
            n_iter_ret = broke ? n_iter + 1 : P.max_iter;
        }
        if (warp == 0) {
            int cnt = 0;
            for (int i = lane; i < c; i += 32) cnt += (w[i] != 0.0);
#pragma unroll
            for (int off = 16; off; off >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, off);
            if (lane == 0) {
                ctl.nnz = cnt;
                double *lg = P.out_probe_log + (size_t)probe * 4;
                lg[0] = alpha_user; lg[1] = (double)cnt; lg[2] = (double)n_iter_ret; lg[3] = gap;
            }
        }
        __syncthreads();
        const int nnz = ctl.nnz;
        __syncthreads();
        ++probe;
        return nnz;
    };

    // ---- alpha search, reference lib/decompose.py:489-525
    double left = 0.0, right = P.right0, alpha = P.right0;
    int nnz = 0;
    bool done = false;
    while (true) {  // :502-515  relax right until fewer than `rank` survive
        if (probe >= P.max_probes) { status = 1; done = true; break; }
        alpha = right;
        nnz = solve(right);
        if (nnz < P.rank) break;
        right = __dmul_rn(right, 2.0);
    }
    while (!done) {  // :516-525  bisection into [lbound, rbound]
        if (probe >= P.max_probes) { status = 1; break; }
        alpha = __dmul_rn(__dadd_rn(left, right), 0.5);
        nnz = solve(alpha);
        if ((double)nnz > P.rbound) left = alpha;
        else if ((double)nnz < P.lbound) right = alpha;
        else break;
    }
    for (int e = tid; e < c; e += WS_THREADS) {
        P.out_idxs[e] = w[e] != 0.0 ? 1 : 0;
        P.out_coef[e] = w[e];
    }
    if (tid == 0) {
        P.out_scalars[0] = alpha;
        P.out_scalars[1] = (double)probe;
        P.out_scalars[2] = (double)status;
        P.out_scalars[3] = (double)nnz;
    }
}

template <int NPB>
int launch_select(const SelectParams &P, cudaStream_t stream) {
    constexpr int CP = 2 * 32 * NBULK * NPB;
    const size_t smem = (size_t)CP * 4 * sizeof(double) + (size_t)QR * 12 * sizeof(double) +
                        (size_t)CP * (4 * sizeof(uint32_t) + 1) + 16;
    static cp_per_device_flag configured;  // per instantiation, per device
    if (bool *done = configured.slot(); !*done) {
        CP_CUDA(cudaFuncSetAttribute(lasso_select_kernel<NPB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        *done = true;
    }
    lasso_select_kernel<NPB><<<1, WS_THREADS, smem, stream>>>(P);
    CP_CHECK_LAUNCH();
    return CP_OK;
}

}  // namespace

#ifdef CP_TIMING
extern "C" int cp_debug_lasso_times(long long *host_out) {  // 384 steps x 8 clock64 stamps (third sweep of the first fit)
    return (int)cudaMemcpyFromSymbol(host_out, cp_lasso_times, sizeof(long long) * 384 * 8);
}
#endif

extern "C" int cp_lasso_build(cp_handle_t h, const double *Gs, const double *Bs, const double *sxs,
                              const double *sys, const double *yys, const double *WW, const double *sw,
                              const float *W2, int c, int k2, int n, int S, double *Q, int ldq, double *qv,
                              double *yn2, cp_stream_t stream_) {
    CP_REQUIRE(h && Gs && Bs && sxs && sys && yys && WW && sw && W2 && Q && qv && yn2, "cp_lasso_build: NULL argument");
    CP_REQUIRE(c > 0 && k2 > 0 && n > 0 && S > 0, "cp_lasso_build: bad shape");
    CP_REQUIRE(ldq >= c && (ldq % 2) == 0, "cp_lasso_build: ldq must be even and >= c (got %d)", ldq);
    cudaStream_t stream = (cudaStream_t)stream_;
    const double m = (double)S * (double)n;
    dim3 grid(cp_cdiv(ldq, 16), cp_cdiv(c, 16));
    lasso_build_Q<<<grid, 256, 0, stream>>>(Gs, WW, sxs, sw, c, k2, m, Q, ldq);
    CP_CHECK_LAUNCH();
    lasso_build_q<<<c, 128, 0, stream>>>(W2, Bs, sxs, sw, sys, yys, c, k2, n, m, qv, yn2);
    CP_CHECK_LAUNCH();
    return CP_OK;
}

extern "C" int cp_lasso_select(cp_handle_t h, const double *Q, int ldq, const double *qv, const double *yn2, int c,
                               double m, int rank, double lbound, double rbound, double right0, double tol,
                               int max_iter, const uint32_t *seeds, int max_probes, uint8_t *out_idxs,
                               double *out_coef, double *out_scalars, double *out_probe_log, cp_stream_t stream_) {
    CP_REQUIRE(h && Q && qv && yn2 && seeds && out_idxs && out_coef && out_scalars && out_probe_log,
               "cp_lasso_select: NULL argument");
    CP_REQUIRE(c > 0 && c <= MAXC, "cp_lasso_select: c=%d outside 1..%d", c, MAXC);
    CP_REQUIRE(ldq >= c && (ldq % 2) == 0 && (((uintptr_t)Q) & 15) == 0,
               "cp_lasso_select: Q rows must be 16-byte aligned (even ldq >= c, aligned base)");
    CP_REQUIRE(max_probes > 0 && max_iter > 0 && right0 > 0 && m > 0, "cp_lasso_select: bad parameters");
    SelectParams P{Q, ldq, qv, yn2, c, m, rank, lbound, rbound, right0, tol, max_iter, seeds, max_probes,
                   out_idxs, out_coef, out_scalars, out_probe_log};
    cudaStream_t stream = (cudaStream_t)stream_;
    if (c <= 256) return launch_select<1>(P, stream);
    if (c <= 512) return launch_select<2>(P, stream);
    if (c <= 1024) return launch_select<4>(P, stream);
    return launch_select<8>(P, stream);
}
