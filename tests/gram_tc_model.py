"""Host models of cp_gram (csrc/gram.cu, csrc/gram_tc2.cu) and of the fp64 product driver (cpgemm::product in
csrc/gemm_f64.cuh), for the statistics tests.

* product_plan / tc_plan restate the split policies of the two arithmetic modes, so that a test can say which branch a
  shape reaches (split or not and why, mirror, kernel, tile walk) and assert that its parametrisation reaches all of them.
* tc_prep emulates the tensor-core mode's operand preparation bit for bit: the fp32 shift fl32(t * (1/N)), the column
  exponent e, xs = fl32(x - s), v = fl32(xs 2^e), hi = fp16_rn(v), lo = fp16_rn(fl32(v - hi)), and the fp64 column
  sums T and squares SQ of xs.  It is exact when every fp64 column sum (of x and of xs) is exact, which
  exact_sum_preconditions checks.
* tc_model puts the prepared operands through reduce_tc2's fp64 formula, with the three products hi'hi + hi'lo + lo'hi
  taken exactly up to the float64 BLAS used for them; it returns the statistics the tensor-core mode would give with an
  exact accumulation, the magnitudes its error bound is built from, and a bound on the modelled arithmetic's own
  distance from X'X (the 22-bit split and the fp32 rounding of x - s).
"""
import numpy as np

BM = 128          # fp64 product tile edge (cpgemm::BM = BN)
BK = 16           # fp64 product reduction stage
KS = 64           # tensor-core stage (rows of one wgmma accumulator run)
TILE = 128        # tensor-core output tile edge
RS = 32           # row splits of the tensor-core statistics passes
MAX_SPLIT_ROWS = 4096
U64 = 2.0 ** -53


def cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------ fp64 products (cpgemm::product)
def num_tiles(M, Nn, sym, T=BM):
    tm, tn = cdiv(M, T), cdiv(Nn, T)
    return tn * (tn + 1) // 2 if sym else tm * tn


def product_plan(M, Nn, R, sym, sms, min_split_r=0, async_operands=False):
    """The split, tile set and kernel cpgemm::product picks.  async_operands: plain fp64 operands of cp_gemm_f64 with
    an r-contiguous A, 16-byte aligned, even leading dimensions (what launch() requires of gemm_async_kernel)."""
    tiles = num_tiles(M, Nn, sym)
    target = 2 * sms
    nsplit, rps, br = 1, R, set()
    tag = "sym" if sym else "all"
    if tiles < target and R > 0 and R >= min_split_r:
        ns = cdiv(target, tiles)
        max_by_rows = cdiv(R, 4 * BK)
        cap = "tiles"
        if ns > max_by_rows:
            ns, cap = max_by_rows, "rows"
        rps = cdiv(cdiv(R, ns), BK) * BK
        nsplit = cdiv(R, rps)
        br.add("%s:split-cap-%s" % (tag, cap) if nsplit > 1 else "%s:unsplit-short-R" % tag)
    elif R > 0:
        br.add("%s:unsplit-%s" % (tag, "tiles" if tiles >= target else "min-split-r"))
    if R > 0:
        br.add("%s:%s" % (tag, "split" if nsplit > 1 else "unsplit"))
        if R % BK:
            br.add("reduction-tail")
        if nsplit == 1 and async_operands:
            br.add("async%d" % (128 if tiles >= sms else 64))
        else:
            br.add("register-staged")
    if sym and M > BM:
        br.add("sym:mirror")
    return dict(nsplit=nsplit, rps=rps, tiles=tiles, branches=br)


# ------------------------------------------------------------------ tensor-core mode (cp_gram_tc2)
def tc_eligible(N, K, ldx, x_aligned, y_dtype, n, ldy, y_aligned, rows, want_y):
    """cp_gram_tc_eligible"""
    if rows or N < 64 or K < 64 or not x_aligned or ldx % 4:
        return False
    if want_y and (y_dtype != "f32" or not y_aligned or ldy % 4 or n < 1):
        return False
    return True


def tc_routes(N, K, ldx, x_aligned, y_dtype, n, ldy, y_aligned, rows, want_B, want_sy, want_yy):
    """True when a mode-1 cp_gram call with these arguments runs the tensor-core pipeline (R > 0)."""
    if want_yy or not tc_eligible(N, K, ldx, x_aligned, y_dtype, n, ldy, y_aligned, rows, want_B or want_sy):
        return False
    return not (want_sy and not want_B)


def tc_plan(N, K, n, want_G, want_B, sms, y_bias=False):
    """Row splits, items and grid of cp_gram_tc2, and the branches of gram_tc2_kernel / reduce_tc2 / tc2_prep the
    call reaches."""
    tjx = cdiv(K, TILE)
    tnb = cdiv(n, TILE) if want_B else 0
    tiles_sym = tjx * (tjx + 1) // 2 if want_G else 0
    ntiles = tiles_sym + tjx * tnb
    SUB = KS
    ns_min = cdiv(N, MAX_SPLIT_ROWS)
    nsplit, rps = ns_min, cdiv(cdiv(N, ns_min), SUB) * SUB
    if ntiles > 0:
        best = 1e300
        max_ns = cdiv(N, SUB)
        for ns in range(ns_min, min(max_ns, ns_min + 31) + 1):
            r = cdiv(cdiv(N, ns), SUB) * SUB
            ns_eff = cdiv(N, r)
            rounds = float(cdiv(ntiles * ns_eff, sms))
            cost = rounds * (1.2 * float(r // KS) + 1.0) + float(ns_eff) * (2.0 * ntiles * TILE * TILE * 4.0 / 3.0e6)
            if cost < best * 0.98:
                best, nsplit, rps = cost, ns_eff, r
    Np = cdiv(N, KS) * KS
    ntile_rows = Np // 64
    tiles_per_split = cdiv(ntile_rows, RS)
    nitems = ntiles * nsplit
    br = {"tc"}
    if want_G:
        br.add("tc:diag-tile")
        if tjx > 1:
            br.add("tc:offdiag-tile")
    if want_B:
        br.add("tc:y-tile")
        if not want_G:
            br.add("tc:G-null")
        if n % TILE:
            br.add("tc:y-tile-partial")
        if y_bias:
            br.add("tc:y-bias")
    if K % TILE:
        br.add("tc:row-tile-partial")
    if N % KS:
        br.add("tc:stage-padded")
    br.add("tc:split" if nsplit > 1 else "tc:unsplit")
    if ns_min > 1:
        br.add("tc:split-cap-4096")
    if tiles_per_split > 1:
        br.add("tc:prep-multi-tile")
    if cdiv(ntile_rows, tiles_per_split) == RS:
        br.add("tc:prep-32-splits")
    if nitems < sms:
        br.add("tc:grid-below-sms")
    if nitems > sms:
        br.add("tc:items-per-cta>1")
        if want_G and tjx > 1:
            br.add("tc:mixed-diag-offdiag-per-cta")
    return dict(nsplit=nsplit, rps=rps, nst=rps // KS, ntiles=ntiles, nitems=nitems, branches=br)


def tau(nst):
    """Relative accumulation error of one fp32 partial of the tensor-core mode, against A (the sum of the absolute
    products):  12 truncating wgmma adds per stage, each within 2 ulp (2^-22) of the sum of the absolute values it
    adds, then nst round-to-nearest adds of the stage results into the split sum, each within 2^-24 of the absolute
    sum so far.  With splits of at most 4096 rows (nst <= 64): (48 + 64) 2^-24 ~ 2^-17.2."""
    return (12 * 4 + nst) * 2.0 ** -24


def col_exponent(mx, clamp="fixed"):
    """colstat_finish's column exponent e (2^e scales the shifted column) from the fp32 column maxima mx.
    clamp="fixed": e = 8 - ilogb(mx) in [-126, 127];  clamp="old": e = 9 - ilogb(fl32(2 mx)) in [-100, 100]."""
    mx = np.asarray(mx, dtype=np.float32)
    e = np.zeros(mx.shape, dtype=np.int64)
    if clamp == "fixed":
        ok = (mx > 0) & np.isfinite(mx)
        e[ok] = np.clip(8 - (np.frexp(mx[ok])[1] - 1), -126, 127)
    else:
        with np.errstate(over="ignore"):
            b = (np.float32(2) * mx).astype(np.float32)
        ok = (b > 0) & np.isfinite(b)
        e[ok] = np.clip(9 - (np.frexp(b[ok])[1] - 1), -100, 100)
    return e


def tc_prep(cols, clamp="fixed"):
    """Bit-exact model of colstat_part/colstat_finish/tc2_prep/tc2_stat_finish for the fp32 columns cols (N x m),
    provided the fp64 column sums of cols and of xs are exact (any summation order then gives the same bits)."""
    cols = np.asarray(cols, dtype=np.float32)
    N = cols.shape[0]
    t = cols.astype(np.float64).sum(0)
    shift = (t * (1.0 / N)).astype(np.float32)
    mx = np.abs(cols).max(0) if N else np.zeros(cols.shape[1], np.float32)
    e = col_exponent(mx, clamp)
    scale = np.ldexp(np.float32(1), e).astype(np.float32)
    xs = cols - shift
    with np.errstate(over="ignore", under="ignore"):
        v = xs * scale
        hi = v.astype(np.float16)
        lo = (v - hi.astype(np.float32)).astype(np.float16)
    x64 = xs.astype(np.float64)
    return dict(N=N, cols=cols, t=t, shift=shift, mx=mx, e=e, scale=scale, inv=np.ldexp(1.0, -e), xs=xs, v=v, hi=hi,
                lo=lo, T=x64.sum(0), SQ=(x64 * x64).sum(0), Tabs=np.abs(x64).sum(0))


def exact_sum_preconditions(cols, quantum, bound):
    """The data conditions under which tc_prep is exact: entries on the grid `quantum` (a power of two) with
    |x| < bound and N bound / quantum < 2^53 (every fp64 partial sum of x, or of x - m, is exact in any order), and
    every column summing to N m with m an fp32 value on the grid, so that the shift is m, xs = x - m is exact and on
    the grid, and T = 0.  Returns the column means m."""
    cols = np.asarray(cols, dtype=np.float64)
    N = cols.shape[0]
    q = cols / quantum
    assert np.array_equal(q, np.round(q)), "entries off the grid"
    assert np.abs(cols).max(initial=0) < bound and N * bound / quantum < 2.0 ** 53
    m = cols.sum(0) / N
    assert np.array_equal(m / quantum, np.round(m / quantum)), "column sums are not N m with m on the grid"
    assert np.array_equal(m.astype(np.float32).astype(np.float64), m)
    return m


def _abs_mm(mm, a, b):
    return mm(np.abs(a), np.abs(b))


def tc_model(px, py=None, y_bias=None, mm=None, want_G=True, with_split=True):
    """reduce_tc2 and tc2_stat_finish on the emulated operands of tc_prep (px for X, py for Y).  mm(a, b) = a' b in
    float64.  Returns dict with the modelled G / B / sx / sy, and per element:
      A        sum_r |hi_i hi_j| + |hi_i lo_j| + |lo_i hi_j|  (the magnitudes the tensor cores accumulate)
      scale    inv_i inv_j (A is in the scaled operand units)
      undo     |s_i| Tabs_j + Tabs_i |u_j| + N |s_i u_j|  (magnitudes of the fp64 shift undo)
      split    bound on |model - exact product| from the 22-bit split and from the fp32 rounding of x - s
               (with_split only)."""
    mm = mm or (lambda a, b: a.T @ b)
    N = px["N"]
    out = {}

    def f64(h):
        return h.astype(np.float64)

    def block(pa, pb, ub, diag):
        ha, la, hb, lb = f64(pa["hi"]), f64(pa["lo"]), f64(pb["hi"]), f64(pb["lo"])
        P = mm(ha, hb) + mm(ha, lb) + mm(la, hb)
        sc = np.outer(pa["inv"], pb["inv"])
        ua = pa["shift"].astype(np.float64)
        val = P * sc + (np.outer(ua, pb["T"]) + np.outer(pa["T"], ub) + N * np.outer(ua, ub))
        A = _abs_mm(mm, ha, hb) + _abs_mm(mm, ha, lb) + _abs_mm(mm, la, hb)
        undo = np.outer(np.abs(ua), pb["Tabs"]) + np.outer(pa["Tabs"], np.abs(ub)) + N * np.abs(np.outer(ua, ub))
        if diag:
            d = np.arange(val.shape[0])
            val[d, d] = pa["SQ"] + (ua * pa["T"] + pa["T"] * ua + N * ua * ua)
        if not with_split:
            return dict(val=val, A=A, scale=sc, undo=undo)
        # model error against the exact X'(Y - b): x = s + xs + dx, v = hi + lo + r
        va, vb = f64(pa["v"]), f64(pb["v"])
        ra, rb = va - ha - la, vb - hb - lb
        dxa = pa["cols"].astype(np.float64) - ua - pa["xs"].astype(np.float64)
        dxb = pb["cols"].astype(np.float64) - pb["shift"].astype(np.float64) - pb["xs"].astype(np.float64)
        xa, xb = pa["xs"].astype(np.float64), pb["xs"].astype(np.float64)
        split = sc * (_abs_mm(mm, la, lb) + _abs_mm(mm, ha + la, rb) + _abs_mm(mm, ra, vb))
        split += np.outer(np.abs(ua), np.abs(dxb).sum(0)) + np.outer(np.abs(dxa).sum(0), np.abs(ub))
        split += _abs_mm(mm, xa, dxb) + _abs_mm(mm, dxa, xb) + _abs_mm(mm, dxa, dxb)
        return dict(val=val, A=A, scale=sc, undo=undo, split=split)

    sx = px["T"] + N * px["shift"].astype(np.float64)
    out["sx"] = dict(val=sx, mag=px["Tabs"] + N * np.abs(px["shift"].astype(np.float64)))
    if want_G:
        out["G"] = block(px, px, px["shift"].astype(np.float64), True)
    if py is not None:
        ub = py["shift"].astype(np.float64) - (y_bias.astype(np.float64) if y_bias is not None else 0.0)
        out["B"] = block(px, py, ub, False)
        out["sy"] = dict(val=py["T"] + N * ub, mag=py["Tabs"] + N * np.abs(ub))
    return out


def tc_bound(blk, nst, N, diag=False, SQ=None):
    """|statistic - model| bound of one G or B block: tau(nst) inv_i inv_j A_ij for the tensor-core accumulation,
    plus (N + 16) 2^-53 of every fp64 magnitude (the model's own BLAS sums, the pipeline's fp64 split sums, the shift
    undo and its possible fused multiply-adds).  diag: G's diagonal comes from the fp64 squares SQ instead."""
    g = (N + 16) * U64
    b = tau(nst) * blk["scale"] * blk["A"] + g * (blk["scale"] * blk["A"] + blk["undo"])
    if diag:
        d = np.arange(b.shape[0])
        b[d, d] = g * (SQ + blk["undo"][d, d])
    return b
