"""CPU: the host model of cp_gram's tensor-core mode (gram_tc_model) against exact rational arithmetic
(fractions.Fraction) at small sizes, the preconditions under which its operand preparation is exact, the column
exponent at the ends of the fp32 range, and the split policies it restates."""
from fractions import Fraction

import numpy as np
import pytest

import gram_tc_model as M

Q = 2.0 ** -12


def grid_columns(rng, N, K, mamp=2.0 ** 7, damp=2.0 ** 7):
    """Columns on the 2^-12 grid that sum to exactly N m (deviations in +-pairs), as the GPU tests build them."""
    m = np.round(rng.uniform(-mamp, mamp, K) / Q) * Q
    h = N // 2
    d = np.round(rng.uniform(-damp, damp, (h, K)) / Q) * Q
    d = rng.permuted(np.concatenate([d, -d, np.zeros((N - 2 * h, K))]), axis=0)
    return (m + d).astype(np.float32)


def F(x):
    return Fraction(float(x))


def test_numpy_fp16_conversion_rounds_to_nearest_even():
    """tc_prep's hi/lo split relies on numpy's float32 -> float16 conversion being __float2half_rn."""
    x = np.float32([2049, 2051, 1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, 2.0 ** -25, 3 * 2.0 ** -25, 65520, -2049])
    want = [2048, 2052, 1, 1 + 2.0 ** -9, 0, 2.0 ** -23, np.inf, -2048]
    with np.errstate(over="ignore"):
        assert np.array_equal(x.astype(np.float16).astype(np.float64), want)


@pytest.mark.parametrize("N,K", [(70, 5), (65, 3), (9, 4)])
def test_prep_is_exact_on_grid_data(N, K):
    rng = np.random.default_rng(N * K)
    X = grid_columns(rng, N, K)
    m = M.exact_sum_preconditions(X, Q, 2.0 ** 8)
    p = M.tc_prep(X)
    for j in range(K):
        col = [F(x) for x in X[:, j]]
        assert F(p["t"][j]) == sum(col)
        assert F(p["shift"][j]) == sum(col) / N == F(m[j])
        xs = [c - F(p["shift"][j]) for c in col]
        assert [F(x) for x in p["xs"][:, j]] == xs
        assert F(p["T"][j]) == sum(xs) == 0
        assert F(p["SQ"][j]) == sum(x * x for x in xs)
        s = Fraction(2) ** int(p["e"][j])
        assert [F(v) for v in p["v"][:, j]] == [x * s for x in xs]
        # 22 bits: hi + lo is v exactly, and |v| <= 2 max|x| 2^e < 2^10
        assert [F(h) + F(lo) for h, lo in zip(p["hi"][:, j], p["lo"][:, j])] == [x * s for x in xs]
        assert max(abs(x * s) for x in xs) <= 2 * F(p["mx"][j]) * s < 2 ** 10


def test_exact_preconditions_reject_bad_data():
    rng = np.random.default_rng(3)
    X = grid_columns(rng, 40, 3)
    M.exact_sum_preconditions(X, Q, 2.0 ** 8)
    off = X.copy()
    off[0, 1] += np.float32(2.0 ** -14)
    with pytest.raises(AssertionError):
        M.exact_sum_preconditions(off, Q, 2.0 ** 8)
    moved = X.copy()
    moved[0, 2] += np.float32(Q)
    with pytest.raises(AssertionError):
        M.exact_sum_preconditions(moved, Q, 2.0 ** 8)
    with pytest.raises(AssertionError):
        M.exact_sum_preconditions(X * 4, Q, 2.0 ** 8)


@pytest.mark.parametrize("seed", [0, 1])
def test_model_formula_against_fractions(seed):
    """tc_model's value is reduce_tc2's formula on the emulated operands: the exact inv_i inv_j (hi'hi + hi'lo + lo'hi)
    + s T' + T s' + N s u' (diagonal: SQ + 2 s T + N s^2), within (N + 16) 2^-53 of its magnitudes; and the exact
    X'(Y - b) lies within the model's split bound of it."""
    rng = np.random.default_rng(seed)
    N, K, n = 67, 4, 3
    X = grid_columns(rng, N, K)
    Y = grid_columns(rng, N, n)
    X[:, 2] = np.float32(rng.standard_normal(N))  # one unstructured column: T != 0, lo and the x - s rounding live
    yb = np.float32(rng.standard_normal(n))
    px, py = M.tc_prep(X), M.tc_prep(Y)
    mod = M.tc_model(px, py, yb)
    g = (N + 16) * M.U64
    for key, pa, pb, bias in (("G", px, px, None), ("B", px, py, yb)):
        blk = mod[key]
        for i in range(pa["hi"].shape[1]):
            for j in range(pb["hi"].shape[1]):
                ha, la = [F(v) for v in pa["hi"][:, i]], [F(v) for v in pa["lo"][:, i]]
                hb, lb = [F(v) for v in pb["hi"][:, j]], [F(v) for v in pb["lo"][:, j]]
                P = sum(a * b + a * d + c * b for a, b, c, d in zip(ha, hb, la, lb))
                sa, sb = F(pa["shift"][i]), F(pb["shift"][j])
                ub = sb - (F(bias[j]) if bias is not None else 0)
                Ta = sum(F(x) for x in pa["xs"][:, i])
                Tb = sum(F(x) for x in pb["xs"][:, j])
                if key == "G" and i == j:
                    exact_model = sum(F(x) ** 2 for x in pa["xs"][:, i]) + 2 * sa * Ta + N * sa * sa
                else:
                    exact_model = P * F(pa["inv"][i]) * F(pb["inv"][j]) + sa * Tb + Ta * ub + N * sa * ub
                mag = blk["scale"][i, j] * blk["A"][i, j] + blk["undo"][i, j]
                assert abs(F(blk["val"][i, j]) - exact_model) <= F(g * mag)
                truth = sum(F(x) * (F(y) - (F(bias[j]) if bias is not None else 0))
                            for x, y in zip(pa["cols"][:, i], pb["cols"][:, j]))
                assert abs(truth - exact_model) <= F(blk["split"][i, j]) * Fraction(1000001, 1000000)


def test_col_exponent_over_the_fp32_range():
    """Fixed exponent: 2^e is a normal fp32, |v| <= 2 max|x| 2^e < 2^10, and e equals the old exponent wherever that
    was inside its clamp; the old exponent broke above 2^116 (too small a scale) and from 2^127 (2 max|x| overflows)."""
    k = np.arange(-149, 128)
    mx = np.concatenate([np.ldexp(np.float32(1), k), np.ldexp(np.float32(1.9990234), k[k > -140])]).astype(np.float32)
    mx = np.concatenate([mx, np.float32([np.finfo(np.float32).max])])
    e = M.col_exponent(mx)
    assert e.min() >= -126 and e.max() <= 127
    v = 2 * mx.astype(np.float64) * np.exp2(e)
    assert v.max() < 2 ** 10
    big = mx >= 2.0 ** -119
    assert np.all(v[big] >= 2 ** 9)
    old = M.col_exponent(mx, clamp="old")
    inside = (np.abs(old) < 100) & np.isfinite(2 * mx.astype(np.float64)) & (2 * mx.astype(np.float64) < 2.0 ** 128)
    assert np.array_equal(e[inside], old[inside])
    assert np.all(old[mx >= 2.0 ** 127] == 0)
    assert np.all(2 * mx[mx > 2.0 ** 117].astype(np.float64) * np.exp2(old[mx > 2.0 ** 117]) >= 2 ** 16)


@pytest.mark.parametrize("k", [-114, 0, 115, 120])
def test_old_clamp_loses_bits_and_the_fixed_one_does_not(k):
    """Emulated on a grid column scaled by 2^k: the fixed exponent keeps all of v in hi + lo at every scale; the old
    clamp drops bits into fp16 subnormals at 2^-114 and overflows fp16 at 2^115 and 2^120."""
    rng = np.random.default_rng(11)
    X = np.ldexp(grid_columns(rng, 200, 2, mamp=2.0, damp=4.0), k).astype(np.float32)
    for clamp in ("fixed", "old"):
        p = M.tc_prep(X, clamp=clamp)
        v = p["xs"].astype(np.float64) * np.exp2(p["e"])
        with np.errstate(invalid="ignore"):
            kept = np.array_equal(p["hi"].astype(np.float64) + p["lo"].astype(np.float64), v)
        assert kept == (clamp == "fixed" or k == 0), (clamp, k)


def test_product_plan_restates_the_split_policy():
    p = M.product_plan(640, 640, 20007, True, 132)
    assert (p["tiles"], p["nsplit"], p["rps"]) == (15, 18, 1120)
    assert {"sym:split-cap-tiles", "sym:mirror", "reduction-tail", "register-staged"} <= p["branches"]
    p = M.product_plan(129, 129, 5000, True, 132)
    assert (p["nsplit"], p["rps"]) == (79, 64) and "sym:split-cap-rows" in p["branches"]
    assert M.product_plan(300, 300, 50, True, 132)["nsplit"] == 1
    assert "async64" in M.product_plan(300, 200, 78, False, 132, 128, True)["branches"]
    assert "async128" in M.product_plan(1536, 1536, 100, False, 132, 128, True)["branches"]
    assert "all:split" in M.product_plan(200, 150, 5003, False, 132, 128, True)["branches"]
    for R in range(1, 3000, 37):
        for K in (64, 129, 640, 3000):
            p = M.product_plan(K, K, R, True, 132)
            assert p["rps"] % M.BK == 0 or p["nsplit"] == 1
            assert p["nsplit"] * p["rps"] >= R > (p["nsplit"] - 1) * p["rps"]


def test_tc_plan_restates_the_split_policy():
    for N in (64, 65, 127, 4095, 4096, 4097, 12289, 50000, 100000):
        for K, n in ((64, 1), (257, 129), (2304, 200)):
            p = M.tc_plan(N, K, n, True, True, 132)
            assert p["rps"] % M.KS == 0 and p["rps"] <= M.MAX_SPLIT_ROWS
            assert p["nsplit"] * p["rps"] >= N > (p["nsplit"] - 1) * p["rps"]
            assert M.tau(p["nst"]) <= 112 * 2.0 ** -24
    assert M.tc_plan(64, 64, 1, True, True, 132)["nitems"] == 2
    assert "tc:G-null" in M.tc_plan(4096, 1000, 129, False, True, 132)["branches"]
    assert M.tc_routes(1000, 128, 128, True, "f32", 20, 20, True, False, True, True, False)
    assert not M.tc_routes(1000, 128, 128, True, "f32", 20, 20, True, False, True, True, True)
    assert not M.tc_routes(1000, 128, 128, True, "f32", 20, 20, True, False, False, True, False)
    assert M.tc_routes(1000, 128, 128, True, "f32", 20, 21, False, False, False, False, False)
