"""GPU: the tensor-core (split-fp16 wgmma, shifted, chunked) Gram path against an fp64 evaluation, and its effect
on the end result (weights) against the oracle.  Floating-point kernel -> tolerances, stated here:
  * Gram entries: |G_tc - G_64| <= 2e-7 * sqrt(G_ii G_jj)   (fp32-level, data-relative)
  * reconstructed weights through the full drop-in path: <= 1e-4 relative Frobenius (north_star)."""
import numpy as np
import pytest

import cases
import cp_oracle as O

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def _dev(a, eng):
    return torch.as_tensor(np.ascontiguousarray(a), device=eng.device)


@pytest.mark.parametrize("N,K,n", [(1024, 256, 128), (5000, 576, 64), (4999, 1152, 200), (2000, 200, 36), (640, 128, 8)])
def test_gram_tc_close_to_fp64(engine, N, K, n):
    r = np.random.RandomState(N + K)
    X = np.maximum(r.standard_normal((N, K)), 0).astype(np.float32)
    Y = (X[:, :min(K, 64)] @ r.standard_normal((min(K, 64), n)) + r.standard_normal((N, n))).astype(np.float32)
    bias = (0.1 * r.standard_normal(n)).astype(np.float32)
    ldy = (n + 3) // 4 * 4
    Yp = torch.zeros(N, ldy, dtype=torch.float32, device=engine.device)
    Yp[:, :n] = _dev(Y, engine)
    g = engine.gram(_dev(X, engine), Yp[:, :n], y_bias=_dev(bias, engine), mode=1)
    X64, Y64 = X.astype(np.float64), Y.astype(np.float64) - bias.astype(np.float64)
    Gr, Br = X64.T @ X64, X64.T @ Y64
    G, B = g["G"].cpu().numpy(), g["B"].cpu().numpy()
    dx = np.sqrt(np.diag(Gr))
    dy = np.sqrt((Y64 ** 2).sum(0))
    eg = np.abs(G - Gr) / np.outer(dx, dx)
    eb = np.abs(B - Br) / np.outer(dx, dy)
    print("max rel err G %.2e  B %.2e" % (eg.max(), eb.max()))
    assert eg.max() <= 1e-6 and eb.max() <= 1e-6
    # diagonal: separate fp64 pass over fl32(x - shift); what is left is the fp32 rounding of the shifted data
    assert np.abs(np.diag(G) - np.diag(Gr)).max() <= 1e-7 * np.diag(Gr).max()
    np.testing.assert_array_equal(G, G.T)
    # the sums are those of the fp32-rounded shifted data (consistent with G), not of the raw data
    np.testing.assert_allclose(g["sx"].cpu().numpy(), X64.sum(0), rtol=1e-7)
    np.testing.assert_allclose(g["sy"].cpu().numpy(), Y64.sum(0), rtol=1e-6, atol=1e-4)
    # centred Gram (what the least squares sees): error relative to its own scale
    xm = X64.mean(0)
    Gc_ref = Gr - N * np.outer(xm, xm)
    sxd = g["sx"].cpu().numpy()
    Gc = G - np.outer(sxd, sxd) / N
    dc = np.sqrt(np.diag(Gc_ref))
    ec = np.abs(Gc - Gc_ref) / np.outer(dc, dc)
    print("max rel err centred G %.2e" % ec.max())
    assert ec.max() <= 1e-6


def test_dictionary_with_tc_gram_meets_north_star_tolerance(engine):
    """c=128 -> K=1152, N=5000: full drop-in path with the tensor-core Gram vs the CPU oracle."""
    from cpb200.lib import cfgs, decompose

    X, W2, Y = cases.dictionary_inputs(c=128, n=64, N=5000, k=3, seed=55)
    rank = int(128 / 1.15)
    st = O.DictState(alpha=1e-3)
    np.random.seed(3)
    oi, oW, oB = O.dictionary(X.astype(np.float64), W2, Y, rank=rank, state=st)
    old = engine.gram_mode
    engine.gram_mode = 1
    try:
        cfgs.alpha = 1e-3
        np.random.seed(3)
        idxs, W, B = decompose.dictionary(X.astype(np.float64), W2, Y, rank=rank)
    finally:
        engine.gram_mode = old
    assert np.array_equal(idxs, oi)
    rel = np.linalg.norm(W - oW) / np.linalg.norm(oW)
    print("rel weight error with 3xTF32 Gram: %.2e" % rel)
    assert rel <= 1e-4 and np.abs(B - oB).max() <= 1e-4


@pytest.mark.parametrize("N,K,n", [(64, 64, 4), (65, 128, 1), (257, 192, 130), (8191, 256, 64), (300, 1000, 12),
                                   (20000, 256, 64)])
def test_gram_tc_edge_shapes(engine, N, K, n):
    """Row counts that are not multiples of the 32-row k-block / 128-row sub-chunk, a single sub-chunk, many
    row splits (tall-skinny: few tiles), one target column, K and n that leave partial tiles, N beyond one
    split's row cap (SURVEY 8d config 5 sweeps N up to 1e5 at this kernel)."""
    r = np.random.RandomState(7 * N + K)
    X = (r.standard_normal((N, K)) * r.uniform(0.1, 3.0, K) + r.uniform(-2, 2, K)).astype(np.float32)
    ldy = (n + 3) // 4 * 4
    Y = r.standard_normal((N, n)).astype(np.float32)
    Yp = torch.zeros(N, ldy, dtype=torch.float32, device=engine.device)
    Yp[:, :n] = _dev(Y, engine)
    g = engine.gram(_dev(X, engine), Yp[:, :n], mode=1)
    X64, Y64 = X.astype(np.float64), Y.astype(np.float64)
    Gr, Br = X64.T @ X64, X64.T @ Y64
    dx, dy = np.sqrt(np.diag(Gr)), np.sqrt((Y64 ** 2).sum(0))
    assert (np.abs(g["G"].cpu().numpy() - Gr) / np.outer(dx, dx)).max() <= 1e-6
    assert (np.abs(g["B"].cpu().numpy() - Br) / np.outer(dx, dy)).max() <= 1e-6
    np.testing.assert_array_equal(g["G"].cpu().numpy(), g["G"].cpu().numpy().T)


def test_gram_tc_single_products(engine):
    """G only and X'Y only (one launch covers both tile kinds; either may be absent)."""
    r = np.random.RandomState(11)
    N, K, n = 1500, 384, 96
    X = np.maximum(r.standard_normal((N, K)), 0).astype(np.float32)
    Y = r.standard_normal((N, n)).astype(np.float32)
    X64, Y64 = X.astype(np.float64), Y.astype(np.float64)
    g1 = engine.gram(_dev(X, engine), None, mode=1)
    assert g1["B"] is None
    np.testing.assert_allclose(g1["G"].cpu().numpy(), X64.T @ X64, rtol=0, atol=1e-6 * np.diag(X64.T @ X64).max())
    g2 = engine.gram(_dev(X, engine), _dev(Y, engine), want_G=False, mode=1)
    assert g2["G"] is None
    ref = X64.T @ Y64
    assert np.abs(g2["B"].cpu().numpy() - ref).max() <= 1e-6 * np.sqrt(np.diag(X64.T @ X64).max() * (Y64 ** 2).sum(0).max())


def test_gram_tc_is_bitwise_reproducible(engine):
    r = np.random.RandomState(5)
    X = _dev(r.standard_normal((3000, 640)).astype(np.float32), engine)
    Y = _dev(r.standard_normal((3000, 64)).astype(np.float32), engine)
    a = engine.gram(X, Y, mode=1)
    b = engine.gram(X, Y, mode=1)
    assert torch.equal(a["G"], b["G"]) and torch.equal(a["B"], b["B"])
