"""GPU: each libcpb200 entry point (called through the C ABI via cffi) against the oracle /
numpy on identical seeded inputs."""
import ctypes
import os

import numpy as np
import pytest

import cases
import cp_oracle as O

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def _dev(a, eng, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(a), device=eng.device)
    return t if dtype is None else t.to(dtype)


def _forward_from(images, specs, weights, biases):
    from make_golden import conv2d_numpy

    cache = {}

    def forward(batch):
        if batch not in cache:
            blobs = {"data": images[batch % len(images)]}
            for s in specs:
                y = conv2d_numpy(blobs[s["bottom"]], weights[s["name"]], biases[s["name"]], s["pad"], s["stride"])
                blobs[s["name"]] = y
                blobs[s["name"] + "_relu"] = np.maximum(y, 0)
            cache[batch] = blobs
        return cache[batch]

    return forward


# ---------------------------------------------------------------------------- gathers (bit exact)
@pytest.mark.parametrize("name", list(cases.NET_CASES))
@pytest.mark.parametrize("layout", ["nchw", "nhwc"])
def test_gathers_bit_exact_vs_reference_golden(engine, golden_dir, name, layout):
    spec = cases.NET_CASES[name]
    g = np.load(os.path.join(golden_dir, "net_%s.npz" % name))
    images, specs, weights, biases = cases.net_inputs(**spec["gen"])
    forward = _forward_from(images, specs, weights, biases)
    nB, P = spec["nBatches"], spec["P"]
    s2 = specs[1]
    k = s2["k"]
    B = images[0].shape[0]
    blobs_x = np.concatenate([forward(b)["conv1"] for b in range(nB)], 0)  # (nB*B, c, H, W)
    blobs_y = np.concatenate([forward(b)["conv2"] for b in range(nB)], 0)
    rx = np.stack([g["randx_conv2_%d" % b] for b in range(nB)]).astype(np.int32)
    ry = np.stack([g["randy_conv2_%d" % b] for b in range(nB)]).astype(np.int32)

    def lay(a):
        return np.ascontiguousarray(a.transpose(0, 2, 3, 1)) if layout == "nhwc" else a

    X = engine.patch_gather(_dev(lay(blobs_x), engine), _dev(rx, engine), _dev(ry, engine), B, P, k, s2["pad"],
                            s2["stride"], relu=False, layout=layout)
    N = nB * P * B
    c = blobs_x.shape[1]
    got = X.view(N, c, k * k).permute(0, 2, 1).reshape(N * k * k, c).cpu().numpy().astype(np.float64)
    np.testing.assert_array_equal(got, g["XY"])  # reference extract_XY, bit exact
    Xr = engine.patch_gather(_dev(lay(blobs_x), engine), _dev(rx, engine), _dev(ry, engine), B, P, k, s2["pad"],
                             s2["stride"], relu=True, layout=layout)
    np.testing.assert_array_equal(Xr.cpu().numpy(), np.maximum(X.cpu().numpy(), 0))
    Yf = engine.point_gather(_dev(lay(blobs_y), engine), _dev(rx, engine), _dev(ry, engine), B, P, layout=layout)
    np.testing.assert_array_equal(Yf.cpu().numpy().astype(np.float64), g["feats_conv2"])


@pytest.mark.parametrize("c,k,pad,stride,H", [(16, 3, 1, 1, 9), (64, 3, 1, 1, 14), (384, 3, 1, 2, 13), (512, 3, 1, 1, 7),
                                              (1024, 1, 0, 1, 6), (96, 5, 2, 1, 8), (2048, 1, 0, 2, 7), (256, 3, 0, 1, 10)])
def test_tma_gather_is_bit_identical_to_the_nchw_kernel(engine, c, k, pad, stride, H):
    """The NHWC TMA path (whole windows by cp.async.bulk.tensor, zero fill for the padding taps, bulk row stores)
    against the SIMT NCHW kernel that the reference goldens pin: every corner and border point is sampled."""
    g = torch.Generator(device=engine.device)
    g.manual_seed(c * 7 + k)
    B, nb = 3, 4
    fm = torch.randn((nb * B, c, H, H), generator=g, device=engine.device)
    Ho = (H + 2 * pad - k) // stride + 1
    pts = [(0, 0), (0, Ho - 1), (Ho - 1, 0), (Ho - 1, Ho - 1), (Ho // 2, Ho // 2), (1 % Ho, Ho - 1), (Ho - 1, 1 % Ho)]
    P = len(pts)
    rx = torch.tensor([[p[0] for p in pts]] * nb, dtype=torch.int32, device=engine.device)
    ry = torch.tensor([[p[1] for p in pts]] * nb, dtype=torch.int32, device=engine.device)
    rx[1] = rx[1].flip(0)
    fm_l = fm.permute(0, 2, 3, 1).contiguous()
    for relu in (False, True):
        want = engine.patch_gather(fm, rx, ry, B, P, k, pad, stride, relu=relu, layout="nchw")
        got = engine.patch_gather(fm_l, rx, ry, B, P, k, pad, stride, relu=relu, layout="nhwc")
        assert torch.equal(want, got)
    # rows with a leading dimension larger than K (X riding in a wider buffer)
    K = c * k * k
    wide = torch.full((nb * P * B, K + 8), -7.0, device=engine.device)
    engine.patch_gather(fm_l, rx, ry, B, P, k, pad, stride, relu=True, layout="nhwc", out=wide[:, :K])
    assert torch.equal(wide[:, :K], want) and bool((wide[:, K:] == -7.0).all())


def test_gather_rejects_bad_arguments(engine):
    import cpb200

    f = torch.zeros(2, 3, 5, 5, device=engine.device)
    r = torch.zeros(1, 2, dtype=torch.int32, device=engine.device)
    with pytest.raises(cpb200._cabi.CpError):
        engine.patch_gather(f, r, r, 2, 2, 4, 1, 1)  # even kernel size (reference asserts odd, net.py:604)


# ---------------------------------------------------------------------------- Gram statistics
@pytest.mark.parametrize("N,K,n", [(600, 288, 16), (1000, 27, 8), (777, 130, 33), (5000, 576, 64)])
def test_gram_fp64_matches_numpy(engine, N, K, n):
    r = np.random.RandomState(N + K)
    X = np.maximum(r.standard_normal((N, K)), 0).astype(np.float32)
    Y = r.standard_normal((N, n)).astype(np.float32)
    bias = (0.1 * r.standard_normal(n)).astype(np.float32)
    g = engine.gram(_dev(X, engine), _dev(Y, engine), y_bias=_dev(bias, engine), want_yy=True, mode=0)
    X64, Y64 = X.astype(np.float64), Y.astype(np.float64) - bias.astype(np.float64)
    G = g["G"].cpu().numpy()
    np.testing.assert_allclose(G, X64.T @ X64, rtol=1e-12, atol=1e-9)
    np.testing.assert_array_equal(G, G.T)
    np.testing.assert_allclose(g["B"].cpu().numpy(), X64.T @ Y64, rtol=1e-11, atol=1e-9)
    np.testing.assert_allclose(g["sx"].cpu().numpy(), X64.sum(0), rtol=1e-12)
    np.testing.assert_allclose(g["sy"].cpu().numpy(), Y64.sum(0), rtol=1e-11, atol=1e-10)
    np.testing.assert_allclose(g["yy"].cpu().numpy()[0], (Y64 ** 2).sum(), rtol=1e-12)


def test_gram_row_subset_with_repeats_and_f64_targets(engine):
    r = np.random.RandomState(5)
    N, K, n = 900, 96, 12
    X = r.standard_normal((N, K)).astype(np.float32)
    Y = r.standard_normal((N, n))  # genuine float64 targets
    rows = r.randint(0, N, 45).astype(np.int32)
    rows[3] = rows[7]  # with replacement (lib/decompose.py:425)
    g = engine.gram(_dev(X, engine), _dev(Y, engine), rows=_dev(rows, engine), want_yy=True, mode=0)
    Xs, Ys = X[rows].astype(np.float64), Y[rows]
    np.testing.assert_allclose(g["G"].cpu().numpy(), Xs.T @ Xs, rtol=1e-12, atol=1e-10)
    np.testing.assert_allclose(g["B"].cpu().numpy(), Xs.T @ Ys, rtol=1e-11, atol=1e-10)
    np.testing.assert_allclose(g["yy"].cpu().numpy()[0], (Ys ** 2).sum(), rtol=1e-12)


def test_gram_empty_and_ragged(engine):
    X = torch.zeros(0, 40, device=engine.device)
    g = engine.gram(X, None, want_B=False, mode=0)
    assert float(g["G"].abs().max()) == 0.0 and float(g["sx"].abs().max()) == 0.0
    # unaligned leading dimension (K=27 like conv1_1) through a strided view
    r = np.random.RandomState(1)
    big = _dev(r.standard_normal((300, 31)).astype(np.float32), engine)
    Xv = big[:, 2:29]
    g = engine.gram(Xv, None, want_B=False, mode=0)
    X64 = Xv.cpu().numpy().astype(np.float64)
    np.testing.assert_allclose(g["G"].cpu().numpy(), X64.T @ X64, rtol=1e-12, atol=1e-10)


# ---------------------------------------------------------------------------- LASSO
def _lasso_problem(c, n, N, k, seed):
    X, W2, Y = cases.dictionary_inputs(c=c, n=n, N=N, k=k, seed=seed)
    S = min(400, N // 20)
    samples = np.random.RandomState(seed + 1).randint(0, N, S)
    reX = np.rollaxis(X.reshape((N, c, -1))[samples], 1, 0).astype(np.float64)
    reW2 = np.transpose(W2.reshape((n, c, -1)), [1, 2, 0]).astype(np.float64)
    Z = np.matmul(reX, reW2).reshape((c, -1)).T
    y = Y[samples].reshape(-1)
    return X, W2, Y, samples, Z, y


@pytest.mark.parametrize("c,n,N,k", [(32, 16, 600, 3), (96, 32, 800, 1), (130, 24, 1000, 3)])
def test_lasso_build_matches_centred_design(engine, c, n, N, k):
    X, W2, Y, samples, Z, y = _lasso_problem(c, n, N, k, 40 + c)
    Xd = _dev(X.reshape(N, -1), engine)
    Yd = _dev(Y.astype(np.float32), engine)
    W2m = _dev(W2.reshape(n, -1), engine)
    sd = _dev(samples.astype(np.int32), engine)
    gs = engine.gram(Xd, Yd, rows=sd, want_yy=True, mode=0)
    gw = engine.gram(W2m, None, want_B=False, mode=0)
    Q, qv, yn2 = engine.lasso_build(gs, gw, W2m, c, k * k, len(samples))
    Zc = Z - Z.mean(0)
    yc = y - y.mean()
    scale = np.abs(Zc.T @ Zc).max()
    np.testing.assert_allclose(Q.cpu().numpy(), Zc.T @ Zc, rtol=0, atol=1e-11 * scale)
    np.testing.assert_allclose(qv.cpu().numpy(), Zc.T @ yc, rtol=0, atol=1e-11 * np.abs(Zc.T @ yc).max())
    np.testing.assert_allclose(yn2.cpu().numpy()[0], yc @ yc, rtol=1e-11)


@pytest.mark.parametrize("c,n,N,k,rank", [(32, 16, 600, 3, 27), (96, 32, 800, 1, 83), (131, 24, 1000, 3, 113),
                                           (300, 24, 1000, 3, 260), (600, 8, 2000, 1, 520), (1100, 16, 3000, 1, 950)])
def test_lasso_select_bit_exact_vs_gram_model(engine, c, n, N, k, rank):
    """Device alpha search == oracle/cd_oracle.c:cp_enet_cd_gram driven by the same search loop,
    fed the device-built (Q, q, |y|^2): identical probes, iteration counts, coefficients (bitwise)."""
    X, W2, Y, samples, Z, y = _lasso_problem(c, n, N, k, 70 + c)
    Zc = Z - Z.mean(0)
    yc = y - y.mean()
    Q = np.ascontiguousarray(Zc.T @ Zc)
    q = np.ascontiguousarray(Zc.T @ yc)
    yn2 = float(yc @ yc)
    m = float(Z.shape[0])
    seeds = np.random.RandomState(9).randint(0, 2147483647, size=64)
    res = engine.lasso_select(_dev(Q, engine), _dev(q, engine), _dev(np.array([yn2]), engine), m, rank, rank,
                              rank + 0.1 * rank, 1e-3, seeds)
    scal = res.scalars.cpu().numpy()
    nprobe = int(scal[1])
    assert int(scal[2]) == 0
    plog = res.probe_log[:nprobe].cpu().numpy()
    # model: same search, C Gram-form CD
    lib = O._clib()
    w = np.zeros(c)
    Qw = np.zeros(c)  # carried between fits, like the kernel
    gap, tol_s = ctypes.c_double(), ctypes.c_double()
    probes = []

    def solve(a):
        it = lib.cp_enet_cd_gram(O._dp(w), O._dp(Qw), a * m, O._dp(Q), c, O._dp(q), yn2, c, 1000, 1e-4,
                                 int(seeds[len(probes)]), 1, 1, ctypes.byref(gap), ctypes.byref(tol_s))
        nnz = int(np.count_nonzero(w))
        probes.append((a, nnz, it, gap.value))
        return nnz

    left, right = 0.0, 1e-3
    while True:
        if solve(right) < rank:
            break
        right *= 2
    while True:
        alpha = (left + right) / 2
        t = solve(alpha)
        if t > rank + 0.1 * rank:
            left = alpha
        elif t < rank:
            right = alpha
        else:
            break
    assert nprobe == len(probes)
    np.testing.assert_array_equal(plog[:, 0], [p[0] for p in probes])  # alphas
    np.testing.assert_array_equal(plog[:, 1], [p[1] for p in probes])  # nnz
    np.testing.assert_array_equal(plog[:, 2], [p[2] for p in probes])  # CD sweeps
    np.testing.assert_array_equal(res.coef.cpu().numpy(), w)  # bitwise
    np.testing.assert_array_equal(plog[:, 3], [p[3] for p in probes])  # duality gaps, bitwise
    assert scal[0] == alpha and int(scal[3]) == probes[-1][1]
    np.testing.assert_array_equal(res.idxs.cpu().numpy().astype(bool), w != 0)


def test_lasso_select_probe_cap_reports_status(engine):
    c = 16
    Q = np.eye(c)
    q = np.linspace(1, 2, c)
    seeds = np.arange(1, 5)
    # window that cannot be hit: nnz jumps across it -> cap
    res = engine.lasso_select(_dev(Q, engine), _dev(q, engine), _dev(np.array([float(q @ q)]), engine), 1.0, 8, 8.2,
                              8.4, 1e-3, seeds)
    scal = res.scalars.cpu().numpy()
    assert int(scal[2]) == 1 and int(scal[1]) == 4


# ---------------------------------------------------------------------------- least squares
@pytest.mark.parametrize("N,K,n,nsel", [(600, 96, 16, 60), (2000, 700, 40, 500), (500, 130, 7, 130)])
def test_ls_solve_matches_lstsq(engine, N, K, n, nsel):
    r = np.random.RandomState(K)
    X = np.maximum(r.standard_normal((N, K)), 0).astype(np.float32)
    Y = (X @ r.standard_normal((K, n)) + r.standard_normal((N, n))).astype(np.float32)
    sel = np.sort(r.choice(K, nsel, replace=False)).astype(np.int32)
    g = engine.gram(_dev(X, engine), _dev(Y, engine), mode=0)
    sel_d = _dev(sel, engine)
    W, b, info, _ = engine.ls_solve(g, sel_d)
    assert int(info.cpu()[0]) == 0
    # the same system factored alone, then solved against the kept factor
    info, _ = engine.ls_factor(g, sel_d)
    assert int(info.cpu()[0]) == 0
    Wr, br = engine.ls_resolve(g["B"], g["sx"], g["sy"], sel_d)
    coef, icpt = O.linear_regression(X[:, sel].astype(np.float64), Y.astype(np.float64))
    for Wx, bx in ((W, b), (Wr, br)):
        assert np.linalg.norm(Wx.cpu().numpy() - coef) <= 1e-9 * np.linalg.norm(coef)
        np.testing.assert_allclose(bx.cpu().numpy(), icpt, atol=1e-9 * max(1, np.abs(icpt).max()))
    # accumulate_into adds the solution to the given tensors in place
    W1, b1 = Wr.cpu().numpy(), br.cpu().numpy()
    Wa, ba = engine.ls_resolve(g["B"], g["sx"], g["sy"], sel_d, accumulate_into=(Wr, br))
    assert Wa is Wr and ba is br
    np.testing.assert_array_equal(Wr.cpu().numpy(), 2 * W1)
    np.testing.assert_array_equal(br.cpu().numpy(), 2 * b1)


def test_ls_solve_dual_minimum_norm(engine):
    r = np.random.RandomState(3)
    N, K, n = 300, 520, 9
    X = np.maximum(r.standard_normal((N, K)), 0).astype(np.float32)
    Y = r.standard_normal((N, n)).astype(np.float32)
    sel = np.arange(K, dtype=np.int32)
    W, b, info, _ = engine.ls_solve_dual(_dev(X, engine), _dev(Y, engine), None, _dev(sel, engine))
    assert int(info.cpu()[0]) == 0
    coef, icpt = O.linear_regression(X.astype(np.float64), Y.astype(np.float64))
    assert np.linalg.norm(W.cpu().numpy() - coef) <= 1e-8 * np.linalg.norm(coef)
    np.testing.assert_allclose(b.cpu().numpy(), icpt, atol=1e-8)


def test_ls_solve_flags_singular_system(engine):
    r = np.random.RandomState(4)
    X = r.standard_normal((400, 20)).astype(np.float32)
    X[:, 7] = X[:, 3]  # exactly collinear columns
    Y = r.standard_normal((400, 3)).astype(np.float32)
    g = engine.gram(_dev(X, engine), _dev(Y, engine), mode=0)
    W, b, info, _ = engine.ls_solve(g, _dev(np.arange(20, dtype=np.int32), engine))
    assert int(info.cpu()[0]) != 0


@pytest.mark.parametrize("mode", [0, 1], ids=["fp64", "3xtf32"])
def test_rank_deficient_system_gets_gelsd_truncated_solution(engine, mode):
    """Exactly collinear columns: the Cholesky flags the system, and fc_kernel returns what the reference's
    LinearRegression returns there -- gelsd's minimum-norm solution with singular values below 1e-6 sigma_max
    dropped (sklearn _base.py:752), the weight shared between the duplicates."""
    from cpb200.lib import decompose

    r = np.random.RandomState(4)
    X = np.maximum(r.standard_normal((900, 120)), 0).astype(np.float32)
    X[:, 70] = X[:, 30]          # exact duplicate
    X[:, 100] = 0.0              # dead column
    Y = (X @ r.standard_normal((120, 8)) + 0.1 * r.standard_normal((900, 8))).astype(np.float32)
    engine.gram_mode = mode
    coef, icpt = decompose.fc_kernel(X.astype(np.float64), Y.astype(np.float64))
    rc, ri = O.linear_regression(X.astype(np.float64), Y.astype(np.float64))
    assert np.linalg.norm(coef - rc) <= 1e-7 * np.linalg.norm(rc) and np.abs(icpt - ri).max() <= 1e-7
    assert np.abs(coef[:, 100]).max() <= 1e-9 and np.abs(coef[:, 70] - coef[:, 30]).max() <= 1e-9


@pytest.mark.parametrize("M,Nn,R,lower", [(700, 300, 256, False), (1030, 520, 128, True), (512, 512, 384, True),
                                          (257, 200, 130, False), (2048, 768, 512, False), (512, 1100, 512, "nc"),
                                          (300, 333, 200, "nc")])
def test_gemm_tc_split_matches_fp64(engine, M, Nn, R, lower):
    """cp_gemm_tc_split (the solver's tensor-core bulk product): C = beta C + alpha A B', rows of very different magnitude
    (power-of-two row scales).  Tolerance: |err| <= 4e-6 * sum_r |a||b|.  The operand split keeps 22 bits (<= 5e-7 of
    sum|a||b|); the rest is the tensor core's fp32 accumulator, which TRUNCATES: 12 additions per accumulator
    run (64 reduction elements), each losing < 2^-23 of the running sum in the same direction when all terms have one sign -- the
    diagonal of a symmetric update, the worst case (mixed signs partly cancel)."""
    r = np.random.RandomState(M + Nn + R)
    A = r.standard_normal((M, R)) * np.exp(3.0 * r.standard_normal((M, 1)))
    if lower is True:
        B = A[:Nn].copy()
    else:
        B = r.standard_normal((Nn, R)) * np.exp(3.0 * r.standard_normal((Nn, 1)))
    C0 = r.standard_normal((M, Nn))
    nc = lower == "nc"   # B handed over reduction-major (R, Nn)
    lower = lower is True
    Ad, Bd, Cd = (torch.as_tensor(x, device=engine.device) for x in (A, np.ascontiguousarray(B.T) if nc else B, C0.copy()))
    engine.gemm_tc_split(Ad, Bd, Cd, alpha=-1.0, beta=1.0, lower=lower, b_nc=nc)
    got = Cd.cpu().numpy()
    ref = C0 - A @ B.T
    bound = np.abs(A) @ np.abs(B).T
    err = np.abs(got - ref) / bound
    if lower:  # 128 x 128 tiles with row tile >= column tile are written; the others must be untouched
        ti, tj = np.arange(M)[:, None] // 128, np.arange(Nn)[None, :] // 128
        touched = ti >= tj
        assert np.array_equal(got[~touched], C0[~touched])
        err = err[touched]
    print("max err / sum|a||b| = %.2e" % err.max())
    assert err.max() <= 4e-6
