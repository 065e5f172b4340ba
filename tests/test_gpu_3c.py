"""GPU: the 3C companions of the pruning path (SURVEY.md 8a-a8 / 8f): dense fp64 blocks through the C ABI, then
VH_decompose / nonlinear_fc / ITQ_decompose against golden outputs of the reference's own code
(tests/golden/vh_*.npz, itq_*.npz, written by oracle/make_golden.py) and against the oracle."""
import os

import numpy as np
import pytest

import cases
import cp_oracle as O

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def _dev(a, eng):
    return torch.as_tensor(np.ascontiguousarray(a), device=eng.device)


def _sign_align(a, b, axis):
    a2 = np.moveaxis(a, axis, 0).copy()
    b2 = np.moveaxis(b, axis, 0)
    for k in range(a2.shape[0]):
        if np.vdot(a2[k], b2[k]) < 0:
            a2[k] = -a2[k]
    return np.moveaxis(a2, 0, axis)


@pytest.mark.parametrize("M,Nn,R", [(1, 48, 48), (130, 70, 33), (64, 64, 5000), (300, 257, 129), (5000, 40, 96)])
def test_gemm_f64_all_layouts(engine, M, Nn, R):
    r = np.random.RandomState(M + Nn)
    A, B = r.standard_normal((M, R)), r.standard_normal((R, Nn))
    want = A @ B
    tol = 1e-12 * np.abs(want).max() * max(1, R) ** .5
    np.testing.assert_allclose(engine.mm(_dev(A, engine), _dev(B, engine)).cpu().numpy(), want, atol=tol)
    np.testing.assert_allclose(engine.mm_nt(_dev(A, engine), _dev(B.T, engine)).cpu().numpy(), want, atol=tol)
    np.testing.assert_allclose(engine.mm_tn(_dev(A.T, engine), _dev(B, engine)).cpu().numpy(), want, atol=tol)
    C0 = r.standard_normal((M, Nn))
    out = _dev(C0, engine)
    engine.gemm(_dev(A.T, engine), _dev(B.T, engine), a_mc=True, b_nc=False, alpha=-2.0, beta=0.5, out=out)
    np.testing.assert_allclose(out.cpu().numpy(), -2.0 * want + 0.5 * C0, atol=3 * tol)


@pytest.mark.parametrize("a_mc,b_nc", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_gemm_f64_empty_reduction_scales_c(engine, a_mc, b_nc):
    # through the C ABI: Engine.gemm passes an empty operand as NULL, which cp_gemm_f64 refuses
    M, Nn = 130, 70
    C0 = np.random.RandomState(4).standard_normal((M, Nn))
    A = torch.full((M, M), float("nan"), dtype=torch.float64, device=engine.device)  # never read at R = 0
    B = torch.full((Nn, Nn), float("nan"), dtype=torch.float64, device=engine.device)
    out = _dev(C0, engine)
    engine._call(engine.lib.cp_gemm_f64(engine.h, a_mc, b_nc, M, Nn, 0, -2.0, engine._p(A, "const double*"), M,
                                        engine._p(B, "const double*"), Nn, 0.5, engine._p(out, "double*"), Nn,
                                        engine._s()))
    assert np.array_equal(out.cpu().numpy(), 0.5 * C0)


@pytest.mark.parametrize("m,n,kind", [(36, 60, "full"), (60, 36, "full"), (200, 200, "full"), (128, 128, "lowrank"),
                                      (768, 300, "decay"), (257, 255, "full")])
def test_svd_jacobi_matches_lapack(engine, m, n, kind):
    r = np.random.RandomState(m * 7 + n)
    F = r.standard_normal((m, n))
    if kind == "lowrank":
        F = r.standard_normal((m, 20)) @ r.standard_normal((20, n))
    elif kind == "decay":
        u, _, vt = np.linalg.svd(F, full_matrices=False)
        F = (u * np.logspace(0, -9, min(m, n))) @ vt
    U, s, Vh = [t.cpu().numpy() for t in engine.svd(_dev(F, engine))]
    k = min(m, n)
    assert U.shape == (m, k) and s.shape == (k,) and Vh.shape == (k, n)
    s_ref = np.linalg.svd(F, compute_uv=False)
    np.testing.assert_allclose(s, s_ref, atol=1e-13 * s_ref[0])
    assert np.all(np.diff(s) <= 0)
    np.testing.assert_allclose((U * s) @ Vh, F, atol=1e-12 * s_ref[0])
    live = s_ref > 1e-12 * s_ref[0]
    np.testing.assert_allclose((U[:, live].T @ U[:, live]), np.eye(live.sum()), atol=1e-11)
    np.testing.assert_allclose((Vh[live] @ Vh[live].T), np.eye(live.sum()), atol=1e-11)


def test_solve_relu_and_pinv(engine):
    from cpb200.lib import decompose

    r = np.random.RandomState(2)
    RU, Z = r.standard_normal((500, 37)), np.maximum(r.standard_normal((500, 37)), 0)
    for lam in (0.1, 1):
        np.testing.assert_array_equal(decompose.solve_relu(RU, Z, lam), O.solve_relu(RU, Z, lam))
    G = r.standard_normal((300, 40)) @ r.standard_normal((40, 40))
    G[:, 7] = G[:, 3]  # rank deficient: the 1e-6 cut-off must drop the null direction
    S = G.T @ G
    np.testing.assert_allclose(decompose.pinv(S), O.pinv(S), atol=1e-9 * np.abs(O.pinv(S)).max())


def test_nonlinear_fc_matches_oracle(engine):
    from cpb200.lib import decompose

    r = np.random.RandomState(5)
    X = np.maximum(r.standard_normal((1200, 90)), 0)
    Y = X @ r.standard_normal((90, 24)) * 0.3 + 0.1 * r.standard_normal((1200, 24))
    W, b = decompose.nonlinear_fc(X, Y)
    Wo, bo = O.nonlinear_fc(X, Y)
    assert np.linalg.norm(W - Wo) <= 1e-8 * np.linalg.norm(Wo) and np.abs(b - bo).max() <= 1e-8
    with pytest.raises(AssertionError):
        decompose.nonlinear_fc(X[None], Y)


@pytest.mark.parametrize("name", list(cases.VH_CASES))
def test_vh_decompose_matches_reference_golden(engine, golden_dir, name):
    from cpb200.lib import decompose

    spec = cases.VH_CASES[name]
    g = np.load(os.path.join(golden_dir, "%s.npz" % name))
    W, X, Y = cases.vh_inputs(**spec["gen"])
    V, H, VHr, b = decompose.VH_decompose(W.astype(np.float64), rank=spec["rank"], DEBUG=0, X=X.astype(np.float64), Y=Y)
    assert V.shape == g["V"].shape and H.shape == g["H"].shape and VHr.shape == g["VHr"].shape and V.dtype == np.float64
    scale = np.abs(g["VHr"]).max()
    assert np.linalg.norm(VHr - g["VHr"]) <= 1e-6 * np.linalg.norm(g["VHr"])   # sign-invariant outputs
    assert np.abs(b - g["b"]).max() <= 1e-6 * max(1.0, np.abs(g["b"]).max())
    np.testing.assert_allclose(_sign_align(V, g["V"], 0), g["V"], atol=1e-8)
    np.testing.assert_allclose(_sign_align(H, g["H"], 1), g["H"], atol=1e-6 * np.abs(g["H"]).max())
    V0, H0, VHr0 = decompose.VH_decompose(W.astype(np.float64), rank=spec["rank"])
    np.testing.assert_allclose(VHr0, g["VHr0"], atol=1e-10 * scale)
    np.testing.assert_allclose(_sign_align(H0, g["H0"], 1), g["H0"], atol=1e-9)


@pytest.mark.parametrize("name", list(cases.ITQ_CASES))
def test_itq_decompose_matches_reference_golden(engine, golden_dir, name):
    from cpb200.lib import decompose

    spec = cases.ITQ_CASES[name]
    g = np.load(os.path.join(golden_dir, "%s.npz" % name))
    feat, gt, H, VHr, bias = cases.itq_inputs(**spec["gen"])
    W1, W2, B, W12 = decompose.ITQ_decompose(feat, gt, H, spec["rank"], bias=bias, DEBUG=0, Wr=VHr)
    assert W1.shape == g["W1"].shape and W2.shape == g["W2"].shape and W12.shape == g["W12"].shape
    assert np.linalg.norm(W12 - g["W12"]) <= 1e-4 * np.linalg.norm(g["W12"])     # sign-invariant outputs
    assert np.abs(B - g["B"]).max() <= 1e-4 * max(1.0, np.abs(g["B"]).max())
    a1, a2 = _sign_align(W1, g["W1"], 0), _sign_align(W2, g["W2"], 1)
    assert np.linalg.norm(a1 - g["W1"]) <= 1e-4 * np.linalg.norm(g["W1"])
    assert np.linalg.norm(a2 - g["W2"]) <= 1e-4 * np.linalg.norm(g["W2"])
