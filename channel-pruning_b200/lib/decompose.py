"""Drop-in for the channel-pruning part of the reference's ``lib/decompose.py``.

Same names, argument meaning, return values and implicit state (``cfgs.alpha``, the
numpy global RNG) as the reference; the arithmetic runs on the H100 through libcpb200
(see include/cpb200.h).  numpy in -> numpy out, exactly like the reference; torch CUDA
tensors are accepted too and avoid the host<->device copies.

  relu, rel_error        lib/decompose.py:22-23, 31-32
  dictionary             lib/decompose.py:386-634  (c3 configuration)
  fc_kernel              lib/decompose.py:636-669  (default LinearRegression branch)
  VH_decompose, ITQ_decompose, nonlinear_fc
                         signatures kept (lib/decompose.py:85,163,671); the 3C companions
                         are SURVEY.md 8(f) "next" and raise NotImplementedError here.
"""
from __future__ import annotations

import numpy as np
import torch

from . import cfgs
from .cfgs import c as dcfgs
from ..engine import MAX_PROBES, RAND_R_MAX, get_engine, settle_ls


def relu(x):
    """lib/decompose.py:22-23"""
    if isinstance(x, torch.Tensor):
        return torch.clamp_min(x, 0.)
    return np.maximum(x, 0.)


def rel_error(A, B):
    """lib/decompose.py:31-32"""
    return np.mean((A - B) ** 2) ** .5 / np.mean(A ** 2) ** .5


def _dev_f32(a, eng):
    if isinstance(a, torch.Tensor):
        return a.to(device=eng.device, dtype=torch.float32).contiguous()
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32), device=eng.device)


def _dev_y(Y, eng):
    """Targets are used exactly: fp32 when every value is fp32-representable, else fp64."""
    if isinstance(Y, torch.Tensor):
        if Y.dtype == torch.float32:
            return Y.to(eng.device).contiguous()
        Yd = Y.to(device=eng.device, dtype=torch.float64).contiguous()
        Y32 = Yd.to(torch.float32)
        return Y32 if bool((Y32.to(torch.float64) == Yd).all()) else Yd
    Y = np.ascontiguousarray(Y)
    if Y.dtype == np.float32:
        return torch.as_tensor(Y, device=eng.device)
    Y = Y.astype(np.float64, copy=False)
    Y32 = Y.astype(np.float32)
    if np.array_equal(Y32.astype(np.float64), Y):
        return torch.as_tensor(Y32, device=eng.device)
    return torch.as_tensor(Y, device=eng.device)


class DictionaryInfo:
    """Diagnostics of the last ``dictionary`` call (alpha probes, CD iterations)."""
    last = None


def dictionary(X, W2, Y, alpha=1e-4, rank=None, DEBUG=0, B2=None, rank_tol=.1, verbose=0):
    """LASSO channel selection + least-squares reconstruction, reference
    lib/decompose.py:386-634.

    X: (N, c, h, w)   W2: (n, c, h, w)   Y: (N, n)   rank: channels to keep
    returns (idxs bool[c], newW2 (n, c', h, w) float64, newB2 (n,) float64)
    h != w (a 1 x 7 or 3 x 1 layer) is accepted: columns are (c, h, w) in that order, as F.unfold gives them.
    Conv3d layers: X (N, c, t, h, w), W2 (n, c, t, h, w) -> newW2 (n, c', t, h, w); columns (c, t, h, w).
    or, with DEBUG, (newX, newW2, newB2) (decompose.py:629-632).

    Reference behaviour that is kept on purpose:
      * ``rank_tol`` argument ignored, dcfgs.dic.rank_tol used (:393); verbose forced off (:387)
      * rows for the LASSO drawn with replacement from the numpy GLOBAL RNG (:425), one
        further global draw per Lasso.fit for its coordinate order (sklearn _cd_fast)
      * alpha search starts at cfgs.alpha and stores the final alpha back (:491, :627);
        with rank == c the LASSO is skipped and cfgs.alpha becomes the *argument* (:487, :627)
      * the reference assumes square kernels, w = h (:401-402); here w is read from X.shape[3].  Square inputs draw
        the same RNG values and give the same results as the reference
    Deviation: the reference's unguarded ``while True`` loops (:502, :516) are capped at
    64 probes; hitting the cap raises RuntimeError instead of spinning forever.
    """
    if dcfgs.autodet or dcfgs.solver != cfgs.solvers.sk or dcfgs.ls != 'linear' or dcfgs.dic.alter or \
            dcfgs.dic.debug or dcfgs.fc_ridge or dcfgs.nonlinear_fc or dcfgs.nofc:
        raise NotImplementedError("only the `train.py -action c3` configuration of dictionary() is implemented")
    eng = get_engine()
    N, c, win = X.shape[0], X.shape[1], tuple(int(v) for v in X.shape[2:])  # win: (h, w), or (t, h, w) for Conv3d
    assert len(win) in (2, 3), "X must be (N, c, h, w) or (N, c, t, h, w)"
    k2 = int(np.prod(win))
    n = W2.shape[0]
    assert tuple(W2.shape) == (n, c) + win and tuple(Y.shape) == (N, n)
    Xd = _dev_f32(X, eng).reshape(N, c * k2)
    W2m = _dev_f32(W2, eng).reshape(n, c * k2)
    Yd = _dev_y(Y, eng)
    idxs, Wd, bd = _dictionary_device(eng, Xd, W2m, Yd, None, c, k2, rank, alpha)
    rank = int(idxs.sum())
    newW2 = Wd.cpu().numpy().reshape((n, rank) + win)
    newB2 = bd.cpu().numpy()
    if DEBUG:
        Xh = X.cpu().numpy() if isinstance(X, torch.Tensor) else np.asarray(X)
        return Xh[:, idxs, ...], newW2, newB2
    return idxs, newW2, newB2


def _dictionary_device(eng, Xd, W2m, Yd, y_bias, c, k2, rank, alpha=1e-4):
    """Body of ``dictionary`` on device buffers: Xd (N, c*k2) fp32 in (c,kh,kw) column order (k2 = kh*kw taps per
    channel), W2m (n, c*k2) fp32, Yd (N, n) fp32|fp64 with optional fp32 ``y_bias`` subtracted exactly.
    Returns (idxs numpy bool[c], W (n, K') fp64 device, b (n,) fp64 device)."""
    rank_tol = dcfgs.dic.rank_tol  # :393
    N = Xd.shape[0]
    S = min(400, N // 20)
    samples = np.random.randint(0, N, S)  # :425 -- consumed even when rank == c, like the reference
    info = {"samples": samples, "probes": [], "alpha": alpha}
    if rank == c:  # :487-488
        idxs = np.array([True] * rank)
        g_full = eng.gram(Xd, Yd, y_bias=y_bias)
    else:
        state = np.random.get_state()
        seeds = np.random.randint(0, RAND_R_MAX, size=MAX_PROBES)
        samples_d = torch.as_tensor(samples.astype(np.int32), device=eng.device)
        g_full, res = eng.select_channels_async(Xd, W2m, Yd, y_bias, samples_d, c, k2, rank, rank_tol, cfgs.alpha,
                                                seeds)
        scal = res.scalars.cpu().numpy()  # synchronises
        nprobe, status = int(scal[1]), int(scal[2])
        np.random.set_state(state)
        if nprobe:
            np.random.randint(0, RAND_R_MAX, size=nprobe)  # the draws the reference's fits would have made
        plog = res.probe_log[:nprobe].cpu().numpy()
        info["probes"] = [(float(a), int(z)) for a, z, _, _ in plog]
        info["cd"] = [(int(it), float(gap)) for _, _, it, gap in plog]
        info["coef"] = res.coef.cpu().numpy()
        if status != 0:
            raise RuntimeError("alpha search hit the %d-probe cap (the reference would loop forever); probes=%r"
                               % (MAX_PROBES, info["probes"]))
        alpha = float(scal[0])
        idxs = res.idxs.cpu().numpy().astype(bool)
    Wd, bd = _solve_ls(eng, g_full, Xd, Yd, y_bias, idxs, k2, info)
    cfgs.alpha = alpha  # :626-627
    info["alpha"] = alpha
    DictionaryInfo.last = info
    return idxs, Wd, bd


def _solve_ls(eng, g_full, Xd, Yd, y_bias, idxs, k2, info=None):
    """LS on the surviving channels, accepted or redone by the conditioning policy of engine.settle_ls."""
    Wd, bd, info_d, stat_d = eng.reconstruct_async(g_full, Xd, Yd, y_bias, idxs, k2)
    fail, ratio = int(info_d.cpu()[0]), float(stat_d.cpu()[0])
    W, b, rec = settle_ls(eng, Xd, Yd, y_bias, idxs, k2, g_full["mode"], fail, ratio)
    if info is not None:
        info["ls"] = rec
    return (Wd, bd) if W is None else (W, b)


def fc_kernel(X, Y, copy_X=True, W=None, B=None, ret_reg=False, fit_intercept=True):
    """Least squares with intercept, reference lib/decompose.py:636-669 (default branch:
    ``LinearRegression(fit_intercept=True).fit(X, Y)``).  Returns (coef (n, K), intercept (n,))."""
    assert copy_X == True  # noqa: E712   (decompose.py:640)
    assert len(X.shape) == 2  # decompose.py:641
    if dcfgs.ls != 'linear' or dcfgs.fc_ridge:
        raise NotImplementedError("only the default LinearRegression branch of fc_kernel is implemented")
    if ret_reg or not fit_intercept:
        raise NotImplementedError("ret_reg / fit_intercept=False are used by nonlinear_fc only (SURVEY.md 8f)")
    eng = get_engine()
    Xd = _dev_f32(X, eng)
    Yd = _dev_y(Y, eng)
    g = eng.gram(Xd, Yd)
    K = Xd.shape[1]
    Wd, bd = _solve_ls(eng, g, Xd, Yd, None, np.ones(K, dtype=bool), 1)
    return Wd.cpu().numpy(), bd.cpu().numpy()


def _dev_f64(a, eng):
    if isinstance(a, torch.Tensor):
        return a.to(device=eng.device, dtype=torch.float64).contiguous()
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device=eng.device)


def solve_relu(RU, Z, Lambda):
    """lib/decompose.py:51-59 (elementwise; cp_solve_relu)."""
    eng = get_engine()
    U = eng.solve_relu(_dev_f64(RU, eng), None, _dev_f64(Z, eng), Lambda)
    return U if isinstance(RU, torch.Tensor) else U.cpu().numpy()


def svd(x):
    """lib/decompose.py:154-156: thin SVD, singular values descending (one-sided Jacobi on the device; singular
    vectors agree with LAPACK's up to the sign of each pair)."""
    eng = get_engine()
    U, s, Vh = eng.svd(_dev_f64(x, eng))
    if isinstance(x, torch.Tensor):
        return U, s, Vh
    return U.cpu().numpy(), s.cpu().numpy(), Vh.cpu().numpy()


def _pinv_device(eng, x, rtol=1e-6):
    U, s, Vh = eng.svd(x)
    keep = s > rtol * s[0]
    inv = torch.where(keep, 1.0 / torch.where(keep, s, torch.ones_like(s)), torch.zeros_like(s))
    return eng.mm_tn(Vh, (U * inv[None, :]).T.contiguous())  # V diag(1/s) U'


def pinv(x):
    """lib/decompose.py:149-152: scipy.linalg.pinv(x, 1e-6) -- singular values below 1e-6 sigma_max dropped."""
    eng = get_engine()
    P = _pinv_device(eng, _dev_f64(x, eng))
    return P if isinstance(x, torch.Tensor) else P.cpu().numpy()


def _nonlinear_fc_device(eng, Xd, Yd):
    """Body of nonlinear_fc on fp64 device buffers: the centred Gram of X is factored ONCE (cp_ls_factor), each of the
    50 refits is X'U (one tall-skinny product) + two triangular substitutions (cp_ls_resolve), a prediction and the
    elementwise ReLU-aware update.  Returns (coef (n, K), intercept (n,)) on the device."""
    N, K = Xd.shape
    G = eng.mm_tn(Xd, Xd)
    sx = eng.colstats(Xd)
    g = dict(G=G, sx=sx, N=N, K=K)
    info_d, stat_d = eng.ls_factor(g)
    fail = int(info_d.cpu()[0])
    if fail:
        raise np.linalg.LinAlgError("nonlinear_fc: X is numerically rank deficient (pivot %d); the reference's gelsd "
                                    "would truncate here" % fail)
    U = Yd.clone()
    Z = torch.clamp_min(Yd, 0.)
    its = [30, 20]
    W = b = None
    for epoch, l in enumerate([10 ** i for i in range(-1, 1)]):  # decompose.py:678
        for _ in range(its[epoch]):
            Bxy = eng.mm_tn(Xd, U)
            sy = eng.colstats(U)
            W, b = eng.ls_resolve(Bxy, sx, sy)  # reg = fc_kernel(X, U, ret_reg=True)
            RUraw = eng.mm_nt(Xd, W)            # reg.predict(X) without the intercept
            U = eng.solve_relu(RUraw, b, Z, l)
    return W, b


def nonlinear_fc(X, Y, copy_X=True, W=None, B=None):
    """lib/decompose.py:671-685.  Returns (coef_ (n, K), intercept_ (n,)) of the last refit, float64."""
    assert len(X.shape) == 2  # :672
    assert copy_X == True  # noqa: E712  (:673)
    assert W is None and B is None  # :674-675
    eng = get_engine()
    Wd, bd = _nonlinear_fc_device(eng, _dev_f64(X, eng), _dev_f64(Y, eng))
    return Wd.cpu().numpy(), bd.cpu().numpy()


def VH_decompose(weights, rank=None, DEBUG=0, X=None, Y=None):
    """Spatial decomposition, reference lib/decompose.py:85-147.
    weights (n, c, h, w) -> V (rank, c, h, 1), H (n, rank, 1, w), VHr (n, c, h, w) [, b (n,)]; with X (N, c, h, w) and
    Y (N, n) the H factor is refitted on data by nonlinear_fc (:129-138).  SVD, projections and the 50 refits run on
    the device in fp64; numpy float64 in and out like the reference."""
    eng = get_engine()
    Wd = _dev_f64(weights, eng)
    n, c, h, w = Wd.shape
    VH = Wd.permute(1, 2, 0, 3).reshape(c * h, n * w).contiguous()  # ch x nw  (:96-99)
    Vm, sig, Hm = eng.svd(VH)
    if rank is None:
        rank = c * h
    Vm = Vm[:, :rank].contiguous()                       # ch x rank
    Hm = (sig[:rank, None] * Hm[:rank, :]).contiguous()  # rank x nw  (:105-111)
    VHr = eng.mm(Vm, Hm).reshape(c, h, n, w)
    H = Hm.reshape(rank, n, w, 1).permute(1, 0, 3, 2).contiguous()  # n rank 1 w
    V = Vm.reshape(c, 1, h, rank).permute(3, 0, 2, 1).contiguous()  # rank c h 1
    b = None
    if X is not None:
        Xd = _dev_f64(X, eng)
        N = Xd.shape[0]
        assert w == 3, "the reference reshapes H to (o, rank, 1, 3) (decompose.py:135)"
        # Xv[N, rank, 1, w] = sum_{c,h} X[N, c, h, w] V[rank, c, h]   (:130-131)
        Xp = Xd.permute(0, 3, 1, 2).reshape(N * w, c * h).contiguous()
        Xv = eng.mm(Xp, Vm).reshape(N, w, rank).permute(0, 2, 1).reshape(N, rank * w).contiguous()
        Hfit, bd = _nonlinear_fc_device(eng, Xv, _dev_f64(Y, eng))
        H = Hfit.reshape(n, rank, 1, 3)
        reH = H.permute(1, 0, 2, 3).reshape(rank, n * 3).contiguous()
        VHr = eng.mm(Vm, reH).reshape(c, h, n, w)  # (:136-138)
        b = bd.cpu().numpy()
    VHr = VHr.permute(2, 0, 1, 3).contiguous()
    if X is not None:
        return V.cpu().numpy(), H.cpu().numpy(), VHr.cpu().numpy(), b
    return V.cpu().numpy(), H.cpu().numpy(), VHr.cpu().numpy()


def ITQ_decompose(feature, gt_feature, weight, rank, bias=None, DEBUG=False, Wr=None):
    """Channel decomposition, reference lib/decompose.py:163-319 (the branch Net.R3 takes: weight (n, r, 1, w),
    ``right = 1``).  Returns W1 (rank, r, 1, w), W2 (n, rank, 1, 1), B (n,), W12 (n, c, h, w), float64.

    Device formulation: every N x n quantity of the loop is G times an n x n matrix (X = G M, M = pinv(G'G) G'UU), so
    the thin SVD of the N x n matrix X (:217) is taken of the n x n matrix F = diag(sqrt(s_S)) V_S' M, which has the
    same singular values and right singular vectors (F'F = M'(G'G)M = X'X, with G'G = V_S diag(s_S) V_S'); per
    iteration only G'UU and G T remain tall products."""
    eng = get_engine()
    Yf = _dev_f64(feature, eng)
    n_ins, nfc = Yf.shape
    gt = _dev_f64(gt_feature, eng)
    assert tuple(gt.shape) == (n_ins, nfc)  # :167-168
    Z = torch.clamp_min(gt, 0.)
    Y_mean, G = eng.colstats(Yf, 1.0 / n_ins, centre=True)  # :180-182
    S = eng.mm_tn(G, G)
    Us, ss, Vhs = eng.svd(S)
    keep = ss > 1e-6 * ss[0]
    inv = torch.where(keep, 1.0 / torch.where(keep, ss, torch.ones_like(ss)), torch.zeros_like(ss))
    PG = eng.mm_tn(Vhs, (Us * inv[None, :]).T.contiguous())  # pinv(G'G), :189
    E = (torch.sqrt(ss)[:, None] * Vhs).contiguous()        # E'E = G'G
    UU = G.clone()
    U_mean = Y_mean.clone()
    T = None
    for Lambda, iters in zip([0.1, 1], [30, 20]):  # :203-204
        for _ in range(iters):
            A1 = eng.mm_tn(G, UU)          # G'UU
            M = eng.mm(PG, A1)             # X = G M  (:213)
            F = eng.mm(E, M)
            _, _, Rh = eng.svd(F)
            Rr = Rh[:rank].contiguous()    # top right singular vectors of X
            MP = eng.mm(eng.mm_nt(M, Rr), Rr)   # M R_r' R_r:  T_big = G (M P)  (:219)
            T = eng.mm(PG, eng.mm(S, MP))       # PGGt.dot(T_big)  (:225)
            RUraw = eng.mm(G, T)                # :226
            U, U_mean_new = eng.solve_relu(RUraw, U_mean, Z, Lambda, want_mean=True)  # :228-240
            U_mean = U_mean_new
            UU = U - U_mean[None, :]
    L, sigma, R = eng.svd(T)  # :250
    L = L[:, :rank].contiguous()
    R = (sigma[:rank, None] * R[:rank, :]).contiguous()
    Wd = _dev_f64(weight, eng)
    dim = tuple(Wd.shape)
    assert len(dim) == 4
    assert dim[3] != nfc and dim[0] == nfc, "only the branch Net.R3 takes (decompose.py:261-262) is implemented"
    wt = Wd.permute(1, 2, 3, 0).contiguous()
    W1 = eng.mm(wt.reshape(-1, nfc), L)  # :265-266
    if Wr is not None:
        wr = _dev_f64(Wr, eng).permute(1, 2, 3, 0).contiguous()
        W12 = eng.mm(wr.reshape(-1, nfc), L)
        shape12 = tuple(wr.shape[:3])
    else:
        W12 = W1
        shape12 = tuple(wt.shape[:3])
    W1 = W1.reshape(tuple(wt.shape[:3]) + (rank,)).permute(3, 0, 1, 2).contiguous()
    W2 = R
    W12 = eng.mm(W12.contiguous(), W2)
    W2 = W2.T.contiguous().reshape(nfc, rank, 1, 1)
    W12 = W12.reshape(shape12 + (nfc,)).permute(3, 0, 1, 2).contiguous()
    B = -eng.mm(Y_mean[None, :].contiguous(), T)[0] + U_mean  # :304
    B = B.cpu().numpy()
    if bias is not None:
        B = B + np.asarray(bias.cpu().numpy() if isinstance(bias, torch.Tensor) else bias, dtype=np.float64)
    return W1.cpu().numpy(), W2.cpu().numpy(), B, W12.cpu().numpy()
