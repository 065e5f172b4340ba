"""GPU: the Cholesky least-squares solver (csrc/ls.cu) entry by entry -- cp_ls_solve, cp_ls_factor / cp_ls_resolve,
cp_ls_solve_dual, cp_ls_residual -- against host references in fp64 and higher, on every branch of its schedule.

The statistics are built outside the library (cuBLAS fp64 products through torch), so a failure points at the
solver.  Error model of the primal solve, in the diagonally scaled system H = D^-1 Gc D^-1 (D = sqrt(diag Gc); the
Cholesky factorisation is invariant to that scaling, and H has a unit diagonal):
  * backward error  |D^-1 (Bc - Gc w)| / (|H| |D w|)  <=  beta = 4 K' u + eta_asm + eta_rhs + eta_ref
      4 K' u:  the factorisation and both substitutions, each element a dot product of at most K' fp64 terms:
               Higham's (3K' + 1) u |L||L'| (Thm 10.4) in norm, with |(|L||L'|)| ~ |H| (entries <= 1 for a
               unit-diagonal H; the worst case K' |H| is not approached by data like these);
      eta_asm: the centred Gram assembled here and by ls_assemble may round G - sx sx'/N differently (FMA
               contraction): |dGc| <= 2u (|G| + |sx sx'|/N), scaled, in the infinity norm (>= the 2-norm, symmetric);
      eta_rhs: the same for the right-hand sides Bc = Bxy - sx sy'/N;
      eta_ref: the residual of the reference itself, u |H| |D w| (it is the exact solution rounded once);
  * forward error   |D (w - w_ref)| / |D w_ref|  <=  kappa(H) beta / (1 - kappa(H) beta);
  * intercept       |b - b_ref| <= (|sx' (w - w_ref)| + 2 (K' + 2) u (|sy| + |sx|'|w|)) / N: the first term is the
                    intercept's exact response to the device's own weights, so b is checked to the rounding of
                    ls_output's sum (measured and bound meet where the weights' error dominates).
The reference is scipy's Cholesky, refined once with a residual in extended precision (np.longdouble): its error is
(kappa K' u)^2, far below the bounds.  Every case prints measured / bound."""
import numpy as np
import pytest
import scipy.linalg

import cp_oracle as O

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

U = 2.0 ** -53
N, K, NT = 2700, 2400, 320   # module problem: rows, columns, targets
NPLAIN = K - 8               # columns K - 8 .. K - 1 are collinear with earlier ones (COLLIN)
LS_RATIO_MIN = 0.005         # engine.LS_RATIO_MIN, checked below
# collinear column -> (partner, 1 - rho^2):  x_j = rho x_i + sqrt(1 - rho^2) z.  With ~1100 other columns selected the
# pivot ratio of x_j is about (1 - rho^2)(1 - K'/N): about 0.06, 0.012, 0.0062 and 1e-6 here (measured by the host
# factor in each case that uses them)
COLLIN = {NPLAIN + 0: (11, 0.1), NPLAIN + 1: (23, 0.02), NPLAIN + 2: (37, 0.0103), NPLAIN + 3: (41, 1.7e-6)}


def make_host_data():
    r = np.random.RandomState(2026)
    X = np.maximum(r.standard_normal((N, K)), 0.0)  # ReLU features: nonzero means, centring cancels
    for j, (i, e) in COLLIN.items():
        X[:, j] = np.sqrt(1.0 - e) * X[:, i] + np.sqrt(e) * np.maximum(r.standard_normal(N), 0.0)
    X = X.astype(np.float32)
    Wt = r.standard_normal((NPLAIN, NT)) / np.sqrt(NPLAIN)
    Y = (X[:, :NPLAIN].astype(np.float64) @ Wt + 0.5 * r.standard_normal((N, NT)) + 0.3).astype(np.float32)
    return X, Y


def selection(kp, extra=()):
    """Ascending subset of kp plain columns with gaps (seeded by kp), plus the given extra columns."""
    r = np.random.RandomState(kp + 7)
    pool = np.setdiff1d(np.arange(NPLAIN), extra)
    base = r.choice(pool, kp - len(extra), replace=False)
    return np.sort(np.concatenate([base, np.asarray(extra, dtype=np.int64)])).astype(np.int32)


# ---------------------------------------------------------------------------- host reference
class Ref:
    """Host solution of the centred normal equations on columns sel, right-hand sides 0..n-1, and what the error model
    needs.  G, Bxy, sx, sy: the host copies of the statistics handed to the solver."""

    def __init__(self, G, Bxy, sx, sy, sel, n, nrows=N):
        invN = 1.0 / nrows
        sxs = sx[sel]
        S = np.outer(sxs, sxs) * invN
        Gs = G[np.ix_(sel, sel)]
        self.Gc = Gs - S                                   # the formula of ls_assemble
        self.Bc = Bxy[sel, :n] - np.outer(sxs, sy[:n]) * invN
        self.kp, self.n, self.invN, self.sx, self.sy = len(sel), n, invN, sxs, sy[:n]
        c = scipy.linalg.cho_factor(self.Gc, lower=True)
        W = scipy.linalg.cho_solve(c, self.Bc)
        ld = np.longdouble
        R = (self.Bc.astype(ld) - self.Gc.astype(ld) @ W.astype(ld)).astype(np.float64)
        self.W = (W + scipy.linalg.cho_solve(c, R)).T      # (n, K')
        self.b = ((sy[:n].astype(ld) - self.W.astype(ld) @ sxs.astype(ld)) * ld(invN)).astype(np.float64)
        self.d = np.sqrt(np.diag(self.Gc))
        self.H = self.Gc / np.outer(self.d, self.d)
        ev = np.linalg.eigvalsh(self.H)
        self.normH, self.kappa = ev[-1], ev[-1] / ev[0]
        self.Ls = np.tril(c[0]) / self.d[:, None]          # Cholesky factor of H
        self.pivots = np.diag(self.Ls) ** 2                # exact pivot / original-diagonal ratios
        self.ratio = self.pivots.min()
        dd = np.outer(self.d, self.d)
        self.eta_asm = (2 * U * (np.abs(Gs) + np.abs(S)) / dd).sum(1).max() / self.normH
        self.e_rhs = 2 * U * (np.abs(Bxy[sel, :n]) + np.abs(np.outer(sxs, sy[:n])) * invN) / self.d[:, None]

    def sliced(self, n):
        """The same reference for the first n right-hand sides."""
        s = Ref.__new__(Ref)
        s.__dict__.update(self.__dict__)
        s.n, s.Bc, s.W, s.b, s.sy, s.e_rhs = n, self.Bc[:, :n], self.W[:n], self.b[:n], self.sy[:n], self.e_rhs[:, :n]
        return s

    def beta(self, Wd):
        """Backward-error bound per right-hand side (fp64 solve) for the device solution Wd (n, K')."""
        y = Wd * self.d
        yn = np.linalg.norm(y, axis=1)
        eta_rhs = np.linalg.norm(self.e_rhs, axis=0) / (self.normH * yn)
        eta_ref = U * np.linalg.norm(np.abs(self.W * self.d) @ np.abs(self.H), axis=1) / (self.normH * yn)
        return 4 * self.kp * U + self.eta_asm + eta_rhs + eta_ref

    def errors(self, Wd):
        """(forward, backward) error per right-hand side, in the scaled system."""
        dy = (Wd - self.W) * self.d
        fwd = np.linalg.norm(dy, axis=1) / np.linalg.norm(self.W * self.d, axis=1)
        bwd = np.linalg.norm(dy @ self.H, axis=1) / (self.normH * np.linalg.norm(Wd * self.d, axis=1))
        return fwd, bwd

    def check(self, Wd, bd, label, extra_beta=0.0):
        """Asserts the error model above (extra_beta: a further backward-error term, the tensor cores') and returns
        the measured forward error."""
        Wd, bd = np.asarray(Wd), np.asarray(bd)
        fwd, bwd = self.errors(Wd)
        beta = self.beta(Wd) + extra_beta
        kb = self.kappa * beta
        assert (kb < 0.5).all(), "bound vacuous for %s" % label
        fb = kb / (1 - kb)
        sdw = np.abs((Wd - self.W) @ self.sx)
        bb = (sdw + 2 * (self.kp + 2) * U * (np.abs(self.sy) + np.abs(Wd) @ np.abs(self.sx))) * self.invN
        eb = np.abs(bd - self.b)
        print("%s: K'=%d n=%d kappa %.0f  fwd %.2e / %.2e  bwd %.2e / %.2e  b %.2e / %.2e" % (
            label, self.kp, self.n, self.kappa, fwd.max(), fb[np.argmax(fwd / fb)], bwd.max(),
            beta[np.argmax(bwd / beta)], eb.max(), bb[np.argmax(eb / np.maximum(bb, 1e-300))]))
        assert (bwd <= beta).all(), (label, (bwd / beta).max())
        assert (fwd <= fb).all(), (label, (fwd / fb).max())
        assert (eb <= bb).all(), (label, (eb / bb).max())
        return fwd.max()

    def tc_beta(self):
        """Backward-error term of the split-precision (22-bit) products: each product of the factorisation, of the
        forward and of the backward substitution errs by at most 4e-6 sum_k |a_k||b_k| per element (cp_gemm_tc_split,
        test_gpu_kernels.py), which adds up, per element of H, to 4e-6 (|L||L'|)_ij for each of the three stages.
        The diagonal gets its bound in full (the accumulator truncates in one direction when every term has one
        sign); off the diagonal the terms have both signs and the errors are independent roundings, so the norm of
        that part is bounded like the norm of a random matrix with those entry bounds: 3 max_i sqrt(sum_j e_ij^2)."""
        A = np.abs(self.Ls)
        E = 3 * 4e-6 * (A @ A.T)
        dg = np.diag(E).copy()
        np.fill_diagonal(E, 0.0)
        return (dg.max() + 3 * np.sqrt((E ** 2).sum(1)).max()) / self.normH


# ---------------------------------------------------------------------------- module problem
class Problem:
    def __init__(self, eng):
        self.eng = eng
        X, Y = make_host_data()
        self.Xh, self.Yh = X, Y
        self.X = torch.as_tensor(X, device=eng.device)
        self.Y = torch.as_tensor(Y, device=eng.device)
        X64, Y64 = self.X.double(), self.Y.double()
        G, B = X64.T @ X64, X64.T @ Y64                # cuBLAS, not this library
        sx, sy = X64.sum(0), Y64.sum(0)
        self.G, self.B, self.sx, self.sy = (t.contiguous() for t in (G, B, sx, sy))
        self.Gh, self.Bh, self.sxh, self.syh = (t.cpu().numpy() for t in (G, B, sx, sy))
        self._g, self._ref, self._sel = {}, {}, {}

    def g(self, n, mode=0):
        """Statistics dict for engine.ls_solve / ls_factor with the first n targets; mode selects the solver's
        tensor-core flag (ls_solve and ls_factor set it from the dict)."""
        if n not in self._g:
            self._g[n] = dict(G=self.G, B=self.B[:, :n].contiguous(), sx=self.sx, sy=self.sy[:n].contiguous(), N=N,
                              K=K, n=n)
        return dict(self._g[n], mode=mode)

    def sel(self, kp, extra=()):
        key = (kp, tuple(extra))
        if key not in self._sel:
            s = selection(kp, extra)
            self._sel[key] = (s, torch.as_tensor(s, device=self.eng.device))
        return self._sel[key]

    def ref(self, kp, n, extra=()):
        """Reference on selection(kp, extra) for the first n targets (computed once for the largest n asked for in
        this module: the right-hand sides are solved independently, so a smaller n is a slice)."""
        key = (kp, tuple(extra))
        nmax = max(n, NMAX.get(kp, 64))
        if key not in self._ref or self._ref[key].n < n:
            self._ref[key] = Ref(self.Gh, self.Bh, self.sxh, self.syh, self.sel(kp, extra)[0], nmax)
        return self._ref[key].sliced(n) if n < self._ref[key].n else self._ref[key]


@pytest.fixture(scope="module")
def P(_engine_session):
    return Problem(_engine_session)


@pytest.fixture(autouse=True)
def fp64_solver(engine):
    """The engine fixture resets only the Gram mode; the solver's tensor-core flag stays on a handle from whatever ran
    before.  Every test here starts and ends with it off, and a test that wants it on says so."""
    engine.ls_tensor_cores(False)
    yield
    engine.ls_tensor_cores(False)


def _np(*ts):
    return tuple(t.cpu().numpy() for t in ts)


# ---------------------------------------------------------------------------- schedule coverage
# K' -> what chol_factor (PB = 128-wide panels, GB = 512-wide groups, panels paired (e, o)) reaches first at that size:
SCHEDULE = [
    45,     # one panel of 45 columns: sub-panels 32 + 13, the other 83 rows padded with the identity
    128,    # one whole panel, nothing after it
    129,    # a second panel of one column: crit update 1 wide
    200,    # crit only (second panel 72 wide; far_a needs more than 256 columns)
    300,    # far_a(0) 44 wide on the side stream, and the half-group merge (the third panel starts at 256)
    384,    # far_a(0) a whole panel wide, pair merge (0, 1), half-group merge over a whole third panel
    500,    # near(0, 1) 116 wide: under the 192 columns a product needs for the tensor cores
    512,    # one whole group: pair merges (0, 1), (2, 3), half-group merge; near(0, 1) 128 wide
    513,    # a second group of one column: its own 1 x 1 inverse block, a second substitution step
    600,    # near(0, 1) 216 wide (>= 192: tensor-core eligible once it has 256 rows, i.e. n >= 40)
    700,    # near2(0, 1), columns 640..699
    900,    # rest(0, 1) on the bulk stream (4 columns), and near2(2, 3) waiting for it on ev_bulk
    1100,   # rest(0, 1) 204 wide: tensor-core eligible; groups 0, 1 and a 76-column third
    1536,   # three whole groups
    2304,   # everything, eight rest updates and their bulk waits; four whole groups and a half one
]
NVAR = {513: (1, 7, 300), 1100: (1, 7, 300), 2304: (1, 7, 300)}   # n = 300: over subst_update's 256 threshold
NMAX = {kp: max(v) for kp, v in NVAR.items()}
SOLVE_CASES = [(kp, 64) for kp in SCHEDULE] + [(kp, n) for kp, ns in NVAR.items() for n in ns]


@pytest.mark.parametrize("kp,n", SOLVE_CASES)
def test_solve_matches_host_reference(engine, P, kp, n):
    sel, sel_d = P.sel(kp)
    W, b, info, stat = engine.ls_solve(P.g(n), sel_d)
    assert int(info.cpu()[0]) == 0
    P.ref(kp, n).check(*_np(W, b), "solve")


@pytest.mark.parametrize("kp", [45, 513, 700, 1100, 2304])
def test_factor_then_resolve_matches_host_reference(engine, P, kp):
    """cp_ls_factor builds the factor with no right-hand side; cp_ls_resolve then runs both substitutions for
    whatever n it is given (here 300 and 7), and accumulate = 1 adds its solution to what the outputs hold."""
    sel, sel_d = P.sel(kp)
    info, stat = engine.ls_factor(P.g(0), sel_d)
    assert int(info.cpu()[0]) == 0
    for n in (300, 7):
        g = P.g(n)
        W, b = engine.ls_resolve(g["B"], g["sx"], g["sy"], sel_d)
        P.ref(kp, n).check(*_np(W, b), "resolve")
    W0 = torch.randn(7, kp, dtype=torch.float64, device=engine.device)
    b0 = torch.randn(7, dtype=torch.float64, device=engine.device)
    Wa, ba = W0.clone(), b0.clone()
    engine.ls_resolve(g["B"], g["sx"], g["sy"], sel_d, accumulate_into=(Wa, ba))
    assert torch.equal(Wa, W0 + W) and torch.equal(ba, b0 + b)   # the same IEEE sum, element by element


# ---------------------------------------------------------------------------- tensor-core dispatch
def tc_runs(kp, n_factor, n_subst):
    """Whether a product of a factorisation with n_factor right-hand-side rows, followed by substitutions for n_subst
    right-hand sides, takes the tensor cores when the handle's flag is on.  dgemm sends a product there when its
    column count Nn >= 192, its row count M >= 256 and 128 <= R <= 1024; subst_update asks for that when n >= 256 and
    Nn >= 512.
      * factorisation: far_a is at most one panel (128) wide, so only the pair updates near / near2 / rest qualify.
        The first that can be 192 wide is near(0, 1): columns 384 .. min(K', 640), rows K' + n_factor - 384.  When it
        does not qualify, K' < 576 (nothing later is 192 wide) or K' + n_factor < 640 (nothing later exists).
      * backward substitution: the updates of groups g >= 1 have Nn = 512 g and R = the group's width, so with
        n >= 256 one qualifies once a second group is 128 wide: K' >= 640;
      * forward substitution (cp_ls_resolve): Nn = K' - 512 (g + 1), R = 512: K' >= 1024, which the above covers."""
    return (kp >= 576 and kp + n_factor >= 640) or (n_subst >= 256 and kp >= 640)


TC_CASES = [(45, 300), (512, 300), (513, 300), (575, 300), (576, 64), (600, 7), (600, 64), (638, 1), (639, 1),
            (700, 64), (1100, 64), (1100, 300), (2304, 300)]


@pytest.mark.parametrize("kp,n", TC_CASES)
def test_tensor_core_mode_solve(engine, P, kp, n):
    """Same bits as fp64 mode where no product qualifies; elsewhere different bits (the split-precision kernel ran)
    within the error model plus the tensor cores' backward-error term (Ref.tc_beta)."""
    sel, sel_d = P.sel(kp)
    W0, b0, _, s0 = engine.ls_solve(P.g(n, 0), sel_d)
    W1, b1, info, s1 = engine.ls_solve(P.g(n, 1), sel_d)
    assert int(info.cpu()[0]) == 0
    if not tc_runs(kp, n, n):
        assert torch.equal(W0, W1) and torch.equal(b0, b1) and torch.equal(s0, s1)
        return
    assert not torch.equal(W0, W1)
    ref = P.ref(kp, n)
    ref.check(*_np(W1, b1), "tc solve", extra_beta=ref.tc_beta())


@pytest.mark.parametrize("kp,n", [(639, 64), (640, 64), (640, 300), (1100, 300)])
def test_tensor_core_mode_resolve(engine, P, kp, n):
    """A factor built without right-hand sides: its own boundary is K' >= 640 (near(0, 1) needs 256 matrix rows)."""
    sel, sel_d = P.sel(kp)
    g = P.g(n)
    out = []
    for mode in (0, 1):
        info, _ = engine.ls_factor(P.g(0, mode), sel_d)
        assert int(info.cpu()[0]) == 0
        out.append(engine.ls_resolve(g["B"], g["sx"], g["sy"], sel_d))
    (W0, b0), (W1, b1) = out
    if not tc_runs(kp, 0, n):
        assert torch.equal(W0, W1) and torch.equal(b0, b1)
        return
    assert not torch.equal(W0, W1)
    ref = P.ref(kp, n)
    ref.check(*_np(W1, b1), "tc resolve", extra_beta=ref.tc_beta())


# ---------------------------------------------------------------------------- state, determinism, defaults
def test_kept_factor_survives_other_work(engine, P):
    """The factor lives in the handle's own allocation: cp_gram, cp_gemm_f64, a dual solve that grows the scratch and
    cp_ls_residual in between change nothing of what cp_ls_resolve computes from it."""
    sel, sel_d = P.sel(1100)
    g = P.g(300)
    info, _ = engine.ls_factor(P.g(0), sel_d)
    assert int(info.cpu()[0]) == 0
    Wa, ba = engine.ls_resolve(g["B"], g["sx"], g["sy"], sel_d)
    engine.gram(P.X[:, :900], P.Y[:, :64], mode=0)
    A = torch.randn(300, 200, dtype=torch.float64, device=engine.device)
    engine.mm_nt(A, A)
    dsel = torch.arange(2200, dtype=torch.int32, device=engine.device)
    _, _, dinfo, _ = engine.ls_solve_dual(P.X[:1800], P.Y[:1800], None, dsel)
    engine.ls_residual(P.X, P.Y[:, :300], None, sel_d, Wa, ba, mode=0)
    Wb, bb = engine.ls_resolve(g["B"], g["sx"], g["sy"], sel_d)
    assert int(dinfo.cpu()[0]) == 0
    assert torch.equal(Wa, Wb) and torch.equal(ba, bb)


@pytest.mark.parametrize("mode", [0, 1], ids=["fp64", "tc"])
def test_solve_is_deterministic(engine, P, mode):
    sel, sel_d = P.sel(1100)
    first = engine.ls_solve(P.g(300, mode), sel_d)
    second = engine.ls_solve(P.g(300, mode), sel_d)
    for x, y in zip(first, second):
        assert torch.equal(x, y)


def test_null_selection_is_every_column(engine, P):
    sel, _ = P.sel(700)
    sub = dict(P.g(64), K=700)
    sub["G"] = P.G[sel][:, sel].contiguous()
    sub["B"] = P.B[sel, :64].contiguous()
    sub["sx"] = P.sx[sel].contiguous()
    a = engine.ls_solve(sub, None)
    b = engine.ls_solve(sub, torch.arange(700, dtype=torch.int32, device=engine.device))
    for x, y in zip(a, b):
        assert torch.equal(x, y)


# ---------------------------------------------------------------------------- pivot status
def _stats_with(P, edits):
    """The module statistics with column dst made an exact copy of column src (src >= 0) or all zero (src < 0)."""
    G, B, sx = P.Gh.copy(), P.Bh.copy(), P.sxh.copy()
    for dst, src in edits:
        if src >= 0:
            G[dst, :], B[dst], sx[dst] = G[src, :], B[src], sx[src]
            G[:, dst] = G[:, src]
        else:
            G[dst, :], G[:, dst], B[dst], sx[dst] = 0.0, 0.0, 0.0, 0.0
    d = P.eng.device
    return dict(G=torch.as_tensor(G, device=d), B=torch.as_tensor(B[:, :64].copy(), device=d),
                sx=torch.as_tensor(sx, device=d), sy=P.sy[:64].contiguous(), N=N, K=K, n=64)


# (selection index j made a copy of selection index i; i = -1: all zero), K' = 700: groups 0 and 1, last panel 60 wide
PIVOT_CASES = {
    "first_panel": [(50, 10)],
    "second_group": [(530, 100)],
    "last_partial_panel": [(680, 600)],
    "two_duplicates": [(530, 7), (300, 5)],
    "zero_column": [(200, -1)],
}


@pytest.mark.parametrize("case", list(PIVOT_CASES))
def test_failed_pivot_reports_its_index_and_a_tiny_ratio(engine, P, case):
    sel, sel_d = P.sel(700)
    g = _stats_with(P, [(int(sel[j]), int(sel[i]) if i >= 0 else -1) for j, i in PIVOT_CASES[case]])
    first = min(j for j, _ in PIVOT_CASES[case])
    W, b, info, stat = engine.ls_solve(dict(g, mode=0), sel_d)
    info, stat = int(info.cpu()[0]), float(stat.cpu()[0])
    print("%s: info %d stat %.3e" % (case, info, stat))
    assert info == first + 1
    assert 0.0 < stat <= 1e-12
    info_f, stat_f = engine.ls_factor(dict(g, mode=0), sel_d)
    assert int(info_f.cpu()[0]) == first + 1 and 0.0 < float(stat_f.cpu()[0]) <= 1e-12


def test_tensor_core_mode_catches_a_duplicate(engine, P):
    """The 22-bit updates may lift the duplicate's pivot above 1e-12 of its diagonal, but never to a ratio the
    acceptance policy (engine.settle_ls) would keep: it re-solves when info != 0 or stat < LS_RATIO_MIN."""
    import cpb200

    assert cpb200.engine.LS_RATIO_MIN == LS_RATIO_MIN
    sel, sel_d = P.sel(1100)
    g = _stats_with(P, [(int(sel[1000]), int(sel[20]))])
    _, _, info, stat = engine.ls_solve(dict(g, mode=1), sel_d)
    info, stat = int(info.cpu()[0]), float(stat.cpu()[0])
    print("tc duplicate: info %d stat %.3e" % (info, stat))
    assert info != 0 or stat < LS_RATIO_MIN


def _pivot_sensitivity(Ls):
    """s_k = 1 + |H11^-1 h_k|^2 per pivot k, H11 the columns before k: a perturbation dH of H moves pivot k by at most
    |dH| s_k (pivot_k = h_kk - h_k' H11^-1 h_k).  H11^-1 h_k = L11^-T l_k, l_k the row of the factor."""
    Li = scipy.linalg.solve_triangular(Ls, np.eye(Ls.shape[0]), lower=True)
    s = np.ones(Ls.shape[0])
    for k in range(1, Ls.shape[0]):
        s[k] += np.sum((Li[:k, :k].T @ Ls[k, :k]) ** 2)
    return s


@pytest.mark.parametrize("kp,extra", [(200, ()), (1100, ()), (2304, ()), (700, (NPLAIN + 1,)), (700, (NPLAIN + 3,))],
                         ids=["200", "1100", "2304", "700-collinear-1e-2", "700-collinear-1e-6"])
def test_pivot_ratio_matches_host_factor(engine, P, kp, extra):
    """stat against the exact ratios min_k L_kk^2 / Gc_kk of the host factor.  Device and host pivots each differ
    from the exact ones by at most |dH| s_k, |dH| = |H| beta (the backward error of the model above): so stat lies in
    [min_k (p_k - 2 |H| beta s_k), p_k* + 2 |H| beta s_k*], k* the host's smallest pivot."""
    if extra:
        extra = extra + (COLLIN[extra[0]][0],)
    sel, sel_d = P.sel(kp, extra)
    ref = P.ref(kp, 64, extra)
    W, b, info, stat = engine.ls_solve(P.g(64), sel_d)
    assert int(info.cpu()[0]) == 0
    stat = float(stat.cpu()[0])
    s = _pivot_sensitivity(ref.Ls)
    dev = 2 * ref.normH * (4 * kp * U + ref.eta_asm) * s
    k = int(np.argmin(ref.pivots))
    lo, hi = (ref.pivots - dev).min(), ref.pivots[k] + dev[k]
    print("K'=%d: stat %.6e host %.6e  |diff| %.2e / %.2e" % (kp, stat, ref.ratio, abs(stat - ref.ratio), dev[k]))
    assert lo <= stat <= hi
    if extra:
        assert k == list(sel).index(extra[0])  # the collinear column is the smallest pivot, as built


# ---------------------------------------------------------------------------- dual (minimum-norm) path
@pytest.mark.parametrize("nr,kp", [(300, 500), (300, 450), (700, 900), (700, 1050), (1100, 1300), (1100, 1650)])
def test_dual_solve_is_minimum_norm_and_always_fp64(engine, P, nr, kp):
    """K' > N - 1: cp_ls_solve_dual against gelsd's minimum-norm answer (oracle linear_regression), bit-identical
    whether or not the handle's tensor-core flag is on.  Error model: the dual system H = Xc Xc' + 11'/N is built in
    fp64 (K' terms) and factored (N terms), a backward error eta <= (4N + K' + 4) u |(|Xc||Xc|')| / |Xc|^2 (the +4:
    the column means); then W = Xc' H^-1 Yc moves by at most |dH| |A| / s_min <= eta kappa(Xc)^2 |W| per target, since
    |A| <= |W| / s_min on the rows' space (A is orthogonal to 1, the one direction Xc' removes)."""
    sel = selection(kp)
    sel_d = torch.as_tensor(sel, device=engine.device)
    X = P.X[:nr]
    Xs = P.Xh[:nr][:, sel].astype(np.float64)
    Xc = Xs - Xs.mean(0)
    sv = np.linalg.svd(Xc, compute_uv=False)
    kap2 = (sv[0] / sv[nr - 2]) ** 2                       # rank N - 1: the centred rows sum to zero
    A = np.abs(Xc)
    eta = (4 * nr + kp + 4) * U * (A @ (A.T @ np.ones(nr))).max() / sv[0] ** 2
    rb = kap2 * eta
    r = np.random.RandomState(nr + kp)
    for ydt, with_bias in ((torch.float32, False), (torch.float64, True)):
        Y = P.Y[:nr, :16].to(ydt).contiguous()
        if ydt == torch.float64:
            Y = Y + torch.as_tensor(1e-3 * r.standard_normal((nr, 16)), device=engine.device)  # not fp32 values
        bias = torch.as_tensor((0.1 * r.standard_normal(16)).astype(np.float32), device=engine.device) if with_bias \
            else None
        engine.ls_tensor_cores(False)
        off = engine.ls_solve_dual(X, Y, bias, sel_d)
        engine.ls_tensor_cores(True)
        on = engine.ls_solve_dual(X, Y, bias, sel_d)
        engine.ls_tensor_cores(False)
        assert int(off[2].cpu()[0]) == 0
        for a, b in zip(off, on):
            assert torch.equal(a, b), "the dual solve depends on the tensor-core flag"
        Yh = Y.cpu().numpy().astype(np.float64)
        if bias is not None:
            Yh = Yh - bias.cpu().numpy().astype(np.float64)
        coef, icpt = O.linear_regression(Xs, Yh)
        W, b = _np(off[0], off[1])
        ew = np.linalg.norm(W - coef, axis=1) / np.linalg.norm(coef, axis=1)
        xm, ym = Xs.mean(0), Yh.mean(0)
        bb = np.linalg.norm(xm) * rb * np.linalg.norm(coef, axis=1) + 2 * (kp + 2) * U * (
            np.abs(ym) + np.abs(W) @ np.abs(xm))
        eb = np.abs(b - icpt)
        print("dual N=%d K'=%d %s: kappa(Xc)^2 %.0f  W %.2e / %.2e  b %.2e / %.2e" % (
            nr, kp, "f64+bias" if with_bias else "f32", kap2, ew.max(), rb, eb.max(), bb[np.argmax(eb / bb)]))
        assert rb < 1e-3 and (ew <= rb).all() and (eb <= bb).all()


# ---------------------------------------------------------------------------- residual
def _residual(engine, X, Y, bias, sel_d, W, b, mode, ldr):
    """cp_ls_residual into an (N, ldr) buffer whose columns n.. must stay untouched."""
    n = Y.shape[1]
    R = torch.full((X.shape[0], ldr), -7.0, dtype=torch.float32, device=engine.device)
    engine._call(engine.lib.cp_ls_residual(
        engine.h, engine._p(X, "const float*"), X.shape[0], X.shape[1], X.stride(0), engine._p(Y, "const void*"),
        0 if Y.dtype == torch.float32 else 1, n, Y.stride(0), engine._p(bias, "const float*"),
        engine._p(sel_d, "const int32_t*"), W.shape[1], engine._p(W, "const double*"), engine._p(b, "const double*"),
        engine._p(R, "float*"), ldr, mode, engine._s()))
    assert bool((R[:, n:] == -7.0).all())
    return R[:, :n].cpu().numpy()


# name -> (rows, columns, selected (None: all), n, f64 targets, y_bias, ldr); mode 1 runs on the tensor cores only
# with rows % 4 == 0, rows >= 128, columns >= 64 and n % 4 == 0, and falls back to the fp64 path otherwise
RESIDUAL_CASES = {
    "f32": (2700, 2400, 1100, 64, False, False, 64),
    "f64_bias_ldr": (2700, 2400, 700, 60, True, True, 68),
    "k4608_split": (512, 4608, None, 32, False, True, 32),
    "k27": (1000, 27, None, 64, False, False, 72),
    "n_not_4": (2700, 2400, 1100, 62, False, True, 64),
    "rows_not_4": (2699, 2400, 1100, 64, True, False, 64),
}


@pytest.mark.parametrize("case", list(RESIDUAL_CASES))
def test_residual_matches_host(engine, P, case):
    """Mode 0: fp64 products and sums, rounded once to fp32: |R - r| <= half an fp32 ulp of r + 2 delta (the half ulp
    is the rounding itself, reached wherever r lies near a midpoint of two fp32 values), delta =
    (K' + 3) u (|y| + |bias| + sum_j |x_j||w_j| + |b|) the fp64 evaluation error (here and on the host).
    Mode 1 on the tensor cores: + 4e-6 sum_j |x_j||w_j| (split operands, fp32 accumulators, weights rounded to fp32);
    mode 1 where it falls back: the same bits as mode 0."""
    nr, kc, ks, n, f64, with_bias, ldr = RESIDUAL_CASES[case]
    r = np.random.RandomState(nr + kc + n)
    if kc == K:
        X, Xh = P.X[:nr], P.Xh[:nr]
        Yh = P.Yh[:nr, :n].astype(np.float64)
    else:
        Xh = np.maximum(r.standard_normal((nr, kc)), 0).astype(np.float32)
        X = torch.as_tensor(Xh, device=engine.device)
        Yh = r.standard_normal((nr, n)).astype(np.float32).astype(np.float64)
    if f64:
        Yh = Yh + 1e-3 * r.standard_normal(Yh.shape)
    sel = selection(ks) if ks else np.arange(kc, dtype=np.int32)
    sel_d = torch.as_tensor(sel, device=engine.device) if ks else None
    Wh = r.standard_normal((n, len(sel))) / np.sqrt(len(sel))
    bh = r.standard_normal(n)
    biash = (0.1 * r.standard_normal(n)).astype(np.float32) if with_bias else None
    Y = torch.as_tensor(Yh if f64 else Yh.astype(np.float32), device=engine.device)
    W, b = torch.as_tensor(Wh, device=engine.device), torch.as_tensor(bh, device=engine.device)
    bias = torch.as_tensor(biash, device=engine.device) if with_bias else None
    y0 = Yh - (biash.astype(np.float64) if with_bias else 0.0)
    Xs = Xh[:, sel].astype(np.float64)
    ref = y0 - Xs @ Wh.T - bh
    S = np.abs(Xs) @ np.abs(Wh).T
    delta = (len(sel) + 3) * U * (np.abs(y0) + S + np.abs(bh))
    half_ulp = 0.5 * np.spacing((np.abs(ref) + 2 * delta).astype(np.float32)).astype(np.float64)
    R0 = _residual(engine, X, Y, bias, sel_d, W, b, 0, ldr)
    e0 = np.abs(R0 - ref)
    b0 = half_ulp + 2 * delta
    R1 = _residual(engine, X, Y, bias, sel_d, W, b, 1, ldr)
    tc = nr % 4 == 0 and nr >= 128 and kc >= 64 and n % 4 == 0
    msg = "residual %s: mode 0 %.2e of its bound" % (case, (e0 / b0).max())
    if tc:
        e1, b1 = np.abs(R1 - ref), half_ulp + 2 * delta + 4e-6 * S
        msg += ", mode 1 (tensor cores) %.2e of its bound, %.2e of 4e-6 sum|x||w|" % ((e1 / b1).max(),
                                                                                  (e1 / (4e-6 * S)).max())
    print(msg)
    assert (e0 <= b0).all()
    if tc:
        assert (e1 <= b1).all() and not np.array_equal(R0, R1)
    else:
        assert np.array_equal(R0, R1)


# ---------------------------------------------------------------------------- refinement (the pipeline's contract)
@pytest.mark.parametrize("extra", [(), (NPLAIN + 0,), (NPLAIN + 1,), (NPLAIN + 2,)],
                         ids=["ratio-0.5", "ratio-0.06", "ratio-0.012", "ratio-0.006"])
def test_refined_tensor_core_solve_meets_the_pipeline_bound(engine, P, extra):
    """What reconstruct_async does with tensor-core statistics: cp_gram mode 1, ls_solve with the tensor-core flag,
    one ls_refine.  Every case here has an exact pivot ratio above LS_RATIO_MIN, so settle_ls keeps it: the refined W
    must meet the pipeline's 1e-4 relative bound (test_gpu_fullsize.py), and the refinement must reduce the error."""
    if extra:
        extra = extra + (COLLIN[extra[0]][0],)
    sel, sel_d = P.sel(1100, extra)
    ref = P.ref(1100, 300, extra)
    Y = P.Y[:, :300]
    g = engine.gram(P.X, Y, mode=1)
    assert g["mode"] == 1
    W, b, info, stat = engine.ls_solve(g, sel_d)
    W0, b0 = _np(W, b)
    engine.ls_refine(g, P.X, Y, None, sel_d, W, b)
    W1, b1 = _np(W, b)
    rel = lambda Wx: np.linalg.norm(Wx - ref.W) / np.linalg.norm(ref.W)  # noqa: E731
    relb = lambda bx: np.abs(bx - ref.b).max() / max(1.0, np.abs(ref.b).max())  # noqa: E731
    stat = float(stat.cpu()[0])
    print("refine: exact ratio %.4f stat %.4f  W %.2e -> %.2e  b %.2e -> %.2e" % (
        ref.ratio, stat, rel(W0), rel(W1), relb(b0), relb(b1)))
    assert ref.ratio > LS_RATIO_MIN and (ref.ratio < 0.0075 if extra and extra[0] == NPLAIN + 2 else True)
    assert int(info.cpu()[0]) == 0 and stat >= LS_RATIO_MIN
    assert rel(W1) <= 1e-4 and relb(b1) <= 1e-4
    assert rel(W1) < rel(W0)
