"""GPU: the LASSO channel search (cp_lasso_select) bit for bit against its executable specification, and the channel
statistics it reads (cp_lasso_build) against exact arithmetic.

The search's specification is oracle/cd_oracle.c:cp_enet_cd_gram driven by the alpha search of lib/decompose.py:489-525
(model_search below).  Every search case launches the kernel twice (the two launches must agree to the bit) and compares
the coefficients, the selection, the scalars and every probe-log row with the model, bit for bit.  Each case names the
kernel path it reaches; the end-to-end parity tests cannot see such paths go wrong, because they compare selections,
not coefficients."""
import ctypes
import math
from fractions import Fraction

import numpy as np
import pytest

import cp_oracle as O

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

U = Fraction(1, 2 ** 53)  # unit roundoff of float64


# ---------------------------------------------------------------------------- the model and the kernel
def model_search(Q, ldq, qv, yn2, m, rank, lbound, rbound, right0, seeds, tol=1e-4, max_iter=1000):
    """The alpha search of lib/decompose.py:489-525 over cp_enet_cd_gram, with cp_lasso_select's probe cap: once
    len(seeds) fits have run, the search stops with status 1 and the last fit's coefficients.  Q: c rows ldq doubles
    apart.  Returns the kernel's outputs (coef, idxs, scalars, probe_log) and, per fit, the warm start it began from
    (starts: (w, Qw) pairs)."""
    lib = O._clib()
    c = len(qv)
    Qf = np.ascontiguousarray(Q, dtype=np.float64).reshape(-1)
    assert Qf.size >= (c - 1) * ldq + c
    qv = np.ascontiguousarray(qv, dtype=np.float64)
    w, Qw = np.zeros(c), np.zeros(c)  # Qw = Q w, carried between fits like the kernel does
    gap, tol_s = ctypes.c_double(), ctypes.c_double()
    log, starts = [], []

    def solve(a):
        starts.append((w.copy(), Qw.copy()))
        it = lib.cp_enet_cd_gram(O._dp(w), O._dp(Qw), a * m, O._dp(Qf), ldq, O._dp(qv), yn2, c, max_iter, tol,
                                 int(seeds[len(log)]), 1, 1, ctypes.byref(gap), ctypes.byref(tol_s))
        log.append((a, np.count_nonzero(w), it, gap.value))
        return log[-1][1]

    left, right, alpha, nnz, status = 0.0, right0, right0, 0, 0
    while True:  # :502-515
        if len(log) >= len(seeds):
            status = 1
            break
        alpha = right
        nnz = solve(right)
        if nnz < rank:
            break
        right *= 2
    while status == 0:  # :516-525
        if len(log) >= len(seeds):
            status = 1
            break
        alpha = (left + right) / 2
        nnz = solve(alpha)
        if nnz > rbound:
            left = alpha
        elif nnz < lbound:
            right = alpha
        else:
            break
    return dict(coef=w, idxs=(w != 0).astype(np.uint8), scalars=np.array([alpha, len(log), status, nnz], np.float64),
                probe_log=np.array(log, np.float64).reshape(-1, 4), starts=starts)


def device_search(engine, Qd, qd, yd, m, rank, lbound, rbound, right0, seeds, tol=1e-4, max_iter=1000):
    """cp_lasso_select on device tensors (Qd: c x c, rows Qd.stride(0) apart); host copies of its outputs."""
    res = engine.lasso_select(Qd, qd, yd, m, rank, lbound, rbound, right0, seeds, tol=tol, max_iter=max_iter)
    return dict(coef=res.coef.cpu().numpy(), idxs=res.idxs.cpu().numpy(), scalars=res.scalars.cpu().numpy(),
                probe_log=res.probe_log.cpu().numpy())


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int64) if a.dtype == np.float64 else a


def assert_bits(got, want, what):
    """Bit equality (so -0 and +0 differ); the message shows the first differing values."""
    got, want = np.ascontiguousarray(got), np.ascontiguousarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    diff = np.flatnonzero(_bits(got) != _bits(want))
    assert diff.size == 0, "%s: %d of %d differ, first at %s: %r != %r" % (
        what, diff.size, got.size, np.unravel_index(diff[0], got.shape), got.flat[diff[0]], want.flat[diff[0]])


def check_search(engine, Qd, qd, yd, m, rank, lbound, rbound, right0, seeds, tol=1e-4, max_iter=1000):
    """Two launches and the model on the very bytes the kernel read; every output bit for bit.  Returns
    (kernel outputs, model outputs)."""
    args = (m, rank, lbound, rbound, right0, seeds, tol, max_iter)
    got = device_search(engine, Qd, qd, yd, *args)
    again = device_search(engine, Qd, qd, yd, *args)
    for key in got:
        assert_bits(again[key], got[key], "second launch: " + key)
    c, ldq = Qd.shape[0], Qd.stride(0)
    Qh = Qd.as_strided((c, ldq), (ldq, 1)).cpu().numpy()  # the rows as the kernel reads them, padding included
    ref = model_search(Qh, ldq, qd.cpu().numpy(), float(yd.cpu()[0]), *args)
    n = int(ref["scalars"][1])
    assert_bits(got["probe_log"][:n], ref["probe_log"], "probe log (alpha, nnz, n_iter, gap)")
    assert not got["probe_log"][n:].any()
    assert_bits(got["scalars"], ref["scalars"], "scalars (alpha, n_probes, status, nnz)")
    assert_bits(got["coef"], ref["coef"], "coef")
    assert_bits(got["idxs"], ref["idxs"], "idxs")
    return got, ref


# ---------------------------------------------------------------------------- problems
def synthetic(c, seed, zrank=None, m=None, dead=(), dup=()):
    """Centred statistics (Q, qv, yn2, m) of a correlated design Z (m x c) = F M with zrank latent factors (by default
    c/2 < zrank < c, so Q is singular), and y = Z w + noise.  Columns in dead are zero (dead ReLU channels); a pair
    (a, b) in dup makes column b an exact copy of column a.  Q is exactly symmetric (upper triangle mirrored)."""
    r = np.random.RandomState(seed)
    zr = zrank or max(1, min(c - 1, 3 * c // 4))
    m = m or c + 32
    Z = r.standard_normal((m, zr)) @ (r.standard_normal((zr, c)) + 0.5)
    for a, b in dup:
        Z[:, b] = Z[:, a]
    Z[:, list(dead)] = 0.0
    noise = 0.3 * (Z.std() or 1.0) * r.standard_normal(m)
    y = Z @ (r.standard_normal(c) * np.exp(-np.arange(c) / (0.3 * c + 1))) + noise
    Zc, yc = Z - Z.mean(0), y - y.mean()
    Q = Zc.T @ Zc
    Q = np.triu(Q) + np.triu(Q, 1).T
    return Q, Zc.T @ yc, float(yc @ yc), float(m)


def to_device(engine, Q, qv, yn2, ldq=None):
    """Device copies; Q as a c x c view of rows ldq apart (zero padding)."""
    c = Q.shape[0]
    ldq = ldq or c + (c & 1)
    Qp = np.zeros((c, ldq))
    Qp[:, :c] = Q
    dev = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device=engine.device)
    return dev(Qp)[:, :c], dev(qv), dev(np.array([yn2]))


def alpha_max(qv, m):
    """The smallest alpha at which w = 0 is optimal: max |q| / m."""
    return float(np.abs(qv).max()) / m


def seeds_for(seed, n=48):
    return np.random.RandomState(seed).randint(0, 2 ** 31 - 1, n)


def window(rank, rank_tol=0.1):
    import cpb200

    return cpb200.engine.window(rank, rank_tol)


def first_screen_evictions(Q, qv, yn2, w, Qw, l1, tol):
    """Nonzero coefficients of a warm start (w, Qw) that the first gap-safe screening of a fit at l1 sets to zero:
    cp_enet_cd_gram's gap (cd_oracle.c:198-213, the warp-order sums) and screening (:229-242) restated in the same
    float64 operations.  0 when the fit returns at its first gap check."""
    c = len(qv)
    w, Qw, qv = [float(v) for v in w], [float(v) for v in Qw], [float(v) for v in qv]

    def warp_sum(terms):  # 32 strided partial sums, then a 5-level butterfly
        p = [0.0] * 32
        for i, t in enumerate(terms):
            p[i % 32] += t
        for off in (16, 8, 4, 2, 1):
            p = [p[l] + p[l ^ off] for l in range(32)]
        return p[0]

    q_dot_w = warp_sum(w[i] * qv[i] for i in range(c))
    wQw = warp_sum(w[i] * Qw[i] for i in range(c))
    R_norm2 = yn2 + wQw - 2.0 * q_dot_w
    Ry = yn2 - q_dot_w
    XtA = [qv[j] - Qw[j] for j in range(c)]
    dn = 0.0
    for a in XtA:
        dn = abs(a) if abs(a) > dn else dn
    primal = 0.5 * (R_norm2 + 0.0) + l1 * warp_sum(abs(v) for v in w)
    scale = l1 / dn if dn > l1 else 1.0
    gap = primal - (-0.5 * (scale * scale) * (R_norm2 + 0.0) + scale * Ry)
    if gap <= tol * yn2:
        return 0
    radius = math.sqrt(2 * abs(gap)) / l1
    den = l1 if l1 > dn else dn
    out = 0
    for j in range(c):
        Qjj = float(Q[j][j])
        if Qjj != 0 and w[j] != 0 and (1 - abs(XtA[j] / den)) / math.sqrt(Qjj) > radius:
            out += 1
    return out


# ---------------------------------------------------------------------------- pipeline input
def pipeline_inputs(c, k2, n, N, S, seed):
    """A layer problem as the pipeline holds it: post-ReLU X (N, c*k2) fp32 with correlated channels and taps, W2
    (n, c*k2) fp32, float64 targets Y with an fp32 bias, S sampled rows (with repeats)."""
    r = np.random.RandomState(seed)
    K = c * k2
    lat = max(4, K // 3)
    X = np.maximum(r.standard_normal((N, lat)) @ (r.standard_normal((lat, K)) / np.sqrt(lat)) + 0.2, 0)
    X = X.astype(np.float32)
    W2 = (r.standard_normal((n, K)) * np.sqrt(2.0 / K)).astype(np.float32)
    Y = X.astype(np.float64) @ W2.T.astype(np.float64)
    Y += 0.05 * Y.std() * r.standard_normal(Y.shape)
    bias = (0.1 * r.standard_normal(n)).astype(np.float32)
    samples = r.randint(0, N, S).astype(np.int32)
    return X, W2, Y + bias.astype(np.float64), bias, samples


def pipeline_statistics(engine, X, W2, Y, bias, samples, c, k2):
    """(gs, gw, W2m, Q, qv, yn2) on the device, built as Engine.select_channels_async builds them."""
    from cpb200.engine import GRAM_FP64

    dev = lambda a: torch.as_tensor(np.ascontiguousarray(a), device=engine.device)
    W2m = dev(W2)
    gs = engine.gram(dev(X), dev(Y), y_bias=dev(bias), rows=dev(samples), want_yy=True, mode=GRAM_FP64)
    gw = engine.gram(W2m, None, want_B=False, mode=GRAM_FP64)
    Q, qv, yn2 = engine.lasso_build(gs, gw, W2m, c, k2, len(samples))
    return gs, gw, W2m, Q, qv, yn2


@pytest.mark.parametrize("k2,c,n", [(1, 96, 16), (9, 64, 16), (27, 40, 8)], ids=["k1", "k3x3", "k3x3x3"])
def test_search_on_the_pipelines_own_statistics(engine, k2, c, n):
    """Q, qv, yn2 straight from cp_gram + cp_lasso_build.  The builder sums the k2^2 products of Q[a, b] in a's tap
    order and those of Q[b, a] in b's, so for k2 > 1 Q is not bitwise symmetric: the search must read each entry
    where its model does (the delta of step s-k applied to Qw[j_s] through row j_{s-k})."""
    X, W2, Y, bias, samples = pipeline_inputs(c, k2, n, N=3000, S=400, seed=100 + k2)
    _, _, _, Q, qv, yn2 = pipeline_statistics(engine, X, W2, Y, bias, samples, c, k2)
    Qh = Q.cpu().numpy()
    if k2 == 1:
        assert_bits(Qh, Qh.T, "k2 = 1: every entry is one rounded product, Q is symmetric")
    else:
        assert (Qh != Qh.T).any(), "expected a Q that is not bitwise symmetric"
    rank = int(0.8 * c)
    lb, rb = window(rank)
    got, _ = check_search(engine, Q, qv, yn2, float(len(samples) * n), rank, lb, rb, 1e-3, seeds_for(k2))
    assert got["scalars"][2] == 0 and lb <= got["scalars"][3] <= rb


# ---------------------------------------------------------------------------- variant edges
# NPB = 1, 2, 4, 8 at c <= 256, 512, 1024, 2048; c < 16 (one guarded chain block), < LAG + 1 = 5, < 32 (one packager
# batch), > 64 (the per-step rings wrap), and MAXC = 2048
@pytest.mark.parametrize("c", [1, 2, 3, 5, 17, 33, 65, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025, 2047, 2048])
def test_search_at_the_variant_edges(engine, c):
    Q, qv, yn2, m = synthetic(c, seed=c)
    rank = max(1, c // 2)  # below the rank of Z (about 3c/4), so the window is reachable
    lb, rb = window(rank)
    got, _ = check_search(engine, *to_device(engine, Q, qv, yn2), m, rank, lb, rb, alpha_max(qv, m) / 8,
                          seeds_for(c))
    assert got["scalars"][2] == 0


# ---------------------------------------------------------------------------- degenerate channels
def test_search_with_dead_channels(engine):
    """Zero columns (dead ReLU channels): the first screening of every fit excludes them (zero diagonal)."""
    c = 70
    dead = list(range(0, c, 7)) + [c - 1]
    Q, qv, yn2, m = synthetic(c, seed=3, dead=dead)
    rank = 30
    lb, rb = window(rank)
    got, _ = check_search(engine, *to_device(engine, Q, qv, yn2), m, rank, lb, rb, alpha_max(qv, m) / 8, seeds_for(3))
    assert not got["coef"][dead].any()


@pytest.mark.parametrize("live", [[23], [5, 23]], ids=["one", "two"])
def test_search_with_few_live_channels(engine, live):
    """All channels but one or two dead.  One active coordinate: every sweep is a single chain step.  Two: about half
    the steps draw the coordinate of the step before, whose w the chain warp prefetched before it changed."""
    c = 40
    Q, qv, yn2, m = synthetic(c, seed=4, dead=[j for j in range(c) if j not in live])
    rank = len(live)
    got, _ = check_search(engine, *to_device(engine, Q, qv, yn2), m, rank, rank, rank + 0.1, alpha_max(qv, m) / 64,
                          seeds_for(4))
    assert got["scalars"][2] == 0 and np.flatnonzero(got["coef"]).tolist() == live


def test_search_with_every_channel_dead(engine):
    """Q = 0, q = 0: every fit returns at its first gap check (n_iter = 0, gap = 0) with nnz = 0; the window [0, 0.1]
    accepts the first bisection probe."""
    c = 36
    Q, qv, yn2, m = synthetic(c, seed=5, dead=range(c))
    assert not Q.any() and not qv.any() and yn2 > 0
    got, _ = check_search(engine, *to_device(engine, Q, qv, yn2), m, 1, 0.0, 0.1, 1e-3, seeds_for(5))
    log = got["probe_log"][:int(got["scalars"][1])]
    assert got["scalars"].tolist() == [5e-4, 2, 0, 0]
    assert not log[:, 1:].any()


def test_search_with_duplicated_channels(engine):
    """Exactly duplicated columns: identical rows and columns of Q, ties in every screening decision."""
    c = 64
    Q, qv, yn2, m = synthetic(c, seed=6, dup=[(0, 1), (5, 40), (5, 41), (63, 62)])
    rank = 32
    lb, rb = window(rank)
    check_search(engine, *to_device(engine, Q, qv, yn2), m, rank, lb, rb, alpha_max(qv, m) / 8, seeds_for(6))


# ---------------------------------------------------------------------------- search paths
def test_search_doubling_from_far_below(engine):
    """right0 twelve doublings below max|q|/m: the first loop runs a chain of fits, each warm-started from the denser
    solution of the one before."""
    c = 96
    Q, qv, yn2, m = synthetic(c, seed=7)
    rank = 20
    lb, rb = window(rank)
    got, _ = check_search(engine, *to_device(engine, Q, qv, yn2), m, rank, lb, rb, alpha_max(qv, m) / 2 ** 12,
                          seeds_for(7))
    alphas = got["probe_log"][:8, 0]
    assert_bits(alphas, alphas[0] * 2.0 ** np.arange(8), "eight fits of the doubling loop")


def test_search_evicting_warm_starts(engine):
    """right0 just below max|q|/m: the first fit keeps a few coefficients barely above the threshold, and at the
    doubled alpha the first screening evicts them (Qw corrected row by row).  A doubling from further below leaves a
    gap too large for the safe region to exclude a nonzero coefficient."""
    c = 120
    Q, qv, yn2, m = synthetic(c, seed=22)
    _, ref = check_search(engine, *to_device(engine, Q, qv, yn2), m, 1, 1, 1.1, 0.9 * alpha_max(qv, m), seeds_for(22))
    evicted = [first_screen_evictions(Q, qv, yn2, w, Qw, a * m, 1e-4)
               for (w, Qw), a in zip(ref["starts"], ref["probe_log"][:, 0])]
    assert sum(evicted) > 0, evicted


def test_search_starting_at_an_optimum(engine):
    """right0 >= max|q|/m: w = 0 is optimal, so the first fit returns at its first gap check (n_iter = 0)."""
    c = 48
    Q, qv, yn2, m = synthetic(c, seed=8)
    rank = 24
    lb, rb = window(rank)
    got, _ = check_search(engine, *to_device(engine, Q, qv, yn2), m, rank, lb, rb, alpha_max(qv, m) * 1.5,
                          seeds_for(8))
    assert got["probe_log"][0, 1:3].tolist() == [0, 0]


@pytest.mark.parametrize("max_iter", [1, 2, 3])
def test_search_with_a_sweep_cap(engine, max_iter):
    """max_iter sweeps per fit: the capped fits end with a gap check and a screening after every sweep."""
    c = 80
    Q, qv, yn2, m = synthetic(c, seed=9)
    rank = 40
    lb, rb = window(rank)
    got, _ = check_search(engine, *to_device(engine, Q, qv, yn2), m, rank, lb, rb, alpha_max(qv, m) / 8,
                          seeds_for(9 + max_iter), max_iter=max_iter)
    assert (got["probe_log"][:int(got["scalars"][1]), 2] == max_iter).any()


@pytest.mark.parametrize("tol", [1e-2, 1e-7])
def test_search_at_loose_and_tight_tolerance(engine, tol):
    c = 72
    Q, qv, yn2, m = synthetic(c, seed=10)
    rank = 36
    lb, rb = window(rank)
    check_search(engine, *to_device(engine, Q, qv, yn2), m, rank, lb, rb, alpha_max(qv, m) / 8, seeds_for(10), tol=tol)


@pytest.mark.parametrize("rank", [1, 47, 48], ids=["one", "c-1", "c"])
def test_search_for_extreme_ranks(engine, rank):
    """Keep one channel, all but one, or all of them (full-rank Z, so small alphas keep every channel)."""
    c = 48
    Q, qv, yn2, m = synthetic(c, seed=11, zrank=c, m=4 * c)
    lb, rb = window(rank)
    got, _ = check_search(engine, *to_device(engine, Q, qv, yn2), m, rank, lb, rb, alpha_max(qv, m) / 64,
                          seeds_for(11))
    assert got["scalars"][2] == 0 and lb <= got["scalars"][3] <= rb


def test_search_for_an_unreachable_window(engine):
    """No integer lies in [rank + 0.2, rank + 0.4]: the search runs into the probe cap (status 1) and returns the
    last fit's coefficients."""
    c = 300
    Q, qv, yn2, m = synthetic(c, seed=12)
    seeds = seeds_for(12, 14)
    got, _ = check_search(engine, *to_device(engine, Q, qv, yn2), m, 150, 150.2, 150.4, alpha_max(qv, m) / 8, seeds)
    assert got["scalars"][1:3].tolist() == [len(seeds), 1]


def test_search_with_edge_seeds(engine):
    """Seeds 0 (which the xorshift maps to 1), 1, 2^31 - 2 and repeated values; seed 0 and seed 1 give the same
    search."""
    c = 40
    Q, qv, yn2, m = synthetic(c, seed=13)
    rank = 20
    lb, rb = window(rank)
    dev = to_device(engine, Q, qv, yn2)
    args = (m, rank, lb, rb, alpha_max(qv, m) / 8)
    check_search(engine, *dev, *args, np.array([0, 1, 2 ** 31 - 2, 7, 7, 7, 0, 2 ** 31 - 2] * 6))
    zeros = device_search(engine, *dev, *args, np.zeros(48, np.int64))
    ones = device_search(engine, *dev, *args, np.ones(48, np.int64))
    for key in zeros:
        assert_bits(zeros[key], ones[key], "seed 0 against seed 1: " + key)


# ---------------------------------------------------------------------------- layout
@pytest.mark.parametrize("c,ldq", [(37, 38), (40, 46)], ids=["odd_c", "padded"])
def test_search_with_padded_rows(engine, c, ldq):
    """Rows of Q ldq apart with zero padding (the model is given the same ldq)."""
    Q, qv, yn2, m = synthetic(c, seed=14 + c)
    rank = 20
    lb, rb = window(rank)
    Qd, qd, yd = to_device(engine, Q, qv, yn2, ldq=ldq)
    assert Qd.stride(0) == ldq
    check_search(engine, Qd, qd, yd, m, rank, lb, rb, alpha_max(qv, m) / 8, seeds_for(14))


# ---------------------------------------------------------------------------- checks without the model
@pytest.mark.parametrize("c", [24, 130])
def test_search_is_invariant_under_powers_of_four(engine, c):
    """Scaling Q, qv, yn2 and right0 by s = 4^k scales every intermediate of the search by s, s^(1/2) = 2^k or 1, and
    correctly rounded + - * / sqrt commute exactly with such scalings (far from overflow and underflow): coef, idxs,
    nnz and n_iter are unchanged to the bit, the logged alphas and gaps scale exactly."""
    Q, qv, yn2, m = synthetic(c, seed=15)
    rank = c // 2
    lb, rb = window(rank)
    right0 = alpha_max(qv, m) / 8
    base = device_search(engine, *to_device(engine, Q, qv, yn2), m, rank, lb, rb, right0, seeds_for(15))
    n = int(base["scalars"][1])
    for s in (4.0 ** 20, 4.0 ** -20):
        got = device_search(engine, *to_device(engine, Q * s, qv * s, yn2 * s), m, rank, lb, rb, right0 * s,
                            seeds_for(15))
        assert_bits(got["coef"], base["coef"], "coef")
        assert_bits(got["idxs"], base["idxs"], "idxs")
        assert_bits(got["scalars"], base["scalars"] * np.array([s, 1, 1, 1]), "scalars")
        assert_bits(got["probe_log"][:n], base["probe_log"][:n] * np.array([s, 1, 1, s]), "probe log")


def _two_prod(a, b):
    """(p, e) with p + e = a * b exactly (Dekker's product, elementwise on float64 arrays)."""
    def split(x):
        t = 134217729.0 * x
        hi = t - (t - x)
        return hi, x - hi

    p = a * b
    ah, al = split(a)
    bh, bl = split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _dot(a, b):
    """Correctly rounded a . b: exact products summed by math.fsum."""
    p, e = _two_prod(np.asarray(a, np.float64), np.asarray(b, np.float64))
    return math.fsum(np.concatenate([p, e]))


def duality_gap(Q, qv, yn2, w, l1):
    """The duality gap of the fit's problem at w (gap_enet with dual_gap_formulation_A), with Q w and every dot
    product correctly rounded and the rest in exact rational arithmetic."""
    c = len(qv)
    Qw = np.array([_dot(Q[j], w) for j in range(c)])
    qw, wQw = Fraction(_dot(qv, w)), Fraction(_dot(w, Qw))
    R_norm2 = Fraction(yn2) + wQw - 2 * qw
    Ry = Fraction(yn2) - qw
    dn = max(abs(Fraction(float(a)) - Fraction(float(b))) for a, b in zip(qv, Qw))
    l1 = Fraction(l1)
    primal = R_norm2 / 2 + l1 * sum(abs(Fraction(float(v))) for v in w)
    scale = l1 / dn if dn > l1 else Fraction(1)
    return float(primal - (-scale * scale * R_norm2 / 2 + scale * Ry))


@pytest.mark.parametrize("c,tol", [(17, 1e-4), (65, 1e-4), (65, 1e-7), (257, 1e-4)])
def test_every_converged_fit_is_optimal(engine, c, tol):
    """The kernel alone: launched with the probe cap at p it returns the coefficients of its p-th fit.  Every fit that
    stopped on its gap (n_iter < max_iter) has a duality gap, recomputed from (Q, qv, yn2, w), within tol * yn2 and
    equal to the logged one up to the rounding of the kernel's carried Q w and its sums: 4 c u (yn2 + |q| |w| +
    |w|' |Q| |w|).  The accepted selection lies in the window."""
    Q, qv, yn2, m = synthetic(c, seed=16 + c)
    rank = max(1, c // 3)
    lb, rb = window(rank)
    dev = to_device(engine, Q, qv, yn2)
    seeds = seeds_for(16)
    args = (m, rank, lb, rb, alpha_max(qv, m) / 8)
    full = device_search(engine, *dev, *args, seeds, tol=tol)
    assert full["scalars"][2] == 0 and lb <= full["scalars"][3] <= rb
    n = int(full["scalars"][1])
    tol_s = tol * yn2
    for p in range(1, n + 1):
        got = device_search(engine, *dev, *args, seeds[:p], tol=tol) if p < n else full
        alpha, nnz, n_iter, gap = got["probe_log"][p - 1]
        assert (alpha, nnz, n_iter, gap) == tuple(full["probe_log"][p - 1])
        w = got["coef"]
        assert np.count_nonzero(w) == nnz
        if n_iter >= 1000:
            continue
        aw = np.abs(w)
        allowance = 4 * c * 2.0 ** -53 * (yn2 + np.abs(qv) @ aw + aw @ np.abs(Q) @ aw)
        exact = duality_gap(Q, qv, yn2, w, alpha * m)
        assert gap <= tol_s and exact <= tol_s + allowance, (p, gap, exact, tol_s)
        assert abs(exact - gap) <= allowance, (p, gap, exact, allowance)


# ---------------------------------------------------------------------------- cp_lasso_build against exact arithmetic
def _ints(a):
    """Float64 values as exact integers: a == ints * 2**e."""
    mant, ex = np.frexp(np.asarray(a, np.float64).ravel())
    mant = (mant * 2.0 ** 53).astype(np.int64)
    e = int(ex.min()) - 53
    return [int(v) << int(s) for v, s in zip(mant, ex - 53 - e)], e


def exact_dot(a, b):
    """sum a_i b_i of two float64 arrays, exactly."""
    ai, ea = _ints(a)
    bi, eb = _ints(b)
    return Fraction(sum(x * y for x, y in zip(ai, bi))) * Fraction(2) ** (ea + eb)


def exact_sum(a):
    ai, e = _ints(a)
    return Fraction(sum(ai)) * Fraction(2) ** e


def gamma(n):
    """Higham's gamma_n = n u / (1 - n u): the bound on the relative error of n successive roundings."""
    return n * U / (1 - n * U)


def exact_build(Gs, Bs, sxs, sys_, yys, WW, sw, W2, c, k2, n, m, entries):
    """Q[a, b] for (a, b) in entries, qv and yn2 in exact arithmetic from the float64 statistics the kernel read, with
    bounds on the error of cp_lasso_build's float64 evaluation: a chain of f fused multiply-adds, a tree of t
    additions, each rounding at most u relative, so the computed sum is within gamma_(f + t) of the exact one
    relative to the sum of the magnitudes of its terms (Higham, Accuracy and Stability, 3.1 and 3.5)."""
    mm = Fraction(m)
    za = [exact_dot(sxs[a * k2:(a + 1) * k2], sw[a * k2:(a + 1) * k2]) for a in range(c)]
    Za = [exact_dot(np.abs(sxs[a * k2:(a + 1) * k2]), np.abs(sw[a * k2:(a + 1) * k2])) for a in range(c)]
    Q = {}
    for a, b in entries:
        g = Gs[a * k2:(a + 1) * k2, b * k2:(b + 1) * k2]
        w = WW[a * k2:(a + 1) * k2, b * k2:(b + 1) * k2]
        # s: k2^2 fmas; za, zb: k2 fmas each, then a product, a division and the subtraction
        bound = gamma(k2 * k2 + 1) * exact_dot(np.abs(g), np.abs(w)) + gamma(2 * k2 + 3) * Za[a] * Za[b] / mm
        Q[a, b] = (exact_dot(g, w) - za[a] * za[b] / mm, bound)
    ysum, Ysum = exact_sum(sys_), exact_sum(np.abs(sys_))
    chain = -(-k2 * n // 128) + 7  # per-thread fma chains of a 128-thread block, then a 7-level tree
    qv = []
    for a in range(c):
        wa = W2[:, a * k2:(a + 1) * k2].T.astype(np.float64)  # (k2, n) like Bs[(a, p), j]
        ba = Bs[a * k2:(a + 1) * k2, :]
        bound = gamma(chain + 1) * exact_dot(np.abs(wa), np.abs(ba)) + gamma(k2 + n + 2) * Za[a] * Ysum / mm
        qv.append((exact_dot(wa, ba) - za[a] * ysum / mm, bound))
    yn2 = (Fraction(float(yys)) - ysum * ysum / mm, gamma(2 * n + 1) * (Fraction(float(yys)) + Ysum * Ysum / mm))
    return Q, qv, yn2


# every k2 the builder meets (1x1, 2x2 / 4x1 / 1x4, 1x7 / 7x1, 3x3, 4x4, 5x5, 3x3x3, 7x7) and each of n, S and c
# with at least two of them
@pytest.mark.parametrize("k2,n,S,c", [(1, 1, 1, 130), (4, 3, 2, 1), (7, 64, 400, 3), (9, 64, 400, 130),
                                      (16, 1, 400, 17), (25, 3, 1, 17), (27, 64, 2, 130), (49, 3, 400, 17)])
def test_lasso_build_against_exact_arithmetic(engine, k2, n, S, c):
    X, W2, Y, bias, samples = pipeline_inputs(c, k2, n, N=max(2 * S, 64), S=S, seed=200 + k2)
    gs, gw, W2m, Q, qv, yn2 = pipeline_statistics(engine, X, W2, Y, bias, samples, c, k2)
    h = {k: v.cpu().numpy() for k, v in dict(Gs=gs["G"], Bs=gs["B"], sxs=gs["sx"], sys_=gs["sy"], WW=gw["G"],
                                                sw=gw["sx"]).items()}
    yys = float(gs["yy"].cpu()[0])
    r = np.random.RandomState(k2)
    if c <= 17:
        entries = [(a, b) for a in range(c) for b in range(c)]
    else:
        entries = [(0, 0), (0, c - 1), (c - 1, 0), (c - 1, c - 1)] + list(zip(r.randint(0, c, 196), r.randint(0, c, 196)))
    m = S * n
    eQ, eq, ey = exact_build(yys=yys, W2=W2, c=c, k2=k2, n=n, m=m, entries=entries, **h)
    Qh, qh, yh = Q.cpu().numpy(), qv.cpu().numpy(), float(yn2.cpu()[0])
    for (a, b), (want, bound) in eQ.items():
        assert abs(Fraction(float(Qh[a, b])) - want) <= bound, ("Q", a, b, float(Qh[a, b]), float(want), float(bound))
    for a, (want, bound) in enumerate(eq):
        assert abs(Fraction(float(qh[a])) - want) <= bound, ("qv", a, float(qh[a]), float(want), float(bound))
    assert abs(Fraction(yh) - ey[0]) <= ey[1], ("yn2", yh, float(ey[0]), float(ey[1]))
    # padding: a wider Q buffer full of NaN gets the same c columns and exact zeros after them
    ldq = c + (c & 1) + 6
    Qw = torch.full((c, ldq), float("nan"), dtype=torch.float64, device=engine.device)
    qw, yw = engine.empty(c), engine.empty(1)
    engine._call(engine.lib.cp_lasso_build(
        engine.h, *[engine._p(t, "const double*") for t in (gs["G"], gs["B"], gs["sx"], gs["sy"], gs["yy"], gw["G"],
                                                             gw["sx"])],
        engine._p(W2m, "const float*"), c, k2, n, S, engine._p(Qw, "double*"), ldq, engine._p(qw, "double*"),
        engine._p(yw, "double*"), engine._s()))
    Qw = Qw.cpu().numpy()
    assert_bits(Qw[:, :c], Qh, "Q in a wider buffer")
    assert_bits(Qw[:, c:], np.zeros((c, ldq - c)), "padding columns")
    assert_bits(qw.cpu().numpy(), qh, "qv")
    assert_bits(yw.cpu().numpy(), yn2.cpu().numpy(), "yn2")
