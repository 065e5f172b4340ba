"""GPU: cp_gram's statistics in both arithmetic modes, the fp64 product driver behind them (cpgemm::product, which
also runs cp_gemm_f64) and cp_colstats_f64, against exact statistics.

Exact data.  Entries are m_col + d with integer column offsets |m_col| < 2^10 and integer deviations |d| <= 7 that
sum to zero in each column (they come in pairs +d, -d, each column permuted on its own).  Targets Y are built the same
way and y_bias is integer-valued.  Then every operation of both modes is exact, the statistics have one correct
value, and the tests require equality with it (value equality: a zero may carry either sign):
  * fp64 mode: products of such fp32 values are exact in fp64 and every sum stays far below 2^53.
  * tensor-core mode: the column sum is exactly N m, so the shift fl32(t (1/N)) is exactly m for any N; xs = d is
    exact; v = d 2^e (|v| < 2^10) fits the fp16 hi half with lo = 0; every product hi_i hi_j is a multiple of
    2^(e_i + e_j) no larger than 49 of those units, so a 64-row stage (< 2^12 units) and a split of at most 4096 rows
    (< 2^18 units) stay far below 2^24 units and every fp32 accumulation is exact whatever its rounding; the fp64 split
    sums, the exact rescale by 2^-(e_i + e_j), T = 0, SQ and the undo N m_i m_j are exact.
  * the reference, float64 BLAS on the same integer-valued data, is exact for the same reason.
exact_data asserts these preconditions on the data each test generates.

Emulation (part 3).  gram_tc_model.tc_prep reproduces the tensor-core mode's operand preparation bit for bit on data
whose fp64 column sums are exact (entries on the 2^-12 grid, |x| < 2^8, columns summing to N m with m on the grid),
and tc_model takes the three products hi'hi + hi'lo + lo'hi in float64 BLAS.  The tensor-core result must then lie
within tau(nst) inv_i inv_j A_ij of the model (gram_tc_model.tau: 12 truncating wgmma adds per 64-row stage within
2 ulp each, then nst round-to-nearest adds per split; about 2^-17.2 at 64 stages), plus an fp64-level term.  Dropping
one of the three products moves an entry by about 2^-11 A, far outside the bound.  On unstructured data the result
must also lie within that bound plus the split and shift-rounding model error of X'X, computed in long double.

Scale invariance (part 4).  Scaling X by 2^kx and Y by 2^ky scales G, B, sx and sy exactly in both modes for as long
as the data stays normal fp32 and x - mean finite: the tensor-core mode's shift, column exponent and operands move
with the scale and its hi/lo halves keep their bits.

Branch coverage.  gram_tc_model.product_plan and tc_plan restate the split policies; the *_reach_every_branch tests
assert that the parametrisations below reach every branch of cpgemm::product and of cp_gram_tc2, on this device's SM
count."""
import numpy as np
import pytest

import gram_tc_model as M

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

F32, F64 = 0, 1
NAN = float("nan")


def _sms(eng):
    return torch.cuda.get_device_properties(eng.device).multi_processor_count


def _gen(eng, seed):
    g = torch.Generator(device=eng.device)
    g.manual_seed(seed)
    return g


def _nan(eng, numel, off=0, dtype=torch.float64):
    """NaN-filled device buffer of numel elements starting `off` elements into its allocation (off = 1: 8 bytes off a
    16-byte boundary for doubles, 4 bytes for floats)."""
    return torch.full((numel + off,), NAN, dtype=dtype, device=eng.device)[off:]


def _place(eng, A, ld, off, dtype):
    """A (rows x cols) copied into a NaN-padded buffer with leading dimension ld, `off` elements into the allocation;
    returns (flat view passed to the kernel, 2-D view of the valid part)."""
    rows, cols = A.shape
    flat = _nan(eng, max(rows * ld, 1), off, dtype)
    view = flat[:rows * ld].view(rows, ld)[:, :cols]
    view.copy_(A)
    return flat, view


def _same_bits(a, b):
    a, b = a.contiguous(), b.contiguous()
    assert a.shape == b.shape
    return torch.equal(a.view(torch.int64), b.view(torch.int64))


def raw_gram(eng, X, N, K, ldx, Y=None, y_dtype=F32, n=0, ldy=0, y_bias=None, rows=None, nrows=0, G=None, B=None,
             sx=None, sy=None, yy=None, mode=0):
    p = eng._p
    eng._call(eng.lib.cp_gram(eng.h, p(X, "const float*"), N, K, ldx, p(Y, "const void*"), y_dtype, n, ldy,
                              p(y_bias, "const float*"), p(rows, "const int32_t*"), nrows, p(G, "double*"),
                              p(B, "double*"), p(sx, "double*"), p(sy, "double*"), p(yy, "double*"), mode, eng._s()))


def exact_data(eng, gen, N, K, moff=1023, dmax=7):
    """(m + d) as float64 on the device (N x K): |m| <= moff integer column offsets, integer deviations |d| <= dmax in
    +-pairs (a zero row when N is odd), rows permuted per column.  Asserts the exactness preconditions."""
    dev = eng.device
    m = torch.randint(-moff, moff + 1, (K,), generator=gen, device=dev, dtype=torch.int64)
    h = N // 2
    d = torch.randint(-dmax, dmax + 1, (h, K), generator=gen, device=dev, dtype=torch.int64)
    d = torch.cat([d, -d, torch.zeros((N - 2 * h, K), dtype=torch.int64, device=dev)])
    if N > 1:
        d = torch.gather(d, 0, torch.argsort(torch.rand(N, K, generator=gen, device=dev), dim=0))
    assert moff < 2 ** 10 and dmax <= 7
    assert int(d.abs().max()) <= dmax if N else True
    assert bool((d.sum(0) == 0).all())
    return (m + d).to(torch.float64)


# ------------------------------------------------------------------ part 1: exact statistics
def _sym_fill_K(sms):
    t = 1
    while t * (t + 1) // 2 < 2 * sms:
        t += 1
    return 128 * t


# name: N, K, n, options.  outs: requested outputs; ldx/ldy: None = packed; xoff/yoff/coff: elements off a 16-byte
# boundary; rows: None, ("repeat", nrows) or "empty" (a valid pointer and nrows = 0); y64: fp64 targets.
FP64_CASES = {
    "sym-unsplit-short-R": dict(N=50, K=300, n=7, bias=True),
    "sym-unsplit-tiles": dict(N=200, K="fill", n=0, outs=("G", "sx")),
    "K128-split-rows": dict(N=1000, K=128, n=1, bias=True),
    "K129-mirror-split-rows": dict(N=5000, K=129, n=129, bias=True),
    "K640-split-tiles-tail": dict(N=20007, K=640, n=300),
    "n128": dict(N=4096, K=256, n=128, bias=True),
    "rows-repeat": dict(N=3000, K=96, n=5, bias=True, rows=("repeat", 4001), outs=("G", "B", "sx", "sy", "yy")),
    "rows-empty": dict(N=500, K=70, n=3, bias=True, rows="empty", outs=("G", "B", "sx", "sy", "yy")),
    "N0": dict(N=0, K=40, n=3, outs=("G", "B", "sx", "sy", "yy")),
    "y64-odd-ldy": dict(N=777, K=100, n=9, y64=True, ldy=11, bias=True, outs=("G", "B", "sx", "sy", "yy")),
    "x-misaligned-ldx": dict(N=1500, K=150, ldx=153, xoff=1, n=20),
    "outputs-misaligned": dict(N=900, K=200, n=130, coff=1, bias=True),
    "G-only": dict(N=2000, K=257, n=0, outs=("G",)),
    "B-only": dict(N=2000, K=64, n=200, outs=("B",)),
    "sx-only": dict(N=3001, K=77, n=0, outs=("sx",)),
    "sy-yy-without-B": dict(N=1234, K=64, n=33, bias=True, outs=("sy", "yy")),
}

# tensor-core mode: shapes across the 64-row stage, the 4096-row split cap, the 32-way preparation split, partial and
# multiple 128-tiles of X and of Y, and persistent-grid loads from below one item per SM to many per CTA
TC_CASES = {
    "N64-K64-n1": dict(N=64, K=64, n=1, bias=True),
    "N65-K65-n3": dict(N=65, K=65, n=3),
    "N127-K127-n4": dict(N=127, K=127, n=4, bias=True),
    "N4095-K128-n127": dict(N=4095, K=128, n=127, bias=True),
    "N4096-K129-n128": dict(N=4096, K=129, n=128),
    "N4097-K257-n129": dict(N=4097, K=257, n=129, bias=True),
    "N12289-K1000-n200": dict(N=12289, K=1000, n=200, bias=True),
    "N50000-K257-n3": dict(N=50000, K=257, n=3, bias=True),
    "N4097-K2304-n200": dict(N=4097, K=2304, n=200, bias=True),
    "N12289-K64-G-only": dict(N=12289, K=64, n=0, outs=("G", "sx")),
    "N4096-K1000-n129-G-null": dict(N=4096, K=1000, n=129, bias=True, outs=("B", "sx", "sy")),
}


def _tc_ld(v):
    return (v + 3) // 4 * 4


def _resolve(case, sms, tc):
    c = dict(case)
    if c["K"] == "fill":
        c["K"] = _sym_fill_K(sms)
    c.setdefault("outs", ("G", "B", "sx", "sy") if c["n"] else ("G", "sx"))
    c.setdefault("ldx", _tc_ld(c["K"]) if tc else c["K"])
    c.setdefault("ldy", _tc_ld(c["n"]) if tc else c["n"])
    return c


def _features(c):
    f = set()
    if c.get("rows") == "empty":
        f.add("nrows-0")
    elif c.get("rows"):
        f.add("rows-repeat")
    if c["N"] == 0:
        f.add("N-0")
    if c.get("bias"):
        f.add("y-bias")
    if c.get("y64") and c["ldy"] % 2:
        f.add("y-f64-odd-ldy")
    if c["ldx"] > c["K"]:
        f.add("ldx>K")
    if c.get("xoff"):
        f.add("x-misaligned")
    if c.get("coff"):
        f.add("outputs-misaligned")
    o = set(c["outs"])
    for name, s in (("G-only", {"G"}), ("B-only", {"B"}), ("sx-only", {"sx"}), ("sy+yy-without-B", {"sy", "yy"})):
        if o == s:
            f.add(name)
    if "G" in o and c["K"] in (128, 129):
        f.add("sym-K%d" % c["K"])
    return f


def _fp64_branches(c, sms):
    R = c["N"] if not c.get("rows") else (c["rows"][1] if c["rows"] != "empty" else 0)
    br = set()
    if "G" in c["outs"]:
        br |= M.product_plan(c["K"], c["K"], R, True, sms)["branches"]
    if "B" in c["outs"]:
        br |= M.product_plan(c["K"], c["n"], R, False, sms)["branches"]
    return br | _features(c)


def _is_tc(c):
    o = set(c["outs"])
    return M.tc_routes(c["N"], c["K"], c["ldx"], not c.get("xoff"), "f64" if c.get("y64") else "f32", c["n"], c["ldy"],
                       not c.get("yoff"), bool(c.get("rows")), "B" in o, "sy" in o, "yy" in o)


def run_exact(eng, c, mode, seed):
    """One cp_gram call on exact data, through the C ABI with the case's strides and offsets; every output must equal
    the float64 reference, and G its own transpose bit for bit."""
    gen = _gen(eng, seed)
    N, K, n = c["N"], c["K"], c["n"]
    X = exact_data(eng, gen, N, K)
    Xf, _ = _place(eng, X.float(), c["ldx"], c.get("xoff", 0), torch.float32)
    assert torch.equal(Xf[:N * c["ldx"]].view(N, c["ldx"])[:, :K].double(), X) if N else True
    Y = Yf = yb = rows = None
    ydt = torch.float64 if c.get("y64") else torch.float32
    if n:
        Y = exact_data(eng, gen, N, n)
        Yf, _ = _place(eng, Y.to(ydt), c["ldy"], c.get("yoff", 0), ydt)
        if c.get("bias"):
            yb = torch.randint(-300, 301, (n,), generator=gen, device=eng.device).float()
    nrows = 0
    if c.get("rows") == "empty":
        rows = torch.zeros(1, dtype=torch.int32, device=eng.device)
    elif c.get("rows"):
        nrows = c["rows"][1]
        rows = torch.randint(0, N, (nrows,), generator=gen, device=eng.device, dtype=torch.int32)
        assert rows.unique().numel() < nrows  # repeats
    off = c.get("coff", 0)
    o = set(c["outs"])
    outs = dict(G=_nan(eng, K * K, off) if "G" in o else None, B=_nan(eng, K * n, off) if "B" in o else None,
                sx=_nan(eng, K, off) if "sx" in o else None, sy=_nan(eng, n, off) if "sy" in o else None,
                yy=_nan(eng, 1, off) if "yy" in o else None)
    raw_gram(eng, Xf if N else _nan(eng, 4, 0, torch.float32), N, K, c["ldx"], Yf, F64 if c.get("y64") else F32, n,
             c["ldy"], yb, rows, nrows, mode=mode, **outs)
    Xr = X[rows.long()] if (rows is not None and nrows) else (X[:0] if rows is not None else X)
    ref = dict(G=Xr.T @ Xr, sx=Xr.sum(0))
    if n:
        Yr = Y[rows.long()] if (rows is not None and nrows) else (Y[:0] if rows is not None else Y)
        Yc = Yr - (yb.double() if yb is not None else 0.0)
        ref.update(B=Xr.T @ Yc, sy=Yc.sum(0), yy=(Yc * Yc).sum().reshape(1))
    torch.cuda.synchronize()
    for k, v in outs.items():
        if v is None:
            continue
        got = v.view(ref[k].shape)
        bad = ~(got == ref[k])
        assert not bool(bad.any()), "%s: %d of %d entries differ from the exact statistic (first %s)" % (
            k, int(bad.sum()), bad.numel(), bad.nonzero()[:3].tolist())
    if outs["G"] is not None:
        G = outs["G"].view(K, K)
        assert _same_bits(G, G.T)
    return outs


def test_fp64_cases_reach_every_product_branch(engine):
    sms = _sms(engine)
    reached = set()
    for name, case in FP64_CASES.items():
        c = _resolve(case, sms, False)
        br = _fp64_branches(c, sms)
        print("%-24s %s" % (name, " ".join(sorted(br))))
        reached |= br
    need = {"sym:split", "sym:unsplit", "sym:mirror", "all:split", "all:unsplit", "sym:split-cap-rows",
            "sym:split-cap-tiles", "all:split-cap-tiles", "sym:unsplit-short-R", "all:unsplit-short-R",
            "sym:unsplit-tiles", "reduction-tail", "register-staged", "rows-repeat", "nrows-0", "N-0", "y-bias",
            "y-f64-odd-ldy", "ldx>K", "x-misaligned", "outputs-misaligned", "G-only", "B-only", "sx-only",
            "sy+yy-without-B", "sym-K128", "sym-K129"}
    assert need <= reached, sorted(need - reached)


def test_tc_cases_reach_every_tensor_core_branch(engine):
    sms = _sms(engine)
    reached = set()
    for name, case in TC_CASES.items():
        c = _resolve(case, sms, True)
        assert _is_tc(c), name
        o = set(c["outs"])
        br = M.tc_plan(c["N"], c["K"], c["n"], "G" in o, "B" in o, sms, c.get("bias", False))["branches"]
        print("%-26s %s" % (name, " ".join(sorted(br))))
        reached |= br
    need = {"tc:diag-tile", "tc:offdiag-tile", "tc:y-tile", "tc:G-null", "tc:y-tile-partial", "tc:y-bias",
            "tc:row-tile-partial", "tc:stage-padded", "tc:split", "tc:unsplit", "tc:split-cap-4096",
            "tc:prep-multi-tile", "tc:prep-32-splits", "tc:grid-below-sms", "tc:items-per-cta>1",
            "tc:mixed-diag-offdiag-per-cta"}
    assert need <= reached, sorted(need - reached)
    assert {64, 65, 127, 128, 129, 257, 1000, 2304} <= {c["K"] for c in TC_CASES.values()}
    assert {1, 3, 4, 127, 128, 129, 200} <= {c["n"] for c in TC_CASES.values()}
    assert {64, 65, 127, 4095, 4096, 4097, 12289, 50000} <= {c["N"] for c in TC_CASES.values()}


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("name", list(FP64_CASES))
def test_gram_exact_statistics(engine, name, mode):
    """Every fp64-product branch; in mode 1 the same calls either fall back to those products or (when eligible)
    run the tensor cores, exact either way on this data."""
    c = _resolve(FP64_CASES[name], _sms(engine), False)
    run_exact(engine, c, mode, seed=sum(map(ord, name)) + mode)


@pytest.mark.parametrize("name", list(TC_CASES))
def test_gram_tc_exact_statistics(engine, name):
    c = _resolve(TC_CASES[name], _sms(engine), True)
    assert _is_tc(c)
    run_exact(engine, c, 1, seed=sum(map(ord, name)))


@pytest.mark.parametrize("mode", [0, 1])
def test_gram_exact_after_nan_scratch(engine, mode):
    """A large call on NaN-containing data leaves NaN in the handle's scratch (split partials, operands, column
    statistics); a smaller exact call on the same handle must not pick any of it up."""
    gen = _gen(engine, 77)
    N, K, n = (12289, 1000, 200) if mode else (20007, 640, 300)
    X = torch.randn(N, K, generator=gen, device=engine.device)
    X[::7, ::3] = NAN
    Y = torch.randn(N, n, generator=gen, device=engine.device)
    Y[::5, ::2] = NAN
    g = engine.gram(X, Y, mode=mode)
    torch.cuda.synchronize()
    assert bool(torch.isnan(g["G"]).any())
    c = _resolve(dict(N=4097, K=129, n=128, bias=True), _sms(engine), True)
    run_exact(engine, c, mode, seed=78)
    c = _resolve(dict(N=1000, K=128, n=1, bias=True), _sms(engine), False)
    run_exact(engine, c, mode, seed=79)


@pytest.mark.parametrize("mode", [0, 1])
def test_gram_is_deterministic(engine, mode):
    gen = _gen(engine, 90 + mode)
    N, K, n = 12289, 1000, 200
    X = torch.randn(N, K, generator=gen, device=engine.device)
    Y = torch.randn(N, n, generator=gen, device=engine.device)
    b = torch.randn(n, generator=gen, device=engine.device)
    a = engine.gram(X, Y, y_bias=b, mode=mode)
    c = engine.gram(X, Y, y_bias=b, mode=mode)
    for k in ("G", "B", "sx", "sy"):
        assert _same_bits(a[k], c[k]), k


# ------------------------------------------------------------------ part 2: which path a mode-1 call takes
ROUTES = {
    # name: (tensor cores expected, call options)
    "rows": (False, dict(rows=True)),
    "N<64": (False, dict(N=63)),
    "K<64": (False, dict(K=63, ldx=64)),
    "X-misaligned": (False, dict(xoff=1)),
    "ldx%4": (False, dict(ldx=130)),
    "Y-f64": (False, dict(y64=True)),
    "Y-misaligned": (False, dict(yoff=1)),
    "ldy%4": (False, dict(ldy=21)),
    "yy": (False, dict(outs=("G", "B", "sx", "sy", "yy"))),
    "sy-without-B": (False, dict(outs=("G", "sx", "sy"))),
    "eligible": (True, dict()),
    "eligible-G-only": (True, dict(outs=("G",))),
    "eligible-G-null": (True, dict(outs=("B", "sx", "sy"))),
    "eligible-Y-misaligned-unused": (True, dict(yoff=1, outs=("G", "sx"))),
}


@pytest.mark.parametrize("name", list(ROUTES))
def test_gram_mode1_routing(engine, name):
    """Ineligible mode-1 calls return exactly the bits of mode 0; eligible ones run the tensor cores, whose bits
    differ from mode 0 on general float data."""
    tc, o = ROUTES[name]
    N, K, n = o.get("N", 1000), o.get("K", 128), 20
    ldx, ldy = o.get("ldx", K), o.get("ldy", n)
    outs = o.get("outs", ("G", "B", "sx", "sy"))
    y64 = o.get("y64", False)
    assert M.tc_routes(N, K, ldx, not o.get("xoff"), "f64" if y64 else "f32", n, ldy, not o.get("yoff"),
                       o.get("rows", False), "B" in outs, "sy" in outs, "yy" in outs) == tc
    gen = _gen(engine, 5)
    X = torch.randn(N, K, generator=gen, device=engine.device)
    Y = torch.randn(N, n, generator=gen, device=engine.device, dtype=torch.float64 if y64 else torch.float32)
    yb = torch.randn(n, generator=gen, device=engine.device)
    Xf, _ = _place(engine, X, ldx, o.get("xoff", 0), torch.float32)
    Yf, _ = _place(engine, Y, ldy, o.get("yoff", 0), Y.dtype)
    rows = torch.randint(0, N, (1500,), generator=gen, device=engine.device, dtype=torch.int32) if o.get("rows") \
        else None
    res = []
    for mode in (0, 1):
        r = dict(G=_nan(engine, K * K) if "G" in outs else None, B=_nan(engine, K * n) if "B" in outs else None,
                 sx=_nan(engine, K) if "sx" in outs else None, sy=_nan(engine, n) if "sy" in outs else None,
                 yy=_nan(engine, 1) if "yy" in outs else None)
        raw_gram(engine, Xf, N, K, ldx, Yf, F64 if y64 else F32, n, ldy, yb, rows, 1500 if rows is not None else 0,
                 mode=mode, **r)
        res.append(r)
    torch.cuda.synchronize()
    for k in outs:
        assert not bool(torch.isnan(res[1][k]).any()), k
    if not tc:
        for k in outs:
            assert _same_bits(res[0][k], res[1][k]), k
    else:
        k = "G" if "G" in outs else "B"
        assert not _same_bits(res[0][k], res[1][k]), "mode 1 gave the fp64 bits: the tensor cores did not run"
        rel = ((res[0][k] - res[1][k]).abs().max() / res[0][k].abs().max()).item()
        assert rel < 1e-6, rel


# ------------------------------------------------------------------ part 3: tensor-core arithmetic vs its emulation
def _gpu_mm(eng):
    def mm(a, b):
        return (torch.from_numpy(np.ascontiguousarray(a)).to(eng.device).T
                @ torch.from_numpy(np.ascontiguousarray(b)).to(eng.device)).cpu().numpy()
    return mm


def grid_data(rng, N, K, mamp=2.0 ** 7, damp=2.0 ** 7, q=2.0 ** -12):
    """Columns m + d on the grid q: |m| < mamp and |d| < damp on the grid, deviations in +-pairs (a zero row when N is
    odd), each column permuted, so that every column sums to exactly N m."""
    m = np.round(rng.uniform(-mamp, mamp, K) / q) * q
    h = N // 2
    d = np.round(rng.uniform(-damp, damp, (h, K)) / q) * q
    d = np.concatenate([d, -d, np.zeros((N - 2 * h, K))])
    d = rng.permuted(d, axis=0)
    return (m + d).astype(np.float32)


def _tc_call(eng, X, Y, yb, want_G=True):
    """mode-1 gram of host arrays through Engine.gram, with 16-byte aligned, ld % 4 == 0 copies"""
    dev = eng.device
    N, K = X.shape
    Xd = torch.zeros(N, _tc_ld(K), device=dev)[:, :K]
    Xd.copy_(torch.from_numpy(X))
    Yd = None
    if Y is not None:
        Yd = torch.zeros(N, _tc_ld(Y.shape[1]), device=dev)[:, :Y.shape[1]]
        Yd.copy_(torch.from_numpy(Y))
    g = eng.gram(Xd, Yd, y_bias=None if yb is None else torch.from_numpy(yb).to(dev), want_G=want_G, mode=1)
    return {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in g.items()}


def _check_model(g, model, plan, N, what, ratios):
    nst = plan["nst"]
    for k in ("G", "B"):
        if k not in model or g[k] is None:
            continue
        blk = model[k]
        diag = k == "G"
        if diag:  # the tensor cores round (i, j) and (j, i) differently; G takes both from one of them
            assert np.array_equal(g[k].view(np.int64), np.ascontiguousarray(g[k].T).view(np.int64))
        bound = M.tc_bound(blk, nst, N, diag=diag, SQ=model.get("SQ"))
        err = np.abs(g[k] - blk["val"])
        r = err / np.maximum(bound, np.finfo(float).tiny)
        if diag:
            d = np.arange(r.shape[0])
            rd = r[d, d].max()
            r[d, d] = 0
            ratios.append(("%s G diag" % what, float(rd)))
            assert rd <= 1.0, rd
        ratios.append(("%s %s" % (what, k), float(r.max())))
        assert np.isfinite(g[k]).all()
        assert r.max() <= 1.0, (k, r.max(), np.unravel_index(np.argmax(r), r.shape))
    for k in ("sx", "sy"):
        if k in model and g[k] is not None:
            err = np.abs(g[k] - model[k]["val"])
            bound = (N + 16) * M.U64 * model[k]["mag"]
            rr = float((err / np.maximum(bound, np.finfo(float).tiny)).max())
            ratios.append(("%s %s" % (what, k), rr))
            assert rr <= 1.0, (k, rr)


EMUL_CASES = ["N64-K64-n1", "N65-K65-n3", "N4095-K128-n127", "N4097-K257-n129", "N12289-K1000-n200",
              "N50000-K257-n3", "N4097-K2304-n200", "N12289-K64-G-only", "N4096-K1000-n129-G-null"]


@pytest.mark.parametrize("name", EMUL_CASES)
def test_gram_tc_matches_emulation(engine, name):
    c = _resolve(TC_CASES[name], _sms(engine), True)
    N, K, n = c["N"], c["K"], c["n"]
    rng = np.random.default_rng(sum(map(ord, name)))
    X = grid_data(rng, N, K)
    M.exact_sum_preconditions(X, 2.0 ** -12, 2.0 ** 8)
    Y = yb = None
    if n:
        Y = grid_data(rng, N, n)
        M.exact_sum_preconditions(Y, 2.0 ** -12, 2.0 ** 8)
        if c.get("bias"):
            yb = (np.round(rng.uniform(-4, 4, n) * 4096) / 4096).astype(np.float32)
    want_G = "G" in c["outs"]
    g = _tc_call(engine, X, Y if "B" in c["outs"] else None, yb, want_G=want_G)
    px = M.tc_prep(X)
    py = M.tc_prep(Y) if (Y is not None and "B" in c["outs"]) else None
    assert np.all(px["T"] == 0) and (py is None or np.all(py["T"] == 0))
    assert np.array_equal(px["v"].astype(np.float64), px["hi"].astype(np.float64) + px["lo"].astype(np.float64))
    assert np.count_nonzero(px["lo"]) > 0
    model = M.tc_model(px, py, yb, mm=_gpu_mm(engine), want_G=want_G, with_split=False)
    model["SQ"] = px["SQ"]
    plan = M.tc_plan(N, K, n if py is not None else 0, want_G, py is not None, _sms(engine))
    # sx, sy: T = 0 and N m exact on this data
    assert np.array_equal(g["sx"], model["sx"]["val"])
    if py is not None:
        assert np.array_equal(g["sy"], model["sy"]["val"])
    ratios = []
    _check_model(g, model, plan, N, name, ratios)
    for what, r in ratios:
        print("measured/bound %-44s %.3f" % (what, r))


def _unstructured(rng, N, K, span):
    """N(0,1) columns times 2^u, u uniform in [-span, span], with every fourth column a near copy of its neighbour
    (strongly correlated off-diagonal products: the accumulation error there comes close to its bound)."""
    X = rng.standard_normal((N, K)) * np.exp2(rng.uniform(-span, span, K)) + rng.uniform(-3, 3, K) * np.exp2(
        rng.uniform(-span, span, K))
    for j in range(1, K, 4):
        X[:, j] = X[:, j - 1] * (1 + 1e-3 * rng.standard_normal(N))
    return X.astype(np.float32)


@pytest.mark.parametrize("N,K,n,span", [(4097, 129, 3, 2), (4096, 96, 5, 30), (1000, 64, 8, 0)])
def test_gram_tc_unstructured_within_model(engine, N, K, n, span):
    """General fp32 data: within the accumulation bound of the emulated model, and within that bound plus the
    model's own error (22-bit split, fp32 rounding of x - s) of the exact X'X and X'(Y - b) in long double."""
    rng = np.random.default_rng(N + K + span)
    X = _unstructured(rng, N, K, span)
    Y = _unstructured(rng, N, n, span)
    yb = (rng.standard_normal(n) * np.abs(Y).max(0)).astype(np.float32)
    g = _tc_call(engine, X, Y, yb)
    px, py = M.tc_prep(X), M.tc_prep(Y)
    model = M.tc_model(px, py, yb, mm=_gpu_mm(engine))
    model["SQ"] = px["SQ"]
    plan = M.tc_plan(N, K, n, True, True, _sms(engine))
    ratios = []
    _check_model(g, model, plan, N, "span%d" % span, ratios)
    XL = X.astype(np.longdouble)
    YL = Y.astype(np.longdouble) - yb.astype(np.longdouble)
    for k, ref in (("G", XL.T @ XL), ("B", XL.T @ YL)):
        blk = model[k]
        bound = M.tc_bound(blk, plan["nst"], N) + blk["split"] * (1 + 1e-6)
        if k == "G":
            d = np.arange(K)
            bound[d, d] = (N + 16) * M.U64 * (px["SQ"] + blk["undo"][d, d]) + blk["split"][d, d] * (1 + 1e-6)
        r = (np.abs(g[k].astype(np.longdouble) - ref) / bound).astype(np.float64)
        ratios.append(("span%d %s vs exact" % (span, k), float(r.max())))
        assert r.max() <= 1.0, (k, r.max())
    for k, ref in (("sx", XL.sum(0)), ("sy", YL.sum(0))):
        p = px if k == "sx" else py
        dx = np.abs(p["cols"].astype(np.float64) - p["shift"].astype(np.float64) - p["xs"].astype(np.float64)).sum(0)
        bound = (N + 16) * M.U64 * model[k]["mag"] + dx * (1 + 1e-6)
        r = (np.abs(g[k].astype(np.longdouble) - ref) / np.maximum(bound, 1e-300)).astype(np.float64)
        ratios.append(("span%d %s vs exact" % (span, k), float(r.max())))
        assert r.max() <= 1.0, (k, r.max())
    for what, r in ratios:
        print("measured/bound %-36s %.3f" % (what, r))


# ------------------------------------------------------------------ part 4: scale invariance
SCALES = [(k, k) for k in (-114, -100, -60, 0, 60, 100, 115, 120)] + [(60, -60), (-114, 120)]


@pytest.fixture(scope="module")
def scale_data():
    rng = np.random.default_rng(2024)
    N, K, n = 4097, 129, 5
    X = grid_data(rng, N, K, mamp=2.0, damp=4.0)
    Y = grid_data(rng, N, n, mamp=2.0, damp=4.0)
    yb = (np.round(rng.uniform(-2, 2, n) * 4096) / 4096).astype(np.float32)
    for A in (X, Y):
        mx = np.abs(A).max(0)
        assert mx.min() >= 4 and mx.max() < 8  # max |x| in [2^2, 2^3): every nonzero entry stays normal at 2^-114
        M.exact_sum_preconditions(A, 2.0 ** -12, 2.0 ** 3)
    return X, Y, yb


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("kx,ky", SCALES)
def test_gram_scales_exactly(engine, scale_data, kx, ky, mode):
    X, Y, yb = scale_data
    base = _scaled_gram(engine, X, Y, yb, 0, 0, mode)
    got = _scaled_gram(engine, X, Y, yb, kx, ky, mode)
    for k, p in (("G", 2 * kx), ("B", kx + ky), ("sx", kx), ("sy", ky)):
        want = base[k] * 2.0 ** p
        assert np.isfinite(got[k]).all(), k
        assert np.array_equal(got[k].view(np.int64), want.view(np.int64)), (
            k, int((got[k] != want).sum()), float(np.abs(got[k] / want - 1).max()))


def _scaled_gram(eng, X, Y, yb, kx, ky, mode):
    Xs = np.ldexp(X, kx).astype(np.float32)
    Ys = np.ldexp(Y, ky).astype(np.float32)
    bs = np.ldexp(yb, ky).astype(np.float32)
    assert np.array_equal(np.ldexp(Xs, -kx), X) and np.array_equal(np.ldexp(Ys, -ky), Y)
    dev = eng.device
    N, K = X.shape
    n = Y.shape[1]
    Xd = torch.zeros(N, _tc_ld(K), device=dev)[:, :K]
    Xd.copy_(torch.from_numpy(Xs))
    Yd = torch.zeros(N, _tc_ld(n), device=dev)[:, :n]
    Yd.copy_(torch.from_numpy(Ys))
    g = eng.gram(Xd, Yd, y_bias=torch.from_numpy(bs).to(dev), mode=mode)
    return {k: g[k].cpu().numpy() for k in ("G", "B", "sx", "sy")}


# ------------------------------------------------------------------ part 5: cp_gemm_f64 and cp_colstats_f64
GEMM_CASES = {
    # name: M, Nn, R, options (alpha, beta; odd: odd leading dimensions; off: operands 8 bytes off 16)
    "async128": dict(M="fill", Nn="fill", R=100),
    "async64": dict(M=300, Nn=200, R=78, beta=0.5),
    "odd-ld": dict(M=200, Nn=130, R=99, odd=True),
    "misaligned": dict(M=190, Nn=260, R=111, off=1, beta=-0.25),
    "split-alpha-beta": dict(M=200, Nn=150, R=5003, alpha=-0.75, beta=0.5),
    "partial-tiles-split": dict(M=130, Nn=70, R=1000, alpha=0.5),
}


def _gemm_resolve(c, sms):
    c = dict(c)
    t = 1
    while t * t < sms:
        t += 1
    if c["M"] == "fill":
        c["M"] = c["Nn"] = 128 * t
    return c


def _gemm_lds(c, a_mc, b_nc):
    lda = c["M"] if a_mc else c["R"]
    ldb = c["Nn"] if b_nc else c["R"]
    if c.get("odd"):
        lda += 1 - lda % 2
        ldb += 1 - ldb % 2
    return lda, ldb


def test_gemm_cases_reach_every_kernel(engine):
    sms = _sms(engine)
    reached = set()
    for name, case in GEMM_CASES.items():
        c = _gemm_resolve(case, sms)
        for a_mc in (0, 1):
            for b_nc in (0, 1):
                lda, ldb = _gemm_lds(c, a_mc, b_nc)
                asy = not a_mc and not c.get("off") and lda % 2 == 0 and ldb % 2 == 0
                br = M.product_plan(c["M"], c["Nn"], c["R"], False, sms, 8 * M.BK, asy)["branches"]
                if "all:split" in br and c.get("beta", 0.0) != 0 and c.get("alpha", 1.0) != 1:
                    br.add("split-alpha-beta")
                if c["M"] % 128 or c["Nn"] % 128:
                    br.add("partial-tiles")
                print("%-20s a_mc=%d b_nc=%d %s" % (name, a_mc, b_nc, " ".join(sorted(br))))
                reached |= br
    need = {"async128", "async64", "register-staged", "all:split", "all:unsplit", "split-alpha-beta",
            "partial-tiles", "reduction-tail", "all:unsplit-min-split-r"}
    assert need <= reached, sorted(need - reached)


@pytest.mark.parametrize("b_nc", [0, 1])
@pytest.mark.parametrize("a_mc", [0, 1])
@pytest.mark.parametrize("name", list(GEMM_CASES))
def test_gemm_f64_exact(engine, name, a_mc, b_nc):
    """Integer operands, dyadic alpha and beta: C = alpha a b' + beta C has one exact value.  C's padding columns
    (ldc > Nn) must stay untouched, and C is not read when beta = 0 (it starts as NaN then)."""
    c = _gemm_resolve(GEMM_CASES[name], _sms(engine))
    Mm, Nn, R = c["M"], c["Nn"], c["R"]
    alpha, beta = c.get("alpha", 1.0), c.get("beta", 0.0)
    lda, ldb = _gemm_lds(c, a_mc, b_nc)
    off = c.get("off", 0)
    gen = _gen(engine, Mm + 3 * Nn + R)
    dev = engine.device
    a = torch.randint(-64, 65, (Mm, R), generator=gen, device=dev).double()
    b = torch.randint(-64, 65, (Nn, R), generator=gen, device=dev).double()
    Af, _ = _place(engine, a.T if a_mc else a, lda, off, torch.float64)
    Bf, _ = _place(engine, b.T if b_nc else b, ldb, off, torch.float64)
    ldc = Nn + 3
    C0 = torch.randint(-1000, 1001, (Mm, Nn), generator=gen, device=dev).double()
    Cf, Cv = _place(engine, C0 if beta else torch.full_like(C0, NAN), ldc, off, torch.float64)
    engine._call(engine.lib.cp_gemm_f64(engine.h, a_mc, b_nc, Mm, Nn, R, alpha, engine._p(Af, "const double*"), lda,
                                        engine._p(Bf, "const double*"), ldb, beta, engine._p(Cf, "double*"), ldc,
                                        engine._s()))
    ref = alpha * (a @ b.T) + (beta * C0 if beta else 0.0)
    torch.cuda.synchronize()
    assert torch.equal(Cv, ref), int((Cv != ref).sum())
    pad = Cf[:Mm * ldc].view(Mm, ldc)[:, Nn:]
    assert bool(torch.isnan(pad).all())


@pytest.mark.parametrize("N,n", [(3001, 70), (64, 1), (100000, 33)])
def test_colstats_f64_exact(engine, N, n):
    gen = _gen(engine, N + n)
    dev = engine.device
    X = torch.randint(-10 ** 6, 10 ** 6 + 1, (N, n), generator=gen, device=dev).double()
    ldx, ldo = n + 5, n + 2
    Xf, _ = _place(engine, X, ldx, 1, torch.float64)
    cs = _nan(engine, n, 1)
    Of = _nan(engine, N * ldo, 1)
    engine._call(engine.lib.cp_colstats_f64(engine.h, engine._p(Xf, "const double*"), ldx, N, n, 0.25,
                                            engine._p(cs, "double*"), engine._p(Of, "double*"), ldo, engine._s()))
    torch.cuda.synchronize()
    ref = 0.25 * X.sum(0)
    assert torch.equal(cs, ref)
    O = Of.view(N, ldo)
    assert torch.equal(O[:, :n], X - ref)
    assert bool(torch.isnan(O[:, n:]).all())
