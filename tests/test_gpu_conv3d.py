"""GPU: patch and point gathers of 3-D feature maps (torch.nn.Conv3d semantics, cp_patch_gather_conv3d /
cp_point_gather3d).  Every path (NCDHW and NDHWC, HBM and pinned host, TMA and SIMT) is checked bit for bit against a
torch gather built from F.pad and strided indexing, the kernel that ran against the one intended, the gathered X
against F.conv3d, refusals of bad geometry, and the solver and pipeline on Conv3d layers against the oracle."""
import zlib

import numpy as np
import pytest

import conv3d_oracle as C3
import cp_oracle as O
import gather_checks as GC

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
F = pytest.importorskip("torch.nn.functional")

# (kernel_size, padding, stride, dilation), ints or (t, h, w) triples as nn.Conv3d takes them
WINDOWS = {
    "1x1x1": (1, 0, 1, 1), "3x3x3": (3, 1, 1, 1), "1x3x3": ((1, 3, 3), (0, 1, 1), 1, 1),
    "3x1x1": ((3, 1, 1), (1, 0, 0), 1, 1), "stem3x7x7": ((3, 7, 7), (1, 3, 3), (1, 2, 2), 1),
    "3x3x3d2": (3, 2, 1, 2), "3x3x3d123": (3, (1, 2, 3), 1, (1, 2, 3)),
}
# path -> (layout, in pinned host memory, channels): c = 64 passes the TMA rules, c = 12 not
PATHS = {"ncdhw": ("ncdhw", False, 12), "ncdhw_host": ("ncdhw", True, 12), "ndhwc_tma": ("ndhwc", False, 64),
         "ndhwc_simt": ("ndhwc", False, 12), "ndhwc_host": ("ndhwc", True, 24)}


def _tr(v):
    return tuple(v) if isinstance(v, tuple) else (v, v, v)


def _out_size(D, H, W, win):
    k, pad, stride, dil = (_tr(v) for v in win)
    return tuple((n + 2 * p - d * (kk - 1) - 1) // s + 1 for n, kk, p, s, d in zip((D, H, W), k, pad, stride, dil))


def _torch_gather(ncdhw, rt, rx, ry, B, win, relu):
    """X of the sampled points from the map widened to fp32 on the CPU: F.pad, then the strided taps of each window
    (padded coordinates stride*point + dil*tap).  ReLU after widening as the kernels apply it (NaN and -0 give +0).
    Rows (batch, point, image), columns (c, u, i, j)."""
    (kt, kh, kw), (pt, ph, pw), (st, sh, sw), (dt, dh, dw) = (_tr(v) for v in win)
    x = ncdhw.float().cpu()
    xp = F.pad(x, (pw, pw + dw * kw, ph, ph + dh * kh, pt, pt + dt * kt))
    c = x.shape[1]
    nb, P = rt.shape
    img = (torch.arange(nb)[:, None, None] * B + torch.arange(B)[None, None, :]).expand(nb, P, B).reshape(-1)
    rep = [r.cpu().long()[:, :, None].expand(nb, P, B).reshape(-1) for r in (rt, rx, ry)]
    it = (st * rep[0][:, None] + dt * torch.arange(kt)[None, :])[:, None, :, None, None]
    iy = (sh * rep[1][:, None] + dh * torch.arange(kh)[None, :])[:, None, None, :, None]
    ix = (sw * rep[2][:, None] + dw * torch.arange(kw)[None, :])[:, None, None, None, :]
    X = xp[img[:, None, None, None, None], torch.arange(c)[None, :, None, None, None], it, iy, ix]
    X = X.reshape(len(img), -1)
    return torch.where(X > 0, X, torch.zeros_like(X)) if relu else X


def _gather(engine, path, ncdhw, rt, rx, ry, B, P, win, relu, out=None):
    layout, host, _ = PATHS[path]
    m = ncdhw if layout == "ncdhw" else ncdhw.permute(0, 2, 3, 4, 1).contiguous()
    if host:
        m = GC.pinned(m)
    k, pad, stride, dil = win
    return engine.patch_gather3d(m, rt, rx, ry, B, P, k, pad, stride, relu=relu, layout=layout, dilation=dil, out=out)


@pytest.mark.parametrize("dtype", list(GC.FMAP_DTYPES))
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("wname", list(WINDOWS))
def test_gather3d_bits_equal_torch(engine, dtype, path, wname):
    win = WINDOWS[wname]
    dev = engine.device
    c = PATHS[path][2]
    D, H, W, B, nb = 5, 9, 8, 3, 2
    To, Ho, Wo = _out_size(D, H, W, win)
    seed = zlib.crc32(("%s/%s/%s" % (wname, path, dtype)).encode()) % 10007
    ncdhw = GC.special_map((nb * B, c, D, H, W), dtype, seed, dev)
    rt, rx, ry, P = GC.points3d(nb, To, Ho, Wo, dev)
    for relu in (False, True):
        got = _gather(engine, path, ncdhw, rt, rx, ry, B, P, win, relu)
        torch.cuda.synchronize()
        GC.assert_same_bits(got, _torch_gather(ncdhw, rt, rx, ry, B, win, relu))


def test_torch_gather_agrees_with_the_numpy_oracle():
    """The torch reference gather and conv3d_oracle.gather3d (per-window numpy) give the same X."""
    r = np.random.RandomState(1)
    x = torch.as_tensor(r.standard_normal((4, 3, 5, 9, 8)).astype(np.float32))
    for win in WINDOWS.values():
        To, Ho, Wo = _out_size(5, 9, 8, win)
        pts = [torch.as_tensor(r.randint(0, hi, (2, 3)).astype(np.int32)) for hi in (To, Ho, Wo)]
        want = C3.gather3d(x.numpy(), *[p.numpy() for p in pts], 2, *win, relu=True)
        assert np.array_equal(_torch_gather(x, *pts, 2, win, True).numpy(), want)


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("wname", ["3x3x3", "1x3x3", "3x3x3d2"])
def test_gather3d_at_r3d18_size(engine, dtype, wname):
    """N = 5000 rows of a 128-channel 8 x 28 x 28 map (r3d_18 layer2; the persistent grids' tails), every path against
    the torch gather, and a row slice of a wider buffer (ldx > K) on the TMA path that leaves the rest alone."""
    win = WINDOWS[wname]
    dev = engine.device
    c, D, H, B, nb, P = 128, 8, 28, 10, 10, 50
    To, Ho, Wo = _out_size(D, H, H, win)
    g = torch.Generator(device=dev)
    g.manual_seed(11)
    ncdhw = torch.randn((nb * B, c, D, H, H), generator=g, device=dev).to(GC.FMAP_DTYPES[dtype])
    r = np.random.RandomState(3)
    rt, rx, ry = (torch.as_tensor(r.randint(0, hi, (nb, P)).astype(np.int32), device=dev) for hi in (To, Ho, Wo))
    want = _torch_gather(ncdhw, rt, rx, ry, B, win, True)
    for path in ("ncdhw", "ndhwc_tma", "ndhwc_host", "ncdhw_host"):
        got = _gather(engine, path, ncdhw, rt, rx, ry, B, P, win, True)
        torch.cuda.synchronize()
        GC.assert_same_bits(got, want)
        del got
    K = want.shape[1]
    wide = torch.full((want.shape[0], K + 40), 7.0, device=dev)
    _gather(engine, "ndhwc_tma", ncdhw, rt, rx, ry, B, P, win, True, out=wide[:, 8:8 + K])
    torch.cuda.synchronize()
    GC.assert_same_bits(wide[:, 8:8 + K].contiguous(), want)
    assert bool((wide[:, :8] == 7.0).all()) and bool((wide[:, 8 + K:] == 7.0).all())


@pytest.mark.parametrize("dtype", list(GC.FMAP_DTYPES))
@pytest.mark.parametrize("layout,host", [("ncdhw", False), ("ndhwc", False), ("ncdhw", True), ("ndhwc", True)])
def test_point_gather3d_bits(engine, dtype, layout, host):
    dev = engine.device
    n, To, Ho, Wo, B, nb = 40, 4, 7, 6, 3, 2
    y = GC.special_map((nb * B, n, To, Ho, Wo), dtype, 17 + n, dev)
    rt, rx, ry, P = GC.points3d(nb, To, Ho, Wo, dev)
    m = y if layout == "ncdhw" else y.permute(0, 2, 3, 4, 1).contiguous()
    m = GC.pinned(m) if host else m
    got = engine.point_gather3d(m, rt, rx, ry, B, P, layout=layout)
    torch.cuda.synchronize()
    yc = y.float().cpu()
    want = torch.stack([yc[b * B + i, :, int(rt[b, p]), int(rx[b, p]), int(ry[b, p])]
                        for b in range(nb) for p in range(P) for i in range(B)])
    GC.assert_same_bits(got, want)


@pytest.mark.parametrize("wname", list(WINDOWS))
@pytest.mark.parametrize("layout", ["ncdhw", "ndhwc"])
def test_gathered_x_reproduces_conv3d(engine, wname, layout):
    """relu(X) W2' + b2 at the sampled points is F.conv3d(relu(x), W2, b2, stride, padding, dilation) there."""
    k, pad, stride, dil = win = WINDOWS[wname]
    dev = engine.device
    g = torch.Generator(device=dev)
    g.manual_seed(5)
    c, n, D, H, W, B, nb = 16, 8, 5, 9, 8, 3, 2
    x = torch.randn((nb * B, c, D, H, W), generator=g, device=dev)
    W2 = torch.randn((n, c) + _tr(k), generator=g, device=dev)
    b2 = torch.randn((n,), generator=g, device=dev)
    To, Ho, Wo = _out_size(D, H, W, win)
    rt, rx, ry, P = GC.points3d(nb, To, Ho, Wo, dev)
    m = x if layout == "ncdhw" else x.permute(0, 2, 3, 4, 1).contiguous()
    X = engine.patch_gather3d(m, rt, rx, ry, B, P, k, pad, stride, relu=True, layout=layout, dilation=dil)
    got = X.double() @ W2.reshape(n, -1).T.double() + b2.double()
    y = F.conv3d(torch.relu(x).double(), W2.double(), b2.double(), stride=stride, padding=pad, dilation=dil)
    assert tuple(y.shape[2:]) == (To, Ho, Wo)
    want = torch.stack([y[b * B + i, :, int(rt[b, p]), int(rx[b, p]), int(ry[b, p])] for b in range(nb)
                        for p in range(P) for i in range(B)])
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5)


def _raw_gather3d(engine, m, c, D, H, W, layout, geom):
    """cp_patch_gather_conv3d with geom = (kt, kh, kw, pt, ph, pw, st, sh, sw, dt, dh, dw); returns (rc, message)."""
    ffi, lib = engine.ffi, engine.lib
    r = torch.zeros((1, 1), dtype=torch.int32, device=engine.device)
    k3 = max(geom[0] * geom[1] * geom[2], 1)
    X = torch.empty((2, c * k3 + 16), device=engine.device)
    ip = ffi.cast("const int32_t*", r.data_ptr())
    rc = lib.cp_patch_gather_conv3d(engine.h, ffi.cast("const void*", m.data_ptr()), lib.CP_F32, 1, 2, c, D, H, W,
                                    layout, ip, ip, ip, 1, *geom, 0, ffi.cast("float*", X.data_ptr()), X.shape[1],
                                    ffi.NULL)
    return rc, ffi.string(lib.cp_last_error()).decode()


_G = (3, 3, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1)


def _with(i, v):
    g = list(_G)
    g[i] = v
    return tuple(g)


@pytest.mark.parametrize("geom,msg", [(_with(0, 0), "kernel_size"), (_with(2, 0), "kernel_size"),
                                      (_with(3, -1), "padding"), (_with(5, -2), "padding"),
                                      (_with(6, 0), "stride"), (_with(8, 0), "stride"),
                                      (_with(9, 0), "dilation"), (_with(10, 0), "dilation"),
                                      ((5, 3, 3, 0, 1, 1, 1, 1, 1, 1, 1, 1), "empty output map"),
                                      ((3, 3, 3, 1, 1, 1, 1, 1, 1, 3, 1, 1), "empty output map"),
                                      ((17, 16, 16, 8, 8, 8, 1, 1, 1, 1, 1, 1), "taps")])
@pytest.mark.parametrize("layout", [0, 1])
def test_bad_geometry_is_refused(engine, geom, msg, layout):
    import cpb200

    f = torch.zeros(2, 16, 3, 7, 7, device=engine.device)
    rc, err = _raw_gather3d(engine, f, 16, 3, 7, 7, layout, geom)
    assert rc == engine.lib.CP_ERR_INVALID and msg in err, err
    kt, kh, kw, pt, ph, pw, st, sh, sw, dt, dh, dw = geom
    r = torch.zeros((1, 1), dtype=torch.int32, device=engine.device)
    with pytest.raises(cpb200._cabi.CpError):
        engine.patch_gather3d(f, r, r, r, 2, 1, (kt, kh, kw), (pt, ph, pw), (st, sh, sw), dilation=(dt, dh, dw))


def test_window_beyond_the_host_reader_is_refused(engine):
    """kt*kh*kw = 392 > 343 on an NDHWC pinned map: CP_ERR_INVALID with a message; the same window on the NDHWC SIMT
    kernel in HBM and on NCDHW maps (HBM and pinned) is gathered."""
    dev = engine.device
    m = torch.randn(2, 8, 9, 9, 3, device=dev)
    geom = (8, 7, 7, 3, 3, 3, 1, 1, 1, 1, 1, 1)
    rc, err = _raw_gather3d(engine, GC.pinned(m), 3, 8, 9, 9, 1, geom)
    assert rc == engine.lib.CP_ERR_INVALID and "8x7x7" in err and "host reader" in err, err
    nc = m.permute(0, 4, 1, 2, 3).contiguous()
    for mm, lay in ((m, 1), (nc, 0), (GC.pinned(nc), 0)):
        rc, err = _raw_gather3d(engine, mm, 3, 8, 9, 9, lay, geom)
        assert rc == 0, err
    torch.cuda.synchronize()


def test_point_gather3d_refuses_an_empty_map(engine):
    ffi, lib = engine.ffi, engine.lib
    r = torch.zeros((1, 1), dtype=torch.int32, device=engine.device)
    f = torch.zeros(2, 4, 2, 2, 2, device=engine.device)
    Y = torch.empty(2, 4, device=engine.device)
    ip = ffi.cast("const int32_t*", r.data_ptr())
    for n, D in ((0, 2), (4, 0)):
        rc = lib.cp_point_gather3d(engine.h, ffi.cast("const void*", f.data_ptr()), lib.CP_F32, 1, 2, n, D, 2, 2, 0,
                                   ip, ip, ip, 1, ffi.cast("float*", Y.data_ptr()), 4, ffi.NULL)
        assert rc == lib.CP_ERR_INVALID and b"empty output map" in ffi.string(lib.cp_last_error())


# kind -> (layout, host, channels, windows)
_KERNEL_CASES = {"tma": ("ndhwc", False, 64, ["3x3x3", "1x3x3", "3x1x1", "1x1x1", "stem3x7x7", "3x3x3d2"]),
                 "simt": ("ndhwc", False, 12, ["3x3x3", "stem3x7x7"]),
                 "host": ("ndhwc", True, 64, ["3x3x3", "3x3x3d123"]),
                 "ncdhw": ("ncdhw", False, 64, ["3x3x3", "1x3x3"]),
                 "ncdhw_host": ("ncdhw", True, 64, ["3x3x3"])}
_REPEAT = 3


def _profile_kernel_cases():
    """Runs every case of _KERNEL_CASES _REPEAT times inside one profiler session; returns (kind, kernel name) of
    every gather launch, in order."""
    import cpb200
    from torch.profiler import ProfilerActivity, profile

    engine = cpb200.get_engine()
    dev = engine.device
    D, H, B, nb = 5, 11, 2, 2
    runs = []
    for kind, (layout, host, c, names) in _KERNEL_CASES.items():
        for wname in names:
            k, pad, stride, dil = win = WINDOWS[wname]
            rt, rx, ry, P = GC.points3d(nb, *_out_size(D, H, H, win), dev)
            shape = (nb * B, D, H, H, c) if layout == "ndhwc" else (nb * B, c, D, H, H)
            m = torch.randn(shape, device=dev)
            if host:
                m = GC.pinned(m)
            call = (lambda m=m, rt=rt, rx=rx, ry=ry, P=P, k=k, pad=pad, stride=stride, dil=dil, layout=layout:
                    engine.patch_gather3d(m, rt, rx, ry, B, P, k, pad, stride, layout=layout, dilation=dil))
            call()  # warm-up (module load)
            runs.append((kind, call))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _, call in runs:
            for _ in range(_REPEAT):
                call()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "patch_gather" in e.name and e.device_type.name == "CUDA"]


def test_intended_kernels_run(engine):
    """One profiler session: eligible NDHWC HBM windows launch the 5-D TMA kernel, c = 12 the NDHWC SIMT kernel,
    NDHWC pinned maps the host reader, NCDHW maps (HBM and pinned) the NCDHW kernel.  Each case runs _REPEAT times, so
    a lost activity record does not decide the check.  The session runs in a child process, so the suite's other
    profiler checks keep their record counts."""

    def kind_of(n):
        for key, kind in (("patch_gather_ndhwc_tma<", "tma"), ("patch_gather_ndhwc_host<", "host"),
                          ("patch_gather_ndhwc<", "simt"), ("patch_gather_ncdhw<", "ncdhw")):
            if key in n:
                return kind
        return n

    want = {k: _REPEAT * len(v[3]) for k, v in _KERNEL_CASES.items()}
    want["ncdhw"] += want.pop("ncdhw_host")  # one kernel, two grids
    GC.assert_launch_counts(GC.launched_gather_kernels("test_gpu_conv3d"), kind_of, want)


def _layer(name, c, n, D, H, k=3, pad=1, stride=1, dilation=1, N=1000, B=10, P=10, rank=None):
    import cpb200

    return cpb200.synth.LayerShape3d(name, c, n, D, H, k=k, pad=pad, stride=stride, dilation=dilation, N=N, B=B, P=P,
                                     rank=rank)


@pytest.mark.parametrize("mode,tol", [(0, 1e-7), (1, 1e-4)], ids=["fp64", "3xtf32"])
@pytest.mark.parametrize("geom", [dict(k=3, pad=1), dict(k=(1, 3, 3), pad=(0, 1, 1))], ids=["3x3x3", "1x3x3"])
def test_dictionary_on_conv3d_layers_matches_oracle(engine, mode, tol, geom):
    """decompose.dictionary on X (N, c, kt, kh, kw) against the oracle: the same mask, alpha probes and numpy RNG
    draws, weights within tol, newW2 shaped (n, c', kt, kh, kw)."""
    import cpb200
    from cpb200.lib import cfgs, decompose

    engine.gram_mode = mode
    s = _layer("L", 32, 24, 4, 8, **geom)
    d = cpb200.synth.make_problem_numpy(s, 9)
    X, W2, Y = d["X"].astype(np.float64), d["W2"], d["feats"].astype(np.float64)
    assert X.shape == (s.N, s.c, s.kt, s.kh, s.kw)
    st = O.DictState(alpha=1e-3)
    info = {}
    np.random.seed(77)
    oi, oW, oB = C3.dictionary(X, W2, Y, rank=s.rank, state=st, info=info)
    after_oracle = np.random.get_state()
    cfgs.alpha = 1e-3
    np.random.seed(77)
    idxs, W, B = decompose.dictionary(X, W2, Y, rank=s.rank)
    after_device = np.random.get_state()
    assert np.array_equal(idxs, oi)
    assert decompose.DictionaryInfo.last["probes"] == info["probes"]
    assert cfgs.alpha == st.alpha
    assert after_oracle[2] == after_device[2] and np.array_equal(after_oracle[1], after_device[1])
    assert W.shape == oW.shape == (s.n, int(idxs.sum()), s.kt, s.kh, s.kw)
    assert GC.rel(W, oW) <= tol and np.abs(B - oB).max() <= tol * max(1.0, np.abs(oB).max())


def _video_layers(N=400, B=4, P=5):
    """Conv3d layers at test size (r3d_18-like 3x3x3, R(2+1)D's 1x3x3 and 3x1x1, a strided and a dilated 3x3x3) and
    one 2-D layer among them."""
    import cpb200

    return [_layer("l1_3x3x3", 32, 24, 4, 14, N=N, B=B, P=P),
            _layer("l2_s2", 32, 48, 4, 14, stride=2, N=N, B=B, P=P),
            _layer("r21d_1x3x3", 48, 32, 4, 8, k=(1, 3, 3), pad=(0, 1, 1), N=N, B=B, P=P),
            _layer("r21d_3x1x1", 32, 32, 4, 8, k=(3, 1, 1), pad=(1, 0, 0), N=N, B=B, P=P),
            _layer("d2", 24, 16, 5, 9, pad=2, dilation=2, N=N, B=B, P=P),
            cpb200.synth.LayerShape("conv2d", 32, 24, 14, N=N, B=B, P=P)]


def _oracle_layer(s, d):
    """The oracle on one Conv3d pipeline problem: conv3d_oracle.gather3d (ReLU'd), then the oracle's dictionary with the
    problem's samples and seeds."""
    fm = d["fmap"].float().cpu().numpy() if d["layout"] == "ncdhw" else \
        d["fmap"].permute(0, 4, 1, 2, 3).float().cpu().numpy()
    pts = [d[k].cpu().numpy() for k in ("randt", "randx", "randy")]
    X = C3.gather3d(fm.astype(np.float64), *pts, s.B, s.k, s.pad, s.stride, s.dilation, relu=True)
    return GC.oracle_on_problem(C3.dictionary, X.reshape((s.N, s.c) + s.window), s, d)


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("host_layout", ["ncdhw", "ndhwc"])
def test_pipeline_on_conv3d_layers(engine, dtype, host_layout):
    """prune_layers on Conv3d layers mixed with a 2-D one: maps in HBM, read in place from pinned host memory ('zc')
    or staged by DMA ('copy') or as the plan decides, NCDHW or NDHWC on the host -- identical masks, alpha, W and b;
    two layers against the oracle (fp64 statistics: W and b within 1e-7)."""
    import cpb200
    from cpb200 import pruner

    eng = cpb200.Engine(nstreams=4)
    eng.gram_mode = 0
    shapes = _video_layers()
    datas = []
    for i, s in enumerate(shapes):
        hl = host_layout if isinstance(s, cpb200.synth.LayerShape3d) else "nchw"
        datas.append(cpb200.synth.make_problem_device(s, 70 + i, eng, pinned_host=True, host_layout=hl,
                                                      dtype=GC.FMAP_DTYPES[dtype]))
    ref = pruner.prune_layers(eng, shapes, datas)
    torch.cuda.synchronize()
    ref = [(r.idxs.copy(), r.alpha, r.nprobe, r.W.cpu(), r.b.cpu()) for r in ref]
    for policy in ("zc", "copy", True):
        got = pruner.prune_layers(eng, shapes, datas, from_host=policy, to_host=True)
        torch.cuda.synchronize()
        for s, (idxs, alpha, nprobe, W, b), r in zip(shapes, ref, got):
            assert np.array_equal(idxs, r.idxs) and alpha == r.alpha and nprobe == r.nprobe, (policy, s.name)
            assert torch.equal(W, r.W) and torch.equal(b, r.b), (policy, s.name)
    if host_layout == "ncdhw":
        for i in (0, 2):  # l1_3x3x3 and r21d_1x3x3
            s, d = shapes[i], datas[i]
            oi, oW, oB, oalpha, onprobe = _oracle_layer(s, d)
            idxs, alpha, nprobe, W, b = ref[i]
            assert np.array_equal(idxs, oi) and alpha == oalpha and nprobe == onprobe, s.name
            W = W.numpy().reshape(oW.shape)
            assert GC.rel(W, oW) <= 1e-7 and np.abs(b.numpy() - oB).max() <= 1e-7, s.name
    eng.close()


def test_pipeline_with_tensor_core_statistics_matches_oracle(engine):
    """The product default (tensor-core statistics with refinement) on a 3x3x3 layer with NDHWC maps in HBM (the TMA
    gather): the oracle's mask and probes, W and b within 1e-4."""
    import cpb200
    from cpb200 import pruner

    eng = cpb200.Engine(nstreams=2)
    eng.gram_mode = 1
    s = _layer("l1_3x3x3", 32, 24, 4, 14, N=400, B=4, P=5)
    d = cpb200.synth.make_problem_device(s, 5, eng, layout="ndhwc")
    r = pruner.prune_layers(eng, [s], [d])[0]
    torch.cuda.synchronize()
    oi, oW, oB, oalpha, onprobe = _oracle_layer(s, d)
    assert np.array_equal(r.idxs, oi) and r.alpha == oalpha and r.nprobe == onprobe
    assert GC.rel(r.W.cpu().numpy().reshape(oW.shape), oW) <= 1e-4
    assert np.abs(r.b.cpu().numpy() - oB).max() <= 1e-4 * max(1.0, np.abs(oB).max())
    eng.close()


def test_prune_network_sharded_returns_5d_weights(engine):
    """One rank: unpack_network gives (n, c', kt, kh, kw) for the Conv3d layers, (n, c', kh, kw) for the 2-D one, with
    the values prune_layers returns."""
    import cpb200
    from cpb200 import pruner

    eng = cpb200.Engine(nstreams=4)
    eng.gram_mode = 0
    shapes = _video_layers()
    datas = [cpb200.synth.make_problem_device(s, 30 + i, eng) for i, s in enumerate(shapes)]
    owner, sizes, allbuf = pruner.prune_network_sharded(eng, shapes, lambda i: datas[i], 0, 1)
    out = pruner.unpack_network(shapes, owner, sizes, allbuf)
    ref = pruner.prune_layers(eng, shapes, datas)
    torch.cuda.synchronize()
    for s, o, r in zip(shapes, out, ref):
        assert o["W"].shape == (s.n, int(r.idxs.sum())) + pruner.window_of(s)
        assert np.array_equal(o["idxs"], r.idxs) and o["alpha"] == r.alpha
        assert np.array_equal(o["W"].reshape(s.n, -1), r.W.cpu().numpy()) and np.array_equal(o["b"], r.b.cpu().numpy())
    assert out[0]["W"].ndim == 5 and out[-1]["W"].ndim == 4
    eng.close()
