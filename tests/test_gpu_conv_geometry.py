"""GPU: patch gathers for general convolution windows -- rectangular kernels, per-axis padding and stride, dilation
(torch.nn.Conv2d semantics, cp_patch_gather_conv).  Every path (NCHW and NHWC, HBM and pinned host, TMA and SIMT) is
checked bit for bit against F.unfold on the CPU, square windows against the reference entry points, the kernel that
ran against the one intended, the gathered X against F.conv2d, and the solver and pipeline on dilated and
rectangular layers against the oracle."""
import zlib

import numpy as np
import pytest

import conv_oracle as CO
import cp_oracle as O
import gather_checks as GC

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
F = pytest.importorskip("torch.nn.functional")

# (kernel_size, padding, stride, dilation), ints or (h, w) pairs as nn.Conv2d takes them
WINDOWS = {
    "1x3": ((1, 3), (0, 1), 1, 1), "3x1": ((3, 1), (1, 0), 1, 1), "1x7": ((1, 7), (0, 3), 1, 1),
    "7x1": ((7, 1), (3, 0), 1, 1), "2x2": ((2, 2), 0, 1, 1), "2x2p1": ((2, 2), 1, 1, 1),
    "3x3d2": (3, 2, 1, 2), "3x3d4": (3, 4, 1, 4), "5x5d3": (5, 6, 1, 3), "3x3d12": (3, 12, 1, 12),
    "3x3s21": (3, 1, (2, 1), 1), "3x7p03": ((3, 7), (0, 3), 1, 1), "3x5d21s12": ((3, 5), (2, 2), (1, 2), (2, 1)),
}
# path -> (layout, in pinned host memory, channels): c = 64 passes the TMA rules (when the window does), c = 12 not
PATHS = {"nchw": ("nchw", False, 12), "nchw_host": ("nchw", True, 12), "nhwc_tma": ("nhwc", False, 64),
         "nhwc_simt": ("nhwc", False, 12), "nhwc_host": ("nhwc", True, 24)}


def _pair(v):
    return tuple(v) if isinstance(v, tuple) else (v, v)


def _out_size(H, W, win):
    (kh, kw), (ph, pw), (sh, sw), (dh, dw) = (_pair(v) for v in win)
    return (H + 2 * ph - dh * (kh - 1) - 1) // sh + 1, (W + 2 * pw - dw * (kw - 1) - 1) // sw + 1


def _points(nb, Ho, Wo, device):
    """Every corner and border of the output map, plus the centre, in varying order per batch."""
    pts = [(0, 0), (0, Wo - 1), (Ho - 1, 0), (Ho - 1, Wo - 1), (Ho // 2, Wo // 2), (1 % Ho, Wo - 1), (Ho - 1, 1 % Wo),
           (0, Wo // 2), (Ho // 2, 0), (Ho - 1, Wo // 2), (Ho // 2, Wo - 1)]
    rx = torch.tensor([[p[0] for p in pts]] * nb, dtype=torch.int32, device=device)
    ry = torch.tensor([[p[1] for p in pts]] * nb, dtype=torch.int32, device=device)
    rx[1] = rx[1].flip(0)
    ry[1] = ry[1].flip(0)
    return rx, ry, len(pts)


def _unfold_oracle(nchw, rx, ry, B, win, relu):
    """X of the sampled points from F.unfold on the CPU, of the map widened to fp32, ReLU after widening with the
    kernels' fmaxf(v, 0) (NaN and -0 give +0).  Rows (batch, point, image), columns F.unfold's (c, i, j)."""
    k, pad, stride, dil = win
    x = nchw.float().cpu()
    _, _, H, W = x.shape
    Ho, Wo = _out_size(H, W, win)
    U = F.unfold(x, _pair(k), dilation=_pair(dil), padding=_pair(pad), stride=_pair(stride))
    assert U.shape[2] == Ho * Wo
    nb, P = rx.shape
    rows = [U[b * B + i, :, int(rx[b, p]) * Wo + int(ry[b, p])] for b in range(nb) for p in range(P) for i in range(B)]
    X = torch.stack(rows)
    if relu:
        X = torch.where(X > 0, X, torch.zeros_like(X))
    return X


def _direct_oracle(nchw, rx, ry, B, win):
    """The same X as _unfold_oracle (ReLU on) by direct indexing: F.unfold of a whole N = 5000 problem would not fit in
    host memory."""
    (kh, kw), (ph, pw), (sh, sw), (dh, dw) = (_pair(v) for v in win)
    x = nchw.float().cpu()
    n, c, H, W = x.shape
    nb, P = rx.shape
    img = (torch.arange(nb)[:, None, None] * B + torch.arange(B)[None, None, :]).expand(nb, P, B).reshape(-1)
    px = rx.cpu().long()[:, :, None].expand(nb, P, B).reshape(-1)
    py = ry.cpu().long()[:, :, None].expand(nb, P, B).reshape(-1)
    iy = (sh * px[:, None] - ph + dh * torch.arange(kh)[None, :])[:, None, :, None]
    ix = (sw * py[:, None] - pw + dw * torch.arange(kw)[None, :])[:, None, None, :]
    inside = (iy >= 0) & (iy < H) & (ix >= 0) & (ix < W)
    X = x[img[:, None, None, None], torch.arange(c)[None, :, None, None], iy.clamp(0, H - 1), ix.clamp(0, W - 1)]
    X = torch.where(inside, X, torch.zeros_like(X))
    X = X.reshape(len(img), c * kh * kw)
    return torch.where(X > 0, X, torch.zeros_like(X))


def _gather(engine, path, nchw, rx, ry, B, P, win, relu, out=None):
    layout, host, _ = PATHS[path]
    m = nchw if layout == "nchw" else nchw.permute(0, 2, 3, 1).contiguous()
    if host:
        m = GC.pinned(m)
    k, pad, stride, dil = win
    return engine.patch_gather(m, rx, ry, B, P, k, pad, stride, relu=relu, layout=layout, dilation=dil, out=out)


@pytest.mark.parametrize("dtype", list(GC.FMAP_DTYPES))
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("wname", list(WINDOWS))
def test_conv_gather_bits_equal_unfold(engine, dtype, path, wname):
    win = WINDOWS[wname]
    dev = engine.device
    c = PATHS[path][2]
    H, W, B, nb = 11, 10, 3, 2
    Ho, Wo = _out_size(H, W, win)
    seed = zlib.crc32(("%s/%s/%s" % (wname, path, dtype)).encode()) % 10007
    nchw = GC.special_map((nb * B, c, H, W), dtype, seed, dev)
    rx, ry, P = _points(nb, Ho, Wo, dev)
    for relu in (False, True):
        got = _gather(engine, path, nchw, rx, ry, B, P, win, relu)
        torch.cuda.synchronize()
        GC.assert_same_bits(got.cpu(), _unfold_oracle(nchw, rx, ry, B, win, relu))


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("wname", ["3x3d2", "3x3d4", "1x7", "7x1", "3x3d12"])
def test_conv_gather_at_deeplab_size(engine, dtype, wname):
    """N = 5000 rows of a 256-channel 28 x 28 map (the persistent grids' tails), every path against F.unfold, and a
    row slice of a wider buffer (ldx > K) on the TMA path that leaves the rest of the buffer alone."""
    win = WINDOWS[wname]
    dev = engine.device
    c, H, B, nb, P = 256, 28, 10, 50, 10
    Ho, Wo = _out_size(H, H, win)
    g = torch.Generator(device=dev)
    g.manual_seed(11)
    nchw = torch.randn((nb * B, c, H, H), generator=g, device=dev).to(GC.FMAP_DTYPES[dtype])
    r = np.random.RandomState(3)
    rx = torch.as_tensor(r.randint(0, Ho, (nb, P)).astype(np.int32), device=dev)
    ry = torch.as_tensor(r.randint(0, Wo, (nb, P)).astype(np.int32), device=dev)
    want = _direct_oracle(nchw, rx, ry, B, win)
    small = slice(0, 2 * P * B)
    GC.assert_same_bits(want[small], _unfold_oracle(nchw[:2 * B], rx[:2], ry[:2], B, win, True))
    for path in ("nchw", "nhwc_tma", "nhwc_host"):
        got = _gather(engine, path, nchw, rx, ry, B, P, win, True)
        torch.cuda.synchronize()
        GC.assert_same_bits(got.cpu(), want)
        del got
    K = want.shape[1]
    wide = torch.full((want.shape[0], K + 40), 7.0, device=dev)
    _gather(engine, "nhwc_tma", nchw, rx, ry, B, P, win, True, out=wide[:, 8:8 + K])
    torch.cuda.synchronize()
    GC.assert_same_bits(wide[:, 8:8 + K].contiguous().cpu(), want)
    assert bool((wide[:, :8] == 7.0).all()) and bool((wide[:, 8 + K:] == 7.0).all())


@pytest.mark.parametrize("dtype", list(GC.FMAP_DTYPES))
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("k,pad,stride", [(1, 0, 1), (1, 0, 2), (3, 1, 1), (3, 0, 2), (5, 2, 1)])
def test_square_windows_give_the_reference_entries_bits(engine, dtype, path, k, pad, stride):
    """A square, odd, undilated window through cp_patch_gather_conv (pairs) gives the bits of cp_patch_gather_typed
    (ints), and of cp_patch_gather for fp32 maps."""
    dev = engine.device
    c = PATHS[path][2]
    layout, host, _ = PATHS[path]
    H, B, nb = 9, 3, 2
    Ho = (H + 2 * pad - k) // stride + 1
    nchw = GC.special_map((nb * B, c, H, H), dtype, c + k * 7 + stride, dev)
    rx, ry, P = _points(nb, Ho, Ho, dev)
    for relu in (False, True):
        a = _gather(engine, path, nchw, rx, ry, B, P, (k, pad, stride, 1), relu)
        b = _gather(engine, path, nchw, rx, ry, B, P, ((k, k), (pad, pad), (stride, stride), (1, 1)), relu)
        torch.cuda.synchronize()
        GC.assert_same_bits(b, a)
        if dtype == "fp32":
            m = nchw if layout == "nchw" else nchw.permute(0, 2, 3, 1).contiguous()
            m = GC.pinned(m) if host else m
            X = torch.empty_like(a)
            ffi, lib = engine.ffi, engine.lib
            rc = lib.cp_patch_gather(engine.h, ffi.cast("const float*", m.data_ptr()), nb, B, c, H, H,
                                     0 if layout == "nchw" else 1, ffi.cast("const int32_t*", rx.data_ptr()),
                                     ffi.cast("const int32_t*", ry.data_ptr()), P, k, pad, stride, int(relu),
                                     ffi.cast("float*", X.data_ptr()), X.stride(0), ffi.NULL)
            assert rc == 0
            torch.cuda.synchronize()
            GC.assert_same_bits(X, a)


def _raw_gather(engine, m, c, H, W, layout, kh, kw, ph, pw, sh, sw, dh, dw, entry="conv"):
    ffi, lib = engine.ffi, engine.lib
    r = torch.zeros((1, 1), dtype=torch.int32, device=engine.device)
    X = torch.empty((2, c * max(kh * kw, 1) + 16), device=engine.device)
    args = (engine.h, ffi.cast("const void*", m.data_ptr()), lib.CP_F32, 1, 2, c, H, W, layout,
            ffi.cast("const int32_t*", r.data_ptr()), ffi.cast("const int32_t*", r.data_ptr()), 1)
    tail = (0, ffi.cast("float*", X.data_ptr()), X.shape[1], ffi.NULL)
    if entry == "conv":
        rc = lib.cp_patch_gather_conv(*args, kh, kw, ph, pw, sh, sw, dh, dw, *tail)
    else:
        rc = lib.cp_patch_gather_typed(*args, kh, ph, sh, *tail)
    return rc, ffi.string(lib.cp_last_error()).decode()


@pytest.mark.parametrize("bad,msg", [((3, 3, 1, 1, 1, 1, 0, 1), "dilation"), ((3, 3, 1, 1, 1, 1, 1, 0), "dilation"),
                                     ((3, 3, 1, 1, 0, 1, 1, 1), "stride"), ((3, 3, 1, 1, 1, 0, 1, 1), "stride"),
                                     ((3, 3, -1, 1, 1, 1, 1, 1), "padding"), ((3, 3, 1, -2, 1, 1, 1, 1), "padding"),
                                     ((0, 3, 0, 1, 1, 1, 1, 1), "kernel_size"), ((3, 0, 1, 0, 1, 1, 1, 1), "kernel_size")])
def test_bad_geometry_is_refused(engine, bad, msg):
    import cpb200

    f = torch.zeros(2, 16, 7, 7, device=engine.device)
    rc, err = _raw_gather(engine, f, 16, 7, 7, 0, *bad)
    assert rc == engine.lib.CP_ERR_INVALID and msg in err, err
    kh, kw, ph, pw, sh, sw, dh, dw = bad
    r = torch.zeros((1, 1), dtype=torch.int32, device=engine.device)
    with pytest.raises(cpb200._cabi.CpError):
        engine.patch_gather(f, r, r, 2, 1, (kh, kw), (ph, pw), (sh, sw), dilation=(dh, dw))


def test_window_beyond_the_host_reader_is_refused(engine):
    """kh*kw = 90 > 81 on an NHWC pinned map: CP_ERR_INVALID with a message; the same window on the NHWC SIMT kernel
    in HBM (kh*kw <= 95) and on NCHW maps is gathered."""
    import cpb200

    dev = engine.device
    m = torch.randn(2, 12, 12, 3, device=dev)
    rc, err = _raw_gather(engine, GC.pinned(m), 3, 12, 12, 1, 9, 10, 4, 4, 1, 1, 1, 1)
    assert rc == engine.lib.CP_ERR_INVALID and "kernel_size 9x10" in err and "host reader" in err, err
    r = torch.zeros((1, 1), dtype=torch.int32, device=dev)
    with pytest.raises(cpb200._cabi.CpError):
        engine.patch_gather(GC.pinned(m), r, r, 2, 1, (9, 10), 4, 1, layout="nhwc")
    for mm, lay in ((m, 1), (m.permute(0, 3, 1, 2).contiguous(), 0)):
        rc, err = _raw_gather(engine, mm, 3, 12, 12, lay, 9, 10, 4, 4, 1, 1, 1, 1)
        assert rc == 0, err
    rc, err = _raw_gather(engine, m, 3, 12, 12, 1, 10, 10, 4, 4, 1, 1, 1, 1)  # 100 taps: beyond the SIMT tile
    assert rc == engine.lib.CP_ERR_INVALID and "kernel_size 10x10" in err, err
    torch.cuda.synchronize()


@pytest.mark.parametrize("dtype", list(GC.FMAP_DTYPES))
def test_largest_nhwc_simt_window_equals_unfold(engine, dtype):
    """kh*kw = 95, the largest window the 2-D entries take on the NHWC SIMT kernel in HBM (kw = 19 is beyond TMA), over
    c = 140 channels (a full and a partial channel tile), against F.unfold."""
    win = ((5, 19), (2, 9), 1, 1)
    H, W, B, nb = 9, 21, 3, 2
    nchw = GC.special_map((nb * B, 140, H, W), dtype, 95, engine.device)
    rx, ry, P = _points(nb, *_out_size(H, W, win), engine.device)
    for relu in (False, True):
        got = _gather(engine, "nhwc_simt", nchw, rx, ry, B, P, win, relu)
        torch.cuda.synchronize()
        GC.assert_same_bits(got.cpu(), _unfold_oracle(nchw, rx, ry, B, win, relu))


def test_reference_entries_still_refuse_even_kernels(engine):
    f = torch.zeros(2, 16, 7, 7, device=engine.device)
    rc, err = _raw_gather(engine, f, 16, 7, 7, 0, 2, 2, 0, 0, 1, 1, 1, 1, entry="typed")
    assert rc == engine.lib.CP_ERR_INVALID and "odd" in err
    ffi, lib = engine.ffi, engine.lib
    r = torch.zeros((1, 1), dtype=torch.int32, device=engine.device)
    X = torch.empty((2, 64), device=engine.device)
    rc = lib.cp_patch_gather(engine.h, ffi.cast("const float*", f.data_ptr()), 1, 2, 16, 7, 7, 0,
                             ffi.cast("const int32_t*", r.data_ptr()), ffi.cast("const int32_t*", r.data_ptr()), 1, 2,
                             0, 1, 0, ffi.cast("float*", X.data_ptr()), 64, ffi.NULL)
    assert rc == lib.CP_ERR_INVALID and b"odd" in ffi.string(lib.cp_last_error())
    rc, err = _raw_gather(engine, f, 16, 7, 7, 0, 2, 2, 0, 0, 1, 1, 1, 1)  # the same window through the new entry
    assert rc == 0, err
    torch.cuda.synchronize()


_KERNEL_CASES = {"tma": ["3x3d2", "3x3d4", "5x5d3", "1x7", "7x1", "1x3", "2x2", "3x5d21s12"],
                 "simt": ["3x3d12"], "host": ["3x3d2", "3x3d12", "1x7", "2x2"]}
_REPEAT = 3


def _profile_kernel_cases():
    """Runs every case of _KERNEL_CASES _REPEAT times inside one profiler session; returns the gather kernels'
    names."""
    import cpb200
    from torch.profiler import ProfilerActivity, profile

    engine = cpb200.get_engine()
    dev = engine.device
    H, B, nb, c = 11, 2, 2, 64
    runs = []
    for kind, names in _KERNEL_CASES.items():
        for wname in names:
            k, pad, stride, dil = win = WINDOWS[wname]
            Ho, Wo = _out_size(H, H, win)
            rx, ry, P = _points(nb, Ho, Wo, dev)
            m = torch.randn((nb * B, H, H, c), device=dev)
            if kind == "host":
                m = GC.pinned(m)
            call = (lambda m=m, rx=rx, ry=ry, P=P, k=k, pad=pad, stride=stride, dil=dil:
                    engine.patch_gather(m, rx, ry, B, P, k, pad, stride, layout="nhwc", dilation=dil))
            call()  # warm-up (module load)
            runs.append(call)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for call in runs:
            for _ in range(_REPEAT):
                call()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "patch_gather" in e.name and e.device_type.name == "CUDA"]


def test_intended_kernels_run(engine):
    """One profiler session: eligible dilated (d <= 8) and rectangular NHWC HBM windows launch the TMA kernel, d = 12
    the NHWC SIMT kernel, NHWC pinned maps the host reader.  Each case runs _REPEAT times, so a lost activity record
    does not decide the check.  The session runs in a child process: a process that has profiled once loses more
    activity records in its later sessions, and other tests of the suite profile too."""

    def kind_of(n):
        if "patch_gather_nhwc_tma<" in n:
            return "tma"
        if "patch_gather_nhwc_host<" in n:
            return "host"
        if "patch_gather_nhwc<" in n:
            return "simt"
        return n

    want = {kind: _REPEAT * len(cases) for kind, cases in _KERNEL_CASES.items()}
    GC.assert_launch_counts(GC.launched_gather_kernels("test_gpu_conv_geometry"), kind_of, want)


@pytest.mark.parametrize("wname", list(WINDOWS))
def test_gathered_x_reproduces_the_convolution(engine, wname):
    """relu(X) W2' + b2 at the sampled points is F.conv2d(relu(x), W2, b2, stride, padding, dilation) there."""
    k, pad, stride, dil = win = WINDOWS[wname]
    (kh, kw) = _pair(k)
    dev = engine.device
    g = torch.Generator(device=dev)
    g.manual_seed(5)
    c, n, H, W, B, nb = 16, 8, 11, 10, 3, 2
    x = torch.randn((nb * B, c, H, W), generator=g, device=dev)
    W2 = torch.randn((n, c, kh, kw), generator=g, device=dev)
    b2 = torch.randn((n,), generator=g, device=dev)
    Ho, Wo = _out_size(H, W, win)
    rx, ry, P = _points(nb, Ho, Wo, dev)
    X = engine.patch_gather(x, rx, ry, B, P, k, pad, stride, relu=True, dilation=dil)
    got = X.double() @ W2.reshape(n, -1).T.double() + b2.double()
    y = F.conv2d(torch.relu(x).double(), W2.double(), b2.double(), stride=stride, padding=pad, dilation=dil)
    assert y.shape[2:] == (Ho, Wo)
    want = torch.stack([y[b * B + i, :, int(rx[b, p]), int(ry[b, p])] for b in range(nb) for p in range(P)
                        for i in range(B)])
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5)


def _layer(name, c, n, H, k, pad, stride=1, dilation=1, N=1000, B=10, P=10, rank=None):
    import cpb200

    return cpb200.synth.LayerShape(name, c, n, H, k=k, pad=pad, stride=stride, dilation=dilation, N=N, B=B, P=P,
                                   rank=rank)


@pytest.mark.parametrize("mode,tol", [(0, 1e-7), (1, 1e-4)], ids=["fp64", "3xtf32"])
@pytest.mark.parametrize("geom", [dict(k=3, pad=2, dilation=2), dict(k=(1, 7), pad=(0, 3))], ids=["3x3d2", "1x7"])
def test_dictionary_on_dilated_and_rectangular_layers_matches_oracle(engine, mode, tol, geom):
    """decompose.dictionary against oracle.dictionary on X gathered with the layer's window: the same mask, alpha
    probes and numpy RNG draws, weights within tol (relative Frobenius) and newW2 shaped (n, c', kh, kw)."""
    import cpb200
    from cpb200.lib import cfgs, decompose

    engine.gram_mode = mode
    s = _layer("L", 64, 48, 14, **geom)
    d = cpb200.synth.make_problem_numpy(s, 9)
    X, W2, Y = d["X"].astype(np.float64), d["W2"], d["feats"].astype(np.float64)
    assert X.shape == (s.N, s.c, s.kh, s.kw)
    st = O.DictState(alpha=1e-3)
    info = {}
    np.random.seed(77)
    oi, oW, oB = CO.dictionary(X, W2, Y, rank=s.rank, state=st, info=info)
    after_oracle = np.random.get_state()
    cfgs.alpha = 1e-3
    np.random.seed(77)
    idxs, W, B = decompose.dictionary(X, W2, Y, rank=s.rank)
    after_device = np.random.get_state()
    assert np.array_equal(idxs, oi)
    assert decompose.DictionaryInfo.last["probes"] == info["probes"]
    assert cfgs.alpha == st.alpha
    assert after_oracle[2] == after_device[2] and np.array_equal(after_oracle[1], after_device[1])
    assert W.shape == oW.shape == (s.n, int(idxs.sum()), s.kh, s.kw)
    assert GC.rel(W, oW) <= tol and np.abs(B - oB).max() <= tol * max(1.0, np.abs(oB).max())


def _deeplab_inception_layers(N=600, B=4, P=5):
    """DeepLabV3 backbone (3x3, dilation 2 and 4), an ASPP branch (dilation 12) and Inception-v3 factorised kernels
    (1x7 / 7x1, 1x3 / 3x1), at test size."""
    return [_layer("layer3_d2", 64, 48, 28, 3, 2, dilation=2, N=N, B=B, P=P),
            _layer("layer4_d4", 64, 48, 28, 3, 4, dilation=4, N=N, B=B, P=P),
            _layer("aspp_d12", 32, 16, 28, 3, 12, dilation=12, N=400, B=B, P=P),
            _layer("mixed6_1x7", 48, 32, 17, (1, 7), (0, 3), N=N, B=B, P=P),
            _layer("mixed6_7x1", 48, 32, 17, (7, 1), (3, 0), N=N, B=B, P=P),
            _layer("mixed7_1x3", 32, 32, 8, (1, 3), (0, 1), N=400, B=B, P=P),
            _layer("mixed7_3x1", 32, 24, 8, (3, 1), (1, 0), N=400, B=B, P=P),
            _layer("s21", 32, 16, 14, 3, 1, stride=(2, 1), N=400, B=B, P=P)]


def _oracle_layer(s, d):
    """The oracle on one pipeline problem: extract_XY_conv with the layer's window, ReLU, oracle.dictionary with the
    problem's samples and seeds (what oracle.dictionary_kernel does for square layers)."""
    import types

    fm = d["fmap"].float().cpu().numpy() if d.get("layout", "nchw") == "nchw" else \
        d["fmap"].permute(0, 3, 1, 2).float().cpu().numpy()
    pd = {"nPointsPerLayer": s.P, "nBatches": s.nbatch}
    for b in range(s.nbatch):
        pd[(b, "y", "randx")] = d["randx"][b].cpu().numpy()
        pd[(b, "y", "randy")] = d["randy"][b].cpu().numpy()
    spec = types.SimpleNamespace(name="y", kernel_size=s.k, pad=s.pad, stride=s.stride, dilation=s.dilation)
    X = CO.extract_XY_conv(lambda b: {"x": fm[b * s.B:(b + 1) * s.B]}, "x", spec, pd)
    newX = O.relu(np.rollaxis(X.reshape((-1, s.kh, s.kw, X.shape[1])), 3, 1).copy())
    return GC.oracle_on_problem(CO.dictionary, newX, s, d)


@pytest.mark.parametrize("host_layout", ["nchw", "nhwc"])
def test_pipeline_on_deeplab_and_inception_layers(engine, host_layout):
    """prune_layers on dilated and rectangular layers: maps in HBM, read in place from pinned host memory ('zc') or
    staged by DMA ('copy'), NCHW or NHWC on the host -- identical masks, alpha, W and b; two layers against the
    oracle."""
    import cpb200
    from cpb200 import pruner

    eng = cpb200.Engine(nstreams=4)
    eng.gram_mode = 0
    shapes = _deeplab_inception_layers()
    datas = [cpb200.synth.make_problem_device(s, 90 + i, eng, pinned_host=True, host_layout=host_layout)
             for i, s in enumerate(shapes)]
    ref = pruner.prune_layers(eng, shapes, datas)
    torch.cuda.synchronize()
    ref = [(r.idxs.copy(), r.alpha, r.nprobe, r.W.cpu(), r.b.cpu()) for r in ref]
    for policy in ("zc", "copy"):
        got = pruner.prune_layers(eng, shapes, datas, from_host=policy, to_host=True)
        torch.cuda.synchronize()
        for s, (idxs, alpha, nprobe, W, b), r in zip(shapes, ref, got):
            assert np.array_equal(idxs, r.idxs) and alpha == r.alpha and nprobe == r.nprobe, (policy, s.name)
            assert torch.equal(W, r.W) and torch.equal(b, r.b), (policy, s.name)
    if host_layout == "nchw":
        for i in (0, 3):  # layer3_d2 and mixed6_1x7
            s, d = shapes[i], datas[i]
            oi, oW, oB, oalpha, onprobe = _oracle_layer(s, d)
            idxs, alpha, nprobe, W, b = ref[i]
            assert np.array_equal(idxs, oi) and alpha == oalpha and nprobe == onprobe, s.name
            W = W.numpy().reshape(oW.shape)
            assert GC.rel(W, oW) <= 1e-7 and np.abs(b.numpy() - oB).max() <= 1e-7, s.name
    eng.close()


def test_net_with_dilated_and_rectangular_convs_matches_oracle(engine):
    """A Net of ConvSpecs with a 1x7 (pad (0, 3)) and a dilated 3x3 conv: extract_XY and dictionary_kernel against
    the oracle's conv-semantics extract_XY and dictionary on the same blobs and points."""
    import types

    from cpb200.lib import cfgs, net as cpnet

    engine.gram_mode = 0
    r = np.random.RandomState(4)
    Bimg, H, nbat = 4, 12, 6
    images = [r.standard_normal((Bimg, 3, H, H)).astype(np.float32) for _ in range(nbat)]
    geo = {"conv1": (3, 16, 3, 1, 1, 1), "conv2": (16, 24, (1, 7), (0, 3), 1, 1), "conv3": (24, 20, 3, 2, 1, 2)}
    specs, weights, biases, bottom = [], {}, {}, "data"
    for nm, (ci, co, k, pad, stride, dil) in geo.items():
        kh, kw = _pair(k)
        specs.append(cpnet.ConvSpec(nm, bottom, co, k, pad, stride, dilation=dil))
        weights[nm] = (r.standard_normal((co, ci, kh, kw)) * np.sqrt(2.0 / (ci * kh * kw))).astype(np.float32)
        biases[nm] = (0.1 * r.standard_normal(co)).astype(np.float32)
        bottom = nm + "_relu"
    net = cpnet.Net(specs, weights, biases, cpnet.ConvStackForward(images_by_batch=lambda b: images[b]))
    cfgs.c.nBatches, cfgs.c.nPointsPerLayer = nbat, 10
    np.random.seed(12)
    feats, points = net.extract_features(list(geo), save=1)
    net.load_frozen(feats_dict=feats, points_dict=points)
    blobs = [{k: v.float().cpu().numpy() for k, v in net.forward(points[(b, 0)]).items()} for b in range(nbat)]
    for X_name, Y_name in (("conv1", "conv2"), ("conv2", "conv3")):
        ci, co, k, pad, stride, dil = geo[Y_name]
        kh, kw = _pair(k)
        spec = types.SimpleNamespace(name=Y_name, kernel_size=k, pad=pad, stride=stride, dilation=dil)
        want = CO.extract_XY_conv(lambda b: blobs[b], X_name, spec, points)
        XY = net.extract_XY(X_name, Y_name)
        assert XY.dtype == np.float64 and XY.shape == (nbat * 10 * Bimg * kh * kw, ci)
        np.testing.assert_array_equal(XY, want)
        d_prime = int(ci / 1.15)
        cfgs.alpha = 1e-3
        np.random.seed(3)
        idxs, W, B = net.dictionary_kernel(X_name, None, d_prime, Y_name, None)
        newX = O.relu(np.rollaxis(want.reshape((-1, kh, kw, ci)), 3, 1).copy())
        st = O.DictState(alpha=1e-3)
        np.random.seed(3)
        oi, oW, oB = CO.dictionary(newX, weights[Y_name], feats[Y_name] - biases[Y_name], rank=d_prime,
                                  B2=biases[Y_name], state=st)
        assert np.array_equal(idxs, oi) and cfgs.alpha == st.alpha, Y_name
        assert W.shape == oW.shape == (co, int(oi.sum()), kh, kw)
        assert GC.rel(W, oW) <= 1e-7 and np.abs(B - oB).max() <= 1e-7, Y_name
