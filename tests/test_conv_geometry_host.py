"""CPU: the host side of general convolution windows (rectangular kernels, per-axis padding and stride, dilation) --
LayerShape's geometry against torch.nn.Conv2d, the numpy and oracle gathers against F.unfold, the TMA box rule the
dilated gather relies on, and the zero-copy line model (an upper bound on a brute-force count, unchanged for square
windows, so every existing transfer plan is unchanged)."""
import types

import numpy as np
import pytest

import conv_oracle as CO
import cp_oracle as O

torch = pytest.importorskip("torch")
F = pytest.importorskip("torch.nn.functional")

# (kernel_size, padding, stride, dilation)
WINDOWS = [((1, 3), (0, 1), 1, 1), ((3, 1), (1, 0), 1, 1), ((1, 7), (0, 3), 1, 1), ((7, 1), (3, 0), 1, 1),
           ((2, 2), 0, 1, 1), ((2, 2), 1, 1, 1), (3, 2, 1, 2), (3, 4, 1, 4), (5, 6, 1, 3), (3, 12, 1, 12),
           (3, 1, (2, 1), 1), ((3, 7), (0, 3), 1, 1), ((3, 5), (2, 2), (1, 2), (2, 1)), (3, 1, 1, 1), (1, 0, 2, 1)]


def _pair(v):
    return tuple(v) if isinstance(v, tuple) else (v, v)


@pytest.mark.parametrize("win", WINDOWS)
def test_layer_shape_geometry_follows_conv2d(win):
    import cpb200

    k, pad, stride, dil = win
    s = cpb200.synth.LayerShape("L", 6, 4, 13, k=k, pad=pad, stride=stride, dilation=dil, W=11, N=60, B=3, P=5)
    (kh, kw), (ph, pw), (sh, sw), (dh, dw) = (_pair(v) for v in win)
    assert (s.kh, s.kw, s.pad_h, s.pad_w, s.stride_h, s.stride_w, s.dil_h, s.dil_w) == (kh, kw, ph, pw, sh, sw, dh, dw)
    assert s.k2 == kh * kw and s.K == 6 * kh * kw and (s.H, s.W) == (13, 11)
    y = F.conv2d(torch.zeros(1, 6, 13, 11), torch.zeros(4, 6, kh, kw), stride=stride, padding=pad, dilation=dil)
    assert (s.Ho, s.Wo) == tuple(y.shape[2:])
    assert s.conv_args() == dict(k=k, pad=pad, stride=stride, dilation=dil)


def test_square_layer_shapes_keep_their_plain_fields():
    import cpb200

    for s in cpb200.synth.vgg16_layers() + cpb200.synth.resnet50_layers():
        assert isinstance(s.k, int) and isinstance(s.pad, int) and isinstance(s.stride, int)
        assert s.k2 == s.k * s.k and s.W == s.H and s.Ho == (s.H + 2 * s.pad - s.k) // s.stride + 1 and s.Wo == s.Ho


def _unfold_rows(fmap, randx, randy, B, win):
    k, pad, stride, dil = win
    x = torch.as_tensor(fmap)
    _, _, H, W = x.shape
    U = F.unfold(x, _pair(k), dilation=_pair(dil), padding=_pair(pad), stride=_pair(stride))
    (kh, kw), (ph, pw), (sh, sw), (dh, dw) = (_pair(v) for v in win)
    Wo = (W + 2 * pw - dw * (kw - 1) - 1) // sw + 1
    nb, P = randx.shape
    return torch.stack([U[b * B + i, :, int(randx[b, p]) * Wo + int(randy[b, p])]
                        for b in range(nb) for p in range(P) for i in range(B)]).numpy()


@pytest.mark.parametrize("win", WINDOWS)
def test_numpy_and_oracle_gathers_equal_unfold(win):
    """synth.gather_patches_numpy and oracle.extract_XY_conv against F.unfold at every output point."""
    import cpb200

    k, pad, stride, dil = win
    s = cpb200.synth.LayerShape("L", 5, 4, 12, k=k, pad=pad, stride=stride, dilation=dil, W=10, N=60, B=3, P=4)
    r = np.random.RandomState(1)
    fmap = r.standard_normal((s.nbatch * s.B, s.c, s.H, s.W)).astype(np.float32)
    randx = r.randint(0, s.Ho, (s.nbatch, s.P)).astype(np.int32)
    randy = r.randint(0, s.Wo, (s.nbatch, s.P)).astype(np.int32)
    randx[0, 0], randy[0, 0], randx[-1, -1], randy[-1, -1] = 0, 0, s.Ho - 1, s.Wo - 1
    want = _unfold_rows(fmap, randx, randy, s.B, win)
    got = cpb200.synth.gather_patches_numpy(fmap, randx, randy, s.B, k, pad, stride, relu=False, dilation=dil)
    np.testing.assert_array_equal(got.reshape(s.N, -1), want)
    pd = {"nPointsPerLayer": s.P, "nBatches": s.nbatch}
    for b in range(s.nbatch):
        pd[(b, "y", "randx")], pd[(b, "y", "randy")] = randx[b], randy[b]
    spec = types.SimpleNamespace(name="y", kernel_size=k, pad=pad, stride=stride, dilation=dil)
    XY = CO.extract_XY_conv(lambda b: {"x": fmap[b * s.B:(b + 1) * s.B]}, "x", spec, pd)
    assert XY.dtype == np.float64 and XY.shape == (s.N * s.k2, s.c)
    np.testing.assert_array_equal(XY.reshape(s.N, s.k2, s.c).transpose(0, 2, 1).reshape(s.N, -1), want)
    if isinstance(k, int) and k % 2 == 1 and dil == 1 and isinstance(pad, int) and isinstance(stride, int):
        square = O.ConvSpec("y", "x", k, pad, stride)  # the reference's statement, for square windows
        np.testing.assert_array_equal(XY, O.extract_XY(lambda b: {"x": fmap[b * s.B:(b + 1) * s.B]}, "x", square, pd))


def _tma_box(cbox, kh, kw, dh, dw):
    return [cbox, (kw - 1) * dw + 1, (kh - 1) * dh + 1, 1], [1, dw, dh, 1]


@pytest.mark.parametrize("kh,kw,dh,dw", [(3, 3, 1, 1), (3, 3, 2, 2), (3, 3, 4, 4), (3, 3, 8, 8), (5, 5, 3, 3),
                                         (1, 7, 1, 1), (7, 1, 1, 1), (16, 16, 1, 1), (3, 5, 2, 1), (2, 2, 7, 5)])
def test_tma_box_delivers_exactly_the_window(kh, kw, dh, dw):
    """CPU model of the dilated TMA stage (csrc/gather_tma.cu): a box (c_box, (kw-1) dw + 1, (kh-1) dh + 1, 1) with
    traversal strides (1, dw, dh, 1) delivers ceil(box / stride) elements per dimension -- the bytes expect_tx must
    announce -- which are exactly the kh x kw taps of the window, in the stage order [i][j][channel]."""
    cbox = 16
    box, estr = _tma_box(cbox, kh, kw, dh, dw)
    assert all(b <= 256 for b in box) and all(e <= 8 for e in estr)
    delivered = [-(-b // e) for b, e in zip(box, estr)]
    assert np.prod(delivered) == cbox * kh * kw
    # the traversal: element m of dimension d sits at box offset m * estr[d]
    taps = [(m2 * estr[2], m1 * estr[1]) for m2 in range(delivered[2]) for m1 in range(delivered[1])]
    assert taps == [(i * dh, j * dw) for i in range(kh) for j in range(kw)]


def _old_zero_copy_lines(s, esize=4, layout="nchw"):
    """zero_copy_lines as it was for square, undilated windows only."""
    if layout == "nhwc":
        run = s.k * s.c * esize
        per_run = -(-run // 128) + (1 if (s.c * esize) % 128 else 0)
        return s.N * s.k * per_run
    row = s.W * esize if hasattr(s, "W") else esize * 64
    lines = min(s.k, -(-((s.k - 1) * row + s.k * esize) // 128) + 1) if s.k > 1 else 1
    return s.N * s.c * lines


def _square_shapes():
    import cpb200

    out = cpb200.synth.vgg16_layers() + cpb200.synth.resnet50_layers()
    for c in (1, 3, 5, 12, 16, 24, 32, 64, 96, 512, 2048):
        for k in (1, 3, 5, 7, 9):
            out.append(cpb200.synth.LayerShape("s", c, 8, 20, k=k, pad=k // 2, N=100, B=2, P=5))
            out.append(types.SimpleNamespace(N=1, c=c, k=k, W=7))
            out.append(types.SimpleNamespace(N=1, c=c, k=k))
    return out


def test_line_model_is_unchanged_for_square_windows():
    from cpb200 import pruner

    for s in _square_shapes():
        for es in (4, 2):
            for layout in ("nchw", "nhwc"):
                assert pruner.zero_copy_lines(s, es, layout) == _old_zero_copy_lines(s, es, layout)


def _brute_nhwc_lines(c, H, W, win, esize, img, x, y):
    """128-byte lines of an NHWC map (base 128-byte aligned) that the in-bounds taps of one window touch."""
    (kh, kw), (ph, pw), (sh, sw), (dh, dw) = (_pair(v) for v in win)
    lines = set()
    for i in range(kh):
        yy = sh * x - ph + dh * i
        if not 0 <= yy < H:
            continue
        for j in range(kw):
            xx = sw * y - pw + dw * j
            if 0 <= xx < W:
                start = ((img * H + yy) * W + xx) * c * esize
                lines.update(range(start // 128, (start + c * esize - 1) // 128 + 1))
    return len(lines)


@pytest.mark.parametrize("esize", [4, 2])
@pytest.mark.parametrize("c", [1, 3, 5, 12, 16, 24, 32, 64, 96, 512])
@pytest.mark.parametrize("win", WINDOWS)
def test_nhwc_line_model_bounds_rectangular_and_dilated_windows(esize, c, win):
    import cpb200
    from cpb200 import pruner

    k, pad, stride, dil = win
    H, W = 27, 26
    s = cpb200.synth.LayerShape("L", c, 4, H, k=k, pad=pad, stride=stride, dilation=dil, W=W, N=1, B=1, P=1)
    model = pruner.zero_copy_lines(s, esize, "nhwc")
    r = np.random.RandomState(c + esize)
    pts = [(0, 0), (0, s.Wo - 1), (s.Ho - 1, 0), (s.Ho - 1, s.Wo - 1)] + \
        [(int(a), int(b)) for a, b in zip(r.randint(0, s.Ho, 40), r.randint(0, s.Wo, 40))]
    for x, y in pts:
        assert _brute_nhwc_lines(c, H, W, win, esize, int(r.randint(0, 4)), x, y) <= model, (x, y, model)


def test_nchw_line_model_of_dilated_and_rectangular_windows():
    """NCHW: a window is c*kh rows of kw taps; the rows of a channel are dil_h*W*esize bytes apart, so dilation only
    spreads them; a dilated fp32 3x3 on a 28-wide map touches a line per row, like the undilated one."""
    import cpb200
    from cpb200 import pruner

    L = cpb200.synth.LayerShape
    und = L("u", 256, 256, 28, k=3, pad=1)
    for d in (2, 4):
        s = L("d", 256, 256, 28, k=3, pad=d, dilation=d)
        assert pruner.zero_copy_lines(s) == pruner.zero_copy_lines(und) == 5000 * 256 * 3
    assert pruner.zero_copy_lines(L("r", 192, 192, 17, k=(1, 7), pad=(0, 3))) == 5000 * 192 * 1
    # 7 rows 68 bytes apart: the whole 412-byte column spans at most 5 lines
    assert pruner.zero_copy_lines(L("r", 192, 192, 17, k=(7, 1), pad=(3, 0))) == 5000 * 192 * 5
    # a dilated row counts the lines of its span, at most one per tap
    assert pruner.zero_copy_lines(L("w", 8, 8, 64, k=(1, 5), pad=(0, 24), dilation=12)) == 5000 * 8 * 2
    assert pruner.zero_copy_lines(L("w", 8, 8, 256, k=(1, 3), pad=(0, 64), dilation=64)) == 5000 * 8 * 3


def test_plans_of_the_square_workloads_are_unchanged(monkeypatch):
    """h2d_plan on the VGG-16 and ResNet-50 workloads gives what the square-only line model gave."""
    import cpb200
    from cpb200 import pruner

    monkeypatch.delenv("CPB200_DMA_MAX_MB", raising=False)
    monkeypatch.delenv("CPB200_DMA_RATIO", raising=False)
    for shapes in (cpb200.synth.vgg16_layers(), cpb200.synth.resnet50_layers()):
        for dtype in (torch.float32, torch.bfloat16):
            for layout in ("nchw", "nhwc"):
                es = torch.empty((), dtype=dtype).element_size()
                datas = []
                for s in shapes:
                    shape = (s.nbatch * s.B, s.H, s.W, s.c) if layout == "nhwc" else (s.nbatch * s.B, s.c, s.H, s.W)
                    datas.append(dict(fmap_host=torch.empty(shape, dtype=dtype, device="meta"), host_layout=layout))
                rate = pruner.ZC_NHWC_LINES_PER_S if layout == "nhwc" else pruner.ZC_LINES_PER_S
                want = []
                for s, d in zip(shapes, datas):
                    nbytes = d["fmap_host"].numel() * es
                    t_zc = _old_zero_copy_lines(s, es, layout) / rate
                    want.append("dma" if (nbytes <= 300e6 and nbytes / 50e9 + 1e-4 < 0.8 * t_zc) else "zc")
                assert pruner.h2d_plan(shapes, datas, True) == want


def test_conv_oracle_dictionary_on_rectangular_layers():
    """The test-side oracle on a 1x3 layer returns (n, c', 1, 3) weights, and the sklearn cross-check selects the same
    channels as the restated coordinate descent; on a square layer it is cp_oracle.dictionary itself."""
    import cpb200

    s = cpb200.synth.LayerShape("L", 24, 16, 10, k=(1, 3), pad=(0, 1), N=600, B=6, P=10)
    d = cpb200.synth.make_problem_numpy(s, 4)
    X, W2, Y = d["X"].astype(np.float64), d["W2"], d["feats"].astype(np.float64)
    samples = np.random.RandomState(0).randint(0, s.N, s.S)
    res = {}
    for engine in ("restated", "sklearn"):
        if engine == "sklearn":
            pytest.importorskip("sklearn")
        st = O.DictState(alpha=1e-3)
        res[engine] = CO.dictionary(X, W2, Y, rank=s.rank, state=st, samples=samples, engine=engine)
    idxs, W, B = res["restated"]
    assert W.shape == (16, int(idxs.sum()), 1, 3)
    assert np.array_equal(idxs, res["sklearn"][0])
    # the weights are the least squares of Y on the kept channels' columns (with an intercept)
    Xk = X[:, idxs].reshape(s.N, -1)
    Xc, Yc = Xk - Xk.mean(0), Y - Y.mean(0)
    Wls = np.linalg.lstsq(Xc, Yc, rcond=None)[0].T
    np.testing.assert_allclose(W.reshape(16, -1), Wls, rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(B, Y.mean(0) - Xk.mean(0) @ Wls.T, rtol=1e-8, atol=1e-10)
    sq = cpb200.synth.LayerShape("Q", 24, 16, 10, k=3, pad=1, N=600, B=6, P=10)
    d = cpb200.synth.make_problem_numpy(sq, 5)
    X, W2, Y = d["X"].astype(np.float64), d["W2"], d["feats"].astype(np.float64)
    a = CO.dictionary(X, W2, Y, rank=sq.rank, state=O.DictState(alpha=1e-3), samples=samples)
    b = O.dictionary(X, W2, Y, rank=sq.rank, state=O.DictState(alpha=1e-3), samples=samples)
    assert all(np.array_equal(u, v) for u, v in zip(a, b))
