"""CPU: Conv3d layer problems -- geometry against PyTorch's output size, the numpy gathers against F.conv3d, the TMA
box rule of the 5-D tensor map, the zero-copy line model of NCDHW and NDHWC host maps against a brute-force count,
the transfer plan, and pack / unpack of 5-D weights."""
import numpy as np
import pytest

import conv3d_oracle as C3

torch = pytest.importorskip("torch")
F = pytest.importorskip("torch.nn.functional")

# (kernel_size, padding, stride, dilation) as nn.Conv3d takes them
WINDOWS = {
    "1x1x1": (1, 0, 1, 1), "3x3x3": (3, 1, 1, 1), "1x3x3": ((1, 3, 3), (0, 1, 1), 1, 1),
    "3x1x1": ((3, 1, 1), (1, 0, 0), 1, 1), "stem3x7x7": ((3, 7, 7), (1, 3, 3), (1, 2, 2), 1),
    "3x3x3d2": (3, 2, 1, 2), "3x3x3d121": (3, (1, 2, 1), 1, (1, 2, 1)), "3x3x3s2": (3, 1, 2, 1),
}


def _shape(win, c=6, n=5, D=7, H=9, W=8, N=60, B=3, P=4):
    import cpb200

    k, pad, stride, dil = win
    return cpb200.synth.LayerShape3d("L", c, n, D, H, k=k, pad=pad, stride=stride, dilation=dil, W=W, N=N, B=B, P=P)


@pytest.mark.parametrize("wname", list(WINDOWS))
def test_geometry_matches_pytorch_output_size(wname):
    k, pad, stride, dil = WINDOWS[wname]
    s = _shape(WINDOWS[wname])
    y = F.conv3d(torch.zeros(1, s.c, s.D, s.H, s.W), torch.zeros((s.n, s.c) + s.window), stride=stride, padding=pad,
                 dilation=dil)
    assert tuple(y.shape[2:]) == (s.To, s.Ho, s.Wo)
    assert s.k2 == s.kt * s.kh * s.kw and s.K == s.c * s.k2
    assert s.conv_args() == dict(k=k, pad=pad, stride=stride, dilation=dil)
    assert s.cost() > 0


@pytest.mark.parametrize("wname", list(WINDOWS))
def test_numpy_gathers_reproduce_conv3d(wname):
    """synth's gather and the test-side oracle's agree bit for bit, and X W' + b is F.conv3d at the points."""
    import cpb200

    k, pad, stride, dil = WINDOWS[wname]
    s = _shape(WINDOWS[wname])
    d = cpb200.synth.make_problem_numpy(s, 3, noise=0.0)
    X = d["X"]
    assert X.shape == (s.N, s.c) + s.window and X.dtype == np.float32
    Xo = C3.gather3d(d["fmap"], d["randt"], d["randx"], d["randy"], s.B, k, pad, stride, dil, relu=True)
    assert np.array_equal(X.reshape(s.N, -1), Xo)
    x = torch.relu(torch.as_tensor(d["fmap"], dtype=torch.float64))
    y = F.conv3d(x, torch.as_tensor(d["W2"], dtype=torch.float64), torch.as_tensor(d["b2"], dtype=torch.float64),
                 stride=stride, padding=pad, dilation=dil).numpy()
    want = np.stack([y[b * s.B + i, :, d["randt"][b, p], d["randx"][b, p], d["randy"][b, p]]
                     for b in range(s.nbatch) for p in range(s.P) for i in range(s.B)])
    got = X.reshape(s.N, -1).astype(np.float64) @ d["W2"].reshape(s.n, -1).T.astype(np.float64) + d["b2"]
    np.testing.assert_allclose(got, want, rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(d["feats"], want, rtol=1e-6, atol=1e-6)  # noise = 0: the targets are the convolution


def _box_rule(c_box, win):
    """Elements a tiled TMA request with the 3-D path's box and traversal strides delivers (ceil(box / stride) per
    dimension), and the window's element count."""
    (kt, kh, kw), _, _, (dt, dh, dw) = (C3._triple(v) for v in win)
    box = [c_box, (kw - 1) * dw + 1, (kh - 1) * dh + 1, (kt - 1) * dt + 1, 1]
    estr = [1, dw, dh, dt, 1]
    return int(np.prod([-(-b // e) for b, e in zip(box, estr)])), c_box * kt * kh * kw


@pytest.mark.parametrize("wname", list(WINDOWS))
def test_tma_box_delivers_exactly_the_window(wname):
    for c_box in (16, 64, 128, 256):
        got, want = _box_rule(c_box, WINDOWS[wname])
        assert got == want
    for d in range(1, 9):  # every traversal stride the tensor map allows, up to 16 taps per axis
        for k in (1, 2, 3, 5, 16):
            got, want = _box_rule(32, (k, 0, 1, d))
            assert got == want and (k - 1) * d + 1 <= 256 or (k - 1) * d + 1 > 256


def _brute_lines(layout, c, D, H, W, win, esize, img, t, x, y):
    """128-byte lines of a map (base 128-byte aligned) that the in-bounds taps of one window touch."""
    (kt, kh, kw), (pt, ph, pw), (st, sh, sw), (dt, dh, dw) = (C3._triple(v) for v in win)
    lines = set()
    for u in range(kt):
        tt = st * t - pt + dt * u
        for i in range(kh):
            yy = sh * x - ph + dh * i
            if not (0 <= tt < D and 0 <= yy < H):
                continue
            for j in range(kw):
                xx = sw * y - pw + dw * j
                if not 0 <= xx < W:
                    continue
                if layout == "ndhwc":
                    start = (((img * D + tt) * H + yy) * W + xx) * c * esize
                    lines.update(range(start // 128, (start + c * esize - 1) // 128 + 1))
                else:
                    for a in range(c):
                        lines.add(((((img * c + a) * D + tt) * H + yy) * W + xx) * esize // 128)
    return len(lines)


@pytest.mark.parametrize("layout", ["ncdhw", "ndhwc"])
@pytest.mark.parametrize("esize", [4, 2])
@pytest.mark.parametrize("c", [3, 16, 24, 64])
@pytest.mark.parametrize("wname", list(WINDOWS))
def test_line_model_bounds_the_brute_force_count(layout, esize, c, wname):
    """NDHWC: the model is an upper bound.  NCDHW: the model counts a short row of taps as one line, the convention of
    the 2-D NCHW count ZC_LINES_PER_S was measured with; a row that straddles a line boundary touches one more, so the
    bound holds up to one line per row (c*kt*kh rows)."""
    import cpb200
    from cpb200 import pruner

    win = WINDOWS[wname]
    k, pad, stride, dil = win
    s = cpb200.synth.LayerShape3d("L", c, 4, 6, 27, k=k, pad=pad, stride=stride, dilation=dil, W=26, N=1, B=1, P=1)
    model = pruner.zero_copy_lines(s, esize, layout)
    r = np.random.RandomState(c + esize)
    pts = [(0, 0, 0), (s.To - 1, s.Ho - 1, s.Wo - 1), (s.To // 2, 0, s.Wo - 1)] + \
        [tuple(int(v) for v in p) for p in zip(r.randint(0, s.To, 12), r.randint(0, s.Ho, 12), r.randint(0, s.Wo, 12))]
    slack = 0 if layout == "ndhwc" else s.c * s.kt * s.kh
    for t, x, y in pts:
        assert _brute_lines(layout, c, s.D, s.H, s.W, win, esize, int(r.randint(0, 3)), t, x, y) <= model + slack


def test_line_model_is_kt_frames_of_the_2d_count():
    """NCDHW: c*kt*kh rows of kw taps; NDHWC: kt*kh runs of kw*c*esize bytes (+ a line per run for a pixel stride off
    the 128-byte grid) -- kt times the count of the same (kh, kw) window on one frame."""
    import cpb200
    from cpb200 import pruner

    L2, L3 = cpb200.synth.LayerShape, cpb200.synth.LayerShape3d
    for c, H in ((64, 56), (128, 28), (256, 14), (512, 7), (3, 112)):
        s3 = L3("a", c, c, 8, H)
        s2 = L2("b", c, c, H)
        for es in (4, 2):
            assert pruner.zero_copy_lines(s3, es, "ncdhw") == 3 * pruner.zero_copy_lines(s2, es, "nchw")
            assert pruner.zero_copy_lines(s3, es, "ndhwc") == 3 * pruner.zero_copy_lines(s2, es, "nhwc")
    # r3d_18 layer4 (c = 512, fp32): 9 runs of 3 x 2048 bytes = 48 lines each
    s = L3("l4", 512, 512, 2, 7)
    assert pruner.zero_copy_lines(s, 4, "ndhwc") == 5000 * 9 * 48
    # NCDHW: per channel and frame, three 28-byte rows of a 7-wide frame span 68 bytes: at most 2 lines, 3 frames
    assert pruner.zero_copy_lines(s, 4, "ncdhw") == 5000 * 512 * 3 * 2


def test_plan_rule_on_r3d18(monkeypatch):
    """h2d_plan on the r3d_18 layers follows the rule of the 2-D layers: DMA when the map is small enough and the copy
    is cheaper than 0.8 of the in-place reader's modelled time for the host map's layout."""
    import cpb200
    from cpb200 import pruner

    monkeypatch.delenv("CPB200_DMA_MAX_MB", raising=False)
    monkeypatch.delenv("CPB200_DMA_RATIO", raising=False)
    shapes = cpb200.synth.r3d18_layers()
    assert [s.k2 for s in shapes] == [27] * 16 and all(s.N == 5000 for s in shapes)
    for dtype in (torch.float32, torch.bfloat16):
        es = torch.empty((), dtype=dtype).element_size()
        for layout in ("ncdhw", "ndhwc"):
            datas = []
            for s in shapes:
                shp = (s.nbatch * s.B, s.D, s.H, s.W, s.c) if layout == "ndhwc" else (s.nbatch * s.B, s.c, s.D, s.H, s.W)
                datas.append(dict(fmap_host=torch.empty(shp, dtype=dtype, device="meta"), host_layout=layout))
            rate = pruner.ZC_NHWC_LINES_PER_S if layout == "ndhwc" else pruner.ZC_LINES_PER_S
            want = []
            for s, d in zip(shapes, datas):
                nbytes = d["fmap_host"].numel() * es
                t_zc = pruner.zero_copy_lines(s, es, layout) / rate
                want.append("dma" if (nbytes <= 300e6 and nbytes / 50e9 + 1e-4 < 0.8 * t_zc) else "zc")
            assert pruner.h2d_plan(shapes, datas, True) == want
            # without a host_layout key a Conv3d layer's map is read as NCDHW
            bare = [dict(fmap_host=d["fmap_host"]) for d in datas]
            if layout == "ncdhw":
                assert pruner.h2d_plan(shapes, bare, True) == want


def test_pack_unpack_round_trip_of_5d_weights():
    import cpb200
    from cpb200 import pruner as pr

    shapes = [cpb200.synth.LayerShape3d("a", 12, 7, 4, 6, k=(3, 1, 2), pad=(1, 0, 1), N=60, B=3, P=4, rank=9),
              cpb200.synth.LayerShape("b", 10, 5, 6, k=3, N=60, B=3, P=4, rank=8)]
    r = np.random.RandomState(2)
    sizes = [pr.slot_size(s.c, s.n, s.k2, s.rank, 0.1) for s in shapes]
    buf = torch.zeros(sum(sizes), dtype=torch.float64)
    want, off = [], 0
    for s, sz in zip(shapes, sizes):
        idxs = np.zeros(s.c, dtype=bool)
        idxs[r.choice(s.c, s.rank, replace=False)] = True
        W = torch.as_tensor(r.standard_normal((s.n, s.rank * s.k2)))
        b = torch.as_tensor(r.standard_normal(s.n))
        pr.pack_result(buf, off, idxs, W, b, 0.25, 3, s.c, s.n, s.k2)
        want.append((idxs, W.numpy(), b.numpy()))
        off += sz
    out = pr.unpack_network(shapes, [0, 0], sizes, buf.view(1, -1))
    assert out[0]["W"].shape == (7, 9, 3, 1, 2) and out[1]["W"].shape == (5, 8, 3, 3)
    for (idxs, W, b), o, s in zip(want, out, shapes):
        assert np.array_equal(o["idxs"], idxs) and np.array_equal(o["b"], b)
        assert np.array_equal(o["W"].reshape(s.n, -1), W) and o["alpha"] == 0.25 and o["nprobe"] == 3
    assert pr.window_of(shapes[0]) == (3, 1, 2) and pr.window_of(shapes[1]) == (3, 3)


def test_conv3d_oracle_dictionary_shapes():
    """The test-side oracle on a 3x3x3 layer returns (n, c', 3, 3, 3) weights: the least squares of Y on the kept
    channels' columns."""
    import cp_oracle as O

    import cpb200

    s = cpb200.synth.LayerShape3d("L", 16, 12, 4, 6, N=600, B=6, P=10)
    d = cpb200.synth.make_problem_numpy(s, 4)
    X, W2, Y = d["X"].astype(np.float64), d["W2"], d["feats"].astype(np.float64)
    samples = np.random.RandomState(0).randint(0, s.N, s.S)
    idxs, W, B = C3.dictionary(X, W2, Y, rank=s.rank, state=O.DictState(alpha=1e-3), samples=samples)
    assert W.shape == (12, int(idxs.sum()), 3, 3, 3)
    Xk = X[:, idxs].reshape(s.N, -1)
    Xc, Yc = Xk - Xk.mean(0), Y - Y.mean(0)
    Wls = np.linalg.lstsq(Xc, Yc, rcond=None)[0].T
    np.testing.assert_allclose(W.reshape(12, -1), Wls, rtol=1e-7, atol=1e-9)
