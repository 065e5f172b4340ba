"""CPU: transposed-convolution layer problems (ConvTranspose2d / ConvTranspose3d) -- the numpy gathers against
F.conv_transpose2d / 3d at every output point, the phase arithmetic of the kernels against brute force, output sizes
against PyTorch's, the zero-copy line model against a brute-force count, and pack / unpack of transposed weights."""
import numpy as np
import pytest

import conv_transpose_oracle as CT

torch = pytest.importorskip("torch")
F = pytest.importorskip("torch.nn.functional")

# (kernel_size, padding, stride, dilation, output_padding) as nn.ConvTranspose2d takes them
GEOMS2D = {
    "k2s2": (2, 0, 2, 1, 0), "k4s2p1": (4, 1, 2, 1, 0), "k3s2p1op1": (3, 1, 2, 1, 1), "k3s2d2": (3, 0, 2, 2, 0),
    "k3s1p1": (3, 1, 1, 1, 0), "rect": ((3, 4), (1, 2), (2, 3), (2, 1), (1, 0)),
    "s4d2": ((3, 5), (1, 0), (4, 3), (2, 2), (0, 1)),
}
# the same for nn.ConvTranspose3d: (1, 2, 2) and 2x2x2 up-convolutions, overlapping and rectangular windows
GEOMS3D = {
    "1x2x2": ((1, 2, 2), 0, (1, 2, 2), 1, 0), "2x2x2": (2, 0, 2, 1, 0), "3x3x3s2p1op1": (3, 1, 2, 1, 1),
    "rect3d": ((2, 3, 4), (0, 1, 2), (2, 1, 3), (1, 2, 1), (1, 0, 2)), "3x3x3s2d2": (3, 1, 2, 2, 0),
}


def _all_points(dims, nbatch):
    """Every output point of a dims-shaped output map, for each batch: (arrays (nbatch, P) per axis, P)."""
    grids = np.meshgrid(*[np.arange(n) for n in dims], indexing="ij")
    pts = [np.tile(g.reshape(1, -1), (nbatch, 1)).astype(np.int32) for g in grids]
    return pts, pts[0].shape[1]


def _shape(name, d3, **kw):
    import cpb200

    k, pad, stride, dil, op = (GEOMS3D if d3 else GEOMS2D)[name]
    if d3:
        return cpb200.synth.LayerShape3d("L", kw.pop("c", 5), kw.pop("n", 4), kw.pop("D", 3), kw.pop("H", 5), k=k,
                                         pad=pad, stride=stride, dilation=dil, output_padding=op, W=kw.pop("W", 4),
                                         transposed=True, **kw)
    return cpb200.synth.LayerShape("L", kw.pop("c", 5), kw.pop("n", 4), kw.pop("H", 6), k=k, pad=pad, stride=stride,
                                   dilation=dil, output_padding=op, W=kw.pop("W", 5), transposed=True, **kw)


@pytest.mark.parametrize("name", list(GEOMS2D))
def test_oracle_reproduces_conv_transpose2d(name):
    """X (every output point) times weight.transpose(0, 1).reshape(n, -1).T is F.conv_transpose2d, in fp64; synth's
    vectorised restatement gives the oracle's X bit for bit."""
    import cpb200

    k, pad, stride, dil, op = GEOMS2D[name]
    s = _shape(name, False, N=1, B=1, P=1)
    r = np.random.RandomState(7)
    B, nb = 2, 2
    x = r.standard_normal((nb * B, s.c, s.H, s.W))
    w = r.standard_normal((s.c, s.n, s.kh, s.kw))  # ConvTranspose2d.weight
    y = F.conv_transpose2d(torch.as_tensor(x), torch.as_tensor(w), stride=stride, padding=pad, output_padding=op,
                           dilation=dil).numpy()
    assert y.shape[2:] == (s.Ho, s.Wo)
    (rx, ry), P = _all_points((s.Ho, s.Wo), nb)
    X = CT.gather_tr(x, rx, ry, B, k, pad, stride, dil)
    got = X @ w.transpose(1, 0, 2, 3).reshape(s.n, -1).T
    want = np.stack([y[b * B + i, :, rx[b, p], ry[b, p]] for b in range(nb) for p in range(P) for i in range(B)])
    assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max())
    Xs = cpb200.synth.gather_patches_tr_numpy(x, rx, ry, B, k, pad, stride, relu=False, dilation=dil)
    assert np.array_equal(Xs.reshape(X.shape), X)
    Xr = cpb200.synth.gather_patches_tr_numpy(x, rx, ry, B, k, pad, stride, relu=True, dilation=dil)
    assert np.array_equal(Xr.reshape(X.shape), CT.gather_tr(x, rx, ry, B, k, pad, stride, dil, relu=True))


@pytest.mark.parametrize("name", list(GEOMS3D))
def test_oracle_reproduces_conv_transpose3d(name):
    import cpb200

    k, pad, stride, dil, op = GEOMS3D[name]
    s = _shape(name, True, N=1, B=1, P=1)
    r = np.random.RandomState(8)
    B, nb = 2, 1
    x = r.standard_normal((nb * B, s.c, s.D, s.H, s.W))
    w = r.standard_normal((s.c, s.n) + s.window)
    y = F.conv_transpose3d(torch.as_tensor(x), torch.as_tensor(w), stride=stride, padding=pad, output_padding=op,
                           dilation=dil).numpy()
    assert y.shape[2:] == (s.To, s.Ho, s.Wo)
    (rt, rx, ry), P = _all_points((s.To, s.Ho, s.Wo), nb)
    X = CT.gather_tr3d(x, rt, rx, ry, B, k, pad, stride, dil)
    got = X @ w.transpose(1, 0, 2, 3, 4).reshape(s.n, -1).T
    want = np.stack([y[b * B + i, :, rt[b, p], rx[b, p], ry[b, p]] for b in range(nb) for p in range(P)
                     for i in range(B)])
    assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max())
    Xs = cpb200.synth.gather_patches_tr3d_numpy(x, rt, rx, ry, B, k, pad, stride, relu=False, dilation=dil)
    assert np.array_equal(Xs.reshape(X.shape), X)


def test_structured_rows():
    """k = s = 2: exactly one of the kh*kw taps is valid per point; k = 3, s = d = 2 on a 6 x 6 map: the 225 - 64
    output points with x or y odd have all-zero rows (x + p off the gcd grid on an axis)."""
    r = np.random.RandomState(1)
    x = r.standard_normal((1, 3, 6, 6)) + 5.0  # no zeros among the map's values
    (rx, ry), P = _all_points((12, 12), 1)
    X = CT.gather_tr(x, rx, ry, 1, 2, 0, 2, 1).reshape(P, 3, 4)
    assert np.array_equal((X != 0).sum(axis=2), np.ones((P, 3), dtype=int))
    Ho = (6 - 1) * 2 + 2 * 2 + 1  # k = 3, s = d = 2: 15
    (rx, ry), P = _all_points((Ho, Ho), 1)
    X = CT.gather_tr(x, rx, ry, 1, 3, 0, 2, 2)
    zero = ~(X != 0).any(axis=1)
    assert P == 225 and zero.sum() == 225 - 64  # only (even, even) points read the map
    assert np.array_equal(zero, ((rx[0] % 2) | (ry[0] % 2)).astype(bool))


def _axes(geoms):
    for name, (k, pad, stride, dil, op) in geoms.items():
        nax = 3 if geoms is GEOMS3D else 2
        tr = CT._triple if nax == 3 else CT._pair
        for kk, pp, ss, dd, oo in zip(*(tr(v) for v in (k, pad, stride, dil, op))):
            yield name, kk, pp, ss, dd, oo


def test_phase_arithmetic_matches_brute_force():
    """tr_taps' first valid tap and step (restated in taps_by_phase) give the brute-force valid-tap set at every output
    coordinate of every axis of the geometry tables, for input extents 1 to 9."""
    seen = 0
    for name, k, p, s, d, op in list(_axes(GEOMS2D)) + list(_axes(GEOMS3D)):
        for n in range(1, 10):
            out = (n - 1) * s - 2 * p + d * (k - 1) + op + 1
            for x in range(max(out, 0)):
                assert CT.taps_by_phase(x, p, s, d, k, n) == CT.taps_brute(x, p, s, d, k, n), (name, n, x)
                seen += 1
    # wider strides and dilations than the tables hold
    for s in range(1, 7):
        for d in range(1, 7):
            for k in (1, 2, 3, 5, 8):
                for p in range(0, d * (k - 1) + 1):
                    for n in (1, 2, 5):
                        out = (n - 1) * s - 2 * p + d * (k - 1) + 1
                        for x in range(max(out, 0)):
                            assert CT.taps_by_phase(x, p, s, d, k, n) == CT.taps_brute(x, p, s, d, k, n)
                            seen += 1
    assert seen > 10000


@pytest.mark.parametrize("name", list(GEOMS2D))
def test_layer_shape_output_size_matches_pytorch(name):
    k, pad, stride, dil, op = GEOMS2D[name]
    s = _shape(name, False, N=60, B=3, P=4)
    y = F.conv_transpose2d(torch.zeros(1, s.c, s.H, s.W), torch.zeros(s.c, s.n, s.kh, s.kw), stride=stride,
                           padding=pad, output_padding=op, dilation=dil)
    assert tuple(y.shape[2:]) == (s.Ho, s.Wo)
    assert s.conv_args() == dict(k=k, pad=pad, stride=stride, dilation=dil, transposed=True)
    assert s.k2 == s.kh * s.kw and s.K == s.c * s.k2 and s.cost() > 0


@pytest.mark.parametrize("name", list(GEOMS3D))
def test_layer_shape3d_output_size_matches_pytorch(name):
    k, pad, stride, dil, op = GEOMS3D[name]
    s = _shape(name, True, N=60, B=3, P=4)
    y = F.conv_transpose3d(torch.zeros(1, s.c, s.D, s.H, s.W), torch.zeros((s.c, s.n) + s.window), stride=stride,
                           padding=pad, output_padding=op, dilation=dil)
    assert tuple(y.shape[2:]) == (s.To, s.Ho, s.Wo)
    assert s.conv_args()["transposed"] is True


def test_invalid_output_padding_is_refused():
    """PyTorch's rule output_padding < max(stride, dilation) per axis, and no output_padding on a plain convolution."""
    import cpb200

    L2, L3 = cpb200.synth.LayerShape, cpb200.synth.LayerShape3d
    with pytest.raises(RuntimeError):  # torch refuses it too
        F.conv_transpose2d(torch.zeros(1, 2, 4, 4), torch.zeros(2, 2, 2, 2), stride=2, output_padding=2)
    for kw in (dict(k=2, stride=2, pad=0, output_padding=2), dict(k=3, stride=1, pad=0, output_padding=1),
               dict(k=3, stride=(2, 1), pad=0, dilation=(1, 2), output_padding=(1, 2))):
        with pytest.raises(AssertionError, match="output_padding"):
            L2("L", 4, 4, 5, N=1, B=1, P=1, transposed=True, **kw)
    with pytest.raises(AssertionError, match="output_padding"):
        L3("L", 4, 4, 3, 5, k=2, stride=(1, 2, 2), pad=0, output_padding=(1, 0, 0), N=1, B=1, P=1, transposed=True)
    with pytest.raises(AssertionError, match="output_padding"):
        L2("L", 4, 4, 5, k=3, stride=2, output_padding=1, N=1, B=1, P=1)
    # the largest valid one is accepted, on the axis with the larger dilation
    s = L2("L", 4, 4, 5, k=3, stride=(2, 1), pad=0, dilation=(1, 3), output_padding=(1, 2), N=1, B=1, P=1,
           transposed=True)
    assert (s.Ho, s.Wo) == (4 * 2 + 2 + 1 + 1, 4 + 6 + 2 + 1)


def _brute_lines(layout, s, esize, img, pt):
    """128-byte lines of a map (base 128-byte aligned) that the valid taps of one output point touch."""
    d3 = hasattr(s, "kt")
    D = s.D if d3 else 1
    tt = CT.taps_brute(pt[0], s.pad_t, s.stride_t, s.dil_t, s.kt, D) if d3 else [(0, 0)]
    hh = CT.taps_brute(pt[-2], s.pad_h, s.stride_h, s.dil_h, s.kh, s.H)
    ww = CT.taps_brute(pt[-1], s.pad_w, s.stride_w, s.dil_w, s.kw, s.W)
    lines = set()
    for _, t in tt:
        for _, h in hh:
            for _, w in ww:
                if layout in ("nhwc", "ndhwc"):
                    start = (((img * D + t) * s.H + h) * s.W + w) * s.c * esize
                    lines.update(range(start // 128, (start + s.c * esize - 1) // 128 + 1))
                else:
                    for a in range(s.c):
                        lines.add(((((img * s.c + a) * D + t) * s.H + h) * s.W + w) * esize // 128)
    return len(lines)


@pytest.mark.parametrize("esize", [4, 2])
@pytest.mark.parametrize("c", [3, 16, 24, 64])
@pytest.mark.parametrize("name", list(GEOMS2D) + ["3d:" + n for n in GEOMS3D])
def test_line_model_bounds_the_brute_force_count(name, c, esize):
    """zero_copy_lines of a transposed layer bounds the lines every output point touches, in both layouts."""
    from cpb200 import pruner

    d3 = name.startswith("3d:")
    s = _shape(name[3:] if d3 else name, d3, c=c, N=1, B=1, P=1, **(dict(D=3, H=7, W=6) if d3 else dict(H=13, W=11)))
    dims = (s.To, s.Ho, s.Wo) if d3 else (s.Ho, s.Wo)
    pts = [tuple(int(g) for g in p) for p in np.ndindex(*dims)]
    for layout in (("ncdhw", "ndhwc") if d3 else ("nchw", "nhwc")):
        model = pruner.zero_copy_lines(s, esize, layout)
        worst = max(_brute_lines(layout, s, esize, img, p) for p in pts for img in (0, 1))
        assert worst <= model, (layout, worst, model)


def test_line_model_of_the_up_convolutions():
    """k = s = 2 reads one input pixel per point: c lines (one per channel) in NCHW, ceil(c*esize / 128) lines of the
    pixel's channels (+1 off the 128-byte grid) in NHWC."""
    import cpb200
    from cpb200 import pruner

    nets = cpb200.synth.conv_transpose_layers()
    for s in nets["unet2d"] + nets["nnunet3d"]:
        for es in (4, 2):
            assert pruner.zero_copy_lines(s, es, "nchw") == s.N * s.c
            assert pruner.zero_copy_lines(s, es, "nhwc") == s.N * -(-s.c * es // 128)


def test_conv_transpose_table():
    """The profile's shapes: transposed, k = s = 2 up-convolutions halving c (the 3-D decoder's first keeps 320) and one
    k = 4, s = 2, p = 1 layer; the synthetic fp32 maps of each network within 10 GB; every layer a well-posed least
    squares at N = 5000 (N - 1 >= K' and, points spread evenly, each k = s phase more rows than kept channels)."""
    import cpb200

    nets = cpb200.synth.conv_transpose_layers()
    assert [s.c for s in nets["unet2d"]] == [1024, 512, 256, 128]
    assert [s.c for s in nets["nnunet3d"]] == [320, 320, 256, 128, 64]
    for net, shapes in nets.items():
        nbytes = 0
        for s in shapes:
            assert s.transposed and s.N == 5000
            assert s.N - 1 >= s.rank * s.k2
            if s.stride == s.k:
                assert s.N / s.k2 > s.rank
            spatial = (s.D * s.H * s.W) if hasattr(s, "kt") else s.H * s.W
            nbytes += s.nbatch * s.B * s.c * spatial * 4
        assert nbytes <= 10e9, (net, nbytes)
    (dc,) = nets["dcgan"]
    assert (dc.k, dc.stride, dc.pad, dc.Ho) == (4, 2, 1, 2 * dc.H)
    assert all(s.Ho == 2 * s.H for s in nets["unet2d"]) and all(s.To == 2 * s.D for s in nets["nnunet3d"])


def test_make_problem_numpy_reproduces_conv_transpose():
    """The targets of a transposed problem are F.conv_transpose2d(relu(x), W2.transpose(0, 1)) + b2 at the points:
    W2 is (n, c, kh, kw), the orientation of every layer problem."""
    import cpb200

    s = _shape("k3s2p1op1", False, c=6, n=5, H=7, W=6, N=60, B=3, P=4)
    d = cpb200.synth.make_problem_numpy(s, 3, noise=0.0)
    assert d["W2"].shape == (s.n, s.c, s.kh, s.kw) and d["X"].shape == (s.N, s.c, s.kh, s.kw)
    x = torch.relu(torch.as_tensor(d["fmap"], dtype=torch.float64))
    y = F.conv_transpose2d(x, torch.as_tensor(d["W2"], dtype=torch.float64).transpose(0, 1),
                           torch.as_tensor(d["b2"], dtype=torch.float64), stride=s.stride, padding=s.pad,
                           output_padding=s.output_padding).numpy()
    want = np.stack([y[b * s.B + i, :, d["randx"][b, p], d["randy"][b, p]]
                     for b in range(s.nbatch) for p in range(s.P) for i in range(s.B)])
    np.testing.assert_allclose(d["feats"], want, rtol=1e-6, atol=1e-6)
    s3 = _shape("2x2x2", True, N=60, B=3, P=4)
    d3 = cpb200.synth.make_problem_numpy(s3, 4, noise=0.0)
    assert d3["X"].shape == (s3.N, s3.c) + s3.window
    Xo = CT.gather_tr3d(d3["fmap"], d3["randt"], d3["randx"], d3["randy"], s3.B, s3.k, s3.pad, s3.stride, relu=True)
    assert np.array_equal(d3["X"].reshape(s3.N, -1), Xo)


def test_pack_unpack_round_trip_of_transposed_weights():
    """W (n, c', *window) round-trips; W.transpose(0, 1) is the kept channels' ConvTranspose weight (c', n, *window)."""
    import cpb200
    from cpb200 import pruner as pr

    shapes = [_shape("rect", False, c=12, n=7, N=60, B=3, P=4, rank=9),
              _shape("2x2x2", True, c=10, n=5, N=60, B=3, P=4, rank=8)]
    r = np.random.RandomState(2)
    sizes = [pr.slot_size(s.c, s.n, s.k2, s.rank, 0.1) for s in shapes]
    buf = torch.zeros(sum(sizes), dtype=torch.float64)
    want, off = [], 0
    for s, sz in zip(shapes, sizes):
        idxs = np.zeros(s.c, dtype=bool)
        idxs[r.choice(s.c, s.rank, replace=False)] = True
        W = torch.as_tensor(r.standard_normal((s.n, s.rank * s.k2)))
        b = torch.as_tensor(r.standard_normal(s.n))
        pr.pack_result(buf, off, idxs, W, b, 0.5, 2, s.c, s.n, s.k2)
        want.append((idxs, W.numpy(), b.numpy()))
        off += sz
    out = pr.unpack_network(shapes, [0, 0], sizes, buf.view(1, -1))
    assert out[0]["W"].shape == (7, 9, 3, 4) and out[1]["W"].shape == (5, 8, 2, 2, 2)
    for (idxs, W, b), o, s in zip(want, out, shapes):
        assert np.array_equal(o["idxs"], idxs) and np.array_equal(o["b"], b)
        assert np.array_equal(o["W"].reshape(s.n, -1), W) and o["alpha"] == 0.5 and o["nprobe"] == 2
        assert np.array_equal(np.swapaxes(o["W"], 0, 1).reshape(-1), W.reshape((s.n, s.rank, s.k2)).transpose(1, 0, 2)
                              .reshape(-1))
