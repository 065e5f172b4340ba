"""GPU: patch gathers of transposed convolutions (nn.ConvTranspose2d / 3d; cp_patch_gather_conv_transpose / _3d).
Every path (channels first and last, HBM and pinned host, 2-D and 3-D) is checked bit for bit against the numpy
restatement, the kernel that ran against the one intended, the gathered X against F.conv_transpose2d / 3d, refusals of
bad geometry, and the solver and pipeline on transposed layers against the oracle -- the structured cases (all-zero
rows, a phase with fewer rows than kept channels, the dual path) included."""
import zlib

import numpy as np
import pytest

import conv3d_oracle as C3
import cp_oracle as O
import gather_checks as GC

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
F = pytest.importorskip("torch.nn.functional")

# (kernel_size, padding, stride, dilation, output_padding) as nn.ConvTranspose2d / 3d take them
GEOMS2D = {
    "k2s2": (2, 0, 2, 1, 0), "k4s2p1": (4, 1, 2, 1, 0), "k3s2p1op1": (3, 1, 2, 1, 1), "k3s2d2": (3, 0, 2, 2, 0),
    "k3s1p1": (3, 1, 1, 1, 0), "rect": ((3, 4), (1, 2), (2, 3), (2, 1), (1, 0)),
}
GEOMS3D = {
    "1x2x2": ((1, 2, 2), 0, (1, 2, 2), 1, 0), "2x2x2": (2, 0, 2, 1, 0), "3x3x3s2p1op1": (3, 1, 2, 1, 1),
    "rect3d": ((2, 3, 4), (0, 1, 2), (2, 1, 3), (1, 2, 1), (1, 0, 2)),
}
# path -> (channels last, in pinned host memory, channels): c = 24 takes 16-byte loads on channels-last maps, c = 5 not
PATHS = {"cf": (False, False, 12), "cf_host": (False, True, 12), "cl": (True, False, 24), "cl_c5": (True, False, 5),
         "cl_host": (True, True, 24), "cl_host_c5": (True, True, 5)}


def _tup(v, n):
    return tuple(v) if isinstance(v, tuple) else (v,) * n


def _out_size(dims, geom):
    k, pad, stride, dil, op = (_tup(v, len(dims)) for v in geom)
    return tuple((n - 1) * s - 2 * p + d * (kk - 1) + o + 1 for n, kk, p, s, d, o in zip(dims, k, pad, stride, dil, op))


def _points2d(nb, Ho, Wo, device):
    """Every output point of the (small) output map, in reversed order for the second batch."""
    xs, ys = np.meshgrid(np.arange(Ho), np.arange(Wo), indexing="ij")
    rx = torch.tensor([xs.reshape(-1)] * nb, dtype=torch.int32, device=device)
    ry = torch.tensor([ys.reshape(-1)] * nb, dtype=torch.int32, device=device)
    if nb > 1:
        rx[1], ry[1] = rx[1].flip(0), ry[1].flip(0)
    return rx, ry, rx.shape[1]


def _ref(ncdhw, pts, B, geom, relu, d3):
    """The numpy restatement (synth) on the map widened to fp32, ReLU'd as the kernels do (NaN and -0 give +0)."""
    import cpb200

    k, pad, stride, dil, _ = geom
    x = ncdhw.float().cpu().numpy()
    p = [t.cpu().numpy() for t in pts]
    if d3:
        X = cpb200.synth.gather_patches_tr3d_numpy(x, *p, B, k, pad, stride, relu=False, dilation=dil)
    else:
        X = cpb200.synth.gather_patches_tr_numpy(x, *p, B, k, pad, stride, relu=False, dilation=dil)
    X = torch.as_tensor(X.reshape(X.shape[0], -1))
    return torch.where(X > 0, X, torch.zeros_like(X)) if relu else X


def _gather(engine, path, ncdhw, pts, B, P, geom, relu, d3, out=None):
    clast, host, _ = PATHS[path]
    m = ncdhw.permute(0, *range(2, ncdhw.dim()), 1).contiguous() if clast else ncdhw
    if host:
        m = GC.pinned(m)
    k, pad, stride, dil, _ = geom
    if d3:
        return engine.patch_gather3d(m, *pts, B, P, k, pad, stride, relu=relu, layout="ndhwc" if clast else "ncdhw",
                                     dilation=dil, out=out, transposed=True)
    return engine.patch_gather(m, *pts, B, P, k, pad, stride, relu=relu, layout="nhwc" if clast else "nchw",
                               dilation=dil, out=out, transposed=True)


@pytest.mark.parametrize("dtype", list(GC.FMAP_DTYPES))
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("gname", ["2d:" + n for n in GEOMS2D] + ["3d:" + n for n in GEOMS3D])
def test_gather_tr_bits_equal_reference(engine, dtype, path, gname):
    d3 = gname.startswith("3d:")
    geom = (GEOMS3D if d3 else GEOMS2D)[gname[3:]]
    dev = engine.device
    c = PATHS[path][2]
    B, nb = 2, 2
    seed = zlib.crc32(("%s/%s/%s" % (gname, path, dtype)).encode()) % 10007
    if d3:
        D, H, W = 3, 5, 4
        To, Ho, Wo = _out_size((D, H, W), geom)
        x = GC.special_map((nb * B, c, D, H, W), dtype, seed, dev)
        rt, rx, ry, P = GC.points3d(nb, To, Ho, Wo, dev)
        pts = (rt, rx, ry)
    else:
        H, W = 6, 5
        Ho, Wo = _out_size((H, W), geom)
        x = GC.special_map((nb * B, c, H, W), dtype, seed, dev)
        rx, ry, P = _points2d(nb, Ho, Wo, dev)
        pts = (rx, ry)
    for relu in (False, True):
        got = _gather(engine, path, x, pts, B, P, geom, relu, d3)
        torch.cuda.synchronize()
        GC.assert_same_bits(got, _ref(x, pts, B, geom, relu, d3))


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("gname", ["2d:k2s2", "2d:k4s2p1", "3d:2x2x2"])
def test_gather_tr_at_decoder_size(engine, dtype, gname):
    """N = 5000 rows of a 160-channel map (the persistent grids' tails, several channel tiles), every path against the
    reference, and a row slice of a wider buffer (ldx > K) that leaves the rest alone."""
    d3 = gname.startswith("3d:")
    geom = (GEOMS3D if d3 else GEOMS2D)[gname[3:]]
    dev = engine.device
    c, B, nb, P = 160, 10, 10, 50
    dims = (6, 14, 14) if d3 else (28, 28)
    out = _out_size(dims, geom)
    g = torch.Generator(device=dev)
    g.manual_seed(11)
    x = torch.randn((nb * B, c) + dims, generator=g, device=dev).to(GC.FMAP_DTYPES[dtype])
    r = np.random.RandomState(3)
    pts = tuple(torch.as_tensor(r.randint(0, hi, (nb, P)).astype(np.int32), device=dev) for hi in out)
    want = _ref(x, pts, B, geom, True, d3)
    for path in ("cf", "cf_host", "cl", "cl_host"):
        got = _gather(engine, path, x, pts, B, P, geom, True, d3)
        torch.cuda.synchronize()
        GC.assert_same_bits(got, want)
        del got
    K = want.shape[1]
    for path in ("cf", "cl"):
        wide = torch.full((want.shape[0], K + 40), 7.0, device=dev)
        _gather(engine, path, x, pts, B, P, geom, True, d3, out=wide[:, 8:8 + K])
        torch.cuda.synchronize()
        GC.assert_same_bits(wide[:, 8:8 + K].contiguous(), want)
        assert bool((wide[:, :8] == 7.0).all()) and bool((wide[:, 8 + K:] == 7.0).all())


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("path", ["cl", "cl_host"])
def test_gather_tr_channel_tiles(engine, dtype, path):
    """Channels last with more channels than one 48 KB tile holds (c = 1400, 3 x 3 stride 1: every tap valid, 1363
    channels per tile): two channel tiles per row, against the reference."""
    dev = engine.device
    geom = GEOMS2D["k3s1p1"]
    B, nb = 2, 1
    x = GC.special_map((nb * B, 1400, 6, 5), dtype, 3, dev)
    rx, ry, P = _points2d(nb, *_out_size((6, 5), geom), dev)
    for relu in (False, True):
        got = _gather(engine, path, x, (rx, ry), B, P, geom, relu, False)
        torch.cuda.synchronize()
        GC.assert_same_bits(got, _ref(x, (rx, ry), B, geom, relu, False))


@pytest.mark.parametrize("gname", ["2d:" + n for n in GEOMS2D] + ["3d:" + n for n in GEOMS3D])
@pytest.mark.parametrize("clast", [False, True])
def test_gathered_x_reproduces_conv_transpose(engine, gname, clast):
    """relu(X) W2' + b2 at the sampled points is F.conv_transpose2d / 3d(relu(x), W2.transpose(0, 1), b2) there."""
    d3 = gname.startswith("3d:")
    k, pad, stride, dil, op = geom = (GEOMS3D if d3 else GEOMS2D)[gname[3:]]
    dev = engine.device
    g = torch.Generator(device=dev)
    g.manual_seed(5)
    c, n, B, nb = 16, 8, 3, 2
    dims = (3, 5, 4) if d3 else (6, 5)
    x = torch.randn((nb * B, c) + dims, generator=g, device=dev)
    W2 = torch.randn((n, c) + _tup(k, len(dims)), generator=g, device=dev)
    b2 = torch.randn((n,), generator=g, device=dev)
    out = _out_size(dims, geom)
    if d3:
        rt, rx, ry, P = GC.points3d(nb, *out, dev)
        pts = (rt, rx, ry)
    else:
        rx, ry, P = _points2d(nb, *out, dev)
        pts = (rx, ry)
    X = _gather(engine, "cl" if clast else "cf", x, pts, B, P, geom, True, d3)
    got = X.double() @ W2.reshape(n, -1).T.double() + b2.double()
    fn = F.conv_transpose3d if d3 else F.conv_transpose2d
    y = fn(torch.relu(x).double(), W2.transpose(0, 1).double(), b2.double(), stride=stride, padding=pad,
           output_padding=op, dilation=dil)
    assert tuple(y.shape[2:]) == out
    idx = [[int(t[b, p]) for t in pts] for b in range(nb) for p in range(P)]
    want = torch.stack([y[(j // P) * B + i, :, *idx[j]] for j in range(nb * P) for i in range(B)])
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5)


def _raw(engine, m, c, dims, layout, geom, ldx=None, dtype=None, null_points=False):
    """cp_patch_gather_conv_transpose(3d) with geom = per-axis (k..., pad..., stride..., dil...); (rc, message)."""
    ffi, lib = engine.ffi, engine.lib
    r = torch.zeros((1, 1), dtype=torch.int32, device=engine.device)
    na = len(dims)
    taps = max(int(np.prod(geom[:na])), 1)
    X = torch.empty((2, c * taps + 16), device=engine.device)
    ip = ffi.NULL if null_points else ffi.cast("const int32_t*", r.data_ptr())
    fn = lib.cp_patch_gather_conv_transpose3d if na == 3 else lib.cp_patch_gather_conv_transpose
    rc = fn(engine.h, ffi.cast("const void*", m.data_ptr()), lib.CP_F32 if dtype is None else dtype, 1, 2, c, *dims,
            layout, *([ip] * na), 1, *geom, 0, ffi.cast("float*", X.data_ptr()),
            X.shape[1] if ldx is None else ldx, ffi.NULL)
    return rc, ffi.string(lib.cp_last_error()).decode()


_G2 = (2, 2, 0, 0, 2, 2, 1, 1)
_G3 = (2, 2, 2, 0, 0, 0, 2, 2, 2, 1, 1, 1)


def _with(base, i, v):
    g = list(base)
    g[i] = v
    return tuple(g)


@pytest.mark.parametrize("d3", [False, True])
@pytest.mark.parametrize("case,msg", [
    ("k0", "kernel_size"), ("pad-1", "padding"), ("s0", "stride"), ("d0", "dilation"), ("taps", "taps"),
    ("ldx", "ldx"), ("layout", "unknown layout"), ("dtype", "dtype"), ("null", "NULL")])
def test_bad_geometry_is_refused(engine, d3, case, msg):
    """CP_ERR_INVALID with the entry's message before any device work, in both layouts; the Python call raises."""
    import cpb200

    base, na = (_G3, 3) if d3 else (_G2, 2)
    dims = (3, 7, 7) if d3 else (7, 7)
    geom, kw, layouts = base, {}, (0, 1)
    if case == "k0":
        geom = _with(base, na - 1, 0)
    elif case == "pad-1":
        geom = _with(base, na, -1)
    elif case == "s0":
        geom = _with(base, 2 * na, 0)
    elif case == "d0":
        geom = _with(base, 3 * na, 0)
    elif case == "taps":
        geom = ((17, 16, 16) if d3 else (65, 64)) + base[na:]
    elif case == "ldx":
        kw["ldx"] = 16 * int(np.prod(base[:na])) - 1
    elif case == "layout":
        layouts = (2,)
    elif case == "dtype":
        kw["dtype"] = 1  # CP_F64
    else:
        kw["null_points"] = True
    f = torch.zeros((2, 16) + dims, device=engine.device)
    name = "cp_patch_gather_conv_transpose3d" if d3 else "cp_patch_gather_conv_transpose"
    for layout in layouts:
        rc, err = _raw(engine, f, 16, dims, layout, geom, **kw)
        assert rc == engine.lib.CP_ERR_INVALID and msg in err and name + ":" in err, err
    if case in ("k0", "pad-1", "s0", "d0", "taps"):
        r = torch.zeros((1, 1), dtype=torch.int32, device=engine.device)
        k, pad, st, dil = (geom[i * na:(i + 1) * na] for i in range(4))
        with pytest.raises(cpb200._cabi.CpError):
            if d3:
                engine.patch_gather3d(f, r, r, r, 2, 1, k, pad, st, dilation=dil, transposed=True)
            else:
                engine.patch_gather(f, r, r, 2, 1, k, pad, st, dilation=dil, transposed=True)


def test_window_wider_than_the_map_is_gathered(engine):
    """No empty-output rule: a 9 x 9 window on a 2 x 2 map (every tap range-checked) gathers like the reference."""
    dev = engine.device
    x = torch.randn(2, 3, 2, 2, device=dev)
    geom = (9, 0, 1, 1, 0)
    rx, ry, P = _points2d(1, *_out_size((2, 2), geom), dev)
    for path in ("cf", "cl"):
        got = _gather(engine, path, x, (rx, ry), 2, P, geom, False, False)
        torch.cuda.synchronize()
        GC.assert_same_bits(got, _ref(x, (rx, ry), 2, geom, False, False))


# kind -> (channels last, d3, channels, geometries); each runs from HBM and from pinned host memory
_KERNEL_CASES = {"nchw": (False, False, 32, ["k2s2", "k4s2p1"]), "ncdhw": (False, True, 32, ["2x2x2"]),
                 "nhwc": (True, False, 32, ["k2s2", "k3s2d2"]), "ndhwc": (True, True, 32, ["2x2x2", "1x2x2"])}
_REPEAT = 3


def _profile_kernel_cases():
    """Every case of _KERNEL_CASES, from HBM and pinned host, _REPEAT times in one profiler session; the names of the
    gather launches in order."""
    import cpb200
    from torch.profiler import ProfilerActivity, profile

    engine = cpb200.get_engine()
    dev = engine.device
    B, nb = 2, 2
    runs = []
    for kind, (clast, d3, c, names) in _KERNEL_CASES.items():
        for gname in names:
            geom = (GEOMS3D if d3 else GEOMS2D)[gname]
            dims = (3, 6, 6) if d3 else (8, 8)
            out = _out_size(dims, geom)
            if d3:
                rt, rx, ry, P = GC.points3d(nb, *out, dev)
                pts = (rt, rx, ry)
            else:
                rx, ry, P = _points2d(nb, *out, dev)
                pts = (rx, ry)
            x = torch.randn((nb * B, c) + dims, device=dev)
            for host in (False, True):
                m = x.permute(0, *range(2, x.dim()), 1).contiguous() if clast else x
                m = GC.pinned(m) if host else m
                lay = ("ndhwc" if d3 else "nhwc") if clast else ("ncdhw" if d3 else "nchw")
                k, pad, stride, dil, _ = geom
                fn = engine.patch_gather3d if d3 else engine.patch_gather
                call = (lambda fn=fn, m=m, pts=pts, P=P, k=k, pad=pad, stride=stride, dil=dil, lay=lay:
                        fn(m, *pts, B, P, k, pad, stride, layout=lay, dilation=dil, transposed=True))
                call()
                runs.append(call)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for call in runs:
            for _ in range(_REPEAT):
                call()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "patch_gather" in e.name and e.device_type.name == "CUDA"]


def test_intended_kernels_run(engine):
    """One profiler session (in a child process, so the suite's other profiler checks keep their record counts): each
    layout and rank launches its own kernel, from HBM and from pinned host memory alike."""

    def kind_of(n):
        for kind in ("ncdhw", "nchw", "ndhwc", "nhwc"):
            if "patch_gather_tr_%s<" % kind in n:
                return kind
        return n

    want = {kind: 2 * _REPEAT * len(v[3]) for kind, v in _KERNEL_CASES.items()}  # HBM and pinned host
    GC.assert_launch_counts(GC.launched_gather_kernels("test_gpu_conv_transpose"), kind_of, want)


# ----------------------------------------------------------------------------- solver and pipeline
def _layer(name, c, n, H, d3=False, N=1000, B=10, P=10, rank=None, **geo):
    import cpb200

    if d3:
        return cpb200.synth.LayerShape3d(name, c, n, geo.pop("D"), H, N=N, B=B, P=P, rank=rank, transposed=True,
                                         **geo)
    return cpb200.synth.LayerShape(name, c, n, H, N=N, B=B, P=P, rank=rank, transposed=True, **geo)


@pytest.mark.parametrize("mode,tol", [(0, 1e-7), (1, 1e-4)], ids=["fp64", "3xtf32"])
@pytest.mark.parametrize("geo", ["k4s2p1", "2x2x2"])
def test_dictionary_on_transposed_layers_matches_oracle(engine, mode, tol, geo):
    """decompose.dictionary on a transposed problem's X against conv3d_oracle.dictionary: the same mask, alpha, probes
    and numpy RNG draws, weights within tol."""
    import cpb200
    from cpb200.lib import cfgs, decompose

    engine.gram_mode = mode
    if geo == "2x2x2":
        s = _layer("L", 32, 24, 6, d3=True, D=4, k=2, stride=2, pad=0)
    else:
        s = _layer("L", 32, 24, 8, k=4, stride=2, pad=1)
    d = cpb200.synth.make_problem_numpy(s, 9)
    X, W2, Y = d["X"].astype(np.float64), d["W2"], d["feats"].astype(np.float64)
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
    assert W.shape == oW.shape
    assert GC.rel(W, oW) <= tol and np.abs(B - oB).max() <= tol * max(1.0, np.abs(oB).max())


def _oracle_layer(s, d):
    """The oracle on one pipeline problem of a transposed layer: synth's numpy transposed gather (fp64, ReLU'd), then
    conv3d_oracle.dictionary with the problem's samples and seeds."""
    import cpb200

    d3 = hasattr(s, "kt")
    fm = d["fmap"]
    if d["layout"] in ("nhwc", "ndhwc"):
        fm = fm.permute(0, fm.dim() - 1, *range(1, fm.dim() - 1))
    fm = fm.float().cpu().numpy().astype(np.float64)
    if d3:
        pts = [d[k].cpu().numpy() for k in ("randt", "randx", "randy")]
        X = cpb200.synth.gather_patches_tr3d_numpy(fm, *pts, s.B, s.k, s.pad, s.stride, True, dilation=s.dilation)
    else:
        pts = [d[k].cpu().numpy() for k in ("randx", "randy")]
        X = cpb200.synth.gather_patches_tr_numpy(fm, *pts, s.B, s.k, s.pad, s.stride, True, dilation=s.dilation)
    return GC.oracle_on_problem(C3.dictionary, X, s, d)


def _decoder_layers(N=800, B=4, P=10):
    """Transposed layers at test size (2-D and 3-D up-convolutions, an overlapping k = 4 window) among a Conv2d and
    a Conv3d layer.  N = 800 leaves every k = s phase of the 2x2x2 layer more rows than kept channels."""
    import cpb200

    return [_layer("up2d", 32, 16, 7, k=2, stride=2, pad=0, N=N, B=B, P=P),
            _layer("dcgan", 24, 16, 6, k=4, stride=2, pad=1, N=N, B=B, P=P),
            _layer("up3d", 32, 16, 4, d3=True, D=3, k=2, stride=2, pad=0, N=N, B=B, P=P),
            cpb200.synth.LayerShape("conv2d", 32, 24, 14, N=N, B=B, P=P),
            cpb200.synth.LayerShape3d("conv3d", 24, 16, 4, 8, N=N, B=B, P=P)]


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("host_layout", ["nchw", "nhwc"])
def test_pipeline_on_transposed_layers(engine, dtype, host_layout):
    """prune_layers on transposed layers mixed with conv layers: maps in HBM, read in place from pinned host memory
    ('zc'), staged by DMA ('copy') or as the plan decides -- identical masks, alpha, W and b; verdict 'ok'; the
    transposed layers against the oracle (fp64 statistics: W and b within 1e-7)."""
    import cpb200
    from cpb200 import pruner

    eng = cpb200.Engine(nstreams=4)
    eng.gram_mode = 0
    shapes = _decoder_layers()
    datas = [cpb200.synth.make_problem_device(s, 90 + i, eng, pinned_host=True, host_layout=host_layout,
                                              dtype=GC.FMAP_DTYPES[dtype]) for i, s in enumerate(shapes)]
    ref = pruner.prune_layers(eng, shapes, datas)
    torch.cuda.synchronize()
    assert [r.info["verdict"] for r in ref] == ["ok"] * len(shapes)
    ref = [(r.idxs.copy(), r.alpha, r.nprobe, r.W.cpu(), r.b.cpu()) for r in ref]
    for policy in ("zc", "copy", True):
        got = pruner.prune_layers(eng, shapes, datas, from_host=policy, to_host=True)
        torch.cuda.synchronize()
        for s, (idxs, alpha, nprobe, W, b), r in zip(shapes, ref, got):
            assert np.array_equal(idxs, r.idxs) and alpha == r.alpha and nprobe == r.nprobe, (policy, s.name)
            assert torch.equal(W, r.W) and torch.equal(b, r.b), (policy, s.name)
            assert r.info["verdict"] == "ok", (policy, s.name, r.info)
    if host_layout == "nchw":
        for i in (0, 1, 2):
            s, d = shapes[i], datas[i]
            oi, oW, oB, oalpha, onprobe = _oracle_layer(s, d)
            idxs, alpha, nprobe, W, b = ref[i]
            assert np.array_equal(idxs, oi) and alpha == oalpha and nprobe == onprobe, s.name
            assert GC.rel(W.numpy().reshape(oW.shape), oW) <= 1e-7 and np.abs(b.numpy() - oB).max() <= 1e-7, s.name
    eng.close()


def test_prune_network_sharded_on_transposed_layers(engine):
    """One rank: unpack_network gives (n, c', *window) weights with the values prune_layers returns."""
    import cpb200
    from cpb200 import pruner

    eng = cpb200.Engine(nstreams=4)
    eng.gram_mode = 0
    shapes = _decoder_layers()
    datas = [cpb200.synth.make_problem_device(s, 30 + i, eng) for i, s in enumerate(shapes)]
    owner, sizes, allbuf = pruner.prune_network_sharded(eng, shapes, lambda i: datas[i], 0, 1)
    out = pruner.unpack_network(shapes, owner, sizes, allbuf)
    ref = pruner.prune_layers(eng, shapes, datas)
    torch.cuda.synchronize()
    for s, o, r in zip(shapes, out, ref):
        assert o["W"].shape == (s.n, int(r.idxs.sum())) + pruner.window_of(s)
        assert np.array_equal(o["idxs"], r.idxs) and o["alpha"] == r.alpha
        assert np.array_equal(o["W"].reshape(s.n, -1), r.W.cpu().numpy()) and np.array_equal(o["b"], r.b.cpu().numpy())
    eng.close()


def _with_points(s, d, eng, pts, noise=0.01, seed=0):
    """Replaces a device problem's sampled points and recomputes its targets from them (the library's gather, fp64)."""
    keys = ("randt", "randx", "randy") if hasattr(s, "kt") else ("randx", "randy")
    for key, p in zip(keys, pts):
        d[key] = torch.as_tensor(np.asarray(p, dtype=np.int32), device=eng.device).contiguous()
    from cpb200 import pruner

    X = pruner._patch_gather(eng, s, d, d["fmap"], d["layout"])
    Y = X.double() @ d["W2"].reshape(s.n, -1).T.double() + d["b2"].double()
    g = torch.Generator(device=eng.device)
    g.manual_seed(seed)
    Y = Y + noise * Y.std() * torch.randn(Y.shape, generator=g, device=eng.device, dtype=torch.float64)
    d["feats"] = Y.float()
    return d


def _run_one(s, d, mode):
    import cpb200
    from cpb200 import pruner

    eng = cpb200.Engine(nstreams=2)
    eng.gram_mode = mode
    r = pruner.prune_layers(eng, [s], [d])[0]
    torch.cuda.synchronize()
    eng.close()
    return r


def _check_against_oracle(s, d, r, tol):
    oi, oW, oB, oalpha, onprobe = _oracle_layer(s, d)
    assert np.array_equal(r.idxs, oi) and r.alpha == oalpha and r.nprobe == onprobe
    assert GC.rel(r.W.cpu().numpy().reshape(oW.shape), oW) <= tol
    assert np.abs(r.b.cpu().numpy() - oB).max() <= tol * max(1.0, np.abs(oB).max())


def test_strided_dilated_layer_with_zero_rows_matches_oracle(engine):
    """k = 3, s = d = 2: points with an odd coordinate read nothing (three quarters of the rows all zero)."""
    import cpb200

    s = _layer("s2d2", 16, 12, 9, k=3, stride=2, dilation=2, pad=0, N=1000, B=5, P=20)
    eng = cpb200.get_engine()
    d = cpb200.synth.make_problem_device(s, 13, eng)
    r = np.random.RandomState(4)
    pts = [r.randint(0, hi, (s.nbatch, s.P)) for hi in (s.Ho, s.Wo)]
    d = _with_points(s, d, eng, pts)
    X = cpb200.synth.gather_patches_tr_numpy(d["fmap"].cpu().numpy(), *pts, s.B, s.k, s.pad, s.stride, True,
                                             dilation=s.dilation).reshape(s.N, -1)
    odd = ((pts[0] % 2) | (pts[1] % 2)).astype(bool)
    assert not X[np.repeat(odd.reshape(-1), s.B)].any() and 0.6 < odd.mean() < 0.9
    res = _run_one(s, d, 0)
    assert res.info["verdict"] == "ok"
    _check_against_oracle(s, d, res, 1e-7)


@pytest.mark.parametrize("mode", [0, 1], ids=["fp64", "3xtf32"])
def test_phase_with_fewer_rows_than_kept_channels_matches_gelsd(engine, mode):
    """2-D k = s = 2: the points are placed so that N - 1 >= K' but phase (0, 0) gets 10 rows for about 14 kept
    channels.  Its taps' columns are then exactly dependent: the Cholesky flags the system and the layer takes the
    truncated solve, whose W and b match the oracle's gelsd minimum-norm answer."""
    import cpb200

    s = _layer("starved", 16, 12, 8, k=2, stride=2, pad=0, N=200, B=2, P=10)
    eng = cpb200.get_engine()
    d = cpb200.synth.make_problem_device(s, 17, eng)
    r = np.random.RandomState(8)
    phase = r.permutation(np.r_[np.zeros(5, int), np.ones(95, int) + r.randint(0, 3, 95)]).reshape(s.nbatch, s.P)
    ph, pw = np.array([0, 0, 1, 1])[phase], np.array([0, 1, 0, 1])[phase]
    pts = [2 * r.randint(0, s.Ho // 2, phase.shape) + ph, 2 * r.randint(0, s.Wo // 2, phase.shape) + pw]
    d = _with_points(s, d, eng, pts)
    res = _run_one(s, d, mode)
    kept = int(res.idxs.sum())
    assert s.N - 1 >= kept * s.k2 and 5 * s.B < kept
    print("phase-starved k = s = 2 layer: verdict %s, %s" % (res.info["verdict"], res.info))
    assert res.info["verdict"] == "truncated"
    _check_against_oracle(s, d, res, 1e-6)


def test_3d_up_convolution_on_the_dual_path_matches_oracle(engine):
    """3-D k = s = 2 with N - 1 < K': the dual (minimum-norm) solve, against the oracle.  Rows of different phases
    are orthogonal, so the dual system is regular only while no phase has more rows than kept channels and no row
    repeats: the points are distinct within each batch and take the eight phases in turn (48 or 52 rows each, for at
    least 55 kept channels)."""
    import cpb200
    from cpb200.engine import ls_dual

    s = _layer("dual3d", 64, 16, 4, d3=True, D=3, k=2, stride=2, pad=0, N=400, B=4, P=10)
    eng = cpb200.get_engine()
    d = cpb200.synth.make_problem_device(s, 21, eng)
    r = np.random.RandomState(5)
    pts = np.zeros((3, s.nbatch, s.P), dtype=np.int32)
    for b in range(s.nbatch):
        used = set()
        for j in range(s.P):
            ph = (b * s.P + j) % 8
            while True:
                p = tuple(2 * int(r.randint(0, n // 2)) + (ph >> (2 - a) & 1) for a, n in enumerate((s.To, s.Ho, s.Wo)))
                if p not in used:
                    break
            used.add(p)
            pts[:, b, j] = p
    d = _with_points(s, d, eng, list(pts))
    res = _run_one(s, d, 0)
    assert res.info["dual"] and ls_dual(s.N, res.idxs, s.k2)
    assert res.info["verdict"] == "ok"
    _check_against_oracle(s, d, res, 1e-7)
