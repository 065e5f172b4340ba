"""GPU: patch gathers through a consumer's input transform (cp_patch_gather_act): Conv-BN-activation networks pruned
from their raw conv outputs.  Every path (channels first and last, TMA, SIMT, pinned host, 2-D, 3-D and transposed)
against the numpy statement bit for bit on maps with -0, +-inf, NaN and subnormals seeded in, every exact act with
and without the folded BatchNorm; SiLU across paths and against float64; the affine-free route against the relu
gathers; which kernel runs; the gathered X against PyTorch's Conv-BN-act-Conv; and the pipeline against the oracle."""
import numpy as np
import pytest

import conv3d_oracle as C3
import gather_checks as GC

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
F = pytest.importorskip("torch.nn.functional")

EXACT_ACTS = [("identity", None), ("relu", None), ("relu6", None), ("leaky_relu", 0.1), ("hardswish", None)]
SILU_ULP = 4  # cpb200.h: SiLU within 4 ulp of the float64 value rounded to fp32

# family -> (geometries (k, pad, stride, dilation)); transposed families take their own points
GEOMS = {
    "conv2d": [(3, 1, 1, 1), ((3, 5), (2, 1), (1, 2), (2, 1)), (7, 3, 2, 1)],
    "conv3d": [(3, 1, 1, 1), ((1, 3, 3), (0, 1, 1), 1, 1)],
    "tr2d": [(4, 1, 2, 1), (3, 1, 1, 1)],
    "tr3d": [(2, 0, 2, 1), (3, 1, 2, 1)],
}
# family -> {path: (channels last, pinned host, channels)}; c = 64 takes the TMA kernel on channels-last HBM maps,
# c = 12 the SIMT kernel
PATHS = {
    "conv2d": {"nchw": (False, False, 12), "nchw_host": (False, True, 12), "nhwc_tma": (True, False, 64),
               "nhwc_simt": (True, False, 12), "nhwc_host": (True, True, 24)},
    "conv3d": {"ncdhw": (False, False, 12), "ncdhw_host": (False, True, 12), "ndhwc_tma": (True, False, 64),
               "ndhwc_simt": (True, False, 12), "ndhwc_host": (True, True, 24)},
    "tr2d": {"tr_nchw": (False, False, 12), "tr_nchw_host": (False, True, 12), "tr_nhwc": (True, False, 24),
             "tr_nhwc_c5": (True, False, 5), "tr_nhwc_host": (True, True, 24)},
    "tr3d": {"tr_ncdhw": (False, False, 12), "tr_ncdhw_host": (False, True, 12), "tr_ndhwc": (True, False, 24),
             "tr_ndhwc_host": (True, True, 24)},
}
DIMS = {"conv2d": (7, 6), "conv3d": (3, 5, 4), "tr2d": (4, 5), "tr3d": (2, 3, 3)}


def _tup(v, n):
    return tuple(v) if isinstance(v, tuple) else (v,) * n


def _out_size(fam, dims, geom):
    k, pad, stride, dil = (_tup(v, len(dims)) for v in geom)
    if fam.startswith("tr"):
        return tuple((n - 1) * s - 2 * p + d * (kk - 1) + 1 for n, kk, p, s, d in zip(dims, k, pad, stride, dil))
    return tuple((n + 2 * p - d * (kk - 1) - 1) // s + 1 for n, kk, p, s, d in zip(dims, k, pad, stride, dil))


def _points(fam, out, nb, dev):
    """Every output point of a 2-D map (reversed in the second batch), the corners and borders of a 3-D one."""
    if len(out) == 3:
        rt, rx, ry, P = GC.points3d(nb, *out, dev)
        return (rt, rx, ry), P
    xs, ys = np.meshgrid(np.arange(out[0]), np.arange(out[1]), indexing="ij")
    rx = torch.tensor([xs.reshape(-1)] * nb, dtype=torch.int32, device=dev)
    ry = torch.tensor([ys.reshape(-1)] * nb, dtype=torch.int32, device=dev)
    rx[1], ry[1] = rx[1].flip(0), ry[1].flip(0)
    return (rx, ry), rx.shape[1]


def _affine(c, kind, dev, seed=3):
    """(scale, shift) on device: 'bn' both (synth.bn_params: shift far from zero), 'scale' / 'shift' one of them."""
    import cpb200

    sc, sh = (torch.as_tensor(v, device=dev) for v in cpb200.synth.bn_params(c, seed))
    return {"none": (None, None), "bn": (sc, sh), "scale": (sc, None), "shift": (None, sh)}[kind]


def _layout(fam, clast):
    d3 = fam.endswith("3d")
    return ("ndhwc" if d3 else "nhwc") if clast else ("ncdhw" if d3 else "nchw")


def _gather(engine, fam, path, x, pts, B, P, geom, act, act_param, scale, shift):
    clast, host, _ = PATHS[fam][path]
    m = x.permute(0, *range(2, x.dim()), 1).contiguous() if clast else x
    if host:
        m = GC.pinned(m)
    k, pad, stride, dil = geom
    fn = engine.patch_gather3d if fam.endswith("3d") else engine.patch_gather
    return fn(m, *pts, B, P, k, pad, stride, layout=_layout(fam, clast), dilation=dil, transposed=fam.startswith("tr"),
              act=act, act_param=act_param, in_scale=scale, in_shift=shift)


def _ref(fam, x, pts, B, geom, act, act_param, scale, shift):
    """synth's numpy gather through input_transform_numpy, on the map widened to fp32."""
    import cpb200

    sy = cpb200.synth
    gather = {"conv2d": sy.gather_patches_numpy, "conv3d": sy.gather_patches3d_numpy,
              "tr2d": sy.gather_patches_tr_numpy, "tr3d": sy.gather_patches_tr3d_numpy}[fam]
    k, pad, stride, dil = geom
    X = gather(x.float().cpu().numpy(), *[p.cpu().numpy() for p in pts], B, k, pad, stride, relu=None, dilation=dil,
               act=act, act_param=act_param, in_scale=None if scale is None else scale.cpu().numpy(),
               in_shift=None if shift is None else shift.cpu().numpy())
    return torch.as_tensor(X.reshape(X.shape[0], -1))


def _cases(fam, dtype, seed, dev, nb=2, B=2):
    """(path, map, points, P, geometry) of every path and geometry of a family."""
    for gi, geom in enumerate(GEOMS[fam]):
        dims = DIMS[fam]
        pts, P = _points(fam, _out_size(fam, dims, geom), nb, dev)
        for path, (_, _, c) in PATHS[fam].items():
            if path.endswith("_tma") and gi == 2 and dtype != "fp32":
                continue  # one 7 x 7 TMA case (k2 > 32) per family is enough
            x = GC.special_map((nb * B, c) + dims, dtype, seed + gi, dev)
            yield path, x, pts, P, geom


@pytest.mark.parametrize("affine", ["none", "bn"])
@pytest.mark.parametrize("act,act_param", EXACT_ACTS, ids=[a for a, _ in EXACT_ACTS])
@pytest.mark.parametrize("dtype", list(GC.FMAP_DTYPES))
@pytest.mark.parametrize("fam", list(GEOMS))
def test_every_path_matches_numpy_bit_for_bit(engine, fam, dtype, act, act_param, affine):
    """Bit identity with the numpy statement on every path, border and corner; with 'bn' the shift is far from zero,
    so a padded or invalid tap given the transform would show."""
    dev = engine.device
    B = 2
    for path, x, pts, P, geom in _cases(fam, dtype, 40, dev, B=B):
        scale, shift = _affine(x.shape[1], affine, dev)
        got = _gather(engine, fam, path, x, pts, B, P, geom, act, act_param, scale, shift)
        torch.cuda.synchronize()
        GC.assert_same_bits(got, _ref(fam, x, pts, B, geom, act, act_param, scale, shift))


@pytest.mark.parametrize("affine", ["scale", "shift"])
@pytest.mark.parametrize("fam", list(GEOMS))
def test_half_affine(engine, fam, affine):
    """Scale without shift and shift without scale (the other pointer NULL)."""
    dev = engine.device
    for path, x, pts, P, geom in _cases(fam, "bf16", 41, dev):
        scale, shift = _affine(x.shape[1], affine, dev)
        got = _gather(engine, fam, path, x, pts, 2, P, geom, "leaky_relu", 0.2, scale, shift)
        torch.cuda.synchronize()
        GC.assert_same_bits(got, _ref(fam, x, pts, 2, geom, "leaky_relu", 0.2, scale, shift))


def _ulp_distance(a, b):
    """|a - b| in units in the last place of fp32 (the ordered integer images), for finite a and b."""
    def ordered(v):
        i = v.view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(ordered(np.asarray(a, np.float32)) - ordered(np.asarray(b, np.float32)))


def _check_silu(got, want64):
    """got (fp32) against the float64 value: NaN where it is NaN, the same infinities, within SILU_ULP elsewhere.
    Returns the largest distance."""
    got = got.cpu().numpy().reshape(-1)
    want = want64.reshape(-1)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan)
    fin = np.isfinite(want.astype(np.float32)) & ~nan
    assert np.array_equal(got[~fin & ~nan], want[~fin & ~nan].astype(np.float32))
    d = _ulp_distance(got[fin], want[fin].astype(np.float32))
    assert d.max() <= SILU_ULP, d.max()
    return int(d.max())


@pytest.mark.parametrize("affine", ["none", "bn"])
@pytest.mark.parametrize("dtype", list(GC.FMAP_DTYPES))
@pytest.mark.parametrize("fam", list(GEOMS))
def test_silu_paths_agree_and_stay_within_the_bound(engine, fam, dtype, affine):
    """SiLU: every path gives the bits of the first; each within SILU_ULP of the float64 value of the transform's
    input, and +0 at the padded or invalid taps."""
    dev = engine.device
    B = 2
    first = {}
    for path, x, pts, P, geom in _cases(fam, dtype, 42, dev, B=B):
        scale, shift = _affine(x.shape[1], affine, dev)
        got = _gather(engine, fam, path, x, pts, B, P, geom, "silu", None, scale, shift)
        torch.cuda.synchronize()
        # the affine's fp32 result, then silu in float64 (numpy statement of the identity transform)
        pre = _ref(fam, x, pts, B, geom, "identity", None, scale, shift).numpy().astype(np.float64)
        inmap = _ref(fam, torch.ones_like(x[:, :1], dtype=torch.float32), pts, B, geom, "identity", None, None, None)
        inmap = np.broadcast_to(inmap.numpy().reshape(inmap.shape[0], 1, -1) != 0,
                                (pre.shape[0], x.shape[1], inmap.shape[1])).reshape(pre.shape)
        with np.errstate(all="ignore"):
            want = np.where(inmap, pre / (1.0 + np.exp(-pre)), 0.0)
        _check_silu(got, want)
        assert not np.signbit(got.cpu().numpy()[~inmap]).any()
        key = (geom, x.shape[1])
        if key in first:
            GC.assert_same_bits(got, first[key])
        else:
            first[key] = got


def test_silu_dense_sweep(engine):
    """SiLU over a dense sweep of fp32 values -- around 0, the subnormals, the tail below -64 where expf(-v) heads for
    overflow, and large magnitudes -- on a channels-first map and on the TMA path: within SILU_ULP, the same bits."""
    dev = engine.device
    r = np.random.RandomState(0)
    v = np.concatenate([np.linspace(-110, 110, 40001), np.linspace(-1, 1, 20001), np.linspace(-90, -60, 20001),
                        r.standard_normal(20000) * 10, np.array([1e-45, -1e-45, 1e-38, -1e-38, 3e38, -3e38, -88.73,
                                                                 -103.9, -104.0, -150.0])]).astype(np.float32)
    c = 64
    v = np.concatenate([v, np.zeros((-len(v)) % c, np.float32)])
    x = torch.as_tensor(v.reshape(-1, c, 1, 1), device=dev)  # one 1 x 1 image per row of c values
    n = x.shape[0]
    rx = torch.zeros((1, 1), dtype=torch.int32, device=dev)
    got_cf = engine.patch_gather(x, rx, rx, n, 1, 1, 0, 1, act="silu")
    got_tma = engine.patch_gather(x.permute(0, 2, 3, 1).contiguous(), rx, rx, n, 1, 1, 0, 1, layout="nhwc",
                                  act="silu")
    torch.cuda.synchronize()
    GC.assert_same_bits(got_cf, got_tma)
    d = v.astype(np.float64)
    with np.errstate(all="ignore"):
        worst = _check_silu(got_cf, d / (1.0 + np.exp(-d)))
    print("silu: largest distance to the rounded float64 value %d ulp" % worst)


@pytest.mark.parametrize("act", ["relu", "identity"])
@pytest.mark.parametrize("fam", list(GEOMS))
def test_affine_free_route_gives_the_relu_gathers_bits(engine, fam, act):
    """cp_patch_gather_act with CP_ACT_RELU (CP_ACT_IDENTITY) and no affine: the bits of relu = 1 (0) of the entry
    the window selects, on every path."""
    from cpb200.engine import ACTS, _gather_map

    dev = engine.device
    B = 2
    d3, tr = fam.endswith("3d"), fam.startswith("tr")
    for path, x, pts, P, geom in _cases(fam, "fp32", 43, dev, B=B):
        clast, host, _ = PATHS[fam][path]
        m = x.permute(0, *range(2, x.dim()), 1).contiguous() if clast else x
        if host:
            m = GC.pinned(m)
        lay = _layout(fam, clast)
        k, pad, stride, dil = geom
        fn = engine.patch_gather3d if d3 else engine.patch_gather
        old = fn(m, *pts, B, P, k, pad, stride, relu=act == "relu", layout=lay, dilation=dil, transposed=tr)
        kk, pp, ss, dd = ((_tup(v, 3) if d3 else (1,) + _tup(v, 2)) for v in geom)
        pp = pp if d3 else (0,) + pp[1:]
        window = kk + pp + ss + dd  # kt, kh, kw, pad_t, ..., dil_w
        geo = _gather_map(m, B, lay, d3)
        new = engine._patch_gather_act(geo, m, tuple(pts) if d3 else (None,) + tuple(pts), B, P,
                                       int(np.prod(kk)), window, tr, (ACTS[act], 0.0, None, None), None)
        torch.cuda.synchronize()
        GC.assert_same_bits(new, old)


def test_refusals(engine):
    """Unknown act, non-finite slope, a scale off the device, a 2-D call with a depth: CP_ERR_INVALID, no launch."""
    dev = engine.device
    x = torch.randn(2, 16, 6, 6, device=dev)
    rx = torch.zeros((1, 1), dtype=torch.int32, device=dev)
    lib, ffi = engine.lib, engine.ffi
    out = torch.empty(2, 16 * 9, device=dev)
    sc = torch.ones(16, device=dev)
    sc_host = GC.pinned(torch.ones(16))
    p = lambda t, ty: ffi.cast(ty, t.data_ptr())  # noqa: E731
    null = ffi.NULL

    def call(act=1, slope=0.0, scale=null, D=1, kt=1):
        return lib.cp_patch_gather_act(engine.h, p(x, "const void*"), 0, 1, 2, 16, D, 6, 6, 0, null,
                                       p(rx, "const int32_t*"), p(rx, "const int32_t*"), 1, kt, 3, 3, 0, 1, 1, 1, 1, 1,
                                       1, 1, 1, 0, act, slope, scale, null, p(out, "float*"), 16 * 9, null)

    assert call(act=3, slope=0.1, scale=p(sc, "const float*")) == 0
    torch.cuda.synchronize()
    for kw in (dict(act=6), dict(act=-1), dict(act=3, slope=float("nan")), dict(act=3, slope=float("inf")),
               dict(scale=p(sc_host, "const float*")), dict(D=2), dict(kt=2)):
        assert call(**kw) == -1, kw  # CP_ERR_INVALID
    with pytest.raises(ValueError):
        engine.patch_gather(x, rx, rx, 2, 1, 3, 1, 1, relu=True, act="silu")
    with pytest.raises(ValueError):
        engine.patch_gather(x, rx, rx, 2, 1, 3, 1, 1, act="relu6", act_param=0.5)
    with pytest.raises(AssertionError):
        engine.patch_gather(x, rx, rx, 2, 1, 3, 1, 1, act="silu", in_scale=torch.ones(15, device=dev))


# ----------------------------------------------------------------------------- which kernel runs
_KERNEL_CASES = [("conv2d", "nchw", "nchw"), ("conv2d", "nchw_host", "nchw"), ("conv2d", "nhwc_tma", "nhwc_tma"),
                 ("conv2d", "nhwc_simt", "nhwc"), ("conv2d", "nhwc_host", "nhwc_host"),
                 ("conv3d", "ncdhw", "ncdhw"), ("conv3d", "ncdhw_host", "ncdhw"), ("conv3d", "ndhwc_tma", "ndhwc_tma"),
                 ("conv3d", "ndhwc_simt", "ndhwc"), ("conv3d", "ndhwc_host", "ndhwc_host"),
                 ("tr2d", "tr_nchw", "tr_nchw"), ("tr2d", "tr_nhwc_host", "tr_nhwc"),
                 ("tr3d", "tr_ncdhw_host", "tr_ncdhw"), ("tr3d", "tr_ndhwc", "tr_ndhwc")]
_REPEAT = 2


def _profile_kernel_cases():
    """Every case of _KERNEL_CASES with BN + SiLU, _REPEAT times in one profiler session; the gather launches' names."""
    import cpb200
    from torch.profiler import ProfilerActivity, profile

    engine = cpb200.get_engine()
    dev = engine.device
    runs = []
    for fam, path, _ in _KERNEL_CASES:
        geom = GEOMS[fam][0]
        pts, P = _points(fam, _out_size(fam, DIMS[fam], geom), 2, dev)
        c = PATHS[fam][path][2]
        x = torch.randn((4, c) + DIMS[fam], device=dev)
        scale, shift = _affine(c, "bn", dev)
        call = (lambda fam=fam, path=path, x=x, pts=pts, P=P, geom=geom, scale=scale, shift=shift:
                _gather(engine, fam, path, x, pts, 2, P, geom, "silu", None, scale, shift))
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
    """Each path launches its own kernel's fused (XFORM = true) instantiation."""
    import re

    def kind_of(n):
        m = re.search(r"patch_gather_([a-z_]+)<", n)
        if not m:
            return n
        return m.group(1) if re.search(r"[<,]true[,>]", n) else "unfused:" + m.group(1)

    want = {}
    for _, _, kind in _KERNEL_CASES:
        want[kind] = want.get(kind, 0) + _REPEAT
    GC.assert_launch_counts(GC.launched_gather_kernels("test_gpu_conv_bn_act"), kind_of, want)


# ----------------------------------------------------------------------------- PyTorch cross-check
TORCH_ACTS = {"relu": (torch.nn.ReLU(), None), "relu6": (torch.nn.ReLU6(), None),
              "leaky_relu": (torch.nn.LeakyReLU(0.1), 0.1), "silu": (torch.nn.SiLU(), None),
              "hardswish": (torch.nn.Hardswish(), None)}


@pytest.mark.parametrize("act", list(TORCH_ACTS))
def test_against_torch_conv_bn_act_conv(engine, act):
    """Conv2d -> BatchNorm2d (eval) -> act -> Conv2d: X gathered from the hooked raw output of the first conv through
    fold_bn equals F.unfold(act(bn(raw))) at the points to 1e-6, and X @ W2.T + b is the second conv's output there."""
    import cpb200

    dev = engine.device
    g = torch.Generator().manual_seed(7)
    conv1, bn, conv2 = torch.nn.Conv2d(8, 16, 3, padding=1), torch.nn.BatchNorm2d(16), torch.nn.Conv2d(16, 12, 3,
                                                                                                        padding=1)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(16, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(16, generator=g))
        bn.running_mean.copy_(torch.randn(16, generator=g) * 0.3)
        bn.running_var.copy_(torch.rand(16, generator=g) + 0.5)
    mod, slope = TORCH_ACTS[act]
    net = torch.nn.Sequential(conv1, bn, mod, conv2).eval().to(dev)
    raw = {}
    conv1.register_forward_hook(lambda m, i, o: raw.__setitem__("x", o.detach()))
    conv2.register_forward_hook(lambda m, i, o: raw.__setitem__("y", o.detach()))
    B, H = 4, 10
    x = torch.randn(B, 8, H, H, generator=g).to(dev)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            net(x)
            want_in = mod(bn(raw["x"]))
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    r = np.random.RandomState(1)
    P = 30
    rx = torch.as_tensor(r.randint(0, H, (1, P)).astype(np.int32), device=dev)
    ry = torch.as_tensor(r.randint(0, H, (1, P)).astype(np.int32), device=dev)
    rx[0, :4], ry[0, :4] = torch.tensor([0, 0, H - 1, H - 1]), torch.tensor([0, H - 1, 0, H - 1])
    scale, shift = cpb200.synth.fold_bn(bn)
    X = engine.patch_gather(raw["x"].contiguous(), rx, ry, B, P, 3, 1, 1, act=act, act_param=slope, in_scale=scale,
                            in_shift=shift)
    cols = F.unfold(want_in, 3, padding=1)  # (B, 16*9, H*W)
    idx = (rx[0] * H + ry[0]).long()
    want = cols[:, :, idx].permute(2, 0, 1).reshape(P * B, -1)  # rows (point, image)
    assert (X - want).norm().item() <= 1e-6 * want.norm().item()
    # the padded taps of the corner point (0, 0) (rows 0 .. B-1): +0, not act(shift)
    corner = X.reshape(P * B, 16, 9)[:B, :, [0, 1, 2, 3, 6]]
    assert (corner == 0).all() and not torch.signbit(corner).any()
    Y = engine.point_gather(raw["y"].contiguous(), rx, ry, B, P)
    Yx = X.double() @ conv2.weight.reshape(12, -1).T.double() + conv2.bias.double()
    assert (Yx - Y.double()).norm().item() <= 1e-5 * Y.double().norm().item()


# ----------------------------------------------------------------------------- pipeline
def _bn_layers(act, N=800, B=4, P=10):
    import cpb200

    sy = cpb200.synth
    kw = dict(N=N, B=B, P=P, act=act, bn=True)
    return [sy.LayerShape("conv2d", 32, 24, 10, **kw),
            sy.LayerShape("conv2d_1x1", 48, 32, 8, k=1, pad=0, **kw),
            sy.LayerShape3d("conv3d", 24, 16, 4, 6, **kw),
            sy.LayerShape("up2d", 32, 16, 6, k=2, stride=2, pad=0, transposed=True, **kw),
            sy.LayerShape3d("up3d", 16, 12, 3, 4, k=2, stride=2, pad=0, transposed=True, **kw)]


@pytest.mark.parametrize("act", ["silu", "relu"])
@pytest.mark.parametrize("host_layout", ["nchw", "nhwc"])
def test_pipeline_on_bn_layers(engine, act, host_layout):
    """prune_layers on BN + act layers (2-D, 1 x 1, 3-D, transposed): maps in HBM, read in place from pinned host
    memory ('zc') or staged by DMA ('copy') -- identical masks, alpha, probe counts, W and b; and the oracle on the
    GPU's own X gives the same masks, alpha and probe counts, W and b within 1e-7 (fp64 statistics)."""
    import cpb200
    from cpb200 import pruner

    eng = cpb200.Engine(nstreams=4)
    eng.gram_mode = 0
    shapes = _bn_layers(act)
    datas = [cpb200.synth.make_problem_device(s, 60 + i, eng, pinned_host=True, host_layout=host_layout)
             for i, s in enumerate(shapes)]
    ref = pruner.prune_layers(eng, shapes, datas)
    torch.cuda.synchronize()
    assert [r.info["verdict"] for r in ref] == ["ok"] * len(shapes)
    ref = [(r.idxs.copy(), r.alpha, r.nprobe, r.W.cpu(), r.b.cpu()) for r in ref]
    for policy in ("zc", "copy"):
        got = pruner.prune_layers(eng, shapes, datas, from_host=policy, to_host=True)
        torch.cuda.synchronize()
        for s, (idxs, alpha, nprobe, W, b), r in zip(shapes, ref, got):
            assert np.array_equal(idxs, r.idxs) and alpha == r.alpha and nprobe == r.nprobe, (policy, s.name)
            assert torch.equal(W, r.W) and torch.equal(b, r.b), (policy, s.name)
    if host_layout == "nchw":
        for s, d, (idxs, alpha, nprobe, W, b) in zip(shapes, datas, ref):
            X = pruner._patch_gather(eng, s, d, d["fmap"], d["layout"])
            X = X.cpu().numpy().astype(np.float64).reshape((s.N, s.c) + pruner.window_of(s))
            oi, oW, oB, oalpha, onprobe = GC.oracle_on_problem(C3.dictionary, X, s, d)
            assert np.array_equal(idxs, oi) and alpha == oalpha and nprobe == onprobe, s.name
            assert GC.rel(W.numpy().reshape(oW.shape), oW) <= 1e-7 and np.abs(b.numpy() - oB).max() <= 1e-7, s.name
    eng.close()


def test_bn_problem_differs_from_the_plain_one_and_pads_with_zeros(engine):
    """The device generator's bn X: the transform of the map inside it, +0 at the padded taps (shift != 0)."""
    import cpb200
    from cpb200 import pruner

    s = cpb200.synth.LayerShape("L", 16, 8, 6, N=200, B=4, P=5, act="silu", bn=True)
    d = cpb200.synth.make_problem_device(s, 5, engine)
    X = pruner._patch_gather(engine, s, d, d["fmap"], d["layout"])
    pts = [d[k].cpu().numpy() for k in ("randx", "randy")]
    inmap = cpb200.synth.gather_patches_numpy(np.ones((s.nbatch * s.B, 1, s.H, s.W), np.float32), *pts, s.B, s.k,
                                              s.pad, s.stride, relu=False) != 0
    inmap = np.broadcast_to(inmap, (s.N, s.c, 3, 3)).reshape(s.N, -1)
    Xn = X.cpu().numpy()
    assert (~inmap).any() and not np.signbit(Xn[~inmap]).any() and (Xn[~inmap] == 0).all()
    assert d["in_shift"].abs().max().item() > 0.3


def test_prune_network_sharded_on_bn_layers(engine):
    """One rank: unpack_network gives the values prune_layers returns, for BN + SiLU layers."""
    import cpb200
    from cpb200 import pruner

    eng = cpb200.Engine(nstreams=4)
    eng.gram_mode = 0
    shapes = _bn_layers("silu")
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
