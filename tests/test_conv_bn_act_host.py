"""CPU: the consumer input transform of Conv-BN-activation networks on the host side -- the numpy statement of every
activation on special values, fold_bn against torch's eval-mode BatchNorm, the layer shape's checks, the zero padding
of a bn problem, and the default generator left as it was."""
import numpy as np
import pytest

import cpb200
from cpb200 import synth

f32 = np.float32
SPECIALS = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, 1.2e-38, -1.2e-38, 1.0, -1.0, 3.0, -3.0,
                     -4.0, 7.0, -100.0], dtype=f32)


def _bits(a):
    return np.asarray(a, dtype=f32).view(np.int32)


def _same(got, want):
    got, want = np.asarray(got, dtype=f32), np.asarray(want, dtype=f32)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (got, want)
    ok = ~np.isnan(want)
    assert np.array_equal(_bits(got[ok]), _bits(want[ok])), (got, want)


def _apply(act, v, **kw):
    return synth.input_transform_numpy(v.reshape(1, -1), act, **kw).reshape(-1)


def test_relu_and_relu6_on_special_values():
    nan_gives = f32(0)  # fmaxf(NaN, 0) is 0, as the relu gathers give it
    want = [0.0, 0.0, np.inf, 0.0, nan_gives, 1e-45, 0.0, 1.2e-38, 0.0, 1.0, 0.0, 3.0, 0.0, 0.0, 7.0, 0.0]
    _same(_apply("relu", SPECIALS), want)
    assert not np.signbit(_apply("relu", SPECIALS)).any()
    want6 = [0.0, 0.0, 6.0, 0.0, 0.0, 1e-45, 0.0, 1.2e-38, 0.0, 1.0, 0.0, 3.0, 0.0, 0.0, 6.0, 0.0]
    _same(_apply("relu6", SPECIALS), want6)


def test_identity_leaky_and_hardswish_on_special_values():
    _same(_apply("identity", SPECIALS), SPECIALS)
    assert np.signbit(_apply("identity", SPECIALS))[1]  # no arithmetic: -0 stays -0
    lk = _apply("leaky_relu", SPECIALS, act_param=0.25)
    want = [0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, f32(-1e-45) * f32(0.25), 1.2e-38, f32(-1.2e-38) * f32(0.25),
            1.0, -0.25, 3.0, -0.75, -1.0, 7.0, -25.0]
    _same(lk, want)
    _same(_apply("leaky_relu", np.array([-2.0], f32)), [f32(-2.0) * f32(0.01)])  # torch's default slope
    hs = _apply("hardswish", SPECIALS)
    # (v * min(max(v + 3, 0), 6)) / 6 in float32: -inf * 0 is NaN, -3 and below give -0 or +0 as the product's sign
    want = [0.0, -0.0, np.inf, np.nan, np.nan, f32(f32(1e-45) * f32(3)) / f32(6), -0.0, f32(f32(1.2e-38) * f32(3)) / f32(6),
            f32(f32(-1.2e-38) * f32(3)) / f32(6), f32(4) / f32(6), f32(-2) / f32(6), 3.0, -0.0, -0.0, 7.0, -0.0]
    _same(hs, want)


def test_silu_is_the_rounded_float64_value():
    v = SPECIALS.astype(np.float64)
    with np.errstate(all="ignore"):
        want = (v / (1.0 + np.exp(-v))).astype(f32)
    _same(_apply("silu", SPECIALS), want)
    assert _apply("silu", np.array([-100.0], f32))[0] < 0  # no overflow to -0 in the tail


def test_affine_is_two_rounded_float32_operations():
    r = np.random.RandomState(3)
    v = r.standard_normal((5, 4, 3)).astype(f32)
    sc, sh = r.uniform(0.5, 1.5, 4).astype(f32), r.standard_normal(4).astype(f32)
    got = synth.input_transform_numpy(v, "identity", scale=sc, shift=sh)
    want = np.empty_like(v)
    for a in range(4):
        for i in np.ndindex(5, 3):
            want[i[0], a, i[1]] = f32(f32(v[i[0], a, i[1]] * sc[a]) + sh[a])
    _same(got, want)
    _same(synth.input_transform_numpy(v, "identity", shift=sh), v + sh.reshape(1, 4, 1))


def test_fold_bn_matches_eval_mode_batchnorm():
    torch = pytest.importorskip("torch")
    g = torch.Generator().manual_seed(0)
    bn = torch.nn.BatchNorm2d(32, eps=1e-3)
    with torch.no_grad():
        bn.weight.copy_(torch.rand(32, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(32, generator=g))
        bn.running_mean.copy_(torch.randn(32, generator=g))
        bn.running_var.copy_(torch.rand(32, generator=g) * 3 + 0.1)
    bn.eval()
    before = {k: v.clone() for k, v in bn.state_dict().items()}
    scale, shift = synth.fold_bn(bn)
    assert scale.dtype == shift.dtype == torch.float32 and scale.is_contiguous() and scale.shape == (32,)
    x = torch.randn(4, 32, 5, 5, generator=g)
    with torch.no_grad():
        want = bn(x).double()
    got = x.double() * scale.double().view(1, -1, 1, 1) + shift.double().view(1, -1, 1, 1)
    assert ((got - want).norm() / want.norm()).item() <= 1e-6
    # float64 then one rounding
    w64 = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
    assert torch.equal(scale, w64.float())
    assert torch.equal(shift, (bn.bias.double() - bn.running_mean.double() * w64).float())
    assert all(torch.equal(v, bn.state_dict()[k]) for k, v in before.items())


def test_layer_shape_checks_its_transform():
    with pytest.raises(ValueError):
        synth.LayerShape("L", 8, 8, 6, act="gelu")
    with pytest.raises(ValueError):
        synth.LayerShape("L", 8, 8, 6, act="relu", act_param=0.1)
    with pytest.raises(ValueError):
        synth.LayerShape3d("L", 8, 8, 4, 6, act="silu", act_param=0.1)
    s = synth.LayerShape("L", 8, 8, 6, act="leaky_relu", act_param=0.1, bn=True)
    assert (s.act, s.act_param, s.bn) == ("leaky_relu", 0.1, True)
    s = synth.LayerShape("L", 8, 8, 6)
    assert (s.act, s.act_param, s.bn) == ("relu", None, False)


def test_resnet50_bn_layers():
    plain, bn = synth.resnet50_layers(), synth.resnet50_layers(bn=True)
    assert [s.name for s in plain] == [s.name for s in bn]
    for s in bn:
        assert s.act == "relu" and s.bn == (not s.name.endswith("branch2a"))
    assert not any(s.bn for s in plain)


@pytest.mark.parametrize("kind", ["conv2d", "conv3d", "tr2d"])
@pytest.mark.parametrize("act", ["silu", "relu", "identity"])
def test_bn_problem_pads_with_zeros(kind, act):
    """A padded layer's X: +0 at every out-of-range tap, the transform of the map elsewhere."""
    if kind == "conv3d":
        s = synth.LayerShape3d("L", 4, 3, 4, 5, k=3, pad=1, N=100, B=2, P=5, act=act, bn=True)
    elif kind == "tr2d":
        s = synth.LayerShape("L", 4, 3, 5, k=4, pad=1, stride=2, N=100, B=2, P=5, act=act, bn=True, transposed=True)
    else:
        s = synth.LayerShape("L", 4, 3, 5, k=3, pad=2, dilation=2, N=100, B=2, P=5, act=act, bn=True)
    d = synth.make_problem_numpy(s, 11)
    sc, sh = d["in_scale"], d["in_shift"]
    assert np.abs(sh).max() > 0.3 and (np.abs(sc) >= 0.5).all()
    pts = [d[k] for k in (("randt", "randx", "randy") if kind == "conv3d" else ("randx", "randy"))]
    gather = {"conv2d": synth.gather_patches_numpy, "conv3d": synth.gather_patches3d_numpy,
              "tr2d": synth.gather_patches_tr_numpy}[kind]
    ones = np.ones_like(d["fmap"])
    inmap = gather(ones, *pts, s.B, s.k, s.pad, s.stride, relu=False, dilation=s.dilation) != 0
    raw = gather(d["fmap"], *pts, s.B, s.k, s.pad, s.stride, relu=False, dilation=s.dilation)
    X = d["X"]
    assert (~inmap).any() and inmap.any()
    assert np.array_equal(_bits(X[~inmap]), np.zeros((~inmap).sum(), np.int32))  # +0, not act(shift)
    _same(X[inmap], synth.input_transform_numpy(raw, act, scale=sc, shift=sh)[inmap])


def test_default_generator_is_unchanged():
    """make_problem_numpy of a default shape draws what it always drew: the stream restated here, and a bn shape of
    the same seed shares every draw but X and the targets."""
    s = synth.LayerShape("L", 6, 5, 7, k=3, pad=1, N=100, B=2, P=5)
    d = synth.make_problem_numpy(s, 5)
    r = np.random.RandomState(5)
    fmap = r.standard_normal((s.nbatch * s.B, s.c, s.H, s.W)).astype(f32)
    randx = r.randint(0, s.Ho, (s.nbatch, s.P)).astype(np.int32)
    randy = r.randint(0, s.Wo, (s.nbatch, s.P)).astype(np.int32)
    W2 = (r.standard_normal((s.n, s.c, s.kh, s.kw)) * np.sqrt(2.0 / (s.c * s.k2))).astype(f32)
    b2 = (0.01 * r.standard_normal(s.n)).astype(f32)
    X = synth.gather_patches_numpy(fmap, randx, randy, s.B, s.k, s.pad, s.stride, relu=True)
    Y = X.reshape(s.N, -1).astype(np.float64) @ W2.reshape(s.n, -1).T.astype(np.float64) + b2
    Y = Y + 0.01 * Y.std() * r.standard_normal(Y.shape)
    samples = r.randint(0, s.N, s.S)
    for k, v in dict(fmap=fmap, randx=randx, randy=randy, W2=W2, b2=b2, X=X, feats=Y.astype(f32),
                     samples=samples).items():
        assert np.array_equal(d[k], v), k
    assert "in_scale" not in d
    sb = synth.LayerShape("L", 6, 5, 7, k=3, pad=1, N=100, B=2, P=5, bn=True)
    db = synth.make_problem_numpy(sb, 5)
    for k in ("fmap", "randx", "randy", "W2", "b2", "samples"):
        assert np.array_equal(db[k], d[k]), k
    assert not np.array_equal(db["X"], d["X"])


def test_engine_refuses_relu_and_act_together():
    from cpb200.engine import input_transform

    with pytest.raises(ValueError):
        input_transform(True, "silu", None, None, None, 4, None)
    with pytest.raises(ValueError):
        input_transform(None, "relu", 0.1, None, None, 4, None)
    with pytest.raises(ValueError):
        input_transform(None, "tanh", None, None, None, 4, None)
    assert input_transform(None, None, None, None, None, 4, None) is None
    assert input_transform(False, None, None, None, None, 4, None) is None
    assert input_transform(None, "identity", None, None, None, 4, None) is None
    assert input_transform(None, "leaky_relu", None, None, None, 4, None) == (3, 0.01, None, None)
    assert cpb200.engine.ACTS["silu"] == 5
