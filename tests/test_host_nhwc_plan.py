"""CPU: the transfer plan of channels-last (NHWC) host maps -- the line model of the in-place NHWC reader against a
brute-force count, and h2d_plan's rule with it (meta tensors: no memory, no GPU)."""
import types

import numpy as np
import pytest

import gather_checks as GC

torch = pytest.importorskip("torch")


def _brute_lines(c, H, W, k, pad, stride, esize, img, x, y):
    """128-byte lines of an NHWC map (base 128-byte aligned) that the in-bounds taps of one window touch."""
    lines = set()
    y0, x0 = stride * x - pad, stride * y - pad
    for py in range(k):
        yy = y0 + py
        if not 0 <= yy < H:
            continue
        xs = [xx for xx in range(x0, x0 + k) if 0 <= xx < W]
        if not xs:
            continue
        start = ((img * H + yy) * W + xs[0]) * c * esize
        end = ((img * H + yy) * W + xs[-1] + 1) * c * esize
        lines.update(range(start // 128, (end - 1) // 128 + 1))
    return len(lines), y0 >= 0 and x0 >= 0 and y0 + k <= H and x0 + k <= W


@pytest.mark.parametrize("esize", [4, 2])
@pytest.mark.parametrize("c", [1, 3, 5, 12, 16, 24, 32, 64, 96, 512])
@pytest.mark.parametrize("k,pad,stride", [(1, 0, 1), (1, 0, 2), (3, 1, 1), (3, 0, 1), (3, 1, 2), (5, 2, 1)])
def test_nhwc_line_model_bounds_the_lines_a_window_touches(esize, c, k, pad, stride):
    """The model never counts fewer lines than a window touches.  For an interior window whose rows share no line, it
    counts at most one more per window row (the line a run starting inside a line adds); with a pixel stride of whole
    lines it is exact for interior windows."""
    from cpb200 import pruner

    H = W = 7
    Ho = (H + 2 * pad - k) // stride + 1
    s = types.SimpleNamespace(N=1, c=c, k=k, W=W)
    model = pruner.zero_copy_lines(s, esize, "nhwc")
    r = np.random.RandomState(c * 10 + k + esize)
    pts = [(0, 0), (0, Ho - 1), (Ho - 1, 0), (Ho - 1, Ho - 1)] + [tuple(p) for p in r.randint(0, Ho, (60, 2))]
    for x, y in pts:
        img = int(r.randint(0, 5))
        got, interior = _brute_lines(c, H, W, k, pad, stride, esize, img, x, y)
        assert got <= model, (x, y, got, model)
        if interior and (W - k) * c * esize >= 128:
            assert model - got <= k, (x, y, got, model)
            if (c * esize) % 128 == 0:
                assert got == model


def test_nhwc_line_model_at_vgg16_shapes():
    """conv4_2 (c 512, k 3): a window row is 6144 fp32 bytes = 48 whole lines, 24 in 16 bit; conv1_1 (c 3): a 36-byte
    row may straddle two lines.  NCHW counts are unchanged by the layout argument's default."""
    import cpb200
    from cpb200 import pruner

    by_name = {s.name: s for s in cpb200.synth.vgg16_layers()}
    assert pruner.zero_copy_lines(by_name["conv4_2"], 4, "nhwc") == 5000 * 3 * 48
    assert pruner.zero_copy_lines(by_name["conv4_2"], 2, "nhwc") == 5000 * 3 * 24
    assert pruner.zero_copy_lines(by_name["conv1_1"], 4, "nhwc") == 5000 * 3 * 2
    for s in by_name.values():
        for es in (4, 2):
            assert pruner.zero_copy_lines(s, es) == pruner.zero_copy_lines(s, es, "nchw")
            assert pruner.zero_copy_lines(s, es, "nhwc") < pruner.zero_copy_lines(s, es, "nchw")


def _maps(shapes, dtype, host_layout=None):
    out = []
    for s in shapes:
        shape = (s.nbatch * s.B, s.H, s.W, s.c) if host_layout == "nhwc" else (s.nbatch * s.B, s.c, s.H, s.W)
        d = dict(fmap_host=torch.empty(shape, dtype=dtype, device="meta"))
        if host_layout is not None:
            d["host_layout"] = host_layout
        out.append(d)
    return out


@pytest.fixture
def default_rule(monkeypatch):
    monkeypatch.delenv("CPB200_DMA_MAX_MB", raising=False)
    monkeypatch.delenv("CPB200_DMA_RATIO", raising=False)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=["fp32", "bf16", "fp16"])
def test_plan_of_nhwc_maps_uses_nhwc_lines_and_their_rate(default_rule, dtype):
    from cpb200 import pruner

    shapes = GC.all_shapes()
    datas = _maps(shapes, dtype, "nhwc")
    es = torch.empty((), dtype=dtype).element_size()
    plan = pruner.h2d_plan(shapes, datas, True)
    for s, d, p in zip(shapes, datas, plan):
        nbytes = d["fmap_host"].numel() * es
        t_zc = pruner.zero_copy_lines(s, es, "nhwc") / pruner.ZC_NHWC_LINES_PER_S
        dma = nbytes <= 300e6 and nbytes / 50e9 + 1e-4 < 0.8 * t_zc
        assert p == ("dma" if dma else "zc"), s.name
    assert pruner.h2d_plan(shapes, datas, "zc") == ["zc"] * len(shapes)
    assert pruner.h2d_plan(shapes, datas, "copy") == ["dma"] * len(shapes)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_maps_without_host_layout_keep_todays_plan(default_rule, dtype):
    """No host_layout key: NCHW lines at ZC_LINES_PER_S, exactly the plan an explicit 'nchw' gets."""
    from cpb200 import pruner

    shapes = GC.all_shapes()
    plain = _maps(shapes, dtype)
    es = torch.empty((), dtype=dtype).element_size()
    want = []
    for s, d in zip(shapes, plain):
        nbytes = d["fmap_host"].numel() * es
        dma = nbytes <= 300e6 and nbytes / 50e9 + 1e-4 < 0.8 * pruner.zero_copy_lines(s, es) / pruner.ZC_LINES_PER_S
        want.append("dma" if dma else "zc")
    assert pruner.h2d_plan(shapes, plain, True) == want
    assert pruner.h2d_plan(shapes, _maps(shapes, dtype, "nchw"), True) == want
    assert pruner.h2d_plan(shapes, plain, "zc") == ["zc"] * len(shapes)
    assert pruner.h2d_plan(shapes, plain, "copy") == ["dma"] * len(shapes)
