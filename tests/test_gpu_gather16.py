"""GPU: gathers of bf16 / fp16 feature maps.  Widening a 16-bit value to fp32 is exact, so every gather of a 16-bit
map must produce the bits the fp32 gather of the widened map produces -- on the TMA and SIMT paths, from HBM and from
pinned host memory, and through the whole pruning walk."""
import numpy as np
import pytest

import cases
import gather_checks as GC

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

DTYPES = pytest.mark.parametrize("dtype", ["bf16", "fp16"])
_T = {"bf16": torch.bfloat16, "fp16": torch.float16}
# (k, pad, stride): every kernel size the kernels specialise, stride 1 and 2
WINDOWS = [(1, 0, 1), (1, 0, 2), (3, 1, 1), (3, 1, 2), (5, 2, 1), (5, 2, 2)]
CHANNELS = [3, 12, 16, 24, 64, 512, 2048]


def _map16(shape, dtype, seed, device):
    """N(0,1) drawn in fp32 and rounded, with -0, +-inf, NaN and subnormals (of fp16 and of bf16) seeded in."""
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    fm = torch.randn(shape, generator=g, device=device)
    flat = fm.view(-1)
    specials = torch.tensor([-0.0, float("inf"), float("-inf"), float("nan"), 6e-8, -3e-6, 4e-5, 1e-39, -5e-39],
                            device=device)
    idx = torch.randperm(flat.numel(), generator=g, device=device)[:max(len(specials), flat.numel() // 40)]
    flat[idx] = specials[torch.arange(idx.numel(), device=device) % len(specials)]
    return fm.to(_T[dtype])


def _points(nb, Ho, device):
    """Every corner and border of the output map, plus the centre, in varying order per batch."""
    pts = [(0, 0), (0, Ho - 1), (Ho - 1, 0), (Ho - 1, Ho - 1), (Ho // 2, Ho // 2), (1 % Ho, Ho - 1), (Ho - 1, 1 % Ho)]
    rx = torch.tensor([[p[0] for p in pts]] * nb, dtype=torch.int32, device=device)
    ry = torch.tensor([[p[1] for p in pts]] * nb, dtype=torch.int32, device=device)
    rx[1] = rx[1].flip(0)
    return rx, ry, len(pts)


@DTYPES
@pytest.mark.parametrize("c", CHANNELS)
@pytest.mark.parametrize("k,pad,stride", WINDOWS)
def test_patch_gather_of_16bit_map_equals_gather_of_widened_map(engine, dtype, c, k, pad, stride):
    dev = engine.device
    H = 9
    B, nb = 3, 4
    m16 = _map16((nb * B, c, H, H), dtype, c * 31 + k * 7 + stride, dev)
    m32 = m16.float()
    rx, ry, P = _points(nb, (H + 2 * pad - k) // stride + 1, dev)
    for layout in ("nchw", "nhwc"):
        a16 = m16 if layout == "nchw" else m16.permute(0, 2, 3, 1).contiguous()
        a32 = m32 if layout == "nchw" else m32.permute(0, 2, 3, 1).contiguous()
        for relu in (False, True):
            want = engine.patch_gather(a32, rx, ry, B, P, k, pad, stride, relu=relu, layout=layout)
            got = engine.patch_gather(a16, rx, ry, B, P, k, pad, stride, relu=relu, layout=layout)
            GC.assert_same_bits(got, want)
            if relu:
                assert not bool(torch.isnan(got).any())  # fmaxf(NaN, 0) = 0, as in the fp32 kernel


PATH_SHAPES = [(16, 3), (24, 5), (64, 1), (512, 3), (2048, 1), (20, 3), (12, 3)]
_PATH_CASES = [(dtype, c, k) for dtype in ("bf16", "fp16") for c, k in PATH_SHAPES]


def _profile_kernel_cases():
    """Gathers every case of _PATH_CASES once inside one profiler session, after a warm-up whose bits are checked
    against the gather of the widened map; returns the gather kernels' names in launch order."""
    import cpb200
    from torch.profiler import ProfilerActivity, profile

    engine = cpb200.get_engine()
    dev = engine.device
    H, B, nb, stride = 7, 2, 2, 1
    rx, ry, P = _points(nb, H, dev)
    runs = []
    for dtype, c, k in _PATH_CASES:
        m16 = _map16((nb * B, H, H, c), dtype, c + k, dev)
        out = engine.patch_gather(m16, rx, ry, B, P, k, k // 2, stride, layout="nhwc")  # warm-up (module load)
        want = engine.patch_gather(m16.float(), rx, ry, B, P, k, k // 2, stride, layout="nhwc")
        GC.assert_same_bits(out, want)
        runs.append((k, m16, out))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k, m16, out in runs:
            engine.patch_gather(m16, rx, ry, B, P, k, k // 2, stride, layout="nhwc", out=out)
        torch.cuda.synchronize()
    kernels = sorted((e for e in prof.events() if "patch_gather" in e.name and e.device_type.name == "CUDA"),
                     key=lambda e: e.time_range.start)
    return [e.name for e in kernels]


def test_16bit_nhwc_path_is_the_one_its_shape_selects(engine):
    """c % 8 == 0 and c >= 16: the TMA kernel must be what ran (a silent SIMT fall-back would pass the bit checks
    above).  c = 20 takes TMA as fp32 but not in 16 bit (40-byte channel stride); c = 12 never does.  One profiler
    session for every case: the launches run in order on one stream, so the i-th kernel belongs to the i-th case.  The
    session runs in a child process: a process that has profiled once may lose activity records in its later
    sessions, and this check counts every launch."""
    names = GC.launched_gather_kernels("test_gpu_gather16")
    assert len(names) == len(_PATH_CASES), names
    for (dtype, c, k), n in zip(_PATH_CASES, names):
        tma = c % 8 == 0 and c >= 16
        assert ("patch_gather_nhwc_tma" in n) == tma, (dtype, c, k, n)
        assert "patch_gather_nhwc" in n and ("bfloat16" if dtype == "bf16" else "half") in n, n


@DTYPES
@pytest.mark.parametrize("c,k,pad,stride", [(3, 3, 1, 1), (64, 3, 1, 2), (256, 1, 0, 1), (96, 5, 2, 1)])
def test_pinned_host_nchw_reader_of_16bit_map(engine, dtype, c, k, pad, stride):
    """The in-place reader over PCIe (the host-resident input path) on a 16-bit pinned map."""
    dev = engine.device
    H, B, nb = 11, 3, 4
    m16 = _map16((nb * B, c, H, H), dtype, 500 + c, dev)
    host = GC.pinned(m16)
    rx, ry, P = _points(nb, (H + 2 * pad - k) // stride + 1, dev)
    for relu in (False, True):
        want = engine.patch_gather(m16.float(), rx, ry, B, P, k, pad, stride, relu=relu)
        got = engine.patch_gather(host, rx, ry, B, P, k, pad, stride, relu=relu)
        torch.cuda.synchronize()
        GC.assert_same_bits(got, want)


@DTYPES
@pytest.mark.parametrize("n", [3, 12, 64, 512, 2048])
def test_point_gather_of_16bit_map_equals_gather_of_widened_map(engine, dtype, n):
    dev = engine.device
    H, B, nb = 9, 3, 4
    m16 = _map16((nb * B, n, H, H), dtype, 900 + n, dev)
    rx, ry, P = _points(nb, H, dev)
    host = GC.pinned(m16)
    want = engine.point_gather(m16.float(), rx, ry, B, P)
    GC.assert_same_bits(engine.point_gather(m16, rx, ry, B, P), want)
    GC.assert_same_bits(engine.point_gather(host, rx, ry, B, P), want)
    torch.cuda.synchronize()
    l16, l32 = m16.permute(0, 2, 3, 1).contiguous(), m16.float().permute(0, 2, 3, 1).contiguous()
    GC.assert_same_bits(engine.point_gather(l16, rx, ry, B, P, layout="nhwc"),
                        engine.point_gather(l32, rx, ry, B, P, layout="nhwc"))


# ---------------------------------------------------------------------------- end to end
class _Widened:
    """A feature provider's blobs widened to fp32 (exact): what a caller had to do before 16-bit maps were read."""

    def __init__(self, inner):
        self.inner = inner

    def data(self, batch):
        return self.inner.data(batch)

    def __call__(self, net, data, upto=None):
        return {k: v.float() for k, v in self.inner(net, data, upto=upto).items()}


@pytest.fixture
def deterministic_convs():
    """The two walks below must see the same bf16 blobs: cuDNN may otherwise pick its algorithm per call."""
    old = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = old


def _r3_walk(engine, widen):
    from cpb200.lib import cfgs
    from cpb200.lib import net as cpnet

    spec = cases.R3_CASES["r3_small"]
    images, specs, weights, biases = cases.r3_inputs(**spec["gen"])
    cs = [cpnet.ConvSpec(s["name"], s["bottom"], weights[s["name"]].shape[0], s["k"], s["pad"], s["stride"],
                         pool_after=(s["name"] == "conv1_2")) for s in specs if s.get("type") != "pool"]
    provider = cpnet.ConvStackForward(lambda b: torch.as_tensor(images[b % len(images)], device=engine.device),
                                      dtype=torch.bfloat16)
    net = cpnet.Net(cs, weights, biases, _Widened(provider) if widen else provider, pool_names={"conv1_2": "pool1"})
    cfgs.c.nBatches, cfgs.c.nPointsPerLayer = spec["nBatches"], spec["P"]
    cfgs.c.dic.vh, cfgs.c.dic.keep = 1, 3.
    cfgs.alpha = 1e-3
    np.random.seed(spec["np_seed"])
    blobs = net.forward(torch.as_tensor(images[0], device=engine.device))
    feats, points = net.freeze()
    WPQ, new_pt = net.R3()
    return dict(blob_dtype=blobs["conv1_1"].dtype, feats=feats, points=points, WPQ=WPQ, new_pt=new_pt,
                sel=dict(net.selection), w={k: v.cpu().numpy() for k, v in net._w.items()},
                b={k: v.cpu().numpy() for k, v in net._b.items()}, alpha=cfgs.alpha, rng=np.random.get_state())


def _same_dict(a, b):
    assert set(a) == set(b)
    for k in a:
        if isinstance(a[k], np.ndarray):
            assert a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k]), k
        else:
            assert a[k] == b[k], k


def test_r3_walk_on_bf16_blobs_equals_the_walk_on_widened_blobs(engine, deterministic_convs):
    """Net on a bf16 forward pass: frozen features, selections, WPQ, final weights, the alpha carried through the walk
    and the RNG draws are those of the same blobs widened to fp32."""
    a = _r3_walk(engine, widen=False)
    b = _r3_walk(engine, widen=True)
    assert a["blob_dtype"] == torch.bfloat16 and b["blob_dtype"] == torch.float32
    _same_dict(a["feats"], b["feats"])
    _same_dict(a["points"], b["points"])
    _same_dict(a["sel"], b["sel"])
    assert len(a["sel"]) > 0
    _same_dict(a["WPQ"], b["WPQ"])
    assert a["new_pt"] == b["new_pt"]
    _same_dict(a["w"], b["w"])
    _same_dict(a["b"], b["b"])
    assert a["alpha"] == b["alpha"]
    sa, sb = a["rng"], b["rng"]
    assert sa[0] == sb[0] and np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]


@pytest.mark.parametrize("policy", [True, "zc", "copy"])
def test_host_resident_pipeline_on_bf16_maps_equals_widened_maps(policy):
    """prune_layers(from_host=...) with bf16 pinned maps against the same maps widened to fp32: identical masks, W
    and b, whatever the transfer plan (it may differ: a 16-bit map is half the DMA and fewer read requests)."""
    import cpb200
    from cpb200 import pruner

    eng = cpb200.Engine(nstreams=4)
    shapes = [cpb200.synth.LayerShape("a", 32, 24, 14, N=600, B=4, P=5), cpb200.synth.LayerShape("b", 48, 16, 28, N=800, B=4, P=5),
              cpb200.synth.LayerShape("c", 16, 16, 56, N=400, B=4, P=5), cpb200.synth.LayerShape("d", 64, 32, 7, N=600, B=4, P=5),
              cpb200.synth.LayerShape("e", 24, 8, 20, k=1, pad=0, N=400, B=4, P=5)]
    d16 = [cpb200.synth.make_problem_device(s, 40 + i, eng, pinned_host=True, dtype=torch.bfloat16)
           for i, s in enumerate(shapes)]
    d32 = []
    for d in d16:
        assert d["fmap"].dtype == torch.bfloat16 and d["fmap_host"].dtype == torch.bfloat16 and d["fmap_host"].is_pinned()
        w = dict(d, fmap=d["fmap"].float(), fmap_host=torch.empty(d["fmap_host"].shape, pin_memory=True))
        w["fmap_host"].copy_(d["fmap_host"].float())
        d32.append(w)
    ref = pruner.prune_layers(eng, shapes, d32, from_host=policy, to_host=True)
    torch.cuda.synchronize()
    got = pruner.prune_layers(eng, shapes, d16, from_host=policy, to_host=True)
    torch.cuda.synchronize()
    for a, b in zip(ref, got):
        assert np.array_equal(a.idxs, b.idxs) and a.alpha == b.alpha and a.nprobe == b.nprobe
        assert torch.equal(a.W, b.W) and torch.equal(a.b, b.b)
    eng.close()
