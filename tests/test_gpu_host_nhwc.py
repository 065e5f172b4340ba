"""GPU: the in-place reader of channels-last (NHWC) feature maps in pinned host memory.  It must produce the bits the
HBM gathers produce for the same values (NHWC by TMA or SIMT, and NCHW), be the kernel that actually ran, refuse what
the HBM NHWC path refuses, and leave the host-resident pruning pipeline's results unchanged."""
import numpy as np
import pytest

import gather_checks as GC

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

DTYPES = pytest.mark.parametrize("dtype", list(GC.FMAP_DTYPES))
# (k, pad, stride)
WINDOWS = [(1, 0, 1), (1, 0, 2), (3, 1, 1), (3, 1, 2), (3, 0, 1), (5, 2, 1), (5, 2, 2)]
CHANNELS = [3, 5, 12, 16, 24, 64, 512, 2048]


def _points(nb, Ho, device):
    """Every corner and border of the output map, plus the centre, in varying order per batch."""
    pts = [(0, 0), (0, Ho - 1), (Ho - 1, 0), (Ho - 1, Ho - 1), (Ho // 2, Ho // 2), (1 % Ho, Ho - 1), (Ho - 1, 1 % Ho),
           (0, Ho // 2), (Ho // 2, 0), (Ho - 1, Ho // 2), (Ho // 2, Ho - 1)]
    rx = torch.tensor([[p[0] for p in pts]] * nb, dtype=torch.int32, device=device)
    ry = torch.tensor([[p[1] for p in pts]] * nb, dtype=torch.int32, device=device)
    rx[1] = rx[1].flip(0)
    return rx, ry, len(pts)


@DTYPES
@pytest.mark.parametrize("c", CHANNELS)
@pytest.mark.parametrize("k,pad,stride", WINDOWS)
def test_host_nhwc_gather_equals_hbm_gathers(engine, dtype, c, k, pad, stride):
    dev = engine.device
    H, B, nb = 9, 3, 4
    nchw = GC.special_map((nb * B, c, H, H), dtype, c * 31 + k * 7 + stride + pad, dev)
    nhwc = nchw.permute(0, 2, 3, 1).contiguous()
    host = GC.pinned(nhwc)
    rx, ry, P = _points(nb, (H + 2 * pad - k) // stride + 1, dev)
    for relu in (False, True):
        a = engine.patch_gather(nchw, rx, ry, B, P, k, pad, stride, relu=relu)
        b = engine.patch_gather(nhwc, rx, ry, B, P, k, pad, stride, relu=relu, layout="nhwc")
        got = engine.patch_gather(host, rx, ry, B, P, k, pad, stride, relu=relu, layout="nhwc")
        torch.cuda.synchronize()
        GC.assert_same_bits(b, a)
        GC.assert_same_bits(got, b)
        if relu:
            assert not bool(torch.isnan(got).any())  # fmaxf(NaN, 0) = 0, as in the HBM kernels


def _conv4_2():
    import cpb200

    return [s for s in cpb200.synth.vgg16_layers() if s.name == "conv4_2"][0]


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_host_nhwc_gather_at_conv4_2_size(engine, dtype):
    """N = 5000 rows of a 512-channel, 28 x 28 map: the persistent grid's tails, against the TMA gather in HBM; and
    the same gather into a row slice of a wider buffer (ldx > K, an offset base), leaving the rest of the buffer
    alone."""
    s = _conv4_2()
    dev = engine.device
    g = torch.Generator(device=dev)
    g.manual_seed(5)
    nhwc = torch.randn((s.nbatch * s.B, s.H, s.W, s.c), generator=g, device=dev).to(GC.FMAP_DTYPES[dtype])
    host = GC.pinned(nhwc)
    r = np.random.RandomState(3)
    rx = torch.as_tensor(r.randint(0, s.Ho, (s.nbatch, s.P)).astype(np.int32), device=dev)
    ry = torch.as_tensor(r.randint(0, s.Ho, (s.nbatch, s.P)).astype(np.int32), device=dev)
    want = engine.patch_gather(nhwc, rx, ry, s.B, s.P, s.k, s.pad, s.stride, layout="nhwc")
    got = engine.patch_gather(host, rx, ry, s.B, s.P, s.k, s.pad, s.stride, layout="nhwc")
    torch.cuda.synchronize()
    GC.assert_same_bits(got, want)
    del got
    wide = torch.full((s.N, s.K + 40), 7.0, device=dev)
    out = wide[:, 8:8 + s.K]
    engine.patch_gather(host, rx, ry, s.B, s.P, s.k, s.pad, s.stride, layout="nhwc", out=out)
    torch.cuda.synchronize()
    GC.assert_same_bits(out.contiguous(), want)
    assert bool((wide[:, :8] == 7.0).all()) and bool((wide[:, 8 + s.K:] == 7.0).all())


PATH_SHAPES = [(3, 3), (5, 1), (12, 5), (16, 3), (24, 3), (64, 1), (512, 3), (2048, 1), (2048, 3)]


def test_host_nhwc_reader_is_what_runs(engine):
    """Every NHWC host map -- aligned or not, any dtype -- must take the host reader, not the HBM SIMT kernel (which
    would pass the bit checks above).  One profiler session, every case launched REPEAT times: in a process that has
    profiled before, the profiler may lose an activity record, so the check does not rest on any single launch.  No
    other gather kernel may appear, and each dtype must show its launches, but for at most LOST records."""
    from torch.profiler import ProfilerActivity, profile

    dev = engine.device
    H, B, nb = 7, 2, 2
    rx, ry, P = _points(nb, H, dev)
    runs = []
    for dtype in GC.FMAP_DTYPES:
        for c, k in PATH_SHAPES:
            host = GC.pinned(GC.special_map((nb * B, H, H, c), dtype, c + k, dev))
            out = engine.patch_gather(host, rx, ry, B, P, k, k // 2, 1, layout="nhwc")  # warm-up (module load)
            runs.append((dtype, c, k, host, out))
    torch.cuda.synchronize()
    REPEAT, LOST = 3, 2
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for dtype, c, k, host, out in runs:
            for _ in range(REPEAT):
                engine.patch_gather(host, rx, ry, B, P, k, k // 2, 1, layout="nhwc", out=out)
        torch.cuda.synchronize()
    kernels = [e.name for e in prof.events() if "patch_gather" in e.name and e.device_type.name == "CUDA"]
    assert kernels and all("patch_gather_nhwc_host" in n for n in kernels), sorted(set(kernels))
    ctype = {"fp32": "float", "bf16": "bfloat16", "fp16": "half"}
    for dtype in GC.FMAP_DTYPES:
        seen = sum(1 for n in kernels if "%s>" % ctype[dtype] in n or "%s >" % ctype[dtype] in n)
        want = REPEAT * sum(1 for r in runs if r[0] == dtype)
        assert want - LOST <= seen <= want, (dtype, seen, want, sorted(set(kernels)))


def test_oversized_window_on_nhwc_host_map_is_refused(engine):
    """k = 11 is refused with CP_ERR_INVALID and a message, as it is for an NHWC map in HBM off the TMA path."""
    ffi, lib = engine.ffi, engine.lib
    dev = engine.device
    H, B, nb, k = 13, 2, 1, 11
    host = GC.pinned(torch.zeros((nb * B, H, H, 3), device=dev))
    rx = torch.zeros((nb, 1), dtype=torch.int32, device=dev)
    X = torch.empty((nb * B, 3 * k * k), device=dev)
    rc = lib.cp_patch_gather_typed(engine.h, ffi.cast("const void*", host.data_ptr()), lib.CP_F32, nb, B, 3, H, H, 1,
                                   ffi.cast("const int32_t*", rx.data_ptr()), ffi.cast("const int32_t*", rx.data_ptr()),
                                   1, k, 5, 1, 1, ffi.cast("float*", X.data_ptr()), 3 * k * k, ffi.NULL)
    assert rc == lib.CP_ERR_INVALID
    assert b"kernel_size 11" in ffi.string(lib.cp_last_error())


def _shapes():
    import cpb200

    S = cpb200.synth.LayerShape
    return [S("a", 32, 24, 14, N=600, B=4, P=5), S("b", 48, 16, 28, N=800, B=4, P=5),
            S("c", 16, 16, 56, N=400, B=4, P=5), S("d", 64, 32, 7, N=600, B=4, P=5),
            S("e", 24, 8, 20, k=1, pad=0, N=400, B=4, P=5), S("f", 12, 8, 9, N=400, B=4, P=5),
            S("g", 128, 16, 4, N=4000, B=2, P=100)]  # a 4 x 4 map sampled 4000 times: DMA in either layout


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("policy", [True, "zc", "copy"])
def test_host_resident_pipeline_on_nhwc_maps_equals_nchw_maps(dtype, policy):
    """prune_layers(from_host=...) on channels-last pinned maps against the same values in NCHW pinned maps: identical
    masks, alpha, probe counts, W and b, whatever the transfer plan (it may differ between the layouts)."""
    import cpb200
    from cpb200 import pruner

    eng = cpb200.Engine(nstreams=4)
    shapes = _shapes()
    dt = None if dtype == "fp32" else GC.FMAP_DTYPES[dtype]
    dn = [cpb200.synth.make_problem_device(s, 70 + i, eng, pinned_host=True, dtype=dt) for i, s in enumerate(shapes)]
    dh = [cpb200.synth.make_problem_device(s, 70 + i, eng, pinned_host=True, dtype=dt, host_layout="nhwc")
          for i, s in enumerate(shapes)]
    for a, b in zip(dn, dh):
        assert "host_layout" not in a and b["host_layout"] == "nhwc" and b["fmap_host"].is_pinned()
        assert torch.equal(a["fmap_host"].permute(0, 2, 3, 1), b["fmap_host"])
    if policy is True:  # the densely sampled map goes by DMA, whatever the layout; the largest is read in place
        for d in (dn, dh):
            plan = pruner.h2d_plan(shapes, d, True)
            assert plan[-1] == "dma" and plan[2] == "zc", plan
    ref = pruner.prune_layers(eng, shapes, dn, from_host=policy, to_host=True)
    torch.cuda.synchronize()
    ref = [(r.idxs.copy(), r.alpha, r.nprobe, r.W.clone(), r.b.clone()) for r in ref]
    got = pruner.prune_layers(eng, shapes, dh, from_host=policy, to_host=True)
    torch.cuda.synchronize()
    for (idxs, alpha, nprobe, W, b), r in zip(ref, got):
        assert np.array_equal(idxs, r.idxs) and alpha == r.alpha and nprobe == r.nprobe
        assert torch.equal(W, r.W) and torch.equal(b, r.b)
    eng.close()
