"""Patch gathers of Conv3d layers (torchvision r3d_18 on a 16 x 112 x 112 clip) on every path, next to the 2-D conv4_2
gather, and one prune_layers step over r3d_18's 3x3x3 convolutions with maps in HBM and in pinned host memory.
    python profiles/conv3d.py [--reps R] [--launches L] [--steps S] [--warmup W] [--no-e2e] [--no-gathers]
Gathers at N = 5000 (B = 10 clips, P = 50 points, 10 batches), fp32 and bf16 maps, paths alternating over the
repetitions (CUDA events over L launches each): NDHWC in HBM (the 5-D TMA kernel), NCDHW in HBM, NDHWC and NCDHW in
pinned host memory (in place).  GB/s is of the algorithmic bytes 8 N K (fp32 map) or 6 N K (16-bit map), K = c kt kh
kw; for the host paths the plan's line model (pruner.zero_copy_lines) and lines/s.  Every path is checked against the
NCDHW gather's bits before it is timed.  conv4_2 (VGG-16, 512 x 28 x 28, 3 x 3) runs the 2-D NHWC TMA and NCHW paths
with the same N, B and P."""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import cpb200
from cpb200 import pruner
from profiles.conv_geometry import _pinned, card

L3 = cpb200.synth.LayerShape3d
# the distinct 3x3x3 shapes of r3d_18's layer1-layer4 (stride-1 convs; the strided first convs read the maps above)
SHAPES = [("layer1_64x16x56", 64, 16, 56), ("layer2_128x8x28", 128, 8, 28), ("layer3_256x4x14", 256, 4, 14),
          ("layer4_512x2x7", 512, 2, 7)]


def _kernel_of(call):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if "patch_gather" in e.name and e.device_type.name == "CUDA"]
    name = names[0] if names else "?"
    for k in ("patch_gather_ndhwc_tma", "patch_gather_ndhwc_host", "patch_gather_ndhwc", "patch_gather_ncdhw",
              "patch_gather_nhwc_tma", "patch_gather_nchw"):
        if k in name:
            return k
    return name


def _time(calls, reps, launches):
    times = {p: [] for p in calls}
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(reps):
        for p, call in calls.items():
            a.record()
            for _ in range(launches):
                call()
            b.record()
            b.synchronize()
            times[p].append(a.elapsed_time(b) / launches)
    return times


def _report(name, K, dt, times, kern, nbytes, lines=None):
    for p, ts in times.items():
        ms = float(np.median(ts))
        extra = "  %.3g lines, %.3g lines/s" % (lines[p], lines[p] / (ms / 1e3)) if lines and p in lines else ""
        print("  %-18s K %5d %-8s %-11s %-24s %8.3f ms (%.3f-%.3f)  %7.1f GB/s%s" % (
            name, K, str(dt).replace("torch.", ""), p, kern[p], ms, min(ts), max(ts), nbytes / (ms / 1e3) / 1e9, extra),
            flush=True)


def gathers(eng, reps, launches):
    print("gathers, N = 5000, %d reps x %d launches, paths alternating; ms median (min-max), GB/s of 8NK / 6NK"
          % (reps, launches), flush=True)
    dev = eng.device
    for name, c, D, H in SHAPES:
        s = L3(name, c, c, D, H, N=5000, B=10, P=50)
        r = np.random.RandomState(2)
        pts = [torch.as_tensor(r.randint(0, hi, (s.nbatch, s.P)).astype(np.int32), device=dev) for hi in (s.To, s.Ho,
                                                                                                           s.Wo)]
        X = eng.empty(s.N, s.K, dtype=torch.float32)
        g = torch.Generator(device=dev)
        g.manual_seed(11)
        for dt in (torch.float32, torch.bfloat16):
            ncdhw = torch.randn((s.nbatch * s.B, s.c, s.D, s.H, s.W), generator=g, device=dev).to(dt)
            ndhwc = ncdhw.permute(0, 2, 3, 4, 1).contiguous()
            maps = {"ndhwc_hbm": (ndhwc, "ndhwc"), "ncdhw_hbm": (ncdhw, "ncdhw"),
                    "ndhwc_host": (_pinned(ndhwc), "ndhwc"), "ncdhw_host": (_pinned(ncdhw), "ncdhw")}
            calls = {p: (lambda m=m, lay=lay: eng.patch_gather3d(m, *pts, s.B, s.P, layout=lay, out=X, **s.conv_args()))
                     for p, (m, lay) in maps.items()}
            want = eng.patch_gather3d(ncdhw, *pts, s.B, s.P, **s.conv_args())
            kern = {}
            for p, call in calls.items():
                call()
                torch.cuda.synchronize()
                assert torch.equal(X, want), (name, dt, p)
                kern[p] = _kernel_of(call)
            del want
            es = ncdhw.element_size()
            lines = {"ndhwc_host": pruner.zero_copy_lines(s, es, "ndhwc"),
                     "ncdhw_host": pruner.zero_copy_lines(s, es, "ncdhw")}
            _report(name, s.K, dt, _time(calls, reps, launches), kern, (8 if es == 4 else 6) * s.N * s.K, lines)
            del maps, calls, ncdhw, ndhwc
        del X
        torch.cuda.empty_cache()
    # the 2-D reference point of the same call: VGG-16 conv4_2
    s = cpb200.synth.LayerShape("conv4_2", 512, 512, 28, N=5000, B=10, P=50)
    r = np.random.RandomState(2)
    rx, ry = (torch.as_tensor(r.randint(0, hi, (s.nbatch, s.P)).astype(np.int32), device=dev) for hi in (s.Ho, s.Wo))
    X = eng.empty(s.N, s.K, dtype=torch.float32)
    for dt in (torch.float32, torch.bfloat16):
        nchw = torch.randn((s.nbatch * s.B, s.c, s.H, s.W), device=dev).to(dt)
        maps = {"nhwc_hbm": (nchw.permute(0, 2, 3, 1).contiguous(), "nhwc"), "nchw_hbm": (nchw, "nchw")}
        calls = {p: (lambda m=m, lay=lay: eng.patch_gather(m, rx, ry, s.B, s.P, layout=lay, out=X, **s.conv_args()))
                 for p, (m, lay) in maps.items()}
        kern = {}
        for p, call in calls.items():
            call()
            kern[p] = _kernel_of(call)
        _report("conv4_2 (2-D)", s.K, dt, _time(calls, reps, launches), kern,
                (8 if nchw.element_size() == 4 else 6) * s.N * s.K)
        del maps, calls, nchw
    del X
    torch.cuda.empty_cache()


def e2e(eng, steps, warmup):
    # The layers with c >= 256 inputs are left out: at N = 5000 their least squares has more columns (K' = 27 c')
    # than rows, and their small output volumes (784 and 98 points per clip) make 50 samples per clip repeat rows, so
    # the minimum-norm solve is rank deficient and goes through the truncated SVD (engine.reconstruct_truncated).  On
    # an H100 a step with layer3 did not finish within 7 minutes; layer4's K' ~ 13000 exceeds cp_svd_jacobi's
    # m <= 12800.  The nine layers with c <= 128 (K' < N) remain.
    shapes = [s for s in cpb200.synth.r3d18_layers() if s.c <= 128]
    datas = [cpb200.synth.make_problem_device(s, 700 + i, eng, pinned_host=True) for i, s in enumerate(shapes)]
    # the same maps channels-last on the host
    datas_nd = []
    for d in datas:
        e = dict(d)
        e["fmap_host"] = _pinned(d["fmap_host"].permute(0, 2, 3, 4, 1))
        e["host_layout"] = "ndhwc"
        datas_nd.append(e)
    torch.cuda.synchronize()
    print("r3d_18: %d layers (c <= 128), N = 5000 (B = 10, P = 50), fp32 maps %.1f GB" % (
        len(shapes), sum(d["fmap"].numel() for d in datas) * 4 / 1e9), flush=True)
    runs = {"hbm": (datas, False), "host_ncdhw": (datas, True), "host_ndhwc": (datas_nd, True)}
    for label, (ds, fh) in runs.items():
        if fh:
            print("  plan %-10s %s" % (label, " ".join(pruner.h2d_plan(shapes, ds, True))), flush=True)
    ref = None
    for label, (ds, fh) in runs.items():
        for _ in range(warmup):
            pruner.prune_layers(eng, shapes, ds, from_host=fh)
            torch.cuda.synchronize()
    walls = {label: [] for label in runs}
    for _ in range(steps):  # alternating
        for label, (ds, fh) in runs.items():
            t0 = time.perf_counter()
            res = pruner.prune_layers(eng, shapes, ds, from_host=fh)
            torch.cuda.synchronize()
            walls[label].append(time.perf_counter() - t0)
            masks = [r.idxs for r in res]
            if ref is None:
                ref = masks
            assert all(np.array_equal(a, b) for a, b in zip(ref, masks)), label
    for label, w in walls.items():
        ms = 1e3 * float(np.median(w))
        print("prune_layers, r3d_18 3x3x3 convs (9 layers, c <= 128), maps %-10s %.1f ms/step (median of %d, %.1f-%.1f)"
              % (label, ms, len(w), 1e3 * min(w), 1e3 * max(w)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--launches", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-gathers", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/conv3d.py measures on the GPU"
    print("card (name, power limit, max SM clock): %s" % card(), flush=True)
    eng = cpb200.Engine(nstreams=9)
    if not args.no_gathers:
        gathers(eng, args.reps, args.launches)
    if not args.no_e2e:
        e2e(eng, args.steps, args.warmup)
    print("card after: %s" % card(), flush=True)


if __name__ == "__main__":
    main()
