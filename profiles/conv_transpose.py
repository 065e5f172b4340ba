"""Patch gathers of transposed convolutions (synth.conv_transpose_layers: a 2-D U-Net's up-convolutions, a 3-D
nnU-Net-style decoder's ConvTranspose3d(k = s = 2), a DCGAN k = 4, s = 2, p = 1 layer) on every path, next to the conv
gather of the same map, and one prune_layers step over each network's transposed layers from HBM and from pinned host
maps.
    python profiles/conv_transpose.py [--reps R] [--launches L] [--steps S] [--warmup W] [--no-e2e] [--no-gathers]
Gathers at N = 5000, fp32 / bf16 / fp16 maps, paths alternating over the repetitions (CUDA events over L launches
each, median): channels first and last, in HBM and in pinned host memory (read in place).  TB/s is of the algorithmic
bytes: the map bytes the sampled rows really read (valid taps x c x element size, counted on the host from the points)
plus 4 N K written.  Every path is checked against the channels-first HBM gather's bits before it is timed.  The conv
gather (3 x 3, pad 1) of the same map runs in the same call, its bytes counted the same way (in-bounds taps), and a
device-to-device copy of the largest X gives the copy rate."""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import cpb200
from cpb200 import pruner
from profiles.conv3d import _kernel_of, _time
from profiles.conv_geometry import _pinned, card

_DT = (torch.float32, torch.bfloat16, torch.float16)


def _is3d(s):
    return hasattr(s, "kt")


def _valid_taps(s, pts, conv=False):
    """Taps of the sampled rows that read the map (each point's count times B), from the points on the host."""
    d3 = _is3d(s)
    axes = ((s.kt, s.pad_t, s.stride_t, s.dil_t, s.D),) if d3 else ()
    axes += ((s.kh, s.pad_h, s.stride_h, s.dil_h, s.H), (s.kw, s.pad_w, s.stride_w, s.dil_w, s.W))
    count = 1
    for p, (k, pad, st, dil, n) in zip(pts, axes):
        p = p.cpu().numpy()
        if conv:  # the conv window on the same map (k = 3, pad = 1, stride 1 on the input grid)
            h = p[..., None] - 1 + np.arange(3)
            ok = (h >= 0) & (h < n)
        else:
            _, ok = cpb200.synth._tr_axis_numpy(p, pad, st, dil, k, n)
        count = count * ok.sum(-1)
    return int(count.sum()) * s.B


def _conv_of(s):
    """The 3 x 3 (x 3), pad 1 conv on the transposed layer's input map: same c, same N, B and P."""
    if _is3d(s):
        return cpb200.synth.LayerShape3d(s.name + "/conv", s.c, s.c, s.D, s.H, N=s.N, B=s.B, P=s.P)
    return cpb200.synth.LayerShape(s.name + "/conv", s.c, s.c, s.H, N=s.N, B=s.B, P=s.P)


def gathers(eng, reps, launches):
    print("gathers, N = 5000, %d reps x %d launches, paths alternating; ms median (min-max), TB/s of valid-tap bytes "
          "read + 4NK written" % (reps, launches), flush=True)
    dev = eng.device
    kmax = 0
    for net, shapes in cpb200.synth.conv_transpose_layers().items():
        for s in shapes:
            d3 = _is3d(s)
            kmax = max(kmax, s.K)
            fn = eng.patch_gather3d if d3 else eng.patch_gather
            r = np.random.RandomState(2)
            out = (s.To, s.Ho, s.Wo) if d3 else (s.Ho, s.Wo)
            pts = [torch.as_tensor(r.randint(0, hi, (s.nbatch, s.P)).astype(np.int32), device=dev) for hi in out]
            sc = _conv_of(s)
            cpts = [torch.as_tensor(r.randint(0, hi, (s.nbatch, s.P)).astype(np.int32), device=dev)
                    for hi in ((sc.To, sc.Ho, sc.Wo) if d3 else (sc.Ho, sc.Wo))]
            vt, vc = _valid_taps(s, pts), _valid_taps(sc, cpts, conv=True)
            X = eng.empty(s.N, s.K, dtype=torch.float32)
            Xc = eng.empty(sc.N, sc.K, dtype=torch.float32)
            g = torch.Generator(device=dev)
            g.manual_seed(11)
            spatial = (s.D, s.H, s.W) if d3 else (s.H, s.W)
            cf, cl = ("ncdhw", "ndhwc") if d3 else ("nchw", "nhwc")
            for dt in _DT:
                first = torch.randn((s.nbatch * s.B, s.c) + spatial, generator=g, device=dev).to(dt)
                last = first.permute(0, *range(2, first.dim()), 1).contiguous()
                maps = {cf + "_hbm": (first, cf), cl + "_hbm": (last, cl), cf + "_host": (_pinned(first), cf),
                        cl + "_host": (_pinned(last), cl)}
                calls = {p: (lambda m=m, lay=lay: fn(m, *pts, s.B, s.P, layout=lay, out=X, **s.conv_args()))
                         for p, (m, lay) in maps.items()}
                want = fn(first, *pts, s.B, s.P, **s.conv_args())
                kern = {}
                for p, call in calls.items():
                    call()
                    torch.cuda.synchronize()
                    assert torch.equal(X, want), (s.name, dt, p)
                    kern[p] = _kernel_of(call)
                del want
                calls["conv_" + cl] = lambda: fn(last, *cpts, s.B, s.P, layout=cl, out=Xc, **sc.conv_args())
                calls["conv_" + cf] = lambda: fn(first, *cpts, s.B, s.P, layout=cf, out=Xc, **sc.conv_args())
                for p in ("conv_" + cl, "conv_" + cf):
                    calls[p]()
                    kern[p] = _kernel_of(calls[p])
                es = first.element_size()
                times = _time(calls, reps, launches)
                for p, ts in times.items():
                    ms = float(np.median(ts))
                    conv = p.startswith("conv_")
                    nbytes = (vc if conv else vt) * s.c * es + 4 * s.N * (sc.K if conv else s.K)
                    lines = ""
                    if p.endswith("_host"):
                        nl = pruner.zero_copy_lines(s, es, p[:-5])
                        lines = "  model %.3g lines, %.3g lines/s" % (nl, nl / (ms / 1e3))
                    print("  %-8s %-10s c %4d K %5d %-8s %-12s %-26s %8.3f ms (%.3f-%.3f) %6.2f TB/s%s" % (
                        net, s.name, s.c, sc.K if conv else s.K, str(dt)[6:], p, kern[p], ms, min(ts), max(ts),
                        nbytes / (ms / 1e3) / 1e12, lines), flush=True)
                del maps, calls, first, last
            del X, Xc
            torch.cuda.empty_cache()
    # the copy rate of the card: a device-to-device copy of the largest X
    a = eng.empty(5000, kmax, dtype=torch.float32)
    b = torch.empty_like(a)
    ts = _time({"copy": lambda: b.copy_(a)}, reps, launches)["copy"]
    ms = float(np.median(ts))
    print("  d2d copy of %.0f MB: %.3f ms, %.2f TB/s (read + write)" % (a.numel() * 4 / 1e6, ms,
                                                                         2 * a.numel() * 4 / (ms / 1e3) / 1e12))
    del a, b
    torch.cuda.empty_cache()


def e2e(eng, steps, warmup):
    for net, shapes in cpb200.synth.conv_transpose_layers().items():
        for dt in (torch.float32, torch.bfloat16):
            for hl in ("nchw", "nhwc"):
                datas = [cpb200.synth.make_problem_device(s, 500 + i, eng, pinned_host=True, host_layout=hl, dtype=dt)
                         for i, s in enumerate(shapes)]
                torch.cuda.synchronize()
                runs = {"hbm": False, "host_" + hl: True} if hl == "nchw" else {"host_" + hl: True}
                for label, fh in runs.items():
                    for _ in range(warmup):
                        pruner.prune_layers(eng, shapes, datas, from_host=fh)
                        torch.cuda.synchronize()
                    walls = []
                    for _ in range(steps):
                        t0 = time.perf_counter()
                        res = pruner.prune_layers(eng, shapes, datas, from_host=fh)
                        torch.cuda.synchronize()
                        walls.append(time.perf_counter() - t0)
                    plan = " ".join(pruner.h2d_plan(shapes, datas, True)) if fh else "-"
                    print("prune_layers %-8s %d layers, %-8s maps %-10s %8.1f ms/step (median of %d, %.1f-%.1f)  "
                          "plan %s  verdicts %s  kept %s" % (
                              net, len(shapes), str(dt)[6:], label, 1e3 * float(np.median(walls)), len(walls),
                              1e3 * min(walls), 1e3 * max(walls), plan,
                              ",".join(r.info["verdict"] for r in res), [int(r.idxs.sum()) for r in res]), flush=True)
                del datas, res
                torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--launches", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-gathers", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/conv_transpose.py measures on the GPU"
    print("card (name, power limit, max SM clock): %s" % card(), flush=True)
    eng = cpb200.Engine(nstreams=6)
    if not args.no_gathers:
        gathers(eng, args.reps, args.launches)
    if not args.no_e2e:
        e2e(eng, args.steps, args.warmup)
    print("card after: %s" % card(), flush=True)


if __name__ == "__main__":
    main()
