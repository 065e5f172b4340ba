"""The consumer input transform of Conv-BN-activation networks (cp_patch_gather_act) against today's relu gather: the
conv4_2 gather (c = 512, 28 x 28, 3 x 3, N = 5000) on every path, and one prune_layers step over
synth.resnet50_layers(bn=True) against synth.resnet50_layers().
    python profiles/conv_bn_act.py [--reps R] [--launches L] [--steps S] [--warmup W] [--no-e2e] [--no-gathers]
Gathers, fp32 and bf16 maps: relu (the relu flag's kernels), BN + ReLU and BN + SiLU (the fused kernels), paths and
transforms alternating over the repetitions (CUDA events over L launches each, median).  TB/s of 8 N K bytes (fp32:
the window read once, the row written once) or 6 N K (bf16).  Paths: NCHW and NHWC in HBM (NHWC: the TMA kernel, and
the SIMT kernel, which an X whose leading dimension is not a multiple of 4 selects), NCHW and NHWC in pinned host
memory read in place.  Every fused gather is checked against the numpy statement on a slice of rows first.
The e2e step: N = 5000 with B = 10, P = 50 (100 images per layer), maps in HBM and NHWC pinned host maps ('zc')."""
import argparse
import os
import re
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import cpb200
from cpb200 import pruner
from profiles.conv3d import _time
from profiles.conv_geometry import _pinned, card


def _kernel_of(call):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    names = [e.name.replace(" ", "") for e in prof.events() if "patch_gather" in e.name and e.device_type.name == "CUDA"]
    name = names[0] if names else "?"
    for k in ("patch_gather_nhwc_tma", "patch_gather_nhwc_host", "patch_gather_nhwc", "patch_gather_nchw"):
        if k in name:
            return k + ("+x" if re.search(r"[<,]true[,>]", name) else "")
    return name


def gathers(eng, reps, launches):
    s = cpb200.synth.LayerShape("conv4_2", 512, 512, 28, N=5000)
    dev = eng.device
    print("gathers at %s (c %d, %dx%d, k 3, N %d), %d reps x %d launches; ms median (min-max), TB/s of 8NK (fp32) / "
          "6NK (bf16)" % (s.name, s.c, s.H, s.W, s.N, reps, launches), flush=True)
    r = np.random.RandomState(3)
    rx = torch.as_tensor(r.randint(0, s.Ho, (s.nbatch, s.P)).astype(np.int32), device=dev)
    ry = torch.as_tensor(r.randint(0, s.Wo, (s.nbatch, s.P)).astype(np.int32), device=dev)
    sc, sh = (torch.as_tensor(v, device=dev) for v in cpb200.synth.bn_params(s.c, 3))
    X = eng.empty(s.N, s.K, dtype=torch.float32)
    Xs = eng.empty(s.N, s.K + 1, dtype=torch.float32)[:, :s.K]  # ldx % 4 != 0: the SIMT kernel
    g = torch.Generator(device=dev)
    g.manual_seed(5)
    for dt in (torch.float32, torch.bfloat16):
        first = torch.randn((s.nbatch * s.B, s.c, s.H, s.W), generator=g, device=dev).to(dt)
        last = first.permute(0, 2, 3, 1).contiguous()
        maps = {"nchw_hbm": (first, "nchw", X), "nhwc_tma": (last, "nhwc", X), "nhwc_simt": (last, "nhwc", Xs),
                "nchw_host": (_pinned(first), "nchw", X), "nhwc_host": (_pinned(last), "nhwc", X)}
        kws = {"relu": dict(relu=True), "bn_relu": dict(act="relu", in_scale=sc, in_shift=sh),
               "bn_silu": dict(act="silu", in_scale=sc, in_shift=sh)}
        # check the fused gathers against numpy on the first 40 rows (nbatch 1 of the points, B = 10: 4 points)
        fm = first[:s.B].float().cpu().numpy()
        for xf in ("bn_relu", "bn_silu"):
            want = cpb200.synth.gather_patches_numpy(fm, rx[:1].cpu().numpy(), ry[:1].cpu().numpy(), s.B, 3, 1, 1,
                                                     None, act=xf[3:], in_scale=sc.cpu().numpy(),
                                                     in_shift=sh.cpu().numpy()).reshape(-1, s.K)
            for p, (m, lay, out) in maps.items():
                eng.patch_gather(m, rx, ry, s.B, s.P, 3, 1, 1, layout=lay, out=out, **kws[xf])
                torch.cuda.synchronize()
                got = out[:want.shape[0]].cpu().numpy()
                if xf == "bn_relu":
                    assert np.array_equal(got.view(np.int32), want.view(np.int32)), (dt, p, xf)
                else:
                    assert np.abs(got - want).max() <= 1e-6 * max(1.0, np.abs(want).max()), (dt, p, xf)
        calls, kern = {}, {}
        for p, (m, lay, out) in maps.items():
            for xf, kw in kws.items():
                call = (lambda m=m, lay=lay, out=out, kw=kw: eng.patch_gather(m, rx, ry, s.B, s.P, 3, 1, 1, layout=lay,
                                                                               out=out, **kw))
                call()
                calls[(p, xf)] = call
                kern[(p, xf)] = _kernel_of(call)
        times = _time(calls, reps, launches)
        nbytes = (8 if dt == torch.float32 else 6) * s.N * s.K
        for p in maps:
            base = float(np.median(times[(p, "relu")]))
            for xf in kws:
                ts = times[(p, xf)]
                ms = float(np.median(ts))
                print("  %-8s %-9s %-8s %-26s %8.3f ms (%.3f-%.3f) %6.2f TB/s  %+6.1f %%" % (
                    str(dt)[6:], p, xf, kern[(p, xf)], ms, min(ts), max(ts), nbytes / (ms / 1e3) / 1e12,
                    100 * (ms / base - 1)), flush=True)
        del maps, calls, first, last
        torch.cuda.empty_cache()


def e2e(eng, steps, warmup):
    for bn in (False, True):
        shapes = cpb200.synth.resnet50_layers(N=5000, B=10, P=50, bn=bn)
        datas = [cpb200.synth.make_problem_device(s, 700 + i, eng, pinned_host=True, host_layout="nhwc")
                 for i, s in enumerate(shapes)]
        torch.cuda.synchronize()
        for label, fh in (("hbm", False), ("host_nhwc", "zc")):
            for _ in range(warmup):
                pruner.prune_layers(eng, shapes, datas, from_host=fh)
                torch.cuda.synchronize()
            walls = []
            for _ in range(steps):
                t0 = time.perf_counter()
                res = pruner.prune_layers(eng, shapes, datas, from_host=fh)
                torch.cuda.synchronize()
                walls.append(time.perf_counter() - t0)
            verdicts = {v: sum(r.info["verdict"] == v for r in res) for v in {r.info["verdict"] for r in res}}
            print("prune_layers resnet50%-8s %d layers, %-9s %8.1f ms/step (median of %d, %.1f-%.1f)  verdicts %s" % (
                "(bn)" if bn else "", len(shapes), label, 1e3 * float(np.median(walls)), len(walls), 1e3 * min(walls),
                1e3 * max(walls), verdicts), flush=True)
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
    assert torch.cuda.is_available(), "profiles/conv_bn_act.py measures on the GPU"
    print("card (name, power limit, max SM clock): %s" % card(), flush=True)
    eng = cpb200.Engine(nstreams=6)
    if not args.no_gathers:
        gathers(eng, args.reps, args.launches)
    if not args.no_e2e:
        e2e(eng, args.steps, args.warmup)
    print("card after: %s" % card(), flush=True)


if __name__ == "__main__":
    main()
