"""Patch gathers of dilated and rectangular convolutions against their undilated, square twins, and one prune_layers
step over DeepLabV3-ResNet50's dilated 3x3 convolutions against the same layers undilated.
    python profiles/conv_geometry.py [--reps R] [--launches L] [--steps S] [--warmup W] [--no-e2e]
Gathers at N = 5000 (B = 10 images, P = 10 points, 50 batches), fp32 and bf16 maps, three paths alternating over the
repetitions (CUDA events over L launches each): NHWC in HBM (the TMA kernel where the window allows it, else the
SIMT kernel; the 'kernel' column says which), NCHW in HBM, NHWC in pinned host memory (the in-place reader).
GB/s is of the algorithmic bytes: 8 N K (fp32 map) or 6 N K (16-bit map), K = c kh kw -- each window read once, the
fp32 row written once.  Every path is checked against the NCHW gather's bits before it is timed."""
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import cpb200
from cpb200 import pruner

L = cpb200.synth.LayerShape
# name, c, H, kernel, pad, dilation -- DeepLabV3-ResNet50 at a 224 input (layer3 d = 2, layer4 d = 4 and an ASPP
# branch, on 28 x 28 maps), the undilated 3x3 twins, Inception-v3 Mixed_6 (17 x 17) and Mixed_7 (8 x 8)
SHAPES = [("deeplab_layer3_3x3_d2", 256, 28, 3, 2, 2), ("twin_layer3_3x3", 256, 28, 3, 1, 1),
          ("deeplab_layer4_3x3_d4", 512, 28, 3, 4, 4), ("twin_layer4_3x3", 512, 28, 3, 1, 1),
          ("inception_mixed6_1x7", 192, 17, (1, 7), (0, 3), 1), ("inception_mixed6_7x1", 192, 17, (7, 1), (3, 0), 1),
          ("inception_mixed7_1x3", 384, 8, (1, 3), (0, 1), 1), ("inception_mixed7_3x1", 384, 8, (3, 1), (1, 0), 1),
          ("aspp_3x3_d12", 2048, 28, 3, 12, 12)]
PATHS = (("nhwc", False), ("nchw", False), ("nhwc", True))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or "nvidia-smi: no answer"
    except Exception as e:  # pragma: no cover
        return "nvidia-smi unavailable (%s); %s" % (e, torch.cuda.get_device_name())


def _pinned(t):
    h = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
    h.copy_(t)
    return h


def _kernel_of(eng, m, rx, ry, s, layout):
    """Name of the gather kernel one launch runs (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.patch_gather(m, rx, ry, s.B, s.P, layout=layout, **s.conv_args())
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if "patch_gather" in e.name and e.device_type.name == "CUDA"]
    name = names[0] if names else "?"
    for k in ("patch_gather_nhwc_tma", "patch_gather_nhwc_host", "patch_gather_nhwc", "patch_gather_nchw"):
        if k in name:
            return k
    return name


def gathers(eng, reps, launches):
    print("gathers, N = 5000, %d reps x %d launches, paths alternating; ms median (min-max), GB/s of 8NK / 6NK"
          % (reps, launches), flush=True)
    for name, c, H, k, pad, dil in SHAPES:
        s = L(name, c, c, H, k=k, pad=pad, dilation=dil, N=5000)
        r = np.random.RandomState(2)
        rx = torch.as_tensor(r.randint(0, s.Ho, (s.nbatch, s.P)).astype(np.int32), device=eng.device)
        ry = torch.as_tensor(r.randint(0, s.Wo, (s.nbatch, s.P)).astype(np.int32), device=eng.device)
        X = eng.empty(s.N, s.K, dtype=torch.float32)
        g = torch.Generator(device=eng.device)
        g.manual_seed(11)
        for dt in (torch.float32, torch.bfloat16):
            nchw = torch.randn((s.nbatch * s.B, s.c, s.H, s.W), generator=g, device=eng.device).to(dt)
            nhwc = nchw.permute(0, 2, 3, 1).contiguous()
            maps = {("nhwc", False): nhwc, ("nchw", False): nchw, ("nhwc", True): _pinned(nhwc)}
            want = eng.patch_gather(nchw, rx, ry, s.B, s.P, **s.conv_args())
            kern = {}
            for (lay, host), m in maps.items():  # warm-up, and every path must give the NCHW gather's bits
                eng.patch_gather(m, rx, ry, s.B, s.P, layout=lay, out=X, **s.conv_args())
                torch.cuda.synchronize()
                assert torch.equal(X, want), (name, dt, lay, host)
                kern[(lay, host)] = _kernel_of(eng, m, rx, ry, s, lay)
            del want
            nbytes = (8 if dt == torch.float32 else 6) * s.N * s.K
            times = {p: [] for p in maps}
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for _ in range(reps):
                for (lay, host), m in maps.items():
                    a.record()
                    for _ in range(launches):
                        eng.patch_gather(m, rx, ry, s.B, s.P, layout=lay, out=X, **s.conv_args())
                    b.record()
                    b.synchronize()
                    times[(lay, host)].append(a.elapsed_time(b) / launches)
            for (lay, host), ts in times.items():
                ms = float(np.median(ts))
                print("  %-22s K %5d %-8s %-4s %-4s %-23s %8.3f ms (%.3f-%.3f)  %7.1f GB/s" % (
                    name, s.K, str(dt).replace("torch.", ""), lay, "host" if host else "hbm", kern[(lay, host)], ms,
                    min(ts), max(ts), nbytes / (ms / 1e3) / 1e9), flush=True)
            del maps, nchw, nhwc
        del X
        torch.cuda.empty_cache()


def _deeplab(dilated):
    """The 3x3 convolutions of DeepLabV3-ResNet50's layer3 (6 blocks, c = 256, d = 2) and layer4 (3 blocks, c = 512,
    d = 4) at a 224 input (28 x 28 maps), N = 5000; undilated: the same layers with d = 1."""
    out = []
    for i in range(6):
        out.append(L("layer3.%d.conv2" % i, 256, 256, 28, k=3, pad=2 if dilated else 1, dilation=2 if dilated else 1))
    for i in range(3):
        out.append(L("layer4.%d.conv2" % i, 512, 512, 28, k=3, pad=4 if dilated else 1, dilation=4 if dilated else 1))
    return out


def e2e(eng, steps, warmup):
    sets = {}
    for label, dilated in (("dilated", True), ("undilated", False)):
        shapes = _deeplab(dilated)
        datas = [cpb200.synth.make_problem_device(s, 500 + i, eng) for i, s in enumerate(shapes)]
        sets[label] = (shapes, datas)
    torch.cuda.synchronize()
    for shapes, datas in sets.values():
        for _ in range(warmup):
            pruner.prune_layers(eng, shapes, datas)
            torch.cuda.synchronize()
    walls = {label: [] for label in sets}
    for _ in range(steps):  # alternating
        for label, (shapes, datas) in sets.items():
            t0 = time.perf_counter()
            pruner.prune_layers(eng, shapes, datas)
            torch.cuda.synchronize()
            walls[label].append(time.perf_counter() - t0)
    for label, w in walls.items():
        ms = 1e3 * float(np.median(w))
        print("prune_layers, DeepLabV3-ResNet50 layer3/layer4 3x3 convs (9 layers, N = 5000, maps in HBM, NCHW) "
              "%-9s %.1f ms/step (median of %d, %.1f-%.1f)" % (label, ms, len(w), 1e3 * min(w), 1e3 * max(w)),
              flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--launches", type=int, default=5)
    ap.add_argument("--steps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-e2e", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/conv_geometry.py measures on the GPU"
    print("card (name, power limit, max SM clock): %s" % card(), flush=True)
    eng = cpb200.Engine(nstreams=9)
    gathers(eng, args.reps, args.launches)
    if not args.no_e2e:
        e2e(eng, args.steps, args.warmup)
    print("card after: %s" % card(), flush=True)


if __name__ == "__main__":
    main()
