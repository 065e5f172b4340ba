"""Channels-last (NHWC) against NCHW feature maps in pinned host memory: the in-place reader alone, and one VGG-16 step
of prune_layers(from_host=True, to_host=True).
    python profiles/host_nhwc.py [--reps R] [--launches L] [--steps S] [--warmup W] [--no-e2e]
Reader: conv2_2, conv3_2, conv4_2 and conv5_1 at N = 5000, fp32 and bf16, the two layouts alternating over repetitions
(CUDA events over L launches).  Lines are the plan's model (pruner.zero_copy_lines) of each layout; window bytes are
the in-bounds taps of the drawn windows (c elements each), exactly counted.  NHWC lines/s is the rate the plan's
ZC_NHWC_LINES_PER_S states.
End to end: never more than one set of fp32 maps pinned at a time (18 GB); the bf16 sets alternate in one process."""
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

LAYERS = ("conv2_2", "conv3_2", "conv4_2", "conv5_1")


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


def window_bytes(s, rx, ry, esize):
    """Bytes of the in-bounds taps of every window (each tap is c elements in either layout)."""
    k = torch.arange(s.k, device=rx.device)
    y = (s.stride * rx.reshape(-1, 1) - s.pad + k)
    x = (s.stride * ry.reshape(-1, 1) - s.pad + k)
    ny = ((y >= 0) & (y < s.H)).sum(1)
    nx = ((x >= 0) & (x < s.W)).sum(1)
    return int((ny * nx).sum()) * s.B * s.c * esize


def reader(eng, reps, launches):
    by_name = {s.name: s for s in cpb200.synth.vgg16_layers()}
    print("reader alone, N = 5000, %d reps x %d launches, layouts alternating; ms median (min-max)" % (reps, launches))
    rates = []
    for name in LAYERS:
        s = by_name[name]
        g = torch.Generator(device=eng.device)
        g.manual_seed(11)
        r = np.random.RandomState(2)
        rx = torch.as_tensor(r.randint(0, s.Ho, (s.nbatch, s.P)).astype(np.int32), device=eng.device)
        ry = torch.as_tensor(r.randint(0, s.Ho, (s.nbatch, s.P)).astype(np.int32), device=eng.device)
        X = eng.empty(s.N, s.K, dtype=torch.float32)
        for dt in (torch.float32, torch.bfloat16):
            dev_map = torch.randn((s.nbatch * s.B, s.c, s.H, s.W), generator=g, device=eng.device).to(dt)
            maps = {"nchw": _pinned(dev_map), "nhwc": _pinned(dev_map.permute(0, 2, 3, 1))}
            want = eng.patch_gather(dev_map, rx, ry, s.B, s.P, s.k, s.pad, s.stride)
            del dev_map
            for lay, m in maps.items():  # warm-up, and both readers must give the HBM gather's bits
                eng.patch_gather(m, rx, ry, s.B, s.P, s.k, s.pad, s.stride, layout=lay, out=X)
                torch.cuda.synchronize()
                assert torch.equal(X, want), (name, dt, lay)
            del want
            es = maps["nchw"].element_size()
            wb = window_bytes(s, rx, ry, es)
            times = {lay: [] for lay in maps}
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for _ in range(reps):
                for lay, m in maps.items():
                    a.record()
                    for _ in range(launches):
                        eng.patch_gather(m, rx, ry, s.B, s.P, s.k, s.pad, s.stride, layout=lay, out=X)
                    b.record()
                    b.synchronize()
                    times[lay].append(a.elapsed_time(b) / launches)
            for lay, ts in times.items():
                ms = float(np.median(ts))
                lines = pruner.zero_copy_lines(s, es, lay)
                print("  %-8s %-5s %-4s %8.3f ms (%.3f-%.3f)  %5.2f M lines  %6.3g lines/s  %5.1f GB/s of %6.1f MB "
                      "window bytes" % (name, str(dt).replace("torch.", ""), lay, ms, min(ts), max(ts), lines / 1e6,
                                        lines / (ms / 1e3), wb / (ms / 1e3) / 1e9, wb / 1e6), flush=True)
                if lay == "nhwc":
                    rates.append(lines / (ms / 1e3))
            del maps
        del X
        torch.cuda.empty_cache()
    print("NHWC model lines/s over the %d cases: min %.3g, median %.3g" % (len(rates), min(rates),
                                                                          float(np.median(rates))), flush=True)


def _datas(eng, dtype, host_layout):
    datas = []
    for i, s in enumerate(cpb200.synth.vgg16_layers()):
        d = cpb200.synth.make_problem_device(s, 1000 + i, eng, pinned_host=True, dtype=dtype, host_layout=host_layout)
        del d["fmap"]  # the maps live in pinned host memory only
        datas.append(d)
    torch.cuda.synchronize()
    return datas


def _steps(eng, shapes, datas, n):
    walls = []
    for _ in range(n):
        t0 = time.perf_counter()
        pruner.prune_layers(eng, shapes, datas, from_host=True, to_host=True)
        torch.cuda.synchronize()
        walls.append(time.perf_counter() - t0)
    return walls


def _report(shapes, datas, label, walls):
    plan = pruner.h2d_plan(shapes, datas, True)
    es = datas[0]["fmap_host"].element_size()
    lay = datas[0].get("host_layout", "nchw")
    dma = sum(int(d["fmap_host"].numel()) * es for d, p in zip(datas, plan) if p == "dma")
    lines = sum(pruner.zero_copy_lines(s, es, lay) for s, p in zip(shapes, plan) if p == "zc")
    ms = 1e3 * float(np.median(walls))
    print("e2e VGG-16 %-10s plan %s  DMA %.2f GB + %.2f M zero-copy lines per step  %.1f ms/step (median of %d, "
          "%.1f-%.1f)  %.1f layers/s" % (label, "".join("D" if p == "dma" else "z" for p in plan), dma / 1e9,
                                          lines / 1e6, ms, len(walls), 1e3 * min(walls), 1e3 * max(walls),
                                          len(shapes) / (ms / 1e3)), flush=True)


def e2e(eng, steps, warmup):
    shapes = cpb200.synth.vgg16_layers()
    for lay in ("nchw", "nhwc"):  # one fp32 set at a time
        datas = _datas(eng, torch.float32, lay)
        _steps(eng, shapes, datas, warmup)
        _report(shapes, datas, "fp32 " + lay, _steps(eng, shapes, datas, steps))
        del datas
        torch.cuda.empty_cache()
    sets = {lay: _datas(eng, torch.bfloat16, lay) for lay in ("nchw", "nhwc")}
    for lay, datas in sets.items():
        _steps(eng, shapes, datas, warmup)
    walls = {lay: [] for lay in sets}
    for _ in range(steps):  # alternating
        for lay, datas in sets.items():
            walls[lay] += _steps(eng, shapes, datas, 1)
    for lay, datas in sets.items():
        _report(shapes, datas, "bf16 " + lay, walls[lay])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--launches", type=int, default=5)
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-e2e", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/host_nhwc.py measures on the GPU"
    print("card (name, power limit, max SM clock): %s" % card(), flush=True)
    eng = cpb200.Engine(nstreams=13)
    reader(eng, args.reps, args.launches)
    if not args.no_e2e:
        e2e(eng, args.steps, args.warmup)
    print("card after: %s" % card(), flush=True)


if __name__ == "__main__":
    main()
