"""bf16 against fp32 feature maps: the conv4_2 patch gather (N = 5000; NHWC by TMA and NCHW) and one end-to-end step
of prune_layers(from_host=True) on the VGG-16 shapes with the maps in pinned host memory.
    python profiles/gather16.py [--reps R] [--steps S]
Gather rates are algorithmic bytes over kernel time (CUDA events over many launches, the two dtypes alternating):
8 N K bytes for fp32 maps (read 4 + write 4 per element of X), 6 N K for 16-bit maps (read 2 + write 4)."""
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


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or "nvidia-smi: no answer"
    except Exception as e:  # pragma: no cover
        return "nvidia-smi unavailable (%s); %s" % (e, torch.cuda.get_device_name())


def gather_rates(eng, reps, launches):
    s = [x for x in cpb200.synth.vgg16_layers() if x.name == "conv4_2"][0]
    g = torch.Generator(device=eng.device)
    g.manual_seed(42)
    f32 = torch.randn((s.nbatch * s.B, s.c, s.H, s.W), generator=g, device=eng.device)
    maps = {("nchw", "fp32"): f32, ("nchw", "bf16"): f32.to(torch.bfloat16)}
    for dt in ("fp32", "bf16"):
        maps[("nhwc", dt)] = maps[("nchw", dt)].permute(0, 2, 3, 1).contiguous()
    r = np.random.RandomState(1)
    rx = torch.as_tensor(r.randint(0, s.Ho, (s.nbatch, s.P)).astype(np.int32), device=eng.device)
    ry = torch.as_tensor(r.randint(0, s.Ho, (s.nbatch, s.P)).astype(np.int32), device=eng.device)
    X = eng.empty(s.N, s.K, dtype=torch.float32)
    for (layout, dt), m in maps.items():  # warm-up; a bf16 gather must equal the gather of the widened map
        eng.patch_gather(m, rx, ry, s.B, s.P, s.k, s.pad, s.stride, layout=layout, out=X)
        if dt == "bf16":
            want = eng.patch_gather(m.float(), rx, ry, s.B, s.P, s.k, s.pad, s.stride, layout=layout)
            assert torch.equal(X, want), "bf16 gather differs from the gather of the widened map"
            del want
    torch.cuda.synchronize()
    times = {k: [] for k in maps}
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(reps):
        for layout in ("nhwc", "nchw"):
            for dt in ("fp32", "bf16"):  # alternating
                m = maps[(layout, dt)]
                a.record()
                for _ in range(launches):
                    eng.patch_gather(m, rx, ry, s.B, s.P, s.k, s.pad, s.stride, layout=layout, out=X)
                b.record()
                b.synchronize()
                times[(layout, dt)].append(a.elapsed_time(b) / launches)
    print("conv4_2 patch gather, N = %d, K = %d (c %d, k %d), %d x %d launches per config:" % (
        s.N, s.K, s.c, s.k, reps, launches))
    for (layout, dt), ts in times.items():
        ms = float(np.median(ts))
        nbytes = (8 if dt == "fp32" else 6) * s.N * s.K
        print("  %-4s %-4s  %7.3f ms  (min %7.3f)  %6.0f GB/s of %.1f MB algorithmic bytes" % (
            layout, dt, ms, min(ts), nbytes / (ms / 1e3) / 1e9, nbytes / 1e6))
    del maps, X


def e2e(eng, dtype, steps, warmup):
    shapes = cpb200.synth.vgg16_layers()
    datas = []
    for i, s in enumerate(shapes):
        d = cpb200.synth.make_problem_device(s, 1000 + i, eng, pinned_host=True, dtype=dtype)
        del d["fmap"]  # the maps live in pinned host memory only
        datas.append(d)
    torch.cuda.synchronize()
    for _ in range(warmup):
        pruner.prune_layers(eng, shapes, datas, from_host=True, to_host=True)
    torch.cuda.synchronize()
    walls = []
    for _ in range(steps):
        t0 = time.perf_counter()
        pruner.prune_layers(eng, shapes, datas, from_host=True, to_host=True)
        torch.cuda.synchronize()
        walls.append(time.perf_counter() - t0)
    plan = pruner.h2d_plan(shapes, datas, True)
    es = datas[0]["fmap_host"].element_size()
    h2d = sum(int(d["fmap_host"].numel()) * es if p == "dma" else int(s.N) * s.K * es
              for s, d, p in zip(shapes, datas, plan))
    resident = sum(int(d["fmap_host"].numel()) * es for d in datas)
    ms = 1e3 * float(np.median(walls))
    print("e2e step, VGG-16, maps %s in pinned host memory (%.1f GB): h2d plan %s, h2d %.2f GB/step, "
          "%.1f ms/step (median of %d; min %.1f), %.1f layers/s" % (
              str(dtype).replace("torch.", ""), resident / 1e9, "".join("D" if p == "dma" else "z" for p in plan),
              h2d / 1e9, ms, steps, 1e3 * min(walls), len(shapes) / (ms / 1e3)), flush=True)
    del datas


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-e2e", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "profiles/gather16.py measures on the GPU"
    print("card: %s" % card(), flush=True)
    eng = cpb200.Engine(nstreams=13)
    gather_rates(eng, args.reps, args.launches)
    if not args.no_e2e:
        # one dtype after the other (both sets of maps at once would pin 27 GB of host memory)
        for dt in (torch.float32, torch.bfloat16):
            e2e(eng, dt, args.steps, args.warmup)
            torch.cuda.empty_cache()
    print("card after: %s" % card(), flush=True)


if __name__ == "__main__":
    main()
