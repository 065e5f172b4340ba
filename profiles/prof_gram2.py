"""Tensor-core Gram (gram_tc2.cu) against an fp64 evaluation.
    python profiles/prof_gram2.py            # accuracy on edge shapes + timing on the conv4_2 shape
Timing: CUDA events around one cp_gram call (all its launches), L2 flushed between repetitions."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import cpb200

eng = cpb200.Engine(gram_mode=1)
dev = eng.device


def check(N, K, n, seed=0, scale=1.0, offset=0.0):
    g = torch.Generator(device=dev).manual_seed(seed)
    X = (torch.randn(N, K, device=dev, generator=g).clamp_min(0) * scale + offset).float()
    Y = (X[:, :min(K, 64)] @ torch.randn(min(K, 64), n, device=dev, generator=g) + torch.randn(N, n, device=dev, generator=g)).float()
    bias = 0.1 * torch.randn(n, device=dev, generator=g)
    ldy = (n + 3) // 4 * 4
    Yp = torch.zeros(N, ldy, device=dev)
    Yp[:, :n] = Y
    out = eng.gram(X, Yp[:, :n], y_bias=bias, mode=1)
    torch.cuda.synchronize()
    X64, Y64 = X.double(), Y.double() - bias.double()
    Gr, Br = X64.T @ X64, X64.T @ Y64
    dx, dy = Gr.diagonal().sqrt(), (Y64 ** 2).sum(0).sqrt()
    eg = ((out["G"] - Gr).abs() / torch.outer(dx, dx)).max().item()
    eb = ((out["B"] - Br).abs() / torch.outer(dx, dy)).max().item()
    xm = X64.mean(0)
    Gc_ref = Gr - N * torch.outer(xm, xm)
    Gc = out["G"] - torch.outer(out["sx"], out["sx"]) / N
    dc = Gc_ref.diagonal().sqrt().clamp_min(1e-300)
    ec = ((Gc - Gc_ref).abs() / torch.outer(dc, dc)).max().item()
    sym = bool((out["G"] == out["G"].T).all().item())
    esx = ((out["sx"] - X64.sum(0)).abs() / X64.sum(0).abs().clamp_min(1e-30)).max().item()
    print("N=%6d K=%5d n=%4d scale=%g off=%g: relG %.2e relB %.2e centred %.2e sx %.1e sym %s" %
          (N, K, n, scale, offset, eg, eb, ec, esx, sym), flush=True)
    return max(eg, eb, ec)


worst = 0.0
for (N, K, n) in [(64, 64, 4), (65, 128, 1), (257, 192, 130), (1024, 256, 128), (4999, 1152, 200), (2000, 200, 36),
                  (640, 128, 8), (300, 1000, 12), (8191, 256, 64), (5000, 576, 64), (5000, 2304, 256)]:
    worst = max(worst, check(N, K, n, seed=N + K))
worst = max(worst, check(3000, 384, 40, seed=1, scale=1e-6), check(3000, 384, 40, seed=2, scale=3e4, offset=100.0))
print("worst", worst, flush=True)

# timing on the bench's widest layer
s = cpb200.synth.LayerShape("conv4_2", 512, 512, 28, N=int(os.environ.get("CP_N", "5000")))
d = cpb200.synth.make_problem_device(s, 5, eng, layout="nhwc")
X = eng.patch_gather(d["fmap"], d["randx"], d["randy"], s.B, s.P, s.k, s.pad, s.stride, relu=True, layout="nhwc")
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
ts, tk = [], []
eng.gram_profile(True)
for it in range(8):
    flush.fill_(it)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = eng.gram(X, d["feats"], y_bias=d["b2"], want_sums=True, mode=1)
    b.record()
    torch.cuda.synchronize()
    ts.append(a.elapsed_time(b))
    tk.append(eng.gram_kernel_ms())
flop = s.N * s.K * (s.K + 1) + 2.0 * s.N * s.K * s.n
print("cp_gram conv4_2 N=%d: %s ms -> best %.4f ms = %.1f TF/s algorithmic" %
      (s.N, ["%.3f" % t for t in ts], min(ts[2:]), flop / (min(ts[2:]) / 1e3) / 1e12), flush=True)
print("GEMM kernel alone: %s ms -> best %.4f ms = %.1f TF/s algorithmic (x3 issued)" %
      (["%.3f" % t for t in tk], min(tk[2:]), flop / (min(tk[2:]) / 1e3) / 1e12), flush=True)
X64 = X.double()
Gr = X64.T @ X64
dx = Gr.diagonal().sqrt()
print("conv4_2 relG %.2e sym %s" % (((out["G"] - Gr).abs() / torch.outer(dx, dx)).max().item(),
                                    bool((out["G"] == out["G"].T).all().item())), flush=True)
