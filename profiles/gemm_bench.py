"""fp64 GEMM kernels of libcpb200 (gemm_f64.cuh through cp_gemm_f64) against cuBLAS on the shapes the solver uses.
cp_gemm_f64 runs the cp.async kernel unless the product has fewer 128 x 128 tiles than twice the SMs and a reduction of
at least 128: those (the substitution, panel-solve and residual shapes) split the reduction over the register-staged
kernel.  The solver itself calls the cp.async kernel directly, without a split.
    python profiles/gemm_bench.py
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import cpb200

eng = cpb200.Engine()
dev = eng.device


def timed(fn, reps=5):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return min(ts)


shapes = [("square 4096^3", 4096, 4096, 4096), ("trailing update 4096 x 4096 x 256", 4096, 4096, 256),
          ("trailing update 4096 x 4096 x 128", 4096, 4096, 128), ("substitution 512 x 3584 x 512", 512, 3584, 512),
          ("substitution 512 x 512 x 512", 512, 512, 512), ("panel solve 4608 x 128 x 128", 4608, 128, 128),
          ("residual 5000 x 512 x 4284", 5000, 512, 4284)]
for name, M, Nn, R in shapes:
    A = torch.randn(M, R, device=dev, dtype=torch.float64)
    B = torch.randn(Nn, R, device=dev, dtype=torch.float64)
    C = torch.zeros(M, Nn, device=dev, dtype=torch.float64)
    flop = 2.0 * M * Nn * R
    t_own = timed(lambda: eng.gemm(A, B, alpha=-1.0, beta=1.0, out=C))
    t_lib = timed(lambda: torch.addmm(C, A, B.T, beta=1.0, alpha=-1.0, out=C))
    print("%-36s own %7.3f ms %5.1f TF/s | cuBLAS %7.3f ms %5.1f TF/s" % (name, t_own, flop / t_own / 1e9, t_lib,
                                                                           flop / t_lib / 1e9))
