"""One least-squares reconstruction (cp_ls_solve [+ refinement]) and one LASSO search of a VGG-shaped problem:
host issue time vs device time, and -- under ncu --profile-from-start off -- the launch list of exactly these calls.
    python profiles/prof_ls.py [c] [H]
    ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv --log-file X.csv python profiles/prof_ls.py"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import cpb200

c = int(sys.argv[1]) if len(sys.argv) > 1 else 512
H = int(sys.argv[2]) if len(sys.argv) > 2 else 28
eng = cpb200.Engine()
s = cpb200.synth.LayerShape("L", c, c, H, N=5000)
d = cpb200.synth.make_problem_device(s, 7, eng)
W2m = d["W2"].reshape(s.n, s.K)
X = eng.patch_gather(d["fmap"], d["randx"], d["randy"], s.B, s.P, s.k, s.pad, s.stride, relu=True)
g_full = eng.gram(X, d["feats"], y_bias=d["b2"])
g_s = eng.gram(X, d["feats"], y_bias=d["b2"], rows=d["samples"], want_yy=True, mode=0)
g_w = eng.gram(W2m, None, want_B=False, mode=0)
Q, qv, yn2 = eng.lasso_build(g_s, g_w, W2m, s.c, 9, s.S)
lb, rb = cpb200.engine.window(s.rank, .1)
res = eng.lasso_select(Q, qv, yn2, float(s.S) * s.n, s.rank, lb, rb, 1e-3, d["seeds"])
idxs = res.idxs.cpu().numpy().astype(bool)
cols = eng._cols_device(idxs, 9, s.K)
lib = cpb200._cabi.load()[1]


def timed(label, fn, reps=3):
    fn()
    torch.cuda.synchronize()
    host, dev, launches = [], [], []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        l0 = lib.cp_launch_count()
        t0 = time.perf_counter()
        a.record()
        fn()
        b.record()
        host.append(time.perf_counter() - t0)
        torch.cuda.synchronize()
        dev.append(a.elapsed_time(b))
        launches.append(lib.cp_launch_count() - l0)
    print("%-34s host issue %.3f ms | device %.3f ms | %d launches" % (label, 1e3 * min(host), min(dev), launches[-1]), flush=True)


print("c=%d K=%d K'=%d n=%d" % (c, s.K, cols.numel(), s.n))
timed("ls_solve (factor+backward)", lambda: eng.ls_solve(g_full, cols))
W, b, info, stat = eng.ls_solve(g_full, cols)
timed("ls_residual", lambda: eng.ls_residual(X, d["feats"], d["b2"], cols, W, b))
R = eng.ls_residual(X, d["feats"], d["b2"], cols, W, b)
timed("gram(X, R) cross products", lambda: eng.gram(X, R, want_G=False))
gr = eng.gram(X, R, want_G=False)
timed("ls_resolve (forward+backward)", lambda: eng.ls_resolve(gr["B"], g_full["sx"], gr["sy"], cols))
timed("reconstruct_async (solve+refine)", lambda: eng.reconstruct_async(g_full, X, d["feats"], d["b2"], idxs, 9))
timed("lasso_select", lambda: eng.lasso_select(Q, qv, yn2, float(s.S) * s.n, s.rank, lb, rb, 1e-3, d["seeds"]), reps=2)
timed("gram full (tc)", lambda: eng.gram(X, d["feats"], y_bias=d["b2"]))
# the profiled region: one solve + refinement, one search
torch.cuda.synchronize()
torch.cuda.profiler.start()
eng.reconstruct_async(g_full, X, d["feats"], d["b2"], idxs, 9)
torch.cuda.synchronize()
torch.cuda.profiler.stop()
# accuracy of the tensor-core path (statistics, bulk products of the solve, residual) against the exact-product fp64 solve
Wt, bt, _, st = eng.reconstruct_async(g_full, X, d["feats"], d["b2"], idxs, 9)
We, be, _, _ = eng.reconstruct_exact_async(X, d["feats"], d["b2"], idxs, 9)
torch.cuda.synchronize()
print("tensor-core path vs exact fp64 solve: rel W %.2e, rel b %.2e, pivot ratio %.3g" % (
    ((Wt - We).norm() / We.norm()).item(), ((bt - be).norm() / be.norm()).item(), st.item()), flush=True)
