"""Read-request rate of the in-place gather over PCIe (pruner.ZC_LINES_PER_S): cp_patch_gather on NCHW maps in pinned
host memory, for the VGG-16 layers that take that path, as 128-byte lines touched (pruner.zero_copy_lines) per second.
    python profiles/zc_rate.py"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import cpb200
from cpb200 import pruner

eng = cpb200.Engine()
print(torch.cuda.get_device_name(), flush=True)
for s in cpb200.synth.vgg16_layers():
    if s.name not in ("conv2_2", "conv3_2", "conv4_2"):
        continue
    d = cpb200.synth.make_problem_device(s, 7, eng, pinned_host=True)
    del d["fmap"]
    X = eng.patch_gather(d["fmap_host"], d["randx"], d["randy"], s.B, s.P, s.k, s.pad, s.stride)
    times = []
    for _ in range(5):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        eng.patch_gather(d["fmap_host"], d["randx"], d["randy"], s.B, s.P, s.k, s.pad, s.stride, out=X)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    t = min(times)
    print("%s: %.3f ms, %.3g lines/s" % (s.name, 1e3 * t, pruner.zero_copy_lines(s) / t), flush=True)
    del d, X
