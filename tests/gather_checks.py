"""Scaffolding shared by the gather tests: feature maps with special values seeded in, pinned copies, bit equality,
the oracle on one pipeline problem with the pipeline's CD seeds, and the check of which gather kernels a set of cases
launches."""
import contextlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import cp_oracle as O

torch = pytest.importorskip("torch")

FMAP_DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}


def special_map(shape, dtype, seed, device):
    """N(0,1) drawn in fp32 and rounded to dtype, with -0, +-inf, NaN and subnormals (of fp32, bf16 and fp16) seeded
    in."""
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    fm = torch.randn(shape, generator=g, device=device)
    flat = fm.view(-1)
    specials = torch.tensor([-0.0, float("inf"), float("-inf"), float("nan"), 6e-8, -3e-6, 4e-5, 1e-39, -5e-39,
                             1e-44], device=device)
    idx = torch.randperm(flat.numel(), generator=g, device=device)[:max(len(specials), flat.numel() // 40)]
    flat[idx] = specials[torch.arange(idx.numel(), device=device) % len(specials)]
    return fm.to(FMAP_DTYPES[dtype])


def points3d(nb, To, Ho, Wo, device):
    """Every corner of the output volume, border points and the centre, in varying order per batch."""
    pts = [(t, x, y) for t in (0, To - 1) for x in (0, Ho - 1) for y in (0, Wo - 1)]
    pts += [(To // 2, Ho // 2, Wo // 2), (0, Ho // 2, Wo - 1), (To - 1, 1 % Ho, Wo // 2), (To // 2, 0, 1 % Wo)]
    out = []
    for axis in range(3):
        v = torch.tensor([[p[axis] for p in pts]] * nb, dtype=torch.int32, device=device)
        v[1] = v[1].flip(0)
        out.append(v)
    return out[0], out[1], out[2], len(pts)


def pinned(t):
    """A copy of t in page-locked host memory."""
    h = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
    h.copy_(t)
    return h


def assert_same_bits(got, want):
    """Bit equality of two fp32 tensors, on either device (so -0 and +0 differ); NaN positions compared separately,
    their payloads not."""
    got, want = got.cpu(), want.cpu()
    assert got.dtype == want.dtype == torch.float32 and got.shape == want.shape
    ng, nw = torch.isnan(got), torch.isnan(want)
    assert torch.equal(ng, nw)
    z = torch.zeros_like(got)
    assert torch.equal(torch.where(ng, z, got).view(torch.int32), torch.where(nw, z, want).view(torch.int32))


def rel(a, b):
    """Relative Frobenius error of a against b."""
    return np.linalg.norm(a - b) / np.linalg.norm(b)


@contextlib.contextmanager
def seeded_lasso(seeds):
    """Every cp_oracle.LassoCD built inside draws its per-fit CD seeds from seeds, in order from the first, as the
    device pipeline does; the oracle's dictionary functions otherwise take them from numpy's global RandomState."""
    orig = O.LassoCD.__init__

    def init(self, alpha, **kw):
        orig(self, alpha, **kw)
        self.rng = O.SeedFeeder(seeds)

    O.LassoCD.__init__ = init
    try:
        yield
    finally:
        O.LassoCD.__init__ = orig


def oracle_on_problem(dictionary, X, s, d):
    """The oracle's dictionary (conv_oracle's or conv3d_oracle's) on one pipeline problem d of layer s, given its
    gathered, ReLU'd X: the problem's W2, targets less b2, samples and CD seeds.  Returns (idxs, W, b, alpha, number
    of alpha probes)."""
    b2 = d["b2"].cpu().numpy()
    st = O.DictState(alpha=1e-3)
    info = {}
    with seeded_lasso(d["seeds"]):
        oi, oW, oB = dictionary(X, d["W2"].cpu().numpy(), d["feats"].cpu().numpy().astype(np.float64) - b2,
                                rank=s.rank, B2=b2, state=st, samples=d["samples"].cpu().numpy(), info=info)
    return oi, oW, oB, st.alpha, len(info["probes"])


def launched_gather_kernels(module_name):
    """Runs <module_name>._profile_kernel_cases() in a child process and returns the names of the kernels it reports,
    spaces removed.  A process that has profiled once loses more activity records in its later sessions, and other
    tests of the suite profile too, so every session gets a process of its own."""
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    code = ("import sys, json; sys.path[:0] = %r; import %s as t; "
            "print('NAMES ' + json.dumps(t._profile_kernel_cases()))"
            % ([root, os.path.join(root, "oracle"), here], module_name))
    flags = ["-s"] if sys.flags.no_user_site else []
    out = subprocess.run([sys.executable] + flags + ["-c", code], cwd=root, capture_output=True, text=True,
                         timeout=600)
    assert out.returncode == 0, out.stderr[-3000:]
    names = json.loads([ln for ln in out.stdout.splitlines() if ln.startswith("NAMES ")][-1][6:])
    return [n.replace(" ", "") for n in names]


def assert_launch_counts(names, classify, want, lost=2):
    """Every launch classifies to a kind of want, and each kind's launch count lies in [want[kind] - lost,
    want[kind]]: the profiler may drop an activity record, so no single launch decides the check."""
    seen = [classify(n) for n in names]
    assert set(seen) <= set(want), sorted(set(names))
    for kind, n in want.items():
        assert n - lost <= seen.count(kind) <= n, (kind, seen.count(kind), n, sorted(set(names)))


def all_shapes():
    """Every VGG-16 and ResNet-50 layer of synth: the shapes the transfer-plan tests run over."""
    import cpb200

    return cpb200.synth.vgg16_layers() + cpb200.synth.resnet50_layers()
