"""GPU: the drop-in entry points (cpb200.lib.decompose / cpb200.lib.net) against
 (a) golden outputs of the reference's own code (tests/golden, oracle/make_golden.py),
 (b) the oracle on BASELINE-config-sized inputs,
 (c) size-independent properties at full size (KKT of the LASSO, normal equations of the LS).
Gates (BASELINE.json north_star): selected-channel set identical; reconstructed weights within
1e-4 relative Frobenius error (in practice ~1e-9 with the fp64 Gram mode)."""
import os

import numpy as np
import pytest

import cases
import cp_oracle as O
import gather_checks as GC

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

W_TOL = 1e-4  # north_star tolerance on reconstructed weights (relative Frobenius)


@pytest.mark.parametrize("mode", [0, 1], ids=["fp64", "3xtf32"])
@pytest.mark.parametrize("name", list(cases.DICTIONARY_CASES))
def test_dictionary_matches_reference_golden(engine, golden_dir, name, mode):
    import cpb200
    from cpb200.lib import cfgs, decompose

    spec = cases.DICTIONARY_CASES[name]
    g = np.load(os.path.join(golden_dir, "dictionary_%s.npz" % name))
    X, W2, Y = cases.case_inputs(spec)
    cfgs.alpha = spec["alpha0"]
    cfgs.c.dic.rank_tol = spec.get("rank_tol", .1)
    old_mode, engine.gram_mode = engine.gram_mode, mode
    try:
        np.random.seed(spec["np_seed"])
        idxs, W, B = decompose.dictionary(X.astype(np.float64), W2, Y, rank=spec["rank"], B2=np.zeros(W2.shape[0]))
        after = np.random.randint(0, 1 << 30)
    finally:
        cfgs.c.dic.rank_tol = .1
        engine.gram_mode = old_mode
    assert idxs.dtype == np.bool_ and np.array_equal(idxs, g["idxs"])  # exact channel set
    assert after == int(g["rng_after"])  # consumed the same global RNG draws as the reference
    assert cfgs.alpha == float(g["alpha_final"])
    assert W.dtype == np.float64 and W.shape == g["W"].shape
    assert GC.rel(W, g["W"]) <= W_TOL
    # what the two arithmetic modes actually deliver; the near-collinear case (cond of the centred Gram 2e10) is
    # limited by the normal equations in fp64, cond * 2e-16
    tight = spec.get("w_tol", 1e-7 if mode == 0 else 2e-5)
    assert GC.rel(W, g["W"]) <= tight
    assert np.abs(B - g["B"]).max() <= tight * max(1.0, np.abs(g["B"]).max())


def test_dictionary_accepts_cuda_tensors(engine, golden_dir):
    from cpb200.lib import cfgs, decompose

    engine.gram_mode = 0

    spec = cases.DICTIONARY_CASES["c32"]
    g = np.load(os.path.join(golden_dir, "dictionary_c32.npz"))
    X, W2, Y = cases.case_inputs(spec)
    cfgs.alpha = spec["alpha0"]
    np.random.seed(spec["np_seed"])
    idxs, W, B = decompose.dictionary(torch.as_tensor(X, device=engine.device), torch.as_tensor(W2, device=engine.device),
                                      torch.as_tensor(Y, device=engine.device), rank=spec["rank"])
    assert np.array_equal(idxs, g["idxs"]) and GC.rel(W, g["W"]) <= 1e-7


def test_fc_kernel_matches_oracle(engine):
    from cpb200.lib import decompose

    engine.gram_mode = 0

    r = np.random.RandomState(8)
    X = np.maximum(r.standard_normal((900, 250)), 0).astype(np.float32)
    Y = (X @ r.standard_normal((250, 20)) + 0.1 * r.standard_normal((900, 20)))
    coef, icpt = decompose.fc_kernel(X.astype(np.float64), Y)
    rc, ri = O.fc_kernel(X.astype(np.float64), Y)
    assert GC.rel(coef, rc) <= 1e-8 and np.abs(icpt - ri).max() <= 1e-8
    with pytest.raises(AssertionError):
        decompose.fc_kernel(X[None], Y)  # reference asserts 2-D input (decompose.py:641)


def _forward_np(images, specs, weights, biases):
    from make_golden import conv2d_numpy

    cache = {}

    def forward(batch):
        if batch not in cache:
            blobs = {"data": images[batch % len(images)]}
            for s in specs:
                y = conv2d_numpy(blobs[s["bottom"]], weights[s["name"]], biases[s["name"]], s["pad"], s["stride"])
                blobs[s["name"]] = y
                blobs[s["name"] + "_relu"] = np.maximum(y, 0)
            cache[batch] = blobs
        return cache[batch]

    return forward


@pytest.mark.parametrize("name", list(cases.NET_CASES))
def test_net_methods_match_reference_golden(engine, golden_dir, name):
    from cpb200.lib import cfgs, net as cpnet

    spec = cases.NET_CASES[name]
    g = np.load(os.path.join(golden_dir, "net_%s.npz" % name))
    images, specs, weights, biases = cases.net_inputs(**spec["gen"])
    fnp = _forward_np(images, specs, weights, biases)
    engine.gram_mode = 0

    def forward(net, batch):  # feature provider: the same blobs the reference saw, on the device
        return {k: torch.as_tensor(v, device=engine.device) for k, v in fnp(batch).items()}

    cs = [cpnet.ConvSpec(s["name"], s["bottom"], weights[s["name"]].shape[0], s["k"], s["pad"], s["stride"])
          for s in specs]
    net = cpnet.Net(cs, weights, biases, forward)
    cfgs.c.nBatches, cfgs.c.nPointsPerLayer = spec["nBatches"], spec["P"]
    cfgs.alpha = 1e-3
    names = [s["name"] for s in specs]
    np.random.seed(spec["np_seed"])
    feats, points = net.extract_features(names, save=1)
    for nm in names:
        assert feats[nm].dtype == np.float64
        np.testing.assert_array_equal(feats[nm], g["feats_" + nm])
        for b in range(spec["nBatches"]):
            np.testing.assert_array_equal(points[(b, nm, "randx")], g["randx_%s_%d" % (nm, b)])
    net.load_frozen(feats_dict=feats, points_dict=points)
    XY = net.extract_XY(spec["xy"][0], spec["xy"][1])
    assert XY.dtype == np.float64
    np.testing.assert_array_equal(XY, g["XY"])
    if spec.get("dictionary_kernel"):
        np.random.seed(spec["np_seed"] + 1)
        idxs, W, B = net.dictionary_kernel(spec["xy"][0], None, int(g["dk_dprime"]), spec["xy"][1], None)
        assert np.array_equal(idxs, g["dk_idxs"])
        assert cfgs.alpha == float(g["dk_alpha"])
        assert GC.rel(W, g["dk_W"]) <= 1e-7 and np.abs(B - g["dk_B"]).max() <= 1e-7


def test_baseline_config1_mask_bit_compare(engine):
    """BASELINE.json configs[0]: single 256->256 3x3 layer, N=1000 patches; oracle = the reference's
    algorithm (sklearn-faithful CD + gelsd) on the CPU; N-1 < K' so the LS is the minimum-norm one."""
    from cpb200.lib import cfgs, decompose

    X, W2, Y = cases.dictionary_inputs(c=256, n=256, N=1000, k=3, seed=101)
    rank = int(256 / 1.15)
    st = O.DictState(alpha=1e-3)
    np.random.seed(77)
    info = {}
    oi, oW, oB = O.dictionary(X.astype(np.float64), W2, Y, rank=rank, state=st, info=info)
    cfgs.alpha = 1e-3
    np.random.seed(77)
    idxs, W, B = decompose.dictionary(X.astype(np.float64), W2, Y, rank=rank)
    assert np.array_equal(idxs, oi)
    assert decompose.DictionaryInfo.last["probes"] == info["probes"]  # same alpha probes and counts
    assert cfgs.alpha == st.alpha
    assert GC.rel(W, oW) <= W_TOL and np.abs(B - oB).max() <= W_TOL


@pytest.mark.parametrize("mode", [0, 1], ids=["fp64", "3xtf32"])
def test_full_size_properties_conv4_shape(engine, mode):
    """c=n=512, k=3, N=5000 (VGG conv4_x; too slow for the CPU oracle in a unit test): check what
    must hold for ANY correct solution -- LASSO KKT conditions on the device-built statistics and
    the normal equations of the reconstruction -- plus agreement of the Gram-form statistics with
    a torch fp64 evaluation."""
    import cpb200

    engine.gram_mode = mode
    gtol, netol = (1e-11, 1e-6) if mode == 0 else (2e-6, 1e-4)
    s = cpb200.synth.LayerShape("conv4_x", 512, 512, 28, N=5000)
    d = cpb200.synth.make_problem_device(s, 123, engine)
    X = engine.patch_gather(d["fmap"], d["randx"], d["randy"], s.B, s.P, s.k, s.pad, s.stride, relu=True)
    assert X.shape == (5000, 4608) and float(X.min()) >= 0
    W2m = d["W2"].reshape(s.n, s.K)
    g_full, res = engine.select_channels_async(X, W2m, d["feats"], d["b2"], d["samples"], s.c, 9, s.rank, .1, 1e-3,
                                               d["seeds"])
    scal = res.scalars.cpu().numpy()
    assert int(scal[2]) == 0
    nnz = int(scal[3])
    assert s.rank <= nnz <= s.rank * 1.1
    # Gram statistics vs torch fp64 on a sub-block
    X64 = X[:, :300].double()
    Yc = d["feats"].double() - d["b2"].double()
    Gref, Bref = X64.T @ X64, X64.T @ Yc
    assert float((g_full["G"][:300, :300] - Gref).abs().max()) <= gtol * float(Gref.abs().max())
    assert float((g_full["B"][:300] - Bref).abs().max()) <= 10 * gtol * float(Bref.abs().max())
    # KKT of the final LASSO fit (duality gap criterion => subgradient condition up to the gap)
    gs = engine.gram(X, d["feats"], y_bias=d["b2"], rows=d["samples"], want_yy=True, mode=0)
    gw = engine.gram(W2m, None, want_B=False, mode=0)
    Q, qv, yn2 = engine.lasso_build(gs, gw, W2m, s.c, 9, s.S)
    w = res.coef
    grad = qv - Q @ w
    l1 = float(scal[0]) * s.S * s.n
    active = w != 0
    assert float((grad[~active].abs()).max()) <= l1 * 1.05
    assert float((grad[active] - l1 * torch.sign(w[active])).abs().max()) <= 5e-2 * l1
    # reconstruction: centred normal equations  Xc'(Yc - Xc W - b) = 0
    idxs = res.idxs.cpu().numpy().astype(bool)
    Wd, bd, info, _ = engine.reconstruct_async(g_full, X, d["feats"], d["b2"], idxs, 9)
    assert int(info.cpu()[0]) == 0
    cols = torch.as_tensor((np.flatnonzero(idxs)[:, None] * 9 + np.arange(9)).reshape(-1), device=engine.device)
    Xs = X[:, cols].double()
    R = Yc - Xs @ Wd.T - bd
    assert float(R.mean(0).abs().max()) <= (1e-9 if mode == 0 else 1e-6)
    assert float((Xs.T @ R).abs().max()) <= netol * float((Xs.T @ Yc).abs().max())


@pytest.mark.parametrize("name", ["res2a_branch2a", "res2b_branch2a", "res3a_branch2a", "res2b_branch2b", "res3b_branch2c"])
def test_resnet50_bottleneck_problem_vs_oracle(engine, name):
    """BASELINE configs[3] shapes (1x1 / 3x3 / stride-2 bottleneck convs, target counts from the reference's
    released resnet-50-cp.prototxt) through the batched pipeline (pruner.prune_layers) against the oracle's
    dictionary_kernel on the same data, N=1000."""
    import cpb200

    row = [r for r in cpb200.synth.RESNET50 if r[0] == name][0]
    nm, c, n, k, H, st, pad, kept = row
    s = cpb200.synth.LayerShape(nm, c, n, H, k=k, pad=pad, stride=st, N=1000, rank=kept)
    d = cpb200.synth.make_problem_device(s, 77, engine)
    res = cpb200.pruner.prune_layers(engine, [s], [d], right0=1e-3)[0]
    torch.cuda.synchronize()
    fm = d["fmap"].cpu().numpy()
    pd = {"nPointsPerLayer": s.P, "nBatches": s.nbatch}
    for b in range(s.nbatch):
        pd[(b, "y", "randx")] = d["randx"][b].cpu().numpy()
        pd[(b, "y", "randy")] = d["randy"][b].cpu().numpy()
    forward = lambda b: {"x": fm[b * s.B:(b + 1) * s.B]}  # noqa: E731
    st_ = O.DictState(alpha=1e-3)
    info = {}
    with GC.seeded_lasso(d["seeds"]):
        oi, oW, oB = O.dictionary_kernel(forward, "x", O.ConvSpec("y", "x", k, pad, st), d["W2"].cpu().numpy(),
                                         d["b2"].cpu().numpy(), d["feats"].cpu().numpy().astype(np.float64), pd, kept,
                                         state=st_, samples=d["samples"].cpu().numpy(), info=info)
    assert np.array_equal(res.idxs, oi)
    if kept != c:
        assert res.alpha == st_.alpha and res.nprobe == len(info["probes"])
    W = res.W.cpu().numpy().reshape(oW.shape)
    assert GC.rel(W, oW) <= W_TOL and np.abs(res.b.cpu().numpy() - oB).max() <= W_TOL


@pytest.mark.parametrize("policy", [True, "zc", "copy"])
def test_host_resident_pipeline_equals_device_resident(policy):
    """prune_layers with the feature maps in pinned host memory (in-place gather over PCIe, whole-map DMA, or the
    per-layer plan) must return bit-identical masks and weights to the device-resident run, and results copied
    back to host buffers must equal the device ones."""
    import cpb200
    from cpb200 import pruner

    eng = cpb200.Engine(nstreams=4)
    shapes = [cpb200.synth.LayerShape("a", 32, 24, 14, N=600, B=4, P=5), cpb200.synth.LayerShape("b", 48, 16, 28, N=800, B=4, P=5),
              cpb200.synth.LayerShape("c", 16, 16, 56, N=400, B=4, P=5), cpb200.synth.LayerShape("d", 64, 32, 7, N=600, B=4, P=5),
              cpb200.synth.LayerShape("e", 24, 8, 20, k=1, pad=0, N=400, B=4, P=5)]
    datas = [cpb200.synth.make_problem_device(s, 40 + i, eng, pinned_host=True) for i, s in enumerate(shapes)]
    ref = pruner.prune_layers(eng, shapes, datas)
    torch.cuda.synchronize()
    got = pruner.prune_layers(eng, shapes, datas, from_host=policy, to_host=True)
    torch.cuda.synchronize()
    for a, b in zip(ref, got):
        assert np.array_equal(a.idxs, b.idxs) and a.alpha == b.alpha and a.nprobe == b.nprobe
        assert not b.W.is_cuda and b.W.is_pinned()
        assert torch.equal(a.W.cpu(), b.W) and torch.equal(a.b.cpu(), b.b)
    eng.close()


def test_pipeline_trace_records_every_stage():
    import cpb200
    from cpb200 import pruner

    eng = cpb200.Engine(nstreams=2)
    shapes = [cpb200.synth.LayerShape("a", 32, 24, 14, N=600, B=4, P=5), cpb200.synth.LayerShape("b", 16, 16, 28, N=400, B=4, P=5)]
    datas = [cpb200.synth.make_problem_device(s, 3 + i, eng, pinned_host=True) for i, s in enumerate(shapes)]
    tr = {}
    pruner.prune_layers(eng, shapes, datas, from_host="zc", to_host=True, trace=tr)
    torch.cuda.synchronize()
    t0 = tr.pop("_t0")
    for s in shapes:
        labels = [lab for lab, _ in tr[s.name]]
        assert labels == ["zc_done", "select_done", "ls_done"]
        times = [t0.elapsed_time(e) for _, e in tr[s.name]]
        assert times == sorted(times) and times[0] >= 0
    eng.close()
