"""Layer-problem driver: one network's independent pruning problems on one or more H100s.

Within a GPU, problems are pipelined over the engine's streams in two phases (the only host
synchronisation points): phase 1 enqueues gather -> Gram statistics -> LASSO search for every
problem; phase 2, once the kept-channel masks are known on the host, enqueues the
least-squares reconstructions.  Across GPUs (one process per GPU, torch.distributed/NCCL) the
problems are assigned by longest-processing-time-first on an analytic cost and the packed
results are re-assembled on every rank with ONE all_gather (static upper-bound payload size, so
no size exchange is needed).  There is no data-path collective: layer problems are independent
(SURVEY.md 8e) -- in the reference's *sequential* R3 mode (lib/net.py:1386,1698) they are
coupled and this sharding does not apply (use lib.net.Net.R3 on one GPU).
"""
from __future__ import annotations

import math
import os
import time

import numpy as np
import torch

from .engine import Engine, conv_pair, ls_dual, settle_ls, window


# ---------------------------------------------------------------------------- assignment
# host threads that issue the reconstructions of phase 2 (an engine with one stream uses the single-threaded loop)
PHASE2_THREADS = 6
_POOLS = {}


def _phase2_pool(n):
    import concurrent.futures

    p = _POOLS.get(n)
    if p is None:
        p = _POOLS[n] = concurrent.futures.ThreadPoolExecutor(max_workers=n, thread_name_prefix="cpb200-phase2")
    return p


def assign_layers(costs, world_size):
    """LPT: returns owner[i] for each problem; deterministic (ties by index)."""
    order = sorted(range(len(costs)), key=lambda i: (-costs[i], i))
    load = [0.0] * world_size
    owner = [0] * len(costs)
    for i in order:
        r = min(range(world_size), key=lambda q: (load[q], q))
        owner[i] = r
        load[r] += costs[i]
    return owner


# ---------------------------------------------------------------------------- packing
def slot_size(c, n, k2, rank, rank_tol):
    """Upper bound (in float64 words) of one packed layer result."""
    _, rbound = window(rank, rank_tol)
    cmax = c if rank == c else min(c, int(np.floor(rbound)))
    return 4 + c + n + n * cmax * k2


def pack_result(buf, offset, idxs, W, b, alpha, nprobe, c, n, k2, eng=None, slot=0):
    """buf: 1-D float64 tensor (any device).  Layout: [c', alpha, nprobe, 0, idxs(c), b(n), W(n*c'*k2)].
    With ``eng`` the host-side scalars/mask are staged through an engine-owned PINNED buffer and every copy is
    asynchronous on the current stream (a pageable copy would make torch synchronise the stream: the pattern
    engine.lasso_select documents as a serialising bug); W / b may live on the device or in pinned host memory."""
    cp = int(idxs.sum())
    if eng is not None:
        head = eng.pinned(("pack", slot), (4 + c,), torch.float64)
        hn = head.numpy()
        hn[0], hn[1], hn[2], hn[3] = cp, alpha, nprobe, 0.0
        hn[4:] = idxs
        buf[offset:offset + 4 + c].copy_(head, non_blocking=True)
        buf[offset + 4 + c:offset + 4 + c + n].copy_(b.reshape(-1), non_blocking=True)
        buf[offset + 4 + c + n:offset + 4 + c + n + n * cp * k2].copy_(W.reshape(-1), non_blocking=True)
        return
    head = torch.tensor([cp, alpha, nprobe, 0.0], dtype=torch.float64)
    buf[offset:offset + 4] = head.to(buf.device)
    buf[offset + 4:offset + 4 + c] = torch.as_tensor(idxs.astype(np.float64)).to(buf.device)
    buf[offset + 4 + c:offset + 4 + c + n] = b.reshape(-1).to(buf.device, torch.float64)
    buf[offset + 4 + c + n:offset + 4 + c + n + n * cp * k2] = W.reshape(-1).to(buf.device, torch.float64)


def unpack_result(buf, offset, c, n, k2, window=None):
    """window: the layer's kernel extents, (kh, kw) or (kt, kh, kw) with product k2 -- W comes back (n, c', *window);
    None: a square k x k window, k = sqrt(k2)."""
    head = buf[offset:offset + 4].cpu().numpy()
    cp = int(head[0])
    idxs = buf[offset + 4:offset + 4 + c].cpu().numpy() != 0
    b = buf[offset + 4 + c:offset + 4 + c + n].cpu().numpy()
    if window is None:
        k = int(round(np.sqrt(k2)))
        window = (k, k)
    assert int(np.prod(window)) == k2, (window, k2)
    W = buf[offset + 4 + c + n:offset + 4 + c + n + n * cp * k2].cpu().numpy().reshape((n, cp) + tuple(window))
    return dict(idxs=idxs, W=W, b=b, alpha=float(head[1]), nprobe=int(head[2]))


def allgather_results(local_buf, world_size, group=None):
    """ONE collective: every rank contributes a buffer of identical (upper-bound) length."""
    import torch.distributed as dist

    out = torch.empty(world_size * local_buf.numel(), dtype=local_buf.dtype, device=local_buf.device)
    dist.all_gather_into_tensor(out, local_buf, group=group)
    return out.view(world_size, -1)


# ---------------------------------------------------------------------------- single-GPU pipeline
class LayerResult:
    __slots__ = ("idxs", "W", "b", "alpha", "nprobe", "probes", "info")


def prune_layers(eng: Engine, shapes, datas, right0=1e-3, rank_tol=.1, from_host=False, to_host=False, trace=None):
    """Runs the layer problems ``shapes[i]`` / ``datas[i]`` (see synth.make_problem_device) on
    ``eng``.  from_host: feature maps are taken from pinned host memory (datas[i]['fmap_host'], float32, bfloat16
    or float16, laid out as datas[i]['host_layout']: 'nchw' (default) or 'nhwc') and copied in the pipeline; to_host:
    results are copied back to pinned host memory.
    Conv3d layers (synth.LayerShape3d, whose data carry randt) may stand alone or among 2-D ones; their layouts are
    'ncdhw' (default) or 'ndhwc'.  Transposed layers (shape.transposed: ConvTranspose2d / 3d) are gathered with their
    own window; W2 and the returned W are (n, c, *window) as for every layer, W.transpose(0, 1) the new weight.
    trace: optional dict; filled with {layer name: [(label, timing event), ...]} plus '_t0' (device timeline
    of the step: profiles/e2e_breakdown.py prints it).
    Batch mode: the problems are INDEPENDENT -- every alpha search starts from ``right0`` and the seeds come with the
    problem (datas[i]['seeds']), so the call neither reads nor writes ``cfgs.alpha`` and draws nothing from numpy's
    global RNG.  The reference's sequential walk carries alpha from layer to layer (lib/decompose.py:491,627) and draws
    one seed per probe; that behaviour lives in lib.decompose.dictionary / Net.R3, which run the layers one after the
    other.  Masks and alphas of the two modes are therefore not comparable layer by layer (DESIGN.md section 8).
    Every reconstruction is verified before it is returned (Cholesky status + pivot ratio, see the end of
    _prune_layers_ordered): r.info['verdict'] is 'ok', 'redo->ok' (re-solved from exact-product statistics) or
    'truncated' (rank deficient: gelsd's minimum-norm solution).
    Returns a list of LayerResult (W, b as device fp64 tensors unless to_host)."""
    nslots = len(eng.streams)
    main = torch.cuda.current_stream(eng.device)
    # longest problems first: their (latency-bound) LASSO searches start early and the short ones fill the GPU
    order = sorted(range(len(shapes)), key=lambda i: (-shapes[i].cost(), i))
    inv = {orig: pos for pos, orig in enumerate(order)}
    shapes_o = [shapes[i] for i in order]
    datas_o = [datas[i] for i in order]
    if trace is not None:
        trace["_t0"] = torch.cuda.Event(enable_timing=True)
        trace["_t0"].record()
    res_o = _prune_layers_ordered(eng, shapes_o, datas_o, right0, rank_tol, from_host, to_host, main, trace)
    return [res_o[inv[i]] for i in range(len(shapes))]


# Both rates were measured for the conv readers.  The transposed-convolution readers (gather_tr.cu) are charged at
# them too: their line rates are not measured.
# read requests per second of the in-place gather over PCIe (profiles/zc_rate.py; H100 80GB HBM3 SXM, PCIe 5)
ZC_LINES_PER_S = 2.6e8
# full 128-byte lines per second of the in-place NHWC reader, whose requests are whole lines of contiguous window rows
# (profiles/host_nhwc.py, conv2_2 to conv5_1 at N = 5000, fp32 and bf16: 6.8e7 to 7.7e7, median 7.1e7, about 9 GB/s,
# on an H100 80GB HBM3 SXM at 700 W whose NCHW reader ran at 2.2e8 to 3.0e8 lines/s, the regime of ZC_LINES_PER_S;
# another such card read 1.9e8 NHWC and 5.7e8 NCHW lines/s: the host link varies, the ratio of the two readers not)
ZC_NHWC_LINES_PER_S = 7.1e7


def window_of(s):
    """Kernel extents of a layer shape: (kh, kw), or (kt, kh, kw) for a Conv3d layer (synth.LayerShape3d)."""
    return (s.kt, s.kh, s.kw) if _is3d(s) else (getattr(s, "kh", s.k), getattr(s, "kw", s.k))


def _is3d(s):
    return hasattr(s, "kt")


def _default_layout(s):
    return "ncdhw" if _is3d(s) else "nchw"


def _patch_gather(eng, s, d, fmap, layout):
    """The gather of layer s from map fmap (layout as the map lies): Engine.patch_gather3d for a Conv3d layer
    (d carries randt), Engine.patch_gather otherwise; through the shape's input transform (s.act, s.act_param; the
    ReLU when the shape has none) and the problem's affine (d['in_scale'], d['in_shift'], when present)."""
    xf = dict(act=getattr(s, "act", "relu"), act_param=getattr(s, "act_param", None), in_scale=d.get("in_scale"),
              in_shift=d.get("in_shift"))
    if _is3d(s):
        return eng.patch_gather3d(fmap, d["randt"], d["randx"], d["randy"], s.B, s.P, layout=layout, **xf,
                                  **s.conv_args())
    return eng.patch_gather(fmap, d["randx"], d["randy"], s.B, s.P, layout=layout, **xf, **s.conv_args())


def zero_copy_lines(s, esize=4, layout="nchw"):
    """128-byte lines the in-place gather touches in host memory (esize: bytes per map element), for a window of
    kh x kw taps with dilation (dil_h, dil_w) (s.kh, s.kw, s.dilation; a shape with only s.k is square, undilated).
    nchw: c*kh rows of kw taps per window, each row counted as the lines its taps span (one for the reference's
    k <= 9 rows); the rows of a channel are dil_h*W*esize bytes apart.
    nhwc: kh window rows; an undilated row is one run of kw*c*esize contiguous bytes, a dilated one kw runs of
    c*esize bytes (or, if fewer, the lines of the span from its first tap to its last); plus one line per run when the
    pixel stride c*esize is not a multiple of 128 bytes (a run may then start inside a line).  An upper bound for a
    map whose base is 128-byte aligned: clipping at the border only removes lines.
    Square, undilated windows give the counts the transfer rates ZC_LINES_PER_S and ZC_NHWC_LINES_PER_S were
    measured with.
    Conv3d layers (s.kt): 'ncdhw' counts c*kt*kh rows of kw taps, 'ndhwc' kt*kh runs of kw*c*esize bytes -- kt times
    the 2-D count of the (kh, kw) window rows of one frame (frames are H*W pixels apart).
    Transposed layers (s.transposed): _zero_copy_lines_tr."""
    if getattr(s, "transposed", False):
        return _zero_copy_lines_tr(s, esize, layout)
    if _is3d(s):
        flat = _Frame(s)
        return s.kt * zero_copy_lines(flat, esize, "nhwc" if layout in ("nhwc", "ndhwc") else "nchw")
    kh, kw = getattr(s, "kh", s.k), getattr(s, "kw", s.k)
    dh, dw = conv_pair(getattr(s, "dilation", 1))
    span_w = (kw - 1) * dw + 1  # elements from the first tap of a window row to its last
    if layout == "nhwc":
        tail = 1 if (s.c * esize) % 128 else 0
        per_row = -(-span_w * s.c * esize // 128) + tail
        if dw > 1:
            per_row = min(per_row, kw * (-(-s.c * esize // 128) + tail))
        return s.N * kh * per_row
    row = s.W * esize if hasattr(s, "W") else esize * 64
    per_row = min(kw, -(-span_w * esize // 128))
    span = (kh - 1) * dh * row + span_w * esize
    lines = min(kh * per_row, -(-span // 128) + 1) if kh * kw > 1 else 1
    return s.N * s.c * lines


def _tr_touched(k, stride, dil):
    """One axis of a transposed window: the most input coordinates one output coordinate's valid taps read,
    ceil(k / (stride / g)), and their spacing dil / g (g = gcd(stride, dil)), whatever the output coordinate's phase."""
    g = math.gcd(stride, dil)
    return -(-k // (stride // g)), dil // g


def _zero_copy_lines_tr(s, esize, layout):
    """128-byte lines the in-place gather of a transposed layer touches, an upper bound over the phases of the points
    for a map whose base is 128-byte aligned.  Per point the valid taps read m_t x m_h input rows (_tr_touched; m_t = 1
    in 2-D) and, in each, m_w pixels sw apart.
    nchw: per channel and row, the m_w elements span ((m_w - 1) sw + 1) * esize bytes: at most one line more than
    that span fills, and never more than m_w lines.
    nhwc: per row, the m_w pixels' c channels span ((m_w - 1) sw + 1) * c * esize bytes (m_w runs of c * esize bytes
    when sw > 1, if that is fewer), plus one line per run when the pixel stride is not a multiple of 128 bytes."""
    axes = ([(s.kt, s.stride_t, s.dil_t)] if _is3d(s) else []) + [(s.kh, s.stride_h, s.dil_h),
                                                                    (s.kw, s.stride_w, s.dil_w)]
    touched = [_tr_touched(*a) for a in axes]
    rows = int(np.prod([m for m, _ in touched[:-1]]))
    mw, sw = touched[-1]
    span = (mw - 1) * sw + 1  # pixels from the first touched one of a row to its last
    if layout in ("nhwc", "ndhwc"):
        tail = 1 if (s.c * esize) % 128 else 0
        per_row = -(-span * s.c * esize // 128) + tail
        if sw > 1:
            per_row = min(per_row, mw * (-(-s.c * esize // 128) + tail))
        return s.N * rows * per_row
    return s.N * s.c * rows * min(mw, -(-span * esize // 128) + 1)


class _Frame:
    """The (kh, kw) window of a Conv3d layer on one frame: what zero_copy_lines counts per temporal tap."""

    def __init__(self, s):
        self.N, self.c, self.W, self.kh, self.kw = s.N, s.c, s.W, s.kh, s.kw
        self.k, self.dilation = s.kh, (s.dil_h, s.dil_w)


def _zero_copy_seconds(s, esize=4, layout="nchw"):
    """Model of the in-place gather over PCIe: it is bound by the number of read requests."""
    rate = ZC_NHWC_LINES_PER_S if layout in ("nhwc", "ndhwc") else ZC_LINES_PER_S
    return zero_copy_lines(s, esize, layout) / rate


def _element_size(fmap):
    """Bytes per element of a host map (float32 4, bfloat16 / float16 2); a map that only reports numel() counts as
    float32."""
    return fmap.element_size() if hasattr(fmap, "element_size") else 4


def h2d_plan(shapes, datas, from_host):
    """Per layer: 'zc' (gather kernel reads the windows in place from pinned host memory) or 'dma' (copy engine
    moves the whole map at full PCIe bandwidth, gather from HBM).  DMA pays off when the windows cover most of
    the map (small spatial maps: conv5_x).  CPB200_DMA_MAX_MB caps the size of a map that may be staged.
    The reader and the copy engine share the link, so moving a map from one to the other buys nothing unless it
    removes bytes.  The reader's cost follows the host map's layout (datas[i]['host_layout'], 'nchw' by default)."""
    if from_host == "zc":
        return ["zc"] * len(shapes)
    if from_host == "copy":
        return ["dma"] * len(shapes)
    cap = float(os.environ.get("CPB200_DMA_MAX_MB", "300")) * 1e6
    ratio = float(os.environ.get("CPB200_DMA_RATIO", "0.8"))
    plan = []
    for s, d in zip(shapes, datas):
        esize = _element_size(d["fmap_host"])
        nbytes = d["fmap_host"].numel() * esize
        t_dma = nbytes / 50e9 + 1e-4
        t_zc = _zero_copy_seconds(s, esize, d.get("host_layout", _default_layout(s)))
        plan.append("dma" if (nbytes <= cap and t_dma < ratio * t_zc) else "zc")
    return plan


def _mark(trace, name, label):
    if trace is not None:
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        trace.setdefault(name, []).append((label, e))


def _prune_layers_ordered(eng, shapes, datas, right0, rank_tol, from_host, to_host, main, trace=None):
    # ---- host-resident inputs: PCIe is the shared resource, so the transfers are issued in the (longest-first)
    # layer order on two dedicated streams -- zero-copy gathers on one, whole-map DMAs on the copy engine --
    # and each layer stream waits only for its own transfer.
    pre = [None] * len(shapes)
    if from_host and len(eng.streams) > 1 and eng.streams[0] is not None:
        plan = h2d_plan(shapes, datas, from_host)
        zc_stream, dma_stream = eng.xfer_streams()
        zc_stream.wait_stream(main)
        dma_stream.wait_stream(main)
        dma_order = sorted((i for i in range(len(shapes)) if plan[i] == "dma"),
                           key=lambda i: (datas[i]["fmap_host"].numel(), i))
        for i in dma_order:
            with torch.cuda.stream(dma_stream):
                st = eng.staging(("fmap", i), datas[i]["fmap_host"].shape, datas[i]["fmap_host"].dtype)
                st.copy_(datas[i]["fmap_host"], non_blocking=True)
                _mark(trace, shapes[i].name, "dma_done")
                ev = torch.cuda.Event()
                ev.record()
            pre[i] = ("dma", st, ev)
        for i, (s, d) in enumerate(zip(shapes, datas)):
            if plan[i] != "zc":
                continue
            eng.use_slot(i)
            with torch.cuda.stream(zc_stream):
                X = _patch_gather(eng, s, d, d["fmap_host"], d.get("host_layout", _default_layout(s)))
                _mark(trace, s.name, "zc_done")
                ev = torch.cuda.Event()
                ev.record()
            pre[i] = ("zc", X, ev)
    phase1 = []
    for i, (s, d) in enumerate(zip(shapes, datas)):
        stream = eng.use_slot(i)
        ctx = torch.cuda.stream(stream) if stream is not None else _null()
        with ctx:
            if stream is not None:
                stream.wait_stream(main)
            X = None
            layout = d.get("host_layout", _default_layout(s))  # of fmap_host, and of its staged copy in HBM
            if pre[i] is not None:
                kind, obj, ev = pre[i]
                stream.wait_event(ev)
                if kind == "zc":
                    X = obj
                else:
                    fmap = obj
            elif from_host == "copy":
                fmap = eng.staging(("fmap", i), d["fmap_host"].shape, d["fmap_host"].dtype)
                fmap.copy_(d["fmap_host"], non_blocking=True)
            elif from_host:
                # zero-copy: the gather kernel reads the sampled windows straight out of pinned host memory;
                # only the touched 32-byte sectors cross PCIe (1-40 % of a feature map), not the whole map
                fmap = d["fmap_host"]
            else:
                fmap = d["fmap"]
                layout = d.get("layout", _default_layout(s))  # HBM layout of fmap
            if X is None:
                X = _patch_gather(eng, s, d, fmap, layout)
            W2m = d["W2"].reshape(s.n, s.K)
            if s.rank == s.c:
                g_full = eng.gram(X, d["feats"], y_bias=d["b2"])
                res = None
                host = None
            else:
                g_full, res = eng.select_channels_async(X, W2m, d["feats"], d["b2"], d["samples"], s.c, s.k2,
                                                        s.rank, rank_tol, right0, d["seeds"])
                host = (eng.pinned(("scal", i), (4,), torch.float64), eng.pinned(("idxs", i), (s.c,), torch.uint8))
                host[0].copy_(res.scalars, non_blocking=True)
                host[1].copy_(res.idxs, non_blocking=True)
            _mark(trace, s.name, "select_done")
            ev = torch.cuda.Event()
            ev.record()
        phase1.append((X, g_full, res, host, ev))
    out = [None] * len(shapes)
    # phase 2 in COMPLETION order of the searches (which layer finishes first depends on sizes and, with
    # host-resident inputs, on the transfer order): poll the events, reconstruct whichever is ready.
    # A reconstruction of a wide layer is hundreds of kernel launches (host time inside libcpb200 calls, which
    # release the GIL): issued from one thread, the c = 512 layers of VGG-16 would queue behind one another on the
    # HOST.  Worker threads issue them side by side; the engine's current (handle, stream) slot is thread-local.
    checks = []

    def reconstruct_layer(i):
        s, d = shapes[i], datas[i]
        X, g_full, res, host, ev = phase1[i]
        if res is not None:
            ev.synchronize()
        torch.cuda.set_device(eng.device)
        stream = eng.use_slot(i)
        r = LayerResult()
        if res is None:
            r.idxs = np.ones(s.c, dtype=bool)
            r.alpha, r.nprobe = 1e-4, 0  # lib/decompose.py:386 argument default survives (:627)
        else:
            scal = host[0].numpy()
            if int(scal[2]) != 0:
                raise RuntimeError("layer %s: alpha search hit the probe cap" % s.name)
            r.idxs = host[1].numpy().astype(bool)
            r.alpha, r.nprobe = float(scal[0]), int(scal[1])
        ctx = torch.cuda.stream(stream) if stream is not None else _null()
        with eng.slot_lock(i), ctx:  # layers that share a slot (more layers than streams) are issued one after the other
            W, b, info, stat = eng.reconstruct_async(g_full, X, d["feats"], d["b2"], r.idxs, s.k2)
            chk = (eng.pinned(("lsinfo", i), (1,), torch.int32), eng.pinned(("lsstat", i), (1,), torch.float64))
            chk[0].copy_(info, non_blocking=True)
            chk[1].copy_(stat, non_blocking=True)
            r.W, r.b = _maybe_to_host(eng, i, W, b, to_host)  # eager: the copy overlaps the other layers' solves
            ev_ls = torch.cuda.Event()
            ev_ls.record()
            _mark(trace, s.name, "ls_done")
        r.probes = res
        r.info = {"mode": g_full["mode"], "dual": ls_dual(g_full["N"], r.idxs, s.k2)}
        out[i] = r
        return (i, chk, ev_ls)

    nworkers = min(PHASE2_THREADS, len(shapes)) if eng.streams[0] is not None else 1
    pool = _phase2_pool(nworkers) if nworkers > 1 else None
    futures = []
    pending = list(reversed(range(len(shapes))))
    while pending:
        ready = [i for i in pending if phase1[i][2] is None or phase1[i][4].query()]
        if not ready:
            time.sleep(2e-5)
            continue
        i = ready[0]
        pending.remove(i)
        if pool is not None:
            futures.append(pool.submit(reconstruct_layer, i))
        else:
            checks.append(reconstruct_layer(i))
    checks.extend(f.result() for f in futures)
    # ---- every reconstruction is CHECKED before it is handed out (Cholesky status + conditioning signal) and, where
    # the policy says so, redone on its layer's slot (engine.settle_ls).
    for i, chk, ev_ls in checks:
        ev_ls.synchronize()
        s, d, r = shapes[i], datas[i], out[i]
        stream = eng.use_slot(i)
        with torch.cuda.stream(stream) if stream is not None else _null():
            W, b, rec = settle_ls(eng, phase1[i][0], d["feats"], d["b2"], r.idxs, s.k2, r.info["mode"],
                                  int(chk[0][0]), float(chk[1][0]))
            if W is not None:
                r.W, r.b = _maybe_to_host(eng, i, W, b, to_host)
        r.info.update(rec)
    for st in eng.streams:
        if st is not None:
            main.wait_stream(st)
    return out


def _maybe_to_host(eng, i, W, b, to_host):
    if not to_host:
        return W, b
    # engine-owned pinned buffers: valid until the next prune_layers call on this engine
    Wh = eng.pinned(("W", i), W.shape, torch.float64)
    bh = eng.pinned(("b", i), b.shape, torch.float64)
    Wh.copy_(W, non_blocking=True)
    bh.copy_(b, non_blocking=True)
    return Wh, bh


class _null:
    def __enter__(self):
        return None

    def __exit__(self, *a):
        return False


# ---------------------------------------------------------------------------- multi-GPU
def prune_network_sharded(eng: Engine, shapes, make_data, rank, world_size, right0=1e-3, rank_tol=.1, group=None):
    """Each rank solves its LPT share and all ranks end with every layer's result.
    make_data(i) -> data dict for problem i (only called for owned problems)."""
    owner = assign_layers([s.cost() for s in shapes], world_size)
    mine = [i for i, o in enumerate(owner) if o == rank]
    datas = [make_data(i) for i in mine]
    res = prune_layers(eng, [shapes[i] for i in mine], datas, right0=right0, rank_tol=rank_tol)
    sizes = [slot_size(s.c, s.n, s.k2, s.rank, rank_tol) for s in shapes]
    # static layout: rank r's buffer holds its problems in index order; pad to the largest rank buffer
    per_rank = [sum(sizes[i] for i in range(len(shapes)) if owner[i] == r) for r in range(world_size)]
    buf = torch.zeros(max(per_rank), dtype=torch.float64, device=eng.device)
    off = 0
    for j, i in enumerate(mine):
        s = shapes[i]
        pack_result(buf, off, res[j].idxs, res[j].W, res[j].b, res[j].alpha, res[j].nprobe, s.c, s.n, s.k2,
                    eng=eng, slot=j)
        off += sizes[i]
    if world_size > 1:
        allbuf = allgather_results(buf, world_size, group)
    else:
        allbuf = buf.view(1, -1)
    return owner, sizes, allbuf


def unpack_network(shapes, owner, sizes, allbuf):
    offs = [0] * allbuf.shape[0]
    out = [None] * len(shapes)
    for i, s in enumerate(shapes):
        r = owner[i]
        out[i] = unpack_result(allbuf[r], offs[r], s.c, s.n, s.k2, window_of(s))
        offs[r] += sizes[i]
    return out
