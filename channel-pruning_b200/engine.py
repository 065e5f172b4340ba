"""Device-side engine: torch tensors as device buffers, libcpb200 kernels as the compute.

One ``Engine`` per process/GPU.  It owns ``nstreams`` CUDA streams, each with its own
libcpb200 handle (scratch workspace is per handle), so that independent layer problems
can overlap: the LASSO search is a single-CTA latency-bound kernel and the Cholesky
panels are small, while the Gram/trailing-update kernels fill the chip -- running
several layers concurrently on separate streams keeps the SMs busy.

Every method enqueues work on the *current* torch stream unless stated; nothing here
touches the CPU oracle, and there is no fallback: without a CUDA device or without
libcpb200.so construction fails.
"""
from __future__ import annotations

import os
import threading

import numpy as np
import torch

from . import _cabi

RAND_R_MAX = 2147483647
MAX_PROBES = 64
# Least squares from tensor-core (3xTF32) statistics: the ~4e-7 relative error of that Gram is amplified by the
# conditioning of the system (profiles/conditioning_map.py maps the weight error against the pivot ratio), so every such solve is followed by ONE step of iterative refinement against the
# same factor with the residual taken from the data (engine.ls_refine) -- which squares the error -- and is accepted
# only while the smallest Cholesky pivot keeps at least LS_RATIO_MIN of its original diagonal entry (1 - R^2 of the
# most collinear column); below that the layer is re-solved from exact-product fp64 statistics (settle_ls).
LS_RATIO_MIN = 0.005

_LAYOUTS = {"nchw": 0, "nhwc": 1}
_LAYOUTS3D = {"ncdhw": 0, "ndhwc": 1}  # the same C codes, with a depth axis
GRAM_FP64, GRAM_3XTF32 = 0, 1
# element types of the feature maps the gathers read (CP_F32, CP_BF16, CP_F16 of include/cpb200.h)
FMAP_DTYPES = {torch.float32: 0, torch.bfloat16: 2, torch.float16: 3}


def conv_pair(v):
    """(h, w) of a Conv2d-style argument given as an int or a pair (kernel_size, padding, stride, dilation)."""
    if isinstance(v, (tuple, list)):
        assert len(v) == 2, v
        return int(v[0]), int(v[1])
    return int(v), int(v)


def conv_triple(v):
    """(t, h, w) of a Conv3d-style argument given as an int or a triple (kernel_size, padding, stride, dilation)."""
    if isinstance(v, (tuple, list)):
        assert len(v) == 3, v
        return int(v[0]), int(v[1]), int(v[2])
    return int(v), int(v), int(v)


def fmap_dtype_code(dtype):
    """The C ABI code of a feature-map dtype; TypeError for a type the gathers do not read."""
    code = FMAP_DTYPES.get(dtype)
    if code is None:
        raise TypeError("feature maps must be float32, bfloat16 or float16, got %s" % (dtype,))
    return code


# the activations of a consumer's input transform: name -> CP_ACT_* of include/cpb200.h
ACTS = {"identity": 0, "relu": 1, "relu6": 2, "leaky_relu": 3, "hardswish": 4, "silu": 5}
LEAKY_SLOPE = 0.01  # torch.nn.LeakyReLU's default negative_slope


def check_act(act, act_param):
    """ValueError for an activation not in ACTS, or a slope given to an activation other than leaky_relu."""
    if act not in ACTS:
        raise ValueError("unknown activation %r (one of %s)" % (act, ", ".join(ACTS)))
    if act_param is not None and act != "leaky_relu":
        raise ValueError("act_param (the negative slope) is an argument of leaky_relu, not of %r" % act)


def input_transform(relu, act, act_param, in_scale, in_shift, c, device):
    """The input transform a gather was asked for: None for the relu flag's gathers (relu True / None, or act 'relu',
    without an affine; relu False or act 'identity' likewise), else (CP_ACT code, slope, scale, shift).  relu and act
    exclude each other; scale and shift are contiguous fp32 tensors of c values on device, or None."""
    if relu is not None and act is not None:
        raise ValueError("pass relu or act, not both")
    if act is None:
        if act_param is not None:
            raise ValueError("act_param without act")
        act = "identity" if relu is False else "relu"
    check_act(act, act_param)
    for t in (in_scale, in_shift):
        if t is not None:
            assert t.dtype == torch.float32 and t.is_contiguous() and t.numel() == c, "scale / shift: %d fp32" % c
            assert t.is_cuda and t.device == device, "scale / shift must live on %s" % device
    if act in ("relu", "identity") and in_scale is None and in_shift is None:
        return None
    slope = float(LEAKY_SLOPE if act_param is None else act_param) if act == "leaky_relu" else 0.0
    return ACTS[act], slope, in_scale, in_shift


def _gather_map(fmap, B, layout, d3):
    """(dtype code, layout code, nbatch, dims) of a gather's map (nbatch*B images): dims is (c, H, W) of a 2-D map and
    (c, D, H, W) of a 3-D one (d3), c the channels whichever the layout.  TypeError for a dtype the gathers do not read,
    before anything else."""
    dt = fmap_dtype_code(fmap.dtype)
    assert fmap.is_contiguous() and fmap.dim() == (5 if d3 else 4)
    lay = (_LAYOUTS3D if d3 else _LAYOUTS)[layout]
    s = tuple(fmap.shape[1:])
    return dt, lay, fmap.shape[0] // B, s if lay == 0 else s[-1:] + s[:-1]


class LassoResult:
    """Device-resident outputs of one channel selection (cp_lasso_select)."""

    __slots__ = ("idxs", "coef", "scalars", "probe_log", "seeds")

    def __init__(self, idxs, coef, scalars, probe_log, seeds):
        self.idxs, self.coef, self.scalars, self.probe_log, self.seeds = idxs, coef, scalars, probe_log, seeds


def gpu_numa_cpus(device_index):
    """CPUs of the NUMA node the GPU hangs off (from sysfs), or None when the platform does not say."""
    try:
        pr = torch.cuda.get_device_properties(device_index)
        bdf = "%04x:%02x:%02x.0" % (pr.pci_domain_id, pr.pci_bus_id, pr.pci_device_id)
        node = int(open("/sys/bus/pci/devices/%s/numa_node" % bdf).read().strip())
        if node < 0:
            return None
        cpus = set()
        for part in open("/sys/devices/system/node/node%d/cpulist" % node).read().strip().split(","):
            lo, _, hi = part.partition("-")
            cpus.update(range(int(lo), int(hi or lo) + 1))
        return cpus or None
    except Exception:
        return None


class numa_local:
    """Context: page-locked host buffers allocated inside are placed on the NUMA node of ``device_index`` (first
    touch under a temporary CPU affinity; a GPU reading host memory of the other socket pays the inter-socket
    link on every PCIe read -- round-1 measurement: 0.75 e2e scaling efficiency at 8 GPUs from one node's memory)."""

    def __init__(self, device_index):
        self.cpus = gpu_numa_cpus(device_index)
        self.old = None

    def __enter__(self):
        if self.cpus:
            try:
                self.old = os.sched_getaffinity(0)
                allowed = self.cpus & self.old
                if allowed:
                    os.sched_setaffinity(0, allowed)
                else:
                    self.old = None
            except Exception:
                self.old = None
        return self

    def __exit__(self, *exc):
        if self.old is not None:
            try:
                os.sched_setaffinity(0, self.old)
            except Exception:
                pass
        return False


class Engine:
    def __init__(self, device=None, nstreams: int = 1, gram_mode: int = None):
        if not torch.cuda.is_available():
            raise RuntimeError("cpb200: no CUDA device visible; the solver has no CPU path")
        self.ffi, self.lib = _cabi.load()
        if device is None:
            device = torch.cuda.current_device()
        self.device = torch.device("cuda", device if isinstance(device, int) else torch.device(device).index or 0)
        if gram_mode is None:  # tensor cores by default; CPB200_GRAM=fp64 selects the exact-product DMMA mode
            gram_mode = GRAM_FP64 if os.environ.get("CPB200_GRAM", "tc").lower() == "fp64" else GRAM_3XTF32
        self.gram_mode = gram_mode
        self._handles = []
        self.streams = []
        with torch.cuda.device(self.device):
            for i in range(max(1, nstreams)):
                hp = self.ffi.new("cp_handle_t*")
                _cabi.check(self.lib.cp_create(hp, self.device.index))
                self._handles.append(hp[0])
                # The pipeline hands its most expensive problems to the first slots: the first half of the slots runs
                # one level higher.  Priorities only order CTAs that are not yet resident, so they matter little when
                # the step is bound by FP64 throughput.
                prio = -2 if i < nstreams // 2 else -1  # 0 is left to the deferred-Gram stream
                self.streams.append(torch.cuda.Stream(self.device, priority=prio) if nstreams > 1 else None)
        self._tls = threading.local()   # current (handle, stream) slot of each host thread (use_slot)
        self._lock = threading.Lock()
        self.launches = 0  # libcpb200 calls issued (each launches >= 1 kernel)
        self._pinned = {}   # (key, shape, dtype) -> page-locked host buffer, allocated once (cudaHostAlloc is slow)
        self._staging = {}  # (key, shape, dtype) -> device staging buffer for maps that are cheaper to DMA whole
        self._xfer = None   # (zero-copy gather stream, DMA stream) of the host-resident input path
        self._aux = None    # (handle, lowest-priority stream) of the deferred full Grams (select_channels_async)

    # ------------------------------------------------------------------ plumbing
    def close(self):
        for h in self._handles:
            self.lib.cp_destroy(h)
        self._handles = []
        if self._aux is not None:
            self.lib.cp_destroy(self._aux[0])
            self._aux = None

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def pinned(self, key, shape, dtype):
        """Engine-owned page-locked host buffer, reused across calls (contents valid until the next call that
        asks for the same key)."""
        k = (key, tuple(shape), dtype)
        t = self._pinned.get(k)
        if t is None:
            with numa_local(self.device.index if self.device.index is not None else 0):
                t = self._pinned[k] = torch.empty(tuple(shape), dtype=dtype, pin_memory=True)
        return t

    def _ring(self):
        """Rotating index for small pinned staging buffers: a buffer is rewritten by the host only 256 calls
        after the asynchronous copy that read it was enqueued (every step synchronises on each layer's search)."""
        with self._lock:
            self._seq = (getattr(self, "_seq", -1) + 1) % 256
            return self._seq

    def staging(self, key, shape, dtype=torch.float32):
        k = (key, tuple(shape), dtype)
        t = self._staging.get(k)
        if t is None:
            t = self._staging[k] = torch.empty(tuple(shape), dtype=dtype, device=self.device)
        return t

    def xfer_streams(self):
        if self._xfer is None:
            self._xfer = (torch.cuda.Stream(self.device), torch.cuda.Stream(self.device))
        return self._xfer

    def use_slot(self, i: int):
        """Select which (handle, stream) pair subsequent calls OF THE CALLING THREAD use (the selection is
        thread-local: pruner.prune_layers issues the reconstructions of different layers from worker threads)."""
        self._tls.cur = i % len(self._handles)
        return self.streams[self._tls.cur]

    def slot_lock(self, i: int):
        """Lock of slot i's (handle, stream) pair: a handle's scratch is reused by every call in stream order, so two
        host threads must not interleave their launches on one slot."""
        with self._lock:
            if not hasattr(self, "_slot_locks"):
                self._slot_locks = [threading.Lock() for _ in self._handles]
        return self._slot_locks[i % len(self._handles)]

    @property
    def _cur(self):
        return getattr(self._tls, "cur", 0)

    @property
    def h(self):
        over = getattr(self._tls, "handle", None)
        return over if over is not None else self._handles[self._cur]

    def aux_slot(self):
        """(handle, stream) for work that may run in the shadow of the channel searches: the lowest stream priority, its
        own handle (scratch), created on first use."""
        if self._aux is None:
            with torch.cuda.device(self.device):
                hp = self.ffi.new("cp_handle_t*")
                _cabi.check(self.lib.cp_create(hp, self.device.index))
                self._aux = (hp[0], torch.cuda.Stream(self.device, priority=0))
        return self._aux

    def _s(self):
        return self.ffi.cast("void*", torch.cuda.current_stream(self.device).cuda_stream)

    def _p(self, t, ctype):
        if t is None:
            return self.ffi.NULL
        if not t.is_cuda:
            # pinned (page-locked) host memory is mapped into the device address space under UVA: kernels may
            # read it in place over PCIe -- used by the sparse gathers, which touch a small part of each map
            assert t.is_pinned(), "host tensors must be pinned to be read by a kernel"
        else:
            assert t.device == self.device, "tensor must live on %s" % self.device
        return self.ffi.cast(ctype, t.data_ptr())

    def _call(self, rc):
        self.launches += 1
        _cabi.check(rc)

    def empty(self, *shape, dtype=torch.float64):
        return torch.empty(*shape, dtype=dtype, device=self.device)

    # ------------------------------------------------------------------ kernels
    def patch_gather(self, fmap, randx, randy, B, P, k, pad, stride, relu=None, layout="nchw", out=None, dilation=1,
                     transposed=False, act=None, act_param=None, in_scale=None, in_shift=None):
        """fmap: (nbatch*B, c, H, W) [nchw] or (nbatch*B, H, W, c) [nhwc], float32 / bfloat16 / float16, on device
        or in pinned host memory (read in place over PCIe); randx/randy: (nbatch, P) int32 on device.  Returns X (nbatch*P*B, c*kh*kw)
        fp32 -- 16-bit maps are widened exactly, so X equals the X of fmap.float().
        k, pad, stride, dilation: an int or an (h, w) pair, with the meaning of torch.nn.Conv2d's arguments (pad: the
        top / left padding; the sampled points already respect the output size).  Columns are in F.unfold's order.
        All ints with dilation 1 is the reference's window, which must be odd (an even square kernel is (k, k)).
        transposed: the window of torch.nn.ConvTranspose2d (k, pad = padding, stride, dilation as it takes them; fmap
        its input map, the points in its output map; cp_patch_gather_conv_transpose).  Then X @
        weight.transpose(0, 1).reshape(n, -1).T is the layer's output at the points, minus its bias.
        relu: True (the default) or False, the ReLU of the reference's VGG maps.  act, act_param, in_scale, in_shift
        instead: the consumer's input transform of a Conv-BN-activation network whose map is the producer's raw conv
        output (input_transform; cp_patch_gather_act).  relu and act exclude each other."""
        geo = _gather_map(fmap, B, layout, False)
        (kh, kw), (ph, pw), (sh, sw), (dh, dw) = (conv_pair(v) for v in (k, pad, stride, dilation))
        xf = input_transform(relu, act, act_param, in_scale, in_shift, geo[3][0], self.device)
        if xf is not None:
            window = (1, kh, kw, 0, ph, pw, 1, sh, sw, 1, dh, dw)
            return self._patch_gather_act(geo, fmap, (None, randx, randy), B, P, kh * kw, window, transposed, xf, out)
        relu = relu is None or relu if act is None else act == "relu"
        if transposed:
            fn, window = self.lib.cp_patch_gather_conv_transpose, (kh, kw, ph, pw, sh, sw, dh, dw)
        elif all(isinstance(v, (int, np.integer)) for v in (k, pad, stride, dilation)) and dilation == 1:
            fn, window = self.lib.cp_patch_gather_typed, (kh, ph, sh)
        else:
            fn, window = self.lib.cp_patch_gather_conv, (kh, kw, ph, pw, sh, sw, dh, dw)
        return self._patch_gather(fn, geo, fmap, (randx, randy), B, P, kh * kw, window, relu, out)

    def point_gather(self, fmap, randx, randy, B, P, layout="nchw", out=None):
        """Y (nbatch*P*B, n) fp32 at the sampled points of fmap (float32 / bfloat16 / float16, widened exactly)."""
        geo = _gather_map(fmap, B, layout, False)
        return self._point_gather(self.lib.cp_point_gather_typed, geo, fmap, (randx, randy), B, P, out)

    def patch_gather3d(self, fmap, randt, randx, randy, B, P, k, pad, stride, relu=None, layout="ncdhw", out=None,
                       dilation=1, transposed=False, act=None, act_param=None, in_scale=None, in_shift=None):
        """fmap: (nbatch*B, c, D, H, W) [ncdhw] or (nbatch*B, D, H, W, c) [ndhwc, channels_last_3d], float32 /
        bfloat16 / float16, on device or in pinned host memory (read in place); randt/randx/randy: (nbatch, P) int32 on
        device, the sampled output points (t, x, y).  Returns X (nbatch*P*B, c*kt*kh*kw) fp32, 16-bit maps widened
        exactly.  k, pad, stride, dilation: an int or a (t, h, w) triple, with the meaning of torch.nn.Conv3d's
        arguments (pad: the front / top / left padding).  Columns are in Conv3d.weight.reshape(n, -1)'s order.
        transposed: the window of torch.nn.ConvTranspose3d, as for patch_gather (cp_patch_gather_conv_transpose3d).
        relu, act, act_param, in_scale, in_shift: as for patch_gather."""
        geo = _gather_map(fmap, B, layout, True)
        (kt, kh, kw), (pt, ph, pw), (st, sh, sw), (dt, dh, dw) = (conv_triple(v) for v in (k, pad, stride, dilation))
        window = (kt, kh, kw, pt, ph, pw, st, sh, sw, dt, dh, dw)
        xf = input_transform(relu, act, act_param, in_scale, in_shift, geo[3][0], self.device)
        if xf is not None:
            return self._patch_gather_act(geo, fmap, (randt, randx, randy), B, P, kt * kh * kw, window, transposed, xf,
                                          out)
        fn = self.lib.cp_patch_gather_conv_transpose3d if transposed else self.lib.cp_patch_gather_conv3d
        relu = relu is None or relu if act is None else act == "relu"
        return self._patch_gather(fn, geo, fmap, (randt, randx, randy), B, P, kt * kh * kw, window, relu, out)

    def point_gather3d(self, fmap, randt, randx, randy, B, P, layout="ncdhw", out=None):
        """Y (nbatch*P*B, n) fp32 at the sampled points (t, x, y) of a Conv3d output map (nbatch*B, n, To, Ho, Wo)
        [ncdhw] or (nbatch*B, To, Ho, Wo, n) [ndhwc], float32 / bfloat16 / float16 widened exactly."""
        geo = _gather_map(fmap, B, layout, True)
        return self._point_gather(self.lib.cp_point_gather3d, geo, fmap, (randt, randx, randy), B, P, out)

    def _patch_gather(self, fn, geo, fmap, points, B, P, taps, window, relu, out):
        """patch_gather and patch_gather3d from here on: fn is the C entry, geo what _gather_map found, points the
        (randx, randy) or (randt, randx, randy) tensors, window the entry's geometry arguments."""
        dt, lay, nbatch, dims = geo
        assert fmap.shape[0] % B == 0
        for r in points:
            assert r.dtype == torch.int32 and r.numel() == nbatch * P and r.is_contiguous()
        rows, K = nbatch * P * B, dims[0] * taps
        if out is None:
            out = self.empty(rows, K, dtype=torch.float32)
        assert out.shape == (rows, K) and out.dtype == torch.float32 and out.stride(1) == 1
        self._call(fn(self.h, self._p(fmap, "const void*"), dt, nbatch, B, *dims, lay,
                      *[self._p(r, "const int32_t*") for r in points], P, *window, int(bool(relu)),
                      self._p(out, "float*"), out.stride(0), self._s()))
        return out

    def _patch_gather_act(self, geo, fmap, points, B, P, taps, window, transposed, xf, out):
        """patch_gather and patch_gather3d through cp_patch_gather_act: points (randt or None, randx, randy), window
        the 12 values kt ... dil_w, xf what input_transform returned."""
        dt, lay, nbatch, dims = geo
        if len(dims) == 3:
            dims = (dims[0], 1) + tuple(dims[1:])  # (c, D = 1, H, W)
        assert fmap.shape[0] % B == 0
        for r in points[1:] if points[0] is None else points:
            assert r.dtype == torch.int32 and r.numel() == nbatch * P and r.is_contiguous()
        rows, K = nbatch * P * B, dims[0] * taps
        if out is None:
            out = self.empty(rows, K, dtype=torch.float32)
        assert out.shape == (rows, K) and out.dtype == torch.float32 and out.stride(1) == 1
        act, slope, scale, shift = xf
        self._call(self.lib.cp_patch_gather_act(
            self.h, self._p(fmap, "const void*"), dt, nbatch, B, *dims, lay,
            *[self._p(r, "const int32_t*") for r in points], P, *window, int(bool(transposed)), act, slope,
            self._p(scale, "const float*"), self._p(shift, "const float*"), self._p(out, "float*"), out.stride(0),
            self._s()))
        return out

    def _point_gather(self, fn, geo, fmap, points, B, P, out):
        """point_gather and point_gather3d from here on (arguments as for _patch_gather)."""
        dt, lay, nbatch, dims = geo
        rows, n = nbatch * P * B, dims[0]
        if out is None:
            out = self.empty(rows, n, dtype=torch.float32)
        assert out.shape == (rows, n) and out.dtype == torch.float32 and out.stride(1) == 1
        self._call(fn(self.h, self._p(fmap, "const void*"), dt, nbatch, B, *dims, lay,
                      *[self._p(r, "const int32_t*") for r in points], P, self._p(out, "float*"), out.stride(0),
                      self._s()))
        return out

    def gram(self, X, Y=None, y_bias=None, rows=None, want_G=True, want_B=True, want_sums=True, want_yy=False,
             mode=None):
        """Sufficient statistics of (X, Y) (optionally over gathered rows).
        Returns dict with G (K,K), B (K,n), sx (K), sy (n), yy (1) as fp64 device tensors."""
        assert X.dtype == torch.float32 and X.dim() == 2 and X.stride(1) == 1
        N, K = X.shape
        out = {}
        n = 0
        y_dt = 0
        if Y is not None:
            assert Y.dim() == 2 and Y.shape[0] == N and Y.stride(1) == 1
            assert Y.dtype in (torch.float32, torch.float64)
            y_dt = 0 if Y.dtype == torch.float32 else 1
            n = Y.shape[1]
        if rows is not None:
            assert rows.dtype == torch.int32 and rows.is_contiguous()
        G = self.empty(K, K) if want_G else None
        Bxy = self.empty(K, n) if (want_B and Y is not None) else None
        sx = self.empty(K) if want_sums else None
        sy = self.empty(n) if (want_sums and Y is not None) else None
        yy = self.empty(1) if (want_yy and Y is not None) else None
        self._call(self.lib.cp_gram(self.h, self._p(X, "const float*"), N, K, X.stride(0),
                                    self._p(Y, "const void*"), y_dt, n, Y.stride(0) if Y is not None else 0,
                                    self._p(y_bias, "const float*"), self._p(rows, "const int32_t*"),
                                    rows.numel() if rows is not None else 0, self._p(G, "double*"),
                                    self._p(Bxy, "double*"), self._p(sx, "double*"), self._p(sy, "double*"),
                                    self._p(yy, "double*"), self.gram_mode if mode is None else mode, self._s()))
        out.update(G=G, B=Bxy, sx=sx, sy=sy, yy=yy, N=N, K=K, n=n, mode=self.gram_mode if mode is None else mode)
        return out

    def gemm_tc_split(self, A, B, C=None, alpha=1.0, beta=0.0, lower=False, b_nc=False):
        """C = alpha A B' + beta C on the tensor cores in 22-bit split precision (cp_gemm_tc_split): A (M, R), B (Nn, R)
        -- or (R, Nn) with b_nc -- C (M, Nn), fp64 device tensors with unit inner stride."""
        assert A.dtype == B.dtype == torch.float64 and A.stride(1) == 1 and B.stride(1) == 1
        M, R = A.shape
        Nn = B.shape[1] if b_nc else B.shape[0]
        assert (B.shape[0] if b_nc else B.shape[1]) == R
        if C is None:
            assert beta == 0.0
            C = self.empty(M, Nn)
        assert C.shape == (M, Nn) and C.dtype == torch.float64 and C.stride(1) == 1
        self._call(self.lib.cp_gemm_tc_split(self.h, M, Nn, R, float(alpha), self._p(A, "const double*"), A.stride(0),
                                             self._p(B, "const double*"), B.stride(0), float(beta), self._p(C, "double*"),
                                             C.stride(0), (1 if lower else 0) | (2 if b_nc else 0), self._s()))
        return C

    def ls_tensor_cores(self, enable):
        """Bulk products of the following ls_solve / ls_factor / ls_resolve calls on the tensor cores (cp_ls_tensor_cores)."""
        self._call(self.lib.cp_ls_tensor_cores(self.h, 1 if enable else 0))

    def gram_profile(self, enable=True):
        """CUDA events around the tensor-core GEMM launch of every following gram() on this engine's handle."""
        self._call(self.lib.cp_gram_profile(self.h, 1 if enable else 0))

    def gram_kernel_ms(self):
        """Elapsed time (ms) of the tensor-core GEMM launch of the last gram() (needs gram_profile(True))."""
        ms = self.ffi.new("float*")
        self._call(self.lib.cp_gram_kernel_ms(self.h, ms))
        return float(ms[0])

    def lasso_build(self, gs, gw, W2m, c, k2, S):
        """gs: gram over sampled rows (with yy); gw: gram of W2 viewed (n, K); W2m: (n, K) fp32."""
        n = W2m.shape[0]
        ldq = c + (c & 1)  # even leading dimension: 16-byte aligned rows for the selection kernel
        Q = self.empty(c, ldq)
        qv = self.empty(c)
        yn2 = self.empty(1)
        self._call(self.lib.cp_lasso_build(self.h, self._p(gs["G"], "const double*"), self._p(gs["B"], "const double*"),
                                           self._p(gs["sx"], "const double*"), self._p(gs["sy"], "const double*"),
                                           self._p(gs["yy"], "const double*"), self._p(gw["G"], "const double*"),
                                           self._p(gw["sx"], "const double*"), self._p(W2m, "const float*"), c, k2, n,
                                           S, self._p(Q, "double*"), ldq, self._p(qv, "double*"),
                                           self._p(yn2, "double*"), self._s()))
        return Q[:, :c], qv, yn2

    def lasso_select(self, Q, qv, yn2, m, rank, lbound, rbound, right0, seeds, tol=1e-4, max_iter=1000):
        c = Q.shape[0]
        if Q.stride(1) != 1 or Q.stride(0) % 2 or Q.data_ptr() % 16:
            Qp = torch.zeros(c, c + (c & 1), dtype=torch.float64, device=self.device)
            Qp[:, :c] = Q
            Q = Qp[:, :c]
        if isinstance(seeds, torch.Tensor) and seeds.is_cuda:
            assert seeds.dtype == torch.int32 and seeds.is_contiguous()
            seeds_d = seeds
        else:
            # staged through an engine-owned pinned buffer: a pageable H2D copy would make torch synchronise
            # the stream, i.e. block the host until everything queued on this layer's stream has run
            sh = np.asarray(seeds, dtype=np.int64).astype(np.int32)
            pin = self.pinned(("seeds", self._ring()), sh.shape, torch.int32)
            pin.numpy()[...] = sh
            seeds_d = pin.to(self.device, non_blocking=True)
        maxp = seeds_d.numel()
        idxs = self.empty(c, dtype=torch.uint8)
        coef = self.empty(c)
        scalars = self.empty(4)
        plog = torch.zeros(maxp, 4, dtype=torch.float64, device=self.device)
        self._call(self.lib.cp_lasso_select(self.h, self._p(Q, "const double*"), Q.stride(0),
                                            self._p(qv, "const double*"),
                                            self._p(yn2, "const double*"), c, float(m), int(rank), float(lbound),
                                            float(rbound), float(right0), float(tol), int(max_iter),
                                            self._p(seeds_d, "const uint32_t*"), maxp, self._p(idxs, "uint8_t*"),
                                            self._p(coef, "double*"), self._p(scalars, "double*"),
                                            self._p(plog, "double*"), self._s()))
        return LassoResult(idxs, coef, scalars, plog, seeds_d)

    def ls_solve(self, g, sel_cols):
        """Centred normal-equation LS on columns ``sel_cols`` (int32 device tensor, ascending; None = all).
        Returns (W (n, Ksel) fp64, b (n,) fp64, info (1,) int32, stat (1,) fp64) on device; stat is the smallest
        pivot / original-diagonal ratio of the Cholesky (conditioning signal, see include/cpb200.h)."""
        Ks = sel_cols.numel() if sel_cols is not None else g["K"]
        n = g["n"]
        W = self.empty(n, Ks)
        b = self.empty(n)
        info = torch.zeros(1, dtype=torch.int32, device=self.device)
        stat = self.empty(1)
        self.ls_tensor_cores(g.get("mode", GRAM_FP64) != GRAM_FP64)
        self._call(self.lib.cp_ls_solve(self.h, self._p(g["G"], "const double*"), self._p(g["B"], "const double*"),
                                        self._p(g["sx"], "const double*"), self._p(g["sy"], "const double*"),
                                        g["N"], g["K"], n, self._p(sel_cols, "const int32_t*"), Ks,
                                        self._p(W, "double*"), self._p(b, "double*"), self._p(info, "int32_t*"),
                                        self._p(stat, "double*"), self._s()))
        return W, b, info, stat

    def ls_solve_dual(self, X, Y, y_bias, sel_cols):
        N, K = X.shape
        n = Y.shape[1]
        Ks = sel_cols.numel() if sel_cols is not None else K
        W = self.empty(n, Ks)
        b = self.empty(n)
        info = torch.zeros(1, dtype=torch.int32, device=self.device)
        stat = self.empty(1)
        self._call(self.lib.cp_ls_solve_dual(self.h, self._p(X, "const float*"), N, K, X.stride(0),
                                             self._p(Y, "const void*"), 0 if Y.dtype == torch.float32 else 1, n,
                                             Y.stride(0), self._p(y_bias, "const float*"),
                                             self._p(sel_cols, "const int32_t*"), Ks, self._p(W, "double*"),
                                             self._p(b, "double*"), self._p(info, "int32_t*"),
                                             self._p(stat, "double*"), self._s()))
        return W, b, info, stat

    def ls_factor(self, g, sel_cols=None):
        """Keeps the Cholesky factor of the centred Gram (columns ``sel_cols``) on the CURRENT handle for
        subsequent ls_resolve calls.  Returns (info (1,) int32, stat (1,) fp64)."""
        Ks = sel_cols.numel() if sel_cols is not None else g["K"]
        info = torch.zeros(1, dtype=torch.int32, device=self.device)
        stat = self.empty(1)
        self.ls_tensor_cores(g.get("mode", GRAM_FP64) != GRAM_FP64)
        self._call(self.lib.cp_ls_factor(self.h, self._p(g["G"], "const double*"), self._p(g["sx"], "const double*"),
                                         g["N"], g["K"], self._p(sel_cols, "const int32_t*"), Ks,
                                         self._p(info, "int32_t*"), self._p(stat, "double*"), self._s()))
        return info, stat

    def ls_resolve(self, Bxy, sx, sy, sel_cols=None, Ks=None, accumulate_into=None):
        """Solve against the factor kept on the CURRENT handle (ls_factor, or the last ls_solve): Bxy (K, n) = X'U,
        sy (n,) = 1'U.  Returns (W (n, Ksel), b (n,)); with accumulate_into=(W, b) the solution is ADDED to those."""
        n = Bxy.shape[1]
        Ks = (sel_cols.numel() if sel_cols is not None else Bxy.shape[0]) if Ks is None else Ks
        if accumulate_into is None:
            W, b, acc = self.empty(n, Ks), self.empty(n), 0
        else:
            (W, b), acc = accumulate_into, 1
            assert W.shape == (n, Ks) and W.is_contiguous() and b.shape == (n,)
        self._call(self.lib.cp_ls_resolve(self.h, self._p(Bxy, "const double*"), self._p(sx, "const double*"),
                                          self._p(sy, "const double*"), n, self._p(sel_cols, "const int32_t*"),
                                          self._p(W, "double*"), self._p(b, "double*"), acc, self._s()))
        return W, b

    def ls_residual(self, X, Y, y_bias, sel_cols, W, b, mode=None):
        """fp32 residual (N, n) of the fit (W, b) on columns sel_cols, computed from the data (cp_ls_residual): prediction
        in fp64 (mode 0) or on the tensor cores (mode 1, default = the engine's Gram mode)."""
        N, K = X.shape
        n = Y.shape[1]
        Ks = sel_cols.numel() if sel_cols is not None else K
        R = self.empty(N, n, dtype=torch.float32)
        self._call(self.lib.cp_ls_residual(self.h, self._p(X, "const float*"), N, K, X.stride(0), self._p(Y, "const void*"),
                                           0 if Y.dtype == torch.float32 else 1, n, Y.stride(0),
                                           self._p(y_bias, "const float*"), self._p(sel_cols, "const int32_t*"), Ks,
                                           self._p(W, "const double*"), self._p(b, "const double*"), self._p(R, "float*"),
                                           R.stride(0), self.gram_mode if mode is None else mode, self._s()))
        return R

    def ls_refine(self, g, X, Y, y_bias, sel_cols, W, b):
        """One step of iterative refinement of (W, b) against the factor the last ls_solve left on this handle:
        residual from the data, its cross products with X on the tensor cores, forward/backward substitution,
        correction added in place.  Removes the error tensor-core statistics put into the solution.  The prediction
        X W' of the residual runs in the statistics' mode: on the tensor cores it is one short persistent launch, and
        it takes 2NK'n flop per layer off the FP64 pipe, the step's scarce resource."""
        R = self.ls_residual(X, Y, y_bias, sel_cols, W, b, mode=g["mode"])
        gr = self.gram(X, R, want_G=False, mode=g["mode"])
        self.ls_resolve(gr["B"], g["sx"], gr["sy"], sel_cols, accumulate_into=(W, b))
        return W, b

    # ------------------------------------------------------------------ data-form LASSO (benchmark kernel)
    def lasso_dataform_build(self, X, W2m, Y, y_bias, samples, c, k2):
        """Materialises the reference's design matrix Z ((S*n) x c, column major fp32) and target y (lib/decompose.py:
        428-437).  Returns (Z as a (c, m) tensor whose rows are the columns of Z, y (m,) fp64)."""
        N, K = X.shape
        n = W2m.shape[0]
        S = samples.numel()
        m = S * n
        Z = self.empty(c, m, dtype=torch.float32)
        y = self.empty(m)
        self._call(self.lib.cp_lasso_dataform_build(self.h, self._p(X, "const float*"), N, K, X.stride(0),
                                                    self._p(W2m, "const float*"), n, c, k2,
                                                    self._p(samples, "const int32_t*"), S, self._p(Y, "const void*"),
                                                    0 if Y.dtype == torch.float32 else 1, Y.stride(0),
                                                    self._p(y_bias, "const float*"), self._p(Z, "float*"), Z.stride(0),
                                                    self._p(y, "double*"), self._s()))
        return Z, y

    def lasso_cd_dataform(self, Z, y, alpha, seed, w=None, tol=1e-4, max_iter=1000):
        """One Lasso.fit in data form (cp_lasso_cd_dataform).  Returns (w (c,), scalars [n_iter, gap, tol, sweeps, checks])."""
        c, m = Z.shape
        if w is None:
            w = torch.zeros(c, dtype=torch.float64, device=self.device)
        out = torch.zeros(8, dtype=torch.float64, device=self.device)
        self._call(self.lib.cp_lasso_cd_dataform(self.h, self._p(Z, "const float*"), Z.stride(0), self._p(y, "const double*"),
                                                 m, c, float(alpha), float(tol), int(max_iter), int(seed) & 0xffffffff,
                                                 self._p(w, "double*"), self._p(out, "double*"), self._s()))
        return w, out

    def dataform_benchmark(self, X, W2m, Y, y_bias, samples, shape, alpha, seed=12345):
        """Times one cold-start data-form fit at ``alpha`` (profiles/sweep_config5.py): bytes of Z streamed per second."""
        Z, y = self.lasso_dataform_build(X, W2m, Y, y_bias, samples, shape.c, shape.k * shape.k)
        self.lasso_cd_dataform(Z, y, alpha, seed)  # warm-up
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        w, out = self.lasso_cd_dataform(Z, y, alpha, seed)
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b)
        o = out.cpu().numpy()
        sweeps, checks = int(o[3]), int(o[4])
        nbytes = 4.0 * Z.shape[0] * Z.shape[1] * (sweeps + checks)  # SURVEY 8(d): 4 m c per sweep (+ per gap check)
        return {"m": int(Z.shape[1]), "c": int(Z.shape[0]), "alpha": alpha, "n_iter": int(o[0]), "sweeps": sweeps,
                "gap_checks": checks, "ms": ms, "stream_gbs": nbytes / (ms / 1e3) / 1e9, "nnz": int((w != 0).sum().item()),
                "algorithmic_bytes": nbytes}

    # ------------------------------------------------------------------ dense fp64 blocks (3C companions)
    def gemm(self, A, B, a_mc=False, b_nc=False, alpha=1.0, beta=0.0, out=None):
        """C[m, nn] = alpha * sum_r a(m, r) b(nn, r) + beta * C   (cp_gemm_f64; fp64 device tensors, unit inner stride)
        a_mc: A is (R, M) else (M, R);  b_nc: B is (R, Nn) else (Nn, R)."""
        assert A.dtype == torch.float64 and B.dtype == torch.float64 and A.dim() == 2 and B.dim() == 2
        assert (A.stride(1) == 1 or A.shape[1] == 1) and (B.stride(1) == 1 or B.shape[1] == 1)
        R, M = (A.shape[0], A.shape[1]) if a_mc else (A.shape[1], A.shape[0])
        Rb, Nn = (B.shape[0], B.shape[1]) if b_nc else (B.shape[1], B.shape[0])
        assert R == Rb, "inner dimensions differ: %d vs %d" % (R, Rb)
        if out is None:
            assert beta == 0.0
            out = self.empty(M, Nn)
        assert out.shape == (M, Nn) and out.dtype == torch.float64 and (out.stride(1) == 1 or Nn == 1)
        self._call(self.lib.cp_gemm_f64(self.h, int(a_mc), int(b_nc), M, Nn, R, float(alpha), self._p(A, "const double*"),
                                        A.stride(0), self._p(B, "const double*"), B.stride(0), float(beta),
                                        self._p(out, "double*"), out.stride(0), self._s()))
        return out

    def mm(self, A, B):
        """A @ B"""
        return self.gemm(A, B, a_mc=False, b_nc=True)

    def mm_nt(self, A, B):
        """A @ B.T"""
        return self.gemm(A, B, a_mc=False, b_nc=False)

    def mm_tn(self, A, B):
        """A.T @ B"""
        return self.gemm(A, B, a_mc=True, b_nc=True)

    def svd(self, F, max_sweeps=40):
        """Thin SVD of a small dense fp64 matrix (m, n) by one-sided Jacobi (cp_svd_jacobi).  Returns (U (m, r),
        s (r,) descending, Vh (r, n)), r = min(m, n) -- the convention of scipy.linalg.svd(full_matrices=False)."""
        assert F.dtype == torch.float64 and F.dim() == 2
        m, n = F.shape
        if m < n:  # orthogonalise the columns of the taller orientation
            U, s, Vh = self.svd(F.T.contiguous(), max_sweeps)
            return Vh.T.contiguous(), s, U.T.contiguous()
        Ft = F.T.contiguous()
        Wt = self.empty(n, n)
        sigma = self.empty(n)
        sweeps = self.ffi.new("int32_t*")
        tol = float(np.sqrt(m)) * 2.220446049250313e-16
        self._call(self.lib.cp_svd_jacobi(self.h, self._p(Ft, "double*"), m, n, Ft.stride(0), self._p(Wt, "double*"),
                                          Wt.stride(0), self._p(sigma, "double*"), 1, tol, max_sweeps, sweeps,
                                          self._s()))
        if sweeps[0] >= max_sweeps:
            raise np.linalg.LinAlgError("Jacobi SVD did not converge in %d sweeps" % max_sweeps)
        order = torch.argsort(sigma, descending=True, stable=True)
        return Ft[order].T.contiguous(), sigma[order].contiguous(), Wt[order].contiguous()

    def solve_relu(self, RUraw, bias, Z, lam, want_mean=False):
        """U = solve_relu(RUraw + bias, Z, lam) (lib/decompose.py:51-59), optional column means of U."""
        N, n = RUraw.shape
        U = self.empty(N, n)
        mean = self.empty(n) if want_mean else None
        self._call(self.lib.cp_solve_relu(self.h, self._p(RUraw, "const double*"), RUraw.stride(0),
                                          self._p(bias, "const double*"), self._p(Z, "const double*"), Z.stride(0),
                                          float(lam), self._p(U, "double*"), U.stride(0), N, n, self._p(mean, "double*"),
                                          self._s()))
        return (U, mean) if want_mean else U

    def colstats(self, X, scale=1.0, centre=False):
        """(scale * column sums, X - that) of an fp64 matrix (cp_colstats_f64); centre with scale = 1/N."""
        N, n = X.shape
        assert X.dtype == torch.float64 and X.stride(1) == 1
        cs = self.empty(n)
        Xc = self.empty(N, n) if centre else None
        self._call(self.lib.cp_colstats_f64(self.h, self._p(X, "const double*"), X.stride(0), N, n, float(scale),
                                            self._p(cs, "double*"), self._p(Xc, "double*"), n, self._s()))
        return (cs, Xc) if centre else cs

    # ------------------------------------------------------------------ composite: one layer problem
    def select_channels_async(self, X, W2m, Y, y_bias, samples, c, k2, rank, rank_tol, right0, seeds):
        """Everything of decompose.dictionary up to (and including) the alpha search, enqueued
        without host synchronisation.  Returns (g_full, LassoResult)."""
        n = W2m.shape[0]
        S = samples.numel()
        # The search needs only the channel-space statistics (Q from the sampled rows and W2); the full Gram feeds the
        # reconstruction.  In the pipeline (one stream per layer) it is therefore enqueued AFTER the search, on a
        # lowest-priority stream with its own handle: the full-GPU launch no longer delays the start of this and of
        # every later layer's single-SM search, it runs in their shadow.
        defer = self.streams[0] is not None
        if defer:
            cur = torch.cuda.current_stream(self.device)
            ev_x = torch.cuda.Event()
            ev_x.record(cur)  # X and Y are complete here (recorded BEFORE the search is enqueued on this stream)
        g_full = None if defer else self.gram(X, Y, y_bias=y_bias)
        g_s = self.gram(X, Y, y_bias=y_bias, rows=samples, want_yy=True, mode=GRAM_FP64)
        g_w = self.gram(W2m, None, want_B=False, mode=GRAM_FP64)
        Q, qv, yn2 = self.lasso_build(g_s, g_w, W2m, c, k2, S)
        lbound, rbound = window(rank, rank_tol)
        res = self.lasso_select(Q, qv, yn2, float(S) * n, rank, lbound, rbound, right0, seeds)
        if defer:
            ah, astream = self.aux_slot()
            self._tls.handle = ah
            try:
                with torch.cuda.stream(astream):
                    astream.wait_event(ev_x)
                    g_full = self.gram(X, Y, y_bias=y_bias)
                    ready = torch.cuda.Event()
                    ready.record(astream)
            finally:
                self._tls.handle = None
            for t in (X, Y, y_bias):
                if t is not None:
                    t.record_stream(astream)
            for key in ("G", "B", "sx", "sy"):
                if g_full.get(key) is not None:
                    g_full[key].record_stream(cur)
            g_full["ready"] = ready
        return g_full, res

    def _cols_device(self, idxs_host, k2, K):
        sel = np.flatnonzero(idxs_host)
        cols = (sel[:, None] * k2 + np.arange(k2)[None, :]).reshape(-1).astype(np.int32)
        pin = self.pinned(("cols", self._ring()), (K,), torch.int32)  # no pageable (synchronising) copy
        pin.numpy()[:cols.size] = cols
        return pin[:cols.size].to(self.device, non_blocking=True)

    def reconstruct_async(self, g_full, X, Y, y_bias, idxs_host, k2):
        """LS on the surviving channels (device outputs; no host sync).  Returns (W, b, info, stat)."""
        if g_full.get("ready") is not None:  # full Gram enqueued on the deferred-Gram stream
            torch.cuda.current_stream(self.device).wait_event(g_full["ready"])
        cols_d = self._cols_device(idxs_host, k2, g_full["K"])
        if not ls_dual(g_full["N"], idxs_host, k2):
            W, b, info, stat = self.ls_solve(g_full, cols_d)
            if g_full["mode"] != GRAM_FP64:
                # statistics from the 3xTF32 Gram carry ~4e-7 relative error, which the conditioning of a wide layer
                # amplifies by orders of magnitude in W and more in b: one refinement step against
                # the same factor, with the residual taken from the data, restores fp64-level accuracy
                self.ls_refine(g_full, X, Y, y_bias, cols_d, W, b)
            return W, b, info, stat
        return self.ls_solve_dual(X, Y, y_bias, cols_d)

    def reconstruct_exact_async(self, X, Y, y_bias, idxs_host, k2):
        """The same solve from exact-product fp64 statistics (the slow path of the conditioning policy)."""
        g = self.gram(X, Y, y_bias=y_bias, mode=GRAM_FP64)
        return self.reconstruct_async(g, X, Y, y_bias, idxs_host, k2)

    def reconstruct_truncated(self, X, Y, y_bias, idxs_host, k2):
        """Minimum-norm least squares with the reference's rank cut-off, for systems the Cholesky flags as numerically
        rank deficient: LinearRegression.fit -> scipy.linalg.lstsq(Xc, Yc, cond=1e-6) (gelsd, sklearn _base.py:752)
        drops singular values below 1e-6 sigma_max.  Here: one-sided Jacobi SVD of the centred selected columns
        (cp_svd_jacobi works on X itself, so small singular values are resolved like gelsd resolves them), then
        W = V diag(1/s) U' Yc over the kept ones.  Slow path (O(10) sweeps over N x K'), rare."""
        cols = self._cols_device(idxs_host, k2, X.shape[1]).long()
        N = X.shape[0]
        Xs = X[:, cols].to(torch.float64).contiguous()
        xm, Xc = self.colstats(Xs, 1.0 / N, centre=True)
        Yd = Y.to(torch.float64)
        if y_bias is not None:
            Yd = Yd - y_bias.to(torch.float64)[None, :]
        ym, Yc = self.colstats(Yd.contiguous(), 1.0 / N, centre=True)
        U, s, Vh = self.svd(Xc)
        keep = s > 1e-6 * s[0]
        inv = torch.where(keep, 1.0 / torch.where(keep, s, torch.ones_like(s)), torch.zeros_like(s))
        UtY = self.mm_tn(U, Yc)                                   # (r, n)
        W = self.mm_tn((inv[:, None] * UtY).contiguous(), Vh)    # (n, K') = (V diag(1/s) U' Yc)'
        b = ym - self.mm(W, xm[:, None].contiguous())[:, 0]
        return W, b, int(keep.sum().item())


def ls_dual(N, idxs_host, k2):
    """True when the K' = kept channels * k2 selected columns leave fewer than K' degrees of freedom in the N centred
    rows: the normal equations are singular by construction, so the solve works on the data (cp_ls_solve_dual)."""
    return N - 1 < int(np.count_nonzero(idxs_host)) * k2


def settle_ls(eng, X, Y, y_bias, idxs_host, k2, mode, fail, ratio):
    """Acceptance policy of a reconstruct_async solve, given its Cholesky status ``fail`` and pivot ratio ``ratio``
    (read back on the host), in statistics mode ``mode``.  Work it adds runs on the current stream.
      - fp64 statistics or the dual path: accepted unless the Cholesky failed ('singular').
      - tensor-core statistics: accepted while the Cholesky succeeded and ratio >= LS_RATIO_MIN (NaN fails);
        otherwise re-solved from exact-product fp64 statistics ('redo->ok', or singular when that fails too).
      - singular (a pivot below 1e-12 of its diagonal, even with exact statistics): numerically rank deficient.  The
        reference's gelsd drops singular values below 1e-6 sigma_max (cond=1e-6, sklearn _base.py:752) and returns
        the minimum-norm solution; reconstruct_truncated applies that rule through the SVD of the data: 'truncated',
        with the rank it kept.
    Returns (W, b, record): W and b replace the first solve's, or are None when it stands; record holds
    pivot_ratio, verdict ('ok' | 'redo->ok' | 'truncated') and, where they apply, pivot_ratio_exact and rank."""
    rec = {"pivot_ratio": ratio}
    if mode == GRAM_FP64 or ls_dual(X.shape[0], idxs_host, k2):
        verdict = "singular" if fail else "ok"
    else:
        verdict = "redo" if fail or not (ratio >= LS_RATIO_MIN) else "ok"
    W = b = None
    if verdict == "redo":
        W, b, info, stat = eng.reconstruct_exact_async(X, Y, y_bias, idxs_host, k2)
        fail, rec["pivot_ratio_exact"] = int(info.cpu()[0]), float(stat.cpu()[0])
        verdict = "singular" if fail else "redo->ok"
    if verdict == "singular":
        W, b, rec["rank"] = eng.reconstruct_truncated(X, Y, y_bias, idxs_host, k2)
        verdict = "truncated"
    rec["verdict"] = verdict
    return W, b, rec


def window(rank, rank_tol):
    """Acceptance window of the alpha search, reference lib/decompose.py:492-501."""
    lbound = rank
    if rank_tol >= 1:
        rbound = rank + rank_tol
    else:
        rbound = rank + rank_tol * rank
        if rank_tol == .2:
            lbound = rank + 0.1 * rank
            rbound = rank + 0.2 * rank
    return lbound, rbound


_ENGINE = None


def get_engine(**kw) -> Engine:
    """Process-wide engine on the current CUDA device."""
    global _ENGINE
    if _ENGINE is None:
        _ENGINE = Engine(**kw)
    return _ENGINE


def reset_engine():
    global _ENGINE
    if _ENGINE is not None:
        _ENGINE.close()
    _ENGINE = None
