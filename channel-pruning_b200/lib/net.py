"""Drop-in for the pruning-path methods of the reference's ``lib.net.Net`` -- without Caffe.

The reference's ``Net`` wraps a pycaffe handle; the hot path only needs (a) the blobs of a
forward pass, (b) conv hyper-parameters, (c) weights.  Here a ``Net`` is built from a plain
list of layer specs + a weight dict + a *feature provider* ``forward(net, data) -> {blob:
CUDA tensor (B, C, H, W)}`` (``ConvStackForward`` below runs a sequential conv/ReLU/pool stack
with torch.nn.functional, standing in for Caffe's GPU forward, which is also library code in
the reference).  Methods keep the reference's names, arguments and return conventions:

  extract_features(names, nBatches=None, points_dict=None, save=False)   lib/net.py:368-532
  extract_XY(X, Y, DEBUG=False, w1=None)                                 lib/net.py:534-684
  freeze_images(check_exist=False, convs=None)                           lib/net.py:749-800
  load_frozen(DEBUG=False, feats_dict=None, points_dict=None)            lib/net.py:839-876
  dictionary_kernel(X_name, weights, d_prime, Y_name, Y, DEBUG=0)        lib/net.py:1685-1735
  R3() -> (WPQ, new_pt)    spatial + channel decomposition + pruning     lib/net.py:1292-1471
  combineHP(WPQ, new_pt), layercomputation(...), computation(...)        lib/net.py:1473-1504, 1049-1081
      (module-level: they work on the WPQ / topology dictionaries R3 returns -- there is no prototxt here)

The gathers run on the device (cp_point_gather / cp_patch_gather); sampled points come from the
numpy global RNG with the reference's call sequence, so a seeded run draws the same points.
Data types (SURVEY.md 8a-a9) follow the reference: ``feats_dict{layer: float64 (N, n)}``,
``points_dict{'nPointsPerLayer', 'nBatches', 'data', 'label', (batch, 0): images, (batch, 1): labels,
(batch, layer, 'randx'|'randy'): int[P]}``, the frozen pickle ``[feats_dict, points_dict]`` (protocol 4),
``WPQ{layer or (layer, 0|1): ndarray}``, ``selection{conv: bool[c]}``.
"""
from __future__ import annotations

import os
import pickle

import numpy as np
import torch
import torch.nn.functional as F

from . import cfgs
from .cfgs import c as dcfgs
from .decompose import ITQ_decompose, VH_decompose, _dictionary_device
from ..engine import conv_pair, get_engine


def underline(*parts):
    """lib/utils.py:52-54"""
    return '_'.join(str(p) for p in parts)


class ConvSpec:
    """What the reference reads from the prototxt for a Convolution layer (net.py:542-553).
    kernel_size, pad, stride and dilation are ints or (h, w) pairs with the meaning of torch.nn.Conv2d's arguments
    (groups == 1): rectangular kernels such as Inception's 1 x 7, per-axis padding and dilated layers such as those
    of DeepLabV3's backbone.  The reference's layers are square, odd and undilated."""

    def __init__(self, name, bottom, num_output, kernel_size=3, pad=1, stride=1, pool_after=False, dilation=1):
        self.name, self.bottom = name, bottom
        self.num_output = num_output
        self.kernel_size, self.pad, self.stride, self.dilation = kernel_size, pad, stride, dilation
        self.pool_after = pool_after  # a 2x2/2 max-pool follows the ReLU (VGG)

    @property
    def kernel_hw(self):
        """(kh, kw)"""
        return conv_pair(self.kernel_size)


class ConvStackForward:
    """Feature provider for a sequential conv -> ReLU (-> pool) stack.  Blob names follow the
    reference after ``seperateConvReLU`` (net.py:1228): blob ``<conv>`` holds the PRE-ReLU conv
    output; the next conv's bottom is ``<conv>_relu`` or ``pool<k>`` (post-ReLU).
    ``images_by_batch(batch) -> (B, 3, H, W)`` supplies the un-frozen batches (Caffe's data layer);
    frozen runs pass the stored images in (net.py:446-447).
    ``dtype``: the type the stack runs in (images and weights are rounded to it; a bfloat16 or float16 forward is
    what autocast hands over on an H100).  The blobs stay in that type: the gathers read 16-bit maps directly."""

    def __init__(self, images_by_batch=None, dtype=torch.float32):
        self.images_by_batch = images_by_batch
        self.dtype = dtype

    def data(self, batch):
        return self.images_by_batch(batch)

    def __call__(self, net, data, upto=None):
        dev = net.eng.device
        x = data if isinstance(data, torch.Tensor) else torch.as_tensor(np.asarray(data, dtype=np.float32))
        x = x.to(dev, torch.float32).to(self.dtype)
        blobs = {"data": x}
        for spec in net._specs:
            w = net._w[spec.name].to(self.dtype)
            b = net._b[spec.name].to(self.dtype)
            y = F.conv2d(blobs[spec.bottom], w, b, stride=spec.stride, padding=spec.pad, dilation=spec.dilation)
            blobs[spec.name] = y
            r = F.relu(y)
            blobs[spec.name + "_relu"] = r
            if spec.pool_after:
                blobs[net._pool_name[spec.name]] = F.max_pool2d(r, 2, 2)
            if upto is not None and spec.name == upto:
                break
        return blobs


# net.py:1309-1321
RANKDIC = {'conv1_1': 17, 'conv1_2': 17, 'conv2_1': 37, 'conv2_2': 47, 'conv3_1': 83, 'conv3_2': 89, 'conv3_3': 106,
           'conv4_1': 175, 'conv4_2': 192, 'conv4_3': 227, 'conv5_1': 398, 'conv5_2': 390, 'conv5_3': 379}


class Net:
    def __init__(self, specs, weights, biases, forward, pool_names=None, frozen=None):
        """specs: ordered list of ConvSpec; weights/biases: {name: array (n,c,k,k) / (n,)};
        forward: feature provider (see ConvStackForward); frozen: path of the frozen-points pickle."""
        self.eng = get_engine()
        dev = self.eng.device
        self._specs = list(specs)
        self._spec = {s.name: s for s in self._specs}
        self.convs = [s.name for s in self._specs]
        self._w = {k: torch.as_tensor(np.asarray(v, dtype=np.float32), device=dev).clone() if not isinstance(
            v, torch.Tensor) else v.to(dev, torch.float32).clone() for k, v in weights.items()}
        self._b = {k: torch.as_tensor(np.asarray(v, dtype=np.float32), device=dev).clone() if not isinstance(
            v, torch.Tensor) else v.to(dev, torch.float32).clone() for k, v in biases.items()}
        self._forward = forward
        self._pool_name = pool_names or {}
        self.bottom_names = {s.name: [s.bottom] for s in self._specs}
        self._mem = True
        self._protocol = 4  # net.py:94
        self._frozen = frozen
        self.WPQ = {}
        self.selection = {}
        self._feats_dict = None
        self._points_dict = None
        self._feats_dev = {}
        self.num = None
        self._batch_iter = 0

    # ---- accessors with the reference's names (net.py:174-286)
    def param_data(self, name):
        return self._w[name]

    def param_b_data(self, name):
        return self._b[name]

    def param_shape(self, name):
        return tuple(self._w[name].shape)

    def set_param_data(self, name, d):
        self._w[name].copy_(torch.as_tensor(np.asarray(d), device=self._w[name].device))

    def set_param_b(self, name, d):
        self._b[name].copy_(torch.as_tensor(np.asarray(d), device=self._b[name].device))

    def conv_param_pad(self, name):
        return self._spec[name].pad

    def conv_param_kernel_size(self, name):
        return self._spec[name].kernel_size

    def conv_param_stride(self, name):
        return self._spec[name].stride

    def forward(self, data=None, upto=None):
        """One forward pass: of the provider's next batch (data=None, like Caffe's data layer) or of given images
        (the frozen path, net.set_input_arrays at net.py:447).  Returns the blob dict."""
        if not hasattr(self._forward, "data"):
            # plain provider ``forward(net, batch) -> blobs`` (a batch index stands in for the frozen images)
            if data is None:
                data = self._batch_iter
                self._batch_iter += 1
            return self._forward(self, data)
        if data is None:
            data = self._forward.data(self._batch_iter)
            self._batch_iter += 1
        self._data = data
        return self._forward(self, data, upto=upto)

    def _frozen_blobs(self, batch, upto=None):
        pd = self._points_dict
        return self.forward(pd[(batch, 0)], upto=upto)

    # ---- extract_features, net.py:368-532 (conv blobs)
    def extract_features(self, names=[], nBatches=None, points_dict=None, save=False):
        assert nBatches is None, "deprecate"  # net.py:369
        nBatches = dcfgs.nBatches
        nPointsPerLayer = dcfgs.nPointsPerLayer
        if not isinstance(names, list):
            names = [names]
        assert len(names) > 0
        frozen_points = False
        if save:
            if points_dict is None:
                points_dict = dict()
                points_dict["nPointsPerLayer"] = nPointsPerLayer
                points_dict["nBatches"] = nBatches
            else:
                frozen_points = True
                nPointsPerLayer = points_dict["nPointsPerLayer"]
                nBatches = points_dict["nBatches"]
        eng = self.eng
        feats_dev = {}
        P = nPointsPerLayer
        last = names[-1] if all(n in self.convs for n in names) else None
        upto = None
        if last is not None:  # the deepest requested blob bounds the forward pass
            upto = max(names, key=self.convs.index)
        for batch in range(nBatches):
            if save and frozen_points and (batch, 0) in points_dict:
                blobs = self.forward(points_dict[(batch, 0)], upto=upto)  # net.py:446-447
            else:
                blobs = self.forward(upto=upto) if hasattr(self._forward, "data") else self.forward(batch)
                if save and not frozen_points and not hasattr(self._forward, "data"):
                    points_dict[(batch, 0)] = batch  # plain provider: the batch index identifies the images
                elif save and not frozen_points:
                    data = blobs["data"]
                    if batch == 0:
                        points_dict["data"] = tuple(data.shape)       # net.py:432-433
                        points_dict["label"] = (data.shape[0], 1, 1, 1)
                    if data.dtype == torch.bfloat16:  # numpy has no bfloat16: stored widened (exact)
                        data = data.float()
                    points_dict[(batch, 0)] = data.cpu().numpy().copy()  # net.py:441-442
                    points_dict[(batch, 1)] = np.zeros((data.shape[0], 1, 1, 1), dtype=np.float32)
            for name in names:
                feat = blobs[name]
                B, n, H, W = feat.shape
                self.num = B
                if name not in feats_dev:
                    feats_dev[name] = eng.empty(nBatches * P * B, n, dtype=torch.float32)
                if save and frozen_points and (batch, name, "randx") in points_dict:
                    randx = points_dict[(batch, name, "randx")]
                    randy = points_dict[(batch, name, "randy")]
                else:
                    randx = np.random.randint(0, H - 0, P)  # net.py:464-465 / 506-507
                    randy = np.random.randint(0, W - 0, P)
                    if save:
                        points_dict[(batch, name, "randx")] = randx.copy()
                        points_dict[(batch, name, "randy")] = randy.copy()
                rx = torch.as_tensor(np.asarray(randx, dtype=np.int32), device=eng.device)
                ry = torch.as_tensor(np.asarray(randy, dtype=np.int32), device=eng.device)
                out = feats_dev[name][batch * P * B:(batch + 1) * P * B]
                eng.point_gather(feat.contiguous(), rx, ry, B, P, out=out)
        self._last_feats_dev = feats_dev
        feats_dict = {k: v.cpu().numpy().astype(np.float64) for k, v in feats_dev.items()}  # fp64, net.py:426
        if save:
            return feats_dict, points_dict
        return feats_dict

    # ---- freeze_images / load_frozen, net.py:749-800, 839-876
    def freeze_images(self, check_exist=False, convs=None, **kwargs):
        """Samples points + features of every conv once and pickles ``[feats_dict, points_dict]`` (protocol 4) to
        ``self._frozen`` exactly like the reference (net.py:799-800).  Returns the path."""
        frozen = self._frozen
        assert frozen is not None, "construct the Net with frozen=<path> to use the pickle round trip"
        if check_exist and os.path.exists(frozen):
            return frozen
        if convs is None:
            convs = self.convs
        feats_dict, points_dict = self.extract_features(names=convs, save=1, **kwargs)
        with open(frozen, 'wb') as f:
            pickle.dump([feats_dict, points_dict], f, protocol=self._protocol)
        return frozen

    def load_frozen(self, DEBUG=False, feats_dict=None, points_dict=None):
        if feats_dict is None:  # net.py:862-864
            with open(self._frozen, 'rb') as f:
                feats_dict, points_dict = pickle.load(f)
        self._feats_dict = feats_dict
        self._points_dict = points_dict
        dev = self.eng.device
        self._feats_dev = {}
        for k, v in feats_dict.items():
            v32 = np.asarray(v, dtype=np.float32)
            self._feats_dev[k] = torch.as_tensor(v32 if np.array_equal(v32.astype(np.float64), v) else np.asarray(v),
                                                 device=dev)
        if DEBUG:  # net.py:866-875: re-extraction at the frozen points reproduces the frozen features exactly
            again, _ = self.extract_features(list(feats_dict), points_dict=points_dict, save=1)
            for i in again:
                assert np.array_equal(again[i], feats_dict[i]), i

    def freeze(self, names=None):
        """freeze_images + load_frozen without touching the disk."""
        names = names or self.convs
        feats_dict, points_dict = self.extract_features(names, save=1)
        self.load_frozen(feats_dict=feats_dict, points_dict=points_dict)
        return feats_dict, points_dict

    # ---- extract_XY, net.py:534-684
    def _extract_X_device(self, X, Y, relu):
        spec = self._spec[Y]
        pd = self._points_dict
        P, nBatches = pd["nPointsPerLayer"], pd["nBatches"]
        eng = self.eng
        # the producing layer bounds the forward pass: blobs after X are not needed
        upto = None
        for s in self._specs:
            if X in (s.name, s.name + "_relu", self._pool_name.get(s.name)):
                upto = s.name
        out = None
        for batch in range(nBatches):
            blob = self._frozen_blobs(batch, upto=upto)[X].contiguous() if (batch, 0) in pd else \
                self.forward(upto=upto)[X].contiguous()
            B, c = blob.shape[0], blob.shape[1]
            if out is None:
                kh, kw = spec.kernel_hw
                out = eng.empty(nBatches * P * B, c * kh * kw, dtype=torch.float32)
            rx = torch.as_tensor(np.asarray(pd[(batch, Y, "randx")], dtype=np.int32), device=eng.device)
            ry = torch.as_tensor(np.asarray(pd[(batch, Y, "randy")], dtype=np.int32), device=eng.device)
            eng.patch_gather(blob, rx, ry, B, P, spec.kernel_size, spec.pad, spec.stride, relu=relu,
                             out=out[batch * P * B:(batch + 1) * P * B], dilation=spec.dilation)
        return out

    def extract_XY(self, X, Y, DEBUG=False, w1=None):
        """Returns the (N*kh*kw, c) float64 matrix of the reference (rows (sample, kh, kw)); kh, kw and the rest of the
        window are those of the consumer Y."""
        assert w1 is None, "the w1 branch (net.py:544-548) is not part of the c3 path"
        kh, kw = self._spec[Y].kernel_hw
        Xd = self._extract_X_device(X, Y, relu=False)
        N = Xd.shape[0]
        c = Xd.shape[1] // (kh * kw)
        out = Xd.view(N, c, kh * kw).permute(0, 2, 1).reshape(N * kh * kw, c)
        return out.cpu().numpy().astype(np.float64)

    # ---- dictionary_kernel, net.py:1685-1735 (VGG branch: relu on X, resY = 0)
    def dictionary_kernel(self, X_name, weights, d_prime, Y_name, Y, DEBUG=0):
        if dcfgs.model in [cfgs.Models.xception, cfgs.Models.resnet] or dcfgs.res.short:
            raise NotImplementedError("ResNet/Xception residual branches (net.py:1716-1719) are not implemented")
        Xd = self._extract_X_device(X_name, Y_name, relu=True)  # :1698 + :1720
        W2 = self._w[Y_name]
        n, c, kh, kw = W2.shape
        feats = self._feats_dev[Y_name]
        bias = self._b[Y_name]
        y_bias = bias if feats.dtype == torch.float32 else None
        Yd = feats if y_bias is not None else feats - bias.to(torch.float64)
        idxs, Wd, bd = _dictionary_device(self.eng, Xd, W2.reshape(n, c * kh * kw), Yd, y_bias, c, kh * kw, d_prime)
        rank = int(idxs.sum())
        return idxs, Wd.cpu().numpy().reshape(n, rank, kh, kw), bd.cpu().numpy()

    # ---- R3, net.py:1292-1471
    def R3(self):
        """The 3C walk of the reference: for every conv after the first, spatial decomposition (VH_decompose, refitted
        on data), channel decomposition (ITQ_decompose on re-extracted features), then -- for the layers of alldic /
        pooldic -- channel pruning of the NEXT conv's input (dictionary_kernel), each stage compensating the error of
        the ones before it because features are re-extracted through the already rewritten weights.
        Returns (WPQ, new_pt): WPQ with the reference's keys (<conv>_V, (<conv>_H, 0|1), (<conv>_P, 0|1)); new_pt
        describes the rewritten topology (the reference writes a prototxt, net.py:1470)."""
        speed_ratio = dcfgs.dic.keep
        prefix = ('3C' if dcfgs.dic.vh else '2C') + str(int(speed_ratio) + 1) + 'x'  # :1296-1300
        convs = self.convs
        self.WPQ = dict()
        self.selection = dict()
        self._mem = True
        end = 5
        alldic = ['conv%d_1' % i for i in range(1, end)] + ['conv%d_2' % i for i in range(3, end)]  # :1307
        pooldic = ['conv1_2', 'conv2_2']
        rankdic = dict(RANKDIC)
        for i in rankdic:
            if 'conv5' in i:
                continue
            rankdic[i] = int(rankdic[i] * 4. / speed_ratio)  # :1323-1326
        c_ratio = 1.15
        dev = self.eng.device

        def getX(name):  # :1329-1331
            x = self.extract_XY(self.bottom_names[name][0], name)
            return np.rollaxis(x.reshape((-1, 3, 3, x.shape[1])), 3, 1).copy()

        def setConv(c, d):  # :1333-1337
            d = torch.as_tensor(np.asarray(d), device=dev, dtype=torch.float32)
            if c in self.selection:
                self._w[c][:, torch.as_tensor(self.selection[c], device=dev), :, :] = d
            else:
                self._w[c].copy_(d)

        topology = []
        trace = getattr(self, "_trace", None)  # optional list: (conv, stage, {name: array}) per stage (debugging aid)
        # optional test hook, called where the reference enters VH_decompose / ITQ_decompose / dictionary_kernel and
        # at the end ('vh' | 'itq' | 'prune' | 'final'); it may inspect and overwrite the live parameters
        checkpoint = getattr(self, "_checkpoint", None) or (lambda stage: None)
        for conv, convnext in zip(convs[1:], convs[2:] + ['pool5']):
            conv_V = underline(conv, 'V')
            conv_H = underline(conv, 'H')
            conv_P = underline(conv, 'P')
            W_shape = self.param_shape(conv)
            d_c = int(W_shape[0] / c_ratio)
            rank = rankdic[conv]
            d_prime = rank
            if d_c < rank:
                d_c = rank  # :1349
            # ---- spatial decomposition (:1351-1380)
            checkpoint("vh")
            weights = self._w[conv]
            if conv in self.selection:
                weights = weights[:, torch.as_tensor(self.selection[conv], device=dev), :, :]
            Y = self._feats_dict[conv] - self._b[conv].cpu().numpy()
            X = getX(conv)
            if conv in self.selection:
                X = X[:, self.selection[conv], :, :]
            V, H, VHr, b = VH_decompose(weights.cpu().numpy().astype(np.float64), rank=rank, DEBUG=True, X=X, Y=Y)
            self.set_param_b(conv, b)
            self.WPQ[conv_V] = V
            setConv(conv, VHr)
            self.WPQ[(conv_H, 0)] = H
            self.WPQ[(conv_H, 1)] = self._b[conv].cpu().numpy()
            if trace is not None:
                trace.append((conv, "vh", dict(VHr=VHr.copy(), b=np.asarray(b).copy(), X=X.copy(), Y=Y.copy())))
            # ---- channel decomposition (:1384-1404)
            checkpoint("itq")
            feats_dict, _ = self.extract_features(names=conv, points_dict=self._points_dict, save=1)
            Yf = feats_dict[conv]
            W1, W2, B, W12 = ITQ_decompose(Yf, self._feats_dict[conv], H, d_prime, bias=self._b[conv].cpu().numpy(),
                                           DEBUG=0, Wr=VHr)
            setConv(conv, W12.copy())
            self.set_param_b(conv, B.copy())
            self.WPQ[(conv_H, 0)] = W1.reshape([d_prime, H.shape[1], H.shape[2], H.shape[3]])
            self.WPQ[(conv_H, 1)] = np.zeros(d_prime)
            self.WPQ[(conv_P, 0)] = W2.reshape([W2.shape[0], W2.shape[1], 1, 1])
            self.WPQ[(conv_P, 1)] = B
            if trace is not None:
                trace.append((conv, "itq", dict(W12=W12.copy(), B=np.asarray(B).copy(), Yf=Yf.copy())))
            # ---- channel pruning (:1406-1459)
            if dcfgs.dic.vh and (conv in alldic or conv in pooldic) and (convnext in self.convs):
                X_name = self.bottom_names[convnext][0] if conv in pooldic else conv  # :1411-1414
                checkpoint("prune")
                idxs, W2n, B2n = self.dictionary_kernel(X_name, None, d_c, convnext, None)
                self.selection[convnext] = idxs
                it = torch.as_tensor(idxs, device=dev)
                self._w[convnext][:, ~it, ...] = 0  # :1446
                self._w[convnext][:, it, ...] = torch.as_tensor(W2n, device=dev, dtype=torch.float32)
                self.set_param_b(convnext, B2n)
                key = conv_P if (conv_P, 0) in self.WPQ else conv_H  # :1450-1456
                self.WPQ[(key, 0)] = self.WPQ[(key, 0)][idxs]
                self.WPQ[(key, 1)] = self.WPQ[(key, 1)][idxs]
                if trace is not None:
                    from .decompose import DictionaryInfo
                    trace.append((conv, "prune", dict(idxs=idxs.copy(), W2=W2n.copy(), B2=np.asarray(B2n).copy(),
                                                      ls=dict(DictionaryInfo.last.get("ls", {})))))
            topology.append({"V": conv_V, "H": conv_H, "P": conv_P, "rank": int(rank),
                             "num_output": int(self.WPQ[(conv_P, 0)].shape[0])})
        checkpoint("final")
        new_pt = {"prefix": prefix, "layers": topology}
        return self.WPQ, new_pt


# ---------------------------------------------------------------------------- model surgery on R3's result
def combineHP(WPQ, new_pt):
    """lib/net.py:1473-1504: after the 3C walk every conv is a chain V (k x 1) -> H (1 x k, m outputs) -> P (1 x 1,
    o outputs).  Where the channel decomposition saved little (3 m >= 2 o) the reference folds P back into H:
        W_H' = P_w . H_w   (o x ...),    b_H' = P_b + P_w . H_b
    and removes P.  The reference edits the Caffe net and writes a prototxt; here the same rule is applied to the
    dictionaries ``Net.R3`` returns.  Returns (WPQ', new_pt') -- new objects, the inputs are left alone."""
    out = dict(WPQ)
    layers = []
    for lay in new_pt["layers"]:
        lay = dict(lay)
        h, p = lay["H"], lay.get("P")
        if p is not None and (h, 0) in out and (p, 0) in out:
            assert h.split('_H')[0] == p.split('_P')[0]  # :1485
            Hshape = out[(h, 0)].shape
            m, o = Hshape[0], out[(p, 0)].shape[0]
            if 3 * m >= 2 * o:  # :1489
                Hw = np.asarray(out[(h, 0)], dtype=np.float64).reshape((m, -1))
                Pw = np.asarray(out[(p, 0)], dtype=np.float64).reshape((o, -1))
                Hb = np.asarray(out[(h, 1)], dtype=np.float64)
                pb = np.asarray(out[(p, 1)], dtype=np.float64)
                out[(h, 0)] = Pw.dot(Hw).reshape((o,) + tuple(Hshape[1:]))  # :1495
                out[(h, 1)] = pb + Pw.dot(Hb)                                # :1496
                del out[(p, 0)], out[(p, 1)]
                lay["P"] = None
                lay["num_output_H"] = int(o)
        layers.append(lay)
    return out, dict(new_pt, layers=layers, prefix="cb" + str(new_pt.get("prefix", "")))


def layercomputation(blob_shape, param_shape, stride=1, spatial=False, channels=1., outputs=1., innerproduct=False):
    """lib/net.py:1049-1067: multiply-accumulates of one layer from the shape of its bottom blob (B, C, H, W) and of its
    weights (n, c, kh, kw); ``spatial`` marks the depth-wise layers of ``Net.spation_convs``."""
    s, p = blob_shape, param_shape
    if innerproduct:
        return int(p[0] * p[1])
    if spatial:
        channels = 1
    else:
        assert s[1] == p[1]
        channels *= p[1]
    outputs *= p[0]
    return int(s[2] * s[3] * outputs * channels * p[2] * p[3] / stride ** 2)


def computation(layers):
    """lib/net.py:1069-1081: total and per-layer cost; ``layers`` = iterable of (name, blob_shape, param_shape, stride).
    Returns (total, {name: flops}) instead of printing."""
    per = {name: layercomputation(bs, ps, st) for name, bs, ps, st in layers}
    return sum(per.values()), per
