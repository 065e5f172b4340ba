"""Synthetic workloads for BASELINE.json's configs (no datasets / checkpoints offline).

A *layer problem* is what one iteration of the reference's pruning loop sees
(lib/net.py:1406-1459): the bottom blob of ``convnext`` for ``nBatches`` batches of ``B``
images, the sampled output points, ``convnext``'s weights/bias and its frozen output features
at those points.  Shapes follow ``temp/vgg.prototxt`` (VGG-16 @224x224): each of the 13 conv
layers has its *input* channels pruned to ``int(c / 1.15)`` (``conv1_1``: c = 3 -> the
``rank == c`` shortcut, lib/decompose.py:487).

Data: pre-ReLU bottom blob ~ N(0,1) fp32 (ReLU is fused into the gather, lib/net.py:1720),
weights ~ N(0, 2/(c k^2)) (MSRA filler, lib/builder.py:385), bias ~ 0.01 N(0,1), frozen output
features = conv(relu(blob)) + bias + 1% noise, rounded to fp32 like a Caffe blob.  Every
batch is an independent draw (as 10 new images per batch are in the reference), so the N =
nBatches*P*B sampled patches are distinct and the least-squares systems are well posed.
"""
from __future__ import annotations

import numpy as np

from .engine import LEAKY_SLOPE, check_act, conv_pair, conv_triple

# (name, c_in, n_out, H=W of the layer's input/output map)  -- temp/vgg.prototxt:53-306
VGG16 = [
    ("conv1_1", 3, 64, 224), ("conv1_2", 64, 64, 224),
    ("conv2_1", 64, 128, 112), ("conv2_2", 128, 128, 112),
    ("conv3_1", 128, 256, 56), ("conv3_2", 256, 256, 56), ("conv3_3", 256, 256, 56),
    ("conv4_1", 256, 512, 28), ("conv4_2", 512, 512, 28), ("conv4_3", 512, 512, 28),
    ("conv5_1", 512, 512, 14), ("conv5_2", 512, 512, 14), ("conv5_3", 512, 512, 14),
]

C_RATIO = 1.15  # lib/net.py:1327

# BASELINE config 4: ResNet-50 bottleneck problems.  (name, c_in, n_out, k, H_in, stride, pad, kept) where `kept`
# is the number of surviving INPUT channels recorded in the reference's released pruned net
# temp/resnet-50-cp.prototxt (branch2a: the block's input selector `<prev>_Filter.num_output`; branch2b /
# branch2c: `num_output` of the producing conv).  kept == c_in means the layer was left alone (LS only).
RESNET50 = [
    ('res2a_branch2a', 64, 64, 1, 56, 1, 0, 35), ('res2a_branch2b', 64, 64, 3, 56, 1, 1, 64),
    ('res2a_branch2c', 64, 256, 1, 56, 1, 0, 55), ('res2b_branch2a', 256, 64, 1, 56, 1, 0, 101),
    ('res2b_branch2b', 64, 64, 3, 56, 1, 1, 51), ('res2b_branch2c', 64, 256, 1, 56, 1, 0, 39),
    ('res2c_branch2a', 256, 64, 1, 56, 1, 0, 97), ('res2c_branch2b', 64, 64, 3, 56, 1, 1, 50),
    ('res2c_branch2c', 64, 256, 1, 56, 1, 0, 37), ('res3a_branch2a', 256, 128, 1, 56, 2, 0, 144),
    ('res3a_branch2b', 128, 128, 3, 28, 1, 1, 128), ('res3a_branch2c', 128, 512, 1, 28, 1, 0, 106),
    ('res3b_branch2a', 512, 128, 1, 28, 1, 0, 205), ('res3b_branch2b', 128, 128, 3, 28, 1, 1, 105),
    ('res3b_branch2c', 128, 512, 1, 28, 1, 0, 72), ('res3c_branch2a', 512, 128, 1, 28, 1, 0, 198),
    ('res3c_branch2b', 128, 128, 3, 28, 1, 1, 105), ('res3c_branch2c', 128, 512, 1, 28, 1, 0, 72),
    ('res3d_branch2a', 512, 128, 1, 28, 1, 0, 288), ('res3d_branch2b', 128, 128, 3, 28, 1, 1, 128),
    ('res3d_branch2c', 128, 512, 1, 28, 1, 0, 110), ('res4a_branch2a', 512, 256, 1, 28, 2, 0, 278),
    ('res4a_branch2b', 256, 256, 3, 14, 1, 1, 256), ('res4a_branch2c', 256, 1024, 1, 14, 1, 0, 225),
    ('res4b_branch2a', 1024, 256, 1, 14, 1, 0, 418), ('res4b_branch2b', 256, 256, 3, 14, 1, 1, 209),
    ('res4b_branch2c', 256, 1024, 1, 14, 1, 0, 147), ('res4c_branch2a', 1024, 256, 1, 14, 1, 0, 407),
    ('res4c_branch2b', 256, 256, 3, 14, 1, 1, 204), ('res4c_branch2c', 256, 1024, 1, 14, 1, 0, 158),
    ('res4d_branch2a', 1024, 256, 1, 14, 1, 0, 423), ('res4d_branch2b', 256, 256, 3, 14, 1, 1, 212),
    ('res4d_branch2c', 256, 1024, 1, 14, 1, 0, 155), ('res4e_branch2a', 1024, 256, 1, 14, 1, 0, 412),
    ('res4e_branch2b', 256, 256, 3, 14, 1, 1, 211), ('res4e_branch2c', 256, 1024, 1, 14, 1, 0, 148),
    ('res4f_branch2a', 1024, 256, 1, 14, 1, 0, 595), ('res4f_branch2b', 256, 256, 3, 14, 1, 1, 256),
    ('res4f_branch2c', 256, 1024, 1, 14, 1, 0, 213), ('res5a_branch2a', 1024, 512, 1, 14, 2, 0, 606),
    ('res5a_branch2b', 512, 512, 3, 7, 1, 1, 512), ('res5a_branch2c', 512, 2048, 1, 7, 1, 0, 433),
    ('res5b_branch2a', 2048, 512, 1, 7, 1, 0, 1222), ('res5b_branch2b', 512, 512, 3, 7, 1, 1, 512),
    ('res5b_branch2c', 512, 2048, 1, 7, 1, 0, 437), ('res5c_branch2a', 2048, 512, 1, 7, 1, 0, 1147),
    ('res5c_branch2b', 512, 512, 3, 7, 1, 1, 512), ('res5c_branch2c', 512, 2048, 1, 7, 1, 0, 440),
]


def _out_size(n, k, pad, stride, dil, output_padding, transposed):
    """One axis of the output map, PyTorch's formula: Conv (n + 2 pad - dil (k - 1) - 1) // stride + 1, ConvTranspose
    (n - 1) stride - 2 pad + dil (k - 1) + output_padding + 1 with output_padding < max(stride, dil)."""
    if transposed:
        assert 0 <= output_padding < max(stride, dil), "output_padding must be smaller than either stride or dilation"
        out = (n - 1) * stride - 2 * pad + dil * (k - 1) + output_padding + 1
    else:
        assert output_padding == 0, "output_padding is an argument of transposed convolutions"
        out = (n + 2 * pad - dil * (k - 1) - 1) // stride + 1
    assert out >= 1, "empty output map"
    return out


def _set_input(s, act, act_param, bn):
    """The consumer's input transform of a layer shape: act (engine.ACTS) after, with bn, the producer's BatchNorm."""
    check_act(act, act_param)
    s.act, s.act_param, s.bn = act, act_param, bool(bn)


def _conv_args(s):
    a = dict(k=s.k, pad=s.pad, stride=s.stride, dilation=s.dilation)
    if s.transposed:
        a["transposed"] = True
    return a


class LayerShape:
    """One layer problem: a convolution with c input and n output channels on an H x W input map (W = H unless
    given).  k, pad, stride and dilation are ints or (h, w) pairs, as torch.nn.Conv2d takes them (groups == 1); the
    reference's layers are square, odd and undilated, and for those k, pad and stride keep their plain int meaning.
    kh, kw, pad_h, pad_w, stride_h, stride_w, dil_h, dil_w: the per-axis geometry; k2 = kh*kw taps per channel;
    Ho x Wo: the output map (PyTorch's formula), the range of the sampled points.
    transposed: a torch.nn.ConvTranspose2d consumer (k, pad = padding, stride, dilation and output_padding as it takes
    them; H x W its input map); W2 is then (n, c, kh, kw) = weight.transpose(0, 1), the orientation of every layer.
    act, act_param, bn: the consumer's input transform (Engine.patch_gather).  The map is the producer's raw conv output
    and X is act(BN(map)) with bn (the problem's in_scale / in_shift, fold_bn of the producer's BatchNorm), act(map)
    without; act 'relu' and no bn is the reference's VGG layer."""

    def __init__(self, name, c, n, H, k=3, pad=1, stride=1, N=5000, B=10, P=10, rank=None, dilation=1, W=None,
                 transposed=False, output_padding=0, act="relu", act_param=None, bn=False):
        _set_input(self, act, act_param, bn)
        self.name, self.c, self.n, self.H, self.W = name, c, n, H, H if W is None else W
        self.k, self.pad, self.stride, self.dilation = k, pad, stride, dilation
        self.transposed, self.output_padding = bool(transposed), output_padding
        self.kh, self.kw = conv_pair(k)
        self.pad_h, self.pad_w = conv_pair(pad)
        self.stride_h, self.stride_w = conv_pair(stride)
        self.dil_h, self.dil_w = conv_pair(dilation)
        self.k2 = self.kh * self.kw
        self.B, self.P = B, P
        assert N % (B * P) == 0, "N must be a multiple of B*P"
        self.nbatch = N // (B * P)
        self.N = N
        self.rank = int(c / C_RATIO) if rank is None else rank
        if c <= 3:
            self.rank = c
        self.K = c * self.k2
        self.S = min(400, N // 20)
        self.Ho, self.Wo = (_out_size(*a, self.transposed) for a in zip(
            (self.H, self.W), (self.kh, self.kw), (self.pad_h, self.pad_w), (self.stride_h, self.stride_w),
            (self.dil_h, self.dil_w), conv_pair(output_padding)))

    def conv_args(self):
        """(k, pad, stride), dilation and (for a transposed layer) transposed, as Engine.patch_gather takes them"""
        return _conv_args(self)

    def cost(self):
        """Rough relative cost (Gram + Cholesky flops) for load balancing across GPUs."""
        kp = self.rank * self.k2
        return self.N * self.K * (self.K + 2 * self.n) + kp ** 3 / 3 + 2.0 * kp * kp * self.n


class LayerShape3d:
    """One layer problem of a Conv3d consumer with c input and n output channels on a D x H x W input map (W = H unless
    given).  k, pad, stride and dilation are ints or (t, h, w) triples, as torch.nn.Conv3d takes them (groups == 1).
    kt, kh, kw, pad_t, ..., dil_w: the per-axis geometry; k2 = kt*kh*kw taps per channel (what the solver sees: X is
    (N, c*k2)); To x Ho x Wo: the output map (PyTorch's formula), the range of the sampled points (t, x, y).
    transposed, output_padding: a torch.nn.ConvTranspose3d consumer; act, act_param, bn: its input transform; as for
    LayerShape."""

    def __init__(self, name, c, n, D, H, k=3, pad=1, stride=1, N=5000, B=10, P=10, rank=None, dilation=1, W=None,
                 transposed=False, output_padding=0, act="relu", act_param=None, bn=False):
        _set_input(self, act, act_param, bn)
        self.name, self.c, self.n, self.D, self.H, self.W = name, c, n, D, H, H if W is None else W
        self.k, self.pad, self.stride, self.dilation = k, pad, stride, dilation
        self.transposed, self.output_padding = bool(transposed), output_padding
        self.kt, self.kh, self.kw = conv_triple(k)
        self.pad_t, self.pad_h, self.pad_w = conv_triple(pad)
        self.stride_t, self.stride_h, self.stride_w = conv_triple(stride)
        self.dil_t, self.dil_h, self.dil_w = conv_triple(dilation)
        self.window = (self.kt, self.kh, self.kw)
        self.k2 = self.kt * self.kh * self.kw
        self.B, self.P = B, P
        assert N % (B * P) == 0, "N must be a multiple of B*P"
        self.nbatch = N // (B * P)
        self.N = N
        self.rank = int(c / C_RATIO) if rank is None else rank
        if c <= 3:
            self.rank = c
        self.K = c * self.k2
        self.S = min(400, N // 20)
        self.To, self.Ho, self.Wo = (_out_size(*a, self.transposed) for a in zip(
            (self.D, self.H, self.W), self.window, (self.pad_t, self.pad_h, self.pad_w),
            (self.stride_t, self.stride_h, self.stride_w), (self.dil_t, self.dil_h, self.dil_w),
            conv_triple(output_padding)))

    def conv_args(self):
        """(k, pad, stride), dilation and (for a transposed layer) transposed, as Engine.patch_gather3d takes them"""
        return _conv_args(self)


    def cost(self):
        """Rough relative cost (Gram + Cholesky flops) for load balancing across GPUs."""
        kp = self.rank * self.k2
        return self.N * self.K * (self.K + 2 * self.n) + kp ** 3 / 3 + 2.0 * kp * kp * self.n


# torchvision's r3d_18 on a 16 x 112 x 112 clip: the 3x3x3 convolutions of layer1-layer4 (two BasicBlocks each).
# (name, c_in, n_out, D = H of the layer's INPUT map, stride); the first conv of layer2-4 halves every axis.
R3D18 = [
    ("layer1.0.conv1", 64, 64, 16, 56, 1), ("layer1.0.conv2", 64, 64, 16, 56, 1),
    ("layer1.1.conv1", 64, 64, 16, 56, 1), ("layer1.1.conv2", 64, 64, 16, 56, 1),
    ("layer2.0.conv1", 64, 128, 16, 56, 2), ("layer2.0.conv2", 128, 128, 8, 28, 1),
    ("layer2.1.conv1", 128, 128, 8, 28, 1), ("layer2.1.conv2", 128, 128, 8, 28, 1),
    ("layer3.0.conv1", 128, 256, 8, 28, 2), ("layer3.0.conv2", 256, 256, 4, 14, 1),
    ("layer3.1.conv1", 256, 256, 4, 14, 1), ("layer3.1.conv2", 256, 256, 4, 14, 1),
    ("layer4.0.conv1", 256, 512, 4, 14, 2), ("layer4.0.conv2", 512, 512, 2, 7, 1),
    ("layer4.1.conv1", 512, 512, 2, 7, 1), ("layer4.1.conv2", 512, 512, 2, 7, 1),
]


def r3d18_layers(N=5000, B=10, P=50):
    """The 16 layer problems of R3D18.  B = 10 clips and P = 50 points per batch (10 batches at N = 5000) keep the
    synthetic fp32 maps at 8.1 GB in all (6.4 GB of them the five 64 x 16 x 56 x 56 maps); with P = 10 they would be
    50 batches, 40 GB."""
    return [LayerShape3d(nm, c, n, D, H, k=3, pad=1, stride=st, N=N, B=B, P=P) for nm, c, n, D, H, st in R3D18]


# The transposed convolutions of three decoder families: (name, c_in, n_out, H = W (3-D: D = H = W) of the layer's
# INPUT map, k, stride, pad), groups == 1.
# A same-padded 2-D U-Net on 256 x 256 images: the up-convolutions ConvTranspose2d(c, c/2, 2, stride 2).
UNET_UP = [("up1", 1024, 512, 16, 2, 2, 0), ("up2", 512, 256, 32, 2, 2, 0), ("up3", 256, 128, 64, 2, 2, 0),
           ("up4", 128, 64, 128, 2, 2, 0)]
# A 3-D nnU-Net-style decoder on 128^3 patches (features 32 ... 320): ConvTranspose3d(k = stride = 2).
NNUNET3D_UP = [("tu0", 320, 320, 4, 2, 2, 0), ("tu1", 320, 256, 8, 2, 2, 0), ("tu2", 256, 128, 16, 2, 2, 0),
               ("tu3", 128, 64, 32, 2, 2, 0), ("tu4", 64, 32, 64, 2, 2, 0)]
# One DCGAN-style generator layer: ConvTranspose2d(256, 128, 4, stride 2, padding 1), overlapping windows.
DCGAN_UP = [("dcgan.up3", 256, 128, 16, 4, 2, 1)]


def conv_transpose_layers(N=5000):
    """{network: its transposed-convolution layer problems} of UNET_UP, NNUNET3D_UP and DCGAN_UP.  B and P keep the
    synthetic fp32 maps within about 10 GB: the 2-D ones at B = 10, P = 50 (100 images, 1.6 GB in all), the 3-D ones at
    B = 5, P = 100 (50 volumes; 3.4 GB of the 4.3 GB the 64 x 64^3 map of tu4)."""
    return {
        "unet2d": [LayerShape(nm, c, n, H, k=k, stride=st, pad=p, N=N, B=10, P=50, transposed=True)
                   for nm, c, n, H, k, st, p in UNET_UP],
        "nnunet3d": [LayerShape3d(nm, c, n, H, H, k=k, stride=st, pad=p, N=N, B=5, P=100, transposed=True)
                     for nm, c, n, H, k, st, p in NNUNET3D_UP],
        "dcgan": [LayerShape(nm, c, n, H, k=k, stride=st, pad=p, N=N, B=10, P=50, transposed=True)
                  for nm, c, n, H, k, st, p in DCGAN_UP],
    }


def vgg16_layers(N=5000, B=10, P=10):
    return [LayerShape(nm, c, n, H, N=N, B=B, P=P) for nm, c, n, H in VGG16]


def resnet50_layers(N=5000, B=10, P=10, bn=False):
    """The 48 bottleneck convolutions of RESNET50.  bn: pruned from the raw conv outputs of a Conv-BN-ReLU network --
    branch2b and branch2c take ReLU(BN(raw output of the branch before)); branch2a keeps the ReLU of its input, the
    block's post-add map."""
    return [LayerShape(nm, c, n, H, k=k, pad=pad, stride=st, N=N, B=B, P=P, rank=kept,
                       bn=bn and not nm.endswith("branch2a"))
            for nm, c, n, k, H, st, pad, kept in RESNET50]


def fold_bn(bn):
    """(scale, shift) of an eval-mode torch.nn.BatchNorm2d / 3d: scale = weight / sqrt(running_var + eps), shift =
    bias - running_mean * scale, computed in float64 and rounded once to float32 (contiguous tensors on bn's device).
    bn itself is left untouched."""
    import torch

    with torch.no_grad():
        var, mean = bn.running_var.double(), bn.running_mean.double()
        w = bn.weight.double() if bn.weight is not None else torch.ones_like(var)
        b = bn.bias.double() if bn.bias is not None else torch.zeros_like(var)
        scale = w / torch.sqrt(var + bn.eps)
        shift = b - mean * scale
        return scale.float().contiguous(), shift.float().contiguous()


def input_transform_numpy(v, act, act_param=None, scale=None, shift=None):
    """The consumer's input transform (cpb200.h, cp_patch_gather_act) on float32 values v, channels on axis 1:
    (v * scale) + shift, each rounded in float32 (either left out when None), then act.  Every act but silu is the
    kernels' expression, bit for bit; silu is the float64 value rounded to float32, which the kernels meet within 4
    ulp."""
    f = np.float32
    v = np.asarray(v, dtype=f)
    cshape = (1, -1) + (1,) * (v.ndim - 2)
    with np.errstate(all="ignore"):
        if scale is not None:
            v = v * np.asarray(scale, dtype=f).reshape(cshape)
        if shift is not None:
            v = v + np.asarray(shift, dtype=f).reshape(cshape)
        if act == "relu":
            return np.fmax(v, f(0))
        if act == "relu6":
            return np.fmin(np.fmax(v, f(0)), f(6))
        if act == "leaky_relu":
            return np.where(v > 0, v, v * f(LEAKY_SLOPE if act_param is None else act_param))
        if act == "hardswish":
            return (v * np.fmin(np.fmax(v + f(3), f(0)), f(6))) / f(6)
        if act == "silu":
            d = v.astype(np.float64)
            return (d / (1.0 + np.exp(-d))).astype(f)
        assert act == "identity", act
        return v


def _transformed(gather, fmap, args, relu, dilation, act, act_param, in_scale, in_shift):
    """gather(fmap, *args, relu=False, dilation=dilation) with the input transform applied to the taps inside the map;
    the others (zero padding, invalid taps of a transposed window) stay +0."""
    if relu:
        raise ValueError("pass relu or act, not both")
    X = gather(fmap, *args, relu=False, dilation=dilation)
    ones = np.ones(fmap.shape[:1] + (1,) + fmap.shape[2:], dtype=np.float32)
    inmap = gather(ones, *args, relu=False, dilation=dilation) != 0
    act = "identity" if act is None else act
    return np.where(inmap, input_transform_numpy(X, act, act_param, in_scale, in_shift), np.float32(0))


def _xform_of(s, d):
    """The gather's transform arguments of layer s and problem d: relu for the reference's layers, act and the
    affine otherwise."""
    if s.act == "relu" and not s.bn:
        return dict(relu=True)
    return dict(relu=None, act=s.act, act_param=s.act_param, in_scale=d.get("in_scale"), in_shift=d.get("in_shift"))


def bn_params(c, seed):
    """A producer BatchNorm's folded (scale, shift), float32, for a synthetic bn layer: |scale| in [0.5, 1.5] with
    every tenth sign flipped, shift ~ N(0, 0.5) -- far enough from zero that a padded tap given the transform shows.
    Drawn from a generator of their own, so the rest of the problem is that of the same seed without bn."""
    r = np.random.RandomState([seed, 0xB7])
    scale = r.uniform(0.5, 1.5, c) * np.where(r.uniform(size=c) < 0.1, -1.0, 1.0)
    shift = 0.5 * r.standard_normal(c)
    return scale.astype(np.float32), shift.astype(np.float32)


def make_problem_numpy(shape: LayerShape, seed: int, noise=0.01):
    """Host (numpy) instance of a layer problem -- used by CPU tests and by the oracle leg.
    Returns dict(fmap (nbatch*B,c,H,W) f32, randx/randy (nbatch,P) i32, W2, b2, feats (N,n) f32,
    samples (S,), X (N,c,kh,kw) f32 relu'd patches -- the shape's input transform of them, with in_scale / in_shift
    (bn_params) for a bn shape)."""
    if isinstance(shape, LayerShape3d):
        return _make_problem3d_numpy(shape, seed, noise)
    r = np.random.RandomState(seed)
    s = shape
    fmap = r.standard_normal((s.nbatch * s.B, s.c, s.H, s.W)).astype(np.float32)
    randx = r.randint(0, s.Ho, (s.nbatch, s.P)).astype(np.int32)
    randy = r.randint(0, s.Wo, (s.nbatch, s.P)).astype(np.int32)
    W2 = (r.standard_normal((s.n, s.c, s.kh, s.kw)) * np.sqrt(2.0 / (s.c * s.k2))).astype(np.float32)
    b2 = (0.01 * r.standard_normal(s.n)).astype(np.float32)
    bn = dict(zip(("in_scale", "in_shift"), bn_params(s.c, seed))) if s.bn else {}
    gather = gather_patches_tr_numpy if s.transposed else gather_patches_numpy
    X = gather(fmap, randx, randy, s.B, s.k, s.pad, s.stride, dilation=s.dilation, **_xform_of(s, bn))
    Y = X.reshape(s.N, -1).astype(np.float64) @ W2.reshape(s.n, -1).T.astype(np.float64) + b2
    Y = Y + noise * Y.std() * r.standard_normal(Y.shape)
    feats = Y.astype(np.float32)
    samples = r.randint(0, s.N, s.S)
    return dict(fmap=fmap, randx=randx, randy=randy, W2=W2, b2=b2, feats=feats, samples=samples, X=X, **bn)


def gather_patches_numpy(fmap, randx, randy, B, k, pad, stride, relu, dilation=1, act=None, act_param=None,
                         in_scale=None, in_shift=None):
    """Plain numpy statement of the patch layout (rows (batch, point, image); columns (c,kh,kw))
    used to build synthetic targets.  (The *checked* restatement of the reference's
    extract_XY lives in the oracle directory; tests compare the two.)  k, pad, stride, dilation: ints or (h, w)
    pairs, as LayerShape takes them.  act, act_param, in_scale, in_shift (relu then None): the input transform of the
    taps inside the map (input_transform_numpy), the padding +0."""
    if act is not None or in_scale is not None or in_shift is not None:
        return _transformed(gather_patches_numpy, fmap, (randx, randy, B, k, pad, stride), relu, dilation, act,
                            act_param, in_scale, in_shift)
    (kh, kw), (ph, pw), (sh, sw), (dh, dw) = (conv_pair(v) for v in (k, pad, stride, dilation))
    nimg, c, H, W = fmap.shape
    nbatch, P = randx.shape
    # taps reach down to stride*(Ho-1) - pad + dil*(k-1) <= H - 1 + pad: a border of pad on each side suffices
    fp = np.zeros((nimg, c, H + 2 * ph, W + 2 * pw), dtype=fmap.dtype)
    fp[:, :, ph:H + ph, pw:W + pw] = fmap
    out = np.empty((nbatch * P * B, c, kh, kw), dtype=fmap.dtype)
    for b in range(nbatch):
        imgs = fp[b * B:(b + 1) * B]
        for p in range(P):
            y0, x0 = sh * randx[b, p], sw * randy[b, p]
            out[(b * P + p) * B:(b * P + p + 1) * B] = imgs[:, :, y0:y0 + dh * (kh - 1) + 1:dh,
                                                            x0:x0 + dw * (kw - 1) + 1:dw]
    if relu:
        np.maximum(out, 0, out=out)
    return out


def _make_problem3d_numpy(s, seed, noise):
    """make_problem_numpy for a LayerShape3d: fmap (nbatch*B, c, D, H, W), randt/randx/randy, X (N, c, kt, kh, kw)."""
    r = np.random.RandomState(seed)
    fmap = r.standard_normal((s.nbatch * s.B, s.c, s.D, s.H, s.W)).astype(np.float32)
    randt = r.randint(0, s.To, (s.nbatch, s.P)).astype(np.int32)
    randx = r.randint(0, s.Ho, (s.nbatch, s.P)).astype(np.int32)
    randy = r.randint(0, s.Wo, (s.nbatch, s.P)).astype(np.int32)
    W2 = (r.standard_normal((s.n, s.c) + s.window) * np.sqrt(2.0 / (s.c * s.k2))).astype(np.float32)
    b2 = (0.01 * r.standard_normal(s.n)).astype(np.float32)
    bn = dict(zip(("in_scale", "in_shift"), bn_params(s.c, seed))) if s.bn else {}
    gather = gather_patches_tr3d_numpy if s.transposed else gather_patches3d_numpy
    X = gather(fmap, randt, randx, randy, s.B, s.k, s.pad, s.stride, dilation=s.dilation, **_xform_of(s, bn))
    Y = X.reshape(s.N, -1).astype(np.float64) @ W2.reshape(s.n, -1).T.astype(np.float64) + b2
    Y = Y + noise * Y.std() * r.standard_normal(Y.shape)
    feats = Y.astype(np.float32)
    samples = r.randint(0, s.N, s.S)
    return dict(fmap=fmap, randt=randt, randx=randx, randy=randy, W2=W2, b2=b2, feats=feats, samples=samples, X=X,
                **bn)


def gather_patches3d_numpy(fmap, randt, randx, randy, B, k, pad, stride, relu, dilation=1, act=None, act_param=None,
                           in_scale=None, in_shift=None):
    """gather_patches_numpy for NCDHW maps and Conv3d windows: rows (batch, point, image), columns (c, kt, kh, kw).
    k, pad, stride, dilation: ints or (t, h, w) triples; act ... in_shift as for gather_patches_numpy."""
    if act is not None or in_scale is not None or in_shift is not None:
        return _transformed(gather_patches3d_numpy, fmap, (randt, randx, randy, B, k, pad, stride), relu, dilation,
                            act, act_param, in_scale, in_shift)
    (kt, kh, kw), (pt, ph, pw), (st, sh, sw), (dt, dh, dw) = (conv_triple(v) for v in (k, pad, stride, dilation))
    nimg, c, D, H, W = fmap.shape
    nbatch, P = randx.shape
    fp = np.zeros((nimg, c, D + 2 * pt, H + 2 * ph, W + 2 * pw), dtype=fmap.dtype)
    fp[:, :, pt:D + pt, ph:H + ph, pw:W + pw] = fmap
    out = np.empty((nbatch * P * B, c, kt, kh, kw), dtype=fmap.dtype)
    for b in range(nbatch):
        imgs = fp[b * B:(b + 1) * B]
        for p in range(P):
            t0, y0, x0 = st * randt[b, p], sh * randx[b, p], sw * randy[b, p]
            out[(b * P + p) * B:(b * P + p + 1) * B] = imgs[:, :, t0:t0 + dt * (kt - 1) + 1:dt,
                                                            y0:y0 + dh * (kh - 1) + 1:dh, x0:x0 + dw * (kw - 1) + 1:dw]
    if relu:
        np.maximum(out, 0, out=out)
    return out


def _tr_axis_numpy(x, pad, stride, dil, k, n):
    """One axis of a transposed window: (input coordinate, valid) of every tap, shape x.shape + (k,).  Tap i of output
    coordinate x reads (x + pad - dil i) / stride when that division is exact and lands in [0, n)."""
    num = x[..., None].astype(np.int64) + pad - dil * np.arange(k)
    ok = (num >= 0) & (num % stride == 0)
    h = np.where(ok, num // stride, 0)
    ok &= h < n
    return np.where(ok, h, 0), ok


def gather_patches_tr3d_numpy(fmap, randt, randx, randy, B, k, pad, stride, relu, dilation=1, act=None,
                              act_param=None, in_scale=None, in_shift=None):
    """The patch gather of torch.nn.ConvTranspose3d in numpy: fmap (nimg, c, D, H, W) is the layer's input map, the
    points (t, x, y) lie in its output map; rows (batch, point, image), columns (c, kt, kh, kw), zero for invalid taps.
    k, pad, stride, dilation: ints or (t, h, w) triples; act ... in_shift as for gather_patches_numpy (the invalid
    taps stay +0)."""
    if act is not None or in_scale is not None or in_shift is not None:
        return _transformed(gather_patches_tr3d_numpy, fmap, (randt, randx, randy, B, k, pad, stride), relu, dilation,
                            act, act_param, in_scale, in_shift)
    (kt, kh, kw), (pt, ph, pw), (st, sh, sw), (dt, dh, dw) = (conv_triple(v) for v in (k, pad, stride, dilation))
    nimg, c, D, H, W = fmap.shape
    nbatch, P = np.asarray(randx).shape
    (tt, ot), (hh, oh), (ww, ow) = (_tr_axis_numpy(np.asarray(r), *a) for r, a in (
        (randt, (pt, st, dt, kt, D)), (randx, (ph, sh, dh, kh, H)), (randy, (pw, sw, dw, kw, W))))
    img = (np.arange(nbatch)[:, None, None] * B + np.arange(B)[None, None, :])[..., None, None, None, None]
    a = np.arange(c)[:, None, None, None]

    def ax(v, axis):  # (nbatch, P, k) -> broadcastable against (nbatch, P, B, c, kt, kh, kw) on tap axis 4 + axis
        shape = [nbatch, P, 1, 1, 1, 1, 1]
        shape[4 + axis] = v.shape[-1]
        return v.reshape(shape)

    vals = fmap[img, a, ax(tt, 0), ax(hh, 1), ax(ww, 2)]
    ok = ax(ot, 0) & ax(oh, 1) & ax(ow, 2)
    out = np.where(ok, vals, np.zeros((), dtype=fmap.dtype)).reshape(nbatch * P * B, c, kt, kh, kw)
    if relu:
        np.maximum(out, 0, out=out)
    return out


def gather_patches_tr_numpy(fmap, randx, randy, B, k, pad, stride, relu, dilation=1, act=None, act_param=None,
                            in_scale=None, in_shift=None):
    """gather_patches_tr3d_numpy for torch.nn.ConvTranspose2d: the one-frame case, columns (c, kh, kw).  k, pad,
    stride, dilation: ints or (h, w) pairs; act ... in_shift as for gather_patches_numpy."""
    if act is not None or in_scale is not None or in_shift is not None:
        return _transformed(gather_patches_tr_numpy, fmap, (randx, randy, B, k, pad, stride), relu, dilation, act,
                            act_param, in_scale, in_shift)
    (kh, kw), (ph, pw), (sh, sw), (dh, dw) = (conv_pair(v) for v in (k, pad, stride, dilation))
    X = gather_patches_tr3d_numpy(fmap[:, :, None], np.zeros_like(randx), randx, randy, B, (1, kh, kw), (0, ph, pw),
                                  (1, sh, sw), relu, dilation=(1, dh, dw))
    return X.reshape(X.shape[0], X.shape[1], kh, kw)


def fmap_nchw(d):
    """The feature map of a problem dict in the reference's blob order (nimg, c, H, W), whatever its HBM layout."""
    return d["fmap"].permute(0, 3, 1, 2) if d.get("layout", "nchw") == "nhwc" else d["fmap"]


def make_problem_device(shape: LayerShape, seed: int, eng, noise=0.01, pinned_host=False, layout="nchw", dtype=None,
                        host_layout="nchw"):
    """Device instance (torch CUDA generator), sized for BASELINE configs (GBs of feature maps).
    feats are produced with the library's own gather + a torch fp64 matmul: this is data
    generation, outside any timed region.
    layout: how the bottom blob sits in HBM.  'nhwc' (channels last, what a device-side forward provider hands over)
    takes the TMA gather; the VALUES are those of the 'nchw' instance of the same seed.
    host_layout: how the pinned host copy (fmap_host) is laid out: the reference's NCHW blob order, or 'nhwc'
    (channels last, what a user offloading a channels_last forward's maps hands over; the same values, and the dict
    then carries host_layout='nhwc').
    dtype: element type of the feature maps (fmap, fmap_host): None / torch.float32, or torch.bfloat16 /
    torch.float16 as a 16-bit forward pass would hand them over -- drawn in fp32 as for float32, then rounded; the
    targets are computed from the rounded map.
    A bn shape's dict carries in_scale / in_shift (bn_params, fp32 on device), and its targets come from X gathered
    through the shape's input transform."""
    import torch

    if isinstance(shape, LayerShape3d):
        return _make_problem3d_device(shape, seed, eng, noise, pinned_host, layout, dtype, host_layout)
    s = shape
    dev = eng.device
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    fmap = torch.randn((s.nbatch * s.B, s.c, s.H, s.W), generator=g, device=dev, dtype=torch.float32)
    if dtype is not None and dtype != torch.float32:
        fmap = fmap.to(dtype)
    r = np.random.RandomState(seed)
    randx = torch.as_tensor(r.randint(0, s.Ho, (s.nbatch, s.P)).astype(np.int32), device=dev)
    randy = torch.as_tensor(r.randint(0, s.Wo, (s.nbatch, s.P)).astype(np.int32), device=dev)
    W2 = torch.randn((s.n, s.c, s.kh, s.kw), generator=g, device=dev, dtype=torch.float32) * float(
        np.sqrt(2.0 / (s.c * s.k2)))
    b2 = 0.01 * torch.randn((s.n,), generator=g, device=dev, dtype=torch.float32)
    bn = {nm: torch.as_tensor(v, device=dev) for nm, v in zip(("in_scale", "in_shift"), bn_params(s.c, seed))} if s.bn else {}
    X = eng.patch_gather(fmap, randx, randy, s.B, s.P, **_xform_of(s, bn), **s.conv_args())
    Y = X.to(torch.float64) @ W2.reshape(s.n, -1).T.to(torch.float64) + b2.to(torch.float64)
    Y = Y + noise * Y.std() * torch.randn(Y.shape, generator=g, device=dev, dtype=torch.float64)
    feats = Y.to(torch.float32)
    samples = torch.as_tensor(r.randint(0, s.N, s.S).astype(np.int32), device=dev)
    seeds = r.randint(0, 2147483647, size=64)
    out = dict(fmap=fmap, randx=randx, randy=randy, W2=W2, b2=b2, feats=feats, samples=samples, seeds=seeds,
               layout=layout, **bn)
    del X, Y
    assert host_layout in ("nchw", "nhwc"), host_layout
    if pinned_host and host_layout == "nhwc":
        src = fmap.permute(0, 2, 3, 1)
        out["fmap_host"] = torch.empty(src.shape, dtype=fmap.dtype, pin_memory=True)
        out["fmap_host"].copy_(src)
        out["host_layout"] = "nhwc"
    elif pinned_host:
        out["fmap_host"] = torch.empty(fmap.shape, dtype=fmap.dtype, pin_memory=True)
        out["fmap_host"].copy_(fmap)
    if layout == "nhwc":
        out["fmap"] = fmap.permute(0, 2, 3, 1).contiguous()
        del fmap
    return out


def _make_problem3d_device(s, seed, eng, noise, pinned_host, layout, dtype, host_layout):
    """make_problem_device for a LayerShape3d.  layout / host_layout: 'ncdhw' or 'ndhwc' ('nchw' / 'nhwc', the 2-D
    defaults, are read as their 3-D forms); the dict carries both keys and randt."""
    import torch

    layout = {"nchw": "ncdhw", "nhwc": "ndhwc"}.get(layout, layout)
    host_layout = {"nchw": "ncdhw", "nhwc": "ndhwc"}.get(host_layout, host_layout)
    assert layout in ("ncdhw", "ndhwc") and host_layout in ("ncdhw", "ndhwc"), (layout, host_layout)
    dev = eng.device
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    fmap = torch.randn((s.nbatch * s.B, s.c, s.D, s.H, s.W), generator=g, device=dev, dtype=torch.float32)
    if dtype is not None and dtype != torch.float32:
        fmap = fmap.to(dtype)
    r = np.random.RandomState(seed)
    pts = [torch.as_tensor(r.randint(0, hi, (s.nbatch, s.P)).astype(np.int32), device=dev) for hi in (s.To, s.Ho, s.Wo)]
    W2 = torch.randn((s.n, s.c) + s.window, generator=g, device=dev, dtype=torch.float32) * float(
        np.sqrt(2.0 / (s.c * s.k2)))
    b2 = 0.01 * torch.randn((s.n,), generator=g, device=dev, dtype=torch.float32)
    bn = {nm: torch.as_tensor(v, device=dev) for nm, v in zip(("in_scale", "in_shift"), bn_params(s.c, seed))} if s.bn else {}
    X = eng.patch_gather3d(fmap, *pts, s.B, s.P, **_xform_of(s, bn), **s.conv_args())
    Y = X.to(torch.float64) @ W2.reshape(s.n, -1).T.to(torch.float64) + b2.to(torch.float64)
    Y = Y + noise * Y.std() * torch.randn(Y.shape, generator=g, device=dev, dtype=torch.float64)
    feats = Y.to(torch.float32)
    samples = torch.as_tensor(r.randint(0, s.N, s.S).astype(np.int32), device=dev)
    seeds = r.randint(0, 2147483647, size=64)
    out = dict(fmap=fmap, randt=pts[0], randx=pts[1], randy=pts[2], W2=W2, b2=b2, feats=feats, samples=samples,
               seeds=seeds, layout=layout, host_layout=host_layout, **bn)
    del X, Y
    if pinned_host:
        src = fmap.permute(0, 2, 3, 4, 1) if host_layout == "ndhwc" else fmap
        out["fmap_host"] = torch.empty(src.shape, dtype=fmap.dtype, pin_memory=True)
        out["fmap_host"].copy_(src)
    if layout == "ndhwc":
        out["fmap"] = fmap.permute(0, 2, 3, 4, 1).contiguous()
        del fmap
    return out
