"""Test-side oracle for transposed convolutions (torch.nn.ConvTranspose2d / ConvTranspose3d semantics, groups == 1).

  gather_tr3d / gather_tr   the transposed patch gather restated in numpy, tap by tap: rows (batch, point, image),
                            columns (c, kt, kh, kw) / (c, kh, kw); fmap is the layer's INPUT map, the points lie in its
                            output map
  taps_brute                the valid taps of one axis, every tap tested
  taps_by_phase             the same from the point's phase (first valid tap and step), as csrc/gather_tr.cu finds them
"""
import math

import numpy as np


def _triple(v):
    return tuple(int(x) for x in v) if isinstance(v, (tuple, list)) else (int(v),) * 3


def _pair(v):
    return tuple(int(x) for x in v) if isinstance(v, (tuple, list)) else (int(v),) * 2


def taps_brute(x, pad, stride, dil, k, n):
    """[(tap i, input coordinate h)] of output coordinate x: h = (x + pad - dil i) / stride exact and 0 <= h < n.  A
    negative numerator is skipped before it is tested for divisibility."""
    out = []
    for i in range(k):
        num = x + pad - dil * i
        if num < 0 or num % stride:
            continue
        if num // stride < n:
            out.append((i, num // stride))
    return out


def taps_by_phase(x, pad, stride, dil, k, n):
    """taps_brute from the phase of x: with g = gcd(stride, dil), nothing unless g divides x + pad; otherwise the taps
    i0, i0 + stride/g, ... (d i0 = x + pad mod stride), clipped to the ones whose input coordinate lies in [0, n),
    consecutive ones dil/g input coordinates apart.  The arithmetic of tr_taps in csrc/gather_tr.cu."""
    num = x + pad
    g = math.gcd(stride, dil)
    if num % g:
        return []
    period = stride // g
    i0 = 0
    while (num - dil * i0) % stride:
        i0 += 1
    over = num - stride * (n - 1)
    lo = -(-over // dil) if over > 0 else 0
    first = i0 + (-(-(lo - i0) // period) * period if lo > i0 else 0)
    last = min(k - 1, num // dil)
    if first > last:
        return []
    h0, step = (num - dil * first) // stride, dil // g
    return [(first + m * period, h0 - m * step) for m in range((last - first) // period + 1)]


def gather_tr3d(fmap, randt, randx, randy, B, k, pad, stride, dilation=1, relu=False):
    """fmap (nimg, c, D, H, W), any float type (kept); the sampled output points (nbatch, P).  Returns
    (nbatch*P*B, c*kt*kh*kw), ReLU'd with np.maximum when relu."""
    (kt, kh, kw), (pt, ph, pw), (st, sh, sw), (dt, dh, dw) = (_triple(v) for v in (k, pad, stride, dilation))
    nimg, c, D, H, W = fmap.shape
    nbatch, P = np.asarray(randx).shape
    X = np.zeros((nbatch * P * B, c, kt, kh, kw), dtype=fmap.dtype)
    for b in range(nbatch):
        for p in range(P):
            rows = slice((b * P + p) * B, (b * P + p + 1) * B)
            for u, t in taps_brute(int(randt[b][p]), pt, st, dt, kt, D):
                for i, h in taps_brute(int(randx[b][p]), ph, sh, dh, kh, H):
                    for j, w in taps_brute(int(randy[b][p]), pw, sw, dw, kw, W):
                        X[rows, :, u, i, j] = fmap[b * B:(b + 1) * B, :, t, h, w]
    X = X.reshape(nbatch * P * B, -1)
    return np.maximum(X, 0) if relu else X


def gather_tr(fmap, randx, randy, B, k, pad, stride, dilation=1, relu=False):
    """gather_tr3d on the one-frame map (nimg, c, 1, H, W): the ConvTranspose2d gather, columns (c, kh, kw)."""
    (kh, kw), (ph, pw), (sh, sw), (dh, dw) = (_pair(v) for v in (k, pad, stride, dilation))
    return gather_tr3d(fmap[:, :, None], np.zeros_like(np.asarray(randx)), randx, randy, B, (1, kh, kw), (0, ph, pw),
                       (1, sh, sw), (1, dh, dw), relu)
