"""Test-side oracle for Conv3d layers (torch.nn.Conv3d semantics, groups == 1), built on oracle/cp_oracle.py without
changing it.

  gather3d      the 3-D patch gather restated in numpy: rows (batch, point, image), columns (c, kt, kh, kw)
  dictionary    cp_oracle.dictionary for X (N, c, kt, kh, kw): its search and least squares see X as (N, c, k2)
"""
import numpy as np

import conv_oracle


def _triple(v):
    return tuple(int(x) for x in v) if isinstance(v, (tuple, list)) else (int(v),) * 3


def gather3d(fmap, randt, randx, randy, B, k, pad, stride, dilation=1, relu=False):
    """fmap (nimg, c, D, H, W) float64 (or any float type, kept); the sampled points (nbatch, P).  Output point
    (t, x, y) reads (st t - pt + dt u, sh x - ph + dh i, sw y - pw + dw j), zero outside the map.  Returns
    (nbatch*P*B, c*kt*kh*kw), ReLU'd with np.maximum when relu."""
    (kt, kh, kw), (pt, ph, pw), (st, sh, sw), (dt, dh, dw) = (_triple(v) for v in (k, pad, stride, dilation))
    nimg, c, D, H, W = fmap.shape
    nbatch, P = np.asarray(randx).shape
    rows = []
    for b in range(nbatch):
        for p in range(P):
            tt = st * int(randt[b][p]) - pt + dt * np.arange(kt)
            yy = sh * int(randx[b][p]) - ph + dh * np.arange(kh)
            xx = sw * int(randy[b][p]) - pw + dw * np.arange(kw)
            inside = ((tt >= 0) & (tt < D))[:, None, None] & ((yy >= 0) & (yy < H))[None, :, None] & \
                ((xx >= 0) & (xx < W))[None, None, :]
            for i in range(B):
                img = fmap[b * B + i]
                win = img[:, np.clip(tt, 0, D - 1)][:, :, np.clip(yy, 0, H - 1)][:, :, :, np.clip(xx, 0, W - 1)]
                rows.append(np.where(inside[None], win, 0).reshape(-1))
    X = np.stack(rows)
    return np.maximum(X, 0) if relu else X


def dictionary(X, W2, Y, **kw):
    """cp_oracle.dictionary on X (N, c, kt, kh, kw), W2 (n, c, kt, kh, kw): run on the (N, c, 1, k2) view (through
    conv_oracle.dictionary, which takes the least-squares weights from fc_kernel for non-square views), then the
    weights reshaped to (n, c', kt, kh, kw).  Same masks, alpha state, probes and RNG draws as the oracle."""
    X = np.asarray(X)
    N, c = X.shape[:2]
    win = tuple(X.shape[2:])
    k2 = int(np.prod(win))
    n = np.asarray(W2).shape[0]
    idxs, W, B = conv_oracle.dictionary(X.reshape(N, c, 1, k2), np.asarray(W2).reshape(n, c, 1, k2), Y, **kw)
    return idxs, W.reshape((n, -1) + win), B
