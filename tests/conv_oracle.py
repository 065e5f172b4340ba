"""Test-side oracle for convolution windows beyond the reference's square, odd, undilated ones (rectangular kernels,
per-axis padding and stride, dilation), built on oracle/cp_oracle.py without changing it.

  extract_XY_conv   cp_oracle.extract_XY restated with the semantics of torch.nn.Conv2d (groups == 1)
  dictionary        cp_oracle.dictionary for X (N, c, kh, kw) with kh != kw
"""
import numpy as np

import cp_oracle


def _pair(v):
    return (int(v[0]), int(v[1])) if isinstance(v, (tuple, list)) else (int(v), int(v))


def extract_XY_conv(forward, X_name, Y_spec, points_dict):
    """Y_spec.kernel_size, .pad, .stride and .dilation (default 1) are ints or (h, w) pairs.  Output point (x, y)
    reads the taps (stride_h x - pad_h + dil_h i, stride_w y - pad_w + dil_w j), i < kh, j < kw, zero outside the map.
    Returns the (N*kh*kw, c) float64 matrix, rows (sample, i, j) -- cp_oracle.extract_XY's layout; for square, odd,
    undilated windows the two agree bit for bit."""
    (kh, kw), (ph, pw), (sh, sw) = _pair(Y_spec.kernel_size), _pair(Y_spec.pad), _pair(Y_spec.stride)
    dh, dw = _pair(getattr(Y_spec, "dilation", 1))
    Y = Y_spec.name
    P = points_dict["nPointsPerLayer"]
    rows = []
    for batch in range(points_dict["nBatches"]):
        blob = forward(batch)[X_name]
        B, c, H, W = blob.shape
        feat = np.zeros((B, c, H + 2 * ph + dh * kh, W + 2 * pw + dw * kw), dtype=blob.dtype)
        feat[:, :, ph:H + ph, pw:W + pw] = blob
        for x, y in zip(points_dict[(batch, Y, "randx")][:P], points_dict[(batch, Y, "randy")][:P]):
            win = feat[:, :, sh * x:sh * x + dh * (kh - 1) + 1:dh, sw * y:sw * y + dw * (kw - 1) + 1:dw]
            rows.append(np.moveaxis(win, 1, -1).reshape((B * kh * kw, c)))
    return np.concatenate(rows).astype(np.float64)


def dictionary(X, W2, Y, **kw):
    """cp_oracle.dictionary on X (N, c, kh, kw), W2 (n, c, kh, kw) with any kh, kw.  Its channel search and least
    squares only see X.reshape(N, c, -1); only its last reshape of the weights assumes w = h (decompose.py:401-402).
    So for kh != kw the least-squares weights are taken as fc_kernel returns them, (n, c'*kh*kw), and the reshape is
    fed a placeholder of the size it expects.  Returns (idxs, newW2 (n, c', kh, kw), newB2) and the same alpha state,
    probes and RNG draws as the oracle."""
    X = np.asarray(X)
    N, c, kh, kw_ = X.shape
    if kh == kw_:
        return cp_oracle.dictionary(X, W2, Y, **kw)
    assert not kw.get("DEBUG"), "DEBUG returns X, not weights: call cp_oracle.dictionary"
    n = np.asarray(W2).shape[0]
    orig = cp_oracle.fc_kernel
    got = {}

    def fc_kernel(Xs, Ys, **a):
        Wn, Bn = orig(Xs, Ys, **a)
        got["W"] = Wn
        rank = Wn.shape[1] // (kh * kw_)
        return np.zeros((n, rank * kh * kh)), Bn  # the shape the oracle's (n, rank, h, h) reshape needs

    cp_oracle.fc_kernel = fc_kernel
    try:
        idxs, _, newB2 = cp_oracle.dictionary(X, W2, Y, **kw)
    finally:
        cp_oracle.fc_kernel = orig
    return idxs, got["W"].reshape((n, -1, kh, kw_)), newB2
