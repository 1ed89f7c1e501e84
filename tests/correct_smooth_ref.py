"""fp64 restatement of the reference's Correct & Smooth (cogdl/models/nn/correct_smooth.py: CorrectSmooth.__call__ with
train_only, and diffusion with p = 1) on a graph given as COO (row, col), numpy only.  Normalisations as the
reference's Graph.normalize on an edge_index-built graph: degrees count each edge at its row, "sym" weighs an edge
d[r]^-1/2 d[c]^-1/2, "row" 1/d[r], "col" 1/d'[c] with d' counting each edge at its column; a zero degree gives 0."""
import numpy as np
import scipy.sparse as sp


def _inv(d, p):
    with np.errstate(divide="ignore"):
        out = np.power(d, p)
    out[~np.isfinite(out)] = 0.0
    return out


def adjacency(row, col, n, norm):
    d_row = np.bincount(row, minlength=n).astype(np.float64)
    d_col = np.bincount(col, minlength=n).astype(np.float64)
    if norm == "sym":
        w = _inv(d_row, -0.5)[row] * _inv(d_row, -0.5)[col]
    elif norm == "row":
        w = _inv(d_row, -1.0)[row]
    elif norm == "col":
        w = _inv(d_col, -1.0)[col]
    else:
        raise ValueError(norm)
    return sp.csr_matrix((w, (row, col)), shape=(n, n))


def propagate(A, labels, alpha, nprop, post):
    out = labels.copy()
    for _ in range(nprop):
        out = post(alpha * (A @ out) + (1.0 - alpha) * labels)
    return out


def correct_smooth_fp64(row, col, n, preds, y, train_mask, autoscale, correct_norm, smooth_norm, correct_alpha,
                        smooth_alpha, nprop_correct, nprop_smooth, scale=1.0):
    preds = preds.astype(np.float64)
    C = int(y.max()) + 1
    train = np.flatnonzero(train_mask)
    onehot = np.eye(C)[y]
    err = np.zeros((n, C))
    err[train] = onehot[train] - preds[train]

    def reset(x):
        x[train] = err[train]
        return x

    clip_correct = (lambda x: np.clip(x, -1.0, 1.0)) if autoscale else reset
    resid = propagate(adjacency(row, col, n, correct_norm), err, correct_alpha, nprop_correct, clip_correct)
    if autoscale:
        orig_diff = np.abs(err[train]).sum() / train.shape[0]
        with np.errstate(divide="ignore", invalid="ignore"):
            s = orig_diff / np.abs(resid).sum(axis=1, keepdims=True)
        s[np.isinf(s) | (s > 1000)] = 1.0
        res = preds + s * resid
        res[np.isnan(res)] = preds[np.isnan(res)]
    else:
        res = preds + scale * resid
    start = res.copy()
    start[train] = onehot[train]
    return propagate(adjacency(row, col, n, smooth_norm), start, smooth_alpha, nprop_smooth,
                     lambda x: np.clip(x, 0.0, 1.0))


def diffusion_fp64(A, x, nhtop, alpha=0.5):
    x = x.astype(np.float64)
    for _ in range(nhtop):
        x = (1.0 - alpha) * x + alpha * (A @ x)
    return x
