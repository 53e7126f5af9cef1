"""float64 numpy restatement of Correct & Smooth (DESIGN.md §16) and of its distributed exchange protocol.

    A = D^-1/2 A D^-1/2 (per edge u -> v: pre[u] * post[v], pre = out_deg^-1/2, post = in_deg^-1/2), APPNP's A
    set-up:  yhat = softmax(z);  e0 = onehot(y) - yhat on the labelled rows (y >= 0), 0 elsewhere;
             sigma = sum |e0| / n_train
    correct: e_{k+1} = P(a1 A e_k + (1 - a1) e0), e_0 = e0, k < K1
             scale None (autoscale): P = clamp(-1, 1); zc = yhat + s e_K, s = sigma / |e_K|_1 per row, s = 1 where
                                     |e_K|_1 = 0 or s > 1000
             scale c (fixed):        P resets the labelled rows to e0;   zc = yhat + c e_K
    smooth:  g0 = zc with the labelled rows replaced by onehot(y);  g_{k+1} = clamp(a2 A g_k + (1 - a2) g0, 0, 1)
    result:  g_K

`monolithic` runs it on a whole graph, `distributed` on every rank of prepared layouts (manager.layout) with each
step's exchange simulated exactly (gat_oracle.exchange); both return the same fields.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence

import numpy as np

from .appnp_oracle import _local, _pow, matrix
from .gat_oracle import exchange, global_from_layouts  # noqa: F401  (re-exported for the tests)

CUTOFF = 1000.0


def softmax(z: np.ndarray) -> np.ndarray:
    z = np.asarray(z, np.float64)
    e = np.exp(z - z.max(1, keepdims=True))
    return e / e.sum(1, keepdims=True)


def onehot(y: np.ndarray, C: int) -> np.ndarray:
    """Rows of onehot(y) where y >= 0, zero rows elsewhere."""
    y = np.asarray(y)
    out = np.zeros((y.size, C))
    lab = np.nonzero(y >= 0)[0]
    out[lab, y[lab]] = 1.0
    return out


def autoscale_ratio(sigma: float, e: np.ndarray) -> np.ndarray:
    """sigma / |e|_1 per row before the cut-off (inf where the row is zero)."""
    l1 = np.abs(e).sum(1)
    with np.errstate(divide="ignore"):
        return np.where(l1 > 0, sigma / np.where(l1 > 0, l1, 1.0), np.inf)


def autoscale(sigma: float, e: np.ndarray) -> np.ndarray:
    r = autoscale_ratio(sigma, e)
    return np.where(np.isfinite(r) & (r <= CUTOFF), r, 1.0)


def _run(prop: Callable[[List[np.ndarray]], List[np.ndarray]], zs: Sequence[np.ndarray], ys: Sequence[np.ndarray],
         k1: int, a1: float, k2: int, a2: float, scale: Optional[float]) -> dict:
    C = np.asarray(zs[0]).shape[1]
    yhat = [softmax(z) for z in zs]
    lab = [np.asarray(y) >= 0 for y in ys]
    hot = [onehot(y, C) for y in ys]
    e0 = [np.where(m[:, None], h - p, 0.0) for m, h, p in zip(lab, hot, yhat)]
    n_train = sum(int(m.sum()) for m in lab)
    sigma = sum(float(np.abs(e).sum()) for e in e0) / max(n_train, 1)
    e = e0
    for _ in range(k1):
        ae = prop(e)
        if scale is None:
            e = [np.clip(a1 * x + (1 - a1) * t, -1.0, 1.0) for x, t in zip(ae, e0)]
        else:
            e = [np.where(m[:, None], t, a1 * x + (1 - a1) * t) for x, t, m in zip(ae, e0, lab)]
    if scale is None:
        ratio = [autoscale_ratio(sigma, x) for x in e]
        zc = [p + autoscale(sigma, x)[:, None] * x for p, x in zip(yhat, e)]
    else:
        ratio = [np.full(x.shape[0], float(scale)) for x in e]
        zc = [p + scale * x for p, x in zip(yhat, e)]
    g0 = [np.where(m[:, None], h, x) for m, h, x in zip(lab, hot, zc)]
    g = g0
    for _ in range(k2):
        ag = prop(g)
        g = [np.clip(a2 * x + (1 - a2) * t, 0.0, 1.0) for x, t in zip(ag, g0)]
    return {"yhat": yhat, "e0": e0, "sigma": sigma, "n_train": n_train, "e": e, "ratio": ratio, "g0": g0, "g": g}


def monolithic(indptr, indices, z, y, k1=50, a1=0.8, k2=50, a2=0.8, scale=None) -> dict:
    """C&S on an unpartitioned graph (no halo); every field a one-element list."""
    deg = np.diff(np.asarray(indptr, np.int64))
    A = matrix(indptr, indices, deg.size, _pow(deg, -0.5), _pow(deg, -0.5))
    return _run(lambda xs: [A @ xs[0]], [z], [y], k1, a1, k2, a2, scale)


def distributed(layouts, zs, ys, k1=50, a1=0.8, k2=50, a2=0.8, scale=None) -> dict:
    """C&S on every rank of `layouts`: each step exchanges the rows it propagates (the fp32 exchange of CS_KEY) and
    applies the rank's forward operator to its inner rows; sigma sums every rank's labelled errors."""
    As = [_local(L, True) for L in layouts]

    def prop(xs):
        halo = exchange(xs, layouts)
        return [A @ np.concatenate([x, h]) for A, x, h in zip(As, xs, halo)]

    return _run(prop, [np.asarray(z, np.float64) for z in zs], ys, k1, a1, k2, a2, scale)
