"""Correct & Smooth (Huang et al., ICLR 2021; DESIGN §16): the parameter check and the host wrappers of its three
kernels -- cs_init_kernel and cs_combine_kernel (csrc/cs.cu) and the propagation step cs_prop_kernel (csrc/spmm.cu).
The distributed schedule of the steps is model/ops.py (_cs_step, correct_and_smooth).

`y` is an int32 tensor with one entry per row: the row's label where the row is fixed (a train row), else -1."""
from __future__ import annotations

import math
from dataclasses import dataclass
from numbers import Integral, Real
from typing import Optional, Tuple

import torch

from . import _lib

CS_CORRECT_LAYERS = 50
CS_CORRECT_ALPHA = 0.8
CS_SMOOTH_LAYERS = 50
CS_SMOOTH_ALPHA = 0.8
CS_SCALE = "auto"
AUTOSCALE_CUTOFF = 1000.0       # an autoscale above it is replaced by 1 (PyG's CorrectAndSmooth)
CLAMP, FIX = 0, 1               # post_mode of adaqp_cs_prop_f32


@dataclass(frozen=True)
class CSParams:
    correct_layers: int
    correct_alpha: float
    smooth_layers: int
    smooth_alpha: float
    scale: Optional[float]          # None: autoscale

    def as_dict(self) -> dict:
        return {"correct_layers": self.correct_layers, "correct_alpha": self.correct_alpha,
                "smooth_layers": self.smooth_layers, "smooth_alpha": self.smooth_alpha,
                "scale": "auto" if self.scale is None else self.scale}


def _layers(name: str, k) -> int:
    if isinstance(k, bool) or not (isinstance(k, Integral) or (isinstance(k, Real) and float(k).is_integer())):
        raise ValueError(f"{name}={k!r} is not an integer")
    if int(k) < 1:
        raise ValueError(f"{name}={k} must be at least 1")
    return int(k)


def _alpha(name: str, a) -> float:
    if isinstance(a, bool) or not isinstance(a, Real) or not 0.0 <= float(a) <= 1.0:
        raise ValueError(f"{name}={a!r} is outside [0, 1]")
    return float(a)


def cs_params(correct_layers=CS_CORRECT_LAYERS, correct_alpha=CS_CORRECT_ALPHA, smooth_layers=CS_SMOOTH_LAYERS,
              smooth_alpha=CS_SMOOTH_ALPHA, scale=CS_SCALE) -> CSParams:
    """The C&S parameters checked: the step counts integers >= 1, the alphas in [0, 1] (alpha = 1 is pure
    propagation), the scale `auto` or a finite number > 0 (a number given as a string is accepted)."""
    sc = None
    if not (isinstance(scale, str) and scale == "auto"):
        try:
            if isinstance(scale, bool):
                raise TypeError
            sc = float(scale)
        except (TypeError, ValueError):
            raise ValueError(f"cs_scale={scale!r} is neither 'auto' nor a number") from None
        if not (math.isfinite(sc) and sc > 0.0):
            raise ValueError(f"cs_scale={scale!r} must be 'auto' or a finite number > 0")
    return CSParams(_layers("cs_correct_layers", correct_layers), _alpha("cs_correct_alpha", correct_alpha),
                    _layers("cs_smooth_layers", smooth_layers), _alpha("cs_smooth_alpha", smooth_alpha), sc)


def _rows(t: torch.Tensor, C: int):
    assert t.dtype == torch.float32 and t.dim() == 2 and t.shape[1] == C and t.stride(1) == 1


def init(z: torch.Tensor, y: torch.Tensor, n_partials: int = 512) -> Tuple[torch.Tensor, torch.Tensor, float]:
    """(yhat, e0, l1): yhat = softmax(z) per row, e0 = onehot(y) - yhat on the fixed rows and 0 elsewhere, and l1 the
    float64 sum of |e0| over the rows -- summed exactly on the host from the kernel's per-CTA partials, so it depends
    only on z, y and n_partials."""
    rows, C = int(z.shape[0]), int(z.shape[1])
    _rows(z, C)
    assert y.dtype == torch.int32 and y.is_contiguous() and y.numel() == rows
    yhat, e0 = torch.empty_like(z), torch.empty_like(z)
    if rows == 0:
        return yhat, e0, 0.0
    partials = torch.empty(n_partials, dtype=torch.float64, device=z.device)
    rc = _lib.load().adaqp_cs_init_f32(z.data_ptr(), z.stride(0), y.data_ptr(), rows, C, yhat.data_ptr(),
                                       yhat.stride(0), e0.data_ptr(), e0.stride(0), partials.data_ptr(), n_partials,
                                       _lib.stream_ptr())
    _lib.check(rc, "adaqp_cs_init_f32")
    return yhat, e0, math.fsum(partials.cpu().tolist())


def combine(yhat: torch.Tensor, e: torch.Tensor, y: torch.Tensor, sigma: Optional[float] = None,
            scale: Optional[float] = None) -> torch.Tensor:
    """g0 = onehot(y) on the fixed rows, yhat + s e elsewhere: s = sigma / |e|_1 per row with `sigma` (autoscale; 1
    where |e|_1 = 0 or the ratio exceeds AUTOSCALE_CUTOFF), else the fixed `scale`."""
    assert (sigma is None) != (scale is None), "exactly one of sigma (autoscale) and scale"
    rows, C = int(yhat.shape[0]), int(yhat.shape[1])
    _rows(yhat, C)
    _rows(e, C)
    assert y.dtype == torch.int32 and y.is_contiguous() and y.numel() == rows and e.shape[0] == rows
    g0 = torch.empty_like(yhat)
    auto = sigma is not None
    rc = _lib.load().adaqp_cs_combine_f32(yhat.data_ptr(), yhat.stride(0), e.data_ptr(), e.stride(0), y.data_ptr(),
                                          rows, C, 1 if auto else 0, float(sigma if auto else scale), g0.data_ptr(),
                                          g0.stride(0), _lib.stream_ptr())
    _lib.check(rc, "adaqp_cs_combine_f32")
    return g0


def prop(graph, x_local: torch.Tensor, x_halo: Optional[torch.Tensor], pre: Optional[torch.Tensor],
         post: Optional[torch.Tensor], scale: float, alpha: float, row_begin: int = 0, row_end: Optional[int] = None,
         out: Optional[torch.Tensor] = None, tele: Optional[torch.Tensor] = None, y: Optional[torch.Tensor] = None,
         fix: Optional[torch.Tensor] = None, lo: float = -math.inf, hi: float = math.inf, stream=None) -> torch.Tensor:
    """One C&S step over whole CSR rows [row_begin, row_end) of a LocalGraph (cs_prop_kernel):
        r[v] = scale * post[v] * sum_u pre[u] x[u]  (+ alpha * tele[v])
    clamped to [lo, hi]; or, with `fix` (and `y`), out[v] = fix[v] on the rows with y >= 0 -- whose gather is
    skipped -- and r[v] without the tele term elsewhere.  tele, y, fix and out are indexed v - row_begin."""
    row_end = graph.n_inner if row_end is None else int(row_end)
    F = int(x_local.shape[1])
    assert x_local.dtype == torch.float32 and x_local.stride(1) == 1
    if out is None:
        out = torch.empty((row_end - row_begin, F), dtype=torch.float32, device=x_local.device)
    if x_halo is not None and x_halo.shape[0] == 0:
        x_halo = None
    for t in (tele, fix):
        assert t is None or (t.dtype == torch.float32 and t.stride(1) == 1 and t.shape[0] >= row_end - row_begin)
    if fix is not None:
        assert y is not None and y.dtype == torch.int32 and y.is_contiguous() and y.numel() >= row_end - row_begin
    rc = _lib.load().adaqp_cs_prop_f32(
        graph.indptr.data_ptr(), graph.indices.data_ptr(), x_local.data_ptr(), x_local.stride(0), graph.n_inner,
        x_halo.data_ptr() if x_halo is not None else None, x_halo.stride(0) if x_halo is not None else 0,
        pre.data_ptr() if pre is not None else None, post.data_ptr() if post is not None else None,
        float(scale), float(alpha), tele.data_ptr() if tele is not None else None,
        tele.stride(0) if tele is not None else 0, y.data_ptr() if fix is not None else None,
        fix.data_ptr() if fix is not None else None, fix.stride(0) if fix is not None else 0,
        FIX if fix is not None else CLAMP, float(lo), float(hi), int(row_begin), row_end, F, out.data_ptr(),
        out.stride(0), _lib.stream_ptr(stream))
    _lib.check(rc, "adaqp_cs_prop_f32")
    return out
