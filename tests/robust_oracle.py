"""Float64 statement of the robust feature-metric loss (banet_level_t::robust): one IRLS step per iteration.  With s_n = sum_c d_c^2 point
n's squared residual norm at the current iterate and c_n its confidence weight (1 without one), point n enters the weighted normal
equations of tests/weighted_oracle.py with w_n = c_n rho'(s_n):
  Huber   rho(s) = s (s <= delta^2), 2 delta sqrt(s) - delta^2      rho'(s) = 1 or delta / sqrt(s)
  Cauchy  rho(s) = delta^2 log(1 + s / delta^2)                    rho'(s) = delta^2 / (delta^2 + s)
H has no rho'' term, and the mean |residual| (lambda) and the in-bounds count stay unweighted.  w_n is a function of the iterate, so
float64 autograd through it carries the rho'' term of the exact gradient; detach_weight=True drops it (the reference for the test that
the kernels keep it)."""
import torch

import weighted_oracle as WO
from oracle import ba_oracle as O


def rho1(kind: str, delta: float, s: torch.Tensor) -> torch.Tensor:
    """rho'(s) of the robust loss `kind` ("huber" or "cauchy") with scale delta; differentiable in s (Huber: away from s = delta^2)."""
    t = float(delta) ** 2
    if kind == "huber":
        return torch.where(s <= t, torch.ones_like(s), float(delta) / torch.sqrt(torch.clamp(s, min=t)))
    if kind == "cauchy":
        return t / (t + s)
    raise ValueError(f"unknown robust loss {kind!r}")


def squared_norms(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, guard_nonfinite: bool = True) -> torch.Tensor:
    """s_n = |d_n|^2 [nb,N] at the iterate (R, T, W); 0 at masked points."""
    _, _, _, diff, m = WO._point_system(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, guard_nonfinite)
    return (diff.squeeze(-1) ** 2).sum(-1) * (m > 0)


def robust_weight(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, kind, delta, weight=None, detach_weight: bool = False,
                  guard_nonfinite: bool = True) -> torch.Tensor:
    """w_n = c_n rho'(s_n) [nb,N,1] at the iterate (R, T, W); weight [nb,N,1] is c_n (None: ones)."""
    s = squared_norms(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, guard_nonfinite)
    w = rho1(kind, delta, s).unsqueeze(-1)
    if detach_weight:
        w = w.detach()
    return w if weight is None else weight * w


def normal_equations(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, kind, delta, weight=None, detach_weight: bool = False,
                     guard_nonfinite: bool = True):
    """H [nb,P,P], g [nb,P,1], rbar [nb,1,C], nvalid [nb] of one robust build (weighted_oracle.normal_equations with w_n)."""
    args = (conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W)
    w = robust_weight(*args, kind, delta, weight, detach_weight, guard_nonfinite)
    return WO.normal_equations(*args, w, guard_nonfinite)


def iteration(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, mlp_params, kind, delta, weight=None, opts: O.IterOptions = O.IterOptions(),
              detach_weight: bool = False):
    """weighted_oracle.iteration with w_n = c_n rho'(s_n) evaluated at (R, T, W) -> (R', T', W' or None)."""
    args = (conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W)
    w = robust_weight(*args, kind, delta, weight, detach_weight, opts.guard_nonfinite)
    return WO.iteration(*args, mlp_params, w, opts)


def solve(levels, kind, deltas, iters_per_level: int, R, T, W, weights=None, opts: O.IterOptions = O.IterOptions()):
    """Coarse-to-fine: `iters_per_level` robust iterations per level (oracle.LevelInputs, its own lambda-MLP), delta per level, W carried."""
    weights = weights if weights is not None else [None] * len(levels)
    for lv, delta, wt in zip(levels, deltas, weights):
        for _ in range(iters_per_level):
            R, T, W = iteration(lv.conv1, lv.conv2, lv.fx, lv.fy, lv.ox, lv.oy, lv.p, lv.D, lv.B, R, T, W, lv.mlp, kind, delta, wt, opts)
    return R, T, W
