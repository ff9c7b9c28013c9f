"""Float64 statement of the feature-metric cost of a level (banet_lm_cost): with s_n = sum_c d_{n,c}^2 point n's squared residual norm at
the iterate (tests/robust_oracle.py: 0 at masked points), c_n its weight (1 without one) and rho the robust loss,
  cost[b] = sum_n c_n rho(s_n)      rho(s) = s (no loss), Huber s (s <= delta^2) / 2 delta sqrt(s) - delta^2, Cauchy delta^2 log(1 + s / delta^2)
whose derivative is robust_oracle.rho1.  Differentiable by float64 autograd in every input, the weight included; the residual is sampled
by the oracle's bilinear resampler, so the gradient is the exact derivative of the cost through the F2 values, not the Gauss-Newton one."""
import torch

import robust_oracle as RO


def rho(kind, delta: float, s: torch.Tensor) -> torch.Tensor:
    """rho(s) of the robust loss `kind` (None, "huber" or "cauchy") with scale delta; rho(0) = 0 for every kind."""
    if kind is None:
        return s
    t = float(delta) ** 2
    if kind == "huber":
        return torch.where(s <= t, s, 2.0 * float(delta) * torch.sqrt(torch.clamp(s, min=t)) - t)
    if kind == "cauchy":
        return t * torch.log1p(s / t)
    raise ValueError(f"unknown robust loss {kind!r}")


def cost_from_norms(s: torch.Tensor, kind=None, delta: float = 0.0, weight=None) -> torch.Tensor:
    """[nb] from the squared norms s [nb,N] (0 at masked points) and weight [nb,N,1] or None."""
    r = rho(kind, delta, s)
    return (r if weight is None else weight.reshape(s.shape) * r).sum(-1)


def cost(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, kind=None, delta: float = 0.0, weight=None, guard_nonfinite: bool = True):
    """cost [nb] of the level at (R, T, W); conv2 is the [F2|gx|gy] map (only its F2 channels enter)."""
    s = RO.squared_norms(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, guard_nonfinite)
    return cost_from_norms(s, kind, delta, weight)
