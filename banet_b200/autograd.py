"""Differentiable BundleIteration / CameraIteration.

Two training paths:
  * `iteration_fused` (default): torch.autograd.Functions over the fused sm_90a kernels — forward banet_lm_build /
    banet_lm_solve_update, backward banet_lm_build_bwd / banet_lm_solve_update_bwd (banet_b200/csrc/lm_bwd.cu): nothing per-pixel
    (J, G, d, the tiled upstream gradients of utils.cu:613-617) is materialised, so it runs at any N and K <= 256.  The lambda-MLP
    (5 dense layers on a [nb,C] vector, bundlenet.py:244-248) stays stock torch in between.  Gradient signature = the reference's:
    conv1, conv2, D, B, R, T, W and the lambda-MLP parameters (TF autodiff + the registered op gradient, bundlenet.py:79-82).
    `window_iteration_fused` is the same for the joint keyframe window (banet_lm_window_solve_update / _bwd after the per-pair build),
    `window_batch_iteration_fused` for a batch of windows (banet_lm_window_batch_solve_update / _bwd).
  * `iteration` (the reference's own split of labour, kept as the A/B baseline and for op-level drop-in use):

    reference:  TF graph ops (warp, resampler, Jacobians, damping, solve, update; TF autodiff)  +  native op
                `equation_construction` with its registered native gradient (bundlenet.py:76-82, 263)
    here:       the same graph in stock torch CUDA ops (torch autograd)                          +  native op
                `ops.equation_construction` = banet_eqc_fwd / banet_eqc_bwd (sm_90a)

This is the TRAINING path: it materialises J[nb,N,2,P], G[nb,N,C,2], d[nb,N,C,1] exactly like the reference does
(so it is meant for the reference's training regime, N <= a few thousand sampled points).  The fused kernels
(`ops.lm_build` ...) are the inference / no-grad path; a fused analytic backward is a later-round item (DESIGN.md §7).
Gradient signature = every float input: conv1, conv2, D, B, R, T, W and the lambda-MLP parameters.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import torch

from . import ops

Tensor = torch.Tensor
_SELU_ALPHA, _SELU_SCALE = 1.6732632423543772, 1.0507009873554805


def _resampler(data: Tensor, x: Tensor, y: Tensor) -> Tensor:
    """bilinear, zero outside (tf.contrib.resampler semantics); differentiable w.r.t. data and coordinates."""
    nb, h, w, C = data.shape
    x0f, y0f = torch.floor(x), torch.floor(y)
    dx, dy = (x - x0f).unsqueeze(-1), (y - y0f).unsqueeze(-1)
    x0, y0 = x0f.long(), y0f.long()
    flat = data.reshape(nb, h * w, C)
    out = 0
    for xi, yi, wg in ((x0, y0, (1 - dx) * (1 - dy)), (x0 + 1, y0, dx * (1 - dy)), (x0, y0 + 1, (1 - dx) * dy), (x0 + 1, y0 + 1, dx * dy)):
        ok = ((xi >= 0) & (xi < w) & (yi >= 0) & (yi < h)).unsqueeze(-1).to(data.dtype)
        idx = (yi.clamp(0, h - 1) * w + xi.clamp(0, w - 1)).unsqueeze(-1).expand(-1, -1, C)
        out = out + torch.gather(flat, 1, idx) * (wg * ok)
    return out


def _rodrigues(w: Tensor) -> Tensor:
    """bundlenet.py:17-37 (theta clamped to 1e-6).  w [nb,3] -> [nb,3,3]"""
    th = torch.sqrt((w * w).sum(1)).clamp_min(1e-6)
    k = w / th.unsqueeze(1)
    c, s = torch.cos(th), torch.sin(th)
    kx, ky, kz = k[:, 0], k[:, 1], k[:, 2]
    oc = 1 - c
    rows = [c + kx * kx * oc, kx * ky * oc - kz * s, ky * s + kx * kz * oc,
            kz * s + kx * ky * oc, c + ky * ky * oc, -kx * s + ky * kz * oc,
            -ky * s + kx * kz * oc, kx * s + ky * kz * oc, c + kz * kz * oc]
    return torch.stack(rows, 1).reshape(-1, 3, 3)


def _vmatrix(w: Tensor) -> Tensor:
    """bundlenet.py:39-46, per pair (series below 1e-4 like the CUDA path)."""
    th2 = (w * w).sum(1)
    th = torch.sqrt(th2.clamp_min(1e-30))
    small = th < 1e-4
    ths = torch.where(small, torch.ones_like(th), th)
    ca = torch.where(small, 0.5 - th2 / 24, (1 - torch.cos(ths)) / (ths * ths))
    cb = torch.where(small, 1.0 / 6 - th2 / 120, (ths - torch.sin(ths)) / (ths * ths * ths))
    z = torch.zeros_like(th)
    K = torch.stack([z, -w[:, 2], w[:, 1], w[:, 2], z, -w[:, 0], -w[:, 1], w[:, 0], z], 1).reshape(-1, 3, 3)
    eye = torch.eye(3, device=w.device, dtype=w.dtype).unsqueeze(0)
    return eye + ca.view(-1, 1, 1) * K + cb.view(-1, 1, 1) * (K @ K)


def lambda_mlp(avg_residual: Tensor, params: Sequence[Tuple[Tensor, Tensor]]) -> Tensor:
    h = avg_residual
    for i, (Wt, b) in enumerate(params):
        h = h @ Wt + b
        h = torch.tanh(h) if i == len(params) - 1 else _SELU_SCALE * torch.where(h > 0, h, _SELU_ALPHA * torch.expm1(h))
    return h


def iteration(conv1, conv2, intr, p, D, B, R, T, W, mlp_params, l2_regularizer_base: Optional[float],
              damping_eps: float = 1e-5, exact_sym: bool = False, lambda_override: Optional[Tensor] = None):
    """One differentiable LM iteration.  B/W None -> CameraIteration (bundlenet.py:122-191), else BundleIteration (:193-278).
    intr [nb,4].  Returns (R', T', W')."""
    nb, N, C = conv1.shape
    h, w = conv2.shape[1], conv2.shape[2]
    fx, fy, ox, oy = [intr[:, i:i + 1] for i in range(4)]
    bundle = B is not None
    Dt = (D + B @ W) if bundle else D                                             # :208
    Rp = R @ p                                                                    # :209
    X = Rp * Dt.transpose(1, 2) + T                                               # :211-214
    Z = X[:, 2]; x = X[:, 0] / Z; y = X[:, 1] / Z                                 # :216-221
    px, py = fx * x + ox, fy * y + oy                                             # :223-224
    ok = (px >= 0) & (px <= w - 1) & (py >= 0) & (py <= h - 1) & torch.isfinite(px) & torch.isfinite(py)   # :231 (+ finite guard)
    pxs, pys = torch.where(ok, px, torch.zeros_like(px)), torch.where(ok, py, torch.zeros_like(py))
    s = _resampler(conv2, pxs, pys)                                               # :230
    m = ok.to(conv1.dtype).unsqueeze(-1)
    diff = ((conv1 - s[..., :C]) * m).unsqueeze(-1)                               # :234,238
    grad = torch.stack([s[..., C:2 * C] * m, s[..., 2 * C:3 * C] * m], dim=-1)    # :235-239
    avg = diff.squeeze(-1).abs().mean(dim=1, keepdim=True)                        # :243
    if lambda_override is not None:
        lam = lambda_override.reshape(nb, 1, 1)
    else:
        lam = torch.pow(torch.linalg.norm(avg, dim=-1, keepdim=True), 2.0 + lambda_mlp(avg, mlp_params))   # :244-249
        if bundle and l2_regularizer_base is not None:
            lam = l2_regularizer_base * lam                                       # :252-253
    iZ = 1.0 / Z
    zeros = torch.zeros_like(x)
    Jx = -fx.unsqueeze(-1) * torch.stack([x * y, -1 - x * x, y, -iZ, zeros, x * iZ], dim=2)      # :49-61
    Jy = -fy.unsqueeze(-1) * torch.stack([1 + y * y, -x * y, -x, zeros, -iZ, y * iZ], dim=2)
    J = torch.stack([Jx, Jy], dim=2)                                              # [nb,N,2,6]
    if bundle:
        jd = torch.stack([fx * ((Rp[:, 0] - Rp[:, 2] * x) * iZ), fy * ((Rp[:, 1] - Rp[:, 2] * y) * iZ)], dim=2)   # :63-74
        J = torch.cat([J, jd.unsqueeze(-1) * B.unsqueeze(-2)], dim=-1)            # :260-261
    J = torch.where(ok.unsqueeze(-1).unsqueeze(-1), J, torch.zeros_like(J))        # masked / non-finite projections: no 0 * inf (the fused kernels skip them)
    AtA, Atb = ops.equation_construction(J.contiguous(), grad.contiguous(), diff.contiguous(), exact_sym)   # :263 (native fwd + bwd)
    diag = torch.diagonal(AtA, dim1=-2, dim2=-1)
    if bundle:
        dvec = torch.cat([diag[:, :-1] + damping_eps, torch.zeros(nb, 1, device=diag.device, dtype=diag.dtype)], dim=-1)   # :266
    else:
        dvec = diag + damping_eps                                                 # :182
    sol = torch.linalg.solve(AtA + torch.diag_embed(dvec * lam.reshape(nb, 1)), Atb)               # :267 / :183
    wv, tv = sol[:, 0:3, 0], sol[:, 3:6, :]
    dr = _rodrigues(wv)
    Rn = dr @ R                                                                   # :274
    Tn = _vmatrix(wv) @ tv + dr @ T                                               # :275
    Wn = (W + sol[:, 6:, :]) if bundle else None                                  # :276
    return Rn, Tn, Wn


# ------------------------------------------------------------------------------------------ fused path
class _LMBuildFn(torch.autograd.Function):
    """(H, g, rbar_sum) = banet_lm_build(...); backward = banet_lm_build_bwd.  conv2 is the [F2|gx|gy] tensor."""

    @staticmethod
    def forward(ctx, conv1, conv2, D, B, R, T, W, intr, p, precision, exact_sym, grid):
        lv = ops.Level(conv1, conv2, intr, p, D, B, grid=grid)
        H, g, rbar, nvalid = ops.lm_build(lv, R, T, W, precision)
        ctx.save_for_backward(conv1, conv2, D, B if B is not None else conv1.new_empty(0), R, T, W if W is not None else conv1.new_empty(0), intr, p)
        ctx.has_basis = B is not None
        ctx.exact_sym = bool(exact_sym); ctx.grid = grid
        ctx.mark_non_differentiable(nvalid)
        return H, g, rbar, nvalid

    @staticmethod
    def backward(ctx, dH, dg, drbar, _dnvalid):
        conv1, conv2, D, B, R, T, W, intr, p = ctx.saved_tensors
        if not ctx.has_basis:
            B = None; W = None
        lv = ops.Level(conv1, conv2, intr, p, D, B, grid=ctx.grid)
        nb = conv1.shape[0]
        P = 6 + (0 if B is None else B.shape[2])
        dH = dH.contiguous() if dH is not None else torch.zeros(nb, P, P, device=conv1.device)
        dg = dg if dg is not None else torch.zeros(nb, P, device=conv1.device)
        drbar = drbar if drbar is not None else torch.zeros(nb, conv1.shape[2], device=conv1.device)
        dconv1, dconv2, dD, dB, dR, dT, dW = ops.lm_build_bwd(lv, R, T, W, dH, dg.contiguous(), drbar.contiguous(), ctx.exact_sym)
        return dconv1, dconv2, dD, dB, dR, dT, dW, None, None, None, None, None


class _LMSolveUpdateFn(torch.autograd.Function):
    """(R', T', W') = banet_lm_solve_update(H, g, lambda, R, T, W); backward = banet_lm_solve_update_bwd."""

    @staticmethod
    def forward(ctx, H, g, lam, R, T, W, damping_eps, undamped_last):
        Rn, Tn, Wn, delta, status = ops.lm_solve_update(H, g, lam, R, T, W, damping_eps=damping_eps, undamped_last=undamped_last)
        ctx.save_for_backward(H, g, lam, delta, R, T)
        ctx.eps = float(damping_eps); ctx.undamped_last = bool(undamped_last); ctx.has_w = W is not None
        ctx.mark_non_differentiable(status)
        if W is None:
            return Rn, Tn, status
        return Rn, Tn, Wn, status

    @staticmethod
    def backward(ctx, *grads):
        H, g, lam, delta, R, T = ctx.saved_tensors
        nb, P = g.shape[0], H.shape[1]
        dRn = grads[0] if grads[0] is not None else torch.zeros_like(R)
        dTn = grads[1] if grads[1] is not None else torch.zeros_like(T)
        dWn = None
        if ctx.has_w:
            dWn = grads[2] if grads[2] is not None else torch.zeros(nb, P - 6, 1, device=H.device)
        dH, dg, dlam, dR, dT, dW = ops.lm_solve_update_bwd(H, g, lam, delta, R, T, dRn.contiguous(), dTn.contiguous(),
                                                           None if dWn is None else dWn.contiguous(), ctx.eps, ctx.undamped_last)
        return dH, dg.reshape(g.shape), dlam.reshape(lam.shape), dR, dT, dW, None, None


class _WindowSolveUpdateFn(torch.autograd.Function):
    """(R' [nf,3,3], T' [nf,3,1], W' [K,1]) = banet_lm_window_solve_update(H, g, lambda [1], R, T, W); backward =
    banet_lm_window_solve_update_bwd.  Saves H, g, lambda, the joint solution, R, T: nothing per-pixel."""

    @staticmethod
    def forward(ctx, H, g, lam, R, T, W, damping_eps):
        Rn, Tn, Wn, delta, status = ops.lm_window_solve_update(H, g, lam, R, T, W, damping_eps=damping_eps)
        ctx.save_for_backward(H, g, lam, delta, R, T)
        ctx.eps = float(damping_eps)
        ctx.mark_non_differentiable(status)
        return Rn, Tn, Wn, status

    @staticmethod
    def backward(ctx, dRn, dTn, dWn, _dstatus):
        H, g, lam, delta, R, T = ctx.saved_tensors
        K = H.shape[1] - 6
        dRn = dRn if dRn is not None else torch.zeros_like(R)
        dTn = dTn if dTn is not None else torch.zeros_like(T)
        dWn = dWn if dWn is not None else torch.zeros(K, 1, device=H.device)
        dH, dg, dlam, dR, dT, dW = ops.lm_window_solve_update_bwd(H, g, lam, delta, R, T, dRn.contiguous(), dTn.contiguous(), dWn.contiguous(), ctx.eps)
        return dH, dg.reshape(g.shape), dlam.reshape(lam.shape), dR, dT, dW, None


class _WindowBatchSolveUpdateFn(torch.autograd.Function):
    """(R' [nw*nf,3,3], T' [nw*nf,3,1], W' [nw,K,1]) = banet_lm_window_batch_solve_update(H, g, lambda [nw], R, T, W); backward =
    banet_lm_window_batch_solve_update_bwd.  Saves H, g, lambda, the windows' solutions, R, T: nothing per-pixel."""

    @staticmethod
    def forward(ctx, H, g, lam, R, T, W, damping_eps):
        Rn, Tn, Wn, delta, status = ops.lm_window_batch_solve_update(H, g, lam, R, T, W, damping_eps=damping_eps)
        ctx.save_for_backward(H, g, lam, delta, R, T)
        ctx.eps = float(damping_eps)
        ctx.mark_non_differentiable(status)
        return Rn, Tn, Wn, status

    @staticmethod
    def backward(ctx, dRn, dTn, dWn, _dstatus):
        H, g, lam, delta, R, T = ctx.saved_tensors
        nw, K = lam.numel(), H.shape[1] - 6
        dRn = dRn if dRn is not None else torch.zeros_like(R)
        dTn = dTn if dTn is not None else torch.zeros_like(T)
        dWn = dWn if dWn is not None else torch.zeros(nw, K, 1, device=H.device)
        dH, dg, dlam, dR, dT, dW = ops.lm_window_batch_solve_update_bwd(H, g, lam, delta, R, T, dRn.contiguous(), dTn.contiguous(), dWn.contiguous(),
                                                                        ctx.eps)
        return dH, dg.reshape(g.shape), dlam.reshape(lam.shape), dR, dT, dW, None


class _GradFixedConcatFn(torch.autograd.Function):
    """[F | grad_fixed(F)] (+ the half swap of bundlenet.py:386), differentiable (banet_grad_fixed_concat / _bwd)."""

    @staticmethod
    def forward(ctx, F, swap_halves):
        ctx.swap = bool(swap_halves)
        return ops.grad_fixed_concat(F, swap_halves=ctx.swap)

    @staticmethod
    def backward(ctx, dconv2):
        return ops.grad_fixed_concat_bwd(dconv2.contiguous(), swap_halves=ctx.swap), None


class _ResampleFn(torch.autograd.Function):
    """tf.contrib.resampler.resampler w.r.t. the map (the points are constants on this path)."""

    @staticmethod
    def forward(ctx, data, xy, coord_scale):
        ctx.save_for_backward(xy); ctx.cs = float(coord_scale); ctx.hw = (data.shape[1], data.shape[2])
        return ops.resample(data, xy, coord_scale)

    @staticmethod
    def backward(ctx, dout):
        (xy,) = ctx.saved_tensors
        return ops.resample_bwd(dout.contiguous(), xy, ctx.cs, ctx.hw[0], ctx.hw[1]), None, None


class _DepthComposeFn(torch.autograd.Function):
    """init_depth + basis . W (bundlenet.py:397)."""

    @staticmethod
    def forward(ctx, init_depth, basis, W):
        ctx.save_for_backward(basis, W)
        return ops.depth_compose(init_depth, basis, W)

    @staticmethod
    def backward(ctx, dout):
        basis, W = ctx.saved_tensors
        dbasis, dW = ops.depth_compose_bwd(dout.contiguous(), basis, W)
        return dout, dbasis, dW


def grad_fixed_concat(F: Tensor, swap_halves: bool = False) -> Tensor:
    return _GradFixedConcatFn.apply(F, swap_halves)


def resample(data: Tensor, xy: Tensor, coord_scale: float = 1.0) -> Tensor:
    return _ResampleFn.apply(data, xy.detach(), coord_scale)


def depth_compose(init_depth: Tensor, basis: Tensor, W: Tensor) -> Tensor:
    return _DepthComposeFn.apply(init_depth, basis, W)


def iteration_fused(conv1, conv2, intr, p, D, B, R, T, W, mlp_params, l2_regularizer_base: Optional[float],
                    damping_eps: float = 1e-5, exact_sym: bool = False, lambda_override: Optional[Tensor] = None,
                    precision: int = 0, grid=None, return_status: bool = False):
    """One differentiable LM iteration on the fused kernels.  Same arguments / returns as `iteration`.
    precision: contraction mode of the FORWARD build (the backward is fp32); default FP32_SIMT, the reference's arithmetic type."""
    nb, N, C = conv1.shape
    bundle = B is not None
    H, g, rbar_sum, _nvalid = _LMBuildFn.apply(conv1, conv2, D, B, R, T, W, intr.detach(), p.detach(), precision, exact_sym, grid)
    if lambda_override is not None:
        lam = lambda_override.reshape(nb)
    else:
        avg = (rbar_sum / float(N)).unsqueeze(1)                                  # tf.reduce_mean over N, :243
        lam = torch.pow(torch.linalg.norm(avg, dim=-1, keepdim=True), 2.0 + lambda_mlp(avg, mlp_params)).reshape(nb)   # :244-249
        if bundle and l2_regularizer_base is not None:
            lam = l2_regularizer_base * lam                                       # :252-253
    out = _LMSolveUpdateFn.apply(H, g, lam, R, T, W, damping_eps, bundle)
    if bundle:
        Rn, Tn, Wn, status = out
    else:
        (Rn, Tn, status), Wn = out, None
    if return_status:
        return Rn, Tn, Wn, status
    return Rn, Tn, Wn


def window_iteration_fused(conv1, conv2, intr, p, D, B, R, T, W, mlp_params, l2_regularizer_base: Optional[float],
                           damping_eps: float = 1e-5, exact_sym: bool = False, lambda_override: Optional[Tensor] = None,
                           precision: int = 0, grid=None, return_status: bool = False):
    """One differentiable LM iteration of a keyframe window (the joint solve of ops.lm_window_run) on the fused kernels: nf pairs
    (keyframe -> frame f) share W [K,1]; R [nf,3,3], T [nf,3,1] and conv2 [nf,h,w,3C] are per frame.  The keyframe tensors conv1, p, D, B
    (and intr) may be given once ([1,...]): they are broadcast to the frames and their gradients summed over them.  lambda: from the mean
    |residual| over all points of all frames through the MLP (times l2_regularizer_base), or lambda_override [1].
    Returns (R', T', W' [K,1]) (, status [nf])."""
    nf = R.shape[0]
    K = B.shape[-1]
    frames = lambda t: t.expand(nf, *t.shape[1:]).contiguous() if t.shape[0] == 1 and nf > 1 else t
    conv1, intr, p, D, B = frames(conv1), frames(intr), frames(p), frames(D), frames(B)
    N = conv1.shape[1]
    Wf = W.reshape(1, K, 1).expand(nf, K, 1).contiguous()                       # every pair builds with the shared W; dW sums over them
    H, g, rbar_sum, _nvalid = _LMBuildFn.apply(conv1, conv2, D, B, R, T, Wf, intr.detach(), p.detach(), precision, exact_sym, grid)
    if lambda_override is not None:
        lam = lambda_override.reshape(1)
    else:
        avg = (rbar_sum.sum(0) / float(nf * N)).reshape(1, 1, -1)               # mean |residual| over all nf * N points
        lam = torch.pow(torch.linalg.norm(avg, dim=-1, keepdim=True), 2.0 + lambda_mlp(avg, mlp_params)).reshape(1)
        if l2_regularizer_base is not None:
            lam = l2_regularizer_base * lam
    Rn, Tn, Wn, status = _WindowSolveUpdateFn.apply(H, g, lam, R, T, W.reshape(K, 1), damping_eps)
    if return_status:
        return Rn, Tn, Wn, status
    return Rn, Tn, Wn


def window_batch_iteration_fused(conv1, conv2, intr, p, D, B, R, T, W, mlp_params, l2_regularizer_base: Optional[float],
                                 damping_eps: float = 1e-5, exact_sym: bool = False, lambda_override: Optional[Tensor] = None,
                                 precision: int = 0, grid=None, return_status: bool = False):
    """One differentiable LM iteration of a batch of nw keyframe windows of nf frames (window_iteration_fused per window, one launch each
    for the build, the step and their backwards).  R [nw,nf,3,3], T [nw,nf,3,1], conv2 [nw,nf,h,w,3C] per frame, W [nw,K,1] per window; the
    keyframe tensors conv1, p, D, B (and intr) are [nw,nf,...] or [nw,1,...] (broadcast to the frames, their gradients summed over them).
    lambda per window: from the mean |residual| over its nf * N points through the MLP (times l2_regularizer_base), or lambda_override [nw].
    Returns (R' [nw,nf,3,3], T' [nw,nf,3,1], W' [nw,K,1]) (, status [nw,nf])."""
    nw, nf = R.shape[0], R.shape[1]
    K = B.shape[-1]
    nb = nw * nf
    pairs = lambda t: (t.expand(nw, nf, *t.shape[2:]) if t.shape[1] == 1 and nf > 1 else t).reshape(nb, *t.shape[2:]).contiguous()
    conv1, conv2, intr, p, D, B = pairs(conv1), pairs(conv2), pairs(intr), pairs(p), pairs(D), pairs(B)
    N, C = conv1.shape[1], conv1.shape[2]
    Wf = W.reshape(nw, 1, K, 1).expand(nw, nf, K, 1).reshape(nb, K, 1).contiguous()   # every pair builds with its window's W
    Rf, Tf = R.reshape(nb, 3, 3), T.reshape(nb, 3, 1)
    H, g, rbar_sum, _nvalid = _LMBuildFn.apply(conv1, conv2, D, B, Rf, Tf, Wf, intr.detach(), p.detach(), precision, exact_sym, grid)
    if lambda_override is not None:
        lam = lambda_override.reshape(nw)
    else:
        avg = (rbar_sum.reshape(nw, nf, C).sum(1) / float(nf * N)).unsqueeze(1)         # mean |residual| over each window's nf * N points
        lam = torch.pow(torch.linalg.norm(avg, dim=-1, keepdim=True), 2.0 + lambda_mlp(avg, mlp_params)).reshape(nw)
        if l2_regularizer_base is not None:
            lam = l2_regularizer_base * lam
    Rn, Tn, Wn, status = _WindowBatchSolveUpdateFn.apply(H, g, lam, Rf, Tf, W.reshape(nw, K, 1), damping_eps)
    Rn, Tn, status = Rn.reshape(nw, nf, 3, 3), Tn.reshape(nw, nf, 3, 1), status.reshape(nw, nf)
    if return_status:
        return Rn, Tn, Wn, status
    return Rn, Tn, Wn
