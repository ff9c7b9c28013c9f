"""Host-side mirror of the reference's BA-layer interface (reference bundlenet.py:86-399), backed by the
sm_90a kernels.  Same method names, argument order, tensor layouts and return values as the reference's
`BundleNet`; arithmetic happens in libbanet.so (no torch maths on the hot path, no CPU fallback).

Differences a reference user should know (all documented in DESIGN.md):
  * fx,fy,ox,oy may be passed as the reference does ([nb,N], constant along N) — column 0 is used;
  * lambda-MLP weights are ordinary parameters named like the TF variables
    (`lambda_{level}_{i}_filters` [cin,cout], `lambda_{level}_{i}_biases`, reference bundlenet.py:105-106);
  * `tf.matrix_solve` (LU) is replaced by a Cholesky factorisation; non-finite projections are masked
    instead of poisoning the sums with NaN; VMatrix is evaluated per pair unless
    `vmatrix_batch_scramble=True` (reference bundlenet.py:45 interleaves pairs for nb > 1).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import ops
from . import autograd as _ag
from ._lib import PREC_AUTO

Tensor = torch.Tensor


def _intr_from_tiled(fx, fy, ox, oy) -> Tensor:
    """[nb,N] (reference) / [nb,1] / [nb] -> [nb,4]."""
    cols = []
    for t in (fx, fy, ox, oy):
        t = t.reshape(t.shape[0], -1)[:, 0]
        cols.append(t)
    return torch.stack(cols, dim=1).to(torch.float32).contiguous()


@dataclass
class ResizeGeometry:
    """Crop / intrinsics fix-ups hard-coded in the reference (bundlenet.py:286-287, 298-302, 397)."""
    sx: float = 320.0; cx: float = 4.0; dx: float = 312.0
    sy: float = 256.0; cy: float = 4.0; dy: float = 232.0
    fx_num: float = 40.0; fx_den: float = 39.0; ox_sub: float = 160.0 / 39.0
    fy_num: float = 32.0; fy_den: float = 29.0; oy_sub: float = 128.0 / 29.0
    out_hw: Tuple[int, int] = (256 // 2, 320 // 2)


class BundleNet(torch.nn.Module):
    """Drop-in for reference `BundleNet` (bundlenet.py:86).  `channels` = feature channels C of the pyramid."""

    def __init__(self, channels: int, levels: Sequence[str] = ("0", "1", "2", "3"), is_training: bool = True,
                 reuse_variables=None, vmatrix_batch_scramble: bool = False, precision: int = PREC_AUTO, seed: int = 7,
                 exact_sym_grad: bool = False, training_path: str = "fused", strict_status: bool = False):
        super().__init__()
        self.is_training = is_training
        self.reuse_variables = reuse_variables
        self.channels = channels
        self.vmatrix_batch_scramble = vmatrix_batch_scramble
        self.precision = precision
        self.exact_sym_grad = exact_sym_grad      # False: the reference's op gradient 2*A*Ghat (utils.cu:648); True: A(Ghat+Ghat^T)
        if training_path not in ("fused", "reference_split"):
            raise ValueError("training_path must be 'fused' or 'reference_split'")
        self.training_path = training_path        # fused: banet_lm_*_bwd kernels; reference_split: torch graph + native equation_construction
        self.strict_status = strict_status
        self.last_status: Optional[Tensor] = None
        self.train(bool(is_training))
        self.geo = ResizeGeometry()
        g = torch.Generator().manual_seed(seed)
        dims = [channels, 2 * channels, 4 * channels, 2 * channels, channels, 1]
        for lv in levels:
            for i in range(5):
                # he_normal filters, zero biases (reference bundlenet.py:105-106)
                w = torch.randn(dims[i], dims[i + 1], generator=g) * math.sqrt(2.0 / dims[i])
                self.register_parameter(f"lambda_{lv}_{i + 1}_filters", torch.nn.Parameter(w))
                self.register_parameter(f"lambda_{lv}_{i + 1}_biases", torch.nn.Parameter(torch.zeros(dims[i + 1])))

    # ---- helpers -------------------------------------------------------------------------------
    def mlp_params(self, level: str) -> List[Tuple[Tensor, Tensor]]:
        return [(getattr(self, f"lambda_{level}_{i}_filters"), getattr(self, f"lambda_{level}_{i}_biases")) for i in range(1, 6)]

    def mlp_packed(self, level: str) -> Tensor:
        return ops.pack_mlp([(w.detach(), b.detach()) for w, b in self.mlp_params(level)])

    def grad_fixed(self, input: Tensor, name=None) -> Tensor:
        """reference bundlenet.py:92-100: [nb,h,w,C] -> [nb,h,w,2C] = [gradx|grady]."""
        return ops.grad_fixed_concat(input)[..., input.shape[-1]:].contiguous()

    def computeCoordinates(self, points2d: Tensor, fx, fy, ox, oy) -> Tensor:
        """reference bundlenet.py:112-120 -> p [nb,3,N] (L2-normalised)."""
        return ops.compute_coordinates(points2d, _intr_from_tiled(fx, fy, ox, oy), normalize=True)

    # ---- one LM iteration ----------------------------------------------------------------------
    def _wants_grad(self, *tensors) -> bool:
        """Gradients are recorded when autograd is on and a DATA input requires grad, or the module is in training mode (then the
        lambda-MLP parameters do).  In eval mode with plain inputs the no-grad kernels run (same forward, nothing saved)."""
        if not torch.is_grad_enabled():
            return False
        if any(isinstance(t, torch.Tensor) and t.requires_grad for t in tensors):
            return True
        return self.training and any(p.requires_grad for p in self.parameters())

    def _check_status(self, status: Tensor) -> None:
        """Keeps the per-pair solver status of the last call (0 ok, 1 non-SPD matrix: step skipped, 2 non-finite input) in
        `self.last_status` (device tensor, no host sync); `strict_status=True` turns a non-zero status into an exception."""
        self.last_status = status
        if self.strict_status and int(status.abs().max()) != 0:
            raise RuntimeError(f"LM solve skipped a step for pairs {torch.nonzero(status).flatten().tolist()} (status {status.tolist()})")

    def _iterate(self, conv1, conv2, intr, p, D, B, R, T, W, base, level, grid=None):
        """One iteration, differentiable or not; returns (R', T', W', aux or None)."""
        bundle = B is not None
        if self._wants_grad(conv1, conv2, D, B, R, T, W):
            if self.vmatrix_batch_scramble:
                raise RuntimeError("vmatrix_batch_scramble=True (the reference's batch-interleaved VMatrix, bundlenet.py:45) is not differentiable here")
            if self.training_path == "reference_split":
                Rn, Tn, Wn = _ag.iteration(conv1, conv2, intr, p, D, B, R, T, W, self.mlp_params(str(level)), base if bundle else None,
                                           exact_sym=self.exact_sym_grad)
                return Rn, Tn, Wn, None
            Rn, Tn, Wn, status = _ag.iteration_fused(conv1, conv2, intr, p, D, B, R, T, W, self.mlp_params(str(level)), base if bundle else None,
                                                     exact_sym=self.exact_sym_grad, precision=self.precision, grid=grid, return_status=True)
            self._check_status(status)
            return Rn, Tn, Wn, None
        lv = ops.Level(conv1, conv2, intr, p, D, B, grid=grid)
        H, g, rbar, nvalid = ops.lm_build(lv, R, T, W, self.precision)
        lam = ops.lm_lambda(rbar, conv1.shape[1], self.mlp_packed(str(level)), float(base) if bundle else 1.0)
        Rn, Tn, Wn, delta, status = ops.lm_solve_update(H, g, lam, R, T, W, undamped_last=bundle, vmatrix_batch_scramble=self.vmatrix_batch_scramble)
        self._check_status(status)
        return Rn, Tn, Wn, dict(AtA=H, Atb=g, lam=lam, rbar_sum=rbar, nvalid=nvalid, solution=delta, status=status)

    def CameraIteration(self, conv1, conv2, fx, fy, ox, oy, p, D, R, T, l2_regularizer_base=None, level=None, return_aux: bool = False):
        """reference bundlenet.py:122-191 -> (updatedR, updatedT).  l2_regularizer_base accepted, unused (as there).
        Differentiable (fused backward kernels) whenever gradients are being recorded; `return_aux` needs the no-grad path."""
        if return_aux:
            with torch.no_grad():
                Rn, Tn, _, aux = self._iterate(conv1, conv2, _intr_from_tiled(fx, fy, ox, oy), p, D, None, R, T, None, 1.0, level)
            return Rn, Tn, aux
        Rn, Tn, _, _ = self._iterate(conv1, conv2, _intr_from_tiled(fx, fy, ox, oy), p, D, None, R, T, None, 1.0, level)
        return Rn, Tn

    def BundleIteration(self, conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, l2_regularizer_base=None, level=None, return_aux: bool = False):
        """reference bundlenet.py:193-278 -> (updatedR, updatedT, updatedW)."""
        base = 1.0 if l2_regularizer_base is None else float(l2_regularizer_base)      # :252-253
        if return_aux:
            with torch.no_grad():
                Rn, Tn, Wn, aux = self._iterate(conv1, conv2, _intr_from_tiled(fx, fy, ox, oy), p, D, B, R, T, W, base, level)
            return Rn, Tn, Wn, aux
        Rn, Tn, Wn, _ = self._iterate(conv1, conv2, _intr_from_tiled(fx, fy, ox, oy), p, D, B, R, T, W, base, level)
        return Rn, Tn, Wn

    def WindowIteration(self, conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, l2_regularizer_base=None, level=None):
        """One joint LM iteration of a keyframe window (an extension; the reference's layer is 2-view): the nf pairs (keyframe -> frame f)
        share the keyframe depth D + B.W.  Arguments as BundleIteration with R [nf,3,3], T [nf,3,1], conv2 [nf,h,w,3C] per frame and
        W [K,1] shared; the keyframe tensors conv1, p, D, B may be given once ([1,...]) or per frame.  -> (updatedR, updatedT, updatedW [K,1]).
        Differentiable (banet_lm_window_solve_update_bwd) whenever gradients are being recorded; there is no reference_split twin.
        A batch of nw windows: R [nw,nf,3,3], T [nw,nf,3,1], conv2 [nw,nf,h,w,3C], W [nw,K,1], keyframe tensors and fx, fy, ox, oy
        [nw,1,...] or [nw,nf,...] -> ([nw,nf,3,3], [nw,nf,3,1], [nw,K,1]), last_status [nw,nf] (banet_lm_window_batch_*)."""
        base = 1.0 if l2_regularizer_base is None else float(l2_regularizer_base)
        if self.vmatrix_batch_scramble:
            raise RuntimeError("vmatrix_batch_scramble=True is a 2-view quirk (bundlenet.py:45); the window solve has per-frame VMatrix only")
        if R.dim() == 4:
            return self._window_batch_iteration(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, base, level)
        nf = R.shape[0]
        intr = _intr_from_tiled(fx, fy, ox, oy)
        if self._wants_grad(conv1, conv2, D, B, R, T, W):
            if self.training_path == "reference_split":
                raise RuntimeError("training_path='reference_split' has no torch-graph twin of the window solve; use training_path='fused'")
            Rn, Tn, Wn, status = _ag.window_iteration_fused(conv1, conv2, intr, p, D, B, R, T, W, self.mlp_params(str(level)), base,
                                                            exact_sym=self.exact_sym_grad, precision=self.precision, return_status=True)
            self._check_status(status)
            return Rn, Tn, Wn
        frames = lambda t: t.expand(nf, *t.shape[1:]) if t.shape[0] == 1 else t
        lv = ops.Level(frames(conv1), conv2, frames(intr), frames(p), frames(D), frames(B))
        Rn, Tn, Wn, status = ops.lm_window_run([lv], 1, R, T, W, mlp_packed=[self.mlp_packed(str(level))], l2_regularizer_base=base,
                                               precision=self.precision)
        self._check_status(status)
        return Rn, Tn, Wn

    def _window_batch_iteration(self, conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, base, level):
        """WindowIteration on a batch of nw windows (R [nw,nf,3,3]): the fused path when gradients are recorded, else one iteration of
        ops.lm_window_batch_run."""
        nw, nf = R.shape[0], R.shape[1]
        intr = torch.stack([t.reshape(t.shape[0], t.shape[1], -1)[..., 0] for t in (fx, fy, ox, oy)], dim=-1).to(torch.float32)   # [nw,1|nf,4]
        if self._wants_grad(conv1, conv2, D, B, R, T, W):
            if self.training_path == "reference_split":
                raise RuntimeError("training_path='reference_split' has no torch-graph twin of the window solve; use training_path='fused'")
            Rn, Tn, Wn, status = _ag.window_batch_iteration_fused(conv1, conv2, intr, p, D, B, R, T, W, self.mlp_params(str(level)), base,
                                                                  exact_sym=self.exact_sym_grad, precision=self.precision, return_status=True)
            self._check_status(status)
            return Rn, Tn, Wn
        pairs = lambda t: (t.expand(nw, nf, *t.shape[2:]) if t.shape[1] == 1 else t).reshape(nw * nf, *t.shape[2:])
        lv = ops.Level(pairs(conv1), pairs(conv2), pairs(intr), pairs(p), pairs(D), pairs(B))
        Rn, Tn, Wn, status = ops.lm_window_batch_run([lv], nw, 1, R.reshape(nw * nf, 3, 3), T.reshape(nw * nf, 3, 1), W,
                                                     mlp_packed=[self.mlp_packed(str(level))], l2_regularizer_base=base, precision=self.precision)
        self._check_status(status.reshape(nw, nf))
        return Rn.reshape(nw, nf, 3, 3), Tn.reshape(nw, nf, 3, 1), Wn

    # ---- level schedulers ----------------------------------------------------------------------
    def _prepare(self, intrisic: Tensor, points: Tensor):
        geo = self.geo
        x = geo.sx * (points[..., 0:1] - geo.cx) / geo.dx
        y = geo.sy * (points[..., 1:2] - geo.cy) / geo.dy
        _points = torch.cat([x, y], dim=-1).contiguous()
        k = intrisic.reshape(intrisic.shape[0], 4)
        intr = torch.stack([geo.fx_num * k[:, 0] / geo.fx_den, geo.fy_num * k[:, 1] / geo.fy_den,
                            geo.fx_num * k[:, 2] / geo.fx_den - geo.ox_sub,
                            geo.fy_num * k[:, 3] / geo.fy_den - geo.oy_sub], dim=1).contiguous()
        return _points.detach(), intr.detach()

    def CameraResize(self, intrisic, layers, points, _depths, reuse_variables=False):
        """reference bundlenet.py:280-329 -> (rotations, translations), levels 0..3 x 1 iteration.  Differentiable w.r.t. the feature
        pyramid and the lambda-MLP parameters when gradients are being recorded (the depth is stop_gradient'ed, :288)."""
        nb = layers[-1].shape[0]
        _points, intr = self._prepare(intrisic, points)
        grad = self._wants_grad(*layers)
        resample, gfc = (_ag.resample, _ag.grad_fixed_concat) if grad else (ops.resample, ops.grad_fixed_concat)
        d = ops.resample(_depths.detach(), _points, 0.5)                       # :289-290
        p = ops.compute_coordinates(_points, intr, True)
        R = torch.eye(3, device=points.device).repeat(nb, 1, 1)
        T = torch.zeros(nb, 3, 1, device=points.device)
        rotations, translations = [], []
        for level in range(0, 4):
            scale = 2 ** (3 - level)
            layer1 = resample(layers[level], _points, 1.0 / scale)             # :320
            layer2 = gfc(layers[level], swap_halves=True)                      # :321-324
            R, T, _, _ = self._iterate(layer1, layer2, intr / scale, p, d, None, R, T, None, 1.0, level)
            rotations.append(R); translations.append(T)
        return rotations, translations

    def BundleResize(self, intrisic, layers, points, basis, init_depth, init_rotation=None, init_translation=None,
                     reuse_variables=False):
        """reference bundlenet.py:332-399 -> (output_rotations, output_translations, output_depths), levels 2,3.  Differentiable w.r.t.
        the feature pyramid, the basis, the initial pose and the lambda-MLP parameters when gradients are being recorded
        (init_depth enters the LM only through stop_gradient, :341, and the output depth directly, :397)."""
        nb = layers[-1].shape[0]
        K = basis.shape[-1]
        _points, intr = self._prepare(intrisic, points)
        grad = self._wants_grad(*layers, basis, init_depth, init_rotation, init_translation)
        resample, gfc, compose = (_ag.resample, _ag.grad_fixed_concat, _ag.depth_compose) if grad else (ops.resample, ops.grad_fixed_concat, ops.depth_compose)
        d = ops.resample(init_depth.detach(), _points, 0.5)                    # :341-343
        b = resample(basis, _points, 0.5)                                      # :344
        p = ops.compute_coordinates(_points, intr, True)                       # :358
        dev = points.device
        R = torch.eye(3, device=dev).repeat(nb, 1, 1) if init_rotation is None else init_rotation
        T = torch.zeros(nb, 3, 1, device=dev) if init_translation is None else init_translation
        W = torch.zeros(nb, K, 1, device=dev)
        oh, ow = self.geo.out_hw
        Rs, Ts, Ds = [], [], []
        for level in range(2, 4):                                              # :376
            scale = 2 ** (3 - level)
            layer1 = resample(layers[level], _points, 1.0 / scale)             # :385
            layer2 = gfc(layers[level], swap_halves=True)                      # :386-389
            R, T, W, _ = self._iterate(layer1, layer2, intr / scale, p, d, b, R, T, W, 1000.0, level)   # :393
            Rs.append(R); Ts.append(T)
            depth = compose(init_depth.reshape(nb, -1), basis.reshape(nb, -1, K), W)   # :397
            Ds.append(depth.reshape(nb, oh, ow, 1))
        return Rs, Ts, Ds

    # ---- training losses (reference bundlenet.py:401-463): stock torch, like the CNN around the layer ---------------------------------
    def lossR(self, predQ: Tensor, gtQ: Tensor) -> Tensor:
        """bundlenet.py:401-404: tf.losses.cosine_distance of unit quaternions = mean(1 - <pred, gt>)."""
        return (1.0 - (predQ * gtQ).sum(dim=1, keepdim=True)).mean()

    def lossT(self, predT: Tensor, gtT: Tensor) -> Tensor:
        """bundlenet.py:411-413 (the second definition, which overrides the angular one of :406-409): mean |predT - gtT|."""
        return (predT - gtT).abs().mean()

    def lossF(self, intrisic: Tensor, depth: Tensor, mask: Tensor, predR: Tensor, predT: Tensor, gtR: Tensor, gtT: Tensor) -> Tensor:
        """bundlenet.py:415-463: masked mean |flow(pred) - flow(gt)| over the dense pixel grid in units of the image width, times total / valid."""
        geo = self.geo
        nb, h, w = depth.shape[0], depth.shape[1], depth.shape[2]
        npix = h * w
        k = intrisic.reshape(nb, 4)
        fx = (geo.fx_num * k[:, 0:1] / geo.fx_den); fy = (geo.fy_num * k[:, 1:2] / geo.fy_den)
        ox = geo.fx_num * k[:, 2:3] / geo.fx_den - geo.ox_sub; oy = geo.fy_num * k[:, 3:4] / geo.fy_den - geo.oy_sub
        yy, xx = torch.meshgrid(torch.arange(h, device=depth.device, dtype=depth.dtype), torch.arange(w, device=depth.device, dtype=depth.dtype), indexing="ij")
        ray = torch.stack([(xx.reshape(1, -1) - ox) / fx, (yy.reshape(1, -1) - oy) / fy, torch.ones(nb, npix, device=depth.device, dtype=depth.dtype)], dim=1)
        p = ray * torch.rsqrt(torch.clamp((ray * ray).sum(dim=1, keepdim=True), min=1e-12))
        m = mask.reshape(nb, npix)

        def flow(Rm, Tm):
            X = (Rm @ p) * depth.reshape(nb, 1, npix) + Tm.reshape(nb, 3, 1)
            return fx * (X[:, 0] / X[:, 2]) + ox, fy * (X[:, 1] / X[:, 2]) + oy

        fxp, fyp = flow(predR, predT); fxg, fyg = flow(gtR, gtT)
        return (float(npix * nb) / m.sum()) * (((fxp - fxg).abs() * m).mean() / w + ((fyp - fyg).abs() * m).mean() / w)


def rotation2quaternion(R: Tensor, name=None) -> Tensor:
    """reference bundlenet.py:6-15: [nb,3,3] -> unit quaternion [nb,4] (w first)."""
    diag = 1.0 + R[:, 0, 0] + R[:, 1, 1] + R[:, 2, 2]
    q0 = torch.sqrt(diag) / 2.0
    q = torch.stack([q0, (R[:, 2, 1] - R[:, 1, 2]) / (4.0 * q0), (R[:, 0, 2] - R[:, 2, 0]) / (4.0 * q0), (R[:, 1, 0] - R[:, 0, 1]) / (4.0 * q0)], dim=1)
    return q * torch.rsqrt(torch.clamp((q * q).sum(dim=1, keepdim=True), min=1e-12))
