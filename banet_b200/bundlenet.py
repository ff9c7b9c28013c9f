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
from typing import Dict, List, Mapping, Optional, Sequence, Tuple, Union

import torch

from . import ops
from . import autograd as _ag
from . import _lib
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

    def _iterate(self, conv1, conv2, intr, p, D, B, R, T, W, base, level, grid=None, weight=None, robust=None, robust_scale=0.0):
        """One iteration, differentiable or not; returns (R', T', W', aux or None).  weight [nb,N,1]: per-point weight of H and g;
        robust, robust_scale: the robust loss of the feature-metric error (ops.Level)."""
        bundle = B is not None
        ops.robust_kind(robust, robust_scale)                                  # argument errors before any kernel runs
        if self._wants_grad(conv1, conv2, D, B, R, T, W, weight):
            if self.vmatrix_batch_scramble:
                raise RuntimeError("vmatrix_batch_scramble=True (the reference's batch-interleaved VMatrix, bundlenet.py:45) is not differentiable here")
            if self.training_path == "reference_split":
                if weight is not None:
                    raise RuntimeError("training_path='reference_split' has no point weights; weighted iterations train on the fused path")
                if robust is not None:
                    raise RuntimeError("training_path='reference_split' has no robust loss; robust iterations train on the fused path")
                if conv1.dtype != torch.float32 or conv2.dtype != torch.float32:
                    raise RuntimeError("training_path='reference_split' takes float32 features; bfloat16 features train on the fused path")
                if bundle and B.dtype != torch.float32:
                    raise RuntimeError("training_path='reference_split' takes a float32 basis; a bfloat16 basis trains on the fused path")
                Rn, Tn, Wn = _ag.iteration(conv1, conv2, intr, p, D, B, R, T, W, self.mlp_params(str(level)), base if bundle else None,
                                           exact_sym=self.exact_sym_grad)
                return Rn, Tn, Wn, None
            Rn, Tn, Wn, status = _ag.iteration_fused(conv1, conv2, intr, p, D, B, R, T, W, self.mlp_params(str(level)), base if bundle else None,
                                                     exact_sym=self.exact_sym_grad, precision=self.precision, grid=grid, return_status=True,
                                                     weight=weight, robust=robust, robust_scale=robust_scale)
            self._check_status(status)
            return Rn, Tn, Wn, None
        lv = ops.Level(conv1, conv2, intr, p, D, B, grid=grid, weight=weight, robust=robust, robust_scale=robust_scale)
        H, g, rbar, nvalid = ops.lm_build(lv, R, T, W, self.precision)
        lam = ops.lm_lambda(rbar, conv1.shape[1], self.mlp_packed(str(level)), float(base) if bundle else 1.0)
        Rn, Tn, Wn, delta, status = ops.lm_solve_update(H, g, lam, R, T, W, undamped_last=bundle, vmatrix_batch_scramble=self.vmatrix_batch_scramble)
        self._check_status(status)
        return Rn, Tn, Wn, dict(AtA=H, Atb=g, lam=lam, rbar_sum=rbar, nvalid=nvalid, solution=delta, status=status)

    def CameraIteration(self, conv1, conv2, fx, fy, ox, oy, p, D, R, T, l2_regularizer_base=None, level=None, return_aux: bool = False, *,
                        weight: Optional[Tensor] = None, robust: Optional[str] = None, robust_scale: float = 0.0):
        """reference bundlenet.py:122-191 -> (updatedR, updatedT).  l2_regularizer_base accepted, unused (as there).
        Differentiable (fused backward kernels) whenever gradients are being recorded; `return_aux` needs the no-grad path.
        weight [nb,N,1] float32 (an extension): per-point confidence of the normal equations, H = sum_n w_n H_n, g = sum_n w_n g_n; the
        damping lambda does not see it.  Differentiable on the fused training path.
        robust "huber" / "cauchy" (an extension) with robust_scale delta > 0 in feature units: a robust loss of the feature-metric error,
        one IRLS step per iteration (each point's weight times rho'(|d_n|^2) at the current iterate; lambda does not see it).
        Differentiable on the fused training path, through the residual the weight depends on."""
        kw = dict(weight=weight, robust=robust, robust_scale=robust_scale)
        if return_aux:
            with torch.no_grad():
                Rn, Tn, _, aux = self._iterate(conv1, conv2, _intr_from_tiled(fx, fy, ox, oy), p, D, None, R, T, None, 1.0, level, **kw)
            return Rn, Tn, aux
        Rn, Tn, _, _ = self._iterate(conv1, conv2, _intr_from_tiled(fx, fy, ox, oy), p, D, None, R, T, None, 1.0, level, **kw)
        return Rn, Tn

    def BundleIteration(self, conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, l2_regularizer_base=None, level=None, return_aux: bool = False, *,
                        weight: Optional[Tensor] = None, robust: Optional[str] = None, robust_scale: float = 0.0):
        """reference bundlenet.py:193-278 -> (updatedR, updatedT, updatedW).  weight [nb,N,1], robust, robust_scale: as in CameraIteration."""
        base = 1.0 if l2_regularizer_base is None else float(l2_regularizer_base)      # :252-253
        kw = dict(weight=weight, robust=robust, robust_scale=robust_scale)
        if return_aux:
            with torch.no_grad():
                Rn, Tn, Wn, aux = self._iterate(conv1, conv2, _intr_from_tiled(fx, fy, ox, oy), p, D, B, R, T, W, base, level, **kw)
            return Rn, Tn, Wn, aux
        Rn, Tn, Wn, _ = self._iterate(conv1, conv2, _intr_from_tiled(fx, fy, ox, oy), p, D, B, R, T, W, base, level, **kw)
        return Rn, Tn, Wn

    def FeatureMetricCost(self, conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, weight: Optional[Tensor] = None, *,
                          robust: Optional[str] = None, robust_scale: float = 0.0) -> Tensor:
        """The energy BundleIteration takes one step on, at (R, T, W) (an extension): [nb] = sum_n c_n rho(|d_n|^2) over the in-bounds
        points, d_n the point's feature-metric residual, c_n its weight [nb,N,1] (ones when None) and rho the robust loss (rho(s) = s
        without one).  Arguments and layouts of BundleIteration (B = None, W = None for pose-only levels; conv2 [F2|gx|gy] or F2 only).
        Differentiable in conv1, conv2, D, B, R, T, W and weight whenever gradients are being recorded (autograd.feature_metric_cost),
        e.g. as a training loss at the solution; otherwise one no-grad kernel (ops.lm_cost)."""
        ops.robust_kind(robust, robust_scale)                                  # argument errors before any kernel runs
        intr = _intr_from_tiled(fx, fy, ox, oy)
        if torch.is_grad_enabled() and any(isinstance(t, Tensor) and t.requires_grad for t in (conv1, conv2, D, B, R, T, W, weight)):
            return _ag.feature_metric_cost(conv1, conv2, D, B, R, T, W, intr, p, weight=weight, robust=robust, robust_scale=robust_scale)
        lv = ops.Level(conv1, conv2, intr, p, D, B, weight=weight, robust=robust, robust_scale=robust_scale)
        return ops.lm_cost(lv, R, T, W)[0]

    def WindowFeatureMetricCost(self, conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, *, weight: Optional[Tensor] = None) -> Tensor:
        """The energy the keyframe form of WindowIteration takes one step on, at (R, T, W) (an extension): [nw,nf], entry (w, f) = sum_n
        c_n |d_n|^2 over the keyframe points of window w in bounds in frame f, d_n the point's feature-metric residual and c_n its weight
        (ones when None).  Arguments as WindowIteration's keyframe form: conv1 [nw,N,C], p [nw,3,N], D [nw,N,1], B [nw,N,K] once per window,
        conv2 [nw,nf,h,w,3C] or F2 only [nw,nf,h,w,C], fx, fy, ox, oy [nw,1|nf,...], R [nw,nf,3,3], T [nw,nf,3,1], W [nw,K,1], weight
        [nw,nf|1,N,1]; float32 only.  Differentiable in conv1, conv2, D, B, R, T, W and weight whenever gradients are being recorded
        (autograd.window_feature_metric_cost), e.g. as a training loss without ground-truth poses; otherwise one no-grad kernel
        (ops.lm_keyframe_cost).  Nothing of the keyframe is copied per frame."""
        intr = torch.stack([t.reshape(t.shape[0], t.shape[1], -1)[..., 0] for t in (fx, fy, ox, oy)], dim=-1).to(torch.float32)   # [nw,1|nf,4]
        return self._window_cost(conv1, conv2, intr, p, D, B, R, T, W, weight)

    def _window_cost(self, conv1, conv2, intr, p, D, B, R, T, W, weight=None) -> Tensor:
        """WindowFeatureMetricCost with intr [nw,1|nf,4]; its arguments are checked against each other before any kernel runs."""
        def fail(name, t, want):
            got = tuple(t.shape) if isinstance(t, torch.Tensor) else type(t).__name__
            raise _lib.BanetError(f"WindowFeatureMetricCost: {name} must be {want}; got {got}")

        for name, t in (("conv1", conv1), ("conv2", conv2), ("D", D), ("B", B), ("R", R), ("T", T), ("W", W)):
            if not isinstance(t, torch.Tensor) or t.dtype != torch.float32:
                raise _lib.BanetError(f"WindowFeatureMetricCost: {name} must be a float32 tensor (the keyframe layout is fp32 only); got "
                                      f"{getattr(t, 'dtype', type(t).__name__)}")
        if R.dim() != 4 or tuple(R.shape[2:]) != (3, 3):
            fail("R", R, "[nw,nf,3,3]")
        nw, nf = R.shape[0], R.shape[1]
        if conv1.dim() != 3 or conv1.shape[0] != nw:
            fail("conv1", conv1, f"[nw={nw},N,C]")
        N, C = conv1.shape[1], conv1.shape[2]
        if B.dim() != 3 or tuple(B.shape[:2]) != (nw, N):
            fail("B", B, f"[nw={nw},N={N},K]")
        K = B.shape[2]
        for name, t, want in (("p", p, (nw, 3, N)), ("D", D, (nw, N, 1)), ("T", T, (nw, nf, 3, 1)), ("W", W, (nw, K, 1))):
            if tuple(t.shape) != want:
                fail(name, t, f"[{','.join(map(str, want))}]")
        if conv2.dim() != 5 or tuple(conv2.shape[:2]) != (nw, nf) or conv2.shape[4] not in (C, 3 * C):
            fail("conv2", conv2, f"[nw={nw},nf={nf},h,w,3C|C] with C={C}")
        if intr.dim() != 3 or intr.shape[0] != nw or intr.shape[1] not in (1, nf):
            fail("fx, fy, ox, oy", intr, f"[nw={nw},1|nf={nf},...]")
        nb = nw * nf
        wf = None if weight is None else _ag.window_weights(weight, nw, nf, N)
        intr = intr.expand(nw, nf, 4).reshape(nb, 4).contiguous()
        conv2 = conv2.reshape(nb, *conv2.shape[2:])
        Rf, Tf = R.reshape(nb, 3, 3), T.reshape(nb, 3, 1)
        if torch.is_grad_enabled() and any(isinstance(t, Tensor) and t.requires_grad for t in (conv1, conv2, D, B, R, T, W, weight)):
            return _ag.window_feature_metric_cost(conv1, conv2, D, B, Rf, Tf, W, intr, p, weight=wf).reshape(nw, nf)
        return ops.lm_keyframe_cost(ops.KeyframeLevel(conv1, conv2, intr, p, D, B, weight=wf), Rf, Tf, W)[0].reshape(nw, nf)

    def WindowIteration(self, conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, l2_regularizer_base=None, level=None, *,
                        weight: Optional[Tensor] = None, robust: Optional[str] = None, robust_scale: float = 0.0):
        """One joint LM iteration of a keyframe window (an extension; the reference's layer is 2-view): the nf pairs (keyframe -> frame f)
        share the keyframe depth D + B.W.  Arguments as BundleIteration with R [nf,3,3], T [nf,3,1], conv2 [nf,h,w,3C] (or F2 only, [nf,h,w,C]) per frame and
        W [K,1] shared; the keyframe tensors conv1, p, D, B may be given once ([1,...]) or per frame.  -> (updatedR, updatedT, updatedW [K,1]).
        Differentiable (banet_lm_window_solve_update_bwd) whenever gradients are being recorded; there is no reference_split twin.
        A batch of nw windows: R [nw,nf,3,3], T [nw,nf,3,1], conv2 [nw,nf,h,w,3C] (or [nw,nf,h,w,C]), W [nw,K,1], keyframe tensors and fx, fy, ox, oy
        [nw,1,...] or [nw,nf,...] -> ([nw,nf,3,3], [nw,nf,3,1], [nw,K,1]), last_status [nw,nf] (banet_lm_window_batch_*).
        weight (an extension) float32: a per-(frame, keyframe point) confidence of the normal equations (see CameraIteration), [nf|1,N,1] for
        one window, [nw,nf|1,N,1] for a batch (a frame axis of 1 is broadcast to the frames); differentiable when it requires grad.
        robust, robust_scale (an extension): the robust loss of every pair's build, as in CameraIteration; the per-pair forms only (keyframe
        tensors with a frame axis): the keyframe form raises."""
        base = 1.0 if l2_regularizer_base is None else float(l2_regularizer_base)
        if self.vmatrix_batch_scramble:
            raise RuntimeError("vmatrix_batch_scramble=True is a 2-view quirk (bundlenet.py:45); the window solve has per-frame VMatrix only")
        ops.robust_kind(robust, robust_scale)
        if R.dim() == 4:
            return self._window_batch_iteration(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, base, level, weight, robust, robust_scale)
        nf = R.shape[0]
        intr = _intr_from_tiled(fx, fy, ox, oy)
        if self._wants_grad(conv1, conv2, D, B, R, T, W, weight):
            if self.training_path == "reference_split":
                raise RuntimeError("training_path='reference_split' has no torch-graph twin of the window solve; use training_path='fused'")
            Rn, Tn, Wn, status = _ag.window_iteration_fused(conv1, conv2, intr, p, D, B, R, T, W, self.mlp_params(str(level)), base,
                                                            exact_sym=self.exact_sym_grad, precision=self.precision, return_status=True,
                                                            weight=weight, robust=robust, robust_scale=robust_scale)
            self._check_status(status)
            return Rn, Tn, Wn
        frames = lambda t: t.expand(nf, *t.shape[1:]) if t.shape[0] == 1 else t
        wf = None if weight is None else _ag.window_weights(weight, None, nf, conv1.shape[1])
        lv = ops.Level(frames(conv1), conv2, frames(intr), frames(p), frames(D), frames(B), weight=wf, robust=robust, robust_scale=robust_scale)
        Rn, Tn, Wn, status = ops.lm_window_run([lv], 1, R, T, W, mlp_packed=[self.mlp_packed(str(level))], l2_regularizer_base=base,
                                               precision=self.precision)
        self._check_status(status)
        return Rn, Tn, Wn

    def _window_batch_iteration(self, conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, base, level, weight=None, robust=None, robust_scale=0.0):
        """WindowIteration on a batch of nw windows (R [nw,nf,3,3]): the fused path when gradients are recorded, else one iteration of
        ops.lm_window_batch_run."""
        nw, nf = R.shape[0], R.shape[1]
        intr = torch.stack([t.reshape(t.shape[0], t.shape[1], -1)[..., 0] for t in (fx, fy, ox, oy)], dim=-1).to(torch.float32)   # [nw,1|nf,4]
        ranks = {t.dim() for t in (conv1, p, D, B)}
        if len(ranks) != 1:
            raise RuntimeError("WindowIteration: conv1, p, D, B must all carry a frame axis ([nw,1|nf,...]) or all come without one ([nw,...])")
        if conv1.dim() == 3:
            self._require_keyframe_plain_loss(robust)
            return self._keyframe_batch_iteration(conv1, conv2, intr, p, D, B, R, T, W, base, level, weight)
        if self._wants_grad(conv1, conv2, D, B, R, T, W, weight):
            if self.training_path == "reference_split":
                raise RuntimeError("training_path='reference_split' has no torch-graph twin of the window solve; use training_path='fused'")
            Rn, Tn, Wn, status = _ag.window_batch_iteration_fused(conv1, conv2, intr, p, D, B, R, T, W, self.mlp_params(str(level)), base,
                                                                  exact_sym=self.exact_sym_grad, precision=self.precision, return_status=True,
                                                                  weight=weight, robust=robust, robust_scale=robust_scale)
            self._check_status(status)
            return Rn, Tn, Wn
        pairs = lambda t: (t.expand(nw, nf, *t.shape[2:]) if t.shape[1] == 1 else t).reshape(nw * nf, *t.shape[2:])
        wf = None if weight is None else _ag.window_weights(weight, nw, nf, conv1.shape[2])
        lv = ops.Level(pairs(conv1), pairs(conv2), pairs(intr), pairs(p), pairs(D), pairs(B), weight=wf, robust=robust, robust_scale=robust_scale)
        Rn, Tn, Wn, status = ops.lm_window_batch_run([lv], nw, 1, R.reshape(nw * nf, 3, 3), T.reshape(nw * nf, 3, 1), W,
                                                     mlp_packed=[self.mlp_packed(str(level))], l2_regularizer_base=base, precision=self.precision)
        self._check_status(status.reshape(nw, nf))
        return Rn.reshape(nw, nf, 3, 3), Tn.reshape(nw, nf, 3, 1), Wn

    def _keyframe_batch_iteration(self, conv1, conv2, intr, p, D, B, R, T, W, base, level, weight=None):
        """WindowIteration on nw windows with the keyframe tensors once per window (conv1 [nw,N,C], p [nw,3,N], D [nw,N,1], B [nw,N,K]):
        the keyframe build (banet_lm_keyframe_*), fused autograd path when gradients are recorded, else one iteration of
        ops.lm_keyframe_run.  fp32 SIMT only: a TF32 precision raises, and so do bfloat16 features and a bfloat16 basis."""
        self._require_keyframe_precision()
        self._require_keyframe_features(conv1, conv2)
        self._require_keyframe_basis(B)
        nw, nf = R.shape[0], R.shape[1]
        if self._wants_grad(conv1, conv2, D, B, R, T, W, weight):
            if self.training_path == "reference_split":
                raise RuntimeError("training_path='reference_split' has no torch-graph twin of the window solve; use training_path='fused'")
            Rn, Tn, Wn, status = _ag.window_batch_iteration_fused(conv1, conv2, intr, p, D, B, R, T, W, self.mlp_params(str(level)), base,
                                                                  exact_sym=self.exact_sym_grad, precision=self.precision, return_status=True,
                                                                  weight=weight)
            self._check_status(status)
            return Rn, Tn, Wn
        wf = None if weight is None else _ag.window_weights(weight, nw, nf, conv1.shape[1])
        lv = ops.KeyframeLevel(conv1, conv2.reshape(nw * nf, *conv2.shape[2:]), intr.expand(nw, nf, 4).reshape(nw * nf, 4), p, D, B, weight=wf)
        Rn, Tn, Wn, status = ops.lm_keyframe_run([lv], 1, R.reshape(nw * nf, 3, 3), T.reshape(nw * nf, 3, 1), W,
                                                 mlp_packed=[self.mlp_packed(str(level))], l2_regularizer_base=base, precision=self.precision)
        self._check_status(status.reshape(nw, nf))
        return Rn.reshape(nw, nf, 3, 3), Tn.reshape(nw, nf, 3, 1), Wn

    @staticmethod
    def _require_keyframe_features(*features) -> None:
        if any(t.dtype != torch.float32 for t in features):
            raise RuntimeError("the keyframe form of WindowIteration / WindowResize takes float32 features only; give the keyframe tensors per "
                               "frame ([nw,1|nf,...]) to WindowIteration for bfloat16 features")

    @staticmethod
    def _require_keyframe_basis(basis: Tensor) -> None:
        if basis.dtype != torch.float32:
            raise RuntimeError(f"the keyframe form of WindowIteration / WindowResize takes a float32 basis only (got {basis.dtype}); give the "
                               "keyframe tensors per frame ([nw,1|nf,...]) to WindowIteration for a bfloat16 basis")

    @staticmethod
    def _require_keyframe_plain_loss(robust: Optional[str]) -> None:
        if robust is not None:
            raise RuntimeError(f"robust={robust!r}: the keyframe form of WindowIteration / WindowResize has no robust loss; give the keyframe "
                               "tensors per frame ([nw,1|nf,...]) to WindowIteration, whose per-pair build has one")

    @staticmethod
    def _robust_scale_at(robust_scale, level) -> float:
        """robust_scale of the Resize methods at one level: a float for every level, or a mapping from level name ("2") to float."""
        if isinstance(robust_scale, Mapping):
            if str(level) not in robust_scale:
                raise RuntimeError(f"robust_scale has no entry for level {str(level)!r} (keys {sorted(robust_scale)})")
            return float(robust_scale[str(level)])
        return float(robust_scale)

    def _require_keyframe_precision(self) -> None:
        if self.precision not in (_lib.PREC_AUTO, _lib.PREC_FP32_SIMT):
            raise RuntimeError(f"precision {self.precision}: the keyframe form of WindowIteration has no tensor-core build; use AUTO or FP32_SIMT")

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

    @staticmethod
    def _swapped_f2(layer: Tensor, gfc):
        """conv2 of bundlenet.py:386-389: the half-swapped pyramid level.  float32: [F2|gx|gy] by grad_fixed_concat (one fused pass); bfloat16:
        the half-swapped F2 only, whose gradient channels the build derives on the fly (no fp32 3C copy)."""
        if layer.dtype == torch.bfloat16:
            h = layer.shape[0] // 2
            return torch.cat([layer[h:], layer[:h]]).contiguous()
        return gfc(layer, swap_halves=True)

    def CameraResize(self, intrisic, layers, points, _depths, reuse_variables=False, weight: Optional[Tensor] = None, *,
                     robust: Optional[str] = None, robust_scale: Union[float, Mapping[str, float]] = 0.0):
        """reference bundlenet.py:280-329 -> (rotations, translations), levels 0..3 x 1 iteration.  Differentiable w.r.t. the feature
        pyramid and the lambda-MLP parameters when gradients are being recorded (the depth is stop_gradient'ed, :288).
        `layers` may be bfloat16 (an autocast encoder's pyramid): conv1 is then the bfloat16 resample and conv2 the half-swapped F2 only.
        weight [nb,N,1] float32 (an extension): a per-point confidence at `points`, the same at every level (see CameraIteration);
        differentiable when it requires grad.
        robust, robust_scale (an extension): the robust loss of every level (see CameraIteration); robust_scale is one float, or a mapping
        from level name ("0" .. "3") to float, since feature magnitudes differ per level."""
        nb = layers[-1].shape[0]
        for level in range(0, 4) if robust is not None else ():
            ops.robust_kind(robust, self._robust_scale_at(robust_scale, level))
        _points, intr = self._prepare(intrisic, points)
        grad = self._wants_grad(*layers, weight)
        resample, gfc = (_ag.resample, _ag.grad_fixed_concat) if grad else (ops.resample, ops.grad_fixed_concat)
        d = ops.resample(_depths.detach(), _points, 0.5)                       # :289-290
        p = ops.compute_coordinates(_points, intr, True)
        R = torch.eye(3, device=points.device).repeat(nb, 1, 1)
        T = torch.zeros(nb, 3, 1, device=points.device)
        rotations, translations = [], []
        for level in range(0, 4):
            scale = 2 ** (3 - level)
            layer1 = resample(layers[level], _points, 1.0 / scale)             # :320
            layer2 = self._swapped_f2(layers[level], gfc)                      # :321-324
            R, T, _, _ = self._iterate(layer1, layer2, intr / scale, p, d, None, R, T, None, 1.0, level, weight=weight, robust=robust,
                                       robust_scale=self._robust_scale_at(robust_scale, level) if robust is not None else 0.0)
            rotations.append(R); translations.append(T)
        return rotations, translations

    def BundleResize(self, intrisic, layers, points, basis, init_depth, init_rotation=None, init_translation=None,
                     reuse_variables=False, weight: Optional[Tensor] = None, *, robust: Optional[str] = None,
                     robust_scale: Union[float, Mapping[str, float]] = 0.0):
        """reference bundlenet.py:332-399 -> (output_rotations, output_translations, output_depths), levels 2,3.  Differentiable w.r.t.
        the feature pyramid, the basis, the initial pose and the lambda-MLP parameters when gradients are being recorded
        (init_depth enters the LM only through stop_gradient, :341, and the output depth directly, :397).
        `layers` may be bfloat16 (an autocast encoder's pyramid): conv1 is then the bfloat16 resample and conv2 the half-swapped F2 only;
        their gradients come back in bfloat16.  `basis` may be bfloat16 too, independently of the pyramid (an autocast decoder's depth basis):
        it is sampled by the bfloat16 resample, the output depth is composed on it (banet_depth_compose_bf16), and its gradient comes back in
        bfloat16.  init_depth stays float32.
        weight [nb,N,1] float32 (an extension): a per-point confidence at `points`, the same at both levels (see CameraIteration);
        differentiable when it requires grad.
        robust, robust_scale (an extension): the robust loss of both levels (see CameraIteration); robust_scale is one float, or a mapping
        from level name ("2", "3") to float, since feature magnitudes differ per level."""
        nb = layers[-1].shape[0]
        K = basis.shape[-1]
        for level in range(2, 4) if robust is not None else ():
            ops.robust_kind(robust, self._robust_scale_at(robust_scale, level))
        _points, intr = self._prepare(intrisic, points)
        grad = self._wants_grad(*layers, basis, init_depth, init_rotation, init_translation, weight)
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
            layer2 = self._swapped_f2(layers[level], gfc)                      # :386-389
            R, T, W, _ = self._iterate(layer1, layer2, intr / scale, p, d, b, R, T, W, 1000.0, level, weight=weight, robust=robust,   # :393
                                       robust_scale=self._robust_scale_at(robust_scale, level) if robust is not None else 0.0)
            Rs.append(R); Ts.append(T)
            depth = compose(init_depth.reshape(nb, -1), basis.reshape(nb, -1, K), W)   # :397
            Ds.append(depth.reshape(nb, oh, ow, 1))
        return Rs, Ts, Ds

    def WindowResize(self, intrisic, key_layers, frame_layers, points, basis, init_depth, init_rotation=None, init_translation=None,
                     weight: Optional[Tensor] = None, *, robust: Optional[str] = None, robust_scale: Union[float, Mapping[str, float]] = 0.0,
                     return_cost: bool = False):
        """BundleResize's schedule (reference bundlenet.py:332-399) for nw keyframe windows of nf frames (an extension): levels 2, 3 x one
        joint window iteration, the keyframe depth init_depth + basis.W shared by the window's frames.
          intrisic [nw,4,1]            one camera per window (keyframe rays and every frame's projection)
          key_layers 4 x [nw,h_l,w_l,C]  the keyframes' feature pyramids;  frame_layers 4 x [nw,nf,h_l,w_l,C]  the frames' (F2 only)
          points [nw,N,2]              keyframe pixels in the reference's crop coordinates
          basis [nw,h/2,w/2,K], init_depth [nw,h/2,w/2,1];  init_rotation [nw,nf,3,3], init_translation [nw,nf,3,1] (default I, 0)
        conv1, p, D, B and W are once per window, conv2, R and T per frame.  -> (Rs [nw,nf,3,3], Ts [nw,nf,3,1], depths [nw,h/2,w/2,1]), one
        entry per level; last_status [nw,nf], or-ed over the levels.
        No gradients recorded: one ops.lm_keyframe_run iteration per level on the frames' F2 maps as they are.  Gradients recorded: the keyframe
        form of autograd.window_batch_iteration_fused per level on [F2|gx|gy] (the keyframe backward takes that layout only); gradients reach
        both pyramids, the basis, the initial pose and the lambda-MLP parameters, init_depth through the output depth only (:341, :397).
        AUTO or FP32_SIMT, float32 pyramids and a float32 basis only, like the keyframe form of WindowIteration.
        weight [nw,nf,N,1] or [nw,1,N,1] float32 (an extension): a per-(frame, point) confidence at `points`, the same at both levels (see
        WindowIteration); differentiable when it requires grad.
        robust: the keyframe build has no robust loss, so a robust loss raises; WindowIteration's per-pair form takes one.
        return_cost=True (an extension) -> (Rs, Ts, depths, Es): Es[i] [nw,nf] is level i's feature-metric cost (WindowFeatureMetricCost) at
        that level's output pose and depth coefficients, on its conv1, rays, depth, basis and weight and the frames' F2 maps as given (no
        [F2|gx|gy] copy); differentiable whenever the resize is, so it can train both pyramids without ground-truth poses.  Rs, Ts, depths and
        last_status are those of return_cost=False."""
        if self.vmatrix_batch_scramble:
            raise RuntimeError("vmatrix_batch_scramble=True is a 2-view quirk (bundlenet.py:45); the window solve has per-frame VMatrix only")
        self._require_keyframe_plain_loss(robust)
        self._require_keyframe_precision()
        self._require_keyframe_features(*key_layers, *frame_layers)
        self._require_keyframe_basis(basis)
        nw, nf, K = self._window_resize_shapes(intrisic, key_layers, frame_layers, points, basis, init_depth, init_rotation, init_translation)
        if weight is not None:
            _ag.window_weights(weight, nw, nf, points.shape[1])                # shape and dtype errors before any kernel runs
        _points, intr = self._prepare(intrisic, points)
        grad = self._wants_grad(*key_layers, *frame_layers, basis, init_rotation, init_translation, weight)
        resample = _ag.resample if grad else ops.resample
        compose = _ag.depth_compose if grad or self._wants_grad(init_depth) else ops.depth_compose
        d = ops.resample(init_depth.detach(), _points, 0.5)                    # :341-343, once per window
        b = resample(basis, _points, 0.5)                                      # :344
        p = ops.compute_coordinates(_points, intr, True)                       # :358
        dev = points.device
        R = torch.eye(3, device=dev).repeat(nw, nf, 1, 1) if init_rotation is None else init_rotation
        T = torch.zeros(nw, nf, 3, 1, device=dev) if init_translation is None else init_translation
        W = torch.zeros(nw, K, 1, device=dev)
        oh, ow = self.geo.out_hw
        Rs, Ts, Ds, Es = [], [], [], []
        status = None
        for level in range(2, 4):                                              # :376
            scale = 2 ** (3 - level)
            conv1 = resample(key_layers[level], _points, 1.0 / scale)         # :385, once per window
            F2 = frame_layers[level]
            if grad:                                                           # :386-389; the keyframe backward takes [F2|gx|gy] only
                conv2 = _ag.grad_fixed_concat(F2.reshape(nw * nf, *F2.shape[2:])).reshape(*F2.shape[:4], 3 * F2.shape[4])
            else:                                                              # the keyframe forward derives gx, gy from F2 itself
                conv2 = F2
            R, T, W = self._keyframe_batch_iteration(conv1, conv2, (intr / scale).unsqueeze(1), p, d, b, R, T, W, 1000.0, level, weight)   # :393
            status = self.last_status if status is None else status | self.last_status
            Rs.append(R); Ts.append(T)
            depth = compose(init_depth.reshape(nw, -1), basis.reshape(nw, -1, K), W)   # :397
            Ds.append(depth.reshape(nw, oh, ow, 1))
            if return_cost:
                Es.append(self._window_cost(conv1, F2, (intr / scale).unsqueeze(1), p, d, b, R, T, W, weight))
        self._check_status(status)
        return (Rs, Ts, Ds, Es) if return_cost else (Rs, Ts, Ds)

    def _window_resize_shapes(self, intrisic, key_layers, frame_layers, points, basis, init_depth, init_rotation, init_translation):
        """WindowResize's arguments checked against each other before any kernel runs -> (nw, nf, K).  nw comes from key_layers[3], nf from
        frame_layers[3]; an error names the argument that disagrees."""
        def fail(name, t, want):
            got = tuple(t.shape) if isinstance(t, torch.Tensor) else type(t).__name__
            raise _lib.BanetError(f"WindowResize: {name} must be {want}; got {got}")

        for name, ls in (("key_layers", key_layers), ("frame_layers", frame_layers)):
            if len(ls) != 4:
                raise _lib.BanetError(f"WindowResize: {name} must hold the 4 pyramid levels 0..3; got {len(ls)}")
        if key_layers[3].dim() != 4:
            fail("key_layers[3]", key_layers[3], "[nw,h,w,C]")
        if frame_layers[3].dim() != 5:
            fail("frame_layers[3]", frame_layers[3], "[nw,nf,h,w,C]")
        nw, nf, C = key_layers[3].shape[0], frame_layers[3].shape[1], key_layers[3].shape[3]
        for l in (2, 3):
            kl, fl = key_layers[l], frame_layers[l]
            if kl.dim() != 4 or kl.shape[0] != nw or kl.shape[3] != C:
                fail(f"key_layers[{l}]", kl, f"[nw={nw},h,w,C={C}]")
            if tuple(fl.shape) != (nw, nf, *kl.shape[1:]):
                fail(f"frame_layers[{l}]", fl, f"[nw,nf,h,w,C] = {(nw, nf, *kl.shape[1:])} (nw of key_layers, the keyframe's map size)")
        if intrisic.shape[0] != nw or intrisic.numel() != 4 * nw:
            fail("intrisic", intrisic, f"[nw={nw},4,1]")
        if points.dim() != 3 or points.shape[0] != nw or points.shape[2] != 2:
            fail("points", points, f"[nw={nw},N,2]")
        oh, ow = self.geo.out_hw
        if basis.dim() != 4 or tuple(basis.shape[:3]) != (nw, oh, ow):
            fail("basis", basis, f"[nw={nw},{oh},{ow},K]")
        if tuple(init_depth.shape) != (nw, oh, ow, 1):
            fail("init_depth", init_depth, f"[nw={nw},{oh},{ow},1]")
        for name, t, tail in (("init_rotation", init_rotation, (3, 3)), ("init_translation", init_translation, (3, 1))):
            if t is not None and tuple(t.shape) != (nw, nf, *tail):
                fail(name, t, f"[nw={nw},nf={nf},{tail[0]},{tail[1]}]")
        return nw, nf, basis.shape[3]

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
