"""Thin torch-facing wrappers over the C-ABI (include/banet_abi.h).  torch is plumbing only: it owns
device memory and streams; all arithmetic happens in libbanet.so.  No fallbacks: CPU tensors or a
missing library raise.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import BanetLevel, BanetSolveOpts, check, load

Tensor = torch.Tensor


_FEATURE_DTYPES = {torch.float32: _lib.DTYPE_F32, torch.bfloat16: _lib.DTYPE_BF16}      # also the basis dtypes


def _chk(t: Tensor, name: str, shape: Optional[Tuple[int, ...]] = None, features: bool = False) -> Tensor:
    """features=True: a feature map (conv1 / conv2 / resampler data) or a depth basis, which may also be bfloat16."""
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise _lib.BanetError(f"{name}: expected a CUDA tensor (banet_b200 has no CPU path)")
    if t.dtype != torch.float32 and not (features and t.dtype == torch.bfloat16):
        raise _lib.BanetError(f"{name}: expected {'float32 or bfloat16' if features else 'float32'}, got {t.dtype}")
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise _lib.BanetError(f"{name}: expected shape {tuple(shape)}, got {tuple(t.shape)}")
    return t.contiguous()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _ws(nbytes: int, device) -> Tensor:
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)


# ------------------------------------------------------------------------------------------ op level
class _EquationConstruction(torch.autograd.Function):
    """Drop-in for the reference TF op `equation_construction` and its registered gradient
    (reference bundlenet.py:76-82; utils.cu:150-171, 420-428)."""

    @staticmethod
    def forward(ctx, jacobian, gradient, difference, exact_sym):
        lib = load()
        J = _chk(jacobian, "jacobian"); nb, N, two, P = J.shape
        Cc = gradient.shape[2]
        G = _chk(gradient, "gradient", (nb, N, Cc, 2)); d = _chk(difference, "difference", (nb, N, Cc, 1))
        if two != 2:
            raise _lib.BanetError("jacobian must be [nb,N,2,P]")
        AtA = torch.empty(nb, P, P, device=J.device, dtype=torch.float32)
        Atb = torch.empty(nb, P, 1, device=J.device, dtype=torch.float32)
        nbytes = lib.banet_eqc_workspace_bytes(nb, N, Cc, P)
        ws = _ws(nbytes, J.device)
        check(lib.banet_eqc_fwd(J.data_ptr(), G.data_ptr(), d.data_ptr(), nb, N, Cc, P, AtA.data_ptr(), Atb.data_ptr(),
                                ws.data_ptr(), ws.numel(), _stream()), "banet_eqc_fwd")
        ctx.save_for_backward(J, G, d)
        ctx.exact_sym = bool(exact_sym)
        return AtA, Atb

    @staticmethod
    def backward(ctx, gAtA, gAtb):
        lib = load()
        J, G, d = ctx.saved_tensors
        nb, N, _, P = J.shape
        Cc = G.shape[2]
        gA = _chk(gAtA, "left_grad", (nb, P, P)); gb = _chk(gAtb, "right_grad", (nb, P, 1))
        dJ = torch.empty_like(J); dG = torch.empty_like(G); dd = torch.empty_like(d)
        check(lib.banet_eqc_bwd(J.data_ptr(), G.data_ptr(), d.data_ptr(), gA.data_ptr(), gb.data_ptr(), nb, N, Cc, P,
                                1 if ctx.exact_sym else 0, dJ.data_ptr(), dG.data_ptr(), dd.data_ptr(), _stream()),
              "banet_eqc_bwd")
        return dJ, dG, dd, None


def equation_construction(jacobian: Tensor, gradient: Tensor, difference: Tensor, exact_sym: bool = False):
    """AtA, Atb = equation_construction(jacobian[nb,N,2,P], gradient[nb,N,C,2], difference[nb,N,C,1]).
    Backward = the reference's `equation_construction_grad` (2*A*Ghat form) unless exact_sym."""
    return _EquationConstruction.apply(jacobian, gradient, difference, exact_sym)


def equation_construction_grad(jacobian, gradient, difference, left_grad, right_grad, exact_sym: bool = False):
    """Direct call of the gradient op (reference utils.cu:420-428)."""
    lib = load()
    J = _chk(jacobian, "jacobian"); nb, N, _, P = J.shape
    Cc = gradient.shape[2]
    G = _chk(gradient, "gradient", (nb, N, Cc, 2)); d = _chk(difference, "difference", (nb, N, Cc, 1))
    gA = _chk(left_grad, "left_grad", (nb, P, P)); gb = _chk(right_grad, "right_grad", (nb, P, 1))
    dJ = torch.empty_like(J); dG = torch.empty_like(G); dd = torch.empty_like(d)
    check(lib.banet_eqc_bwd(J.data_ptr(), G.data_ptr(), d.data_ptr(), gA.data_ptr(), gb.data_ptr(), nb, N, Cc, P,
                            1 if exact_sym else 0, dJ.data_ptr(), dG.data_ptr(), dd.data_ptr(), _stream()), "banet_eqc_bwd")
    return dJ, dG, dd


# ------------------------------------------------------------------------------------------ pre-steps
def compute_coordinates(points: Tensor, intr: Tensor, normalize: bool = True) -> Tensor:
    lib = load()
    pts = _chk(points, "points"); nb, N, _ = pts.shape
    it = _chk(intr, "intr", (nb, 4))
    p = torch.empty(nb, 3, N, device=pts.device, dtype=torch.float32)
    check(lib.banet_compute_coordinates(pts.data_ptr(), it.data_ptr(), nb, N, int(normalize), p.data_ptr(), _stream()),
          "banet_compute_coordinates")
    return p


def grad_fixed_concat(F: Tensor, swap_halves: bool = False, out: Optional[Tensor] = None) -> Tensor:
    """[nb,h,w,C] -> [nb,h,w,3C] = [F | gradx | grady] (reference bundlenet.py:92-100 + the concat of :386-389); `out` reuses a buffer."""
    lib = load()
    f = _chk(F, "F"); nb, h, w, Cc = f.shape
    if out is None:
        out = torch.empty(nb, h, w, 3 * Cc, device=f.device, dtype=torch.float32)
    else:
        out = _chk(out, "out", (nb, h, w, 3 * Cc))
    check(lib.banet_grad_fixed_concat(f.data_ptr(), nb, h, w, Cc, int(swap_halves), out.data_ptr(), _stream()),
          "banet_grad_fixed_concat")
    return out


def resample(data: Tensor, xy: Tensor, coord_scale: float = 1.0) -> Tensor:
    """Bilinear sampler, zero outside: data [nb,h,w,C] (float32, or bfloat16: banet_resample_bf16, fp32 arithmetic, the result rounded to
    bfloat16), xy [nb,N,2] -> [nb,N,C] in data's dtype."""
    lib = load()
    dt = _chk(data, "data", features=True); nb, h, w, Cc = dt.shape
    pts = _chk(xy, "xy"); N = pts.shape[1]
    out = torch.empty(nb, N, Cc, device=dt.device, dtype=dt.dtype)
    fn = lib.banet_resample_bf16 if dt.dtype == torch.bfloat16 else lib.banet_resample
    check(fn(dt.data_ptr(), pts.data_ptr(), float(coord_scale), nb, h, w, Cc, N, out.data_ptr(), _stream()),
          "banet_resample_bf16" if dt.dtype == torch.bfloat16 else "banet_resample")
    return out


def interpolate2d(data: Tensor, xy: Tensor, coord_scale: float = 1.0, with_mask: bool = False):
    """The legacy sampler (legacy/utils_python.py:61-117, 177-232): bilinear with clamped tap indices -> out [nb,N,C] (, mask [nb,N,1])."""
    lib = load()
    dt = _chk(data, "data"); nb, h, w, Cc = dt.shape
    pts = _chk(xy, "xy"); N = pts.shape[1]
    out = torch.empty(nb, N, Cc, device=dt.device, dtype=torch.float32)
    mask = torch.empty(nb, N, 1, device=dt.device, dtype=torch.float32) if with_mask else None
    check(lib.banet_interpolate2d(dt.data_ptr(), pts.data_ptr(), float(coord_scale), nb, h, w, Cc, N, out.data_ptr(), _ptr(mask), _stream()), "banet_interpolate2d")
    return (out, mask) if with_mask else out


def depth_compose(init_depth: Tensor, basis: Tensor, W: Tensor) -> Tensor:
    """init_depth [nb,M], basis [nb,M,K], W [nb,K,1] -> [nb,M]   (reference bundlenet.py:397).  basis may be bfloat16
    (banet_depth_compose_bf16: widened where it is read); everything else and the result are float32."""
    lib = load()
    bs = _chk(basis, "basis", features=True); nb, M, K = bs.shape
    d0 = _chk(init_depth, "init_depth", (nb, M)); Wt = _chk(W, "W", (nb, K, 1))
    out = torch.empty(nb, M, device=bs.device, dtype=torch.float32)
    name = "banet_depth_compose_bf16" if bs.dtype == torch.bfloat16 else "banet_depth_compose"
    check(getattr(lib, name)(d0.data_ptr(), bs.data_ptr(), Wt.data_ptr(), nb, M, K, out.data_ptr(), _stream()), name)
    return out


# ------------------------------------------------------------------------------------------ layer level
_ROBUST_KINDS = {None: _lib.ROBUST_NONE, "huber": _lib.ROBUST_HUBER, "cauchy": _lib.ROBUST_CAUCHY}


def robust_kind(robust: Optional[str], robust_scale: float) -> Tuple[int, float]:
    """(banet_level_t::robust, ::robust_scale) of a robust loss given by name: None, "huber" or "cauchy", with a finite scale > 0."""
    if robust not in _ROBUST_KINDS:
        raise _lib.BanetError(f"robust={robust!r}: expected None, 'huber' or 'cauchy'")
    if robust is None:
        return _lib.ROBUST_NONE, 0.0
    scale = float(robust_scale)
    if not (math.isfinite(scale) and scale > 0.0):
        raise _lib.BanetError(f"robust_scale={robust_scale!r}: a {robust} loss needs a finite scale > 0")
    return _ROBUST_KINDS[robust], scale


@dataclass
class Level:
    """One pyramid level in the reference's tensor layouts (see banet_level in include/banet_abi.h)."""
    conv1: Tensor             # [nb,N,C]      float32, or bfloat16 (conv1 and conv2 the same dtype)
    conv2: Tensor             # [nb,h,w,3C]  ([nb,h,w,C]: F2 only, gradients derived on the fly)
    intr: Tensor              # [nb,4]
    p: Tensor                 # [nb,3,N]
    D: Tensor                 # [nb,N,1]
    B: Optional[Tensor]       # [nb,N,K] or None; float32 or bfloat16, independent of the features' dtype
    grid: Optional[Tuple[int, int]] = None   # (grid_w, grid_h) if the N points are a row-major raster grid (locality hint)
    weight: Optional[Tensor] = None          # [nb,N,1] float32 per-point weight of the normal equations (H, g); None = unweighted
    robust: Optional[str] = None             # robust loss of the feature-metric error: None (squared), "huber" or "cauchy" (IRLS weight
    robust_scale: float = 0.0                # w_n = weight_n rho'(|d_n|^2) at each build); its scale delta > 0 in feature units

    def as_struct(self) -> Tuple[BanetLevel, list]:
        conv1 = _chk(self.conv1, "conv1", features=True); nb, N, Cc = conv1.shape
        conv2 = _chk(self.conv2, "conv2", features=True); _, h, w, c2 = conv2.shape
        if conv1.dtype != conv2.dtype:
            raise _lib.BanetError(f"conv1 ({conv1.dtype}) and conv2 ({conv2.dtype}) must have the same dtype (float32 or bfloat16)")
        intr = _chk(self.intr, "intr", (nb, 4)); p = _chk(self.p, "p", (nb, 3, N)); D = _chk(self.D, "D", (nb, N, 1))
        B = None if self.B is None else _chk(self.B, "B", features=True)
        K = 0 if B is None else B.shape[2]
        if B is not None and tuple(B.shape[:2]) != (nb, N):
            raise _lib.BanetError(f"B: expected [nb,N,K]=[{nb},{N},K], got {tuple(B.shape)}")
        if conv2.shape[0] != nb:
            raise _lib.BanetError("conv2 batch mismatch")
        wt = None if self.weight is None else _chk(self.weight, "weight", (nb, N, 1))
        keep = [conv1, conv2, intr, p, D, B, wt]
        gw, gh = (0, 0) if self.grid is None else self.grid
        if gw * gh not in (0, N):
            raise _lib.BanetError(f"grid {gw}x{gh} does not match N={N}")
        kind, scale = robust_kind(self.robust, self.robust_scale)
        return BanetLevel(nb, N, Cc, K, h, w, c2, conv1.data_ptr(), conv2.data_ptr(), intr.data_ptr(), p.data_ptr(),
                          D.data_ptr(), _ptr(B), gw, gh, _FEATURE_DTYPES[conv1.dtype], _FEATURE_DTYPES[torch.float32 if B is None else B.dtype],
                          _ptr(wt), kind, scale), keep


def lm_build(level: Level, R: Tensor, T: Tensor, W: Optional[Tensor], precision: int = _lib.PREC_AUTO):
    """H [nb,P,P], g [nb,P], rbar_sum [nb,C], nvalid [nb] of one iteration at the current (R,T,W)."""
    lib = load()
    st, keep = level.as_struct()
    nb, K, Cc = st.nb, st.K, st.C
    P = 6 + K
    R = _chk(R, "R", (nb, 3, 3)); T = _chk(T, "T", (nb, 3, 1))
    Wt = None if K == 0 else _chk(W, "W", (nb, K, 1))
    dev = R.device
    H = torch.empty(nb, P, P, device=dev, dtype=torch.float32); g = torch.empty(nb, P, device=dev, dtype=torch.float32)
    rbar = torch.empty(nb, Cc, device=dev, dtype=torch.float32); nvalid = torch.empty(nb, device=dev, dtype=torch.float32)
    ws = _ws(lib.banet_lm_build_workspace_bytes(C.byref(st), precision), dev)
    check(lib.banet_lm_build(C.byref(st), R.data_ptr(), T.data_ptr(), _ptr(Wt), precision, H.data_ptr(), g.data_ptr(),
                             rbar.data_ptr(), nvalid.data_ptr(), ws.data_ptr(), ws.numel(), _stream()), "banet_lm_build")
    return H, g, rbar, nvalid


def lm_cost(level: Level, R: Tensor, T: Tensor, W: Optional[Tensor], per_point: bool = False):
    """Feature-metric cost of the level at (R, T, W) (banet_lm_cost): cost [nb] = sum_n c_n rho(s_n) over the in-bounds points, s_n the
    squared norm of the build's residual, c_n the point weight and rho the level's robust loss (rho(s) = s without one), and nvalid [nb],
    bit for bit lm_build's.  per_point=True appends s [nb,N,1] (0 at masked points) and mask [nb,N,1]."""
    lib = load()
    st, keep = level.as_struct()
    nb, K, N = st.nb, st.K, st.N
    R = _chk(R, "R", (nb, 3, 3)); T = _chk(T, "T", (nb, 3, 1))
    Wt = None if K == 0 else _chk(W, "W", (nb, K, 1))
    dev = R.device
    cost = torch.empty(nb, device=dev, dtype=torch.float32); nvalid = torch.empty(nb, device=dev, dtype=torch.float32)
    s = torch.empty(nb, N, 1, device=dev, dtype=torch.float32) if per_point else None
    mask = torch.empty(nb, N, 1, device=dev, dtype=torch.float32) if per_point else None
    nbytes = lib.banet_lm_cost_workspace_bytes(C.byref(st))
    if nbytes == 0:
        check(lib.banet_lm_cost(C.byref(st), R.data_ptr(), T.data_ptr(), _ptr(Wt), cost.data_ptr(), nvalid.data_ptr(), None, None, None, 0,
                                _stream()), "banet_lm_cost")
    ws = _ws(nbytes, dev)
    check(lib.banet_lm_cost(C.byref(st), R.data_ptr(), T.data_ptr(), _ptr(Wt), cost.data_ptr(), nvalid.data_ptr(), _ptr(s), _ptr(mask),
                            ws.data_ptr(), ws.numel(), _stream()), "banet_lm_cost")
    return (cost, nvalid, s, mask) if per_point else (cost, nvalid)


def lm_cost_bwd(level: Level, R: Tensor, T: Tensor, W: Optional[Tensor], dcost: Tensor, return_dweight: bool = False):
    """Backward of lm_cost's cost (banet_lm_cost_bwd): dcost [nb] -> dconv1, dconv2, dD, dB, dR, dT, dW (+ dweight [nb,N,1] =
    dcost rho(s_n) with return_dweight), the exact derivative of the cost through the bilinear sample of F2.  dconv2 has conv2's layout
    (on [F2|gx|gy] its gradient channels are zero); dconv1, dconv2 and dB are float32 whatever the dtypes of the features and the basis."""
    lib = load()
    st, keep = level.as_struct()
    nb, K, Cc, N = st.nb, st.K, st.C, st.N
    R = _chk(R, "R", (nb, 3, 3)); T = _chk(T, "T", (nb, 3, 1))
    Wt = None if K == 0 else _chk(W, "W", (nb, K, 1))
    dc = _chk(dcost.reshape(-1), "dcost", (nb,))
    dev = R.device
    dconv1 = torch.empty(nb, N, Cc, device=dev); dconv2 = torch.empty(nb, st.h, st.w, st.conv2_channels, device=dev)
    dD = torch.empty(nb, N, 1, device=dev); dB = None if K == 0 else torch.empty(nb, N, K, device=dev)
    dR = torch.empty(nb, 3, 3, device=dev); dT = torch.empty(nb, 3, 1, device=dev); dW = None if K == 0 else torch.empty(nb, K, 1, device=dev)
    dweight = torch.empty(nb, N, 1, device=dev) if return_dweight else None
    check(lib.banet_lm_cost_bwd(C.byref(st), R.data_ptr(), T.data_ptr(), _ptr(Wt), dc.data_ptr(), dconv1.data_ptr(), dconv2.data_ptr(),
                                dD.data_ptr(), _ptr(dB), dR.data_ptr(), dT.data_ptr(), _ptr(dW), _ptr(dweight), _stream()), "banet_lm_cost_bwd")
    out = (dconv1, dconv2, dD, dB, dR, dT, dW)
    return out + (dweight,) if return_dweight else out


def pack_mlp(params: Sequence[Tuple[Tensor, Tensor]]) -> Tensor:
    """[(W1[cin,cout], b1[cout]), ...x5] -> packed fp32 buffer expected by banet_lm_lambda."""
    return torch.cat([t.reshape(-1).to(torch.float32) for wb in params for t in wb]).contiguous()


def lm_lambda(rbar_sum: Tensor, N: int, mlp_packed: Tensor, base: float) -> Tensor:
    lib = load()
    rb = _chk(rbar_sum, "rbar_sum"); nb, Cc = rb.shape
    mp = _chk(mlp_packed, "mlp_packed")
    if mp.numel() != lib.banet_mlp_param_count(Cc):
        raise _lib.BanetError(f"mlp_packed has {mp.numel()} params, expected {lib.banet_mlp_param_count(Cc)} for C={Cc}")
    lam = torch.empty(nb, device=rb.device, dtype=torch.float32)
    check(lib.banet_lm_lambda(rb.data_ptr(), nb, int(N), Cc, mp.data_ptr(), float(base), lam.data_ptr(), _stream()), "banet_lm_lambda")
    return lam


def lm_solve_update(H: Tensor, g: Tensor, lam: Tensor, R: Tensor, T: Tensor, W: Optional[Tensor],
                    damping_eps: float = 1e-5, undamped_last: Optional[bool] = None, vmatrix_batch_scramble: bool = False):
    """-> R', T', W', delta [nb,P], status [nb] (int32).  undamped_last None: True for K > 0 (bundlenet.py:266), False for pose-only (:182)."""
    lib = load()
    Hc = _chk(H, "H"); nb, P, _ = Hc.shape
    K = P - 6
    if undamped_last is None:
        undamped_last = K > 0
    gc = _chk(g.reshape(nb, P), "g", (nb, P)); lc = _chk(lam.reshape(nb), "lambda", (nb,))
    R = _chk(R, "R", (nb, 3, 3)); T = _chk(T, "T", (nb, 3, 1))
    Wt = None if K == 0 else _chk(W, "W", (nb, K, 1))
    dev = Hc.device
    Ro = torch.empty_like(R); To = torch.empty_like(T); Wo = None if K == 0 else torch.empty_like(Wt)
    delta = torch.empty(nb, P, device=dev, dtype=torch.float32)
    status = torch.empty(nb, device=dev, dtype=torch.int32)
    opts = BanetSolveOpts(float(damping_eps), int(undamped_last), int(vmatrix_batch_scramble))
    check(lib.banet_lm_solve_update(Hc.data_ptr(), gc.data_ptr(), lc.data_ptr(), nb, K, C.byref(opts), R.data_ptr(), T.data_ptr(),
                                    _ptr(Wt), Ro.data_ptr(), To.data_ptr(), _ptr(Wo), delta.data_ptr(), status.data_ptr(),
                                    None, 0, _stream()), "banet_lm_solve_update")
    return Ro, To, Wo, delta, status


def lm_step(H: Tensor, g: Tensor, rbar_sum: Optional[Tensor], N: int, mlp_packed: Optional[Tensor], base: float, R: Tensor, T: Tensor,
            W: Optional[Tensor], lam: Optional[Tensor] = None, damping_eps: float = 1e-5, undamped_last: Optional[bool] = None):
    """banet_lm_step: lambda-MLP (or the given `lam`) + damping + solve + update in one launch -> R', T', W', delta, lambda, status."""
    lib = load()
    Hc = _chk(H, "H"); nb, P, _ = Hc.shape
    K = P - 6
    gc = _chk(g.reshape(nb, P), "g", (nb, P))
    R = _chk(R, "R", (nb, 3, 3)); T = _chk(T, "T", (nb, 3, 1)); Wt = None if K == 0 else _chk(W, "W", (nb, K, 1))
    rb = None if rbar_sum is None else _chk(rbar_sum, "rbar_sum"); mp = None if mlp_packed is None else _chk(mlp_packed, "mlp_packed")
    lin = None if lam is None else _chk(lam.reshape(nb), "lambda", (nb,))
    Cc = 1 if rb is None else rb.shape[1]
    if undamped_last is None:
        undamped_last = K > 0
    dev = Hc.device
    Ro = torch.empty_like(R); To = torch.empty_like(T); Wo = None if K == 0 else torch.empty_like(Wt)
    delta = torch.empty(nb, P, device=dev); lout = torch.empty(nb, device=dev); status = torch.empty(nb, device=dev, dtype=torch.int32)
    opts = BanetSolveOpts(float(damping_eps), int(undamped_last), 0)
    check(lib.banet_lm_step(Hc.data_ptr(), gc.data_ptr(), _ptr(rb), nb, int(N), Cc, K, _ptr(mp), float(base), _ptr(lin), C.byref(opts), R.data_ptr(),
                            T.data_ptr(), _ptr(Wt), Ro.data_ptr(), To.data_ptr(), _ptr(Wo), delta.data_ptr(), lout.data_ptr(), status.data_ptr(), _stream()),
          "banet_lm_step")
    return Ro, To, Wo, delta, lout, status


def _prepare_run(levels, query, query_args, mlp_packed, l2_regularizer_base, damping_eps, undamped_last, vmatrix_batch_scramble):
    """Argument block of the whole-solve wrappers and LMRunGraph: the structs of the levels (Level or KeyframeLevel), lambda-MLP pointers,
    options and the workspace size from the C-ABI query `query(structs, nlevels, *query_args)`, 0 when the query rejects the levels."""
    lib = load()
    structs, keep = [], []
    for lv in levels:
        s, k = lv.as_struct(); structs.append(s); keep.append(k)
    arr = (type(structs[0]) * len(structs))(*structs)
    K = structs[0].K
    if undamped_last is None:
        undamped_last = K > 0
    if l2_regularizer_base is None:              # BundleIteration scales lambda by 1000 (bundlenet.py:252-253, 393); CameraIteration ignores the base (:165-173)
        l2_regularizer_base = 1000.0 if K > 0 else 1.0
    mlp_ptrs = (C.c_void_p * len(structs))()
    have = False
    for i in range(len(structs)):
        m = None if mlp_packed is None else mlp_packed[i]
        if m is not None:
            m = _chk(m, "mlp_packed"); keep.append(m); have = True
            if m.numel() != lib.banet_mlp_param_count(structs[i].C):
                raise _lib.BanetError("mlp_packed size mismatch")
        mlp_ptrs[i] = None if m is None else m.data_ptr()
    opts = BanetSolveOpts(float(damping_eps), int(undamped_last), int(vmatrix_batch_scramble))
    nbytes = query(arr, len(structs), *query_args)
    return arr, (mlp_ptrs if have else None), float(l2_regularizer_base), opts, int(nbytes), keep


def lm_run(levels: Sequence[Level], iters_per_level: int, R: Tensor, T: Tensor, W: Optional[Tensor],
           mlp_packed: Optional[Sequence[Optional[Tensor]]] = None, l2_regularizer_base: Optional[float] = None,
           lambda_fixed: float = -1.0, damping_eps: float = 1e-5, undamped_last: Optional[bool] = None,
           vmatrix_batch_scramble: bool = False, precision: int = _lib.PREC_AUTO, workspace: Optional[Tensor] = None):
    """Whole coarse-to-fine solve on the device (banet_lm_run).  Returns new (R,T,W,status); inputs are not modified."""
    lib = load()
    arr, mlp_ptrs, base, opts, nbytes, _keep = _prepare_run(levels, lib.banet_lm_run_workspace_bytes, (precision,), mlp_packed, l2_regularizer_base,
                                                            damping_eps, undamped_last, vmatrix_batch_scramble)
    if nbytes == 0:
        check(-4, "banet_lm_run_workspace_bytes")
    nb, K = arr[0].nb, arr[0].K
    R = _chk(R, "R", (nb, 3, 3)).clone(); T = _chk(T, "T", (nb, 3, 1)).clone()
    Wt = None if K == 0 else _chk(W, "W", (nb, K, 1)).clone()
    ws = workspace if workspace is not None and workspace.numel() >= nbytes else _ws(nbytes, R.device)
    status = torch.empty(nb, device=R.device, dtype=torch.int32)
    check(lib.banet_lm_run(arr, len(arr), int(iters_per_level), mlp_ptrs, base, float(lambda_fixed), C.byref(opts), precision,
                           R.data_ptr(), T.data_ptr(), _ptr(Wt), status.data_ptr(), ws.data_ptr(), ws.numel(), _stream()), "banet_lm_run")
    return R, T, Wt, status


def lm_window_run(levels: Sequence[Level], iters_per_level: int, R: Tensor, T: Tensor, W: Tensor,
                  mlp_packed: Optional[Sequence[Optional[Tensor]]] = None, l2_regularizer_base: Optional[float] = None,
                  lambda_fixed: float = -1.0, damping_eps: float = 1e-5, undamped_last: bool = True,
                  precision: int = _lib.PREC_AUTO, workspace: Optional[Tensor] = None):
    """Joint coarse-to-fine solve of a keyframe window (banet_lm_window_run; an extension, SURVEY.md section 8f-4): the nf pairs of every
    level are (keyframe -> frame f) and share ONE depth-coefficient vector.  R [nf,3,3], T [nf,3,1] per frame, W [K,1] (or [1,K,1]) shared.
    Returns new (R, T, W [K,1], status [nf])."""
    lib = load()
    arr, mlp_ptrs, base, opts, nbytes, _keep = _prepare_run(levels, lib.banet_lm_window_run_workspace_bytes, (precision,), mlp_packed,
                                                            l2_regularizer_base, damping_eps, undamped_last, False)
    if nbytes == 0:
        check(-4, "banet_lm_window_run_workspace_bytes")
    nf, K = arr[0].nb, arr[0].K
    R = _chk(R, "R", (nf, 3, 3)).clone(); T = _chk(T, "T", (nf, 3, 1)).clone()
    Wt = _chk(W.reshape(1, K, 1), "W", (1, K, 1)).repeat(nf, 1, 1).contiguous()
    ws = workspace if workspace is not None and workspace.numel() >= nbytes else _ws(nbytes, R.device)
    status = torch.empty(nf, device=R.device, dtype=torch.int32)
    check(lib.banet_lm_window_run(arr, len(arr), int(iters_per_level), mlp_ptrs, base, float(lambda_fixed), C.byref(opts), precision,
                                  R.data_ptr(), T.data_ptr(), Wt.data_ptr(), status.data_ptr(), ws.data_ptr(), ws.numel(), _stream()),
          "banet_lm_window_run")
    return R, T, Wt[0].clone(), status


def lm_window_solve_update(H: Tensor, g: Tensor, lam: Tensor, R: Tensor, T: Tensor, W: Tensor, damping_eps: float = 1e-5, undamped_last: bool = True):
    """One iteration of a keyframe window after the build (banet_lm_window_solve_update): H [nf,P,P], g [nf,P] from lm_build with nb = nf,
    lam [1], R [nf,3,3], T [nf,3,1], W [K,1] shared -> R', T', W' [K,1], delta [6 nf + K] (the joint solution), status [nf] (int32)."""
    lib = load()
    Hc = _chk(H, "H"); nf, P, _ = Hc.shape
    K = P - 6
    gc = _chk(g.reshape(nf, P), "g", (nf, P)); lc = _chk(lam.reshape(1), "lambda", (1,))
    R = _chk(R, "R", (nf, 3, 3)); T = _chk(T, "T", (nf, 3, 1)); Wt = _chk(W.reshape(K, 1), "W", (K, 1))
    dev = Hc.device
    Ro = torch.empty_like(R); To = torch.empty_like(T); Wo = torch.empty_like(Wt)
    delta = torch.empty(6 * nf + K, device=dev); status = torch.empty(nf, device=dev, dtype=torch.int32)
    opts = BanetSolveOpts(float(damping_eps), int(undamped_last), 0)
    ws = _ws(lib.banet_lm_window_solve_update_workspace_bytes(nf, K), dev)
    check(lib.banet_lm_window_solve_update(Hc.data_ptr(), gc.data_ptr(), lc.data_ptr(), nf, K, C.byref(opts), R.data_ptr(), T.data_ptr(), Wt.data_ptr(),
                                           Ro.data_ptr(), To.data_ptr(), Wo.data_ptr(), delta.data_ptr(), status.data_ptr(), ws.data_ptr(), ws.numel(),
                                           _stream()), "banet_lm_window_solve_update")
    return Ro, To, Wo, delta, status


def lm_window_batch_run(levels: Sequence[Level], nw: int, iters_per_level: int, R: Tensor, T: Tensor, W: Tensor,
                        mlp_packed: Optional[Sequence[Optional[Tensor]]] = None, l2_regularizer_base: Optional[float] = None,
                        lambda_fixed: float = -1.0, damping_eps: float = 1e-5, undamped_last: bool = True,
                        precision: int = _lib.PREC_AUTO, workspace: Optional[Tensor] = None):
    """Joint coarse-to-fine solve of a batch of nw keyframe windows (banet_lm_window_batch_run): every level holds nb = nw * nf pairs, pair
    w * nf + f = (keyframe of window w -> frame f).  R [nb,3,3], T [nb,3,1] per frame, W [nw,K,1] per window.  Returns new
    (R, T, W [nw,K,1], status [nb])."""
    lib = load()
    arr, mlp_ptrs, base, opts, nbytes, _keep = _prepare_run(levels, lib.banet_lm_window_batch_run_workspace_bytes, (int(nw), precision), mlp_packed,
                                                            l2_regularizer_base, damping_eps, undamped_last, False)
    nb, K = arr[0].nb, arr[0].K
    if nbytes == 0:
        check(-4 if nw > 0 and nb % nw == 0 else -1, "banet_lm_window_batch_run_workspace_bytes")
    R = _chk(R, "R", (nb, 3, 3)).clone(); T = _chk(T, "T", (nb, 3, 1)).clone()
    Wt = _chk(W.reshape(nw, K, 1), "W", (nw, K, 1)).clone()
    ws = workspace if workspace is not None and workspace.numel() >= nbytes else _ws(nbytes, R.device)
    status = torch.empty(nb, device=R.device, dtype=torch.int32)
    check(lib.banet_lm_window_batch_run(arr, len(arr), int(nw), int(iters_per_level), mlp_ptrs, base, float(lambda_fixed), C.byref(opts), precision,
                                        R.data_ptr(), T.data_ptr(), Wt.data_ptr(), status.data_ptr(), ws.data_ptr(), ws.numel(), _stream()),
          "banet_lm_window_batch_run")
    return R, T, Wt, status


def lm_window_batch_solve_update(H: Tensor, g: Tensor, lam: Tensor, R: Tensor, T: Tensor, W: Tensor, damping_eps: float = 1e-5,
                                 undamped_last: bool = True):
    """One iteration of nw keyframe windows after the build (banet_lm_window_batch_solve_update): H [nw*nf,P,P], g [nw*nf,P] from lm_build,
    lam [nw], R [nw*nf,3,3], T [nw*nf,3,1], W [nw,K,1] -> R', T', W' [nw,K,1], delta [nw, 6 nf + K], status [nw*nf] (int32)."""
    lib = load()
    Hc = _chk(H, "H"); nb, P, _ = Hc.shape
    K = P - 6
    nw = lam.numel()
    if nw == 0 or nb % nw:
        raise _lib.BanetError(f"lambda has {nw} windows, which does not divide the {nb} pairs")
    nf = nb // nw
    gc = _chk(g.reshape(nb, P), "g", (nb, P)); lc = _chk(lam.reshape(nw), "lambda", (nw,))
    R = _chk(R, "R", (nb, 3, 3)); T = _chk(T, "T", (nb, 3, 1)); Wt = _chk(W.reshape(nw, K, 1), "W", (nw, K, 1))
    dev = Hc.device
    Ro = torch.empty_like(R); To = torch.empty_like(T); Wo = torch.empty_like(Wt)
    delta = torch.empty(nw, 6 * nf + K, device=dev); status = torch.empty(nb, device=dev, dtype=torch.int32)
    opts = BanetSolveOpts(float(damping_eps), int(undamped_last), 0)
    ws = _ws(lib.banet_lm_window_batch_solve_update_workspace_bytes(nw, nf, K), dev)
    check(lib.banet_lm_window_batch_solve_update(Hc.data_ptr(), gc.data_ptr(), lc.data_ptr(), nw, nf, K, C.byref(opts), R.data_ptr(), T.data_ptr(),
                                                 Wt.data_ptr(), Ro.data_ptr(), To.data_ptr(), Wo.data_ptr(), delta.data_ptr(), status.data_ptr(),
                                                 ws.data_ptr(), ws.numel(), _stream()), "banet_lm_window_batch_solve_update")
    return Ro, To, Wo, delta, status


@dataclass
class KeyframeLevel:
    """One pyramid level of nw keyframe windows with the keyframe tensors given once per window (banet_keyframe_level in
    include/banet_abi.h).  Pair w * nf + f is (keyframe of window w -> frame f)."""
    conv1: Tensor             # [nw,N,C]
    conv2: Tensor             # [nw*nf,h,w,3C]  ([nw*nf,h,w,C]: F2 only, forward only)
    intr: Tensor              # [nw*nf,4]
    p: Tensor                 # [nw,3,N]
    D: Tensor                 # [nw,N,1]
    B: Tensor                 # [nw,N,K]
    weight: Optional[Tensor] = None          # [nw*nf,N,1] float32 per-(frame, point) weight of the normal equations; None = unweighted

    def as_struct(self) -> Tuple[_lib.BanetKeyframeLevel, list]:
        if self.conv1.dtype != torch.float32 or self.conv2.dtype != torch.float32:
            raise _lib.BanetError(f"keyframe levels take float32 features only (conv1 {self.conv1.dtype}, conv2 {self.conv2.dtype})")
        conv1 = _chk(self.conv1, "conv1"); nw, N, Cc = conv1.shape
        conv2 = _chk(self.conv2, "conv2"); nb, h, w, c2 = conv2.shape
        if nb % nw:
            raise _lib.BanetError(f"conv2 has {nb} pairs, which is not a multiple of the {nw} windows")
        nf = nb // nw
        B = _chk(self.B, "B"); K = B.shape[2]
        _chk(B, "B", (nw, N, K))
        intr = _chk(self.intr, "intr", (nb, 4)); p = _chk(self.p, "p", (nw, 3, N)); D = _chk(self.D, "D", (nw, N, 1))
        wt = None if self.weight is None else _chk(self.weight, "weight", (nb, N, 1))
        keep = [conv1, conv2, intr, p, D, B, wt]
        return _lib.BanetKeyframeLevel(nw, nf, N, Cc, K, h, w, c2, conv1.data_ptr(), p.data_ptr(), D.data_ptr(), B.data_ptr(),
                                       conv2.data_ptr(), intr.data_ptr(), _ptr(wt)), keep


def lm_keyframe_build(level: KeyframeLevel, R: Tensor, T: Tensor, W: Tensor):
    """The keyframe build (banet_lm_keyframe_build): R [nw*nf,3,3], T [nw*nf,3,1], W [nw,K,1] -> the window-reduced per-pair system
    H [nw*nf,P,P], g [nw*nf,P], rbar_sum [nw*nf,C], nvalid [nw*nf]: banet_lm_build's per-pair values except that frame 0's depth block holds
    the window's whole depth block and the other frames' depth blocks are zero."""
    lib = load()
    st, keep = level.as_struct()
    nw, nb, K, Cc = st.nw, st.nw * st.nf, st.K, st.C
    P = 6 + K
    R = _chk(R, "R", (nb, 3, 3)); T = _chk(T, "T", (nb, 3, 1)); Wt = _chk(W.reshape(nw, K, 1), "W", (nw, K, 1))
    dev = R.device
    H = torch.empty(nb, P, P, device=dev); g = torch.empty(nb, P, device=dev)
    rbar = torch.empty(nb, Cc, device=dev); nvalid = torch.empty(nb, device=dev)
    nbytes = lib.banet_lm_keyframe_build_workspace_bytes(C.byref(st))
    ws = _ws(nbytes, dev)
    check(lib.banet_lm_keyframe_build(C.byref(st), R.data_ptr(), T.data_ptr(), Wt.data_ptr(), H.data_ptr(), g.data_ptr(), rbar.data_ptr(),
                                      nvalid.data_ptr(), ws.data_ptr(), ws.numel(), _stream()), "banet_lm_keyframe_build")
    return H, g, rbar, nvalid


def lm_keyframe_build_bwd(level: KeyframeLevel, R: Tensor, T: Tensor, W: Tensor, dH: Tensor, dg: Tensor, drbar_sum: Tensor,
                          exact_sym: bool = False, return_dweight: bool = False):
    """Backward of lm_keyframe_build (banet_lm_keyframe_build_bwd) -> dconv1 [nw,N,C], dconv2 [nw*nf,h,w,3C], dD [nw,N,1], dB [nw,N,K],
    dR, dT [nw*nf,...], dW [nw,K,1].  Only frame 0's depth block of dH is read.  On a weighted level every gradient carries the point
    weights.  return_dweight=True appends dweight [nw*nf,N,1] (banet_lm_keyframe_build_bwd_weighted; on an unweighted level, the gradient
    at weights of ones)."""
    lib = load()
    st, keep = level.as_struct()
    nw, nb, K, Cc, N = st.nw, st.nw * st.nf, st.K, st.C, st.N
    P = 6 + K
    R = _chk(R, "R", (nb, 3, 3)); T = _chk(T, "T", (nb, 3, 1)); Wt = _chk(W.reshape(nw, K, 1), "W", (nw, K, 1))
    dH = _chk(dH, "dH", (nb, P, P)); dg = _chk(dg.reshape(nb, P), "dg", (nb, P)); dr = _chk(drbar_sum, "drbar_sum", (nb, Cc))
    dev = R.device
    dconv1 = torch.empty(nw, N, Cc, device=dev); dconv2 = torch.empty(nb, st.h, st.w, 3 * Cc, device=dev)
    dD = torch.empty(nw, N, 1, device=dev); dB = torch.empty(nw, N, K, device=dev)
    dR = torch.empty(nb, 3, 3, device=dev); dT = torch.empty(nb, 3, 1, device=dev); dW = torch.empty(nw, K, 1, device=dev)
    if not return_dweight:
        check(lib.banet_lm_keyframe_build_bwd(C.byref(st), R.data_ptr(), T.data_ptr(), Wt.data_ptr(), dH.data_ptr(), dg.data_ptr(), dr.data_ptr(),
                                              int(bool(exact_sym)), dconv1.data_ptr(), dconv2.data_ptr(), dD.data_ptr(), dB.data_ptr(), dR.data_ptr(),
                                              dT.data_ptr(), dW.data_ptr(), _stream()), "banet_lm_keyframe_build_bwd")
        return dconv1, dconv2, dD, dB, dR, dT, dW
    dweight = torch.empty(nb, N, 1, device=dev)
    check(lib.banet_lm_keyframe_build_bwd_weighted(C.byref(st), R.data_ptr(), T.data_ptr(), Wt.data_ptr(), dH.data_ptr(), dg.data_ptr(),
                                                   dr.data_ptr(), int(bool(exact_sym)), dconv1.data_ptr(), dconv2.data_ptr(), dD.data_ptr(),
                                                   dB.data_ptr(), dR.data_ptr(), dT.data_ptr(), dW.data_ptr(), dweight.data_ptr(), _stream()),
          "banet_lm_keyframe_build_bwd_weighted")
    return dconv1, dconv2, dD, dB, dR, dT, dW, dweight


def lm_keyframe_cost(level: KeyframeLevel, R: Tensor, T: Tensor, W: Tensor, per_point: bool = False):
    """Feature-metric cost of keyframe windows at (R, T, W) (banet_lm_keyframe_cost): R [nw*nf,3,3], T [nw*nf,3,1], W [nw,K,1] -> cost
    [nw*nf] = sum_n c_n s_n over the in-bounds points of each pair (w*nf + f), s_n the squared norm of the keyframe build's residual and c_n
    the level's weight, and nvalid [nw*nf], bit for bit lm_keyframe_build's.  Bit for bit lm_cost on the keyframe replicated per frame.
    per_point=True appends s [nw*nf,N,1] (0 at masked points) and mask [nw*nf,N,1]."""
    lib = load()
    st, keep = level.as_struct()
    nw, nb, K, N = st.nw, st.nw * st.nf, st.K, st.N
    R = _chk(R, "R", (nb, 3, 3)); T = _chk(T, "T", (nb, 3, 1)); Wt = _chk(W, "W", (nw, K, 1))
    dev = R.device
    cost = torch.empty(nb, device=dev); nvalid = torch.empty(nb, device=dev)
    s = torch.empty(nb, N, 1, device=dev) if per_point else None
    mask = torch.empty(nb, N, 1, device=dev) if per_point else None
    ws = _ws(lib.banet_lm_keyframe_cost_workspace_bytes(C.byref(st)), dev)
    check(lib.banet_lm_keyframe_cost(C.byref(st), R.data_ptr(), T.data_ptr(), Wt.data_ptr(), cost.data_ptr(), nvalid.data_ptr(), _ptr(s),
                                     _ptr(mask), ws.data_ptr(), ws.numel(), _stream()), "banet_lm_keyframe_cost")
    return (cost, nvalid, s, mask) if per_point else (cost, nvalid)


def lm_keyframe_cost_bwd(level: KeyframeLevel, R: Tensor, T: Tensor, W: Tensor, dcost: Tensor, return_dweight: bool = False):
    """Backward of lm_keyframe_cost's cost (banet_lm_keyframe_cost_bwd): dcost [nw*nf] -> dconv1 [nw,N,C], dconv2 (conv2's layout, zero
    gradient channels on [F2|gx|gy]), dD [nw,N,1], dB [nw,N,K], dR, dT [nw*nf,...], dW [nw,K,1] (+ dweight [nw*nf,N,1] = dcost s_n with
    return_dweight): the exact derivative through the bilinear sample of F2, the keyframe's gradients summed over the frames."""
    lib = load()
    st, keep = level.as_struct()
    nw, nb, K, Cc, N = st.nw, st.nw * st.nf, st.K, st.C, st.N
    R = _chk(R, "R", (nb, 3, 3)); T = _chk(T, "T", (nb, 3, 1)); Wt = _chk(W, "W", (nw, K, 1))
    dc = _chk(dcost.reshape(-1), "dcost", (nb,))
    dev = R.device
    dconv1 = torch.empty(nw, N, Cc, device=dev); dconv2 = torch.empty(nb, st.h, st.w, st.conv2_channels, device=dev)
    dD = torch.empty(nw, N, 1, device=dev); dB = torch.empty(nw, N, K, device=dev)
    dR = torch.empty(nb, 3, 3, device=dev); dT = torch.empty(nb, 3, 1, device=dev); dW = torch.empty(nw, K, 1, device=dev)
    dweight = torch.empty(nb, N, 1, device=dev) if return_dweight else None
    check(lib.banet_lm_keyframe_cost_bwd(C.byref(st), R.data_ptr(), T.data_ptr(), Wt.data_ptr(), dc.data_ptr(), dconv1.data_ptr(),
                                         dconv2.data_ptr(), dD.data_ptr(), dB.data_ptr(), dR.data_ptr(), dT.data_ptr(), dW.data_ptr(),
                                         _ptr(dweight), _stream()), "banet_lm_keyframe_cost_bwd")
    out = (dconv1, dconv2, dD, dB, dR, dT, dW)
    return out + (dweight,) if return_dweight else out


def lm_keyframe_run(levels: Sequence[KeyframeLevel], iters_per_level: int, R: Tensor, T: Tensor, W: Tensor,
                    mlp_packed: Optional[Sequence[Optional[Tensor]]] = None, l2_regularizer_base: float = 1000.0,
                    lambda_fixed: float = -1.0, damping_eps: float = 1e-5, undamped_last: bool = True,
                    precision: int = _lib.PREC_AUTO, workspace: Optional[Tensor] = None):
    """Joint coarse-to-fine solve of nw keyframe windows with the keyframe tensors once per window (banet_lm_keyframe_run): per iteration
    one keyframe build and one window step.  R [nw*nf,3,3], T [nw*nf,3,1], W [nw,K,1].  Returns new (R, T, W [nw,K,1], status [nw*nf])."""
    lib = load()
    arr, mlp_ptrs, base, opts, nbytes, _keep = _prepare_run(levels, lib.banet_lm_keyframe_run_workspace_bytes, (int(precision),), mlp_packed,
                                                            l2_regularizer_base, damping_eps, undamped_last, False)
    # a query of 0 is left to the run, which names the fault: the query sets no message for levels that disagree
    nw, nb, K = arr[0].nw, arr[0].nw * arr[0].nf, arr[0].K
    R = _chk(R, "R", (nb, 3, 3)).clone(); T = _chk(T, "T", (nb, 3, 1)).clone(); Wt = _chk(W.reshape(nw, K, 1), "W", (nw, K, 1)).clone()
    ws = workspace if workspace is not None and workspace.numel() >= nbytes else _ws(nbytes, R.device)
    status = torch.empty(nb, device=R.device, dtype=torch.int32)
    check(lib.banet_lm_keyframe_run(arr, len(arr), int(iters_per_level), mlp_ptrs, base, float(lambda_fixed),
                                    C.byref(opts), int(precision), R.data_ptr(), T.data_ptr(), Wt.data_ptr(), status.data_ptr(), ws.data_ptr(),
                                    ws.numel(), _stream()), "banet_lm_keyframe_run")
    return R, T, Wt, status


class LMRunGraph:
    """`banet_lm_run` captured ONCE into a CUDA graph and replayed: the library call allocates nothing and never synchronises, so the whole
    coarse-to-fine loop (3 launches per LM iteration) is capturable as it is.  For small or sparse problems (the reference's 4096-point
    tracking mode, coarse levels), where launch gaps are a visible share of a solve (SURVEY.md section 8f-2).  Results are bit-identical to
    `lm_run`.  The level tensors, lambda-MLP weights and the workspace are baked into the graph by address: keep them alive and refill them in
    place between solves; `solve` copies the start iterate into the graph's static buffers and returns clones of the result."""

    def __init__(self, levels: Sequence[Level], iters_per_level: int, mlp_packed: Optional[Sequence[Optional[Tensor]]] = None,
                 l2_regularizer_base: Optional[float] = None, lambda_fixed: float = -1.0, damping_eps: float = 1e-5,
                 undamped_last: Optional[bool] = None, precision: int = _lib.PREC_AUTO):
        self._lib = load()
        (self._arr, self._mlp_ptrs, self._base, self._opts, nbytes, self._keep) = _prepare_run(
            levels, self._lib.banet_lm_run_workspace_bytes, (precision,), mlp_packed, l2_regularizer_base, damping_eps, undamped_last, False)
        if nbytes == 0:
            check(-4, "banet_lm_run_workspace_bytes")
        self.nb, self.K = self._arr[0].nb, self._arr[0].K
        self._iters, self._lambda_fixed, self._prec = int(iters_per_level), float(lambda_fixed), int(precision)
        dev = levels[0].conv1.device
        self.R = torch.zeros(self.nb, 3, 3, device=dev); self.T = torch.zeros(self.nb, 3, 1, device=dev)
        self.W = None if self.K == 0 else torch.zeros(self.nb, self.K, 1, device=dev)
        self.status = torch.zeros(self.nb, device=dev, dtype=torch.int32)
        self._ws = _ws(nbytes, dev)
        self.R.copy_(torch.eye(3, device=dev).expand(self.nb, 3, 3))
        side = torch.cuda.Stream(device=dev)                       # eager warm-up off the default stream (sets the kernels' attributes), then capture
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            self._launch()
        torch.cuda.current_stream(dev).wait_stream(side)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._launch()

    def _launch(self):
        check(self._lib.banet_lm_run(self._arr, len(self._arr), self._iters, self._mlp_ptrs, self._base, self._lambda_fixed, C.byref(self._opts),
                                     self._prec, self.R.data_ptr(), self.T.data_ptr(), _ptr(self.W), self.status.data_ptr(),
                                     self._ws.data_ptr(), self._ws.numel(), _stream()), "banet_lm_run")

    def solve(self, R: Tensor, T: Tensor, W: Optional[Tensor]):
        """-> new (R, T, W, status) like `lm_run`."""
        self.R.copy_(_chk(R, "R", (self.nb, 3, 3))); self.T.copy_(_chk(T, "T", (self.nb, 3, 1)))
        if self.K:
            self.W.copy_(_chk(W, "W", (self.nb, self.K, 1)))
        self.graph.replay()
        return self.R.clone(), self.T.clone(), None if self.W is None else self.W.clone(), self.status.clone()


def lm_run_workspace_bytes(levels: Sequence[Level], precision: int = _lib.PREC_AUTO) -> int:
    lib = load()
    structs = [lv.as_struct()[0] for lv in levels]
    arr = (BanetLevel * len(structs))(*structs)
    return int(lib.banet_lm_run_workspace_bytes(arr, len(structs), precision))


# ------------------------------------------------------------------------------------------ backward of one iteration
def lm_build_bwd(level: Level, R: Tensor, T: Tensor, W: Optional[Tensor], dH: Tensor, dg: Tensor, drbar_sum: Tensor, exact_sym: bool = False,
                 return_dweight: bool = False):
    """Backward of lm_build (banet_lm_build_bwd) -> dconv1, dconv2, dD, dB, dR, dT, dW.  dconv2 has conv2's layout: [nb,h,w,3C] for
    [F2|gx|gy], [nb,h,w,C] for F2 only (the adjoint of the on-the-fly gradient stencil is applied inside the kernel).  dconv1 and dconv2
    are float32 also for bfloat16 features (the kernel accumulates them with fp32 atomics), and dB is float32 also for a bfloat16 basis.
    On a weighted level every gradient carries the point weights.  return_dweight=True appends dweight [nb,N,1] = <dH, H_n> + <dg, g_n>
    (banet_lm_build_bwd_weighted; on an unweighted level, the gradient at weights of ones)."""
    lib = load()
    st, keep = level.as_struct()
    nb, K, Cc, N = st.nb, st.K, st.C, st.N
    P = 6 + K
    R = _chk(R, "R", (nb, 3, 3)); T = _chk(T, "T", (nb, 3, 1))
    Wt = None if K == 0 else _chk(W, "W", (nb, K, 1))
    dH = _chk(dH, "dH", (nb, P, P)); dg = _chk(dg.reshape(nb, P), "dg", (nb, P)); dr = _chk(drbar_sum, "drbar_sum", (nb, Cc))
    dev = R.device
    dconv1 = torch.empty(nb, N, Cc, device=dev); dconv2 = torch.empty(nb, st.h, st.w, st.conv2_channels, device=dev)
    dD = torch.empty(nb, N, 1, device=dev); dB = None if K == 0 else torch.empty(nb, N, K, device=dev)
    dR = torch.empty(nb, 3, 3, device=dev); dT = torch.empty(nb, 3, 1, device=dev); dW = None if K == 0 else torch.empty(nb, K, 1, device=dev)
    if not return_dweight:
        check(lib.banet_lm_build_bwd(C.byref(st), R.data_ptr(), T.data_ptr(), _ptr(Wt), dH.data_ptr(), dg.data_ptr(), dr.data_ptr(), int(bool(exact_sym)),
                                     dconv1.data_ptr(), dconv2.data_ptr(), dD.data_ptr(), _ptr(dB), dR.data_ptr(), dT.data_ptr(), _ptr(dW), _stream()),
              "banet_lm_build_bwd")
        return dconv1, dconv2, dD, dB, dR, dT, dW
    dweight = torch.empty(nb, N, 1, device=dev)
    check(lib.banet_lm_build_bwd_weighted(C.byref(st), R.data_ptr(), T.data_ptr(), _ptr(Wt), dH.data_ptr(), dg.data_ptr(), dr.data_ptr(),
                                          int(bool(exact_sym)), dconv1.data_ptr(), dconv2.data_ptr(), dD.data_ptr(), _ptr(dB), dR.data_ptr(),
                                          dT.data_ptr(), _ptr(dW), dweight.data_ptr(), _stream()),
          "banet_lm_build_bwd_weighted")
    return dconv1, dconv2, dD, dB, dR, dT, dW, dweight


def lm_solve_update_bwd(H: Tensor, g: Tensor, lam: Tensor, delta: Tensor, R: Tensor, T: Tensor, dRn: Tensor, dTn: Tensor, dWn: Optional[Tensor],
                        damping_eps: float = 1e-5, undamped_last: bool = True):
    """Backward of lm_solve_update (banet_lm_solve_update_bwd) -> dH, dg, dlambda, dR, dT, dW."""
    lib = load()
    Hc = _chk(H, "H"); nb, P, _ = Hc.shape
    K = P - 6
    gc = _chk(g.reshape(nb, P), "g", (nb, P)); lc = _chk(lam.reshape(nb), "lambda", (nb,)); dl = _chk(delta, "delta", (nb, P))
    R = _chk(R, "R", (nb, 3, 3)); T = _chk(T, "T", (nb, 3, 1))
    gR = _chk(dRn, "dR_out", (nb, 3, 3)); gT = _chk(dTn, "dT_out", (nb, 3, 1)); gW = None if K == 0 else _chk(dWn, "dW_out", (nb, K, 1))
    dev = Hc.device
    dH = torch.empty(nb, P, P, device=dev); dg = torch.empty(nb, P, device=dev); dlam = torch.empty(nb, device=dev)
    dR = torch.empty(nb, 3, 3, device=dev); dT = torch.empty(nb, 3, 1, device=dev); dW = None if K == 0 else torch.empty(nb, K, 1, device=dev)
    opts = BanetSolveOpts(float(damping_eps), int(undamped_last), 0)
    check(lib.banet_lm_solve_update_bwd(Hc.data_ptr(), gc.data_ptr(), lc.data_ptr(), dl.data_ptr(), nb, K, C.byref(opts), R.data_ptr(), T.data_ptr(),
                                        gR.data_ptr(), gT.data_ptr(), _ptr(gW), dH.data_ptr(), dg.data_ptr(), dlam.data_ptr(), dR.data_ptr(),
                                        dT.data_ptr(), _ptr(dW), _stream()), "banet_lm_solve_update_bwd")
    return dH, dg, dlam, dR, dT, dW


def lm_step_bwd(H: Tensor, g: Tensor, rbar_sum: Optional[Tensor], N: int, mlp_packed: Optional[Tensor], lam: Tensor, delta: Tensor, R: Tensor,
                T: Tensor, dRn: Tensor, dTn: Tensor, dWn: Optional[Tensor], damping_eps: float = 1e-5, undamped_last: Optional[bool] = None,
                base: float = 1000.0, workspace: Optional[Tensor] = None):
    """Backward of lm_step (banet_lm_step_bwd).  lam, delta: the lambda and delta lm_step returned; rbar_sum, N as given to lm_step (rbar_sum
    also sets the storage plan when lambda was given, as in the forward).  -> dH [nb,P,P], dg [nb,P], drbar_sum [nb,C] (None without the MLP),
    dmlp (packed like mlp_packed; None without it), dlambda [nb], dR, dT, dW.  workspace: a uint8 buffer to use when it is large enough."""
    lib = load()
    Hc = _chk(H, "H"); nb, P, _ = Hc.shape
    K = P - 6
    if undamped_last is None:
        undamped_last = K > 0
    gc = _chk(g.reshape(nb, P), "g", (nb, P)); lc = _chk(lam.reshape(nb), "lambda", (nb,)); dl = _chk(delta, "delta", (nb, P))
    rb = None if rbar_sum is None else _chk(rbar_sum, "rbar_sum"); mp = None if mlp_packed is None else _chk(mlp_packed, "mlp_packed")
    Cc = 1 if rb is None else rb.shape[1]
    R = _chk(R, "R", (nb, 3, 3)); T = _chk(T, "T", (nb, 3, 1))
    gR = _chk(dRn, "dR_out", (nb, 3, 3)); gT = _chk(dTn, "dT_out", (nb, 3, 1)); gW = None if K == 0 else _chk(dWn, "dW_out", (nb, K, 1))
    dev = Hc.device
    dH = torch.empty(nb, P, P, device=dev); dg = torch.empty(nb, P, device=dev); dlam = torch.empty(nb, device=dev)
    dR = torch.empty(nb, 3, 3, device=dev); dT = torch.empty(nb, 3, 1, device=dev); dW = None if K == 0 else torch.empty(nb, K, 1, device=dev)
    drb = None if mp is None else torch.empty(nb, Cc, device=dev)
    dmlp = None if mp is None else torch.empty_like(mp)
    ws = None
    if mp is not None:
        if mp.numel() != lib.banet_mlp_param_count(Cc):
            raise _lib.BanetError(f"mlp_packed has {mp.numel()} params, expected {lib.banet_mlp_param_count(Cc)} for C={Cc}")
        nbytes = lib.banet_lm_step_bwd_workspace_bytes(nb, Cc, K)
        ws = workspace if workspace is not None and workspace.numel() >= nbytes else _ws(nbytes, dev)
    opts = BanetSolveOpts(float(damping_eps), int(undamped_last), 0)
    check(lib.banet_lm_step_bwd(Hc.data_ptr(), gc.data_ptr(), _ptr(rb), nb, int(N), Cc, K, _ptr(mp), float(base), lc.data_ptr(), dl.data_ptr(),
                                C.byref(opts), R.data_ptr(), T.data_ptr(), gR.data_ptr(), gT.data_ptr(), _ptr(gW), dH.data_ptr(), dg.data_ptr(),
                                _ptr(drb), _ptr(dmlp), dlam.data_ptr(), dR.data_ptr(), dT.data_ptr(), _ptr(dW), _ptr(ws),
                                0 if ws is None else ws.numel(), _stream()), "banet_lm_step_bwd")
    return dH, dg, drb, dmlp, dlam, dR, dT, dW


def lm_step_supported(nb: int, C: int, K: int) -> bool:
    """Whether banet_lm_step and its backward take K depth bases at MLP width C (C = 1 when lambda is given without rbar_sum)."""
    return load().banet_lm_step_bwd_workspace_bytes(int(nb), int(C), int(K)) > 0


def lm_window_solve_update_bwd(H: Tensor, g: Tensor, lam: Tensor, delta: Tensor, R: Tensor, T: Tensor, dRn: Tensor, dTn: Tensor, dWn: Tensor,
                               damping_eps: float = 1e-5, undamped_last: bool = True):
    """Backward of lm_window_solve_update (banet_lm_window_solve_update_bwd) -> dH [nf,P,P], dg [nf,P], dlambda [1], dR, dT, dW [K,1]."""
    lib = load()
    Hc = _chk(H, "H"); nf, P, _ = Hc.shape
    K = P - 6
    gc = _chk(g.reshape(nf, P), "g", (nf, P)); lc = _chk(lam.reshape(1), "lambda", (1,)); dl = _chk(delta, "delta", (6 * nf + K,))
    R = _chk(R, "R", (nf, 3, 3)); T = _chk(T, "T", (nf, 3, 1))
    gR = _chk(dRn, "dR_out", (nf, 3, 3)); gT = _chk(dTn, "dT_out", (nf, 3, 1)); gW = _chk(dWn.reshape(K, 1), "dW_out", (K, 1))
    dev = Hc.device
    dH = torch.empty(nf, P, P, device=dev); dg = torch.empty(nf, P, device=dev); dlam = torch.empty(1, device=dev)
    dR = torch.empty(nf, 3, 3, device=dev); dT = torch.empty(nf, 3, 1, device=dev); dW = torch.empty(K, 1, device=dev)
    opts = BanetSolveOpts(float(damping_eps), int(undamped_last), 0)
    ws = _ws(lib.banet_lm_window_solve_update_bwd_workspace_bytes(nf, K), dev)
    check(lib.banet_lm_window_solve_update_bwd(Hc.data_ptr(), gc.data_ptr(), lc.data_ptr(), dl.data_ptr(), nf, K, C.byref(opts), R.data_ptr(), T.data_ptr(),
                                               gR.data_ptr(), gT.data_ptr(), gW.data_ptr(), dH.data_ptr(), dg.data_ptr(), dlam.data_ptr(), dR.data_ptr(),
                                               dT.data_ptr(), dW.data_ptr(), ws.data_ptr(), ws.numel(), _stream()), "banet_lm_window_solve_update_bwd")
    return dH, dg, dlam, dR, dT, dW


def lm_window_batch_solve_update_bwd(H: Tensor, g: Tensor, lam: Tensor, delta: Tensor, R: Tensor, T: Tensor, dRn: Tensor, dTn: Tensor, dWn: Tensor,
                                     damping_eps: float = 1e-5, undamped_last: bool = True):
    """Backward of lm_window_batch_solve_update (banet_lm_window_batch_solve_update_bwd) -> dH [nw*nf,P,P], dg [nw*nf,P], dlambda [nw],
    dR, dT, dW [nw,K,1]."""
    lib = load()
    Hc = _chk(H, "H"); nb, P, _ = Hc.shape
    K = P - 6
    nw = lam.numel()
    if nw == 0 or nb % nw:
        raise _lib.BanetError(f"lambda has {nw} windows, which does not divide the {nb} pairs")
    nf = nb // nw
    gc = _chk(g.reshape(nb, P), "g", (nb, P)); lc = _chk(lam.reshape(nw), "lambda", (nw,)); dl = _chk(delta, "delta", (nw, 6 * nf + K))
    R = _chk(R, "R", (nb, 3, 3)); T = _chk(T, "T", (nb, 3, 1))
    gR = _chk(dRn, "dR_out", (nb, 3, 3)); gT = _chk(dTn, "dT_out", (nb, 3, 1)); gW = _chk(dWn.reshape(nw, K, 1), "dW_out", (nw, K, 1))
    dev = Hc.device
    dH = torch.empty(nb, P, P, device=dev); dg = torch.empty(nb, P, device=dev); dlam = torch.empty(nw, device=dev)
    dR = torch.empty(nb, 3, 3, device=dev); dT = torch.empty(nb, 3, 1, device=dev); dW = torch.empty(nw, K, 1, device=dev)
    opts = BanetSolveOpts(float(damping_eps), int(undamped_last), 0)
    ws = _ws(lib.banet_lm_window_batch_solve_update_bwd_workspace_bytes(nw, nf, K), dev)
    check(lib.banet_lm_window_batch_solve_update_bwd(Hc.data_ptr(), gc.data_ptr(), lc.data_ptr(), dl.data_ptr(), nw, nf, K, C.byref(opts), R.data_ptr(),
                                                     T.data_ptr(), gR.data_ptr(), gT.data_ptr(), gW.data_ptr(), dH.data_ptr(), dg.data_ptr(),
                                                     dlam.data_ptr(), dR.data_ptr(), dT.data_ptr(), dW.data_ptr(), ws.data_ptr(), ws.numel(), _stream()),
          "banet_lm_window_batch_solve_update_bwd")
    return dH, dg, dlam, dR, dT, dW


def grad_fixed_concat_bwd(dconv2: Tensor, swap_halves: bool = False) -> Tensor:
    lib = load()
    g = _chk(dconv2, "dconv2"); nb, h, w, c3 = g.shape
    dF = torch.empty(nb, h, w, c3 // 3, device=g.device)
    check(lib.banet_grad_fixed_concat_bwd(g.data_ptr(), nb, h, w, c3 // 3, int(swap_halves), dF.data_ptr(), _stream()), "banet_grad_fixed_concat_bwd")
    return dF


def resample_bwd(dout: Tensor, xy: Tensor, coord_scale: float, h: int, w: int) -> Tensor:
    lib = load()
    g = _chk(dout, "dout"); nb, N, Cc = g.shape
    pts = _chk(xy, "xy", (nb, N, 2))
    dd = torch.empty(nb, h, w, Cc, device=g.device)
    check(lib.banet_resample_bwd(g.data_ptr(), pts.data_ptr(), float(coord_scale), nb, h, w, Cc, N, dd.data_ptr(), _stream()), "banet_resample_bwd")
    return dd


def depth_compose_bwd(dout: Tensor, basis: Tensor, W: Tensor):
    """-> dbasis [nb,M,K], dW [nb,K,1], both float32 (also for a bfloat16 basis: banet_depth_compose_bwd_bf16)."""
    lib = load()
    bs = _chk(basis, "basis", features=True); nb, M, K = bs.shape
    g = _chk(dout, "dout", (nb, M)); Wt = _chk(W, "W", (nb, K, 1))
    dbasis = torch.empty(nb, M, K, device=bs.device); dW = torch.empty(nb, K, 1, device=bs.device)
    name = "banet_depth_compose_bwd_bf16" if bs.dtype == torch.bfloat16 else "banet_depth_compose_bwd"
    check(getattr(lib, name)(g.data_ptr(), bs.data_ptr(), Wt.data_ptr(), nb, M, K, dbasis.data_ptr(), dW.data_ptr(), _stream()), name)
    return dbasis, dW


# ------------------------------------------------------------------------------------------ legacy tracker loop
def lm_track_legacy(levels: Sequence[Level], level_iters: Sequence[int], R: Tensor, T: Tensor, mlp_packed: Optional[Sequence[Optional[Tensor]]] = None,
                    early_termination: bool = True, angle_change: float = 0.002 * (3.14 / 180.0), translation_change: float = 0.0002,
                    residual_ratio: float = 1.0):
    """banet_lm_track_legacy (legacy/ba.py:83-145 on the device) -> R, T, iters_done [nlevels,nb], valid_ratio [nb], status [nb]."""
    lib = load()
    structs, keep = [], []
    for lv in levels:
        s, k = lv.as_struct(); structs.append(s); keep.append(k)
    arr = (BanetLevel * len(structs))(*structs)
    nb = structs[0].nb
    R = _chk(R, "R", (nb, 3, 3)).clone(); T = _chk(T, "T", (nb, 3, 1)).clone()
    iters = (C.c_int * len(structs))(*[int(i) for i in level_iters])
    mlp_ptrs = (C.c_void_p * len(structs))()
    for i in range(len(structs)):
        m = None if mlp_packed is None else mlp_packed[i]
        if m is not None:
            m = _chk(m, "mlp_packed"); keep.append(m)
        mlp_ptrs[i] = None if m is None else m.data_ptr()
    opts = _lib.BanetLegacyOpts(int(early_termination), float(angle_change), float(translation_change), float(residual_ratio))
    nbytes = lib.banet_lm_track_legacy_workspace_bytes(arr, len(structs))
    if nbytes == 0:
        check(-1, "banet_lm_track_legacy_workspace_bytes")
    ws = _ws(nbytes, R.device)
    done = torch.zeros(len(structs), nb, device=R.device, dtype=torch.int32)
    ratio = torch.zeros(nb, device=R.device); status = torch.empty(nb, device=R.device, dtype=torch.int32)
    check(lib.banet_lm_track_legacy(arr, len(structs), iters, mlp_ptrs, C.byref(opts), R.data_ptr(), T.data_ptr(), done.data_ptr(), ratio.data_ptr(),
                                    status.data_ptr(), ws.data_ptr(), ws.numel(), _stream()), "banet_lm_track_legacy")
    return R, T, done, ratio, status
