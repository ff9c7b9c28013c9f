"""Float64 statement of the point-weighted keyframe window: every pair (keyframe -> frame f) builds its weighted normal equations
(weighted_oracle.normal_equations, the window's W broadcast to the frames, one weight per (frame, keyframe point)), the window's block-arrow
system is assembled from them (oracle.window_assemble), and oracle.window_iteration's damping, solve and update follow.  The mean |residual|
that drives lambda stays unweighted.  A weighted window_resize (the schedule of window_resize_oracle.window_resize) is stated on it.
tests/test_window_weights.py ties both to the oracle with weights of ones.  Differentiable by float64 autograd in every input."""
import torch

from oracle import ba_oracle as O
import weighted_oracle as WO


def window_system(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, weight=None, guard_nonfinite: bool = True):
    """One window of nf pairs (the keyframe tensors per frame, [nf,...]), W [K,1] shared, weight [nf,N,1] or None (= ones) ->
    per-pair H [nf,P,P], g [nf,P,1], rbar [nf,1,C] (unweighted), and the assembled Hj [Pj,Pj], gj [Pj,1] (Pj = 6 nf + K)."""
    nf = conv1.shape[0]
    K = B.shape[-1]
    H, g, rbar, _ = WO.normal_equations(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W.reshape(1, K, 1).expand(nf, K, 1), weight, guard_nonfinite)
    Hj, gj = O.window_assemble(H, g)
    return H, g, rbar, Hj, gj


def window_iteration(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, mlp_params, weight=None, opts: O.IterOptions = O.IterOptions()):
    """oracle.window_iteration with the weighted per-pair normal equations -> (R' [nf,3,3], T' [nf,3,1], W' [K,1])."""
    nf = conv1.shape[0]
    K = B.shape[-1]
    _, _, rbar, Hj, gj = window_system(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, weight, opts.guard_nonfinite)
    avg = rbar.mean(dim=0, keepdim=True)                              # every frame has N points: mean over all nf * N
    if opts.lambda_override is not None:
        lam = opts.lambda_override.reshape(-1)[0].to(conv1.dtype)
    else:
        lam = torch.pow(torch.linalg.norm(avg, dim=-1, keepdim=True), 2.0 + O.lambda_mlp(avg, mlp_params)).reshape(())
        if opts.l2_regularizer_base is not None:
            lam = opts.l2_regularizer_base * lam
    diag = torch.diagonal(Hj)
    dvec = diag + opts.damping_eps
    if opts.undamped_last:
        dvec = torch.cat([dvec[:-1], torch.zeros(1, dtype=diag.dtype)])
    sol = torch.linalg.solve(Hj + torch.diag(dvec * lam), gj)
    Rn, Tn = O._update(sol[:6 * nf].reshape(nf, 6, 1), R, T, opts)
    return Rn, Tn, W.reshape(K, 1) + sol[6 * nf:]


def window_solve(levels, weights, iters_per_level: int, R, T, W, opts: O.IterOptions = O.IterOptions()):
    """Coarse-to-fine loop of the weighted window_iteration over oracle.LevelInputs (nb = nf pairs per level); weights[l] [nf,N_l,1]."""
    for lv, wt in zip(levels, weights):
        for _ in range(iters_per_level):
            R, T, W = window_iteration(lv.conv1, lv.conv2, lv.fx, lv.fy, lv.ox, lv.oy, lv.p, lv.D, lv.B, R, T, W, lv.mlp, wt, opts)
    return R, T, W


def window_resize(intrisic, key_layers, frame_layers, points, basis, init_depth, mlp_params_by_level, init_rotation=None, init_translation=None,
                  weight=None, opts: O.IterOptions = O.IterOptions(), geo: O.ResizeGeometry = O.ResizeGeometry()):
    """window_resize_oracle.window_resize with the weighted window_iteration; weight [nw,nf|1,N,1] (at `points`, the same at both levels)
    or None."""
    nw, nf = frame_layers[-1].shape[0], frame_layers[-1].shape[1]
    K = basis.shape[-1]
    _points, sfx, sfy, sox, soy = O._prepare(intrisic, points, geo)     # :338-339, :354-357
    d = O.resampler(init_depth.detach(), _points / 2)                    # :341-343
    b = O.resampler(basis, _points / 2)                                  # :344
    p = O.compute_coordinates(_points, sfx, sfy, sox, soy)              # :358
    dt = frame_layers[-1].dtype
    R = torch.eye(3, dtype=dt).repeat(nw, nf, 1, 1) if init_rotation is None else init_rotation
    T = torch.zeros(nw, nf, 3, 1, dtype=dt) if init_translation is None else init_translation
    W = [torch.zeros(K, 1, dtype=dt) for _ in range(nw)]
    Rs, Ts, Ds = [], [], []
    for level in range(2, 4):                                            # :376
        scale = 2 ** (3 - level)
        fx, fy, ox, oy = sfx / scale, sfy / scale, sox / scale, soy / scale
        layer1 = O.resampler(key_layers[level], _points / scale)        # :385
        Rl, Tl = [], []
        for w in range(nw):
            F2 = frame_layers[level][w]
            layer2 = torch.cat([F2, O.grad_fixed(F2)], dim=-1)           # :388-389, per frame
            kf = lambda t: t[w:w + 1].expand(nf, *t.shape[1:])          # the keyframe's tensors, the same for every frame
            wt = None if weight is None else weight[w].expand(nf, *weight.shape[2:])
            Rn, Tn, W[w] = window_iteration(kf(layer1), layer2, kf(fx), kf(fy), kf(ox), kf(oy), kf(p), kf(d), kf(b), R[w], T[w], W[w],
                                            mlp_params_by_level[str(level)], wt, opts)   # :391-393
            Rl.append(Rn); Tl.append(Tn)
        R, T = torch.stack(Rl), torch.stack(Tl)
        Rs.append(R); Ts.append(T)
        Wb = torch.stack(W)                                              # [nw,K,1]
        Ds.append(init_depth + (basis.reshape(nw, -1, K) @ Wb).reshape(nw, geo.out_hw[0], geo.out_hw[1], 1))   # :397
    return Rs, Ts, Ds
