"""Float64 statement of the point-weighted iteration: every point n of a pair adds w_n J_n^T M_n J_n to H and w_n J_n^T q_n to g
(M_n = G_n^T G_n, q_n = G_n^T d_n, the block form of DESIGN.md §2), while the mean |residual| that drives lambda and the in-bounds count
stay unweighted.  Built on the oracle's own warp, sampler and Jacobians (oracle/ba_oracle.py), without changing them:
tests/test_point_weights.py ties it to oracle.bundle_iteration / camera_iteration with weights of ones.  Differentiable by float64 autograd
in every input, the weight included."""
import torch

from oracle import ba_oracle as O


def _point_system(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, guard_nonfinite):
    """J [nb,N,2,P] (zero at masked points), M [nb,N,2,2], q [nb,N,2,1], diff [nb,N,C,1], mask [nb,N]."""
    Dt = D if B is None else D + B @ W
    Rp, x, y, Z, px, py = O._warp(p, Dt, R, T, fx, fy, ox, oy)
    diff, grad, m = O._sample_diff_grad(conv1, conv2, px, py, guard_nonfinite)
    J = O.camera_jacobian_matrix(x, y, Z, fx, fy)                                         # [nb,N,2,6]
    if B is not None:
        jd = O.depth_jacobian_matrix(Rp[:, 0:1], Rp[:, 1:2], Rp[:, 2:3], x, y, Z, fx, fy)  # [nb,N,2]
        J = torch.cat([J, jd.unsqueeze(-1) * B.unsqueeze(-2)], dim=-1)                    # [nb,N,2,6+K]
    J = torch.where(m > 0, J, torch.zeros_like(J))                                        # masked points contribute nothing
    M = grad.transpose(-1, -2) @ grad
    q = grad.transpose(-1, -2) @ diff
    return J, M, q, diff, m.reshape(m.shape[0], m.shape[1])


def point_terms(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, guard_nonfinite: bool = True):
    """Per-point unweighted contributions H_n [nb,N,P,P] and g_n [nb,N,P] (small N only)."""
    J, M, q, _, _ = _point_system(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, guard_nonfinite)
    return J.transpose(-1, -2) @ M @ J, (J.transpose(-1, -2) @ q).squeeze(-1)


def normal_equations(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, weight=None, guard_nonfinite: bool = True, chunk: int = 32768):
    """H [nb,P,P], g [nb,P,1], rbar [nb,1,C] (unweighted mean |diff|), nvalid [nb] (unweighted); weight [nb,N,1] or None (= ones).
    Summed over point chunks (bounded memory)."""
    nb, N, C = conv1.shape
    H = g = None
    rsum = torch.zeros(nb, 1, C, dtype=conv1.dtype)
    nvalid = torch.zeros(nb, dtype=conv1.dtype)
    for a in range(0, N, chunk):
        b = min(N, a + chunk)
        J, M, q, diff, m = _point_system(conv1[:, a:b], conv2, fx[:, a:b], fy[:, a:b], ox[:, a:b], oy[:, a:b], p[:, :, a:b], D[:, a:b],
                                         None if B is None else B[:, a:b], R, T, W, guard_nonfinite)
        MJ, qv = M @ J, q.squeeze(-1)
        if weight is not None:
            w = weight[:, a:b].reshape(nb, b - a)
            MJ, qv = MJ * w[..., None, None], qv * w[..., None]
        Hc = torch.einsum("bnip,bniq->bpq", J, MJ)
        gc = torch.einsum("bnip,bni->bp", J, qv).unsqueeze(-1)
        H = Hc if H is None else H + Hc
        g = gc if g is None else g + gc
        rsum = rsum + diff.squeeze(-1).abs().sum(dim=1, keepdim=True)
        nvalid = nvalid + m.sum(1)
    return H, g, rsum / float(N), nvalid


def iteration(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, mlp_params, weight=None, opts: O.IterOptions = O.IterOptions()):
    """oracle.bundle_iteration (B given) / camera_iteration (B None) with the weighted normal equations -> (R', T', W' or None)."""
    nb = conv1.shape[0]
    bundle = B is not None
    H, g, rbar, _ = normal_equations(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, weight, opts.guard_nonfinite)
    if opts.lambda_override is not None:
        lam = opts.lambda_override.reshape(-1, 1, 1).to(conv1.dtype)
    else:
        lam = torch.pow(torch.linalg.norm(rbar, dim=-1, keepdim=True), 2.0 + O.lambda_mlp(rbar, mlp_params))
        if bundle and opts.l2_regularizer_base is not None:
            lam = opts.l2_regularizer_base * lam
    diag = torch.diagonal(H, dim1=-2, dim2=-1)
    if bundle and opts.undamped_last:
        dvec = torch.cat([diag[:, :-1] + opts.damping_eps, torch.zeros(nb, 1, dtype=diag.dtype)], dim=-1)
    else:
        dvec = diag + opts.damping_eps
    sol = torch.linalg.solve(H + torch.diag_embed(dvec * lam.reshape(nb, 1)), g)
    Rn, Tn = O._update(sol[:, :6, :], R, T, opts)
    return Rn, Tn, (W + sol[:, 6:, :]) if bundle else None


def solve(levels, weights, iters_per_level: int, R, T, W, opts: O.IterOptions = O.IterOptions()):
    """Coarse-to-fine: `iters_per_level` weighted iterations per level (oracle.LevelInputs, its own lambda-MLP), W carried across levels."""
    for lv, wt in zip(levels, weights):
        for _ in range(iters_per_level):
            R, T, W = iteration(lv.conv1, lv.conv2, lv.fx, lv.fy, lv.ox, lv.oy, lv.p, lv.D, lv.B, R, T, W, lv.mlp, wt, opts)
    return R, T, W
