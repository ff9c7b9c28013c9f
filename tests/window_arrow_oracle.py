"""Float64 statement of the block-arrow window step (banet_lm_window_batch_*): the per-frame pose blocks eliminated by a Schur complement,
the K x K depth system factored, the pose steps back-substituted.  tests/test_window_batch.py proves it equal to the dense solve of the
assembled window system (oracle.window_assemble), values and gradients, and the GPU kernels are checked against the oracle's iteration."""
import torch


def window_arrow_solve(H, g, lam, damping_eps: float = 1e-5, undamped_last: bool = True):
    """H [nf,P,P], g [nf,P,1] (one window's per-pair normal equations, P = 6 + K), lam scalar -> the window's step [6 nf + K, 1] (frame f's
    pose at 6f, the depth at 6 nf).  Damping as bundlenet.py:264-266 on the joint system: lam (diag + eps) on every pose diagonal and on the
    frame-summed depth diagonal, except the last depth coefficient when undamped_last."""
    nf, P, _ = H.shape
    K = P - 6
    Hcc, Hcd, Hdd = H[:, :6, :6], H[:, :6, 6:], H[:, 6:, 6:]
    gc, gd = g[:, :6], g[:, 6:]
    Acc = Hcc + torch.diag_embed((torch.diagonal(Hcc, dim1=-2, dim2=-1) + damping_eps) * lam)        # damped 6x6 per frame
    Dsum = Hdd.sum(0)
    ddamp = (torch.diagonal(Dsum) + damping_eps) * lam
    if undamped_last:
        ddamp = torch.cat([ddamp[:-1], torch.zeros(1, dtype=H.dtype)])
    L = torch.linalg.cholesky(Acc)                                                                   # Acc_f = L_f L_f^T
    Y = torch.linalg.solve_triangular(L, Hcd, upper=False)                                           # Y_f = L_f^-1 Hcd_f      [nf,6,K]
    z = torch.linalg.solve_triangular(L, gc, upper=False)                                            # z_f = L_f^-1 g_f        [nf,6,1]
    S = Dsum + torch.diag(ddamp) - (Y.transpose(1, 2) @ Y).sum(0)                                    # Schur complement       [K,K]
    r = gd.sum(0) - (Y.transpose(1, 2) @ z).sum(0)
    xd = torch.cholesky_solve(r, torch.linalg.cholesky(S))
    xf = torch.cholesky_solve(gc - Hcd @ xd, L)                                                      # x_f = Acc_f^-1 (g_f - Hcd_f x_d)
    return torch.cat([xf.reshape(6 * nf, 1), xd], 0)
