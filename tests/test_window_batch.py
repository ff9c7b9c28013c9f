"""Batches of keyframe windows (banet_lm_window_batch_*, autograd.window_batch_iteration_fused, BundleNet.WindowIteration on [nw,nf,...]):
the block-arrow elimination is proved equal to the dense window solve on the CPU (values and gradients, float64); on the GPU the new entries
are compared with the single-window entries, with the float64 oracle (a loop of window_iteration over the windows) and with themselves
(windows independent, bit-reproducible), including windows the dense single-window solve rejects."""
import ctypes

import pytest
import torch

from helpers import O, scene_case, oracle_level_inputs, mlp_for, rel_fro, to_cuda32
from window_arrow_oracle import window_arrow_solve


def _opts(**kw):
    from banet_b200._lib import BanetSolveOpts
    return BanetSolveOpts(kw.get("eps", 1e-5), kw.get("undamped_last", 1), kw.get("scramble", 0))


# ------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("nf,K,undamped_last", [(1, 5, True), (3, 5, True), (4, 9, False)])
def test_arrow_elimination_is_the_dense_window_solve(nf, K, undamped_last):
    sc = scene_case(nb=nf, H=24, W=32, C=3, K=K, level_ids=(3,), seed=17 + nf, shared_depth=True)
    a = oracle_level_inputs(sc.levels[0])
    W = (sc.W_true[0] * 0.5).expand(nf, K, 1)
    H, g, _, _ = O.normal_equations_structured(a["conv1"], a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"], sc.R0, sc.T0, W)
    gen = torch.Generator().manual_seed(nf)
    c = torch.randn(6 * nf + K, 1, generator=gen, dtype=torch.float64)
    M = H.clone().requires_grad_(); gg = g.clone().requires_grad_(); lam = torch.tensor(0.3, dtype=torch.float64, requires_grad=True)
    eps = 1e-5

    def dense(M, gg, lam):
        Hj, gj = O.window_assemble(0.5 * (M + M.transpose(1, 2)), gg)
        dvec = torch.diagonal(Hj) + eps
        if undamped_last:
            dvec = torch.cat([dvec[:-1], torch.zeros(1, dtype=dvec.dtype)])
        return torch.linalg.solve(Hj + torch.diag(dvec * lam), gj)

    def arrow(M, gg, lam):                                           # H enters through its symmetric part in both
        return window_arrow_solve(0.5 * (M + M.transpose(1, 2)), gg, lam, eps, undamped_last)

    xd, xa = dense(M, gg, lam), arrow(M, gg, lam)
    assert rel_fro(xa, xd) < 1e-12
    gd = torch.autograd.grad((xd * c).sum(), (M, gg, lam))
    ga = torch.autograd.grad((xa * c).sum(), (M, gg, lam))
    for name, u, v in zip(("H", "g", "lambda"), ga, gd):
        assert rel_fro(u, v) < 1e-12, name


def test_window_batch_entries_reject_bad_arguments_without_gpu():
    from banet_b200 import _lib
    lib = _lib.load()
    opts = _opts()
    p = 1                                                            # non-null dummy pointers: every check below fires before a CUDA call
    fwd = lambda nw, nf, K, o=opts, H=p, ws=p, nbytes=1 << 30: lib.banet_lm_window_batch_solve_update(
        H, p, p, nw, nf, K, ctypes.byref(o), p, p, p, p, p, p, p, p, ws, nbytes, None)
    bwd = lambda nw, nf, K, o=opts, H=p, ws=p, nbytes=1 << 30: lib.banet_lm_window_batch_solve_update_bwd(
        H, p, p, p, nw, nf, K, ctypes.byref(o), p, p, p, p, p, p, p, p, p, p, p, ws, nbytes, None)
    for call in (fwd, bwd):
        assert call(2, 4, 128, H=None) == -1 and b"null" in lib.banet_last_error()
        assert call(0, 4, 128) == -1 and call(2, 0, 128) == -1 and call(2, 4, 0) == -1
        assert call(2, 4, 128, o=_opts(scramble=1)) == -1
        assert call(2, 4, 257) == -4 and b"K=257" in lib.banet_last_error()
        assert call(2, 4, 128, ws=None) == -2
        assert call(2, 4, 128, nbytes=16) == -2
    assert lib.banet_lm_window_batch_solve_update_workspace_bytes(2, 4, 128) > 0
    assert lib.banet_lm_window_batch_solve_update_workspace_bytes(0, 4, 128) == 0 and lib.banet_lm_window_batch_solve_update_bwd_workspace_bytes(2, 4, 0) == 0

    lv = _lib.BanetLevel(8, 4096, 64, 128, 120, 160, 192, 1, 1, 1, 1, 1, 1, 0, 0)          # nb = 8 pairs
    arr = (_lib.BanetLevel * 1)(lv)
    run = lambda nw, o=opts, R=p, ws=p, nbytes=1 << 34, lvs=arr: lib.banet_lm_window_batch_run(lvs, 1, nw, 1, None, 1000.0, 0.5, ctypes.byref(o), 0,
                                                                                               R, p, p, p, ws, nbytes, None)
    assert run(2, R=None) == -1 and b"null" in lib.banet_last_error()
    assert run(0) == -1
    assert run(3) == -1 and b"nw * nf" in lib.banet_last_error()                               # 8 pairs are not 3 windows
    assert run(2, o=_opts(scramble=1)) == -1
    assert run(2, ws=None) == -2 and run(2, nbytes=16) == -2
    big = (_lib.BanetLevel * 1)(_lib.BanetLevel(8, 4096, 64, 300, 120, 160, 192, 1, 1, 1, 1, 1, 1, 0, 0))
    assert run(2, lvs=big) == -4
    assert lib.banet_lm_window_batch_run_workspace_bytes(arr, 1, 2, 0) > 0
    assert lib.banet_lm_window_batch_run_workspace_bytes(arr, 1, 3, 0) == 0


# ------------------------------------------------------------------------------------------ GPU
def _batch_scene(nw, nf, C, K, seed=83, n_points=400, H=48, W=64, level_ids=(3,), dtype=torch.float32):
    return scene_case(nb=nw * nf, H=H, W=W, C=C, K=K, level_ids=level_ids, seed=seed, n_points=n_points, shared_depth=True,
                      window_frames=nf, dtype=dtype)


def _gpu_level(l):
    from banet_b200 import ops
    return ops.Level(to_cuda32(l.conv1), to_cuda32(l.conv2), to_cuda32(l.intr), to_cuda32(l.p), to_cuda32(l.D), to_cuda32(l.B), grid=l.grid)


def _built(nw, nf, C, K, seed=83, n_points=400, H=48, W=64, precision=0):
    """Per-pair normal equations of nw windows (ops.lm_build on nw * nf pairs) and the start iterate, on the GPU."""
    from banet_b200 import ops
    sc = _batch_scene(nw, nf, C, K, seed=seed, n_points=n_points, H=H, W=W)
    lv = _gpu_level(sc.levels[0])
    R, T = to_cuda32(sc.R0), to_cuda32(sc.T0)
    Wb = to_cuda32(sc.W0.reshape(nw, nf, K, 1)[:, 0]) + 0.01 * torch.arange(1, nw + 1, device="cuda").reshape(nw, 1, 1)
    Hm, g, _, _ = ops.lm_build(lv, R, T, Wb.repeat_interleave(nf, 0).contiguous(), precision)
    return lv, Hm, g, R, T, Wb


@pytest.mark.gpu
@pytest.mark.parametrize("nf,K", [(1, 16), (1, 128), (4, 16), (4, 128)])
def test_one_window_agrees_with_the_single_window_entries(nf, K):
    from banet_b200 import ops, _lib
    _lib.require_device()
    _, Hm, g, R, T, W = _built(1, nf, 32, K, n_points=2048)
    lam = torch.tensor([0.5], device="cuda")
    a = ops.lm_window_batch_solve_update(Hm, g, lam, R, T, W)
    b = ops.lm_window_solve_update(Hm, g, lam, R, T, W[0])
    assert int(a[4].abs().max()) == 0 and int(b[4].abs().max()) == 0
    errs = [rel_fro(x, y.reshape(x.shape)) for x, y in zip(a[:4], b[:4])]
    print(f"nf={nf} K={K} forward R', T', W', delta: " + " ".join(f"{e:.1e}" for e in errs))
    gen = torch.Generator(device="cuda").manual_seed(4)
    dR, dT, dW = (torch.randn(s, generator=gen, device="cuda") for s in ((nf, 3, 3), (nf, 3, 1), (1, K, 1)))
    ga = ops.lm_window_batch_solve_update_bwd(Hm, g, lam, a[3], R, T, dR, dT, dW)
    gb = ops.lm_window_solve_update_bwd(Hm, g, lam, b[3], R, T, dR, dT, dW[0])
    berrs = [rel_fro(x, y.reshape(x.shape)) for x, y in zip(ga, gb)]
    print(f"nf={nf} K={K} backward dH, dg, dlambda, dR, dT, dW: " + " ".join(f"{e:.1e}" for e in berrs))
    assert max(errs) < 1e-5 and max(berrs) < 1e-5


@pytest.mark.gpu
def test_windows_of_a_batch_are_independent_bit_for_bit():
    from banet_b200 import ops, _lib
    _lib.require_device()
    nw, nf, K = 5, 3, 16
    sc = _batch_scene(nw, nf, 16, K, seed=5, level_ids=(2, 3), H=96, W=128, n_points=None)
    levels = [_gpu_level(l) for l in sc.levels]
    lv, R, T = levels[-1], to_cuda32(sc.R0), to_cuda32(sc.T0)
    W = 0.01 * torch.randn(nw, K, 1, generator=torch.Generator(device="cuda").manual_seed(2), device="cuda")
    Hm, g, _, _ = ops.lm_build(lv, R, T, W.repeat_interleave(nf, 0).contiguous(), 0)
    lam = torch.linspace(0.2, 0.6, nw, device="cuda")
    a = ops.lm_window_batch_solve_update(Hm, g, lam, R, T, W)
    gen = torch.Generator(device="cuda").manual_seed(9)
    dR, dT, dW = (torch.randn(s, generator=gen, device="cuda") for s in ((nw * nf, 3, 3), (nw * nf, 3, 1), (nw, K, 1)))
    ga = ops.lm_window_batch_solve_update_bwd(Hm, g, lam, a[3], R, T, dR, dT, dW)
    packed = [ops.pack_mlp(mlp_for(16, l.level, torch.float32)).cuda() for l in sc.levels]
    ra = ops.lm_window_batch_run(levels, nw, 2, R, T, W, mlp_packed=packed, l2_regularizer_base=1000.0, precision=0)
    assert int(a[4].abs().max()) == 0 and int(ra[3].abs().max()) == 0
    for w in range(nw):
        s = slice(w * nf, (w + 1) * nf)
        one = ops.lm_window_batch_solve_update(Hm[s], g[s], lam[w:w + 1], R[s], T[s], W[w:w + 1])
        for x, y in zip(one, (a[0][s], a[1][s], a[2][w:w + 1], a[3][w:w + 1], a[4][s])):
            assert torch.equal(x, y)
        gone = ops.lm_window_batch_solve_update_bwd(Hm[s], g[s], lam[w:w + 1], one[3], R[s], T[s], dR[s], dT[s], dW[w:w + 1])
        for x, y in zip(gone, (ga[0][s], ga[1][s], ga[2][w:w + 1], ga[3][s], ga[4][s], ga[5][w:w + 1])):
            assert torch.equal(x, y)
    # The whole run: the build sums each pair's tiles in a partition that depends on how many pairs share the launch, so a window run alone
    # matches its batched run to rounding; with the batch size fixed, a window's bits do not depend on what the other windows hold.
    for w in range(nw):
        s = slice(w * nf, (w + 1) * nf)
        lvw = [ops.Level(l.conv1[s], l.conv2[s], l.intr[s], l.p[s], l.D[s], l.B[s], grid=l.grid) for l in levels]
        rone = ops.lm_window_batch_run(lvw, 1, 2, R[s], T[s], W[w:w + 1], mlp_packed=packed, l2_regularizer_base=1000.0, precision=0)
        for x, y in zip(rone[:3], (ra[0][s], ra[1][s], ra[2][w:w + 1])):
            assert rel_fro(x, y) < 1e-6
        assert torch.equal(rone[3], ra[3][s])
        other = torch.ones(nw * nf, 1, 1, 1, device="cuda"); other[:s.start] = 1.1; other[s.stop:] = 0.9
        lvo = [ops.Level(l.conv1, (l.conv2 * other).contiguous(), l.intr, l.p, l.D, l.B, grid=l.grid) for l in levels]
        ro = ops.lm_window_batch_run(lvo, nw, 2, R, T, W, mlp_packed=packed, l2_regularizer_base=1000.0, precision=0)
        assert not torch.equal(ro[0], ra[0])
        for x, y in zip((ro[0][s], ro[1][s], ro[2][w:w + 1], ro[3][s]), (ra[0][s], ra[1][s], ra[2][w:w + 1], ra[3][s])):
            assert torch.equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize("nf,C,K", [(3, 16, 16), (4, 128, 128)])
def test_one_batch_run_iteration_is_build_plus_batch_step(nf, C, K):
    from banet_b200 import ops, _lib
    _lib.require_device()
    nw = 2
    lv, Hm, g, R, T, W = _built(nw, nf, C, K)
    lam = torch.full((nw,), 0.5, device="cuda")
    Rn, Tn, Wn, _, status = ops.lm_window_batch_solve_update(Hm, g, lam, R, T, W)
    R2, T2, W2, status2 = ops.lm_window_batch_run([lv], nw, 1, R, T, W, lambda_fixed=0.5, precision=_lib.PREC_FP32_SIMT)
    assert int(status.abs().max()) == 0
    assert torch.equal(Rn, R2) and torch.equal(Tn, T2) and torch.equal(Wn, W2) and torch.equal(status, status2)


@pytest.mark.gpu
def test_window_batch_step_is_reproducible_and_ignores_the_workspace():
    from banet_b200 import ops, _lib
    _lib.require_device()
    nw, nf, K = 3, 4, 128
    _, Hm, g, R, T, W = _built(nw, nf, 32, K, n_points=2048)
    lib = _lib.load()
    lam = torch.tensor([0.3, 0.4, 0.5], device="cuda")
    opts = _opts()
    gen = torch.Generator(device="cuda").manual_seed(6)
    dRn, dTn, dWn = (torch.randn(s, generator=gen, device="cuda") for s in ((nw * nf, 3, 3), (nw * nf, 3, 1), (nw, K, 1)))
    outs = []
    for fill in ("nan", "random", "nan"):
        nbytes = lib.banet_lm_window_batch_solve_update_workspace_bytes(nw, nf, K)
        ws = torch.empty(nbytes // 4 + 1, device="cuda")
        ws.fill_(float("nan")) if fill == "nan" else ws.uniform_(-1e3, 1e3)
        o = [torch.empty_like(R), torch.empty_like(T), torch.empty_like(W), torch.empty(nw, 6 * nf + K, device="cuda"),
             torch.empty(nw * nf, device="cuda", dtype=torch.int32)]
        _lib.check(lib.banet_lm_window_batch_solve_update(Hm.data_ptr(), g.data_ptr(), lam.data_ptr(), nw, nf, K, ctypes.byref(opts), R.data_ptr(),
                                                          T.data_ptr(), W.data_ptr(), *[x.data_ptr() for x in o], ws.data_ptr(), ws.numel() * 4,
                                                          ops._stream()), "banet_lm_window_batch_solve_update")
        ws.fill_(float("nan")) if fill == "nan" else ws.uniform_(-1e3, 1e3)
        b = [torch.empty(nw * nf, 6 + K, 6 + K, device="cuda"), torch.empty(nw * nf, 6 + K, device="cuda"), torch.empty(nw, device="cuda"),
             torch.empty_like(R), torch.empty_like(T), torch.empty_like(W)]
        _lib.check(lib.banet_lm_window_batch_solve_update_bwd(Hm.data_ptr(), g.data_ptr(), lam.data_ptr(), o[3].data_ptr(), nw, nf, K, ctypes.byref(opts),
                                                              R.data_ptr(), T.data_ptr(), dRn.data_ptr(), dTn.data_ptr(), dWn.data_ptr(),
                                                              *[x.data_ptr() for x in b], ws.data_ptr(), ws.numel() * 4, ops._stream()),
                   "banet_lm_window_batch_solve_update_bwd")
        outs.append(o + b)
    assert int(outs[0][4].abs().max()) == 0
    for other in outs[1:]:
        for x, y in zip(outs[0], other):
            assert torch.equal(x, y)


def _mlp_leaves(C, level=3):
    return [(w.clone().requires_grad_(), b.clone().requires_grad_()) for w, b in mlp_for(C, level)]


def _gradients_vs_oracle(nw, nf, C, K, n_points, fixed_lambda, seed=71, tol=2e-3):
    """window_batch_iteration_fused against a loop of the float64 oracle's window_iteration over the windows, outputs and gradients of a
    random linear functional (tolerances of test_window_gradients_match_oracle_autograd)."""
    from banet_b200 import autograd as ag
    H, Wd = (48, 64) if n_points <= 400 else (120, 160)
    sc = _batch_scene(nw, nf, C, K, seed=seed, n_points=n_points, H=H, W=Wd)
    lv = sc.levels[0]
    a = oracle_level_inputs(lv)
    names = ["conv1", "conv2", "D", "B"]
    for n in names:
        a[n] = a[n].clone().requires_grad_()
    R = sc.R0.double().clone().requires_grad_(); T = sc.T0.double().clone().requires_grad_()
    W = (sc.W0.reshape(nw, nf, K, 1)[:, 0].double() + 0.01 * torch.randn(nw, K, 1, generator=torch.Generator().manual_seed(3), dtype=torch.float64)).requires_grad_()
    mlp64 = [] if fixed_lambda is not None else _mlp_leaves(C)
    g = torch.Generator().manual_seed(5)
    cR, cT, cW = (torch.randn(nw * nf, 3, 3, generator=g, dtype=torch.float64), torch.randn(nw * nf, 3, 1, generator=g, dtype=torch.float64),
                  torch.randn(nw, K, 1, generator=g, dtype=torch.float64))
    oR, oT, oW = [], [], []
    for w in range(nw):
        s = slice(w * nf, (w + 1) * nf)
        lam = None if fixed_lambda is None else torch.tensor([fixed_lambda], dtype=torch.float64)
        r = O.window_iteration(a["conv1"][s], a["conv2"][s], a["fx"][s], a["fy"][s], a["ox"][s], a["oy"][s], a["p"][s], a["D"][s], a["B"][s],
                               R[s], T[s], W[w], mlp64, O.IterOptions(l2_regularizer_base=1000.0, guard_nonfinite=True, lambda_override=lam))
        oR.append(r[0]); oT.append(r[1]); oW.append(r[2])
    oR, oT, oW = torch.cat(oR), torch.cat(oT), torch.stack(oW)
    ((oR * cR).sum() + (oT * cT).sum() + (oW * cW).sum()).backward()

    bw = lambda t: to_cuda32(t.detach()).reshape(nw, nf, *t.shape[1:]).requires_grad_()
    t = {n: bw(a[n]) for n in names}
    Rg, Tg = bw(R), bw(T)
    Wg = to_cuda32(W.detach()).requires_grad_()
    mlp32 = [(to_cuda32(w.detach()).requires_grad_(), to_cuda32(b.detach()).requires_grad_()) for w, b in mlp64]
    lam32 = None if fixed_lambda is None else torch.full((nw,), fixed_lambda, device="cuda")
    intr = to_cuda32(lv.intr).reshape(nw, nf, 4); p = to_cuda32(lv.p).reshape(nw, nf, 3, -1)
    gR, gT, gW, status = ag.window_batch_iteration_fused(t["conv1"], t["conv2"], intr, p, t["D"], t["B"], Rg, Tg, Wg, mlp32, 1000.0, exact_sym=True,
                                                         lambda_override=lam32, return_status=True)
    assert int(status.abs().max()) == 0
    e = (rel_fro(gR.reshape(oR.shape), oR), rel_fro(gT.reshape(oT.shape), oT), rel_fro(gW, oW))
    print(f"batch nw={nw} nf={nf} C={C} K={K}: outputs R {e[0]:.1e} T {e[1]:.1e} W {e[2]:.1e}")
    assert e[0] < 1e-5 and e[1] < 1e-4 and e[2] < 1e-3
    ((gR * to_cuda32(cR).reshape(gR.shape)).sum() + (gT * to_cuda32(cT).reshape(gT.shape)).sum() + (gW * to_cuda32(cW)).sum()).backward()
    for nm, x, y in [(n, t[n], a[n]) for n in names] + [("R", Rg, R), ("T", Tg, T), ("W", Wg, W)]:
        err = rel_fro(x.grad.reshape(y.grad.shape), y.grad)
        print(f"grad {nm}: {err:.2e}")
        assert err < tol, nm
    for i, ((w32, _), (w64, _)) in enumerate(zip(mlp32, mlp64)):
        err = rel_fro(w32.grad, w64.grad)
        print(f"grad lambda filters {i + 1}: {err:.2e}")
        assert err < tol


@pytest.mark.gpu
@pytest.mark.parametrize("nw,nf,C,K,n_points,fixed_lambda", [(3, 2, 8, 5, 400, None), (3, 4, 8, 5, 400, None), (2, 4, 64, 128, 4096, 0.4)])
def test_window_batch_gradients_match_oracle_autograd(nw, nf, C, K, n_points, fixed_lambda):
    from banet_b200 import _lib
    _lib.require_device()
    _gradients_vs_oracle(nw, nf, C, K, n_points, fixed_lambda)


def _run_vs_oracle(nw, nf, C, K, iters, precision, tolW, level_ids=(2, 3), H=96, W=128, seed=41):
    from banet_b200 import ops
    sc = _batch_scene(nw, nf, C, K, seed=seed, n_points=None, H=H, W=W, level_ids=level_ids, dtype=torch.float64)
    lvs = []
    for l in sc.levels:
        a = oracle_level_inputs(l)
        lvs.append((a, mlp_for(C, l.level)))
    oR, oT, oW = [], [], []
    for w in range(nw):
        s = slice(w * nf, (w + 1) * nf)
        olv = [O.LevelInputs(a["conv1"][s], a["conv2"][s], a["fx"][s], a["fy"][s], a["ox"][s], a["oy"][s], a["p"][s], a["D"][s], a["B"][s], m) for a, m in lvs]
        r = O.window_solve(olv, iters, sc.R0[s], sc.T0[s], sc.W0[w * nf])
        oR.append(r[0]); oT.append(r[1]); oW.append(r[2])
    oR, oT, oW = torch.cat(oR), torch.cat(oT), torch.stack(oW)
    levels = [_gpu_level(l) for l in sc.levels]
    packed = [ops.pack_mlp([(w.float(), b.float()) for w, b in m]).cuda() for _, m in lvs]
    W0 = to_cuda32(sc.W0.reshape(nw, nf, K, 1)[:, 0])
    R, T, Wn, st = ops.lm_window_batch_run(levels, nw, iters, to_cuda32(sc.R0), to_cuda32(sc.T0), W0, mlp_packed=packed, l2_regularizer_base=1000.0,
                                           precision=precision)
    assert int(st.abs().max()) == 0
    e = (rel_fro(R, oR), rel_fro(T, oT), rel_fro(Wn, oW))
    print(f"batch run nw={nw} nf={nf} C={C} K={K} prec={precision}: R {e[0]:.1e} T {e[1]:.1e} W {e[2]:.1e}")
    assert e[0] < 1e-5 and e[1] < 1e-4 and e[2] < tolW
    return levels, packed, sc


@pytest.mark.gpu
@pytest.mark.parametrize("nw,nf,C,K", [(2, 3, 16, 16), (2, 4, 128, 128)])
def test_window_batch_run_matches_oracle(nw, nf, C, K):
    from banet_b200 import _lib
    _lib.require_device()
    _run_vs_oracle(nw, nf, C, K, 3, _lib.PREC_FP32_SIMT, 2e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("nf,K", [(60, 5), (40, 128)])
def test_windows_beyond_the_dense_limit_run_and_match_the_oracle(nf, K):
    from banet_b200 import ops, _lib
    _lib.require_device()
    C = 8 if K == 5 else 16
    levels, packed, sc = _run_vs_oracle(1, nf, C, K, 2, _lib.PREC_FP32_SIMT, 2e-4, level_ids=(3,), H=48 if K == 5 else 96, W=64 if K == 5 else 128)
    R0, T0, W0 = to_cuda32(sc.R0), to_cuda32(sc.T0), to_cuda32(sc.W0[0])
    with pytest.raises(_lib.BanetError, match="code -4"):
        ops.lm_window_run(levels, 1, R0, T0, W0, mlp_packed=packed, l2_regularizer_base=1000.0, precision=_lib.PREC_FP32_SIMT)
    Hm, g, _, _ = ops.lm_build(levels[0], R0, T0, W0.reshape(1, K, 1).expand(nf, K, 1).contiguous(), _lib.PREC_FP32_SIMT)
    lam = torch.tensor([0.5], device="cuda")
    with pytest.raises(_lib.BanetError, match="code -4"):
        ops.lm_window_solve_update(Hm, g, lam, R0, T0, W0)
    with pytest.raises(_lib.BanetError, match="code -4"):
        ops.lm_window_solve_update_bwd(Hm, g, lam, torch.zeros(6 * nf + K, device="cuda"), R0, T0, torch.zeros_like(R0), torch.zeros_like(T0), W0)
    if K == 5:
        _gradients_vs_oracle(1, nf, 8, 5, 400, None, seed=72)


@pytest.mark.gpu
def test_k256_windows_match_the_oracle():
    from banet_b200 import _lib
    _lib.require_device()
    _run_vs_oracle(2, 4, 16, 256, 2, _lib.PREC_FP32_SIMT, 1e-3, level_ids=(3,))


@pytest.mark.gpu
def test_a_skipped_window_stays_contained():
    from banet_b200 import ops, autograd as ag, _lib
    _lib.require_device()
    nw, nf, C, K = 3, 3, 8, 5
    sc = _batch_scene(nw, nf, C, K, seed=13)
    l = sc.levels[0]
    lv = _gpu_level(l)
    bad = ops.Level(lv.conv1.clone(), lv.conv2, lv.intr, lv.p, lv.D, lv.B)
    bad.conv1[nf + 1, 3, 0] = float("nan")                             # window 1, frame 1
    R, T = to_cuda32(sc.R0), to_cuda32(sc.T0)
    W = to_cuda32(sc.W0.reshape(nw, nf, K, 1)[:, 0]) + 0.01
    packed = [ops.pack_mlp(mlp_for(C, 3, torch.float32)).cuda()]
    a = ops.lm_window_batch_run([lv], nw, 2, R, T, W, mlp_packed=packed, l2_regularizer_base=1000.0, precision=0)
    b = ops.lm_window_batch_run([bad], nw, 2, R, T, W, mlp_packed=packed, l2_regularizer_base=1000.0, precision=0)
    st = b[3].reshape(nw, nf)
    assert bool((st[1] != 0).all()) and int(st[0].abs().max()) == 0 and int(st[2].abs().max()) == 0
    ok = [0, 1, 2, nf * 2, nf * 2 + 1, nf * 2 + 2]
    assert torch.equal(a[0][ok], b[0][ok]) and torch.equal(a[1][ok], b[1][ok]) and torch.equal(a[2][[0, 2]], b[2][[0, 2]])
    assert torch.equal(b[2][1], W[1])                                  # a skipped window keeps its W (every iteration skipped: NaN stays)
    # step and backward on the poisoned build: window 1 zero dH, dg, dlambda, pass-through; the others as without the NaN
    Wp = W.repeat_interleave(nf, 0).contiguous()
    lam = torch.full((nw,), 0.5, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(3)
    dR, dT, dW = (torch.randn(s, generator=gen, device="cuda") for s in ((nw * nf, 3, 3), (nw * nf, 3, 1), (nw, K, 1)))
    res = []
    for level in (lv, bad):
        Hm, g, _, _ = ops.lm_build(level, R, T, Wp, 0)
        f = ops.lm_window_batch_solve_update(Hm, g, lam, R, T, W)
        res.append((f, ops.lm_window_batch_solve_update_bwd(Hm, g, lam, f[3], R, T, dR, dT, dW)))
    (fa, ga), (fb, gb) = res
    s1 = slice(nf, 2 * nf)
    assert bool((fb[4][s1] != 0).all()) and not bool(fb[3][1].any())
    assert not bool(gb[0][s1].any()) and not bool(gb[1][s1].any()) and float(gb[2][1]) == 0.0
    assert torch.equal(gb[3][s1], dR[s1]) and torch.equal(gb[4][s1], dT[s1]) and torch.equal(gb[5][1], dW[1])
    for w in (0, 2):
        s = slice(w * nf, (w + 1) * nf)
        assert torch.equal(fa[3][w], fb[3][w]) and torch.equal(ga[0][s], gb[0][s]) and torch.equal(ga[1][s], gb[1][s]) and torch.equal(ga[2][w], gb[2][w])


def _net_and_batch(nw=2, nf=3, C=8, K=5, seed=91, once=False):
    from banet_b200.bundlenet import BundleNet
    from banet_b200 import _lib
    sc = _batch_scene(nw, nf, C, K, seed=seed, n_points=500)
    lv = sc.levels[0]
    net = BundleNet(C, levels=("3",), exact_sym_grad=True, precision=_lib.PREC_FP32_SIMT, strict_status=True).cuda()
    for i, (w, b) in enumerate(mlp_for(C, 3)):
        getattr(net, f"lambda_3_{i + 1}_filters").data.copy_(w); getattr(net, f"lambda_3_{i + 1}_biases").data.copy_(b)
    fr = lambda t: to_cuda32(t).reshape(nw, nf, *t.shape[1:])
    x = dict(conv1=fr(lv.conv1), conv2=fr(lv.conv2), p=fr(lv.p), D=fr(lv.D), B=fr(lv.B), R=fr(sc.R0), T=fr(sc.T0),
             W=to_cuda32(sc.W0.reshape(nw, nf, K, 1)[:, 0]) + 0.01)
    fx, fy, ox, oy = [fr(t) for t in lv.intr_tiled()]
    call = lambda d: net.WindowIteration(d["conv1"], d["conv2"], fx, fy, ox, oy, d["p"], d["D"], d["B"], d["R"], d["T"], d["W"], 1000.0, "3")
    return net, x, call


@pytest.mark.gpu
def test_batched_window_iteration_grad_and_no_grad_paths_agree():
    from banet_b200 import _lib
    _lib.require_device()
    net, x, call = _net_and_batch()
    with torch.no_grad():
        a = call(x)
    b = call({k: v.clone().requires_grad_() for k, v in x.items()})
    assert all(t.requires_grad for t in b) and not any(t.requires_grad for t in a)
    assert tuple(net.last_status.shape) == (2, 3) and int(net.last_status.abs().max()) == 0
    assert tuple(a[0].shape) == (2, 3, 3, 3) and tuple(a[1].shape) == (2, 3, 3, 1) and tuple(a[2].shape) == (2, 5, 1)
    for u, v in zip(a, b):
        assert rel_fro(u, v.detach()) < 1e-5


@pytest.mark.gpu
def test_batched_window_iteration_strict_status_raises_on_a_skipped_window():
    from banet_b200 import _lib
    _lib.require_device()
    net, x, call = _net_and_batch()
    x["conv1"] = x["conv1"].clone(); x["conv1"][1, 0, 0, 0] = float("nan")
    with torch.no_grad(), pytest.raises(RuntimeError, match="skipped"):
        call(x)
    with pytest.raises(RuntimeError, match="skipped"):
        call({k: v.clone().requires_grad_() for k, v in x.items()})
    assert bool((net.last_status[1] != 0).all()) and int(net.last_status[0].abs().max()) == 0


@pytest.mark.gpu
def test_batched_window_iteration_broadcast_keyframe_gets_the_frame_summed_gradient():
    from banet_b200 import _lib
    _lib.require_device()
    net, x, call = _net_and_batch()
    nf = x["R"].shape[1]
    key = ("conv1", "p", "D", "B")
    once = {k: (v[:, :1].clone() if k in key else v.clone()).requires_grad_(k != "p") for k, v in x.items()}
    per_frame = {k: (v[:, :1].repeat(1, nf, *[1] * (v.dim() - 2)) if k in key else v.clone()).requires_grad_(k != "p") for k, v in x.items()}
    outs = [call(d) for d in (once, per_frame)]
    gen = torch.Generator(device="cuda").manual_seed(12)
    c = [torch.randn(t.shape, generator=gen, device="cuda") for t in outs[0]]
    for o in outs:
        sum((t * ci).sum() for t, ci in zip(o, c)).backward()
    for u, v in zip(outs[0], outs[1]):
        assert torch.equal(u, v)
    for k in ("conv1", "D", "B"):                                    # the build's backward accumulates with atomics: equal up to summation order
        assert rel_fro(once[k].grad[:, 0], per_frame[k].grad.sum(1)) < 1e-5, k
    for k in ("conv2", "R", "T", "W"):
        assert rel_fro(once[k].grad, per_frame[k].grad) < 1e-5, k
