"""The differentiable joint keyframe window (banet_lm_window_solve_update / _bwd, autograd.window_iteration_fused, BundleNet.WindowIteration):
the float64 oracle's window_iteration is the reference (its own gradients checked by gradcheck on the CPU), the GPU gradients are compared
with its autograd, nf = 1 must be the 2-view entries bit for bit, and the one-iteration forward the step banet_lm_window_run takes."""
import ctypes

import pytest
import torch

from helpers import O, scene_case, oracle_level_inputs, mlp_for, rel_fro, to_cuda32


def _oracle_args(lv):
    a = oracle_level_inputs(lv)
    return [a[k] for k in ("conv1", "conv2", "fx", "fy", "ox", "oy", "p", "D", "B")]


# ------------------------------------------------------------------------------------------ CPU
def test_oracle_window_iteration_passes_gradcheck():
    nf, C, K = 2, 3, 3
    sc = scene_case(nb=nf, H=24, W=32, C=C, K=K, level_ids=(3,), seed=19, shared_depth=True)
    conv1, conv2, fx, fy, ox, oy, p, D, B = _oracle_args(sc.levels[0])
    mlp = mlp_for(C, 3)
    W0 = sc.W0[0].double() + 0.01

    def f(R, T, W, conv2, B):
        return O.window_iteration(conv1, conv2, fx, fy, ox, oy, p, D, B, R, T, W, mlp, O.IterOptions(l2_regularizer_base=1000.0))

    R, T, W, conv2, B = (t.double().clone().requires_grad_() for t in (sc.R0, sc.T0, W0, conv2, B))
    # every Jacobian entry w.r.t. the pose and W; the large feature map and basis through random projections (fast mode)
    assert torch.autograd.gradcheck(lambda R, T, W: f(R, T, W, conv2.detach(), B.detach()), (R, T, W), eps=1e-7, atol=1e-6, rtol=1e-4)
    assert torch.autograd.gradcheck(f, (R, T, W, conv2, B), eps=1e-7, atol=1e-6, rtol=1e-4, fast_mode=True)


def _opts(**kw):
    from banet_b200._lib import BanetSolveOpts
    return BanetSolveOpts(kw.get("eps", 1e-5), kw.get("undamped_last", 1), kw.get("scramble", 0))


def test_window_solve_update_entries_reject_bad_arguments_without_gpu():
    from banet_b200 import _lib
    lib = _lib.load()
    opts = _opts()
    p = 1                                                            # non-null dummy pointers: every check below fires before a CUDA call
    fwd = lambda nf, K, o=opts, H=p, ws=p, nbytes=1 << 30: lib.banet_lm_window_solve_update(H, p, p, nf, K, ctypes.byref(o), p, p, p, p, p, p, p, p, ws, nbytes, None)
    bwd = lambda nf, K, o=opts, dW=p, ws=p, nbytes=1 << 30: lib.banet_lm_window_solve_update_bwd(p, p, p, p, nf, K, ctypes.byref(o), p, p, p, p, dW,
                                                                                                 p, p, p, p, p, p, ws, nbytes, None)
    assert fwd(4, 128, H=None) == -1 and b"null" in lib.banet_last_error()
    assert bwd(4, 128, dW=None) == -1 and b"null" in lib.banet_last_error()
    for call in (fwd, bwd):
        assert call(0, 128) == -1
        assert call(4, 0) == -1
        assert call(4, 128, o=_opts(scramble=1)) == -1
        assert call(4, 4096) == -4 and b"do not fit" in lib.banet_last_error()           # 6 nf + K beyond the fused solve
        assert call(40, 128) == -4
        assert call(4, 128, ws=None) == -2
        assert call(4, 128, nbytes=16) == -2
    assert lib.banet_lm_window_solve_update_workspace_bytes(4, 128) > 0 and lib.banet_lm_window_solve_update_bwd_workspace_bytes(4, 128) > 0
    assert lib.banet_lm_window_solve_update_workspace_bytes(0, 128) == 0 and lib.banet_lm_window_solve_update_bwd_workspace_bytes(4, 0) == 0


# ------------------------------------------------------------------------------------------ GPU
def _mlp_leaves(C, level=3):
    return [(w.clone().requires_grad_(), b.clone().requires_grad_()) for w, b in mlp_for(C, level)]


@pytest.mark.gpu
@pytest.mark.parametrize("nf,C,K,n_points,fixed_lambda", [(2, 8, 5, 400, None), (4, 8, 5, 400, None), (4, 64, 128, 4096, 0.4)])
def test_window_gradients_match_oracle_autograd(nf, C, K, n_points, fixed_lambda):
    from banet_b200 import autograd as ag, _lib
    _lib.require_device()
    H, Wd = (48, 64) if n_points <= 400 else (120, 160)
    sc = scene_case(nb=nf, H=H, W=Wd, C=C, K=K, level_ids=(3,), seed=71, n_points=n_points, shared_depth=True, dtype=torch.float32)
    lv = sc.levels[0]
    a = oracle_level_inputs(lv)
    names = ["conv1", "conv2", "D", "B"]
    for n in names:
        a[n] = a[n].clone().requires_grad_()
    R = sc.R0.double().clone().requires_grad_(); T = sc.T0.double().clone().requires_grad_()
    W = (sc.W0[0].double() + 0.01 * torch.randn(K, 1, generator=torch.Generator().manual_seed(3), dtype=torch.float64)).requires_grad_()
    mlp64 = [] if fixed_lambda is not None else _mlp_leaves(C)
    lam = None if fixed_lambda is None else torch.tensor([fixed_lambda], dtype=torch.float64)
    g = torch.Generator().manual_seed(5)
    cR, cT, cW = (torch.randn(nf, 3, 3, generator=g, dtype=torch.float64), torch.randn(nf, 3, 1, generator=g, dtype=torch.float64),
                  torch.randn(K, 1, generator=g, dtype=torch.float64))
    oR, oT, oW = O.window_iteration(a["conv1"], a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"], R, T, W, mlp64,
                                    O.IterOptions(l2_regularizer_base=1000.0, guard_nonfinite=True, lambda_override=lam))
    ((oR * cR).sum() + (oT * cT).sum() + (oW * cW).sum()).backward()

    t = {n: to_cuda32(a[n].detach()).requires_grad_() for n in names}
    Rg, Tg, Wg = (to_cuda32(x.detach()).requires_grad_() for x in (R, T, W))
    mlp32 = [(to_cuda32(w.detach()).requires_grad_(), to_cuda32(b.detach()).requires_grad_()) for w, b in mlp64]
    gR, gT, gW, status = ag.window_iteration_fused(t["conv1"], t["conv2"], to_cuda32(lv.intr), to_cuda32(lv.p), t["D"], t["B"], Rg, Tg, Wg, mlp32,
                                                   1000.0, exact_sym=True, lambda_override=None if lam is None else to_cuda32(lam),
                                                   return_status=True)
    assert int(status.abs().max()) == 0
    e = (rel_fro(gR, oR), rel_fro(gT, oT), rel_fro(gW, oW))
    print(f"window nf={nf} C={C} K={K}: outputs R {e[0]:.1e} T {e[1]:.1e} W {e[2]:.1e}")
    assert e[0] < 1e-5 and e[1] < 1e-4 and e[2] < 1e-3
    ((gR * to_cuda32(cR)).sum() + (gT * to_cuda32(cT)).sum() + (gW * to_cuda32(cW)).sum()).backward()
    tol = 2e-3
    for nm, x, y in [(n, t[n], a[n]) for n in names] + [("R", Rg, R), ("T", Tg, T), ("W", Wg, W)]:
        err = rel_fro(x.grad, y.grad)
        print(f"grad {nm}: {err:.2e}")
        assert err < tol, nm
    for i, ((w32, _), (w64, _)) in enumerate(zip(mlp32, mlp64)):
        err = rel_fro(w32.grad, w64.grad)
        print(f"grad lambda filters {i + 1}: {err:.2e}")
        assert err < tol


def _built_pairs(nf, C, K, seed=83, n_points=None, H=48, W=64):
    """Per-pair normal equations of a window (ops.lm_build, fp32 SIMT) and its start iterate, on the GPU."""
    from banet_b200 import ops, _lib
    sc = scene_case(nb=nf, H=H, W=W, C=C, K=K, level_ids=(3,), seed=seed, n_points=n_points, shared_depth=True, dtype=torch.float32)
    l = sc.levels[0]
    lv = ops.Level(to_cuda32(l.conv1), to_cuda32(l.conv2), to_cuda32(l.intr), to_cuda32(l.p), to_cuda32(l.D), to_cuda32(l.B), grid=l.grid)
    R, T = to_cuda32(sc.R0), to_cuda32(sc.T0)
    W = to_cuda32(sc.W0[0]) + 0.01
    Hm, g, _, _ = ops.lm_build(lv, R, T, W.reshape(1, K, 1).expand(nf, K, 1), _lib.PREC_FP32_SIMT)
    return lv, Hm, g, R, T, W


@pytest.mark.gpu
def test_one_frame_window_is_the_two_view_step_bit_for_bit():
    from banet_b200 import ops, _lib
    _lib.require_device()
    K = 16
    _, Hm, g, R, T, W = _built_pairs(1, 16, K)
    lam = torch.tensor([0.7], device="cuda")
    Rn, Tn, Wn, delta, status = ops.lm_window_solve_update(Hm, g, lam, R, T, W)
    R2, T2, W2, delta2, _, status2 = ops.lm_step(Hm, g, None, 1, None, 1.0, R, T, W.reshape(1, K, 1), lam=lam)
    assert int(status.abs().max()) == 0
    assert torch.equal(Rn, R2) and torch.equal(Tn, T2) and torch.equal(Wn, W2[0]) and torch.equal(delta, delta2[0]) and torch.equal(status, status2)
    gen = torch.Generator(device="cuda").manual_seed(4)
    dR, dT, dW = (torch.randn(s, generator=gen, device="cuda") for s in ((1, 3, 3), (1, 3, 1), (K, 1)))
    a = ops.lm_window_solve_update_bwd(Hm, g, lam, delta, R, T, dR, dT, dW)
    b = ops.lm_solve_update_bwd(Hm, g, lam, delta.reshape(1, -1), R, T, dR, dT, dW.reshape(1, K, 1))
    for x, y in zip(a, b):
        assert torch.equal(x, y.reshape(x.shape))


@pytest.mark.gpu
@pytest.mark.parametrize("nf,C,K", [(3, 16, 16), (4, 128, 128)])
def test_build_plus_window_solve_update_is_one_step_of_the_window_run(nf, C, K):
    from banet_b200 import ops, _lib
    _lib.require_device()
    lv, Hm, g, R, T, W = _built_pairs(nf, C, K)
    Rn, Tn, Wn, _, status = ops.lm_window_solve_update(Hm, g, torch.tensor([0.5], device="cuda"), R, T, W)
    R2, T2, W2, status2 = ops.lm_window_run([lv], 1, R, T, W, lambda_fixed=0.5, precision=_lib.PREC_FP32_SIMT)
    assert int(status.abs().max()) == 0
    assert torch.equal(Rn, R2) and torch.equal(Tn, T2) and torch.equal(Wn, W2) and torch.equal(status, status2)


@pytest.mark.gpu
def test_window_solve_update_ignores_what_the_workspace_held():
    import ctypes as C
    from banet_b200 import ops, _lib
    from banet_b200._lib import BanetSolveOpts
    _lib.require_device()
    nf, K = 4, 128
    _, Hm, g, R, T, W = _built_pairs(nf, 32, K, n_points=2048)
    lib = _lib.load()
    lam = torch.tensor([0.3], device="cuda")
    opts = BanetSolveOpts(1e-5, 1, 0)
    nbytes = lib.banet_lm_window_solve_update_workspace_bytes(nf, K)
    outs = []
    for fill in ("nan", "random"):
        ws = torch.empty(nbytes // 4 + 1, device="cuda")
        ws.fill_(float("nan")) if fill == "nan" else ws.uniform_(-1e3, 1e3)
        o = [torch.empty_like(R), torch.empty_like(T), torch.empty_like(W), torch.empty(6 * nf + K, device="cuda"), torch.empty(nf, device="cuda", dtype=torch.int32)]
        _lib.check(lib.banet_lm_window_solve_update(Hm.data_ptr(), g.data_ptr(), lam.data_ptr(), nf, K, C.byref(opts), R.data_ptr(), T.data_ptr(), W.data_ptr(),
                                                    *[x.data_ptr() for x in o], ws.data_ptr(), ws.numel() * 4, ops._stream()), "banet_lm_window_solve_update")
        outs.append(o)
    assert int(outs[0][4].abs().max()) == 0
    for x, y in zip(*outs):
        assert torch.equal(x, y)


@pytest.mark.gpu
def test_skipped_window_step_zeroes_the_system_gradients_and_passes_the_rest_through():
    from banet_b200 import ops, _lib
    _lib.require_device()
    nf, K = 3, 8
    _, Hm, g, R, T, W = _built_pairs(nf, 8, K)
    Hm = Hm.clone(); Hm[1, 2, 2] = float("inf")                   # on the diagonal: status 2 only (off it, the factorisation also fails: 1)
    lam = torch.tensor([0.5], device="cuda")
    Rn, Tn, Wn, delta, status = ops.lm_window_solve_update(Hm, g, lam, R, T, W)
    assert status.tolist() == [2] * nf
    assert not bool(delta.any()) and torch.equal(Wn, W)
    gen = torch.Generator(device="cuda").manual_seed(8)
    dRn, dTn, dWn = (torch.randn(s, generator=gen, device="cuda") for s in ((nf, 3, 3), (nf, 3, 1), (K, 1)))
    dH, dg, dlam, dR, dT, dW = ops.lm_window_solve_update_bwd(Hm, g, lam, delta, R, T, dRn, dTn, dWn)
    assert not bool(dH.any()) and not bool(dg.any()) and not bool(dlam.any())
    assert torch.equal(dR, dRn) and torch.equal(dT, dTn) and torch.equal(dW, dWn)


def _net_and_inputs(nf=3, C=8, K=5, seed=91):
    from banet_b200.bundlenet import BundleNet
    from banet_b200 import _lib
    sc = scene_case(nb=nf, H=48, W=64, C=C, K=K, level_ids=(3,), seed=seed, n_points=500, shared_depth=True, dtype=torch.float32)
    lv = sc.levels[0]
    net = BundleNet(C, levels=("3",), exact_sym_grad=True, precision=_lib.PREC_FP32_SIMT, strict_status=True).cuda()
    for i, (w, b) in enumerate(mlp_for(C, 3)):
        getattr(net, f"lambda_3_{i + 1}_filters").data.copy_(w); getattr(net, f"lambda_3_{i + 1}_biases").data.copy_(b)
    x = dict(conv1=to_cuda32(lv.conv1), conv2=to_cuda32(lv.conv2), p=to_cuda32(lv.p), D=to_cuda32(lv.D), B=to_cuda32(lv.B),
             R=to_cuda32(sc.R0), T=to_cuda32(sc.T0), W=to_cuda32(sc.W0[0]) + 0.01)
    fx, fy, ox, oy = [to_cuda32(t) for t in lv.intr_tiled()]
    call = lambda d: net.WindowIteration(d["conv1"], d["conv2"], fx, fy, ox, oy, d["p"], d["D"], d["B"], d["R"], d["T"], d["W"], 1000.0, "3")
    return net, x, call


@pytest.mark.gpu
def test_window_iteration_grad_and_no_grad_paths_agree():
    from banet_b200 import _lib
    _lib.require_device()
    net, x, call = _net_and_inputs()
    with torch.no_grad():
        a = call(x)
    b = call({k: v.clone().requires_grad_() for k, v in x.items()})
    assert all(t.requires_grad for t in b) and not any(t.requires_grad for t in a)
    assert int(net.last_status.abs().max()) == 0
    for u, v in zip(a, b):
        assert rel_fro(u, v.detach()) < 1e-5


@pytest.mark.gpu
def test_window_iteration_strict_status_raises_on_a_skipped_step():
    from banet_b200 import _lib
    _lib.require_device()
    net, x, call = _net_and_inputs()
    x["conv1"] = x["conv1"].clone(); x["conv1"][0, 0, 0] = float("nan")
    with torch.no_grad(), pytest.raises(RuntimeError, match="skipped"):
        call(x)
    with pytest.raises(RuntimeError, match="skipped"):
        call({k: v.clone().requires_grad_() for k, v in x.items()})
    assert bool((net.last_status != 0).all())


@pytest.mark.gpu
def test_window_iteration_broadcast_keyframe_gets_the_frame_summed_gradient():
    from banet_b200 import _lib
    _lib.require_device()
    net, x, call = _net_and_inputs()
    nf = x["R"].shape[0]
    key = ("conv1", "p", "D", "B")
    once = {k: (v[:1].clone() if k in key else v.clone()).requires_grad_(k != "p") for k, v in x.items()}
    per_frame = {k: (v[:1].repeat(nf, *[1] * (v.dim() - 1)) if k in key else v.clone()).requires_grad_(k != "p") for k, v in x.items()}
    outs = [call(d) for d in (once, per_frame)]
    gen = torch.Generator(device="cuda").manual_seed(12)
    c = [torch.randn(t.shape, generator=gen, device="cuda") for t in outs[0]]
    for o in outs:
        sum((t * ci).sum() for t, ci in zip(o, c)).backward()
    for u, v in zip(outs[0], outs[1]):
        assert torch.equal(u, v)
    for k in ("conv1", "D", "B"):                                    # the build's backward accumulates with atomics: equal up to summation order
        assert rel_fro(once[k].grad[0], per_frame[k].grad.sum(0)) < 1e-5, k
    for k in ("conv2", "R", "T", "W"):
        assert rel_fro(once[k].grad, per_frame[k].grad) < 1e-5, k
