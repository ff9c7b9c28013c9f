"""Training on the F2-only feature layout: banet_lm_build_bwd with conv2 [nb,h,w,C], whose gradient channels the build derives on the fly
with the REFLECT-by-one stencil.  The backward of that layout must be the adjoint of the stencil: the 3C backward followed by
grad_fixed_concat_bwd, which is what a user gets by materialising [F2|gx|gy] with autograd.grad_fixed_concat.  Checked kernel against
kernel (every gradient, border points included), layer against the float64 oracle (both training paths), on the window forms, behind the
tensor-core forward, and for the memory it saves."""
import pytest
import torch

from helpers import O, scene_case, oracle_level_inputs, mlp_for, rel_fro, to_cuda32

pytestmark = pytest.mark.gpu


def _border_level(nb, C, K, h=24, w=32, seed=0):
    """A level whose projections are exact in fp32 (R = I, T = 0, W = 0, D = 1, fx = fy = 1, ox = oy = 0, p = (u, v, 1)): the kernel's
    u, v are the p given.  The points fill the border band (x0 = 0, x1 = w-1 and the same in y), sit exactly on u = w-1 and v = h-1
    (where the tap clamps), on u = 0 and v = 0, and in the interior."""
    g = torch.Generator().manual_seed(seed)
    edge_u = torch.tensor([0.0, 0.25, 0.75, w - 2.0, w - 1.75, w - 1.25, w - 1.0, w - 1.0, 0.0, w - 1.0])
    edge_v = torch.tensor([h - 1.0, 0.5, h - 1.0, 0.0, 0.25, h - 1.5, 3.5, h - 1.0, 0.0, 0.5])
    n_in = 200
    u = torch.cat([edge_u, torch.rand(n_in, generator=g) * (w - 1), torch.rand(n_in, generator=g) * (w - 1)])
    v = torch.cat([edge_v, torch.rand(n_in, generator=g) * (h - 1), torch.cat([torch.rand(n_in // 2, generator=g) * 1.0,
                                                                               h - 2 + torch.rand(n_in // 2, generator=g)])])
    N = u.numel()
    p = torch.stack([u, v, torch.ones(N)]).unsqueeze(0).repeat(nb, 1, 1)
    F2 = torch.randn(nb, h, w, C, generator=g)
    conv1 = torch.randn(nb, N, C, generator=g)
    D = torch.ones(nb, N, 1)
    B = torch.randn(nb, N, K, generator=g) if K else None
    W = torch.zeros(nb, K, 1) if K else None
    intr = torch.tensor([1.0, 1.0, 0.0, 0.0]).repeat(nb, 1)
    R, T = torch.eye(3).repeat(nb, 1, 1), torch.zeros(nb, 3, 1)
    x0, y0 = u.floor(), v.floor()
    assert bool(((x0 == 0) & (y0 == 0)).any()) and bool(((x0 == w - 2) | (u == w - 1)).any()) and bool((u == w - 1).any())
    assert bool((v == h - 1).any()) and bool(((u == w - 1) & (v == h - 1)).any()) and bool(((y0 == 0) & (x0 > 0)).any())
    assert bool(((x0 >= 1) & (x0 + 2 <= w - 1) & (y0 >= 1) & (y0 + 2 <= h - 1)).any())
    return F2, conv1, intr, p, D, B, R, T, W, None


def _scene_level(nb, C, K, points, seed):
    sc = scene_case(nb=nb, H=48, W=64, C=C, K=K, level_ids=(3,), seed=seed, n_points=400 if points == "sparse" else None, dtype=torch.float32)
    lv = sc.levels[0]
    W = None if K == 0 else sc.W0 + 0.01 * torch.randn(sc.W0.shape, generator=torch.Generator().manual_seed(seed))
    return lv.conv2[..., :C].contiguous(), lv.conv1, lv.intr, lv.p, lv.D, lv.B, sc.R0, sc.T0, W, lv.grid


@pytest.mark.parametrize("exact", [0, 1])
@pytest.mark.parametrize("K", [0, 16, 128, 200])
@pytest.mark.parametrize("C", [5, 8, 64, 128])
@pytest.mark.parametrize("points", ["sparse", "dense", "border"])
def test_f2_backward_is_the_adjoint_of_the_stencil(points, C, K, exact):
    """dF2 of the F2-only backward == grad_fixed_concat_bwd of the 3C backward's dconv2; every other gradient equal to the 3C one."""
    from banet_b200 import ops, _lib
    _lib.require_device()
    nb = 2
    if points == "border":
        F2, conv1, intr, p, D, B, R, T, W, grid = _border_level(nb, C, K, seed=C + K)
    else:
        F2, conv1, intr, p, D, B, R, T, W, grid = _scene_level(nb, C, K, points, seed=31 + C + K)
    cu = to_cuda32
    F2, conv1, intr, p, D, B, R, T, W = (cu(t) for t in (F2, conv1, intr, p, D, B, R, T, W))
    conv2 = ops.grad_fixed_concat(F2)
    P = 6 + K
    gen = torch.Generator(device="cuda").manual_seed(K + C)
    dH = torch.randn(nb, P, P, generator=gen, device="cuda")
    dg = torch.randn(nb, P, generator=gen, device="cuda")
    dr = torch.randn(nb, C, generator=gen, device="cuda")
    lv3 = ops.Level(conv1, conv2, intr, p, D, B, grid=grid)
    lv1 = ops.Level(conv1, F2, intr, p, D, B, grid=grid)
    _, _, _, nvalid = ops.lm_build(lv1, R, T, W, _lib.PREC_FP32_SIMT)
    assert float(nvalid.min()) > 0
    r3 = ops.lm_build_bwd(lv3, R, T, W, dH, dg, dr, bool(exact))
    r1 = ops.lm_build_bwd(lv1, R, T, W, dH, dg, dr, bool(exact))
    assert r1[1].shape == F2.shape
    assert rel_fro(r1[1], ops.grad_fixed_concat_bwd(r3[1])) <= 1e-5
    for name, a, b in zip(("dconv1", "dD", "dB", "dR", "dT", "dW"), (r1[0],) + r1[2:], (r3[0],) + r3[2:]):
        if b is None:
            assert a is None and K == 0, name
            continue
        assert rel_fro(a, b) <= 1e-5, name


@pytest.mark.parametrize("path", ["fused", "reference_split"])
@pytest.mark.parametrize("K,exact", [(6, False), (0, False), (6, True), (0, True)])
def test_f2_iteration_gradients_match_oracle_autograd(K, exact, path):
    """BundleIteration / CameraIteration with an F2-only conv2 against the oracle on cat([F2, grad_fixed(F2)]), F2 the leaf on both sides."""
    from banet_b200.bundlenet import BundleNet
    from banet_b200 import _lib
    _lib.require_device()
    C = 8
    sc = scene_case(nb=2, C=C, K=K, level_ids=(3,), seed=61, n_points=400, dtype=torch.float32)
    lv = sc.levels[0]
    mlp = mlp_for(C, 3)
    a = oracle_level_inputs(lv)
    a["F2"] = a.pop("conv2")[..., :C].contiguous()
    names = ["conv1", "F2", "D"] + (["B"] if K else [])
    for n in names:
        a[n] = a[n].clone().requires_grad_()
    conv2_o = torch.cat([a["F2"], O.grad_fixed(a["F2"])], dim=-1)
    R = sc.R0.double().clone().requires_grad_(); T = sc.T0.double().clone().requires_grad_()
    W = (sc.W0.double() + 0.01).clone().requires_grad_() if K else None
    mlp64 = [(w.clone().requires_grad_(), b.clone().requires_grad_()) for w, b in mlp]
    g = torch.Generator().manual_seed(5)
    cR, cT = torch.randn(2, 3, 3, generator=g, dtype=torch.float64), torch.randn(2, 3, 1, generator=g, dtype=torch.float64)
    cW = torch.randn(2, K, 1, generator=g, dtype=torch.float64) if K else None
    if K:
        oR, oT, oW = O.bundle_iteration(a["conv1"], conv2_o, a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"], R, T, W, mlp64,
                                        O.IterOptions(l2_regularizer_base=1000.0, guard_nonfinite=True, reference_op_grad=not exact))
        loss = (oR * cR).sum() + (oT * cT).sum() + (oW * cW).sum()
    else:
        oR, oT = O.camera_iteration(a["conv1"], conv2_o, a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], R, T, mlp64,
                                    O.IterOptions(guard_nonfinite=True, reference_op_grad=not exact))
        loss = (oR * cR).sum() + (oT * cT).sum()
    loss.backward()
    net = BundleNet(C, levels=("3",), exact_sym_grad=exact, training_path=path, precision=_lib.PREC_FP32_SIMT, strict_status=True).cuda()
    for i, (w, b) in enumerate(mlp):
        getattr(net, f"lambda_3_{i + 1}_filters").data.copy_(w); getattr(net, f"lambda_3_{i + 1}_biases").data.copy_(b)
    t = {n: to_cuda32(a[n].detach()).requires_grad_() for n in names}
    Rg = to_cuda32(sc.R0).requires_grad_(); Tg = to_cuda32(sc.T0).requires_grad_()
    Wg = to_cuda32(sc.W0 + 0.01).requires_grad_() if K else None
    fx, fy, ox, oy = [to_cuda32(x) for x in lv.intr_tiled()]
    if K:
        gR, gT, gW = net.BundleIteration(t["conv1"], t["F2"], fx, fy, ox, oy, to_cuda32(lv.p), t["D"], t["B"], Rg, Tg, Wg, 1000.0, "3")
        lossg = (gR * cR.float().cuda()).sum() + (gT * cT.float().cuda()).sum() + (gW * cW.float().cuda()).sum()
        assert rel_fro(gW, oW) < 1e-4
    else:
        gR, gT = net.CameraIteration(t["conv1"], t["F2"], fx, fy, ox, oy, to_cuda32(lv.p), t["D"], Rg, Tg, 1.0, "3")
        lossg = (gR * cR.float().cuda()).sum() + (gT * cT.float().cuda()).sum()
    assert rel_fro(gR, oR) < 1e-5 and rel_fro(gT, oT) < 1e-4
    lossg.backward()
    tol = 2e-3
    for n in names:
        assert rel_fro(t[n].grad, a[n].grad) < tol, n
    assert rel_fro(Rg.grad, R.grad) < tol and rel_fro(Tg.grad, T.grad) < tol
    if K:
        assert rel_fro(Wg.grad, W.grad) < tol
    for i, (w64, b64) in enumerate(mlp64):
        assert rel_fro(getattr(net, f"lambda_3_{i + 1}_filters").grad, w64.grad) < tol
        assert rel_fro(getattr(net, f"lambda_3_{i + 1}_biases").grad, b64.grad) < 5 * tol


def _mlp_leaves(C, seed=7):
    g = torch.Generator().manual_seed(seed); dims = [C, 2 * C, 4 * C, 2 * C, C, 1]
    return [((torch.randn(dims[i], dims[i + 1], generator=g) * (2.0 / dims[i]) ** 0.5).cuda().requires_grad_(),
             torch.zeros(dims[i + 1], device="cuda").requires_grad_()) for i in range(5)]


@pytest.mark.parametrize("form", ["batch", "single"])
def test_f2_window_iterations_match_the_3c_route(form):
    """window_batch_iteration_fused (per-frame form, conv2 [nw,nf,h,w,C]) and window_iteration_fused (conv2 [nf,h,w,C]) against the same
    call on [F2|gx|gy] built by autograd.grad_fixed_concat."""
    from banet_b200 import autograd as ag, _lib
    _lib.require_device()
    nw, nf, C, K = (3, 4, 16, 12) if form == "batch" else (1, 4, 16, 12)
    sc = scene_case(nb=nw * nf, C=C, K=K, level_ids=(3,), seed=43, n_points=300, dtype=torch.float32, shared_depth=True, window_frames=nf)
    lv = sc.levels[0]
    mlp = _mlp_leaves(C)
    leaf = lambda t: to_cuda32(t).requires_grad_()
    shape = (lambda t: t.reshape(nw, nf, *t.shape[1:])) if form == "batch" else (lambda t: t)
    F2 = leaf(shape(lv.conv2[..., :C]))
    conv1, D, B, R, T = (leaf(shape(t)) for t in (lv.conv1, lv.D, lv.B, sc.R0, sc.T0))
    W = leaf(sc.W0.reshape(nw, nf, K, 1)[:, 0] + 0.01) if form == "batch" else leaf(sc.W0[0] + 0.01)
    intr, p = to_cuda32(shape(lv.intr)), to_cuda32(shape(lv.p))
    fn = ag.window_batch_iteration_fused if form == "batch" else ag.window_iteration_fused
    leaves = [F2, conv1, D, B, R, T, W, *[x for wb in mlp for x in wb]]

    def run(route):
        for x in leaves:
            x.grad = None
        if route == "f2":
            conv2 = F2
        else:
            conv2 = ag.grad_fixed_concat(F2.reshape(-1, *F2.shape[-3:])).reshape(*F2.shape[:-1], 3 * C)
        out = fn(conv1, conv2, intr, p, D, B, R, T, W, mlp, 1000.0)
        (out[0].sum() + out[1].sum() + (out[2] * out[2]).sum()).backward()
        return [o.detach().clone() for o in out], [x.grad.clone() for x in leaves]

    (o1, g1), (o3, g3) = run("f2"), run("3c")
    for a, b in zip(o1, o3):
        assert rel_fro(a, b) < 1e-5
    for i, (a, b) in enumerate(zip(g1, g3)):
        assert rel_fro(a, b) < 1e-4, i


def test_f2_training_behind_the_tensor_core_forward():
    """iteration_fused at AUTO on a dense grid (C=64, K=128: the tensor-core build on both layouts): the F2 route's gradients equal the 3C
    route's."""
    from banet_b200 import autograd as ag, _lib
    _lib.require_device()
    C, K, nb = 64, 128, 2
    sc = scene_case(nb=nb, C=C, K=K, level_ids=(3,), seed=52, dtype=torch.float32)
    lv = sc.levels[0]
    assert lv.grid is not None
    intr, p = to_cuda32(lv.intr), to_cuda32(lv.p)
    mlp = _mlp_leaves(C, seed=9)
    leaf = lambda t: to_cuda32(t).requires_grad_()
    F2, conv1, D, B, R, T, W = (leaf(t) for t in (lv.conv2[..., :C], lv.conv1, lv.D, lv.B, sc.R0, sc.T0, sc.W0 + 0.01))
    leaves = [F2, conv1, D, B, R, T, W, *[x for wb in mlp for x in wb]]

    def run(route):
        for x in leaves:
            x.grad = None
        conv2 = F2 if route == "f2" else ag.grad_fixed_concat(F2)
        out = ag.iteration_fused(conv1, conv2, intr, p, D, B, R, T, W, mlp, 1000.0, precision=_lib.PREC_AUTO, grid=lv.grid)
        (out[0].sum() + out[1].sum() + (out[2] * out[2]).sum()).backward()
        return [o.detach().clone() for o in out], [x.grad.clone() for x in leaves]

    (o1, g1), (o3, g3) = run("f2"), run("3c")
    for a, b in zip(o1, o3):
        assert rel_fro(a, b) < 1e-4
    for i, (a, b) in enumerate(zip(g1, g3)):
        assert rel_fro(a, b) < 1e-4, i


def test_f2_training_saves_a_3c_tensor_of_peak_memory():
    """Dense 320x240, nb=4, C=128: one F2-route training iteration peaks below the 3C route by at least one [nb,h,w,3C] tensor."""
    from banet_b200 import autograd as ag, synth, _lib
    _lib.require_device()
    nb, C, K = 4, 128, 128
    sc = synth.make_scene(nb=nb, H=240, W=320, C=C, K=K, level_ids=(3,), seed=8, device="cuda", dtype=torch.float32)
    lv = sc.levels[0]
    leaf = lambda t: t.detach().clone().requires_grad_()
    F2 = leaf(lv.conv2[..., :C].contiguous())
    conv1, D, B, R, T, W = (leaf(t) for t in (lv.conv1, lv.D, lv.B, sc.R0, sc.T0, sc.W0 + 0.01))
    mlp = _mlp_leaves(C)
    leaves = [F2, conv1, D, B, R, T, W, *[x for wb in mlp for x in wb]]

    def peak(route):
        for x in leaves:
            x.grad = None
        torch.cuda.synchronize(); torch.cuda.empty_cache(); torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        conv2 = F2 if route == "f2" else ag.grad_fixed_concat(F2)
        out = ag.iteration_fused(conv1, conv2, lv.intr, lv.p, D, B, R, T, W, mlp, 1000.0, grid=lv.grid)
        (out[0].sum() + out[1].sum() + (out[2] * out[2]).sum()).backward()
        del conv2, out
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    p3, p1 = peak("3c"), peak("f2")
    assert p3 - p1 >= nb * 240 * 320 * 3 * C * 4, (p3, p1)
