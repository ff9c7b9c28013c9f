"""bfloat16 feature maps (banet_level_t::feature_dtype = BANET_DTYPE_BF16): conv1 / conv2 read as bf16 by the build kernels, their
backward, BundleNet and the host pipeline.  bf16 -> fp32 is exact, so every run on bf16 features is checked against the same fp32 call on
the widened tensors (x.bfloat16().float()): bitwise where the kernel keeps the fp32 lane <-> channel map and summation order (the SIMT build,
the tensor-core build at C = 64), to fp32 rounding where it does not (the tensor-core build at C = 128 sums a lane's 8 contiguous channels).
CPU tests: argument checks through the loaded library."""
import ctypes

import pytest
import torch

from helpers import O, scene_case, oracle_level_inputs, mlp_for, rel_fro, to_cuda32
from banet_b200 import _lib

gpu = pytest.mark.gpu
BF = torch.bfloat16


# ------------------------------------------------------------------------------------------------ CPU: the C-ABI
def _level(**kw):
    lv = _lib.BanetLevel(2, 4096, 64, 0, 48, 64, 192, 1, 1, 1, 1, 1, 1, 0, 0)
    for k, v in kw.items():
        setattr(lv, k, v)
    return lv


def test_struct_built_without_the_field_keeps_fp32():
    assert _level().feature_dtype == _lib.DTYPE_F32 == 0
    assert _lib.DTYPE_BF16 == 1


def test_bad_feature_dtype_is_rejected():
    lib = _lib.load()
    for bad in (2, -1, 7):
        lv = _level(feature_dtype=bad)
        rc = lib.banet_lm_build(ctypes.byref(lv), 1, 1, None, 0, 1, 1, 1, 1, 1, 1 << 20, None)
        assert rc == -1 and b"feature_dtype" in lib.banet_last_error()
        arr = (_lib.BanetLevel * 1)(lv)
        rc = lib.banet_lm_run(arr, 1, 1, None, 1.0, 0.5, ctypes.byref(_lib.BanetSolveOpts(1e-5, 0, 0)), 0, 1, 1, None, 1, 1, 1 << 20, None)
        assert rc == -1 and b"feature_dtype" in lib.banet_last_error()


def test_legacy_tracker_rejects_bf16_levels():
    lib = _lib.load()
    arr = (_lib.BanetLevel * 1)(_level(feature_dtype=_lib.DTYPE_BF16))
    iters = (ctypes.c_int * 1)(3)
    opts = _lib.BanetLegacyOpts(1, 1e-5, 2e-4, 1.0)
    rc = lib.banet_lm_track_legacy(arr, 1, iters, None, ctypes.byref(opts), 1, 1, None, 1, 1, 1, 1 << 20, None)
    assert rc == -4 and b"bf16" in lib.banet_last_error()


# ------------------------------------------------------------------------------------------------ GPU helpers
def _widened(t):
    return t.to(BF).float()


def _build_case(C, K, points, layout, seed):
    """A seeded level on the GPU with its features rounded to bf16: (bf16 level, widened fp32 level, R, T, W)."""
    from banet_b200 import ops
    sc = scene_case(nb=2, H=48, W=64, C=C, K=K, level_ids=(3,), seed=seed, n_points=400 if points == "sparse" else None, dtype=torch.float32)
    lv = sc.levels[0]
    conv2 = lv.conv2 if layout == "3C" else lv.conv2[..., :C].contiguous()
    c1, c2 = lv.conv1.cuda().to(BF), conv2.cuda().to(BF)
    W = None if K == 0 else to_cuda32(sc.W0 + 0.01 * torch.randn(sc.W0.shape, generator=torch.Generator().manual_seed(seed)))
    rest = (to_cuda32(lv.intr), to_cuda32(lv.p), to_cuda32(lv.D), to_cuda32(lv.B))
    mk = lambda a, b: ops.Level(a, b, *rest, grid=lv.grid)
    return mk(c1, c2), mk(c1.float(), c2.float()), to_cuda32(sc.R0), to_cuda32(sc.T0), W


MODES = {"SIMT": _lib.PREC_FP32_SIMT, "X1": _lib.PREC_TF32X1, "X2": _lib.PREC_TF32X2, "X3": _lib.PREC_TF32X3, "AUTO": _lib.PREC_AUTO}


@gpu
@pytest.mark.parametrize("points", ["dense", "sparse"])
@pytest.mark.parametrize("layout", ["3C", "F2"])
@pytest.mark.parametrize("C", [64, 128])
@pytest.mark.parametrize("K", [128, 64, 32, 0])
@pytest.mark.parametrize("mode", list(MODES))
def test_build_matches_the_widened_fp32_build(mode, K, C, layout, points):
    from banet_b200 import ops
    _lib.require_device()
    if K == 0 and mode not in ("SIMT", "AUTO"):
        pytest.skip("the tensor-core modes need a depth basis")
    lb, lf, R, T, W = _build_case(C, K, points, layout, seed=7 * C + K)
    prec = MODES[mode]
    Hb, gb, rb, nb_ = ops.lm_build(lb, R, T, W, prec)
    Hf, gf, rf, nf_ = ops.lm_build(lf, R, T, W, prec)
    assert torch.equal(nb_, nf_) and float(nf_.min()) > 0
    tensor_cores = K > 0 and mode != "SIMT"
    if not tensor_cores or C == 64:              # the fp32 lane map and channel order: the same bits
        for a, b in ((Hb, Hf), (gb, gf), (rb, rf)):
            assert torch.equal(a, b)
    else:                                        # C = 128: a lane's 8 channels are contiguous, the per-pixel sums are reordered
        tol = 1e-6 if mode == "X3" or (mode == "AUTO" and lb.conv1.shape[1] < 65536) else 1e-5
        assert rel_fro(Hb, Hf) <= tol and rel_fro(gb, gf) <= tol
        assert rel_fro(rb, rf) <= 1e-6


@gpu
@pytest.mark.parametrize("layout", ["3C", "F2"])
@pytest.mark.parametrize("C,K", [(64, 128), (128, 128), (128, 0), (8, 16)])
def test_build_backward_matches_the_widened_backward(C, K, layout):
    """dconv1 / dconv2 come back fp32 for bf16 levels; every gradient equals the widened run's up to the order of the fp32 atomics."""
    from banet_b200 import ops
    _lib.require_device()
    lb, lf, R, T, W = _build_case(C, K, "sparse", layout, seed=3 + C + K)
    P = 6 + K
    g = torch.Generator(device="cuda").manual_seed(4)
    dH = torch.randn(2, P, P, device="cuda", generator=g); dg = torch.randn(2, P, device="cuda", generator=g)
    dr = torch.randn(2, C, device="cuda", generator=g)
    ob = ops.lm_build_bwd(lb, R, T, W, dH, dg, dr)
    of = ops.lm_build_bwd(lf, R, T, W, dH, dg, dr)
    assert ob[0].dtype == torch.float32 and ob[1].dtype == torch.float32 and ob[1].shape == lb.conv2.shape
    for a, b in zip(ob, of):
        if b is not None:
            assert rel_fro(a, b) <= 1e-5


@gpu
def test_mixed_feature_dtypes_are_rejected():
    from banet_b200 import ops
    c1 = torch.zeros(1, 4, 8, device="cuda", dtype=BF); c2 = torch.zeros(1, 4, 4, 8, device="cuda")
    lv = ops.Level(c1, c2, torch.zeros(1, 4, device="cuda"), torch.zeros(1, 3, 4, device="cuda"), torch.zeros(1, 4, 1, device="cuda"), None)
    with pytest.raises(_lib.BanetError, match="conv1.*conv2"):
        lv.as_struct()


@gpu
def test_resample_bf16_is_the_fp32_resample_rounded():
    from banet_b200 import ops
    _lib.require_device()
    g = torch.Generator(device="cuda").manual_seed(2)
    data = torch.randn(3, 20, 30, 64, device="cuda", generator=g).to(BF)
    xy = torch.rand(3, 500, 2, device="cuda", generator=g) * torch.tensor([34.0, 24.0], device="cuda") - 2.0
    out = ops.resample(data, xy, 1.0)
    assert out.dtype == BF
    assert torch.equal(out, ops.resample(data.float(), xy, 1.0).to(BF))


def _run_scene(nb, C, K, seed, levels=(0, 1, 2, 3), layout="F2", **kw):
    from banet_b200 import ops, synth
    sc = synth.make_scene(nb=nb, H=96, W=128, C=C, K=K, level_ids=levels, seed=seed, device="cuda", **kw)
    mk = lambda l, dt: ops.Level(l.conv1.to(dt), (l.conv2 if layout == "3C" else l.conv2[..., :C].contiguous()).to(dt), l.intr, l.p, l.D, l.B,
                                 grid=l.grid)
    lb = [mk(l, BF) for l in sc.levels]
    lf = [ops.Level(l.conv1.float(), l.conv2.float(), l.intr, l.p, l.D, l.B, grid=l.grid) for l in lb]
    return sc, lb, lf


def _mlps(C, n, seed=9):
    from banet_b200 import ops
    g = torch.Generator().manual_seed(seed)
    dims = [C, 2 * C, 4 * C, 2 * C, C, 1]
    return [ops.pack_mlp([(torch.randn(dims[i], dims[i + 1], generator=g) * (2.0 / dims[i]) ** 0.5, torch.zeros(dims[i + 1])) for i in range(5)]).cuda()
            for _ in range(n)]


@gpu
@pytest.mark.parametrize("layout", ["3C", "F2"])
def test_lm_run_matches_the_widened_run(layout):
    from banet_b200 import ops
    _lib.require_device()
    sc, lb, lf = _run_scene(4, 128, 128, seed=13, layout=layout)
    mlps = _mlps(128, 4)
    Rb, Tb, Wb, sb = ops.lm_run(lb, 2, sc.R0, sc.T0, sc.W0, mlp_packed=mlps, l2_regularizer_base=1000.0)
    Rf, Tf, Wf, sf = ops.lm_run(lf, 2, sc.R0, sc.T0, sc.W0, mlp_packed=mlps, l2_regularizer_base=1000.0)
    assert int(sb.abs().max()) == 0 and int(sf.abs().max()) == 0
    assert rel_fro(Rb, Rf) < 1e-4 and rel_fro(Tb, Tf) < 1e-4 and rel_fro(Wb, Wf) < 1e-4


@gpu
def test_lm_window_batch_run_matches_the_widened_run():
    from banet_b200 import ops, synth
    _lib.require_device()
    nw, nf, C, K = 2, 3, 64, 128
    sc = synth.make_scene(nb=nw * nf, H=96, W=128, C=C, K=K, level_ids=(2, 3), seed=17, device="cuda", shared_depth=True, window_frames=nf)
    lb = [ops.Level(l.conv1.to(BF), l.conv2[..., :C].contiguous().to(BF), l.intr, l.p, l.D, l.B, grid=l.grid) for l in sc.levels]
    lf = [ops.Level(l.conv1.float(), l.conv2.float(), l.intr, l.p, l.D, l.B, grid=l.grid) for l in lb]
    W0 = sc.W0.reshape(nw, nf, K, 1)[:, 0].contiguous()
    mlps = _mlps(C, 2)
    out_b = ops.lm_window_batch_run(lb, nw, 2, sc.R0, sc.T0, W0, mlp_packed=mlps)
    out_f = ops.lm_window_batch_run(lf, nw, 2, sc.R0, sc.T0, W0, mlp_packed=mlps)
    assert int(out_b[3].abs().max()) == 0
    for a, b in zip(out_b[:3], out_f[:3]):
        assert rel_fro(a, b) < 1e-4


@gpu
def test_bf16_solve_is_bit_reproducible_from_poisoned_workspaces():
    from banet_b200 import ops
    _lib.require_device()
    sc, lb, _ = _run_scene(4, 128, 128, seed=19)
    mlps = _mlps(128, 4)
    outs = []
    for _ in range(2):
        ws = torch.empty(ops.lm_run_workspace_bytes(lb), dtype=torch.uint8, device="cuda")
        ws.view(torch.float32)[: ws.numel() // 4].fill_(float("nan"))
        outs.append(ops.lm_run(lb, 2, sc.R0, sc.T0, sc.W0, mlp_packed=mlps, l2_regularizer_base=1000.0, workspace=ws))
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)


@gpu
def test_planted_solution_converges_on_bf16_features():
    """The accuracy cost of storing the features in bf16: the planted-solution solve of tests/test_oracle_consistency.py (3 levels, 5
    iterations each, lambda 1e-2) on bf16 F2 features next to fp32 3C features.  Rounding the features moves the minimum by about the bf16
    rounding (2^-9 relative), so the bf16 solve still lands near the planted pose and W."""
    from banet_b200 import ops
    _lib.require_device()
    sc = scene_case(nb=2, H=96, W=128, C=8, K=4, level_ids=(1, 2, 3), seed=3, dtype=torch.float32)
    cu = lambda t: None if t is None else t.cuda()
    errs = {}
    for name, dt, layout in (("fp32 3C", torch.float32, "3C"), ("bf16 F2", BF, "F2")):
        levels = [ops.Level(cu(l.conv1).to(dt), cu(l.conv2 if layout == "3C" else l.conv2[..., :8].contiguous()).to(dt), cu(l.intr), cu(l.p),
                            cu(l.D), cu(l.B), grid=l.grid) for l in sc.levels]
        R, T, W, st = ops.lm_run(levels, 5, cu(sc.R0), cu(sc.T0), cu(sc.W0), lambda_fixed=0.01, precision=_lib.PREC_FP32_SIMT)
        assert int(st.abs().max()) == 0
        errs[name] = [float((x.cpu() - y).norm()) for x, y in ((R, sc.R_true), (T, sc.T_true), (W, sc.W_true))]
    start = [float((x - y).norm()) for x, y in ((sc.R0, sc.R_true), (sc.T0, sc.T_true), (sc.W0, sc.W_true))]
    print("planted-solution errors |R - R*|, |T - T*|, |W - W*|: start", start, errs)
    for i in range(3):
        assert errs["fp32 3C"][i] < 0.01 * start[i] + 1e-5
        assert errs["bf16 F2"][i] < 0.05 * start[i] + 1e-4


# ------------------------------------------------------------------------------------------------ GPU: BundleNet and training
def _net(C, levels, **kw):
    from banet_b200.bundlenet import BundleNet
    kw.setdefault("strict_status", True)
    return BundleNet(C, levels=levels, **kw).cuda()


@gpu
@pytest.mark.parametrize("layout", ["3C", "F2"])
def test_bundle_iteration_takes_bf16_features(layout):
    from banet_b200.bundlenet import BundleNet
    _lib.require_device()
    sc, lb, lf = _run_scene(2, 64, 32, seed=29, levels=(3,), layout=layout)
    net = _net(64, ("3",)).eval()
    fx, fy, ox, oy = [sc.levels[0].intr[:, i:i + 1] for i in range(4)]
    args = lambda lv: (lv.conv1, lv.conv2, fx, fy, ox, oy, lv.p, lv.D, lv.B, sc.R0, sc.T0, sc.W0, 1000.0, "3")
    with torch.no_grad():
        ob = net.BundleIteration(*args(lb[0])); of = net.BundleIteration(*args(lf[0]))
    for a, b in zip(ob, of):
        assert rel_fro(a, b) < 1e-4


@gpu
def test_training_gradients_reach_bf16_features_in_bf16():
    """iteration_fused on bf16 features: the feature gradients are the widened run's gradients rounded to bf16 (within one bf16 ulp: the
    backward's atomics reorder the fp32 sums); R, T, W, D, B get the widened run's fp32 gradients."""
    from banet_b200 import autograd as ag
    _lib.require_device()
    C, K = 64, 32
    lb, lf, R, T, W = _build_case(C, K, "sparse", "F2", seed=37)
    mlp = [(w.cuda().float(), b.cuda().float()) for w, b in mlp_for(C, 3)]
    g = torch.Generator(device="cuda").manual_seed(6)
    cR, cT, cW = (torch.randn(s, device="cuda", generator=g) for s in ((2, 3, 3), (2, 3, 1), (2, K, 1)))

    def run(lv):
        ins = [t.detach().clone().requires_grad_() for t in (lv.conv1, lv.conv2, lv.D, lv.B, R, T, W)]
        Rn, Tn, Wn = ag.iteration_fused(ins[0], ins[1], lv.intr, lv.p, ins[2], ins[3], ins[4], ins[5], ins[6], mlp, 1000.0)
        ((Rn * cR).sum() + (Tn * cT).sum() + (Wn * cW).sum()).backward()
        return [t.grad for t in ins]

    gb, gf = run(lb), run(lf)
    for i in (0, 1):
        assert gb[i].dtype == BF
        ref = gf[i].to(BF).float()
        ulp = torch.where(ref != 0, ref.abs() * 2.0 ** -7, torch.full_like(ref, 1e-30))
        assert bool(((gb[i].float() - ref).abs() <= ulp + 1e-6 * ref.abs().max()).all())
    for a, b in zip(gb[2:], gf[2:]):
        assert a.dtype == torch.float32 and rel_fro(a, b) < 1e-5


@gpu
def test_bf16_training_gradients_match_the_float64_oracle():
    """One iteration on a small widened case: bf16 features through BundleNet's fused training path against float64 autograd of the oracle
    on the same (widened) features.  The feature gradients are stored in bf16 (relative rounding 2^-9)."""
    _lib.require_device()
    C, K = 8, 6
    sc = scene_case(nb=2, C=C, K=K, level_ids=(3,), seed=61, n_points=400, dtype=torch.float32)
    lv = sc.levels[0]
    mlp = mlp_for(C, 3)
    a = oracle_level_inputs(lv)
    a["conv1"] = _widened(a["conv1"]).double(); a["conv2"] = _widened(a["conv2"]).double()
    names = ["conv1", "conv2", "D", "B"]
    for n in names:
        a[n] = a[n].clone().requires_grad_()
    R = sc.R0.double().clone().requires_grad_(); T = sc.T0.double().clone().requires_grad_(); W = (sc.W0.double() + 0.01).clone().requires_grad_()
    gen = torch.Generator().manual_seed(5)
    cR, cT, cW = (torch.randn(s, generator=gen, dtype=torch.float64) for s in ((2, 3, 3), (2, 3, 1), (2, K, 1)))
    oR, oT, oW = O.bundle_iteration(a["conv1"], a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"], R, T, W,
                                    [(w.clone(), b.clone()) for w, b in mlp],
                                    O.IterOptions(l2_regularizer_base=1000.0, guard_nonfinite=True, reference_op_grad=True))
    ((oR * cR).sum() + (oT * cT).sum() + (oW * cW).sum()).backward()
    net = _net(C, ("3",), precision=_lib.PREC_FP32_SIMT)
    for i, (w, b) in enumerate(mlp):
        getattr(net, f"lambda_3_{i + 1}_filters").data.copy_(w); getattr(net, f"lambda_3_{i + 1}_biases").data.copy_(b)
    t = {n: (a[n].detach().cuda().to(BF) if n.startswith("conv") else to_cuda32(a[n].detach())).requires_grad_() for n in names}
    Rg, Tg, Wg = (to_cuda32(x.detach()).requires_grad_() for x in (R, T, W))
    fx, fy, ox, oy = [to_cuda32(x) for x in lv.intr_tiled()]
    gR, gT, gW = net.BundleIteration(t["conv1"], t["conv2"], fx, fy, ox, oy, to_cuda32(lv.p), t["D"], t["B"], Rg, Tg, Wg, 1000.0, "3")
    assert rel_fro(gR, oR) < 1e-5 and rel_fro(gT, oT) < 1e-4 and rel_fro(gW, oW) < 1e-4
    ((gR * cR.float().cuda()).sum() + (gT * cT.float().cuda()).sum() + (gW * cW.float().cuda()).sum()).backward()
    for n in names:
        tol = 8e-3 if n.startswith("conv") else 1e-3
        assert t[n].grad.dtype == t[n].dtype and rel_fro(t[n].grad.double().cpu(), a[n].grad) < tol, n
    for x, y in ((Rg, R), (Tg, T), (Wg, W)):
        assert rel_fro(x.grad.double().cpu(), y.grad) < 1e-3


def _resize_inputs(nimg, C, K, seed):
    from banet_b200 import synth
    sc = synth.make_resize_scene(nimg, 96, 128, C, K, level_ids=(2, 3), seed=seed, device="cuda")
    return sc, [l.to(BF) for l in sc.layers]


@gpu
@pytest.mark.parametrize("grad", [False, True])
def test_bundle_and_camera_resize_on_a_bf16_pyramid(grad):
    """BundleResize / CameraResize on a bf16 pyramid against the same calls on the widened pyramid.  The two routes differ only by the
    bf16 rounding of the resampled conv1 (at most 2^-9 relative per element) and by F2 with on-the-fly gradients in place of the
    materialised 3C map (the same values, summed in another order); the poses and depths move by a small fraction of that rounding."""
    import gen_golden
    _lib.require_device()
    x = gen_golden.resize_inputs(nb=4, C=16, K=8)
    C = 16
    net = _net(C, ("0", "1", "2", "3"), strict_status=False)
    net.train(grad)
    f32 = {k: to_cuda32(x[k]) for k in ("intr", "points", "basis", "depth", "R0", "T0")}

    def call(layers):
        ls = [l.detach().clone().requires_grad_(grad) for l in layers]
        b = f32["basis"].clone().requires_grad_(grad)
        with torch.set_grad_enabled(grad):
            Rs, Ts, Ds = net.BundleResize(f32["intr"], ls, f32["points"], b, f32["depth"], f32["R0"], f32["T0"])
            cR, cT = net.CameraResize(f32["intr"], ls, f32["points"], f32["depth"])
            if grad:
                (sum(r.sum() for r in Rs + cR) + sum(t.sum() for t in Ts + cT) + sum(d.sum() for d in Ds)).backward()
        return Rs + cR, Ts + cT, Ds, ls, b

    lb = [to_cuda32(l).to(BF) for l in x["layers"]]
    Rb, Tb, Db, lsb, bb = call(lb)
    Rf, Tf, Df, lsf, bf = call([l.float() for l in lb])
    for xs, ys in ((Rb, Rf), (Tb, Tf), (Db, Df)):
        for u, v in zip(xs, ys):
            assert u.dtype == torch.float32 and rel_fro(u, v) < 1e-3
    if grad:
        for u, v in zip(lsb, lsf):
            assert u.grad.dtype == BF and rel_fro(u.grad.float(), v.grad) < 5e-2
        assert bb.grad.dtype == torch.float32 and rel_fro(bb.grad, bf.grad) < 5e-2


@gpu
def test_keyframe_forms_reject_bf16():
    from banet_b200 import ops
    _lib.require_device()
    nw, nf, N, C, K = 1, 2, 64, 8, 4
    z = lambda *s, dt=torch.float32: torch.zeros(*s, device="cuda", dtype=dt)
    kl = ops.KeyframeLevel(z(nw, N, C, dt=BF), z(nw * nf, 8, 8, C, dt=BF), z(nw * nf, 4), z(nw, 3, N), z(nw, N, 1), z(nw, N, K))
    with pytest.raises(_lib.BanetError, match="float32"):
        kl.as_struct()
    net = _net(C, ("3",)).eval()
    with pytest.raises(RuntimeError, match="float32"):
        net.WindowIteration(z(nw, N, C, dt=BF), z(nw, nf, 8, 8, C, dt=BF), *[z(nw, 1, 1)] * 4, z(nw, 3, N), z(nw, N, 1), z(nw, N, K),
                            torch.eye(3, device="cuda").repeat(nw, nf, 1, 1), z(nw, nf, 3, 1), z(nw, K, 1), 1000.0, "3")


@gpu
@pytest.mark.parametrize("chunks", [2, 4])
def test_resize_host_solver_keeps_a_bf16_pyramid(chunks):
    """A bf16 host pyramid stays bf16 on the device (2 bytes per element over PCIe) and solves like the device-level lm_run on the same bf16
    levels (tolerance of the fp32 pipeline test: a different batch per call reorders the fp32 partial sums)."""
    from banet_b200 import ops
    from banet_b200.host_pipeline import ResizeHostSolver
    _lib.require_device()
    nimg, C, K = 8, 64, 128
    sc, lb = _resize_inputs(nimg, C, K, seed=41)
    scales = sc.scales
    pin = lambda t: t.cpu().pin_memory()
    hs = ResizeHostSolver([pin(l) for l in lb], pin(sc.basis), pin(sc.init_depth), pin(sc.intr), scales, chunks=chunks, precision=0)
    assert all(d.dtype == BF for d in hs.d_layers)
    assert hs.h2d_bytes == 2 * sum(l.numel() for l in lb) + 4 * (sc.basis.numel() + sc.init_depth.numel() + sc.intr.numel())
    R, T, W, st = hs.solve(pin(sc.R0), pin(sc.T0), pin(sc.W0), 4, lambda_fixed=0.5)
    torch.cuda.synchronize()
    assert int(st.abs().max()) == 0
    half = nimg // 2
    levels = []
    for lay, s in zip(lb, scales):
        h, w = lay.shape[1], lay.shape[2]
        vv, uu = torch.meshgrid(torch.arange(h, device="cuda", dtype=torch.float32), torch.arange(w, device="cuda", dtype=torch.float32), indexing="ij")
        pts = torch.stack([uu.reshape(-1), vv.reshape(-1)], -1).unsqueeze(0).repeat(nimg, 1, 1).contiguous()
        intr_l = sc.intr / s
        levels.append(ops.Level(lay.reshape(nimg, h * w, C), torch.cat([lay[half:], lay[:half]], 0).contiguous(), intr_l,
                                ops.compute_coordinates(pts, intr_l, True), ops.resample(sc.init_depth, pts, s / 2.0),
                                ops.resample(sc.basis, pts, s / 2.0), grid=(w, h)))
    R1, T1, W1, st1 = ops.lm_run(levels, 4, sc.R0, sc.T0, sc.W0, lambda_fixed=0.5, precision=0)
    assert rel_fro(R, R1) < 2e-5 and rel_fro(T, T1) < 1e-3 and rel_fro(W, W1) < 5e-3
