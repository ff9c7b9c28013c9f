"""Per-point confidence weights of the normal equations (banet_level_t::weight): H = sum_n w_n J_n^T M_n J_n, g = sum_n w_n J_n^T q_n, with
the mean |residual| (lambda) and the in-bounds count unweighted.  The float64 statement (tests/weighted_oracle.py) is tied to the oracle on
the CPU; the build kernels, their backward, the whole solves and BundleNet are held to it on the GPU.  Weights of ones must give the
unweighted bits in every precision mode (x * 1.0f is exact)."""
import ctypes

import pytest
import torch

from helpers import O, scene_case, oracle_level_inputs, mlp_for, rel_fro, to_cuda32
import weighted_oracle as WO
from banet_b200 import _lib

gpu = pytest.mark.gpu
BF = torch.bfloat16


# ------------------------------------------------------------------------------------------------ CPU: the weighted statement
def _oracle_case(K, seed=3, n_points=300):
    sc = scene_case(nb=2, C=8, K=K, level_ids=(3,), seed=seed, n_points=n_points)
    a = oracle_level_inputs(sc.levels[0])
    W = None if K == 0 else sc.W0 + 0.01
    return sc, a, W


def _ne(a, R, T, W, weight=None):
    return WO.normal_equations(a["conv1"], a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"], R, T, W, weight)


@pytest.mark.parametrize("K", [0, 5])
def test_weights_of_ones_are_the_oracle(K):
    sc, a, W = _oracle_case(K)
    args = (a["conv1"], a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"])
    ones = torch.ones(2, a["conv1"].shape[1], 1, dtype=torch.float64)
    H, g, rbar, nv = _ne(a, sc.R0, sc.T0, W, ones)
    rH, rg, rrbar, rnv = O.normal_equations_structured(*args, a["B"], sc.R0, sc.T0, W, guard_nonfinite=True)
    assert rel_fro(H, rH) < 1e-12 and rel_fro(g, rg) < 1e-12 and rel_fro(rbar, rrbar) < 1e-12 and torch.equal(nv, rnv)
    mlp = mlp_for(8, 3)
    opts = O.IterOptions(l2_regularizer_base=1000.0, guard_nonfinite=True)
    mine = WO.iteration(*args, a["B"], sc.R0, sc.T0, W, mlp, ones, opts)
    if K:
        ref = O.bundle_iteration(*args, a["B"], sc.R0, sc.T0, W, mlp, opts)
    else:
        ref = O.camera_iteration(*args, sc.R0, sc.T0, mlp, opts)
    for x, y in zip(mine, ref):
        assert rel_fro(x, y) < 1e-12


def _select(a, idx):
    """The oracle inputs restricted to (or repeating) the points idx (a LongTensor over N)."""
    out = dict(a)
    for k in ("conv1", "D", "B"):
        if a[k] is not None:
            out[k] = a[k][:, idx]
    for k in ("fx", "fy", "ox", "oy"):
        out[k] = a[k][:, idx]
    out["p"] = a["p"][:, :, idx]
    return out


def test_weight_two_duplicates_a_point_and_zero_removes_it():
    sc, a, W = _oracle_case(5, seed=4)
    N = a["conv1"].shape[1]
    g = torch.Generator().manual_seed(0)
    two, zero = torch.randperm(N, generator=g)[:40], torch.randperm(N, generator=g)[:60]
    zero = zero[~torch.isin(zero, two)]
    w = torch.ones(2, N, 1, dtype=torch.float64)
    w[:, two] = 2.0
    w[:, zero] = 0.0
    H, gv, _, _ = _ne(a, sc.R0, sc.T0, W, w)
    keep = torch.tensor([n for n in range(N) if n not in set(zero.tolist())])
    idx = torch.cat([keep, two])                          # the weight-2 points twice, the weight-0 points gone
    rH, rg, _, _ = _ne(_select(a, idx), sc.R0, sc.T0, W)
    assert rel_fro(H, rH) < 1e-12 and rel_fro(gv, rg) < 1e-12


def test_autograd_dweight_is_the_inner_product_with_the_point_terms():
    sc, a, W = _oracle_case(5, seed=5)
    N = a["conv1"].shape[1]
    gen = torch.Generator().manual_seed(1)
    w = (2 * torch.rand(2, N, 1, generator=gen, dtype=torch.float64)).requires_grad_()
    P = 11
    cH, cg = torch.randn(2, P, P, generator=gen, dtype=torch.float64), torch.randn(2, P, 1, generator=gen, dtype=torch.float64)
    H, g, _, _ = _ne(a, sc.R0, sc.T0, W, w)
    ((H * cH).sum() + (g * cg).sum()).backward()
    Hn, gn = WO.point_terms(a["conv1"], a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"], sc.R0, sc.T0, W)
    expect = torch.einsum("bnpq,bpq->bn", Hn, cH) + torch.einsum("bnp,bp->bn", gn, cg.squeeze(-1))
    assert rel_fro(w.grad.squeeze(-1), expect) < 1e-12


# ------------------------------------------------------------------------------------------------ CPU: the C-ABI
def _level(**kw):
    lv = _lib.BanetLevel(2, 4096, 64, 32, 48, 64, 192, 1, 1, 1, 1, 1, 1, 0, 0)
    for k, v in kw.items():
        setattr(lv, k, v)
    return lv


def test_struct_built_without_the_field_is_unweighted():
    assert _level().weight is None
    assert _lib.BanetLevel.weight.offset > _lib.BanetLevel.basis_dtype.offset


def test_weighted_backward_rejects_bad_arguments_before_any_cuda_call():
    lib = _lib.load()
    bwd = lib.banet_lm_build_bwd_weighted
    rc = bwd(ctypes.byref(_level(weight=1, nb=0)), 1, 1, 1, 1, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1, 1, None)
    assert rc == -1 and b"bad shape" in lib.banet_last_error()
    rc = bwd(ctypes.byref(_level(weight=1)), 1, 1, 1, None, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1, 1, None)
    assert rc == -1 and b"null pointer" in lib.banet_last_error()
    rc = bwd(ctypes.byref(_level(weight=1)), 1, 1, 1, 1, 1, 1, 0, 1, 1, 1, 1, 1, 1, None, 1, None)
    assert rc == -1 and b"dW" in lib.banet_last_error()
    rc = bwd(ctypes.byref(_level(weight=1, basis_dtype=5)), 1, 1, 1, 1, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1, 1, None)
    assert rc == -1 and b"basis_dtype" in lib.banet_last_error()


def test_legacy_tracker_rejects_weighted_levels():
    lib = _lib.load()
    arr = (_lib.BanetLevel * 1)(_level(K=0, weight=1))
    iters = (ctypes.c_int * 1)(3)
    rc = lib.banet_lm_track_legacy(arr, 1, iters, None, ctypes.byref(_lib.BanetLegacyOpts(1, 1e-5, 2e-4, 1.0)), 1, 1, None, 1, 1, 1, 1 << 20, None)
    assert rc == -4 and b"weights" in lib.banet_last_error()


# ------------------------------------------------------------------------------------------------ GPU
PRECS = {"simt": _lib.PREC_FP32_SIMT, "x1": _lib.PREC_TF32X1, "x2": _lib.PREC_TF32X2, "x3": _lib.PREC_TF32X3, "auto": _lib.PREC_AUTO}


def _gpu_scene(C, K, seed, H=48, W=64, n_points=None):
    from banet_b200 import synth
    sc = synth.make_scene(nb=2, H=H, W=W, C=C, K=K, level_ids=(3,), seed=seed, device="cuda", dtype=torch.float32, n_points=n_points)
    Wt = None if K == 0 else sc.W0 + 0.01 * torch.randn(sc.W0.shape, generator=torch.Generator().manual_seed(seed)).cuda()
    return sc, sc.levels[0], Wt


def _level_of(lv, layout, feat, basis, grid, weight=None):
    from banet_b200 import ops
    C = lv.conv1.shape[2]
    conv2 = lv.conv2 if layout == "3c" else lv.conv2[..., :C].contiguous()
    conv1 = lv.conv1
    if feat == "bf16":
        conv1, conv2 = conv1.to(BF), conv2.to(BF)
    B = lv.B if (lv.B is None or basis == "f32") else lv.B.to(BF)
    return ops.Level(conv1, conv2, lv.intr, lv.p, lv.D, B, grid=lv.grid if grid else None, weight=weight)


@gpu
@pytest.mark.parametrize("basis", ["f32", "bf16"])
@pytest.mark.parametrize("feat", ["f32", "bf16"])
@pytest.mark.parametrize("layout", ["3c", "f2"])
@pytest.mark.parametrize("K", [128, 64, 32, 16, 200, 0])
def test_weights_of_ones_give_the_unweighted_bits(K, layout, feat, basis):
    from banet_b200 import ops
    _lib.require_device()
    if K == 0 and basis == "bf16":
        pytest.skip("no basis")
    sc, lv, Wt = _gpu_scene(64, K, seed=17 + K)
    ones = torch.ones(2, lv.N, 1, device="cuda")
    precs = ("simt", "x1", "x2", "x3", "auto") if K in (32, 64, 128) else ("simt", "auto")
    for grid in (True, False):
        for pn in precs:
            a = ops.lm_build(_level_of(lv, layout, feat, basis, grid), sc.R0, sc.T0, Wt, PRECS[pn])
            b = ops.lm_build(_level_of(lv, layout, feat, basis, grid, ones), sc.R0, sc.T0, Wt, PRECS[pn])
            for x, y, name in zip(a, b, ("H", "g", "rbar_sum", "nvalid")):
                assert torch.equal(x, y), (grid, pn, name)


def _weighted_reference(lv, sc, Wt, weight):
    a = oracle_level_inputs(lv)
    a = {k: (None if v is None else v.cpu()) for k, v in a.items()}
    return WO.normal_equations(a["conv1"], a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"], sc.R0.cpu().double(),
                               sc.T0.cpu().double(), None if Wt is None else Wt.cpu().double(), None if weight is None else weight.cpu().double())


@gpu
@pytest.mark.parametrize("layout", ["3c", "f2"])
@pytest.mark.parametrize("grid", [True, False])
def test_random_weights_match_the_float64_statement(layout, grid):
    from banet_b200 import ops
    _lib.require_device()
    sc, lv, Wt = _gpu_scene(128, 128, seed=23)
    w = 2 * torch.rand(2, lv.N, 1, generator=torch.Generator().manual_seed(2)).cuda()
    rH, rg, rrbar, rnv = _weighted_reference(lv, sc, Wt, w)
    for pn, tol in (("simt", 2e-5), ("x1", 5e-4), ("x2", 1e-4), ("x3", 2e-6)):
        H, g, rbar, nv = ops.lm_build(_level_of(lv, layout, "f32", "f32", grid, w), sc.R0, sc.T0, Wt, PRECS[pn])
        print(f"{layout} grid={grid} {pn}: relH={rel_fro(H, rH):.2e} relg={rel_fro(g, rg.squeeze(-1)):.2e}")
        assert rel_fro(H, rH) < tol and rel_fro(g, rg.squeeze(-1)) < tol, pn
        assert rel_fro(rbar / lv.N, rrbar.squeeze(1)) < 2e-5 and torch.equal(nv.cpu().double(), rnv)


@gpu
@pytest.mark.parametrize("layout", ["3c", "f2"])
def test_zero_weights_equal_a_build_on_the_other_points(layout):
    from banet_b200 import ops
    _lib.require_device()
    sc, lv, Wt = _gpu_scene(128, 128, seed=29)
    N = lv.N
    keep = torch.rand(N, generator=torch.Generator().manual_seed(3)) < 0.5
    w = keep.float().reshape(1, N, 1).repeat(2, 1, 1).cuda()
    idx = torch.nonzero(keep).flatten().cuda()
    C = 128
    conv2 = lv.conv2 if layout == "3c" else lv.conv2[..., :C].contiguous()
    half = ops.Level(lv.conv1[:, idx].contiguous(), conv2, lv.intr, lv.p[:, :, idx].contiguous(), lv.D[:, idx].contiguous(), lv.B[:, idx].contiguous())
    for pn in ("simt", "x3"):
        H, g, rbar, nv = ops.lm_build(ops.Level(lv.conv1, conv2, lv.intr, lv.p, lv.D, lv.B, grid=lv.grid, weight=w), sc.R0, sc.T0, Wt, PRECS[pn])
        Hh, gh, _, _ = ops.lm_build(half, sc.R0, sc.T0, Wt, PRECS[pn])
        _, _, rbar0, nv0 = ops.lm_build(ops.Level(lv.conv1, conv2, lv.intr, lv.p, lv.D, lv.B, grid=lv.grid), sc.R0, sc.T0, Wt, PRECS[pn])
        assert rel_fro(H, Hh) < 1e-5 and rel_fro(g, gh) < 1e-5, pn
        assert torch.equal(rbar, rbar0) and torch.equal(nv, nv0), pn


def _poisoned_ws(pattern):
    def make(nbytes, device):
        n = max(int(nbytes), 256)
        if pattern == "nan":
            return torch.full((n,), 0xFF, dtype=torch.uint8, device=device)
        g = torch.Generator(device="cuda").manual_seed(n % 9973 + 1)
        return torch.randint(0, 256, (n,), dtype=torch.uint8, device=device, generator=g)
    return make


@gpu
@pytest.mark.parametrize("layout", ["3c", "f2"])
def test_weighted_builds_are_bit_reproducible(layout, monkeypatch):
    from banet_b200 import ops
    _lib.require_device()
    sc, lv, Wt = _gpu_scene(128, 128, seed=31, H=120, W=160)
    w = 2 * torch.rand(2, lv.N, 1, generator=torch.Generator().manual_seed(4)).cuda()
    L = _level_of(lv, layout, "f32", "f32", True, w)
    for pn in PRECS:
        outs = []
        for pattern in ("nan", "random"):
            monkeypatch.setattr(ops, "_ws", _poisoned_ws(pattern))
            outs.append(ops.lm_build(L, sc.R0, sc.T0, Wt, precision=PRECS[pn]))
        for a, b in zip(*outs):
            assert torch.equal(a, b), pn
        assert bool(torch.isfinite(outs[0][0]).all())


@gpu
@pytest.mark.parametrize("exact", [1, 0])
@pytest.mark.parametrize("feat", ["f32", "bf16"])
@pytest.mark.parametrize("layout", ["3c", "f2"])
@pytest.mark.parametrize("K", [6, 0])
def test_iteration_gradients_match_float64_autograd(K, layout, feat, exact):
    """iteration_fused with a weight that requires grad against float64 autograd of the weighted statement: every input's gradient at
    exact_sym = 1 (the true adjoint); dweight, which both conventions share, at exact_sym = 0."""
    from banet_b200 import autograd as AG
    _lib.require_device()
    C = 8
    sc = scene_case(nb=2, C=C, K=K, level_ids=(3,), seed=61 + K, n_points=400, dtype=torch.float32)
    lv = sc.levels[0]
    a = oracle_level_inputs(lv)
    if feat == "bf16":
        a["conv1"] = a["conv1"].to(BF).double()
        a["conv2"] = a["conv2"].to(BF).double()
    a["F2"] = a["conv2"][..., :C].contiguous()
    a["weight"] = 2 * torch.rand(2, lv.N, 1, generator=torch.Generator().manual_seed(K), dtype=torch.float64)
    names = ["conv1", "F2" if layout == "f2" else "conv2", "D", "weight"] + (["B"] if K else [])
    for n in names:
        a[n] = a[n].clone().requires_grad_()
    conv2_o = torch.cat([a["F2"], O.grad_fixed(a["F2"])], dim=-1) if layout == "f2" else a["conv2"]
    R = sc.R0.double().clone().requires_grad_(); T = sc.T0.double().clone().requires_grad_()
    W = (sc.W0.double() + 0.01).clone().requires_grad_() if K else None
    mlp = mlp_for(C, 3)
    g = torch.Generator().manual_seed(5)
    cR, cT = torch.randn(2, 3, 3, generator=g, dtype=torch.float64), torch.randn(2, 3, 1, generator=g, dtype=torch.float64)
    cW = torch.randn(2, K, 1, generator=g, dtype=torch.float64) if K else None
    opts = O.IterOptions(l2_regularizer_base=1000.0, guard_nonfinite=True)
    oR, oT, oW = WO.iteration(a["conv1"], conv2_o, a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"], R, T, W, mlp, a["weight"], opts)
    loss = (oR * cR).sum() + (oT * cT).sum() + ((oW * cW).sum() if K else 0.0)
    loss.backward()
    dt = BF if feat == "bf16" else torch.float32
    t = {n: a[n].detach().to("cuda", dt if n in ("conv1", "conv2", "F2") else torch.float32).contiguous().requires_grad_() for n in names}
    Rg = to_cuda32(sc.R0).requires_grad_(); Tg = to_cuda32(sc.T0).requires_grad_()
    Wg = to_cuda32(sc.W0 + 0.01).requires_grad_() if K else None
    mlp32 = [(to_cuda32(w), to_cuda32(b)) for w, b in mlp]
    conv2_key = "F2" if layout == "f2" else "conv2"
    gR, gT, gW = AG.iteration_fused(t["conv1"], t[conv2_key], to_cuda32(lv.intr), to_cuda32(lv.p), t["D"], t.get("B"), Rg, Tg, Wg, mlp32,
                                    1000.0 if K else None, exact_sym=bool(exact), weight=t["weight"])
    assert rel_fro(gR, oR) < 1e-5 and rel_fro(gT, oT) < 1e-4
    lossg = (gR * cR.float().cuda()).sum() + (gT * cT.float().cuda()).sum() + ((gW * cW.float().cuda()).sum() if K else 0.0)
    lossg.backward()
    tol = 2e-3 if feat == "f32" else 5e-3
    check = names + ["R", "T"] + (["W"] if K else []) if exact else ["weight"]
    got = dict(t, R=Rg, T=Tg, W=Wg)
    want = dict(a, R=R, T=T, W=W)
    for n in check:
        e = rel_fro(got[n].grad.float(), want[n].grad)
        print(f"K={K} {layout} {feat} exact={exact} d{n}: {e:.2e}")
        assert e < tol, n


@gpu
@pytest.mark.parametrize("layout", ["3c", "f2"])
def test_all_ones_backward_is_the_unweighted_backward(layout):
    from banet_b200 import ops
    _lib.require_device()
    sc, lv, Wt = _gpu_scene(64, 32, seed=37)
    P = 38
    gen = torch.Generator(device="cuda").manual_seed(9)
    dH, dg, dr = torch.randn(2, P, P, generator=gen, device="cuda"), torch.randn(2, P, generator=gen, device="cuda"), torch.randn(2, 64, generator=gen, device="cuda")
    ones = torch.ones(2, lv.N, 1, device="cuda")
    a = ops.lm_build_bwd(_level_of(lv, layout, "f32", "f32", True), sc.R0, sc.T0, Wt, dH, dg, dr, True)
    b = ops.lm_build_bwd(_level_of(lv, layout, "f32", "f32", True, ones), sc.R0, sc.T0, Wt, dH, dg, dr, True, return_dweight=True)
    c = ops.lm_build_bwd(_level_of(lv, layout, "f32", "f32", True), sc.R0, sc.T0, Wt, dH, dg, dr, True, return_dweight=True)
    for name, x, y in zip(("dconv1", "dconv2", "dD", "dB", "dR", "dT", "dW"), a, b):
        assert rel_fro(y, x) < 1e-6, name
    for name in (0, 2, 3):                                 # one writer per element: bitwise
        assert torch.equal(a[name], b[name]), name
    assert torch.equal(b[7], c[7]) and bool(torch.isfinite(b[7]).all())


def _resize_net(C):
    from banet_b200.bundlenet import BundleNet
    return BundleNet(C, levels=("0", "1", "2", "3"), precision=_lib.PREC_AUTO).cuda()


@gpu
def test_resize_with_weights():
    import gen_golden
    _lib.require_device()
    x = gen_golden.resize_inputs(nb=4, C=16, K=8)
    net = _resize_net(16)
    f = {k: to_cuda32(x[k]) for k in ("intr", "points", "basis", "depth", "R0", "T0")}
    layers = [to_cuda32(l) for l in x["layers"]]
    N = f["points"].shape[1]
    ones = torch.ones(4, N, 1, device="cuda")
    net.eval()
    with torch.no_grad():
        a = net.BundleResize(f["intr"], layers, f["points"], f["basis"], f["depth"], f["R0"], f["T0"])
        b = net.BundleResize(f["intr"], layers, f["points"], f["basis"], f["depth"], f["R0"], f["T0"], weight=ones)
        ca = net.CameraResize(f["intr"], layers, f["points"], f["depth"])
        cb = net.CameraResize(f["intr"], layers, f["points"], f["depth"], weight=ones)
    for xs, ys in zip(a + ca, b + cb):
        for u, v in zip(xs, ys):
            assert torch.equal(u, v)
    w = (0.5 + torch.rand(4, N, 1, generator=torch.Generator().manual_seed(6))).cuda().requires_grad_()
    Rs, Ts, Ds = net.BundleResize(f["intr"], layers, f["points"], f["basis"], f["depth"], f["R0"], f["T0"], weight=w)
    cR, cT = net.CameraResize(f["intr"], layers, f["points"], f["depth"], weight=w)
    (sum(r.sum() for r in Rs + cR) + sum(t.sum() for t in Ts + cT) + sum(d.sum() for d in Ds)).backward()
    assert w.grad is not None and bool(torch.isfinite(w.grad).all()) and float(w.grad.abs().sum()) > 0
    split = _resize_net(16)
    split.training_path = "reference_split"
    with pytest.raises(RuntimeError, match="point weights"):
        split.BundleResize(f["intr"], layers, f["points"], f["basis"], f["depth"], f["R0"], f["T0"], weight=w)
    with pytest.raises(RuntimeError, match="point weights"):
        split.CameraResize(f["intr"], layers, f["points"], f["depth"], weight=w)


@gpu
def test_weighted_whole_solve_at_auto_matches_the_float64_statement():
    from banet_b200 import ops, synth
    _lib.require_device()
    sc = synth.make_scene(nb=1, H=240, W=320, C=128, K=128, level_ids=(0, 1, 2, 3), seed=1236, device="cuda", dtype=torch.float32)
    mlps = [O.init_lambda_mlp(128, seed=7 + l.level, dtype=torch.float32) for l in sc.levels]
    ws = [(0.5 + torch.rand(1, l.N, 1, generator=torch.Generator().manual_seed(l.level))).cuda() for l in sc.levels]
    olv = []
    for l, m in zip(sc.levels, mlps):
        a = oracle_level_inputs(l)
        a = {k: (None if v is None else v.cpu()) for k, v in a.items()}
        olv.append(O.LevelInputs(a["conv1"], a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"],
                                 [(w.double(), b.double()) for w, b in m]))
    oR, oT, oW = WO.solve(olv, [w.cpu().double() for w in ws], 5, sc.R0.cpu().double(), sc.T0.cpu().double(), sc.W0.cpu().double())
    packed = [ops.pack_mlp(m).cuda() for m in mlps]
    for layout in ("3c", "f2"):
        levels = [ops.Level(l.conv1, l.conv2 if layout == "3c" else l.conv2[..., :128].contiguous(), l.intr, l.p, l.D, l.B, grid=l.grid, weight=w)
                  for l, w in zip(sc.levels, ws)]
        for name, prec in (("fp32", _lib.PREC_FP32_SIMT), ("auto", _lib.PREC_AUTO)):
            R, T, W, st = ops.lm_run(levels, 5, sc.R0, sc.T0, sc.W0, mlp_packed=packed, l2_regularizer_base=1000.0, precision=prec)
            e = dict(R=rel_fro(R, oR), T=rel_fro(T, oT), W=rel_fro(W, oW))
            print(layout, name, e)
            assert int(st.abs().max()) == 0 and max(e.values()) < 1e-4, (layout, name, e)
        unweighted = [ops.Level(l.conv1, lv.conv2, l.intr, l.p, l.D, l.B, grid=l.grid) for l, lv in zip(sc.levels, levels)]
        R0, _, _, _ = ops.lm_run(unweighted, 5, sc.R0, sc.T0, sc.W0, mlp_packed=packed, l2_regularizer_base=1000.0, precision=_lib.PREC_AUTO)
        assert not torch.equal(R, R0)                      # the weights do act


@gpu
def test_window_of_one_frame_with_weights_is_the_two_view_solve():
    from banet_b200 import ops, synth
    _lib.require_device()
    sc = synth.make_scene(nb=1, H=96, W=128, C=128, K=128, level_ids=(2, 3), seed=41, device="cuda", dtype=torch.float32, shared_depth=True)
    levels = [ops.Level(l.conv1, l.conv2, l.intr, l.p, l.D, l.B, grid=l.grid,
                        weight=2 * torch.rand(1, l.N, 1, generator=torch.Generator().manual_seed(l.level)).cuda()) for l in sc.levels]
    packed = [ops.pack_mlp(O.init_lambda_mlp(128, seed=100 + l.level, dtype=torch.float32)).cuda() for l in sc.levels]
    for prec in (_lib.PREC_AUTO, _lib.PREC_FP32_SIMT):
        R, T, W, st = ops.lm_window_run(levels, 3, sc.R0, sc.T0, sc.W0[0], mlp_packed=packed, l2_regularizer_base=1000.0, precision=prec)
        R2, T2, W2, _ = ops.lm_run(levels, 3, sc.R0, sc.T0, sc.W0, mlp_packed=packed, l2_regularizer_base=1000.0, precision=prec)
        assert int(st.abs().max()) == 0
        assert torch.equal(R, R2) and torch.equal(T, T2) and torch.equal(W, W2[0]), prec
