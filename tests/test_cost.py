"""The feature-metric cost of a level (banet_lm_cost / banet_lm_cost_bwd, ops.lm_cost, autograd.feature_metric_cost,
BundleNet.FeatureMetricCost): cost[b] = sum_n c_n rho(s_n), s_n the squared norm of the build's residual.  On the CPU: the float64
statement (tests/cost_oracle.py) against the robust weights and, on feature maps that are affine in (x, y), against the weighted normal
equations (the descent identity: the gradient of the cost w.r.t. the LM update at 0 is -2 g); the C-ABI's argument errors.  On the GPU:
the forward and the backward against float64, the bitwise identities, the same descent identity on the library, batches past 65 535 pairs
and the Python layers."""
import ctypes
import math

import pytest
import torch

from helpers import O, scene_case, oracle_level_inputs, rel_fro, to_cuda32
import cost_oracle as CO
import robust_oracle as RO
import weighted_oracle as WO
from banet_b200 import _lib

gpu = pytest.mark.gpu
BF = torch.bfloat16
KINDS = [None, "huber", "cauchy"]


def _args(a):
    return (a["conv1"], a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"])


# ------------------------------------------------------------------------------------------------ CPU: the float64 statement
def test_rho1_is_the_derivative_of_rho():
    s = torch.tensor([0.05, 0.3, 1.0, 2.5, 7.0, 30.0], dtype=torch.float64, requires_grad=True)     # Huber kink at 1.44: not hit
    for kind in ("huber", "cauchy"):
        (d,) = torch.autograd.grad(CO.rho(kind, 1.2, s).sum(), s)
        assert torch.allclose(d, RO.rho1(kind, 1.2, s.detach()), rtol=1e-13, atol=0), kind
        assert torch.autograd.gradcheck(lambda x: CO.rho(kind, 1.2, x), (s,))
    assert torch.equal(CO.rho(None, 0.0, s), s)
    z = torch.zeros(3, dtype=torch.float64)
    for kind in KINDS:
        assert torch.equal(CO.rho(kind, 0.7, z), z)


def _skew(w):
    z = torch.zeros_like(w[:, 0])
    return torch.stack([torch.stack([z, -w[:, 2], w[:, 1]], -1), torch.stack([w[:, 2], z, -w[:, 0]], -1),
                        torch.stack([-w[:, 1], w[:, 0], z], -1)], -2)


def _lm_update(R, T, W, xi, dl):
    """The LM update at (xi, dl) to first order at 0 (bundlenet.py:269-276): R <- exp(w) R, T <- V(w) t + exp(w) T, W <- W + dl;
    V(0) = I, and V(w) t has no first-order term in w at t = 0."""
    E = torch.matrix_exp(_skew(xi[:, :3]))
    return E @ R, E @ T + xi[:, 3:].unsqueeze(-1), None if W is None else W + dl.unsqueeze(-1)


def _affine_case(K, seed, weighted):
    """A scene whose conv2 is affine in (x, y) per channel, [F2 | gx | gy] with the exact slopes, restricted to the points whose taps and
    gradient stencil lie inside the map: there the bilinear sample's derivative is the build's G, so the descent identity is exact."""
    sc = scene_case(nb=2, C=8, K=K, level_ids=(3,), seed=seed, n_points=600)
    a = oracle_level_inputs(sc.levels[0])
    W = None if K == 0 else sc.W0 + 0.01
    Dt = a["D"] if K == 0 else a["D"] + a["B"] @ W
    _, _, _, _, px, py = O._warp(a["p"], Dt, sc.R0, sc.T0, a["fx"], a["fy"], a["ox"], a["oy"])
    nb, h, w, C = 2, a["conv2"].shape[1], a["conv2"].shape[2], a["conv1"].shape[2]
    ok = (px >= 2) & (px <= w - 3) & (py >= 2) & (py <= h - 3)
    n = int(ok.sum(1).min())
    assert n >= 100
    idx = torch.stack([torch.nonzero(ok[b]).flatten()[:n] for b in range(nb)])
    take = lambda t: None if t is None else torch.gather(t, 1, idx.unsqueeze(-1).expand(-1, -1, t.shape[2]))
    g = torch.Generator().manual_seed(seed)
    A0, ax, ay = (torch.rand(nb, 1, 1, C, generator=g, dtype=torch.float64) for _ in range(3))
    ax, ay = ax - 0.5, ay - 0.5
    F2 = A0 + ax * torch.arange(w, dtype=torch.float64).reshape(1, 1, w, 1) + ay * torch.arange(h, dtype=torch.float64).reshape(1, h, 1, 1)
    out = dict(conv1=take(a["conv1"]), conv2=torch.cat([F2, ax.expand(nb, h, w, C), ay.expand(nb, h, w, C)], -1),
               fx=a["fx"][:, :n], fy=a["fy"][:, :n], ox=a["ox"][:, :n], oy=a["oy"][:, :n],
               p=torch.gather(a["p"], 2, idx.unsqueeze(1).expand(-1, 3, -1)), D=take(a["D"]), B=take(a["B"]))
    c = (0.5 + torch.rand(nb, n, 1, generator=g, dtype=torch.float64)) if weighted else None
    return sc, out, W, c


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("K", [0, 5])
def test_descent_identity_on_the_float64_statement(K, kind, weighted):
    sc, a, W, c = _affine_case(K, 17 + K, weighted)
    R, T = sc.R0, sc.T0
    s = RO.squared_norms(*_args(a), R, T, W)
    delta = math.sqrt(float(s[s > 0].median()))
    w = c if kind is None else RO.robust_weight(*_args(a), R, T, W, kind, delta, c)
    _, g, _, _ = WO.normal_equations(*_args(a), R, T, W, w)
    xi = torch.zeros(2, 6, dtype=torch.float64, requires_grad=True)
    dl = torch.zeros(2, K, dtype=torch.float64, requires_grad=True)
    Rn, Tn, Wn = _lm_update(R, T, W, xi, dl)
    cost = CO.cost(*_args(a), Rn, Tn, Wn, kind, delta, c)
    grads = torch.autograd.grad(cost.sum(), (xi, dl) if K else (xi,))
    got = torch.cat([t.reshape(2, -1) for t in grads], -1)
    assert rel_fro(got, -2.0 * g.squeeze(-1)) < 1e-10


# ------------------------------------------------------------------------------------------------ CPU: the C-ABI
def _level(**kw):
    lv = _lib.BanetLevel(2, 4096, 64, 32, 48, 64, 192, 1, 1, 1, 1, 1, 1, 0, 0)
    for k, v in kw.items():
        setattr(lv, k, v)
    return lv


def _fwd(lib, lv, R=1, T=1, W=1, cost=1, nvalid=1, ws=1, ws_bytes=1 << 30):
    return lib.banet_lm_cost(ctypes.byref(lv), R, T, W, cost, nvalid, None, None, ws, ws_bytes, None)


def _bwd(lib, lv, **kw):
    a = dict(R=1, T=1, W=1, dcost=1, dconv1=1, dconv2=1, dD=1, dB=1, dR=1, dT=1, dW=1)
    a.update(kw)
    return lib.banet_lm_cost_bwd(ctypes.byref(lv), a["R"], a["T"], a["W"], a["dcost"], a["dconv1"], a["dconv2"], a["dD"], a["dB"], a["dR"],
                                 a["dT"], a["dW"], None, None)


def test_cost_entries_reject_bad_arguments_without_gpu():
    lib = _lib.load()
    err = lambda: lib.banet_last_error()
    good = _level()
    need = lib.banet_lm_cost_workspace_bytes(ctypes.byref(good))
    assert 0 < need < (1 << 20)
    # the level's own checks: bad shape, layout, dtype, robust kind or scale, a null tensor, K > 0 without B
    for bad in (dict(nb=0), dict(conv2_channels=100), dict(feature_dtype=2), dict(basis_dtype=5), dict(robust=3, robust_scale=1.0),
                dict(robust=1, robust_scale=0.0), dict(robust=2, robust_scale=float("nan")), dict(conv1=None), dict(B=None),
                dict(grid_w=7, grid_h=7)):
        lv = _level(**bad)
        assert _fwd(lib, lv) == -1, bad
        assert _bwd(lib, lv) == -1, bad
        assert lib.banet_lm_cost_workspace_bytes(ctypes.byref(lv)) == 0, bad
    assert lib.banet_lm_cost_workspace_bytes(None) == 0
    assert lib.banet_lm_cost(None, 1, 1, 1, 1, 1, None, None, 1, 1 << 30, None) == -1
    # null pointers
    for k in ("R", "T", "cost", "nvalid"):
        assert _fwd(lib, good, **{k: None}) == -1 and b"null" in err(), k
    for k in ("R", "T", "dcost", "dconv1", "dconv2", "dD", "dR", "dT"):
        assert _bwd(lib, good, **{k: None}) == -1 and b"null" in err(), k
    # K > 0 needs W (and dB, dW in the backward); K = 0 needs none of them
    assert _fwd(lib, good, W=None) == -1 and b"W is null" in err()
    for k in ("W", "dB", "dW"):
        assert _bwd(lib, good, **{k: None}) == -1 and b"null" in err(), k
    # K > 256
    big = _level(K=257)
    assert _fwd(lib, big) == -4 and b"K=257" in err()
    assert _bwd(lib, big) == -4 and b"K=257" in err()
    assert lib.banet_lm_cost_workspace_bytes(ctypes.byref(big)) == 0
    assert lib.banet_lm_cost_workspace_bytes(ctypes.byref(_level(K=256))) > 0
    # the workspace
    assert _fwd(lib, good, ws=None) == -2 and b"workspace" in err()
    assert _fwd(lib, good, ws_bytes=need - 1) == -2 and b"workspace" in err()
    # the grid hint only changes the tiling: 8 x 8 tiles of a 64 x 64 grid
    assert lib.banet_lm_cost_workspace_bytes(ctypes.byref(_level(grid_w=64, grid_h=64))) >= 64 * 2 * 16


def test_lm_cost_rejects_bad_arguments_in_python_without_gpu():
    from banet_b200 import ops
    with pytest.raises(_lib.BanetError, match="robust"):
        ops.robust_kind("tukey", 1.0)
    lv = ops.Level(torch.zeros(1, 4, 2), torch.zeros(1, 2, 2, 6), torch.zeros(1, 4), torch.zeros(1, 3, 4), torch.zeros(1, 4, 1), None)
    with pytest.raises(_lib.BanetError, match="CUDA"):
        ops.lm_cost(lv, torch.eye(3)[None], torch.zeros(1, 3, 1), None)


# ------------------------------------------------------------------------------------------------ GPU
def _gpu_scene(C, K, seed, H=48, W=64, nb=2):
    from banet_b200 import synth
    sc = synth.make_scene(nb=nb, H=H, W=W, C=C, K=K, level_ids=(3,), seed=seed, device="cuda", dtype=torch.float32)
    Wt = None if K == 0 else sc.W0 + 0.01 * torch.randn(sc.W0.shape, generator=torch.Generator().manual_seed(seed)).cuda()
    return sc, sc.levels[0], Wt


def _level_of(lv, layout, feat, basis, grid=True, weight=None, robust=None, scale=0.0):
    from banet_b200 import ops
    C = lv.conv1.shape[2]
    conv2 = lv.conv2 if layout == "3c" else lv.conv2[..., :C].contiguous()
    conv1 = lv.conv1
    if feat == "bf16":
        conv1, conv2 = conv1.to(BF), conv2.to(BF)
    B = lv.B if (lv.B is None or basis == "f32") else lv.B.to(BF)
    return ops.Level(conv1, conv2, lv.intr, lv.p, lv.D, B, grid=lv.grid if grid else None, weight=weight, robust=robust, robust_scale=scale)


def _oracle_inputs(lv, feat, basis):
    """Oracle inputs of a GPU scene level as the kernels read them (bf16 tensors rounded first); the cost reads F2 only, so one map serves
    both layouts."""
    a = {k: (None if v is None else v.cpu()) for k, v in oracle_level_inputs(lv).items()}
    rnd = (lambda t: t.to(BF).cpu().double()) if feat == "bf16" else (lambda t: t.cpu().double())
    a["conv1"], a["conv2"] = rnd(lv.conv1), rnd(lv.conv2)
    if basis == "bf16" and a["B"] is not None:
        a["B"] = lv.B.to(BF).cpu().double()
    return a


def _delta(s):
    """delta with half of the valid points above delta^2 (down-weighted by Huber; Cauchy down-weights every point, these the most)."""
    v = s[s > 0]
    return math.sqrt(float(v.median())), float((v > v.median()).double().mean())


@gpu
@pytest.mark.parametrize("C", [16, 64, 128, 13])
@pytest.mark.parametrize("K", [0, 16, 128, 256])
def test_forward_matches_float64(K, C):
    from banet_b200 import ops
    _lib.require_device()
    sc, lv, Wt = _gpu_scene(C, K, seed=101 + K + C)
    R0d, T0d, Wd = sc.R0.cpu().double(), sc.T0.cpu().double(), None if Wt is None else Wt.cpu().double()
    c = (0.5 + torch.rand(2, lv.N, 1, generator=torch.Generator().manual_seed(7))).cuda()
    worst = 0.0
    for feat in ("f32", "bf16"):
        for basis in (("f32", "bf16") if K else ("f32",)):
            a = _oracle_inputs(lv, feat, basis)
            s = RO.squared_norms(*_args(a), R0d, T0d, Wd)
            m = (s > 0).double()
            delta, frac = _delta(s)
            print(f"K={K} C={C} {feat}/{basis}: delta={delta:.4g}, {100 * frac:.0f} % of the valid points above delta^2")
            assert 0.4 <= frac <= 0.6
            for weight in (None, c):
                wd = None if weight is None else weight.cpu().double()
                for kind in KINDS:
                    ref = CO.cost_from_norms(s, kind, delta, wd)
                    for layout in ("3c", "f2"):
                        for grid in (True, False):
                            L = _level_of(lv, layout, feat, basis, grid, weight, kind, delta if kind else 0.0)
                            cost, nv, sk, mk = ops.lm_cost(L, sc.R0, sc.T0, Wt, per_point=True)
                            e = rel_fro(cost.cpu().double(), ref)
                            worst = max(worst, e)
                            assert e < 2e-5, (feat, basis, weight is None, kind, layout, grid, e)
                            assert torch.equal(mk.squeeze(-1).cpu().double(), m) and torch.equal(nv.cpu().double(), m.sum(1))
                            assert rel_fro(sk.squeeze(-1).cpu().double(), s) < 2e-5
                            assert bool((sk.squeeze(-1)[mk.squeeze(-1) == 0] == 0).all())
    print(f"largest relative cost error {worst:.2e}")


PRECS = {"simt": _lib.PREC_FP32_SIMT, "x1": _lib.PREC_TF32X1, "x2": _lib.PREC_TF32X2, "x3": _lib.PREC_TF32X3, "auto": _lib.PREC_AUTO}


@gpu
@pytest.mark.parametrize("C", [64, 128, 13])
@pytest.mark.parametrize("K", [0, 16, 128])
def test_nvalid_is_the_builds_in_every_precision_mode(K, C):
    from banet_b200 import ops
    _lib.require_device()
    sc, lv, Wt = _gpu_scene(C, K, seed=131 + K + C)
    R = sc.R0.clone()
    R[1] = torch.linalg.matrix_exp(torch.tensor([[0.0, -0.12, 0.05], [0.12, 0.0, -0.08], [-0.05, 0.08, 0.0]], device="cuda")) @ R[1]  # masks some points
    tc = K == 128 and C in (64, 128)
    for layout in ("3c", "f2"):
        for feat in ("f32", "bf16"):
            for basis in (("f32", "bf16") if K else ("f32",)):
                for kind in (None, "cauchy"):
                    L = _level_of(lv, layout, feat, basis, True, None, kind, 2.0 if kind else 0.0)
                    _, nv = ops.lm_cost(L, R, sc.T0, Wt)
                    assert float(nv.min()) > 0
                    for pn in (PRECS if tc else ("simt", "auto")):
                        _, _, _, bn = ops.lm_build(L, R, sc.T0, Wt, PRECS[pn])
                        assert torch.equal(nv, bn), (layout, feat, basis, kind, pn)


def _poisoned_ws(pattern):
    def make(nbytes, device):
        n = max(int(nbytes), 256)
        if pattern == "nan":
            return torch.full((n,), 0xFF, dtype=torch.uint8, device=device)
        g = torch.Generator(device="cuda").manual_seed(n % 9973 + 1)
        return torch.randint(0, 256, (n,), dtype=torch.uint8, device=device, generator=g)
    return make


@gpu
@pytest.mark.parametrize("K", [0, 16, 128, 256])
def test_bitwise_identities(K, monkeypatch):
    from banet_b200 import ops
    _lib.require_device()
    for C in (16, 13):
        sc, lv, Wt = _gpu_scene(C, K, seed=151 + K + C)
        s = ops.lm_cost(_level_of(lv, "3c", "f32", "f32"), sc.R0, sc.T0, Wt, per_point=True)[2]
        big = 10.0 * math.sqrt(float(s.max()))
        ones = torch.ones(2, lv.N, 1, device="cuda")
        for feat in ("f32", "bf16"):
            for basis in (("f32", "bf16") if K else ("f32",)):
                for kind in KINDS:
                    scale = 3.0 if kind else 0.0
                    ref = ops.lm_cost(_level_of(lv, "3c", feat, basis, True, None, kind, scale), sc.R0, sc.T0, Wt, per_point=True)
                    # the F2-only layout reads the same channels
                    f2 = ops.lm_cost(_level_of(lv, "f2", feat, basis, True, None, kind, scale), sc.R0, sc.T0, Wt, per_point=True)
                    # weights of ones are no weights
                    w1 = ops.lm_cost(_level_of(lv, "3c", feat, basis, True, ones, kind, scale), sc.R0, sc.T0, Wt, per_point=True)
                    for x, y, z in zip(ref, f2, w1):
                        assert torch.equal(x, y) and torch.equal(x, z), (C, feat, basis, kind)
                    # poisoned workspaces: the slots are written before they are read
                    for pattern in ("nan", "random"):
                        monkeypatch.setattr(ops, "_ws", _poisoned_ws(pattern))
                        again = ops.lm_cost(_level_of(lv, "f2", feat, basis, False, None, kind, scale), sc.R0, sc.T0, Wt, per_point=True)
                        monkeypatch.undo()
                        if pattern == "nan":
                            first = again
                        else:
                            for x, y in zip(first, again):
                                assert torch.equal(x, y), (C, feat, basis, kind)
                    assert bool(torch.isfinite(first[0]).all())
                # Huber above every residual is the plain loss
                hub = ops.lm_cost(_level_of(lv, "3c", feat, basis, True, None, "huber", big), sc.R0, sc.T0, Wt, per_point=True)
                plain = ops.lm_cost(_level_of(lv, "3c", feat, basis, True, None), sc.R0, sc.T0, Wt, per_point=True)
                for x, y in zip(hub, plain):
                    assert torch.equal(x, y), (C, feat, basis)
        # bf16 maps and basis against the fp32 path on the widened values.  Both dtypes read 4 channels per lane when C % 4 == 0 and
        # the maps are aligned (8 B for bf16, 16 B for fp32: true of every torch allocation here), and one channel per lane otherwise, so
        # every lane sums the same channels in the same order and the bits agree.
        from banet_b200 import ops as _o
        widen = lambda t: t.to(BF).float()
        for kind in KINDS:
            scale = 3.0 if kind else 0.0
            Bb = None if lv.B is None else lv.B.to(BF)
            a = _o.lm_cost(_o.Level(lv.conv1.to(BF), lv.conv2.to(BF), lv.intr, lv.p, lv.D, Bb, grid=lv.grid, robust=kind, robust_scale=scale),
                           sc.R0, sc.T0, Wt, per_point=True)
            b = _o.lm_cost(_o.Level(widen(lv.conv1), widen(lv.conv2), lv.intr, lv.p, lv.D, None if Bb is None else Bb.float(), grid=lv.grid,
                                    robust=kind, robust_scale=scale), sc.R0, sc.T0, Wt, per_point=True)
            for x, y in zip(a, b):
                assert torch.equal(x, y), (C, kind)


def _backward_case(feat, basis, seed=67):
    C, K = 8, 6
    sc = scene_case(nb=2, C=C, K=K, level_ids=(3,), seed=seed, n_points=400, dtype=torch.float32)
    lv = sc.levels[0]
    a = oracle_level_inputs(lv)
    if feat == "bf16":
        a["conv1"], a["conv2"] = a["conv1"].to(BF).double(), a["conv2"].to(BF).double()
    if basis == "bf16":
        a["B"] = a["B"].to(BF).double()
    a["F2"] = a["conv2"][..., :C].contiguous()
    a["weight"] = 0.5 + torch.rand(2, lv.N, 1, generator=torch.Generator().manual_seed(8), dtype=torch.float64)
    return sc, lv, a, C, K


@gpu
@pytest.mark.parametrize("basis", ["f32", "bf16"])
@pytest.mark.parametrize("feat", ["f32", "bf16"])
@pytest.mark.parametrize("layout", ["3c", "f2"])
@pytest.mark.parametrize("kind", KINDS)
def test_backward_matches_float64_autograd(kind, layout, feat, basis):
    from banet_b200 import ops
    _lib.require_device()
    sc, lv, a, C, K = _backward_case(feat, basis)
    R0d, T0d, W0d = sc.R0.double(), sc.T0.double(), sc.W0.double() + 0.01
    s = RO.squared_norms(a["conv1"], a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"], R0d, T0d, W0d)
    delta = _delta(s)[0] if kind else 0.0
    dcost = torch.tensor([0.7, -1.3], dtype=torch.float64)
    names = ["conv1", "F2" if layout == "f2" else "conv2", "D", "B", "weight"]
    t = {n: a[n].clone().requires_grad_() for n in names}
    conv2_o = torch.cat([t["F2"], O.grad_fixed(t["F2"])], dim=-1) if layout == "f2" else t["conv2"]
    R, T, W = R0d.clone().requires_grad_(), T0d.clone().requires_grad_(), W0d.clone().requires_grad_()
    ref = CO.cost(t["conv1"], conv2_o, a["fx"], a["fy"], a["ox"], a["oy"], a["p"], t["D"], t["B"], R, T, W, kind, delta, t["weight"])
    (ref * dcost).sum().backward()
    want = dict({n: t[n].grad for n in names}, R=R.grad, T=T.grad, W=W.grad)
    dt = BF if feat == "bf16" else torch.float32
    conv2 = a["conv2"] if layout == "3c" else a["F2"]
    L = ops.Level(a["conv1"].to("cuda", dt), conv2.to("cuda", dt).contiguous(), to_cuda32(lv.intr), to_cuda32(lv.p), to_cuda32(a["D"]),
                  a["B"].to("cuda", BF if basis == "bf16" else torch.float32), weight=to_cuda32(a["weight"]), robust=kind, robust_scale=delta)
    Wg = to_cuda32(W0d)
    cost = ops.lm_cost(L, to_cuda32(R0d), to_cuda32(T0d), Wg)[0]
    assert rel_fro(cost.cpu().double(), ref.detach()) < 1e-5
    dconv1, dconv2, dD, dB, dR, dT, dW, dweight = ops.lm_cost_bwd(L, to_cuda32(R0d), to_cuda32(T0d), Wg, to_cuda32(dcost), return_dweight=True)
    got = {"conv1": dconv1, names[1]: dconv2, "D": dD, "B": dB, "weight": dweight, "R": dR, "T": dT, "W": dW}
    for n in names + ["R", "T", "W"]:
        e = rel_fro(got[n].cpu().double(), want[n])
        print(f"  d{n}: {e:.2e}")
        assert e < 2e-4, n
    if layout == "3c":
        assert bool((dconv2[..., C:] == 0).all())
    # a pair with dcost = 0 gets zero gradients, and the other pair's are unchanged
    z = ops.lm_cost_bwd(L, to_cuda32(R0d), to_cuda32(T0d), Wg, torch.tensor([0.7, 0.0], device="cuda"), return_dweight=True)
    for x, y in zip(z, (dconv1, dconv2, dD, dB, dR, dT, dW, dweight)):
        assert bool((x[1] == 0).all())
        assert rel_fro(x[0].cpu().double(), y[0].cpu().double()) < 1e-6


def _affine_gpu(K, seed, weighted):
    sc, a, W, c = _affine_case(K, seed, weighted)
    intr = torch.stack([a["fx"][:, 0], a["fy"][:, 0], a["ox"][:, 0], a["oy"][:, 0]], -1)
    g = {k: to_cuda32(v) for k, v in a.items()}
    return sc, g, to_cuda32(intr), to_cuda32(W), to_cuda32(c), a


@gpu
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("K", [0, 16])
def test_descent_identity_on_the_library(K, kind, weighted):
    """-2 g of ops.lm_build (FP32_SIMT) equals the gradient of autograd.feature_metric_cost through the SE(3) / W update at 0: the new
    kernels are tied to the build's Jacobians and to the update's sign convention."""
    from banet_b200 import ops, autograd as AG
    _lib.require_device()
    sc, g, intr, W, c, a = _affine_gpu(K, 23 + K, weighted)
    R, T = to_cuda32(sc.R0), to_cuda32(sc.T0)
    s = RO.squared_norms(*_args(a), sc.R0, sc.T0, None if W is None else W.cpu().double())
    delta = math.sqrt(float(s[s > 0].median())) if kind else 0.0
    for layout in ("3c", "f2"):
        C = g["conv1"].shape[2]
        conv2 = g["conv2"] if layout == "3c" else g["conv2"][..., :C].contiguous()
        L = ops.Level(g["conv1"], conv2, intr, g["p"], g["D"], g["B"], weight=c, robust=kind, robust_scale=delta)
        _, gb, _, nv = ops.lm_build(L, R, T, W, _lib.PREC_FP32_SIMT)
        assert float(nv.min()) == g["conv1"].shape[1]
        xi = torch.zeros(2, 6, device="cuda", requires_grad=True)
        dl = torch.zeros(2, K, device="cuda", requires_grad=True)
        Rn, Tn, Wn = _lm_update(R, T, W, xi, dl)
        cost = AG.feature_metric_cost(g["conv1"], conv2, g["D"], g["B"], Rn, Tn, Wn, intr, g["p"], weight=c, robust=kind, robust_scale=delta)
        grads = torch.autograd.grad(cost.sum(), (xi, dl) if K else (xi,))
        got = torch.cat([t.reshape(2, -1) for t in grads], -1)
        e = rel_fro(got, -2.0 * gb)
        print(f"K={K} {kind} weighted={weighted} {layout}: {e:.2e}")
        assert e < 1e-4, layout


@gpu
def test_batches_past_65535_pairs():
    from banet_b200 import ops
    _lib.require_device()
    nb, N, C, K, h, w = 65537, 16, 4, 2, 8, 8
    g = torch.Generator(device="cuda").manual_seed(5)
    r = lambda *s: torch.rand(*s, device="cuda", generator=g)
    fx = fy = 6.0
    ox, oy = 3.5, 3.5
    u, v = 0.5 + r(nb, N) * (w - 2), 0.5 + r(nb, N) * (h - 2)
    p = torch.stack([(u - ox) / fx, (v - oy) / fy, torch.ones_like(u)], 1).contiguous()
    D = (1.0 + r(nb, N, 1)).contiguous()
    B = (0.1 * r(nb, N, K)).contiguous()
    W = (0.1 * r(nb, K, 1) - 0.05).contiguous()
    intr = torch.tensor([fx, fy, ox, oy], device="cuda").expand(nb, 4).contiguous()
    Rm = torch.linalg.matrix_exp(_skew(0.02 * (r(nb, 3) - 0.5)))
    T = (0.02 * (r(nb, 3, 1) - 0.5)).contiguous()
    conv1, conv2 = r(nb, N, C), r(nb, h, w, 3 * C)
    weight = 0.5 + r(nb, N, 1)
    full = ops.Level(conv1, conv2, intr, p, D, B, weight=weight, robust="cauchy", robust_scale=0.5)
    out = ops.lm_cost(full, Rm, T, W, per_point=True)
    dcost = r(nb) - 0.5
    bw = ops.lm_cost_bwd(full, Rm, T, W, dcost, return_dweight=True)
    assert float(out[1].min()) > 0
    pick = torch.tensor([0, 1, 2, 40000, 65534, 65535, 65536], device="cuda")
    sub = lambda t: t[pick].contiguous()
    small = ops.Level(sub(conv1), sub(conv2), sub(intr), sub(p), sub(D), sub(B), weight=sub(weight), robust="cauchy", robust_scale=0.5)
    out_s = ops.lm_cost(small, sub(Rm), sub(T), sub(W), per_point=True)
    for x, y in zip(out, out_s):
        assert torch.equal(x[pick], y)
    bw_s = ops.lm_cost_bwd(small, sub(Rm), sub(T), sub(W), sub(dcost), return_dweight=True)
    # one writer per element (dconv1, dD, dB, dweight), and dR, dT, dW of a one-tile pair (two warp sums: their order cannot matter)
    for i in (0, 2, 3, 4, 5, 6, 7):
        assert torch.equal(bw[i][pick], bw_s[i]), i
    assert rel_fro(bw[1][pick], bw_s[1]) < 1e-6                     # dconv2: taps shared by points, accumulated with atomics


@gpu
def test_python_layers():
    from banet_b200 import ops, autograd as AG
    from banet_b200.bundlenet import BundleNet
    _lib.require_device()
    sc, lv, Wt = _gpu_scene(16, 8, seed=171)
    fx, fy, ox, oy = lv.intr_tiled()
    c = (0.5 + torch.rand(2, lv.N, 1, generator=torch.Generator().manual_seed(3))).cuda()
    net = BundleNet(16, levels=("3",)).cuda()
    for kind in KINDS:
        scale = 2.0 if kind else 0.0
        for B, W in ((lv.B, Wt), (None, None)):
            for weight in (None, c):
                L = ops.Level(lv.conv1, lv.conv2, lv.intr, lv.p, lv.D, B, weight=weight, robust=kind, robust_scale=scale)
                ref = ops.lm_cost(L, sc.R0, sc.T0, W)[0]
                with torch.no_grad():
                    got = net.FeatureMetricCost(lv.conv1, lv.conv2, fx, fy, ox, oy, lv.p, lv.D, B, sc.R0, sc.T0, W, weight, robust=kind,
                                                robust_scale=scale)
                assert torch.equal(got, ref)
                # with gradients: the autograd function, whose gradients are ops.lm_cost_bwd's
                leaves = dict(conv1=lv.conv1.clone().requires_grad_(), conv2=lv.conv2.clone().requires_grad_(), D=lv.D.clone().requires_grad_(),
                              R=sc.R0.clone().requires_grad_(), T=sc.T0.clone().requires_grad_())
                if B is not None:
                    leaves.update(B=B.clone().requires_grad_(), W=W.clone().requires_grad_())
                if weight is not None:
                    leaves["weight"] = weight.clone().requires_grad_()
                cost = net.FeatureMetricCost(leaves["conv1"], leaves["conv2"], fx, fy, ox, oy, lv.p, leaves["D"], leaves.get("B"), leaves["R"],
                                             leaves["T"], leaves.get("W"), leaves.get("weight"), robust=kind, robust_scale=scale)
                assert torch.equal(cost.detach(), ref) and cost.requires_grad
                dc = torch.tensor([0.3, -2.0], device="cuda")
                (cost * dc).sum().backward()
                want = ops.lm_cost_bwd(L, sc.R0, sc.T0, W, dc, return_dweight=True)
                names = ["conv1", "conv2", "D", "B", "R", "T", "W", "weight"]
                for n, x in zip(names, want):
                    if n in leaves:
                        atomic = n in ("conv2", "R", "T", "W")
                        assert (rel_fro(leaves[n].grad, x) < 1e-6) if atomic else torch.equal(leaves[n].grad, x), (kind, B is None, n)
    # bf16 inputs: gradients come back in bf16
    c1, c2 = lv.conv1.to(BF).requires_grad_(), lv.conv2.to(BF).requires_grad_()
    Bb = lv.B.to(BF).requires_grad_()
    AG.feature_metric_cost(c1, c2, lv.D, Bb, sc.R0, sc.T0, Wt, lv.intr, lv.p).sum().backward()
    assert c1.grad.dtype == BF and c2.grad.dtype == BF and Bb.grad.dtype == BF
    # argument errors before any kernel
    with pytest.raises(_lib.BanetError, match="robust"):
        net.FeatureMetricCost(lv.conv1, lv.conv2, fx, fy, ox, oy, lv.p, lv.D, lv.B, sc.R0, sc.T0, Wt, robust="tukey", robust_scale=1.0)
    with pytest.raises(_lib.BanetError, match="robust_scale"):
        net.FeatureMetricCost(lv.conv1.clone().requires_grad_(), lv.conv2, fx, fy, ox, oy, lv.p, lv.D, lv.B, sc.R0, sc.T0, Wt, robust="huber")
    with pytest.raises(_lib.BanetError, match="R: expected shape"):
        net.FeatureMetricCost(lv.conv1, lv.conv2, fx, fy, ox, oy, lv.p, lv.D, lv.B, sc.R0[:1], sc.T0, Wt)
    with pytest.raises(_lib.BanetError, match="W: expected shape"):
        AG.feature_metric_cost(lv.conv1.clone().requires_grad_(), lv.conv2, lv.D, lv.B, sc.R0, sc.T0, Wt[:, :3], lv.intr, lv.p)
