"""Robust losses of the feature-metric error (banet_level_t::robust, robust_scale): each build is one IRLS step, point n weighted by
w_n = c_n rho'(|d_n|^2) on the point-weight path, with lambda and the in-bounds count unweighted.  The float64 statement
(tests/robust_oracle.py) is tied to the weighted statement on the CPU and fixes the planted-outlier constants; the build kernels, their
backward (with the rho'' term of the weight), the whole solves, the per-pair windows and BundleNet are held to it on the GPU."""
import ctypes
import math
import os
import subprocess

import pytest
import torch

from helpers import O, scene_case, oracle_level_inputs, mlp_for, rel_fro, to_cuda32
import robust_oracle as RO
import weighted_oracle as WO
import weighted_window_oracle as WWO
from banet_b200 import _lib

gpu = pytest.mark.gpu
BF = torch.bfloat16
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# The planted-outlier scene: 20 % of the points' conv1 rows are another point's features.  Two levels x 3 iterations at lambda = 0.01,
# delta = 1 (features have unit variance per channel, C = 16).  Pose errors |R - R*|_F + |T - T*| of the float64 solves (measured here):
# L2 4.19e-3, Huber 9.0e-4, Cauchy 6.5e-4.
OUTLIER_ITERS, OUTLIER_LAMBDA, OUTLIER_DELTA = 3, 0.01, 1.0
OUTLIER_L2_MIN, OUTLIER_CAUCHY_MAX, OUTLIER_MARGIN = 3e-3, 1e-3, 4.0


def outlier_scene(device="cpu", dtype=torch.float64, seed=71, frac=0.2, C=16, K=16):
    sc = scene_case(nb=1, H=96, W=128, C=C, K=K, level_ids=(2, 3), seed=seed, dtype=torch.float64)
    g = torch.Generator().manual_seed(seed)
    for lv in sc.levels:
        N = lv.N
        bad = torch.randperm(N, generator=g)[: int(frac * N)]
        src = torch.randperm(N, generator=g)[: bad.numel()]
        lv.conv1[:, bad] = lv.conv1[:, src].clone()
    return sc


def _oracle_levels(sc, C):
    out = []
    for l in sc.levels:
        a = {k: (None if v is None else v.cpu().double()) for k, v in oracle_level_inputs(l).items()}
        out.append(O.LevelInputs(a["conv1"], a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"], mlp_for(C, l.level)))
    return out


def _pose_err(sc, R, T):
    return float((R.cpu().double() - sc.R_true.cpu().double()).norm() + (T.cpu().double() - sc.T_true.cpu().double()).norm())


def _outlier_solves():
    sc = outlier_scene()
    lvs = _oracle_levels(sc, 16)
    opts = O.IterOptions(l2_regularizer_base=1000.0, guard_nonfinite=True, lambda_override=torch.tensor([OUTLIER_LAMBDA], dtype=torch.float64))
    out = {"l2": WO.solve(lvs, [None, None], OUTLIER_ITERS, sc.R0, sc.T0, sc.W0, opts)}
    for kind in ("huber", "cauchy"):
        out[kind] = RO.solve(lvs, kind, [OUTLIER_DELTA] * 2, OUTLIER_ITERS, sc.R0, sc.T0, sc.W0, opts=opts)
    return sc, out


# ------------------------------------------------------------------------------------------------ CPU: the robust statement
def _case(K, seed=3, n_points=300, C=8):
    sc = scene_case(nb=2, C=C, K=K, level_ids=(3,), seed=seed, n_points=n_points)
    a = oracle_level_inputs(sc.levels[0])
    W = None if K == 0 else sc.W0 + 0.01
    return sc, a, W


def _args(a):
    return (a["conv1"], a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"])


@pytest.mark.parametrize("K", [0, 5])
def test_huber_above_every_residual_is_the_weighted_statement(K):
    sc, a, W = _case(K)
    s = RO.squared_norms(*_args(a), sc.R0, sc.T0, W)
    delta = 1.01 * math.sqrt(float(s.max()))
    c = 2 * torch.rand(2, a["conv1"].shape[1], 1, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    for weight in (None, c):
        mine = RO.normal_equations(*_args(a), sc.R0, sc.T0, W, "huber", delta, weight)
        ref = WO.normal_equations(*_args(a), sc.R0, sc.T0, W, weight)
        for x, y in zip(mine, ref):
            assert torch.equal(x, y)


def test_weight_functions_pass_gradcheck():
    s = torch.tensor([0.1, 0.5, 2.0, 3.5, 9.0], dtype=torch.float64, requires_grad=True)      # Huber kink at delta^2 = 1.44: not hit
    for kind in ("huber", "cauchy"):
        assert torch.autograd.gradcheck(lambda x: RO.rho1(kind, 1.2, x), (s,))
    # and rho'' is what the kernels use
    r = RO.rho1("cauchy", 1.2, s)
    (d2,) = torch.autograd.grad(r.sum(), s)
    assert torch.allclose(d2, -1.44 / (1.44 + s.detach()) ** 2)
    r = RO.rho1("huber", 1.2, s)
    (d2,) = torch.autograd.grad(r.sum(), s)
    sd = s.detach()
    assert torch.allclose(d2, torch.where(sd > 1.44, -0.5 * 1.2 / sd ** 1.5, torch.zeros_like(sd)))


def test_robust_gradient_carries_the_rho_second_derivative_term():
    sc, a, W = _case(5, seed=6)
    conv1 = a["conv1"].clone().requires_grad_()
    args = (conv1,) + _args(a)[1:]
    s = RO.squared_norms(*_args(a), sc.R0, sc.T0, W)
    delta = math.sqrt(float(s[s > 0].median()))
    gens = []
    for detach in (False, True):
        H, g, _, _ = RO.normal_equations(*args, sc.R0, sc.T0, W, "cauchy", delta, None, detach)
        (gr,) = torch.autograd.grad(H.sum() + g.sum(), conv1)
        gens.append(gr)
    assert rel_fro(gens[0], gens[1]) > 1e-2


def test_planted_outliers_are_resisted_by_the_robust_losses():
    sc, out = _outlier_solves()
    e = {k: _pose_err(sc, R, T) for k, (R, T, _) in out.items()}
    print("planted-outlier pose errors (float64):", e)
    assert e["l2"] > OUTLIER_L2_MIN and e["cauchy"] < OUTLIER_CAUCHY_MAX and e["l2"] > OUTLIER_MARGIN * e["cauchy"]
    assert e["huber"] < e["l2"]


# ------------------------------------------------------------------------------------------------ CPU: the C-ABI
def _level(**kw):
    lv = _lib.BanetLevel(2, 4096, 64, 32, 48, 64, 192, 1, 1, 1, 1, 1, 1, 0, 0)
    for k, v in kw.items():
        setattr(lv, k, v)
    return lv


BAD_ROBUST = [dict(robust=3, robust_scale=1.0), dict(robust=-1, robust_scale=1.0)] + \
             [dict(robust=k, robust_scale=s) for k in (1, 2) for s in (0.0, -1.0, float("nan"), float("inf"))]


def _entries(lib, lv):
    """(name, rc) of every level-taking entry on one level lv (dummy device pointers: only argument checks may run)."""
    arr = (_lib.BanetLevel * 1)(lv)
    opts = _lib.BanetSolveOpts(1e-5, 1, 0)
    out = [("lm_build", lib.banet_lm_build(ctypes.byref(lv), 1, 1, 1, 0, 1, 1, 1, 1, 1, 1 << 30, None)),
           ("lm_build_bwd", lib.banet_lm_build_bwd(ctypes.byref(lv), 1, 1, 1, 1, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1, None)),
           ("lm_build_bwd_weighted", lib.banet_lm_build_bwd_weighted(ctypes.byref(lv), 1, 1, 1, 1, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1, 1, None)),
           ("lm_run", lib.banet_lm_run(arr, 1, 1, None, 1000.0, 1.0, ctypes.byref(opts), 0, 1, 1, 1, 1, 1, 1 << 30, None)),
           ("lm_window_run", lib.banet_lm_window_run(arr, 1, 1, None, 1000.0, 1.0, ctypes.byref(opts), 0, 1, 1, 1, 1, 1, 1 << 30, None)),
           ("lm_window_batch_run", lib.banet_lm_window_batch_run(arr, 1, 1, 1, None, 1000.0, 1.0, ctypes.byref(opts), 0, 1, 1, 1, 1, 1, 1 << 30,
                                                                  None))]
    return out


def _workspace_queries(lib, lv):
    arr = (_lib.BanetLevel * 1)(lv)
    return [lib.banet_lm_build_workspace_bytes(ctypes.byref(lv), 0), lib.banet_lm_run_workspace_bytes(arr, 1, 0),
            lib.banet_lm_window_run_workspace_bytes(arr, 1, 0), lib.banet_lm_window_batch_run_workspace_bytes(arr, 1, 1, 0)]


@pytest.mark.parametrize("bad", BAD_ROBUST, ids=lambda d: f"{d['robust']}-{d['robust_scale']}")
def test_level_entries_reject_bad_robust_arguments_without_gpu(bad):
    lib = _lib.load()
    for name, rc in _entries(lib, _level(**bad)):
        assert rc == -1 and b"robust" in lib.banet_last_error(), name
    assert _workspace_queries(lib, _level(**bad)) == [0, 0, 0, 0]


def test_legacy_tracker_rejects_robust_levels_and_none_takes_any_scale():
    lib = _lib.load()
    iters = (ctypes.c_int * 1)(3)
    legacy = _lib.BanetLegacyOpts(1, 1e-5, 2e-4, 1.0)
    for kind in (1, 2):
        arr = (_lib.BanetLevel * 1)(_level(K=0, robust=kind, robust_scale=0.5))
        rc = lib.banet_lm_track_legacy(arr, 1, iters, None, ctypes.byref(legacy), 1, 1, None, 1, 1, 1, 1 << 20, None)
        assert rc == -4 and b"robust" in lib.banet_last_error()
    # robust = 0 ignores the scale: the entries fail on the (deliberately) bad shape, never on the scale
    for scale in (0.0, -1.0, float("nan"), float("inf")):
        lv = _level(robust=0, robust_scale=scale, nb=0)
        for name, rc in _entries(lib, lv):
            assert rc == -1 and b"robust" not in lib.banet_last_error(), name
        assert _workspace_queries(lib, _level(robust=0, robust_scale=scale))[0] > 0


def test_struct_matches_the_header(tmp_path):
    assert _lib.BanetLevel(2, 1, 1, 1, 2, 2, 3).robust == 0
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "banet_abi.h"\n'
                   'int main(void) { printf("%zu %zu %zu %d %d %d\\n", sizeof(banet_level_t), offsetof(banet_level_t, robust), '
                   'offsetof(banet_level_t, robust_scale), BANET_ROBUST_NONE, BANET_ROBUST_HUBER, BANET_ROBUST_CAUCHY); return 0; }\n')
    exe = tmp_path / "layout"
    cc = os.environ.get("CC", "cc")
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    want = [ctypes.sizeof(_lib.BanetLevel), _lib.BanetLevel.robust.offset, _lib.BanetLevel.robust_scale.offset,
            _lib.ROBUST_NONE, _lib.ROBUST_HUBER, _lib.ROBUST_CAUCHY]
    assert [int(x) for x in got] == want


def test_ops_level_validates_the_robust_loss():
    from banet_b200 import ops
    assert ops.robust_kind(None, -3.0) == (0, 0.0)
    assert ops.robust_kind("huber", 2) == (1, 2.0) and ops.robust_kind("cauchy", 0.5) == (2, 0.5)
    for kind, scale in (("tukey", 1.0), ("huber", 0.0), ("cauchy", -1.0), ("huber", float("nan")), ("cauchy", float("inf"))):
        with pytest.raises(_lib.BanetError, match="robust"):
            ops.robust_kind(kind, scale)


# ------------------------------------------------------------------------------------------------ GPU
PRECS = {"simt": _lib.PREC_FP32_SIMT, "x1": _lib.PREC_TF32X1, "x2": _lib.PREC_TF32X2, "x3": _lib.PREC_TF32X3, "auto": _lib.PREC_AUTO}
TOL = {"simt": 2e-5, "x1": 5e-4, "x2": 1e-4, "x3": 2e-6}


def _gpu_scene(C, K, seed, H=48, W=64):
    from banet_b200 import synth
    sc = synth.make_scene(nb=2, H=H, W=W, C=C, K=K, level_ids=(3,), seed=seed, device="cuda", dtype=torch.float32)
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


def _oracle_inputs(lv, layout, feat, basis):
    """Oracle inputs of a GPU scene level as the kernels read them: bf16 tensors rounded first, and in the F2-only layout the gradient
    channels derived from F2 as the build derives them."""
    a = {k: (None if v is None else v.cpu()) for k, v in oracle_level_inputs(lv).items()}
    rnd = (lambda t: t.to(BF).cpu().double()) if feat == "bf16" else (lambda t: t.cpu().double())
    a["conv1"] = rnd(lv.conv1)
    C = lv.conv1.shape[2]
    a["conv2"] = rnd(lv.conv2) if layout == "3c" else torch.cat([rnd(lv.conv2[..., :C]), O.grad_fixed(rnd(lv.conv2[..., :C]))], dim=-1)
    if basis == "bf16" and a["B"] is not None:
        a["B"] = lv.B.to(BF).cpu().double()
    return a


def _pick_delta(s, lo=0.4, hi=0.7, kink=True):
    """delta^2 in the widest relative gap of the sorted valid s between their lo and hi quantiles, so that 30-60 % of the valid points are
    down-weighted; kink: and no valid point lies within 1e-3 relative of Huber's delta^2 (the fp32 and float64 s could fall on opposite
    sides of it, where rho'' jumps).  A solve moves s away from where it was checked, so the whole-solve tests, which compare forward
    results only (rho' is continuous at the kink), do not ask for it."""
    v = torch.sort(s[s > 0].flatten()).values
    i0, i1 = int(lo * v.numel()), int(hi * v.numel())
    rel = (v[i0 + 1:i1 + 1] - v[i0:i1]) / v[i0:i1]
    j = i0 + int(torch.argmax(rel))
    t = math.sqrt(float(v[j] * v[j + 1]))
    if kink:
        assert float(((v - t).abs() / t).min()) > 1e-3
    return math.sqrt(t), float((v > t).double().mean())


@gpu
@pytest.mark.parametrize("kind", ["huber", "cauchy"])
@pytest.mark.parametrize("C", [64, 128])
@pytest.mark.parametrize("K", [128, 16, 0])
def test_robust_build_matches_the_float64_statement(K, C, kind):
    from banet_b200 import ops
    _lib.require_device()
    sc, lv, Wt = _gpu_scene(C, K, seed=43 + K + C)
    R0d, T0d, Wd = sc.R0.cpu().double(), sc.T0.cpu().double(), None if Wt is None else Wt.cpu().double()
    c = (0.5 + torch.rand(2, lv.N, 1, generator=torch.Generator().manual_seed(5))).cuda()
    precs = ("simt", "x1", "x2", "x3", "auto") if K == 128 else ("simt", "auto")
    for feat in ("f32", "bf16"):
        for basis in (("f32", "bf16") if K else ("f32",)):
            for layout in ("3c", "f2"):
                a = _oracle_inputs(lv, layout, feat, basis)
                s = RO.squared_norms(*_args(a), R0d, T0d, Wd)
                delta, frac = _pick_delta(s)
                print(f"K={K} C={C} {kind} {feat}/{basis}/{layout}: delta={delta:.4g}, {100 * frac:.0f} % of the valid points down-weighted")
                assert 0.3 <= frac <= 0.6
                for weight in (None, c):
                    rH, rg, rrbar, rnv = RO.normal_equations(*_args(a), R0d, T0d, Wd, kind, delta, None if weight is None else weight.cpu().double())
                    for pn in precs:
                        tol = TOL["x3" if K == 128 else "simt"] if pn == "auto" else TOL[pn]
                        L = _level_of(lv, layout, feat, basis, True, weight, kind, delta)
                        H, g, rbar, nv = ops.lm_build(L, sc.R0, sc.T0, Wt, PRECS[pn])
                        eH, eg = rel_fro(H.cpu().double(), rH), rel_fro(g.cpu().double(), rg.squeeze(-1))
                        assert eH < tol and eg < tol, (feat, basis, weight is None, layout, pn, eH, eg)
                        assert rel_fro(rbar.cpu().double() / lv.N, rrbar.squeeze(1)) < 2e-5 and torch.equal(nv.cpu().double(), rnv)


@gpu
@pytest.mark.parametrize("K", [128, 32, 16, 0])
def test_huber_above_every_residual_gives_the_plain_bits(K):
    from banet_b200 import ops
    _lib.require_device()
    sc, lv, Wt = _gpu_scene(64, K, seed=53 + K)
    a = oracle_level_inputs(lv)
    a = {k: (None if v is None else v.cpu()) for k, v in a.items()}
    s = RO.squared_norms(*_args(a), sc.R0.cpu().double(), sc.T0.cpu().double(), None if Wt is None else Wt.cpu().double())
    big = 10.0 * math.sqrt(float(s.max()))
    c = (0.5 + torch.rand(2, lv.N, 1, generator=torch.Generator().manual_seed(6))).cuda()
    precs = ("simt", "x1", "x2", "x3", "auto") if K in (32, 64, 128) else ("simt", "auto")
    for layout in ("3c", "f2"):
        for feat in ("f32", "bf16"):
            for basis in (("f32", "bf16") if K else ("f32",)):
                for weight in (None, c):
                    for pn in precs:
                        x = ops.lm_build(_level_of(lv, layout, feat, basis, True, weight), sc.R0, sc.T0, Wt, PRECS[pn])
                        y = ops.lm_build(_level_of(lv, layout, feat, basis, True, weight, "huber", big), sc.R0, sc.T0, Wt, PRECS[pn])
                        for u, v, name in zip(x, y, ("H", "g", "rbar_sum", "nvalid")):
                            assert torch.equal(u, v), (layout, feat, basis, weight is None, pn, name)


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
def test_robust_builds_are_bit_reproducible(layout, monkeypatch):
    from banet_b200 import ops
    _lib.require_device()
    sc, lv, Wt = _gpu_scene(128, 128, seed=61, H=120, W=160)
    for kind in ("huber", "cauchy"):
        L = _level_of(lv, layout, "f32", "f32", True, None, kind, 4.0)
        for pn in PRECS:
            outs = []
            for pattern in ("nan", "random"):
                monkeypatch.setattr(ops, "_ws", _poisoned_ws(pattern))
                outs.append(ops.lm_build(L, sc.R0, sc.T0, Wt, precision=PRECS[pn]))
            for a, b in zip(*outs):
                assert torch.equal(a, b), (kind, pn)
            assert bool(torch.isfinite(outs[0][0]).all())


@gpu
@pytest.mark.parametrize("basis", ["f32", "bf16"])
@pytest.mark.parametrize("feat", ["f32", "bf16"])
@pytest.mark.parametrize("layout", ["3c", "f2"])
@pytest.mark.parametrize("kind", ["huber", "cauchy"])
def test_robust_iteration_gradients_match_float64_autograd(kind, layout, feat, basis):
    """iteration_fused with a robust loss (and a confidence weight that requires grad) against float64 autograd of the robust statement at
    exact_sym = 1: every input's gradient.  The rho'' term is checked to be there: dconv1 is far closer to the full reference than to the
    reference with w_n detached."""
    from banet_b200 import autograd as AG
    _lib.require_device()
    C, K = 8, 6
    sc = scene_case(nb=2, C=C, K=K, level_ids=(3,), seed=67, n_points=400, dtype=torch.float32)
    lv = sc.levels[0]
    a = oracle_level_inputs(lv)
    if feat == "bf16":
        a["conv1"] = a["conv1"].to(BF).double()
        a["conv2"] = a["conv2"].to(BF).double()
    if basis == "bf16":
        a["B"] = a["B"].to(BF).double()
    a["F2"] = a["conv2"][..., :C].contiguous()
    a["weight"] = 0.5 + torch.rand(2, lv.N, 1, generator=torch.Generator().manual_seed(8), dtype=torch.float64)
    R0d, T0d, W0d = sc.R0.double(), sc.T0.double(), sc.W0.double() + 0.01
    s = RO.squared_norms(a["conv1"], a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"], R0d, T0d, W0d)
    delta, frac = _pick_delta(s)
    print(f"{kind} {layout} {feat}/{basis}: delta={delta:.4g}, {100 * frac:.0f} % down-weighted")
    names = ["conv1", "F2" if layout == "f2" else "conv2", "D", "B", "weight"]
    mlp = mlp_for(C, 3)
    g = torch.Generator().manual_seed(5)
    cR, cT, cW = (torch.randn(2, 3, 3, generator=g, dtype=torch.float64), torch.randn(2, 3, 1, generator=g, dtype=torch.float64),
                  torch.randn(2, K, 1, generator=g, dtype=torch.float64))
    opts = O.IterOptions(l2_regularizer_base=1000.0, guard_nonfinite=True)
    refs = {}
    for detach in (False, True):
        t = {n: a[n].clone().requires_grad_() for n in names}
        conv2_o = torch.cat([t["F2"], O.grad_fixed(t["F2"])], dim=-1) if layout == "f2" else t["conv2"]
        R, T, W = R0d.clone().requires_grad_(), T0d.clone().requires_grad_(), W0d.clone().requires_grad_()
        oR, oT, oW = RO.iteration(t["conv1"], conv2_o, a["fx"], a["fy"], a["ox"], a["oy"], a["p"], t["D"], t["B"], R, T, W, mlp, kind, delta,
                                  t["weight"], opts, detach_weight=detach)
        ((oR * cR).sum() + (oT * cT).sum() + (oW * cW).sum()).backward()
        refs[detach] = (dict({n: t[n].grad for n in names}, R=R.grad, T=T.grad, W=W.grad), oR, oT)
    want, oR, oT = refs[False]
    dt = BF if feat == "bf16" else torch.float32
    bdt = BF if basis == "bf16" else torch.float32
    tg = {n: a[n].detach().to("cuda", dt if n in ("conv1", "conv2", "F2") else (bdt if n == "B" else torch.float32)).contiguous().requires_grad_()
          for n in names}
    Rg, Tg, Wg = to_cuda32(sc.R0).requires_grad_(), to_cuda32(sc.T0).requires_grad_(), to_cuda32(sc.W0 + 0.01).requires_grad_()
    mlp32 = [(to_cuda32(w), to_cuda32(b)) for w, b in mlp]
    gR, gT, gW = AG.iteration_fused(tg["conv1"], tg[names[1]], to_cuda32(lv.intr), to_cuda32(lv.p), tg["D"], tg["B"], Rg, Tg, Wg, mlp32, 1000.0,
                                    exact_sym=True, weight=tg["weight"], robust=kind, robust_scale=delta)
    assert rel_fro(gR.cpu().double(), oR) < 1e-5 and rel_fro(gT.cpu().double(), oT) < 1e-4
    ((gR * cR.float().cuda()).sum() + (gT * cT.float().cuda()).sum() + (gW * cW.float().cuda()).sum()).backward()
    tol = 2e-3 if feat == "f32" and basis == "f32" else 5e-3
    got = dict(tg, R=Rg, T=Tg, W=Wg)
    for n in names + ["R", "T", "W"]:
        e = rel_fro(got[n].grad.float().cpu().double(), want[n].cpu())
        print(f"  d{n}: {e:.2e}")
        assert e < tol, n
    gap = rel_fro(refs[True][0]["conv1"], want["conv1"])
    print(f"  dconv1: full vs detached-weight reference {gap:.2e}")
    assert gap > 10 * tol
    assert rel_fro(tg["conv1"].grad.float().cpu().double(), want["conv1"]) < 0.1 * gap


def _solve_levels(sc, kind, deltas, weights=None, layout="3c"):
    from banet_b200 import ops
    out = []
    for i, l in enumerate(sc.levels):
        C = l.conv1.shape[2]
        conv2 = l.conv2 if layout == "3c" else l.conv2[..., :C].contiguous()
        out.append(ops.Level(l.conv1, conv2, l.intr, l.p, l.D, l.B, grid=l.grid, weight=None if weights is None else weights[i],
                             robust=kind, robust_scale=deltas[i] if kind else 0.0))
    return out


@gpu
@pytest.mark.parametrize("kind", ["huber", "cauchy"])
def test_robust_whole_solves_match_the_float64_statement(kind):
    from banet_b200 import ops, autograd as AG, synth
    _lib.require_device()
    C, K = 64, 16
    sc = synth.make_scene(nb=2, H=96, W=128, C=C, K=K, level_ids=(2, 3), seed=73, device="cuda", dtype=torch.float32)
    olv = _oracle_levels(sc, C)
    deltas = []
    for l, o in zip(sc.levels, olv):
        s = RO.squared_norms(o.conv1, o.conv2, o.fx, o.fy, o.ox, o.oy, o.p, o.D, o.B, sc.R0.cpu().double(), sc.T0.cpu().double(),
                             sc.W0.cpu().double())
        deltas.append(_pick_delta(s, kink=False)[0])
    opts = O.IterOptions(l2_regularizer_base=1000.0, guard_nonfinite=True)
    oR, oT, oW = RO.solve(olv, kind, deltas, 2, sc.R0.cpu().double(), sc.T0.cpu().double(), sc.W0.cpu().double(), opts=opts)
    mlps = [mlp_for(C, l.level, torch.float32) for l in sc.levels]
    packed = [ops.pack_mlp(m).cuda() for m in mlps]
    levels = _solve_levels(sc, kind, deltas)
    for prec in (_lib.PREC_FP32_SIMT, _lib.PREC_AUTO):
        R, T, W, st = ops.lm_run(levels, 2, sc.R0, sc.T0, sc.W0, mlp_packed=packed, l2_regularizer_base=1000.0, precision=prec)
        e = dict(R=rel_fro(R.cpu().double(), oR), T=rel_fro(T.cpu().double(), oT), W=rel_fro(W.cpu().double(), oW))
        print(kind, prec, e)
        assert int(st.abs().max()) == 0 and max(e.values()) < 1e-4, (prec, e)
        mlp_cuda = [[(w.cuda(), b.cuda()) for w, b in m] for m in mlps]
        aR, aT, aW = AG.lm_run(levels, 2, sc.R0, sc.T0, sc.W0, mlp_params=mlp_cuda, l2_regularizer_base=1000.0, precision=prec)
        assert torch.equal(aR, R) and torch.equal(aT, T) and torch.equal(aW, W)
        graph = ops.LMRunGraph(levels, 2, packed, l2_regularizer_base=1000.0, precision=prec)
        gR, gT, gW, _ = graph.solve(sc.R0, sc.T0, sc.W0)
        assert torch.equal(gR, R) and torch.equal(gT, T) and torch.equal(gW, W)
    plain = _solve_levels(sc, None, deltas)
    R0, _, _, _ = ops.lm_run(plain, 2, sc.R0, sc.T0, sc.W0, mlp_packed=packed, l2_regularizer_base=1000.0)
    assert not torch.equal(R0, R)


@gpu
def test_planted_outliers_on_the_gpu():
    from banet_b200 import ops
    _lib.require_device()
    sc, out = _outlier_solves()
    gsc = outlier_scene()
    for l in gsc.levels:
        for k in ("conv1", "conv2", "intr", "p", "D", "B"):
            setattr(l, k, to_cuda32(getattr(l, k)))
    R0, T0, W0 = to_cuda32(sc.R0), to_cuda32(sc.T0), to_cuda32(sc.W0)
    errs = {}
    for kind in ("l2", "huber", "cauchy"):
        levels = _solve_levels(gsc, None if kind == "l2" else kind, [OUTLIER_DELTA] * 2)
        R, T, W, st = ops.lm_run(levels, OUTLIER_ITERS, R0, T0, W0, lambda_fixed=OUTLIER_LAMBDA, l2_regularizer_base=1000.0,
                                 precision=_lib.PREC_FP32_SIMT)
        oR, oT, oW = out[kind]
        errs[kind] = _pose_err(sc, R, T)
        print(kind, "pose error", errs[kind], "float64", _pose_err(sc, oR, oT), "rel T", rel_fro(T.cpu().double(), oT))
        assert int(st.abs().max()) == 0 and rel_fro(R.cpu().double(), oR) < 1e-4 and rel_fro(T.cpu().double(), oT) < 1e-3
    assert errs["l2"] > OUTLIER_MARGIN * errs["cauchy"]


@gpu
def test_robust_window_batch_run_and_window_iteration():
    from banet_b200 import ops, synth, autograd as AG
    from banet_b200.bundlenet import BundleNet
    _lib.require_device()
    nw, nf, C, K = 2, 2, 64, 32
    sc = synth.make_scene(nb=nw * nf, H=48, W=64, C=C, K=K, level_ids=(3,), seed=79, device="cuda", dtype=torch.float32, shared_depth=True,
                          window_frames=nf)
    l = sc.levels[0]
    delta = 3.0
    lv = ops.Level(l.conv1, l.conv2, l.intr, l.p, l.D, l.B, grid=l.grid, robust="cauchy", robust_scale=delta)
    Ww = sc.W0.reshape(nw, nf, K, 1)[:, 0].contiguous()
    lam = 0.05
    R, T, W, st = ops.lm_window_batch_run([lv], nw, 1, sc.R0, sc.T0, Ww, lambda_fixed=lam, precision=_lib.PREC_FP32_SIMT)
    opts = O.IterOptions(l2_regularizer_base=1000.0, guard_nonfinite=True, lambda_override=torch.tensor([lam], dtype=torch.float64))
    a = {k: (None if v is None else v.cpu()) for k, v in oracle_level_inputs(l).items()}
    for w in range(nw):
        sl = slice(w * nf, (w + 1) * nf)
        aw = {k: (None if v is None else v[sl]) for k, v in a.items()}
        Rw, Tw = sc.R0[sl].cpu().double(), sc.T0[sl].cpu().double()
        Wd = Ww[w].cpu().double()
        cw = RO.robust_weight(*_args(aw), Rw, Tw, Wd.expand(nf, K, 1), "cauchy", delta)
        oR, oT, oW = WWO.window_iteration(*_args(aw), Rw, Tw, Wd, None, cw, opts)
        assert rel_fro(R[sl].cpu().double(), oR) < 1e-5 and rel_fro(W[w].cpu().double(), oW) < 1e-4, w
    assert int(st.abs().max()) == 0
    # the per-pair WindowIteration: no-grad equals lm_window_batch_run, the grad path equals window_batch_iteration_fused
    net = BundleNet(C, levels=("3",), precision=_lib.PREC_FP32_SIMT).cuda()
    net.eval()
    per = lambda t: t.reshape(nw, nf, *t.shape[1:])
    fx, fy, ox, oy = [per(t) for t in l.intr_tiled()]
    args = (per(l.conv1), per(l.conv2), fx, fy, ox, oy, per(l.p), per(l.D), per(l.B), per(sc.R0), per(sc.T0), Ww)
    with torch.no_grad():
        nR, nT, nW = net.WindowIteration(*args, 1000.0, "3", robust="cauchy", robust_scale=delta)
    bR, bT, bW, _ = ops.lm_window_batch_run([lv], nw, 1, sc.R0, sc.T0, Ww, mlp_packed=[net.mlp_packed("3")], l2_regularizer_base=1000.0,
                                            precision=_lib.PREC_FP32_SIMT)
    assert torch.equal(nR.reshape(-1, 3, 3), bR) and torch.equal(nW, bW)
    c1 = args[0].clone().requires_grad_()
    gR, gT, gW = net.WindowIteration(c1, *args[1:], 1000.0, "3", robust="cauchy", robust_scale=delta)
    (gR.sum() + gT.sum() + gW.sum()).backward()
    c2 = args[0].clone().requires_grad_()
    fR, fT, fW = AG.window_batch_iteration_fused(c2, args[1], torch.stack([t[..., 0] for t in (fx, fy, ox, oy)], -1), *args[6:], net.mlp_params("3"),
                                                  1000.0, exact_sym=net.exact_sym_grad, precision=_lib.PREC_FP32_SIMT, robust="cauchy",
                                                  robust_scale=delta)
    (fR.sum() + fT.sum() + fW.sum()).backward()
    assert torch.equal(gR, fR) and rel_fro(c1.grad, c2.grad) < 1e-6
    # the keyframe form and WindowResize have no robust loss
    key = (l.conv1.reshape(nw, nf, -1, C)[:, 0].contiguous(), args[1], fx, fy, ox, oy, per(l.p)[:, 0].contiguous(), per(l.D)[:, 0].contiguous(),
           per(l.B)[:, 0].contiguous(), args[9], args[10], Ww)
    with pytest.raises(RuntimeError, match="robust"):
        with torch.no_grad():
            net.WindowIteration(*key, 1000.0, "3", robust="huber", robust_scale=delta)
    with pytest.raises(RuntimeError, match="robust"):
        net.WindowResize(None, None, None, None, None, None, robust="huber", robust_scale=1.0)


@gpu
def test_resize_with_a_robust_loss():
    import gen_golden
    from banet_b200 import autograd as AG
    from banet_b200.bundlenet import BundleNet
    _lib.require_device()
    x = gen_golden.resize_inputs(nb=4, C=16, K=8)
    net = BundleNet(16, levels=("0", "1", "2", "3"), precision=_lib.PREC_AUTO).cuda()
    f = {k: to_cuda32(x[k]) for k in ("intr", "points", "basis", "depth", "R0", "T0")}
    layers = [to_cuda32(l) for l in x["layers"]]
    net.eval()
    scales = {"0": 2.0, "1": 2.0, "2": 1.5, "3": 1.0}
    with torch.no_grad():
        a = net.BundleResize(f["intr"], layers, f["points"], f["basis"], f["depth"], f["R0"], f["T0"], robust="cauchy", robust_scale=scales)
        b = net.BundleResize(f["intr"], layers, f["points"], f["basis"], f["depth"], f["R0"], f["T0"])
        ca = net.CameraResize(f["intr"], layers, f["points"], f["depth"], robust="huber", robust_scale=1.0)
    assert not torch.equal(a[0][-1], b[0][-1])
    assert all(bool(torch.isfinite(t).all()) for xs in a + ca for t in xs)
    # BundleIteration: no-grad equals ops, the grad path equals iteration_fused
    from banet_b200 import synth, ops
    sc = synth.make_scene(nb=2, H=48, W=64, C=16, K=8, level_ids=(3,), seed=83, device="cuda", dtype=torch.float32)
    l = sc.levels[0]
    fx, fy, ox, oy = l.intr_tiled()
    bnet = BundleNet(16, levels=("3",), precision=_lib.PREC_FP32_SIMT).cuda()
    with torch.no_grad():
        nR, nT, nW, aux = bnet.BundleIteration(l.conv1, l.conv2, fx, fy, ox, oy, l.p, l.D, l.B, sc.R0, sc.T0, sc.W0, 1000.0, "3", return_aux=True,
                                               robust="huber", robust_scale=2.0)
    H, g, _, _ = ops.lm_build(ops.Level(l.conv1, l.conv2, l.intr, l.p, l.D, l.B, robust="huber", robust_scale=2.0), sc.R0, sc.T0, sc.W0,
                              _lib.PREC_FP32_SIMT)
    assert torch.equal(aux["AtA"], H) and torch.equal(aux["Atb"], g)
    c1 = l.conv1.clone().requires_grad_()
    gR, gT, gW = bnet.BundleIteration(c1, l.conv2, fx, fy, ox, oy, l.p, l.D, l.B, sc.R0, sc.T0, sc.W0, 1000.0, "3", robust="huber", robust_scale=2.0)
    (gR.sum() + gT.sum() + gW.sum()).backward()
    c2 = l.conv1.clone().requires_grad_()
    fR, fT, fW = AG.iteration_fused(c2, l.conv2, l.intr, l.p, l.D, l.B, sc.R0, sc.T0, sc.W0, bnet.mlp_params("3"), 1000.0,
                                    exact_sym=bnet.exact_sym_grad, robust="huber", robust_scale=2.0)
    (fR.sum() + fT.sum() + fW.sum()).backward()
    assert torch.equal(gR, fR) and rel_fro(c1.grad, c2.grad) < 1e-6
