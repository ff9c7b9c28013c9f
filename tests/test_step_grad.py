"""The backward of the fused LM step (banet_lm_step_bwd: lambda-MLP, damping, Cholesky, SE(3) / W update) and the differentiable whole solve
autograd.lm_run built on it.

CPU: argument errors before any CUDA call, the (K, C) rejection edge equal to banet_lm_step's (tests/solve_plan_model.py), the workspace query.
GPU: the step backward against float64 autograd of the oracle's lambda-MLP + damping + solve + update on systems from a real build, on both
sides of every storage switch of lm_step at C = 5, 64, 128, 256; with lambda given, the same gradients as banet_lm_solve_update_bwd; the skip
contract; bit-reproducibility from poisoned workspaces; autograd.lm_run's forward equal to ops.lm_run bit for bit; its gradients against
float64 autograd of oracle.lm_solve, next to the iteration_fused loop's; its peak memory next to that loop's.
"""
import ctypes
import json
import os
import subprocess
import sys

import pytest
import torch

from helpers import ROOT, rel_fro, scene_case, mlp_for, oracle_level_inputs, to_cuda32
from oracle import ba_oracle as O
import solve_plan_model as M

U32 = 2.0 ** -24
EPS32 = float(torch.tensor(1e-5, dtype=torch.float32))
F64 = (M.SQUARE64, M.PACKED64)


def _opts(scramble=0, undamped_last=1):
    from banet_b200 import _lib
    return _lib.BanetSolveOpts(1e-5, undamped_last, scramble)


# ------------------------------------------------------------------------------------------ CPU
def test_step_bwd_rejects_bad_arguments_without_gpu():
    from banet_b200 import _lib
    lib = _lib.load()
    p = 1                                                            # non-null dummy pointers: every call below fails before a CUDA call
    args = dict(H=p, g=p, rbar=p, nb=2, N=100, C=8, K=4, mlp=p, lam=p, delta=p, opts=None, R=p, T=p, dRo=p, dTo=p, dWo=p, dH=p, dg=p, drb=p,
                dmlp=p, dlam=p, dR=p, dT=p, dW=p, ws=p, nbytes=1 << 34)

    def bwd(**kw):
        a = dict(args, **kw)
        o = a["opts"] or _opts()
        return lib.banet_lm_step_bwd(a["H"], a["g"], a["rbar"], a["nb"], a["N"], a["C"], a["K"], a["mlp"], 1000.0, a["lam"], a["delta"],
                                     ctypes.byref(o), a["R"], a["T"], a["dRo"], a["dTo"], a["dWo"], a["dH"], a["dg"], a["drb"], a["dmlp"],
                                     a["dlam"], a["dR"], a["dT"], a["dW"], a["ws"], a["nbytes"], None)

    for name in ("H", "g", "lam", "delta", "R", "T", "dRo", "dTo", "dH", "dg", "dlam", "dR", "dT"):
        assert bwd(**{name: None}) == -1, name
    for bad in (dict(nb=0), dict(K=-1), dict(dWo=None), dict(dW=None), dict(rbar=None), dict(drb=None), dict(dmlp=None), dict(N=0), dict(C=0)):
        assert bwd(**bad) == -1, bad
    assert bwd(K=0, dWo=None, dW=None, ws=None) == -2                 # K = 0 needs no dW: past the argument checks, to the workspace check
    assert bwd(opts=_opts(scramble=1)) == -4 and b"vmatrix_batch_scramble" in lib.banet_last_error()
    assert bwd(K=400) == -4 and b"K=400" in lib.banet_last_error()
    assert bwd(ws=None) == -2 and bwd(nbytes=16) == -2
    ws = lambda nb, C=8, K=4: lib.banet_lm_step_bwd_workspace_bytes(nb, C, K)
    assert ws(1) > 0 and ws(64) > ws(8) > ws(1)
    for bad in (dict(nb=0), dict(nb=1, C=0), dict(nb=1, K=-1), dict(nb=1, K=400)):
        assert ws(**bad) == 0, bad


_PROBE = r"""
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from banet_b200 import _lib
lib = _lib.load()
o = _lib.BanetSolveOpts(1e-5, 1, 0)
p = 1                                        # non-null dummy pointers: nothing below may reach a kernel, and no device is visible
out = {}
def bwd(P, C, mlp):
    return lib.banet_lm_step_bwd(p, p, p if mlp else None, 1, 100, C, P - 6, p if mlp else None, 1000.0, p, p, ctypes.byref(o), p, p, p, p, p,
                                 p, p, p if mlp else None, p if mlp else None, p, p, p, p, None, 0, None)
def fwd(P, C, mlp):
    return lib.banet_lm_step(p, p, p if mlp else None, 1, 100, C, P - 6, p if mlp else None, 1.0, None if mlp else p, ctypes.byref(o),
                             p, p, p, p, p, p, p, p, p, None)
for P, C, mlp in json.loads(sys.argv[2]):
    out[f"{P}:{C}:{mlp}"] = [bwd(P, C, mlp), fwd(P, C, mlp), lib.banet_last_error().decode()]
print(json.dumps(out))
"""


def test_rejection_edge_is_lm_steps():
    """-4 from banet_lm_step_bwd exactly where banet_lm_step rejects (the model's edge, which tests/test_solve_edges.py ties to the forward),
    at C = 5, 128, 256 with the MLP and with lambda given.  One size below, the backward gets past every size check: -2 (no workspace, MLP)
    or -3 (its first CUDA call, no device visible)."""
    asks = []
    for name, C, mlp in (("lm_step_mlp_C5", 5, True), ("lm_step_mlp_C128", 128, True), ("lm_step_mlp_C256", 256, True),
                         ("lm_step_lambda_given", 1, False)):
        ok, rej = M.rejection_edge(name)
        asks += [(ok, C, mlp), (rej, C, mlp)]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", _PROBE, ROOT, json.dumps(asks)], env=env, capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    got = json.loads(res.stdout.strip().splitlines()[-1])
    for P, C, mlp in asks:
        rc_b, rc_f, msg = got[f"{P}:{C}:{mlp}"]
        if M.step_plan(P, C if mlp else 0) == M.REJECT:
            assert rc_b == -4 and rc_f == -4, (P, C, mlp, rc_b, rc_f, msg)
        else:
            assert rc_b == (-2 if mlp else -3) and rc_f == -3, (P, C, mlp, rc_b, rc_f, msg)


# ------------------------------------------------------------------------------------------ GPU: one step
_BUILT = {}


def built():
    """Per-pair H, g of a real FP32_SIMT build at K = 256 (4 pairs, a 96 x 128 scene, level 3, C = 16): a leading block H[:P, :P], g[:P] is
    the system of the first P - 6 basis columns."""
    if not _BUILT:
        from banet_b200 import ops, _lib
        sc = scene_case(nb=4, H=96, W=128, C=16, K=256, level_ids=(3,), seed=29, dtype=torch.float32)
        lv = sc.levels[0]
        level = ops.Level(to_cuda32(lv.conv1), to_cuda32(lv.conv2), to_cuda32(lv.intr), to_cuda32(lv.p), to_cuda32(lv.D), to_cuda32(lv.B), grid=lv.grid)
        W = to_cuda32(sc.W0) + 0.01 * torch.randn(4, 256, 1, generator=torch.Generator(device="cuda").manual_seed(3), device="cuda")
        H, g, _, _ = ops.lm_build(level, to_cuda32(sc.R0), to_cuda32(sc.T0), W, _lib.PREC_FP32_SIMT)
        torch.cuda.synchronize()
        _BUILT["v"] = (H.cpu().double(), g.cpu().double())
    return _BUILT["v"]


def graded_spd(P, kappa, seed):
    gen = torch.Generator().manual_seed(seed)
    Q, _ = torch.linalg.qr(torch.randn(P, P, generator=gen, dtype=torch.float64))
    s = kappa ** -torch.linspace(0, 1, P, dtype=torch.float64)
    H = (Q * s) @ Q.T
    return ((H + H.T) / 2).float().double()


def pair_systems(P, nb, seed):
    """Leading blocks of the real build where P <= 262, graded systems (kappa = 1e4) beyond."""
    if P <= 262:
        H, g = built()
        idx = [i % 4 for i in range(nb)]
        return H[idx, :P, :P].contiguous(), g[idx, :P].contiguous()
    H = torch.stack([graded_spd(P, 1e4, seed + i) for i in range(nb)])
    g = torch.randn(nb, P, generator=torch.Generator().manual_seed(seed + 99), dtype=torch.float64).float().double()
    return H, g


def iterate(nb, K, seed=1):
    gen = torch.Generator().manual_seed(seed)
    ang = 0.01 * torch.randn(nb, 3, 1, generator=gen, dtype=torch.float64)
    R = O.angle_axis_rotation(ang[:, 0:1], ang[:, 1:2], ang[:, 2:3]).float().double()
    T = (0.1 * torch.randn(nb, 3, 1, generator=gen, dtype=torch.float64)).float().double()
    W = (0.01 * torch.randn(nb, K, 1, generator=gen, dtype=torch.float64)).float().double()
    return R, T, W


def cu(t):
    return None if t is None else t.to(device="cuda", dtype=torch.float32).contiguous()


def damped(H, lam, ndamped, eps=EPS32):
    P = H.shape[-1]
    d = torch.diagonal(H, dim1=-2, dim2=-1)
    mask = (torch.arange(P) < ndamped).to(H.dtype)
    return H + torch.diag_embed((d + eps) * lam.reshape(-1, 1) * mask)


def step64(H, g, lam, R, T, W, undamped_last):
    """The pair step after lambda in float64: damped solve, SE(3) update, W' = W + delta_d (differentiable)."""
    P = H.shape[-1]
    delta = torch.linalg.solve(damped(H, lam, P - 1 if undamped_last else P), g.unsqueeze(-1))
    Rn, Tn = O._update(delta, R, T, O.IterOptions())
    return Rn, Tn, (None if W is None else W + delta[:, 6:])


def mlp_lambda64(rbar_sum, N, mlp, base):
    """lambda = base ||rbar||^(2 + MLP(rbar)), rbar = rbar_sum / N (bundlenet.py:243-253) with the oracle's MLP, float64."""
    avg = (rbar_sum / N).unsqueeze(1)
    return (base * torch.pow(torch.linalg.norm(avg, dim=-1, keepdim=True), 2.0 + O.lambda_mlp(avg, mlp))).reshape(-1)


def cotangents(nb, K, seed):
    g = torch.Generator().manual_seed(seed)
    cR = torch.randn(nb, 3, 3, generator=g, dtype=torch.float64).float().double()
    cT = torch.randn(nb, 3, 1, generator=g, dtype=torch.float64).float().double()
    cW = torch.randn(nb, K, 1, generator=g, dtype=torch.float64).float().double() if K else None
    return cR, cT, cW


def step_case(P, C, use_mlp, nb=2, seed=5, base=1000.0, lam_given=0.1):
    """One step forward + backward on the GPU and in float64 autograd.  -> (storage variant, kappa, {output: relative error})."""
    from banet_b200 import ops
    K = P - 6
    H, g = pair_systems(P, nb, seed)
    R, T, W = iterate(nb, K, seed)
    W = W if K else None
    N = 4096
    rb = (0.02 * (1 + torch.rand(nb, C, generator=torch.Generator().manual_seed(seed))) * N).float().double()
    mlp32 = mlp_for(C, 3, torch.float32)
    cR, cT, cW = cotangents(nb, K, seed + 1)
    if use_mlp:
        out = ops.lm_step(cu(H), cu(g), cu(rb), N, ops.pack_mlp(mlp32).cuda(), base, cu(R), cu(T), cu(W))
    else:
        lam_in = torch.full((nb,), lam_given, dtype=torch.float32)
        out = ops.lm_step(cu(H), cu(g), cu(rb), N, None, base, cu(R), cu(T), cu(W), lam=cu(lam_in))
    delta, lout, status = out[3], out[4], out[5]
    assert int(status.abs().max()) == 0
    grads = ops.lm_step_bwd(cu(H), cu(g), cu(rb), N, ops.pack_mlp(mlp32).cuda() if use_mlp else None, lout, delta, cu(R), cu(T), cu(cR), cu(cT),
                            cu(cW), base=base)
    torch.cuda.synchronize()
    dH, dg, drb, dmlp, dlam, dR, dT, dW = [None if t is None else t.double().cpu() for t in grads]
    # float64: leaves in float64, lambda at the kernel's value with the float64 MLP's derivative
    leaf = lambda t: None if t is None else t.clone().requires_grad_()
    Hl, gl, rbl, Rl, Tl, Wl = leaf(H), leaf(g), leaf(rb), leaf(R), leaf(T), leaf(W)
    mlp64 = [(w.double().clone().requires_grad_(), b.double().clone().requires_grad_()) for w, b in mlp32]
    lk = lout.double().cpu()
    if use_mlp:
        l64 = mlp_lambda64(rbl, N, mlp64, base)
        lam = l64 + (lk - l64).detach()
    else:
        lam = lk.clone().requires_grad_()
    lam.retain_grad()
    Rn, Tn, Wn = step64(Hl, gl, lam, Rl, Tl, Wl, K > 0)
    loss = (Rn * cR).sum() + (Tn * cT).sum() + ((Wn * cW).sum() if K else 0.0)
    loss.backward()
    err = {"dH": rel_fro(dH, Hl.grad), "dg": rel_fro(dg, gl.grad), "dlambda": rel_fro(dlam, lam.grad), "dR": rel_fro(dR, Rl.grad),
           "dT": rel_fro(dT, Tl.grad)}
    if K:
        err["dW"] = rel_fro(dW, Wl.grad)
    if use_mlp:
        err["drbar_sum"] = rel_fro(drb, rbl.grad)
        off = 0
        for i, (w, b) in enumerate(mlp64):
            err[f"filters{i + 1}"] = rel_fro(dmlp[off:off + w.numel()].reshape(w.shape), w.grad); off += w.numel()
            err[f"biases{i + 1}"] = rel_fro(dmlp[off:off + b.numel()], b.grad); off += b.numel()
    ndamped = P - 1 if K else P
    kap = max(float(torch.linalg.cond(damped(H[i:i + 1], lk[i:i + 1], ndamped)[0])) for i in range(nb))
    # dlambda = -sum_i u_i delta_i (H_ii + eps) cancels: its condition number sum |t_i| / |sum t_i| scales its bound
    t = -(gl.grad * torch.linalg.solve(damped(H, lk, ndamped), g.unsqueeze(-1)).squeeze(-1) * (torch.diagonal(H, dim1=-2, dim2=-1) + EPS32))[:, :ndamped]
    cond_sum = float((t.abs().sum(1) / t.sum(1).abs().clamp_min(1e-300)).max())
    return M.step_plan(P, C if use_mlp else 0), kap, cond_sum, err


def sizes_for(C):
    """6 + K for K in {0, 16, 128, 200} where accepted, and both sides of every storage switch of lm_step at this C."""
    plan = lambda P: M.step_plan(P, C)
    s = {6 + K for K in (0, 16, 128, 200)}
    for a, b, _ in M.switches(plan, 7, 400):
        s.update((a, b))
    return sorted(P for P in s if plan(P) != M.REJECT)


# Bounds, stated per output family (relative Frobenius error against float64; kappa: 2-norm condition number of the damped system):
#   * fp64 storage: the solve's outputs (dH, dg, dR, dT, dW) within a few fp32 roundings: 16 u32 (u32 = 2^-24 ~ 6e-8) -- the kernel
#     rounds the pose adjoint, the forward's delta and each output once;
#   * fp32 storage: P kappa u32 (the Cholesky solve's classical n kappa u), and at least the fp64 bound;
#   * dlambda, a sum of P products that cancel, gets its family's bound times the sum's condition number sum |t_i| / |sum t_i|;
#   * the lambda path (drbar_sum, each layer's filters and biases) is dlambda times the MLP's fp32 backward: dlambda's bound + 2e-5.
# Largest measured on an H100 80GB HBM3 over C = 5, 64, 128, 256: fp64 7.1e-8 (dH), 4.5e-8 (dg, dR, dT), 1.9e-6 (dlambda, at a sum
# condition number above 2), 6.9e-7 (drbar_sum, filters, biases); fp32 2.0e-4 (dT at P = 327, kappa = 157: 0.065 P kappa u32).
SOLVE_ROUNDINGS = 16


def _bound(variant, P, kap, cond_sum, name):
    b = SOLVE_ROUNDINGS * U32 if variant in F64 else max(P * kap * U32, SOLVE_ROUNDINGS * U32)
    if name.startswith(("dlambda", "drbar", "filters", "biases")):
        b *= max(cond_sum, 1.0)
    if name.startswith(("drbar", "filters", "biases")):
        b += 2e-5
    return b


@pytest.mark.gpu
@pytest.mark.parametrize("C", [5, 64, 128, 256])
def test_step_bwd_matches_float64(C):
    """Every output of the step backward against float64 autograd, at K = 0, 16, 128, 200 and both sides of each storage switch of lm_step at
    this C, with the lambda-MLP (base 1000) and with lambda given."""
    worst, fails = {}, []
    for P in sizes_for(C):
        for use_mlp in (True, False):
            variant, kap, cond_sum, err = step_case(P, C, use_mlp)
            for name, e in err.items():
                key = (variant, name)
                worst[key] = max(worst.get(key, 0.0), e)
                fails += [] if e <= _bound(variant, P, kap, cond_sum, name) else [(P, use_mlp, variant, name, e, kap, cond_sum)]
    print(f"C={C} largest errors:", {f"{v}:{n}": f"{e:.2e}" for (v, n), e in sorted(worst.items())})
    assert not fails, fails


@pytest.mark.gpu
@pytest.mark.parametrize("P", [22, 134, 200, 250])
def test_lambda_given_is_the_existing_solve_backward(P):
    """With lambda given, dH, dg, dlambda, dR, dT, dW equal banet_lm_solve_update_bwd's bit for bit (the same kernel), and so do the forwards."""
    from banet_b200 import ops
    nb, K = 3, P - 6
    H, g = pair_systems(P, nb, 11)
    R, T, W = iterate(nb, K, 2)
    lam = cu(torch.tensor([1e-3, 0.1, 10.0]))
    cR, cT, cW = cotangents(nb, K, 3)
    out = ops.lm_step(cu(H), cu(g), None, 1, None, 1.0, cu(R), cu(T), cu(W), lam=lam)
    a = ops.lm_step_bwd(cu(H), cu(g), None, 1, None, out[4], out[3], cu(R), cu(T), cu(cR), cu(cT), cu(cW))
    ref = ops.lm_solve_update(cu(H), cu(g), lam, cu(R), cu(T), cu(W))
    b = ops.lm_solve_update_bwd(cu(H), cu(g), lam, ref[3], cu(R), cu(T), cu(cR), cu(cT), cu(cW))
    for name, x, y in zip(("R", "T", "W", "delta", "status"), (out[0], out[1], out[2], out[3], out[5]), ref):
        assert torch.equal(x, y), (P, name)
    for name, x, y in zip(("dH", "dg", "dlambda", "dR", "dT", "dW"), (a[0], a[1], a[4], a[5], a[6], a[7]), b):
        assert torch.equal(x, y), (P, name, rel_fro(x, y))


def _skip_batch(use_mlp, C=128, K=16):
    """5 pairs: 0 and 4 ordinary, 1 not positive definite, 2 with NaN in g, 3 with a non-finite lambda (given, or from an infinite rbar_sum)."""
    P = 6 + K
    H, g = pair_systems(P, 5, 21)
    H = H.clone(); g = g.clone()
    H[1, 0, 0] = -1e6
    g[2, 3] = float("nan")
    rb = (0.02 * (1 + torch.rand(5, C, generator=torch.Generator().manual_seed(4))) * 4096).float().double()
    lam = torch.tensor([0.1, 0.1, 0.1, float("inf"), 0.1], dtype=torch.float64)
    if use_mlp:
        rb[3, 7] = float("inf")
    R, T, W = iterate(5, K, 8)
    return H, g, rb, lam, R, T, W


def _step_and_bwd(H, g, rb, lam, R, T, W, use_mlp, C, cots, workspace=None):
    from banet_b200 import ops
    mlp = ops.pack_mlp(mlp_for(C, 3, torch.float32)).cuda() if use_mlp else None
    out = ops.lm_step(cu(H), cu(g), cu(rb), 4096, mlp, 1000.0, cu(R), cu(T), cu(W), lam=None if use_mlp else cu(lam))
    grads = ops.lm_step_bwd(cu(H), cu(g), cu(rb), 4096, mlp, out[4], out[3], cu(R), cu(T), *[cu(c) for c in cots], workspace=workspace)
    return out, grads


@pytest.mark.gpu
@pytest.mark.parametrize("use_mlp", [True, False])
def test_skip_contract(use_mlp):
    """Skipped pairs (status != 0) get zero dH, dg, dlambda, drbar_sum, no share of dmlp, and pass dR', dT', dW' through; the other pairs equal
    the same pairs run alone, bit for bit, and dmlp equals that of the ordinary pairs alone."""
    C, K = 128, 16
    H, g, rb, lam, R, T, W = _skip_batch(use_mlp, C, K)
    cots = cotangents(5, K, 9)
    out, grads = _step_and_bwd(H, g, rb, lam, R, T, W, use_mlp, C, cots)
    status = out[5].cpu()
    assert status.tolist()[0] == 0 and status.tolist()[4] == 0 and all(s != 0 for s in status.tolist()[1:4]), status
    dH, dg, drb, dmlp, dlam, dR, dT, dW = grads
    for b in (1, 2, 3):
        assert not dH[b].any() and not dg[b].any() and float(dlam[b]) == 0.0
        if use_mlp:
            assert not drb[b].any()
        assert torch.equal(dR[b], cu(cots[0])[b]) and torch.equal(dT[b], cu(cots[1])[b]) and torch.equal(dW[b], cu(cots[2])[b])
    keep = [0, 4]
    sub = lambda t: None if t is None else t[keep]
    _, alone = _step_and_bwd(sub(H), sub(g), sub(rb), sub(lam), sub(R), sub(T), sub(W), use_mlp, C, [sub(c) for c in cots])
    for name, x, y in zip(("dH", "dg", "drbar_sum", "dmlp", "dlambda", "dR", "dT", "dW"), grads, alone):
        if x is None:
            continue
        assert torch.equal(x if name == "dmlp" else x[keep], y), name


@pytest.mark.gpu
def test_bitwise_reproducible_from_poisoned_workspaces():
    from banet_b200 import ops
    C, K, nb = 128, 128, 8
    P = 6 + K
    H, g = pair_systems(P, nb, 31)
    R, T, W = iterate(nb, K, 4)
    rb = (0.02 * (1 + torch.rand(nb, C, generator=torch.Generator().manual_seed(6))) * 4096).float().double()
    cots = cotangents(nb, K, 5)
    nbytes = ops.load().banet_lm_step_bwd_workspace_bytes(nb, C, K)
    runs = []
    for fill in (0x00, 0xFF):
        ws = torch.full((nbytes,), fill, dtype=torch.uint8, device="cuda")
        runs.append(_step_and_bwd(H, g, rb, None, R, T, W, True, C, cots, workspace=ws)[1])
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda").view(torch.float32).fill_(float("nan")).view(torch.uint8)
    runs.append(_step_and_bwd(H, g, rb, None, R, T, W, True, C, cots, workspace=ws)[1])
    for r in runs[1:]:
        for x, y in zip(runs[0], r):
            assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------ GPU: the whole solve
def _levels(sc, K, f2=False, bf16=False, weights=False, bf16_basis=False, grad=False, seed=3):
    """ops.Level per scene level (fp32 or bf16 features, 3C or F2 only, optional point weights) and the leaves that need gradients."""
    from banet_b200 import ops
    levels, leaves = [], []
    gen = torch.Generator().manual_seed(seed)
    for lv in sc.levels:
        C = lv.conv1.shape[2]
        fdt = torch.bfloat16 if bf16 else torch.float32
        conv2 = lv.conv2[..., :C] if f2 else lv.conv2
        t = dict(conv1=to_cuda32(lv.conv1).to(fdt), conv2=to_cuda32(conv2).to(fdt).contiguous(), D=to_cuda32(lv.D),
                 B=None if K == 0 else to_cuda32(lv.B).to(torch.bfloat16 if bf16_basis else torch.float32))
        if weights:
            t["weight"] = (0.5 + torch.rand(lv.conv1.shape[0], lv.conv1.shape[1], 1, generator=gen)).cuda()
        if grad:
            for k, v in t.items():
                if v is not None:
                    v.requires_grad_()
        leaves.append(t)
        levels.append(ops.Level(t["conv1"], t["conv2"], to_cuda32(lv.intr), to_cuda32(lv.p), t["D"], t["B"], grid=lv.grid, weight=t.get("weight")))
    return levels, leaves


RUN_VARIANTS = [(prec, bf16, f2, wt, K) for prec in ("AUTO", "FP32_SIMT") for bf16 in (False, True) for f2 in (False, True)
                for wt in (False, True) for K in (0, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("prec,bf16,f2,weights,K", RUN_VARIANTS)
def test_lm_run_forward_is_ops_lm_run(prec, bf16, f2, weights, K):
    """autograd.lm_run's forward (2 levels x 3 iterations) returns ops.lm_run's bits."""
    from banet_b200 import ops, _lib
    from banet_b200 import autograd as ag
    C = 64
    sc = scene_case(nb=2, H=48, W=64, C=C, K=K, level_ids=(2, 3), seed=41, dtype=torch.float32)
    levels, _ = _levels(sc, K, f2=f2, bf16=bf16, weights=weights)
    mlps = [[(w.cuda(), b.cuda()) for w, b in mlp_for(C, lv.level, torch.float32)] for lv in sc.levels]
    precision = _lib.PREC_AUTO if prec == "AUTO" else _lib.PREC_FP32_SIMT
    R0, T0, W0 = to_cuda32(sc.R0), to_cuda32(sc.T0), to_cuda32(sc.W0) if K else None
    a = ops.lm_run(levels, 3, R0, T0, W0, mlp_packed=[ops.pack_mlp(m) for m in mlps], precision=precision)
    with torch.no_grad():
        b = ag.lm_run(levels, 3, R0, T0, W0, mlp_params=mlps, precision=precision, return_status=True)
    for name, x, y in zip(("R", "T", "W", "status"), a, b):
        if x is None:
            assert y is None
            continue
        assert torch.equal(x, y), name


def _run_grads(route, sc, K, C, exact, cR, cT, cW, precision, f2=False):
    """Gradients of <cR, R'> + <cT, T'> + <cW, W'> after 2 levels x 2 iterations, through autograd.lm_run or an iteration_fused loop."""
    from banet_b200 import autograd as ag
    levels, leaves = _levels(sc, K, f2=f2, grad=True)
    mlps = [[(w.cuda().requires_grad_(), b.cuda().requires_grad_()) for w, b in mlp_for(C, lv.level, torch.float32)] for lv in sc.levels]
    R = to_cuda32(sc.R0).requires_grad_(); T = to_cuda32(sc.T0).requires_grad_(); W = to_cuda32(sc.W0).requires_grad_() if K else None
    if route == "lm_run":
        Rn, Tn, Wn = ag.lm_run(levels, 2, R, T, W, mlp_params=mlps, precision=precision, exact_sym=exact)
    else:
        Rn, Tn, Wn = R, T, W
        for lv, m in zip(levels, mlps):
            for _ in range(2):
                Rn, Tn, Wn = ag.iteration_fused(lv.conv1, lv.conv2, lv.intr, lv.p, lv.D, lv.B, Rn, Tn, Wn, m, 1000.0 if K else None,
                                                exact_sym=exact, precision=precision, grid=lv.grid)
    loss = (Rn * cu(cR)).sum() + (Tn * cu(cT)).sum() + ((Wn * cu(cW)).sum() if K else 0.0)
    loss.backward()
    out = {"R0": R.grad, "T0": T.grad}
    if K:
        out["W0"] = W.grad
    for i, (t, m) in enumerate(zip(leaves, mlps)):
        for k, v in t.items():
            if v is not None:
                out[f"{k}{i}"] = v.grad
        for j, (w, b) in enumerate(m):
            out[f"filters{i}_{j + 1}"] = w.grad; out[f"biases{i}_{j + 1}"] = b.grad
    return out, (Rn.detach(), Tn.detach(), None if Wn is None else Wn.detach())


# Allowance for run-to-run noise: the build backward accumulates dR, dT, dW and dconv2 with atomics, so these gradients move slightly from
# run to run.  With a depth basis both routes' errors agree to 3 digits at every leaf.  The pose-only version of this schedule is not a
# usable yardstick: after four iterations its gradients are dominated by fp32 noise (the oracle evaluated in float32 misses dT0 by 2e-2; on
# the GPU the level-1 lambda-MLP biases were 4e-3 from float64 in both routes, and each route's errors moved by up to 2.6e-4 between runs,
# so either route came out ahead).  Its step backward is held to float64 in test_step_bwd_matches_float64 (P = 6).
NOISE = 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize("K,f2", [(16, False), (16, True)])
def test_lm_run_gradients_match_float64(K, f2):
    """Gradients of every leaf after 2 levels x 2 iterations (FP32_SIMT) against float64 autograd of oracle.lm_solve on the same schedule:
    autograd.lm_run's agreement is at least as tight as the iteration_fused loop's on the same case (within 10 %; both printed, with the
    difference between the two routes)."""
    from banet_b200 import _lib
    C, exact = 8, False
    sc = scene_case(nb=2, H=48, W=64, C=C, K=K, level_ids=(2, 3), seed=61, n_points=300, dtype=torch.float32)
    cR, cT, cW = cotangents(2, K, 13)
    olevels, oleaves = [], []
    for lv in sc.levels:
        a = oracle_level_inputs(lv)
        if f2:
            a["conv2"] = a["conv2"][..., :C].contiguous()
        for k in ("conv1", "conv2", "D", "B"):
            if a[k] is not None:
                a[k] = a[k].clone().requires_grad_()
        conv2 = torch.cat([a["conv2"], O.grad_fixed(a["conv2"])], dim=-1) if f2 else a["conv2"]
        mlp = [(w.clone().requires_grad_(), b.clone().requires_grad_()) for w, b in mlp_for(C, lv.level)]
        oleaves.append((a, mlp))
        olevels.append(O.LevelInputs(a["conv1"], conv2, a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"], mlp))
    R = sc.R0.double().clone().requires_grad_(); T = sc.T0.double().clone().requires_grad_()
    W = sc.W0.double().clone().requires_grad_() if K else None
    oR, oT, oW = O.lm_solve(olevels, 2, R, T, W, O.IterOptions(l2_regularizer_base=1000.0, guard_nonfinite=True, reference_op_grad=not exact))
    loss = (oR * cR).sum() + (oT * cT).sum() + ((oW * cW).sum() if K else 0.0)
    loss.backward()
    ref = {"R0": R.grad, "T0": T.grad}
    if K:
        ref["W0"] = W.grad
    for i, (a, mlp) in enumerate(oleaves):
        for k in ("conv1", "conv2", "D", "B"):
            if a[k] is not None:
                ref[f"{k}{i}"] = a[k].grad
        for j, (w, b) in enumerate(mlp):
            ref[f"filters{i}_{j + 1}"] = w.grad; ref[f"biases{i}_{j + 1}"] = b.grad
    run, run_out = _run_grads("lm_run", sc, K, C, exact, cR, cT, cW, _lib.PREC_FP32_SIMT, f2)
    loop, _ = _run_grads("loop", sc, K, C, exact, cR, cT, cW, _lib.PREC_FP32_SIMT, f2)
    assert set(run) == set(ref) == set(loop)
    assert rel_fro(run_out[0], oR.detach()) < 1e-4 and rel_fro(run_out[1], oT.detach()) < 1e-3
    # The start pose is held as one leaf: after four LM iterations the solve has converged and |dT0| is small next to |dR0|, so T0's own
    # relative error is mostly rounding noise; R0 and T0 are printed on their own.
    pose = lambda d: torch.cat([d["R0"].reshape(-1).double().cpu(), d["T0"].reshape(-1).double().cpu()])
    for d in (ref, run, loop):
        d["pose0"] = pose(d)
    report, bad = {}, []
    for k in ref:
        e_run, e_loop = rel_fro(run[k], ref[k]), rel_fro(loop[k], ref[k])
        report[k] = (f"{e_run:.2e}", f"{e_loop:.2e}", f"{rel_fro(run[k], loop[k]):.2e}")
        if k not in ("R0", "T0") and not (e_run <= max(1.1 * e_loop, e_loop + NOISE) and e_run < 2e-2):
            bad.append((k, e_run, e_loop))
    print(f"K={K} f2={f2} relative errors against float64 (lm_run, iteration_fused loop, lm_run against the loop):", report)
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("bf16,weights", [(True, False), (False, True), (True, True)])
def test_lm_run_gradients_reach_bf16_and_weighted_leaves(bf16, weights):
    """With bfloat16 features and basis, or point weights, every leaf (the weights included) gets autograd.lm_run's gradient, and it agrees
    with the iteration_fused loop's (the same build backward; the steps differ in their factorisation and lambda-MLP arithmetic)."""
    from banet_b200 import _lib
    from banet_b200 import autograd as ag
    C, K = 16, 16
    sc = scene_case(nb=2, H=48, W=64, C=C, K=K, level_ids=(2, 3), seed=67, n_points=300, dtype=torch.float32)
    cR, cT, cW = cotangents(2, K, 17)
    grads = {}
    for route in ("lm_run", "loop"):
        levels, leaves = _levels(sc, K, bf16=bf16, bf16_basis=bf16, weights=weights, grad=True, seed=9)
        mlps = [[(w.cuda().requires_grad_(), b.cuda().requires_grad_()) for w, b in mlp_for(C, lv.level, torch.float32)] for lv in sc.levels]
        R = to_cuda32(sc.R0).requires_grad_(); T = to_cuda32(sc.T0).requires_grad_(); W = to_cuda32(sc.W0).requires_grad_()
        if route == "lm_run":
            Rn, Tn, Wn = ag.lm_run(levels, 2, R, T, W, mlp_params=mlps, precision=_lib.PREC_FP32_SIMT)
        else:
            Rn, Tn, Wn = R, T, W
            for lv, m in zip(levels, mlps):
                for _ in range(2):
                    Rn, Tn, Wn = ag.iteration_fused(lv.conv1, lv.conv2, lv.intr, lv.p, lv.D, lv.B, Rn, Tn, Wn, m, 1000.0, precision=_lib.PREC_FP32_SIMT,
                                                    weight=lv.weight)
        ((Rn * cu(cR)).sum() + (Tn * cu(cT)).sum() + (Wn * cu(cW)).sum()).backward()
        g = {"R0": R.grad, "T0": T.grad, "W0": W.grad}
        for i, (t, m) in enumerate(zip(leaves, mlps)):
            for k, v in t.items():
                g[f"{k}{i}"] = v.grad
                assert v.grad is not None and v.grad.dtype == v.dtype, (route, k, i)
            for j, (w, b) in enumerate(m):
                g[f"filters{i}_{j + 1}"] = w.grad; g[f"biases{i}_{j + 1}"] = b.grad
        grads[route] = g
    for k, v in grads["lm_run"].items():
        assert torch.isfinite(v.float()).all(), k
        assert rel_fro(v.float(), grads["loop"][k].float()) < (2e-2 if bf16 else 2e-3), (k, rel_fro(v.float(), grads["loop"][k].float()))


@pytest.mark.gpu
def test_lm_run_peak_memory_is_no_larger_than_the_loop():
    """Peak device memory of a differentiable 2-level x 3-iteration solve with its backward: autograd.lm_run against the iteration_fused
    loop (both printed)."""
    from banet_b200 import _lib
    C, K = 64, 128
    sc = scene_case(nb=4, H=96, W=128, C=C, K=K, level_ids=(2, 3), seed=71, dtype=torch.float32)
    cR, cT, cW = cotangents(4, K, 19)
    peak = {}
    for route in ("loop", "lm_run", "loop", "lm_run"):
        torch.cuda.synchronize(); torch.cuda.empty_cache(); torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        _run_grads(route, sc, K, C, False, cR, cT, cW, _lib.PREC_FP32_SIMT)
        torch.cuda.synchronize()
        peak[route] = torch.cuda.max_memory_allocated() - base
    print("peak bytes above the start:", peak)
    assert peak["lm_run"] <= peak["loop"], peak


@pytest.mark.gpu
def test_lm_run_raises_where_the_fused_step_does_not_fit():
    from banet_b200 import _lib
    from banet_b200 import autograd as ag
    C, K = 8, 400
    sc = scene_case(nb=1, H=48, W=64, C=C, K=4, level_ids=(3,), seed=5, n_points=64, dtype=torch.float32)
    lv = sc.levels[0]
    from banet_b200 import ops
    B = torch.zeros(1, lv.conv1.shape[1], K, device="cuda")
    level = ops.Level(to_cuda32(lv.conv1), to_cuda32(lv.conv2), to_cuda32(lv.intr), to_cuda32(lv.p), to_cuda32(lv.D), B)
    with pytest.raises(_lib.BanetError, match="fused step"):
        ag.lm_run([level], 1, to_cuda32(sc.R0), to_cuda32(sc.T0), torch.zeros(1, K, 1, device="cuda"),
                  mlp_params=[[(w.cuda(), b.cuda()) for w, b in mlp_for(C, 3, torch.float32)]])
