"""The damped solve of an LM iteration at the storage switches of its kernels, against float64.

Both solvers (lm_step_kernel, which is also the pair solve with lambda given and the dense window, and the arrow) pick their shared-memory
storage by size (tests/solve_plan_model.py): square fp64, packed fp64 or packed fp32, or reject the size.  These tests run every kernel
instantiation on both sides of every switch:
  * CPU: the plan model, the rejection edges of the built library (asked through the C-ABI with no device visible, so that a size the
    library accepts fails only at its first CUDA call), and the float64 references the GPU tests use;
  * GPU: forwards against a float64 solve of the same fp32 inputs on systems from a real build, with bounds c * kappa * u; each switch
    crossed by padding a system with decoupled unknowns; backwards against float64 autograd; the skip contract (status bits, zero step,
    unchanged iterate, zero gradients) for every skip cause; the backward's skip equal to the forward's status on systems whose
    definiteness depends on the precision or on the order of the factorisation; the entries that share lm_step's code bitwise equal to it;
    the arrow's thread- and warp-per-frame loops past their wraps; and a profiler pass that lists every instantiation.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import ROOT, scene_case, mlp_for, to_cuda32
from oracle import ba_oracle as O
import solve_plan_model as M
from window_arrow_oracle import window_arrow_solve

U64, U32 = 2.0 ** -53, 2.0 ** -24
EPS32 = float(np.float32(1e-5))
F64 = (M.SQUARE64, M.PACKED64)
LAMS = (1e-3, 0.1, 10.0)

# c of the forward bounds err <= c kappa u (+ 2^-23 for the fp64 variants, whose step is stored in fp32); kappa = 2-norm condition number
# of the damped system.  Largest measured (err - 2^-23) / (kappa u) on an H100 80GB HBM3 over the realistic and graded systems of
# test_forward_matches_float64: 0 for every fp64 variant (errors <= 2.9e-8: the final rounding alone), 0.39 for the fp32 ones;
# DESIGN.md section 4 has each variant.
C_FWD = {"fp64": 4.0, "fp32": 1.0}


# ------------------------------------------------------------------------------------------ float64 references
def damped(H, lam, ndamped, eps=EPS32):
    """H [...,P,P] -> H + lam diag(diag H + eps) on the first ndamped diagonal entries (bundlenet.py:264-266)."""
    P = H.shape[-1]
    d = torch.diagonal(H, dim1=-2, dim2=-1)
    mask = (torch.arange(P) < ndamped).to(H.dtype)
    return H + torch.diag_embed((d + eps) * lam * mask)


def pair_step64(H, g, lam, R, T, W, undamped_last=True):
    """The pair iteration after the build in float64: damped solve, SE(3) update (O._update), W' = W + delta_d.  Differentiable."""
    P = H.shape[-1]
    delta = torch.linalg.solve(damped(H, lam.reshape(-1, 1), P - 1 if undamped_last else P), g.unsqueeze(-1))
    Rn, Tn = O._update(delta, R, T, O.IterOptions())
    return Rn, Tn, W + delta[:, 6:], delta.squeeze(-1)


def dense_window_step64(H, g, lam, R, T, W, undamped_last=True, fp32_assembly=False):
    """The joint keyframe window (one W for nf frames) in float64 on the assembled system: H [nf,P,P], g [nf,P], W [K,1]."""
    nf = H.shape[0]
    Hj, gj = O.window_assemble(H, g.unsqueeze(-1))
    if fp32_assembly:                                               # the kernel assembles the frame-summed blocks in float
        Hj = Hj + (Hj.detach().float().double() - Hj.detach()); gj = gj + (gj.detach().float().double() - gj.detach())
    Pj = Hj.shape[0]
    delta = torch.linalg.solve(damped(Hj, lam.reshape(()), Pj - 1 if undamped_last else Pj), gj)
    Rn, Tn = O._update(delta[:6 * nf].reshape(nf, 6, 1), R, T, O.IterOptions())
    return Rn, Tn, W + delta[6 * nf:], delta.squeeze(-1)


def arrow_step64(H, g, lam, R, T, W, nw, undamped_last=True, fp32_damping_diag=True):
    """nw block-arrow windows in float64 (tests/window_arrow_oracle.py): H [nw nf,P,P], g [nw nf,P], lam [nw], W [nw,K,1]."""
    nb, P, _ = H.shape
    nf = nb // nw
    outs = [window_arrow_solve(H[w * nf:(w + 1) * nf], g[w * nf:(w + 1) * nf].unsqueeze(-1), lam[w], EPS32, undamped_last, fp32_damping_diag)
            for w in range(nw)]
    delta = torch.stack([o.squeeze(-1) for o in outs])             # [nw, 6 nf + K]
    Rn, Tn = O._update(delta[:, :6 * nf].reshape(nb, 6, 1), R, T, O.IterOptions())
    return Rn, Tn, W + delta[:, 6 * nf:].unsqueeze(-1), delta


def graded_spd(P, kappa, seed, dtype=torch.float64):
    """Q diag(kappa^-t) Q^T, t uniform in [0, 1]: a symmetric positive definite system of known condition number, rounded to fp32."""
    gen = torch.Generator().manual_seed(seed)
    Q, _ = torch.linalg.qr(torch.randn(P, P, generator=gen, dtype=torch.float64))
    s = kappa ** -torch.linspace(0, 1, P, dtype=torch.float64)
    H = (Q * s) @ Q.T
    return ((H + H.T) / 2).float().to(dtype)


def rand_g(P, seed, n=1):
    return torch.randn(n, P, generator=torch.Generator().manual_seed(seed), dtype=torch.float64).float().double()


def kappa(A):
    return float(torch.linalg.cond(A))


# ------------------------------------------------------------------------------------------ CPU: the model and the library
# (last fp64 size, first rejected size) of every entry before its MLP buffers shared the matrix's storage and every pair and dense-window
# solve ran on lm_step_kernel's code: the sizes each entry accepted and the fp64 range it had, which the one plan must keep (but where stated)
PREVIOUS = {"lm_step_lambda_given": (220, 330), "lm_step_mlp_C5": (220, 329), "lm_step_mlp_C128": (218, 326), "lm_step_mlp_C256": (215, 323),
            "lm_solve": (223, 334), "lm_solve_bwd_pairs": (223, 333), "dense_window": (220, 330), "lm_solve_bwd_dense_window": (220, 330),
            "arrow_lambda_given": (215, 257), "arrow_bwd": (215, 257), "arrow_mlp_C5": (213, 257), "arrow_mlp_C128": (211, 257),
            "arrow_mlp_C256": (209, 257)}


def test_plan_model_switch_table():
    step = [(157, 158), (222, 223), (332, 333)]
    arrow = [(154, 155), (215, 216), (256, 257)]
    for name, (plan, (lo, hi)) in M.PLANS.items():
        edges = [(a, b) for a, b, _ in M.switches(plan, lo, hi)]
        if name.startswith(("lm_step_width", "lm_lambda_width")):
            assert edges == {"lm_step_width_P7": [(4690, 4691)], "lm_step_width_P262": [(4649, 4650)], "lm_lambda_width": [(4693, 4694)]}[name]
        else:
            assert edges == (arrow if name.startswith("arrow") else step), name
    for name in M.PLANS:
        sizes = [s for s in M.edge_sizes(name) if M.PLANS[name][0](s) != M.REJECT]
        assert {s % 4 for s in sizes} == {0, 1, 2, 3}, name
    # inference and training factor alike: the step with the MLP at any width and with lambda given, forward and backward, one plan
    for P in range(7, 400):
        assert len({M.PLANS[n][0](P) for n in M.PLANS if n.startswith(("lm_step_mlp", "lm_step_lambda", "lm_solve", "dense_window"))}) == 1, P
    # every entry keeps every size it accepted and its fp64 range, but for the pair solve and its backward at P = 223 (now fp32) and
    # banet_lm_solve_update at P = 333 (now rejected, as its backward was)
    moved = {"lm_solve": [(223, "fp32"), (333, "rejected")], "lm_solve_bwd_pairs": [(223, "fp32")]}
    for name, (last64, rej) in PREVIOUS.items():
        plan, (lo, hi) = M.PLANS[name]
        got = []
        for n in range(lo, rej):
            v = plan(n)
            if v == M.REJECT:
                got.append((n, "rejected"))
            elif n <= last64 and v not in F64:
                got.append((n, "fp32"))
        assert got == moved.get(name, []), (name, got)
    # banet_lm_lambda now rejects C >= 4694 (before: C > 5120); lm_run with the MLP from C = 4650 (P = 262) to 4691 (P = 7)
    assert M.rejection_edge("lm_lambda_width") == (4693, 4694)


_PROBE = r"""
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from banet_b200 import _lib
lib = _lib.load()
o = _lib.BanetSolveOpts(1e-5, 1, 0)
p = 1                                        # non-null dummy pointers: nothing below may reach a kernel, and no device is visible
out = {}
def step(P, C, mlp):
    return lib.banet_lm_step(p, p, p if mlp else None, 1, 100, C, P - 6, p if mlp else None, 1.0, None if mlp else p, ctypes.byref(o),
                             p, p, p, p, p, p, p, p, p, None)
def lam(C): return lib.banet_lm_lambda(p, 1, 100, C, p, 1.0, p, None)
def solve(P): return lib.banet_lm_solve_update(p, p, p, 1, P - 6, ctypes.byref(o), p, p, p, p, p, p, p, p, None, 0, None)
def solve_bwd(P): return lib.banet_lm_solve_update_bwd(p, p, p, p, 1, P - 6, ctypes.byref(o), p, p, p, p, p, p, p, p, p, p, p, None)
def win(Pj): return lib.banet_lm_window_solve_update(p, p, p, 1, Pj - 6, ctypes.byref(o), p, p, p, p, p, p, p, p, None, 0, None)
def win_bwd(Pj): return lib.banet_lm_window_solve_update_bwd(p, p, p, p, 1, Pj - 6, ctypes.byref(o), p, p, p, p, p, p, p, p, p, p, p, None, 0, None)
def arrow(K): return lib.banet_lm_window_batch_solve_update(p, p, p, 2, 3, K, ctypes.byref(o), p, p, p, p, p, p, p, p, None, 0, None)
def arrow_bwd(K): return lib.banet_lm_window_batch_solve_update_bwd(p, p, p, p, 2, 3, K, ctypes.byref(o), p, p, p, p, p, p, p, p, p, p, p, None, 0, None)
def arrow_run(K, C):
    lv = (_lib.BanetLevel * 1)(_lib.BanetLevel(6, 4096, C, K, 120, 160, 3 * C, 1, 1, 1, 1, 1, 1, 0, 0))
    mlp = (ctypes.c_void_p * 1)(p)
    return lib.banet_lm_window_batch_run(lv, 1, 2, 1, mlp, 1000.0, -1.0, ctypes.byref(o), 0, p, p, p, p, None, 0, None)
calls = {"lm_step_lambda_given": lambda n: step(n, 1, False), "lm_step_mlp_C5": lambda n: step(n, 5, True),
         "lm_step_mlp_C128": lambda n: step(n, 128, True), "lm_step_mlp_C256": lambda n: step(n, 256, True),
         "lm_step_width_P7": lambda n: step(7, n, True), "lm_step_width_P262": lambda n: step(262, n, True), "lm_lambda_width": lam,
         "lm_solve": solve, "lm_solve_bwd_pairs": solve_bwd, "lm_solve_bwd_dense_window": win_bwd, "dense_window": win,
         "arrow_lambda_given": arrow, "arrow_bwd": arrow_bwd, "arrow_mlp_C5": lambda n: arrow_run(n, 5),
         "arrow_mlp_C128": lambda n: arrow_run(n, 128), "arrow_mlp_C256": lambda n: arrow_run(n, 256)}
for name, n in json.loads(sys.argv[2]):
    out[f"{name}:{n}"] = [calls[name](n), lib.banet_last_error().decode()]
print(json.dumps(out))
"""


def test_rejection_edges_come_from_the_library():
    """-4 exactly where the model rejects; one size below, the call gets past every size check: it fails at its first CUDA call (-3,
    no device is visible to the probe) or at the workspace check that follows (-2, no workspace given).  A rejection that came after a
    CUDA call would show as -3 as well, so -4 also proves the check runs before any CUDA call."""
    asks = []
    for name in M.PLANS:
        ok, rej = M.rejection_edge(name)
        asks += [(name, ok), (name, rej)]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", _PROBE, ROOT, json.dumps(asks)], env=env, capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    got = json.loads(res.stdout.strip().splitlines()[-1])
    for name, n in asks:
        rc, msg = got[f"{name}:{n}"]
        ok, rej = M.rejection_edge(name)
        if n == rej:
            assert rc == -4, (name, n, rc, msg)
        else:
            assert rc in (-2, -3), (name, n, rc, msg)


def test_float64_references_agree():
    """The three float64 statements the GPU tests use agree with each other: one frame of the arrow is the pair solve, and the arrow equals
    the dense solve of the assembled window (with the same fp32 rounding of the summed depth diagonal)."""
    nf, K = 3, 9
    P = 6 + K
    H = torch.stack([graded_spd(P, 1e3, s) for s in range(nf)]).double()
    g = rand_g(P, 5, nf)
    lam = torch.tensor([0.3], dtype=torch.float64)
    R = torch.eye(3, dtype=torch.float64).repeat(nf, 1, 1); T = torch.zeros(nf, 3, 1, dtype=torch.float64)
    W = torch.zeros(1, K, 1, dtype=torch.float64)
    a = arrow_step64(H, g, lam, R, T, W, 1, fp32_damping_diag=False)
    d = dense_window_step64(H, g, lam, R, T, W[0])
    assert torch.allclose(a[3][0], d[3], rtol=1e-10, atol=1e-12)
    one = arrow_step64(H[:1], g[:1], lam, R[:1], T[:1], W, 1)
    pr = pair_step64(H[:1], g[:1], lam, R[:1], T[:1], W)
    assert torch.allclose(one[3][0], pr[3][0], rtol=1e-10, atol=1e-12)


# ------------------------------------------------------------------------------------------ GPU
def _built_systems():
    """Per-pair H, g of a real build (FP32_SIMT, K = 256, a 96 x 128 scene at level 3, C = 16): 4 pairs, two windows of two frames.
    A leading block H[:6+K, :6+K], g[:6+K] is exactly the system of the first K basis columns."""
    from banet_b200 import ops, _lib
    sc = scene_case(nb=4, H=96, W=128, C=16, K=256, level_ids=(3,), seed=29, shared_depth=True, window_frames=2, dtype=torch.float32)
    lv = sc.levels[0]
    level = ops.Level(to_cuda32(lv.conv1), to_cuda32(lv.conv2), to_cuda32(lv.intr), to_cuda32(lv.p), to_cuda32(lv.D), to_cuda32(lv.B), grid=lv.grid)
    W = to_cuda32(sc.W0) + 0.01 * torch.randn(4, 256, 1, generator=torch.Generator(device="cuda").manual_seed(3), device="cuda")
    H, g, _, _ = ops.lm_build(level, to_cuda32(sc.R0), to_cuda32(sc.T0), W, _lib.PREC_FP32_SIMT)
    torch.cuda.synchronize()
    return H.cpu().double(), g.cpu().double(), sc.R0.double(), sc.T0.double()


_BUILT = {}


def built():
    if not _BUILT:
        _BUILT["v"] = _built_systems()
    return _BUILT["v"]


def pair_systems(P, nb, seed):
    """nb pair systems of size P: leading blocks of the real build where P <= 262, graded (kappa = 1e4) beyond."""
    if P <= 262:
        H, g, _, _ = built()
        idx = [i % 4 for i in range(nb)]
        return H[idx, :P, :P].contiguous(), g[idx, :P].contiguous(), "build"
    return torch.stack([graded_spd(P, 1e4, seed + i) for i in range(nb)]).double(), rand_g(P, seed + 99, nb), "graded"


def _iterate(nb, K, seed=1):
    gen = torch.Generator().manual_seed(seed)
    ang = 0.01 * torch.randn(nb, 3, 1, generator=gen, dtype=torch.float64)
    R = O.angle_axis_rotation(ang[:, 0:1], ang[:, 1:2], ang[:, 2:3]).float().double()
    T = (0.1 * torch.randn(nb, 3, 1, generator=gen, dtype=torch.float64)).float().double()
    W = (0.01 * torch.randn(nb, K, 1, generator=gen, dtype=torch.float64)).float().double()
    return R, T, W


def cu(t):
    return t.to(device="cuda", dtype=torch.float32).contiguous()


def _rel(a, b):
    a = torch.as_tensor(a).double().cpu(); b = torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _bound(variant, kap, lam=None):
    c = C_FWD["fp64" if variant in F64 else "fp32"]
    if variant in F64:
        return c * kap * U64 + 2 * U32
    return min(c * kap * U32, ERR_CAP_FP32[lam])


# c kappa u32 exceeds 1 on the realistic systems at lambda = 1e-3 (kappa ~1e8), so the fp32 variants are also held to an absolute cap per
# lambda (None: the lambda-MLP).  Largest errors measured on an H100 80GB HBM3, realistic and graded systems together: 2.0e-4 at
# lambda = 1e-3, 6.1e-6 at 0.1, 1.5e-6 at 10, 7.1e-7 with the MLP.
ERR_CAP_FP32 = {1e-3: 1e-3, 0.1: 3e-5, 10.0: 1e-5, None: 1e-4}


def _fwd_case(entry, n, lam, seed):
    """Run one forward on the GPU and its float64 reference.  -> (variant, kappa, error of the step, source of the system)."""
    from banet_b200 import ops
    if entry in ("lm_step_lambda_given", "lm_step_mlp_C5", "lm_step_mlp_C128", "lm_step_mlp_C256", "lm_solve"):
        H, g, src = pair_systems(n, 2, seed)
        R, T, W = _iterate(2, n - 6)
        if entry.startswith("lm_step_mlp_C"):
            Cm = int(entry[len("lm_step_mlp_C"):])
            rb = 0.02 * (1 + torch.rand(2, Cm, generator=torch.Generator().manual_seed(seed))) * 4096
            mlp = ops.pack_mlp(mlp_for(Cm, 3, torch.float32)).cuda()
            out = ops.lm_step(cu(H), cu(g), cu(rb), 4096, mlp, 1000.0, cu(R), cu(T), cu(W))
            lamv = out[4].double().cpu()                             # the reference solves at the lambda the kernel reports
            variant = M.step_plan(n, Cm)
        elif entry == "lm_step_lambda_given":
            lamv = torch.full((2,), lam, dtype=torch.float32).double()
            out = ops.lm_step(cu(H), cu(g), None, 1, None, 1.0, cu(R), cu(T), cu(W), lam=cu(lamv))
            variant = M.step_plan(n)
        else:
            lamv = torch.full((2,), lam, dtype=torch.float32).double()
            out = ops.lm_solve_update(cu(H), cu(g), cu(lamv), cu(R), cu(T), cu(W))
            variant = M.step_plan(n)
        delta, status = out[3].cpu().double(), out[-1].cpu()
        ref = pair_step64(H, g, lamv, R, T, W)[3]
        kap = max(kappa(damped(H[i], lamv[i], n - 1)) for i in range(2))
        err = max(_rel(delta[i], ref[i]) for i in range(2))
    elif entry == "dense_window":
        nf = 2
        K = n - 6 * nf
        H, g, src = pair_systems(6 + K, nf, seed)
        R, T, W = _iterate(nf, K)
        lamv = torch.tensor([lam], dtype=torch.float32).double()
        out = ops.lm_window_solve_update(cu(H), cu(g), cu(lamv), cu(R), cu(T), cu(W[0]))
        delta, status = out[3].cpu().double(), out[4].cpu()
        ref = dense_window_step64(H, g, lamv, R, T, W[0], fp32_assembly=True)[3]
        Hj, _ = O.window_assemble(H, g.unsqueeze(-1))
        kap = kappa(damped(Hj.float().double(), lamv, n - 1))
        err = _rel(delta, ref)
        variant = M.step_plan(n)
    else:                                                            # arrow: two windows of two frames
        nw, nf, K = 2, 2, n
        H, g, src = pair_systems(6 + K, nw * nf, seed)
        R, T, W = _iterate(nw * nf, K)
        W = W[:nw]
        lamv = torch.full((nw,), lam, dtype=torch.float32).double()
        out = ops.lm_window_batch_solve_update(cu(H), cu(g), cu(lamv), cu(R), cu(T), cu(W))
        delta, status = out[3].cpu().double(), out[4].cpu()
        ref = arrow_step64(H, g, lamv, R, T, W, nw)[3]
        kap = 0.0
        for w in range(nw):
            Hj, _ = O.window_assemble(H[w * nf:(w + 1) * nf], g[w * nf:(w + 1) * nf].unsqueeze(-1))
            kap = max(kap, kappa(damped(Hj, lamv[w], 6 * nf + K - 1)))
        err = max(_rel(delta[w], ref[w]) for w in range(nw))
        variant = M.arrow_plan(K, 0)
    return variant, kap, err, src, status


def accepted_edges(name):
    return [s for s in M.edge_sizes(name) if M.PLANS[name][0](s) != M.REJECT]


FWD_SIZES = {
    "lm_step_lambda_given": accepted_edges("lm_step_lambda_given"),
    "lm_step_mlp_C5": accepted_edges("lm_step_mlp_C5"),
    "lm_step_mlp_C128": accepted_edges("lm_step_mlp_C128"),
    "lm_step_mlp_C256": accepted_edges("lm_step_mlp_C256"),
    "lm_solve": accepted_edges("lm_solve") + [225],
    "dense_window": accepted_edges("dense_window"),
    "arrow": accepted_edges("arrow_lambda_given") + [153],
}


@pytest.mark.gpu
@pytest.mark.parametrize("entry", list(FWD_SIZES))
def test_forward_matches_float64(entry):
    """Step of every variant against the float64 solve of the same fp32 inputs, on realistic systems (leading blocks of one real build, at
    three lambdas) and on graded ones of known condition: err <= c kappa u (+ 2^-23 for the fp64 variants, whose step is stored in fp32).
    c = C_FWD is small enough that one fp32 intermediate in an fp64 variant would fail."""
    from banet_b200 import _lib
    _lib.require_device()
    rows, worst = [], {"fp64": 0.0, "fp32": 0.0}
    lams = (None,) if entry.startswith("lm_step_mlp_C") else LAMS
    for n in FWD_SIZES[entry]:
        for lam in lams:
            variant, kap, err, src, status = _fwd_case(entry, n, lam, seed=n)
            prec = "fp64" if variant in F64 else "fp32"
            u = U64 if prec == "fp64" else U32
            c = max(err - (2 * U32 if prec == "fp64" else 0.0), 0.0) / (kap * u)
            rows.append((n, lam, variant, src, f"{kap:.1e}", f"{err:.1e}", f"{c:.2g}", status.tolist()))
            worst[prec] = max(worst[prec], c)
            assert int(status.abs().max()) == 0, rows[-1]                # every one of these systems is solved, fp32 variants included
            assert err <= _bound(variant, kap, lam), rows[-1]
    for r in rows:
        print(entry, *r)
    print(f"{entry}: measured c = {worst}")


# ---- the step inside the window runs, with the lambda-MLP at C = 128 (at the arrow's switches, K = 154/155 and 215/216)
RUN_K = [s for s in M.edge_sizes("arrow_mlp_C128") if 140 < s < 240]
_RUN_SCENE = {}


def _run_scene():
    """Two windows of two frames, C = 128, 4096 keyframe points on the 120 x 160 map of level 3, K = 216 (smaller K: the leading basis
    columns)."""
    if not _RUN_SCENE:
        _RUN_SCENE["v"] = scene_case(nb=4, H=120, W=160, C=128, K=max(RUN_K), level_ids=(3,), seed=47, n_points=4096, shared_depth=True,
                                     window_frames=2, dtype=torch.float32)
    return _RUN_SCENE["v"]


def _mlp_lambda64(rbar_sum, N, nf, mlp32, base=1000.0):
    """The window's lambda in float64 from the run's own per-pair residual sums: rbar = (sum over the frames, rounded to float) / (nf N),
    lambda = base ||rbar||^(2 + MLP(rbar)) (bundlenet.py:241-253)."""
    nw = rbar_sum.shape[0] // nf
    acc = rbar_sum.double().reshape(nw, nf, -1).sum(1).float()
    r = (acc * np.float32(1.0 / (N * nf))).double()
    h = O.lambda_mlp(r.unsqueeze(1), [(w.double(), b.double()) for w, b in mlp32]).reshape(nw)
    return base * torch.linalg.norm(r, dim=-1) ** (2.0 + h)


@pytest.mark.gpu
@pytest.mark.parametrize("run", ["window_batch_run", "keyframe_run"])
def test_window_runs_with_the_mlp_match_float64(run):
    """One iteration of lm_window_batch_run / lm_keyframe_run with the lambda-MLP at C = 128, at the arrow's switch sizes for that C,
    against the float64 block-arrow step (tests/window_arrow_oracle.py) of the same build (the run's build is bitwise ops.lm_build at
    FP32_SIMT / ops.lm_keyframe_build).  The run does not report its lambda, so the reference takes lambda in float64 from the same
    residual sums; the bound adds the step's change under a 1e-5 relative change of lambda, which covers the fp32 MLP's rounding, and the
    fp32 rounding of W' = W + delta_d."""
    from banet_b200 import ops, _lib
    _lib.require_device()
    sc = _run_scene()
    l = sc.levels[0]
    nw, nf = 2, 2
    mlp32 = mlp_for(128, 3, torch.float32)
    packed = ops.pack_mlp(mlp32).cuda()
    N = l.conv1.shape[1]
    for K in RUN_K:
        variant = M.arrow_plan(K, 128)
        R, T = cu(sc.R0), cu(sc.T0)
        W = (cu(sc.W0.reshape(nw, nf, -1, 1)[:, 0, :K]) + 0.01 * torch.arange(1, nw + 1, device="cuda").reshape(nw, 1, 1)).contiguous()
        B = l.B[..., :K].contiguous()
        if run == "window_batch_run":
            lv = ops.Level(cu(l.conv1), cu(l.conv2), cu(l.intr), cu(l.p), cu(l.D), cu(B), grid=l.grid)
            Rn, Tn, Wn, st = ops.lm_window_batch_run([lv], nw, 1, R, T, W, mlp_packed=[packed], l2_regularizer_base=1000.0,
                                                     precision=_lib.PREC_FP32_SIMT)
            H, g, rb, _ = ops.lm_build(lv, R, T, W.repeat_interleave(nf, 0).contiguous(), _lib.PREC_FP32_SIMT)
        else:
            k = lambda t: cu(t.reshape(nw, nf, *t.shape[1:])[:, 0])
            kl = ops.KeyframeLevel(k(l.conv1), cu(l.conv2), cu(l.intr), k(l.p), k(l.D), k(B))
            Rn, Tn, Wn, st = ops.lm_keyframe_run([kl], 1, R, T, W, mlp_packed=[packed], l2_regularizer_base=1000.0,
                                                 precision=_lib.PREC_FP32_SIMT)
            H, g, rb, _ = ops.lm_keyframe_build(kl, R, T, W)
        assert int(st.abs().max()) == 0, (run, K)
        H64, g64 = H.cpu().double(), g.cpu().double()
        R64, T64, W64 = R.cpu().double(), T.cpu().double(), W.cpu().double()
        lam = _mlp_lambda64(rb.cpu(), N, nf, mlp32)
        ref = arrow_step64(H64, g64, lam, R64, T64, W64, nw)
        ref2 = arrow_step64(H64, g64, lam * (1 + 1e-5), R64, T64, W64, nw)
        kap = 0.0
        for w in range(nw):
            Hj, _ = O.window_assemble(H64[w * nf:(w + 1) * nf], g64[w * nf:(w + 1) * nf].unsqueeze(-1))
            kap = max(kap, kappa(damped(Hj, lam[w], 6 * nf + K - 1)))
        for w in range(nw):
            dd = (ref[2][w] - W64[w]).norm()
            err = float((Wn[w].cpu().double() - ref[2][w]).norm() / dd)
            sens = float((ref2[2][w] - ref[2][w]).norm() / dd)
            bound = _bound(variant, kap, None) + sens + 2 * U32 * float(W64[w].norm() / dd)
            print(run, K, variant, f"lambda {float(lam[w]):.3g} kappa {kap:.1e} err {err:.1e} bound {bound:.1e} (lambda sensitivity {sens:.1e})")
            assert err <= bound, (run, K, w, variant, err, bound)
            assert _rel(Tn[w * nf:(w + 1) * nf], ref[1][w * nf:(w + 1) * nf]) <= 1e-5, (run, K, w)


def _pad(H, g, extra):
    """[n,P,P], [n,P] -> the same systems with `extra` decoupled identity unknowns appended (zero right-hand side, so zero steps)."""
    n, P, _ = H.shape
    Hp = torch.zeros(n, P + extra, P + extra, dtype=H.dtype)
    Hp[:, :P, :P] = H
    Hp[:, P:, P:] = torch.eye(extra, dtype=H.dtype)
    return Hp, torch.cat([g, torch.zeros(n, extra, dtype=g.dtype)], 1)


SWITCHES = {
    "lm_step_lambda_given": [(a, b) for a, b, _ in M.switches(M.PLANS["lm_step_lambda_given"][0], 7, 400)][:2],
    "lm_step_mlp_C128": [(a, b) for a, b, _ in M.switches(M.PLANS["lm_step_mlp_C128"][0], 7, 400)][:2],
    "lm_solve": [(a, b) for a, b, _ in M.switches(M.PLANS["lm_solve"][0], 7, 400)][:2],
    "dense_window": [(a, b) for a, b, _ in M.switches(M.PLANS["dense_window"][0], 7, 400)][:2],
    "arrow": [(a, b) for a, b, _ in M.switches(M.PLANS["arrow_lambda_given"][0], 1, 300)][:2],
}


@pytest.mark.gpu
@pytest.mark.parametrize("entry", list(SWITCHES))
def test_each_switch_is_crossed_by_padding(entry):
    """The same system solved by the variant below a switch and, padded with decoupled identity unknowns, by the variant above it.  Two
    fp64 variants agree to within one fp32 rounding of the stored step; with an fp32 side, to the fp32 bound.  A wrong packed index
    shows here at any tolerance."""
    from banet_b200 import ops, _lib
    _lib.require_device()
    for a, b in SWITCHES[entry]:
        lam = torch.tensor([0.1], dtype=torch.float32).double()
        if entry in ("lm_step_lambda_given", "lm_step_mlp_C128", "lm_solve"):
            H = torch.stack([graded_spd(a, 1e3, a)]).double(); g = rand_g(a, a)
            R, T, W = _iterate(1, b - 6)
            Hp, gp = _pad(H, g, b - a)
            if entry == "lm_step_lambda_given":
                run = lambda H_, g_, W_: ops.lm_step(cu(H_), cu(g_), None, 1, None, 1.0, cu(R), cu(T), cu(W_), lam=cu(lam), undamped_last=False)[3]
                plan = M.step_plan
            elif entry == "lm_step_mlp_C128":                        # lambda depends on the residual sums only: the same on both sides
                rb = 0.02 * (1 + torch.rand(1, 128, generator=torch.Generator().manual_seed(a))) * 4096
                mlp = ops.pack_mlp(mlp_for(128, 3, torch.float32)).cuda()
                run = lambda H_, g_, W_: ops.lm_step(cu(H_), cu(g_), cu(rb), 4096, mlp, 1000.0, cu(R), cu(T), cu(W_), undamped_last=False)[3]
                plan = lambda s: M.step_plan(s, 128)
            else:
                run = lambda H_, g_, W_: ops.lm_solve_update(cu(H_), cu(g_), cu(lam), cu(R), cu(T), cu(W_), undamped_last=False)[3]
                plan = M.step_plan
            da = run(H, g, W[:, :a - 6]).cpu().double()[0]
            db = run(Hp, gp, W).cpu().double()[0][:a]
        elif entry == "dense_window":
            nf = 2
            Hs = torch.stack([graded_spd(a - 6, 1e3, a + f) for f in range(nf)]).double(); g = rand_g(a - 6, a, nf)
            Hs[:, :6, 6:] *= 0.3; Hs[:, 6:, :6] *= 0.3
            Hs = Hs.float().double()
            Hs = torch.stack([h + 2 * torch.eye(a - 6, dtype=torch.float64) for h in Hs]).float().double()
            R, T, W = _iterate(nf, b - 12)
            # pad the depth block of frame 0 only: the frame-summed depth block gets the identity once
            Hp, gp = _pad(Hs, g, b - a); Hp[1, a - 6:, a - 6:] = 0
            run = lambda H_, g_, W_: ops.lm_window_solve_update(cu(H_), cu(g_), cu(lam), cu(R), cu(T), cu(W_), undamped_last=False)[3]
            da = run(Hs, g, W[0, :a - 12]).cpu().double()
            db = run(Hp, gp, W[0]).cpu().double()[:a]
            plan = M.step_plan
        else:
            nf = 2
            Hs = torch.stack([graded_spd(6 + a, 1e3, a + f) for f in range(nf)]).double()
            Hs = torch.stack([h + 2 * torch.eye(6 + a, dtype=torch.float64) for h in Hs]).float().double()
            g = rand_g(6 + a, a, nf)
            R, T, W = _iterate(nf, b)
            Hp, gp = _pad(Hs, g, b - a); Hp[1, 6 + a:, 6 + a:] = 0
            run = lambda H_, g_, W_: ops.lm_window_batch_solve_update(cu(H_), cu(g_), cu(lam), cu(R), cu(T), cu(W_), undamped_last=False)[3]
            da = run(Hs, g, W[:1, :a]).cpu().double()[0]
            db = run(Hp, gp, W[:1]).cpu().double()[0][:6 * nf + a]
            plan = lambda s: M.arrow_plan(s, 0)
        va, vb = plan(a), plan(b)
        assert va != vb
        if va in F64 and vb in F64:
            ulp = torch.from_numpy(np.spacing(da.abs().float().numpy())).double()
            assert bool(((da - db).abs() <= 1e-12 * da.abs().max() + ulp).all()), (entry, a, b, float((da - db).abs().max()))
        else:
            # graded systems of kappa ~1e3: c kappa u32 with the forward's c is below 1e-4; 1e-3 leaves room for the windows' coupling
            assert _rel(db, da) <= 1e-3, (entry, a, b, _rel(db, da))
        print(entry, a, va, b, vb, f"max |diff| {float((da - db).abs().max()):.2e}")


BWD_SWITCHES = {"pairs": [(a, b) for a, b, _ in M.switches(M.PLANS["lm_solve_bwd_pairs"][0], 7, 400)][:2],
                "dense_window": [(a, b) for a, b, _ in M.switches(M.PLANS["lm_solve_bwd_dense_window"][0], 7, 400)][:2]}


@pytest.mark.gpu
@pytest.mark.parametrize("entry", list(BWD_SWITCHES))
def test_each_backward_switch_is_crossed_by_padding(entry):
    """The backward's switches (square fp64 to packed fp64 at 157/158, packed fp64 to packed fp32 at 222/223), crossed as the forward's: the same
    system and upstream gradients below the switch, and padded with decoupled identity unknowns (zero g, zero dW') above it.  Every
    gradient of the first unknowns agrees to the fp32 bound, and the padding gets exactly zero dH, dg."""
    from banet_b200 import ops, _lib
    _lib.require_device()
    lam = torch.tensor([0.1], dtype=torch.float32).double()
    for a, b in BWD_SWITCHES[entry]:
        assert M.PLANS["lm_solve_bwd_pairs" if entry == "pairs" else "lm_solve_bwd_dense_window"][0](a) in F64
        if entry == "pairs":
            H = torch.stack([graded_spd(a, 1e3, a)]).double(); g = rand_g(a, a)
            Hp, gp = _pad(H, g, b - a)
            R, T, W = _iterate(1, b - 6)
            gR, gT, gW = _grad_inputs(((1, 3, 3), (1, 3, 1), (1, b - 6, 1)), a)
            gW[:, a - 6:] = 0

            def both(H_, g_, n):
                f = ops.lm_solve_update(cu(H_), cu(g_), cu(lam), cu(R), cu(T), cu(W[:, :n - 6]), undamped_last=False)
                assert int(f[4].abs().max()) == 0
                return ops.lm_solve_update_bwd(cu(H_), cu(g_), cu(lam), f[3], cu(R), cu(T), cu(gR), cu(gT), cu(gW[:, :n - 6]), undamped_last=False)
            ga, gb = both(H, g, a), both(Hp, gp, b)
            cut = [lambda x: x[:, :a, :a], lambda x: x[:, :a], lambda x: x, lambda x: x, lambda x: x, lambda x: x[:, :a - 6]]
            pads = (gb[0][:, a:, :].abs().max(), gb[0][:, :, a:].abs().max(), gb[1][:, a:].abs().max())
        else:
            nf = 2
            Hs = torch.stack([graded_spd(a - 6, 1e3, a + f) for f in range(nf)]).double(); g = rand_g(a - 6, a, nf)
            Hs = torch.stack([h + 2 * torch.eye(a - 6, dtype=torch.float64) for h in Hs]).float().double()
            Hp, gp = _pad(Hs, g, b - a); Hp[1, a - 6:, a - 6:] = 0
            R, T, W = _iterate(nf, b - 12)
            gR, gT, gW = _grad_inputs(((nf, 3, 3), (nf, 3, 1), (b - 12, 1)), a)
            gW[a - 12:] = 0

            def both(H_, g_, n):
                f = ops.lm_window_solve_update(cu(H_), cu(g_), cu(lam), cu(R), cu(T), cu(W[0, :n - 12]), undamped_last=False)
                assert int(f[4].abs().max()) == 0
                return ops.lm_window_solve_update_bwd(cu(H_), cu(g_), cu(lam), f[3], cu(R), cu(T), cu(gR), cu(gT), cu(gW[:n - 12]),
                                                      undamped_last=False)
            ga, gb = both(Hs, g, a), both(Hp, gp, b)
            P = a - 6
            cut = [lambda x: x[:, :P, :P], lambda x: x[:, :P], lambda x: x, lambda x: x, lambda x: x, lambda x: x[:a - 12]]
            pads = (gb[0][:, P:, :].abs().max(), gb[0][:, :, P:].abs().max(), gb[1][:, P:].abs().max())
        errs = [_rel(c(y), x) for c, x, y in zip(cut, ga, gb)]
        print(entry, a, b, "dH, dg, dlambda, dR, dT, dW:", " ".join(f"{e:.1e}" for e in errs))
        # graded systems of kappa ~1e3: c kappa u32 is below 1e-4 for the fp32 side
        assert max(errs) <= 1e-3, (entry, a, b, errs)
        assert all(float(x) == 0.0 for x in pads), (entry, a, b, pads)


# ---- backward against float64 autograd
def _grad_inputs(shapes, seed):
    gen = torch.Generator().manual_seed(seed)
    return [torch.randn(s, generator=gen, dtype=torch.float64).float().double() for s in shapes]


def _bwd_case(entry, n, seed):
    """-> (variant, {name: rel error}) of one backward against float64 autograd of the same fp32 inputs (lambda = 0.1)."""
    from banet_b200 import ops
    lam0 = float(np.float32(0.1))
    if entry == "pairs":
        H, g, _ = pair_systems(n, 2, seed)
        R, T, W = _iterate(2, n - 6)
        lam = torch.full((2,), lam0, dtype=torch.float64)
        gR, gT, gW = _grad_inputs(((2, 3, 3), (2, 3, 1), (2, n - 6, 1)), seed)
        fwd = ops.lm_solve_update(cu(H), cu(g), cu(lam), cu(R), cu(T), cu(W))
        got = ops.lm_solve_update_bwd(cu(H), cu(g), cu(lam), fwd[3], cu(R), cu(T), cu(gR), cu(gT), cu(gW))
        step = lambda *a: pair_step64(*a)
        variant = M.step_plan(n)
    elif entry == "dense_window":
        nf = 2
        H, g, _ = pair_systems(n - 6 * nf + 6, nf, seed)
        K = n - 12
        R, T, W = _iterate(nf, K); W = W[0]
        lam = torch.tensor([lam0], dtype=torch.float64)
        gR, gT, gW = _grad_inputs(((nf, 3, 3), (nf, 3, 1), (K, 1)), seed)
        fwd = ops.lm_window_solve_update(cu(H), cu(g), cu(lam), cu(R), cu(T), cu(W))
        got = ops.lm_window_solve_update_bwd(cu(H), cu(g), cu(lam), fwd[3], cu(R), cu(T), cu(gR), cu(gT), cu(gW))
        step = lambda *a: dense_window_step64(*a, fp32_assembly=True)
        variant = M.step_plan(n)
    else:
        nw, nf, K = 2, 2, n
        H, g, _ = pair_systems(6 + K, nw * nf, seed)
        R, T, W = _iterate(nw * nf, K); W = W[:nw]
        lam = torch.full((nw,), lam0, dtype=torch.float64)
        gR, gT, gW = _grad_inputs(((nw * nf, 3, 3), (nw * nf, 3, 1), (nw, K, 1)), seed)
        fwd = ops.lm_window_batch_solve_update(cu(H), cu(g), cu(lam), cu(R), cu(T), cu(W))
        got = ops.lm_window_batch_solve_update_bwd(cu(H), cu(g), cu(lam), fwd[3], cu(R), cu(T), cu(gR), cu(gT), cu(gW))
        step = lambda *a: arrow_step64(*a, nw)
        variant = M.arrow_plan(K, 0)
    assert int(fwd[-1].abs().max()) == 0
    leaves = [t.clone().requires_grad_() for t in (H, g, lam, R, T, W)]
    Rn, Tn, Wn, _ = step(*leaves)
    ((Rn * gR).sum() + (Tn * gT).sum() + (Wn * gW).sum()).backward()
    names = ("dH", "dg", "dlambda", "dR", "dT", "dW")
    errs = {k: _rel(_sym(x.reshape(l.shape)) if k == "dH" else x.reshape(l.shape), _sym(l.grad) if k == "dH" else l.grad)
            for k, x, l in zip(names, got, leaves)}
    return variant, errs


def _sym(dH):
    """The kernels read the lower triangle of each symmetric H and write dH = -u delta^T; the float64 statements read other entries of
    the same symmetric matrix.  dH + dH^T is the gradient both give for a symmetric perturbation."""
    dH = torch.as_tensor(dH).double().cpu()
    return dH + dH.transpose(-1, -2)


BWD_SIZES = {
    "pairs": accepted_edges("lm_solve_bwd_pairs"),
    "dense_window": accepted_edges("lm_solve_bwd_dense_window"),
    "arrow": [s for s in M.edge_sizes("arrow_lambda_given") if M.arrow_plan(s, 0) != M.REJECT] + [153],
}
# bounds of the backward on the realistic systems at lambda = 0.1 (kappa up to ~3e6) and the graded ones (kappa = 1e4).  Largest measured
# errors on an H100 80GB HBM3: 4.5e-7 (fp64 variants, the arrow) and 2.4e-4 (fp32 variants, the dense window); DESIGN.md section 4
BWD_BOUND = {"fp64": 5e-6, "fp32": 2e-3}


@pytest.mark.gpu
@pytest.mark.parametrize("entry", list(BWD_SIZES))
def test_backward_matches_float64_autograd(entry):
    from banet_b200 import _lib
    _lib.require_device()
    worst = {"fp64": 0.0, "fp32": 0.0}
    for n in BWD_SIZES[entry]:
        variant, errs = _bwd_case(entry, n, seed=n)
        prec = "fp64" if variant in F64 else "fp32"
        worst[prec] = max(worst[prec], max(errs.values()))
        print(entry, n, variant, " ".join(f"{k} {v:.1e}" for k, v in errs.items()))
        assert max(errs.values()) <= BWD_BOUND[prec], (entry, n, variant, errs)
    print(f"{entry}: worst backward error {worst}")


# ---- the skip contract
CAUSES = ("pivot_col0", "pivot_last_panel", "undamped_last_zero", "nonfinite_H", "nonfinite_g", "nonfinite_lambda")


def last_panel_col(n):
    """First column of the last panel of 4 when a system of n unknowns is factored in panels of STEP_NB = 4 (partial when n % 4 != 0)."""
    return M.STEP_NB * ((n - 1) // M.STEP_NB)


def _poison(H, g, lam, cause, P, panel_col):
    """Poison one per-pair system of size P in place.  panel_col: the row of this pair's H that becomes the first column of the last
    panel of the factored system (the pair's own, the assembled window's, or the arrow's K x K depth system)."""
    if cause == "pivot_col0":
        H[0, 0] = -1.0
    elif cause == "pivot_last_panel":
        H[panel_col, panel_col] = -1e6                              # negative after damping, and after the sum over a window's frames
    elif cause == "undamped_last_zero":
        H[P - 1, :] = 0; H[:, P - 1] = 0                            # a basis column zero on every valid pixel
    elif cause == "nonfinite_H":
        H[3, 3] = float("inf")
    elif cause == "nonfinite_g":
        g[5] = float("nan")
    else:
        lam.fill_(float("inf"))


# every size has a partial last panel of 4 (n % 4 != 0): the "pivot_last_panel" cause poisons its first column
SKIP_SIZES = {
    "lm_step_lambda_given": [157, 222, 223],
    "lm_step_mlp_C128": [157, 222, 223],
    "lm_solve": [157, 222, 223],
    "dense_window": [157, 222, 223],
    "arrow": [153, 155, 217],
}


def _skip_fwd(entry, n, cause):
    """-> clean outputs, poisoned outputs, the poisoned batch index set, expected status bits, inputs (CPU)."""
    from banet_b200 import ops
    lam0 = float(np.float32(0.3))
    if entry in ("lm_step_lambda_given", "lm_step_mlp_C128", "lm_solve"):
        nb, P = 2, n
        H = torch.stack([graded_spd(P, 1e3, P + i) for i in range(nb)]).double(); g = rand_g(P, P, nb)
        R, T, W = _iterate(nb, P - 6)
        lam = torch.full((nb,), lam0, dtype=torch.float64)
        rb = 0.02 * (1 + torch.rand(nb, 128, generator=torch.Generator().manual_seed(n))) * 4096
        if entry == "lm_step_mlp_C128":
            mlp = ops.pack_mlp(mlp_for(128, 3, torch.float32)).cuda()
            run = lambda H_, g_, lam_, rb_: ops.lm_step(cu(H_), cu(g_), cu(rb_), 4096, mlp, 1000.0, cu(R), cu(T), cu(W))
        elif entry == "lm_step_lambda_given":
            run = lambda H_, g_, lam_, rb_: ops.lm_step(cu(H_), cu(g_), None, 1, None, 1.0, cu(R), cu(T), cu(W), lam=cu(lam_))
        else:
            run = lambda H_, g_, lam_, rb_: ops.lm_solve_update(cu(H_), cu(g_), cu(lam_), cu(R), cu(T), cu(W))
        clean = run(H, g, lam, rb)
        Hp, gp, lp, rbp = H.clone(), g.clone(), lam.clone(), rb.clone()
        if cause == "nonfinite_lambda" and entry == "lm_step_mlp_C128":
            rbp[1, 7] = float("inf")                                 # lambda comes from the MLP: a non-finite residual statistic
        else:
            _poison(Hp[1], gp[1], lp[1:2], cause, P, last_panel_col(P))
        bad = run(Hp, gp, lp, rbp)
        return clean, bad, [1], (R, T, W), (H, g, lam, Hp, gp, lp)
    if entry == "dense_window":
        nf, Pj = 2, n
        K = Pj - 12
        H = torch.stack([graded_spd(6 + K, 1e3, n + f) for f in range(nf)]).double(); g = rand_g(6 + K, n, nf)
        R, T, W = _iterate(nf, K); W = W[0]
        lam = torch.tensor([lam0], dtype=torch.float64)
        run = lambda H_, g_, lam_: ops.lm_window_solve_update(cu(H_), cu(g_), cu(lam_), cu(R), cu(T), cu(W))
        clean = run(H, g, lam)
        Hp, gp, lp = H.clone(), g.clone(), lam.clone()
        # frame 0 carries the poison; in the assembled system the last depth row is the sum over the frames, so zero it in both
        col = 6 + last_panel_col(Pj) - 6 * nf                      # column last_panel_col(Pj) of the assembled system is depth unknown col - 6
        _poison(Hp[0], gp[0], lp, cause, 6 + K, col)
        if cause == "undamped_last_zero":
            _poison(Hp[1], gp[1], lp, cause, 6 + K, col)
        bad = run(Hp, gp, lp)
        return clean, bad, [0, 1], (R, T, W), (H, g, lam, Hp, gp, lp)
    nw, nf, K = 2, 2, n
    H = torch.stack([graded_spd(6 + K, 1e3, n + f) for f in range(nw * nf)]).double(); g = rand_g(6 + K, n, nw * nf)
    R, T, W = _iterate(nw * nf, K); W = W[:nw]
    lam = torch.full((nw,), lam0, dtype=torch.float64)
    run = lambda H_, g_, lam_: ops.lm_window_batch_solve_update(cu(H_), cu(g_), cu(lam_), cu(R), cu(T), cu(W))
    clean = run(H, g, lam)
    Hp, gp, lp = H.clone(), g.clone(), lam.clone()
    col = 6 + last_panel_col(K)                                      # the arrow factors the K x K depth system in panels
    _poison(Hp[2], gp[2], lp[1:2], cause, 6 + K, col)                 # window 1, frame 0
    if cause == "undamped_last_zero":
        _poison(Hp[3], gp[3], lp[1:2], cause, 6 + K, col)
    bad = run(Hp, gp, lp)
    return clean, bad, [1], (R, T, W), (H, g, lam, Hp, gp, lp)


def _expected_bits(cause, status):
    if cause in ("pivot_col0", "pivot_last_panel", "undamped_last_zero"):
        return status == 1
    return (status & 2) == 2


@pytest.mark.gpu
@pytest.mark.parametrize("entry", list(SKIP_SIZES))
def test_skip_contract_forward(entry):
    """Every skip cause at every variant: the status bits, a zero step, R, T, W unchanged bit for bit, and the other pairs or windows
    bitwise as without the poison."""
    from banet_b200 import _lib
    _lib.require_device()
    for n in SKIP_SIZES[entry]:
        for cause in CAUSES:
            clean, bad, _, (R, T, W), _ = _skip_fwd(entry, n, cause)
            st = bad[-1].cpu()
            assert int(clean[-1].abs().max()) == 0, (entry, n, cause)
            Rc, Tc = cu(R), cu(T)
            if entry in ("lm_step_lambda_given", "lm_step_mlp_C128", "lm_solve"):
                assert _expected_bits(cause, int(st[1])) and int(st[0]) == 0, (entry, n, cause, st)
                assert bool((bad[3][1] == 0).all())
                assert torch.equal(bad[0][1], Rc[1]) and torch.equal(bad[1][1], Tc[1]) and torch.equal(bad[2][1], cu(W)[1])
                for a, b in zip(bad[:4], clean[:4]):
                    assert torch.equal(a[0], b[0]), (entry, n, cause)
            elif entry == "dense_window":
                assert all(_expected_bits(cause, int(s)) for s in st), (entry, n, cause, st)
                assert bool((bad[3] == 0).all())
                assert torch.equal(bad[0], Rc) and torch.equal(bad[1], Tc) and torch.equal(bad[2], cu(W))
            else:
                assert int(st[:2].abs().max()) == 0 and all(_expected_bits(cause, int(s)) for s in st[2:]), (entry, n, cause, st)
                assert bool((bad[3][1] == 0).all())
                assert torch.equal(bad[0][2:], Rc[2:]) and torch.equal(bad[1][2:], Tc[2:]) and torch.equal(bad[2][1], cu(W)[1])
                for a, b in zip(bad[:4], clean[:4]):
                    k = 1 if a.shape[0] == 2 else 2
                    assert torch.equal(a[:k], b[:k]), (entry, n, cause)


BWD_SKIP_SIZES = {"pairs": [157, 222, 223], "dense_window": [157, 222, 223], "arrow": [153, 155, 217]}


@pytest.mark.gpu
@pytest.mark.parametrize("entry", list(BWD_SKIP_SIZES))
def test_skip_contract_backward(entry):
    """Every skip cause at every variant of the backwards: dH = dg = dlambda = 0, dR, dT, dW passed through, the others bitwise as
    without the poison."""
    from banet_b200 import ops, _lib
    _lib.require_device()
    fwd_entry = {"pairs": "lm_solve", "dense_window": "dense_window", "arrow": "arrow"}[entry]
    for n in BWD_SKIP_SIZES[entry]:
        for cause in CAUSES:
            clean, bad, _, (R, T, W), (H, g, lam, Hp, gp, lp) = _skip_fwd(fwd_entry, n, cause)
            nb = H.shape[0]
            K = H.shape[-1] - 6
            gR, gT = _grad_inputs(((nb, 3, 3), (nb, 3, 1)), n)
            gW = _grad_inputs((W.shape,), n + 1)[0]
            bwd = {"pairs": ops.lm_solve_update_bwd, "dense_window": ops.lm_window_solve_update_bwd,
                   "arrow": ops.lm_window_batch_solve_update_bwd}[entry]
            gc = bwd(cu(H), cu(g), cu(lam), clean[3], cu(R), cu(T), cu(gR), cu(gT), cu(gW))
            gb = bwd(cu(Hp), cu(gp), cu(lp), bad[3], cu(R), cu(T), cu(gR), cu(gT), cu(gW))
            dH, dg, dl, dR, dT, dW = gb
            if entry == "pairs":
                s = 1
                for x in (dH[s], dg[s], dl[s]):
                    assert bool((x == 0).all()), (entry, n, cause)
                assert torch.equal(dW[s], cu(gW)[s])
                assert torch.allclose(dR[s], cu(gR)[s], rtol=1e-6, atol=0) and torch.allclose(dT[s], cu(gT)[s], rtol=1e-6, atol=0)
                for a, b in zip(gb, gc):
                    assert torch.equal(a[0], b[0]), (entry, n, cause)
            elif entry == "dense_window":
                for x in (dH, dg, dl):
                    assert bool((x == 0).all()), (entry, n, cause)
                assert torch.equal(dW, cu(gW))
                assert torch.allclose(dR, cu(gR), rtol=1e-6, atol=0) and torch.allclose(dT, cu(gT), rtol=1e-6, atol=0)
            else:
                for x in (dH[2:], dg[2:], dl[1]):
                    assert bool((x == 0).all()), (entry, n, cause)
                assert torch.equal(dW[1], cu(gW)[1])
                assert torch.allclose(dR[2:], cu(gR)[2:], rtol=1e-6, atol=0) and torch.allclose(dT[2:], cu(gT)[2:], rtol=1e-6, atol=0)
                for a, b in zip(gb, gc):
                    k = 1 if a.shape[0] == 2 else 2
                    assert torch.equal(a[:k], b[:k]), (entry, n, cause)


# ---- the backward's skip is the forward's status where definiteness depends on the precision
def _precision_dependent(P, j):
    """A graded system (kappa = 1e3) with a decoupled 2 x 2 block at unknowns j, j+1: [[1, h], [h, 2^-149]], h = 2^-75 (1 + 2^-23).  Its
    second pivot 2^-149 - h^2 = 2^-150 (1 - 2^-22 - 2^-46) is positive, and every fp64 factorisation finds it.  In fp32 it lies below half
    the smallest subnormal: h^2 (or 2^-149 - h^2 in one fused operation) rounds so that the pivot is exactly 0, whatever the order of the
    factorisation, so every fp32 factorisation reports a non-positive pivot (lambda = 0: no damping moves it)."""
    H = graded_spd(P, 1e3, P).double()
    H[j, :] = 0; H[:, j] = 0; H[j + 1, :] = 0; H[:, j + 1] = 0
    h = 2.0 ** -75 * (1 + 2.0 ** -23)
    H[j, j] = 1.0; H[j, j + 1] = H[j + 1, j] = h; H[j + 1, j + 1] = 2.0 ** -149
    assert bool((H.float().double() == H).all())                     # exactly representable in fp32
    return H


def _emulate_fp32_lm_solve_notpd(H):
    """float32 restatement of a column-by-column Cholesky factorisation: does it meet a non-positive pivot?"""
    A = np.tril(H.numpy().astype(np.float32))
    P = A.shape[0]
    with np.errstate(all="ignore"):
        for j in range(P):
            d = A[j, j]
            if not d > 0:
                return True
            invd = np.float32(1) / d
            ci = A[j + 1:, j] * invd
            A[j + 1:, j + 1:] -= np.tril(np.outer(ci, A[j + 1:, j]).astype(np.float32))
    return False


def test_precision_dependent_system_is_definite_only_in_fp64():
    P = 223
    H = _precision_dependent(P, 200)
    torch.linalg.cholesky(H)                                         # positive definite in float64
    assert _emulate_fp32_lm_solve_notpd(H)
    assert not _emulate_fp32_lm_solve_notpd(graded_spd(P, 1e3, P).double())


@pytest.mark.gpu
@pytest.mark.parametrize("entry,n", [("pairs", 223), ("pairs", 224), ("pairs", 222), ("pairs", 225), ("dense_window", 220),
                                     ("dense_window", 221), ("dense_window", 222), ("dense_window", 223), ("dense_window", 224)])
def test_backward_skip_equals_forward_status(entry, n):
    """Up to P = 222 the pair and dense-window solves factor in fp64, from 223 in fp32.  The backward must reach the same skip decision:
    zero dH, dg, dlambda exactly when the forward's status is non-zero."""
    from banet_b200 import ops, _lib
    _lib.require_device()
    lam = torch.zeros(1, dtype=torch.float64)
    if entry == "pairs":
        H = _precision_dependent(n, 200)[None]
        g = rand_g(n, n); g[0, 200:202] = 0
        R, T, W = _iterate(1, n - 6)
        gR, gT, gW = _grad_inputs(((1, 3, 3), (1, 3, 1), (1, n - 6, 1)), n)
        gW[0, 194:196] = 0                                           # no adjoint on the 2 x 2 block
        fwd = ops.lm_solve_update(cu(H), cu(g), cu(lam), cu(R), cu(T), cu(W))
        bwd = ops.lm_solve_update_bwd(cu(H), cu(g), cu(lam), fwd[3], cu(R), cu(T), cu(gR), cu(gT), cu(gW))
        want_fp64 = M.step_plan(n) in F64
    else:
        nf, K = 2, n - 12
        k = 188                                                      # depth unknown 188 is column 200 of the assembled system: a panel start
        H = torch.stack([_precision_dependent(6 + K, 6 + k), graded_spd(6 + K, 1e3, n).double()])
        H[1, 6 + k:8 + k, :] = 0; H[1, :, 6 + k:8 + k] = 0            # frame 1 adds nothing to the block's rows of the depth system
        g = rand_g(6 + K, n, nf); g[:, 6 + k:8 + k] = 0
        R, T, W = _iterate(nf, K); W = W[0]
        gR, gT, gW = _grad_inputs(((nf, 3, 3), (nf, 3, 1), (K, 1)), n)
        gW[k:k + 2] = 0
        fwd = ops.lm_window_solve_update(cu(H), cu(g), cu(lam), cu(R), cu(T), cu(W))
        bwd = ops.lm_window_solve_update_bwd(cu(H), cu(g), cu(lam), fwd[3], cu(R), cu(T), cu(gR), cu(gT), cu(gW))
        want_fp64 = M.step_plan(n) in F64
    status = int(fwd[-1].abs().max())
    zero_grad = all(bool((x == 0).all()) for x in bwd[:3])
    print(entry, n, "forward status", status, "backward zero", zero_grad)
    assert status == (0 if want_fp64 else 1)
    assert zero_grad == (status != 0)
    if status == 0:
        assert all(bool(torch.isfinite(x).all()) for x in bwd)


# ---- the backward's skip is the forward's status where definiteness depends on the order of the factorisation
def _fma32(a, b, c):
    """fp32 fused multiply-add of fp32 operands (the product is exact in float64)."""
    return np.float32(float(a) * float(b) + float(c))


def _emulate_fp32_column_notpd(B):
    """float32 restatement, with fused multiply-adds, of the column-by-column factorisation (one column at a time, the trailing matrix
    updated with the unscaled column times 1/d): does it meet a non-positive pivot?"""
    A = np.tril(np.asarray(B, dtype=np.float32))
    n, notpd = A.shape[0], False
    for j in range(n):
        d = A[j, j]
        if not d > 0:
            notpd, d = True, np.float32(1)
        invd = np.float32(1) / d
        for i in range(j + 1, n):
            ci = np.float32(A[i, j] * invd)
            for k in range(j + 1, i + 1):
                A[i, k] = _fma32(-ci, A[k, j], A[i, k])
    return notpd


def _emulate_fp32_panel_notpd(B):
    """float32 restatement, with fused multiply-adds, of step_cholesky_solve (lm_step.cuh): panels of STEP_NB columns, each diagonal block
    factored with reciprocal square roots, the rows below solved against it, the trailing matrix updated with one sum per entry.  The
    hardware's reciprocal square root is approximate; this one is correctly rounded.  Does it meet a non-positive pivot?"""
    A = np.tril(np.asarray(B, dtype=np.float32))
    n, notpd = A.shape[0], False
    for j0 in range(0, n, M.STEP_NB):
        jb = min(M.STEP_NB, n - j0)
        L, inv = A[j0:j0 + jb, j0:j0 + jb].copy(), np.zeros(jb, dtype=np.float32)
        for c in range(jb):
            d = L[c, c]
            for m in range(c):
                d = _fma32(-L[c, m], L[c, m], d)
            if not d > 0:
                notpd, d = True, np.float32(1)
            inv[c] = np.float32(1.0 / np.sqrt(float(d)))
            L[c, c] = np.float32(d * inv[c])
            for r in range(c + 1, jb):
                v = L[r, c]
                for m in range(c):
                    v = _fma32(-L[r, m], L[c, m], v)
                L[r, c] = np.float32(v * inv[c])
        A[j0:j0 + jb, j0:j0 + jb] = np.tril(L)
        for i in range(j0 + jb, n):
            for c in range(jb):
                v = A[i, j0 + c]
                for m in range(c):
                    v = _fma32(-A[i, j0 + m], L[c, m], v)
                A[i, j0 + c] = np.float32(v * inv[c])
        for i in range(j0 + jb, n):
            for k in range(j0 + jb, i + 1):
                sv = np.float32(0)
                for c in range(jb):
                    sv = _fma32(A[i, j0 + c], A[k, j0 + c], sv)
                A[i, k] = np.float32(A[i, k] - sv)
    return notpd


def _order_dependent_blocks(count=4, m=6):
    """m x m fp32 blocks V V^T (V: m x (m - 1)) with a tiny positive multiple of e_m e_m^T: their last pivot is a few ulps from zero, fed by
    every earlier column.  -> (seed, block, column order's verdict, panel order's verdict) for the first `count` seeds whose verdicts
    differ, panels starting at the block's first column."""
    out = []
    for seed in range(4000):
        gen = torch.Generator().manual_seed(seed)
        V = torch.randn(m, m - 1, generator=gen, dtype=torch.float64)
        B = V @ V.T
        B[m - 1, m - 1] += 2.0 ** -22 * float(B[m - 1, m - 1])
        B = B.float().double()
        col, pan = _emulate_fp32_column_notpd(B.numpy()), _emulate_fp32_panel_notpd(B.numpy())
        if col != pan:
            out.append((seed, B, col, pan))
            if len(out) == count:
                break
    return out


ORDER_BLOCKS = {}


def order_blocks():
    if not ORDER_BLOCKS:
        ORDER_BLOCKS["v"] = _order_dependent_blocks()
    return ORDER_BLOCKS["v"]


def test_order_dependent_blocks_exist():
    """The emulations agree with float64 on a well-conditioned system and disagree with each other on the blocks the GPU test uses, in both
    directions among them."""
    good = graded_spd(12, 1e2, 3).double().numpy()
    assert not _emulate_fp32_column_notpd(good) and not _emulate_fp32_panel_notpd(good)
    blocks = order_blocks()
    assert len(blocks) == 4
    assert {(c, p) for _, _, c, p in blocks} == {(True, False), (False, True)}, [(sd, c, p) for sd, _, c, p in blocks]


@pytest.mark.gpu
def test_backward_skip_equals_forward_status_order_dependent():
    """Dense windows of Pj = 224 unknowns (fp32 storage) holding a decoupled block whose last pivot is within a few ulps of zero, fed by five
    earlier columns, at a panel start: whether the factorisation meets a non-positive pivot depends on the order of its operations.  The
    backward must reach the forward's skip decision: zero dH, dg, dlambda exactly when the forward's status is non-zero."""
    from banet_b200 import ops, _lib
    _lib.require_device()
    nf, n = 2, 224
    K, k = n - 12, 188                                               # depth unknown 188 is column 200 of the assembled system: a panel start
    assert M.step_plan(n) == M.PACKED32
    lam = torch.zeros(1, dtype=torch.float64)
    rows = []
    for seed, Bk, col, pan in order_blocks():
        m = Bk.shape[0]
        H = torch.stack([graded_spd(6 + K, 1e3, n).double(), graded_spd(6 + K, 1e3, n + 1).double()])
        H[:, 6 + k:6 + k + m, :] = 0; H[:, :, 6 + k:6 + k + m] = 0
        H[0, 6 + k:6 + k + m, 6 + k:6 + k + m] = Bk                 # frame 1 adds nothing to the block's rows of the depth system
        g = rand_g(6 + K, n, nf); g[:, 6 + k:6 + k + m] = 0
        R, T, W = _iterate(nf, K); W = W[0]
        gR, gT, gW = _grad_inputs(((nf, 3, 3), (nf, 3, 1), (K, 1)), n)
        gW[k:k + m] = 0                                              # no adjoint on the block
        fwd = ops.lm_window_solve_update(cu(H), cu(g), cu(lam), cu(R), cu(T), cu(W))
        bwd = ops.lm_window_solve_update_bwd(cu(H), cu(g), cu(lam), fwd[3], cu(R), cu(T), cu(gR), cu(gT), cu(gW))
        status = int(fwd[-1].abs().max())
        zero_grad = all(bool((x == 0).all()) for x in bwd[:3])
        rows.append((seed, col, pan, status, zero_grad))
        print("seed", seed, "column order not PD", col, "panel order not PD", pan, "forward status", status, "backward zero", zero_grad)
    assert all(z == (st != 0) for _, _, _, st, z in rows), rows


# ---- the arrow's per-frame loops past their wraps
@pytest.mark.gpu
@pytest.mark.parametrize("nf", [1, 32, 33, 1024, 1025])
def test_arrow_frame_wraps(nf):
    """Thread-per-frame loops wrap at 1024 frames, warp-per-frame loops at 32: forward and backward against float64 at K = 5, 6, 7."""
    from banet_b200 import ops, _lib
    _lib.require_device()
    for K in (5, 6, 7):
        P = 6 + K
        H = torch.stack([graded_spd(P, 1e2, 1000 * K + f) for f in range(nf)]).double(); g = rand_g(P, K, nf)
        R, T, W = _iterate(nf, K); W = W[:1]
        lam = torch.tensor([float(np.float32(0.2))], dtype=torch.float64)
        fwd = ops.lm_window_batch_solve_update(cu(H), cu(g), cu(lam), cu(R), cu(T), cu(W))
        assert int(fwd[4].abs().max()) == 0
        ref = arrow_step64(H, g, lam, R, T, W, 1)
        errs = [_rel(fwd[i], ref[i]) for i in range(4)]
        gR, gT, gW = _grad_inputs(((nf, 3, 3), (nf, 3, 1), (1, K, 1)), K)
        got = ops.lm_window_batch_solve_update_bwd(cu(H), cu(g), cu(lam), fwd[3], cu(R), cu(T), cu(gR), cu(gT), cu(gW))
        leaves = [t.clone().requires_grad_() for t in (H, g, lam, R, T, W)]
        Rn, Tn, Wn, _ = arrow_step64(*leaves, 1)
        ((Rn * gR).sum() + (Tn * gT).sum() + (Wn * gW).sum()).backward()
        berrs = [_rel(_sym(x.reshape(l.shape)), _sym(l.grad)) if i == 0 else _rel(x.reshape(l.shape), l.grad)
                 for i, (x, l) in enumerate(zip(got, leaves))]
        print(nf, K, " ".join(f"{e:.1e}" for e in errs), "|", " ".join(f"{e:.1e}" for e in berrs))
        assert max(errs) < 1e-5 and max(berrs) < 1e-4, (nf, K, errs, berrs)


# ---- the entries that share lm_step's code
@pytest.mark.gpu
def test_solve_update_is_lm_step_with_lambda_given():
    """banet_lm_solve_update equals banet_lm_step with lambda_in, and their backwards are equal, bit for bit at every edge size."""
    from banet_b200 import ops, _lib
    _lib.require_device()
    for n in accepted_edges("lm_solve"):
        H, g, _ = pair_systems(n, 2, n)
        R, T, W = _iterate(2, n - 6)
        lam = cu(torch.tensor([0.1, 10.0]))
        gR, gT, gW = _grad_inputs(((2, 3, 3), (2, 3, 1), (2, n - 6, 1)), n)
        a = ops.lm_solve_update(cu(H), cu(g), lam, cu(R), cu(T), cu(W))
        b = ops.lm_step(cu(H), cu(g), None, 1, None, 1.0, cu(R), cu(T), cu(W), lam=lam)
        for name, x, y in zip(("R", "T", "W", "delta", "status"), a, (b[0], b[1], b[2], b[3], b[5])):
            assert torch.equal(x, y), (n, name)
        da = ops.lm_solve_update_bwd(cu(H), cu(g), lam, a[3], cu(R), cu(T), cu(gR), cu(gT), cu(gW))
        db = ops.lm_step_bwd(cu(H), cu(g), None, 1, None, b[4], b[3], cu(R), cu(T), cu(gR), cu(gT), cu(gW))
        for name, x, y in zip(("dH", "dg", "dlambda", "dR", "dT", "dW"), da, (db[0], db[1], db[4], db[5], db[6], db[7])):
            assert torch.equal(x, y), (n, name)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [5, 128, 256])
def test_lm_lambda_is_lm_steps_lambda(C):
    """banet_lm_lambda computes, bit for bit, the lambda lm_step reports with the MLP."""
    from banet_b200 import ops, _lib
    _lib.require_device()
    H, g, _ = pair_systems(22, 3, 1)
    R, T, W = _iterate(3, 16)
    rb = cu(0.02 * (1 + torch.rand(3, C, generator=torch.Generator().manual_seed(C))) * 4096)
    mlp = ops.pack_mlp(mlp_for(C, 3, torch.float32)).cuda()
    out = ops.lm_step(cu(H), cu(g), rb, 4096, mlp, 1000.0, cu(R), cu(T), cu(W))
    assert torch.equal(ops.lm_lambda(rb, 4096, mlp, 1000.0), out[4])


@pytest.mark.gpu
def test_inference_and_training_factor_alike():
    """lm_step with the lambda-MLP at C = 128 equals lm_step given the lambda it reported, bit for bit, at P = 219..222 (where the MLP's
    buffers used to move the step to fp32 storage while the training forward stayed in fp64)."""
    from banet_b200 import ops, _lib
    _lib.require_device()
    mlp = ops.pack_mlp(mlp_for(128, 3, torch.float32)).cuda()
    for n in range(219, 223):
        H, g, _ = pair_systems(n, 2, n)
        R, T, W = _iterate(2, n - 6)
        rb = cu(0.02 * (1 + torch.rand(2, 128, generator=torch.Generator().manual_seed(n))) * 4096)
        a = ops.lm_step(cu(H), cu(g), rb, 4096, mlp, 1000.0, cu(R), cu(T), cu(W))
        b = ops.lm_step(cu(H), cu(g), None, 1, None, 1.0, cu(R), cu(T), cu(W), lam=a[4])
        for name, x, y in zip(("R", "T", "W", "delta", "lambda", "status"), a, b):
            assert torch.equal(x, y), (n, name)


# ---- every instantiation runs
@pytest.mark.gpu
def test_profiler_lists_every_instantiation():
    from banet_b200 import _lib
    from torch.profiler import profile, ProfilerActivity
    _lib.require_device()
    built()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for n in (157, 158, 223):
            _fwd_case("lm_step_mlp_C128", n, None, 1)
            _fwd_case("lm_step_lambda_given", n, 0.1, 1)
            _fwd_case("lm_solve", n, 0.1, 1)
            _bwd_case("pairs", n, 1)
        for n in (154, 155, 216):
            _fwd_case("arrow", n, 0.1, 1)
            _bwd_case("arrow", n, 1)
        torch.cuda.synchronize()
    names = {e.key for e in prof.key_averages()}
    want = [f"{k}<{s}>" for k in ("lm_step_kernel", "lm_step_bwd_kernel", "window_arrow_step_kernel", "window_arrow_step_bwd_kernel")
             for s in ("double, true", "double, false", "float, false")]
    missing = [w for w in want if not any(w in n for n in names)]
    print(sorted(n for n in names if "kernel<" in n))
    assert not missing, missing
