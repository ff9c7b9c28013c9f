"""Every entry point at batches past 65 535 pairs or windows, and with per-pair offsets past 2^31 elements, against float64.

CUDA caps gridDim.y and gridDim.z at 65 535.  Launches that put the pair or window index on grid.y (the build's and the keyframe build's
reduce, depth_compose's backward) stride over it, so a batch of any size runs; eqc keeps its documented limit of 65 535 pairs, which its
entry points reject before any CUDA call.

  * CPU: banet_eqc_fwd / _bwd reject nb = 65 536 with BANET_ERR_UNSUPPORTED and get past that check at nb = 65 535.
  * GPU, at nb in {65 535, 65 536, 65 537, 131 073}: every pair has its own map, points, pose, intrinsics, W and weights, and fits one
    tile, so one pair that reads another's slot or row shows up.  H at K = 128 in float64 would not fit host memory, so the oracle sees a
    fixed sample of pairs (the first and last 64, 65 534 to 65 537, every 997th); kernels whose float64 statement is cheap are checked on the
    whole batch.  Where a pair's result does not depend on the rest of the batch it must also equal, bit for bit, the same pairs launched
    as a small batch at the same indices (the head of 65 535 pairs; for the paths without a pair-index dither, any slice).
  * GPU, past 2^31 elements: nb * P^2 > 2^31 with nb < 65 536, so one pair's H block straddles element 2^31 and the last lies beyond it.
"""
import json
import os
import subprocess
import sys

import pytest
import torch

import solve_plan_model as SM
import test_build_edges as BE
import test_solve_edges as SE
import test_step_grad as SG
from helpers import ROOT, O, mlp_for

LIMIT = 65535                                       # gridDim.y / gridDim.z
NBS = [65535, 65536, 65537, 131073]
SIMT, X1, X2, X3, AUTO = BE.SIMT, BE.X1, BE.X2, BE.X3, BE.AUTO
U32 = 2.0 ** -24


# ------------------------------------------------------------------------------------------------------------------------------------
# CPU: eqc's batch limit
# ------------------------------------------------------------------------------------------------------------------------------------
_EQC_PROBE = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from banet_b200 import _lib
lib = _lib.load()
p = 1                                        # non-null dummy pointers: nothing may reach a kernel, and no device is visible
out = {}
for nb in (65535, 65536):
    out[f"fwd:{nb}"] = [lib.banet_eqc_fwd(p, p, p, nb, 16, 8, 12, p, p, None, 0, None), lib.banet_last_error().decode()]
    out[f"bwd:{nb}"] = [lib.banet_eqc_bwd(p, p, p, p, p, nb, 16, 8, 12, 0, p, p, p, None), lib.banet_last_error().decode()]
print(json.dumps(out))
"""


def test_eqc_rejects_more_than_65535_pairs_before_any_cuda_call():
    """nb = 65 536: -4 (unsupported) naming nb, with no device visible, so before any CUDA call.  nb = 65 535 gets past the check: the
    forward stops at its workspace check (-2, no workspace given), the backward at its first CUDA call (-3)."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", _EQC_PROBE, ROOT], env=env, capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    got = json.loads(res.stdout.strip().splitlines()[-1])
    for d in ("fwd", "bwd"):
        rc, msg = got[f"{d}:65536"]
        assert rc == -4 and "nb=65536" in msg, (d, rc, msg)
    assert got["fwd:65535"][0] == -2, got["fwd:65535"]
    assert got["bwd:65535"][0] == -3, got["bwd:65535"]


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: cases, samples and small batches
# ------------------------------------------------------------------------------------------------------------------------------------
def _case(nb, N, C, K, h, w, seed, f2=False, weighted=False, inside=False):
    """test_build_edges.Case's distribution drawn on the device, with per-pair intrinsics as well: points whose projections land on the
    map or up to one texel outside it (inside=True: on the map at the start, so a solve sees every point of its pair)."""
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(seed)
    rand = lambda *s: torch.rand(*s, generator=g, device=dev)
    randn = lambda *s: torch.randn(*s, generator=g, device=dev)
    c = BE.Case.__new__(BE.Case)
    c.nb, c.N, c.C, c.K, c.h, c.w, c.f2 = nb, N, C, K, h, w, f2
    fx = float(max(h, w)) * (1.0 + 0.25 * rand(nb, 1))
    fy = fx * (1.0 + 0.1 * rand(nb, 1))
    ox = (w - 1) / 2.0 + 0.5 * (rand(nb, 1) - 0.5)
    oy = (h - 1) / 2.0 + 0.5 * (rand(nb, 1) - 0.5)
    u = rand(nb, N) * (w - 1) if inside else rand(nb, N) * (w + 1) - 1.0
    v = rand(nb, N) * (h - 1) if inside else rand(nb, N) * (h + 1) - 1.0
    c.p = torch.stack([(u - ox) / fx, (v - oy) / fy, torch.ones(nb, N, device=dev)], 1).contiguous()
    c.intr = torch.cat([fx, fy, ox, oy], 1).contiguous()
    c.D = 2.0 + rand(nb, N, 1)
    c.B = 0.5 * randn(nb, N, K) if K else None
    c.W = 0.02 * randn(nb, K, 1) if K else None
    wv = 0.01 * torch.randn(nb, 3, generator=g, device=dev, dtype=torch.float64)
    S = torch.zeros(nb, 3, 3, dtype=torch.float64, device=dev)
    S[:, 0, 1], S[:, 0, 2], S[:, 1, 2] = -wv[:, 2], wv[:, 1], -wv[:, 0]
    c.R = torch.linalg.matrix_exp(S - S.transpose(1, 2)).float().contiguous()
    c.T = 0.02 * randn(nb, 3, 1)
    c.conv1 = randn(nb, N, C)
    c.conv2 = randn(nb, h, w, C if f2 else 3 * C)
    c.weight = None
    if weighted:
        c.weight = 2.0 * rand(nb, N, 1)
        c.weight[rand(nb, N, 1) < 0.1] = 0.0
    return c


_FIELDS = ("p", "intr", "D", "B", "W", "R", "T", "conv1", "conv2", "weight")


def _map(c, fn, nb):
    s = BE.Case.__new__(BE.Case)
    s.__dict__.update(c.__dict__)
    for k in _FIELDS:
        t = getattr(c, k)
        setattr(s, k, None if t is None else fn(t))
    s.nb = nb
    return s


def _slice(c, lo, hi):
    return _map(c, lambda t: t[lo:hi], hi - lo)


def _cpu_subset(c, idx):
    ix = torch.tensor(idx, device="cuda")
    return _map(c, lambda t: t[ix].cpu().contiguous(), len(idx))


def _sample(nb):
    """The first and last 64 pairs, 65 534 to 65 537 (those that exist) and every 997th pair."""
    return sorted(set(range(min(64, nb))) | set(range(max(0, nb - 64), nb)) | {i for i in range(LIMIT - 1, LIMIT + 2) if i < nb} |
                  set(range(0, nb, 997)))


def _pieces(nb, n=1024):
    """Small batches of the same pairs at their own indices: the first and last n pairs, and n pairs from 65 535 on."""
    p = [(0, min(n, nb)), (max(0, nb - n), nb)]
    if nb > LIMIT:
        p.append((LIMIT, min(nb, LIMIT + n)))
    return p


def _dev():
    from banet_b200 import _lib
    _lib.require_device()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _build(c, prec, fb=False, bb=False, grid=None):
    from banet_b200 import ops
    return ops.lm_build(BE._level(c, fb, bb, grid), c.R, c.T, c.W, prec)


def _oracle_build(c, idx, fb=False, bb=False):
    """Float64 H, g, rbar_sum, nvalid of the pairs idx.  K = 0: the pose block of the system with one zero basis column and W = 0."""
    s = _cpu_subset(c, idx)
    if c.K == 0:
        s.K, s.B, s.W = 1, torch.zeros(s.nb, s.N, 1), torch.zeros(s.nb, 1, 1)
        H, g, rb, nv = BE._oracle(s, BE._oracle_inputs(s, fb, bb))
        return H[:, :6, :6], g[:, :6], rb, nv
    return BE._oracle(s, BE._oracle_inputs(s, fb, bb))


def _assert_pieces_equal(full, run, pieces, label):
    for lo, hi in pieces:
        small = run(lo, hi)
        for i, (x, y) in enumerate(zip(full, small)):
            if x is not None:
                assert torch.equal(x[lo:hi], y), (label, "small batch", lo, hi, i)


def _check_build(c, modes, label, fb=False, bb=False, grid=None):
    idx = _sample(c.nb)
    ref = _oracle_build(c, idx, fb, bb)
    worst = {}
    for prec in modes:
        lab = f"{label} {BE.MODE_NAME[prec]}"
        out = _build(c, prec, fb, bb, grid)
        tol = BE.TOL[BE._auto(c.K, c.N) if prec == AUTO else prec]
        worst[prec] = BE._check_forward(lab, [t[idx].cpu() for t in out], ref, tol)
        run = lambda lo, hi: _build(_slice(c, lo, hi), prec, fb, bb, grid)
        if c.nb > LIMIT:                             # the head as one launch of 65 535 pairs: same indices, so also TF32X1's dither
            _assert_pieces_equal(out, run, [(0, LIMIT)], lab)
        if prec in (SIMT, X2, X3) or (prec == AUTO and BE._auto(c.K, c.N) != X1):
            _assert_pieces_equal(out, run, _pieces(c.nb), lab)
        else:
            _assert_pieces_equal(out, run, [(0, 1024)], lab)
        del out
    return worst


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: the build
# ------------------------------------------------------------------------------------------------------------------------------------
BUILD_CFGS = {"3c-f32": ("3c", False, False, False, False), "f2-f32-w-hint": ("f2", False, False, True, True),
              "3c-bf16-w": ("3c", True, True, True, False), "f2-bf16feat-hint": ("f2", True, False, False, True),
              "f2-bf16basis-w": ("f2", False, True, True, False)}
BUILD_RUNS = [(65537, k) for k in BUILD_CFGS] + [(nb, k) for nb in (65535, 65536, 131073) for k in ("3c-f32", "f2-f32-w-hint")]


@pytest.mark.gpu
@pytest.mark.parametrize("nb,cfg", BUILD_RUNS)
def test_build_past_grid_y(nb, cfg):
    """lm_build in SIMT, TF32X2, TF32X3 and AUTO at K = 32, C = 64, N = 40 (one tile per pair) on the sample against the oracle, and the
    small batches bit for bit."""
    _dev()
    layout, fb, bb, weighted, hint = BUILD_CFGS[cfg]
    c = _case(nb, 40, 64, 32, 5, 7, seed=nb + 7 * list(BUILD_CFGS).index(cfg), f2=layout == "f2", weighted=weighted)
    _check_build(c, [SIMT, X2, X3, AUTO], f"batch nb={nb} {cfg}", fb, bb, (5, 8) if hint else None)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["3c", "f2"])
def test_build_K128_every_mode_past_grid_y(layout):
    """K = 128 at nb = 65 537: SIMT, TF32X1, X2, X3 and AUTO, weighted, with the grid hint on F2."""
    _dev()
    c = _case(65537, 40, 64, 128, 5, 7, seed=128 + (layout == "f2"), f2=layout == "f2", weighted=True)
    _check_build(c, [SIMT, X1, X2, X3, AUTO], f"batch K=128 {layout}", grid=(5, 8) if layout == "f2" else None)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [0, 16])
@pytest.mark.parametrize("nb", [65536, 131073])
def test_build_small_K_simt_past_grid_y(nb, K):
    _dev()
    c = _case(nb, 40, 64, K, 5, 7, seed=nb + K, weighted=K == 16)
    _check_build(c, [SIMT], f"batch K={K} nb={nb}")


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["3c-f32-w", "f2-bf16-w"])
def test_build_backward_past_grid_y(cfg):
    """lm_build_bwd (exact_sym, with dweight) at nb = 65 537 on the sample against float64 autograd of the oracle build: feature adjoints,
    dD, dB and dweight over the sample, dR, dT, dW per pair."""
    from banet_b200 import ops
    _dev()
    f2, bf = cfg.startswith("f2"), "bf16" in cfg
    nb, N, C, K = 65537, 40, 64, 32
    c = BE._clear_kinks(_case(nb, N, C, K, 5, 7, seed=1300 + f2, f2=f2, weighted=True))
    P = 6 + K
    gen = torch.Generator(device="cuda").manual_seed(5)
    dH = torch.randn(nb, P, P, generator=gen, device="cuda")
    dg = torch.randn(nb, P, generator=gen, device="cuda")
    dr = torch.randn(nb, C, generator=gen, device="cuda")
    got = ops.lm_build_bwd(BE._level(c, bf, bf), c.R, c.T, c.W, dH, dg, dr, True, return_dweight=True)
    idx = _sample(nb)
    ix = torch.tensor(idx, device="cuda")
    names = ("conv1", "conv2", "D", "B", "R", "T", "W", "weight")
    got = {k: t[ix].cpu() for k, t in zip(names, got)}
    s = _cpu_subset(c, idx)
    want = BE._oracle_grads(s, BE._oracle_inputs(s, bf, bf, requires_grad=True), dH[ix].cpu(), dg[ix].cpu(), dr[ix].cpu())
    BE._check_backward(f"batch bwd nb={nb} {cfg}", got, want, 1e-4)


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: keyframe windows
# ------------------------------------------------------------------------------------------------------------------------------------
def _rel_per_pair(x, ref):
    nb = ref.shape[0]
    x, ref = x.double().reshape(nb, -1), ref.double().reshape(nb, -1)
    return float(((x - ref).norm(dim=1) / ref.norm(dim=1).clamp_min(1e-300)).max())


def _rel(x, ref):
    x, ref = x.double(), ref.double()
    return float((x - ref).norm() / ref.norm().clamp_min(1e-300))


def _keyframe_case(nw, nf, N, C, K, seed):
    c = _case(nw * nf, N, C, K, 5, 7, seed=seed, weighted=True)
    first = torch.arange(nw, device="cuda") * nf
    for k in ("p", "D", "B", "conv1", "W"):                          # one keyframe per window: frame 0's tensors in every frame
        setattr(c, k, getattr(c, k)[first].repeat_interleave(nf, 0).contiguous())
    return c, first


@pytest.mark.gpu
@pytest.mark.parametrize("nw,nf", [(65537, 1), (32769, 2)])
def test_keyframe_build_and_backward_past_grid_y(nw, nf):
    """lm_keyframe_build and its backward at nw = 65 537 windows of one frame, and at 32 769 windows of two (more than 65 535 pairs, fewer
    windows): on the whole batch against the window-reduced per-pair build and backward, and on the sample windows against the oracle."""
    from banet_b200 import ops
    _dev()
    N, C, K = 40, 32, 64
    nb, P = nw * nf, 6 + K
    c, first = _keyframe_case(nw, nf, N, C, K, seed=1400 + nf)
    key = ops.KeyframeLevel(c.conv1[first], c.conv2, c.intr, c.p[first], c.D[first], c.B[first], weight=c.weight)
    W = c.W[first].contiguous()
    H, g, rb, nv = ops.lm_keyframe_build(key, c.R, c.T, W)
    Hr, gr, rbr, nvr = _build(c, SIMT)
    assert torch.equal(H, H.transpose(1, 2)) and torch.equal(nv, nvr)
    assert not bool(H.reshape(nw, nf, P, P)[:, 1:, 6:, 6:].any())
    Hw = Hr.reshape(nw, nf, P, P).clone()
    Hw[:, 0, 6:, 6:] = Hr.reshape(nw, nf, P, P)[:, :, 6:, 6:].sum(1)
    Hw[:, 1:, 6:, 6:] = 0
    eb = max(_rel_per_pair(H, Hw.reshape(nb, P, P)), _rel_per_pair(g, gr), _rel_per_pair(rb, rbr))
    del Hr, Hw
    wins = _sample(nw)
    pairs = [w * nf + f for w in wins for f in range(nf)]
    s = _cpu_subset(c, pairs)
    oH, og, orb, onv = BE._oracle(s, BE._oracle_inputs(s))
    n = len(wins)
    oHw = oH.clone().reshape(n, nf, P, P)
    oHw[:, 0, 6:, 6:] = oH.reshape(n, nf, P, P)[:, :, 6:, 6:].sum(1)
    oHw[:, 1:, 6:, 6:] = 0
    ix = torch.tensor(pairs, device="cuda")
    eo = max(_rel_per_pair(H[ix].cpu(), oHw.reshape(-1, P, P)), _rel_per_pair(g[ix].cpu(), og), _rel_per_pair(rb[ix].cpu(), orb))
    assert torch.equal(nv[ix].cpu().double(), onv)
    gen = torch.Generator(device="cuda").manual_seed(nw)
    dH = 1e-2 * torch.randn(nb, P, P, generator=gen, device="cuda")
    dg = 1e-2 * torch.randn(nb, P, generator=gen, device="cuda")
    dr = 1e-2 * torch.randn(nb, C, generator=gen, device="cuda")
    a = ops.lm_keyframe_build_bwd(key, c.R, c.T, W, dH, dg, dr, True, return_dweight=True)
    rH = dH.reshape(nw, nf, P, P).clone()
    rH[:, :, 6:, 6:] = rH[:, :1, 6:, 6:]
    r = ops.lm_build_bwd(BE._level(c), c.R, c.T, c.W, rH.reshape(nb, P, P), dg, dr, True, return_dweight=True)
    del rH
    fsum = lambda t: t.reshape(nw, nf, *t.shape[1:]).sum(1)
    ew = dict(conv1=_rel(a[0], fsum(r[0])), conv2=_rel(a[1], r[1]), D=_rel(a[2], fsum(r[2])), B=_rel(a[3], fsum(r[3])),
              R=_rel_per_pair(a[4], r[4]), T=_rel_per_pair(a[5], r[5]), W=_rel_per_pair(a[6], fsum(r[6])), weight=_rel(a[7], r[7]))
    print(f"BATCH keyframe nw={nw} nf={nf}: build vs per-pair {eb:.2e}, vs oracle {eo:.2e}; backward vs per-pair " +
          " ".join(f"d{k} {v:.1e}" for k, v in ew.items()))
    assert eb < 1e-5 and eo < BE.TOL[SIMT] and max(ew.values()) < 1e-5


@pytest.mark.gpu
def test_keyframe_run_past_grid_y():
    """lm_keyframe_run at nw = 65 537 windows of one frame: every window equals its run in a small batch, bit for bit."""
    from banet_b200 import ops
    _dev()
    nw, nf, N, C, K = 65537, 1, 40, 32, 16
    c, first = _keyframe_case(nw, nf, N, C, K, seed=1500)
    cu = lambda t, lo, hi: t[lo:hi].contiguous()
    def run(lo, hi):
        key = ops.KeyframeLevel(cu(c.conv1, lo, hi), cu(c.conv2, lo, hi), cu(c.intr, lo, hi), cu(c.p, lo, hi), cu(c.D, lo, hi),
                                cu(c.B, lo, hi), weight=cu(c.weight, lo, hi))
        mlp = ops.pack_mlp(mlp_for(C, 2, torch.float32)).cuda()
        return ops.lm_keyframe_run([key], 2, cu(c.R, lo, hi), cu(c.T, lo, hi), cu(c.W, lo, hi), mlp_packed=[mlp])
    full = run(0, nw)
    assert int(full[3].abs().max()) == 0
    assert bool(torch.isfinite(full[0]).all() and torch.isfinite(full[2]).all())
    _assert_pieces_equal(full, run, _pieces(nw), "keyframe run")


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: the damped step and its backward
# ------------------------------------------------------------------------------------------------------------------------------------
def _cap_key(lam):
    """The lambda of test_solve_edges.ERR_CAP_FP32 whose cap covers lam: the largest one at or below it (a smaller lambda, a larger cap)."""
    return max([k for k in (1e-3, 0.1, 10.0) if k <= lam * (1 + 1e-6)] or [1e-3])


@pytest.mark.gpu
@pytest.mark.parametrize("use_mlp", [True, False])
def test_step_and_backward_past_grid_y(use_mlp):
    """lm_step (lambda-MLP, or a lambda per pair) and lm_step_bwd at nb = 65 537, K = 16, C = 64 on systems from a real build: every pair
    against float64 autograd (dmlp: the fixed-order sum over all pairs), the small batches bit for bit; lm_lambda and lm_solve_update(_bwd)
    bit for bit against lm_step's; and the SE(3) update with the reference's batch-scrambled VMatrix against the oracle's."""
    from banet_b200 import ops
    _dev()
    nb, N, C, K = 65537, 40, 64, 16
    P = 6 + K
    c = _case(nb, N, C, K, 5, 7, seed=1600)
    H, g, rb, _ = _build(c, SIMT)
    mlp32 = mlp_for(C, 3, torch.float32)
    mlp = ops.pack_mlp(mlp32).cuda() if use_mlp else None
    lam_in = None if use_mlp else (10.0 ** (4 * torch.rand(nb, generator=torch.Generator().manual_seed(3)) - 3)).cuda()
    cR, cT, cW = [t.cuda().float() for t in SG.cotangents(nb, K, 7)]

    def run(lo, hi):
        sl = lambda t: None if t is None else t[lo:hi].contiguous()
        out = ops.lm_step(sl(H), sl(g), sl(rb), N, mlp, 1000.0, sl(c.R), sl(c.T), sl(c.W), lam=sl(lam_in))
        grads = ops.lm_step_bwd(sl(H), sl(g), sl(rb), N, mlp, out[4], out[3], sl(c.R), sl(c.T), sl(cR), sl(cT), sl(cW), base=1000.0)
        return out, grads

    out, grads = run(0, nb)
    assert int(out[5].abs().max()) == 0
    per_pair = lambda o, gr: list(o) + [t for i, t in enumerate(gr) if i != 3]          # all but dmlp
    _assert_pieces_equal(per_pair(out, grads), lambda lo, hi: per_pair(*run(lo, hi)), _pieces(nb), "lm_step")
    # the entries that share lm_step's code: bit for bit on the whole batch (lm_lambda with the MLP; the solve with lambda given)
    lam = out[4]
    if use_mlp:
        assert torch.equal(ops.lm_lambda(rb, N, mlp, 1000.0), lam)
    su = ops.lm_solve_update(H, g, lam, c.R, c.T, c.W)
    assert int(su[4].abs().max()) == 0
    if not use_mlp:
        for name, x, y in zip(("R", "T", "W", "delta", "status"), (out[0], out[1], out[2], out[3], out[5]), su):
            assert torch.equal(x, y), name
        sb = ops.lm_solve_update_bwd(H, g, lam, out[3], c.R, c.T, cR, cT, cW)
        for name, x, y in zip(("dH", "dg", "dlambda", "dR", "dT", "dW"), (grads[0], grads[1], grads[4], grads[5], grads[6], grads[7]), sb):
            assert torch.equal(x, y), name
    # float64 autograd of every pair at the kernel's lambda (with the float64 MLP's derivative), on the host
    H64, g64, rb64 = H.double().cpu(), g.double().cpu(), rb.double().cpu()
    R64, T64, W64 = c.R.double().cpu(), c.T.double().cpu(), c.W.double().cpu()
    leaf = lambda t: t.clone().requires_grad_()
    Hl, gl, rbl, Rl, Tl, Wl = leaf(H64), leaf(g64), leaf(rb64), leaf(R64), leaf(T64), leaf(W64)
    mlp64 = [(w.double().clone().requires_grad_(), b.double().clone().requires_grad_()) for w, b in mlp32]
    lk = lam.double().cpu()
    if use_mlp:
        l64 = SG.mlp_lambda64(rbl, N, mlp64, 1000.0)
        assert float(((lk - l64.detach()).abs() / l64.detach().abs()).max()) < 1e-4
        lamv = l64 + (lk - l64).detach()
    else:
        lamv = lk.clone().requires_grad_()
    lamv.retain_grad()
    Rn, Tn, Wn = SG.step64(Hl, gl, lamv, Rl, Tl, Wl, True)
    (((Rn * cR.double().cpu()).sum() + (Tn * cT.double().cpu()).sum() + (Wn * cW.double().cpu()).sum())).backward()
    dH, dg, drb, dmlp, dlam, dR, dT, dW = [None if t is None else t.double().cpu() for t in grads]
    variant = SM.step_plan(P, C if use_mlp else 0)
    ndamped = P - 1
    kap = torch.linalg.cond(SG.damped(H64, lk, ndamped))
    t = -(gl.grad * torch.linalg.solve(SG.damped(H64, lk, ndamped), g64.unsqueeze(-1)).squeeze(-1) *
          (torch.diagonal(H64, dim1=-2, dim2=-1) + SG.EPS32))[:, :ndamped]
    cond_sum = t.abs().sum(1) / t.sum(1).abs().clamp_min(1e-300)
    pp = lambda x, ref: (x.reshape(nb, -1) - ref.reshape(nb, -1)).norm(dim=1) / ref.reshape(nb, -1).norm(dim=1).clamp_min(1e-300)
    errs = {"R": pp(out[0].double().cpu(), Rn), "T": pp(out[1].double().cpu(), Tn), "W": pp(out[2].double().cpu(), Wn),
            "dH": pp(dH, Hl.grad), "dg": pp(dg, gl.grad), "dR": pp(dR, Rl.grad), "dT": pp(dT, Tl.grad), "dW": pp(dW, Wl.grad),
            "dlambda": (dlam - lamv.grad).abs() / lamv.grad.abs().clamp_min(1e-300)}
    if use_mlp:
        errs["drbar_sum"] = pp(drb, rbl.grad)
    # per pair, test_step_grad's bounds for the backward (with this pair's kappa and sum condition number); the updated R', T', W': a few
    # fp32 roundings of the update on top of the step's own bound
    fails = []
    for name, e in errs.items():
        if name in ("R", "T", "W"):
            b = torch.tensor([SE._bound(variant, float(kap[i]), None if use_mlp else _cap_key(float(lk[i]))) for i in range(nb)],
                             dtype=torch.float64) + 64 * U32
        else:
            b = torch.tensor([SG._bound(variant, P, float(kap[i]), float(cond_sum[i]), name) for i in range(nb)], dtype=torch.float64)
        worst = int(torch.argmax(e / b))
        print(f"BATCH lm_step mlp={int(use_mlp)} {name}: per-pair max {float(e.max()):.2e}, largest share of its bound "
              f"{float(e[worst] / b[worst]):.2f} (pair {worst})")
        if bool((e > b).any()):
            fails.append((name, worst, float(e[worst]), float(b[worst])))
    if use_mlp:
        off, de = 0, {}
        for i, (w, b) in enumerate(mlp64):
            de[f"filters{i + 1}"] = SE._rel(dmlp[off:off + w.numel()].reshape(w.shape), w.grad); off += w.numel()
            de[f"biases{i + 1}"] = SE._rel(dmlp[off:off + b.numel()], b.grad); off += b.numel()
        print("BATCH lm_step dmlp:", " ".join(f"{k} {v:.1e}" for k, v in de.items()))
        # a sum over 65 537 pairs of contributions each within the lambda path's per-pair bound
        bound = SG._bound(variant, P, 0.0, float(cond_sum.max()), "filters")
        fails += [(k, v) for k, v in de.items() if v > bound]
    assert not fails, fails
    # the reference's VMatrix quirk couples pairs through the flat index b * 9 + q: the whole batch against the oracle on the same delta
    Rs, Ts, Ws, ds, sts = ops.lm_solve_update(H, g, lam, c.R, c.T, c.W, vmatrix_batch_scramble=True)
    assert torch.equal(ds, su[3]) and torch.equal(Rs, su[0]) and torch.equal(Ws, su[2])
    _, Tref = O._update(ds.double().cpu().unsqueeze(-1), R64, T64, O.IterOptions(vmatrix_batch_scramble=True))
    e = (Ts.double().cpu() - Tref).norm(dim=(1, 2)) / Tref.norm(dim=(1, 2))
    print(f"BATCH scrambled VMatrix: per-pair max T' {float(e.max()):.2e}")
    assert float(e.max()) < 1e-5


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: whole solves
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("prec", [SIMT, AUTO])
def test_lm_run_past_grid_y(prec):
    """ops.lm_run (two levels, two iterations, K = 16, the lambda-MLP) at nb = 65 537: every pair equals its run in a small batch, bit for
    bit; autograd.lm_run returns the same bits and its gradients reach R and T of every pair."""
    from banet_b200 import ops, autograd
    _dev()
    nb, C, K = 65537, 64, 16
    # a depth block of K = 16 needs at least 16 valid points: the points start on the map
    cs = [_case(nb, N, C, K, h, w, seed=1700 + N, weighted=True, inside=True) for N, h, w in ((32, 4, 5), (64, 6, 8))]
    mlps = [mlp_for(C, l, torch.float32) for l in (3, 2)]
    packed = [ops.pack_mlp(m).cuda() for m in mlps]

    def run(lo, hi):
        lv = [BE._level(_slice(c, lo, hi)) for c in cs]
        sl = lambda t: t[lo:hi].contiguous()
        return ops.lm_run(lv, 2, sl(cs[0].R), sl(cs[0].T), sl(cs[0].W), mlp_packed=packed, precision=prec)

    full = run(0, nb)
    skipped = int((full[3] != 0).sum())                             # random pairs: a rare one may meet a system that is not definite
    print(f"BATCH lm_run {BE.MODE_NAME[prec]}: {skipped} of {nb} pairs with a skipped step")
    assert skipped <= nb // 10000
    _assert_pieces_equal(full, run, _pieces(nb), f"lm_run {BE.MODE_NAME[prec]}")
    R0, T0 = cs[0].R.clone().requires_grad_(), cs[0].T.clone().requires_grad_()
    mp = [[(w.cuda(), b.cuda()) for w, b in m] for m in mlps]
    Ra, Ta, Wa = autograd.lm_run([BE._level(c) for c in cs], 2, R0, T0, cs[0].W, mlp_params=mp, precision=prec)
    assert torch.equal(Ra, full[0]) and torch.equal(Ta, full[1]) and torch.equal(Wa, full[2])
    (Ra.sum() + Ta.sum()).backward()
    assert bool(torch.isfinite(R0.grad).all() and torch.isfinite(T0.grad).all())
    assert bool((R0.grad.reshape(nb, -1).abs().amax(1) > 0).all())


@pytest.mark.gpu
def test_lm_track_legacy_past_grid_y():
    """lm_track_legacy at nb = 65 537: every pair equals its run in a small batch, bit for bit."""
    from banet_b200 import ops
    _dev()
    nb, C = 65537, 32
    cs = [_case(nb, N, C, 0, h, w, seed=1800 + N) for N, h, w in ((16, 3, 4), (40, 5, 7))]
    packed = [ops.pack_mlp(mlp_for(C, l, torch.float32)).cuda() for l in (3, 2)]

    def run(lo, hi):
        lv = [BE._level(_slice(c, lo, hi)) for c in cs]
        R, T, done, ratio, status = ops.lm_track_legacy(lv, [2, 2], cs[0].R[lo:hi].contiguous(), cs[0].T[lo:hi].contiguous(),
                                                        mlp_packed=packed)
        return R, T, done.t(), ratio, status                        # iterations done [nlevels, nb] -> per pair

    full = run(0, nb)
    _assert_pieces_equal(full, run, _pieces(nb), "lm_track_legacy")


@pytest.mark.gpu
def test_window_batch_run_past_grid_y():
    """lm_window_batch_run at nw = 16 385 windows of 4 frames (65 540 pairs): every window equals its run in a small batch, bit for bit."""
    from banet_b200 import ops
    _dev()
    nw, nf, N, C, K = 16385, 4, 40, 32, 16
    c, first = _keyframe_case(nw, nf, N, C, K, seed=1900)
    packed = [ops.pack_mlp(mlp_for(C, 2, torch.float32)).cuda()]
    W = c.W[first].contiguous()

    def run(lo, hi):
        s = _slice(c, lo * nf, hi * nf)
        return ops.lm_window_batch_run([BE._level(s)], hi - lo, 2, s.R, s.T, W[lo:hi].contiguous(), mlp_packed=packed)

    full = run(0, nw)
    assert int(full[3].abs().max()) == 0
    for lo, hi in _pieces(nw, 256):                                  # the last windows hold pairs 65 535 and 65 536
        small = run(lo, hi)
        for i, (x, y) in enumerate(zip(full, small)):
            rows = slice(lo, hi) if i == 2 else slice(lo * nf, hi * nf)
            assert torch.equal(x[rows], y), ("window batch run", lo, hi, i)


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: pre- and post-step kernels on the whole batch
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("nb", NBS)
def test_depth_compose_past_grid_y(nb):
    """depth_compose and its backward, fp32 and bf16 basis, on the whole batch against float64: dbasis = dout W exactly (one rounding),
    out and dW within a few roundings of the sum of the magnitudes of their terms."""
    from banet_b200 import ops
    _dev()
    M, K = 40, 16
    gen = torch.Generator(device="cuda").manual_seed(nb)
    d0 = 2.0 + torch.rand(nb, M, generator=gen, device="cuda")
    basis = torch.randn(nb, M, K, generator=gen, device="cuda")
    W = 0.1 * torch.randn(nb, K, 1, generator=gen, device="cuda")
    dout = torch.randn(nb, M, generator=gen, device="cuda")
    for bdt in (torch.float32, torch.bfloat16):
        b = basis.to(bdt)
        b64, W64 = b.double(), W.double()
        out = ops.depth_compose(d0, b, W)
        ref = d0.double() + (b64 @ W64).squeeze(-1)
        mag = d0.double().abs() + (b64.abs() @ W64.abs()).squeeze(-1)
        e_out = float(((out.double() - ref).abs() / mag).max())
        db, dW = ops.depth_compose_bwd(dout, b, W)
        assert torch.equal(db, dout.unsqueeze(-1) * W.transpose(1, 2)), (nb, bdt, "dbasis")
        refW = (b64 * dout.double().unsqueeze(-1)).sum(1).unsqueeze(-1)
        magW = (b64.abs() * dout.double().abs().unsqueeze(-1)).sum(1).unsqueeze(-1)
        e_dW = float(((dW.double() - refW).abs() / magW).max())
        print(f"BATCH depth_compose nb={nb} {bdt}: out {e_out:.1e} dW {e_dW:.1e} (relative to the sum of |terms|)")
        assert e_out < 64 * U32 and e_dW < 64 * U32, (nb, bdt, e_out, e_dW)


@pytest.mark.gpu
@pytest.mark.parametrize("nb", [65536, 131073])
def test_sampling_kernels_past_grid_y(nb):
    """resample (fp32, bf16) and resample_bwd, grad_fixed_concat(_bwd) (with swap_halves at even nb), interpolate2d and compute_coordinates
    on the whole batch against float64."""
    from banet_b200 import ops
    _dev()
    h, w, C, N = 5, 7, 8, 16
    gen = torch.Generator(device="cuda").manual_seed(nb + 1)
    data = torch.randn(nb, h, w, C, generator=gen, device="cuda")
    xy = torch.stack([torch.rand(nb, N, generator=gen, device="cuda") * (w + 2) - 1.5,
                      torch.rand(nb, N, generator=gen, device="cuda") * (h + 2) - 1.5], -1).contiguous()
    d64, xy64 = data.double(), xy.double()
    ref = O.resampler(d64, xy64)
    mag = O.resampler(d64.abs(), xy64)
    e = float(((ops.resample(data, xy).double() - ref).abs() / mag.clamp_min(1e-300)).max())
    db16 = data.bfloat16()
    ref16 = O.resampler(db16.double(), xy64)
    e16 = float(((ops.resample(db16, xy).double() - ref16).abs() - 2.0 ** -8 * ref16.abs() - 8 * U32 * mag).max())
    dout = torch.randn(nb, N, C, generator=gen, device="cuda")
    dd = d64.clone().requires_grad_()
    (O.resampler(dd, xy64) * dout.double()).sum().backward()
    da = d64.clone().requires_grad_()
    (O.resampler(da, xy64) * dout.double().abs()).sum().backward()
    e_bwd = float(((ops.resample_bwd(dout, xy, 1.0, h, w).double() - dd.grad).abs() / da.grad.clamp_min(1e-300)).max())
    swap = nb % 2 == 0
    F = data
    cat = ops.grad_fixed_concat(F, swap_halves=swap)
    Fl = d64.clone().requires_grad_()
    rc = torch.cat([Fl, O.grad_fixed(Fl)], -1)
    if swap:
        rc = O._swap_halves(rc)
    e_cat = float((cat.double() - rc.detach()).abs().max() / d64.abs().max())
    dc = torch.randn(nb, h, w, 3 * C, generator=gen, device="cuda")
    (rc * dc.double()).sum().backward()
    e_cat_bwd = float((ops.grad_fixed_concat_bwd(dc, swap_halves=swap).double() - Fl.grad).abs().max() / dc.abs().max())
    out, mask = ops.interpolate2d(data, xy, 1.0, with_mask=True)
    ri, rm = O.interpolate2d(d64, xy64[..., 0], xy64[..., 1])
    mi, _ = O.interpolate2d(d64.abs(), xy64[..., 0], xy64[..., 1])
    assert torch.equal(mask.double(), rm)
    e_int = float(((out.double() - ri).abs() / mi.clamp_min(1e-300)).max())
    intr = torch.cat([100 + 50 * torch.rand(nb, 2, generator=gen, device="cuda"), 50 * torch.rand(nb, 2, generator=gen, device="cuda")], 1)
    pts = 100 * torch.rand(nb, N, 2, generator=gen, device="cuda")
    i64 = intr.double()
    rp = O.compute_coordinates(pts.double(), *[i64[:, k:k + 1] for k in range(4)])
    e_cc = _rel_per_pair(ops.compute_coordinates(pts, intr).transpose(1, 2), rp.transpose(1, 2))
    errs = dict(resample=e, resample_bf16=e16, resample_bwd=e_bwd, grad_fixed_concat=e_cat, grad_fixed_concat_bwd=e_cat_bwd,
                interpolate2d=e_int, compute_coordinates=e_cc)
    print(f"BATCH sampling nb={nb} swap={int(swap)}: " + " ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    assert e < 16 * U32 and e16 <= 0.0 and e_bwd < 64 * U32 and e_int < 16 * U32 and e_cc < 16 * U32
    assert e_cat < 4 * U32 and e_cat_bwd < 16 * U32


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: per-pair offsets past 2^31 elements
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_step_and_build_past_2_31_elements():
    """K = 244 (P = 250): nb = 34 361 pairs take nb P^2 > 2^31 elements, pair 34 359's H block straddles element 2^31 and pair 34 360 lies
    wholly beyond it.  lm_build (whose reduce writes H there), lm_step and lm_step_bwd with lambda given: the straddling pair, its
    neighbours and the last pair against float64, and bit for bit against the same pair run alone."""
    from banet_b200 import ops
    _dev()
    nb, N, C, K = 34361, 40, 16, 244
    P = 6 + K
    b0 = (2 ** 31 - 1) // (P * P)
    assert b0 * P * P < 2 ** 31 < (b0 + 1) * P * P and (nb - 1) * P * P >= 2 ** 31 and nb - 1 == b0 + 1
    need = 3 * nb * P * P * 4 + (4 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    c = _case(nb, N, C, K, 3, 4, seed=2031)
    H, g, rb, _ = _build(c, SIMT)
    picks = [0, b0 - 1, b0, b0 + 1]
    ref = _oracle_build(c, picks)
    BE._check_forward("2^31 build", [t[picks].cpu() for t in (H, g, rb, _)], ref, BE.TOL[SIMT])
    for b in picks:
        alone = _build(_slice(c, b, b + 1), SIMT)
        assert all(torch.equal(x[b:b + 1], y) for x, y in zip((H, g, rb), alone)), ("2^31 build alone", b)
    lam = torch.full((nb,), 0.1, device="cuda")
    cR, cT, cW = [t.cuda().float() for t in SG.cotangents(nb, K, 9)]

    def run(lo, hi):
        sl = lambda t: t[lo:hi].contiguous()
        out = ops.lm_step(sl(H), sl(g), None, 1, None, 1.0, sl(c.R), sl(c.T), sl(c.W), lam=sl(lam))
        grads = ops.lm_step_bwd(sl(H), sl(g), None, 1, None, out[4], out[3], sl(c.R), sl(c.T), sl(cR), sl(cT), sl(cW))
        return [t for t in out] + [t for t in grads if t is not None]

    full = run(0, nb)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert int(full[5][picks].abs().max()) == 0
    for b in picks:
        alone = run(b, b + 1)
        assert all(torch.equal(x[b:b + 1], y) for x, y in zip(full, alone)), ("2^31 step alone", b)
    ix = torch.tensor(picks, device="cuda")
    H64, g64 = H[ix].double().cpu(), g[ix].double().cpu()
    leaf = lambda t: t[ix].double().cpu().clone().requires_grad_()
    Hl, gl, Rl, Tl, Wl = H64.clone().requires_grad_(), g64.clone().requires_grad_(), leaf(c.R), leaf(c.T), leaf(c.W)
    lk = lam[ix].double().cpu()
    Rn, Tn, Wn = SG.step64(Hl, gl, lk, Rl, Tl, Wl, True)
    ((Rn * cR[ix].double().cpu()).sum() + (Tn * cT[ix].double().cpu()).sum() + (Wn * cW[ix].double().cpu()).sum()).backward()
    variant = SM.step_plan(P, 0)
    kap = max(float(torch.linalg.cond(SG.damped(H64[i:i + 1], lk[i:i + 1], P - 1)[0])) for i in range(len(picks)))
    dH, dg = full[6][ix].double().cpu(), full[7][ix].double().cpu()
    errs = dict(W=SE._rel(full[2][ix], Wn.detach()), T=SE._rel(full[1][ix], Tn.detach()), dH=SE._rel(dH, Hl.grad), dg=SE._rel(dg, gl.grad))
    # P kappa u (test_step_grad's fp32 bound) is vacuous at this kappa; hold the backward to ten times the forward's cap at this lambda
    # (test_solve_edges.ERR_CAP_FP32): it solves once more and forms the outer products of u and delta
    bwd_bound = min(SG._bound(variant, P, kap, 1.0, "dH"), 10 * SE._bound(variant, kap, 0.1))
    print(f"BATCH 2^31: variant {variant}, kappa {kap:.1e}, " + " ".join(f"{k} {v:.1e}" for k, v in errs.items()) +
          f"; fwd bound {SE._bound(variant, kap, 0.1):.1e}, bwd bound {bwd_bound:.1e}; peak device memory {peak / 2**30:.2f} GiB")
    assert errs["W"] <= SE._bound(variant, kap, 0.1) and errs["T"] <= SE._bound(variant, kap, 0.1)
    assert errs["dH"] <= bwd_bound and errs["dg"] <= bwd_bound
    del full, H, g, rb, c
    torch.cuda.empty_cache()
    assert peak < 24 * 2 ** 30                                       # 17.7 GiB measured on an H100 80GB HBM3
