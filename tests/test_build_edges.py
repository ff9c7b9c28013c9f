"""The build kernels at the edges of the batch partition and of the image, against the float64 oracle.

Every build kernel runs on a persistent grid whose CTAs each own a contiguous tile range, write one partial slot per pair they touch
(a "span") and leave the reduce to find those slots again by recomputing the partition.  These tests drive the partition where it is
easy to get wrong: many pairs smaller than one tile (every tile a pair change, 8-16 spans per CTA), a grid of exactly total_tiles - 1,
total_tiles and total_tiles + 1 CTAs, and one pair spread over every CTA; and the image where it is easy to get wrong: projections
exactly on the first and last row and column, one representable step outside them, maps of 2 x 2 texels, maps 65600 texels wide or tall,
and per-image offsets next to 2^31 elements.

The CPU part restates the partition in Python (build_edges_model.py) and sweeps it.  The GPU part compares every path against the float64
oracle per pair, since one wrong slot among 2000 pairs disappears in a batch norm; where a pair fits one tile it also asserts bitwise
properties that any stale accumulator or wrong slot would break.  Grid-dependent shapes derive from banet_num_sms()."""
import math

import pytest
import torch

import build_edges_model as M
from helpers import O, rel_fro
import weighted_oracle as WO

# ------------------------------------------------------------------------------------------------------------------------------------
# A. CPU model of the partition
# ------------------------------------------------------------------------------------------------------------------------------------
SWEEP_NB_N = [(1, 1), (1, 40), (1, 64), (1, 65), (1, 132 * 64 * 3 + 17), (1, 264 * 64 + 17), (2, 40), (3, 129), (113, 40), (114, 40),
              (115, 40), (131, 40), (132, 40), (133, 40), (263, 40), (264, 40), (265, 40), (700, 65), (2000, 40), (2000, 1), (3000, 1),
              (57, 4096 + 17), (32, 307200), (250_000, 40), (1_000_000, 1), (40_000, 250), (1, 10_000_000)]
SWEEP_GRIDS = [None, (2, 2), (3, 5), (7, 9), (8, 8), (9, 17), (20, 9), (80, 60), (160, 120), (640, 480)]


@pytest.mark.parametrize("num_sms", [114, 132])
def test_partition_model_simt_and_tensor_core_builds(num_sms):
    """build_plan (per_sm 1 at K = 128, 2 at K = 64 / 32) and build_plan_tc, without and with the dense-grid hint, up to nb * N = 10^7."""
    worst_span, worst_ctas = 0, 0
    for nb, N in SWEEP_NB_N:
        for K in (128, 64):
            for plan in (M.build_plan(nb, N, K, 64, num_sms), M.build_plan_tc(nb, N, K, 64, num_sms)):
                s, c = M.check_partition(plan, nb)
                worst_span, worst_ctas = max(worst_span, s), max(worst_ctas, c)
    for gw_gh in SWEEP_GRIDS[1:]:
        N = gw_gh[0] * gw_gh[1]
        for nb in (1, 2, num_sms - 1, num_sms, num_sms + 1, 2000):
            if nb * N > 2 * 10 ** 7:
                continue
            s, c = M.check_partition(M.build_plan_tc(nb, N, 128, 128, num_sms, gw_gh), nb)
            worst_span, worst_ctas = max(worst_span, s), max(worst_ctas, c)
    assert worst_span >= 16 and worst_ctas == 2 * num_sms         # the sweep reached many spans per CTA and a pair over the whole grid


@pytest.mark.parametrize("num_sms", [114, 132])
def test_partition_model_grid_of_total_tiles_plus_minus_one(num_sms):
    """total_tiles = grid - 1, grid, grid + 1 for each plan's own grid, with tiles_per_pair 1, 2 and 3."""
    for K, per_sm in ((128, 1), (64, 2), (32, 2)):
        G = num_sms * per_sm
        for tpp in (1, 2, 3):
            for total in (G - 1, G, G + 1, 2 * G - 1, 2 * G + 1):
                if total % tpp:
                    continue
                nb, N = total // tpp, 64 * tpp - 13
                plan = M.build_plan(nb, N, K, 64, num_sms)
                assert plan.total_tiles == total
                M.check_partition(plan, nb)
                M.check_partition(M.build_plan_tc(nb, N, K, 64, num_sms), nb)


@pytest.mark.parametrize("num_sms", [114, 132])
def test_partition_model_keyframe_windows(num_sms):
    """keyframe_plan: tiles per window, window slots of nf frames (nw * nf in the hundreds and beyond)."""
    for nw, nf, N in ((1000, 2, 40), (64, 16, 40), (64, 48, 40), (1, 48, 132 * 64 * 2 + 5), (300, 4, 65), (5000, 3, 1), (2, 16, 4096),
                      (num_sms - 1, 2, 40), (num_sms, 2, 40), (num_sms + 1, 2, 40), (2 * num_sms + 1, 2, 40)):
        for K in (128, 64):
            plan = M.keyframe_plan(nw, nf, N, K, 64, num_sms)
            M.check_partition(plan, nw)


def test_partition_model_catches_slot_bugs():
    """The model is not vacuous: one span too few, a reduce that rounds the partition the other way, and an off-by-one span in the
    reduce each fail the check on a shape of the sweep."""
    nb, N = 2000, 40
    plan = M.build_plan_tc(nb, N, 128, 64, 132)
    M.check_partition(plan, nb)
    short = M.build_plan_tc(nb, N, 128, 64, 132)
    short.max_span -= 1
    ceil_part = lambda total, parts, i: (total * i + parts - 1) // parts
    for bad in (lambda: M.check_partition(short, nb),
                lambda: M.check_partition(M.build_plan_tc(nb, 65, 128, 64, 132), nb, partition_reduce=ceil_part),
                lambda: M.check_partition(plan, nb, span_offset=1)):
        with pytest.raises(AssertionError):
            bad()


# ------------------------------------------------------------------------------------------------------------------------------------
# GPU: cases, oracle and comparison
# ------------------------------------------------------------------------------------------------------------------------------------
SIMT, X1, X2, X3, AUTO = 0, 1, 2, 3, -1
# Per pair, relative Frobenius, H and g against the float64 oracle (largest errors measured on an H100 80GB HBM3 at 700 W in brackets).
# A pair of 40 points has no averaging to hide behind, so these are looser than the whole-batch bounds of the other suites
# (SIMT 2e-5, X3 2e-6, X2 1e-4, X1 5e-4):
# - H, g and the pose block are sums of a few dozen terms of both signs.  The fp32 SIMT build itself reaches 1.2e-5 on one pair's g and
#   pose block, and X3 (fp32-grade) 1.2e-5 on H at N = 1, so both share an fp32 bound of 5e-5 (measured 2.0e-5).
# - X2 rounds every R operand to nearest once.  Over one pair these errors do not average out: 2.0e-4 measured, bound 4e-4.
# - X1 adds the stochastic rounding of the basis: 3.3e-4 measured, bound 5e-4 (unchanged).
TOL = {SIMT: 5e-5, X1: 5e-4, X2: 4e-4, X3: 5e-5}
TOL_POSE = 5e-5                                       # pose block of H and g (never through the tensor cores): fp32 bound as above
TOL_RBAR = 2e-5                                       # rbar_sum (measured 1.1e-6)
MODE_NAME = {SIMT: "simt", X1: "x1", X2: "x2", X3: "x3", AUTO: "auto"}


def _modes(K):
    return [SIMT, X1, X2, X3, AUTO] if K == 128 else [SIMT, X2, X3, AUTO]


def _auto(K, N):
    return (X3 if N < 65536 else X1) if K == 128 else X2


def _rotation(nb, g, scale):
    w = torch.randn(nb, 3, generator=g, dtype=torch.float64) * scale
    S = torch.zeros(nb, 3, 3, dtype=torch.float64)
    S[:, 0, 1], S[:, 0, 2], S[:, 1, 2] = -w[:, 2], w[:, 1], -w[:, 0]
    return torch.linalg.matrix_exp(S - S.transpose(1, 2)).float()


class Case:
    """One level on the CPU in fp32: random maps and points whose projections land on the map or up to one texel outside it."""

    def __init__(self, nb, N, C, K, h, w, seed, f2, weighted=False):
        g = torch.Generator().manual_seed(seed)
        self.nb, self.N, self.C, self.K, self.h, self.w, self.f2 = nb, N, C, K, h, w, f2
        fx = fy = float(max(h, w))
        ox, oy = (w - 1) / 2.0, (h - 1) / 2.0
        u = torch.rand(nb, N, generator=g) * (w + 1) - 1.0
        v = torch.rand(nb, N, generator=g) * (h + 1) - 1.0
        self.p = torch.stack([(u - ox) / fx, (v - oy) / fy, torch.ones(nb, N)], 1).contiguous()
        self.intr = torch.tensor([fx, fy, ox, oy]).repeat(nb, 1)
        self.D = 2.0 + torch.rand(nb, N, 1, generator=g)
        self.B = 0.5 * torch.randn(nb, N, K, generator=g)
        self.W = 0.02 * torch.randn(nb, K, 1, generator=g)
        self.R = _rotation(nb, g, 0.01)
        self.T = 0.02 * torch.randn(nb, 3, 1, generator=g)
        self.conv1 = torch.randn(nb, N, C, generator=g)
        self.conv2 = torch.randn(nb, h, w, C if f2 else 3 * C, generator=g)
        self.weight = None
        if weighted:
            self.weight = 2.0 * torch.rand(nb, N, 1, generator=g)
            self.weight[torch.rand(nb, N, 1, generator=g) < 0.1] = 0.0

    def subset(self, idx):
        """The same level restricted to the pairs idx (in that order)."""
        c = Case.__new__(Case)
        c.__dict__.update(self.__dict__)
        for k in ("p", "intr", "D", "B", "W", "R", "T", "conv1", "conv2", "weight"):
            t = getattr(self, k)
            setattr(c, k, None if t is None else t[idx].contiguous())
        c.nb = len(idx)
        return c


def _feat(t, bf16):
    return t.bfloat16() if bf16 else t


def _level(c, feat_bf16=False, basis_bf16=False, grid=None):
    from banet_b200 import ops
    cu = lambda t: None if t is None else t.cuda().contiguous()
    return ops.Level(cu(_feat(c.conv1, feat_bf16)), cu(_feat(c.conv2, feat_bf16)), cu(c.intr), cu(c.p), cu(c.D), cu(_feat(c.B, basis_bf16)),
                     grid=grid, weight=cu(c.weight))


def _build(c, prec, feat_bf16=False, basis_bf16=False, grid=None):
    from banet_b200 import ops
    return [t.cpu() for t in ops.lm_build(_level(c, feat_bf16, basis_bf16, grid), c.R.cuda(), c.T.cuda(), c.W.cuda(), prec)]


def _oracle_inputs(c, feat_bf16=False, basis_bf16=False, requires_grad=False):
    f64 = torch.float64
    wid = lambda t, bf: _feat(t, bf).to(f64)
    a = dict(conv1=wid(c.conv1, feat_bf16), conv2=wid(c.conv2, feat_bf16), p=c.p.double(), D=c.D.double(), B=wid(c.B, basis_bf16),
             R=c.R.double(), T=c.T.double(), W=c.W.double(), weight=None if c.weight is None else c.weight.double())
    if requires_grad:
        for k, t in a.items():
            if t is not None:
                t.requires_grad_()
    return a


def _oracle(c, a):
    """H [nb,P,P], g [nb,P], rbar_sum [nb,C], nvalid [nb] in float64 (3C maps from F2 by the REFLECT stencil)."""
    conv2 = torch.cat([a["conv2"], O.grad_fixed(a["conv2"])], -1) if c.f2 else a["conv2"]
    fx, fy, ox, oy = [c.intr[:, i:i + 1].double().expand(c.nb, c.N) for i in range(4)]
    if a["weight"] is None:
        H, g, rbar, nv = O.normal_equations_structured_chunked(a["conv1"], conv2, fx, fy, ox, oy, a["p"], a["D"], a["B"], a["R"], a["T"], a["W"])
    else:
        H, g, rbar, nv = WO.normal_equations(a["conv1"], conv2, fx, fy, ox, oy, a["p"], a["D"], a["B"], a["R"], a["T"], a["W"], a["weight"])
    return H, g.reshape(c.nb, -1), rbar.reshape(c.nb, -1) * c.N, nv


def _per_pair(x, ref):
    nb = ref.shape[0]
    x, ref = x.double().reshape(nb, -1), ref.detach().double().reshape(nb, -1)
    return (x - ref).norm(dim=1) / ref.norm(dim=1).clamp_min(1e-300)


def _check_forward(label, out, ref, tol):
    """Per-pair errors of one build against the oracle; returns the largest ones (printed for the record)."""
    H, g, rb, nv = out
    rH, rg, rrb, rnv = ref
    assert torch.equal(nv.double(), rnv.double()), (label, "nvalid")
    assert torch.equal(H, H.transpose(1, 2)), (label, "H not exactly symmetric")
    e = dict(H=float(_per_pair(H, rH).max()), g=float(_per_pair(g, rg).max()),
             pose=float(max(_per_pair(H[:, :6, :6], rH[:, :6, :6]).max(), _per_pair(g[:, :6], rg[:, :6]).max())),
             rbar=float(_per_pair(rb, rrb).max()))
    print(f"EDGE {label}: per-pair max H {e['H']:.2e} g {e['g']:.2e} pose {e['pose']:.2e} rbar {e['rbar']:.2e} (tol {tol:.0e})")
    assert e["H"] < tol and e["g"] < tol, (label, e)
    assert e["pose"] < TOL_POSE and e["rbar"] < TOL_RBAR, (label, e)
    return e


def _num_sms():
    from banet_b200 import _lib
    _lib.require_device()
    return int(_lib.load().banet_num_sms())


def _bitwise_pair_properties(c, prec, label, **kw):
    """tiles_per_pair == 1: the build of a permuted batch is the permuted build, and a pair built alone is that pair of the batch, bit
    for bit (not in TF32X1, whose dither seed includes the pair index)."""
    full = _build(c, prec, **kw)
    gen = torch.Generator().manual_seed(c.nb)
    perm = torch.randperm(c.nb, generator=gen)
    permuted = _build(c.subset(perm), prec, **kw)
    for x, y in zip(full, permuted):
        assert torch.equal(x[perm], y), (label, "permuted batch")
    sms = _num_sms()
    picks = sorted({0, c.nb - 1} | {min(c.nb - 1, M.part_begin(c.nb, sms, i)) for i in range(0, sms, max(1, sms // 8))} |
                   {int(i) for i in torch.randint(0, c.nb, (6,), generator=gen)})
    for b in picks:
        alone = _build(c.subset([b]), prec, **kw)
        for x, y in zip(full, alone):
            assert torch.equal(x[b:b + 1], y), (label, "pair built alone", b)


# ------------------------------------------------------------------------------------------------------------------------------------
# B. forward builds on partition edges
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("hint", [False, True])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("feat,basis", [("f32", "f32"), ("bf16", "f32"), ("f32", "bf16"), ("bf16", "bf16")])
@pytest.mark.parametrize("layout", ["3c", "f2"])
def test_many_subtile_pairs_match_the_oracle_per_pair(layout, feat, basis, weighted, hint):
    """nb = 2000 pairs of N = 40 (a 5 x 8 grid under the hint): every tile is a pair change and each CTA walks 8-16 spans."""
    fb, bb = feat == "bf16", basis == "bf16"
    c = Case(2000, 40, 64, 128, 6, 9, seed=1000 + 8 * fb + 4 * bb + 2 * weighted + hint + 16 * (layout == "f2"), f2=layout == "f2", weighted=weighted)
    grid = (5, 8) if hint else None
    ref = _oracle(c, _oracle_inputs(c, fb, bb))
    for prec in _modes(128):
        lab = f"subtile {layout} feat={feat} basis={basis} w={int(weighted)} hint={int(hint)} {MODE_NAME[prec]}"
        _check_forward(lab, _build(c, prec, fb, bb, grid), ref, TOL[_auto(128, c.N) if prec == AUTO else prec])
        if prec != X1:
            _bitwise_pair_properties(c, prec, lab, feat_bf16=fb, basis_bf16=bb, grid=grid)


@pytest.mark.gpu
@pytest.mark.parametrize("hint", [False, True])
@pytest.mark.parametrize("layout", ["3c", "f2"])
@pytest.mark.parametrize("K", [64, 32])
def test_many_subtile_pairs_small_K(K, layout, hint):
    c = Case(2000, 40, 64, K, 6, 9, seed=1100 + K + hint + 2 * (layout == "f2"), f2=layout == "f2", weighted=hint)
    grid = (5, 8) if hint else None
    ref = _oracle(c, _oracle_inputs(c))
    for prec in _modes(K):
        lab = f"subtile K={K} {layout} hint={int(hint)} {MODE_NAME[prec]}"
        _check_forward(lab, _build(c, prec, grid=grid), ref, TOL[_auto(K, c.N) if prec == AUTO else prec])
        _bitwise_pair_properties(c, prec, lab, grid=grid)


def _shape(kind, K, prec, sms):
    """(nb, N, grid) of a partition-edge shape for the path (K, prec): its own grid G is sms CTAs, or 2 sms for SIMT below K = 128."""
    G = sms * (2 if prec == SIMT and K < 128 else 1)
    if kind.startswith("grid"):
        return G + {"grid-1": -1, "grid": 0, "grid+1": 1}[kind], 40, None
    if kind == "spread":
        return 1, G * 64 * 3 + 17, None
    if kind == "n1":
        return 3000, 1, None
    if kind == "n65":
        return 700, 65, None
    gw, gh = {"g2x2": (2, 2), "g3x5": (3, 5), "g7x9": (7, 9), "g13x11": (13, 11), "g20x9": (20, 9)}[kind]
    return 300, gw * gh, (gw, gh)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["3c", "f2"])
@pytest.mark.parametrize("K", [128, 64])
@pytest.mark.parametrize("kind", ["grid-1", "grid", "grid+1", "spread", "n1", "n65", "g2x2", "g3x5", "g7x9", "g13x11", "g20x9"])
def test_partition_edge_shapes_match_the_oracle_per_pair(kind, K, layout):
    """total_tiles = G - 1, G, G + 1 for each path's own grid G; one pair over every CTA; N = 1; N = 65 (the second tile holds one point);
    dense grids smaller than one 8 x 8 tile and grids that are not multiples of 8."""
    sms = _num_sms()
    done = {}
    for prec in _modes(K):
        nb, N, grid = _shape(kind, K, prec, sms)
        if (nb, N) not in done:
            c = Case(nb, N, 64, K, 7, 10, seed=nb * 7 + N + K, f2=layout == "f2", weighted=kind in ("grid", "n65", "g3x5"))
            done[(nb, N)] = (c, _oracle(c, _oracle_inputs(c)))
        c, ref = done[(nb, N)]
        lab = f"shape {kind} K={K} {layout} nb={nb} N={N} {MODE_NAME[prec]}"
        _check_forward(lab, _build(c, prec, grid=grid), ref, TOL[_auto(K, N) if prec == AUTO else prec])


# ------------------------------------------------------------------------------------------------------------------------------------
# C. backward on the same shapes
# ------------------------------------------------------------------------------------------------------------------------------------
def _oracle_grads(c, a, dH, dg, dr):
    H, g, rb, _ = _oracle(c, a)
    loss = (dH.double() * H).sum() + (dg.double() * g).sum() + (dr.double() * rb).sum()
    names = [k for k in ("conv1", "conv2", "D", "B", "R", "T", "W", "weight") if a[k] is not None]
    grads = torch.autograd.grad(loss, [a[k] for k in names])
    return dict(zip(names, grads))


def _clear_kinks(c, margin=1e-3):
    """Nudge points whose float64 projection lies within `margin` texels of an integer row or column: there the bilinear sample has a
    kink, so its derivative is one-sided and the fp32 and fp64 projections may take different sides."""
    for _ in range(4):
        fx, fy, ox, oy = [c.intr[:, i:i + 1].double().expand(c.nb, c.N) for i in range(4)]
        _, _, _, _, px, py = O._warp(c.p.double(), c.D.double() + c.B.double() @ c.W.double(), c.R.double(), c.T.double(), fx, fy, ox, oy)
        near = lambda q: (q - q.round()).abs() < margin
        bad = near(px) | near(py)
        if not bool(bad.any()):
            return c
        c.p[:, 0][bad] += (4 * margin / fx[bad]).float()
        c.p[:, 1][bad] += (4 * margin / fy[bad]).float()
    raise AssertionError("could not move the points off the texel lines")


def _bwd(c, dH, dg, dr, feat_bf16=False, basis_bf16=False):
    from banet_b200 import ops
    out = ops.lm_build_bwd(_level(c, feat_bf16, basis_bf16), c.R.cuda(), c.T.cuda(), c.W.cuda(), dH.cuda(), dg.cuda(), dr.cuda(), True,
                           return_dweight=True)
    return dict(zip(("conv1", "conv2", "D", "B", "R", "T", "W", "weight"), [t.cpu() for t in out]))


def _check_backward(label, got, want, tol):
    e = {}
    for k, ref in want.items():
        e[k] = float(_per_pair(got[k], ref).max()) if k in ("R", "T", "W") else rel_fro(got[k], ref)
    print(f"EDGE {label}: " + " ".join(f"d{k} {v:.2e}" for k, v in e.items()) + f" (tol {tol:.0e}; dR, dT, dW per pair)")
    assert max(e.values()) < tol, (label, e)
    return e


BWD_CASES = [("3c", "f32", "f32", False), ("3c", "f32", "f32", True), ("f2", "f32", "f32", False), ("f2", "f32", "f32", True),
             ("3c", "bf16", "bf16", True), ("f2", "bf16", "f32", False), ("f2", "f32", "bf16", True)]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["subtile", "spread"])
@pytest.mark.parametrize("layout,feat,basis,weighted", BWD_CASES)
def test_backward_on_partition_edges_matches_oracle_autograd(layout, feat, basis, weighted, shape):
    """lm_build_bwd (exact_sym) against float64 autograd of the oracle build with loss <dH,H> + <dg,g> + <dr,rbar_sum>: nb = 2000 x
    N = 40, and one pair spread over the whole backward grid.  bf16 inputs: also against the fp32 backward on the widened inputs."""
    fb, bb = feat == "bf16", basis == "bf16"
    sms = _num_sms()
    nb, N = (2000, 40) if shape == "subtile" else (1, 2 * sms * 64 + 17)
    K, C = 32, 64
    c = _clear_kinks(Case(nb, N, C, K, 6, 9, seed=1300 + nb + 2 * fb + bb + 4 * weighted, f2=layout == "f2", weighted=weighted))
    g = torch.Generator().manual_seed(nb + 5)
    P = 6 + K
    dH, dg, dr = torch.randn(nb, P, P, generator=g), torch.randn(nb, P, generator=g), torch.randn(nb, C, generator=g)
    want = _oracle_grads(c, _oracle_inputs(c, fb, bb, requires_grad=True), dH, dg, dr)
    got = _bwd(c, dH, dg, dr, fb, bb)
    if not weighted:
        want["weight"] = _oracle_grads(c, dict(_oracle_inputs(c, fb, bb, requires_grad=True),
                                               weight=torch.ones(nb, N, 1, dtype=torch.float64, requires_grad=True)), dH, dg, dr)["weight"]
    _check_backward(f"bwd {shape} {layout} feat={feat} basis={basis} w={int(weighted)}", got, want, 1e-4)
    if fb or bb:
        cw = c.subset(list(range(nb)))
        cw.conv1, cw.conv2, cw.B = _feat(c.conv1, fb).float(), _feat(c.conv2, fb).float(), _feat(c.B, bb).float()
        ref32 = _bwd(cw, dH, dg, dr)
        for k in got:
            assert rel_fro(got[k], ref32[k]) < 1e-5, (k, "bf16 backward vs fp32 backward on the widened inputs")


# ------------------------------------------------------------------------------------------------------------------------------------
# D. keyframe forms with many windows of sub-tile N
# ------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("nw,nf", [(1000, 2), (64, 16)])
def test_keyframe_many_subtile_windows(nw, nf, weighted):
    """lm_keyframe_build / _bwd against the window-reduced per-pair build and backward, and the build against the oracle."""
    from banet_b200 import ops
    N, C, K = 40, 32, 64
    nb, P = nw * nf, 6 + K
    c = Case(nb, N, C, K, 6, 9, seed=1400 + nw + weighted, f2=False, weighted=weighted)
    first = torch.arange(nw) * nf
    for k in ("p", "D", "B", "conv1", "W"):                          # one keyframe per window: frame 0's tensors in every frame
        setattr(c, k, getattr(c, k)[first].repeat_interleave(nf, 0).contiguous())
    cu = lambda t: None if t is None else t.cuda().contiguous()
    key = ops.KeyframeLevel(cu(c.conv1[first]), cu(c.conv2), cu(c.intr), cu(c.p[first]), cu(c.D[first]), cu(c.B[first]), weight=cu(c.weight))
    R, T, W = c.R.cuda(), c.T.cuda(), c.W[first].cuda()
    H, g, rb, nv = [t.cpu() for t in ops.lm_keyframe_build(key, R, T, W)]
    Hr, gr, rbr, nvr = _build(c, SIMT)
    assert torch.equal(H, H.transpose(1, 2)) and torch.equal(nv, nvr)
    dd, ddr = H.reshape(nw, nf, P, P)[:, :, 6:, 6:], Hr.reshape(nw, nf, P, P)[:, :, 6:, 6:]
    assert not bool(dd[:, 1:].any())
    Hw = Hr.clone().reshape(nw, nf, P, P)
    Hw[:, 0, 6:, 6:] = ddr.sum(1)
    Hw[:, 1:, 6:, 6:] = 0
    eb = max(float(_per_pair(H, Hw.reshape(nb, P, P)).max()), float(_per_pair(g, gr).max()), float(_per_pair(rb, rbr).max()))
    oH, og, orb, onv = _oracle(c, _oracle_inputs(c))
    oHw = oH.clone().reshape(nw, nf, P, P)
    oHw[:, 0, 6:, 6:] = oH.reshape(nw, nf, P, P)[:, :, 6:, 6:].sum(1)
    oHw[:, 1:, 6:, 6:] = 0
    eo = max(float(_per_pair(H, oHw.reshape(nb, P, P)).max()), float(_per_pair(g, og).max()), float(_per_pair(rb, orb).max()))
    assert torch.equal(nv.double(), onv)
    gen = torch.Generator().manual_seed(nw)
    dH, dg, dr = 1e-2 * torch.randn(nb, P, P, generator=gen), 1e-2 * torch.randn(nb, P, generator=gen), 1e-2 * torch.randn(nb, C, generator=gen)
    a = [t.cpu() for t in ops.lm_keyframe_build_bwd(key, R, T, W, dH.cuda(), dg.cuda(), dr.cuda(), True, return_dweight=True)]
    rH = dH.clone().reshape(nw, nf, P, P)
    rH[:, :, 6:, 6:] = rH[:, :1, 6:, 6:]
    r = _bwd(c, rH.reshape(nb, P, P), dg, dr)
    fsum = lambda t: t.reshape(nw, nf, *t.shape[1:]).sum(1)
    ew = dict(conv1=rel_fro(a[0], fsum(r["conv1"])), conv2=rel_fro(a[1], r["conv2"]), D=rel_fro(a[2], fsum(r["D"])), B=rel_fro(a[3], fsum(r["B"])),
              R=float(_per_pair(a[4], r["R"]).max()), T=float(_per_pair(a[5], r["T"]).max()), W=float(_per_pair(a[6], fsum(r["W"])).max()),
              weight=rel_fro(a[7], r["weight"]))
    print(f"EDGE keyframe nw={nw} nf={nf} w={int(weighted)}: build vs per-pair {eb:.2e}, vs oracle {eo:.2e}; backward vs per-pair " +
          " ".join(f"d{k} {v:.1e}" for k, v in ew.items()))
    assert eb < 1e-5 and eo < TOL[SIMT] and max(ew.values()) < 1e-5


# ------------------------------------------------------------------------------------------------------------------------------------
# E. image edges with exact projections
# ------------------------------------------------------------------------------------------------------------------------------------
STEP = 2.0 ** -7            # one step outside the map that stays exact in fp32 through (u - t) + t for every map here (w, h < 2^17)
SHIFT = 0.25                # T = (t, t, 0) in camera units: x = ((u / f - t) + t) / 1 = u / f exactly (y alike); depth Jacobian -f t (1, 1)


def _edge_case(h, w, C=64, K=128, seed=0, f2=True):
    """Points on u in {0, w-1}, v in {0, h-1}, the corners, one STEP outside each edge, interior fractions, two Z < 0 points that are in
    bounds, and for a wide map the columns around 65536; padded to a multiple of 8 points.  R = I, D = 1, W = 0, o = 0, fx = fy = f the
    power of two at or above the map's size (camera coordinates of order one, as in a real camera), T = (t, t, 0) and
    p = (Z u / f - t, Z v / f - t, Z): the projection is exactly (u, v) in fp32 and in fp64."""
    us = [0.0, w - 1.0, -STEP, w - 1.0 + STEP, 0.5 * (w - 1), min(0.25, w - 1.0), w - 1.25 if w > 2 else 0.75]
    vs = [0.0, h - 1.0, -STEP, h - 1.0 + STEP, 0.5 * (h - 1), min(0.75, h - 1.0)]
    if w > 65536:
        us += [65534.5, 65535.0, 65535.75, 65536.0, 65536.25, 65537.0, w - 2.5]
    if h > 65536:
        vs += [65535.0, 65536.5, h - 2.25]
    pts = [(u, v, 1.0) for u in us for v in vs] + [(0.5 * (w - 1), 0.25 * (h - 1), -1.0), (w - 1.0, h - 1.0, -1.0)]
    while len(pts) % 8:
        pts.append((0.25 * (w - 1), 0.5 * (h - 1), 1.0))
    u = torch.tensor([q[0] for q in pts]); v = torch.tensor([q[1] for q in pts]); z = torch.tensor([q[2] for q in pts])
    N, nb = u.numel(), 1 if max(h, w) > 1000 else 2
    c = Case(nb, N, C, K, 2, 2, seed=seed, f2=f2)
    g = torch.Generator().manual_seed(seed + 1)
    c.h, c.w = h, w
    c.conv2 = torch.randn(nb, h, w, C if f2 else 3 * C, generator=g)
    # Z = z: X = px + t must be z * u / f so that f * X / Z = u; every step is exact in fp32 for these u (y alike)
    f = _edge_focal(h, w)
    px, py = z * u / f - SHIFT, z * v / f - SHIFT
    c.p = torch.stack([px, py, z]).unsqueeze(0).repeat(nb, 1, 1).contiguous()
    assert torch.equal(f * ((px + SHIFT) / z), u) and torch.equal(f * ((py + SHIFT) / z), v)
    c.intr = torch.tensor([f, f, 0.0, 0.0]).repeat(nb, 1)
    c.D = torch.ones(nb, N, 1)
    c.W = torch.zeros(nb, K, 1)
    c.R = torch.eye(3).repeat(nb, 1, 1)
    c.T = torch.tensor([SHIFT, SHIFT, 0.0]).reshape(1, 3, 1).repeat(nb, 1, 1)
    return c, (8, N // 8)


def _edge_focal(h, w):
    return 2.0 ** math.ceil(math.log2(max(h, w)))


EDGE_MAPS = {"2x2": (2, 2), "2x3": (2, 3), "3x2": (3, 2), "16x20": (16, 20), "wide": (2, 65600), "tall": (65600, 2)}


@pytest.mark.gpu
@pytest.mark.parametrize("feat", ["f32", "bf16"])
@pytest.mark.parametrize("layout", ["3c", "f2"])
@pytest.mark.parametrize("shape", list(EDGE_MAPS))
def test_image_edges_forward_every_path(shape, layout, feat):
    """Every forward path (SIMT, TF32X1/X2/X3, AUTO, with and without the grid hint) with projections exactly on the map's first and
    last rows and columns.  An F2 map 65536 texels or wider stays off the tensor cores' packed 16-bit tap
    columns: AUTO resolves to SIMT and an explicit TF32 mode is refused with a message that names the width."""
    from banet_b200 import _lib
    h, w = EDGE_MAPS[shape]
    fb = feat == "bf16"
    c, grid = _edge_case(h, w, f2=layout == "f2", seed=h + w)
    ref = _oracle(c, _oracle_inputs(c, fb, False))
    assert float(ref[3].min()) < c.N and float(ref[3].min()) > 0          # some points out, some in
    wide_f2 = layout == "f2" and w >= 65536
    for prec in _modes(128):
        for hint in (None, grid):
            lab = f"edges {shape} {layout} feat={feat} {MODE_NAME[prec]} hint={int(hint is not None)}"
            tol = TOL[SIMT] if wide_f2 and prec == AUTO else TOL[_auto(128, c.N) if prec == AUTO else prec]
            try:
                out = _build(c, prec, fb, grid=hint)
            except _lib.BanetError as e:
                assert wide_f2 and prec in (X1, X2, X3) and "w < 65536" in str(e) and "w=65600" in str(e), (lab, str(e))
                print(f"EDGE {lab}: refused (F2 width)")
                continue
            _check_forward(lab, out, ref, tol)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["3c", "f2"])
@pytest.mark.parametrize("shape", list(EDGE_MAPS))
def test_image_edges_backward(shape, layout):
    """lm_build_bwd with the same edge points against oracle autograd.  The feature-map adjoints and dweight are compared with every point;
    the gradients through the projection without the points exactly on u = w-1 or v = h-1, where the kernel's clamped tap and the
    oracle's zero tap give different one-sided derivatives of the bilinear sample."""
    h, w = EDGE_MAPS[shape]
    K, C = 32, 64
    c, _ = _edge_case(h, w, C=C, K=K, f2=layout == "f2", seed=3 * h + w)
    c.W = 0.0 * c.W
    P = 6 + K
    g = torch.Generator().manual_seed(7)
    dH, dg, dr = torch.randn(c.nb, P, P, generator=g), torch.randn(c.nb, P, generator=g), torch.randn(c.nb, C, generator=g)
    a = _oracle_inputs(c, requires_grad=True)
    a["weight"] = torch.ones(c.nb, c.N, 1, dtype=torch.float64, requires_grad=True)
    want = _oracle_grads(c, a, dH, dg, dr)
    got = _bwd(c, dH, dg, dr)
    _check_backward(f"bwd edges {shape} {layout} features", got, {k: want[k] for k in ("conv1", "conv2", "weight")}, 1e-4)
    f = _edge_focal(h, w)
    u = f * ((c.p[0, 0] + SHIFT) / c.p[0, 2])
    v = f * ((c.p[0, 1] + SHIFT) / c.p[0, 2])
    keep = torch.nonzero((u != w - 1) & (v != h - 1)).flatten().tolist()
    ci = c.subset(list(range(c.nb)))
    ci.p, ci.conv1, ci.D, ci.B, ci.N = c.p[:, :, keep].contiguous(), c.conv1[:, keep].contiguous(), c.D[:, keep].contiguous(), c.B[:, keep].contiguous(), len(keep)
    a = _oracle_inputs(ci, requires_grad=True)
    want = _oracle_grads(ci, a, dH, dg, dr)
    got = _bwd(ci, dH, dg, dr)
    _check_backward(f"bwd edges {shape} {layout} geometry", got, {k: want[k] for k in ("D", "B", "R", "T", "W")}, 1e-4)


# ------------------------------------------------------------------------------------------------------------------------------------
# F. per-image offsets near 2^31 elements
# ------------------------------------------------------------------------------------------------------------------------------------
def _big_map_case(h, w, nb, C=128, K=128, seed=5):
    """Points in the bottom-right 64 x 64 block, two or more texels from its inner edges, at multiples of 1/64; the map is zero outside the
    block.  Returns the full-map level (bf16 features) and the same level cropped to the block for the oracle, whose principal point
    is moved by the block's origin so that the projections land in the block at the same camera coordinates."""
    g = torch.Generator().manual_seed(seed)
    N = 64
    gu = torch.randint(2 * 64, 62 * 64 + 1, (N,), generator=g).float() / 64.0        # block coordinates in [2, 62], multiples of 1/64
    gv = torch.randint(2 * 64, 62 * 64 + 1, (N,), generator=g).float() / 64.0
    gu[:4] = torch.tensor([63.0, 62.5, 63.0, 2.0]); gv[:4] = torch.tensor([63.0, 63.0, 2.0, 63.0])   # on the true last column / row
    crop = Case(nb, N, C, K, 64, 64, seed=seed, f2=True)
    crop.conv2 = torch.randn(nb, 64, 64, C, generator=g).bfloat16().float()
    crop.conv1 = crop.conv1.bfloat16().float()
    crop.intr = torch.tensor([1.0, 1.0, 0.0, 0.0]).repeat(nb, 1)
    crop.R = torch.eye(3).repeat(nb, 1, 1)
    crop.T = torch.tensor([SHIFT, SHIFT, 0.0]).reshape(1, 3, 1).repeat(nb, 1, 1)
    crop.D = torch.ones(nb, N, 1)
    crop.W = torch.zeros(nb, K, 1)
    crop.p = torch.stack([gu - SHIFT, gv - SHIFT, torch.ones(N)]).unsqueeze(0).repeat(nb, 1, 1).contiguous()
    crop.p[:, 0] += float(w - 64)
    crop.p[:, 1] += float(h - 64)
    full = crop.subset(list(range(nb)))
    full.h, full.w = h, w
    # the oracle sees the same points (so the same Jacobians) on the block: its principal point moves by the block's origin instead
    crop.intr = torch.tensor([1.0, 1.0, -float(w - 64), -float(h - 64)]).repeat(nb, 1)
    return full, crop


def _big_level(full, crop, dev_map):
    from banet_b200 import ops
    return ops.Level(crop.conv1.bfloat16().cuda(), dev_map, full.intr.cuda(), full.p.cuda(), full.D.cuda(), full.B.cuda())


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["below", "above"])
def test_offsets_near_2_31(which):
    """below: an F2 map of 4095 x 4096 x 128 bf16 (h w C just below 2^31), nb = 2, so the tensor-core path runs with its largest 32-bit
    per-image offsets and pair 1 starts beyond 2^31 elements.  above: 4097 x 4096 x 128, where AUTO falls back to SIMT and the TF32 modes
    are refused.  Both against the oracle on the cropped bottom-right block, with the projections moved into it by the principal point."""
    from banet_b200 import ops, _lib
    _lib.require_device()
    h, w, C, nb = (4095, 4096, 128, 2) if which == "below" else (4097, 4096, 128, 1)
    assert (h * w * C < 2 ** 31) == (which == "below")
    need = nb * h * w * C * 2 + (1 << 28)
    free, _ = torch.cuda.mem_get_info()
    if free < need + (1 << 30):
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")
    full, crop = _big_map_case(h, w, nb)
    torch.cuda.synchronize(); torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    dev_map = torch.zeros(nb, h, w, C, dtype=torch.bfloat16, device="cuda")
    dev_map[:, h - 64:, w - 64:, :] = crop.conv2.bfloat16().cuda()
    lv = _big_level(full, crop, dev_map)
    ref = _oracle(crop, _oracle_inputs(crop))
    assert float(ref[3].min()) == crop.N
    R, T, W = full.R.cuda(), full.T.cuda(), full.W.cuda()
    for prec in (SIMT, X1, X2, X3, AUTO):
        lab = f"offsets {which} {MODE_NAME[prec]}"
        if which == "above" and prec in (X1, X2, X3):
            with pytest.raises(_lib.BanetError):
                ops.lm_build(lv, R, T, W, prec)
            print(f"EDGE {lab}: refused")
            continue
        out = [t.cpu() for t in ops.lm_build(lv, R, T, W, prec)]
        tol = TOL[SIMT] if which == "above" else TOL[_auto(128, crop.N) if prec == AUTO else prec]
        _check_forward(lab, out, ref, tol)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print(f"EDGE offsets {which}: peak device memory {peak / 2**30:.2f} GiB")
    del lv, dev_map
    torch.cuda.empty_cache()
    assert peak < 10 * 2 ** 30
