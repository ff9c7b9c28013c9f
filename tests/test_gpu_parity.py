"""GPU parity tests (run with `-m gpu` on an H100): every C-ABI entry point against the CPU oracle on the
same seeded inputs, and against the committed golden fixtures.  All arithmetic on the path is fp32;
tolerances are relative Frobenius errors against the float64 oracle, written beside each assert.
The headline bar (BASELINE.json north_star) is 1e-4 rel-fro on pose/depth outputs."""
import numpy as np
import pytest
import torch

from helpers import O, scene_case, oracle_level_inputs, mlp_for, rel_fro, to_cuda32, GOLDEN_DIR

pytestmark = pytest.mark.gpu

TOL_SUMS = 2e-5      # H, g, rbar: fp32 sums over N pixels vs float64
TOL_OUT = 1e-4       # R, T, W, depth: the north-star tolerance


def _ops():
    from banet_b200 import ops, _lib
    _lib.require_device()
    return ops


def _level(ops, lv, fly=False):
    conv2 = lv.conv2[..., :lv.conv1.shape[2]] if fly else lv.conv2
    return ops.Level(to_cuda32(lv.conv1), to_cuda32(conv2), to_cuda32(lv.intr), to_cuda32(lv.p), to_cuda32(lv.D), to_cuda32(lv.B))


def _oracle_build(lv, R, T, W):
    a = oracle_level_inputs(lv)
    return O.normal_equations_structured(a["conv1"], a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"],
                                         R.double(), T.double(), None if W is None else W.double())


# ---------------------------------------------------------------------------------------------- op level
@pytest.mark.parametrize("nb,N,C,P", [(2, 70, 12, 22), (1, 33, 5, 6), (3, 257, 128, 134), (1, 100, 8, 150)])
def test_equation_construction_fwd_bwd(nb, N, C, P):
    ops = _ops()
    g = torch.Generator().manual_seed(nb * 1000 + N)
    J = torch.randn(nb, N, 2, P, generator=g); G = torch.randn(nb, N, C, 2, generator=g); d = torch.randn(nb, N, C, 1, generator=g)
    lg = torch.randn(nb, P, P, generator=g); rg = torch.randn(nb, P, 1, generator=g)
    AtA, Atb = ops.equation_construction(J.cuda(), G.cuda(), d.cuda())
    rA, rb = O.equation_construction(J.double(), G.double(), d.double())
    assert rel_fro(AtA, rA) < 1e-5 and rel_fro(Atb, rb) < 1e-5
    assert torch.equal(AtA, AtA.transpose(1, 2))                       # exactly symmetric
    for exact in (False, True):
        dJ, dG, dd = ops.equation_construction_grad(J.cuda(), G.cuda(), d.cuda(), lg.cuda(), rg.cuda(), exact_sym=exact)
        lgo = (0.5 * (lg + lg.transpose(1, 2))) if exact else lg       # A(Ghat+Ghat^T) == 2 A sym(Ghat)
        oJ, oG, od = O.equation_construction_grad(J.double(), G.double(), d.double(), lgo.double(), rg.double())
        assert rel_fro(dJ, oJ) < 1e-5 and rel_fro(dG, oG) < 1e-5 and rel_fro(dd, od) < 1e-5


def test_equation_construction_autograd_and_golden():
    ops = _ops()
    ref = np.load(f"{GOLDEN_DIR}/eqc.npz")
    J, G, d = [torch.tensor(ref[k], dtype=torch.float32, device="cuda").requires_grad_() for k in ("in_J", "in_G", "in_d")]
    lg = torch.tensor(ref["in_left_grad"], dtype=torch.float32, device="cuda")
    rg = torch.tensor(ref["in_right_grad"], dtype=torch.float32, device="cuda")
    AtA, Atb = ops.equation_construction(J, G, d)
    assert rel_fro(AtA, ref["out_AtA"]) < 1e-5 and rel_fro(Atb, ref["out_Atb"]) < 1e-5
    ((AtA * lg).sum() + (Atb * rg).sum()).backward()
    assert rel_fro(J.grad, ref["out_dJ"]) < 1e-5 and rel_fro(G.grad, ref["out_dG"]) < 1e-5 and rel_fro(d.grad, ref["out_dd"]) < 1e-5


# ---------------------------------------------------------------------------------------------- pre-steps
def test_pre_steps_match_oracle():
    ops = _ops()
    g = torch.Generator().manual_seed(5)
    nb, h, w, C, N = 2, 19, 23, 12, 200
    F = torch.randn(nb, h, w, C, generator=g)
    out = ops.grad_fixed_concat(F.cuda())
    ref = torch.cat([F.double(), O.grad_fixed(F.double())], -1)
    assert rel_fro(out, ref) < 1e-6
    out = ops.grad_fixed_concat(F.cuda(), swap_halves=True)
    Fs = torch.cat([F[1:], F[:1]], 0).double()
    assert rel_fro(out, torch.cat([Fs, O.grad_fixed(Fs)], -1)) < 1e-6
    pts = torch.rand(nb, N, 2, generator=g) * torch.tensor([w + 4.0, h + 4.0]) - 2.0      # some outside the map
    s = ops.resample(F.cuda(), pts.cuda(), 1.0)
    assert rel_fro(s, O.resampler(F.double(), pts.double())) < 1e-6
    s = ops.resample(F.cuda(), pts.cuda(), 0.5)
    assert rel_fro(s, O.resampler(F.double(), pts.double() / 2)) < 1e-6
    s2, m2 = ops.interpolate2d(F.cuda(), pts.cuda(), 1.0, with_mask=True)                 # legacy sampler: clamped indices + in-bounds mask
    o2, om = O.interpolate2d(F.double(), pts[..., 0].double(), pts[..., 1].double())
    assert rel_fro(s2, o2) < 1e-6 and torch.equal(m2.cpu().double(), om)
    intr = torch.tensor([[20.0, 21.0, 11.0, 9.0]]).repeat(nb, 1)
    p = ops.compute_coordinates(pts.cuda(), intr.cuda(), True)
    t = [intr[:, i:i + 1].expand(-1, N).double() for i in range(4)]
    assert rel_fro(p, O.compute_coordinates(pts.double(), *t)) < 1e-6
    basis = torch.randn(nb, 50, 7, generator=g); W = torch.randn(nb, 7, 1, generator=g); d0 = torch.randn(nb, 50, generator=g)
    out = ops.depth_compose(d0.cuda(), basis.cuda(), W.cuda())
    assert rel_fro(out, d0.double() + (basis.double() @ W.double()).squeeze(-1)) < 1e-6


# ---------------------------------------------------------------------------------------------- build
@pytest.mark.parametrize("C,K,n_points,fly", [
    (8, 4, None, False), (8, 0, None, False), (128, 128, None, False), (6, 5, 333, False), (5, 16, 100, False),
    (12, 32, None, True), (16, 64, 1000, False), (128, 16, None, True), (16, 256, 700, False), (8, 200, None, False)])
def test_lm_build_matches_oracle(C, K, n_points, fly):
    ops = _ops()
    sc = scene_case(nb=3, H=24 if C == 128 else 48, W=32 if C == 128 else 64, C=C, K=K, level_ids=(3,), seed=7 + C + K,
                    n_points=n_points, dtype=torch.float32)
    lv = sc.levels[0]
    W = None if K == 0 else sc.W0 + 0.01 * torch.randn(sc.W0.shape, generator=torch.Generator().manual_seed(1))
    H, g, rbar, nvalid = ops.lm_build(_level(ops, lv, fly), to_cuda32(sc.R0), to_cuda32(sc.T0), to_cuda32(W))
    rH, rg, rrbar, rnv = _oracle_build(lv, sc.R0, sc.T0, W)
    assert torch.equal(nvalid.cpu().double(), rnv)
    assert rel_fro(H, rH) < TOL_SUMS and rel_fro(g, rg.squeeze(-1)) < TOL_SUMS
    assert rel_fro(rbar / lv.N, rrbar.squeeze(1)) < TOL_SUMS
    assert torch.equal(H, H.transpose(1, 2))


def test_lm_build_edge_cases():
    """All points out of bounds for one pair (huge translation) -> zero equations, nvalid 0; nb=1; tiny N."""
    ops = _ops()
    sc = scene_case(nb=2, C=8, K=4, level_ids=(3,), seed=9, n_points=7, dtype=torch.float32)
    lv = sc.levels[0]
    T = sc.T0.clone(); T[1, 0, 0] = 1e4
    H, g, rbar, nvalid = ops.lm_build(_level(ops, lv), to_cuda32(sc.R0), to_cuda32(T), to_cuda32(sc.W0))
    assert nvalid[1].item() == 0 and H[1].abs().max().item() == 0 and g[1].abs().max().item() == 0 and rbar[1].abs().max().item() == 0
    rH, rg, _, rnv = _oracle_build(lv, sc.R0, T, sc.W0)
    assert rel_fro(H[0], rH[0]) < TOL_SUMS and nvalid[0].item() == rnv[0].item()
    # non-finite projection (Z == 0) is masked, not propagated
    T2 = sc.T0.clone(); D0 = lv.D.clone(); D0[0, 0, 0] = 0.0; T2[0] = 0.0
    lv2 = ops.Level(to_cuda32(lv.conv1), to_cuda32(lv.conv2), to_cuda32(lv.intr), to_cuda32(lv.p), to_cuda32(D0), to_cuda32(lv.B))
    H, g, rbar, nvalid = ops.lm_build(lv2, to_cuda32(sc.R0), to_cuda32(T2), to_cuda32(sc.W0))
    assert torch.isfinite(H).all() and torch.isfinite(g).all()


def test_lm_build_is_deterministic():
    ops = _ops()
    sc = scene_case(nb=4, C=16, K=16, level_ids=(3,), seed=13, dtype=torch.float32)
    lvl = _level(ops, sc.levels[0])
    a = ops.lm_build(lvl, to_cuda32(sc.R0), to_cuda32(sc.T0), to_cuda32(sc.W0))
    b = ops.lm_build(lvl, to_cuda32(sc.R0), to_cuda32(sc.T0), to_cuda32(sc.W0))
    for x, y in zip(a, b):
        assert torch.equal(x, y)


# ---------------------------------------------------------------------------------------------- lambda / solve
@pytest.mark.parametrize("C", [8, 128])
def test_lambda_mlp(C):
    ops = _ops()
    g = torch.Generator().manual_seed(C)
    nb, N = 3, 500
    rbar_sum = torch.rand(nb, C, generator=g) * N * 0.2
    mlp = mlp_for(C, 2)
    lam = ops.lm_lambda(rbar_sum.cuda(), N, ops.pack_mlp(mlp).cuda(), 1000.0)
    avg = (rbar_sum.double() / N).unsqueeze(1)
    ref = 1000.0 * torch.pow(torch.linalg.norm(avg, dim=-1, keepdim=True), 2.0 + O.lambda_mlp(avg, mlp))
    assert rel_fro(lam, ref.reshape(-1)) < 1e-4


@pytest.mark.parametrize("K,undamped_last,scramble", [(0, False, False), (4, True, False), (128, True, False), (250, True, False), (3, True, True)])
def test_solve_update(K, undamped_last, scramble):
    ops = _ops()
    g = torch.Generator().manual_seed(K + 1)
    nb, P = 3, 6 + K
    A = torch.randn(nb, P, 3 * P, generator=g, dtype=torch.float64)
    H = (A @ A.transpose(1, 2)) / (3 * P); gv = torch.randn(nb, P, 1, generator=g, dtype=torch.float64) * 1e-2
    lam = torch.rand(nb, generator=g, dtype=torch.float64) + 0.1
    H32, g32, lam32 = H.float(), gv.float(), lam.float()
    R = O.angle_axis_rotation(*[torch.randn(nb, 1, 1, generator=g, dtype=torch.float64) * 0.1 for _ in range(3)]).float()
    T = torch.randn(nb, 3, 1, generator=g); W = torch.randn(nb, K, 1, generator=g) if K else None
    Rn, Tn, Wn, delta, status = ops.lm_solve_update(H32.cuda(), g32.cuda(), lam32.cuda(), R.cuda(), T.cuda(), to_cuda32(W),
                                                    undamped_last=undamped_last, vmatrix_batch_scramble=scramble)
    assert status.abs().max().item() == 0
    Hd = H32.double(); diag = torch.diagonal(Hd, dim1=1, dim2=2)
    dvec = (diag + 1e-5) * lam32.double().unsqueeze(-1)
    if undamped_last:
        dvec[:, -1] = 0
    sol = torch.linalg.solve(Hd + torch.diag_embed(dvec), g32.double())
    assert rel_fro(delta, sol.squeeze(-1)) < 1e-5
    oR, oT = O._update(sol[:, :6], R.double(), T.double(), O.IterOptions(vmatrix_batch_scramble=scramble))
    assert rel_fro(Rn, oR) < 1e-6 and rel_fro(Tn, oT) < 1e-6
    if K:
        assert rel_fro(Wn, W.double() + sol[:, 6:]) < 1e-6


def test_solve_flags_bad_matrices():
    ops = _ops()
    nb, P = 3, 10
    H = torch.eye(P).repeat(nb, 1, 1); H[1, 3, 3] = -5.0; H[2, 0, 0] = float("nan")
    gv = torch.ones(nb, P); lam = torch.zeros(nb)
    R = torch.eye(3).repeat(nb, 1, 1); T = torch.zeros(nb, 3, 1); W = torch.zeros(nb, P - 6, 1)
    Rn, Tn, Wn, delta, status = ops.lm_solve_update(H.cuda(), gv.cuda(), lam.cuda(), R.cuda(), T.cuda(), W.cuda(), undamped_last=False)
    assert status.tolist()[0] == 0 and status.tolist()[1] & 1 and status.tolist()[2] & 2
    assert delta[1:].abs().max().item() == 0 and torch.equal(Rn[1:].cpu(), R[1:]) and torch.equal(Wn[1:].cpu(), W[1:])


# ---------------------------------------------------------------------------------------------- whole iterations
def test_bundle_iteration_golden_and_mirror_api():
    """Reference-shaped call (BundleNet.BundleIteration, bundlenet.py:193) against the committed fixture."""
    _ops()
    import gen_golden
    from banet_b200.bundlenet import BundleNet
    ref = np.load(f"{GOLDEN_DIR}/bundle_iteration.npz")
    sc = gen_golden._scene(2, 48, 64, 8, 4, (3,), 21)
    lv = sc.levels[0]
    net = BundleNet(8, levels=("3",)).cuda()
    for i, (w, b) in enumerate(gen_golden.mlp_for(8, 3)):
        getattr(net, f"lambda_3_{i + 1}_filters").data.copy_(w); getattr(net, f"lambda_3_{i + 1}_biases").data.copy_(b)
    fx, fy, ox, oy = [to_cuda32(t) for t in lv.intr_tiled()]
    W = (sc.W0.double() + 0.01).float()
    Rn, Tn, Wn, aux = net.BundleIteration(to_cuda32(lv.conv1), to_cuda32(lv.conv2), fx, fy, ox, oy, to_cuda32(lv.p), to_cuda32(lv.D),
                                          to_cuda32(lv.B), to_cuda32(sc.R0), to_cuda32(sc.T0), to_cuda32(W), 1000.0, "3", return_aux=True)
    assert rel_fro(aux["AtA"], ref["out_AtA"]) < TOL_SUMS and rel_fro(aux["Atb"], ref["out_Atb"].squeeze(-1)) < TOL_SUMS
    assert rel_fro(aux["lam"], ref["out_lam"].reshape(-1)) < 1e-4
    assert rel_fro(aux["solution"], ref["out_solution"].squeeze(-1)) < TOL_OUT
    assert rel_fro(Rn, ref["out_R"]) < TOL_OUT and rel_fro(Tn, ref["out_T"]) < TOL_OUT and rel_fro(Wn, ref["out_W"]) < TOL_OUT


def test_camera_iteration_golden():
    _ops()
    import gen_golden
    from banet_b200.bundlenet import BundleNet
    ref = np.load(f"{GOLDEN_DIR}/camera_iteration.npz")
    sc = gen_golden._scene(2, 48, 64, 6, 0, (3,), 22, n_points=300)
    lv = sc.levels[0]
    net = BundleNet(6, levels=("3",)).cuda()
    for i, (w, b) in enumerate(gen_golden.mlp_for(6, 3)):
        getattr(net, f"lambda_3_{i + 1}_filters").data.copy_(w); getattr(net, f"lambda_3_{i + 1}_biases").data.copy_(b)
    fx, fy, ox, oy = [to_cuda32(t) for t in lv.intr_tiled()]
    Rn, Tn, aux = net.CameraIteration(to_cuda32(lv.conv1), to_cuda32(lv.conv2), fx, fy, ox, oy, to_cuda32(lv.p), to_cuda32(lv.D),
                                      to_cuda32(sc.R0), to_cuda32(sc.T0), 1.0, "3", return_aux=True)
    assert rel_fro(aux["AtA"], ref["out_AtA"]) < TOL_SUMS and rel_fro(aux["solution"], ref["out_solution"].squeeze(-1)) < TOL_OUT
    assert rel_fro(Rn, ref["out_R"]) < TOL_OUT and rel_fro(Tn, ref["out_T"]) < TOL_OUT


def test_lm_run_golden_and_convergence():
    ops = _ops()
    import gen_golden
    ref = np.load(f"{GOLDEN_DIR}/lm_solve.npz")
    sc = gen_golden._scene(2, 48, 64, 8, 16, (2, 3), 23)
    levels = [_level(ops, lv) for lv in sc.levels]
    R, T, W, status = ops.lm_run(levels, 3, to_cuda32(sc.R0), to_cuda32(sc.T0), to_cuda32(sc.W0), lambda_fixed=0.05)
    assert status.abs().max().item() == 0
    assert rel_fro(R, ref["out_R"]) < TOL_OUT and rel_fro(T, ref["out_T"]) < TOL_OUT and rel_fro(W, ref["out_W"]) < TOL_OUT


def test_bundle_and_camera_resize_golden():
    """Reference schedulers BundleResize / CameraResize (bundlenet.py:280-399) end to end."""
    _ops()
    import gen_golden
    from banet_b200.bundlenet import BundleNet
    ref = np.load(f"{GOLDEN_DIR}/bundle_resize.npz")
    x = gen_golden.resize_inputs()
    net = BundleNet(4).cuda()
    for l in range(4):
        for i, (w, b) in enumerate(gen_golden.mlp_for(4, l)):
            getattr(net, f"lambda_{l}_{i + 1}_filters").data.copy_(w); getattr(net, f"lambda_{l}_{i + 1}_biases").data.copy_(b)
    layers = [to_cuda32(t) for t in x["layers"]]
    Rs, Ts, Ds = net.BundleResize(to_cuda32(x["intr"]), layers, to_cuda32(x["points"]), to_cuda32(x["basis"]), to_cuda32(x["depth"]),
                                  to_cuda32(x["R0"]), to_cuda32(x["T0"]))
    for i in range(2):
        assert rel_fro(Rs[i], ref[f"out_R{i}"]) < TOL_OUT and rel_fro(Ts[i], ref[f"out_T{i}"]) < TOL_OUT
        assert rel_fro(Ds[i], ref[f"out_D{i}"]) < TOL_OUT
    rot, tr = net.CameraResize(to_cuda32(x["intr"]), layers, to_cuda32(x["points"]), to_cuda32(x["depth"]))
    for i in range(4):
        assert rel_fro(rot[i], ref[f"out_camR{i}"]) < TOL_OUT and rel_fro(tr[i], ref[f"out_camT{i}"]) < TOL_OUT


def test_full_size_properties():
    """BASELINE-size level (640x480, C=K=128), one pair: size-independent properties instead of the oracle —
    additivity over pixel subsets (H(all) == H(first half) + H(second half)), symmetry, determinism."""
    ops = _ops()
    from banet_b200 import synth
    sc = synth.make_scene(nb=1, H=480, W=640, C=128, K=128, level_ids=(3,), seed=77, device="cuda", dtype=torch.float32,
                          rot_deg=0.03, trans_m=0.002, start_trans_noise_m=0.001)      # inside the fine level's basin
    lv = sc.levels[0]
    full = ops.Level(lv.conv1, lv.conv2, lv.intr, lv.p, lv.D, lv.B)
    H, g, rbar, nv = ops.lm_build(full, sc.R0, sc.T0, sc.W0)
    half = lv.N // 2
    parts = []
    for sl in (slice(0, half), slice(half, lv.N)):
        part = ops.Level(lv.conv1[:, sl].contiguous(), lv.conv2, lv.intr, lv.p[:, :, sl].contiguous(), lv.D[:, sl].contiguous(),
                         lv.B[:, sl].contiguous())
        parts.append(ops.lm_build(part, sc.R0, sc.T0, sc.W0))
    assert rel_fro(parts[0][0] + parts[1][0], H) < 1e-5 and rel_fro(parts[0][1] + parts[1][1], g) < 1e-5
    assert rel_fro(parts[0][2] + parts[1][2], rbar) < 1e-5 and (parts[0][3] + parts[1][3]).item() == nv.item()
    assert torch.equal(H, H.transpose(1, 2))
    R, T, W, status = ops.lm_run([full], 5, sc.R0, sc.T0, sc.W0, lambda_fixed=1e-2)
    assert status.item() == 0
    e0 = (sc.T0 - sc.T_true).norm().item(); e1 = (T - sc.T_true).norm().item()
    assert e1 < 0.05 * e0 and (W - sc.W_true).norm().item() < 0.2 * sc.W_true.norm().item()


@pytest.mark.parametrize("C", [128, 32])
def test_cfg1_reference_cpu_case(C):
    """BASELINE.json configs[0] — the reference's own CPU-runnable case: one 2-frame pair, 160x120 single scale, K=16 depth
    bases, 3 LM iterations with the lambda-MLP, at the pyramid width of the headline configs (C=128) and at C=32 — whole solve against
    the oracle's reference-faithful materialised form at the north-star tolerance, through banet_lm_run."""
    ops = _ops()
    sc = scene_case(nb=1, H=120, W=160, C=C, K=16, level_ids=(3,), seed=1235, dtype=torch.float32)
    lv = sc.levels[0]
    mlp = mlp_for(C, 3)
    a = oracle_level_inputs(lv)
    ol = O.LevelInputs(a["conv1"], a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"], mlp)
    oR, oT, oW = O.lm_solve([ol], 3, sc.R0.double(), sc.T0.double(), sc.W0.double(), O.IterOptions(l2_regularizer_base=1000.0))
    packed = ops.pack_mlp([(w.float(), b.float()) for w, b in mlp]).cuda()
    R, T, W, status = ops.lm_run([_level(ops, lv)], 3, to_cuda32(sc.R0), to_cuda32(sc.T0), to_cuda32(sc.W0), mlp_packed=[packed],
                                 l2_regularizer_base=1000.0)
    assert status.abs().max().item() == 0
    assert rel_fro(R, oR) < TOL_OUT and rel_fro(T, oT) < TOL_OUT and rel_fro(W, oW) < TOL_OUT
    depth = ops.depth_compose(to_cuda32(lv.D).reshape(1, -1), to_cuda32(lv.B), W)
    assert rel_fro(depth, (a["D"] + a["B"] @ oW).reshape(1, -1)) < TOL_OUT


@pytest.mark.parametrize("K,C", [(0, 8), (4, 8), (128, 128), (250, 16), (37, 5)])
def test_lm_step_fused_lambda_solve_update(K, C):
    """banet_lm_step (lambda-MLP + damping + blocked Cholesky with the rhs as an extra row + update, one launch) against float64 LU and the
    oracle's lambda MLP / SE(3) update, and against the separate banet_lm_lambda + banet_lm_solve_update kernels."""
    ops = _ops()
    g = torch.Generator().manual_seed(100 + K)
    nb, P, N = 3, 6 + K, 700
    A = torch.randn(nb, P, 3 * P, generator=g, dtype=torch.float64)
    H = ((A @ A.transpose(1, 2)) / (3 * P)).float(); gv = (torch.randn(nb, P, generator=g, dtype=torch.float64) * 1e-2).float()
    rbar_sum = torch.rand(nb, C, generator=g) * N * 0.2
    mlp = mlp_for(C, 2)
    base = 1000.0 if K else 1.0
    R = O.angle_axis_rotation(*[torch.randn(nb, 1, 1, generator=g, dtype=torch.float64) * 0.1 for _ in range(3)]).float()
    T = torch.randn(nb, 3, 1, generator=g); W = torch.randn(nb, K, 1, generator=g) if K else None
    Rn, Tn, Wn, delta, lam, status = ops.lm_step(H.cuda(), gv.cuda(), rbar_sum.cuda(), N, ops.pack_mlp(mlp).cuda(), base, R.cuda(), T.cuda(), to_cuda32(W))
    assert status.abs().max().item() == 0
    avg = (rbar_sum.double() / N).unsqueeze(1)
    olam = base * torch.pow(torch.linalg.norm(avg, dim=-1, keepdim=True), 2.0 + O.lambda_mlp(avg, mlp)).reshape(nb)
    assert rel_fro(lam, olam) < 1e-4
    Hd = H.double(); diag = torch.diagonal(Hd, dim1=1, dim2=2)
    dvec = (diag + 1e-5) * lam.cpu().double().unsqueeze(-1)
    if K:
        dvec[:, -1] = 0
    sol = torch.linalg.solve(Hd + torch.diag_embed(dvec), gv.double().unsqueeze(-1))
    assert rel_fro(delta, sol.squeeze(-1)) < 1e-5
    oR, oT = O._update(sol[:, :6], R.double(), T.double(), O.IterOptions())
    assert rel_fro(Rn, oR) < 1e-6 and rel_fro(Tn, oT) < 1e-6
    if K:
        assert rel_fro(Wn, W.double() + sol[:, 6:]) < 1e-6
    lam2 = ops.lm_lambda(rbar_sum.cuda(), N, ops.pack_mlp(mlp).cuda(), base)
    R2, T2, W2, d2, st2 = ops.lm_solve_update(H.cuda(), gv.cuda(), lam2, R.cuda(), T.cuda(), to_cuda32(W), undamped_last=K > 0)
    assert rel_fro(lam, lam2) < 1e-5 and rel_fro(delta, d2) < 1e-5 and rel_fro(Rn, R2) < 1e-6 and rel_fro(Tn, T2) < 1e-6
    # a given lambda instead of the MLP, and a non-SPD matrix (flagged, step skipped)
    Rn3, Tn3, Wn3, d3, lam3, st3 = ops.lm_step(H.cuda(), gv.cuda(), None, N, None, 1.0, R.cuda(), T.cuda(), to_cuda32(W), lam=lam2)
    assert rel_fro(d3, d2) < 1e-5 and torch.equal(lam3, lam2)
    Hbad = H.clone(); Hbad[1] = -Hbad[1]
    Rb, Tb, Wb, db, lb, stb = ops.lm_step(Hbad.cuda(), gv.cuda(), None, N, None, 1.0, R.cuda(), T.cuda(), to_cuda32(W), lam=lam2)
    assert stb.tolist()[1] == 1 and stb.tolist()[0] == 0 and float(db[1].abs().max()) == 0.0 and rel_fro(Tb[1], T[1]) < 1e-7
