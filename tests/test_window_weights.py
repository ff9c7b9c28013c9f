"""Per-point confidence weights in keyframe windows: one weight per (frame, keyframe point), pair w*nf + f, with the semantics of
banet_level_t::weight per pair (H = sum w J^T M J, g = sum w J^T q; the mean |residual| and nvalid stay unweighted).  The float64 statement
(tests/weighted_window_oracle.py) is tied to the oracle on the CPU; the keyframe build (banet_keyframe_level_t::weight), its backward
(banet_lm_keyframe_build_bwd_weighted), the window runs, autograd and BundleNet.WindowIteration / WindowResize are held to it on the GPU.
Weights of ones must give the unweighted bits (x * 1.0f is exact)."""
import ctypes
import dataclasses

import pytest
import torch

from helpers import O, scene_case, oracle_level_inputs, mlp_for, rel_fro, to_cuda32
import weighted_oracle as WO
import weighted_window_oracle as WWO
from window_resize_oracle import window_resize as window_resize_oracle
from banet_b200 import _lib

gpu = pytest.mark.gpu
F64 = torch.float64


# ------------------------------------------------------------------------------------------------ CPU: the weighted statement
def _window_case(nf, K=5, C=8, seed=3, n_points=300):
    """One window of nf pairs (float64, CPU), the keyframe tensors (frame 0's) given per frame."""
    sc = scene_case(nb=nf, C=C, K=K, level_ids=(3,), seed=seed, n_points=n_points, shared_depth=True)
    a = oracle_level_inputs(sc.levels[0])
    kf = lambda t: t[:1].expand(nf, *t.shape[1:]).contiguous()
    for k in ("conv1", "D", "B", "p"):
        a[k] = kf(a[k])
    W = sc.W0[0] + 0.01
    return sc, a, W


def _args(a):
    return (a["conv1"], a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"])


def test_weighted_window_statement_with_weights_of_ones_is_the_oracle():
    nf = 3
    sc, a, W = _window_case(nf)
    ones = torch.ones(nf, a["conv1"].shape[1], 1, dtype=F64)
    opts = O.IterOptions(l2_regularizer_base=1000.0, guard_nonfinite=True)
    mine = WWO.window_iteration(*_args(a), sc.R0, sc.T0, W, mlp_for(8, 3), ones, opts)
    ref = O.window_iteration(*_args(a), sc.R0, sc.T0, W, mlp_for(8, 3), opts)
    for x, y in zip(mine, ref):
        assert rel_fro(x, y) < 1e-12


def test_weighted_window_resize_with_weights_of_ones_is_window_resize():
    from banet_b200 import synth
    nw, nf, C, K = 2, 3, 4, 3
    sc = synth.make_window_resize_scene(nw, nf, C, K, n_points=300, seed=8, dtype=F64)
    mlps = {str(l): mlp_for(C, l) for l in (2, 3)}
    args = (sc.intrisic, sc.key_layers, sc.frame_layers, sc.points, sc.basis, sc.init_depth, mlps, sc.R0, sc.T0)
    opts = O.IterOptions(guard_nonfinite=True)
    ref = window_resize_oracle(*args, opts)
    for wt in (torch.ones(nw, nf, sc.points.shape[1], 1, dtype=F64), torch.ones(nw, 1, sc.points.shape[1], 1, dtype=F64)):
        mine = WWO.window_resize(*args, wt, opts)
        for xs, ys in zip(mine, ref):
            for x, y in zip(xs, ys):
                assert rel_fro(x, y) < 1e-12


def test_weighted_window_of_one_frame_is_the_weighted_two_view_iteration():
    sc, a, W = _window_case(1, seed=4)
    w = 2 * torch.rand(1, a["conv1"].shape[1], 1, generator=torch.Generator().manual_seed(1), dtype=F64)
    opts = O.IterOptions(l2_regularizer_base=1000.0, guard_nonfinite=True)
    mine = WWO.window_iteration(*_args(a), sc.R0, sc.T0, W, mlp_for(8, 3), w, opts)
    ref = WO.iteration(*_args(a), sc.R0, sc.T0, W.reshape(1, *W.shape), mlp_for(8, 3), w, opts)
    for x, y in zip(mine, (ref[0], ref[1], ref[2][0])):
        assert rel_fro(x, y) < 1e-12


def _select(a, idx):
    """The per-frame oracle inputs restricted to (or repeating) the keyframe points idx."""
    out = dict(a)
    for k in ("conv1", "D", "B", "fx", "fy", "ox", "oy"):
        out[k] = a[k][:, idx]
    out["p"] = a["p"][:, :, idx]
    return out


def test_weight_two_duplicates_a_point_and_zero_in_one_frame_removes_it_there():
    nf = 3
    sc, a, W = _window_case(nf, seed=5)
    N = a["conv1"].shape[1]
    g = torch.Generator().manual_seed(0)
    two = torch.randperm(N, generator=g)[:40]
    w = torch.ones(nf, N, 1, dtype=F64)
    w[:, two] = 2.0
    _, _, _, Hj, gj = WWO.window_system(*_args(a), sc.R0, sc.T0, W, w)
    _, _, _, rHj, rgj = WWO.window_system(*_args(_select(a, torch.cat([torch.arange(N), two]))), sc.R0, sc.T0, W)
    assert rel_fro(Hj, rHj) < 1e-12 and rel_fro(gj, rgj) < 1e-12
    # zero weights in frame 1 only: frame 1's pair system on the remaining points, the other frames' on all of them
    zero = torch.randperm(N, generator=g)[:70]
    keep = torch.tensor([n for n in range(N) if n not in set(zero.tolist())])
    w = torch.ones(nf, N, 1, dtype=F64)
    w[1, zero] = 0.0
    _, _, _, Hj, gj = WWO.window_system(*_args(a), sc.R0, sc.T0, W, w)
    H, gv, _, _, _ = WWO.window_system(*_args(a), sc.R0, sc.T0, W)
    s = _select(a, keep)
    H1, g1, _, _, _ = WWO.window_system(*[t[1:2] for t in _args(s)], sc.R0[1:2], sc.T0[1:2], W)
    H, gv = H.clone(), gv.clone()
    H[1], gv[1] = H1[0], g1[0]
    rHj, rgj = O.window_assemble(H, gv)
    assert rel_fro(Hj, rHj) < 1e-12 and rel_fro(gj, rgj) < 1e-12


def test_autograd_dweight_is_the_inner_product_with_the_assembled_adjoint():
    nf, K = 3, 5
    sc, a, W = _window_case(nf, K=K, seed=6)
    N, P = a["conv1"].shape[1], 6 + K
    gen = torch.Generator().manual_seed(2)
    w = (2 * torch.rand(nf, N, 1, generator=gen, dtype=F64)).requires_grad_()
    Pj = 6 * nf + K
    cH, cg = torch.randn(Pj, Pj, generator=gen, dtype=F64), torch.randn(Pj, 1, generator=gen, dtype=F64)
    _, _, _, Hj, gj = WWO.window_system(*_args(a), sc.R0, sc.T0, W, w)
    ((Hj * cH).sum() + (gj * cg).sum()).backward()
    Hn, gn = WO.point_terms(*_args(a), sc.R0, sc.T0, W.reshape(1, K, 1).expand(nf, K, 1))
    for f in range(nf):                                 # frame f's adjoint: its pose rows / columns, the window's depth block
        s = slice(6 * f, 6 * f + 6)
        dH = torch.zeros(P, P, dtype=F64); dg = torch.zeros(P, dtype=F64)
        dH[:6, :6] = cH[s, s]; dH[:6, 6:] = cH[s, 6 * nf:]; dH[6:, :6] = cH[6 * nf:, s]; dH[6:, 6:] = cH[6 * nf:, 6 * nf:]
        dg[:6] = cg[s, 0]; dg[6:] = cg[6 * nf:, 0]
        expect = torch.einsum("npq,pq->n", Hn[f], dH) + gn[f] @ dg
        assert rel_fro(w.grad[f, :, 0], expect) < 1e-12, f


def test_window_weights_shape_and_dtype_errors_name_the_weight():
    from banet_b200 import autograd as AG
    ok = torch.ones(2, 3, 10, 1)
    assert tuple(AG.window_weights(ok, 2, 3, 10).shape) == (6, 10, 1)
    assert tuple(AG.window_weights(torch.ones(2, 1, 10, 1), 2, 3, 10).shape) == (6, 10, 1)
    assert tuple(AG.window_weights(torch.ones(1, 10, 1), None, 3, 10).shape) == (3, 10, 1)
    for bad in (ok.double(), ok.bfloat16(), torch.ones(2, 2, 10, 1), torch.ones(2, 3, 10), torch.ones(6, 10, 1), torch.ones(2, 3, 9, 1), None):
        with pytest.raises(_lib.BanetError, match="weight"):
            AG.window_weights(bad, 2, 3, 10)


# ------------------------------------------------------------------------------------------------ CPU: the C-ABI
def _klevel(**kw):
    lv = _lib.BanetKeyframeLevel(2, 4, 4096, 64, 128, 120, 160, 192, 1, 1, 1, 1, 1, 1)
    for k, v in kw.items():
        setattr(lv, k, v)
    return lv


def test_keyframe_struct_built_without_the_field_is_unweighted():
    assert _klevel().weight is None
    assert _lib.BanetKeyframeLevel.weight.offset > _lib.BanetKeyframeLevel.intr.offset


def test_weighted_keyframe_backward_rejects_bad_arguments_before_any_cuda_call():
    lib = _lib.load()
    bwd = lambda lv, dH=1, dweight=1: lib.banet_lm_keyframe_build_bwd_weighted(ctypes.byref(lv), 1, 1, 1, dH, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1,
                                                                               dweight, None)
    assert bwd(_klevel(weight=1, nw=0)) == -1 and b"bad shape" in lib.banet_last_error()
    assert bwd(_klevel(weight=1), dH=None) == -1 and b"null pointer" in lib.banet_last_error()
    assert bwd(_klevel(weight=1, conv2_channels=64)) == -4 and b"3C" in lib.banet_last_error()
    assert bwd(_klevel(weight=1, K=257)) == -4 and b"K=257" in lib.banet_last_error()
    assert bwd(_klevel(weight=1, K=256, C=128, conv2_channels=384), dweight=None) == -4 and b"shared memory" in lib.banet_last_error()


# ------------------------------------------------------------------------------------------------ GPU
def _gscene(nw, nf, C, K, n_points=1000, seed=1, H=48, W=64):
    from banet_b200 import synth
    return synth.make_scene(nb=nw * nf, H=H, W=W, C=C, K=K, level_ids=(3,), seed=seed, device="cuda", dtype=torch.float32,
                            n_points=n_points, shared_depth=True, window_frames=nf)


def _levels(sc, nw, nf, layout="3c", weight=None, lv=None):
    """The keyframe level (frame 0's keyframe tensors once per window) and the per-pair level on copies of them."""
    from banet_b200 import ops
    l = sc.levels[0] if lv is None else lv
    C = l.conv1.shape[2]
    kf = lambda t: t.reshape(nw, nf, *t.shape[1:])[:, 0].contiguous()
    r = lambda t: t.repeat_interleave(nf, 0).contiguous()
    conv2 = l.conv2 if layout == "3c" else l.conv2[..., :C].contiguous()
    key = ops.KeyframeLevel(kf(l.conv1), conv2, l.intr, kf(l.p), kf(l.D), kf(l.B), weight=weight)
    rep = ops.Level(r(key.conv1), conv2, l.intr, r(key.p), r(key.D), r(key.B), weight=weight)
    return key, rep


def _start(sc, nw, nf, K):
    W = sc.W0.reshape(nw, nf, K, 1)[:, 0] + 0.01 * torch.arange(1, nw + 1, device="cuda").reshape(nw, 1, 1)
    return sc.R0, sc.T0, W.contiguous()


def _rand_w(nb, N, seed, lo=0.0, hi=2.0):
    return lo + (hi - lo) * torch.rand(nb, N, 1, generator=torch.Generator().manual_seed(seed)).cuda()


@gpu
@pytest.mark.parametrize("C", [128, 10])
@pytest.mark.parametrize("K", [5, 16, 64, 128, 200])
def test_keyframe_build_weights_of_ones_give_the_unweighted_bits(K, C):
    from banet_b200 import ops
    _lib.require_device()
    nw = 2
    for nf in (1, 3, 16):
        sc = _gscene(nw, nf, C, K, n_points=700, seed=K + nf)
        R, T, W = _start(sc, nw, nf, K)
        ones = torch.ones(nw * nf, sc.levels[0].N, 1, device="cuda")
        for layout in ("3c", "f2"):
            a = ops.lm_keyframe_build(_levels(sc, nw, nf, layout)[0], R, T, W)
            b = ops.lm_keyframe_build(_levels(sc, nw, nf, layout, ones)[0], R, T, W)
            for x, y, name in zip(a, b, ("H", "g", "rbar_sum", "nvalid")):
                assert torch.equal(x, y), (nf, layout, name)


def _f64_window_reduced(lv, sc, nw, nf, W, weight):
    """The float64 statement per pair on the replicated keyframe: H [nb,P,P] with frame 0's depth block the window's sum, the others zero."""
    a = {k: (None if v is None else v.cpu()) for k, v in oracle_level_inputs(lv).items()}
    rp = lambda t: t.reshape(nw, nf, *t.shape[1:])[:, :1].expand(nw, nf, *t.shape[1:]).reshape(t.shape)
    H, g, rbar, nv = WO.normal_equations(rp(a["conv1"]), a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], rp(a["p"]), rp(a["D"]), rp(a["B"]),
                                         sc.R0.cpu().double(), sc.T0.cpu().double(), W.cpu().double().repeat_interleave(nf, 0),
                                         None if weight is None else weight.cpu().double())
    return _reduce(H, nw, nf), g.squeeze(-1), rbar.squeeze(1), nv


def _reduce(H, nw, nf):
    P = H.shape[-1]
    Hw = H.reshape(nw, nf, P, P).clone()
    Hw[:, 0, 6:, 6:] = Hw[:, :, 6:, 6:].sum(1)
    Hw[:, 1:, 6:, 6:] = 0
    return Hw.reshape(nw * nf, P, P)


@gpu
@pytest.mark.parametrize("layout", ["3c", "f2"])
@pytest.mark.parametrize("nw,nf,C,K", [(2, 4, 8, 16), (2, 3, 128, 128), (2, 4, 128, 200), (1, 16, 10, 64)])
def test_weighted_keyframe_build_is_the_window_reduced_weighted_per_pair_build(nw, nf, C, K, layout):
    from banet_b200 import ops
    _lib.require_device()
    sc = _gscene(nw, nf, C, K, n_points=1500, seed=11 + K)
    R, T, W = _start(sc, nw, nf, K)
    w = _rand_w(nw * nf, sc.levels[0].N, seed=K)
    key, rep = _levels(sc, nw, nf, layout, w)
    H, g, rb, nv = ops.lm_keyframe_build(key, R, T, W)
    Hr, gr, rbr, nvr = ops.lm_build(rep, R, T, W.repeat_interleave(nf, 0).contiguous(), _lib.PREC_FP32_SIMT)
    nb, P = nw * nf, 6 + K
    e = (rel_fro(H, _reduce(Hr, nw, nf)), rel_fro(g, gr), rel_fro(rb, rbr))
    print(f"nw={nw} nf={nf} C={C} K={K} {layout}: vs weighted per-pair build H {e[0]:.1e} g {e[1]:.1e} rbar {e[2]:.1e}")
    assert max(e) < 1e-5 and torch.equal(nv, nvr) and torch.equal(H, H.transpose(1, 2))
    oH, og, orb, onv = _f64_window_reduced(sc.levels[0], sc, nw, nf, W, w)
    eo = (rel_fro(H, oH), rel_fro(g, og), rel_fro(rb / key.conv1.shape[1], orb))
    print(f"  vs float64 statement H {eo[0]:.1e} g {eo[1]:.1e} rbar {eo[2]:.1e}")
    assert max(eo) < 1e-5 and torch.equal(nv.cpu().double(), onv)
    H0, _, rb0, nv0 = ops.lm_keyframe_build(_levels(sc, nw, nf, layout)[0], R, T, W)
    assert torch.equal(rb, rb0) and torch.equal(nv, nv0) and rel_fro(H, H0) > 1e-3       # lambda's inputs unweighted; H weighted


@gpu
def test_zero_weights_remove_points_from_the_keyframe_build():
    from banet_b200 import ops
    _lib.require_device()
    nw, nf, C, K = 2, 4, 128, 128
    sc = _gscene(nw, nf, C, K, n_points=1500, seed=5)
    R, T, W = _start(sc, nw, nf, K)
    l = sc.levels[0]
    N = l.N
    keep = torch.rand(N, generator=torch.Generator().manual_seed(3)) < 0.5
    idx = torch.nonzero(keep).flatten().cuda()
    w = keep.float().reshape(1, N, 1).repeat(nw * nf, 1, 1).cuda()
    H, g, _, _ = ops.lm_keyframe_build(_levels(sc, nw, nf, weight=w)[0], R, T, W)
    key, _ = _levels(sc, nw, nf)
    half = ops.KeyframeLevel(key.conv1[:, idx].contiguous(), key.conv2, key.intr, key.p[:, :, idx].contiguous(), key.D[:, idx].contiguous(),
                             key.B[:, idx].contiguous())
    Hh, gh, _, _ = ops.lm_keyframe_build(half, R, T, W)
    assert rel_fro(H, Hh) < 1e-5 and rel_fro(g, gh) < 1e-5
    # zero weights in frame 2 of each window only, against the float64 statement
    w1 = torch.ones(nw, nf, N, 1, device="cuda")
    w1[:, 2, ~keep.cuda()] = 0.0
    w1 = w1.reshape(nw * nf, N, 1)
    H1, g1, _, _ = ops.lm_keyframe_build(_levels(sc, nw, nf, weight=w1)[0], R, T, W)
    oH, og, _, _ = _f64_window_reduced(l, sc, nw, nf, W, w1)
    assert rel_fro(H1, oH) < 1e-5 and rel_fro(g1, og) < 1e-5


def _poisoned_ws(pattern):
    def make(nbytes, device):
        n = max(int(nbytes), 256)
        if pattern == "nan":
            return torch.full((n,), 0xFF, dtype=torch.uint8, device=device)
        g = torch.Generator(device="cuda").manual_seed(n % 9973 + 1)
        return torch.randint(0, 256, (n,), dtype=torch.uint8, device=device, generator=g)
    return make


@gpu
def test_weighted_keyframe_build_and_run_are_bit_reproducible(monkeypatch):
    from banet_b200 import ops
    _lib.require_device()
    nw, nf, C, K = 3, 4, 32, 128
    sc = _gscene(nw, nf, C, K, n_points=2000, seed=9)
    R, T, W = _start(sc, nw, nf, K)
    key, _ = _levels(sc, nw, nf, weight=_rand_w(nw * nf, sc.levels[0].N, seed=4))
    packed = [ops.pack_mlp(mlp_for(C, 3, torch.float32)).cuda()]
    outs = []
    for pattern in ("nan", "random", "nan"):
        monkeypatch.setattr(ops, "_ws", _poisoned_ws(pattern))
        outs.append(list(ops.lm_keyframe_build(key, R, T, W)) + list(ops.lm_keyframe_run([key], 2, R, T, W, mlp_packed=packed)))
    assert int(outs[0][-1].abs().max()) == 0 and bool(torch.isfinite(outs[0][0]).all())
    for other in outs[1:]:
        for x, y in zip(outs[0], other):
            assert torch.equal(x, y)


@gpu
@pytest.mark.parametrize("exact_sym", [True, False])
def test_keyframe_backward_with_weights(exact_sym):
    from banet_b200 import ops
    _lib.require_device()
    nw, nf, C, K = 2, 4, 32, 128
    sc = _gscene(nw, nf, C, K, n_points=2000, seed=21)
    R, T, W = _start(sc, nw, nf, K)
    nb, P, N = nw * nf, 6 + K, sc.levels[0].N
    gen = torch.Generator(device="cuda").manual_seed(21)
    dH = 1e-3 * torch.randn(nb, P, P, generator=gen, device="cuda")
    dg = 1e-3 * torch.randn(nb, P, generator=gen, device="cuda"); dr = 1e-3 * torch.randn(nb, C, generator=gen, device="cuda")
    ones = torch.ones(nb, N, 1, device="cuda")
    key0, _ = _levels(sc, nw, nf)
    key1, _ = _levels(sc, nw, nf, weight=ones)
    a = ops.lm_keyframe_build_bwd(key0, R, T, W, dH, dg, dr, exact_sym)
    b = ops.lm_keyframe_build_bwd(key1, R, T, W, dH, dg, dr, exact_sym, return_dweight=True)
    c = ops.lm_keyframe_build_bwd(key0, R, T, W, dH, dg, dr, exact_sym, return_dweight=True)
    for i in (0, 2, 3):                                    # dconv1, dD, dB: stored without atomics
        assert torch.equal(a[i], b[i]) and torch.equal(a[i], c[i]), i
    for i in (1, 4, 5, 6):                                 # dconv2, dR, dT, dW: atomics
        assert rel_fro(b[i], a[i]) < 1e-6, i
    assert torch.equal(b[7], c[7]) and bool(torch.isfinite(b[7]).all())
    # the per-pair weighted backward on the replicated layout, every frame's dH depth block set to frame 0's
    rH = dH.clone().reshape(nw, nf, P, P)
    rH[:, :, 6:, 6:] = rH[:, :1, 6:, 6:]
    fsum = lambda t: t.reshape(nw, nf, *t.shape[1:]).sum(1)
    for w in (ones, _rand_w(nb, N, seed=7)):
        key, rep = _levels(sc, nw, nf, weight=w)
        k = ops.lm_keyframe_build_bwd(key, R, T, W, dH, dg, dr, exact_sym, return_dweight=True)
        r = ops.lm_build_bwd(rep, R, T, W.repeat_interleave(nf, 0).contiguous(), rH.reshape(nb, P, P), dg, dr, exact_sym, return_dweight=True)
        e = (rel_fro(k[0], fsum(r[0])), rel_fro(k[1], r[1]), rel_fro(k[2], fsum(r[2])), rel_fro(k[3], fsum(r[3])), rel_fro(k[4], r[4]),
             rel_fro(k[5], r[5]), rel_fro(k[6], fsum(r[6])), rel_fro(k[7], r[7]))
        print("weighted keyframe backward vs per-pair: " + " ".join(f"{n} {v:.1e}" for n, v in zip(("conv1", "conv2", "D", "B", "R", "T", "W", "weight"), e)))
        assert max(e) < 1e-5


def _grad_case(nw, nf, C, K, n_points, seed):
    sc = scene_case(nb=nw * nf, C=C, K=K, level_ids=(3,), seed=seed, n_points=n_points, dtype=F64, shared_depth=True, window_frames=nf)
    lv = sc.levels[0]
    a = oracle_level_inputs(lv)
    W = sc.W0.reshape(nw, nf, K, 1)[:, 0].double() + 0.01 * torch.randn(nw, K, 1, generator=torch.Generator().manual_seed(3), dtype=F64)
    g = torch.Generator().manual_seed(5)
    c = (torch.randn(nw * nf, 3, 3, generator=g, dtype=F64), torch.randn(nw * nf, 3, 1, generator=g, dtype=F64), torch.randn(nw, K, 1, generator=g, dtype=F64))
    return sc, lv, a, W, c


@gpu
@pytest.mark.parametrize("exact_sym", [True, False])
@pytest.mark.parametrize("wframes", ["nf", "1"])
@pytest.mark.parametrize("form", ["keyframe", "pairs"])
def test_window_iteration_gradients_with_weights_match_float64_autograd(form, wframes, exact_sym):
    """window_batch_iteration_fused with a weight that requires grad against float64 autograd of the weighted window statement: every input
    at exact_sym = True (the true adjoint), the weight at both (its gradient is the same in both conventions)."""
    from banet_b200 import autograd as AG
    _lib.require_device()
    nw, nf, C, K, lam = 2, 3, 8, 5, 0.4
    sc, lv, a, W, (cR, cT, cW) = _grad_case(nw, nf, C, K, 400, seed=71)
    N = lv.N
    fw = nf if wframes == "nf" else 1
    w0 = 0.5 + torch.rand(nw, fw, N, 1, generator=torch.Generator().manual_seed(9), dtype=F64)
    kf64 = lambda t: t.reshape(nw, nf, *t.shape[1:])[:, 0].clone().requires_grad_()
    o = {n: kf64(a[n]) for n in ("conv1", "D", "B")}
    o["conv2"] = a["conv2"].clone().requires_grad_()
    o["weight"] = w0.clone().requires_grad_()
    R = sc.R0.double().clone().requires_grad_(); T = sc.T0.double().clone().requires_grad_(); W64 = W.clone().requires_grad_()
    opts = O.IterOptions(l2_regularizer_base=1000.0, guard_nonfinite=True, lambda_override=torch.tensor([lam], dtype=F64))
    oR, oT, oW = [], [], []
    for w in range(nw):
        s = slice(w * nf, (w + 1) * nf)
        ex = lambda t: t[w:w + 1].expand(nf, *t.shape[1:])
        p_key = a["p"].reshape(nw, nf, *a["p"].shape[1:])[w, :1].expand(nf, *a["p"].shape[1:])
        r = WWO.window_iteration(ex(o["conv1"]), o["conv2"][s], a["fx"][s], a["fy"][s], a["ox"][s], a["oy"][s], p_key, ex(o["D"]), ex(o["B"]),
                                 R[s], T[s], W64[w], [], o["weight"][w].expand(nf, N, 1), opts)
        oR.append(r[0]); oT.append(r[1]); oW.append(r[2])
    oR, oT, oW = torch.cat(oR), torch.cat(oT), torch.stack(oW)
    ((oR * cR).sum() + (oT * cT).sum() + (oW * cW).sum()).backward()
    kf = lambda t: to_cuda32(t.reshape(nw, nf, *t.shape[1:])[:, 0])
    once = form == "keyframe"
    t = {n: (kf(a[n]) if once else kf(a[n]).unsqueeze(1).repeat(1, nf, *[1] * (a[n].dim() - 1))).requires_grad_() for n in ("conv1", "D", "B")}
    t["conv2"] = to_cuda32(a["conv2"]).reshape(nw, nf, *a["conv2"].shape[1:]).requires_grad_()
    t["weight"] = to_cuda32(w0).requires_grad_()
    Rg = to_cuda32(sc.R0).reshape(nw, nf, 3, 3).requires_grad_(); Tg = to_cuda32(sc.T0).reshape(nw, nf, 3, 1).requires_grad_()
    Wg = to_cuda32(W).requires_grad_()
    p = kf(lv.p) if once else kf(lv.p).unsqueeze(1)
    gR, gT, gW, status = AG.window_batch_iteration_fused(t["conv1"], t["conv2"], to_cuda32(lv.intr).reshape(nw, nf, 4), p, t["D"], t["B"], Rg, Tg, Wg, [],
                                                         1000.0, exact_sym=exact_sym, lambda_override=torch.full((nw,), lam, device="cuda"),
                                                         return_status=True, weight=t["weight"])
    assert int(status.abs().max()) == 0
    e = (rel_fro(gR.reshape(oR.shape), oR), rel_fro(gT.reshape(oT.shape), oT), rel_fro(gW, oW))
    print(f"{form} weight [nw,{wframes},N,1]: outputs R {e[0]:.1e} T {e[1]:.1e} W {e[2]:.1e}")
    assert e[0] < 1e-5 and e[1] < 1e-4 and e[2] < 1e-3
    ((gR * to_cuda32(cR).reshape(gR.shape)).sum() + (gT * to_cuda32(cT).reshape(gT.shape)).sum() + (gW * to_cuda32(cW)).sum()).backward()
    got = dict(t, R=Rg, T=Tg, W=Wg)
    want = dict(o, R=R, T=T, W=W64)
    for n in (["conv1", "conv2", "D", "B", "R", "T", "W", "weight"] if exact_sym else ["weight"]):
        g = got[n].grad.sum(1) if (not once and n in ("conv1", "D", "B")) else got[n].grad     # the per-frame copies' gradients, summed
        err = rel_fro(g.reshape(want[n].grad.shape), want[n].grad)
        print(f"  exact_sym={exact_sym} grad {n}: {err:.2e}")
        assert err < 2e-3, n


def _run_case(nw, nf, C, K, iters, seed=41):
    sc = scene_case(nb=nw * nf, H=96, W=128, C=C, K=K, level_ids=(2, 3), seed=seed, dtype=F64, shared_depth=True, window_frames=nf)
    ws = [0.5 + torch.rand(nw * nf, l.N, 1, generator=torch.Generator().manual_seed(l.level), dtype=F64) for l in sc.levels]
    mlps = [mlp_for(C, l.level) for l in sc.levels]
    oR, oT, oW = [], [], []
    for w in range(nw):
        s = slice(w * nf, (w + 1) * nf)
        olv = []
        for l, m in zip(sc.levels, mlps):
            a = oracle_level_inputs(l)
            kf = lambda t: t[w * nf:w * nf + 1].expand(nf, *t.shape[1:])
            olv.append(O.LevelInputs(kf(a["conv1"]), a["conv2"][s], a["fx"][s], a["fy"][s], a["ox"][s], a["oy"][s], kf(a["p"]), kf(a["D"]), kf(a["B"]), m))
        r = WWO.window_solve(olv, [x[s] for x in ws], iters, sc.R0[s], sc.T0[s], sc.W0[w * nf], O.IterOptions(l2_regularizer_base=1000.0))
        oR.append(r[0]); oT.append(r[1]); oW.append(r[2])
    return sc, ws, mlps, (torch.cat(oR), torch.cat(oT), torch.stack(oW))


@gpu
def test_weighted_window_runs_match_the_float64_statement():
    from banet_b200 import ops
    _lib.require_device()
    nw, nf, C, K, iters = 2, 3, 16, 16, 3
    sc, ws, mlps, (oR, oT, oW) = _run_case(nw, nf, C, K, iters)
    packed = [ops.pack_mlp([(w.float(), b.float()) for w, b in m]).cuda() for m in mlps]
    R0, T0 = to_cuda32(sc.R0), to_cuda32(sc.T0)
    W0 = to_cuda32(sc.W0.reshape(nw, nf, K, 1)[:, 0])
    cuda = lambda l: dataclasses.replace(l, **{k: to_cuda32(getattr(l, k)) for k in ("conv1", "conv2", "intr", "p", "D", "B")})
    cl = [_levels(sc, nw, nf, lv=cuda(l), weight=to_cuda32(w)) for l, w in zip(sc.levels, ws)]
    cl0 = [_levels(sc, nw, nf, lv=cuda(l)) for l in sc.levels]
    runs = {"keyframe_run": lambda i: ops.lm_keyframe_run([k for k, _ in i], iters, R0, T0, W0, mlp_packed=packed, l2_regularizer_base=1000.0),
            "window_batch_run": lambda i: ops.lm_window_batch_run([r for _, r in i], nw, iters, R0, T0, W0, mlp_packed=packed, l2_regularizer_base=1000.0,
                                                                  precision=_lib.PREC_FP32_SIMT)}
    for name, fn in runs.items():
        R, T, Wn, st = fn(cl)
        R_, _, W_, _ = fn(cl0)
        assert int(st.abs().max()) == 0
        e = (rel_fro(R, oR), rel_fro(T, oT), rel_fro(Wn, oW))
        print(f"{name} with weights vs float64 statement: R {e[0]:.1e} T {e[1]:.1e} W {e[2]:.1e}; unweighted differs by {rel_fro(Wn, W_):.1e}")
        assert e[0] < 1e-5 and e[1] < 1e-4 and e[2] < 2e-4
        assert rel_fro(Wn, W_) > 1e-3                     # the weights act
    # lm_window_run (one window, nf > 1): window 0
    s = slice(0, nf)
    lv0 = [ops.Level(r.conv1[s], r.conv2[s], r.intr[s], r.p[s], r.D[s], r.B[s], weight=r.weight[s]) for _, r in cl]
    R, T, Wn, st = ops.lm_window_run(lv0, iters, R0[s], T0[s], W0[0], mlp_packed=packed, l2_regularizer_base=1000.0, precision=_lib.PREC_FP32_SIMT)
    assert int(st.abs().max()) == 0
    e = (rel_fro(R, oR[s]), rel_fro(T, oT[s]), rel_fro(Wn, oW[0]))
    _, _, Wb, _ = runs["window_batch_run"](cl)
    lu = [ops.Level(r.conv1[s], r.conv2[s], r.intr[s], r.p[s], r.D[s], r.B[s]) for _, r in cl0]
    _, _, Wu, _ = ops.lm_window_run(lu, iters, R0[s], T0[s], W0[0], mlp_packed=packed, l2_regularizer_base=1000.0, precision=_lib.PREC_FP32_SIMT)
    _, _, Wub, _ = runs["window_batch_run"](cl0)
    print(f"window_run with weights vs float64 statement: R {e[0]:.1e} T {e[1]:.1e} W {e[2]:.1e}; vs the batch run's window 0 "
          f"{rel_fro(Wn, Wb[0]):.1e}; unweighted window_run vs unweighted batch run {rel_fro(Wu, Wub[0]):.1e}")
    # W of window 0 alone is small against its fp32 rounding (the batch run's window 0 is as far from the float64 statement); the dense
    # window step and the block-arrow step are the same maths, and the batch run is held to the statement above
    assert e[0] < 1e-5 and e[1] < 1e-4 and rel_fro(Wn, Wb[0]) < 1e-5 and rel_fro(Wb[0], oW[0]) > 10 * rel_fro(Wn, Wb[0])
    assert rel_fro(Wn, Wu) > 1e-3


def _net(C, levels=("3",)):
    from banet_b200.bundlenet import BundleNet
    net = BundleNet(C, levels=levels, exact_sym_grad=True, precision=_lib.PREC_FP32_SIMT, strict_status=True).cuda()
    for lv in levels:
        for i, (w, b) in enumerate(mlp_for(C, lv)):
            getattr(net, f"lambda_{lv}_{i + 1}_filters").data.copy_(w); getattr(net, f"lambda_{lv}_{i + 1}_biases").data.copy_(b)
    return net


@gpu
def test_window_iteration_with_weights_grad_and_no_grad_paths_agree():
    _lib.require_device()
    nw, nf, C, K = 2, 3, 8, 5
    sc = _gscene(nw, nf, C, K, n_points=500, seed=91)
    lv = sc.levels[0]
    kf = lambda t: t.reshape(nw, nf, *t.shape[1:])[:, 0].contiguous()
    fr = lambda t: t.reshape(nw, nf, *t.shape[1:])
    x = dict(conv1=kf(lv.conv1), conv2=fr(lv.conv2), p=kf(lv.p), D=kf(lv.D), B=kf(lv.B), R=fr(sc.R0), T=fr(sc.T0),
             W=sc.W0.reshape(nw, nf, K, 1)[:, 0] + 0.01)
    intr = [fr(t) for t in lv.intr_tiled()]
    w = 0.5 + torch.rand(nw, nf, lv.N, 1, generator=torch.Generator().manual_seed(2)).cuda()
    net = _net(C)
    call = lambda d, weight: net.WindowIteration(d["conv1"], d["conv2"], *d["intr"], d["p"], d["D"], d["B"], d["R"], d["T"], d["W"], 1000.0, "3",
                                                 weight=weight)
    one = lambda t: t[0]
    forms = {"keyframe": dict(x, intr=intr),
             "pairs": dict(x, intr=intr, **{k: x[k].unsqueeze(1) for k in ("conv1", "p", "D", "B")}),
             "single": dict(conv1=x["conv1"][:1], conv2=one(x["conv2"]), intr=[one(t) for t in intr], p=x["p"][:1], D=x["D"][:1], B=x["B"][:1],
                            R=one(x["R"]), T=one(x["T"]), W=one(x["W"]))}
    for name, d in forms.items():
        wt = w[0] if name == "single" else w
        with torch.no_grad():
            a = call(d, wt)
            a0 = call(d, None)
        b = call(d, wt.clone().requires_grad_())
        assert all(t.requires_grad for t in b), name
        for u, v, u0 in zip(a, b, a0):
            assert rel_fro(u, v.detach()) < 1e-5, name
        assert rel_fro(a[2], a0[2]) > 1e-4, name              # the weights act
        sum(t.sum() for t in b).backward()
        with torch.no_grad():                                   # weights of ones: the unweighted bits on the no-grad path
            c = call(d, torch.ones_like(wt[:, :1] if name != "single" else wt[:1]))
        for u, v in zip(a0, c):
            assert torch.equal(u, v), name


def _resize_inputs(nw, nf, C, K, n_points, seed):
    from banet_b200 import synth
    sc = synth.make_window_resize_scene(nw, nf, C, K, n_points=n_points, seed=seed)
    x = dict(intr=to_cuda32(sc.intrisic), key=[to_cuda32(l) for l in sc.key_layers], frames=[to_cuda32(l) for l in sc.frame_layers],
             points=to_cuda32(sc.points), basis=to_cuda32(sc.basis), depth=to_cuda32(sc.init_depth), R0=to_cuda32(sc.R0), T0=to_cuda32(sc.T0))
    return sc, x


def _resize_call(net, x, weight=None, **over):
    x = {**x, **over}
    return net.WindowResize(x["intr"], x["key"], x["frames"], x["points"], x["basis"], x["depth"], x["R0"], x["T0"], weight=weight)


@gpu
def test_window_resize_with_weights_matches_the_float64_statement():
    _lib.require_device()
    nw, nf, C, K = 2, 3, 8, 5
    sc, x = _resize_inputs(nw, nf, C, K, 400, seed=31)
    N = sc.points.shape[1]
    w64 = 0.5 + torch.rand(nw, nf, N, 1, generator=torch.Generator().manual_seed(3), dtype=F64)
    f = lambda t: t.to(F64).clone().requires_grad_()
    o = dict(key=[f(l) for l in sc.key_layers], frames=[f(l) for l in sc.frame_layers], basis=f(sc.basis), R0=f(sc.R0), T0=f(sc.T0), weight=w64.clone().requires_grad_())
    mlps = {str(l): [(w.clone(), b.clone()) for w, b in mlp_for(C, l)] for l in (2, 3)}
    oR, oT, oD = WWO.window_resize(sc.intrisic.to(F64), o["key"], o["frames"], sc.points.to(F64), o["basis"], sc.init_depth.to(F64), mlps,
                                   o["R0"], o["T0"], o["weight"], O.IterOptions(guard_nonfinite=True))
    net = _net(C, levels=("2", "3"))
    with torch.no_grad():
        Rs, Ts, Ds = _resize_call(net, x, to_cuda32(w64))
        U = _resize_call(net, x)
        ones = _resize_call(net, x, torch.ones(nw, 1, N, 1, device="cuda"))
    for i in range(2):
        e = (rel_fro(Rs[i], oR[i]), rel_fro(Ts[i], oT[i]), rel_fro(Ds[i], oD[i]))
        print(f"WindowResize inference with weights, level {i + 2} vs float64: R {e[0]:.1e} T {e[1]:.1e} depth {e[2]:.1e}")
        assert e[0] < 1e-5 and e[1] < 1e-4 and e[2] < 2e-4
        for u, v in zip(U, ones):
            assert torch.equal(u[i], v[i])
    assert rel_fro(Ds[1], U[2][1]) > 1e-6
    # training: outputs and gradients (the weight's included) against float64 autograd
    g = torch.Generator().manual_seed(4)
    cs = [(torch.randn(nw, nf, 3, 3, generator=g, dtype=F64), torch.randn(nw, nf, 3, 1, generator=g, dtype=F64),
           torch.randn(nw, 128, 160, 1, generator=g, dtype=F64)) for _ in range(2)]
    loss = lambda R, T, D, cv: sum((R[i] * cv(c[0])).sum() + (T[i] * cv(c[1])).sum() + 1e-2 * (D[i] * cv(c[2])).sum() for i, c in enumerate(cs))
    loss(oR, oT, oD, lambda c: c).backward()
    xl = {**x, "key": [l.clone().requires_grad_() for l in x["key"]], "frames": [l.clone().requires_grad_() for l in x["frames"]],
          "basis": x["basis"].clone().requires_grad_(), "R0": x["R0"].clone().requires_grad_(), "T0": x["T0"].clone().requires_grad_()}
    wg = to_cuda32(w64).requires_grad_()
    Rt, Tt, Dt = _resize_call(net, xl, wg)
    for i in range(2):
        assert rel_fro(Rt[i], oR[i]) < 1e-5 and rel_fro(Tt[i], oT[i]) < 1e-4 and rel_fro(Dt[i], oD[i]) < 2e-4
    loss(Rt, Tt, Dt, to_cuda32).backward()
    pairs = [("weight", wg, o["weight"]), ("basis", xl["basis"], o["basis"]), ("init_rotation", xl["R0"], o["R0"])]
    pairs += [(f"key_layers[{l}]", xl["key"][l], o["key"][l]) for l in (2, 3)] + [(f"frame_layers[{l}]", xl["frames"][l], o["frames"][l]) for l in (2, 3)]
    for name, t, r in pairs:
        err = rel_fro(t.grad, r.grad)
        print(f"WindowResize grad {name}: {err:.2e}")
        assert err < 2e-3, name


@gpu
def test_weight_shape_and_dtype_errors_name_the_argument():
    from banet_b200 import ops, autograd as AG
    _lib.require_device()
    nw, nf, C, K = 2, 3, 8, 5
    sc = _gscene(nw, nf, C, K, n_points=300, seed=43)
    N = sc.levels[0].N
    R, T, W = _start(sc, nw, nf, K)
    for bad in (torch.ones(nw * nf, N, 1, device="cuda", dtype=F64), torch.ones(nw * nf, N, device="cuda"), torch.ones(nw, N, 1, device="cuda")):
        with pytest.raises(_lib.BanetError, match="weight"):
            ops.lm_keyframe_build(_levels(sc, nw, nf, weight=bad)[0], R, T, W)
    key, _ = _levels(sc, nw, nf)
    args = (key.conv1, key.conv2.reshape(nw, nf, *key.conv2.shape[1:]), key.intr.reshape(nw, nf, 4), key.p, key.D, key.B,
            R.reshape(nw, nf, 3, 3), T.reshape(nw, nf, 3, 1), W, [], 1000.0)
    for bad in (torch.ones(nw, nf, N, 1, device="cuda", dtype=torch.bfloat16), torch.ones(nw, 2, N, 1, device="cuda"), torch.ones(nw * nf, N, 1, device="cuda")):
        with pytest.raises(_lib.BanetError, match="weight"):
            AG.window_batch_iteration_fused(*args, lambda_override=torch.full((nw,), 0.5, device="cuda"), weight=bad)
    _, x = _resize_inputs(nw, nf, C, K, 300, seed=43)
    net = _net(C, levels=("2", "3"))
    with torch.no_grad(), pytest.raises(_lib.BanetError, match="weight"):
        _resize_call(net, x, torch.ones(nw, nf, x["points"].shape[1] + 1, 1, device="cuda"))
    with torch.no_grad(), pytest.raises(_lib.BanetError, match="weight"):
        _resize_call(net, x, torch.ones(nw, nf, x["points"].shape[1], 1, device="cuda", dtype=F64))
