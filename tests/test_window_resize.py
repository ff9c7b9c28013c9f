"""BundleNet.WindowResize: BundleResize's coarse-to-fine schedule (reference bundlenet.py:332-399) for keyframe windows.  On the CPU the float64
statement of the schedule (tests/window_resize_oracle.py) is tied to oracle.bundle_resize and shown to move towards a planted solution; on the
GPU the inference and training paths are compared with it, with BundleResize and with each other, and their memory and error paths are pinned."""
import pytest
import torch

from helpers import O, mlp_for, rel_fro, to_cuda32
from window_resize_oracle import window_resize

F64 = torch.float64


# ------------------------------------------------------------------------------------------ CPU
def test_window_resize_oracle_with_one_frame_is_bundle_resize():
    """nf = 1, nw = nb/2: window w is pair w of bundle_resize (keyframe = image w, frame = image w + nb/2, the half swap of :386)."""
    import gen_golden as GG
    nb = 4
    x = GG.resize_inputs(seed=24, nb=nb, C=4, K=3, N=500)
    mlps = {str(l): GG.mlp_for(4, l) for l in range(4)}
    Rs, Ts, Ds = O.bundle_resize(x["intr"], x["layers"], x["points"], x["basis"], x["depth"], mlps, x["R0"], x["T0"])
    h = nb // 2
    wR, wT, wD = window_resize(x["intr"][:h], [l[:h] for l in x["layers"]], [l[h:].unsqueeze(1) for l in x["layers"]], x["points"][:h],
                               x["basis"][:h], x["depth"][:h], mlps, x["R0"][:h].unsqueeze(1), x["T0"][:h].unsqueeze(1))
    for i in range(2):
        e = (rel_fro(wR[i][:, 0], Rs[i][:h]), rel_fro(wT[i][:, 0], Ts[i][:h]), rel_fro(wD[i], Ds[i][:h]))
        print(f"level {i + 2}: R {e[0]:.1e} T {e[1]:.1e} depth {e[2]:.1e}")
        assert max(e) < 1e-12


def _angle(Ra, Rb):
    c = ((Ra.transpose(-1, -2) @ Rb).diagonal(dim1=-2, dim2=-1).sum(-1) - 1.0) / 2.0
    return float(torch.arccos(c.clamp(-1.0, 1.0)).norm())


def test_window_resize_oracle_moves_towards_the_planted_solution():
    """A motion of a quarter degree and a fixed small lambda: one iteration per level converges; the untrained lambda-MLP times
    l2_regularizer_base = 1000 damps the step to almost nothing."""
    from banet_b200 import synth
    nw, nf, C, K = 2, 3, 8, 4
    sc = synth.make_window_resize_scene(nw, nf, C, K, n_points=600, seed=5, dtype=F64, rot_deg=0.25, start_trans_noise_m=0.005)
    Rs, Ts, Ds = window_resize(sc.intrisic, sc.key_layers, sc.frame_layers, sc.points, sc.basis, sc.init_depth, {"2": [], "3": []}, sc.R0, sc.T0,
                               O.IterOptions(guard_nonfinite=True, lambda_override=torch.tensor([0.01], dtype=F64)))
    Dtrue = sc.init_depth + (sc.basis.reshape(nw, -1, K) @ sc.W_true).reshape(sc.init_depth.shape)
    eR = [_angle(sc.R0, sc.R_true)] + [_angle(R, sc.R_true) for R in Rs]
    eT = [float((sc.T0 - sc.T_true).norm())] + [float((T - sc.T_true).norm()) for T in Ts]
    eD = [float((sc.init_depth - Dtrue).norm())] + [float((D - Dtrue).norm()) for D in Ds]   # B (W - W*): the error in W, through the basis
    print(f"start / level 2 / level 3: R {eR}  T {eT}  depth {eD}")
    for e in (eR, eT, eD):
        assert e[2] < e[1] < e[0]


# ------------------------------------------------------------------------------------------ GPU
def _scene(nw, nf, C, K, n_points, seed=17):
    from banet_b200 import synth
    return synth.make_window_resize_scene(nw, nf, C, K, n_points=n_points, seed=seed)


def _cuda(sc):
    return dict(intr=to_cuda32(sc.intrisic), key=[to_cuda32(l) for l in sc.key_layers], frames=[to_cuda32(l) for l in sc.frame_layers],
                points=to_cuda32(sc.points), basis=to_cuda32(sc.basis), depth=to_cuda32(sc.init_depth), R0=to_cuda32(sc.R0), T0=to_cuda32(sc.T0))


def _net(C, precision=None, strict=True):
    from banet_b200.bundlenet import BundleNet
    from banet_b200 import _lib
    net = BundleNet(C, levels=("2", "3"), exact_sym_grad=True, precision=_lib.PREC_FP32_SIMT if precision is None else precision,
                    strict_status=strict).cuda()
    for lv in (2, 3):
        for i, (w, b) in enumerate(mlp_for(C, lv)):
            getattr(net, f"lambda_{lv}_{i + 1}_filters").data.copy_(w); getattr(net, f"lambda_{lv}_{i + 1}_biases").data.copy_(b)
    return net


def _call(net, x, **over):
    x = {**x, **over}
    return net.WindowResize(x["intr"], x["key"], x["frames"], x["points"], x["basis"], x["depth"], x["R0"], x["T0"])


def _oracle(sc, leaves=None):
    """window_resize in float64 on the scene's (float32) values; leaves: name -> float64 leaf tensors to use instead."""
    d = dict(intr=sc.intrisic.to(F64), key=[l.to(F64) for l in sc.key_layers], frames=[l.to(F64) for l in sc.frame_layers],
             points=sc.points.to(F64), basis=sc.basis.to(F64), depth=sc.init_depth.to(F64), R0=sc.R0.to(F64), T0=sc.T0.to(F64),
             mlps={str(l): mlp_for(sc.key_layers[0].shape[-1], l) for l in (2, 3)})
    d.update(leaves or {})
    return window_resize(d["intr"], d["key"], d["frames"], d["points"], d["basis"], d["depth"], d["mlps"], d["R0"], d["T0"],
                         O.IterOptions(guard_nonfinite=True))


@pytest.mark.gpu
@pytest.mark.parametrize("C,K,n_points", [(8, 8, 512), (128, 128, 1024)])
def test_window_resize_inference_matches_the_oracle(C, K, n_points):
    from banet_b200 import _lib
    _lib.require_device()
    nw, nf = 2, 4
    sc = _scene(nw, nf, C, K, n_points)
    oR, oT, oD = _oracle(sc)
    net = _net(C, precision=_lib.PREC_AUTO)
    with torch.no_grad():
        Rs, Ts, Ds = _call(net, _cuda(sc))
    assert tuple(net.last_status.shape) == (nw, nf) and int(net.last_status.abs().max()) == 0
    for i in range(2):
        assert tuple(Rs[i].shape) == (nw, nf, 3, 3) and tuple(Ts[i].shape) == (nw, nf, 3, 1) and tuple(Ds[i].shape) == (nw, 128, 160, 1)
        e = (rel_fro(Rs[i], oR[i]), rel_fro(Ts[i], oT[i]), rel_fro(Ds[i], oD[i]))
        print(f"C={C} K={K} N={n_points} level {i + 2} vs oracle: R {e[0]:.1e} T {e[1]:.1e} depth {e[2]:.1e}")
        assert e[0] < 1e-5 and e[1] < 1e-4 and e[2] < 2e-4


@pytest.mark.gpu
def test_window_resize_with_one_frame_agrees_with_bundle_resize():
    from banet_b200 import _lib
    _lib.require_device()
    nw, C, K = 3, 16, 16
    x = _cuda(_scene(nw, 1, C, K, 800, seed=23))
    net = _net(C, strict=False)
    with torch.no_grad():
        Rs, Ts, Ds = _call(net, x)
        assert int(net.last_status.abs().max()) == 0
        two = lambda t: torch.cat([t, t], 0)                         # pairs nw.. are the reverse pairs of BundleResize's half swap
        layers = [torch.cat([k, f[:, 0]], 0) for k, f in zip(x["key"], x["frames"])]
        bR, bT, bD = net.BundleResize(two(x["intr"]), layers, two(x["points"]), two(x["basis"]), two(x["depth"]), two(x["R0"][:, 0]),
                                      two(x["T0"][:, 0]))
    for i in range(2):
        e = (rel_fro(Rs[i][:, 0], bR[i][:nw]), rel_fro(Ts[i][:, 0], bT[i][:nw]), rel_fro(Ds[i], bD[i][:nw]))
        print(f"level {i + 2} vs BundleResize: R {e[0]:.1e} T {e[1]:.1e} depth {e[2]:.1e}")
        assert e[0] < 1e-5 and e[1] < 1e-4 and e[2] < 1e-4


def _leaves(x):
    return {**x, "key": [l.clone().requires_grad_() for l in x["key"]], "frames": [l.clone().requires_grad_() for l in x["frames"]],
            "basis": x["basis"].clone().requires_grad_(), "depth": x["depth"].clone().requires_grad_(), "R0": x["R0"].clone().requires_grad_(),
            "T0": x["T0"].clone().requires_grad_()}


@pytest.mark.gpu
def test_window_resize_training_outputs_are_the_inference_outputs():
    from banet_b200 import _lib
    _lib.require_device()
    nw, nf, C, K = 2, 4, 32, 32
    x = _cuda(_scene(nw, nf, C, K, 512, seed=29))
    net = _net(C)
    with torch.no_grad():
        a = _call(net, x)
    b = _call(net, _leaves(x))
    for i in range(2):
        assert all(t[i].requires_grad for t in b) and not any(t[i].requires_grad for t in a)
        e = [rel_fro(u[i], v[i].detach()) for u, v in zip(a, b)]
        print(f"level {i + 2} training vs inference: R {e[0]:.1e} T {e[1]:.1e} depth {e[2]:.1e}")
        assert e[0] < 1e-5 and e[1] < 1e-4 and e[2] < 1e-4


@pytest.mark.gpu
def test_window_resize_gradients_match_oracle_autograd():
    from banet_b200 import _lib
    _lib.require_device()
    nw, nf, C, K = 2, 3, 8, 5
    sc = _scene(nw, nf, C, K, 400, seed=31)
    f = lambda t: t.to(F64).clone().requires_grad_()
    o = dict(key=[f(l) for l in sc.key_layers], frames=[f(l) for l in sc.frame_layers], basis=f(sc.basis), R0=f(sc.R0), T0=f(sc.T0),
             mlps={str(l): [(w.clone().requires_grad_(), b.clone().requires_grad_()) for w, b in mlp_for(C, l)] for l in (2, 3)})
    oR, oT, oD = _oracle(sc, o)
    g = torch.Generator().manual_seed(4)
    cs = [(torch.randn(nw, nf, 3, 3, generator=g, dtype=F64), torch.randn(nw, nf, 3, 1, generator=g, dtype=F64),
           torch.randn(nw, 128, 160, 1, generator=g, dtype=F64)) for _ in range(2)]
    loss = lambda R, T, D, cv: sum((R[i] * cv(c[0])).sum() + (T[i] * cv(c[1])).sum() + 1e-2 * (D[i] * cv(c[2])).sum() for i, c in enumerate(cs))
    loss(oR, oT, oD, lambda c: c).backward()
    net = _net(C)
    x = _leaves(_cuda(sc))
    Rs, Ts, Ds = _call(net, x)
    assert int(net.last_status.abs().max()) == 0
    for i in range(2):
        e = (rel_fro(Rs[i], oR[i]), rel_fro(Ts[i], oT[i]), rel_fro(Ds[i], oD[i]))
        print(f"level {i + 2} outputs vs oracle: R {e[0]:.1e} T {e[1]:.1e} depth {e[2]:.1e}")
    loss(Rs, Ts, Ds, to_cuda32).backward()
    tol = 2e-3
    pairs = [(f"key_layers[{l}]", x["key"][l], o["key"][l]) for l in (2, 3)] + [(f"frame_layers[{l}]", x["frames"][l], o["frames"][l]) for l in (2, 3)]
    pairs += [("basis", x["basis"], o["basis"]), ("init_rotation", x["R0"], o["R0"]), ("init_translation", x["T0"], o["T0"])]
    for lv in (2, 3):
        for i, (w, b) in enumerate(o["mlps"][str(lv)]):
            pairs.append((f"lambda_{lv}_{i + 1}_filters", getattr(net, f"lambda_{lv}_{i + 1}_filters"), w))
    for name, t, r in pairs:
        err = rel_fro(t.grad, r.grad)
        print(f"grad {name}: {err:.2e}")
        assert err < tol, name
    assert x["key"][0].grad is None and x["frames"][1].grad is None                   # levels 0, 1 are not used
    # init_depth: through the output depth only (:341 stop_gradient, :397), i.e. the sum of the depth outputs' upstream gradients
    ref = sum(1e-2 * to_cuda32(c[2]) for c in cs)
    assert rel_fro(x["depth"].grad, ref) < 1e-6


def _peak(fn):
    torch.cuda.synchronize(); torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn(); torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


@pytest.mark.gpu
def test_window_resize_memory_layout():
    """Training holds no per-frame copy of the keyframe; inference makes no [F2|gx|gy] tensor."""
    from banet_b200 import _lib
    _lib.require_device()
    nw, nf, C, K = 1, 8, 32, 32
    x = _cuda(_scene(nw, nf, C, K, 512, seed=37))
    net = _net(C)
    xl = _leaves(x)

    def window():
        Rs, Ts, Ds = _call(net, xl)
        sum(R.sum() + T.sum() + D.sum() for R, T, D in zip(Rs, Ts, Ds)).backward()

    rep = lambda t: t.repeat_interleave(nf, 0)
    two = lambda t: torch.cat([t, t], 0)
    layers = [torch.cat([rep(k), f.reshape(nw * nf, *f.shape[2:])], 0).requires_grad_() for k, f in zip(x["key"], x["frames"])]
    pair_args = [two(rep(x[n])) for n in ("intr", "points")] + [two(rep(x["basis"])).requires_grad_(), two(rep(x["depth"]))]
    R0, T0 = two(x["R0"].reshape(-1, 3, 3)).requires_grad_(), two(x["T0"].reshape(-1, 3, 1)).requires_grad_()

    def pairs():
        net.strict_status = False
        Rs, Ts, Ds = net.BundleResize(pair_args[0], layers, pair_args[1], pair_args[2], pair_args[3], R0, T0)
        sum(R.sum() + T.sum() + D.sum() for R, T, D in zip(Rs, Ts, Ds)).backward()
        net.strict_status = True

    pw, pp = _peak(window), _peak(pairs)
    print(f"training peak: WindowResize {pw / 2**20:.1f} MiB, BundleResize on repeated keyframes {pp / 2**20:.1f} MiB")
    assert pw < pp
    with torch.no_grad():
        pi = _peak(lambda: _call(net, x))
    h, w = x["frames"][3].shape[2:4]
    one3c = nw * nf * h * w * 3 * C * 4
    print(f"inference peak {pi / 2**20:.1f} MiB, one [nw*nf,h,w,3C] tensor {one3c / 2**20:.1f} MiB")
    assert pi < one3c


@pytest.mark.gpu
def test_window_resize_inference_is_reproducible():
    from banet_b200 import _lib
    _lib.require_device()
    x = _cuda(_scene(2, 4, 32, 64, 700, seed=41))
    net = _net(32)
    with torch.no_grad():
        a, b = _call(net, x), _call(net, x)
    for u, v in zip(a, b):
        for s, t in zip(u, v):
            assert torch.equal(s, t)


@pytest.mark.gpu
def test_window_resize_errors_and_status():
    from banet_b200 import _lib
    from banet_b200.bundlenet import BundleNet
    _lib.require_device()
    nw, nf, C, K = 2, 3, 8, 5
    x = _cuda(_scene(nw, nf, C, K, 300, seed=43))
    for prec in (_lib.PREC_TF32X1, _lib.PREC_TF32X3, _lib.PREC_TF32_LEVELWISE):
        with torch.no_grad(), pytest.raises(RuntimeError, match="tensor-core"):
            _call(_net(C, precision=prec), x)
    net = _net(C)
    bad = [("points", dict(points=x["points"][:1])), ("intrisic", dict(intr=x["intr"][:1])), ("basis", dict(basis=x["basis"][:1])),
           ("init_depth", dict(depth=x["depth"][:1])), (r"key_layers\[2\]", dict(key=[*x["key"][:2], x["key"][2][:1], x["key"][3]])),
           (r"frame_layers\[2\]", dict(frames=[*x["frames"][:2], x["frames"][2][:, :2], x["frames"][3]])),
           ("init_rotation", dict(R0=x["R0"][:, :2])), ("init_translation", dict(T0=x["T0"][:1]))]
    for name, over in bad:
        with torch.no_grad(), pytest.raises(_lib.BanetError, match=name):
            _call(net, x, **over)
    with pytest.raises(RuntimeError, match="vmatrix_batch_scramble"):
        BundleNet(C, vmatrix_batch_scramble=True).cuda().WindowResize(x["intr"], x["key"], x["frames"], x["points"], x["basis"], x["depth"])
    split = BundleNet(C, training_path="reference_split").cuda()
    with pytest.raises(RuntimeError, match="reference_split"):
        split.WindowResize(x["intr"], x["key"], x["frames"], x["points"], x["basis"], x["depth"], x["R0"], x["T0"])
    # window 1 with a zero basis: its depth block is exactly zero and the undamped last depth coefficient (:266) makes its system singular
    flat = x["basis"].clone()
    flat[1] = 0.0
    with torch.no_grad(), pytest.raises(RuntimeError, match="skipped"):
        _call(net, x, basis=flat)
    with pytest.raises(RuntimeError, match="skipped"):
        _call(net, _leaves(x), basis=flat.clone().requires_grad_())
    loose = _net(C, strict=False)
    with torch.no_grad():
        _call(loose, x, basis=flat)
        st = loose.last_status
        assert tuple(st.shape) == (nw, nf) and bool((st[1] != 0).all()) and int(st[0].abs().max()) == 0
        _call(loose, x)
        assert tuple(loose.last_status.shape) == (nw, nf) and int(loose.last_status.abs().max()) == 0
