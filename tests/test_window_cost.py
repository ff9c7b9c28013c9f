"""The feature-metric cost of keyframe windows (banet_lm_keyframe_cost / _bwd, ops.lm_keyframe_cost, autograd.window_feature_metric_cost,
BundleNet.WindowFeatureMetricCost, WindowResize(return_cost=True)): banet_lm_cost on the keyframe layout, the keyframe's tensors once per
window.  On the CPU: the C-ABI's and the Python layer's argument errors.  On the GPU: the forward against float64 (tests/cost_oracle.py on
the keyframe replicated per frame) and bit for bit against the pair cost on the replicated layout, the backward against float64 autograd
and the pair backward's frame sums, the descent identity against the keyframe build, batches past 65 535 pairs and the Python layers."""
import ctypes

import pytest
import torch

from helpers import O, scene_case, oracle_level_inputs, rel_fro, to_cuda32
import cost_oracle as CO
from banet_b200 import _lib

gpu = pytest.mark.gpu


def _klevel(nw=2, nf=4, N=4096, C=64, K=128, h=120, w=160, c2=None, ptr=1):
    return _lib.BanetKeyframeLevel(nw, nf, N, C, K, h, w, 3 * C if c2 is None else c2, ptr, ptr, ptr, ptr, ptr, ptr)


# ------------------------------------------------------------------------------------------ CPU
def test_keyframe_cost_entries_reject_bad_arguments_without_gpu():
    lib = _lib.load()
    err = lambda: lib.banet_last_error()
    p = 1                                                            # non-null dummy pointers: every check below fires before a CUDA call

    def fwd(lv, R=p, T=p, W=p, cost=p, nvalid=p, ws=p, nbytes=1 << 34):
        return lib.banet_lm_keyframe_cost(ctypes.byref(lv), R, T, W, cost, nvalid, None, None, ws, nbytes, None)

    def bwd(lv, **kw):
        a = dict(R=p, T=p, W=p, dcost=p, dconv1=p, dconv2=p, dD=p, dB=p, dR=p, dT=p, dW=p)
        a.update(kw)
        return lib.banet_lm_keyframe_cost_bwd(ctypes.byref(lv), a["R"], a["T"], a["W"], a["dcost"], a["dconv1"], a["dconv2"], a["dD"], a["dB"],
                                              a["dR"], a["dT"], a["dW"], None, None)

    ws = lambda lv: lib.banet_lm_keyframe_cost_workspace_bytes(ctypes.byref(lv))
    for k in ("R", "T", "W", "cost", "nvalid"):
        assert fwd(_klevel(), **{k: None}) == -1 and b"null" in err(), k
    for k in ("R", "T", "W", "dcost", "dconv1", "dconv2", "dD", "dB", "dR", "dT", "dW"):
        assert bwd(_klevel(), **{k: None}) == -1 and b"null" in err(), k
    for call in (fwd, bwd):
        assert call(_klevel(ptr=None)) == -1 and b"null" in err()
        for bad in (dict(nw=0), dict(nf=0), dict(N=0), dict(C=0), dict(K=0), dict(h=1), dict(w=1), dict(c2=100)):
            assert call(_klevel(**bad)) == -1, bad
        assert call(_klevel(K=257)) == -4 and b"K=257" in err()
        assert call(_klevel(C=4096)) == -4 and b"C=4096" in err()
    assert fwd(_klevel(), ws=None) == -2 and b"workspace" in err()
    need = ws(_klevel())
    assert need == 2 * 4 * 64 * 2 * 8                                 # one fp64 pair (cost, count) per (pair, 64-point tile)
    assert fwd(_klevel(), nbytes=need - 1) == -2 and b"workspace" in err()
    assert ws(_klevel(nf=16)) > ws(_klevel(nf=4)) and ws(_klevel(c2=64)) == need
    for bad in (dict(nw=0), dict(nf=0), dict(K=0), dict(K=257), dict(C=4096), dict(c2=100), dict(ptr=None)):
        assert ws(_klevel(**bad)) == 0, bad
    assert lib.banet_lm_keyframe_cost_workspace_bytes(None) == 0


def _cpu_window_args(nw=2, nf=3, N=10, C=4, K=3, h=6, w=8):
    z = lambda *s: torch.zeros(*s)
    return dict(conv1=z(nw, N, C), conv2=z(nw, nf, h, w, 3 * C), fx=z(nw, 1, 1), fy=z(nw, 1, 1), ox=z(nw, 1, 1), oy=z(nw, 1, 1), p=z(nw, 3, N),
                D=z(nw, N, 1), B=z(nw, N, K), R=torch.eye(3).expand(nw, nf, 3, 3).contiguous(), T=z(nw, nf, 3, 1), W=z(nw, K, 1))


def test_window_cost_rejects_bad_arguments_in_python_without_gpu():
    from banet_b200 import ops
    from banet_b200.bundlenet import BundleNet
    net = BundleNet(4, levels=("3",))
    a = _cpu_window_args()
    call = lambda **kw: net.WindowFeatureMetricCost(*[{**a, **kw}[k] for k in ("conv1", "conv2", "fx", "fy", "ox", "oy", "p", "D", "B", "R", "T", "W")],
                                                    weight=kw.get("weight"))
    bad = [(dict(conv1=a["conv1"].to(torch.bfloat16)), "conv1"), (dict(B=a["B"].double()), "B"), (dict(conv2=a["conv2"].half()), "conv2"),
           (dict(R=a["R"][0]), "R"), (dict(conv1=a["conv1"][:1]), "conv1"), (dict(B=a["B"][:, :5]), "B"), (dict(p=a["p"][:, :2]), "p"),
           (dict(D=a["D"][:, :, :0]), "D"), (dict(T=a["T"][:, :2]), "T"), (dict(W=a["W"][:, :2]), "W"), (dict(conv2=a["conv2"][..., :5]), "conv2"),
           (dict(conv2=a["conv2"][:, :2]), "conv2"), (dict(fx=torch.zeros(2, 2, 1), fy=torch.zeros(2, 2, 1), ox=torch.zeros(2, 2, 1), oy=torch.zeros(2, 2, 1)), "fx"), (dict(weight=torch.zeros(2, 2, 10, 1)), "weight"),
           (dict(weight=torch.zeros(2, 3, 10, 1).double()), "weight")]
    for kw, name in bad:
        with pytest.raises(_lib.BanetError, match=name):
            call(**kw)
    with pytest.raises(_lib.BanetError, match="CUDA"):                # shapes right: the kernel wrapper refuses CPU tensors
        call()
    lv = ops.KeyframeLevel(a["conv1"], a["conv2"].reshape(6, 6, 8, 12), torch.zeros(6, 4), a["p"], a["D"], a["B"])
    with pytest.raises(_lib.BanetError, match="CUDA"):
        ops.lm_keyframe_cost(lv, a["R"].reshape(6, 3, 3), a["T"].reshape(6, 3, 1), a["W"])


# ------------------------------------------------------------------------------------------ GPU
def _scene(nw, nf, C, K, n_points, seed):
    """Sparse: n_points keyframe points on the 120 x 160 map of level 3; dense (n_points None): the 60 x 80 grid of level 2."""
    return scene_case(nb=nw * nf, H=120, W=160, C=C, K=K, level_ids=(3,) if n_points else (2,), seed=seed, n_points=n_points, shared_depth=True,
                      window_frames=nf, dtype=torch.float32)


class Win:
    """A keyframe level on the GPU (frame 0's keyframe tensors once per window) and the same level replicated per pair."""

    def __init__(self, sc, nw, nf, layout="3c", weight=None):
        from banet_b200 import ops
        l = sc.levels[0]
        C, K = l.conv1.shape[2], l.B.shape[2]
        self.nw, self.nf, self.nb, self.N, self.C, self.K = nw, nf, nw * nf, l.conv1.shape[1], C, K
        k = lambda t: to_cuda32(t.reshape(nw, nf, *t.shape[1:])[:, 0])
        self.conv1, self.p, self.D, self.B = k(l.conv1), k(l.p), k(l.D), k(l.B)
        conv2 = to_cuda32(l.conv2)
        self.conv2 = conv2 if layout == "3c" else conv2[..., :C].contiguous()
        self.intr, self.weight = to_cuda32(l.intr), weight
        self.R, self.T = to_cuda32(sc.R0), to_cuda32(sc.T0)
        self.W = (to_cuda32(sc.W0.reshape(nw, nf, K, 1)[:, 0]) + 0.01 * torch.arange(1, nw + 1, device="cuda").reshape(nw, 1, 1)).contiguous()
        self.key = ops.KeyframeLevel(self.conv1, self.conv2, self.intr, self.p, self.D, self.B, weight=weight)
        r = lambda t: t.repeat_interleave(nf, 0).contiguous()
        self.rep = ops.Level(r(self.conv1), self.conv2, self.intr, r(self.p), r(self.D), r(self.B), weight=weight)
        self.Wrep = r(self.W)

    def oracle_cost(self, weight):
        a = {n: t.cpu().double() for n, t in (("conv1", self.rep.conv1), ("p", self.rep.p), ("D", self.rep.D), ("B", self.rep.B))}
        conv2 = self.conv2.cpu().double()
        fx, fy, ox, oy = [self.intr[:, i:i + 1].expand(self.nb, self.N).cpu().double() for i in range(4)]
        return CO.cost(a["conv1"], conv2, fx, fy, ox, oy, a["p"], a["D"], a["B"], self.R.cpu().double(), self.T.cpu().double(),
                       self.Wrep.cpu().double(), weight=None if weight is None else weight.cpu().double())


def _weights(nb, nf, N, seed):
    g = torch.Generator().manual_seed(seed)
    c = (0.5 + torch.rand(nb, N, 1, generator=g)).cuda()
    z = c.clone()
    z[min(1, nf - 1)::nf] = 0.0                                      # every window's frame 1 (frame 0 when nf = 1) weighs nothing
    return {"none": None, "random": c, "zero frame": z}


FWD_CASES = [(2, 1, 13, 1, 4096), (2, 3, 64, 16, 4096), (1, 16, 128, 128, 4096), (2, 3, 128, 200, 4096), (1, 3, 64, 256, 4096),
             (2, 3, 13, 16, None), (1, 16, 64, 128, None), (2, 1, 128, 256, None)]


@gpu
@pytest.mark.parametrize("nw,nf,C,K,n_points", FWD_CASES)
def test_forward_matches_float64_and_is_the_pair_cost_bit_for_bit(nw, nf, C, K, n_points, monkeypatch):
    from banet_b200 import ops
    _lib.require_device()
    sc = _scene(nw, nf, C, K, n_points, seed=301 + K + C + nf)
    worst = 0.0
    for wname, weight in _weights(nw * nf, nf, sc.levels[0].conv1.shape[1], seed=K + C).items():
        outs = {}
        for layout in ("3c", "f2"):
            x = Win(sc, nw, nf, layout, weight)
            out = ops.lm_keyframe_cost(x.key, x.R, x.T, x.W, per_point=True)
            rep = ops.lm_cost(x.rep, x.R, x.T, x.Wrep, per_point=True)
            for a, b in zip(out, rep):                                   # cost, nvalid, s, mask: the pair cost on the replicated layout
                assert torch.equal(a, b), (wname, layout)
            outs[layout] = out
            if layout == "3c":
                _, _, _, nvb = ops.lm_keyframe_build(x.key, x.R, x.T, x.W)
                assert torch.equal(out[1], nvb)                          # the keyframe build's nvalid
                ref = x.oracle_cost(weight)
                e = rel_fro(out[0].cpu().double(), ref)
                worst = max(worst, e)
                assert e < 2e-5, (wname, e)
                if wname == "zero frame":
                    assert not bool(out[0][min(1, nf - 1)::nf].any())
        for a, b in zip(outs["3c"], outs["f2"]):                         # the F2-only layout reads the same channels
            assert torch.equal(a, b), wname
    assert float(outs["3c"][1].min()) > 0
    # weights of ones are no weights; two differently poisoned workspaces give the same bits
    x = Win(sc, nw, nf, "f2", torch.ones(nw * nf, x.N, 1, device="cuda"))
    ones = ops.lm_keyframe_cost(x.key, x.R, x.T, x.W, per_point=True)
    x0 = Win(sc, nw, nf, "f2")
    plain = ops.lm_keyframe_cost(x0.key, x0.R, x0.T, x0.W, per_point=True)
    for a, b in zip(ones, plain):
        assert torch.equal(a, b)
    runs = []
    for fill in (0xFF, 0x7F):
        monkeypatch.setattr(ops, "_ws", lambda n, dev, f=fill: torch.full((max(int(n), 256),), f, dtype=torch.uint8, device=dev))
        runs.append(ops.lm_keyframe_cost(x0.key, x0.R, x0.T, x0.W, per_point=True))
        monkeypatch.undo()
    for a, b, c in zip(runs[0], runs[1], plain):
        assert torch.equal(a, b) and torch.equal(a, c)
    print(f"nw={nw} nf={nf} C={C} K={K} N={n_points}: largest relative error against float64 {worst:.1e}")


def _frame_sum(t, nw, nf):
    return t.reshape(nw, nf, *t.shape[1:]).sum(1)


@gpu
@pytest.mark.parametrize("layout", ["3c", "f2"])
@pytest.mark.parametrize("nw,nf", [(2, 3), (1, 20)])
def test_backward_matches_float64_autograd_and_the_pair_backward(nw, nf, layout):
    """nf = 20 walks the frames in two chunks (16 + 4)."""
    from banet_b200 import ops
    _lib.require_device()
    C, K = 8, 6
    sc = _scene(nw, nf, C, K, 400, seed=67 + nf)
    nb = nw * nf
    weight = (0.5 + torch.rand(nb, 400, 1, generator=torch.Generator().manual_seed(8))).cuda()
    # the sampler's coordinate derivative jumps at texel edges: a projection within fp32 rounding of one may take the other side than in
    # float64, so those (frame, point) pairs weigh nothing here (their s, and so dweight, stays continuous)
    x = Win(sc, nw, nf, layout, weight)
    a = oracle_level_inputs(sc.levels[0])
    Dt = x.rep.D.cpu().double() + x.rep.B.cpu().double() @ x.Wrep.cpu().double()
    _, _, _, _, px, py = O._warp(x.rep.p.cpu().double(), Dt, x.R.cpu().double(), x.T.cpu().double(), a["fx"], a["fy"], a["ox"], a["oy"])
    edge = ((px - px.round()).abs() < 1e-4) | ((py - py.round()).abs() < 1e-4)
    weight[edge.cuda().unsqueeze(-1)] = 0.0
    x = Win(sc, nw, nf, layout, weight)
    dcost = (torch.rand(nb, generator=torch.Generator().manual_seed(3)) - 0.5).cuda()
    got = ops.lm_keyframe_cost_bwd(x.key, x.R, x.T, x.W, dcost, return_dweight=True)
    names = ["conv1", "conv2", "D", "B", "R", "T", "W", "weight"]
    # float64 autograd at every leaf, the keyframe given once
    f64 = lambda t: t.detach().cpu().double().clone().requires_grad_()
    t = {n: f64(v) for n, v in (("conv1", x.conv1), ("conv2", x.conv2), ("D", x.D), ("B", x.B), ("R", x.R), ("T", x.T), ("W", x.W),
                                ("weight", weight))}
    rp = lambda v: v.repeat_interleave(nf, 0)
    conv2_o = t["conv2"] if layout == "3c" else torch.cat([t["conv2"], O.grad_fixed(t["conv2"])], dim=-1)
    fx, fy, ox, oy = [x.intr[:, i:i + 1].expand(nb, x.N).cpu().double() for i in range(4)]
    ref = CO.cost(rp(t["conv1"]), conv2_o, fx, fy, ox, oy, rp(x.p.cpu().double()), rp(t["D"]), rp(t["B"]), t["R"], t["T"], rp(t["W"]),
                  weight=t["weight"])
    (ref * dcost.cpu().double()).sum().backward()
    for n, g in zip(names, got):
        e = rel_fro(g.cpu().double(), t[n].grad)
        print(f"  d{n}: {e:.2e} against float64")
        assert e < 2e-4, n
    if layout == "3c":
        assert not bool(got[1][..., C:].any())
    # the pair backward on the replicated layout, the keyframe's gradients summed over the frames
    pr = ops.lm_cost_bwd(x.rep, x.R, x.T, x.Wrep, dcost, return_dweight=True)
    want = [_frame_sum(pr[0], nw, nf), pr[1], _frame_sum(pr[2], nw, nf), _frame_sum(pr[3], nw, nf), pr[4], pr[5], _frame_sum(pr[6], nw, nf), pr[7]]
    for n, g, w in zip(names, got, want):
        assert rel_fro(g, w) < 1e-5, n
    assert torch.equal(got[7], pr[7])                                   # dweight = dcost s: the pair kernel's arithmetic
    # one writer per element: dconv1, dD, dB and dweight are bitwise the same in a second run
    again = ops.lm_keyframe_cost_bwd(x.key, x.R, x.T, x.W, dcost, return_dweight=True)
    for i in (0, 2, 3, 7):
        assert torch.equal(got[i], again[i]), names[i]
    # pairs with dcost = 0 contribute nothing
    dz = dcost.clone()
    dz[1::2] = 0.0
    z = ops.lm_keyframe_cost_bwd(x.key, x.R, x.T, x.W, dz, return_dweight=True)
    for i in (1, 4, 5, 7):
        assert not bool(z[i][1::2].any()), names[i]
    zr = ops.lm_cost_bwd(x.rep, x.R, x.T, x.Wrep, dz, return_dweight=True)
    assert rel_fro(z[0], _frame_sum(zr[0], nw, nf)) < 1e-5 and rel_fro(z[2], _frame_sum(zr[2], nw, nf)) < 1e-5


def _skew(w):
    z = torch.zeros_like(w[:, 0])
    return torch.stack([torch.stack([z, -w[:, 2], w[:, 1]], -1), torch.stack([w[:, 2], z, -w[:, 0]], -1),
                        torch.stack([-w[:, 1], w[:, 0], z], -1)], -2)


@gpu
@pytest.mark.parametrize("weighted", [False, True])
def test_descent_identity_on_the_library(weighted):
    """On feature maps affine in (x, y), restricted to points whose taps and gradient stencil lie inside every frame's map, the gradient of
    sum_f cost w.r.t. the window's LM update at 0 is -2 g of the keyframe build: each frame's pose part, and the depth part summed over the
    frames (the LM update: R <- exp(w) R, T <- exp(w) T + t, W <- W + dl, to first order at 0)."""
    from banet_b200 import ops, autograd as AG
    _lib.require_device()
    nw, nf, C, K = 2, 3, 8, 16
    sc = _scene(nw, nf, C, K, 1500, seed=29)
    x = Win(sc, nw, nf)
    nb, h, w = nw * nf, x.conv2.shape[1], x.conv2.shape[2]
    a = oracle_level_inputs(sc.levels[0])
    Dt = x.rep.D.cpu().double() + x.rep.B.cpu().double() @ x.Wrep.cpu().double()
    _, _, _, _, px, py = O._warp(x.rep.p.cpu().double(), Dt, sc.R0.double(), sc.T0.double(), a["fx"], a["fy"], a["ox"], a["oy"])
    ok = ((px >= 2) & (px <= w - 3) & (py >= 2) & (py <= h - 3)).reshape(nw, nf, -1).all(1)
    n = int(ok.sum(1).min())
    assert n >= 100
    idx = torch.stack([torch.nonzero(ok[i]).flatten()[:n] for i in range(nw)]).cuda()
    take = lambda t: torch.gather(t, 1, idx.unsqueeze(-1).expand(-1, -1, t.shape[2])).contiguous()
    conv1, D, B, p = take(x.conv1), take(x.D), take(x.B), torch.gather(x.p, 2, idx.unsqueeze(1).expand(-1, 3, -1)).contiguous()
    g = torch.Generator().manual_seed(5)
    A0, ax, ay = (torch.rand(nb, 1, 1, C, generator=g) for _ in range(3))
    ax, ay = ax - 0.5, ay - 0.5
    F2 = A0 + ax * torch.arange(w, dtype=torch.float32).reshape(1, 1, w, 1) + ay * torch.arange(h, dtype=torch.float32).reshape(1, h, 1, 1)
    conv2 = torch.cat([F2, ax.expand(nb, h, w, C), ay.expand(nb, h, w, C)], -1).cuda().contiguous()
    c = (0.5 + torch.rand(nb, n, 1, generator=g)).cuda() if weighted else None
    _, gk, _, nv = ops.lm_keyframe_build(ops.KeyframeLevel(conv1, conv2, x.intr, p, D, B, weight=c), x.R, x.T, x.W)
    assert float(nv.min()) == n
    for layout in ("3c", "f2"):
        cv2 = conv2 if layout == "3c" else conv2[..., :C].contiguous()
        xi = torch.zeros(nb, 6, device="cuda", requires_grad=True)
        dl = torch.zeros(nw, K, device="cuda", requires_grad=True)
        E = torch.matrix_exp(_skew(xi[:, :3]))
        cost = AG.window_feature_metric_cost(conv1, cv2, D, B, E @ x.R, E @ x.T + xi[:, 3:].unsqueeze(-1), x.W + dl.unsqueeze(-1), x.intr, p,
                                             weight=c)
        gxi, gdl = torch.autograd.grad(cost.sum(), (xi, dl))
        e = (rel_fro(gxi, -2.0 * gk[:, :6]), rel_fro(gdl, -2.0 * gk[:, 6:].reshape(nw, nf, K).sum(1)))
        print(f"weighted={weighted} {layout}: pose {e[0]:.1e} depth {e[1]:.1e}")
        assert max(e) < 1e-4, layout


@gpu
def test_batches_past_65535_pairs():
    from banet_b200 import ops
    _lib.require_device()
    nw, nf, N, C, K, h, w = 16385, 4, 16, 4, 2, 8, 8
    nb = nw * nf
    g = torch.Generator(device="cuda").manual_seed(5)
    r = lambda *s: torch.rand(*s, device="cuda", generator=g)
    fx = fy = 6.0
    ox, oy = 3.5, 3.5
    u, v = 0.5 + r(nw, N) * (w - 2), 0.5 + r(nw, N) * (h - 2)
    p = torch.stack([(u - ox) / fx, (v - oy) / fy, torch.ones_like(u)], 1).contiguous()
    D, B, W = 1.0 + r(nw, N, 1), 0.1 * r(nw, N, K), (0.1 * r(nw, K, 1) - 0.05).contiguous()
    intr = torch.tensor([fx, fy, ox, oy], device="cuda").expand(nb, 4).contiguous()
    R = torch.linalg.matrix_exp(_skew(0.02 * (r(nb, 3) - 0.5))).contiguous()
    T = (0.02 * (r(nb, 3, 1) - 0.5)).contiguous()
    conv1, conv2, weight = r(nw, N, C), r(nb, h, w, 3 * C), 0.5 + r(nb, N, 1)
    key = ops.KeyframeLevel(conv1, conv2, intr, p, D, B, weight=weight)
    out = ops.lm_keyframe_cost(key, R, T, W, per_point=True)
    dcost = r(nb) - 0.5
    bw = ops.lm_keyframe_cost_bwd(key, R, T, W, dcost, return_dweight=True)
    assert float(out[1].min()) > 0
    wins = torch.tensor([0, 1, 9000, 16383, 16384], device="cuda")
    pairs = (wins.reshape(-1, 1) * nf + torch.arange(nf, device="cuda")).reshape(-1)
    rw, sp = lambda t: t[wins].repeat_interleave(nf, 0).contiguous(), lambda t: t[pairs].contiguous()
    small = ops.Level(rw(conv1), sp(conv2), sp(intr), rw(p), rw(D), rw(B), weight=sp(weight))
    out_s = ops.lm_cost(small, sp(R), sp(T), rw(W), per_point=True)
    for a, b in zip(out, out_s):
        assert torch.equal(a[pairs], b)
    bw_s = ops.lm_cost_bwd(small, sp(R), sp(T), rw(W), sp(dcost), return_dweight=True)
    k = len(wins)
    fs = lambda t: t.reshape(k, nf, *t.shape[1:]).sum(1)
    for i, (a, b) in enumerate(zip((bw[0][wins], bw[1][pairs], bw[2][wins], bw[3][wins], bw[4][pairs], bw[5][pairs], bw[6][wins], bw[7][pairs]),
                                   (fs(bw_s[0]), bw_s[1], fs(bw_s[2]), fs(bw_s[3]), bw_s[4], bw_s[5], fs(bw_s[6]), bw_s[7]))):
        assert rel_fro(a, b) < 1e-5, i
    assert torch.equal(bw[7][pairs], bw_s[7])


def _net(C):
    from banet_b200.bundlenet import BundleNet
    return BundleNet(C, levels=("2", "3"), exact_sym_grad=True, precision=_lib.PREC_FP32_SIMT, strict_status=False).cuda()


@gpu
def test_python_layers():
    from banet_b200 import ops, autograd as AG
    _lib.require_device()
    nw, nf, C, K = 2, 3, 16, 8
    sc = _scene(nw, nf, C, K, 600, seed=171)
    net = _net(C).eval()
    c = (0.5 + torch.rand(nw, nf, 600, 1, generator=torch.Generator().manual_seed(3))).cuda()
    for layout in ("3c", "f2"):
        for weight in (None, c):
            x = Win(sc, nw, nf, layout, None if weight is None else weight.reshape(nw * nf, 600, 1))
            fx, fy, ox, oy = [x.intr[:, i].reshape(nw, nf, 1) for i in range(4)]
            args = lambda **lv: [lv.get(n, getattr(x, n)) for n in ("conv1",)] + [lv.get("conv2", x.conv2).reshape(nw, nf, *x.conv2.shape[1:])] + \
                [fx, fy, ox, oy] + [lv.get(n, getattr(x, n)) for n in ("p", "D", "B")] + \
                [lv.get("R", x.R).reshape(nw, nf, 3, 3), lv.get("T", x.T).reshape(nw, nf, 3, 1), lv.get("W", x.W)]
            ref = ops.lm_keyframe_cost(x.key, x.R, x.T, x.W)[0]
            with torch.no_grad():
                got = net.WindowFeatureMetricCost(*args(), weight=weight)
            assert got.shape == (nw, nf) and torch.equal(got.reshape(-1), ref)
            leaves = {n: getattr(x, n).clone().requires_grad_() for n in ("conv1", "conv2", "D", "B", "R", "T", "W")}
            wl = None if weight is None else weight.clone().requires_grad_()
            cost = net.WindowFeatureMetricCost(*args(**leaves), weight=wl)
            assert torch.equal(cost.detach().reshape(-1), ref) and cost.requires_grad
            dc = torch.linspace(-1.0, 2.0, nw * nf, device="cuda")
            (cost.reshape(-1) * dc).sum().backward()
            want = ops.lm_keyframe_cost_bwd(x.key, x.R, x.T, x.W, dc, return_dweight=True)
            for n, wv in zip(("conv1", "conv2", "D", "B", "R", "T", "W"), want):
                atomic = n in ("conv2", "R", "T", "W")
                assert (rel_fro(leaves[n].grad, wv) < 1e-6) if atomic else torch.equal(leaves[n].grad, wv), (layout, n)
            if wl is not None:
                assert torch.equal(wl.grad.reshape(-1, 600, 1), want[7])
            direct = AG.window_feature_metric_cost(x.conv1, x.conv2, x.D, x.B, x.R, x.T, x.W, x.intr, x.p, weight=x.weight)
            assert torch.equal(direct, ref)


def _resize_inputs(nw, nf, C, K, seed=17):
    from banet_b200 import synth
    sc = synth.make_window_resize_scene(nw, nf, C, K, n_points=500, seed=seed)
    return dict(intr=to_cuda32(sc.intrisic), key=[to_cuda32(l) for l in sc.key_layers], frames=[to_cuda32(l) for l in sc.frame_layers],
                points=to_cuda32(sc.points), basis=to_cuda32(sc.basis), depth=to_cuda32(sc.init_depth), R0=to_cuda32(sc.R0), T0=to_cuda32(sc.T0))


def _resize(net, x, weight=None, **kw):
    return net.WindowResize(x["intr"], x["key"], x["frames"], x["points"], x["basis"], x["depth"], x["R0"], x["T0"], weight=weight, **kw)


@gpu
def test_window_resize_return_cost():
    from banet_b200 import ops
    _lib.require_device()
    nw, nf, C, K = 2, 3, 8, 4
    x = _resize_inputs(nw, nf, C, K)
    weight = (0.5 + torch.rand(nw, 1, 500, 1, generator=torch.Generator().manual_seed(4))).cuda()
    net = _net(C).eval()
    with torch.no_grad():
        Rs, Ts, Ds = _resize(net, x, weight)
        st = net.last_status.clone()
        Rc, Tc, Dc, Es = _resize(net, x, weight, return_cost=True)
    for a, b in zip(Rs + Ts + Ds, Rc + Tc + Dc):
        assert torch.equal(a, b)
    assert torch.equal(st, net.last_status)
    # Es[i] is WindowFeatureMetricCost at level i's inputs and outputs; the level's iteration is replayed to get its W
    pts, intr = net._prepare(x["intr"], x["points"])
    d, b = ops.resample(x["depth"], pts, 0.5), ops.resample(x["basis"], pts, 0.5)
    p = ops.compute_coordinates(pts, intr, True)
    R, T, W = x["R0"], x["T0"], torch.zeros(nw, K, 1, device="cuda")
    for i, level in enumerate((2, 3)):
        scale = 2 ** (3 - level)
        conv1 = ops.resample(x["key"][level], pts, 1.0 / scale)
        fx, fy, ox, oy = [(intr[:, j] / scale).reshape(nw, 1, 1) for j in range(4)]
        with torch.no_grad():
            R, T, W = net.WindowIteration(conv1, x["frames"][level], fx, fy, ox, oy, p, d, b, R, T, W, 1000.0, level, weight=weight)
            assert torch.equal(R, Rc[i]) and torch.equal(T, Tc[i])
            want = net.WindowFeatureMetricCost(conv1, x["frames"][level], fx, fy, ox, oy, p, d, b, R, T, W, weight=weight)
        assert Es[i].shape == (nw, nf) and torch.equal(Es[i], want), level
        assert float(Es[i].min()) > 0
    # with gradients: the costs are the same, and their gradient reaches both pyramids, the basis, the initial pose and the weight
    net.train()
    leaves = dict(key=[t.clone().requires_grad_() for t in x["key"]], frames=[t.clone().requires_grad_() for t in x["frames"]],
                  basis=x["basis"].clone().requires_grad_(), R0=x["R0"].clone().requires_grad_(), T0=x["T0"].clone().requires_grad_())
    wl = weight.clone().requires_grad_()
    Rg, Tg, Dg, Eg = _resize(net, {**x, **leaves}, wl, return_cost=True)
    for a, b in zip(Eg, Es):
        assert rel_fro(a.detach(), b) < 1e-5
    sum(e.sum() for e in Eg).backward()
    for name, t in (("key_layers[3]", leaves["key"][3]), ("key_layers[2]", leaves["key"][2]), ("frame_layers[3]", leaves["frames"][3]),
                    ("frame_layers[2]", leaves["frames"][2]), ("basis", leaves["basis"]), ("init_rotation", leaves["R0"]),
                    ("init_translation", leaves["T0"]), ("weight", wl)):
        assert t.grad is not None and bool(torch.isfinite(t.grad).all()) and bool(t.grad.any()), name

