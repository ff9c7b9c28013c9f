"""Cost of per-point weights in keyframe windows (banet_keyframe_level_t::weight) on an H100, and the unweighted keyframe build against a
comparison tree's library (GPU).

    python scripts/time_window_weights.py [--base-tree /path/to/other/checkout] [--rounds 5] [--reps 10] [--out profiles/h100_window_weights.json]

Workloads of profiles/h100_window_keyframe.json: (i) nw = 32, nf = 4, 4096 keyframe points per window, C = K = 128; (ii) nw = 4, nf = 4, the
dense 320 x 240 grid, C = K = 128.  Unweighted against weighted (weights in [0.5, 1.5], one per (frame, point)):
  (a) banet_lm_keyframe_build alone, at (i) and (ii);
  (b) forward + backward of one differentiable keyframe iteration (autograd.window_batch_iteration_fused, lambda-MLP), the weight requiring
      grad, at (i) and (ii);
  (c) BundleNet.WindowResize inference (two levels, one keyframe iteration each) at (i).
(d) --base-tree: this library's unweighted banet_lm_keyframe_build against the comparison tree's (its own libbanet.so, bound through its own
    _lib.py), at (i) and (ii): whether the outputs are bitwise equal, and the times.
Every case alternates its contenders --rounds times; a round times --reps calls of each after three warm-up calls (CUDA events).  The report
gives median [min - max] per contender over all timed calls, and the card's name and power limit read in the same call."""
import argparse, importlib.util, json, os, statistics, sys
import ctypes as C
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from banet_b200 import synth, autograd as ag, ops, _lib
from banet_b200.bundlenet import BundleNet
from time_window_training_step import card

CK = 128


def timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return ms


def alternate(cases, rounds, reps):
    ms = {k: [] for k in cases}
    for _ in range(rounds):
        for k, fn in cases.items():
            ms[k] += timed(fn, reps)
    return {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v), "n": len(v)} for k, v in ms.items()}


def workload(name):
    nw, nf, n_points, level = (32, 4, 4096, 1) if name == "i" else (4, 4, None, 3)     # (ii): the dense 320 x 240 grid of level 3
    sc = synth.make_scene(nb=nw * nf, H=240, W=320, C=CK, K=CK, level_ids=(level,), seed=21, device="cuda", dtype=torch.float32,
                          n_points=n_points, shared_depth=True, window_frames=nf)
    l = sc.levels[0]
    kf = lambda t: t.reshape(nw, nf, *t.shape[1:])[:, 0].contiguous()
    w = 0.5 + torch.rand(nw * nf, l.N, 1, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    return dict(nw=nw, nf=nf, N=l.N, sc=sc, l=l, conv1=kf(l.conv1), p=kf(l.p), D=kf(l.D), B=kf(l.B), W=sc.W0.reshape(nw, nf, CK, 1)[:, 0].contiguous(), w=w)


def key_level(x, weight=None):
    return ops.KeyframeLevel(x["conv1"], x["l"].conv2, x["l"].intr, x["p"], x["D"], x["B"], weight=weight)


def mlp_leaves():
    g = torch.Generator().manual_seed(7); dims = [CK, 2 * CK, 4 * CK, 2 * CK, CK, 1]
    return [((torch.randn(dims[i], dims[i + 1], generator=g) * (2.0 / dims[i]) ** 0.5).cuda().requires_grad_(),
             torch.zeros(dims[i + 1], device="cuda").requires_grad_()) for i in range(5)]


def build_cases(x):
    sc = x["sc"]
    lv0, lv1 = key_level(x), key_level(x, x["w"])
    return {"unweighted": lambda: ops.lm_keyframe_build(lv0, sc.R0, sc.T0, x["W"]), "weighted": lambda: ops.lm_keyframe_build(lv1, sc.R0, sc.T0, x["W"])}


def train_cases(x):
    nw, nf, sc, l = x["nw"], x["nf"], x["sc"], x["l"]
    mlp = mlp_leaves()
    bw = lambda t: t.reshape(nw, nf, *t.shape[1:])
    leaf = lambda t: t.detach().clone().requires_grad_()
    t = {n: leaf(x[n]) for n in ("conv1", "D", "B")}
    conv2, R, T, W = leaf(bw(l.conv2)), leaf(bw(sc.R0)), leaf(bw(sc.T0)), leaf(x["W"])
    wt = leaf(x["w"].reshape(nw, nf, x["N"], 1))

    def step(weight):
        o = ag.window_batch_iteration_fused(t["conv1"], conv2, bw(l.intr), x["p"], t["D"], t["B"], R, T, W, mlp, 1000.0, weight=weight)
        (o[0].sum() + o[1].sum() + (o[2] * o[2]).sum()).backward()

    return {"unweighted": lambda: step(None), "weighted (requires grad)": lambda: step(wt)}


def resize_cases():
    nw, nf = 32, 4
    sc = synth.make_window_resize_scene(nw, nf, CK, CK, n_points=4096, seed=5, device="cuda")
    net = BundleNet(CK, levels=("2", "3"), precision=_lib.PREC_FP32_SIMT).cuda().eval()
    w = 0.5 + torch.rand(nw, nf, 4096, 1, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))

    def run(weight):
        with torch.no_grad():
            net.WindowResize(sc.intrisic, sc.key_layers, sc.frame_layers, sc.points, sc.basis, sc.init_depth, sc.R0, sc.T0, weight=weight)

    return {"unweighted": lambda: run(None), "weighted": lambda: run(w)}


def base_cases(x, base_tree):
    """banet_lm_keyframe_build of this library and of base_tree's, unweighted, on the same tensors and into separate outputs."""
    spec = importlib.util.spec_from_file_location("banet_base_lib", os.path.join(base_tree, "banet_b200", "_lib.py"))
    base = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(base)
    sc, l, nw, nf = x["sc"], x["l"], x["nw"], x["nf"]
    nb, P = nw * nf, 6 + CK
    R, T, W = sc.R0.contiguous(), sc.T0.contiguous(), x["W"]
    stream = torch.cuda.current_stream().cuda_stream

    def make(mod):
        lib = mod.load()
        st = mod.BanetKeyframeLevel(nw, nf, x["N"], CK, CK, l.conv2.shape[1], l.conv2.shape[2], l.conv2.shape[3], x["conv1"].data_ptr(),
                                    x["p"].data_ptr(), x["D"].data_ptr(), x["B"].data_ptr(), l.conv2.data_ptr(), l.intr.data_ptr())
        ws = torch.empty(max(lib.banet_lm_keyframe_build_workspace_bytes(C.byref(st)), 256), dtype=torch.uint8, device="cuda")
        out = [torch.empty(nb, P, P, device="cuda"), torch.empty(nb, P, device="cuda"), torch.empty(nb, CK, device="cuda"), torch.empty(nb, device="cuda")]

        def fn():
            mod.check(lib.banet_lm_keyframe_build(C.byref(st), R.data_ptr(), T.data_ptr(), W.data_ptr(), *[o.data_ptr() for o in out], ws.data_ptr(),
                                                  ws.numel(), stream), "banet_lm_keyframe_build")
        return fn, out

    (f_this, o_this), (f_base, o_base) = make(_lib), make(base)
    res = alternate({"this tree": f_this, "base tree": f_base}, ARGS.rounds, ARGS.reps)
    f_this(); f_base(); torch.cuda.synchronize()
    res["outputs_bitwise_equal"] = all(torch.equal(a, b) for a, b in zip(o_this, o_base))
    return res


def main():
    global ARGS
    ap = argparse.ArgumentParser()
    ap.add_argument("--base-tree", default=None, help="a checkout (library built) whose unweighted keyframe build is compared with this tree's")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_window_weights.json"))
    ARGS = a = ap.parse_args()
    _lib.require_device()
    rep = {"script": "scripts/time_window_weights.py", **card(), "rounds": a.rounds, "reps_per_round": a.reps, "cases": {}}
    for name in ("i", "ii"):
        x = workload(name)
        shape = f"nw={x['nw']} nf={x['nf']} N={x['N']} C=K={CK}"
        rep["cases"][f"(a) keyframe build ({name}) {shape}"] = alternate(build_cases(x), a.rounds, a.reps)
        rep["cases"][f"(b) keyframe iteration fwd+bwd ({name}) {shape}"] = alternate(train_cases(x), a.rounds, a.reps)
        if a.base_tree:
            rep["cases"][f"(d) unweighted keyframe build, this vs base tree ({name}) {shape}"] = base_cases(x, os.path.abspath(a.base_tree))
        print(json.dumps(rep, indent=1), flush=True)
        del x
        torch.cuda.empty_cache()
    rep["cases"]["(c) WindowResize inference (i) nw=32 nf=4 N=4096 C=K=128"] = alternate(resize_cases(), a.rounds, a.reps)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rep, f, indent=1)
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    main()
