"""Keyframe-layout windows (banet_lm_keyframe_*: the keyframe tensors once per window) against the [nw,1,...] broadcast form (the per-pair
build on copies of the keyframe), timed with CUDA events, warm-ups, the contenders alternated in one loop, medians and min-max reported.
Every row also reports each contender's peak memory and the relative difference of outputs and gradients between the contenders.  Prints one
JSON document with the card's name and power limit; --out also writes it to a file.
  i)   nw = 32, nf = 4, 4096 points per window, C = K = 128, lambda-MLP: forward + backward of one differentiable iteration;
  ii)  nw = 4, nf = 4, the dense 320 x 240 grid, C = K = 128, lambda-MLP: the same;
  iii) nw = 8, nf = 16, 4096 points, C = K = 128, lambda-MLP: the same;
  iv)  the build kernels alone (forward, backward) at (i) and (iii): banet_lm_keyframe_build(_bwd) against banet_lm_build(_bwd) (FP32_SIMT) on
       pre-replicated per-pair tensors;
  v)   no-grad: one iteration of banet_lm_keyframe_run against banet_lm_window_batch_run at AUTO (the tensor-core per-pair build) at (ii)."""
import argparse, json, os, statistics, sys
import torch
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from banet_b200 import synth, autograd as ag, ops, _lib
from time_window_training_step import card
from time_window_batch import timed

C = K = 128


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300))


def peak_mib(fn):
    """Peak device memory above what was allocated before one call of fn (MiB), gradients included."""
    torch.cuda.synchronize(); torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn(); torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2**20


def scene(nw, nf, n_points, seed):
    level = 3 if n_points is None else 1                            # dense: the 320 x 240 grid; sparse: 4096 points on an 80 x 60 map
    return synth.make_scene(nb=nw * nf, H=240, W=320, C=C, K=K, level_ids=(level,), seed=seed, device="cuda", dtype=torch.float32,
                            n_points=n_points, shared_depth=True, window_frames=nf)


def mlp_leaves():
    g = torch.Generator().manual_seed(7); dims = [C, 2 * C, 4 * C, 2 * C, C, 1]         # he_normal filters, zero biases (bundlenet.py:102-110)
    return [((torch.randn(dims[i], dims[i + 1], generator=g) * (2.0 / dims[i]) ** 0.5).cuda().requires_grad_(),
             torch.zeros(dims[i + 1], device="cuda").requires_grad_()) for i in range(5)]


def training_case(name, nw, nf, n_points, args):
    sc = scene(nw, nf, n_points, seed=21)
    lv = sc.levels[0]
    mlp = mlp_leaves()
    leaf = lambda t: t.detach().clone().requires_grad_()
    bw = lambda t: t.reshape(nw, nf, *t.shape[1:])
    kf = lambda t: bw(t)[:, 0].contiguous()
    conv2, R, T = leaf(bw(lv.conv2)), leaf(bw(sc.R0)), leaf(bw(sc.T0))
    W = leaf(sc.W0.reshape(nw, nf, K, 1)[:, 0])
    intr = bw(lv.intr)
    key = {n: leaf(kf(getattr(lv, n))) for n in ("conv1", "D", "B")}
    bc = {n: leaf(kf(getattr(lv, n)).unsqueeze(1)) for n in ("conv1", "D", "B")}
    pk = kf(lv.p)
    shared = [conv2, R, T, W, *[x for wb in mlp for x in wb]]

    def run(form):
        t, p = (key, pk) if form == "keyframe" else (bc, pk.unsqueeze(1))
        for x in shared + list(t.values()):
            x.grad = None
        return ag.window_batch_iteration_fused(t["conv1"], conv2, intr, p, t["D"], t["B"], R, T, W, mlp, 1000.0)

    loss = lambda o: o[0].sum() + o[1].sum() + (o[2] * o[2]).sum()
    fns = {f: (lambda f=f: loss(run(f)), lambda l: l.backward()) for f in ("keyframe", "broadcast_nw1")}
    res = timed(fns, args.warmup, args.reps)
    grads = {}
    for f in fns:
        for x in shared + list(key.values()) + list(bc.values()):    # the peak is taken above the inputs alone
            x.grad = None
        res[f]["peak_MiB"] = peak_mib(lambda f=f: fns[f][1](fns[f][0]()))
        o = run(f); loss(o).backward()
        t = key if f == "keyframe" else bc
        grads[f] = ([x.detach().clone() for x in o], {n: t[n].grad.reshape(nw, *t[n].shape[-2:]).clone() for n in t},
                    [x.grad.clone() for x in shared])
    (ok, kg, ks), (ob, bg, bs) = grads["keyframe"], grads["broadcast_nw1"]
    diffs = {"outputs_R_T_W": max(rel(x, y) for x, y in zip(ok, ob)), **{f"grad_{n}": rel(kg[n], bg[n]) for n in kg},
             "grad_conv2_R_T_W_mlp": max(rel(x, y) for x, y in zip(ks, bs))}
    return {"case": name, "nw": nw, "nf": nf, "N_per_window": lv.N, "C": C, "K": K, "lambda": "mlp", "precision": "FP32_SIMT", "reps": args.reps,
            "rel_diff_keyframe_vs_broadcast": diffs, **res}


def build_case(name, nw, nf, args):
    sc = scene(nw, nf, 4096, seed=22)
    l = sc.levels[0]
    kf = lambda t: t.reshape(nw, nf, *t.shape[1:])[:, 0].contiguous()
    key = ops.KeyframeLevel(kf(l.conv1), l.conv2, l.intr, kf(l.p), kf(l.D), kf(l.B))
    r = lambda t: t.repeat_interleave(nf, 0).contiguous()
    rep = ops.Level(r(key.conv1), key.conv2, key.intr, r(key.p), r(key.D), r(key.B))
    W = sc.W0.reshape(nw, nf, K, 1)[:, 0].contiguous() + 0.01
    Wp = r(W)
    P, nb = 6 + K, nw * nf
    gen = torch.Generator(device="cuda").manual_seed(3)
    dH = 1e-3 * torch.randn(nb, P, P, generator=gen, device="cuda")
    dH.reshape(nw, nf, P, P)[:, :, 6:, 6:] = dH.reshape(nw, nf, P, P)[:, :1, 6:, 6:].clone()      # the window steps' backward: one depth block
    dg = 1e-3 * torch.randn(nb, P, generator=gen, device="cuda"); dr = 1e-3 * torch.randn(nb, C, generator=gen, device="cuda")
    fns = {"keyframe_build": (lambda: ops.lm_keyframe_build(key, sc.R0, sc.T0, W),
                              lambda o: ops.lm_keyframe_build_bwd(key, sc.R0, sc.T0, W, dH, dg, dr, True)),
           "per_pair_build": (lambda: ops.lm_build(rep, sc.R0, sc.T0, Wp, _lib.PREC_FP32_SIMT),
                              lambda o: ops.lm_build_bwd(rep, sc.R0, sc.T0, Wp, dH, dg, dr, True))}
    res = timed(fns, args.warmup, args.reps)
    for f in fns:
        res[f]["peak_MiB"] = peak_mib(lambda f=f: fns[f][1](fns[f][0]()))
    a, b = fns["keyframe_build"][0](), fns["per_pair_build"][0]()
    m = torch.ones(nb, P, P, device="cuda"); m[:, 6:, 6:] = 0
    Ha, Hb = a[0].reshape(nw, nf, P, P), b[0].reshape(nw, nf, P, P)
    ga, gb = fns["keyframe_build"][1](a), fns["per_pair_build"][1](b)
    fsum = lambda t: t.reshape(nw, nf, *t.shape[1:]).sum(1)
    diffs = {"H_depth_block": rel(Ha[:, 0, 6:, 6:], Hb[:, :, 6:, 6:].sum(1)), "H_rest": rel(a[0] * m, b[0] * m), "g": rel(a[1], b[1]),
             "dconv1": rel(ga[0], fsum(gb[0])), "dconv2": rel(ga[1], gb[1]), "dD": rel(ga[2], fsum(gb[2])), "dB": rel(ga[3], fsum(gb[3])),
             "dR": rel(ga[4], gb[4]), "dT": rel(ga[5], gb[5]), "dW": rel(ga[6], fsum(gb[6]))}
    return {"case": name, "nw": nw, "nf": nf, "N_per_window": l.N, "C": C, "K": K, "reps": args.reps, "timed": "forward = build, backward = build backward",
            "rel_diff_keyframe_vs_per_pair": diffs, **res}


def run_case(args):
    nw, nf = 4, 4
    sc = scene(nw, nf, None, seed=23)
    l = sc.levels[0]
    kf = lambda t: t.reshape(nw, nf, *t.shape[1:])[:, 0].contiguous()
    key = ops.KeyframeLevel(kf(l.conv1), l.conv2, l.intr, kf(l.p), kf(l.D), kf(l.B))
    r = lambda t: t.repeat_interleave(nf, 0).contiguous()
    rep = ops.Level(r(key.conv1), key.conv2, key.intr, r(key.p), r(key.D), r(key.B), grid=l.grid)
    W = sc.W0.reshape(nw, nf, K, 1)[:, 0].contiguous()
    packed = [ops.pack_mlp([(w.detach(), b.detach()) for w, b in mlp_leaves()])]
    fns = {"keyframe_run_FP32_SIMT": (lambda: ops.lm_keyframe_run([key], 1, sc.R0, sc.T0, W, mlp_packed=packed), lambda o: None),
           "window_batch_run_AUTO": (lambda: ops.lm_window_batch_run([rep], nw, 1, sc.R0, sc.T0, W, mlp_packed=packed, l2_regularizer_base=1000.0,
                                                                     precision=_lib.PREC_AUTO), lambda o: None),
           "window_batch_run_FP32_SIMT": (lambda: ops.lm_window_batch_run([rep], nw, 1, sc.R0, sc.T0, W, mlp_packed=packed, l2_regularizer_base=1000.0,
                                                                          precision=_lib.PREC_FP32_SIMT), lambda o: None)}
    with torch.no_grad():
        res = timed(fns, args.warmup, args.reps)
        for f in fns:
            res[f]["peak_MiB"] = peak_mib(fns[f][0])
        outs = {f: fns[f][0]() for f in fns}
    k = outs["keyframe_run_FP32_SIMT"]
    diffs = {f: {"R": rel(k[0], o[0]), "T": rel(k[1], o[1]), "W": rel(k[2], o[2])} for f, o in outs.items() if f != "keyframe_run_FP32_SIMT"}
    return {"case": "v", "nw": nw, "nf": nf, "N_per_window": l.N, "C": C, "K": K, "lambda": "mlp", "iterations": 1, "reps": args.reps,
            "timed": "forward = the whole no-grad iteration", "rel_diff_keyframe_vs": diffs, **res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    _lib.require_device()
    rows = []
    for fn in (lambda: training_case("i", 32, 4, 4096, args), lambda: training_case("ii", 4, 4, None, args),
               lambda: training_case("iii", 8, 16, 4096, args), lambda: build_case("iv-i", 32, 4, args), lambda: build_case("iv-iii", 8, 16, args),
               lambda: run_case(args)):
        rows.append(fn())
        print(json.dumps(rows[-1]), flush=True)
        torch.cuda.empty_cache()
    doc = {"script": "scripts/time_window_keyframe.py", **card(), "rows": rows}
    print(json.dumps(doc, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
