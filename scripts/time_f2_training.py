"""Training on the F2-only feature layout against the 3C route, timed with CUDA events, warm-ups, the routes alternated in one loop, medians
and min-max reported.  Forward + backward of one differentiable iteration_fused, lambda-MLP on:
  3C route: F2 (requires grad) -> autograd.grad_fixed_concat -> the build on [F2|gx|gy] (what a user had to do before the F2-only backward);
  F2 route: F2 straight into the build (banet_lm_build_bwd applies the adjoint of the on-the-fly gradient stencil).
Workloads:
  a) 4096 sampled points at 160 x 120, nb = 32, C = 64, K = 128, FP32_SIMT (the reference's training regime);
  b) dense 320 x 240, nb = 32, C = K = 128, at FP32_SIMT and at AUTO;
  c) dense 640 x 480, nb = 16, C = K = 128, AUTO.
Every row reports each route's peak memory (above the inputs) and the largest relative difference of outputs and of gradients between the
routes; each workload also times the two backward kernels alone (banet_lm_build_bwd on the 3C map and on the F2 map, same dH, dg, drbar).
Prints one JSON document with the card's name and power limit; --out also writes it to a file."""
import argparse, json, os, sys
import torch
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from banet_b200 import synth, autograd as ag, ops, _lib
from time_window_training_step import card
from time_window_batch import timed
from time_window_keyframe import rel, peak_mib

PREC = {"FP32_SIMT": _lib.PREC_FP32_SIMT, "AUTO": _lib.PREC_AUTO}


def mlp_leaves(C):
    g = torch.Generator().manual_seed(7); dims = [C, 2 * C, 4 * C, 2 * C, C, 1]         # he_normal filters, zero biases (bundlenet.py:102-110)
    return [((torch.randn(dims[i], dims[i + 1], generator=g) * (2.0 / dims[i]) ** 0.5).cuda().requires_grad_(),
             torch.zeros(dims[i + 1], device="cuda").requires_grad_()) for i in range(5)]


def case(name, nb, H, W, C, K, n_points, precisions, args):
    sc = synth.make_scene(nb=nb, H=H, W=W, C=C, K=K, level_ids=(3,), seed=31, device="cuda", dtype=torch.float32, n_points=n_points)
    lv = sc.levels[0]
    leaf = lambda t: t.detach().clone().requires_grad_()
    F2 = leaf(lv.conv2[..., :C].contiguous())
    conv1, D, B, R, T, Wt = (leaf(t) for t in (lv.conv1, lv.D, lv.B, sc.R0, sc.T0, sc.W0 + 0.01))
    intr, p, grid = lv.intr, lv.p, lv.grid
    lv.conv2 = None
    del sc
    mlp = mlp_leaves(C)
    leaves = [F2, conv1, D, B, R, T, Wt, *[x for wb in mlp for x in wb]]
    loss = lambda o: o[0].sum() + o[1].sum() + (o[2] * o[2]).sum()
    rows = []
    for prec in precisions:
        def fwd(route, prec=prec):
            for x in leaves:
                x.grad = None
            conv2 = F2 if route == "f2" else ag.grad_fixed_concat(F2)
            return ag.iteration_fused(conv1, conv2, intr, p, D, B, R, T, Wt, mlp, 1000.0, precision=PREC[prec], grid=grid)
        routes = {"route_3c": "3c", "route_f2": "f2"}
        fns = {r: (lambda r=r: loss(fwd(routes[r])), lambda l: l.backward()) for r in routes}
        res = timed(fns, args.warmup, args.reps)
        got = {}
        for r in fns:
            for x in leaves:
                x.grad = None
            torch.cuda.empty_cache()
            res[r]["peak_MiB"] = peak_mib(lambda r=r: fns[r][1](fns[r][0]()))
            o = fwd(routes[r]); loss(o).backward()
            got[r] = ([x.detach().clone() for x in o], [x.grad.clone() for x in leaves])
        (o3, g3), (o1, g1) = got["route_3c"], got["route_f2"]
        names = ["F2", "conv1", "D", "B", "R", "T", "W"]
        diffs = {"outputs_R_T_W": max(rel(a, b) for a, b in zip(o1, o3)), **{f"grad_{n}": rel(a, b) for n, a, b in zip(names, g1, g3)},
                 "grad_mlp": max(rel(a, b) for a, b in zip(g1[7:], g3[7:]))}
        rows.append({"case": name, "nb": nb, "map": [W, H], "N": lv.N, "C": C, "K": K, "lambda": "mlp", "precision": prec, "reps": args.reps,
                     "timed": "forward + backward of one differentiable iteration_fused", "max_rel_diff_f2_vs_3c": diffs, **res})
        print(json.dumps(rows[-1]), flush=True)
        del got, o3, g3, o1, g1
        torch.cuda.empty_cache()
    # the backward kernels alone, on the level both routes see
    with torch.no_grad():
        conv2 = ops.grad_fixed_concat(F2.detach())
        lv3 = ops.Level(conv1.detach(), conv2, intr, p, D.detach(), B.detach(), grid=grid)
        lv1 = ops.Level(conv1.detach(), F2.detach(), intr, p, D.detach(), B.detach(), grid=grid)
        P = 6 + K
        gen = torch.Generator(device="cuda").manual_seed(3)
        dH = 1e-3 * torch.randn(nb, P, P, generator=gen, device="cuda")
        dg = 1e-3 * torch.randn(nb, P, generator=gen, device="cuda"); dr = 1e-3 * torch.randn(nb, C, generator=gen, device="cuda")
        Rd, Td, Wd = R.detach(), T.detach(), Wt.detach()
        fns = {"lm_build_bwd_3c": (lambda: None, lambda _: ops.lm_build_bwd(lv3, Rd, Td, Wd, dH, dg, dr, True)),
               "lm_build_bwd_f2": (lambda: None, lambda _: ops.lm_build_bwd(lv1, Rd, Td, Wd, dH, dg, dr, True))}
        res = timed(fns, args.warmup, args.reps)
        for r in res:
            del res[r]["forward_ms_median"], res[r]["forward_ms_min_max"]
        a, b = fns["lm_build_bwd_f2"][1](None), fns["lm_build_bwd_3c"][1](None)
        diffs = {"dF2": rel(a[1], ops.grad_fixed_concat_bwd(b[1])),
                 **{n: rel(x, y) for n, x, y in zip(("dconv1", "dD", "dB", "dR", "dT", "dW"), (a[0],) + a[2:], (b[0],) + b[2:])}}
        rows.append({"case": name + "-kernel", "nb": nb, "map": [W, H], "N": lv.N, "C": C, "K": K, "reps": args.reps,
                     "timed": "backward = banet_lm_build_bwd alone (dconv2 memset included)", "rel_diff_f2_vs_3c": diffs, **res})
        print(json.dumps(rows[-1]), flush=True)
        del a, b, conv2, lv3
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    _lib.require_device()
    rows = []
    rows += case("a", 32, 120, 160, 64, 128, 4096, ["FP32_SIMT"], args)
    rows += case("b", 32, 240, 320, 128, 128, None, ["FP32_SIMT", "AUTO"], args)
    rows += case("c", 16, 480, 640, 128, 128, None, ["AUTO"], args)
    doc = {"script": "scripts/time_f2_training.py", **card(), "rows": rows}
    print(json.dumps(doc, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
