"""Cost of training through the fused LM step on an H100 (GPU).

    python scripts/time_step_bwd.py [--reps 20] [--out profiles/h100_step_bwd.json]
    python scripts/time_step_bwd.py --profile [--out profiles/h100_step_bwd_profile.json]

(a) One step, forward + backward, after a real build (nb = 32, C = K = 128; FP32_SIMT build of a synthetic scene with 4096 random points per
    pair and with the dense 320 x 240 grid): autograd._LMStepFn (banet_lm_step + banet_lm_step_bwd) against the lambda-MLP in stock torch +
    autograd._LMSolveUpdateFn (banet_lm_solve_update + banet_lm_solve_update_bwd), the route of iteration_fused.  Only the step is timed.
(b) A whole differentiable solve, forward + backward, 2 levels x 5 iterations (FP32_SIMT), at the same sizes (levels 2 and 3 of each scene):
    autograd.lm_run against a Python loop of iteration_fused.  The outputs and gradients of the two routes are compared (max relative
    difference and relative Frobenius difference, per tensor: R', T', W' and the gradients of R0, T0, W0, conv1, conv2, D, B and every
    lambda-MLP parameter), next to the loop against a second run of itself: the build backward accumulates with atomics, so that is the
    run-to-run spread of the gradients.
(c) --profile, a run of its own: torch.profiler over one forward + backward of autograd.lm_run (4096 points), listing every CUDA kernel with
    its launch count and device time, and the launches per LM iteration.
Each timed case runs 3 warm-up rounds, then --reps rounds alternating the two routes, each timed with CUDA events; the report gives median
[min - max] in ms, and the card name and power limit read in the same call.
"""
import argparse, json, os, statistics, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from banet_b200 import autograd as ag, ops, synth, _lib  # noqa: E402

NB, C, K = 32, 128, 128


def gpu_identity():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
    return {"name": q[0], "power_limit_w": float(q[1])}


def scene(n_points, level_ids):
    return synth.make_scene(nb=NB, H=240, W=320, C=C, K=K, level_ids=level_ids, seed=1234, n_points=n_points, device="cuda", dtype=torch.float32)


def levels_of(sc, grad):
    out = []
    for lv in sc.levels:
        t = [x.detach().clone().requires_grad_(grad) for x in (lv.conv1, lv.conv2, lv.D, lv.B)]
        out.append(ops.Level(t[0], t[1], lv.intr, lv.p, t[2], t[3], grid=lv.grid))
    return out


def mlps(levels):
    """Per level: five (filters [cin,cout], biases [cout]) with he-normal filters and zero biases (bundlenet.py:105-106), seeded."""
    dims = [C, 2 * C, 4 * C, 2 * C, C, 1]
    out = []
    for i in range(len(levels)):
        g = torch.Generator().manual_seed(100 + i)
        out.append([((torch.randn(dims[l], dims[l + 1], generator=g) * (2.0 / dims[l]) ** 0.5).cuda().requires_grad_(),
                     torch.zeros(dims[l + 1], device="cuda").requires_grad_()) for l in range(5)])
    return out


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b)


def stats(xs):
    return {"median_ms": statistics.median(xs), "min_ms": min(xs), "max_ms": max(xs), "n": len(xs)}


def alternate(routes, reps):
    for _ in range(3):
        for fn in routes.values():
            fn()
    torch.cuda.synchronize()
    t = {k: [] for k in routes}
    for _ in range(reps):
        for k, fn in routes.items():
            t[k].append(timed(fn))
    return {k: stats(v) for k, v in t.items()}


def max_rel(a, b):
    """(max |a - b| / max |b|, ||a - b|| / ||b||)"""
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30)), float((a - b).norm() / b.norm().clamp_min(1e-30))


def case_step(n_points, reps):
    sc = scene(n_points, (3,))
    lv = levels_of(sc, False)[0]
    N = lv.conv1.shape[1]
    W0 = sc.W0 + 0.01
    H, g, rbar, _ = ops.lm_build(lv, sc.R0, sc.T0, W0, _lib.PREC_FP32_SIMT)
    mlp = mlps([lv])[0]
    gen = torch.Generator(device="cuda").manual_seed(5)
    cR, cT, cW = [torch.randn(s, device="cuda", generator=gen) for s in ((NB, 3, 3), (NB, 3, 1), (NB, K, 1))]

    def leaves():
        return [t.detach().clone().requires_grad_() for t in (H, g, rbar, sc.R0, sc.T0, W0)]

    def fused():
        h, gg, rb, R, T, W = leaves()
        Rn, Tn, Wn, _ = ag._LMStepFn.apply(h, gg, rb, None, R, T, W, N, 1000.0, 1e-5, True, *[t for wb in mlp for t in wb])
        ((Rn * cR).sum() + (Tn * cT).sum() + (Wn * cW).sum()).backward()

    def torch_mlp():
        h, gg, rb, R, T, W = leaves()
        avg = (rb / float(N)).unsqueeze(1)
        lam = 1000.0 * torch.pow(torch.linalg.norm(avg, dim=-1, keepdim=True), 2.0 + ag.lambda_mlp(avg, mlp)).reshape(NB)
        Rn, Tn, Wn, _ = ag._LMSolveUpdateFn.apply(h, gg, lam, R, T, W, 1e-5, True)
        ((Rn * cR).sum() + (Tn * cT).sum() + (Wn * cW).sum()).backward()

    return {"points_per_pair": N, "times": alternate({"LMStepFn": fused, "torch_mlp+LMSolveUpdateFn": torch_mlp}, reps)}


def solve_routes(sc):
    gen = torch.Generator(device="cuda").manual_seed(7)
    cR, cT, cW = [torch.randn(s, device="cuda", generator=gen) for s in ((NB, 3, 3), (NB, 3, 1), (NB, K, 1))]
    levels = levels_of(sc, True)
    mlp = mlps(levels)

    def run(route):
        R, T, W = [t.detach().clone().requires_grad_() for t in (sc.R0, sc.T0, sc.W0)]
        if route == "lm_run":
            Rn, Tn, Wn = ag.lm_run(levels, 5, R, T, W, mlp_params=mlp, precision=_lib.PREC_FP32_SIMT)
        else:
            Rn, Tn, Wn = R, T, W
            for lv, m in zip(levels, mlp):
                for _ in range(5):
                    Rn, Tn, Wn = ag.iteration_fused(lv.conv1, lv.conv2, lv.intr, lv.p, lv.D, lv.B, Rn, Tn, Wn, m, 1000.0,
                                                    precision=_lib.PREC_FP32_SIMT, grid=lv.grid)
        ((Rn * cR).sum() + (Tn * cT).sum() + (Wn * cW).sum()).backward()
        return R, T, W, (Rn, Tn, Wn)
    return levels, mlp, run


def case_solve(n_points, reps):
    sc = scene(n_points, (2, 3))
    levels, mlp, run = solve_routes(sc)
    leaves = [t for lv in levels for t in (lv.conv1, lv.conv2, lv.D, lv.B)] + [t for m in mlp for wb in m for t in wb]
    res = {}
    for route in ("lm_run", "loop", "loop_again"):
        for t in leaves:
            t.grad = None
        R, T, W, outs = run(route.replace("_again", ""))
        res[route] = dict(R=outs[0], T=outs[1], W=outs[2], dR0=R.grad, dT0=T.grad, dW0=W.grad,
                          **{f"d{n}{i}": getattr(lv, n).grad.clone() for i, lv in enumerate(levels) for n in ("conv1", "conv2", "D", "B")},
                          **{f"dmlp{i}_{j}": t.grad.clone() for i, m in enumerate(mlp) for j, t in enumerate(x for wb in m for x in wb)})
    diffs = {k: max_rel(res["lm_run"][k], res["loop"][k]) for k in res["loop"]}
    noise = {k: max_rel(res["loop_again"][k], res["loop"][k]) for k in res["loop"]}
    times = alternate({"lm_run": lambda: run("lm_run"), "iteration_fused_loop": lambda: run("loop")}, reps)
    return {"points_per_pair_per_level": [lv.conv1.shape[1] for lv in levels], "times": times,
            "rel_diff_lm_run_vs_loop": {"outputs": {k: diffs[k] for k in ("R", "T", "W")},
                                        "gradients": {k: v for k, v in diffs.items() if k.startswith("d")}},
            "rel_diff_loop_vs_itself": {"outputs": {k: noise[k] for k in ("R", "T", "W")},
                                        "gradients": {k: v for k, v in noise.items() if k.startswith("d")}}}


def profile():
    from torch.profiler import profile as tprofile, ProfilerActivity
    sc = scene(4096, (2, 3))
    _, _, run = solve_routes(sc)
    run("lm_run"); torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        run("lm_run"); torch.cuda.synchronize()
    counts, us = {}, {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset")):
            counts[e.name] = counts.get(e.name, 0) + 1
            us[e.name] = us.get(e.name, 0.0) + float(getattr(e, "device_time", 0.0) or 0.0)
    banet = {k: v for k, v in counts.items() if "banet" in k}
    iters = 2 * 5
    kernels = {k: {"launches": counts[k], "total_us": us[k], "mean_us": us[k] / counts[k]} for k in sorted(counts, key=lambda k: -us[k])}
    return {"iterations": iters, "kernels": kernels, "banet_launches_per_iteration": sum(banet.values()) / iters,
            "all_launches_per_iteration": sum(counts.values()) / iters, "kernel_time_total_us": sum(us.values())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    _lib.require_device()
    rep = {"gpu": gpu_identity(), "nb": NB, "C": C, "K": K}
    if a.profile:
        rep["profile_lm_run_4096_points"] = profile()
        out = a.out or os.path.join(ROOT, "profiles", "h100_step_bwd_profile.json")
    else:
        rep["reps"] = a.reps
        rep["a_step"] = {"4096_points": case_step(4096, a.reps), "320x240": case_step(None, a.reps)}
        rep["b_solve_2x5"] = {"4096_points": case_solve(4096, a.reps), "320x240": case_solve(None, a.reps)}
        out = a.out or os.path.join(ROOT, "profiles", "h100_step_bwd.json")
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    with open(out, "w") as f:
        json.dump(rep, f, indent=1, default=str)
    print(json.dumps(rep, indent=1, default=str))


if __name__ == "__main__":
    main()
