"""bfloat16 against float32 feature maps on the GPU: build per level, whole solve, host-pipeline step, one training iteration.

    python scripts/time_bf16_features.py [--reps 20] [--out profiles/h100_bf16_features.json]

(a) lm_build per cfg2 level (80x60 .. 640x480, 32 pairs, C = K = 128, AUTO) for fp32-3C, fp32-F2, bf16-F2 and bf16-3C, with the
    achieved bytes/s against each variant's algorithmic bytes (conv1 + conv2 + basis + p + D, each read once).
(b) the whole 4-level solve (5 iterations per level, fixed lambda) for fp32 3C, fp32 F2 and bf16 F2, with the W and finest-level depth
    difference of each against the fp32 3C solve.
(c) one ResizeHostSolver step (32 images, 4 levels, pinned host inputs) with a fp32 and a bf16 host pyramid, with the H2D bytes.
(d) one differentiable iteration (autograd.iteration_fused, F2 layout) at dense 320x240, 8 pairs: forward + backward and peak memory.
Every case is warmed up, then the variants of a group are timed alternately, `--reps` times each (CUDA events); the report gives the
median and min - max.  The card's name and power limit are read in the same run.
"""
import argparse, json, os, statistics, subprocess, sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def alternate(fns, reps, warm=2):
    """fns: name -> callable.  Warm each, then time them round-robin; -> name -> {median_ms, min_ms, max_ms}."""
    import torch
    for fn in fns.values():
        for _ in range(warm):
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in fns}
    for _ in range(reps):
        for k, fn in fns.items():
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record(); torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1))
    return {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)} for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bf16_features.json"))
    ap.add_argument("--profile", default=None, help="only write a torch.profiler kernel table of the 640x480 F2 builds (fp32 and bf16) to this file")
    args = ap.parse_args()
    import torch
    from banet_b200 import ops, synth, autograd as ag, _lib
    from banet_b200.host_pipeline import ResizeHostSolver
    _lib.require_device()
    BF = torch.bfloat16
    dev = torch.device("cuda")
    rel = lambda a, b: float((a - b).norm() / b.norm())
    report = {"card": card(), "reps": args.reps}
    nb, C, K = 32, 128, 128

    # ---- (a) build per level, (b) whole solve
    sc = synth.make_scene(nb=nb, H=480, W=640, C=C, K=K, level_ids=(0, 1, 2, 3), seed=1234 + 2, device=dev, dtype=torch.float32)
    var = {}
    for name, dt, layout in (("fp32-3C", torch.float32, "3C"), ("fp32-F2", torch.float32, "F2"), ("bf16-F2", BF, "F2"), ("bf16-3C", BF, "3C")):
        var[name] = [ops.Level(l.conv1.to(dt), (l.conv2 if layout == "3C" else l.conv2[..., :C]).contiguous().to(dt), l.intr, l.p, l.D, l.B, grid=l.grid)
                     for l in sc.levels]
    if args.profile:
        from torch.profiler import profile, ProfilerActivity
        fns = {k: (lambda lv=var[k][-1]: ops.lm_build(lv, sc.R0, sc.T0, sc.W0, _lib.PREC_AUTO)) for k in ("fp32-F2", "bf16-F2")}
        alternate(fns, 2)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                for fn in fns.values():
                    fn()
            torch.cuda.synchronize()
        with open(args.profile, "w") as f:
            f.write(f"{report['card']}\n640x480, 32 pairs, C = K = {C}, AUTO (TF32X1), F2 layout, 5 builds each\n")
            f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=12, max_name_column_width=110))
        print(open(args.profile).read())
        return
    builds = []
    for li, l in enumerate(sc.levels):
        N = l.N
        fns = {k: (lambda lv=v[li]: ops.lm_build(lv, sc.R0, sc.T0, sc.W0, _lib.PREC_AUTO)) for k, v in var.items()}
        t = alternate(fns, args.reps)
        row = {"level": f"{l.conv2.shape[2]}x{l.conv2.shape[1]}", "N": N}
        for k, v in var.items():
            es = v[li].conv1.element_size()
            c2 = v[li].conv2.shape[-1]
            by = nb * N * ((C + c2) * es + (K + 4) * 4)
            row[k] = dict(t[k], algorithmic_bytes=by, achieved_GBs=by / (t[k]["median_ms"] * 1e-3) / 1e9)
        builds.append(row)
        print(json.dumps(row))
    report["a_build_per_level"] = builds
    solves = {k: var[k] for k in ("fp32-3C", "fp32-F2", "bf16-F2")}
    fns = {k: (lambda lv=v: ops.lm_run(lv, 5, sc.R0, sc.T0, sc.W0, lambda_fixed=0.05)) for k, v in solves.items()}
    t = alternate(fns, max(5, args.reps // 2), warm=1)
    outs = {k: fn() for k, fn in fns.items()}
    fin = sc.levels[-1]
    depth = lambda W: fin.D + fin.B @ W
    ref = outs["fp32-3C"]
    report["b_solve"] = {k: dict(t[k], W_rel_vs_fp32_3C=rel(o[2], ref[2]), depth_rel_vs_fp32_3C=rel(depth(o[2]), depth(ref[2])),
                                 W_rel_vs_planted=rel(o[2], sc.W_true)) for k, o in outs.items()}
    print(json.dumps(report["b_solve"]))
    del var, solves, fns, outs, sc
    torch.cuda.empty_cache()

    # ---- (c) host pipeline step
    rs = synth.make_resize_scene(nb, 480, 640, C, K, level_ids=(0, 1, 2, 3), seed=1234 + 3, device=dev)
    pin = lambda x: x.cpu().pin_memory()
    hb, hd, hi = pin(rs.basis), pin(rs.init_depth), pin(rs.intr)
    R0, T0, W0 = pin(rs.R0), pin(rs.T0), pin(rs.W0)
    solvers = {"fp32": ResizeHostSolver([pin(l) for l in rs.layers], hb, hd, hi, rs.scales, chunks=4),
               "bf16": ResizeHostSolver([pin(l.to(BF)) for l in rs.layers], hb, hd, hi, rs.scales, chunks=4)}
    del rs
    torch.cuda.empty_cache()
    fns = {k: (lambda s=s: s.solve(R0, T0, W0, 5, lambda_fixed=0.05)) for k, s in solvers.items()}
    t = alternate(fns, max(5, args.reps // 2), warm=1)
    outs = {k: fn() for k, fn in fns.items()}
    report["c_e2e_host_step"] = {k: dict(t[k], h2d_bytes=solvers[k].h2d_bytes, W_rel_vs_fp32=rel(outs[k][2], outs["fp32"][2])) for k in solvers}
    print(json.dumps(report["c_e2e_host_step"]))
    del solvers, fns, outs
    torch.cuda.empty_cache()

    # ---- (d) one differentiable iteration, dense 320x240, F2 layout
    sc = synth.make_scene(nb=8, H=240, W=320, C=C, K=K, level_ids=(3,), seed=1234 + 4, device=dev, dtype=torch.float32)
    l = sc.levels[0]
    g = torch.Generator().manual_seed(3)
    dims = [C, 2 * C, 4 * C, 2 * C, C, 1]
    mlp = [((torch.randn(dims[i], dims[i + 1], generator=g) * (2.0 / dims[i]) ** 0.5).cuda().requires_grad_(), torch.zeros(dims[i + 1], device=dev).requires_grad_())
           for i in range(5)]
    train = {}
    for name, dt in (("fp32-F2", torch.float32), ("bf16-F2", BF)):
        c1 = l.conv1.to(dt).requires_grad_(); c2 = l.conv2[..., :C].contiguous().to(dt).requires_grad_()
        B = l.B.clone().requires_grad_(); R = sc.R0.clone().requires_grad_(); T = sc.T0.clone().requires_grad_(); W = sc.W0.clone().requires_grad_()

        def step(c1=c1, c2=c2, B=B, R=R, T=T, W=W):
            Rn, Tn, Wn = ag.iteration_fused(c1, c2, l.intr, l.p, l.D, B, R, T, W, mlp, 1000.0, precision=_lib.PREC_AUTO, grid=l.grid)
            (Rn.sum() + Tn.sum() + Wn.sum()).backward()
        train[name] = step
    peaks = {}
    for k, fn in train.items():
        fn(); torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(); base = torch.cuda.memory_allocated()
        fn(); torch.cuda.synchronize()
        peaks[k] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    t = alternate(train, args.reps)
    report["d_training_iteration_320x240"] = {k: dict(t[k], peak_extra_MiB=peaks[k]) for k in train}
    print(json.dumps(report["d_training_iteration_320x240"]))
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(report, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
