"""bfloat16 against float32 depth basis on the GPU: build per level, the dropped split-A pass, whole solve, host-pipeline step, one training
iteration.

    python scripts/time_bf16_basis.py [--reps 20] [--out profiles/h100_bf16_basis.json]

(a) lm_build per cfg2 level (80x60 .. 640x480, 32 pairs, C = K = 128, AUTO) with an fp32 and a bf16 basis, on bf16 F2 features and on
    fp32 3C features, with the achieved bytes/s against each variant's algorithmic bytes (conv1 + conv2 + basis + p + D, each read once).
(b) TF32X2 at K = 64 and K = 32 at 640x480 (the first 64 / 32 basis columns of (a)'s scene), fp32 against bf16 basis: the bf16 basis
    makes it one MMA pass instead of two.
(c) the whole 4-level solve (5 iterations per level, fixed lambda, AUTO, bf16 F2 features) on the fp32 basis and on its bf16 rounding, with
    the W and finest-level depth difference of the bf16-basis solve against the fp32-basis solve on the unrounded basis.
(d) one ResizeHostSolver step (32 images, 4 levels, pinned host inputs, bf16 pyramid) with an fp32 and a bf16 host basis, with the H2D bytes.
(e) one differentiable iteration (autograd.iteration_fused, bf16 F2 features) at dense 320x240, 8 pairs, fp32 against bf16 basis: forward +
    backward time and peak memory.
Every case is warmed up, then the variants of a group are timed alternately, `--reps` times each (CUDA events); the report gives the
median and min - max.  The card's name and power limit are read in the same run.
"""
import argparse, json, os, sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from time_bf16_features import alternate, card        # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_bf16_basis.json"))
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

    # ---- (a) build per level
    sc = synth.make_scene(nb=nb, H=480, W=640, C=C, K=K, level_ids=(0, 1, 2, 3), seed=1234 + 2, device=dev, dtype=torch.float32)
    Bbf = [l.B.to(BF) for l in sc.levels]
    var = {}
    for fname, dt, layout in (("bf16-F2", BF, "F2"), ("fp32-3C", torch.float32, "3C")):
        for bname in ("fp32", "bf16"):
            var[f"{fname}/B-{bname}"] = [ops.Level(l.conv1.to(dt), (l.conv2 if layout == "3C" else l.conv2[..., :C]).contiguous().to(dt), l.intr, l.p, l.D,
                                                   l.B if bname == "fp32" else Bbf[i], grid=l.grid) for i, l in enumerate(sc.levels)]
    builds = []
    for li, l in enumerate(sc.levels):
        N = l.N
        fns = {k: (lambda lv=v[li]: ops.lm_build(lv, sc.R0, sc.T0, sc.W0, _lib.PREC_AUTO)) for k, v in var.items()}
        t = alternate(fns, args.reps)
        row = {"level": f"{l.conv2.shape[2]}x{l.conv2.shape[1]}", "N": N}
        for k, v in var.items():
            lv = v[li]
            by = nb * N * ((C + lv.conv2.shape[-1]) * lv.conv1.element_size() + K * lv.B.element_size() + 4 * 4)
            row[k] = dict(t[k], algorithmic_bytes=by, achieved_GBs=by / (t[k]["median_ms"] * 1e-3) / 1e9)
        builds.append(row)
        print(json.dumps(row))
    report["a_build_per_level"] = builds
    del var
    torch.cuda.empty_cache()

    # ---- (b) TF32X2 at K = 64 / 32, 640x480 (the second MMA pass is dropped on a bf16 basis)
    fin = sc.levels[-1]
    c1, c2 = fin.conv1.to(BF), fin.conv2[..., :C].contiguous().to(BF)
    smallk = {}
    for k in (64, 32):
        Bk = fin.B[..., :k].contiguous()
        Wk = sc.W0[:, :k].contiguous()
        lv = {"B-fp32": ops.Level(c1, c2, fin.intr, fin.p, fin.D, Bk, grid=fin.grid), "B-bf16": ops.Level(c1, c2, fin.intr, fin.p, fin.D, Bk.to(BF), grid=fin.grid)}
        fns = {n: (lambda v=v, Wk=Wk: ops.lm_build(v, sc.R0, sc.T0, Wk, _lib.PREC_TF32X2)) for n, v in lv.items()}
        smallk[f"K={k}"] = alternate(fns, args.reps)
        print(json.dumps({f"K={k}": smallk[f"K={k}"]}))
        del lv, fns, Bk
    report["b_tf32x2_smallk_640x480"] = smallk
    del c1, c2
    torch.cuda.empty_cache()

    # ---- (c) whole solve on bf16 F2 features
    mk = lambda l, B: ops.Level(l.conv1.to(BF), l.conv2[..., :C].contiguous().to(BF), l.intr, l.p, l.D, B, grid=l.grid)
    solves = {"B-fp32": [mk(l, l.B) for l in sc.levels], "B-bf16": [mk(l, Bbf[i]) for i, l in enumerate(sc.levels)]}
    fns = {k: (lambda lv=v: ops.lm_run(lv, 5, sc.R0, sc.T0, sc.W0, lambda_fixed=0.05)) for k, v in solves.items()}
    t = alternate(fns, max(5, args.reps // 2), warm=1)
    outs = {k: fn() for k, fn in fns.items()}
    depth = lambda W: fin.D + fin.B @ W                     # the unrounded basis
    ref = outs["B-fp32"]
    report["c_solve_bf16_F2"] = {k: dict(t[k], W_rel_vs_fp32_basis=rel(o[2], ref[2]), depth_rel_vs_fp32_basis=rel(depth(o[2]), depth(ref[2])),
                                         W_rel_vs_planted=rel(o[2], sc.W_true)) for k, o in outs.items()}
    print(json.dumps(report["c_solve_bf16_F2"]))
    del solves, fns, outs, sc, Bbf, fin
    torch.cuda.empty_cache()

    # ---- (d) host pipeline step, bf16 pyramid
    rs = synth.make_resize_scene(nb, 480, 640, C, K, level_ids=(0, 1, 2, 3), seed=1234 + 3, device=dev)
    pin = lambda x: x.cpu().pin_memory()
    hl = [pin(l.to(BF)) for l in rs.layers]
    hd, hi = pin(rs.init_depth), pin(rs.intr)
    R0, T0, W0 = pin(rs.R0), pin(rs.T0), pin(rs.W0)
    solvers = {"B-fp32": ResizeHostSolver(hl, pin(rs.basis), hd, hi, rs.scales, chunks=4),
               "B-bf16": ResizeHostSolver(hl, pin(rs.basis.to(BF)), hd, hi, rs.scales, chunks=4)}
    del rs
    torch.cuda.empty_cache()
    fns = {k: (lambda s=s: s.solve(R0, T0, W0, 5, lambda_fixed=0.05)) for k, s in solvers.items()}
    t = alternate(fns, max(5, args.reps // 2), warm=1)
    outs = {k: fn() for k, fn in fns.items()}
    report["d_e2e_host_step_bf16_pyramid"] = {k: dict(t[k], h2d_bytes=solvers[k].h2d_bytes, W_rel_vs_fp32_basis=rel(outs[k][2], outs["B-fp32"][2]))
                                              for k in solvers}
    print(json.dumps(report["d_e2e_host_step_bf16_pyramid"]))
    del solvers, fns, outs
    torch.cuda.empty_cache()

    # ---- (e) one differentiable iteration, dense 320x240, bf16 F2 features
    sc = synth.make_scene(nb=8, H=240, W=320, C=C, K=K, level_ids=(3,), seed=1234 + 4, device=dev, dtype=torch.float32)
    l = sc.levels[0]
    g = torch.Generator().manual_seed(3)
    dims = [C, 2 * C, 4 * C, 2 * C, C, 1]
    mlp = [((torch.randn(dims[i], dims[i + 1], generator=g) * (2.0 / dims[i]) ** 0.5).cuda().requires_grad_(), torch.zeros(dims[i + 1], device=dev).requires_grad_())
           for i in range(5)]
    train = {}
    for name, bdt in (("B-fp32", torch.float32), ("B-bf16", BF)):
        c1 = l.conv1.to(BF).requires_grad_(); c2 = l.conv2[..., :C].contiguous().to(BF).requires_grad_()
        B = l.B.to(bdt).requires_grad_(); R = sc.R0.clone().requires_grad_(); T = sc.T0.clone().requires_grad_(); W = sc.W0.clone().requires_grad_()

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
    report["e_training_iteration_320x240"] = {k: dict(t[k], peak_extra_MiB=peaks[k], basis_MiB=l.B.numel() * (2 if k == "B-bf16" else 4) / 2 ** 20)
                                              for k in train}
    print(json.dumps(report["e_training_iteration_320x240"]))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(report, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
