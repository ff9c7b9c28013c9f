"""Cost of per-point weights (banet_level_t::weight) on an H100, and the default bench line against a comparison tree (GPU).

    python scripts/time_point_weights.py [--base-tree /path/to/other/checkout] [--rounds 3] [--reps 8] [--bench-rounds 2] [--out profiles/h100_point_weights.json]

(a) lm_build at AUTO on bench.py's cfg2 scene at half its pairs (nb=16, C=K=128, dense levels 80x60 .. 640x480, seed 1234+2), fp32 [F2|gx|gy] and bf16
    F2-only, each unweighted and weighted (weights in [0.5, 1.5]);
(b) a 4-level lm_run, 5 iterations per level, lambda fixed, unweighted and weighted;
(c) one differentiable iteration (autograd.iteration_fused, FP32_SIMT forward, 8 pairs, dense 320x240, F2-only), forward + backward,
    without a weight and with a weight that requires grad;
(d) bench.py's default line of this tree and of --base-tree, alternated --bench-rounds times in one call.
Cases (a)-(c) alternate the unweighted and weighted variants --rounds times, each round timing --reps calls after three warm-up calls
(CUDA events).  The report gives median [min - max] per case, and the card name and power limit read in the same call.
"""
import argparse, json, os, statistics, subprocess, sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
NB = 16        # pairs of the kernel scenes: cfg2's 32 at 640x480 plus the bf16 copies need more free device memory than a shared card may have


def timed(fn, reps):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return ms


def summary(ms):
    return {"median_ms": statistics.median(ms), "min_ms": min(ms), "max_ms": max(ms), "n": len(ms)}


def kernels(rounds, reps):
    sys.path.insert(0, ROOT)
    import torch
    from banet_b200 import ops, synth, autograd as AG, _lib
    dev = torch.device("cuda")
    sc = synth.make_scene(nb=NB, H=480, W=640, C=128, K=128, level_ids=(0, 1, 2, 3), seed=1234 + 2, device=dev, dtype=torch.float32)
    g = torch.Generator(device="cuda").manual_seed(0)
    wts = [0.5 + torch.rand(NB, l.N, 1, device=dev, generator=g) for l in sc.levels]
    names = ["80x60", "160x120", "320x240", "640x480"]
    cases = {}
    for layout in ("fp32-3C", "bf16-F2"):
        for li, l in enumerate(sc.levels):
            c1, c2 = (l.conv1, l.conv2) if layout == "fp32-3C" else (l.conv1.bfloat16(), l.conv2[..., :128].bfloat16().contiguous())
            for wname, w in (("unweighted", None), ("weighted", wts[li])):
                lv = ops.Level(c1, c2, l.intr, l.p, l.D, l.B, grid=l.grid, weight=w)
                cases[f"(a) lm_build {layout} {names[li]} {wname}"] = (lambda lv=lv: ops.lm_build(lv, sc.R0, sc.T0, sc.W0, precision=_lib.PREC_AUTO))
    for wname, use in (("unweighted", False), ("weighted", True)):
        lvs = [ops.Level(l.conv1, l.conv2, l.intr, l.p, l.D, l.B, grid=l.grid, weight=wts[i] if use else None) for i, l in enumerate(sc.levels)]
        cases[f"(b) lm_run 4 levels x 5 iters {wname}"] = (lambda lvs=lvs: ops.lm_run(lvs, 5, sc.R0, sc.T0, sc.W0, lambda_fixed=0.01, precision=_lib.PREC_AUTO))
    l2 = sc.levels[2]
    nb8 = 8
    sl = lambda t: t[:nb8].contiguous()
    F2 = sl(l2.conv2)[..., :128].contiguous()
    dims = [128, 256, 512, 256, 128, 1]                                  # the lambda-MLP (he_normal filters, zero biases)
    gm = torch.Generator().manual_seed(9)
    mlp = [((torch.randn(dims[i], dims[i + 1], generator=gm) * (2.0 / dims[i]) ** 0.5).cuda(), torch.zeros(dims[i + 1], device=dev)) for i in range(5)]
    w8 = (0.5 + torch.rand(nb8, l2.N, 1, device=dev, generator=g))

    def train_step(weight):
        conv1 = sl(l2.conv1).requires_grad_(); f2 = F2.clone().requires_grad_(); B = sl(l2.B).requires_grad_()
        wt = None if weight is None else weight.clone().requires_grad_()
        R, T, W = AG.iteration_fused(conv1, f2, sl(l2.intr), sl(l2.p), sl(l2.D), B, sl(sc.R0), sl(sc.T0), sl(sc.W0), mlp, 1000.0,
                                     grid=l2.grid, weight=wt)
        (R.sum() + T.sum() + W.sum()).backward()

    cases["(c) iteration_fused fwd+bwd 320x240 x8 F2 unweighted"] = lambda: train_step(None)
    cases["(c) iteration_fused fwd+bwd 320x240 x8 F2 weighted (requires grad)"] = lambda: train_step(w8)
    ms = {k: [] for k in cases}
    for _ in range(rounds):
        for k, fn in cases.items():
            ms[k] += timed(fn, reps)
    return {k: summary(v) for k, v in ms.items()}


def bench_lines(base_tree, rounds):
    """bench.py's default line (--gpus 1 --steps 5 --warmup 3) of this tree and of base_tree, alternated."""
    runs = {"this tree": [], "base tree": []}
    for _ in range(rounds):
        for name, tree in (("this tree", ROOT), ("base tree", base_tree)):
            out = subprocess.run([sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", "5", "--warmup", "3"],
                                 capture_output=True, text=True, cwd=tree, timeout=1800)
            line = [x for x in out.stdout.splitlines() if x.startswith("{")]
            if out.returncode != 0 or not line:
                raise RuntimeError(f"bench.py in {tree} failed: {out.stderr[-2000:]}")
            runs[name].append(json.loads(line[-1])["value"])
    return {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "values": v, "unit": "pair-iters/s"} for k, v in runs.items()}


def gpu_identity():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
    return {"name": q[0], "power_limit_w": float(q[1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base-tree", default=None, help="a checkout (library built) whose bench.py line is compared with this tree's")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=8)
    ap.add_argument("--bench-rounds", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_point_weights.json"))
    a = ap.parse_args()
    rep = {"gpu": gpu_identity(), "rounds": a.rounds, "reps_per_round": a.reps}
    rep["kernels"] = kernels(a.rounds, a.reps)
    if a.base_tree:
        rep["bench_default_line"] = bench_lines(os.path.abspath(a.base_tree), a.bench_rounds)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rep, f, indent=1)
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    main()
