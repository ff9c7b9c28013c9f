"""Cost of the robust losses (banet_level_t::robust) on an H100, the non-robust build against a comparison library, and the default bench line
against a comparison tree (GPU).

    python scripts/time_robust.py --base-lib /path/to/other/libbanet.so --base-tree /path/to/other/checkout [--rounds 3] [--reps 8]
                                  [--bench-rounds 3] [--out profiles/h100_robust.json]

(a) lm_build at AUTO, non-robust, on bench.py's cfg2 scene at half its pairs (16 pairs, C = K = 128, dense levels 80x60 .. 640x480, seed 1234+2), fp32 [F2|gx|gy]
    and bf16 F2-only: this library against --base-lib, both loaded in this process (one level per call, so the comparison library reads
    the leading fields of the level struct it knows);
(b) the same levels on this library with Huber and Cauchy (delta = 4) against non-robust;
(c) one differentiable iteration (autograd.iteration_fused, FP32_SIMT forward, 8 pairs, dense 320x240, F2-only), forward + backward,
    Cauchy against non-robust;
(d) bench.py's default line of this tree and of --base-tree, alternated --bench-rounds times;
(e) the planted-outlier scene (tests/test_robust.py: 20 % of conv1 rows replaced by other points' features, 2 levels x 3 iterations,
    lambda 0.01, delta 1): pose errors |R - R*|_F + |T - T*| of the FP32_SIMT solve with L2, Huber and Cauchy.
Cases (a)-(c) alternate their variants --rounds times, each round timing --reps calls after three warm-up calls (CUDA events).  The
report gives median [min - max] per case, and the card name and power limit read in the same call.  --sections picks what runs (default
all: kernels = (a)-(c), outliers = (e), bench = (d)); the sections run are written into --out, keeping the others it already holds, and
bench values add to the ones it holds (rounds of one order per call, --base-first for the other).
"""
import argparse, json, os, statistics, subprocess, sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
NB = 16        # pairs of the kernel scenes: cfg2 has 32; at 640x480 the fp32 3C maps and their bf16 copies need more free memory than a shared card may have


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


def kernels(base_lib, rounds, reps):
    sys.path.insert(0, ROOT)
    import torch
    from banet_b200 import ops, synth, autograd as AG, _lib
    handles = {"this": _lib.load()}
    if base_lib:
        _lib._lib, _lib.LIB_PATH = None, os.path.abspath(base_lib)
        handles["base"] = _lib.load()
        _lib._lib = handles["this"]

    def on(name, fn):
        def run():
            _lib._lib = handles[name]
            try:
                return fn()
            finally:
                _lib._lib = handles["this"]
        return run

    dev = torch.device("cuda")
    sc = synth.make_scene(nb=NB, H=480, W=640, C=128, K=128, level_ids=(0, 1, 2, 3), seed=1234 + 2, device=dev, dtype=torch.float32)
    names = ["80x60", "160x120", "320x240", "640x480"]
    groups = []
    for layout in ("fp32-3C", "bf16-F2"):
        for li, l in enumerate(sc.levels):
            c1, c2 = (l.conv1, l.conv2) if layout == "fp32-3C" else (l.conv1.bfloat16(), l.conv2[..., :128].bfloat16().contiguous())
            lv = {k: ops.Level(c1, c2, l.intr, l.p, l.D, l.B, grid=l.grid, robust=k, robust_scale=4.0 if k else 0.0) for k in (None, "huber", "cauchy")}
            build = lambda L: (lambda: ops.lm_build(L, sc.R0, sc.T0, sc.W0, precision=_lib.PREC_AUTO))
            g = {f"(a) lm_build {layout} {names[li]} non-robust, this library": build(lv[None])}
            if base_lib:
                g[f"(a) lm_build {layout} {names[li]} non-robust, base library"] = on("base", build(lv[None]))
            groups.append(g)
            groups.append({f"(b) lm_build {layout} {names[li]} {k or 'non-robust'}": build(lv[k]) for k in (None, "huber", "cauchy")})
        del c1, c2
    l2 = sc.levels[2]
    nb8 = 8
    sl = lambda t: t[:nb8].contiguous()
    F2 = sl(l2.conv2)[..., :128].contiguous()
    dims = [128, 256, 512, 256, 128, 1]
    gm = torch.Generator().manual_seed(9)
    mlp = [((torch.randn(dims[i], dims[i + 1], generator=gm) * (2.0 / dims[i]) ** 0.5).cuda(), torch.zeros(dims[i + 1], device=dev)) for i in range(5)]

    def train_step(robust):
        conv1 = sl(l2.conv1).requires_grad_(); f2 = F2.clone().requires_grad_(); B = sl(l2.B).requires_grad_()
        R, T, W = AG.iteration_fused(conv1, f2, sl(l2.intr), sl(l2.p), sl(l2.D), B, sl(sc.R0), sl(sc.T0), sl(sc.W0), mlp, 1000.0,
                                     grid=l2.grid, robust=robust, robust_scale=4.0)
        (R.sum() + T.sum() + W.sum()).backward()

    groups.append({"(c) iteration_fused fwd+bwd 320x240 x8 F2 non-robust": lambda: train_step(None),
                   "(c) iteration_fused fwd+bwd 320x240 x8 F2 cauchy": lambda: train_step("cauchy")})
    ms = {}
    for g in groups:
        for k in g:
            ms[k] = []
        for _ in range(rounds):
            for k, fn in g.items():
                ms[k] += timed(fn, reps)
        for k in g:
            print(k, summary(ms[k]), flush=True)
    return {k: summary(v) for k, v in ms.items()}


def outliers():
    """(e): the planted-outlier scene of tests/test_robust.py, built from synth alone."""
    sys.path.insert(0, ROOT)
    import torch
    from banet_b200 import ops, synth, _lib
    sc = synth.make_scene(nb=1, H=96, W=128, C=16, K=16, level_ids=(2, 3), seed=71, dtype=torch.float64)
    g = torch.Generator().manual_seed(71)
    for lv in sc.levels:
        bad = torch.randperm(lv.N, generator=g)[: int(0.2 * lv.N)]
        src = torch.randperm(lv.N, generator=g)[: bad.numel()]
        lv.conv1[:, bad] = lv.conv1[:, src].clone()
    cu = lambda t: t.to("cuda", torch.float32).contiguous()
    out = {}
    for kind in (None, "huber", "cauchy"):
        levels = [ops.Level(cu(l.conv1), cu(l.conv2), cu(l.intr), cu(l.p), cu(l.D), cu(l.B), grid=l.grid, robust=kind,
                            robust_scale=1.0 if kind else 0.0) for l in sc.levels]
        R, T, W, st = ops.lm_run(levels, 3, cu(sc.R0), cu(sc.T0), cu(sc.W0), lambda_fixed=0.01, l2_regularizer_base=1000.0,
                                 precision=_lib.PREC_FP32_SIMT)
        err = float((R.cpu().double() - sc.R_true).norm() + (T.cpu().double() - sc.T_true).norm())
        out[kind or "l2"] = {"pose_error": err, "status": int(st.abs().max())}
    return out


def bench_lines(base_tree, rounds, runs=None, base_first=False):
    """bench.py's default line (--gpus 1 --steps 5 --warmup 3) of this tree and of base_tree, alternated; appended to the values in runs
    (earlier calls).  base_first: each round starts with base_tree (an earlier call can measure the other order)."""
    runs = {"this tree": [], "base tree": []} if runs is None else {k: list(v["values"]) for k, v in runs.items()}
    order = (("this tree", ROOT), ("base tree", base_tree))
    for _ in range(rounds):
        for name, tree in (order[::-1] if base_first else order):
            out = subprocess.run([sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", "5", "--warmup", "3"],
                                 capture_output=True, text=True, cwd=tree, timeout=1800)
            line = [x for x in out.stdout.splitlines() if x.startswith("{")]
            if out.returncode != 0 or not line:
                raise RuntimeError(f"bench.py in {tree} failed: {out.stderr[-2000:]}")
            runs[name].append(json.loads(line[-1])["value"])
            print("bench", name, runs[name][-1], flush=True)
    return {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "values": v, "unit": "pair-iters/s"} for k, v in runs.items()}


def gpu_identity():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
    return {"name": q[0], "power_limit_w": float(q[1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base-lib", default=None, help="a comparison libbanet.so for (a)")
    ap.add_argument("--base-tree", default=None, help="a checkout (library built) whose bench.py line is compared with this tree's")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=8)
    ap.add_argument("--bench-rounds", type=int, default=3)
    ap.add_argument("--sections", default="kernels,outliers,bench")
    ap.add_argument("--base-first", action="store_true", help="bench rounds start with --base-tree")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_robust.json"))
    a = ap.parse_args()
    sections = a.sections.split(",")
    rep = {}
    if os.path.exists(a.out):
        with open(a.out) as f:
            rep = json.load(f)
    gpu = gpu_identity()
    if "kernels" in sections:
        rep["kernels"] = {"gpu": gpu, "rounds": a.rounds, "reps_per_round": a.reps, "cases": kernels(a.base_lib, a.rounds, a.reps)}
    if "outliers" in sections:
        rep["planted_outliers"] = {"gpu": gpu, "errors": outliers()}
    if "bench" in sections and a.base_tree:
        prev = rep.get("bench_default_line", {}).get("runs")
        rep["bench_default_line"] = {"gpu": gpu, "runs": bench_lines(os.path.abspath(a.base_tree), a.bench_rounds, prev, a.base_first)}
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rep, f, indent=1)
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    main()
