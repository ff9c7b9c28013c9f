"""Timing of the feature-metric cost (banet_lm_cost / banet_lm_cost_bwd) on an H100 against the build on the same tensors, and the default
bench line against a comparison tree (GPU).

    python scripts/time_cost.py [--base-tree /path/to/other/checkout] [--rounds 3] [--reps 8] [--bench-rounds 3] [--sections kernels,bench]
                                [--out profiles/h100_cost.json]

(a) lm_cost against lm_build at AUTO and at FP32_SIMT on bench.py's cfg2 scene at half its pairs (16 pairs, C = K = 128, dense levels
    80x60 .. 640x480, seed 1234+2), fp32 [F2|gx|gy] and bf16 F2-only, non-robust and Cauchy (delta = 4): the three calls alternate in
    each round.  Each case also reports the rate against the algorithmic bytes of the cost, N (2 C e_f + K e_b + 16) per pair (conv1 and
    one F2 sample per point, the basis row, D, p; e_f, e_b the element sizes of the features and the basis).
(b) one autograd.feature_metric_cost forward + backward at dense 320x240, 8 pairs, fp32 F2-only, next to one autograd.iteration_fused
    forward + backward (FP32_SIMT forward) on the same tensors, for scale.
(c) bench.py's default line of this tree and of --base-tree, alternated --bench-rounds times.
Cases (a) and (b) alternate their variants --rounds times, each round timing --reps calls after three warm-up calls (CUDA events); the
report gives median [min - max] per case, and the card name and power limit read in the same call.
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


def summary(ms, nbytes=None):
    out = {"median_ms": statistics.median(ms), "min_ms": min(ms), "max_ms": max(ms), "n": len(ms)}
    if nbytes:
        out["cost_bytes"] = nbytes
        out["GB_per_s_at_median"] = nbytes / (out["median_ms"] * 1e-3) / 1e9
    return out


def cost_bytes(nb, N, C, K, e_f, e_b):
    return nb * N * (2 * C * e_f + K * e_b + 16)


def kernels(rounds, reps):
    sys.path.insert(0, ROOT)
    import torch
    from banet_b200 import ops, synth, autograd as AG, _lib
    dev = torch.device("cuda")
    sc = synth.make_scene(nb=NB, H=480, W=640, C=128, K=128, level_ids=(0, 1, 2, 3), seed=1234 + 2, device=dev, dtype=torch.float32)
    names = ["80x60", "160x120", "320x240", "640x480"]
    groups = []
    for layout in ("fp32-3C", "bf16-F2"):
        for li, l in enumerate(sc.levels):
            c1, c2 = (l.conv1, l.conv2) if layout == "fp32-3C" else (l.conv1.bfloat16(), l.conv2[..., :128].bfloat16().contiguous())
            e_f = 4 if layout == "fp32-3C" else 2
            for kind in (None, "cauchy"):
                L = ops.Level(c1, c2, l.intr, l.p, l.D, l.B, grid=l.grid, robust=kind, robust_scale=4.0 if kind else 0.0)
                tag = f"{layout} {names[li]} {kind or 'non-robust'}"
                nbytes = cost_bytes(NB, l.N, 128, 128, e_f, 4)
                groups.append(({f"(a) lm_cost {tag}": (lambda L=L: ops.lm_cost(L, sc.R0, sc.T0, sc.W0)),
                                f"(a) lm_build AUTO {tag}": (lambda L=L: ops.lm_build(L, sc.R0, sc.T0, sc.W0, precision=_lib.PREC_AUTO)),
                                f"(a) lm_build FP32_SIMT {tag}": (lambda L=L: ops.lm_build(L, sc.R0, sc.T0, sc.W0, precision=_lib.PREC_FP32_SIMT))},
                               nbytes))
        del c1, c2
    l2 = sc.levels[2]
    nb8 = 8
    sl = lambda t: t[:nb8].contiguous()
    F2 = sl(l2.conv2)[..., :128].contiguous()
    dims = [128, 256, 512, 256, 128, 1]
    gm = torch.Generator().manual_seed(9)
    mlp = [((torch.randn(dims[i], dims[i + 1], generator=gm) * (2.0 / dims[i]) ** 0.5).cuda(), torch.zeros(dims[i + 1], device=dev)) for i in range(5)]

    def leaves():
        return sl(l2.conv1).requires_grad_(), F2.clone().requires_grad_(), sl(l2.B).requires_grad_(), sl(sc.W0).requires_grad_()

    def cost_step():
        conv1, f2, B, W = leaves()
        AG.feature_metric_cost(conv1, f2, sl(l2.D), B, sl(sc.R0), sl(sc.T0), W, sl(l2.intr), sl(l2.p), grid=l2.grid).sum().backward()

    def train_step():
        conv1, f2, B, W = leaves()
        R, T, Wn = AG.iteration_fused(conv1, f2, sl(l2.intr), sl(l2.p), sl(l2.D), B, sl(sc.R0), sl(sc.T0), W, mlp, 1000.0, grid=l2.grid)
        (R.sum() + T.sum() + Wn.sum()).backward()

    groups.append(({"(b) feature_metric_cost fwd+bwd 320x240 x8 F2": cost_step, "(b) iteration_fused fwd+bwd 320x240 x8 F2": train_step}, None))
    out = {}
    for g, nbytes in groups:
        ms = {k: [] for k in g}
        for _ in range(rounds):
            for k, fn in g.items():
                ms[k] += timed(fn, reps)
        for k in g:
            out[k] = summary(ms[k], nbytes if k.startswith("(a) lm_cost") else None)
            print(k, out[k], flush=True)
    return out


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
            print("bench", name, runs[name][-1], flush=True)
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
    ap.add_argument("--bench-rounds", type=int, default=3)
    ap.add_argument("--sections", default="kernels,bench")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_cost.json"))
    a = ap.parse_args()
    sections = a.sections.split(",")
    rep = {}
    if os.path.exists(a.out):
        with open(a.out) as f:
            rep = json.load(f)
    gpu = gpu_identity()
    if "kernels" in sections:
        rep["kernels"] = {"gpu": gpu, "rounds": a.rounds, "reps_per_round": a.reps, "pairs": NB, "cases": kernels(a.rounds, a.reps)}
    if "bench" in sections and a.base_tree:
        rep["bench_default_line"] = {"gpu": gpu, "runs": bench_lines(os.path.abspath(a.base_tree), a.bench_rounds)}
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rep, f, indent=1)
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    main()
