"""Timing of the keyframe-window feature-metric cost (banet_lm_keyframe_cost / _bwd) on an H100 (GPU).

    python scripts/time_window_cost.py [--base-tree /path/to/other/checkout] [--rounds 3] [--reps 10] [--out profiles/h100_window_cost.json]

(a) ops.lm_keyframe_cost and ops.lm_keyframe_cost_bwd against ops.lm_cost / ops.lm_cost_bwd on the replicated layout, the per-frame copies
    of conv1, p, D, B and W (and the frame sums of the keyframe gradients) inside the timed call, at WindowResize's sparse (nw = 8, nf = 4,
    N = 4096, 64 x 80 maps) and dense (nw = 4, nf = 4, N = 81920, 256 x 320 maps) workloads, C = K = 128, F2-only fp32 maps; with the peak
    device memory of each call above what was allocated before it.
(b) one WindowResize training step (forward, loss, backward) with return_cost=False and with return_cost=True (the loss adds sum Es) at
    nw = 8, nf = 4, N = 4096, C = K = 128.
(c) bench.py's default line of this tree and of --base-tree, alternated.
The variants of a case alternate --rounds times, each round timing --reps calls after three warm-up calls (CUDA events); median [min - max].
The card's name and power limit are read in the same call.
"""
import argparse, json, os, statistics, subprocess, sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)


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


def peak_mib(fn):
    import torch
    torch.cuda.synchronize(); torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn(); torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def summary(ms):
    return {"median_ms": statistics.median(ms), "min_ms": min(ms), "max_ms": max(ms), "n": len(ms)}


def alternate(fns, rounds, reps):
    ms = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            ms[k] += timed(fn, reps)
    return {k: summary(v) for k, v in ms.items()}


def window_level(nw, nf, N, C, K, h, w, seed):
    import torch
    from banet_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.rand(*s, device="cuda", generator=g)
    nb = nw * nf
    fx, fy, ox, oy = 0.9 * w, 0.9 * w, (w - 1) / 2, (h - 1) / 2
    u, v = r(nw, N) * (w - 1), r(nw, N) * (h - 1)
    p = torch.stack([(u - ox) / fx, (v - oy) / fy, torch.ones_like(u)], 1)
    p = (p / p.norm(dim=1, keepdim=True)).contiguous()
    D, B, W = 2.0 + r(nw, N, 1), 0.01 * (r(nw, N, K) - 0.5), 0.1 * (r(nw, K, 1) - 0.5)
    intr = torch.tensor([fx, fy, ox, oy], device="cuda").expand(nb, 4).contiguous()
    th = 0.01 * (r(nb, 3) - 0.5)
    z = torch.zeros_like(th[:, 0])
    S = torch.stack([torch.stack([z, -th[:, 2], th[:, 1]], -1), torch.stack([th[:, 2], z, -th[:, 0]], -1), torch.stack([-th[:, 1], th[:, 0], z], -1)], -2)
    R, T = torch.linalg.matrix_exp(S).contiguous(), (0.02 * (r(nb, 3, 1) - 0.5)).contiguous()
    key = ops.KeyframeLevel(r(nw, N, C), r(nb, h, w, C), intr, p, D, B)
    return key, R, T, W


def kernels(rounds, reps):
    import torch
    from banet_b200 import ops
    out = {}
    for name, (nw, nf, N, h, w) in (("sparse nw=8 nf=4 N=4096 64x80", (8, 4, 4096, 64, 80)),
                                    ("dense nw=4 nf=4 N=81920 256x320", (4, 4, 81920, 256, 320))):
        key, R, T, W = window_level(nw, nf, N, 128, 128, h, w, seed=11)
        dcost = torch.linspace(-1.0, 1.0, nw * nf, device="cuda")
        rp = lambda t: t.repeat_interleave(nf, 0)
        fs = lambda t: t.reshape(nw, nf, *t.shape[1:]).sum(1)

        def rep_level():
            return ops.Level(rp(key.conv1), key.conv2, key.intr, rp(key.p), rp(key.D), rp(key.B))

        fns = {"keyframe cost fwd": lambda: ops.lm_keyframe_cost(key, R, T, W),
               "pair cost fwd, replicated (copies included)": lambda: ops.lm_cost(rep_level(), R, T, rp(W)),
               "keyframe cost bwd": lambda: ops.lm_keyframe_cost_bwd(key, R, T, W, dcost),
               "pair cost bwd, replicated (copies and frame sums included)":
                   lambda: [fs(t) if i in (0, 2, 3, 6) else t for i, t in enumerate(ops.lm_cost_bwd(rep_level(), R, T, rp(W), dcost))]}
        res = alternate(fns, rounds, reps)
        for k, fn in fns.items():
            res[k]["peak_MiB"] = peak_mib(fn)
            print(name, k, res[k], flush=True)
        a = ops.lm_keyframe_cost(key, R, T, W)
        b = ops.lm_cost(rep_level(), R, T, rp(W))
        res["outputs bitwise equal"] = bool(torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]))
        out[name] = res
        del key
    return out


def resize_step(rounds, reps):
    import torch
    from banet_b200.bundlenet import BundleNet
    from banet_b200 import _lib
    nw, nf, N, C, K = 8, 4, 4096, 128, 128
    g = torch.Generator(device="cuda").manual_seed(3)
    r = lambda *s: torch.rand(*s, device="cuda", generator=g)
    key = [r(nw, 32 * 2 ** l, 40 * 2 ** l, C) for l in range(4)]
    frames = [r(nw, nf, 32 * 2 ** l, 40 * 2 ** l, C) for l in range(4)]
    intr = torch.tensor([280.0, 280.0, 160.0, 128.0], device="cuda").reshape(1, 4, 1).expand(nw, 4, 1).contiguous()
    points = torch.stack([4 + r(nw, N) * 300, 4 + r(nw, N) * 220], -1)
    basis, depth = 0.01 * (r(nw, 128, 160, K) - 0.5), 2.0 + r(nw, 128, 160, 1)
    net = BundleNet(C, levels=("2", "3"), precision=_lib.PREC_FP32_SIMT).cuda().train()

    def step(return_cost):
        kl = [t.clone().requires_grad_() for t in key]
        out = net.WindowResize(intr, kl, frames, points, basis, depth, return_cost=return_cost)
        loss = sum(t.sum() for t in out[0] + out[1] + out[2])
        if return_cost:
            loss = loss + sum(e.sum() for e in out[3])
        loss.backward()

    fns = {"WindowResize training step": lambda: step(False), "WindowResize training step, return_cost=True": lambda: step(True)}
    res = alternate(fns, rounds, reps)
    for k, fn in fns.items():
        res[k]["peak_MiB"] = peak_mib(fn)
        print(k, res[k], flush=True)
    return {"shape": dict(nw=nw, nf=nf, N=N, C=C, K=K), **res}


def bench_lines(base_tree, rounds):
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
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--bench-rounds", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_window_cost.json"))
    a = ap.parse_args()
    rep = {"script": "scripts/time_window_cost.py", "gpu": gpu_identity(), "rounds": a.rounds, "reps_per_round": a.reps}
    rep["kernels"] = kernels(a.rounds, a.reps)
    rep["window_resize_training_step"] = resize_step(a.rounds, max(a.reps // 2, 3))
    if a.base_tree:
        rep["bench_default_line"] = bench_lines(os.path.abspath(a.base_tree), a.bench_rounds)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rep, f, indent=1)
    print(json.dumps(rep, indent=1))


if __name__ == "__main__":
    main()
