"""Forward + backward of one differentiable keyframe-window iteration (banet_b200.autograd.window_iteration_fused) against the same 4 frames as
4 independent pairs (autograd.iteration_fused), timed with CUDA events in alternation.  nf = 4, C = K = 128 (BA-Net's 5-frame setting):
4096 sampled points per frame (the reference's training regime) and a dense 320x240 level.  Prints one JSON document with the card's name and
power limit; --out also writes it to a file."""
import argparse, json, os, statistics, subprocess, sys
import torch
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from banet_b200 import synth, autograd as ag, _lib


def card():
    """The card's name and power limit: an absolute time means little without them."""
    name, limit = torch.cuda.get_device_name(), "unknown"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    if q.returncode == 0 and q.stdout.strip():
        name, limit = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")][:2]
    return {"gpu": name, "power_limit": limit}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    _lib.require_device()
    nf, C, K = 4, 128, 128
    g = torch.Generator().manual_seed(7); dims = [C, 2 * C, 4 * C, 2 * C, C, 1]       # he_normal filters, zero biases (bundlenet.py:102-110)
    mlp = [((torch.randn(dims[i], dims[i + 1], generator=g) * (2.0 / dims[i]) ** 0.5).cuda().requires_grad_(), torch.zeros(dims[i + 1], device="cuda").requires_grad_())
           for i in range(5)]
    rows = []
    for label, H, W, npts in (("sparse4096", 120, 160, 4096), ("dense320x240", 240, 320, None)):
        sc = synth.make_scene(nb=nf, H=H, W=W, C=C, K=K, level_ids=(3,), seed=21, device="cuda", dtype=torch.float32, n_points=npts, shared_depth=True)
        lv = sc.levels[0]
        leaf = lambda t: t.detach().clone().requires_grad_()
        conv1, conv2, D, B, R, T = leaf(lv.conv1), leaf(lv.conv2), leaf(lv.D), leaf(lv.B), leaf(sc.R0), leaf(sc.T0)
        Wwin, Wpairs = leaf(sc.W0[0]), leaf(sc.W0)
        def window():
            Rn, Tn, Wn = ag.window_iteration_fused(conv1, conv2, lv.intr, lv.p, D, B, R, T, Wwin, mlp, 1000.0, grid=lv.grid)
            return Rn.sum() + Tn.sum() + (Wn * Wn).sum()
        def pairs():
            Rn, Tn, Wn = ag.iteration_fused(conv1, conv2, lv.intr, lv.p, D, B, R, T, Wpairs, mlp, 1000.0, grid=lv.grid)
            return Rn.sum() + Tn.sum() + (Wn * Wn).sum()
        ev = lambda: torch.cuda.Event(enable_timing=True)
        times = {"window": ([], []), "pairs": ([], [])}
        for it in range(args.warmup + args.reps):
            for name, fn in (("window", window), ("pairs", pairs)):             # alternate the two in one loop: same clocks, same neighbours
                for t in (conv1, conv2, D, B, R, T, Wwin, Wpairs, *[x for wb in mlp for x in wb]):
                    t.grad = None
                e0, e1, e2 = ev(), ev(), ev()
                e0.record(); loss = fn(); e1.record(); loss.backward(); e2.record()
                torch.cuda.synchronize()
                if it >= args.warmup:
                    times[name][0].append(e0.elapsed_time(e1)); times[name][1].append(e1.elapsed_time(e2))
        row = {"case": label, "nf": nf, "N_per_frame": lv.N, "C": C, "K": K, "lambda": "mlp", "precision": "FP32_SIMT (autograd default)", "reps": args.reps}
        for name, (tf, tb) in times.items():
            row[name] = {"forward_ms_median": statistics.median(tf), "backward_ms_median": statistics.median(tb),
                         "forward_ms_min_max": [min(tf), max(tf)], "backward_ms_min_max": [min(tb), max(tb)]}
        rows.append(row)
        print(json.dumps(row), flush=True)
        del conv1, conv2, D, B, sc, lv
        torch.cuda.empty_cache()
    doc = {"script": "scripts/time_window_training_step.py", **card(), "rows": rows}
    print(json.dumps(doc, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
