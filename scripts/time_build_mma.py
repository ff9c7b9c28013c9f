"""lm_build at the four cfg2 bench levels against a comparison build of the library: timing and bitwise outputs (GPU).

    python scripts/time_build_mma.py --base /path/to/other/libbanet.so [--rounds 4] [--reps 6] [--out profiles/h100_build_mma.json]

The scene is bench.py's cfg2 scene (nb=32, C=K=128, [F2|gx|gy] layout, raster grids, seed 1234+2).  Each level is built in the mode
PREC_AUTO picks there (TF32X3 below 65 536 points per pair, TF32X1 above), and 640x480 once more in TF32X2.  Worker processes load
one library each (BANET_LIB_PATH) and run alternately, `--rounds` times per library; every worker times `--reps` launches per case
after three warm-up launches (CUDA events).  The report gives median [min - max] per case and library, and whether H, g, rbar and
nvalid of the two libraries are bitwise equal.
"""
import argparse, hashlib, json, os, statistics, subprocess, sys, tempfile

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
CASES = [("80x60", 0, "auto"), ("160x120", 1, "auto"), ("320x240", 2, "auto"), ("640x480", 3, "auto"), ("640x480", 3, "tf32x2")]


def worker(out_path, reps):
    sys.path.insert(0, ROOT)
    import torch
    from banet_b200 import ops, synth, _lib
    prec = {"auto": _lib.PREC_AUTO, "tf32x2": _lib.PREC_TF32X2}
    dev = torch.device("cuda")
    sc = synth.make_scene(nb=32, H=480, W=640, C=128, K=128, level_ids=(0, 1, 2, 3), seed=1234 + 2, device=dev, dtype=torch.float32)
    levels = [ops.Level(l.conv1, l.conv2, l.intr, l.p, l.D, l.B, grid=l.grid) for l in sc.levels]
    res = {}
    for name, li, mode in CASES:
        fn = lambda: ops.lm_build(levels[li], sc.R0, sc.T0, sc.W0, precision=prec[mode])
        for _ in range(3):
            out = fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(reps):
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record(); torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        digest = {k: hashlib.sha256(v.contiguous().cpu().numpy().tobytes()).hexdigest() for k, v in zip(("H", "g", "rbar", "nvalid"), out)}
        res[f"{name} {mode}"] = {"ms": ms, "sha256": digest}
    with open(out_path, "w") as f:
        json.dump(res, f)


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"name": q[0], "power_limit_w": float(q[1])}
    except Exception as e:                       # the identity is informative only
        return {"name": None, "power_limit_w": None, "note": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="libbanet.so to compare against")
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_build_mma.json"))
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a.worker, a.reps)
    libs = {"base": os.path.abspath(a.base), "new": os.path.abspath(os.path.join(ROOT, "banet_b200", "libbanet.so"))}
    runs = {k: [] for k in libs}
    with tempfile.TemporaryDirectory() as td:
        for r in range(a.rounds):
            for k, path in libs.items():
                p = os.path.join(td, f"{k}{r}.json")
                subprocess.run([sys.executable, os.path.abspath(__file__), "--base", a.base, "--reps", str(a.reps), "--worker", p],
                               env=dict(os.environ, BANET_LIB_PATH=path), check=True)
                with open(p) as f:
                    runs[k].append(json.load(f))
    report = {"gpu": gpu_identity(), "libs": {"base": "comparison build (--base)", "new": "banet_b200/libbanet.so"},
              "rounds": a.rounds, "reps_per_round": a.reps, "cases": {}}
    all_equal = True
    for name, _, mode in CASES:
        key = f"{name} {mode}"
        row = {}
        for k in libs:
            ms = sorted(x for run in runs[k] for x in run[key]["ms"])
            row[k] = {"median_ms": statistics.median(ms), "min_ms": ms[0], "max_ms": ms[-1], "n": len(ms)}
        digests = {k: {json.dumps(run[key]["sha256"], sort_keys=True) for run in runs[k]} for k in libs}
        row["deterministic"] = all(len(v) == 1 for v in digests.values())
        row["bitwise_equal"] = row["deterministic"] and digests["base"] == digests["new"]
        row["speedup"] = row["base"]["median_ms"] / row["new"]["median_ms"]
        all_equal &= row["bitwise_equal"]
        report["cases"][key] = row
        print(f"{key:18s} base {row['base']['median_ms']:8.3f} [{row['base']['min_ms']:.3f}-{row['base']['max_ms']:.3f}] ms   "
              f"new {row['new']['median_ms']:8.3f} [{row['new']['min_ms']:.3f}-{row['new']['max_ms']:.3f}] ms   x{row['speedup']:.2f}   "
              f"bitwise_equal={row['bitwise_equal']}", flush=True)
    report["all_bitwise_equal"] = all_equal
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(report, f, indent=1)
    if not all_equal:
        sys.exit("time_build_mma: outputs differ between the two libraries")


if __name__ == "__main__":
    main()
