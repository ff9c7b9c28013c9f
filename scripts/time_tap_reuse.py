"""lm_build per cfg2 level and whole lm_run solves against a comparison build of the library: timing and bitwise outputs (GPU).

    python scripts/time_tap_reuse.py --base /path/to/other/libbanet.so [--variant name=/path/to/libbanet.so ...]
                                     [--rounds 4] [--reps 8] [--solves 3] [--out profiles/h100_tap_reuse.json]

The scene is bench.py's cfg2 scene (nb = 32, C = K = 128, [F2|gx|gy] layout, dense raster grids at 80x60 .. 640x480, seed 1234 + 2, the
default motion), built at the precision bench.py times (PREC_AUTO: TF32X3 below 65 536 points per pair, TF32X1 above).  One process builds
the scene once and loads every library (each one its own handle); the libraries take turns, `--rounds` times each.  A turn times `--reps`
lm_build launches per level after three warm-up launches, and `--solves` whole lm_run solves (4 levels x 5 iterations, bench.py's
lambda-MLP, after one warm-up solve), with CUDA events.  The report gives the card and its power limit, median [min - max] per case and
library, and whether H, g, rbar, nvalid of every level and R, T, W of the solve are bitwise equal between base and new (and across the
rounds of each).  `--variant` adds more libraries (e.g. an ablation) to the rotation; they are timed, not compared.
"""
import argparse, hashlib, json, os, statistics, subprocess, sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
LEVELS = ("80x60", "160x120", "320x240", "640x480")


def use_library(path):
    from banet_b200 import _lib
    _lib.LIB_PATH, _lib._lib = path, None
    _lib.load()


def measure(levels, sc, packed, ws, reps, solves):
    import torch
    from banet_b200 import ops, _lib
    digest = lambda ts: {k: hashlib.sha256(v.contiguous().cpu().numpy().tobytes()).hexdigest() for k, v in ts.items()}

    def timed(fn, n):
        ms = []
        for _ in range(n):
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record(); out = fn(); e1.record(); torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        return ms, out

    res = {}
    for name, lv in zip(LEVELS, levels):
        fn = lambda: ops.lm_build(lv, sc.R0, sc.T0, sc.W0, precision=_lib.PREC_AUTO)
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ms, out = timed(fn, reps)
        res[f"lm_build {name}"] = {"ms": ms, "sha256": digest(dict(zip(("H", "g", "rbar", "nvalid"), out)))}
    fn = lambda: ops.lm_run(levels, 5, sc.R0, sc.T0, sc.W0, mlp_packed=packed, l2_regularizer_base=1000.0, workspace=ws, precision=_lib.PREC_AUTO)
    fn()
    torch.cuda.synchronize()
    ms, (R, T, W, status) = timed(fn, solves)
    assert int(status.abs().max()) == 0
    res["lm_run cfg2 solve"] = {"ms": ms, "sha256": digest({"R": R, "T": T, "W": W})}
    return res


def gpu_identity():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"name": q[0], "power_limit_w": float(q[1]), "max_sm_clock_mhz": float(q[2])}
    except Exception as e:                       # the identity is informative only
        return {"name": None, "power_limit_w": None, "note": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="libbanet.so to compare against")
    ap.add_argument("--variant", action="append", default=[], help="name=path: another library to time in the same rotation")
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--reps", type=int, default=8)
    ap.add_argument("--solves", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_tap_reuse.json"))
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import torch
    from banet_b200 import ops, synth, _lib
    libs = {"base": os.path.abspath(a.base), "new": os.path.abspath(os.path.join(ROOT, "banet_b200", "libbanet.so"))}
    for v in a.variant:
        k, p = v.split("=", 1)
        libs[k] = os.path.abspath(p)
    dev = torch.device("cuda")
    sc = synth.make_scene(nb=32, H=480, W=640, C=128, K=128, level_ids=(0, 1, 2, 3), seed=1234 + 2, device=dev, dtype=torch.float32)
    levels = [ops.Level(l.conv1, l.conv2, l.intr, l.p, l.D, l.B, grid=l.grid) for l in sc.levels]
    g = torch.Generator().manual_seed(7)                          # bench.py's he-normal lambda-MLP
    dims = [128, 256, 512, 256, 128, 1]
    packed = []
    for _ in levels:
        params = [(torch.randn(dims[i], dims[i + 1], generator=g) * (2.0 / dims[i]) ** 0.5, torch.zeros(dims[i + 1])) for i in range(5)]
        packed.append(ops.pack_mlp(params).to(dev))
    print("scene built; libraries:", libs, flush=True)
    runs = {k: [] for k in libs}
    for r in range(a.rounds):
        for k, path in libs.items():
            use_library(path)
            ws = torch.empty(ops.lm_run_workspace_bytes(levels, _lib.PREC_AUTO), dtype=torch.uint8, device=dev)
            runs[k].append(measure(levels, sc, packed, ws, a.reps, a.solves))
            del ws
            print(f"round {r} {k}: " + "  ".join(f"{c} {statistics.median(v['ms']):.3f}" for c, v in runs[k][-1].items()), flush=True)
    report = {"gpu": gpu_identity(), "libs": {k: ("banet_b200/libbanet.so" if k == "new" else os.path.basename(os.path.dirname(v)) + "/libbanet.so")
                                              for k, v in libs.items()},
              "scene": "bench.py cfg2: nb=32, C=K=128, [F2|gx|gy], PREC_AUTO, seed 1236", "rounds": a.rounds, "reps_per_round": a.reps,
              "solves_per_round": a.solves, "cases": {}}
    all_equal = True
    for key in [f"lm_build {n}" for n in LEVELS] + ["lm_run cfg2 solve"]:
        row = {}
        for k in libs:
            ms = sorted(x for run in runs[k] for x in run[key]["ms"])
            row[k] = {"median_ms": statistics.median(ms), "min_ms": ms[0], "max_ms": ms[-1], "n": len(ms)}
        digests = {k: {json.dumps(run[key]["sha256"], sort_keys=True) for run in runs[k]} for k in libs}
        row["deterministic"] = all(len(digests[k]) == 1 for k in ("base", "new"))
        row["bitwise_equal"] = row["deterministic"] and digests["base"] == digests["new"]
        for k in libs:
            if k != "base":
                row[f"speedup_{k}"] = row["base"]["median_ms"] / row[k]["median_ms"]
        all_equal &= row["bitwise_equal"]
        report["cases"][key] = row
        print(f"{key:20s} " + "   ".join(f"{k} {row[k]['median_ms']:8.3f} [{row[k]['min_ms']:.3f}-{row[k]['max_ms']:.3f}]" for k in libs)
              + f"   x{row['speedup_new']:.3f}   bitwise_equal={row['bitwise_equal']}", flush=True)
    report["all_bitwise_equal"] = all_equal
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(report, f, indent=1)
    if not all_equal:
        sys.exit("time_tap_reuse: outputs differ between the two libraries")


if __name__ == "__main__":
    main()
