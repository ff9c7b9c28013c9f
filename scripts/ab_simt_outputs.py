"""Bitwise A/B of the fp32 SIMT build kernels against a comparison build of the library (GPU), and interleaved timings of them.

    python scripts/ab_simt_outputs.py --base /path/to/other/libbanet.so [--rounds 3] [--out result.json]

Outputs: one worker process loads both libraries (two ctypes handles) and runs every seeded case on each.  Forward outputs and the
single-writer gradients (dconv1, dD, dB, dweight) must be bitwise equal.  An atomic output (dconv2, dR, dT, dW: fp32 atomics in a
run-dependent order) may differ from the nearest of five base runs by no more (max abs) than two base runs differ from each other.  Cases:
  lm_build at PREC_FP32_SIMT and lm_build_bwd (both exact_sym, with dweight): K in {0, 16, 32, 64, 128, 200}, C in {64, 128, 30} (30: the
    VEC = 1 path), fp32 / bf16 features and basis, [F2|gx|gy] and F2-only maps, with and without point weights, on 4096 sampled points
    (nb = 4), a dense 160 x 120 grid (nb = 2) and 2000 pairs x 40 points;
  lm_keyframe_build: (nw, nf) in {(2,1), (4,4), (2,16)}, K in {16, 32, 64, 128, 256}, both maps, with and without weights; its backward
    (K <= 128) on the [F2|gx|gy] map, including nf = 64 frames at C = K = 128 (more frames than one shared-memory chunk holds);
  lm_run and lm_keyframe_run at FP32_SIMT.
Timing (--rounds): worker processes load one library each (BANET_LIB_PATH) and alternate; each times, with CUDA events after three warm-up
calls, lm_build FP32_SIMT at the bench's cfg2 levels, lm_build_bwd on cfg2's 160 x 120 and 320 x 240 levels (both maps), lm_build and
lm_build_bwd at K in {0, 16, 32, 64} on 32 pairs x 4096 points (the two-CTA variants), and the keyframe build and backward at
nw x nf = 32 x 4 (K = 16, 32, 64, 128) and 8 x 16 (4096 points) and 4 x 4 (dense 320 x 240), C = 128.  The report gives median [min - max]
per case and library, and the card's name and power limit.
"""
import argparse, json, os, statistics, subprocess, sys, tempfile

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
ATOMIC = {"dconv2", "dR", "dT", "dW"}


class Libs:
    """Both libraries loaded into one process (two ctypes handles), switched per call, so outputs can be compared element by element."""
    def __init__(self, paths):
        from banet_b200 import _lib
        self._mod, self.handles = _lib, {}
        for name, path in paths.items():
            _lib._lib, _lib.LIB_PATH = None, path
            self.handles[name] = _lib.load()

    def run(self, name, fn):
        self._mod._lib = self.handles[name]
        out = fn()
        return out


def maxdiff(a, b):
    return float((a.double() - b.double()).abs().nan_to_num(float("inf")).max()) if a.numel() else 0.0


def compare(libs, case, names, fn, bad, counts, base_runs=5):
    """Bitwise for every output not in ATOMIC.  An atomic output passes when its distance (max abs) to the nearest of base_runs base runs is at
    most the largest distance between two base runs: the new output differs from the base's outputs by no more than those differ from each
    other."""
    b1, n = libs.run("base", fn), libs.run("new", fn)
    bases = None
    for i, (name, x, y) in enumerate(zip(names, b1, n)):
        if x is None:
            continue
        counts[0] += 1
        if torch_equal(x, y):
            continue
        if name not in ATOMIC:
            bad.append(f"{case}: {name} differs by {maxdiff(y, x):.3g}")
            continue
        if bases is None:
            bases = [b1] + [libs.run("base", fn) for _ in range(base_runs - 1)]
        near = min(maxdiff(y, b[i]) for b in bases)
        spread = max(maxdiff(bases[p][i], bases[q][i]) for p in range(base_runs) for q in range(p))
        if near <= spread:
            counts[1] += 1
        else:
            bad.append(f"{case}: {name} is {near:.3g} from the nearest of {base_runs} base runs (base run to run at most {spread:.3g})")


def torch_equal(a, b):
    return a.shape == b.shape and bool(((a == b) | (a.isnan() & b.isnan())).all())


def correctness(libs, ops, synth, torch, prec):
    dev, bad, counts = torch.device("cuda"), [], [0, 0]
    FWD, BWD, RUN = ("H", "g", "rbar", "nvalid"), ("dconv1", "dconv2", "dD", "dB", "dR", "dT", "dW", "dweight"), ("R", "T", "W", "status")
    ncase = 0
    for shape, (nb, lv, npts) in (("sparse", (4, 1, 4096)), ("dense", (2, 2, None)), ("pairs", (2000, 0, 40))):
        for C in (64, 128, 30):
            print("check", shape, C, flush=True)
            sc = synth.make_scene(nb=nb, H=240, W=320, C=C, K=200, level_ids=(lv,), seed=7 + C, device=dev, dtype=torch.float32, n_points=npts)
            l = sc.levels[0]
            wt = torch.rand(l.D.shape, device=dev, generator=torch.Generator(device=dev).manual_seed(3)) + 0.5
            for K in (0, 16, 32, 64, 128, 200):
                for fd in (torch.float32, torch.bfloat16):
                    for bd in ((torch.float32, torch.bfloat16) if K else (torch.float32,)):
                        for lay in ("3C", "F2"):
                            for weighted in (False, True):
                                c2 = l.conv2 if lay == "3C" else l.conv2[..., :C].contiguous()
                                B = None if K == 0 else l.B[..., :K].contiguous().to(bd)
                                W = None if K == 0 else sc.W0[:, :K].contiguous() + 0.01
                                lev = ops.Level(l.conv1.to(fd), c2.to(fd), l.intr, l.p, l.D, B, weight=wt if weighted else None)
                                case = f"{shape} C{C} K{K} {fd}/{bd} {lay} w{int(weighted)}"
                                compare(libs, "build " + case, FWD, lambda: ops.lm_build(lev, sc.R0, sc.T0, W, precision=prec), bad, counts)
                                P = 6 + K
                                gen = torch.Generator(device=dev).manual_seed(K + C)
                                dH = torch.randn(nb, P, P, device=dev, generator=gen) * 1e-3
                                dg = torch.randn(nb, P, device=dev, generator=gen) * 1e-3
                                dr = torch.randn(nb, C, device=dev, generator=gen) * 1e-3
                                for es in (False, True):
                                    compare(libs, f"bwd {case} es{int(es)}", BWD,
                                            lambda: ops.lm_build_bwd(lev, sc.R0, sc.T0, W, dH, dg, dr, exact_sym=es, return_dweight=True), bad, counts)
                                ncase += 3
            if shape == "sparse":
                lev = ops.Level(l.conv1, l.conv2, l.intr, l.p, l.D, l.B[..., :64].contiguous())
                compare(libs, f"run C{C}", RUN, lambda: ops.lm_run([lev], 3, sc.R0, sc.T0, sc.W0[:, :64].contiguous(), lambda_fixed=1.0, precision=prec),
                        bad, counts)
                ncase += 1
            del sc, l, lev
            torch.cuda.empty_cache()
    for nw, nf, Ks, C in ((2, 1, (16, 32, 64, 128, 256), 64), (4, 4, (16, 32, 64, 128, 256), 64), (2, 16, (16, 32, 64, 128, 256), 64), (1, 64, (128,), 128)):
        print("check keyframe", nw, nf, flush=True)
        sc = synth.make_scene(nb=nw * nf, H=240, W=320, C=C, K=256, level_ids=(1,), seed=11 + nf, device=dev, dtype=torch.float32,
                              n_points=4096, shared_depth=True, window_frames=nf)
        l = sc.levels[0]
        kf = lambda t: t.reshape(nw, nf, *t.shape[1:])[:, 0].contiguous()
        wt = torch.rand(l.D.shape, device=dev, generator=torch.Generator(device=dev).manual_seed(5)) + 0.5
        for K in Ks:
            W = sc.W0.reshape(nw, nf, 256, 1)[:, 0, :K].contiguous() + 0.01
            for lay in (("3C", "F2") if nf < 64 else ("3C",)):
                for weighted in (False, True):
                    c2 = l.conv2 if lay == "3C" else l.conv2[..., :C].contiguous()
                    key = ops.KeyframeLevel(kf(l.conv1), c2, l.intr, kf(l.p), kf(l.D), kf(l.B)[..., :K].contiguous(), weight=wt if weighted else None)
                    case = f"keyframe {nw}x{nf} C{C} K{K} {lay} w{int(weighted)}"
                    if nf < 64:
                        compare(libs, case, FWD, lambda: ops.lm_keyframe_build(key, sc.R0, sc.T0, W), bad, counts)
                        ncase += 1
                    if lay == "3C" and K <= 128:                      # the backward keeps S_dd in shared memory: K <= 128 at these C
                        P, nb = 6 + K, nw * nf
                        gen = torch.Generator(device=dev).manual_seed(K)
                        dH = torch.randn(nb, P, P, device=dev, generator=gen) * 1e-3
                        dg = torch.randn(nb, P, device=dev, generator=gen) * 1e-3
                        dr = torch.randn(nb, C, device=dev, generator=gen) * 1e-3
                        for es in (False, True):
                            compare(libs, f"bwd {case} es{int(es)}", BWD,
                                    lambda: ops.lm_keyframe_build_bwd(key, sc.R0, sc.T0, W, dH, dg, dr, exact_sym=es, return_dweight=True), bad, counts)
                            ncase += 1
        if nf == 4:
            key = ops.KeyframeLevel(kf(l.conv1), l.conv2, l.intr, kf(l.p), kf(l.D), kf(l.B)[..., :64].contiguous())
            W = sc.W0.reshape(nw, nf, 256, 1)[:, 0, :64].contiguous()
            compare(libs, f"keyframe run {nw}x{nf}", RUN, lambda: ops.lm_keyframe_run([key], 3, sc.R0, sc.T0, W, lambda_fixed=1.0, precision=prec),
                    bad, counts)
            ncase += 1
    return {"cases": ncase, "outputs": counts[0], "atomic_outputs_within_base_spread": counts[1], "mismatches": bad}


def timing(ops, synth, torch, prec, reps):
    dev, res = torch.device("cuda"), {}

    def timed(name, fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(reps):
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record(); torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        res[name] = ms
        print("timed", name, flush=True)

    sc = synth.make_scene(nb=32, H=480, W=640, C=128, K=128, level_ids=(0, 1, 2, 3), seed=1234 + 2, device=dev, dtype=torch.float32)
    for l in sc.levels:
        lev = ops.Level(l.conv1, l.conv2, l.intr, l.p, l.D, l.B, grid=l.grid)
        name = f"{l.conv2.shape[2]}x{l.conv2.shape[1]}"
        timed(f"build {name}", lambda: ops.lm_build(lev, sc.R0, sc.T0, sc.W0, precision=prec))
        if l.conv2.shape[2] in (160, 320):
            P, nb = 134, 32
            dH = torch.randn(nb, P, P, device=dev) * 1e-3; dg = torch.randn(nb, P, device=dev) * 1e-3; dr = torch.randn(nb, 128, device=dev) * 1e-3
            for lay in ("3C", "F2"):
                lv2 = lev if lay == "3C" else ops.Level(l.conv1, l.conv2[..., :128].contiguous(), l.intr, l.p, l.D, l.B, grid=l.grid)
                timed(f"bwd {name} {lay}", lambda: ops.lm_build_bwd(lv2, sc.R0, sc.T0, sc.W0, dH, dg, dr))
    s = synth.make_scene(nb=32, H=240, W=320, C=128, K=64, level_ids=(1,), seed=21, device=dev, dtype=torch.float32, n_points=4096)
    l = s.levels[0]
    for K in (0, 16, 32, 64):                       # the two-CTA variants, 4096 points per pair
        lev = ops.Level(l.conv1, l.conv2, l.intr, l.p, l.D, None if K == 0 else l.B[..., :K].contiguous())
        W = None if K == 0 else s.W0[:, :K].contiguous() + 0.01
        timed(f"build 4096pt K{K}", lambda: ops.lm_build(lev, s.R0, s.T0, W, precision=prec))
        P = 6 + K
        dH = torch.randn(32, P, P, device=dev) * 1e-3; dg = torch.randn(32, P, device=dev) * 1e-3; dr = torch.randn(32, 128, device=dev) * 1e-3
        timed(f"bwd 4096pt K{K}", lambda: ops.lm_build_bwd(lev, s.R0, s.T0, W, dH, dg, dr))
    for nw, nf, npts in ((32, 4, 4096), (4, 4, None), (8, 16, 4096)):
        s = synth.make_scene(nb=nw * nf, H=240, W=320, C=128, K=128, level_ids=(1 if npts else 3,), seed=22, device=dev, dtype=torch.float32,
                             n_points=npts, shared_depth=True, window_frames=nf)
        l = s.levels[0]
        kf = lambda t: t.reshape(nw, nf, *t.shape[1:])[:, 0].contiguous()
        key = ops.KeyframeLevel(kf(l.conv1), l.conv2, l.intr, kf(l.p), kf(l.D), kf(l.B))
        W = s.W0.reshape(nw, nf, 128, 1)[:, 0].contiguous() + 0.01
        P, nb = 134, nw * nf
        dH = torch.randn(nb, P, P, device=dev) * 1e-3; dg = torch.randn(nb, P, device=dev) * 1e-3; dr = torch.randn(nb, 128, device=dev) * 1e-3
        timed(f"keyframe build {nw}x{nf}", lambda: ops.lm_keyframe_build(key, s.R0, s.T0, W))
        timed(f"keyframe bwd {nw}x{nf}", lambda: ops.lm_keyframe_build_bwd(key, s.R0, s.T0, W, dH, dg, dr))
        if nw == 32:
            for K in (16, 32, 64):                  # the two-CTA forward variants and the smaller backward ones
                keyK = ops.KeyframeLevel(key.conv1, key.conv2, key.intr, key.p, key.D, key.B[..., :K].contiguous())
                WK = W[:, :K].contiguous()
                dHK = dH[:, :6 + K, :6 + K].contiguous(); dgK = dg[:, :6 + K].contiguous()
                timed(f"keyframe build {nw}x{nf} K{K}", lambda: ops.lm_keyframe_build(keyK, s.R0, s.T0, WK))
                timed(f"keyframe bwd {nw}x{nf} K{K}", lambda: ops.lm_keyframe_build_bwd(keyK, s.R0, s.T0, WK, dHK, dgK, dr))
    return res


def worker(path, mode, reps, libs):
    sys.path.insert(0, ROOT)
    import torch
    from banet_b200 import ops, synth, _lib
    if mode == "check":
        res = correctness(Libs(libs), ops, synth, torch, _lib.PREC_FP32_SIMT)
    else:
        res = timing(ops, synth, torch, _lib.PREC_FP32_SIMT, reps)
    with open(path, "w") as f:
        json.dump(res, f)


def gpu_identity():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
    return {"name": q[0], "power_limit_w": float(q[1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="libbanet.so to compare against")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", nargs=2, default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    libs = {"base": os.path.abspath(a.base), "new": os.path.abspath(os.path.join(ROOT, "banet_b200", "libbanet.so"))}
    if a.worker:
        return worker(a.worker[0], a.worker[1], a.reps, libs)

    def run(lib, mode, td, tag):
        p = os.path.join(td, f"{tag}.json")
        subprocess.run([sys.executable, os.path.abspath(__file__), "--base", a.base, "--reps", str(a.reps), "--worker", p, mode],
                       env=dict(os.environ, BANET_LIB_PATH=libs[lib]), check=True)
        with open(p) as f:
            return json.load(f)

    report = {"gpu": gpu_identity()}
    with tempfile.TemporaryDirectory() as td:
        report["check"] = chk = run("new", "check", td, "check")
        times = {k: [] for k in libs}
        for r in range(a.rounds):
            for k in libs:
                times[k].append(run(k, "time", td, f"t{k}{r}"))
    bad = chk["mismatches"]
    report["timing_ms"] = {}
    for case in times["base"][0] if a.rounds else []:
        row = {}
        for k in libs:
            ms = sorted(x for run_ in times[k] for x in run_[case])
            row[k] = {"median": statistics.median(ms), "min": ms[0], "max": ms[-1]}
        report["timing_ms"][case] = row
        print(f"{case:28s} base {row['base']['median']:8.3f} [{row['base']['min']:.3f}-{row['base']['max']:.3f}]   "
              f"new {row['new']['median']:8.3f} [{row['new']['min']:.3f}-{row['new']['max']:.3f}] ms", flush=True)
    print(f"{chk['cases']} cases, {chk['outputs']} outputs compared, {chk['atomic_outputs_within_base_spread']} atomic outputs within the "
          f"base's run-to-run spread, {len(bad)} mismatches", *bad[:20], sep="\n")
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)
    if bad:
        sys.exit("ab_simt_outputs: outputs differ between the two libraries")


if __name__ == "__main__":
    main()
