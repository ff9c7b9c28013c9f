"""Error A/B of the four whole-solve entries (banet_lm_run, banet_lm_window_run, banet_lm_window_batch_run, banet_lm_keyframe_run) and
their workspace queries against a comparison build of the library.  CPU only: every call carries at least one fault that the library
reports before any CUDA call (the workspace is always 16 bytes).

    python scripts/ab_run_errors.py --base /path/to/other/libbanet.so

One process loads both libraries (two ctypes handles, as scripts/ab_solve_outputs.py).  Each fault of the table below alone and every
pair of them, on each of the four forms: the run's return code and banet_last_error(), then the query's size and banet_last_error(),
must be equal.  A robust-loss message that names a different *_workspace_bytes query is reported apart.  Then the four queries' sizes
over a grid of valid configurations.  The pair queries do not check level shapes, so no fault sets N = 0 (their build plan divides by it).
"""
import argparse, ctypes as C, itertools, os, sys
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from banet_b200 import _lib

ap = argparse.ArgumentParser()
ap.add_argument("--base", required=True, help="libbanet.so to compare against")
args = ap.parse_args()
libs = {}
for k, p in {"old": os.path.abspath(args.base), "new": os.path.join(ROOT, "banet_b200", "libbanet.so")}.items():
    _lib._lib, _lib.LIB_PATH = None, p
    libs[k] = _lib.load()

P = 1 << 20


def plevel(nb=4, N=4096, Cc=64, K=32, h=48, w=64, c2=None, robust=0, scale=0.0):
    return _lib.BanetLevel(nb, N, Cc, K, h, w, 3 * Cc if c2 is None else c2, P, P, P, P, P, P, 0, 0, 0, 0, None, robust, scale)


def klevel(nw=2, nf=2, N=1024, Cc=32, K=32, h=48, w=64, c2=None):
    return _lib.BanetKeyframeLevel(nw, nf, N, Cc, K, h, w, 3 * Cc if c2 is None else c2, P, P, P, P, P, P, None)


# the arguments of one run and its query; each fault edits them
def base(form):
    lv = [klevel(), klevel(N=256, h=24, w=32)] if form == "key" else [plevel(), plevel(N=1024, h=24, w=32, Cc=32)]
    return dict(form=form, levels=lv, nlevels=None, iters=2, mlp="none", lf=0.5, scramble=0, prec=0, R=P, T=P, W=P, status=P, opts=True,
                ws=P, ws_bytes=16, nw=2)


def lvset(attr, val, which=-1):
    """A fault on a level field; on a form whose level struct has no such field the fault does not apply and the call is skipped."""
    def f(a):
        for i, lv in enumerate(a["levels"]):
            if attr not in (name for name, _ in type(lv)._fields_):
                a["skip"] = True
            elif which < 0 or i == which:
                setattr(lv, attr, val)
    return f


def argset(**kw):
    return lambda a: a.update(kw)


FAULTS = {
    "R0": argset(R=None), "T0": argset(T=None), "W0": argset(W=None), "status0": argset(status=None), "opts0": argset(opts=False),
    "ws0": argset(ws=None), "nlev0": argset(nlevels=0), "iters0": argset(iters=0), "nw0": argset(nw=0), "nw3": argset(nw=3),
    "nbdis": lvset("nb", 6, 1), "Kdis": lvset("K", 16, 1), "nwdis": lvset("nw", 3, 1), "nfdis": lvset("nf", 3, 1),
    "nomlp": argset(lf=-1.0), "halfmlp": argset(mlp="half", lf=-1.0), "K0": lvset("K", 0), "scramble": argset(scramble=1),
    "robust_kind": lvset("robust", 3), "robust_scale": lambda a: (lvset("robust", 1)(a), lvset("robust_scale", -1.0)(a)),
    "prec9": argset(prec=9), "precm2": argset(prec=-2), "prec1": argset(prec=1), "prec3": argset(prec=3), "prec4": argset(prec=4),
    "K257": lvset("K", 257), "C4096": lvset("C", 4096), "C2048": lvset("C", 2048), "bigC_mlp": lambda a: (lvset("C", 1024)(a), a.update(mlp="all", lf=-1.0)),
    "badshape": lvset("conv2_channels", 100, 0), "nullconv": lvset("conv1", None, 1), "mlp_ok": argset(mlp="all", lf=-1.0),
    "K200": lvset("K", 200), "nb0": lvset("nb", 0),
}


def call(lib, a):
    form, lvs = a["form"], a["levels"]
    T = _lib.BanetKeyframeLevel if form == "key" else _lib.BanetLevel
    arr = (T * len(lvs))(*lvs)
    n = len(lvs) if a["nlevels"] is None else a["nlevels"]
    mlp = None
    if a["mlp"] != "none":
        mlp = (C.c_void_p * len(lvs))(*[P if (a["mlp"] == "all" or i == 0) else None for i in range(len(lvs))])
    opts = _lib.BanetSolveOpts(1e-5, 1, a["scramble"])
    op = C.byref(opts) if a["opts"] else None
    tail = (a["R"], a["T"], a["W"], a["status"], a["ws"], a["ws_bytes"], None)
    if form == "pair":
        rc = lib.banet_lm_run(arr, n, a["iters"], mlp, 1000.0, a["lf"], op, a["prec"], *tail)
        e1 = lib.banet_last_error()
        q = lib.banet_lm_run_workspace_bytes(arr, n, a["prec"])
    elif form == "win":
        rc = lib.banet_lm_window_run(arr, n, a["iters"], mlp, 1000.0, a["lf"], op, a["prec"], *tail)
        e1 = lib.banet_last_error()
        q = lib.banet_lm_window_run_workspace_bytes(arr, n, a["prec"])
    elif form == "batch":
        rc = lib.banet_lm_window_batch_run(arr, n, a["nw"], a["iters"], mlp, 1000.0, a["lf"], op, a["prec"], *tail)
        e1 = lib.banet_last_error()
        q = lib.banet_lm_window_batch_run_workspace_bytes(arr, n, a["nw"], a["prec"])
    else:
        rc = lib.banet_lm_keyframe_run(arr, n, a["iters"], mlp, 1000.0, a["lf"], op, a["prec"], *tail)
        e1 = lib.banet_last_error()
        q = lib.banet_lm_keyframe_run_workspace_bytes(arr, n, a["prec"])
    return rc, e1, q, lib.banet_last_error()


def make(form, faults):
    a = base(form)
    for f in faults:
        FAULTS[f](a)
    return a


names = sorted(FAULTS)
n = bad = 0
diffs = []
for form in ("pair", "win", "batch", "key"):
    for combo in [(f,) for f in names] + list(itertools.combinations(names, 2)):
        if make(form, combo).get("skip"):
            continue
        ro, rn = call(libs["old"], make(form, combo)), call(libs["new"], make(form, combo))
        n += 1
        if ro != rn:
            bad += 1
            diffs.append((form, combo, ro, rn))
print(f"error A/B: {n} calls, {bad} differ")
allowed = 0
for d in diffs:
    form, combo, ro, rn = d
    # a failing query's robust-loss message names the query that was called (before: lm_run_workspace_bytes for all three pair queries)
    if ro[:3] == rn[:3] and ro[3].startswith(b"lm_run_workspace_bytes: robust") and rn[3].split(b":")[0].endswith(b"_workspace_bytes"):
        allowed += 1
        continue
    print("DIFF", form, combo, "\n   old", ro, "\n   new", rn)
print(f"  of which the allowed robust-query naming: {allowed}")

# workspace sizes over a grid of valid configurations
grid_n = 0
gbad = 0
for nb in (1, 2, 4, 6, 33, 100, 1000):
    for Cc in (8, 16, 32, 64, 128, 512):
        for K in (0, 1, 16, 32, 64, 128, 200, 256):
            for prec in (-1, 0, 1, 2, 3, 4):
                for nl in (1, 2, 3):
                    lvs = [plevel(nb=nb, Cc=max(Cc >> i, 1), K=K, N=4096 >> (2 * i), h=48 >> i, w=64 >> i) for i in range(nl)]
                    arr = (_lib.BanetLevel * nl)(*lvs)
                    for nw in (1, 2, 3):
                        r = [(lib.banet_lm_run_workspace_bytes(arr, nl, prec), lib.banet_lm_window_run_workspace_bytes(arr, nl, prec),
                              lib.banet_lm_window_batch_run_workspace_bytes(arr, nl, nw, prec)) for lib in (libs["old"], libs["new"])]
                        grid_n += 1
                        if r[0] != r[1]:
                            gbad += 1
                            print("SIZE DIFF", nb, Cc, K, prec, nl, nw, r)
for nw in (1, 2, 5, 64):
    for nf in (1, 2, 3, 16, 40):
        for Cc in (8, 32, 128, 2048):
            for K in (1, 16, 128, 255, 256):
                for prec in (-1, 0, 1):
                    for nl in (1, 2):
                        lvs = [klevel(nw=nw, nf=nf, Cc=Cc, K=K, N=4096 >> (2 * i), h=48 >> i, w=64 >> i) for i in range(nl)]
                        arr = (_lib.BanetKeyframeLevel * nl)(*lvs)
                        r = [lib.banet_lm_keyframe_run_workspace_bytes(arr, nl, prec) for lib in (libs["old"], libs["new"])]
                        grid_n += 1
                        if r[0] != r[1]:
                            gbad += 1
                            print("KEY SIZE DIFF", nw, nf, Cc, K, prec, nl, r)
print(f"workspace grid: {grid_n} configurations, {gbad} differ")
sys.exit(1 if gbad or bad > allowed else 0)
