"""Bitwise A/B of every build path on non-robust levels against a comparison build of the library that predates banet_level_t::robust (GPU).

    python scripts/ab_robust_outputs.py --base /path/to/other/libbanet.so [--out result.json]

One process loads both libraries (two ctypes handles).  The comparison library's level struct lacks the trailing robust and robust_scale
fields, so its calls take a struct of its own layout (the leading fields, copied) and level arrays of its stride.  Forward outputs and the
single-writer gradients (dconv1, dD, dB, dweight) must be bitwise equal; an atomic gradient (dconv2, dR, dT, dW) may differ from the
nearest of twelve base runs by no more than two base runs differ from each other (scripts/ab_simt_outputs.py).  Cases, on a dense 64 x 48
grid (nb = 2) and 4096 sampled points (nb = 4):
  lm_build in FP32_SIMT, TF32X1, TF32X2, TF32X3 and AUTO (the TF32 modes where they apply): K in {0, 16, 32, 64, 128}, C in {64, 128},
    fp32 / bf16 features and basis, [F2|gx|gy] and F2-only maps, with and without point weights;
  lm_build_bwd with dweight (exact_sym 0 and 1) on the same levels;
  lm_run, 2 levels x 2 iterations, at FP32_SIMT and AUTO.
"""
import argparse, ctypes as C, json, os, sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ab_simt_outputs import compare          # noqa: E402


class Libs:
    """Both libraries in one process; calls on 'base' see a level struct without the robust fields."""
    def __init__(self, base_path):
        from banet_b200 import _lib, ops
        self._lib, self._ops = _lib, ops
        fields = [f for f in _lib.BanetLevel._fields_ if f[0] not in ("robust", "robust_scale")]

        class ParentLevel(C.Structure):
            _fields_ = fields

            def __init__(self, *args):
                super().__init__(*args[:len(fields)])

        self.Parent = ParentLevel
        self.handles = {"new": _lib.load()}
        _lib._lib, _lib.LIB_PATH = None, base_path
        base = _lib.load()
        for name, (_, args) in _lib.SIGNATURES.items():
            fn = getattr(base, name)
            fn.argtypes = [C.POINTER(ParentLevel) if a is C.POINTER(_lib.BanetLevel) else a for a in args]
        self.handles["base"] = base
        _lib._lib = self.handles["new"]

    def run(self, name, fn):
        self._lib._lib = self.handles[name]
        self._ops.BanetLevel = self.Parent if name == "base" else self._lib.BanetLevel
        try:
            return fn()
        finally:
            self._lib._lib = self.handles["new"]
            self._ops.BanetLevel = self._lib.BanetLevel


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from banet_b200 import ops, synth, _lib
    libs = Libs(os.path.abspath(a.base))
    P = {"simt": _lib.PREC_FP32_SIMT, "x1": _lib.PREC_TF32X1, "x2": _lib.PREC_TF32X2, "x3": _lib.PREC_TF32X3, "auto": _lib.PREC_AUTO}
    FWD, BWD, RUN = ("H", "g", "rbar", "nvalid"), ("dconv1", "dconv2", "dD", "dB", "dR", "dT", "dW", "dweight"), ("R", "T", "W", "status")
    bad, counts, ncase = [], [0, 0], 0
    for shape, (nb, npts) in (("dense", (2, None)), ("sparse", (4, 4096))):
        for C_ in (64, 128):
            for K in (0, 16, 32, 64, 128):
                sc = synth.make_scene(nb=nb, H=48, W=64, C=C_, K=K, level_ids=(2, 3), seed=5 + K + C_, device="cuda", dtype=torch.float32,
                                      n_points=npts)
                l = sc.levels[1]
                Wt = None if K == 0 else sc.W0 + 0.01
                wt = (0.5 + torch.rand(nb, l.N, 1, generator=torch.Generator().manual_seed(K))).cuda()
                P_ = 6 + K
                gen = torch.Generator(device="cuda").manual_seed(K + C_)
                dH, dg, dr = (torch.randn(nb, P_, P_, generator=gen, device="cuda"), torch.randn(nb, P_, generator=gen, device="cuda"),
                              torch.randn(nb, C_, generator=gen, device="cuda"))
                precs = ("simt", "x1", "x2", "x3", "auto") if K in (32, 64, 128) else ("simt", "auto")
                for layout in ("3c", "f2"):
                    for feat in ("f32", "bf16"):
                        for basis in (("f32", "bf16") if K else ("f32",)):
                            c1 = l.conv1 if feat == "f32" else l.conv1.bfloat16()
                            c2 = l.conv2 if layout == "3c" else l.conv2[..., :C_].contiguous()
                            c2 = c2 if feat == "f32" else c2.bfloat16()
                            B = l.B if (K == 0 or basis == "f32") else l.B.bfloat16()
                            for wname, w in (("unweighted", None), ("weighted", wt)):
                                lv = ops.Level(c1, c2, l.intr, l.p, l.D, B, grid=l.grid, weight=w)
                                tag = f"{shape} C{C_} K{K} {layout} {feat}/{basis} {wname}"
                                for pn in precs:
                                    ncase += 1
                                    compare(libs, f"lm_build {pn} {tag}", FWD, lambda: ops.lm_build(lv, sc.R0, sc.T0, Wt, P[pn]), bad, counts, base_runs=12)
                                for ex in (0, 1):
                                    ncase += 1
                                    compare(libs, f"lm_build_bwd exact={ex} {tag}", BWD,
                                            lambda: ops.lm_build_bwd(lv, sc.R0, sc.T0, Wt, dH, dg, dr, ex, return_dweight=True), bad, counts, base_runs=12)
                print("checked", shape, C_, K, len(bad), flush=True)
                if K in (0, 16, 128):
                    lvs = [ops.Level(x.conv1, x.conv2, x.intr, x.p, x.D, x.B, grid=x.grid) for x in sc.levels]
                    for pn in ("simt", "auto"):
                        ncase += 1
                        compare(libs, f"lm_run {pn} {shape} C{C_} K{K}", RUN,
                                lambda: ops.lm_run(lvs, 2, sc.R0, sc.T0, sc.W0, lambda_fixed=0.1, precision=P[pn]), bad, counts, base_runs=12)
    rep = {"cases": ncase, "outputs_compared": counts[0], "atomic_outputs_within_base_spread": counts[1], "mismatches": bad}
    print(json.dumps(rep, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rep, f, indent=1)
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
