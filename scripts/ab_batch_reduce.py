"""Bitwise A/B of the batch-indexed reduce launches against a comparison build of the library (GPU).

    python scripts/ab_batch_reduce.py --base /path/to/other/libbanet.so [--out result.json]

The build's and the keyframe build's reduce, and depth_compose's backward, take the pair or window index from blockIdx.y and stride by
gridDim.y past 65 535.  Up to 65 535 the launch shape and each element's summation order are unchanged, so the outputs must be bit for bit
those of the comparison library: H, g, rbar_sum, nvalid of lm_build (FP32_SIMT and TF32X3, K = 128, C = 64, one 40-point tile per pair)
and of lm_keyframe_build (nf = 1, K = 64, C = 32), and depth_compose_bwd's dbasis, at nb in {1, 2000, 65535}.  Both libraries are loaded
into one process (scripts/ab_simt_outputs.py's Libs).
"""
import argparse, json, os, sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="libbanet.so to compare against")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from ab_simt_outputs import Libs, gpu_identity, torch_equal
    from banet_b200 import ops, _lib
    import test_batch_edges as TB
    import test_build_edges as BE
    libs = Libs({"base": os.path.abspath(a.base), "new": os.path.abspath(os.path.join(ROOT, "banet_b200", "libbanet.so"))})
    rows, bad = [], []

    def compare(case, fn):
        x, y = libs.run("base", fn), libs.run("new", fn)
        torch.cuda.synchronize()
        same = all(torch_equal(p, q) for p, q in zip(x, y))
        rows.append((case, same))
        print(f"{case:40s} {'bitwise equal' if same else 'DIFFERS'}", flush=True)
        if not same:
            bad.append(case)

    for nb in (1, 2000, 65535):
        c = TB._case(nb, 40, 64, 128, 5, 7, seed=nb, weighted=True)
        lv = BE._level(c)
        for prec in (_lib.PREC_FP32_SIMT, _lib.PREC_TF32X3):
            compare(f"lm_build nb={nb} {BE.MODE_NAME[prec]}", lambda: ops.lm_build(lv, c.R, c.T, c.W, prec))
        del c, lv
        k, _ = TB._keyframe_case(nb, 1, 40, 32, 64, seed=nb + 1)
        key = ops.KeyframeLevel(k.conv1, k.conv2, k.intr, k.p, k.D, k.B, weight=k.weight)
        compare(f"lm_keyframe_build nw={nb} nf=1", lambda: ops.lm_keyframe_build(key, k.R, k.T, k.W))
        del k, key
        gen = torch.Generator(device="cuda").manual_seed(nb)
        basis = torch.randn(nb, 40, 16, generator=gen, device="cuda")
        W = torch.randn(nb, 16, 1, generator=gen, device="cuda")
        dout = torch.randn(nb, 40, generator=gen, device="cuda")
        compare(f"depth_compose_bwd nb={nb} dbasis", lambda: ops.depth_compose_bwd(dout, basis, W)[:1])
        torch.cuda.empty_cache()
    report = {"gpu": gpu_identity(), "cases": rows, "mismatches": bad}
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)
    if bad:
        sys.exit("ab_batch_reduce: outputs differ between the two libraries")


if __name__ == "__main__":
    main()
