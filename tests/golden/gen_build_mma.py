"""Writes tests/golden/build_mma.json: SHA-256 digests of the tensor-core lm_build outputs (H, g, rbar, nvalid) on a seeded scene, in
every precision mode, both conv2 layouts and K = 128 / 64 / 32 (GPU).  tests/test_gpu_build_mma.py holds
the library to them bit for bit.  Run on an H100 with the library whose results are to be frozen:

    python tests/golden/gen_build_mma.py [OUT.json]          (BANET_LIB_PATH selects another build of the library)

The outputs depend on the partition of the tiles over the CTAs, i.e. on the SM count: the fixture records it, and the test skips
on a device with a different count.
"""
import hashlib
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# (K, layout, precision mode); K = 64 / 32 take modes 2 and 3
CASES = [(128, lay, m) for lay in ("3c", "f2") for m in (1, 2, 3)] + [(k, "3c", m) for k in (64, 32) for m in (2, 3)]


def case_id(K, lay, mode):
    return f"gen6_K{K}_{lay}_x{mode}"       # gen6: the tensor-core kernel, lm_build_tc6_kernel


def outputs():
    """{case id: {tensor name: sha256 hex}} of the library that banet_b200 loads, plus the device identity."""
    from banet_b200 import ops, synth
    dev = torch.device("cuda")
    res = {}
    scenes = {}
    for K, lay, mode in CASES:
        if K not in scenes:      # 320x240, 2 pairs: 1 200 tiles per pair, spans of several pairs per CTA and pair changes inside a CTA
            scenes[K] = synth.make_scene(nb=2, H=240, W=320, C=128, K=K, level_ids=(3,), seed=4100 + K, device=dev, dtype=torch.float32)
        sc = scenes[K]
        lv = sc.levels[0]
        conv2 = lv.conv2 if lay == "3c" else lv.conv2[..., :128].contiguous()
        L = ops.Level(lv.conv1, conv2, lv.intr, lv.p, lv.D, lv.B, grid=lv.grid)
        W = sc.W0 + 0.01 * torch.randn(sc.W0.shape, generator=torch.Generator().manual_seed(3)).to(dev)
        out = ops.lm_build(L, sc.R0, sc.T0, W, precision=mode)
        torch.cuda.synchronize()
        res[case_id(K, lay, mode)] = {k: hashlib.sha256(v.contiguous().cpu().numpy().tobytes()).hexdigest()
                                      for k, v in zip(("H", "g", "rbar", "nvalid"), out)}
    p = torch.cuda.get_device_properties(0)
    return {"device": p.name, "sm_count": p.multi_processor_count, "cases": res}


if __name__ == "__main__":
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "build_mma.json")
    with open(out, "w") as f:
        json.dump(outputs(), f, indent=1, sort_keys=True)
    print("wrote", out)
