"""Writes ref_op_timing.json: wall times of the reference's OWN compiled op (EquationConstruction + Grad, utils.cu, built unmodified by
oracle/Makefile into oracle/_ref/) at the shapes of tests/test_gpu_reference_pin.py::test_reference_op_timed_beside_the_b200_kernels,
with the card name and power limit they were measured at.  Needs a GPU and oracle/_ref/libbanet_ref_eqc.so:
    python tests/golden/gen_ref_timing_golden.py [outdir]"""
import json
import os
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_lib                                                      # noqa: E402
from test_gpu_reference_pin import TIMING_SHAPES, timing_inputs, wall_ms       # noqa: E402

out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
rows = []
for nb, gh, gw in TIMING_SHAPES:
    J, G, d, lg, rg = timing_inputs(nb, gh, gw)
    rows.append({"nb": nb, "gh": gh, "gw": gw,
                 "reference_fwd_ms": wall_ms(lambda: ref_lib.equation_construction(J, G, d)),
                 "reference_bwd_ms": wall_ms(lambda: ref_lib.equation_construction_grad(J, G, d, lg, rg))})
    del J, G, d
    torch.cuda.empty_cache()
doc = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": float(power), "cuda": torch.version.cuda, "rows": rows}
os.makedirs(out_dir, exist_ok=True)
json.dump(doc, open(os.path.join(out_dir, "ref_op_timing.json"), "w"), indent=1)
print(json.dumps(doc))
