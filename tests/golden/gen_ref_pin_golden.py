"""Writes ref_eqc_pin.npz: outputs of the reference's OWN compiled op kernels (EquationConstruction + Grad, utils.cu, built unmodified
by oracle/Makefile into oracle/_ref/) on the seeded cases of tests/test_gpu_reference_pin.py, so that the test compares against them
without the reference library.  Needs a GPU and oracle/_ref/libbanet_ref_eqc.so:  python tests/golden/gen_ref_pin_golden.py [outdir]
AtA / Atb are stored whole; the gradients as a fixed seeded sample of 4096 entries each (tests/test_gpu_reference_pin.py:sample_index)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_lib                                  # noqa: E402
from test_gpu_reference_pin import CASES, _inputs, sample_index   # noqa: E402

out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
z = {"meta": np.array([torch.cuda.get_device_name(0), torch.version.cuda])}
for i, (nb, N, C, P) in enumerate(CASES):
    J, G, d, lg, rg = _inputs(nb, N, C, P)
    A, b = ref_lib.equation_construction(J.cuda(), G.cuda(), d.cuda())
    dJ, dG, dd = ref_lib.equation_construction_grad(J.cuda(), G.cuda(), d.cuda(), lg.cuda(), rg.cuda())
    z[f"c{i}_AtA"] = A.cpu().numpy(); z[f"c{i}_Atb"] = b.cpu().numpy()
    for name, t in (("dJ", dJ), ("dG", dG), ("dd", dd)):
        t = t.cpu().reshape(-1)
        z[f"c{i}_{name}_sample"] = t[sample_index(t.numel(), i)].numpy()
os.makedirs(out_dir, exist_ok=True)
np.savez_compressed(os.path.join(out_dir, "ref_eqc_pin.npz"), **z)
print("wrote", os.path.join(out_dir, "ref_eqc_pin.npz"))
