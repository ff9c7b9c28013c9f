"""CPU oracle for the BA-layer LM hot path.  TEST INFRASTRUCTURE ONLY.

This package restates, line by line, the maths of frobelbest/BANet's BA layer (`bundlenet.py`, `utils.cu`, `legacy/ba.py`,
`legacy/utils_python.py`) in plain torch-CPU (float64 by default, float32 for the timed CPU baseline).  It is the checker that
the CUDA path in `banet_b200/` is compared against.

Rules (enforced by tests/test_abi_symbols.py::test_product_never_touches_the_oracle):
  * only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` legs may import it;
  * nothing under `banet_b200/` may import, call or fall back to it.

PARITY PINNED (round 2).  The reference ships no tests, golden vectors or fixtures, and TensorFlow-1.x / Python-2 cannot be
installed here — but the reference's own code does run, two ways, and the oracle is held to both:
  1. its Python: `oracle/tf1_shim.py` is a torch-backed emulation of the TF-1 API subset the reference touches; with it registered as
     `tensorflow`, /root/reference/bundlenet.py, legacy/ba.py and legacy/utils_python.py execute from their own source text
     (tests/golden/gen_ref_golden.py -> tests/golden/ref_*.npz).  tests/test_oracle_pinned.py holds every oracle function —
     SE(3) helpers, Jacobians, grad_fixed, rays, BundleIteration, CameraIteration, BundleResize, CameraResize, the legacy
     CameraIteration / CameraIteration2 (accept / reject) and the tracker loop — to those outputs at 1e-10.
     Third-party restatement is confined to the shim (resampler, LU / QR solves, selu, l2_normalize, REFLECT pad) and listed there.
  2. its CUDA: `oracle/Makefile` compiles /root/reference/utils.cu UNMODIFIED (EquationConstruction + EquationConstructionGrad: real
     cuBLAS batched GEMMs + the reference's own reduction / tiling kernels) against stand-in TensorFlow headers (oracle/tf_stub) into
     oracle/_ref/libbanet_ref_eqc.so.  On the GPU, tests/test_gpu_reference_pin.py compares the kernels AND the oracle with it (through stored outputs, tests/golden/ref_eqc_pin.npz);
     tests/golden/ref_eqc.npz (written by that compiled kernel on a B200) pins the oracle and the cuBLAS-chain replay
     (oracle/gemm_chain.py) on the CPU (tests/test_oracle_pinned_eqc.py).
Further self-consistency checks (tests/test_oracle_consistency.py): materialised reference form == structured block form == chunked
form; planted-solution scenes converge.
"""
