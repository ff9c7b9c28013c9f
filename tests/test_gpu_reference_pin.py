"""GPU: the reference's OWN native op — EquationConstruction / EquationConstructionGrad compiled unmodified from utils.cu
(oracle/_ref, built by oracle/Makefile against the TensorFlow stand-in headers) — against (a) the float64 oracle and (b) the kernels
banet_eqc_fwd / banet_eqc_bwd on the same inputs.  The reference op's outputs on these seeded cases are stored in
tests/golden/ref_eqc_pin.npz (tests/golden/gen_ref_pin_golden.py): AtA / Atb whole, the gradients as a fixed sample of 4096 entries.
This pins SURVEY §8 rows a8-a10."""
import os

import numpy as np
import pytest
import torch

from helpers import O, rel_fro, GOLDEN_DIR

pytestmark = pytest.mark.gpu
CASES = [(2, 70, 12, 22), (1, 33, 5, 6), (2, 257, 128, 134), (1, 64, 8, 38)]
SAMPLE = 4096


def _inputs(nb, N, C, P):
    g = torch.Generator().manual_seed(nb * 1000 + N + P)
    mk = lambda *s: torch.randn(*s, generator=g)
    return mk(nb, N, 2, P), mk(nb, N, C, 2), mk(nb, N, C, 1), mk(nb, P, P), mk(nb, P, 1)


def sample_index(numel, case):
    """Fixed seeded sample of flat indices (all of them when the tensor is small)."""
    if numel <= SAMPLE:
        return torch.arange(numel)
    return torch.randperm(numel, generator=torch.Generator().manual_seed(100 + case))[:SAMPLE].sort().values


def _golden():
    return np.load(os.path.join(GOLDEN_DIR, "ref_eqc_pin.npz"))


def _rel_sample(t, z, key, case):
    """Relative Frobenius error on the stored sample of the reference tensor."""
    t = t.detach().double().cpu().reshape(-1)[sample_index(t.numel(), case)]
    ref = torch.from_numpy(z[f"c{case}_{key}_sample"]).double()
    return float((t - ref).norm() / ref.norm().clamp_min(1e-300))


@pytest.mark.parametrize("nb,N,C,P", CASES)
def test_reference_op_vs_oracle_and_b200_kernels(nb, N, C, P):
    from banet_b200 import ops
    case = CASES.index((nb, N, C, P))
    z = _golden()
    J, G, d, lg, rg = _inputs(nb, N, C, P)
    rA, rb = z[f"c{case}_AtA"], z[f"c{case}_Atb"]
    oA, ob = O.equation_construction(J.double(), G.double(), d.double())
    # the reference sums N per-pixel fp32 matrices serially in fp32 (utils.cu:181-198): ~1e-6 per element
    assert rel_fro(rA, oA) < 2e-5 and rel_fro(rb, ob) < 2e-5
    A, b = ops.equation_construction(J.cuda(), G.cuda(), d.cuda())
    assert rel_fro(A, rA) < 2e-5 and rel_fro(b, rb) < 2e-5
    oJ, oG, od = O.equation_construction_grad(J.double(), G.double(), d.double(), lg.double(), rg.double())      # the 2*A*Ghat form, utils.cu:648
    assert _rel_sample(oJ, z, "dJ", case) < 2e-5 and _rel_sample(oG, z, "dG", case) < 2e-5 and _rel_sample(od, z, "dd", case) < 2e-5
    dJ, dG, dd = ops.equation_construction_grad(J.cuda(), G.cuda(), d.cuda(), lg.cuda(), rg.cuda(), exact_sym=False)
    assert _rel_sample(dJ, z, "dJ", case) < 2e-5 and _rel_sample(dG, z, "dG", case) < 2e-5 and _rel_sample(dd, z, "dd", case) < 2e-5
    print(f"nb={nb} N={N} C={C} P={P}: ref vs oracle AtA {rel_fro(rA, oA):.1e}; kernels vs ref AtA {rel_fro(A, rA):.1e} "
          f"dJ {_rel_sample(dJ, z, 'dJ', case):.1e}")


def test_reference_op_reproduces_committed_golden():
    """tests/golden/ref_eqc.npz holds inputs and outputs of the compiled reference op (tests/golden/gen_ref_eqc_golden.py); the CPU suite
    holds the oracle to it (tests/test_oracle_pinned_eqc.py).  Here the same op boundary, served by banet_eqc_fwd / banet_eqc_bwd
    (exact_sym=False: the reference's 2*A*Ghat form), must reproduce it."""
    from banet_b200 import ops
    z = np.load(os.path.join(GOLDEN_DIR, "ref_eqc.npz"))
    J, G, d, lg, rg = [torch.tensor(z[k]).cuda() for k in ("in_J", "in_G", "in_d", "in_left_grad", "in_right_grad")]
    A, b = ops.equation_construction(J, G, d)
    dJ, dG, dd = ops.equation_construction_grad(J, G, d, lg, rg, exact_sym=False)
    for got, key in ((A, "out_AtA"), (b, "out_Atb"), (dJ, "out_dJ"), (dG, "out_dG"), (dd, "out_dd")):
        assert rel_fro(got, z[key]) < 2e-5, key


# timing shapes: the reference's own scale (nb=2, 4096 sampled points, legacy/seq_example.py:12) and a 160x120 level
TIMING_SHAPES = ((2, 64, 64), (4, 120, 160))


def timing_inputs(nb, gh, gw):
    N, C, K = gh * gw, 128, 128; P = K + 6
    g = torch.Generator().manual_seed(7)
    J = torch.randn(nb, N, 2, P, generator=g).cuda(); G = torch.randn(nb, N, C, 2, generator=g).cuda(); d = torch.randn(nb, N, C, 1, generator=g).cuda()
    lg = torch.randn(nb, P, P, generator=g).cuda(); rg = torch.randn(nb, P, 1, generator=g).cuda()
    return J, G, d, lg, rg


def wall_ms(fn, reps=5):
    """Median wall time of synchronous calls (the reference harness synchronises the device itself)."""
    import time
    fn(); torch.cuda.synchronize(); ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); fn(); torch.cuda.synchronize(); ts.append(time.perf_counter() - t0)
    return sorted(ts)[len(ts) // 2] * 1e3


def test_reference_op_timed_beside_the_b200_kernels():
    """The reference's own CUDA op (cuBLAS batched SGEMM chain + its serial column reduction, utils.cu:331-414 / :613-690) against the
    kernels behind the same op boundary, at TIMING_SHAPES.  The reference op's times were measured on an H100 80GB HBM3 and are stored in
    tests/golden/ref_op_timing.json (tests/golden/gen_ref_timing_golden.py, card and power limit recorded there); the kernels are timed
    here.  Also the fused layer-level build (never materialises J, G, d) at the same shape, reported.  The single assertion is that the
    replacement is not slower."""
    import json
    from banet_b200 import ops, synth
    ref = json.load(open(os.path.join(GOLDEN_DIR, "ref_op_timing.json")))
    for nb, gh, gw in TIMING_SHAPES:
        J, G, d, lg, rg = timing_inputs(nb, gh, gw)
        stored = next(r for r in ref["rows"] if (r["nb"], r["gh"], r["gw"]) == (nb, gh, gw))
        row = {"nb": nb, "N": gh * gw, "reference_fwd_ms": stored["reference_fwd_ms"], "reference_bwd_ms": stored["reference_bwd_ms"],
               "eqc_fwd_ms": wall_ms(lambda: ops.equation_construction(J, G, d)),
               "eqc_bwd_ms": wall_ms(lambda: ops.equation_construction_grad(J, G, d, lg, rg))}
        del J, G, d
        sc = synth.make_scene(nb=nb, H=gh, W=gw, C=128, K=128, level_ids=(3,), seed=11, device="cuda", dtype=torch.float32)
        lv = sc.levels[0]; L = ops.Level(lv.conv1, lv.conv2, lv.intr, lv.p, lv.D, lv.B, grid=lv.grid)
        row["fused_build_fp32_ms"] = wall_ms(lambda: ops.lm_build(L, sc.R0, sc.T0, sc.W0, precision=0))
        row["fused_build_auto_ms"] = wall_ms(lambda: ops.lm_build(L, sc.R0, sc.T0, sc.W0, precision=-1))
        print(row)
        assert row["eqc_fwd_ms"] < row["reference_fwd_ms"] and row["eqc_bwd_ms"] < row["reference_bwd_ms"]
