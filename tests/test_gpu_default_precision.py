"""GPU: the SHIPPED default precision policy, whole solves, against the float64 oracle at the north-star tolerance.

cfg2-shaped case, sized so that the float64 oracle finishes in about a minute of host time:
nb = 1, 4 dense levels 40x30 .. 320x240 (the finest level is above the 65536-point threshold of the level-wise policy, so both TF32X3 and TF32X1 run),
C = K = 128, lambda-MLP in the loop, 5 LM iterations per level; both conv2 layouts (the reference's [F2|gx|gy] and F2-only).  Asserted at 1e-4 rel-fro on R, T, W and the depth output D + B.W (bundlenet.py:397) for AUTO (what
bench.py times) and for the fp32-grade modes; the other modes are printed."""
import pytest
import torch

from helpers import O, oracle_level_inputs, rel_fro

pytestmark = pytest.mark.gpu
TOL = 1e-4


@pytest.fixture(scope="module")
def cfg2_case():
    from banet_b200 import ops, synth
    nb = 1
    sc = synth.make_scene(nb=nb, H=240, W=320, C=128, K=128, level_ids=(0, 1, 2, 3), seed=1236, device="cuda", dtype=torch.float32)
    mlps = [O.init_lambda_mlp(128, seed=7 + l.level, dtype=torch.float32) for l in sc.levels]
    olv = []
    for l, m in zip(sc.levels, mlps):
        class _L:
            pass
        cl = _L()
        cl.conv1, cl.conv2, cl.intr, cl.p, cl.D, cl.B = [t.cpu() for t in (l.conv1, l.conv2, l.intr, l.p, l.D, l.B)]
        cl.N = l.N
        cl.intr_tiled = lambda cl=cl: tuple(cl.intr[:, i:i + 1].expand(-1, cl.N).contiguous() for i in range(4))
        a = oracle_level_inputs(cl)
        olv.append(O.LevelInputs(a["conv1"], a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"], [(w.double(), b.double()) for w, b in m]))
    oR, oT, oW = O.lm_solve_structured(olv, 5, sc.R0.cpu().double(), sc.T0.cpu().double(), sc.W0.cpu().double())
    oD = olv[-1].D + olv[-1].B @ oW
    del olv
    return sc, [ops.pack_mlp(m).cuda() for m in mlps], (oR, oT, oW, oD)


@pytest.mark.parametrize("layout", ["3c", "f2"])
def test_default_precision_whole_solve_vs_oracle(cfg2_case, layout):
    from banet_b200 import ops, _lib
    sc, packed, (oR, oT, oW, oD) = cfg2_case
    levels = [ops.Level(l.conv1, l.conv2 if layout == "3c" else l.conv2[..., :128].contiguous(), l.intr, l.p, l.D, l.B, grid=l.grid) for l in sc.levels]
    fin = sc.levels[-1]
    for name, prec, asserted in (("auto", _lib.PREC_AUTO, True), ("fp32", _lib.PREC_FP32_SIMT, True), ("tf32x3", _lib.PREC_TF32X3, True),
                                 ("levelwise", _lib.PREC_TF32_LEVELWISE, False), ("tf32x2", _lib.PREC_TF32X2, False), ("tf32x1", _lib.PREC_TF32X1, False)):
        R, T, W, st = ops.lm_run(levels, 5, sc.R0, sc.T0, sc.W0, mlp_packed=packed, l2_regularizer_base=1000.0, precision=prec)
        d = fin.D.cpu().double() + fin.B.cpu().double() @ W.cpu().double()
        e = dict(R=rel_fro(R, oR), T=rel_fro(T, oT), W=rel_fro(W, oW), depth=rel_fro(d, oD))
        print(f"{layout}/{name}: " + " ".join(f"{k}={v:.2e}" for k, v in e.items()))
        assert int(st.abs().max()) == 0
        if asserted:
            assert max(e.values()) < TOL, (layout, name, e)
