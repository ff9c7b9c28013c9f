"""GPU tests of the generation-7 tensor-core build kernel (TMA-staged F2 windows, banet_b200/csrc/lm_build_tc7.cu): against the
float64 oracle and the FP32 SIMT path (itself pinned to the oracle in test_gpu_parity.py) on shapes that exercise edge tiles, the
band tile order, pair changes inside a CTA, the per-tile global-tap fallback and its forced variant."""
import numpy as np
import pytest
import torch

from helpers import O, oracle_level_inputs, rel_fro, to_cuda32

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _restore_tuning():
    from banet_b200 import _lib
    yield
    _lib.set_tuning()


def _scene(nb, H, W, C, seed, device="cuda", **kw):
    from banet_b200 import synth
    return synth.make_scene(nb=nb, H=H, W=W, C=C, K=128, level_ids=(3,), seed=seed, device=device, dtype=torch.float32, **kw)


def _f2_level(ops, lv, grid=True):
    C = lv.conv1.shape[2]
    return ops.Level(lv.conv1, lv.conv2[..., :C].contiguous(), lv.intr, lv.p, lv.D, lv.B, grid=lv.grid if grid else None)


@pytest.mark.parametrize("C", [64, 128])
@pytest.mark.parametrize("prec", [1, 2])
def test_tc7_matches_oracle(prec, C):
    """Small dense level (ragged 8x8 edge tiles: 44x52) against the float64 oracle's block form."""
    from banet_b200 import ops, _lib
    sc = _scene(3, 44, 52, C, seed=70 + C, device="cpu")
    lv = sc.levels[0]
    Wt = sc.W0 + 0.01 * torch.randn(sc.W0.shape, generator=torch.Generator().manual_seed(2))
    a = oracle_level_inputs(lv)
    rH, rg, rrbar, rnv = O.normal_equations_structured(a["conv1"], a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], a["p"], a["D"], a["B"],
                                                       sc.R0.double(), sc.T0.double(), Wt.double())
    L = ops.Level(to_cuda32(lv.conv1), to_cuda32(lv.conv2[..., :C]), to_cuda32(lv.intr), to_cuda32(lv.p), to_cuda32(lv.D), to_cuda32(lv.B), grid=lv.grid)
    _lib.set_tuning(tc_generation=7)
    H, g, rbar, nv = ops.lm_build(L, to_cuda32(sc.R0), to_cuda32(sc.T0), to_cuda32(Wt), precision=prec)
    tol = {1: 2e-4, 2: 2e-5}[prec]       # N = 2288 points per pair: tf32 rounding of H averages out as 1/sqrt(N)
    print(f"prec={prec} C={C}: relH {rel_fro(H, rH):.2e} relg {rel_fro(g, rg.squeeze(-1)):.2e}")
    assert torch.equal(nv.cpu().double(), rnv)
    assert rel_fro(H, rH) < tol and rel_fro(g, rg.squeeze(-1)) < tol
    assert rel_fro(H[:, :6, :6], rH[:, :6, :6]) < 2e-5 and rel_fro(g[:, :6], rg[:, :6, 0]) < 2e-5      # pose block: fp32 only
    assert rel_fro(rbar / lv.N, rrbar.squeeze(1)) < 2e-5
    assert torch.equal(H, H.transpose(1, 2))


@pytest.mark.parametrize("band", [1, 3, 4, 30])
def test_tc7_band_order_and_generation6_agree(band):
    """240x320, 2 pairs = 2400 tiles over 132 CTAs (ring wrap, two pair spans per CTA): every band order gives
    the generation-6 result up to fp32 summation order, run-to-run bit reproducible."""
    from banet_b200 import ops, _lib
    sc = _scene(2, 240, 320, 128, seed=17)
    L = _f2_level(ops, sc.levels[0])
    Wt = sc.W0 + 0.01 * torch.randn(sc.W0.shape, generator=torch.Generator().manual_seed(3)).cuda()
    Hs, gs, rbs, nvs = ops.lm_build(L, sc.R0, sc.T0, Wt, precision=0)
    for prec in (1, 2):
        _lib.set_tuning(tc_generation=6)
        H6, g6, rb6, nv6 = ops.lm_build(L, sc.R0, sc.T0, Wt, precision=prec)
        _lib.set_tuning(tc_generation=7, tc7_band_rows=band)
        H, g, rbar, nv = ops.lm_build(L, sc.R0, sc.T0, Wt, precision=prec)
        H2, g2, rbar2, nv2 = ops.lm_build(L, sc.R0, sc.T0, Wt, precision=prec)
        assert torch.equal(H, H2) and torch.equal(g, g2) and torch.equal(rbar, rbar2)
        assert torch.equal(nv, nvs) and torch.equal(nv6, nvs)
        tol = {1: 5e-4, 2: 1e-4}[prec]
        print(f"band={band} prec={prec}: vs simt relH {rel_fro(H, Hs):.2e} relg {rel_fro(g, gs):.2e}; vs gen6 relH {rel_fro(H, H6):.2e}")
        assert rel_fro(H, Hs) < tol and rel_fro(g, gs) < tol
        assert rel_fro(H[:, :6, :6], Hs[:, :6, :6]) < 2e-5 and rel_fro(rbar, rbs) < 2e-5
        assert rel_fro(H[:, :6, :6], H6[:, :6, :6]) < 2e-5 and rel_fro(rbar, rb6) < 2e-5


@pytest.mark.parametrize("force", [False, True])
def test_tc7_large_motion_fallback(force):
    """Strong zoom / rotation (8 degrees, 25 cm): many tiles overflow the staged window and take the global-tap fallback (all of them when
    forced); the result must not depend on which path a tile took."""
    from banet_b200 import ops, _lib
    sc = _scene(2, 120, 160, 64, seed=23, rot_deg=8.0, trans_m=0.25)
    L = _f2_level(ops, sc.levels[0])
    Wt = sc.W0 + 0.02 * torch.randn(sc.W0.shape, generator=torch.Generator().manual_seed(4)).cuda()
    Hs, gs, rbs, nvs = ops.lm_build(L, sc.R0, sc.T0, Wt, precision=0)
    _lib.set_tuning(tc_generation=7, tc7_force_direct=force)
    H, g, rbar, nv = ops.lm_build(L, sc.R0, sc.T0, Wt, precision=2)
    print(f"force={force}: nvalid {nv.tolist()} relH {rel_fro(H, Hs):.2e} relg {rel_fro(g, gs):.2e}")
    assert torch.equal(nv, nvs) and float(nv.min()) > 1000
    assert rel_fro(H, Hs) < 1e-4 and rel_fro(g, gs) < 1e-4 and rel_fro(rbar, rbs) < 2e-5
    assert rel_fro(H[:, :6, :6], Hs[:, :6, :6]) < 2e-5


def test_tc7_whole_solve_under_the_default_policy():
    """A 2-level solve through banet_lm_run under the AUTO (level-wise) policy: 120x160 -> TF32X3 (generation 6), 240x320 -> TF32X1 on the
    generation-6 or (forced) generation-7 kernel; against the FP32 SIMT path (held to the oracle in test_gpu_parity.py) at the north-star tolerance."""
    from banet_b200 import ops, _lib, synth
    sc = synth.make_scene(nb=2, H=240, W=320, C=128, K=128, level_ids=(2, 3), seed=31, device="cuda", dtype=torch.float32)
    levels = [_f2_level(ops, l) for l in sc.levels]
    R0, T0, W0, st0 = ops.lm_run(levels, 4, sc.R0, sc.T0, sc.W0, lambda_fixed=0.5, precision=_lib.PREC_FP32_SIMT)
    out = {}
    for gen in (6, 7):
        _lib.set_tuning(tc_generation=gen)
        R, T, W, st = ops.lm_run(levels, 4, sc.R0, sc.T0, sc.W0, lambda_fixed=0.5, precision=_lib.PREC_AUTO)
        assert int(st.abs().max()) == 0
        fin = sc.levels[-1]
        d = ops.depth_compose(fin.D.reshape(2, -1), fin.B, W); d0 = ops.depth_compose(fin.D.reshape(2, -1), fin.B, W0)
        e = dict(R=rel_fro(R, R0), T=rel_fro(T, T0), W=rel_fro(W, W0), depth=rel_fro(d, d0))
        print(f"generation {gen}: " + " ".join(f"{k}={v:.2e}" for k, v in e.items()))
        assert e["R"] < 1e-4 and e["T"] < 1e-4 and e["depth"] < 1e-4
