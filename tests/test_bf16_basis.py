"""bfloat16 depth basis (banet_level_t::basis_dtype = BANET_DTYPE_BF16): B read as bf16 by the build kernels, their backward, depth_compose,
BundleNet and the host pipeline, independently of the features' dtype.  bf16 -> fp32 is exact, so every run on a bf16 basis is checked against
the same call on the widened basis (B.bfloat16().float()).  The forward keeps the fp32 summation orders and, on the tensor cores, only skips
products of an exactly zero A_lo, so the build and the whole solve are bitwise those of the widened run.
CPU tests: argument checks through the loaded library and a host-side model of the bf16 basis tile of the tensor-core build."""
import ctypes
import itertools

import pytest
import torch

from helpers import scene_case, rel_fro, to_cuda32
from banet_b200 import _lib

gpu = pytest.mark.gpu
BF = torch.bfloat16


# ------------------------------------------------------------------------------------------------ CPU: the C-ABI
def _level(**kw):
    lv = _lib.BanetLevel(2, 4096, 64, 32, 48, 64, 192, 1, 1, 1, 1, 1, 1, 0, 0)
    for k, v in kw.items():
        setattr(lv, k, v)
    return lv


def test_struct_built_without_the_field_keeps_an_fp32_basis():
    assert _level().basis_dtype == _lib.DTYPE_F32 == 0
    assert _level(feature_dtype=_lib.DTYPE_BF16).basis_dtype == 0


@pytest.mark.parametrize("bad", [2, -1, 7])
def test_bad_basis_dtype_is_rejected_before_any_cuda_call(bad):
    lib = _lib.load()
    opts = ctypes.byref(_lib.BanetSolveOpts(1e-5, 1, 0))
    lv = _level(basis_dtype=bad)
    rc = lib.banet_lm_build(ctypes.byref(lv), 1, 1, 1, 0, 1, 1, 1, 1, 1, 1 << 20, None)
    assert rc == -1 and b"basis_dtype" in lib.banet_last_error()
    rc = lib.banet_lm_build_bwd(ctypes.byref(lv), 1, 1, 1, 1, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1, None)
    assert rc == -1 and b"basis_dtype" in lib.banet_last_error()
    arr = (_lib.BanetLevel * 1)(lv)
    rc = lib.banet_lm_run(arr, 1, 1, None, 1.0, 0.5, opts, 0, 1, 1, 1, 1, 1, 1 << 20, None)
    assert rc == -1 and b"basis_dtype" in lib.banet_last_error()
    rc = lib.banet_lm_window_batch_run(arr, 1, 1, 1, None, 1.0, 0.5, opts, 0, 1, 1, 1, 1, 1, 1 << 20, None)
    assert rc == -1 and b"basis_dtype" in lib.banet_last_error()


def test_levels_without_a_basis_still_check_the_field():
    lib = _lib.load()
    arr = (_lib.BanetLevel * 1)(_level(K=0, basis_dtype=3))
    iters = (ctypes.c_int * 1)(3)
    rc = lib.banet_lm_track_legacy(arr, 1, iters, None, ctypes.byref(_lib.BanetLegacyOpts(1, 1e-5, 2e-4, 1.0)), 1, 1, None, 1, 1, 1, 1 << 20, None)
    assert rc == -1 and b"basis_dtype" in lib.banet_last_error()


# ------------------------------------------------------------------------------------------------ CPU: model of the bf16 basis tile
# lm_build_tc6.cu with TB = bf16: one stage holds KBLK blocks of [64 px][32 columns x 2 B] (4096 B each), 64B swizzle.
def sw64_off(r, c):                               # tc_utils.cuh
    return r * 64 + ((c ^ ((r >> 1) & 3)) << 4)


def sw128_off(r, c):
    return r * 128 + ((c ^ (r & 7)) << 4)


def bf16_col(off):                                # byte offset inside a block -> (pixel row, basis column in the block)
    r, rem = divmod(off, 64)
    chunk, byte = divmod(rem, 16)
    return r, 8 * (chunk ^ ((r >> 1) & 3)) + byte // 2


def _ways(offs, width):
    """Wavefronts of one access of `width` bytes per lane, relative to the conflict-free count: a wavefront serves 128 B (LDS.128 per
    quarter-warp, LDS.64 per half-warp, LDS.32 per warp); ways = the most distinct 128-B lines any bank is asked for within one phase."""
    phase = 128 // width
    worst = 0
    for p0 in range(0, 32, phase):
        use = {}
        for off in offs[p0:p0 + phase]:
            for b in range(0, width, 4):
                use.setdefault(((off + b) % 128) // 4, set()).add((off + b) // 128)
        worst = max(worst, max(len(v) for v in use.values()))
    return worst


def test_sw64_is_a_bijection_on_a_block():
    slots = [sw64_off(r, c) for r in range(64) for c in range(4)]
    assert sorted(slots) == list(range(0, 4096, 16))
    for r, c in itertools.product(range(64), range(4)):
        for e in range(8):
            assert bf16_col(sw64_off(r, c) + 2 * e) == (r, 8 * c + e)


def _geometry_walk(lane, gwi, kblk):
    """The b.W walk of geometry warp gwi: lane (r16, hf) reads one LDS.128 per even step i and takes 4 columns per step."""
    r16, hf = lane & 15, lane >> 4
    nlr = gwi * 16 + r16
    loads, cols = [], []
    for i in range(16):
        blk, c = 2 * hf + (i >> 3), i & 7
        if blk >= kblk:
            continue
        off = blk * 4096 + sw64_off(nlr, c >> 1)
        if c % 2 == 0:
            loads.append(off)
        col0 = [bf16_col(off - blk * 4096 + 2 * (4 * (c & 1) + e)) for e in range(4)]
        assert all(r == nlr for r, _ in col0)
        cols.append([blk * 32 + cc for _, cc in col0])
    return loads, cols


@pytest.mark.parametrize("kblk", [4, 2, 1])
def test_bw_walk_covers_the_row_in_the_fp32_order(kblk):
    for gwi in range(4):
        for r16 in range(16):
            seen = []
            for hf in range(2):
                _, cols = _geometry_walk(r16 + 16 * hf, gwi, kblk)
                # fp32 walk: step i reads float4 chunk c of block blk = columns blk*32 + 4c .. +3, acc.x..w in that order
                want = [[blk * 32 + 4 * c + e for e in range(4)] for i in range(16) for blk, c in [(2 * hf + (i >> 3), i & 7)] if blk < kblk]
                assert cols == want
                seen += [x for step in cols for x in step]
            assert sorted(seen) == list(range(32 * kblk))


def test_bw_walk_loads_are_conflict_free():
    for gwi, k in itertools.product(range(4), range(8)):
        offs = [_geometry_walk(lane, gwi, 4)[0][k] for lane in range(32)]
        assert _ways(offs, 16) == 1


def _r_walk(lane, awi, kblk):
    """The algebra warps' R rows on a bf16 tile: lane (r16, hf) reads 16-B chunk m of block blk (LDS.128) and writes fp32 chunks 2m, 2m+1
    of the R row (two STS.128)."""
    r16, hf = lane & 15, lane >> 4
    nlr = awi * 16 + r16
    out = []
    for i in range(8):
        blk, m = 2 * hf + (i >> 2), i & 3
        if blk >= kblk:
            continue
        src = blk * 4096 + sw64_off(nlr, m)
        dst = [blk * 8192 + sw128_off(nlr, 2 * m + hc) for hc in range(2)]
        out.append((src, dst, nlr, [blk * 32 + bf16_col(src - blk * 4096 + 2 * e)[1] for e in range(8)]))
    return out


@pytest.mark.parametrize("kblk", [4, 2, 1])
def test_r_walk_writes_every_column_of_its_row_once(kblk):
    for awi, r16 in itertools.product(range(4), range(16)):
        written = {}
        for hf in range(2):
            for src, dst, nlr, cols in _r_walk(r16 + 16 * hf, awi, kblk):
                for hc in range(2):
                    blk, rem = divmod(dst[hc], 8192)
                    r, rr = divmod(rem, 128)
                    assert r == nlr
                    chunk = (rr // 16) ^ (r & 7)
                    for e in range(4):                 # the fp32 R element at (row, column) gets the bf16 basis column it multiplies
                        written.setdefault(blk * 32 + 4 * chunk + e, []).append(cols[4 * hc + e])
        assert sorted(written) == list(range(32 * kblk))
        assert all(v == [k] for k, v in written.items())


def test_r_walk_loads_and_stores_are_conflict_free():
    for awi, i in itertools.product(range(4), range(8)):
        walk = [_r_walk(lane, awi, 4)[i] for lane in range(32)]
        assert _ways([w[0] for w in walk], 16) == 1
        for hc in range(2):
            assert _ways([w[1][hc] for w in walk], 16) == 1


def test_a_fragment_lds32_reads_the_mapped_columns_with_a_two_way_conflict():
    """mma_role.cuh, BB: lane (g, t) reads the word of columns 16mb+2g, 16mb+2g+1 at pixel rows t and t+4 of step kk (LDS.32 each)."""
    for mb, kk in itertools.product(range(8), range(8)):
        lo, hi = [], []
        for lane in range(32):
            g, t = lane >> 2, lane & 3
            oab = t * 64 + (((g >> 2) ^ (t >> 1)) << 4) + (g & 3) * 4
            base = (mb >> 1) * 4096 + kk * 512
            o_lo = base + oab + 32 * (mb & 1)
            o_hi = base + 256 + oab + 32 * ((mb & 1) ^ 1)
            for off, px in ((o_lo, t), (o_hi, t + 4)):
                r, col = bf16_col(off - (mb >> 1) * 4096)
                assert (r, col) == (8 * kk + px, 16 * (mb & 1) + 2 * g)
            lo.append(o_lo); hi.append(o_hi)
        assert _ways(lo, 4) == 2 and _ways(hi, 4) == 2


# ------------------------------------------------------------------------------------------------ GPU helpers
def _widened(t):
    return t.to(BF).float()


def _build_case(C, K, points, layout, fdt, seed):
    """A seeded level on the GPU with its basis rounded to bf16: (bf16-basis level, widened level, R, T, W).  fdt: the features' dtype."""
    from banet_b200 import ops
    sc = scene_case(nb=2, H=48, W=64, C=C, K=K, level_ids=(3,), seed=seed, n_points=400 if points == "sparse" else None, dtype=torch.float32)
    lv = sc.levels[0]
    conv2 = lv.conv2 if layout == "3C" else lv.conv2[..., :C].contiguous()
    c1, c2 = lv.conv1.cuda().to(fdt), conv2.cuda().to(fdt)
    B = lv.B.cuda().to(BF)
    W = to_cuda32(sc.W0 + 0.01 * torch.randn(sc.W0.shape, generator=torch.Generator().manual_seed(seed)))
    mk = lambda b: ops.Level(c1, c2, to_cuda32(lv.intr), to_cuda32(lv.p), to_cuda32(lv.D), b, grid=lv.grid)
    return mk(B), mk(B.float()), to_cuda32(sc.R0), to_cuda32(sc.T0), W


def _assert_build_equal(lb, lf, R, T, W, prec):
    from banet_b200 import ops
    ob = ops.lm_build(lb, R, T, W, prec)
    of = ops.lm_build(lf, R, T, W, prec)
    assert float(of[3].min()) > 0
    for a, b in zip(ob, of):
        assert torch.equal(a, b)


MODES = {"X1": _lib.PREC_TF32X1, "X2": _lib.PREC_TF32X2, "X3": _lib.PREC_TF32X3, "AUTO": _lib.PREC_AUTO}
FEATURES = {"fp32": torch.float32, "bf16": BF}


@gpu
@pytest.mark.parametrize("points", ["dense", "sparse"])
@pytest.mark.parametrize("layout", ["3C", "F2"])
@pytest.mark.parametrize("K", [16, 128, 256])
def test_simt_build_is_bitwise_the_widened_build(K, layout, points):
    _lib.require_device()
    for fname, fdt in FEATURES.items():
        lb, lf, R, T, W = _build_case(64, K, points, layout, fdt, seed=K + 5)
        _assert_build_equal(lb, lf, R, T, W, _lib.PREC_FP32_SIMT)


@gpu
@pytest.mark.parametrize("features", list(FEATURES))
@pytest.mark.parametrize("points", ["dense", "sparse"])
@pytest.mark.parametrize("layout", ["3C", "F2"])
@pytest.mark.parametrize("C", [64, 128])
@pytest.mark.parametrize("K", [32, 64, 128])
@pytest.mark.parametrize("mode", list(MODES))
def test_tensor_core_build_is_bitwise_the_widened_build(mode, K, C, layout, points, features):
    _lib.require_device()
    lb, lf, R, T, W = _build_case(C, K, points, layout, FEATURES[features], seed=7 * C + K)
    _assert_build_equal(lb, lf, R, T, W, MODES[mode])


@gpu
@pytest.mark.parametrize("layout", ["3C", "F2"])
@pytest.mark.parametrize("C,K", [(64, 128), (128, 64), (8, 16)])
def test_build_backward_matches_the_widened_backward(C, K, layout):
    """dB comes back fp32 for a bf16 basis; every gradient equals the widened run's up to the order of the fp32 atomics."""
    from banet_b200 import ops
    _lib.require_device()
    for fdt in FEATURES.values():
        lb, lf, R, T, W = _build_case(C, K, "sparse", layout, fdt, seed=3 + C + K)
        P = 6 + K
        g = torch.Generator(device="cuda").manual_seed(4)
        dH = torch.randn(2, P, P, device="cuda", generator=g); dg = torch.randn(2, P, device="cuda", generator=g)
        dr = torch.randn(2, C, device="cuda", generator=g)
        ob = ops.lm_build_bwd(lb, R, T, W, dH, dg, dr)
        of = ops.lm_build_bwd(lf, R, T, W, dH, dg, dr)
        assert ob[3].dtype == torch.float32 and ob[3].shape == lb.B.shape
        for a, b in zip(ob, of):
            assert rel_fro(a, b) <= 1e-5


@gpu
def test_depth_compose_on_a_bf16_basis():
    from banet_b200 import ops
    _lib.require_device()
    g = torch.Generator(device="cuda").manual_seed(8)
    basis = torch.randn(3, 700, 40, device="cuda", generator=g).to(BF)
    d0 = torch.randn(3, 700, device="cuda", generator=g); W = torch.randn(3, 40, 1, device="cuda", generator=g)
    out = ops.depth_compose(d0, basis, W)
    assert out.dtype == torch.float32 and torch.equal(out, ops.depth_compose(d0, basis.float(), W))
    dout = torch.randn(3, 700, device="cuda", generator=g)
    db, dW = ops.depth_compose_bwd(dout, basis, W)
    db1, dW1 = ops.depth_compose_bwd(dout, basis.float(), W)
    assert db.dtype == torch.float32 and torch.equal(db, db1) and rel_fro(dW, dW1) <= 1e-6


def _run_scene(nb, C, K, seed, fdt=torch.float32, levels=(0, 1, 2, 3), layout="F2", **kw):
    from banet_b200 import ops, synth
    sc = synth.make_scene(nb=nb, H=96, W=128, C=C, K=K, level_ids=levels, seed=seed, device="cuda", **kw)
    mk = lambda l, B: ops.Level(l.conv1.to(fdt), (l.conv2 if layout == "3C" else l.conv2[..., :C].contiguous()).to(fdt), l.intr, l.p, l.D, B,
                                grid=l.grid)
    lb = [mk(l, l.B.to(BF)) for l in sc.levels]
    lf = [mk(l, l.B.to(BF).float()) for l in sc.levels]
    return sc, lb, lf


def _mlps(C, n, seed=9):
    from banet_b200 import ops
    g = torch.Generator().manual_seed(seed)
    dims = [C, 2 * C, 4 * C, 2 * C, C, 1]
    return [ops.pack_mlp([(torch.randn(dims[i], dims[i + 1], generator=g) * (2.0 / dims[i]) ** 0.5, torch.zeros(dims[i + 1])) for i in range(5)]).cuda()
            for _ in range(n)]


@gpu
@pytest.mark.parametrize("features", list(FEATURES))
def test_lm_run_is_bitwise_the_widened_run(features):
    from banet_b200 import ops
    _lib.require_device()
    sc, lb, lf = _run_scene(4, 128, 128, seed=13, fdt=FEATURES[features])
    mlps = _mlps(128, 4)
    ob = ops.lm_run(lb, 2, sc.R0, sc.T0, sc.W0, mlp_packed=mlps, l2_regularizer_base=1000.0)
    of = ops.lm_run(lf, 2, sc.R0, sc.T0, sc.W0, mlp_packed=mlps, l2_regularizer_base=1000.0)
    assert int(ob[3].abs().max()) == 0
    for a, b in zip(ob, of):
        assert torch.equal(a, b)


@gpu
def test_lm_window_batch_run_is_bitwise_the_widened_run():
    from banet_b200 import ops, synth
    _lib.require_device()
    nw, nf, C, K = 2, 3, 64, 128
    sc = synth.make_scene(nb=nw * nf, H=96, W=128, C=C, K=K, level_ids=(2, 3), seed=17, device="cuda", shared_depth=True, window_frames=nf)
    lb = [ops.Level(l.conv1, l.conv2[..., :C].contiguous(), l.intr, l.p, l.D, l.B.to(BF), grid=l.grid) for l in sc.levels]
    lf = [ops.Level(l.conv1, l.conv2, l.intr, l.p, l.D, l.B.float(), grid=l.grid) for l in lb]
    W0 = sc.W0.reshape(nw, nf, K, 1)[:, 0].contiguous()
    mlps = _mlps(C, 2)
    out_b = ops.lm_window_batch_run(lb, nw, 2, sc.R0, sc.T0, W0, mlp_packed=mlps)
    out_f = ops.lm_window_batch_run(lf, nw, 2, sc.R0, sc.T0, W0, mlp_packed=mlps)
    assert int(out_b[3].abs().max()) == 0
    for a, b in zip(out_b, out_f):
        assert torch.equal(a, b)


@gpu
@pytest.mark.parametrize("precision", [_lib.PREC_AUTO, _lib.PREC_FP32_SIMT, _lib.PREC_TF32X1])
def test_bf16_basis_build_is_bit_reproducible_from_poisoned_workspaces(precision, monkeypatch):
    from banet_b200 import ops
    _lib.require_device()
    lb, _, R, T, W = _build_case(128, 128, "dense", "F2", BF, seed=19)
    outs = []
    for fill in ("nan", "rand"):
        def make(nbytes, device, fill=fill):
            ws = torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)
            if fill == "nan":
                ws.view(torch.float32)[: ws.numel() // 4].fill_(float("nan"))
            else:
                ws.random_(0, 256)
            return ws
        monkeypatch.setattr(ops, "_ws", make)
        outs.append(ops.lm_build(lb, R, T, W, precision))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ GPU: BundleNet and the host pipeline
def _net(C, levels, **kw):
    from banet_b200.bundlenet import BundleNet
    kw.setdefault("strict_status", True)
    return BundleNet(C, levels=levels, **kw).cuda()


@gpu
@pytest.mark.parametrize("grad", [False, True])
def test_bundle_iteration_takes_a_bf16_basis(grad):
    _lib.require_device()
    sc, lb, lf = _run_scene(2, 64, 32, seed=29, levels=(3,))
    net = _net(64, ("3",)).train(grad)
    fx, fy, ox, oy = [sc.levels[0].intr[:, i:i + 1] for i in range(4)]

    def call(lv):
        B = lv.B.detach().clone().requires_grad_(grad)
        with torch.set_grad_enabled(grad):
            out = net.BundleIteration(lv.conv1, lv.conv2, fx, fy, ox, oy, lv.p, lv.D, B, sc.R0, sc.T0, sc.W0, 1000.0, "3")
            if grad:
                sum(o.sum() for o in out).backward()
        return out, B

    (ob, Bb), (of, Bf) = call(lb[0]), call(lf[0])
    for a, b in zip(ob, of):
        assert rel_fro(a, b) < 1e-6
    if grad:
        assert Bb.grad.dtype == BF and rel_fro(Bb.grad.float(), Bf.grad) < 1e-2


@gpu
def test_reference_split_rejects_a_bf16_basis():
    _lib.require_device()
    sc, lb, _ = _run_scene(2, 64, 32, seed=31, levels=(3,))
    net = _net(64, ("3",), training_path="reference_split").train()
    fx, fy, ox, oy = [sc.levels[0].intr[:, i:i + 1] for i in range(4)]
    lv = lb[0]
    B = lv.B.detach().clone().requires_grad_()
    with pytest.raises(RuntimeError, match="basis"):
        net.BundleIteration(lv.conv1, lv.conv2, fx, fy, ox, oy, lv.p, lv.D, B, sc.R0, sc.T0, sc.W0, 1000.0, "3")


@gpu
def test_bundle_resize_with_a_bf16_basis_and_bf16_layers():
    """Differentiable BundleResize on a bf16 basis and a bf16 pyramid against the same call with both widened (the tolerances of the bf16
    pyramid test: the sampled basis and conv1 are rounded to bf16)."""
    import gen_golden
    _lib.require_device()
    x = gen_golden.resize_inputs(nb=4, C=16, K=8)
    net = _net(16, ("0", "1", "2", "3"), strict_status=False).train()
    f32 = {k: to_cuda32(x[k]) for k in ("intr", "points", "depth", "R0", "T0")}
    lb = [to_cuda32(l).to(BF) for l in x["layers"]]
    bb = to_cuda32(x["basis"]).to(BF)

    def call(layers, basis):
        ls = [l.detach().clone().requires_grad_() for l in layers]
        b = basis.detach().clone().requires_grad_()
        Rs, Ts, Ds = net.BundleResize(f32["intr"], ls, f32["points"], b, f32["depth"], f32["R0"], f32["T0"])
        (sum(r.sum() for r in Rs) + sum(t.sum() for t in Ts) + sum(d.sum() for d in Ds)).backward()
        return Rs, Ts, Ds, ls, b

    Rb, Tb, Db, lsb, b1 = call(lb, bb)
    Rf, Tf, Df, lsf, b2 = call([l.float() for l in lb], bb.float())
    for xs, ys in ((Rb, Rf), (Tb, Tf), (Db, Df)):
        for u, v in zip(xs, ys):
            assert u.dtype == torch.float32 and rel_fro(u, v) < 1e-3
    assert b1.grad.dtype == BF and rel_fro(b1.grad.float(), b2.grad) < 5e-2
    for u, v in zip(lsb[2:], lsf[2:]):                   # BundleResize reads levels 2 and 3
        assert u.grad.dtype == BF and rel_fro(u.grad.float(), v.grad) < 5e-2


@gpu
def test_keyframe_forms_reject_a_bf16_basis():
    from banet_b200 import ops
    _lib.require_device()
    nw, nf, N, C, K = 1, 2, 64, 8, 4
    z = lambda *s, dt=torch.float32: torch.zeros(*s, device="cuda", dtype=dt)
    kl = ops.KeyframeLevel(z(nw, N, C), z(nw * nf, 8, 8, C), z(nw * nf, 4), z(nw, 3, N), z(nw, N, 1), z(nw, N, K, dt=BF))
    with pytest.raises(_lib.BanetError, match="B"):
        kl.as_struct()
    net = _net(C, ("3",)).eval()
    with pytest.raises(RuntimeError, match="basis"):
        net.WindowIteration(z(nw, N, C), z(nw, nf, 8, 8, C), *[z(nw, 1, 1)] * 4, z(nw, 3, N), z(nw, N, 1), z(nw, N, K, dt=BF),
                            torch.eye(3, device="cuda").repeat(nw, nf, 1, 1), z(nw, nf, 3, 1), z(nw, K, 1), 1000.0, "3")


@gpu
def test_resize_host_solver_keeps_a_bf16_basis():
    """A bf16 host basis stays bf16 on the device (2 bytes per element over PCIe), is sampled by banet_resample_bf16 and solves like the
    device-level lm_run on the same bf16 levels (the tolerances of the bf16 pyramid test)."""
    from banet_b200 import ops, synth
    from banet_b200.host_pipeline import ResizeHostSolver
    _lib.require_device()
    nimg, C, K = 8, 64, 128
    sc = synth.make_resize_scene(nimg, 96, 128, C, K, level_ids=(2, 3), seed=41, device="cuda")
    lb = [l.to(BF) for l in sc.layers]
    basis = sc.basis.to(BF)
    pin = lambda t: t.cpu().pin_memory()
    hs = ResizeHostSolver([pin(l) for l in lb], pin(basis), pin(sc.init_depth), pin(sc.intr), sc.scales, chunks=4, precision=0)
    assert hs.d_basis.dtype == BF
    assert hs.h2d_bytes == 2 * (sum(l.numel() for l in lb) + basis.numel()) + 4 * (sc.init_depth.numel() + sc.intr.numel())
    R, T, W, st = hs.solve(pin(sc.R0), pin(sc.T0), pin(sc.W0), 4, lambda_fixed=0.5)
    torch.cuda.synchronize()
    assert int(st.abs().max()) == 0
    half = nimg // 2
    levels = []
    for lay, s in zip(lb, sc.scales):
        h, w = lay.shape[1], lay.shape[2]
        vv, uu = torch.meshgrid(torch.arange(h, device="cuda", dtype=torch.float32), torch.arange(w, device="cuda", dtype=torch.float32), indexing="ij")
        pts = torch.stack([uu.reshape(-1), vv.reshape(-1)], -1).unsqueeze(0).repeat(nimg, 1, 1).contiguous()
        intr_l = sc.intr / s
        B = ops.resample(basis, pts, s / 2.0)
        assert B.dtype == BF
        levels.append(ops.Level(lay.reshape(nimg, h * w, C), torch.cat([lay[half:], lay[:half]], 0).contiguous(), intr_l,
                                ops.compute_coordinates(pts, intr_l, True), ops.resample(sc.init_depth, pts, s / 2.0), B, grid=(w, h)))
    R1, T1, W1, st1 = ops.lm_run(levels, 4, sc.R0, sc.T0, sc.W0, lambda_fixed=0.5, precision=0)
    assert rel_fro(R, R1) < 2e-5 and rel_fro(T, T1) < 1e-3 and rel_fro(W, W1) < 5e-3
