"""Keyframe-layout window batches (banet_lm_keyframe_*, ops.KeyframeLevel, the rank-3 keyframe form of window_batch_iteration_fused and
BundleNet.WindowIteration): the keyframe tensors once per window, the window-reduced per-pair system (frame 0 carries the window's whole depth
block, the other frames' depth blocks are zero).  On the GPU the new build is compared with the per-pair build on the replicated layout and with
the float64 oracle, the window steps and the run with their replicated-layout results, the gradients with the float64 oracle's autograd and the
replicated path's frame sums."""
import ctypes

import pytest
import torch

from helpers import O, scene_case, oracle_level_inputs, mlp_for, rel_fro, to_cuda32


def _opts(**kw):
    from banet_b200._lib import BanetSolveOpts
    return BanetSolveOpts(kw.get("eps", 1e-5), kw.get("undamped_last", 1), kw.get("scramble", 0))


def _klevel(nw=2, nf=4, N=4096, C=64, K=128, h=120, w=160, c2=None, ptr=1):
    from banet_b200 import _lib
    return _lib.BanetKeyframeLevel(nw, nf, N, C, K, h, w, 3 * C if c2 is None else c2, ptr, ptr, ptr, ptr, ptr, ptr)


# ------------------------------------------------------------------------------------------ CPU
def test_keyframe_entries_reject_bad_arguments_without_gpu():
    from banet_b200 import _lib
    lib = _lib.load()
    p = 1                                                            # non-null dummy pointers: every check below fires before a CUDA call
    fwd = lambda lv, R=p, ws=p, nbytes=1 << 34: lib.banet_lm_keyframe_build(ctypes.byref(lv), R, p, p, p, p, p, p, ws, nbytes, None)
    bwd = lambda lv, R=p: lib.banet_lm_keyframe_build_bwd(ctypes.byref(lv), R, p, p, p, p, p, 0, p, p, p, p, p, p, p, None)

    def run(lv, o=None, prec=0, R=p, ws=p, nbytes=1 << 34, lambda_fixed=0.5):
        arr = (_lib.BanetKeyframeLevel * 1)(lv)
        return lib.banet_lm_keyframe_run(arr, 1, 1, None, 1000.0, lambda_fixed, ctypes.byref(o or _opts()), prec, R, p, p, p, ws, nbytes, None)

    for call in (fwd, bwd, run):
        assert call(_klevel(), R=None) == -1 and b"null" in lib.banet_last_error()
        assert call(_klevel(ptr=None)) == -1 and b"null" in lib.banet_last_error()
        for bad in (dict(nw=0), dict(nf=0), dict(N=0), dict(C=0), dict(K=0), dict(h=1), dict(c2=100)):
            assert call(_klevel(**bad)) == -1, bad
        assert call(_klevel(K=257)) == -4 and b"K=257" in lib.banet_last_error()
        assert call(_klevel(C=4096)) == -4
    assert bwd(_klevel(c2=64)) == -4 and b"3C" in lib.banet_last_error()                      # F2-only conv2 in the backward
    assert bwd(_klevel(K=256, C=128)) == -4 and b"shared memory" in lib.banet_last_error()     # S_dd of K = 256 does not fit
    assert run(_klevel(), o=_opts(scramble=1)) == -1
    assert run(_klevel(), lambda_fixed=-1.0) == -1                                             # no MLP and no fixed lambda
    for prec in (1, 2, 3, 4):
        assert run(_klevel(), prec=prec) == -4 and b"keyframe build" in lib.banet_last_error()
    assert run(_klevel(), prec=9) == -1
    for call in (fwd, run):
        assert call(_klevel(), ws=None) == -2 and call(_klevel(), nbytes=16) == -2

    ws = lambda lv: lib.banet_lm_keyframe_build_workspace_bytes(ctypes.byref(lv))
    assert ws(_klevel()) > 0 and ws(_klevel(nf=16)) > ws(_klevel(nf=4))
    for bad in (dict(nw=0), dict(nf=0), dict(K=0), dict(K=257), dict(c2=100)):
        assert ws(_klevel(**bad)) == 0, bad
    rws = lambda lvs, prec=0: lib.banet_lm_keyframe_run_workspace_bytes((_lib.BanetKeyframeLevel * len(lvs))(*lvs), len(lvs), prec)
    assert rws([_klevel()]) > 0 and rws([_klevel(), _klevel(N=1024, h=60, w=80)]) > 0 and rws([_klevel()], -1) == rws([_klevel()], 0)
    assert rws([_klevel()], 1) == 0 and rws([_klevel(K=0)]) == 0 and rws([_klevel(), _klevel(nf=3)]) == 0


class _StructLevel:
    """A level that is only its C struct (dummy device pointers), for the wrappers' argument path on the CPU."""
    def __init__(self, st):
        self.st = st

    def as_struct(self):
        return self.st, []


def test_run_wrappers_report_the_library_message_without_gpu(monkeypatch):
    """The whole-solve wrappers raise BanetError with the library's own message: a rejected keyframe run reaches banet_lm_keyframe_run (its
    workspace query sets no message for levels that disagree), a bad nw of a window batch is BANET_ERR_BAD_ARG.  CPU tensors stand in for
    the device tensors; every call fails in the library before any CUDA call."""
    from banet_b200 import ops, _lib
    monkeypatch.setattr(ops, "_chk", lambda t, name, shape=None, features=False: t)
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    z = torch.zeros
    key = [_StructLevel(_klevel(nw=2, nf=4, K=16)), _StructLevel(_klevel(nw=2, nf=2, K=16))]
    with pytest.raises(_lib.BanetError, match=r"banet_lm_keyframe_run failed \(code -1\): lm_keyframe_run: nw/nf/K must agree across levels"):
        ops.lm_keyframe_run(key, 1, z(8, 3, 3), z(8, 3, 1), z(2, 16, 1), lambda_fixed=0.5)
    with pytest.raises(_lib.BanetError, match=r"banet_lm_keyframe_run failed \(code -4\): lm_keyframe_run: precision mode 1 \(tensor cores\)"):
        ops.lm_keyframe_run(key[:1], 1, z(8, 3, 3), z(8, 3, 1), z(2, 16, 1), lambda_fixed=0.5, precision=_lib.PREC_TF32X1)
    pair = [_StructLevel(_lib.BanetLevel(4, 4096, 64, 16, 48, 64, 192, 1, 1, 1, 1, 1, 1, 0, 0))]
    with pytest.raises(_lib.BanetError, match=r"banet_lm_window_batch_run_workspace_bytes failed \(code -1\)"):
        ops.lm_window_batch_run(pair, 3, 1, z(4, 3, 3), z(4, 3, 1), z(3, 16, 1), lambda_fixed=0.5)
    with pytest.raises(_lib.BanetError, match=r"banet_lm_run_workspace_bytes failed \(code -4\): unknown precision mode 9"):
        ops.lm_run(pair, 1, z(4, 3, 3), z(4, 3, 1), z(4, 16, 1), lambda_fixed=0.5, precision=9)


# ------------------------------------------------------------------------------------------ GPU
def _scene(nw, nf, C, K, n_points, seed=83, dtype=torch.float32, level_ids=None, H=120, W=160):
    """Sparse: n_points keyframe points on the 120 x 160 map of level 3; dense (n_points None): the 60 x 80 grid of level 2."""
    level_ids = level_ids or ((3,) if n_points else (2,))
    return scene_case(nb=nw * nf, H=H, W=W, C=C, K=K, level_ids=level_ids, seed=seed, n_points=n_points, shared_depth=True,
                      window_frames=nf, dtype=dtype)


def _key_levels(sc, nw, nf):
    """Frame 0's keyframe tensors ([:, 0]) once per window, and the same tensors replicated per pair."""
    from banet_b200 import ops
    key, rep = [], []
    for l in sc.levels:
        k = lambda t: to_cuda32(t.reshape(nw, nf, *t.shape[1:])[:, 0])
        kl = ops.KeyframeLevel(k(l.conv1), to_cuda32(l.conv2), to_cuda32(l.intr), k(l.p), k(l.D), k(l.B))
        r = lambda t: t.repeat_interleave(nf, 0).contiguous()
        key.append(kl)
        rep.append(ops.Level(r(kl.conv1), kl.conv2, kl.intr, r(kl.p), r(kl.D), r(kl.B)))
    return key, rep


def _start(sc, nw, nf, K):
    W = to_cuda32(sc.W0.reshape(nw, nf, K, 1)[:, 0]) + 0.01 * torch.arange(1, nw + 1, device="cuda").reshape(nw, 1, 1)
    return to_cuda32(sc.R0), to_cuda32(sc.T0), W.contiguous()


def _depth_mask(nb, P):
    m = torch.ones(nb, P, P, device="cuda")
    m[:, 6:, 6:] = 0
    return m


BUILD_CASES = [(2, 4, 8, 16, 4096), (2, 1, 128, 128, 4096), (2, 16, 8, 16, None), (2, 4, 128, 256, 4096), (1, 16, 128, 128, None),
               (2, 4, 8, 128, None)]


@pytest.mark.gpu
@pytest.mark.parametrize("nw,nf,C,K,n_points", BUILD_CASES)
def test_keyframe_build_is_the_window_reduced_per_pair_build(nw, nf, C, K, n_points):
    from banet_b200 import ops, _lib
    _lib.require_device()
    sc = _scene(nw, nf, C, K, n_points)
    (key,), (rep,) = _key_levels(sc, nw, nf)
    R, T, W = _start(sc, nw, nf, K)
    nb, P = nw * nf, 6 + K
    H, g, rb, nv = ops.lm_keyframe_build(key, R, T, W)
    Hr, gr, rbr, nvr = ops.lm_build(rep, R, T, W.repeat_interleave(nf, 0).contiguous(), _lib.PREC_FP32_SIMT)
    assert torch.equal(H, H.transpose(1, 2))
    dd, ddr = H.reshape(nw, nf, P, P)[:, :, 6:, 6:], Hr.reshape(nw, nf, P, P)[:, :, 6:, 6:]
    assert not bool(dd[:, 1:].any())
    m = _depth_mask(nb, P)
    e = (rel_fro(dd[:, 0], ddr.sum(1)), rel_fro(H * m, Hr * m), rel_fro(g, gr), rel_fro(rb, rbr))
    print(f"nw={nw} nf={nf} C={C} K={K} N={n_points}: vs per-pair build  Hdd {e[0]:.1e} rest of H {e[1]:.1e} g {e[2]:.1e} rbar {e[3]:.1e}")
    assert max(e) < 1e-5 and torch.equal(nv, nvr)
    # float64 oracle, per pair on the replicated keyframe, depth blocks summed over the frames
    f64 = torch.float64
    l = sc.levels[0]
    a = oracle_level_inputs(l)
    rp = lambda t: t.to(f64).reshape(nw, nf, *t.shape[1:])[:, :1].expand(nw, nf, *t.shape[1:]).reshape(t.shape)
    oH, og, orb, onv = O.normal_equations_structured(rp(a["conv1"]), a["conv2"], a["fx"], a["fy"], a["ox"], a["oy"], rp(a["p"]), rp(a["D"]), rp(a["B"]),
                                                     sc.R0.to(f64), sc.T0.to(f64), W.double().cpu().repeat_interleave(nf, 0))
    oH = oH.reshape(nw, nf, P, P)
    mc = m.cpu().double()
    eo = (rel_fro(dd[:, 0], oH[:, :, 6:, 6:].sum(1)), rel_fro(H.cpu().double() * mc, oH.reshape(nb, P, P) * mc), rel_fro(g, og.reshape(nb, P)),
          rel_fro(rb / key.conv1.shape[1], orb.reshape(nb, -1)))                   # the oracle's rbar is the mean over the N points
    print(f"  vs float64 oracle  Hdd {eo[0]:.1e} rest of H {eo[1]:.1e} g {eo[2]:.1e} rbar {eo[3]:.1e}")
    assert max(eo) < 1e-5 and torch.equal(nv.cpu().double(), onv.reshape(nb))


@pytest.mark.gpu
@pytest.mark.parametrize("nf,C,K", [(4, 8, 16), (3, 128, 128)])
def test_keyframe_build_f2_only_layout_agrees_with_3c(nf, C, K):
    from banet_b200 import ops, _lib
    _lib.require_device()
    nw = 2
    sc = _scene(nw, nf, C, K, 4096)
    (key,), _ = _key_levels(sc, nw, nf)
    R, T, W = _start(sc, nw, nf, K)
    f2 = key.conv2[..., :C].contiguous()
    a = ops.lm_keyframe_build(ops.KeyframeLevel(key.conv1, f2, key.intr, key.p, key.D, key.B), R, T, W)
    b = ops.lm_keyframe_build(ops.KeyframeLevel(key.conv1, ops.grad_fixed_concat(f2), key.intr, key.p, key.D, key.B), R, T, W)
    for x, y in zip(a[:3], b[:3]):
        assert rel_fro(x, y) < 1e-5
    assert torch.equal(a[3], b[3])


@pytest.mark.gpu
@pytest.mark.parametrize("nw,nf,C,K", [(3, 4, 8, 16), (2, 16, 128, 128), (1, 4, 32, 128)])
def test_window_steps_take_the_reduced_layout(nw, nf, C, K):
    from banet_b200 import ops, _lib
    _lib.require_device()
    sc = _scene(nw, nf, C, K, 4096)
    (key,), (rep,) = _key_levels(sc, nw, nf)
    R, T, W = _start(sc, nw, nf, K)
    H, g, _, _ = ops.lm_keyframe_build(key, R, T, W)
    Hr, gr, _, _ = ops.lm_build(rep, R, T, W.repeat_interleave(nf, 0).contiguous(), _lib.PREC_FP32_SIMT)
    lam = torch.linspace(0.3, 0.6, nw, device="cuda")
    a = ops.lm_window_batch_solve_update(H, g, lam, R, T, W)
    b = ops.lm_window_batch_solve_update(Hr, gr, lam, R, T, W)
    assert int(a[4].abs().max()) == 0 and int(b[4].abs().max()) == 0
    e = [rel_fro(x, y) for x, y in zip(a[:4], b[:4])]
    print(f"batch step, reduced vs replicated layout: R' {e[0]:.1e} T' {e[1]:.1e} W' {e[2]:.1e} delta {e[3]:.1e}")
    assert max(e) < 1e-5
    if nw == 1:                                                      # the single-window (3c) step too
        c = ops.lm_window_solve_update(H, g, lam, R, T, W[0])
        d = ops.lm_window_solve_update(Hr, gr, lam, R, T, W[0])
        e = [rel_fro(x, y) for x, y in zip(c[:4], d[:4])]
        print(f"single-window step, reduced vs replicated layout: " + " ".join(f"{v:.1e}" for v in e))
        assert max(e) < 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("nw,nf,C,K", [(2, 3, 16, 16), (2, 4, 128, 128)])
def test_keyframe_run_matches_the_oracle_and_the_replicated_run(nw, nf, C, K):
    from banet_b200 import ops, _lib
    _lib.require_device()
    iters = 3
    sc = _scene(nw, nf, C, K, None, seed=41, dtype=torch.float64, level_ids=(2, 3), H=96, W=128)
    key, rep = _key_levels(sc, nw, nf)
    mlps = [mlp_for(C, l.level) for l in sc.levels]
    oR, oT, oW = [], [], []
    for w in range(nw):
        s = slice(w * nf, (w + 1) * nf)
        olv = []
        for l, m in zip(sc.levels, mlps):
            a = oracle_level_inputs(l)
            kf = lambda t: t[w * nf:w * nf + 1].expand(nf, *t.shape[1:])
            olv.append(O.LevelInputs(kf(a["conv1"]), a["conv2"][s], a["fx"][s], a["fy"][s], a["ox"][s], a["oy"][s], kf(a["p"]), kf(a["D"]), kf(a["B"]), m))
        r = O.window_solve(olv, iters, sc.R0[s], sc.T0[s], sc.W0[w * nf])
        oR.append(r[0]); oT.append(r[1]); oW.append(r[2])
    oR, oT, oW = torch.cat(oR), torch.cat(oT), torch.stack(oW)
    packed = [ops.pack_mlp([(w.float(), b.float()) for w, b in m]).cuda() for m in mlps]
    R0, T0 = to_cuda32(sc.R0), to_cuda32(sc.T0)
    W0 = to_cuda32(sc.W0.reshape(nw, nf, K, 1)[:, 0])
    R, T, Wn, st = ops.lm_keyframe_run(key, iters, R0, T0, W0, mlp_packed=packed, l2_regularizer_base=1000.0)
    assert int(st.abs().max()) == 0
    e = (rel_fro(R, oR), rel_fro(T, oT), rel_fro(Wn, oW))
    print(f"keyframe run nw={nw} nf={nf} C={C} K={K} vs oracle: R {e[0]:.1e} T {e[1]:.1e} W {e[2]:.1e}")
    assert e[0] < 1e-5 and e[1] < 1e-4 and e[2] < 2e-4
    Rr, Tr, Wr, str_ = ops.lm_window_batch_run(rep, nw, iters, R0, T0, W0, mlp_packed=packed, l2_regularizer_base=1000.0,
                                               precision=_lib.PREC_FP32_SIMT)
    er = (rel_fro(R, Rr), rel_fro(T, Tr), rel_fro(Wn, Wr))
    print(f"  vs lm_window_batch_run on the replicated layout: R {er[0]:.1e} T {er[1]:.1e} W {er[2]:.1e}")
    assert max(er) < 1e-4 and torch.equal(st, str_)


@pytest.mark.gpu
@pytest.mark.parametrize("nf,C,K", [(3, 16, 16), (4, 128, 128)])
def test_one_keyframe_run_iteration_is_the_build_plus_the_batch_step(nf, C, K):
    from banet_b200 import ops, _lib
    _lib.require_device()
    nw = 2
    sc = _scene(nw, nf, C, K, 4096)
    (key,), _ = _key_levels(sc, nw, nf)
    R, T, W = _start(sc, nw, nf, K)
    H, g, _, _ = ops.lm_keyframe_build(key, R, T, W)
    lam = torch.full((nw,), 0.5, device="cuda")
    Rn, Tn, Wn, _, status = ops.lm_window_batch_solve_update(H, g, lam, R, T, W)
    R2, T2, W2, status2 = ops.lm_keyframe_run([key], 1, R, T, W, lambda_fixed=0.5, precision=_lib.PREC_FP32_SIMT)
    assert int(status.abs().max()) == 0
    assert torch.equal(Rn, R2) and torch.equal(Tn, T2) and torch.equal(Wn, W2) and torch.equal(status, status2)


@pytest.mark.gpu
def test_keyframe_build_and_run_are_reproducible_and_ignore_the_workspace():
    from banet_b200 import ops, _lib
    _lib.require_device()
    lib = _lib.load()
    nw, nf, C, K = 3, 4, 32, 128
    sc = _scene(nw, nf, C, K, 4096)
    (key,), _ = _key_levels(sc, nw, nf)
    R, T, W = _start(sc, nw, nf, K)
    st, _keep = key.as_struct()
    P, nb = 6 + K, nw * nf
    packed = [ops.pack_mlp(mlp_for(C, 3, torch.float32)).cuda()]
    outs = []
    for fill in ("nan", "random", "nan"):
        nbytes = lib.banet_lm_keyframe_build_workspace_bytes(ctypes.byref(st))
        ws = torch.empty(nbytes // 4 + 1, device="cuda")
        ws.fill_(float("nan")) if fill == "nan" else ws.uniform_(-1e3, 1e3)
        o = [torch.empty(nb, P, P, device="cuda"), torch.empty(nb, P, device="cuda"), torch.empty(nb, C, device="cuda"), torch.empty(nb, device="cuda")]
        _lib.check(lib.banet_lm_keyframe_build(ctypes.byref(st), R.data_ptr(), T.data_ptr(), W.data_ptr(), *[x.data_ptr() for x in o], ws.data_ptr(),
                                               ws.numel() * 4, ops._stream()), "banet_lm_keyframe_build")
        rws = torch.empty(lib.banet_lm_keyframe_run_workspace_bytes((_lib.BanetKeyframeLevel * 1)(st), 1, 0) // 4 + 1, device="cuda")
        rws.fill_(float("nan")) if fill == "nan" else rws.uniform_(-1e3, 1e3)
        r = ops.lm_keyframe_run([key], 2, R, T, W, mlp_packed=packed, workspace=rws)
        outs.append(o + list(r))
    assert int(outs[0][-1].abs().max()) == 0
    for other in outs[1:]:
        for x, y in zip(outs[0], other):
            assert torch.equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize("exact_sym", [True, False])
def test_keyframe_backward_reads_frame_0s_depth_block_and_is_the_per_pair_backward_summed(exact_sym):
    from banet_b200 import ops, _lib
    _lib.require_device()
    nw, nf, C, K = 2, 4, 32, 128
    sc = _scene(nw, nf, C, K, 4096)
    (key,), (rep,) = _key_levels(sc, nw, nf)
    R, T, W = _start(sc, nw, nf, K)
    nb, P = nw * nf, 6 + K
    gen = torch.Generator(device="cuda").manual_seed(21)
    dH = 1e-3 * torch.randn(nb, P, P, generator=gen, device="cuda")
    dg = 1e-3 * torch.randn(nb, P, generator=gen, device="cuda"); dr = 1e-3 * torch.randn(nb, C, generator=gen, device="cuda")
    a = ops.lm_keyframe_build_bwd(key, R, T, W, dH, dg, dr, exact_sym)
    b = ops.lm_keyframe_build_bwd(key, R, T, W, dH, dg, dr, exact_sym)
    for i in (0, 2, 3):                                             # dconv1, dD, dB: no atomics, bit-reproducible
        assert torch.equal(a[i], b[i])
    junk = dH.clone().reshape(nw, nf, P, P)
    junk[:, 1:, 6:, 6:] = 7.0 * torch.randn(nw, nf - 1, K, K, generator=gen, device="cuda")
    c = ops.lm_keyframe_build_bwd(key, R, T, W, junk.reshape(nb, P, P), dg, dr, exact_sym)
    for x, y in zip((a[0], a[2], a[3]), (c[0], c[2], c[3])):
        assert torch.equal(x, y)
    for x, y in zip((a[1], a[4], a[5], a[6]), (c[1], c[4], c[5], c[6])):
        assert rel_fro(x, y) < 1e-6
    # the per-pair backward on the replicated layout with frame 0's depth block in every frame, summed over the frames
    rH = dH.clone().reshape(nw, nf, P, P)
    rH[:, :, 6:, 6:] = rH[:, :1, 6:, 6:]
    r = ops.lm_build_bwd(rep, R, T, W.repeat_interleave(nf, 0).contiguous(), rH.reshape(nb, P, P), dg, dr, exact_sym)
    fsum = lambda t: t.reshape(nw, nf, *t.shape[1:]).sum(1)
    e = (rel_fro(a[0], fsum(r[0])), rel_fro(a[1], r[1]), rel_fro(a[2], fsum(r[2])), rel_fro(a[3], fsum(r[3])), rel_fro(a[4], r[4]),
         rel_fro(a[5], r[5]), rel_fro(a[6], fsum(r[6])))
    print("keyframe backward vs per-pair backward summed: " + " ".join(f"{n} {v:.1e}" for n, v in zip(("conv1", "conv2", "D", "B", "R", "T", "W"), e)))
    assert max(e) < 1e-5


def _grad_inputs(nw, nf, C, K, n_points, seed):
    sc = _scene(nw, nf, C, K, n_points, seed=seed, dtype=torch.float64)
    lv = sc.levels[0]
    a = oracle_level_inputs(lv)
    W = sc.W0.reshape(nw, nf, K, 1)[:, 0].double() + 0.01 * torch.randn(nw, K, 1, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    g = torch.Generator().manual_seed(5)
    c = (torch.randn(nw * nf, 3, 3, generator=g, dtype=torch.float64), torch.randn(nw * nf, 3, 1, generator=g, dtype=torch.float64),
         torch.randn(nw, K, 1, generator=g, dtype=torch.float64))
    return sc, lv, a, W, c


def _keyframe_call(lv, a, sc, W, nw, nf, mlp, lam, exact_sym, once=True):
    """window_batch_iteration_fused on float32 CUDA copies: the keyframe form (once) or the per-frame replicated form; returns outputs and
    leaves."""
    from banet_b200 import autograd as ag
    key = ("conv1", "D", "B")
    kf = lambda t: to_cuda32(t.reshape(nw, nf, *t.shape[1:])[:, 0])
    t = {n: (kf(a[n]) if once else kf(a[n]).unsqueeze(1).repeat(1, nf, *[1] * (a[n].dim() - 1))).requires_grad_() for n in key}
    t["conv2"] = to_cuda32(a["conv2"]).reshape(nw, nf, *a["conv2"].shape[1:]).requires_grad_()
    Rg = to_cuda32(sc.R0).reshape(nw, nf, 3, 3).requires_grad_(); Tg = to_cuda32(sc.T0).reshape(nw, nf, 3, 1).requires_grad_()
    Wg = to_cuda32(W).requires_grad_()
    p = kf(lv.p) if once else kf(lv.p).unsqueeze(1).repeat(1, nf, 1, 1)
    intr = to_cuda32(lv.intr).reshape(nw, nf, 4)
    out = ag.window_batch_iteration_fused(t["conv1"], t["conv2"], intr, p, t["D"], t["B"], Rg, Tg, Wg, mlp, 1000.0, exact_sym=exact_sym,
                                          lambda_override=lam, return_status=True)
    t.update(R=Rg, T=Tg, W=Wg)
    return out, t


@pytest.mark.gpu
@pytest.mark.parametrize("nw,nf,C,K,n_points,fixed_lambda", [(2, 3, 8, 5, 400, None), (2, 3, 128, 128, 4096, 0.4)])
def test_keyframe_gradients_match_oracle_autograd_and_the_replicated_path(nw, nf, C, K, n_points, fixed_lambda):
    from banet_b200 import _lib
    _lib.require_device()
    sc, lv, a, W, (cR, cT, cW) = _grad_inputs(nw, nf, C, K, n_points, seed=71)
    names = ["conv1", "conv2", "D", "B"]
    kf64 = lambda t: t.reshape(nw, nf, *t.shape[1:])[:, 0].clone().requires_grad_()
    o = {n: kf64(a[n]) for n in ("conv1", "D", "B")}
    o["conv2"] = a["conv2"].clone().requires_grad_()
    R = sc.R0.double().clone().requires_grad_(); T = sc.T0.double().clone().requires_grad_(); W64 = W.clone().requires_grad_()
    mlp64 = [] if fixed_lambda is not None else [(w.clone().requires_grad_(), b.clone().requires_grad_()) for w, b in mlp_for(C, 3)]
    oR, oT, oW = [], [], []
    for w in range(nw):
        s = slice(w * nf, (w + 1) * nf)
        ex = lambda t: t[w:w + 1].expand(nf, *t.shape[1:])
        p_key = a["p"].reshape(nw, nf, *a["p"].shape[1:])[w, :1].expand(nf, *a["p"].shape[1:])
        lam = None if fixed_lambda is None else torch.tensor([fixed_lambda], dtype=torch.float64)
        r = O.window_iteration(ex(o["conv1"]), o["conv2"][s], a["fx"][s], a["fy"][s], a["ox"][s], a["oy"][s], p_key, ex(o["D"]), ex(o["B"]),
                               R[s], T[s], W64[w], mlp64, O.IterOptions(l2_regularizer_base=1000.0, guard_nonfinite=True, lambda_override=lam))
        oR.append(r[0]); oT.append(r[1]); oW.append(r[2])
    oR, oT, oW = torch.cat(oR), torch.cat(oT), torch.stack(oW)
    ((oR * cR).sum() + (oT * cT).sum() + (oW * cW).sum()).backward()
    lam32 = None if fixed_lambda is None else torch.full((nw,), fixed_lambda, device="cuda")
    res = {}
    for exact_sym in (True, False):
        for once in (True, False):
            mlp32 = [(to_cuda32(w.detach()).requires_grad_(), to_cuda32(b.detach()).requires_grad_()) for w, b in mlp64]
            (gR, gT, gW, status), t = _keyframe_call(lv, a, sc, W, nw, nf, mlp32, lam32, exact_sym, once)
            assert int(status.abs().max()) == 0
            ((gR * to_cuda32(cR).reshape(gR.shape)).sum() + (gT * to_cuda32(cT).reshape(gT.shape)).sum() + (gW * to_cuda32(cW)).sum()).backward()
            res[(exact_sym, once)] = ((gR, gT, gW), t, mlp32)
    (gR, gT, gW), t, mlp32 = res[(True, True)]
    e = (rel_fro(gR.reshape(oR.shape), oR), rel_fro(gT.reshape(oT.shape), oT), rel_fro(gW, oW))
    print(f"keyframe nw={nw} nf={nf} C={C} K={K}: outputs R {e[0]:.1e} T {e[1]:.1e} W {e[2]:.1e}")
    assert e[0] < 1e-5 and e[1] < 1e-4 and e[2] < 1e-3
    for nm, x, y in [(n, t[n], o[n]) for n in names] + [("R", t["R"], R), ("T", t["T"], T), ("W", t["W"], W64)]:
        err = rel_fro(x.grad.reshape(y.grad.shape), y.grad)
        print(f"grad {nm} vs oracle: {err:.2e}")
        assert err < 2e-3, nm
    for i, ((w32, _), (w64, _)) in enumerate(zip(mlp32, mlp64)):
        assert rel_fro(w32.grad, w64.grad) < 2e-3, i
    for exact_sym in (True, False):                                 # against the replicated path's frame-summed gradients
        (ko, kt, km), (ro, rt, rm) = res[(exact_sym, True)], res[(exact_sym, False)]
        for x, y in zip(ko, ro):
            assert rel_fro(x, y) < 1e-5
        for n in ("conv1", "D", "B"):
            err = rel_fro(kt[n].grad, rt[n].grad.sum(1))
            print(f"exact_sym={exact_sym} grad {n} vs replicated frame sum: {err:.1e}")
            assert err < 1e-5, n
        for n in ("conv2", "R", "T", "W"):
            assert rel_fro(kt[n].grad, rt[n].grad) < 1e-5, n
        for (w1, _), (w2, _) in zip(km, rm):
            assert rel_fro(w1.grad, w2.grad) < 1e-5


@pytest.mark.gpu
def test_a_skipped_keyframe_window_stays_contained():
    from banet_b200 import ops, _lib
    _lib.require_device()
    nw, nf, C, K = 3, 3, 8, 5
    sc = _scene(nw, nf, C, K, 400, seed=13)
    (key,), _ = _key_levels(sc, nw, nf)
    R, T, W = _start(sc, nw, nf, K)
    bad = ops.KeyframeLevel(key.conv1.clone(), key.conv2, key.intr, key.p, key.D, key.B)
    bad.conv1[1, 3, 0] = float("nan")                                # window 1's keyframe
    packed = [ops.pack_mlp(mlp_for(C, 3, torch.float32)).cuda()]
    a = ops.lm_keyframe_run([key], 2, R, T, W, mlp_packed=packed)
    b = ops.lm_keyframe_run([bad], 2, R, T, W, mlp_packed=packed)
    st = b[3].reshape(nw, nf)
    assert bool((st[1] != 0).all()) and int(st[0].abs().max()) == 0 and int(st[2].abs().max()) == 0
    ok = [0, 1, 2, 2 * nf, 2 * nf + 1, 2 * nf + 2]
    assert torch.equal(a[0][ok], b[0][ok]) and torch.equal(a[1][ok], b[1][ok]) and torch.equal(a[2][[0, 2]], b[2][[0, 2]])
    assert torch.equal(b[2][1], W[1])
    # one differentiable iteration: the other windows' values and keyframe gradients are those without the NaN
    from banet_b200 import autograd as ag
    lam = torch.full((nw,), 0.5, device="cuda")
    res = []
    for lv in (key, bad):
        t = {n: getattr(lv, n).clone().requires_grad_() for n in ("conv1", "D", "B")}
        Rg, Tg, Wg = R.reshape(nw, nf, 3, 3).clone().requires_grad_(), T.reshape(nw, nf, 3, 1).clone().requires_grad_(), W.clone().requires_grad_()
        Rn, Tn, Wn, status = ag.window_batch_iteration_fused(t["conv1"], lv.conv2.reshape(nw, nf, *lv.conv2.shape[1:]), lv.intr.reshape(nw, nf, 4),
                                                             lv.p, t["D"], t["B"], Rg, Tg, Wg, [], 1000.0, lambda_override=lam, return_status=True)
        (Rn.sum() + Tn.sum() + Wn.sum()).backward()
        res.append((Rn, Tn, Wn, status, t, Rg, Tg, Wg))
    (Ra, Ta, Wa, sa, ta, Rga, Tga, Wga), (Rb, Tb, Wb, sb, tb, Rgb, Tgb, Wgb) = res
    assert bool((sb[1] != 0).all()) and int(sb[[0, 2]].abs().max()) == 0
    for w in (0, 2):
        assert torch.equal(Ra[w], Rb[w]) and torch.equal(Ta[w], Tb[w]) and torch.equal(Wa[w], Wb[w])
        for n in ("conv1", "D", "B"):
            assert torch.equal(ta[n].grad[w], tb[n].grad[w]), n
        assert rel_fro(Rgb.grad[w], Rga.grad[w]) < 1e-6 and rel_fro(Wgb.grad[w], Wga.grad[w]) < 1e-6


@pytest.mark.gpu
def test_keyframe_form_does_not_replicate_the_keyframe():
    from banet_b200 import _lib
    _lib.require_device()
    nw, nf, C, K, N = 2, 16, 128, 128, 4096
    sc = _scene(nw, nf, C, K, N, seed=7, level_ids=(0,))             # a 15 x 20 map: the basis, not conv2, dominates the inputs
    (key,), _ = _key_levels(sc, nw, nf)
    R, T, W = _start(sc, nw, nf, K)
    from banet_b200 import autograd as ag
    lib = _lib.load()
    st, _keep = key.as_struct()
    build_ws = lib.banet_lm_keyframe_build_workspace_bytes(ctypes.byref(st))
    t = {n: getattr(key, n).clone().requires_grad_() for n in ("conv1", "D", "B")}
    conv2 = key.conv2.reshape(nw, nf, *key.conv2.shape[1:]).clone().requires_grad_()
    Rg, Tg, Wg = R.reshape(nw, nf, 3, 3).clone().requires_grad_(), T.reshape(nw, nf, 3, 1).clone().requires_grad_(), W.clone().requires_grad_()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    Rn, Tn, Wn = ag.window_batch_iteration_fused(t["conv1"], conv2, key.intr.reshape(nw, nf, 4), key.p, t["D"], t["B"], Rg, Tg, Wg, [], 1000.0,
                                                 lambda_override=torch.full((nw,), 0.5, device="cuda"))
    (Rn.sum() + Tn.sum() + Wn.sum()).backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    P = 6 + K
    inputs = sum(x.numel() * 4 for x in (t["conv1"], conv2, t["D"], t["B"]))     # one gradient per input
    system = 4 * nw * nf * P * P * 4                                              # H, dH and their transients
    bound = build_ws + inputs + system + (4 << 20)
    replicated = nw * nf * N * K * 4                                              # one [nw*nf,N,K] tensor
    print(f"peak {peak / 2**20:.1f} MiB, bound {bound / 2**20:.1f} MiB, one replicated basis {replicated / 2**20:.1f} MiB")
    assert bound < replicated and peak <= bound


def _net(C, precision=None, strict=True):
    from banet_b200.bundlenet import BundleNet
    from banet_b200 import _lib
    net = BundleNet(C, levels=("3",), exact_sym_grad=True, precision=_lib.PREC_FP32_SIMT if precision is None else precision, strict_status=strict).cuda()
    for i, (w, b) in enumerate(mlp_for(C, 3)):
        getattr(net, f"lambda_3_{i + 1}_filters").data.copy_(w); getattr(net, f"lambda_3_{i + 1}_biases").data.copy_(b)
    return net


def _net_inputs(nw=2, nf=3, C=8, K=5, seed=91):
    sc = _scene(nw, nf, C, K, 500, seed=seed)
    lv = sc.levels[0]
    kf = lambda t: to_cuda32(t).reshape(nw, nf, *t.shape[1:])[:, 0].contiguous()
    fr = lambda t: to_cuda32(t).reshape(nw, nf, *t.shape[1:])
    x = dict(conv1=kf(lv.conv1), conv2=fr(lv.conv2), p=kf(lv.p), D=kf(lv.D), B=kf(lv.B), R=fr(sc.R0), T=fr(sc.T0),
             W=to_cuda32(sc.W0.reshape(nw, nf, K, 1)[:, 0]) + 0.01)
    intr = [fr(t) for t in lv.intr_tiled()]
    return x, intr


def _call(net, d, intr):
    fx, fy, ox, oy = intr
    return net.WindowIteration(d["conv1"], d["conv2"], fx, fy, ox, oy, d["p"], d["D"], d["B"], d["R"], d["T"], d["W"], 1000.0, "3")


@pytest.mark.gpu
def test_keyframe_window_iteration_grad_and_no_grad_paths_agree():
    from banet_b200 import _lib
    _lib.require_device()
    x, intr = _net_inputs()
    net = _net(8, precision=_lib.PREC_AUTO)
    with torch.no_grad():
        a = _call(net, x, intr)
    b = _call(net, {k: v.clone().requires_grad_(k != "p") for k, v in x.items()}, intr)
    assert all(t.requires_grad for t in b) and not any(t.requires_grad for t in a)
    assert tuple(net.last_status.shape) == (2, 3) and int(net.last_status.abs().max()) == 0
    assert tuple(a[0].shape) == (2, 3, 3, 3) and tuple(a[1].shape) == (2, 3, 3, 1) and tuple(a[2].shape) == (2, 5, 1)
    for u, v in zip(a, b):
        assert rel_fro(u, v.detach()) < 1e-5
    # the same windows in the [nw,1,...] broadcast form
    once = {k: (v.unsqueeze(1) if k in ("conv1", "p", "D", "B") else v) for k, v in x.items()}
    with torch.no_grad():
        c = _call(net, once, intr)
    for u, v in zip(a, c):
        assert rel_fro(u, v) < 1e-5


@pytest.mark.gpu
def test_keyframe_window_iteration_strict_status_precision_and_mixed_forms():
    from banet_b200 import _lib
    _lib.require_device()
    x, intr = _net_inputs()
    net = _net(8)
    bad = dict(x); bad["conv1"] = x["conv1"].clone(); bad["conv1"][1, 0, 0] = float("nan")
    with torch.no_grad(), pytest.raises(RuntimeError, match="skipped"):
        _call(net, bad, intr)
    with pytest.raises(RuntimeError, match="skipped"):
        _call(net, {k: v.clone().requires_grad_(k != "p") for k, v in bad.items()}, intr)
    assert bool((net.last_status[1] != 0).all()) and int(net.last_status[0].abs().max()) == 0
    for prec in (_lib.PREC_TF32X1, _lib.PREC_TF32X3, _lib.PREC_TF32_LEVELWISE):
        with torch.no_grad(), pytest.raises(RuntimeError, match="tensor-core"):
            _call(_net(8, precision=prec), x, intr)
    mixed = dict(x); mixed["B"] = x["B"].unsqueeze(1)
    with torch.no_grad(), pytest.raises(RuntimeError, match="frame axis"):
        _call(net, mixed, intr)
