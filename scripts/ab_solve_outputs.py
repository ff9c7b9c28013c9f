"""A/B of the damped solve, its backward and the LM runs against a comparison build of the library (GPU), and interleaved timings.

    python scripts/ab_solve_outputs.py --base /path/to/other/libbanet.so [--rounds 5] [--out result.json]

Outputs: one process loads both libraries (two ctypes handles, as scripts/ab_simt_outputs.py) and runs every seeded case on each, at K = 16, 64,
128, 200 and at the storage edges of lm_step (P = 157, 158, 222, 223, 332) and of the arrow (K = 154, 155, 215, 216):
  * bitwise expected: lm_step with the MLP (C = 128) and with lambda given, lm_run (fixed lambda and MLP), lm_window_run, lm_window_batch_run
    and lm_keyframe_run (MLP), the arrow's solve and its backward, at every size where the storage variant of the comparison build (the
    `previous` rules below) is the one the new build picks;
  * expected to change, reported as the relative distance from a float64 statement (torch) next to the comparison build's: lm_solve_update
    and its backward (pairs; per pair, lambda in {1e-3, 0.1, 10, 0.3}; the backward through W' = W + delta_d), the dense window's backward,
    lm_lambda (against a float64 MLP) and lm_run with vmatrix_batch_scramble (against the other build).
Systems are graded (condition number 1e4 for the solves, 1e3 for the arrow and the timings); runs use a synthetic sparse scene.
Timing (--rounds): in the same process, rounds alternate the two libraries; each times with CUDA events, after three warm-up calls, 20 calls of
lm_solve_update + lm_solve_update_bwd at nb = 32 and K = 128, 64, 32, lm_window_solve_update_bwd at nf = 4 and 16 (K = 128) and lm_lambda at
nb = 32, C = 128.  The report gives median [min - max] per case and library, and the card's name and power limit.
"""
import argparse, json, os, statistics, subprocess, sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)


def previous_step_variant(P, C):
    """The comparison build's lm_step storage: the MLP's buffers (C, 1 with lambda given) beside the matrix."""
    mlp = (8 * C + max(4 * C, 1024)) * 4
    size = lambda full, e: ((P + 1) * ((P + 1) | 1) if full else (P + 1) * (P + 2) // 2) * e + (2 * P + 4) * e + mlp
    if size(True, 8) <= 200 * 1024:
        return "square_fp64"
    if size(False, 8) <= 200 * 1024:
        return "packed_fp64"
    return "packed_fp32" if size(False, 4) <= 220 * 1024 else "rejected"


def previous_arrow_variant(K, C):
    mlp = (8 * C + max(4 * C, 1024)) * 4 if C else 0
    size = lambda full, e: (((K + 1) * ((K + 1) | 1) if full else (K + 1) * (K + 2) // 2) + 9 * K + 4) * e + mlp
    if size(True, 8) <= 200 * 1024:
        return "square_fp64"
    return "packed_fp64" if size(False, 8) <= 200 * 1024 else "packed_fp32"


class Libs:
    def __init__(self, paths):
        from banet_b200 import _lib
        self._mod, self.handles = _lib, {}
        for name, path in paths.items():
            _lib._lib, _lib.LIB_PATH = None, path
            self.handles[name] = _lib.load()

    def run(self, name, fn):
        self._mod._lib = self.handles[name]
        return fn()


# ---- seeded inputs and float64 statements (torch only)
def graded_spd(torch, P, kappa, seed):
    """Q diag(kappa^-t) Q^T, t uniform in [0, 1], rounded to fp32: symmetric positive definite of condition number kappa."""
    gen = torch.Generator().manual_seed(seed)
    Q, _ = torch.linalg.qr(torch.randn(P, P, generator=gen, dtype=torch.float64))
    H = (Q * kappa ** -torch.linspace(0, 1, P, dtype=torch.float64)) @ Q.T
    return ((H + H.T) / 2).float().double()


def randn(torch, shape, seed, scale=1.0):
    return (scale * torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)).float().double()


def iterate(torch, nb, K, seed):
    w = randn(torch, (nb, 3), seed, 0.01)
    sk = torch.zeros(nb, 3, 3, dtype=torch.float64)
    sk[:, 0, 1], sk[:, 0, 2], sk[:, 1, 2] = -w[:, 2], w[:, 1], -w[:, 0]
    R = torch.linalg.matrix_exp(sk - sk.transpose(1, 2)).float().double()
    return R, randn(torch, (nb, 3, 1), seed + 1, 0.1), randn(torch, (nb, K, 1), seed + 2, 0.01)


def damped(torch, H, lam, ndamped, eps=1e-5):
    P = H.shape[-1]
    d = torch.diagonal(H, dim1=-2, dim2=-1)
    return H + torch.diag_embed((d + float(torch.tensor(eps).float())) * lam.reshape(-1, 1) * (torch.arange(P) < ndamped).to(H.dtype))


def assemble(torch, H, g):
    """The joint window system of nf pairs sharing W (the depth blocks summed, rounded to fp32 as the kernel stores them)."""
    nf, P = g.shape
    K, np_ = P - 6, 6 * nf
    Hj = torch.zeros(np_ + K, np_ + K, dtype=H.dtype); gj = torch.zeros(np_ + K, dtype=H.dtype)
    for f in range(nf):
        Hj[6 * f:6 * f + 6, 6 * f:6 * f + 6] = H[f, :6, :6]
        Hj[6 * f:6 * f + 6, np_:] = H[f, :6, 6:]
        Hj[np_:, 6 * f:6 * f + 6] = H[f, 6:, :6]
        gj[6 * f:6 * f + 6] = g[f, :6]
    Hd, gd = H[:, 6:, 6:].sum(0), g[:, 6:].sum(0)
    Hj[np_:, np_:] = Hd + (Hd.detach().float().double() - Hd.detach())
    gj[np_:] = gd + (gd.detach().float().double() - gd.detach())
    return Hj, gj


def mlp_params(torch, C, seed):
    gen, dims = torch.Generator().manual_seed(seed), [C, 2 * C, 4 * C, 2 * C, C, 1]
    return [(torch.randn(dims[i], dims[i + 1], generator=gen) * (1.0 / dims[i]) ** 0.5, 0.01 * torch.randn(dims[i + 1], generator=gen))
            for i in range(5)]


def lambda64(torch, rbar_sum, N, params, base=1000.0):
    """lambda = base ||rbar||^(2 + MLP(rbar)), rbar = rbar_sum / N (bundlenet.py:243-253) in float64."""
    r = rbar_sum.double() / N
    a = r
    for i, (w, b) in enumerate(params):
        a = a @ w.double() + b.double()
        a = torch.tanh(a) if i == 4 else torch.nn.functional.selu(a)
    return base * torch.linalg.norm(r, dim=-1) ** (2.0 + a[:, 0])


def rel(torch, a, b):
    a = torch.as_tensor(a).double().cpu(); b = torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def equal(a, b):
    return a.shape == b.shape and bool(((a == b) | (a.isnan() & b.isnan())).all())


def correctness(libs):
    import torch
    from banet_b200 import ops, synth, _lib
    cu = lambda t: t.to(device="cuda", dtype=torch.float32).contiguous()
    r = lambda a, b: rel(torch, a, b)
    res = {"bitwise": [], "mismatch": [], "changed": []}

    def both(case, names, fn, expect_bitwise):
        a, b = libs.run("base", fn), libs.run("new", fn)
        for name, x, y in zip(names, a, b):
            if x is None:
                continue
            row = f"{case} {name}"
            if equal(x, y):
                res["bitwise"].append(row)
            elif expect_bitwise:
                res["mismatch"].append(f"{row}: max |diff| {float((x.double() - y.double()).abs().max()):.3g}")
        return a, b

    def sym(x):
        x = torch.as_tensor(x).double().cpu()
        return x + x.transpose(-1, -2)

    def new_step_variant(P):
        size = lambda full, e: ((P + 1) * ((P + 1) | 1) if full else (P + 1) * (P + 2) // 2) * e + (2 * P + 4) * e
        if size(True, 8) <= 200 * 1024:
            return "square_fp64"
        return "packed_fp64" if size(False, 8) <= 200 * 1024 else "packed_fp32"

    def new_arrow_variant(K):
        return previous_arrow_variant(K, 0)

    mlp128 = ops.pack_mlp(mlp_params(torch, 128, 3)).cuda()
    for P in sorted({6 + K for K in (16, 64, 128, 200)} | {157, 158, 222, 223, 332}):
        K = P - 6
        H = torch.stack([graded_spd(torch, P, 1e4, P + i) for i in range(4)]); g = randn(torch, (4, P), P)
        R, T, W = iterate(torch, 4, K, P)
        lam = torch.tensor([1e-3, 0.1, 10.0, 0.3], dtype=torch.float32).double()
        rb = (0.02 * (1 + torch.rand(4, 128, generator=torch.Generator().manual_seed(P))) * 4096).float()
        new_v = new_step_variant(P)
        for C, tag in ((128, "mlp"), (1, "lambda given")):
            prev = previous_step_variant(P, C)
            if prev == "rejected":
                continue
            fn = ((lambda: ops.lm_step(cu(H), cu(g), cu(rb), 4096, mlp128, 1000.0, cu(R), cu(T), cu(W))) if tag == "mlp" else
                  (lambda: ops.lm_step(cu(H), cu(g), None, 1, None, 1.0, cu(R), cu(T), cu(W), lam=cu(lam))))
            both(f"lm_step {tag} P={P} ({prev} -> {new_v})", ("R", "T", "W", "delta", "lambda", "status"), fn, prev == new_v)
        # the pair solve and its backward (through W' = W + delta_d, dR' = dT' = 0) against float64 autograd, per lambda, both libraries
        gW = randn(torch, (4, K, 1), P + 7)
        z3, z1 = torch.zeros(4, 3, 3), torch.zeros(4, 3, 1)
        leaves = [t.clone().requires_grad_() for t in (H, g, lam)]
        delta64 = torch.linalg.solve(damped(torch, leaves[0], leaves[2], P - 1), leaves[1].unsqueeze(-1)).squeeze(-1)
        (delta64[:, 6:] * gW.squeeze(-1)).sum().backward()
        row = {"case": f"pairs P={P}", "variant": new_v, "lambda": lam.tolist()}
        for lib in ("base", "new"):
            try:
                f = libs.run(lib, lambda: ops.lm_solve_update(cu(H), cu(g), cu(lam), cu(R), cu(T), cu(W)))
                d = libs.run(lib, lambda: ops.lm_solve_update_bwd(cu(H), cu(g), cu(lam), f[3], cu(R), cu(T), cu(z3), cu(z1), cu(gW)))
            except Exception as e:                                  # a size one of the two rejects
                row[lib] = str(e)[:80]
                continue
            row[lib] = [{"delta": r(f[3][i], delta64[i].detach()), "dH": r(sym(d[0][i]), sym(leaves[0].grad[i])), "dg": r(d[1][i], leaves[1].grad[i]),
                         "dlambda": r(d[2][i], leaves[2].grad[i]), "dW": r(d[5][i], gW[i])} for i in range(4)]
        res["changed"].append(row)
    # the dense window's backward (nf = 2, lambda = 0.1, through W' only) against float64 autograd
    for Pj in (44, 140, 157, 158, 222, 223, 332):
        K = Pj - 12
        H = torch.stack([graded_spd(torch, 6 + K, 1e4, Pj + f) for f in range(2)]); g = randn(torch, (2, 6 + K), Pj)
        R, T, W = iterate(torch, 2, K, Pj); W = W[0]
        lam = torch.tensor([0.1], dtype=torch.float32).double()
        gW = randn(torch, (K, 1), Pj + 7)
        leaves = [t.clone().requires_grad_() for t in (H, g, lam)]
        Hj, gj = assemble(torch, leaves[0], leaves[1])
        dj = torch.linalg.solve(damped(torch, Hj[None], leaves[2], Pj - 1)[0], gj)
        (dj[12:] * gW.squeeze(-1)).sum().backward()
        row = {"case": f"dense window backward Pj={Pj}", "variant": new_step_variant(Pj)}
        f = libs.run("new", lambda: ops.lm_window_solve_update(cu(H), cu(g), cu(lam), cu(R), cu(T), cu(W)))
        for lib in ("base", "new"):
            try:
                d = libs.run(lib, lambda: ops.lm_window_solve_update_bwd(cu(H), cu(g), cu(lam), f[3], cu(R), cu(T), cu(torch.zeros(2, 3, 3)),
                                                                         cu(torch.zeros(2, 3, 1)), cu(gW)))
            except Exception as e:
                row[lib] = str(e)[:80]
                continue
            row[lib] = {"dH": r(sym(d[0]), sym(leaves[0].grad)), "dg": r(d[1], leaves[1].grad), "dlambda": r(d[2], leaves[2].grad)}
        res["changed"].append(row)
    # lm_lambda against a float64 MLP
    for C in (5, 128, 256):
        params = mlp_params(torch, C, C)
        rb = (0.02 * (1 + torch.rand(32, C, generator=torch.Generator().manual_seed(C))) * 4096).float()
        ref = lambda64(torch, rb, 4096, params)
        row = {"case": f"lm_lambda C={C}"}
        for lib in ("base", "new"):
            row[lib] = r(libs.run(lib, lambda: ops.lm_lambda(cu(rb), 4096, ops.pack_mlp(params).cuda(), 1000.0)), ref)
        res["changed"].append(row)
    # the arrow (lambda given), forward and backward
    for K in (16, 64, 128, 154, 155, 200, 215, 216):
        H = torch.stack([graded_spd(torch, 6 + K, 1e3, K + f) + 2 * torch.eye(6 + K, dtype=torch.float64) for f in range(4)]).float().double()
        g = randn(torch, (4, 6 + K), K)
        R, T, W = iterate(torch, 4, K, K); W = W[:2]
        lam = torch.tensor([0.1, 1.0], dtype=torch.float64)
        gR, gT, gW = randn(torch, (4, 3, 3), K + 1), randn(torch, (4, 3, 1), K + 2), randn(torch, (2, K, 1), K + 3)
        same = previous_arrow_variant(K, 0) == new_arrow_variant(K)
        f, _ = both(f"arrow K={K}", ("R", "T", "W", "delta", "status"),
                    lambda: ops.lm_window_batch_solve_update(cu(H), cu(g), cu(lam), cu(R), cu(T), cu(W)), same)
        both(f"arrow backward K={K}", ("dH", "dg", "dlambda", "dR", "dT", "dW"),
             lambda: ops.lm_window_batch_solve_update_bwd(cu(H), cu(g), cu(lam), f[3], cu(R), cu(T), cu(gR), cu(gT), cu(gW)), same)
    # the runs: a sparse scene (4 pairs, 4096 points, C = 128), two levels
    dev = torch.device("cuda")
    sc = synth.make_scene(nb=4, H=240, W=320, C=128, K=200, level_ids=(2, 3), seed=17, device=dev, dtype=torch.float32, n_points=4096,
                          shared_depth=True, window_frames=2)
    mlps = [ops.pack_mlp(mlp_params(torch, 128, 5 + i)).cuda() for i in range(2)]
    RUN = ("R", "T", "W", "status")
    for K in (16, 64, 128, 200):
        levels = [ops.Level(l.conv1, l.conv2, l.intr, l.p, l.D, l.B[..., :K].contiguous()) for l in sc.levels]
        W0 = sc.W0[:, :K].contiguous()
        both(f"lm_run mlp K={K}", RUN, lambda: ops.lm_run(levels, 2, sc.R0, sc.T0, W0, mlp_packed=mlps, l2_regularizer_base=1000.0,
                                                           precision=_lib.PREC_FP32_SIMT),
             previous_step_variant(6 + K, 128) == new_step_variant(6 + K))
        both(f"lm_run fixed lambda K={K}", RUN, lambda: ops.lm_run(levels, 2, sc.R0, sc.T0, W0, lambda_fixed=0.05, precision=_lib.PREC_FP32_SIMT),
             previous_step_variant(6 + K, 1) == new_step_variant(6 + K))
        scr = lambda: ops.lm_run(levels, 2, sc.R0, sc.T0, W0, mlp_packed=mlps, l2_regularizer_base=1000.0, precision=_lib.PREC_FP32_SIMT,
                                 vmatrix_batch_scramble=True)
        a, b = libs.run("base", scr), libs.run("new", scr)
        res["changed"].append({"case": f"lm_run scramble K={K}", "new vs base": {n: r(y, x) for n, x, y in zip(RUN[:3], a, b)},
                               "status": [int(a[3].abs().max()), int(b[3].abs().max())]})
        both(f"lm_window_run K={K}", RUN, lambda: ops.lm_window_run(levels, 2, sc.R0, sc.T0, W0[0].contiguous(), mlp_packed=mlps,
                                                                    l2_regularizer_base=1000.0, precision=_lib.PREC_FP32_SIMT), True)
        same_arrow = previous_arrow_variant(K, 128) == new_arrow_variant(K)
        Ww = W0.reshape(2, 2, K, 1)[:, 0].contiguous()
        both(f"lm_window_batch_run K={K}", RUN, lambda: ops.lm_window_batch_run(levels, 2, 2, sc.R0, sc.T0, Ww, mlp_packed=mlps,
                                                                                l2_regularizer_base=1000.0, precision=_lib.PREC_FP32_SIMT), same_arrow)
        kf = lambda t: t.reshape(2, 2, *t.shape[1:])[:, 0].contiguous()
        keys = [ops.KeyframeLevel(kf(l.conv1), l.conv2, l.intr, kf(l.p), kf(l.D), kf(l.B)[..., :K].contiguous()) for l in sc.levels]
        both(f"lm_keyframe_run K={K}", RUN, lambda: ops.lm_keyframe_run(keys, 2, sc.R0, sc.T0, Ww, mlp_packed=mlps, l2_regularizer_base=1000.0,
                                                                        precision=_lib.PREC_AUTO), same_arrow)
    return res


def timing(libs, rounds, reps):
    import torch
    from banet_b200 import ops
    cu = lambda t: t.to(device="cuda", dtype=torch.float32).contiguous()
    cases = {}
    for K in (128, 64, 32):
        H = torch.stack([graded_spd(torch, 6 + K, 1e3, i) for i in range(32)]); g = randn(torch, (32, 6 + K), K)
        R, T, W = [cu(t) for t in iterate(torch, 32, K, K)]
        Hc, gc, lam = cu(H), cu(g), cu(torch.full((32,), 0.1))
        gR, gT, gW = cu(randn(torch, (32, 3, 3), 1)), cu(randn(torch, (32, 3, 1), 2)), cu(randn(torch, (32, K, 1), 3))

        def fb(Hc=Hc, gc=gc, lam=lam, R=R, T=T, W=W, gR=gR, gT=gT, gW=gW):
            f = ops.lm_solve_update(Hc, gc, lam, R, T, W)
            ops.lm_solve_update_bwd(Hc, gc, lam, f[3], R, T, gR, gT, gW)
        cases[f"lm_solve_update + bwd nb=32 K={K}"] = fb
    for nf in (4, 16):
        K = 128
        H = torch.stack([graded_spd(torch, 6 + K, 1e3, 50 + f) for f in range(nf)]); g = randn(torch, (nf, 6 + K), nf)
        R, T, W = [cu(t) for t in iterate(torch, nf, K, nf)]; W = W[0].contiguous()
        Hc, gc, lam = cu(H), cu(g), cu(torch.tensor([0.1]))
        gR, gT, gW = cu(randn(torch, (nf, 3, 3), 1)), cu(randn(torch, (nf, 3, 1), 2)), cu(randn(torch, (K, 1), 3))
        f = libs.run("new", lambda: ops.lm_window_solve_update(Hc, gc, lam, R, T, W))
        cases[f"lm_window_solve_update_bwd nf={nf} K={K}"] = (lambda Hc=Hc, gc=gc, lam=lam, d=f[3], R=R, T=T, gR=gR, gT=gT, gW=gW:
                                                              ops.lm_window_solve_update_bwd(Hc, gc, lam, d, R, T, gR, gT, gW))
    rb = cu(0.02 * (1 + torch.rand(32, 128, generator=torch.Generator().manual_seed(1))) * 4096)
    mlp = ops.pack_mlp(mlp_params(torch, 128, 1)).cuda()
    cases["lm_lambda nb=32 C=128"] = lambda: ops.lm_lambda(rb, 4096, mlp, 1000.0)
    out = {name: {"base": [], "new": []} for name in cases}
    for _ in range(rounds):
        for lib in ("base", "new"):
            for name, fn in cases.items():
                def timed():
                    for _ in range(3):
                        fn()
                    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(reps):
                        fn()
                    e1.record(); torch.cuda.synchronize()
                    return e0.elapsed_time(e1) / reps
                out[name][lib].append(libs.run(lib, timed))
    return out


def gpu_identity():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
    return {"name": q[0], "power_limit_w": float(q[1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="libbanet.so to compare against")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    libs = Libs({"base": os.path.abspath(a.base), "new": os.path.abspath(os.path.join(ROOT, "banet_b200", "libbanet.so"))})
    report = {"gpu": gpu_identity(), "check": correctness(libs)}
    chk = report["check"]
    print(f"{len(chk['bitwise'])} outputs bitwise equal, {len(chk['mismatch'])} expected-bitwise outputs differ", *chk["mismatch"], sep="\n")
    for row in chk["changed"]:
        print(json.dumps(row))
    report["timing_ms"] = {}
    if a.rounds:
        t = timing(libs, a.rounds, a.reps)
        for name, row in t.items():
            s = {k: {"median": statistics.median(v), "min": min(v), "max": max(v)} for k, v in row.items()}
            report["timing_ms"][name] = s
            print(f"{name:44s} base {s['base']['median']:8.4f} [{s['base']['min']:.4f}-{s['base']['max']:.4f}]   "
                  f"new {s['new']['median']:8.4f} [{s['new']['min']:.4f}-{s['new']['max']:.4f}] ms")
    print(report["gpu"])
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)
    if chk["mismatch"]:
        sys.exit("ab_solve_outputs: outputs expected to be bitwise equal differ")


if __name__ == "__main__":
    main()
