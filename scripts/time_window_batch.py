"""Batches of keyframe windows (banet_lm_window_batch_*) against the single-window path, timed with CUDA events, warm-ups, the contenders
alternated in one loop, medians reported.  Prints one JSON document with the card's name and power limit; --out also writes it to a file.
  a) nw = 32 windows x nf = 4 frames, 4096 points per frame, C = K = 128, lambda-MLP, forward + backward of one differentiable iteration:
     autograd.window_batch_iteration_fused against a loop of 32 autograd.window_iteration_fused calls;
  b) the window step alone (lambda given), forward + backward, nf = 4 and nf = 16 at K = 128: banet_lm_window_batch_solve_update(_bwd) with
     nw = 1 against banet_lm_window_solve_update(_bwd) (dense fp64 at nf = 4, dense fp32 at nf = 16);
  c) nf = 48, K = 128: a window only the block-arrow step runs (the dense one rejects 416 unknowns)."""
import argparse, json, os, statistics, sys
import torch
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from banet_b200 import synth, autograd as ag, ops, _lib
from time_window_training_step import card


def timed(fns, warmup, reps):
    """fns: name -> callable returning (forward time end event recorded inside) ... each call: forward, then backward; alternated."""
    ev = lambda: torch.cuda.Event(enable_timing=True)
    out = {n: ([], []) for n in fns}
    for it in range(warmup + reps):
        for name, (fwd, bwd) in fns.items():
            e0, e1, e2 = ev(), ev(), ev()
            e0.record(); state = fwd(); e1.record(); bwd(state); e2.record()
            torch.cuda.synchronize()
            if it >= warmup:
                out[name][0].append(e0.elapsed_time(e1)); out[name][1].append(e1.elapsed_time(e2))
    return {n: {"forward_ms_median": statistics.median(tf), "backward_ms_median": statistics.median(tb),
                "forward_ms_min_max": [min(tf), max(tf)], "backward_ms_min_max": [min(tb), max(tb)]} for n, (tf, tb) in out.items()}


def case_a(args):
    nw, nf, C, K = 32, 4, 128, 128
    g = torch.Generator().manual_seed(7); dims = [C, 2 * C, 4 * C, 2 * C, C, 1]       # he_normal filters, zero biases (bundlenet.py:102-110)
    mlp = [((torch.randn(dims[i], dims[i + 1], generator=g) * (2.0 / dims[i]) ** 0.5).cuda().requires_grad_(), torch.zeros(dims[i + 1], device="cuda").requires_grad_())
           for i in range(5)]
    sc = synth.make_scene(nb=nw * nf, H=120, W=160, C=C, K=K, level_ids=(3,), seed=21, device="cuda", dtype=torch.float32, n_points=4096,
                          shared_depth=True, window_frames=nf)
    lv = sc.levels[0]
    leaf = lambda t: t.detach().clone().requires_grad_()
    bw = lambda t: t.reshape(nw, nf, *t.shape[1:])
    conv1, conv2, D, B, R, T = (leaf(bw(t)) for t in (lv.conv1, lv.conv2, lv.D, lv.B, sc.R0, sc.T0))
    W = leaf(sc.W0.reshape(nw, nf, K, 1)[:, 0])
    intr, p = bw(lv.intr), bw(lv.p)
    params = (conv1, conv2, D, B, R, T, W, *[x for wb in mlp for x in wb])

    def batched():
        for t in params: t.grad = None
        Rn, Tn, Wn = ag.window_batch_iteration_fused(conv1, conv2, intr, p, D, B, R, T, W, mlp, 1000.0)
        return Rn.sum() + Tn.sum() + (Wn * Wn).sum()

    def loop():
        for t in params: t.grad = None
        loss = 0
        for w in range(nw):
            Rn, Tn, Wn = ag.window_iteration_fused(conv1[w], conv2[w], intr[w], p[w], D[w], B[w], R[w], T[w], W[w], mlp, 1000.0)
            loss = loss + Rn.sum() + Tn.sum() + (Wn * Wn).sum()
        return loss

    with torch.no_grad():                                            # both compute the same iteration
        a = ag.window_batch_iteration_fused(conv1, conv2, intr, p, D, B, R, T, W, mlp, 1000.0)
        b = [ag.window_iteration_fused(conv1[w], conv2[w], intr[w], p[w], D[w], B[w], R[w], T[w], W[w], mlp, 1000.0) for w in range(nw)]
        diff = max(float((a[0] - torch.stack([x[0] for x in b])).norm() / a[0].norm()), float((a[2] - torch.stack([x[2] for x in b])).norm() / a[2].norm()))
    res = timed({"batched": (batched, lambda l: l.backward()), "loop_of_single_windows": (loop, lambda l: l.backward())}, args.warmup, args.reps)
    return {"case": "a", "nw": nw, "nf": nf, "N_per_frame": lv.N, "C": C, "K": K, "lambda": "mlp", "precision": "FP32_SIMT (autograd default)",
            "reps": args.reps, "rel_diff_R_W_batched_vs_loop": diff, **res}


def step_case(nf, K, args, with_dense):
    nw, C = 1, 32
    sc = synth.make_scene(nb=nf, H=96, W=128, C=C, K=K, level_ids=(3,), seed=23, device="cuda", dtype=torch.float32, n_points=2048, shared_depth=True)
    l = sc.levels[0]
    lv = ops.Level(l.conv1, l.conv2, l.intr, l.p, l.D, l.B)
    W = sc.W0[0] + 0.01
    Hm, g, _, _ = ops.lm_build(lv, sc.R0, sc.T0, W.reshape(1, K, 1).expand(nf, K, 1).contiguous(), _lib.PREC_FP32_SIMT)
    lam = torch.tensor([0.5], device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(1)
    dR, dT, dW = (torch.randn(s, generator=gen, device="cuda") for s in ((nf, 3, 3), (nf, 3, 1), (K, 1)))
    fns = {"block_arrow": (lambda: ops.lm_window_batch_solve_update(Hm, g, lam, sc.R0, sc.T0, W.reshape(1, K, 1)),
                           lambda o: ops.lm_window_batch_solve_update_bwd(Hm, g, lam, o[3], sc.R0, sc.T0, dR, dT, dW.reshape(1, K, 1)))}
    row = {"case": "b" if with_dense else "c", "nw": nw, "nf": nf, "K": K, "unknowns": 6 * nf + K, "lambda": "given", "reps": args.reps}
    if with_dense:
        fns["dense_single_window"] = (lambda: ops.lm_window_solve_update(Hm, g, lam, sc.R0, sc.T0, W),
                                      lambda o: ops.lm_window_solve_update_bwd(Hm, g, lam, o[3], sc.R0, sc.T0, dR, dT, dW))
        a, b = fns["block_arrow"][0](), fns["dense_single_window"][0]()
        row["rel_diff_delta"] = float((a[3].reshape(-1) - b[3]).norm() / b[3].norm())
    else:
        try:
            ops.lm_window_solve_update(Hm, g, lam, sc.R0, sc.T0, W)
            row["dense_single_window"] = "ran"
        except _lib.BanetError as e:
            row["dense_single_window"] = "rejected: " + str(e).split(":")[0]
    row.update(timed(fns, args.warmup, args.reps))
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    _lib.require_device()
    rows = []
    for fn in (lambda: case_a(args), lambda: step_case(4, 128, args, True), lambda: step_case(16, 128, args, True), lambda: step_case(48, 128, args, False)):
        rows.append(fn())
        print(json.dumps(rows[-1]), flush=True)
        torch.cuda.empty_cache()
    doc = {"script": "scripts/time_window_batch.py", **card(), "rows": rows}
    print(json.dumps(doc, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
