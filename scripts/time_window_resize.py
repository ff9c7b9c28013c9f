"""BundleNet.WindowResize (BundleResize's schedule for keyframe windows: conv1, p, D, B and W once per window) against the route a user has
without it: BundleResize on the nw*nf (keyframe -> frame) pairs with the keyframe's tensors repeated per frame.  BundleResize pairs image b with
image b + nb/2 (its half swap, bundlenet.py:386), so it runs on 2*nw*nf images (the repeated keyframes, then the frames) and also solves the
nw*nf reverse pairs (frame -> keyframe).  The two routes solve different problems (shared W against per-pair W): only their times and peak
memory are compared.  Timed with CUDA events, warm-ups, the contenders alternated in one loop, medians and min-max reported, both at the
BundleNet defaults (AUTO precision, lambda-MLP, l2_regularizer_base = 1000):
  inference: no gradients recorded;
  training:  forward + backward of one step with a loss on both levels' R, T and depth;
  a) the reference's sparse regime: nw = 8, nf = 4, N = 4096 points, C = K = 128;
  b) the dense level-3 grid at the reference's 320 x 256 resolution (N = 81920): nw = 4, nf = 4, C = K = 128.
A torch.profiler pass over WindowResize's inference at (a), after the timing, reports the summed kernel time per call and its share of the
wall time.  Prints one JSON document with the card's name and power limit; --out also writes it to a file."""
import argparse, json, os, sys
import torch
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from banet_b200 import synth, _lib
from banet_b200.bundlenet import BundleNet
from time_window_training_step import card
from time_window_batch import timed
from time_window_keyframe import peak_mib

C = K = 128


def loss(outs):
    Rs, Ts, Ds = outs
    return sum(R.sum() + T.sum() + (D * D).sum() for R, T, D in zip(Rs, Ts, Ds))


def case(name, nw, nf, n_points, args):
    sc = synth.make_window_resize_scene(nw, nf, C, K, n_points=n_points, seed=21, device="cuda")
    net = BundleNet(C, levels=("2", "3")).cuda()
    leaf = lambda t: t.detach().clone().requires_grad_()
    rep = lambda t: t.repeat_interleave(nf, 0)
    two = lambda t: torch.cat([t, t], 0)
    win = dict(key=[leaf(l) for l in sc.key_layers], frames=[leaf(l) for l in sc.frame_layers], basis=leaf(sc.basis), depth=leaf(sc.init_depth),
               R0=leaf(sc.R0), T0=leaf(sc.T0))
    pairs = dict(layers=[leaf(torch.cat([rep(k), f.reshape(nw * nf, *f.shape[2:])], 0)) for k, f in zip(sc.key_layers, sc.frame_layers)],
                 intr=two(rep(sc.intrisic)), points=two(rep(sc.points)), basis=leaf(two(rep(sc.basis))), depth=leaf(two(rep(sc.init_depth))),
                 R0=leaf(two(sc.R0.reshape(-1, 3, 3))), T0=leaf(two(sc.T0.reshape(-1, 3, 1))))
    leaves = [*win["key"], *win["frames"], win["basis"], win["depth"], win["R0"], win["T0"], *pairs["layers"], pairs["basis"], pairs["depth"],
              pairs["R0"], pairs["T0"], *net.parameters()]

    def window():
        for t in leaves: t.grad = None
        return net.WindowResize(sc.intrisic, win["key"], win["frames"], sc.points, win["basis"], win["depth"], win["R0"], win["T0"])

    def bundle():
        for t in leaves: t.grad = None
        return net.BundleResize(pairs["intr"], pairs["layers"], pairs["points"], pairs["basis"], pairs["depth"], pairs["R0"], pairs["T0"])

    row = {"case": name, "nw": nw, "nf": nf, "N_per_window": sc.points.shape[1], "C": C, "K": K, "lambda": "mlp, l2_regularizer_base 1000",
           "precision": "AUTO (BundleNet default)", "reps": args.reps, "warmup": args.warmup,
           "contender": f"BundleResize on {2 * nw * nf} images: the {nw * nf} keyframe->frame pairs and their {nw * nf} reverses"}
    with torch.no_grad():
        fns = {"WindowResize": (window, lambda o: None), "BundleResize_repeated_keyframes": (bundle, lambda o: None)}
        inf = timed(fns, args.warmup, args.reps)
        for f in fns:
            inf[f]["peak_MiB"] = peak_mib(fns[f][0])
        status = {}
        for f in fns:
            fns[f][0]()
            status[f] = int(net.last_status.count_nonzero())
        inf["last_status_nonzero"] = status
    row["inference"] = {"timed": "forward = the whole no-grad call", **inf}
    fns = {"WindowResize": (lambda: loss(window()), lambda l: l.backward()),
           "BundleResize_repeated_keyframes": (lambda: loss(bundle()), lambda l: l.backward())}
    tr = timed(fns, args.warmup, args.reps)
    for f in fns:
        tr[f]["peak_MiB"] = peak_mib(lambda f=f: fns[f][1](fns[f][0]()))
    row["training"] = {"timed": "forward = the call and the loss, backward = loss.backward()", **tr}
    if args.profile and name == "a":
        row["profile_inference_WindowResize"] = profile(window, args)
    return row


def profile(fn, args):
    """Summed device-kernel time per no-grad call against its CUDA-event wall time: what is left is launch and host overhead."""
    from torch.profiler import profile as prof, ProfilerActivity
    calls = 10
    with torch.no_grad():
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        with prof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
            for _ in range(calls):
                fn()
            torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(calls):
            fn()
        e1.record(); torch.cuda.synchronize()
    kernels = {}
    for ev in p.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            k = kernels.setdefault(ev.name, [0, 0.0])
            k[0] += 1; k[1] += ev.device_time_total / 1000.0
    total = sum(v[1] for v in kernels.values()) / calls
    wall = e0.elapsed_time(e1) / calls
    top = sorted(kernels.items(), key=lambda kv: -kv[1][1])[:12]
    return {"calls": calls, "kernel_ms_per_call": total, "wall_ms_per_call_unprofiled": wall, "kernel_share_of_wall": total / wall,
            "kernels_per_call": sum(v[0] for v in kernels.values()) / calls,
            "top_kernels_ms_per_call": {n[:90]: round(v[1] / calls, 4) for n, v in top}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    _lib.require_device()
    rows = []
    for fn in (lambda: case("a", 8, 4, 4096, args), lambda: case("b", 4, 4, None, args)):
        rows.append(fn())
        print(json.dumps(rows[-1]), flush=True)
        torch.cuda.empty_cache()
    doc = {"script": "scripts/time_window_resize.py", **card(), "rows": rows}
    print(json.dumps(doc, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
