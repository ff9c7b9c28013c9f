"""Float64 statement of BundleNet.WindowResize: the schedule of oracle.bundle_resize (reference bundlenet.py:332-399) with oracle.window_iteration
per keyframe window in place of bundle_iteration per pair.  tests/test_window_resize.py ties it to bundle_resize (itself held to the reference's
own code by tests/test_oracle_pinned.py): with one frame per window the two are the same computation."""
import torch

from oracle import ba_oracle as O


def window_resize(intrisic, key_layers, frame_layers, points, basis, init_depth, mlp_params_by_level, init_rotation=None, init_translation=None,
                  opts: O.IterOptions = O.IterOptions(), geo: O.ResizeGeometry = O.ResizeGeometry()):
    """intrisic [nw,4,1]; key_layers 4 x [nw,h_l,w_l,C]; frame_layers 4 x [nw,nf,h_l,w_l,C] (F2); points [nw,N,2]; basis [nw,h/2,w/2,K];
    init_depth [nw,h/2,w/2,1]; init_rotation [nw,nf,3,3], init_translation [nw,nf,3,1].  -> (Rs [nw,nf,3,3], Ts [nw,nf,3,1], depths
    [nw,h/2,w/2,1]), one entry per level (2, 3).  conv1, p, D, B and W are per window; conv2 = [F2 | grad_fixed(F2)], R and T per frame."""
    nw, nf = frame_layers[-1].shape[0], frame_layers[-1].shape[1]
    K = basis.shape[-1]
    _points, sfx, sfy, sox, soy = O._prepare(intrisic, points, geo)     # :338-339, :354-357
    d = O.resampler(init_depth.detach(), _points / 2)                    # :341-343
    b = O.resampler(basis, _points / 2)                                  # :344
    p = O.compute_coordinates(_points, sfx, sfy, sox, soy)              # :358
    dt = frame_layers[-1].dtype
    R = torch.eye(3, dtype=dt).repeat(nw, nf, 1, 1) if init_rotation is None else init_rotation
    T = torch.zeros(nw, nf, 3, 1, dtype=dt) if init_translation is None else init_translation
    W = [torch.zeros(K, 1, dtype=dt) for _ in range(nw)]
    Rs, Ts, Ds = [], [], []
    for level in range(2, 4):                                            # :376
        scale = 2 ** (3 - level)
        fx, fy, ox, oy = sfx / scale, sfy / scale, sox / scale, soy / scale
        layer1 = O.resampler(key_layers[level], _points / scale)        # :385
        Rl, Tl = [], []
        for w in range(nw):
            F2 = frame_layers[level][w]
            layer2 = torch.cat([F2, O.grad_fixed(F2)], dim=-1)           # :388-389, per frame
            kf = lambda t: t[w:w + 1].expand(nf, *t.shape[1:])          # the keyframe's tensors, the same for every frame
            Rn, Tn, W[w] = O.window_iteration(kf(layer1), layer2, kf(fx), kf(fy), kf(ox), kf(oy), kf(p), kf(d), kf(b), R[w], T[w], W[w],
                                              mlp_params_by_level[str(level)], opts)   # :391-393
            Rl.append(Rn); Tl.append(Tn)
        R, T = torch.stack(Rl), torch.stack(Tl)
        Rs.append(R); Ts.append(T)
        Wb = torch.stack(W)                                              # [nw,K,1]
        Ds.append(init_depth + (basis.reshape(nw, -1, K) @ Wb).reshape(nw, geo.out_hw[0], geo.out_hw[1], 1))   # :397
    return Rs, Ts, Ds
