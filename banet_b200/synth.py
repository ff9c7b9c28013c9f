"""Seeded synthetic frame-pair scenes with a planted solution (SURVEY.md §8d "Synthetic data").

Pure torch, device-agnostic data generation for tests and bench.py — not part of the LM path.
Per level: F2 = unit-variance Gaussian-blurred noise, conv2 = [F2 | grad_fixed(F2)], basis =
blurred noise scaled by rsqrt(var+1e-3) (the decoder's output contract, reference dec.py:107-108),
D0 = blurred U[1,3] m, and conv1 = F2 sampled at the warp of the level's pixel grid under the
planted (R*, T*, D0 + B W*), so the feature-metric residual is 0 at the planted solution.

The start pose is NOT (I, 0): at zero motion the depth Jacobian (reference bundlenet.py:63-74)
vanishes identically and the reference's undamped last depth coefficient (:266) makes the normal
matrix singular; the solve starts from a perturbed copy of the planted translation, as if it came
from the pose-only stage (`CameraResize`, bundlenet.py:280-329).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Optional

import torch
import torch.nn.functional as F

TUM_INTRINSICS = (535.4, 539.2, 320.1, 247.6)       # reference legacy/seq_example.py:114, at 640x480


def _gauss_kernel(sigma: float, device, dtype):
    r = max(1, int(math.ceil(3.0 * sigma)))
    x = torch.arange(-r, r + 1, device=device, dtype=dtype)
    k = torch.exp(-0.5 * (x / sigma) ** 2)
    return k / k.sum(), r


def gaussian_blur_nchw(x: torch.Tensor, sigma: float) -> torch.Tensor:
    """Separable Gaussian blur, reflect padding.  x [n,c,h,w]."""
    k, r = _gauss_kernel(sigma, x.device, x.dtype)
    r = min(r, x.shape[-1] - 1, x.shape[-2] - 1)
    k = k[len(k) // 2 - r: len(k) // 2 + r + 1]
    k = k / k.sum()
    n, c, h, w = x.shape
    x = x.reshape(n * c, 1, h, w)
    x = F.conv2d(F.pad(x, (r, r, 0, 0), mode="reflect"), k.view(1, 1, 1, -1))
    x = F.conv2d(F.pad(x, (0, 0, r, r), mode="reflect"), k.view(1, 1, -1, 1))
    return x.reshape(n, c, h, w)


def grad_fixed_nhwc(f: torch.Tensor) -> torch.Tensor:
    """[F | gx | gy] with reflect-pad central differences (layout of the reference's conv2)."""
    p = F.pad(f.permute(0, 3, 1, 2), (1, 1, 1, 1), mode="reflect").permute(0, 2, 3, 1)
    h, w = f.shape[1], f.shape[2]
    gx = 0.5 * (p[:, 1:h + 1, 2:w + 2] - p[:, 1:h + 1, 0:w])
    gy = 0.5 * (p[:, 2:h + 2, 1:w + 1] - p[:, 0:h, 1:w + 1])
    return torch.cat([f, gx, gy], dim=-1)


def bilinear_zero_pad(data: torch.Tensor, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """data [nb,h,w,C], x,y [nb,N] -> [nb,N,C]; texels outside the map read 0."""
    nb, h, w, C = data.shape
    x0f, y0f = torch.floor(x), torch.floor(y)
    dx, dy = (x - x0f).unsqueeze(-1), (y - y0f).unsqueeze(-1)
    x0, y0 = x0f.long(), y0f.long()
    flat = data.reshape(nb, h * w, C)
    out = torch.zeros(nb, x.shape[1], C, device=data.device, dtype=data.dtype)
    for xi, yi, wg in ((x0, y0, (1 - dx) * (1 - dy)), (x0 + 1, y0, dx * (1 - dy)),
                       (x0, y0 + 1, (1 - dx) * dy), (x0 + 1, y0 + 1, dx * dy)):
        ok = ((xi >= 0) & (xi < w) & (yi >= 0) & (yi < h)).unsqueeze(-1).to(data.dtype)
        idx = (yi.clamp(0, h - 1) * w + xi.clamp(0, w - 1)).unsqueeze(-1).expand(-1, -1, C)
        out += torch.gather(flat, 1, idx) * wg * ok
    return out


def rodrigues(w: torch.Tensor) -> torch.Tensor:
    """w [nb,3] -> R [nb,3,3]."""
    th = w.norm(dim=1).clamp_min(1e-12).view(-1, 1, 1)
    k = w / th.view(-1, 1)
    z = torch.zeros_like(k[:, 0])
    Kx = torch.stack([z, -k[:, 2], k[:, 1], k[:, 2], z, -k[:, 0], -k[:, 1], k[:, 0], z], 1).view(-1, 3, 3)
    eye = torch.eye(3, device=w.device, dtype=w.dtype).unsqueeze(0)
    return eye + torch.sin(th) * Kx + (1 - torch.cos(th)) * (Kx @ Kx)


@dataclass
class SceneLevel:
    level: int                 # reference level index: scale = 2**(3-level)  (bundlenet.py:378)
    h: int
    w: int
    conv1: torch.Tensor        # [nb,N,C]
    conv2: torch.Tensor        # [nb,h,w,3C]
    intr: torch.Tensor         # [nb,4]  fx,fy,ox,oy at this level
    p: torch.Tensor            # [nb,3,N]
    D: torch.Tensor            # [nb,N,1]
    B: Optional[torch.Tensor]  # [nb,N,K]
    points: torch.Tensor       # [nb,N,2] level-pixel coordinates
    grid: Optional[tuple] = None   # (w,h) when the points are the dense row-major pixel grid

    @property
    def N(self):
        return self.conv1.shape[1]

    def intr_tiled(self):
        """fx,fy,ox,oy as the reference passes them: [nb,N] each."""
        n = self.N
        return tuple(self.intr[:, i:i + 1].expand(-1, n).contiguous() for i in range(4))


@dataclass
class Scene:
    levels: List[SceneLevel]
    R_true: torch.Tensor; T_true: torch.Tensor; W_true: Optional[torch.Tensor]
    R0: torch.Tensor; T0: torch.Tensor; W0: Optional[torch.Tensor]


def make_scene(nb: int, H: int, W: int, C: int, K: int, level_ids=(0, 1, 2, 3), seed: int = 1234,
               device="cpu", dtype=torch.float32, n_points: Optional[int] = None,
               rot_deg: float = 1.0, trans_m: float = 0.02, w_std: float = 0.02,
               start_trans_noise_m: float = 0.01, pair_chunk: int = 4, shared_depth: bool = False,
               window_frames: Optional[int] = None) -> Scene:
    """Build a planted-solution scene.  (H,W) is the finest (level-3) resolution; level l has
    (H,W)/2**(3-l).  K == 0 -> pose-only scene (B None).  n_points: if given, use that many random
    sub-pixel points per level instead of the dense grid (the reference's sparse mode,
    legacy/seq_example.py:12,72-82).  shared_depth: the nb pairs are (keyframe -> frame f) of one window: same D, B and planted W for
    every pair, own pose and own frame features (the joint window solve, ops.lm_window_run).  window_frames = nf (with shared_depth): nb / nf
    independent windows (ops.lm_window_batch_run), pairs w nf .. w nf + nf - 1 share window w's depth, basis and planted W; None: one window."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    dev = torch.device(device)

    def randn(*s):
        return torch.randn(*s, generator=g, dtype=torch.float32).to(dev, dtype)

    def rand(*s):
        return torch.rand(*s, generator=g, dtype=torch.float32).to(dev, dtype)

    w_true = randn(nb, 3) * math.radians(rot_deg)
    R_true = rodrigues(w_true)
    T_true = (randn(nb, 3) * trans_m).unsqueeze(-1)
    W_true = (randn(nb, K) * w_std).unsqueeze(-1) if K > 0 else None
    gf = nb if window_frames is None else int(window_frames)         # pairs per window
    if shared_depth and nb % gf:
        raise ValueError(f"window_frames={gf} does not divide nb={nb}")
    ng = nb // gf
    if shared_depth and K > 0:
        W_true = W_true[::gf].repeat_interleave(gf, 0)
    R0 = torch.eye(3, device=dev, dtype=dtype).repeat(nb, 1, 1)
    T0 = T_true + randn(nb, 3, 1) * start_trans_noise_m
    W0 = torch.zeros(nb, K, 1, device=dev, dtype=dtype) if K > 0 else None

    levels = []
    for lid in level_ids:
        scale = 2 ** (3 - lid)
        h, w = H // scale, W // scale
        intr = torch.tensor(TUM_INTRINSICS, device=dev, dtype=dtype) * (W / 640.0) / scale
        intr = intr.unsqueeze(0).repeat(nb, 1)
        if n_points is None:
            vv, uu = torch.meshgrid(torch.arange(h, device=dev, dtype=dtype),
                                    torch.arange(w, device=dev, dtype=dtype), indexing="ij")
            pts = torch.stack([uu.reshape(-1), vv.reshape(-1)], -1).unsqueeze(0).repeat(nb, 1, 1)
        else:
            pts = rand(nb, n_points, 2) * torch.tensor([w - 1.0, h - 1.0], device=dev, dtype=dtype)
        N = pts.shape[1]
        fx, fy, ox, oy = [intr[:, i:i + 1] for i in range(4)]
        ray = torch.stack([(pts[..., 0] - ox) / fx, (pts[..., 1] - oy) / fy, torch.ones_like(pts[..., 0])], 1)
        p = ray / ray.norm(dim=1, keepdim=True)

        conv1 = torch.empty(nb, N, C, device=dev, dtype=dtype)
        conv2 = torch.empty(nb, h, w, 3 * C, device=dev, dtype=dtype)
        D = torch.empty(nb, N, 1, device=dev, dtype=dtype)
        Bm = torch.empty(nb, N, K, device=dev, dtype=dtype) if K > 0 else None
        sig_b = max(1.0, 8.0 / scale)
        shared_dmap = gaussian_blur_nchw(1.0 + 2.0 * rand(ng, 1, h, w), sig_b).permute(0, 2, 3, 1) if shared_depth else None
        shared_bm = gaussian_blur_nchw(randn(ng, K, h, w), sig_b) if shared_depth and K > 0 else None
        for b0 in range(0, nb, pair_chunk):                 # chunked so cfg2-sized scenes fit comfortably
            b1 = min(nb, b0 + pair_chunk)
            n = b1 - b0
            f2 = gaussian_blur_nchw(randn(n, C, h, w), 2.0)
            f2 = f2 / f2.flatten(2).std(dim=2).clamp_min(1e-6).view(n, C, 1, 1)
            f2 = f2.permute(0, 2, 3, 1).contiguous()
            conv2[b0:b1] = grad_fixed_nhwc(f2)
            grp = torch.arange(b0, b1, device=dev) // gf                                   # the window of each pair
            dmap = shared_dmap[grp] if shared_depth else gaussian_blur_nchw(1.0 + 2.0 * rand(n, 1, h, w), sig_b).permute(0, 2, 3, 1)
            # rescale the blurred map back to span ~[1,3] m
            dmin = dmap.flatten(1).min(1).values.view(n, 1, 1, 1); dmax = dmap.flatten(1).max(1).values.view(n, 1, 1, 1)
            dmap = 1.0 + 2.0 * (dmap - dmin) / (dmax - dmin).clamp_min(1e-6)
            xs, ys = pts[b0:b1, :, 0], pts[b0:b1, :, 1]
            D[b0:b1] = bilinear_zero_pad(dmap.contiguous(), xs, ys)
            Dt = D[b0:b1]
            if K > 0:
                bm = shared_bm[grp] if shared_depth else gaussian_blur_nchw(randn(n, K, h, w), sig_b)
                bm = bm * torch.rsqrt(bm.flatten(2).var(dim=2) + 1e-3).view(n, K, 1, 1)
                Bm[b0:b1] = bilinear_zero_pad(bm.permute(0, 2, 3, 1).contiguous(), xs, ys)
                Dt = Dt + Bm[b0:b1] @ W_true[b0:b1]
            X = (R_true[b0:b1] @ p[b0:b1]) * Dt.transpose(1, 2) + T_true[b0:b1]
            px = fx[b0:b1] * (X[:, 0] / X[:, 2]) + ox[b0:b1]
            py = fy[b0:b1] * (X[:, 1] / X[:, 2]) + oy[b0:b1]
            conv1[b0:b1] = bilinear_zero_pad(f2, px, py)
        levels.append(SceneLevel(lid, h, w, conv1, conv2, intr, p.contiguous(), D, Bm, pts, (w, h) if n_points is None else None))
    return Scene(levels, R_true, T_true, W_true, R0, T0, W0)


@dataclass
class ResizeScene:
    """Inputs at the layer boundary of the reference's BundleResize (bundlenet.py:332-399) for dense pyramid levels: a batch of `nimg` images,
    pair b = (image b, image (b + nimg/2) % nimg) (the half swap of :386)."""
    layers: List[torch.Tensor]          # per level (coarse -> fine) [nimg,h_l,w_l,C] feature maps of every image
    basis: torch.Tensor                 # [nimg,H/2,W/2,K] depth basis of every image (as frame 1 of its pair)
    init_depth: torch.Tensor            # [nimg,H/2,W/2,1]
    intr: torch.Tensor                  # [nimg,4] fx,fy,ox,oy at the finest level
    scales: List[int]                   # per level: finest-level pixels per level pixel
    R0: torch.Tensor; T0: torch.Tensor; W0: torch.Tensor


def make_resize_scene(nimg: int, H: int, W: int, C: int, K: int, level_ids=(0, 1, 2, 3), seed: int = 1234, device="cpu", dtype=torch.float32,
                      rot_deg: float = 1.0, trans_m: float = 0.02, w_std: float = 0.02, start_trans_noise_m: float = 0.01, pair_chunk: int = 4) -> ResizeScene:
    """Planted-solution batch for the BundleResize boundary.  For the first nimg/2 pairs (b, b + nimg/2) the features of image b at every
    level are the features of image b + nimg/2 sampled at the warp of the level's pixel grid under a planted (R*, T*, D + B.W*), with D and B
    resampled from the half-resolution depth / basis maps exactly as the solver derives them; the second half of the pairs are the same
    image pairs in the opposite direction (a genuine, non-zero-residual LM problem)."""
    assert nimg % 2 == 0
    g = torch.Generator(device="cpu").manual_seed(seed)
    dev = torch.device(device)
    half = nimg // 2

    def randn(*s_):
        return torch.randn(*s_, generator=g, dtype=torch.float32).to(dev, dtype)

    def rand(*s_):
        return torch.rand(*s_, generator=g, dtype=torch.float32).to(dev, dtype)

    hb, wb = H // 2, W // 2
    intr = torch.tensor(TUM_INTRINSICS, device=dev, dtype=dtype).mul(W / 640.0).unsqueeze(0).repeat(nimg, 1)
    basis = torch.empty(nimg, hb, wb, K, device=dev, dtype=dtype)
    depth = torch.empty(nimg, hb, wb, 1, device=dev, dtype=dtype)
    for b0 in range(0, nimg, pair_chunk):
        b1 = min(nimg, b0 + pair_chunk); n = b1 - b0
        bm = gaussian_blur_nchw(randn(n, K, hb, wb), 4.0)
        basis[b0:b1] = (bm * torch.rsqrt(bm.flatten(2).var(dim=2) + 1e-3).view(n, K, 1, 1)).permute(0, 2, 3, 1)
        dm = gaussian_blur_nchw(1.0 + 2.0 * rand(n, 1, hb, wb), 4.0).permute(0, 2, 3, 1)
        dmin = dm.flatten(1).min(1).values.view(n, 1, 1, 1); dmax = dm.flatten(1).max(1).values.view(n, 1, 1, 1)
        depth[b0:b1] = 1.0 + 2.0 * (dm - dmin) / (dmax - dmin).clamp_min(1e-6)
    w_true = randn(half, 3) * math.radians(rot_deg)
    R_true = rodrigues(w_true); T_true = (randn(half, 3) * trans_m).unsqueeze(-1); W_true = (randn(half, K) * w_std).unsqueeze(-1)
    layers, scales = [], []
    for lid in level_ids:
        s_ = 2 ** (3 - lid); scales.append(s_)
        h, w = H // s_, W // s_
        feat = torch.empty(nimg, h, w, C, device=dev, dtype=dtype)
        li = intr / s_
        vv, uu = torch.meshgrid(torch.arange(h, device=dev, dtype=dtype), torch.arange(w, device=dev, dtype=dtype), indexing="ij")
        pts = torch.stack([uu.reshape(-1), vv.reshape(-1)], -1)
        for b0 in range(0, half, pair_chunk):
            b1 = min(half, b0 + pair_chunk); n = b1 - b0
            f2 = gaussian_blur_nchw(randn(n, C, h, w), 2.0)
            f2 = (f2 / f2.flatten(2).std(dim=2).clamp_min(1e-6).view(n, C, 1, 1)).permute(0, 2, 3, 1).contiguous()
            feat[half + b0:half + b1] = f2                                              # frame 2 of pair b = image b + half
            fx, fy, ox, oy = [li[b0:b1, i:i + 1] for i in range(4)]
            px_, py_ = pts[:, 0].unsqueeze(0).expand(n, -1), pts[:, 1].unsqueeze(0).expand(n, -1)
            ray = torch.stack([(px_ - ox) / fx, (py_ - oy) / fy, torch.ones_like(px_)], 1)
            p = ray / ray.norm(dim=1, keepdim=True)
            xs, ys = px_ * (s_ / 2.0), py_ * (s_ / 2.0)                                 # level pixel -> half-resolution map coordinates
            Dl = bilinear_zero_pad(depth[b0:b1].contiguous(), xs, ys)
            Bl = bilinear_zero_pad(basis[b0:b1].contiguous(), xs, ys)
            Dt = Dl + Bl @ W_true[b0:b1]
            X = (R_true[b0:b1] @ p) * Dt.transpose(1, 2) + T_true[b0:b1]
            u = fx * (X[:, 0] / X[:, 2]) + ox; v = fy * (X[:, 1] / X[:, 2]) + oy
            feat[b0:b1] = bilinear_zero_pad(f2, u, v).reshape(n, h, w, C)               # frame 1 of pair b = image b
        layers.append(feat)
    R0 = torch.eye(3, device=dev, dtype=dtype).repeat(nimg, 1, 1)
    T0 = torch.cat([T_true + randn(half, 3, 1) * start_trans_noise_m, -T_true + randn(half, 3, 1) * start_trans_noise_m], 0)
    W0 = torch.zeros(nimg, K, 1, device=dev, dtype=dtype)
    return ResizeScene(layers, basis, depth, intr, scales, R0, T0, W0)
