"""How often do the two pixels of a gather unit share a bilinear tap column?  (CPU; bounds the gain of lm_build_tc6_kernel's shared-column
load path.)

    python scripts/count_tap_sharing.py [--motion default|large] [--nb 32] [--out profiles/tap_sharing_default.json]

The scene is bench.py's cfg2 scene (nb = 32, 640x480 at the finest of four levels, C = K = 128, seed 1234 + 2; `--motion large` is bench.py's
4 deg / 8 cm).  Only its geometry is needed (p, D, B, intrinsics, poses), so the script replays synth.make_scene's random stream and skips
the feature maps; `--check` first proves the replay equal to synth.make_scene at a small size.  Pixels are projected in float64 with the
reference's warp (bundlenet.py:209-224: X = R p (D + B W) + T, u = fx X/Z + ox, v = fy Y/Z + oy) at two iterates: the start of the solve
(R0, T0, W0) and the planted solution, where the solve ends.

In lm_build_tc6_kernel a gather warp walks one 8-pixel row of an 8 x 8 tile, two pixels at a time: pixel 2k on half-warp 0 and 2k+1 on
half-warp 1, each with taps (x0, y0), (x1, y0), (x0, y1), (x1, y1) and 3 components [F2 | gx | gy] per texel.  Per level the script counts
  - share: of the pairs whose two pixels are both in bounds, the fraction whose right tap column of pixel 2k is the left tap column of
    pixel 2k+1 (o_2k.y == o_2k+1.x and o_2k.w == o_2k+1.z in the kernel's records): those load 18 texel-chunks instead of 24;
  - chunks_per_pair: the texel-chunks the gather requests per such pair, before (24) and with the shared column loaded once;
  - distinct_per_pair_in_tile: the distinct texel-chunks of a whole tile per pair (what an ideal per-tile cache would fetch).
"""
import argparse, json, math, os, sys

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from banet_b200 import synth                                      # noqa: E402

H_FULL, W_FULL, LEVEL_IDS, SEED = 480, 640, (0, 1, 2, 3), 1234 + 2
MOTION = {"default": {}, "large": dict(rot_deg=4.0, trans_m=0.08, start_trans_noise_m=0.02)}


def scene_geometry(nb, H, W, C, K, level_ids, seed, rot_deg=1.0, trans_m=0.02, w_std=0.02, start_trans_noise_m=0.01, pair_chunk=4):
    """synth.make_scene's draws in its order (dense grid, no shared depth), keeping p, D, B, intr and the poses only."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    randn = lambda *s: torch.randn(*s, generator=g, dtype=torch.float32)
    rand = lambda *s: torch.rand(*s, generator=g, dtype=torch.float32)
    R_true = synth.rodrigues(randn(nb, 3) * math.radians(rot_deg))
    T_true = (randn(nb, 3) * trans_m).unsqueeze(-1)
    W_true = (randn(nb, K) * w_std).unsqueeze(-1)
    R0, T0, W0 = torch.eye(3).repeat(nb, 1, 1), T_true + randn(nb, 3, 1) * start_trans_noise_m, torch.zeros(nb, K, 1)
    levels = []
    for lid in level_ids:
        scale = 2 ** (3 - lid)
        h, w = H // scale, W // scale
        intr = (torch.tensor(synth.TUM_INTRINSICS, dtype=torch.float32) * (W / 640.0) / scale).unsqueeze(0).repeat(nb, 1)
        vv, uu = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
        pts = torch.stack([uu.reshape(-1), vv.reshape(-1)], -1).unsqueeze(0).repeat(nb, 1, 1)
        fx, fy, ox, oy = [intr[:, i:i + 1] for i in range(4)]
        ray = torch.stack([(pts[..., 0] - ox) / fx, (pts[..., 1] - oy) / fy, torch.ones_like(pts[..., 0])], 1)
        p = ray / ray.norm(dim=1, keepdim=True)
        N = pts.shape[1]
        D, Bm = torch.empty(nb, N, 1), torch.empty(nb, N, K)
        sig_b = max(1.0, 8.0 / scale)
        for b0 in range(0, nb, pair_chunk):
            b1 = min(nb, b0 + pair_chunk)
            n = b1 - b0
            randn(n, C, h, w)                                     # the feature maps' draw (not needed here)
            dmap = synth.gaussian_blur_nchw(1.0 + 2.0 * rand(n, 1, h, w), sig_b).permute(0, 2, 3, 1)
            dmin = dmap.flatten(1).min(1).values.view(n, 1, 1, 1); dmax = dmap.flatten(1).max(1).values.view(n, 1, 1, 1)
            dmap = 1.0 + 2.0 * (dmap - dmin) / (dmax - dmin).clamp_min(1e-6)
            xs, ys = pts[b0:b1, :, 0], pts[b0:b1, :, 1]
            D[b0:b1] = synth.bilinear_zero_pad(dmap.contiguous(), xs, ys)
            bm = synth.gaussian_blur_nchw(randn(n, K, h, w), sig_b)
            bm = bm * torch.rsqrt(bm.flatten(2).var(dim=2) + 1e-3).view(n, K, 1, 1)
            Bm[b0:b1] = synth.bilinear_zero_pad(bm.permute(0, 2, 3, 1).contiguous(), xs, ys)
        levels.append(dict(h=h, w=w, intr=intr, p=p, D=D, B=Bm))
    return levels, {"start": (R0, T0, W0), "planted": (R_true, T_true, W_true)}


def count_level(lv, R, T, W):
    f64 = torch.float64
    h, w = lv["h"], lv["w"]
    nb = lv["p"].shape[0]
    Dt = lv["D"].to(f64) + lv["B"].to(f64) @ W.to(f64)
    fx, fy, ox, oy = [lv["intr"][:, i:i + 1].to(f64) for i in range(4)]
    X = (R.to(f64) @ lv["p"].to(f64)) * Dt.transpose(1, 2) + T.to(f64)          # [nb,3,N]
    Z = X[:, 2]
    px, py = fx * (X[:, 0] / Z) + ox, fy * (X[:, 1] / Z) + oy
    valid = (px >= 0) & (px <= w - 1) & (py >= 0) & (py <= h - 1) & torch.isfinite(1.0 / Z)
    x0 = torch.where(valid, torch.floor(px), torch.zeros_like(px)).long()
    y0 = torch.where(valid, torch.floor(py), torch.zeros_like(py)).long()
    x1, y1 = (x0 + 1).clamp(max=w - 1), (y0 + 1).clamp(max=h - 1)
    taps = torch.stack([y0 * w + x0, y0 * w + x1, y1 * w + x0, y1 * w + x1], -1).view(nb, h, w, 4)     # texel index of o.x .. o.w
    valid = valid.view(nb, h, w)
    # pixels padded to whole 8 x 8 tiles (pixels outside the map are masked, as in the kernel)
    th, tw = -(-h // 8) * 8, -(-w // 8) * 8
    tp = torch.zeros(nb, th, tw, 4, dtype=torch.long); tp[:, :h, :w] = taps
    vp = torch.zeros(nb, th, tw, dtype=torch.bool); vp[:, :h, :w] = valid
    a, b = tp[:, :, 0::2], tp[:, :, 1::2]                         # pixel 2k and 2k+1 of every gather row
    va, vb = vp[:, :, 0::2], vp[:, :, 1::2]
    both = va & vb
    share = both & (a[..., 1] == b[..., 0]) & (a[..., 3] == b[..., 2])
    n_both, n_share = int(both.sum()), int(share.sum())
    # distinct texels per tile (x3 components): union over the tile's valid pixels
    tiles = tp.view(nb, th // 8, 8, tw // 8, 8, 4).permute(0, 1, 3, 2, 4, 5).reshape(-1, 256)
    tv = vp.view(nb, th // 8, 8, tw // 8, 8).permute(0, 1, 3, 2, 4).reshape(-1, 64).repeat_interleave(4, 1)
    ids = torch.where(tv, tiles, torch.full_like(tiles, -1))
    srt = ids.sort(1).values
    distinct = int(((srt[:, 1:] != srt[:, :-1]) & (srt[:, 1:] >= 0)).sum() + (srt[:, 0] >= 0).sum())
    n_valid_px = int(vp.sum())
    pairs_px = n_valid_px / 2.0
    return {"level": f"{w}x{h}", "pixels_in_bounds": n_valid_px, "pairs_both_in_bounds": n_both,
            "share": n_share / max(n_both, 1),
            "chunks_per_pair": {"before": 24.0, "shared_column_once": 24.0 - 6.0 * n_share / max(n_both, 1)},
            "distinct_per_pair_in_tile": 3.0 * distinct / max(pairs_px, 1.0)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--motion", default="default", choices=list(MOTION))
    ap.add_argument("--nb", type=int, default=32)
    ap.add_argument("--out", default=None)
    ap.add_argument("--check", action="store_true", help="first prove the replayed geometry equal to synth.make_scene at a small size")
    a = ap.parse_args()
    if a.check:
        sc = synth.make_scene(nb=5, H=48, W=64, C=8, K=16, level_ids=(2, 3), seed=11, **MOTION[a.motion])
        lv, it = scene_geometry(5, 48, 64, 8, 16, (2, 3), 11, **MOTION[a.motion])
        for s, r in zip(sc.levels, lv):
            assert torch.equal(s.p, r["p"]) and torch.equal(s.D, r["D"]) and torch.equal(s.B, r["B"]) and torch.equal(s.intr, r["intr"])
        assert torch.equal(sc.T0, it["start"][1]) and torch.equal(sc.R_true, it["planted"][0]) and torch.equal(sc.W_true, it["planted"][2])
        print("replayed geometry equals synth.make_scene", flush=True)
    levels, iterates = scene_geometry(a.nb, H_FULL, W_FULL, 128, 128, LEVEL_IDS, SEED, **MOTION[a.motion])
    report = {"scene": f"bench.py cfg2 geometry, nb={a.nb}, motion={a.motion}", "iterates": {}}
    for name, (R, T, W) in iterates.items():
        rows = [count_level(lv, R, T, W) for lv in levels]
        report["iterates"][name] = rows
        for r in rows:
            print(f"{name:8s} {r['level']:8s} share {r['share']:.3f}  chunks/pair 24 -> {r['chunks_per_pair']['shared_column_once']:.2f}  "
                  f"distinct in tile per pair {r['distinct_per_pair_in_tile']:.2f}", flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
