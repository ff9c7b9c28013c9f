"""Solve frame-pairs whose level tensors live in host memory: the call a user makes when the feature pyramid comes off a
data loader / another process.  Mirrors the layer boundary of the reference's `BundleResize` (bundlenet.py:376-399): feature
maps in, `[F2|gx|gy]` derived on the device (:386-389), coarse-to-fine LM solve (:376-399), (R, T, W) out.

Pairs are independent, so the batch is cut into chunks: the host->device copies of chunk k+1 (copy stream, pinned buffers)
overlap the solve of chunk k (compute stream); the PCIe transfer is the long pole (20 GB per 32-pair cfg2 batch vs 51 ms of
compute), so the solve hides behind it except for the last chunk.  No CPU fallback: everything after the copy is the C-ABI."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import ops
from ._lib import PREC_AUTO

Tensor = torch.Tensor
_NAMES = ("conv1", "conv2", "intr", "p", "D", "B")


def chunk_ranges(nb: int, chunks: int) -> List[Tuple[int, int]]:
    """Contiguous, balanced pair ranges (first ranges one longer); never empty ranges."""
    chunks = max(1, min(int(chunks), int(nb)))
    base, rem = divmod(nb, chunks)
    out, a = [], 0
    for c in range(chunks):
        b = a + base + (1 if c < rem else 0)
        out.append((a, b)); a = b
    return out



class numa_local_to:
    """Context manager: while it is active the calling thread runs on the CPUs of the NUMA node the given GPU hangs off, so that host buffers
    allocated (and pinned) inside it are placed in the memory next to that GPU's PCIe root (first-touch placement).  With several GPUs per
    host this keeps every rank's host->device traffic off the inter-socket link.  Restores the previous affinity on exit.  A no-op (with
    `.info` saying why) when the topology cannot be read — it never fails the caller."""

    def __init__(self, device, _bdf: Optional[str] = None, _sysfs: str = "/sys"):
        self.device = torch.device(device)
        self.info = {"node": None, "cpus": None, "note": "not applied"}
        self._saved = None
        self._bdf, self._sysfs = _bdf, _sysfs                      # test hooks: PCI address and sysfs root

    def __enter__(self):
        import os
        try:
            bdf = self._bdf
            if bdf is None:
                pr = torch.cuda.get_device_properties(self.device)
                bdf = "%04x:%02x:%02x.0" % (int(pr.pci_domain_id), int(pr.pci_bus_id), int(pr.pci_device_id))
            node = int(open(f"{self._sysfs}/bus/pci/devices/{bdf}/numa_node").read().strip())
            if node < 0:
                self.info["note"] = f"{bdf}: numa_node unknown (-1)"
                return self
            cpus = set()
            for part in open(f"{self._sysfs}/devices/system/node/node{node}/cpulist").read().strip().split(","):
                a, _, b = part.partition("-")
                cpus.update(range(int(a), int(b or a) + 1))
            self._saved = os.sched_getaffinity(0)
            use = cpus & self._saved
            if not use:
                self.info["note"] = f"node {node}: none of its CPUs is in this process's affinity mask"
                self._saved = None
                return self
            os.sched_setaffinity(0, use)
            self.info = {"node": node, "cpus": len(use), "note": f"{bdf}: host buffers allocated on NUMA node {node}"}
        except Exception as ex:                                    # sysfs not mounted, property missing, permission: stay as we are
            self.info["note"] = f"topology unavailable ({type(ex).__name__})"
            self._saved = None
        return self

    def __exit__(self, *exc):
        import os
        if self._saved is not None:
            try:
                os.sched_setaffinity(0, self._saved)
            except Exception:
                pass
        return False

class HostSolver:
    """host_levels: one dict per level (coarse -> fine) with host tensors conv1 [nb,N,C], conv2 [nb,h,w,C] (features; gradients
    are derived on the device) or [nb,h,w,3C] (already [F2|gx|gy]) when derive_gradients=False, intr [nb,4], p [nb,3,N],
    D [nb,N,1], B [nb,N,K], and optionally grid=(w,h).  Pinned host tensors make the copies asynchronous."""

    def __init__(self, host_levels: Sequence[Dict], derive_gradients: bool = True, chunks: int = 4, device=None,
                 precision: int = PREC_AUTO):
        self.dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.host = list(host_levels)
        self.derive = bool(derive_gradients)
        self.precision = precision
        self.nb = int(self.host[0]["conv1"].shape[0])
        self.ranges = chunk_ranges(self.nb, chunks)
        self.copy_stream = torch.cuda.Stream(self.dev)
        self.compute_stream = torch.cuda.Stream(self.dev)
        self.dev_levels: List[Dict[str, Tensor]] = []
        self.h2d_bytes = 0
        for hl in self.host:
            d = {}
            for name in _NAMES:
                t = hl.get(name)
                if t is None:                     # pose-only levels carry no basis
                    d[name] = None
                    continue
                d[name] = torch.empty(t.shape, dtype=torch.float32, device=self.dev)
                self.h2d_bytes += t.numel() * 4
            if self.derive:                       # staging of the feature maps; conv2 on the device is the 3C tensor
                C = hl["conv2"].shape[-1]
                d["feat"] = d["conv2"]
                d["conv2"] = torch.empty(*hl["conv2"].shape[:-1], 3 * C, dtype=torch.float32, device=self.dev)
            self.dev_levels.append(d)
        self._ws: Optional[Tensor] = None

    def _levels(self, a: int, b: int) -> List[ops.Level]:
        return [ops.Level(d["conv1"][a:b], d["conv2"][a:b], d["intr"][a:b], d["p"][a:b], d["D"][a:b], None if d["B"] is None else d["B"][a:b], grid=hl.get("grid"))
                for d, hl in zip(self.dev_levels, self.host)]

    def solve(self, R0: Tensor, T0: Tensor, W0: Tensor, iters_per_level: int, mlp_packed=None, l2_regularizer_base: float = 1000.0,
              lambda_fixed: float = -1.0, out: Optional[Tuple[Tensor, Tensor, Tensor]] = None):
        """R0 [nb,3,3], T0 [nb,3,1], W0 [nb,K,1] on the host (pinned for async copies).  Returns device (R, T, W, status); when
        `out` = three host tensors is given they receive the results too (device->host inside the pipeline)."""
        nb, dev = self.nb, self.dev
        R = torch.empty(nb, 3, 3, device=dev); T = torch.empty(nb, 3, 1, device=dev)
        W = None if W0 is None else torch.empty(W0.shape, device=dev)
        status = torch.empty(nb, dtype=torch.int32, device=dev)
        dR = torch.empty_like(R); dT = torch.empty_like(T); dW = None if W is None else torch.empty_like(W)
        self.copy_stream.wait_stream(torch.cuda.current_stream(dev))
        self.compute_stream.wait_stream(torch.cuda.current_stream(dev))
        events = []
        with torch.cuda.stream(self.copy_stream):
            for a, b in self.ranges:
                for d, hl in zip(self.dev_levels, self.host):
                    for name in _NAMES:
                        dst = d["feat"] if (name == "conv2" and self.derive) else d[name]
                        if dst is not None:
                            dst[a:b].copy_(hl[name][a:b], non_blocking=True)
                dR[a:b].copy_(R0[a:b], non_blocking=True); dT[a:b].copy_(T0[a:b], non_blocking=True); (dW is not None) and dW[a:b].copy_(W0[a:b], non_blocking=True)
                ev = torch.cuda.Event(); ev.record(self.copy_stream); events.append(ev)
        with torch.cuda.stream(self.compute_stream):
            for (a, b), ev in zip(self.ranges, events):
                self.compute_stream.wait_event(ev)
                if self.derive:
                    for d in self.dev_levels:
                        ops.grad_fixed_concat(d["feat"][a:b], out=d["conv2"][a:b])
                lv = self._levels(a, b)
                if self._ws is None:
                    self._ws = torch.empty(ops.lm_run_workspace_bytes(lv, self.precision), dtype=torch.uint8, device=dev)
                r, t, w, st = ops.lm_run(lv, iters_per_level, dR[a:b], dT[a:b], None if dW is None else dW[a:b], mlp_packed=mlp_packed,
                                         l2_regularizer_base=l2_regularizer_base, lambda_fixed=lambda_fixed, workspace=self._ws,
                                         precision=self.precision)
                R[a:b] = r; T[a:b] = t; status[a:b] = st
                if W is not None:
                    W[a:b] = w
                if out is not None:
                    out[0][a:b].copy_(r, non_blocking=True); out[1][a:b].copy_(t, non_blocking=True)
                    if W is not None:
                        out[2][a:b].copy_(w, non_blocking=True)
        torch.cuda.current_stream(dev).wait_stream(self.compute_stream)
        for t_ in (R, T, W, status, dR, dT, dW):
            if t_ is not None:
                t_.record_stream(self.compute_stream)
        return R, T, W, status


class ResizeHostSolver:
    """The reference's `BundleResize` boundary (bundlenet.py:332-399) with HOST inputs, for dense pyramid levels: a batch of `nimg` images
    comes in as feature maps `layers[l]` [nimg,h_l,w_l,C] (coarse -> fine), half-resolution `basis` [nimg,H/2,W/2,K] and `init_depth`
    [nimg,H/2,W/2,1] and finest-level intrinsics `intr` [nimg,4]; pair b = (image b, image (b + nimg/2) % nimg) (:386).  Everything the
    reference derives in its graph is derived on the device, nothing derivable crosses PCIe:
        conv1 = layers[l] itself (the points are the level's own pixel grid, so resampler(layers[l], points) is the identity: zero copy);
        conv2 = the other half of the same buffer, F2 only (gradients on the fly in the build kernel, bundlenet.py:92-100, 386-389);
        p = computeCoordinates(points_l, intr / scale_l) (:358);  D, B = resampler(init_depth | basis, points / 2) (:343-344).
    Pairs are cut into chunks inside each half of the batch; the H2D copies of the images a later chunk needs overlap the solve of the
    current one (copy stream / compute stream).
    The pyramid keeps the host layers' dtype on the device: a bfloat16 pyramid (an autocast encoder's output) is copied at 2 bytes per
    element and solved as bfloat16 levels.  So does the basis, independently: a bfloat16 host basis is copied at 2 bytes per element and
    sampled by banet_resample_bf16 into bfloat16 levels.  Depth and intrinsics are float32.  `h2d_bytes` counts the real element sizes."""

    def __init__(self, layers: Sequence[Tensor], basis: Tensor, init_depth: Tensor, intr: Tensor, scales: Sequence[int], chunks: int = 4,
                 device=None, precision: int = PREC_AUTO):
        self.dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.h_layers = list(layers); self.h_basis = basis; self.h_depth = init_depth; self.h_intr = intr
        self.scales = [int(s) for s in scales]
        self.precision = precision
        self.nimg = int(basis.shape[0]); self.half = self.nimg // 2
        if self.nimg % 2:
            raise ValueError("the half-swap pairing of bundlenet.py:386 needs an even batch")
        # chunk order: (pairs a..b of the first half) then (the same image set in the other direction, pairs a+half..b+half): both read images
        # a..b and a+half..b+half, so each image set is copied once and two chunks of compute follow it; the copies of the next set overlap them
        per_half = max(1, int(chunks) // 2)
        self.ranges = [(o + a, o + b) for a, b in chunk_ranges(self.half, per_half) for o in (0, self.half)]
        self.copy_stream = torch.cuda.Stream(self.dev); self.compute_stream = torch.cuda.Stream(self.dev)
        dev = self.dev
        fdt = self.h_layers[0].dtype
        if fdt not in (torch.float32, torch.bfloat16) or any(t.dtype != fdt for t in self.h_layers):
            raise ValueError(f"layers must all be float32 or all bfloat16; got {[t.dtype for t in self.h_layers]}")
        self.d_layers = [torch.empty(t.shape, dtype=fdt, device=dev) for t in self.h_layers]
        if basis.dtype not in (torch.float32, torch.bfloat16):
            raise ValueError(f"basis must be float32 or bfloat16; got {basis.dtype}")
        self.d_basis = torch.empty(basis.shape, dtype=basis.dtype, device=dev)
        self.d_depth = torch.empty(init_depth.shape, dtype=torch.float32, device=dev)
        self.d_intr = torch.empty(intr.shape, dtype=torch.float32, device=dev)
        self.h2d_bytes = sum(t.numel() * t.element_size() for t in (*self.h_layers, basis, init_depth, intr))
        self.K = int(basis.shape[-1]); self.C = int(self.h_layers[0].shape[-1])
        nmax = max(b - a for a, b in self.ranges)
        self.pts, self.scr = [], []
        for t, s in zip(self.h_layers, self.scales):                      # per level: dense pixel grid + scratch for the derived tensors of one chunk
            h, w = int(t.shape[1]), int(t.shape[2]); N = h * w
            vv, uu = torch.meshgrid(torch.arange(h, device=dev, dtype=torch.float32), torch.arange(w, device=dev, dtype=torch.float32), indexing="ij")
            self.pts.append(torch.stack([uu.reshape(-1), vv.reshape(-1)], -1).unsqueeze(0).repeat(nmax, 1, 1).contiguous())
            self.scr.append({"B": torch.empty(nmax, N, self.K, dtype=basis.dtype, device=dev), "D": torch.empty(nmax, N, 1, device=dev), "p": torch.empty(nmax, 3, N, device=dev)})
        self._ws: Optional[Tensor] = None

    def _chunk_levels(self, a: int, b: int) -> List[ops.Level]:
        n = b - a
        a2 = (a + self.half) % self.nimg
        lib = ops.load()
        levels = []
        for l, (dl, s) in enumerate(zip(self.d_layers, self.scales)):
            h, w = int(dl.shape[1]), int(dl.shape[2]); N = h * w
            pts = self.pts[l][:n]; scr = self.scr[l]
            intr_l = (self.d_intr[a:b] / float(s)).contiguous()
            ops.check(lib.banet_compute_coordinates(pts.data_ptr(), intr_l.data_ptr(), n, N, 1, scr["p"].data_ptr(), ops._stream()), "banet_compute_coordinates")
            ops.check(lib.banet_resample(self.d_depth[a:b].data_ptr(), pts.data_ptr(), s / 2.0, n, int(self.d_depth.shape[1]), int(self.d_depth.shape[2]), 1, N,
                                         scr["D"].data_ptr(), ops._stream()), "banet_resample")
            rs = "banet_resample_bf16" if self.d_basis.dtype == torch.bfloat16 else "banet_resample"
            ops.check(getattr(lib, rs)(self.d_basis[a:b].data_ptr(), pts.data_ptr(), s / 2.0, n, int(self.d_basis.shape[1]), int(self.d_basis.shape[2]), self.K, N,
                                       scr["B"].data_ptr(), ops._stream()), rs)
            levels.append(ops.Level(dl[a:b].reshape(n, N, self.C), dl[a2:a2 + n], intr_l, scr["p"][:n], scr["D"][:n], scr["B"][:n], grid=(w, h)))
        return levels

    def solve(self, R0: Tensor, T0: Tensor, W0: Tensor, iters_per_level: int, mlp_packed=None, l2_regularizer_base: float = 1000.0,
              lambda_fixed: float = -1.0, out: Optional[Tuple[Tensor, Tensor, Tensor]] = None):
        """R0 [nimg,3,3], T0 [nimg,3,1], W0 [nimg,K,1] on the host.  Returns device (R, T, W, status); `out` = three host tensors receive them too."""
        nimg, dev = self.nimg, self.dev
        R = torch.empty(nimg, 3, 3, device=dev); T = torch.empty(nimg, 3, 1, device=dev); W = torch.empty(W0.shape, device=dev)
        status = torch.empty(nimg, dtype=torch.int32, device=dev)
        dR = torch.empty_like(R); dT = torch.empty_like(T); dW = torch.empty_like(W)
        cur = torch.cuda.current_stream(dev)
        self.copy_stream.wait_stream(cur); self.compute_stream.wait_stream(cur)
        events, resident = [], set()
        with torch.cuda.stream(self.copy_stream):
            self.d_intr.copy_(self.h_intr, non_blocking=True)
            for a, b in self.ranges:
                a2 = (a + self.half) % nimg
                for lo, hi in ((a, b), (a2, a2 + (b - a))):                  # images this chunk reads (frame 1, frame 2) that are not on the device yet
                    if (lo, hi) in resident:
                        continue
                    resident.add((lo, hi))
                    for dl, hl in zip(self.d_layers, self.h_layers):
                        dl[lo:hi].copy_(hl[lo:hi], non_blocking=True)
                self.d_basis[a:b].copy_(self.h_basis[a:b], non_blocking=True); self.d_depth[a:b].copy_(self.h_depth[a:b], non_blocking=True)
                dR[a:b].copy_(R0[a:b], non_blocking=True); dT[a:b].copy_(T0[a:b], non_blocking=True); dW[a:b].copy_(W0[a:b], non_blocking=True)
                ev = torch.cuda.Event(); ev.record(self.copy_stream); events.append(ev)
        with torch.cuda.stream(self.compute_stream):
            for (a, b), ev in zip(self.ranges, events):
                self.compute_stream.wait_event(ev)
                lv = self._chunk_levels(a, b)
                if self._ws is None:
                    self._ws = torch.empty(ops.lm_run_workspace_bytes(lv, self.precision), dtype=torch.uint8, device=dev)
                r, t, w, st = ops.lm_run(lv, iters_per_level, dR[a:b], dT[a:b], dW[a:b], mlp_packed=mlp_packed, l2_regularizer_base=l2_regularizer_base,
                                         lambda_fixed=lambda_fixed, workspace=self._ws, precision=self.precision)
                R[a:b] = r; T[a:b] = t; W[a:b] = w; status[a:b] = st
                if out is not None:
                    out[0][a:b].copy_(r, non_blocking=True); out[1][a:b].copy_(t, non_blocking=True); out[2][a:b].copy_(w, non_blocking=True)
        cur.wait_stream(self.compute_stream)
        for t_ in (R, T, W, status, dR, dT, dW):
            t_.record_stream(self.compute_stream)
        return R, T, W, status
