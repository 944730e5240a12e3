"""Drop-in for the reference's Mip-NeRF 360 renderer (models/mipnerf360/model.py:30-365), SURVEY.md section 8(a) row a18.

`MipNeRF360.forward(batch, train_frac, randomized, is_train, near, far)` returns the reference's
`(renderings: list[3] of {"rgb"}, ray_history: list[3] of {"density","rgb","sdist","weights"})` (model.py:359-365).  Parameter and
buffer names equal the reference's (`mlps.{0,1,2}.pts_linear.{i}`, `density_layer`, `bottleneck_layer`, `views_linear.0`,
`rgb_layer`, `pos_basis_t`).  Arithmetic: fp32 CUDA cores in the reference formulation (csrc/mip.cu); CUDA only."""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Tuple

import torch
import torch.nn as nn

from . import _lib as L
from .mip_basis import POS_BASIS_T


class MipNeRF360MLP(nn.Module):
    def __init__(self, netdepth: int = 8, netwidth: int = 256, disable_rgb: bool = False):
        super().__init__()
        self.netdepth, self.netwidth, self.disable_rgb = netdepth, netwidth, disable_rgb
        self.register_buffer("pos_basis_t", POS_BASIS_T.clone())
        pos = 12 * 2 * 21
        layers = [nn.Linear(pos, netwidth)]
        for idx in range(netdepth - 1):
            layers.append(nn.Linear(netwidth + pos if (idx % 4 == 0 and idx > 0) else netwidth, netwidth))
        self.pts_linear = nn.ModuleList(layers)
        self.density_layer = nn.Linear(netwidth, 1)
        if not disable_rgb:
            self.bottleneck_layer = nn.Linear(netwidth, 256)
            self.views_linear = nn.ModuleList([nn.Linear(256 + 27, 128)])
            self.rgb_layer = nn.Linear(128, 3)
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.kaiming_uniform_(m.weight)

    def c_params(self, keep: list) -> L.NeoMipMLPParams:
        p = L.NeoMipMLPParams()
        f = lambda t: (keep.append(t.detach().contiguous().float()) or keep[-1])
        p.depth, p.width = self.netdepth, self.netwidth
        p.basis = L.ptr(f(self.pos_basis_t))
        for i in range(self.netdepth):
            p.w[i] = L.ptr(f(self.pts_linear[i].weight))
            p.b[i] = L.ptr(f(self.pts_linear[i].bias))
        p.wsig, p.bsig = L.ptr(f(self.density_layer.weight)), L.ptr(f(self.density_layer.bias))
        if not self.disable_rgb:
            p.wb, p.bb = L.ptr(f(self.bottleneck_layer.weight)), L.ptr(f(self.bottleneck_layer.bias))
            p.wv0, p.bv0 = L.ptr(f(self.views_linear[0].weight)), L.ptr(f(self.views_linear[0].bias))
            p.wrgb, p.brgb = L.ptr(f(self.rgb_layer.weight)), L.ptr(f(self.rgb_layer.bias))
        return p


class NeRFMLP(MipNeRF360MLP):
    def __init__(self, netdepth: int = 8, netwidth: int = 1024):
        super().__init__(netdepth=netdepth, netwidth=netwidth)


class PropMLP(MipNeRF360MLP):
    def __init__(self, netdepth: int = 4, netwidth: int = 256):
        super().__init__(netdepth=netdepth, netwidth=netwidth, disable_rgb=True)


class MipNeRF360(nn.Module):
    def __init__(self, num_prop_samples: int = 64, num_nerf_samples: int = 32, num_levels: int = 3, precision: str = "fp32",
                 **reference_defaults):
        super().__init__()
        self.precision = precision          # "fp32": CUDA-core SGEMM chain (tight parity); "tc": every dense layer on the tensor cores (fp16 operands)
        if num_levels != 3 or reference_defaults:
            raise NotImplementedError("reference defaults only (models/mipnerf360/model.py:199-223)")
        self.num_prop_samples, self.num_nerf_samples = num_prop_samples, num_nerf_samples
        self.mlps = nn.ModuleList([PropMLP(), PropMLP(), NeRFMLP()])
        self._ws = None

    def forward(self, batch: Dict[str, torch.Tensor], train_frac: float, randomized: bool, is_train: bool, near, far) -> Tuple[List[dict], List[dict]]:
        if torch.is_grad_enabled() and self.training and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("backward through the CUDA path is not built yet; call under torch.no_grad() / .eval()")
        o = batch["rays_o"].contiguous().float()
        if not o.is_cuda:
            raise RuntimeError("neo360_b200 needs CUDA tensors (no CPU fallback)")
        d, vd = batch["rays_d"].contiguous().float(), batch["viewdirs"].contiguous().float()
        radii = batch["radii"].reshape(-1).contiguous().float()
        lib = L.load()
        n, dev = o.shape[0], o.device
        keep = []
        arr = (L.NeoMipMLPParams * 3)(*[m.to(dev).c_params(keep) for m in self.mlps])
        cfg = L.NeoMipCfg()
        cfg.n_prop, cfg.n_nerf = self.num_prop_samples, self.num_nerf_samples
        cfg.near_plane, cfg.far_plane, cfg.train_frac = float(near), float(far), float(train_frac)
        cfg.precision = {"fp32": L.NEO_PREC_FP32, "tc": L.NEO_PREC_TC}[self.precision]
        if randomized:
            jit = batch.get("_uniforms") or [torch.rand((n, 1), device=dev) for _ in range(3)]     # helper.py:361 (single_jitter)
            for i in range(3):
                j = jit[i].reshape(-1).contiguous()
                keep.append(j)
                cfg.jitter[i] = j.data_ptr()
        need = lib.neo_mip_workspace_bytes(n, C.byref(cfg), self.mlps[2].netwidth)
        if need == 0:
            raise RuntimeError("neo360_b200: " + lib.neo_last_error().decode())
        if self._ws is None or self._ws.numel() < need or self._ws.device != dev:
            self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
        ns = (cfg.n_prop, cfg.n_prop, cfg.n_nerf)
        out = L.NeoMipOut()
        ren, hist = [], []
        for l in range(3):
            T = {"rgb": torch.empty(n, 3, device=dev), "density": torch.empty(n, ns[l], device=dev), "rgb_s": torch.empty(n, ns[l], 3, device=dev),
                 "sdist": torch.empty(n, ns[l] + 1, device=dev), "weights": torch.empty(n, ns[l], device=dev)}
            for k, t in T.items():
                getattr(out, k)[l] = t.data_ptr()
            ren.append({"rgb": T["rgb"]})
            hist.append({"density": T["density"], "rgb": T["rgb_s"], "sdist": T["sdist"], "weights": T["weights"]})
        with torch.cuda.device(dev):
            L.check(lib.neo_mip_render_fwd(arr, L.ptr(o), L.ptr(d), L.ptr(vd), L.ptr(radii), n, C.byref(cfg), C.byref(out), self._ws.data_ptr(),
                                           self._ws.numel(), torch.cuda.current_stream().cuda_stream))
        return ren, hist
