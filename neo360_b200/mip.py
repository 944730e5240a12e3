"""Drop-in for the reference's Mip-NeRF 360 renderer (models/mipnerf360/model.py:30-365), SURVEY.md section 8(a) row a18.

`MipNeRF360.forward(batch, train_frac, randomized, is_train, near, far)` returns the reference's
`(renderings: list[3] of {"rgb"}, ray_history: list[3] of {"density","rgb","sdist","weights"})` (model.py:359-365).  Parameter and
buffer names equal the reference's (`mlps.{0,1,2}.pts_linear.{i}`, `density_layer`, `bottleneck_layer`, `views_linear.0`,
`rgb_layer`, `pos_basis_t`).  Arithmetic (csrc/mip.cu): `precision = "fp32"` (default) runs the MLPs as fp32 CUDA-core SGEMMs in the
reference formulation; `"tc"` runs every dense layer on the tensor cores (fp16 operands).  CUDA only, no CPU fallback.

Training: with autograd on, the module in train mode and parameters that require grad, `MipNeRF360.forward` returns the same
`(renderings, ray_history)` differentiable w.r.t. every MLP parameter (LitMipNeRF360.training_step, model.py:427-456): `density`, `rgb`
and `weights` of every level and each level's rendered `rgb` carry gradients, `sdist` is detached (model.py:309-310) and the proposal
levels' `rgb` are zeros.  Resampling, IPE features, direction encoding and compositing forward and backward are hand-written CUDA; the
dense layers are framework fp32 GEMMs under autograd, or with `train_precision="tc"` bf16 tensor-core GEMMs forward and backward
(training._MLPTrainTC, csrc/dense_train.cu).  `precision` applies to inference only.
`training_loss` is the reference's training loss on those outputs.
Ray gradients, as the reference's plain-PyTorch module has them: when grad is enabled and a ray tensor requires grad, `forward` takes the
autograd path (also with frozen parameters or in eval mode).  `viewdirs` gets the gradient of its direction encoding (`neo_mip_encode_bwd`)
and `rays_d` that of the |rays_d| scaling of the intervals (`neo_mip_composite_bwd_rays_d`).  The reference's `contract` returns detached
Gaussians (models/mipnerf360/helper.py:63-66), so, as there, `rays_o` and `radii` get no gradient and `rays_d` none through the frustums
(DESIGN.md section 12)."""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib as L
from .mip_basis import POS_BASIS_T
from .training import check_train_precision, distortion_loss, mlp_train_tc, rays_need_grad


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
                 train_precision: str = "fp32", **reference_defaults):
        super().__init__()
        self.train_precision = check_train_precision(train_precision)   # "fp32": framework GEMMs; "tc": bf16 tensor cores (training only)
        self.precision = precision          # "fp32": CUDA-core SGEMM chain (tight parity); "tc": every dense layer on the tensor cores (fp16 operands)
        if num_levels != 3 or reference_defaults:
            raise NotImplementedError("reference defaults only (models/mipnerf360/model.py:199-223)")
        self.num_prop_samples, self.num_nerf_samples = num_prop_samples, num_nerf_samples
        self.mlps = nn.ModuleList([PropMLP(), PropMLP(), NeRFMLP()])
        self._ws = None

    def forward(self, batch: Dict[str, torch.Tensor], train_frac: float, randomized: bool, is_train: bool, near, far) -> Tuple[List[dict], List[dict]]:
        if torch.is_grad_enabled() and ((self.training and any(p.requires_grad for p in self.parameters())) or rays_need_grad(batch)):
            return self._forward_train(batch, train_frac, randomized, near, far)
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
                cfg.jitter[i] = L.ptr(j)
        self._ws = L.grow(self._ws, lib.neo_mip_workspace_bytes(n, C.byref(cfg), self.mlps[2].netwidth), dev)
        ns = (cfg.n_prop, cfg.n_prop, cfg.n_nerf)
        out = L.NeoMipOut()
        ren, hist = [], []
        for l in range(3):
            T = {"rgb": torch.empty(n, 3, device=dev), "density": torch.empty(n, ns[l], device=dev), "rgb_s": torch.empty(n, ns[l], 3, device=dev),
                 "sdist": torch.empty(n, ns[l] + 1, device=dev), "weights": torch.empty(n, ns[l], device=dev)}
            for k, t in T.items():
                getattr(out, k)[l] = L.ptr(t)
            ren.append({"rgb": T["rgb"]})
            hist.append({"density": T["density"], "rgb": T["rgb_s"], "sdist": T["sdist"], "weights": T["weights"]})
        with L.on(dev) as s:
            L.check(lib.neo_mip_render_fwd(arr, L.ptr(o), L.ptr(d), L.ptr(vd), L.ptr(radii), n, C.byref(cfg), C.byref(out), L.ptr(self._ws),
                                           self._ws.numel(), s))
        return ren, hist

    @torch.no_grad()
    def field(self, rays: Dict[str, torch.Tensor], t: torch.Tensor, level: int, var, precision: Optional[str] = None, rgb: bool = True):
        """MLP `level` (0, 1: PropMLP; 2: NeRFMLP) at Gaussians with mean rays_o + t viewdirs and covariance diag(var), var a 3-sequence
        of per-axis variances; viewdirs is the direction input (neo_mip_field_eval).  t (n_rays, N) -> (rgb (n_rays, N, 3) or None,
        density (n_rays, N)) after their activations, in `precision` (default: the module's).  rgb is None at the proposal levels,
        which have no colour head, and when rgb=False."""
        o, vd = rays["rays_o"].contiguous().float(), rays["viewdirs"].contiguous().float()
        if not o.is_cuda:
            raise RuntimeError("neo360_b200 needs CUDA tensors (no CPU fallback)")
        prec = precision or self.precision
        if prec not in ("fp32", "tc"):
            raise ValueError(f"precision must be 'fp32' or 'tc', got {prec!r}")
        lib = L.load()
        t = t.contiguous().float()
        n, N = t.shape
        dev = o.device
        keep = []
        arr = (L.NeoMipMLPParams * 3)(*[m.to(dev).c_params(keep) for m in self.mlps])
        P = {"fp32": L.NEO_PREC_FP32, "tc": L.NEO_PREC_TC}[prec]
        need = lib.neo_mip_field_workspace_bytes(n * N, self.mlps[level].netwidth if 0 <= level < 3 else 0, P)
        if need == 0:
            raise ValueError(f"Mip-NeRF 360 field: bad level {level} or size {n} x {N}")
        ws = L.workspace(need, dev)
        r = L.NeoRays()
        r.n_rays, r.chunk = n, 0
        r.rays_o, r.rays_d, r.viewdirs = L.ptr(o), L.ptr(vd), L.ptr(vd)
        v = (C.c_float * 3)(*[float(x) for x in var])
        out_rgb = torch.empty(n, N, 3, device=dev) if rgb and level == 2 else None
        density = torch.empty(n, N, device=dev)
        with L.on(dev) as s:
            L.check(lib.neo_mip_field_eval(arr, int(level), C.byref(r), L.ptr(t), N, v, P, L.ptr(out_rgb), L.ptr(density), L.ptr(ws), need,
                                           s))
        return out_rgb, density

    def density_grid(self, resolution, bbox=((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)), level: int = 2, precision: Optional[str] = None,
                     slab_rays: Optional[int] = None, var=None) -> torch.Tensor:
        """density of MLP `level` on an (R_z, R_y, R_x) lattice over `bbox`; see neo360_b200.mesh.density_grid."""
        from . import mesh
        return mesh.density_grid(self, resolution, bbox, level, precision, slab_rays, var=var)

    def _forward_train(self, batch: Dict[str, torch.Tensor], train_frac: float, randomized: bool, near, far) -> Tuple[List[dict], List[dict]]:
        """MipNeRF360.forward under autograd (what LitMipNeRF360.training_step calls, model.py:427-456).  Per level: `neo_mip_resample` on the
        detached previous weights, `neo_mip_encode`, the MLP as `F.linear` on the modules' own parameters (fp32 whatever `self.precision`
        is; bf16 tensor-core GEMMs, `training.mlp_train_tc`, with `self.train_precision == "tc"`), then `_MipComposite` (the eval path's compositing kernel forward, `neo_mip_composite_bwd` backward)."""
        o = batch["rays_o"].contiguous().float()
        if not o.is_cuda:
            raise RuntimeError("neo360_b200 needs CUDA tensors (no CPU fallback)")
        d, vd = batch["rays_d"].contiguous().float(), batch["viewdirs"].contiguous().float()
        radii = batch["radii"].reshape(-1).contiguous().float()
        lib = L.load()
        n, dev = o.shape[0], o.device
        jit = [None] * 3
        if randomized:
            jit = batch.get("_uniforms") or [torch.rand((n, 1), device=dev) for _ in range(3)]     # helper.py:361 (single_jitter)
            jit = [j.reshape(-1).contiguous().float() for j in jit]
        ns = (self.num_prop_samples, self.num_prop_samples, self.num_nerf_samples)
        tc = check_train_precision(self.train_precision) == "tc"
        ren, hist = [], []
        sdist = w = None
        for lvl, mlp in enumerate(self.mlps):
            N = ns[lvl]
            with L.on(dev) as s:
                s1, t1 = torch.empty(n, N + 1, device=dev), torch.empty(n, N + 1, device=dev)
                wp = w.detach().contiguous() if lvl else None
                L.check(lib.neo_mip_resample(L.ptr(sdist), L.ptr(wp), n, ns[lvl - 1] if lvl else 1, lvl, N, float(near), float(far),
                                             float(train_frac), L.ptr(jit[lvl]), L.ptr(s1), L.ptr(t1), s))
                sdist = s1
                basis = mlp.pos_basis_t.to(dev).contiguous().float()
                if vd.requires_grad:
                    feats, denc = _MipEncode.apply(o, d, vd, radii, t1, basis)
                else:
                    feats, denc = torch.empty(n * N, 504, device=dev), torch.empty(n, 27, device=dev)
                    L.check(lib.neo_mip_encode(L.ptr(o), L.ptr(d), L.ptr(vd), L.ptr(radii), L.ptr(t1), L.ptr(basis), n, N, L.ptr(feats),
                                               L.ptr(denc), s))
            if tc:
                raw_density, raw_rgb = mlp_train_tc(mlp, feats, denc, n, N)
                raw_density = raw_density.reshape(n, N)
            else:
                raw_density, raw_rgb = _mlp_train(mlp, feats, denc, n, N)
            rgb, w, density, rgb_s = _MipComposite.apply(raw_density, raw_rgb, t1, d)
            ren.append({"rgb": rgb})
            hist.append({"density": density, "rgb": rgb_s, "sdist": sdist, "weights": w})
        return ren, hist


def _mlp_train(m: MipNeRF360MLP, feats: torch.Tensor, denc: torch.Tensor, n: int, N: int):
    """MipNeRF360MLP.forward (model.py:111-173) up to the activations, as framework GEMMs on the module's parameters: feats (n*N, 504),
    denc (n, 27) -> raw density (n, N), raw rgb (n, N, 3) or None (PropMLP).  The skip concatenation follows layer 4 (model.py:122-126);
    views_linear.0 sees [bottleneck | dir_enc], and its dir_enc columns are applied once per ray and broadcast over the ray's N samples
    (the same sum, re-associated)."""
    lin = lambda layer, x: F.linear(x, layer.weight, layer.bias)
    x = feats
    for i in range(m.netdepth):
        x = torch.relu(lin(m.pts_linear[i], x))
        if i % 4 == 0 and i > 0:
            x = torch.cat([x, feats], -1)
    raw_density = lin(m.density_layer, x).reshape(n, N)
    if m.disable_rgb:
        return raw_density, None
    beta = lin(m.bottleneck_layer, x)
    v = m.views_linear[0]
    kb = beta.shape[-1]
    y = F.linear(beta, v.weight[:, :kb], v.bias).reshape(n, N, -1) + F.linear(denc, v.weight[:, kb:])[:, None, :]
    return raw_density, lin(m.rgb_layer, torch.relu(y))


class _MipEncode(torch.autograd.Function):
    """neo_mip_encode under autograd: (rays_o, rays_d, viewdirs (n,3), radii (n), tdist (n,N+1), basis) -> feats (n*N, 504), dir_enc (n, 27).
    The backward (neo_mip_encode_bwd) gives viewdirs the gradient of its direction encoding; the IPE features give the rays none, as the
    reference's detached `contract` (helper.py:63-66)."""

    @staticmethod
    def forward(ctx, o, d, vd, radii, tdist, basis):
        lib = L.load()
        o, d, vd, radii, tdist = (x.detach().contiguous().float() for x in (o, d, vd, radii, tdist))
        n, N = tdist.shape[0], tdist.shape[1] - 1
        feats, denc = torch.empty(n * N, 504, device=o.device), torch.empty(n, 27, device=o.device)
        with L.on(o) as s:
            L.check(lib.neo_mip_encode(L.ptr(o), L.ptr(d), L.ptr(vd), L.ptr(radii), L.ptr(tdist), L.ptr(basis), n, N, L.ptr(feats), L.ptr(denc),
                                       s))
        ctx.save_for_backward(vd)
        return feats, denc

    @staticmethod
    def backward(ctx, g_feats, g_denc):
        lib = L.load()
        (vd,) = ctx.saved_tensors
        n = vd.shape[0]
        g_vd = torch.zeros(n, 3, device=vd.device)
        if g_denc is not None:
            with L.on(vd) as s:
                L.check(lib.neo_mip_encode_bwd(L.ptr(vd), n, L.ptr(g_denc.contiguous().float()), L.ptr(g_vd),
                                               s))
        return None, None, g_vd, None, None, None


class _MipComposite(torch.autograd.Function):
    """Head activations + compute_alpha_weights(opaque_background) + volumetric_rendering, white background (helper.py:234-274):
    raw density (n,N), raw rgb (n,N,3) or None (proposal level), tdist (n,N+1), rays_d (n,3) -> rgb (n,3), weights (n,N), density (n,N),
    rgb_s (n,N,3) (zeros for a proposal level).  Forward `neo_mip_composite` (the eval path's kernel), backward `neo_mip_composite_bwd`."""

    @staticmethod
    def forward(ctx, raw_density, raw_rgb, tdist, rays_d):
        lib = L.load()
        rd = raw_density.detach().contiguous().float()
        rc = raw_rgb.detach().contiguous().float() if raw_rgb is not None else None
        t, d = tdist.detach().contiguous().float(), rays_d.detach().contiguous().float()
        n, N = rd.shape
        dev = rd.device
        rgb, w, dens, rgb_s = torch.empty(n, 3, device=dev), torch.empty(n, N, device=dev), torch.empty(n, N, device=dev), torch.empty(n, N, 3, device=dev)
        with L.on(dev) as s:
            L.check(lib.neo_mip_composite(L.ptr(rd), L.ptr(rc), L.ptr(t), L.ptr(d), n, N, L.ptr(rgb), L.ptr(w), L.ptr(dens), L.ptr(rgb_s),
                                          s))
        ctx.save_for_backward(rd, rc, t, d)
        ctx.want_d = rays_d.requires_grad
        if rc is None:
            ctx.mark_non_differentiable(rgb_s)
        return rgb, w, dens, rgb_s

    @staticmethod
    def backward(ctx, g_rgb, g_w, g_dens, g_rgb_s):
        lib = L.load()
        rd, rc, t, d = ctx.saved_tensors
        n, N = rd.shape
        dev = rd.device
        d_rd = torch.empty(n, N, device=dev)
        d_rc = torch.empty(n, N, 3, device=dev) if rc is not None else None
        f = lambda g: None if g is None else g.contiguous().float()
        gs = [L.ptr(f(g_rgb)), L.ptr(f(g_w)), L.ptr(f(g_dens)), L.ptr(f(g_rgb_s) if rc is not None else None)]
        g_d = None
        with L.on(dev) as s:
            if ctx.needs_input_grad[3]:
                g_d = torch.empty(n, 3, device=dev)
                L.check(lib.neo_mip_composite_bwd_rays_d(L.ptr(rd), L.ptr(rc), L.ptr(t), L.ptr(d), n, N, *gs, L.ptr(d_rd), L.ptr(d_rc), L.ptr(g_d),
                                                         s))
            else:
                L.check(lib.neo_mip_composite_bwd(L.ptr(rd), L.ptr(rc), L.ptr(t), L.ptr(d), n, N, *gs, L.ptr(d_rd), L.ptr(d_rc),
                                                  s))
        return d_rd, d_rc, None, g_d


def _outer_weights(t: torch.Tensor, t_env: torch.Tensor, w_env: torch.Tensor) -> torch.Tensor:
    """w_outer of helper.inner_outer (helper.py:117-134): the envelope mass over each interval of t.  The reference's mask-based
    searchsorted (helper.py:108-113) is torch.searchsorted(t_env, t, right=True) = r, lo = max(r - 1, 0), hi = min(r, len(t_env) - 1)."""
    r = torch.searchsorted(t_env.contiguous(), t.contiguous(), right=True)
    lo, hi = (r - 1).clamp(min=0), r.clamp(max=t_env.shape[-1] - 1)
    cy = torch.cat([torch.zeros_like(w_env[..., :1]), torch.cumsum(w_env, -1)], -1)
    return torch.gather(cy, -1, hi)[..., 1:] - torch.gather(cy, -1, lo)[..., :-1]


class _Interlevel(torch.autograd.Function):
    """One proposal level of the interlevel loss per ray (neo_interlevel_loss, backward neo_interlevel_loss_bwd): sdist (n,Nc+1), weights
    (n,Nc) of the NeRF level (no gradient), sdist_env (n,Np+1), weights_env (n,Np) of the proposal level -> (n,); the gradient flows to
    weights_env.  Fixed-order sums, no atomics."""

    @staticmethod
    def forward(ctx, c, w, t_env, w_env):
        lib = L.load()
        ts = [x.detach().contiguous().float() for x in (c, w, t_env, w_env)]
        n, Nc = ts[1].shape
        Np = ts[3].shape[1]
        out = torch.empty(n, device=ts[0].device)
        with L.on(out) as s:
            L.check(lib.neo_interlevel_loss(*[L.ptr(x) for x in ts], n, Nc, Np, L.ptr(out), s))
        ctx.save_for_backward(*ts)
        return out

    @staticmethod
    def backward(ctx, g):
        lib = L.load()
        ts = ctx.saved_tensors
        n, Nc = ts[1].shape
        Np = ts[3].shape[1]
        d_we = torch.empty_like(ts[3])
        with L.on(d_we) as s:
            L.check(lib.neo_interlevel_loss_bwd(*[L.ptr(x) for x in ts], n, Nc, Np, L.ptr(g.contiguous().float()), L.ptr(d_we),
                                                s))
        return None, None, None, d_we


def training_loss(renderings: List[dict], ray_history: List[dict], target: torch.Tensor, charb_padding: float = 0.001,
                  interlevel_mult: float = 1.0, distortion_mult: float = 0.01) -> torch.Tensor:
    """LitMipNeRF360.training_step's loss (model.py:442-449): sqrt(mse + charb_padding^2) of the last rendering, plus the interlevel loss
    (lossfun_outer of every proposal level against the detached NeRF-level sdist / weights, model.py:725-734, helper.py:138-141), plus
    distortion_mult times the distortion loss of the NeRF level (model.py:736-741, helper.py:145-152; `training.distortion_loss` is the same
    functional in O(N) form for ascending sdist).  Under torch.use_deterministic_algorithms on CUDA tensors the interlevel terms come from
    neo_interlevel_loss (the same searchsorted / lo / hi semantics as `_outer_weights`, without its cumulative sums)."""
    mse = ((renderings[-1]["rgb"] - target) ** 2).mean()
    loss = torch.sqrt(mse + charb_padding ** 2)
    last = ray_history[-1]
    c, w = last["sdist"].detach(), last["weights"].detach()
    eps = 1.1920929e-07                                                           # helper.py:18
    inter = 0.0
    det = torch.are_deterministic_algorithms_enabled() and c.is_cuda           # torch.cumsum raises in deterministic mode
    for h in ray_history[:-1]:
        if det:
            inter = inter + _Interlevel.apply(c.reshape(-1, c.shape[-1]), w.reshape(-1, w.shape[-1]), h["sdist"].reshape(-1, h["sdist"].shape[-1]),
                                              h["weights"].reshape(-1, h["weights"].shape[-1])).mean()
            continue
        w_outer = _outer_weights(c, h["sdist"], h["weights"])
        inter = inter + (torch.clip(w - w_outer, min=0) ** 2 / (w + eps)).mean()
    s, wl = last["sdist"], last["weights"]
    dist = distortion_loss(wl, 0.5 * (s[..., 1:] + s[..., :-1]), s[..., 1:] - s[..., :-1])
    return loss + interlevel_mult * inter + distortion_mult * dist
