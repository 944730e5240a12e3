"""Drop-in for the reference's vanilla NeRF renderer (models/vanilla_nerf/model.py:44-216), SURVEY.md section 8(a) row a17.

`NeRF.forward(rays, randomized, white_bkgd, near, far)` returns the reference's `list[2]` of `(comp_rgb, acc, depth)`
(model.py:214).  Parameter names and shapes equal the reference's (`coarse_mlp.pts_linears.0.weight`, ...), so its checkpoints
load.  Arithmetic (csrc/vanilla.cu): `self.precision = "fp32"` (default) runs the layers on fp32 CUDA cores in the reference
formulation; `"tc"` runs them as fp16 wgmma GEMMs with fp32 accumulation (csrc/gemm_tc.cu).  CUDA only, no CPU fallback.

Training: with autograd on, the module in train mode and parameters that require grad, `NeRF.forward` returns the same tuples
differentiable w.r.t. every MLP parameter (LitNeRF.training_step, model.py:273-299).  Sampling, encodings and compositing forward and
backward are hand-written CUDA; the dense layers are framework fp32 GEMMs under autograd, or with `train_precision="tc"` bf16 tensor-core
GEMMs forward and backward (training._MLPTrainTC, csrc/dense_train.cu).  `precision` applies to inference only.  After an optimiser step the next inference call re-packs the weights (`_ensure` keys on each
parameter's storage and version).

Ray and pose gradients: when grad is enabled and `rays_o`, `rays_d` or `viewdirs` requires grad, `forward` takes the same autograd path,
also with the MLPs frozen or the module in eval mode, and the outputs are differentiable w.r.t. those rays as the reference's plain-PyTorch
module is: the points o + t viewdirs and the direction encoding through `neo_vanilla_encode_bwd`, |rays_d| through the compositing (the
sample positions t carry no gradient, as in the reference).  With `ops.sample_rays` / `ops.get_rays` on a `c2w` that requires grad and
`cameras.PoseCorrection`, this refines camera poses by photometric gradient.  With no ray requiring grad, nothing of this runs."""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib as L
from .training import _Composite, check_train_precision, mlp_train_tc, rays_need_grad


class NeRFMLP(nn.Module):
    def __init__(self, min_deg_point=0, max_deg_point=10, deg_view=4, netdepth: int = 8, netwidth: int = 256, netdepth_condition: int = 1,
                 netwidth_condition: int = 128, skip_layer: int = 4, input_ch: int = 3, input_ch_view: int = 3, num_rgb_channels: int = 3,
                 num_density_channels: int = 1):
        super().__init__()
        if (min_deg_point, max_deg_point, deg_view, netdepth, netwidth, netdepth_condition, netwidth_condition, skip_layer, input_ch,
                input_ch_view) != (0, 10, 4, 8, 256, 1, 128, 4, 3, 3):
            raise NotImplementedError("the CUDA path implements the reference's default NeRFMLP architecture")
        pos = ((max_deg_point - min_deg_point) * 2 + 1) * input_ch
        view = (deg_view * 2 + 1) * input_ch_view
        layers = [nn.Linear(pos, netwidth)]
        for idx in range(netdepth - 1):
            layers.append(nn.Linear(netwidth + pos if (idx % skip_layer == 0 and idx > 0) else netwidth, netwidth))
        self.pts_linears = nn.ModuleList(layers)
        self.views_linear = nn.ModuleList([nn.Linear(netwidth + view, netwidth_condition)])
        self.bottleneck_layer = nn.Linear(netwidth, netwidth)
        self.density_layer = nn.Linear(netwidth, num_density_channels)
        self.rgb_layer = nn.Linear(netwidth_condition, num_rgb_channels)
        for m in list(self.pts_linears) + [self.bottleneck_layer, self.density_layer, self.rgb_layer]:
            nn.init.xavier_uniform_(m.weight)

    def c_params(self, keep: list) -> L.NeoVanillaMLPParams:
        p = L.NeoVanillaMLPParams()
        f = lambda t: (keep.append(t.detach().contiguous().float()) or keep[-1])
        for i in range(8):
            p.w[i] = L.ptr(f(self.pts_linears[i].weight))
            p.b[i] = L.ptr(f(self.pts_linears[i].bias))
        for wn, bn, lin in (("wb", "bb", self.bottleneck_layer), ("wsig", "bsig", self.density_layer),
                            ("wv0", "bv0", self.views_linear[0]), ("wrgb", "brgb", self.rgb_layer)):
            setattr(p, wn, L.ptr(f(lin.weight)))
            setattr(p, bn, L.ptr(f(lin.bias)))
        return p

    def forward(self, *a, **k):
        raise RuntimeError("NeRFMLP is evaluated inside the CUDA path; call NeRF.forward")


def _mlp_train(m: NeRFMLP, enc: torch.Tensor, denc: torch.Tensor, n: int, N: int):
    """NeRFMLP.forward (model.py:100-125) as framework GEMMs on the module's parameters: enc (n*N, 63), denc (n, 27) -> raw rgb (n, N, 3),
    raw sigma (n, N, 1).  views_linear.0 sees [bottleneck | dir_enc]; its dir_enc columns are applied once per ray and broadcast over the
    ray's N samples (the same sum, re-associated)."""
    lin = lambda layer, x: F.linear(x, layer.weight, layer.bias)
    x = enc
    for i in range(8):
        x = torch.relu(lin(m.pts_linears[i], x))
        if i == 4:
            x = torch.cat([x, enc], -1)
    raw_sigma = lin(m.density_layer, x)
    beta = lin(m.bottleneck_layer, x)
    v = m.views_linear[0]
    kb = beta.shape[-1]
    y = F.linear(beta, v.weight[:, :kb], v.bias).reshape(n, N, -1) + F.linear(denc, v.weight[:, kb:])[:, None, :]
    raw_rgb = lin(m.rgb_layer, torch.relu(y))
    return raw_rgb, raw_sigma.reshape(n, N, 1)


class _VanillaEncode(torch.autograd.Function):
    """neo_vanilla_encode under autograd: rays_o, viewdirs (n,3), t (n,N) -> enc (n*N, 63), dir_enc (n, 27).  The backward
    (neo_vanilla_encode_bwd) gives rays_o and viewdirs their gradients; t carries none (the reference's sample positions are detached)."""

    @staticmethod
    def forward(ctx, o, vd, t):
        lib = L.load()
        o_c, vd_c, t_c = (x.detach().contiguous().float() for x in (o, vd, t))
        n, N = t_c.shape
        enc, denc = torch.empty(n * N, 63, device=o_c.device), torch.empty(n, 27, device=o_c.device)
        with L.on(o_c) as s:
            L.check(lib.neo_vanilla_encode(L.ptr(o_c), L.ptr(vd_c), L.ptr(t_c), n, N, L.ptr(enc), L.ptr(denc), s))
        ctx.save_for_backward(o_c, vd_c, t_c)
        return enc, denc

    @staticmethod
    def backward(ctx, g_enc, g_denc):
        lib = L.load()
        o_c, vd_c, t_c = ctx.saved_tensors
        n, N = t_c.shape
        dev = o_c.device
        g_enc = torch.zeros(n * N, 63, device=dev) if g_enc is None else g_enc.contiguous().float()
        g_denc = torch.zeros(n, 27, device=dev) if g_denc is None else g_denc.contiguous().float()
        g_o, g_vd = torch.empty(n, 3, device=dev), torch.empty(n, 3, device=dev)
        with L.on(dev) as s:
            L.check(lib.neo_vanilla_encode_bwd(L.ptr(o_c), L.ptr(vd_c), L.ptr(t_c), n, N, L.ptr(g_enc), L.ptr(g_denc), L.ptr(g_o), L.ptr(g_vd),
                                               s))
        return g_o, g_vd, None


class NeRF(nn.Module):
    def __init__(self, num_levels: int = 2, min_deg_point: int = 0, max_deg_point: int = 10, deg_view: int = 4, num_coarse_samples: int = 64,
                 num_fine_samples: int = 128, use_viewdirs: bool = True, noise_std: float = 0.0, lindisp: bool = False,
                 train_precision: str = "fp32"):
        super().__init__()
        self.train_precision = check_train_precision(train_precision)   # "fp32": framework GEMMs; "tc": bf16 tensor cores (training only)
        if num_levels != 2 or lindisp or noise_std != 0.0 or not use_viewdirs:
            raise NotImplementedError("reference defaults only (models/vanilla_nerf/model.py:129-139)")
        self.num_coarse_samples, self.num_fine_samples = num_coarse_samples, num_fine_samples
        self.coarse_mlp = NeRFMLP(min_deg_point, max_deg_point, deg_view)
        self.fine_mlp = NeRFMLP(min_deg_point, max_deg_point, deg_view)
        self._handle = None
        self._key = None
        self._ws = None

    def _ensure(self, dev):
        key = tuple((p.data_ptr(), p._version) for p in self.parameters())
        if self._handle is None or key != self._key:
            self.release()
            lib = L.load()
            keep = []
            arr = (L.NeoVanillaMLPParams * 2)(self.coarse_mlp.to(dev).c_params(keep), self.fine_mlp.to(dev).c_params(keep))
            h = C.c_void_p()
            with L.on(dev) as s:
                L.check(lib.neo_vanilla_create(arr, C.byref(h), s))
            self._handle, self._key = h, tuple((p.data_ptr(), p._version) for p in self.parameters())
        return self._handle

    def release(self):
        if self._handle is not None:
            L.load().neo_vanilla_free(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    def forward(self, rays: Dict[str, torch.Tensor], randomized: bool, white_bkgd: bool, near, far, debug: bool = False) -> List[tuple]:
        if torch.is_grad_enabled() and ((self.training and any(p.requires_grad for p in self.parameters())) or rays_need_grad(rays)):
            return self._forward_train(rays, randomized, white_bkgd, near, far, debug)
        o = rays["rays_o"].contiguous().float()
        d = rays["rays_d"].contiguous().float()
        vd = rays["viewdirs"].contiguous().float()
        if not o.is_cuda:
            raise RuntimeError("neo360_b200 needs CUDA tensors (no CPU fallback)")
        lib = L.load()
        h = self._ensure(o.device)
        n, dev = o.shape[0], o.device
        nc, nf = self.num_coarse_samples, self.num_fine_samples
        cfg = L.NeoVanillaCfg()
        cfg.n_coarse, cfg.n_fine, cfg.white_bkgd = nc, nf, int(bool(white_bkgd))
        cfg.near_plane, cfg.far_plane = float(near), float(far)
        cfg.precision = {"fp32": L.NEO_PREC_FP32, "tc": L.NEO_PREC_TC}[getattr(self, "precision", "fp32")]
        keep = []
        if randomized:
            u = rays.get("_uniforms") or [torch.rand((n, nc + 1), device=dev), torch.rand((n, nf), device=dev)]   # helper.py:438, 587
            keep.extend(u)
            cfg.u0, cfg.u1 = L.ptr(u[0].contiguous()), L.ptr(u[1].contiguous())
        r = L.NeoRays()
        r.n_rays, r.chunk = n, 0
        r.rays_o, r.rays_d, r.viewdirs = L.ptr(o), L.ptr(d), L.ptr(vd)
        self._ws = L.grow(self._ws, lib.neo_vanilla_workspace_bytes(n, C.byref(cfg)), dev)
        out = L.NeoVanillaOut()
        T = {k: [] for k in L.VANILLA_OUT_FIELDS}
        N = (nc + 1, nc + 1 + nf)
        for lvl in range(2):
            shapes = {"comp_rgb": (n, 3), "acc": (n,), "depth": (n,)}
            if debug:
                shapes.update({"t": (n, N[lvl]), "sigma": (n, N[lvl], 1), "rgb_s": (n, N[lvl], 3), "weights": (n, N[lvl])})
            for k, shp in shapes.items():
                t = torch.empty(*shp, device=dev)
                T[k].append(t)
                getattr(out, k)[lvl] = L.ptr(t)
        with L.on(dev) as s:
            L.check(lib.neo_vanilla_render_fwd(h, C.byref(r), C.byref(cfg), C.byref(out), L.ptr(self._ws), self._ws.numel(), s))
        if debug:
            self.last_debug = T
        return [(T["comp_rgb"][lvl], T["acc"][lvl], T["depth"][lvl]) for lvl in range(2)]

    @torch.no_grad()
    def field(self, rays: Dict[str, torch.Tensor], t: torch.Tensor, level: int, precision: Optional[str] = None):
        """The NeRFMLP of `level` (0 coarse, 1 fine) at the points rays_o + t viewdirs of t (n_rays, N), viewdirs its direction input:
        rgb (n_rays, N, 3), sigma (n_rays, N) after their activations (neo_vanilla_field_eval), in `precision` (default: the module's).
        The same code as `forward`'s per-level field: at the render's own t the same bits as its `rgb_s` / `sigma`."""
        o, vd = rays["rays_o"].contiguous().float(), rays["viewdirs"].contiguous().float()
        if not o.is_cuda:
            raise RuntimeError("neo360_b200 needs CUDA tensors (no CPU fallback)")
        prec = precision or getattr(self, "precision", "fp32")
        if prec not in ("fp32", "tc"):
            raise ValueError(f"precision must be 'fp32' or 'tc', got {prec!r}")
        lib = L.load()
        t = t.contiguous().float()
        n, N = t.shape
        dev = o.device
        h = self._ensure(dev)
        P = {"fp32": L.NEO_PREC_FP32, "tc": L.NEO_PREC_TC}[prec]
        need = lib.neo_vanilla_field_workspace_bytes(n * N, P)
        if need:            # 0: the fp32 field needs no workspace
            self._ws = L.grow(self._ws, need, dev)
        r = L.NeoRays()
        r.n_rays, r.chunk = n, 0
        r.rays_o, r.rays_d, r.viewdirs = L.ptr(o), L.ptr(vd), L.ptr(vd)
        rgb, sigma = torch.empty(n, N, 3, device=dev), torch.empty(n, N, device=dev)
        with L.on(dev) as s:
            L.check(lib.neo_vanilla_field_eval(h, C.byref(r), L.ptr(t), N, int(level), P, L.ptr(rgb), L.ptr(sigma),
                                               L.ptr(self._ws) if need else None, need, s))
        return rgb, sigma

    def density_grid(self, resolution, bbox=((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)), level: int = 1, precision: Optional[str] = None,
                     slab_rays: Optional[int] = None) -> torch.Tensor:
        """sigma of the NeRFMLP of `level` on an (R_z, R_y, R_x) lattice over `bbox`; see neo360_b200.mesh.density_grid."""
        from . import mesh
        return mesh.density_grid(self, resolution, bbox, level, precision, slab_rays)

    def _forward_train(self, rays: Dict[str, torch.Tensor], randomized: bool, white_bkgd: bool, near, far, debug: bool = False) -> List[tuple]:
        """NeRF.forward under autograd (what LitNeRF.training_step calls, models/vanilla_nerf/model.py:273-299): the same tuples,
        differentiable w.r.t. every parameter of coarse_mlp and fine_mlp.  Sampling, encodings and compositing (forward and backward) are
        the library's stages; the NeRFMLP layers are framework GEMMs (`F.linear`) on the modules' own parameters, in fp32 whatever
        `self.precision` is, or with `self.train_precision == "tc"` bf16 tensor-core GEMMs (`training.mlp_train_tc`).  `debug=True` keeps each level's sample positions and (detached) weights in `self.last_debug`."""
        o = rays["rays_o"].contiguous().float()
        d = rays["rays_d"].contiguous().float()
        vd = rays["viewdirs"].contiguous().float()
        if not o.is_cuda:
            raise RuntimeError("neo360_b200 needs CUDA tensors (no CPU fallback)")
        lib = L.load()
        n, dev = o.shape[0], o.device
        nc, nf = self.num_coarse_samples, self.num_fine_samples
        u = [None, None]
        if randomized:
            u = rays.get("_uniforms") or [torch.rand((n, nc + 1), device=dev), torch.rand((n, nf), device=dev)]   # helper.py:438, 587
            u = [x.contiguous().float() for x in u]
        tc = check_train_precision(self.train_precision) == "tc"
        ray_grad = o.requires_grad or vd.requires_grad
        ret, t, w = [], None, None
        dbg = {"t": [], "weights": []}
        for lvl, mlp in enumerate((self.coarse_mlp, self.fine_mlp)):
            with L.on(dev) as s:
                if lvl == 0:
                    t = torch.empty(n, nc + 1, device=dev)
                    L.check(lib.neo_vanilla_sample_along_rays(L.ptr(o.detach()), L.ptr(vd.detach()), n, nc, float(near), float(far), L.ptr(u[0]), L.ptr(t), s))
                else:       # bins = mids(t), weights[1:-1] of the DETACHED level-0 weights (helper.py:613)
                    t1 = torch.empty(n, t.shape[1] + nf, device=dev)
                    L.check(lib.neo_sample_pdf(L.ptr(o.detach()), L.ptr(vd.detach()), None, L.ptr(t), L.ptr(w.detach().contiguous()), n, t.shape[1], nf, 1, 0.0,
                                               L.ptr(u[1]), L.ptr(t1), None, None, s))
                    t = t1
                N = t.shape[1]
                if ray_grad:
                    enc, denc = _VanillaEncode.apply(o, vd, t)
                else:
                    enc, denc = torch.empty(n * N, 63, device=dev), torch.empty(n, 27, device=dev)
                    L.check(lib.neo_vanilla_encode(L.ptr(o), L.ptr(vd), L.ptr(t), n, N, L.ptr(enc), L.ptr(denc), s))
            if tc:
                raw_sigma, raw_rgb = mlp_train_tc(mlp, enc, denc, n, N)
                raw_sigma = raw_sigma.reshape(n, N, 1)
            else:
                raw_rgb, raw_sigma = _mlp_train(mlp, enc, denc, n, N)
            rgb = torch.sigmoid(raw_rgb) * (1 + 2 * 0.001) - 0.001              # model.py:197-205
            sigma = F.softplus(raw_sigma - 1.0)
            comp, acc, w, _, depth = _Composite.apply(rgb, sigma, t, d, None, white_bkgd, 2)
            ret.append((comp, acc, depth))
            dbg["t"].append(t)
            dbg["weights"].append(w.detach())
        if debug:
            self.last_debug = dbg
        return ret
