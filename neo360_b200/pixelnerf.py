"""Drop-in for the reference's PixelNeRF renderer (models/vanilla_nerf/model_pixel.py:35-258), SURVEY.md section 2 row 11.

`PixelNeRF.forward(rays, randomized, white_bkgd, near, far)` takes the NeO-360 batch dict (rays_o / rays_d / viewdirs and src_imgs /
src_poses / src_focal / src_c, datasets/nerds360_ae.py with model_type="pixelnerf") and returns the reference's `list[2]` of
`(comp_rgb, acc, depth)`.  Parameter names equal the reference's (`coarse_mlp.pts_linears.0.weight`, ..., `encoder.model.*`), so its
checkpoints load.  CUDA only, no CPU fallback.  The rays get no gradient (unlike the reference's plain-PyTorch module): that needs the
spatial gradient of the pixel-aligned lookup; vanilla NeRF has ray and pose gradients (DESIGN.md section 12).

Inference: sampling, the per-level field (csrc/pixelnerf.cu, fp32 CUDA cores in the reference formulation) and compositing run in the
library.  The encoder is hoisted: it runs once per `src_imgs` tensor and in-place version (the same deliberate difference as NeO-360's
quirk Q5), and its latent is kept channel-last.  `precision` selects the field's arithmetic: "fp32" (default, CUDA cores, the parity path) or "tc" (each dense layer
on the tensor cores through gemm_tc.cu, fp16 operands and fp32 accumulation; view means and activations in hand-written kernels).

Training (autograd on, module in train mode, parameters that require grad): the encoder runs under autograd on every call so its
convolutions train; sampling, encodings, the latent lookup and its backward (neo_index_maps / neo_index_maps_bwd, or the order-fixed
_det form under torch.use_deterministic_algorithms) and compositing forward and backward are the library's.  `train_precision` selects the
MLP's arithmetic: "fp32" (default) runs the dense layers as framework fp32 / TF32 GEMMs on the modules' parameters in the reference
formulation, as in vanilla NeRF's default training; "tc" applies the latent columns of pts_linears.0 to the latent map once per step
(P0 = latent . W0[:, 63:575]^T under autograd, exact re-association: the lookup is linear), looks up 128 projected channels instead of 512,
runs layers 0-3 and the view mean forward and backward on the tensor cores (training._PixelTrunkTC: bf16 operands, fp32 accumulation) and
the head once per point on the view mean (training.view_mean_head, fp32)."""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib as L
from .encoder import SpatialEncoder
from .renderer import Scene
from .training import _Composite, _PixelTrunkTC, _index_maps_bwd_det, check_train_precision, view_mean_head


class NeRFMLP(nn.Module):
    """model_pixel.py:35-93 at the defaults PixelNeRF uses: trunk [enc 63 | latent 512] -> 128 x4, views 155 -> 128 -> 128, rgb 128 -> 3."""

    def __init__(self, min_deg_point=0, max_deg_point=10, deg_view=4, netdepth: int = 4, netwidth: int = 128, netdepth_condition: int = 2,
                 netwidth_condition: int = 128, skip_layer: int = 4, input_ch: int = 3, input_ch_view: int = 3, num_rgb_channels: int = 3,
                 num_density_channels: int = 1, latent_size: int = 512, combine_layer: int = 3, combine_type="average"):
        super().__init__()
        if (min_deg_point, max_deg_point, deg_view, netdepth, netwidth, netdepth_condition, netwidth_condition, skip_layer, input_ch,
                input_ch_view, num_rgb_channels, num_density_channels, latent_size, combine_layer, combine_type) != \
                (0, 10, 4, 4, 128, 2, 128, 4, 3, 3, 3, 1, 512, 3, "average"):
            raise NotImplementedError("the CUDA path implements the reference's default PixelNeRF NeRFMLP architecture")
        pos = (max_deg_point - min_deg_point) * 2 * input_ch + input_ch + latent_size
        self.pts_linears = nn.ModuleList([nn.Linear(pos, netwidth)] + [nn.Linear(netwidth, netwidth) for _ in range(netdepth - 1)])
        self.views_linear = nn.ModuleList([nn.Linear(netwidth + (deg_view * 2 + 1) * input_ch_view, netwidth_condition),
                                           nn.Linear(netwidth_condition, netwidth_condition)])
        self.bottleneck_layer = nn.Linear(netwidth, netwidth)
        self.density_layer = nn.Linear(netwidth, num_density_channels)
        self.rgb_layer = nn.Linear(netwidth_condition, num_rgb_channels)
        for m in list(self.pts_linears) + [self.views_linear[1], self.bottleneck_layer, self.density_layer, self.rgb_layer]:
            nn.init.xavier_uniform_(m.weight)           # views_linear.0 keeps nn.Linear's default init, as in the reference

    def c_params(self, keep: list) -> L.NeoPixelMLPParams:
        p = L.NeoPixelMLPParams()
        t = lambda x: (keep.append(x.detach().float().t().contiguous()) or L.ptr(keep[-1]))
        f = lambda x: (keep.append(x.detach().float().contiguous()) or L.ptr(keep[-1]))
        for i in range(4):
            p.wt[i], p.b[i] = t(self.pts_linears[i].weight), f(self.pts_linears[i].bias)
        p.wbt, p.bb = t(self.bottleneck_layer.weight), f(self.bottleneck_layer.bias)
        p.wsig, p.bsig = f(self.density_layer.weight), f(self.density_layer.bias)
        p.wv0t, p.bv0 = t(self.views_linear[0].weight), f(self.views_linear[0].bias)
        p.wv1t, p.bv1 = t(self.views_linear[1].weight), f(self.views_linear[1].bias)
        p.wrgb, p.brgb = f(self.rgb_layer.weight), f(self.rgb_layer.bias)
        return p

    def tc_params(self, keep: list) -> L.NeoPixelTCParams:
        """fp16 weights (out, in) with the input width padded to a multiple of 64 (pts_linears.0: 576, views_linear.0: 192), fp32 biases
        and heads: the operands of neo_pixelnerf_field_tc."""
        p = L.NeoPixelTCParams()

        def h(lin):
            w = lin.weight.detach().float()
            k = -(-w.shape[1] // 64) * 64
            keep.append(F.pad(w, (0, k - w.shape[1])).half().contiguous())
            return L.ptr(keep[-1])

        f = lambda x: (keep.append(x.detach().float().contiguous()) or L.ptr(keep[-1]))
        for i in range(4):
            p.w16[i], p.b[i] = h(self.pts_linears[i]), f(self.pts_linears[i].bias)
        p.wb16, p.bb = h(self.bottleneck_layer), f(self.bottleneck_layer.bias)
        p.wsig, p.bsig = f(self.density_layer.weight), f(self.density_layer.bias)
        p.wv016, p.bv0 = h(self.views_linear[0]), f(self.views_linear[0].bias)
        p.wv116, p.bv1 = h(self.views_linear[1]), f(self.views_linear[1].bias)
        p.wrgb, p.brgb = f(self.rgb_layer.weight), f(self.rgb_layer.bias)
        return p

    def forward(self, *a, **k):
        raise RuntimeError("NeRFMLP is evaluated inside the CUDA path; call PixelNeRF.forward")


def _mlp_train(m: NeRFMLP, enc: torch.Tensor, dir_tile: torch.Tensor, local: torch.Tensor, nv: int):
    """NeRFMLP.forward (model_pixel.py:95-131) as framework GEMMs: enc (nv*M,63), dir_tile (nv*M,27), local (nv*M,512) -> raw rgb (M,3),
    raw sigma (M,1)."""
    lin = lambda layer, x: F.linear(x, layer.weight, layer.bias)
    h = torch.cat([enc, local], -1)
    for i in range(4):
        h = torch.relu(lin(m.pts_linears[i], h))
    M = h.shape[0] // nv
    beta = lin(m.bottleneck_layer, h)
    raw_sigma = lin(m.density_layer, h.reshape(nv, M, -1).mean(0))
    q = torch.relu(lin(m.views_linear[0], torch.cat([beta, dir_tile], -1)).reshape(nv, M, -1).mean(0))
    return lin(m.rgb_layer, torch.relu(lin(m.views_linear[1], q))), raw_sigma


def _mlp_train_tc(m: NeRFMLP, cam: torch.Tensor, dir_tile: torch.Tensor, p0: torch.Tensor, nv: int):
    """`_mlp_train` with the latent columns of layer 0 already applied (p0 (nv*M, 128) = looked-up rows of latent . W0[:, 63:]^T): the
    trunk on the tensor cores from the camera-frame points cam (nv, M, 3), the head once per point -> raw rgb (M,3), raw sigma (M,1)."""
    p = m.pts_linears
    hbar = _PixelTrunkTC.apply(cam, p0, p[0].weight[:, :63], p[0].bias, p[1].weight, p[1].bias, p[2].weight, p[2].bias, p[3].weight,
                               p[3].bias)
    return view_mean_head(m, hbar, dir_tile, nv)


class _LatentLookup(torch.autograd.Function):
    """SpatialEncoder.index rows of world points pts (M,3): latent_cl (nv,Hl,Wl,512) -> (nv*M,512); the backward scatters into the
    channel-last latent gradient (neo_index_maps_bwd, or neo_index_maps_bwd_det under deterministic algorithms)."""

    @staticmethod
    def forward(ctx, pts, latent_cl, sc):
        lib = L.load()
        M, Cc = pts.shape[0], latent_cl.shape[-1]
        lat = latent_cl.detach().contiguous()
        out = torch.empty(sc.nv * M, Cc, device=pts.device)
        with L.on(pts) as s:
            L.check(lib.neo_index_maps(sc.handle, L.ptr(pts), M, Cc, L.ptr(lat), None, None, None, L.ptr(out), None, s))
        ctx.save_for_backward(pts)
        ctx.sc, ctx.shape = sc, latent_cl.shape
        ctx.det = torch.are_deterministic_algorithms_enabled()
        return out

    @staticmethod
    def backward(ctx, g):
        lib = L.load()
        (pts,) = ctx.saved_tensors
        sc, M = ctx.sc, pts.shape[0]
        g = g.contiguous().float()
        g_lat = torch.zeros(ctx.shape, device=pts.device)
        if ctx.det:
            _index_maps_bwd_det(sc, pts, M, ctx.shape[-1], g, None, g_lat, [None] * 3)
        else:
            with L.on(pts) as s:
                L.check(lib.neo_index_maps_bwd(sc.handle, L.ptr(pts), M, ctx.shape[-1], L.ptr(g), None, L.ptr(g_lat), None, None, None, s))
        return None, g_lat, None


class PixelNeRF(nn.Module):
    def __init__(self, num_levels: int = 2, min_deg_point: int = 0, max_deg_point: int = 10, deg_view: int = 4, num_coarse_samples: int = 64,
                 num_fine_samples: int = 64, use_viewdirs: bool = True, noise_std: float = 0.0, lindisp: bool = False, num_src_views: int = 3,
                 train_precision: str = "fp32"):
        super().__init__()
        if num_levels != 2 or lindisp or noise_std != 0.0 or not use_viewdirs:
            raise NotImplementedError("reference defaults only (models/vanilla_nerf/model_pixel.py:134-147)")
        self.num_levels, self.num_src_views = num_levels, num_src_views
        self.num_coarse_samples, self.num_fine_samples = num_coarse_samples, num_fine_samples
        self.precision = "fp32"
        self.train_precision = check_train_precision(train_precision)   # "fp32": framework GEMMs; "tc": bf16 tensor cores (training only)
        self.encoder = SpatialEncoder()
        self.coarse_mlp = NeRFMLP(min_deg_point, max_deg_point, deg_view)
        self.fine_mlp = NeRFMLP(min_deg_point, max_deg_point, deg_view)
        self._packed = None                 # (key, precision, keep, params[2])
        self._ws = None                     # workspace of the tensor-core field
        self._scene = None                  # (key, Scene)
        self._latent = None                 # (key, latent_cl) of the hoisted encoder

    @staticmethod
    def _key(tensors):
        return tuple((id(t), t._version) for t in tensors)

    def _ensure_weights(self, precision: str):
        params = list(self.coarse_mlp.parameters()) + list(self.fine_mlp.parameters())
        key = tuple((p.data_ptr(), p._version) for p in params)
        if self._packed is None or self._packed[0] != key or self._packed[1] != precision:
            keep = []
            pack = (lambda m: m.c_params(keep)) if precision == "fp32" else (lambda m: m.tc_params(keep))
            self._packed = (key, precision, keep, [pack(self.coarse_mlp), pack(self.fine_mlp)])
        return self._packed[3]

    def _ensure_scene(self, rays, lat_hw):
        """Cameras-only NeoScene from the source poses with the camera y axis negated (include/neo360_b200.h, PixelNeRF section)."""
        src = [rays[k] for k in ("src_poses", "src_focal", "src_c", "src_imgs")]
        key = (self._key(src), tuple(rays["src_imgs"].shape[-2:]), tuple(lat_hw))
        if self._scene is not None and self._scene[0] == key and all(a is b for a, b in zip(self._scene[2], src)):
            return self._scene[1]
        poses = rays["src_poses"].detach().float().clone()
        poses[:, :3, 1] = -poses[:, :3, 1]
        nv = poses.shape[0]
        if nv != self.num_src_views:
            raise ValueError(f"batch has {nv} source views, the model was built for {self.num_src_views}")
        focal, c = rays["src_focal"].detach().float().contiguous(), rays["src_c"].detach().float().contiguous()
        dummy = torch.zeros(4, device=poses.device)
        d = L.NeoSceneDesc()
        d.nv, d.world_ch, d.plane_h, d.plane_w = nv, 128, 2, 2
        d.local_ch, (d.lat_h, d.lat_w) = 512, lat_hw
        d.img_w, d.img_h = int(rays["src_imgs"].shape[-1]), int(rays["src_imgs"].shape[-2])
        d.planes_xz = d.planes_xy = d.planes_yz = d.latent = L.ptr(dummy)     # not read by a cameras-only scene
        d.src_poses, d.src_focal, d.src_c = L.ptr(poses), L.ptr(focal), L.ptr(c)
        h = C.c_void_p()
        with L.on(poses) as s:
            L.check(L.load().neo_scene_create(C.byref(d), (L.NeoMLPParams * 4)(), 0, C.byref(h), s))
        sc = Scene(h, 0)
        sc.nv = nv
        self._scene = (key, sc, src)
        return sc

    def _hoisted_latent(self, imgs):
        """encoder(src_imgs) once per src_imgs tensor, in-place version and version of the trunk's parameters and batch-norm statistics;
        channel-last (nv,Hl,Wl,512)."""
        trunk = list(self.encoder.model.parameters()) + list(self.encoder.model.buffers())
        key = (id(imgs), imgs._version, self.encoder.training, tuple((p.data_ptr(), p._version) for p in trunk))
        if self._latent is None or self._latent[0] != key or self._latent[2] is not imgs:
            with torch.no_grad():
                lat = self.encoder(imgs)
            self._latent = (key, lat.permute(0, 2, 3, 1).contiguous(), imgs)
        return self._latent[1]

    def _rays(self, rays, chunk):
        o, d, vd = (rays[k].contiguous().float() for k in ("rays_o", "rays_d", "viewdirs"))
        if not o.is_cuda:
            raise RuntimeError("neo360_b200 needs CUDA tensors (no CPU fallback)")
        r = L.NeoRays()
        r.n_rays, r.chunk = o.shape[0], int(chunk or 0)
        r.rays_o, r.rays_d, r.viewdirs, r.ray_order = L.ptr(o), L.ptr(d), L.ptr(vd), None
        return r, (o, d, vd)

    def _uniforms(self, rays, randomized, n, dev):
        if not randomized:
            return [None, None]
        u = rays.get("_uniforms") or [torch.rand((n, self.num_coarse_samples + 1), device=dev), torch.rand((n, self.num_fine_samples), device=dev)]
        return [x.contiguous().float() for x in u]          # helper.py:438, 587

    def _sample(self, lvl, o, d, t, w, n, near, far, u):
        lib, dev = L.load(), o.device
        with L.on(o) as s:
            if lvl == 0:
                t1 = torch.empty(n, self.num_coarse_samples + 1, device=dev)
                L.check(lib.neo_vanilla_sample_along_rays(L.ptr(o), L.ptr(d), n, self.num_coarse_samples, float(near), float(far), L.ptr(u),
                                                          L.ptr(t1), s))
            else:       # bins = mids(t), weights[1:-1] of the detached level-0 weights (model_pixel.py:195-204)
                t1 = torch.empty(n, t.shape[1] + self.num_fine_samples, device=dev)
                L.check(lib.neo_sample_pdf(L.ptr(o), L.ptr(d), None, L.ptr(t), L.ptr(w.detach().contiguous()), n, t.shape[1],
                                           self.num_fine_samples, 1, 0.0, L.ptr(u), L.ptr(t1), None, None, s))
        return t1

    def _field(self, r, sc, lat, t, lvl, precision: str):
        lib, dev = L.load(), t.device
        n, N = t.shape
        mlp = self._ensure_weights(precision)[lvl]
        rgb, sigma = torch.empty(n, N, 3, device=dev), torch.empty(n, N, device=dev)
        with L.on(t) as s:
            if precision == "fp32":
                L.check(lib.neo_pixelnerf_field(sc.handle, L.ptr(lat), C.byref(mlp), C.byref(r), L.ptr(t), N, L.ptr(rgb), L.ptr(sigma), s))
            else:
                self._ws = L.grow(self._ws, lib.neo_pixelnerf_tc_workspace_bytes(sc.nv, n * N), dev)
                L.check(lib.neo_pixelnerf_field_tc(sc.handle, L.ptr(lat), C.byref(mlp), C.byref(r), L.ptr(t), N, L.ptr(rgb), L.ptr(sigma),
                                                   L.ptr(self._ws), self._ws.numel(), s))
        return rgb, sigma

    @torch.no_grad()
    def field(self, rays: Dict[str, torch.Tensor], t: torch.Tensor, level: int, chunk: Optional[int] = None, precision: Optional[str] = None):
        """The field of one level at the caller's sample distances t (n_rays, N), in `precision` (default: `self.precision`): rgb
        (n_rays, N, 3), sigma (n_rays, N) after their activations (model_pixel.py:207-246).  `rays` also holds the src_* entries of
        `forward`'s batch; `chunk` is `forward`'s (quirk Q1)."""
        prec = precision or self.precision
        if prec not in ("fp32", "tc"):
            raise ValueError(f"PixelNeRF precision must be 'fp32' or 'tc', got {prec!r}")
        r, _ = self._rays(rays, chunk)
        lat = self._hoisted_latent(rays["src_imgs"])
        sc = self._ensure_scene(rays, lat.shape[1:3])
        return self._field(r, sc, lat, t.contiguous().float(), level, prec)

    def density_grid(self, resolution, bbox=((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)), level: int = 1, precision: Optional[str] = None,
                     slab_rays: Optional[int] = None, batch: Optional[Dict[str, torch.Tensor]] = None) -> torch.Tensor:
        """sigma of the MLP of `level` on an (R_z, R_y, R_x) lattice over `bbox`, seen by the source views of `batch` (its src_*
        entries, as `forward` takes them); see neo360_b200.mesh.density_grid."""
        from . import mesh
        return mesh.density_grid(self, resolution, bbox, level, precision, slab_rays, batch)

    def forward(self, rays: Dict[str, torch.Tensor], randomized: bool, white_bkgd: bool, near, far, chunk: Optional[int] = None) -> List[tuple]:
        """model_pixel.py:174-258.  `chunk` (default: the whole call) is the caller's chunk size for quirk Q1: a sample's direction
        encoding comes from ray (j mod B) of its own chunk, as when the reference is called chunk by chunk."""
        if self.precision not in ("fp32", "tc"):
            raise ValueError(f"PixelNeRF precision must be 'fp32' or 'tc', got {self.precision!r}")
        if torch.is_grad_enabled() and self.training and any(p.requires_grad for p in self.parameters()):
            return self._forward_train(rays, randomized, white_bkgd, near, far, chunk)
        lib = L.load()
        r, (o, d, vd) = self._rays(rays, chunk)
        n, dev = o.shape[0], o.device
        with L.on(dev) as s:
            lat = self._hoisted_latent(rays["src_imgs"])
            sc = self._ensure_scene(rays, lat.shape[1:3])
            u = self._uniforms(rays, randomized, n, dev)
            ret, t, w = [], None, None
            for lvl in range(2):
                t = self._sample(lvl, o, d, t, w, n, near, far, u[lvl])
                N = t.shape[1]
                rgb, sigma = self._field(r, sc, lat, t, lvl, self.precision)
                comp, acc, w, depth = torch.empty(n, 3, device=dev), torch.empty(n, device=dev), torch.empty(n, N, device=dev), torch.empty(n, device=dev)
                L.check(lib.neo_volumetric_rendering(L.ptr(rgb), L.ptr(sigma), L.ptr(t), L.ptr(d), None, n, N, int(bool(white_bkgd)), 2,
                                                     L.ptr(comp), L.ptr(acc), L.ptr(w), None, L.ptr(depth), s))
                ret.append((comp, acc, depth))
        return ret

    def _forward_train(self, rays, randomized, white_bkgd, near, far, chunk) -> List[tuple]:
        """PixelNeRF.forward under autograd (LitPixelNeRF.training_step, model_pixel.py:322-347): differentiable w.r.t. every MLP and
        encoder parameter."""
        lib = L.load()
        tc = check_train_precision(self.train_precision) == "tc"
        r, (o, d, vd) = self._rays(rays, chunk)
        n, dev = o.shape[0], o.device
        nv = self.num_src_views
        with L.on(dev) as s:
            latent = self.encoder(rays["src_imgs"])
            lat_cl = latent.permute(0, 2, 3, 1)                         # channel-last: the lookup's layout, the projection contracts it
            if not tc:
                lat_cl = lat_cl.contiguous()
            sc = self._ensure_scene(rays, lat_cl.shape[1:3])
            u = self._uniforms(rays, randomized, n, dev)
            ret, t, w = [], None, None
            for lvl, mlp in enumerate((self.coarse_mlp, self.fine_mlp)):
                t = self._sample(lvl, o, d, t, w, n, near, far, u[lvl])
                N = t.shape[1]
                M = n * N
                enc, dtile, pts = torch.empty(nv * M, 63, device=dev), torch.empty(nv * M, 27, device=dev), torch.empty(M, 3, device=dev)
                L.check(lib.neo_pixelnerf_encode(sc.handle, C.byref(r), L.ptr(t), N, L.ptr(enc), L.ptr(dtile), L.ptr(pts), s))
                if tc:
                    p0 = _LatentLookup.apply(pts, lat_cl @ mlp.pts_linears[0].weight[:, 63:].t(), sc)
                    raw_rgb, raw_sigma = _mlp_train_tc(mlp, enc[:, :3].reshape(nv, M, 3), dtile, p0, nv)
                else:
                    local = _LatentLookup.apply(pts, lat_cl, sc)
                    raw_rgb, raw_sigma = _mlp_train(mlp, enc, dtile, local, nv)
                rgb = torch.sigmoid(raw_rgb).reshape(n, N, 3)               # model_pixel.py:245-246
                sigma = torch.relu(raw_sigma).reshape(n, N, 1)
                comp, acc, w, _, depth = _Composite.apply(rgb, sigma, t, d, None, white_bkgd, 2)
                ret.append((comp, acc, depth))
        return ret
