"""Drop-in for the reference's NeO-360 renderer behind its own call surface.  The rays get no gradient (unlike the reference's plain
PyTorch): that needs the spatial gradient of the tri-plane and projected-map lookups; vanilla NeRF has ray and pose gradients
(DESIGN.md section 12).

    reference                                         here
    ---------------------------------------------     ------------------------------------------------
    models/neo360/model.py:37   NeRFPPMLP             NeRFPPMLP  (same parameter names / shapes; weights only)
    models/neo360/model.py:162  NeRF_TP               NeRF_TP    (same ctor args, same forward signature + returns)
    model.py:861-907 render_rays_test chunk loop      NeRF_TP.render_rays_test(batch, chunk)  (one call, same result)

`forward(rays, randomized, white_bkgd, near, far, out_depth=False)` returns the reference's `list[2]` of tuples
(model.py:525-527 / 577-579).  The encoder (GridEncoder, out of scope: SURVEY.md section 8(f1)) is hoisted out of the
chunk loop (quirk Q5): call `set_scene(...)` once per scene with its outputs, or pass them in the `rays` dict under
`planes_xz|planes_xy|planes_yz|latent`; or hand an `encoder` module to the constructor and it is run once per new set
of `src_*` tensors.  All arithmetic runs in libneo360_b200.so (hand-written CUDA, sm_90a); there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional

import torch
import torch.nn as nn

from . import _lib as L

PRECISIONS = {"fp32": L.NEO_PREC_FP32, "tc": L.NEO_PREC_TC}


class NeRFPPMLP(nn.Module):
    """Parameter container with the reference's layout (models/neo360/model.py:37-108).  Evaluation happens in CUDA."""

    def __init__(self, min_deg_point, max_deg_point, deg_view, netdepth: int = 4, netwidth: int = 128,
                 netdepth_condition: int = 2, netwidth_condition: int = 64, skip_layer: int = 2, input_ch: int = 3,
                 input_ch_view: int = 3, num_rgb_channels: int = 3, num_density_channels: int = 1,
                 local_latent_size: int = 512, world_latent_size: int = 128, combine_layer: int = 3,
                 combine_type="average", out_nocs=False, num_src_views=3):
        super().__init__()
        if (netdepth, netwidth, netdepth_condition, netwidth_condition, skip_layer, combine_layer, combine_type,
                local_latent_size, world_latent_size, out_nocs) != (4, 128, 2, 64, 2, 3, "average", 512, 128, False):
            raise NotImplementedError("the CUDA path implements the reference's default NeRFPPMLP architecture")
        if (min_deg_point, max_deg_point, deg_view) != (0, 10, 4) or input_ch not in (3, 4):
            raise NotImplementedError("pos-enc degrees are fixed to the reference's (0,10,4)")
        self.input_ch = input_ch
        pos = ((max_deg_point - min_deg_point) * 2 + 1) * input_ch + local_latent_size + world_latent_size
        view = (deg_view * 2 + 1) * input_ch_view
        layers = [nn.Linear(pos, netwidth)]
        for idx in range(netdepth - 1):
            layers.append(nn.Linear(netwidth + pos if (idx % skip_layer == 0 and idx > 0) else netwidth, netwidth))
        self.pts_linears = nn.ModuleList(layers)
        self.views_linear = nn.ModuleList([nn.Linear(netwidth + view, netwidth_condition),
                                           nn.Linear(netwidth_condition, netwidth_condition)])
        self.bottleneck_layer = nn.Linear(netwidth, netwidth)
        self.density_layer = nn.Linear(netwidth, num_density_channels)
        self.rgb_layer = nn.Linear(netwidth_condition, num_rgb_channels)
        for m in list(self.pts_linears) + [self.views_linear[1], self.bottleneck_layer, self.density_layer, self.rgb_layer]:
            nn.init.xavier_uniform_(m.weight)

    def c_params(self, keep: list) -> L.NeoMLPParams:
        p = L.NeoMLPParams()
        p.in_ch = self.input_ch

        def put(wn, bn, lin):
            w, b = lin.weight.detach().contiguous().float(), lin.bias.detach().contiguous().float()
            keep.extend([w, b])
            setattr(p, wn, L.ptr(w)); setattr(p, bn, L.ptr(b))

        for i in range(4):
            put(f"w{i}", f"b{i}", self.pts_linears[i])
        put("wb", "bb", self.bottleneck_layer)
        put("wsig", "bsig", self.density_layer)
        put("wv0", "bv0", self.views_linear[0])
        put("wv1", "bv1", self.views_linear[1])
        put("wrgb", "brgb", self.rgb_layer)
        return p

    def forward(self, *a, **k):
        raise RuntimeError("NeRFPPMLP is evaluated inside the fused CUDA path; call NeRF_TP.forward")


class Scene:
    """Owns a NeoScene handle (re-laid-out feature maps + packed weights) for one scene + parameter version."""

    def __init__(self, handle, nbytes):
        self.handle = handle
        self.nbytes = nbytes

    def __del__(self):
        try:
            if self.handle:
                L.load().neo_scene_free(self.handle)
                self.handle = None
        except Exception:
            pass


class NeRF_TP(nn.Module):
    def __init__(self, num_levels: int = 2, min_deg_point: int = 0, max_deg_point: int = 10, deg_view: int = 4,
                 num_coarse_samples: int = 128, num_fine_samples: int = 256, use_viewdirs: bool = True,
                 num_src_views: int = 3, density_noise: float = 0.0, lindisp: bool = False, encoder: Optional[nn.Module] = None,
                 precision: str = "tc", chunk: Optional[int] = None, train_precision: str = "fp32", **unused):
        super().__init__()
        if num_levels != 2 or lindisp or density_noise != 0.0 or not use_viewdirs:
            raise NotImplementedError("reference defaults only: 2 levels, lindisp=False, density_noise=0 (model.py:165-175)")
        self.num_coarse_samples, self.num_fine_samples, self.num_src_views = num_coarse_samples, num_fine_samples, num_src_views
        self.precision = precision
        # arithmetic of the MLPs in a training step: "fp32" (framework layers under autograd) or "tc" (bf16 tensor-core trunk,
        # projected formulation only; training._TrunkTC).  An attribute like train_projected.
        self.train_precision = train_precision
        self.chunk = chunk
        self.encoder = encoder
        mk = lambda ch: NeRFPPMLP(min_deg_point, max_deg_point, deg_view, num_src_views=num_src_views, input_ch=ch)
        self.fg_coarse_mlp, self.fg_fine_mlp = mk(3), mk(3)
        self.bg_coarse_mlp, self.bg_fine_mlp = mk(4), mk(4)
        self._scene: Optional[Scene] = None
        self._scene_src = None          # (tensors, versions) the scene was built from: compared by identity, never by address
        self._scene_inputs = None       # arguments of the last set_scene (to re-pack when the parameters change)
        self._param_key = None
        self._ws = None

    # ---- scene handling (encoder hoisted, quirk Q5) ----
    def _mlps(self):
        return [self.fg_coarse_mlp, self.bg_coarse_mlp, self.fg_fine_mlp, self.bg_fine_mlp]

    def _params_version(self):
        """Identity of the packed weights: every parameter's storage and in-place version (optimizer steps, load_state_dict)."""
        return tuple((p.data_ptr(), p._version) for m in self._mlps() for p in m.parameters())

    def set_scene(self, planes_xz, planes_xy, planes_yz, latent, src_poses, src_focal, src_c, img_wh, precisions=None):
        """Build the per-scene state (pre-projected feature maps, cameras, packed weights).  The scene snapshots the CURRENT
        parameters; `forward` re-packs it when they have changed since (training steps, load_state_dict)."""
        lib = L.load()
        dev = planes_xz.device
        if dev.type != "cuda":
            raise RuntimeError("neo360_b200 needs CUDA tensors (no CPU fallback)")
        nv = planes_xz.shape[0]
        if planes_xz.dim() != 4 or latent.dim() != 4:
            raise ValueError("planes must be (NV,128,Hp,Wp) and latent (NV,512,Hl,Wl)")
        if not (planes_xy.shape == planes_xz.shape == planes_yz.shape):
            raise ValueError(f"tri-planes must share one shape, got {tuple(planes_xz.shape)} {tuple(planes_xy.shape)} {tuple(planes_yz.shape)}")
        if latent.shape[0] != nv or nv != self.num_src_views:
            raise ValueError(f"scene has {nv} plane views / {latent.shape[0]} latent views, the model was built for {self.num_src_views}")
        if src_poses.shape[0] != nv or tuple(src_poses.shape[1:]) != (4, 4):
            raise ValueError(f"src_poses must be ({nv},4,4), got {tuple(src_poses.shape)}")
        if int(img_wh[0]) <= 0 or int(img_wh[1]) <= 0:
            raise ValueError(f"img_wh must be positive, got {img_wh}")
        self._scene_inputs = (planes_xz, planes_xy, planes_yz, latent, src_poses, src_focal, src_c, tuple(img_wh), precisions)
        keep = []
        f = lambda t: (keep.append(t.detach().contiguous().float()) or keep[-1])
        d = L.NeoSceneDesc()
        d.nv, d.world_ch, d.plane_h, d.plane_w = planes_xz.shape
        _, d.local_ch, d.lat_h, d.lat_w = latent.shape
        d.img_w, d.img_h = int(img_wh[0]), int(img_wh[1])
        d.planes_xz, d.planes_xy, d.planes_yz = L.ptr(f(planes_xz)), L.ptr(f(planes_xy)), L.ptr(f(planes_yz))
        d.latent = L.ptr(f(latent))
        d.src_poses, d.src_focal, d.src_c = L.ptr(f(src_poses)), L.ptr(f(src_focal)), L.ptr(f(src_c))
        arr = (L.NeoMLPParams * 4)(*[m.to(dev).c_params(keep) for m in self._mlps()])
        precisions = [self.precision] if precisions is None else precisions      # [] = cameras / geometry only (projected-map training)
        mask = 0
        for p in precisions:
            mask |= 1 << PRECISIONS[p]
        h = C.c_void_p()
        with torch.cuda.device(dev):
            L.check(lib.neo_scene_create(C.byref(d), arr, mask, C.byref(h), torch.cuda.current_stream().cuda_stream))
        self._scene = Scene(h, lib.neo_scene_bytes(h))
        self._scene.nv = nv
        self._scene.mask = mask
        self._param_key = self._params_version()
        self._scene_src = None
        return self._scene

    def _same_source(self, tensors) -> bool:
        """True when the scene was built from exactly these tensor OBJECTS at their current in-place versions.  Addresses are
        not compared: the caching allocator hands a freed block back at the same address for the next scene."""
        src = self._scene_src
        return (src is not None and len(src[0]) == len(tensors) and all(a is b for a, b in zip(src[0], tensors))
                and src[1] == tuple(t._version for t in tensors))

    def _ensure_scene(self, rays, precision: Optional[str] = None):
        precision = precision or self.precision
        if all(k in rays for k in ("planes_xz", "planes_xy", "planes_yz", "latent")):
            keyed = tuple(rays[k] for k in ("planes_xz", "planes_xy", "planes_yz", "latent", "src_poses"))
            if not self._same_source(keyed):
                W, H = rays["src_imgs"].shape[-1], rays["src_imgs"].shape[-2]
                self.set_scene(rays["planes_xz"], rays["planes_xy"], rays["planes_yz"], rays["latent"], rays["src_poses"],
                               rays["src_focal"], rays["src_c"], (W, H))
                self._scene_src = (keyed, tuple(t._version for t in keyed))
        elif self.encoder is not None and "src_imgs" in rays:
            keyed = tuple(rays[k] for k in ("src_imgs", "src_poses", "src_focal", "src_c"))
            if not self._same_source(keyed):
                with torch.no_grad():
                    xz, xy, yz = self.encoder(rays["src_imgs"], rays["src_poses"], rays["src_focal"], rays["src_c"])
                    latent = self.encoder.spatial_encoder.latent
                W, H = rays["src_imgs"].shape[-1], rays["src_imgs"].shape[-2]
                self.set_scene(xz, xy, yz, latent, rays["src_poses"], rays["src_focal"], rays["src_c"], (W, H))
                self._scene_src = (keyed, tuple(t._version for t in keyed))
        if self._scene is None:
            raise RuntimeError("no scene: call set_scene(...) or pass planes_*/latent in `rays`, or give an encoder")
        need = 1 << PRECISIONS[precision]
        if self._param_key != self._params_version() or not (self._scene.mask & need):
            # the packed weights (fp32 transposes, swizzled weight images, W0/W3-projected feature maps) are stale, or the scene was last built for
            # another use (a training step leaves a cameras-only scene): re-pack from the kept inputs
            src = self._scene_src
            a = self._scene_inputs
            prec = a[8]
            if prec is None and precision != self.precision:
                prec = [self.precision]
            if prec is not None and not any(PRECISIONS[p] == PRECISIONS[precision] for p in prec):
                prec = list(prec) + [precision]
            self.set_scene(*a[:8], precisions=prec)
            self._scene_src = src
        return self._scene

    # ---- the reference's call surface ----
    def forward(self, rays: Dict[str, torch.Tensor], randomized: bool, white_bkgd: bool, near=None, far=None,
                out_depth: bool = False, chunk: Optional[int] = None, debug: bool = False) -> List[tuple]:
        """near/far are ignored exactly as the reference ignores them (quirk Q4, model.py:277-278)."""
        if torch.is_grad_enabled() and self.training and any(p.requires_grad for p in self.parameters()):
            return self._forward_train(rays, randomized, white_bkgd, out_depth)
        lib = L.load()
        sc = self._ensure_scene(rays)
        o = rays["rays_o"].contiguous().float()
        d = rays["rays_d"].contiguous().float()
        vd = rays["viewdirs"].contiguous().float()
        if not o.is_cuda:
            raise RuntimeError("neo360_b200 needs CUDA tensors (no CPU fallback)")
        n, dev = o.shape[0], o.device
        nc, nf = self.num_coarse_samples, self.num_fine_samples
        N = (nc + 1, nc + 1 + nf)
        cfg = L.NeoCfg()
        cfg.n_coarse, cfg.n_fine = nc, nf
        cfg.white_bkgd, cfg.out_depth = int(bool(white_bkgd)), int(bool(out_depth))
        cfg.precision = PRECISIONS[self.precision]
        keep = []
        if randomized:
            # same draw order and shapes as the reference: helper.py:50 (fg, bg) then helper.py:199 (fg, bg)
            u = [torch.rand((n, nc + 1), device=dev), torch.rand((n, nc + 1), device=dev),
                 torch.rand((n, nf), device=dev), torch.rand((n, nf), device=dev)]
            u = rays.get("_uniforms", u)
            keep.extend(u)
            cfg.u_fg0, cfg.u_bg0, cfg.u_fg1, cfg.u_bg1 = [L.ptr(x.contiguous()) for x in u]
        r = L.NeoRays()
        r.n_rays = n
        r.chunk = int(chunk if chunk is not None else (self.chunk or 0))
        r.rays_o, r.rays_d, r.viewdirs = L.ptr(o), L.ptr(d), L.ptr(vd)
        order = rays.get("_ray_order")
        if order is not None:
            keep.append(order)
            r.ray_order = order.data_ptr()
        need = lib.neo_render_workspace_bytes(n, C.byref(cfg))
        if need == 0:
            raise RuntimeError("neo360_b200: " + lib.neo_last_error().decode())
        if self._ws is None or self._ws.numel() < need or self._ws.device != dev:
            self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
        out = L.NeoOut()
        T: Dict[str, list] = {}

        def want(name, *shape_fn):
            T[name] = []
            for lvl in range(2):
                t = torch.empty(*[s(lvl) if callable(s) else s for s in shape_fn], device=dev)
                T[name].append(t)
                getattr(out, name)[lvl] = t.data_ptr()

        NL = lambda lvl: N[lvl]
        want("comp_rgb", n, 3)
        if out_depth:
            want("fg_rgb", n, 3); want("bg_rgb", n, 3); want("fg_acc", n); want("bg_lambda", n, 1); want("depth", n)
        else:
            want("fg_w", n, NL); want("bg_w", n, NL); want("fg_sdist", n, NL); want("bg_sdist", n, NL); want("bg_acc", n)
        if debug:
            for k in ("fg_t", "bg_s", "fg_sigma", "bg_sigma"):
                want(k, n, NL)
            want("fg_rgb_s", n, NL, 3); want("bg_rgb_s", n, NL, 3)
            if out_depth:
                want("fg_w", n, NL); want("bg_w", n, NL)
        with torch.cuda.device(dev):
            L.check(lib.neo_render_fwd(sc.handle, C.byref(r), C.byref(cfg), C.byref(out), self._ws.data_ptr(), self._ws.numel(),
                                       torch.cuda.current_stream().cuda_stream))
        ret = []
        for lvl in range(2):
            if out_depth:
                ret.append(tuple(T[k][lvl] for k in ("comp_rgb", "fg_rgb", "bg_rgb", "fg_acc", "bg_lambda", "depth")))
            else:
                ret.append(tuple(T[k][lvl] for k in ("comp_rgb", "fg_w", "bg_w", "fg_sdist", "bg_sdist", "bg_acc")))
        if debug:
            self.last_debug = T
        return ret

    def _forward_train(self, rays, randomized, white_bkgd, out_depth):
        """Training mode (models/neo360/model.py:725-732): the same tuples, differentiable w.r.t. the MLP parameters and the encoder
        outputs.  The feature maps come from the `rays` dict (`planes_xz|xy|yz`, `latent`), from `self.encoder` (run WITH autograd, so
        its parameters train too) or from the last `set_scene`.  See neo360_b200/training.py for what is hand-written CUDA."""
        from . import training
        if all(k in rays for k in ("planes_xz", "planes_xy", "planes_yz", "latent")):
            maps = [rays[k] for k in ("planes_xz", "planes_xy", "planes_yz", "latent")]
            cams = [rays[k] for k in ("src_poses", "src_focal", "src_c")]
            wh = (rays["src_imgs"].shape[-1], rays["src_imgs"].shape[-2]) if "src_imgs" in rays else self._scene_inputs[7]
        elif self.encoder is not None and "src_imgs" in rays:
            xz, xy, yz = self.encoder(rays["src_imgs"], rays["src_poses"], rays["src_focal"], rays["src_c"])
            maps = [xz, xy, yz, self.encoder.spatial_encoder.latent]
            cams = [rays[k] for k in ("src_poses", "src_focal", "src_c")]
            wh = (rays["src_imgs"].shape[-1], rays["src_imgs"].shape[-2])
        elif self._scene_inputs is not None:
            a = self._scene_inputs
            maps, cams, wh = list(a[:4]), list(a[4:7]), a[7]
        else:
            raise RuntimeError("no scene: call set_scene(...) or pass planes_*/latent in `rays`, or give an encoder")
        # reference formulation: the lookups read the scene's channel-last copies of THESE maps; projected formulation (default): the
        # scene only carries the cameras and grid geometry, the maps are projected under autograd in training.render_train
        self.set_scene(*maps, *cams, wh, precisions=[] if getattr(self, "train_projected", True) else ["fp32"])
        r = dict(rays)
        r["src_poses"] = cams[0]
        return training.render_train(self, r, maps[:3], maps[3], randomized, white_bkgd, out_depth, uniforms=rays.get("_uniforms"))

    # ---- stage-level operators that need the scene (parity tests) ----
    def index_grid(self, samples: torch.Tensor) -> torch.Tensor:
        """encoder_tp_fusion_conv.py:122-209: samples (...,3) world -> (NV*M,128), rows ordered (view, point)."""
        pts = samples.reshape(-1, 3).contiguous().float()
        out = torch.empty(self._scene.nv * pts.shape[0], 128, device=pts.device)
        with torch.cuda.device(pts.device):
            L.check(L.load().neo_index_grid(self._scene.handle, L.ptr(pts), pts.shape[0], L.ptr(out),
                                            torch.cuda.current_stream().cuda_stream))
        return out

    def get_local_feats(self, samples: torch.Tensor) -> torch.Tensor:
        """model.py:239-264: samples (...,3) world -> (NV*M,512)."""
        pts = samples.reshape(-1, 3).contiguous().float()
        out = torch.empty(self._scene.nv * pts.shape[0], 512, device=pts.device)
        with torch.cuda.device(pts.device):
            L.check(L.load().neo_index_local(self._scene.handle, L.ptr(pts), pts.shape[0], L.ptr(out),
                                             torch.cuda.current_stream().cuda_stream))
        return out

    def field_eval(self, rays, far, t_vals, mlp_index: int, chunk: int = 0, precision: Optional[str] = None,
                   ray_order: Optional[torch.Tensor] = None):
        """`predict` (model.py:343-407) of one branch: t/s (n,N) -> rgb (n,N,3), sigma (n,N,1).  `ray_order` (n) int32, a permutation
        of the rays, only changes the order in which the TC kernel visits them (NeoRays.ray_order); rows stay indexed by ray."""
        o, d, vd = (rays[k].contiguous().float() for k in ("rays_o", "rays_d", "viewdirs"))
        t = t_vals.contiguous().float()
        fr = far.reshape(-1).contiguous().float()
        n, N = t.shape
        r = L.NeoRays()
        r.n_rays, r.chunk = n, int(chunk)
        r.rays_o, r.rays_d, r.viewdirs = L.ptr(o), L.ptr(d), L.ptr(vd)
        if ray_order is not None:
            if ray_order.dtype != torch.int32 or ray_order.numel() != n or ray_order.device != t.device:
                raise ValueError("ray_order must be an int32 permutation of the rays on their device")
            ray_order = ray_order.contiguous()
            r.ray_order = ray_order.data_ptr()
        rgb = torch.empty(n, N, 3, device=t.device)
        sig = torch.empty(n, N, 1, device=t.device)
        with torch.cuda.device(t.device):
            L.check(L.load().neo_field_eval(self._scene.handle, C.byref(r), L.ptr(fr), L.ptr(t), N, mlp_index,
                                            PRECISIONS[precision or self.precision], L.ptr(rgb), L.ptr(sig),
                                            torch.cuda.current_stream().cuda_stream))
        return rgb, sig

    def density_grid(self, resolution, bbox=((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)), level: int = 1, precision: Optional[str] = None,
                     slab_rays: int = 16384, batch: Optional[Dict[str, torch.Tensor]] = None) -> torch.Tensor:
        """sigma of the foreground MLP of `level` on an (R_z, R_y, R_x) lattice over `bbox`; see neo360_b200.mesh.density_grid."""
        from . import mesh
        return mesh.density_grid(self, resolution, bbox, level, precision, slab_rays, batch)

    def check(self):
        """Synchronise and surface deferred device-side errors (the reference's asserts, helper.py:271,426)."""
        L.check(L.load().neo_check_async(self._scene.handle, torch.cuda.current_stream().cuda_stream))

    def _blocked_order(self, n: int, img_wh, dev) -> torch.Tensor:
        """Permutation visiting a row-major W x H frame in 8x4 pixel blocks: the 32 rays of a TC tile then hit neighbouring
        texels at every sample (L1 locality).  Pure scheduling: every ray's result is unchanged."""
        key = (n, int(img_wh[0]), int(img_wh[1]), str(dev))
        if getattr(self, "_order_key", None) != key:
            W = int(img_wh[0])
            idx = torch.arange(n, device=dev)
            y, x = idx // W, idx % W
            k = ((y // 4) * ((W + 7) // 8) + x // 8) * 32 + (y % 4) * 8 + (x % 8)
            self._order = torch.argsort(k).to(torch.int32).contiguous()
            self._order_key = key
        return self._order

    @torch.no_grad()
    def render_rays_test(self, batch: Dict[str, torch.Tensor], chunk: int = 1024, white_bkgd: bool = False, img_wh=None):
        """models/neo360/model.py:861-907 without the Python chunk loop: one call over every ray of the frame; the
        reference's per-chunk view-direction conditioning (quirk Q1) is reproduced from `chunk`.  `img_wh=(W,H)` (rays are the
        row-major pixels of a frame) lets the kernel walk the frame in 8x4 pixel blocks."""
        if img_wh is not None and batch["rays_o"].shape[0] == int(img_wh[0]) * int(img_wh[1]):
            batch = dict(batch)
            batch["_ray_order"] = self._blocked_order(batch["rays_o"].shape[0], img_wh, batch["rays_o"].device)
        out = self.forward(batch, False, white_bkgd, None, None, out_depth=True, chunk=chunk)[1]
        return {"rgb": out[0], "fg_rgb": out[1], "bg_rgb": out[2], "depth": out[5], "fg_acc": out[3]}
