"""Differentiable (training) form of the NeO-360 hot path: `NeRF_TP.forward(..., out_depth=False)` under autograd.

Reference: models/neo360/model.py:266-581 (train tuple 564-579), training_step 697-820, distortion loss 1246-1260, DDP run.py:154.

What runs where
  * hand-written CUDA through the C ABI: ray / sphere intersection, stratified + inverse-CDF sampling (no gradient: the reference
    detaches sample positions, helper.py:225), the tri-plane and pixel-aligned lookups (forward `neo_index_grid|local`, backward
    `neo_index_grid_bwd|local_bwd`: 16-byte vector reductions into channel-last gradient maps), alpha compositing (forward
    `neo_volumetric_rendering`, backward `neo_volumetric_rendering_bwd`);
  * host framework (autograd + plain library GEMMs): the dense layers of NeRFPPMLP, activations, positional encodings, losses and the
    optimiser.
  * formulation: by default (`net.train_projected`, True) the training step uses the same exact re-association as the tensor-core
    inference kernel -- the lookups are linear, so the latent / tri-plane columns of layers 0 and 3 are applied to the feature MAPS once per
    step (`P = F . [W0_map ; W3_map]^T`, 0.4 M texels) instead of to every looked-up row (7.9 M point-views): the K = 703 / 831 input
    layers shrink to K = 63|84 and the lookups fetch 2 x 256 projected channels (`neo_index_maps`, backward `neo_index_maps_bwd`).  Autograd
    differentiates through the projection, so the map-column weights and the encoder outputs get exactly the reference's gradients (to
    fp32 re-association).  `train_projected = False` keeps the reference formulation row by row.
  * NCCL: ONE all-reduce over the flat gradient slab of the four MLPs per step (`allreduce_flat`), as the reference's DDP does.
  * under torch.use_deterministic_algorithms(True) the lookups' backward is the order-fixed `neo_index_maps_bwd_det` (sort + segmented
    reduction, bit-reproducible) and the distortion loss comes from `neo_distortion_loss`; with the flag off the code above runs unchanged.
There is no CPU fallback: every op raises on CPU tensors.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from . import _lib as L
from . import ops

Tensor = torch.Tensor


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _index_maps_bwd_det(sc, p, M, Cc, g_local, g_world, g_lat, g_pl):
    """neo_index_maps_bwd_det (no floating-point atomics, bit-reproducible) with a workspace of the queried size; a None row gradient skips
    its maps."""
    lib = L.load()
    need = lib.neo_index_maps_bwd_det_workspace_bytes(sc.handle, M, Cc)
    if need == 0:
        L.check(-1)
    ws = torch.empty(need, dtype=torch.uint8, device=p.device)
    f = lambda g: None if g is None else g.contiguous().float()
    L.check(lib.neo_index_maps_bwd_det(sc.handle, L.ptr(p), M, Cc, L.ptr(f(g_local)), L.ptr(f(g_world)), L.ptr(g_lat), *[L.ptr(t) for t in g_pl],
                                       L.ptr(ws), need, _stream()))


class _Lookup(torch.autograd.Function):
    """index_grid + get_local_feats (encoder_tp_fusion_conv.py:122-209, model.py:239-264) of world points (M,3):
    -> world (NV*M,128), local (NV*M,512); gradients flow to the three tri-planes and the latent image."""

    @staticmethod
    def forward(ctx, pts, planes_xz, planes_xy, planes_yz, latent, net):
        lib = L.load()
        p = pts.detach().reshape(-1, 3).contiguous().float()
        sc = net._scene
        M, nv = p.shape[0], sc.nv
        world = torch.empty(nv * M, 128, device=p.device)
        local = torch.empty(nv * M, 512, device=p.device)
        with torch.cuda.device(p.device):
            L.check(lib.neo_index_grid(sc.handle, L.ptr(p), M, L.ptr(world), _stream()))
            L.check(lib.neo_index_local(sc.handle, L.ptr(p), M, L.ptr(local), _stream()))
        ctx.save_for_backward(p)
        ctx.net, ctx.scene = net, sc
        ctx.shapes = (planes_xz.shape, latent.shape)
        ctx.det = torch.are_deterministic_algorithms_enabled()
        return world, local

    @staticmethod
    def backward(ctx, g_world, g_local):
        lib = L.load()
        (p,) = ctx.saved_tensors
        sc = ctx.scene
        (nv, cw, hp, wp), (_, cl, hl, wl) = ctx.shapes
        M = p.shape[0]
        g_planes = [torch.zeros(nv, hp, wp, cw, device=p.device) for _ in range(3)]
        g_lat = torch.zeros(nv, hl, wl, cl, device=p.device)
        with torch.cuda.device(p.device):
            if ctx.det:
                _index_maps_bwd_det(sc, p, M, cw, None, g_world, None, g_planes)
                _index_maps_bwd_det(sc, p, M, cl, g_local, None, g_lat, [None] * 3)
            else:
                L.check(lib.neo_index_grid_bwd(sc.handle, L.ptr(p), M, L.ptr(g_world.contiguous().float()), L.ptr(g_planes[0]),
                                               L.ptr(g_planes[1]), L.ptr(g_planes[2]), _stream()))
                L.check(lib.neo_index_local_bwd(sc.handle, L.ptr(p), M, L.ptr(g_local.contiguous().float()), L.ptr(g_lat), _stream()))
        nchw = lambda t: t.permute(0, 3, 1, 2)
        return None, nchw(g_planes[0]), nchw(g_planes[1]), nchw(g_planes[2]), nchw(g_lat), None


class _LookupMaps(torch.autograd.Function):
    """The two lookups over caller-owned channel-last maps of C channels (projected maps): lat_cl (NV,Hl,Wl,C), three planes
    (NV,Hp,Wp,C) -> local (NV*M,C), world (NV*M,C); gradients are scatter-added into channel-last gradient maps."""

    @staticmethod
    def forward(ctx, pts, lat_cl, xz_cl, xy_cl, yz_cl, net):
        lib = L.load()
        p = pts.detach().reshape(-1, 3).contiguous().float()
        sc = net._scene
        M, nv, Cc = p.shape[0], sc.nv, lat_cl.shape[-1]
        maps = [t.detach().contiguous().float() for t in (lat_cl, xz_cl, xy_cl, yz_cl)]
        local = torch.empty(nv * M, Cc, device=p.device)
        world = torch.empty(nv * M, Cc, device=p.device)
        with torch.cuda.device(p.device):
            L.check(lib.neo_index_maps(sc.handle, L.ptr(p), M, Cc, *[L.ptr(t) for t in maps], L.ptr(local), L.ptr(world), _stream()))
        ctx.save_for_backward(p)
        ctx.scene, ctx.C = sc, Cc
        ctx.shapes = (lat_cl.shape, xz_cl.shape)
        ctx.det = torch.are_deterministic_algorithms_enabled()
        return local, world

    @staticmethod
    def backward(ctx, g_local, g_world):
        lib = L.load()
        (p,) = ctx.saved_tensors
        sc, Cc = ctx.scene, ctx.C
        M = p.shape[0]
        g_lat = torch.zeros(ctx.shapes[0], device=p.device)
        g_pl = [torch.zeros(ctx.shapes[1], device=p.device) for _ in range(3)]
        with torch.cuda.device(p.device):
            if ctx.det:
                _index_maps_bwd_det(sc, p, M, Cc, g_local, g_world, g_lat, g_pl)
            else:
                L.check(lib.neo_index_maps_bwd(sc.handle, L.ptr(p), M, Cc, L.ptr(g_local.contiguous().float()),
                                               L.ptr(g_world.contiguous().float()), L.ptr(g_lat), L.ptr(g_pl[0]), L.ptr(g_pl[1]), L.ptr(g_pl[2]),
                                               _stream()))
        return None, g_lat, g_pl[0], g_pl[1], g_pl[2], None


class _Composite(torch.autograd.Function):
    """volumetric_rendering (helper.py:128-171): (rgb (B,N,3), sigma (B,N,1), t (B,N)) -> comp, acc, weights, bg_lambda, depth.
    `mode`: True / 1 = NeO-360 fg (reads far), False / 0 = NeO-360 bg, 2 = vanilla NeRF (models/vanilla_nerf/helper.py:521-559; far is
    None, bg_lambda is zeros, backward through neo_vanilla_composite_bwd)."""

    @staticmethod
    def forward(ctx, rgb, sigma, t, d, far, white, mode):
        lib = L.load()
        mode = int(mode)
        rgb_c, sig_c = rgb.detach().contiguous().float(), sigma.detach().reshape(sigma.shape[0], -1).contiguous().float()
        t_c, d_c = t.detach().contiguous().float(), d.detach().contiguous().float()
        far_c = far.detach().reshape(-1).contiguous().float() if far is not None else None
        n, N = t_c.shape
        dev = t_c.device
        comp, acc = torch.empty(n, 3, device=dev), torch.empty(n, device=dev)
        w, depth = torch.empty(n, N, device=dev), torch.empty(n, device=dev)
        lam = torch.empty(n, 1, device=dev) if mode == 1 else torch.zeros(n, 1, device=dev)
        with torch.cuda.device(dev):
            L.check(lib.neo_volumetric_rendering(L.ptr(rgb_c), L.ptr(sig_c), L.ptr(t_c), L.ptr(d_c), L.ptr(far_c), n, N, int(bool(white)),
                                                 mode, L.ptr(comp), L.ptr(acc), L.ptr(w), L.ptr(lam) if mode == 1 else None,
                                                 L.ptr(depth), _stream()))
        ctx.save_for_backward(rgb_c, sig_c, t_c, d_c, far_c)
        ctx.flags = (int(bool(white)), mode)
        return comp, acc, w, lam, depth

    @staticmethod
    def backward(ctx, g_comp, g_acc, g_w, g_lam, g_depth):
        lib = L.load()
        rgb_c, sig_c, t_c, d_c, far_c = ctx.saved_tensors
        white, mode = ctx.flags
        n, N = t_c.shape
        dev = t_c.device
        d_rgb, d_sig = torch.empty(n, N, 3, device=dev), torch.empty(n, N, device=dev)
        f = lambda g: None if g is None else g.contiguous().float()
        with torch.cuda.device(dev):
            if mode == 2:
                gs = [f(g_comp), f(g_acc), f(g_w), f(g_depth)]
                L.check(lib.neo_vanilla_composite_bwd(L.ptr(rgb_c), L.ptr(sig_c), L.ptr(t_c), L.ptr(d_c), n, N, white,
                                                      *[L.ptr(g) for g in gs], L.ptr(d_rgb), L.ptr(d_sig), _stream()))
            else:
                gs = [f(g_comp), f(g_acc), f(g_w), f(g_lam) if mode else None, f(g_depth)]
                L.check(lib.neo_volumetric_rendering_bwd(L.ptr(rgb_c), L.ptr(sig_c), L.ptr(t_c), L.ptr(d_c), L.ptr(far_c), n, N, white, mode,
                                                         *[L.ptr(g) for g in gs], L.ptr(d_rgb), L.ptr(d_sig), _stream()))
        return d_rgb, d_sig.reshape(n, N, 1), None, None, None, None, None


def _pos_enc(x: Tensor, min_deg: int, max_deg: int) -> Tensor:
    """helper.py:121-125"""
    scales = torch.tensor([2.0 ** i for i in range(min_deg, max_deg)], dtype=x.dtype, device=x.device)
    xb = (x[..., None, :] * scales[:, None]).reshape(*x.shape[:-1], -1)
    return torch.cat([x, torch.sin(torch.cat([xb, xb + 0.5 * math.pi], -1))], -1)


def _world2camera(x: Tensor, c2w: Tensor) -> Tensor:
    """util.py:52-70: (M,3) world points, (NV,4,4) camera-to-world -> (NV,M,3)."""
    rot = c2w[:, :3, :3].transpose(1, 2)
    trans = -torch.bmm(rot, c2w[:, :3, 3:])
    return torch.matmul(rot[:, None], x[None, :, :, None])[..., 0] + trans[:, None, :, 0]


def _world2camera_dirs(v: Tensor, c2w: Tensor) -> Tensor:
    rot = c2w[:, :3, :3].transpose(1, 2)
    return torch.matmul(rot[:, None], v[None, :, :, None])[..., 0]


def _mlp(mlp, enc: Tensor, dir_tile: Tensor, world: Tensor, local: Tensor, nv: int):
    """NeRFPPMLP.forward (model.py:110-158): enc (NV,M,63|84), dir_tile (NV*M,27), world (NV*M,128), local (NV*M,512)."""
    M = enc.shape[1]
    lin = lambda m, x: F.linear(x, m.weight, m.bias)
    inp = torch.cat([enc.reshape(-1, enc.shape[-1]), local, world], -1)
    h = torch.relu(lin(mlp.pts_linears[0], inp))
    h = torch.relu(lin(mlp.pts_linears[1], h))
    h = torch.relu(lin(mlp.pts_linears[2], h))
    h = torch.relu(lin(mlp.pts_linears[3], torch.cat([h, inp], -1)))
    beta = lin(mlp.bottleneck_layer, h)
    raw_sigma = lin(mlp.density_layer, h.reshape(nv, M, -1).mean(0))
    q = lin(mlp.views_linear[0], torch.cat([beta, dir_tile], -1)).reshape(nv, M, -1).mean(0)
    q = torch.relu(lin(mlp.views_linear[1], torch.relu(q)))
    return lin(mlp.rgb_layer, q), raw_sigma


def _project_maps(mlp, enc_dim: int, latent_cl: Tensor, planes_cl: List[Tensor]):
    """[P0 | P3] = F . [W0_map ; W3_map]^T per map: the latent (512) / tri-plane (128) columns of layers 0 and 3 applied to the channel-last
    feature maps (model.py:110-158: x = [enc | local 512 | world 128], layer 3 sees [h 128 | x])."""
    w0, w3 = mlp.pts_linears[0].weight, mlp.pts_linears[3].weight
    wl = torch.cat([w0[:, enc_dim:enc_dim + 512], w3[:, 128 + enc_dim:128 + enc_dim + 512]], 0)       # (256, 512)
    ww = torch.cat([w0[:, enc_dim + 512:], w3[:, 128 + enc_dim + 512:]], 0)                              # (256, 128)
    return latent_cl @ wl.t(), [pc @ ww.t() for pc in planes_cl]


def _mlp_projected(mlp, enc: Tensor, dir_tile: Tensor, local_p: Tensor, world_p: Tensor, nv: int):
    """NeRFPPMLP.forward with the map columns of layers 0 / 3 already applied: local_p, world_p (NV*M, 256) = looked-up [P0 | P3]."""
    M, E = enc.shape[1], enc.shape[-1]
    lin = lambda m, x: F.linear(x, m.weight, m.bias)
    e = enc.reshape(-1, E)
    w0, w3 = mlp.pts_linears[0], mlp.pts_linears[3]
    pm = local_p + world_p
    h = torch.relu(F.linear(e, w0.weight[:, :E], w0.bias) + pm[:, :128])
    h = torch.relu(lin(mlp.pts_linears[1], h))
    h = torch.relu(lin(mlp.pts_linears[2], h))
    h = torch.relu(F.linear(torch.cat([h, e], -1), w3.weight[:, :128 + E], w3.bias) + pm[:, 128:])
    beta = lin(mlp.bottleneck_layer, h)
    raw_sigma = lin(mlp.density_layer, h.reshape(nv, M, -1).mean(0))
    q = lin(mlp.views_linear[0], torch.cat([beta, dir_tile], -1)).reshape(nv, M, -1).mean(0)
    q = torch.relu(lin(mlp.views_linear[1], torch.relu(q)))
    return lin(mlp.rgb_layer, q), raw_sigma


def render_train(net, rays: Dict[str, Tensor], planes: List[Tensor], latent: Tensor, randomized: bool, white_bkgd: bool,
                 out_depth: bool = False, uniforms: Optional[List[Tensor]] = None):
    """NeRF_TP.forward (model.py:266-581, encoder hoisted) with autograd through the MLP parameters, `planes` (xz, xy, yz) and `latent`.
    `net` must hold a scene built from exactly these feature maps with the fp32 path prepared (`set_scene(..., precisions=["fp32"])`)."""
    o, d, vd = (rays[k].contiguous().float() for k in ("rays_o", "rays_d", "viewdirs"))
    if not o.is_cuda:
        raise RuntimeError("neo360_b200 needs CUDA tensors (no CPU fallback)")
    B, nv = o.shape[0], net._scene.nv
    nc, nf = net.num_coarse_samples, net.num_fine_samples
    poses = rays["src_poses"].float() if "src_poses" in rays else net._scene_inputs[4].float()
    far = ops.intersect_sphere(o, d)                                            # (B,1); near / far arguments ignored (quirk Q4)
    near = torch.full_like(far, 1e-4)
    dirs_cam = _world2camera_dirs(vd, poses)                                     # (NV,B,3)
    denc = _pos_enc(dirs_cam, 0, 4)                                              # (NV,B,27)
    u = uniforms if uniforms is not None else [None] * 4
    mlps = net._mlps()                                                           # fg_coarse, bg_coarse, fg_fine, bg_fine
    projected = getattr(net, "train_projected", True)
    if projected:
        latent_cl = latent.permute(0, 2, 3, 1)                                   # channel-last views: the projection contracts the last axis
        planes_cl = [pl.permute(0, 2, 3, 1) for pl in planes]
    ret = []
    fg_t = bg_s = fg_w = bg_w = None
    for level in range(2):
        if level == 0:
            fg_t, fg_pts = ops.sample_along_rays(o, d, nc, near, far, randomized, False, True, 3.0, u_rand=u[0])
            bg_s, bg_pts, bg_lin = ops.sample_along_rays(o, d, nc, near, far, randomized, False, False, 3.0, u_rand=u[1])
        else:
            fg_t, fg_pts = ops.sample_pdf(fg_t, fg_w.detach(), o, d, nf, randomized, True, far, 3.0, u_rand=u[2])
            bg_s, bg_pts, bg_lin = ops.sample_pdf(bg_s, bg_w.detach(), o, d, nf, randomized, False, far, 3.0, u_rand=u[3])
        N = fg_t.shape[1]
        dir_tile = denc[:, None].repeat(1, 1, N, 1).reshape(-1, denc.shape[-1])  # quirk Q1: row j sees ray (j mod B)
        out = []
        for b, (enc_pts, look_pts, tvals) in enumerate(((fg_pts, fg_pts, fg_t), (bg_pts, bg_lin, bg_s))):
            cam = _world2camera(enc_pts[..., :3].reshape(-1, 3), poses)          # (NV,B*N,3)
            if b == 1:
                cam = torch.cat([cam, enc_pts[..., 3].reshape(1, -1, 1).repeat(nv, 1, 1)], -1)
            mlp = mlps[2 * level + b]
            if projected:
                pl_cl, pp_cl = _project_maps(mlp, 63 if b == 0 else 84, latent_cl, planes_cl)
                local_p, world_p = _LookupMaps.apply(look_pts.reshape(-1, 3), pl_cl, pp_cl[0], pp_cl[1], pp_cl[2], net)
                raw_rgb, raw_sigma = _mlp_projected(mlp, _pos_enc(cam, 0, 10), dir_tile, local_p, world_p, nv)
            else:
                world, local = _Lookup.apply(look_pts.reshape(-1, 3), planes[0], planes[1], planes[2], latent, net)
                raw_rgb, raw_sigma = _mlp(mlp, _pos_enc(cam, 0, 10), dir_tile, world, local, nv)
            sigma = F.softplus(raw_sigma.reshape(B, N, 1) - 1.0)                 # model.py:392-393
            rgb = torch.sigmoid(raw_rgb.reshape(B, N, 3)) * (1 + 2 * 0.001) - 0.001
            wb = False if out_depth else white_bkgd                              # model.py:501,519 vs 551,560
            out.append(_Composite.apply(rgb, sigma, tvals, d, far, wb, b == 0))
        (fg_c, fg_acc, fg_w, lam, fg_depth), (bg_c, bg_acc, bg_w, _, bg_depth) = out
        comp = fg_c + lam * bg_c
        if out_depth:
            ret.append((comp, fg_c, bg_c, fg_acc, lam, fg_depth + lam.squeeze(-1) * bg_depth))
        else:
            fg_m = 0.5 * (fg_t[..., 1:] + fg_t[..., :-1])
            fg_m = torch.cat([fg_m, (fg_m[:, -1] + (fg_m[:, -1] - fg_m[:, -2]))[:, None]], -1)
            bg_m = torch.cat([0.5 * (bg_s[..., 1:] + bg_s[..., :-1]), bg_s[..., -1:]], -1)
            ret.append((comp, fg_w, bg_w, fg_m, bg_m, bg_acc))
    return ret


class _Distortion(torch.autograd.Function):
    """Per-ray distortion regulariser (neo_distortion_loss, backward neo_distortion_loss_bwd): w, m, interval (n,N) -> (n,).  Fixed-order
    sums, no atomics; m and interval carry no gradient."""

    @staticmethod
    def forward(ctx, w, m, interval):
        lib = L.load()
        wc, mc, ic = (t.detach().contiguous().float() for t in (w, m, interval))
        n, N = wc.shape
        out = torch.empty(n, device=wc.device)
        with torch.cuda.device(wc.device):
            L.check(lib.neo_distortion_loss(L.ptr(wc), L.ptr(mc), L.ptr(ic), 0.0, n, N, L.ptr(out), _stream()))
        ctx.save_for_backward(wc, mc, ic)
        return out

    @staticmethod
    def backward(ctx, g):
        lib = L.load()
        wc, mc, ic = ctx.saved_tensors
        n, N = wc.shape
        d_w = torch.empty_like(wc)
        with torch.cuda.device(wc.device):
            L.check(lib.neo_distortion_loss_bwd(L.ptr(wc), L.ptr(mc), L.ptr(ic), 0.0, n, N, L.ptr(g.contiguous().float()), L.ptr(d_w), _stream()))
        return d_w, None, None


def distortion_loss(w: Tensor, m: Tensor, interval: Tensor) -> Tensor:
    """The O(N) form of the regulariser the reference applies through `eff_distloss` (models/neo360/model.py:1246-1260; same functional
    as the in-tree O(N^2) lossfun_distortion, helper.py:111-118):  1/3 sum_i interval_i w_i^2 + 2 sum_i w_i (m_i W_{<i} - (wm)_{<i}).
    Under torch.use_deterministic_algorithms on CUDA tensors (where torch.cumsum raises) the per-ray values come from neo_distortion_loss."""
    if torch.are_deterministic_algorithms_enabled() and w.is_cuda:
        N = w.shape[-1]
        flat = lambda t: t.expand_as(w).reshape(-1, N)
        return _Distortion.apply(w.reshape(-1, N), flat(m), flat(interval)).mean()
    loss_uni = (1.0 / 3.0) * (interval * w.pow(2)).sum(-1).mean()
    wm = w * m
    w_cum, wm_cum = w.cumsum(-1), wm.cumsum(-1)
    loss_bi = 2.0 * (wm[..., 1:] * w_cum[..., :-1] - w[..., 1:] * wm_cum[..., :-1]).sum(-1).mean()
    return loss_uni + loss_bi


LPIPS_LAMBDA = 0.3      # model.py:1308


def lpips_loss(rgb: Tensor, target: Tensor, model) -> Tensor:
    """NeRF_TP.lpips_loss (model.py:1283-1309): 0.3 LPIPS of the 30x30 patch whose (900, 3) colours are `rgb` (patch order of
    batches.patch_batch) against `target`, with lpips' scaling (csrc/lpips.cu form 1) and an `neo360_b200.lpips.LPIPS` model.  The
    gradient flows to `rgb`.  The 1x1 layers have no dropout: the term is the reference's in eval mode (DESIGN.md section 8)."""
    from .lpips import FORM_LPIPS
    from .batches import PATCH
    d = model(rgb.reshape(1, PATCH, PATCH, 3), target.reshape(1, PATCH, PATCH, 3), FORM_LPIPS)
    return d.float()[0] * LPIPS_LAMBDA


def setup_finetune_lpips(net) -> List[torch.nn.Parameter]:
    """What configure_optimizers does for --finetune_lpips (model.py:957-981): freeze the encoder's spatial_encoder and put it in eval
    mode, put every BatchNorm2d of `net` in eval mode.  Returns the parameters that still train, for the optimiser and the gradient clip;
    the LPIPS model is not part of `net`, so its parameters stay out of both.  Call it after `net.train()`, which would undo the eval
    modes."""
    if getattr(net, "encoder", None) is not None:
        net.encoder.spatial_encoder.requires_grad_(False)
        net.encoder.spatial_encoder.eval()
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.eval()
    return [p for p in net.parameters() if p.requires_grad]


def training_loss(ret, target: Tensor, dist_weight: float = 0.01, lpips_model=None) -> Tensor:
    """MSE of both levels + distortion regulariser on the fine level (model.py:740-748, 1246-1260).  With `lpips_model` (the
    --finetune_lpips variant, model.py:750-755) the LPIPS loss of both levels' patch colours is added before the regulariser."""
    loss = ((ret[0][0] - target) ** 2).mean() + ((ret[1][0] - target) ** 2).mean()
    if lpips_model is not None:
        loss = loss + (lpips_loss(ret[0][0], target, lpips_model) + lpips_loss(ret[1][0], target, lpips_model))
    _, fg_w, bg_w, fg_m, bg_m, _ = ret[1]
    n = fg_w.shape[-1]
    loss = loss + dist_weight * (distortion_loss(fg_w, fg_m, torch.full_like(fg_w, 1.0 / n)) + distortion_loss(bg_w, bg_m, torch.full_like(bg_w, 1.0 / n)))
    return loss


def allreduce_flat(params, world: int, dist) -> Tensor:
    """ONE NCCL all-reduce over the flat slab of every parameter gradient (mean over ranks), written back in place."""
    grads = [p.grad if p.grad is not None else torch.zeros_like(p) for p in params]
    flat = torch._utils._flatten_dense_tensors(grads)
    if dist is not None and world > 1:
        dist.all_reduce(flat, op=dist.ReduceOp.SUM)
        flat.div_(world)
        for p, g in zip(params, torch._utils._unflatten_dense_tensors(flat, grads)):
            p.grad = g.clone() if p.grad is None else p.grad.copy_(g)
    return flat


def bench_train(args, rank, world, local, dev, dist, pk, base, sampler, timed):
    """BASELINE configs[3]: `--batch-rays` rays per step split over the ranks, synthetic NERDS360-shaped scene per rank (encoder out of
    scope: its outputs are leaf tensors that receive gradients), targets = a fixed random image, Adam + clip 0.05 (model.py:1003-1025)."""
    import bench as Bm
    from . import NeRF_TP, synth
    from .encoder import GridEncoder
    with_encoder = not getattr(args, "freeze_encoder", False)
    tf32 = getattr(args, "train_matmul", "fp32") == "tf32"
    torch.backends.cuda.matmul.allow_tf32 = tf32                # forward and backward GEMMs of the dense layers (and the encoder's linears)
    torch.backends.cudnn.allow_tf32 = tf32                      # encoder convolutions
    sc = synth.make_scene((Bm.IMG_W, Bm.IMG_H), Bm.NV, (120, 160), seed=rank)
    torch.manual_seed(0)                                        # identical initial weights on every rank (what DDP's broadcast gives)
    enc = GridEncoder() if with_encoder else None
    net = NeRF_TP(num_coarse_samples=Bm.N_COARSE, num_fine_samples=Bm.N_FINE, num_src_views=Bm.NV, precision="fp32", encoder=enc)
    sd = net.state_dict()
    sd.update(synth.make_mlp_params(0))
    net.load_state_dict(sd)
    net = net.to(dev).train()
    net.train_projected = getattr(args, "train_formulation", "projected") == "projected"
    cams = [sc[k].to(dev) for k in ("src_poses", "src_focal", "src_c")]
    if with_encoder:
        # the reference's training step (models/neo360/model.py:697-820): the encoder runs inside the step and trains through the renderer
        g0 = torch.Generator().manual_seed(77 + rank)
        src_imgs = (torch.rand(Bm.NV, 3, Bm.IMG_H, Bm.IMG_W, generator=g0) * 2 - 1).to(dev)
        maps = {}
        params = [p for p in net.parameters() if p.requires_grad]
    else:
        maps = {k: sc[k].to(dev).requires_grad_(True) for k in ("planes_xz", "planes_xy", "planes_yz", "latent")}
        params = [p for m in net._mlps() for p in m.parameters()]
    opt = torch.optim.Adam(params, lr=5e-4)
    per = args.batch_rays // world
    # dataset side (row f3): 20 target views of this rank's scene resident in HBM; per step the host draws `pix_inds` exactly like
    # nerds360_ae.py:730-732 and the sampled rays + target colours are produced on the device (batches.train_batch)
    from . import batches
    g = torch.Generator().manual_seed(1234 + rank)
    tposes = torch.stack([synth.target_pose((5 * k + rank) % 100, 100)[:3, :4] for k in range(batches.NUM_TARGET_VIEWS)]).to(dev)
    timgs = torch.rand(batches.NUM_TARGET_VIEWS, Bm.IMG_H, Bm.IMG_W, 3, generator=g).to(dev)
    views = batches.TargetViews(tposes, timgs, 0.8 * Bm.IMG_W)
    pix_host = torch.empty(per, dtype=torch.int64).pin_memory()
    state = {}

    def step(s):
        pix_host.copy_(batches.draw_pix_inds(views.T, views.H, views.W, per, g))
        src = {"src_poses": cams[0], "src_focal": cams[1], "src_c": cams[2]}
        if with_encoder:
            src["src_imgs"] = src_imgs
        else:
            src["src_imgs"] = torch.empty(Bm.NV, 3, Bm.IMG_H, Bm.IMG_W, device="meta")      # only its shape is read (image size)
        batch = batches.train_batch(views, src, pix_inds=pix_host)
        if not with_encoder:
            batch.update(maps)
        tgt = batch["target"]
        ret = net(batch, True, False, None, None, out_depth=False)
        loss = training_loss(ret, tgt)
        opt.zero_grad(set_to_none=True)
        for t in maps.values():
            t.grad = None
        loss.backward()
        flat = allreduce_flat(params, world, dist)
        torch.nn.utils.clip_grad_norm_(params, 0.05)
        opt.step()
        state["loss"] = loss.detach()
        state["grad_elems"] = flat.numel()

    if sampler:
        sampler.start()
    ms = timed(step, args.steps, args.warmup, dev, dist)
    if sampler:
        sampler.stop_flag = True
    loss = float(state["loss"].item())
    rays = per * world * args.steps
    return dict(base, metric="training rays/sec, neo360 generalisable training, 4096-ray batches", value=rays / (ms * 1e-3),
                ms_per_step=ms / args.steps, scaling="strong", dtype="tf32" if tf32 else "f32",
                config={"workload": "neo360 training step (BASELINE configs[3]): stratified + PDF sampling, lookups, NeRFPPMLP x4, compositing, "
                                    "MSE + distortion loss, backward, NCCL gradient all-reduce, clip 0.05, Adam",
                        "batch_rays": per * world, "rays_per_rank": per, "samples": "128+64",
                        "precision": "fp32 (reference formulation)" + ("; framework GEMMs / convolutions in TF32 (the reference's torch-1.11 default)" if tf32 else ""),
                        "parallelism": f"data parallel x{world}: one all-reduce over a flat {state['grad_elems']}-element gradient slab per step",
                        "encoder": "GridEncoder inside the step (dense_train: grid lookup and softmax pillar sums forward / backward in hand-written "
                                   "CUDA, dense layers as framework GEMMs; ResNet and conv stacks framework), its gradients in the all-reduced slab"
                                   if with_encoder
                                   else "frozen / absent: encoder outputs are leaf tensors (finetune mode, model.py:969-979)",
                        "batch": "pix_inds drawn on the host as the reference dataset does, rays + targets of the sampled pixels generated on the device "
                                 "from 20 resident target views (neo_sample_rays)",
                        "formulation": "projected maps: [W0_map; W3_map] applied to the 0.4 M map texels once per step under autograd, lookups of 2x256 projected "
                                       "channels, K=63|84 input layers (exact re-association)" if net.train_projected
                                       else "reference: row-by-row K=703/831 input layers on the looked-up 640 raw channels",
                        "hand_written": "pixel sampling, ray sampling, lookups fwd/bwd, compositing fwd/bwd", "library": "dense layers, encoder GEMMs and convolutions (autograd), Adam"},
                e2e={"value": rays / (ms * 1e-3), "unit": "rays/s", "h2d_bytes_per_step": per * 8, "d2h_bytes_per_step": 4},
                final_loss=loss, clocks=sampler.result() if sampler else None)
