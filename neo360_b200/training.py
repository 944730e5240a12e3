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
  * `net.train_precision = "tc"` (projected formulation only): layers 0-3 of the four MLPs and their view mean run forward and
    backward on the tensor cores in bf16 with fp32 accumulation (`_TrunkTC`, csrc/field_train.cu); the head runs once per point on the
    view mean (exact re-association).  The default "fp32" runs `_mlp_projected` under autograd.
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
        g_d = None
        if mode == 2 and ctx.needs_input_grad[3]:
            # alpha_i depends on sigma_i and |rays_d| only through sigma_i delta_i |rays_d|: dL/d|d| = sum_i g_sigma_i sigma_i / |d|
            g_d = (d_sig * sig_c).sum(-1, keepdim=True) / (d_c * d_c).sum(-1, keepdim=True) * d_c
        return d_rgb, d_sig.reshape(n, N, 1), None, g_d, None, None, None


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


def _trunk_workspace(need: int, dev) -> Tensor:
    """A byte buffer of the size a `*_train_workspace_bytes` query returned (0: the query refused the sizes)."""
    if need == 0:
        L.check(-1)
    return torch.empty(need, dtype=torch.uint8, device=dev)


def _trunk_grads(E: int, k3: int, dev) -> List[Tensor]:
    """Outputs of a trunk backward: gw0 (128, E), gb0, gw1 (128, 128), gb1, gw2 (128, 128), gb2, gw3 (128, k3), gb3."""
    return [torch.empty(128, E, device=dev), torch.empty(128, device=dev), torch.empty(128, 128, device=dev), torch.empty(128, device=dev),
            torch.empty(128, 128, device=dev), torch.empty(128, device=dev), torch.empty(128, k3, device=dev), torch.empty(128, device=dev)]


class _TrunkTC(torch.autograd.Function):
    """Layers 0-3 of a NeRFPPMLP and the view mean, projected formulation, on the tensor cores (csrc/field_train.cu, bf16 operands, fp32
    accumulation): cam (NV, M, in_ch) camera-frame encoding points, local_p / world_p (NV*M, 256) looked-up [P0 | P3], the encoding and
    h columns of layers 0 / 3 -> hbar (M, 128) = mean over the views of h3.  The backward returns one row gradient for local_p and
    world_p (their sum enters the layers) and every weight / bias gradient; no floating-point atomics."""

    @staticmethod
    def forward(ctx, cam, local_p, world_p, w0e, b0, w1, b1, w2, b2, w3e, b3):
        lib = L.load()
        nv, M, ich = cam.shape
        f = lambda t: t.detach().contiguous().float()
        cam_c, lp, wp = f(cam), f(local_p), f(world_p)
        ws = [f(t) for t in (w0e, b0, w1, b1, w2, b2, w3e, b3)]
        need = lib.neo_field_train_workspace_bytes(nv, M, ich, 0)
        saved = _trunk_workspace(need, cam.device)
        hbar = torch.empty(M, 128, device=cam.device)
        with torch.cuda.device(cam.device):
            L.check(lib.neo_field_train_fwd(L.ptr(cam_c), L.ptr(lp), L.ptr(wp), nv, M, ich, *[L.ptr(t) for t in ws], L.ptr(hbar),
                                            L.ptr(saved), need, _stream()))
        ctx.save_for_backward(saved, ws[2], ws[4], ws[6])
        ctx.dims = (nv, M, ich)
        return hbar

    @staticmethod
    def backward(ctx, g_hbar):
        lib = L.load()
        saved, w1, w2, w3e = ctx.saved_tensors
        nv, M, ich = ctx.dims
        E, dev = 21 * ich, saved.device
        need = lib.neo_field_train_workspace_bytes(nv, M, ich, 1)
        scratch = _trunk_workspace(need, dev)
        d_pm = torch.empty(nv * M, 256, device=dev)
        g = _trunk_grads(E, 128 + E, dev)
        with torch.cuda.device(dev):
            L.check(lib.neo_field_train_bwd(L.ptr(g_hbar.contiguous().float()), nv, M, ich, L.ptr(w1), L.ptr(w2), L.ptr(w3e), L.ptr(saved),
                                            saved.numel(), L.ptr(d_pm), *[L.ptr(t) for t in g], L.ptr(scratch), need, _stream()))
        return (None, d_pm, d_pm, *g)


class _PixelTrunkTC(torch.autograd.Function):
    """Layers 0-3 of PixelNeRF's NeRFMLP trunk and the view mean, projected formulation, on the tensor cores (the PixelNeRF form of
    csrc/field_train.cu): cam (NV, M, 3) camera-frame points, p0 (NV*M, 128) looked-up rows of latent . W0[:, 63:575]^T, the encoding
    columns of layer 0, layers 1-3 (no skip at layer 3) -> hbar (M, 128) = mean over the views of h3.  The backward returns the row
    gradient of p0 and every weight / bias gradient; no floating-point atomics."""

    @staticmethod
    def forward(ctx, cam, p0, w0e, b0, w1, b1, w2, b2, w3, b3):
        lib = L.load()
        nv, M, _ = cam.shape
        f = lambda t: t.detach().contiguous().float()
        cam_c, p0c = f(cam), f(p0)
        ws = [f(t) for t in (w0e, b0, w1, b1, w2, b2, w3, b3)]
        saved = _trunk_workspace(lib.neo_pixelnerf_train_workspace_bytes(nv, M, 0), cam.device)
        hbar = torch.empty(M, 128, device=cam.device)
        with torch.cuda.device(cam.device):
            L.check(lib.neo_pixelnerf_train_fwd(L.ptr(cam_c), L.ptr(p0c), nv, M, *[L.ptr(t) for t in ws], L.ptr(hbar), L.ptr(saved),
                                                saved.numel(), _stream()))
        ctx.save_for_backward(saved, ws[2], ws[4], ws[6])
        ctx.dims = (nv, M)
        return hbar

    @staticmethod
    def backward(ctx, g_hbar):
        lib = L.load()
        saved, w1, w2, w3 = ctx.saved_tensors
        nv, M = ctx.dims
        dev = saved.device
        need = lib.neo_pixelnerf_train_workspace_bytes(nv, M, 1)
        scratch = _trunk_workspace(need, dev)
        d_p0 = torch.empty(nv * M, 128, device=dev)
        g = _trunk_grads(63, 128, dev)
        with torch.cuda.device(dev):
            L.check(lib.neo_pixelnerf_train_bwd(L.ptr(g_hbar.contiguous().float()), nv, M, L.ptr(w1), L.ptr(w2), L.ptr(w3), L.ptr(saved),
                                                saved.numel(), L.ptr(d_p0), *[L.ptr(t) for t in g], L.ptr(scratch), need, _stream()))
        return (None, d_p0, *g)


def view_mean_head(mlp, hbar: Tensor, dir_tile: Tensor, nv: int):
    """The head after a view-averaged trunk, once per point: raw rgb and raw sigma from hbar (M, 128) and dir_tile (NV*M, 27).  Exact
    re-association of the per-view head: bottleneck -> views_linear.0 is linear and so is the view mean, so it runs on hbar and the view
    mean of the direction encodings, in fp32.  NeRFPPMLP and PixelNeRF's NeRFMLP share this head."""
    lin = lambda m, x: F.linear(x, m.weight, m.bias)
    M = hbar.shape[0]
    raw_sigma = lin(mlp.density_layer, hbar)
    dbar = dir_tile.reshape(nv, M, -1).mean(0)
    q = lin(mlp.views_linear[0], torch.cat([lin(mlp.bottleneck_layer, hbar), dbar], -1))
    q = torch.relu(lin(mlp.views_linear[1], torch.relu(q)))
    return lin(mlp.rgb_layer, q), raw_sigma


def _mlp_projected_tc(mlp, cam: Tensor, dir_tile: Tensor, local_p: Tensor, world_p: Tensor, nv: int):
    """`_mlp_projected` with the trunk (layers 0-3 and the view mean) on the tensor cores (`_TrunkTC`) and the head once per point
    (`view_mean_head`)."""
    E = 21 * cam.shape[-1]
    p = mlp.pts_linears
    hbar = _TrunkTC.apply(cam, local_p, world_p, p[0].weight[:, :E], p[0].bias, p[1].weight, p[1].bias, p[2].weight, p[2].bias,
                          p[3].weight[:, :128 + E], p[3].bias)
    return view_mean_head(mlp, hbar, dir_tile, nv)


TRAIN_PRECISIONS = ("fp32", "tc")
RAY_KEYS = ("rays_o", "rays_d", "viewdirs", "radii")


def rays_need_grad(rays: Dict[str, Tensor]) -> bool:
    """True when a ray tensor of the batch requires grad: vanilla NeRF and Mip-NeRF 360 then take their autograd path even with frozen parameters or in eval
    mode, so the rays (and, through ops.sample_rays, the camera poses) get gradients."""
    return any(k in rays and torch.is_tensor(rays[k]) and rays[k].requires_grad for k in RAY_KEYS)


def check_train_precision(p: str) -> str:
    if p not in TRAIN_PRECISIONS:
        raise ValueError(f"train_precision must be one of {TRAIN_PRECISIONS}, got {p!r}")
    return p


def _bf16(*shape, dev):
    return torch.empty(*shape, dtype=torch.bfloat16, device=dev)


def _ceil64(x: int) -> int:
    return (x + 63) // 64 * 64


class _MLPTrainTC(torch.autograd.Function):
    """The dense layers of vanilla NeRF's NeRFMLP and Mip-NeRF 360's PropMLP / NeRFMLP on the tensor cores (csrc/dense_train.cu and
    gemm_tc.cu: bf16 operands, fp32 accumulation, no floating-point atomics).  `depth` ReLU layers of width W on feats (M, F), the
    features concatenated after layer 4 when depth > 5, then the density head (bf16 rowdot) and, when the bottleneck parameters are
    given, the bottleneck and the beta columns of views_linear.0 (no bias).  params = w_i, b_i for every layer, density w, b, then
    optionally bottleneck w, b and views_linear.0.weight[:, :256] -> raw sigma (M, 1) fp32 and, with the bottleneck, y_beta (M, 128) fp32.
    Activations live in bf16: feats sit beside h4 in one [h4 | feats] buffer, so the skip layer reads one operand and the concatenation
    is never copied.  The backward runs dgrad (ReLU mask of the saved layer input in its epilogue, the density head's rank-1 gradient
    added to the last activation's) and wgrad per layer."""

    @staticmethod
    def forward(ctx, depth, feats, *params):
        lib = L.load()
        dev, s = feats.device, _stream()
        M, F = feats.shape
        f = lambda t: t.detach().contiguous().float()
        P = [f(t) for t in params]
        ws = [(P[2 * i], P[2 * i + 1]) for i in range(depth)]
        wsig, bsig = P[2 * depth], P[2 * depth + 1]
        rgb = len(P) > 2 * depth + 2
        W, Kf = ws[0][0].shape[0], _ceil64(F)
        skip = depth > 5
        fo = W if skip else 0
        XS = _bf16(M, fo + Kf, dev=dev)                                          # [h4 | feats] (feats alone without a skip)
        e = XS.data_ptr() + 2 * fo
        fc = f(feats)
        with torch.cuda.device(dev):
            L.check(lib.neo_tc_pack_bf16(L.ptr(fc), M, F, F, e, Kf, fo + Kf, 0, s))
            H, Wp, WT, X = [], [], [], []
            for i, (w, b) in enumerate(ws):
                kin = Kf if i == 0 else (W + Kf if skip and i == 5 else W)
                wp = _bf16(W, kin, dev=dev)
                L.check(lib.neo_tc_pack_bf16(L.ptr(w), W, w.shape[1], w.shape[1], wp.data_ptr(), kin, kin, 0, s))
                Wp.append(wp)
                if i > 0:
                    wt = _bf16(W, W, dev=dev)
                    L.check(lib.neo_tc_pack_bf16(L.ptr(w), W, w.shape[1], w.shape[1], wt.data_ptr(), W, W, 1, s))
                    WT.append(wt)
                x = (e, fo + Kf) if i == 0 else ((XS.data_ptr(), W + Kf) if skip and i == 5 else (H[-1].data_ptr(), W))
                X.append(x + (kin,))
                h = XS if skip and i == 4 else _bf16(M, W, dev=dev)
                L.check(lib.neo_tc_gemm_bf16(x[0], x[1], wp.data_ptr(), kin, L.ptr(b), h.data_ptr(), W + Kf if h is XS else W, M, W, kin, 0, s))
                H.append(h)
            hl = H[-1]
            sig = torch.empty(M, 1, device=dev)
            L.check(lib.neo_tc_rowdot_bf16(hl.data_ptr(), W, W, L.ptr(wsig), L.ptr(bsig), 1, M, L.ptr(sig), s))
            out, saved = (sig,), []
            if rgb:
                wb, bb, wv = P[2 * depth + 2], P[2 * depth + 3], P[2 * depth + 4]
                nb, nv = wb.shape[0], wv.shape[0]
                wbp, wvp, wbt, wvt = _bf16(nb, W, dev=dev), _bf16(nv, nb, dev=dev), _bf16(W, nb, dev=dev), _bf16(nb, nv, dev=dev)
                L.check(lib.neo_tc_pack_bf16(L.ptr(wb), nb, W, W, wbp.data_ptr(), W, W, 0, s))
                L.check(lib.neo_tc_pack_bf16(L.ptr(wv), nv, nb, nb, wvp.data_ptr(), nb, nb, 0, s))
                L.check(lib.neo_tc_pack_bf16(L.ptr(wb), nb, W, W, wbt.data_ptr(), W, nb, 1, s))
                L.check(lib.neo_tc_pack_bf16(L.ptr(wv), nv, nb, nb, wvt.data_ptr(), nb, nv, 1, s))
                beta = _bf16(M, nb, dev=dev)
                yb = torch.empty(M, nv, device=dev)
                L.check(lib.neo_tc_gemm_bf16(hl.data_ptr(), W, wbp.data_ptr(), W, L.ptr(bb), beta.data_ptr(), nb, M, nb, W, 1, s))
                L.check(lib.neo_tc_gemm_bf16(beta.data_ptr(), nb, wvp.data_ptr(), nb, None, yb.data_ptr(), nv, M, nv, nb, 2, s))
                out, saved = (sig, yb), [beta, wbt, wvt]
            # the input rows' gradient (pose refinement) reads W0^T and the skip layer's feature columns transposed, zero padded to Kf
            wft = []
            if feats.requires_grad:
                for i, c0 in ((0, 0),) + (((5, W),) if skip else ()):
                    w = ws[i][0]
                    wt = torch.zeros(Kf, W, dtype=torch.bfloat16, device=dev)
                    L.check(lib.neo_tc_pack_bf16(w.data_ptr() + 4 * c0, W, F, w.shape[1], wt.data_ptr(), F, W, 1, s))
                    wft.append((i, wt))
        ctx.save_for_backward(XS, *H, *WT, wsig, *saved)
        ctx.wft = wft
        ctx.meta = (depth, M, F, W, Kf, fo, X, [w.shape[1] for w, _ in ws], rgb)
        return out if rgb else sig

    @staticmethod
    def backward(ctx, g_sig, g_yb=None):
        lib = L.load()
        depth, M, F, W, Kf, fo, X, kvalid, rgb = ctx.meta
        T = ctx.saved_tensors
        XS, H, WT, wsig = T[0], T[1:1 + depth], T[1 + depth:2 * depth], T[2 * depth]
        hl = H[-1]
        dev, s = XS.device, _stream()
        g_sig = torch.zeros(M, 1, device=dev) if g_sig is None else g_sig.contiguous().float()
        calls = [(M, 64, W)] + [(M, W, x[2]) for x in X]
        if rgb:
            beta, wbt, wvt = T[2 * depth + 1:]
            nb, nv = beta.shape[1], wvt.shape[1]
            calls += [(M, nv, nb), (M, nb, W)]
        need = max(lib.neo_tc_wgrad_bf16_workspace_bytes(*c) for c in calls)
        if need == 0:
            L.check(-1)
        ws = torch.empty(need, dtype=torch.uint8, device=dev)
        wg = lambda dy, ldy, x, ldx, N, K, dw, kv, db: L.check(lib.neo_tc_wgrad_bf16(dy, ldy, x, ldx, M, N, K, L.ptr(dw), kv, L.ptr(db),
                                                                                     L.ptr(ws), need, s))
        G = [_bf16(M, W, dev=dev), _bf16(M, W, dev=dev)]
        grads = [None] * (2 * depth + 2)
        wft = dict(ctx.wft)
        g_in = {i: torch.empty(M, Kf, device=dev) for i in wft}
        extra = []
        with torch.cuda.device(dev):
            if rgb:
                g_yb = torch.zeros(M, nv, device=dev) if g_yb is None else g_yb.contiguous().float()
                dyb, dbeta = _bf16(M, nv, dev=dev), _bf16(M, nb, dev=dev)
                gwv, gwb, gbb = torch.empty(nv, nb, device=dev), torch.empty(nb, W, device=dev), torch.empty(nb, device=dev)
                L.check(lib.neo_tc_pack_bf16(L.ptr(g_yb), M, nv, nv, dyb.data_ptr(), nv, nv, 0, s))
                wg(dyb.data_ptr(), nv, beta.data_ptr(), nb, nv, nb, gwv, nb, None)
                L.check(lib.neo_tc_dgrad_bf16(dyb.data_ptr(), nv, wvt.data_ptr(), nv, None, 0, None, None, dbeta.data_ptr(), nb, M, nb, nv, s))
                wg(dbeta.data_ptr(), nb, hl.data_ptr(), W, nb, W, gwb, W, gbb)
                L.check(lib.neo_tc_dgrad_bf16(dbeta.data_ptr(), nb, wbt.data_ptr(), nb, hl.data_ptr(), W, L.ptr(g_sig), L.ptr(wsig),
                                              G[0].data_ptr(), W, M, W, nb, s))
                extra = [gwb, gbb, gwv]
            else:
                L.check(lib.neo_tc_relu_rank1_bf16(L.ptr(g_sig), L.ptr(wsig), hl.data_ptr(), W, M, W, G[0].data_ptr(), W, s))
            gs = _bf16(M, 64, dev=dev)
            gwsig = torch.empty(64, W, device=dev)
            L.check(lib.neo_tc_pack_bf16(L.ptr(g_sig), M, 1, 1, gs.data_ptr(), 64, 64, 0, s))
            wg(gs.data_ptr(), 64, hl.data_ptr(), W, 64, W, gwsig, W, None)
            grads[2 * depth], grads[2 * depth + 1] = gwsig[:1].clone(), g_sig.sum(0)
            for i in range(depth - 1, -1, -1):
                xp, ldx, kin = X[i]
                gw, gb = torch.empty(W, kvalid[i], device=dev), torch.empty(W, device=dev)
                wg(G[0].data_ptr(), W, xp, ldx, W, kin, gw, kvalid[i], gb)
                grads[2 * i], grads[2 * i + 1] = gw, gb
                if i in wft:        # dL/dz_i . W_i[:, feature columns] in fp32 (fp32 epilogue of the bf16 GEMM)
                    L.check(lib.neo_tc_gemm_bf16(G[0].data_ptr(), W, wft[i].data_ptr(), W, None, g_in[i].data_ptr(), Kf, M, Kf, W, 2, s))
                if i > 0:
                    L.check(lib.neo_tc_dgrad_bf16(G[0].data_ptr(), W, WT[i - 1].data_ptr(), W, xp, ldx, None, None, G[1].data_ptr(), W, M, W, W, s))
                    G.reverse()
        g_feats = None
        if g_in:
            g_feats = (g_in[0] + g_in[5] if 5 in g_in else g_in[0])[:, :F]
        return (None, g_feats, *grads, *extra)


def mlp_train_tc(m, feats: Tensor, denc: Tensor, n: int, N: int):
    """`_mlp_train` of vanilla.NeRFMLP, mip.PropMLP or mip.NeRFMLP with the dense layers on the tensor cores (`_MLPTrainTC`): feats
    (n*N, F), denc (n, 27) -> raw sigma (n*N, 1), raw rgb (n, N, 3) or None.  The direction columns of views_linear.0 with its bias and
    ReLU, and rgb_layer, stay fp32 framework ops, the direction columns applied once per ray."""
    layers = m.pts_linears if hasattr(m, "pts_linears") else m.pts_linear
    params = [t for lin in layers for t in (lin.weight, lin.bias)] + [m.density_layer.weight, m.density_layer.bias]
    rgb = hasattr(m, "rgb_layer")
    if not rgb:
        return _MLPTrainTC.apply(len(layers), feats, *params), None
    v, kb = m.views_linear[0], m.bottleneck_layer.out_features
    params += [m.bottleneck_layer.weight, m.bottleneck_layer.bias, v.weight[:, :kb]]
    sig, yb = _MLPTrainTC.apply(len(layers), feats, *params)
    y = yb.reshape(n, N, -1) + F.linear(denc, v.weight[:, kb:], v.bias)[:, None, :]
    return sig, F.linear(torch.relu(y), m.rgb_layer.weight, m.rgb_layer.bias)


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
    tc = getattr(net, "train_precision", "fp32")
    if tc not in TRAIN_PRECISIONS:
        raise ValueError(f"train_precision must be one of {TRAIN_PRECISIONS}, got {tc!r}")
    tc = tc == "tc"
    if tc and not projected:
        raise ValueError("train_precision='tc' runs the projected formulation only: set train_projected=True")
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
                if tc:
                    raw_rgb, raw_sigma = _mlp_projected_tc(mlp, cam, dir_tile, local_p, world_p, nv)
                else:
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


TEST_TIME_LR = 5e-6      # model.py:960-967: 5e-6 when the run resumes from a checkpoint, which run.py:84-92 always does


def test_time_optimizer(net, lr: float = TEST_TIME_LR, eval_modules: bool = True) -> torch.optim.Adam:
    """configure_optimizers for --is_optimize, the reference's test-time optimisation of a trained model on the source views of a new scene
    (model.py:957-981): the encoder's spatial_encoder (ResNet-34) is frozen, and Adam with betas (0.9, 0.999) runs over every parameter of
    `net` (the frozen ones never get a gradient).  optimizer_step then steps it with no learning-rate schedule and no gradient clipping
    (model.py:999-1000): see `test_time_step`.
    `eval_modules` (default True, configure_optimizers' evident intent) puts the spatial_encoder and every BatchNorm2d in eval mode, so
    their running statistics stay as trained and GridEncoder runs the frozen ResNet once per set of source images.  False leaves the
    modes alone: that is what the reference gets if its training loop calls `model.train()` after configure_optimizers (DESIGN.md
    section 8)."""
    if getattr(net, "encoder", None) is not None:
        net.encoder.spatial_encoder.requires_grad_(False)
    if eval_modules:
        setup_finetune_lpips(net)
    return torch.optim.Adam(net.parameters(), lr=lr, betas=(0.9, 0.999))


def test_time_step(net, opt: torch.optim.Optimizer, batch: Dict[str, Tensor], lpips_model=None) -> Tensor:
    """One step of the reference's test-time optimisation (training_step, model.py:697-820, and the --is_optimize branch of
    optimizer_step, model.py:999-1000): randomized forward, `training_loss` (with `lpips_model` for a --finetune_lpips patch batch),
    backward and a plain optimiser step: no schedule, no clip.  Returns the loss."""
    ret = net(batch, True, False, None, None, out_depth=False)
    loss = training_loss(ret, batch["target"], lpips_model=lpips_model)
    opt.zero_grad(set_to_none=True)
    loss.backward()
    opt.step()
    return loss.detach()


test_time_optimizer.__test__ = test_time_step.__test__ = False      # library functions, not pytest tests, when a test module imports them


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
