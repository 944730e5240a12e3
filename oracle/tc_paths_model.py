"""TEST INFRASTRUCTURE ONLY -- float64 models of the vanilla NeRF, Mip-NeRF 360 and GridEncoder tensor-core paths.

Each function restates, point by point (or pillar by pillar), what the NEO_PREC_TC path of `csrc/vanilla.cu`, `csrc/mip.cu` or
`csrc/encoder.cu` computes, with every fp16 rounding it applies made explicit (`tc_model._round`):

* vanilla_tc_field: points x = fp32(o + fp32(t viewdirs)); encoding [x | sin 2^k x (k-major) | cos | 0] fp16 (64 columns), direction
  encoding fp16 (27 columns, zero padded); weights fp16 packed as `neo_vanilla_create` packs them (layer 5 = [h4 | enc] split at column
  256); fp32 biases added in the epilogue, ReLU, fp16 after every trunk layer; bottleneck fp16 without ReLU; view layer fp16 after ReLU;
  sigma / rgb heads = fp16 rows times the fp32 weights (`rowdot_f16`) + bias, then softplus(x - 1) / sigmoid * 1.002 - 0.001.
* mip_tc_field: cast_cone -> contract -> ipe_features in float64, rounded to fp16 (504 columns, zero padded to 512); the same layer chain
  with the [h4 | features] skip at layer 5; `rowdot_f16` heads; activations of `mip::composite_kernel`.
* encoder_tc_dense: gathered row [bilinear latent | cam xyz | masked unit direction | 0] fp16; DepthPillarEncoder with fp16 weights,
  Ha / Hb fp16 after ReLU, L fp16 without; coordinate column fp16; aggregator hidden layer fp16 after ReLU; logits = fp16 Ha times the
  fp32 second aggregator layer + bias; softmax over the 64 cells and the weighted sum of the fp16 L rows.  Only the cells of the
  requested pillars are evaluated.

`fp16=False` turns every rounding into the identity; each model then equals its oracle (`vanilla_oracle.mlp_forward`, `mip_oracle.mlp`,
`GridEncoder.dense_torch`) to 1e-9 in float64 (tests/test_tc_paths_model.py).  `mutation=` applies one named value-level bug (the
*_MUTATIONS tuples), used on the CPU to show that the GPU bounds (*_TOL below, tests/test_gpu_tc_paths.py) would catch it.
Nothing under `neo360_b200/` imports this file.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn.functional as F

from . import mip_oracle as mo
from . import neo360_oracle as orc
from .tc_model import _round, blend

Tensor = torch.Tensor

# Bounds of the GPU tests (tests/test_gpu_tc_paths.py), set at 2-3x the largest values measured there on an H100 80GB HBM3 at a 400 W
# power limit (measured in the comments; DESIGN.md section 2).  Per point: |rgb - model| <= *_RGB_TOL and the sigma / density error in
# units of its pre-activation, |sigma - model| / (1 - exp(-model)), <= *_SIGMA_TOL; per case, the means of those errors <= *_MEAN_TOL.
# The per-point maxima are fp16 rounding noise: the kernels' fp32 geometry and angle doubling move an encoding by up to ~1 fp16 ulp,
# and once one fp16 rounding of a point differs, its later roundings decorrelate from the model's.  The means stay an order lower.
VAN_RGB_TOL, VAN_SIGMA_TOL, VAN_RGB_MEAN_TOL, VAN_SIGMA_MEAN_TOL = 4e-3, 1e-2, 5e-4, 1e-3      # measured 1.5e-3, 4.3e-3, 1.9e-4, 3.4e-4
MIP_RGB_TOL, MIP_SIGMA_TOL, MIP_RGB_MEAN_TOL, MIP_SIGMA_MEAN_TOL = 1e-3, 1.5e-3, 2.5e-4, 2e-4  # measured 3.3e-4, 5.3e-4, 8.7e-5, 7.4e-5
# encoder pillar sums, relative to the largest |pillar sum| of the case: per element and the per-case mean (measured 1.9e-4, 2.9e-6)
ENC_TOL, ENC_MEAN_TOL = 5e-4, 8e-6

VANILLA_MUTATIONS = ("sigma_short", "l6_no_bias", "dir_swap34", "l5_enc_shift", "oct9_cos_early")
MIP_MUTATIONS = ("skip_offset", "ipe_var_2k", "dir_cos_zero", "rgb_short")
ENCODER_MUTATIONS = ("no_dir_mask", "cam_dir_swap", "no_size_ratio", "coord_axis", "border_clamp")


def _check(mutation, allowed):
    if mutation is not None and mutation not in allowed:
        raise ValueError(f"unknown mutation {mutation!r}")


def sigma_error(got: Tensor, model: Tensor) -> Tensor:
    """|sigma - model| in units of the pre-activation x of sigma = softplus(x): d sigma / dx = 1 - exp(-sigma).  Absolute for a dense
    point, relative for a nearly empty one (where the transmittance of the 1e10 last interval still sees it)."""
    return (got.double() - model).abs() / (-torch.expm1(-model)).clamp(min=1e-30)


def _head_act(raw_sigma, raw_rgb):
    sigma = F.softplus(raw_sigma - 1.0)
    rgb = None if raw_rgb is None else torch.sigmoid(raw_rgb) * 1.002 - 0.001
    return sigma, rgb


# ---------------------------------------------------------------------------------------------------------------------------------
# vanilla NeRF (csrc/vanilla.cu, NEO_PREC_TC)
# ---------------------------------------------------------------------------------------------------------------------------------

def vanilla_tc_field(P: Dict[str, Tensor], pre: str, rays: Dict[str, Tensor], t: Tensor, fp16: bool = True,
                     mutation: Optional[str] = None):
    """rays_o / viewdirs (n, 3), t (n, N) -> rgb (n, N, 3), sigma (n, N, 1), float64 on the device of `t`."""
    _check(mutation, VANILLA_MUTATIONS)
    h = _round(fp16)
    f32 = (lambda x: x.float().double()) if fp16 else (lambda x: x)
    dev = t.device
    g = lambda x: x.detach().to(device=dev, dtype=torch.float64)
    Wt = lambda name: g(P[pre + name + ".weight"])
    Bs = lambda name: g(P[pre + name + ".bias"])
    o, vd, tt = g(rays["rays_o"]), g(rays["viewdirs"]), g(t)
    n, N = tt.shape
    x = f32(o[:, None, :] + f32(tt[..., None] * vd[:, None, :])).reshape(-1, 3)           # enc16_kernel: add_(o, mul_(t, d))
    enc = orc.pos_enc(x, 0, 10)
    if mutation == "oct9_cos_early":                                                     # cos(2^9 x) replaced by cos(2^8 x)
        enc = enc.clone()
        enc[:, 60:63] = enc[:, 57:60]
    enc = h(enc)
    denc = orc.pos_enc(vd, 0, 4)
    if mutation == "dir_swap34":
        denc = denc[:, [0, 1, 2, 4, 3] + list(range(5, 27))]
    denc = h(denc)[:, None, :].expand(n, N, 27).reshape(-1, 27)
    layer = lambda name, a, relu=True: h(torch.relu(a @ h(Wt(name)).T + Bs(name)) if relu else a @ h(Wt(name)).T + Bs(name))
    a = enc
    for i in range(8):
        name = f"pts_linears.{i}"
        if i == 5:
            e5 = torch.cat([torch.zeros_like(enc[:, :1]), enc[:, :62]], -1) if mutation == "l5_enc_shift" else enc
            a = h(torch.relu(torch.cat([a, e5], -1) @ h(Wt(name)).T + Bs(name)))
        elif i == 6 and mutation == "l6_no_bias":
            a = h(torch.relu(a @ h(Wt(name)).T))
        else:
            a = layer(name, a)
    wsig = Wt("density_layer")
    if mutation == "sigma_short":                                                        # density head without its last 8 columns
        wsig = wsig.clone()
        wsig[:, 248:] = 0
    raw_sigma = a @ wsig.T + Bs("density_layer")
    beta = layer("bottleneck_layer", a, relu=False)
    v = layer("views_linear.0", torch.cat([beta, denc], -1))
    raw_rgb = v @ Wt("rgb_layer").T + Bs("rgb_layer")
    sigma, rgb = _head_act(raw_sigma, raw_rgb)
    return rgb.reshape(n, N, 3), sigma.reshape(n, N, 1)


# ---------------------------------------------------------------------------------------------------------------------------------
# Mip-NeRF 360 (csrc/mip.cu, NEO_PREC_TC)
# ---------------------------------------------------------------------------------------------------------------------------------

def mip_features(rays_o, rays_d, radii, tdist, basis, mutation: Optional[str] = None):
    """cast_cone -> contract -> ipe_features (mip_oracle), float64: (n, N, 504).  `ipe_var_2k`: variance scaled by 2^k, not 4^k."""
    mean, cov = mo.cast_cone(tdist, rays_o, rays_d, radii)
    z, zc = mo.contract(mean, cov)
    if mutation != "ipe_var_2k":
        return mo.ipe_features(z, zc, basis)
    m = z @ basis
    v = torch.sum(basis[None, None] * (zc @ basis), dim=-2)
    sc = 2.0 ** torch.arange(0, 12, dtype=z.dtype, device=z.device)
    sm = (m[..., None, :] * sc[:, None]).reshape(*m.shape[:-1], -1)
    sv = (v[..., None, :] * sc[:, None]).reshape(*v.shape[:-1], -1)
    return torch.exp(-0.5 * torch.cat([sv, sv], -1)) * torch.sin(torch.cat([sm, sm + 0.5 * torch.pi], -1))


def mip_tc_field(P: Dict[str, Tensor], pre: str, depth: int, disable_rgb: bool, rays: Dict[str, Tensor], radii: Tensor, tdist: Tensor,
                 fp16: bool = True, mutation: Optional[str] = None):
    """One Mip-NeRF 360 MLP (`pre` = "mlps.{l}.") at intervals tdist (n, N+1) -> density (n, N), rgb (n, N, 3) (zeros when
    disable_rgb), float64 on the device of `tdist`."""
    _check(mutation, MIP_MUTATIONS)
    h = _round(fp16)
    dev = tdist.device
    g = lambda x: x.detach().to(device=dev, dtype=torch.float64)
    Wt = lambda name: g(P[pre + name + ".weight"])
    Bs = lambda name: g(P[pre + name + ".bias"])
    o, d, vd, rad, td = g(rays["rays_o"]), g(rays["rays_d"]), g(rays["viewdirs"]), g(radii).reshape(-1, 1), g(tdist)
    n, N = td.shape[0], td.shape[1] - 1
    feats = h(mip_features(o, d, rad, td, g(P[pre + "pos_basis_t"]), mutation)).reshape(-1, 504)
    a = feats
    for i in range(depth):
        name = f"pts_linear.{i}"
        if i == 5:
            f5 = torch.cat([torch.zeros_like(feats[:, :1]), feats[:, :503]], -1) if mutation == "skip_offset" else feats
            a = torch.cat([a, f5], -1)
        a = h(torch.relu(a @ h(Wt(name)).T + Bs(name)))
    raw_sigma = (a @ Wt("density_layer").T + Bs("density_layer"))[:, 0]
    if disable_rgb:
        density, _ = _head_act(raw_sigma, None)
        return density.reshape(n, N), torch.zeros(n, N, 3, dtype=torch.float64, device=dev)
    beta = h(a @ h(Wt("bottleneck_layer")).T + Bs("bottleneck_layer"))
    de = mo.dir_enc(vd)
    if mutation == "dir_cos_zero":
        de = torch.cat([de[:, :15], torch.zeros_like(de[:, 15:])], -1)
    de = h(de)[:, None, :].expand(n, N, 27).reshape(-1, 27)
    v = h(torch.relu(torch.cat([beta, de], -1) @ h(Wt("views_linear.0")).T + Bs("views_linear.0")))
    wrgb = Wt("rgb_layer")
    if mutation == "rgb_short":                                                          # rgb head without its last 8-wide k group
        wrgb = wrgb.clone()
        wrgb[:, 120:] = 0
    density, rgb = _head_act(raw_sigma, v @ wrgb.T + Bs("rgb_layer"))
    return density.reshape(n, N), rgb.reshape(n, N, 3)


# ---------------------------------------------------------------------------------------------------------------------------------
# GridEncoder dense part (csrc/encoder.cu)
# ---------------------------------------------------------------------------------------------------------------------------------

def pillar_cells(pillars: Tensor, G: int) -> Tensor:
    """pillars (K, 4) = (view, axis, p, q) -> (K, G, 3) integer grid indices (ix, iy, iz): `axis` runs over 0..G-1, the two other axes
    (in x, y, z order) are (p, q) -- the (p, q) pixel of the floor plan that sums over `axis` (yz: axis 0, xz: 1, xy: 2)."""
    K = pillars.shape[0]
    i = torch.arange(G)[None, :].expand(K, G)
    idx = torch.zeros(K, G, 3, dtype=torch.long)
    for k, (_, axis, p, q) in enumerate(pillars.tolist()):
        others = [a for a in range(3) if a != axis]
        idx[k, :, axis] = i[k]
        idx[k, :, others[0]] = p
        idx[k, :, others[1]] = q
    return idx


def encoder_geometry(pillars: Tensor, G: int, poses: Tensor, focal: float, c: Tensor, W: int, H: int, lat_hw, mutation=None):
    """World xyz, camera xyz, masked unit direction and latent grid coordinates of every cell of every pillar, float64, with the
    constants of `GridEncoder.dense_torch`: the grid linspace in the default dtype (float32, as the kernel's), the latent scaling
    in float32."""
    dev = poses.device
    ax = [torch.linspace(-1, 1, G), torch.linspace(-1, 1, G), torch.linspace(0, 1, G)]
    idx = pillar_cells(pillars, G)
    world = torch.stack([ax[a][idx[..., a]] for a in range(3)], -1).to(device=dev, dtype=torch.float64)   # (K, G, 3)
    pose = poses.to(torch.float64)[pillars[:, 0].to(dev)]                                   # (K, 4, 4)
    rot = pose[:, :3, :3].transpose(1, 2)
    trans = -torch.bmm(rot, pose[:, :3, 3:])
    cam = torch.einsum("kij,kgj->kgi", rot, world) + trans[:, None, :, 0]
    mask = cam[..., 2] < 1e-3
    if mutation == "no_dir_mask":
        mask = torch.ones_like(mask)
    dvec = world - pose[:, None, :3, 3]
    dvec = dvec / torch.norm(dvec + 1e-9, dim=-1, keepdim=True) * mask[..., None]
    f2 = torch.tensor([focal, -focal], dtype=torch.float64, device=dev)
    uv = -cam[..., :2] / (cam[..., 2:] + 1e-9) * f2 + c.to(device=dev, dtype=torch.float64).reshape(1, 1, 2)
    lh, lw = lat_hw
    ls = torch.tensor([lw, lh], dtype=torch.float32)
    scale = (2.0 / torch.tensor([W, H], dtype=torch.float32)) if mutation == "no_size_ratio" else \
        ((ls / (ls - 1) * 2.0) / torch.tensor([W, H], dtype=torch.float32))
    uv = uv * scale.to(device=dev, dtype=torch.float64) - 1.0
    return world, cam, dvec, uv


def encoder_tc_dense(module, latent: Tensor, poses: Tensor, focal, c, W: int, H: int, pillars: Tensor, fp16: bool = True,
                     mutation: Optional[str] = None) -> Tensor:
    """`neo_grid_encoder_dense` at the given pillars (K, 4) = (view, axis, p, q): -> (K, 512) float64 = plane[axis][view, :, p, q] of
    the (xz, xy, yz) = (axis 1, 2, 0) floor planes.  Runs on the device of `latent`; G = module.GRID cells per pillar."""
    _check(mutation, ENCODER_MUTATIONS)
    h = _round(fp16)
    dev = latent.device
    g = lambda x: x.detach().to(device=dev, dtype=torch.float64)
    G = module.GRID
    pillars = pillars.long().cpu()
    K = pillars.shape[0]
    focal = float(focal[0]) if torch.is_tensor(focal) else float(focal)
    c0 = (c[0] if torch.is_tensor(c) and c.dim() == 2 else torch.as_tensor(c)).double()
    lat = g(latent)
    world, cam, dvec, uv = encoder_geometry(pillars, G, g(poses), focal, c0, W, H, lat.shape[-2:], mutation)
    gx, gy = uv[..., 0], uv[..., 1]
    if mutation == "border_clamp":                  # clamp the sample position into the image instead of zero padding outside it
        gx, gy = gx.clamp(-1, 1), gy.clamp(-1, 1)
    feat = torch.zeros(K, G, lat.shape[1], dtype=torch.float64, device=dev)
    views = pillars[:, 0].to(dev)
    for v in pillars[:, 0].unique().tolist():
        sel = views == v
        feat[sel] = blend(lat[v:v + 1], gx[sel].reshape(1, -1), gy[sel].reshape(1, -1))[0].reshape(-1, G, lat.shape[1])
    tail = [dvec, cam] if mutation == "cam_dir_swap" else [cam, dvec]
    row = h(torch.cat([feat] + tail, -1))                                               # (K, G, 518)
    fc = [module.depth_fc.common_branch[0], module.depth_fc.common_branch[2], module.depth_fc.depth_encoder]
    lin = lambda m, a: a @ h(g(m.weight)).T + g(m.bias)
    ha = h(torch.relu(lin(fc[0], row)))
    hb = h(torch.relu(lin(fc[1], ha)))
    L = h(lin(fc[2], hb))                                                               # (K, G, 512)
    out = torch.empty(K, L.shape[-1], dtype=torch.float64, device=dev)
    names = {0: "yz", 1: "xz", 2: "xy"}
    axes = pillars[:, 1].to(dev)
    for axis in range(3):
        sel = axes == axis
        if not bool(sel.any()):
            continue
        agg = getattr(module, f"pillar_aggregator_{names[axis]}")
        coord = world[sel][..., ((axis + 1) % 3) if mutation == "coord_axis" else axis][..., None]
        a = h(torch.relu(lin(agg[0], torch.cat([L[sel], h(coord)], -1))))
        logits = (a @ g(agg[2].weight).T + g(agg[2].bias))[..., 0]                     # (k, G)
        out[sel] = (torch.softmax(logits, -1)[..., None] * L[sel]).sum(1)
    return out
