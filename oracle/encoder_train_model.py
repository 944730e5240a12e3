"""TEST INFRASTRUCTURE ONLY -- float64 model of the four stages of the GridEncoder training path (csrc/encoder.cu).

* features_fwd / features_bwd: `neo_grid_encoder_features` and its adjoint `neo_grid_encoder_features_bwd`.  Rows v * G^3 + cell
  (cells (ix, iy, iz) row-major, as `cell_xyz`) = [bilinear latent lookup | cam xyz | masked unit direction]; the geometry is
  `tc_paths_model.encoder_geometry` over the pillars along z (which enumerate the cells in row order), the taps, the gather and the
  `index_add_` adjoint are `train_stage_model`'s.  With `fp32=True` the taps are taken at the kernel's own fp32 coordinates as
  `train_stage_model.lookup_taps` models them (fp32 grid linspace, fp32 focal / principal point / latent scaling), each row with a
  first-order bound on its fp32 tap-coordinate error; the forward returns sum |w F| per element and that error term, the adjoint sum
  |w g|, the contribution count per texel and the error term.  With `fp32=False` everything is float64 of the inputs (the grid linspace
  in the default dtype, as `dense_torch` builds it) and the model equals autograd through `GridEncoder.dense_torch`
  (tests/test_encoder_train_model.py).
* pool_fwd / pool_bwd: `neo_grid_encoder_pool` and `neo_grid_encoder_pool_bwd`: softmax of each pillar's logits and the weighted sum of
  its rows; backward d_lat = sum_a s_a g_a, d_logits = s (g.lat - sum s (g.lat)).  Each result comes with its magnitude (the same sum with
  every term in absolute value), the unit the GPU bounds are stated in.
G is read from the module (`module.GRID`), so the CPU tests can run an 8^3 grid.  Nothing under `neo360_b200/` imports this file.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import tc_paths_model as tpm
from . import train_stage_model as tsm

Tensor = torch.Tensor
AXES = ("yz", "xz", "xy")       # axis 0 / 1 / 2: the floor plan that sums over x / y / z


def _cells(G: int, nv: int) -> Tensor:
    """The pillars along z of every view: their cells are the grid rows v * G^3 + (ix * G + iy) * G + iz in order."""
    return torch.tensor([(v, 2, p, q) for v in range(nv) for p in range(G) for q in range(G)])


def features_taps(G: int, latent_hw, poses: Tensor, focal: float, c, W: int, H: int, fp32: bool = True):
    """Tap set of every row (train_stage_model._taps layout) and the cam / direction columns (R, 3) of the lookup rows, float64."""
    nv = poses.shape[0]
    lh, lw = latent_hw
    pil = _cells(G, nv)
    c = torch.as_tensor(c, dtype=torch.float64).reshape(-1)
    world, cam, dvec, uv = tpm.encoder_geometry(pil, G, poses.double(), float(focal), c, W, H, (lh, lw))
    if fp32:
        grid = torch.stack(torch.meshgrid(*[torch.linspace(-1, 1, G), torch.linspace(-1, 1, G), torch.linspace(0, 1, G)], indexing="ij"), -1)
        pts = grid.reshape(-1, 3).to(device=poses.device, dtype=torch.float64)
        tp = tsm.lookup_taps(pts, poses.float(), None, (lh, lw), float(focal), float(c[0]), float(c[1]), (W, H), local=True)[0]
    else:
        uv = uv.reshape(-1, 2)
        z = torch.zeros_like(uv[:, 0])
        tp = tsm._taps(uv[:, 0], uv[:, 1], z, z, lw, lh)
    return tp, cam.reshape(-1, 3), dvec.reshape(-1, 3)


def features_fwd(latent: Tensor, tp, cam: Tensor, dvec: Tensor) -> Dict[str, Tensor]:
    """latent (NV,512,Hl,Wl) -> X (R, 518) float64 and, for the 512 lookup columns, mag = sum |w F| and derr (coordinate-error term)."""
    nv = latent.shape[0]
    lk = tsm.lookup_fwd([tp], [latent.double().permute(0, 2, 3, 1).contiguous()], nv)
    return dict(X=torch.cat([lk["val"], cam, dvec], -1), mag=lk["mag"], derr=lk["derr"])


def features_bwd(tp, g_X: Tensor, nv: int) -> Dict[str, Tensor]:
    """g_X (R, >= 512): columns 0..511 scattered into the channel-last latent gradient (NV,Hl,Wl,512): val, mag = sum |w g|, n (count
    of non-zero contributions per texel), derr and reach (texels some row's taps may touch)."""
    return tsm.lookup_bwd(tp, g_X[:, :512].double(), nv)


def _softmax(logits: Tensor, nv: int, G: int):
    """s of every axis: (3, NV, G, G, G) float64, each softmaxed along its axis (dims 2 / 3 / 4 = x / y / z)."""
    lg = logits.double().reshape(3, nv, G, G, G)
    return torch.stack([torch.softmax(lg[a], dim=1 + a) for a in range(3)])


def pool_fwd(lat: Tensor, logits: Tensor, nv: int, G: int) -> Dict[str, Tensor]:
    """lat (R, 512), logits (3, R) -> planes {"xz", "xy", "yz"} (NV,512,G,G) float64 and their magnitudes sum s |lat|."""
    s = _softmax(logits, nv, G)
    L = lat.double().reshape(nv, G, G, G, -1)
    out = {}
    for a, name in enumerate(AXES):
        out[name] = (s[a][..., None] * L).sum(1 + a).permute(0, 3, 1, 2)
        out[name + "_mag"] = (s[a][..., None] * L.abs()).sum(1 + a).permute(0, 3, 1, 2)
    return out


def pool_bwd(lat: Tensor, logits: Tensor, nv: int, G: int, g_xz: Optional[Tensor] = None, g_xy: Optional[Tensor] = None,
             g_yz: Optional[Tensor] = None) -> Dict[str, Tensor]:
    """d_lat (R, 512), d_logits (3, R) float64 and their magnitudes; None upstream planes are zero."""
    s = _softmax(logits, nv, G)
    L = lat.double().reshape(nv, G, G, G, -1)
    gs = dict(yz=g_yz, xz=g_xz, xy=g_xy)
    d_lat, d_lat_m = torch.zeros_like(L), torch.zeros_like(L)
    d_lg, d_lg_m = [], []
    for a, name in enumerate(AXES):
        g = gs[name]
        if g is None:
            d_lg.append(torch.zeros_like(s[a]))
            d_lg_m.append(torch.zeros_like(s[a]))
            continue
        gb = g.double().permute(0, 2, 3, 1).unsqueeze(1 + a)                          # (NV, ..., 512) broadcast along the pillar axis
        d_lat = d_lat + s[a][..., None] * gb
        d_lat_m = d_lat_m + s[a][..., None] * gb.abs()
        gl = (gb * L).sum(-1)
        glm = (gb.abs() * L.abs()).sum(-1)
        d_lg.append(s[a] * (gl - (s[a] * gl).sum(1 + a, keepdim=True)))
        d_lg_m.append(s[a] * (glm + (s[a] * glm).sum(1 + a, keepdim=True)))
    R = nv * G ** 3
    return dict(d_lat=d_lat.reshape(R, -1), d_lat_mag=d_lat_m.reshape(R, -1), d_logits=torch.stack(d_lg).reshape(3, R),
                d_logits_mag=torch.stack(d_lg_m).reshape(3, R))


def dense_layers(module, X: Tensor):
    """depth_fc and the three aggregators' logits as `dense_train` applies them (framework ops, the module's dtype): lat (R, 512),
    logits (3, R)."""
    G = module.GRID
    nv = X.shape[0] // G ** 3
    lat = module.depth_fc(X)
    ax = [torch.linspace(-1, 1, G, dtype=X.dtype), torch.linspace(-1, 1, G, dtype=X.dtype), torch.linspace(0, 1, G, dtype=X.dtype)]
    grid = torch.stack(torch.meshgrid(*ax, indexing="ij"), -1).reshape(1, -1, 3).expand(nv, -1, -1).reshape(-1, 3).to(X.device)
    logits = [getattr(module, f"pillar_aggregator_{n}")(torch.cat([lat, grid[:, a:a + 1]], -1))[:, 0] for a, n in enumerate(AXES)]
    return lat, torch.stack(logits)
