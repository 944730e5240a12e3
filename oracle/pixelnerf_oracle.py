"""TEST INFRASTRUCTURE ONLY -- CPU restatement (oracle) of the PixelNeRF renderer of the reference
(models/vanilla_nerf/model_pixel.py:35-258, models/vanilla_nerf/util.py:13-63, models/vanilla_nerf/encoder.py:101-130,
models/vanilla_nerf/helper.py:415-616), SURVEY.md section 2 row 11.

Pinned to the unmodified reference by oracle/make_golden_pixelnerf.py (tests/golden/pixelnerf_reference_vectors.npz).
Differentiable: with float64 inputs it is the gradient reference of the GPU training tests."""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn.functional as F

from .neo360_oracle import pos_enc, world2camera, world2camera_dirs
from .vanilla_oracle import sample_along_rays, sample_pdf, composite

Tensor = torch.Tensor


def project(p_cam: Tensor, focal: float, cx: float, cy: float) -> Tensor:
    """util.py:36-51 with focal = src_focal[0] on both axes and c = src_c[0] for every view (model_pixel.py:210-212).  Unlike
    NeO-360's get_local_feats (models/neo360/model.py:243) the y focal is NOT negated."""
    uv = -p_cam[..., :2] / (p_cam[..., 2:] + 1e-9)
    return uv * focal + torch.tensor([cx, cy], dtype=p_cam.dtype, device=p_cam.device)


def index(latent: Tensor, uv: Tensor, img_w: int, img_h: int) -> Tensor:
    """SpatialEncoder.index (encoder.py:101-130): bilinear, zeros padding, align_corners=True.  latent (NV,C,Hl,Wl), uv (NV,M,2)
    -> (NV*M, C), rows ordered (view, point) (model_pixel.py:214-219)."""
    nv, C, Hl, Wl = latent.shape
    ls = torch.tensor([float(Wl), float(Hl)], dtype=torch.float32)
    ls = (ls / (ls - 1) * 2.0).to(uv)                                         # encoder.py:182-184 (fp32 buffer)
    g = uv * (ls / torch.tensor([float(img_w), float(img_h)], dtype=uv.dtype, device=uv.device)) - 1.0
    out = F.grid_sample(latent, g[:, :, None, :], align_corners=True, mode="bilinear", padding_mode="zeros")[..., 0]
    return out.transpose(1, 2).reshape(-1, C)


def mlp_forward(P: Dict[str, Tensor], pre: str, enc: Tensor, dir_tile: Tensor, latent: Tensor, nv: int):
    """NeRFMLP.forward (model_pixel.py:95-131): enc (NV,M,63), dir_tile (NV*M,27), latent (NV*M,512) -> raw rgb (M,3), raw sigma (M,1).
    Trunk 575 -> 128 -> 128 -> 128 -> 128 with ReLU, no skip; after layer 3 the bottleneck is taken per view and the trunk is averaged
    over views (combine_interleaved, util.py:53-63); views_linear.0 is averaged over views before its ReLU."""
    M = enc.shape[1]
    lin = lambda name, x: F.linear(x, P[pre + name + ".weight"], P[pre + name + ".bias"])
    h = torch.cat([enc.reshape(-1, enc.shape[-1]), latent], -1)
    for i in range(4):
        h = torch.relu(lin(f"pts_linears.{i}", h))
    beta = lin("bottleneck_layer", h)
    raw_sigma = lin("density_layer", h.reshape(nv, M, -1).mean(0))
    q = torch.relu(lin("views_linear.0", torch.cat([beta, dir_tile], -1)).reshape(nv, M, -1).mean(0))
    q = torch.relu(lin("views_linear.1", q))
    return lin("rgb_layer", q), raw_sigma


def stages(pts: Tensor, viewdirs: Tensor, sc: Dict, N: int):
    """Per-view inputs of one level (model_pixel.py:207-232): pts (B,N,3) -> enc (NV,B*N,63), dir_tile (NV*B*N,27), latent rows
    (NV*B*N,512).  Quirk Q1: the direction encoding is tiled along the ray axis, so row j = b*N+s of a view sees ray (j mod B)."""
    p_cam = world2camera(pts.reshape(-1, 3), sc["src_poses"])
    uv = project(p_cam, sc["focal"], sc["cx"], sc["cy"])
    latent = index(sc["latent"], uv, sc["img_w"], sc["img_h"])
    enc = pos_enc(p_cam, 0, 10)
    denc = pos_enc(world2camera_dirs(viewdirs, sc["src_poses"]), 0, 4)        # (NV,B,27)
    dir_tile = torch.tile(denc[:, None, :], (1, N, 1, 1)).reshape(-1, denc.shape[-1])
    return dict(p_cam=p_cam, uv=uv, latent=latent, enc=enc, dir_tile=dir_tile)


def render(rays: Dict[str, Tensor], sc: Dict, P: Dict[str, Tensor], n_coarse: int, n_fine: int, near: float, far: float,
           white_bkgd: bool = False, rand: Optional[Dict[str, Tensor]] = None, return_aux: bool = False):
    """PixelNeRF.forward (model_pixel.py:174-258) with the encoder output `sc["latent"]` given.  Marches along rays_d with the caller's
    near / far; rgb = sigmoid(raw), sigma = relu(raw) (model_pixel.py:164-165, 245-246)."""
    o, d, vd = rays["rays_o"], rays["rays_d"], rays["viewdirs"]
    nv = sc["src_poses"].shape[0]
    ret, aux = [], []
    t = w = None
    for lvl in range(2):
        if lvl == 0:
            t, pts = sample_along_rays(o, d, n_coarse, near, far, None if rand is None else rand.get("u0"))
        else:
            t, pts = sample_pdf(o, d, t, w.detach(), n_fine, None if rand is None else rand.get("u1"))
        B, N = t.shape
        st = stages(pts, vd, sc, N)
        pre = "coarse_mlp." if lvl == 0 else "fine_mlp."
        raw_rgb, raw_sigma = mlp_forward(P, pre, st["enc"], st["dir_tile"], st["latent"], nv)
        rgb = torch.sigmoid(raw_rgb.reshape(B, N, 3))
        sigma = torch.relu(raw_sigma.reshape(B, N, 1))
        comp, acc, w, depth = composite(rgb, sigma, t, d, white_bkgd)
        ret.append((comp, acc, depth))
        aux.append(dict(t=t, rgb=rgb, sigma=sigma, w=w, **st))
    return (ret, aux) if return_aux else ret


def scene(latent: Tensor, src_poses: Tensor, src_focal: Tensor, src_c: Tensor, img_wh) -> Dict:
    """The per-call scene of the oracle from the batch's src_* entries (model_pixel.py:176-178, 210-211)."""
    return dict(latent=latent, src_poses=src_poses, focal=float(src_focal[0]), cx=float(src_c[0, 0]), cy=float(src_c[0, 1]),
                img_w=int(img_wh[0]), img_h=int(img_wh[1]))
