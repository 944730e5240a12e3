"""Seeded synthetic NERDS360-shaped inputs (SURVEY.md section 8(d)).

There is no dataset / checkpoint access, so benches and tests run on synthetic scenes of the right
SHAPE: a turntable of target cameras inside the unit sphere (OpenGL convention, -z forward, as
produced by datasets/ray_utils.py:329-332 in the reference), NV source cameras at equally spaced
azimuths, band-limited random tri-planes (NV,128,120,160) x3 and pixel-aligned latent (NV,512,H/2,W/2)
standing in for the (out-of-scope) encoder's outputs, and xavier-initialised MLP parameters under the
reference's state-dict names (models/neo360/model.py:215-237; SURVEY.md section 8(b)).
"""
from __future__ import annotations

import math
from typing import Dict, Tuple

import torch

Tensor = torch.Tensor

MLP_PREFIXES = ("fg_coarse_mlp.", "bg_coarse_mlp.", "fg_fine_mlp.", "bg_fine_mlp.")
LOCAL_CH = 512
WORLD_CH = 128


def look_at_pose(azim_deg: float, height: float, radius: float) -> Tensor:
    """Camera-to-world (4,4), camera at (r cos a, r sin a, h) looking at the origin, -z forward, +y up-ish."""
    a = math.radians(azim_deg)
    p = torch.tensor([radius * math.cos(a), radius * math.sin(a), height], dtype=torch.float64)
    fwd = -p / p.norm()
    z = -fwd
    up = torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64)
    x = torch.linalg.cross(up, z)
    x = x / x.norm()
    y = torch.linalg.cross(z, x)
    m = torch.eye(4, dtype=torch.float64)
    m[:3, 0], m[:3, 1], m[:3, 2], m[:3, 3] = x, y, z, p
    return m.float()


def _smooth_field(shape, gen, k=5) -> Tensor:
    x = torch.randn(shape, generator=gen) * 0.5
    n, c, h, w = shape
    x = torch.nn.functional.avg_pool2d(x.reshape(1, n * c, h, w), k, stride=1, padding=k // 2,
                                       count_include_pad=True).reshape(shape)
    return (x / x.std() * 0.5).contiguous()


def make_scene(img_wh: Tuple[int, int] = (640, 480), nv: int = 3, plane_hw: Tuple[int, int] = (120, 160),
               seed: int = 0) -> Dict[str, Tensor]:
    """Returns the `src_*` part of the reference batch dict (nerds360_ae.py:1007-1023) plus the
    encoder outputs (`planes_xz|xy|yz`, `latent`) that the hot path consumes."""
    W, H = img_wh
    g = torch.Generator().manual_seed(seed)
    poses = torch.stack([look_at_pose(360.0 * v / nv + 10.0, 0.3, 0.8) for v in range(nv)])
    hp, wp = plane_hw
    return {
        "src_poses": poses,
        "src_focal": torch.full((nv,), 0.8 * W),
        "src_c": torch.tensor([[W / 2.0, H / 2.0]] * nv),
        "img_wh": (W, H),
        "planes_xz": _smooth_field((nv, WORLD_CH, hp, wp), g),
        "planes_xy": _smooth_field((nv, WORLD_CH, hp, wp), g),
        "planes_yz": _smooth_field((nv, WORLD_CH, hp, wp), g),
        "latent": _smooth_field((nv, LOCAL_CH, H // 2, W // 2), g),
    }


def _linear(out_f, in_f, gen, xavier=True):
    if xavier:
        bound = math.sqrt(6.0 / (in_f + out_f))
    else:
        bound = 1.0 / math.sqrt(in_f)
    w = (torch.rand((out_f, in_f), generator=gen) * 2 - 1) * bound
    b = (torch.rand((out_f,), generator=gen) * 2 - 1) / math.sqrt(in_f)
    return w, b


# Gains on top of xavier init so that the random-weight field has trained-network-like dynamic range
# (rgb spanning most of [0,1], accumulated opacity spanning (0,1)) instead of sitting at sigmoid(0).
GAINS = {"pts_linears.0": 1.5, "pts_linears.1": 1.5, "pts_linears.2": 1.5, "pts_linears.3": 1.5,
         "views_linear.0": 2.0, "views_linear.1": 2.0, "bottleneck_layer": 1.5, "density_layer": 3.0,
         "rgb_layer": 4.0}


def make_mlp_params(seed: int = 0, density_bias_shift: float = 1.0) -> Dict[str, Tensor]:
    """Four NeRFPPMLP parameter sets (fg/bg x coarse/fine) with the reference's shapes:
    (128,703|724) (128,128)x2 (128,831|852) | bottleneck (128,128) | density (1,128) | views (64,155),(64,64) | rgb (3,64)."""
    g = torch.Generator().manual_seed(1000 + seed)
    P: Dict[str, Tensor] = {}
    for pre in MLP_PREFIXES:
        pos = (63 if pre.startswith("fg") else 84) + LOCAL_CH + WORLD_CH
        shapes = {
            "pts_linears.0": (128, pos), "pts_linears.1": (128, 128), "pts_linears.2": (128, 128),
            "pts_linears.3": (128, 128 + pos), "views_linear.0": (64, 128 + 27), "views_linear.1": (64, 64),
            "bottleneck_layer": (128, 128), "density_layer": (1, 128), "rgb_layer": (3, 64),
        }
        for name, (o, i) in shapes.items():
            w, b = _linear(o, i, g, xavier=(name != "views_linear.0"))
            w = w * GAINS[name]
            if name == "density_layer":
                b = b + density_bias_shift
            P[pre + name + ".weight"] = w
            P[pre + name + ".bias"] = b
    return P


def target_pose(view: int = 0, n_views: int = 100) -> Tensor:
    """Turntable target camera `view` of `n_views` (radius 0.6-0.9, height 0.2-0.4, inside the unit sphere)."""
    f = view / max(n_views, 1)
    return look_at_pose(360.0 * f + 47.0, 0.3 + 0.1 * math.sin(2 * math.pi * f), 0.75 + 0.15 * math.cos(2 * math.pi * f))


VANILLA_PREFIXES = ("coarse_mlp.", "fine_mlp.")


def make_vanilla_params(seed: int = 0, density_bias_shift: float = 1.0) -> Dict[str, Tensor]:
    """Two NeRFMLP parameter sets with the reference's shapes (models/vanilla_nerf/model.py:44-98): pts_linears.0 (256,63),
    .1-.4/.6/.7 (256,256), .5 (256,319), views_linear.0 (128,283), bottleneck (256,256), density (1,256), rgb (3,128)."""
    g = torch.Generator().manual_seed(2000 + seed)
    P: Dict[str, Tensor] = {}
    for pre in VANILLA_PREFIXES:
        shapes = {f"pts_linears.{i}": (256, 63 if i == 0 else (319 if i == 5 else 256)) for i in range(8)}
        shapes.update({"views_linear.0": (128, 283), "bottleneck_layer": (256, 256), "density_layer": (1, 256), "rgb_layer": (3, 128)})
        for name, (o, i) in shapes.items():
            w, b = _linear(o, i, g, xavier=(name != "views_linear.0"))
            gain = {"density_layer": 3.0, "rgb_layer": 4.0, "views_linear.0": 2.0}.get(name, 1.3)
            w = w * gain
            if name == "density_layer":
                b = b + density_bias_shift
            P[pre + name + ".weight"] = w
            P[pre + name + ".bias"] = b
    return P


def make_pixelnerf_params(seed: int = 0, density_bias_shift: float = 1.0) -> Dict[str, Tensor]:
    """Two PixelNeRF NeRFMLP parameter sets with the reference's shapes (models/vanilla_nerf/model_pixel.py:35-93): pts_linears.0
    (128,575), .1-.3 (128,128), views_linear.0 (128,155), .1 (128,128), bottleneck (128,128), density (1,128), rgb (3,128)."""
    g = torch.Generator().manual_seed(3000 + seed)
    P: Dict[str, Tensor] = {}
    for pre in VANILLA_PREFIXES:
        shapes = {f"pts_linears.{i}": (128, 63 + LOCAL_CH if i == 0 else 128) for i in range(4)}
        shapes.update({"views_linear.0": (128, 155), "views_linear.1": (128, 128), "bottleneck_layer": (128, 128),
                       "density_layer": (1, 128), "rgb_layer": (3, 128)})
        for name, (o, i) in shapes.items():
            w, b = _linear(o, i, g, xavier=(name != "views_linear.0"))
            w = w * {"density_layer": 3.0, "rgb_layer": 4.0, "views_linear.0": 2.0}.get(name, 1.5)
            if name == "density_layer":
                b = b + density_bias_shift
            P[pre + name + ".weight"] = w
            P[pre + name + ".bias"] = b
    return P


def make_mip_params(seed: int = 0, width: int = 1024) -> Dict[str, Tensor]:
    """MipNeRF360 parameter set (models/mipnerf360/model.py:176-234): two PropMLPs (4x256, density only) and one NeRFMLP
    (8 x `width`, default 1024) under the reference's state-dict names, plus the `pos_basis_t` buffers."""
    from .mip_basis import POS_BASIS_T
    g = torch.Generator().manual_seed(3000 + seed)
    P: Dict[str, Tensor] = {}
    for lvl in range(3):
        pre = f"mlps.{lvl}."
        w_, depth = (256, 4) if lvl < 2 else (width, 8)
        P[pre + "pos_basis_t"] = POS_BASIS_T.clone()
        shapes = {f"pts_linear.{i}": (w_, 504 if i == 0 else (w_ + 504 if (i == 5) else w_)) for i in range(depth)}
        shapes["density_layer"] = (1, w_)
        if lvl == 2:
            shapes.update({"bottleneck_layer": (256, w_), "views_linear.0": (128, 283), "rgb_layer": (3, 128)})
        for name, (o, i) in shapes.items():
            bound = math.sqrt(6.0 / i)                      # kaiming_uniform_ (a=0), model.py:76-110
            wgt = (torch.rand((o, i), generator=g) * 2 - 1) * bound
            b = (torch.rand((o,), generator=g) * 2 - 1) / math.sqrt(i)
            gain = {"density_layer": 0.6, "rgb_layer": 1.5}.get(name, 0.8)
            if name == "density_layer":
                b = b + 1.0
            P[pre + name + ".weight"] = wgt * gain
            P[pre + name + ".bias"] = b
    return P
