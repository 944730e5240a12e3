"""TEST INFRASTRUCTURE ONLY -- float64 models of Mip-NeRF 360's MLPs at an arbitrary Gaussian, for neo_mip_field_eval.

neo_mip_field_eval reads each point as a Gaussian with its mean at the point and covariance diag(var); the render reads the Gaussian of
a conical frustum.  Both go through the same contraction, lift and IPE, then the same MLP.  This module takes the Gaussian as an input:

* point_gaussian(pts, var): the Gaussian neo_mip_field_eval gives a point.
* gaussian_features(mean, cov, basis): contract + lift_and_diagonalize + integrated_pos_enc (mip_oracle), float64.
* point_features(pts, var, basis): gaussian_features of point_gaussian.
* mip_tc_gaussian_field: the NEO_PREC_TC path at given Gaussians, every fp16 rounding of tc_paths_model.mip_tc_field made explicit in
  the same places.  At the render's frustums (mip_oracle.cast_cone) it equals tc_paths_model.mip_tc_field bit for bit
  (tests/test_mesh_models.py), so the frustum model is unchanged and this one only swaps the Gaussian's source.

Nothing under `neo360_b200/` imports this file.
"""
from __future__ import annotations

from typing import Dict

import torch
from torch import Tensor

from . import mip_oracle as mo
from . import tc_paths_model as tpm


def point_gaussian(pts: Tensor, var):
    """mean pts (..., 3), covariance diag(var) (..., 3, 3), var a per-axis 3-sequence."""
    v = torch.as_tensor(var, dtype=pts.dtype, device=pts.device)
    return pts, torch.diag_embed(v.expand(pts.shape))


def gaussian_features(mean: Tensor, cov: Tensor, basis: Tensor) -> Tensor:
    """(n, N, 3), (n, N, 3, 3) -> IPE features (n, N, 504)."""
    return mo.ipe_features(*mo.contract(mean, cov), basis)


def point_features(pts: Tensor, var, basis: Tensor) -> Tensor:
    return gaussian_features(*point_gaussian(pts, var), basis)


def mip_tc_gaussian_field(P: Dict[str, Tensor], pre: str, depth: int, disable_rgb: bool, viewdirs: Tensor, mean: Tensor, cov: Tensor,
                          fp16: bool = True):
    """One Mip-NeRF 360 MLP (`pre` = "mlps.{l}.") at Gaussians mean (n, N, 3), cov (n, N, 3, 3), viewdirs (n, 3) its direction input
    -> density (n, N), rgb (n, N, 3) (zeros when disable_rgb), float64 on the device of `mean`."""
    h = tpm._round(fp16)
    dev = mean.device
    g = lambda x: x.detach().to(device=dev, dtype=torch.float64)
    Wt = lambda name: g(P[pre + name + ".weight"])
    Bs = lambda name: g(P[pre + name + ".bias"])
    n, N = mean.shape[0], mean.shape[1]
    feats = h(gaussian_features(g(mean), g(cov), g(P[pre + "pos_basis_t"]))).reshape(-1, 504)
    a = feats
    for i in range(depth):
        if i == 5:
            a = torch.cat([a, feats], -1)
        a = h(torch.relu(a @ h(Wt(f"pts_linear.{i}")).T + Bs(f"pts_linear.{i}")))
    raw_sigma = (a @ Wt("density_layer").T + Bs("density_layer"))[:, 0]
    if disable_rgb:
        density, _ = tpm._head_act(raw_sigma, None)
        return density.reshape(n, N), torch.zeros(n, N, 3, dtype=torch.float64, device=dev)
    beta = h(a @ h(Wt("bottleneck_layer")).T + Bs("bottleneck_layer"))
    de = h(mo.dir_enc(g(viewdirs)))[:, None, :].expand(n, N, 27).reshape(-1, 27)
    v = h(torch.relu(torch.cat([beta, de], -1) @ h(Wt("views_linear.0")).T + Bs("views_linear.0")))
    density, rgb = tpm._head_act(raw_sigma, v @ Wt("rgb_layer").T + Bs("rgb_layer"))
    return density.reshape(n, N), rgb.reshape(n, N, 3)
