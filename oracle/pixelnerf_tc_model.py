"""TEST INFRASTRUCTURE ONLY -- float64 model of the PixelNeRF tensor-core field (`neo_pixelnerf_field_tc`, csrc/pixelnerf.cu).

`tc_field` restates, point by point, what the NEO_PREC_TC field of one level computes, with every fp16 rounding made explicit
(`tc_model._round`): points fp32(o + fp32(t rays_d)); per view the row [pos_enc(camera point) 63 | bilinear latent 512 | 0] in fp16;
weights fp16, fp32 biases added in the epilogue, fp16 after each trunk layer's ReLU (4 layers); bottleneck fp16 without ReLU beside
the fp16 direction encoding; the view mean of h3 rounded to fp16 times the fp32 density weights; views_linear.0 fp16, its view mean +
ReLU fp16; views_linear.1 fp16 after ReLU; the rgb head = fp16 rows times the fp32 weights; sigma = relu, rgb = sigmoid.  Geometry,
encodings and the lookup are float64 (the kernels' fp32 arithmetic differs from them by fp32 rounding, below one fp16 ulp).

`fp16=False` turns every rounding into the identity; the model then equals `pixelnerf_oracle.mlp_forward` on the same inputs to 1e-9
(tests/test_pixelnerf_tc_model.py).  The bounds below hold the GPU against it (tests/test_gpu_pixelnerf.py).
Nothing under `neo360_b200/` imports this file."""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from . import pixelnerf_oracle as por
from .tc_model import _round

Tensor = torch.Tensor

# Per point: |rgb - model| <= RGB_TOL and |sigma - model| / (1 + |model|) <= SIGMA_TOL; per case the means of those errors <= *_MEAN_TOL.
# Set at about 3x the largest values measured on an H100 80GB HBM3 at a 700 W power limit (measured in the comment).  The per-point
# maxima are fp16 rounding noise: once one rounding of a point differs from the model's, its later roundings decorrelate.
RGB_TOL, SIGMA_TOL, RGB_MEAN_TOL, SIGMA_MEAN_TOL = 1e-2, 1.5e-2, 4e-4, 3e-4       # measured 3.8e-3, 5.9e-3, 1.45e-4, 9.2e-5


def tc_field(P: Dict[str, Tensor], pre: str, rays: Dict[str, Tensor], t: Tensor, sc: Dict, fp16: bool = True):
    """rays (n, 3 each, fp32), t (n, N) fp32, sc = pixelnerf_oracle.scene(...) -> rgb (n, N, 3), sigma (n, N) float64.  One chunk of n
    rays (quirk Q1)."""
    r = _round(fp16)
    o, d, vd = rays["rays_o"].float(), rays["rays_d"].float(), rays["viewdirs"].float()
    n, N = t.shape
    pts = (o[:, None, :] + t.float()[..., None] * d[:, None, :]).double()
    sc64 = dict(sc, latent=sc["latent"].double(), src_poses=sc["src_poses"].double())
    st = por.stages(pts, vd.double(), sc64, N)
    nv = sc["src_poses"].shape[0]
    W = lambda name: r(P[pre + name + ".weight"].double())
    B = lambda name: P[pre + name + ".bias"].double()
    x = r(torch.cat([st["enc"].reshape(-1, 63), st["latent"]], -1))
    h = x
    for i in range(4):
        h = r(torch.relu(F.linear(h, W(f"pts_linears.{i}"), B(f"pts_linears.{i}"))))
    beta = r(F.linear(h, W("bottleneck_layer"), B("bottleneck_layer")))
    hbar = r(h.reshape(nv, -1, 128).mean(0))
    raw_sigma = F.linear(hbar, P[pre + "density_layer.weight"].double(), B("density_layer"))
    v = r(F.linear(torch.cat([beta, r(st["dir_tile"])], -1), W("views_linear.0"), B("views_linear.0")))
    q0 = r(torch.relu(v.reshape(nv, -1, 128).mean(0)))
    q1 = r(torch.relu(F.linear(q0, W("views_linear.1"), B("views_linear.1"))))
    raw_rgb = F.linear(q1, P[pre + "rgb_layer.weight"].double(), B("rgb_layer"))
    return torch.sigmoid(raw_rgb).reshape(n, N, 3), torch.relu(raw_sigma).reshape(n, N)


def errors(rgb: Tensor, sigma: Tensor, m_rgb: Tensor, m_sigma: Tensor):
    """(max, mean) of the rgb and sigma errors in the units of the bounds above."""
    e_rgb = (rgb.double().cpu() - m_rgb).abs()
    e_sig = (sigma.double().cpu() - m_sigma).abs() / (1.0 + m_sigma.abs())
    return float(e_rgb.max()), float(e_rgb.mean()), float(e_sig.max()), float(e_sig.mean())
