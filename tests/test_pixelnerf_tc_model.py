"""oracle/pixelnerf_tc_model.py with its fp16 roundings off equals the PixelNeRF oracle's field (the formulation the tensor-core path
computes is the reference's), and with them on differs from it by fp16 noise only."""
import torch

from neo360_b200 import synth
from oracle import pixelnerf_oracle as por
from oracle import pixelnerf_tc_model as ptm


def _case(nv=3, n=16, N=9, seed=3):
    W, H = 64, 48
    sc = synth.make_scene((W, H), nv, (8, 8), seed)
    g = torch.Generator().manual_seed(seed)
    o = torch.randn(n, 3, generator=g) * 0.1 + torch.tensor([0.6, 0.2, 0.3])
    d = -o + torch.randn(n, 3, generator=g) * 0.2
    rays = {"rays_o": o, "rays_d": d, "viewdirs": d / d.norm(dim=-1, keepdim=True)}
    t = torch.sort(torch.rand(n, N, generator=g) * 1.5 + 0.02, -1).values
    osc = por.scene(sc["latent"], sc["src_poses"], sc["src_focal"], sc["src_c"], (W, H))
    return rays, t, osc, synth.make_pixelnerf_params(seed)


def test_model_without_rounding_is_the_oracle():
    rays, t, osc, P = _case()
    n, N = t.shape
    rgb, sigma = ptm.tc_field(P, "coarse_mlp.", rays, t, osc, fp16=False)
    pts = (rays["rays_o"][:, None, :] + t[..., None] * rays["rays_d"][:, None, :]).double()
    P64 = {k: v.double() for k, v in P.items()}
    sc64 = dict(osc, latent=osc["latent"].double(), src_poses=osc["src_poses"].double())
    st = por.stages(pts, rays["viewdirs"].double(), sc64, N)
    raw_rgb, raw_sigma = por.mlp_forward(P64, "coarse_mlp.", st["enc"], st["dir_tile"], st["latent"], 3)
    assert float((rgb - torch.sigmoid(raw_rgb).reshape(n, N, 3)).abs().max()) < 1e-9
    assert float((sigma - torch.relu(raw_sigma).reshape(n, N)).abs().max()) < 1e-9


def test_fp16_roundings_stay_small():
    rays, t, osc, P = _case()
    a = ptm.tc_field(P, "fine_mlp.", rays, t, osc, fp16=True)
    b = ptm.tc_field(P, "fine_mlp.", rays, t, osc, fp16=False)
    e = ptm.errors(a[0], a[1], b[0], b[1])
    assert 0 < e[0] < 5e-2 and e[2] < 1e-1
