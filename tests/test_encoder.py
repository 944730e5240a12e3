"""Tri-plane builder (SURVEY.md 8(f1)): neo360_b200.encoder.GridEncoder against vectors minted from the UNMODIFIED reference module
(oracle/make_golden_encoder.py: state dicts bit-identical under the same seed, outputs bit-identical on CPU), and the hand-written
CUDA dense part (wgmma) against the module's own fp32 framework-op form."""
import os

import numpy as np
import pytest
import torch

from neo360_b200 import synth

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "encoder_reference_vectors.npz")
T = lambda a: torch.from_numpy(np.asarray(a))


def _setup():
    from neo360_b200.encoder import GridEncoder
    g = np.load(GOLD)
    seed, W, H, NV = [int(x) for x in g["cfg"]]
    torch.manual_seed(seed)
    enc = GridEncoder().eval()
    sc = synth.make_scene((W, H), NV, (12, 16), seed)
    return g, enc, sc, T(g["imgs"]), W, H


def test_grid_encoder_framework_form_matches_reference_vectors():
    """CPU: seeded construction + framework-op forward reproduce the reference's planes and latent (strided samples) to 1e-5."""
    g, enc, sc, imgs, W, H = _setup()
    with torch.no_grad():
        lat = enc.spatial_encoder(imgs)
        fl = enc.dense_torch(lat, sc["src_poses"], sc["src_focal"], sc["src_c"], W, H)
        planes = {"xz": enc.floorplan_convnet_xz(fl[0]), "xy": enc.floorplan_convnet_xy(fl[1]), "yz": enc.floorplan_convnet_yz(fl[2])}
    assert float((lat[:, ::16, ::3, ::4] - T(g["latent_s"])).abs().max()) < 1e-4
    for k, p in planes.items():
        assert p.shape == (3, 128, 120, 160)
        assert float((p[:, ::8, ::6, ::8] - T(g[f"plane_{k}_s"])).abs().max()) < 1e-5, k
    for k, f in zip(("xz", "xy", "yz"), fl):
        assert float((f[:, ::16, ::4, ::4] - T(g[f"floor_{k}_s"])).abs().max()) < 1e-5, k


@pytest.mark.gpu
def test_grid_encoder_cuda_dense_part(tmp_path):
    """GPU: `neo_grid_encoder_dense` (gather + DepthPillarEncoder + pillar aggregators on the tensor cores, fp16 operands) against the fp32
    framework-op form of the same module and weights; then the whole forward against the reference planes.
    Stated: pillar sums within 2e-2 of their scale (fp16 weights / activations through 4 dense layers + softmax); planes within 3e-2 of scale."""
    assert torch.cuda.is_available()
    from neo360_b200 import build
    build.build()
    dev = torch.device("cuda:0")
    g, enc, sc, imgs, W, H = _setup()
    enc = enc.to(dev)
    poses, focal, c = sc["src_poses"].to(dev), sc["src_focal"].to(dev), sc["src_c"].to(dev)
    with torch.no_grad():
        lat = enc.spatial_encoder(imgs.to(dev))
        ref = enc.dense_torch(lat, poses, focal, c, W, H)
        got = enc.dense_cuda(lat, poses, focal, c, W, H)
        torch.cuda.synchronize()
        for k, a, b in zip(("xz", "xy", "yz"), got, ref):
            scale = float(b.abs().max())
            err = float((a - b).abs().max())
            print(f"pillar sums {k}: max err {err:.3e}, scale {scale:.3f}")
            assert err < 2e-2 * scale, (k, err, scale)
        xz, xy, yz = enc(imgs.to(dev), poses, focal, c)          # eval + no_grad: the CUDA dense part
    for k, p in (("xz", xz), ("xy", xy), ("yz", yz)):
        refp = T(g[f"plane_{k}_s"])
        err = float((p[:, ::8, ::6, ::8].cpu() - refp).abs().max())
        print(f"plane {k} vs reference: max err {err:.3e}, scale {float(refp.abs().max()):.3f}")
        assert err < 3e-2 * float(refp.abs().max()), (k, err)


@pytest.mark.gpu
def test_renderer_with_grid_encoder_handoff():
    """The `encoder=` hand-off of NeRF_TP (renderer.py): real GridEncoder output magnitudes (random ResNet) through the tensor-core
    renderer against the fp32 CUDA path on the same planes: L-inf <= 1e-2 on rgb, PSNR >= 45 dB."""
    from neo360_b200 import NeRF_TP
    from neo360_b200.encoder import GridEncoder
    from oracle import neo360_oracle as orc
    dev = torch.device("cuda:0")
    W, H, nc, nf = 64, 48, 24, 12
    torch.manual_seed(2)
    enc = GridEncoder().eval()
    net = NeRF_TP(num_coarse_samples=nc, num_fine_samples=nf, encoder=enc, precision="tc").eval()
    sd = net.state_dict()
    sd.update(synth.make_mlp_params(2))
    net.load_state_dict(sd)
    net = net.to(dev)
    sc = synth.make_scene((W, H), 3, (12, 16), 2)
    pose = synth.target_pose(9, 100)
    ro, vd, rd, _ = orc.rays_from_pose(orc.ray_directions(H, W, 0.8 * W), pose[:3, :4])
    g = torch.Generator().manual_seed(2)
    batch = {"rays_o": ro[500:600].contiguous().to(dev), "rays_d": rd[500:600].contiguous().to(dev), "viewdirs": vd[500:600].contiguous().to(dev),
             "src_imgs": (torch.rand(3, 3, H, W, generator=g) * 2 - 1).to(dev), "src_poses": sc["src_poses"].to(dev),
             "src_focal": sc["src_focal"].to(dev), "src_c": sc["src_c"].to(dev)}
    with torch.no_grad():
        a = net(batch, False, False, None, None, out_depth=True)[1]
        net.check()
        net.precision = "fp32"
        net._scene_src = None                      # rebuild the scene with the fp32 path prepared
        b = net(batch, False, False, None, None, out_depth=True)[1]
        net.check()
    err = float((a[0] - b[0]).abs().max())
    ps = orc.psnr(a[0].cpu(), b[0].cpu())
    print(f"encoder hand-off: TC vs fp32 CUDA on real encoder planes: L-inf {err:.2e}, PSNR {ps:.1f} dB")
    assert err < 1e-2 and ps > 45.0
