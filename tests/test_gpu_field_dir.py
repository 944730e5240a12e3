"""GPU: the direction fragments of the NEO_PREC_TC field kernel (csrc/field_tc.cu, dir_frag_kernel).

The view-mean direction encoding that conditions the colour head depends only on the conditioning ray and the source cameras, so it
is computed once per ray and call and read by every field launch.  These tests check
* the fragments against a float64 rotation and sine of the same columns, within half an fp16 ulp plus the fp32 error of the kernel's
  rotation and argument, with the padding columns 27-31 exactly zero, for nv 1, 3 and 8;
* that neo_field_eval (fragments in a pool block) and neo_render_fwd (fragments in the render workspace) give the same field rows
  for the same rays and samples, bit for bit.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from neo360_b200 import _lib as L
from neo360_b200 import ops, synth
from oracle import neo360_oracle as orc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cuda():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()
    return torch.device("cuda:0")


def tc_net(cuda, nv, seed, nc=8, nf=4):
    from neo360_b200 import NeRF_TP
    sc = synth.make_scene((37, 23), nv, (13, 17), seed)
    P = synth.make_mlp_params(seed)
    net = NeRF_TP(num_coarse_samples=nc, num_fine_samples=nf, num_src_views=nv, precision="tc").eval()
    net.load_state_dict(P)
    net = net.to(cuda)
    net.set_scene(*[sc[k].to(cuda) for k in ("planes_xz", "planes_xy", "planes_yz", "latent", "src_poses", "src_focal", "src_c")],
                  sc["img_wh"], precisions=["tc"])
    return net, sc


def random_rays(cuda, n, seed):
    g = torch.Generator().manual_seed(seed)
    o = (torch.rand(n, 3, generator=g) - 0.5) * 1.0
    d = torch.randn(n, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True)
    return {"rays_o": o.to(cuda), "rays_d": d.to(cuda), "viewdirs": d.to(cuda)}


def dir_fragments(net, rays):
    """neo_tc_dir_fragments -> (n, 32) float64 columns, decoded from the 64-byte per-ray records."""
    n = rays["viewdirs"].shape[0]
    o, d, vd = (rays[k].contiguous().float() for k in ("rays_o", "rays_d", "viewdirs"))
    r = L.NeoRays()
    r.n_rays, r.chunk = n, 0
    r.rays_o, r.rays_d, r.viewdirs = L.ptr(o), L.ptr(d), L.ptr(vd)
    out = torch.empty(n, 64, dtype=torch.uint8, device=vd.device)
    L.check(L.load().neo_tc_dir_fragments(net._scene.handle, C.byref(r), L.ptr(out), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    h = out.cpu().numpy().view(np.float16).reshape(n, 4, 4, 2)          # [ray][thread t][word 2 ks + h][pair element e]
    cols = np.empty(n * 32, np.float64).reshape(n, 32)
    for t in range(4):
        for w in range(4):
            for e in range(2):
                cols[:, 16 * (w >> 1) + 8 * (w & 1) + 2 * t + e] = h[:, t, w, e]
    return cols


def dir_model(vd, poses):
    """float64 view mean of pos_enc(R^T d, 0, 4) (model.py:357-360), zero-padded to 32 columns."""
    dc = orc.world2camera_dirs(vd.double().cpu(), poses.double().cpu())   # (nv, n, 3)
    enc = orc.pos_enc(dc, 0, 4).mean(0)                                  # (n, 27)
    return torch.cat([enc, torch.zeros(enc.shape[0], 5, dtype=torch.float64)], -1).numpy()


def half_ulp16(a):
    """half the fp16 spacing at magnitude a (subnormal spacing 2^-24 below 2^-14)."""
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return 0.5 * 2.0 ** (e - 10)


@pytest.mark.parametrize("nv", [1, 3, 8])
def test_dir_fragments_vs_float64(cuda, nv):
    """Every column of every ray within half an fp16 ulp of the float64 value, plus 8e-6 for the fp32 rotation (|d| = 1, a few
    units of 2^-23), scaled by up to 2^3 in the highest level's argument, and sinf; padding columns exactly zero."""
    net, sc = tc_net(cuda, nv, 70 + nv)
    rays = random_rays(cuda, 2000, 700 + nv)
    got = dir_fragments(net, rays)
    ref = dir_model(rays["viewdirs"], sc["src_poses"])
    assert np.all(got[:, 27:] == 0.0)
    slack = 8e-6
    bound = half_ulp16(np.abs(ref) + slack) + slack
    err = np.abs(got - ref)
    print(f"dir fragments nv={nv}: max |err| {err.max():.3e}, max err / bound {(err / bound).max():.3f}")
    assert np.all(err <= bound), np.unravel_index(np.argmax(err / bound), err.shape)


@pytest.mark.parametrize("chunk", [0, 24])
def test_field_eval_matches_render(cuda, chunk):
    """neo_field_eval on the t / s values neo_render_fwd sampled gives the render's per-sample rgb and sigma bit for bit: both
    compute the direction fragments with the same kernel and the field launches read them the same way (quirk Q1 chunks: 0 = one
    chunk, 24 = several chunks, the last one ragged)."""
    net, sc = tc_net(cuda, 3, 91)
    rays = random_rays(cuda, 100, 910 + chunk)
    with torch.no_grad():
        net(rays, False, False, None, None, out_depth=True, chunk=chunk, debug=True)
        net.check()
        dbg = {k: [t.clone() for t in v] for k, v in net.last_debug.items()}
        far = ops.intersect_sphere(rays["rays_o"], rays["rays_d"])
        for lvl in range(2):
            for b, (tk, rk, sk) in enumerate((("fg_t", "fg_rgb_s", "fg_sigma"), ("bg_s", "bg_rgb_s", "bg_sigma"))):
                rgb, sig = net.field_eval(rays, far, dbg[tk][lvl], 2 * lvl + b, chunk=chunk, precision="tc")
                net.check()
                assert torch.equal(rgb, dbg[rk][lvl]), (lvl, b)
                assert torch.equal(sig[..., 0], dbg[sk][lvl]), (lvl, b)
