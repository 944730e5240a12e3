"""CPU: the float64 restatements of the training step's hand-written stages (oracle/train_stage_model.py) against torch.autograd
through the oracle (oracle/neo360_oracle.py) in float64.

* compositing: the explicit backward (G_i, S_i, dalpha_i = G_i T_i - S_i / a_i) equals autograd through `orc.composite` to 1e-12 of the
  magnitude unit, fg and bg, white and black, every upstream gradient alone and all together, on rays with opaque runs, all-zero sigma,
  N = 1 and duplicate t;
* lookups: the gather forward and the `index_add_` backward of the tri-plane and pixel-aligned taps equal `orc.triplane_lookup` /
  `orc.local_lookup` and their autograd, with points outside the maps and behind the cameras; the first-order coordinate-error
  estimate bounds what fp32 arithmetic actually does to the tap coordinates.
"""
import pytest
import torch

from neo360_b200 import synth
from oracle import neo360_oracle as orc
from oracle import train_stage_model as tsm

GRADS = ("g_comp", "g_acc", "g_w", "g_lam", "g_depth")


def composite_case(N, in_sphere, seed):
    """Rays of every regime: realistic, a run of 6 opaque samples (T ~ 1e-60 behind it), one opaque first sample, all-zero sigma,
    duplicate t (delta = 0) and a tiny sigma on the bg 1e10 interval."""
    g = torch.Generator().manual_seed(seed)
    n = 6
    t = torch.sort(torch.rand(n, N, generator=g, dtype=torch.float64), -1, descending=not in_sphere)[0]
    if in_sphere:
        t = t * 1.5 + 1e-4
    sig = torch.nn.functional.softplus(torch.randn(n, N, generator=g, dtype=torch.float64) * 2 - 1)
    if N >= 8:
        sig[1, 1:7] = 1e3
        t[4, 2:5] = t[4, 1]
    sig[2, 0] = 40.0 / max(float((t[2, 1] - t[2, 0]).abs()) if N > 1 else 1.0, 1e-3)
    sig[3] = 0.0
    if not in_sphere:
        sig[5, -1] = 1e-12
    rgb = torch.rand(n, N, 3, generator=g, dtype=torch.float64)
    d = torch.randn(n, 3, generator=g, dtype=torch.float64)
    far = t.abs().amax(1, keepdim=True) + 0.2
    ups = {"g_comp": torch.randn(n, 3, generator=g, dtype=torch.float64), "g_acc": torch.randn(n, generator=g, dtype=torch.float64),
           "g_w": torch.randn(n, N, generator=g, dtype=torch.float64), "g_lam": torch.randn(n, generator=g, dtype=torch.float64),
           "g_depth": torch.randn(n, generator=g, dtype=torch.float64)}
    return rgb, sig, t, d, far, ups


@pytest.mark.parametrize("N", [1, 2, 9, 40])
@pytest.mark.parametrize("in_sphere", [True, False], ids=["fg", "bg"])
@pytest.mark.parametrize("white", [True, False], ids=["white", "black"])
def test_composite_backward_equals_autograd(N, in_sphere, white):
    rgb, sig, t, d, far, ups = composite_case(N, in_sphere, 7 * N + 2 * in_sphere + white)
    names = [k for k in GRADS if in_sphere or k != "g_lam"]
    for use in [[k] for k in names] + [names]:
        r, s = rgb.clone().requires_grad_(True), sig.clone().requires_grad_(True)
        comp, acc, w, lam, depth = orc.composite(r, s[..., None], t, d, white, in_sphere, far)
        outs = {"g_comp": comp, "g_acc": acc, "g_w": w, "g_lam": lam[:, 0] if in_sphere else None, "g_depth": depth}
        loss = sum((outs[k] * ups[k]).sum() for k in use)
        gr, gs = torch.autograd.grad(loss, [r, s], allow_unused=True, materialize_grads=True)
        m = tsm.composite_bwd(rgb, sig, t, d, far, white, in_sphere, fp32=False, **{k: ups[k] for k in use})
        for got, ref, mag in ((m["d_sigma"], gs, m["d_sigma_mag"]), (m["d_rgb"], gr, m["d_rgb_mag"])):
            err = (got - ref).abs()
            assert bool((err <= 1e-12 * mag + 1e-300).all()), (use, float((err / mag.clamp_min(1e-300)).max()))
    f = tsm.composite_fwd(rgb, sig, t, d, far, white, in_sphere, fp32=False)
    comp, acc, w, lam, depth = orc.composite(rgb, sig[..., None], t, d, white, in_sphere, far)
    for a, b in ((f["comp"], comp), (f["acc"], acc), (f["w"], w), (f["depth"], depth)) + (((f["lam"], lam[:, 0]),) if in_sphere else ()):
        assert float((a - b).abs().max()) <= 1e-13 * max(1.0, float(t.abs().max()))


def test_composite_fp32_model_is_on_the_kernels_side_of_the_alpha_rounding():
    """With fp32 rounding on, a sample with e < 2^-25 has alpha = 1 and a = 1e-10 (what the kernel computes); one with e just above
    keeps a = 2^-24 + 1e-10; without it a = e + 1e-10."""
    t = torch.tensor([[0.0, 1.0, 2.0]], dtype=torch.float64)
    d = torch.tensor([[1.0, 0.0, 0.0]], dtype=torch.float64)
    far = torch.tensor([[3.0]], dtype=torch.float64)
    for sd, a32 in ((18.0, tsm.EPS32), (17.0, 2.0 ** -24 + tsm.EPS32)):
        sig = torch.tensor([[sd, 0.5, 0.5]], dtype=torch.float64)
        k = tsm.composite_terms(sig, t, d, far, True, fp32=True)
        assert float(k["a"][0, 0]) == a32
        k64 = tsm.composite_terms(sig, t, d, far, True, fp32=False)
        assert abs(float(k64["a"][0, 0]) - (torch.exp(torch.tensor(-sd, dtype=torch.float64)).item() + 1e-10)) < 1e-16


def lookup_case(seed, nv=3):
    W, H = 64, 48
    sc = synth.make_scene((W, H), nv, (12, 16), seed)
    mp = {k: sc[k].double() for k in ("planes_xz", "planes_xy", "planes_yz", "latent")}
    osc = orc.Scene(mp["planes_xz"], mp["planes_xy"], mp["planes_yz"], mp["latent"], sc["src_poses"].double(),
                    float(sc["src_focal"][0]), float(sc["src_c"][0, 0]), float(sc["src_c"][0, 1]), W, H)
    g = torch.Generator().manual_seed(seed)
    pts = ((torch.rand(400, 3, generator=g) - 0.5) * 3.2)                   # up to 1.6 from the origin: outside the planes
    pts[:50] = sc["src_poses"][0, :3, 3] + torch.randn(50, 3, generator=g) * 0.3     # around (and behind) camera 0
    return sc, osc, pts.float(), (W, H)


@pytest.mark.parametrize("local", [False, True], ids=["triplane", "local"])
def test_lookup_scatter_equals_autograd(local):
    sc, osc, pts, wh = lookup_case(3)
    nv = sc["src_poses"].shape[0]
    planes = [osc.planes_xz, osc.planes_xy, osc.planes_yz]
    taps = tsm.lookup_taps(pts, sc["src_poses"], planes[0].shape[-2:], osc.latent.shape[-2:], osc.focal, osc.cx, osc.cy, wh, local)
    maps = [osc.latent] if local else planes
    leaves = [m.clone().requires_grad_(True) for m in maps]
    if local:
        osc2 = orc.Scene(*planes, leaves[0], osc.src_poses, osc.focal, osc.cx, osc.cy, *wh)
    else:
        osc2 = orc.Scene(*leaves, osc.latent, osc.src_poses, osc.focal, osc.cx, osc.cy, *wh)
    cam = orc.world2camera(pts.double(), osc.src_poses)
    ref = (orc.local_lookup if local else orc.triplane_lookup)(cam, osc2).reshape(nv * pts.shape[0], -1)
    C = ref.shape[1]
    assert sum(float((tp["w"] != 0).sum()) for tp in taps) > 0
    cl = [m.permute(0, 2, 3, 1).contiguous() for m in maps]
    f = tsm.lookup_fwd(taps, cl, nv)
    assert bool(((f["val"] - ref.detach()).abs() <= 1e-12 * f["mag"] + 1e-300).all())
    G = torch.randn(nv * pts.shape[0], C, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    (ref * G).sum().backward()
    for tp, leaf in zip(taps, leaves):
        b = tsm.lookup_bwd(tp, G, nv, chunk_elems=1 << 14)
        want = leaf.grad.permute(0, 2, 3, 1)
        assert bool(((b["val"] - want).abs() <= 1e-12 * b["mag"] + 1e-300).all())
        assert bool((want[~b["reach"]] == 0).all())
        assert float(b["n"].sum()) == float((tp["w"] != 0).sum())
    if local:   # some rows project behind the camera, some off the latent grid
        assert bool((taps[0]["z"] > 0).any()) and bool((taps[0]["w"].sum(1) == 0).any())


def test_lookup_coordinate_error_estimate_bounds_fp32():
    """|ix_fp32 - ix| + |iy_fp32 - iy| <= the model's first-order estimate, for the tap coordinates evaluated with fp32 arithmetic
    (rows with |z_cam| >= 1e-4)."""
    sc, osc, pts, wh = lookup_case(11)
    poses = sc["src_poses"]
    Hl, Wl = osc.latent.shape[-2:]
    for local in (False, True):
        taps = tsm.lookup_taps(pts, poses, osc.planes_xz.shape[-2:], (Hl, Wl), osc.focal, osc.cx, osc.cy, wh, local)
        c = orc.world2camera(pts, poses).reshape(-1, 3)                       # fp32
        if local:
            sc32 = orc.Scene(osc.planes_xz.float(), osc.planes_xy.float(), osc.planes_yz.float(), osc.latent.float(), poses,
                             osc.focal, osc.cx, osc.cy, *wh)
            uv = -c[:, :2] / (c[:, 2:] + 1e-9)
            uv = uv * torch.tensor([sc32.focal, -sc32.focal]) + torch.tensor([sc32.cx, sc32.cy])
            ls = torch.tensor([float(Wl), float(Hl)])
            g = uv * (ls / (ls - 1) * 2.0 / torch.tensor([float(wh[0]), float(wh[1])])) - 1.0
            coords = [(g[:, 0], g[:, 1], Wl, Hl)]
            keep = taps[0]["z"].abs() >= 1e-4
        else:
            Hp, Wp = osc.planes_xz.shape[-2:]
            coords = [(c[:, 0], c[:, 2], Wp, Hp), (c[:, 0], c[:, 1], Wp, Hp), (c[:, 1], c[:, 2], Wp, Hp)]
            keep = torch.ones(c.shape[0], dtype=torch.bool)
        for tp, (gx, gy, W, H) in zip(taps, coords):
            ix, iy = ((gx + 1) / 2 * (W - 1)).double(), ((gy + 1) / 2 * (H - 1)).double()
            err = (ix - tp["ix"]).abs() + (iy - tp["iy"]).abs()
            k = keep & tp["finite"]
            assert bool((err[k] <= tp["derr"][k]).all()), float((err[k] / tp["derr"][k]).max())
