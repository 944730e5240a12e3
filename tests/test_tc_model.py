"""CPU: the float64 model of the tensor-core field kernel (oracle/tc_model.py), which the GPU tests in test_gpu_tc_kernels.py hold the
kernel to.  The model is pinned to the oracle here, without a GPU:

* with fp16=False it is an exact re-association of `neo360_oracle.field` (the folded head, the b0 / b3 constant-one column, the
  projected maps and quirk Q1 all checked to 1e-9 in float64);
* with fp16=True it stays within the kernel's existing bounds of the fp32 oracle;
* every bug of a catalogue of value-level layout bugs moves its output by more than 3x the GPU bounds, so the GPU test would catch it.
"""
import numpy as np
import pytest
import torch

from neo360_b200 import synth
from oracle import neo360_oracle as orc
from oracle import tc_model as tcm

T = lambda a: torch.from_numpy(np.asarray(a))


def scene64(img_wh, nv, plane_hw, seed):
    sc = synth.make_scene(img_wh, nv, plane_hw, seed)
    W, H = img_wh
    d = lambda k: sc[k].double()
    return orc.Scene(d("planes_xz"), d("planes_xy"), d("planes_yz"), d("latent"), d("src_poses"),
                     float(sc["src_focal"][0]), float(sc["src_c"][0, 0]), float(sc["src_c"][0, 1]), W, H)


def random_inputs(n, N, bg, seed):
    """Rays inside the unit sphere, their far distances and t (fg, partly beyond `far`) or descending s (bg) values."""
    g = torch.Generator().manual_seed(seed)
    o = (torch.rand(n, 3, generator=g, dtype=torch.float64) - 0.5) * 1.0
    d = torch.randn(n, 3, generator=g, dtype=torch.float64)
    d = d / d.norm(dim=-1, keepdim=True)
    far = orc.intersect_sphere(o, d)
    u = torch.sort(torch.rand(n, N, generator=g, dtype=torch.float64), -1).values
    t = torch.flip(u, [-1]) if bg else u * far * 1.3
    return {"rays_o": o, "rays_d": d, "viewdirs": d}, far, t


def oracle_field(rays, far, t, mlp_index, sc, P, chunk):
    """neo360_oracle.field over the caller's chunks, fed exactly as `neo360_oracle.render` feeds it (float64 when the inputs are)."""
    o, d, vd = rays["rays_o"], rays["rays_d"], rays["viewdirs"]
    n, N = t.shape
    nv = sc.src_poses.shape[0]
    pre = orc.MLP_NAMES[mlp_index]
    ch = chunk if chunk > 0 else n
    out_rgb, out_sig = [], []
    for c0 in range(0, n, ch):
        sl = slice(c0, min(c0 + ch, n))
        oc, dc, tc, fc = o[sl], d[sl], t[sl], far[sl].reshape(-1, 1)
        B = oc.shape[0]
        dirs_cam = orc.world2camera_dirs(vd[sl], sc.src_poses)
        if mlp_index & 1:
            pts = orc.depth2pts_outside(oc, dc, tc)
            lin = oc[:, None, :] + (fc * (1.0 - tc) + 3.0 * tc)[..., None] * dc[:, None, :]
            cam = orc.world2camera(pts[..., :3].reshape(-1, 3), sc.src_poses)
            enc_in = torch.cat([cam, pts[..., 3].reshape(1, -1, 1).repeat(nv, 1, 1)], -1)
            look = orc.world2camera(lin.reshape(-1, 3), sc.src_poses)
        else:
            pts = oc[:, None, :] + tc[..., None] * dc[:, None, :]
            enc_in = look = orc.world2camera(pts.reshape(-1, 3), sc.src_poses)
        rgb, sig = orc.field(P, pre, enc_in, dirs_cam, orc.triplane_lookup(look, sc).reshape(-1, 128),
                             orc.local_lookup(look, sc).reshape(-1, sc.latent.shape[1]), B, N, nv)
        out_rgb.append(rgb)
        out_sig.append(sig)
    return torch.cat(out_rgb, 0), torch.cat(out_sig, 0)


def md(a, b):
    return float((a.double() - b.double()).abs().max())


@pytest.mark.parametrize("nv", [1, 3, 8])
@pytest.mark.parametrize("mlp_index", [0, 1, 2, 3])
def test_model_without_rounding_is_the_oracle(mlp_index, nv):
    """fp16=False: the kernel's formulation (projected maps, folded head, b0 / b3 on the constant-one column, Q1 from the chunk) is an
    exact re-association of the oracle: <= 1e-9 in float64.  Odd map sizes (plane 13 x 17, latent 18 x 11), ragged n and N, no chunk
    and a chunk that leaves a ragged last chunk."""
    sc = scene64((37, 23), nv, (13, 17), 40 + nv)
    P = {k: v.double() for k, v in synth.make_mlp_params(7).items()}
    rays, far, t = random_inputs(23, 13, mlp_index & 1, 100 + mlp_index)
    for chunk in (0, 7):
        with torch.no_grad():
            rgb, sig = tcm.tc_field(rays, far, t, mlp_index, sc, P, chunk=chunk, fp16=False)
            rr, rs = oracle_field(rays, far, t, mlp_index, sc, P, chunk)
        assert rgb.shape == (23, 13, 3) and sig.shape == (23, 13, 1)
        assert md(rgb, rr) <= 1e-9 and md(sig, rs) <= 1e-9 * (1 + float(rs.abs().max())), (chunk, md(rgb, rr), md(sig, rs))
    # the chunk matters (Q1 is real in this input), and the ray order does not
    a = tcm.tc_field(rays, far, t, mlp_index, sc, P, chunk=7, fp16=False)[0]
    b = tcm.tc_field(rays, far, t, mlp_index, sc, P, chunk=0, fp16=False, ray_order=torch.randperm(23).int())[0]
    assert md(a, b) > 1e-6


def test_q1_source_matches_the_oracle_tiling():
    """Quirk Q1: point (b, s) of a chunk of B rays is conditioned on ray (b N + s) mod B of that chunk (oracle `field`'s repeat)."""
    n, N, chunk = 11, 5, 4
    src = tcm.q1_source(n, N, chunk)
    for c0 in range(0, n, chunk):
        B = min(chunk, n - c0)
        tile = torch.arange(B)[None].repeat(1, N).reshape(-1)            # the oracle's dir_tile row -> ray
        assert torch.equal(src[c0:c0 + B].reshape(-1), c0 + tile)


@pytest.mark.parametrize("tag", ["tiny", "small"])
def test_model_with_rounding_is_within_tc_bounds_of_the_oracle(golden, tag):
    """fp16=True against the fp32 oracle on the golden configs, same t values: within the bounds the TC kernel is held to against the
    oracle (|rgb| 2e-2, sigma 2e-2 + 2 %).  Measured here: rgb 2.8e-3 / 3.0e-3, sigma 4.0e-3 / 3.6e-3 (tiny / small), the size of the
    kernel's own error against the oracle (DESIGN.md section 2)."""
    g = golden
    W, H, hp, wp, B, nc, nf, seed, start = [int(x) for x in g[f"{tag}_cfg"]]
    sc = synth.make_scene((W, H), 3, (hp, wp), seed)
    P = synth.make_mlp_params(seed)
    osc = orc.Scene(sc["planes_xz"], sc["planes_xy"], sc["planes_yz"], sc["latent"], sc["src_poses"],
                    float(sc["src_focal"][0]), float(sc["src_c"][0, 0]), float(sc["src_c"][0, 1]), W, H)
    rays = {k: T(g[f"{tag}_{k}"]) for k in ("rays_o", "rays_d", "viewdirs")}
    with torch.no_grad():
        _, aux = orc.render(rays, osc, P, nc, nf, False, True, return_aux=True)
        worst = [0.0, 0.0]
        for lvl in range(2):
            for b, (tk, rk, sk) in enumerate((("fg_t", "fg_rgb", "fg_sigma"), ("bg_s", "bg_rgb", "bg_sigma"))):
                rgb, sig = tcm.tc_field(rays, aux[lvl]["far"], aux[lvl][tk], 2 * lvl + b, osc, P)
                ref_s = aux[lvl][sk].double()
                ds = (sig - ref_s).abs()
                assert float((ds - 0.02 * ref_s.abs()).max()) < 2e-2, (lvl, b, float(ds.max()))
                assert md(rgb, aux[lvl][rk]) < 2e-2, (lvl, b)
                worst = [max(worst[0], md(rgb, aux[lvl][rk])), max(worst[1], float(ds.max()))]
    print(f"tc model (fp16) vs fp32 oracle [{tag}]: rgb {worst[0]:.2e}, sigma {worst[1]:.2e}")
    assert worst[0] < 5e-3


def test_mutation_catalogue_exceeds_gpu_bounds():
    """Each value-level bug of tc_model.MUTATIONS, applied to the model, must move rgb or sigma by more than 3x a GPU bound (the per-point
    tc_model.RGB_TOL / SIGMA_TOL or the per-case mean RGB_MEAN_TOL / SIGMA_MEAN_TOL) on these inputs (nv = 3, odd map sizes, all four
    MLPs, ragged chunks); the GPU test, which compares the kernel with the unmutated model at those bounds, then fails for the same bug
    in the kernel.

    Measured here (first column), and the same bug against the fp32 oracle at the old field bound (|rgb| 2e-2, sigma 2e-2 + 2 %) on
    the inputs of test_gpu_parity.py::test_field_eval_tc_vs_oracle (75 frame rays, 16 + 8 samples, both levels):
      mutation      x GPU bound   vs oracle, old inputs   the bug
      pmap_swap     68            rgb 4.8e-1              two channels of the projected-map order exchanged
      sigma_no_inv  1289          sigma 1.3e1             sigma row of the folded head not divided by nv
      b0_off        13            rgb 6.7e-2              b0 missing from the constant-one column
      b3_off        33            rgb 9.3e-2              b3 missing from the constant-one column
      tap_edge      86            rgb 4.9e-1              right / bottom taps past the last texel read it
      no_q1         229           rgb 6.6e-1              direction term from the point's own ray (no Q1)
      no_w3enc      458           rgb 8.8e-1              the W3enc block of layer 3 dropped
      dir_colmap    46            rgb 9.1e-2              two columns of the direction-term column map exchanged
    None of these whole-channel / whole-block bugs would have been missed by the old 2e-2 bound on its own inputs (the closest, b0_off,
    clears it by 3x).  The test prints the values it measures."""
    sc = scene64((37, 23), 3, (13, 17), 8)
    P = synth.make_mlp_params(3)
    cases = []
    for mlp_index in range(4):
        rays, far, t = random_inputs(40, 24, mlp_index & 1, 200 + mlp_index)
        with torch.no_grad():
            base = tcm.tc_field(rays, far, t, mlp_index, sc, P, chunk=16)
        cases.append((rays, far, t, mlp_index, base))
    # the old test's inputs (test_gpu_parity.py::test_field_eval_tc_vs_oracle)
    s0 = synth.make_scene((64, 48), 3, (24, 32), 0)
    P0 = synth.make_mlp_params(0)
    osc = orc.Scene(s0["planes_xz"], s0["planes_xy"], s0["planes_yz"], s0["latent"], s0["src_poses"],
                    float(s0["src_focal"][0]), float(s0["src_c"][0, 0]), float(s0["src_c"][0, 1]), 64, 48)
    ro, vd, rd, _ = orc.rays_from_pose(orc.ray_directions(48, 64, 0.8 * 64), synth.target_pose(3, 100)[:3, :4])
    old_rays = {"rays_o": ro[1000:1075], "rays_d": rd[1000:1075], "viewdirs": vd[1000:1075]}
    with torch.no_grad():
        _, aux = orc.render(old_rays, osc, P0, 16, 8, False, True, return_aux=True)
    report = []
    for mut in tcm.MUTATIONS:
        seen, old_rgb, old_sig = 0.0, 0.0, 0.0
        with torch.no_grad():
            for rays, far, t, mlp_index, (rgb0, sig0) in cases:
                rgb, sig = tcm.tc_field(rays, far, t, mlp_index, sc, P, chunk=16, mutation=mut)
                dr, dsig = (rgb - rgb0).abs().amax(-1), (sig - sig0).abs() / (1 + sig0)
                seen = max(seen, float(dr.max()) / tcm.RGB_TOL, float(dsig.max()) / tcm.SIGMA_TOL,
                           float(dr.mean()) / tcm.RGB_MEAN_TOL, float(dsig.mean()) / tcm.SIGMA_MEAN_TOL)
            for lvl in range(2):
                for b, (tk, rk, sk) in enumerate((("fg_t", "fg_rgb", "fg_sigma"), ("bg_s", "bg_rgb", "bg_sigma"))):
                    rgb, sig = tcm.tc_field(old_rays, aux[lvl]["far"], aux[lvl][tk], 2 * lvl + b, osc, P0, mutation=mut)
                    rs = aux[lvl][sk].double()
                    old_rgb = max(old_rgb, md(rgb, aux[lvl][rk]))
                    old_sig = max(old_sig, float(((sig - rs).abs() - 0.02 * rs.abs()).max()))
        caught_old = old_rgb >= 2e-2 or old_sig >= 2e-2
        report.append(f"{mut:13s} {seen:9.1f} x GPU bound | vs oracle, old test's inputs: rgb {old_rgb:.1e} sigma {old_sig:.1e} "
                      f"({'caught' if caught_old else 'MISSED'} by the 2e-2 bound)")
        assert seen > 3.0, report[-1]
    print("\n" + "\n".join(report))
