"""GPU: the vanilla NeRF, Mip-NeRF 360 and GridEncoder tensor-core paths stage by stage against float64 models of the same computation
(oracle/tc_paths_model.py, pinned to the oracles on the CPU by tests/test_tc_paths_model.py), and `rowdot_f16`, the head kernel they
share, against a float64 dot product of its own operands.

* rowdot_f16 at its callers' K and row strides, N 1 / 3, M from 1 to 10^6: element-wise bound, sentinel past row M.
* vanilla NeRF, each level: sigma / rgb per point against the model at the kernel's own t; weights / rgb / acc / depth per ray against
  `vanilla_oracle.composite` in float64 of the kernel's own sigma, rgb and t; white and black backgrounds.
* Mip-NeRF 360, each level: (i) the kernel's sdist against `max_dilate_weights` + `sample_intervals` of its previous level in fp32,
  (ii) density / rgb per point against the model at the kernel's own intervals (TC), (iii) weights / rgb per ray against
  `alpha_weights` in float64 of the kernel's own density and rgb.  (i) and (iii) in both precisions.
* GridEncoder dense part: pillar sums of `dense_cuda` on a synthetic latent against the model at seeded pillars.

Bounds: tc_paths_model.*_TOL and the constants below; the values measured on an H100 are in the docstrings and DESIGN.md section 2.
Run with `-m gpu -s`: every comparison prints its per-point maximum and its mean.
"""
import math

import pytest
import torch

from neo360_b200 import synth
from oracle import mip_oracle as mo
from oracle import neo360_oracle as orc
from oracle import tc_paths_model as tpm
from oracle import vanilla_oracle as vo

pytestmark = pytest.mark.gpu

# Measured on an H100 80GB HBM3 at a 400 W power limit; each bound is 2-3x the largest value measured.
# rowdot_f16: |got - ref| <= ROWDOT_C 2^-24 (sum_k |h_k w_k| + |b|)  (measured 1.54)
ROWDOT_C = 4.0
# vanilla compositing of the kernel's own sigma / rgb / t against float64: weights, rgb, acc; depth relative to far  (measured 4.9e-7)
VAN_COMP_TOL = 1.5e-6
# Mip-NeRF 360: (i) >= 99 % of sdist within MIP_S_TOL, every one within one interval (measured: none beyond 2e-6, max 7.2e-7);
# (iii) weights and rgb (measured 1.5e-6)
MIP_S_TOL = 2e-6
MIP_COMP_TOL = 4e-6
SUBSET = 16384          # points (pillars) of a large case compared with the model, plus every point of the last 128-row tile


@pytest.fixture(scope="module")
def cuda():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()
    return torch.device("cuda:0")


def subset(M, seed, device):
    """Row indices compared with a float64 model: all of them, or SUBSET seeded rows plus the whole last (ragged) 128-row tile."""
    if M <= SUBSET:
        return torch.arange(M, device=device)
    g = torch.Generator().manual_seed(seed)
    last = torch.arange(M - ((M - 1) % 128 + 1), M)
    return torch.unique(torch.cat([torch.randperm(M, generator=g)[:SUBSET], last])).to(device)


def stats(e):
    return float(e.max()), float(e.mean())


# ---------------- rowdot_f16 ----------------

ROWDOT_KLD = [(128, 128), (256, 320), (256, 768), (512, 512), (1024, 1536)]     # (K, row stride) as csrc/vanilla.cu, mip.cu, encoder.cu
ROWDOT_M = [1, 127, 128, 129, 4097, 1_000_003]


@pytest.mark.parametrize("K,ld", ROWDOT_KLD, ids=[f"K{k}-ld{l}" for k, l in ROWDOT_KLD])
def test_rowdot_f16_vs_float64(cuda, K, ld):
    """out = H . W^T + b for fp16 rows H (padding columns NaN, so a read past K shows), fp32 W and b, against float64 of the same
    operands, N in {1, 3}, M in {1, 127, 128, 129, 4097, 1000003}.  Stated, element-wise: |got - ref| <= ROWDOT_C 2^-24 (sum_k |h w| + |b|);
    rows >= M keep their sentinel."""
    from neo360_b200 import _lib as L
    lib = L.load()
    worst = 0.0
    for N in (1, 3):
        for M in ROWDOT_M:
            g = torch.Generator(device=cuda).manual_seed(K * 7 + N * 3 + M)
            hbuf = torch.full((M, ld), float("nan"), device=cuda, dtype=torch.float16)
            hbuf[:, :K] = torch.randn(M, K, generator=g, device=cuda).half()
            w = torch.randn(N, K, generator=g, device=cuda) / math.sqrt(K)
            b = torch.randn(N, generator=g, device=cuda)
            out = torch.full((M + 3, N), 0x7FBADBAD, dtype=torch.int32, device=cuda)
            L.check(lib.neo_tc_rowdot_f16(hbuf.data_ptr(), ld, K, w.data_ptr(), b.data_ptr(), N, M, out.data_ptr(),
                                          torch.cuda.current_stream().cuda_stream))
            torch.cuda.synchronize()
            h64, w64 = hbuf[:, :K].double(), w.double()
            ref = h64 @ w64.T + b.double()
            scale = h64.abs() @ w64.abs().T + b.double().abs()
            got = out[:M].view(torch.float32).double()
            ratio = float(((got - ref).abs() / scale).max()) * 2.0 ** 24 if bool(torch.isfinite(got).all()) else float("inf")
            sentinel = bool((out[M:] == 0x7FBADBAD).all())
            print(f"rowdot_f16 K={K:4d} ld={ld:4d} N={N} M={M:7d}: max |err| / (2^-24 sum|hw| + |b|) = {ratio:.2f}, "
                  f"sentinel {'intact' if sentinel else 'OVERWRITTEN'}")
            assert sentinel, (K, ld, N, M)
            worst = max(worst, ratio)
    print(f"rowdot_f16 K={K} ld={ld}: worst {worst:.2f} x 2^-24 (bound {ROWDOT_C})")
    assert worst <= ROWDOT_C, worst


# ---------------- vanilla NeRF ----------------

def frame_rays(W, H, view, idx):
    ro, vd, rd, radii = orc.rays_from_pose(orc.ray_directions(H, W, 0.8 * W), synth.target_pose(view, 100)[:3, :4])
    return {"rays_o": ro[idx].contiguous(), "rays_d": rd[idx].contiguous(), "viewdirs": vd[idx].contiguous()}, radii[idx].contiguous()


def spread(n, total):
    return torch.linspace(0, total - 1, n).long()


def vanilla_rays(kind):
    if kind == "v_cfg1":
        import os
        import numpy as np
        g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vanilla_reference_vectors.npz"))
        return {k: torch.from_numpy(g[f"v_cfg1_{k}"]) for k in ("rays_o", "rays_d", "viewdirs")}
    if kind == "slice":                        # 65536 consecutive pixels (rows 120..256) of a 640 x 480 frame: one library call
        return frame_rays(640, 480, 3, torch.arange(120 * 640, 120 * 640 + 65536))[0]
    return frame_rays(64, 48, 7, spread(kind, 64 * 48))[0]


# name, rays, n_coarse, n_fine, density bias shift (-25: nearly empty rays, acc well inside (0, 1))
VAN_CASES = [("1 ray 3+1", 1, 3, 1, 1.0), ("33 rays 16+8", 33, 16, 8, 1.0), ("33 rays 16+8 nearly empty", 33, 16, 8, -25.0),
             ("configs[0] 1024 rays 64+64", "v_cfg1", 64, 64, 1.0), ("640x480 slice 65536 rays 64+128", "slice", 64, 128, 1.0)]


@pytest.mark.parametrize("case", VAN_CASES, ids=[c[0] for c in VAN_CASES])
def test_vanilla_tc_levels_match_model(cuda, case):
    """Each level: the kernel's sigma / rgb per point against tc_paths_model.vanilla_tc_field at the kernel's own t (bounds VAN_*_TOL), the
    black-background run's field bit-identical to the white one, and weights / rgb / acc / depth per ray against
    `vanilla_oracle.composite` in float64 of the kernel's own sigma, rgb and t (VAN_COMP_TOL; depth relative to far = 3)."""
    from neo360_b200.vanilla import NeRF
    name, kind, nc, nf, shift = case
    P = synth.make_vanilla_params(4, density_bias_shift=shift)
    net = NeRF(num_coarse_samples=nc, num_fine_samples=nf).eval()
    net.precision = "tc"
    net.load_state_dict(P)
    net = net.to(cuda)
    rays = {k: v.to(cuda) for k, v in vanilla_rays(kind).items()}
    runs = {}
    with torch.no_grad():
        for white in (True, False):
            ev = net(rays, False, white, 0.2, 3.0, debug=True)
            runs[white] = (ev, {k: [t.clone() for t in v] for k, v in net.last_debug.items()})
    torch.cuda.synchronize()
    worst = {}
    for lvl, pre in enumerate(("coarse_mlp.", "fine_mlp.")):
        dbg = runs[True][1]
        t, sig, rgb = dbg["t"][lvl], dbg["sigma"][lvl], dbg["rgb_s"][lvl]
        assert torch.equal(sig, runs[False][1]["sigma"][lvl]) and torch.equal(rgb, runs[False][1]["rgb_s"][lvl])
        n, N = t.shape
        idx = subset(n * N, lvl, cuda)
        b = torch.div(idx, N, rounding_mode="floor")
        sub = {k: v[b] for k, v in rays.items()}
        with torch.no_grad():
            mr, ms = tpm.vanilla_tc_field(P, pre, sub, t.reshape(-1)[idx][:, None])
        er = (rgb.reshape(-1, 3)[idx].double() - mr[:, 0]).abs().amax(-1)
        es = tpm.sigma_error(sig.reshape(-1)[idx], ms[:, 0, 0])
        f = (*stats(er), *stats(es))
        print(f"vanilla tc [{name}] level {lvl}: {idx.numel()} of {n * N} points: rgb max {f[0]:.2e} mean {f[1]:.2e}, "
              f"sigma (pre-activation units) max {f[2]:.2e} mean {f[3]:.2e}")
        assert f[0] <= tpm.VAN_RGB_TOL and f[1] <= tpm.VAN_RGB_MEAN_TOL, f
        assert f[2] <= tpm.VAN_SIGMA_TOL and f[3] <= tpm.VAN_SIGMA_MEAN_TOL, f
        for white in (True, False):
            ev, dbg = runs[white]
            comp, acc, w, depth = vo.composite(rgb.double(), sig.double(), t.double(), rays["rays_d"].double(), white)
            e = {"weights": float((dbg["weights"][lvl].double() - w).abs().max()), "rgb": float((ev[lvl][0].double() - comp).abs().max()),
                 "acc": float((ev[lvl][1].double() - acc).abs().max()), "depth/far": float((ev[lvl][2].double() - depth).abs().max()) / 3.0}
            print(f"vanilla tc [{name}] level {lvl} {'white' if white else 'black'}: compositing vs float64: " +
                  ", ".join(f"{k} {v:.1e}" for k, v in e.items()) + f"; acc in [{float(acc.min()):.3f}, {float(acc.max()):.3f}]")
            for k, v in e.items():
                worst[k] = max(worst.get(k, 0.0), v)
            if shift < 0:
                assert float(acc.min()) < 0.5 and float(acc.max()) > 0.05, "the nearly empty case must leave acc inside (0, 1)"
    assert all(v <= VAN_COMP_TOL for v in worst.values()), worst


# ---------------- Mip-NeRF 360 ----------------

# name, rays, n_prop, n_nerf, far, train_frac, jitter
MIP_CASES = [("1 ray 2/2", 1, 2, 2, 6.0, 1.0, False), ("33 rays 2/2", 33, 2, 2, 6.0, 1.0, False),
             ("37 rays 160/160", 37, 160, 160, 6.0, 1.0, False), ("129 rays 16/8 jitter train_frac 0.5", 129, 16, 8, 6.0, 0.5, True),
             ("configs[2] 8191 rays 64/64 far 100", 8191, 64, 64, 100.0, 1.0, False)]
NEAR = 0.2


def s_to_t32(s, far):
    sf, sn = torch.tensor(1.0) / torch.tensor(far), torch.tensor(1.0) / torch.tensor(NEAR)
    return 1.0 / (s * sf.to(s.device) + (1.0 - s) * sn.to(s.device))


@pytest.mark.parametrize("case", MIP_CASES, ids=[c[0] for c in MIP_CASES])
def test_mip360_levels_match_models(cuda, case):
    """Every level of both precisions, from the kernel's own ray history:
    (i) sdist against max_dilate_weights + sample_intervals of the kernel's previous level in fp32: >= 99 % within MIP_S_TOL, all within
        the widest interval of their ray;
    (ii) TC only: density / rgb per point against tc_paths_model.mip_tc_field at the kernel's intervals (t recomputed in fp32 from
        sdist): bounds MIP_*_TOL; fp32 only, configs[2] (far 100): density / rgb against mip_oracle.mlp in fp32 at the oracle tolerance
        (>= 99 % within 2e-4, L-inf 5e-3);
    (iii) weights and rgb per ray against alpha_weights in float64 of the kernel's own density and rgb: MIP_COMP_TOL."""
    from neo360_b200.mip import MipNeRF360
    name, nr, npp, nn_, far, tf, jitter = case
    P = synth.make_mip_params(2)
    rays, radii = frame_rays(640, 480, 5, spread(nr, 640 * 480))
    batch = {k: v.to(cuda) for k, v in rays.items()}
    batch["radii"] = radii.to(cuda)
    if jitter:
        batch["_uniforms"] = [torch.rand(nr, 1, generator=torch.Generator().manual_seed(i)).to(cuda) for i in range(3)]
    anneal = (10 * tf) / (9 * tf + 1)
    for prec in ("fp32", "tc"):
        net = MipNeRF360(num_prop_samples=npp, num_nerf_samples=nn_, precision=prec).eval()
        net.load_state_dict(P)
        net = net.to(cuda)
        with torch.no_grad():
            ren, hist = net(batch, tf, jitter, False, NEAR, far)
        torch.cuda.synchronize()
        prod = 1
        for lvl in range(3):
            n = npp if lvl < 2 else nn_
            dil = 0.0025 + 0.5 / prod
            prod *= n
            sd, dens, rgb, wts = (hist[lvl][k] for k in ("sdist", "density", "rgb", "weights"))
            # (i) resampling
            if lvl == 0:
                s_prev = torch.tensor([[0.0, 1.0]], device=cuda).expand(nr, 2)
                w_prev = torch.ones(nr, 1, device=cuda)
            else:
                s_prev, w_prev = mo.max_dilate_weights(hist[lvl - 1]["sdist"], hist[lvl - 1]["weights"], dil)
                s_prev, w_prev = s_prev[..., 1:-1], w_prev[..., 1:-1]
            logits = torch.where(s_prev[..., 1:] > s_prev[..., :-1], anneal * torch.log(w_prev), torch.full_like(w_prev, -torch.inf))
            s_ref = mo.sample_intervals(s_prev, logits, n, batch["_uniforms"][lvl] if jitter else None)
            ds = (sd - s_ref).abs()
            frac = float((ds > MIP_S_TOL).float().mean())
            width = (s_ref[:, 1:] - s_ref[:, :-1]).amax(-1, keepdim=True)
            print(f"mip {prec} [{name}] level {lvl} (i) sdist: max {float(ds.max()):.1e}, {100 * frac:.2f} % > {MIP_S_TOL:.0e}, "
                  f"max / widest interval {float((ds / width).max()):.2e}")
            assert frac <= 0.01 and bool((ds <= width).all()), (prec, lvl)
            td = s_to_t32(sd, far)
            # (iii) compositing
            w64 = mo.alpha_weights(dens.double(), td.double(), batch["rays_d"].double())
            r64 = (w64[..., None] * rgb.double()).sum(-2) + (1 - w64.sum(-1, keepdim=True)).clamp(min=0)
            ew, ec = float((wts.double() - w64).abs().max()), float((ren[lvl]["rgb"].double() - r64).abs().max())
            print(f"mip {prec} [{name}] level {lvl} (iii) compositing vs float64: weights {ew:.1e}, rgb {ec:.1e}")
            assert ew <= MIP_COMP_TOL and ec <= MIP_COMP_TOL, (prec, lvl, ew, ec)
            # (ii) field
            pre, depth = f"mlps.{lvl}.", (4 if lvl < 2 else 8)
            if prec == "tc":
                M = nr * n
                idx = subset(M, lvl, cuda)
                b, k = torch.div(idx, n, rounding_mode="floor"), idx % n
                sub = {kk: v[b] for kk, v in batch.items() if kk != "_uniforms"}
                with torch.no_grad():
                    md_, mr_ = tpm.mip_tc_field(P, pre, depth, lvl < 2, sub, sub["radii"], torch.stack([td[b, k], td[b, k + 1]], -1))
                ed = tpm.sigma_error(dens.reshape(-1)[idx], md_[:, 0])
                er = (rgb.reshape(-1, 3)[idx].double() - mr_[:, 0]).abs().amax(-1)
                f = (*stats(er), *stats(ed))
                print(f"mip tc [{name}] level {lvl} (ii) field: {idx.numel()} of {M} points: rgb max {f[0]:.2e} mean {f[1]:.2e}, "
                      f"density (pre-activation units) max {f[2]:.2e} mean {f[3]:.2e}")
                assert f[0] <= tpm.MIP_RGB_TOL and f[1] <= tpm.MIP_RGB_MEAN_TOL, f
                assert f[2] <= tpm.MIP_SIGMA_TOL and f[3] <= tpm.MIP_SIGMA_MEAN_TOL, f
            elif far == 100.0:
                P32 = {kk: v.to(cuda) for kk, v in P.items()}
                with torch.no_grad():
                    mean, cov = mo.cast_cone(td, batch["rays_o"], batch["rays_d"], batch["radii"][:, None])
                    z, zc = mo.contract(mean, cov)
                    rd, rr = mo.mlp(P32, pre, mo.ipe_features(z, zc, P32[pre + "pos_basis_t"]), batch["viewdirs"], depth, lvl < 2)
                for what, got, ref in (("density", dens, rd), ("rgb", rgb, rr)):
                    diff = (got - ref).abs()
                    print(f"mip fp32 [{name}] level {lvl} (ii) {what} vs mip_oracle.mlp (fp32): max {float(diff.max()):.1e}, "
                          f"{100 * float((diff > 2e-4).float().mean()):.3f} % > 2e-4")
                    assert float(diff.max()) < 5e-3 and float((diff > 2e-4).float().mean()) <= 0.01, (lvl, what)


# ---------------- GridEncoder dense part ----------------

def encoder_poses(nv):
    """The synthetic source cameras, with view 0 replaced by the identity pose (the grid's z = 0 plane lies on z_cam = 0, every other
    cell is behind the camera) and view 1 by the identity moved to (0, 0, 0.5) (half the grid in front); lookups of the synthetic
    cameras fall both inside and far outside the latent."""
    poses = synth.make_scene((36, 22), nv, (4, 4), 0)["src_poses"].clone()
    poses[0] = torch.eye(4)
    if nv > 1:
        poses[1] = torch.eye(4)
        poses[1, 2, 3] = 0.5
    return poses


def seeded_pillars(nv, G, per, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for v in range(nv):
        for a in range(3):
            fixed = [(0, 0), (0, G - 1), (G - 1, 0), (G - 1, G - 1), (0, int(torch.randint(G, (1,), generator=g))),
                     (int(torch.randint(G, (1,), generator=g)), G - 1)]
            pq = fixed + [tuple(torch.randint(G, (2,), generator=g).tolist()) for _ in range(per - len(fixed))]
            out += [(v, a, p, q) for p, q in pq]
    return torch.tensor(out)


@pytest.mark.parametrize("nv,lat_hw", [(1, (11, 18)), (3, (19, 12)), (8, (11, 18))])
def test_grid_encoder_dense_matches_model(cuda, nv, lat_hw):
    """`dense_cuda` on a seeded nonnegative latent of ResNet magnitude (the ResNet bypassed), odd latent sizes, cameras with cells
    behind them, on z_cam = 0 and projecting outside the image, against tc_paths_model.encoder_tc_dense at 64 seeded pillars per view
    and axis (corners and other border pillars included).  Pillars with a cell whose mask or projection is ill-conditioned in fp32
    (|z_cam - 1e-3| < 1e-5, or |z_cam| < 1e-4 with a lookup near the image) are left out and counted.  Bounds, relative to the case's
    largest |pillar sum|: per element ENC_TOL, mean ENC_MEAN_TOL."""
    from neo360_b200.encoder import GridEncoder
    torch.manual_seed(3)
    enc = GridEncoder().eval().to(cuda)
    lh, lw = lat_hw
    W, H = 2 * lw, 2 * lh
    latent = (torch.rand(nv, 512, lh, lw, generator=torch.Generator().manual_seed(nv)) ** 2 * 2).to(cuda)
    poses = encoder_poses(nv).to(cuda)
    focal, c = torch.full((nv,), 0.8 * W, device=cuda), torch.tensor([[W / 2.0, H / 2.0]] * nv, device=cuda)
    with torch.no_grad():
        xz, xy, yz = enc.dense_cuda(latent, poses, focal, c, W, H)
    torch.cuda.synchronize()
    planes = {0: yz, 1: xz, 2: xy}
    pil = seeded_pillars(nv, 64, 64, nv)
    _, cam, _, uv = tpm.encoder_geometry(pil, 64, poses.double(), float(focal[0]), c[0].cpu().double(), W, H, (lh, lw))
    z = cam[..., 2]
    ill = ((z - 1e-3).abs() < 1e-5) | ((z.abs() < 1e-4) & (uv.abs().amax(-1) < 1e3))
    keep = ~ill.any(-1).cpu()
    cover = {"behind": int((z >= 1e-3).sum()), "on z_cam = 0": int((z == 0).sum()), "outside": int((uv.abs().amax(-1) > 1).sum()),
             "inside": int((uv.abs().amax(-1) < 1).sum())}
    pil = pil[keep]
    with torch.no_grad():
        model = tpm.encoder_tc_dense(enc, latent, poses, focal, c, W, H, pil)
    got = torch.stack([planes[a][v, :, p, q] for v, a, p, q in pil.tolist()]).double()
    scale = float(model.abs().max())
    e = (got - model).abs() / scale
    print(f"encoder nv={nv} latent {lh}x{lw}: {pil.shape[0]} pillars ({int((~keep).sum())} left out), cells {cover}: "
          f"max {float(e.max()):.2e} mean {float(e.mean()):.2e} of scale {scale:.3f}")
    assert all(v > 0 for v in cover.values()), cover
    assert float(e.max()) <= tpm.ENC_TOL and float(e.mean()) <= tpm.ENC_MEAN_TOL
