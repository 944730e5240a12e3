"""GPU: the hand-written CUDA of the NeO-360 training step against float64 restatements of the same operations
(oracle/train_stage_model.py, pinned to autograd through the oracle on the CPU by tests/test_train_stage_model.py).

* compositing, forward `neo_volumetric_rendering` and backward `neo_volumetric_rendering_bwd`: fg and bg, white and black,
  N in {1, 2, 31, 32, 33, 64, 65, 129, 193, 257} (one and several 32-sample blocks of the forward's warp scan), n in {1, 127, 128, 129, 4096}
  (one and several 128-ray blocks of the backward); every ray batch mixes the sigma * delta regimes: transparent, realistic (t from the
  library's own samplers at 129 / 193), one opaque sample (sigma delta in {17, 18, 30, 1e3}), runs of >= 5 opaque samples (T underflows),
  all-zero sigma, duplicate t, an opaque first / last sample and a tiny sigma on the bg 1e10 interval (a large d sigma).  Each upstream
  gradient alone with the others NULL, then all together.
  Bounds: forward |got - model| <= COMP_FWD_K 2^-24 N (depth relative to max |t|); backward |got - model| <= COMP_BWD_K 2^-24 N
  (magnitude + 2^-126 (max |G| + |g_lam|) / a) + the rounding of a subnormal output (2^-149): fp32 products below the normal range
  are held absolutely.
* lookups: raw maps (`neo_index_grid|local`, `neo_index_grid_bwd|local_bwd`, C 128 / 512) at nv 1 / 3; projected maps (`neo_index_maps`,
  `neo_index_maps_bwd`) at nv 1 / 3 / 8 and C in {4, 124, 128, 132, 252, 256, 260, 512} (one and two trips of the float4 loop in both
  thread-count branches).  Points: the level-1 points (fg and the bg `pts_lin`, up to 3 units along the ray) of the per-rank batch of
  the 640 x 480 training scene at 8 GPUs (512 rays) and at 1 GPU (4096 rays); 10^5 points inside one texel; an exact-geometry scene
  (signed-permutation cameras, map sides 2^k + 1) with points on texel centres, on gx = +-1, one ulp inside and outside, and beyond.
  Gradient maps start from a sentinel pattern: where the model's taps reach, the result is sentinel + scatter within
  LOOK_K 2^-24 (n_t + 1)(sum |w g| + |sentinel|) + sum |g| (|dix| + |diy|); everywhere else it is bit-identical to the sentinel.
  Forward rows within LOOK_K 2^-24 n sum |w F| + the coordinate term.
  Rows with |z_cam| < TAU are ill-conditioned for the pixel-aligned projection: their points are left out of the element-wise check and
  held instead to two identities on the kernel's own taps: <fwd(F), G> = <F, bwd(G)> per channel, and the backward's mass per channel =
  sum_rows coverage g (coverage = forward of an all-ones map), both within ADJ_K 2^-24 (rows + 4) of the absolute sums.
* one case of each through `training._Composite`, `_Lookup` and `_LookupMaps` (the NCHW / channel-last wrappers).

Bounds are 2-3x the largest values measured on an H100 80GB HBM3 at a 400 W power limit (DESIGN.md section 2).  Run with `-m gpu -s` to
see every case's max and mean.
"""
import functools
import math

import pytest
import torch

from neo360_b200 import synth
from oracle import neo360_oracle as orc
from oracle import train_stage_model as tsm

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
DENORM = 2.0 ** -126      # below fp32's normal range products are held absolutely (2^-149 = 2^-24 2^-125)
OUT_ROUND = 2.0 ** -149   # absolute rounding of a backward output in fp32's subnormal range
COMP_FWD_K = 5.0          # measured 1.79
COMP_BWD_K = 10.0         # measured 4.03 (at N = 1), mean 0.018
LOOK_K = 1.2              # measured 0.469
ADJ_K = 0.3               # measured 0.113
TAU = 1e-4

COMP_N = [1, 2, 31, 32, 33, 64, 65, 129, 193, 257]
COMP_RAYS = [1, 127, 128, 129, 4096]
MAP_C = [4, 124, 128, 132, 252, 256, 260, 512]
IMG_WH, PLANE_HW, LAT_HW = (640, 480), (120, 160), (240, 320)


@pytest.fixture(scope="module")
def cuda():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()
    return torch.device("cuda:0")


def lib():
    from neo360_b200 import _lib as L
    return L.load()


def call(name, *args):
    from neo360_b200 import _lib as L
    L.check(getattr(lib(), name)(*args, torch.cuda.current_stream().cuda_stream))


def P(t):
    from neo360_b200 import _lib as L
    return L.ptr(t)


def report(label, ratio):
    r = ratio.reshape(-1)
    mx, mean = (float(r.max()), float(r.mean())) if r.numel() else (0.0, 0.0)
    print(f"{label}: max {mx:.3g}  mean {mean:.3g}")
    return mx


# ---------------------------------------------------------------- compositing

@functools.lru_cache(maxsize=8)
def _view_rays(view):
    ro, vd, rd, _ = orc.rays_from_pose(orc.ray_directions(IMG_WH[1], IMG_WH[0], 0.8 * IMG_WH[0]), synth.target_pose(view, 100)[:3, :4])
    return ro, rd


def frame_rays(n, seed, dev):
    g = torch.Generator().manual_seed(seed)
    ro, rd = _view_rays(seed % 7)
    idx = torch.randint(0, ro.shape[0], (n,), generator=g)
    return ro[idx].contiguous().to(dev), rd[idx].contiguous().to(dev)


def sampled_t(o, d, far, N, in_sphere, g):
    """t / s of the library's own samplers: stratified (129) and, for 193, inverse-CDF on realistic level-0 weights."""
    from neo360_b200 import ops
    n = o.shape[0]
    near = torch.full_like(far, 1e-4)
    u0 = torch.rand(n, 129, generator=g, device=o.device)
    t0 = ops.sample_along_rays(o, d, 128, near, far, True, False, in_sphere, 3.0, u_rand=u0)[0]
    if N == 129:
        return t0
    w0 = torch.rand(n, 129, generator=g, device=o.device) ** 4
    u1 = torch.rand(n, 64, generator=g, device=o.device)
    return ops.sample_pdf(t0, w0, o, d, 64, True, in_sphere, far, 3.0, u_rand=u1)[0]


def comp_inputs(n, N, in_sphere, seed, dev):
    from neo360_b200 import ops
    g = torch.Generator(device=dev).manual_seed(seed)
    o, d = frame_rays(n, seed, dev)
    far = ops.intersect_sphere(o, d)
    if N in (129, 193):
        t = sampled_t(o, d, far, N, in_sphere, g)
    else:
        t = torch.sort(torch.rand(n, N, generator=g, device=dev), -1, descending=not in_sphere)[0]
        if in_sphere:
            t = 1e-4 + t * (far - 1e-4)
    reg = (torch.arange(n, device=dev) + seed) % 8
    t = t.clone()
    dup = reg == 5                                   # duplicate t: every third sample repeats its predecessor (delta = 0)
    if N > 1:
        j = torch.arange(1, N, 3, device=dev)
        t[dup.nonzero()[:, 0][:, None], j[None]] = t[dup.nonzero()[:, 0][:, None], (j - 1)[None]]
    t64 = t.double()
    if in_sphere:
        dist = torch.cat([t64[:, 1:], far.double()], 1) - t64
        dist = dist * d.double().norm(dim=-1, keepdim=True)
    else:
        dist = torch.cat([t64[:, :-1] - t64[:, 1:], torch.full_like(t64[:, :1], 1e10)], 1)
    sig = torch.nn.functional.softplus(torch.randn(n, N, generator=g, device=dev, dtype=torch.float64) * 2 - 1)
    sig[reg == 0] *= 1e-3                                                            # transparent
    sig[reg == 4] = 0.0                                                              # all-zero sigma
    vals = torch.tensor([17.0, 18.0, 30.0, 1e3], device=dev, dtype=torch.float64)
    k1 = torch.randint(0, N, (n,), generator=g, device=dev)
    rows = torch.arange(n, device=dev)
    ok = dist > 1e-6

    def opaque(mask, col, v):
        m = mask & ok[rows, col]
        sig[rows[m], col[m]] = (v / dist[rows, col])[m]

    opaque(reg == 2, k1, vals[rows % 4])                                             # one opaque sample
    opaque(reg == 7, torch.zeros_like(k1), vals[rows % 4])                           # opaque first sample
    if in_sphere:
        opaque(reg == 6, torch.full_like(k1, N - 1), vals[rows % 4])                 # opaque last sample
    else:
        sig[reg == 6, N - 1] = 1e-12                                                 # tiny sigma on the 1e10 interval
    if N >= 6:                                                                       # runs of 5..8 opaque samples
        k0 = torch.randint(0, max(1, N - 8), (n,), generator=g, device=dev)
        for r in range(8):
            col = (k0 + r).clamp(max=N - 1)
            opaque((reg == 3) & (r < 5 + rows % 4), col, 18.0 + 3 * r)
    rgb = torch.rand(n, N, 3, generator=g, device=dev)
    ups = {"g_comp": torch.randn(n, 3, generator=g, device=dev), "g_acc": torch.randn(n, generator=g, device=dev),
           "g_w": torch.randn(n, N, generator=g, device=dev), "g_lam": torch.randn(n, generator=g, device=dev),
           "g_depth": torch.randn(n, generator=g, device=dev)}
    return rgb.contiguous(), sig.float().contiguous(), t.contiguous(), d.contiguous(), far.reshape(-1).contiguous(), ups


def comp_fwd_kernel(rgb, sig, t, d, far, white, in_sphere):
    n, N = t.shape
    dev = t.device
    out = dict(comp=torch.empty(n, 3, device=dev), acc=torch.empty(n, device=dev), w=torch.empty(n, N, device=dev),
               lam=torch.empty(n, device=dev) if in_sphere else None, depth=torch.empty(n, device=dev))
    call("neo_volumetric_rendering", P(rgb), P(sig), P(t), P(d), P(far), n, N, int(white), int(in_sphere), P(out["comp"]), P(out["acc"]),
         P(out["w"]), P(out["lam"]), P(out["depth"]))
    return out


def comp_bwd_kernel(rgb, sig, t, d, far, white, in_sphere, gs):
    n, N = t.shape
    d_rgb = torch.full((n, N, 3), float("nan"), device=t.device)
    d_sig = torch.full((n, N), float("nan"), device=t.device)
    call("neo_volumetric_rendering_bwd", P(rgb), P(sig), P(t), P(d), P(far), n, N, int(white), int(in_sphere),
         *[P(gs.get(k)) for k in ("g_comp", "g_acc", "g_w", "g_lam", "g_depth")], P(d_rgb), P(d_sig))
    return d_rgb, d_sig


def comp_fwd_ratio(got, m, t, N, in_sphere):
    tmax = t.double().abs().amax(1).clamp_min(1e-30)
    errs = [(got["comp"].double() - m["comp"]).abs().amax(1), (got["acc"].double() - m["acc"]).abs(),
            (got["w"].double() - m["w"]).abs().amax(1), (got["depth"].double() - m["depth"]).abs() / tmax]
    if in_sphere:
        errs.append((got["lam"].double() - m["lam"]).abs())
    return torch.stack(errs, 1).amax(1) / (U * N)


def comp_bwd_ratio(d_rgb, d_sig, m, gs, N):
    """|got - model| in units of 2^-24 N (magnitude + subnormal floor), after the absolute rounding of a subnormal fp32 output:
    d_sigma = (dalpha dist) e is two roundings (<= 2^-150 each, the first scaled by e < 1), d_rgb = (alpha T) g_comp rounds w and then
    the product (<= 2^-150 (|g_comp| + 1))."""
    gmax = (m["G_mag"].amax(1) + m["g_lam_abs"])[:, None]
    floor_s = DENORM * gmax / m["a"] * m["dist"] * m["e"]
    es = ((d_sig.double() - m["d_sigma"]).abs() - OUT_ROUND).clamp_min(0)
    rs = es / (U * N * (m["d_sigma_mag"] + floor_s)).clamp_min(1e-300)
    gc = gs["g_comp"].double().abs()[:, None, :] if "g_comp" in gs else torch.zeros_like(m["d_rgb"])
    er = ((d_rgb.double() - m["d_rgb"]).abs() - OUT_ROUND / 2 * (gc + 1)).clamp_min(0)
    rr = er / (U * N * (m["d_rgb_mag"] + DENORM * gc)).clamp_min(1e-300)
    rs = torch.where(torch.isnan(d_sig), torch.full_like(rs, float("inf")), rs)
    rr = torch.where(torch.isnan(d_rgb), torch.full_like(rr, float("inf")), rr)
    return torch.cat([rs.reshape(-1), rr.reshape(-1)])


@pytest.mark.parametrize("white", [True, False], ids=["white", "black"])
@pytest.mark.parametrize("in_sphere", [True, False], ids=["fg", "bg"])
def test_composite_forward_backward_vs_float64(cuda, in_sphere, white):
    names = [k for k in ("g_comp", "g_acc", "g_w", "g_lam", "g_depth") if in_sphere or k != "g_lam"]
    worst_f, worst_b, means_f, means_b, where_b = 0.0, 0.0, [], [], None
    for N in COMP_N:
        for n in COMP_RAYS:
            rgb, sig, t, d, far, ups = comp_inputs(n, N, in_sphere, 1000 * N + n + 7 * in_sphere + 3 * white, cuda)
            got = comp_fwd_kernel(rgb, sig, t, d, far, white, in_sphere)
            rf = comp_fwd_ratio(got, tsm.composite_fwd(rgb, sig, t, d, far, white, in_sphere), t, N, in_sphere)
            worst_f = max(worst_f, float(rf.max()))
            means_f.append(float(rf.mean()))
            for use in [[k] for k in names] + [names]:
                gs = {k: ups[k] for k in use}
                d_rgb, d_sig = comp_bwd_kernel(rgb, sig, t, d, far, white, in_sphere, gs)
                m = tsm.composite_bwd(rgb, sig, t, d, far, white, in_sphere, **gs)
                rb = comp_bwd_ratio(d_rgb, d_sig, m, gs, N)
                if float(rb.max()) > worst_b:
                    worst_b, where_b = float(rb.max()), (N, n, use)
                means_b.append(float(rb.mean()))
    tag = f"composite {'fg' if in_sphere else 'bg'} {'white' if white else 'black'}"
    print(f"{tag} forward: max {worst_f:.3g} mean {sum(means_f) / len(means_f):.3g} x 2^-24 N (bound {COMP_FWD_K})")
    print(f"{tag} backward: max {worst_b:.3g} at (N, n, upstream) {where_b}, mean {sum(means_b) / len(means_b):.3g} x 2^-24 N magnitude "
          f"(bound {COMP_BWD_K})")
    assert worst_f <= COMP_FWD_K and worst_b <= COMP_BWD_K, (worst_f, worst_b, where_b)


def test_composite_autograd_wrapper(cuda):
    """training._Composite: the same kernels behind autograd, every output used, fg and bg."""
    from neo360_b200.training import _Composite
    for in_sphere in (True, False):
        rgb, sig, t, d, far, ups = comp_inputs(129, 65, in_sphere, 5, cuda)
        r, s = rgb.clone().requires_grad_(True), sig[..., None].clone().requires_grad_(True)
        comp, acc, w, lam, depth = _Composite.apply(r, s, t, d, far[:, None], True, in_sphere)
        loss = (comp * ups["g_comp"]).sum() + (acc * ups["g_acc"]).sum() + (w * ups["g_w"]).sum() + (depth * ups["g_depth"]).sum()
        if in_sphere:
            loss = loss + (lam[:, 0] * ups["g_lam"]).sum()
        loss.backward()
        gs = {k: v for k, v in ups.items() if in_sphere or k != "g_lam"}
        m = tsm.composite_bwd(rgb, sig, t, d, far, True, in_sphere, **gs)
        rb = comp_bwd_ratio(r.grad, s.grad[..., 0], m, gs, 65)
        assert report(f"_Composite {'fg' if in_sphere else 'bg'}", rb) <= COMP_BWD_K


# ---------------------------------------------------------------- lookups

def training_poses(nv):
    return torch.stack([synth.look_at_pose(360.0 * v / nv + 10.0, 0.3, 0.8) for v in range(nv)])


def perm_poses(nv):
    """Signed axis permutations (to_camera is exact), centred at the origin."""
    perms = [(0, 1, 2), (1, 2, 0), (2, 0, 1), (0, 2, 1), (2, 1, 0), (1, 0, 2), (0, 1, 2), (2, 0, 1)]
    signs = [(1, 1, 1), (1, -1, 1), (-1, 1, 1), (1, 1, -1), (-1, -1, 1), (1, -1, -1), (-1, -1, -1), (-1, 1, -1)]
    out = []
    for v in range(nv):
        m = torch.eye(4)
        m[:3, :3] = 0
        for r in range(3):
            m[r, perms[v][r]] = signs[v][r]
        out.append(m)
    return torch.stack(out)


class Geo:
    """A scene handle with the given cameras and map sizes (fp32 raw maps attached when `raw` is given)."""

    def __init__(self, poses, plane_hw, lat_hw, img_wh, dev, raw=None):
        from neo360_b200 import NeRF_TP
        nv = poses.shape[0]
        self.nv, self.poses, self.plane_hw, self.lat_hw, self.img_wh = nv, poses.to(dev), plane_hw, lat_hw, img_wh
        self.focal, self.cx, self.cy = 0.8 * img_wh[0], img_wh[0] / 2.0, img_wh[1] / 2.0
        self.net = NeRF_TP(num_coarse_samples=8, num_fine_samples=4, num_src_views=nv, precision="fp32")
        self.net.load_state_dict(synth.make_mlp_params(0))
        self.net = self.net.to(dev)
        if raw is None:
            pl = [torch.empty(nv, 128, *plane_hw, device=dev) for _ in range(3)]
            lat = torch.empty(nv, 512, *lat_hw, device=dev)
        else:
            pl, lat = raw[:3], raw[3]
        self.net.set_scene(*pl, lat, poses.to(dev), torch.full((nv,), self.focal, device=dev),
                           torch.tensor([[self.cx, self.cy]] * nv, device=dev), img_wh, precisions=["fp32"] if raw is not None else [])
        self.h = self.net._scene.handle

    def taps(self, pts, local):
        return tsm.lookup_taps(pts, self.poses, self.plane_hw, self.lat_hw, self.focal, self.cx, self.cy, self.img_wh, local)


def level1_points(n_rays, seed, dev):
    """Level-1 points of a training batch: fg points and the bg `pts_lin` lookup points (M,3)."""
    from neo360_b200 import ops
    g = torch.Generator(device=dev).manual_seed(seed)
    o, d = frame_rays(n_rays, seed, dev)
    far = ops.intersect_sphere(o, d)
    fg = sampled_t(o, d, far, 193, True, g)
    near = torch.full_like(far, 1e-4)
    t0, _, _ = ops.sample_along_rays(o, d, 128, near, far, True, False, False, 3.0, u_rand=torch.rand(n_rays, 129, generator=g, device=dev))
    w0 = torch.rand(n_rays, 129, generator=g, device=dev) ** 4
    _, _, lin = ops.sample_pdf(t0, w0, o, d, 64, True, False, far, 3.0, u_rand=torch.rand(n_rays, 64, generator=g, device=dev))
    fg_pts = o[:, None, :] + fg[..., None] * d[:, None, :]
    return torch.cat([fg_pts.reshape(-1, 3), lin.reshape(-1, 3)]).contiguous()


def contention_points(dev, n=100_000):
    g = torch.Generator(device=dev).manual_seed(17)
    base = torch.tensor([0.1234, -0.0567, 0.2101], device=dev)
    return (base + (torch.rand(n, 3, generator=g, device=dev) - 0.5) * 2e-4).contiguous()


def edge_points(geo, dev):
    """Camera-frame coordinates of view 0 from {texel centres of the 2^k + 1 sides, +-1, one ulp inside / outside, beyond}, mapped
    back to the world with the exact signed permutation."""
    vals = [k / 16 - 1 for k in range(33)] + [1 - 2 ** -24, 1 + 2 ** -23, -1 + 2 ** -24, -1 - 2 ** -23, 1.5, -1.5, 3.0, 1 / 32 - 1]
    v = torch.tensor(vals, dtype=torch.float32)
    g = torch.Generator().manual_seed(23)
    c = v[torch.randint(0, len(vals), (6000, 3), generator=g)]
    R = geo.poses[0, :3, :3].cpu()
    return (c @ R.T).contiguous().to(dev)


def split_near(geo, pts):
    z = geo.taps(pts, True)[0]["z"].reshape(geo.nv, -1)
    near = (z.abs() < TAU).any(0)
    return pts[~near].contiguous(), pts[near].contiguous()


def rows_of(t, nv):
    return t.reshape(nv, -1, t.shape[-1])


def sentinel(shape, dev):
    k = torch.arange(math.prod(shape), device=dev, dtype=torch.float32).reshape(shape)
    return ((k % 7) - 3.0) * 0.25 + 0.125


def check_scatter(label, got, sent, tp, G, nv, chunk):
    b = tsm.lookup_bwd(tp, G, nv, chunk_elems=chunk)
    want = sent.double() + b["val"]
    err = (got.double() - want).abs()
    unit = U * (b["n"][..., None] + 1) * (b["mag"] + sent.double().abs())
    reach = b["reach"]
    ratio = ((err - b["derr"]).clamp_min(0) / unit.clamp_min(1e-300))[reach]
    untouched_ok = bool((got[~reach] == sent[~reach]).all())
    mx = report(f"{label} (texels reached {int(reach.sum())}, max n_t {int(b['n'].max())})", ratio)
    assert untouched_ok, f"{label}: texels no row reaches changed"
    assert mx <= LOOK_K, (label, mx)
    return mx


def check_rows(label, got, f, n_terms):
    err = (got.double() - f["val"]).abs()
    ratio = (err - f["derr"]).clamp_min(0) / (U * n_terms * f["mag"]).clamp_min(1e-300)
    mx = report(label, ratio)
    assert mx <= LOOK_K, (label, mx)


def maps_fwd(geo, pts, C, lat, pl):
    M = pts.shape[0]
    ol = torch.empty(geo.nv * M, C, device=pts.device) if lat is not None else None
    ow = torch.empty(geo.nv * M, C, device=pts.device) if pl is not None else None
    call("neo_index_maps", geo.h, P(pts), M, C, P(lat), *(P(x) for x in (pl or [None] * 3)), P(ol), P(ow))
    return ol, ow


def maps_bwd(geo, pts, C, gl, gw, glat, gpl):
    call("neo_index_maps_bwd", geo.h, P(pts), pts.shape[0], C, P(gl), P(gw), P(glat), *(P(x) for x in (gpl or [None] * 3)))


def check_identities(label, geo, pts, C, dev):
    """Rows near z_cam = 0: adjointness and mass conservation of the pixel-aligned lookup, on the kernel's own taps."""
    if pts.shape[0] == 0:
        return
    g = torch.Generator(device=dev).manual_seed(C)
    Hl, Wl = geo.lat_hw
    F = torch.randn(geo.nv, Hl, Wl, C, generator=g, device=dev)
    R = geo.nv * pts.shape[0]
    G = torch.randn(R, C, generator=g, device=dev)
    out, _ = maps_fwd(geo, pts, C, F, None)
    outa, _ = maps_fwd(geo, pts, C, F.abs().contiguous(), None)
    cov, _ = maps_fwd(geo, pts, C, torch.ones_like(F), None)
    gm = torch.zeros_like(F)
    maps_bwd(geo, pts, C, G, None, gm, None)
    lhs = (out.double() * G.double()).sum(0)
    rhs = (F.double() * gm.double()).reshape(-1, C).sum(0)
    scale = (outa.double() * G.double().abs()).sum(0)
    mass = gm.double().reshape(-1, C).sum(0)
    want = (cov.double() * G.double()).sum(0)
    mscale = (cov.double() * G.double().abs()).sum(0)
    r1 = (lhs - rhs).abs() / (U * (R + 4) * scale).clamp_min(1e-300)
    r2 = (mass - want).abs() / (U * (R + 4) * mscale).clamp_min(1e-300)
    mx = max(report(f"{label} near-z rows ({R}): <fwd F, G> - <F, bwd G>", r1), report(f"{label} near-z rows: backward mass", r2))
    assert mx <= ADJ_K, (label, mx)


def run_projected(label, geo, pts, C, dev, chunk=1 << 26):
    """neo_index_maps(_bwd) on random projected maps of C channels against the model; world rows at every point, local rows at the
    points away from z_cam = 0 (the others through check_identities)."""
    g = torch.Generator(device=dev).manual_seed(C + 7 * geo.nv)
    nv, (Hp, Wp), (Hl, Wl) = geo.nv, geo.plane_hw, geo.lat_hw
    lat = torch.randn(nv, Hl, Wl, C, generator=g, device=dev)
    pl = [torch.randn(nv, Hp, Wp, C, generator=g, device=dev) for _ in range(3)]
    reg, near = split_near(geo, pts)
    step = 1 if pts.shape[0] <= 300_000 else 8         # large batches: the forward (row-independent) on every 8th point
    pf, rf = pts[::step].contiguous(), reg[::step].contiguous()
    _, ow = maps_fwd(geo, pf, C, None, pl)
    check_rows(f"{label} world fwd", ow, tsm.lookup_fwd(geo.taps(pf, False), pl, nv, chunk), 12)
    del ow
    ol, _ = maps_fwd(geo, rf, C, lat, None)
    check_rows(f"{label} local fwd", ol, tsm.lookup_fwd(geo.taps(rf, True), [lat], nv, chunk), 4)
    del ol
    tw, tl = geo.taps(pts, False), geo.taps(reg, True)
    Gw = torch.randn(nv * pts.shape[0], C, generator=g, device=dev)
    gpl = [sentinel((nv, Hp, Wp, C), dev) for _ in range(3)]
    sp = [x.clone() for x in gpl]
    maps_bwd(geo, pts, C, None, Gw, None, gpl)
    for name, tp, got, s in zip(("xz", "xy", "yz"), tw, gpl, sp):
        check_scatter(f"{label} bwd {name}", got, s, tp, Gw, nv, chunk)
    del Gw, gpl, sp
    Gl = torch.randn(nv * reg.shape[0], C, generator=g, device=dev)
    glat = sentinel((nv, Hl, Wl, C), dev)
    sl = glat.clone()
    maps_bwd(geo, reg, C, Gl, None, glat, None)
    check_scatter(f"{label} bwd latent", glat, sl, tl[0], Gl, nv, chunk)
    check_identities(label, geo, near, C, dev)


@pytest.mark.parametrize("nv", [1, 3, 8])
def test_projected_lookups_vs_float64(cuda, nv):
    """Every C at nv 1 / 3 / 8 on a 64-ray slice of the training batch, on 10^5 points inside one texel and on the exact-geometry scene."""
    geo = Geo(training_poses(nv), PLANE_HW, LAT_HW, IMG_WH, cuda)
    pts = level1_points(64, 11, cuda)
    cont = contention_points(cuda)
    edge_geo = Geo(perm_poses(nv), (17, 33), (9, 17), (64, 32), cuda)
    epts = edge_points(edge_geo, cuda)
    for C in MAP_C:
        run_projected(f"maps nv={nv} C={C} train-64", geo, pts, C, cuda)
        run_projected(f"maps nv={nv} C={C} edge", edge_geo, epts, C, cuda)
        if C in (4, 256, 260):
            run_projected(f"maps nv={nv} C={C} contention", geo, cont, C, cuda)


@pytest.mark.parametrize("n_rays", [512, 4096], ids=["8gpu-batch", "1gpu-batch"])
def test_projected_lookups_training_batch(cuda, n_rays):
    """The training configuration: nv 3, C = 256 projected channels, every level-1 point of a per-rank batch."""
    geo = Geo(training_poses(3), PLANE_HW, LAT_HW, IMG_WH, cuda)
    run_projected(f"maps nv=3 C=256 batch {n_rays} rays", geo, level1_points(n_rays, 29, cuda), 256, cuda, chunk=1 << 28)


@pytest.mark.parametrize("nv", [1, 3])
def test_raw_lookups_vs_float64(cuda, nv):
    """neo_index_grid / neo_index_local and their backward on the scene's own raw maps (C 128 / 512), 8-GPU batch and contention."""
    g = torch.Generator(device=cuda).manual_seed(nv)
    (Hp, Wp), (Hl, Wl) = PLANE_HW, LAT_HW
    raw = [torch.randn(nv, 128, Hp, Wp, generator=g, device=cuda) for _ in range(3)] + [torch.randn(nv, 512, Hl, Wl, generator=g, device=cuda)]
    geo = Geo(training_poses(nv), PLANE_HW, LAT_HW, IMG_WH, cuda, raw=raw)
    cl = [x.permute(0, 2, 3, 1).contiguous() for x in raw]
    for label, pts in ((f"raw nv={nv} batch 512 rays", level1_points(512, 31, cuda)), (f"raw nv={nv} contention", contention_points(cuda))):
        reg, near = split_near(geo, pts)
        M, Mr = pts.shape[0], reg.shape[0]
        ow = torch.empty(nv * M, 128, device=cuda)
        call("neo_index_grid", geo.h, P(pts), M, P(ow))
        tw = geo.taps(pts, False)
        check_rows(f"{label} grid fwd", ow, tsm.lookup_fwd(tw, cl[:3], nv), 12)
        ol = torch.empty(nv * Mr, 512, device=cuda)
        call("neo_index_local", geo.h, P(reg), Mr, P(ol))
        tl = geo.taps(reg, True)
        check_rows(f"{label} local fwd", ol, tsm.lookup_fwd(tl, cl[3:], nv), 4)
        Gw = torch.randn(nv * M, 128, generator=g, device=cuda)
        gpl = [sentinel((nv, Hp, Wp, 128), cuda) for _ in range(3)]
        sp = [x.clone() for x in gpl]
        call("neo_index_grid_bwd", geo.h, P(pts), M, P(Gw), *[P(x) for x in gpl])
        for name, tp, got, s in zip(("xz", "xy", "yz"), tw, gpl, sp):
            check_scatter(f"{label} grid bwd {name}", got, s, tp, Gw, nv, 1 << 26)
        Gl = torch.randn(nv * Mr, 512, generator=g, device=cuda)
        glat = sentinel((nv, Hl, Wl, 512), cuda)
        sl = glat.clone()
        call("neo_index_local_bwd", geo.h, P(reg), Mr, P(Gl), P(glat))
        check_scatter(f"{label} local bwd", glat, sl, tl[0], Gl, nv, 1 << 26)


def test_lookup_autograd_wrappers(cuda):
    """training._Lookup (NCHW maps, raw) and training._LookupMaps (channel-last projected maps) against the model, forward and backward."""
    from neo360_b200.training import _Lookup, _LookupMaps
    nv = 3
    g = torch.Generator(device=cuda).manual_seed(41)
    (Hp, Wp), (Hl, Wl) = PLANE_HW, LAT_HW
    raw = [torch.randn(nv, 128, Hp, Wp, generator=g, device=cuda) for _ in range(3)] + [torch.randn(nv, 512, Hl, Wl, generator=g, device=cuda)]
    geo = Geo(training_poses(nv), PLANE_HW, LAT_HW, IMG_WH, cuda, raw=raw)
    reg, _ = split_near(geo, level1_points(16, 43, cuda))
    tw, tl = geo.taps(reg, False), geo.taps(reg, True)
    leaves = [x.clone().requires_grad_(True) for x in raw]
    world, local = _Lookup.apply(reg, *leaves, geo.net)
    cl = [x.permute(0, 2, 3, 1) for x in raw]
    check_rows("_Lookup world fwd", world, tsm.lookup_fwd(tw, cl[:3], nv), 12)
    check_rows("_Lookup local fwd", local, tsm.lookup_fwd(tl, cl[3:], nv), 4)
    Gw, Gl = torch.randn_like(world), torch.randn_like(local)
    ((world * Gw).sum() + (local * Gl).sum()).backward()
    zero = lambda x: torch.zeros(x.shape[0], x.shape[2], x.shape[3], x.shape[1], device=cuda)
    for name, tp, leaf in zip(("xz", "xy", "yz"), tw, leaves[:3]):
        check_scatter(f"_Lookup bwd {name}", leaf.grad.permute(0, 2, 3, 1), zero(leaf), tp, Gw, nv, 1 << 26)
    check_scatter("_Lookup bwd latent", leaves[3].grad.permute(0, 2, 3, 1), zero(leaves[3]), tl[0], Gl, nv, 1 << 26)
    C = 256
    geo2 = Geo(training_poses(nv), PLANE_HW, LAT_HW, IMG_WH, cuda)
    lat = torch.randn(nv, Hl, Wl, C, generator=g, device=cuda, requires_grad=True)
    pl = [torch.randn(nv, Hp, Wp, C, generator=g, device=cuda, requires_grad=True) for _ in range(3)]
    lp, wp = _LookupMaps.apply(reg, lat, *pl, geo2.net)
    check_rows("_LookupMaps local fwd", lp, tsm.lookup_fwd(tl, [lat.detach()], nv), 4)
    check_rows("_LookupMaps world fwd", wp, tsm.lookup_fwd(tw, [x.detach() for x in pl], nv), 12)
    Gl, Gw = torch.randn_like(lp), torch.randn_like(wp)
    ((lp * Gl).sum() + (wp * Gw).sum()).backward()
    check_scatter("_LookupMaps bwd latent", lat.grad, torch.zeros_like(lat), tl[0], Gl, nv, 1 << 26)
    for name, tp, leaf in zip(("xz", "xy", "yz"), tw, pl):
        check_scatter(f"_LookupMaps bwd {name}", leaf.grad, torch.zeros_like(leaf), tp, Gw, nv, 1 << 26)
