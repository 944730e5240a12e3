"""GPU: the projected-map blend of the NEO_PREC_TC field kernel (csrc/field_tc.cu, blend_maps) on tiles that mix points with no tap
of non-zero weight, with some and with all 16.

A thread blends the 16 taps (4 maps x 4 bilinear taps) of its two points, rows r0 and r0 + 8 of the tile, and skips those of zero
weight, so the lanes of a warp take different paths through the blend whenever their points differ in which taps are in range.
Random rays rarely put that mix inside one warp, so the rays and samples here are chosen for it: a single source camera with the
identity pose (camera frame = world frame), and per point the 16-bit mask of non-zero taps (bit 4 m + k: map m, tap k) computed in
float64 from the lookup point.  A 64-point tile is 32 consecutive rays x 2 samples; warp w holds sample w // 2 of rays
16 (w % 2) .. 16 (w % 2) + 15, and its lane quad q rays 16 (w % 2) + q and 16 (w % 2) + q + 8 (a thread's rows r0 and r0 + 8).
Among 16 chosen rays, ray k < 8 has 4 samples of category PAIRS[k][0] and ray k + 8 of PAIRS[k][1]; the call lines up 8 copies of
them, so every warp has the row pairs (0, 16), (16, 0), (some, 16), (16, some), (0, some), (some, 0) non-zero taps and two pairs
where one row has taps only in maps 0-1 and the other only in maps 2-3.  (The layout holds for any tile of 16 j rays.)  Copy c pairs
ray k with ray 8 + (k + c) % 8, and a permutation of the rays mixes all of them across tiles and lanes.

Checked, for every MLP: the kernel against oracle/tc_model.py at the bounds of test_gpu_tc_kernels.py, and that a permutation of the
rays (other tiles, other lanes) gives the same rows bit for bit.
"""
import pytest
import torch

from neo360_b200 import synth
from oracle import neo360_oracle as orc
from oracle import tc_model as tcm

pytestmark = pytest.mark.gpu

ZERO, FULL, SOME, LO, HI = "zero", "full", "some", "lo", "hi"
# categories of (row r0, row r0 + 8) of a warp's 8 lane quads
PAIRS = [(ZERO, FULL), (FULL, ZERO), (SOME, FULL), (FULL, SOME), (ZERO, SOME), (SOME, ZERO), (LO, HI), (HI, LO)]
MARGIN = 2e-3          # texels: a tap counts only if every grid coordinate is this far from a texel centre (fp32 vs float64)


@pytest.fixture(scope="module")
def cuda():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()
    return torch.device("cuda:0")


def scene():
    sc = synth.make_scene((37, 23), 1, (13, 17), 11)
    sc["src_poses"] = torch.eye(4)[None]
    d = lambda k: sc[k].to(torch.float64)
    W, H = sc["img_wh"]
    osc = orc.Scene(d("planes_xz"), d("planes_xy"), d("planes_yz"), d("latent"), d("src_poses"),
                    float(sc["src_focal"][0]), float(sc["src_c"][0, 0]), float(sc["src_c"][0, 1]), W, H)
    return sc, osc


def quad_mask(gx, gy, W, H):
    """tap_quad's non-zero taps {nw, ne, sw, se} as 4 bits, and the distance of (ix, iy) from the nearest texel centre."""
    ix, iy = (gx + 1) / 2 * (W - 1), (gy + 1) / 2 * (H - 1)
    inr = (ix >= -1) & (ix < W) & (iy >= -1) & (iy < H)
    x0, y0 = torch.floor(ix), torch.floor(iy)
    vx = [(x0 + a >= 0) & (x0 + a < W) for a in (0, 1)]
    vy = [(y0 + a >= 0) & (y0 + a < H) for a in (0, 1)]
    bits = torch.zeros_like(ix, dtype=torch.int64)
    for k in range(4):
        bits |= (inr & vx[k & 1] & vy[k >> 1]).long() << k
    margin = torch.minimum((ix - torch.round(ix)).abs(), (iy - torch.round(iy)).abs())
    return bits, margin


def tap_masks(p, osc):
    """16-bit tap masks (bit 4 m + k) of lookup points p (..., 3) in the camera frame = world frame, and their margin."""
    Hp, Wp = osc.planes_xz.shape[-2:]
    Hl, Wl = osc.latent.shape[-2:]
    gx, gy = tcm.latent_coords(p, osc)
    coords = [(gx, gy, Wl, Hl), (p[..., 0], p[..., 2], Wp, Hp), (p[..., 0], p[..., 1], Wp, Hp), (p[..., 1], p[..., 2], Wp, Hp)]
    mask = torch.zeros(p.shape[:-1], dtype=torch.int64)
    margin = torch.full(p.shape[:-1], float("inf"), dtype=torch.float64)
    for m, (a, b, W, H) in enumerate(coords):
        bits, mg = quad_mask(a, b, W, H)
        mask |= bits << (4 * m)
        margin = torch.minimum(margin, mg)
    margin = torch.where(p[..., 2].abs() < 0.05, torch.zeros_like(margin), margin)      # near the latent projection's pole
    return mask, margin


def category(mask):
    lo, hi = mask & 0xFF, mask >> 8
    return {ZERO: mask == 0, FULL: mask == 0xFFFF, SOME: (mask != 0) & (mask != 0xFFFF) & (lo != 0) & (hi != 0),
            LO: (lo != 0) & (hi == 0), HI: (lo == 0) & (hi != 0)}


def chosen_inputs(osc, bg, seed):
    """16 rays x 4 samples, every point of ray k in tap mask category PAIRS[k % 8][k // 8]: per ray a random origin and direction,
    then 4 t (fg) or s (bg) values from a fine grid whose lookup points have that category."""
    g = torch.Generator().manual_seed(seed)
    grid = torch.linspace(0.0, 3.0, 3001, dtype=torch.float64) if not bg else torch.linspace(0.0, 1.0, 2001, dtype=torch.float64)
    os_, ds, ts = [], [], []
    for k in range(16):
        want = PAIRS[k % 8][k // 8]
        for _ in range(1000):
            o = (torch.rand(3, generator=g, dtype=torch.float64) - 0.5) * 0.8
            d = torch.randn(3, generator=g, dtype=torch.float64)
            d = d / d.norm()
            far = orc.intersect_sphere(o[None].float(), d[None].float()).double()[0]
            tl = far * (1 - grid) + tcm.FAR_UNC * grid if bg else grid
            mask, margin = tap_masks(o + tl[:, None] * d, osc)
            idx = torch.nonzero(category(mask)[want] & (margin > MARGIN)).flatten()
            if idx.numel() >= 4:
                break
        else:
            raise AssertionError(f"no ray found for category {want}")
        os_.append(o)
        ds.append(d)
        ts.append(grid[idx[torch.randperm(idx.numel(), generator=g)[:4]]])
    o, d, t = torch.stack(os_).float(), torch.stack(ds).float(), torch.stack(ts).float()
    far = orc.intersect_sphere(o, d)
    return {"rays_o": o, "rays_d": d, "viewdirs": d}, far, t


def check_mix(rays, far, t, osc, bg):
    """The tile's tap masks, recomputed from the fp32 inputs in float64, have the intended mix in every warp."""
    o, d, t64 = rays["rays_o"].double(), rays["rays_d"].double(), t.double()
    tl = far.double().reshape(-1, 1) * (1 - t64) + tcm.FAR_UNC * t64 if bg else t64
    mask, margin = tap_masks(o[:, None, :] + tl[..., None] * d[:, None, :], osc)
    assert bool((margin > MARGIN / 2).all()), "a lookup point lies too close to a texel centre"
    cat = category(mask)
    for rl in range(16):
        for w in range(4):
            c = PAIRS[rl % 8][rl // 8]
            assert bool(cat[c][rl, w]), (rl, w, c, hex(int(mask[rl, w])))
    counts = [int(x) for x in torch.unique(torch.tensor([bin(int(x)).count("1") for x in mask.flatten()]))]
    assert 0 in counts and 16 in counts and any(0 < c < 16 for c in counts), counts
    return counts


@pytest.mark.parametrize("mlp_index", [0, 1, 2, 3])
def test_tc_field_mixed_taps(cuda, mlp_index):
    """Kernel vs float64 model on tiles that mix 0, some and 16 non-zero taps in every warp, and bit identity under a permutation
    of the rays.  Copy c < 8 of the 16 chosen rays (half a tile each) pairs ray k with ray 8 + (k + c) % 8, so that every category
    pair shares a thread somewhere."""
    from neo360_b200 import NeRF_TP
    sc, osc = scene()
    bg = bool(mlp_index & 1)
    rays, far, t = chosen_inputs(osc, bg, 100 + mlp_index)
    counts = check_mix(rays, far, t, osc, bg)
    order = torch.cat([torch.tensor(list(range(8)) + [8 + (k + c) % 8 for k in range(8)]) for c in range(8)])
    rays = {k: v[order] for k, v in rays.items()}
    far, t = far[order], t[order]
    P = synth.make_mlp_params(11)
    net = NeRF_TP(num_coarse_samples=8, num_fine_samples=4, num_src_views=1, precision="tc").eval()
    net.load_state_dict(P)
    net = net.to(cuda)
    net.set_scene(*[sc[k].to(cuda) for k in ("planes_xz", "planes_xy", "planes_yz", "latent", "src_poses", "src_focal", "src_c")],
                  sc["img_wh"], precisions=["tc"])
    osc_dev = orc.Scene(*[x.to(cuda) for x in (osc.planes_xz, osc.planes_xy, osc.planes_yz, osc.latent, osc.src_poses)],
                        osc.focal, osc.cx, osc.cy, osc.img_w, osc.img_h)
    rays = {k: v.to(cuda) for k, v in rays.items()}
    far, t = far.to(cuda), t.to(cuda)
    n = t.shape[0]
    with torch.no_grad():
        rgb, sig = net.field_eval(rays, far, t, mlp_index, precision="tc")
        perm = torch.randperm(n, generator=torch.Generator().manual_seed(mlp_index)).to(torch.int32).to(cuda)
        prgb, psig = net.field_eval(rays, far, t, mlp_index, precision="tc", ray_order=perm)
        net.check()
        mr, ms = tcm.tc_field(rays, far, t, mlp_index, osc_dev, P)
    er = (rgb.double() - mr).abs().amax(-1)
    es = ((sig.double() - ms).abs() / (1 + ms))[..., 0]
    print(f"tc field mixed taps mlp={mlp_index} (non-zero taps per point: {counts}): max rgb {float(er.max()):.2e} "
          f"sigma/(1+sigma) {float(es.max()):.2e}, mean rgb {float(er.mean()):.2e} sigma/(1+sigma) {float(es.mean()):.2e}")
    assert torch.isfinite(rgb).all() and torch.isfinite(sig).all()
    assert float(er.max()) <= tcm.RGB_TOL and float(es.max()) <= tcm.SIGMA_TOL
    assert float(er.mean()) <= tcm.RGB_MEAN_TOL and float(es.mean()) <= tcm.SIGMA_MEAN_TOL
    assert torch.equal(prgb, rgb) and torch.equal(psig, sig), "a ray permutation changed the output bits"
