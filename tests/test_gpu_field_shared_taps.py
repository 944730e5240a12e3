"""GPU: the projected-map blend of the NEO_PREC_TC field kernel (csrc/field_tc.cu, blend_maps) when a thread's two points share
texels.

A thread blends rows r0 and r0 + 8 of a tile: the same sample of rays 16 (w % 2) + q and 16 (w % 2) + q + 8 (warp w, lane quad q).
In the foreground kernel both rows' loads of a tap are in flight together, and when tap k of map m is the same texel for both rows
and both weights are non-zero (TapTable::share), the texel is fetched once and blended into both rows; the background kernel blends
one row's tap at a time and is checked on the same pairs.  The rays here are chosen per lane quad, with a single source camera of identity pose (camera frame = world
frame), so that every warp holds these row pairs, for both samples of the tile:
  same      every tap of every map shared;
  shift +x  the xz quad of row r0 + 8 is one texel right of row r0's (no tap shared in that map: the same texel is another tap);
  shift -x  one texel left;
  shift y   the xz quad one texel down;
  some      a pair shifted along world y: the xz quad shared, the xy and yz quads not;
  edge a    xz: row r0's nw tap out of range (weight 0, index 0), row r0 + 8's nw tap in range at texel 0;
  edge b    the same with the rows swapped.
The categories are checked in float64 from the fp32 inputs.  Checked, for every MLP: the kernel against oracle/tc_model.py at the
bounds of test_gpu_tc_kernels.py, and that a ray order that splits every row pair across threads (row r0's ray then shares a
thread with another pair's ray) gives the same rows bit for bit, so the shared and unshared paths compute the same sums.
"""
import pytest
import torch

from neo360_b200 import synth
from oracle import neo360_oracle as orc
from oracle import tc_model as tcm

pytestmark = pytest.mark.gpu

SAME, SHIFT_X, SHIFT_XN, SHIFT_Y, SOME, EDGE_A, EDGE_B = "same", "shift +x", "shift -x", "shift y", "some", "edge a", "edge b"
PAIRS = [SAME, SHIFT_X, SHIFT_XN, SHIFT_Y, SOME, EDGE_A, EDGE_B, SAME]       # lane quad q of every warp
COPIES = 4                                                                  # 16 rays each (8 pairs), 2 per tile
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


def quads(p, osc):
    """Per map m (latent, xz, xy, yz) of lookup points p (..., 3): tap_quad's base texel x0, y0 (..., 4), the in-range taps
    {nw, ne, sw, se} as bits 4 m + k (...), and the distance of the grid coordinates from the nearest texel centre."""
    Hp, Wp = osc.planes_xz.shape[-2:]
    Hl, Wl = osc.latent.shape[-2:]
    gx, gy = tcm.latent_coords(p, osc)
    coords = [(gx, gy, Wl, Hl), (p[..., 0], p[..., 2], Wp, Hp), (p[..., 0], p[..., 1], Wp, Hp), (p[..., 1], p[..., 2], Wp, Hp)]
    x0s, y0s = [], []
    bits = torch.zeros(p.shape[:-1], dtype=torch.int64)
    margin = torch.full(p.shape[:-1], float("inf"), dtype=torch.float64)
    for m, (a, b, W, H) in enumerate(coords):
        ix, iy = (a + 1) / 2 * (W - 1), (b + 1) / 2 * (H - 1)
        inr = (ix >= -1) & (ix < W) & (iy >= -1) & (iy < H)
        x0, y0 = torch.floor(ix), torch.floor(iy)
        vx = [(x0 + e >= 0) & (x0 + e < W) for e in (0, 1)]
        vy = [(y0 + e >= 0) & (y0 + e < H) for e in (0, 1)]
        for k in range(4):
            bits |= (inr & vx[k & 1] & vy[k >> 1]).long() << (4 * m + k)
        x0s.append(x0.long())
        y0s.append(y0.long())
        margin = torch.minimum(margin, torch.minimum((ix - torch.round(ix)).abs(), (iy - torch.round(iy)).abs()))
    margin = torch.where(p[..., 2].abs() < 0.05, torch.zeros_like(margin), margin)      # near the latent projection's pole
    return torch.stack(x0s, -1), torch.stack(y0s, -1), bits, margin


def share_mask(qa, qb):
    """TapTable::share of two points from their quads(): bit 4 m + k when tap k of map m is in range for both at the same texel."""
    same = (qa[0] == qb[0]) & (qa[1] == qb[1])                                    # (..., 4 maps)
    same16 = sum(same[..., m].long() * (0xF << (4 * m)) for m in range(4))
    return qa[2] & qb[2] & same16


def is_category(cat, qa, qb):
    """Row pair (a, b) has category cat, for every sample (qa, qb: quads() of the two rows)."""
    xa, ya, ba, _ = qa
    xb, yb, bb, _ = qb
    sh = share_mask(qa, qb)
    xz_full = ((ba >> 4) & 0xF == 0xF) & ((bb >> 4) & 0xF == 0xF)
    if cat == SAME:
        ok = sh == 0xFFFF
    elif cat in (SHIFT_X, SHIFT_XN, SHIFT_Y):
        dx, dy = {SHIFT_X: (1, 0), SHIFT_XN: (-1, 0), SHIFT_Y: (0, 1)}[cat]
        ok = xz_full & (xb[..., 1] == xa[..., 1] + dx) & (yb[..., 1] == ya[..., 1] + dy)
    elif cat == SOME:
        nib = lambda x, m: (x >> (4 * m)) & 0xF
        ok = (nib(sh, 1) == 0xF) & (nib(sh, 2) == 0) & (nib(ba & bb, 2) != 0) & (nib(sh, 3) == 0) & (nib(ba & bb, 3) != 0)
    else:                                                                          # edge: nw tap (k = 0) of the xz map
        (xo, yo, bo), (xi, yi, bi) = ((xa, ya, ba), (xb, yb, bb)) if cat == EDGE_A else ((xb, yb, bb), (xa, ya, ba))
        ok = (((bo >> 4) & 1) == 0) & (((bi >> 4) & 1) == 1) & (xi[..., 1] == 0) & (yi[..., 1] == 0) & (xo[..., 1] == -1)
    return bool(ok.all())


def lookup_points(o, d, far, t, bg):
    """Lookup points (n, N, 3), float64 from the fp32 inputs: the sample point (fg) or far (1 - s) + 3 s along the ray (bg)."""
    o, d, t64 = o.double(), d.double(), t.double()
    tl = far.double().reshape(-1, 1) * (1 - t64) + tcm.FAR_UNC * t64 if bg else t64
    return o[:, None, :] + tl[..., None] * d[:, None, :]


def make_pair(cat, osc, bg, g):
    """Rays a, b (origin, direction) and their 2 samples, with row pair (a, b) of category cat at both samples.  Ray b is ray a moved
    by delta; a sample sits at distance L along its ray from the origin (fg: t = L, bg: s with far (1 - s) + 3 s = L)."""
    Hp, Wp = osc.planes_xz.shape[-2:]
    tx, ty = 2.0 / (Wp - 1), 2.0 / (Hp - 1)                    # one plane texel in world x, and in world z (y of the xz map)
    u = lambda: float(torch.rand((), generator=g, dtype=torch.float64))
    for _ in range(20000):
        if cat in (EDGE_A, EDGE_B):
            ix, iy = -1 + 0.1 + 0.8 * u(), 0.1 + 0.8 * u()     # xz: x0 = -1, y0 = 0; one texel right, x0 = 0: nw tap = texel 0
            pa = torch.tensor([2 * ix / (Wp - 1) - 1, 1.6 * u() - 0.8, 2 * iy / (Hp - 1) - 1], dtype=torch.float64)
            delta = torch.tensor([tx, 0.0, 0.0], dtype=torch.float64)
            if cat == EDGE_B:                                   # row r0 in range at texel 0, row r0 + 8 one texel left
                pa, delta = pa + delta, -delta
        else:
            pa = (torch.rand(3, generator=g, dtype=torch.float64) * 2 - 1) * 0.9
            delta = {SAME: torch.randn(3, generator=g, dtype=torch.float64) * 1e-3 * tx, SHIFT_X: torch.tensor([tx, 0.0, 0.0]),
                     SHIFT_XN: torch.tensor([-tx, 0.0, 0.0]), SHIFT_Y: torch.tensor([0.0, 0.0, ty]),
                     SOME: torch.tensor([0.0, 2.0 / (osc.planes_xy.shape[-2] - 1), 0.0])}[cat].double()
        if bg and float(pa.norm()) < 1.05:                      # bg lookup points lie beyond the unit sphere
            continue
        o = torch.randn(3, generator=g, dtype=torch.float64)
        o = o / o.norm() * 0.4 * u()
        L0 = float((pa - o).norm())
        d = (pa - o) / L0
        L = torch.tensor([L0, L0 + 0.3 * tx * u()], dtype=torch.float64)
        rays = []
        for oo in (o, o + delta):
            o32, d32 = oo.float(), d.float()
            far = orc.intersect_sphere(o32[None], d32[None])[0]
            f = far.double()
            t = ((L - f) / (tcm.FAR_UNC - f) if bg else L).float()
            rays.append((o32, d32, far, t))
        if bg and not all(bool(((r[3] > 0) & (r[3] < 1)).all()) for r in rays):
            continue
        q = [quads(lookup_points(o32[None], d32[None], far, t[None], bg)[0], osc) for o32, d32, far, t in rays]
        if bool((q[0][3] > MARGIN).all()) and bool((q[1][3] > MARGIN).all()) and is_category(cat, q[0], q[1]):
            return rays
    raise AssertionError(f"no row pair found for category {cat}")


def chosen_inputs(osc, bg, seed):
    """COPIES x 16 rays: copy c is [a of pair 0..7, b of pair 0..7], pair q of category PAIRS[q], so that in every tile lane quad q
    of each warp blends pair q."""
    g = torch.Generator().manual_seed(seed)
    os_, ds, fars, ts = [], [], [], []
    for _ in range(COPIES):
        pairs = [make_pair(cat, osc, bg, g) for cat in PAIRS]
        for side in (0, 1):
            for p in pairs:
                o, d, far, t = p[side]
                os_.append(o); ds.append(d); fars.append(far); ts.append(t)
    o, d = torch.stack(os_), torch.stack(ds)
    return {"rays_o": o, "rays_d": d, "viewdirs": d}, torch.stack(fars), torch.stack(ts)


def shared_taps(rays, far, t, osc, bg, order):
    """Taps of non-zero weight, and the shared ones, over the row pairs the kernel forms when it visits the rays in `order`."""
    q = quads(lookup_points(rays["rays_o"][order], rays["rays_d"][order], far[order], t[order], bg), osc)
    a = torch.arange(q[2].shape[0]).reshape(-1, 16)
    ra, rb = a[:, :8].flatten(), a[:, 8:].flatten()
    qa, qb = [x[ra] for x in q], [x[rb] for x in q]
    taps = sum(bin(int(x)).count("1") for x in q[2].flatten())
    shared = sum(bin(int(x)).count("1") for x in share_mask(qa, qb).flatten())
    return taps, shared


@pytest.mark.parametrize("mlp_index", [0, 1, 2, 3])
def test_tc_field_shared_taps(cuda, mlp_index):
    """Kernel vs float64 model on row pairs that share all, some or none of their texels, or meet at the edge of a map; and bit
    identity with a ray order that pairs every row with another pair's ray."""
    from neo360_b200 import NeRF_TP
    sc, osc = scene()
    bg = bool(mlp_index & 1)
    rays, far, t = chosen_inputs(osc, bg, 200 + mlp_index)
    n = t.shape[0]
    # slot 16 j + 8 + q takes ray b of pair (q + 1) % 8: every row pair of the natural order is split across threads
    split = torch.tensor([16 * j + (k if k < 8 else 8 + (k - 8 + 1) % 8) for j in range(n // 16) for k in range(16)])
    taps, shared = shared_taps(rays, far, t, osc, bg, torch.arange(n))
    _, shared_split = shared_taps(rays, far, t, osc, bg, split)
    assert shared > 0
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
    with torch.no_grad():
        rgb, sig = net.field_eval(rays, far, t, mlp_index, precision="tc")
        srgb, ssig = net.field_eval(rays, far, t, mlp_index, precision="tc", ray_order=split.to(torch.int32).to(cuda))
        net.check()
        mr, ms = tcm.tc_field(rays, far, t, mlp_index, osc_dev, P)
    er = (rgb.double() - mr).abs().amax(-1)
    es = ((sig.double() - ms).abs() / (1 + ms))[..., 0]
    print(f"tc field shared taps mlp={mlp_index}: {taps} taps, {shared} shared by a thread's rows ({shared_split} with the rows "
          f"split): max rgb {float(er.max()):.2e} sigma/(1+sigma) {float(es.max()):.2e}, mean rgb {float(er.mean()):.2e} "
          f"sigma/(1+sigma) {float(es.mean()):.2e}")
    assert torch.isfinite(rgb).all() and torch.isfinite(sig).all()
    assert float(er.max()) <= tcm.RGB_TOL and float(es.max()) <= tcm.SIGMA_TOL
    assert float(er.mean()) <= tcm.RGB_MEAN_TOL and float(es.mean()) <= tcm.SIGMA_MEAN_TOL
    assert torch.equal(srgb, rgb) and torch.equal(ssig, sig), "splitting the row pairs changed the output bits"
