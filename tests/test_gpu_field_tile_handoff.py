"""GPU: the hand-off of a tile's geometry from the producer warpgroup to a consumer of the NEO_PREC_TC field kernel
(csrc/field_tc.cu) when every consumer runs several tiles.

The producer builds tile T + 1's rows, the background's view-independent s columns (which travel with the rows) and its first
view's encodings and tap table while the consumer still works on tile T.  A tap table stores one texel index per (point, map), the
quad's nw tap, and the blend derives the other three taps from it; at a map's edge (x0 or y0 = -1) that index lies outside the map,
in a source view v > 0 inside the previous view's texels.  The cases here:
  * enough rays that every consumer warpgroup of the device runs at least three tiles, and a tile count that is not a multiple of
    the consumer count, so the last round leaves some consumers idle;
  * every source camera with the identity pose (camera frame = world frame), so the edge lookups of test_gpu_tc_kernels.py's edge
    scene (grid coordinates on, just inside and just outside the maps' edges) hit the map corners in every view;
  * those edge rays repeated through the ray order, so they land in consumers' later tiles.
Checked, for all four MLPs at NV = 1, 3 and 8: the full call bit for bit against each chunk evaluated on its own (most consumers
then run one tile or none) and against a permuted ray order; at NV = 3, the full call against oracle/tc_model.py at the bounds of
test_gpu_tc_kernels.py.
"""
import pytest
import torch

from neo360_b200 import synth
from oracle import neo360_oracle as orc
from oracle import tc_model as tcm

pytestmark = pytest.mark.gpu

TILE_RAYS, TILE_SAMPLES = 32, 2          # a tile: 32 consecutive slots of the ray order x 2 consecutive samples (field_tc.cu)
PLANE_HW = (13, 17)
CHUNK = 8 * TILE_RAYS                    # a chunk evaluated on its own has fewer tiles than a device has consumers
EDGE_EVERY = 200                         # a copy of the edge rays every this many rays


@pytest.fixture(scope="module")
def cuda():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()
    return torch.device("cuda:0")


def md(a, b):
    return float((a.detach().double() - b.detach().to(a.device).double()).abs().max()) if a.numel() else 0.0


def tc_net(cuda, nv, seed):
    """NeRF_TP with a NEO_PREC_TC scene whose nv source cameras all have the identity pose, and the same scene for the model."""
    from neo360_b200 import NeRF_TP
    sc = synth.make_scene((37, 23), nv, PLANE_HW, seed)
    sc["src_poses"] = torch.eye(4)[None].repeat(nv, 1, 1)
    P = synth.make_mlp_params(seed)
    net = NeRF_TP(num_coarse_samples=8, num_fine_samples=4, num_src_views=nv, precision="tc").eval()
    net.load_state_dict(P)
    net = net.to(cuda)
    net.set_scene(*[sc[k].to(cuda) for k in ("planes_xz", "planes_xy", "planes_yz", "latent", "src_poses", "src_focal", "src_c")],
                  sc["img_wh"], precisions=["tc"])
    W, H = sc["img_wh"]
    d = lambda k: sc[k].to(cuda, torch.float64)
    osc = orc.Scene(d("planes_xz"), d("planes_xy"), d("planes_yz"), d("latent"), d("src_poses"),
                    float(sc["src_focal"][0]), float(sc["src_c"][0, 0]), float(sc["src_c"][0, 1]), W, H)
    return net, osc, P


def edge_rays(bg):
    """The edge scene of test_gpu_tc_kernels.py: axis-aligned rays whose t (fg) or s (bg) values put the lookups on, half a texel
    out, just inside and just outside the plane grids' edges, far outside, and on z_cam = 0 (the latent projection's pole)."""
    Hp, Wp = PLANE_HW
    targets = sorted({0.0, 0.5, 1.0} | {1.0 + 2.0 * f / (L - 1) for L in (Hp, Wp) for f in (0.5, 0.999, 1.001, 1.5, 4.0)})
    rays = [((0.0, 0.05, 0.0), 0), ((0.0, 0.05, -0.3), 0), ((0.05, 0.0, 0.0), 1), ((0.05, 0.0, -0.3), 1),
            ((0.05, 0.03, 0.0), 2), ((-0.2, 0.1, 0.0), 2)]
    o, d = [], []
    for org, axis in rays:
        for sign in (1.0, -1.0):
            o.append(org)
            d.append([sign if k == axis else 0.0 for k in range(3)])
    o, d = torch.tensor(o), torch.tensor(d)
    far = orc.intersect_sphere(o, d)
    tgt = torch.tensor(targets + [2.0, 2.5, 3.0])[None].expand(o.shape[0], -1)
    if bg:      # lookup distance far (1 - s) + 3 s = target
        t = torch.sort(((tgt - far) / (3.0 - far)).clamp(0.0, 1.0), -1, descending=True).values
    else:
        t = tgt
    return o, d, far, t.contiguous()


def inputs(cuda, n_sm, bg, seed):
    """Random rays inside the unit sphere with the edge rays spliced in every EDGE_EVERY rays; the ray count gives every consumer
    (2 per SM) at least three tiles, a tile count that is not a multiple of 2 n_sm and a ragged last ray group."""
    eo, ed, ef, et = edge_rays(bg)
    N = et.shape[1]
    sg = (N + TILE_SAMPLES - 1) // TILE_SAMPLES
    groups = (3 * 2 * n_sm + sg - 1) // sg + 1
    while (groups * sg) % (2 * n_sm) == 0:
        groups += 1
    n = groups * TILE_RAYS - 5
    g = torch.Generator().manual_seed(seed)
    o = (torch.rand(n, 3, generator=g) - 0.5) * 1.0
    d = torch.randn(n, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True)
    far = orc.intersect_sphere(o, d)
    u = torch.sort(torch.rand(n, N, generator=g), -1).values
    t = torch.flip(u, [-1]) if bg else u * far * 1.2
    for lo in range(0, n - eo.shape[0], EDGE_EVERY):
        sl = slice(lo, lo + eo.shape[0])
        o[sl], d[sl], far[sl], t[sl] = eo, ed, ef, et
    rays = {"rays_o": o.to(cuda), "rays_d": d.to(cuda), "viewdirs": d.to(cuda)}
    return rays, far.to(cuda), t.contiguous().to(cuda), groups * sg


def lookups(rays, far, t, bg):
    """float64 lookup points (n, N, 3) of the world frame (= every camera's frame here)."""
    o, dd, t64 = rays["rays_o"].double(), rays["rays_d"].double(), t.double()
    tl = far.double().reshape(-1, 1) * (1 - t64) + 3.0 * t64 if bg else t64
    return o[:, None, :] + tl[..., None] * dd[:, None, :]


@pytest.mark.parametrize("nv", [1, 3, 8])
def test_tc_field_tile_handoff(cuda, nv):
    """Bit for bit: the full call = every chunk on its own = a permuted ray order, for all four MLPs.  At NV = 3 also the model
    bounds, where the latent projection is well conditioned (|z_cam| >= 1e-2) or puts the lookup far outside the map."""
    n_sm = torch.cuda.get_device_properties(cuda).multi_processor_count
    net, osc, P = tc_net(cuda, nv, 40 + nv)
    Hp, Wp = PLANE_HW
    for mlp_index in range(4):
        bg = mlp_index & 1
        rays, far, t, tiles = inputs(cuda, n_sm, bg, 500 + 10 * nv + mlp_index)
        n, N = t.shape
        assert tiles >= 3 * 2 * n_sm and tiles % (2 * n_sm) != 0, (tiles, n_sm)
        # map corners: plane quads with x0 = -1 (x on the xz / xy planes) and with y0 = -1 (z on the xz plane), in every view
        xl = lookups(rays, far, t, bg)
        ix, iz = ((xl[..., 0] + 1) / 2) * (Wp - 1), ((xl[..., 2] + 1) / 2) * (Hp - 1)
        corner_x, corner_y = int(((ix > -1) & (ix < 0)).sum()), int(((iz > -1) & (iz < 0)).sum())
        assert corner_x > 0 and corner_y > 0, (corner_x, corner_y)
        with torch.no_grad():
            rgb, sig = net.field_eval(rays, far, t, mlp_index, chunk=CHUNK, precision="tc")
            assert torch.isfinite(rgb).all() and torch.isfinite(sig).all(), mlp_index
            perm = torch.randperm(n, generator=torch.Generator().manual_seed(nv + mlp_index)).to(torch.int32).to(cuda)
            prgb, psig = net.field_eval(rays, far, t, mlp_index, chunk=CHUNK, precision="tc", ray_order=perm)
            res = [("permuted", md(prgb, rgb), md(psig, sig))]
            for lo in range(0, n, CHUNK):
                hi = min(lo + CHUNK, n)
                sub = {k: v[lo:hi].contiguous() for k, v in rays.items()}
                srgb, ssig = net.field_eval(sub, far[lo:hi], t[lo:hi], mlp_index, chunk=CHUNK, precision="tc")
                res.append((f"rays [{lo}, {hi}) alone", md(srgb, rgb[lo:hi]), md(ssig, sig[lo:hi])))
        net.check()
        print(f"tile hand-off nv={nv} mlp={mlp_index}: {n} rays x {N} samples, {tiles} tiles on {n_sm} SMs, "
              f"{corner_x} / {corner_y} corner lookups (x0 / y0 = -1) per view, {len(res) - 1} chunks")
        for name, a, b in res:
            assert a == 0 and b == 0, (nv, mlp_index, name, a, b)
        if nv == 3:
            with torch.no_grad():
                mr, ms = tcm.tc_field(rays, far, t, mlp_index, osc, P, chunk=CHUNK)
            gx, gy = tcm.latent_coords(xl.reshape(1, -1, 3), osc)
            keep = (xl[..., 2].abs() >= 1e-2) | (torch.maximum(gx.abs(), gy.abs()) > 100).reshape(n, N)
            er = (rgb.double() - mr).abs().amax(-1)[keep]
            es = ((sig.double() - ms).abs() / (1 + ms))[..., 0][keep]
            e = (float(er.max()), float(es.max()), float(er.mean()), float(es.mean()))
            print(f"tile hand-off nv={nv} mlp={mlp_index} vs model: max rgb {e[0]:.2e} sigma/(1+sigma) {e[1]:.2e}, mean rgb "
                  f"{e[2]:.2e} sigma/(1+sigma) {e[3]:.2e} ({int(keep.sum())} of {n * N} points compared)")
            assert e[0] <= tcm.RGB_TOL and e[1] <= tcm.SIGMA_TOL, e
            assert e[2] <= tcm.RGB_MEAN_TOL and e[3] <= tcm.SIGMA_MEAN_TOL, e
