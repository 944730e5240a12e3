"""GPU: the two tensor-core kernels against high-precision models of the SAME computation, at bounds that fail for a subtle error.

* The NEO_PREC_TC field kernel (csrc/field_tc.cu) point by point against oracle/tc_model.py (float64, with the kernel's fp16
  roundings), which tests/test_tc_model.py pins to the oracle on the CPU.  Bounds: tc_model.RGB_TOL / SIGMA_TOL.
* Its schedule invariance: every point's blend is a per-thread fp32 loop in a fixed order and a wgmma row does not depend on the
  other rows, so a point's output is bit-identical wherever it lands in a tile.
* gemm_f16 (csrc/gemm_tc.cu) at the strides, bias modes and buffer aliasing of its callers against a float64 matmul of the same
  fp16 operands, with C's untouched rows / columns checked against a sentinel.

Run with `-m gpu -s` on an H100: the measured errors are printed per case.
"""
import math

import pytest
import torch

from neo360_b200 import synth
from oracle import neo360_oracle as orc
from oracle import tc_model as tcm

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cuda():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from neo360_b200 import build
    build.build()
    return torch.device("cuda:0")


def md(a, b):
    return float((a.detach().double() - b.detach().to(a.device).double()).abs().max()) if a.numel() else 0.0


def tc_net(cuda, img_wh, nv, plane_hw, seed, poses=None):
    """NeRF_TP with a NEO_PREC_TC scene, and the same scene for the model (float64 maps and cameras)."""
    from neo360_b200 import NeRF_TP
    sc = synth.make_scene(img_wh, nv, plane_hw, seed)
    if poses is not None:
        sc["src_poses"] = poses
    P = synth.make_mlp_params(seed)
    net = NeRF_TP(num_coarse_samples=8, num_fine_samples=4, num_src_views=nv, precision="tc").eval()
    net.load_state_dict(P)
    net = net.to(cuda)
    net.set_scene(*[sc[k].to(cuda) for k in ("planes_xz", "planes_xy", "planes_yz", "latent", "src_poses", "src_focal", "src_c")],
                  sc["img_wh"], precisions=["tc"])
    W, H = img_wh
    d = lambda k: sc[k].to(cuda, torch.float64)
    osc = orc.Scene(d("planes_xz"), d("planes_xy"), d("planes_yz"), d("latent"), d("src_poses"),
                    float(sc["src_focal"][0]), float(sc["src_c"][0, 0]), float(sc["src_c"][0, 1]), W, H)
    return net, osc, P


def random_inputs(cuda, n, N, bg, seed):
    """fp32 rays inside the unit sphere, far, and t (fg, up to 1.2 far) or descending s (bg) values."""
    g = torch.Generator().manual_seed(seed)
    o = (torch.rand(n, 3, generator=g) - 0.5) * 1.0
    d = torch.randn(n, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True)
    far = orc.intersect_sphere(o, d)
    u = torch.sort(torch.rand(n, N, generator=g), -1).values
    t = torch.flip(u, [-1]) if bg else u * far * 1.2
    return {"rays_o": o.to(cuda), "rays_d": d.to(cuda), "viewdirs": d.to(cuda)}, far.to(cuda), t.to(cuda)


def field_errors(net, osc, P, rays, far, t, mlp_index, chunk, ray_order=None, mask=None):
    """Kernel vs model: (max |rgb diff|, max |sigma diff| / (1 + sigma)) over the points selected by `mask` (n, N)."""
    with torch.no_grad():
        rgb, sig = net.field_eval(rays, far, t, mlp_index, chunk=chunk, precision="tc", ray_order=ray_order)
        net.check()
        mr, ms = tcm.tc_field(rays, far, t, mlp_index, osc, P, chunk=chunk)
    er = (rgb.double() - mr).abs().amax(-1)
    es = ((sig.double() - ms).abs() / (1 + ms))[..., 0]
    if mask is not None:
        er, es = er[mask], es[mask]
    return (float(er.max()), float(es.max()), float(er.mean()), float(es.mean())), rgb, sig


def check_field(worst, errs):
    """Fold one case's (max rgb, max sigma, mean rgb, mean sigma) errors into `worst`."""
    return [max(a, b) for a, b in zip(worst, errs)]


def assert_field_bounds(worst):
    assert worst[0] <= tcm.RGB_TOL and worst[1] <= tcm.SIGMA_TOL, worst
    assert worst[2] <= tcm.RGB_MEAN_TOL and worst[3] <= tcm.SIGMA_MEAN_TOL, worst


# n_rays x N x chunk: every n_rays in {1, 15, 17, 33} and N in {5, 17, 129, 385}, chunk 0 and ragged last chunks; (33, 385) has
# 3 x 97 = 291 tiles and (300, 129) 19 x 33 = 627 tiles, more than 2 per SM on a 132-SM H100, so every warpgroup loops
CELLS = [(1, 5, 0), (15, 385, 4), (17, 129, 0), (33, 17, 10), (33, 385, 0), (300, 129, 128)]


@pytest.mark.parametrize("nv", [1, 3, 8])
def test_tc_field_matches_model(cuda, nv):
    """Every MLP, nv in {1, 3, 8} (8 = kMaxViews, the largest shared-memory footprint), odd map sizes (plane 13 x 17; image 37 x 23,
    latent 18 x 11, so the pre-projection's M is ragged against 128) over the CELLS matrix.
    Stated, per point: |rgb - model| <= tc_model.RGB_TOL (1e-2), |sigma - model| / (1 + sigma) <= SIGMA_TOL (4e-3); per case, the means
    of those errors <= RGB_MEAN_TOL (1e-3) / SIGMA_MEAN_TOL (4e-4).  Measured on an H100 80GB HBM3 (700 W), max over all nv and cells:
    per point rgb 4.4e-3, sigma 1.4e-3; largest case mean rgb 3.8e-4, sigma 1.1e-4.  The per-point maximum is fp16 rounding noise
    (see tc_model.py), not one fp32 rounding; the means are what a layout bug moves by orders of magnitude."""
    net, osc, P = tc_net(cuda, (37, 23), nv, (13, 17), 30 + nv)
    worst = [0.0] * 4
    for mlp_index in range(4):
        for ci, (n, N, chunk) in enumerate(CELLS):
            rays, far, t = random_inputs(cuda, n, N, mlp_index & 1, 1000 * nv + 10 * mlp_index + ci)
            e, _, _ = field_errors(net, osc, P, rays, far, t, mlp_index, chunk)
            print(f"tc field nv={nv} mlp={mlp_index} n={n:3d} N={N:3d} chunk={chunk:3d}: max rgb {e[0]:.2e} sigma/(1+sigma) {e[1]:.2e}, "
                  f"mean rgb {e[2]:.2e} sigma/(1+sigma) {e[3]:.2e}")
            worst = check_field(worst, e)
    print(f"tc field nv={nv}: max rgb {worst[0]:.2e}, sigma/(1+sigma) {worst[1]:.2e}; largest cell mean rgb {worst[2]:.2e}, "
          f"sigma/(1+sigma) {worst[3]:.2e}")
    assert_field_bounds(worst)


def edge_inputs(cuda, bg, plane_hw):
    """Axis-aligned rays through a scene whose single source camera has the identity pose (camera frame = world frame), with
    t (fg) or s (bg) values that put the lookups exactly on the plane grids' edges: grid coordinate +-1 (ix = 0 and ix = W-1), half a
    texel out, just inside and just outside [-1, W), far outside (bg lookups out to radius 3), and points on z_cam = 0 (the latent
    projection's pole).  Every origin has coordinate 0 along its ray's axis, so that coordinate is +-(distance along the ray)."""
    Hp, Wp = plane_hw
    targets = sorted({0.0, 0.5, 1.0} | {1.0 + 2.0 * f / (L - 1) for L in (Hp, Wp) for f in (0.5, 0.999, 1.001, 1.5, 4.0)})
    rays = [((0.0, 0.05, 0.0), 0), ((0.0, 0.05, -0.3), 0), ((0.05, 0.0, 0.0), 1), ((0.05, 0.0, -0.3), 1),
            ((0.05, 0.03, 0.0), 2), ((-0.2, 0.1, 0.0), 2)]                   # (origin, axis); z = 0 rays lie on the pole plane
    o, d = [], []
    for org, axis in rays:
        for sign in (1.0, -1.0):
            o.append(org)
            d.append([sign if k == axis else 0.0 for k in range(3)])
    o, d = torch.tensor(o), torch.tensor(d)
    far = orc.intersect_sphere(o, d)
    tgt = torch.tensor(targets + [2.0, 2.5, 3.0])[None].expand(o.shape[0], -1)
    if bg:      # lookup distance far (1 - s) + 3 s = target  (targets short of `far` clamp to s = 0)
        t = torch.sort(((tgt - far) / (3.0 - far)).clamp(0.0, 1.0), -1, descending=True).values
    else:
        t = tgt
    return {"rays_o": o.to(cuda), "rays_d": d.to(cuda), "viewdirs": d.to(cuda)}, far.to(cuda), t.contiguous().to(cuda)


def test_tc_field_edge_scene(cuda):
    """Lookups exactly on and around the edges of the maps (edge_inputs), every MLP, chunk 0 and a ragged chunk.  Where the latent
    projection is ill-conditioned (|z_cam| < 1e-2) only finiteness is asserted, unless the model puts the latent lookup far
    outside the map (|grid coordinate| > 100): then far-outside taps must contribute exactly what the model says, nothing.
    Everywhere else: the bounds of test_tc_field_matches_model.  Measured on an H100: per point rgb 1.7e-3, sigma 1.3e-3; case mean
    rgb 2.3e-4, sigma 8.8e-5."""
    plane_hw = (13, 17)
    net, osc, P = tc_net(cuda, (37, 23), 1, plane_hw, 5, poses=torch.eye(4)[None])
    Hp, Wp = plane_hw
    worst = [0.0] * 4
    cover = {"edge": 0, "inside_last": 0, "outside_last": 0, "far": 0, "pole": 0}
    for mlp_index in range(4):
        rays, far, t = edge_inputs(cuda, mlp_index & 1, plane_hw)
        n, N = t.shape
        # lookup points of the model (float64): the camera frame is the world frame
        o, dd, t64 = rays["rays_o"].double(), rays["rays_d"].double(), t.double()
        tl = far.double().reshape(-1, 1) * (1 - t64) + 3.0 * t64 if mlp_index & 1 else t64
        xl = o[:, None, :] + tl[..., None] * dd[:, None, :]
        ix = ((xl[..., 0] + 1) / 2) * (Wp - 1)                       # x on the xz / xy planes
        cover["edge"] += int(((ix - (Wp - 1)).abs() < 1e-5).sum() + (ix.abs() < 1e-5).sum())
        cover["inside_last"] += int(((ix > Wp - 1 + 1e-5) & (ix < Wp)).sum() + ((ix > -1) & (ix < -1e-5)).sum())
        cover["outside_last"] += int(((ix >= Wp) & (ix < Wp + 1)).sum() + ((ix <= -1) & (ix > -2)).sum())
        cover["far"] += int((ix > Wp + 4).sum())
        gx, gy = tcm.latent_coords(xl.reshape(1, -1, 3), osc)
        z = xl[..., 2]
        ill = z.abs() < 1e-2
        far_out = (torch.maximum(gx.abs(), gy.abs()) > 100).reshape(n, N)
        cover["pole"] += int((z == 0).sum())
        keep = ~ill | far_out
        for chunk in (0, 5):
            e, rgb, sig = field_errors(net, osc, P, rays, far, t, mlp_index, chunk, mask=keep)
            assert torch.isfinite(rgb).all() and torch.isfinite(sig).all(), (mlp_index, chunk)
            print(f"tc field edge scene mlp={mlp_index} chunk={chunk}: max rgb {e[0]:.2e} sigma/(1+sigma) {e[1]:.2e}, mean rgb "
                  f"{e[2]:.2e} sigma/(1+sigma) {e[3]:.2e} ({int(keep.sum())} of {n * N} points compared)")
            worst = check_field(worst, e)
    print("edge scene coverage (lookups):", cover)
    assert all(v > 0 for v in cover.values()), cover
    assert_field_bounds(worst)


def test_tc_field_is_schedule_invariant(cuda):
    """A random ray order, and whole chunks evaluated on their own (quirk Q1 conditions on the chunk, so a chunk is the unit that
    can be split off), reproduce the full call's rows bit for bit: a point's result does not depend on its tile or row."""
    net, osc, P = tc_net(cuda, (37, 23), 3, (13, 17), 9)
    n, N, chunk = 100, 37, 32                            # chunks 32, 32, 32, 4
    for mlp_index in range(4):
        rays, far, t = random_inputs(cuda, n, N, mlp_index & 1, 77 + mlp_index)
        with torch.no_grad():
            rgb, sig = net.field_eval(rays, far, t, mlp_index, chunk=chunk, precision="tc")
            perm = torch.randperm(n, generator=torch.Generator().manual_seed(mlp_index)).to(torch.int32).to(cuda)
            prgb, psig = net.field_eval(rays, far, t, mlp_index, chunk=chunk, precision="tc", ray_order=perm)
            res = [("permuted", md(prgb, rgb), md(psig, sig))]
            for lo, hi in ((32, 64), (96, 100), (0, 96)):
                sub = {k: v[lo:hi].contiguous() for k, v in rays.items()}
                srgb, ssig = net.field_eval(sub, far[lo:hi], t[lo:hi], mlp_index, chunk=chunk, precision="tc")
                res.append((f"rays [{lo}, {hi}) alone", md(srgb, rgb[lo:hi]), md(ssig, sig[lo:hi])))
            sub = {k: v[32:64].contiguous() for k, v in rays.items()}
            sp = torch.randperm(32, generator=torch.Generator().manual_seed(9)).to(torch.int32).to(cuda)
            srgb, ssig = net.field_eval(sub, far[32:64], t[32:64], mlp_index, chunk=chunk, precision="tc", ray_order=sp)
            res.append(("rays [32, 64) alone, permuted", md(srgb, rgb[32:64]), md(ssig, sig[32:64])))
        net.check()
        for name, a, b in res:
            print(f"tc field schedule mlp={mlp_index} {name}: md rgb {a} sigma {b}")
            assert a == 0 and b == 0, (mlp_index, name, a, b)


# ---------------- gemm_f16 ----------------

SENTINEL = 0x7E00                                       # fp16 NaN bit pattern


def f16_ulp(x):
    """One fp16 ulp at |x| (normal range), 2^-24 in the subnormal range and at 0."""
    e = torch.frexp(x.abs())[1]                         # |x| in [2^(e-1), 2^e)
    ulp = torch.exp2((e - 11).to(x.dtype))
    return torch.where(x == 0, torch.full_like(x, 2.0 ** -24), torch.clamp(ulp, min=2.0 ** -24))


def run_gemm(cuda, M, N, K, relu, use_bias, lda=None, ldw=None, ldc=None, a_off=None, seed=0):
    """One neo_tc_gemm_f16 call.  C lives in a sentinel-filled (M + 3) x ldc buffer; with `a_off` the A operand is columns
    [a_off, a_off + K) of C's own rows (the Mip-NeRF 360 / vanilla activation buffers), else its own M x lda buffer whose padding
    columns are NaN, as are W's.  Returns (max error / bound, sentinel intact, A intact, max of (error - 1 ulp) / sum_k |a_k w_k| in
    units of 2^-24)."""
    from neo360_b200 import _lib as L
    lib = L.load()
    lda = lda or (ldc if a_off is not None else K)
    ldw = ldw or K
    ldc = ldc or N
    g = torch.Generator(device=cuda).manual_seed(seed)
    a = torch.randn(M, K, generator=g, device=cuda).half()
    w = (torch.randn(N, K, generator=g, device=cuda) / math.sqrt(K)).half()
    bias = torch.randn(N, generator=g, device=cuda) if use_bias else None
    cbuf = torch.full((M + 3, ldc), SENTINEL, dtype=torch.int16, device=cuda).view(torch.float16)
    wbuf = torch.full((N, ldw), SENTINEL, dtype=torch.int16, device=cuda).view(torch.float16)
    wbuf[:, :K] = w
    if a_off is not None:
        assert lda == ldc and a_off >= N and a_off + K <= ldc
        cbuf[:M, a_off:a_off + K] = a
        a_ptr = cbuf[:, a_off:].data_ptr()
        abuf = None
    else:
        abuf = torch.full((M, lda), SENTINEL, dtype=torch.int16, device=cuda).view(torch.float16)
        abuf[:, :K] = a
        a_ptr = abuf.data_ptr()
    before = cbuf.clone()
    L.check(lib.neo_tc_gemm_f16(a_ptr, lda, wbuf.data_ptr(), ldw, bias.data_ptr() if use_bias else None, cbuf.data_ptr(), ldc,
                                M, N, K, relu, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    a64, w64 = a.double(), w.double()
    ref = a64 @ w64.T
    if use_bias:
        ref = ref + bias.double()
    if relu:
        ref = torch.relu(ref)
    absum = a64.abs() @ w64.abs().T
    got = cbuf[:M, :N].double()
    ulp = f16_ulp(ref)
    err = (got - ref.half().double()).abs()
    ratio = float((err / (ulp + 2.0 ** -21 * absum)).max())
    acc_c = float(((err - ulp).clamp(min=0) / absum.clamp(min=1e-30)).max()) * 2.0 ** 24
    if not torch.isfinite(got).all():
        ratio = float("inf")
    raw, raw0 = cbuf.view(torch.int16), before.view(torch.int16)
    untouched = torch.ones_like(raw, dtype=torch.bool)
    untouched[:M, :N] = False
    sentinel_ok = bool((raw[untouched] == raw0[untouched]).all())
    a_ok = True if a_off is None else bool(torch.equal(cbuf[:M, a_off:a_off + K], a))
    return ratio, sentinel_ok, a_ok, acc_c


GEMM_M = [1, 127, 128, 129, 70000]
GEMM_N = [64, 128, 192, 256, 320, 1024]
GEMM_K = [64, 192, 1536]


@pytest.mark.parametrize("N", GEMM_N)
@pytest.mark.parametrize("M", GEMM_M)
def test_gemm_f16_vs_float64(cuda, M, N):
    """gemm_f16 at every M (1, one short of / exactly / one over a 128-row tile, many tiles) x N (BN = 64 with several column tiles
    for 192 and 320, BN = 128 otherwise) x K (64: one k-block, fewer than the 3 stages; 192; 1536), relu on / off and bias on / NULL
    alternating, against a float64 matmul of the same fp16 operands + the fp32 bias.  Stated, element-wise:
    |got - fp16(ref)| <= 1 fp16 ulp of ref + 2^-21 sum_k |a_k w_k|; every element of C outside [0, M) x [0, N) keeps its sentinel.
    Measured on an H100: beyond the 1-ulp term the error reaches 2.0 x 2^-24 sum_k |a_k w_k| (wgmma's fp32 accumulation over up to 96
    k-steps); 2^-22 was exceeded (by 1.2x) at M = 70000, K = 1536 with a bias, hence 2^-21."""
    mi, ni = GEMM_M.index(M), GEMM_N.index(N)
    for ki, K in enumerate(GEMM_K):
        relu, use_bias = (mi + ki) % 2, (ni + ki) % 2 == 0
        ratio, sent, _, acc_c = run_gemm(cuda, M, N, K, relu, use_bias, seed=M * 7 + N * 3 + K)
        print(f"gemm_f16 M={M:5d} N={N:4d} K={K:4d} relu={relu} bias={'yes' if use_bias else 'NULL'}: "
              f"max err / bound {ratio:.3f} (beyond 1 ulp: {acc_c:.2f} x 2^-24 sum|aw|), sentinel {'intact' if sent else 'OVERWRITTEN'}")
        assert ratio <= 1.0 and sent, (M, N, K, relu, use_bias, ratio, sent)


GEMM_CALLS = [
    # name, M, N, K, lda, ldw, ldc, a_off, relu, bias
    ("vanilla layer 0: A = cols [256, 320) of C's rows", 4099, 256, 64, 320, 64, 320, 256, 1, True),
    ("vanilla hidden layer, ld 320", 4099, 256, 256, 320, 256, 320, None, 1, True),
    ("vanilla view layer, K 320", 777, 128, 320, 320, 320, 128, None, 1, True),
    ("mip layer 0, W 320: A = cols [W, W+512) of C's rows", 3001, 320, 512, 832, 512, 832, 320, 1, True),
    ("mip layer 0, W 1024", 2049, 1024, 512, 1536, 512, 1536, 1024, 1, True),
    ("mip layer 5, reads [0, W+512), W 256", 1025, 256, 768, 768, 768, 768, None, 1, True),
    ("mip bottleneck, no relu, ld W+512", 1000, 256, 1024, 1536, 1024, 256, None, 0, True),
    ("pre-projection: latent, no bias, ragged M", 198, 256, 512, 512, 512, 256, None, 0, False),
    ("pre-projection: plane, no bias", 221, 256, 128, 128, 128, 256, None, 0, False),
    ("strided W rows (ldw = K + 64)", 300, 192, 192, 200, 256, 264, None, 1, False),
]


@pytest.mark.parametrize("case", GEMM_CALLS, ids=[c[0] for c in GEMM_CALLS])
def test_gemm_f16_call_patterns(cuda, case):
    """gemm_f16 at its callers' call patterns (csrc/vanilla.cu, csrc/mip.cu, the scene pre-projection in csrc/field_tc.cu): strided rows,
    NULL bias, and A inside C's own buffer at disjoint columns, which is only correct if the epilogue writes no column >= N.  Same
    bound as test_gemm_f16_vs_float64; the sentinel outside [0, M) x [0, N) and, when aliased, A itself must be intact."""
    name, M, N, K, lda, ldw, ldc, a_off, relu, use_bias = case
    ratio, sent, a_ok, acc_c = run_gemm(cuda, M, N, K, relu, use_bias, lda, ldw, ldc, a_off, seed=M + N + K)
    print(f"gemm_f16 [{name}] M={M} N={N} K={K} lda={lda} ldw={ldw} ldc={ldc}: max err / bound {ratio:.3f} ({acc_c:.2f} x 2^-24), "
          f"sentinel {'intact' if sent else 'OVERWRITTEN'}, A {'intact' if a_ok else 'OVERWRITTEN'}")
    assert ratio <= 1.0 and sent and a_ok, (name, ratio, sent, a_ok)
