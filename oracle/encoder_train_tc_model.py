"""Float64 model of the tensor-core training form of GridEncoder's dense part (csrc/encoder.cu, csrc/gemm_tc.cu, csrc/dense_train.cu,
encoder._DenseTC) with every bf16 rounding the kernels apply made explicit, its hand-written adjoint, and the bounds the GPU tests hold the
kernels to.

Forward, rows r = v 64^3 + cell of the lookup rows X (R, 518) (`neo_grid_encoder_features`), depth_fc weights w_i, b_i, aggregator a
(0 yz, 1 xz, 2 xy) weights u_a (512, 513), c_a (512), q_a (1, 512), e_a (1):
    x = bf(X);  h_0 = bf(relu(x bf(w_0)^T + b_0));  h_1 = bf(relu(h_0 bf(w_1)^T + b_1));  lat = bf(h_1 bf(w_2)^T + b_2)
    Lb = [lat | bf(world x, y, z of the cell) | 0]                                   (R, 576)
    A = bf(relu(Lb bf(U)^T + c))   (R, 1536): U (1536, 576) stacks the aggregators, row block a = [u_a[:, :512] | 0 .. u_a[:, 512] at
                                    column 512 + a .. 0], c = [c_0 | c_1 | c_2]; so A[:, 512a:512a+512] is aggregator a's own first layer
    logits_a = A_a q_a^T + e_a      (A_a = A[:, 512a:512a+512]; q_a fp32: the bf16 rowdot head)
    planes = softmax pillar sums of lat with the logits (encoder_train_model.pool_fwd), fp32
Backward, upstream g_xz, g_xy, g_yz:
    d_pool, d_logits = encoder_train_model.pool_bwd(lat, logits, g)                  (fp32, unrounded)
    dA_a = bf(d_logits_a q_a [A_a > 0]);  dU = dA^T Lb (columns < 515);  dc = sum_rows dA;  dq_a = bf(d_logits_a)^T A_a;  de_a = sum d_logits_a
    d_lat = bf(d_pool + dA bf(U)[:, :512])
    dw_2 = d_lat^T h_1;  dh_1 = bf((d_lat bf(w_2)) [h_1 > 0]);  dw_1 = dh_1^T h_0;  dh_0 = bf((dh_1 bf(w_1)) [h_0 > 0]);  dw_0 = dh_0^T x
    db_i = sum_rows of the gradient into layer i's output;  g_X = dh_0 bf(w_0)[:, :512]   (fp32, the lookup columns only)
bf() rounds an fp32 value to bf16 (nearest even).  Biases, accumulators, logits, softmax, floor plans, d_logits, d_pool and g_X stay
fp32 and unrounded.  With `rnd=False` every bf() is the identity and the model is autograd through `GridEncoder.dense_torch` in float64
(tests/test_encoder_train_tc_model.py).  G is read from the module (`module.GRID`), so the CPU tests can run an 8^3 grid.

Bounds, as ||kernel - model|| / ||model|| per tensor (Frobenius), the model fed the kernel's own fp32 lookup rows:
* POOL_BOUND: the bf16 pool forward and backward at identical inputs (bf16 lat, fp32 logits): fp32 exp / sum orders only.
* FWD_BOUND / BWD_BOUND: the whole dense part, forward (three floor plans) and backward (g_X and every parameter gradient).  The kernels
  sum in other fp32 orders than float64, which flips a bf16 rounding now and then (2^-8 of an element) and a ReLU mask where a
  pre-activation sits within that error of zero; the backward carries those flips through four more products.
* STEP_BOUND: the tc form against the fp32 `dense_train` at identical upstream gradients: the bf16 roundings themselves (the bound of the
  other tensor-core training paths).
* ENC_STEP_BOUND: the NeO-360 step with both the renderer and the encoder in tc against the all-fp32 step.  Here the two forms' planes
  and their upstream gradients already differ by the renderer's bf16 roundings (feature-map gradients 0.05-0.07 with a frozen encoder,
  DESIGN.md section 6), and the encoder's gradients sum those differences over the 64^3 x 3 grid rows on top of its own, so 0.15 does
  not hold: the step's encoder gradients measure up to 0.21.
Measured on an H100 80GB HBM3 at 700 W (tests/test_gpu_encoder_train_tc.py): pool forward and backward 1.3e-7 to 1.9e-7; dense part
forward 9.7e-5 to 1.4e-4, backward 4.3e-4 (depth_encoder bias) to 7.2e-3 (the aggregators' first-layer biases and weights, sums over all
grid rows); against the fp32 `dense_train` up to 0.080; the whole step up to 0.206.  Each bound is 2-3x its measured maximum, except
STEP_BOUND, the shared a-priori bound of the tensor-core training paths.
"""
from __future__ import annotations

import torch

from . import encoder_train_model as etm

AXES = etm.AXES                 # aggregator a = 0 / 1 / 2: yz / xz / xy, coordinate x / y / z
LAT, LD, NA = 512, 576, 3

POOL_BOUND = 5e-7
FWD_BOUND = 4e-4
BWD_BOUND = 2e-2
STEP_BOUND = 0.15
ENC_STEP_BOUND = 0.45


def bf(x, on=True):
    return x.float().bfloat16().double() if on else x


def params_of(module):
    """float64 copies of the parameters of depth_fc and the three aggregators (axis order yz, xz, xy)."""
    d = lambda t: t.detach().double().clone()
    fc = module.depth_fc
    lins = [fc.common_branch[0], fc.common_branch[2], fc.depth_encoder]
    P = {"w": [d(m.weight) for m in lins], "b": [d(m.bias) for m in lins]}
    for k in ("u", "c", "q", "e"):
        P[k] = []
    for n in AXES:
        agg = getattr(module, f"pillar_aggregator_{n}")
        P["u"].append(d(agg[0].weight)); P["c"].append(d(agg[0].bias)); P["q"].append(d(agg[2].weight)); P["e"].append(d(agg[2].bias))
    return P


def stack_first_layers(u):
    """U (1536, 576): row block a = u_a's 512 latent columns, its coordinate column at column 512 + a, zeros elsewhere."""
    U = torch.zeros(NA * LAT, LD, dtype=u[0].dtype, device=u[0].device)
    for a in range(NA):
        U[a * LAT:(a + 1) * LAT, :LAT] = u[a][:, :LAT]
        U[a * LAT:(a + 1) * LAT, LAT + a] = u[a][:, LAT]
    return U


def grid_coords(G: int, nv: int, dtype=torch.float32, device=None):
    """(nv G^3, 3) world x, y, z of every grid row, torch.linspace in `dtype` as dense_torch / dense_train build the grid."""
    ax = [torch.linspace(-1, 1, G, dtype=dtype), torch.linspace(-1, 1, G, dtype=dtype), torch.linspace(0, 1, G, dtype=dtype)]
    g = torch.stack(torch.meshgrid(*ax, indexing="ij"), -1).reshape(-1, 3)
    return g.repeat(nv, 1).to(device=device, dtype=torch.float64)


def forward(X, coords, P, nv: int, G: int, rnd=True):
    """X (R, >= 518) lookup rows, coords (R, 3) -> planes {"xz", "xy", "yz"} (nv, 512, G, G), logits (3, R), saved state."""
    r = lambda t: bf(t, rnd)
    x = r(X[:, :518].double())
    h0 = r(torch.relu(x @ r(P["w"][0]).T + P["b"][0]))
    h1 = r(torch.relu(h0 @ r(P["w"][1]).T + P["b"][1]))
    lat = r(h1 @ r(P["w"][2]).T + P["b"][2])
    Lb = torch.cat([lat, r(coords.double()), torch.zeros(lat.shape[0], LD - LAT - 3, dtype=lat.dtype, device=lat.device)], -1)
    U = stack_first_layers(P["u"])
    A = r(torch.relu(Lb @ r(U).T + torch.cat(P["c"])))
    logits = torch.stack([A[:, a * LAT:(a + 1) * LAT] @ P["q"][a][0] + P["e"][a][0] for a in range(NA)])
    planes = etm.pool_fwd(lat, logits, nv, G)
    S = dict(x=x, h0=h0, h1=h1, lat=lat, Lb=Lb, A=A, U=U, logits=logits)
    return {n: planes[n] for n in ("xz", "xy", "yz")}, logits, S


def backward(g_xz, g_xy, g_yz, S, P, nv: int, G: int, rnd=True):
    """Adjoint of `forward` -> dict: g_X (R, 512) and every parameter gradient in nn.Linear layout (w0..2, b0..2, {axis}_w0 / _b0 / _w1 /
    _b1), plus the pool's d_pool and d_logits."""
    r = lambda t: bf(t, rnd)
    pb = etm.pool_bwd(S["lat"], S["logits"], nv, G, g_xz=g_xz, g_xy=g_xy, g_yz=g_yz)
    d_pool, d_lg = pb["d_lat"], pb["d_logits"]
    A, Lb, U = S["A"], S["Lb"], S["U"]
    dA = torch.cat([r(d_lg[a][:, None] * P["q"][a] * (A[:, a * LAT:(a + 1) * LAT] > 0)) for a in range(NA)], -1)
    dU, dc = dA.T @ Lb, dA.sum(0)
    out = dict(d_pool=d_pool, d_logits=d_lg)
    for a, n in enumerate(AXES):
        rows = slice(a * LAT, (a + 1) * LAT)
        out[f"{n}_w0"] = torch.cat([dU[rows, :LAT], dU[rows, LAT + a:LAT + a + 1]], -1)
        out[f"{n}_b0"] = dc[rows]
        out[f"{n}_w1"] = (r(d_lg[a]) @ A[:, rows])[None]
        out[f"{n}_b1"] = d_lg[a].sum(0, keepdim=True)
    d_lat = r(d_pool + dA @ r(U)[:, :LAT])
    out["w2"], out["b2"] = d_lat.T @ S["h1"], d_lat.sum(0)
    dh1 = r((d_lat @ r(P["w"][2])) * (S["h1"] > 0))
    out["w1"], out["b1"] = dh1.T @ S["h0"], dh1.sum(0)
    dh0 = r((dh1 @ r(P["w"][1])) * (S["h0"] > 0))
    out["w0"], out["b0"] = dh0.T @ S["x"], dh0.sum(0)
    out["g_X"] = dh0 @ r(P["w"][0])[:, :LAT]
    return out


def rel_err(a, b):
    """||a - b|| / ||b||"""
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))
