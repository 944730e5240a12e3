"""Float64 model of the tensor-core training form of the vanilla NeRF and Mip-NeRF 360 MLPs (csrc/dense_train.cu, csrc/gemm_tc.cu,
training._MLPTrainTC) with every bf16 rounding the kernels apply made explicit, its hand-written adjoint, and the bounds the GPU tests
hold the kernels to.

Forward, rows r of feats (M, F); layer i has weight w_i (W, K_i), bias b_i; layer 5 of an 8-layer MLP sees [h4 | feats]:
    x_0 = bf(feats);  h_i = relu(x_i bf(w_i)^T + b_i);  x_{i+1} = bf(h_i)  (= [bf(h_4) | x_0] for i = 4 when depth > 5)
    raw_sigma = x_d w_sig^T + b_sig      (w_sig fp32: the bf16 rowdot head)
    beta = bf(x_d bf(w_b)^T + b_b);  y_beta = beta bf(w_vb)^T  (fp32)
    raw_rgb = rgb_layer(relu(y_beta + (denc w_vd^T + b_v) broadcast over the ray's samples))     (fp32 framework ops)
Backward, g_sig (M, 1), g_yb (M, 128):
    dyb = bf(g_yb);  dbeta = bf(dyb bf(w_vb));  dz_{d-1} = bf((dbeta bf(w_b) + g_sig w_sig) [x_d > 0])  (PropMLP: no dbeta term)
    dz_{i-1} = bf((dz_i bf(w_i))[:, :W] [x_i[:, :W] > 0]);  dw_i = dz_i^T x_i;  db_i = sum_rows dz_i
    dw_b = dbeta^T x_d;  db_b = sum_rows dbeta;  dw_vb = dyb^T beta;  dw_sig = bf(g_sig)^T x_d;  db_sig = sum_rows g_sig
bf() rounds an fp32 value to bf16 (nearest even).  The biases, the accumulators and the rank-1 density term stay fp32 and unrounded.
With `rnd=False` every bf() is the identity and the model is vanilla._mlp_train / mip._mlp_train in float64
(tests/test_dense_train_model.py).

Bounds, as ||kernel - model|| / ||model|| per tensor (Frobenius).  One product form against the model at identical rounding points
differs only by fp32 accumulation order (K <= 1536 products: ~1e-6 relative) and the bf16 output roundings it flips (2^-8 of an
element, rare): PRODUCT_BOUND.  The whole MLP adds ReLU masks that flip where a pre-activation sits within that error of zero; each flip
moves a whole element of that layer's gradient, and the 8-layer chain carries them through 7 more products, so the backward bound is
the one field_train uses.  STEP_BOUND holds the whole training step against the "fp32" path: the bf16 roundings themselves.

Measured on an H100 80GB HBM3 at 700 W (tests/test_gpu_dense_train.py): each product form within 6.6e-5 of the model at identical
rounding points (forward 9e-6 to 4.9e-5, dgrad 1.0e-5 to 6.6e-5, wgrad and bias sums 5e-8 to 3.3e-6), so PRODUCT_BOUND stays at its
a-priori 1e-3.  Whole MLPs: vanilla 8 x 256 forward 2.6e-4 to 4.2e-4, gradients up to 7.2e-3; PropMLP 3.5e-4 and 5.2e-3.  The Mip-NeRF 360
8 x 1024 NeRFMLP measures 3.4e-3 forward and 2.2e-2 to 4.0e-2 on the gradients: its products are as exact as the others, but its
Kaiming-initialised 1024-wide layers amplify each layer's rounding flips about 1.7x per layer (the product-level 4e-5 becomes 3.4e-3 after
eight layers and the head), where the Xavier-initialised 256-wide vanilla chain does not.  So that MLP is held to WIDE_FWD_BOUND and
WIDE_BWD_BOUND (2.5 and 2 times the narrow ones), and every mutation of the catalogue still moves some tensor past twice the wide bounds.
"""
import torch

PRODUCT_BOUND = 1e-3
FWD_BOUND = 2e-3
BWD_BOUND = 3e-2
WIDE_FWD_BOUND = 5e-3            # the 8 x 1024 Mip-NeRF 360 NeRFMLP: see above
WIDE_BWD_BOUND = 6e-2
STEP_BOUND = 0.15


def bf(x, on=True):
    return x.float().bfloat16().double() if on else x


def params_of(m):
    """float64 copies of the parameters of vanilla.NeRFMLP, mip.PropMLP or mip.NeRFMLP."""
    d = lambda t: t.detach().double().clone()
    layers = m.pts_linears if hasattr(m, "pts_linears") else m.pts_linear
    P = {"w": [d(l.weight) for l in layers], "b": [d(l.bias) for l in layers], "wsig": d(m.density_layer.weight),
         "bsig": d(m.density_layer.bias)}
    if hasattr(m, "rgb_layer"):
        kb = m.bottleneck_layer.out_features
        v = m.views_linear[0]
        P.update(wb=d(m.bottleneck_layer.weight), bb=d(m.bottleneck_layer.bias), wvb=d(v.weight[:, :kb]), wvd=d(v.weight[:, kb:]),
                 bv=d(v.bias), wrgb=d(m.rgb_layer.weight), brgb=d(m.rgb_layer.bias))
    return P


def forward(feats, P, rnd=True, mut=None):
    """feats (M, F) float64 -> raw_sigma (M, 1), y_beta (M, 128) or None, saved state."""
    r = lambda x: bf(x, rnd)
    depth = len(P["w"])
    e = r(feats)
    x = e
    X = []
    for i in range(depth):
        X.append(x)
        z = x @ r(P["w"][i]).T
        h = torch.relu(z) + P["b"][i] if mut == "bias_after_relu" else torch.relu(z + P["b"][i])
        x = r(h)
        if i == 4 and depth > 5:
            x = torch.cat([x, 0 * e if mut == "no_skip" else e], -1)
    sig = x @ P["wsig"].T + P["bsig"]
    S = dict(X=X, xd=x)
    if "wb" not in P:
        return sig, None, S
    beta = r(x @ r(P["wb"]).T + P["bb"])
    S["beta"] = beta
    return sig, beta @ r(P["wvb"]).T, S


def head(yb, denc, P, n, N):
    """the fp32 framework ops after y_beta: raw rgb (n, N, 3)."""
    y = yb.reshape(n, N, -1) + (denc @ P["wvd"].T + P["bv"])[:, None, :]
    return torch.relu(y) @ P["wrgb"].T + P["brgb"]


def backward(g_sig, g_yb, S, P, rnd=True, mut=None):
    """Adjoint of `forward`: -> dict of gradients (nn.Linear layout; "wvb" the beta columns of views_linear.0)."""
    r = lambda x: bf(x, rnd)
    depth, W = len(P["w"]), P["w"][0].shape[0]
    xd = S["xd"]
    G = {}
    dh = 0 if mut == "no_density_addend" else g_sig @ P["wsig"]
    if "wb" in P:
        dyb = r(g_yb)
        G["wvb"] = dyb.T @ S["beta"]
        dbeta = r(dyb @ r(P["wvb"]))
        G["wb"], G["bb"] = dbeta.T @ xd, dbeta.sum(0)
        dh = dh + dbeta @ r(P["wb"])
    dz = r(dh * (xd > 0))
    G["wsig"], G["bsig"] = r(g_sig).T @ xd, g_sig.sum(0)
    for i in range(depth - 1, -1, -1):
        X = S["X"][i]
        G[f"w{i}"] = dz.T @ (S["X"][1] if mut == "wgrad_wrong_input" and i == 2 else X)
        G[f"b{i}"] = dz.sum(0)
        if i > 0:
            d = (dz @ r(P["w"][i]))[:, :W]
            dz = r(d if mut == "no_relu_mask" else d * (X[:, :W] > 0))
    return G


def rel_err(a, b):
    """||a - b|| / ||b||"""
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


MUTATIONS = ("no_skip", "no_relu_mask", "wgrad_wrong_input", "no_density_addend", "bias_after_relu")
