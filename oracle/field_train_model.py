"""Float64 model of the tensor-core training trunk (csrc/field_train.cu, training._TrunkTC) with every bf16 rounding the kernels apply
made explicit, its hand-written adjoint, the per-point head it feeds, and the bounds the GPU tests hold the kernels to.

Forward (rows r = v M + j, point j seen from source view v):
    enc = bf(_pos_enc(cam, 0, 10));  pm = local_p + world_p  (fp32 rows, never rounded)
    h0 = relu(enc bf(W0e)^T + b0 + pm[:, :128]);   h1 = relu(bf(h0) bf(W1)^T + b1);   h2 = relu(bf(h1) bf(W2)^T + b2)
    h3 = relu(bf(h2) bf(W3h)^T + enc bf(W3e)^T + b3 + pm[:, 128:]);   hbar = mean_v h3 (h3 unrounded)
Backward, g = d hbar:
    dz3 = (g / NV)[h3 > 0];  dz2 = (bf(dz3) bf(W3h))[h2 > 0];  dz1 = (bf(dz2) bf(W2))[h1 > 0];  dz0 = (bf(dz1) bf(W1))[h0 > 0]
    d_pm = [dz0 | dz3];  dW0e = bf(dz0)^T enc;  dW1 = bf(dz1)^T bf(h0);  dW2 = bf(dz2)^T bf(h1);  dW3 = bf(dz3)^T [bf(h2) | enc];
    db_l = sum_rows bf(dz_l)
bf() rounds an fp32 value to bf16 (nearest even).  With `rnd=False` every bf() is the identity and the model is training._mlp_projected
re-associated exactly (head on the view mean), which tests/test_field_train_model.py checks in float64.

Bounds, as ||kernel - model|| / ||model|| per tensor (Frobenius).  What remains between the kernels and this model is fp32
accumulation (K <= 224 products of bf16 operands: ~1e-6 relative), bf16 rounding flips where an fp32 value sits within that error of a
rounding boundary (2^-8 of one operand), and ReLU masks that flip where a pre-activation is within that error of zero (the whole
element of that layer's gradient).  Both are rare, so the norm moves by far less than the bounds; a max-entry measure would not do,
one flipped mask moves its entry by all of itself.  The backward chains three products and its masks come from the forward, so
its bound is wider.  Measured on an H100 80GB HBM3 (tests/test_gpu_field_train.py, 900-1000 points, NV 1-5): hbar 5e-5 to 8e-5,
d_pm 7e-4 to 7e-3, weight and bias gradients up to 1.1e-2; every mutation of the catalogue moves some tensor past twice the bound.
"""
import math

import torch

FWD_BOUND = 2e-3
BWD_BOUND = 3e-2
# the whole training step against the "fp32" path: the bf16 roundings themselves.  Measured on the model (tests/test_field_train_model.py,
# 1200 rows): 0.002 on hbar, 0.02-0.08 on the gradients, almost all of it from ReLU masks that flip between the rounded and the exact
# forward (with the forward state held fixed the backward's roundings give 0.002-0.004)
STEP_BOUND = 0.15


def bf(x, on=True):
    return x.float().bfloat16().double() if on else x


def pos_enc(x):
    """training._pos_enc(x, 0, 10) in float64."""
    scales = torch.tensor([2.0 ** i for i in range(10)], dtype=x.dtype)
    xb = (x[..., None, :] * scales[:, None]).reshape(*x.shape[:-1], -1)
    return torch.cat([x, torch.sin(torch.cat([xb, xb + 0.5 * math.pi], -1))], -1)


def forward(cam, local_p, world_p, W, rnd=True, mut=None):
    """cam (NV, M, in_ch), local_p / world_p (NV*M, 256), W = dict(w0e, b0, w1, b1, w2, b2, w3e, b3) float64 -> hbar (M, 128), saved."""
    nv, M, ich = cam.shape
    E = 21 * ich
    r = lambda x: bf(x, rnd)
    enc = r(pos_enc(cam).reshape(nv * M, E))
    if mut == "cos_as_sin":
        enc = r(pos_enc_noshift(cam).reshape(nv * M, E))
    pm = local_p + (0 * world_p if mut == "no_world" else world_p)
    h0 = torch.relu(enc @ r(W["w0e"]).T + W["b0"] + pm[:, :128])
    h1 = torch.relu(r(h0) @ r(W["w1"]).T + (0 if mut == "no_b1" else W["b1"]))
    h2 = torch.relu(r(h1) @ r(W["w2"]).T + W["b2"])
    w3 = r(W["w3e"])
    z3 = r(h2) @ w3[:, :128].T + W["b3"] + pm[:, 128:]
    if mut != "no_w3e":
        z3 = z3 + enc @ w3[:, 128:].T
    h3 = torch.relu(z3)
    hbar = h3.reshape(nv, M, 128)[0] if mut == "view0" else h3.reshape(nv, M, 128).mean(0)
    return hbar, dict(enc=enc, h0=h0, h1=h1, h2=h2, h3=h3, nv=nv)


def pos_enc_noshift(x):
    scales = torch.tensor([2.0 ** i for i in range(10)], dtype=x.dtype)
    xb = (x[..., None, :] * scales[:, None]).reshape(*x.shape[:-1], -1)
    return torch.cat([x, torch.sin(torch.cat([xb, xb], -1))], -1)


def backward(g_hbar, S, W, rnd=True, mut=None):
    """Adjoint of `forward`: g_hbar (M, 128) -> d_pm (NV*M, 256) and dict of weight / bias gradients (nn.Linear layout)."""
    r = lambda x: bf(x, rnd)
    nv = S["nv"]
    g = g_hbar.repeat(nv, 1) / (1 if mut == "no_inv_nv" else nv)
    dz3 = g * (S["h3"] > 0)
    w3 = r(W["w3e"])
    dz2 = r(dz3) @ w3[:, :128]
    if mut != "no_mask2":
        dz2 = dz2 * (S["h2"] > 0)
    dz1 = (r(dz2) @ r(W["w2"])) * (S["h1"] > 0)
    dz0 = (r(dz1) @ r(W["w1"])) * (S["h0"] > 0)
    d_pm = torch.cat([dz0, dz3], -1)
    G = {}
    G["w0e"] = r(dz0).T @ S["enc"]
    G["w1"] = r(dz1).T @ r(S["h1"] if mut == "dw1_wrong_input" else S["h0"])
    G["w2"] = r(dz2).T @ r(S["h1"])
    G["w3e"] = r(dz3).T @ torch.cat([r(S["h2"]), S["enc"]], -1)
    for k, dz in (("b0", dz0), ("b1", dz1), ("b2", dz2), ("b3", dz3)):
        G[k] = r(dz).sum(0)
    return d_pm, G


def head(mlp, hbar, dir_tile, nv):
    """The head of training._mlp_projected_tc: once per point on hbar and the view mean of the direction encodings."""
    lin = lambda m, x: torch.nn.functional.linear(x, m.weight, m.bias)
    M = hbar.shape[0]
    raw_sigma = lin(mlp.density_layer, hbar)
    dbar = dir_tile.reshape(nv, M, -1).mean(0)
    q = lin(mlp.views_linear[0], torch.cat([lin(mlp.bottleneck_layer, hbar), dbar], -1))
    q = torch.relu(lin(mlp.views_linear[1], torch.relu(q)))
    return lin(mlp.rgb_layer, q), raw_sigma


def weights_of(mlp, ich):
    """The trunk inputs of `_TrunkTC` from a NeRFPPMLP (float64 copies)."""
    E = 21 * ich
    p = mlp.pts_linears
    d = lambda t: t.detach().double().clone()
    return dict(w0e=d(p[0].weight[:, :E]), b0=d(p[0].bias), w1=d(p[1].weight), b1=d(p[1].bias), w2=d(p[2].weight), b2=d(p[2].bias),
                w3e=d(p[3].weight[:, :128 + E]), b3=d(p[3].bias))


def rel_err(a, b):
    """||a - b|| / ||b||"""
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


MUTATIONS = ("cos_as_sin", "no_world", "no_b1", "no_w3e", "view0", "no_inv_nv", "no_mask2", "dw1_wrong_input")
