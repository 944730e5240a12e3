// Dense part of the tri-plane builder `GridEncoder.forward` (SURVEY.md section 8(f1); models/neo360/encoder_tp_fusion_conv.py:472-597)
// between the ResNet feature extractor and the three floor-plan conv stacks (both stay in the host framework):
//   world grid 64^3 -> per source view: camera transform, projection, bilinear lookup of the 512-channel latent image (zeros padding),
//   [latent | camera xyz | unit direction to the camera * (z_cam < 1e-3)] -> DepthPillarEncoder 518 -> 512 -> 512 -> 512,
//   three pillar aggregators (Linear 513 -> 512, ReLU, Linear 512 -> 1, softmax along one grid axis) -> weighted pillar sums.
// 786 432 rows per scene at NV = 3: every dense layer runs on the tensor cores through gemm_f16 (csrc/gemm_tc.cu); the gather, the logit
// reduction and the softmax-weighted pillar sum are the kernels below.  fp16 weights / activations, fp32 accumulation and softmax.
#include "common.cuh"
#include <cuda_fp16.h>

namespace neo {
namespace enc {

constexpr int kG = 64, kNC = kG * kG * kG, kLat = 512, kIn = 518, kLd = 576;      // 518 -> 576 (multiple of 64) zero padded

// torch.linspace(a, b, n)[i] (ATen: symmetric evaluation around the midpoint)
__device__ __forceinline__ float lin(float a, float b, int i, int n) {
    const float step = (b - a) / (float)(n - 1);
    return (i < n / 2) ? a + step * (float)i : b - step * (float)(n - 1 - i);
}
__device__ __forceinline__ void cell_xyz(int cell, float* x) {
    const int ix = cell / (kG * kG), iy = (cell / kG) % kG, iz = cell % kG;
    x[0] = lin(-1.f, 1.f, ix, kG); x[1] = lin(-1.f, 1.f, iy, kG); x[2] = lin(0.f, 1.f, iz, kG);     // side_lengths [1,1,1]: z in [0,1]
}

// one block (128 threads = 512 channels / 4) per (view, grid cell): row = [latent lookup (512) | cam xyz (3) | direction (3) | 0 ...]
__global__ void __launch_bounds__(128) grid_gather_kernel(const float* __restrict__ lat_cl, int lh, int lw, const float* __restrict__ poses,
                                                          float focal, float cx, float cy, float sx, float sy, __half* __restrict__ X) {
    const long long row = blockIdx.x;
    const int v = (int)(row / kNC), cell = (int)(row % kNC);
    float xw[3];
    cell_xyz(cell, xw);
    const float* m = poses + 16 * v;                     // camera-to-world
    float cam[3], dir[3];
    for (int r = 0; r < 3; ++r) {
        // rot = c2w[:3,:3]^T ; trans = -(rot @ t) ; cam = rot @ x + trans   (util.py:52-70)
        const float rot0 = m[0 * 4 + r], rot1 = m[1 * 4 + r], rot2 = m[2 * 4 + r];
        const float tr = -(rot0 * m[3] + rot1 * m[7] + rot2 * m[11]);
        cam[r] = (rot0 * xw[0] + rot1 * xw[1] + rot2 * xw[2]) + tr;
    }
    {
        const float d0 = xw[0] - m[3], d1 = xw[1] - m[7], d2 = xw[2] - m[11];
        const float e0 = d0 + 1e-9f, e1 = d1 + 1e-9f, e2 = d2 + 1e-9f;
        const float nrm = sqrtf(e0 * e0 + e1 * e1 + e2 * e2);
        const float mk = (cam[2] < 1e-3f) ? 1.f : 0.f;      // points in front of the camera (-z forward)
        dir[0] = d0 / nrm * mk; dir[1] = d1 / nrm * mk; dir[2] = d2 / nrm * mk;
    }
    // projection (util.py:92-111) with focal (f, -f), then SpatialEncoder.index (encoder_pn.py:101-152): uv * latent_scaling / image_size - 1
    const float z = cam[2] + 1e-9f;
    const float u = (-cam[0] / z) * focal + cx, w = (-cam[1] / z) * (-focal) + cy;
    Taps t;
    bilinear_taps(u * sx - 1.0f, w * sy - 1.0f, lw, lh, t);
    const float* base = lat_cl + (size_t)v * lh * lw * kLat;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int tp = 0; tp < 4; ++tp) {
        const float wt = t.w[tp];
        if (wt != 0.f) {
            const float4 f = __ldg(reinterpret_cast<const float4*>(base + (size_t)t.idx[tp] * kLat) + threadIdx.x);
            acc.x += f.x * wt; acc.y += f.y * wt; acc.z += f.z * wt; acc.w += f.w * wt;
        }
    }
    __half* xr = X + row * kLd;
    __half2 lo = __floats2half2_rn(acc.x, acc.y), hi = __floats2half2_rn(acc.z, acc.w);
    uint2 pk;
    pk.x = *reinterpret_cast<uint32_t*>(&lo); pk.y = *reinterpret_cast<uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(xr + 4 * threadIdx.x) = pk;
    if (threadIdx.x < kLd - kLat) {
        const int c = threadIdx.x;
        const float val = c < 3 ? cam[c] : (c < 6 ? dir[c - 3] : 0.f);
        xr[kLat + c] = __float2half_rn(val);
    }
}

// column 512 of every row = the world coordinate of its cell along `axis` (the aggregator's extra input); columns 513.. = 0
__global__ void coord_col_kernel(__half* __restrict__ L, long long rows, int axis) {
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= rows * (kLd - kLat)) return;
    const long long row = gid / (kLd - kLat);
    const int c = (int)(gid % (kLd - kLat));
    float val = 0.f;
    if (c == 0) {
        float x[3];
        cell_xyz((int)(row % kNC), x);
        val = x[axis];
    }
    L[row * kLd + kLat + c] = __float2half_rn(val);
}

// softmax of the 64 logits of a pillar along `axis` and the weighted sum of its latent rows: out (nv, 512, 64, 64) NCHW, plane dims =
// the two remaining grid axes in (x, y, z) order.  One block (128 threads x 4 channels) per pillar.
__global__ void __launch_bounds__(128) pillar_sum_kernel(const __half* __restrict__ L, const float* __restrict__ logits, int axis, float* __restrict__ out) {
    const int pillar = blockIdx.x % (kG * kG), v = blockIdx.x / (kG * kG);
    const int p = pillar / kG, q = pillar % kG;
    const int stride = axis == 0 ? kG * kG : (axis == 1 ? kG : 1);
    const int base = axis == 0 ? p * kG + q : (axis == 1 ? p * kG * kG + q : (p * kG + q) * kG);
    __shared__ float wsm[kG];
    if (threadIdx.x < kG) wsm[threadIdx.x] = logits[(size_t)v * kNC + base + threadIdx.x * stride];
    __syncthreads();
    float mx = -INFINITY;
    for (int i = 0; i < kG; ++i) mx = fmaxf(mx, wsm[i]);
    float den = 0.f;
    for (int i = 0; i < kG; ++i) den += expf(wsm[i] - mx);
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    for (int i = 0; i < kG; ++i) {
        const float wgt = expf(wsm[i] - mx) / den;
        const uint2 pk = *reinterpret_cast<const uint2*>(L + ((size_t)v * kNC + base + (size_t)i * stride) * kLd + 4 * threadIdx.x);
        const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&pk.x)), f1 = __half22float2(*reinterpret_cast<const __half2*>(&pk.y));
        a0 += wgt * f0.x; a1 += wgt * f0.y; a2 += wgt * f1.x; a3 += wgt * f1.y;
    }
    float* o = out + (((size_t)v * kLat + 4 * threadIdx.x) * kG + p) * kG + q;
    o[0] = a0; o[(size_t)kG * kG] = a1; o[(size_t)2 * kG * kG] = a2; o[(size_t)3 * kG * kG] = a3;
}

struct WS { float* lat_cl; __half *X, *Ha, *Hb, *L, *W; float* logits; };
size_t carve(Carve& c, int nv, int lh, int lw, WS& w) {
    const size_t R = (size_t)nv * kNC;
    w.lat_cl = c.take<float>((size_t)nv * lh * lw * kLat);
    w.X = c.take<__half>(R * kLd);
    w.Ha = c.take<__half>(R * kLat);
    w.Hb = c.take<__half>(R * kLat);
    w.L = c.take<__half>(R * kLd);
    w.W = c.take<__half>((size_t)kLat * kLd + 2 * (size_t)kLat * kLat + 3 * (size_t)kLat * kLd);
    w.logits = c.take<float>(R);
    return c.used;
}

}  // namespace enc
}  // namespace neo

using namespace neo;

extern "C" size_t neo_grid_encoder_workspace_bytes(int nv, int lat_h, int lat_w) {
    if (nv < 1 || lat_h < 2 || lat_w < 2) return 0;
    Carve c{nullptr, 0};
    enc::WS w;
    return enc::carve(c, nv, lat_h, lat_w, w);
}

extern "C" int neo_grid_encoder_dense(const NeoGridEncoderParams* p, const float* latent, int nv, int lat_h, int lat_w, int img_w, int img_h,
                                      const float* src_poses, float focal, float cx, float cy, float* floor_xz, float* floor_xy, float* floor_yz,
                                      void* workspace, size_t workspace_bytes, void* stream) {
    using namespace enc;
    if (!p || !latent || !src_poses || !floor_xz || !floor_xy || !floor_yz || nv < 1 || lat_h < 2 || lat_w < 2 || img_w <= 0 || img_h <= 0) {
        set_error("neo_grid_encoder_dense: bad arguments");
        return NEO_ERR_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    Carve c{static_cast<unsigned char*>(workspace), 0};
    WS w;
    const size_t need = carve(c, nv, lat_h, lat_w, w);
    if (!workspace || workspace_bytes < need) { set_error("workspace too small: need %zu bytes, got %zu", need, workspace_bytes); return NEO_ERR_WORKSPACE; }
    const long long R = (long long)nv * kNC;
    int rc;
    if ((rc = launch_nchw_to_nhwc(latent, w.lat_cl, nv, kLat, lat_h * lat_w, s))) return rc;
    // latent_scaling = size / (size - 1) * 2 ; scale = latent_scaling / image_size   (encoder_pn.py:119, 204-206)
    const float sx = (float)lat_w / ((float)lat_w - 1.0f) * 2.0f / (float)img_w, sy = (float)lat_h / ((float)lat_h - 1.0f) * 2.0f / (float)img_h;
    grid_gather_kernel<<<(unsigned)R, 128, 0, s>>>(w.lat_cl, lat_h, lat_w, src_poses, focal, cx, cy, sx, sy, w.X);
    NEO_LAUNCH_CHECK("grid_gather_kernel");
    // DepthPillarEncoder: 518 -> 512 (ReLU) -> 512 (ReLU) -> 512
    __half* wp = w.W;
    __half* w0 = wp; wp += (size_t)kLat * kLd;
    __half* w1 = wp; wp += (size_t)kLat * kLat;
    __half* w2 = wp; wp += (size_t)kLat * kLat;
    if ((rc = f32_to_f16_pad(p->fc_w[0], kLat, kIn, kIn, w0, kLd, kLd, s))) return rc;
    if ((rc = f32_to_f16_pad(p->fc_w[1], kLat, kLat, kLat, w1, kLat, kLat, s))) return rc;
    if ((rc = f32_to_f16_pad(p->fc_w[2], kLat, kLat, kLat, w2, kLat, kLat, s))) return rc;
    if ((rc = gemm_f16(w.X, kLd, w0, kLd, p->fc_b[0], w.Ha, kLat, R, kLat, kLd, 1, s))) return rc;
    if ((rc = gemm_f16(w.Ha, kLat, w1, kLat, p->fc_b[1], w.Hb, kLat, R, kLat, kLat, 1, s))) return rc;
    if ((rc = gemm_f16(w.Hb, kLat, w2, kLat, p->fc_b[2], w.L, kLd, R, kLat, kLat, 0, s))) return rc;
    // pillar aggregators: yz sums over x (input coordinate x), xz over y, xy over z   (encoder_tp_fusion_conv.py:556-570)
    const float* aw0[3] = {p->agg_yz_w0, p->agg_xz_w0, p->agg_xy_w0};
    const float* ab0[3] = {p->agg_yz_b0, p->agg_xz_b0, p->agg_xy_b0};
    const float* aw1[3] = {p->agg_yz_w1, p->agg_xz_w1, p->agg_xy_w1};
    const float* ab1[3] = {p->agg_yz_b1, p->agg_xz_b1, p->agg_xy_b1};
    float* outs[3] = {floor_yz, floor_xz, floor_xy};
    for (int axis = 0; axis < 3; ++axis) {
        __half* wa = wp; wp += (size_t)kLat * kLd;
        if ((rc = f32_to_f16_pad(aw0[axis], kLat, kLat + 1, kLat + 1, wa, kLd, kLd, s))) return rc;
        coord_col_kernel<<<(unsigned)((R * (kLd - kLat) + 255) / 256), 256, 0, s>>>(w.L, R, axis);
        NEO_LAUNCH_CHECK("coord_col_kernel");
        if ((rc = gemm_f16(w.L, kLd, wa, kLd, ab0[axis], w.Ha, kLat, R, kLat, kLd, 1, s))) return rc;
        if ((rc = launch_rowdot_f16(w.Ha, kLat, kLat, aw1[axis], ab1[axis], 1, R, w.logits, s))) return rc;
        pillar_sum_kernel<<<(unsigned)(nv * kG * kG), 128, 0, s>>>(w.L, w.logits, axis, outs[axis]);
        NEO_LAUNCH_CHECK("pillar_sum_kernel");
    }
    return NEO_OK;
}
