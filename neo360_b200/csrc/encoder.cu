// Dense part of the tri-plane builder `GridEncoder.forward` (SURVEY.md section 8(f1); models/neo360/encoder_tp_fusion_conv.py:472-597)
// between the ResNet feature extractor and the three floor-plan conv stacks (both stay in the host framework):
//   world grid 64^3 -> per source view: camera transform, projection, bilinear lookup of the 512-channel latent image (zeros padding),
//   [latent | camera xyz | unit direction to the camera * (z_cam < 1e-3)] -> DepthPillarEncoder 518 -> 512 -> 512 -> 512,
//   three pillar aggregators (Linear 513 -> 512, ReLU, Linear 512 -> 1, softmax along one grid axis) -> weighted pillar sums.
// 786 432 rows per scene at NV = 3: every dense layer runs on the tensor cores through gemm_f16 (csrc/gemm_tc.cu); the gather, the logit
// reduction and the softmax-weighted pillar sum are the kernels below.  fp16 weights / activations, fp32 accumulation and softmax.
// Training (GridEncoder.dense_train) uses the same gather and pillar-sum kernels in fp32, their backward kernels below, and the host
// framework's GEMMs for the dense layers.  Its tensor-core form (GridEncoder.dense_train_tc) uses their bf16 instances around gemm_tc.cu's
// bf16 products: lookup rows and the latent buffer L = [lat | x y z | 0] (coords_kernel) in bf16, the pillar sums and their backward
// reading lat from L, and lat_grad_kernel joining the pool's and the aggregators' latent gradients.
#include "common.cuh"
#include <cuda_fp16.h>
#include <cuda_bf16.h>

namespace neo {
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

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

// What one grid cell `row` = v * 64^3 + cell looks like from source view v: camera xyz, unit direction to the camera masked to the
// points in front of it, and the four bilinear taps of its latent lookup.  The lookup's forward and backward both take their taps from
// here, so a cell's backward taps are its forward taps bit for bit.
struct CellView { float cam[3], dir[3]; Taps t; };
__device__ __forceinline__ void cell_view(long long row, int lh, int lw, const float* __restrict__ poses, float focal, float cx, float cy,
                                          float sx, float sy, CellView& o) {
    const int v = (int)(row / kNC), cell = (int)(row % kNC);
    float xw[3];
    cell_xyz(cell, xw);
    const float* m = poses + 16 * v;                     // camera-to-world
    for (int r = 0; r < 3; ++r) {
        // rot = c2w[:3,:3]^T ; trans = -(rot @ t) ; cam = rot @ x + trans   (util.py:52-70)
        const float rot0 = m[0 * 4 + r], rot1 = m[1 * 4 + r], rot2 = m[2 * 4 + r];
        const float tr = -(rot0 * m[3] + rot1 * m[7] + rot2 * m[11]);
        o.cam[r] = (rot0 * xw[0] + rot1 * xw[1] + rot2 * xw[2]) + tr;
    }
    {
        const float d0 = xw[0] - m[3], d1 = xw[1] - m[7], d2 = xw[2] - m[11];
        const float e0 = d0 + 1e-9f, e1 = d1 + 1e-9f, e2 = d2 + 1e-9f;
        const float nrm = sqrtf(e0 * e0 + e1 * e1 + e2 * e2);
        const float mk = (o.cam[2] < 1e-3f) ? 1.f : 0.f;    // points in front of the camera (-z forward)
        o.dir[0] = d0 / nrm * mk; o.dir[1] = d1 / nrm * mk; o.dir[2] = d2 / nrm * mk;
    }
    // projection (util.py:92-111) with focal (f, -f), then SpatialEncoder.index (encoder_pn.py:101-152): uv * latent_scaling / image_size - 1
    const float z = o.cam[2] + 1e-9f;
    const float u = (-o.cam[0] / z) * focal + cx, w = (-o.cam[1] / z) * (-focal) + cy;
    bilinear_taps(u * sx - 1.0f, w * sy - 1.0f, lw, lh, o.t);
}

__device__ __forceinline__ void store4(float* p, float4 a) { *reinterpret_cast<float4*>(p) = a; }
__device__ __forceinline__ void store4(__half* p, float4 a) {
    __half2 lo = __floats2half2_rn(a.x, a.y), hi = __floats2half2_rn(a.z, a.w);
    uint2 pk;
    pk.x = *reinterpret_cast<uint32_t*>(&lo); pk.y = *reinterpret_cast<uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(p) = pk;
}
__device__ __forceinline__ void store4(__nv_bfloat16* p, float4 a) {
    __nv_bfloat162 lo = __floats2bfloat162_rn(a.x, a.y), hi = __floats2bfloat162_rn(a.z, a.w);
    uint2 pk;
    pk.x = *reinterpret_cast<uint32_t*>(&lo); pk.y = *reinterpret_cast<uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(p) = pk;
}
__device__ __forceinline__ float4 load4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 load4(const __half* p) {
    const uint2 pk = *reinterpret_cast<const uint2*>(p);
    const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&pk.x)), f1 = __half22float2(*reinterpret_cast<const __half2*>(&pk.y));
    return make_float4(f0.x, f0.y, f1.x, f1.y);
}
__device__ __forceinline__ float4 load4(const __nv_bfloat16* p) {
    const uint2 pk = *reinterpret_cast<const uint2*>(p);
    const float2 f0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&pk.x));
    const float2 f1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&pk.y));
    return make_float4(f0.x, f0.y, f1.x, f1.y);
}
__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }

// one block (128 threads = 512 channels / 4) per (view, grid cell): row (stride ld, 518 <= ld <= 640) =
// [latent lookup (512) | cam xyz (3) | direction (3) | 0 ...].  T = __half: the tensor-core eval path; T = float: the training path;
// T = __nv_bfloat16: its tensor-core form (every element the fp32 instance's value rounded once).
template <class T>
__global__ void __launch_bounds__(128) grid_gather_kernel(const float* __restrict__ lat_cl, int lh, int lw, const float* __restrict__ poses,
                                                          float focal, float cx, float cy, float sx, float sy, T* __restrict__ X, int ld) {
    const long long row = blockIdx.x;
    CellView cv;
    cell_view(row, lh, lw, poses, focal, cx, cy, sx, sy, cv);
    const float* base = lat_cl + (size_t)(row / kNC) * lh * lw * kLat;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int tp = 0; tp < 4; ++tp) {
        const float wt = cv.t.w[tp];
        if (wt != 0.f) {
            const float4 f = __ldg(reinterpret_cast<const float4*>(base + (size_t)cv.t.idx[tp] * kLat) + threadIdx.x);
            acc.x += f.x * wt; acc.y += f.y * wt; acc.z += f.z * wt; acc.w += f.w * wt;
        }
    }
    T* xr = X + row * ld;
    store4(xr + 4 * threadIdx.x, acc);
    if (threadIdx.x < ld - kLat) {
        const int c = threadIdx.x;
        const float val = c < 3 ? cv.cam[c] : (c < 6 ? cv.dir[c - 3] : 0.f);
        xr[kLat + c] = from_f32<T>(val);
    }
}

// adjoint of the lookup columns of grid_gather_kernel<float>: g_lat_cl[v][tap texel][:] += w_tap * g_X[row][0..512) with the 16-byte
// vector reductions of index_bwd_kernel (csrc/field_fp32.cu).  g_X rows (stride ldg, even) are read as float2 pairs: autograd hands the
// gradient of a (R, 518) input over with a row stride of 518.
__global__ void __launch_bounds__(128) grid_gather_bwd_kernel(int lh, int lw, const float* __restrict__ poses, float focal, float cx, float cy,
                                                              float sx, float sy, const float* __restrict__ gX, long long ldg, float* __restrict__ g_lat) {
    const long long row = blockIdx.x;
    CellView cv;
    cell_view(row, lh, lw, poses, focal, cx, cy, sx, sy, cv);
    const float2* g = reinterpret_cast<const float2*>(gX + row * ldg) + 2 * threadIdx.x;
    const float2 a = g[0], b = g[1];
    float* base = g_lat + (size_t)(row / kNC) * lh * lw * kLat;
#pragma unroll
    for (int tp = 0; tp < 4; ++tp) {
        const float w = cv.t.w[tp];
        if (w != 0.f) atomicAdd(reinterpret_cast<float4*>(base + (size_t)cv.t.idx[tp] * kLat) + threadIdx.x, make_float4(a.x * w, a.y * w, b.x * w, b.y * w));
    }
}

// entries of the same adjoint for the order-fixed scatter (csrc/det.cu): e = row*4 + tap, key = v*lh*lw + texel, or T for a zero weight
__global__ void grid_gather_entries_kernel(long long rows, int lh, int lw, const float* __restrict__ poses, float focal, float cx, float cy,
                                           float sx, float sy, unsigned T, unsigned* __restrict__ keys, unsigned* __restrict__ ids,
                                           float* __restrict__ wts) {
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= rows) return;
    CellView cv;
    cell_view(row, lh, lw, poses, focal, cx, cy, sx, sy, cv);
    const unsigned base = (unsigned)(row / kNC) * lh * lw;
#pragma unroll
    for (int tp = 0; tp < 4; ++tp) {
        const unsigned e = (unsigned)row * 4 + tp;
        const float w = cv.t.w[tp];
        keys[e] = w != 0.f ? base + cv.t.idx[tp] : T;
        ids[e] = e;
        wts[e] = w;
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

// columns 512, 513, 514 of every row (stride ld) = the world x, y, z of its cell in bf16, columns 515..ld-1 = 0: the coordinate inputs of
// the three aggregators' stacked first layer (aggregator a reads column 512 + a)
__global__ void coords_kernel(__nv_bfloat16* __restrict__ L, long long rows, int ld) {
    const int w = ld - kLat;
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= rows * w) return;
    const long long row = gid / w;
    const int c = (int)(gid % w);
    float x[3];
    cell_xyz((int)(row % kNC), x);
    L[row * ld + kLat + c] = __float2bfloat16_rn(c == 0 ? x[0] : c == 1 ? x[1] : c == 2 ? x[2] : 0.f);
}

// d_lat (rows, 512) bf16 = bf16(d_pool + d_agg), both fp32 (rows, 512): the latent gradient of the tensor-core training form, rounded once
__global__ void lat_grad_kernel(const float4* __restrict__ a, const float4* __restrict__ b, long long n4, uint2* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const float4 x = a[i], y = b[i];
    __nv_bfloat162 lo = __floats2bfloat162_rn(x.x + y.x, x.y + y.y), hi = __floats2bfloat162_rn(x.z + y.z, x.w + y.w);
    uint2 pk;
    pk.x = *reinterpret_cast<uint32_t*>(&lo); pk.y = *reinterpret_cast<uint32_t*>(&hi);
    out[i] = pk;
}

// The 64 cells of pillar (p, q) along `axis` (plane dims = the two remaining grid axes in (x, y, z) order): cell i = base + i * stride.
__device__ __forceinline__ void pillar_cells(int axis, int p, int q, int& base, int& stride) {
    stride = axis == 0 ? kG * kG : (axis == 1 ? kG : 1);
    base = axis == 0 ? p * kG + q : (axis == 1 ? p * kG * kG + q : (p * kG + q) * kG);
}
// max and softmax denominator of a pillar's 64 logits (every thread scans them in the same order)
__device__ __forceinline__ void pillar_softmax(const float* wsm, float& mx, float& den) {
    mx = -INFINITY;
    for (int i = 0; i < kG; ++i) mx = fmaxf(mx, wsm[i]);
    den = 0.f;
    for (int i = 0; i < kG; ++i) den += expf(wsm[i] - mx);
}

// softmax of the 64 logits of a pillar along `axis` and the weighted sum of its latent rows (row stride ld): out (nv, 512, 64, 64) NCHW.
// One block (128 threads x 4 channels) per pillar.  T = __half: the eval path's L; T = float: the training path's depth_fc output;
// T = __nv_bfloat16: the latent columns of its tensor-core form's L.
template <class T>
__global__ void __launch_bounds__(128) pillar_sum_kernel(const T* __restrict__ L, int ld, const float* __restrict__ logits, int axis, float* __restrict__ out) {
    const int pillar = blockIdx.x % (kG * kG), v = blockIdx.x / (kG * kG);
    const int p = pillar / kG, q = pillar % kG;
    int base, stride;
    pillar_cells(axis, p, q, base, stride);
    __shared__ float wsm[kG];
    if (threadIdx.x < kG) wsm[threadIdx.x] = logits[(size_t)v * kNC + base + threadIdx.x * stride];
    __syncthreads();
    float mx, den;
    pillar_softmax(wsm, mx, den);
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    for (int i = 0; i < kG; ++i) {
        const float wgt = expf(wsm[i] - mx) / den;
        const float4 f = load4(L + ((size_t)v * kNC + base + (size_t)i * stride) * ld + 4 * threadIdx.x);
        a0 += wgt * f.x; a1 += wgt * f.y; a2 += wgt * f.z; a3 += wgt * f.w;
    }
    float* o = out + (((size_t)v * kLat + 4 * threadIdx.x) * kG + p) * kG + q;
    o[0] = a0; o[(size_t)kG * kG] = a1; o[(size_t)2 * kG * kG] = a2; o[(size_t)3 * kG * kG] = a3;
}

// ---- backward of the pillar sums: out_a[v, c, p, q] = sum_i s_i lat[cell_i, c], s = softmax over the pillar's logits ----
//   d_lat[r, c]    = sum_a s_a(r) g_a[v, c, plane_a(r)]                                 (every element written once, no atomics)
//   d_logits[a, r] = s_a(r) (gl_a(r) - sum_{j in pillar_a(r)} s_a(j) gl_a(j)),  gl_a(r) = sum_c g_a[v, c, plane_a(r)] lat[r, c]
// Three launches: (1) s of the yz (axis 0) and xz (axis 1) pillars into d_logits[0..1]; (2) one block per xy pillar (64 consecutive
// rows, iz = 0..63): d_lat, gl of the three axes, the finished xy d_logits, gl of axes 0 / 1 into d_logits[0..1] (replacing s); (3) the
// yz / xz pillars again: d_logits = s (gl - sum s gl).  Fixed summation orders throughout: two calls give bit-identical results.

// launches (1) and (3): one block of 64 threads (one per cell) per pillar of axis blockIdx.y (0 or 1)
__global__ void __launch_bounds__(64) pillar_softmax_bwd_kernel(const float* __restrict__ logits, float* __restrict__ dl, long long R, int finish) {
    const int axis = blockIdx.y, pillar = blockIdx.x % (kG * kG), v = blockIdx.x / (kG * kG);
    int base, stride;
    pillar_cells(axis, pillar / kG, pillar % kG, base, stride);
    const size_t r = (size_t)v * kNC + base + (size_t)threadIdx.x * stride;
    __shared__ float wsm[kG], sg[kG];
    wsm[threadIdx.x] = logits[axis * R + r];
    __syncthreads();
    float mx, den;
    pillar_softmax(wsm, mx, den);
    const float s = expf(wsm[threadIdx.x] - mx) / den;
    if (!finish) { dl[axis * R + r] = s; return; }
    const float gl = dl[axis * R + r];
    sg[threadIdx.x] = s * gl;
    __syncthreads();
    float S = 0.f;
    for (int i = 0; i < kG; ++i) S += sg[i];
    dl[axis * R + r] = s * (gl - S);
}

// launch (2): 256 threads per xy pillar (v, ix, iy); channels in chunks of 32, lane = channel, warp w = rows iz = w, w + 8, ...
// lat rows have stride ld (T = float: the fp32 training path, ld 512; T = __nv_bfloat16: its tensor-core form's L); d_lat has stride 512.
template <class T>
__global__ void __launch_bounds__(256) pool_bwd_rows_kernel(const T* __restrict__ lat, long long ld, const float* __restrict__ logits, const float* __restrict__ g_yz,
                                                            const float* __restrict__ g_xz, const float* __restrict__ g_xy, float* __restrict__ d_lat,
                                                            float* __restrict__ dl, long long R) {
    constexpr int kCh = 32, kRows = kG / 8;
    const int v = blockIdx.x / (kG * kG), ix = (blockIdx.x / kG) % kG, iy = blockIdx.x % kG;
    const size_t r0 = (size_t)v * kNC + (size_t)(ix * kG + iy) * kG;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __shared__ float s[3][kG], gl[3][kG], g0[kCh][kG + 1], g1[kCh][kG + 1], g2[kCh];
    if (threadIdx.x < kG) {
        s[0][threadIdx.x] = dl[r0 + threadIdx.x];
        s[1][threadIdx.x] = dl[R + r0 + threadIdx.x];
        s[2][threadIdx.x] = logits[2 * R + r0 + threadIdx.x];
    }
    __syncthreads();
    float e2 = 0.f;
    if (threadIdx.x < kG) {
        float mx, den;
        pillar_softmax(s[2], mx, den);
        e2 = expf(s[2][threadIdx.x] - mx) / den;
    }
    __syncthreads();        // every thread has read the xy logits before they are replaced by their softmax
    if (threadIdx.x < kG) s[2][threadIdx.x] = e2;
    __syncthreads();
    float acc[3][kRows];
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int k = 0; k < kRows; ++k) acc[a][k] = 0.f;
    for (int c0 = 0; c0 < kLat; c0 += kCh) {
        // g_yz[v, c, iy, iz] and g_xz[v, c, ix, iz]: 64 consecutive floats per channel
        for (int e = threadIdx.x; e < kCh * kG; e += blockDim.x) {
            const int c = e / kG, iz = e % kG;
            const size_t cc = (size_t)v * kLat + c0 + c;
            g0[c][iz] = g_yz ? g_yz[(cc * kG + iy) * kG + iz] : 0.f;
            g1[c][iz] = g_xz ? g_xz[(cc * kG + ix) * kG + iz] : 0.f;
        }
        if (threadIdx.x < kCh) g2[threadIdx.x] = g_xy ? g_xy[(((size_t)v * kLat + c0 + threadIdx.x) * kG + ix) * kG + iy] : 0.f;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < kRows; ++k) {
            const int iz = warp + 8 * k;
            const size_t e = (r0 + iz) * kLat + c0 + lane;
            const float x = to_f32(lat[(r0 + iz) * ld + c0 + lane]), a0 = g0[lane][iz], a1 = g1[lane][iz], a2 = g2[lane];
            d_lat[e] = (s[0][iz] * a0 + s[1][iz] * a1) + s[2][iz] * a2;
            acc[0][k] += a0 * x; acc[1][k] += a1 * x; acc[2][k] += a2 * x;
        }
        __syncthreads();
    }
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int k = 0; k < kRows; ++k) {
            const float t = warp_sum(acc[a][k]);
            if (lane == 0) gl[a][warp + 8 * k] = t;
        }
    __syncthreads();
    if (threadIdx.x < kG) {
        const int i = threadIdx.x;
        float S = 0.f;
        for (int j = 0; j < kG; ++j) S += s[2][j] * gl[2][j];
        dl[r0 + i] = gl[0][i];
        dl[R + r0 + i] = gl[1][i];
        dl[2 * R + r0 + i] = s[2][i] * (gl[2][i] - S);
    }
}

// latent_scaling = size / (size - 1) * 2 ; scale = latent_scaling / image_size   (encoder_pn.py:119, 204-206)
inline void lat_scale(int lat_h, int lat_w, int img_w, int img_h, float& sx, float& sy) {
    sx = (float)lat_w / ((float)lat_w - 1.0f) * 2.0f / (float)img_w;
    sy = (float)lat_h / ((float)lat_h - 1.0f) * 2.0f / (float)img_h;
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
    float sx, sy;
    lat_scale(lat_h, lat_w, img_w, img_h, sx, sy);
    grid_gather_kernel<__half><<<(unsigned)R, 128, 0, s>>>(w.lat_cl, lat_h, lat_w, src_poses, focal, cx, cy, sx, sy, w.X, kLd);
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
        pillar_sum_kernel<__half><<<(unsigned)(nv * kG * kG), 128, 0, s>>>(w.L, kLd, w.logits, axis, outs[axis]);
        NEO_LAUNCH_CHECK("pillar_sum_kernel");
    }
    return NEO_OK;
}

// ---- training path (fp32): stage-level entry points, caller-owned buffers, asynchronous on `stream`, nothing allocated ----

static bool enc_geometry_ok(const char* who, int nv, int lat_h, int lat_w, int img_w, int img_h, const float* poses) {
    if (!poses || nv < 1 || lat_h < 2 || lat_w < 2 || img_w <= 0 || img_h <= 0) {
        set_error("%s: bad arguments (nv %d, latent %dx%d, image %dx%d)", who, nv, lat_h, lat_w, img_w, img_h);
        return false;
    }
    return true;
}
static bool aligned(const void* p, size_t a) { return ((uintptr_t)p & (a - 1)) == 0; }

extern "C" int neo_grid_encoder_features(const float* latent_cl, int nv, int lat_h, int lat_w, int img_w, int img_h, const float* src_poses,
                                         float focal, float cx, float cy, float* X, int ldx, void* stream) {
    using namespace enc;
    if (!enc_geometry_ok("neo_grid_encoder_features", nv, lat_h, lat_w, img_w, img_h, src_poses)) return NEO_ERR_INVALID;
    if (!latent_cl || !X || ldx < kIn || ldx > kLat + 128 || ldx % 4 || !aligned(latent_cl, 16) || !aligned(X, 16)) {
        set_error("neo_grid_encoder_features: NULL or unaligned buffer, or row stride %d outside [518, 640] or not a multiple of 4", ldx);
        return NEO_ERR_INVALID;
    }
    float sx, sy;
    lat_scale(lat_h, lat_w, img_w, img_h, sx, sy);
    grid_gather_kernel<float><<<(unsigned)((long long)nv * kNC), 128, 0, (cudaStream_t)stream>>>(latent_cl, lat_h, lat_w, src_poses, focal, cx, cy,
                                                                                                sx, sy, X, ldx);
    NEO_LAUNCH_CHECK("grid_gather_kernel<float>");
    return NEO_OK;
}

extern "C" int neo_grid_encoder_features_bwd(int nv, int lat_h, int lat_w, int img_w, int img_h, const float* src_poses, float focal, float cx,
                                             float cy, const float* g_X, long long ldg, float* g_latent_cl, void* stream) {
    using namespace enc;
    if (!enc_geometry_ok("neo_grid_encoder_features_bwd", nv, lat_h, lat_w, img_w, img_h, src_poses)) return NEO_ERR_INVALID;
    if (!g_X || !g_latent_cl || ldg < kLat || ldg % 2 || !aligned(g_X, 8) || !aligned(g_latent_cl, 16)) {
        set_error("neo_grid_encoder_features_bwd: NULL buffer, g_X not 8-byte aligned with an even row stride >= 512 (got %lld), or the "
                  "gradient map not 16-byte aligned", ldg);
        return NEO_ERR_INVALID;
    }
    float sx, sy;
    lat_scale(lat_h, lat_w, img_w, img_h, sx, sy);
    grid_gather_bwd_kernel<<<(unsigned)((long long)nv * kNC), 128, 0, (cudaStream_t)stream>>>(lat_h, lat_w, src_poses, focal, cx, cy, sx, sy, g_X,
                                                                                              ldg, g_latent_cl);
    NEO_LAUNCH_CHECK("grid_gather_bwd_kernel");
    return NEO_OK;
}

// E = nv * 64^3 * 4 entries, T = nv * lat_h * lat_w texels
static bool features_det_sizes(const char* who, int nv, int lat_h, int lat_w, long long& E, long long& T) {
    E = 4LL * nv * enc::kNC;
    T = (long long)nv * lat_h * lat_w;
    if (nv < 1 || lat_h < 2 || lat_w < 2 || E >= (1LL << 31) - 1 || T >= (1LL << 31) - 1) {
        set_error("%s: bad sizes (nv %d, latent %dx%d) or more than 2^31 - 2 entries", who, nv, lat_h, lat_w);
        return false;
    }
    return true;
}

extern "C" size_t neo_grid_encoder_features_bwd_det_workspace_bytes(int nv, int lat_h, int lat_w) {
    long long E, T;
    if (!features_det_sizes("neo_grid_encoder_features_bwd_det_workspace_bytes", nv, lat_h, lat_w, E, T)) return 0;
    return det_carve(nullptr, E, T).total;
}

extern "C" int neo_grid_encoder_features_bwd_det(int nv, int lat_h, int lat_w, int img_w, int img_h, const float* src_poses, float focal, float cx,
                                                 float cy, const float* g_X, long long ldg, float* g_latent_cl, void* workspace,
                                                 size_t workspace_bytes, void* stream) {
    using namespace enc;
    if (!enc_geometry_ok("neo_grid_encoder_features_bwd_det", nv, lat_h, lat_w, img_w, img_h, src_poses)) return NEO_ERR_INVALID;
    if (!g_X || !g_latent_cl || !workspace || ldg < kLat || ldg % 2 || !aligned(g_X, 8) || !aligned(g_latent_cl, 16) || !aligned(workspace, 16)) {
        set_error("neo_grid_encoder_features_bwd_det: NULL buffer, g_X not 8-byte aligned with an even row stride >= 512 (got %lld), or the "
                  "gradient map / workspace not 16-byte aligned", ldg);
        return NEO_ERR_INVALID;
    }
    long long E, T;
    if (!features_det_sizes("neo_grid_encoder_features_bwd_det", nv, lat_h, lat_w, E, T)) return NEO_ERR_INVALID;
    const DetBuffers b = det_carve(workspace, E, T);
    if (!b.total) return NEO_ERR_CUDA;
    if (workspace_bytes < b.total) {
        set_error("neo_grid_encoder_features_bwd_det: workspace of %zu bytes, %zu needed", workspace_bytes, b.total);
        return NEO_ERR_INVALID;
    }
    float sx, sy;
    lat_scale(lat_h, lat_w, img_w, img_h, sx, sy);
    cudaStream_t s = (cudaStream_t)stream;
    const long long rows = (long long)nv * kNC;
    grid_gather_entries_kernel<<<(unsigned)((rows + 127) / 128), 128, 0, s>>>(rows, lat_h, lat_w, src_poses, focal, cx, cy, sx, sy, (unsigned)T,
                                                                             b.keys, b.ids, b.wts);
    NEO_LAUNCH_CHECK("grid_gather_entries_kernel");
    const DetSrc src{{g_X, g_X}, {ldg, ldg}, {0u, 0xffffffffu}, {4, 4}};
    const DetDst dst{{g_latent_cl, g_latent_cl, g_latent_cl, g_latent_cl}, {0, T, T, T}};
    return det_sort_reduce(b, E, T, kLat, 2, src, dst, s);
}

extern "C" int neo_grid_encoder_pool(const float* lat, const float* logits, int nv, float* floor_xz, float* floor_xy, float* floor_yz, void* stream) {
    using namespace enc;
    if (!lat || !logits || !floor_xz || !floor_xy || !floor_yz || nv < 1 || !aligned(lat, 16)) {
        set_error("neo_grid_encoder_pool: bad arguments (NULL buffer, nv %d < 1 or lat not 16-byte aligned)", nv);
        return NEO_ERR_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const long long R = (long long)nv * kNC;
    float* outs[3] = {floor_yz, floor_xz, floor_xy};
    for (int axis = 0; axis < 3; ++axis) {
        pillar_sum_kernel<float><<<(unsigned)(nv * kG * kG), 128, 0, s>>>(lat, kLat, logits + axis * R, axis, outs[axis]);
        NEO_LAUNCH_CHECK("pillar_sum_kernel<float>");
    }
    return NEO_OK;
}

extern "C" int neo_grid_encoder_pool_bwd(const float* lat, const float* logits, int nv, const float* g_xz, const float* g_xy, const float* g_yz,
                                         float* d_lat, float* d_logits, void* stream) {
    using namespace enc;
    if (!lat || !logits || !d_lat || !d_logits || nv < 1) {
        set_error("neo_grid_encoder_pool_bwd: bad arguments (NULL buffer or nv %d < 1)", nv);
        return NEO_ERR_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const long long R = (long long)nv * kNC;
    pillar_softmax_bwd_kernel<<<dim3((unsigned)(nv * kG * kG), 2), kG, 0, s>>>(logits, d_logits, R, 0);
    NEO_LAUNCH_CHECK("pillar_softmax_bwd_kernel");
    pool_bwd_rows_kernel<float><<<(unsigned)(nv * kG * kG), 256, 0, s>>>(lat, kLat, logits, g_yz, g_xz, g_xy, d_lat, d_logits, R);
    NEO_LAUNCH_CHECK("pool_bwd_rows_kernel");
    pillar_softmax_bwd_kernel<<<dim3((unsigned)(nv * kG * kG), 2), kG, 0, s>>>(logits, d_logits, R, 1);
    NEO_LAUNCH_CHECK("pillar_softmax_bwd_kernel");
    return NEO_OK;
}

// ---- tensor-core training form (bf16 rows; GridEncoder.dense_train_tc): same contracts as the fp32 entries above ----

extern "C" int neo_grid_encoder_features_bf16(const float* latent_cl, int nv, int lat_h, int lat_w, int img_w, int img_h, const float* src_poses,
                                              float focal, float cx, float cy, void* X, int ldx, void* stream) {
    using namespace enc;
    if (!enc_geometry_ok("neo_grid_encoder_features_bf16", nv, lat_h, lat_w, img_w, img_h, src_poses)) return NEO_ERR_INVALID;
    if (!latent_cl || !X || ldx < kIn || ldx > kLat + 128 || ldx % 8 || !aligned(latent_cl, 16) || !aligned(X, 16)) {
        set_error("neo_grid_encoder_features_bf16: NULL or unaligned buffer, or row stride %d outside [518, 640] or not a multiple of 8", ldx);
        return NEO_ERR_INVALID;
    }
    float sx, sy;
    lat_scale(lat_h, lat_w, img_w, img_h, sx, sy);
    grid_gather_kernel<__nv_bfloat16><<<(unsigned)((long long)nv * kNC), 128, 0, (cudaStream_t)stream>>>(latent_cl, lat_h, lat_w, src_poses, focal,
                                                                                                        cx, cy, sx, sy, (__nv_bfloat16*)X, ldx);
    NEO_LAUNCH_CHECK("grid_gather_kernel<bf16>");
    return NEO_OK;
}

extern "C" int neo_grid_encoder_coords_bf16(void* L, int nv, int ld, void* stream) {
    using namespace enc;
    if (!L || nv < 1 || ld < kLat + 3 || ld > kLat + 128 || ld % 8 || !aligned(L, 16)) {
        set_error("neo_grid_encoder_coords_bf16: NULL or unaligned buffer, nv %d < 1, or row stride %d outside [520, 640] or not a multiple of 8",
                  nv, ld);
        return NEO_ERR_INVALID;
    }
    const long long rows = (long long)nv * kNC, n = rows * (ld - kLat);
    coords_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>((__nv_bfloat16*)L, rows, ld);
    NEO_LAUNCH_CHECK("coords_kernel");
    return NEO_OK;
}

extern "C" int neo_grid_encoder_pool_bf16(const void* lat, long long ld, const float* logits, int nv, float* floor_xz, float* floor_xy,
                                          float* floor_yz, void* stream) {
    using namespace enc;
    if (!lat || !logits || !floor_xz || !floor_xy || !floor_yz || nv < 1 || ld < kLat || ld % 8 || !aligned(lat, 16)) {
        set_error("neo_grid_encoder_pool_bf16: bad arguments (NULL buffer, nv %d < 1, row stride %lld < 512 or not a multiple of 8, or lat not "
                  "16-byte aligned)", nv, ld);
        return NEO_ERR_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const long long R = (long long)nv * kNC;
    float* outs[3] = {floor_yz, floor_xz, floor_xy};
    for (int axis = 0; axis < 3; ++axis) {
        pillar_sum_kernel<__nv_bfloat16><<<(unsigned)(nv * kG * kG), 128, 0, s>>>((const __nv_bfloat16*)lat, (int)ld, logits + axis * R, axis,
                                                                                 outs[axis]);
        NEO_LAUNCH_CHECK("pillar_sum_kernel<bf16>");
    }
    return NEO_OK;
}

extern "C" int neo_grid_encoder_pool_bwd_bf16(const void* lat, long long ld, const float* logits, int nv, const float* g_xz, const float* g_xy,
                                              const float* g_yz, float* d_lat, float* d_logits, void* stream) {
    using namespace enc;
    if (!lat || !logits || !d_lat || !d_logits || nv < 1 || ld < kLat) {
        set_error("neo_grid_encoder_pool_bwd_bf16: bad arguments (NULL buffer, nv %d < 1 or row stride %lld < 512)", nv, ld);
        return NEO_ERR_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const long long R = (long long)nv * kNC;
    pillar_softmax_bwd_kernel<<<dim3((unsigned)(nv * kG * kG), 2), kG, 0, s>>>(logits, d_logits, R, 0);
    NEO_LAUNCH_CHECK("pillar_softmax_bwd_kernel");
    pool_bwd_rows_kernel<__nv_bfloat16><<<(unsigned)(nv * kG * kG), 256, 0, s>>>((const __nv_bfloat16*)lat, ld, logits, g_yz, g_xz, g_xy, d_lat,
                                                                                d_logits, R);
    NEO_LAUNCH_CHECK("pool_bwd_rows_kernel<bf16>");
    pillar_softmax_bwd_kernel<<<dim3((unsigned)(nv * kG * kG), 2), kG, 0, s>>>(logits, d_logits, R, 1);
    NEO_LAUNCH_CHECK("pillar_softmax_bwd_kernel");
    return NEO_OK;
}

extern "C" int neo_grid_encoder_lat_grad_bf16(const float* d_pool, const float* d_agg, int nv, void* d_lat, void* stream) {
    using namespace enc;
    if (!d_pool || !d_agg || !d_lat || nv < 1 || !aligned(d_pool, 16) || !aligned(d_agg, 16) || !aligned(d_lat, 8)) {
        set_error("neo_grid_encoder_lat_grad_bf16: bad arguments (NULL buffer, nv %d < 1, or inputs not 16-byte / output not 8-byte aligned)", nv);
        return NEO_ERR_INVALID;
    }
    const long long n4 = (long long)nv * kNC * kLat / 4;
    lat_grad_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, (cudaStream_t)stream>>>((const float4*)d_pool, (const float4*)d_agg, n4, (uint2*)d_lat);
    NEO_LAUNCH_CHECK("lat_grad_kernel");
    return NEO_OK;
}
