// Shared device helpers for the NeO-360 hot path (sm_90a).  All math is fp32 and follows the order of
// operations of the reference's eager PyTorch ops (separate mul / add kernels => no FMA contraction) wherever
// a value feeds a discrete decision (sample positions, CDF brackets); see SURVEY.md Appendix A.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <math.h>
#include <vector>
#include "../../include/neo360_b200.h"

namespace neo {

constexpr int kMaxViews = 8;
constexpr int kWorldCh = 128;
constexpr int kLocalCh = 512;
constexpr int kHidden = 128;
constexpr int kDirEnc = 27;   // deg_view = 4  -> 3 + 3*2*4
constexpr int kPosDeg = 10;   // max_deg_point

// R^T and -(R^T t) of one source camera (models/neo360/util.py:52-70)
struct ViewXform {
    float rt[9];
    float tr[3];
    float pad[4];
};

struct SceneDev {
    int nv, plane_h, plane_w, lat_h, lat_w, img_w, img_h;
    float focal, cx, cy;          // src_focal[0], src_c[0]   (model.py:242-244)
    float lat_scale_x, lat_scale_y;  // latent_scaling / image_size (encoder_pn.py:119,204-206)
    const ViewXform* views;       // device, nv entries
    // channel-last fp32 copies (exact path): (nv, H, W, C)
    const float* planes_cl[3];    // xz, xy, yz
    const float* latent_cl;
};

void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);

#define NEO_CUDA(call)                                              \
    do {                                                            \
        cudaError_t _e = (call);                                    \
        if (_e != cudaSuccess) return neo::cuda_fail(_e, #call);    \
    } while (0)

#define NEO_LAUNCH_CHECK(name)                                      \
    do {                                                            \
        cudaError_t _e = cudaGetLastError();                        \
        if (_e != cudaSuccess) return neo::cuda_fail(_e, name);     \
    } while (0)

// ---- rounding-explicit arithmetic (mimics separate eager kernels) ----
__device__ __forceinline__ float mul_(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add_(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub_(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float dot3_(const float* a, const float* b) {
    return add_(add_(mul_(a[0], b[0]), mul_(a[1], b[1])), mul_(a[2], b[2]));
}

// torch.linspace(0, 1, steps)[i]  (ATen RangeFactories: symmetric evaluation around the midpoint)
__device__ __forceinline__ float linspace01(int i, int steps) {
    if (steps == 1) return 0.f;
    float step = __fdiv_rn(1.0f, (float)(steps - 1));
    int half = steps / 2;
    return (i < half) ? mul_(step, (float)i) : sub_(1.0f, mul_(step, (float)(steps - i - 1)));
}

// Per-ray constants of the NeRF++ parametrisation (helper.py:253-273 and 401-436).
struct RayGeom {
    float o[3], d[3];
    float far;        // intersect_sphere
    float rho;        // |p_mid|
    float phi;        // asin(rho)
    float psph[3];    // sphere hit point
    float axis[3];    // normalised rotation axis
    float check;      // 1 - |p_mid|^2  (must be >= 0)
};

__device__ __forceinline__ void ray_geom(const float* __restrict__ o, const float* __restrict__ d, RayGeom& g,
                                         bool need_bg) {
    g.o[0] = o[0]; g.o[1] = o[1]; g.o[2] = o[2];
    g.d[0] = d[0]; g.d[1] = d[1]; g.d[2] = d[2];
    float dd = dot3_(g.d, g.d);
    float d1 = __fdiv_rn(-dot3_(g.d, g.o), dd);
    float p[3] = {add_(g.o[0], mul_(d1, g.d[0])), add_(g.o[1], mul_(d1, g.d[1])), add_(g.o[2], mul_(d1, g.d[2]))};
    float inv = __fdiv_rn(1.0f, __fsqrt_rn(dd));
    float p2 = dot3_(p, p);
    g.check = sub_(1.0f, p2);
    g.far = add_(d1, mul_(__fsqrt_rn(sub_(1.0f, p2)), inv));
    if (need_bg) {
        // depth2pts_outside uses norm(p_mid) and rho*rho instead of the squared sum (helper.py:422-428)
        g.rho = __fsqrt_rn(p2);
        float d2 = mul_(__fsqrt_rn(sub_(1.0f, mul_(g.rho, g.rho))), inv);
        float s = add_(d1, d2);
        for (int i = 0; i < 3; ++i) g.psph[i] = add_(g.o[i], mul_(s, g.d[i]));
        float ax[3] = {sub_(mul_(g.o[1], g.psph[2]), mul_(g.o[2], g.psph[1])),
                       sub_(mul_(g.o[2], g.psph[0]), mul_(g.o[0], g.psph[2])),
                       sub_(mul_(g.o[0], g.psph[1]), mul_(g.o[1], g.psph[0]))};
        float an = __fsqrt_rn(dot3_(ax, ax));
        for (int i = 0; i < 3; ++i) g.axis[i] = __fdiv_rn(ax[i], an);
        g.phi = asinf(g.rho);
    }
}

__device__ __forceinline__ void fg_point(const RayGeom& g, float t, float* x) {
    for (int i = 0; i < 3; ++i) x[i] = add_(g.o[i], mul_(t, g.d[i]));
}

// bg: s = inverse radius.  xhat = depth2pts_outside (unit vector), lin = o + (far(1-s) + far_unc*s) d (quirk Q2)
__device__ __forceinline__ void bg_point(const RayGeom& g, float s, float far_unc, float* xhat, float* lin) {
    float theta = asinf(mul_(g.rho, s));
    float ang = sub_(g.phi, theta);
    float ca = cosf(ang), sa = sinf(ang);
    const float* a = g.axis;
    const float* p = g.psph;
    float cr[3] = {sub_(mul_(a[1], p[2]), mul_(a[2], p[1])), sub_(mul_(a[2], p[0]), mul_(a[0], p[2])),
                   sub_(mul_(a[0], p[1]), mul_(a[1], p[0]))};
    float ap = dot3_(a, p);
    float omc = sub_(1.0f, ca);
    float q[3];
    for (int i = 0; i < 3; ++i) q[i] = add_(add_(mul_(p[i], ca), mul_(cr[i], sa)), mul_(mul_(a[i], ap), omc));
    float qn = add_(__fsqrt_rn(dot3_(q, q)), 1e-10f);
    for (int i = 0; i < 3; ++i) xhat[i] = __fdiv_rn(q[i], qn);
    if (lin) {
        float tl = add_(mul_(g.far, sub_(1.0f, s)), mul_(far_unc, s));
        for (int i = 0; i < 3; ++i) lin[i] = add_(g.o[i], mul_(tl, g.d[i]));
    }
}

__device__ __forceinline__ void to_camera(const ViewXform& v, const float* x, float* c) {
    c[0] = fmaf(v.rt[2], x[2], fmaf(v.rt[1], x[1], v.rt[0] * x[0])) + v.tr[0];
    c[1] = fmaf(v.rt[5], x[2], fmaf(v.rt[4], x[1], v.rt[3] * x[0])) + v.tr[1];
    c[2] = fmaf(v.rt[8], x[2], fmaf(v.rt[7], x[1], v.rt[6] * x[0])) + v.tr[2];
}
__device__ __forceinline__ void rotate_to_camera(const ViewXform& v, const float* x, float* c) {
    c[0] = fmaf(v.rt[2], x[2], fmaf(v.rt[1], x[1], v.rt[0] * x[0]));
    c[1] = fmaf(v.rt[5], x[2], fmaf(v.rt[4], x[1], v.rt[3] * x[0]));
    c[2] = fmaf(v.rt[8], x[2], fmaf(v.rt[7], x[1], v.rt[6] * x[0]));
}

// grid_sample(align_corners=True, zeros) tap set: indices (clamped) and weights (0 when out of range)
struct Taps {
    int idx[4];     // y*W + x of nw, ne, sw, se (valid even when weight is 0)
    float w[4];
};
__device__ __forceinline__ void bilinear_taps(float gx, float gy, int W, int H, Taps& t) {
    float ix = ((gx + 1.f) / 2.f) * (float)(W - 1);
    float iy = ((gy + 1.f) / 2.f) * (float)(H - 1);
    float x0f = floorf(ix), y0f = floorf(iy);
    float fx = ix - x0f, fy = iy - y0f;      // (ix - ix_nw)
    float gx1 = (x0f + 1.f) - ix, gy1 = (y0f + 1.f) - iy;  // (ix_se - ix)
    // NaN / huge coordinates: every tap is out of range -> 0
    bool finite = (ix == ix) && (iy == iy) && fabsf(ix) < 1e9f && fabsf(iy) < 1e9f;
    int x0 = finite ? (int)x0f : -2, y0 = finite ? (int)y0f : -2;
    int x1 = x0 + 1, y1 = y0 + 1;
    bool vx0 = (x0 >= 0) & (x0 < W), vx1 = (x1 >= 0) & (x1 < W);
    bool vy0 = (y0 >= 0) & (y0 < H), vy1 = (y1 >= 0) & (y1 < H);
    int cx0 = min(max(x0, 0), W - 1), cx1 = min(max(x1, 0), W - 1);
    int cy0 = min(max(y0, 0), H - 1), cy1 = min(max(y1, 0), H - 1);
    t.idx[0] = cy0 * W + cx0; t.w[0] = (vx0 & vy0) ? gx1 * gy1 : 0.f;
    t.idx[1] = cy0 * W + cx1; t.w[1] = (vx1 & vy0) ? fx * gy1 : 0.f;
    t.idx[2] = cy1 * W + cx0; t.w[2] = (vx0 & vy1) ? gx1 * fy : 0.f;
    t.idx[3] = cy1 * W + cx1; t.w[3] = (vx1 & vy1) ? fx * fy : 0.f;
}

// projection (util.py:92-111) + latent grid coords (encoder_pn.py:116-120)
__device__ __forceinline__ void local_grid_coords(const SceneDev& sc, const float* c, float& gx, float& gy) {
    float z = c[2] + 1e-9f;
    float u = (-c[0] / z) * sc.focal + sc.cx;
    float v = (-c[1] / z) * (-sc.focal) + sc.cy;
    gx = u * sc.lat_scale_x - 1.0f;
    gy = v * sc.lat_scale_y - 1.0f;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Column c of the reference positional encoding of x[0..ich) (helper.py:121-125, also the vanilla NeRF and Mip-NeRF 360 direction
// encodings): [x | sin(x 2^k), k-major, k < deg | sin(x 2^k + pi/2)].  The fp32 parity paths depend on this exact mul / add / sinf
// sequence; the tensor-core paths' angle-doubling encodings are different arithmetic and do not use it.
__device__ __forceinline__ float pos_enc_col(const float* x, int ich, int deg, int c) {
    if (c < ich) return x[c];
    int q = c - ich;
    const bool shifted = q >= ich * deg;
    if (shifted) q -= ich * deg;
    const float xb = mul_(x[q % ich], (float)(1 << (q / ich)));
    return sinf(shifted ? add_(xb, 1.57079637f) : xb);
}
// dL/dx_j of one row of pos_enc_col's encoding of x (ich coordinates, deg octaves) whose upstream gradient is g: the identity
// column, then 2^k cos(2^k x_j) for sin(2^k x_j) and -2^k sin(2^k x_j) for its shifted twin sin(2^k x_j + pi/2).  2^k x_j is exact.
__device__ __forceinline__ float pos_enc_grad(float xj, const float* __restrict__ g, int j, int ich, int deg) {
    float s = g[j];
    for (int k = 0; k < deg; ++k) {
        const float sc = (float)(1 << k);
        float sn, cs;
        sincosf(mul_(xj, sc), &sn, &cs);
        s += sc * (g[ich + ich * k + j] * cs - g[ich + ich * deg + ich * k + j] * sn);
    }
    return s;
}

// Head activations of the reference MLPs: density = softplus_(raw - 1), rgb = rgb_act(raw)   (models/neo360/model.py:392-397)
__device__ __forceinline__ float softplus_(float x) { return x > 20.f ? x : log1pf(expf(x)); }
__device__ __forceinline__ float sigmoid_(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float rgb_act(float x) { return sigmoid_(x) * 1.002f - 0.001f; }

// acc[r] += A[r][0..K) . Wt[0..K)[j] for ROWS rows of A (row stride lda, 16-byte aligned rows); Wt is (in, out) with row stride ldw.
// One thread per output neuron j: the weight loads are coalesced across the block, the activation rows are shared-memory broadcasts.
template <int ROWS>
__device__ __forceinline__ void dense_rows(const float* __restrict__ Wt, int ldw, int K, const float* __restrict__ A, int lda, float* acc, int j) {
    int k = 0;
    for (; k + 4 <= K; k += 4) {
        float w0 = __ldg(Wt + (size_t)(k + 0) * ldw + j), w1 = __ldg(Wt + (size_t)(k + 1) * ldw + j);
        float w2 = __ldg(Wt + (size_t)(k + 2) * ldw + j), w3 = __ldg(Wt + (size_t)(k + 3) * ldw + j);
#pragma unroll
        for (int r = 0; r < ROWS; ++r) {
            float4 a = *reinterpret_cast<const float4*>(A + r * lda + k);
            acc[r] = fmaf(a.w, w3, fmaf(a.z, w2, fmaf(a.y, w1, fmaf(a.x, w0, acc[r]))));
        }
    }
    for (; k < K; ++k) {
        float w0 = __ldg(Wt + (size_t)k * ldw + j);
#pragma unroll
        for (int r = 0; r < ROWS; ++r) acc[r] = fmaf(A[r * lda + k], w0, acc[r]);
    }
}

template <class T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }

// ---- host side shared between translation units ----
// Bump allocation of a caller-provided workspace: every block starts on a 256-byte boundary.  With base == nullptr it only counts,
// so the same carving code computes the workspace size and the pointers.
struct Carve {
    unsigned char* base;
    size_t used;
    template <class T> T* take(size_t count) {
        T* p = base ? reinterpret_cast<T*>(base + used) : nullptr;
        used += (count * sizeof(T) + 255) & ~size_t(255);
        return p;
    }
};

// Copies n floats of a workspace result to an optional output; NULL (not wanted) or the same buffer is a no-op.
inline int copy_out(float* dst, const float* src, size_t n, cudaStream_t s) {
    if (!dst || dst == src) return NEO_OK;
    NEO_CUDA(cudaMemcpyAsync(dst, src, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return NEO_OK;
}

struct MLPFp32 {   // weights transposed to (in, out) for coalesced reads by output-neuron threads
    int in_ch, enc_dim, in_dim;   // 3|4, 63|84, enc+512+128
    const float *w0t, *b0, *w1t, *b1, *w2t, *b2, *w3t, *b3, *wbt, *bb, *wsig, *bsig, *wv0t, *bv0, *wv1t, *bv1, *wrgb, *brgb;
};

}  // namespace neo

struct NeoScene {
    neo::SceneDev dev;
    NeoSceneDesc desc;
    int precision_mask;
    neo::MLPFp32 mlp32[4];
    void* tc_state;            // opaque state of the tensor-core path (field_tc.cu)
    int* err_flag;             // device int
    std::vector<std::pair<void*, size_t>> allocations;
    size_t bytes;
};

namespace neo {
// scene.cu
int scene_alloc_bytes(NeoScene* sc, void** p, size_t bytes);
// Device blocks of destroyed scenes (and the scene builder's temporaries) are kept, per device and up to a cap, for the next scene of
// the same shape: a scene change then costs its kernels, not cudaMalloc / cudaFree (which are slow, erratic and device-synchronising).
int pool_alloc(void** p, size_t bytes);
void pool_release(void* p, size_t bytes);
// (n, C, HW) fp32 -> (n, HW, C) fp32 or fp16 (round to nearest): channel-last copies of feature maps
int launch_nchw_to_nhwc(const float* in, float* out, int n, int C, int HW, cudaStream_t s);
int launch_nchw_to_nhwc(const float* in, __half* out, int n, int C, int HW, cudaStream_t s);
// nn.Linear weight (out_f, in_f) -> (in_f, out_f), for the CUDA-core MLPs' coalesced weight reads (dense_rows)
int launch_transpose(const float* w, float* wt, int out_f, int in_f, cudaStream_t s);
// sampling.cu
int launch_far(const float* o, const float* d, int n, float* far, int* err, cudaStream_t s);
int launch_sample_coarse(const float* o, const float* d, const float* far, int n, int num_samples, int in_sphere,
                         float far_unc, const float* u_rand, float* t, float* pts, float* pts_lin, cudaStream_t s);
int launch_resample(const float* o, const float* d, const float* far, const float* t_old, const float* w, int n,
                    int n_old, int m, int in_sphere, float far_unc, const float* u_rand, float* t, float* pts,
                    float* pts_lin, cudaStream_t s);
int launch_composite(const float* rgb, const float* sigma, const float* t, const float* d, const float* far, int n,
                     int N, int white, int in_sphere, float* comp, float* acc, float* w, float* lam, float* depth,
                     cudaStream_t s);
int launch_composite_bwd(const float* rgb, const float* sigma, const float* t, const float* d, const float* far, int n, int N, int white,
                         int in_sphere, const float* g_comp, const float* g_acc, const float* g_w, const float* g_lam, const float* g_depth,
                         float* d_rgb, float* d_sigma, cudaStream_t s);
int launch_combine(int n, int N, const float* fg_c, const float* bg_c, const float* lam, const float* fg_depth,
                   const float* bg_depth, const float* fg_t, const float* bg_s, float* comp, float* depth,
                   float* fg_sdist, float* bg_sdist, cudaStream_t s);
// mask NULL: every value; otherwise one byte per (pixel, 3) value triple, and *count = the number of values summed
int launch_clipped_sq_err(const float* a, const float* b, const unsigned char* mask, long long n, double* out, unsigned long long* count,
                          cudaStream_t s);
int launch_sample_rays(int n, const long long* pix, int T, int H, int W, float focal, const float* c2w, const float* images,
                       float* o, float* vd, float* rd, float* radii, float* target, int* err, cudaStream_t s);
int launch_get_rays(int H, int W, float focal, const float* c2w, float* o, float* vd, float* rd, float* radii,
                    cudaStream_t s);
size_t sample_rays_bwd_workspace(int n, int T);
int launch_sample_rays_bwd(int n, const long long* pix, int T, int H, int W, float focal, const float* c2w, const float* g_o, const float* g_vd,
                           const float* g_rd, float* g_c2w, void* ws, cudaStream_t s);
// field_fp32.cu
int launch_field_fp32(const NeoScene* sc, const NeoRays* rays, const float* far, const float* t, int N, int mlp_index,
                      float* rgb, float* sigma, cudaStream_t s);
int launch_index_grid(const NeoScene* sc, const float* pts, int M, float* out, cudaStream_t s);
int launch_index_local(const NeoScene* sc, const float* pts, int M, float* out, cudaStream_t s);
int launch_index_maps(const NeoScene* sc, const float* pts, int M, int C, const float* lat, const float* xz, const float* xy, const float* yz,
                      float* out_local, float* out_world, cudaStream_t s);
int launch_index_maps_bwd(const NeoScene* sc, const float* pts, int M, int C, const float* g_local, const float* g_world, float* g_lat, float* g_xz,
                          float* g_xy, float* g_yz, cudaStream_t s);
int launch_index_bwd(const NeoScene* sc, const float* pts, int M, int local, const float* g_out, float* g_lat, float* g_xz, float* g_xy,
                     float* g_yz, cudaStream_t s);
// det.cu: order-fixed scatter (deterministic adjoint of the lookups).  The caller's entry kernel writes, for entry e in [0, E), keys[e]
// (texel key in [0, T), or T for a zero-weight tap), ids[e] = e and wts[e]; det_sort_reduce sorts and reduces.  Workspace blocks, in
// this order and each starting on a 256-byte boundary of the workspace: keys, keys_sorted, ids, ids_sorted (E u32 each), wts (E f32),
// starts (T + 1 u32), sort scratch.
struct DetBuffers {
    unsigned *keys, *keys_sorted, *ids, *ids_sorted;
    float* wts;
    unsigned* starts;
    void* scratch;
    size_t scratch_bytes, total;     // total = 0: the sort's scratch query failed (neo_last_error says why)
};
DetBuffers det_carve(void* ws, long long E, long long T);
// Entry e belongs to source s = (e >= e0[1]), row (e - e0[s]) / taps[s] of g[s] (row stride ld[s] floats).
struct DetSrc { const float* g[2]; long long ld[2]; unsigned e0[2]; int taps[2]; };
// Keys [key0[m], key0[m+1]) address map m (channel-last rows of C floats); unused maps repeat the last key0.
constexpr int kDetMaps = 4;
struct DetDst { float* map[kDetMaps]; long long key0[kDetMaps]; };
// vec = 4: rows and maps are read as float4 (C % 4 == 0, 16-byte aligned); 2: float2 (C, ld even, 8-byte aligned)
int det_sort_reduce(const DetBuffers& b, long long E, long long T, int C, int vec, const DetSrc& src, const DetDst& dst, cudaStream_t s);
int launch_index_maps_bwd_det(const NeoScene* sc, const float* pts, int M, int C, const float* g_local, const float* g_world, float* g_lat,
                              float* g_xz, float* g_xy, float* g_yz, const DetBuffers& b, cudaStream_t s);
// E and T of neo_index_maps_bwd_det for the maps that receive a gradient
void index_det_sizes(const NeoScene* sc, int M, bool local, bool world, long long& E, long long& T);
// field_tc.cu
int tc_scene_create(NeoScene* sc, const NeoMLPParams mlps[4], cudaStream_t s);
void tc_scene_free(NeoScene* sc);
// direction fragments of every ray for the field launches of one call: kDirFragBytes per ray, 16-byte aligned
constexpr size_t kDirFragBytes = 64;
int launch_dir_frags(const NeoScene* sc, const NeoRays* rays, void* dir, cudaStream_t s);
int launch_field_tc(const NeoScene* sc, const NeoRays* rays, const float* far, const float* t, int N, int mlp_index, const void* dir,
                    float* rgb, float* sigma, cudaStream_t s);
// gemm_tc.cu: the tensor-core dense layer, fp16 operand packing and the tiny-N head (contracts at their definitions)
int gemm_f16(const void* A, long long lda, const void* W, long long ldw, const float* bias, void* C, long long ldc, long long M, int N, int K,
             int relu, cudaStream_t s);
int f32_to_f16_pad(const float* in, long long rows, int cols_in, long long ld_in, void* out, int cols_out, long long ld_out, cudaStream_t s,
                   int bf16 = 0);
int launch_rowdot_f16(const void* H, long long ld, int K, const float* W, const float* b, int N, long long M, float* out, cudaStream_t s,
                      int bf16 = 0);
// gemm_tc.cu: the bf16 training forms of the same dense layer (csrc/dense_train.cu)
int gemm_bf16(const void* A, long long lda, const void* W, long long ldw, const float* bias, void* C, long long ldc, long long M, int N, int K,
              int epi, cudaStream_t s);
int dgrad_bf16(const void* dY, long long ldy, const void* Wt, long long ldwt, const void* X, long long ldx, const float* g_sig,
               const float* w_sig, void* dX, long long lddx, long long M, int N, int K, cudaStream_t s);
int wgrad_bf16_partials(const void* dY, long long ldy, const void* X, long long ldx, long long M, int N, int K, int splits, float* part,
                        cudaStream_t s);
}  // namespace neo
