// Output side and LPIPS fine-tuning (SURVEY.md 8(f4)): the LPIPS-specific arithmetic around a VGG-16 trunk that the host framework runs.
// LPIPS of frames x, y in [0, 1] (LitModel.lpips_each, models/interface.py:113-122, with piqa's LPIPS(network="vgg"); the fine-tuning
// loss NeRF_TP.lpips_loss, models/neo360/model.py:1283-1309, with lpips.LPIPS(net="vgg")) is pinned here as:
//   - inputs clipped to [0, 1] first (torch.clamp: NaN stays NaN);
//   - scaling, two forms that agree in real arithmetic but round differently in fp32, each in its package's operation order:
//       form 0 (piqa, evaluation):  (x - mean_c) / std_c                  mean = (0.485, 0.456, 0.406), std = (0.229, 0.224, 0.225)
//       form 1 (lpips, training):   ((2 x - 1) - shift_c) / scale_c        shift = (-0.030, -0.088, -0.188), scale = (0.458, 0.448, 0.450)
//   - features: relu1_2, relu2_2, relu3_3, relu4_3, relu5_3 of torchvision's vgg16().features[:30] (framework convolutions, not here):
//     layer k has C_k = 64, 128, 256, 512, 512 channels on an (H >> k, W >> k) grid (2x2 max pools floor);
//   - per layer k and pixel p: u = f_x / (||f_x||_2 + eps), v = f_y / (||f_y||_2 + eps), norms over the channels, eps = 1e-10
//     (lpips' normalize_tensor); d_p = sum_c w_kc (u_c - v_c)^2 with w_k the layer's 1x1 weights;
//   - LPIPS = sum_k mean_p d_p.
//
// neo_lpips_head: one thread per pixel, so each channel step reads one coalesced row of a plane.  Per pixel, a norm pass (fma chains in
// channel order) and a distance pass (e = u - v with both divisions rounded, d as an fma chain in channel order); the CTA's sum in double
// (per thread, XOR butterfly per warp, warps in index order) goes to the workspace, and a second launch adds each frame's partials layer by
// layer in index order.  The CTA partition depends on H and W only and there are no floating-point atomics: two calls are bit-identical,
// a frame gives the same bits alone or in any batch, LPIPS(x, x) is exactly 0 and LPIPS(x, y) and LPIPS(y, x) have the same bits.
//
// neo_lpips_head_bwd, for a per-frame upstream g: with D = ||f|| + eps, r = w (u - v) and a = 2 g / (H_k W_k),
//   dLPIPS / df_j = a (r_j / D - f_j (sum_c r_c f_c) / (||f|| D^2)),
// written as (a / D) r_j - f_j ((a / D) t / (||f|| D)) with t = sum_c r_c f_c.  A pixel whose channels are all zero gets 0: the norm has no
// derivative there, and in the framework the ReLU in front of the head zeroes that gradient anyway.  The y side is the same with -r.
#include "common.cuh"

namespace neo {
namespace lpips {

constexpr int kLayers = 5, kThreads = 128, kWarps = kThreads / 32;
constexpr int kMinSize = 1 << (kLayers - 1);       // relu5_3 needs H >> 4, W >> 4 >= 1
constexpr float kEps = 1e-10f;
__constant__ float c_mean[3] = {0.485f, 0.456f, 0.406f}, c_std[3] = {0.229f, 0.224f, 0.225f};
__constant__ float c_shift[3] = {-0.030f, -0.088f, -0.188f}, c_scale[3] = {0.458f, 0.448f, 0.450f};
__host__ __device__ constexpr int channels(int k) { return k < 3 ? 64 << k : 512; }   // 64, 128, 256, 512, 512

struct Layers {
    const float* fx[kLayers];
    const float* fy[kLayers];
    const float* w[kLayers];
    float* gx[kLayers];
    float* gy[kLayers];
    long long P[kLayers];        // pixels per frame of each layer
    int tile0[kLayers + 1];      // first CTA of each layer within a frame; tile0[kLayers] = CTAs per frame
};

__device__ __forceinline__ float clamp01(float v) { return v < 0.f ? 0.f : (v > 1.f ? 1.f : v); }   // torch.clamp: NaN stays NaN

__global__ void __launch_bounds__(256) prepare_kernel(const float* __restrict__ img, long long n_pix, long long HW, int form,
                                                     float* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_pix) return;
    const long long f = i / HW, p = i - f * HW;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float x = clamp01(img[3 * i + c]);
        const float s = form == 0 ? __fsub_rn(x, c_mean[c]) : __fsub_rn(__fsub_rn(__fmul_rn(2.f, x), 1.f), c_shift[c]);
        out[(f * 3 + c) * HW + p] = __fdiv_rn(s, form == 0 ? c_std[c] : c_scale[c]);
    }
}

// Autograd's chain through the same operations: division backward g / s, the factor 2 of form 1, then clamp's mask, inclusive at 0 and 1.
__global__ void __launch_bounds__(256) prepare_bwd_kernel(const float* __restrict__ img, const float* __restrict__ g_out, long long n_pix,
                                                         long long HW, int form, float* __restrict__ g_img) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_pix) return;
    const long long f = i / HW, p = i - f * HW;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float x = img[3 * i + c], g = g_out[(f * 3 + c) * HW + p];
        const float d = form == 0 ? __fdiv_rn(g, c_std[c]) : __fmul_rn(__fdiv_rn(g, c_scale[c]), 2.f);
        g_img[3 * i + c] = (x >= 0.f && x <= 1.f) ? d : 0.f;
    }
}

// Norm pass: sum_c f_c^2 of both images as fma chains in channel order; returns ||f|| + eps of each.
template <int C>
__device__ __forceinline__ void norms(const float* __restrict__ fx, const float* __restrict__ fy, long long P, float* nx, float* ny) {
    float sx = 0.f, sy = 0.f;
#pragma unroll 8
    for (int c = 0; c < C; ++c) {
        const float a = __ldg(fx + c * P), b = __ldg(fy + c * P);
        sx = __fmaf_rn(a, a, sx);
        sy = __fmaf_rn(b, b, sy);
    }
    *nx = __fsqrt_rn(sx);
    *ny = __fsqrt_rn(sy);
}

template <int C>
__device__ __forceinline__ float head_pixel(const float* __restrict__ fx, const float* __restrict__ fy, const float* __restrict__ w,
                                            long long P) {
    float nx, ny;
    norms<C>(fx, fy, P, &nx, &ny);
    const float dx = __fadd_rn(nx, kEps), dy = __fadd_rn(ny, kEps);
    float d = 0.f;
#pragma unroll 8
    for (int c = 0; c < C; ++c) {
        const float e = __fsub_rn(__fdiv_rn(__ldg(fx + c * P), dx), __fdiv_rn(__ldg(fy + c * P), dy));
        d = __fmaf_rn(__ldg(w + c), __fmul_rn(e, e), d);
    }
    return d;
}

// The layer of CTA t of a frame.
__device__ __forceinline__ int layer_of(const Layers& L, int t) {
    int k = 0;
    while (k + 1 < kLayers && t >= L.tile0[k + 1]) ++k;
    return k;
}

// Deterministic block sum; the result is valid in thread 0.  Callable repeatedly.
__device__ __forceinline__ double block_sum(double v, double* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < kWarps; ++w) t += red[w];
    __syncthreads();
    return t;
}

__global__ void __launch_bounds__(kThreads) head_tile_kernel(const Layers L, double* __restrict__ partial) {
    __shared__ double red[kWarps];
    const int tpf = L.tile0[kLayers];
    const int f = blockIdx.x / tpf, t = blockIdx.x - f * tpf, k = layer_of(L, t);
    const long long P = L.P[k], p = (long long)(t - L.tile0[k]) * kThreads + threadIdx.x;
    double acc = 0.0;
    if (p < P) {
        const long long base = (long long)f * channels(k) * P + p;
        const float* fx = L.fx[k] + base;
        const float* fy = L.fy[k] + base;
        float d;
        switch (k) {
            case 0: d = head_pixel<64>(fx, fy, L.w[0], P); break;
            case 1: d = head_pixel<128>(fx, fy, L.w[1], P); break;
            case 2: d = head_pixel<256>(fx, fy, L.w[2], P); break;
            default: d = head_pixel<512>(fx, fy, L.w[k], P); break;
        }
        acc = (double)d;
    }
    const double s = block_sum(acc, red);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// One block per frame: each layer's CTA sums in index order over its pixel count, then the layers in order.
__global__ void __launch_bounds__(kThreads) head_frame_kernel(const Layers L, const double* __restrict__ partial, double* __restrict__ out,
                                                              double* __restrict__ per_layer) {
    __shared__ double red[kWarps];
    const int tpf = L.tile0[kLayers];
    const double* p = partial + (long long)blockIdx.x * tpf;
    double total = 0.0;
    for (int k = 0; k < kLayers; ++k) {
        double acc = 0.0;
        for (int i = L.tile0[k] + threadIdx.x; i < L.tile0[k + 1]; i += kThreads) acc += p[i];
        const double v = block_sum(acc, red) / (double)L.P[k];
        total += v;
        if (threadIdx.x == 0 && per_layer) per_layer[blockIdx.x * kLayers + k] = v;
    }
    if (threadIdx.x == 0) out[blockIdx.x] = total;
}

// One side of the adjoint at one pixel: g_j = (a / D) s r_j - f_j k, s = +1 for x, -1 for y, k = (a / D) t / (||f|| D).
template <int C>
__device__ __forceinline__ void bwd_pixel(const float* __restrict__ fx, const float* __restrict__ fy, const float* __restrict__ w,
                                          long long P, float a, float* __restrict__ gx, float* __restrict__ gy) {
    float nx, ny;
    norms<C>(fx, fy, P, &nx, &ny);
    const float dx = __fadd_rn(nx, kEps), dy = __fadd_rn(ny, kEps);
    float tx = 0.f, ty = 0.f;
#pragma unroll 8
    for (int c = 0; c < C; ++c) {
        const float a_ = __ldg(fx + c * P), b_ = __ldg(fy + c * P);
        const float r = __fmul_rn(__ldg(w + c), __fsub_rn(__fdiv_rn(a_, dx), __fdiv_rn(b_, dy)));
        tx = __fmaf_rn(r, a_, tx);
        ty = __fmaf_rn(-r, b_, ty);
    }
    const float ax = __fdiv_rn(a, dx), ay = __fdiv_rn(a, dy);
    const float kx = nx > 0.f ? __fdiv_rn(__fmul_rn(ax, tx), __fmul_rn(nx, dx)) : 0.f;
    const float ky = ny > 0.f ? __fdiv_rn(__fmul_rn(ay, ty), __fmul_rn(ny, dy)) : 0.f;
#pragma unroll 8
    for (int c = 0; c < C; ++c) {
        const float a_ = __ldg(fx + c * P), b_ = __ldg(fy + c * P);
        const float r = __fmul_rn(__ldg(w + c), __fsub_rn(__fdiv_rn(a_, dx), __fdiv_rn(b_, dy)));
        gx[c * P] = nx > 0.f ? __fsub_rn(__fmul_rn(ax, r), __fmul_rn(kx, a_)) : 0.f;
        if (gy) gy[c * P] = ny > 0.f ? __fsub_rn(__fmul_rn(ay, -r), __fmul_rn(ky, b_)) : 0.f;
    }
}

__global__ void __launch_bounds__(kThreads) head_bwd_kernel(const Layers L, const float* __restrict__ g) {
    const int tpf = L.tile0[kLayers];
    const int f = blockIdx.x / tpf, t = blockIdx.x - f * tpf, k = layer_of(L, t);
    const long long P = L.P[k], p = (long long)(t - L.tile0[k]) * kThreads + threadIdx.x;
    if (p >= P) return;
    const long long base = (long long)f * channels(k) * P + p;
    const float a = __fdiv_rn(__fmul_rn(2.f, g[f]), (float)P);
    const float *fx = L.fx[k] + base, *fy = L.fy[k] + base;
    float *gx = L.gx[k] + base, *gy = L.gy[k] ? L.gy[k] + base : nullptr;
    switch (k) {
        case 0: bwd_pixel<64>(fx, fy, L.w[0], P, a, gx, gy); break;
        case 1: bwd_pixel<128>(fx, fy, L.w[1], P, a, gx, gy); break;
        case 2: bwd_pixel<256>(fx, fy, L.w[2], P, a, gx, gy); break;
        default: bwd_pixel<512>(fx, fy, L.w[k], P, a, gx, gy); break;
    }
}

// Layer sizes and the CTA partition of one frame; false when the sizes are invalid or the call does not fit one launch / int64 indexing.
bool head_shape(int n, int H, int W, Layers* L) {
    if (n < 1 || H < kMinSize || W < kMinSize) return false;
    long long elems;
    if (__builtin_mul_overflow((long long)n, (long long)H, &elems) || __builtin_mul_overflow(elems, (long long)W, &elems) ||
        __builtin_mul_overflow(elems, 64LL, &elems))
        return false;
    long long tiles = 0;
    for (int k = 0; k < kLayers; ++k) {
        L->P[k] = (long long)(H >> k) * (W >> k);
        L->tile0[k] = (int)tiles;
        tiles += (L->P[k] + kThreads - 1) / kThreads;
        if (tiles * n > 0x7fffffffLL) return false;
    }
    L->tile0[kLayers] = (int)tiles;
    return true;
}

// Host arrays of five device pointers: every entry must be set.
bool all_set(const void* const* a) {
    if (!a) return false;
    for (int k = 0; k < kLayers; ++k)
        if (!a[k]) return false;
    return true;
}

}  // namespace lpips
}  // namespace neo

using namespace neo;

static int prepare_check(const char* who, const void* a, const void* b, const void* c, int n, int H, int W, int form) {
    if (!a || !b || !c) { set_error("%s: NULL buffer", who); return NEO_ERR_INVALID; }
    long long e;
    if (n < 1 || H < 1 || W < 1 || __builtin_mul_overflow((long long)n * H, (long long)W * 3, &e) || (form != 0 && form != 1)) {
        set_error("%s: n %d, H %d, W %d must be >= 1 and fit int64 elements, form %d must be 0 (piqa) or 1 (lpips)", who, n, H, W, form);
        return NEO_ERR_INVALID;
    }
    return NEO_OK;
}

extern "C" int neo_lpips_prepare(const float* img, int n, int H, int W, int form, float* out, void* stream) {
    if (int rc = prepare_check("neo_lpips_prepare", img, out, out, n, H, W, form)) return rc;
    const long long n_pix = (long long)n * H * W;
    lpips::prepare_kernel<<<(unsigned)((n_pix + 255) / 256), 256, 0, (cudaStream_t)stream>>>(img, n_pix, (long long)H * W, form, out);
    NEO_LAUNCH_CHECK("lpips::prepare_kernel");
    return NEO_OK;
}

extern "C" int neo_lpips_prepare_bwd(const float* img, const float* g_out, int n, int H, int W, int form, float* g_img, void* stream) {
    if (int rc = prepare_check("neo_lpips_prepare_bwd", img, g_out, g_img, n, H, W, form)) return rc;
    const long long n_pix = (long long)n * H * W;
    lpips::prepare_bwd_kernel<<<(unsigned)((n_pix + 255) / 256), 256, 0, (cudaStream_t)stream>>>(img, g_out, n_pix, (long long)H * W, form,
                                                                                                   g_img);
    NEO_LAUNCH_CHECK("lpips::prepare_bwd_kernel");
    return NEO_OK;
}

extern "C" size_t neo_lpips_workspace_bytes(int n, int H, int W) {
    lpips::Layers L;
    if (!lpips::head_shape(n, H, W, &L)) return 0;
    return (size_t)n * L.tile0[lpips::kLayers] * sizeof(double);
}

extern "C" int neo_lpips_head(const float* const* fx, const float* const* fy, const float* const* w, int n, int H, int W, double* lpips_out,
                              double* per_layer, void* workspace, size_t workspace_bytes, void* stream) {
    using namespace lpips;
    Layers L = {};
    if (!all_set((const void* const*)fx) || !all_set((const void* const*)fy) || !all_set((const void* const*)w) || !lpips_out || !workspace) {
        set_error("neo_lpips_head: NULL feature / weight pointer, lpips or workspace");
        return NEO_ERR_INVALID;
    }
    if (!head_shape(n, H, W, &L)) {
        set_error("neo_lpips_head: n %d must be >= 1 and H %d, W %d >= %d, and the call must fit int64 elements and 2^31 - 1 CTAs", n, H, W,
                  kMinSize);
        return NEO_ERR_INVALID;
    }
    const size_t need = (size_t)n * L.tile0[kLayers] * sizeof(double);
    if (workspace_bytes < need || (uintptr_t)workspace % alignof(double)) {
        set_error("neo_lpips_head: workspace needs %zu bytes, 8-byte aligned (got %zu)", need, workspace_bytes);
        return NEO_ERR_WORKSPACE;
    }
    for (int k = 0; k < kLayers; ++k) {
        L.fx[k] = fx[k];
        L.fy[k] = fy[k];
        L.w[k] = w[k];
    }
    cudaStream_t s = (cudaStream_t)stream;
    head_tile_kernel<<<(unsigned)(n * L.tile0[kLayers]), kThreads, 0, s>>>(L, (double*)workspace);
    NEO_LAUNCH_CHECK("lpips::head_tile_kernel");
    head_frame_kernel<<<(unsigned)n, kThreads, 0, s>>>(L, (const double*)workspace, lpips_out, per_layer);
    NEO_LAUNCH_CHECK("lpips::head_frame_kernel");
    return NEO_OK;
}

extern "C" int neo_lpips_head_bwd(const float* const* fx, const float* const* fy, const float* const* w, int n, int H, int W, const float* g,
                                  float* const* g_fx, float* const* g_fy, void* stream) {
    using namespace lpips;
    Layers L = {};
    if (!all_set((const void* const*)fx) || !all_set((const void* const*)fy) || !all_set((const void* const*)w) || !g ||
        !all_set((const void* const*)g_fx) || (g_fy && !all_set((const void* const*)g_fy))) {
        set_error("neo_lpips_head_bwd: NULL feature / weight / gradient pointer (g_fy may be NULL as a whole)");
        return NEO_ERR_INVALID;
    }
    if (!head_shape(n, H, W, &L)) {
        set_error("neo_lpips_head_bwd: n %d must be >= 1 and H %d, W %d >= %d, and the call must fit int64 elements and 2^31 - 1 CTAs", n, H,
                  W, kMinSize);
        return NEO_ERR_INVALID;
    }
    for (int k = 0; k < kLayers; ++k) {
        L.fx[k] = fx[k];
        L.fy[k] = fy[k];
        L.w[k] = w[k];
        L.gx[k] = g_fx[k];
        L.gy[k] = g_fy ? g_fy[k] : nullptr;
    }
    head_bwd_kernel<<<(unsigned)(n * L.tile0[kLayers]), kThreads, 0, (cudaStream_t)stream>>>(L, g);
    NEO_LAUNCH_CHECK("lpips::head_bwd_kernel");
    return NEO_OK;
}
