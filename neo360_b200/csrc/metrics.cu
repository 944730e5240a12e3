// Output side (SURVEY.md 8(f4)): SSIM of rendered frames, as LitModel.ssim_each (models/interface.py:101-111) computes it with piqa's
// SSIM() at its defaults.  piqa is pinned by its definition:
//   - window: 11 taps, sigma = 1.5, built in fp32 as k = exp(-((arange(11) - 5)^2 / (2 sigma^2))), k /= k.sum() (the values below are
//     torch's fp32 results of that construction), applied separably with NO padding: the SSIM map of a (H, W) channel is (H-10, W-10);
//   - mu_x = G*x, mu_y = G*y, s_xx = G*(x x) - mu_x^2, s_yy = G*(y y) - mu_y^2, s_xy = G*(x y) - mu_x mu_y, C1 = 0.01^2, C2 = 0.03^2;
//   - cs = (2 s_xy + C2) / (s_xx + s_yy + C2), ss = (2 mu_x mu_y + C1) / (mu_x^2 + mu_y^2 + C1) * cs;
//   - a frame's SSIM is the mean of ss over its three channels and every valid pixel;
//   - inputs are clipped to [0, 1] first (ssim_each clips before it calls piqa).
//
// One CTA per (frame, 16 x 32 tile of the SSIM map).  It stages the tile's 26 x 42 input pixels (all three channels, the 10-row / column
// halo included, clipped) of both images in shared memory, then per channel runs the horizontal pass of the five moments into shared
// memory and the vertical pass, the map and the tile's sum in registers.  The tile partition depends on H and W only, and every sum has a
// fixed order (per thread in program order, an XOR butterfly per warp, warps in index order, the tiles of a frame in index order in a
// second launch): no floating-point atomics, so two calls are bit-identical and a frame gives the same bits alone or inside any batch.
#include "common.cuh"

namespace neo {
namespace metrics {

constexpr int kTaps = 11, kLost = kTaps - 1;
constexpr int kTileH = 16, kTileW = 32, kInH = kTileH + kLost, kInW = kTileW + kLost;
constexpr int kThreads = 256, kWarps = kThreads / 32;
constexpr float kC1 = 1.0e-4f, kC2 = 9.0e-4f;   // float(0.01 ** 2), float(0.03 ** 2): the scalars piqa's fp32 ops see
static_assert(kThreads == kTileW * kTileH / 2, "the vertical pass gives every thread two rows of one column");

__constant__ float c_win[kTaps] = {0x1.0d957p-10f, 0x1.f1fe02p-8f, 0x1.26eb18p-5f, 0x1.bff0fep-4f, 0x1.b43c3ep-3f, 0x1.10656p-2f,
                                   0x1.b43c3ep-3f, 0x1.bff0fep-4f, 0x1.26eb18p-5f, 0x1.f1fe02p-8f, 0x1.0d957p-10f};

__device__ __forceinline__ float clip01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }

// Deterministic block sum; the result is valid in thread 0.
__device__ __forceinline__ double block_sum(double v, double* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < kWarps; ++w) t += red[w];
    return t;
}

// Every operation is written with an explicit rounding (no FMA contraction), so that for x == y the numerators and denominators round
// identically and SSIM(x, x) is exactly 1: 2 s_xy + C2 and (s_xx + s_yy) + C2 are then the same fp32 value, as are 2 mu_x mu_y + C1 and
// (mu_x^2 + mu_y^2) + C1.  The window sums are fma chains in tap order, the same instructions for x x, y y and x y.
__global__ void __launch_bounds__(kThreads) ssim_tile_kernel(const float* __restrict__ x, const float* __restrict__ y, int H, int W, int tiles_x,
                                                             int tiles_per_frame, float* __restrict__ ss_map, double* __restrict__ partial) {
    __shared__ float sx[kInH][kInW * 3], sy[kInH][kInW * 3];   // channel-last, as in global memory
    __shared__ float sh[5][kInH][kTileW];                       // horizontal pass of x, y, x x, y y, x y for one channel
    __shared__ double red[kWarps];
    const int f = blockIdx.x / tiles_per_frame, t = blockIdx.x - f * tiles_per_frame;
    const int oy0 = (t / tiles_x) * kTileH, ox0 = (t % tiles_x) * kTileW;
    const int Ho = H - kLost, Wo = W - kLost;
    const long long row3 = 3LL * W, frame = (long long)f * H * row3;
    for (int i = threadIdx.x; i < kInH * kInW * 3; i += kThreads) {
        const int r = i / (kInW * 3), c = i - r * (kInW * 3);
        const long long gx = 3LL * ox0 + c;
        float a = 0.f, b = 0.f;
        if (oy0 + r < H && gx < row3) {
            const long long g = frame + (oy0 + r) * row3 + gx;
            a = clip01(x[g]);
            b = clip01(y[g]);
        }
        sx[r][c] = a;
        sy[r][c] = b;
    }
    __syncthreads();
    const int col = threadIdx.x & 31, r0 = (threadIdx.x >> 5) * 2, ox = ox0 + col;
    double acc = 0.0;
    for (int ch = 0; ch < 3; ++ch) {
        for (int i = threadIdx.x; i < kInH * kTileW; i += kThreads) {
            const int r = i / kTileW, c = i - r * kTileW;
            float m[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int k = 0; k < kTaps; ++k) {
                const float w = c_win[k], a = sx[r][(c + k) * 3 + ch], b = sy[r][(c + k) * 3 + ch];
                m[0] = __fmaf_rn(w, a, m[0]);
                m[1] = __fmaf_rn(w, b, m[1]);
                m[2] = __fmaf_rn(w, __fmul_rn(a, a), m[2]);
                m[3] = __fmaf_rn(w, __fmul_rn(b, b), m[3]);
                m[4] = __fmaf_rn(w, __fmul_rn(a, b), m[4]);
            }
#pragma unroll
            for (int q = 0; q < 5; ++q) sh[q][r][c] = m[q];
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int r = r0 + j, oy = oy0 + r;
            float m[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int k = 0; k < kTaps; ++k)
#pragma unroll
                for (int q = 0; q < 5; ++q) m[q] = __fmaf_rn(c_win[k], sh[q][r + k][col], m[q]);
            const float mxx = __fmul_rn(m[0], m[0]), myy = __fmul_rn(m[1], m[1]), mxy = __fmul_rn(m[0], m[1]);
            const float sxx = __fsub_rn(m[2], mxx), syy = __fsub_rn(m[3], myy), sxy = __fsub_rn(m[4], mxy);
            const float cs = __fdiv_rn(__fadd_rn(__fmul_rn(2.f, sxy), kC2), __fadd_rn(__fadd_rn(sxx, syy), kC2));
            const float ss = __fmul_rn(__fdiv_rn(__fadd_rn(__fmul_rn(2.f, mxy), kC1), __fadd_rn(__fadd_rn(mxx, myy), kC1)), cs);
            if (oy < Ho && ox < Wo) {
                acc += (double)ss;
                if (ss_map) ss_map[(((long long)f * Ho + oy) * Wo + ox) * 3 + ch] = ss;
            }
        }
        __syncthreads();   // sh is rewritten for the next channel
    }
    const double s = block_sum(acc, red);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// One block per frame: the frame's tile sums in a fixed order, divided by the number of map values.
__global__ void __launch_bounds__(kThreads) ssim_frame_kernel(const double* __restrict__ partial, int tiles_per_frame, double count,
                                                              double* __restrict__ out) {
    __shared__ double red[kWarps];
    const double* p = partial + (long long)blockIdx.x * tiles_per_frame;
    double acc = 0.0;
    for (int i = threadIdx.x; i < tiles_per_frame; i += kThreads) acc += p[i];
    const double s = block_sum(acc, red);
    if (threadIdx.x == 0) out[blockIdx.x] = s / count;
}

// Tiles per frame and in the whole call; false when the sizes are invalid or the call does not fit one launch / int64 indexing.
bool ssim_shape(int n, int H, int W, int* tiles_x, int* tiles_per_frame) {
    if (n < 1 || H < kTaps || W < kTaps) return false;
    long long elems;
    if (__builtin_mul_overflow((long long)n, (long long)H, &elems) || __builtin_mul_overflow(elems, (long long)W, &elems) ||
        __builtin_mul_overflow(elems, 3LL, &elems))
        return false;
    const long long tx = (W - kLost + kTileW - 1) / kTileW, ty = (H - kLost + kTileH - 1) / kTileH;
    if (tx * ty * n > 0x7fffffffLL) return false;
    *tiles_x = (int)tx;
    *tiles_per_frame = (int)(tx * ty);
    return true;
}

}  // namespace metrics
}  // namespace neo

using namespace neo;

extern "C" size_t neo_ssim_workspace_bytes(int n, int H, int W) {
    int tx, tpf;
    if (!metrics::ssim_shape(n, H, W, &tx, &tpf)) return 0;
    return (size_t)n * tpf * sizeof(double);
}

extern "C" int neo_ssim(const float* pred, const float* gt, int n, int H, int W, double* ssim, float* ss_map, void* workspace,
                        size_t workspace_bytes, void* stream) {
    using namespace metrics;
    int tx, tpf;
    if (!pred || !gt || !ssim || !workspace) { set_error("neo_ssim: NULL pred / gt / ssim / workspace"); return NEO_ERR_INVALID; }
    if (!ssim_shape(n, H, W, &tx, &tpf)) {
        set_error("neo_ssim: n %d must be >= 1 and H %d, W %d >= 11, and the call must fit int64 elements and 2^31 - 1 tiles", n, H, W);
        return NEO_ERR_INVALID;
    }
    if (workspace_bytes < (size_t)n * tpf * sizeof(double) || (uintptr_t)workspace % alignof(double)) {
        set_error("neo_ssim: workspace needs %zu bytes, 8-byte aligned (got %zu)", (size_t)n * tpf * sizeof(double), workspace_bytes);
        return NEO_ERR_WORKSPACE;
    }
    double* partial = (double*)workspace;
    cudaStream_t s = (cudaStream_t)stream;
    ssim_tile_kernel<<<(unsigned)(n * tpf), kThreads, 0, s>>>(pred, gt, H, W, tx, tpf, ss_map, partial);
    NEO_LAUNCH_CHECK("ssim_tile_kernel");
    ssim_frame_kernel<<<(unsigned)n, kThreads, 0, s>>>(partial, tpf, 3.0 * (H - kLost) * (W - kLost), ssim);
    NEO_LAUNCH_CHECK("ssim_frame_kernel");
    return NEO_OK;
}
