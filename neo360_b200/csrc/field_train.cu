// Training form of the NeO-360 trunk (layers 0-3 of a NeRFPPMLP, projected formulation) on Hopper tensor cores: bf16 operands,
// fp32 accumulation, forward and backward.  Definition (training._mlp_projected, models/neo360/model.py:110-158):
//   enc = _pos_enc(cam, 0, 10)                                        (E = 21 in_ch columns, the reference's order)
//   h0 = relu(W0e enc + b0 + P0),  h1 = relu(W1 h0 + b1),  h2 = relu(W2 h1 + b2),  h3 = relu(W3h h2 + W3e enc + b3 + P3)
//   hbar = mean over the NV views of h3                               (row v M + j of the trunk is point j seen from view v)
// with [P0 | P3] = local_p + world_p, the looked-up projected rows (fp32, added to the accumulators unrounded).  The head after
// hbar stays with the caller: bottleneck -> views_linear.0 is linear and so is the view mean, so the head runs once per point.
//
// Rounding points (oracle/field_train_model.py): enc, W*, and the layer inputs h0, h1, h2 are bf16; h3 enters the mean in fp32.
// Backward: dz3 = (g_hbar / NV) [h3 > 0]; dz2 = (W3h^T bf16(dz3)) [h2 > 0]; dz1, dz0 likewise through W2, W1.  d_pm = [dz0 | dz3]
// (fp32) is the row gradient of both local_p and world_p.  Weight gradients are sums over rows of bf16(dz) x (the bf16 layer input);
// bias gradients are the sums of bf16(dz) (the constant-one column E of the saved encoding).
//
// Kernels: trunk_fwd / trunk_dgrad keep every weight matrix of the pass in shared memory (128-byte-swizzled K-major bf16 tiles) and
// run each layer as wgmma m64n128k16 with the activations as register A fragments, two warpgroups per CTA, one 64-point tile per
// warpgroup at a time, all NV views of a tile in turn.  The forward saves [enc | h0 | h1 | h2 | h3] per row in bf16, the dgrad
// [dz0 | dz1 | dz2 | dz3]; wgrad reduces them with mma.sync (ldmatrix.trans of row-major tiles) split over row ranges, and
// wgrad_reduce sums the partials in a fixed order: no floating-point atomics, two calls are bit-identical.
//
// PixelNeRF form (template parameter PIX; pixelnerf.NeRFMLP, models/vanilla_nerf/model_pixel.py:95-131 at skip_layer = netdepth = 4):
//   h0 = relu(W0e enc + b0 + p0),  h1, h2 as above,  h3 = relu(W3 h2 + b3),  hbar = mean over the NV views of h3
// with in_ch = 3 and p0 (nv*M, 128) = the looked-up rows of latent . W0[:, 63:575]^T.  Layer 3 has no encoding columns and no projected
// term, so the forward image is W0e | W1 | W2 | W3, the dgrad writes d_p0 = dz0 only, and wgrad job 4 is b3 alone (the constant-one
// encoding column, as b1 / b2).  The saved rows, the rounding points and the fixed-order reduction are those of the NeO-360 form
// (model: oracle/pixelnerf_train_tc_model.py).
#include "common.cuh"
#include "hopper.cuh"
#include <cuda_bf16.h>
#include <algorithm>

namespace neo {
namespace ftrain {
using namespace hopper;

constexpr int kTile = 64;                       // rows of one wgmma
constexpr int kWarpgroups = 2;
constexpr int kThreads = 128 * kWarpgroups;
constexpr uint32_t SLAB = 128 * 128;            // one 64-column slab of a 128-row bf16 tile
constexpr int kSplits = 128;                    // row ranges of the weight-gradient reduction (fixed: the sum order does not depend on the GPU)
constexpr int kJobs = 7;
constexpr int kPad = 136;                       // row stride (bf16) of the wgrad shared-memory tiles: ldmatrix rows on distinct banks

__host__ __device__ constexpr int enc_slabs(int KE) { return KE / 64 + (KE % 64 != 0); }
// forward image: W0e | W1 | W2 | W3h | W3e (128 rows each, K-major slabs; the PixelNeRF form ends at W3); backward image: W3h^T | W2^T | W1^T
__host__ __device__ constexpr uint32_t fwd_off(int KE, int seg) { return seg == 0 ? 0u : (uint32_t)(enc_slabs(KE) + 2 * (seg - 1)) * SLAB; }
__host__ __device__ constexpr uint32_t fwd_bytes(int KE, bool pix = false) { return fwd_off(KE, 4) + (pix ? 0u : (uint32_t)enc_slabs(KE) * SLAB); }
constexpr uint32_t BWD_BYTES = 6 * SLAB;

struct Dims {
    int nv, M, ich, E, KE, XS;                  // XS: bf16 per saved row = KE + 512
    long long R;                                // nv * M trunk rows
};
__host__ __device__ inline Dims make_dims(int nv, int M, int ich) {
    Dims d;
    d.nv = nv; d.M = M; d.ich = ich; d.E = 21 * ich; d.KE = ich == 3 ? 64 : 96; d.XS = d.KE + 512; d.R = (long long)nv * M;
    return d;
}
static size_t align_up(size_t x) { return (x + 1023) & ~(size_t)1023; }
static size_t saved_bytes(const Dims& d, bool pix = false) { return align_up((size_t)d.R * d.XS * 2) + align_up(fwd_bytes(d.KE, pix)); }
static size_t scratch_bytes(const Dims& d) {
    return align_up((size_t)d.R * 512 * 2) + align_up(BWD_BYTES) + (size_t)kSplits * kJobs * 128 * 128 * 4;
}

__device__ __forceinline__ uint32_t pack_bf2(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack_bf2(uint32_t u) { return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u)); }

// column c of _pos_enc(x, 0, 10) (helper.py:121-125): [x, sin(2^l x_c) (l-major), sin(2^l x_c + pi/2)]; column E is the constant
// one that carries the bias gradients; zero beyond
template <int ICH>
__device__ __forceinline__ float enc_val(const float (&x)[4], int c) {
    constexpr int E = 21 * ICH;
    if (c < ICH) return x[c];
    if (c < E) {
        const bool shifted = c >= 11 * ICH;
        const int k = c - (shifted ? 11 * ICH : ICH), l = k / ICH, cc = k - l * ICH;
        const float xb = x[cc] * (float)(1 << l);
        return sinf(shifted ? xb + 1.57079637f : xb);
    }
    return c == E ? 1.f : 0.f;
}

// ld3: row stride of w3, 128 + E with its encoding columns (segment W3e follows), 128 without (PixelNeRF form: no segment 4)
__global__ void fwd_img_kernel(const float* __restrict__ w0, const float* __restrict__ w1, const float* __restrict__ w2,
                               const float* __restrict__ w3, int E, int KE, int ld3, unsigned char* __restrict__ img) {
    const int es = enc_slabs(KE) * 64, KW = (ld3 > 128 ? 2 * es : es) + 384;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= KW * 128) return;
    const int n = idx / KW, kk = idx % KW;
    int seg, k;
    float x;
    if (kk < es) { seg = 0; k = kk; x = k < E ? w0[n * E + k] : 0.f; }
    else if (kk < es + 128) { seg = 1; k = kk - es; x = w1[n * 128 + k]; }
    else if (kk < es + 256) { seg = 2; k = kk - es - 128; x = w2[n * 128 + k]; }
    else if (kk < es + 384) { seg = 3; k = kk - es - 256; x = w3[n * ld3 + k]; }
    else { seg = 4; k = kk - es - 384; x = k < E ? w3[n * ld3 + 128 + k] : 0.f; }
    *reinterpret_cast<__nv_bfloat16*>(img + fwd_off(KE, seg) + sw128_off(n, k, 128)) = __float2bfloat16_rn(x);
}
// element (n, k) of W^T for W = W3h, W2, W1: B operand of dh_in = dz_out . W (ld3: row stride of w3)
__global__ void bwd_img_kernel(const float* __restrict__ w1, const float* __restrict__ w2, const float* __restrict__ w3, int ld3,
                               unsigned char* __restrict__ img) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= 3 * 128 * 128) return;
    const int s = idx / (128 * 128), n = (idx / 128) % 128, k = idx % 128;
    const float x = s == 0 ? w3[k * ld3 + n] : s == 1 ? w2[k * 128 + n] : w1[k * 128 + n];
    *reinterpret_cast<__nv_bfloat16*>(img + (uint32_t)s * 2 * SLAB + sw128_off(n, k, 128)) = __float2bfloat16_rn(x);
}

__device__ __forceinline__ uint64_t wdesc(uint32_t base, int ks) { return desc_sw128(base + (uint32_t)(ks >> 2) * SLAB + (uint32_t)(ks & 3) * 32u); }

// cooperative copy of a weight image into shared memory, then made visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void load_image(unsigned char* dst, const unsigned char* src, uint32_t bytes) {
    const uint4* s = reinterpret_cast<const uint4*>(src);
    uint4* d = reinterpret_cast<uint4*>(dst);
    for (uint32_t i = threadIdx.x; i < bytes / 16; i += blockDim.x) d[i] = __ldg(s + i);
    fence_proxy_async();
    __syncthreads();
}

struct FwdParams {
    const float *cam, *local_p, *world_p, *b0, *b1, *b2, *b3;    // PixelNeRF form: local_p = p0 (nv*M, 128), world_p unused
    const unsigned char* img;
    Dims d;
    int n_tiles;
    float* hbar;
    __nv_bfloat16* X;
};

// accumulator element k = 4 j + 2 i + e of a thread (warp w, lane l): row 16 w + l / 4 + 8 i, column 8 j + 2 (l % 4) + e
template <int ICH, bool PIX>
__global__ void __launch_bounds__(kThreads, 1) trunk_fwd(const __grid_constant__ FwdParams P) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
    unsigned char* sgen = smem_raw + (sbase - smem_u32(smem_raw));
    constexpr int KE = ICH == 3 ? 64 : 96, KS = KE / 16;
    load_image(sgen, P.img, fwd_bytes(KE, PIX));
    const Dims& D = P.d;
    const int wg = threadIdx.x >> 7, wt = threadIdx.x & 127, warp = wt >> 5, lane = threadIdx.x & 31, t = lane & 3;
    const int r0 = warp * 16 + (lane >> 2);
    const float inv_nv = 1.0f / (float)D.nv;
    for (int tile = blockIdx.x * kWarpgroups + wg; tile < P.n_tiles; tile += gridDim.x * kWarpgroups) {
        int jr[2];
        bool ok[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) { jr[i] = tile * kTile + r0 + 8 * i; ok[i] = jr[i] < D.M; }
#pragma unroll 1
        for (int v = 0; v < D.nv; ++v) {
            long long row[2];
            uint32_t enc[KS][4];
            {
                float x[2][4];
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    row[i] = (long long)v * D.M + jr[i];
#pragma unroll
                    for (int c = 0; c < 4; ++c) x[i][c] = (ok[i] && c < ICH) ? P.cam[row[i] * ICH + c] : 0.f;
                }
#pragma unroll
                for (int ks = 0; ks < KS; ++ks)
#pragma unroll
                    for (int r = 0; r < 4; ++r) {
                        const int c = 16 * ks + 8 * (r >> 1) + 2 * t;
                        enc[ks][r] = pack_bf2(enc_val<ICH>(x[r & 1], c), enc_val<ICH>(x[r & 1], c + 1));
                    }
            }
            auto seed = [&](float (&acc)[64], int half, const float* b) {      // projected rows + bias, fp32
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int c = 8 * j + 2 * t;
                    const float2 bb = make_float2(__ldg(b + c), __ldg(b + c + 1));
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        float2 s = make_float2(0.f, 0.f);
                        if (PIX && half == 0 && ok[i]) {
                            s = __ldg(reinterpret_cast<const float2*>(P.local_p + row[i] * 128 + c));
                        } else if (!PIX && half >= 0 && ok[i]) {
                            const float2 l = __ldg(reinterpret_cast<const float2*>(P.local_p + row[i] * 256 + 128 * half + c));
                            const float2 w = __ldg(reinterpret_cast<const float2*>(P.world_p + row[i] * 256 + 128 * half + c));
                            s = make_float2(l.x + w.x, l.y + w.y);
                        }
                        acc[4 * j + 2 * i] = s.x + bb.x;
                        acc[4 * j + 2 * i + 1] = s.y + bb.y;
                    }
                }
            };
            // rectify, save as bf16 at column offset `col0` of the saved row, and pack as the next layer's A fragments
            auto relu_save = [&](float (&acc)[64], uint32_t (&a)[8][4], int col0) {
#pragma unroll
                for (int ks = 0; ks < 8; ++ks)
#pragma unroll
                    for (int r = 0; r < 4; ++r) {
                        acc[8 * ks + 2 * r] = fmaxf(acc[8 * ks + 2 * r], 0.f);
                        acc[8 * ks + 2 * r + 1] = fmaxf(acc[8 * ks + 2 * r + 1], 0.f);
                        a[ks][r] = pack_bf2(acc[8 * ks + 2 * r], acc[8 * ks + 2 * r + 1]);
                        const int i = r & 1, c = 16 * ks + 8 * (r >> 1) + 2 * t;
                        if (ok[i]) *reinterpret_cast<uint32_t*>(P.X + row[i] * D.XS + col0 + c) = a[ks][r];
                    }
            };
            float acc[64];
            uint32_t a[8][4];
            seed(acc, 0, P.b0);
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) wgmma_rs_n128_bf16(acc, enc[ks], wdesc(sbase + fwd_off(KE, 0), ks));
            wgmma_commit();
            wgmma_wait<0>();
            relu_save(acc, a, KE);
#pragma unroll 1
            for (int l = 1; l <= 2; ++l) {
                seed(acc, -1, l == 1 ? P.b1 : P.b2);
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < 8; ++ks) wgmma_rs_n128_bf16(acc, a[ks], wdesc(sbase + fwd_off(KE, l), ks));
                wgmma_commit();
                wgmma_wait<0>();
                relu_save(acc, a, KE + 128 * l);
            }
            seed(acc, PIX ? -1 : 1, P.b3);
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) wgmma_rs_n128_bf16(acc, a[ks], wdesc(sbase + fwd_off(KE, 3), ks));
            if constexpr (!PIX) {
#pragma unroll
                for (int ks = 0; ks < KS; ++ks) wgmma_rs_n128_bf16(acc, enc[ks], wdesc(sbase + fwd_off(KE, 4), ks));
            }
            wgmma_commit();
            wgmma_wait<0>();
            relu_save(acc, a, KE + 384);
            // hbar: the view sum runs in this thread's own elements of the output (registers would spill), in view order
#pragma unroll
            for (int j = 0; j < 16; ++j)
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    if (!ok[i]) continue;
                    float2* dst = reinterpret_cast<float2*>(P.hbar + (long long)jr[i] * 128 + 8 * j + 2 * t);
                    float2 h = make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
                    if (v > 0) { const float2 p = *dst; h = make_float2(p.x + h.x, p.y + h.y); }
                    if (v == D.nv - 1) h = make_float2(h.x * inv_nv, h.y * inv_nv);
                    *dst = h;
                }
#pragma unroll
            for (int ks = 0; ks < KS; ++ks)
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const int i = r & 1;
                    if (ok[i]) *reinterpret_cast<uint32_t*>(P.X + row[i] * D.XS + 16 * ks + 8 * (r >> 1) + 2 * t) = enc[ks][r];
                }
        }
    }
}

struct BwdParams {
    const float* g_hbar;
    const __nv_bfloat16* X;
    const unsigned char* img;
    Dims d;
    int n_tiles;
    float* d_pm;                                   // PixelNeRF form: d_p0 (nv*M, 128)
    __nv_bfloat16* G;
};

template <bool PIX>
__global__ void __launch_bounds__(kThreads, 1) trunk_dgrad(const __grid_constant__ BwdParams P) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
    unsigned char* sgen = smem_raw + (sbase - smem_u32(smem_raw));
    load_image(sgen, P.img, BWD_BYTES);
    const Dims& D = P.d;
    const int wg = threadIdx.x >> 7, wt = threadIdx.x & 127, warp = wt >> 5, lane = threadIdx.x & 31, t = lane & 3;
    const int r0 = warp * 16 + (lane >> 2);
    const float fnv = (float)D.nv;
    for (int tile = blockIdx.x * kWarpgroups + wg; tile < P.n_tiles; tile += gridDim.x * kWarpgroups) {
        int jr[2];
        bool ok[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) { jr[i] = tile * kTile + r0 + 8 * i; ok[i] = jr[i] < D.M; }
        float gb[64];
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                float2 g = make_float2(0.f, 0.f);
                if (ok[i]) g = __ldg(reinterpret_cast<const float2*>(P.g_hbar + (long long)jr[i] * 128 + 8 * j + 2 * t));
                gb[4 * j + 2 * i] = g.x / fnv;
                gb[4 * j + 2 * i + 1] = g.y / fnv;
            }
#pragma unroll 1
        for (int v = 0; v < D.nv; ++v) {
            long long row[2];
#pragma unroll
            for (int i = 0; i < 2; ++i) row[i] = (long long)v * D.M + jr[i];
            // dz = dh [h > 0] with h the saved bf16 activation at column xcol; saved at G column gcol (bf16) and, for layers 0 and 3
            // (layer 0 alone in the PixelNeRF form), written to d_pm (fp32); packed as the A fragments of the next product
            constexpr int ldpm = PIX ? 128 : 256;
            auto mask_save = [&](float (&dz)[64], uint32_t (&a)[8][4], int xcol, int gcol, int pmcol) {
#pragma unroll
                for (int j = 0; j < 16; ++j)
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        const int c = 8 * j + 2 * t;
                        float2 h = make_float2(0.f, 0.f);
                        if (ok[i]) h = unpack_bf2(__ldg(reinterpret_cast<const unsigned int*>(P.X + row[i] * D.XS + xcol + c)));
                        float& z0 = dz[4 * j + 2 * i];
                        float& z1 = dz[4 * j + 2 * i + 1];
                        z0 = h.x > 0.f ? z0 : 0.f;
                        z1 = h.y > 0.f ? z1 : 0.f;
                        const uint32_t p = pack_bf2(z0, z1);
                        a[j >> 1][2 * (j & 1) + i] = p;
                        if (ok[i]) {
                            *reinterpret_cast<uint32_t*>(P.G + row[i] * 512 + gcol + c) = p;
                            if (pmcol >= 0) *reinterpret_cast<float2*>(P.d_pm + row[i] * ldpm + pmcol + c) = make_float2(z0, z1);
                        }
                    }
            };
            float dz[64];
            uint32_t a[8][4];
#pragma unroll
            for (int k = 0; k < 64; ++k) dz[k] = gb[k];
            mask_save(dz, a, D.KE + 384, 384, PIX ? -1 : 128);            // dz3
#pragma unroll 1
            for (int l = 0; l < 3; ++l) {                                 // through W3h, W2, W1: dz2, dz1, dz0
#pragma unroll
                for (int k = 0; k < 64; ++k) dz[k] = 0.f;
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < 8; ++ks) wgmma_rs_n128_bf16(dz, a[ks], wdesc(sbase + (uint32_t)l * 2 * SLAB, ks));
                wgmma_commit();
                wgmma_wait<0>();
                mask_save(dz, a, D.KE + 256 - 128 * l, 256 - 128 * l, l == 2 ? 0 : -1);
            }
        }
    }
}

// Weight-gradient jobs: dW_job[o][k] = sum over rows of G[row][gcol + o] X[row][xcol + k], o < 128, k < K
struct Job { int gcol, xcol, K; };
__host__ __device__ inline Job job_of(int j, int KE, bool pix) {
    switch (j) {
        case 0: return {0, 0, KE};                   // W0e | b0 (constant-one column E)
        case 1: return {128, KE, 128};               // W1
        case 2: return {256, KE + 128, 128};         // W2
        case 3: return {384, KE + 256, 128};         // W3h
        case 4: return pix ? Job{384, KE - 16, 16}   // b3 (PixelNeRF form: W3 has no encoding columns)
                           : Job{384, 0, KE};        // W3e | b3
        case 5: return {128, KE - 16, 16};           // b1 (the constant-one column within the last 16 encoding columns)
        default: return {256, KE - 16, 16};          // b2
    }
}

__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

struct WgradParams {
    const __nv_bfloat16 *X, *G;
    Dims d;
    long long chunks;                              // 64-row chunks
    float* part;                                   // [split][job][128][128]
};

// CTA (job, split): 8 warps, warp w owns output rows o = 16 w .. 16 w + 15 and every k; the 64-row chunks of the split stream through
// row-major shared-memory tiles, read as transposed fragments by ldmatrix.trans
template <int KMAX>
__device__ __forceinline__ void wgrad_body(const WgradParams& P, const Job jb, int split, __nv_bfloat16 (*Gs)[kPad], __nv_bfloat16 (*Xs)[kPad]) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float acc[KMAX / 8][4];
#pragma unroll
    for (int n = 0; n < KMAX / 8; ++n)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[n][e] = 0.f;
    const long long c0 = P.chunks * split / kSplits, c1 = P.chunks * (split + 1) / kSplits;
    const int K = jb.K;
    for (long long ch = c0; ch < c1; ++ch) {
        __syncthreads();
        for (int idx = threadIdx.x; idx < 64 * 16; idx += kThreads) {         // G: 64 rows x 128 columns, 16-byte pieces
            const int r = idx >> 4, p = idx & 15;
            const long long row = ch * 64 + r;
            uint4 q = make_uint4(0, 0, 0, 0);
            if (row < P.d.R) q = __ldg(reinterpret_cast<const uint4*>(P.G + row * 512 + jb.gcol) + p);
            *reinterpret_cast<uint4*>(&Gs[r][8 * p]) = q;
        }
        for (int idx = threadIdx.x; idx < 64 * (K / 8); idx += kThreads) {
            const int r = idx / (K / 8), p = idx % (K / 8);
            const long long row = ch * 64 + r;
            uint4 q = make_uint4(0, 0, 0, 0);
            if (row < P.d.R) q = __ldg(reinterpret_cast<const uint4*>(P.X + row * P.d.XS + jb.xcol) + p);
            *reinterpret_cast<uint4*>(&Xs[r][8 * p]) = q;
        }
        __syncthreads();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            uint32_t a[4];
            ldsm_x4_t(a, smem_u32(&Gs[16 * ks + (lane & 7) + ((lane >> 4) << 3)][16 * warp + ((lane >> 3) & 1) * 8]));
#pragma unroll
            for (int p = 0; p < KMAX / 16; ++p) {
                if (16 * p >= K) break;
                uint32_t b[4];
                ldsm_x4_t(b, smem_u32(&Xs[16 * ks + (lane & 7) + ((lane >> 3) & 1) * 8][16 * p + (lane >> 4) * 8]));
                mma_bf16(acc[2 * p], a, b[0], b[1]);
                mma_bf16(acc[2 * p + 1], a, b[2], b[3]);
            }
        }
    }
    const int g = lane >> 2, t = lane & 3;
    float* out = P.part + ((size_t)split * kJobs + blockIdx.x % kJobs) * 128 * 128;
#pragma unroll
    for (int n = 0; n < KMAX / 8; ++n) {
        if (8 * n >= K) break;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int o = 16 * warp + g + 8 * h, k = 8 * n + 2 * t;
            *reinterpret_cast<float2*>(out + o * 128 + k) = make_float2(acc[n][2 * h], acc[n][2 * h + 1]);
        }
    }
}

template <bool PIX>
__global__ void __launch_bounds__(kThreads) wgrad(const __grid_constant__ WgradParams P) {
    __shared__ __align__(16) __nv_bfloat16 Gs[64][kPad];
    __shared__ __align__(16) __nv_bfloat16 Xs[64][kPad];
    const int job = blockIdx.x % kJobs, split = blockIdx.x / kJobs;
    const Job jb = job_of(job, P.d.KE, PIX);
    if (jb.K == 16) wgrad_body<16>(P, jb, split, Gs, Xs);
    else wgrad_body<128>(P, jb, split, Gs, Xs);
}

struct GradOut { float *gw0, *gb0, *gw1, *gb1, *gw2, *gb2, *gw3, *gb3; };

// fixed-order sum of the partials of every job, scattered into nn.Linear layout: gw0 (128, E), gw3 (128, 128 + E; PixelNeRF form (128, 128))
template <bool PIX>
__global__ void wgrad_reduce(const float* __restrict__ part, Dims D, GradOut out) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= kJobs * 128 * 128) return;
    const int job = idx / (128 * 128), o = (idx / 128) % 128, k = idx % 128;
    const Job jb = job_of(job, D.KE, PIX);
    if (k >= jb.K) return;
    const int E = D.E, one = E - (D.KE - 16);
    float* dst = nullptr;
    switch (job) {
        case 0: dst = k < E ? out.gw0 + o * E + k : k == E ? out.gb0 + o : nullptr; break;
        case 1: dst = out.gw1 + o * 128 + k; break;
        case 2: dst = out.gw2 + o * 128 + k; break;
        case 3: dst = out.gw3 + o * (PIX ? 128 : 128 + E) + k; break;
        case 4: dst = PIX ? (k == one ? out.gb3 + o : nullptr) : k < E ? out.gw3 + o * (128 + E) + 128 + k : k == E ? out.gb3 + o : nullptr; break;
        case 5: dst = k == one ? out.gb1 + o : nullptr; break;
        default: dst = k == one ? out.gb2 + o : nullptr; break;
    }
    if (!dst) return;
    float s = 0.f;
    for (int sp = 0; sp < kSplits; ++sp) s += part[((size_t)sp * kJobs + job) * 128 * 128 + o * 128 + k];
    *dst = s;
}

static int n_sms() {
    static int n_sm_of[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 0;
    if (!n_sm_of[dev]) cudaDeviceGetAttribute(&n_sm_of[dev], cudaDevAttrMultiProcessorCount, dev);
    return n_sm_of[dev];
}

static int check_dims(int nv, int M, int in_ch) {
    if (nv < 1 || nv > kMaxViews) { set_error("field_train: nv = %d outside 1..%d", nv, kMaxViews); return NEO_ERR_INVALID; }
    if (in_ch != 3 && in_ch != 4) { set_error("field_train: in_ch = %d, must be 3 or 4", in_ch); return NEO_ERR_INVALID; }
    if (M <= 0) { set_error("field_train: M = %d, must be positive", M); return NEO_ERR_INVALID; }
    if ((long long)nv * M > (1LL << 31) / 64) { set_error("field_train: nv * M = %lld rows is too many", (long long)nv * M); return NEO_ERR_INVALID; }
    return NEO_OK;
}

// The launches of the forward and backward once the arguments are checked.  PIX: p0 in local_p, world_p unused, w3 (128, 128).
template <bool PIX>
static int launch_fwd(const char* name, const float* cam, const float* local_p, const float* world_p, const Dims& d, const float* w0,
                      const float* b0, const float* w1, const float* b1, const float* w2, const float* b2, const float* w3, const float* b3,
                      float* hbar, void* saved, cudaStream_t s) {
    unsigned char* base = (unsigned char*)saved;
    FwdParams P;
    P.cam = cam; P.local_p = local_p; P.world_p = world_p; P.b0 = b0; P.b1 = b1; P.b2 = b2; P.b3 = b3;
    P.d = d; P.hbar = hbar;
    P.X = (__nv_bfloat16*)base;
    unsigned char* img = base + align_up((size_t)d.R * d.XS * 2);
    P.img = img;
    const int nimg = ((PIX ? 1 : 2) * enc_slabs(d.KE) * 64 + 384) * 128;
    fwd_img_kernel<<<(nimg + 255) / 256, 256, 0, s>>>(w0, w1, w2, w3, d.E, d.KE, PIX ? 128 : 128 + d.E, img);
    NEO_LAUNCH_CHECK("fwd_img_kernel");
    P.n_tiles = (d.M + kTile - 1) / kTile;
    const int nsm = n_sms();
    if (nsm <= 0) { set_error("%s: no device", name); return NEO_ERR_CUDA; }
    const int grid = std::min((P.n_tiles + kWarpgroups - 1) / kWarpgroups, nsm);
    const size_t smem = fwd_bytes(d.KE, PIX) + 1024;
    void (*kern)(const FwdParams) = trunk_fwd<3, PIX>;
    if constexpr (!PIX) if (d.ich == 4) kern = trunk_fwd<4, false>;
    NEO_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, kThreads, smem, s>>>(P);
    NEO_LAUNCH_CHECK("trunk_fwd");
    return NEO_OK;
}

template <bool PIX>
static int launch_bwd(const char* name, const float* g_hbar, const Dims& d, const float* w1, const float* w2, const float* w3,
                      const void* saved, float* d_pm, const GradOut& go, void* scratch, cudaStream_t s) {
    unsigned char* sc = (unsigned char*)scratch;
    BwdParams P;
    P.g_hbar = g_hbar; P.X = (const __nv_bfloat16*)saved; P.d = d; P.d_pm = d_pm;
    P.G = (__nv_bfloat16*)sc;
    unsigned char* img = sc + align_up((size_t)d.R * 512 * 2);
    float* part = (float*)(img + align_up(BWD_BYTES));
    P.img = img;
    bwd_img_kernel<<<(3 * 128 * 128 + 255) / 256, 256, 0, s>>>(w1, w2, w3, PIX ? 128 : 128 + d.E, img);
    NEO_LAUNCH_CHECK("bwd_img_kernel");
    P.n_tiles = (d.M + kTile - 1) / kTile;
    const int nsm = n_sms();
    if (nsm <= 0) { set_error("%s: no device", name); return NEO_ERR_CUDA; }
    const int grid = std::min((P.n_tiles + kWarpgroups - 1) / kWarpgroups, nsm);
    const size_t smem = BWD_BYTES + 1024;
    NEO_CUDA(cudaFuncSetAttribute(trunk_dgrad<PIX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    trunk_dgrad<PIX><<<grid, kThreads, smem, s>>>(P);
    NEO_LAUNCH_CHECK("trunk_dgrad");
    WgradParams W;
    W.X = P.X; W.G = P.G; W.d = d; W.chunks = (d.R + 63) / 64; W.part = part;
    wgrad<PIX><<<kSplits * kJobs, kThreads, 0, s>>>(W);
    NEO_LAUNCH_CHECK("wgrad");
    wgrad_reduce<PIX><<<(kJobs * 128 * 128 + 255) / 256, 256, 0, s>>>(part, d, go);
    NEO_LAUNCH_CHECK("wgrad_reduce");
    return NEO_OK;
}

}  // namespace ftrain
}  // namespace neo

using namespace neo::ftrain;

extern "C" size_t neo_field_train_workspace_bytes(int nv, int M, int in_ch, int which) {
    if (check_dims(nv, M, in_ch) != NEO_OK || (which != 0 && which != 1)) return 0;
    const Dims d = make_dims(nv, M, in_ch);
    return which == 0 ? saved_bytes(d) : scratch_bytes(d);
}

extern "C" int neo_field_train_fwd(const float* cam, const float* local_p, const float* world_p, int nv, int M, int in_ch,
                                   const float* w0, const float* b0, const float* w1, const float* b1, const float* w2, const float* b2,
                                   const float* w3, const float* b3, float* hbar, void* saved, size_t saved_size, void* stream) {
    int rc = check_dims(nv, M, in_ch);
    if (rc) return rc;
    if (!cam || !local_p || !world_p || !w0 || !b0 || !w1 || !b1 || !w2 || !b2 || !w3 || !b3 || !hbar || !saved) {
        neo::set_error("neo_field_train_fwd: NULL buffer"); return NEO_ERR_INVALID;
    }
    const Dims d = make_dims(nv, M, in_ch);
    if (saved_size < saved_bytes(d)) { neo::set_error("neo_field_train_fwd: saved-state workspace of %zu bytes, %zu needed", saved_size, saved_bytes(d)); return NEO_ERR_WORKSPACE; }
    if ((reinterpret_cast<uintptr_t>(local_p) | reinterpret_cast<uintptr_t>(world_p) | reinterpret_cast<uintptr_t>(hbar) |
         reinterpret_cast<uintptr_t>(saved)) & 15) { neo::set_error("neo_field_train_fwd: buffers must be 16-byte aligned"); return NEO_ERR_INVALID; }
    return launch_fwd<false>("neo_field_train_fwd", cam, local_p, world_p, d, w0, b0, w1, b1, w2, b2, w3, b3, hbar, saved, (cudaStream_t)stream);
}

extern "C" int neo_field_train_bwd(const float* g_hbar, int nv, int M, int in_ch, const float* w1, const float* w2, const float* w3,
                                   const void* saved, size_t saved_size, float* d_pm, float* gw0, float* gb0, float* gw1, float* gb1,
                                   float* gw2, float* gb2, float* gw3, float* gb3, void* scratch, size_t scratch_size, void* stream) {
    int rc = check_dims(nv, M, in_ch);
    if (rc) return rc;
    if (!g_hbar || !w1 || !w2 || !w3 || !saved || !d_pm || !gw0 || !gb0 || !gw1 || !gb1 || !gw2 || !gb2 || !gw3 || !gb3 || !scratch) {
        neo::set_error("neo_field_train_bwd: NULL buffer"); return NEO_ERR_INVALID;
    }
    const Dims d = make_dims(nv, M, in_ch);
    if (saved_size < saved_bytes(d) || scratch_size < scratch_bytes(d)) {
        neo::set_error("neo_field_train_bwd: workspaces of %zu / %zu bytes, %zu / %zu needed", saved_size, scratch_size, saved_bytes(d), scratch_bytes(d));
        return NEO_ERR_WORKSPACE;
    }
    if ((reinterpret_cast<uintptr_t>(g_hbar) | reinterpret_cast<uintptr_t>(d_pm) | reinterpret_cast<uintptr_t>(saved) |
         reinterpret_cast<uintptr_t>(scratch)) & 15) { neo::set_error("neo_field_train_bwd: buffers must be 16-byte aligned"); return NEO_ERR_INVALID; }
    return launch_bwd<false>("neo_field_train_bwd", g_hbar, d, w1, w2, w3, saved, d_pm, GradOut{gw0, gb0, gw1, gb1, gw2, gb2, gw3, gb3},
                             scratch, (cudaStream_t)stream);
}

// PixelNeRF form: in_ch = 3, p0 (nv*M, 128) in place of [P0 | P3], w3 (128, 128), d_p0 (nv*M, 128)
extern "C" size_t neo_pixelnerf_train_workspace_bytes(int nv, int M, int which) {
    if (check_dims(nv, M, 3) != NEO_OK || (which != 0 && which != 1)) return 0;
    const Dims d = make_dims(nv, M, 3);
    return which == 0 ? saved_bytes(d, true) : scratch_bytes(d);
}

extern "C" int neo_pixelnerf_train_fwd(const float* cam, const float* p0, int nv, int M, const float* w0, const float* b0, const float* w1,
                                       const float* b1, const float* w2, const float* b2, const float* w3, const float* b3, float* hbar,
                                       void* saved, size_t saved_size, void* stream) {
    int rc = check_dims(nv, M, 3);
    if (rc) return rc;
    if (!cam || !p0 || !w0 || !b0 || !w1 || !b1 || !w2 || !b2 || !w3 || !b3 || !hbar || !saved) {
        neo::set_error("neo_pixelnerf_train_fwd: NULL buffer"); return NEO_ERR_INVALID;
    }
    const Dims d = make_dims(nv, M, 3);
    if (saved_size < saved_bytes(d, true)) {
        neo::set_error("neo_pixelnerf_train_fwd: saved-state workspace of %zu bytes, %zu needed", saved_size, saved_bytes(d, true));
        return NEO_ERR_WORKSPACE;
    }
    if ((reinterpret_cast<uintptr_t>(p0) | reinterpret_cast<uintptr_t>(hbar) | reinterpret_cast<uintptr_t>(saved)) & 15) {
        neo::set_error("neo_pixelnerf_train_fwd: buffers must be 16-byte aligned"); return NEO_ERR_INVALID;
    }
    return launch_fwd<true>("neo_pixelnerf_train_fwd", cam, p0, nullptr, d, w0, b0, w1, b1, w2, b2, w3, b3, hbar, saved, (cudaStream_t)stream);
}

extern "C" int neo_pixelnerf_train_bwd(const float* g_hbar, int nv, int M, const float* w1, const float* w2, const float* w3, const void* saved,
                                       size_t saved_size, float* d_p0, float* gw0, float* gb0, float* gw1, float* gb1, float* gw2, float* gb2,
                                       float* gw3, float* gb3, void* scratch, size_t scratch_size, void* stream) {
    int rc = check_dims(nv, M, 3);
    if (rc) return rc;
    if (!g_hbar || !w1 || !w2 || !w3 || !saved || !d_p0 || !gw0 || !gb0 || !gw1 || !gb1 || !gw2 || !gb2 || !gw3 || !gb3 || !scratch) {
        neo::set_error("neo_pixelnerf_train_bwd: NULL buffer"); return NEO_ERR_INVALID;
    }
    const Dims d = make_dims(nv, M, 3);
    if (saved_size < saved_bytes(d, true) || scratch_size < scratch_bytes(d)) {
        neo::set_error("neo_pixelnerf_train_bwd: workspaces of %zu / %zu bytes, %zu / %zu needed", saved_size, scratch_size,
                       saved_bytes(d, true), scratch_bytes(d));
        return NEO_ERR_WORKSPACE;
    }
    if ((reinterpret_cast<uintptr_t>(g_hbar) | reinterpret_cast<uintptr_t>(d_p0) | reinterpret_cast<uintptr_t>(saved) |
         reinterpret_cast<uintptr_t>(scratch)) & 15) { neo::set_error("neo_pixelnerf_train_bwd: buffers must be 16-byte aligned"); return NEO_ERR_INVALID; }
    return launch_bwd<true>("neo_pixelnerf_train_bwd", g_hbar, d, w1, w2, w3, saved, d_p0, GradOut{gw0, gb0, gw1, gb1, gw2, gb2, gw3, gb3},
                            scratch, (cudaStream_t)stream);
}
