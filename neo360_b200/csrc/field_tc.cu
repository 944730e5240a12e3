// NEO_PREC_TC: the radiance field of NeO-360 on Hopper tensor cores (sm_90a wgmma), weights resident in shared memory.
//
// Formulation (exact re-association of models/neo360/model.py:110-158, see DESIGN.md "TC path"):
//   * bilinear lookups are linear, so the latent columns of layers 0 and 3 are applied to the feature maps once per
//     scene:  P0 = W0[:, enc:] . F,  P3 = W3[:, 128+enc:] . F  (F = pixel-aligned latent or a tri-plane).  Per sample
//     the kernel blends 4 taps of [P0|P3] (256 fp16 channels) from 4 maps instead of 4 taps of 512+3*128 raw channels.
//   * bottleneck_layer -> views_linear.0 has no nonlinearity in between and the view mean is linear, so
//       q = (Wv0[:, :128] Wb / NV) . sum_v h3_v + Wv0[:, 128:] . mean_v(dir_enc_v) + (Wv0[:, :128] bb + bv0)
//       sigma_raw = (w_sigma / NV) . sum_v h3_v + b_sigma
//     i.e. the cross-view means become one register accumulator summed over the views.
//   * b0 and b3 ride on a constant-one column of the positional encoding; b1, b2 and the head biases seed the accumulators.
//
// Layout: one persistent CTA per SM, three warpgroups.  Two consumer warpgroups each work on their own tiles of 64 points (32 rays x 2
// consecutive samples); the producer warpgroup builds their geometry (points, camera-frame encodings, tap tables: 64 threads per
// consumer, one point each) and hands it over through full / empty mbarrier pairs, so the consumers only blend and multiply.  A tile's
// rows (and, in the background, its view-independent s encoding columns) go over once per tile, then the encodings and tap table of
// one view at a time: the producer builds the next tile's rows and first view while the consumer is still on its current tile.
// setmaxnreg moves registers from the producer (56) to the consumers (224).
// The rays of a tile are 32 consecutive slots of the ray order (one 8x4 pixel block of a frame, renderer._blocked_order): rays that
// close together read the same texels at a sample, while consecutive samples move on to the next texel, so a tile that spans more
// rays and fewer samples reads fewer distinct texels per point (on H100 the field launches are 1.11x faster than with 16 rays x 4
// samples, DESIGN.md §5).
// Every weight matrix of the branch's MLP (trunk, folded head, colour head: up to 200 KB fp16, 128-byte-swizzled K-major tiles) is
// copied into shared memory once per CTA by TMA bulk copies.  Per (tile, view) a warpgroup runs the whole MLP as wgmma.mma_async
// m64nNk16 with the activations as REGISTER A fragments: the fp32 accumulator of one layer is rectified, packed to fp16 and fed to
// the next layer without touching shared memory.  The projected-map blends are added straight into the accumulators of layers 0 and
// 3: the projected maps are stored with their channels in the accumulator-fragment order (pmap_logical), so the 32 channels a thread
// owns for a point are four 16-byte chunks of each texel, one per 64-byte block (four 16-byte loads per tap; each load of a quad
// of lanes is one contiguous 64-byte block, the four together a whole 256-byte half row).
#include "common.cuh"
#include "hopper.cuh"
#include <cuda.h>
#include <cuda_fp16.h>
#include <cstdio>
#include <cstring>

namespace neo {
namespace tc {
using namespace hopper;

constexpr int kTileRays = 32;
constexpr int kTileSamples = 2;
constexpr int kTilePts = kTileRays * kTileSamples;  // = the M of one wgmma
constexpr int kConsumers = 2;                        // MMA warpgroups 0, 1; warpgroup 2 is the producer
constexpr int kThreads = 128 * (kConsumers + 1);
// setmaxnreg only moves registers within the CTA's launch allocation (kLaunchRegs per thread, what __launch_bounds__ leaves ptxas:
// 168 x 384 = 64 512, not the SM's 65 536): a split that asks for more leaves a consumer warp waiting for registers forever.
constexpr int kLaunchRegs = 65536 / kThreads / 8 * 8;
constexpr int kConsumerRegs = 224, kProducerRegs = 56;
static_assert(kConsumers * 128 * kConsumerRegs + 128 * kProducerRegs == kThreads * kLaunchRegs, "setmaxnreg split must fill the CTA's registers");
static_assert(kConsumers * kTilePts == 128, "the producer warpgroup has one thread per point of each consumer's tile");

// head weights image (B operands, 128-byte swizzle): Whead_h 80 x 128 | Whead_dir 80 x 64 | Wv1 64 x 64 | Wrgb 16 x 64
constexpr uint32_t WH_H = 0, WH_DIR = 20480, WH_V1 = 30720, WH_RGB = 38912, WH_BYTES = 40960;
constexpr int BIAS_FLOATS = 512 + 64 + 64 + 4 + 4;   // fp32: b0..b3 (512) | bq (64) | bv1 (64) | brgb (4) | bsig (1)
constexpr uint32_t BIAS_BYTES = 2624;                // BIAS_FLOATS * 4 rounded up to 64
constexpr uint32_t SLAB = 128 * 128;                 // one 64-column slab of a 128-row weight tile

// trunk weights image: W0enc | W1 | W2 | W3h | W3enc, each 128 rows (neurons) x K, K-major in 64-column slabs.  The background's
// KE = 96 fills only half of each encoding segment's last slab, so W3enc's columns 64-95 are packed into columns 32-63 of W0enc's
// last slab (w3enc_tail): W3enc takes one slab instead of two, and the 16 KB go to the encoding staging rows.
__host__ __device__ constexpr int enc_slabs(int KE) { return (KE + 63) / 64; }
__host__ __device__ constexpr uint32_t trunk_off(int KE, int seg) { return seg == 0 ? 0u : (uint32_t)(enc_slabs(KE) + 2 * (seg - 1)) * SLAB; }
__host__ __device__ constexpr uint32_t trunk_bytes(int KE) { return trunk_off(KE, 4) + (uint32_t)(KE / 64) * SLAB; }
__host__ __device__ constexpr uint32_t w3enc_tail(int KE) { return trunk_off(KE, 0) + (uint32_t)(KE / 64) * SLAB; }
// byte offset of W3enc's 16-column k-step ks (a wgmma descriptor start address relative to the image)
__host__ __device__ constexpr uint32_t w3enc_kstep(int KE, int ks) {
    return ks < 4 * (KE / 64) ? trunk_off(KE, 4) + (uint32_t)(ks >> 2) * SLAB + (uint32_t)(ks & 3) * 32u
                              : w3enc_tail(KE) + (uint32_t)(ks - 4 * (KE / 64) + 2) * 32u;
}

// channel order of the projected maps: physical channel p of a texel holds logical channel pmap_logical(p) of [P0 | P3], so that
// thread t (lane % 4) of an accumulator fragment finds its channels 8 j + 2 t + e (j < 16, e < 2) of a half at
// p = 32 (j / 4) + 8 t + 2 (j % 4) + e: in 16-byte chunk u = j / 4 of a 64-byte block per t, the four lanes of a quad reading one
// contiguous 64-byte block per load.  (With each thread's 64 bytes contiguous instead, one warp load of 8 points touches two
// 128-byte lines per point rather than one, and the blends' L1 wavefronts double.)
__host__ __device__ inline int pmap_logical(int p) {
    const int q = p & 127, u = q >> 5, t = (q >> 3) & 3, jj = (q >> 1) & 3, e = q & 1;
    return (p & 128) + 8 * (4 * u + jj) + 2 * t + e;
}

struct PtsRow {        // 48 bytes: view-independent data of one point of a tile
    float xe[3];       // point fed to the positional encoding (fg: sample point, bg: unit-sphere point)
    float tv;          // t (fg) or inverse radius s (bg)
    float xl[3];       // lookup point (fg: same point, bg: far(1-s)+3s along the ray, quirk Q2)
    int rid, sidx;     // ray and sample index
    int src;           // ray whose view direction conditions this point (quirk Q1)
    int valid;         // 0: padding row of the tile, its outputs are not stored
    int pad;
};

struct MlpTc {
    int in_ch, enc_dim, KE;          // 3|4, 63|84, 64|96
    const unsigned char* trunkimg;   // trunk_bytes(KE), pre-swizzled
    const unsigned char* headimg;    // WH_BYTES, pre-swizzled
    const float* bias;               // BIAS_FLOATS
    const __half* pmap[4];           // projected maps [P0|P3] of latent, xz, xy, yz: [nv][H][W][256] fp16 in pmap_logical order
};

struct State {
    MlpTc mlp[4];
};

struct Params {
    const float *rays_o, *rays_d, *far, *tvals;
    const uint4* dir;   // direction fragments of every ray (dir_frag_kernel), 4 per ray
    const int* ray_order;
    int n_rays, N, chunk, nv, n_tiles, sg;
    float far_unc;
    SceneDev sc;
    MlpTc mlp;
    float* rgb_out;
    float* sigma_out;
    int* trap;          // host-mapped int[8]: who timed out on which mbarrier (wait_timeout)
#ifdef NEO_FIELD_PHASES
    int phase_slot;     // row of g_phase_cycles this launch adds to
#endif
};

// Phase clocks (diagnostic build only, -DNEO_FIELD_PHASES; read by tools/field_phases.py): the first thread of every consumer
// warpgroup and of every producer half adds the clock() cycles between consecutive marks to its phase (32-bit: one register less
// than clock64() in the background consumers, and a phase lasts far less than 2^32 cycles), and at the end of the kernel the sums
// (and the consumers' tile counts) go into the launch's row of g_phase_cycles.  The marks bound the phases as the
// compiler scheduled them, which is close to, but not exactly, the source order.  Without the macro the kernel has no marks at all.
#ifdef NEO_FIELD_PHASES
enum Phase {
    kPhWait, kPhRows, kPhBlend0, kPhLayers, kPhBlend3, kPhLayer3, kPhDir, kPhColour,          // consumers
    kPhSetup, kPhEnc, kPhTaps, kPhSlot,                                                      // producer
    kPhases
};
// the phases, then tiles, taps of non-zero weight, and those of them that row n shares with row n + 8 (TapTable::share)
constexpr int kPhaseCols = kPhases + 3;
constexpr int kPhaseUnits = 2 * kConsumers;                              // the consumers, then the producer halves
constexpr uint32_t kPhaseBytes = kPhaseUnits * (kPhases + 1) * 8;        // per-unit sums (phases, tiles) in shared memory
constexpr int kPhaseSlots = 64;
__device__ unsigned long long g_phase_cycles[kPhaseSlots][kPhaseCols];    // [launch][column]
static int g_phase_launches = 0;
#define FIELD_PHASE_INIT(unit, lead) \
    unsigned ph_t = clock();         \
    unsigned long long ph_taps = 0;  \
    unsigned long long ph_shared = 0; \
    const int ph_unit = (unit);      \
    const bool ph_lead = (lead)
#define FIELD_PHASE(p)                                        \
    do {                                                      \
        const unsigned now_ = clock();                        \
        if (ph_lead) ph_acc[ph_unit][p] += now_ - ph_t;       \
        ph_t = now_;                                          \
    } while (0)
#else
constexpr uint32_t kPhaseBytes = 0;
#define FIELD_PHASE_INIT(unit, lead) do {} while (0)
#define FIELD_PHASE(p) do {} while (0)
#endif

// ------------------------------------------------------------------------------------------------
// per-scene preparation kernels
// ------------------------------------------------------------------------------------------------
// Per scene and MLP the latent columns of layers 0 and 3 are applied to the raw feature maps once (linearity of the lookups):
// P[v][pixel][p] = sum_c Wsel[p][c] * F[v][c][pixel],  p in [0,256) = [P0 | P3] in pmap_logical order -- a plain contraction, run on
// the tensor cores by gemm_f16 (csrc/gemm_tc.cu) from the channel-last fp16 maps (launch_nchw_to_nhwc) and the weight rows below.
// Wsel[p][c] fp16, p in [0,256): logical row r = pmap_logical(p); rows 0..127 = W0[r][col0 + c], rows 128..255 = W3[r - 128][col3 + c]
// (the latent columns of layers 0 and 3)
__global__ void wsel_kernel(const float* __restrict__ w0, int ld0, int col0, const float* __restrict__ w3, int ld3, int col3, int C, __half* __restrict__ out) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= 256 * C) return;
    const int r = pmap_logical(idx / C), c = idx % C;
    out[idx] = __float2half_rn(r < 128 ? w0[(size_t)r * ld0 + col0 + c] : w3[(size_t)(r - 128) * ld3 + col3 + c]);
}

// ---- positional encoding of the camera-frame point (helper.py:121-125), tensor-core operand layout ----
// The MMA does not care about the ORDER of the K columns as long as W0enc / W3enc use the same one (trunk_img_kernel), so the
// columns are grouped per coordinate: [x, sin(2^0 x) .. sin(2^9 x), cos(2^0 x) .. cos(2^9 x)] -- 21 columns per coordinate, stride 21
// (3 coordinates + the constant-one column 63 = 64 = KE) or stride 24 (4 coordinates, column 21 = constant one, KE = 96).
struct EncCol { int kind, cc, lvl; };          // kind 0: zero, 1: constant one, 2: x, 3: sin level, 4: cos level
template <int ICH>
__host__ __device__ constexpr EncCol enc_col(int col) {
    constexpr int STRIDE = (ICH == 3) ? 21 : 24;
    const int cc = col / STRIDE, j = col % STRIDE;
    if (ICH == 3 && col == 63) return {1, 0, 0};
    if (ICH == 4 && col == 21) return {1, 0, 0};
    if (cc >= ICH || j >= 21) return {0, 0, 0};
    if (j == 0) return {2, cc, 0};
    if (j <= 10) return {3, cc, j - 1};
    return {4, cc, j - 11};
}
// index of an encoding column in the reference's ordering (x, then per level all coordinates' sines, then the cosines); -1: none
template <int ICH>
__host__ __device__ constexpr int enc_col_ref_index(int col) {
    const EncCol e = enc_col<ICH>(col);
    if (e.kind == 2) return e.cc;
    if (e.kind == 3) return ICH + e.lvl * ICH + e.cc;
    if (e.kind == 4) return ICH + kPosDeg * ICH + e.lvl * ICH + e.cc;
    return -1;
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
// trunk weights image (shared-memory bytes, 128-byte swizzle): element (neuron n, k) of segment s at trunk_off(KE, s) +
// sw128_off(n, k, 128); segments W0enc (KE) | W1 | W2 | W3h (128 each) | W3enc (KE); W3enc's columns from 64 (KE / 64) on at
// w3enc_tail(KE) + sw128_off(n, 32 + k - 64 (KE / 64), 128)
__global__ void trunk_img_kernel(NeoMLPParams p, int enc_dim, int KE, unsigned char* __restrict__ img) {
    const int KW = 2 * KE + 384;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= KW * 128) return;
    const int n = idx / KW, kk = idx % KW;
    const int in_dim = enc_dim + kLocalCh + kWorldCh;
    const bool bg = (KE == 96);
    // encoding column `col` of the kernel's operand layout (enc_col<>): reference column, bias (constant-one column) or zero
    auto enc_w = [&](const float* w, size_t stride, size_t off0, const float* bias, int col) -> float {
        const EncCol e = bg ? enc_col<4>(col) : enc_col<3>(col);
        if (e.kind == 1) return bias[n];
        const int ref = bg ? enc_col_ref_index<4>(col) : enc_col_ref_index<3>(col);
        return ref >= 0 ? w[(size_t)n * stride + off0 + ref] : 0.f;
    };
    int seg, k;
    float x;
    if (kk < KE) { seg = 0; k = kk; x = enc_w(p.w0, in_dim, 0, p.b0, k); }
    else if (kk < KE + 128) { seg = 1; k = kk - KE; x = p.w1[n * 128 + k]; }
    else if (kk < KE + 256) { seg = 2; k = kk - KE - 128; x = p.w2[n * 128 + k]; }
    else if (kk < KE + 384) { seg = 3; k = kk - KE - 256; x = p.w3[(size_t)n * (128 + in_dim) + k]; }
    else { seg = 4; k = kk - KE - 384; x = enc_w(p.w3, 128 + in_dim, 128, p.b3, k); }
    const int full = 64 * (KE / 64);
    const uint32_t off = (seg == 4 && k >= full) ? w3enc_tail(KE) + sw128_off(n, 32 + k - full, 128) : trunk_off(KE, seg) + sw128_off(n, k, 128);
    *reinterpret_cast<__half*>(img + off) = __float2half_rn(x);
}

// head weights (pre-swizzled smem image) + folded biases
__global__ void head_kernel(NeoMLPParams p, int nv, unsigned char* __restrict__ img, float* __restrict__ bias) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    __half* im = reinterpret_cast<__half*>(img);
    const float inv = 1.0f / (float)nv;
    if (idx < 80 * 128) {                 // Whead_h  (rows: 64 q rows, 1 sigma row, 15 zero rows)
        int r = idx / 128, k = idx % 128;
        float x = 0.f;
        if (r < 64) { for (int j = 0; j < 128; ++j) x = fmaf(p.wv0[r * 155 + j], p.wb[j * 128 + k], x); x *= inv; }
        else if (r == 64) x = p.wsig[k] * inv;
        im[(WH_H + sw128_off(r, k, 80)) / 2] = __float2half_rn(x);
    } else if (idx < 80 * 128 + 80 * 64) { // Whead_dir
        int e = idx - 80 * 128, r = e / 64, k = e % 64;
        float x = (r < 64 && k < kDirEnc) ? p.wv0[r * 155 + 128 + k] : 0.f;
        im[(WH_DIR + sw128_off(r, k, 80)) / 2] = __float2half_rn(x);
    } else if (idx < 80 * 128 + 80 * 64 + 64 * 64) {
        int e = idx - 80 * 128 - 80 * 64, r = e / 64, k = e % 64;
        im[(WH_V1 + sw128_off(r, k, 64)) / 2] = __float2half_rn(p.wv1[r * 64 + k]);
    } else if (idx < 80 * 128 + 80 * 64 + 64 * 64 + 16 * 64) {
        int e = idx - 80 * 128 - 80 * 64 - 64 * 64, r = e / 64, k = e % 64;
        im[(WH_RGB + sw128_off(r, k, 16)) / 2] = __float2half_rn(r < 3 ? p.wrgb[r * 64 + k] : 0.f);
    }
    if (idx < BIAS_FLOATS) {
        float x = 0.f;
        if (idx < 128) x = p.b0[idx];
        else if (idx < 256) x = p.b1[idx - 128];
        else if (idx < 384) x = p.b2[idx - 256];
        else if (idx < 512) x = p.b3[idx - 384];
        else if (idx < 576) { int r = idx - 512; x = p.bv0[r]; for (int j = 0; j < 128; ++j) x = fmaf(p.wv0[r * 155 + j], p.bb[j], x); }
        else if (idx < 640) x = p.bv1[idx - 576];
        else if (idx < 643) x = p.brgb[idx - 640];
        else if (idx == 644) x = p.bsig[0];
        bias[idx] = x;
    }
}

// Fast-math restatement of ray_geom / fg_point / bg_point (common.cuh) for the TC path: the results only feed fp16
// operands and bilinear coordinates, so FMA contraction, rsqrt and approximate division are fine here.
struct RayFast { float o[3], d[3], far, rho, phi, psph[3], axis[3]; };
__device__ __forceinline__ void ray_fast(const float* __restrict__ o, const float* __restrict__ d, float far, RayFast& g, bool need_bg) {
    g.o[0] = o[0]; g.o[1] = o[1]; g.o[2] = o[2]; g.d[0] = d[0]; g.d[1] = d[1]; g.d[2] = d[2]; g.far = far;
    if (need_bg) {
        const float dd = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
        const float inv_dd = __fdividef(1.0f, dd);
        const float d1 = -(d[0] * o[0] + d[1] * o[1] + d[2] * o[2]) * inv_dd;
        const float p[3] = {o[0] + d1 * d[0], o[1] + d1 * d[1], o[2] + d1 * d[2]};
        const float p2 = p[0] * p[0] + p[1] * p[1] + p[2] * p[2];
        g.rho = sqrtf(p2);
        const float s = d1 + sqrtf(fmaxf(1.0f - p2, 0.f)) * rsqrtf(dd);
        for (int i = 0; i < 3; ++i) g.psph[i] = o[i] + s * d[i];
        float ax[3] = {o[1] * g.psph[2] - o[2] * g.psph[1], o[2] * g.psph[0] - o[0] * g.psph[2], o[0] * g.psph[1] - o[1] * g.psph[0]};
        const float an = rsqrtf(ax[0] * ax[0] + ax[1] * ax[1] + ax[2] * ax[2]);
        for (int i = 0; i < 3; ++i) g.axis[i] = ax[i] * an;
        g.phi = asinf(g.rho);
    }
}
__device__ __forceinline__ void bg_point_fast(const RayFast& g, float s, float far_unc, float* xhat, float* lin) {
    const float ang = g.phi - asinf(g.rho * s);
    float sa, ca;
    __sincosf(ang, &sa, &ca);
    const float* a = g.axis;
    const float* p = g.psph;
    const float cr[3] = {a[1] * p[2] - a[2] * p[1], a[2] * p[0] - a[0] * p[2], a[0] * p[1] - a[1] * p[0]};
    const float ap = (a[0] * p[0] + a[1] * p[1] + a[2] * p[2]) * (1.0f - ca);
    float q[3];
    for (int i = 0; i < 3; ++i) q[i] = p[i] * ca + cr[i] * sa + a[i] * ap;
    const float qn = __fdividef(1.0f, sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]) + 1e-10f);
    for (int i = 0; i < 3; ++i) xhat[i] = q[i] * qn;
    const float tl = g.far * (1.0f - s) + far_unc * s;
    for (int i = 0; i < 3; ++i) lin[i] = g.o[i] + tl * g.d[i];
}

// 2x2 tap quad of F.grid_sample(bilinear, align_corners=True, padding_mode="zeros") -- same arithmetic as bilinear_taps
// (common.cuh) but keeping the unclamped base texel: x0 in [-1, W-1], y0 in [-1, H-1]; w = {nw, ne, sw, se}, 0 when out of range.
struct TapQuad { int x0, y0; float w[4]; };
__device__ __forceinline__ void tap_quad(float gx, float gy, int W, int H, TapQuad& t) {
    const float ix = ((gx + 1.f) / 2.f) * (float)(W - 1);
    const float iy = ((gy + 1.f) / 2.f) * (float)(H - 1);
    const float x0f = floorf(ix), y0f = floorf(iy);
    const float fx = ix - x0f, fy = iy - y0f;
    const float gx1 = (x0f + 1.f) - ix, gy1 = (y0f + 1.f) - iy;
    // NaN / far-away coordinates: every tap is out of range
    const bool inr = (ix >= -1.f) && (ix < (float)W) && (iy >= -1.f) && (iy < (float)H);
    const int x0 = inr ? (int)x0f : -2, y0 = inr ? (int)y0f : -2;
    const bool vx0 = (x0 >= 0) & (x0 < W), vx1 = (x0 + 1 >= 0) & (x0 + 1 < W);
    const bool vy0 = (y0 >= 0) & (y0 < H), vy1 = (y0 + 1 >= 0) & (y0 + 1 < H);
    t.x0 = x0; t.y0 = y0;
    t.w[0] = (inr & vx0 & vy0) ? gx1 * gy1 : 0.f;
    t.w[1] = (inr & vx1 & vy0) ? fx * gy1 : 0.f;
    t.w[2] = (inr & vx0 & vy1) ? gx1 * fy : 0.f;
    t.w[3] = (inr & vx1 & vy1) ? fx * fy : 0.f;
}

// ------------------------------------------------------------------------------------------------
// the field kernel
// ------------------------------------------------------------------------------------------------
// Hand-off between the producer and consumer c: mbarrier 1 + kChans c + k of the CTA (mbarrier 0: the weight copies).  A full
// barrier completes when the consumer's 64 producer threads have written, an empty one when its 128 threads have read.
enum Chan { kRowsFull, kRowsEmpty, kStageFull, kStageEmpty, kTapsFull, kTapsEmpty, kChans };
constexpr int kBars = 1 + kChans * kConsumers;

// records who timed out on which mbarrier (id: 0 the weight copies, 1 + kChans c + k channel k of consumer c), then traps
__device__ __noinline__ void wait_timeout(int* trapinfo, uint32_t bar, int id) {
    if (trapinfo) {
        volatile int* t = trapinfo;
        if (t[0] == 0) {
            t[1] = (int)blockIdx.x; t[2] = (int)threadIdx.x; t[3] = (int)bar; t[4] = id; t[5] = (int)gridDim.x;
            t[0] = 1000;
        }
        __threadfence_system();
    }
    asm volatile("trap;");
}
// bounded wait for the phase of parity `parity` of mbarrier id (bar0: the address of mbarrier 0)
__device__ __forceinline__ void bar_wait(int* trapinfo, uint32_t bar0, int id, uint32_t parity) {
    const uint32_t b = bar0 + 8u * (uint32_t)id;
    if (!mbar_wait_bounded(b, parity)) wait_timeout(trapinfo, b, id);
}

__device__ __forceinline__ float sel4(const float* x, int i) { return i == 0 ? x[0] : i == 1 ? x[1] : i == 2 ? x[2] : x[3]; }

// Encoding staging: per (tile, view) the producer computes a consumer's 64 points' camera-frame encodings once, as a flat set of
// items, into one row of 64 fp16 per point; then every thread of the consumer loads its A-fragment columns from the rows.  (The
// background's s columns do not depend on the view and go with the tile's rows instead: kSRow.)  Row slot 21 j + k holds column k
// of coordinate j: k = 0 the coordinate, 1 + l sin(2^l x), 11 + l cos(2^l x), the order of enc_col<3> (slot == column for the
// foreground).  The 32-bit words of a row are XOR-swizzled by the point (bits 2-4), so
// that the 8 points x 4 words a warp loads per fragment register fall on 32 distinct banks.
constexpr int kStageRow = 64;
__device__ __forceinline__ int stage_slot(int n, int k) { return n * kStageRow + ((((k >> 1) ^ ((n & 7) << 2))) << 1 | (k & 1)); }

// items first .. first + count - 1 of one point (item i: staged coordinate i / 10, level i % 10): sin and cos of 2^l x, rounded to
// fp16 as pack_h2 does, into rows[slot(k)] for row slot k.  Rolled, so the kernel has one sincosf call site per use instead of one
// sinf / cosf per fragment column.
template <typename Slot>
__device__ __forceinline__ void stage_items(__half* rows, Slot slot, const float (&x)[3], int first, int count) {
#pragma unroll 1
    for (int i = first; i < first + count; ++i) {
        const int j = i / 10, l = i - 10 * j;
        const float xc = j == 0 ? x[0] : j == 1 ? x[1] : x[2];
        float s, c;
        sincosf(xc * (float)(1 << l), &s, &c);           // exact: power-of-two scaling
        rows[slot(21 * j + 1 + l)] = __float2half_rn(s);
        rows[slot(21 * j + 11 + l)] = __float2half_rn(c);
    }
}

// fp16 bits of encoding column c = c0 + u (enc_col<ICH> order; c0 a multiple of 8, u < 8, c < 72 in the background) of point n,
// from the staging rows.  Beyond a coordinate's 21 columns: the constant one (column 21 of the background) or zero.
template <int ICH>
__device__ __forceinline__ uint32_t enc_staged(const __half* stage, int n, int c0, int u) {
    if (ICH == 3) {                                      // stride 21: the slot is the column
        const int c = c0 + u;
        return c == 63 ? 0x3c00u : __half_as_ushort(stage[stage_slot(n, c)]);
    }
    const int j = c0 / 24, k = c0 % 24 + u;              // c0 % 24 <= 16: the 8 columns from c0 share one coordinate block
    if (k >= 21) return (j == 0 && k == 21) ? 0x3c00u : 0u;
    return __half_as_ushort(stage[stage_slot(n, 21 * j + k)]);
}
// the slot arithmetic above, checked against enc_col<> for every column
template <int ICH>
constexpr bool stage_layout_ok() {
    for (int c = 0; c < (ICH == 3 ? 64 : 96); ++c) {
        const EncCol e = enc_col<ICH>(c);
        const int k = e.kind == 2 ? 0 : e.kind == 3 ? 1 + e.lvl : 11 + e.lvl;
        if (ICH == 3 && e.kind >= 2 && c != 21 * e.cc + k) return false;
        if (ICH == 4) {
            const int j = c / 24, kk = c % 24;
            if (e.kind >= 2 && (kk >= 21 || j != e.cc || kk != k)) return false;
            if (e.kind < 2 && kk < 21) return false;
            if ((e.kind == 1) != (j == 0 && kk == 21)) return false;
        }
        if (ICH == 3 && (e.kind == 1) != (c == 63)) return false;
        if (ICH == 3 && e.kind == 0) return false;
    }
    return true;
}
static_assert(stage_layout_ok<3>() && stage_layout_ok<4>(), "enc_staged does not match enc_col");

// The background's s columns 72-95 (coordinate 3 of enc_col<4>: the inverse radius tv, its sin / cos levels and three zero columns)
// do not depend on the view.  The producer writes them once per tile, with the tile's PtsRows and before the same rows-full arrive,
// into one row of kSRow fp16 per point, slot k = column 72 + k; the consumer loads its A-fragment words of them when it copies the
// rows.  So the staging rows hold one view's encodings and nothing else, and the producer can build the next tile's first view while
// the consumer still works on the current tile.  A fragment word (columns 72 + 8 h' + 2 t, + 1) is one 32-bit load at slot
// 8 h' + 2 t: the 8 rows x 4 threads t of a warp's load fall on 32 distinct banks with the plain 48-byte row stride.
constexpr int kSRow = 24;
constexpr int kSCol0 = 72;
__device__ __forceinline__ uint32_t s_word(const __half* srows, int n, int k) {
    return *reinterpret_cast<const uint32_t*>(srows + n * kSRow + k);
}
constexpr bool s_layout_ok() {
    for (int k = 0; k < kSRow; ++k) {
        const EncCol e = enc_col<4>(kSCol0 + k);
        const int slot = e.kind == 2 ? 0 : e.kind == 3 ? 1 + e.lvl : 11 + e.lvl;
        if (k < 21 && (e.kind < 2 || e.cc != 3 || slot != k)) return false;
        if (k >= 21 && e.kind != 0) return false;
    }
    if (kSCol0 + kSRow != 96 || kSRow % 2) return false;
    for (int h = 0; h < 3; ++h) {                        // fragment words at slots 8 h + 2 t of rows r .. r + 7
        unsigned banks = 0;
        for (int r = 0; r < 8; ++r)
            for (int t = 0; t < 4; ++t) banks |= 1u << ((r * kSRow + 8 * h + 2 * t) / 2 % 32);
        if (banks != 0xffffffffu) return false;
    }
    return true;
}
static_assert(s_layout_ok(), "s rows do not match enc_col<4> or their fragment loads conflict on banks");

// column e of the direction encoding of the conditioning ray in one source camera's frame (model.py:357-360): [d, sin(2^k d),
// sin(2^k d + pi/2)], 27 columns, zero beyond
__device__ __forceinline__ float dir_value(const float* dc, int e) {
    if (e >= kDirEnc) return 0.f;
    if (e < 3) return sel4(dc, e);
    const int q0 = e - 3;
    const bool shifted = q0 >= 12;
    const int qq = shifted ? q0 - 12 : q0;
    const float xb = sel4(dc, qq % 3) * (float)(1 << (qq / 3));
    return sinf(shifted ? xb + 1.57079637f : xb);
}

// Direction fragments.  The direction term of the head, hacc += mean_v(dir_enc_v) . Whead_dir^T (K = 32: 27 columns + zero padding),
// has an A operand that depends only on the conditioning ray of the point (quirk Q1) and the source cameras, so it is computed once
// per ray and call (dir_frag_kernel) and every field launch of the call loads it.  Record of a ray: 64 bytes, 16 per thread t (lane
// % 4) of an accumulator quad: word 2 ks + h packs columns 16 ks + 8 h + 2 t + {0, 1}, i.e. the thread's A-fragment words (k-step ks,
// half h) of one row.  The view sum runs over the views in order, then is scaled by 1 / nv and rounded to fp16.
__device__ __forceinline__ uint4 dir_words(const ViewXform* vxs, int nv, const float (&wd)[3], int t) {
    float dsum[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) dsum[c] = 0.f;
    for (int vv = 0; vv < nv; ++vv) {
        float dc[3];
        rotate_to_camera(vxs[vv], wd, dc);
#pragma unroll
        for (int c = 0; c < 8; ++c) dsum[c] += dir_value(dc, 16 * (c >> 2) + 8 * ((c >> 1) & 1) + 2 * t + (c & 1));
    }
    const float inv = 1.0f / (float)nv;
    return make_uint4(pack_h2(dsum[0] * inv, dsum[1] * inv), pack_h2(dsum[2] * inv, dsum[3] * inv), pack_h2(dsum[4] * inv, dsum[5] * inv),
                      pack_h2(dsum[6] * inv, dsum[7] * inv));
}
// thread 4 r + t writes the 16 bytes of thread t of ray r's record
__global__ void dir_frag_kernel(const float* __restrict__ viewdirs, int n_rays, const ViewXform* __restrict__ views, int nv, uint4* __restrict__ out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= 4LL * n_rays) return;
    const long long r = idx >> 2;
    const float wd[3] = {viewdirs[3 * r], viewdirs[3 * r + 1], viewdirs[3 * r + 2]};
    out[idx] = dir_words(views, nv, wd, (int)(idx & 3));
}

// rectified accumulator (NC columns) -> fp16 A fragments of the next layer (K = NC, NC / 16 k-steps)
template <int NC>
__device__ __forceinline__ void relu_to_frags(const float (&d)[NC / 2], uint32_t (&a)[NC / 16][4]) {
#pragma unroll
    for (int ks = 0; ks < NC / 16; ++ks)
#pragma unroll
        for (int r = 0; r < 4; ++r) a[ks][r] = pack_h2(fmaxf(d[8 * ks + 2 * r], 0.f), fmaxf(d[8 * ks + 2 * r + 1], 0.f));
}
// accumulator (NC columns) seeded with a bias vector (shared memory)
template <int NC>
__device__ __forceinline__ void seed_bias(float (&d)[NC / 2], const float* b, int t) {
#pragma unroll
    for (int j = 0; j < NC / 8; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i) { d[4 * j + 2 * i] = b[8 * j + 2 * t]; d[4 * j + 2 * i + 1] = b[8 * j + 2 * t + 1]; }
}
// descriptor of k-step ks of a 128-byte-swizzled K-major weight tile whose 64-column slabs are `slab` bytes apart
__device__ __forceinline__ uint64_t wdesc(uint32_t base, int ks, uint32_t slab) { return desc_sw128(base + (uint32_t)(ks >> 2) * slab + (uint32_t)(ks & 3) * 32u); }

// Tap table of one (tile, view), per consumer in shared memory: for every point n of the tile and map m (latent, xz, xy, yz), the
// texel index (view included) of the quad's nw tap and the bilinear weights of its four taps {nw, ne, sw, se}; tap k is texel
// base + (k >> 1) mw + (k & 1) (tap_index), mw the map's width.  Arrays [m][n], so that the 8 points a warp reads at once fall on
// distinct banks.  A consumer thread blends rows r0 and r0 + 8 (r0 % 16 < 8): the same sample of two vertically adjacent pixels,
// which mostly read the same texels.  Foreground only: share[share_pair(r0)] has bit 4 m + k set when tap k of map m is the same
// texel for both rows and both weights are non-zero, so the blend fetches it once.
struct TapTable {
    int base[4][kTilePts];
    float4 w[4][kTilePts];
    uint16_t share[kTilePts / 2];
};
__host__ __device__ constexpr int share_pair(int r0) { return (r0 >> 4) * 8 + (r0 & 7); }
__device__ __forceinline__ float comp4(const float4& x, int k) { return k == 0 ? x.x : k == 1 ? x.y : k == 2 ? x.z : x.w; }
// texel index of tap k of the quad whose nw tap is texel `base` of a map mw texels wide
__device__ __forceinline__ int tap_index(int base, int mw, int k) { return base + (k >> 1) * mw + (k & 1); }

// entry (point n, map m) of the tap table from the camera-frame lookup point cl: grid_sample(bilinear, align_corners=True, zeros)
// taps of the map in source view v.  A tap out of range has weight 0, and a tap of weight 0 is never loaded (blend_maps), so only
// the taps of non-zero weight need tap_index to be a texel of the map: at a map's edge (x0 or y0 = -1) the base and the other taps
// may lie outside it.  A quad whose four weights are all zero (e.g. x0, y0 = -2: off the map) stores base 0.  With SHARE, returns in the
// threads with n % 16 < 8 bit k set when tap k is a texel of non-zero weight that is also tap k of point n + 8 with non-zero weight
// (lane n + 8 of the same warp; every lane of the warp must call this together).
template <bool SHARE>
__device__ __forceinline__ uint32_t tap_entry(TapTable& tab, const SceneDev& sc, const float (&cl)[3], int v, int n, int m) {
    float gx, gy;
    int mw, mh;
    if (m == 0) {
        local_grid_coords(sc, cl, gx, gy);
        mw = sc.lat_w; mh = sc.lat_h;
    } else {
        gx = (m == 3) ? cl[1] : cl[0];
        gy = (m == 2) ? cl[1] : cl[2];          // xz, xy, yz
        mw = sc.plane_w; mh = sc.plane_h;
    }
    TapQuad tq;
    tap_quad(gx, gy, mw, mh, tq);
    int tx[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) tx[k] = tq.w[k] == 0.f ? 0 : (v * mh + tq.y0 + (k >> 1)) * mw + tq.x0 + (k & 1);
    const bool any = (tq.w[0] != 0.f) | (tq.w[1] != 0.f) | (tq.w[2] != 0.f) | (tq.w[3] != 0.f);
    tab.base[m][n] = any ? (v * mh + tq.y0) * mw + tq.x0 : 0;
    tab.w[m][n] = make_float4(tq.w[0], tq.w[1], tq.w[2], tq.w[3]);
    if (!SHARE) return 0;
    uint32_t shared = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int key = tq.w[k] == 0.f ? -1 : tx[k];              // a zero-weight tap (index 0) matches nothing
        const int other = __shfl_down_sync(0xffffffffu, key, 8);
        shared |= (uint32_t)(key >= 0 && key == other) << k;
    }
    return shared;
}

// acc[4 j + 2 I + e] += w * (channel 8 j + 2 t + e of the texel chunks q): one tap of the point in row r0 + 8 I
template <int I>
__device__ __forceinline__ void blend_tap(float (&acc)[64], float w, const uint4 (&q)[4]) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const uint32_t wd[4] = {q[u].x, q[u].y, q[u].z, q[u].w};
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
            const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&wd[jj]));
            const int j = 4 * u + jj;
            acc[4 * j + 2 * I] = fmaf(w, f.x, acc[4 * j + 2 * I]);
            acc[4 * j + 2 * I + 1] = fmaf(w, f.y, acc[4 * j + 2 * I + 1]);
        }
    }
}

// acc[4 j + 2 i + e] += bilinear blend (grid_sample, align_corners=True, zeros) of channel 8 j + 2 t + e of half HALF of [P0 | P3]
// over the four maps, at this thread's two points (rows r0, r0 + 8 of the tile); fp32 blend of fp16 texels.
// The taps' geometry comes from the tap table.  For each map and tap k the thread blends tap k of row r0, then tap k of row r0 + 8;
// a tap of zero weight is skipped (zeros padding: no contribution), and its texel index, which may lie outside the map, is never
// formed into a load.  Each accumulator belongs to one row and gets its taps in (m, k) order with the same fmaf operands whatever
// the path, so the sums are bit for bit those of blending each row on its own.  All lanes step through (m, k) together, so lanes of
// a quarter-warp that read the same line in one load still share it.
// PAIR: both rows' loads of tap k are issued before either row's FMAs, two texels in flight instead of one (the blends wait on each
// texel's first fetch, DESIGN.md §5).  SHARE (foreground, with PAIR): a tap the table marks as the same texel for both rows
// (TapTable::share) is loaded once, row r0 + 8 blending row r0's chunks; the background producer builds no mask.  The background
// kernel has no registers for the second set of chunks in its P3 blend (it spills), so there it loads and blends one row's tap at a
// time.  (Issuing a map's four taps ahead of their FMAs needs the skip replaced by masking, 64 more live registers and the FMAs of
// out-of-range taps; measured on H100 that made the field launches 10 % slower than one tap at a time, see DESIGN.md §5.)
template <int HALF, bool PAIR, bool SHARE>
__device__ __forceinline__ void blend_maps(float (&acc)[64], const Params& P, const TapTable& tab, int r0, int t) {
    static_assert(PAIR || !SHARE, "a shared tap is blended into both rows from one load: the paired form");
    uint32_t share = SHARE ? tab.share[share_pair(r0)] : 0u;
#pragma unroll 1
    for (int m = 0; m < 4; ++m, share >>= 4) {
        const float4 wv0 = tab.w[m][r0], wv1 = tab.w[m][r0 + 8];
        const int* bx0 = &tab.base[m][r0];                             // read per tap, behind its skip: fewer live registers
        const int* bx1 = &tab.base[m][r0 + 8];
        const int mw = m == 0 ? P.sc.lat_w : P.sc.plane_w;
        const uint4* base = reinterpret_cast<const uint4*>(P.mlp.pmap[m] + HALF * 128 + t * 8);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float w0 = comp4(wv0, k), w1 = comp4(wv1, k);
            const bool both = (share >> k) & 1u;                       // shared: w0, w1 != 0 and q0 holds row r0 + 8's texel
            uint4 q0[4], q1[4];
            if (w0 != 0.f) {
                const int tx = tap_index(*bx0, mw, k);
#pragma unroll
                for (int u = 0; u < 4; ++u) q0[u] = __ldg(base + (size_t)tx * 32 + 4 * u);   // 32 uint4 per texel
                if (!PAIR) blend_tap<0>(acc, w0, q0);
            }
            if (w1 != 0.f && !both) {
                const int tx = tap_index(*bx1, mw, k);
#pragma unroll
                for (int u = 0; u < 4; ++u) q1[u] = __ldg(base + (size_t)tx * 32 + 4 * u);
            }
            if (PAIR && w0 != 0.f) blend_tap<0>(acc, w0, q0);
            if (w1 != 0.f) {
                if (both)
#pragma unroll
                    for (int u = 0; u < 4; ++u) q1[u] = q0[u];
                blend_tap<1>(acc, w1, q1);
            }
        }
    }
}

template <int KE>
struct SmemMap {
    static constexpr uint32_t HEAD = trunk_bytes(KE), BIAS = HEAD + WH_BYTES, VIEWS = BIAS + BIAS_BYTES,
                              PTS = VIEWS + kMaxViews * 64, TAPS = PTS + kConsumers * kTilePts * (uint32_t)sizeof(PtsRow),
                              STAGE = TAPS + kConsumers * (uint32_t)sizeof(TapTable),
                              SROWS = STAGE + kConsumers * kTilePts * kStageRow * (uint32_t)sizeof(__half),
                              BAR = SROWS + (KE == 96 ? kConsumers * kTilePts * kSRow * (uint32_t)sizeof(__half) : 0u),
                              PHASES = BAR + (kBars * 8 + 15) / 16 * 16, TOTAL = PHASES + kPhaseBytes;
    static_assert(KE % 64 == 0 || KE % 64 == 32, "an encoding segment ends on a whole or a half slab (w3enc_tail)");
    static_assert(TOTAL + 1024 <= 227u * 1024u, "field kernel shared memory exceeds the 227 KB an sm_90 CTA can have");
};

template <int ICH>
__global__ void __launch_bounds__(kThreads, 1) field_tc_kernel(const __grid_constant__ Params P) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
    unsigned char* sgen = smem_raw + (sbase - smem_u32(smem_raw));
    constexpr int KE = (ICH == 3) ? 64 : 96, KS = KE / 16;
    constexpr bool IS_BG = (ICH == 4);
    using SM = SmemMap<KE>;
    const uint32_t bar = sbase + SM::BAR;

    // ---- one-time setup: every weight of the MLP -> shared memory (TMA bulk copies), source-camera transforms, hand-off barriers ----
    if (threadIdx.x == 0) {
        mbar_init(bar, 1);
        for (int c = 0; c < kConsumers; ++c)
            for (int k = 0; k < kChans; ++k) mbar_init(bar + 8u * (1 + kChans * c + k), (k & 1) ? 128 : kTilePts);   // empty: consumer
        mbar_init_fence();
        constexpr uint32_t TB = trunk_bytes(KE);
        mbar_expect_tx(bar, TB + WH_BYTES + BIAS_FLOATS * 4);
        for (uint32_t off = 0; off < TB; off += 32768u) bulk_load(sbase + off, P.mlp.trunkimg + off, min(32768u, TB - off), bar);
        bulk_load(sbase + SM::HEAD, P.mlp.headimg, WH_BYTES, bar);
        bulk_load(sbase + SM::BIAS, P.mlp.bias, BIAS_FLOATS * 4, bar);
    }
    {
        float* vsm = reinterpret_cast<float*>(sgen + SM::VIEWS);
        const float* vsrc = reinterpret_cast<const float*>(P.sc.views);
        for (int i = threadIdx.x; i < P.nv * 16; i += kThreads) vsm[i] = __ldg(vsrc + i);
    }
#ifdef NEO_FIELD_PHASES
    auto ph_acc = reinterpret_cast<unsigned long long (*)[kPhases + 1]>(sgen + SM::PHASES);
    if (threadIdx.x < kPhaseUnits * (kPhases + 1)) (&ph_acc[0][0])[threadIdx.x] = 0ull;
#endif
    __syncthreads();

    const int wg = threadIdx.x >> 7;
    const ViewXform* vxs = reinterpret_cast<const ViewXform*>(sgen + SM::VIEWS);
    const int nv = P.nv, N = P.N;

    if (wg == kConsumers) {
        // ================= producer: thread pt builds point n of consumer c's tiles =================
        setmaxnreg_dec<kProducerRegs>();
        const int pt = threadIdx.x - 128 * kConsumers, c = pt / kTilePts, n = pt % kTilePts;
        PtsRow* pts = reinterpret_cast<PtsRow*>(sgen + SM::PTS) + c * kTilePts;
        TapTable* tab = reinterpret_cast<TapTable*>(sgen + SM::TAPS) + c;
        __half* stage = reinterpret_cast<__half*>(sgen + SM::STAGE) + c * kTilePts * kStageRow;
        __half* srows = reinterpret_cast<__half*>(sgen + SM::SROWS) + c * kTilePts * kSRow;   // background only
        const int cb = 1 + kChans * c;                   // id of this consumer's first channel barrier
        uint32_t k_rows = 0, k_stage = 0, k_taps = 0;   // fills so far: the producer's wait for fill k is on parity (k & 1) ^ 1
        FIELD_PHASE_INIT(kConsumers + c, n == 0);
        for (int tile = blockIdx.x * kConsumers + c; tile < P.n_tiles; tile += gridDim.x * kConsumers) {
            const int g = tile / P.sg, q = tile % P.sg;
            bar_wait(P.trap, bar, cb + kRowsEmpty, (k_rows & 1) ^ 1);        // the consumer has copied the previous tile's rows
            FIELD_PHASE(kPhSlot);
            {
                const int rl = n % kTileRays, sl = n / kTileRays;
                const int slot = g * kTileRays + rl, s = q * kTileSamples + sl;
                const int slot_c = min(slot, P.n_rays - 1), s_c = min(s, N - 1);
                const int rid = P.ray_order ? P.ray_order[slot_c] : slot_c;
                PtsRow pr;
                pr.rid = rid; pr.sidx = s_c; pr.valid = (slot < P.n_rays) && (s < N);
                pr.tv = P.tvals[(long long)rid * N + s_c];
                RayFast rg;
                ray_fast(P.rays_o + 3 * rid, P.rays_d + 3 * rid, P.far[rid], rg, IS_BG);
                if (IS_BG) bg_point_fast(rg, pr.tv, P.far_unc, pr.xe, pr.xl);
                else for (int i = 0; i < 3; ++i) { pr.xe[i] = rg.o[i] + pr.tv * rg.d[i]; pr.xl[i] = pr.xe[i]; }
                // quirk Q1: the direction of ray (j mod B) of the ray's chunk, j = flat (ray, sample) index inside the chunk
                const int ch = P.chunk > 0 ? P.chunk : P.n_rays;
                const int c0 = (rid / ch) * ch;
                const int Bc = min(ch, P.n_rays - c0);
                const long long jl = (long long)(rid - c0) * N + s_c;
                pr.src = c0 + (int)(jl % Bc);
                pr.pad = 0;
                pts[n] = pr;
                if constexpr (IS_BG) {
                    // the s columns 72-95, once per tile: they travel with the rows
                    const float sx[3] = {pr.tv, 0.f, 0.f};
                    __half* srow = srows + n * kSRow;
                    srow[0] = __float2half_rn(sx[0]);
                    stage_items(srow, [](int k) { return k; }, sx, 0, 10);
#pragma unroll
                    for (int k = 21; k < kSRow; ++k) srow[k] = __float2half_rn(0.f);
                }
            }
            mbar_arrive(bar + 8u * (cb + kRowsFull));
            ++k_rows;
            FIELD_PHASE(kPhSetup);
#pragma unroll 1
            for (int v = 0; v < nv; ++v) {
                float ce[3];
                to_camera(vxs[v], pts[n].xe, ce);
                bar_wait(P.trap, bar, cb + kStageEmpty, (k_stage & 1) ^ 1);  // the consumer has loaded the previous encodings
                FIELD_PHASE(kPhSlot);
#pragma unroll
                for (int j = 0; j < 3; ++j) stage[stage_slot(n, 21 * j)] = __float2half_rn(ce[j]);
                stage_items(stage, [n](int k) { return stage_slot(n, k); }, ce, 0, 30);
                mbar_arrive(bar + 8u * (cb + kStageFull));
                ++k_stage;
                FIELD_PHASE(kPhEnc);
                float cl[3] = {ce[0], ce[1], ce[2]};            // foreground: xl == xe, the lookup point IS the encoded point
                if constexpr (IS_BG) to_camera(vxs[v], pts[n].xl, cl);
                bar_wait(P.trap, bar, cb + kTapsEmpty, (k_taps & 1) ^ 1);    // the consumer's blends have read the previous table
                FIELD_PHASE(kPhSlot);
                uint32_t shared = 0;
#pragma unroll 1
                for (int m = 0; m < 4; ++m) {
                    shared |= tap_entry<!IS_BG>(*tab, P.sc, cl, v, n, m) << (4 * m);
#ifdef NEO_FIELD_PHASES
                    for (int k = 0; k < 4; ++k) ph_taps += comp4(tab->w[m][n], k) != 0.f;
#endif
                }
                if (!IS_BG && (n & 15) < 8) {
                    tab->share[share_pair(n)] = (uint16_t)shared;
#ifdef NEO_FIELD_PHASES
                    ph_shared += __popc(shared);
#endif
                }
                mbar_arrive(bar + 8u * (cb + kTapsFull));
                ++k_taps;
                FIELD_PHASE(kPhTaps);
            }
        }
#ifdef NEO_FIELD_PHASES
        if (ph_lead)
            for (int p = kPhSetup; p < kPhases; ++p) atomicAdd(&g_phase_cycles[P.phase_slot][p], ph_acc[ph_unit][p]);
        atomicAdd(&g_phase_cycles[P.phase_slot][kPhases + 1], ph_taps);
        atomicAdd(&g_phase_cycles[P.phase_slot][kPhases + 2], ph_shared);
#endif
        return;
    }

    // ================= consumer wg: blends and tensor-core MLP of its tiles =================
    setmaxnreg_inc<kConsumerRegs>();
    bar_wait(P.trap, bar, 0, 0);                         // the weight copies
    const int wt = threadIdx.x & 127, warp = wt >> 5, lane = threadIdx.x & 31, t = lane & 3;
    const PtsRow* pts = reinterpret_cast<const PtsRow*>(sgen + SM::PTS) + wg * kTilePts;
    const TapTable* tab = reinterpret_cast<const TapTable*>(sgen + SM::TAPS) + wg;
    const __half* stage = reinterpret_cast<const __half*>(sgen + SM::STAGE) + wg * kTilePts * kStageRow;
    const __half* srows = reinterpret_cast<const __half*>(sgen + SM::SROWS) + wg * kTilePts * kSRow;   // background only
    const int cb = 1 + kChans * wg;
    uint32_t k_rows = 0, k_stage = 0, k_taps = 0;       // fills consumed so far: the wait for fill k is on parity k & 1
    const float* sb = reinterpret_cast<const float*>(sgen + SM::BIAS);
    const uint32_t sW = sbase, sH = sbase + SM::HEAD;
    const int r0 = warp * 16 + (lane >> 2);          // this thread's accumulator rows (points) r0, r0 + 8
    FIELD_PHASE_INIT(wg, wt == 0);

    for (int tile = blockIdx.x * kConsumers + wg; tile < P.n_tiles; tile += gridDim.x * kConsumers) {
        // the tile's rows: what the direction term and the stores need, copied so that the producer can move on to the next tile
        bar_wait(P.trap, bar, cb + kRowsFull, k_rows & 1);
        FIELD_PHASE(kPhWait);
        long long gp[2];                                 // output index rid * N + sidx of rows r0, r0 + 8, -1: padding row
        int src[2];
        // A-fragment columns 16 ks + 8 h + 2 t + e of rows r0, r0 + 8 (e: the low / high half of a word)
        uint32_t enc[KS][4];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const PtsRow& pr = pts[r0 + 8 * i];
            gp[i] = pr.valid ? (long long)pr.rid * N + pr.sidx : -1;
            src[i] = pr.src;
            if constexpr (IS_BG) {                       // the s columns 72-95: enc[4][2..3], enc[5][*]
                enc[KS - 2][2 + i] = s_word(srows, r0 + 8 * i, 2 * t);
                enc[KS - 1][i] = s_word(srows, r0 + 8 * i, 8 + 2 * t);
                enc[KS - 1][2 + i] = s_word(srows, r0 + 8 * i, 16 + 2 * t);
            }
        }
        mbar_arrive(bar + 8u * (cb + kRowsEmpty));
        ++k_rows;
#ifdef NEO_FIELD_PHASES
        if (wt == 0) ph_acc[wg][kPhases] += 1ull;
#endif
        auto load_enc = [&](int ks, int h) {             // the columns as enc_staged reads them (c0 = 16 ks + 8 h, u = 2 t + e)
#pragma unroll
            for (int i = 0; i < 2; ++i)
                enc[ks][2 * h + i] = enc_staged<ICH>(stage, r0 + 8 * i, 16 * ks + 8 * h, 2 * t) |
                                     enc_staged<ICH>(stage, r0 + 8 * i, 16 * ks + 8 * h, 2 * t + 1) << 16;
        };
        FIELD_PHASE(kPhRows);

        float hacc[40];                                 // folded head: [q (64) | sigma | pad], summed over the views
#pragma unroll
        for (int i = 0; i < 40; ++i) hacc[i] = 0.f;
#pragma unroll 1
        for (int v = 0; v < nv; ++v) {
            bar_wait(P.trap, bar, cb + kStageFull, k_stage & 1);
            FIELD_PHASE(kPhWait);
#pragma unroll
            for (int ks = 0; ks < 4; ++ks)
#pragma unroll
                for (int h = 0; h < 2; ++h) load_enc(ks, h);
            if constexpr (IS_BG) load_enc(4, 0);                               // columns 64-71: the last levels of coordinate 2
            mbar_arrive(bar + 8u * (cb + kStageEmpty));
            ++k_stage;
            FIELD_PHASE(kPhRows);
            bar_wait(P.trap, bar, cb + kTapsFull, k_taps & 1);
            FIELD_PHASE(kPhWait);
            float acc[64];
            uint32_t a[8][4];
            // layer 0: blend of P0 + W0enc . enc (b0 on the constant-one column)
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] = 0.f;
            blend_maps<0, !IS_BG, !IS_BG>(acc, P, *tab, r0, t);
            FIELD_PHASE(kPhBlend0);
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) wgmma_rs_n128(acc, enc[ks], wdesc(sW + trunk_off(KE, 0), ks, SLAB));
            wgmma_commit();
            wgmma_wait<0>();
            relu_to_frags<128>(acc, a);
            // layers 1, 2
#pragma unroll 1
            for (int l = 1; l <= 2; ++l) {
                seed_bias<128>(acc, sb + 128 * l, t);
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < 8; ++ks) wgmma_rs_n128(acc, a[ks], wdesc(sW + trunk_off(KE, l), ks, SLAB));
                wgmma_commit();
                wgmma_wait<0>();
                relu_to_frags<128>(acc, a);
            }
            // layer 3: blend of P3 + W3h . h2 + W3enc . enc (b3 on the constant-one column)
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] = 0.f;
            FIELD_PHASE(kPhLayers);
            blend_maps<1, !IS_BG, !IS_BG>(acc, P, *tab, r0, t);
            mbar_arrive(bar + 8u * (cb + kTapsEmpty));                              // the producer may build the next table
            ++k_taps;
            FIELD_PHASE(kPhBlend3);
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) wgmma_rs_n128(acc, a[ks], wdesc(sW + trunk_off(KE, 3), ks, SLAB));
#pragma unroll
            for (int ks = 0; ks < KS; ++ks) wgmma_rs_n128(acc, enc[ks], desc_sw128(sW + w3enc_kstep(KE, ks)));
            wgmma_commit();
            wgmma_wait<0>();
            relu_to_frags<128>(acc, a);
            // folded head: hacc += h3 . Whead_h^T
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) wgmma_rs_n80(hacc, a[ks], wdesc(sH + WH_H, ks, 80 * 128));
            wgmma_commit();
            wgmma_wait<0>();
            FIELD_PHASE(kPhLayer3);
        }
        // direction term: hacc += mean_v(dir_enc_v) . Whead_dir^T, A = the direction fragments of the points' conditioning rays
        {
            const uint4 d0 = __ldg(P.dir + 4LL * src[0] + t), d1 = __ldg(P.dir + 4LL * src[1] + t);
            const uint32_t dfr[2][4] = {{d0.x, d1.x, d0.y, d1.y}, {d0.z, d1.z, d0.w, d1.w}};
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) wgmma_rs_n80(hacc, dfr[ks], wdesc(sH + WH_DIR, ks, 80 * 128));
            wgmma_commit();
            wgmma_wait<0>();
        }
        FIELD_PHASE(kPhDir);
        // sigma (column 64: thread t = 0 of each quad), q = relu(hacc + bq) -> colour head 64 x 64 -> relu -> 64 x 3 -> sigmoid
        if (t == 0) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const float xs = (hacc[32 + 2 * i] + sb[644]) - 1.0f;                   // model.py:392-393
                if (gp[i] >= 0) P.sigma_out[gp[i]] = softplus_(xs);
            }
        }
        uint32_t qa[4][4];
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int c = 16 * ks + 8 * (r >> 1) + 2 * t;                           // column of hacc[8 ks + 2 r]
                qa[ks][r] = pack_h2(fmaxf(hacc[8 * ks + 2 * r] + sb[512 + c], 0.f), fmaxf(hacc[8 * ks + 2 * r + 1] + sb[512 + c + 1], 0.f));
            }
        float v1[32];
        seed_bias<64>(v1, sb + 576, t);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) wgmma_rs_n64(v1, qa[ks], wdesc(sH + WH_V1, ks, 64 * 128));
        wgmma_commit();
        wgmma_wait<0>();
        relu_to_frags<64>(v1, qa);
        float o[8];
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int c = 8 * j + 2 * t + e;
                    o[4 * j + 2 * i + e] = c < 3 ? sb[640 + c] : 0.f;
                }
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) wgmma_rs_n16(o, qa[ks], wdesc(sH + WH_RGB, ks, 16 * 128));
        wgmma_commit();
        wgmma_wait<0>();
        if (t < 2) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                if (gp[i] < 0) continue;
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int c = 2 * t + e;
                    if (c < 3) P.rgb_out[gp[i] * 3 + c] = rgb_act(o[2 * i + e]);   // model.py:395-397
                }
            }
        }
        FIELD_PHASE(kPhColour);
    }
#ifdef NEO_FIELD_PHASES
    if (ph_lead) {
        for (int p = 0; p < kPhSetup; ++p) atomicAdd(&g_phase_cycles[P.phase_slot][p], ph_acc[ph_unit][p]);
        atomicAdd(&g_phase_cycles[P.phase_slot][kPhases], ph_acc[ph_unit][kPhases]);
    }
#endif
}

}  // namespace tc

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static int* g_trap_host = nullptr;   // host-mapped int[8] written by wait_timeout before a trap
static int* g_trap_dev = nullptr;

static int trap_buffer() {
    if (g_trap_host) return NEO_OK;
    void* h = nullptr;
    NEO_CUDA(cudaHostAlloc(&h, 8 * sizeof(int), cudaHostAllocMapped));
    memset(h, 0, 8 * sizeof(int));
    void* dptr = nullptr;
    NEO_CUDA(cudaHostGetDevicePointer(&dptr, h, 0));
    g_trap_host = (int*)h;
    g_trap_dev = (int*)dptr;
    return NEO_OK;
}
const char* tc_trap_info() {
    static char buf[256];
    if (!g_trap_host || g_trap_host[0] == 0) return "";
    volatile int* t = g_trap_host;
    static const char* chans[tc::kChans] = {"rows full", "rows empty", "staging full", "staging empty", "tap table full", "tap table empty"};
    const int id = t[4];
    char what[64];
    if (id == 0) snprintf(what, sizeof(what), "weight copies");
    else if (id > 0 && id < tc::kBars) snprintf(what, sizeof(what), "%s, consumer %d", chans[(id - 1) % tc::kChans], (id - 1) / tc::kChans);
    else snprintf(what, sizeof(what), "barrier %d", id);
    snprintf(buf, sizeof(buf), " [TC field kernel: wait on the %s mbarrier timed out: CTA %d of %d, thread %d, barrier smem 0x%x]",
             what, t[1], t[5], t[2], (unsigned)t[3]);
    return buf;
}

int tc_scene_create(NeoScene* sc, const NeoMLPParams mlps[4], cudaStream_t s) {
    using namespace tc;
    const NeoSceneDesc& d = sc->desc;
    State* st = new State();
    sc->tc_state = st;
    const float* planes[3] = {d.planes_xz, d.planes_xy, d.planes_yz};
    // channel-last fp16 copies of the raw feature maps (temporary: shared by the four MLPs' pre-projections) and the packed weight rows
    struct Temps {                                   // handed back to the block pool on every exit path (after the stream has drained)
        __half* feat16[4] = {nullptr, nullptr, nullptr, nullptr};
        size_t bytes[4] = {0, 0, 0, 0};
        __half* wsel = nullptr;
        cudaStream_t s;
        ~Temps() {
            cudaStreamSynchronize(s);
            for (int k = 0; k < 4; ++k) pool_release(feat16[k], bytes[k]);
            pool_release(wsel, (size_t)256 * kLocalCh * 2);
        }
    } tmp;
    tmp.s = s;
    if ((long long)d.nv * d.lat_h * d.lat_w > 0x7fffffffLL || (long long)d.nv * d.plane_h * d.plane_w > 0x7fffffffLL) {
        set_error("feature maps too large: the tap table holds 32-bit texel indices");
        return NEO_ERR_UNSUPPORTED;
    }
    __half** feat16 = tmp.feat16;
    __half*& wsel = tmp.wsel;
    {
        const float* srcs[4] = {d.latent, planes[0], planes[1], planes[2]};
        int rc;
        for (int k = 0; k < 4; ++k) {
            const int C = k ? kWorldCh : kLocalCh, hw = k ? d.plane_h * d.plane_w : d.lat_h * d.lat_w;
            tmp.bytes[k] = (size_t)d.nv * hw * C * 2;
            if ((rc = pool_alloc((void**)&feat16[k], tmp.bytes[k]))) return rc;
            if ((rc = launch_nchw_to_nhwc(srcs[k], feat16[k], d.nv, C, hw, s))) return rc;
        }
        if ((rc = pool_alloc((void**)&wsel, (size_t)256 * kLocalCh * 2))) return rc;
    }
    for (int i = 0; i < 4; ++i) {
        const NeoMLPParams& p = mlps[i];
        if (p.in_ch != 3 && p.in_ch != 4) { set_error("mlp %d: in_ch must be 3 or 4", i); return NEO_ERR_INVALID; }
        if ((i & 1) != (p.in_ch == 4)) { set_error("mlps must be ordered fg_coarse, bg_coarse, fg_fine, bg_fine"); return NEO_ERR_INVALID; }
        MlpTc& m = st->mlp[i];
        m.in_ch = p.in_ch;
        m.enc_dim = p.in_ch * 21;
        m.KE = (p.in_ch == 3) ? 64 : 96;
        const int in_dim = m.enc_dim + kLocalCh + kWorldCh;
        void* q = nullptr;
        int rc;
        const uint32_t tbytes = trunk_bytes(m.KE);
        if ((rc = scene_alloc_bytes(sc, &q, tbytes))) return rc;
        m.trunkimg = (const unsigned char*)q;
        const int nelem = (2 * m.KE + 384) * 128;
        trunk_img_kernel<<<(nelem + 255) / 256, 256, 0, s>>>(p, m.enc_dim, m.KE, (unsigned char*)q);
        NEO_LAUNCH_CHECK("trunk_img_kernel");
        void* hb = nullptr; void* bb = nullptr;
        if ((rc = scene_alloc_bytes(sc, &hb, WH_BYTES))) return rc;
        if ((rc = scene_alloc_bytes(sc, &bb, BIAS_BYTES))) return rc;
        NEO_CUDA(cudaMemsetAsync(hb, 0, WH_BYTES, s));
        NEO_CUDA(cudaMemsetAsync(bb, 0, BIAS_BYTES, s));
        head_kernel<<<(80 * 128 + 80 * 64 + 64 * 64 + 16 * 64 + 255) / 256, 256, 0, s>>>(p, d.nv, (unsigned char*)hb, (float*)bb);
        NEO_LAUNCH_CHECK("head_kernel");
        m.headimg = (const unsigned char*)hb;
        m.bias = (const float*)bb;
        // pre-projected feature maps [P0 | P3] in pmap_logical channel order, [nv][H][W][256]: P = F . Wsel^T is a plain contraction
        // over the raw channels, one N = 256 gemm_f16 per view (fp16 features x fp16 weights, fp32 accumulate)
        for (int k = 0; k < 4; ++k) {
            const int C = k ? kWorldCh : kLocalCh, mh = k ? d.plane_h : d.lat_h, mw = k ? d.plane_w : d.lat_w, hw = mh * mw;
            const int col = m.enc_dim + (k ? kLocalCh : 0);
            void* pp = nullptr;
            if ((rc = scene_alloc_bytes(sc, &pp, (size_t)d.nv * hw * 256 * 2))) return rc;
            m.pmap[k] = (const __half*)pp;
            wsel_kernel<<<(256 * C + 255) / 256, 256, 0, s>>>(p.w0, in_dim, col, p.w3, 128 + in_dim, 128 + col, C, wsel);
            NEO_LAUNCH_CHECK("wsel_kernel");
            for (int v = 0; v < d.nv; ++v)
                if ((rc = gemm_f16(feat16[k] + (size_t)v * hw * C, C, wsel, C, nullptr, (__half*)pp + (size_t)v * hw * 256, 256, hw, 256, C, 0, s)))
                    return rc;
        }
        NEO_CUDA(cudaStreamSynchronize(s));          // wsel is reused by the next MLP
    }
    NEO_CUDA(cudaStreamSynchronize(s));              // the temporaries are released when `tmp` goes out of scope
    return NEO_OK;
}

void tc_scene_free(NeoScene* sc) {
    if (sc && sc->tc_state) { delete reinterpret_cast<tc::State*>(sc->tc_state); sc->tc_state = nullptr; }
}

int launch_dir_frags(const NeoScene* sc, const NeoRays* rays, void* dir, cudaStream_t s) {
    if (!rays->viewdirs || !dir || (uintptr_t)dir % 16) { set_error("direction fragments: need viewdirs and a 16-byte aligned output"); return NEO_ERR_INVALID; }
    const long long threads = 4LL * rays->n_rays;
    if (threads <= 0) return NEO_OK;
    tc::dir_frag_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(rays->viewdirs, rays->n_rays, sc->dev.views, sc->dev.nv,
                                                                         static_cast<uint4*>(dir));
    NEO_LAUNCH_CHECK("dir_frag_kernel");
    return NEO_OK;
}

int launch_field_tc(const NeoScene* sc, const NeoRays* rays, const float* far, const float* t, int N, int mlp_index, const void* dir,
                    float* rgb, float* sigma, cudaStream_t s) {
    using namespace tc;
    if (!(sc->precision_mask & (1 << NEO_PREC_TC)) || !sc->tc_state) { set_error("scene was not prepared for NEO_PREC_TC"); return NEO_ERR_INVALID; }
    if (!dir) { set_error("NEO_PREC_TC field launch without direction fragments"); return NEO_ERR_INVALID; }
    const State* st = reinterpret_cast<const State*>(sc->tc_state);
    static int n_sm_of[64] = {0};          // per device: a process may drive several GPUs
    int dev = 0;
    NEO_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64) { set_error("device index %d out of range", dev); return NEO_ERR_UNSUPPORTED; }
    if (!n_sm_of[dev]) NEO_CUDA(cudaDeviceGetAttribute(&n_sm_of[dev], cudaDevAttrMultiProcessorCount, dev));
    const int n_sm = n_sm_of[dev];
    Params P;
    P.rays_o = rays->rays_o; P.rays_d = rays->rays_d; P.far = far; P.tvals = t;
    P.dir = static_cast<const uint4*>(dir);
    P.ray_order = rays->ray_order;
    P.n_rays = rays->n_rays; P.N = N; P.chunk = rays->chunk; P.nv = sc->dev.nv;
    P.sg = (N + kTileSamples - 1) / kTileSamples;
    const long long groups = ((long long)rays->n_rays + kTileRays - 1) / kTileRays;
    const long long n_tiles = groups * P.sg;
    if (n_tiles > 0x3fffffffLL) { set_error("too many tiles"); return NEO_ERR_UNSUPPORTED; }
    P.n_tiles = (int)n_tiles;
    P.far_unc = 3.0f;
    P.sc = sc->dev;
    P.mlp = st->mlp[mlp_index];
    P.rgb_out = rgb; P.sigma_out = sigma;
    { int rc0 = trap_buffer(); if (rc0) return rc0; }
    P.trap = g_trap_dev;
#ifdef NEO_FIELD_PHASES
    P.phase_slot = g_phase_launches++ % kPhaseSlots;
#endif
    const long long ctas = (n_tiles + kConsumers - 1) / kConsumers;
    const int grid = (int)(ctas < n_sm ? ctas : n_sm);
    auto launch = [&](auto kern, size_t smem) -> int {
        cudaFuncAttributes fa;
        NEO_CUDA(cudaFuncGetAttributes(&fa, kern));
        if (fa.numRegs != kLaunchRegs) {              // the setmaxnreg split would not fit: refuse rather than hang
            set_error("field_tc_kernel was compiled for %d registers per thread, its warpgroup split needs %d", fa.numRegs, kLaunchRegs);
            return NEO_ERR_UNSUPPORTED;
        }
        NEO_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, kThreads, smem, s>>>(P);
        return NEO_OK;
    };
    int rc;
    if (mlp_index & 1) rc = launch(field_tc_kernel<4>, SmemMap<96>::TOTAL + 1024);
    else rc = launch(field_tc_kernel<3>, SmemMap<64>::TOTAL + 1024);
    if (rc != NEO_OK) return rc;
    NEO_LAUNCH_CHECK("field_tc_kernel");
    return NEO_OK;
}

}  // namespace neo

extern "C" int neo_tc_enc_column(int in_ch, int col) {
    using namespace neo::tc;
    if ((in_ch != 3 && in_ch != 4) || col < 0 || col >= (in_ch == 3 ? 64 : 96)) return -3;
    const EncCol e = (in_ch == 3) ? enc_col<3>(col) : enc_col<4>(col);
    if (e.kind == 1) return -1;
    if (e.kind == 0) return -2;
    return (in_ch == 3) ? enc_col_ref_index<3>(col) : enc_col_ref_index<4>(col);
}
extern "C" const char* neo_tc_trap_info(void) { return neo::tc_trap_info(); }

#ifdef NEO_FIELD_PHASES
// diagnostic build only (not part of include/neo360_b200.h): zero the phase clocks, and read them back after a synchronise as
// [launch][kPhases + 3] (cycles per phase, then tiles, taps of non-zero weight and shared taps), one row per field launch since the
// reset; returns the number of launches
extern "C" int neo_field_phases_reset(void) {
    neo::tc::g_phase_launches = 0;
    void* p = nullptr;
    if (cudaGetSymbolAddress(&p, neo::tc::g_phase_cycles) != cudaSuccess) return -1;
    return cudaMemset(p, 0, sizeof(neo::tc::g_phase_cycles)) == cudaSuccess ? 0 : -1;
}
extern "C" int neo_field_phases_read(unsigned long long* out, int max_launches) {
    using namespace neo::tc;
    if (g_phase_launches > kPhaseSlots) return -1;          // rows have wrapped
    const int n = g_phase_launches < max_launches ? g_phase_launches : max_launches;
    if (n > 0 && cudaMemcpyFromSymbol(out, g_phase_cycles, sizeof(unsigned long long) * n * kPhaseCols) != cudaSuccess) return -1;
    return n;
}
#endif
