// Vanilla two-level NeRF renderer of the reference (SURVEY.md section 8(a) row a17), fp32 CUDA cores, reference formulation.
// Reference: models/vanilla_nerf/model.py:44-216 (NeRFMLP 8x256 with skip after layer 4, NeRF.forward),
// models/vanilla_nerf/helper.py:415-442 (sampling), 445-449 (pos-enc), 521-559 (compositing), 567-616 (inverse CDF).
// Sampling marches along `viewdirs`, compositing scales by |rays_d| (quirk Q15); depth gets nan_to_num(inf) (quirk Q10).
#include "common.cuh"
#include <cuda_fp16.h>

struct NeoVanilla {
    struct Mlp {
        const float* wt[8];   // transposed (in,out)
        const float* b[8];
        const float *wbt, *bb, *wsig, *bsig, *wv0t, *bv0, *wrgb, *brgb;
        // tensor-core path (NEO_PREC_TC): nn.Linear layout (out, in padded to a multiple of 64) in fp16
        const void* w16[8];   // (256, 64) | (256,256) x4 | (256, 256+64) | (256,256) x2
        const void *wb16, *wv016;   // (256,256), (128, 256+64)
    } mlp[2];
    std::vector<void*> allocations;
    size_t bytes;
};

namespace neo {
namespace van {

constexpr int kW = 256, kEnc = 63, kP = 8, kThreads = 256, kCond = 128;

// helper.py:415-442, deterministic or jittered; points = o + t * viewdirs
__global__ void sample_kernel(const float* __restrict__ o, const float* __restrict__ vd, int n, int ns, float near, float far,
                              const float* __restrict__ u_rand, float* __restrict__ t_out) {
    int steps = ns + 1;
    long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (long long)n * steps) return;
    int b = (int)(gid / steps), k = (int)(gid % steps);
    auto tv = [&](int kk) { float u = linspace01(kk, steps); return add_(mul_(near, sub_(1.0f, u)), mul_(far, u)); };
    float t = tv(k);
    if (u_rand) {
        float lower = (k > 0) ? mul_(0.5f, add_(t, tv(k - 1))) : t;
        float upper = (k < ns) ? mul_(0.5f, add_(tv(k + 1), t)) : t;
        t = add_(lower, mul_(sub_(upper, lower), u_rand[(long long)b * steps + k]));
    }
    t_out[gid] = t;
}

__global__ void __launch_bounds__(kThreads) field_kernel(NeoVanilla::Mlp m, const float* __restrict__ rays_o,
                                                         const float* __restrict__ viewdirs, const float* __restrict__ tvals,
                                                         int n_rays, int N, float* __restrict__ rgb_out, float* __restrict__ sigma_out) {
    __shared__ __align__(16) float X[kP][64];
    __shared__ __align__(16) float Ha[kP][kW + 4];
    __shared__ __align__(16) float Hb[kP][kW + 4];
    __shared__ __align__(16) float Dn[kP][28];
    __shared__ float xp[kP][3];
    __shared__ float red[8][kP];
    const int j = threadIdx.x;
    const long long total = (long long)n_rays * N, tile0 = (long long)blockIdx.x * kP;
    if (j < kP) {
        long long gp = min(tile0 + j, total - 1);
        int b = (int)(gp / N);
        float t = tvals[gp];
        for (int c = 0; c < 3; ++c) xp[j][c] = add_(rays_o[3 * b + c], mul_(t, viewdirs[3 * b + c]));   // cast_rays along viewdirs
    }
    __syncthreads();
    for (int e = j; e < kP * 64; e += kThreads) {
        int p = e / 64, c = e % 64;
        X[p][c] = c < kEnc ? pos_enc_col(xp[p], 3, 10, c) : 0.f;
    }
    for (int e = j; e < kP * 28; e += kThreads) {
        int p = e / 28, c = e % 28;
        long long gp = min(tile0 + p, total - 1);
        Dn[p][c] = c < kDirEnc ? pos_enc_col(viewdirs + 3 * (gp / N), 3, 4, c) : 0.f;
    }
    __syncthreads();
    float acc[kP];
    auto init = [&](const float* b) { float v = __ldg(b + j); for (int r = 0; r < kP; ++r) acc[r] = v; };
    auto relu_to = [&](float (*H)[kW + 4]) { for (int r = 0; r < kP; ++r) H[r][j] = fmaxf(acc[r], 0.f); };
    float (*src)[kW + 4] = Ha;
    float (*dst)[kW + 4] = Hb;
    // layer 0
    init(m.b[0]); dense_rows<kP>(m.wt[0], kW, kEnc, &X[0][0], 64, acc, j); relu_to(Ha); __syncthreads();
    for (int l = 1; l < 8; ++l) {
        init(m.b[l]);
        dense_rows<kP>(m.wt[l], kW, kW, &src[0][0], kW + 4, acc, j);
        if (l == 5) dense_rows<kP>(m.wt[l] + (size_t)kW * kW, kW, kEnc, &X[0][0], 64, acc, j);      // cat([h, inputs]) after layer 4
        relu_to(dst);
        __syncthreads();
        float (*tmp)[kW + 4] = src; src = dst; dst = tmp;
    }
    // src = h7.  density head
    {
        float ws = __ldg(m.wsig + j);
        for (int p = 0; p < kP; ++p) {
            float part = warp_sum(src[p][j] * ws);
            if ((j & 31) == 0) red[j >> 5][p] = part;
        }
    }
    // bottleneck -> dst
    init(m.bb); dense_rows<kP>(m.wbt, kW, kW, &src[0][0], kW + 4, acc, j);
    for (int r = 0; r < kP; ++r) dst[r][j] = acc[r];
    __syncthreads();
    if (j < kP) {
        long long gp = tile0 + j;
        if (gp < total) {
            float raw = __ldg(m.bsig);
            for (int w = 0; w < 8; ++w) raw += red[w][j];
            sigma_out[gp] = softplus_(raw - 1.0f);
        }
    }
    // view branch: [bottleneck | dir_enc] -> 128 relu  (result into src rows, first 128 columns)
    float a2[kP];
    if (j < kCond) {
        float v = __ldg(m.bv0 + j);
        for (int r = 0; r < kP; ++r) a2[r] = v;
        dense_rows<kP>(m.wv0t, kCond, kW, &dst[0][0], kW + 4, a2, j);
        dense_rows<kP>(m.wv0t + (size_t)kW * kCond, kCond, kDirEnc, &Dn[0][0], 28, a2, j);
    }
    __syncthreads();
    if (j < kCond) for (int r = 0; r < kP; ++r) src[r][j] = fmaxf(a2[r], 0.f);
    __syncthreads();
    if (j < kP * 3) {
        int p = j / 3, c = j % 3;
        long long gp = tile0 + p;
        if (gp < total) {
            float a = __ldg(m.brgb + c);
            for (int k = 0; k < kCond; ++k) a = fmaf(src[p][k], __ldg(m.wrgb + c * kCond + k), a);
            rgb_out[gp * 3 + c] = rgb_act(a);
        }
    }
}

// ---- tensor-core path: positional encodings as fp16 rows (63 -> 64, 27 -> 64 zero padded), activations of the heads ----
// One thread per sample row: the point and its 10 octaves (one sincosf per coordinate, then angle doubling, whose error grows with the
// octave), then the direction encoding of its ray (4 octaves).  Against exact sin / cos of the fp32 point rounded to fp16
// (oracle/tc_paths_model.py), the field's per-point error stays fp16 rounding noise: tests/test_gpu_tc_paths.py measured up to 1.5e-3 in
// rgb and 4.3e-3 in sigma (pre-activation units) per point, 1.9e-4 / 3.4e-4 per case mean, on an H100.  Rows are 128 bytes; a lane owns a row,
// so each row is assembled in a per-warp shared-memory tile ([32 rows][128 B], 16-byte pieces XOR-swizzled by row) and written out as
// whole lines, 4 rows per store instruction (the one-thread-per-element version spent 15 % of the frame here).
__device__ __forceinline__ void put_h(unsigned char* stage, int lane, int c, float v) {
    const int byte = c * 2;
    *reinterpret_cast<__half*>(stage + lane * 128 + ((((byte >> 4) ^ (lane & 7)) << 4) | (byte & 15))) = __float2half_rn(v);
}
__device__ __forceinline__ void flush_rows(const unsigned char* stage, int lane, __half* __restrict__ dst, long long ld, long long row0, long long M) {
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int rr = i * 4 + (lane >> 3), p = lane & 7;
        const uint4 val = *reinterpret_cast<const uint4*>(stage + rr * 128 + ((p ^ (rr & 7)) << 4));
        if (row0 + rr < M) *reinterpret_cast<uint4*>(dst + (row0 + rr) * ld + p * 8) = val;
    }
    __syncwarp();
}
__global__ void __launch_bounds__(256) enc16_kernel(const float* __restrict__ rays_o, const float* __restrict__ viewdirs, const float* __restrict__ tvals,
                                                    long long M, int N, __half* __restrict__ X16, long long ldx, __half* __restrict__ D16, long long ldd) {
    __shared__ __align__(16) unsigned char stage_all[8][32 * 128];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned char* stage = stage_all[warp];
    const long long row0 = ((long long)blockIdx.x * 8 + warp) * 32, m = row0 + lane;
    const bool live = m < M;
    const int b = live ? (int)(m / N) : 0;
    const float t = live ? tvals[m] : 0.f;
    float d[3], x[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) { d[j] = viewdirs[3 * b + j]; x[j] = add_(rays_o[3 * b + j], mul_(t, d[j])); }
    // point encoding: [x (3) | sin(x 2^k) k-major (30) | cos (30) | 0]
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        put_h(stage, lane, j, x[j]);
        float sn, cs;
        sincosf(x[j], &sn, &cs);
#pragma unroll
        for (int k = 0; k < 10; ++k) {
            put_h(stage, lane, 3 + 3 * k + j, sn);
            put_h(stage, lane, 33 + 3 * k + j, cs);
            const float s2 = 2.f * sn * cs, c2 = (cs - sn) * (cs + sn);
            sn = s2; cs = c2;
        }
    }
    put_h(stage, lane, 63, 0.f);
    flush_rows(stage, lane, X16, ldx, row0, M);
    // direction encoding: [d (3) | sin (12) | cos (12) | 0 ... 0]
#pragma unroll
    for (int p = 3; p < 8; ++p) *reinterpret_cast<uint4*>(stage + lane * 128 + ((p ^ (lane & 7)) << 4)) = make_uint4(0u, 0u, 0u, 0u);
    __syncwarp();
    for (int c = 27; c < 32; ++c) put_h(stage, lane, c, 0.f);
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        put_h(stage, lane, j, d[j]);
        float sn, cs;
        sincosf(d[j], &sn, &cs);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            put_h(stage, lane, 3 + 3 * k + j, sn);
            put_h(stage, lane, 15 + 3 * k + j, cs);
            const float s2 = 2.f * sn * cs, c2 = (cs - sn) * (cs + sn);
            sn = s2; cs = c2;
        }
    }
    flush_rows(stage, lane, D16, ldd, row0, M);
}
__global__ void head_act_kernel(const float* __restrict__ raw_sigma, const float* __restrict__ raw_rgb, long long M, float* __restrict__ sigma,
                                float* __restrict__ rgb) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= M * 4) return;
    const long long m = i >> 2;
    const int c = (int)(i & 3);
    if (c == 3) sigma[m] = softplus_(raw_sigma[m] - 1.0f);
    else rgb[m * 3 + c] = rgb_act(raw_rgb[m * 3 + c]);
}

// Training path (neo360_b200/vanilla.py): the fp32 encodings the field kernel builds in shared memory, written out for the framework's
// dense layers.  Elements [0, M*63) are point-encoding columns (row = sample, helper.py:445-449 column order), [M*63, M*63 + n*27) are
// direction-encoding columns (row = ray); the point and pos_enc_col are field_kernel's own arithmetic, so the values are bit-identical.
__global__ void encode_kernel(const float* __restrict__ rays_o, const float* __restrict__ viewdirs, const float* __restrict__ tvals, int n, int N,
                              float* __restrict__ enc, float* __restrict__ dir_enc) {
    const long long M = (long long)n * N, gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid < M * kEnc) {
        const long long m = gid / kEnc;
        const int c = (int)(gid % kEnc), b = (int)(m / N);
        const float t = tvals[m];
        float x[3];
        for (int j = 0; j < 3; ++j) x[j] = add_(rays_o[3 * b + j], mul_(t, viewdirs[3 * b + j]));
        enc[gid] = pos_enc_col(x, 3, 10, c);
    } else if (gid < M * kEnc + (long long)n * kDirEnc) {
        const long long e = gid - M * kEnc;
        dir_enc[e] = pos_enc_col(viewdirs + 3 * (e / kDirEnc), 3, 4, (int)(e % kDirEnc));
    }
}

}  // namespace van
}  // namespace neo

using namespace neo;

namespace {
// Scratch of one level's field: the tensor-core chain's fp16 activation rows and raw head outputs (the fp32 field kernel needs none)
struct WSF { __half *A16[2], *B16, *V16; float *rawd, *rawc; };
struct WSV { float *t0, *w0, *t1, *w1, *sig, *rgb; WSF f; };
constexpr int kLdA = 256 + 64, kLdB = 256 + 64;      // activation rows: [h (256) | padded encoding (64)], [bottleneck (256) | padded direction encoding (64)]
void carve_field(Carve& c, size_t M, WSF& w, int precision) {
    if (precision != NEO_PREC_TC) return;
    for (int i = 0; i < 2; ++i) w.A16[i] = c.take<__half>(M * kLdA);
    w.B16 = c.take<__half>(M * kLdB);
    w.V16 = c.take<__half>(M * 128);
    w.rawd = c.take<float>(M); w.rawc = c.take<float>(M * 3);
}
size_t carve(Carve& c, int n, int N0, int N1, WSV& w, int precision) {
    w.t0 = c.take<float>((size_t)n * N0); w.w0 = c.take<float>((size_t)n * N0); w.t1 = c.take<float>((size_t)n * N1); w.w1 = c.take<float>((size_t)n * N1);
    w.sig = c.take<float>((size_t)n * N1); w.rgb = c.take<float>((size_t)n * N1 * 3);
    carve_field(c, (size_t)n * N1, w.f, precision);
    return c.used;
}
// One level's NeRFMLP at the points o + t viewdirs of t (n, N): activated rgb (n, N, 3) and sigma (n, N).  The render and
// neo_vanilla_field_eval both run this, so the two give the same bits.
int field(const NeoVanilla::Mlp& m, const float* rays_o, const float* viewdirs, const float* t, int n, int N, int precision, const WSF& w,
          float* rgb, float* sig, cudaStream_t s) {
    const long long total = (long long)n * N;
    int rc;
    if (precision == NEO_PREC_TC) {
        // NeRFMLP (models/vanilla_nerf/model.py:44-125) layer by layer on the tensor cores (csrc/gemm_tc.cu), fp16 activations; the skip concatenation
        // by keeping h4 and the encoding in ONE buffer (layer 5 is a single K = 320 GEMM)
        __half* buf[2] = {w.A16[0], w.A16[1]};
        __half* B = w.B16;
        van::enc16_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(rays_o, viewdirs, t, total, N, buf[0] + 256, kLdA, B + 256, kLdB);
        NEO_LAUNCH_CHECK("vanilla enc16_kernel");
        if ((rc = gemm_f16(buf[0] + 256, kLdA, m.w16[0], 64, m.b[0], buf[0], kLdA, total, 256, 64, 1, s))) return rc;
        for (int l = 1; l < 8; ++l) {
            const int K = l == 5 ? 320 : 256;
            if ((rc = gemm_f16(buf[(l - 1) & 1], kLdA, m.w16[l], K, m.b[l], buf[l & 1], kLdA, total, 256, K, 1, s))) return rc;
        }
        const __half* h = buf[1];
        if ((rc = launch_rowdot_f16(h, kLdA, 256, m.wsig, m.bsig, 1, total, w.rawd, s))) return rc;
        if ((rc = gemm_f16(h, kLdA, m.wb16, 256, m.bb, B, kLdB, total, 256, 256, 0, s))) return rc;
        if ((rc = gemm_f16(B, kLdB, m.wv016, 320, m.bv0, w.V16, 128, total, 128, 320, 1, s))) return rc;
        if ((rc = launch_rowdot_f16(w.V16, 128, 128, m.wrgb, m.brgb, 3, total, w.rawc, s))) return rc;
        van::head_act_kernel<<<(unsigned)((total * 4 + 255) / 256), 256, 0, s>>>(w.rawd, w.rawc, total, sig, rgb);
        NEO_LAUNCH_CHECK("vanilla head_act_kernel");
    } else {
        van::field_kernel<<<(unsigned)((total + van::kP - 1) / van::kP), van::kThreads, 0, s>>>(m, rays_o, viewdirs, t, n, N, rgb, sig);
        NEO_LAUNCH_CHECK("vanilla field_kernel");
    }
    return NEO_OK;
}
int check(const NeoVanillaCfg* c) {
    if (!c || c->n_coarse < 3 || c->n_fine < 1 || c->n_coarse > 4096 || c->n_fine > 4096) { set_error("vanilla: bad sample counts"); return NEO_ERR_INVALID; }
    if (c->precision != NEO_PREC_FP32 && c->precision != NEO_PREC_TC) { set_error("vanilla: bad precision %d", c->precision); return NEO_ERR_INVALID; }
    return NEO_OK;
}
}  // namespace

extern "C" int neo_vanilla_create(const NeoVanillaMLPParams mlps[2], NeoVanilla** out, void* stream) {
    if (!mlps || !out) { set_error("neo_vanilla_create: null argument"); return NEO_ERR_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    NeoVanilla* v = new NeoVanilla();
    v->bytes = 0;
    auto fail = [&](int rc) { neo_vanilla_free(v); return rc; };
    auto dup = [&](const float* src, size_t n, const float** dst, int out_f, int in_f) -> int {
        void* q = nullptr;
        cudaError_t e = cudaMalloc(&q, n * sizeof(float));
        if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc(vanilla)");
        v->allocations.push_back(q);
        v->bytes += n * sizeof(float);
        *dst = (const float*)q;
        return out_f > 0 ? launch_transpose(src, (float*)q, out_f, in_f, s) : copy_out((float*)q, src, n, s);
    };
    for (int i = 0; i < 2; ++i) {
        const NeoVanillaMLPParams& p = mlps[i];
        NeoVanilla::Mlp& m = v->mlp[i];
        int rc;
        for (int l = 0; l < 8; ++l) {
            int in_f = l == 0 ? 63 : (l == 5 ? 319 : 256);
            if ((rc = dup(p.w[l], (size_t)256 * in_f, &m.wt[l], 256, in_f))) return fail(rc);
            if ((rc = dup(p.b[l], 256, &m.b[l], 0, 0))) return fail(rc);
        }
        if ((rc = dup(p.wb, 256 * 256, &m.wbt, 256, 256))) return fail(rc);
        if ((rc = dup(p.bb, 256, &m.bb, 0, 0))) return fail(rc);
        if ((rc = dup(p.wsig, 256, &m.wsig, 0, 0))) return fail(rc);
        if ((rc = dup(p.bsig, 1, &m.bsig, 0, 0))) return fail(rc);
        if ((rc = dup(p.wv0, 128 * 283, &m.wv0t, 128, 283))) return fail(rc);
        if ((rc = dup(p.bv0, 128, &m.bv0, 0, 0))) return fail(rc);
        if ((rc = dup(p.wrgb, 3 * 128, &m.wrgb, 0, 0))) return fail(rc);
        if ((rc = dup(p.brgb, 3, &m.brgb, 0, 0))) return fail(rc);
        // fp16 images for the tensor-core path: K padded to a multiple of 64; the skip layer's [h | inputs] columns land at [0,256) | [256,319)
        auto pack16 = [&](const float* src, int rows, int c0, int ncols, int ld_in, void* dst, int off, int pad_cols, int ld_out) -> int {
            return f32_to_f16_pad(src + c0, rows, ncols, ld_in, (__half*)dst + off, pad_cols, ld_out, s);
        };
        auto alloc16 = [&](size_t halves, const void** dst) -> int {
            void* q = nullptr;
            cudaError_t e = cudaMalloc(&q, halves * 2);
            if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc(vanilla fp16)");
            v->allocations.push_back(q);
            v->bytes += halves * 2;
            *dst = q;
            return NEO_OK;
        };
        for (int l = 0; l < 8; ++l) {
            const int in_f = l == 0 ? 63 : (l == 5 ? 319 : 256), kp = l == 0 ? 64 : (l == 5 ? 320 : 256);
            if ((rc = alloc16((size_t)256 * kp, &m.w16[l]))) return fail(rc);
            if (l == 5) {
                if ((rc = pack16(p.w[l], 256, 0, 256, in_f, (void*)m.w16[l], 0, 256, kp))) return fail(rc);
                if ((rc = pack16(p.w[l], 256, 256, 63, in_f, (void*)m.w16[l], 256, 64, kp))) return fail(rc);
            } else if ((rc = pack16(p.w[l], 256, 0, in_f, in_f, (void*)m.w16[l], 0, kp, kp))) return fail(rc);
        }
        if ((rc = alloc16((size_t)256 * 256, &m.wb16))) return fail(rc);
        if ((rc = pack16(p.wb, 256, 0, 256, 256, (void*)m.wb16, 0, 256, 256))) return fail(rc);
        if ((rc = alloc16((size_t)128 * 320, &m.wv016))) return fail(rc);
        if ((rc = pack16(p.wv0, 128, 0, 256, 283, (void*)m.wv016, 0, 256, 320))) return fail(rc);
        if ((rc = pack16(p.wv0, 128, 256, 27, 283, (void*)m.wv016, 256, 64, 320))) return fail(rc);
    }
    cudaError_t e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return fail(cuda_fail(e, "neo_vanilla_create sync"));
    *out = v;
    return NEO_OK;
}

extern "C" void neo_vanilla_free(NeoVanilla* v) {
    if (!v) return;
    for (void* p : v->allocations) cudaFree(p);
    delete v;
}

extern "C" size_t neo_vanilla_workspace_bytes(int n_rays, const NeoVanillaCfg* cfg) {
    if (n_rays <= 0 || check(cfg)) return 0;
    Carve c{nullptr, 0};
    WSV w;
    return carve(c, n_rays, cfg->n_coarse + 1, cfg->n_coarse + 1 + cfg->n_fine, w, cfg->precision);
}

extern "C" int neo_vanilla_render_fwd(const NeoVanilla* v, const NeoRays* rays, const NeoVanillaCfg* cfg, NeoVanillaOut* out,
                                      void* workspace, size_t workspace_bytes, void* stream) {
    if (!v || !rays || !out) { set_error("neo_vanilla_render_fwd: null argument"); return NEO_ERR_INVALID; }
    int rc = check(cfg);
    if (rc) return rc;
    if (rays->n_rays <= 0 || !rays->rays_o || !rays->rays_d || !rays->viewdirs) { set_error("neo_vanilla_render_fwd: empty rays"); return NEO_ERR_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    const int n = rays->n_rays, N0 = cfg->n_coarse + 1, N1 = N0 + cfg->n_fine;
    Carve c{static_cast<unsigned char*>(workspace), 0};
    WSV w;
    size_t need = carve(c, n, N0, N1, w, cfg->precision);
    if (!workspace || workspace_bytes < need) { set_error("workspace too small: need %zu bytes, got %zu", need, workspace_bytes); return NEO_ERR_WORKSPACE; }
    for (int lvl = 0; lvl < 2; ++lvl) {
        const int N = lvl ? N1 : N0;
        float* t = lvl ? w.t1 : w.t0;
        float* wt = lvl ? w.w1 : w.w0;
        if (lvl == 0) {
            long long total = (long long)n * N0;
            van::sample_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(rays->rays_o, rays->viewdirs, n, cfg->n_coarse, cfg->near_plane,
                                                                               cfg->far_plane, cfg->u0, t);
            NEO_LAUNCH_CHECK("vanilla sample_kernel");
        } else {
            // sample_pdf: bins = mids(t), weights[1:-1]; same ascending-bin inverse CDF + merge as the NeO-360 foreground branch
            if ((rc = launch_resample(rays->rays_o, rays->viewdirs, nullptr, w.t0, w.w0, n, N0, cfg->n_fine, 1, 0.f, cfg->u1, t, nullptr, nullptr, s))) return rc;
        }
        if ((rc = field(v->mlp[lvl], rays->rays_o, rays->viewdirs, t, n, N, cfg->precision, w.f, w.rgb, w.sig, s))) return rc;
        // mode 2: ascending t, last interval 1e10, scaled by |rays_d|, depth nan_to_num(inf)
        if ((rc = launch_composite(w.rgb, w.sig, t, rays->rays_d, nullptr, n, N, cfg->white_bkgd, 2, out->comp_rgb[lvl], out->acc[lvl], wt, nullptr,
                                   out->depth[lvl], s))) return rc;
        if ((rc = copy_out(out->t[lvl], t, (size_t)n * N, s))) return rc;
        if ((rc = copy_out(out->sigma[lvl], w.sig, (size_t)n * N, s))) return rc;
        if ((rc = copy_out(out->rgb_s[lvl], w.rgb, (size_t)n * N * 3, s))) return rc;
        if ((rc = copy_out(out->weights[lvl], wt, (size_t)n * N, s))) return rc;
    }
    return NEO_OK;
}

extern "C" size_t neo_vanilla_field_workspace_bytes(long long n_points, int precision) {
    if (n_points <= 0) return 0;
    Carve c{nullptr, 0};
    WSF w;
    carve_field(c, (size_t)n_points, w, precision);
    return c.used;
}

extern "C" int neo_vanilla_field_eval(const NeoVanilla* v, const NeoRays* rays, const float* t_vals, int N, int level, int precision, float* rgb,
                                      float* sigma, void* ws, size_t ws_bytes, void* stream) {
    if (!v || !rays || !t_vals || !rgb || !sigma) { set_error("neo_vanilla_field_eval: null argument"); return NEO_ERR_INVALID; }
    if (rays->n_rays <= 0 || !rays->rays_o || !rays->viewdirs || N < 1) { set_error("neo_vanilla_field_eval: empty rays or N < 1"); return NEO_ERR_INVALID; }
    if (level != 0 && level != 1) { set_error("neo_vanilla_field_eval: level must be 0 (coarse) or 1 (fine), got %d", level); return NEO_ERR_INVALID; }
    if (precision != NEO_PREC_FP32 && precision != NEO_PREC_TC) { set_error("neo_vanilla_field_eval: bad precision %d", precision); return NEO_ERR_INVALID; }
    const long long M = (long long)rays->n_rays * N;
    if (M > ((long long)1 << 31) - 1) { set_error("neo_vanilla_field_eval: n_rays * N must be below 2^31"); return NEO_ERR_INVALID; }
    Carve c{static_cast<unsigned char*>(ws), 0};
    WSF w;
    carve_field(c, (size_t)M, w, precision);
    if (c.used && (!ws || ws_bytes < c.used)) { set_error("workspace too small: need %zu bytes, got %zu", c.used, ws_bytes); return NEO_ERR_WORKSPACE; }
    return field(v->mlp[level], rays->rays_o, rays->viewdirs, t_vals, rays->n_rays, N, precision, w, rgb, sigma, (cudaStream_t)stream);
}

// ---- stage-level entry points of the training path (neo360_b200/vanilla.py): sampling and encodings have no backward; the compositing
// backward is composite_bwd_kernel in mode 2 (csrc/sampling.cu); the dense layers are differentiated by the host framework ----
extern "C" int neo_vanilla_sample_along_rays(const float* rays_o, const float* viewdirs, int n_rays, int n_coarse, float near_plane, float far_plane,
                                             const float* u_rand, float* t_vals, void* stream) {
    if (!rays_o || !viewdirs || !t_vals || n_rays <= 0 || n_coarse < 1) { set_error("neo_vanilla_sample_along_rays: bad arguments"); return NEO_ERR_INVALID; }
    const long long total = (long long)n_rays * (n_coarse + 1);
    van::sample_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(rays_o, viewdirs, n_rays, n_coarse, near_plane, far_plane,
                                                                                          u_rand, t_vals);
    NEO_LAUNCH_CHECK("vanilla sample_kernel");
    return NEO_OK;
}

extern "C" int neo_vanilla_encode(const float* rays_o, const float* viewdirs, const float* t_vals, int n_rays, int N, float* enc, float* dir_enc,
                                  void* stream) {
    if (!rays_o || !viewdirs || !t_vals || !enc || !dir_enc || n_rays <= 0 || N < 1) { set_error("neo_vanilla_encode: bad arguments"); return NEO_ERR_INVALID; }
    const long long total = (long long)n_rays * N * van::kEnc + (long long)n_rays * kDirEnc;
    van::encode_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(rays_o, viewdirs, t_vals, n_rays, N, enc, dir_enc);
    NEO_LAUNCH_CHECK("vanilla encode_kernel");
    return NEO_OK;
}

extern "C" int neo_vanilla_composite_bwd(const float* rgb, const float* sigma, const float* t_vals, const float* rays_d, int n_rays, int N, int white_bkgd,
                                         const float* g_comp_rgb, const float* g_acc, const float* g_weights, const float* g_depth, float* d_rgb,
                                         float* d_sigma, void* stream) {
    if (!rgb || !sigma || !t_vals || !rays_d || !d_rgb || !d_sigma || n_rays <= 0 || N < 1) {
        set_error("neo_vanilla_composite_bwd: bad arguments");
        return NEO_ERR_INVALID;
    }
    return launch_composite_bwd(rgb, sigma, t_vals, rays_d, nullptr, n_rays, N, white_bkgd, 2, g_comp_rgb, g_acc, g_weights, nullptr, g_depth,
                                d_rgb, d_sigma, (cudaStream_t)stream);
}
