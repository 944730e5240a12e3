// PixelNeRF (models/vanilla_nerf/model_pixel.py:35-258): the per-view field of one level in the reference formulation on fp32 CUDA cores
// (the parity path) and on the tensor cores (gemm_f16), and the per-view encodings of the training path.  Sampling, the 512-channel lookup's training form and compositing are the library's
// existing stages (vanilla sampling, neo_index_maps*, neo_volumetric_rendering mode 2 and neo_vanilla_composite_bwd).
//
// Cameras: the scene passed here is built from the source poses with the camera y axis negated (column 1 of each rotation).  Negation
// is exact, so its camera-frame points are PixelNeRF's with y negated bit for bit, and the shared projection (local_grid_coords, which
// negates the y focal as NeO-360's get_local_feats does, models/neo360/model.py:243) then gives exactly PixelNeRF's pixel coordinates
// (util.py:36-51 with an un-negated focal).  The encodings negate y back.
#include "common.cuh"

namespace neo {
namespace {

constexpr int kThreads = 128;                       // one thread per hidden unit
constexpr int kEnc = 63;                            // pos_enc(cam xyz, 0, 10)
constexpr int kIn = kEnc + kLocalCh;                // 575: [enc | latent]
constexpr int kLdx = 580;                           // row stride of the input tile (16-byte rows)
constexpr int kLdh = kHidden + 4;

// Rays of one call; row j = b*N + s of a view is conditioned on ray (j mod B_chunk) of its chunk (quirk Q1, model_pixel.py:227-232).
__device__ __forceinline__ int q1_source(int b, int s, int N, int n_rays, int chunk) {
    const int ch = chunk > 0 ? chunk : n_rays;
    const int c0 = (b / ch) * ch;
    const int Bc = min(ch, n_rays - c0);
    return c0 + (int)(((long long)(b - c0) * N + s) % Bc);
}

// Camera-frame sample point (y restored) and direction of the conditioning ray in view v; helper.py:20-26 (o + t d along rays_d).
__device__ __forceinline__ void row_geometry(const SceneDev& sc, int v, const float* __restrict__ o, const float* __restrict__ d,
                                             const float* __restrict__ vd, float t, float* cam, float* dir) {
    float x[3] = {add_(o[0], mul_(t, d[0])), add_(o[1], mul_(t, d[1])), add_(o[2], mul_(t, d[2]))};
    to_camera(sc.views[v], x, cam);
    rotate_to_camera(sc.views[v], vd, dir);
    dir[1] = -dir[1];
}

struct RowGeo {
    float enc_in[3];
    float dir[3];
    Taps local;
    int valid;
};

template <int NV>
struct Tile { static constexpr int P = NV <= 4 ? 8 : 4; static constexpr int ROWS = NV * P; };

template <int NV>
__global__ void __launch_bounds__(kThreads)
pixel_field_kernel(SceneDev sc, const float* __restrict__ latent_cl, NeoPixelMLPParams m, const float* __restrict__ rays_o,
                   const float* __restrict__ rays_d, const float* __restrict__ viewdirs, const float* __restrict__ tvals, int n_rays, int N,
                   int chunk, float* __restrict__ rgb_out, float* __restrict__ sigma_out) {
    constexpr int P = Tile<NV>::P, ROWS = Tile<NV>::ROWS;
    extern __shared__ __align__(16) float smem[];
    float* X = smem;                                // [ROWS][kLdx]   [enc | latent]
    float* Ha = X + ROWS * kLdx;                    // [ROWS][kLdh]
    float* Hb = Ha + ROWS * kLdh;                   // [ROWS][kLdh]
    float* Dn = Hb + ROWS * kLdh;                   // [ROWS][28]     direction encodings
    float* Q = Dn + ROWS * 28;                      // [P][kLdh] x 2
    RowGeo* geo = reinterpret_cast<RowGeo*>(Q + 2 * P * kLdh);
    const int j = threadIdx.x;
    const long long total = (long long)n_rays * N;
    const long long tile0 = (long long)blockIdx.x * P;

    // ---- geometry per (view, point) row ----
    if (j < ROWS) {
        const int v = j / P, p = j % P;
        const long long gp = tile0 + p;
        RowGeo& rg = geo[j];
        rg.valid = gp < total;
        if (rg.valid) {
            const int b = (int)(gp / N), s = (int)(gp % N);
            float cam[3];
            row_geometry(sc, v, rays_o + 3 * b, rays_d + 3 * b, viewdirs + 3 * q1_source(b, s, N, n_rays, chunk), tvals[gp], cam, rg.dir);
            float gx, gy;
            local_grid_coords(sc, cam, gx, gy);
            bilinear_taps(gx, gy, sc.lat_w, sc.lat_h, rg.local);
            rg.enc_in[0] = cam[0]; rg.enc_in[1] = -cam[1]; rg.enc_in[2] = cam[2];
        }
    }
    __syncthreads();

    // ---- inputs X = [pos_enc | latent lookup], Dn = direction pos_enc ----
    for (int e = j; e < ROWS * kEnc; e += kThreads) {
        const int r = e / kEnc, c = e % kEnc;
        X[r * kLdx + c] = geo[r].valid ? pos_enc_col(geo[r].enc_in, 3, kPosDeg, c) : 0.f;
    }
    for (int e = j; e < ROWS * 28; e += kThreads) {
        const int r = e / 28, c = e % 28;
        Dn[e] = (geo[r].valid && c < kDirEnc) ? pos_enc_col(geo[r].dir, 3, 4, c) : 0.f;
    }
    for (int r = 0; r < ROWS; ++r) {
        const RowGeo& rg = geo[r];
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
        if (rg.valid) {
            const float* lat = latent_cl + (size_t)(r / P) * sc.lat_h * sc.lat_w * kLocalCh;
#pragma unroll
            for (int tp = 0; tp < 4; ++tp) {
                const float w = rg.local.w[tp];
                const float4 f = __ldg(reinterpret_cast<const float4*>(lat + (size_t)rg.local.idx[tp] * kLocalCh) + j);
                a.x += f.x * w; a.y += f.y * w; a.z += f.z * w; a.w += f.w * w;
            }
        }
        float* xr = X + r * kLdx + kEnc;
        xr[4 * j + 0] = a.x; xr[4 * j + 1] = a.y; xr[4 * j + 2] = a.z; xr[4 * j + 3] = a.w;
    }
    __syncthreads();

    // ---- trunk 575 -> 128 x4 (ReLU), per view ----
    float acc[ROWS];
    auto bias_init = [&](const float* bp) {
        const float bv = __ldg(bp + j);
#pragma unroll
        for (int r = 0; r < ROWS; ++r) acc[r] = bv;
    };
    auto store_relu = [&](float* H) {
#pragma unroll
        for (int r = 0; r < ROWS; ++r) H[r * kLdh + j] = fmaxf(acc[r], 0.f);
    };
    bias_init(m.b[0]); dense_rows<ROWS>(m.wt[0], kHidden, kIn, X, kLdx, acc, j); store_relu(Ha); __syncthreads();
    bias_init(m.b[1]); dense_rows<ROWS>(m.wt[1], kHidden, kHidden, Ha, kLdh, acc, j); store_relu(Hb); __syncthreads();
    bias_init(m.b[2]); dense_rows<ROWS>(m.wt[2], kHidden, kHidden, Hb, kLdh, acc, j); store_relu(Ha); __syncthreads();
    bias_init(m.b[3]); dense_rows<ROWS>(m.wt[3], kHidden, kHidden, Ha, kLdh, acc, j); store_relu(Hb); __syncthreads();
    // ---- per-view bottleneck -> Ha; view mean of h3 -> density (ReLU) ----
    bias_init(m.bb); dense_rows<ROWS>(m.wbt, kHidden, kHidden, Hb, kLdh, acc, j);
#pragma unroll
    for (int r = 0; r < ROWS; ++r) Ha[r * kLdh + j] = acc[r];
    {
        const float ws = __ldg(m.wsig + j);
        float* red = Q;                             // [4 warps][P]
#pragma unroll
        for (int p = 0; p < P; ++p) {
            float s = 0.f;
#pragma unroll
            for (int v = 0; v < NV; ++v) s += Hb[(v * P + p) * kLdh + j];
            const float part = warp_sum((s / (float)NV) * ws);
            if ((j & 31) == 0) red[(j >> 5) * P + p] = part;
        }
    }
    __syncthreads();
    if (j < P) {
        const long long gp = tile0 + j;
        if (gp < total) sigma_out[gp] = fmaxf(((Q[j] + Q[P + j]) + (Q[2 * P + j] + Q[3 * P + j])) + __ldg(m.bsig), 0.f);
    }
    __syncthreads();
    // ---- view branch: [bottleneck | dir] (155) -> 128, mean over views, ReLU, 128 -> 128 ReLU, 128 -> 3 sigmoid ----
    float* q0 = Q;
    float* q1 = Q + P * kLdh;
    bias_init(m.bv0);
    dense_rows<ROWS>(m.wv0t, kHidden, kHidden, Ha, kLdh, acc, j);
    dense_rows<ROWS>(m.wv0t + (size_t)kHidden * kHidden, kHidden, kDirEnc, Dn, 28, acc, j);
#pragma unroll
    for (int p = 0; p < P; ++p) {
        float s = 0.f;
#pragma unroll
        for (int v = 0; v < NV; ++v) s += acc[v * P + p];
        q0[p * kLdh + j] = fmaxf(s / (float)NV, 0.f);
    }
    __syncthreads();
    {
        float a2[P];
        const float bv = __ldg(m.bv1 + j);
#pragma unroll
        for (int p = 0; p < P; ++p) a2[p] = bv;
        dense_rows<P>(m.wv1t, kHidden, kHidden, q0, kLdh, a2, j);
#pragma unroll
        for (int p = 0; p < P; ++p) q1[p * kLdh + j] = fmaxf(a2[p], 0.f);
    }
    __syncthreads();
    if (j < P * 3) {
        const int p = j / 3, c = j % 3;
        const long long gp = tile0 + p;
        if (gp < total) {
            float a = __ldg(m.brgb + c);
            for (int k = 0; k < kHidden; ++k) a = fmaf(q1[p * kLdh + k], __ldg(m.wrgb + c * kHidden + k), a);
            rgb_out[gp * 3 + c] = sigmoid_(a);
        }
    }
}

template <int NV>
size_t field_smem() {
    constexpr int P = Tile<NV>::P, ROWS = Tile<NV>::ROWS;
    return ((size_t)ROWS * kLdx + 2 * (size_t)ROWS * kLdh + (size_t)ROWS * 28 + 2 * (size_t)P * kLdh) * sizeof(float)
           + (size_t)ROWS * sizeof(RowGeo);
}

template <int NV>
int launch_nv(const NeoScene* sc, const float* lat, const NeoPixelMLPParams& m, const NeoRays* r, const float* t, int N, float* rgb,
              float* sigma, cudaStream_t s) {
    const size_t smem = field_smem<NV>();
    NEO_CUDA(cudaFuncSetAttribute(pixel_field_kernel<NV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long long total = (long long)r->n_rays * N;
    const unsigned grid = (unsigned)((total + Tile<NV>::P - 1) / Tile<NV>::P);
    pixel_field_kernel<NV><<<grid, kThreads, smem, s>>>(sc->dev, lat, m, r->rays_o, r->rays_d, r->viewdirs, t, r->n_rays, N, r->chunk, rgb,
                                                        sigma);
    NEO_LAUNCH_CHECK("pixel_field_kernel");
    return NEO_OK;
}

// enc (nv*M, 63), dir_tile (nv*M, 27), pts (M, 3) world points; M = n_rays * N, rows ordered (view, point)
__global__ void pixel_encode_kernel(SceneDev sc, const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                    const float* __restrict__ viewdirs, const float* __restrict__ tvals, int n_rays, int N, int chunk,
                                    float* __restrict__ enc, float* __restrict__ dir_tile, float* __restrict__ pts) {
    const long long M = (long long)n_rays * N;
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= (long long)sc.nv * M) return;
    const int v = (int)(row / M);
    const long long gp = row % M;
    const int b = (int)(gp / N), s = (int)(gp % N);
    const float* o = rays_o + 3 * b;
    const float* d = rays_d + 3 * b;
    const float t = tvals[gp];
    float cam[3], dir[3];
    row_geometry(sc, v, o, d, viewdirs + 3 * q1_source(b, s, N, n_rays, chunk), t, cam, dir);
    cam[1] = -cam[1];
    for (int c = 0; c < kEnc; ++c) enc[row * kEnc + c] = pos_enc_col(cam, 3, kPosDeg, c);
    for (int c = 0; c < kDirEnc; ++c) dir_tile[row * kDirEnc + c] = pos_enc_col(dir, 3, 4, c);
    if (v == 0 && pts)
        for (int i = 0; i < 3; ++i) pts[gp * 3 + i] = add_(o[i], mul_(t, d[i]));
}


// ---- NEO_PREC_TC: the reference formulation layer by layer on gemm_f16 (fp16 operands, fp32 accumulation) ----
constexpr int kLdX = 576;                           // [enc 63 | latent 512 | 0]
constexpr int kLdD = 192;                           // [bottleneck 128 | dir 27 | 0]: views_linear.0's operand
constexpr long long kSlice = 65536;                 // points per pass: bounds the workspace (about 2 KB per point and view)

// One warp per (view, point) row: the fp16 rows X and the direction columns of D, the field kernel's geometry and lookup arithmetic.
__global__ void __launch_bounds__(256) pixel_rows16_kernel(SceneDev sc, const float* __restrict__ latent_cl, const float* __restrict__ rays_o,
                                                           const float* __restrict__ rays_d, const float* __restrict__ viewdirs,
                                                           const float* __restrict__ tvals, int n_rays, int N, int chunk, long long p0,
                                                           long long Ms, __half* __restrict__ X, __half* __restrict__ D) {
    const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= (long long)sc.nv * Ms) return;
    const int v = (int)(row / Ms);
    const long long gp = p0 + row % Ms;
    const int b = (int)(gp / N), s = (int)(gp % N);
    float cam[3], dir[3];
    row_geometry(sc, v, rays_o + 3 * b, rays_d + 3 * b, viewdirs + 3 * q1_source(b, s, N, n_rays, chunk), tvals[gp], cam, dir);
    Taps tp;
    float gx, gy;
    local_grid_coords(sc, cam, gx, gy);
    bilinear_taps(gx, gy, sc.lat_w, sc.lat_h, tp);
    cam[1] = -cam[1];
    __half* x = X + row * kLdX;
    __half* d = D + row * kLdD;
    for (int c = lane; c < 64; c += 32) x[c] = __float2half_rn(c < kEnc ? pos_enc_col(cam, 3, kPosDeg, c) : 0.f);
    for (int c = lane; c < 64; c += 32) d[kHidden + c] = __float2half_rn(c < kDirEnc ? pos_enc_col(dir, 3, 4, c) : 0.f);
    const float* lat = latent_cl + (size_t)v * sc.lat_h * sc.lat_w * kLocalCh;
    for (int q = lane; q < kLocalCh / 4; q += 32) {
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float w = tp.w[k];
            const float4 f = __ldg(reinterpret_cast<const float4*>(lat + (size_t)tp.idx[k] * kLocalCh) + q);
            a.x += f.x * w; a.y += f.y * w; a.z += f.z * w; a.w += f.w * w;
        }
        __half* o = x + kEnc + 4 * q;                 // column 63 + 4q: not 8-byte aligned, so four stores
        o[0] = __float2half_rn(a.x); o[1] = __float2half_rn(a.y); o[2] = __float2half_rn(a.z); o[3] = __float2half_rn(a.w);
    }
    if (lane == 0) x[kLdX - 1] = __float2half_rn(0.f);
}

// out (Ms, 128) fp16 = [ReLU](mean over the nv views of in (nv*Ms rows, row stride ld) fp16), summed in view order in fp32
__global__ void pixel_view_mean_kernel(const __half* __restrict__ in, long long ld, int nv, long long Ms, int relu, __half* __restrict__ out) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= Ms * kHidden) return;
    const long long p = e / kHidden;
    const int c = (int)(e % kHidden);
    float s = 0.f;
    for (int v = 0; v < nv; ++v) s += __half2float(in[((long long)v * Ms + p) * ld + c]);
    s = s / (float)nv;
    out[e] = __float2half_rn(relu ? fmaxf(s, 0.f) : s);
}

// sigma = relu(raw), rgb = sigmoid(raw) (model_pixel.py:164-165)
__global__ void pixel_act_kernel(const float* __restrict__ raw_sigma, const float* __restrict__ raw_rgb, long long Ms,
                                 float* __restrict__ sigma, float* __restrict__ rgb) {
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= Ms) return;
    sigma[p] = fmaxf(raw_sigma[p], 0.f);
    for (int c = 0; c < 3; ++c) rgb[3 * p + c] = sigmoid_(raw_rgb[3 * p + c]);
}

struct TCWork { __half *X, *Ha, *Hb, *D, *hbar, *q0, *q1; float *rs, *rr; };
TCWork tc_carve(void* base, int nv, long long Ms, size_t* used) {
    Carve c{(unsigned char*)base, 0};
    const long long R = nv * Ms;
    TCWork w;
    w.X = c.take<__half>(R * kLdX); w.Ha = c.take<__half>(R * kHidden); w.Hb = c.take<__half>(R * kHidden); w.D = c.take<__half>(R * kLdD);
    w.hbar = c.take<__half>(Ms * kHidden); w.q0 = c.take<__half>(Ms * kHidden); w.q1 = c.take<__half>(Ms * kHidden);
    w.rs = c.take<float>(Ms); w.rr = c.take<float>(Ms * 3);
    *used = c.used;
    return w;
}

bool check_rays(const char* who, const NeoScene* sc, const NeoRays* r, const float* t, int N) {
    if (!sc || !r || !t || !r->rays_o || !r->rays_d || !r->viewdirs || r->n_rays <= 0 || N <= 0) {
        set_error("%s: null argument or empty batch", who);
        return false;
    }
    if ((long long)r->n_rays * N * sc->dev.nv >= (1LL << 31)) {
        set_error("%s: n_rays * N * nv must stay below 2^31", who);
        return false;
    }
    return true;
}

}  // namespace
}  // namespace neo

using namespace neo;

extern "C" int neo_pixelnerf_field(const NeoScene* sc, const float* latent_cl, const NeoPixelMLPParams* mlp, const NeoRays* rays,
                                   const float* t_vals, int N, float* rgb, float* sigma, void* stream) {
    if (!check_rays("neo_pixelnerf_field", sc, rays, t_vals, N)) return NEO_ERR_INVALID;
    if (!latent_cl || !mlp || !rgb || !sigma) { set_error("neo_pixelnerf_field: null argument"); return NEO_ERR_INVALID; }
    const NeoPixelMLPParams& m = *mlp;
    for (int i = 0; i < 4; ++i)
        if (!m.wt[i] || !m.b[i]) { set_error("neo_pixelnerf_field: null weight"); return NEO_ERR_INVALID; }
    if (!m.wbt || !m.bb || !m.wsig || !m.bsig || !m.wv0t || !m.bv0 || !m.wv1t || !m.bv1 || !m.wrgb || !m.brgb) {
        set_error("neo_pixelnerf_field: null weight");
        return NEO_ERR_INVALID;
    }
    if (((uintptr_t)latent_cl & 15) || ((uintptr_t)m.wt[0] & 15) || ((uintptr_t)m.wt[1] & 15) || ((uintptr_t)m.wt[2] & 15) ||
        ((uintptr_t)m.wt[3] & 15) || ((uintptr_t)m.wbt & 15) || ((uintptr_t)m.wv0t & 15) || ((uintptr_t)m.wv1t & 15)) {
        set_error("neo_pixelnerf_field: latent and transposed weights must be 16-byte aligned");
        return NEO_ERR_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    switch (sc->dev.nv) {
        case 1: return launch_nv<1>(sc, latent_cl, m, rays, t_vals, N, rgb, sigma, s);
        case 2: return launch_nv<2>(sc, latent_cl, m, rays, t_vals, N, rgb, sigma, s);
        case 3: return launch_nv<3>(sc, latent_cl, m, rays, t_vals, N, rgb, sigma, s);
        case 4: return launch_nv<4>(sc, latent_cl, m, rays, t_vals, N, rgb, sigma, s);
        case 5: return launch_nv<5>(sc, latent_cl, m, rays, t_vals, N, rgb, sigma, s);
        case 6: return launch_nv<6>(sc, latent_cl, m, rays, t_vals, N, rgb, sigma, s);
        case 7: return launch_nv<7>(sc, latent_cl, m, rays, t_vals, N, rgb, sigma, s);
        case 8: return launch_nv<8>(sc, latent_cl, m, rays, t_vals, N, rgb, sigma, s);
    }
    set_error("neo_pixelnerf_field: 1..8 source views (got %d)", sc->dev.nv);
    return NEO_ERR_UNSUPPORTED;
}

extern "C" int neo_pixelnerf_encode(const NeoScene* sc, const NeoRays* rays, const float* t_vals, int N, float* enc, float* dir_tile,
                                    float* pts, void* stream) {
    if (!check_rays("neo_pixelnerf_encode", sc, rays, t_vals, N)) return NEO_ERR_INVALID;
    if (!enc || !dir_tile) { set_error("neo_pixelnerf_encode: null output"); return NEO_ERR_INVALID; }
    const long long rows = (long long)sc->dev.nv * rays->n_rays * N;
    pixel_encode_kernel<<<(unsigned)((rows + 127) / 128), 128, 0, (cudaStream_t)stream>>>(sc->dev, rays->rays_o, rays->rays_d, rays->viewdirs,
                                                                                       t_vals, rays->n_rays, N, rays->chunk, enc, dir_tile, pts);
    NEO_LAUNCH_CHECK("pixel_encode_kernel");
    return NEO_OK;
}

extern "C" size_t neo_pixelnerf_tc_workspace_bytes(int nv, long long M) {
    if (nv < 1 || nv > kMaxViews || M <= 0) return 0;
    size_t used = 0;
    tc_carve(nullptr, nv, M < kSlice ? M : kSlice, &used);
    return used;
}

extern "C" int neo_pixelnerf_field_tc(const NeoScene* sc, const float* latent_cl, const NeoPixelTCParams* mlp, const NeoRays* rays,
                                      const float* t_vals, int N, float* rgb, float* sigma, void* workspace, size_t workspace_bytes,
                                      void* stream) {
    if (!check_rays("neo_pixelnerf_field_tc", sc, rays, t_vals, N)) return NEO_ERR_INVALID;
    if (!latent_cl || !mlp || !rgb || !sigma || !workspace || ((uintptr_t)latent_cl & 15) || ((uintptr_t)workspace & 255)) {
        set_error("neo_pixelnerf_field_tc: null argument, or latent not 16-byte / workspace not 256-byte aligned");
        return NEO_ERR_INVALID;
    }
    const NeoPixelTCParams& m = *mlp;
    for (int i = 0; i < 4; ++i)
        if (!m.w16[i] || !m.b[i]) { set_error("neo_pixelnerf_field_tc: null weight"); return NEO_ERR_INVALID; }
    if (!m.wb16 || !m.bb || !m.wsig || !m.bsig || !m.wv016 || !m.bv0 || !m.wv116 || !m.bv1 || !m.wrgb || !m.brgb) {
        set_error("neo_pixelnerf_field_tc: null weight");
        return NEO_ERR_INVALID;
    }
    const int nv = sc->dev.nv;
    const long long M = (long long)rays->n_rays * N;
    if (workspace_bytes < neo_pixelnerf_tc_workspace_bytes(nv, M)) { set_error("neo_pixelnerf_field_tc: workspace too small"); return NEO_ERR_WORKSPACE; }
    cudaStream_t s = (cudaStream_t)stream;
    for (long long p0 = 0; p0 < M; p0 += kSlice) {
        const long long Ms = M - p0 < kSlice ? M - p0 : kSlice, R = nv * Ms;
        size_t used;
        const TCWork w = tc_carve(workspace, nv, Ms, &used);
        pixel_rows16_kernel<<<(unsigned)((R * 32 + 255) / 256), 256, 0, s>>>(sc->dev, latent_cl, rays->rays_o, rays->rays_d, rays->viewdirs,
                                                                            t_vals, rays->n_rays, N, rays->chunk, p0, Ms, w.X, w.D);
        NEO_LAUNCH_CHECK("pixel_rows16_kernel");
        int rc;
        if ((rc = gemm_f16(w.X, kLdX, m.w16[0], kLdX, m.b[0], w.Ha, kHidden, R, kHidden, kLdX, 1, s))) return rc;
        if ((rc = gemm_f16(w.Ha, kHidden, m.w16[1], kHidden, m.b[1], w.Hb, kHidden, R, kHidden, kHidden, 1, s))) return rc;
        if ((rc = gemm_f16(w.Hb, kHidden, m.w16[2], kHidden, m.b[2], w.Ha, kHidden, R, kHidden, kHidden, 1, s))) return rc;
        if ((rc = gemm_f16(w.Ha, kHidden, m.w16[3], kHidden, m.b[3], w.Hb, kHidden, R, kHidden, kHidden, 1, s))) return rc;   // h3
        if ((rc = gemm_f16(w.Hb, kHidden, m.wb16, kHidden, m.bb, w.D, kLdD, R, kHidden, kHidden, 0, s))) return rc;           // bottleneck
        const unsigned g = (unsigned)((Ms * kHidden + 255) / 256);
        pixel_view_mean_kernel<<<g, 256, 0, s>>>(w.Hb, kHidden, nv, Ms, 0, w.hbar);
        NEO_LAUNCH_CHECK("pixel_view_mean_kernel(trunk)");
        if ((rc = launch_rowdot_f16(w.hbar, kHidden, kHidden, m.wsig, m.bsig, 1, Ms, w.rs, s))) return rc;
        if ((rc = gemm_f16(w.D, kLdD, m.wv016, kLdD, m.bv0, w.Ha, kHidden, R, kHidden, kLdD, 0, s))) return rc;
        pixel_view_mean_kernel<<<g, 256, 0, s>>>(w.Ha, kHidden, nv, Ms, 1, w.q0);
        NEO_LAUNCH_CHECK("pixel_view_mean_kernel(views)");
        if ((rc = gemm_f16(w.q0, kHidden, m.wv116, kHidden, m.bv1, w.q1, kHidden, Ms, kHidden, kHidden, 1, s))) return rc;
        if ((rc = launch_rowdot_f16(w.q1, kHidden, kHidden, m.wrgb, m.brgb, 3, Ms, w.rr, s))) return rc;
        pixel_act_kernel<<<(unsigned)((Ms + 255) / 256), 256, 0, s>>>(w.rs, w.rr, Ms, sigma + p0, rgb + 3 * p0);
        NEO_LAUNCH_CHECK("pixel_act_kernel");
    }
    return NEO_OK;
}
