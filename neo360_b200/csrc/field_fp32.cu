// Exact-arithmetic (CUDA-core fp32) evaluation of the NeO-360 radiance field in the REFERENCE formulation:
// world->camera, tri-plane + pixel-aligned bilinear lookups, positional encoding, NeRFPPMLP with the
// cross-view means, activations.  This is the tight-parity path (NEO_PREC_FP32) and the on-GPU check for the
// tensor-core path in field_tc.cu.  Reference: models/neo360/model.py:110-158, 239-264, 339-472;
// encoder_tp_fusion_conv.py:122-209; encoder_pn.py:101-152; util.py:45-111; helper.py:121-125.
#include "common.cuh"

namespace neo {

constexpr int kThreads = 128;  // one thread per hidden unit
constexpr int kMaxInDim = 4 * (2 * kPosDeg + 1) + kLocalCh + kWorldCh;   // background MLP: [pos_enc(xyz, 1/r) | local | world]
constexpr size_t kSmemLimit = 227 * 1024;                               // opt-in dynamic shared memory per block on sm_90

// Points per CTA.  Each point has one row per view in shared memory, so the tile shrinks from 8 to 4 points above 6 views to stay
// within kSmemLimit.  A point's arithmetic does not depend on the tile: only which CTA evaluates it changes.
__host__ __device__ constexpr int points_per_cta(int nv) { return nv <= 6 ? 8 : 4; }

struct RowGeo {
    float enc_in[4];    // camera-frame position fed to pos_enc (+ 1/r for bg)
    float dir[3];       // camera-frame view direction of the (quirk-Q1) conditioning ray
    Taps local;
    Taps plane[3];      // xz, xy, yz
    int valid;
};

template <int NV>
__global__ void __launch_bounds__(kThreads)
field_fp32_kernel(SceneDev sc, MLPFp32 mlp, const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                  const float* __restrict__ viewdirs, const float* __restrict__ far, const float* __restrict__ tvals,
                  int n_rays, int N, int chunk, int is_bg, float far_unc, float* __restrict__ rgb_out,
                  float* __restrict__ sigma_out) {
    constexpr int kP = points_per_cta(NV);
    constexpr int ROWS = NV * kP;
    extern __shared__ __align__(16) float smem[];
    const int in_dim = mlp.in_dim;                 // enc + 512 + 128
    const int ldx = (in_dim + 3) / 4 * 4 + 4;
    float* X = smem;                               // [ROWS][ldx]   inputs  [enc | local | world]
    float* Ha = X + ROWS * ldx;                    // [ROWS][128+4]
    float* Hb = Ha + ROWS * (kHidden + 4);         // [ROWS][128+4]
    float* Dn = Hb + ROWS * (kHidden + 4);         // [ROWS][28]  direction encodings
    float* Q = Dn + ROWS * 28;                     // [kP][64+4] x2
    RowGeo* geo = reinterpret_cast<RowGeo*>(Q + 2 * kP * 68);
    const int ldh = kHidden + 4;
    const int j = threadIdx.x;
    const long long total = (long long)n_rays * N;
    const long long tile0 = (long long)blockIdx.x * kP;

    // ---- phase A: geometry per (view, point) row ----
    if (j < ROWS) {
        int v = j / kP, p = j % kP;
        long long gp = tile0 + p;
        RowGeo& rg = geo[j];
        rg.valid = gp < total;
        if (rg.valid) {
            int b = (int)(gp / N), s = (int)(gp % N);
            RayGeom g;
            ray_geom(rays_o + 3 * b, rays_d + 3 * b, g, is_bg);
            g.far = far[b];
            float tv = tvals[gp];
            float xe[3], xl[3];
            if (is_bg) bg_point(g, tv, far_unc, xe, xl);
            else { fg_point(g, tv, xe); xl[0] = xe[0]; xl[1] = xe[1]; xl[2] = xe[2]; }
            const ViewXform& vx = sc.views[v];
            float ce[3], cl[3];
            to_camera(vx, xe, ce);
            to_camera(vx, xl, cl);
            rg.enc_in[0] = ce[0]; rg.enc_in[1] = ce[1]; rg.enc_in[2] = ce[2]; rg.enc_in[3] = tv;
            // quirk Q1: row (b_local*N + s) of the chunk is conditioned on ray ((b_local*N + s) mod B_chunk)
            int ch = chunk > 0 ? chunk : n_rays;
            int c0 = (b / ch) * ch;
            int Bc = min(ch, n_rays - c0);
            long long jl = (long long)(b - c0) * N + s;
            int src = c0 + (int)(jl % Bc);
            rotate_to_camera(vx, viewdirs + 3 * src, rg.dir);
            float gx, gy;
            local_grid_coords(sc, cl, gx, gy);
            bilinear_taps(gx, gy, sc.lat_w, sc.lat_h, rg.local);
            bilinear_taps(cl[0], cl[2], sc.plane_w, sc.plane_h, rg.plane[0]);   // xz
            bilinear_taps(cl[0], cl[1], sc.plane_w, sc.plane_h, rg.plane[1]);   // xy
            bilinear_taps(cl[1], cl[2], sc.plane_w, sc.plane_h, rg.plane[2]);   // yz
        }
    }
    __syncthreads();

    // ---- phase B: inputs  X = [pos_enc | local latent | world latent],  Dn = dir pos_enc ----
    const int ich = mlp.in_ch, enc = mlp.enc_dim;
    for (int e = j; e < ROWS * enc; e += kThreads) {
        int r = e / enc, c = e % enc;
        const RowGeo& rg = geo[r];
        X[r * ldx + c] = rg.valid ? pos_enc_col(rg.enc_in, ich, kPosDeg, c) : 0.f;
    }
    for (int e = j; e < ROWS * 28; e += kThreads) {
        int r = e / 28, c = e % 28;
        const RowGeo& rg = geo[r];
        Dn[e] = (rg.valid && c < kDirEnc) ? pos_enc_col(rg.dir, 3, 4, c) : 0.f;
    }
    for (int r = 0; r < ROWS; ++r) {
        const RowGeo& rg = geo[r];
        int v = r / kP;
        float4 accl = make_float4(0.f, 0.f, 0.f, 0.f);
        float accw = 0.f;
        if (rg.valid) {
            const float* lat = sc.latent_cl + (size_t)v * sc.lat_h * sc.lat_w * kLocalCh;
#pragma unroll
            for (int tp = 0; tp < 4; ++tp) {
                float w = rg.local.w[tp];
                float4 f = __ldg(reinterpret_cast<const float4*>(lat + (size_t)rg.local.idx[tp] * kLocalCh) + j);
                accl.x += f.x * w; accl.y += f.y * w; accl.z += f.z * w; accl.w += f.w * w;
            }
            float pl[3];
#pragma unroll
            for (int pi = 0; pi < 3; ++pi) {
                const float* pp = sc.planes_cl[pi] + (size_t)v * sc.plane_h * sc.plane_w * kWorldCh;
                float a = 0.f;
#pragma unroll
                for (int tp = 0; tp < 4; ++tp)
                    a += __ldg(pp + (size_t)rg.plane[pi].idx[tp] * kWorldCh + j) * rg.plane[pi].w[tp];
                pl[pi] = a;
            }
            accw = (pl[0] + pl[1]) + pl[2];        // torch.sum(stack([xz, xy, yz]), 0)
        }
        float* xr = X + r * ldx + enc;
        xr[4 * j + 0] = accl.x; xr[4 * j + 1] = accl.y; xr[4 * j + 2] = accl.z; xr[4 * j + 3] = accl.w;
        xr[kLocalCh + j] = accw;
    }
    __syncthreads();

    // ---- phase C: MLP ----
    float acc[ROWS];
    auto bias_init = [&](const float* bptr) {
        float bv = __ldg(bptr + j);
#pragma unroll
        for (int r = 0; r < ROWS; ++r) acc[r] = bv;
    };
    auto store_relu = [&](float* H) {
#pragma unroll
        for (int r = 0; r < ROWS; ++r) H[r * ldh + j] = fmaxf(acc[r], 0.f);
    };
    bias_init(mlp.b0); dense_rows<ROWS>(mlp.w0t, kHidden, in_dim, X, ldx, acc, j); store_relu(Ha); __syncthreads();
    bias_init(mlp.b1); dense_rows<ROWS>(mlp.w1t, kHidden, kHidden, Ha, ldh, acc, j); store_relu(Hb); __syncthreads();
    bias_init(mlp.b2); dense_rows<ROWS>(mlp.w2t, kHidden, kHidden, Hb, ldh, acc, j); store_relu(Ha); __syncthreads();
    bias_init(mlp.b3);
    dense_rows<ROWS>(mlp.w3t, kHidden, kHidden, Ha, ldh, acc, j);                              // [h2 | inputs]
    dense_rows<ROWS>(mlp.w3t + (size_t)kHidden * kHidden, kHidden, in_dim, X, ldx, acc, j);
    store_relu(Hb); __syncthreads();                                                          // Hb = h3 (per view)
    // bottleneck (per view) -> Ha ; hbar = mean_v h3 -> density
    bias_init(mlp.bb); dense_rows<ROWS>(mlp.wbt, kHidden, kHidden, Hb, ldh, acc, j);
#pragma unroll
    for (int r = 0; r < ROWS; ++r) Ha[r * ldh + j] = acc[r];
    {
        float ws = __ldg(mlp.wsig + j);
        float* red = Q;                     // [4 warps][kP]
#pragma unroll
        for (int p = 0; p < kP; ++p) {
            float m = 0.f;
#pragma unroll
            for (int v = 0; v < NV; ++v) m += Hb[(v * kP + p) * ldh + j];
            m = m / (float)NV;
            float part = warp_sum(m * ws);
            if ((j & 31) == 0) red[(j >> 5) * kP + p] = part;
        }
    }
    __syncthreads();
    if (j < kP) {
        long long gp = tile0 + j;
        if (gp < total) {
            float raw = ((Q[0 * kP + j] + Q[1 * kP + j]) + (Q[2 * kP + j] + Q[3 * kP + j])) + __ldg(mlp.bsig);
            sigma_out[gp] = softplus_(raw - 1.0f);                                  // model.py:392-393
        }
    }
    __syncthreads();
    // view branch: [bottleneck | dir_enc] -> 64, mean over views, relu, 64->64 relu, 64->3
    float* q0 = Q;
    float* q1 = Q + kP * 68;
    if (j < 64) {
        float bv = __ldg(mlp.bv0 + j);
#pragma unroll
        for (int r = 0; r < ROWS; ++r) acc[r] = bv;
        for (int k = 0; k < kHidden; ++k) {
            float w = __ldg(mlp.wv0t + (size_t)k * 64 + j);
#pragma unroll
            for (int r = 0; r < ROWS; ++r) acc[r] = fmaf(Ha[r * ldh + k], w, acc[r]);
        }
        for (int k = 0; k < kDirEnc; ++k) {
            float w = __ldg(mlp.wv0t + (size_t)(kHidden + k) * 64 + j);
#pragma unroll
            for (int r = 0; r < ROWS; ++r) acc[r] = fmaf(Dn[r * 28 + k], w, acc[r]);
        }
#pragma unroll
        for (int p = 0; p < kP; ++p) {
            float m = 0.f;
#pragma unroll
            for (int v = 0; v < NV; ++v) m += acc[v * kP + p];
            q0[p * 68 + j] = fmaxf(m / (float)NV, 0.f);
        }
    }
    __syncthreads();
    if (j < 64) {
        float a2[kP];
        float bv = __ldg(mlp.bv1 + j);
#pragma unroll
        for (int p = 0; p < kP; ++p) a2[p] = bv;
        for (int k = 0; k < 64; ++k) {
            float w = __ldg(mlp.wv1t + (size_t)k * 64 + j);
#pragma unroll
            for (int p = 0; p < kP; ++p) a2[p] = fmaf(q0[p * 68 + k], w, a2[p]);
        }
#pragma unroll
        for (int p = 0; p < kP; ++p) q1[p * 68 + j] = fmaxf(a2[p], 0.f);
    }
    __syncthreads();
    if (j < kP * 3) {
        int p = j / 3, c = j % 3;
        long long gp = tile0 + p;
        if (gp < total) {
            float a = __ldg(mlp.brgb + c);
            for (int k = 0; k < 64; ++k) a = fmaf(q1[p * 68 + k], __ldg(mlp.wrgb + c * 64 + k), a);
            rgb_out[gp * 3 + c] = rgb_act(a);                                       // model.py:395-397
        }
    }
}

static constexpr size_t field_fp32_smem(int nv, int in_dim) {
    const int kP = points_per_cta(nv);
    const int rows = nv * kP;
    const int ldx = (in_dim + 3) / 4 * 4 + 4;
    const size_t fl = (size_t)rows * ldx + 2 * (size_t)rows * (kHidden + 4) + (size_t)rows * 28 + 2 * kP * 68;
    return fl * sizeof(float) + (size_t)rows * sizeof(RowGeo);
}

template <int NV>
static int launch_nv(const NeoScene* sc, const NeoRays* rays, const float* far, const float* t, int N, int mi,
                     float* rgb, float* sigma, cudaStream_t s) {
    constexpr int kP = points_per_cta(NV);
    static_assert(field_fp32_smem(NV, kMaxInDim) <= kSmemLimit, "field_fp32_kernel tile exceeds shared memory");
    static_assert(NV * kP <= kThreads && 3 * kP <= kThreads, "phase A and the rgb head need one thread per row");
    const MLPFp32& m = sc->mlp32[mi];
    size_t smem = field_fp32_smem(NV, m.in_dim);
    NEO_CUDA(cudaFuncSetAttribute(field_fp32_kernel<NV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    long long total = (long long)rays->n_rays * N;
    unsigned grid = (unsigned)((total + kP - 1) / kP);
    field_fp32_kernel<NV><<<grid, kThreads, smem, s>>>(sc->dev, m, rays->rays_o, rays->rays_d, rays->viewdirs, far, t,
                                                       rays->n_rays, N, rays->chunk, mi & 1, 3.0f, rgb, sigma);
    NEO_LAUNCH_CHECK("field_fp32_kernel");
    return NEO_OK;
}

int launch_field_fp32(const NeoScene* sc, const NeoRays* rays, const float* far, const float* t, int N, int mlp_index,
                      float* rgb, float* sigma, cudaStream_t s) {
    if (!(sc->precision_mask & (1 << NEO_PREC_FP32))) { set_error("scene was not prepared for NEO_PREC_FP32"); return NEO_ERR_INVALID; }
    switch (sc->dev.nv) {
        case 1: return launch_nv<1>(sc, rays, far, t, N, mlp_index, rgb, sigma, s);
        case 2: return launch_nv<2>(sc, rays, far, t, N, mlp_index, rgb, sigma, s);
        case 3: return launch_nv<3>(sc, rays, far, t, N, mlp_index, rgb, sigma, s);
        case 4: return launch_nv<4>(sc, rays, far, t, N, mlp_index, rgb, sigma, s);
        case 5: return launch_nv<5>(sc, rays, far, t, N, mlp_index, rgb, sigma, s);
        case 6: return launch_nv<6>(sc, rays, far, t, N, mlp_index, rgb, sigma, s);
        case 7: return launch_nv<7>(sc, rays, far, t, N, mlp_index, rgb, sigma, s);
        case 8: return launch_nv<8>(sc, rays, far, t, N, mlp_index, rgb, sigma, s);
    }
    static_assert(kMaxViews == 8, "instantiate field_fp32_kernel for every view count up to kMaxViews");
    set_error("NEO_PREC_FP32 supports 1..%d source views (got %d)", kMaxViews, sc->dev.nv);
    return NEO_ERR_UNSUPPORTED;
}

// ------------------------------------------------------------------------------------------------
// stage-level lookups (index_grid / get_local_feats): rows ordered (view, point), channels contiguous
// ------------------------------------------------------------------------------------------------
// Maps are passed explicitly (channel-last (nv, H, W, C), spatial sizes = the scene's): the scene's own raw maps for index_grid /
// get_local_feats, or caller-owned maps of any channel count C % 4 == 0 for the training path's projected maps (neo_index_maps*).
struct MapSet { const float* lat; const float* pl[3]; };
struct MapSetW { float* lat; float* pl[3]; };

__global__ void index_kernel(SceneDev sc, const float* __restrict__ pts, int M, int local, int C, MapSet maps, float* __restrict__ out) {
    long long row = blockIdx.x;           // v*M + m
    int v = (int)(row / M), m = (int)(row % M);
    float c[3];
    to_camera(sc.views[v], pts + 3 * (size_t)m, c);
    if (local) {
        float gx, gy;
        Taps t;
        local_grid_coords(sc, c, gx, gy);
        bilinear_taps(gx, gy, sc.lat_w, sc.lat_h, t);
        const float* lat = maps.lat + (size_t)v * sc.lat_h * sc.lat_w * C;
        for (int ch = threadIdx.x; ch < C; ch += blockDim.x) {
            float val = 0.f;
            for (int tp = 0; tp < 4; ++tp) val += __ldg(lat + (size_t)t.idx[tp] * C + ch) * t.w[tp];
            out[row * C + ch] = val;
        }
    } else {
        const float ga[3] = {c[0], c[0], c[1]}, gb[3] = {c[2], c[1], c[2]};
        Taps t[3];
        for (int pi = 0; pi < 3; ++pi) bilinear_taps(ga[pi], gb[pi], sc.plane_w, sc.plane_h, t[pi]);
        for (int ch = threadIdx.x; ch < C; ch += blockDim.x) {
            float pl[3];
            for (int pi = 0; pi < 3; ++pi) {
                const float* pp = maps.pl[pi] + (size_t)v * sc.plane_h * sc.plane_w * C;
                float a = 0.f;
                for (int tp = 0; tp < 4; ++tp) a += __ldg(pp + (size_t)t[pi].idx[tp] * C + ch) * t[pi].w[tp];
                pl[pi] = a;
            }
            out[row * C + ch] = (pl[0] + pl[1]) + pl[2];
        }
    }
}


// ------------------------------------------------------------------------------------------------
// backward of the stage-level lookups: scatter-add of the row gradients into channel-last gradient maps
// (nv, H, W, C): d map[v][tap texel][:] += w_tap * d out[row][:].  A row's channels are contiguous in both tensors, so the
// atomics of one warp are 16-byte vector reductions on consecutive addresses (red.global.add.v4.f32).
// ------------------------------------------------------------------------------------------------
__global__ void index_bwd_kernel(SceneDev sc, const float* __restrict__ pts, int M, int local, int C, const float* __restrict__ g_out, MapSetW maps) {
    const long long row = blockIdx.x;           // v*M + m
    const int v = (int)(row / M), m = (int)(row % M);
    float c[3];
    to_camera(sc.views[v], pts + 3 * (size_t)m, c);
    const float4* g = reinterpret_cast<const float4*>(g_out + row * C);
    if (local) {
        float gx, gy;
        Taps t;
        local_grid_coords(sc, c, gx, gy);
        bilinear_taps(gx, gy, sc.lat_w, sc.lat_h, t);
        float* base = maps.lat + (size_t)v * sc.lat_h * sc.lat_w * C;
        for (int q = threadIdx.x; q < C / 4; q += blockDim.x) {
            const float4 gv = g[q];
            for (int tp = 0; tp < 4; ++tp) {
                const float w = t.w[tp];
                if (w != 0.f) atomicAdd(reinterpret_cast<float4*>(base + (size_t)t.idx[tp] * C) + q, make_float4(gv.x * w, gv.y * w, gv.z * w, gv.w * w));
            }
        }
    } else {
        const float ga[3] = {c[0], c[0], c[1]}, gb[3] = {c[2], c[1], c[2]};
        for (int pi = 0; pi < 3; ++pi) {
            Taps t;
            bilinear_taps(ga[pi], gb[pi], sc.plane_w, sc.plane_h, t);
            float* base = maps.pl[pi] + (size_t)v * sc.plane_h * sc.plane_w * C;
            for (int q = threadIdx.x; q < C / 4; q += blockDim.x) {
                const float4 gv = g[q];
                for (int tp = 0; tp < 4; ++tp) {
                    const float w = t.w[tp];
                    if (w != 0.f) atomicAdd(reinterpret_cast<float4*>(base + (size_t)t.idx[tp] * C) + q, make_float4(gv.x * w, gv.y * w, gv.z * w, gv.w * w));
                }
            }
        }
    }
}

int launch_index_bwd(const NeoScene* sc, const float* pts, int M, int local, const float* g_out, float* g_lat, float* g_xz, float* g_xy,
                     float* g_yz, cudaStream_t s) {
    const int C = local ? kLocalCh : kWorldCh;
    index_bwd_kernel<<<(unsigned)((long long)sc->dev.nv * M), local ? 128 : 32, 0, s>>>(sc->dev, pts, M, local, C, g_out, MapSetW{g_lat, {g_xz, g_xy, g_yz}});
    NEO_LAUNCH_CHECK("index_bwd_kernel");
    return NEO_OK;
}

int launch_index_grid(const NeoScene* sc, const float* pts, int M, float* out, cudaStream_t s) {
    index_kernel<<<(unsigned)((long long)sc->dev.nv * M), 128, 0, s>>>(sc->dev, pts, M, 0, kWorldCh,
                                                                        MapSet{nullptr, {sc->dev.planes_cl[0], sc->dev.planes_cl[1], sc->dev.planes_cl[2]}}, out);
    NEO_LAUNCH_CHECK("index_kernel(grid)");
    return NEO_OK;
}
int launch_index_local(const NeoScene* sc, const float* pts, int M, float* out, cudaStream_t s) {
    index_kernel<<<(unsigned)((long long)sc->dev.nv * M), 128, 0, s>>>(sc->dev, pts, M, 1, kLocalCh, MapSet{sc->dev.latent_cl, {nullptr, nullptr, nullptr}}, out);
    NEO_LAUNCH_CHECK("index_kernel(local)");
    return NEO_OK;
}
// caller-owned maps (training on projected maps): lookups and their scatter-add backward with the scene's cameras / grid geometry
int launch_index_maps(const NeoScene* sc, const float* pts, int M, int C, const float* lat, const float* xz, const float* xy, const float* yz,
                      float* out_local, float* out_world, cudaStream_t s) {
    const unsigned grid = (unsigned)((long long)sc->dev.nv * M);
    const int threads = C >= 128 ? 128 : 64;
    if (lat) { index_kernel<<<grid, threads, 0, s>>>(sc->dev, pts, M, 1, C, MapSet{lat, {nullptr, nullptr, nullptr}}, out_local); NEO_LAUNCH_CHECK("index_kernel(maps, local)"); }
    if (xz) { index_kernel<<<grid, threads, 0, s>>>(sc->dev, pts, M, 0, C, MapSet{nullptr, {xz, xy, yz}}, out_world); NEO_LAUNCH_CHECK("index_kernel(maps, world)"); }
    return NEO_OK;
}
int launch_index_maps_bwd(const NeoScene* sc, const float* pts, int M, int C, const float* g_local, const float* g_world, float* g_lat, float* g_xz,
                          float* g_xy, float* g_yz, cudaStream_t s) {
    const unsigned grid = (unsigned)((long long)sc->dev.nv * M);
    const int threads = C / 4 >= 64 ? 64 : 32;
    if (g_local) { index_bwd_kernel<<<grid, threads, 0, s>>>(sc->dev, pts, M, 1, C, g_local, MapSetW{g_lat, {nullptr, nullptr, nullptr}}); NEO_LAUNCH_CHECK("index_bwd_kernel(maps, local)"); }
    if (g_world) { index_bwd_kernel<<<grid, threads, 0, s>>>(sc->dev, pts, M, 0, C, g_world, MapSetW{nullptr, {g_xz, g_xy, g_yz}}); NEO_LAUNCH_CHECK("index_bwd_kernel(maps, world)"); }
    return NEO_OK;
}

// ---- deterministic backward (csrc/det.cu): the entries of the scatter that index_bwd_kernel does with atomics ----
// Row r = v*M + m.  Local entries e = r*4 + tap, key = v*Hl*Wl + texel; world entries e = e0 + r*12 + plane*4 + tap,
// key = key0 + (plane*nv + v)*Hp*Wp + texel (planes xz, xy, yz).  A zero-weight tap gets the key `T` and is never reduced.
__global__ void index_entries_kernel(SceneDev sc, const float* __restrict__ pts, int M, int local, unsigned e0, unsigned key0, unsigned T,
                                     unsigned* __restrict__ keys, unsigned* __restrict__ ids, float* __restrict__ wts) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= (long long)sc.nv * M) return;
    const int v = (int)(r / M), m = (int)(r % M);
    float c[3];
    to_camera(sc.views[v], pts + 3 * (size_t)m, c);
    auto put = [&](unsigned e, unsigned key, float w) { keys[e] = w != 0.f ? key : T; ids[e] = e; wts[e] = w; };
    if (local) {
        float gx, gy;
        Taps t;
        local_grid_coords(sc, c, gx, gy);
        bilinear_taps(gx, gy, sc.lat_w, sc.lat_h, t);
        const unsigned base = key0 + (unsigned)v * sc.lat_h * sc.lat_w;
        for (int tp = 0; tp < 4; ++tp) put(e0 + (unsigned)r * 4 + tp, base + t.idx[tp], t.w[tp]);
    } else {
        const float ga[3] = {c[0], c[0], c[1]}, gb[3] = {c[2], c[1], c[2]};
        const unsigned hw = (unsigned)sc.plane_h * sc.plane_w;
        for (int pi = 0; pi < 3; ++pi) {
            Taps t;
            bilinear_taps(ga[pi], gb[pi], sc.plane_w, sc.plane_h, t);
            const unsigned base = key0 + ((unsigned)pi * sc.nv + v) * hw;
            for (int tp = 0; tp < 4; ++tp) put(e0 + (unsigned)r * 12 + pi * 4 + tp, base + t.idx[tp], t.w[tp]);
        }
    }
}

void index_det_sizes(const NeoScene* sc, int M, bool local, bool world, long long& E, long long& T) {
    const long long rows = (long long)sc->dev.nv * M;
    E = (local ? 4 * rows : 0) + (world ? 12 * rows : 0);
    T = (local ? (long long)sc->dev.nv * sc->dev.lat_h * sc->dev.lat_w : 0) + (world ? 3LL * sc->dev.nv * sc->dev.plane_h * sc->dev.plane_w : 0);
}

int launch_index_maps_bwd_det(const NeoScene* sc, const float* pts, int M, int C, const float* g_local, const float* g_world, float* g_lat,
                              float* g_xz, float* g_xy, float* g_yz, const DetBuffers& b, cudaStream_t s) {
    long long E, T;
    index_det_sizes(sc, M, g_local != nullptr, g_world != nullptr, E, T);
    const long long rows = (long long)sc->dev.nv * M;
    const unsigned grid = (unsigned)((rows + 127) / 128);
    const long long T_lat = g_local ? (long long)sc->dev.nv * sc->dev.lat_h * sc->dev.lat_w : 0;
    const unsigned e_world = g_local ? (unsigned)(4 * rows) : 0u;
    if (g_local) {
        index_entries_kernel<<<grid, 128, 0, s>>>(sc->dev, pts, M, 1, 0u, 0u, (unsigned)T, b.keys, b.ids, b.wts);
        NEO_LAUNCH_CHECK("index_entries_kernel(local)");
    }
    if (g_world) {
        index_entries_kernel<<<grid, 128, 0, s>>>(sc->dev, pts, M, 0, e_world, (unsigned)T_lat, (unsigned)T, b.keys, b.ids, b.wts);
        NEO_LAUNCH_CHECK("index_entries_kernel(world)");
    }
    const long long hw = (long long)sc->dev.nv * sc->dev.plane_h * sc->dev.plane_w;
    DetSrc src{{g_local ? g_local : g_world, g_world}, {C, C}, {0u, g_local && g_world ? e_world : 0xffffffffu}, {g_local ? 4 : 12, 12}};
    DetDst dst{{g_local ? g_lat : g_xz, g_xz, g_xy, g_yz}, {0, T_lat, T_lat + hw, T_lat + 2 * hw}};
    if (!g_local) dst = DetDst{{g_xz, g_xy, g_yz, g_yz}, {0, hw, 2 * hw, 3 * hw}};
    else if (!g_world) dst = DetDst{{g_lat, g_lat, g_lat, g_lat}, {0, T, T, T}};
    return det_sort_reduce(b, E, T, C, 4, src, dst, s);
}

}  // namespace neo
