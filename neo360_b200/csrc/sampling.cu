// HBM-bound per-ray kernels of the NeO-360 hot path: ray generation, sphere intersection, stratified sampling,
// inverse-CDF resampling (+merge), alpha compositing, fg/bg combine.
// Reference: datasets/ray_utils.py:84-176, models/neo360/helper.py:24-75,128-273,401-450, model.py:521-579.
#include "common.cuh"

namespace neo {

// ------------------------------------------------------------------------------------------------
// a1/a2  get_ray_directions + get_rays   (ray_utils.py:84-104,133-176)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void raw_dir(int i, int j, int H, int W, float focal, const float* c2w, float* d) {
    // directions = ((i - W/2)/f, -(j - H/2)/f, -1);  rays_d = directions @ c2w[:, :3].T
    float c[3] = {__fdiv_rn(sub_((float)i, (float)W / 2.f), focal), -__fdiv_rn(sub_((float)j, (float)H / 2.f), focal),
                  -1.0f};
    for (int r = 0; r < 3; ++r) d[r] = fmaf(c[2], c2w[r * 4 + 2], fmaf(c[1], c2w[r * 4 + 1], c[0] * c2w[r * 4 + 0]));
}

// One pixel (i, j) of one view -> ray slot q.  Shared by the whole-frame and the sampled-pixel kernels so both give the same bits.
__device__ __forceinline__ void ray_at(int i, int j, int H, int W, float focal, const float* m, size_t q, float* __restrict__ o,
                                       float* __restrict__ vd, float* __restrict__ rd, float* __restrict__ radii) {
    float d[3];
    raw_dir(i, j, H, W, focal, m, d);
    if (radii) {
        // dx between image rows j and j+1 (last row copies row H-2), * 2/sqrt(12)   (ray_utils.py:153-160)
        int ja = (j < H - 1) ? j : H - 2;
        float a[3], b[3];
        raw_dir(i, ja, H, W, focal, m, a);
        raw_dir(i, ja + 1, H, W, focal, m, b);
        float e[3] = {sub_(a[0], b[0]), sub_(a[1], b[1]), sub_(a[2], b[2])};
        float dx = __fsqrt_rn(dot3_(e, e));
        radii[q] = __fdiv_rn(mul_(dx, 2.0f), __fsqrt_rn(12.0f));
    }
    float n = __fsqrt_rn(dot3_(d, d));
    for (int r = 0; r < 3; ++r) {
        float v = __fdiv_rn(d[r], n);   // quirk Q3: rays_d is normalised in place through the viewdirs alias
        if (vd) vd[q * 3 + r] = v;
        if (rd) rd[q * 3 + r] = v;
        if (o) o[q * 3 + r] = m[r * 4 + 3];
    }
}

__global__ void get_rays_kernel(int H, int W, float focal, const float* __restrict__ c2w, float* __restrict__ o,
                                float* __restrict__ vd, float* __restrict__ rd, float* __restrict__ radii) {
    int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= H * W) return;
    float m[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) m[k] = c2w[k];
    ray_at(p % W, p / W, H, W, focal, m, (size_t)p, o, vd, rd, radii);
}

int launch_get_rays(int H, int W, float focal, const float* c2w, float* o, float* vd, float* rd, float* radii,
                    cudaStream_t s) {
    int n = H * W;
    get_rays_kernel<<<(n + 255) / 256, 256, 0, s>>>(H, W, focal, c2w, o, vd, rd, radii);
    NEO_LAUNCH_CHECK("get_rays_kernel");
    return NEO_OK;
}

// f3  training-batch pixel sampling (nerds360_ae.py:730-748): the reference builds all T x H x W rays of the target views on the
// host and keeps `n` of them by `pix_inds`; here only the kept rays are ever computed.  pix indexes the flattened (T, H, W) stack.
__global__ void sample_rays_kernel(int n, const long long* __restrict__ pix, int T, int H, int W, float focal,
                                   const float* __restrict__ c2w, const float* __restrict__ images, float* __restrict__ o,
                                   float* __restrict__ vd, float* __restrict__ rd, float* __restrict__ radii,
                                   float* __restrict__ target, int* __restrict__ err) {
    int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n) return;
    long long p = pix[q];
    if (p < 0 || p >= (long long)T * H * W) { atomicExch(err, NEO_ERR_INVALID); return; }
    int t = (int)(p / ((long long)H * W)), r = (int)(p % ((long long)H * W));
    float m[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) m[k] = c2w[t * 12 + k];
    ray_at(r % W, r / W, H, W, focal, m, (size_t)q, o, vd, rd, radii);
    if (target && images)
        for (int c = 0; c < 3; ++c) target[(size_t)q * 3 + c] = images[(size_t)p * 3 + c];
}

int launch_sample_rays(int n, const long long* pix, int T, int H, int W, float focal, const float* c2w, const float* images,
                       float* o, float* vd, float* rd, float* radii, float* target, int* err, cudaStream_t s) {
    if (n == 0) return NEO_OK;
    sample_rays_kernel<<<(n + 255) / 256, 256, 0, s>>>(n, pix, T, H, W, focal, c2w, images, o, vd, rd, radii, target, err);
    NEO_LAUNCH_CHECK("sample_rays_kernel");
    return NEO_OK;
}

// ------------------------------------------------------------------------------------------------
// a3  intersect_sphere   (helper.py:253-273)
// ------------------------------------------------------------------------------------------------
__global__ void far_kernel(const float* __restrict__ o, const float* __restrict__ d, int n, float* __restrict__ far,
                           int* __restrict__ err) {
    int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n) return;
    RayGeom g;
    ray_geom(o + 3 * b, d + 3 * b, g, false);
    far[b] = g.far;
    if (!(g.check >= 0.f) && err) atomicExch(err, 1);   // the reference asserts here (helper.py:271)
}

int launch_far(const float* o, const float* d, int n, float* far, int* err, cudaStream_t s) {
    far_kernel<<<(n + 255) / 256, 256, 0, s>>>(o, d, n, far, err);
    NEO_LAUNCH_CHECK("far_kernel");
    return NEO_OK;
}

// ------------------------------------------------------------------------------------------------
// a4  sample_along_rays   (helper.py:24-75)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float coarse_param(int k, int steps, bool in_sphere, float near, float far) {
    float u = linspace01(k, steps);
    return in_sphere ? add_(mul_(near, sub_(1.0f, u)), mul_(far, u)) : u;
}

__global__ void sample_coarse_kernel(const float* __restrict__ o, const float* __restrict__ d,
                                     const float* __restrict__ far, int n, int ns, int in_sphere, float far_unc,
                                     const float* __restrict__ u_rand, float* __restrict__ t_out,
                                     float* __restrict__ pts, float* __restrict__ pts_lin) {
    int steps = ns + 1;
    long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (long long)n * steps) return;
    int b = (int)(gid / steps), i = (int)(gid % steps);
    // output index i; for the bg branch the arrays are stored flipped (s: 1 -> 0), so the source index is ns - i
    int k = in_sphere ? i : ns - i;
    float fr = far[b];
    const float near = 1e-4f;   // quirk Q4 (model.py:277)
    float t = coarse_param(k, steps, in_sphere, near, fr);
    if (u_rand) {
        float tm = (k > 0) ? coarse_param(k - 1, steps, in_sphere, near, fr) : t;
        float tp = (k < ns) ? coarse_param(k + 1, steps, in_sphere, near, fr) : t;
        float lower = (k > 0) ? mul_(0.5f, add_(t, tm)) : t;
        float upper = (k < ns) ? mul_(0.5f, add_(tp, t)) : t;
        t = add_(lower, mul_(sub_(upper, lower), u_rand[(long long)b * steps + k]));
    }
    t_out[(long long)b * steps + i] = t;
    if (pts || pts_lin) {
        RayGeom g;
        ray_geom(o + 3 * b, d + 3 * b, g, !in_sphere);
        if (in_sphere) {
            float x[3];
            fg_point(g, t, x);
            for (int c = 0; c < 3; ++c) pts[((long long)b * steps + i) * 3 + c] = x[c];
        } else {
            float xh[3], lin[3];
            bg_point(g, t, far_unc, xh, lin);
            if (pts) {
                float* p = pts + ((long long)b * steps + i) * 4;
                p[0] = xh[0]; p[1] = xh[1]; p[2] = xh[2]; p[3] = t;
            }
            if (pts_lin)
                for (int c = 0; c < 3; ++c) pts_lin[((long long)b * steps + i) * 3 + c] = lin[c];
        }
    }
}

int launch_sample_coarse(const float* o, const float* d, const float* far, int n, int num_samples, int in_sphere,
                         float far_unc, const float* u_rand, float* t, float* pts, float* pts_lin, cudaStream_t s) {
    long long total = (long long)n * (num_samples + 1);
    sample_coarse_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(o, d, far, n, num_samples, in_sphere, far_unc,
                                                                       u_rand, t, pts, pts_lin);
    NEO_LAUNCH_CHECK("sample_coarse_kernel");
    return NEO_OK;
}

// ------------------------------------------------------------------------------------------------
// a14/a15  sorted_piecewise_constant_pdf + sample_pdf   (helper.py:174-249)
// One warp per ray.  Shared memory per warp: bins[K] cdf[K] pmax[K] smin[K] sort[P2]  (K = n_old-1).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_incl_scan_add(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        float n = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v = add_(v, n);
    }
    return v;
}

__global__ void resample_kernel(const float* __restrict__ o, const float* __restrict__ d,
                                const float* __restrict__ far, const float* __restrict__ t_old,
                                const float* __restrict__ w, int n, int n_old, int m, int in_sphere, float far_unc,
                                const float* __restrict__ u_rand, float* __restrict__ t_out, float* __restrict__ pts,
                                float* __restrict__ pts_lin, int p2) {
    extern __shared__ float sm[];
    const int warps = blockDim.x / 32, wid = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int K = n_old - 1;              // number of bins (= mids)
    const int per_warp = 4 * K + p2;
    float* bins = sm + wid * per_warp;
    float* cdf = bins + K;
    float* pmax = cdf + K;
    float* smin = pmax + K;
    float* srt = smin + K;
    int b = blockIdx.x * warps + wid;
    if (b >= n) return;                    // whole warp exits together
    const float* tb = t_old + (long long)b * n_old;
    const float* wb = w + (long long)b * n_old;
    const int nw = K - 1;                  // weights[..., 1:-1]

    // bins = 0.5 * (t[1:] + t[:-1]);   weight sum
    float part = 0.f;
    for (int j = lane; j < K; j += 32) bins[j] = mul_(0.5f, add_(tb[j + 1], tb[j]));
    for (int j = lane; j < nw; j += 32) part += wb[j + 1];
    float wsum = warp_sum(part);
    float pad = fmaxf(0.f, sub_(1e-5f, wsum));
    float padw = __fdiv_rn(pad, (float)nw);
    wsum = add_(wsum, pad);
    // cdf = [0, min(1, cumsum(pdf[:-1])), 1]   (K entries)
    float carry = 0.f;
    for (int base = 0; base < nw - 1; base += 32) {
        int j = base + lane;
        float pdf = (j < nw - 1) ? __fdiv_rn(add_(wb[j + 1], padw), wsum) : 0.f;
        float sc = add_(warp_incl_scan_add(pdf, lane), carry);
        // note: the carry is added after the in-warp scan; fp32 association differs from a sequential cumsum by <= a few ulp
        if (j < nw - 1) cdf[j + 1] = fminf(1.0f, sc);
        carry = __shfl_sync(0xffffffffu, sc, 31);
    }
    if (lane == 0) { cdf[0] = 0.f; cdf[K - 1] = 1.0f; }
    __syncwarp();
    // prefix max / suffix min of bins by VALUE (mask max/min semantics, quirk Q17)
    {
        float run = -INFINITY;
        for (int base = 0; base < K; base += 32) {
            int j = base + lane;
            float v = (j < K) ? bins[j] : -INFINITY;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                float nb = __shfl_up_sync(0xffffffffu, v, o);
                if (lane >= o) v = fmaxf(v, nb);
            }
            v = fmaxf(v, run);
            if (j < K) pmax[j] = v;
            run = __shfl_sync(0xffffffffu, v, 31);
        }
        run = INFINITY;
        for (int base = 0; base < K; base += 32) {
            int j = K - 1 - (base + lane);
            float v = (j >= 0) ? bins[j] : INFINITY;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                float nb = __shfl_up_sync(0xffffffffu, v, o);
                if (lane >= o) v = fminf(v, nb);
            }
            v = fminf(v, run);
            if (j >= 0) smin[j] = v;
            run = __shfl_sync(0xffffffffu, v, 31);
        }
    }
    __syncwarp();
    // sort buffer: old values then new samples, padded with +inf
    for (int j = lane; j < p2; j += 32) srt[j] = (j < n_old) ? tb[j] : INFINITY;
    __syncwarp();   // lane j % 32 pads srt[j] and lane q % 32 writes srt[n_old + q]: the padding must land first
    for (int q = lane; q < m; q += 32) {
        float u = u_rand ? u_rand[(long long)b * m + q] : linspace01(q, m);   // linspace(0, 1-2^-32, m): end == 1.0f (Q7)
        // a j with cdf[j] <= u < cdf[j+1] (the last such j while the fp32 cdf is non-decreasing; where two lanes rounded a zero-weight
        // bin differently it can step back one ulp, and the search then returns one valid bracket of the several)
        int lo = 0, hi = K;               // invariant: cdf[lo] <= u, (hi == K or cdf[hi] > u)
        while (hi - lo > 1) {
            int mid = (lo + hi) >> 1;
            if (cdf[mid] <= u) lo = mid; else hi = mid;
        }
        float c0 = cdf[lo];
        float c1 = (lo + 1 < K) ? cdf[lo + 1] : cdf[K - 1];
        float b0 = pmax[lo];
        float b1 = (lo + 1 < K) ? smin[lo + 1] : bins[K - 1];
        float tau = __fdiv_rn(sub_(u, c0), sub_(c1, c0));
        if (tau != tau) tau = 0.f;        // nan_to_num(., 0)
        tau = fminf(fmaxf(tau, 0.f), 1.f);
        srt[n_old + q] = add_(b0, mul_(tau, sub_(b1, b0)));
    }
    __syncwarp();
    // bitonic sort ascending over p2 elements
    for (int k2 = 2; k2 <= p2; k2 <<= 1) {
        for (int j2 = k2 >> 1; j2 > 0; j2 >>= 1) {
            for (int i = lane; i < p2; i += 32) {
                int l = i ^ j2;
                if (l > i) {
                    float a = srt[i], c = srt[l];
                    bool up = ((i & k2) == 0);
                    if ((a > c) == up) { srt[i] = c; srt[l] = a; }
                }
            }
            __syncwarp();
        }
    }
    const int N1 = n_old + m;
    RayGeom g;
    if (pts || pts_lin) ray_geom(o + 3 * b, d + 3 * b, g, !in_sphere);
    for (int i = lane; i < N1; i += 32) {
        float v = in_sphere ? srt[i] : srt[N1 - 1 - i];   // bg: flipped to descending (helper.py:234-239)
        t_out[(long long)b * N1 + i] = v;
        if (in_sphere) {
            if (pts) {
                float x[3];
                fg_point(g, v, x);
                for (int c = 0; c < 3; ++c) pts[((long long)b * N1 + i) * 3 + c] = x[c];
            }
        } else if (pts || pts_lin) {
            float xh[3], lin[3];
            bg_point(g, v, far_unc, xh, lin);
            if (pts) {
                float* p = pts + ((long long)b * N1 + i) * 4;
                p[0] = xh[0]; p[1] = xh[1]; p[2] = xh[2]; p[3] = v;
            }
            if (pts_lin)
                for (int c = 0; c < 3; ++c) pts_lin[((long long)b * N1 + i) * 3 + c] = lin[c];
        }
    }
}

int launch_resample(const float* o, const float* d, const float* far, const float* t_old, const float* w, int n,
                    int n_old, int m, int in_sphere, float far_unc, const float* u_rand, float* t, float* pts,
                    float* pts_lin, cudaStream_t s) {
    if (n_old < 4 || m < 1) { set_error("sample_pdf needs n_old >= 4 and num_samples >= 1"); return NEO_ERR_INVALID; }
    int p2 = 1;
    while (p2 < n_old + m) p2 <<= 1;
    int K = n_old - 1;
    const int warps = 4;
    size_t smem = (size_t)warps * (4 * K + p2) * sizeof(float);
    if (smem > 200 * 1024) { set_error("sample_pdf: too many samples per ray (%d+%d)", n_old, m); return NEO_ERR_UNSUPPORTED; }
    if (smem > 48 * 1024)
        NEO_CUDA(cudaFuncSetAttribute(resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    resample_kernel<<<(n + warps - 1) / warps, warps * 32, smem, s>>>(o, d, far, t_old, w, n, n_old, m, in_sphere,
                                                                     far_unc, u_rand, t, pts, pts_lin, p2);
    NEO_LAUNCH_CHECK("resample_kernel");
    return NEO_OK;
}

// ------------------------------------------------------------------------------------------------
// a12  volumetric_rendering   (helper.py:128-171).  One warp per ray, multiplicative warp scan.
// ------------------------------------------------------------------------------------------------
__global__ void composite_kernel(const float* __restrict__ rgb, const float* __restrict__ sigma,
                                 const float* __restrict__ t, const float* __restrict__ d,
                                 const float* __restrict__ far, int n, int N, int white, int in_sphere,
                                 float* __restrict__ comp, float* __restrict__ acc_out, float* __restrict__ w_out,
                                 float* __restrict__ lam_out, float* __restrict__ depth_out) {
    const int warps = blockDim.x / 32, wid = threadIdx.x / 32, lane = threadIdx.x % 32;
    int b = blockIdx.x * warps + wid;
    if (b >= n) return;
    const float* tb = t + (long long)b * N;
    const float* sb = sigma + (long long)b * N;
    const float* cb = rgb + (long long)b * N * 3;
    // in_sphere: 1 = NeO-360 fg (last interval far - t_N, |d| scale), 0 = NeO-360 bg (descending s, last 1e10),
    //            2 = vanilla NeRF (ascending t, last 1e10, |d| scale, depth nan_to_num)   vanilla_nerf/helper.py:521-559
    float dn = 1.f, fr = 0.f;
    if (in_sphere) {
        const float* dd = d + 3 * b;
        dn = __fsqrt_rn(dot3_(dd, dd));
        if (in_sphere == 1) fr = far[b];
    }
    float carry = 1.f;      // T of everything before this 32-sample block
    float acc = 0.f, r = 0.f, gch = 0.f, bch = 0.f, dep = 0.f;
    for (int base = 0; base < N; base += 32) {
        int k = base + lane;
        bool ok = k < N;
        float tk = ok ? tb[k] : 0.f;
        float dist;
        if (in_sphere == 1) {
            float nxt = (k + 1 < N) ? tb[min(k + 1, N - 1)] : fr;
            dist = mul_(sub_(nxt, tk), dn);
        } else if (in_sphere == 2) {
            dist = mul_((k + 1 < N) ? sub_(tb[min(k + 1, N - 1)], tk) : 1e10f, dn);
        } else {
            dist = (k + 1 < N) ? sub_(tk, tb[min(k + 1, N - 1)]) : 1e10f;
        }
        float alpha = ok ? sub_(1.0f, expf(-mul_(sb[k], dist))) : 0.f;
        float f = ok ? add_(sub_(1.0f, alpha), 1e-10f) : 1.f;      // quirk Q9: eps inside the product
        float sc = f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            float nb = __shfl_up_sync(0xffffffffu, sc, o);
            if (lane >= o) sc = mul_(sc, nb);
        }
        float incl = mul_(carry, sc);
        float excl = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) excl = carry;
        float wk = mul_(alpha, excl);
        if (ok) {
            if (w_out) w_out[(long long)b * N + k] = wk;
            acc += wk;
            r += wk * cb[k * 3 + 0];
            gch += wk * cb[k * 3 + 1];
            bch += wk * cb[k * 3 + 2];
            dep += wk * tk;
        }
        carry = __shfl_sync(0xffffffffu, incl, 31);
    }
    acc = warp_sum(acc); r = warp_sum(r); gch = warp_sum(gch); bch = warp_sum(bch); dep = warp_sum(dep);
    if (lane == 0) {
        if (white) { float bgc = sub_(1.0f, acc); r += bgc; gch += bgc; bch += bgc; }
        if (comp) { comp[b * 3 + 0] = r; comp[b * 3 + 1] = gch; comp[b * 3 + 2] = bch; }
        if (acc_out) acc_out[b] = acc;
        if (lam_out) lam_out[b] = carry;     // T[..., -1]
        if (in_sphere == 2 && dep != dep) dep = INFINITY;      // torch.nan_to_num(depth, inf), quirk Q10
        if (depth_out) depth_out[b] = dep;
    }
}

int launch_composite(const float* rgb, const float* sigma, const float* t, const float* d, const float* far, int n,
                     int N, int white, int in_sphere, float* comp, float* acc, float* w, float* lam, float* depth,
                     cudaStream_t s) {
    const int warps = 8;
    composite_kernel<<<(n + warps - 1) / warps, warps * 32, 0, s>>>(rgb, sigma, t, d, far, n, N, white, in_sphere, comp,
                                                                   acc, w, lam, depth);
    NEO_LAUNCH_CHECK("composite_kernel");
    return NEO_OK;
}


// ------------------------------------------------------------------------------------------------
// backward of a12 (volumetric_rendering, helper.py:128-171) w.r.t. the per-sample rgb and sigma (t is detached in the reference:
// sample positions carry no gradient, helper.py:225).  One thread per ray, two sequential passes over its N samples:
//   forward  : T_i = prod_{j<i} (1 - alpha_j + 1e-10)                       (kept in the d_sigma row as scratch)
//   backward : G_i = g_comp.c_i + g_w_i + g_acc + g_depth t_i - white * sum(g_comp)        (dL/dw_i)
//              S_i = sum_{j>i} G_j w_j + g_lam T_N                                          (everything downstream of factor a_i)
//              dL/dalpha_i = G_i T_i - S_i / a_i ,   dL/dsigma_i = dL/dalpha_i * delta_i (1 - alpha_i) ,   dL/dc_i = w_i g_comp
// in_sphere 2 (vanilla NeRF, entry point neo_vanilla_composite_bwd): ascending t, last interval 1e10, every interval times |d|, no far and
// no g_lam; the forward's depth is nan_to_num(sum w t, inf) clamped to its own chunk-wide min / max (quirk Q10), whose gradient passes
// where sum w t is finite and is zero where it was substituted.
// ------------------------------------------------------------------------------------------------
__global__ void composite_bwd_kernel(const float* __restrict__ rgb, const float* __restrict__ sigma, const float* __restrict__ t,
                                     const float* __restrict__ d, const float* __restrict__ far, int n, int N, int white, int in_sphere,
                                     const float* __restrict__ g_comp, const float* __restrict__ g_acc, const float* __restrict__ g_w,
                                     const float* __restrict__ g_lam, const float* __restrict__ g_depth,
                                     float* __restrict__ d_rgb, float* __restrict__ d_sigma) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n) return;
    const float* tb = t + (long long)b * N;
    const float* sb = sigma + (long long)b * N;
    const float* cb = rgb + (long long)b * N * 3;
    float* ds = d_sigma + (long long)b * N;
    float* dc = d_rgb + (long long)b * N * 3;
    float dn = 1.f, fr = 0.f;
    if (in_sphere) {
        const float* dd = d + 3 * b;
        dn = __fsqrt_rn(dot3_(dd, dd));
        if (in_sphere == 1) fr = far[b];
    }
    auto dist_of = [&](int k) -> float {
        if (in_sphere == 1) return mul_(sub_((k + 1 < N) ? tb[k + 1] : fr, tb[k]), dn);
        if (in_sphere == 2) return mul_((k + 1 < N) ? sub_(tb[k + 1], tb[k]) : 1e10f, dn);
        return (k + 1 < N) ? sub_(tb[k], tb[k + 1]) : 1e10f;
    };
    float T = 1.f, dep = 0.f;
    for (int k = 0; k < N; ++k) {
        ds[k] = T;
        const float alpha = sub_(1.0f, expf(-mul_(sb[k], dist_of(k))));
        if (in_sphere == 2) dep += alpha * T * tb[k];
        T = mul_(T, add_(sub_(1.0f, alpha), 1e-10f));
    }
    const float gc[3] = {g_comp ? g_comp[b * 3] : 0.f, g_comp ? g_comp[b * 3 + 1] : 0.f, g_comp ? g_comp[b * 3 + 2] : 0.f};
    const float ga = (g_acc ? g_acc[b] : 0.f) - (white ? (gc[0] + gc[1] + gc[2]) : 0.f);
    const float gd = (g_depth && (in_sphere != 2 || isfinite(dep))) ? g_depth[b] : 0.f;
    float S = (g_lam ? g_lam[b] : 0.f) * T;
    for (int k = N - 1; k >= 0; --k) {
        const float Tk = ds[k];
        const float dist = dist_of(k);
        const float e = expf(-mul_(sb[k], dist));
        const float alpha = sub_(1.0f, e);
        const float a = add_(sub_(1.0f, alpha), 1e-10f);
        const float w = alpha * Tk;
        const float G = gc[0] * cb[3 * k] + gc[1] * cb[3 * k + 1] + gc[2] * cb[3 * k + 2] + (g_w ? g_w[(long long)b * N + k] : 0.f) + ga + gd * tb[k];
        const float dalpha = G * Tk - S / a;
        ds[k] = dalpha * dist * e;            // d alpha / d sigma = delta exp(-sigma delta)
        dc[3 * k] = w * gc[0]; dc[3 * k + 1] = w * gc[1]; dc[3 * k + 2] = w * gc[2];
        S += G * w;
    }
}

int launch_composite_bwd(const float* rgb, const float* sigma, const float* t, const float* d, const float* far, int n, int N, int white,
                         int in_sphere, const float* g_comp, const float* g_acc, const float* g_w, const float* g_lam, const float* g_depth,
                         float* d_rgb, float* d_sigma, cudaStream_t s) {
    composite_bwd_kernel<<<(n + 127) / 128, 128, 0, s>>>(rgb, sigma, t, d, far, n, N, white, in_sphere, g_comp, g_acc, g_w, g_lam, g_depth,
                                                         d_rgb, d_sigma);
    NEO_LAUNCH_CHECK("composite_bwd_kernel");
    return NEO_OK;
}

// ------------------------------------------------------------------------------------------------
// a13  fg + bg_lambda * bg, sdist outputs   (model.py:521-527, 564-579)
// ------------------------------------------------------------------------------------------------
__global__ void combine_kernel(int n, int N, const float* __restrict__ fg_c, const float* __restrict__ bg_c,
                               const float* __restrict__ lam, const float* __restrict__ fg_depth,
                               const float* __restrict__ bg_depth, const float* __restrict__ fg_t,
                               const float* __restrict__ bg_s, float* __restrict__ comp, float* __restrict__ depth,
                               float* __restrict__ fg_sdist, float* __restrict__ bg_sdist) {
    long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid < n) {
        int b = (int)gid;
        float l = lam[b];
        if (comp)
            for (int c = 0; c < 3; ++c) comp[b * 3 + c] = add_(fg_c[b * 3 + c], mul_(l, bg_c[b * 3 + c]));
        if (depth) depth[b] = add_(fg_depth[b], mul_(l, bg_depth[b]));   // quirk Q8
    }
    if (gid < (long long)n * N && (fg_sdist || bg_sdist)) {
        int b = (int)(gid / N), k = (int)(gid % N);
        if (fg_sdist) {
            const float* tb = fg_t + (long long)b * N;
            float v;
            if (k < N - 1) v = mul_(0.5f, add_(tb[k + 1], tb[k]));
            else {
                float m1 = mul_(0.5f, add_(tb[N - 1], tb[N - 2])), m2 = mul_(0.5f, add_(tb[N - 2], tb[N - 3]));
                v = add_(m1, sub_(m1, m2));
            }
            fg_sdist[gid] = v;
        }
        if (bg_sdist) {
            const float* sb = bg_s + (long long)b * N;
            bg_sdist[gid] = (k < N - 1) ? mul_(0.5f, add_(sb[k + 1], sb[k])) : sb[N - 1];
        }
    }
}

int launch_combine(int n, int N, const float* fg_c, const float* bg_c, const float* lam, const float* fg_depth,
                   const float* bg_depth, const float* fg_t, const float* bg_s, float* comp, float* depth,
                   float* fg_sdist, float* bg_sdist, cudaStream_t s) {
    long long total = (fg_sdist || bg_sdist) ? (long long)n * N : n;
    combine_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(n, N, fg_c, bg_c, lam, fg_depth, bg_depth, fg_t, bg_s,
                                                                 comp, depth, fg_sdist, bg_sdist);
    NEO_LAUNCH_CHECK("combine_kernel");
    return NEO_OK;
}


// ------------------------------------------------------------------------------------------------
// output side (SURVEY.md 8(f4)): sum of squared differences of two images after clipping to [0,1] -- the reduction under
// LitModel.psnr_each (models/interface.py:53-61).  Grid-stride, warp + block reduction, one double atomicAdd per block.
// MASKED: the object PSNR of get_obj_rgbs_from_segmap (models/utils.py:102-109): only the values of pixels whose mask byte is non-zero
// (mask has one byte per pixel, the values are (pixel, 3) channel-last) enter the sum, and *count receives their number.
// ------------------------------------------------------------------------------------------------
template <bool MASKED>
__global__ void clipped_sq_err_kernel(const float* __restrict__ a, const float* __restrict__ b, const unsigned char* __restrict__ mask,
                                      long long n, double* __restrict__ out, unsigned long long* __restrict__ count) {
    double acc = 0.0;
    unsigned long long cnt = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        if (MASKED) {
            if (!mask[i / 3]) continue;
            ++cnt;
        }
        const float x = fminf(fmaxf(a[i], 0.f), 1.f) - fminf(fmaxf(b[i], 0.f), 1.f);
        acc += (double)(x * x);
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    __shared__ double red[8];
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    if (MASKED) {
        for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        __shared__ unsigned long long red_cnt[8];
        if ((threadIdx.x & 31) == 0) red_cnt[threadIdx.x >> 5] = cnt;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long c = 0;
            for (int w = 0; w < (int)(blockDim.x >> 5); ++w) c += red_cnt[w];
            atomicAdd(count, c);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
        atomicAdd(out, t);
    }
}
int launch_clipped_sq_err(const float* a, const float* b, const unsigned char* mask, long long n, double* out, unsigned long long* count,
                          cudaStream_t s) {
    NEO_CUDA(cudaMemsetAsync(out, 0, sizeof(double), s));
    if (mask) NEO_CUDA(cudaMemsetAsync(count, 0, sizeof(unsigned long long), s));
    const int blocks = (int)((n + 255) / 256 < 592 ? (n + 255) / 256 : 592);
    if (mask)
        clipped_sq_err_kernel<true><<<blocks > 0 ? blocks : 1, 256, 0, s>>>(a, b, mask, n, out, count);
    else
        clipped_sq_err_kernel<false><<<blocks > 0 ? blocks : 1, 256, 0, s>>>(a, b, nullptr, n, out, nullptr);
    NEO_LAUNCH_CHECK("clipped_sq_err_kernel");
    return NEO_OK;
}

}  // namespace neo
