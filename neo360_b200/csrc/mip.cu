// Mip-NeRF 360 renderer of the reference (SURVEY.md section 8(a) row a18 / Appendix A.6), fp32 CUDA cores, reference formulation.
// Reference: models/mipnerf360/model.py:30-365; models/mipnerf360/helper.py: max_dilate_weights 152-192, sample_intervals 343-396
// (sorted_interp 207-222), construct_ray_warps 168-172, cast_rays / conical_frustum_to_gaussian / lift_gaussian 278-339,
// contract 33-66 (closed-form Jacobian instead of functorch.jacrev), lift_and_diagonalize 70-73, integrated_pos_enc 77-88,
// compute_alpha_weights 234-260, volumetric_rendering 264-274.
// Structure per level: resample (warp per ray) -> IPE features (warp per sample) -> MLP as a chain of tiled SGEMMs with fused
// bias/ReLU/concat -> compositing (warp per ray).  This is the validation-grade path for this row (no tensor cores yet).
#include "common.cuh"
#include <cuda_fp16.h>

namespace neo {
namespace mip {

constexpr float kEps = 1.1920929e-07f;
constexpr int kFeat = 504, kBasis = 21, kDeg = 12;

// ------------------------------------------------------------------------------------------------
// proposal resampling: dilation + annealed softmax + inverse CDF at interval centres  (one warp per ray)
// shared per warp: t[3n+1 -> P2] | lo[n] | hi[n] | p[n] | wd[P2] | cw[P2]
// ------------------------------------------------------------------------------------------------
__global__ void resample_kernel(const float* __restrict__ s_prev, const float* __restrict__ w_prev, int n_rays, int n_prev, int level,
                                float dilation, float anneal, int n_new, float near, float far, const float* __restrict__ jitter,
                                float* __restrict__ s_out, float* __restrict__ t_out, int p2) {
    extern __shared__ float sm[];
    const int warps = blockDim.x / 32, wid = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int per_warp = 3 * p2 + 3 * n_prev;
    float* td = sm + wid * per_warp;       // sorted dilated positions (p2)
    float* wd = td + p2;                   // dilated weights / pdf (p2)
    float* cw = wd + p2;                   // cdf (p2)
    float* lo = cw + p2;                   // t0_j (n_prev)
    float* hi = lo + n_prev;               // t1_j
    float* pp = hi + n_prev;               // p_j
    const int b = blockIdx.x * warps + wid;
    if (b >= n_rays) return;
    int ns, nw;                            // entries of the (dilated) step function: ns positions, nw = ns-1 weights
    if (level == 0) {
        if (lane == 0) { td[0] = 0.f; td[1] = 1.f; wd[0] = 1.f; }
        ns = 2; nw = 1;
        __syncwarp();
    } else {
        const float* t = s_prev + (size_t)b * (n_prev + 1);
        const float* w = w_prev + (size_t)b * n_prev;
        for (int j = lane; j < n_prev; j += 32) {
            const float a = t[j], c = t[j + 1];
            pp[j] = __fdiv_rn(w[j], fmaxf(sub_(c, a), kEps));          // weight_to_pdf
            lo[j] = sub_(a, dilation);
            hi[j] = add_(c, dilation);
        }
        const int total = 3 * n_prev + 1;
        for (int i = lane; i < p2; i += 32) {
            float v = INFINITY;
            if (i <= n_prev) v = t[i];
            else if (i < 2 * n_prev + 1) v = sub_(t[i - n_prev - 1], dilation);
            else if (i < total) v = add_(t[i - 2 * n_prev], dilation);
            td[i] = v;
        }
        __syncwarp();
        for (int k2 = 2; k2 <= p2; k2 <<= 1)
            for (int j2 = k2 >> 1; j2 > 0; j2 >>= 1) {
                for (int i = lane; i < p2; i += 32) {
                    int l = i ^ j2;
                    if (l > i) {
                        float a = td[i], c = td[l];
                        bool up = ((i & k2) == 0);
                        if ((a > c) == up) { td[i] = c; td[l] = a; }
                    }
                }
                __syncwarp();
            }
        for (int i = lane; i < total; i += 32) td[i] = fminf(fmaxf(td[i], 0.f), 1.f);       // clip to the domain (0,1)
        __syncwarp();
        // p_dilate_i = max_j { p_j : t0_j <= td_i < t1_j }, weights = p * dt, renormalise
        float part = 0.f;
        for (int i = lane; i < total - 1; i += 32) {
            const float x = td[i];
            float m = 0.f;
            for (int j = 0; j < n_prev; ++j)
                if (lo[j] <= x && hi[j] > x) m = fmaxf(m, pp[j]);
            const float wv = mul_(m, sub_(td[i + 1], x));
            wd[i] = wv;
            part += wv;
        }
        const float tot = fmaxf(warp_sum(part), kEps);
        __syncwarp();
        // drop first/last: positions td[1..total-2], weights wd[1..total-3]
        ns = total - 2; nw = total - 3;
        for (int i = lane; i < nw; i += 32) cw[i] = __fdiv_rn(wd[i + 1], tot);
        __syncwarp();
        for (int i = lane; i < nw; i += 32) wd[i] = cw[i];
        for (int i = lane; i < ns; i += 32) cw[i] = td[i + 1];
        __syncwarp();
        for (int i = lane; i < ns; i += 32) td[i] = cw[i];
        __syncwarp();
    }
    // logits = anneal * log(w) where the interval is non-empty, else -inf ; softmax
    float mx = -INFINITY;
    for (int i = lane; i < nw; i += 32) {
        const float lg = (td[i + 1] > td[i]) ? mul_(anneal, logf(wd[i])) : -INFINITY;
        wd[i] = lg;
        mx = fmaxf(mx, lg);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float se = 0.f;
    for (int i = lane; i < nw; i += 32) { const float e = expf(wd[i] - mx); wd[i] = e; se += e; }
    se = warp_sum(se);
    __syncwarp();
    // cw = [0, min(cumsum(w[:-1]), 1), 1]  (ns entries)
    float carry = 0.f;
    for (int base = 0; base < nw - 1; base += 32) {
        const int i = base + lane;
        float v = (i < nw - 1) ? __fdiv_rn(wd[i], se) : 0.f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { float nb = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v = add_(v, nb); }
        v = add_(v, carry);
        if (i < nw - 1) cw[i + 1] = fminf(v, 1.0f);
        carry = __shfl_sync(0xffffffffu, v, 31);
    }
    if (lane == 0) { cw[0] = 0.f; cw[ns - 1] = 1.0f; }
    __syncwarp();
    // quirk Q18: a NaN logit (anneal 0 on an empty-weight, non-empty interval: 0 * log 0) or all logits -inf make the reference's
    // softmax NaN; cumsum and clip keep the NaN and sorted_interp's min then puts every centre on the first knot.  With one weight the
    // reference cdf is [0, 1] whatever the softmax, so the ordinary path below already agrees.  (se is warp-uniform.)
    const bool collapse = (se != se) && nw >= 2;
    // centres = sorted_interp(u, cw, td) ; reuse wd for the centres
    for (int k = lane; k < n_new; k += 32) {
        if (collapse) { wd[k] = td[0]; continue; }
        float u;
        if (jitter) {
            const float u_max = kEps + (1.f - kEps) / (float)n_new;
            const float max_jitter = (1.f - u_max) / (float)(n_new - 1) - kEps;
            // torch.linspace(0, 1-u_max, n)[k] + rand * max_jitter
            const float end = 1.f - u_max, step = end / (float)(n_new - 1);
            const float base = (k < n_new / 2) ? step * (float)k : end - step * (float)(n_new - 1 - k);
            u = base + jitter[b] * max_jitter;
        } else {
            const float pad = 1.f / (2.f * (float)n_new);
            const float start = pad, end = 1.f - pad - kEps, step = (end - start) / (float)(n_new - 1);
            u = (n_new == 1) ? start : ((k < n_new / 2) ? start + step * (float)k : end - step * (float)(n_new - 1 - k));
        }
        int a = 0, c = ns;                     // last j with cw[j] <= u
        while (c - a > 1) { int mid = (a + c) >> 1; if (cw[mid] <= u) a = mid; else c = mid; }
        const float x0 = cw[a], x1 = (a + 1 < ns) ? cw[a + 1] : cw[ns - 1];
        const float f0 = td[a], f1 = (a + 1 < ns) ? td[a + 1] : td[ns - 1];
        float off = __fdiv_rn(sub_(u, x0), sub_(x1, x0));
        if (off != off) off = 0.f;
        off = fminf(fmaxf(off, 0.f), 1.f);
        wd[k] = add_(f0, mul_(off, sub_(f1, f0)));
    }
    __syncwarp();
    float* so = s_out + (size_t)b * (n_new + 1);
    float* to = t_out + (size_t)b * (n_new + 1);
    const float sn = 1.f / near, sf = 1.f / far;
    for (int k = lane; k <= n_new; k += 32) {
        float s;
        if (k == 0) s = fmaxf(2.f * wd[0] - 0.5f * (wd[1] + wd[0]), 0.f);
        else if (k == n_new) s = fminf(2.f * wd[n_new - 1] - 0.5f * (wd[n_new - 1] + wd[n_new - 2]), 1.f);
        else s = 0.5f * (wd[k] + wd[k - 1]);
        so[k] = s;
        to[k] = 1.f / (s * sf + (1.f - s) * sn);                                 // s_to_t
    }
}

// ------------------------------------------------------------------------------------------------
// conical frustum -> Gaussian -> contraction -> 21-direction lift -> integrated positional encoding (one warp per sample)
// ------------------------------------------------------------------------------------------------
// Sources of the Gaussian (mean, cov) of sample m that the IPE features encode.  The encoding itself (contraction, lift, IPE) is
// the same code for both: features_kernel and features16_kernel take the source as a template parameter.
// conical frustum [t0, t1] of sample k of ray b, m = b * n + k (helper.py:293-339): the render's samples
struct FrustumSrc {          // read-only inputs: loaded through the non-coherent path (__ldg), as the kernels' __restrict__ arguments were
    const float *rays_o, *rays_d, *radii, *tdist;
    int n;
    __device__ __forceinline__ void operator()(long long m, float (&mean)[3], float (&cov)[3][3]) const {
        const int b = (int)(m / n), k = (int)(m % n);
        const float t0 = __ldg(tdist + (size_t)b * (n + 1) + k), t1 = __ldg(tdist + (size_t)b * (n + 1) + k + 1);
        const float d[3] = {__ldg(rays_d + 3 * b), __ldg(rays_d + 3 * b + 1), __ldg(rays_d + 3 * b + 2)};
        const float o[3] = {__ldg(rays_o + 3 * b), __ldg(rays_o + 3 * b + 1), __ldg(rays_o + 3 * b + 2)};
        const float rad = __ldg(radii + b);
        const float mu = (t0 + t1) / 2.f, hw = (t1 - t0) / 2.f;
        const float denom = fmaxf(3.f * mu * mu + hw * hw, kEps);
        const float t_mean = mu + (2.f * mu * hw * hw) / denom;
        const float hw4 = hw * hw * hw * hw;
        const float t_var = (hw * hw) / 3.f - (4.f / 15.f) * hw4 * (12.f * mu * mu - hw * hw) / (denom * denom);
        const float r_var = ((mu * mu) / 4.f + (5.f / 12.f) * hw * hw - (4.f / 15.f) * hw4 / denom) * rad * rad;
        const float dmag = fmaxf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2], 1e-10f);
        for (int i = 0; i < 3; ++i) {
            mean[i] = d[i] * t_mean + o[i];
            for (int j = 0; j < 3; ++j) cov[i][j] = t_var * d[i] * d[j] + r_var * ((i == j ? 1.f : 0.f) - d[i] * (d[j] / dmag));
        }
    }
};
// a point o + t viewdirs of sample k of ray b (fp32, each operation rounded) with covariance diag(var): neo_mip_field_eval
struct PointSrc {
    const float *rays_o, *viewdirs, *t;
    int n;
    float var[3];
    __device__ __forceinline__ void operator()(long long m, float (&mean)[3], float (&cov)[3][3]) const {
        const int b = (int)(m / n);
        const float tm = __ldg(t + m);
        for (int i = 0; i < 3; ++i) {
            mean[i] = add_(__ldg(rays_o + 3 * b + i), mul_(tm, __ldg(viewdirs + 3 * b + i)));
            for (int j = 0; j < 3; ++j) cov[i][j] = i == j ? var[i] : 0.f;
        }
    }
};
// contraction with its Jacobian (helper.py:33-66): z = x (r<=1) | ((2r-1)/r^2) x ; J = f I + ((2-2r)/r^4) x x^T ; zc = J cov J^T
__device__ __forceinline__ void contract_gaussian(const float (&mean)[3], const float (&cov)[3][3], float (&z)[3], float (&zc)[3][3]) {
    const float r2 = fmaxf(mean[0] * mean[0] + mean[1] * mean[1] + mean[2] * mean[2], 1e-32f);
    if (r2 <= 1.f) {
        for (int i = 0; i < 3; ++i) { z[i] = mean[i]; for (int j = 0; j < 3; ++j) zc[i][j] = cov[i][j]; }
    } else {
        const float r = sqrtf(r2), f = (2.f * r - 1.f) / r2, g = (2.f - 2.f * r) / (r2 * r2);
        float J[3][3], Tm[3][3];
        for (int i = 0; i < 3; ++i) { z[i] = f * mean[i]; for (int j = 0; j < 3; ++j) J[i][j] = (i == j ? f : 0.f) + g * mean[i] * mean[j]; }
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Tm[i][j] = J[i][0] * cov[0][j] + J[i][1] * cov[1][j] + J[i][2] * cov[2][j];
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) zc[i][j] = Tm[i][0] * J[j][0] + Tm[i][1] * J[j][1] + Tm[i][2] * J[j][2];
    }
}
template <class Src>
__device__ __forceinline__ void contracted_gaussian(const Src& src, long long m, float (&z)[3], float (&zc)[3][3]) {
    float mean[3], cov[3][3];
    src(m, mean, cov);
    contract_gaussian(mean, cov, z, zc);
}

// fp32 path (tight parity): one warp per sample, the reference's own sin(x), sin(x + pi/2) formulation
template <class Src>
__global__ void features_kernel(Src src, const float* __restrict__ basis, long long M, float* __restrict__ X) {
    const long long m = (long long)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    const int lane = threadIdx.x % 32;
    if (m >= M) return;
    float z[3], zc[3][3];
    contracted_gaussian(src, m, z, zc);
    if (lane < kBasis) {
        const float p[3] = {basis[lane], basis[kBasis + lane], basis[2 * kBasis + lane]};
        const float lm = z[0] * p[0] + z[1] * p[1] + z[2] * p[2];
        float cp[3];
        for (int i = 0; i < 3; ++i) cp[i] = zc[i][0] * p[0] + zc[i][1] * p[1] + zc[i][2] * p[2];
        const float lv = p[0] * cp[0] + p[1] * cp[1] + p[2] * cp[2];
        float sc = 1.f;
        float* x = X + (size_t)m * kFeat;
        for (int kk = 0; kk < kDeg; ++kk) {
            const float sm_ = lm * sc, e = expf(-0.5f * (lv * sc * sc));
            x[kk * kBasis + lane] = e * sinf(sm_);
            x[kDeg * kBasis + kk * kBasis + lane] = e * sinf(sm_ + 1.57079637f);
            sc *= 2.f;
        }
    }
}

// tensor-core path: fp16 rows of the activation buffer (row stride ld16 halfs, 504 features + 8 zero columns = 1 KB per sample).
// Thread = (sample, basis direction): 12 samples x 21 directions per block, no idle lanes.  The per-sample Gaussian is computed once
// into shared memory; sin / cos of the 12 octaves come from three accurate sincosf calls (octaves 0, 4, 8) and angle doubling in
// between.  Against float64 features rounded to fp16 (oracle/tc_paths_model.py), the field's per-point error stays fp16 rounding noise:
// tests/test_gpu_tc_paths.py measured up to 3.3e-4 in rgb and 5.3e-4 in density (pre-activation units) per point on an H100;
// the row is assembled in shared memory and leaves as 16-byte coalesced stores (the 2-byte scattered stores of the warp-per-sample
// kernel were the bottleneck: r2 launch list, 15.9 % of the Mip-NeRF 360 frame).
constexpr int kFeatSamples = 12, kFeatThreads = kFeatSamples * kBasis;     // 252
template <class Src>
__global__ void __launch_bounds__(kFeatThreads) features16_kernel(Src src, const float* __restrict__ basis, long long M, __half* __restrict__ X16,
                                                                  long long ld16) {
    __shared__ float zs[kFeatSamples][12];
    __shared__ __align__(16) __half row[kFeatSamples][kFeat + 8];
    const int tid = threadIdx.x;
    const long long m0 = (long long)blockIdx.x * kFeatSamples;
    const int nrows = (int)((M - m0) < kFeatSamples ? (M - m0) : kFeatSamples);
    if (tid < nrows) {
        float z[3], zc[3][3];
        contracted_gaussian(src, m0 + tid, z, zc);
        for (int i = 0; i < 3; ++i) { zs[tid][i] = z[i]; for (int j = 0; j < 3; ++j) zs[tid][3 + 3 * i + j] = zc[i][j]; }
    }
    if (tid < kFeatSamples * 8) row[tid / 8][kFeat + (tid % 8)] = __float2half_rn(0.f);
    __syncthreads();
    const int sidx = tid / kBasis, dir = tid % kBasis;
    if (sidx < nrows) {
        const float p[3] = {basis[dir], basis[kBasis + dir], basis[2 * kBasis + dir]};
        const float* zz = zs[sidx];
        const float lm = zz[0] * p[0] + zz[1] * p[1] + zz[2] * p[2];
        float lv = 0.f;
        for (int i = 0; i < 3; ++i) lv += p[i] * (zz[3 + 3 * i] * p[0] + zz[4 + 3 * i] * p[1] + zz[5 + 3 * i] * p[2]);
        __half* x = row[sidx];
        float sc = 1.f;
#pragma unroll
        for (int g = 0; g < kDeg / 4; ++g) {
            float sn, cs;
            sincosf(lm * sc, &sn, &cs);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int kk = 4 * g + j;
                const float e = __expf(-0.5f * (lv * sc * sc));
                x[kk * kBasis + dir] = __float2half_rn(e * sn);
                x[kDeg * kBasis + kk * kBasis + dir] = __float2half_rn(e * cs);
                const float s2 = 2.f * sn * cs, c2 = (cs - sn) * (cs + sn);
                sn = s2; cs = c2;
                sc *= 2.f;
            }
        }
    }
    __syncthreads();
    constexpr int kVec = (kFeat + 8) / 8;                       // 16-byte pieces per row
    for (int i = tid; i < nrows * kVec; i += kFeatThreads) {
        const int r = i / kVec, c = i % kVec;
        reinterpret_cast<uint4*>(X16 + (size_t)(m0 + r) * ld16)[c] = reinterpret_cast<const uint4*>(row[r])[c];
    }
}

// direction encoding broadcast to samples: out[m][c] for c < cols (27, or the fp16 operand's 64 with zero padding), row stride ld
template <class T>
__global__ void dir_kernel(const float* __restrict__ viewdirs, long long M, int n, T* __restrict__ out, long long ld, int cols) {
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= M * cols) return;
    const long long m = gid / cols;
    const int c = (int)(gid % cols);
    out[m * ld + c] = from_f32<T>(c < kDirEnc ? pos_enc_col(viewdirs + 3 * (m / n), 3, 4, c) : 0.f);
}

// ------------------------------------------------------------------------------------------------
// out[M][N] = act( A1[M][K1] . W[:, 0:K1]^T + A2[M][K2] . W[:, K1:K1+K2]^T + bias )      W is (N, K1+K2) row-major (nn.Linear)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) sgemm_kernel(const float* __restrict__ A1, int K1, const float* __restrict__ A2, int K2,
                                                    const float* __restrict__ W, const float* __restrict__ bias, long long M, int N,
                                                    int relu, float* __restrict__ out) {
    __shared__ float As[16][64 + 4];
    __shared__ float Bs[16][64 + 4];
    const long long m0 = (long long)blockIdx.x * 64;
    const int n0 = blockIdx.y * 64;
    const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
    const int ldw = K1 + K2;
    float acc[4][4] = {};
    for (int seg = 0; seg < 2; ++seg) {
        const float* A = seg ? A2 : A1;
        const int K = seg ? K2 : K1, wo = seg ? K1 : 0;
        if (!A || K == 0) continue;
        for (int k0 = 0; k0 < K; k0 += 16) {
            for (int e = threadIdx.x; e < 16 * 64; e += 256) {
                const int mm = e / 16, kk = e % 16;
                const long long mrow = m0 + mm;
                As[kk][mm] = (mrow < M && k0 + kk < K) ? A[(size_t)mrow * K + k0 + kk] : 0.f;
                const int nn = mm;
                Bs[kk][nn] = (n0 + nn < N && k0 + kk < K) ? W[(size_t)(n0 + nn) * ldw + wo + k0 + kk] : 0.f;
            }
            __syncthreads();
#pragma unroll
            for (int kk = 0; kk < 16; ++kk) {
                float a[4], b[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) { a[i] = As[kk][ty * 4 + i]; b[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
            }
            __syncthreads();
        }
    }
    for (int i = 0; i < 4; ++i) {
        const long long mrow = m0 + ty * 4 + i;
        if (mrow >= M) continue;
        for (int j = 0; j < 4; ++j) {
            const int nn = n0 + tx * 4 + j;
            if (nn >= N) continue;
            float v = acc[i][j] + (bias ? bias[nn] : 0.f);
            if (relu) v = fmaxf(v, 0.f);
            out[(size_t)mrow * N + nn] = v;
        }
    }
}

// composite_kernel's head activations without the compositing (neo_mip_field_eval): density = softplus(raw - 1), rgb = 1.002 sigmoid - 0.001
__global__ void field_act_kernel(const float* __restrict__ raw_density, const float* __restrict__ raw_rgb, long long M, float* __restrict__ density,
                                 float* __restrict__ rgb) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= M * 4) return;
    const long long m = i >> 2;
    const int c = (int)(i & 3);
    if (c == 3) density[m] = softplus_(raw_density[m] - 1.0f);
    else if (rgb) rgb[m * 3 + c] = rgb_act(raw_rgb[m * 3 + c]);
}

// ------------------------------------------------------------------------------------------------
// activations + compute_alpha_weights(opaque_background) + volumetric_rendering (white background weight)   (one warp per ray)
// ------------------------------------------------------------------------------------------------
__global__ void composite_kernel(const float* __restrict__ raw_density, const float* __restrict__ raw_rgb, const float* __restrict__ tdist,
                                 const float* __restrict__ rays_d, int n_rays, int n, float* __restrict__ density_out,
                                 float* __restrict__ rgb_s_out, float* __restrict__ w_out, float* __restrict__ rgb_out) {
    const int warps = blockDim.x / 32, wid = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int b = blockIdx.x * warps + wid;
    if (b >= n_rays) return;
    const float* dd3 = rays_d + 3 * b;
    const float dn = __fsqrt_rn(dot3_(dd3, dd3));
    const float* t = tdist + (size_t)b * (n + 1);
    float carry = 0.f, acc = 0.f, cr = 0.f, cg = 0.f, cb = 0.f;
    for (int base = 0; base < n; base += 32) {
        const int k = base + lane;
        const bool ok = k < n;
        float dens = 0.f, dd = 0.f, col[3] = {0.f, 0.f, 0.f};
        if (ok) {
            dens = softplus_(raw_density[(size_t)b * n + k] - 1.0f);
            dd = (k == n - 1) ? INFINITY : mul_(dens, mul_(sub_(t[k + 1], t[k]), dn));
            for (int c = 0; c < 3; ++c) col[c] = raw_rgb ? rgb_act(raw_rgb[((size_t)b * n + k) * 3 + c]) : 0.f;
        }
        float sc = ok ? ((k == n - 1) ? 0.f : dd) : 0.f;       // cumsum runs over dd[:-1]
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { float nb = __shfl_up_sync(0xffffffffu, sc, o); if (lane >= o) sc = add_(sc, nb); }
        const float incl = add_(sc, carry);
        float excl = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) excl = carry;
        if (ok) {
            const float alpha = 1.f - expf(-dd);
            const float wv = alpha * expf(-excl);
            if (density_out) density_out[(size_t)b * n + k] = dens;
            if (w_out) w_out[(size_t)b * n + k] = wv;
            if (rgb_s_out) for (int c = 0; c < 3; ++c) rgb_s_out[((size_t)b * n + k) * 3 + c] = col[c];
            acc += wv; cr += wv * col[0]; cg += wv * col[1]; cb += wv * col[2];
        }
        carry = __shfl_sync(0xffffffffu, incl, 31);
    }
    acc = warp_sum(acc); cr = warp_sum(cr); cg = warp_sum(cg); cb = warp_sum(cb);
    if (lane == 0 && rgb_out) {
        const float bg = fmaxf(1.f - acc, 0.f);                 // bg_intensity_range = (1, 1)
        rgb_out[3 * b] = cr + bg; rgb_out[3 * b + 1] = cg + bg; rgb_out[3 * b + 2] = cb + bg;
    }
}

// ------------------------------------------------------------------------------------------------
// backward of composite_kernel w.r.t. the raw density and raw rgb (sample positions carry no gradient: model.py:309-310)  (one warp per ray)
//   x_k = softplus(r_k - 1) delta_k (x_{N-1} = inf),  T_k = exp(-sum_{j<k} x_j),  w_k = (1 - e^{-x_k}) T_k,  rgb = sum w c + clip(1 - acc, 0)
//   G_k = g_w_k + g_rgb . c_k - m sum(g_rgb),   m = [1 - acc >= 0]   (the gradient clip passes, decided on this kernel's own fp32 acc)
//   dL/dx_k = G_k e^{-x_k} T_k - sum_{j>k} G_j w_j  (0 for the last, infinite, interval)
//   d_raw_density_k = (delta_k dL/dx_k + g_density_k) softplus'(r_k - 1),   d_raw_rgb_k = (w_k g_rgb + g_rgb_s_k) 1.002 s (1 - s)
// Pass 1 repeats composite_kernel's operations for w and acc and keeps the exclusive scan in the d_raw_density
// row; pass 2 walks the chunks backwards with a suffix scan of G w.
// ------------------------------------------------------------------------------------------------
__global__ void composite_bwd_kernel(const float* __restrict__ raw_density, const float* __restrict__ raw_rgb, const float* __restrict__ tdist,
                                     const float* __restrict__ rays_d, int n_rays, int n, const float* __restrict__ g_rgb,
                                     const float* __restrict__ g_w, const float* __restrict__ g_density, const float* __restrict__ g_rgb_s,
                                     float* __restrict__ d_raw_density, float* __restrict__ d_raw_rgb) {
    const int warps = blockDim.x / 32, wid = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int b = blockIdx.x * warps + wid;
    if (b >= n_rays) return;
    const float* dd3 = rays_d + 3 * b;
    const float dn = __fsqrt_rn(dot3_(dd3, dd3));
    const float* t = tdist + (size_t)b * (n + 1);
    const float* rd = raw_density + (size_t)b * n;
    float* gd = d_raw_density + (size_t)b * n;
    auto x_of = [&](int k, float& delta) -> float {
        delta = mul_(sub_(t[k + 1], t[k]), dn);
        return (k == n - 1) ? INFINITY : mul_(softplus_(rd[k] - 1.0f), delta);
    };
    float carry = 0.f, acc = 0.f;
    for (int base = 0; base < n; base += 32) {
        const int k = base + lane;
        const bool ok = k < n;
        float delta, dd = ok ? x_of(k, delta) : 0.f;
        float sc = ok ? ((k == n - 1) ? 0.f : dd) : 0.f;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { float nb = __shfl_up_sync(0xffffffffu, sc, o); if (lane >= o) sc = add_(sc, nb); }
        const float incl = add_(sc, carry);
        float excl = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) excl = carry;
        if (ok) {
            gd[k] = excl;
            acc += (1.f - expf(-dd)) * expf(-excl);
        }
        carry = __shfl_sync(0xffffffffu, incl, 31);
    }
    acc = warp_sum(acc);
    const float gc[3] = {g_rgb ? g_rgb[3 * b] : 0.f, g_rgb ? g_rgb[3 * b + 1] : 0.f, g_rgb ? g_rgb[3 * b + 2] : 0.f};
    const float gbg = (1.f - acc >= 0.f) ? gc[0] + gc[1] + gc[2] : 0.f;
    float S = 0.f;                                              // sum_{j >= next chunk} G_j w_j
    for (int base = ((n - 1) / 32) * 32; base >= 0; base -= 32) {
        const int k = base + lane;
        const bool ok = k < n;
        float v = 0.f, dx = 0.f, delta = 0.f, w = 0.f, T = 0.f, e = 0.f, s[3] = {0.f, 0.f, 0.f};
        if (ok) {
            const float dd = x_of(k, delta);
            T = expf(-gd[k]);
            e = expf(-dd);
            w = (1.f - e) * T;
            float G = (g_w ? g_w[(size_t)b * n + k] : 0.f) - gbg;
            if (raw_rgb)
                for (int c = 0; c < 3; ++c) {
                    s[c] = raw_rgb[((size_t)b * n + k) * 3 + c];
                    G += gc[c] * rgb_act(s[c]);
                }
            v = G * w;
            dx = G * e * T;
        }
        float incl = v;                                         // suffix scan within the chunk
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { float nb = __shfl_down_sync(0xffffffffu, incl, o); if (lane + o < 32) incl += nb; }
        float after = __shfl_down_sync(0xffffffffu, incl, 1);
        if (lane == 31) after = 0.f;
        const float chunk = __shfl_sync(0xffffffffu, incl, 0);
        if (ok) {
            dx = (k == n - 1) ? 0.f : dx - (after + S);
            const float z = rd[k] - 1.0f;
            const float sp = z > 20.f ? 1.f : 1.f / (1.f + expf(-z));            // softplus'(z), threshold 20 as F.softplus
            gd[k] = (delta * dx + (g_density ? g_density[(size_t)b * n + k] : 0.f)) * sp;
            if (raw_rgb)
                for (int c = 0; c < 3; ++c) {
                    const float q = expf(-fabsf(s[c]));                           // s (1 - s) = q / (1 + q)^2 without cancellation
                    const float up = w * gc[c] + (g_rgb_s ? g_rgb_s[((size_t)b * n + k) * 3 + c] : 0.f);
                    d_raw_rgb[((size_t)b * n + k) * 3 + c] = up * (1.002f * (q / ((1.f + q) * (1.f + q))));
                }
        }
        S += chunk;
    }
}

}  // namespace mip
}  // namespace neo

using namespace neo;

namespace {
struct WSM {
    float *s[3], *t, *w[3], *X, *Ha, *Hb, *beta, *DE, *V, *rawd, *rawc;
    // tensor-core path (fp16): two activation buffers [M][width + 512] whose tail columns hold the padded IPE features of buffer 0,
    // [M][256 + 64] = bottleneck | padded direction encoding, [M][128], and the packed weights
    __half *A16[2], *B16, *V16, *W16;
};
constexpr int kFeatPad = 512, kDirPad = 64;
size_t tc_weight_halves(int width) {      // fp16 elements of one MLP's packed weights (upper bound: the 8-layer NeRF MLP)
    return (size_t)width * kFeatPad + 6 * (size_t)width * width + (size_t)width * (width + kFeatPad) + 256 * (size_t)width + 128 * (256 + kDirPad);
}
// the buffers of one MLP evaluation over M samples (features, activations, raw heads; the packed fp16 weights on the tensor-core path)
void carve_mlp(Carve& c, size_t M, int width, bool tcp, WSM& w) {
    w.X = c.take<float>(tcp ? 0 : M * mip::kFeat);          // the fp32 activation buffers are not needed on the tensor-core path
    w.Ha = c.take<float>(tcp ? 0 : M * width); w.Hb = c.take<float>(tcp ? 0 : M * width);
    w.beta = c.take<float>(tcp ? 0 : M * 256); w.DE = c.take<float>(tcp ? 0 : M * 27); w.V = c.take<float>(tcp ? 0 : M * 128);
    w.rawd = c.take<float>(M); w.rawc = c.take<float>(M * 3);
    if (tcp) {
        for (int i = 0; i < 2; ++i) w.A16[i] = c.take<__half>(M * (size_t)(width + kFeatPad));
        w.B16 = c.take<__half>(M * (256 + kDirPad));
        w.V16 = c.take<__half>(M * 128);
        w.W16 = c.take<__half>(tc_weight_halves(width));
    }
}
size_t carve(Carve& c, int n, const NeoMipCfg* cfg, int width, WSM& w) {
    const int ns[3] = {cfg->n_prop, cfg->n_prop, cfg->n_nerf};
    int nmax = cfg->n_prop > cfg->n_nerf ? cfg->n_prop : cfg->n_nerf;
    for (int l = 0; l < 3; ++l) { w.s[l] = c.take<float>((size_t)n * (ns[l] + 1)); w.w[l] = c.take<float>((size_t)n * ns[l]); }
    w.t = c.take<float>((size_t)n * (nmax + 1));
    carve_mlp(c, (size_t)n * nmax, width, cfg->precision == NEO_PREC_TC, w);
    return c.used;
}
int check(const NeoMipCfg* c) {
    if (!c || c->n_prop < 2 || c->n_nerf < 2 || c->n_prop > 160 || c->n_nerf > 160) { set_error("mip: sample counts must be in [2,160]"); return NEO_ERR_INVALID; }
    if (!(c->near_plane > 0.f) || !(c->far_plane > c->near_plane)) { set_error("mip: need 0 < near < far"); return NEO_ERR_INVALID; }
    if (c->precision != NEO_PREC_FP32 && c->precision != NEO_PREC_TC) { set_error("mip: bad precision %d", c->precision); return NEO_ERR_INVALID; }
    return NEO_OK;
}
// One level of proposal resampling (max_dilate_weights + annealed logits + sample_intervals + s_to_t): sdist / tdist (n_rays, n + 1).
// Level 0 reads no previous level; level l > 0 reads the (n_rays, n_prev + 1) sdist and (n_rays, n_prev) weights of level l - 1.
// dilation = 0.0025 + 0.5 / prod(sample counts of the levels before), model.py:265-272.
int launch_resample(const float* s_prev, const float* w_prev, int n_rays, int n_prev, int level, float dilation, float anneal, int n, float near,
                    float far, const float* jitter, float* s_out, float* t_out, cudaStream_t s) {
    int p2 = 2;
    while (p2 < 3 * n_prev + 1 || p2 < n + 1) p2 <<= 1;
    const int warps = 4;
    const size_t smem = (size_t)warps * (3 * p2 + 3 * n_prev) * sizeof(float);
    if (smem > 48 * 1024) NEO_CUDA(cudaFuncSetAttribute(mip::resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    mip::resample_kernel<<<(n_rays + warps - 1) / warps, warps * 32, smem, s>>>(s_prev, w_prev, n_rays, n_prev, level, dilation, anneal, n, near, far,
                                                                               jitter, s_out, t_out, p2);
    NEO_LAUNCH_CHECK("mip resample_kernel");
    return NEO_OK;
}
float anneal_of(float train_frac) { return (10.f * train_frac) / (9.f * train_frac + 1.f); }     // bias(train_frac, anneal_slope=10)
constexpr int kCompWarps = 8;
int gemm(const float* A1, int K1, const float* A2, int K2, const float* W, const float* b, long long M, int N, int relu, float* out, cudaStream_t s) {
    dim3 grid((unsigned)((M + 63) / 64), (unsigned)((N + 63) / 64));
    mip::sgemm_kernel<<<grid, 256, 0, s>>>(A1, K1, A2, K2, W, b, M, N, relu, out);
    NEO_LAUNCH_CHECK("mip sgemm_kernel");
    return NEO_OK;
}

// One MLP of Mip-NeRF 360 (models/mipnerf360/model.py:30-195) on tensor cores: fp16 activations, every dense layer a gemm_f16 launch
// (csrc/gemm_tc.cu), the skip concatenation by laying h4 and the features out in ONE buffer (layer 5 is a single K = width + 512 GEMM).
int mlp_tc(const NeoMipMLPParams& p, const WSM& w, long long M, int n, const float* viewdirs, float* rawd, float* rawc, cudaStream_t s) {
    const int W = p.width, ld = W + kFeatPad;
    if (W % 64) { set_error("mip tc: width must be a multiple of 64 (got %d)", W); return NEO_ERR_UNSUPPORTED; }
    __half* buf[2] = {w.A16[0], w.A16[1]};
    __half* wp = w.W16;
    int rc;
    // the IPE features were written by features_kernel as fp16 into the tail columns of buffer 0 (zero padded to 512)
    auto pack = [&](const float* src, int rows, int cols_in, int cols_out) -> __half* {
        __half* dst = wp;
        wp += (size_t)rows * cols_out;
        return f32_to_f16_pad(src, rows, cols_in, cols_in, dst, cols_out, cols_out, s) ? nullptr : dst;
    };
    __half* w0 = pack(p.w[0], W, mip::kFeat, kFeatPad);
    if (!w0) return NEO_ERR_CUDA;
    if ((rc = gemm_f16(buf[0] + W, ld, w0, kFeatPad, p.b[0], buf[0], ld, M, W, kFeatPad, 1, s))) return rc;
    for (int l = 1; l < p.depth; ++l) {
        const bool skip_in = (l == 5);                      // cat([h, inputs]) after layer 4 feeds layer 5 (model.py:122-128)
        __half* wl;
        int K;
        if (skip_in) {
            // W5 is (width, width + 504): columns [0, width) stay, the 504 feature columns are padded to 512
            wl = wp;
            wp += (size_t)W * (W + kFeatPad);
            if ((rc = f32_to_f16_pad(p.w[l], W, W, W + mip::kFeat, wl, W, W + kFeatPad, s))) return rc;
            if ((rc = f32_to_f16_pad(p.w[l] + W, W, mip::kFeat, W + mip::kFeat, wl + W, kFeatPad, W + kFeatPad, s))) return rc;
            K = W + kFeatPad;
        } else {
            wl = pack(p.w[l], W, W, W);
            if (!wl) return NEO_ERR_CUDA;
            K = W;
        }
        if ((rc = gemm_f16(buf[(l - 1) & 1], ld, wl, K, p.b[l], buf[l & 1], ld, M, W, K, 1, s))) return rc;
    }
    const __half* h = buf[(p.depth - 1) & 1];
    if ((rc = launch_rowdot_f16(h, ld, W, p.wsig, p.bsig, 1, M, rawd, s))) return rc;
    if (p.wrgb) {
        __half* B = w.B16;
        __half* V = w.V16;
        const int ldb = 256 + kDirPad;
        __half* wb = pack(p.wb, 256, W, W);
        if (!wb) return NEO_ERR_CUDA;
        if ((rc = gemm_f16(h, ld, wb, W, p.bb, B, ldb, M, 256, W, 0, s))) return rc;
        mip::dir_kernel<<<(unsigned)((M * kDirPad + 255) / 256), 256, 0, s>>>(viewdirs, M, n, B + 256, ldb, kDirPad);
        NEO_LAUNCH_CHECK("mip dir_kernel");
        __half* wv = wp;
        wp += (size_t)128 * ldb;
        if ((rc = f32_to_f16_pad(p.wv0, 128, 256, 256 + 27, wv, 256, ldb, s))) return rc;
        if ((rc = f32_to_f16_pad(p.wv0 + 256, 128, 27, 256 + 27, wv + 256, kDirPad, ldb, s))) return rc;
        if ((rc = gemm_f16(B, ldb, wv, ldb, p.bv0, V, 128, M, 128, ldb, 1, s))) return rc;
        if ((rc = launch_rowdot_f16(V, 128, 128, p.wrgb, p.brgb, 3, M, rawc, s))) return rc;
    }
    return NEO_OK;
}

// One MLP of Mip-NeRF 360 as the chain of fp32 SGEMMs with fused bias / ReLU / concatenation (the reference formulation).
int mlp_fp32(const NeoMipMLPParams& p, const WSM& w, long long M, int n, const float* viewdirs, float* rawd, float* rawc, cudaStream_t s) {
    int rc;
    float* src = w.Ha;
    float* dst = w.Hb;
    if ((rc = gemm(w.X, mip::kFeat, nullptr, 0, p.w[0], p.b[0], M, p.width, 1, src, s))) return rc;
    for (int l = 1; l < p.depth; ++l) {
        const bool skip_in = (l == 5);                      // cat([h, inputs]) after layer 4 feeds layer 5
        if ((rc = gemm(src, p.width, skip_in ? w.X : nullptr, skip_in ? mip::kFeat : 0, p.w[l], p.b[l], M, p.width, 1, dst, s))) return rc;
        float* tmp = src; src = dst; dst = tmp;
    }
    if ((rc = gemm(src, p.width, nullptr, 0, p.wsig, p.bsig, M, 1, 0, rawd, s))) return rc;
    if (p.wrgb) {
        if ((rc = gemm(src, p.width, nullptr, 0, p.wb, p.bb, M, 256, 0, w.beta, s))) return rc;
        mip::dir_kernel<<<(unsigned)((M * 27 + 255) / 256), 256, 0, s>>>(viewdirs, M, n, w.DE, 27, 27);
        NEO_LAUNCH_CHECK("mip dir_kernel");
        if ((rc = gemm(w.beta, 256, w.DE, 27, p.wv0, p.bv0, M, 128, 1, w.V, s))) return rc;
        if ((rc = gemm(w.V, 128, nullptr, 0, p.wrgb, p.brgb, M, 3, 0, rawc, s))) return rc;
    }
    return NEO_OK;
}
// features (of the Gaussians of `src`) and then the MLP of one level, in either precision: raw density (M), raw rgb (M, 3) if p has a colour head
template <class Src>
int features_mlp(const NeoMipMLPParams& p, Src src, const WSM& w, long long M, int n, const float* viewdirs, int precision, cudaStream_t s) {
    if (precision == NEO_PREC_TC) {
        mip::features16_kernel<<<(unsigned)((M + mip::kFeatSamples - 1) / mip::kFeatSamples), mip::kFeatThreads, 0, s>>>(
            src, p.basis, M, w.A16[0] + p.width, p.width + kFeatPad);
        NEO_LAUNCH_CHECK("mip features16_kernel");
        return mlp_tc(p, w, M, n, viewdirs, w.rawd, w.rawc, s);
    }
    mip::features_kernel<<<(unsigned)((M + 7) / 8), 256, 0, s>>>(src, p.basis, M, w.X);
    NEO_LAUNCH_CHECK("mip features_kernel");
    return mlp_fp32(p, w, M, n, viewdirs, w.rawd, w.rawc, s);
}
int check_mlp(const NeoMipMLPParams& p, int l) {
    if (p.depth < 1 || p.depth > 8 || p.width < 64 || p.width % 4 || !p.basis) { set_error("mip mlp %d: bad depth/width", l); return NEO_ERR_INVALID; }
    if ((l == 2) != (p.wrgb != nullptr)) { set_error("mip: mlps must be {prop, prop, nerf}"); return NEO_ERR_INVALID; }
    return NEO_OK;
}
}  // namespace

extern "C" size_t neo_mip_workspace_bytes(int n_rays, const NeoMipCfg* cfg, int nerf_width) {
    if (n_rays <= 0 || check(cfg) || nerf_width < 64) return 0;
    Carve c{nullptr, 0};
    WSM w;
    return carve(c, n_rays, cfg, nerf_width > 256 ? nerf_width : 256, w);
}

extern "C" int neo_mip_render_fwd(const NeoMipMLPParams mlps[3], const float* rays_o, const float* rays_d, const float* viewdirs,
                                  const float* radii, int n_rays, const NeoMipCfg* cfg, NeoMipOut* out, void* workspace,
                                  size_t workspace_bytes, void* stream) {
    if (!mlps || !rays_o || !rays_d || !viewdirs || !radii || !out || n_rays <= 0) { set_error("neo_mip_render_fwd: bad arguments"); return NEO_ERR_INVALID; }
    int rc = check(cfg);
    if (rc) return rc;
    for (int l = 0; l < 3; ++l)
        if ((rc = check_mlp(mlps[l], l))) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const int width = mlps[2].width > 256 ? mlps[2].width : 256;
    Carve c{static_cast<unsigned char*>(workspace), 0};
    WSM w;
    size_t need = carve(c, n_rays, cfg, width, w);
    if (!workspace || workspace_bytes < need) { set_error("workspace too small: need %zu bytes, got %zu", need, workspace_bytes); return NEO_ERR_WORKSPACE; }
    const int ns[3] = {cfg->n_prop, cfg->n_prop, cfg->n_nerf};
    const float anneal = anneal_of(cfg->train_frac);
    long long prod = 1;
    for (int lvl = 0; lvl < 3; ++lvl) {
        const int n = ns[lvl], n_prev = lvl ? ns[lvl - 1] : 1;
        const float dilation = 0.0025f + 0.5f / (float)prod;
        prod *= n;
        if ((rc = launch_resample(lvl ? w.s[lvl - 1] : nullptr, lvl ? w.w[lvl - 1] : nullptr, n_rays, n_prev, lvl, dilation, anneal, n, cfg->near_plane,
                                  cfg->far_plane, cfg->jitter[lvl], w.s[lvl], w.t, s))) return rc;
        const long long M = (long long)n_rays * n;
        const NeoMipMLPParams& p = mlps[lvl];
        if ((rc = features_mlp(p, mip::FrustumSrc{rays_o, rays_d, radii, w.t, n}, w, M, n, viewdirs, cfg->precision, s))) return rc;
        const float* rawc = p.wrgb ? w.rawc : nullptr;
        if (!p.wrgb && out->rgb_s[lvl]) NEO_CUDA(cudaMemsetAsync(out->rgb_s[lvl], 0, (size_t)M * 3 * sizeof(float), s));     // disable_rgb: zeros
        const int cw = kCompWarps;
        mip::composite_kernel<<<(n_rays + cw - 1) / cw, cw * 32, 0, s>>>(w.rawd, rawc, w.t, rays_d, n_rays, n, out->density[lvl],
                                                                        rawc ? out->rgb_s[lvl] : nullptr, w.w[lvl], out->rgb[lvl]);
        NEO_LAUNCH_CHECK("mip composite_kernel");
        if ((rc = copy_out(out->sdist[lvl], w.s[lvl], (size_t)n_rays * (n + 1), s))) return rc;
        if ((rc = copy_out(out->weights[lvl], w.w[lvl], (size_t)M, s))) return rc;
    }
    return NEO_OK;
}

extern "C" size_t neo_mip_field_workspace_bytes(long long n_points, int width, int precision) {
    if (n_points <= 0 || width < 64 || (precision != NEO_PREC_FP32 && precision != NEO_PREC_TC)) return 0;
    Carve c{nullptr, 0};
    WSM w;
    carve_mlp(c, (size_t)n_points, width > 256 ? width : 256, precision == NEO_PREC_TC, w);
    return c.used;
}

extern "C" int neo_mip_field_eval(const NeoMipMLPParams mlps[3], int level, const NeoRays* rays, const float* t_vals, int N, const float var[3],
                                  int precision, float* rgb, float* density, void* ws, size_t ws_bytes, void* stream) {
    if (!mlps || !rays || !t_vals || !var || !density) { set_error("neo_mip_field_eval: null argument"); return NEO_ERR_INVALID; }
    if (level < 0 || level > 2) { set_error("neo_mip_field_eval: level must be 0, 1 or 2 (got %d)", level); return NEO_ERR_INVALID; }
    if (rgb && level < 2) { set_error("neo_mip_field_eval: proposal level %d has no colour head (pass rgb = NULL)", level); return NEO_ERR_INVALID; }
    if (precision != NEO_PREC_FP32 && precision != NEO_PREC_TC) { set_error("neo_mip_field_eval: bad precision %d", precision); return NEO_ERR_INVALID; }
    if (rays->n_rays <= 0 || !rays->rays_o || !rays->viewdirs || N < 1) { set_error("neo_mip_field_eval: empty rays or N < 1"); return NEO_ERR_INVALID; }
    for (int i = 0; i < 3; ++i)
        if (!(var[i] >= 0.f && var[i] <= 3.4e38f)) { set_error("neo_mip_field_eval: var must be finite and >= 0"); return NEO_ERR_INVALID; }
    int rc = check_mlp(mlps[level], level);
    if (rc) return rc;
    const NeoMipMLPParams& p = mlps[level];
    const long long M = (long long)rays->n_rays * N;
    if (M > ((long long)1 << 31) - 1) { set_error("neo_mip_field_eval: n_rays * N must be below 2^31"); return NEO_ERR_INVALID; }
    Carve c{static_cast<unsigned char*>(ws), 0};
    WSM w;
    carve_mlp(c, (size_t)M, p.width > 256 ? p.width : 256, precision == NEO_PREC_TC, w);
    if (!ws || ws_bytes < c.used) { set_error("workspace too small: need %zu bytes, got %zu", c.used, ws_bytes); return NEO_ERR_WORKSPACE; }
    cudaStream_t s = (cudaStream_t)stream;
    const mip::PointSrc src{rays->rays_o, rays->viewdirs, t_vals, N, {var[0], var[1], var[2]}};
    if ((rc = features_mlp(p, src, w, M, N, rays->viewdirs, precision, s))) return rc;
    mip::field_act_kernel<<<(unsigned)((M * 4 + 255) / 256), 256, 0, s>>>(w.rawd, p.wrgb ? w.rawc : nullptr, M, density, rgb);
    NEO_LAUNCH_CHECK("mip field_act_kernel");
    return NEO_OK;
}

// ---- stage-level entry points of the training path (neo360_b200/mip.py): resampling and encodings have no backward (the sample positions
// are detached, model.py:309-310, and contract returns detached values, helper.py:63-66); compositing forward is composite_kernel itself and
// its backward composite_bwd_kernel; the dense layers are differentiated by the host framework ----
extern "C" int neo_mip_resample(const float* sdist_prev, const float* weights_prev, int n_rays, int n_prev, int level, int n_new, float near_plane,
                                float far_plane, float train_frac, const float* jitter, float* sdist, float* tdist, void* stream) {
    if (level < 0 || level > 2) { set_error("neo_mip_resample: level must be 0, 1 or 2 (got %d)", level); return NEO_ERR_INVALID; }
    if (!sdist || !tdist || n_rays <= 0 || n_new < 2 || n_new > 160 || (level > 0 && (!sdist_prev || !weights_prev || n_prev < 1 || n_prev > 160))) {
        set_error("neo_mip_resample: bad arguments");
        return NEO_ERR_INVALID;
    }
    if (!(near_plane > 0.f) || !(far_plane > near_plane)) { set_error("neo_mip_resample: need 0 < near < far"); return NEO_ERR_INVALID; }
    // levels 0 and 1 both take num_prop_samples, so the sample counts before level l multiply to n_prev^l
    float prod = 1.f;
    for (int l = 0; l < level; ++l) prod *= (float)n_prev;
    return launch_resample(level ? sdist_prev : nullptr, level ? weights_prev : nullptr, n_rays, level ? n_prev : 1, level, 0.0025f + 0.5f / prod,
                           anneal_of(train_frac), n_new, near_plane, far_plane, jitter, sdist, tdist, (cudaStream_t)stream);
}

extern "C" int neo_mip_encode(const float* rays_o, const float* rays_d, const float* viewdirs, const float* radii, const float* tdist, const float* basis,
                              int n_rays, int N, float* feats, float* dir_enc, void* stream) {
    if (!rays_o || !rays_d || !viewdirs || !radii || !tdist || !basis || !feats || !dir_enc || n_rays <= 0 || N < 1) {
        set_error("neo_mip_encode: bad arguments");
        return NEO_ERR_INVALID;
    }
    cudaStream_t s = (cudaStream_t)stream;
    const long long M = (long long)n_rays * N;
    mip::features_kernel<<<(unsigned)((M + 7) / 8), 256, 0, s>>>(mip::FrustumSrc{rays_o, rays_d, radii, tdist, N}, basis, M, feats);
    NEO_LAUNCH_CHECK("mip features_kernel");
    mip::dir_kernel<<<(unsigned)(((long long)n_rays * kDirEnc + 255) / 256), 256, 0, s>>>(viewdirs, (long long)n_rays, 1, dir_enc, kDirEnc, kDirEnc);
    NEO_LAUNCH_CHECK("mip dir_kernel");
    return NEO_OK;
}

extern "C" int neo_mip_composite(const float* raw_density, const float* raw_rgb, const float* tdist, const float* rays_d, int n_rays, int N, float* rgb,
                                 float* weights, float* density, float* rgb_s, void* stream) {
    if (!raw_density || !tdist || !rays_d || n_rays <= 0 || N < 1) { set_error("neo_mip_composite: bad arguments"); return NEO_ERR_INVALID; }
    mip::composite_kernel<<<(n_rays + kCompWarps - 1) / kCompWarps, kCompWarps * 32, 0, (cudaStream_t)stream>>>(raw_density, raw_rgb, tdist, rays_d,
                                                                                                              n_rays, N, density, rgb_s, weights, rgb);
    NEO_LAUNCH_CHECK("mip composite_kernel");
    return NEO_OK;
}

extern "C" int neo_mip_composite_bwd(const float* raw_density, const float* raw_rgb, const float* tdist, const float* rays_d, int n_rays, int N,
                                     const float* g_rgb, const float* g_weights, const float* g_density, const float* g_rgb_s, float* d_raw_density,
                                     float* d_raw_rgb, void* stream) {
    if (!raw_density || !tdist || !rays_d || !d_raw_density || (raw_rgb && !d_raw_rgb) || n_rays <= 0 || N < 1) {
        set_error("neo_mip_composite_bwd: bad arguments");
        return NEO_ERR_INVALID;
    }
    mip::composite_bwd_kernel<<<(n_rays + kCompWarps - 1) / kCompWarps, kCompWarps * 32, 0, (cudaStream_t)stream>>>(
        raw_density, raw_rgb, tdist, rays_d, n_rays, N, g_rgb, g_weights, g_density, g_rgb_s, d_raw_density, d_raw_rgb);
    NEO_LAUNCH_CHECK("mip composite_bwd_kernel");
    return NEO_OK;
}
