// Deterministic backward kernels of the training step: what runs when torch.are_deterministic_algorithms_enabled() is true.
//
//  * Order-fixed scatter (the lookups' adjoint without floating-point atomics).  An entry kernel owned by each lookup
//    (csrc/field_fp32.cu, csrc/encoder.cu) writes one entry per (row, tap, map): an integer texel key, a weight and its own entry id.
//    A stable CUB radix sort orders the (key, id) pairs by key, keeping ascending entry ids within a key; zero-weight taps carry the
//    key T (past every texel) and are never reduced.  A segment kernel turns the sorted keys into segment starts, and one warp per
//    texel sums its segment into the texel's existing value as acc = __fadd_rn(acc, __fmul_rn(w, g)) in sorted order, channels
//    spread over the lanes.  Every step is a function of the inputs only, so two calls are bit-identical.  Segments are not split:
//    a texel that one warp reduces alone costs its entry count in dependent additions (about 10 ms for 10^5 entries).
//  * Per-ray training losses with a backward (one warp per ray, fixed-order sums, no atomics): the distortion regulariser of
//    training.distortion_loss and one proposal level of Mip-NeRF 360's interlevel loss.
//  * Adjoint of the bilinear upsampling with align_corners=True (F.interpolate): a gather that writes each input element once.
#include "common.cuh"
#include <cub/device/device_radix_sort.cuh>

namespace neo {

// ---- order-fixed scatter ----

static int key_bits(long long T) {
    int b = 1;
    while ((1LL << b) <= T) ++b;
    return b;
}

static size_t sort_scratch_bytes(long long E, long long T) {
    size_t bytes = 0;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const unsigned*)nullptr, (unsigned*)nullptr, (const unsigned*)nullptr,
                                                    (unsigned*)nullptr, (int)E, 0, key_bits(T));
    if (e != cudaSuccess) {
        cudaGetLastError();
        set_error("order-fixed scatter: sort scratch query failed: %s", cudaGetErrorString(e));
        return 0;
    }
    return bytes;
}

DetBuffers det_carve(void* ws, long long E, long long T) {
    Carve c{static_cast<unsigned char*>(ws), 0};
    DetBuffers b;
    b.keys = c.take<unsigned>(E);
    b.keys_sorted = c.take<unsigned>(E);
    b.ids = c.take<unsigned>(E);
    b.ids_sorted = c.take<unsigned>(E);
    b.wts = c.take<float>(E);
    b.starts = c.take<unsigned>(T + 1);
    b.scratch_bytes = sort_scratch_bytes(E, T);
    b.scratch = c.take<unsigned char>(b.scratch_bytes);
    b.total = b.scratch_bytes ? c.used : 0;
    return b;
}

// starts[k] = first sorted position whose key >= k, k in [0, T]; thread i in [0, E] fills the keys in (key[i-1], key[i]].
__global__ void segment_starts_kernel(const unsigned* __restrict__ keys, long long E, long long T, unsigned* __restrict__ starts) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i > E) return;
    const long long prev = i == 0 ? -1 : (long long)keys[i - 1];
    const long long cur = i == E ? T : min((long long)keys[i], T);
    for (long long k = prev + 1; k <= cur; ++k) starts[k] = (unsigned)i;
}

template <int V> struct VecT;
template <> struct VecT<4> { using T = float4; };
template <> struct VecT<2> { using T = float2; };
__device__ __forceinline__ void fma_rn(float4& a, float w, float4 g) {
    a.x = __fadd_rn(a.x, __fmul_rn(w, g.x)); a.y = __fadd_rn(a.y, __fmul_rn(w, g.y));
    a.z = __fadd_rn(a.z, __fmul_rn(w, g.z)); a.w = __fadd_rn(a.w, __fmul_rn(w, g.w));
}
__device__ __forceinline__ void fma_rn(float2& a, float w, float2 g) {
    a.x = __fadd_rn(a.x, __fmul_rn(w, g.x)); a.y = __fadd_rn(a.y, __fmul_rn(w, g.y));
}

constexpr int kSegVecs = 4;     // vectors per lane held in registers per pass over a segment

// one warp per texel key k in [0, T): map[k][:] = map[k][:] + sum over the segment of w * g[row][:], in sorted order
template <int V>
__global__ void __launch_bounds__(256) segment_reduce_kernel(const unsigned* __restrict__ starts, const unsigned* __restrict__ ids,
                                                             const float* __restrict__ wts, long long T, int C, DetSrc src, DetDst dst) {
    using Vec = typename VecT<V>::T;
    const long long k = (long long)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    if (k >= T) return;
    const int lane = threadIdx.x & 31;
    const unsigned s0 = starts[k], s1 = starts[k + 1];
    if (s0 == s1) return;                                   // no entry reaches this texel: it keeps its value
    // selects instead of indexing the parameter arrays, which would copy them to local memory
    float* map = dst.map[0];
    long long k0 = dst.key0[0];
#pragma unroll
    for (int m = 1; m < kDetMaps; ++m)
        if (k >= dst.key0[m]) { map = dst.map[m]; k0 = dst.key0[m]; }
    Vec* out = reinterpret_cast<Vec*>(map + (size_t)(k - k0) * C);
    const int nvec = C / V;
    for (int q0 = 0; q0 < nvec; q0 += 32 * kSegVecs) {
        Vec acc[kSegVecs];
#pragma unroll
        for (int j = 0; j < kSegVecs; ++j) {
            const int q = q0 + 32 * j + lane;
            if (q < nvec) acc[j] = out[q];
        }
#pragma unroll 4
        for (unsigned i = s0; i < s1; ++i) {
            const unsigned e = ids[i];
            const float w = wts[e];
            const bool sec = e >= src.e0[1];
            const long long row = (long long)(e - (sec ? src.e0[1] : src.e0[0])) / (sec ? src.taps[1] : src.taps[0]);
            const Vec* g = reinterpret_cast<const Vec*>((sec ? src.g[1] : src.g[0]) + row * (sec ? src.ld[1] : src.ld[0]));
#pragma unroll
            for (int j = 0; j < kSegVecs; ++j) {
                const int q = q0 + 32 * j + lane;
                if (q < nvec) fma_rn(acc[j], w, __ldg(g + q));
            }
        }
#pragma unroll
        for (int j = 0; j < kSegVecs; ++j) {
            const int q = q0 + 32 * j + lane;
            if (q < nvec) out[q] = acc[j];
        }
    }
}

int det_sort_reduce(const DetBuffers& b, long long E, long long T, int C, int vec, const DetSrc& src, const DetDst& dst, cudaStream_t s) {
    size_t scratch = b.scratch_bytes;
    NEO_CUDA(cub::DeviceRadixSort::SortPairs(b.scratch, scratch, b.keys, b.keys_sorted, b.ids, b.ids_sorted, (int)E, 0, key_bits(T), s));
    segment_starts_kernel<<<(unsigned)((E + 1 + 255) / 256), 256, 0, s>>>(b.keys_sorted, E, T, b.starts);
    NEO_LAUNCH_CHECK("segment_starts_kernel");
    const unsigned grid = (unsigned)((T + 7) / 8);
    if (vec == 4) segment_reduce_kernel<4><<<grid, 256, 0, s>>>(b.starts, b.ids_sorted, b.wts, T, C, src, dst);
    else segment_reduce_kernel<2><<<grid, 256, 0, s>>>(b.starts, b.ids_sorted, b.wts, T, C, src, dst);
    NEO_LAUNCH_CHECK("segment_reduce_kernel");
    return NEO_OK;
}

// ---- distortion loss: 1/3 sum_i I_i w_i^2 + 2 sum_k (w_k m_k W_<k - w_k (wm)_<k), as written (no |m_i - m_j|) ----
// Exclusive prefix sums over chunks of 32 samples: a Hillis-Steele scan in registers plus the carry of the previous chunks.
__device__ __forceinline__ float warp_incl_scan(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v = __fadd_rn(v, u);
    }
    return v;
}

__device__ __forceinline__ float interval_at(const float* iv, float iv_scalar, long long idx) { return iv ? iv[idx] : iv_scalar; }

__global__ void distortion_kernel(const float* __restrict__ w, const float* __restrict__ m, const float* __restrict__ iv, float iv_scalar,
                                  int n, int N, float* __restrict__ loss) {
    const int ray = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
    if (ray >= n) return;
    const float* wr = w + (size_t)ray * N;
    const float* mr = m + (size_t)ray * N;
    float cw = 0.f, cwm = 0.f, uni = 0.f, bi = 0.f;            // carries W_<chunk, (wm)_<chunk; lane partial sums
    for (int k0 = 0; k0 < N; k0 += 32) {
        const int k = k0 + lane;
        const bool ok = k < N;
        const float wk = ok ? wr[k] : 0.f, mk = ok ? mr[k] : 0.f;
        const float wm = __fmul_rn(wk, mk);
        const float iw = warp_incl_scan(wk, lane), iwm = warp_incl_scan(wm, lane);
        const float W_lt = __fadd_rn(cw, __fsub_rn(iw, wk)), WM_lt = __fadd_rn(cwm, __fsub_rn(iwm, wm));
        if (ok) {
            uni = __fadd_rn(uni, __fmul_rn(interval_at(iv, iv_scalar, (size_t)ray * N + k), __fmul_rn(wk, wk)));
            bi = __fadd_rn(bi, __fsub_rn(__fmul_rn(wm, W_lt), __fmul_rn(wk, WM_lt)));
        }
        cw = __fadd_rn(cw, __shfl_sync(0xffffffffu, iw, 31));
        cwm = __fadd_rn(cwm, __shfl_sync(0xffffffffu, iwm, 31));
    }
    uni = warp_sum(uni);
    bi = warp_sum(bi);
    if (lane == 0) loss[ray] = __fadd_rn(__fmul_rn(1.0f / 3.0f, uni), __fmul_rn(2.0f, bi));
}

// d/dw_i = 2/3 I_i w_i + 2 (m_i W_<i - (wm)_<i + (wm)_>i - m_i W_>i), times the ray's upstream gradient
__global__ void distortion_bwd_kernel(const float* __restrict__ w, const float* __restrict__ m, const float* __restrict__ iv, float iv_scalar,
                                      int n, int N, const float* __restrict__ g_loss, float* __restrict__ d_w) {
    const int ray = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
    if (ray >= n) return;
    const float* wr = w + (size_t)ray * N;
    const float* mr = m + (size_t)ray * N;
    float tw = 0.f, twm = 0.f;
    for (int k = lane; k < N; k += 32) { tw = __fadd_rn(tw, wr[k]); twm = __fadd_rn(twm, __fmul_rn(wr[k], mr[k])); }
    tw = warp_sum(tw);
    twm = warp_sum(twm);
    const float g = g_loss[ray];
    float cw = 0.f, cwm = 0.f;
    for (int k0 = 0; k0 < N; k0 += 32) {
        const int k = k0 + lane;
        const bool ok = k < N;
        const float wk = ok ? wr[k] : 0.f, mk = ok ? mr[k] : 0.f;
        const float wm = __fmul_rn(wk, mk);
        const float iw = warp_incl_scan(wk, lane), iwm = warp_incl_scan(wm, lane);
        const float W_le = __fadd_rn(cw, iw), WM_le = __fadd_rn(cwm, iwm);
        const float W_lt = __fsub_rn(W_le, wk), WM_lt = __fsub_rn(WM_le, wm);
        const float W_gt = __fsub_rn(tw, W_le), WM_gt = __fsub_rn(twm, WM_le);
        if (ok) {
            const float pair = __fadd_rn(__fsub_rn(__fmul_rn(mk, W_lt), WM_lt), __fsub_rn(WM_gt, __fmul_rn(mk, W_gt)));
            const float d = __fadd_rn(__fmul_rn(2.0f / 3.0f, __fmul_rn(interval_at(iv, iv_scalar, (size_t)ray * N + k), wk)), __fmul_rn(2.0f, pair));
            d_w[(size_t)ray * N + k] = __fmul_rn(d, g);
        }
        cw = __fadd_rn(cw, __shfl_sync(0xffffffffu, iw, 31));
        cwm = __fadd_rn(cwm, __shfl_sync(0xffffffffu, iwm, 31));
    }
}

// ---- interlevel loss of one proposal level (helper.py:117-141 via mip._outer_weights) ----
// r = searchsorted(t_env, t, right=True) = the number of t_env knots <= t;  lo = max(r-1, 0), hi = min(r, Np)
__device__ __forceinline__ int count_le(const float* te, int len, float x) {
    int a = 0, b = len;
    while (a < b) {
        const int mid = (a + b) >> 1;
        if (te[mid] <= x) a = mid + 1; else b = mid;
    }
    return a;
}
// w_outer_j = sum of w_env over [lo_j, hi_{j+1}) in ascending order
__device__ __forceinline__ void outer_range(const float* t, const float* te, int Np, int j, int& lo, int& hi) {
    lo = max(count_le(te, Np + 1, t[j]) - 1, 0);
    hi = min(count_le(te, Np + 1, t[j + 1]), Np);
}
constexpr float kInterEps = 1.1920929e-07f;

__global__ void interlevel_kernel(const float* __restrict__ t, const float* __restrict__ w, const float* __restrict__ te,
                                  const float* __restrict__ we, int n, int Nc, int Np, float* __restrict__ loss) {
    const int ray = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
    if (ray >= n) return;
    const float *tr = t + (size_t)ray * (Nc + 1), *wr = w + (size_t)ray * Nc, *ter = te + (size_t)ray * (Np + 1), *wer = we + (size_t)ray * Np;
    float part = 0.f;
    for (int j = lane; j < Nc; j += 32) {
        int lo, hi;
        outer_range(tr, ter, Np, j, lo, hi);
        float wo = 0.f;
        for (int k = lo; k < hi; ++k) wo = __fadd_rn(wo, wer[k]);
        const float c = fmaxf(__fsub_rn(wr[j], wo), 0.f);
        part = __fadd_rn(part, __fdiv_rn(__fmul_rn(c, c), __fadd_rn(wr[j], kInterEps)));
    }
    part = warp_sum(part);
    if (lane == 0) loss[ray] = __fdiv_rn(part, (float)Nc);
}

// d w_env[k] = sum over the j whose range [lo_j, hi_{j+1}) holds k of -2 clip(w_j - w_outer_j, 0) / (w_j + eps) / Nc, times g
__global__ void interlevel_bwd_kernel(const float* __restrict__ t, const float* __restrict__ w, const float* __restrict__ te,
                                      const float* __restrict__ we, int n, int Nc, int Np, const float* __restrict__ g_loss, float* __restrict__ d_we) {
    extern __shared__ float sm[];
    const int wid = threadIdx.x / 32, lane = threadIdx.x & 31;
    const int ray = blockIdx.x * (blockDim.x / 32) + wid;
    if (ray >= n) return;
    float* dwo = sm + (size_t)wid * Nc;
    int* rng = reinterpret_cast<int*>(sm + (size_t)(blockDim.x / 32) * Nc) + (size_t)wid * 2 * Nc;
    const float *tr = t + (size_t)ray * (Nc + 1), *wr = w + (size_t)ray * Nc, *ter = te + (size_t)ray * (Np + 1), *wer = we + (size_t)ray * Np;
    const float g = __fdiv_rn(g_loss[ray], (float)Nc);
    for (int j = lane; j < Nc; j += 32) {
        int lo, hi;
        outer_range(tr, ter, Np, j, lo, hi);
        float wo = 0.f;
        for (int k = lo; k < hi; ++k) wo = __fadd_rn(wo, wer[k]);
        const float c = fmaxf(__fsub_rn(wr[j], wo), 0.f);
        dwo[j] = __fmul_rn(__fdiv_rn(__fmul_rn(-2.0f, c), __fadd_rn(wr[j], kInterEps)), g);
        rng[2 * j] = lo;
        rng[2 * j + 1] = hi;
    }
    __syncwarp();
    for (int k = lane; k < Np; k += 32) {
        float acc = 0.f;
        for (int j = 0; j < Nc; ++j)
            if (rng[2 * j] <= k && k < rng[2 * j + 1]) acc = __fadd_rn(acc, dwo[j]);
        d_we[(size_t)ray * Np + k] = acc;
    }
}

// ---- adjoint of upsample_bilinear2d(align_corners=True) ----
// The forward's source row of output row o: h1r = scale * o (scale = (in-1)/(out-1), 0 for out == 1), h1 = (int)h1r,
// h1p = h1 < in-1, lambda1 = h1r - h1, lambda0 = 1 - lambda1 (ATen UpSampleBilinear2d.cu).
struct Tap1 { int h1, h1p; float l0, l1; };
__device__ __forceinline__ Tap1 up_tap(float scale, int o, int in) {
    const float r = __fmul_rn(scale, (float)o);
    Tap1 t;
    t.h1 = (int)r;
    t.h1p = t.h1 < in - 1 ? 1 : 0;
    t.l1 = __fsub_rn(r, (float)t.h1);
    t.l0 = __fsub_rn(1.0f, t.l1);
    return t;
}
// weight of input index y in output index o
__device__ __forceinline__ float up_weight(const Tap1& t, int y) {
    return (t.h1 == y ? t.l0 : 0.f) + (t.h1 + t.h1p == y ? t.l1 : 0.f);
}
// first output index o in [0, out] with h1(o) >= y (h1 is non-decreasing in o)
__device__ __forceinline__ int first_h1_ge(float scale, int in, int out, int y) {
    int a = 0, b = out;
    while (a < b) {
        const int mid = (a + b) >> 1;
        if (up_tap(scale, mid, in).h1 >= y) b = mid; else a = mid + 1;
    }
    return a;
}

// g_in[p][y][x] = sum over o_y in [first_h1_ge(y-1), first_h1_ge(y+1)) of wy * (sum over o_x in the same range along x of wx * g_out)
__global__ void upsample_bwd_kernel(const float* __restrict__ g_out, long long planes, int Hi, int Wi, int Ho, int Wo, float sh, float sw,
                                    float* __restrict__ g_in) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= planes * Hi * Wi) return;
    const int x = (int)(i % Wi), y = (int)((i / Wi) % Hi);
    const long long p = i / ((long long)Hi * Wi);
    const int oy0 = first_h1_ge(sh, Hi, Ho, y - 1), oy1 = first_h1_ge(sh, Hi, Ho, y + 1);
    const int ox0 = first_h1_ge(sw, Wi, Wo, x - 1), ox1 = first_h1_ge(sw, Wi, Wo, x + 1);
    const float* g = g_out + p * Ho * Wo;
    float acc = 0.f;
    for (int oy = oy0; oy < oy1; ++oy) {
        const float wy = up_weight(up_tap(sh, oy, Hi), y);
        if (wy == 0.f) continue;
        float row = 0.f;
        for (int ox = ox0; ox < ox1; ++ox) {
            const float wx = up_weight(up_tap(sw, ox, Wi), x);
            if (wx != 0.f) row = __fadd_rn(row, __fmul_rn(wx, g[(long long)oy * Wo + ox]));
        }
        acc = __fadd_rn(acc, __fmul_rn(wy, row));
    }
    g_in[i] = acc;
}

}  // namespace neo

using namespace neo;

extern "C" int neo_distortion_loss(const float* w, const float* m, const float* interval, float interval_scalar, int n, int N, float* loss,
                                   void* stream) {
    if (!w || !m || !loss || n < 1 || N < 1) { set_error("neo_distortion_loss: NULL w / m / loss, or n, N < 1"); return NEO_ERR_INVALID; }
    distortion_kernel<<<(unsigned)((n + 7) / 8), 256, 0, (cudaStream_t)stream>>>(w, m, interval, interval_scalar, n, N, loss);
    NEO_LAUNCH_CHECK("distortion_kernel");
    return NEO_OK;
}

extern "C" int neo_distortion_loss_bwd(const float* w, const float* m, const float* interval, float interval_scalar, int n, int N,
                                       const float* g_loss, float* d_w, void* stream) {
    if (!w || !m || !g_loss || !d_w || n < 1 || N < 1) {
        set_error("neo_distortion_loss_bwd: NULL w / m / g_loss / d_w, or n, N < 1");
        return NEO_ERR_INVALID;
    }
    distortion_bwd_kernel<<<(unsigned)((n + 7) / 8), 256, 0, (cudaStream_t)stream>>>(w, m, interval, interval_scalar, n, N, g_loss, d_w);
    NEO_LAUNCH_CHECK("distortion_bwd_kernel");
    return NEO_OK;
}

static bool interlevel_args_ok(const char* who, const float* t, const float* w, const float* te, const float* we, int n, int Nc, int Np) {
    if (!t || !w || !te || !we || n < 1 || Nc < 1 || Np < 1 || Nc > 1024) {
        set_error("%s: NULL input, n or Np < 1, or Nc outside [1, 1024]", who);
        return false;
    }
    return true;
}

extern "C" int neo_interlevel_loss(const float* sdist, const float* weights, const float* sdist_env, const float* weights_env, int n, int Nc,
                                   int Np, float* loss, void* stream) {
    if (!interlevel_args_ok("neo_interlevel_loss", sdist, weights, sdist_env, weights_env, n, Nc, Np)) return NEO_ERR_INVALID;
    if (!loss) { set_error("neo_interlevel_loss: NULL loss"); return NEO_ERR_INVALID; }
    interlevel_kernel<<<(unsigned)((n + 7) / 8), 256, 0, (cudaStream_t)stream>>>(sdist, weights, sdist_env, weights_env, n, Nc, Np, loss);
    NEO_LAUNCH_CHECK("interlevel_kernel");
    return NEO_OK;
}

extern "C" int neo_interlevel_loss_bwd(const float* sdist, const float* weights, const float* sdist_env, const float* weights_env, int n, int Nc,
                                       int Np, const float* g_loss, float* d_weights_env, void* stream) {
    if (!interlevel_args_ok("neo_interlevel_loss_bwd", sdist, weights, sdist_env, weights_env, n, Nc, Np)) return NEO_ERR_INVALID;
    if (!g_loss || !d_weights_env) { set_error("neo_interlevel_loss_bwd: NULL g_loss / d_weights_env"); return NEO_ERR_INVALID; }
    const int warps = 4;
    const size_t smem = (size_t)warps * Nc * 3 * sizeof(float);
    interlevel_bwd_kernel<<<(unsigned)((n + warps - 1) / warps), 32 * warps, smem, (cudaStream_t)stream>>>(sdist, weights, sdist_env, weights_env,
                                                                                                           n, Nc, Np, g_loss, d_weights_env);
    NEO_LAUNCH_CHECK("interlevel_bwd_kernel");
    return NEO_OK;
}

extern "C" int neo_upsample_bilinear_bwd(const float* g_out, long long planes, int H_in, int W_in, int H_out, int W_out, float* g_in,
                                         void* stream) {
    if (!g_out || !g_in || planes < 1 || H_in < 1 || W_in < 1 || H_out < 1 || W_out < 1) {
        set_error("neo_upsample_bilinear_bwd: NULL buffer or a size < 1");
        return NEO_ERR_INVALID;
    }
    // area_pixel_compute_scale(align_corners=True): (in - 1) / (out - 1) in fp32, 0 for a single output row / column
    const float sh = H_out > 1 ? (float)(H_in - 1) / (float)(H_out - 1) : 0.f;
    const float sw = W_out > 1 ? (float)(W_in - 1) / (float)(W_out - 1) : 0.f;
    const long long total = planes * H_in * W_in;
    upsample_bwd_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(g_out, planes, H_in, W_in, H_out, W_out, sh, sw, g_in);
    NEO_LAUNCH_CHECK("upsample_bwd_kernel");
    return NEO_OK;
}
