// Per-scene state: channel-last feature maps, source-camera transforms, fp32 weight transposes.
// Consumes the outputs of the (out-of-scope) encoder: encoder_tp_fusion_conv.py:585-595 (planes),
// encoder_pn.py:203-206 (latent + latent_scaling); cameras per util.py:52-70.
#include "common.cuh"
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <map>
#include <mutex>
#include <utility>

namespace neo {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
int cuda_fail(cudaError_t e, const char* what) {
    set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
    return NEO_ERR_CUDA;
}
const char* last_error() { return g_err; }

// (n, C, HW) -> (n, HW, C), tiled through shared memory so both sides are coalesced
template <class T>
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ in, T* __restrict__ out, int C, int HW) {
    __shared__ float tile[32][33];
    int n = blockIdx.z;
    int c0 = blockIdx.y * 32, p0 = blockIdx.x * 32;
    const float* src = in + (size_t)n * C * HW;
    T* dst = out + (size_t)n * C * HW;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int c = c0 + i, p = p0 + threadIdx.x;
        if (c < C && p < HW) tile[i][threadIdx.x] = src[(size_t)c * HW + p];
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int p = p0 + i, c = c0 + threadIdx.x;
        if (c < C && p < HW) dst[(size_t)p * C + c] = from_f32<T>(tile[threadIdx.x][i]);
    }
}

template <class T>
static int nchw_to_nhwc(const float* in, T* out, int n, int C, int HW, cudaStream_t s) {
    dim3 grid((HW + 31) / 32, (C + 31) / 32, n), block(32, 8);
    nchw_to_nhwc_kernel<T><<<grid, block, 0, s>>>(in, out, C, HW);
    NEO_LAUNCH_CHECK("nchw_to_nhwc_kernel");
    return NEO_OK;
}
int launch_nchw_to_nhwc(const float* in, float* out, int n, int C, int HW, cudaStream_t s) { return nchw_to_nhwc(in, out, n, C, HW, s); }
int launch_nchw_to_nhwc(const float* in, __half* out, int n, int C, int HW, cudaStream_t s) { return nchw_to_nhwc(in, out, n, C, HW, s); }

// (out,in) -> (in,out)
__global__ void transpose_kernel(const float* __restrict__ w, float* __restrict__ wt, int out_f, int in_f) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= out_f * in_f) return;
    int o = idx / in_f, i = idx % in_f;
    wt[(size_t)i * out_f + o] = w[idx];
}

int launch_transpose(const float* w, float* wt, int out_f, int in_f, cudaStream_t s) {
    int n = out_f * in_f;
    transpose_kernel<<<(n + 255) / 256, 256, 0, s>>>(w, wt, out_f, in_f);
    NEO_LAUNCH_CHECK("transpose_kernel");
    return NEO_OK;
}

__global__ void view_xform_kernel(const float* __restrict__ poses, int nv, ViewXform* __restrict__ out) {
    int v = threadIdx.x;
    if (v >= nv) return;
    const float* m = poses + 16 * v;
    ViewXform x;
    // rot = c2w[:3,:3]^T ; trans = -(rot @ c2w[:3,3])   (util.py:64-66)
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) x.rt[r * 3 + c] = m[c * 4 + r];
    for (int r = 0; r < 3; ++r)
        x.tr[r] = -fmaf(x.rt[r * 3 + 2], m[11], fmaf(x.rt[r * 3 + 1], m[7], x.rt[r * 3 + 0] * m[3]));
    for (int k = 0; k < 4; ++k) x.pad[k] = 0.f;
    out[v] = x;
}

__global__ void scalar_fetch_kernel(const float* focal, const float* c, float* out) {
    out[0] = focal[0]; out[1] = c[0]; out[2] = c[1];
}

// ---- block pool ----
namespace {
struct BlockPool {
    std::mutex mu;
    std::multimap<std::pair<int, size_t>, void*> free_blocks;     // (device, bytes) -> block
    size_t held = 0;
};
BlockPool g_pool;
constexpr size_t kPoolCap = 6ull << 30;       // bytes kept across all devices; beyond it blocks go back to the driver
constexpr size_t kPoolMinBlock = 1 << 16;     // small blocks are not worth keeping
}  // namespace

int pool_alloc(void** p, size_t bytes) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (bytes >= kPoolMinBlock) {
        std::lock_guard<std::mutex> lk(g_pool.mu);
        auto it = g_pool.free_blocks.find({dev, bytes});
        if (it != g_pool.free_blocks.end()) {
            *p = it->second;
            g_pool.free_blocks.erase(it);
            g_pool.held -= bytes;
            return NEO_OK;
        }
    }
    cudaError_t e = cudaMalloc(p, bytes);
    if (e != cudaSuccess) {                   // give the cached blocks back and retry once
        cudaGetLastError();
        neo_release_cached();
        e = cudaMalloc(p, bytes);
    }
    if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc(scene)");
    return NEO_OK;
}

// The caller guarantees that no kernel still uses the block (neo_scene_free synchronises the device first, as cudaFree would).
void pool_release(void* p, size_t bytes) {
    if (!p) return;
    int dev = 0;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) == cudaSuccess) dev = at.device; else cudaGetLastError();
    {
        std::lock_guard<std::mutex> lk(g_pool.mu);
        if (bytes >= kPoolMinBlock && g_pool.held + bytes <= kPoolCap) {
            g_pool.free_blocks.insert({{dev, bytes}, p});
            g_pool.held += bytes;
            return;
        }
    }
    cudaFree(p);
}

template <typename T>
static int dev_alloc(NeoScene* sc, T** p, size_t count) {
    void* q = nullptr;
    int rc = pool_alloc(&q, count * sizeof(T));
    if (rc) return rc;
    sc->allocations.push_back({q, count * sizeof(T)});
    sc->bytes += count * sizeof(T);
    *p = reinterpret_cast<T*>(q);
    return NEO_OK;
}

int scene_alloc_bytes(NeoScene* sc, void** p, size_t bytes) {
    unsigned char* q = nullptr;
    int rc = dev_alloc(sc, &q, bytes);
    *p = q;
    return rc;
}

static int transpose_to(NeoScene* sc, const float* w, int out_f, int in_f, const float** dst, cudaStream_t s) {
    float* t = nullptr;
    int rc = dev_alloc(sc, &t, (size_t)out_f * in_f);
    if (rc || (rc = launch_transpose(w, t, out_f, in_f, s))) return rc;
    *dst = t;
    return NEO_OK;
}

static int to_channel_last(NeoScene* sc, const float* src, int n, int C, int HW, const float** dst, cudaStream_t s) {
    float* t = nullptr;
    int rc = dev_alloc(sc, &t, (size_t)n * C * HW);
    if (rc || (rc = launch_nchw_to_nhwc(src, t, n, C, HW, s))) return rc;
    *dst = t;
    return NEO_OK;
}

}  // namespace neo

using namespace neo;

extern "C" int neo_scene_create(const NeoSceneDesc* d, const NeoMLPParams mlps[4], int precision_mask, NeoScene** out,
                                void* stream) {
    if (!d || !mlps || !out) { set_error("neo_scene_create: null argument"); return NEO_ERR_INVALID; }
    if (d->nv < 1 || d->nv > kMaxViews || d->world_ch != kWorldCh || d->local_ch != kLocalCh) {
        set_error("neo_scene_create: need 1..%d views, world_ch=128, local_ch=512 (got nv=%d world=%d local=%d)", kMaxViews,
                  d->nv, d->world_ch, d->local_ch);
        return NEO_ERR_UNSUPPORTED;
    }
    if (d->plane_h < 2 || d->plane_w < 2 || d->lat_h < 2 || d->lat_w < 2) {
        set_error("neo_scene_create: feature maps must be at least 2x2");
        return NEO_ERR_INVALID;
    }
    if (d->img_w <= 0 || d->img_h <= 0) {
        set_error("neo_scene_create: img_w / img_h must be positive (got %d x %d)", d->img_w, d->img_h);
        return NEO_ERR_INVALID;
    }
    if (!d->planes_xz || !d->planes_xy || !d->planes_yz || !d->latent || !d->src_poses || !d->src_focal || !d->src_c) {
        set_error("neo_scene_create: null feature map / camera pointer");
        return NEO_ERR_INVALID;
    }
    if (precision_mask & ~((1 << NEO_PREC_FP32) | (1 << NEO_PREC_TC))) {
        set_error("neo_scene_create: unknown bits in the precision mask (%d)", precision_mask);
        return NEO_ERR_INVALID;
    }
    // precision_mask == 0: cameras and grid geometry only (neo_index_maps* of the training path); rendering such a scene is an error
    cudaStream_t s = (cudaStream_t)stream;
    NeoScene* sc = new NeoScene();
    sc->desc = *d;
    sc->precision_mask = precision_mask;
    sc->tc_state = nullptr;
    sc->bytes = 0;
    int rc = NEO_OK;
    auto fail = [&](int code) { neo_scene_free(sc); return code; };

    SceneDev& dv = sc->dev;
    dv.nv = d->nv; dv.plane_h = d->plane_h; dv.plane_w = d->plane_w; dv.lat_h = d->lat_h; dv.lat_w = d->lat_w;
    dv.img_w = d->img_w; dv.img_h = d->img_h;
    // latent_scaling = size / (size - 1) * 2 ; scale = latent_scaling / image_size   (fp32, encoder_pn.py:119,204-206)
    float lsx = (float)d->lat_w / ((float)d->lat_w - 1.0f) * 2.0f;
    float lsy = (float)d->lat_h / ((float)d->lat_h - 1.0f) * 2.0f;
    dv.lat_scale_x = lsx / (float)d->img_w;
    dv.lat_scale_y = lsy / (float)d->img_h;

    ViewXform* views = nullptr;
    if ((rc = dev_alloc(sc, &views, d->nv))) return fail(rc);
    view_xform_kernel<<<1, 32, 0, s>>>(d->src_poses, d->nv, views);
    dv.views = views;
    float* scal = nullptr;
    if ((rc = dev_alloc(sc, &scal, 4))) return fail(rc);
    scalar_fetch_kernel<<<1, 1, 0, s>>>(d->src_focal, d->src_c, scal);
    float h[3];
    cudaError_t e = cudaMemcpyAsync(h, scal, 3 * sizeof(float), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return fail(cuda_fail(e, "scene scalars"));
    dv.focal = h[0]; dv.cx = h[1]; dv.cy = h[2];
    if ((rc = dev_alloc(sc, &sc->err_flag, 1))) return fail(rc);
    if ((e = cudaMemsetAsync(sc->err_flag, 0, sizeof(int), s)) != cudaSuccess) return fail(cuda_fail(e, "memset"));

    dv.latent_cl = nullptr;
    dv.planes_cl[0] = dv.planes_cl[1] = dv.planes_cl[2] = nullptr;
    if (precision_mask & (1 << NEO_PREC_FP32)) {
        const float* planes[3] = {d->planes_xz, d->planes_xy, d->planes_yz};
        for (int i = 0; i < 3; ++i)
            if ((rc = to_channel_last(sc, planes[i], d->nv, kWorldCh, d->plane_h * d->plane_w, &dv.planes_cl[i], s)))
                return fail(rc);
        if ((rc = to_channel_last(sc, d->latent, d->nv, kLocalCh, d->lat_h * d->lat_w, &dv.latent_cl, s))) return fail(rc);
        for (int i = 0; i < 4; ++i) {
            const NeoMLPParams& p = mlps[i];
            MLPFp32& m = sc->mlp32[i];
            if (p.in_ch != 3 && p.in_ch != 4) { set_error("mlp %d: in_ch must be 3 or 4", i); return fail(NEO_ERR_INVALID); }
            m.in_ch = p.in_ch;
            m.enc_dim = p.in_ch * (2 * kPosDeg + 1);
            m.in_dim = m.enc_dim + kLocalCh + kWorldCh;
            if ((rc = transpose_to(sc, p.w0, kHidden, m.in_dim, &m.w0t, s))) return fail(rc);
            if ((rc = transpose_to(sc, p.w1, kHidden, kHidden, &m.w1t, s))) return fail(rc);
            if ((rc = transpose_to(sc, p.w2, kHidden, kHidden, &m.w2t, s))) return fail(rc);
            if ((rc = transpose_to(sc, p.w3, kHidden, kHidden + m.in_dim, &m.w3t, s))) return fail(rc);
            if ((rc = transpose_to(sc, p.wb, kHidden, kHidden, &m.wbt, s))) return fail(rc);
            if ((rc = transpose_to(sc, p.wv0, 64, kHidden + kDirEnc, &m.wv0t, s))) return fail(rc);
            if ((rc = transpose_to(sc, p.wv1, 64, 64, &m.wv1t, s))) return fail(rc);
            m.b0 = p.b0; m.b1 = p.b1; m.b2 = p.b2; m.b3 = p.b3; m.bb = p.bb; m.wsig = p.wsig; m.bsig = p.bsig;
            m.bv0 = p.bv0; m.bv1 = p.bv1; m.wrgb = p.wrgb; m.brgb = p.brgb;
            // small vectors are copied so the scene does not alias caller memory after creation
            const float** small[] = {&m.b0, &m.b1, &m.b2, &m.b3, &m.bb, &m.wsig, &m.bsig, &m.bv0, &m.bv1, &m.wrgb, &m.brgb};
            const int sizes[] = {128, 128, 128, 128, 128, 128, 1, 64, 64, 192, 3};
            for (int k = 0; k < 11; ++k) {
                float* c = nullptr;
                if ((rc = dev_alloc(sc, &c, sizes[k]))) return fail(rc);
                e = cudaMemcpyAsync(c, *small[k], sizes[k] * sizeof(float), cudaMemcpyDeviceToDevice, s);
                if (e != cudaSuccess) return fail(cuda_fail(e, "copy bias"));
                *small[k] = c;
            }
        }
    }
    if (precision_mask & (1 << NEO_PREC_TC)) {
        if ((rc = tc_scene_create(sc, mlps, s))) return fail(rc);
    }
    e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return fail(cuda_fail(e, "neo_scene_create sync"));
    *out = sc;
    return NEO_OK;
}

extern "C" void neo_scene_free(NeoScene* sc) {
    if (!sc) return;
    tc_scene_free(sc);
    cudaDeviceSynchronize();                       // what cudaFree would do implicitly: nothing may still read the blocks
    for (auto& a : sc->allocations) pool_release(a.first, a.second);
    delete sc;
}

extern "C" void neo_release_cached(void) {
    std::vector<void*> blocks;
    {
        std::lock_guard<std::mutex> lk(g_pool.mu);
        for (auto& kv : g_pool.free_blocks) blocks.push_back(kv.second);
        g_pool.free_blocks.clear();
        g_pool.held = 0;
    }
    for (void* p : blocks) cudaFree(p);
}

extern "C" size_t neo_scene_bytes(const NeoScene* sc) { return sc ? sc->bytes : 0; }

namespace neo { const char* last_error(); }
extern "C" const char* neo_last_error(void) { return neo::last_error(); }
extern "C" const char* neo_version(void) { return "neo360_b200 0.1.0 sm_90a"; }
