// Orchestration of one NeRF_TP.forward (models/neo360/model.py:266-581, encoder hoisted) plus the
// stage-level C-ABI wrappers.  Per level: sample -> field(fg), field(bg) -> composite x2 -> combine.
// All intermediates live in the caller-provided workspace; nothing is allocated here.
#include "common.cuh"

using namespace neo;

namespace {

struct WS {
    float *far, *t0[2], *w0[2], *t1[2], *w1[2], *sig[2], *rgb[2];
    float *c[2], *acc[2], *lam, *dep[2];
    unsigned char* dir;      // NEO_PREC_TC: direction fragments of every ray (launch_dir_frags), shared by the four field launches
};

size_t carve(Carve& cv, int n, int N0, int N1, WS& w) {
    w.far = cv.take<float>(n);
    for (int b = 0; b < 2; ++b) {
        w.t0[b] = cv.take<float>((size_t)n * N0);
        w.w0[b] = cv.take<float>((size_t)n * N0);
        w.t1[b] = cv.take<float>((size_t)n * N1);
        w.w1[b] = cv.take<float>((size_t)n * N1);
        w.sig[b] = cv.take<float>((size_t)n * N1);
        w.rgb[b] = cv.take<float>((size_t)n * N1 * 3);
        w.c[b] = cv.take<float>((size_t)n * 3);
        w.acc[b] = cv.take<float>(n);
        w.dep[b] = cv.take<float>(n);
    }
    w.lam = cv.take<float>(n);
    w.dir = cv.take<unsigned char>((size_t)n * kDirFragBytes);
    return cv.used;
}

int check_cfg(const NeoCfg* cfg) {
    if (!cfg) { set_error("null cfg"); return NEO_ERR_INVALID; }
    if (cfg->n_coarse < 3 || cfg->n_fine < 1 || cfg->n_coarse > 4096 || cfg->n_fine > 4096) {
        set_error("n_coarse must be in [3,4096], n_fine in [1,4096] (got %d, %d)", cfg->n_coarse, cfg->n_fine);
        return NEO_ERR_INVALID;
    }
    if (cfg->precision != NEO_PREC_FP32 && cfg->precision != NEO_PREC_TC) { set_error("bad precision %d", cfg->precision); return NEO_ERR_INVALID; }
    return NEO_OK;
}

// ---- optional profiling: CUDA events around every field-kernel launch, on the launching stream ----
struct Prof {
    bool on = false;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pool;
    size_t used = 0;
    unsigned long long launches = 0;     // kernels launched by this library since the last reset
    double field_points = 0;             // (ray, sample) points pushed through field kernels
} g_prof;

int field(const NeoScene* sc, const NeoRays* rays, const float* far, const float* t, int N, int mi, int prec, const void* dir,
          float* rgb, float* sigma, cudaStream_t s) {
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (g_prof.on) {
        if (g_prof.used == g_prof.pool.size()) {
            cudaEvent_t a, b;
            NEO_CUDA(cudaEventCreate(&a));
            NEO_CUDA(cudaEventCreate(&b));
            g_prof.pool.emplace_back(a, b);
        }
        e0 = g_prof.pool[g_prof.used].first;
        e1 = g_prof.pool[g_prof.used].second;
        g_prof.used++;
        NEO_CUDA(cudaEventRecord(e0, s));
    }
    int rc = (prec == NEO_PREC_FP32) ? launch_field_fp32(sc, rays, far, t, N, mi, rgb, sigma, s)
                                     : launch_field_tc(sc, rays, far, t, N, mi, dir, rgb, sigma, s);
    if (g_prof.on && e1) NEO_CUDA(cudaEventRecord(e1, s));
    g_prof.launches += 1;
    g_prof.field_points += (double)rays->n_rays * N;
    return rc;
}

}  // namespace

extern "C" size_t neo_render_workspace_bytes(int n_rays, const NeoCfg* cfg) {
    if (n_rays <= 0 || check_cfg(cfg)) return 0;
    Carve cv{nullptr, 0};
    WS w;
    return carve(cv, n_rays, cfg->n_coarse + 1, cfg->n_coarse + 1 + cfg->n_fine, w);
}

extern "C" int neo_render_fwd(const NeoScene* sc, const NeoRays* rays, const NeoCfg* cfg, NeoOut* out, void* workspace,
                              size_t workspace_bytes, void* stream) {
    if (!sc || !rays || !out) { set_error("neo_render_fwd: null argument"); return NEO_ERR_INVALID; }
    int rc = check_cfg(cfg);
    if (rc) return rc;
    if (rays->n_rays <= 0 || !rays->rays_o || !rays->rays_d || !rays->viewdirs) { set_error("neo_render_fwd: empty rays"); return NEO_ERR_INVALID; }
    if (!(sc->precision_mask & (1 << cfg->precision))) { set_error("scene not prepared for precision %d", cfg->precision); return NEO_ERR_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    const int n = rays->n_rays, N0 = cfg->n_coarse + 1, N1 = N0 + cfg->n_fine;
    Carve cv{static_cast<unsigned char*>(workspace), 0};
    WS w;
    size_t need = carve(cv, n, N0, N1, w);
    if (!workspace || workspace_bytes < need) { set_error("workspace too small: need %zu bytes, got %zu", need, workspace_bytes); return NEO_ERR_WORKSPACE; }

    if ((rc = launch_far(rays->rays_o, rays->rays_d, n, w.far, sc->err_flag, s))) return rc;
    g_prof.launches += 1 + 2 * (2 + 2 + 1);      // far + per level: 2 sampling, 2 composite, 1 combine (field counted in field())
    if (cfg->precision == NEO_PREC_TC) {
        if ((rc = launch_dir_frags(sc, rays, w.dir, s))) return rc;
        g_prof.launches += 1;
    }
    const int white = cfg->out_depth ? 0 : cfg->white_bkgd;       // model.py:501,519 vs 551,560
    for (int lvl = 0; lvl < 2; ++lvl) {
        const int N = lvl ? N1 : N0;
        float* t[2] = {lvl ? w.t1[0] : w.t0[0], lvl ? w.t1[1] : w.t0[1]};
        float* wt[2] = {lvl ? w.w1[0] : w.w0[0], lvl ? w.w1[1] : w.w0[1]};
        if (lvl == 0) {
            if ((rc = launch_sample_coarse(rays->rays_o, rays->rays_d, w.far, n, cfg->n_coarse, 1, 3.0f, cfg->u_fg0, t[0], nullptr, nullptr, s))) return rc;
            if ((rc = launch_sample_coarse(rays->rays_o, rays->rays_d, w.far, n, cfg->n_coarse, 0, 3.0f, cfg->u_bg0, t[1], nullptr, nullptr, s))) return rc;
        } else {
            if ((rc = launch_resample(rays->rays_o, rays->rays_d, w.far, w.t0[0], w.w0[0], n, N0, cfg->n_fine, 1, 3.0f, cfg->u_fg1, t[0], nullptr, nullptr, s))) return rc;
            if ((rc = launch_resample(rays->rays_o, rays->rays_d, w.far, w.t0[1], w.w0[1], n, N0, cfg->n_fine, 0, 3.0f, cfg->u_bg1, t[1], nullptr, nullptr, s))) return rc;
        }
        for (int b = 0; b < 2; ++b)
            if ((rc = field(sc, rays, w.far, t[b], N, 2 * lvl + b, cfg->precision, w.dir, w.rgb[b], w.sig[b], s))) return rc;
        if ((rc = launch_composite(w.rgb[0], w.sig[0], t[0], rays->rays_d, w.far, n, N, white, 1, w.c[0], w.acc[0], wt[0], w.lam, w.dep[0], s))) return rc;
        if ((rc = launch_composite(w.rgb[1], w.sig[1], t[1], rays->rays_d, w.far, n, N, white, 0, w.c[1], w.acc[1], wt[1], nullptr, w.dep[1], s))) return rc;
        if ((rc = launch_combine(n, N, w.c[0], w.c[1], w.lam, w.dep[0], w.dep[1], t[0], t[1], out->comp_rgb[lvl],
                                 out->depth[lvl], out->fg_sdist[lvl], out->bg_sdist[lvl], s))) return rc;
        if ((rc = copy_out(out->fg_rgb[lvl], w.c[0], (size_t)n * 3, s))) return rc;
        if ((rc = copy_out(out->bg_rgb[lvl], w.c[1], (size_t)n * 3, s))) return rc;
        if ((rc = copy_out(out->fg_acc[lvl], w.acc[0], n, s))) return rc;
        if ((rc = copy_out(out->bg_acc[lvl], w.acc[1], n, s))) return rc;
        if ((rc = copy_out(out->bg_lambda[lvl], w.lam, n, s))) return rc;
        if ((rc = copy_out(out->fg_w[lvl], wt[0], (size_t)n * N, s))) return rc;
        if ((rc = copy_out(out->bg_w[lvl], wt[1], (size_t)n * N, s))) return rc;
        if ((rc = copy_out(out->fg_t[lvl], t[0], (size_t)n * N, s))) return rc;
        if ((rc = copy_out(out->bg_s[lvl], t[1], (size_t)n * N, s))) return rc;
        if ((rc = copy_out(out->fg_sigma[lvl], w.sig[0], (size_t)n * N, s))) return rc;
        if ((rc = copy_out(out->bg_sigma[lvl], w.sig[1], (size_t)n * N, s))) return rc;
        if ((rc = copy_out(out->fg_rgb_s[lvl], w.rgb[0], (size_t)n * N * 3, s))) return rc;
        if ((rc = copy_out(out->bg_rgb_s[lvl], w.rgb[1], (size_t)n * N * 3, s))) return rc;
    }
    return NEO_OK;
}

namespace neo { const char* tc_trap_info(); }
extern "C" int neo_check_async(const NeoScene* sc, void* stream) {
    if (!sc) { set_error("null scene"); return NEO_ERR_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    int flag = 0;
    NEO_CUDA(cudaMemcpyAsync(&flag, sc->err_flag, sizeof(int), cudaMemcpyDeviceToHost, s));
    NEO_CUDA(cudaStreamSynchronize(s));
    if (flag) {
        cudaMemsetAsync(sc->err_flag, 0, sizeof(int), s);
        set_error("1.0 - p_norm_sq should be greater than 0: a ray misses the unit sphere (helper.py:271)");
        return NEO_ERR_GEOMETRY;
    }
    return NEO_OK;
}

// ---- stage-level entry points ----
namespace {
// index_bwd_kernel reads its row gradients and reduces into the gradient maps as float4 (16-byte vector atomics)
bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
}  // namespace
extern "C" int neo_get_rays(int H, int W, float focal, const float* c2w, float* o, float* vd, float* rd, float* radii, void* stream) {
    if (H < 2 || W < 1 || !c2w) { set_error("neo_get_rays: bad arguments"); return NEO_ERR_INVALID; }
    return launch_get_rays(H, W, focal, c2w, o, vd, rd, radii, (cudaStream_t)stream);
}
extern "C" int neo_sample_rays(int n, const long long* pix_inds, int n_views, int H, int W, float focal, const float* c2w,
                               const float* images, float* rays_o, float* viewdirs, float* rays_d, float* radii, float* target,
                               int* err_flag, void* stream) {
    if (n == 0) return NEO_OK;                     // an empty batch is valid (and its buffers may be null)
    if (n < 0 || n_views < 1 || H < 2 || W < 1 || !pix_inds || !c2w || !err_flag || (target && !images)) {
        set_error("neo_sample_rays: bad arguments");
        return NEO_ERR_INVALID;
    }
    return launch_sample_rays(n, pix_inds, n_views, H, W, focal, c2w, images, rays_o, viewdirs, rays_d, radii, target, err_flag,
                              (cudaStream_t)stream);
}
extern "C" int neo_intersect_sphere(const float* o, const float* d, int n, float* far, int* err_flag, void* stream) {
    if (n <= 0) { set_error("neo_intersect_sphere: n_rays <= 0"); return NEO_ERR_INVALID; }
    return launch_far(o, d, n, far, err_flag, (cudaStream_t)stream);
}
extern "C" int neo_sample_along_rays(const float* o, const float* d, const float* far, int n, int num_samples, int in_sphere,
                                     float far_unc, const float* u_rand, float* t, float* pts, float* pts_lin, void* stream) {
    if (n <= 0 || num_samples < 1) { set_error("neo_sample_along_rays: bad sizes"); return NEO_ERR_INVALID; }
    if (in_sphere < 0 || in_sphere > 1) { set_error("neo_sample_along_rays: in_sphere must be 0 or 1 (got %d)", in_sphere); return NEO_ERR_INVALID; }
    if (!far || !t || ((pts || pts_lin) && (!o || !d))) {
        set_error("neo_sample_along_rays: null far / t_vals, or pts / pts_linear without rays_o / rays_d");
        return NEO_ERR_INVALID;
    }
    return launch_sample_coarse(o, d, far, n, num_samples, in_sphere, far_unc, u_rand, t, pts, pts_lin, (cudaStream_t)stream);
}
extern "C" int neo_sample_pdf(const float* o, const float* d, const float* far, const float* t_old, const float* weights, int n,
                              int n_old, int num_samples, int in_sphere, float far_unc, const float* u_rand, float* t, float* pts,
                              float* pts_lin, void* stream) {
    if (n <= 0) { set_error("neo_sample_pdf: n_rays <= 0"); return NEO_ERR_INVALID; }
    if (in_sphere < 0 || in_sphere > 1) { set_error("neo_sample_pdf: in_sphere must be 0 or 1 (got %d)", in_sphere); return NEO_ERR_INVALID; }
    if (!t_old || !weights || !t || ((pts || pts_lin) && (!o || !d))) {
        set_error("neo_sample_pdf: null t_old / weights / t_vals, or pts / pts_linear without rays_o / rays_d");
        return NEO_ERR_INVALID;
    }
    return launch_resample(o, d, far, t_old, weights, n, n_old, num_samples, in_sphere, far_unc, u_rand, t, pts, pts_lin, (cudaStream_t)stream);
}
extern "C" int neo_volumetric_rendering(const float* rgb, const float* sigma, const float* t, const float* d, const float* far, int n,
                                        int N, int white, int in_sphere, float* comp, float* acc, float* w, float* lam, float* depth,
                                        void* stream) {
    if (n <= 0 || N < 1) { set_error("neo_volumetric_rendering: bad sizes"); return NEO_ERR_INVALID; }
    if (in_sphere < 0 || in_sphere > 2) { set_error("neo_volumetric_rendering: in_sphere must be 0, 1 or 2 (got %d)", in_sphere); return NEO_ERR_INVALID; }
    if (!rgb || !sigma || !t || (in_sphere && !d) || (in_sphere == 1 && !far)) {
        set_error("neo_volumetric_rendering: null rgb / sigma / t, or rays_d (in_sphere 1, 2) / far (in_sphere 1)");
        return NEO_ERR_INVALID;
    }
    return launch_composite(rgb, sigma, t, d, far, n, N, white, in_sphere, comp, acc, w, lam, depth, (cudaStream_t)stream);
}
extern "C" int neo_clipped_sq_err(const float* pred, const float* gt, long long n, double* out_sum, void* stream) {
    if (n <= 0 || !pred || !gt || !out_sum) { set_error("neo_clipped_sq_err: bad arguments"); return NEO_ERR_INVALID; }
    return launch_clipped_sq_err(pred, gt, nullptr, n, out_sum, nullptr, (cudaStream_t)stream);
}
extern "C" int neo_clipped_sq_err_masked(const float* pred, const float* gt, const uint8_t* mask, long long n_pix, double* out_sum,
                                         unsigned long long* out_count, void* stream) {
    if (n_pix <= 0 || n_pix > (1LL << 61) || !pred || !gt || !mask || !out_sum || !out_count) {
        set_error("neo_clipped_sq_err_masked: bad arguments (NULL buffer or n_pix %lld outside [1, 2^61])", n_pix);
        return NEO_ERR_INVALID;
    }
    return launch_clipped_sq_err(pred, gt, mask, 3 * n_pix, out_sum, out_count, (cudaStream_t)stream);
}
extern "C" int neo_volumetric_rendering_bwd(const float* rgb, const float* sigma, const float* t, const float* d, const float* far, int n, int N,
                                            int white, int in_sphere, const float* g_comp, const float* g_acc, const float* g_w,
                                            const float* g_lam, const float* g_depth, float* d_rgb, float* d_sigma, void* stream) {
    if (n <= 0 || N < 1 || !rgb || !sigma || !t || !d_rgb || !d_sigma) { set_error("neo_volumetric_rendering_bwd: bad arguments"); return NEO_ERR_INVALID; }
    if (in_sphere != 0 && in_sphere != 1) { set_error("neo_volumetric_rendering_bwd: in_sphere must be 0 or 1"); return NEO_ERR_UNSUPPORTED; }
    if (in_sphere && (!d || !far)) { set_error("neo_volumetric_rendering_bwd: in_sphere 1 reads rays_d and far"); return NEO_ERR_INVALID; }
    return launch_composite_bwd(rgb, sigma, t, d, far, n, N, white, in_sphere, g_comp, g_acc, g_w, g_lam, g_depth, d_rgb, d_sigma, (cudaStream_t)stream);
}
extern "C" int neo_index_grid_bwd(const NeoScene* sc, const float* pts, int M, const float* g_out, float* g_xz, float* g_xy, float* g_yz, void* stream) {
    if (!sc || M <= 0 || !pts || !g_out || !g_xz || !g_xy || !g_yz) { set_error("neo_index_grid_bwd: bad arguments"); return NEO_ERR_INVALID; }
    if (!aligned16(g_out) || !aligned16(g_xz) || !aligned16(g_xy) || !aligned16(g_yz)) {
        set_error("neo_index_grid_bwd: g_out and the gradient maps must be 16-byte aligned");
        return NEO_ERR_INVALID;
    }
    return launch_index_bwd(sc, pts, M, 0, g_out, nullptr, g_xz, g_xy, g_yz, (cudaStream_t)stream);
}
extern "C" int neo_index_local_bwd(const NeoScene* sc, const float* pts, int M, const float* g_out, float* g_latent, void* stream) {
    if (!sc || M <= 0 || !pts || !g_out || !g_latent) { set_error("neo_index_local_bwd: bad arguments"); return NEO_ERR_INVALID; }
    if (!aligned16(g_out) || !aligned16(g_latent)) { set_error("neo_index_local_bwd: g_out and g_latent must be 16-byte aligned"); return NEO_ERR_INVALID; }
    return launch_index_bwd(sc, pts, M, 1, g_out, g_latent, nullptr, nullptr, nullptr, (cudaStream_t)stream);
}
extern "C" int neo_index_maps(const NeoScene* sc, const float* pts, int M, int C, const float* latent_cl, const float* xz_cl, const float* xy_cl,
                              const float* yz_cl, float* out_local, float* out_world, void* stream) {
    if (!sc || M <= 0 || !pts || C < 4 || (C % 4) || (latent_cl && !out_local) || (xz_cl && !(xy_cl && yz_cl && out_world)) || !(latent_cl || xz_cl)) {
        set_error("neo_index_maps: bad arguments (C %% 4 == 0, a latent map and/or all three planes, outputs for what is given)");
        return NEO_ERR_INVALID;
    }
    return launch_index_maps(sc, pts, M, C, latent_cl, xz_cl, xy_cl, yz_cl, out_local, out_world, (cudaStream_t)stream);
}
extern "C" int neo_index_maps_bwd(const NeoScene* sc, const float* pts, int M, int C, const float* g_local, const float* g_world, float* g_latent_cl,
                                  float* g_xz_cl, float* g_xy_cl, float* g_yz_cl, void* stream) {
    if (!sc || M <= 0 || !pts || C < 4 || (C % 4) || (g_local && !g_latent_cl) || (g_world && !(g_xz_cl && g_xy_cl && g_yz_cl)) || !(g_local || g_world)) {
        set_error("neo_index_maps_bwd: bad arguments");
        return NEO_ERR_INVALID;
    }
    if (!aligned16(g_local) || !aligned16(g_world) || !aligned16(g_latent_cl) || !aligned16(g_xz_cl) || !aligned16(g_xy_cl) || !aligned16(g_yz_cl)) {
        set_error("neo_index_maps_bwd: row gradients and gradient maps must be 16-byte aligned");
        return NEO_ERR_INVALID;
    }
    return launch_index_maps_bwd(sc, pts, M, C, g_local, g_world, g_latent_cl, g_xz_cl, g_xy_cl, g_yz_cl, (cudaStream_t)stream);
}
namespace {
// entry ids and keys are 32-bit; the sort's item count is an int
bool det_sizes_ok(const char* who, long long E, long long T) {
    if (E >= (1LL << 31) - 1 || T >= (1LL << 31) - 1) { set_error("%s: %lld entries / %lld texels exceed 2^31 - 2", who, E, T); return false; }
    return true;
}
}  // namespace
extern "C" size_t neo_index_maps_bwd_det_workspace_bytes(const NeoScene* sc, int M, int C) {
    if (!sc || M <= 0 || C < 4 || (C % 4)) { set_error("neo_index_maps_bwd_det_workspace_bytes: bad arguments"); return 0; }
    size_t need = 0;
    for (int which = 1; which <= 3; ++which) {             // local only, world only, both: the largest layout
        long long E, T;
        index_det_sizes(sc, M, which & 1, which & 2, E, T);
        if (!det_sizes_ok("neo_index_maps_bwd_det_workspace_bytes", E, T)) return 0;
        const DetBuffers b = det_carve(nullptr, E, T);
        if (!b.total) return 0;
        need = b.total > need ? b.total : need;
    }
    return need;
}
extern "C" int neo_index_maps_bwd_det(const NeoScene* sc, const float* pts, int M, int C, const float* g_local, const float* g_world, float* g_latent_cl,
                                      float* g_xz_cl, float* g_xy_cl, float* g_yz_cl, void* workspace, size_t workspace_bytes, void* stream) {
    if (!sc || M <= 0 || !pts || C < 4 || (C % 4) || (g_local && !g_latent_cl) || (g_world && !(g_xz_cl && g_xy_cl && g_yz_cl)) || !(g_local || g_world) ||
        !workspace) {
        set_error("neo_index_maps_bwd_det: bad arguments");
        return NEO_ERR_INVALID;
    }
    if (!aligned16(g_local) || !aligned16(g_world) || !aligned16(g_latent_cl) || !aligned16(g_xz_cl) || !aligned16(g_xy_cl) || !aligned16(g_yz_cl) ||
        !aligned16(workspace)) {
        set_error("neo_index_maps_bwd_det: row gradients, gradient maps and the workspace must be 16-byte aligned");
        return NEO_ERR_INVALID;
    }
    long long E, T;
    index_det_sizes(sc, M, g_local != nullptr, g_world != nullptr, E, T);
    if (!det_sizes_ok("neo_index_maps_bwd_det", E, T)) return NEO_ERR_INVALID;
    const DetBuffers b = det_carve(workspace, E, T);
    if (!b.total) return NEO_ERR_CUDA;
    if (workspace_bytes < b.total) {
        set_error("neo_index_maps_bwd_det: workspace of %zu bytes, %zu needed", workspace_bytes, b.total);
        return NEO_ERR_INVALID;
    }
    return launch_index_maps_bwd_det(sc, pts, M, C, g_local, g_world, g_latent_cl, g_xz_cl, g_xy_cl, g_yz_cl, b, (cudaStream_t)stream);
}
extern "C" int neo_index_grid(const NeoScene* sc, const float* pts, int M, float* out, void* stream) {
    if (!sc || M <= 0 || !sc->dev.planes_cl[0]) { set_error("neo_index_grid: needs a scene prepared with NEO_PREC_FP32"); return NEO_ERR_INVALID; }
    return launch_index_grid(sc, pts, M, out, (cudaStream_t)stream);
}
extern "C" int neo_index_local(const NeoScene* sc, const float* pts, int M, float* out, void* stream) {
    if (!sc || M <= 0 || !sc->dev.latent_cl) { set_error("neo_index_local: needs a scene prepared with NEO_PREC_FP32"); return NEO_ERR_INVALID; }
    return launch_index_local(sc, pts, M, out, (cudaStream_t)stream);
}
extern "C" int neo_field_eval(const NeoScene* sc, const NeoRays* rays, const float* far, const float* t, int N, int mlp_index,
                              int precision, float* rgb, float* sigma, void* stream) {
    if (!sc || !rays || mlp_index < 0 || mlp_index > 3 || N < 1) { set_error("neo_field_eval: bad arguments"); return NEO_ERR_INVALID; }
    cudaStream_t s = (cudaStream_t)stream;
    if (precision == NEO_PREC_FP32) return field(sc, rays, far, t, N, mlp_index, precision, nullptr, rgb, sigma, s);
    // no caller workspace here: the direction fragments go to a pool block, handed back once the stream has drained
    if (rays->n_rays <= 0) { set_error("neo_field_eval: empty rays"); return NEO_ERR_INVALID; }
    const size_t bytes = (size_t)rays->n_rays * kDirFragBytes;
    void* dir = nullptr;
    int rc = pool_alloc(&dir, bytes);
    if (rc) return rc;
    if (!(rc = launch_dir_frags(sc, rays, dir, s))) {
        g_prof.launches += 1;
        rc = field(sc, rays, far, t, N, mlp_index, precision, dir, rgb, sigma, s);
    }
    const cudaError_t e = cudaStreamSynchronize(s);
    pool_release(dir, bytes);
    if (rc) return rc;
    NEO_CUDA(e);
    return NEO_OK;
}
extern "C" int neo_tc_dir_fragments(const NeoScene* sc, const NeoRays* rays, void* out, void* stream) {
    if (!sc || !rays || rays->n_rays <= 0) { set_error("neo_tc_dir_fragments: bad arguments"); return NEO_ERR_INVALID; }
    return launch_dir_frags(sc, rays, out, (cudaStream_t)stream);
}

// ---- profiling / accounting (bench.py) ----
extern "C" int neo_profile(int enable) {
    g_prof.on = enable != 0;
    g_prof.used = 0;
    g_prof.launches = 0;
    g_prof.field_points = 0;
    return NEO_OK;
}
// Synchronises the device.  field_ms = summed event time of the field-kernel launches since neo_profile(1);
// n_field = their count; launches = all kernels this library launched; points = (ray,sample) points evaluated.
extern "C" int neo_profile_read(float* field_ms, int* n_field, unsigned long long* launches, double* points) {
    NEO_CUDA(cudaDeviceSynchronize());
    float total = 0.f;
    for (size_t i = 0; i < g_prof.used; ++i) {
        float ms = 0.f;
        NEO_CUDA(cudaEventElapsedTime(&ms, g_prof.pool[i].first, g_prof.pool[i].second));
        total += ms;
    }
    if (field_ms) *field_ms = total;
    if (n_field) *n_field = (int)g_prof.used;
    if (launches) *launches = g_prof.launches;
    if (points) *points = g_prof.field_points;
    return NEO_OK;
}
