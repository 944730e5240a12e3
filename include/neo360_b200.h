/*
 * neo360_b200 -- C ABI of the B200-native NeO-360 ray-marching hot path.
 *
 * The reference (zubair-irshad/NeO-360) is pure Python; it has no FFI / operator registry.  The seam
 * this library sits behind is the Python call `self.model(rays, randomized, white_bkgd, near, far,
 * out_depth)` made by models/neo360/model.py:725-732, 841-843, 882-884 (SURVEY.md section 8(b)).
 * `neo360_b200/renderer.py` mirrors that call and binds the entry points below through ctypes;
 * INTEGRATION.md shows the reference-side stub.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer to contiguous fp32 unless marked HOST; the caller (PyTorch)
 *     owns all buffers, the library borrows them for the duration of the call;
 *   - the only library-owned object is the opaque NeoScene (re-laid-out feature maps + packed weights),
 *     released with neo_scene_free;
 *   - calls are asynchronous on `stream` (a cudaStream_t passed as void*); no call synchronises except
 *     neo_scene_create (once per scene) and neo_check_async;
 *   - return value 0 = ok, negative = NeoStatus; neo_last_error() gives the message (per thread);
 *     nothing throws across the ABI.  One caller thread per process / GPU.
 */
#ifndef NEO360_B200_H
#define NEO360_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    NEO_OK = 0,
    NEO_ERR_INVALID = -1,   /* bad argument */
    NEO_ERR_CUDA = -2,      /* CUDA runtime error, see neo_last_error */
    NEO_ERR_WORKSPACE = -3, /* workspace too small */
    NEO_ERR_GEOMETRY = -4,  /* a ray misses the unit sphere: the reference asserts (helper.py:271,426) */
    NEO_ERR_UNSUPPORTED = -5
} NeoStatus;

/* arithmetic of the density/colour MLP */
typedef enum {
    NEO_PREC_FP32 = 0, /* CUDA-core fp32, reference formulation; tightest parity (debug / validation) */
    NEO_PREC_TC = 1    /* tcgen05 tensor cores, 16-bit operands, fp32 accumulate (the fast path) */
} NeoPrecision;

/* One NeRFPPMLP (models/neo360/model.py:37-158).  nn.Linear layout: weight (out,in) row-major, bias (out). */
typedef struct {
    int in_ch;              /* 3 = fg (63-d pos-enc), 4 = bg (84-d) */
    const float *w0, *b0;   /* pts_linears.0   (128, 63|84 + 512 + 128) */
    const float *w1, *b1;   /* pts_linears.1   (128,128) */
    const float *w2, *b2;   /* pts_linears.2   (128,128) */
    const float *w3, *b3;   /* pts_linears.3   (128, 128 + 63|84 + 512 + 128) */
    const float *wb, *bb;   /* bottleneck_layer (128,128) */
    const float *wsig, *bsig; /* density_layer (1,128) */
    const float *wv0, *bv0; /* views_linear.0  (64, 128+27) */
    const float *wv1, *bv1; /* views_linear.1  (64,64) */
    const float *wrgb, *brgb; /* rgb_layer     (3,64) */
} NeoMLPParams;

/* What the (out-of-scope) encoder produced for one scene + the source cameras.
 * Replaces: encoder outputs consumed by index_grid (encoder_tp_fusion_conv.py:122-209) and
 * SpatialEncoder.index (encoder_pn.py:101-152); rays["src_poses"|"src_focal"|"src_c"|"src_imgs"] of
 * NeRF_TP.forward (model.py:266-274). */
typedef struct {
    int nv;                       /* number of source views (reference: 3) */
    int plane_h, plane_w;         /* tri-plane size (reference: 120 x 160) */
    int world_ch;                 /* 128 */
    int lat_h, lat_w, local_ch;   /* pixel-aligned latent (reference: H/2, W/2, 512) */
    int img_w, img_h;             /* src_imgs.shape[-1], [-2] (model.py:267-269) */
    const float* planes_xz;       /* (nv, world_ch, plane_h, plane_w) NCHW */
    const float* planes_xy;
    const float* planes_yz;
    const float* latent;          /* (nv, local_ch, lat_h, lat_w) NCHW */
    const float* src_poses;       /* (nv,4,4) camera-to-world */
    const float* src_focal;       /* (nv,)  only [0] is used (model.py:242) */
    const float* src_c;           /* (nv,2) only [0] is used (model.py:244) */
} NeoSceneDesc;

typedef struct NeoScene NeoScene;

/* Build the per-scene state: channel-last feature maps, R^T / -R^T t per view, MLP weights packed for
 * the selected precision.  mlps[4] = {fg_coarse, bg_coarse, fg_fine, bg_fine} (model.py:215-237).
 * `precision_mask` is a bit-or of (1<<NEO_PREC_FP32) | (1<<NEO_PREC_TC): which paths to prepare; 0 = cameras and grid geometry only
 * (enough for neo_index_maps / neo_index_maps_bwd; rendering such a scene returns NEO_ERR_INVALID). */
int neo_scene_create(const NeoSceneDesc* desc, const NeoMLPParams mlps[4], int precision_mask,
                     NeoScene** out, void* stream);
void neo_scene_free(NeoScene* scene);
/* bytes of device memory held by the scene */
size_t neo_scene_bytes(const NeoScene* scene);
/* neo_scene_free keeps the device blocks of a destroyed scene (per device, up to 6 GB in total) for the next scene of the same shape, so
 * that a scene change costs its kernels and not cudaMalloc / cudaFree.  This returns every kept block to the driver. */
void neo_release_cached(void);

/* rays of one call: rays["rays_o"|"rays_d"|"viewdirs"] (nerds360_ae.py:1007-1023). */
typedef struct {
    int n_rays;
    int chunk;               /* the reference's --chunk (opt.py:195-200): rays are conditioned on the view
                                direction of ray ((b*N+s) mod B) of their own chunk (quirk Q1, model.py:358-360);
                                chunk <= 0 means one chunk = n_rays (what a direct model(...) call does) */
    const float* rays_o;     /* (n_rays,3) */
    const float* rays_d;     /* (n_rays,3) */
    const float* viewdirs;   /* (n_rays,3) */
    const int* ray_order;    /* optional (n_rays) permutation used only for locality: the TC kernel's g-th tile covers rays
                                ray_order[32g..32g+31] (e.g. 8x4 pixel blocks of a frame); results are unchanged.  NULL = identity */
} NeoRays;

typedef struct {
    int n_coarse;            /* NeRF_TP.num_coarse_samples (level 0 evaluates n_coarse+1 points, quirk Q6) */
    int n_fine;              /* NeRF_TP.num_fine_samples   (level 1 evaluates n_coarse+1+n_fine points) */
    int white_bkgd;          /* only honoured when out_depth == 0 (model.py:501,519 vs 551,560) */
    int out_depth;           /* 1: eval tuple, 0: train tuple */
    int precision;           /* NeoPrecision */
    /* randomized=True: uniforms the reference would draw with torch.rand (helper.py:50,199); NULL = deterministic */
    const float* u_fg0;      /* (n_rays, n_coarse+1) */
    const float* u_bg0;      /* (n_rays, n_coarse+1) */
    const float* u_fg1;      /* (n_rays, n_fine) */
    const float* u_bg1;      /* (n_rays, n_fine) */
} NeoCfg;

/* Per level l in {0,1}; N_l = n_coarse+1 (+ n_fine).  NULL pointers are skipped.
 * eval tuple  (model.py:525-527): comp_rgb, fg_rgb, bg_rgb, fg_acc, bg_lambda, depth
 * train tuple (model.py:577-579): comp_rgb, fg_w, bg_w, fg_sdist, bg_sdist, bg_acc */
typedef struct {
    float* comp_rgb[2];   /* (n_rays,3) */
    float* fg_rgb[2];     /* (n_rays,3) */
    float* bg_rgb[2];     /* (n_rays,3) */
    float* fg_acc[2];     /* (n_rays)   */
    float* bg_lambda[2];  /* (n_rays,1) */
    float* depth[2];      /* (n_rays)   */
    float* bg_acc[2];     /* (n_rays)   */
    float* fg_w[2];       /* (n_rays,N_l) */
    float* bg_w[2];       /* (n_rays,N_l) */
    float* fg_sdist[2];   /* (n_rays,N_l) */
    float* bg_sdist[2];   /* (n_rays,N_l) */
    /* optional debug taps (parity tests): per-sample values of level l */
    float* fg_t[2];       /* (n_rays,N_l) */
    float* bg_s[2];       /* (n_rays,N_l) */
    float* fg_sigma[2];   /* (n_rays,N_l) */
    float* bg_sigma[2];   /* (n_rays,N_l) */
    float* fg_rgb_s[2];   /* (n_rays,N_l,3) */
    float* bg_rgb_s[2];   /* (n_rays,N_l,3) */
} NeoOut;

/* Workspace (device) the caller must provide to neo_render_fwd for n_rays rays. */
size_t neo_render_workspace_bytes(int n_rays, const NeoCfg* cfg);

/* NeRF_TP.forward with the encoder hoisted (model.py:266-581 minus :272-274).  Replaces the call at
 * model.py:725-732 / 841-843 / 882-884. */
int neo_render_fwd(const NeoScene* scene, const NeoRays* rays, const NeoCfg* cfg, NeoOut* out,
                   void* workspace, size_t workspace_bytes, void* stream);

/* Synchronise `stream` and report deferred device-side errors (the reference's two asserts,
 * helper.py:271,426, are host syncs; here they are a flag checked on demand). */
int neo_check_async(const NeoScene* scene, void* stream);

/* ---- stage-level entry points (mirror the reference helpers one to one; used by the parity tests) ---- */

/* datasets/ray_utils.py:84-104 + 133-176: pixel grid + c2w (3,4 row-major, device) -> rays. */
int neo_get_rays(int H, int W, float focal, const float* c2w, float* rays_o, float* viewdirs, float* rays_d,
                 float* radii, void* stream);
/* datasets/nerds360_ae.py:730-748 (train __getitem__): `n` sampled pixels of `n_views` target views.  pix_inds (n) int64 index the
 * flattened (n_views, H, W) stack exactly as the reference's `torch.randint(0, T*H*W)` does; c2w (n_views,3,4); images
 * (n_views,H,W,3) fp32 or NULL.  Outputs (n,3)/(n) as neo_get_rays, target (n,3) = images[pix]; any output may be NULL.  Each ray is
 * bit-identical to the same pixel of neo_get_rays.  Out-of-range indices raise *err_flag (device int) = NEO_ERR_INVALID. */
int neo_sample_rays(int n, const long long* pix_inds, int n_views, int H, int W, float focal, const float* c2w,
                    const float* images, float* rays_o, float* viewdirs, float* rays_d, float* radii, float* target,
                    int* err_flag, void* stream);
/* models/neo360/helper.py:253-273 */
int neo_intersect_sphere(const float* rays_o, const float* rays_d, int n_rays, float* far, int* err_flag,
                         void* stream);
/* models/neo360/helper.py:24-75.  in_sphere=1: t (n,N+1), pts (n,N+1,3).  in_sphere=0: t=s (n,N+1) descending,
 * pts (n,N+1,4), pts_linear (n,N+1,3).  u_rand NULL = deterministic.  far (n) and t_vals are always read / written, rays_o / rays_d
 * when pts or pts_linear is given; a NULL one of these, or in_sphere other than 0 / 1, is NEO_ERR_INVALID. */
int neo_sample_along_rays(const float* rays_o, const float* rays_d, const float* far, int n_rays, int num_samples,
                          int in_sphere, float far_uncontracted, const float* u_rand, float* t_vals, float* pts,
                          float* pts_linear, void* stream);
/* models/neo360/helper.py:218-249 (sorted_piecewise_constant_pdf 174-215 inside): bins=mids(t_old), weights[1:-1].  t_old / weights
 * (n,n_old), n_old >= 4; t_vals (n,n_old+num_samples), ascending for in_sphere=1, descending for 0 (bg s).  far is not read (the bg
 * lookup points use the sphere intersection of rays_o / rays_d) and may be NULL; rays_o / rays_d are read only for pts / pts_linear.
 * NULL t_old / weights / t_vals, pts or pts_linear without rays_o / rays_d, or in_sphere other than 0 / 1 is NEO_ERR_INVALID. */
int neo_sample_pdf(const float* rays_o, const float* rays_d, const float* far, const float* t_old,
                   const float* weights, int n_rays, int n_old, int num_samples, int in_sphere,
                   float far_uncontracted, const float* u_rand, float* t_vals, float* pts, float* pts_linear,
                   void* stream);
/* models/neo360/helper.py:128-171.  rgb (n,N,3), sigma (n,N), t (n,N).  in_sphere 1 = fg (reads rays_d and far), 0 = bg (descending s),
 * 2 = vanilla NeRF (reads rays_d); any other value, or a NULL input the branch reads, is NEO_ERR_INVALID.  Outputs may be NULL. */
int neo_volumetric_rendering(const float* rgb, const float* sigma, const float* t_vals, const float* rays_d,
                             const float* far, int n_rays, int N, int white_bkgd, int in_sphere, float* comp_rgb,
                             float* acc, float* weights, float* bg_lambda, float* depth, void* stream);
/* The same two lookups over CALLER-OWNED channel-last maps (nv,H,W,C) fp32 of any channel count C % 4 == 0, with the scene's cameras and
 * grid geometry (spatial sizes = the scene's latent / plane sizes).  Used by the training path, which looks up maps projected through the
 * current first / skip layer weights (linearity of encoder_tp_fusion_conv.py:122-209 and encoder_pn.py:101-152).  latent_cl or the three
 * planes may be NULL (then that output is skipped).  out_local / out_world: (nv*M, C), rows ordered (view, point). */
int neo_index_maps(const NeoScene* scene, const float* pts, int M, int C, const float* latent_cl, const float* xz_cl, const float* xy_cl,
                   const float* yz_cl, float* out_local, float* out_world, void* stream);
/* Backward of neo_index_maps: scatter-add of the row gradients (nv*M, C) into zero-initialised channel-last gradient maps.  Row gradients
 * and gradient maps must be 16-byte aligned (float4 reductions). */
int neo_index_maps_bwd(const NeoScene* scene, const float* pts, int M, int C, const float* g_local, const float* g_world,
                       float* g_latent_cl, float* g_xz_cl, float* g_xy_cl, float* g_yz_cl, void* stream);
/* Deterministic form of neo_index_maps_bwd, the same contract (accumulates into caller-zeroed maps, the same NULL and alignment rules) plus a
 * caller-owned workspace (16-byte aligned) of at least neo_index_maps_bwd_det_workspace_bytes(scene, M, C) bytes (0 = bad arguments or a
 * CUDA error).  No floating-point atomics: two calls are bit-identical.  neo_index_grid_bwd is this call with g_world and C = 128,
 * neo_index_local_bwd with g_local and C = 512.  Algorithm (csrc/det.cu): one entry per (view, point, tap, map), taps bit for bit the
 * forward's; a stable radix sort of (texel key, entry id); then each touched texel is written once, map = map + w * g summed in sorted order
 * as fp32 round-to-nearest multiply then add.
 * With rows = nv*M, the entries are:  local (if g_local) e = r*4 + tap, row r of g_local;  world (if g_world) e = E_local + r*12 + plane*4 + tap,
 * row r of g_world (planes xz, xy, yz), E_local = 4 rows if g_local else 0.  E = the entry count.  Texel keys: latent (if g_local)
 * v*lat_h*lat_w + texel, then plane p of view v at T_lat + (p*nv + v)*plane_h*plane_w + texel; T = the texel count; a zero-weight tap has
 * the key T and is not summed.  Workspace blocks, in this order, each at the next multiple of 256 bytes from the workspace start:
 * keys (E u32, entry order), sorted keys (E u32), entry ids (E u32), sorted entry ids (E u32), weights (E f32, entry order), segment
 * starts (T + 1 u32: the first sorted position with key >= k), sort scratch.  The sorted entries (texel, row, weight) are
 * (sorted key[i], row of sorted id[i], weight[sorted id[i]]).  Any entry past 2^31 - 2, or texel count, is NEO_ERR_INVALID. */
size_t neo_index_maps_bwd_det_workspace_bytes(const NeoScene* scene, int M, int C);
int neo_index_maps_bwd_det(const NeoScene* scene, const float* pts, int M, int C, const float* g_local, const float* g_world,
                           float* g_latent_cl, float* g_xz_cl, float* g_xy_cl, float* g_yz_cl, void* workspace, size_t workspace_bytes,
                           void* stream);
/* encoder_tp_fusion_conv.py:122-209: pts (M,3) world -> (nv*M,128), rows ordered (view, point). */
int neo_index_grid(const NeoScene* scene, const float* pts, int M, float* out, void* stream);
/* model.py:239-264 (get_local_feats): pts (M,3) world -> (nv*M,512). */
int neo_index_local(const NeoScene* scene, const float* pts, int M, float* out, void* stream);
/* Output side (models/interface.py:53-61, LitModel.psnr_each): *out_sum (device double) = sum_i (clip(pred_i,0,1) - clip(gt_i,0,1))^2 over n
 * floats; PSNR = -10 log10(out_sum / n). */
int neo_clipped_sq_err(const float* pred, const float* gt, long long n, double* out_sum, void* stream);
/* Object PSNR (models/utils.py:102-109 get_obj_rgbs_from_segmap, then psnr_each): pred / gt (n_pix, 3), mask (n_pix) one byte per pixel,
 * non-zero = selected.  *out_sum (device double) = the same sum over the values of the selected pixels only, *out_count (device) = their
 * number (3 per pixel); object PSNR = -10 log10(out_sum / out_count), NaN when out_count is 0.  The kernel of neo_clipped_sq_err. */
int neo_clipped_sq_err_masked(const float* pred, const float* gt, const uint8_t* mask, long long n_pix, double* out_sum,
                              unsigned long long* out_count, void* stream);
/* SSIM as LitModel.ssim_each computes it with piqa's SSIM() at its defaults (models/interface.py:101-111; definition in
 * csrc/metrics.cu): pred / gt (n, H, W, 3) fp32 channel-last, clipped to [0, 1] inside.  ssim (n) device doubles, one per frame;
 * ss_map (n, H-10, W-10, 3) fp32 or NULL.  Workspace: neo_ssim_workspace_bytes(n, H, W) bytes, 8-byte aligned, caller-owned (0 = invalid
 * sizes).  NULL pred / gt / ssim / workspace, n < 1, H or W < 11, or a size past int64 elements is NEO_ERR_INVALID before any launch.
 * No floating-point atomics: two calls are bit-identical, and a frame gives the same bits alone or inside any batch. */
size_t neo_ssim_workspace_bytes(int n, int H, int W);
int neo_ssim(const float* pred, const float* gt, int n, int H, int W, double* ssim, float* ss_map, void* workspace, size_t workspace_bytes,
             void* stream);
/* LPIPS (VGG) around a trunk the caller runs (definition in csrc/lpips.cu): LitModel.lpips_each with piqa's LPIPS (models/interface.py:
 * 113-122) and the fine-tuning loss with lpips.LPIPS (models/neo360/model.py:1283-1309).  Asynchronous on `stream`, nothing allocated,
 * NEO_ERR_INVALID before any launch on a NULL buffer or sizes out of range.
 * neo_lpips_prepare: img (n, H, W, 3) fp32 channel-last, clipped to [0, 1] -> out (n, 3, H, W), scaled by form 0 (piqa: (x - mean) / std)
 * or form 1 (lpips: ((2x - 1) - shift) / scale).  neo_lpips_prepare_bwd: g_out (n, 3, H, W) -> g_img (n, H, W, 3), zero where img is
 * outside [0, 1] (inclusive bounds pass, as torch.clamp's backward). */
int neo_lpips_prepare(const float* img, int n, int H, int W, int form, float* out, void* stream);
int neo_lpips_prepare_bwd(const float* img, const float* g_out, int n, int H, int W, int form, float* g_img, void* stream);
/* neo_lpips_head: fx, fy, w are host arrays of 5 device pointers: the features of relu1_2 .. relu5_3 of the frames (n, C_k, H >> k, W >> k)
 * fp32 NCHW with C = 64, 128, 256, 512, 512, and the layers' 1x1 weights (C_k).  lpips (n) device doubles; per_layer (n, 5) device doubles
 * or NULL.  Workspace: neo_lpips_workspace_bytes(n, H, W) bytes, 8-byte aligned, caller-owned (0 = invalid sizes: n >= 1, H, W >= 16).
 * No floating-point atomics: two calls are bit-identical and a frame gives the same bits alone or in any batch.
 * neo_lpips_head_bwd: g (n) fp32 device, the upstream gradient of each frame's value; writes every element of g_fx[k] (shaped as fx[k]) and,
 * when g_fy is not NULL, of g_fy[k].  A pixel whose features are all zero gets a zero gradient. */
size_t neo_lpips_workspace_bytes(int n, int H, int W);
int neo_lpips_head(const float* const* fx, const float* const* fy, const float* const* w, int n, int H, int W, double* lpips, double* per_layer,
                   void* workspace, size_t workspace_bytes, void* stream);
int neo_lpips_head_bwd(const float* const* fx, const float* const* fy, const float* const* w, int n, int H, int W, const float* g,
                       float* const* g_fx, float* const* g_fy, void* stream);

/* ---- backward of the hand-written stages (training: models/neo360/model.py:697-820 differentiates through this path) ----
 * The field's backward is split: the lookups' scatter and the compositing backward are the entry points below; the dense layers of
 * NeRFPPMLP are differentiated by the host framework (plain library GEMMs) in neo360_b200/training.py.  Sample positions carry no
 * gradient (the reference detaches them, helper.py:225). */
/* d(volumetric_rendering)/d(rgb, sigma): upstream gradients of comp_rgb (n,3), acc (n), weights (n,N), bg_lambda (n), depth (n) -- any
 * may be NULL -- -> d_rgb (n,N,3), d_sigma (n,N).  Same rgb / sigma / t / rays_d / far as the forward call; in_sphere 0 or 1. */
int neo_volumetric_rendering_bwd(const float* rgb, const float* sigma, const float* t_vals, const float* rays_d, const float* far,
                                 int n_rays, int N, int white_bkgd, int in_sphere, const float* g_comp_rgb, const float* g_acc,
                                 const float* g_weights, const float* g_bg_lambda, const float* g_depth, float* d_rgb, float* d_sigma,
                                 void* stream);
/* d(index_grid)/d(planes): g_out (nv*M,128) -> ACCUMULATES into channel-last gradient maps (nv, plane_h, plane_w, 128) x3 (zeroed by the caller).
 * g_out and the gradient maps of this and neo_index_local_bwd must be 16-byte aligned. */
int neo_index_grid_bwd(const NeoScene* scene, const float* pts, int M, const float* g_out, float* g_planes_xz, float* g_planes_xy,
                       float* g_planes_yz, void* stream);
/* d(get_local_feats)/d(latent): g_out (nv*M,512) -> ACCUMULATES into the channel-last gradient map (nv, lat_h, lat_w, 512). */
int neo_index_local_bwd(const NeoScene* scene, const float* pts, int M, const float* g_out, float* g_latent, void* stream);
/* `predict` (model.py:343-407) for one branch of one level: t/s (n,N) -> rgb (n,N,3), sigma (n,N).
 * mlp_index in 0..3 = {fg_coarse,bg_coarse,fg_fine,bg_fine}; is_bg selects the NeRF++ background parametrisation. */
int neo_field_eval(const NeoScene* scene, const NeoRays* rays, const float* far, const float* t_vals, int N,
                   int mlp_index, int precision, float* rgb, float* sigma, void* stream);

/* ---- geometry export: density grid, marching tetrahedra, normals (csrc/mesh.cu, neo360_b200/mesh.py) ----
 * A lattice of nx * ny * nz points, each axis >= 2 points, at most 2^28 points in all.  Point (i, j, k) lies at
 * (origin[0] + i * step[0], origin[1] + j * step[1], origin[2] + k * step[2]), each product and sum rounded to nearest in fp32.
 * Grid values (sigma) are fp32, laid out (nz, ny, nx) with x fastest; row r = k * ny + j is the x-row of points (*, j, k).
 * Every call validates its arguments before any launch and returns NEO_ERR_INVALID on a bad one. */
typedef struct {
    int nx, ny, nz;
    float origin[3];          /* x, y, z of point (0, 0, 0): finite */
    float step[3];            /* spacing along x, y, z: finite and > 0 */
} NeoGrid;
/* Rays that make neo_field_eval evaluate a foreground MLP at the lattice points of rows [row0, row0 + n_rows): row r gets
 * rays_o = (origin[0], y_j, z_k), dirs = (1, 0, 0) (pass it as rays_d and viewdirs) and t_vals (n_rows, nx) = i * step[0], so that
 * o + t d is the lattice point bit for bit.  rays_o and dirs are (n_rows, 3). */
int neo_grid_rays(const NeoGrid* grid, long long row0, int n_rows, float* rays_o, float* dirs, float* t_vals, void* stream);
/* sigma_rows (n_rows, nx), rows [row0, row0 + n_rows) of a grid: sets sigma = 0 at every point with x*x + y*y + z*z > 1 (fp32, in that
 * order).  The foreground branch is only sampled inside the unit sphere, so the density grid defines sigma = 0 outside it. */
int neo_grid_mask_sphere(const NeoGrid* grid, long long row0, int n_rows, float* sigma_rows, void* stream);
/* Marching tetrahedra over a grid (sigma, (nz, ny, nx)).  Inside means sigma >= iso (a NaN is outside).  Every cell is split into the 6
 * Kuhn tetrahedra sharing its main diagonal; point p owns the 7 edges from p to p + e, e in type order (1,0,0) (0,1,0) (0,0,1) (1,1,0)
 * (1,0,1) (0,1,1) (1,1,1).  A vertex lies on each owned edge whose end points are on different sides, at
 * w = (iso - s_a) / (s_b - s_a), x = p_a + w * (p_b - p_a) per coordinate (a = p, b = p + e; fp32, each operation rounded to nearest).
 * Vertex ids follow (point, edge type) order; faces (int32 vertex ids) follow (cell, tetrahedron, triangle) order, cells in point order,
 * and wind counter-clockwise seen from outside (lower sigma).  No atomics: two calls give identical bits.
 * Workspace: neo_mt_workspace_bytes(grid) bytes (0 = bad grid), 256-byte aligned, caller-owned.  neo_mt_count writes V and F to
 * *n_verts / *n_faces (HOST ints) and synchronises `stream` once; NEO_ERR_UNSUPPORTED when either exceeds 2^31 - 1.
 * neo_mt_emit reads the block offsets neo_mt_count left in the workspace (same sigma, grid, iso and workspace, same stream), writes
 * verts (n_verts, 3) and faces (n_faces, 3), and never writes past n_verts / n_faces. */
size_t neo_mt_workspace_bytes(const NeoGrid* grid);
int neo_mt_count(const float* sigma, const NeoGrid* grid, float iso, void* workspace, size_t workspace_bytes, int* n_verts, int* n_faces,
                 void* stream);
int neo_mt_emit(const float* sigma, const NeoGrid* grid, float iso, void* workspace, size_t workspace_bytes, float* verts, int n_verts,
                int* faces, int n_faces, void* stream);
/* normals (n_verts, 3) = -grad sigma / |grad sigma| at each vertex (0 where the gradient is 0): the gradient at the lattice points by central
 * differences (one-sided on the grid's faces), trilinearly interpolated in the cell that holds the vertex (clamped into the grid). */
int neo_grid_normals(const float* sigma, const NeoGrid* grid, const float* verts, int n_verts, float* normals, void* stream);

/* ---- vanilla two-level NeRF (SURVEY.md section 8(a) row a17): models/vanilla_nerf/model.py:44-216 ---- */
typedef struct {
    const float* w[8];        /* pts_linears.{0..7}.weight: (256,63) (256,256)x4 (256,319) (256,256)x2 */
    const float* b[8];
    const float *wb, *bb;     /* bottleneck_layer (256,256) */
    const float *wsig, *bsig; /* density_layer (1,256) */
    const float *wv0, *bv0;   /* views_linear.0 (128, 256+27) */
    const float *wrgb, *brgb; /* rgb_layer (3,128) */
} NeoVanillaMLPParams;
typedef struct NeoVanilla NeoVanilla;
typedef struct {
    int n_coarse, n_fine, white_bkgd;
    float near_plane, far_plane;   /* the scalar near / far the caller passes to NeRF.forward (model.py:154) */
    const float* u0;               /* randomized: (n_rays, n_coarse+1) uniforms, helper.py:438; NULL = deterministic */
    const float* u1;               /* randomized: (n_rays, n_fine) uniforms, helper.py:587 */
    int precision;                 /* NeoPrecision: NEO_PREC_FP32 = fused fp32 CUDA-core field kernel (tight parity), NEO_PREC_TC = NeRFMLP layer by layer
                                      on tcgen05 (csrc/gemm_tc.cu), fp16 weights / activations */
} NeoVanillaCfg;
typedef struct {
    float* comp_rgb[2];  /* (n_rays,3)   model.py:214 returns (comp_rgb, acc, depth) per level */
    float* acc[2];       /* (n_rays) */
    float* depth[2];     /* (n_rays) */
    float* t[2];         /* optional debug taps: (n_rays,N_l) */
    float* sigma[2];
    float* rgb_s[2];     /* (n_rays,N_l,3) */
    float* weights[2];
} NeoVanillaOut;
/* mlps[2] = {coarse_mlp, fine_mlp} */
int neo_vanilla_create(const NeoVanillaMLPParams mlps[2], NeoVanilla** out, void* stream);
void neo_vanilla_free(NeoVanilla* v);
size_t neo_vanilla_workspace_bytes(int n_rays, const NeoVanillaCfg* cfg);
/* NeRF.forward (models/vanilla_nerf/model.py:154-216); rays->chunk is ignored (no cross-ray coupling in this model) */
int neo_vanilla_render_fwd(const NeoVanilla* v, const NeoRays* rays, const NeoVanillaCfg* cfg, NeoVanillaOut* out,
                           void* workspace, size_t workspace_bytes, void* stream);
/* The NeRFMLP of one level (0 coarse, 1 fine) at caller-given points: sample s of ray b is rays_o[b] + t_vals[b, s] * viewdirs[b], as the
 * render casts it (rays_d is not read), and its direction input is viewdirs[b].  t_vals (n_rays, N) -> activated rgb (n_rays, N, 3) and
 * sigma (n_rays, N), the render's `rgb_s` / `sigma` at its own samples.  The render runs the same code per level, so the two give the same
 * bits.  precision NEO_PREC_FP32 (the fused field kernel) or NEO_PREC_TC (the fp16 layer chain).  Workspace: 256-byte aligned,
 * neo_vanilla_field_workspace_bytes(n_rays * N, precision) bytes; NEO_PREC_FP32 needs none (0 bytes, ws may be NULL).
 * n_rays * N < 2^31.  sigma does not depend on viewdirs. */
size_t neo_vanilla_field_workspace_bytes(long long n_points, int precision);
int neo_vanilla_field_eval(const NeoVanilla* v, const NeoRays* rays, const float* t_vals, int N, int level, int precision, float* rgb,
                           float* sigma, void* ws, size_t ws_bytes, void* stream);
/* Stages of the differentiable NeRF.forward (training, models/vanilla_nerf/model.py:154-216 under autograd; neo360_b200/vanilla.py).
 * Hand-written: sampling, encodings, compositing forward and backward; the NeRFMLP dense layers are differentiated by the host framework.
 * The fine level resamples with neo_sample_pdf(rays_o, viewdirs, NULL, t0, weights0, n, n_coarse+1, n_fine, 1, 0, u1, t1, NULL, NULL)
 * and composites forward with neo_volumetric_rendering(..., in_sphere = 2, ...), the calls neo_vanilla_render_fwd makes. */
/* helper.py:415-442 along viewdirs (quirk Q15): t_vals (n_rays, n_coarse+1); u_rand (n_rays, n_coarse+1) or NULL = deterministic.
 * The same kernel as neo_vanilla_render_fwd's level 0: bit-identical t. */
int neo_vanilla_sample_along_rays(const float* rays_o, const float* viewdirs, int n_rays, int n_coarse, float near_plane, float far_plane,
                                  const float* u_rand, float* t_vals, void* stream);
/* fp32 positional encodings (helper.py:445-449 column order) of the points o + t viewdirs: enc (n_rays*N, 63), and of the view
 * directions: dir_enc (n_rays, 27).  The same arithmetic as the NEO_PREC_FP32 field kernel (bit-identical).  No backward. */
int neo_vanilla_encode(const float* rays_o, const float* viewdirs, const float* t_vals, int n_rays, int N, float* enc, float* dir_enc,
                       void* stream);
/* Backward of neo_volumetric_rendering in mode 2 (helper.py:521-559): upstream gradients of comp_rgb (n,3), acc (n), weights (n,N),
 * depth (n) -- any may be NULL -- -> d_rgb (n,N,3), d_sigma (n,N).  The depth gradient passes where sum w t was finite (nan_to_num +
 * clamp, quirk Q10) and is zero elsewhere.  Same rgb / sigma / t / rays_d as the forward call. */
int neo_vanilla_composite_bwd(const float* rgb, const float* sigma, const float* t_vals, const float* rays_d, int n_rays, int N, int white_bkgd,
                              const float* g_comp_rgb, const float* g_acc, const float* g_weights, const float* g_depth, float* d_rgb,
                              float* d_sigma, void* stream);

/* ---- PixelNeRF (SURVEY.md section 2 row 11): models/vanilla_nerf/model_pixel.py:35-258, csrc/pixelnerf.cu ----
 * Sampling, lookup backward and compositing are the stages above: neo_vanilla_sample_along_rays and neo_sample_pdf (t only, so rays_d
 * may be passed as the direction), neo_index_maps / neo_index_maps_bwd(_det) on the caller's channel-last latent, and
 * neo_volumetric_rendering mode 2 / neo_vanilla_composite_bwd on the activated rgb and sigma.
 * `scene` below is a cameras-only NeoScene (precision_mask 0) built from the source poses with column 1 of each rotation negated
 * (camera y flipped) and the image size of src_imgs: with it the shared projection gives PixelNeRF's pixel coordinates exactly, for
 * these entry points and for neo_index_maps*.  One NeRFMLP: nn.Linear layers with the weights TRANSPOSED to (in, out), row-major,
 * 16-byte aligned. */
typedef struct {
    const float* wt[4];         /* pts_linears.{0..3}.weight^T: (575,128) (128,128)x3 */
    const float* b[4];
    const float *wbt, *bb;      /* bottleneck_layer^T (128,128) */
    const float *wsig, *bsig;   /* density_layer (1,128), not transposed */
    const float *wv0t, *bv0;    /* views_linear.0^T (155,128) */
    const float *wv1t, *bv1;    /* views_linear.1^T (128,128) */
    const float *wrgb, *brgb;   /* rgb_layer (3,128), not transposed */
} NeoPixelMLPParams;
/* The field of one level, fp32 CUDA cores in the reference formulation: for t_vals (n_rays, N) the points o + t rays_d, per source view
 * the camera transform, the view-0 projection, the bilinear lookup of latent_cl (nv, lat_h, lat_w, 512; zeros padding), the encodings
 * of the camera-frame point (63) and of the camera-frame view direction (27; row b*N+s of a chunk of rays->chunk rays, <= 0 = all, is
 * conditioned on ray ((b*N+s) mod B) of its chunk, quirk Q1), the 4x128 trunk, the per-view bottleneck, the view means, and
 * rgb = sigmoid, sigma = relu -> rgb (n_rays, N, 3), sigma (n_rays, N).  1..8 views. */
int neo_pixelnerf_field(const NeoScene* scene, const float* latent_cl, const NeoPixelMLPParams* mlp, const NeoRays* rays,
                        const float* t_vals, int N, float* rgb, float* sigma, void* stream);
/* The training path's inputs of one level, the field kernel's arithmetic: enc (nv*M, 63), dir_tile (nv*M, 27) with rows ordered
 * (view, point), M = n_rays*N, and pts (M,3) = o + t rays_d (or NULL), the world points neo_index_maps looks up. */
int neo_pixelnerf_encode(const NeoScene* scene, const NeoRays* rays, const float* t_vals, int N, float* enc, float* dir_tile,
                         float* pts, void* stream);

/* NEO_PREC_TC form of neo_pixelnerf_field: the same layers in the reference formulation on the tensor-core dense layer (gemm_f16: fp16
 * operands, fp32 accumulation).  Per pass of up to 65536 points: fp16 rows [enc 63 | latent 512 | 0] (nv*M, 576); the trunk, fp16 after
 * each bias + ReLU; the bottleneck (fp16, no ReLU) beside the fp16 direction encoding in rows [bottleneck | dir 27 | 0] (192); the view
 * mean of h3 (fp32 sum, fp16) times density_layer (fp32, rowdot); views_linear.0 (fp16), its view mean + ReLU (fp16); views_linear.1
 * (fp16 after ReLU); rgb_layer (fp32, rowdot); sigma = relu, rgb = sigmoid.  Weights fp16 nn.Linear layout (out, in) with the input
 * width zero-padded: pts_linears.0 (128, 576), views_linear.0 (128, 192), the rest (128, 128); 16-byte aligned.  Workspace:
 * neo_pixelnerf_tc_workspace_bytes(nv, n_rays*N) bytes, 256-byte aligned (0 = invalid sizes). */
typedef struct {
    const void* w16[4];         /* pts_linears.{0..3}.weight fp16 */
    const float* b[4];
    const void* wb16;           /* bottleneck_layer fp16 (128,128) */
    const float* bb;
    const float *wsig, *bsig;   /* density_layer fp32 (1,128) */
    const void* wv016;          /* views_linear.0 fp16 (128,192) */
    const float* bv0;
    const void* wv116;          /* views_linear.1 fp16 (128,128) */
    const float* bv1;
    const float *wrgb, *brgb;   /* rgb_layer fp32 (3,128) */
} NeoPixelTCParams;
size_t neo_pixelnerf_tc_workspace_bytes(int nv, long long M);
int neo_pixelnerf_field_tc(const NeoScene* scene, const float* latent_cl, const NeoPixelTCParams* mlp, const NeoRays* rays,
                           const float* t_vals, int N, float* rgb, float* sigma, void* workspace, size_t workspace_bytes, void* stream);

/* ---- Mip-NeRF 360 (SURVEY.md section 8(a) row a18): models/mipnerf360/model.py:30-365 ---- */
typedef struct {
    int depth, width;          /* PropMLP: 4 x 256 (density only), NeRFMLP: 8 x 1024 (model.py:176-195) */
    const float* basis;        /* pos_basis_t (3,21) */
    const float* w[8];         /* pts_linear.{i}.weight: (width,504), (width,width)..., layer 5 of a depth-8 MLP is (width, width+504) */
    const float* b[8];
    const float *wsig, *bsig;  /* density_layer (1,width) */
    const float *wb, *bb;      /* bottleneck_layer (256,width)      -- NULL for a PropMLP (disable_rgb) */
    const float *wv0, *bv0;    /* views_linear.0 (128, 256+27) */
    const float *wrgb, *brgb;  /* rgb_layer (3,128) */
} NeoMipMLPParams;
typedef struct {
    int n_prop, n_nerf;            /* MipNeRF360.num_prop_samples / num_nerf_samples (two proposal levels + one NeRF level) */
    float near_plane, far_plane;   /* near / far passed to MipNeRF360.forward (model.py:236) */
    float train_frac;              /* anneals the proposal logits (model.py:288-292) */
    const float* jitter[3];        /* randomized: one (n_rays) uniform per level (single_jitter, helper.py:357-363); NULL = deterministic */
    int precision;                 /* NeoPrecision: NEO_PREC_FP32 = fp32 CUDA-core SGEMM chain (tight parity), NEO_PREC_TC = fp16 activations / weights,
                                      every dense layer on tcgen05 (csrc/gemm_tc.cu) */
} NeoMipCfg;
typedef struct {                   /* per level: renderings[l]["rgb"], ray_history[l]{"density","rgb","sdist","weights"} (model.py:359-365) */
    float* rgb[3];       /* (n_rays,3) */
    float* density[3];   /* (n_rays,n_l) */
    float* rgb_s[3];     /* (n_rays,n_l,3) -- zeros for the proposal levels */
    float* sdist[3];     /* (n_rays,n_l+1) */
    float* weights[3];   /* (n_rays,n_l) */
} NeoMipOut;
size_t neo_mip_workspace_bytes(int n_rays, const NeoMipCfg* cfg, int nerf_width);
/* MipNeRF360.forward (models/mipnerf360/model.py:236-365); mlps[3] = {PropMLP, PropMLP, NeRFMLP}; radii (n_rays) */
int neo_mip_render_fwd(const NeoMipMLPParams mlps[3], const float* rays_o, const float* rays_d, const float* viewdirs,
                       const float* radii, int n_rays, const NeoMipCfg* cfg, NeoMipOut* out, void* workspace,
                       size_t workspace_bytes, void* stream);
/* Stages of the differentiable MipNeRF360.forward (training, LitMipNeRF360.training_step, models/mipnerf360/model.py:427-456 under autograd;
 * neo360_b200/mip.py).  Hand-written: resampling, IPE features and direction encoding (no backward: sdist is detached, model.py:309-310, and
 * contract returns detached values, helper.py:63-66), compositing forward and backward; the MLP dense layers are differentiated by the host
 * framework.  Each launches the same kernel as neo_mip_render_fwd's NEO_PREC_FP32 path, so training and eval share their arithmetic. */
/* One level of max_dilate_weights + annealed logits + sample_intervals + s_to_t (model.py:262-312): sdist, tdist (n_rays, n_new+1).
 * level 0 reads no previous level (sdist_prev / weights_prev may be NULL); level 1 or 2 reads the previous level's sdist (n_rays, n_prev+1)
 * and weights (n_rays, n_prev).  The dilation is 0.0025 + 0.5 / n_prev^level (both proposal levels take num_prop_samples).  n_new in
 * [2,160], n_prev in [1,160]; jitter (n_rays) or NULL = deterministic.  Bit-identical to neo_mip_render_fwd's resampling of that level. */
int neo_mip_resample(const float* sdist_prev, const float* weights_prev, int n_rays, int n_prev, int level, int n_new, float near_plane,
                     float far_plane, float train_frac, const float* jitter, float* sdist, float* tdist, void* stream);
/* fp32 integrated positional encoding of the conical frustums of tdist (n_rays, N+1) (cast_rays + contract + lift_and_diagonalize +
 * integrated_pos_enc): feats (n_rays*N, 504); and the direction encoding of viewdirs, one row per ray: dir_enc (n_rays, 27).  basis is
 * pos_basis_t (3,21).  The NEO_PREC_FP32 path's own kernels (bit-identical).  No backward. */
int neo_mip_encode(const float* rays_o, const float* rays_d, const float* viewdirs, const float* radii, const float* tdist, const float* basis,
                   int n_rays, int N, float* feats, float* dir_enc, void* stream);
/* Head activations + compute_alpha_weights(opaque_background) + volumetric_rendering with a white background (helper.py:234-274) of raw
 * density (n_rays,N) and raw rgb (n_rays,N,3) at tdist (n_rays,N+1): rgb (n_rays,3), weights (n_rays,N), density (n_rays,N), rgb_s
 * (n_rays,N,3).  raw_rgb NULL = a proposal level (rgb_s is written as zeros).  Outputs may be NULL.  The eval path's compositing kernel. */
int neo_mip_composite(const float* raw_density, const float* raw_rgb, const float* tdist, const float* rays_d, int n_rays, int N, float* rgb,
                      float* weights, float* density, float* rgb_s, void* stream);
/* Backward of neo_mip_composite: upstream gradients of rgb (n,3), weights (n,N), density (n,N), rgb_s (n,N,3) -- any may be NULL -- ->
 * d_raw_density (n,N) and, unless raw_rgb is NULL, d_raw_rgb (n,N,3).  Same raw_density / raw_rgb / tdist / rays_d as the forward call.
 * The gradient of clip(1 - acc, min=0) passes where 1 - acc >= 0 of this call's own fp32 acc; the last (infinite) interval has no
 * density gradient through the weights. */
int neo_mip_composite_bwd(const float* raw_density, const float* raw_rgb, const float* tdist, const float* rays_d, int n_rays, int N,
                          const float* g_rgb, const float* g_weights, const float* g_density, const float* g_rgb_s, float* d_raw_density,
                          float* d_raw_rgb, void* stream);
/* One MLP of Mip-NeRF 360 (level 0, 1: PropMLP; 2: NeRFMLP) at caller-given points.  The MLP reads a Gaussian: here its mean is the point
 * rays_o[b] + t_vals[b, s] * viewdirs[b] (fp32, each operation rounded; rays_d is not read) and its covariance diag(var), var >= 0 per
 * axis.  The Gaussian goes through the render's own encoding (contraction with its Jacobian, 21-direction lift, 12-octave IPE), then the
 * render's layer chain in `precision` (fp32 SGEMMs or fp16 tensor-core GEMMs) with viewdirs[b] as the direction input.  Outputs: density
 * (n_rays, N) = softplus(raw - 1) and, at level 2 only, rgb (n_rays, N, 3) = 1.002 sigmoid(raw) - 0.001, or NULL.  A non-NULL rgb at a
 * proposal level is an error: those MLPs have no colour head.  mlps[3] as for neo_mip_render_fwd; only mlps[level] is read.  Workspace:
 * neo_mip_field_workspace_bytes(n_rays * N, mlps[level].width, precision) bytes, 256-byte aligned (0 = invalid sizes).  n_rays * N < 2^31. */
size_t neo_mip_field_workspace_bytes(long long n_points, int width, int precision);
int neo_mip_field_eval(const NeoMipMLPParams mlps[3], int level, const NeoRays* rays, const float* t_vals, int N, const float var[3],
                       int precision, float* rgb, float* density, void* ws, size_t ws_bytes, void* stream);

/* ---- tri-plane builder, dense part (SURVEY.md section 8(f1)): models/neo360/encoder_tp_fusion_conv.py:472-597 between the ResNet feature
 * extractor and the floor-plan conv stacks (both stay in the host framework).  64^3 world grid x nv views: latent lookup, DepthPillarEncoder
 * 518->512->512->512, three pillar aggregators (513->512->1, softmax along one grid axis), softmax-weighted pillar sums.  At inference
 * (neo_grid_encoder_dense) every dense layer runs on wgmma through gemm_f16 (csrc/gemm_tc.cu, fp16 weights / activations, fp32
 * accumulation); nn.Linear layout (out,in) fp32 device pointers.  Training uses the four fp32 stage entry points below around the host
 * framework's dense layers.  Grid rows: row = v*64^3 + cell, cell = (ix*64 + iy)*64 + iz; axis 0 / 1 / 2 = the yz / xz / xy floor plan
 * (the pillar runs along x / y / z). ---- */
typedef struct {
    const float* fc_w[3];   /* depth_fc.common_branch.0 (512,518), depth_fc.common_branch.2 (512,512), depth_fc.depth_encoder (512,512) */
    const float* fc_b[3];
    const float *agg_xz_w0, *agg_xz_b0, *agg_xz_w1, *agg_xz_b1;   /* pillar_aggregator_xz.{0,2}: (512,513), (512), (1,512), (1) */
    const float *agg_yz_w0, *agg_yz_b0, *agg_yz_w1, *agg_yz_b1;
    const float *agg_xy_w0, *agg_xy_b0, *agg_xy_w1, *agg_xy_b1;
} NeoGridEncoderParams;
size_t neo_grid_encoder_workspace_bytes(int nv, int lat_h, int lat_w);
/* latent (nv,512,lat_h,lat_w) NCHW = SpatialEncoder output; src_poses (nv,4,4) camera-to-world; focal / (cx,cy) = src_focal[0] / src_c[0].
 * Outputs: the three pillar-aggregated floor plans (nv,512,64,64) NCHW that feed floorplan_convnet_{xz,xy,yz}. */
int neo_grid_encoder_dense(const NeoGridEncoderParams* params, const float* latent, int nv, int lat_h, int lat_w, int img_w, int img_h,
                           const float* src_poses, float focal, float cx, float cy, float* floor_xz, float* floor_xy, float* floor_yz,
                           void* workspace, size_t workspace_bytes, void* stream);
/* Training path, fp32, caller-owned buffers, asynchronous on `stream`, nothing allocated.  All four return NEO_ERR_INVALID before any
 * launch on a NULL buffer, nv < 1, lat_h or lat_w < 2, img_w or img_h <= 0, or a stride / alignment the kernels cannot address.
 * Lookup rows: latent_cl (nv,lat_h,lat_w,512) channel-last (16-byte aligned) -> X (nv*64^3, ldx) rows
 * [bilinear latent lookup 512 | cam xyz 3 | masked unit direction 3 | 0 ...] = the input of depth_fc; 518 <= ldx <= 640, ldx % 4 == 0,
 * X 16-byte aligned (so X[:, :518] of a 520-wide buffer is a strided GEMM operand). */
int neo_grid_encoder_features(const float* latent_cl, int nv, int lat_h, int lat_w, int img_w, int img_h, const float* src_poses, float focal,
                              float cx, float cy, float* X, int ldx, void* stream);
/* Adjoint of the lookup columns: g_latent_cl (nv,lat_h,lat_w,512) channel-last, caller-zeroed, 16-byte aligned += sum over rows of the
 * tap weights times g_X[row][0..512) (16-byte vector atomics; the order of the additions is not fixed).  g_X row stride ldg >= 512 and
 * even, 8-byte aligned; columns >= 512 are not read (poses do not train).  The taps are the forward's, bit for bit. */
int neo_grid_encoder_features_bwd(int nv, int lat_h, int lat_w, int img_w, int img_h, const float* src_poses, float focal, float cx, float cy,
                                  const float* g_X, long long ldg, float* g_latent_cl, void* stream);
/* Deterministic form of neo_grid_encoder_features_bwd, the same geometry, contract and argument rules plus a caller-owned 16-byte aligned
 * workspace of neo_grid_encoder_features_bwd_det_workspace_bytes(nv, lat_h, lat_w) bytes (0 = bad sizes or a CUDA error).  The order-fixed
 * scatter of neo_index_maps_bwd_det: entries e = row*4 + tap (row of g_X), keys v*lat_h*lat_w + texel (T = nv*lat_h*lat_w for a zero weight),
 * the same workspace layout with E = 4 nv 64^3.  g_X is read as float2 pairs.  Two calls are bit-identical. */
size_t neo_grid_encoder_features_bwd_det_workspace_bytes(int nv, int lat_h, int lat_w);
int neo_grid_encoder_features_bwd_det(int nv, int lat_h, int lat_w, int img_w, int img_h, const float* src_poses, float focal, float cx,
                                      float cy, const float* g_X, long long ldg, float* g_latent_cl, void* workspace, size_t workspace_bytes,
                                      void* stream);
/* Softmax pillar sums: lat (nv*64^3, 512) row-major, 16-byte aligned, logits (3, nv*64^3) by axis -> floor plans (nv,512,64,64) NCHW. */
int neo_grid_encoder_pool(const float* lat, const float* logits, int nv, float* floor_xz, float* floor_xy, float* floor_yz, void* stream);
/* Backward of neo_grid_encoder_pool: upstream g_xz / g_xy / g_yz (nv,512,64,64), each may be NULL (zero) -> d_lat (nv*64^3, 512) = the
 * sum of the three axes' contributions and d_logits (3, nv*64^3) = s (g.lat - sum_pillar s (g.lat)); every element written, no
 * floating-point atomics (two calls give bit-identical results). */
int neo_grid_encoder_pool_bwd(const float* lat, const float* logits, int nv, const float* g_xz, const float* g_xy, const float* g_yz,
                              float* d_lat, float* d_logits, void* stream);
/* Tensor-core training form (GridEncoder.dense_train_tc): bf16 rows around the neo_tc_*_bf16 products.  Each returns NEO_ERR_INVALID
 * before any launch on a NULL buffer, nv < 1, or a stride / alignment its kernel cannot address; the geometry rules are those above.
 * neo_grid_encoder_features_bf16: the rows of neo_grid_encoder_features as bf16, each element the fp32 entry's value rounded once;
 *   518 <= ldx <= 640, ldx % 8 == 0, X 16-byte aligned.
 * neo_grid_encoder_coords_bf16: columns 512, 513, 514 of every row of L (nv*64^3, ld) = the cell's world x, y, z in bf16, columns
 *   515..ld-1 = 0 (L = [lat | x y z | 0], the input of the aggregators' stacked first layer); 520 <= ld <= 640, ld % 8 == 0, 16-byte aligned.
 * neo_grid_encoder_pool_bf16 / _pool_bwd_bf16: neo_grid_encoder_pool / _pool_bwd with lat the first 512 bf16 columns of rows of stride
 *   ld >= 512 (pool: ld % 8 == 0 and lat 16-byte aligned); logits, the floor plans, d_lat (nv*64^3, 512) and d_logits stay fp32, with the
 *   same fixed orders (two calls are bit-identical).
 * neo_grid_encoder_lat_grad_bf16: d_lat (nv*64^3, 512) bf16 = bf16(d_pool + d_agg), both fp32 (nv*64^3, 512), inputs 16-byte and the
 *   output 8-byte aligned. */
int neo_grid_encoder_features_bf16(const float* latent_cl, int nv, int lat_h, int lat_w, int img_w, int img_h, const float* src_poses,
                                   float focal, float cx, float cy, void* X, int ldx, void* stream);
int neo_grid_encoder_coords_bf16(void* L, int nv, int ld, void* stream);
int neo_grid_encoder_pool_bf16(const void* lat, long long ld, const float* logits, int nv, float* floor_xz, float* floor_xy, float* floor_yz,
                               void* stream);
int neo_grid_encoder_pool_bwd_bf16(const void* lat, long long ld, const float* logits, int nv, const float* g_xz, const float* g_xy,
                                   const float* g_yz, float* d_lat, float* d_logits, void* stream);
int neo_grid_encoder_lat_grad_bf16(const float* d_pool, const float* d_agg, int nv, void* d_lat, void* stream);

/* ---- per-ray training losses and the encoder's upsampling adjoint, for training under torch.use_deterministic_algorithms (csrc/det.cu):
 * one warp per ray with fixed-order sums, every output written once, no floating-point atomics; two calls are bit-identical.  All return
 * NEO_ERR_INVALID before any launch on a NULL buffer they read or write or a size out of range. ---- */
/* training.distortion_loss per ray: loss[r] = 1/3 sum_i I_i w_i^2 + 2 sum_k (w_k m_k W_<k - w_k (wm)_<k), W_<k = sum_{i<k} w_i, exactly as
 * written (for descending m this is minus sum w_i w_j |m_i - m_j|, as the reference's eff_distloss gives).  w, m (n,N); interval (n,N) or
 * NULL = interval_scalar for every sample.  The caller takes the mean over rays. */
int neo_distortion_loss(const float* w, const float* m, const float* interval, float interval_scalar, int n, int N, float* loss, void* stream);
/* d_w (n,N) = g_loss[r] * d loss[r] / d w (m and interval carry no gradient). */
int neo_distortion_loss_bwd(const float* w, const float* m, const float* interval, float interval_scalar, int n, int N, const float* g_loss,
                            float* d_w, void* stream);
/* One proposal level of the Mip-NeRF 360 interlevel loss per ray (helper.py:117-141 lossfun_outer): sdist (n,Nc+1), weights (n,Nc) of the
 * NeRF level, sdist_env (n,Np+1), weights_env (n,Np) of the proposal level.  r_i = the number of sdist_env knots <= sdist_i (searchsorted
 * right=True), lo_i = max(r_i - 1, 0), hi_i = min(r_i, Np); w_outer_j = sum of weights_env over [lo_j, hi_{j+1}) in ascending order;
 * loss[r] = sum_j clip(w_j - w_outer_j, 0)^2 / (w_j + 1.1920929e-07) / Nc.  1 <= Nc <= 1024. */
int neo_interlevel_loss(const float* sdist, const float* weights, const float* sdist_env, const float* weights_env, int n, int Nc, int Np,
                        float* loss, void* stream);
/* d_weights_env (n,Np) = g_loss[r] * d loss[r] / d weights_env. */
int neo_interlevel_loss_bwd(const float* sdist, const float* weights, const float* sdist_env, const float* weights_env, int n, int Nc, int Np,
                            const float* g_loss, float* d_weights_env, void* stream);
/* Adjoint of F.interpolate(mode="bilinear", align_corners=True) on NCHW fp32: g_out (planes, H_out, W_out) -> g_in (planes, H_in, W_in),
 * every element written once as a gather over the output rows / columns whose taps reach it, with the tap weights of ATen's
 * upsample_bilinear2d forward (source index scale * o in fp32, scale = (in-1)/(out-1)). */
int neo_upsample_bilinear_bwd(const float* g_out, long long planes, int H_in, int W_in, int H_out, int W_out, float* g_in, void* stream);

/* bench support: CUDA events around every field-kernel launch on the launching stream + launch accounting.
 * neo_profile(1) resets and enables, neo_profile(0) resets and disables; neo_profile_read synchronises. */
int neo_profile(int enable);
int neo_profile_read(float* field_ms, int* n_field, unsigned long long* launches, double* points);

/* Stage-level entry point of the tensor-core dense layer used by the wide MLPs (csrc/gemm_tc.cu: 2-D TMA tile loads, wgmma with
 * register accumulators), on caller-owned fp16 operands with explicit row strides (in elements), as the library's own callers use it:
 * C (M,N; row stride ldc) = act(A (M,K; lda) . W (N,K; ldw)^T + bias) rounded to fp16; A, W, C fp16 device, bias (N) fp32 or NULL.
 * K % 64 == 0, N % 64 == 0, strides % 8 == 0, lda, ldw >= K, ldc >= N, 16-byte aligned pointers.  Writes only columns [0, N) of
 * rows [0, M) of C, so A may sit in other columns of C's own rows.  Asynchronous on `stream`. */
int neo_tc_gemm_f16(const void* A, long long lda, const void* W, long long ldw, const float* bias, void* C, long long ldc, long long M,
                    int N, int K, int relu, void* stream);
/* Stage-level entry point of the tiny-N head used by the vanilla NeRF, Mip-NeRF 360 and encoder tensor-core paths (csrc/gemm_tc.cu
 * rowdot_f16): out (M,N) fp32 = H (M,K; row stride ld) fp16 . W (N,K)^T fp32 + b (N) fp32, fp32 accumulation.  N in {1, 3},
 * K % 8 == 0, ld % 8 == 0, K <= ld, N*K*4 <= 48 KB, H 16-byte aligned, no NULL pointer; M <= 0 does nothing.  Writes only rows
 * [0, M) of out.  Asynchronous on `stream`. */
int neo_tc_rowdot_f16(const void* H, long long ld, int K, const float* W, const float* b, int N, long long M, float* out, void* stream);
/* Host-side view of the TC kernel's encoding-column layout (csrc/field_tc.cu enc_col<>): for in_ch = 3|4 and operand column
 * `col` in [0, KE = 64|96) returns the reference's positional-encoding index (helper.py:121-125 order) in [0, 21*in_ch),
 * -1 for the constant-one (bias) column, -2 for a zero padding column, -3 for invalid arguments.  Pure host code (no GPU). */
int neo_tc_enc_column(int in_ch, int col);

/* NEO_PREC_TC: the direction fragments of `rays` (exposed for tests; neo_render_fwd and neo_field_eval compute them before their field
 * launches).  For every ray r, the mean over the scene's source views of the direction encoding of viewdirs[r] in the view's camera
 * frame (model.py:357-360: [d, sin(2^k d), sin(2^k d + pi/2)], k < 4, 27 columns, then 5 zero columns), fp16, as the field kernel's
 * A fragments: out + 64 r + 16 t (t < 4) holds the fp16 pairs of columns {16 ks + 8 h + 2 t, + 1} in the order (ks, h) = (0,0),
 * (0,1), (1,0), (1,1).  out: n_rays * 64 bytes, 16-byte aligned. */
int neo_tc_dir_fragments(const NeoScene* scene, const NeoRays* rays, void* out, void* stream);

/* "" or a description of the mbarrier wait that timed out inside the NEO_PREC_TC field kernel (the kernel bounds its waits for the
 * weight copies and for the hand-off between its producer and consumer warpgroups, and traps instead of hanging; the barrier and the
 * waiter's identity are recorded in host-mapped memory, which survives the failed context). */
const char* neo_tc_trap_info(void);
const char* neo_last_error(void);
/* "neo360_b200 <version> sm_90a" */
const char* neo_version(void);

/* ---- NeO-360 training on the tensor cores (csrc/field_train.cu): layers 0-3 of one NeRFPPMLP in the projected formulation, bf16
 * operands, fp32 accumulation.  cam (nv*M, in_ch) camera-frame encoding points (row v M + j: point j in source view v); local_p,
 * world_p (nv*M, 256) looked-up projected rows [P0 | P3]; w0 (128, 21 in_ch) = pts_linears.0 encoding columns, w3 (128, 128 + 21 in_ch)
 * = pts_linears.3 [h | encoding] columns, w1 / w2 (128,128), biases (128), all fp32 nn.Linear layout.  hbar (M, 128) = the view mean of
 * h3.  Saved state: neo_field_train_workspace_bytes(..., 0) bytes written by the forward and read by the backward; the backward's
 * scratch: (..., 1) bytes (0 = invalid sizes).  Backward: g_hbar (M,128) -> d_pm (nv*M, 256), the row gradient of both local_p and
 * world_p, and every weight / bias gradient in the layout of the inputs (written, not accumulated).  NEO_ERR_INVALID before any launch
 * on a NULL buffer, nv outside 1..8, in_ch not 3 or 4, M <= 0, or a buffer not 16-byte aligned; NEO_ERR_WORKSPACE on a short
 * workspace.  No floating-point atomics: two calls are bit-identical. ---- */
size_t neo_field_train_workspace_bytes(int nv, int M, int in_ch, int which);
int neo_field_train_fwd(const float* cam, const float* local_p, const float* world_p, int nv, int M, int in_ch,
                        const float* w0, const float* b0, const float* w1, const float* b1, const float* w2, const float* b2,
                        const float* w3, const float* b3, float* hbar, void* saved, size_t saved_bytes, void* stream);
int neo_field_train_bwd(const float* g_hbar, int nv, int M, int in_ch, const float* w1, const float* w2, const float* w3,
                        const void* saved, size_t saved_bytes, float* d_pm, float* gw0, float* gb0, float* gw1, float* gb1,
                        float* gw2, float* gb2, float* gw3, float* gb3, void* scratch, size_t scratch_bytes, void* stream);

/* ---- PixelNeRF training on the tensor cores (csrc/field_train.cu, the PixelNeRF form of the kernels above): layers 0-3 of one
 * pixelnerf.NeRFMLP trunk in the projected formulation, bf16 operands, fp32 accumulation.  cam (nv*M, 3) camera-frame points (row v M + j:
 * point j in source view v, the frame of neo_pixelnerf_encode's first three enc columns); p0 (nv*M, 128) looked-up rows of
 * latent . W0[:, 63:575]^T, added to layer 0's pre-activation unrounded; w0 (128, 63) = pts_linears.0 encoding columns, w1 / w2 / w3
 * (128,128), biases (128), all fp32 nn.Linear layout.  Layer 3 has no skip: h3 = relu(w3 h2 + b3).  hbar (M, 128) = the view mean of
 * h3.  Saved state: neo_pixelnerf_train_workspace_bytes(nv, M, 0) bytes written by the forward and read by the backward; the backward's
 * scratch: (nv, M, 1) bytes (0 = invalid sizes).  Backward: g_hbar (M,128) -> d_p0 (nv*M, 128) and every weight / bias gradient in the
 * layout of the inputs (written, not accumulated).  NEO_ERR_INVALID before any launch on a NULL buffer, nv outside 1..8, M <= 0, more
 * than 2^25 rows (nv*M), or a p0 / hbar / g_hbar / d_p0 / workspace buffer not 16-byte aligned; NEO_ERR_WORKSPACE on a short workspace.
 * No floating-point atomics: two calls are bit-identical. ---- */
size_t neo_pixelnerf_train_workspace_bytes(int nv, int M, int which);
int neo_pixelnerf_train_fwd(const float* cam, const float* p0, int nv, int M, const float* w0, const float* b0, const float* w1,
                            const float* b1, const float* w2, const float* b2, const float* w3, const float* b3, float* hbar,
                            void* saved, size_t saved_bytes, void* stream);
int neo_pixelnerf_train_bwd(const float* g_hbar, int nv, int M, const float* w1, const float* w2, const float* w3, const void* saved,
                            size_t saved_bytes, float* d_p0, float* gw0, float* gb0, float* gw1, float* gb1, float* gw2, float* gb2,
                            float* gw3, float* gb3, void* scratch, size_t scratch_bytes, void* stream);

/* ---- Vanilla NeRF and Mip-NeRF 360 training on the tensor cores (csrc/dense_train.cu, csrc/gemm_tc.cu): the products of their dense
 * layers, bf16 operands (row-major, row strides in elements), fp32 accumulation, asynchronous on `stream`, no floating-point atomics.
 * Each returns NEO_ERR_INVALID before any launch on a NULL buffer it needs, a shape or stride outside its contract, or a misaligned
 * operand, with neo_last_error naming the entry point.
 * neo_tc_gemm_bf16: C (M,N; ldc) = A (M,K; lda) . W (N,K; ldw)^T + bias (N, fp32 or NULL), then epilogue 0 = ReLU -> bf16, 1 -> bf16,
 *   2 = no bias -> fp32.  Shape rules of neo_tc_gemm_f16 (K % 64, N % 64, strides % 8, 16-byte aligned); writes columns [0, N) of C only.
 * neo_tc_dgrad_bf16: dX (M,N; lddx) bf16 = (dY (M,K; ldy) . Wt (N,K; ldwt)^T + g_sig w_sig^T) [X > 0]: Wt = W^T of the layer's weight,
 *   X (M,N; ldx) its saved bf16 input (NULL: no mask), g_sig (M) and w_sig (N) fp32 or both NULL.  Shape rules of neo_tc_gemm_bf16.
 * neo_tc_wgrad_bf16: dW (N, k_valid) fp32 = dY (M,N; ldy)^T X (M,K; ldx), columns k >= k_valid dropped; db (N) = column sums of dY, or
 *   NULL.  N % 64, K % 64, N*K*4 <= 32 MB, strides % 8, 16-byte aligned dY, X and workspace; the workspace is
 *   neo_tc_wgrad_bf16_workspace_bytes(M, N, K) bytes (0 = invalid shape), NEO_ERR_WORKSPACE if short.  Written, not accumulated.
 * neo_tc_pack_bf16: bf16 copy of an fp32 (rows, cols_in; ld_in) matrix: transpose 0 -> out (rows, cols_out; ld_out), zero columns past
 *   cols_in; transpose 1 -> out (cols_out, rows; ld_out) = the first cols_out columns transposed.
 * neo_tc_relu_rank1_bf16: out (M,N; ldo) bf16 = (g (M) w (N)^T) [X (M,N; ldx) > 0], fp32 product rounded once.
 * neo_tc_rowdot_bf16: neo_tc_rowdot_f16 with a bf16 H (the density head over the last trunk activation). ---- */
int neo_tc_gemm_bf16(const void* A, long long lda, const void* W, long long ldw, const float* bias, void* C, long long ldc, long long M,
                     int N, int K, int epilogue, void* stream);
int neo_tc_dgrad_bf16(const void* dY, long long ldy, const void* Wt, long long ldwt, const void* X, long long ldx, const float* g_sig,
                      const float* w_sig, void* dX, long long lddx, long long M, int N, int K, void* stream);
size_t neo_tc_wgrad_bf16_workspace_bytes(long long M, int N, int K);
int neo_tc_wgrad_bf16(const void* dY, long long ldy, const void* X, long long ldx, long long M, int N, int K, float* dW, int k_valid,
                      float* db, void* workspace, size_t workspace_bytes, void* stream);
int neo_tc_pack_bf16(const float* in, long long rows, int cols_in, long long ld_in, void* out, int cols_out, long long ld_out, int transpose,
                     void* stream);
int neo_tc_relu_rank1_bf16(const float* g, const float* w, const void* X, long long ldx, long long M, int N, void* out, long long ldo,
                           void* stream);
int neo_tc_rowdot_bf16(const void* H, long long ld, int K, const float* W, const float* b, int N, long long M, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NEO360_B200_H */
